// The ResNet stem (default path; PSB200_STEM=im2col falls back) — 7x7 / stride 2 / pad 3 convolution, 3 → 64 channels — as
// ONE implicit-GEMM kernel on wgmma, replacing psb_im2col_stem (writes a 1.13 GB patch matrix at batch 256) + the GEMM that
// reads it back + the BatchNorm statistics pass over the 411 MB output.
//
// One tile = one output row (n, oh): OW <= 128 pixels x 64 channels, K = 176 (7 kernel rows x 24 columns — 21 real,
// 3 zero — + 8 zero columns: the layout of ops/stem.py, so the same [64,176] weight matrix is used).
//
//   warpgroup 0     builders   cp.async the 7 input rows of the NEXT tile into a zero-margined smem patch while building
//                              the CURRENT tile's A operand: thread m copies, for each kernel row, the 42 contiguous
//                              bytes x[n, 2oh-3+kh, 2m-3 .. 2m+3, 0..2] into the 128B-swizzled K-major wgmma layout
//                              (three [128 x 64] bf16 blocks; the same canonical layout TMA would have produced)
//   warpgroups 1-2  MMA +      64 pixel rows each: 11 x wgmma m64n64k16 per tile; the [64,176] weight operand is TMA-loaded
//                   epilogue   once per CTA.  Then bf16 → swizzled staging tile → ONE cp.async.bulk.tensor store per output row
//                              (NHWC: the row is 14 KB contiguous), and the per-channel Σy / Σy² of the staged bf16 values
//                              (exactly what psb_bn_stats would read back) accumulated in registers, summed in CTA order
#include "gemm_common.cuh"

namespace {

constexpr int SK = 176;                 // GEMM K (ops/stem.py STEM_K)
constexpr int S_THREADS = 384;          // builder + 2 MMA / epilogue warpgroups
constexpr int SA_BLK = 128 * 128;       // one k-block of A: 128 rows x 128 B
constexpr int SA_BYTES = 3 * SA_BLK;    // 48 KB per A buffer
constexpr int SB_BLK = 64 * 128;        // one k-block of B (64 output channels)
constexpr int SB_BYTES = 3 * SB_BLK;    // 24 KB
constexpr int SO_BYTES = 128 * 128;     // staging tile: 128 rows x 64 bf16
constexpr int MARGIN = 48;              // zero bytes left and right of a patch row (>= 18 needed, 16-byte multiple)
constexpr int MAX_W = 256;
constexpr int PATCH_PITCH_MAX = MARGIN + MAX_W * 6 + MARGIN;
constexpr int PATCH_BYTES = 7 * PATCH_PITCH_MAX;             // 11 424
constexpr int OFF_A = 0;
constexpr int OFF_B = OFF_A + 2 * SA_BYTES;                   // 98 304
constexpr int OFF_O = OFF_B + SB_BYTES;                       // 122 880 (1024-aligned)
constexpr int OFF_P = OFF_O + 2 * SO_BYTES;                   // 155 648
constexpr int OFF_BAR = OFF_P + 2 * PATCH_BYTES;              // 178 496
constexpr int STEM_SMEM = OFF_BAR + 256 + 1024;               // + barriers + alignment slack
static_assert(OFF_O % 1024 == 0 && OFF_B % 1024 == 0, "swizzled tiles must be 1024-byte aligned");
static_assert(STEM_SMEM <= 232448, "shared memory budget");

struct StemParams {
  const __nv_bfloat16* x;     // [N, H, W, 3] bf16 (channels-last, already normalised)
  float* sums;                // [gridDim.x][128]: this CTA's Σy[64] | Σy²[64] (summed in CTA order afterwards); nullable
  int N, H, W, OH, OW;
  // The broadcast gate (as in bcast_gemm*.cu): the weight matrix lives IN the symmetric parameter arena in the [64,176]
  // GEMM layout (layout.py custom placement) and the lane that TMA-loads it first acquires the PS's PARAMS_READY epoch, so
  // this kernel — the first consumer of parameters in a ResNet forward — is the req.Wait() of the broadcast
  // (/root/reference/mpi_comms.py:120-124) and workers queue no separate wait kernel.
  const uint64_t* ready_flag; // nullable
  uint64_t ready_epoch;
  uint64_t* err_slot;
  unsigned long long timeout_ns;
};

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void sts_v4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ uint32_t lds_u16(uint32_t addr) {
  uint16_t v;
  asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t lds_u32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}

// queue the 7 input rows of output row `tile` into `patch` (cp.async; rows outside the image are zero-filled)
__device__ __forceinline__ void load_patch(const StemParams& p, int tile, uint32_t patch, int pitch, int bt) {
  const int n = tile / p.OH, oh = tile - n * p.OH;
  const int chunks = p.W * 6 / 16;                                    // 16-byte pieces per input row
  for (int i = bt; i < 7 * chunks; i += 128) {
    const int kh = i / chunks, c = i - kh * chunks;
    const int ih = 2 * oh - 3 + kh;
    const uint32_t dst = patch + kh * pitch + MARGIN + c * 16;
    if (ih >= 0 && ih < p.H) {
      const uint8_t* src = reinterpret_cast<const uint8_t*>(p.x) + ((size_t)(n * p.H + ih) * p.W) * 6 + (size_t)c * 16;
      cp_async16(dst, src);
    } else {
      sts_v4(dst, 0u, 0u, 0u, 0u);
    }
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
}

// A-operand row `bt` (output pixel ow = bt) of one tile: for each kernel row the 42 contiguous patch bytes
// x[ih, 2ow-3 .. 2ow+3, 0..2] → three 16-byte chunks of the 128B-swizzled [128 x 64] k-blocks.  The same tile serves
// the forward (K-major A operand) and the weight gradient (MN-major operand: rows are then the reduction dimension).
__device__ __forceinline__ void build_row(uint32_t patch, uint32_t a_tile, int pitch, int bt) {
  const uint32_t prow = patch + 30 + 12 * bt;                               // MARGIN + (2*ow - 3) * 6 bytes
  const uint32_t arow = a_tile + (bt >> 3) * 1024 + (bt & 7) * 128;
#pragma unroll
  for (int kh = 0; kh < 7; ++kh) {
    const uint32_t q = prow + kh * pitch;              // 2-mod-4 aligned: one 2-byte and ten 4-byte loads
    const uint32_t first = lds_u16(q);
    uint32_t w4[10], v[12];
#pragma unroll
    for (int j = 0; j < 10; ++j) w4[j] = lds_u32(q + 2 + 4 * j);
    v[0] = first | (w4[0] << 16);
#pragma unroll
    for (int j = 1; j < 10; ++j) v[j] = (w4[j - 1] >> 16) | (w4[j] << 16);
    v[10] = w4[9] >> 16;
    v[11] = 0u;
#pragma unroll
    for (int c3 = 0; c3 < 3; ++c3) {
      const int qc = kh * 3 + c3;                      // 16-byte chunk index within the 352-byte logical row
      sts_v4(arow + (qc >> 3) * SA_BLK + (((qc & 7) ^ (bt & 7)) << 4), v[4 * c3], v[4 * c3 + 1], v[4 * c3 + 2],
             v[4 * c3 + 3]);
    }
  }
  // chunk 21 (columns 168..175) stays zero from the initial clear
}

__global__ void __launch_bounds__(S_THREADS, 1)
psb_stem_fwd_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_y,
                    const __grid_constant__ StemParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
  uint64_t* b_full = bars;            // [1]  weights landed
  uint64_t* a_full = bars + 1;        // [2]  4 builder warps arrive
  uint64_t* a_empty = bars + 3;       // [2]  the wgmmas of both MMA warpgroups that read A[buf] have retired

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles = p.N * p.OH;
  const int per = (tiles + gridDim.x - 1) / gridDim.x;
  const int t0 = blockIdx.x * per, t1 = min(t0 + per, tiles);
  const int pitch = MARGIN + p.W * 6 + MARGIN;
  const uint32_t sA = smem_u32(smem + OFF_A), sB = smem_u32(smem + OFF_B), sO = smem_u32(smem + OFF_O),
                 sP = smem_u32(smem + OFF_P);

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_w) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_y) : "memory");
    mbar_init(b_full, 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&a_full[i], 4);
      mbar_init(&a_empty[i], 2);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // zero both A buffers (rows >= OW and the K padding are never written again) and the patch margins
  for (int i = threadIdx.x; i < (2 * SA_BYTES) / 16; i += S_THREADS) sts_v4(sA + i * 16, 0u, 0u, 0u, 0u);
  for (int i = threadIdx.x; i < (2 * PATCH_BYTES) / 16; i += S_THREADS) sts_v4(sP + i * 16, 0u, 0u, 0u, 0u);
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // the zero rows / columns of A are read by the tensor core
  __syncthreads();

  if (warp < 4) {
    // ============================== builders ==============================
    const int bt = threadIdx.x;                        // 0..127 == the A row (output pixel ow) this thread fills
    if (t0 < t1) load_patch(p, t0, sP, pitch, bt);
    for (int t = t0, i = 0; t < t1; ++t, ++i) {
      const int buf = i & 1;
      if (t + 1 < t1) {
        load_patch(p, t + 1, sP + (buf ^ 1) * PATCH_BYTES, pitch, bt);      // patch[buf^1]: last read one tile ago (barrier below)
        asm volatile("cp.async.wait_group 1;" ::: "memory");
      } else {
        asm volatile("cp.async.wait_group 0;" ::: "memory");
      }
      named_bar(1, 128);                               // everybody's copies of patch[buf] have landed
      mbar_wait(&a_empty[buf], ((i >> 1) & 1) ^ 1);    // the MMAs that read A[buf] two tiles ago are done
      if (bt < p.OW) build_row(sP + buf * PATCH_BYTES, sA + buf * SA_BYTES, pitch, bt);
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");          // generic writes → visible to the tensor core
      __syncwarp();
      if (lane == 0) mbar_arrive(&a_full[buf]);
      named_bar(1, 128);                               // everybody finished READING patch[buf] (refilled during the next tile)
    }
  } else {
    // ============================== MMA + epilogue ==============================
    const int et = threadIdx.x - 128;                  // 0..255
    const int c = et >> 7, wt = et & 127;              // warpgroup c owns pixel rows c*64 .. c*64+63 of the tile
    const int frow = c * 64 + (wt >> 5) * 16 + ((lane) >> 2), fcol = 2 * (lane & 3);   // fragment origin (wgmma_m64n64)
    if (et == 0) {
      if (p.ready_flag != nullptr) {       // patch loads / A-tile builds of the first tiles already run in the builders
        psb::spin_until_ge(p.ready_flag, p.ready_epoch, p.err_slot, p.timeout_ns);
        asm volatile("fence.proxy.async;" ::: "memory");   // generic-proxy acquire → async-proxy (TMA) reads
      }
      mbar_expect_tx(b_full, SB_BYTES);
      for (int b = 0; b < 3; ++b) tma_load_2d(&tmap_w, b_full, smem + OFF_B + b * SB_BLK, b * 64, 0);
    }
    mbar_wait(b_full, 0);
    const int ch = et & 63, part = et >> 6;            // column sums: channel ch over a quarter of the rows
    const int rq = (p.OW + 3) >> 2;
    const int r0 = part * rq, r1 = min(p.OW, r0 + rq);
    float s_sum = 0.f, s_sq = 0.f;
    float acc[32];
    for (int t = t0, i = 0; t < t1; ++t, ++i) {
      const int buf = i & 1;
      mbar_wait(&a_full[buf], (i >> 1) & 1);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < SK / WG_K; ++kk) {
        const uint64_t da = make_desc(sA + buf * SA_BYTES + (kk >> 2) * SA_BLK + c * 64 * 128 + 32 * (kk & 3));
        const uint64_t db = make_desc(sB + (kk >> 2) * SB_BLK + 32 * (kk & 3));
        wgmma_m64n64<0, 0>(acc, da, db, kk != 0);
      }
      wgmma_commit();
      wgmma_wait<0>();
      if (wt == 0) mbar_arrive(&a_empty[buf]);         // A[buf] may be rebuilt for tile i+2

      // staging buffer `buf`: the bulk store issued from it two tiles ago must have finished reading it
      if (et == 0) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
      named_bar(2, 256);
      const uint32_t so = sO + buf * SO_BYTES;
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = frow + 8 * h;
          asm volatile("st.shared.u32 [%0], %1;" ::"r"(so + r * 128 + ((j ^ (r & 7)) << 4) + fcol * 2),
                       "r"(psb::pack_bf16x2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]))
                       : "memory");
        }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      named_bar(2, 256);
      if (et == 0) {
        tma_store_2d(&tmap_y, so, 0, t * p.OW);
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      }
      if (p.sums != nullptr) {
        // column sums of the bf16 values just staged (what a separate statistics pass would read back)
        const uint32_t cbase = so + (ch & 7) * 2;
        for (int rr = r0; rr < r1; ++rr) {
          const float v = __uint_as_float(lds_u16(cbase + rr * 128 + (((ch >> 3) ^ (rr & 7)) << 4)) << 16);
          s_sum += v;
          s_sq = fmaf(v, v, s_sq);
        }
      }
    }
    if (p.sums != nullptr) {        // the four row quarters of each channel, added in a fixed order: no float atomics
      __shared__ float red[2][4][64];
      red[0][part][ch] = s_sum;
      red[1][part][ch] = s_sq;
      named_bar(2, 256);
      if (et < 128) {
        const float* r = red[et >> 6][0] + ch;
        p.sums[(size_t)blockIdx.x * 128 + et] = ((r[0] + r[64]) + r[128]) + r[192];
      }
    }
    if (et == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  }
}

// ==========================================================================================================
// Weight gradient of the stem, implicit too:  dW2d[co][k] = Σ_pixels gy[p][co] · A[p][k].
// The reduction runs over PIXELS, so both operands are MN-major for the tensor core — which is exactly how they already sit
// in shared memory: the im2col tile built by build_row ([pixel rows][k], k contiguous) is the M-side operand, the TMA-loaded
// gy tile ([pixel rows][64 channels]) the N-side one.  Three wgmma m64n64k16 per 16 pixels cover k-blocks 0, 1, 2
// (k = 0..191; k >= 176 is zero).  The accumulators stay in registers for the CTA's whole life; each CTA writes one fp32
// partial [176][64] and the host sums the partials (deterministic, 132 x 45 KB).
//   warpgroup 0  builders (as in the forward); thread 0 also TMA-loads the gy tile of the buffer it fills
//   warpgroup 1  MMA issuer, then the final register → global epilogue
// ==========================================================================================================
constexpr int WG_THREADS = 256;
constexpr int SG_BYTES = 128 * 128;                              // gy tile: up to 128 pixel rows x 64 bf16
constexpr int WOFF_A = 0;
constexpr int WOFF_G = WOFF_A + 2 * SA_BYTES;                    // 98 304
constexpr int WOFF_P = WOFF_G + 2 * SG_BYTES;                    // 131 072
constexpr int WOFF_BAR = WOFF_P + 2 * PATCH_BYTES;
constexpr int WGRAD_SMEM = WOFF_BAR + 256 + 1024;
static_assert(WOFF_G % 1024 == 0, "swizzled tiles must be 1024-byte aligned");
static_assert(WGRAD_SMEM <= 232448, "shared memory budget");

struct StemWgradParams {
  const __nv_bfloat16* x;     // [N, H, W, 3] bf16
  float* partial;             // [gridDim.x][176][64] fp32
  int N, H, W, OH, OW;
};

__global__ void __launch_bounds__(WG_THREADS, 1)
psb_stem_wgrad_kernel(const __grid_constant__ CUtensorMap tmap_g, const __grid_constant__ StemWgradParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + WOFF_BAR);
  uint64_t* a_full = bars;            // [2]  4 builder warps arrive
  uint64_t* g_full = bars + 2;        // [2]  TMA bytes of the gy tile
  uint64_t* empty = bars + 4;         // [2]  the wgmmas that read A[buf] and G[buf] have retired

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles = p.N * p.OH;
  const int per = (tiles + gridDim.x - 1) / gridDim.x;
  const int t0 = blockIdx.x * per, t1 = min(t0 + per, tiles);
  const int pitch = MARGIN + p.W * 6 + MARGIN;
  const uint32_t sA = smem_u32(smem + WOFF_A), sG = smem_u32(smem + WOFF_G), sP = smem_u32(smem + WOFF_P);

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_g) : "memory");
    for (int i = 0; i < 2; ++i) {
      mbar_init(&a_full[i], 4);
      mbar_init(&g_full[i], 1);
      mbar_init(&empty[i], 1);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // rows >= OW of A and of the gy tiles take part in the last K step: they must be zero, not stale bits
  for (int i = threadIdx.x; i < (2 * SA_BYTES + 2 * SG_BYTES) / 16; i += WG_THREADS) sts_v4(sA + i * 16, 0u, 0u, 0u, 0u);
  for (int i = threadIdx.x; i < (2 * PATCH_BYTES) / 16; i += WG_THREADS) sts_v4(sP + i * 16, 0u, 0u, 0u, 0u);
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  StemParams lp{};                                     // load_patch only reads x / H / W / OH
  lp.x = p.x, lp.N = p.N, lp.H = p.H, lp.W = p.W, lp.OH = p.OH, lp.OW = p.OW;

  if (warp < 4) {
    // ============================== builders ==============================
    const int bt = threadIdx.x;
    if (t0 < t1) load_patch(lp, t0, sP, pitch, bt);
    for (int t = t0, i = 0; t < t1; ++t, ++i) {
      const int buf = i & 1;
      if (t + 1 < t1) {
        load_patch(lp, t + 1, sP + (buf ^ 1) * PATCH_BYTES, pitch, bt);
        asm volatile("cp.async.wait_group 1;" ::: "memory");
      } else {
        asm volatile("cp.async.wait_group 0;" ::: "memory");
      }
      named_bar(1, 128);
      mbar_wait(&empty[buf], ((i >> 1) & 1) ^ 1);
      if (bt == 0) {
        mbar_expect_tx(&g_full[buf], (uint32_t)p.OW * 128u);
        tma_load_2d(&tmap_g, &g_full[buf], smem + WOFF_G + buf * SG_BYTES, 0, t * p.OW);
      }
      if (bt < p.OW) build_row(sP + buf * PATCH_BYTES, sA + buf * SA_BYTES, pitch, bt);
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncwarp();
      if (lane == 0) mbar_arrive(&a_full[buf]);
      named_bar(1, 128);
    }
  } else {
    // ============================== MMA, then this CTA's partial dW2d^T [176][64] ==============================
    const int wt = threadIdx.x - 128;
    const int frow = (wt >> 5) * 16 + (lane >> 2), fcol = 2 * (lane & 3);   // fragment origin (wgmma_m64n64)
    const int ksteps = (p.OW + 15) >> 4;               // 16 pixel rows per wgmma K step (rows >= OW are zero)
    float acc[3][32];
    for (int t = t0, i = 0; t < t1; ++t, ++i) {
      const int buf = i & 1;
      const uint32_t par = (i >> 1) & 1;
      mbar_wait(&a_full[buf], par);
      mbar_wait(&g_full[buf], par);
      wgmma_fence();
#pragma unroll 1
      for (int ks = 0; ks < ksteps; ++ks) {
        const uint64_t dg = make_desc(sG + buf * SG_BYTES + ks * 2048, SG_BYTES);
#pragma unroll
        for (int b = 0; b < 3; ++b)                    // k-block b → k = 64b .. 64b+63
          wgmma_m64n64<1, 1>(acc[b], make_desc(sA + buf * SA_BYTES + b * SA_BLK + ks * 2048, SA_BLK), dg, (i | ks) != 0);
      }
      wgmma_commit();
      wgmma_wait<0>();
      if (wt == 0) mbar_arrive(&empty[buf]);
    }
    float* out = p.partial + (size_t)blockIdx.x * SK * 64;
#pragma unroll
    for (int b = 0; b < 3; ++b)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int k = 64 * b + frow + 8 * h;
        if (k < SK) {
#pragma unroll
          for (int j = 0; j < 8; ++j)
            *reinterpret_cast<float2*>(out + (size_t)k * 64 + 8 * j + fcol) =
                t0 < t1 ? make_float2(acc[b][4 * j + 2 * h], acc[b][4 * j + 2 * h + 1]) : make_float2(0.f, 0.f);
        }
      }
  }
}

// dW2d[co][k] = Σ_cta partial[cta][k][co]  (fp32 sum in CTA order → deterministic), cast to bf16.
// Thread t handles (k = t / 64, co = t % 64): the reads of one warp are 128 contiguous bytes of each partial.
__global__ void __launch_bounds__(256) psb_stem_wgrad_finalize_kernel(const float* __restrict__ partial, int grid,
                                                                      __nv_bfloat16* __restrict__ out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= SK * 64) return;
  const int k = t >> 6, co = t & 63;
  float acc = 0.f;
  int g = 0;
  for (; g + 4 <= grid; g += 4) {
    const float a0 = partial[(size_t)(g + 0) * SK * 64 + t], a1 = partial[(size_t)(g + 1) * SK * 64 + t],
                a2 = partial[(size_t)(g + 2) * SK * 64 + t], a3 = partial[(size_t)(g + 3) * SK * 64 + t];
    acc += a0;
    acc += a1;
    acc += a2;
    acc += a3;
  }
  for (; g < grid; ++g) acc += partial[(size_t)g * SK * 64 + t];
  out[co * SK + k] = __float2bfloat16_rn(acc);
}

}  // namespace

void psb_stem_wgrad_finalize_launch(cudaStream_t s, const float* partial, int grid, void* out_bf16) {
  psb_count_launch(1);
  psb_stem_wgrad_finalize_kernel<<<(SK * 64 + 255) / 256, 256, 0, s>>>(partial, grid, reinterpret_cast<__nv_bfloat16*>(out_bf16));
}

namespace {
// sums[j] = Σ_cta part[cta][j] in CTA order (deterministic), j < 128
__global__ void __launch_bounds__(128) psb_stem_sums_kernel(const float* __restrict__ part, int grid, float* __restrict__ sums) {
  float acc = 0.f;
  for (int g = 0; g < grid; ++g) acc += part[(size_t)g * 128 + threadIdx.x];
  sums[threadIdx.x] = acc;
}

}  // namespace

int psb_stem_fwd_smem_bytes() { return STEM_SMEM; }

// tmap_w: [64,176] bf16 weights, box 64 x 64, SWIZZLE_128B.  tmap_y: [N*OH*OW, 64] bf16 output, box 64 columns x OW rows,
// SWIZZLE_128B.  `sums` (nullable): 128 floats, Σy | Σy² per channel; `part`: num_sms x 128 floats of per-CTA partials.
void psb_stem_fwd_launch(cudaStream_t s, const void* tmap_w, const void* tmap_y, const void* x, float* sums, float* part, int N,
                         int H, int W,
                         int num_sms, const uint64_t* ready_flag, uint64_t ready_epoch, unsigned long long timeout_ns) {
  static bool configured = false;
  if (!configured) {
    cudaFuncSetAttribute(psb_stem_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, STEM_SMEM);
    configured = true;
  }
  StemParams p{};
  p.x = reinterpret_cast<const __nv_bfloat16*>(x);
  p.sums = sums != nullptr ? part : nullptr;
  p.N = N, p.H = H, p.W = W;
  p.OH = (H - 1) / 2 + 1, p.OW = (W - 1) / 2 + 1;
  p.ready_flag = ready_flag;
  p.ready_epoch = ready_epoch;
  p.err_slot = ready_flag != nullptr ? const_cast<uint64_t*>(ready_flag) - SIG_PARAMS_READY + SIG_ERROR : nullptr;
  p.timeout_ns = timeout_ns;
  const int tiles = N * p.OH;
  const int grid = tiles < num_sms ? tiles : num_sms;
  psb_count_launch(1);
  psb_stem_fwd_kernel<<<grid, S_THREADS, STEM_SMEM, s>>>(*reinterpret_cast<const CUtensorMap*>(tmap_w),
                                                        *reinterpret_cast<const CUtensorMap*>(tmap_y), p);
  if (sums != nullptr) {
    psb_count_launch(1);
    psb_stem_sums_kernel<<<1, 128, 0, s>>>(part, grid, sums);
  }
}

// tmap_g: [N*OH*OW, 64] bf16 output gradient (channels-last), box 64 columns x OW rows, SWIZZLE_128B.
// `partial`: [grid][176][64] fp32, fully written (no zeroing needed).
int psb_stem_wgrad_grid(int N, int H, int num_sms) {
  const int tiles = N * ((H - 1) / 2 + 1);
  return tiles < num_sms ? tiles : num_sms;
}
void psb_stem_wgrad_launch(cudaStream_t s, const void* tmap_g, const void* x, float* partial, int N, int H, int W, int num_sms) {
  static bool configured = false;
  if (!configured) {
    cudaFuncSetAttribute(psb_stem_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, WGRAD_SMEM);
    configured = true;
  }
  StemWgradParams p{};
  p.x = reinterpret_cast<const __nv_bfloat16*>(x);
  p.partial = partial;
  p.N = N, p.H = H, p.W = W;
  p.OH = (H - 1) / 2 + 1, p.OW = (W - 1) / 2 + 1;
  psb_count_launch(1);
  psb_stem_wgrad_kernel<<<psb_stem_wgrad_grid(N, H, num_sms), WG_THREADS, WGRAD_SMEM, s>>>(
      *reinterpret_cast<const CUtensorMap*>(tmap_g), p);
}
