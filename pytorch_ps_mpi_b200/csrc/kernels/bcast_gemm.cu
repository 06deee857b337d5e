// bcast_gemm: Y[M,N] = act(X[M,K] · W[N,K]^T + bias) in bf16 with fp32 accumulation on the Hopper tensor cores
// (wgmma.mma_async, accumulators in registers, operands staged by TMA into 128B-swizzled shared memory), whose WEIGHT
// operand is the tile the parameter server just broadcast.
//
// The weight tensor map points INTO the symmetric parameter arena (the Ibcast + Wait + first forward matmul of the
// reference's mpi_comms.py, K4 in SURVEY §2.6): the TMA producer acquires the PARAMS_READY epoch flag (ld.acquire.sys +
// fence.proxy.async) right before its first weight load, so this GEMM *is* the req.Wait() of the forward pass.
//
// Structure (one CTA per SM, persistent over output tiles; a CTA computes 128 x BN, BN = 64 or 128):
//   warpgroup 0      TMA producer   one thread: cp.async.bulk.tensor.2d → smem ring of {A 128x64, B BNx64} stages
//   warpgroups 1, 2  consumers      64 rows each: 4 x wgmma m64nBNk16 per stage (one wgmma group kept in flight, the stage
//                                   before it released), then the epilogue straight from the accumulator registers
// CL = 2 (a cluster of two CTAs on 256 x BN tiles): each CTA TMA-loads its own 128 rows of A and HALF of the B tile, and
// multicasts that half into both CTAs, so each weight byte is fetched from L2 once per pair.  A stage is then refilled by
// two producers, so the consumers of each CTA release it in both CTAs (remote mbarrier arrive).
//
// Epilogues (template EPI; fragment → +bias → ReLU → bf16):
//   EPI 3  (default when N % 8 == 0)  TMA store: each consumer warpgroup packs its 64 rows into 128B-swizzled 64-column
//          staging tiles and one thread issues cp.async.bulk.tensor.2d.global.shared::cta; bounds are clipped by the TMA unit.
//   EPI 1  (default otherwise)  staged: the warpgroup's rows go through padded shared memory and leave as full 16-byte
//          row-contiguous stores; handles any N.
//   EPI 0  direct 4-byte stores from the accumulator fragment (the A/B baseline of the two above).
#include "gemm_common.cuh"

namespace {

constexpr int BM = 128;
constexpr int THREADS = 384;

template <int BN, int EPI>
struct Cfg {
  static constexpr int A_BYTES = BM * BK * 2;                            // 16 KB
  static constexpr int B_BYTES = BN * BK * 2;                            // 8 / 16 KB
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = BN == 128 ? 5 : 7;
  static constexpr int BAR_BYTES = 1024;                                 // keeps the staging area 1024-byte aligned (swizzle)
  static constexpr int PITCH = BN * 2 + 16;                              // EPI 1: padded row, conflict-free both ways
  static constexpr int WG_STAGING = EPI == 3 ? 64 * BN * 2 : (EPI == 1 ? 64 * PITCH : 0);
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align slack*/ + BAR_BYTES + 2 * WG_STAGING;
  static_assert(SMEM_BYTES <= 232448, "exceeds the 227 KB of shared memory a CTA may opt into");
};

__device__ __forceinline__ void st_shared_u32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
__device__ __forceinline__ uint4 ld_shared_v4(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr) : "memory");
  return v;
}

template <int BN, int CL, int EPI>
__global__ void __launch_bounds__(THREADS, 1)
psb_bcast_gemm_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                      const __grid_constant__ CUtensorMap tmap_c, const __grid_constant__ GemmParams p) {
  using C = Cfg<BN, EPI>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + C::STAGES * C::STAGE_BYTES);   // [STAGES]
  uint64_t* empty = full + C::STAGES;                                                // [STAGES]
  uint8_t* staging = smem + C::STAGES * C::STAGE_BYTES + C::BAR_BYTES;

  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const uint32_t cta = CL == 2 ? cluster_ctarank() : 0;
  const int ncl = gridDim.x / CL, cl = blockIdx.x / CL;
  const int tiles_m = (p.M + BM * CL - 1) / (BM * CL), tiles_n = (p.N + BN - 1) / BN;
  const int num_tiles = tiles_m * tiles_n;
  const int num_kb = (p.K + BK - 1) / BK;

  if (threadIdx.x == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_a) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_b) : "memory");
    if constexpr (EPI == 3) asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap_c) : "memory");
    for (int i = 0; i < C::STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 2 * CL);        // one arrival per consumer warpgroup of every CTA that fills this stage
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if constexpr (CL == 2) cluster_sync_all();   // the peer's barriers exist before anything is multicast into / arrives on them
  else __syncthreads();

  if (wg == 0) {
    // ===================== TMA producer =====================
    if (t == 0) {
      // The broadcast gate: do not touch a weight tile before the server published this epoch.
      if (p.ready_flag != nullptr) {
        psb::spin_until_ge(p.ready_flag, p.ready_epoch, p.err_slot, p.timeout_ns);
        asm volatile("fence.proxy.async;" ::: "memory");   // generic-proxy acquire → async-proxy (TMA) reads
      }
      uint32_t stage = 0, phase = 0;
      for (int tile = cl; tile < num_tiles; tile += ncl) {
        const int m0 = (tile / tiles_n) * BM * CL + (int)cta * BM, n0 = (tile % tiles_n) * BN;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1);
          uint8_t* sa = smem + stage * C::STAGE_BYTES;
          mbar_expect_tx(&full[stage], C::STAGE_BYTES);
          tma_load_2d(&tmap_a, &full[stage], sa, kb * BK, m0);
          if constexpr (CL == 1) {
            tma_load_2d(&tmap_b, &full[stage], sa + C::A_BYTES, kb * BK, n0);
          } else {
            tma_load_2d_mc(&tmap_b, &full[stage], sa + C::A_BYTES + cta * (BN / 2) * 128, kb * BK, n0 + (int)cta * (BN / 2),
                           (uint16_t)3);
          }
          if (++stage == C::STAGES) stage = 0, phase ^= 1;
        }
      }
    }
  } else {
    // ===================== consumers: wgmma + epilogue =====================
    const int c = wg - 1;                                  // rows c*64 .. c*64+63 of the CTA's 128
    const int warp = t >> 5, lane = t & 31;
    const int frow = warp * 16 + (lane >> 2), fcol = 2 * (lane & 3);   // fragment origin (see wgmma_m64n64)
    const bool vec_ok = (p.N % 8) == 0;
    const uint32_t stg = smem_u32(staging + c * C::WG_STAGING);
    auto release = [&](uint32_t s) {
      if constexpr (CL == 1) {
        if (t == 0) mbar_arrive(&empty[s]);
      } else {
        if (t < 2) mbar_arrive_cluster(&empty[s], (uint32_t)t);     // both CTAs' producers refill this stage
      }
    };
    float acc[BN / 2];
    uint32_t stage = 0, phase = 0;
    for (int tile = cl; tile < num_tiles; tile += ncl) {
      const int m0 = (tile / tiles_n) * BM * CL + (int)cta * BM + c * 64, n0 = (tile % tiles_n) * BN;
      uint32_t prev = 0;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full[stage], phase);
        const uint32_t sa = smem_u32(smem + stage * C::STAGE_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / WG_K; ++k)
          wgmma_tile<BN>(acc, make_desc(sa + c * 64 * 128 + 32 * k), make_desc(sa + C::A_BYTES + 32 * k), (kb | k) != 0);
        wgmma_commit();
        wgmma_wait<1>();                                   // the previous stage's wgmmas have retired: its slot is free
        if (kb > 0) release(prev);
        prev = stage;
        if (++stage == C::STAGES) stage = 0, phase ^= 1;
      }
      wgmma_wait<0>();
      release(prev);

      auto value = [&](int i, int col) {                  // accumulator i (at column col) → +bias → ReLU
        float v = acc[i];
        if (p.bias != nullptr && col < p.N) v += p.bias[col];
        // ReLU as F.relu: NaN stays NaN.  fmaxf would return the 0; max.NaN returns NaN when an operand is NaN by the
        // instruction's definition, so no math-mode flag can drop it, and it keeps every instantiation's register count.
        if (p.relu) asm("max.NaN.f32 %0, %0, 0f00000000;" : "+f"(v));
        return v;
      };
      if constexpr (EPI == 0) {
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int col = n0 + 8 * j + fcol;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = m0 + frow + 8 * h;
            const float a = value(4 * j + 2 * h, col), b = value(4 * j + 2 * h + 1, col + 1);
            if (row < p.M && col < p.N) {
              __nv_bfloat16* o = p.out + (size_t)row * p.N + col;
              if ((p.N % 2) == 0) *reinterpret_cast<uint32_t*>(o) = psb::pack_bf16x2(a, b);
              else {
                o[0] = __float2bfloat16_rn(a);
                if (col + 1 < p.N) o[1] = __float2bfloat16_rn(b);
              }
            }
          }
        }
      } else if constexpr (EPI == 1) {
        named_bar(1 + c, 128);                             // the previous tile's rows have left the staging buffer
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int col = n0 + 8 * j + fcol;
#pragma unroll
          for (int h = 0; h < 2; ++h)
            st_shared_u32(stg + (frow + 8 * h) * C::PITCH + (8 * j + fcol) * 2,
                          psb::pack_bf16x2(value(4 * j + 2 * h, col), value(4 * j + 2 * h + 1, col + 1)));
        }
        named_bar(1 + c, 128);
        constexpr int CHUNKS = BN / 8, ROWS_PER_PASS = 128 / CHUNKS;          // 16-byte pieces per row
        const int ch = t % CHUNKS;
#pragma unroll 1
        for (int r = t / CHUNKS; r < 64; r += ROWS_PER_PASS) {
          const int grow = m0 + r, gcol = n0 + ch * 8;
          if (grow >= p.M || gcol >= p.N) continue;
          const uint4 v = ld_shared_v4(stg + r * C::PITCH + ch * 16);
          __nv_bfloat16* o = p.out + (size_t)grow * p.N + gcol;
          if (vec_ok && gcol + 8 <= p.N) {
            *reinterpret_cast<uint4*>(o) = v;
          } else {
            const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int e = 0; e < 8; ++e)
              if (gcol + e < p.N) reinterpret_cast<uint16_t*>(o)[e] = (uint16_t)(w[e >> 1] >> ((e & 1) * 16));
          }
        }
      } else {
        // the bulk stores issued from this buffer for the previous tile have finished READING it
        if (t == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
        named_bar(1 + c, 128);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int col = n0 + 8 * j + fcol, q = j >> 3;   // 64-column staging tile q; 16-byte chunk (j & 7) ^ (row & 7)
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int r = frow + 8 * h;
            st_shared_u32(stg + q * 8192 + r * 128 + (((j & 7) ^ (r & 7)) << 4) + fcol * 2,
                          psb::pack_bf16x2(value(4 * j + 2 * h, col), value(4 * j + 2 * h + 1, col + 1)));
          }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // generic-proxy writes → visible to the TMA unit
        named_bar(1 + c, 128);
        if (t == 0) {
#pragma unroll
          for (int q = 0; q < BN / 64; ++q)
#pragma unroll
            for (int h = 0; h < 2; ++h)                    // the output map's box is 64 columns x 32 rows
              if (n0 + q * 64 < p.N && m0 + h * 32 < p.M) tma_store_2d(&tmap_c, stg + q * 8192 + h * 4096, n0 + q * 64, m0 + h * 32);
          asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
      }
    }
    if constexpr (EPI == 3) {
      if (t == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");   // all output tiles written before exit
    }
  }
  // no CTA of a pair exits while its peer may still multicast into its shared memory or arrive on its barriers
  if constexpr (CL == 2) cluster_sync_all();
}

template <int BN, int CL, int EPI>
void launch(cudaStream_t s, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc, const GemmParams& p, int grid) {
  using C = Cfg<BN, EPI>;
  static bool configured = false;
  if (!configured) {
    cudaFuncSetAttribute(psb_bcast_gemm_kernel<BN, CL, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
    configured = true;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(THREADS);
  cfg.dynamicSmemBytes = C::SMEM_BYTES;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CL;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  cudaLaunchKernelEx(&cfg, psb_bcast_gemm_kernel<BN, CL, EPI>, ta, tb, tc, p);
}

template <int BN, int CL>
void launch_e(cudaStream_t s, int epi, const CUtensorMap& ta, const CUtensorMap& tb, const CUtensorMap& tc, const GemmParams& p,
              int grid) {
  if (epi == 3) launch<BN, CL, 3>(s, ta, tb, tc, p, grid);
  else if (epi == 1) launch<BN, CL, 1>(s, ta, tb, tc, p, grid);
  else launch<BN, CL, 0>(s, ta, tb, tc, p, grid);
}

}  // namespace

int psb_bcast_gemm_bn(int N) { return N <= 64 ? 64 : 128; }

int psb_bcast_gemm_smem_bytes() { return Cfg<128, 3>::SMEM_BYTES; }

void psb_launch_bcast_gemm(cudaStream_t s, const BcastGemmArgs& a, int num_sms, int epi) {
  if (epi < 0) epi = (a.tmap_out != nullptr && a.N % 8 == 0) ? 3 : 1;
  GemmParams p{};
  p.bias = a.bias;
  p.out = reinterpret_cast<__nv_bfloat16*>(const_cast<void*>(a.tmap_c));   // tmap_c carries the output pointer
  p.ready_flag = a.ready_flag;
  p.ready_epoch = a.ready_epoch;
  p.err_slot = a.ready_flag != nullptr ? const_cast<uint64_t*>(a.ready_flag) - SIG_PARAMS_READY + SIG_ERROR : nullptr;
  p.M = a.M, p.N = a.N, p.K = a.K, p.relu = a.relu;
  p.timeout_ns = a.timeout_ns;
  psb_count_launch(1);
  const int bn = psb_bcast_gemm_bn(a.N), cl = a.two_cta ? 2 : 1;
  const int tiles = ((a.M + BM * cl - 1) / (BM * cl)) * ((a.N + bn - 1) / bn);
  int clusters = num_sms / cl;
  if (tiles < clusters) clusters = tiles;
  const CUtensorMap& ta = *reinterpret_cast<const CUtensorMap*>(a.tmap_a);
  const CUtensorMap& tb = *reinterpret_cast<const CUtensorMap*>(a.tmap_b);
  const CUtensorMap& tc = a.tmap_out != nullptr ? *reinterpret_cast<const CUtensorMap*>(a.tmap_out) : ta;   // unused unless EPI 3
  if (bn == 64) {
    if (cl == 2) launch_e<64, 2>(s, epi, ta, tb, tc, p, 2 * clusters);
    else launch_e<64, 1>(s, epi, ta, tb, tc, p, clusters);
  } else {
    if (cl == 2) launch_e<128, 2>(s, epi, ta, tb, tc, p, 2 * clusters);
    else launch_e<128, 1>(s, epi, ta, tb, tc, p, clusters);
  }
}
