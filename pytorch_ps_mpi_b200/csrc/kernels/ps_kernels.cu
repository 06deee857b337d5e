// Parameter-server hot path for sm_90a: gradient encode, fused gather-reduce-decode-update-
// broadcast, and the epoch-flag signalling kernels.
//
// What these replace in the reference (citations into /root/reference):
//   * encode + to_np + pickle + blosc per parameter on a thread pool (ps.py:92-101,
//     mpi_comms.py:186-193)                         → psb_encode_kernel (one launch per bucket)
//   * Igatherv / Iallgatherv of host bytes (mpi_comms.py:88,162), H2D copies (mpi_comms.py:48-50),
//     decode (ps.py:165-167), sum(grads) (ps.py:176), the eager SGD/Adam ops (ps.py:197-261) and
//     the Ibcast of fresh parameters (mpi_comms.py:132)  → psb_update_kernel: ONE launch that
//     pulls every rank's wire tile over NVLink (P2P loads, or one multimem.ld_reduce through the
//     switch), decodes and sums in registers / shared memory in fixed rank order, applies the
//     optimizer to fp32 master state and publishes the new parameter tile to every GPU
//     (multimem.st through the switch, or unicast peer stores), then raises the epoch flag.
//   * MPI requests / req.Wait() (ps.py:146, mpi_comms.py:110,121)  → monotonically increasing epoch
//     flags in the symmetric signal pad (st.release.sys / ld.acquire.sys), bounded spins.
#include <algorithm>
#include <cstdlib>

#include "kernels.h"

namespace {
using namespace psb;

// ------------------------------------------------------------------------------------------
// small block-level helpers
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t block_excl_scan(uint32_t v, uint32_t* warp_tot /*[8]*/, uint32_t* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t incl = v;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    uint32_t n = __shfl_up_sync(0xffffffffu, incl, off);
    if (lane >= off) incl += n;
  }
  if (lane == 31) warp_tot[warp] = incl;
  __syncthreads();
  uint32_t base = 0, tot = 0;
#pragma unroll
  for (int w = 0; w < PSB_THREADS / 32; ++w) {
    uint32_t t = warp_tot[w];
    if (w < warp) base += t;
    tot += t;
  }
  __syncthreads();   // warp_tot may be reused by the caller
  if (total) *total = tot;
  return base + incl - v;
}

__device__ __forceinline__ float block_max(float v, float* red /*[8]*/) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, off));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float m = red[0];
#pragma unroll
  for (int w = 1; w < PSB_THREADS / 32; ++w) m = fmaxf(m, red[w]);
  __syncthreads();
  return m;
}

// Fixed-order fp32 block sum: an xor butterfly over offsets 16, 8, 4, 2, 1 in every warp, then the 8 warp sums in index order,
// every addition an explicit add_rn, so the device and a host build of this code (the CPU emulator) add the same way.  `red` may
// be written again only after the caller's next barrier.
__device__ __forceinline__ float block_sum_rn(float s, float* red /*[8]*/) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) s = add_rn(s, __shfl_xor_sync(0xffffffffu, s, off));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  s = red[0];
#pragma unroll
  for (int w = 1; w < PSB_THREADS / 32; ++w) s = add_rn(s, red[w]);
  return s;
}

// which batch entry / arena tile does this CTA work on
__device__ __forceinline__ void locate(const EncodeBatch& b, int cta, int& entry, int& tile) {
  int e = 0;
  while (e + 1 < b.n && b.cum[e + 1] <= cta) ++e;
  entry = e;
  tile = b.first_tile[e] + (cta - b.cum[e]);
}

__device__ __forceinline__ void load_grad8(const EncodeArgs& a, int entry, const TileInfo& ti, int tile, float* g) {
  const size_t off = (size_t)(tile - ti.first) * PSB_TILE + threadIdx.x * PSB_EPT;
  const int base = threadIdx.x * PSB_EPT;
  if (base < ti.valid) {
    load8_local(a.batch.src[entry], a.grad_dt, off, g);
#pragma unroll
    for (int j = 0; j < PSB_EPT; ++j)
      if (base + j >= ti.valid) g[j] = 0.f;
  } else {
#pragma unroll
    for (int j = 0; j < PSB_EPT; ++j) g[j] = 0.f;
  }
}

// this thread's 8 elements of the fp32 carry (arena-shaped: element i of tile t at t * PSB_TILE + i)
__device__ __forceinline__ float4* carry8(const EncodeArgs& a, int tile) {
  return reinterpret_cast<float4*>(a.residual + (size_t)tile * PSB_TILE + threadIdx.x * PSB_EPT);
}

__device__ __forceinline__ void add_carry8(const EncodeArgs& a, int tile, float* g) {
  const float4* r = carry8(a, tile);
  const float4 r0 = r[0], r1 = r[1];
  g[0] += r0.x, g[1] += r0.y, g[2] += r0.z, g[3] += r0.w;
  g[4] += r1.x, g[5] += r1.y, g[6] += r1.z, g[7] += r1.w;
}

// ------------------------------------------------------------------------------------------
// gradient accumulation (no_sync): carry += gradient in fp32, one add per element, one launch per bucket; padding lanes add 0
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(PSB_THREADS) psb_accumulate_kernel(const __grid_constant__ EncodeArgs a) {
  int entry, tile;
  locate(a.batch, blockIdx.x, entry, tile);
  const TileInfo ti = a.tiles[tile];
  float g[PSB_EPT];
  load_grad8(a, entry, ti, tile, g);
  float4* r = carry8(a, tile);
  const float4 r0 = r[0], r1 = r[1];
  r[0] = make_float4(r0.x + g[0], r0.y + g[1], r0.z + g[2], r0.w + g[3]);
  r[1] = make_float4(r1.x + g[4], r1.y + g[5], r1.z + g[6], r1.w + g[7]);
}

// ------------------------------------------------------------------------------------------
// abs-max pre-pass for Scale codings: one atomicMax per tile into amax_bits[param]
// ------------------------------------------------------------------------------------------
// CARRY: the instantiation for a.residual != nullptr (the plain pass keeps its registers)
template <bool CARRY>
__global__ void __launch_bounds__(PSB_THREADS) psb_absmax_kernel(const __grid_constant__ EncodeArgs a) {
  __shared__ float red[PSB_THREADS / 32];
  int entry, tile;
  locate(a.batch, blockIdx.x, entry, tile);
  const TileInfo ti = a.tiles[tile];
  float g[PSB_EPT];
  load_grad8(a, entry, ti, tile, g);
  if constexpr (CARRY) add_carry8(a, tile, g);   // the abs-max of what the encode will see
  float m = 0.f;
#pragma unroll
  for (int j = 0; j < PSB_EPT; ++j) m = fmaxf(m, isfinite(g[j]) ? fabsf(g[j]) : 0.f);   // amax over finite elements only
  m = block_max(m, red);
  if (threadIdx.x == 0) atomicMax(a.amax_bits + ti.param, __float_as_uint(m));
}

// ------------------------------------------------------------------------------------------
// encode: gradient tile → wire tile (dense cast | abs-max scaled | block-wise top-k | block-wise QSGD | block-wise sign)
// ------------------------------------------------------------------------------------------
// `saturate` = false only when the fp16 wire carries an fp16 gradient: then it is an exact copy, +-Inf included.
template <int WIRE>
__device__ __forceinline__ void store_dense(void* wire_tile, const float* q, bool saturate) {
  const int tid = threadIdx.x;
  if constexpr (WIRE == WIRE_F32) {
    uint4* p = reinterpret_cast<uint4*>(reinterpret_cast<float*>(wire_tile) + tid * PSB_EPT);
    st_v4(p, make_uint4(__float_as_uint(q[0]), __float_as_uint(q[1]), __float_as_uint(q[2]), __float_as_uint(q[3])));
    st_v4(p + 1, make_uint4(__float_as_uint(q[4]), __float_as_uint(q[5]), __float_as_uint(q[6]), __float_as_uint(q[7])));
  } else if constexpr (WIRE == WIRE_BF16) {
    st_v4(reinterpret_cast<uint16_t*>(wire_tile) + tid * PSB_EPT,
          make_uint4(pack_bf16x2(q[0], q[1]), pack_bf16x2(q[2], q[3]), pack_bf16x2(q[4], q[5]), pack_bf16x2(q[6], q[7])));
  } else if constexpr (WIRE == WIRE_F16) {
    st_v4(reinterpret_cast<uint16_t*>(wire_tile) + tid * PSB_EPT,
          saturate ? make_uint4(pack_f16x2_sat(q[0], q[1]), pack_f16x2_sat(q[2], q[3]), pack_f16x2_sat(q[4], q[5]),
                                pack_f16x2_sat(q[6], q[7]))
                   : make_uint4(pack_f16x2(q[0], q[1]), pack_f16x2(q[2], q[3]), pack_f16x2(q[4], q[5]), pack_f16x2(q[6], q[7])));
  } else if constexpr (WIRE == WIRE_E4M3 || WIRE == WIRE_E5M2) {
    uint2 v = make_uint2(pack_fp8x4<WIRE>(q[0], q[1], q[2], q[3]), pack_fp8x4<WIRE>(q[4], q[5], q[6], q[7]));
    *reinterpret_cast<uint2*>(reinterpret_cast<uint8_t*>(wire_tile) + tid * PSB_EPT) = v;
  } else {  // WIRE_I8
    uint2 v = make_uint2(pack_i8x4(q[0], q[1], q[2], q[3]), pack_i8x4(q[4], q[5], q[6], q[7]));
    *reinterpret_cast<uint2*>(reinterpret_cast<uint8_t*>(wire_tile) + tid * PSB_EPT) = v;
  }
}

// Block-wise QSGD (KIND_QSGD): one wire tile = the 2048 codes (int8, or int4 two per byte with element 2i in the low nibble),
// then a 16-byte header holding the fp32 scale and 12 zero bytes.  The rules are those of DESIGN.md (wire numerics); every
// float operation is an explicit round-to-nearest (mul_rn / add_rn / __fdiv_rn / __fsqrt_rn), so no FMA contraction changes a
// bit and a host build of this code (the CPU emulator) computes the same codes.
template <int WIRE>
constexpr int qsgd_payload_bytes() {
  return WIRE == WIRE_I4 ? PSB_TILE / 2 : PSB_TILE;
}

template <int WIRE>
__device__ __forceinline__ void qsgd_encode_tile(const EncodeArgs& a, int tile, uint8_t* wire_tile, const float* g) {
  __shared__ float red[PSB_THREADS / 32];
  const int tid = threadIdx.x;
  // norm = m * r: m = abs-max over the finite elements (exact, so its reduction order is free), r = sqrt(sum of (|g| / m)^2) —
  // the tile scaled by m first, so no finite input overflows; sum order: per thread in index order, xor butterfly, warps in order
  float m = 0.f;
#pragma unroll
  for (int j = 0; j < PSB_EPT; ++j) m = fmaxf(m, isfinite(g[j]) ? fabsf(g[j]) : 0.f);
  m = block_max(m, red);
  const bool any = m > 0.f;
  if (!any) m = 1.f;
  float t[PSB_EPT], s = 0.f;
#pragma unroll
  for (int j = 0; j < PSB_EPT; ++j) {
    t[j] = isfinite(g[j]) ? __fdiv_rn(fabsf(g[j]), m) : 0.f;
    s = add_rn(s, mul_rn(t[j], t[j]));
  }
  s = block_sum_rn(s, red);
  const float r = any ? __fsqrt_rn(s) : 1.f;   // >= 1 when any: the abs-max element contributes exactly 1
  const int levels = a.levels;
  const float lv = (float)levels;

  // q = sign(g) * (floor(x) + [u < x - floor(x)]), x = |g| / m / r * levels; u = (Philox word >> 8) * 2^-24
  const uint32_t k0 = (uint32_t)a.seed, k1 = (uint32_t)(a.seed >> 32);
  const Philox4 ra = philox4x32_10(2 * tid, (uint32_t)tile, a.step, a.rank, k0, k1);
  const Philox4 rb = philox4x32_10(2 * tid + 1, (uint32_t)tile, a.step, a.rank, k0, k1);
  constexpr uint32_t NAN_CODE = WIRE == WIRE_I4 ? 0x8u : 0x80u;
  constexpr uint32_t MASK = WIRE == WIRE_I4 ? 0xfu : 0xffu;
  uint32_t code[PSB_EPT];
#pragma unroll
  for (int j = 0; j < PSB_EPT; ++j) {
    const uint32_t w = j < 4 ? ra.w[j] : rb.w[j - 4];
    const float u = mul_rn((float)(w >> 8), 5.9604644775390625e-8f);   // 2^-24
    int qi;
    if (!isfinite(g[j])) {
      qi = levels;                                                          // +-Inf saturates (NaN: replaced below)
    } else {
      const float x = mul_rn(__fdiv_rn(t[j], r), lv);
      const float fl = floorf(x);
      qi = min((int)fl + (u < add_rn(x, -fl) ? 1 : 0), levels);
    }
    const int q = (__float_as_uint(g[j]) >> 31) ? -qi : qi;
    code[j] = (__float_as_uint(g[j]) & 0x7fffffffu) > 0x7f800000u ? NAN_CODE : (uint32_t)q & MASK;
  }
  if constexpr (WIRE == WIRE_I4) {
    uint32_t v = 0;
#pragma unroll
    for (int j = 0; j < PSB_EPT; ++j) v |= code[j] << (4 * j);
    *reinterpret_cast<uint32_t*>(wire_tile + tid * 4) = v;
  } else {
    const uint2 v = make_uint2(code[0] | code[1] << 8 | code[2] << 16 | code[3] << 24,
                               code[4] | code[5] << 8 | code[6] << 16 | code[7] << 24);
    *reinterpret_cast<uint2*>(wire_tile + tid * 8) = v;
  }
  if (tid == 0) {
    float scale = mul_rn(m, __fdiv_rn(r, lv));          // norm / levels, without the overflow of forming norm first
    if (!(scale <= 3.40282346638528859811704183484516925e+38f)) scale = 3.40282346638528859811704183484516925e+38f;
    st_v4(wire_tile + qsgd_payload_bytes<WIRE>(), make_uint4(__float_as_uint(scale), 0u, 0u, 0u));
  }
}

// Block-wise scaled sign (KIND_SIGN, WIRE_B1): one wire tile = 256 payload bytes, bit j of byte t the sign bit of element 8t + j,
// then a 16-byte header holding the fp32 scale and 12 zero bytes.  Only the tile's real elements (a.real_mask) take part: the
// others get bit 0 and count nowhere.  The rules are those of DESIGN.md (wire numerics); the float operations are explicit
// round-to-nearest ones, as in the QSGD encode.  On return g holds the error-feedback residual: p - decode on the real elements,
// 0 elsewhere.
__device__ __forceinline__ uint32_t real_bits8(const uint32_t* mask, int tile) {   // this thread's 8 elements of the mask
  return mask[(size_t)tile * (PSB_TILE / 32) + (threadIdx.x >> 2)] >> (8 * (threadIdx.x & 3)) & 0xffu;
}

__device__ __forceinline__ void sign_encode_tile(const EncodeArgs& a, int tile, uint8_t* wire_tile, float* g) {
  __shared__ float red[PSB_THREADS / 32];
  __shared__ int cnt[PSB_THREADS / 32];
  const int tid = threadIdx.x;
  const uint32_t real = real_bits8(a.real_mask, tile);
  // m = abs-max over the real elements (exact, so its reduction order is free); a NaN or +-Inf among them makes it +Inf
  float m = 0.f;
#pragma unroll
  for (int j = 0; j < PSB_EPT; ++j)
    if (real >> j & 1u) m = fmaxf(m, isfinite(g[j]) ? fabsf(g[j]) : __uint_as_float(0x7f800000u));
  m = block_max(m, red);
  float scale;
  if (!(m <= 3.40282346638528859811704183484516925e+38f)) {
    scale = __uint_as_float(0x7fffffffu);   // one bit has no NaN code: the whole tile decodes to NaN
  } else if (m == 0.f) {
    scale = 0.f;
  } else {
    // scale = m * (sum of |p| / m over the real elements) / |R|: the mean magnitude, without overflow for any finite input
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < PSB_EPT; ++j)
      if (real >> j & 1u) s = add_rn(s, __fdiv_rn(fabsf(g[j]), m));
    int n = __popc(real);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) n += __shfl_xor_sync(0xffffffffu, n, off);
    if ((tid & 31) == 0) cnt[tid >> 5] = n;
    s = block_sum_rn(s, red);                // (its barrier also publishes cnt)
    n = 0;
#pragma unroll
    for (int w = 0; w < PSB_THREADS / 32; ++w) n += cnt[w];
    scale = mul_rn(m, __fdiv_rn(s, (float)n));
    if (!(scale <= 3.40282346638528859811704183484516925e+38f)) scale = 3.40282346638528859811704183484516925e+38f;
  }
  // the sign bit; a NaN sends 0: adding the carry leaves a NaN's sign to the processor, and the tile decodes to NaN regardless
  uint32_t bits = 0;
#pragma unroll
  for (int j = 0; j < PSB_EPT; ++j) {
    const uint32_t u = __float_as_uint(g[j]);
    bits |= (u >> 31 & real >> j & ((u & 0x7fffffffu) <= 0x7f800000u ? 1u : 0u)) << j;
  }
  wire_tile[tid] = (uint8_t)bits;
  if (tid == 0) st_v4(wire_tile + PSB_TILE / 8, make_uint4(__float_as_uint(scale), 0u, 0u, 0u));
#pragma unroll
  for (int j = 0; j < PSB_EPT; ++j) g[j] = (real >> j & 1u) ? g[j] - ((bits >> j & 1u) ? -scale : scale) : 0.f;
}

// int4 wire: eight two's-complement nibbles, element j in bits [4j, 4j + 4); -8 is the NaN code
__device__ __forceinline__ void unpack_i4x8(uint32_t w, float* f) {
#pragma unroll
  for (int j = 0; j < PSB_EPT; ++j) {
    const int c = (int)(w << (28 - 4 * j)) >> 28;
    f[j] = c == -8 ? __uint_as_float(0x7fffffffu) : (float)c;
  }
}

// CARRY: the instantiation for a.residual != nullptr, so the plain encode keeps its registers.  Top-k always has CARRY = false
// and tests a.residual at run time: its error-feedback residual is older than gradient accumulation.
template <int KIND, int WIRE, bool CARRY>
__global__ void __launch_bounds__(PSB_THREADS) psb_encode_kernel(const __grid_constant__ EncodeArgs a) {
  const bool carry = KIND == KIND_TOPK ? a.residual != nullptr : CARRY;
  int entry, tile;
  locate(a.batch, blockIdx.x, entry, tile);
  const TileInfo ti = a.tiles[tile];
  const int tid = threadIdx.x;
  uint8_t* wire_tile = reinterpret_cast<uint8_t*>(a.wire) + (size_t)tile * a.bytes_per_tile;
  float g[PSB_EPT];
  load_grad8(a, entry, ti, tile, g);
  if (carry) add_carry8(a, tile, g);

  if constexpr (KIND == KIND_DENSE) {
    store_dense<WIRE>(wire_tile, g, a.grad_dt != DT_F16);
  } else if constexpr (KIND == KIND_SCALED) {
    float amax = __uint_as_float(a.amax_bits[ti.param]);
    if (!(amax > 0.f) || !isfinite(amax)) amax = 1.f;
    const float inv = __fdiv_rn(amax, wire_qmax(WIRE));
    if (tile == ti.first && tid == 0) a.scales[ti.param] = inv;
    float q[PSB_EPT];
#pragma unroll
    for (int j = 0; j < PSB_EPT; ++j) q[j] = __fdiv_rn(g[j], inv);
    store_dense<WIRE>(wire_tile, q, true);
  } else if constexpr (KIND == KIND_QSGD) {
    qsgd_encode_tile<WIRE>(a, tile, wire_tile, g);
  } else if constexpr (KIND == KIND_SIGN) {
    sign_encode_tile(a, tile, wire_tile, g);
  } else {  // KIND_TOPK: block-wise magnitude top-k, ties → lower index, entries in index order
    __shared__ uint32_t hist[256];
    __shared__ uint32_t warp_tot[PSB_THREADS / 32];
    __shared__ uint32_t s_prefix, s_k;
    uint32_t key[PSB_EPT];
#pragma unroll
    for (int j = 0; j < PSB_EPT; ++j) key[j] = (tid * PSB_EPT + j < ti.valid) ? (__float_as_uint(g[j]) & 0x7fffffffu) : 0u;
    int k = (int)ceil((double)a.ratio * (double)ti.valid - 1e-9);
    k = max(1, min(ti.valid, k));
    uint32_t prefix = 0, mask = 0, kk = (uint32_t)k;
#pragma unroll 1
    for (int shift = 24; shift >= 0; shift -= 8) {
      hist[tid] = 0;
      __syncthreads();
#pragma unroll
      for (int j = 0; j < PSB_EPT; ++j)
        if ((key[j] & mask) == prefix) atomicAdd(&hist[(key[j] >> shift) & 0xffu], 1u);
      __syncthreads();
      if (tid < 32) {
        uint32_t c[8], sum = 0;
#pragma unroll
        for (int b = 0; b < 8; ++b) {
          c[b] = hist[255 - 8 * tid - b];
          sum += c[b];
        }
        uint32_t incl = sum;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
          uint32_t n = __shfl_up_sync(0xffffffffu, incl, off);
          if (tid >= off) incl += n;
        }
        const uint32_t excl = incl - sum;
        if (excl < kk && kk <= incl) {
          uint32_t run = excl;
#pragma unroll
          for (int b = 0; b < 8; ++b) {
            if (run + c[b] >= kk) {
              s_prefix = prefix | ((uint32_t)(255 - 8 * tid - b) << shift);
              s_k = kk - run;
              break;
            }
            run += c[b];
          }
        }
      }
      __syncthreads();
      prefix = s_prefix;
      kk = s_k;
      mask |= 0xffu << shift;
      __syncthreads();
    }
    const uint32_t T = prefix;   // k-th largest magnitude; take every key > T and the first kk keys == T
    uint32_t eqc = 0;
#pragma unroll
    for (int j = 0; j < PSB_EPT; ++j) eqc += (key[j] == T);
    uint32_t eq_before = block_excl_scan(eqc, warp_tot, nullptr);
    uint32_t selbits = 0, selc = 0;
#pragma unroll
    for (int j = 0; j < PSB_EPT; ++j) {
      bool s = key[j] > T;
      if (key[j] == T) {
        s = eq_before < kk;
        ++eq_before;
      }
      if (s) {
        selbits |= 1u << j;
        ++selc;
      }
    }
    uint32_t total = 0;
    uint32_t pos = block_excl_scan(selc, warp_tot, &total);
#pragma unroll
    for (int j = 0; j < PSB_EPT; ++j) {
      if (selbits >> j & 1u) {
        const uint32_t idx = tid * PSB_EPT + j;
        if constexpr (WIRE == WIRE_BF16) {
          __nv_bfloat16 hv = __float2bfloat16_rn(g[j]);
          const uint32_t bits = *reinterpret_cast<uint16_t*>(&hv);
          reinterpret_cast<uint32_t*>(wire_tile)[pos] = (idx << 16) | bits;
          g[j] -= __bfloat162float(hv);       // what stays behind as residual
        } else {
          reinterpret_cast<uint2*>(wire_tile)[pos] = make_uint2(idx, __float_as_uint(g[j]));
          g[j] = 0.f;
        }
        ++pos;
      }
    }
    for (uint32_t p = total + tid; p < (uint32_t)a.cap; p += PSB_THREADS) {   // pad: idx == PSB_TILE is "no entry"
      if constexpr (WIRE == WIRE_BF16) reinterpret_cast<uint32_t*>(wire_tile)[p] = (uint32_t)PSB_TILE << 16;
      else reinterpret_cast<uint2*>(wire_tile)[p] = make_uint2(PSB_TILE, 0u);
    }
  }
  if (carry) {   // the carry is consumed: the error-feedback kinds keep what the wire did not carry, everything else zero
    const bool keep = (KIND == KIND_TOPK || KIND == KIND_SIGN) && !a.drop_leftover;
    float4* r = carry8(a, tile);
    r[0] = keep ? make_float4(g[0], g[1], g[2], g[3]) : make_float4(0.f, 0.f, 0.f, 0.f);
    r[1] = keep ? make_float4(g[4], g[5], g[6], g[7]) : make_float4(0.f, 0.f, 0.f, 0.f);
  }

  // ---- fused flag raise (last encode launch of the step): the last CTA to finish publishes GRAD_READY ----
  if (a.nsig > 0) {
    __shared__ int s_last;
    __syncthreads();
    if (tid == 0) {
      __threadfence_system();                       // this CTA's wire tile is visible system-wide
      s_last = (atomicAdd(a.sig_counter, 1u) == gridDim.x - 1);
    }
    __syncthreads();
    if (s_last) {
      if (tid == 0) *a.sig_counter = 0;
      __threadfence_system();
      if (tid < a.nsig && a.sig_targets[tid] != nullptr) st_release_sys(a.sig_targets[tid] + a.sig_slot, a.sig_value);
    }
  }
}

// ------------------------------------------------------------------------------------------
// the fused PS kernel
// ------------------------------------------------------------------------------------------
template <int WIRE>
__device__ __forceinline__ void issue_dense(const void* wire_base, size_t tile_byte_off, uint4& v0, uint4& v1) {
  const uint8_t* p = reinterpret_cast<const uint8_t*>(wire_base) + tile_byte_off +
                     (size_t)threadIdx.x * PSB_EPT * wire_elem_bytes(WIRE);
  if constexpr (WIRE == WIRE_F32) {
    v0 = ld_sys_v4(p);
    v1 = ld_sys_v4(p + 16);
  } else if constexpr (WIRE == WIRE_BF16 || WIRE == WIRE_F16) {
    v0 = ld_sys_v4(p);
  } else {
    uint2 t = ld_sys_v2(p);
    v0.x = t.x, v0.y = t.y;
  }
}

template <int WIRE>
__device__ __forceinline__ void decode_dense(const uint4& v0, const uint4& v1, float* f) {
  if constexpr (WIRE == WIRE_F32) {
    f[0] = __uint_as_float(v0.x), f[1] = __uint_as_float(v0.y), f[2] = __uint_as_float(v0.z), f[3] = __uint_as_float(v0.w);
    f[4] = __uint_as_float(v1.x), f[5] = __uint_as_float(v1.y), f[6] = __uint_as_float(v1.z), f[7] = __uint_as_float(v1.w);
  } else if constexpr (WIRE == WIRE_BF16) {
    unpack_bf16x8(v0, f);
  } else if constexpr (WIRE == WIRE_F16) {
    unpack_f16x8(v0, f);
  } else if constexpr (WIRE == WIRE_E4M3 || WIRE == WIRE_E5M2) {
    unpack_fp8x8<WIRE>(make_uint2(v0.x, v0.y), f);
  } else {
    unpack_i8x8(make_uint2(v0.x, v0.y), f);
  }
}

// Publish one thread's packed parameter vectors (`nv` of `out`) at byte offset `pbytes` of the parameter arena: through the
// switch (multicast), into every rank's arena (unicast peer stores), or into this rank's own.  The publication of
// apply_and_publish below, for psb_publish_kernel.
__device__ __forceinline__ void publish_packed(int bcast, void* param_mc, void* const* param_dst, void* param_local, int world,
                                               size_t pbytes, const uint4* out, int nv) {
  if (bcast == BCAST_MULTICAST) {
    uint8_t* p = reinterpret_cast<uint8_t*>(param_mc) + pbytes;
    multimem_st_v4(p, out[0]);
    if (nv == 2) multimem_st_v4(p + 16, out[1]);
  } else if (bcast == BCAST_UNICAST) {
    for (int r = 0; r < world; ++r) {
      uint8_t* p = reinterpret_cast<uint8_t*>(param_dst[r]) + pbytes;
      st_sys_v4(p, out[0]);
      if (nv == 2) st_sys_v4(p + 16, out[1]);
    }
  } else {
    uint8_t* p = reinterpret_cast<uint8_t*>(param_local) + pbytes;
    st_v4(p, out[0]);
    if (nv == 2) st_v4(p + 16, out[1]);
  }
}

// Optimizer + publication for ONE tile whose summed gradient is already in `acc` (and whose state
// `w`, `b0`, `b1`, `b2` has been loaded): the epilogue shared by every gather flavour.
template <int OPT>
__device__ __forceinline__ void apply_and_publish(const UpdateArgs& a, const TileInfo& ti, size_t e0, float inv_count,
                                                  const float* acc, float* w, float* m, float* v, float* vm) {
  GroupHyper h = a.groups[ti.group];
  if (a.param_hyper != nullptr) {
    // parameters whose step count differs from their group's (a gradient that first arrived late, a layer that was frozen
    // for a while): the reference keeps state PER PARAMETER (/root/reference/ps.py:203-205,226-241), so the bias-corrected
    // Adam step size and SGD's first-step momentum rule come from a per-parameter table
    const float2 ph = a.param_hyper[ti.param];
    h.step_size = ph.x;
    if constexpr (OPT == OPT_ADAMW) h.beta1 = ph.y;   // c2 (common.cuh)
    else h.first_step = ph.y != 0.f;
  }
  float g[PSB_EPT];
#pragma unroll
  for (int j = 0; j < PSB_EPT; ++j) g[j] = acc[j] * inv_count;
  if constexpr (OPT != OPT_ADAMW) {   // coupled L2 decay; AdamW decays the weight itself
    if (h.weight_decay != 0.f) {
#pragma unroll
      for (int j = 0; j < PSB_EPT; ++j) g[j] = fmaf(h.weight_decay, w[j], g[j]);
    }
  }
  if constexpr (OPT == OPT_ADAMW) {   // DESIGN.md, optimizer rule A1: torch.optim.AdamW's fp32 sequence
    // torch's lerp_(g, a): fma(a, g - m, m) for a < 0.5, fma(a - 1, g - m, g) otherwise (a - 1 is exact there)
    const bool small = h.momentum < 0.5f;
    const float wa = small ? h.momentum : add_rn(h.momentum, -1.f);
#pragma unroll
    for (int j = 0; j < PSB_EPT; ++j) {
      if (h.weight_decay != 1.f) w[j] = mul_rn(w[j], h.weight_decay);
      m[j] = fma_rn(wa, add_rn(g[j], -m[j]), small ? m[j] : g[j]);
      v[j] = fma_rn(mul_rn(h.dampening, g[j]), g[j], mul_rn(v[j], h.beta2));
    }
#pragma unroll
    for (int j = 0; j < PSB_EPT; ++j) {
      float den_src = v[j];
      if (h.amsgrad) {
        vm[j] = max_nan(vm[j], v[j]);
        den_src = vm[j];
      }
      const float den = add_rn(__fdiv_rn(__fsqrt_rn(den_src), h.beta1), h.eps);
      w[j] = add_rn(w[j], __fdiv_rn(mul_rn(-h.step_size, m[j]), den));
    }
    float4* mp = reinterpret_cast<float4*>(a.buf0 + e0);
    mp[0] = make_float4(m[0], m[1], m[2], m[3]);
    mp[1] = make_float4(m[4], m[5], m[6], m[7]);
    float4* vp = reinterpret_cast<float4*>(a.buf1 + e0);
    vp[0] = make_float4(v[0], v[1], v[2], v[3]);
    vp[1] = make_float4(v[4], v[5], v[6], v[7]);
    if (h.amsgrad) {
      float4* xp = reinterpret_cast<float4*>(a.buf2 + e0);
      xp[0] = make_float4(vm[0], vm[1], vm[2], vm[3]);
      xp[1] = make_float4(vm[4], vm[5], vm[6], vm[7]);
    }
  } else if constexpr (OPT == OPT_SGD) {   // /root/reference/ps.py:197-214
    if (h.momentum != 0.f) {
#pragma unroll
      for (int j = 0; j < PSB_EPT; ++j) {
        m[j] = h.first_step ? g[j] : fmaf(h.momentum, m[j], (1.f - h.dampening) * g[j]);
        g[j] = h.nesterov ? fmaf(h.momentum, m[j], g[j]) : m[j];
      }
      float4* bp = reinterpret_cast<float4*>(a.buf0 + e0);
      bp[0] = make_float4(m[0], m[1], m[2], m[3]);
      bp[1] = make_float4(m[4], m[5], m[6], m[7]);
    }
#pragma unroll
    for (int j = 0; j < PSB_EPT; ++j) w[j] = fmaf(-h.lr, g[j], w[j]);
  } else {                          // /root/reference/ps.py:218-261
#pragma unroll
    for (int j = 0; j < PSB_EPT; ++j) {
      m[j] = fmaf(h.beta1, m[j], (1.f - h.beta1) * g[j]);
      v[j] = fmaf(h.beta2, v[j], (1.f - h.beta2) * g[j] * g[j]);
      float den_src = v[j];
      if (h.amsgrad) {
        vm[j] = fmaxf(vm[j], v[j]);
        den_src = vm[j];
      }
      const float denom = __fsqrt_rn(den_src) + h.eps;
      w[j] = fmaf(-h.step_size, __fdiv_rn(m[j], denom), w[j]);
    }
    float4* mp = reinterpret_cast<float4*>(a.buf0 + e0);
    mp[0] = make_float4(m[0], m[1], m[2], m[3]);
    mp[1] = make_float4(m[4], m[5], m[6], m[7]);
    float4* vp = reinterpret_cast<float4*>(a.buf1 + e0);
    vp[0] = make_float4(v[0], v[1], v[2], v[3]);
    vp[1] = make_float4(v[4], v[5], v[6], v[7]);
    if (h.amsgrad) {
      float4* xp = reinterpret_cast<float4*>(a.buf2 + e0);
      xp[0] = make_float4(vm[0], vm[1], vm[2], vm[3]);
      xp[1] = make_float4(vm[4], vm[5], vm[6], vm[7]);
    }
  }
  if (a.master != nullptr) {
    float4* wp = reinterpret_cast<float4*>(a.master + e0);
    wp[0] = make_float4(w[0], w[1], w[2], w[3]);
    wp[1] = make_float4(w[4], w[5], w[6], w[7]);
  }
  // publish the fresh parameter tile (the Ibcast of mpi_comms.py:132)
  uint4 out[2];
  const int nv = pack8(a.param_dt, w, out);
  const size_t pbytes = e0 * (a.param_dt == DT_F32 ? 4 : 2);
  // (the same stores as publish_packed; calling it here changes the SASS of the dense update kernels, so they stay inline)
  if (a.bcast == BCAST_MULTICAST) {
    uint8_t* p = reinterpret_cast<uint8_t*>(a.param_mc) + pbytes;
    multimem_st_v4(p, out[0]);
    if (nv == 2) multimem_st_v4(p + 16, out[1]);
  } else if (a.bcast == BCAST_UNICAST) {
    for (int r = 0; r < a.world; ++r) {
      uint8_t* p = reinterpret_cast<uint8_t*>(a.param_dst[r]) + pbytes;
      st_sys_v4(p, out[0]);
      if (nv == 2) st_sys_v4(p + 16, out[1]);
    }
  } else {
    uint8_t* p = reinterpret_cast<uint8_t*>(a.param_local) + pbytes;
    st_v4(p, out[0]);
    if (nv == 2) st_v4(p + 16, out[1]);
  }
}

// Issue the (local, independent) optimizer-state loads for one tile: they fly while the peer loads do.
template <int OPT>
__device__ __forceinline__ void load_state(const UpdateArgs& a, const TileInfo& ti, size_t e0, float* w, float* m, float* v,
                                           float* vm) {
  if (a.master != nullptr) load8_local(a.master, DT_F32, e0, w);
  else load8_local(a.param_local, a.param_dt, e0, w);
  const GroupHyper& h = a.groups[ti.group];
  if constexpr (OPT == OPT_SGD) {
    if (h.momentum != 0.f) load8_local(a.buf0, DT_F32, e0, m);
  } else {
    load8_local(a.buf0, DT_F32, e0, m);
    load8_local(a.buf1, DT_F32, e0, v);
    if (h.amsgrad) load8_local(a.buf2, DT_F32, e0, vm);
  }
}

// One launch covers arena tiles [tile_begin, tile_end): the whole model, or ONE CHUNK of the per-bucket pipeline — the
// device analogue of the reference posting one non-blocking collective per parameter and consuming each as it completes
// (/root/reference/ps.py:140-148,159-162).  The engine launches chunk k's update while backward is still producing
// chunk k+1; GRAD_READY carries a monotone progress value ((epoch-1)*nchunks + chunk + 1), so one flag per rank serves
// every chunk.
//
// NVLS_U = tiles a thread keeps in flight on the multimem.ld_reduce path: one 16-byte switch reduction per tile is far too
// little to cover the NVLS round trip, so four are issued back to back before the first is consumed.
constexpr int NVLS_U = 4;

template <int KIND, int WIRE, int OPT>
__global__ void __launch_bounds__(PSB_THREADS, 3) psb_update_kernel(const __grid_constant__ UpdateArgs a) {
  __shared__ float s_acc[KIND == KIND_TOPK ? PSB_TILE : 1];
  __shared__ int s_flag;
  const int tid = threadIdx.x;
  uint64_t* err_slot = a.signal_local + SIG_ERROR;
  uint32_t contrib = a.contrib_mask, ack = a.ack_mask;
  float inv_count = a.inv_count;
  if (a.select_out != nullptr) {   // async: the contributor set was chosen on the device
    contrib = (uint32_t)a.select_out[0];
    ack = a.ack_last ? contrib : 0u;
    const uint32_t cnt = (uint32_t)a.select_out[1];
    if (cnt == 0) return;          // nothing to apply (all workers finished, or the select timed out)
    if (a.average_dynamic) inv_count = 1.f / (float)cnt;
  }

  // ---- 1. the req.Wait() of the reference: every contributor's progress flag ----
  // (the pipelined engine waits in a one-warp kernel queued just ahead of this one instead — a full update grid spinning
  //  on its peers would hold every SM's registers while this rank's backward still runs; then only the error slot is checked:
  //  a timed-out wait must not be followed by an update over stale tiles)
  if (a.wait_grads) {
    bool ok = true;
    if (tid < a.world && (contrib & a.wait_mask) >> tid & 1u)
      ok = spin_until_ge(a.signal_local + SIG_GRAD_READY + tid, a.wait_value, err_slot, a.timeout_ns);
    if (!__syncthreads_and(ok)) return;
  } else if (a.world > 1) {
    bool ok = true;
    if (tid == 0) ok = ld_relaxed_sys_u64(err_slot) == 0;
    if (!__syncthreads_and(ok)) return;
  }

  if constexpr (KIND == KIND_TOPK) {
    // ---- block-wise top-k: every rank's (index, value) entries are fetched with 16-byte peer loads, ALL ranks in
    // flight at once (2 vectors per thread per round), then scatter-added into a shared-memory tile rank by rank
    // (rank order = summation order, so the sum stays bit-reproducible) ----
    constexpr int ENT = (WIRE == WIRE_BF16) ? 4 : 2;     // entries per 16-byte vector
    constexpr int VPT = 2;                               // vectors per thread per round
    const int nv = a.bytes_per_tile >> 4;                // vectors per rank per tile
    const int total = a.world * nv;
    for (int tile = a.tile_begin + blockIdx.x; tile < a.tile_end; tile += gridDim.x) {
      const TileInfo ti = a.tiles[tile];
      if (a.active != nullptr && a.active[ti.param] == 0) continue;
      const size_t e0 = (size_t)tile * PSB_TILE + tid * PSB_EPT;
      const size_t tile_off = (size_t)tile * a.bytes_per_tile;
      float w[PSB_EPT], m[PSB_EPT], v[PSB_EPT], vm[PSB_EPT];
      load_state<OPT>(a, ti, e0, w, m, v, vm);           // local; flies while the peer loads do
      for (int j = tid; j < PSB_TILE; j += PSB_THREADS) s_acc[j] = 0.f;
      __syncthreads();
      for (int base = 0; base < total; base += VPT * PSB_THREADS) {
        uint4 q[VPT];
        int qr[VPT], qj[VPT];
#pragma unroll
        for (int k = 0; k < VPT; ++k) {
          const int vid = base + k * PSB_THREADS + tid;
          qr[k] = -1;
          qj[k] = 0;
          if (vid < total) {
            const int r = vid / nv;
            if (contrib >> r & 1u) {
              qr[k] = r;
              qj[k] = vid - r * nv;
              q[k] = ld_sys_v4(reinterpret_cast<const uint8_t*>(a.wire[r]) + tile_off + 16 * (size_t)qj[k]);
            }
          }
        }
        const int r_lo = base / nv, r_hi = (min(total, base + VPT * PSB_THREADS) - 1) / nv;
        for (int r = r_lo; r <= r_hi; ++r) {
#pragma unroll
          for (int k = 0; k < VPT; ++k) {
            if (qr[k] != r) continue;
            const uint32_t wd[4] = {q[k].x, q[k].y, q[k].z, q[k].w};
#pragma unroll
            for (int e = 0; e < ENT; ++e) {
              if (qj[k] * ENT + e >= a.cap) break;       // alignment padding behind the last entry
              uint32_t idx;
              float val;
              if constexpr (WIRE == WIRE_BF16) {
                idx = wd[e] >> 16;
                val = __uint_as_float(wd[e] << 16);
              } else {
                idx = wd[2 * e];
                val = __uint_as_float(wd[2 * e + 1]);
              }
              if (idx < PSB_TILE) s_acc[idx] += val;     // indices are unique within one rank's tile
            }
          }
          __syncthreads();
        }
      }
      float acc[PSB_EPT];
#pragma unroll
      for (int j = 0; j < PSB_EPT; ++j) acc[j] = s_acc[tid * PSB_EPT + j];
      __syncthreads();
      apply_and_publish<OPT>(a, ti, e0, inv_count, acc, w, m, v, vm);
    }
  } else if constexpr (KIND == KIND_QSGD) {
    // ---- block-wise QSGD over P2P: each rank's codes (8 bytes per thread on the int8 wire, 4 on the int4 wire) and the scale
    // in that rank's tile header, up to CH ranks in flight; q * scale summed in rank order ----
    constexpr int CH = 4;
    constexpr int PAY = qsgd_payload_bytes<WIRE>();
    for (int tile = a.tile_begin + blockIdx.x; tile < a.tile_end; tile += gridDim.x) {
      const TileInfo ti = a.tiles[tile];
      if (a.active != nullptr && a.active[ti.param] == 0) continue;
      const size_t e0 = (size_t)tile * PSB_TILE + tid * PSB_EPT;
      const size_t tile_off = (size_t)tile * a.bytes_per_tile;
      float acc[PSB_EPT], w[PSB_EPT], m[PSB_EPT], v[PSB_EPT], vm[PSB_EPT];
#pragma unroll
      for (int j = 0; j < PSB_EPT; ++j) acc[j] = 0.f;
      load_state<OPT>(a, ti, e0, w, m, v, vm);
      for (int r0 = 0; r0 < a.world; r0 += CH) {
        uint2 q[CH];
        float sc[CH];
#pragma unroll
        for (int c = 0; c < CH; ++c) {
          const int r = r0 + c;
          sc[c] = 0.f;
          if (r < a.world && (contrib >> r & 1u)) {
            const uint8_t* p = reinterpret_cast<const uint8_t*>(a.wire[r]) + tile_off;
            if constexpr (WIRE == WIRE_I4) q[c].x = ld_sys_u32(p + tid * 4);
            else q[c] = ld_sys_v2(p + tid * 8);
            sc[c] = ld_sys_f32(reinterpret_cast<const float*>(p + PAY));
          }
        }
#pragma unroll
        for (int c = 0; c < CH; ++c) {       // fixed rank order → deterministic fp32 sum
          const int r = r0 + c;
          if (r < a.world && (contrib >> r & 1u)) {
            float f[PSB_EPT];
            if constexpr (WIRE == WIRE_I4) unpack_i4x8(q[c].x, f);
            else unpack_i8x8(q[c], f);
#pragma unroll
            for (int j = 0; j < PSB_EPT; ++j) acc[j] += f[j] * sc[c];
          }
        }
      }
      apply_and_publish<OPT>(a, ti, e0, inv_count, acc, w, m, v, vm);
    }
  } else if constexpr (KIND == KIND_SIGN) {
    // ---- block-wise sign over P2P: each rank's payload word holding this thread's byte and the scale in that rank's tile header,
    // up to CH ranks in flight; +-scale summed in rank order, then every lane outside the tile's real elements set to 0, so
    // padding, master and optimizer state stay exactly 0 ----
    constexpr int CH = 8;
    for (int tile = a.tile_begin + blockIdx.x; tile < a.tile_end; tile += gridDim.x) {
      const TileInfo ti = a.tiles[tile];
      if (a.active != nullptr && a.active[ti.param] == 0) continue;
      const size_t e0 = (size_t)tile * PSB_TILE + tid * PSB_EPT;
      const size_t tile_off = (size_t)tile * a.bytes_per_tile;
      const uint32_t real = real_bits8(a.real_mask, tile);
      float acc[PSB_EPT], w[PSB_EPT], m[PSB_EPT], v[PSB_EPT], vm[PSB_EPT];
#pragma unroll
      for (int j = 0; j < PSB_EPT; ++j) acc[j] = 0.f;
      load_state<OPT>(a, ti, e0, w, m, v, vm);
      for (int r0 = 0; r0 < a.world; r0 += CH) {
        uint32_t q[CH];
        float sc[CH];
#pragma unroll
        for (int c = 0; c < CH; ++c) {
          const int r = r0 + c;
          q[c] = 0u, sc[c] = 0.f;
          if (r < a.world && (contrib >> r & 1u)) {
            const uint8_t* p = reinterpret_cast<const uint8_t*>(a.wire[r]) + tile_off;
            q[c] = ld_sys_u32(p + (tid & ~3));
            sc[c] = ld_sys_f32(reinterpret_cast<const float*>(p + PSB_TILE / 8));
          }
        }
#pragma unroll
        for (int c = 0; c < CH; ++c) {       // fixed rank order → deterministic fp32 sum
          const int r = r0 + c;
          if (r < a.world && (contrib >> r & 1u)) {
            const uint32_t b = q[c] >> (8 * (tid & 3));
#pragma unroll
            for (int j = 0; j < PSB_EPT; ++j) acc[j] += (b >> j & 1u) ? -sc[c] : sc[c];
          }
        }
      }
#pragma unroll
      for (int j = 0; j < PSB_EPT; ++j)
        if (!(real >> j & 1u)) acc[j] = 0.f;
      apply_and_publish<OPT>(a, ti, e0, inv_count, acc, w, m, v, vm);
    }
  } else {
    constexpr bool NVLS_OK = KIND == KIND_DENSE && (WIRE == WIRE_F32 || WIRE == WIRE_BF16 || WIRE == WIRE_F16);
    if (NVLS_OK && a.reduce == REDUCE_NVLS) {
      if constexpr (NVLS_OK) {
        // ---- the switch adds all ranks (multimem.ld_reduce): server ingress is 1x the vector, not (N-1)x ----
        for (int tile0 = a.tile_begin + blockIdx.x; tile0 < a.tile_end; tile0 += NVLS_U * gridDim.x) {
          uint4 v0[NVLS_U], v1[NVLS_U];
          TileInfo ti[NVLS_U];
          bool live[NVLS_U];
#pragma unroll
          for (int u = 0; u < NVLS_U; ++u) {
            const int tile = tile0 + u * gridDim.x;
            live[u] = tile < a.tile_end;
            if (live[u]) {
              ti[u] = a.tiles[tile];
              if (a.active != nullptr && a.active[ti[u].param] == 0) live[u] = false;
            }
            if (live[u]) {
              const uint8_t* p = reinterpret_cast<const uint8_t*>(a.wire_mc) + (size_t)tile * a.bytes_per_tile +
                                 (size_t)tid * PSB_EPT * wire_elem_bytes(WIRE);
              if constexpr (WIRE == WIRE_F32) {
                v0[u] = multimem_ld_reduce_f32x4(p);
                v1[u] = multimem_ld_reduce_f32x4(p + 16);
              } else if constexpr (WIRE == WIRE_BF16) {
                v0[u] = multimem_ld_reduce_bf16x8(p);
              } else {
                v0[u] = multimem_ld_reduce_f16x8(p);
              }
            }
          }
#pragma unroll
          for (int u = 0; u < NVLS_U; ++u) {
            if (!live[u]) continue;
            const size_t e0 = (size_t)(tile0 + u * gridDim.x) * PSB_TILE + tid * PSB_EPT;
            float acc[PSB_EPT], w[PSB_EPT], m[PSB_EPT], v[PSB_EPT], vm[PSB_EPT];
            load_state<OPT>(a, ti[u], e0, w, m, v, vm);
            decode_dense<WIRE>(v0[u], v1[u], acc);
            apply_and_publish<OPT>(a, ti[u], e0, inv_count, acc, w, m, v, vm);
          }
        }
      }
    } else {
      // ---- dense / scaled wires over P2P: up to CH ranks of 16-byte peer loads in flight per thread, local optimizer
      // state issued first (independent of the gather, so it overlaps the NVLink latency) ----
      constexpr int CH = 4;
      for (int tile = a.tile_begin + blockIdx.x; tile < a.tile_end; tile += gridDim.x) {
        const TileInfo ti = a.tiles[tile];
        if (a.active != nullptr && a.active[ti.param] == 0) continue;
        const size_t e0 = (size_t)tile * PSB_TILE + tid * PSB_EPT;
        float acc[PSB_EPT], w[PSB_EPT], m[PSB_EPT], v[PSB_EPT], vm[PSB_EPT];
#pragma unroll
        for (int j = 0; j < PSB_EPT; ++j) acc[j] = 0.f;
        load_state<OPT>(a, ti, e0, w, m, v, vm);
        for (int r0 = 0; r0 < a.world; r0 += CH) {
          uint4 v0[CH], v1[CH];
          float sc[CH];
#pragma unroll
          for (int c = 0; c < CH; ++c) {
            const int r = r0 + c;
            sc[c] = 1.f;
            if (r < a.world && (contrib >> r & 1u)) {
              issue_dense<WIRE>(a.wire[r], (size_t)tile * a.bytes_per_tile, v0[c], v1[c]);
              if constexpr (KIND == KIND_SCALED) sc[c] = ld_sys_f32(a.scales[r] + ti.param);
            }
          }
#pragma unroll
          for (int c = 0; c < CH; ++c) {       // fixed rank order → deterministic fp32 sum
            const int r = r0 + c;
            if (r < a.world && (contrib >> r & 1u)) {
              float f[PSB_EPT];
              decode_dense<WIRE>(v0[c], v1[c], f);
#pragma unroll
              for (int j = 0; j < PSB_EPT; ++j) {
                if constexpr (KIND == KIND_SCALED) acc[j] += f[j] * sc[c];
                else acc[j] += f[j];
              }
            }
          }
        }
        apply_and_publish<OPT>(a, ti, e0, inv_count, acc, w, m, v, vm);
      }
    }
  }

  // ---- completion: the last CTA raises the epoch flags ----
  // Launches that raise nothing (every pipeline chunk but the last; any launch at N = 1) skip the block: the system-scope
  // fence + completion atomic cost each CTA a round trip its warps wait out at the barrier (ncu: `barrier` was the top
  // stall of a 2-3-tile chunk launch).  Their stores are ordered before the last chunk's flag by the stream: a kernel's
  // writes — peer and multimem stores included — are complete when the kernel is.
  if (a.signal_mode == SIGNAL_NONE && ack == 0u) return;
  __syncthreads();
  if (tid == 0) {
    __threadfence_system();
    const unsigned prev = atomicAdd(a.done_counter, 1u);
    s_flag = (prev == gridDim.x - 1);
  }
  __syncthreads();
  if (s_flag) {
    if (tid == 0) {
      *a.done_counter = 0;
      if (a.stats) atomicAdd(a.stats, 1u);
    }
    __threadfence_system();
    if (tid < a.world) {
      if (a.signal_mode == SIGNAL_PARAMS_READY) {
        st_release_sys(a.signal_peer[tid] + SIG_VERSION, a.version);
        st_release_sys(a.signal_peer[tid] + SIG_PARAMS_READY, a.epoch);
      } else if (a.signal_mode == SIGNAL_CONSUMED) {
        st_release_sys(a.signal_peer[tid] + SIG_CONSUMED + a.rank, a.epoch);
      } else if (a.signal_mode == SIGNAL_PARAMS_READY_ADD) {
        // mode='sharded': N servers each add 1 after publishing their share, so e*N means "all of step e is published".
        // Adds are read-modify-writes of one location, so they form a release sequence (PTX memory model): an acquire
        // that reads e*N — the value written by the LAST add — synchronizes with EVERY earlier release-add, and thus sees
        // every server's parameter stores, not only the last server's.
        red_release_sys_add_u64(a.signal_peer[tid] + SIG_PARAMS_READY, 1ull);
      }
      if (ack >> tid & 1u) {
        const uint64_t e = ld_relaxed_sys_u64(a.signal_local + SIG_GRAD_READY + tid);
        st_release_sys(a.signal_peer[tid] + SIG_ACK, e);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// flags
// ------------------------------------------------------------------------------------------
struct SignalArgs {
  uint64_t* targets[PSB_MAX_RANKS];
  int32_t n, slot;
  uint64_t value;
  uint64_t* extra_base;
  int32_t extra_slot;
  uint64_t extra_value;
  // async staleness accounting: when set, the kernel first posts "the parameter version this gradient was computed on"
  // (sampled into `version_local[SIG_SEEN_VERSION]` when the PREVIOUS gradient was posted, i.e. right before the forward
  // pass that produced this one started) into targets[t][version_slot], then re-samples the latest published version.
  uint64_t* version_local;
  int32_t version_slot;
  int32_t add;       // targets[t][slot] += value instead of the store (a server of mode='sharded' that updated nothing last)
};

__global__ void psb_signal_kernel(const __grid_constant__ SignalArgs a) {
  __threadfence_system();
  const int t = threadIdx.x;
  uint64_t seen = 0;
  if (a.version_local != nullptr) seen = ld_relaxed_sys_u64(a.version_local + SIG_SEEN_VERSION);
  if (t < a.n) {
    if (a.extra_base != nullptr && a.targets[t] != nullptr) st_release_sys(a.targets[t] + a.extra_slot, a.extra_value);
    if (a.version_local != nullptr && a.targets[t] != nullptr) st_release_sys(a.targets[t] + a.version_slot, seen);
    if (a.targets[t] != nullptr) {
      if (a.add) red_release_sys_add_u64(a.targets[t] + a.slot, a.value);
      else st_release_sys(a.targets[t] + a.slot, a.value);
    }
  }
  __syncwarp();      // every lane has read `seen` before lane 0 replaces it (several targets: one lane each)
  if (a.version_local != nullptr && t == 0)
    st_release_sys(a.version_local + SIG_SEEN_VERSION, ld_acquire_sys(a.version_local + SIG_VERSION));
}

__global__ void psb_wait_kernel(const uint64_t* signal_local, int slot0, uint32_t mask, uint64_t want,
                                unsigned long long timeout_ns) {
  const int t = threadIdx.x;
  if (mask >> t & 1u)
    spin_until_ge(signal_local + slot0 + t, want, const_cast<uint64_t*>(signal_local) + SIG_ERROR, timeout_ns);
}

// async PS: wait until `quota` candidate workers (ANY source, README.md:65-70) have a gradient newer
// than what was consumed.  Workers that posted the DONE epoch are reported in out[40] and never chosen.
// The whole server iteration is device-resident: this kernel also
//   * opens the consistent-read sequence lock (SIG_STAGE_BEGIN = version on every rank) iff something was selected,
//   * records the staleness of every selected gradient (updates applied since the parameters it was computed on):
//     out[44 + r] = (version - 1) - SIG_GRAD_VERSION[r],
// so the host never has to look at the result before queueing the update kernel and the next select.
#define PSB_DONE_EPOCH (1ull << 62)
struct SelectArgs {
  const uint64_t* signal_local;
  uint64_t* consumed;
  uint64_t* out;
  uint64_t* begin_targets[PSB_MAX_RANKS];   // every rank's signal pad (consistent=True) or all nullptr
  int32_t nbegin;
  uint32_t cand_mask;
  int32_t quota;
  uint64_t version;                          // the version the following update kernel will publish
  unsigned long long timeout_ns;
};

__global__ void psb_select_kernel(const __grid_constant__ SelectArgs a) {
  const uint64_t* signal_local = a.signal_local;
  uint64_t* consumed = a.consumed;
  uint64_t* out = a.out;
  const uint32_t cand_mask = a.cand_mask;
  const int quota = a.quota;
  const int t = threadIdx.x;   // one warp
  uint64_t* err = const_cast<uint64_t*>(signal_local) + SIG_ERROR;
  unsigned long long t0 = 0;
  uint32_t ready = 0, fin = 0;
  uint64_t e = 0;
  int need = 0;
  while (true) {
    const bool cand = cand_mask >> t & 1u;
    e = cand ? ld_acquire_sys(signal_local + SIG_GRAD_READY + t) : 0;
    const bool f = cand && e >= PSB_DONE_EPOCH;
    const bool r = cand && !f && e > consumed[t];
    ready = __ballot_sync(0xffffffffu, r);
    fin = __ballot_sync(0xffffffffu, f);
    need = min(quota, __popc(cand_mask & ~fin));
    if (need == 0 || __popc(ready) >= need) break;
    unsigned long long now;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(now));
    if (t0 == 0) t0 = now;
    bool bad = (now - t0 > a.timeout_ns) || ld_relaxed_sys_u64(err) != 0;
    if (__any_sync(0xffffffffu, bad)) {
      if (t == 0) {
        st_release_sys(err, 2ull);
        out[0] = 0;
        out[1] = 0;
        out[40] = fin;
      }
      return;
    }
    __nanosleep(200);
  }
  // rotating priority so no worker starves: start after the last served rank
  const int start = (int)(consumed[63] % 32);
  uint32_t chosen = 0;
  int cnt = 0;
  for (int i = 0; i < 32 && cnt < need; ++i) {
    const int r = (start + 1 + i) % 32;
    if (ready >> r & 1u) {
      chosen |= 1u << r;
      ++cnt;
    }
  }
  __syncwarp();
  if (chosen >> t & 1u) {
    consumed[t] = e;
    out[2 + t] = e;
    const uint64_t gv = ld_acquire_sys(signal_local + SIG_GRAD_VERSION + t);
    out[44 + t] = a.version - 1 >= gv ? a.version - 1 - gv : 0;
  }
  if (chosen != 0 && t < a.nbegin && a.begin_targets[t] != nullptr)
    st_release_sys(a.begin_targets[t] + SIG_STAGE_BEGIN, a.version);   // sequence lock: BEGIN(v) … stores … VERSION(v)
  if (t == 0) {
    if (chosen) consumed[63] = (uint64_t)(31 - __clz(chosen));
    out[0] = chosen;
    out[1] = (uint64_t)cnt;
    out[40] = fin;
    out[41] = a.version;
  }
}

// ------------------------------------------------------------------------------------------
// consistent reads (async, README.md:79-81 "a buffered broadcast"): device-side sequence-lock snapshot
// ------------------------------------------------------------------------------------------
// The server publishes version v into every rank's STAGING arena between SIG_STAGE_BEGIN = v and SIG_VERSION = v.
// A worker adopts whole versions only, with no host involvement:
//   psb_snapshot_fetch   every CTA: read BEGIN / VERSION; if they agree on a version newer than the adopted one, copy its
//                        slice staging → shadow and re-read BEGIN; any disagreement (publication in progress, torn copy,
//                        CTAs that saw different versions) vetoes.  The last CTA writes the verdict: status = v or 0.
//   psb_snapshot_commit  if status != 0: shadow → live parameter arena (purely local, the server never writes there), and the
//                        adopted version becomes v.  A vetoed attempt leaves the live parameters on the previous whole version.
struct SnapshotArgs {
  const uint64_t* signal_local;
  const uint4* stage;
  uint4* shadow;
  uint4* params;
  size_t nvec;                   // 16-byte vectors
  unsigned long long* scratch;   // [0] veto  [1] min version  [2] max version  [3] CTAs done  [4] status  [5] adopted version
};

__global__ void __launch_bounds__(256) psb_snapshot_fetch(const __grid_constant__ SnapshotArgs a) {
  __shared__ unsigned long long s_v;
  __shared__ int s_go;
  if (threadIdx.x == 0) {
    const uint64_t vb = ld_acquire_sys(a.signal_local + SIG_STAGE_BEGIN), ve = ld_acquire_sys(a.signal_local + SIG_VERSION);
    s_v = ve;
    s_go = (vb == ve) && (ve != a.scratch[5]) && (ve != 0);
  }
  __syncthreads();
  const unsigned long long v = s_v;
  bool veto = !s_go;
  if (s_go) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.nvec; i += (size_t)gridDim.x * blockDim.x)
      a.shadow[i] = ld_sys_v4(a.stage + i);       // coherent loads: the server's multimem.st / peer stores land here
    __syncthreads();
    if (threadIdx.x == 0) veto = ld_acquire_sys(a.signal_local + SIG_STAGE_BEGIN) != v;
  }
  if (threadIdx.x == 0) {
    if (veto) atomicOr(a.scratch + 0, 1ull);
    atomicMin(a.scratch + 1, v);
    atomicMax(a.scratch + 2, v);
    __threadfence();
    if (atomicAdd(a.scratch + 3, 1ull) == gridDim.x - 1) {
      __threadfence();
      const bool ok = a.scratch[0] == 0 && a.scratch[1] == a.scratch[2];
      a.scratch[4] = ok ? a.scratch[1] : 0ull;
      a.scratch[0] = 0, a.scratch[1] = ~0ull, a.scratch[2] = 0, a.scratch[3] = 0;
    }
  }
}

__global__ void __launch_bounds__(256) psb_snapshot_commit(const __grid_constant__ SnapshotArgs a) {
  const unsigned long long v = a.scratch[4];
  if (v == 0) return;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < a.nvec; i += (size_t)gridDim.x * blockDim.x)
    a.params[i] = a.shadow[i];
  if (blockIdx.x == 0 && threadIdx.x == 0) a.scratch[5] = v;     // stream-ordered: the next fetch reads it after this kernel
}

template <int KIND, int WIRE, int OPT>
void launch_update_t(cudaStream_t s, const UpdateArgs& a, int grid) {
  // (a variant with two P2P tiles in flight per thread and no state prefetch measured slower on the ResNet-18 arena at
  //  N = 1, and was removed)
  if (a.state_shift == 0) {
    psb_update_kernel<KIND, WIRE, OPT><<<grid, PSB_THREADS, 0, s>>>(a);
    return;
  }
  // compact optimizer state (mode='sharded'): the kernel indexes master / buf0-2 by arena element, so hand it those pointers
  // moved back by state_shift tiles — it only ever touches elements of tiles >= state_shift, i.e. the compact buffers.  A
  // shift applied to the pointers here costs the kernel nothing: an index shift inside it cost registers and spills.
  UpdateArgs b = a;
  const size_t d = (size_t)a.state_shift * PSB_TILE;
  if (b.master) b.master -= d;
  if (b.buf0) b.buf0 -= d;
  if (b.buf1) b.buf1 -= d;
  if (b.buf2) b.buf2 -= d;
  b.state_shift = 0;
  psb_update_kernel<KIND, WIRE, OPT><<<grid, PSB_THREADS, 0, s>>>(b);
}
template <int KIND, int WIRE>
void launch_update_o(cudaStream_t s, int opt, const UpdateArgs& a, int grid) {
  if (opt == OPT_SGD) launch_update_t<KIND, WIRE, OPT_SGD>(s, a, grid);
  else if (opt == OPT_ADAMW) launch_update_t<KIND, WIRE, OPT_ADAMW>(s, a, grid);
  else launch_update_t<KIND, WIRE, OPT_ADAM>(s, a, grid);
}

// ------------------------------------------------------------------------------------------
// exponential moving average of the weights (DESIGN.md, rule E1) and the publication of stored weights (ema_weights())
// ------------------------------------------------------------------------------------------
// One pass over the update launch's tiles, queued right behind it: it reads what the update wrote (the master, or the published
// parameter) and the compact fp32 average, and writes the average.  No peer access, no flag.  Padding lanes stay +0: the source
// is +0 there and the average starts from it.
__global__ void __launch_bounds__(PSB_THREADS) psb_ema_kernel(const __grid_constant__ EmaArgs a) {
  if (a.select_out != nullptr && a.select_out[1] == 0) return;   // async: nothing was applied, nothing is averaged
  const bool first = a.count != nullptr ? a.count[0] == 0 : a.first != 0;
  // torch's lerp_(w, a): fma(a, w - e, e) for a < 0.5, fma(a - 1, w - e, w) otherwise (a - 1 is exact there)
  const bool small = a.weight < 0.5f;
  const float wa = small ? a.weight : add_rn(a.weight, -1.f);
  for (int tile = a.tile_begin + blockIdx.x; tile < a.tile_end; tile += gridDim.x) {
    const size_t e0 = (size_t)tile * PSB_TILE + threadIdx.x * PSB_EPT;
    float w[PSB_EPT], e[PSB_EPT];
    if (a.master != nullptr) load8_local(a.master, DT_F32, e0, w);
    else load8_local(a.param, a.param_dt, e0, w);
    if (!first) {
      load8_local(a.ema, DT_F32, e0, e);
#pragma unroll
      for (int j = 0; j < PSB_EPT; ++j) w[j] = fma_rn(wa, add_rn(w[j], -e[j]), small ? e[j] : w[j]);
    }
    float4* ep = reinterpret_cast<float4*>(a.ema + e0);
    ep[0] = make_float4(w[0], w[1], w[2], w[3]);
    ep[1] = make_float4(w[4], w[5], w[6], w[7]);
  }
  if (a.count != nullptr) {
    // async: every CTA has read count[0] before it arrives here; the last one to arrive counts this average
    __shared__ int s_last;
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence();
      s_last = atomicAdd(a.count + 1, 1ull) == gridDim.x - 1;
    }
    __syncthreads();
    if (s_last && threadIdx.x == 0) {
      a.count[1] = 0;
      a.count[0] += 1;
    }
  }
}

__global__ void __launch_bounds__(PSB_THREADS) psb_publish_kernel(const __grid_constant__ PublishArgs a) {
  const int esz = a.param_dt == DT_F32 ? 4 : 2;
  for (int tile = a.tile_begin + blockIdx.x; tile < a.tile_end; tile += gridDim.x) {
    const size_t e0 = (size_t)tile * PSB_TILE + threadIdx.x * PSB_EPT;
    uint4 out[2];
    int nv;
    if (a.src_dt == a.param_dt) {   // the saved parameters: their bits, NaN payloads included
      const uint8_t* p = reinterpret_cast<const uint8_t*>(a.src) + e0 * esz;
      nv = esz == 4 ? 2 : 1;
      out[0] = ld_stream_v4(p);
      if (nv == 2) out[1] = ld_stream_v4(p + 16);
    } else {                        // the fp32 average, rounded once to the parameter dtype
      float f[PSB_EPT];
      load8_local(a.src, DT_F32, e0, f);
      nv = pack8(a.param_dt, f, out);
    }
    publish_packed(a.bcast, a.param_mc, a.param_dst, a.param_local, a.world, e0 * esz, out, nv);
  }
}

int small_grid(int tiles, int num_sms) { return std::max(1, std::min(tiles, num_sms * 8)); }

}  // namespace

// ------------------------------------------------------------------------------------------
// launchers
// ------------------------------------------------------------------------------------------
#include <atomic>
static std::atomic<unsigned long long> g_psb_launches{0};
void psb_count_launch(int n) { g_psb_launches.fetch_add((unsigned long long)n, std::memory_order_relaxed); }
unsigned long long psb_launch_count() { return g_psb_launches.load(std::memory_order_relaxed); }

void psb_launch_absmax(cudaStream_t s, const EncodeArgs& a) {
  const int ctas = a.batch.cum[a.batch.n];
  if (ctas > 0) {
    if (a.residual) psb_absmax_kernel<true><<<ctas, PSB_THREADS, 0, s>>>(a);
    else psb_absmax_kernel<false><<<ctas, PSB_THREADS, 0, s>>>(a);
    psb_count_launch(1);
  }
}

void psb_launch_accumulate(cudaStream_t s, const EncodeArgs& a) {
  const int ctas = a.batch.cum[a.batch.n];
  if (ctas > 0) {
    psb_accumulate_kernel<<<ctas, PSB_THREADS, 0, s>>>(a);
    psb_count_launch(1);
  }
}

void psb_launch_encode(cudaStream_t s, int kind, int wire, const EncodeArgs& a) {
  const int ctas = a.batch.cum[a.batch.n];
  if (ctas <= 0) return;
  psb_count_launch(1);
#define ENC(K, W)                                                     \
  if (kind == K && wire == W) {                                       \
    if constexpr (K != KIND_TOPK) {                                   \
      if (a.residual) {                                               \
        psb_encode_kernel<K, W, true><<<ctas, PSB_THREADS, 0, s>>>(a); \
        return;                                                       \
      }                                                               \
    }                                                                 \
    psb_encode_kernel<K, W, false><<<ctas, PSB_THREADS, 0, s>>>(a);   \
    return;                                                           \
  }
  ENC(KIND_DENSE, WIRE_F32) ENC(KIND_DENSE, WIRE_BF16) ENC(KIND_DENSE, WIRE_F16) ENC(KIND_DENSE, WIRE_E4M3)
  ENC(KIND_DENSE, WIRE_E5M2) ENC(KIND_SCALED, WIRE_I8) ENC(KIND_SCALED, WIRE_E4M3) ENC(KIND_SCALED, WIRE_E5M2)
  ENC(KIND_SCALED, WIRE_F16) ENC(KIND_TOPK, WIRE_F32) ENC(KIND_TOPK, WIRE_BF16)
  ENC(KIND_QSGD, WIRE_I8) ENC(KIND_QSGD, WIRE_I4) ENC(KIND_SIGN, WIRE_B1)
#undef ENC
}

void psb_launch_update(cudaStream_t s, int kind, int wire, int opt, const UpdateArgs& a, int grid) {
  psb_count_launch(1);
#define UPD(K, W)                                \
  if (kind == K && wire == W) {                  \
    launch_update_o<K, W>(s, opt, a, grid);      \
    return;                                      \
  }
  UPD(KIND_DENSE, WIRE_F32) UPD(KIND_DENSE, WIRE_BF16) UPD(KIND_DENSE, WIRE_F16) UPD(KIND_DENSE, WIRE_E4M3)
  UPD(KIND_DENSE, WIRE_E5M2) UPD(KIND_SCALED, WIRE_I8) UPD(KIND_SCALED, WIRE_E4M3) UPD(KIND_SCALED, WIRE_E5M2)
  UPD(KIND_SCALED, WIRE_F16) UPD(KIND_TOPK, WIRE_F32) UPD(KIND_TOPK, WIRE_BF16)
  UPD(KIND_QSGD, WIRE_I8) UPD(KIND_QSGD, WIRE_I4) UPD(KIND_SIGN, WIRE_B1)
#undef UPD
}

int psb_update_max_grid(int kind, int wire, int opt) {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  (void)kind, (void)wire, (void)opt;
  return sms * 3;   // __launch_bounds__(256, 3) for every (kind, wire, opt): all CTAs co-resident (the completion counter needs no more)
}

void psb_launch_ema(cudaStream_t s, const EmaArgs& a, int num_sms) {
  // the compact buffers are handed over moved back by state_shift tiles, as the update's state (launch_update_t)
  EmaArgs b = a;
  const size_t d = (size_t)a.state_shift * PSB_TILE;
  if (b.master) b.master -= d;
  b.ema -= d;
  b.state_shift = 0;
  psb_ema_kernel<<<small_grid(a.tile_end - a.tile_begin, num_sms), PSB_THREADS, 0, s>>>(b);
  psb_count_launch(1);
}

void psb_launch_publish(cudaStream_t s, const PublishArgs& a, int num_sms) {
  PublishArgs b = a;
  b.src = reinterpret_cast<const uint8_t*>(a.src) - (size_t)a.src_shift * PSB_TILE * (a.src_dt == DT_F32 ? 4 : 2);
  b.src_shift = 0;
  psb_publish_kernel<<<small_grid(a.tile_end - a.tile_begin, num_sms), PSB_THREADS, 0, s>>>(b);
  psb_count_launch(1);
}

void psb_launch_signal(cudaStream_t s, uint64_t* const* targets, int ntargets, int slot, uint64_t value,
                       uint64_t* extra_slot_base, int extra_slot, uint64_t extra_value, uint64_t* version_local,
                       int version_slot) {
  SignalArgs a{};
  a.n = ntargets;
  for (int i = 0; i < ntargets && i < PSB_MAX_RANKS; ++i) a.targets[i] = targets[i];
  a.slot = slot;
  a.value = value;
  a.extra_base = extra_slot_base;
  a.extra_slot = extra_slot;
  a.extra_value = extra_value;
  a.version_local = version_local;
  a.version_slot = version_slot;
  psb_signal_kernel<<<1, 32, 0, s>>>(a);
  psb_count_launch(1);
}

void psb_launch_signal_add(cudaStream_t s, uint64_t* const* targets, int ntargets, int slot, uint64_t value) {
  SignalArgs a{};
  a.n = ntargets;
  for (int i = 0; i < ntargets && i < PSB_MAX_RANKS; ++i) a.targets[i] = targets[i];
  a.slot = slot;
  a.value = value;
  a.add = 1;
  psb_signal_kernel<<<1, 32, 0, s>>>(a);
  psb_count_launch(1);
}

void psb_launch_snapshot(cudaStream_t s, const uint64_t* signal_local, const void* stage, void* shadow, void* params, size_t nbytes,
                         unsigned long long* scratch, int attempts, int num_sms) {
  SnapshotArgs a{};
  a.signal_local = signal_local;
  a.stage = reinterpret_cast<const uint4*>(stage);
  a.shadow = reinterpret_cast<uint4*>(shadow);
  a.params = reinterpret_cast<uint4*>(params);
  a.nvec = nbytes / 16;
  a.scratch = scratch;
  const int grid = (int)std::max<size_t>(1, std::min<size_t>((size_t)num_sms * 4, (a.nvec + 255) / 256));
  for (int i = 0; i < attempts; ++i) {
    psb_snapshot_fetch<<<grid, 256, 0, s>>>(a);
    psb_snapshot_commit<<<grid, 256, 0, s>>>(a);
    psb_count_launch(2);
  }
}

void psb_launch_wait(cudaStream_t s, const uint64_t* signal_local, int slot0, uint32_t mask, uint64_t want,
                     unsigned long long timeout_ns) {
  psb_wait_kernel<<<1, 32, 0, s>>>(signal_local, slot0, mask, want, timeout_ns);
  psb_count_launch(1);
}

void psb_launch_select(cudaStream_t s, const uint64_t* signal_local, uint64_t* consumed, uint32_t cand_mask,
                       int quota, uint64_t* out, unsigned long long timeout_ns, uint64_t version,
                       uint64_t* const* begin_targets, int nbegin) {
  SelectArgs a{};
  a.signal_local = signal_local;
  a.consumed = consumed;
  a.out = out;
  a.cand_mask = cand_mask;
  a.quota = quota;
  a.version = version;
  a.timeout_ns = timeout_ns;
  a.nbegin = nbegin;
  for (int i = 0; i < nbegin && i < PSB_MAX_RANKS; ++i) a.begin_targets[i] = begin_targets[i];
  psb_select_kernel<<<1, 32, 0, s>>>(a);
  psb_count_launch(1);
}
