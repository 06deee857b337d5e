// 3x3 / stride-2 / pad-1 max pooling for channels-last bf16 activations, forward + backward.
// ATen's max_pool_{forward,backward}_nhwc are slow for the ~0.6 GB of traffic of a ResNet-18 step; these move 16 bytes per thread,
// keep a 1-byte window position per output element for the backward, and the backward GATHERS
// (each input pixel looks at the <= 4 windows covering it) so it needs no atomics and writes dx once.
#include <cuda_bf16.h>

#include "kernels.h"

namespace {
using namespace psb;

struct PoolGeom {
  int N, H, W, C, OH, OW, groups;
};

__global__ void __launch_bounds__(256) psb_maxpool_fwd(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y,
                                                       uint8_t* __restrict__ arg, PoolGeom g) {
  const long long total = (long long)g.N * g.OH * g.OW * g.groups;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int cg = (int)(i % g.groups);
    long long p = i / g.groups;
    const int ow = (int)(p % g.OW);
    p /= g.OW;
    const int oh = (int)(p % g.OH);
    const int n = (int)(p / g.OH);
    float best[8];
    uint32_t pos[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) best[j] = -INFINITY, pos[j] = 255;
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
      const int h = oh * 2 - 1 + kh;
      if (h < 0 || h >= g.H) continue;
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const int w = ow * 2 - 1 + kw;
        if (w < 0 || w >= g.W) continue;
        float v[8];
        uint4 raw = *reinterpret_cast<const uint4*>(x + (((long long)n * g.H + h) * g.W + w) * g.C + cg * 8);
        unpack_bf16x8(raw, v);
#pragma unroll
        for (int j = 0; j < 8; ++j)
          if (v[j] > best[j]) {          // strictly greater: the first maximum wins ties (ATen's rule)
            best[j] = v[j];
            pos[j] = kh * 3 + kw;
          }
      }
    }
    const long long o = (((long long)n * g.OH + oh) * g.OW + ow) * g.C + cg * 8;
    *reinterpret_cast<uint4*>(y + o) = make_uint4(pack_bf16x2(best[0], best[1]), pack_bf16x2(best[2], best[3]),
                                                  pack_bf16x2(best[4], best[5]), pack_bf16x2(best[6], best[7]));
    *reinterpret_cast<uint2*>(arg + o) =
        make_uint2(pos[0] | (pos[1] << 8) | (pos[2] << 16) | (pos[3] << 24), pos[4] | (pos[5] << 8) | (pos[6] << 16) | (pos[7] << 24));
  }
}

__global__ void __launch_bounds__(256) psb_maxpool_bwd(const __nv_bfloat16* __restrict__ dy, const uint8_t* __restrict__ arg,
                                                       __nv_bfloat16* __restrict__ dx, PoolGeom g) {
  const long long total = (long long)g.N * g.H * g.W * g.groups;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int cg = (int)(i % g.groups);
    long long p = i / g.groups;
    const int w = (int)(p % g.W);
    p /= g.W;
    const int h = (int)(p % g.H);
    const int n = (int)(p / g.H);
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    // windows covering (h, w): oh*2-1 <= h <= oh*2+1
    const int oh0 = h >> 1 /* floor(h/2) covers h = 2oh or 2oh+1 */, ow0 = w >> 1;
#pragma unroll
    for (int a = 0; a < 2; ++a) {
      const int oh = oh0 + a;
      const int kh = h - (oh * 2 - 1);
      if (oh >= g.OH || kh < 0 || kh > 2) continue;
#pragma unroll
      for (int b = 0; b < 2; ++b) {
        const int ow = ow0 + b;
        const int kw = w - (ow * 2 - 1);
        if (ow >= g.OW || kw < 0 || kw > 2) continue;
        const long long o = (((long long)n * g.OH + oh) * g.OW + ow) * g.C + cg * 8;
        const uint2 pr = *reinterpret_cast<const uint2*>(arg + o);
        float d[8];
        uint4 raw = *reinterpret_cast<const uint4*>(dy + o);
        unpack_bf16x8(raw, d);
        const uint32_t want = (uint32_t)(kh * 3 + kw);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const uint32_t pj = ((j < 4 ? pr.x : pr.y) >> (8 * (j & 3))) & 0xffu;
          if (pj == want) acc[j] += d[j];
        }
      }
    }
    *reinterpret_cast<uint4*>(dx + (((long long)n * g.H + h) * g.W + w) * g.C + cg * 8) =
        make_uint4(pack_bf16x2(acc[0], acc[1]), pack_bf16x2(acc[2], acc[3]), pack_bf16x2(acc[4], acc[5]), pack_bf16x2(acc[6], acc[7]));
  }
}

// ---- row-based variants (round 2) -----------------------------------------------------------------------------------
// The kernels above spend most of their instructions on 64-bit div/mod index chains (one per 16 bytes).  Here a CTA walks whole rows with 32-bit
// indices; tx = channel group of 8, ty = pixel lane, so a warp covers 32 / groups consecutive NHWC pixels.
// (min-blocks 1: ptxas for sm_90a otherwise caps it at 40 registers and spills; it takes 48 without the cap)
__global__ void __launch_bounds__(256, 1) psb_maxpool_fwd_rows(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y,
                                                            uint8_t* __restrict__ arg, PoolGeom g, int lanes) {
  const int tx = threadIdx.x % g.groups, ty = threadIdx.x / g.groups;
  if (ty >= lanes) return;
  const int rows = g.N * g.OH;
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {
    const int n = row / g.OH, oh = row - n * g.OH;
    const int h0 = oh * 2 - 1;
    const __nv_bfloat16* xin = x + (size_t)n * g.H * g.W * g.C + tx * 8;
    for (int ow = ty; ow < g.OW; ow += lanes) {
      const int w0 = ow * 2 - 1;
      float best[8];
      uint32_t pos[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) best[j] = -INFINITY, pos[j] = 255;
#pragma unroll
      for (int kh = 0; kh < 3; ++kh) {
        const int h = h0 + kh;
        if (h < 0 || h >= g.H) continue;
#pragma unroll
        for (int kw = 0; kw < 3; ++kw) {
          const int w = w0 + kw;
          if (w < 0 || w >= g.W) continue;
          float v[8];
          unpack_bf16x8(*reinterpret_cast<const uint4*>(xin + ((size_t)h * g.W + w) * g.C), v);
#pragma unroll
          for (int j = 0; j < 8; ++j)
            if (v[j] > best[j]) {          // strictly greater: the first maximum wins ties (ATen's rule)
              best[j] = v[j];
              pos[j] = kh * 3 + kw;
            }
        }
      }
      const size_t o = ((size_t)row * g.OW + ow) * g.C + tx * 8;
      *reinterpret_cast<uint4*>(y + o) = make_uint4(pack_bf16x2(best[0], best[1]), pack_bf16x2(best[2], best[3]),
                                                    pack_bf16x2(best[4], best[5]), pack_bf16x2(best[6], best[7]));
      *reinterpret_cast<uint2*>(arg + o) = make_uint2(pos[0] | (pos[1] << 8) | (pos[2] << 16) | (pos[3] << 24),
                                                      pos[4] | (pos[5] << 8) | (pos[6] << 16) | (pos[7] << 24));
    }
  }
}

// Backward by 2x2 input QUADS (H, W even): the quad (h0..h0+1, w0..w0+1), h0 / w0 even, is covered by exactly the four windows
// (oh0 + a, ow0 + b), oh0 = h0/2, ow0 = w0/2, and the nine window taps that fall into the quad partition 0..8 —
// window (0,0): taps 4,5,7,8 → pixels (0,0),(0,1),(1,0),(1,1);  (0,1): taps 3,6 → (0,1),(1,1);  (1,0): taps 1,2 → (1,0),(1,1);
// (1,1): tap 0 → (1,1).  One thread: 4 x (arg 8 B + dy 16 B) in, 4 x 16 B of dx out, no branches on loaded data.
__global__ void __launch_bounds__(256) psb_maxpool_bwd_quads(const __nv_bfloat16* __restrict__ dy, const uint8_t* __restrict__ arg,
                                                             __nv_bfloat16* __restrict__ dx, PoolGeom g, int lanes) {
  const int tx = threadIdx.x % g.groups, ty = threadIdx.x / g.groups;
  if (ty >= lanes) return;
  const int hp = g.H >> 1, wq = g.W >> 1;
  const int rows = g.N * hp;
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {
    const int n = row / hp, oh0 = row - n * hp;
    const size_t on = (size_t)n * g.OH * g.OW * g.C + tx * 8;
    const size_t xbase = ((size_t)n * g.H + 2 * oh0) * g.W * g.C + tx * 8;
    for (int qd = ty; qd < wq; qd += lanes) {
      uint2 pr[4];
      uint4 dv[4];
#pragma unroll
      for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int b = 0; b < 2; ++b) {
          const int i = a * 2 + b;
          pr[i] = make_uint2(0xffffffffu, 0xffffffffu);          // tap 255 matches nothing
          dv[i] = make_uint4(0u, 0u, 0u, 0u);
          if (oh0 + a < g.OH && qd + b < g.OW) {
            const size_t o = on + ((size_t)(oh0 + a) * g.OW + (qd + b)) * g.C;
            pr[i] = *reinterpret_cast<const uint2*>(arg + o);
            dv[i] = *reinterpret_cast<const uint4*>(dy + o);
          }
        }
      float f[4][8], d[4][8];
#pragma unroll
      for (int i = 0; i < 4; ++i) unpack_bf16x8(dv[i], f[i]);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        uint32_t t[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) t[i] = ((j < 4 ? pr[i].x : pr[i].y) >> (8 * (j & 3))) & 0xffu;
        d[0][j] = (t[0] == 4u ? f[0][j] : 0.f);
        d[1][j] = (t[0] == 5u ? f[0][j] : 0.f) + (t[1] == 3u ? f[1][j] : 0.f);
        d[2][j] = (t[0] == 7u ? f[0][j] : 0.f) + (t[2] == 1u ? f[2][j] : 0.f);
        d[3][j] = (t[0] == 8u ? f[0][j] : 0.f) + (t[1] == 6u ? f[1][j] : 0.f) + (t[2] == 2u ? f[2][j] : 0.f) +
                  (t[3] == 0u ? f[3][j] : 0.f);
      }
#pragma unroll
      for (int p = 0; p < 4; ++p)
        *reinterpret_cast<uint4*>(dx + xbase + ((size_t)(p >> 1) * g.W + 2 * qd + (p & 1)) * g.C) =
            make_uint4(pack_bf16x2(d[p][0], d[p][1]), pack_bf16x2(d[p][2], d[p][3]), pack_bf16x2(d[p][4], d[p][5]),
                       pack_bf16x2(d[p][6], d[p][7]));
    }
  }
}

int pool_grid(long long total) {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  long long want = (total + 255) / 256;
  long long cap = (long long)sms * 16;
  return (int)(want < cap ? (want > 0 ? want : 1) : cap);
}

}  // namespace

void psb_maxpool3x3s2_forward(cudaStream_t s, const void* x, void* y, void* arg, int N, int H, int W, int C) {
  psb_count_launch(1);
  PoolGeom g{N, H, W, C, (H + 2 - 3) / 2 + 1, (W + 2 - 3) / 2 + 1, C / 8};
  const long long total = (long long)N * g.OH * g.OW * g.groups;
  if (g.groups <= 256 && 256 % g.groups == 0) {       // row-based kernel (channel groups tile the CTA)
    const int lanes = 256 / g.groups, rows = N * g.OH, cap = pool_grid(total);
    psb_maxpool_fwd_rows<<<rows < cap ? rows : cap, 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(x),
                                                                   reinterpret_cast<__nv_bfloat16*>(y), reinterpret_cast<uint8_t*>(arg),
                                                                   g, lanes);
    return;
  }
  psb_maxpool_fwd<<<pool_grid(total), 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(x), reinterpret_cast<__nv_bfloat16*>(y),
                                                   reinterpret_cast<uint8_t*>(arg), g);
}

void psb_maxpool3x3s2_backward(cudaStream_t s, const void* dy, const void* arg, void* dx, int N, int H, int W, int C) {
  psb_count_launch(1);
  PoolGeom g{N, H, W, C, (H + 2 - 3) / 2 + 1, (W + 2 - 3) / 2 + 1, C / 8};
  const long long total = (long long)N * H * W * g.groups;
  if (H % 2 == 0 && W % 2 == 0 && g.groups <= 256 && 256 % g.groups == 0) {   // quad-based kernel
    const int lanes = 256 / g.groups, rows = N * (H / 2), cap = pool_grid(total / 4);
    psb_maxpool_bwd_quads<<<rows < cap ? rows : cap, 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(dy),
                                                                    reinterpret_cast<const uint8_t*>(arg),
                                                                    reinterpret_cast<__nv_bfloat16*>(dx), g, lanes);
    return;
  }
  psb_maxpool_bwd<<<pool_grid(total), 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(dy), reinterpret_cast<const uint8_t*>(arg),
                                                   reinterpret_cast<__nv_bfloat16*>(dx), g);
}

// ---- input pre-processing: uint8 NCHW image → normalised bf16 NHWC padded to 8 channels --------------
// One pass instead of ATen's float() / sub / div / to(bf16) / contiguous(channels_last) chain, and the
// 8-channel (16-byte) pixel lets cuDNN run the 7x7 stem convolution on its aligned tensor-core kernels
// (C=3 defeats them).
namespace {
__global__ void __launch_bounds__(256) psb_normalize_pad8(const uint8_t* __restrict__ x, __nv_bfloat16* __restrict__ y,
                                                          float m0, float m1, float m2, float s0, float s1, float s2, int N,
                                                          long long HW) {
  const long long total = (long long)N * HW;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long n = i / HW, p = i % HW;
    const uint8_t* base = x + n * 3 * HW + p;
    const float a = ((float)base[0] - m0) * s0, b = ((float)base[HW] - m1) * s1, c = ((float)base[2 * HW] - m2) * s2;
    *reinterpret_cast<uint4*>(y + i * 8) = make_uint4(psb::pack_bf16x2(a, b), psb::pack_bf16x2(c, 0.f), 0u, 0u);
  }
}
}  // namespace

void psb_normalize_pad8_launch(cudaStream_t s, const void* x, void* y, const float* mean, const float* inv_std, int N, long long HW) {
  psb_count_launch(1);
  const long long total = (long long)N * HW;
  psb_normalize_pad8<<<pool_grid(total), 256, 0, s>>>(reinterpret_cast<const uint8_t*>(x), reinterpret_cast<__nv_bfloat16*>(y),
                                                      mean[0], mean[1], mean[2], inv_std[0], inv_std[1], inv_std[2], N, HW);
}

// ---- ResNet stem as an implicit GEMM on OUR wgmma kernel -----------------------------------------------
// cuDNN's 7x7/stride-2 convolution with 3 input channels cannot use its tensor-core paths (C=3).  We lower it
// ourselves: psb_im2col_stem writes the
// [N*OH*OW, 176] patch matrix (7 kernel rows x (21 real + 3 zero) columns + 8 zero columns), the forward
// is psb_bcast_gemm (wgmma/TMA) against the matching [64,176] weight matrix and lands
// directly in NHWC, and the weight gradient is one library GEMM dY^T · A.
namespace {
constexpr int STEM_K = 176;   // 7 kernel rows x 24 (21 = 7*3 real + 3 zero, so every row starts 16-byte aligned) + 8 pad → 11 wgmma K steps

// One thread = one (output pixel, kernel row): the 21 input values x[n, ih, iw0..iw0+6, 0..2] are CONTIGUOUS
// in NHWC memory (42 bytes, always 2-mod-4 aligned because iw0 = 2*ow - 3 is odd), so they are fetched with
// one 2-byte and ten 4-byte loads and written as three 16-byte stores (plus the 16-byte zero tail by kh == 6).
__global__ void __launch_bounds__(256) psb_im2col_stem(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ a,
                                                       int N, int H, int W, int OH, int OW) {
  const long long total = (long long)N * OH * OW * 7;
  const unsigned short* xs = reinterpret_cast<const unsigned short*>(x);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int kh = (int)(i % 7);
    long long p = i / 7;
    const long long row = p;
    const int ow = (int)(p % OW);
    p /= OW;
    const int oh = (int)(p % OH);
    const int n = (int)(p / OH);
    const int ih = oh * 2 - 3 + kh, iw0 = ow * 2 - 3;
    uint32_t v[12];
#pragma unroll
    for (int j = 0; j < 12; ++j) v[j] = 0u;
    if (ih >= 0 && ih < H) {
      const unsigned short* src = xs + (((long long)n * H + ih) * W) * 3;   // row start; element e of the window = src[iw0*3 + e]
      if (iw0 >= 0 && iw0 + 7 <= W) {
        const unsigned short* q = src + (long long)iw0 * 3;                // 2-mod-4 byte aligned
        const uint32_t first = q[0];
        const uint32_t* q4 = reinterpret_cast<const uint32_t*>(q + 1);      // 4-byte aligned
        uint32_t w4[10];
#pragma unroll
        for (int j = 0; j < 10; ++j) w4[j] = q4[j];
        // element e: e=0 → first; e=2j+1, 2j+2 → w4[j] low / high
        v[0] = first | (w4[0] << 16);
#pragma unroll
        for (int j = 1; j < 10; ++j) v[j] = (w4[j - 1] >> 16) | (w4[j] << 16);
        v[10] = (w4[9] >> 16);                                              // element 20, then zero
      } else {
#pragma unroll
        for (int e = 0; e < 21; ++e) {
          const int iw = iw0 + e / 3;
          const uint32_t val = (iw >= 0 && iw < W) ? xs[(((long long)n * H + ih) * W + iw) * 3 + (e % 3)] : 0u;
          v[e >> 1] |= val << (16 * (e & 1));
        }
      }
    }
    uint4* dst = reinterpret_cast<uint4*>(a + row * STEM_K + kh * 24);
    dst[0] = make_uint4(v[0], v[1], v[2], v[3]);
    dst[1] = make_uint4(v[4], v[5], v[6], v[7]);
    dst[2] = make_uint4(v[8], v[9], v[10], v[11]);
    if (kh == 6) dst[3] = make_uint4(0u, 0u, 0u, 0u);                       // columns 168..175
  }
}

// uint8 NCHW image → normalised bf16 NHWC (3 channels), one pass
__global__ void __launch_bounds__(256) psb_normalize_nhwc3(const uint8_t* __restrict__ x, __nv_bfloat16* __restrict__ y, float m0,
                                                           float m1, float m2, float s0, float s1, float s2, int N, long long HW) {
  const long long total = (long long)N * HW;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long n = i / HW, p = i % HW;
    const uint8_t* base = x + n * 3 * HW + p;
    y[i * 3 + 0] = __float2bfloat16_rn(((float)base[0] - m0) * s0);
    y[i * 3 + 1] = __float2bfloat16_rn(((float)base[HW] - m1) * s1);
    y[i * 3 + 2] = __float2bfloat16_rn(((float)base[2 * HW] - m2) * s2);
  }
}
}  // namespace

void psb_im2col_stem_launch(cudaStream_t s, const void* x, void* a, int N, int H, int W) {
  psb_count_launch(1);
  const int OH = (H + 6 - 7) / 2 + 1, OW = (W + 6 - 7) / 2 + 1;
  const long long total = (long long)N * OH * OW * 7;
  psb_im2col_stem<<<pool_grid(total), 256, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(x), reinterpret_cast<__nv_bfloat16*>(a), N,
                                                   H, W, OH, OW);
}

void psb_normalize_nhwc3_launch(cudaStream_t s, const void* x, void* y, const float* mean, const float* inv_std, int N, long long HW) {
  psb_count_launch(1);
  const long long total = (long long)N * HW;
  psb_normalize_nhwc3<<<pool_grid(total), 256, 0, s>>>(reinterpret_cast<const uint8_t*>(x), reinterpret_cast<__nv_bfloat16*>(y),
                                                       mean[0], mean[1], mean[2], inv_std[0], inv_std[1], inv_std[2], N, HW);
}
