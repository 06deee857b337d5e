// Fused training BatchNorm for channels-last (NHWC) bf16 activations on sm_90a.
//
// Why it exists: ATen's channels-last BatchNorm + the separate add / ReLU kernels are a large share of a
// ResNet-18 step and make 5-6 HBM passes.  BatchNorm is pure HBM traffic, so the framework ships its own:
//   forward : psb_bn_stats   (1 read of x, fp32 sum / sum-of-squares per channel)
//             psb_bn_finalize (C threads: mean, rstd, running stats, fused scale/shift)
//             psb_bn_apply   (read x [+ residual] → y = act(x*scale + shift [+ residual]), 1 write)
//   backward: psb_bn_bwd_reduce (read dy, x, y → Σdy', Σdy'·x̂ with the ReLU mask folded in)
//             psb_bn_bwd_finalize
//             psb_bn_bwd_apply  (write dx and, for residual blocks, the masked skip gradient)
// Every pass moves 16 bytes per thread, a warp touches 512 contiguous bytes, accumulation is fp32.
#include <cuda_bf16.h>

#include "kernels.h"

namespace {
using namespace psb;

constexpr int BN_THREADS = 256;

struct BnGeom {
  long long pixels;   // N*H*W
  int C;              // channels (multiple of 8)
  int groups;         // C / 8
  int lanes;          // BN_THREADS / groups  (pixels processed in parallel by a CTA)
};

__device__ __forceinline__ void ld8(const __nv_bfloat16* p, float* f) {
  uint4 v = *reinterpret_cast<const uint4*>(p);
  unpack_bf16x8(v, f);
}
__device__ __forceinline__ void ld8_stream(const __nv_bfloat16* p, float* f) {
  uint4 v = ld_stream_v4(p);
  unpack_bf16x8(v, f);
}
__device__ __forceinline__ void st8(__nv_bfloat16* p, const float* f) {
  *reinterpret_cast<uint4*>(p) = make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]),
                                             pack_bf16x2(f[6], f[7]));
}

// Block-level reduction of per-thread 8-channel partials over the pixel lanes, then one plain store per channel into this
// CTA's row of the partials (no atomics: the finalize kernels add the rows in CTA order, so every run sums in the same order
// and gets the same bits).  smem layout: [lanes][C] floats.
__device__ __forceinline__ void reduce_lanes(float* smem, const float* part, int tx, int ty, const BnGeom& g, float* out) {
  if (ty < g.lanes) {   // threads beyond lanes*groups (C/8 not dividing 256) hold no partials
    float4* row = reinterpret_cast<float4*>(smem + (size_t)ty * g.C + tx * 8);
    row[0] = make_float4(part[0], part[1], part[2], part[3]);
    row[1] = make_float4(part[4], part[5], part[6], part[7]);
  }
  __syncthreads();
  for (int c = threadIdx.x; c < g.C; c += BN_THREADS) {
    float s = 0.f;
    for (int l = 0; l < g.lanes; ++l) s += smem[(size_t)l * g.C + c];
    out[c] = s;
  }
  __syncthreads();
}

// ---- forward ------------------------------------------------------------------------------
__global__ void __launch_bounds__(BN_THREADS) psb_bn_stats(const __nv_bfloat16* __restrict__ x, float* __restrict__ part,
                                                            BnGeom g) {
  extern __shared__ float smem[];
  const int tx = threadIdx.x % g.groups, ty = threadIdx.x / g.groups;
  float s[8], q[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) s[j] = q[j] = 0.f;
  const long long per_cta = (g.pixels + gridDim.x - 1) / gridDim.x;
  const long long p0 = (long long)blockIdx.x * per_cta;
  const long long p1 = p0 + per_cta < g.pixels ? p0 + per_cta : g.pixels;
  if (ty < g.lanes) {
    long long p = p0 + ty;
    for (; p + 3LL * g.lanes < p1; p += 4LL * g.lanes) {   // 4 independent 16-byte loads in flight
      float a[4][8];
#pragma unroll
      for (int u = 0; u < 4; ++u) ld8_stream(x + (p + (long long)u * g.lanes) * g.C + tx * 8, a[u]);
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          s[j] += a[u][j];
          q[j] = fmaf(a[u][j], a[u][j], q[j]);
        }
    }
    for (; p < p1; p += g.lanes) {
      float a[8];
      ld8_stream(x + p * g.C + tx * 8, a);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        s[j] += a[j];
        q[j] = fmaf(a[j], a[j], q[j]);
      }
    }
  }
  reduce_lanes(smem, s, tx, ty, g, part + (size_t)blockIdx.x * 2 * g.C);
  reduce_lanes(smem, q, tx, ty, g, part + (size_t)blockIdx.x * 2 * g.C + g.C);
}

// Σ over `nparts` rows of per-CTA partials [nparts][2C] for the block's FIN_CH channels, in a fixed order: slice i adds rows
// i, i + FIN_SLICES, ... and thread 0 of each channel adds the slices in order.  Returns false on threads that hold no result.
// A slice loads FIN_BATCH of its rows before it adds them (in the same order): the grid is only C / FIN_CH CTAs, so one load
// in flight per thread left these kernels waiting on L2 latency for up to 132 rows (~21 us each on H100).
constexpr int FIN_CH = 32, FIN_SLICES = 8, FIN_THREADS = FIN_CH * FIN_SLICES, FIN_BATCH = 16;
__device__ __forceinline__ bool sum_partials(const float* __restrict__ part, int nparts, int C, float& s, float& q, int& c) {
  __shared__ float red[2][FIN_SLICES][FIN_CH];
  const int cl = threadIdx.x % FIN_CH, sl = threadIdx.x / FIN_CH;
  c = blockIdx.x * FIN_CH + cl;
  s = 0.f, q = 0.f;
  if (c < C)
    for (int b0 = sl; b0 < nparts; b0 += FIN_SLICES * FIN_BATCH) {
      float vs[FIN_BATCH], vq[FIN_BATCH];
#pragma unroll
      for (int u = 0; u < FIN_BATCH; ++u) {
        const int b = b0 + u * FIN_SLICES;
        vs[u] = b < nparts ? part[(size_t)b * 2 * C + c] : 0.f;
        vq[u] = b < nparts ? part[(size_t)b * 2 * C + C + c] : 0.f;
      }
#pragma unroll
      for (int u = 0; u < FIN_BATCH; ++u)
        if (b0 + u * FIN_SLICES < nparts) s += vs[u], q += vq[u];
    }
  red[0][sl][cl] = s;
  red[1][sl][cl] = q;
  __syncthreads();
  if (sl != 0 || c >= C) return false;
  s = 0.f, q = 0.f;
  for (int i = 0; i < FIN_SLICES; ++i) s += red[0][i][cl], q += red[1][i][cl];
  return true;
}

// partials of Σx | Σx² → mean/rstd (saved for backward), running stats, fused scale/shift
__global__ void __launch_bounds__(FIN_THREADS) psb_bn_finalize(const float* __restrict__ part, int nparts,
                                                                const __nv_bfloat16* __restrict__ gamma,
                                                                const __nv_bfloat16* __restrict__ beta, float* __restrict__ mean,
                                                                float* __restrict__ rstd, float* __restrict__ scale,
                                                                float* __restrict__ shift, float* running_mean, float* running_var,
                                                                int C, long long pixels, float eps, float momentum) {
  float sx, sxx;
  int c;
  if (!sum_partials(part, nparts, C, sx, sxx, c)) return;
  const float inv_n = 1.f / (float)pixels;
  const float m = sx * inv_n;
  float var = fmaf(-m, m, sxx * inv_n);
  var = fmaxf(var, 0.f);
  const float r = rsqrtf(var + eps);
  mean[c] = m;
  rstd[c] = r;
  const float gsc = gamma ? __bfloat162float(gamma[c]) : 1.f;
  const float b = beta ? __bfloat162float(beta[c]) : 0.f;
  scale[c] = gsc * r;
  shift[c] = fmaf(-m, gsc * r, b);
  if (running_mean) {
    const float unbiased = pixels > 1 ? var * (float)pixels / (float)(pixels - 1) : var;
    running_mean[c] = fmaf(momentum, m - running_mean[c], running_mean[c]);
    running_var[c] = fmaf(momentum, unbiased - running_var[c], running_var[c]);
  }
}

template <bool RES, bool RELU>
__global__ void __launch_bounds__(BN_THREADS) psb_bn_apply(const __nv_bfloat16* __restrict__ x,
                                                            const __nv_bfloat16* __restrict__ res,
                                                            const float* __restrict__ scale, const float* __restrict__ shift,
                                                            __nv_bfloat16* __restrict__ y, uint8_t* __restrict__ mask, BnGeom g) {
  // `mask` (RELU, training): one bit per element, y > 0 — the backward reads this 1/16-size tensor instead of y
  const int tx = threadIdx.x % g.groups, ty = threadIdx.x / g.groups;
  if (ty >= g.lanes) return;
  float sc[8], sh[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    sc[j] = scale[tx * 8 + j];
    sh[j] = shift[tx * 8 + j];
  }
  const long long stride = (long long)gridDim.x * g.lanes;
  for (long long p = (long long)blockIdx.x * g.lanes + ty; p < g.pixels; p += stride) {
    const long long off = p * g.C + tx * 8;
    float a[8], r[8];
    ld8_stream(x + off, a);
    if (RES) ld8_stream(res + off, r);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float v = fmaf(a[j], sc[j], sh[j]);
      if (RES) v += r[j];
      if (RELU) v = fmaxf(v, 0.f);
      a[j] = v;
    }
    st8(y + off, a);
    if (RELU && mask != nullptr) {
      uint32_t m = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) m |= (__bfloat162float(__float2bfloat16_rn(a[j])) > 0.f ? 1u : 0u) << j;
      mask[p * g.groups + tx] = (uint8_t)m;
    }
  }
}

// ---- backward -----------------------------------------------------------------------------
// ReLU mask of 8 consecutive channels: from the 1-bit mask tensor (MASKED) or from the saved output y
template <bool MASKED>
__device__ __forceinline__ uint32_t relu_bits(const __nv_bfloat16* __restrict__ y, const uint8_t* __restrict__ mask, long long p,
                                              long long off, int groups, int tx) {
  if (MASKED) return mask[p * groups + tx];
  float o[8];
  ld8_stream(y + off, o);
  uint32_t m = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) m |= (o[j] > 0.f ? 1u : 0u) << j;
  return m;
}

template <bool RELU, bool MASKED>
__global__ void __launch_bounds__(BN_THREADS) psb_bn_bwd_reduce(const __nv_bfloat16* __restrict__ dy,
                                                                 const __nv_bfloat16* __restrict__ x,
                                                                 const __nv_bfloat16* __restrict__ y,
                                                                 const uint8_t* __restrict__ mask,
                                                                 const float* __restrict__ mean, const float* __restrict__ rstd,
                                                                 float* __restrict__ part, BnGeom g) {
  extern __shared__ float smem[];
  const int tx = threadIdx.x % g.groups, ty = threadIdx.x / g.groups;
  float s[8], q[8], mu[8], rs[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    s[j] = q[j] = 0.f;
    mu[j] = mean[tx * 8 + j];
    rs[j] = rstd[tx * 8 + j];
  }
  const long long per_cta = (g.pixels + gridDim.x - 1) / gridDim.x;
  const long long p0 = (long long)blockIdx.x * per_cta;
  const long long p1 = p0 + per_cta < g.pixels ? p0 + per_cta : g.pixels;
  if (ty < g.lanes) {
    long long p = p0 + ty;
    for (; p + (long long)g.lanes < p1; p += 2LL * g.lanes) {
      float d[2][8], a[2][8];
      uint32_t mk[2] = {0xffu, 0xffu};
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const long long pp = p + (long long)u * g.lanes;
        const long long off = pp * g.C + tx * 8;
        ld8_stream(dy + off, d[u]);
        ld8_stream(x + off, a[u]);
        if (RELU) mk[u] = relu_bits<MASKED>(y, mask, pp, off, g.groups, tx);
      }
#pragma unroll
      for (int u = 0; u < 2; ++u)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float dd = (RELU && !(mk[u] >> j & 1u)) ? 0.f : d[u][j];
          s[j] += dd;
          q[j] = fmaf(dd, (a[u][j] - mu[j]) * rs[j], q[j]);
        }
    }
    for (; p < p1; p += g.lanes) {
      const long long off = p * g.C + tx * 8;
      float d[8], a[8];
      ld8_stream(dy + off, d);
      ld8_stream(x + off, a);
      const uint32_t mk = RELU ? relu_bits<MASKED>(y, mask, p, off, g.groups, tx) : 0xffu;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float dd = (RELU && !(mk >> j & 1u)) ? 0.f : d[j];
        s[j] += dd;
        q[j] = fmaf(dd, (a[j] - mu[j]) * rs[j], q[j]);
      }
    }
  }
  reduce_lanes(smem, s, tx, ty, g, part + (size_t)blockIdx.x * 2 * g.C);
  reduce_lanes(smem, q, tx, ty, g, part + (size_t)blockIdx.x * 2 * g.C + g.C);
}

// dx = gamma*rstd * (dy' - mean(dy') - x̂ * mean(dy'·x̂))  =  dy'*a + x*b + c   per channel
__global__ void __launch_bounds__(FIN_THREADS) psb_bn_bwd_finalize(const float* __restrict__ part, int nparts,
                                                                    const __nv_bfloat16* __restrict__ gamma,
                                                                    const float* __restrict__ mean, const float* __restrict__ rstd,
                                                                    float* __restrict__ ca, float* __restrict__ cb,
                                                                    float* __restrict__ cc, __nv_bfloat16* __restrict__ dgamma,
                                                                    __nv_bfloat16* __restrict__ dbeta, int C, long long pixels) {
  float sdy, sdyx;
  int c;
  if (!sum_partials(part, nparts, C, sdy, sdyx, c)) return;
  const float inv_n = 1.f / (float)pixels;
  const float g = gamma ? __bfloat162float(gamma[c]) : 1.f;
  const float r = rstd[c], m = mean[c];
  const float a = g * r;
  const float k = sdyx * inv_n * r;           // coefficient of (x - m)
  ca[c] = a;
  cb[c] = -a * k;
  cc[c] = a * (k * m - sdy * inv_n);
  if (dgamma) dgamma[c] = __float2bfloat16_rn(sdyx);
  if (dbeta) dbeta[c] = __float2bfloat16_rn(sdy);
}

template <bool RES, bool RELU, bool MASKED>
__global__ void __launch_bounds__(BN_THREADS) psb_bn_bwd_apply(const __nv_bfloat16* __restrict__ dy,
                                                                const __nv_bfloat16* __restrict__ x,
                                                                const __nv_bfloat16* __restrict__ y,
                                                                const uint8_t* __restrict__ mask, const float* __restrict__ ca,
                                                                const float* __restrict__ cb, const float* __restrict__ cc,
                                                                __nv_bfloat16* __restrict__ dx, __nv_bfloat16* __restrict__ dres,
                                                                BnGeom g) {
  const int tx = threadIdx.x % g.groups, ty = threadIdx.x / g.groups;
  if (ty >= g.lanes) return;
  float a[8], b[8], c[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    a[j] = ca[tx * 8 + j];
    b[j] = cb[tx * 8 + j];
    c[j] = cc[tx * 8 + j];
  }
  const long long stride = (long long)gridDim.x * g.lanes;
  for (long long p = (long long)blockIdx.x * g.lanes + ty; p < g.pixels; p += stride) {
    const long long off = p * g.C + tx * 8;
    float d[8], xv[8];
    ld8_stream(dy + off, d);
    ld8_stream(x + off, xv);
    const uint32_t mk = RELU ? relu_bits<MASKED>(y, mask, p, off, g.groups, tx) : 0xffu;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      if (RELU && !(mk >> j & 1u)) d[j] = 0.f;
      xv[j] = fmaf(d[j], a[j], fmaf(xv[j], b[j], c[j]));
    }
    st8(dx + off, xv);
    if (RES) st8(dres + off, d);
  }
}

// ---- ResNet stem tail: BatchNorm + ReLU + 3x3/s2/p1 max-pool (training, H and W even) -------------------------------------
// The unfused chain writes the full-resolution BN output y only for the pool to read it, and the pool backward writes the
// full-resolution gradient only for the BN backward to read it.  Here the forward pools straight from x, and both backward
// passes gather the pooled gradient themselves, so neither tensor exists.  (Round 2 had a fused forward that gathered per output
// pixel and was deleted because it lost to the unfused kernels; what is different now: the backward, which moves most of the
// bytes, is fused too, and the forward walks rows like psb_maxpool_fwd_rows.)  Every value is bit-identical to the unfused chain:
// the taps are rounded to bf16 exactly as psb_bn_apply stores them, the pool's rule picks the maximum, and the gather forms
// each pixel's gradient with psb_maxpool_bwd_quads' expression.  A window whose maximum is not > 0 stores tap 255 ("routes
// nothing") in place of the ReLU mask: in the unfused chain its gradient lands on a pixel whose mask bit is 0.
struct TailGeom {
  int N, H, W, OH, OW;   // input (even H, W) and pooled extents
};

__global__ void __launch_bounds__(BN_THREADS, 1) psb_bn_relu_maxpool_fwd(const __nv_bfloat16* __restrict__ x,
                                                                          const float* __restrict__ scale,
                                                                          const float* __restrict__ shift,
                                                                          __nv_bfloat16* __restrict__ y, uint8_t* __restrict__ arg,
                                                                          BnGeom g, TailGeom t) {
  const int tx = threadIdx.x % g.groups, ty = threadIdx.x / g.groups;
  if (ty >= g.lanes) return;
  float sc[8], sh[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    sc[j] = scale[tx * 8 + j];
    sh[j] = shift[tx * 8 + j];
  }
  const int rows = t.N * t.OH;
  for (int row = blockIdx.x; row < rows; row += gridDim.x) {   // one pooled row per CTA: L1 / L2 absorb the window overlap
    const int n = row / t.OH, oh = row - n * t.OH;
    const int h0 = oh * 2 - 1;
    const __nv_bfloat16* xin = x + (size_t)n * t.H * t.W * g.C + tx * 8;
    for (int ow = ty; ow < t.OW; ow += g.lanes) {
      const int w0 = ow * 2 - 1;
      float best[8];
      uint32_t pos[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) best[j] = -INFINITY, pos[j] = 255;
#pragma unroll
      for (int kh = 0; kh < 3; ++kh) {
        const int h = h0 + kh;
        if (h < 0 || h >= t.H) continue;
#pragma unroll
        for (int kw = 0; kw < 3; ++kw) {
          const int w = w0 + kw;
          if (w < 0 || w >= t.W) continue;
          float v[8];
          ld8(xin + ((size_t)h * t.W + w) * g.C, v);
#pragma unroll
          for (int j = 0; j < 8; ++j) v[j] = fmaxf(fmaf(v[j], sc[j], sh[j]), 0.f);   // psb_bn_apply<false, true>
          unpack_bf16x8(make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]),
                                   pack_bf16x2(v[6], v[7])), v);                          // the bf16 value y would hold
#pragma unroll
          for (int j = 0; j < 8; ++j)
            if (v[j] > best[j]) {          // strictly greater: the first maximum wins ties (psb_maxpool_fwd_rows)
              best[j] = v[j];
              pos[j] = kh * 3 + kw;
            }
        }
      }
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (!(best[j] > 0.f)) pos[j] = 255;
      const size_t o = ((size_t)row * t.OW + ow) * g.C + tx * 8;
      st8(y + o, best);
      *reinterpret_cast<uint2*>(arg + o) = make_uint2(pos[0] | (pos[1] << 8) | (pos[2] << 16) | (pos[3] << 24),
                                                      pos[4] | (pos[5] << 8) | (pos[6] << 16) | (pos[7] << 24));
    }
  }
}

// The masked BN-input gradient dy' of 8 channels at input pixel p, gathered from the pooled gradient `dp` and the forward's taps:
// what psb_maxpool_bwd_quads writes for this pixel's position in its 2x2 quad, same terms in the same order, rounded to bf16.
// Window (a, b) of the quad's four (oh0 + a, ow0 + b) covers the pixel at (ph, pw) iff a <= ph and b <= pw, with tap
// (ph + 1 - 2a) * 3 + (pw + 1 - 2b).
__device__ __forceinline__ void pooled_grad8(const __nv_bfloat16* __restrict__ dp, const uint8_t* __restrict__ arg, int p, int C,
                                             int tx, const TailGeom& t, float* d) {
  const int w = p % t.W, nh = p / t.W, h = nh % t.H, n = nh / t.H;
  const int ph = h & 1, pw = w & 1, oh0 = h >> 1, ow0 = w >> 1;
  uint2 pr[4];
  float f[4][8];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int a = i >> 1, b = i & 1;
    pr[i] = make_uint2(0xffffffffu, 0xffffffffu);          // tap 255 matches nothing
    uint4 dv = make_uint4(0u, 0u, 0u, 0u);
    if (a <= ph && b <= pw && oh0 + a < t.OH && ow0 + b < t.OW) {
      const size_t o = (((size_t)n * t.OH + oh0 + a) * t.OW + ow0 + b) * C + tx * 8;
      pr[i] = *reinterpret_cast<const uint2*>(arg + o);
      dv = *reinterpret_cast<const uint4*>(dp + o);
    }
    unpack_bf16x8(dv, f[i]);
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    float acc = 0.f;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int a = i >> 1, b = i & 1;
      if (a > ph || b > pw) continue;
      const uint32_t tap = ((j < 4 ? pr[i].x : pr[i].y) >> (8 * (j & 3))) & 0xffu;
      const float v = tap == (uint32_t)((ph + 1 - 2 * a) * 3 + (pw + 1 - 2 * b)) ? f[i][j] : 0.f;
      acc = i == 0 ? v : acc + v;
    }
    d[j] = acc;
  }
  unpack_bf16x8(make_uint4(pack_bf16x2(d[0], d[1]), pack_bf16x2(d[2], d[3]), pack_bf16x2(d[4], d[5]), pack_bf16x2(d[6], d[7])),
                d);
}

// psb_bn_bwd_reduce<true, true> with the dy load and the mask test replaced by pooled_grad8: the same CTA ranges, lanes and
// per-thread pixel order, so every partial sum adds the same values in the same order
__global__ void __launch_bounds__(BN_THREADS, 3) psb_bn_relu_maxpool_bwd_reduce(const __nv_bfloat16* __restrict__ dp,
                                                                              const uint8_t* __restrict__ arg,
                                                                              const __nv_bfloat16* __restrict__ x,
                                                                              const float* __restrict__ mean,
                                                                              const float* __restrict__ rstd,
                                                                              float* __restrict__ part, BnGeom g, TailGeom t) {
  extern __shared__ float smem[];
  const int tx = threadIdx.x % g.groups, ty = threadIdx.x / g.groups;
  float s[8], q[8], mu[8], rs[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    s[j] = q[j] = 0.f;
    mu[j] = mean[tx * 8 + j];
    rs[j] = rstd[tx * 8 + j];
  }
  const long long per_cta = (g.pixels + gridDim.x - 1) / gridDim.x;
  const long long p0 = (long long)blockIdx.x * per_cta;
  const long long p1 = p0 + per_cta < g.pixels ? p0 + per_cta : g.pixels;
  if (ty < g.lanes) {
    for (long long p = p0 + ty; p < p1; p += g.lanes) {   // min-blocks 3: 80 registers, no spills (92 without the cap)
      float d[8], a[8];
      ld8_stream(x + p * g.C + tx * 8, a);
      pooled_grad8(dp, arg, (int)p, g.C, tx, t, d);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        s[j] += d[j];
        q[j] = fmaf(d[j], (a[j] - mu[j]) * rs[j], q[j]);
      }
    }
  }
  reduce_lanes(smem, s, tx, ty, g, part + (size_t)blockIdx.x * 2 * g.C);
  reduce_lanes(smem, q, tx, ty, g, part + (size_t)blockIdx.x * 2 * g.C + g.C);
}

// psb_bn_bwd_apply<false, true, true> with the same gather
__global__ void __launch_bounds__(BN_THREADS) psb_bn_relu_maxpool_bwd_apply(const __nv_bfloat16* __restrict__ dp,
                                                                             const uint8_t* __restrict__ arg,
                                                                             const __nv_bfloat16* __restrict__ x,
                                                                             const float* __restrict__ ca, const float* __restrict__ cb,
                                                                             const float* __restrict__ cc, __nv_bfloat16* __restrict__ dx,
                                                                             BnGeom g, TailGeom t) {
  const int tx = threadIdx.x % g.groups, ty = threadIdx.x / g.groups;
  if (ty >= g.lanes) return;
  float a[8], b[8], c[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    a[j] = ca[tx * 8 + j];
    b[j] = cb[tx * 8 + j];
    c[j] = cc[tx * 8 + j];
  }
  const long long stride = (long long)gridDim.x * g.lanes;
  for (long long p = (long long)blockIdx.x * g.lanes + ty; p < g.pixels; p += stride) {
    const long long off = p * g.C + tx * 8;
    float d[8], xv[8];
    ld8_stream(x + off, xv);
    pooled_grad8(dp, arg, (int)p, g.C, tx, t, d);
#pragma unroll
    for (int j = 0; j < 8; ++j) xv[j] = fmaf(d[j], a[j], fmaf(xv[j], b[j], c[j]));
    st8(dx + off, xv);
  }
}

BnGeom geom(long long pixels, int C) {
  BnGeom g;
  g.pixels = pixels;
  g.C = C;
  g.groups = C / 8;
  g.lanes = BN_THREADS / g.groups;
  if (g.lanes < 1) g.lanes = 1;
  return g;
}

int grid_for(long long pixels, const BnGeom& g, int min_iters = 1) {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  long long want = (pixels + (long long)g.lanes * min_iters - 1) / ((long long)g.lanes * min_iters);   // >= min_iters pixel batches per CTA
  long long cap = (long long)sms * 8;
  return (int)(want < cap ? (want > 0 ? want : 1) : cap);
}
// The reducing kernels write 2C partials per CTA that the finalize kernels add up: on the small late-stage tensors thousands of
// CTAs of ~3 pixel batches each would make that sum the bottleneck.  They get at least 8 batches per CTA.
constexpr int REDUCE_MIN_ITERS = 8;

}  // namespace

// floats of per-CTA partials the reducing kernels write for a tensor of `pixels` x C (the `part` argument below)
long long psb_bn_partial_floats(long long pixels, int C) {
  return (long long)grid_for(pixels, geom(pixels, C), REDUCE_MIN_ITERS) * 2 * C;
}

// C must be a multiple of 8 and <= 2048 (groups <= 256)
void psb_bn_forward(cudaStream_t s, const void* x, const void* res, const void* gamma, const void* beta, void* y,
                    float* part /*psb_bn_partial_floats*/, float* mean, float* rstd, float* scale, float* shift, float* running_mean,
                    float* running_var, long long pixels, int C, float eps, float momentum, int relu, int training, void* mask) {
  auto MK = reinterpret_cast<uint8_t*>(mask);
  const BnGeom g = geom(pixels, C);
  const int grid = grid_for(pixels, g);
  auto X = reinterpret_cast<const __nv_bfloat16*>(x);
  auto R = reinterpret_cast<const __nv_bfloat16*>(res);
  auto Y = reinterpret_cast<__nv_bfloat16*>(y);
  psb_count_launch(training ? 3 : 1);
  if (training) {
    const int rgrid = grid_for(pixels, g, REDUCE_MIN_ITERS);
    psb_bn_stats<<<rgrid, BN_THREADS, sizeof(float) * g.lanes * C, s>>>(X, part, g);
    psb_bn_finalize<<<(C + FIN_CH - 1) / FIN_CH, FIN_THREADS, 0, s>>>(part, rgrid, reinterpret_cast<const __nv_bfloat16*>(gamma),
                                                     reinterpret_cast<const __nv_bfloat16*>(beta), mean, rstd, scale, shift,
                                                     running_mean, running_var, C, pixels, eps, momentum);
  }
  if (res != nullptr) {
    if (relu) psb_bn_apply<true, true><<<grid, BN_THREADS, 0, s>>>(X, R, scale, shift, Y, MK, g);
    else psb_bn_apply<true, false><<<grid, BN_THREADS, 0, s>>>(X, R, scale, shift, Y, MK, g);
  } else {
    if (relu) psb_bn_apply<false, true><<<grid, BN_THREADS, 0, s>>>(X, R, scale, shift, Y, MK, g);
    else psb_bn_apply<false, false><<<grid, BN_THREADS, 0, s>>>(X, R, scale, shift, Y, MK, g);
  }
}

// Training forward whose per-channel sums were produced elsewhere (the fused stem kernel's epilogue, stem_kernels.cu):
// finalize + apply only — the statistics pass over x is skipped (the fused stem, default).
void psb_bn_forward_presummed(cudaStream_t s, const void* x, const void* res, const void* gamma, const void* beta, void* y,
                              const float* sums /*2C, filled by the producer*/, float* mean, float* rstd, float* scale,
                              float* shift, float* running_mean, float* running_var, long long pixels, int C, float eps,
                              float momentum, int relu, void* mask) {
  auto MK = reinterpret_cast<uint8_t*>(mask);
  const BnGeom g = geom(pixels, C);
  const int grid = grid_for(pixels, g);
  auto X = reinterpret_cast<const __nv_bfloat16*>(x);
  auto R = reinterpret_cast<const __nv_bfloat16*>(res);
  auto Y = reinterpret_cast<__nv_bfloat16*>(y);
  psb_count_launch(2);
  psb_bn_finalize<<<(C + FIN_CH - 1) / FIN_CH, FIN_THREADS, 0, s>>>(sums, 1, reinterpret_cast<const __nv_bfloat16*>(gamma),
                                                   reinterpret_cast<const __nv_bfloat16*>(beta), mean, rstd, scale, shift,
                                                   running_mean, running_var, C, pixels, eps, momentum);
  if (res != nullptr) {
    if (relu) psb_bn_apply<true, true><<<grid, BN_THREADS, 0, s>>>(X, R, scale, shift, Y, MK, g);
    else psb_bn_apply<true, false><<<grid, BN_THREADS, 0, s>>>(X, R, scale, shift, Y, MK, g);
  } else {
    if (relu) psb_bn_apply<false, true><<<grid, BN_THREADS, 0, s>>>(X, R, scale, shift, Y, MK, g);
    else psb_bn_apply<false, false><<<grid, BN_THREADS, 0, s>>>(X, R, scale, shift, Y, MK, g);
  }
}

void psb_bn_backward(cudaStream_t s, const void* dy, const void* x, const void* y, const void* gamma, const float* mean,
                     const float* rstd, float* part /*psb_bn_partial_floats*/, float* coef /*3C*/, void* dx, void* dres, void* dgamma, void* dbeta,
                     long long pixels, int C, int relu, const void* mask) {
  auto MK = reinterpret_cast<const uint8_t*>(mask);
  const BnGeom g = geom(pixels, C);
  const int grid = grid_for(pixels, g);
  auto DY = reinterpret_cast<const __nv_bfloat16*>(dy);
  auto X = reinterpret_cast<const __nv_bfloat16*>(x);
  auto Y = reinterpret_cast<const __nv_bfloat16*>(y);
  psb_count_launch(3);
  const size_t sm = sizeof(float) * g.lanes * C;
  const int rgrid = grid_for(pixels, g, REDUCE_MIN_ITERS);
  if (relu && MK) psb_bn_bwd_reduce<true, true><<<rgrid, BN_THREADS, sm, s>>>(DY, X, Y, MK, mean, rstd, part, g);
  else if (relu) psb_bn_bwd_reduce<true, false><<<rgrid, BN_THREADS, sm, s>>>(DY, X, Y, MK, mean, rstd, part, g);
  else psb_bn_bwd_reduce<false, false><<<rgrid, BN_THREADS, sm, s>>>(DY, X, Y, MK, mean, rstd, part, g);
  psb_bn_bwd_finalize<<<(C + FIN_CH - 1) / FIN_CH, FIN_THREADS, 0, s>>>(part, rgrid, reinterpret_cast<const __nv_bfloat16*>(gamma),
                                                                         mean, rstd, coef,
                                                       coef + C, coef + 2 * C, reinterpret_cast<__nv_bfloat16*>(dgamma),
                                                       reinterpret_cast<__nv_bfloat16*>(dbeta), C, pixels);
  auto DX = reinterpret_cast<__nv_bfloat16*>(dx);
  auto DR = reinterpret_cast<__nv_bfloat16*>(dres);
#define PSB_APPLY(RES_, RELU_, MASKED_) \
  psb_bn_bwd_apply<RES_, RELU_, MASKED_><<<grid, BN_THREADS, 0, s>>>(DY, X, Y, MK, coef, coef + C, coef + 2 * C, DX, DR, g)
  if (dres != nullptr) {
    if (relu && MK) PSB_APPLY(true, true, true);
    else if (relu) PSB_APPLY(true, true, false);
    else PSB_APPLY(true, false, false);
  } else {
    if (relu && MK) PSB_APPLY(false, true, true);
    else if (relu) PSB_APPLY(false, true, false);
    else PSB_APPLY(false, false, false);
  }
#undef PSB_APPLY
}

// The ResNet stem tail, training (see psb_bn_relu_maxpool_fwd): finalize on the producer's sums, then BN + ReLU + 3x3/s2/p1
// max-pool in one pass → pooled [N, H/2, W/2, C] and its 1-byte taps (255: the window routes no gradient).  H, W even.
void psb_bn_relu_maxpool_forward_presummed(cudaStream_t s, const void* x, const void* gamma, const void* beta, const float* sums,
                                           float* mean, float* rstd, float* scale, float* shift, float* running_mean,
                                           float* running_var, int N, int H, int W, int C, float eps, float momentum, void* y,
                                           void* arg) {
  const long long pixels = (long long)N * H * W;
  const BnGeom g = geom(pixels, C);
  const TailGeom t{N, H, W, H / 2, W / 2};
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int rows = N * t.OH, grid = rows < sms * 16 ? rows : sms * 16;
  psb_count_launch(2);
  psb_bn_finalize<<<(C + FIN_CH - 1) / FIN_CH, FIN_THREADS, 0, s>>>(sums, 1, reinterpret_cast<const __nv_bfloat16*>(gamma),
                                                   reinterpret_cast<const __nv_bfloat16*>(beta), mean, rstd, scale, shift,
                                                   running_mean, running_var, C, pixels, eps, momentum);
  psb_bn_relu_maxpool_fwd<<<grid, BN_THREADS, 0, s>>>(reinterpret_cast<const __nv_bfloat16*>(x), scale, shift,
                                                       reinterpret_cast<__nv_bfloat16*>(y), reinterpret_cast<uint8_t*>(arg), g, t);
}

// Backward of the stem tail from the pooled gradient `dy` [N, H/2, W/2, C] and the forward's taps: reduce → finalize → apply,
// as psb_bn_backward with relu and the mask, bit for bit.
void psb_bn_relu_maxpool_backward(cudaStream_t s, const void* dy, const void* arg, const void* x, const void* gamma,
                                  const float* mean, const float* rstd, float* part /*psb_bn_partial_floats*/, float* coef /*3C*/,
                                  void* dx, void* dgamma, void* dbeta, int N, int H, int W, int C) {
  const long long pixels = (long long)N * H * W;
  const BnGeom g = geom(pixels, C);
  const TailGeom t{N, H, W, H / 2, W / 2};
  auto DY = reinterpret_cast<const __nv_bfloat16*>(dy);
  auto A = reinterpret_cast<const uint8_t*>(arg);
  auto X = reinterpret_cast<const __nv_bfloat16*>(x);
  psb_count_launch(3);
  const int rgrid = grid_for(pixels, g, REDUCE_MIN_ITERS);
  psb_bn_relu_maxpool_bwd_reduce<<<rgrid, BN_THREADS, sizeof(float) * g.lanes * C, s>>>(DY, A, X, mean, rstd, part, g, t);
  psb_bn_bwd_finalize<<<(C + FIN_CH - 1) / FIN_CH, FIN_THREADS, 0, s>>>(part, rgrid, reinterpret_cast<const __nv_bfloat16*>(gamma),
                                                                         mean, rstd, coef, coef + C, coef + 2 * C,
                                                                         reinterpret_cast<__nv_bfloat16*>(dgamma),
                                                                         reinterpret_cast<__nv_bfloat16*>(dbeta), C, pixels);
  psb_bn_relu_maxpool_bwd_apply<<<grid_for(pixels, g), BN_THREADS, 0, s>>>(DY, A, X, coef, coef + C, coef + 2 * C,
                                                                           reinterpret_cast<__nv_bfloat16*>(dx), g, t);
}
