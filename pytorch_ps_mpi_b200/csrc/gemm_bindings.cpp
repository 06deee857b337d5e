// Bindings of the broadcast-gated wgmma GEMM (csrc/kernels/bcast_gemm.cu): builds the TMA
// tensor maps with cuTensorMapEncodeTiled (resolved through the runtime, no -lcuda) and launches.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAStream.h>
#include <cuda.h>
#include <torch/extension.h>

#include "kernels.h"

namespace py = pybind11;
int psb_bcast_gemm_smem_bytes();

namespace {

using EncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                              const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                              CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeFn encode_fn() {
  static EncodeFn f = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || p == nullptr)
      throw std::runtime_error("cuTensorMapEncodeTiled not available");
    return reinterpret_cast<EncodeFn>(p);
  }();
  return f;
}

// 2-D bf16 row-major [rows, cols] tensor, box = [box_rows, 64 cols] (128 bytes), 128B swizzle
CUtensorMap make_map(uint64_t ptr, int64_t rows, int64_t cols, int64_t row_stride_elems, int box_rows) {
  CUtensorMap m;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)row_stride_elems * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = encode_fn()(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, reinterpret_cast<void*>(ptr), dims, strides, box, estr,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) throw std::runtime_error("cuTensorMapEncodeTiled failed (code " + std::to_string((int)r) + ")");
  return m;
}

// y[M,N] = act(x[M,K] @ w[N,K]^T + bias).  `w_ptr` may be any mapped address holding the [N,K] bf16
// weight (this rank's parameter arena, or the server's arena over NVLink).  `flag_ptr` (optional) is
// the SIG_PARAMS_READY slot the TMA producer acquires before its first weight load.
at::Tensor bcast_gemm(const at::Tensor& x, uint64_t w_ptr, int64_t N, int64_t K, c10::optional<at::Tensor> bias, bool relu,
                      uint64_t flag_ptr, uint64_t epoch, double timeout_s, int variant) {
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == at::kBFloat16 && x.dim() == 2 && x.is_contiguous(), "x must be [M,K] bf16 contiguous");
  TORCH_CHECK(x.size(1) == K && K % 8 == 0, "K mismatch / K must be a multiple of 8");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(x.data_ptr()) % 16 == 0 && w_ptr % 16 == 0, "operands must be 16-byte aligned");
  const int64_t M = x.size(0);
  auto y = at::empty({M, N}, x.options());
  if (M == 0) return y;
  // a pair of CTAs (one cluster, the B tile multicast to both) whenever there are at least 256 rows; `variant & 15` forces
  // one CTA (1) / a pair (2).  Bits 4-7: epilogue — 0 auto (TMA store when N % 8 == 0, else staged), 1 staged, 3 TMA store,
  // 4 direct stores from the accumulator fragment (bench/gemm_variants.py)
  const int base = variant & 15, epi_sel = (variant >> 4) & 15;
  TORCH_CHECK(base <= 2 && (epi_sel == 0 || epi_sel == 1 || epi_sel == 3 || epi_sel == 4) && (variant >> 8) == 0,
              "unknown bcast_gemm variant ", variant);
  const int epi = epi_sel == 0 ? -1 : (epi_sel == 4 ? 0 : epi_sel);
  TORCH_CHECK(epi != 3 || N % 8 == 0, "the TMA-store epilogue needs N % 8 == 0 (16-byte row pitch)");
  const bool two_cta = base == 2 || (base == 0 && M >= 256);
  CUtensorMap ma = make_map(reinterpret_cast<uint64_t>(x.data_ptr()), M, K, K, 128);
  const int bn = psb_bcast_gemm_bn((int)N);
  CUtensorMap mb = make_map(w_ptr, N, K, K, two_cta ? bn / 2 : bn);   // B box: half tile per CTA of a pair, or the whole tile
  CUtensorMap mc;
  BcastGemmArgs a{};
  a.tmap_a = &ma;
  a.tmap_b = &mb;
  a.tmap_c = y.data_ptr();
  if (N % 8 == 0 && (epi == 3 || epi < 0)) {
    mc = make_map(reinterpret_cast<uint64_t>(y.data_ptr()), M, N, N, 32);      // box: 64 columns x 32 rows, 128B swizzle
    a.tmap_out = &mc;
  }
  const float* bp = nullptr;
  at::Tensor bias_f;
  if (bias.has_value() && bias->defined()) {
    bias_f = bias->to(at::kFloat).contiguous();
    bp = bias_f.data_ptr<float>();
  }
  a.bias = bp;
  a.ready_flag = reinterpret_cast<const uint64_t*>(flag_ptr);
  a.ready_epoch = epoch;
  a.M = (int)M, a.N = (int)N, a.K = (int)K;
  a.relu = relu ? 1 : 0;
  a.two_cta = two_cta ? 1 : 0;
  a.timeout_ns = (unsigned long long)(timeout_s * 1e9);
  const int sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  psb_launch_bcast_gemm(c10::cuda::getCurrentCUDAStream().stream(), a, sms, epi);
  cudaError_t e = cudaGetLastError();
  TORCH_CHECK(e == cudaSuccess, "psb_bcast_gemm_kernel launch: ", cudaGetErrorString(e));
  return y;
}

void check_nhwc(const at::Tensor& t, const char* name) {
  TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kBFloat16 && t.dim() == 4, name, " must be a 4-D CUDA bf16 tensor");
  TORCH_CHECK(t.is_contiguous(at::MemoryFormat::ChannelsLast), name, " must be channels_last contiguous");
}

// y = act(BN(x) [+ res]);  returns (y, mean, rstd)
std::vector<at::Tensor> bn_forward(const at::Tensor& x, c10::optional<at::Tensor> res, const at::Tensor& gamma,
                                   const at::Tensor& beta, at::Tensor running_mean, at::Tensor running_var, double eps,
                                   double momentum, bool relu, bool training) {
  check_nhwc(x, "x");
  const int C = (int)x.size(1);
  TORCH_CHECK(C % 8 == 0 && C <= 2048, "channels must be a multiple of 8 and <= 2048");
  const long long pixels = x.numel() / C;
  const void* rp = nullptr;
  if (res.has_value() && res->defined()) {
    check_nhwc(*res, "residual");
    TORCH_CHECK(res->sizes() == x.sizes(), "residual shape mismatch");
    rp = res->data_ptr();
  }
  TORCH_CHECK(running_mean.scalar_type() == at::kFloat && running_var.scalar_type() == at::kFloat, "running stats must be fp32");
  auto y = at::empty_like(x);
  auto fo = x.options().dtype(at::kFloat);
  auto scratch = at::empty({4 * C}, fo);   // mean | rstd | scale | shift
  float* sp = scratch.data_ptr<float>();
  at::Tensor mean = scratch.narrow(0, 0, C), rstd = scratch.narrow(0, C, C);
  at::Tensor part = training ? at::empty({psb_bn_partial_floats(pixels, C)}, fo) : at::Tensor();
  // ReLU + training: a 1-bit-per-element mask (y > 0) for the backward, which then never re-reads y
  at::Tensor mask = (relu && training) ? at::empty({pixels * (C / 8)}, x.options().dtype(at::kByte)) : at::Tensor();
  if (!training) {   // inference: scale/shift from the running statistics
    auto r = (running_var + eps).rsqrt();
    auto sc = gamma.to(at::kFloat) * r;
    scratch.narrow(0, 2 * C, C).copy_(sc);
    scratch.narrow(0, 3 * C, C).copy_(beta.to(at::kFloat) - running_mean * sc);
  }
  psb_bn_forward(c10::cuda::getCurrentCUDAStream().stream(), x.data_ptr(), rp, gamma.data_ptr(), beta.data_ptr(), y.data_ptr(),
                 part.defined() ? part.data_ptr<float>() : nullptr, sp, sp + C, sp + 2 * C, sp + 3 * C, running_mean.data_ptr<float>(),
                 running_var.data_ptr<float>(), pixels, C, (float)eps, (float)momentum, relu ? 1 : 0, training ? 1 : 0,
                 mask.defined() ? mask.data_ptr() : nullptr);
  cudaError_t e = cudaGetLastError();
  TORCH_CHECK(e == cudaSuccess, "psb_bn_forward: ", cudaGetErrorString(e));
  return {y, mean, rstd, mask};
}

// returns (dx, dres or undefined, dgamma, dbeta)
// `out_dgamma` / `out_dbeta` (optional): where to write the parameter gradients — the PS device engine hands out views of its
// wire arena (DeviceEngine.grad_out) so these gradients need no encode pass.
std::vector<at::Tensor> bn_backward(const at::Tensor& dy, const at::Tensor& x, const at::Tensor& y, const at::Tensor& gamma,
                                    const at::Tensor& mean, const at::Tensor& rstd, bool relu, bool has_res,
                                    c10::optional<at::Tensor> out_dgamma, c10::optional<at::Tensor> out_dbeta,
                                    c10::optional<at::Tensor> pool_arg) {
  // relu: `y` is either the saved output (bf16, same shape as x) or the forward's 1-bit mask (uint8, numel/8 bytes)
  // pool_arg: the taps of bn_forward_presummed(pool=True); `dy` is then the pooled gradient and `y` is unused
  const bool pooled = pool_arg.has_value() && pool_arg->defined();
  const bool masked = !pooled && relu && y.scalar_type() == at::kByte;
  if (masked) TORCH_CHECK(y.numel() * 8 == x.numel() && y.is_contiguous(), "bn_backward: mask size mismatch");
  check_nhwc(dy, "dy");
  check_nhwc(x, "x");
  const int C = (int)x.size(1);
  const long long pixels = x.numel() / C;
  const int N = (int)x.size(0), H = (int)x.size(2), W = (int)x.size(3);
  if (pooled) {
    TORCH_CHECK(relu && !has_res, "bn_backward(pool_arg): ReLU and no residual only");
    TORCH_CHECK(H % 2 == 0 && W % 2 == 0 && C % 8 == 0 && C <= 2048 && pixels < (1LL << 31),
                "bn_backward(pool_arg): H and W must be even, C a multiple of 8 and <= 2048");
    TORCH_CHECK(dy.size(0) == N && dy.size(1) == C && dy.size(2) == H / 2 && dy.size(3) == W / 2, "bn_backward: pooled dy shape");
    TORCH_CHECK(pool_arg->scalar_type() == at::kByte && pool_arg->sizes() == dy.sizes() &&
                    pool_arg->is_contiguous(at::MemoryFormat::ChannelsLast),
                "bn_backward: pool_arg must be the forward's channels-last uint8 taps");
  }
  auto dx = at::empty_like(x);
  at::Tensor dres;
  if (has_res) dres = at::empty_like(x);
  auto pick = [&](c10::optional<at::Tensor>& o) {
    if (o.has_value() && o->defined()) {
      TORCH_CHECK(o->is_cuda() && o->scalar_type() == gamma.scalar_type() && o->numel() == gamma.numel() && o->is_contiguous(),
                  "bn_backward: out gradient must be a contiguous tensor like gamma");
      return *o;
    }
    return at::empty_like(gamma);
  };
  auto dgamma = pick(out_dgamma), dbeta = pick(out_dbeta);
  auto scratch = at::empty({3 * C}, x.options().dtype(at::kFloat));
  auto part = at::empty({psb_bn_partial_floats(pixels, C)}, x.options().dtype(at::kFloat));
  float* sp = scratch.data_ptr<float>();
  if (pooled) {
    psb_bn_relu_maxpool_backward(c10::cuda::getCurrentCUDAStream().stream(), dy.data_ptr(), pool_arg->data_ptr(), x.data_ptr(),
                                 gamma.data_ptr(), mean.data_ptr<float>(), rstd.data_ptr<float>(), part.data_ptr<float>(), sp,
                                 dx.data_ptr(), dgamma.data_ptr(), dbeta.data_ptr(), N, H, W, C);
    cudaError_t e = cudaGetLastError();
    TORCH_CHECK(e == cudaSuccess, "psb_bn_relu_maxpool_backward: ", cudaGetErrorString(e));
    return {dx, dres, dgamma, dbeta};
  }
  psb_bn_backward(c10::cuda::getCurrentCUDAStream().stream(), dy.data_ptr(), x.data_ptr(),
                  (relu && !masked) ? y.data_ptr() : nullptr, gamma.data_ptr(), mean.data_ptr<float>(), rstd.data_ptr<float>(),
                  part.data_ptr<float>(), sp, dx.data_ptr(), has_res ? dres.data_ptr() : nullptr, dgamma.data_ptr(), dbeta.data_ptr(), pixels, C,
                  relu ? 1 : 0, masked ? y.data_ptr() : nullptr);
  cudaError_t e = cudaGetLastError();
  TORCH_CHECK(e == cudaSuccess, "psb_bn_backward: ", cudaGetErrorString(e));
  return {dx, dres, dgamma, dbeta};
}

std::vector<at::Tensor> maxpool_forward(const at::Tensor& x) {
  check_nhwc(x, "x");
  const int N = (int)x.size(0), C = (int)x.size(1), H = (int)x.size(2), W = (int)x.size(3);
  TORCH_CHECK(C % 8 == 0, "channels must be a multiple of 8");
  const int OH = (H - 1) / 2 + 1, OW = (W - 1) / 2 + 1;
  auto y = at::empty({N, C, OH, OW}, x.options().memory_format(at::MemoryFormat::ChannelsLast));
  auto arg = at::empty({N, C, OH, OW}, x.options().dtype(at::kByte).memory_format(at::MemoryFormat::ChannelsLast));
  psb_maxpool3x3s2_forward(c10::cuda::getCurrentCUDAStream().stream(), x.data_ptr(), y.data_ptr(), arg.data_ptr(), N, H, W, C);
  cudaError_t e = cudaGetLastError();
  TORCH_CHECK(e == cudaSuccess, "psb_maxpool_fwd: ", cudaGetErrorString(e));
  return {y, arg};
}

at::Tensor maxpool_backward(const at::Tensor& dy, const at::Tensor& arg, int64_t H, int64_t W) {
  check_nhwc(dy, "dy");
  const int N = (int)dy.size(0), C = (int)dy.size(1);
  auto dx = at::empty({N, C, H, W}, dy.options().memory_format(at::MemoryFormat::ChannelsLast));
  psb_maxpool3x3s2_backward(c10::cuda::getCurrentCUDAStream().stream(), dy.data_ptr(), arg.data_ptr(), dx.data_ptr(), N, (int)H,
                            (int)W, C);
  cudaError_t e = cudaGetLastError();
  TORCH_CHECK(e == cudaSuccess, "psb_maxpool_bwd: ", cudaGetErrorString(e));
  return dx;
}

// uint8 [N,3,H,W] (NCHW) → bf16 [N,8,H,W] channels_last, (x - mean) / std, channels 3..7 zero
at::Tensor normalize_pad8(const at::Tensor& x, std::vector<double> mean, std::vector<double> std) {
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == at::kByte && x.dim() == 4 && x.size(1) == 3 && x.is_contiguous(),
              "x must be a contiguous uint8 [N,3,H,W] CUDA tensor");
  TORCH_CHECK(mean.size() == 3 && std.size() == 3, "mean/std need 3 entries");
  const int N = (int)x.size(0);
  const long long HW = x.size(2) * x.size(3);
  auto y = at::empty({N, 8, x.size(2), x.size(3)}, x.options().dtype(at::kBFloat16).memory_format(at::MemoryFormat::ChannelsLast));
  float m[3] = {(float)mean[0], (float)mean[1], (float)mean[2]};
  float is[3] = {(float)(1.0 / std[0]), (float)(1.0 / std[1]), (float)(1.0 / std[2])};
  psb_normalize_pad8_launch(c10::cuda::getCurrentCUDAStream().stream(), x.data_ptr(), y.data_ptr(), m, is, N, HW);
  cudaError_t e = cudaGetLastError();
  TORCH_CHECK(e == cudaSuccess, "psb_normalize_pad8: ", cudaGetErrorString(e));
  return y;
}

// bf16 NHWC [N,3,H,W] (channels_last) → patch matrix [N*OH*OW, 176] for the 7x7/s2/p3 stem
// training BatchNorm forward whose Σx / Σx² were produced by the fused stem kernel; returns (y, mean, rstd, mask)
// pool: the ResNet stem tail — BN + ReLU + 3x3/s2/p1 max-pool in one pass (no residual, even H and W); returns
// (pooled, mean, rstd, arg) where arg holds each window's tap, 255 where the window routes no gradient (bn_backward's pool_arg)
std::vector<at::Tensor> bn_forward_presummed(const at::Tensor& x, c10::optional<at::Tensor> res, const at::Tensor& gamma,
                                             const at::Tensor& beta, at::Tensor running_mean, at::Tensor running_var, double eps,
                                             double momentum, bool relu, const at::Tensor& sums, bool pool) {
  check_nhwc(x, "x");
  const int C = (int)x.size(1);
  TORCH_CHECK(C % 8 == 0 && C <= 2048, "channels must be a multiple of 8 and <= 2048");
  TORCH_CHECK(sums.is_cuda() && sums.scalar_type() == at::kFloat && sums.numel() == 2 * C && sums.is_contiguous(),
              "sums must be a contiguous fp32 CUDA tensor of 2*C elements");
  const long long pixels = x.numel() / C;
  if (pool) {
    const int N = (int)x.size(0), H = (int)x.size(2), W = (int)x.size(3);
    TORCH_CHECK(relu && !(res.has_value() && res->defined()), "bn_forward_presummed(pool=True): ReLU and no residual only");
    TORCH_CHECK(H % 2 == 0 && W % 2 == 0 && H > 0 && W > 0, "bn_forward_presummed(pool=True): H and W must be even");
    TORCH_CHECK(pixels < (1LL << 31), "bn_forward_presummed(pool=True): more than 2^31 pixels");
    TORCH_CHECK(running_mean.scalar_type() == at::kFloat && running_var.scalar_type() == at::kFloat, "running stats must be fp32");
    auto y = at::empty({N, C, H / 2, W / 2}, x.options().memory_format(at::MemoryFormat::ChannelsLast));
    auto arg = at::empty({N, C, H / 2, W / 2}, x.options().dtype(at::kByte).memory_format(at::MemoryFormat::ChannelsLast));
    auto scratch = at::empty({4 * C}, x.options().dtype(at::kFloat));   // mean | rstd | scale | shift
    float* sp = scratch.data_ptr<float>();
    psb_bn_relu_maxpool_forward_presummed(c10::cuda::getCurrentCUDAStream().stream(), x.data_ptr(), gamma.data_ptr(),
                                          beta.data_ptr(), sums.data_ptr<float>(), sp, sp + C, sp + 2 * C, sp + 3 * C,
                                          running_mean.data_ptr<float>(), running_var.data_ptr<float>(), N, H, W, C, (float)eps,
                                          (float)momentum, y.data_ptr(), arg.data_ptr());
    cudaError_t e = cudaGetLastError();
    TORCH_CHECK(e == cudaSuccess, "psb_bn_relu_maxpool_forward_presummed: ", cudaGetErrorString(e));
    return {y, scratch.narrow(0, 0, C), scratch.narrow(0, C, C), arg};
  }
  const void* rp = nullptr;
  if (res.has_value() && res->defined()) {
    check_nhwc(*res, "residual");
    TORCH_CHECK(res->sizes() == x.sizes(), "residual shape mismatch");
    rp = res->data_ptr();
  }
  TORCH_CHECK(running_mean.scalar_type() == at::kFloat && running_var.scalar_type() == at::kFloat, "running stats must be fp32");
  auto y = at::empty_like(x);
  auto scratch = at::empty({4 * C}, x.options().dtype(at::kFloat));   // mean | rstd | scale | shift
  float* sp = scratch.data_ptr<float>();
  at::Tensor mask = relu ? at::empty({pixels * (C / 8)}, x.options().dtype(at::kByte)) : at::Tensor();
  psb_bn_forward_presummed(c10::cuda::getCurrentCUDAStream().stream(), x.data_ptr(), rp, gamma.data_ptr(), beta.data_ptr(),
                           y.data_ptr(), sums.data_ptr<float>(), sp, sp + C, sp + 2 * C, sp + 3 * C,
                           running_mean.data_ptr<float>(), running_var.data_ptr<float>(), pixels, C, (float)eps, (float)momentum,
                           relu ? 1 : 0, mask.defined() ? mask.data_ptr() : nullptr);
  cudaError_t e = cudaGetLastError();
  TORCH_CHECK(e == cudaSuccess, "psb_bn_forward_presummed: ", cudaGetErrorString(e));
  return {y, scratch.narrow(0, 0, C), scratch.narrow(0, C, C), mask};
}

// fused stem: x [N,3,H,W] bf16 channels-last, w2d [64,176] bf16 (ops/stem.py layout)
// → (y [N,64,OH,OW] bf16 channels-last, sums [128] fp32 = Σy | Σy² per channel, or an empty tensor)
std::vector<at::Tensor> stem_fwd(const at::Tensor& x, const at::Tensor& w2d, bool want_sums, uint64_t flag_ptr, uint64_t epoch,
                                 double timeout_s) {
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == at::kBFloat16 && x.dim() == 4 && x.size(1) == 3, "x must be [N,3,H,W] bf16");
  TORCH_CHECK(x.is_contiguous(at::MemoryFormat::ChannelsLast), "x must be channels_last contiguous");
  TORCH_CHECK(w2d.is_cuda() && w2d.scalar_type() == at::kBFloat16 && w2d.dim() == 2 && w2d.size(0) == 64 && w2d.size(1) == 176 &&
                  w2d.is_contiguous(),
              "w2d must be a contiguous [64,176] bf16 matrix");
  const int N = (int)x.size(0), H = (int)x.size(2), W = (int)x.size(3);
  TORCH_CHECK(W % 8 == 0 && W <= 256 && W >= 8 && H >= 1, "fused stem: W must be a multiple of 8 and <= 256");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(x.data_ptr()) % 16 == 0 && reinterpret_cast<uintptr_t>(w2d.data_ptr()) % 16 == 0,
              "operands must be 16-byte aligned");
  const int OH = (H - 1) / 2 + 1, OW = (W - 1) / 2 + 1;
  auto y = at::empty({N, OH, OW, 64}, x.options());
  const int sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  at::Tensor sums = want_sums ? at::empty({128}, x.options().dtype(at::kFloat)) : at::Tensor();
  at::Tensor part = want_sums ? at::empty({sms, 128}, x.options().dtype(at::kFloat)) : at::Tensor();
  CUtensorMap mw = make_map(reinterpret_cast<uint64_t>(w2d.data_ptr()), 64, 176, 176, 64);
  CUtensorMap my = make_map(reinterpret_cast<uint64_t>(y.data_ptr()), (int64_t)N * OH * OW, 64, 64, OW);
  psb_stem_fwd_launch(c10::cuda::getCurrentCUDAStream().stream(), &mw, &my, x.data_ptr(), want_sums ? sums.data_ptr<float>() : nullptr,
                      want_sums ? part.data_ptr<float>() : nullptr, N, H, W, sms, reinterpret_cast<const uint64_t*>(flag_ptr), epoch, (unsigned long long)(timeout_s * 1e9));
  cudaError_t e = cudaGetLastError();
  TORCH_CHECK(e == cudaSuccess, "psb_stem_fwd_kernel launch: ", cudaGetErrorString(e));
  return {y.permute({0, 3, 1, 2}), sums};
}

// implicit weight gradient of the stem: x [N,3,H,W], gy [N,64,OH,OW] (both bf16 channels-last)
// → per-CTA partials [grid,176,64] fp32 of dW2d^T (sum over dim 0 on the caller's side)
at::Tensor stem_wgrad(const at::Tensor& x, const at::Tensor& gy) {
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == at::kBFloat16 && x.dim() == 4 && x.size(1) == 3, "x must be [N,3,H,W] bf16");
  TORCH_CHECK(x.is_contiguous(at::MemoryFormat::ChannelsLast), "x must be channels_last contiguous");
  const int N = (int)x.size(0), H = (int)x.size(2), W = (int)x.size(3);
  TORCH_CHECK(W % 8 == 0 && W <= 256 && W >= 8, "fused stem: W must be a multiple of 8 and <= 256");
  const int OH = (H - 1) / 2 + 1, OW = (W - 1) / 2 + 1;
  check_nhwc(gy, "gy");
  TORCH_CHECK(gy.size(0) == N && gy.size(1) == 64 && gy.size(2) == OH && gy.size(3) == OW, "gy shape mismatch");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(x.data_ptr()) % 16 == 0 && reinterpret_cast<uintptr_t>(gy.data_ptr()) % 16 == 0,
              "operands must be 16-byte aligned");
  const int sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  const int grid = psb_stem_wgrad_grid(N, H, sms);
  auto partial = at::empty({grid, 176, 64}, x.options().dtype(at::kFloat));
  CUtensorMap mg = make_map(reinterpret_cast<uint64_t>(gy.data_ptr()), (int64_t)N * OH * OW, 64, 64, OW);
  psb_stem_wgrad_launch(c10::cuda::getCurrentCUDAStream().stream(), &mg, x.data_ptr(), partial.data_ptr<float>(), N, H, W, sms);
  cudaError_t e = cudaGetLastError();
  TORCH_CHECK(e == cudaSuccess, "psb_stem_wgrad_kernel launch: ", cudaGetErrorString(e));
  return partial;
}

// Σ over the per-CTA partials of psb_stem_wgrad_kernel, transposed and cast: [grid,176,64] fp32 → dW2d [64,176] bf16, written
// into `out` when given (the wire-arena slot of the stem weight: no encode pass) — one kernel instead of sum + t + to.
at::Tensor stem_wgrad_finalize(const at::Tensor& partial, c10::optional<at::Tensor> out) {
  TORCH_CHECK(partial.is_cuda() && partial.scalar_type() == at::kFloat && partial.dim() == 3 && partial.size(1) == 176 &&
                  partial.size(2) == 64 && partial.is_contiguous(), "partial must be [grid,176,64] fp32");
  at::Tensor o;
  if (out.has_value() && out->defined()) {
    TORCH_CHECK(out->is_cuda() && out->scalar_type() == at::kBFloat16 && out->numel() == 64 * 176 && out->is_contiguous(),
                "out must be a contiguous bf16 tensor of 64*176 elements");
    o = out->view({64, 176});
  } else {
    o = at::empty({64, 176}, partial.options().dtype(at::kBFloat16));
  }
  psb_stem_wgrad_finalize_launch(c10::cuda::getCurrentCUDAStream().stream(), partial.data_ptr<float>(), (int)partial.size(0),
                                 o.data_ptr());
  cudaError_t e = cudaGetLastError();
  TORCH_CHECK(e == cudaSuccess, "psb_stem_wgrad_finalize: ", cudaGetErrorString(e));
  return o;
}

at::Tensor im2col_stem(const at::Tensor& x) {
  check_nhwc(x, "x");
  TORCH_CHECK(x.size(1) == 3, "stem input must have 3 channels");
  const int N = (int)x.size(0), H = (int)x.size(2), W = (int)x.size(3);
  const int OH = (H - 1) / 2 + 1, OW = (W - 1) / 2 + 1;
  auto a = at::empty({(int64_t)N * OH * OW, 176}, x.options());
  psb_im2col_stem_launch(c10::cuda::getCurrentCUDAStream().stream(), x.data_ptr(), a.data_ptr(), N, H, W);
  cudaError_t e = cudaGetLastError();
  TORCH_CHECK(e == cudaSuccess, "psb_im2col_stem: ", cudaGetErrorString(e));
  return a;
}

// uint8 [N,3,H,W] NCHW → bf16 [N,3,H,W] channels_last, (x - mean) / std
at::Tensor normalize_nhwc3(const at::Tensor& x, std::vector<double> mean, std::vector<double> std) {
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == at::kByte && x.dim() == 4 && x.size(1) == 3 && x.is_contiguous(),
              "x must be a contiguous uint8 [N,3,H,W] CUDA tensor");
  const int N = (int)x.size(0);
  const long long HW = x.size(2) * x.size(3);
  auto y = at::empty({N, 3, x.size(2), x.size(3)}, x.options().dtype(at::kBFloat16).memory_format(at::MemoryFormat::ChannelsLast));
  float m[3] = {(float)mean[0], (float)mean[1], (float)mean[2]};
  float is[3] = {(float)(1.0 / std[0]), (float)(1.0 / std[1]), (float)(1.0 / std[2])};
  psb_normalize_nhwc3_launch(c10::cuda::getCurrentCUDAStream().stream(), x.data_ptr(), y.data_ptr(), m, is, N, HW);
  cudaError_t e = cudaGetLastError();
  TORCH_CHECK(e == cudaSuccess, "psb_normalize_nhwc3: ", cudaGetErrorString(e));
  return y;
}

}  // namespace

void bind_gemm(py::module_& m) {
  m.def("im2col_stem", &im2col_stem, "bf16 NHWC(3) image → [N*OH*OW,176] patch matrix of the 7x7/s2/p3 stem");
  m.def("normalize_nhwc3", &normalize_nhwc3, "uint8 NCHW image → normalised bf16 NHWC (3 channels)");
  m.def("normalize_pad8", &normalize_pad8, "uint8 NCHW image → normalised bf16 NHWC padded to 8 channels");
  m.def("maxpool_forward", &maxpool_forward, "channels-last bf16 3x3/s2/p1 max pool → (y, argpos)");
  m.def("maxpool_backward", &maxpool_backward, "gather-style backward of maxpool_forward");
  m.def("bn_forward", &bn_forward, "fused channels-last bf16 BatchNorm(+residual)(+ReLU) forward");
  m.def("bn_forward_presummed", &bn_forward_presummed, py::arg("x"), py::arg("res"), py::arg("gamma"), py::arg("beta"),
        py::arg("running_mean"), py::arg("running_var"), py::arg("eps"), py::arg("momentum"), py::arg("relu"), py::arg("sums"),
        py::arg("pool") = false,
        "BN forward with sums produced by the fused stem kernel; pool=True: + ReLU + 3x3/s2/p1 max-pool → (pooled, mean, rstd, arg)");
  m.def("stem_fwd", &stem_fwd, py::arg("x"), py::arg("w2d"), py::arg("want_sums") = true, py::arg("flag_ptr") = 0,
        py::arg("epoch") = 0, py::arg("timeout_s") = 30.0,
        "fused implicit-GEMM ResNet stem (+ BN statistics) on wgmma; flag_ptr/epoch: PARAMS_READY gate of the weight load");
  m.def("stem_wgrad_finalize", &stem_wgrad_finalize, py::arg("partial"), py::arg("out") = c10::nullopt,
        "sum the per-CTA partials → dW2d [64,176] bf16 (optionally straight into the PS wire arena)");
  m.def("stem_wgrad", &stem_wgrad, "implicit weight gradient of the stem → per-CTA fp32 partials [grid,176,64]");
  m.def("bn_backward", &bn_backward, py::arg("dy"), py::arg("x"), py::arg("y"), py::arg("gamma"), py::arg("mean"), py::arg("rstd"),
        py::arg("relu"), py::arg("has_res"), py::arg("out_dgamma") = c10::nullopt, py::arg("out_dbeta") = c10::nullopt,
        py::arg("pool_arg") = c10::nullopt,
        "fused channels-last bf16 BatchNorm(+residual)(+ReLU) backward; pool_arg: dy is the pooled gradient of the stem tail");
  m.def("bcast_gemm", &bcast_gemm, py::arg("x"), py::arg("w_ptr"), py::arg("N"), py::arg("K"), py::arg("bias"),
        py::arg("relu"), py::arg("flag_ptr") = 0, py::arg("epoch") = 0, py::arg("timeout_s") = 30.0, py::arg("variant") = 0,
        "wgmma/TMA GEMM whose weight tiles are gated on the PS broadcast epoch flag");
  m.def("bcast_gemm_smem_bytes", &psb_bcast_gemm_smem_bytes);
}
