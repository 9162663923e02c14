// PyTorch bindings of the unicore_b200 sm_90a kernels (module ``unicore_b200._C``).
// Only this translation unit sees the PyTorch headers; kernels are declared in csrc/api.h.
#include <ATen/cuda/CUDAContext.h>
#include <ATen/cuda/CUDAGeneratorImpl.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include <mutex>
#include <optional>
#include <tuple>
#include <vector>

#include "api.h"
#include "attn/fmha_api.h"
#include "comm/comm_api.h"

namespace {

using torch::Tensor;
using OptTensor = std::optional<Tensor>;

int dtype_tag(const Tensor& t) {
  switch (t.scalar_type()) {
    case at::kFloat: return ub::kF32;
    case at::kHalf: return ub::kF16;
    case at::kBFloat16: return ub::kBF16;
    default: TORCH_CHECK(false, "unsupported dtype ", t.scalar_type());
  }
  return -1;
}

cudaStream_t cur_stream() { return at::cuda::getCurrentCUDAStream().stream(); }

void check_cuda_contig(const Tensor& t, const char* name) {
  TORCH_CHECK(t.is_cuda(), name, " must be a CUDA tensor");
  TORCH_CHECK(t.is_contiguous(), name, " must be contiguous");
}

const void* opt_ptr(const OptTensor& t) { return t.has_value() && t->defined() ? t->data_ptr() : nullptr; }

// Reserve `increment` Philox counters from the default CUDA generator: (seed, offset).
std::pair<uint64_t, uint64_t> philox_reserve(uint64_t increment) {
  auto gen = at::get_generator_or_default<at::CUDAGeneratorImpl>(std::nullopt,
                                                                 at::cuda::detail::getDefaultCUDAGenerator());
  std::lock_guard<std::mutex> lock(gen->mutex_);
  at::PhiloxCudaState st = gen->philox_cuda_state(increment);
  TORCH_CHECK(!st.captured_, "unicore_b200 kernels do not support RNG under CUDA graph capture yet");
  return {st.seed_.val, st.offset_.val};
}

void check_launch(const char* what) {
  cudaError_t err = cudaGetLastError();
  TORCH_CHECK(err == cudaSuccess, what, " launch failed: ", cudaGetErrorString(err));
}

// ---------------------------------------------------------------------------------------------------
// optimizer ops
// ---------------------------------------------------------------------------------------------------
Tensor multi_tensor_l2norm(const std::vector<Tensor>& tensors) {
  TORCH_CHECK(!tensors.empty(), "empty tensor list");
  const c10::cuda::CUDAGuard guard(tensors[0].device());
  const int max_ctas = ub::l2norm_max_ctas();
  // [0] running sum of squares, [1] ticket counter (as uint32), [2] result, [3..] per-CTA partials
  Tensor ws = torch::zeros({3 + max_ctas}, tensors[0].options().dtype(at::kFloat));
  float* base = ws.data_ptr<float>();
  const size_t n = tensors.size();
  for (size_t begin = 0; begin < n; begin += ub::kMaxTensorsPerLaunch) {
    ub::NormTensors t{};
    const size_t end = std::min(n, begin + (size_t)ub::kMaxTensorsPerLaunch);
    for (size_t i = begin; i < end; ++i) {
      check_cuda_contig(tensors[i], "l2norm input");
      t.ptr[i - begin] = tensors[i].data_ptr();
      t.numel[i - begin] = tensors[i].numel();
      t.dtype[i - begin] = dtype_tag(tensors[i]);
    }
    t.count = (int)(end - begin);
    ub::launch_l2norm(t, base, base + 3, reinterpret_cast<unsigned*>(base + 1), base + 2, end == n ? 1 : 0,
                      cur_stream());
  }
  check_launch("l2norm");
  return ws.select(0, 2);  // 0-dim view
}

void multi_tensor_scale(const std::vector<Tensor>& tensors, double scale, const OptTensor& scale_dev) {
  if (tensors.empty()) return;
  const c10::cuda::CUDAGuard guard(tensors[0].device());
  const float* sd = nullptr;
  if (scale_dev.has_value() && scale_dev->defined()) {
    TORCH_CHECK(scale_dev->is_cuda() && scale_dev->scalar_type() == at::kFloat && scale_dev->numel() == 1);
    sd = scale_dev->data_ptr<float>();
  }
  const size_t n = tensors.size();
  for (size_t begin = 0; begin < n; begin += ub::kMaxTensorsPerLaunch) {
    ub::ScaleTensors t{};
    const size_t end = std::min(n, begin + (size_t)ub::kMaxTensorsPerLaunch);
    for (size_t i = begin; i < end; ++i) {
      check_cuda_contig(tensors[i], "scale input");
      t.ptr[i - begin] = tensors[i].data_ptr();
      t.numel[i - begin] = tensors[i].numel();
      t.dtype[i - begin] = dtype_tag(tensors[i]);
    }
    t.count = (int)(end - begin);
    ub::launch_scale(t, (float)scale, sd, cur_stream());
  }
  check_launch("scale");
}

void multi_tensor_adam(const std::vector<Tensor>& p, const std::vector<Tensor>& g, const std::vector<Tensor>& m,
                       const std::vector<Tensor>& v, const std::vector<OptTensor>& p_half,
                       const std::vector<double>& lr, const std::vector<double>& beta1,
                       const std::vector<double>& beta2, const std::vector<double>& eps,
                       const std::vector<int64_t>& step, const std::vector<bool>& bias_correction,
                       const std::vector<double>& weight_decay, double grad_scale, const OptTensor& scale_dev,
                       bool zero_grad, bool stochastic_rounding, const std::vector<OptTensor>& ema, double ema_decay) {
  const size_t n = p.size();
  TORCH_CHECK(n > 0 && g.size() == n && m.size() == n && v.size() == n && p_half.size() == n);
  TORCH_CHECK(ema.empty() || ema.size() == n, "ema: one (optional) fp32 buffer per tensor");
  const c10::cuda::CUDAGuard guard(p[0].device());
  ub::AdamLaunch cfg{};
  cfg.inv_scale = (float)(1.0 / grad_scale);
  cfg.scale_dev = nullptr;
  if (scale_dev.has_value() && scale_dev->defined()) {
    TORCH_CHECK(scale_dev->is_cuda() && scale_dev->scalar_type() == at::kFloat && scale_dev->numel() == 1);
    cfg.scale_dev = scale_dev->data_ptr<float>();
  }
  cfg.zero_grad = zero_grad ? 1 : 0;
  cfg.stochastic_rounding = stochastic_rounding ? 1 : 0;
  cfg.ema_decay = (float)ema_decay;
  cfg.seed = cfg.offset = 0;
  if (stochastic_rounding) {
    auto so = philox_reserve(4);
    cfg.seed = so.first;
    cfg.offset = so.second;
  }
  unsigned long long elem_base = 0;
  for (size_t begin = 0; begin < n; begin += ub::kMaxTensorsPerLaunch) {
    ub::AdamTensors t{};
    const size_t end = std::min(n, begin + (size_t)ub::kMaxTensorsPerLaunch);
    for (size_t i = begin; i < end; ++i) {
      const size_t k = i - begin;
      check_cuda_contig(p[i], "adam p");
      check_cuda_contig(g[i], "adam g");
      check_cuda_contig(m[i], "adam m");
      check_cuda_contig(v[i], "adam v");
      TORCH_CHECK(m[i].scalar_type() == at::kFloat && v[i].scalar_type() == at::kFloat, "moments must be fp32");
      TORCH_CHECK(p[i].numel() == g[i].numel() && p[i].numel() == m[i].numel() && p[i].numel() == v[i].numel(),
                  "adam tensors must have equal numel");
      t.p[k] = p[i].data_ptr();
      t.g[k] = g[i].data_ptr();
      t.m[k] = m[i].data_ptr<float>();
      t.v[k] = v[i].data_ptr<float>();
      t.p_dtype[k] = dtype_tag(p[i]);
      t.g_dtype[k] = dtype_tag(g[i]);
      t.p_half[k] = nullptr;
      t.half_dtype[k] = ub::kF16;
      if (p_half[i].has_value() && p_half[i]->defined()) {
        check_cuda_contig(*p_half[i], "adam p_half");
        TORCH_CHECK(p_half[i]->numel() == p[i].numel());
        t.p_half[k] = p_half[i]->data_ptr();
        t.half_dtype[k] = dtype_tag(*p_half[i]);
      }
      t.ema[k] = nullptr;
      if (!ema.empty() && ema[i].has_value() && ema[i]->defined()) {
        // EMA of the updated fp32 weights in the same pass: ema -= (1 - decay) * (ema - p)
        check_cuda_contig(*ema[i], "adam ema");
        TORCH_CHECK(ema[i]->scalar_type() == at::kFloat && ema[i]->numel() == p[i].numel(), "ema must be fp32, same length");
        t.ema[k] = ema[i]->data_ptr<float>();
      }
      t.numel[k] = p[i].numel();
      double step_size = lr[i];
      if (bias_correction[i]) {
        const double bc1 = 1.0 - std::pow(beta1[i], (double)step[i]);
        const double bc2 = 1.0 - std::pow(beta2[i], (double)step[i]);
        step_size = lr[i] * std::sqrt(bc2) / bc1;
      }
      t.step_size[k] = (float)step_size;
      t.decay_mul[k] = (float)(1.0 - step_size * weight_decay[i]);
      t.beta1[k] = (float)beta1[i];
      t.beta2[k] = (float)beta2[i];
      t.eps[k] = (float)eps[i];
      t.elem_base[k] = elem_base;
      elem_base += ((unsigned long long)p[i].numel() + 7ull) & ~7ull;
    }
    t.count = (int)(end - begin);
    ub::launch_adam(t, cfg, cur_stream());
  }
  check_launch("adam");
}

void fp32_to_bf16_sr(const Tensor& in, Tensor out) {
  check_cuda_contig(in, "in");
  check_cuda_contig(out, "out");
  TORCH_CHECK(in.scalar_type() == at::kFloat && out.scalar_type() == at::kBFloat16 && in.numel() == out.numel());
  const c10::cuda::CUDAGuard guard(in.device());
  auto so = philox_reserve(4);
  ub::launch_fp32_to_bf16_sr(in.data_ptr<float>(), out.data_ptr(), in.numel(), so.first, so.second, cur_stream());
  check_launch("fp32_to_bf16_sr");
}

void ema_update(Tensor ema, const Tensor& p, double decay) {
  check_cuda_contig(ema, "ema");
  check_cuda_contig(p, "p");
  TORCH_CHECK(ema.scalar_type() == at::kFloat && p.scalar_type() == at::kFloat && ema.numel() == p.numel());
  const c10::cuda::CUDAGuard guard(ema.device());
  ub::launch_ema(ema.data_ptr<float>(), p.data_ptr<float>(), ema.numel(), (float)decay, cur_stream());
  check_launch("ema");
}

// ---------------------------------------------------------------------------------------------------
// norms
// ---------------------------------------------------------------------------------------------------
// The norm kernels read rows, gamma, beta and bias with 16-byte vector loads and bulk copies from the first element on.
void check_norm_operand(const Tensor& t, const char* name) {
  check_cuda_contig(t, name);
  TORCH_CHECK((reinterpret_cast<uintptr_t>(t.data_ptr()) & 15) == 0, name, " must be 16-byte aligned");
}

void check_norm_width(const Tensor& x) {
  TORCH_CHECK(x.dim() == 2, "norm input must be 2-D [rows, cols]");
  TORCH_CHECK(ub::norm_plan((int)x.size(0), (int)x.size(1), dtype_tag(x), ub::kNormFwd).gen != 0,
              "no norm kernel for this row width and dtype");
}

std::tuple<Tensor, Tensor, Tensor> layernorm_fwd(const Tensor& x, const Tensor& gamma, const Tensor& beta, double eps) {
  check_norm_operand(x, "x");
  check_norm_operand(gamma, "gamma");
  check_norm_operand(beta, "beta");
  check_norm_width(x);
  TORCH_CHECK(gamma.numel() == x.size(1) && beta.numel() == x.size(1));
  TORCH_CHECK(gamma.scalar_type() == x.scalar_type() && beta.scalar_type() == x.scalar_type());
  const c10::cuda::CUDAGuard guard(x.device());
  const int rows = (int)x.size(0), cols = (int)x.size(1);
  Tensor y = torch::empty_like(x);
  Tensor mean = torch::empty({rows}, x.options().dtype(at::kFloat));
  Tensor rstd = torch::empty({rows}, x.options().dtype(at::kFloat));
  ub::launch_layernorm_fwd(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), y.data_ptr(), mean.data_ptr<float>(),
                           rstd.data_ptr<float>(), rows, cols, (float)eps, dtype_tag(x), cur_stream());
  check_launch("layernorm_fwd");
  return {y, mean, rstd};
}

// A parameter-gradient "sink": the parameter's view of the optimizer's flat gradient arena.  When given, the kernel
// ADDS its result to the sink (and the sink is returned) - no temporary, no separate AccumulateGrad add kernel.
static Tensor grad_out(const OptTensor& sink, const Tensor& like, int bit, int& acc_mask) {
  if (sink.has_value() && sink->defined()) {
    TORCH_CHECK(sink->is_cuda() && sink->is_contiguous() && sink->scalar_type() == like.scalar_type() &&
                    sink->numel() == like.numel(),
                "gradient sink must match the parameter (dtype, length, contiguous)");
    acc_mask |= 1 << bit;
    return *sink;
  }
  return torch::empty_like(like);
}

std::tuple<Tensor, Tensor, Tensor> layernorm_bwd(const Tensor& dy, const Tensor& x, const Tensor& mean,
                                                 const Tensor& rstd, const Tensor& gamma, const OptTensor& dgamma_sink,
                                                 const OptTensor& dbeta_sink) {
  check_norm_operand(dy, "dy");
  check_norm_operand(x, "x");
  check_norm_operand(gamma, "gamma");
  check_norm_width(x);
  TORCH_CHECK(dy.sizes() == x.sizes() && dy.scalar_type() == x.scalar_type() && gamma.numel() == x.size(1));
  const c10::cuda::CUDAGuard guard(x.device());
  const int rows = (int)x.size(0), cols = (int)x.size(1);
  Tensor dx = torch::empty_like(x);
  int acc = 0;
  Tensor dgamma = grad_out(dgamma_sink, gamma, 0, acc), dbeta = grad_out(dbeta_sink, gamma, 1, acc);
  const int parts = ub::norm_bwd_parts(rows, cols, dtype_tag(x));
  Tensor part = torch::empty({3, parts, cols}, x.options().dtype(at::kFloat));
  ub::launch_layernorm_bwd(dy.data_ptr(), x.data_ptr(), mean.data_ptr<float>(), rstd.data_ptr<float>(),
                           gamma.data_ptr(), dx.data_ptr(), dgamma.data_ptr(), dbeta.data_ptr(),
                           part.data_ptr<float>(), rows, cols, dtype_tag(x), cur_stream(), acc,
                           at::globalContext().deterministicAlgorithms());
  check_launch("layernorm_bwd");
  return {dx, dgamma, dbeta};
}

std::tuple<Tensor, Tensor> rmsnorm_fwd(const Tensor& x, const Tensor& gamma, double eps) {
  check_norm_operand(x, "x");
  check_norm_operand(gamma, "gamma");
  check_norm_width(x);
  TORCH_CHECK(gamma.numel() == x.size(1) && gamma.scalar_type() == x.scalar_type());
  const c10::cuda::CUDAGuard guard(x.device());
  const int rows = (int)x.size(0), cols = (int)x.size(1);
  Tensor y = torch::empty_like(x);
  Tensor rstd = torch::empty({rows}, x.options().dtype(at::kFloat));
  ub::launch_rmsnorm_fwd(x.data_ptr(), gamma.data_ptr(), y.data_ptr(), rstd.data_ptr<float>(), rows, cols, (float)eps,
                         dtype_tag(x), cur_stream());
  check_launch("rmsnorm_fwd");
  return {y, rstd};
}

std::tuple<Tensor, Tensor> rmsnorm_bwd(const Tensor& dy, const Tensor& x, const Tensor& rstd, const Tensor& gamma,
                                       const OptTensor& dgamma_sink) {
  check_norm_operand(dy, "dy");
  check_norm_operand(x, "x");
  check_norm_operand(gamma, "gamma");
  check_norm_width(x);
  TORCH_CHECK(dy.sizes() == x.sizes() && dy.scalar_type() == x.scalar_type() && gamma.numel() == x.size(1));
  const c10::cuda::CUDAGuard guard(x.device());
  const int rows = (int)x.size(0), cols = (int)x.size(1);
  Tensor dx = torch::empty_like(x);
  int acc = 0;
  Tensor dgamma = grad_out(dgamma_sink, gamma, 0, acc);
  const int parts = ub::norm_bwd_parts(rows, cols, dtype_tag(x));
  Tensor part = torch::empty({3, parts, cols}, x.options().dtype(at::kFloat));
  ub::launch_rmsnorm_bwd(dy.data_ptr(), x.data_ptr(), rstd.data_ptr<float>(), gamma.data_ptr(), dx.data_ptr(),
                         dgamma.data_ptr(), part.data_ptr<float>(), rows, cols, dtype_tag(x), cur_stream(), acc,
                         at::globalContext().deterministicAlgorithms());
  check_launch("rmsnorm_bwd");
  return {dx, dgamma};
}

// Launch plans (no kernel runs): what the launchers do for a shape, so tests can check which path a shape reaches.
pybind11::dict norm_plan(int64_t rows, int64_t cols, at::ScalarType dtype, const std::string& kind) {
  TORCH_CHECK(kind == "fwd" || kind == "bwd" || kind == "fused", "kind must be fwd, bwd or fused (the fused forward)");
  TORCH_CHECK(dtype == at::kFloat || dtype == at::kHalf || dtype == at::kBFloat16, "unsupported dtype ", dtype);
  const int tag = dtype == at::kFloat ? ub::kF32 : (dtype == at::kHalf ? ub::kF16 : ub::kBF16);
  const ub::NormPlan p = ub::norm_plan((int)rows, (int)cols, tag,
                                       kind == "fwd" ? ub::kNormFwd : (kind == "bwd" ? ub::kNormBwd : ub::kNormFusedFwd));
  pybind11::dict d;
  d["gen"] = p.gen;
  d["nvec"] = p.nvec;
  d["vpl"] = p.vpl;
  d["lpr"] = p.lpr;
  d["r"] = p.r;
  d["tpr"] = p.tpr;
  d["groups"] = p.groups;
  d["vpt"] = p.vpt;
  d["full"] = (bool)p.full;
  d["grid"] = p.grid;
  d["threads"] = p.threads;
  d["tile_rows"] = p.tile_rows;
  d["units"] = p.units;
  d["rows_per_sweep"] = p.rows_per_sweep;
  d["tiles_min"] = p.tiles_min;
  d["tiles_max"] = p.tiles_max;
  return d;
}

pybind11::dict softmax_plan(int64_t rows, int64_t K, at::ScalarType dtype, bool aligned, const std::string& kind) {
  TORCH_CHECK(kind == "fwd" || kind == "bwd", "kind must be fwd or bwd");
  TORCH_CHECK(dtype == at::kFloat || dtype == at::kHalf || dtype == at::kBFloat16, "unsupported dtype ", dtype);
  const int tag = dtype == at::kFloat ? ub::kF32 : (dtype == at::kHalf ? ub::kF16 : ub::kBF16);
  const ub::SoftmaxPlan p = ub::softmax_plan(rows, (int)K, tag, aligned, kind == "bwd");
  pybind11::dict d;
  d["vec"] = (bool)p.vec;
  d["vpt"] = p.vpt;
  d["tpr"] = p.tpr;
  d["grid"] = p.grid;
  d["threads"] = p.threads;
  d["rows_per_sweep"] = p.rows_per_sweep;
  d["sweeps"] = p.sweeps;
  return d;
}

// ---------------------------------------------------------------------------------------------------
// softmax + dropout
// ---------------------------------------------------------------------------------------------------
struct SmBroadcast {
  long long rows, mask_div = 1, bias_rows = 1;
  int K;
};

static SmBroadcast softmax_broadcast_plan(const Tensor& x, const OptTensor& mask, const OptTensor& bias) {
  check_cuda_contig(x, "input");
  TORCH_CHECK(x.dim() == 3, "input must be 3-D [batch, q, k]");
  SmBroadcast b;
  b.rows = x.size(0) * x.size(1);
  b.K = (int)x.size(2);
  if (mask.has_value() && mask->defined()) {
    check_cuda_contig(*mask, "mask");
    TORCH_CHECK(mask->scalar_type() == x.scalar_type() && mask->dim() == 3 && mask->size(2) == b.K);
    const long long mask_rows = mask->size(0) * mask->size(1);
    TORCH_CHECK(mask_rows > 0 && b.rows % mask_rows == 0, "mask rows must divide input rows");
    b.mask_div = b.rows / mask_rows;
  }
  if (bias.has_value() && bias->defined()) {
    check_cuda_contig(*bias, "bias");
    TORCH_CHECK(bias->scalar_type() == x.scalar_type() && bias->dim() == 3 && bias->size(2) == b.K);
    b.bias_rows = bias->size(0) * bias->size(1);
    TORCH_CHECK(b.bias_rows > 0 && b.rows % b.bias_rows == 0, "bias rows must divide input rows");
  }
  return b;
}

// Returns (out, probs, seed, offset).  in_place: the probabilities overwrite x (the reference's contract, probs IS x);
// otherwise x is left untouched and the probabilities go to a fresh tensor - no clone pass in front of the kernel.
// Without dropout `out` and `probs` are the same tensor.
std::tuple<Tensor, Tensor, int64_t, int64_t> softmax_dropout_fwd(Tensor x, const OptTensor& mask, const OptTensor& bias,
                                                                 double p, bool training, bool in_place) {
  const SmBroadcast b = softmax_broadcast_plan(x, mask, bias);
  const c10::cuda::CUDAGuard guard(x.device());
  const float pf = training ? (float)p : 0.f;
  uint64_t seed = 0, offset = 0;
  Tensor probs = in_place ? x : torch::empty_like(x);
  Tensor out = probs;
  if (pf > 0.f) {
    auto so = philox_reserve(4);
    seed = so.first;
    offset = so.second;
    out = torch::empty_like(x);
  }
  ub::launch_softmax_dropout_fwd(x.data_ptr(), out.data_ptr(), opt_ptr(mask), opt_ptr(bias), b.rows, b.K, b.mask_div,
                                 b.bias_rows, pf, seed, offset, dtype_tag(x), cur_stream(), nullptr, nullptr,
                                 probs.data_ptr());
  check_launch("softmax_dropout_fwd");
  return {out, probs, (int64_t)seed, (int64_t)offset};
}

// Logits mode: x is read-only; returns (dropout(softmax(z)), z = x + mask + bias, row log-sum-exp, seed, offset).
std::tuple<Tensor, Tensor, Tensor, int64_t, int64_t> softmax_dropout_logits_fwd(const Tensor& x, const OptTensor& mask,
                                                                                 const OptTensor& bias, double p,
                                                                                 bool training) {
  const SmBroadcast b = softmax_broadcast_plan(x, mask, bias);
  const c10::cuda::CUDAGuard guard(x.device());
  const float pf = training ? (float)p : 0.f;
  uint64_t seed = 0, offset = 0;
  if (pf > 0.f) {
    auto so = philox_reserve(4);
    seed = so.first;
    offset = so.second;
  }
  Tensor out = torch::empty_like(x), logits = torch::empty_like(x);
  Tensor lse = torch::empty({x.size(0), x.size(1)}, x.options().dtype(torch::kFloat32));
  ub::launch_softmax_dropout_fwd(x.data_ptr(), out.data_ptr(), opt_ptr(mask), opt_ptr(bias), b.rows, b.K, b.mask_div,
                                 b.bias_rows, pf, seed, offset, dtype_tag(x), cur_stream(), logits.data_ptr(),
                                 lse.data_ptr<float>());
  check_launch("softmax_dropout_logits_fwd");
  return {out, logits, lse, (int64_t)seed, (int64_t)offset};
}

Tensor softmax_dropout_logits_bwd(const Tensor& dy, const Tensor& logits, const Tensor& lse, const OptTensor& addend,
                                  double p, int64_t seed, int64_t offset) {
  check_cuda_contig(dy, "grad_output");
  check_cuda_contig(logits, "logits");
  check_cuda_contig(lse, "lse");
  TORCH_CHECK(dy.dim() == 3 && dy.sizes() == logits.sizes() && dy.scalar_type() == logits.scalar_type());
  TORCH_CHECK(lse.scalar_type() == torch::kFloat32 && lse.numel() == dy.size(0) * dy.size(1));
  if (addend.has_value() && addend->defined()) {
    check_cuda_contig(*addend, "grad_logits");
    TORCH_CHECK(addend->sizes() == dy.sizes() && addend->scalar_type() == dy.scalar_type());
  }
  const c10::cuda::CUDAGuard guard(dy.device());
  Tensor dx = torch::empty_like(dy);
  ub::launch_softmax_dropout_bwd(dy.data_ptr(), dx.data_ptr(), logits.data_ptr(), dy.size(0) * dy.size(1),
                                 (int)dy.size(2), (float)p, (uint64_t)seed, (uint64_t)offset, dtype_tag(dy),
                                 cur_stream(), lse.data_ptr<float>(), opt_ptr(addend));
  check_launch("softmax_dropout_logits_bwd");
  return dx;
}

Tensor softmax_dropout_bwd(Tensor dy, const Tensor& probs, double p, int64_t seed, int64_t offset) {
  check_cuda_contig(dy, "grad_output");
  check_cuda_contig(probs, "softmax_results");
  TORCH_CHECK(dy.dim() == 3 && dy.sizes() == probs.sizes() && dy.scalar_type() == probs.scalar_type());
  const c10::cuda::CUDAGuard guard(dy.device());
  // out of place: autograd may hand the same grad tensor to several consumers
  Tensor dx = torch::empty_like(dy);
  ub::launch_softmax_dropout_bwd(dy.data_ptr(), dx.data_ptr(), probs.data_ptr(), dy.size(0) * dy.size(1),
                                 (int)dy.size(2), (float)p, (uint64_t)seed, (uint64_t)offset, dtype_tag(dy),
                                 cur_stream());
  check_launch("softmax_dropout_bwd");
  return dx;
}

// ---------------------------------------------------------------------------------------------------
// fused element-wise
// ---------------------------------------------------------------------------------------------------
Tensor bias_gelu_fwd(const Tensor& x, const OptTensor& bias) {
  check_cuda_contig(x, "x");
  const c10::cuda::CUDAGuard guard(x.device());
  const int cols = (int)x.size(-1);
  TORCH_CHECK(cols % 8 == 0 && (x.scalar_type() == at::kHalf || x.scalar_type() == at::kBFloat16));
  Tensor y = torch::empty_like(x);
  ub::launch_bias_gelu_fwd(x.data_ptr(), opt_ptr(bias), y.data_ptr(), x.numel() / cols, cols, dtype_tag(x),
                           cur_stream());
  check_launch("bias_gelu_fwd");
  return y;
}

// returns (dx, dbias); dbias (column sums of dx, produced by the same pass) only when a bias was given
std::tuple<Tensor, OptTensor> bias_gelu_bwd(const Tensor& dy, const Tensor& x, const OptTensor& bias,
                                            const OptTensor& dbias_sink) {
  check_cuda_contig(dy, "dy");
  check_cuda_contig(x, "x");
  const c10::cuda::CUDAGuard guard(x.device());
  const int cols = (int)x.size(-1);
  const long long rows = x.numel() / cols;
  Tensor dx = torch::empty_like(x);
  OptTensor dbias;
  Tensor part;
  const bool has_bias = bias.has_value() && bias->defined();
  int acc = 0;
  if (has_bias) {
    dbias = grad_out(dbias_sink, *bias, 0, acc);
    part = torch::empty({ub::bias_gelu_parts(rows, cols), cols}, x.options().dtype(at::kFloat));
  }
  ub::launch_bias_gelu_bwd(dy.data_ptr(), x.data_ptr(), opt_ptr(bias), dx.data_ptr(),
                           has_bias ? dbias->data_ptr() : nullptr, has_bias ? part.data_ptr<float>() : nullptr, rows,
                           cols, dtype_tag(x), cur_stream(), acc);
  check_launch("bias_gelu_bwd");
  return {dx, dbias};
}

// column sums over all leading dims: x [..., cols] -> [cols] (bias gradient of a Linear layer)
Tensor column_sum(const Tensor& x, const OptTensor& sink) {
  check_cuda_contig(x, "x");
  TORCH_CHECK(x.scalar_type() == at::kHalf || x.scalar_type() == at::kBFloat16, "column_sum supports fp16 / bf16");
  const int cols = (int)x.size(-1);
  TORCH_CHECK(cols % 8 == 0 && (reinterpret_cast<uintptr_t>(x.data_ptr()) & 15) == 0, "column_sum needs 16-byte rows");
  const long long rows = x.numel() / cols;
  TORCH_CHECK(rows < (1ll << 31), "too many rows");
  const c10::cuda::CUDAGuard guard(x.device());
  int acc = 0;
  Tensor out = grad_out(sink, torch::empty({cols}, x.options()), 0, acc);
  Tensor part = torch::empty({ub::bias_gelu_parts(rows, cols), cols}, x.options().dtype(at::kFloat));
  ub::launch_column_sum(x.data_ptr(), out.data_ptr(), part.data_ptr<float>(), rows, cols, dtype_tag(x), cur_stream(),
                        acc);
  check_launch("column_sum");
  return out;
}

// grad[tokens[r], :] (+)= dy[r, :]  (csrc/fused/embedding.cu); scratch fp32 [V, D] and touched uint8 [V] are persistent,
// zero between calls.  `grad` is either the parameter's arena view (accumulate) or a zero-filled tensor.
void embedding_bwd(const Tensor& dy, const Tensor& tokens, int64_t padding_idx, Tensor scratch, Tensor touched, Tensor grad,
                   bool accumulate) {
  check_cuda_contig(dy, "dy");
  check_cuda_contig(tokens, "tokens");
  check_cuda_contig(grad, "grad");
  TORCH_CHECK(dy.scalar_type() == at::kHalf || dy.scalar_type() == at::kBFloat16, "embedding_bwd supports fp16 / bf16");
  TORCH_CHECK(grad.scalar_type() == dy.scalar_type() && grad.dim() == 2 && tokens.scalar_type() == at::kLong);
  const int cols = (int)grad.size(1);
  const long long vocab = grad.size(0);
  TORCH_CHECK(dy.size(-1) == cols && cols % 8 == 0 && dy.numel() / cols == tokens.numel(), "embedding_bwd: shape mismatch");
  TORCH_CHECK((reinterpret_cast<uintptr_t>(dy.data_ptr()) & 15) == 0 && (reinterpret_cast<uintptr_t>(grad.data_ptr()) & 15) == 0,
              "embedding_bwd needs 16-byte aligned rows");
  TORCH_CHECK(scratch.is_cuda() && scratch.is_contiguous() && scratch.scalar_type() == at::kFloat && scratch.numel() == vocab * cols);
  TORCH_CHECK(touched.is_cuda() && touched.is_contiguous() && touched.scalar_type() == at::kByte && touched.numel() == vocab);
  const c10::cuda::CUDAGuard guard(dy.device());
  if (at::globalContext().deterministicAlgorithms()) {
    // fixed summation order: each vocabulary row sums its rows in ascending original order (scratch / touched unused)
    const auto sorted = at::sort(tokens.reshape({-1}), /*stable=*/true, /*dim=*/0, /*descending=*/false);
    const Tensor& ids = std::get<0>(sorted);
    const Tensor& perm = std::get<1>(sorted);
    ub::launch_embedding_bwd_sorted(dy.data_ptr(), reinterpret_cast<const long long*>(ids.data_ptr<int64_t>()),
                                    reinterpret_cast<const long long*>(perm.data_ptr<int64_t>()), grad.data_ptr(),
                                    tokens.numel(), cols, vocab, padding_idx, accumulate ? 1 : 0, dtype_tag(dy),
                                    cur_stream());
    check_launch("embedding_bwd");
    return;
  }
  ub::launch_embedding_bwd(dy.data_ptr(), tokens.data_ptr<int64_t>() == nullptr ? nullptr : reinterpret_cast<const long long*>(tokens.data_ptr<int64_t>()),
                           scratch.data_ptr<float>(), touched.data_ptr<uint8_t>(), grad.data_ptr(), tokens.numel(), cols, vocab,
                           padding_idx, accumulate ? 1 : 0, dtype_tag(dy), cur_stream());
  check_launch("embedding_bwd");
}

std::tuple<Tensor, Tensor, Tensor, Tensor, int64_t, int64_t> bias_dropout_add_ln_fwd(
    const Tensor& x, const OptTensor& bias, const Tensor& residual, const Tensor& gamma, const Tensor& beta, double p,
    double eps) {
  check_norm_operand(x, "x");
  check_norm_operand(residual, "residual");
  check_norm_operand(gamma, "gamma");
  check_norm_operand(beta, "beta");
  if (bias.has_value() && bias->defined()) check_norm_operand(*bias, "bias");
  check_norm_width(x);
  TORCH_CHECK(x.scalar_type() == at::kHalf || x.scalar_type() == at::kBFloat16, "bias_dropout_add_ln supports fp16 / bf16");
  TORCH_CHECK(residual.sizes() == x.sizes() && residual.scalar_type() == x.scalar_type());
  TORCH_CHECK(gamma.scalar_type() == x.scalar_type() && beta.scalar_type() == x.scalar_type());
  const c10::cuda::CUDAGuard guard(x.device());
  const int rows = (int)x.size(0), cols = (int)x.size(1);
  Tensor y = torch::empty_like(x), summed = torch::empty_like(x);
  Tensor mean = torch::empty({rows}, x.options().dtype(at::kFloat));
  Tensor rstd = torch::empty({rows}, x.options().dtype(at::kFloat));
  uint64_t seed = 0, offset = 0;
  if (p > 0.0) {
    auto so = philox_reserve(4);
    seed = so.first;
    offset = so.second;
  }
  ub::launch_bias_dropout_add_ln_fwd(x.data_ptr(), opt_ptr(bias), residual.data_ptr(), gamma.data_ptr(),
                                     beta.data_ptr(), y.data_ptr(), summed.data_ptr(), mean.data_ptr<float>(),
                                     rstd.data_ptr<float>(), rows, cols, (float)p, (float)eps, seed, offset,
                                     dtype_tag(x), cur_stream());
  check_launch("bias_dropout_add_ln_fwd");
  return {y, mean, rstd, summed, (int64_t)seed, (int64_t)offset};
}

// returns (dsum, dx, dgamma, dbeta, dbias); dbias is undefined unless `need_dbias` and the geometry allows
// the in-kernel column sums (the caller then reduces dx itself)
std::tuple<Tensor, Tensor, Tensor, Tensor, OptTensor> bias_dropout_add_ln_bwd(const Tensor& dy, const Tensor& summed,
                                                                              const Tensor& mean, const Tensor& rstd,
                                                                              const Tensor& gamma, double p,
                                                                              int64_t seed, int64_t offset,
                                                                              bool need_dbias,
                                                                              const OptTensor& dgamma_sink,
                                                                              const OptTensor& dbeta_sink,
                                                                              const OptTensor& dbias_sink) {
  check_norm_operand(dy, "dy");
  check_norm_operand(summed, "summed");
  check_norm_operand(gamma, "gamma");
  check_norm_width(summed);
  TORCH_CHECK(summed.scalar_type() == at::kHalf || summed.scalar_type() == at::kBFloat16,
              "bias_dropout_add_ln supports fp16 / bf16");
  TORCH_CHECK(dy.sizes() == summed.sizes() && dy.scalar_type() == summed.scalar_type() && gamma.numel() == summed.size(1));
  const c10::cuda::CUDAGuard guard(dy.device());
  const int rows = (int)summed.size(0), cols = (int)summed.size(1);
  Tensor dsum = torch::empty_like(summed);
  Tensor dx = p > 0.0 ? torch::empty_like(summed) : dsum;
  int acc = 0;
  Tensor dgamma = grad_out(dgamma_sink, gamma, 0, acc), dbeta = grad_out(dbeta_sink, gamma, 1, acc);
  const int parts = ub::norm_bwd_parts(rows, cols, dtype_tag(summed));
  Tensor part = torch::empty({3, parts, cols}, summed.options().dtype(at::kFloat));
  OptTensor dbias;
  if (need_dbias && ub::norm_v2_supported(cols, dtype_tag(summed))) dbias = grad_out(dbias_sink, gamma, 2, acc);
  ub::launch_bias_dropout_add_ln_bwd(dy.data_ptr(), summed.data_ptr(), mean.data_ptr<float>(),
                                     rstd.data_ptr<float>(), gamma.data_ptr(), dsum.data_ptr(), dx.data_ptr(),
                                     dgamma.data_ptr(), dbeta.data_ptr(), dbias.has_value() ? dbias->data_ptr() : nullptr,
                                     part.data_ptr<float>(), rows, cols, (float)p, (uint64_t)seed, (uint64_t)offset,
                                     dtype_tag(summed), cur_stream(), acc,
                                     at::globalContext().deterministicAlgorithms());
  check_launch("bias_dropout_add_ln_bwd");
  return {dsum, dx, dgamma, dbeta, dbias};
}

// `logits` is [rows, stride] contiguous of which the first `valid_cols` columns are the vocabulary (the
// rest is GEMM-alignment padding); valid_cols <= 0 means all columns.
std::tuple<Tensor, Tensor> softmax_xent_fwd(const Tensor& logits, const Tensor& target, int64_t ignore_index,
                                            int64_t valid_cols) {
  check_cuda_contig(logits, "logits");
  check_cuda_contig(target, "target");
  TORCH_CHECK(logits.dim() == 2 && target.dim() == 1 && target.size(0) == logits.size(0));
  TORCH_CHECK(target.scalar_type() == at::kLong);
  TORCH_CHECK(valid_cols <= logits.size(1));
  const c10::cuda::CUDAGuard guard(logits.device());
  const int rows = (int)logits.size(0), stride = (int)logits.size(1);
  const int cols = valid_cols > 0 ? (int)valid_cols : stride;
  Tensor loss = torch::empty({rows}, logits.options().dtype(at::kFloat));
  Tensor lse = torch::empty({rows}, logits.options().dtype(at::kFloat));
  ub::launch_softmax_xent_fwd(logits.data_ptr(), (const long long*)target.data_ptr<int64_t>(), loss.data_ptr<float>(),
                              lse.data_ptr<float>(), rows, cols, stride, ignore_index, dtype_tag(logits), cur_stream());
  check_launch("softmax_xent_fwd");
  return {loss, lse};
}

Tensor softmax_xent_bwd(const Tensor& logits, const Tensor& target, const Tensor& lse, const Tensor& dloss,
                        int64_t ignore_index, int64_t valid_cols) {
  check_cuda_contig(logits, "logits");
  TORCH_CHECK(dloss.is_cuda() && dloss.scalar_type() == at::kFloat && dloss.numel() == 1);
  const c10::cuda::CUDAGuard guard(logits.device());
  const int rows = (int)logits.size(0), stride = (int)logits.size(1);
  const int cols = valid_cols > 0 ? (int)valid_cols : stride;
  Tensor dlogits = torch::empty_like(logits);
  ub::launch_softmax_xent_bwd(logits.data_ptr(), (const long long*)target.data_ptr<int64_t>(), lse.data_ptr<float>(),
                              dloss.data_ptr<float>(), dlogits.data_ptr(), rows, cols, stride, ignore_index,
                              dtype_tag(logits), cur_stream());
  check_launch("softmax_xent_bwd");
  return dlogits;
}

// ---------------------------------------------------------------------------------------------------
// head split / merge
// ---------------------------------------------------------------------------------------------------
static void check_head_geometry(const Tensor& ref, int64_t D) {
  TORCH_CHECK(ref.scalar_type() == at::kHalf || ref.scalar_type() == at::kBFloat16 || ref.scalar_type() == at::kFloat,
              "head permute supports fp16 / bf16 / fp32");
  TORCH_CHECK((D * ref.element_size()) % 16 == 0, "head_dim must span whole 16-byte vectors");
}

// x: [B, L, T*H*D] contiguous -> T tensors [B, H, L, D] (slices of one allocation); slice 0 scaled by scale0
std::vector<Tensor> split_heads(const Tensor& x, int64_t T, int64_t H, double scale0) {
  check_cuda_contig(x, "input");
  TORCH_CHECK(x.dim() == 3 && T >= 1 && T <= 4 && H >= 1 && x.size(2) % (T * H) == 0, "expected [B, L, T*H*D]");
  const int64_t B = x.size(0), L = x.size(1), D = x.size(2) / (T * H);
  check_head_geometry(x, D);
  TORCH_CHECK((reinterpret_cast<uintptr_t>(x.data_ptr()) & 15) == 0, "input must be 16-byte aligned");
  const c10::cuda::CUDAGuard guard(x.device());
  Tensor packed = torch::empty({T, B, H, L, D}, x.options());
  std::vector<Tensor> out;
  void* ptrs[4] = {nullptr, nullptr, nullptr, nullptr};
  for (int64_t t = 0; t < T; ++t) {
    out.push_back(packed.select(0, t));
    ptrs[t] = out.back().data_ptr();
  }
  ub::launch_head_permute(x.data_ptr(), ptrs, (int)B, (int)L, (int)T, (int)H, (int)D, (float)scale0, true, dtype_tag(x),
                          cur_stream());
  check_launch("split_heads");
  return out;
}

// heads: T optional tensors [B, H, L, D] (undefined = zeros) -> [B, L, T*H*D]; slice 0 scaled by scale0
Tensor merge_heads(const std::vector<OptTensor>& heads, double scale0) {
  const int64_t T = (int64_t)heads.size();
  TORCH_CHECK(T >= 1 && T <= 4);
  const Tensor* ref = nullptr;
  for (const auto& h : heads)
    if (h.has_value() && h->defined()) ref = &*h;
  TORCH_CHECK(ref != nullptr, "merge_heads needs at least one defined tensor");
  TORCH_CHECK(ref->dim() == 4, "expected [B, H, L, D]");
  const int64_t B = ref->size(0), H = ref->size(1), L = ref->size(2), D = ref->size(3);
  check_head_geometry(*ref, D);
  void* ptrs[4] = {nullptr, nullptr, nullptr, nullptr};
  for (int64_t t = 0; t < T; ++t) {
    if (!(heads[t].has_value() && heads[t]->defined())) continue;
    const Tensor& h = *heads[t];
    check_cuda_contig(h, "head-major tensor");
    TORCH_CHECK(h.sizes() == ref->sizes() && h.scalar_type() == ref->scalar_type());
    TORCH_CHECK((reinterpret_cast<uintptr_t>(h.data_ptr()) & 15) == 0, "head-major tensors must be 16-byte aligned");
    ptrs[t] = h.data_ptr();
  }
  const c10::cuda::CUDAGuard guard(ref->device());
  Tensor out = torch::empty({B, L, T * H * D}, ref->options());
  ub::launch_head_permute(out.data_ptr(), ptrs, (int)B, (int)L, (int)T, (int)H, (int)D, (float)scale0, false,
                          dtype_tag(*ref), cur_stream());
  check_launch("merge_heads");
  return out;
}

// ---------------------------------------------------------------------------------------------------
// pair representation relayout
// ---------------------------------------------------------------------------------------------------
static void check_pair_operand(const Tensor& t, const char* what) {
  check_cuda_contig(t, what);
  TORCH_CHECK(t.dim() == 4, what, " must be 4-D");
  TORCH_CHECK(t.scalar_type() == at::kHalf || t.scalar_type() == at::kBFloat16, what, " must be fp16 / bf16");
  TORCH_CHECK((reinterpret_cast<uintptr_t>(t.data_ptr()) & 15) == 0, what, " must be 16-byte aligned");
}

static const unsigned char* key_pad_ptr(const OptTensor& key_pad, int64_t B, int64_t Lk) {
  if (!(key_pad.has_value() && key_pad->defined())) return nullptr;
  check_cuda_contig(*key_pad, "key_padding_mask");
  TORCH_CHECK(key_pad->element_size() == 1 && key_pad->dim() == 2 && key_pad->size(0) == B && key_pad->size(1) == Lk,
              "key_padding_mask must be a [B, Lk] bool / uint8 tensor");
  return reinterpret_cast<const unsigned char*>(key_pad->data_ptr());
}

// to_pair: [B, H, Lq, Lk] -> [B, Lq, Lk, H];  otherwise the inverse
Tensor pair_transpose(const Tensor& x, bool to_pair) {
  check_pair_operand(x, "input");
  const int64_t B = x.size(0);
  const int64_t H = to_pair ? x.size(1) : x.size(3);
  const int64_t Lq = to_pair ? x.size(2) : x.size(1), Lk = to_pair ? x.size(3) : x.size(2);
  TORCH_CHECK(H % 8 == 0 && (Lq * Lk) % 8 == 0, "pair_transpose needs H % 8 == 0 and Lq * Lk % 8 == 0");
  const c10::cuda::CUDAGuard guard(x.device());
  Tensor out = to_pair ? torch::empty({B, Lq, Lk, H}, x.options()) : torch::empty({B, H, Lq, Lk}, x.options());
  ub::launch_pair_transpose(x.data_ptr(), out.data_ptr(), (int)B, (int)H, Lq * Lk, to_pair, cur_stream());
  check_launch("pair_transpose");
  return out;
}

std::tuple<Tensor, Tensor> pair_tail_fwd(const Tensor& z, const Tensor& z0, const OptTensor& key_pad) {
  check_pair_operand(z, "logits");
  check_pair_operand(z0, "input bias");
  TORCH_CHECK(z.sizes() == z0.sizes() && z.scalar_type() == z0.scalar_type());
  const int64_t B = z.size(0), H = z.size(1), Lq = z.size(2), Lk = z.size(3);
  TORCH_CHECK(H % 8 == 0 && Lk % 8 == 0, "pair_tail needs H % 8 == 0 and Lk % 8 == 0");
  const unsigned char* pad = key_pad_ptr(key_pad, B, Lk);
  const c10::cuda::CUDAGuard guard(z.device());
  Tensor pair = torch::empty({B, Lq, Lk, H}, z.options()), delta = torch::empty({B, Lq, Lk, H}, z.options());
  ub::launch_pair_tail_fwd(z.data_ptr(), z0.data_ptr(), pad, pair.data_ptr(), delta.data_ptr(), (int)B, (int)H, (int)Lq,
                           (int)Lk, dtype_tag(z), cur_stream());
  check_launch("pair_tail_fwd");
  return {pair, delta};
}

std::tuple<Tensor, Tensor> pair_tail_bwd(const OptTensor& d_pair, const OptTensor& d_delta, const Tensor& z,
                                         const OptTensor& key_pad) {
  check_pair_operand(z, "logits");
  const int64_t B = z.size(0), H = z.size(1), Lq = z.size(2), Lk = z.size(3);
  for (const OptTensor* g : {&d_pair, &d_delta}) {
    if (!(g->has_value() && (*g)->defined())) continue;
    check_pair_operand(**g, "gradient");
    TORCH_CHECK((*g)->size(0) == B && (*g)->size(1) == Lq && (*g)->size(2) == Lk && (*g)->size(3) == H &&
                (*g)->scalar_type() == z.scalar_type());
  }
  const unsigned char* pad = key_pad_ptr(key_pad, B, Lk);
  const c10::cuda::CUDAGuard guard(z.device());
  Tensor dz = torch::empty_like(z), dz0 = torch::empty_like(z);
  ub::launch_pair_tail_bwd(opt_ptr(d_pair), opt_ptr(d_delta), z.data_ptr(), pad, dz.data_ptr(), dz0.data_ptr(), (int)B,
                           (int)H, (int)Lq, (int)Lk, dtype_tag(z), cur_stream());
  check_launch("pair_tail_bwd");
  return {dz, dz0};
}

// ---------------------------------------------------------------------------------------------------
// Gaussian basis (Uni-Mol)
// ---------------------------------------------------------------------------------------------------
Tensor gbf_fwd(const Tensor& d, const Tensor& edge, const Tensor& mul_w, const Tensor& bias_w, const Tensor& means,
               const Tensor& stds) {
  check_cuda_contig(d, "d");
  check_cuda_contig(edge, "edge");
  TORCH_CHECK(edge.scalar_type() == at::kLong && edge.numel() == d.numel());
  TORCH_CHECK(d.scalar_type() == at::kHalf || d.scalar_type() == at::kBFloat16);
  for (const Tensor* t : {&mul_w, &bias_w, &means, &stds})
    TORCH_CHECK(t->is_cuda() && t->is_contiguous() && t->scalar_type() == d.scalar_type());
  const int K = (int)means.numel();
  TORCH_CHECK(K % 8 == 0 && K / 8 <= 32 && ((K / 8) & (K / 8 - 1)) == 0 && stds.numel() == K, "K must be 8 * 2^i <= 256");
  const c10::cuda::CUDAGuard guard(d.device());
  auto sizes = d.sizes().vec();
  sizes.push_back(K);
  Tensor y = torch::empty(sizes, d.options());
  ub::launch_gbf_fwd(d.data_ptr(), (const long long*)edge.data_ptr<int64_t>(), mul_w.data_ptr(), bias_w.data_ptr(),
                     means.data_ptr(), stds.data_ptr(), y.data_ptr(), d.numel(), K, dtype_tag(d), cur_stream());
  check_launch("gbf_fwd");
  return y;
}

// returns (d mul [E], d bias [E], d means [K], d stds_abs [K]) in fp32
std::tuple<Tensor, Tensor, Tensor, Tensor> gbf_bwd(const Tensor& dy, const Tensor& d, const Tensor& edge,
                                                   const Tensor& mul_w, const Tensor& bias_w, const Tensor& means,
                                                   const Tensor& stds) {
  check_cuda_contig(dy, "dy");
  const int K = (int)means.numel(), E = (int)mul_w.numel();
  TORCH_CHECK(dy.scalar_type() == d.scalar_type() && dy.numel() == d.numel() * K && bias_w.numel() == E);
  TORCH_CHECK(E <= 8192, "edge-type table too large for the shared-memory histogram");
  const c10::cuda::CUDAGuard guard(d.device());
  const int parts = ub::gbf_parts(d.numel(), K);
  Tensor part = torch::empty({parts, 2 * K}, d.options().dtype(at::kFloat));
  Tensor hist = torch::zeros({2, E}, d.options().dtype(at::kFloat));
  if (at::globalContext().deterministicAlgorithms()) {
    // fixed summation order: per-row (dt * dist, dt) summed per edge type over the stable-sorted ids
    Tensor rowg = torch::empty({d.numel(), 2}, d.options().dtype(at::kFloat));
    const auto sorted = at::sort(edge.reshape({-1}), /*stable=*/true, /*dim=*/0, /*descending=*/false);
    ub::launch_gbf_bwd_det(dy.data_ptr(), d.data_ptr(), (const long long*)edge.data_ptr<int64_t>(), mul_w.data_ptr(),
                           bias_w.data_ptr(), means.data_ptr(), stds.data_ptr(), part.data_ptr<float>(),
                           rowg.data_ptr<float>(), (const long long*)std::get<0>(sorted).data_ptr<int64_t>(),
                           (const long long*)std::get<1>(sorted).data_ptr<int64_t>(), hist.data_ptr<float>(), d.numel(),
                           K, E, dtype_tag(d), cur_stream());
    check_launch("gbf_bwd");
    Tensor cols = part.sum(0);
    return {hist[0], hist[1], cols.slice(0, 0, K), cols.slice(0, K, 2 * K)};
  }
  ub::launch_gbf_bwd(dy.data_ptr(), d.data_ptr(), (const long long*)edge.data_ptr<int64_t>(), mul_w.data_ptr(),
                     bias_w.data_ptr(), means.data_ptr(), stds.data_ptr(), part.data_ptr<float>(), hist.data_ptr<float>(),
                     d.numel(), K, E, dtype_tag(d), cur_stream());
  check_launch("gbf_bwd");
  Tensor cols = part.sum(0);
  return {hist[0], hist[1], cols.slice(0, 0, K), cols.slice(0, K, 2 * K)};
}

}  // namespace

// defined in attn/fmha_bind.cpp and comm/comm_bind.cpp
void register_fmha(pybind11::module_& m);
void register_comm(pybind11::module_& m);
void register_symm_mem(pybind11::module_& m);

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "unicore_b200 sm_90a kernels";
  m.def("multi_tensor_l2norm", &multi_tensor_l2norm);
  m.def("multi_tensor_scale", &multi_tensor_scale);
  m.def("multi_tensor_adam", &multi_tensor_adam);
  m.def("fp32_to_bf16_sr", &fp32_to_bf16_sr);
  m.def("ema_update", &ema_update);
  m.def("layernorm_fwd", &layernorm_fwd);
  m.def("layernorm_bwd", &layernorm_bwd, pybind11::arg("dy"), pybind11::arg("x"), pybind11::arg("mean"), pybind11::arg("rstd"),
        pybind11::arg("gamma"), pybind11::arg("dgamma_sink") = pybind11::none(), pybind11::arg("dbeta_sink") = pybind11::none());
  m.def("rmsnorm_fwd", &rmsnorm_fwd);
  m.def("rmsnorm_bwd", &rmsnorm_bwd, pybind11::arg("dy"), pybind11::arg("x"), pybind11::arg("rstd"), pybind11::arg("gamma"),
        pybind11::arg("dgamma_sink") = pybind11::none());
  m.def("norm_plan", &norm_plan, pybind11::arg("rows"), pybind11::arg("cols"), pybind11::arg("dtype"), pybind11::arg("kind"));
  m.def("softmax_plan", &softmax_plan, pybind11::arg("rows"), pybind11::arg("K"), pybind11::arg("dtype"),
        pybind11::arg("aligned") = true, pybind11::arg("kind") = "fwd");
  m.def("softmax_dropout_fwd", &softmax_dropout_fwd);
  m.def("softmax_dropout_bwd", &softmax_dropout_bwd);
  m.def("softmax_dropout_logits_fwd", &softmax_dropout_logits_fwd);
  m.def("softmax_dropout_logits_bwd", &softmax_dropout_logits_bwd);
  m.def("bias_gelu_fwd", &bias_gelu_fwd);
  m.def("bias_gelu_bwd", &bias_gelu_bwd, pybind11::arg("dy"), pybind11::arg("x"), pybind11::arg("bias"),
        pybind11::arg("dbias_sink") = pybind11::none());
  m.def("embedding_bwd", &embedding_bwd);
  m.def("column_sum", &column_sum, pybind11::arg("x"), pybind11::arg("sink") = pybind11::none());
  m.def("bias_dropout_add_ln_fwd", &bias_dropout_add_ln_fwd);
  m.def("bias_dropout_add_ln_bwd", &bias_dropout_add_ln_bwd, pybind11::arg("dy"), pybind11::arg("summed"), pybind11::arg("mean"),
        pybind11::arg("rstd"), pybind11::arg("gamma"), pybind11::arg("p"), pybind11::arg("seed"), pybind11::arg("offset"),
        pybind11::arg("need_dbias"), pybind11::arg("dgamma_sink") = pybind11::none(),
        pybind11::arg("dbeta_sink") = pybind11::none(), pybind11::arg("dbias_sink") = pybind11::none());
  m.def("softmax_xent_fwd", &softmax_xent_fwd);
  m.def("softmax_xent_bwd", &softmax_xent_bwd);
  m.def("split_heads", &split_heads);
  m.def("merge_heads", &merge_heads);
  m.def("pair_transpose", &pair_transpose);
  m.def("pair_tail_fwd", &pair_tail_fwd);
  m.def("pair_tail_bwd", &pair_tail_bwd);
  m.def("gbf_fwd", &gbf_fwd);
  m.def("gbf_bwd", &gbf_bwd);
  register_fmha(m);
  register_comm(m);
  register_symm_mem(m);
}
