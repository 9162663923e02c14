// PyTorch bindings of the unicore_b200 sm_90a kernels (module ``unicore_b200._C``).
// Only the binding translation units see the PyTorch headers; kernels are declared in csrc/api.h.
#include <c10/cuda/CUDAGuard.h>

#include <tuple>
#include <vector>

#include "api.h"
#include "bind_util.h"

namespace {

using namespace ub_bind;

// ---------------------------------------------------------------------------------------------------
// optimizer ops
// ---------------------------------------------------------------------------------------------------
Tensor multi_tensor_l2norm(const std::vector<Tensor>& tensors) {
  TORCH_CHECK(!tensors.empty(), "empty tensor list");
  const c10::Device dev = tensors[0].device();
  for (const Tensor& t : tensors) check_operand(t, "l2norm input", dev, kFloating);
  const c10::cuda::CUDAGuard guard(dev);
  const int max_ctas = ub::l2norm_max_ctas();
  // [0] running sum of squares, [1] ticket counter (as uint32), [2] result, [3..] per-CTA partials
  Tensor ws = torch::zeros({3 + max_ctas}, tensors[0].options().dtype(at::kFloat));
  float* base = ws.data_ptr<float>();
  const size_t n = tensors.size();
  for (size_t begin = 0; begin < n; begin += ub::kMaxTensorsPerLaunch) {
    ub::NormTensors t{};
    const size_t end = std::min(n, begin + (size_t)ub::kMaxTensorsPerLaunch);
    for (size_t i = begin; i < end; ++i) {
      t.ptr[i - begin] = tensors[i].data_ptr();
      t.numel[i - begin] = tensors[i].numel();
      t.dtype[i - begin] = dtype_tag(tensors[i].scalar_type());
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
  const c10::Device dev = tensors[0].device();
  for (const Tensor& t : tensors) check_operand(t, "scale input", dev, kFloating);
  check_operand(scale_dev, "scale_dev", dev, {at::kFloat}, {1}, kNumel);
  const c10::cuda::CUDAGuard guard(dev);
  const float* sd = has(scale_dev) ? scale_dev->data_ptr<float>() : nullptr;
  const size_t n = tensors.size();
  for (size_t begin = 0; begin < n; begin += ub::kMaxTensorsPerLaunch) {
    ub::ScaleTensors t{};
    const size_t end = std::min(n, begin + (size_t)ub::kMaxTensorsPerLaunch);
    for (size_t i = begin; i < end; ++i) {
      t.ptr[i - begin] = tensors[i].data_ptr();
      t.numel[i - begin] = tensors[i].numel();
      t.dtype[i - begin] = dtype_tag(tensors[i].scalar_type());
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
  TORCH_CHECK(n > 0, "empty tensor list");
  for (size_t len : {g.size(), m.size(), v.size(), p_half.size(), lr.size(), beta1.size(), beta2.size(), eps.size(),
                     step.size(), bias_correction.size(), weight_decay.size()})
    TORCH_CHECK(len == n, "adam: every per-tensor list needs one entry per parameter");
  TORCH_CHECK(ema.empty() || ema.size() == n, "ema: one (optional) fp32 buffer per tensor");
  const c10::Device dev = p[0].device();
  for (size_t i = 0; i < n; ++i) {
    const int64_t len = p[i].numel();
    check_operand(p[i], "p", dev, kFloating);
    check_operand(g[i], "g", dev, kFloating, {len}, kContig | kNumel);
    check_operand(m[i], "m", dev, {at::kFloat}, {len}, kContig | kNumel);
    check_operand(v[i], "v", dev, {at::kFloat}, {len}, kContig | kNumel);
    check_operand(p_half[i], "p_half", dev, kFloating, {len}, kContig | kNumel);
    // EMA of the updated fp32 weights in the same pass: ema -= (1 - decay) * (ema - p)
    if (!ema.empty()) check_operand(ema[i], "ema", dev, {at::kFloat}, {len}, kContig | kNumel);
  }
  check_operand(scale_dev, "scale_dev", dev, {at::kFloat}, {1}, kNumel);
  const c10::cuda::CUDAGuard guard(dev);
  ub::AdamLaunch cfg{};
  cfg.inv_scale = (float)(1.0 / grad_scale);
  cfg.scale_dev = has(scale_dev) ? scale_dev->data_ptr<float>() : nullptr;
  cfg.zero_grad = zero_grad ? 1 : 0;
  cfg.stochastic_rounding = stochastic_rounding ? 1 : 0;
  cfg.ema_decay = (float)ema_decay;
  cfg.seed = cfg.offset = 0;
  if (stochastic_rounding) std::tie(cfg.seed, cfg.offset) = philox_reserve(4);
  unsigned long long elem_base = 0;
  for (size_t begin = 0; begin < n; begin += ub::kMaxTensorsPerLaunch) {
    ub::AdamTensors t{};
    const size_t end = std::min(n, begin + (size_t)ub::kMaxTensorsPerLaunch);
    for (size_t i = begin; i < end; ++i) {
      const size_t k = i - begin;
      t.p[k] = p[i].data_ptr();
      t.g[k] = g[i].data_ptr();
      t.m[k] = m[i].data_ptr<float>();
      t.v[k] = v[i].data_ptr<float>();
      t.p_dtype[k] = dtype_tag(p[i].scalar_type());
      t.g_dtype[k] = dtype_tag(g[i].scalar_type());
      t.p_half[k] = has(p_half[i]) ? p_half[i]->data_ptr() : nullptr;
      t.half_dtype[k] = has(p_half[i]) ? dtype_tag(p_half[i]->scalar_type()) : ub::kF16;
      t.ema[k] = !ema.empty() && has(ema[i]) ? ema[i]->data_ptr<float>() : nullptr;
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
  check_operand(in, "in", in.device(), {at::kFloat});
  check_operand(out, "out", in.device(), {at::kBFloat16}, {in.numel()}, kContig | kNumel);
  const c10::cuda::CUDAGuard guard(in.device());
  auto so = philox_reserve(4);
  ub::launch_fp32_to_bf16_sr(in.data_ptr<float>(), out.data_ptr(), in.numel(), so.first, so.second, cur_stream());
  check_launch("fp32_to_bf16_sr");
}

void ema_update(Tensor ema, const Tensor& p, double decay) {
  check_operand(ema, "ema", ema.device(), {at::kFloat});
  check_operand(p, "p", ema.device(), {at::kFloat}, {ema.numel()}, kContig | kNumel);
  const c10::cuda::CUDAGuard guard(ema.device());
  ub::launch_ema(ema.data_ptr<float>(), p.data_ptr<float>(), ema.numel(), (float)decay, cur_stream());
  check_launch("ema");
}

// ---------------------------------------------------------------------------------------------------
// norms
// ---------------------------------------------------------------------------------------------------
// The norm kernels read rows, gamma, beta and bias with 16-byte vector loads and bulk copies from the first element on,
// so every norm operand but mean / rstd is kVec.  x: [rows, cols] with a width some norm kernel handles.
void check_norm_width(const Tensor& x, const char* name, DTypes dtypes) {
  check_operand(x, name, x.device(), dtypes, any_shape(2), kVec);
  TORCH_CHECK(ub::norm_plan((int)x.size(0), (int)x.size(1), dtype_tag(x.scalar_type()), ub::kNormFwd).gen != 0,
              "no norm kernel for this row width and dtype");
}

// A parameter-gradient "sink": the parameter's view of the optimizer's flat gradient arena.  When given, the kernel
// ADDS its result to the sink (and the sink is returned) - no temporary, no separate AccumulateGrad add kernel.
void check_sink(const OptTensor& sink, const char* name, const Tensor& param) {
  check_operand(sink, name, param.device(), {param.scalar_type()}, {param.numel()}, kContig | kNumel);
}

Tensor grad_out(const OptTensor& sink, const Tensor& param, int bit, int& acc_mask) {
  if (!has(sink)) return torch::empty_like(param);
  acc_mask |= 1 << bit;
  return *sink;
}

std::tuple<Tensor, Tensor, Tensor> layernorm_fwd(const Tensor& x, const Tensor& gamma, const Tensor& beta, double eps) {
  check_norm_width(x, "x", kFloating);
  const int rows = (int)x.size(0), cols = (int)x.size(1), tag = dtype_tag(x.scalar_type());
  check_operand(gamma, "gamma", x.device(), {x.scalar_type()}, {cols}, kVec | kNumel);
  check_operand(beta, "beta", x.device(), {x.scalar_type()}, {cols}, kVec | kNumel);
  const c10::cuda::CUDAGuard guard(x.device());
  Tensor y = torch::empty_like(x);
  Tensor mean = torch::empty({rows}, x.options().dtype(at::kFloat));
  Tensor rstd = torch::empty({rows}, x.options().dtype(at::kFloat));
  ub::launch_layernorm_fwd(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), y.data_ptr(), mean.data_ptr<float>(),
                           rstd.data_ptr<float>(), rows, cols, (float)eps, tag, cur_stream());
  check_launch("layernorm_fwd");
  return {y, mean, rstd};
}

std::tuple<Tensor, Tensor, Tensor> layernorm_bwd(const Tensor& dy, const Tensor& x, const Tensor& mean,
                                                 const Tensor& rstd, const Tensor& gamma, const OptTensor& dgamma_sink,
                                                 const OptTensor& dbeta_sink) {
  check_norm_width(x, "x", kFloating);
  const int rows = (int)x.size(0), cols = (int)x.size(1), tag = dtype_tag(x.scalar_type());
  check_operand(dy, "dy", x.device(), {x.scalar_type()}, x.sizes(), kVec);
  check_operand(mean, "mean", x.device(), {at::kFloat}, {rows});
  check_operand(rstd, "rstd", x.device(), {at::kFloat}, {rows});
  check_operand(gamma, "gamma", x.device(), {x.scalar_type()}, {cols}, kVec | kNumel);
  check_sink(dgamma_sink, "dgamma_sink", gamma);
  check_sink(dbeta_sink, "dbeta_sink", gamma);
  const c10::cuda::CUDAGuard guard(x.device());
  Tensor dx = torch::empty_like(x);
  int acc = 0;
  Tensor dgamma = grad_out(dgamma_sink, gamma, 0, acc), dbeta = grad_out(dbeta_sink, gamma, 1, acc);
  Tensor part = torch::empty({3, ub::norm_bwd_parts(rows, cols, tag), cols}, x.options().dtype(at::kFloat));
  ub::launch_layernorm_bwd(dy.data_ptr(), x.data_ptr(), mean.data_ptr<float>(), rstd.data_ptr<float>(),
                           gamma.data_ptr(), dx.data_ptr(), dgamma.data_ptr(), dbeta.data_ptr(),
                           part.data_ptr<float>(), rows, cols, tag, cur_stream(), acc);
  check_launch("layernorm_bwd");
  return {dx, dgamma, dbeta};
}

std::tuple<Tensor, Tensor> rmsnorm_fwd(const Tensor& x, const Tensor& gamma, double eps) {
  check_norm_width(x, "x", kFloating);
  const int rows = (int)x.size(0), cols = (int)x.size(1), tag = dtype_tag(x.scalar_type());
  check_operand(gamma, "gamma", x.device(), {x.scalar_type()}, {cols}, kVec | kNumel);
  const c10::cuda::CUDAGuard guard(x.device());
  Tensor y = torch::empty_like(x);
  Tensor rstd = torch::empty({rows}, x.options().dtype(at::kFloat));
  ub::launch_rmsnorm_fwd(x.data_ptr(), gamma.data_ptr(), y.data_ptr(), rstd.data_ptr<float>(), rows, cols, (float)eps,
                         tag, cur_stream());
  check_launch("rmsnorm_fwd");
  return {y, rstd};
}

std::tuple<Tensor, Tensor> rmsnorm_bwd(const Tensor& dy, const Tensor& x, const Tensor& rstd, const Tensor& gamma,
                                       const OptTensor& dgamma_sink) {
  check_norm_width(x, "x", kFloating);
  const int rows = (int)x.size(0), cols = (int)x.size(1), tag = dtype_tag(x.scalar_type());
  check_operand(dy, "dy", x.device(), {x.scalar_type()}, x.sizes(), kVec);
  check_operand(rstd, "rstd", x.device(), {at::kFloat}, {rows});
  check_operand(gamma, "gamma", x.device(), {x.scalar_type()}, {cols}, kVec | kNumel);
  check_sink(dgamma_sink, "dgamma_sink", gamma);
  const c10::cuda::CUDAGuard guard(x.device());
  Tensor dx = torch::empty_like(x);
  int acc = 0;
  Tensor dgamma = grad_out(dgamma_sink, gamma, 0, acc);
  Tensor part = torch::empty({3, ub::norm_bwd_parts(rows, cols, tag), cols}, x.options().dtype(at::kFloat));
  ub::launch_rmsnorm_bwd(dy.data_ptr(), x.data_ptr(), rstd.data_ptr<float>(), gamma.data_ptr(), dx.data_ptr(),
                         dgamma.data_ptr(), part.data_ptr<float>(), rows, cols, tag, cur_stream(), acc);
  check_launch("rmsnorm_bwd");
  return {dx, dgamma};
}

// Launch plans (no kernel runs): what the launchers do for a shape, so tests can check which path a shape reaches.
pybind11::dict norm_plan(int64_t rows, int64_t cols, at::ScalarType dtype, const std::string& kind) {
  TORCH_CHECK(kind == "fwd" || kind == "bwd" || kind == "fused", "kind must be fwd, bwd or fused (the fused forward)");
  const ub::NormPlan p = ub::norm_plan((int)rows, (int)cols, dtype_tag(dtype),
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
  const ub::SoftmaxPlan p = ub::softmax_plan(rows, (int)K, dtype_tag(dtype), aligned, kind == "bwd");
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

// bias_gelu's forward (kind "fwd"), or its backward and column_sum (kind "bwd")
pybind11::dict bias_gelu_plan(int64_t rows, int64_t cols, const std::string& kind) {
  TORCH_CHECK(kind == "fwd" || kind == "bwd", "kind must be fwd or bwd (the backward and column_sum)");
  TORCH_CHECK(rows >= 1 && cols > 0 && cols % 8 == 0, "bias_gelu_plan needs rows >= 1 and a positive multiple of 8 columns");
  const ub::ColumnPlan p = ub::bias_gelu_plan(rows, (int)cols, kind == "fwd");
  pybind11::dict d;
  d["nvec"] = p.nvec;
  d["col_blocks"] = p.col_blocks;
  d["slices"] = p.slices;
  d["rows_per_sweep"] = p.rows_per_sweep;
  d["sweeps"] = p.sweeps;
  return d;
}

pybind11::dict gbf_plan(int64_t n, int64_t K, int64_t E) {
  TORCH_CHECK(n >= 1 && K % 8 == 0 && K / 8 >= 1 && K / 8 <= 32 && ((K / 8) & (K / 8 - 1)) == 0 && E >= 1 && E <= 8192,
              "gbf_plan needs n >= 1, K = 8 * 2^i <= 256 and 1 <= E <= 8192");
  const ub::GbfPlan p = ub::gbf_plan(n, (int)K, (int)E);
  pybind11::dict d;
  d["grid"] = p.grid;
  d["kvec"] = p.kvec;
  d["rows_per_cta"] = p.rows_per_cta;
  d["rows_per_sweep"] = p.rows_per_sweep;
  d["sweeps"] = p.sweeps;
  d["smem"] = p.smem;
  return d;
}

pybind11::dict sweep_dict(const ub::SweepPlan& p) {
  pybind11::dict d;
  d["grid"] = p.grid;
  d["items"] = p.items;
  d["items_per_sweep"] = p.items_per_sweep;
  d["sweeps"] = p.sweeps;
  return d;
}

pybind11::dict head_permute_plan(int64_t B, int64_t L, int64_t T, int64_t H, int64_t D, at::ScalarType dtype) {
  const int64_t esz = c10::elementSize(dtype);
  TORCH_CHECK(B >= 1 && L >= 1 && T >= 1 && T <= 4 && H >= 1 && D >= 1 && (D * esz) % 16 == 0,
              "head_permute_plan needs positive sizes, 1 <= T <= 4 and a head_dim of whole 16-byte vectors");
  return sweep_dict(ub::head_permute_plan((int)B, (int)L, (int)T, (int)H, (int)D, dtype_tag(dtype)));
}

pybind11::dict pair_plan(int64_t B, int64_t H, int64_t M) {
  TORCH_CHECK(B >= 1 && H >= 8 && H % 8 == 0 && M >= 8 && M % 8 == 0,
              "pair_plan needs B >= 1 and positive multiples of 8 for H and M");
  return sweep_dict(ub::pair_plan((int)B, (int)H, M));
}

pybind11::dict embedding_plan(int64_t rows, int64_t vocab) {
  TORCH_CHECK(rows >= 0 && vocab >= 1, "embedding_plan needs rows >= 0 and vocab >= 1");
  const ub::EmbeddingPlan p = ub::embedding_plan(rows, vocab);
  pybind11::dict d;
  d["scatter"] = sweep_dict(p.scatter);
  d["finalize"] = sweep_dict(p.finalize);
  d["sorted"] = sweep_dict(p.sorted);
  return d;
}

// ---------------------------------------------------------------------------------------------------
// softmax + dropout
// ---------------------------------------------------------------------------------------------------
struct SmBroadcast {
  long long rows, mask_div = 1, bias_rows = 1;
  int K;
};

// x [batch, q, k]; mask and bias [*, *, k] whose rows (the product of the first two dims) divide those of x
static SmBroadcast softmax_broadcast_plan(const Tensor& x, const OptTensor& mask, const OptTensor& bias) {
  check_operand(x, "input", x.device(), kFloating, any_shape(3));
  SmBroadcast b;
  b.rows = x.size(0) * x.size(1);
  b.K = (int)x.size(2);
  check_operand(mask, "mask", x.device(), {x.scalar_type()}, {kAnySize, kAnySize, b.K});
  check_operand(bias, "bias", x.device(), {x.scalar_type()}, {kAnySize, kAnySize, b.K});
  if (has(mask)) {
    const long long mask_rows = mask->size(0) * mask->size(1);
    TORCH_CHECK(mask_rows > 0 && b.rows % mask_rows == 0, "mask rows must divide input rows");
    b.mask_div = b.rows / mask_rows;
  }
  if (has(bias)) {
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
    std::tie(seed, offset) = philox_reserve(4);
    out = torch::empty_like(x);
  }
  ub::launch_softmax_dropout_fwd(x.data_ptr(), out.data_ptr(), opt_ptr(mask), opt_ptr(bias), b.rows, b.K, b.mask_div,
                                 b.bias_rows, pf, seed, offset, dtype_tag(x.scalar_type()), cur_stream(), nullptr,
                                 nullptr, probs.data_ptr());
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
  if (pf > 0.f) std::tie(seed, offset) = philox_reserve(4);
  Tensor out = torch::empty_like(x), logits = torch::empty_like(x);
  Tensor lse = torch::empty({x.size(0), x.size(1)}, x.options().dtype(torch::kFloat32));
  ub::launch_softmax_dropout_fwd(x.data_ptr(), out.data_ptr(), opt_ptr(mask), opt_ptr(bias), b.rows, b.K, b.mask_div,
                                 b.bias_rows, pf, seed, offset, dtype_tag(x.scalar_type()), cur_stream(),
                                 logits.data_ptr(), lse.data_ptr<float>());
  check_launch("softmax_dropout_logits_fwd");
  return {out, logits, lse, (int64_t)seed, (int64_t)offset};
}

Tensor softmax_dropout_logits_bwd(const Tensor& dy, const Tensor& logits, const Tensor& lse, const OptTensor& addend,
                                  double p, int64_t seed, int64_t offset) {
  check_operand(dy, "grad_output", dy.device(), kFloating, any_shape(3));
  check_operand(logits, "logits", dy.device(), {dy.scalar_type()}, dy.sizes());
  check_operand(lse, "lse", dy.device(), {at::kFloat}, {dy.size(0) * dy.size(1)}, kContig | kNumel);
  check_operand(addend, "grad_logits", dy.device(), {dy.scalar_type()}, dy.sizes());
  const c10::cuda::CUDAGuard guard(dy.device());
  Tensor dx = torch::empty_like(dy);
  ub::launch_softmax_dropout_bwd(dy.data_ptr(), dx.data_ptr(), logits.data_ptr(), dy.size(0) * dy.size(1),
                                 (int)dy.size(2), (float)p, (uint64_t)seed, (uint64_t)offset,
                                 dtype_tag(dy.scalar_type()), cur_stream(), lse.data_ptr<float>(), opt_ptr(addend));
  check_launch("softmax_dropout_logits_bwd");
  return dx;
}

Tensor softmax_dropout_bwd(Tensor dy, const Tensor& probs, double p, int64_t seed, int64_t offset) {
  check_operand(dy, "grad_output", dy.device(), kFloating, any_shape(3));
  check_operand(probs, "softmax_results", dy.device(), {dy.scalar_type()}, dy.sizes());
  const c10::cuda::CUDAGuard guard(dy.device());
  // out of place: autograd may hand the same grad tensor to several consumers
  Tensor dx = torch::empty_like(dy);
  ub::launch_softmax_dropout_bwd(dy.data_ptr(), dx.data_ptr(), probs.data_ptr(), dy.size(0) * dy.size(1),
                                 (int)dy.size(2), (float)p, (uint64_t)seed, (uint64_t)offset,
                                 dtype_tag(dy.scalar_type()), cur_stream());
  check_launch("softmax_dropout_bwd");
  return dx;
}

// ---------------------------------------------------------------------------------------------------
// fused element-wise
// ---------------------------------------------------------------------------------------------------
// The bias + GELU kernels read x, dy and the bias as 16-byte vectors of 8 elements from the first element on.
static int check_bias_gelu_operands(const Tensor& x, const OptTensor& bias) {
  check_operand(x, "x", x.device(), k16Bit, {}, kVec);
  TORCH_CHECK(x.dim() >= 1 && x.size(-1) > 0 && x.size(-1) % 8 == 0, "bias_gelu needs a positive multiple of 8 columns");
  const int cols = (int)x.size(-1);
  check_operand(bias, "bias", x.device(), {x.scalar_type()}, {cols}, kVec | kNumel);
  return cols;
}

Tensor bias_gelu_fwd(const Tensor& x, const OptTensor& bias) {
  const int cols = check_bias_gelu_operands(x, bias);
  const c10::cuda::CUDAGuard guard(x.device());
  Tensor y = torch::empty_like(x);
  ub::launch_bias_gelu_fwd(x.data_ptr(), opt_ptr(bias), y.data_ptr(), x.numel() / cols, cols,
                           dtype_tag(x.scalar_type()), cur_stream());
  check_launch("bias_gelu_fwd");
  return y;
}

// returns (dx, dbias); dbias (column sums of dx, produced by the same pass) only when a bias was given
std::tuple<Tensor, OptTensor> bias_gelu_bwd(const Tensor& dy, const Tensor& x, const OptTensor& bias,
                                            const OptTensor& dbias_sink) {
  const int cols = check_bias_gelu_operands(x, bias);
  TORCH_CHECK(dy.sizes() == x.sizes(), "bias_gelu_bwd: dy must match x");
  check_operand(dy, "dy", x.device(), {x.scalar_type()}, {}, kVec);
  const bool has_bias = has(bias);
  if (has_bias) check_sink(dbias_sink, "dbias_sink", *bias);
  const c10::cuda::CUDAGuard guard(x.device());
  const long long rows = x.numel() / cols;
  Tensor dx = torch::empty_like(x);
  OptTensor dbias;
  Tensor part;
  int acc = 0;
  if (has_bias) {
    dbias = grad_out(dbias_sink, *bias, 0, acc);
    part = torch::empty({ub::bias_gelu_parts(rows, cols), cols}, x.options().dtype(at::kFloat));
  }
  ub::launch_bias_gelu_bwd(dy.data_ptr(), x.data_ptr(), opt_ptr(bias), dx.data_ptr(),
                           has_bias ? dbias->data_ptr() : nullptr, has_bias ? part.data_ptr<float>() : nullptr, rows,
                           cols, dtype_tag(x.scalar_type()), cur_stream(), acc);
  check_launch("bias_gelu_bwd");
  return {dx, dbias};
}

// column sums over all leading dims: x [..., cols] -> [cols] (bias gradient of a Linear layer)
Tensor column_sum(const Tensor& x, const OptTensor& sink) {
  check_operand(x, "x", x.device(), k16Bit, {}, kVec);
  TORCH_CHECK(x.dim() >= 1 && x.size(-1) > 0 && x.size(-1) % 8 == 0,
              "column_sum needs a positive multiple of 8 columns");
  const int cols = (int)x.size(-1);
  const long long rows = x.numel() / cols;
  TORCH_CHECK(rows < (1ll << 31), "too many rows");
  check_operand(sink, "sink", x.device(), {x.scalar_type()}, {cols}, kContig | kNumel);
  const c10::cuda::CUDAGuard guard(x.device());
  Tensor out = has(sink) ? *sink : torch::empty({cols}, x.options());
  Tensor part = torch::empty({ub::bias_gelu_parts(rows, cols), cols}, x.options().dtype(at::kFloat));
  ub::launch_column_sum(x.data_ptr(), out.data_ptr(), part.data_ptr<float>(), rows, cols, dtype_tag(x.scalar_type()),
                        cur_stream(), has(sink) ? 1 : 0);
  check_launch("column_sum");
  return out;
}

// grad[tokens[r], :] (+)= dy[r, :]  (csrc/fused/embedding.cu); scratch fp32 [V, D] and touched uint8 [V] are persistent,
// zero between calls.  `grad` is either the parameter's arena view (accumulate) or a zero-filled tensor.  dy and grad
// are read as 16-byte vectors, scratch with float4 loads and red.global.add.v4.f32, so all three are kVec.
void embedding_bwd(const Tensor& dy, const Tensor& tokens, int64_t padding_idx, Tensor scratch, Tensor touched, Tensor grad,
                   bool accumulate) {
  check_operand(dy, "dy", dy.device(), k16Bit, {}, kVec);
  check_operand(grad, "grad", dy.device(), {dy.scalar_type()}, any_shape(2), kVec);
  const int cols = (int)grad.size(1);
  const long long vocab = grad.size(0);
  TORCH_CHECK(cols > 0 && cols % 8 == 0 && dy.dim() >= 1 && dy.size(-1) == cols, "embedding_bwd: shape mismatch");
  check_operand(tokens, "tokens", dy.device(), {at::kLong}, {dy.numel() / cols}, kContig | kNumel);
  check_operand(scratch, "scratch", dy.device(), {at::kFloat}, {vocab * cols}, kVec | kNumel);
  check_operand(touched, "touched", dy.device(), {at::kByte}, {vocab}, kContig | kNumel);
  const c10::cuda::CUDAGuard guard(dy.device());
  const int tag = dtype_tag(dy.scalar_type());
  if (at::globalContext().deterministicAlgorithms()) {
    // fixed summation order: each vocabulary row sums its rows in ascending original order (scratch / touched unused)
    const auto sorted = at::sort(tokens.reshape({-1}), /*stable=*/true, /*dim=*/0, /*descending=*/false);
    const Tensor& ids = std::get<0>(sorted);
    const Tensor& perm = std::get<1>(sorted);
    ub::launch_embedding_bwd_sorted(dy.data_ptr(), reinterpret_cast<const long long*>(ids.data_ptr<int64_t>()),
                                    reinterpret_cast<const long long*>(perm.data_ptr<int64_t>()), grad.data_ptr(),
                                    tokens.numel(), cols, vocab, padding_idx, accumulate ? 1 : 0, tag, cur_stream());
    check_launch("embedding_bwd");
    return;
  }
  ub::launch_embedding_bwd(dy.data_ptr(), reinterpret_cast<const long long*>(tokens.data_ptr<int64_t>()),
                           scratch.data_ptr<float>(), touched.data_ptr<uint8_t>(), grad.data_ptr(), tokens.numel(),
                           cols, vocab, padding_idx, accumulate ? 1 : 0, tag, cur_stream());
  check_launch("embedding_bwd");
}

std::tuple<Tensor, Tensor, Tensor, Tensor, int64_t, int64_t> bias_dropout_add_ln_fwd(
    const Tensor& x, const OptTensor& bias, const Tensor& residual, const Tensor& gamma, const Tensor& beta, double p,
    double eps) {
  check_norm_width(x, "x", k16Bit);
  const int rows = (int)x.size(0), cols = (int)x.size(1);
  check_operand(residual, "residual", x.device(), {x.scalar_type()}, x.sizes(), kVec);
  check_operand(gamma, "gamma", x.device(), {x.scalar_type()}, {cols}, kVec | kNumel);
  check_operand(beta, "beta", x.device(), {x.scalar_type()}, {cols}, kVec | kNumel);
  check_operand(bias, "bias", x.device(), {x.scalar_type()}, {cols}, kVec | kNumel);
  const c10::cuda::CUDAGuard guard(x.device());
  Tensor y = torch::empty_like(x), summed = torch::empty_like(x);
  Tensor mean = torch::empty({rows}, x.options().dtype(at::kFloat));
  Tensor rstd = torch::empty({rows}, x.options().dtype(at::kFloat));
  uint64_t seed = 0, offset = 0;
  if (p > 0.0) std::tie(seed, offset) = philox_reserve(4);
  ub::launch_bias_dropout_add_ln_fwd(x.data_ptr(), opt_ptr(bias), residual.data_ptr(), gamma.data_ptr(),
                                     beta.data_ptr(), y.data_ptr(), summed.data_ptr(), mean.data_ptr<float>(),
                                     rstd.data_ptr<float>(), rows, cols, (float)p, (float)eps, seed, offset,
                                     dtype_tag(x.scalar_type()), cur_stream());
  check_launch("bias_dropout_add_ln_fwd");
  return {y, mean, rstd, summed, (int64_t)seed, (int64_t)offset};
}

// returns (dsum, dx, dgamma, dbeta, dbias); dbias (column sums of dx) exactly when `need_dbias`
std::tuple<Tensor, Tensor, Tensor, Tensor, OptTensor> bias_dropout_add_ln_bwd(const Tensor& dy, const Tensor& summed,
                                                                              const Tensor& mean, const Tensor& rstd,
                                                                              const Tensor& gamma, double p,
                                                                              int64_t seed, int64_t offset,
                                                                              bool need_dbias,
                                                                              const OptTensor& dgamma_sink,
                                                                              const OptTensor& dbeta_sink,
                                                                              const OptTensor& dbias_sink) {
  check_norm_width(summed, "summed", k16Bit);
  const int rows = (int)summed.size(0), cols = (int)summed.size(1), tag = dtype_tag(summed.scalar_type());
  check_operand(dy, "dy", summed.device(), {summed.scalar_type()}, summed.sizes(), kVec);
  check_operand(mean, "mean", summed.device(), {at::kFloat}, {rows});
  check_operand(rstd, "rstd", summed.device(), {at::kFloat}, {rows});
  check_operand(gamma, "gamma", summed.device(), {summed.scalar_type()}, {cols}, kVec | kNumel);
  check_sink(dgamma_sink, "dgamma_sink", gamma);
  check_sink(dbeta_sink, "dbeta_sink", gamma);
  check_sink(dbias_sink, "dbias_sink", gamma);
  const c10::cuda::CUDAGuard guard(summed.device());
  Tensor dsum = torch::empty_like(summed);
  Tensor dx = p > 0.0 ? torch::empty_like(summed) : dsum;
  int acc = 0;
  Tensor dgamma = grad_out(dgamma_sink, gamma, 0, acc), dbeta = grad_out(dbeta_sink, gamma, 1, acc);
  Tensor part = torch::empty({3, ub::norm_bwd_parts(rows, cols, tag), cols}, summed.options().dtype(at::kFloat));
  OptTensor dbias;
  if (need_dbias) dbias = grad_out(dbias_sink, gamma, 2, acc);
  ub::launch_bias_dropout_add_ln_bwd(dy.data_ptr(), summed.data_ptr(), mean.data_ptr<float>(),
                                     rstd.data_ptr<float>(), gamma.data_ptr(), dsum.data_ptr(), dx.data_ptr(),
                                     dgamma.data_ptr(), dbeta.data_ptr(), has(dbias) ? dbias->data_ptr() : nullptr,
                                     part.data_ptr<float>(), rows, cols, (float)p, (uint64_t)seed, (uint64_t)offset,
                                     tag, cur_stream(), acc);
  check_launch("bias_dropout_add_ln_bwd");
  return {dsum, dx, dgamma, dbeta, dbias};
}

// `logits` is [rows, stride] contiguous of which the first `valid_cols` columns are the vocabulary (the
// rest is GEMM-alignment padding); valid_cols <= 0 means all columns.  Returns the vocabulary width.
static int check_xent_operands(const Tensor& logits, const Tensor& target, int64_t valid_cols) {
  check_operand(logits, "logits", logits.device(), kFloating, any_shape(2));
  check_operand(target, "target", logits.device(), {at::kLong}, {logits.size(0)});
  TORCH_CHECK(valid_cols <= logits.size(1), "valid_cols must not exceed the row length of logits");
  return valid_cols > 0 ? (int)valid_cols : (int)logits.size(1);
}

std::tuple<Tensor, Tensor> softmax_xent_fwd(const Tensor& logits, const Tensor& target, int64_t ignore_index,
                                            int64_t valid_cols) {
  const int cols = check_xent_operands(logits, target, valid_cols);
  const c10::cuda::CUDAGuard guard(logits.device());
  const int rows = (int)logits.size(0), stride = (int)logits.size(1);
  Tensor loss = torch::empty({rows}, logits.options().dtype(at::kFloat));
  Tensor lse = torch::empty({rows}, logits.options().dtype(at::kFloat));
  ub::launch_softmax_xent_fwd(logits.data_ptr(), (const long long*)target.data_ptr<int64_t>(), loss.data_ptr<float>(),
                              lse.data_ptr<float>(), rows, cols, stride, ignore_index, dtype_tag(logits.scalar_type()),
                              cur_stream());
  check_launch("softmax_xent_fwd");
  return {loss, lse};
}

Tensor softmax_xent_bwd(const Tensor& logits, const Tensor& target, const Tensor& lse, const Tensor& dloss,
                        int64_t ignore_index, int64_t valid_cols) {
  const int cols = check_xent_operands(logits, target, valid_cols);
  check_operand(lse, "lse", logits.device(), {at::kFloat}, {logits.size(0)});
  check_operand(dloss, "dloss", logits.device(), {at::kFloat}, {1}, kNumel);
  const c10::cuda::CUDAGuard guard(logits.device());
  const int rows = (int)logits.size(0), stride = (int)logits.size(1);
  Tensor dlogits = torch::empty_like(logits);
  ub::launch_softmax_xent_bwd(logits.data_ptr(), (const long long*)target.data_ptr<int64_t>(), lse.data_ptr<float>(),
                              dloss.data_ptr<float>(), dlogits.data_ptr(), rows, cols, stride, ignore_index,
                              dtype_tag(logits.scalar_type()), cur_stream());
  check_launch("softmax_xent_bwd");
  return dlogits;
}

// ---------------------------------------------------------------------------------------------------
// head split / merge
// ---------------------------------------------------------------------------------------------------
// x: [B, L, T*H*D] contiguous -> T tensors [B, H, L, D] (slices of one allocation); slice 0 scaled by scale0
std::vector<Tensor> split_heads(const Tensor& x, int64_t T, int64_t H, double scale0) {
  check_operand(x, "input", x.device(), kFloating, any_shape(3), kVec);
  TORCH_CHECK(T >= 1 && T <= 4 && H >= 1 && x.size(2) % (T * H) == 0, "expected [B, L, T*H*D]");
  const int64_t B = x.size(0), L = x.size(1), D = x.size(2) / (T * H);
  TORCH_CHECK((D * x.element_size()) % 16 == 0, "head_dim must span whole 16-byte vectors");
  const c10::cuda::CUDAGuard guard(x.device());
  Tensor packed = torch::empty({T, B, H, L, D}, x.options());
  std::vector<Tensor> out;
  void* ptrs[4] = {nullptr, nullptr, nullptr, nullptr};
  for (int64_t t = 0; t < T; ++t) {
    out.push_back(packed.select(0, t));
    ptrs[t] = out.back().data_ptr();
  }
  ub::launch_head_permute(x.data_ptr(), ptrs, (int)B, (int)L, (int)T, (int)H, (int)D, (float)scale0, true,
                          dtype_tag(x.scalar_type()), cur_stream());
  check_launch("split_heads");
  return out;
}

// heads: T optional tensors [B, H, L, D] (undefined = zeros) -> [B, L, T*H*D]; slice 0 scaled by scale0
Tensor merge_heads(const std::vector<OptTensor>& heads, double scale0) {
  const int64_t T = (int64_t)heads.size();
  TORCH_CHECK(T >= 1 && T <= 4, "merge_heads takes 1 to 4 tensors");
  const Tensor* ref = nullptr;
  for (const auto& h : heads)
    if (has(h)) ref = &*h;
  TORCH_CHECK(ref != nullptr, "merge_heads needs at least one defined tensor");
  check_operand(*ref, "heads", ref->device(), kFloating, any_shape(4), kVec);
  const int64_t B = ref->size(0), H = ref->size(1), L = ref->size(2), D = ref->size(3);
  TORCH_CHECK((D * ref->element_size()) % 16 == 0, "head_dim must span whole 16-byte vectors");
  void* ptrs[4] = {nullptr, nullptr, nullptr, nullptr};
  for (int64_t t = 0; t < T; ++t) {
    check_operand(heads[t], "heads", ref->device(), {ref->scalar_type()}, ref->sizes(), kVec);
    if (has(heads[t])) ptrs[t] = heads[t]->data_ptr();
  }
  const c10::cuda::CUDAGuard guard(ref->device());
  Tensor out = torch::empty({B, L, T * H * D}, ref->options());
  ub::launch_head_permute(out.data_ptr(), ptrs, (int)B, (int)L, (int)T, (int)H, (int)D, (float)scale0, false,
                          dtype_tag(ref->scalar_type()), cur_stream());
  check_launch("merge_heads");
  return out;
}

// ---------------------------------------------------------------------------------------------------
// rotary position embeddings
// ---------------------------------------------------------------------------------------------------
constexpr int64_t kRotaryMaxDim = 512;   // the cos / sin tile of 8 tokens stays within 16 KB of shared memory

pybind11::dict rotary_plan(int64_t B, int64_t L, int64_t N, int64_t D, int64_t rd, at::ScalarType dtype, bool aligned) {
  TORCH_CHECK(B >= 1 && L >= 1 && N >= 1 && rd >= 2 && rd % 2 == 0 && rd <= D && rd <= kRotaryMaxDim &&
                  (dtype == at::kHalf || dtype == at::kBFloat16),
              "rotary_plan needs positive sizes, an even 2 <= rotary_dim <= min(head_dim, 512) and fp16 / bf16");
  const ub::RotaryPlan p = ub::rotary_plan((int)B, (int)L, (int)N, (int)D, (int)rd, dtype_tag(dtype), aligned);
  pybind11::dict d = sweep_dict(p.sweep);
  d["vec"] = p.vec;
  d["tile_tokens"] = p.tile_tokens;
  d["smem"] = p.smem;
  return d;
}

// x: [B, L, N, D] with a contiguous last dim and head stride D -> a new contiguous [B, L, N, D], heads 0 ..
// rotated_heads-1 rotated on their first 2 * inv_freq.numel() columns (the inverse rotation when `inverse`)
Tensor rotary_embedding(const Tensor& x, const Tensor& inv_freq, int64_t rotated_heads, const OptTensor& position_offsets,
                        bool inverse) {
  check_operand(x, "x", x.device(), k16Bit, any_shape(4), 0);
  const int64_t B = x.size(0), L = x.size(1), N = x.size(2), D = x.size(3);
  TORCH_CHECK(x.stride(3) == 1 && (N == 1 || x.stride(2) == D), "x must have a contiguous last dim and head stride D");
  check_operand(inv_freq, "inv_freq", x.device(), {at::kFloat}, any_shape(1));
  const int64_t rd = 2 * inv_freq.size(0);
  TORCH_CHECK(rd >= 2 && rd <= D && rd <= kRotaryMaxDim, "inv_freq must have 1 .. min(head_dim, 512) / 2 entries, not ",
              inv_freq.size(0));
  TORCH_CHECK(rotated_heads >= 0 && rotated_heads <= N, "rotated_heads must be in [0, ", N, "], not ", rotated_heads);
  check_operand(position_offsets, "position_offsets", x.device(), {at::kInt}, {B});
  const c10::cuda::CUDAGuard guard(x.device());
  Tensor out = torch::empty({B, L, N, D}, x.options());
  if (out.numel() == 0) return out;
  const bool aligned = aligned16(x.data_ptr()) && x.stride(0) % 8 == 0 && x.stride(1) % 8 == 0;
  ub::launch_rotary(x.data_ptr(), out.data_ptr(), inv_freq.data_ptr<float>(),
                    has(position_offsets) ? position_offsets->data_ptr<int>() : nullptr, x.stride(0), x.stride(1),
                    (int)B, (int)L, (int)N, (int)D, (int)rd, (int)rotated_heads, aligned, inverse,
                    dtype_tag(x.scalar_type()), cur_stream());
  check_launch("rotary_embedding");
  return out;
}

// ---------------------------------------------------------------------------------------------------
// pair representation relayout
// ---------------------------------------------------------------------------------------------------
// Every pair operand is a 4-D fp16 / bf16 tensor read as 16-byte vectors; key_padding_mask is bool / uint8 [B, Lk],
// read 8 flags at a time with 8-byte loads, so it is kVec too.
static const unsigned char* key_pad_ptr(const OptTensor& key_pad, const Tensor& z, int64_t Lk) {
  check_operand(key_pad, "key_padding_mask", z.device(), {at::kBool, at::kByte}, {z.size(0), Lk}, kVec);
  return static_cast<const unsigned char*>(opt_ptr(key_pad));
}

// to_pair: [B, H, Lq, Lk] -> [B, Lq, Lk, H];  otherwise the inverse
Tensor pair_transpose(const Tensor& x, bool to_pair) {
  check_operand(x, "input", x.device(), k16Bit, any_shape(4), kVec);
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
  check_operand(z, "logits", z.device(), k16Bit, any_shape(4), kVec);
  check_operand(z0, "input bias", z.device(), {z.scalar_type()}, z.sizes(), kVec);
  const int64_t B = z.size(0), H = z.size(1), Lq = z.size(2), Lk = z.size(3);
  TORCH_CHECK(H % 8 == 0 && Lk % 8 == 0, "pair_tail needs H % 8 == 0 and Lk % 8 == 0");
  const unsigned char* pad = key_pad_ptr(key_pad, z, Lk);
  const c10::cuda::CUDAGuard guard(z.device());
  Tensor pair = torch::empty({B, Lq, Lk, H}, z.options()), delta = torch::empty({B, Lq, Lk, H}, z.options());
  ub::launch_pair_tail_fwd(z.data_ptr(), z0.data_ptr(), pad, pair.data_ptr(), delta.data_ptr(), (int)B, (int)H, (int)Lq,
                           (int)Lk, dtype_tag(z.scalar_type()), cur_stream());
  check_launch("pair_tail_fwd");
  return {pair, delta};
}

std::tuple<Tensor, Tensor> pair_tail_bwd(const OptTensor& d_pair, const OptTensor& d_delta, const Tensor& z,
                                         const OptTensor& key_pad) {
  check_operand(z, "logits", z.device(), k16Bit, any_shape(4), kVec);
  const int64_t B = z.size(0), H = z.size(1), Lq = z.size(2), Lk = z.size(3);
  check_operand(d_pair, "d_pair", z.device(), {z.scalar_type()}, {B, Lq, Lk, H}, kVec);
  check_operand(d_delta, "d_delta", z.device(), {z.scalar_type()}, {B, Lq, Lk, H}, kVec);
  const unsigned char* pad = key_pad_ptr(key_pad, z, Lk);
  const c10::cuda::CUDAGuard guard(z.device());
  Tensor dz = torch::empty_like(z), dz0 = torch::empty_like(z);
  ub::launch_pair_tail_bwd(opt_ptr(d_pair), opt_ptr(d_delta), z.data_ptr(), pad, dz.data_ptr(), dz0.data_ptr(), (int)B,
                           (int)H, (int)Lq, (int)Lk, dtype_tag(z.scalar_type()), cur_stream());
  check_launch("pair_tail_bwd");
  return {dz, dz0};
}

// ---------------------------------------------------------------------------------------------------
// Gaussian basis (Uni-Mol)
// ---------------------------------------------------------------------------------------------------
// d [...] distances with an edge type each; mul_w / bias_w one entry per edge type; means / stds the K Gaussians,
// K = 8 * 2^i <= 256 (the kernels' vector widths).  Returns K.
static int check_gbf_operands(const Tensor& d, const Tensor& edge, const Tensor& mul_w, const Tensor& bias_w,
                              const Tensor& means, const Tensor& stds) {
  check_operand(d, "d", d.device(), k16Bit);
  check_operand(edge, "edge", d.device(), {at::kLong}, {d.numel()}, kContig | kNumel);
  check_operand(mul_w, "mul_w", d.device(), {d.scalar_type()});
  check_operand(bias_w, "bias_w", d.device(), {d.scalar_type()}, {mul_w.numel()}, kContig | kNumel);
  check_operand(means, "means", d.device(), {d.scalar_type()});
  const int K = (int)means.numel();
  check_operand(stds, "stds", d.device(), {d.scalar_type()}, {K}, kContig | kNumel);
  TORCH_CHECK(K >= 8 && K % 8 == 0 && K / 8 <= 32 && ((K / 8) & (K / 8 - 1)) == 0, "K must be 8 * 2^i <= 256");
  return K;
}

Tensor gbf_fwd(const Tensor& d, const Tensor& edge, const Tensor& mul_w, const Tensor& bias_w, const Tensor& means,
               const Tensor& stds) {
  const int K = check_gbf_operands(d, edge, mul_w, bias_w, means, stds);
  const c10::cuda::CUDAGuard guard(d.device());
  auto sizes = d.sizes().vec();
  sizes.push_back(K);
  Tensor y = torch::empty(sizes, d.options());
  ub::launch_gbf_fwd(d.data_ptr(), (const long long*)edge.data_ptr<int64_t>(), mul_w.data_ptr(), bias_w.data_ptr(),
                     means.data_ptr(), stds.data_ptr(), y.data_ptr(), d.numel(), K, dtype_tag(d.scalar_type()),
                     cur_stream());
  check_launch("gbf_fwd");
  return y;
}

// returns (d mul [E], d bias [E], d means [K], d stds_abs [K]) in fp32
std::tuple<Tensor, Tensor, Tensor, Tensor> gbf_bwd(const Tensor& dy, const Tensor& d, const Tensor& edge,
                                                   const Tensor& mul_w, const Tensor& bias_w, const Tensor& means,
                                                   const Tensor& stds) {
  const int K = check_gbf_operands(d, edge, mul_w, bias_w, means, stds), E = (int)mul_w.numel();
  check_operand(dy, "dy", d.device(), {d.scalar_type()}, {d.numel() * K}, kContig | kNumel);
  TORCH_CHECK(E <= 8192, "edge-type table too large for the shared-memory histogram");
  const c10::cuda::CUDAGuard guard(d.device());
  const int parts = ub::gbf_parts(d.numel(), K), tag = dtype_tag(d.scalar_type());
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
                           K, E, tag, cur_stream());
  } else {
    ub::launch_gbf_bwd(dy.data_ptr(), d.data_ptr(), (const long long*)edge.data_ptr<int64_t>(), mul_w.data_ptr(),
                       bias_w.data_ptr(), means.data_ptr(), stds.data_ptr(), part.data_ptr<float>(),
                       hist.data_ptr<float>(), d.numel(), K, E, tag, cur_stream());
  }
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
  m.def("bias_gelu_plan", &bias_gelu_plan, pybind11::arg("rows"), pybind11::arg("cols"), pybind11::arg("kind"));
  m.def("gbf_plan", &gbf_plan, pybind11::arg("n"), pybind11::arg("K"), pybind11::arg("E"));
  m.def("head_permute_plan", &head_permute_plan, pybind11::arg("B"), pybind11::arg("L"), pybind11::arg("T"),
        pybind11::arg("H"), pybind11::arg("D"), pybind11::arg("dtype"));
  m.def("pair_plan", &pair_plan, pybind11::arg("B"), pybind11::arg("H"), pybind11::arg("M"));
  m.def("embedding_plan", &embedding_plan, pybind11::arg("rows"), pybind11::arg("vocab"));
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
  // its own submodule, _C.rotary, as _C.kvcache; tests/test_gpu_rotary.py runs the operand-rejection table of
  // tests/test_gpu_bindings.py over it
  auto rot = m.def_submodule("rotary", "rotary position embeddings");
  rot.def("rotary_embedding", &rotary_embedding, pybind11::arg("x"), pybind11::arg("inv_freq"),
          pybind11::arg("rotated_heads"), pybind11::arg("position_offsets"), pybind11::arg("inverse") = false);
  rot.def("rotary_plan", &rotary_plan, pybind11::arg("B"), pybind11::arg("L"), pybind11::arg("N"), pybind11::arg("D"),
          pybind11::arg("rd"), pybind11::arg("dtype"), pybind11::arg("aligned") = true);
  register_fmha(m);
  register_comm(m);
  register_symm_mem(m);
}
