// PyTorch bindings of the fused attention kernels.
#include <ATen/cuda/CUDAContext.h>
#include <ATen/cuda/CUDAGeneratorImpl.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <optional>

#include "fmha_api.h"
#include "tma_map.h"

namespace {
using torch::Tensor;
using OptTensor = std::optional<Tensor>;

std::pair<uint64_t, uint64_t> reserve_philox(uint64_t increment) {
  auto gen = at::get_generator_or_default<at::CUDAGeneratorImpl>(std::nullopt,
                                                                 at::cuda::detail::getDefaultCUDAGenerator());
  std::lock_guard<std::mutex> lock(gen->mutex_);
  at::PhiloxCudaState st = gen->philox_cuda_state(increment);
  TORCH_CHECK(!st.captured_, "fmha: RNG under CUDA graph capture is not supported yet");
  return {st.seed_.val, st.offset_.val};
}

void fill_common(ub::FmhaFwdParams& p, const Tensor& q, const Tensor& k, const Tensor& v, const OptTensor& bias,
                 const OptTensor& kpm, double p_drop, double scale, bool forward) {
  TORCH_CHECK(q.is_cuda() && k.is_cuda() && v.is_cuda());
  TORCH_CHECK(q.dim() == 4 && k.dim() == 4 && v.dim() == 4, "q/k/v must be [B, L, H, D]");
  const int64_t D = q.size(3);
  TORCH_CHECK(ub::fmha_head_dim_supported(D) && k.size(3) == D && v.size(3) == D,
              "head_dim must be the same for q/k/v and a multiple of 8 from 8 to 128 (8, 16, ..., 128)");
  TORCH_CHECK(q.stride(3) == 1 && k.stride(3) == 1 && v.stride(3) == 1, "last dim must be contiguous");
  TORCH_CHECK(q.scalar_type() == at::kHalf || q.scalar_type() == at::kBFloat16);
  TORCH_CHECK(k.scalar_type() == q.scalar_type() && v.scalar_type() == q.scalar_type());
  TORCH_CHECK(k.size(0) == q.size(0) && v.size(0) == q.size(0) && k.size(2) == q.size(2) && v.size(2) == q.size(2));
  TORCH_CHECK(k.size(1) == v.size(1));
  TORCH_CHECK(q.size(1) % 8 == 0 && k.size(1) % 8 == 0, "sequence lengths must be multiples of 8");
  for (const Tensor* t : {&q, &k, &v}) {
    TORCH_CHECK(t->stride(0) % 8 == 0 && t->stride(1) % 8 == 0 && t->stride(2) % 8 == 0 &&
                    (reinterpret_cast<uintptr_t>(t->data_ptr()) & 15) == 0,
                "q/k/v must be 16-byte aligned with strides that are multiples of 8 elements");
  }
  p.q = q.data_ptr();
  p.k = k.data_ptr();
  p.v = v.data_ptr();
  p.q_sb = q.stride(0); p.q_sl = q.stride(1); p.q_sh = q.stride(2);
  p.k_sb = k.stride(0); p.k_sl = k.stride(1); p.k_sh = k.stride(2);
  p.v_sb = v.stride(0); p.v_sl = v.stride(1); p.v_sh = v.stride(2);
  p.B = (int)q.size(0);
  p.Lq = (int)q.size(1);
  p.H = (int)q.size(2);
  p.Lk = (int)k.size(1);
  p.D = (int)D;
  p.is_bf16 = q.scalar_type() == at::kBFloat16 ? 1 : 0;
  p.bias = nullptr;
  p.bias_batch = 1;
  p.bias_is_f32 = 0;
  if (bias.has_value() && bias->defined()) {
    TORCH_CHECK(bias->is_cuda() && bias->is_contiguous() && bias->dim() == 4);
    TORCH_CHECK((bias->size(0) == 1 || bias->size(0) == p.B) && bias->size(1) == p.H && bias->size(2) == p.Lq &&
                bias->size(3) == p.Lk, "bias must be [1|B, H, Lq, Lk]");
    TORCH_CHECK(bias->scalar_type() == q.scalar_type(), "bias must have the dtype of q");
    TORCH_CHECK((reinterpret_cast<uintptr_t>(bias->data_ptr()) & 15) == 0, "bias must be 16-byte aligned");
    p.bias = bias->data_ptr();
    p.bias_batch = (int)bias->size(0);
  }
  p.drop_bits = nullptr;
  p.kpm = nullptr;
  if (kpm.has_value() && kpm->defined()) {
    TORCH_CHECK(kpm->is_cuda() && kpm->is_contiguous() && kpm->scalar_type() == at::kBool && kpm->dim() == 2 &&
                kpm->size(0) == p.B && kpm->size(1) == p.Lk, "key_padding_mask must be bool [B, Lk]");
    p.kpm = reinterpret_cast<const uint8_t*>(kpm->data_ptr());
  }
  p.p_drop = (float)p_drop;
  p.scale = (float)scale;
  // The driver API behind cuTensorMapEncodeTiled needs a current context in THIS thread; autograd worker
  // threads only have the c10 device guard's notion of the device, so bind the primary context explicitly.
  cudaSetDevice(q.get_device());
  // TMA descriptors: heads must be contiguous (stride D) so that (head, 16-byte chunk) is one dimension
  TORCH_CHECK(q.stride(2) == D && k.stride(2) == D && v.stride(2) == D, "q/k/v head stride must be head_dim");
  const bool bf16 = p.is_bf16 != 0;
  const int q_box_rows = forward ? ub::kFwdQBoxRows : ub::kBwdBoxRows;
  const int kv_box_rows = forward ? ub::fmha_fwd_kv_box_rows(p.D) : ub::kBwdBoxRows;
  bool ok = ub::make_head_tile_map_sw128(&p.sw_q, p.q, bf16, p.B, p.Lq, p.H, p.D, p.q_sb, p.q_sl, p.q_sh, q_box_rows);
  ok = ok && ub::make_head_tile_map_sw128(&p.sw_k, p.k, bf16, p.B, p.Lk, p.H, p.D, p.k_sb, p.k_sl, p.k_sh, kv_box_rows);
  ok = ok && ub::make_head_tile_map_sw128(&p.sw_v, p.v, bf16, p.B, p.Lk, p.H, p.D, p.v_sb, p.v_sl, p.v_sh, kv_box_rows);
  if (p.bias != nullptr) ok = ok && ub::make_bias_tile_map_sw128(&p.sw_bias, p.bias, bf16, p.bias_batch * p.H, p.Lq, p.Lk);
  TORCH_CHECK(ok, "cuTensorMapEncodeTiled failed for the attention operands");
}

// (out, lse, keep bits, logits); the logits z = scale * q k^T + bias + key mask only when `logits` is set
std::tuple<Tensor, Tensor, OptTensor, OptTensor> fwd_impl(const Tensor& q, const Tensor& k, const Tensor& v,
                                                          const OptTensor& bias, const OptTensor& kpm, double p_drop,
                                                          double scale, bool logits, bool causal) {
  TORCH_CHECK(!(logits && causal), "fmha: causal attention does not return logits");
  const c10::cuda::CUDAGuard guard(q.device());
  ub::FmhaFwdParams p{};
  fill_common(p, q, k, v, bias, kpm, p_drop, scale, /*forward=*/true);
  p.causal = causal ? 1 : 0;
  Tensor out = torch::empty({p.B, p.Lq, p.H, p.D}, q.options());
  Tensor lse = torch::empty({p.B, p.H, p.Lq}, q.options().dtype(at::kFloat));
  p.out = out.data_ptr();
  p.lse = lse.data_ptr<float>();
  OptTensor z;
  p.logits = nullptr;
  if (logits) {
    z = torch::empty({p.B, p.H, p.Lq, p.Lk}, q.options());
    p.logits = z->data_ptr();
    TORCH_CHECK(ub::make_bias_tile_map_sw128(&p.sw_logits, p.logits, p.is_bf16 != 0, p.B * p.H, p.Lq, p.Lk),
                "cuTensorMapEncodeTiled failed for the logits");
  }
  p.seed = p.offset = 0;
  OptTensor bits;
  if (p_drop > 0.0) {
    auto so = reserve_philox(4);
    p.seed = so.first;
    p.offset = so.second;
    // 1 keep-bit per (query, key): 1/16 of the size of a 16-bit score tensor
    bits = torch::empty({p.B, p.H, p.Lq, (p.Lk + 31) / 32}, q.options().dtype(at::kInt));
    p.drop_bits = reinterpret_cast<uint32_t*>(bits->data_ptr());
  }
  ub::launch_fmha_fwd(p, at::cuda::getCurrentCUDAStream().stream());
  cudaError_t err = cudaGetLastError();
  TORCH_CHECK(err == cudaSuccess, "fmha_fwd launch failed: ", cudaGetErrorString(err));
  return {out, lse, bits, z};
}

// causal: key j is visible to query i iff j <= i (fmha_api.h)
std::tuple<Tensor, Tensor, OptTensor> fmha_fwd(const Tensor& q, const Tensor& k, const Tensor& v,
                                                      const OptTensor& bias, const OptTensor& kpm, double p_drop,
                                                      double scale, bool causal) {
  auto r = fwd_impl(q, k, v, bias, kpm, p_drop, scale, /*logits=*/false, causal);
  return {std::get<0>(r), std::get<1>(r), std::get<2>(r)};
}

// also returns the logits z [B, H, Lq, Lk] (dtype of q, -inf at masked keys); z is [B, H, ...] even for a [1, H, ...]
// bias
std::tuple<Tensor, Tensor, OptTensor, Tensor> fmha_fwd_logits(const Tensor& q, const Tensor& k, const Tensor& v,
                                                              const OptTensor& bias, const OptTensor& kpm,
                                                              double p_drop, double scale) {
  auto r = fwd_impl(q, k, v, bias, kpm, p_drop, scale, /*logits=*/true, /*causal=*/false);
  return {std::get<0>(r), std::get<1>(r), std::get<2>(r), *std::get<3>(r)};
}

std::tuple<Tensor, Tensor, Tensor, OptTensor> fmha_bwd(const Tensor& dout, const Tensor& q, const Tensor& k,
                                                       const Tensor& v, const Tensor& out, const Tensor& lse,
                                                       const OptTensor& bias, const OptTensor& kpm, double p_drop,
                                                       double scale, const OptTensor& drop_bits, bool need_dbias,
                                                       bool packed_grad, const OptTensor& dlogits, bool causal) {
  // packed_grad: q/k/v are slices [:, :, i] of one [B, L, 3, H, D] tensor; the gradients are then
  // written straight into one packed [B, L, 3, H, D] tensor (returned three times as views), which
  // spares autograd three zero-filled select-backward tensors and two full-size adds per layer.
  // dlogits: gradient of the logits output of fmha_fwd_logits, [B, H, Lq, Lk]; None means zero.
  // causal: the backward of fmha_fwd(..., causal=True); its keep bits cover only the key tiles that forward walked.
  const bool has_dlogits = dlogits.has_value() && dlogits->defined();
  TORCH_CHECK(!(causal && has_dlogits), "fmha_bwd: causal attention has no logits output, so dlogits must be None");
  const c10::cuda::CUDAGuard guard(q.device());
  ub::FmhaBwdParams p{};
  fill_common(p.f, q, k, v, bias, kpm, p_drop, scale, /*forward=*/false);
  p.f.causal = causal ? 1 : 0;
  const int D = p.f.D;
  TORCH_CHECK(dout.is_contiguous() && out.is_contiguous() && lse.is_contiguous());
  TORCH_CHECK(dout.dim() == 4 && dout.size(0) == p.f.B && dout.size(1) == p.f.Lq && dout.size(2) == p.f.H &&
                  dout.size(3) == D && out.sizes() == dout.sizes(),
              "dout / out must be [B, Lq, H, D]");
  p.f.out = out.data_ptr();
  p.f.lse = lse.data_ptr<float>();
  if (p_drop > 0.0) {
    TORCH_CHECK(drop_bits.has_value() && drop_bits->defined() && drop_bits->is_contiguous(), "dropout bits missing");
    p.f.drop_bits = reinterpret_cast<uint32_t*>(drop_bits->data_ptr());
  }
  p.dout = dout.data_ptr();
  TORCH_CHECK(ub::make_head_tile_map_sw128(&p.sw_do, p.dout, p.f.is_bf16 != 0, p.f.B, p.f.Lq, p.f.H, D,
                                           (long long)p.f.Lq * p.f.H * D, (long long)p.f.H * D, D, ub::kBwdBoxRows),
              "cuTensorMapEncodeTiled failed for dO");
  Tensor delta = torch::empty({p.f.B, p.f.H, p.f.Lq}, q.options().dtype(at::kFloat));
  // zeroed by the launcher; padded to whole 64-row query tiles and to the kernel's padded head width.  Under
  // torch.use_deterministic_algorithms (warn-only included) the int32 turn counters of the ordered dQ reductions,
  // one per (b, h, query tile), follow in the same allocation.
  const bool det = at::globalContext().deterministicAlgorithms();
  const int64_t n_qt = (p.f.Lq + 63) / 64;
  const int64_t acc_floats = (int64_t)p.f.B * p.f.H * n_qt * 64 * ub::fmha_padded_head_dim(D);
  Tensor dq_acc = torch::empty({acc_floats + (det ? (int64_t)p.f.B * p.f.H * n_qt : 0)}, q.options().dtype(at::kFloat));
  p.dq_turn = det ? reinterpret_cast<int*>(dq_acc.data_ptr<float>() + acc_floats) : nullptr;
  Tensor dq, dk, dv;
  if (packed_grad) {
    TORCH_CHECK(p.f.Lq == p.f.Lk, "packed gradients need self-attention shapes");
    Tensor dqkv = torch::empty({p.f.B, p.f.Lq, 3, p.f.H, D}, q.options());
    dq = dqkv.select(2, 0);
    dk = dqkv.select(2, 1);
    dv = dqkv.select(2, 2);
  } else {
    dq = torch::empty({p.f.B, p.f.Lq, p.f.H, D}, q.options());
    dk = torch::empty({p.f.B, p.f.Lk, p.f.H, D}, q.options());
    dv = torch::empty({p.f.B, p.f.Lk, p.f.H, D}, q.options());
  }
  p.dq_sb = dq.stride(0); p.dq_sl = dq.stride(1); p.dq_sh = dq.stride(2);
  p.dk_sb = dk.stride(0); p.dk_sl = dk.stride(1); p.dk_sh = dk.stride(2);
  p.dv_sb = dv.stride(0); p.dv_sl = dv.stride(1); p.dv_sh = dv.stride(2);
  OptTensor dbias;
  Tensor ds_buf;
  p.dbias = nullptr;
  p.ds_buf = nullptr;
  if (need_dbias && p.f.bias != nullptr) {
    ds_buf = torch::empty({p.f.B, p.f.H, p.f.Lq, p.f.Lk}, q.options());
    p.ds_buf = ds_buf.data_ptr();
    dbias = (p.f.bias_batch == p.f.B) ? ds_buf : torch::empty({p.f.bias_batch, p.f.H, p.f.Lq, p.f.Lk}, q.options());
    p.dbias = dbias->data_ptr();
    TORCH_CHECK(ub::make_bias_tile_map_sw128(&p.sw_ds, p.ds_buf, p.f.is_bf16 != 0, p.f.B * p.f.H, p.f.Lq, p.f.Lk),
                "cuTensorMapEncodeTiled failed for the dS scratch tensor");
  }
  p.dlogits = nullptr;
  if (has_dlogits) {
    TORCH_CHECK(dlogits->is_cuda() && dlogits->is_contiguous() && dlogits->dim() == 4 && dlogits->size(0) == p.f.B &&
                    dlogits->size(1) == p.f.H && dlogits->size(2) == p.f.Lq && dlogits->size(3) == p.f.Lk,
                "dlogits must be contiguous [B, H, Lq, Lk]");
    TORCH_CHECK(dlogits->scalar_type() == q.scalar_type(), "dlogits must have the dtype of q");
    TORCH_CHECK((reinterpret_cast<uintptr_t>(dlogits->data_ptr()) & 15) == 0, "dlogits must be 16-byte aligned");
    p.dlogits = dlogits->data_ptr();
    TORCH_CHECK(ub::make_bias_tile_map_sw128(&p.sw_dz, p.dlogits, p.f.is_bf16 != 0, p.f.B * p.f.H, p.f.Lq, p.f.Lk),
                "cuTensorMapEncodeTiled failed for dlogits");
  }
  p.delta = delta.data_ptr<float>();
  p.dq_acc = dq_acc.data_ptr<float>();
  p.dq = dq.data_ptr();
  p.dk = dk.data_ptr();
  p.dv = dv.data_ptr();
  ub::launch_fmha_bwd(p, at::cuda::getCurrentCUDAStream().stream());
  cudaError_t err = cudaGetLastError();
  TORCH_CHECK(err == cudaSuccess, "fmha_bwd launch failed: ", cudaGetErrorString(err));
  return {dq, dk, dv, dbias};
}
}  // namespace

void register_fmha(pybind11::module_& m) {
  namespace py = pybind11;
  m.def("fmha_fwd", &fmha_fwd, py::arg("q"), py::arg("k"), py::arg("v"), py::arg("bias"), py::arg("kpm"),
        py::arg("p_drop"), py::arg("scale"), py::arg("causal") = false);
  m.def("fmha_fwd_logits", &fmha_fwd_logits);
  m.def("fmha_bwd", &fmha_bwd, py::arg("dout"), py::arg("q"), py::arg("k"), py::arg("v"), py::arg("out"),
        py::arg("lse"), py::arg("bias"), py::arg("kpm"), py::arg("p_drop"), py::arg("scale"), py::arg("drop_bits"),
        py::arg("need_dbias"), py::arg("packed_grad"), py::arg("dlogits") = py::none(), py::arg("causal") = false);
  m.def("fmha_det_timeouts", [] { return (int64_t)ub::fmha_det_timeouts_take(); },
        "deterministic-mode dQ turn waits that timed out on the current device since the last call (reset on read)");
}
