// PyTorch bindings of the fused attention kernels.
#include <c10/cuda/CUDAGuard.h>

#include "../bind_util.h"
#include "fmha_api.h"
#include "tma_map.h"

namespace {
using namespace ub_bind;

// q [B, Lq, H, D] and k / v [B, Lk, H_kv, D] with H_kv dividing H (grouped-query attention; heads contiguous, strides
// that are multiples of 8 elements), bias [1|B, H, Lq, Lk] and the bool key_padding_mask [B, Lk]: what the TMA tile
// maps of fill_common need.
void check_common(const Tensor& q, const Tensor& k, const Tensor& v, const OptTensor& bias, const OptTensor& kpm) {
  check_operand(q, "q", q.device(), k16Bit, any_shape(4), kAligned);
  check_operand(k, "k", q.device(), {q.scalar_type()}, any_shape(4), kAligned);
  check_operand(v, "v", q.device(), {q.scalar_type()}, any_shape(4), kAligned);
  const int64_t B = q.size(0), Lq = q.size(1), H = q.size(2), D = q.size(3), Lk = k.size(1), H_kv = v.size(2);
  TORCH_CHECK(ub::fmha_head_dim_supported(D) && k.size(3) == D && v.size(3) == D,
              "head_dim must be the same for q/k/v and a multiple of 8 from 8 to 128 (8, 16, ..., 128)");
  TORCH_CHECK(k.size(0) == B && v.size(0) == B && k.size(2) == H_kv && v.size(1) == Lk,
              "k / v must be [B, Lk, H_kv, D] with the B and D of q");
  kv_group(H, H_kv, "v");
  TORCH_CHECK(Lq % 8 == 0 && Lk % 8 == 0, "sequence lengths must be multiples of 8");
  for (const Tensor* t : {&q, &k, &v}) {
    // TMA descriptors: heads must be contiguous (stride D) so that (head, 16-byte chunk) is one dimension
    TORCH_CHECK(t->stride(3) == 1 && t->stride(2) == D, "q/k/v head stride must be head_dim");
    TORCH_CHECK(t->stride(0) % 8 == 0 && t->stride(1) % 8 == 0, "q/k/v strides must be multiples of 8 elements");
  }
  check_operand(bias, "bias", q.device(), {q.scalar_type()}, {kAnySize, H, Lq, Lk}, kVec);
  TORCH_CHECK(!has(bias) || bias->size(0) == 1 || bias->size(0) == B, "bias must be [1|B, H, Lq, Lk]");
  check_operand(kpm, "key_padding_mask", q.device(), {at::kBool}, {B, Lk});
}

// The parameters and TMA tile maps of operands check_common accepted.
void fill_common(ub::FmhaFwdParams& p, const Tensor& q, const Tensor& k, const Tensor& v, const OptTensor& bias,
                 const OptTensor& kpm, double p_drop, double scale, bool forward) {
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
  p.D = (int)q.size(3);
  p.kv_group = (int)(q.size(2) / v.size(2));
  const int H_kv = (int)v.size(2);
  p.is_bf16 = q.scalar_type() == at::kBFloat16 ? 1 : 0;
  p.bias = has(bias) ? bias->data_ptr() : nullptr;
  p.bias_batch = has(bias) ? (int)bias->size(0) : 1;
  p.bias_is_f32 = 0;
  p.drop_bits = nullptr;
  p.kpm = static_cast<const uint8_t*>(opt_ptr(kpm));
  p.p_drop = (float)p_drop;
  p.scale = (float)scale;
  // The driver API behind cuTensorMapEncodeTiled needs a current context in THIS thread; autograd worker
  // threads only have the c10 device guard's notion of the device, so bind the primary context explicitly.
  cudaSetDevice(q.get_device());
  const bool bf16 = p.is_bf16 != 0;
  const int q_box_rows = forward ? ub::kFwdQBoxRows : ub::kBwdBoxRows;
  const int kv_box_rows = forward ? ub::fmha_fwd_kv_box_rows(p.D) : ub::kBwdBoxRows;
  bool ok = ub::make_head_tile_map_sw128(&p.sw_q, p.q, bf16, p.B, p.Lq, p.H, p.D, p.q_sb, p.q_sl, p.q_sh, q_box_rows);
  // k / v have the batch of q, except the caches of packed chunks (fmha_kvcache_varlen_fwd), whose q is one batch
  const int B_kv = (int)k.size(0);
  ok = ok && ub::make_head_tile_map_sw128(&p.sw_k, p.k, bf16, B_kv, p.Lk, H_kv, p.D, p.k_sb, p.k_sl, p.k_sh, kv_box_rows);
  ok = ok && ub::make_head_tile_map_sw128(&p.sw_v, p.v, bf16, B_kv, p.Lk, H_kv, p.D, p.v_sb, p.v_sl, p.v_sh, kv_box_rows);
  if (p.bias != nullptr) ok = ok && ub::make_bias_tile_map_sw128(&p.sw_bias, p.bias, bf16, p.bias_batch * p.H, p.Lq, p.Lk);
  TORCH_CHECK(ok, "cuTensorMapEncodeTiled failed for the attention operands");
}

// (out, lse, keep bits, logits); the logits z = scale * q k^T + bias + key mask only when `logits` is set
std::tuple<Tensor, Tensor, OptTensor, OptTensor> fwd_impl(const Tensor& q, const Tensor& k, const Tensor& v,
                                                          const OptTensor& bias, const OptTensor& kpm, double p_drop,
                                                          double scale, bool logits, bool causal) {
  TORCH_CHECK(!(logits && causal), "fmha: causal attention does not return logits");
  check_common(q, k, v, bias, kpm);
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
    std::tie(p.seed, p.offset) = philox_reserve(4);
    // 1 keep-bit per (query, key): 1/16 of the size of a 16-bit score tensor
    bits = torch::empty({p.B, p.H, p.Lq, (p.Lk + 31) / 32}, q.options().dtype(at::kInt));
    p.drop_bits = reinterpret_cast<uint32_t*>(bits->data_ptr());
  }
  ub::launch_fmha_fwd(p, cur_stream());
  check_launch("fmha_fwd");
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
  // packed_grad: q/k/v are the head slices [0, H), [H, H + H_kv), [H + H_kv, H + 2 H_kv) of one [B, L, H + 2 H_kv, D]
  // tensor (a contiguous [B, L, 3, H, D] tensor is that layout with H_kv = H); the gradients are then written straight
  // into one packed tensor of that layout (returned three times as views), which spares autograd three zero-filled
  // slice-backward tensors and two full-size adds per layer.  dK / dV are [B, Lk, H_kv, D]: the sum over each group.
  // dlogits: gradient of the logits output of fmha_fwd_logits, [B, H, Lq, Lk]; None means zero.
  // causal: the backward of fmha_fwd(..., causal=True); its keep bits cover only the key tiles that forward walked.
  TORCH_CHECK(!(causal && has(dlogits)), "fmha_bwd: causal attention has no logits output, so dlogits must be None");
  check_common(q, k, v, bias, kpm);
  const int64_t B = q.size(0), Lq = q.size(1), H = q.size(2), Lk = k.size(1), H_kv = k.size(2);
  // dO is read through a TMA tile map, so it is kVec like dlogits
  check_operand(dout, "dout", q.device(), {q.scalar_type()}, q.sizes(), kVec);
  check_operand(out, "out", q.device(), {q.scalar_type()}, q.sizes());
  check_operand(lse, "lse", q.device(), {at::kFloat}, {B, H, Lq});
  TORCH_CHECK(p_drop <= 0.0 || has(drop_bits), "dropout bits missing");
  if (p_drop > 0.0) check_operand(drop_bits, "drop_bits", q.device(), {at::kInt}, {B, H, Lq, (Lk + 31) / 32});
  check_operand(dlogits, "dlogits", q.device(), {q.scalar_type()}, {B, H, Lq, Lk}, kVec);
  TORCH_CHECK(!packed_grad || Lq == Lk, "packed gradients need self-attention shapes");
  const c10::cuda::CUDAGuard guard(q.device());
  ub::FmhaBwdParams p{};
  fill_common(p.f, q, k, v, bias, kpm, p_drop, scale, /*forward=*/false);
  p.f.causal = causal ? 1 : 0;
  const int D = p.f.D;
  p.f.out = out.data_ptr();
  p.f.lse = lse.data_ptr<float>();
  if (p_drop > 0.0) p.f.drop_bits = reinterpret_cast<uint32_t*>(drop_bits->data_ptr());
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
    Tensor dqkv = torch::empty({B, Lq, H + 2 * H_kv, D}, q.options());
    dq = dqkv.narrow(2, 0, H);
    dk = dqkv.narrow(2, H, H_kv);
    dv = dqkv.narrow(2, H + H_kv, H_kv);
  } else {
    dq = torch::empty({B, Lq, H, D}, q.options());
    dk = torch::empty({B, Lk, H_kv, D}, q.options());
    dv = torch::empty({B, Lk, H_kv, D}, q.options());
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
  if (has(dlogits)) {
    p.dlogits = dlogits->data_ptr();
    TORCH_CHECK(ub::make_bias_tile_map_sw128(&p.sw_dz, p.dlogits, p.f.is_bf16 != 0, p.f.B * p.f.H, p.f.Lq, p.f.Lk),
                "cuTensorMapEncodeTiled failed for dlogits");
  }
  p.delta = delta.data_ptr<float>();
  p.dq_acc = dq_acc.data_ptr<float>();
  p.dq = dq.data_ptr();
  p.dk = dk.data_ptr();
  p.dv = dv.data_ptr();
  ub::launch_fmha_bwd(p, cur_stream());
  check_launch("fmha_bwd");
  return {dq, dk, dv, dbias};
}

// An operand of `sizes` (the last one D) with the dtype of q, read as 16-byte vectors: a contiguous last dim and
// every other stride a multiple of 8 elements
void check_row_operand(const Tensor& t, const char* name, const Tensor& q, at::IntArrayRef sizes) {
  check_operand(t, name, q.device(), {q.scalar_type()}, sizes, kAligned);
  bool ok = t.stride(-1) == 1;
  for (int64_t d = 0; d + 1 < t.dim(); ++d) ok = ok && t.stride(d) % 8 == 0;
  TORCH_CHECK(ok, name, " needs a contiguous last dim and strides that are multiples of 8 elements");
}

// q / k_cache / v_cache / k_new / v_new: [B, L, heads, D] with the B, D and dtype of q, read as 16-byte vectors
void check_decode_operand(const Tensor& t, const char* name, const Tensor& q, int64_t L, int64_t heads) {
  check_row_operand(t, name, q, {q.size(0), L, heads, q.size(3)});
}

// The value cache [B, C, H_kv, D] (D that of q, [..., H, D]) fixes the key / value head count H_kv, which must divide
// the H query heads of q (grouped-query attention); k_cache, k_new and v_new are then checked against it.  Returns H_kv.
int64_t check_cache_heads(const Tensor& q, int64_t B, const Tensor& v_cache) {
  check_row_operand(v_cache, "v_cache", q, {B, kAnySize, kAnySize, q.size(-1)});
  kv_group(q.size(-2), v_cache.size(2), "v_cache");
  return v_cache.size(2);
}

// Paged caches (fmha_api.h): with a block table (int32 [B, M >= 1] on the device of q), k_cache / v_cache are pools
// [num_blocks, block_size, H_kv, D] with one block size, a multiple of 128.  Returns the leading extent the caches are
// checked with afterwards: num_blocks, or B without a table.
int64_t check_paged(const OptTensor& block_table, const Tensor& q, int64_t B, const Tensor& k_cache,
                    const Tensor& v_cache) {
  if (!has(block_table)) return B;
  check_operand(*block_table, "block_table", q.device(), {at::kInt}, {B, kAnySize});
  TORCH_CHECK(block_table->size(1) >= 1, "block_table must have M >= 1 columns");
  check_operand(k_cache, "k_cache", q.device(), {q.scalar_type()}, any_shape(4), kAligned);
  check_operand(v_cache, "v_cache", q.device(), {q.scalar_type()}, any_shape(4), kAligned);
  const int64_t nb = v_cache.size(0), bs = v_cache.size(1);
  TORCH_CHECK(nb >= 1 && k_cache.size(0) == nb && k_cache.size(1) == bs,
              "paged k_cache / v_cache must be pools [num_blocks >= 1, block_size, H_kv, D] of the same shape");
  TORCH_CHECK(bs >= 128 && bs % 128 == 0, "the block size of paged caches must be a multiple of 128, not ", bs);
  TORCH_CHECK(block_table->size(1) * bs <= INT32_MAX, "block_table covers more rows than int32 indexes");
  return nb;
}

// The per-sequence capacity: M * block_size with a block table, else the rows of the caches
int64_t cache_capacity(const OptTensor& block_table, const Tensor& k_cache) {
  return has(block_table) ? block_table->size(1) * k_cache.size(1) : k_cache.size(1);
}

// The paged fields of FmhaFwdParams, FmhaDecodeParams or KvCacheAppendParams (all null / 0 without a table)
template <typename P>
void set_paged(P& p, const OptTensor& block_table, const Tensor& k_cache) {
  p.block_table = has(block_table) ? block_table->data_ptr<int>() : nullptr;
  p.block_size = has(block_table) ? (int)k_cache.size(1) : 0;
  p.blocks_per_seq = has(block_table) ? (int)block_table->size(1) : 0;
  p.num_blocks = has(block_table) ? (int)k_cache.size(0) : 0;
}

// One query row per (b, h) against a [B, C, H_kv, D] key / value cache (fmha_api.h).  max_len is a host bound on
// seqlens (the device values are never read here, so a decode step does not synchronise); with k_new / v_new the row
// seqlens[b] is appended first and counts as visible, so up to max_len + 1 keys are.  num_splits = 0 picks the split
// count from the shapes; any other value forces it.  split_by_length: each (b, h) divides its own device length n_b
// over the splits instead of the host bound (for a CUDA graph captured with the capacity as the bound, where the
// true lengths are far below it); the split count still comes from the bound.
Tensor fmha_decode(const Tensor& q, const Tensor& k_cache, const Tensor& v_cache, const OptTensor& seqlens,
                   int64_t max_len, const OptTensor& k_new, const OptTensor& v_new, const OptTensor& bias,
                   const OptTensor& kpm, double scale, int64_t num_splits, bool split_by_length,
                   const OptTensor& block_table) {
  check_operand(q, "q", q.device(), k16Bit, {kAnySize, 1, kAnySize, kAnySize}, kAligned);
  const int64_t B = q.size(0), H = q.size(2), D = q.size(3);
  TORCH_CHECK(ub::fmha_head_dim_supported(D), "head_dim must be a multiple of 8 from 8 to 128 (8, 16, ..., 128)");
  check_decode_operand(q, "q", q, kAnySize, H);
  const int64_t Bc = check_paged(block_table, q, B, k_cache, v_cache);
  const int64_t H_kv = check_cache_heads(q, Bc, v_cache);
  check_row_operand(k_cache, "k_cache", q, {Bc, kAnySize, H_kv, D});
  TORCH_CHECK(v_cache.size(1) == k_cache.size(1) && k_cache.size(1) >= 1,
              "k_cache / v_cache must have the same capacity C >= 1");
  const int64_t C = cache_capacity(block_table, k_cache);
  const bool append = has(k_new);
  TORCH_CHECK(append == has(v_new), "k_new and v_new go together");
  TORCH_CHECK(!append || has(seqlens), "appending needs seqlens (the row to write)");
  if (append) {
    check_decode_operand(*k_new, "k_new", q, 1, H_kv);
    check_decode_operand(*v_new, "v_new", q, 1, H_kv);
  }
  check_operand(seqlens, "seqlens", q.device(), {at::kInt}, {B});
  if (!has(seqlens)) max_len = C;
  const int64_t bound = max_len + (append ? 1 : 0);   // visible keys of any batch
  TORCH_CHECK(max_len >= 0, "max_len must not be negative");
  TORCH_CHECK(bound <= C, "max_len (+ 1 when appending) exceeds the cache capacity");
  check_operand(bias, "bias", q.device(), {q.scalar_type()}, {kAnySize, H, 1, kAnySize}, 0);
  if (has(bias)) {
    TORCH_CHECK((bias->size(0) == 1 || bias->size(0) == B) && bias->stride(3) == 1,
                "bias must be [1|B, H, 1, Lb] with a contiguous last dim");
    TORCH_CHECK(bias->size(3) >= bound, "bias must have a column for every key that can be visible");
  }
  check_operand(kpm, "key_padding_mask", q.device(), {at::kBool}, {B, kAnySize}, 0);
  TORCH_CHECK(!has(kpm) || (kpm->stride(1) == 1 && kpm->size(1) >= bound),
              "key_padding_mask must have a contiguous last dim and a column for every key that can be visible");
  const c10::cuda::CUDAGuard guard(q.device());
  ub::FmhaDecodeParams p{};
  p.B = (int)B;
  p.H = (int)H;
  p.D = (int)D;
  p.C = (int)C;
  p.kv_group = (int)(H / H_kv);
  p.is_bf16 = q.scalar_type() == at::kBFloat16 ? 1 : 0;
  p.scale = (float)scale;
  p.q = q.data_ptr();
  p.q_sb = q.stride(0); p.q_sh = q.stride(2);
  p.k_cache = k_cache.data_ptr();
  p.kc_sb = k_cache.stride(0); p.kc_sl = k_cache.stride(1); p.kc_sh = k_cache.stride(2);
  p.v_cache = v_cache.data_ptr();
  p.vc_sb = v_cache.stride(0); p.vc_sl = v_cache.stride(1); p.vc_sh = v_cache.stride(2);
  set_paged(p, block_table, k_cache);
  if (append) {
    p.k_new = k_new->data_ptr();
    p.kn_sb = k_new->stride(0); p.kn_sh = k_new->stride(2);
    p.v_new = v_new->data_ptr();
    p.vn_sb = v_new->stride(0); p.vn_sh = v_new->stride(2);
  }
  p.seqlens = has(seqlens) ? seqlens->data_ptr<int>() : nullptr;
  if (has(bias)) {
    p.bias = bias->data_ptr();
    p.bias_batch = (int)bias->size(0);
    p.bias_sb = bias->stride(0); p.bias_sh = bias->stride(1);
    p.bias_cols = (int)bias->size(3);
  }
  if (has(kpm)) {
    p.kpm = reinterpret_cast<const uint8_t*>(kpm->data_ptr());
    p.kpm_sb = kpm->stride(0);
    p.kpm_cols = (int)kpm->size(1);
  }
  if (num_splits == 0) {
    const int sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
    num_splits = ub::fmha_decode_num_splits(p.B, p.H, (int)bound, sms);
  }
  TORCH_CHECK(num_splits >= 1 && num_splits <= ub::kDecodeMaxSplits,
              "num_splits must be 0 (heuristic) or 1 .. fmha_decode_max_splits()");
  p.num_splits = (int)num_splits;
  p.chunk = split_by_length ? 0 : (int)std::max<int64_t>(1, (bound + num_splits - 1) / num_splits);
  Tensor out = torch::empty({p.B, 1, p.H, p.D}, q.options());
  p.out = out.data_ptr();
  Tensor work;
  if (p.num_splits > 1) {
    const int64_t parts = (int64_t)p.B * p.H * p.num_splits;
    work = torch::empty({parts * (D + 2)}, q.options().dtype(at::kFloat));
    p.part_o = work.data_ptr<float>();
    p.part_ml = p.part_o + parts * D;
  }
  ub::launch_fmha_decode(p, cur_stream());
  check_launch("fmha_decode");
  return out;
}

// The checks a chunk into a key / value cache shares in its padded (fmha_kvcache_fwd) and packed
// (fmha_kvcache_varlen_fwd) forms, for B sequences of up to T new queries with the H heads and head dim D of q
// ([..., H, D]): the [B, C, H_kv, D] caches (H_kv dividing H, one capacity C >= 1), k_new / v_new given together and
// exactly when seqlens is, the host bound max_len + T <= C, a bias [1|B, H, T, Lb] with Lb % 8 == 0 (its TMA row
// stride) and a bool key mask [B, Lk], each with a column for every key that can be visible.  k_new / v_new are the
// caller's to check (their layout is the form's).  With a block table the caches are pools (check_paged) and C =
// M * block_size.  Returns {H_kv, kv_cap}.
std::pair<int64_t, int64_t> check_cache_chunk(const Tensor& q, int64_t B, int64_t T, const Tensor& k_cache,
                                              const Tensor& v_cache, const OptTensor& seqlens, int64_t max_len,
                                              const OptTensor& k_new, const OptTensor& v_new, const OptTensor& bias,
                                              const OptTensor& kpm, const OptTensor& block_table) {
  const int64_t H = q.size(-2);
  TORCH_CHECK(ub::fmha_head_dim_supported(q.size(-1)),
              "head_dim must be a multiple of 8 from 8 to 128 (8, 16, ..., 128)");
  const int64_t Bc = check_paged(block_table, q, B, k_cache, v_cache);
  const int64_t H_kv = check_cache_heads(q, Bc, v_cache);
  check_row_operand(k_cache, "k_cache", q, {Bc, kAnySize, H_kv, q.size(-1)});
  TORCH_CHECK(v_cache.size(1) == k_cache.size(1) && k_cache.size(1) >= 1,
              "k_cache / v_cache must have the same capacity C >= 1");
  const int64_t C = cache_capacity(block_table, k_cache);
  const bool append = has(k_new);
  TORCH_CHECK(append == has(v_new), "k_new and v_new go together");
  TORCH_CHECK(append == has(seqlens), "a chunk with seqlens appends k_new / v_new, and one without does not");
  check_operand(seqlens, "seqlens", q.device(), {at::kInt}, {B});
  TORCH_CHECK(max_len >= 0, "max_len must not be negative");
  const int64_t bound = append ? max_len + T : C;   // visible keys of any batch
  TORCH_CHECK(bound <= C, "max_len + T exceeds the cache capacity");
  check_operand(bias, "bias", q.device(), {q.scalar_type()}, {kAnySize, H, T, kAnySize}, kVec);
  if (has(bias)) {
    TORCH_CHECK(bias->size(0) == 1 || bias->size(0) == B, "bias must be [1|B, H, T, Lb]");
    TORCH_CHECK(bias->size(3) % 8 == 0, "bias columns Lb must be a multiple of 8 (the TMA row stride)");
    TORCH_CHECK(bias->size(3) >= bound, "bias must have a column for every key that can be visible");
  }
  check_operand(kpm, "key_padding_mask", q.device(), {at::kBool}, {B, kAnySize});
  TORCH_CHECK(!has(kpm) || kpm->size(1) >= bound, "key_padding_mask must have a column for every key that can be visible");
  int64_t cap = C;
  if (has(bias)) cap = std::min<int64_t>(cap, bias->size(3));
  if (has(kpm)) cap = std::min<int64_t>(cap, kpm->size(1));
  return {H_kv, cap};
}

// Runs a chunk that check_cache_chunk accepted: q4 is [B', T, H, D] as the q map reads it (the padded chunk, or the
// packed rows as the one batch of a [1, N, H, D] view) and out its result; k_new / v_new are appended first (a launch
// of its own), from [B, T, H_kv, D] or, with cu_seqlens, from packed [N, H_kv, D] rows.
void run_cache_chunk(const Tensor& q4, int64_t B, int64_t T, const Tensor& k_cache, const Tensor& v_cache,
                     const OptTensor& seqlens, const OptTensor& k_new, const OptTensor& v_new, const OptTensor& bias,
                     const OptTensor& kpm, int64_t cap, double scale, const Tensor* cu_seqlens,
                     const OptTensor& block_table, Tensor& out) {
  ub::FmhaFwdParams p{};
  // q / k / v as the forward takes them (K / V maps over the C cache rows of the B caches, or over the block_size
  // rows of the num_blocks pool blocks); the bias has Lb columns, not C, so its map is made below
  fill_common(p, q4, k_cache, v_cache, std::nullopt, kpm, 0.0, scale, /*forward=*/true);
  p.B = (int)B;
  p.Lq = (int)T;
  p.Lk = (int)cache_capacity(block_table, k_cache);
  set_paged(p, block_table, k_cache);
  if (has(bias)) {
    p.bias = bias->data_ptr();
    p.bias_batch = (int)bias->size(0);
    TORCH_CHECK(ub::make_bias_tile_map_sw128(&p.sw_bias, p.bias, p.is_bf16 != 0, p.bias_batch * p.H, p.Lq,
                                             (int)bias->size(3)),
                "cuTensorMapEncodeTiled failed for the bias");
  }
  p.kvcache = 1;
  p.seqlens = has(seqlens) ? seqlens->data_ptr<int>() : nullptr;
  p.kpm_cols = has(kpm) ? (int)kpm->size(1) : 0;
  p.kv_cap = (int)cap;
  if (cu_seqlens != nullptr) {
    p.varlen = 1;
    p.cu_seqlens = cu_seqlens->data_ptr<int>();
    p.packed_rows = (int)q4.size(1);
  }
  p.out = out.data_ptr();
  p.lse = nullptr;
  if (has(k_new)) {
    const bool packed = cu_seqlens != nullptr;   // [N, H_kv, D] rows: no batch stride
    ub::KvCacheAppendParams a{};
    a.k_new = k_new->data_ptr();
    a.v_new = v_new->data_ptr();
    a.k_cache = k_cache.data_ptr();
    a.v_cache = v_cache.data_ptr();
    a.seqlens = p.seqlens;
    a.kn_sb = packed ? 0 : k_new->stride(0); a.kn_sl = k_new->stride(packed ? 0 : 1); a.kn_sh = k_new->stride(-2);
    a.vn_sb = packed ? 0 : v_new->stride(0); a.vn_sl = v_new->stride(packed ? 0 : 1); a.vn_sh = v_new->stride(-2);
    a.kc_sb = p.k_sb; a.kc_sl = p.k_sl; a.kc_sh = p.k_sh;
    a.vc_sb = p.v_sb; a.vc_sl = p.v_sl; a.vc_sh = p.v_sh;
    a.B = p.B; a.T = p.Lq; a.H = (int)k_cache.size(2); a.D = p.D; a.C = p.Lk;
    a.cu_seqlens = p.cu_seqlens;
    a.packed_rows = p.packed_rows;
    set_paged(a, block_table, k_cache);
    ub::launch_kv_cache_append(a, cur_stream());
    check_launch("kv_cache_append");
  }
  ub::launch_fmha_fwd(p, cur_stream());
}

// A chunk of T >= 2 queries per sequence against a [B, C, H, D] key / value cache, in the KV-cache mode of the wgmma
// forward (fmha_api.h).  With seqlens the T rows of k_new / v_new are first appended at rows seqlens[b] + i (a launch
// of its own), and query i sees the keys j <= seqlens[b] + i; without seqlens every query sees all C rows.  max_len
// is a host bound on seqlens, as in fmha_decode.  The bias is [1|B, H, T, Lb] with Lb % 8 == 0 (its TMA row stride).
Tensor fmha_kvcache_fwd(const Tensor& q, const Tensor& k_cache, const Tensor& v_cache, const OptTensor& seqlens,
                        int64_t max_len, const OptTensor& k_new, const OptTensor& v_new, const OptTensor& bias,
                        const OptTensor& kpm, double scale, const OptTensor& block_table) {
  check_operand(q, "q", q.device(), k16Bit, any_shape(4), kAligned);
  const int64_t B = q.size(0), T = q.size(1), H = q.size(2), D = q.size(3);
  TORCH_CHECK(T >= 2, "fmha_kvcache_fwd takes chunks of T >= 2 queries (fmha_decode takes T = 1)");
  check_decode_operand(q, "q", q, kAnySize, H);
  const auto [H_kv, cap] = check_cache_chunk(q, B, T, k_cache, v_cache, seqlens, max_len, k_new, v_new, bias, kpm,
                                             block_table);
  if (has(k_new)) {
    check_decode_operand(*k_new, "k_new", q, T, H_kv);
    check_decode_operand(*v_new, "v_new", q, T, H_kv);
  }
  const c10::cuda::CUDAGuard guard(q.device());
  Tensor out = torch::empty({B, T, H, D}, q.options());
  run_cache_chunk(q, B, T, k_cache, v_cache, seqlens, k_new, v_new, bias, kpm, cap, scale, nullptr, block_table, out);
  check_launch("fmha_kvcache_fwd");
  return out;
}

// Packed chunks into a [B, C, H_kv, D] key / value cache: q [N, H, D] holds B sequences back to back, sequence b's
// T_b new queries on rows s_b .. s_b + T_b - 1 with {s_b, T_b} clamped from cu_seqlens (int32 [B + 1] on the device)
// as in the varlen mode (fmha_api.h), and max_seqlen a host bound on T_b (any value >= 1: the KV-cache mode takes
// any T).  With seqlens the rows of k_new / v_new [N, H_kv, D] are first appended at rows seqlens[b] + i, i < T_b
// (rows at or past C are skipped), and query i sees the keys j <= seqlens[b] + i; without seqlens every query sees
// all C rows.  max_len is a host bound on seqlens.  The bias is [1|B, H, max_seqlen, Lb] (row i for query i of every
// sequence) with Lb % 8 == 0, the key mask [B, Lk].  Returns [N, H, D]; rows of no sequence are not written.
Tensor fmha_kvcache_varlen_fwd(const Tensor& q, const Tensor& k_cache, const Tensor& v_cache, const Tensor& cu_seqlens,
                               int64_t max_seqlen, const OptTensor& seqlens, int64_t max_len, const OptTensor& k_new,
                               const OptTensor& v_new, const OptTensor& bias, const OptTensor& kpm, double scale,
                               const OptTensor& block_table) {
  check_operand(q, "q", q.device(), k16Bit, any_shape(3), kAligned);
  const int64_t N = q.size(0), H = q.size(1), D = q.size(2);
  check_row_operand(q, "q", q, {kAnySize, H, D});
  TORCH_CHECK(N >= 1, "q must have N >= 1 packed rows");
  TORCH_CHECK(q.stride(1) == D, "q head stride must be head_dim");   // (head, 16-byte chunk) is one TMA dimension
  check_operand(cu_seqlens, "cu_seqlens", q.device(), {at::kInt}, {kAnySize});
  const int64_t B = cu_seqlens.size(0) - 1;
  TORCH_CHECK(B >= 1, "cu_seqlens must have B + 1 >= 2 entries");
  TORCH_CHECK(max_seqlen >= 1, "max_seqlen must be positive");
  const auto [H_kv, cap] = check_cache_chunk(q, B, max_seqlen, k_cache, v_cache, seqlens, max_len, k_new, v_new, bias,
                                             kpm, block_table);
  if (has(k_new)) {
    check_row_operand(*k_new, "k_new", q, {N, H_kv, D});
    check_row_operand(*v_new, "v_new", q, {N, H_kv, D});
  }
  const c10::cuda::CUDAGuard guard(q.device());
  Tensor out = torch::empty({N, H, D}, q.options());
  run_cache_chunk(q.unsqueeze(0), B, max_seqlen, k_cache, v_cache, seqlens, k_new, v_new, bias, kpm, cap, scale,
                  &cu_seqlens, block_table, out);
  check_launch("fmha_kvcache_varlen_fwd");
  return out;
}

// The append of fmha_kvcache_fwd alone: rows i of k_new / v_new [B, T, H_kv, D] go to rows seqlens[b] + i of the
// [B, C, H_kv, D] caches, or with a block table through it into the pools (fmha_api.h); rows at or past C, and rows
// whose table entry is outside the pool, are skipped.  Bitwise.
void kv_cache_append(const Tensor& k_new, const Tensor& v_new, const Tensor& k_cache, const Tensor& v_cache,
                     const Tensor& seqlens, const OptTensor& block_table) {
  check_operand(k_new, "k_new", k_new.device(), k16Bit, any_shape(4), kAligned);
  const int64_t B = k_new.size(0), T = k_new.size(1), H_kv = k_new.size(2), D = k_new.size(3);
  TORCH_CHECK(ub::fmha_head_dim_supported(D), "head_dim must be a multiple of 8 from 8 to 128 (8, 16, ..., 128)");
  TORCH_CHECK(B >= 1 && T >= 1, "k_new must have B >= 1 sequences of T >= 1 rows");
  check_row_operand(k_new, "k_new", k_new, {B, T, H_kv, D});
  check_row_operand(v_new, "v_new", k_new, {B, T, H_kv, D});
  const int64_t Bc = check_paged(block_table, k_new, B, k_cache, v_cache);
  check_row_operand(k_cache, "k_cache", k_new, {Bc, kAnySize, H_kv, D});
  check_row_operand(v_cache, "v_cache", k_new, {Bc, k_cache.size(1), H_kv, D});
  TORCH_CHECK(k_cache.size(1) >= 1, "k_cache / v_cache must have C >= 1 rows");
  check_operand(seqlens, "seqlens", k_new.device(), {at::kInt}, {B});
  const c10::cuda::CUDAGuard guard(k_new.device());
  ub::KvCacheAppendParams a{};
  a.k_new = k_new.data_ptr();
  a.v_new = v_new.data_ptr();
  a.k_cache = k_cache.data_ptr();
  a.v_cache = v_cache.data_ptr();
  a.seqlens = seqlens.data_ptr<int>();
  a.kn_sb = k_new.stride(0); a.kn_sl = k_new.stride(1); a.kn_sh = k_new.stride(2);
  a.vn_sb = v_new.stride(0); a.vn_sl = v_new.stride(1); a.vn_sh = v_new.stride(2);
  a.kc_sb = k_cache.stride(0); a.kc_sl = k_cache.stride(1); a.kc_sh = k_cache.stride(2);
  a.vc_sb = v_cache.stride(0); a.vc_sl = v_cache.stride(1); a.vc_sh = v_cache.stride(2);
  a.B = (int)B; a.T = (int)T; a.H = (int)H_kv; a.D = (int)D; a.C = (int)cache_capacity(block_table, k_cache);
  set_paged(a, block_table, k_cache);
  ub::launch_kv_cache_append(a, cur_stream());
  check_launch("kv_cache_append");
}

// The block allocator of paged caches (fmha_api.h): block_table int32 [B, M], free_list int32 [num_blocks >= 1],
// free_count and overflow int32 [1], lengths int32 [B], all contiguous on one device.
ub::KvBlocksParams check_kv_blocks(const Tensor& block_table, const Tensor& free_list, const Tensor& free_count,
                                   const Tensor& lengths, int64_t block_size, const Tensor* overflow) {
  const c10::Device dev = block_table.device();
  check_operand(block_table, "block_table", dev, {at::kInt}, any_shape(2));
  const int64_t B = block_table.size(0), M = block_table.size(1);
  TORCH_CHECK(B >= 1 && M >= 1, "block_table must be [B >= 1, M >= 1]");
  check_operand(free_list, "free_list", dev, {at::kInt}, {kAnySize});
  TORCH_CHECK(free_list.size(0) >= 1 && free_list.size(0) <= INT32_MAX, "free_list must have num_blocks >= 1 entries");
  check_operand(free_count, "free_count", dev, {at::kInt}, {1}, kContig | kNumel);
  check_operand(lengths, "lengths", dev, {at::kInt}, {B});
  if (overflow != nullptr) check_operand(*overflow, "overflow", dev, {at::kInt}, {1}, kContig | kNumel);
  TORCH_CHECK(block_size >= 1 && M * block_size <= INT32_MAX,
              "block_size must be positive, and M * block_size fit int32");
  ub::KvBlocksParams p{};
  p.block_table = block_table.data_ptr<int>();
  p.free_list = free_list.data_ptr<int>();
  p.free_count = free_count.data_ptr<int>();
  p.overflow = overflow != nullptr ? overflow->data_ptr<int>() : nullptr;
  p.lengths = lengths.data_ptr<int>();
  p.B = (int)B;
  p.blocks_per_seq = (int)M;
  p.block_size = (int)block_size;
  p.num_blocks = (int)free_list.size(0);
  return p;
}

void kv_blocks_reserve(const Tensor& block_table, const Tensor& free_list, const Tensor& free_count,
                       const Tensor& lengths, int64_t block_size, const Tensor& overflow) {
  const ub::KvBlocksParams p = check_kv_blocks(block_table, free_list, free_count, lengths, block_size, &overflow);
  const c10::cuda::CUDAGuard guard(block_table.device());
  ub::launch_kv_blocks_reserve(p, cur_stream());
  check_launch("kv_blocks_reserve");
}

void kv_blocks_release(const Tensor& block_table, const Tensor& free_list, const Tensor& free_count,
                       const Tensor& lengths, int64_t block_size) {
  const ub::KvBlocksParams p = check_kv_blocks(block_table, free_list, free_count, lengths, block_size, nullptr);
  const c10::cuda::CUDAGuard guard(block_table.device());
  ub::launch_kv_blocks_release(p, cur_stream());
  check_launch("kv_blocks_release");
}
// ---- varlen: packed sequences described by cu_seqlens (fmha_api.h) ------------------------------------------------
// q [N_q, H, D], k / v [N_k, H_kv, D] (head slices of one projection are fine), cu_seqlens int32 [B + 1] on the
// device, max_seqlen a host bound on the query lengths (a multiple of 8: the row stride of the bias, LSE, keep-bit and
// dS maps), bias [1|B, H, max_seqlen, max_seqlen_k].  cu_seqlens_k (int32 [B + 1] on the device, the same B) describes
// separate key sequences, and max_seqlen_k bounds their lengths (0: max_seqlen); without it the keys are the queries'
// own rows (N_k == N_q).  No key padding mask: the lengths take its place.  Causal needs the queries' own keys.
// Returns {B, max_seqlen_k}.
std::pair<int64_t, int64_t> check_varlen(const Tensor& q, const Tensor& k, const Tensor& v, const Tensor& cu_seqlens,
                                         int64_t max_seqlen, const OptTensor& bias, const OptTensor& cu_seqlens_k,
                                         int64_t max_seqlen_k, bool causal) {
  check_operand(q, "q", q.device(), k16Bit, any_shape(3), kAligned);
  check_operand(k, "k", q.device(), {q.scalar_type()}, any_shape(3), kAligned);
  check_operand(v, "v", q.device(), {q.scalar_type()}, any_shape(3), kAligned);
  const int64_t N = q.size(0), H = q.size(1), D = q.size(2), H_kv = v.size(1), N_k = k.size(0);
  TORCH_CHECK(ub::fmha_head_dim_supported(D) && k.size(2) == D && v.size(2) == D,
              "head_dim must be the same for q/k/v and a multiple of 8 from 8 to 128 (8, 16, ..., 128)");
  TORCH_CHECK(N >= 1 && N_k >= 1 && v.size(0) == N_k && k.size(1) == H_kv,
              "k / v must be [N_k, H_kv, D] with N_k >= 1 packed rows each and the D of q");
  TORCH_CHECK(has(cu_seqlens_k) || N_k == N,
              "k / v must be [N, H_kv, D] with the N packed rows of q when cu_seqlens_k is not given");
  kv_group(H, H_kv, "v");
  for (const Tensor* t : {&q, &k, &v}) {
    TORCH_CHECK(t->stride(2) == 1 && t->stride(1) == D, "q/k/v head stride must be head_dim");
    TORCH_CHECK(t->stride(0) % 8 == 0, "q/k/v row strides must be multiples of 8 elements");
  }
  check_operand(cu_seqlens, "cu_seqlens", q.device(), {at::kInt}, {kAnySize});
  const int64_t B = cu_seqlens.size(0) - 1;
  TORCH_CHECK(B >= 1, "cu_seqlens must have B + 1 >= 2 entries");
  check_operand(cu_seqlens_k, "cu_seqlens_k", q.device(), {at::kInt}, {B + 1});
  TORCH_CHECK(!(causal && has(cu_seqlens_k)), "causal attention is not defined with separate key sequences "
              "(cu_seqlens_k)");
  TORCH_CHECK(max_seqlen >= 1 && max_seqlen % 8 == 0, "max_seqlen must be a positive multiple of 8");
  const int64_t Lk = max_seqlen_k == 0 ? max_seqlen : max_seqlen_k;
  TORCH_CHECK(Lk >= 1 && Lk % 8 == 0, "max_seqlen_k must be 0 or a positive multiple of 8");
  TORCH_CHECK(has(cu_seqlens_k) || Lk == max_seqlen, "max_seqlen_k other than max_seqlen needs cu_seqlens_k");
  check_operand(bias, "bias", q.device(), {q.scalar_type()}, {kAnySize, H, max_seqlen, Lk}, kVec);
  TORCH_CHECK(!has(bias) || bias->size(0) == 1 || bias->size(0) == B,
              "bias must be [1|B, H, max_seqlen, max_seqlen_k]");
  return {B, Lk};
}

// The parameters of a varlen call: q / k / v maps over the N_q / N_k packed rows (B = 1), everything else at
// B x max_seqlen (x max_seqlen_k); the key description is the query one when cu_seqlens_k is not given
void fill_varlen(ub::FmhaFwdParams& p, const Tensor& q, const Tensor& k, const Tensor& v, const Tensor& cu_seqlens,
                 int64_t B, int64_t max_seqlen, const OptTensor& cu_seqlens_k, int64_t max_seqlen_k,
                 const OptTensor& bias, double p_drop, double scale, bool causal, bool forward) {
  fill_common(p, q.unsqueeze(0), k.unsqueeze(0), v.unsqueeze(0), std::nullopt, std::nullopt, p_drop, scale, forward);
  p.B = (int)B;
  p.Lq = (int)max_seqlen;
  p.Lk = (int)max_seqlen_k;
  p.causal = causal ? 1 : 0;
  p.varlen = 1;
  p.cu_seqlens = cu_seqlens.data_ptr<int>();
  p.packed_rows = (int)q.size(0);
  p.cu_seqlens_k = has(cu_seqlens_k) ? cu_seqlens_k->data_ptr<int>() : p.cu_seqlens;
  p.packed_rows_k = (int)k.size(0);
  if (has(bias)) {
    p.bias = bias->data_ptr();
    p.bias_batch = (int)bias->size(0);
    TORCH_CHECK(ub::make_bias_tile_map_sw128(&p.sw_bias, p.bias, p.is_bf16 != 0, p.bias_batch * p.H, p.Lq, p.Lk),
                "cuTensorMapEncodeTiled failed for the bias");
  }
}

// (out [N_q, H, D], lse [B, H, max_seqlen], keep bits [B, H, max_seqlen, ceil(max_seqlen_k / 32)] or None); rows of
// LSE and of the keep bits past each sequence's query length are not written
std::tuple<Tensor, Tensor, OptTensor> fmha_varlen_fwd(const Tensor& q, const Tensor& k, const Tensor& v,
                                                      const Tensor& cu_seqlens, int64_t max_seqlen, const OptTensor& bias,
                                                      double p_drop, double scale, bool causal,
                                                      const OptTensor& cu_seqlens_k, int64_t max_seqlen_k) {
  const auto [B, Lk] = check_varlen(q, k, v, cu_seqlens, max_seqlen, bias, cu_seqlens_k, max_seqlen_k, causal);
  const c10::cuda::CUDAGuard guard(q.device());
  ub::FmhaFwdParams p{};
  fill_varlen(p, q, k, v, cu_seqlens, B, max_seqlen, cu_seqlens_k, Lk, bias, p_drop, scale, causal, /*forward=*/true);
  Tensor out = torch::empty({q.size(0), p.H, p.D}, q.options());
  Tensor lse = torch::empty({p.B, p.H, p.Lq}, q.options().dtype(at::kFloat));
  p.out = out.data_ptr();
  p.lse = lse.data_ptr<float>();
  p.seed = p.offset = 0;
  OptTensor bits;
  if (p_drop > 0.0) {
    std::tie(p.seed, p.offset) = philox_reserve(4);
    bits = torch::empty({p.B, p.H, p.Lq, (p.Lk + 31) / 32}, q.options().dtype(at::kInt));
    p.drop_bits = reinterpret_cast<uint32_t*>(bits->data_ptr());
  }
  ub::launch_fmha_fwd(p, cur_stream());
  check_launch("fmha_varlen_fwd");
  return {out, lse, bits};
}

// packed_grad: q / k / v are the head slices of one [N, H + 2 H_kv, D] projection, and the gradients are written into
// one tensor of that layout (returned three times as views), as fmha_bwd does for [B, L, H + 2 H_kv, D]; self-attention
// only.  dK / dV are [N_k, H_kv, D].  dBias is 0 outside every sequence's n_q x n_k block.
std::tuple<Tensor, Tensor, Tensor, OptTensor> fmha_varlen_bwd(const Tensor& dout, const Tensor& q, const Tensor& k,
                                                              const Tensor& v, const Tensor& out, const Tensor& lse,
                                                              const Tensor& cu_seqlens, int64_t max_seqlen,
                                                              const OptTensor& bias, double p_drop, double scale,
                                                              const OptTensor& drop_bits, bool need_dbias,
                                                              bool packed_grad, bool causal,
                                                              const OptTensor& cu_seqlens_k, int64_t max_seqlen_k) {
  const auto [B, Lk] = check_varlen(q, k, v, cu_seqlens, max_seqlen, bias, cu_seqlens_k, max_seqlen_k, causal);
  const int64_t N = q.size(0), H = q.size(1), D = q.size(2), N_k = k.size(0), H_kv = k.size(1), L = max_seqlen;
  check_operand(dout, "dout", q.device(), {q.scalar_type()}, q.sizes(), kVec);
  check_operand(out, "out", q.device(), {q.scalar_type()}, q.sizes());
  check_operand(lse, "lse", q.device(), {at::kFloat}, {B, H, L});
  TORCH_CHECK(p_drop <= 0.0 || has(drop_bits), "dropout bits missing");
  if (p_drop > 0.0) check_operand(drop_bits, "drop_bits", q.device(), {at::kInt}, {B, H, L, (Lk + 31) / 32});
  TORCH_CHECK(!(packed_grad && has(cu_seqlens_k)), "packed gradients need self-attention (no cu_seqlens_k)");
  const c10::cuda::CUDAGuard guard(q.device());
  ub::FmhaBwdParams p{};
  fill_varlen(p.f, q, k, v, cu_seqlens, B, max_seqlen, cu_seqlens_k, Lk, bias, p_drop, scale, causal,
              /*forward=*/false);
  p.f.out = out.data_ptr();
  p.f.lse = lse.data_ptr<float>();
  if (p_drop > 0.0) p.f.drop_bits = reinterpret_cast<uint32_t*>(drop_bits->data_ptr());
  p.dout = dout.data_ptr();
  TORCH_CHECK(ub::make_head_tile_map_sw128(&p.sw_do, p.dout, p.f.is_bf16 != 0, 1, (int)N, (int)H, (int)D, N * H * D,
                                           H * D, D, ub::kBwdBoxRows),
              "cuTensorMapEncodeTiled failed for dO");
  Tensor delta = torch::empty({B, H, L}, q.options().dtype(at::kFloat));
  const bool det = at::globalContext().deterministicAlgorithms();
  const int64_t n_qt = (L + 63) / 64;
  const int64_t acc_floats = B * H * n_qt * 64 * ub::fmha_padded_head_dim((int)D);
  Tensor dq_acc = torch::empty({acc_floats + (det ? B * H * n_qt : 0)}, q.options().dtype(at::kFloat));
  p.dq_turn = det ? reinterpret_cast<int*>(dq_acc.data_ptr<float>() + acc_floats) : nullptr;
  Tensor dq, dk, dv;
  if (packed_grad) {
    Tensor dqkv = torch::empty({N, H + 2 * H_kv, D}, q.options());
    dq = dqkv.narrow(1, 0, H);
    dk = dqkv.narrow(1, H, H_kv);
    dv = dqkv.narrow(1, H + H_kv, H_kv);
  } else {
    dq = torch::empty({N, H, D}, q.options());
    dk = torch::empty({N_k, H_kv, D}, q.options());
    dv = torch::empty({N_k, H_kv, D}, q.options());
  }
  // the kernels address row r of sequence b as row s_b + r through the row stride; the batch stride is unused
  p.dq_sb = p.dk_sb = p.dv_sb = 0;
  p.dq_sl = dq.stride(0); p.dq_sh = dq.stride(1);
  p.dk_sl = dk.stride(0); p.dk_sh = dk.stride(1);
  p.dv_sl = dv.stride(0); p.dv_sh = dv.stride(1);
  OptTensor dbias;
  Tensor ds_buf;
  if (need_dbias && p.f.bias != nullptr) {
    // zeroed by the launcher: the kernels store the tiles inside each sequence's block only
    ds_buf = torch::empty({B, H, L, Lk}, q.options());
    p.ds_buf = ds_buf.data_ptr();
    dbias = (p.f.bias_batch == B) ? ds_buf : torch::empty({p.f.bias_batch, H, L, Lk}, q.options());
    p.dbias = dbias->data_ptr();
    TORCH_CHECK(ub::make_bias_tile_map_sw128(&p.sw_ds, p.ds_buf, p.f.is_bf16 != 0, (int)(B * H), (int)L, (int)Lk),
                "cuTensorMapEncodeTiled failed for the dS scratch tensor");
  }
  p.delta = delta.data_ptr<float>();
  p.dq_acc = dq_acc.data_ptr<float>();
  p.dq = dq.data_ptr();
  p.dk = dk.data_ptr();
  p.dv = dv.data_ptr();
  ub::launch_fmha_bwd(p, cur_stream());
  check_launch("fmha_varlen_bwd");
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
  m.def("fmha_decode", &fmha_decode, py::arg("q"), py::arg("k_cache"), py::arg("v_cache"), py::arg("seqlens"),
        py::arg("max_len"), py::arg("k_new"), py::arg("v_new"), py::arg("bias"), py::arg("key_padding_mask"),
        py::arg("scale"), py::arg("num_splits") = 0, py::arg("split_by_length") = false,
        py::arg("block_table") = py::none());
  // its own submodule, _C.kvcache; tests/test_gpu_attention_kvcache_chunk.py runs the operand-rejection table of
  // tests/test_gpu_bindings.py over it
  auto kv = m.def_submodule("kvcache", "multi-token steps into a key / value cache");
  kv.def("fmha_kvcache_fwd", &fmha_kvcache_fwd, py::arg("q"), py::arg("k_cache"), py::arg("v_cache"),
         py::arg("seqlens"), py::arg("max_len"), py::arg("k_new"), py::arg("v_new"), py::arg("bias"),
         py::arg("key_padding_mask"), py::arg("scale"), py::arg("block_table") = py::none());
  kv.def("fmha_kvcache_varlen_fwd", &fmha_kvcache_varlen_fwd, py::arg("q"), py::arg("k_cache"), py::arg("v_cache"),
         py::arg("cu_seqlens"), py::arg("max_seqlen"), py::arg("seqlens"), py::arg("max_len"), py::arg("k_new"),
         py::arg("v_new"), py::arg("bias"), py::arg("key_padding_mask"), py::arg("scale"),
         py::arg("block_table") = py::none());
  // paged caches: the append on its own (a prefill's rows, a reorder's rows written back) and the block allocator
  kv.def("kv_cache_append", &kv_cache_append, py::arg("k_new"), py::arg("v_new"), py::arg("k_cache"),
         py::arg("v_cache"), py::arg("seqlens"), py::arg("block_table") = py::none());
  kv.def("kv_blocks_reserve", &kv_blocks_reserve, py::arg("block_table"), py::arg("free_list"), py::arg("free_count"),
         py::arg("lengths"), py::arg("block_size"), py::arg("overflow"));
  kv.def("kv_blocks_release", &kv_blocks_release, py::arg("block_table"), py::arg("free_list"), py::arg("free_count"),
         py::arg("lengths"), py::arg("block_size"));
  // packed variable-length sequences: its own submodule, _C.varlen
  auto vl = m.def_submodule("varlen", "packed variable-length sequences described by cu_seqlens");
  vl.def("fmha_varlen_fwd", &fmha_varlen_fwd, py::arg("q"), py::arg("k"), py::arg("v"), py::arg("cu_seqlens"),
         py::arg("max_seqlen"), py::arg("bias"), py::arg("p_drop"), py::arg("scale"), py::arg("causal") = false,
         py::arg("cu_seqlens_k") = py::none(), py::arg("max_seqlen_k") = 0);
  vl.def("fmha_varlen_bwd", &fmha_varlen_bwd, py::arg("dout"), py::arg("q"), py::arg("k"), py::arg("v"),
         py::arg("out"), py::arg("lse"), py::arg("cu_seqlens"), py::arg("max_seqlen"), py::arg("bias"),
         py::arg("p_drop"), py::arg("scale"), py::arg("drop_bits"), py::arg("need_dbias"), py::arg("packed_grad"),
         py::arg("causal") = false, py::arg("cu_seqlens_k") = py::none(), py::arg("max_seqlen_k") = 0);
  m.def("fmha_decode_max_splits", [] { return (int64_t)ub::kDecodeMaxSplits; });
  m.def("fmha_decode_num_splits", [](int64_t B, int64_t H, int64_t len_bound) {
    return (int64_t)ub::fmha_decode_num_splits((int)B, (int)H, (int)len_bound,
                                               at::cuda::getCurrentDeviceProperties()->multiProcessorCount);
  }, "split count fmha_decode picks with num_splits = 0 for B x H rows and at most len_bound visible keys");
  m.def("fmha_det_timeouts", [] { return (int64_t)ub::fmha_det_timeouts_take(); },
        "deterministic-mode dQ turn waits that timed out on the current device since the last call (reset on read)");
}
