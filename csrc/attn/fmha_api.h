// Host launchers of the wgmma fused attention kernels (csrc/attn/fmha_*_sm90.cu).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace ub {

// Head dims the kernels take: D % 8 == 0 and 8 <= D <= 128.  D <= 64 runs on the 64-column kernels, larger D on the
// 128-column ones; the TMA unit zero-fills the columns D..63 / D..127 of every tile in shared memory.
constexpr int kMaxHeadDim = 128;
inline bool fmha_head_dim_supported(long long d) { return d >= 8 && d <= kMaxHeadDim && d % 8 == 0; }
inline int fmha_padded_head_dim(int d) { return d <= 64 ? 64 : 128; }

// rows of the TMA boxes of q / k / v (and dO): the forward walks 128-key tiles (64-key tiles at padded width 128)
// with 64 query rows per CTA, the backward walks 64-row query tiles with 64 keys per CTA
constexpr int kFwdQBoxRows = 64, kBwdBoxRows = 64;
inline int fmha_fwd_kv_box_rows(int d) { return d <= 64 ? 128 : 64; }

struct FmhaFwdParams {
  const void* q;   // [B, Lq, H, D] via strides (elements)
  const void* k;   // [B, Lk, H, D]
  const void* v;
  void* out;       // [B, Lq, H, D] contiguous
  float* lse;      // [B, H, Lq]
  const void* bias;        // [bias_batch (1 or B), H, Lq, Lk] contiguous, same 16-bit type as q; may be null
  const uint8_t* kpm;      // [B, Lk] bool, nonzero = masked; may be null
  // [B, H, Lq, ceil(Lk/32)] dropout keep bits (written by fwd, read by bwd); null if p == 0.  Word w of a row holds
  // keys 32w .. 32w + 31: key 32w + 2i in bit i, key 32w + 2i + 1 in bit 16 + i.
  uint32_t* drop_bits;
  long long q_sb, q_sl, q_sh, k_sb, k_sl, k_sh, v_sb, v_sl, v_sh;
  int B, H, Lq, Lk, D;
  int bias_batch, bias_is_f32, is_bf16;
  float scale, p_drop;
  unsigned long long seed, offset;
  // TMA descriptors (csrc/attn/tma_map.h), 128-byte swizzle: row tiles of q / k / v, 64 x 64 tiles of the bias
  CUtensorMap sw_q, sw_k, sw_v, sw_bias;
  // Logits mode (forward only): z = scale * Q K^T + bias + key mask, [B, H, Lq, Lk] contiguous in the dtype of q,
  // -inf at masked keys; null otherwise.  sw_logits: 64 x 64 boxes of z (the bias map's layout, B * H matrices).
  void* logits;
  // Causal: key j is visible to query i iff j <= i (top-left aligned for any Lq, Lk, the mask
  // triu(full((Lq, Lk), -inf), 1)).  Key tiles wholly above the diagonal are skipped; not combined with logits mode.
  int causal;
  CUtensorMap sw_logits;
};
void launch_fmha_fwd(const FmhaFwdParams& p, cudaStream_t stream);

struct FmhaBwdParams {
  FmhaFwdParams f;   // same inputs as forward (out/lse hold the forward results)
  const void* dout;  // [B, Lq, H, D] contiguous
  float* delta;      // [B, H, Lq] scratch: rowsum(dO * O)
  float* dq_acc;     // [B, H, ceil(Lq / 64) * 64, DP] fp32 (DP = padded head width), zeroed: every key tile adds its
                     // dQ share with bulk reductions.  Row q keeps its 8-column groups in the order group ^ (q & 7)
                     // (the conflict-free layout of the tile in shared memory); only the dQ convert kernel reads it.
  void* dq;          // [B, Lq, H, D] 16-bit results, addressed through (batch, seq, head) element strides so
  void* dk;          // that they can be slices of one packed [B, L, 3, H, D] gradient tensor
  void* dv;
  long long dq_sb, dq_sl, dq_sh, dk_sb, dk_sl, dk_sh, dv_sb, dv_sl, dv_sh;
  // Bias gradient: every CTA stores its 16-bit dS tile (already in shared memory for the dQ product) with one TMA
  // store into ds_buf [B, H, Lq, Lk]; a follow-up kernel sums it over the batch into dbias (fp32 accumulate)
  // when the bias is shared by the batch.  Both null when the bias needs no gradient.
  void* ds_buf;      // [B, H, Lq, Lk] 16-bit
  void* dbias;       // [bias_batch, H, Lq, Lk] 16-bit; == ds_buf when bias_batch == B
  CUtensorMap sw_ds;   // 128-byte-swizzled map of ds_buf (64 x 64 boxes)
  CUtensorMap sw_do;   // 64-row x 64-column boxes of dO (128-byte swizzle)
  // Logits mode: the incoming gradient dz of the forward's logits output, [B, H, Lq, Lk] contiguous 16-bit, added to
  // dS everywhere (dS_total = P o (drop(dP) - delta) + dz feeds dQ, dK and dBias); null runs the plain backward.
  const void* dlogits;
  CUtensorMap sw_dz;   // 64 x 64 boxes of dlogits (the bias map's layout, B * H matrices)
  // Deterministic mode (torch.use_deterministic_algorithms): one int32 turn counter per (b, h, query tile),
  // [B, H, ceil(Lq / 64)], stored right after dq_acc in the same allocation and zeroed with it.  The key tiles then add
  // their dQ shares into each query tile in ascending key-tile order, so dQ does not depend on the CTA schedule.
  // Null runs the default kernels, which add in completion order.
  int* dq_turn;
};
void launch_fmha_bwd(const FmhaBwdParams& p, cudaStream_t stream);
// Number of deterministic-mode waits for a turn that gave up after ~10 s (and added out of order) on the current
// device since the last call; reading resets it.  Any value other than 0 is a bug.
unsigned int fmha_det_timeouts_take();

}  // namespace ub
