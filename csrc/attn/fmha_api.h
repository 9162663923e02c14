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
  // KV-cache mode (fmha_kvcache_fwd; appended so that no earlier field moves): q is a chunk of Lq = T queries per
  // sequence, k / v are [B, C, H, D] caches (Lk = C).  With p_b = clamp(seqlens[b], 0, C) and
  // n_b = min(p_b + T, kv_cap), query i of sequence b sees key j iff j < n_b and j <= p_b + i (the future mask of the
  // whole sequence, aligned bottom-right per sequence); with seqlens null, p_b = C: every row below kv_cap is visible
  // to every query (cross-attention).  kv_cap = min(C, bias columns, key-mask columns); the bias map is
  // [bias_batch * H, T, Lb], the key mask [B, kpm_cols] contiguous.  No dropout, no keep bits, lse may be null.
  const int* seqlens;
  int kvcache, kv_cap, kpm_cols;
  // Grouped-query attention (appended so that no earlier field moves): k / v hold H / kv_group heads, and query head h
  // reads key / value head h / kv_group (the order of repeat_interleave(kv_group, dim=2)).  1 = one per query head.
  // Everything else - bias, key mask, keep bits, Philox counters, LSE, logits - stays per query head.
  int kv_group;
  // Varlen mode (fmha_varlen_fwd / fmha_varlen_bwd; appended so that no earlier field moves): the B sequences are
  // packed back to back.  q is [N, H, D], k / v [N, H_kv, D] (strided views with B = 1 in the TMA maps, L = N), and
  // sequence b holds rows s_b .. s_b + n_b - 1 with s_b = clamp(cu_seqlens[b], 0, N) and
  // n_b = clamp(cu_seqlens[b + 1] - cu_seqlens[b], 0, min(Lq, N - s_b)); Lq = Lk = max_seqlen (self-attention; the
  // key description below generalises this to separate key sequences).  O [N, H, D] (and dO) are
  // packed too.  Everything per (b, h, row) keeps the padded layout of B sequences of Lq rows: LSE, keep bits, Philox
  // counters, delta, the dQ accumulator and turn counters, the bias [1|B, H, Lq, Lk] (sequence b reads its top-left
  // n_b x n_b block) and dS / dBias.  Query i of sequence b sees keys j < n_b (and j <= i when causal): the result at
  // every row i < n_b is that of the padded call with key_padding_mask = (j >= n_b).  kpm must be null; no logits.
  const int* cu_seqlens;   // [B + 1] int32 on the device
  int varlen, packed_rows; // packed_rows = N
  // Varlen keys (appended so that no earlier field moves): every varlen call reads its key ranges from these.  k / v
  // are [N_k, H_kv, D] and sequence b's keys are rows s_k + 0 .. s_k + n_k - 1 with {s_k, n_k} =
  // fmha_varlen_seq(cu_seqlens_k, b, Lk, N_k), while its queries keep {s_q, n_q} from cu_seqlens, Lq and N_q; Lq =
  // max_seqlen and Lk = max_seqlen_k may differ (cross-attention).  Self-attention sets cu_seqlens_k = cu_seqlens and
  // packed_rows_k = packed_rows.  Query i < n_q of sequence b sees keys j < n_k, reads bias[b', h, i, j] of its top-left
  // n_q x n_k block, and gets the result of the padded call with key_padding_mask = (j >= n_k).  A sequence with
  // n_k = 0 < n_q follows the kernels' fully-masked contract: O = 0, LSE = -inf, dQ = 0 and no gradient elsewhere.
  // Causal is defined only for cu_seqlens_k == cu_seqlens (the bindings refuse it otherwise).
  const int* cu_seqlens_k;   // [B + 1] int32 on the device
  int packed_rows_k;         // N_k
  // Packed chunks into a cache (fmha_kvcache_varlen_fwd): varlen and kvcache both set.  q / O are packed [N, H, D] as
  // in varlen mode, with {s_b, T_b} = fmha_varlen_seq(cu_seqlens, b, Lq, N) and Lq = max_seqlen; k / v are the
  // [B, C, H_kv, D] caches of the KV-cache mode (Lk = C).  Query i < T_b of sequence b sees key j iff j < n_b and
  // j <= p_b + i, with p_b as above and n_b = min(p_b + T_b, kv_cap); the bias is [bias_batch * H, Lq, Lb] (row i for
  // query i) and the key mask [B, kpm_cols].  cu_seqlens_k is not read.  No dropout, lse null.
  // Paged caches (KV-cache mode, padded or packed; appended so that no earlier field moves): k / v are pools
  // [num_blocks, block_size, H_kv, D] named by block_table [B, blocks_per_seq] (see fmha_paged_block below), and
  // Lk = C = blocks_per_seq * block_size.  Every rule above holds with cache row j of sequence b read from row
  // j % block_size of its block j / block_size.  block_size is a multiple of 128, so each key tile of the forward lies
  // inside one block.  Null: the [B, C, H, D] caches above.
  const int* block_table;
  int block_size, blocks_per_seq, num_blocks;
};
void launch_fmha_fwd(const FmhaFwdParams& p, cudaStream_t stream);

// Paged key / value caches (fmha_kvcache_fwd, fmha_kvcache_varlen_fwd, fmha_decode and the cache append with a
// block_table): a pool [num_blocks, block_size, H_kv, D] holds the rows of every sequence in blocks of block_size
// rows (a multiple of 128), and block_table [B, M] (int32 on the device) names them: entry (b, i) is the block that
// holds rows i * block_size .. (i + 1) * block_size - 1 of sequence b, -1 none.  The per-sequence capacity is
// C = M * block_size, and with the rows so mapped every kernel computes what it computes on a [B, C, H_kv, D] cache:
// bitwise the result of the contiguous call on the cache gathered through the table.  An entry outside
// [0, num_blocks) never causes a write (the append skips that row); a read through it is clamped into the pool, so
// its value is unspecified but no table value reaches outside a tensor.  The block allocator (kv_blocks.cu) never
// hands out such entries.
#ifdef __CUDACC__
// the pool block of row `row` of sequence b, clamped into the pool (for reads)
__device__ __forceinline__ int fmha_paged_block(const int* block_table, int b, int row, int block_size, int m,
                                                int num_blocks) {
  const int blk = block_table[(long long)b * m + row / block_size];
  return blk < 0 ? 0 : (blk >= num_blocks ? num_blocks - 1 : blk);
}

// Varlen mode: {s_b, n_b} of sequence b (L = max_seqlen, N = packed rows), clamped as documented above, so that no
// value of cu_seqlens makes a kernel reach outside a tensor
__device__ __forceinline__ int2 fmha_varlen_seq(const int* cu_seqlens, int b, int L, int N) {
  const long long c0 = cu_seqlens[b], c1 = cu_seqlens[b + 1];
  const long long s = c0 < 0 ? 0 : (c0 > N ? N : c0);
  const long long cap = (long long)L < N - s ? (long long)L : N - s;
  const long long n = c1 - c0;
  return make_int2((int)s, (int)(n < 0 ? 0 : (n > cap ? cap : n)));
}
#endif

// Copies the T new rows of k_new / v_new [B, T, H, D] into rows p_b + i of the [B, C, H, D] caches, p_b =
// clamp(seqlens[b], 0, C), bitwise, with 16-byte vectors; rows at or past C are skipped.  H is the caches' head count
// (H_kv under grouped-query attention).  It runs as a launch of its own before the KV-cache forward, which reads those
// rows from every query tile of a (b, h).  Packed chunks (cu_seqlens set): k_new / v_new are [N, H, D] (batch strides
// 0), T is max_seqlen, and sequence b copies its T_b rows s_b + i, {s_b, T_b} = fmha_varlen_seq(cu_seqlens, b, T, N),
// into rows p_b + i.
struct KvCacheAppendParams {
  const void* k_new;       // [B, T, H, D] via strides (elements)
  const void* v_new;
  void* k_cache;           // [B, C, H, D] via strides
  void* v_cache;
  const int* seqlens;      // [B] int32 on the device
  long long kn_sb, kn_sl, kn_sh, vn_sb, vn_sl, vn_sh;
  long long kc_sb, kc_sl, kc_sh, vc_sb, vc_sl, vc_sh;
  int B, T, H, D, C;
  const int* cu_seqlens;   // [B + 1] int32 on the device, or null (padded [B, T, H, D] rows); appended so that no
  int packed_rows;         // earlier field moves.  packed_rows = N
  // Paged caches (appended so that no earlier field moves): k_cache / v_cache are pools [num_blocks, block_size, H,
  // D] (kc_sb / vc_sb the block strides) and row pos of sequence b goes to block block_table[b, pos / block_size],
  // row pos % block_size; C = blocks_per_seq * block_size.  A row whose entry is outside [0, num_blocks) is skipped.
  const int* block_table;  // [B, blocks_per_seq] int32 on the device, or null
  int block_size, blocks_per_seq, num_blocks;
};
void launch_kv_cache_append(const KvCacheAppendParams& p, cudaStream_t stream);

// Block allocator of paged caches (kv_blocks.cu).  One CTA each, no atomics: the sequences are walked in order with a
// block-wide scan, so the block ids handed out depend only on the inputs, and nothing is read on the host (both can be
// captured in a CUDA graph).  free_list [num_blocks] is a stack whose top is free_list[*free_count - 1]; *free_count
// is clamped to [0, num_blocks] on entry, lengths[b] to [0, C] with C = blocks_per_seq * block_size.
//  * reserve: every entry (b, i) with i < ceil(lengths[b] / block_size) and block_table[b, i] < 0 takes the next block
//    off the top of the stack, in the order (b, i) ascending.  When the stack runs out the entry stays -1 and
//    *overflow is set to 1 (it is never cleared here).
//  * release: every entry (b, i) with i >= ceil(lengths[b] / block_size) becomes -1; the ones in [0, num_blocks) are
//    pushed onto the stack in the order (b, i) ascending (a push past num_blocks, only possible for a table that names
//    a block twice, is dropped).
struct KvBlocksParams {
  int* block_table;        // [B, blocks_per_seq]
  int* free_list;          // [num_blocks]
  int* free_count;         // [1]
  int* overflow;           // [1] (reserve only)
  const int* lengths;      // [B]
  int B, blocks_per_seq, block_size, num_blocks;
};
void launch_kv_blocks_reserve(const KvBlocksParams& p, cudaStream_t stream);
void launch_kv_blocks_release(const KvBlocksParams& p, cudaStream_t stream);

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

// Decode attention (fmha_decode_sm90.cu): one query row per (b, h) against the first n_b rows of a [B, C, H, D] key /
// value cache, n_b = min(seqlens[b], C) (all C rows without seqlens), plus row seqlens[b] itself when k_new / v_new
// are given: that row is first written with k_new / v_new, bitwise.  n_b is also clamped to the columns of the bias
// and of the key mask, so no device value of seqlens reaches outside a tensor.
struct FmhaDecodeParams {
  const void* q;           // [B, 1, H, D] via strides (elements)
  const void* k_new;       // [B, 1, H, D] via strides, or null (no append)
  const void* v_new;
  void* k_cache;           // [B, C, H, D] via strides
  void* v_cache;
  const int* seqlens;      // [B] int32 on the device, or null (all C rows visible)
  const void* bias;        // [bias_batch, H, 1, bias_cols] via (batch, head) strides, contiguous rows; may be null
  const uint8_t* kpm;      // [B, kpm_cols] bool rows, nonzero = masked; may be null
  void* out;               // [B, 1, H, D] contiguous
  float* part_o;           // [B, H, num_splits, D] fp32 partials (num_splits > 1)
  float* part_ml;          // [B, H, num_splits, 2] (row max in log2 units, row sum)
  long long q_sb, q_sh, kn_sb, kn_sh, vn_sb, vn_sh;
  long long kc_sb, kc_sl, kc_sh, vc_sb, vc_sl, vc_sh;
  long long bias_sb, bias_sh, kpm_sb;
  int B, H, D, C;
  int bias_batch, bias_cols, kpm_cols;
  // split s takes keys [s * chunk, (s + 1) * chunk); the last one runs to n_b.  chunk == 0 derives it per (b, h) from
  // the device length: chunk_b = max(1, ceil(n_b / num_splits)), so that a host bound far above n_b (the capacity,
  // in a captured CUDA graph) still spreads the n_b keys over every split.  Both give the same ranges when n_b equals
  // the bound the host chunk was computed from.
  int num_splits, chunk;
  int is_bf16;
  float scale;
  // query head h reads cache head h / kv_group (grouped-query attention; the caches and k_new / v_new hold
  // H / kv_group heads); 1 = one cache head per query head
  int kv_group;
  // Paged caches (appended so that no earlier field moves): k_cache / v_cache are pools [num_blocks, block_size,
  // H_kv, D] (kc_sb / vc_sb the block strides), C = blocks_per_seq * block_size, and key j of sequence b is row
  // j % block_size of block block_table[b, j / block_size] (fmha_paged_block).  The new row is stored only when its
  // entry is in [0, num_blocks).  Null: [B, C, H, D] caches.
  const int* block_table;
  int block_size, blocks_per_seq, num_blocks;
};
constexpr int kDecodeCtasPerSm = 3;        // 72 KB of shared memory each
constexpr int kDecodeMinSplitKeys = 256;   // the split heuristic makes no shorter split
constexpr int kDecodeMaxSplits = 128;
// split count for B x H rows and at most len_bound visible keys (a host bound: the device lengths are never read)
int fmha_decode_num_splits(int B, int H, int len_bound, int num_sms);
void launch_fmha_decode(const FmhaDecodeParams& p, cudaStream_t stream);

}  // namespace ub
