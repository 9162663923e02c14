// Host-callable launchers of the unicore_b200 kernels (plain C++/CUDA-runtime types only, so the
// .cu translation units do not need the PyTorch headers and compile in seconds).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace ub {

// dtype tags shared by host and device code
enum DType : int { kF32 = 0, kF16 = 1, kBF16 = 2 };

constexpr int kMaxTensorsPerLaunch = 24;

// ---- multi-tensor L2 norm / scale -----------------------------------------------------------------
struct NormTensors {
  const void* ptr[kMaxTensorsPerLaunch];
  long long numel[kMaxTensorsPerLaunch];
  int dtype[kMaxTensorsPerLaunch];
  int count;
};
// acc: float[1] running sum of squares (zeroed by the caller before the first launch)
// partials: float[>= max_ctas] scratch, counter: unsigned[1] zeroed scratch
// out: float[1] receives sqrt(acc) when finalize != 0
void launch_l2norm(const NormTensors& t, float* acc, float* partials, unsigned* counter, float* out, int finalize,
                   cudaStream_t stream);
int l2norm_max_ctas();

struct ScaleTensors {
  void* ptr[kMaxTensorsPerLaunch];
  long long numel[kMaxTensorsPerLaunch];
  int dtype[kMaxTensorsPerLaunch];
  int count;
};
// x *= scale * (scale_dev ? *scale_dev : 1)
void launch_scale(const ScaleTensors& t, float scale, const float* scale_dev, cudaStream_t stream);

// ---- multi-tensor Adam ---------------------------------------------------------------------------------
struct AdamTensors {
  void* p[kMaxTensorsPerLaunch];       // fp32 master (or 16-bit param)
  void* g[kMaxTensorsPerLaunch];       // gradient
  float* m[kMaxTensorsPerLaunch];
  float* v[kMaxTensorsPerLaunch];
  void* p_half[kMaxTensorsPerLaunch];  // optional 16-bit copy of the updated param
  float* ema[kMaxTensorsPerLaunch];    // optional fp32 EMA buffer updated in the same pass
  long long numel[kMaxTensorsPerLaunch];
  int p_dtype[kMaxTensorsPerLaunch], g_dtype[kMaxTensorsPerLaunch], half_dtype[kMaxTensorsPerLaunch];
  float step_size[kMaxTensorsPerLaunch];   // lr * sqrt(1-b2^t)/(1-b1^t) (or lr)
  float decay_mul[kMaxTensorsPerLaunch];   // 1 - step_size * weight_decay
  float beta1[kMaxTensorsPerLaunch], beta2[kMaxTensorsPerLaunch], eps[kMaxTensorsPerLaunch];
  unsigned long long elem_base[kMaxTensorsPerLaunch];  // RNG stream offset of the tensor's first element
  int count;
};
struct AdamLaunch {
  float inv_scale;            // grads are multiplied by inv_scale / (*scale_dev if given)
  const float* scale_dev;     // optional device scalar divisor
  int zero_grad;              // clear g after reading it
  int stochastic_rounding;    // bf16 p_half written with stochastic rounding
  float ema_decay;
  unsigned long long seed, offset;  // philox key for stochastic rounding
};
void launch_adam(const AdamTensors& t, const AdamLaunch& cfg, cudaStream_t stream);

void launch_fp32_to_bf16_sr(const float* in, void* out, long long n, unsigned long long seed,
                            unsigned long long offset, cudaStream_t stream);
void launch_ema(float* ema, const float* p, long long n, float decay, cudaStream_t stream);

// ---- LayerNorm / RMSNorm -----------------------------------------------------------------------------------
// Launch plan of the norm kernels for a [rows, cols] input: which kernel generation and template case runs, on what
// grid, and how the rows are dealt out.  The launchers run exactly this plan.  Every kernel loops over tiles of
// `tile_rows` consecutive rows; tile t goes to unit t % units (a unit is a warp for v3, a CTA for v2 and v1), so a
// unit runs tiles_min or tiles_max tiles.  The generation changes only speed and summation order: the backward has
// one contract (outputs, fixed-order sums, scratch layout, finisher) at every width.
enum NormKind : int { kNormFwd = 0, kNormBwd = 1, kNormFusedFwd = 2 };  // the fused op's backward runs kNormBwd
struct NormPlan {
  int gen;          // 3: one warp per row, 2: bulk-copy input ring, 1: rows in registers; 0: no kernel for this width
  int nvec;         // 16-byte vectors per row
  int vpl, lpr, r;  // v3: vectors per lane, lanes per row; v3 and v2: rows per warp (v3) or row group (v2) and tile
  int tpr, groups;  // v2 and v1: threads per row, row groups per CTA
  int vpt;          // v1: vectors per thread
  int full;         // the row has no partial vector slot (v3: nvec == vpl * lpr, v2 / v1: every thread has all slots)
  int grid, threads, tile_rows;
  long long units, rows_per_sweep, tiles_min, tiles_max;
};
NormPlan norm_plan(int rows, int cols, int dtype, int kind);
void launch_layernorm_fwd(const void* x, const void* gamma, const void* beta, void* y, float* mean, float* rstd,
                          int rows, int cols, float eps, int dtype, cudaStream_t stream);
// part: float[3 * norm_bwd_parts(...) * cols] scratch (per-CTA partial column sums); dgamma/dbeta in `dtype`
int norm_bwd_parts(int rows, int cols, int dtype);
// Every backward sums its parameter gradients in a fixed order (bitwise reproducible in both modes of
// torch.use_deterministic_algorithms) and finishes them through colsum_finalize_kernel.
// accumulate (bit 0: dgamma, bit 1: dbeta, bit 2: dbias): add to what the output already holds (gradient arena)
void launch_layernorm_bwd(const void* dy, const void* x, const float* mean, const float* rstd, const void* gamma,
                          void* dx, void* dgamma, void* dbeta, float* part, int rows, int cols, int dtype,
                          cudaStream_t stream, int accumulate = 0);
void launch_rmsnorm_fwd(const void* x, const void* gamma, void* y, float* rstd, int rows, int cols, float eps,
                        int dtype, cudaStream_t stream);
void launch_rmsnorm_bwd(const void* dy, const void* x, const float* rstd, const void* gamma, void* dx, void* dgamma,
                        float* part, int rows, int cols, int dtype, cudaStream_t stream, int accumulate = 0);
// out[cols] (16-bit `dtype`) = column sums of the fp32 partial rows part[parts][cols] (parts == 0: zeros), in the
// summation order of the norm backward's parameter gradients; accumulate != 0 adds them to what out holds
void launch_colsum_finalize(const float* part, int parts, int cols, void* out, int accumulate, int dtype,
                            cudaStream_t stream);

// ---- softmax + dropout ---------------------------------------------------------------------------------------
// Launch plan of the softmax-dropout kernels (the launchers run exactly this plan).  `aligned`: every buffer of the
// call is 16-byte aligned.  Vector path: a row is owned by `tpr` threads holding `vpt` 16-byte vectors each; scalar
// path (vec == 0): one warp per row.  Both are grid-stride loops over rows, `sweeps` passes of the whole grid.
struct SoftmaxPlan {
  int vec, vpt, tpr, grid, threads;
  long long rows_per_sweep, sweeps;
};
SoftmaxPlan softmax_plan(long long rows, int K, int dtype, bool aligned, bool bwd);
// x: [rows, K] overwritten with softmax probabilities; out: dropout result (may alias x when p == 0)
// mask row = row / mask_div (mask_rows = rows / mask_div), bias row = row % bias_rows
void launch_softmax_dropout_fwd(void* x, void* out, const void* mask, const void* bias, long long rows, int K,
                                long long mask_div, long long bias_rows, float p, unsigned long long seed,
                                unsigned long long offset, int dtype, cudaStream_t stream, void* logits = nullptr,
                                float* lse = nullptr, void* probs = nullptr);
// (plain mode writes the probabilities backward needs into `probs`; nullptr = over x itself, the in-place contract)
// dx may alias dy.  Logits mode (lse != nullptr): `probs` holds the logits forward wrote; `addend` (nullable) is
// added to dx before the store.
void launch_softmax_dropout_bwd(const void* dy, void* dx, const void* probs, long long rows, int K, float p,
                                unsigned long long seed, unsigned long long offset, int dtype, cudaStream_t stream,
                                const float* lse = nullptr, const void* addend = nullptr);

// ---- fused element-wise ---------------------------------------------------------------------------------------
// Launch plan of bias_gelu fwd / bwd and column_sum (the launchers run exactly this plan): a grid of (col_blocks,
// slices) CTAs.  A thread owns one 16-byte column vector (nvec per row, 128 per column block: the last block is
// partial unless nvec % 128 == 0) in one of a CTA's two row lanes, and walks the rows of its (slice, lane) in groups
// of 4; one pass of every slice over its rows covers rows_per_sweep rows, `sweeps` passes cover all rows.  `fwd`:
// the plan of bias_gelu's forward, else the one of its backward and of column_sum.
struct ColumnPlan {
  int nvec, col_blocks, slices;
  long long rows_per_sweep, sweeps;
};
ColumnPlan bias_gelu_plan(long long rows, int cols, bool fwd);
void launch_bias_gelu_fwd(const void* x, const void* bias, void* y, long long rows, int cols, int dtype,
                          cudaStream_t stream);
// dbias (nullable) = column sums of dx; part = float[bias_gelu_parts(rows, cols) * cols] scratch
int bias_gelu_parts(long long rows, int cols);
// out[cols] (16-bit) = column sums of x[rows, cols] (cols % 8 == 0), fp32 accumulation; same scratch size
void launch_column_sum(const void* x, void* out, float* part, long long rows, int cols, int dtype, cudaStream_t stream,
                       int accumulate = 0);
void launch_bias_gelu_bwd(const void* dy, const void* x, const void* bias, void* dx, void* dbias, float* part,
                          long long rows, int cols, int dtype, cudaStream_t stream, int accumulate = 0);
// y = LN(residual + dropout(x + bias)); summed = residual + dropout(x + bias) (saved for backward)
void launch_bias_dropout_add_ln_fwd(const void* x, const void* bias, const void* residual, const void* gamma,
                                    const void* beta, void* y, void* summed, float* mean, float* rstd, int rows,
                                    int cols, float p, float eps, unsigned long long seed, unsigned long long offset,
                                    int dtype, cudaStream_t stream);
// dsum = dLN(dy); dx = dropout_mask * dsum / P(keep); dbias (nullable) = column sums of dx at every width: v3 / v2 sum
// the fp32 values in the same pass, v1 sums the rounded dx with launch_column_sum afterwards (two more launches)
void launch_bias_dropout_add_ln_bwd(const void* dy, const void* summed, const float* mean, const float* rstd,
                                    const void* gamma, void* dsum, void* dx, void* dgamma, void* dbeta,
                                    void* dbias, float* part, int rows, int cols, float p, unsigned long long seed,
                                    unsigned long long offset, int dtype, cudaStream_t stream, int accumulate = 0);
// ---- Gaussian radial basis of (mul[edge] * d + bias[edge]) (Uni-Mol pair features), csrc/fused/gaussian.cu ----------
// y: [n, K] in `dtype` (fp16 / bf16), K a multiple of 8 with K / 8 a power of two <= 32

// Launch plan of a grid-stride kernel: `grid` CTAs take `items_per_sweep` of its `items` work items per pass over the
// grid, `sweeps` passes cover them all (the last one ragged unless items % items_per_sweep == 0).
struct SweepPlan {
  int grid;
  long long items, items_per_sweep, sweeps;
};

// token-major [B, L, T, H, D] <-> T head-major [B, H, L, D] tensors (null head pointer = zeros when gathering);
// slice 0 is multiplied by scale0 in either direction.  D * sizeof(elem) must be a multiple of 16.
// The launcher runs head_permute_plan: an item is one 16-byte vector of one of a pair of neighbouring tokens (an odd
// L leaves the second token of the last pair idle), 256 threads per CTA, at most 16 CTAs per SM.
SweepPlan head_permute_plan(int B, int L, int T, int H, int D, int dtype);
void launch_head_permute(void* token_major, void* const* head_major, int B, int L, int T, int H, int D, float scale0,
                         bool to_heads, int dtype, cudaStream_t stream);

// Rotary position embeddings (rotate-half form), csrc/fused/rotary.cu.  x [B, L, N, D] 16-bit with a contiguous last dim,
// head stride D and token / batch strides sl / sb (elements); out a new contiguous [B, L, N, D].  Heads 0 .. rotated_heads-1
// are rotated on their first rd columns at positions l + offsets[b] (offsets: nullable int32 [B], read on the device),
// everything else is copied bitwise; `inverse` rotates by -theta (the backward).  2 <= rd <= min(D, 512), rd even.
// The launcher runs rotary_plan: an item is a tile of tile_tokens tokens, 256 threads per CTA, at most 8 CTAs per SM,
// `smem` bytes of dynamic shared memory (the tile's cos / sin).  vec: the 16-byte path (8 pairs per thread), taken when
// `aligned` (x 16-byte aligned, sb and sl multiples of 8) and rd / 2 and D are multiples of 8; else one pair per thread.
struct RotaryPlan {
  SweepPlan sweep;
  bool vec;
  int tile_tokens, smem;
};
RotaryPlan rotary_plan(int B, int L, int N, int D, int rd, int dtype, bool aligned);
void launch_rotary(const void* x, void* out, const float* inv_freq, const int* offsets, long long sb, long long sl,
                   int B, int L, int N, int D, int rd, int rotated_heads, bool aligned, bool inverse, int dtype,
                   cudaStream_t stream);

// head-major [B, H, M] <-> pair-major [B, M, H] for 16-bit elements (H % 8 == 0, M % 8 == 0)
// The transpose and both tail kernels run pair_plan: an item is one 8 x 8 tile (8 heads x 8 pair rows), 256 threads
// per CTA, at most 8 CTAs per SM.
SweepPlan pair_plan(int B, int H, long long M);
void launch_pair_transpose(const void* in, void* out, int B, int H, long long M, bool to_pair, cudaStream_t stream);
// encoder tail of pair-bias models: pair = T(z) with -inf -> 0, delta = T(z - z0) with padded keys -> 0 (Lk % 8 == 0)
void launch_pair_tail_fwd(const void* z, const void* z0, const unsigned char* key_pad, void* pair, void* delta, int B,
                          int H, int Lq, int Lk, int dtype, cudaStream_t stream);
void launch_pair_tail_bwd(const void* d_pair, const void* d_delta, const void* z, const unsigned char* key_pad, void* dz,
                          void* dz0, int B, int H, int Lq, int Lk, int dtype, cudaStream_t stream);

// Launch plan of the embedding-gradient kernels (at most 16 CTAs per SM each): the scatter runs a warp per row of dy
// and the finalize a warp per vocabulary row (8 per CTA); the sorted kernel runs a CTA per vocabulary row (grid 0:
// the launcher launches nothing).
struct EmbeddingPlan {
  SweepPlan scatter, finalize, sorted;
};
EmbeddingPlan embedding_plan(long long rows, long long vocab);
// Embedding gradient without a sort: grad[token[r], :] (+)= dy[r, :], fp32 accumulation in `scratch` [vocab, cols]
// (persistent, all zero between calls) with `touched` [vocab] row flags; rows equal to padding_idx contribute nothing.
// accumulate != 0: add to grad (the optimizer's arena view); else touched rows are overwritten (grad pre-zeroed).
void launch_embedding_bwd(const void* dy, const long long* tokens, float* scratch, unsigned char* touched, void* grad,
                          long long rows, int cols, long long vocab, long long padding_idx, int accumulate, int dtype,
                          cudaStream_t stream);
// The same gradient in a fixed summation order (deterministic mode): `sorted` [rows] are the token ids stable-sorted
// ascending and `perm` [rows] their original row indices; vocabulary row v sums dy over its run in ascending row order
// in fp32 from 0, then adds the 16-bit grad (accumulate) and rounds once.  Padding and out-of-range ids are skipped.
void launch_embedding_bwd_sorted(const void* dy, const long long* sorted, const long long* perm, void* grad,
                                 long long rows, int cols, long long vocab, long long padding_idx, int accumulate,
                                 int dtype, cudaStream_t stream);

void launch_gbf_fwd(const void* d, const long long* edge, const void* mul_w, const void* bias_w, const void* means,
                    const void* stds, void* y, long long n, int K, int dtype, cudaStream_t stream);
// Launch plan of the Gaussian-basis kernels: `grid` CTAs of 256 threads, a row of K outputs per kvec = K / 8 threads
// (rows_per_cta rows per CTA), grid-stride over the rows in `sweeps` passes of rows_per_sweep rows.  The backward's
// shared memory (histogram of E edge types + 2K column sums) is `smem` bytes, above 48 KB it needs the opt-in.
struct GbfPlan {
  int grid, kvec, rows_per_cta;
  long long rows_per_sweep, sweeps;
  int smem;
};
GbfPlan gbf_plan(long long n, int K, int E);
// part: float[gbf_parts(n, K)][2 * K] per-CTA partial (d mean, d std); hist: float[2 * E] zero-initialised (d mul, d bias)
int gbf_parts(long long n, int K);
void launch_gbf_bwd(const void* dy, const void* d, const long long* edge, const void* mul_w, const void* bias_w,
                    const void* means, const void* stds, float* part, float* hist, long long n, int K, int E, int dtype,
                    cudaStream_t stream);
// The same gradients in a fixed summation order (deterministic mode): rowg float[n][2] scratch; sorted / perm: the
// edge types stable-sorted and their row indices; d mul / d bias of a type sum its rows in ascending order
void launch_gbf_bwd_det(const void* dy, const void* d, const long long* edge, const void* mul_w, const void* bias_w,
                        const void* means, const void* stds, float* part, float* rowg, const long long* sorted,
                        const long long* perm, float* hist, long long n, int K, int E, int dtype, cudaStream_t stream);
// loss_rows[i] = lse_i - logit_i[target_i] (0 when target == ignore_index); lse saved for backward
void launch_softmax_xent_fwd(const void* logits, const long long* target, float* loss_rows, float* lse, int rows,
                             int cols, int stride, long long ignore_index, int dtype, cudaStream_t stream);
// dlogits = (softmax - onehot) * dloss (0 for ignored rows), written in `dtype`
void launch_softmax_xent_bwd(const void* logits, const long long* target, const float* lse, const float* dloss,
                             void* dlogits, int rows, int cols, int stride, long long ignore_index, int dtype,
                             cudaStream_t stream);

}  // namespace ub
