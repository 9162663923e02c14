// Fused multi-head attention forward for sm_90a (head_dim D % 8 == 0, 8 <= D <= 128, fp16/bf16):
//   O = dropout(softmax(scale * Q K^T + bias + key_padding)) V        LSE = logsumexp of the logits
// One kernel for what the reference runs as bmm -> masked_fill -> softmax_dropout -> bmm plus four transposes
// (unicore/modules/multihead_attention.py:47-113, csrc/softmax_dropout/softmax_fast.h:207-434).
//
// The kernel is a template on the padded head width DP (64 or 128 columns = one or two 128-byte-swizzled boxes per
// row); the head dim D is a runtime value.  The TMA maps span D columns, so the unit zero-fills columns D..DP-1 in
// shared memory: zero columns of Q and K add nothing to S, zero columns of V give zero columns of O, which the
// epilogue does not store.
// One CTA = one warpgroup (128 threads) = one 64-row query tile of one (batch, head); it walks the key tiles
// (kBlockN = 128 keys at DP = 64, 64 keys at DP = 128, which keeps o[64] + s[32] in registers):
//   1. TMA (128-byte-swizzled boxes, csrc/attn/tma_map.h): K, V and the bias tile of key tile j+1 are requested into
//      the other of two stages while tile j is computed; one thread issues every copy, completion on an mbarrier.
//   2. S = Q K_j^T           DP/16 x wgmma m64n{kBlockN}k16, both operands K-major from shared memory, fp32 in registers
//   3. softmax in registers: logits = S*scale + bias + key mask, row max across the 4 threads of a quad, online
//      rescaling of O and of the row sum, Philox dropout on packed 16-bit pairs (the keep bits are stored for the
//      backward pass), P converted in place into the register A operand of the next product.  Each Philox call is
//      made by one thread of the quad that needs its words, and a 4 x 4 word transpose in the quad (quad_transpose4)
//      distributes them.
//   4. O += P V_j            kBlockN/16 x wgmma m64n{DP}k16, A (P) from registers, V presented MN-major from its
//                            row-major bytes (at DP = 128 the descriptor steps to the second box through its LBO)
//   q/k/v are read through strides straight out of the packed in_proj output; O is written as [B, Lq, H, D] so
//   that out_proj consumes it without a transpose.  Grouped-query attention: the K / V maps span H / kv_group heads
//   and the CTA of query head h loads head h / kv_group; its arithmetic is that of the same call on expanded K / V.
// 106 KB (DP = 64) / 98 KB (DP = 128) of shared memory and <= 255 registers per thread: two CTAs (8 warps) per SM,
// so one CTA's softmax overlaps the other's tensor-core work and copies.
// Logits mode (template flag kLogits, p.logits set) also writes z = S*scale + bias + key mask as [B, H, Lq, Lk]: the
// 16-bit logits go back over the bias tile in shared memory and leave by TMA store while P V runs (same shared memory).
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <math_constants.h>

#include "../common.cuh"
#include "fmha_api.h"
#include "wgmma.cuh"

namespace ub {
namespace {

using namespace tc;

constexpr int kBlockM = 64;    // query rows per CTA
constexpr int kFwdThreads = 128;

// Tile geometry and shared memory map of the padded head width DP; every box is 128-byte-swizzled rows of 64 columns
template <int DP>
struct FwdCfg {
  static constexpr int kBlockN = DP == 64 ? 128 : 64;            // keys per tile
  static constexpr int kBoxes = DP / 64;                         // 64-column boxes per row
  static constexpr uint32_t kQBox = kBlockM * 128;               // one 64-column box of the Q tile
  static constexpr uint32_t kKVBox = kBlockN * 128;              // one 64-column box of a K / V tile
  static constexpr uint32_t kKVStage = kBoxes * kKVBox;
  static constexpr uint32_t kBiasStage = kBlockM * kBlockN * 2;  // kBlockN / 64 boxes of 64 rows x 64 keys
  static constexpr uint32_t kSmemQ = 0;
  static constexpr uint32_t kSmemK = kSmemQ + kBoxes * kQBox;    // 2 stages
  static constexpr uint32_t kSmemV = kSmemK + 2 * kKVStage;      // 2 stages
  static constexpr uint32_t kSmemBias = kSmemV + 2 * kKVStage;   // 2 stages
  static constexpr uint32_t kSmemKAdd = kSmemBias + 2 * kBiasStage;   // 2 stages x float[kBlockN]: 0 or -inf per key
  static constexpr uint32_t kSmemBar = kSmemKAdd + 2 * kBlockN * 4;
  static constexpr uint32_t kSmemBytes = kSmemBar + 64 + 1024;   // + alignment slack of the 1024-byte-aligned base
};
static_assert(FwdCfg<64>::kSmemBytes == 108608, "DP = 64 keeps the shared memory map of the 64-only kernel");

// w[j] <- w[j ^ x] for x in 0..3 (per-thread), as two conditional swaps: 8 selects, no runtime-indexed array
UB_DEVICE void xor_permute4(uint32_t (&w)[4], int x) {
  const bool s1 = (x & 1) != 0, s2 = (x & 2) != 0;
  uint32_t a0 = s1 ? w[1] : w[0], a1 = s1 ? w[0] : w[1], a2 = s1 ? w[3] : w[2], a3 = s1 ? w[2] : w[3];
  w[0] = s2 ? a2 : a0;
  w[1] = s2 ? a3 : a1;
  w[2] = s2 ? a0 : a2;
  w[3] = s2 ? a1 : a3;
}

// 4 x 4 word transpose inside a quad: thread c holds the four words of Philox call c and leaves with word c of calls
// 0..3 (w[k] = word c of call k).  After the first permutation w[m] is the word that partner c ^ m needs, so each of the
// three shuffles sends a fixed register; the received w[m] is word c of call c ^ m, and the second permutation puts
// it in place.
UB_DEVICE void quad_transpose4(uint32_t (&w)[4], int c) {
  xor_permute4(w, c);
  w[1] = __shfl_xor_sync(0xffffffffu, w[1], 1);
  w[2] = __shfl_xor_sync(0xffffffffu, w[2], 2);
  w[3] = __shfl_xor_sync(0xffffffffu, w[3], 3);
  xor_permute4(w, c);
}

// kLogits: also write z = scale * Q K^T + bias + key mask (fmha_api.h).  Each thread writes its 16-bit logits back over
// the bias elements it has just read from the swizzled bias stage (no other thread touches them; the region exists
// without a bias too), and one thread stores the tile with a TMA store, clipped at Lq / Lk.  The stage is refilled
// by the prefetch of tile j + 2, so that prefetch first waits until the store has read shared memory.
// kCausal: key j is visible to row i iff j <= i.  The tile loop (and with it the prefetch of tile j + 1) stops at the
// last key tile with key0 <= q0 + 63; the 64 keys q0 .. q0 + 63 of the diagonal lie in that one tile (q0 is a multiple
// of 64, kBlockN of 64), so only there do some elements get -inf, by index, in registers.  The skipped tiles would
// have added exact zeros (alpha = ex2(0) = 1, l += 0, P = +0), so O, LSE and the keep words written are bitwise those
// of the plain kernel given bias + the future mask.  The CTAs take the query tiles longest first.
// kKVCache: a chunk of T queries against a [B, C, H, D] cache (fmha_api.h): query i of sequence b sees key j iff
// j < n_b and j <= p_b + i.  p_b is read from the device and is not tile-aligned, so the tile loop (and the prefetch)
// stops at the tile holding key min(n_b, p_b + q0 + 64) - 1, and every tile that reaches past key p_b + q0 (the band
// may span two) sets the invisible elements to -inf by index.  Cache rows at or past n_b lie inside the tensor, so TMA
// loads them and they may hold anything, NaN included: their scores are replaced (never added to), and their V rows
// are zeroed in shared memory before P V (0 x NaN is NaN).  Only the last tile walked can hold such rows.  No dropout.
// kVarlen: packed sequences (fmha_api.h).  The CTA of (query tile, h, b) reads query rows s_q + q0 .. of the packed q
// and key rows s_k + j * kBlockN .. of the packed k / v through B = 1 maps, and exits when q0 >= n_q.  Its tile loop
// (and the prefetch) stops at the tile holding key n_k - 1; the padded call would walk the later tiles as wholly masked
// ones, which add exact zeros (see kCausal), so O, LSE and the keep words at rows below n_q are bitwise those of that
// call.  In the last tile the keys at or past n_k (rows of the next sequence, or TMA zero fill past N_k) get -inf by
// assignment and their V rows are zeroed, as in the KV-cache mode.  A sequence with n_k = 0 walks tile 0 wholly masked
// (Q arrives with the first tile), so its rows get O = 0 and LSE = -inf.  Only rows below n_q are stored.  Causal
// composes (its diagonal is per sequence, with the keys the queries' own rows); logits mode does not.
// kKVCache && kVarlen: packed chunks into a cache (fmha_api.h).  Queries and O are packed as in varlen mode (rows s_b +
// i, CTAs past n_q exit, only rows below n_q are stored); keys and values come from the caches at batch coordinate b,
// and the visibility, tile count, stale-row handling and tile order are the KV-cache mode's with T_b = n_q in place of
// Lq.  The varlen key description (cu_seqlens_k) is not read.
// kPaged (with kKVCache, padded or packed): k / v are pools [num_blocks, block_size, H_kv, D] (fmha_api.h).  Key tile
// j lies inside one block (block_size is a multiple of kBlockN), so load_tile takes the batch coordinate of its K / V
// boxes from the block table and the row from j * kBlockN % block_size; the tiles, their order and the arithmetic are
// the contiguous call's.
template <typename T, int DP, bool kLogits, bool kCausal, bool kKVCache, bool kVarlen = false, bool kPaged = false>
__global__ void __launch_bounds__(kFwdThreads, 2) fmha_fwd_kernel(const __grid_constant__ FmhaFwdParams p) {
  static_assert(!(kLogits && kCausal), "causal attention is not instantiated in logits mode");
  static_assert(!(kKVCache && (kLogits || kCausal)), "the KV-cache mode is neither causal nor logits mode");
  static_assert(!(kVarlen && kLogits), "the varlen mode is not logits mode");
  static_assert(!kPaged || kKVCache, "paged caches are a KV-cache mode");
  using C = FwdCfg<DP>;
  constexpr int kBlockN = C::kBlockN;
  constexpr int kWords = kBlockN / 32;   // keep-bit words per row of a key tile
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_base = smem_u32(smem_raw);
  const uint32_t smem_base = (raw_base + 1023u) & ~1023u;   // 128-byte swizzle: tiles must be 1024-byte aligned
  uint8_t* smem = smem_raw + (smem_base - raw_base);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, c = lane & 3;
  const int q_tile = (kCausal || kKVCache) ? (int)(gridDim.x - 1 - blockIdx.x) : (int)blockIdx.x;
  const int q0 = q_tile * kBlockM, h = blockIdx.y, b = blockIdx.z;
  const int hk = h / p.kv_group;   // key / value head of query head h (fmha_api.h)
  // varlen: the sequence's first packed query row and query count, and its first packed key row and key count; its
  // rows are addressed as batch 0 of the B = 1 maps
  int vl_s = 0, vl_n = 0, vk_s = 0, vk_n = 0;
  if constexpr (kVarlen) {
    const int2 sn = fmha_varlen_seq(p.cu_seqlens, b, p.Lq, p.packed_rows);
    vl_s = sn.x;
    vl_n = sn.y;
    if (q0 >= vl_n) return;
    if constexpr (!kKVCache) {
      const int2 sk = fmha_varlen_seq(p.cu_seqlens_k, b, p.Lk, p.packed_rows_k);
      vk_s = sk.x;
      vk_n = sk.y;
    }
  }
  const int tb = kVarlen ? 0 : b;   // batch coordinate of the q map
  const int tbk = (kVarlen && !kKVCache) ? 0 : b;   // and of the k / v maps (a cache keeps the padded layout)
  const int row_lim = kVarlen ? vl_n : p.Lq;   // rows stored
  const uint32_t bar0 = smem_base + C::kSmemBar;   // bar0 + 8 * stage: K / V / bias of a key tile (+ Q on the first)
  float* kadd = reinterpret_cast<float*>(smem + C::kSmemKAdd);

  const bool has_bias = p.bias != nullptr;
  const int n_key_tiles = (p.Lk + kBlockN - 1) / kBlockN;
  // KV-cache mode: kv_p = p_b, kv_n = n_b, and kv_lim = the first key that some row of this query tile does not see
  int kv_p = 0, kv_n = 0, kv_lim = 0;
  if constexpr (kKVCache) {
    kv_p = p.seqlens != nullptr ? min(max(p.seqlens[b], 0), p.Lk) : p.Lk;
    kv_n = min(kv_p + (kVarlen ? vl_n : p.Lq), p.kv_cap);
    kv_lim = min(kv_n, kv_p + q0 + 1);
  }
  // causal: key tiles 0 .. (q0 + 63) / kBlockN hold a key visible to one of the rows q0 .. q0 + 63.  varlen: a
  // sequence without keys still walks one wholly masked tile, which loads Q and gives O = 0, LSE = -inf
  const int n_key_walk = kVarlen ? max(1, (vk_n + kBlockN - 1) / kBlockN) : n_key_tiles;
  const int n_tiles = kCausal ? min(n_key_walk, (q0 + kBlockM - 1) / kBlockN + 1)
                      : kKVCache ? max(1, (min(kv_n, kv_p + q0 + kBlockM) + kBlockN - 1) / kBlockN)
                                 : n_key_walk;
  const int bias_nb = (p.bias_batch > 1 ? b : 0) * p.H + h;
  // the TMA unit counts the zero-filled columns D..DP-1 of a box as transferred bytes
  constexpr uint32_t kKVBytes = C::kKVStage, kBiasBytes = C::kBiasStage, kQBytes = C::kBoxes * C::kQBox;
  // paged: the pool block of key tile j.  Thread 0 loads the block of tile j + 2 right after requesting tile j + 1, so
  // the table load's latency passes during tile j's math instead of delaying the next request (and the warpgroup)
  auto tile_block = [&](int j) {
    return fmha_paged_block(p.block_table, b, j * kBlockN, p.block_size, p.blocks_per_seq, p.num_blocks);
  };
  int next_block = 0;
  auto load_tile = [&](int j) {   // one thread; the first tile's phase also covers Q (one arrival per phase)
    const uint32_t st = (uint32_t)(j & 1), bar = bar0 + 8u * st;
    mbar_expect_tx(bar, 2 * kKVBytes + (has_bias ? kBiasBytes : 0u) + (j == 0 ? kQBytes : 0u));
    int kv_row = vk_s + j * kBlockN, kv_b = tbk;   // paged: the tile's block and its row inside it
    if constexpr (kPaged) {
      kv_b = j == 0 ? tile_block(0) : next_block;
      kv_row = j * kBlockN % p.block_size;
      if (j + 1 < n_tiles) next_block = tile_block(j + 1);
    }
#pragma unroll
    for (int x = 0; x < C::kBoxes; ++x) {   // column boxes 0..63 and 64..127
      if (j == 0) tma_load_4d(smem_base + C::kSmemQ + x * C::kQBox, &p.sw_q, 64 * x, h, vl_s + q0, tb, bar);
      tma_load_4d(smem_base + C::kSmemK + st * C::kKVStage + x * C::kKVBox, &p.sw_k, 64 * x, hk, kv_row, kv_b, bar);
      tma_load_4d(smem_base + C::kSmemV + st * C::kKVStage + x * C::kKVBox, &p.sw_v, 64 * x, hk, kv_row, kv_b, bar);
    }
    if (has_bias) {   // 64 rows x kBlockN keys = kBlockN / 64 boxes of 64 keys
#pragma unroll
      for (int x = 0; x < kBlockN / 64; ++x)
        tma_load_3d(smem_base + C::kSmemBias + st * C::kBiasStage + x * 8192, &p.sw_bias, j * kBlockN + 64 * x, q0, bias_nb,
                    bar);
    }
  };
  if (tid == 0) {
    mbar_init(bar0, 1);
    mbar_init(bar0 + 8, 1);
    fence_mbarrier_init();
    load_tile(0);
  }

  const int rl0 = warp * 16 + g, rl1 = rl0 + 8;   // my two rows of the tile
  const int row0 = q0 + rl0, row1 = q0 + rl1;
  const uint8_t* kpm_row = p.kpm != nullptr ? p.kpm + (long long)b * (kKVCache ? p.kpm_cols : p.Lk) : nullptr;
  const bool drop = !kKVCache && p.p_drop > 0.f;
  const uint32_t t14 = dropout_thresh14(p.p_drop);
  const uint32_t t14x2 = t14 | (t14 << 16);
  // the 1/(1-p) of the kept probabilities is applied once, to the normalised output row
  const float keep_scale = drop ? dropout_keep_scale14(t14) : 1.f;
  const unsigned long long bh = (unsigned long long)b * p.H + h;
  const unsigned long long lin0 = bh * p.Lq + (row0 < row_lim ? row0 : 0), lin1 = bh * p.Lq + (row1 < row_lim ? row1 : 0);
  const int words_per_row = (p.Lk + 31) / 32;
  // Philox counter of element (lin, key) is (lin * Lk + key) >> 3, one call per (row, 8 keys).  For each pair of 8-key
  // groups (i, i + 1) the quad needs four calls - rows rl0 / rl1 x groups i / i + 1 - and thread c computes call c:
  // row rl0 for even c, rl1 for odd c, group i + (c >> 1).  ctr_c is that call's (lin * Lk + key) at group pair 0 of
  // tile 0; a tile adds kBlockN, a group pair 16.
  const unsigned long long ctr_c = ((c & 1) ? lin1 : lin0) * p.Lk + 8 * (c >> 1);

  constexpr float kLog2e = 1.4426950408889634f;
  float m0 = -CUDART_INF_F, m1 = -CUDART_INF_F, l0 = 0.f, l1 = 0.f;   // running max (in use) and partial row sums
  float o[DP / 2];
#pragma unroll
  for (int i = 0; i < DP / 2; ++i) o[i] = 0.f;

  for (int j = 0; j < n_tiles; ++j) {
    const uint32_t st = (uint32_t)(j & 1);
    const int key0 = j * kBlockN;
    bool masked = false;
    if (tid < kBlockN) {
      const int key = key0 + tid;
      // KV-cache mode: kpm_cols >= kv_cap >= kv_n, so the key mask is read only below kv_n
      masked = key >= (kKVCache ? kv_n : kVarlen ? vk_n : p.Lk) || (kpm_row != nullptr && kpm_row[key] != 0);
      kadd[st * kBlockN + tid] = masked ? -CUDART_INF_F : 0.f;
    }
    // barrier: every thread is done with tile j-1, so its stage may be refilled with tile j+1
    const bool tile_masked = __syncthreads_or(masked) != 0;
    if (kLogits && tid == 0) bulk_wait_read();   // the logits store of tile j-1 has read the stage tile j+1 fills
    if (tid == 0 && j + 1 < n_tiles) load_tile(j + 1);
    mbar_wait(bar0 + 8u * st, (uint32_t)((j >> 1) & 1));
    if constexpr (kKVCache || kVarlen) {
      const int v_lim = kKVCache ? kv_n : vk_n;
      if (key0 + kBlockN > v_lim) {   // zero the V rows at or past n_b: whole 128-byte rows of every column box
        const int r0 = max(v_lim - key0, 0), chunks = (kBlockN - r0) * 8;
        uint8_t* sv = smem + C::kSmemV + st * C::kKVStage;
        for (int x = tid; x < C::kBoxes * chunks; x += kFwdThreads) {
          const int box = x / chunks, r = r0 + (x % chunks) / 8;
          *reinterpret_cast<uint4*>(sv + box * C::kKVBox + r * 128 + (x % 8) * 16) = make_uint4(0u, 0u, 0u, 0u);
        }
        fence_proxy_async_smem();   // the generic-proxy stores, before wgmma reads V
        __syncthreads();
      }
    }

    // ---- S = Q K^T --------------------------------------------------------------------------------------
    float s[kBlockN / 2];
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < DP / 16; ++kk) {   // k-step kk: box kk / 4, +32 bytes per step inside the box
      const uint64_t da = make_desc_sw128(smem_base + C::kSmemQ + (kk >> 2) * C::kQBox + (kk & 3) * 32);
      const uint64_t db = make_desc_sw128(smem_base + C::kSmemK + st * C::kKVStage + (kk >> 2) * C::kKVBox + (kk & 3) * 32);
      if constexpr (kBlockN == 128) wgmma_m64n128_ss<T, 0>(s, da, db, kk > 0 ? 1u : 0u);
      else wgmma_m64n64_ss<T, 0>(s, da, db, kk > 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    fence_operands(s);

    // ---- logits, row max ----------------------------------------------------------------------------------
    float mx0 = -CUDART_INF_F, mx1 = -CUDART_INF_F;
    uint8_t* bias_tile = smem + C::kSmemBias + st * C::kBiasStage;
#pragma unroll
    for (int i = 0; i < kBlockN / 8; ++i) {
      const int col = 8 * i + 2 * c;
      float2 b0 = make_float2(0.f, 0.f), b1 = make_float2(0.f, 0.f);
      if (has_bias) {
        const uint8_t* box = bias_tile + (i >> 3) * 8192 + c * 4;
        b0 = unpack2<T>(*reinterpret_cast<const uint32_t*>(box + sw128_off(rl0, i & 7)));
        b1 = unpack2<T>(*reinterpret_cast<const uint32_t*>(box + sw128_off(rl1, i & 7)));
      }
      if (tile_masked) {
        const float2 ka = *reinterpret_cast<const float2*>(kadd + st * kBlockN + col);
        b0.x += ka.x; b0.y += ka.y; b1.x += ka.x; b1.y += ka.y;
      }
      s[4 * i + 0] = fmaf(s[4 * i + 0], p.scale, b0.x);
      s[4 * i + 1] = fmaf(s[4 * i + 1], p.scale, b0.y);
      s[4 * i + 2] = fmaf(s[4 * i + 2], p.scale, b1.x);
      s[4 * i + 3] = fmaf(s[4 * i + 3], p.scale, b1.y);
      if constexpr (kCausal) {   // the diagonal tile: keys past the row are -inf, as the future mask would make them
        if (j == n_tiles - 1) {
          const int key = key0 + col;
          if (key > row0) s[4 * i + 0] = -CUDART_INF_F;
          if (key + 1 > row0) s[4 * i + 1] = -CUDART_INF_F;
          if (key > row1) s[4 * i + 2] = -CUDART_INF_F;
          if (key + 1 > row1) s[4 * i + 3] = -CUDART_INF_F;
        }
      }
      if constexpr (kKVCache) {   // assigned, not added: a stale score may be NaN
        if (key0 + kBlockN > kv_lim) {
          const int key = key0 + col;
          const int lim0 = min(kv_n, kv_p + row0 + 1), lim1 = min(kv_n, kv_p + row1 + 1);
          if (key >= lim0) s[4 * i + 0] = -CUDART_INF_F;
          if (key + 1 >= lim0) s[4 * i + 1] = -CUDART_INF_F;
          if (key >= lim1) s[4 * i + 2] = -CUDART_INF_F;
          if (key + 1 >= lim1) s[4 * i + 3] = -CUDART_INF_F;
        }
      }
      // the last tile: keys of the next sequence, assigned (their bias is not this one's).  Not with a cache, whose
      // stale rows the KV-cache branch above has hidden (vk_n is 0 there)
      if constexpr (kVarlen && !kKVCache) {
        if (key0 + kBlockN > vk_n) {
          const int key = key0 + col;
          if (key >= vk_n) s[4 * i + 0] = s[4 * i + 2] = -CUDART_INF_F;
          if (key + 1 >= vk_n) s[4 * i + 1] = s[4 * i + 3] = -CUDART_INF_F;
        }
      }
      if constexpr (kLogits) {   // the same swizzled positions as the bias elements above
        uint8_t* box = bias_tile + (i >> 3) * 8192 + c * 4;
        *reinterpret_cast<uint32_t*>(box + sw128_off(rl0, i & 7)) = pack2<T>(s[4 * i + 0], s[4 * i + 1]);
        *reinterpret_cast<uint32_t*>(box + sw128_off(rl1, i & 7)) = pack2<T>(s[4 * i + 2], s[4 * i + 3]);
      }
      mx0 = fmaxf(mx0, fmaxf(s[4 * i + 0], s[4 * i + 1]));
      mx1 = fmaxf(mx1, fmaxf(s[4 * i + 2], s[4 * i + 3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float mn0 = fmaxf(m0, mx0), mn1 = fmaxf(m1, mx1);
    // exponent offset: the running max, or 0 while every key seen so far is masked (the max itself stays -inf, so the
    // first tile with a finite logit rescales from it and the offset follows that row's real maximum)
    const float mu0 = mn0 == -CUDART_INF_F ? 0.f : mn0, mu1 = mn1 == -CUDART_INF_F ? 0.f : mn1;
    const float alpha0 = ex2_approx((m0 - mu0) * kLog2e), alpha1 = ex2_approx((m1 - mu1) * kLog2e);   // m = -inf -> 0
    m0 = mn0;
    m1 = mn1;
    l0 *= alpha0;
    l1 *= alpha1;
#pragma unroll
    for (int i = 0; i < DP / 8; ++i) {
      o[4 * i + 0] *= alpha0;
      o[4 * i + 1] *= alpha0;
      o[4 * i + 2] *= alpha1;
      o[4 * i + 3] *= alpha1;
    }

    // ---- probabilities, dropout, P -> register A operand ---------------------------------------------------------
    const float nm0 = -mu0 * kLog2e, nm1 = -mu1 * kLog2e;
    uint32_t pa[kBlockN / 4];        // pa[2i] = row rl0, keys 8i + 2c, +1; pa[2i + 1] = row rl1
    uint32_t kw0[kWords], kw1[kWords];   // keep bits, one word per 32 keys
#pragma unroll
    for (int w = 0; w < kWords; ++w) kw0[w] = kw1[w] = 0u;
    const unsigned long long ctr_tile = ctr_c + (unsigned long long)key0;
#pragma unroll
    for (int i2 = 0; i2 < kBlockN / 16; ++i2) {   // 8-key groups i = 2 i2, 2 i2 + 1
      // km[2h + r]: keep masks of group 2 i2 + h, row rl0 (r = 0) / rl1 (r = 1); word c decides the pair of keys
      // 8i + 2c, +1 (bit layout of fmha_api.h)
      uint32_t km[4] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu};
      if (drop) {
        const Philox4 r = philox4x32<7>(p.seed, p.offset, (ctr_tile + 16u * i2) >> 3);
        uint32_t w[4] = {r.x, r.y, r.z, r.w};
        quad_transpose4(w, c);
#pragma unroll
        for (int k = 0; k < 4; ++k) km[k] = keep_mask2(w[k], t14x2);
      }
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        const int i = 2 * i2 + hh;
        const float p00 = ex2_approx(fmaf(s[4 * i + 0], kLog2e, nm0)), p01 = ex2_approx(fmaf(s[4 * i + 1], kLog2e, nm0));
        const float p10 = ex2_approx(fmaf(s[4 * i + 2], kLog2e, nm1)), p11 = ex2_approx(fmaf(s[4 * i + 3], kLog2e, nm1));
        l0 += p00 + p01;
        l1 += p10 + p11;
        const uint32_t km0 = km[2 * hh], km1 = km[2 * hh + 1];
        const uint32_t bit = 0x00010001u << (4 * (i & 3) + c);
        kw0[i >> 2] |= km0 & bit;
        kw1[i >> 2] |= km1 & bit;
        pa[2 * i] = pack2<T>(p00, p01) & km0;
        pa[2 * i + 1] = pack2<T>(p10, p11) & km1;
      }
    }
    if (drop && p.drop_bits != nullptr) {
#pragma unroll
      for (int w = 0; w < kWords; ++w) {
        kw0[w] |= __shfl_xor_sync(0xffffffffu, kw0[w], 1);
        kw0[w] |= __shfl_xor_sync(0xffffffffu, kw0[w], 2);
        kw1[w] |= __shfl_xor_sync(0xffffffffu, kw1[w], 1);
        kw1[w] |= __shfl_xor_sync(0xffffffffu, kw1[w], 2);
      }
      // thread c of the quad stores word c of both rows
      uint32_t w0, w1;
      if constexpr (kWords == 4) {
        w0 = c == 0 ? kw0[0] : (c == 1 ? kw0[1] : (c == 2 ? kw0[2] : kw0[3]));
        w1 = c == 0 ? kw1[0] : (c == 1 ? kw1[1] : (c == 2 ? kw1[2] : kw1[3]));
      } else {
        w0 = c == 0 ? kw0[0] : kw0[1];
        w1 = c == 0 ? kw1[0] : kw1[1];
      }
      if (c < kWords && key0 + 32 * c < p.Lk) {
        const int wi = (key0 >> 5) + c;
        if (row0 < row_lim) p.drop_bits[lin0 * words_per_row + wi] = w0;
        if (row1 < row_lim) p.drop_bits[lin1 * words_per_row + wi] = w1;
      }
    }

    // ---- O += P V ---------------------------------------------------------------------------------------
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kBlockN / 16; ++kk) {   // 16 keys = 16 rows of 128 bytes per step
      const uint32_t a[4] = {pa[4 * kk], pa[4 * kk + 1], pa[4 * kk + 2], pa[4 * kk + 3]};
      const uint32_t v_addr = smem_base + C::kSmemV + st * C::kKVStage + kk * 2048;
      if constexpr (DP == 64) wgmma_m64n64_rs<T, 1>(o, a, make_desc_sw128(v_addr), 1u);
      else wgmma_m64n128_rs<T, 1>(o, a, make_desc_sw128_mn(v_addr, C::kKVBox), 1u);
    }
    wgmma_commit();
    if constexpr (kLogits) {   // while the product runs: the logits tile leaves through one TMA store per 64 keys
      fence_proxy_async_smem();
      __syncthreads();
      if (tid == 0) {
#pragma unroll
        for (int x = 0; x < kBlockN / 64; ++x)
          tma_store_3d(&p.sw_logits, key0 + 64 * x, q0, (int)bh, smem_base + C::kSmemBias + st * C::kBiasStage + x * 8192);
        bulk_commit();
      }
    }
    wgmma_wait<0>();
    fence_operands(o);
  }

  // ---- epilogue ---------------------------------------------------------------------------------------
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float inv0 = l0 > 0.f ? keep_scale / l0 : 0.f, inv1 = l1 > 0.f ? keep_scale / l1 : 0.f;
  T* out = reinterpret_cast<T*>(p.out);
  const int D = p.D;   // columns 8i + 2c, +1 exist iff 8i < D (D % 8 == 0)
  // padded: row (b, i) of [B, Lq, H, D]; varlen: packed row s_b + i of [N, H, D]
  const long long orow0 = kVarlen ? (long long)vl_s : (long long)b * p.Lq;
  if (row0 < row_lim) {
    uint32_t* og = reinterpret_cast<uint32_t*>(out + ((orow0 + row0) * p.H + h) * D + 2 * c);
#pragma unroll
    for (int i = 0; i < DP / 8; ++i)
      if (8 * i < D) og[4 * i] = pack2<T>(o[4 * i + 0] * inv0, o[4 * i + 1] * inv0);
    if (c == 0 && (!kKVCache || p.lse != nullptr))
      p.lse[lin0] = l0 > 0.f ? m0 + __logf(l0) : -CUDART_INF_F;   // natural-log LSE of the logits
  }
  if (row1 < row_lim) {
    uint32_t* og = reinterpret_cast<uint32_t*>(out + ((orow0 + row1) * p.H + h) * D + 2 * c);
#pragma unroll
    for (int i = 0; i < DP / 8; ++i)
      if (8 * i < D) og[4 * i] = pack2<T>(o[4 * i + 2] * inv1, o[4 * i + 3] * inv1);
    if (c == 0 && (!kKVCache || p.lse != nullptr)) p.lse[lin1] = l1 > 0.f ? m1 + __logf(l1) : -CUDART_INF_F;
  }
  if constexpr (kLogits) {
    if (tid == 0) bulk_wait_all();   // shared memory must outlive the last logits store's reads
  }
}

}  // namespace

void launch_fmha_fwd(const FmhaFwdParams& p, cudaStream_t stream) {
  dim3 grid((p.Lq + kBlockM - 1) / kBlockM, p.H, p.B);
  auto run = [&](auto kern, uint32_t smem_bytes) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes);
    kern<<<grid, kFwdThreads, smem_bytes, stream>>>(p);
  };
  auto dispatch = [&](auto logits, auto causal, auto kvcache, auto varlen, auto paged) {
    constexpr bool kLogits = decltype(logits)::value, kCausal = decltype(causal)::value;
    constexpr bool kKV = decltype(kvcache)::value, kVL = decltype(varlen)::value, kPg = decltype(paged)::value;
    if (p.D <= 64) {
      if (p.is_bf16) run(fmha_fwd_kernel<__nv_bfloat16, 64, kLogits, kCausal, kKV, kVL, kPg>, FwdCfg<64>::kSmemBytes);
      else run(fmha_fwd_kernel<__half, 64, kLogits, kCausal, kKV, kVL, kPg>, FwdCfg<64>::kSmemBytes);
    } else {
      if (p.is_bf16) run(fmha_fwd_kernel<__nv_bfloat16, 128, kLogits, kCausal, kKV, kVL, kPg>, FwdCfg<128>::kSmemBytes);
      else run(fmha_fwd_kernel<__half, 128, kLogits, kCausal, kKV, kVL, kPg>, FwdCfg<128>::kSmemBytes);
    }
  };
  // causal + logits is refused by the binding (fmha_bind.cpp); the KV-cache mode sets neither, and the varlen
  // bindings never set logits
  const std::false_type no;
  const std::true_type yes;
  const bool paged = p.kvcache && p.block_table != nullptr;   // the bindings set a block table in KV-cache mode only
  if (p.varlen) {
    if (paged) dispatch(no, no, yes, yes, yes);
    else if (p.kvcache) dispatch(no, no, yes, yes, no);
    else if (p.causal) dispatch(no, yes, no, yes, no);
    else dispatch(no, no, no, yes, no);
  } else if (paged) dispatch(no, no, yes, no, yes);
  else if (p.kvcache) dispatch(no, no, yes, no, no);
  else if (p.logits != nullptr) dispatch(yes, no, no, no, no);
  else if (p.causal) dispatch(no, yes, no, no, no);
  else dispatch(no, no, no, no, no);
}

}  // namespace ub
