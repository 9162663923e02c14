// Decode attention for sm_90a: one query row per (batch, head) against the first n_b rows of a key / value cache,
//   O[b, h] = softmax(scale * q k^T + bias + key mask) V          (fp16 / bf16 in and out, fp32 math)
// with an optional append of the new token's key / value into row seqlens[b] of the caches in the same launch.
//
// M = 1 leaves nothing for wgmma: each key is a dot product and an axpy, and a step has to stream K and V once at HBM
// bandwidth.  So the kernel is a copy pipeline feeding the CUDA cores:
//   * Grouped-query attention: query head h reads key / value head h / G (G = kv_group).  The grid stays (splits, H,
//     B): placing the G CTAs that read the same rows next to each other (x = s * G + g) measured no faster on an H100.
//   * Split-KV: CTA (s, h, b) takes the contiguous key range [s * chunk, (s + 1) * chunk) of (b, h) (the last split
//     runs to n_b); chunk comes from the host bound, or with p.chunk == 0 from n_b itself (a CUDA graph captured at
//     the capacity).  With one split it writes O; otherwise it writes an fp32 partial (o[D] unnormalised, m, l) and
//     fmha_decode_combine_kernel merges the splits in ascending order.  No atomics: for a given split count the
//     result does not depend on the schedule.
//   * Streaming: warp 0 requests the K and V rows of key tile t + kStages with one cp.async.bulk per row (rows are
//     D * 2 bytes, a multiple of 16; no tensor map to encode on the host) into stage t % kStages, completion on that
//     stage's mbarrier.  kStages * 16 KB are in flight per CTA, three CTAs per SM.
//   * Math: 16 groups of 8 lanes; lane j of a group holds 16-byte chunks j and j + 8 of the pre-scaled query
//     (scale * log2e) in fp32.  Group g takes keys g, g + 16, ... of a tile: partial dot products, three xor
//     shuffles, then the online softmax with ex2 over the group's keys of the tile and P V into the lane's fp32
//     chunks.  At the end the 16 group states are merged in shared memory in group order.
//   * Append (k_new / v_new set): the new token's key and value are row pos = seqlens[b] of the caches, and that row
//     is always the last visible key (n_b = pos + 1).  The CTAs whose range holds pos bulk-copy that row into their
//     stage straight from k_new / v_new (not from the cache), and the one of the first query head of the group stores
//     it bitwise into the caches.  No CTA reads row pos of (b, h / G) from the caches - every other key range ends
//     before it - so the write needs no ordering against any read, and one launch both appends and attends.
//   * Paged caches (kPaged, fmha_api.h): the row of key j is row j % block_size of pool block
//     block_table[b, j / block_size].  Warp 0 loads the blocks of tile t + kStages before the math of tile t and
//     issues its copies after it, so the table load's latency is hidden; the owner stores the new row through the
//     table too, and skips the store when its entry is outside the pool.  Ranges, splits and the combine are
//     unchanged.
//   * Bounds: n_b is clamped to the cache capacity C (and to the columns of the bias / key mask), pos to n_b - 1, for
//     any device value of seqlens: no read or write outside the tensors.  A row whose visible keys are all masked
//     gives O = 0.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <math_constants.h>

#include <algorithm>
#include <type_traits>

#include "../common.cuh"
#include "fmha_api.h"

namespace ub {
namespace {

constexpr int kThreads = 128;
constexpr int kGroups = kThreads / 8;   // 8 lanes per key
constexpr int kStages = 4;
constexpr float kLog2e = 1.4426950408889634f;

// NC = 16-byte chunks per lane: 1 for D <= 64, 2 for D <= 128.  A stage holds kTile K rows and kTile V rows of at
// most 64 * NC columns: 16 KB either way.
template <int NC>
struct DecCfg {
  static constexpr int kTile = NC == 1 ? 64 : 32;               // keys per tile
  static constexpr int kKeysPerGroup = kTile / kGroups;          // 4 or 2
  static constexpr uint32_t kRowMax = 64 * NC * 2;               // bytes of the widest row
  static constexpr uint32_t kStageBytes = 2 * kTile * kRowMax;   // K rows, then V rows
  static constexpr uint32_t kSmemRedO = kStages * kStageBytes;   // float[kGroups][64 * NC]
  static constexpr uint32_t kSmemRedML = kSmemRedO + kGroups * 64 * NC * 4;   // float[2][kGroups]
  static constexpr uint32_t kSmemBar = kSmemRedML + 2 * kGroups * 4;
  static constexpr uint32_t kSmemBytes = kSmemBar + kStages * 8;
};

UB_DEVICE int clampi(int x, int lo, int hi) { return x < lo ? lo : (x > hi ? hi : x); }

template <typename T, int NC, bool kPaged>
__global__ void __launch_bounds__(kThreads) fmha_decode_kernel(const FmhaDecodeParams p) {
  using C = DecCfg<NC>;
  extern __shared__ __align__(16) unsigned char smem[];
  const int tid = threadIdx.x, lane = tid & 31, g = tid >> 3, j8 = tid & 7;
  // query head h = hk * G + gq reads cache head hk (fmha_api.h)
  const int G = p.kv_group, s = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int hk = h / G, gq = h % G;
  const int D = p.D, nch = D / 8;
  const uint32_t row_bytes = (uint32_t)D * 2;

  // ---- visible keys of (b, h) and this CTA's range --------------------------------------------------------------
  int cap = p.C;
  if (p.bias != nullptr) cap = min(cap, p.bias_cols);
  if (p.kpm != nullptr) cap = min(cap, p.kpm_cols);
  const bool append = p.k_new != nullptr;
  const int len = p.seqlens != nullptr ? p.seqlens[b] : cap;
  const int pos = append ? clampi(len, 0, cap - 1) : -1;   // row of the new token
  const int n = append ? pos + 1 : clampi(len, 0, cap);
  const int chunk = p.chunk > 0 ? p.chunk : max(1, (n + p.num_splits - 1) / p.num_splits);
  const int start = s * chunk;
  const int end = s == p.num_splits - 1 ? n : min(start + chunk, n);

  // contiguous: batch b of the caches; paged: the pools, whose block is chosen per row
  const long long kc_b = kPaged ? 0LL : (long long)b * p.kc_sb, vc_b = kPaged ? 0LL : (long long)b * p.vc_sb;
  const T* kc = reinterpret_cast<const T*>(p.k_cache) + kc_b + (long long)hk * p.kc_sh;
  const T* vc = reinterpret_cast<const T*>(p.v_cache) + vc_b + (long long)hk * p.vc_sh;
  // offsets (elements) of row `key` from kc / vc
  auto k_row = [&](int key) -> long long {
    if constexpr (kPaged)
      return (long long)fmha_paged_block(p.block_table, b, key, p.block_size, p.blocks_per_seq, p.num_blocks) *
                 p.kc_sb + (long long)(key % p.block_size) * p.kc_sl;
    else
      return (long long)key * p.kc_sl;
  };
  auto v_row = [&](int key) -> long long {
    if constexpr (kPaged)
      return (long long)fmha_paged_block(p.block_table, b, key, p.block_size, p.blocks_per_seq, p.num_blocks) *
                 p.vc_sb + (long long)(key % p.block_size) * p.vc_sl;
    else
      return (long long)key * p.vc_sl;
  };
  const T* kn = append ? reinterpret_cast<const T*>(p.k_new) + (long long)b * p.kn_sb + (long long)hk * p.kn_sh : nullptr;
  const T* vn = append ? reinterpret_cast<const T*>(p.v_new) + (long long)b * p.vn_sb + (long long)hk * p.vn_sh : nullptr;
  // one CTA of the group stores the new row; the other G - 1 take it from k_new / v_new into their stage only
  bool owner = append && gq == 0 && start <= pos && pos < end;
  if constexpr (kPaged) {   // no write through an entry outside the pool
    if (owner) {
      const int blk = p.block_table[(long long)b * p.blocks_per_seq + pos / p.block_size];
      owner = blk >= 0 && blk < p.num_blocks;
    }
  }
  if (owner && tid < 2 * nch) {
    // bitwise copy of the new row into the caches (see the append invariant above)
    const int c = tid % nch;
    const bool is_v = tid >= nch;
    const Vec16 w = ld_global_v4((is_v ? vn : kn) + 8 * c);
    T* dst = const_cast<T*>(is_v ? vc + v_row(pos) : kc + k_row(pos));
    st_global_v4(dst + 8 * c, w);
  }

  const int ntiles = end > start ? (end - start + C::kTile - 1) / C::kTile : 0;
  const uint32_t smem0 = smem_addr_u32(smem);
  const uint32_t bar0 = smem0 + C::kSmemBar;
  auto issue = [&](int t) {   // warp 0: K and V rows of tile t into stage t % kStages
    const int st = t % kStages, r0 = start + t * C::kTile, nrows = min(C::kTile, end - r0);
    const uint32_t bar = bar0 + 8 * st, dk = smem0 + st * C::kStageBytes, dv = dk + C::kTile * row_bytes;
    if (lane == 0) bulk_expect_tx(bar, 2u * nrows * row_bytes);
    __syncwarp();
    for (int r = lane; r < nrows; r += 32) {
      const int key = r0 + r;
      const bool is_new = key == pos;
      bulk_g2s(dk + r * row_bytes, is_new ? kn : kc + k_row(key), row_bytes, bar);
      bulk_g2s(dv + r * row_bytes, is_new ? vn : vc + v_row(key), row_bytes, bar);
    }
  };
  // paged: lane l of warp 0 copies rows l and l + 32 of a tile; their pool blocks are loaded a tile ahead (before the
  // math of tile t for the copies of tile t + kStages), so the table load's latency does not hold up warp 0
  // A tile (kTile <= 64 rows) spans at most two blocks (block_size >= 128), so one division per tile places its rows.
  constexpr int kRowsPerLane = C::kTile / 32;
  auto row_blocks = [&](int t, int (&blk)[kRowsPerLane], int (&row)[kRowsPerLane]) {
    const int r0 = start + t * C::kTile, nrows = min(C::kTile, end - r0);
    const int e0 = r0 / p.block_size, off0 = r0 - e0 * p.block_size;
#pragma unroll
    for (int i = 0; i < kRowsPerLane; ++i) {
      const int r = lane + 32 * i, o = off0 + r;
      const bool next = o >= p.block_size;
      row[i] = next ? o - p.block_size : o;
      blk[i] = 0;
      if (r < nrows) {
        const int x = p.block_table[(long long)b * p.blocks_per_seq + e0 + (next ? 1 : 0)];
        blk[i] = x < 0 ? 0 : (x >= p.num_blocks ? p.num_blocks - 1 : x);   // fmha_paged_block's clamp
      }
    }
  };
  auto issue_paged = [&](int t, const int (&blk)[kRowsPerLane], const int (&row)[kRowsPerLane]) {
    const int st = t % kStages, r0 = start + t * C::kTile, nrows = min(C::kTile, end - r0);
    const uint32_t bar = bar0 + 8 * st, dk = smem0 + st * C::kStageBytes, dv = dk + C::kTile * row_bytes;
    if (lane == 0) bulk_expect_tx(bar, 2u * nrows * row_bytes);
    __syncwarp();
#pragma unroll
    for (int i = 0; i < kRowsPerLane; ++i) {
      const int r = lane + 32 * i;
      if (r < nrows) {
        const int key = r0 + r;
        const bool is_new = key == pos;
        const T* ks = is_new ? kn : kc + blk[i] * p.kc_sb + (long long)row[i] * p.kc_sl;
        const T* vs = is_new ? vn : vc + blk[i] * p.vc_sb + (long long)row[i] * p.vc_sl;
        bulk_g2s(dk + r * row_bytes, ks, row_bytes, bar);
        bulk_g2s(dv + r * row_bytes, vs, row_bytes, bar);
      }
    }
  };
  if (tid == 0) {
    for (int st = 0; st < kStages; ++st) bulk_bar_init(bar0 + 8 * st, 1);
    bulk_bar_init_fence();
  }
  __syncthreads();
  if (tid < 32) {
    if constexpr (kPaged) {   // every table load of the first stages first, so that their latencies overlap
      int blk[kStages][kRowsPerLane], row[kStages][kRowsPerLane];
#pragma unroll
      for (int t = 0; t < kStages; ++t)
        if (t < ntiles) row_blocks(t, blk[t], row[t]);
#pragma unroll
      for (int t = 0; t < kStages; ++t)
        if (t < ntiles) issue_paged(t, blk[t], row[t]);
    } else {
      for (int t = 0; t < min(kStages, ntiles); ++t) issue(t);
    }
  }

  // ---- query chunks of this lane, pre-scaled by scale * log2e ------------------------------------------------------
  const float qs = p.scale * kLog2e;
  float qf[8 * NC], acc[8 * NC];
  const T* q = reinterpret_cast<const T*>(p.q) + (long long)b * p.q_sb + (long long)h * p.q_sh;
#pragma unroll
  for (int c = 0; c < NC; ++c) {
    const int ch = j8 + 8 * c;
    if (ch < nch) {
      unpack<T>(ld_global_v4(q + 8 * ch), qf + 8 * c);
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e) qf[8 * c + e] = 0.f;
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      qf[8 * c + e] *= qs;
      acc[8 * c + e] = 0.f;
    }
  }
  const T* bias = p.bias != nullptr
                      ? reinterpret_cast<const T*>(p.bias) + (p.bias_batch > 1 ? (long long)b * p.bias_sb : 0LL) +
                            (long long)h * p.bias_sh
                      : nullptr;
  const uint8_t* kpm = p.kpm != nullptr ? p.kpm + (long long)b * p.kpm_sb : nullptr;

  float m = -CUDART_INF_F, l = 0.f;
  for (int t = 0; t < ntiles; ++t) {
    int next_blk[kRowsPerLane], next_row[kRowsPerLane];   // paged: tile t + kStages's rows, placed before the math
    if constexpr (kPaged) {
      if (tid < 32 && t + kStages < ntiles) row_blocks(t + kStages, next_blk, next_row);
    }
    const int st = t % kStages, r0 = start + t * C::kTile, nrows = min(C::kTile, end - r0);
    bulk_wait(bar0 + 8 * st, (t / kStages) & 1);
    const unsigned char* sk = smem + st * C::kStageBytes;
    const unsigned char* sv = sk + C::kTile * row_bytes;
    float sc[C::kKeysPerGroup];
#pragma unroll
    for (int i = 0; i < C::kKeysPerGroup; ++i) {
      const int r = g + kGroups * i;
      float d = 0.f;
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        const int ch = j8 + 8 * c;
        if (ch < nch) {
          float kf[8];
          unpack<T>(*reinterpret_cast<const Vec16*>(sk + r * row_bytes + 16 * ch), kf);
#pragma unroll
          for (int e = 0; e < 8; ++e) d = fmaf(qf[8 * c + e], kf[e], d);
        }
      }
      d += __shfl_xor_sync(0xffffffffu, d, 1);
      d += __shfl_xor_sync(0xffffffffu, d, 2);
      d += __shfl_xor_sync(0xffffffffu, d, 4);
      // rows past the range hold stale bytes: their score is replaced, and their V row is never read
      const int key = r0 + r;
      if (r < nrows) {
        if (bias != nullptr) d = fmaf(to_f32<T>(bias[key]), kLog2e, d);
        if (kpm != nullptr && kpm[key] != 0) d = -CUDART_INF_F;
      } else {
        d = -CUDART_INF_F;
      }
      sc[i] = d;
    }
    float mt = sc[0];
#pragma unroll
    for (int i = 1; i < C::kKeysPerGroup; ++i) mt = fmaxf(mt, sc[i]);
    const float m_new = fmaxf(m, mt);
    if (m_new != -CUDART_INF_F) {   // else every key so far is masked: l and acc stay 0
      const float alpha = ex2_approx(m - m_new);   // m = -inf -> 0
      l *= alpha;
#pragma unroll
      for (int e = 0; e < 8 * NC; ++e) acc[e] *= alpha;
#pragma unroll
      for (int i = 0; i < C::kKeysPerGroup; ++i) {
        const int r = g + kGroups * i;
        if (r < nrows) {
          const float pk = ex2_approx(sc[i] - m_new);
          l += pk;
#pragma unroll
          for (int c = 0; c < NC; ++c) {
            const int ch = j8 + 8 * c;
            if (ch < nch) {
              float vf[8];
              unpack<T>(*reinterpret_cast<const Vec16*>(sv + r * row_bytes + 16 * ch), vf);
#pragma unroll
              for (int e = 0; e < 8; ++e) acc[8 * c + e] = fmaf(pk, vf[e], acc[8 * c + e]);
            }
          }
        }
      }
      m = m_new;
    }
    __syncthreads();   // every thread is done with stage st
    if (tid < 32 && t + kStages < ntiles) {
      if constexpr (kPaged) issue_paged(t + kStages, next_blk, next_row);
      else issue(t + kStages);
    }
  }

  // ---- merge the 16 group states in group order --------------------------------------------------------------------
  float* red_o = reinterpret_cast<float*>(smem + C::kSmemRedO);
  float* red_m = reinterpret_cast<float*>(smem + C::kSmemRedML);
  float* red_l = red_m + kGroups;
  if (j8 == 0) {
    red_m[g] = m;
    red_l[g] = l;
  }
#pragma unroll
  for (int c = 0; c < NC; ++c) {
    const int ch = j8 + 8 * c;
    if (ch < nch) {
#pragma unroll
      for (int e = 0; e < 8; ++e) red_o[g * 64 * NC + 8 * ch + e] = acc[8 * c + e];
    }
  }
  __syncthreads();
  float mm = red_m[0];
#pragma unroll
  for (int i = 1; i < kGroups; ++i) mm = fmaxf(mm, red_m[i]);
  if (tid < D) {
    float o = 0.f, ls = 0.f;
    if (mm != -CUDART_INF_F) {
#pragma unroll
      for (int i = 0; i < kGroups; ++i) {
        const float w = ex2_approx(red_m[i] - mm);
        ls = fmaf(red_l[i], w, ls);
        o = fmaf(red_o[i * 64 * NC + tid], w, o);
      }
    }
    const long long bh = (long long)b * p.H + h;
    if (p.num_splits == 1) {
      reinterpret_cast<T*>(p.out)[bh * D + tid] = from_f32<T>(ls > 0.f ? o / ls : 0.f);
    } else {
      const long long part = bh * p.num_splits + s;
      p.part_o[part * D + tid] = o;   // o = 0, m = -inf, l = 0: the neutral partial of an empty range
      if (tid == 0) {
        p.part_ml[2 * part] = mm;
        p.part_ml[2 * part + 1] = ls;
      }
    }
  }
}

// O[b, h] from the num_splits partials of (b, h), added in ascending split order.  One CTA per (b, h), thread d owns
// column d.
template <typename T>
__global__ void __launch_bounds__(kThreads) fmha_decode_combine_kernel(const FmhaDecodeParams p) {
  const int h = blockIdx.x, b = blockIdx.y, d = threadIdx.x;
  if (d >= p.D) return;
  const long long bh = (long long)b * p.H + h;
  const float* ml = p.part_ml + 2 * bh * p.num_splits;
  const float* po = p.part_o + bh * p.num_splits * p.D + d;
  float mm = -CUDART_INF_F;
  for (int s = 0; s < p.num_splits; ++s) mm = fmaxf(mm, ml[2 * s]);
  float o = 0.f, ls = 0.f;
  if (mm != -CUDART_INF_F) {
    for (int s = 0; s < p.num_splits; ++s) {
      const float w = ex2_approx(ml[2 * s] - mm);
      ls = fmaf(ml[2 * s + 1], w, ls);
      o = fmaf(po[(long long)s * p.D], w, o);
    }
  }
  reinterpret_cast<T*>(p.out)[bh * p.D + d] = from_f32<T>(ls > 0.f ? o / ls : 0.f);
}

// Row i of k_new / v_new -> row p_b + i of the caches (fmha_api.h).  CTA (i, b) copies all H cache heads of K and V,
// one 16-byte vector per thread and step; a row at or past C is skipped.  kPacked: k_new / v_new are packed [N, H, D]
// and sequence b's rows are s_b + i, i < T_b ({s_b, T_b} = fmha_varlen_seq(cu_seqlens, b, T, N)).  kPaged: the row
// goes through the block table into the pools, and a row whose entry is outside the pool is skipped.
template <bool kPacked, bool kPaged>
__global__ void __launch_bounds__(kThreads) kv_cache_append_kernel(const KvCacheAppendParams p) {
  const int i = blockIdx.x, b = blockIdx.y;
  int s_b = 0;   // packed: the first row of sequence b in k_new / v_new, whose batch stride is 0
  if constexpr (kPacked) {
    const int2 sn = fmha_varlen_seq(p.cu_seqlens, b, p.T, p.packed_rows);
    if (i >= sn.y) return;
    s_b = sn.x;
  }
  const int pos = min(max(p.seqlens[b], 0), p.C) + i;
  if (pos >= p.C) return;
  long long cb = b, cl = pos;   // cache batch (pool block) and row
  if constexpr (kPaged) {   // a row whose entry is outside the pool is skipped
    const int blk = p.block_table[(long long)b * p.blocks_per_seq + pos / p.block_size];
    if (blk < 0 || blk >= p.num_blocks) return;
    cb = blk;
    cl = pos % p.block_size;
  }
  const int nch = p.D / 8, per = p.H * nch;   // 16-byte chunks of one row of one tensor
  for (int x = threadIdx.x; x < 2 * per; x += kThreads) {
    const bool is_v = x >= per;
    const int h = (x % per) / nch, c = x % nch;
    const uint16_t* src = reinterpret_cast<const uint16_t*>(is_v ? p.v_new : p.k_new) +
                          (long long)b * (is_v ? p.vn_sb : p.kn_sb) + (long long)(s_b + i) * (is_v ? p.vn_sl : p.kn_sl) +
                          (long long)h * (is_v ? p.vn_sh : p.kn_sh) + 8 * c;
    uint16_t* dst = reinterpret_cast<uint16_t*>(is_v ? p.v_cache : p.k_cache) +
                    cb * (is_v ? p.vc_sb : p.kc_sb) + cl * (is_v ? p.vc_sl : p.kc_sl) +
                    (long long)h * (is_v ? p.vc_sh : p.kc_sh) + 8 * c;
    st_global_v4(dst, ld_global_v4(src));
  }
}

}  // namespace

void launch_kv_cache_append(const KvCacheAppendParams& p, cudaStream_t stream) {
  const dim3 grid(p.T, p.B);
  if (p.block_table != nullptr) {
    if (p.cu_seqlens != nullptr) kv_cache_append_kernel<true, true><<<grid, kThreads, 0, stream>>>(p);
    else kv_cache_append_kernel<false, true><<<grid, kThreads, 0, stream>>>(p);
  } else {
    if (p.cu_seqlens != nullptr) kv_cache_append_kernel<true, false><<<grid, kThreads, 0, stream>>>(p);
    else kv_cache_append_kernel<false, false><<<grid, kThreads, 0, stream>>>(p);
  }
}

int fmha_decode_num_splits(int B, int H, int len_bound, int num_sms) {
  // As many splits as fit the num_sms * kDecodeCtasPerSm resident CTAs in one wave (a partial second wave would
  // leave most SMs idle at its end); no split shorter than kDecodeMinSplitKeys (its partial and the second launch
  // would cost more than its keys).  B * H above half the resident slots runs with one split.
  const long long bh = (long long)B * H, slots = (long long)num_sms * kDecodeCtasPerSm;
  long long s = slots / bh;
  s = std::min<long long>(s, (len_bound + kDecodeMinSplitKeys - 1) / kDecodeMinSplitKeys);
  return (int)std::max<long long>(1, std::min<long long>(s, kDecodeMaxSplits));
}

void launch_fmha_decode(const FmhaDecodeParams& p, cudaStream_t stream) {
  const dim3 grid(p.num_splits, p.H, p.B);
  auto run = [&](auto kern, auto combine, uint32_t smem_bytes) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes);
    kern<<<grid, kThreads, smem_bytes, stream>>>(p);
    if (p.num_splits > 1) combine<<<dim3(p.H, p.B), kThreads, 0, stream>>>(p);
  };
  auto by_type = [&](auto paged) {
    constexpr bool kPg = decltype(paged)::value;
    if (p.D <= 64) {
      if (p.is_bf16) run(fmha_decode_kernel<__nv_bfloat16, 1, kPg>, fmha_decode_combine_kernel<__nv_bfloat16>, DecCfg<1>::kSmemBytes);
      else run(fmha_decode_kernel<__half, 1, kPg>, fmha_decode_combine_kernel<__half>, DecCfg<1>::kSmemBytes);
    } else {
      if (p.is_bf16) run(fmha_decode_kernel<__nv_bfloat16, 2, kPg>, fmha_decode_combine_kernel<__nv_bfloat16>, DecCfg<2>::kSmemBytes);
      else run(fmha_decode_kernel<__half, 2, kPg>, fmha_decode_combine_kernel<__half>, DecCfg<2>::kSmemBytes);
    }
  };
  if (p.block_table != nullptr) by_type(std::true_type{});
  else by_type(std::false_type{});
}

}  // namespace ub
