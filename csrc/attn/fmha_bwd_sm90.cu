// Fused multi-head attention backward for sm_90a (head_dim D % 8 == 0, 8 <= D <= 128, fp16/bf16), flash-attention style
// (reference: autograd through unicore/modules/multihead_attention.py:47-113 + softmax_fast.h:513-666):
// probabilities are recomputed from the saved log-sum-exp; the dropout keep bits come from the
// forward pass (1 bit / element).
//
//   Templated on the padded head width DP (64 or 128): Q / K / V / dO tiles are DP / 64 column boxes whose columns
//   D..DP-1 the TMA unit zero-fills, so they add nothing to S, dP or the products, and the epilogues store columns
//   below D only.
//   grid = (64-key tiles, H, B); one CTA = one warpgroup owns K_j, V_j and walks the 64-row query tiles i.  The
//   products are computed transposed (keys are the M dimension), so that P^T and dS^T are accumulator tiles whose
//   16-bit conversions are directly the register A operands of the dV / dK products:
//     S^T  = K_j Q_i^T                      wgmma m64n64, both operands K-major from shared memory
//     dP^T = V_j dO_i^T                     wgmma m64n64, a commit group of its own: P is formed while it runs
//     P = exp2((S*scale + bias + kmask) * log2e - LSE_i * log2e) ;  dS = P o (drop(dP) - delta_i)
//                                           (keep bits read once per tile into registers, applied as selects)
//     dV_j += drop(P)^T dO_i                wgmma m64n{DP}, A from registers, dO MN-major
//     dK_j += dS^T Q_i                      wgmma m64n{DP}, A from registers, Q MN-major
//     dQ_i += dS K_j                        wgmma m64n64 per 64-column half of K (one dq[32] reused, so that DP = 128
//                                           fits the registers next to dV and dK), dS from shared memory
//                                           (stmatrix.trans of the registers, written in place over the consumed bias
//                                           tile), K MN-major; the fp32 tile (bank-conflict-free column order,
//                                           dq_swz_col) is added to a global fp32 accumulator of the same order
//                                           with ONE bulk reduction (cp.reduce.async.bulk)
//     dS tile (16-bit, in shared memory for the dQ product) -> TMA store; a follow-up kernel sums it over the batch
//     into dBias.
//   Q_i, dO_i and the bias tile are fetched one query tile ahead (two stages), one thread issues every copy.
// Pre-pass: delta = rowsum(dO o O).   Post-pass: dq = scale * the fp32 accumulator (and dbias = batch sum of dS).
// Logits mode (template flag kLogits, bp.dlogits set): the gradient dz of the forward's logits output arrives by TMA next
// to the bias tile (two more 8 KB stages) and is added to dS in fp32, so dS_total = P o (drop(dP) - delta) + dz reaches
// dK, dQ and dBias.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <math_constants.h>

#include <algorithm>

#include "../common.cuh"
#include "fmha_api.h"
#include "wgmma.cuh"

namespace ub {
namespace {

using namespace tc;

constexpr int kBM = 64, kBN = 64;   // query rows per step, keys per CTA
constexpr int kBwdThreads = 128;

// shared memory map (bytes) of the padded head width DP; every box is 64 rows x 128 B, 128-byte swizzled, and a
// Q / K / V / dO tile is DP / 64 boxes of 8 KB.  Logits mode adds two 8 KB stages of the incoming logits gradient dz.
template <int DP, bool kLogits = false>
struct BwdCfg {
  static constexpr int kBoxes = DP / 64;
  static constexpr uint32_t kTile = kBoxes * 8192;
  static constexpr uint32_t kOffK = 0;
  static constexpr uint32_t kOffV = kOffK + kTile;
  static constexpr uint32_t kOffQ = kOffV + kTile;        // 2 stages
  static constexpr uint32_t kOffDO = kOffQ + 2 * kTile;   // 2 stages
  static constexpr uint32_t kOffDS = kOffDO + 2 * kTile;  // 2 stages x 8 KB: bias tile [q][key], then dS in place
  static constexpr uint32_t kOffDZ = kOffDS + 2 * 8192;   // logits mode: 2 stages x 8 KB dz tile [q][key]
  static constexpr uint32_t kOffDQ = kOffDZ + (kLogits ? 2 * 8192 : 0);   // fp32 [64][DP] dQ tile (dq_swz_col)
  static constexpr uint32_t kOffStats = kOffDQ + kBM * DP * 4;   // 2 stages x {float lse2[64], delta[64], bits[2][64]}
  static constexpr uint32_t kOffBar = kOffStats + 2048;
  static constexpr uint32_t kSmemBytes = kOffBar + 32 + 1024;   // + alignment slack of the 1024-byte-aligned base
};
static_assert(BwdCfg<64>::kOffStats == 81920 && BwdCfg<64>::kSmemBytes == 85024,
              "DP = 64 keeps the shared memory map of the 64-only kernel");

template <typename T>
UB_DEVICE uint32_t bwd_pack2(float a, float b);
template <>
UB_DEVICE uint32_t bwd_pack2<__half>(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
template <>
UB_DEVICE uint32_t bwd_pack2<__nv_bfloat16>(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
template <typename T>
UB_DEVICE float2 bwd_unpack2(uint32_t w) {
  if constexpr (std::is_same<T, __half>::value) {
    return __half22float2(*reinterpret_cast<const __half2*>(&w));
  } else {
    return make_float2(__uint_as_float(w << 16), __uint_as_float(w & 0xffff0000u));
  }
}

// Column layout of the fp32 dQ tile in shared memory and of its accumulator rows in global memory (the bulk reduction
// copies the tile linearly): the 8-column (32-byte) group of column `col` in row q is stored at group ^ (q & 7).  A
// warp's float2 stores cover 8 rows x 8 columns of one group; unswizzled, every row of 256 or 512 bytes starts in the
// same bank and the store takes 8 wavefronts, swizzled it takes the minimum, 2.
UB_DEVICE int dq_swz_col(int q, int col) { return (((col >> 3) ^ (q & 7)) << 3) | (col & 7); }

// ---- deterministic mode: ordered dQ reductions -----------------------------------------------------------------
__device__ unsigned int g_det_timeouts;   // waits that gave up (fmha_det_timeouts_take)

UB_DEVICE int ld_acquire_gpu(const int* p) {
  int v;
  asm volatile("ld.acquire.gpu.global.b32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
UB_DEVICE void red_release_gpu_add(int* p, int v) {
  asm volatile("red.release.gpu.global.add.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// orders this thread's generic-proxy accesses of global memory with its async-proxy (bulk copy) accesses
UB_DEVICE void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }
UB_DEVICE unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// One thread: wait until the turn counter of a query tile reaches `turn` (the CTA's key tile index).  The wait is
// bounded: after ~10 s it gives up, counts a timeout and lets the caller add out of order rather than hang the GPU.
UB_DEVICE void det_wait_turn(const int* counter, int turn) {
  if (ld_acquire_gpu(counter) != turn) {
    const unsigned long long t0 = globaltimer_ns();
    unsigned int ns = 32;
    while (ld_acquire_gpu(counter) != turn) {
      __nanosleep(ns);
      ns = ns < 1024 ? 2 * ns : ns;
      if (globaltimer_ns() - t0 > 10000000000ull) {
        atomicAdd(&g_det_timeouts, 1u);
        break;
      }
    }
  }
  // the acquire made the previous key tile's reduction visible to this thread; the proxy fence orders it before the
  // reduction this thread issues next through the async proxy
  fence_proxy_async_global();
}

// ---- pre-pass: delta[b,h,q] = sum_d dO * O -----------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) fmha_delta_kernel(const T* __restrict__ dout, const T* __restrict__ out,
                                                           float* __restrict__ delta, int B, int H, int Lq, int D) {
  // 8 threads per (b, q, h) row of D elements; thread `part` sums the 8-element chunks part, part + 8
  const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long rowi = gid >> 3;
  const int part = (int)(gid & 7);
  const long long nrows = (long long)B * Lq * H;
  float acc = 0.f;
  if (rowi < nrows) {
    for (int ch = part; ch < D / 8; ch += 8) {
      float a[8], o[8];
      unpack<T>(ld_global_nc_v4(dout + rowi * D + ch * 8), a);
      unpack<T>(ld_global_nc_v4(out + rowi * D + ch * 8), o);
#pragma unroll
      for (int e = 0; e < 8; ++e) acc += a[e] * o[e];
    }
  }
  acc += __shfl_xor_sync(0xffffffffu, acc, 1);
  acc += __shfl_xor_sync(0xffffffffu, acc, 2);
  acc += __shfl_xor_sync(0xffffffffu, acc, 4);
  if (rowi < nrows && part == 0) {
    const long long hq = rowi % ((long long)Lq * H);
    const long long b = rowi / ((long long)Lq * H);
    const int q = (int)(hq / H), h = (int)(hq % H);
    delta[(b * H + h) * Lq + q] = acc;
  }
}

// ---- post-pass: dq = scale * fp32 accumulator, written through (batch, seq, head) strides -------------------------
template <typename T>
__global__ void __launch_bounds__(256) fmha_dq_convert_kernel(const float* __restrict__ acc, T* __restrict__ out, int H,
                                                                int Lq, int Lq_pad, int D, int DP, long long nvec, float scale,
                                                                long long sb, long long sl, long long sh) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  const int groups = D / 8;   // the accumulator rows are DP wide; columns D..DP-1 are not stored
  for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += stride) {
    // v enumerates [b][h][q][D / 8 groups of 8 columns]
    const int part = (int)(v % groups);
    const long long row = v / groups;
    const int q = (int)(row % Lq);
    const long long bh = row / Lq;
    const int h = (int)(bh % H);
    const long long b = bh / H;
    const float4* src = reinterpret_cast<const float4*>(acc + ((bh * Lq_pad + q) * DP + dq_swz_col(q, part * 8)));
    const float4 x0 = src[0], x1 = src[1];
    const float x[8] = {x0.x * scale, x0.y * scale, x0.z * scale, x0.w * scale,
                        x1.x * scale, x1.y * scale, x1.z * scale, x1.w * scale};
    st_global_v4(out + b * sb + (long long)q * sl + (long long)h * sh + part * 8, pack<T>(x));
  }
}

// ---- main kernel ----------------------------------------------------------------------------------------------
// kLogits: the forward also returned z, and dz (fmha_api.h) is added to dS before it is packed, so that the dK operand,
// the dQ tile and the dBias store all carry dS_total = P o (drop(dP) - delta) + dz
// kCausal: only queries >= key0 see the CTA's keys, so the query-tile loop starts at i0 = key0 / 64 (kBM == kBN: tile i0
// is the diagonal one, where P = dS = 0 at key > query through an additive -inf, as the future mask gives).  Stages and
// mbarrier phases count from i0.  A CTA with key0 >= Lq has no query tile: it loads nothing and stores dK = dV = 0.
// dBias above the diagonal is exactly 0: with a per-batch bias (ds_buf == dbias) the CTA stores a zero tile for each
// skipped query tile i < i0; with a shared bias the reduction kernel writes the zeros and never reads those tiles.
// kDet (deterministic mode, bp.dq_turn set): the key tiles add their dQ shares into query tile i strictly in ascending
// key-tile order j, so dQ_i = ((0 + dQ_i^0) + dQ_i^1) + ... whatever the schedule.  Before its reduction, thread 0 of
// key tile j waits until the turn counter of (b, h, i) is j; after the reduction has completed it increments the
// counter.  The chain has no gap: every key tile walks every query tile, and in causal mode key tile j starts at query
// tile j, so the tiles that reach query tile i are exactly 0 .. min(i, n_kt - 1).  Forward progress: a CTA only ever
// waits on the CTA of the same (b, h) with the next lower blockIdx.x, whose linear block index is lower, so the
// hardware dispatched it before this one; by induction down to key tile 0, which never waits, the chain completes.
// The wait is at the last point, with the dQ tile already staged, so a CTA does not hold up the chain while it
// computes.  dK, dV and dS are computed exactly as in the default mode.
template <typename T, int DP, bool kLogits, bool kCausal, bool kDet = false>
__global__ void __launch_bounds__(kBwdThreads, DP == 64 ? 2 : 1) fmha_bwd_kernel(const __grid_constant__ FmhaBwdParams bp) {
  static_assert(!(kLogits && kCausal), "causal attention is not instantiated in logits mode");
  using C = BwdCfg<DP, kLogits>;
  constexpr uint32_t kOffK = C::kOffK, kOffV = C::kOffV, kOffQ = C::kOffQ, kOffDO = C::kOffDO, kOffDS = C::kOffDS,
                     kOffDQ = C::kOffDQ, kOffStats = C::kOffStats, kOffBar = C::kOffBar, kTile = C::kTile;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_base = smem_u32(smem_raw);
  const uint32_t smem_base = (raw_base + 1023u) & ~1023u;   // 128-byte swizzle: tiles must be 1024-byte aligned
  uint8_t* smem = smem_raw + (smem_base - raw_base);
  const FmhaFwdParams& p = bp.f;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, c = lane & 3;
  const int key0 = blockIdx.x * kBN, h = blockIdx.y, b = blockIdx.z;
  const uint32_t bar_kv = smem_base + kOffBar, bar_in0 = smem_base + kOffBar + 8;   // + 8 * stage
  const bool has_bias = p.bias != nullptr;
  const bool drop = p.p_drop > 0.f && p.drop_bits != nullptr;
  const int n_qtiles = (p.Lq + kBM - 1) / kBM;
  const int Lq_pad = n_qtiles * kBM;
  // first query tile: causal CTAs skip the tiles whose queries all precede key0 (i0 == n_qtiles: none is left)
  const int i0 = kCausal ? min(key0 / kBM, n_qtiles) : 0;
  const long long bh = (long long)b * p.H + h;
  const int bias_nb = (p.bias_batch > 1 ? b : 0) * p.H + h;
  const int words_per_row = (p.Lk + 31) / 32;
  // the TMA unit counts the zero-filled columns D..DP-1 of a box as transferred bytes
  auto load_tile = [&](int i) {   // one thread: Q_i, dO_i (and the bias and dz tiles) -> stage (i - i0) & 1
    const uint32_t st = (uint32_t)((i - i0) & 1), bar = bar_in0 + 8u * st;
    mbar_expect_tx(bar, 2 * kTile + (has_bias ? 8192u : 0u) + (kLogits ? 8192u : 0u));
#pragma unroll
    for (int x = 0; x < C::kBoxes; ++x) {   // column boxes 0..63 and 64..127
      tma_load_4d(smem_base + kOffQ + st * kTile + x * 8192, &p.sw_q, 64 * x, h, i * kBM, b, bar);
      tma_load_4d(smem_base + kOffDO + st * kTile + x * 8192, &bp.sw_do, 64 * x, h, i * kBM, b, bar);
    }
    if (has_bias) tma_load_3d(smem_base + kOffDS + st * 8192, &p.sw_bias, key0, i * kBM, bias_nb, bar);
    if constexpr (kLogits) tma_load_3d(smem_base + C::kOffDZ + st * 8192, &bp.sw_dz, key0, i * kBM, (int)bh, bar);
  };
  // causal: the keep words (key0 >> 5) + {0, 1} are read for query tiles i >= key0 / 64 only; the causal forward of such
  // a tile walked the keys up to at least i * 64 + 63 >= key0 + 63, so it wrote both words of every row it read here
  auto load_stats = [&](int i) {  // all threads: LSE (log2 units, +inf = row contributes nothing), delta, keep bits
    uint8_t* s = smem + kOffStats + ((i - i0) & 1) * 1024;
    const int q = i * kBM + (tid & 63);
    const bool ok = q < p.Lq;
    if (tid < 64) {
      const float lse = ok ? p.lse[bh * p.Lq + q] : -CUDART_INF_F;
      reinterpret_cast<float*>(s)[tid] = lse == -CUDART_INF_F ? CUDART_INF_F : lse * 1.4426950408889634f;
    } else {
      reinterpret_cast<float*>(s + 256)[tid - 64] = ok ? bp.delta[bh * p.Lq + q] : 0.f;
    }
    if (drop) {   // bits[w][q]: word w of the tile's two for query q, so that queries q, q + 1 are one 8-byte load
      const int qb = i * kBM + (tid >> 1), wi = (key0 >> 5) + (tid & 1);
      reinterpret_cast<uint32_t*>(s + 512)[(tid & 1) * 64 + (tid >> 1)] =
          (qb < p.Lq && wi < words_per_row) ? p.drop_bits[(bh * p.Lq + qb) * words_per_row + wi] : 0xffffffffu;
    }
  };

  const bool any_q = !kCausal || i0 < n_qtiles;   // a copy must not outlive the CTA: no query tile, no load
  if (tid == 0) {
    mbar_init(bar_kv, 1);
    mbar_init(bar_in0, 1);
    mbar_init(bar_in0 + 8, 1);
    fence_mbarrier_init();
    if (any_q) {
      mbar_expect_tx(bar_kv, 2 * kTile);
#pragma unroll
      for (int x = 0; x < C::kBoxes; ++x) {
        tma_load_4d(smem_base + kOffK + x * 8192, &p.sw_k, 64 * x, h, key0, b, bar_kv);
        tma_load_4d(smem_base + kOffV + x * 8192, &p.sw_v, 64 * x, h, key0, b, bar_kv);
      }
      load_tile(i0);
    }
  }
  if (any_q) load_stats(i0);
  // causal, per-batch dBias: the skipped tiles (i < i0, every key above every query) are zero.  The first 8 KB of the
  // dQ staging tile are zeroed and stored over each of them; the first dQ tile is written after the bulk_wait_read of
  // the loop's first barrier (A), when the stores have read it.
  const bool zero_ds = kCausal && i0 > 0 && bp.ds_buf != nullptr && bp.ds_buf == bp.dbias;
  if (zero_ds) {
    uint4* zt = reinterpret_cast<uint4*>(smem + kOffDQ);
#pragma unroll
    for (int e = 0; e < 8192 / 16 / kBwdThreads; ++e) zt[e * kBwdThreads + tid] = make_uint4(0u, 0u, 0u, 0u);
    fence_proxy_async_smem();
  }

  // my two keys (accumulator rows) and their additive masks
  const int kl0 = warp * 16 + g, kl1 = kl0 + 8;
  const int kr0 = key0 + kl0, kr1 = key0 + kl1;
  const float kadd0 = (kr0 >= p.Lk || (p.kpm != nullptr && p.kpm[(long long)b * p.Lk + kr0] != 0)) ? -CUDART_INF_F : 0.f;
  const float kadd1 = (kr1 >= p.Lk || (p.kpm != nullptr && p.kpm[(long long)b * p.Lk + kr1] != 0)) ? -CUDART_INF_F : 0.f;
  // keep-bit positions of my keys inside their 32-key word (word (warp >> 1) of the tile's two)
  const int kk0 = 16 * (warp & 1) + g, kk1 = kk0 + 8;
  const int bit0 = (kk0 & 1) * 16 + (kk0 >> 1), bit1 = (kk1 & 1) * 16 + (kk1 >> 1);
  const int kword = warp >> 1;

  const float keep_scale = p.p_drop > 0.f ? dropout_keep_scale14(dropout_thresh14(p.p_drop)) : 1.f;
  constexpr float kLog2e = 1.4426950408889634f;
  // lane -> address of its row for ldmatrix / stmatrix (.trans) of a 16-query x 16-key block of the [q][key] tile
  const int lm = lane >> 3, lj = lane & 7;
  const int ld_q = (lm >> 1) * 8 + lj, ld_chunk = 2 * warp + (lm & 1);

  float dv[DP / 2], dk[DP / 2];
#pragma unroll
  for (int e = 0; e < DP / 2; ++e) {
    dv[e] = 0.f;
    dk[e] = 0.f;
  }
  __syncthreads();   // barriers initialised, stats of tile i0 in shared memory
  if (zero_ds && tid == 0) {
    for (int i = 0; i < i0; ++i) tma_store_3d(&bp.sw_ds, key0, i * kBM, (int)bh, smem_base + kOffDQ);
    bulk_commit();
  }
  if (any_q) mbar_wait(bar_kv, 0);

  for (int i = i0; i < n_qtiles; ++i) {
    const uint32_t st = (uint32_t)((i - i0) & 1);
    __syncthreads();   // (A) tile i-1 is finished by every thread: its stage, stats and dQ staging may be reused
    if (tid == 0) {
      bulk_wait_read();   // the dS store and the dQ reduction of tile i-1 have read shared memory
      if (i + 1 < n_qtiles) load_tile(i + 1);
    }
    if (i + 1 < n_qtiles) load_stats(i + 1);
    mbar_wait(bar_in0 + 8u * st, (uint32_t)(((i - i0) >> 1) & 1));

    const uint32_t sQ = smem_base + kOffQ + st * kTile, sDO = smem_base + kOffDO + st * kTile;
    const uint32_t sDS = smem_base + kOffDS + st * 8192;
    float s[32], dp[32];
    wgmma_fence();
    // k-step kk: box kk / 4, +32 bytes per step inside the box
#pragma unroll
    for (int kk = 0; kk < DP / 16; ++kk) {
      const uint32_t off = (kk >> 2) * 8192 + (kk & 3) * 32;
      wgmma_m64n64_ss<T, 0>(s, make_desc_sw128(smem_base + kOffK + off), make_desc_sw128(sQ + off), kk > 0 ? 1u : 0u);
    }
    wgmma_commit();   // S^T and dP^T are separate groups: P is formed while dP^T is still on the tensor cores
#pragma unroll
    for (int kk = 0; kk < DP / 16; ++kk) {
      const uint32_t off = (kk >> 2) * 8192 + (kk & 3) * 32;
      wgmma_m64n64_ss<T, 0>(dp, make_desc_sw128(smem_base + kOffV + off), make_desc_sw128(sDO + off), kk > 0 ? 1u : 0u);
    }
    wgmma_commit();

    const uint8_t* stats = smem + kOffStats + st * 1024;
    const float* lse2_s = reinterpret_cast<const float*>(stats);
    const float* delta_s = reinterpret_cast<const float*>(stats + 256);
    const uint32_t* bits_s = reinterpret_cast<const uint32_t*>(stats + 512) + 64 * kword;

    // ---- P^T = exp2(logits - LSE), in place over S^T ------------------------------------------------------------
    wgmma_wait<1>();
    fence_operands(s);
#pragma unroll
    for (int sb = 0; sb < 4; ++sb) {
      uint32_t bias_r[4] = {0u, 0u, 0u, 0u};
      const uint32_t addr = sDS + sw128_off(16 * sb + ld_q, ld_chunk);
      if (has_bias) ldmatrix_x4_trans(addr, bias_r);
#pragma unroll
      for (int r = 0; r < 4; ++r) {   // r: rows (key kl0 or kl1) x query half (16sb + 2c or 16sb + 8 + 2c)
        const int e = 8 * sb + 2 * r;
        const int ql = 16 * sb + 8 * (r >> 1) + 2 * c;
        const float2 bb = has_bias ? bwd_unpack2<T>(bias_r[r]) : make_float2(0.f, 0.f);
        const float ka = (r & 1) ? kadd1 : kadd0;
        const float2 l2 = *reinterpret_cast<const float2*>(lse2_s + ql);
        float ka0 = ka, ka1 = ka;
        if constexpr (kCausal) {   // diagonal tile (key0 == i0 * 64): local key index > local query index is future
          const int kl = (r & 1) ? kl1 : kl0;
          if (i == i0) {
            if (kl > ql) ka0 = -CUDART_INF_F;
            if (kl > ql + 1) ka1 = -CUDART_INF_F;
          }
        }
        const float x0 = fmaf(s[e], p.scale, bb.x + ka0), x1 = fmaf(s[e + 1], p.scale, bb.y + ka1);
        s[e] = ex2_approx(fmaf(x0, kLog2e, -l2.x));
        s[e + 1] = ex2_approx(fmaf(x1, kLog2e, -l2.y));
      }
    }

    // ---- dS^T = P o (drop(dP) - delta) (+ dz), both packed into register A operands ----------------------------------
    wgmma_wait<0>();
    fence_operands(s);
    fence_operands(dp);
    uint32_t pa[4][4], da[4][4];   // [16-query block][A-operand register] of drop(P)^T and dS^T
#pragma unroll
    for (int sb = 0; sb < 4; ++sb) {
      uint32_t dz_r[4];   // dz has the bias tile's layout
      if constexpr (kLogits) ldmatrix_x4_trans(smem_base + C::kOffDZ + st * 8192 + sw128_off(16 * sb + ld_q, ld_chunk), dz_r);
      // keep bits of my queries 16sb + 2c, +1 and 16sb + 8 + 2c, +1 in word kword: two 8-byte loads, read once per
      // tile and applied below as selects
      uint2 kb[2];
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
        kb[hh] = drop ? *reinterpret_cast<const uint2*>(bits_s + 16 * sb + 8 * hh + 2 * c) : make_uint2(~0u, ~0u);
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int e = 8 * sb + 2 * r;
        const int ql = 16 * sb + 8 * (r >> 1) + 2 * c;
        const int bit = (r & 1) ? bit1 : bit0;
        const uint2 w = kb[r >> 1];   // queries ql, ql + 1
        const bool k0 = (w.x >> bit) & 1u, k1 = (w.y >> bit) & 1u;
        const float2 dl = *reinterpret_cast<const float2*>(delta_s + ql);
        const float p0 = s[e], p1 = s[e + 1];
        float ds0 = p0 * (dp[e] * (k0 ? keep_scale : 0.f) - dl.x);
        float ds1 = p1 * (dp[e + 1] * (k1 ? keep_scale : 0.f) - dl.y);
        if constexpr (kLogits) {
          const float2 dz = bwd_unpack2<T>(dz_r[r]);
          ds0 += dz.x;
          ds1 += dz.y;
        }
        pa[sb][r] = bwd_pack2<T>(k0 ? p0 : 0.f, k1 ? p1 : 0.f);   // keep_scale is applied to dV in the epilogue
        da[sb][r] = bwd_pack2<T>(ds0, ds1);                         // the softmax scale to dQ / dK at read-out
      }
    }

    // ---- dS -> shared memory as [q][key] (in place over the bias tile: each warp rewrites exactly what it read);
    //      before the products below, which read the same registers asynchronously ---------------------------------
#pragma unroll
    for (int sb = 0; sb < 4; ++sb) stmatrix_x4_trans(sDS + sw128_off(16 * sb + ld_q, ld_chunk), da[sb]);
    fence_proxy_async_smem();

    // ---- dV += drop(P)^T dO, dK += dS^T Q ---------------------------------------------------------------------
    wgmma_fence();
    // 16 queries = 16 rows of 128 bytes per step; at DP = 128 the descriptor steps to the second box through its LBO
#pragma unroll
    for (int sb = 0; sb < 4; ++sb) {
      if constexpr (DP == 64) wgmma_m64n64_rs<T, 1>(dv, pa[sb], make_desc_sw128(sDO + sb * 2048), 1u);
      else wgmma_m64n128_rs<T, 1>(dv, pa[sb], make_desc_sw128_mn(sDO + sb * 2048, 8192), 1u);
    }
#pragma unroll
    for (int sb = 0; sb < 4; ++sb) {
      if constexpr (DP == 64) wgmma_m64n64_rs<T, 1>(dk, da[sb], make_desc_sw128(sQ + sb * 2048), 1u);
      else wgmma_m64n128_rs<T, 1>(dk, da[sb], make_desc_sw128_mn(sQ + sb * 2048, 8192), 1u);
    }
    wgmma_commit();
    __syncthreads();   // (B) the whole dS tile is in shared memory

    // ---- dQ = dS K, one 64-column box of K at a time ------------------------------------------------------------
    float* dq_s = reinterpret_cast<float*>(smem + kOffDQ);
#pragma unroll
    for (int x = 0; x < C::kBoxes; ++x) {
      float dq[32];
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kBN / 16; ++kk)
        wgmma_m64n64_ss<T, 1>(dq, make_desc_sw128(sDS + kk * 32), make_desc_sw128(smem_base + kOffK + x * 8192 + kk * 2048),
                              kk > 0 ? 1u : 0u);
      wgmma_commit();
      if (x == 0 && tid == 0 && bp.ds_buf != nullptr) {   // bias gradient: the dS tile leaves through one TMA store
        tma_store_3d(&bp.sw_ds, key0, i * kBM, (int)bh, sDS);
        bulk_commit();
      }
      wgmma_wait<0>();
      if (x == 0) {
        fence_operands(dv);
        fence_operands(dk);
      }
      fence_operands(dq);
      // rows kl0 and kl1 are both = g (mod 8), and so are the global rows i * 64 + kl0 / kl1
#pragma unroll
      for (int n = 0; n < 8; ++n) {
        const int col = dq_swz_col(g, 64 * x + 8 * n + 2 * c);
        *reinterpret_cast<float2*>(dq_s + kl0 * DP + col) = make_float2(dq[4 * n], dq[4 * n + 1]);
        *reinterpret_cast<float2*>(dq_s + kl1 * DP + col) = make_float2(dq[4 * n + 2], dq[4 * n + 3]);
      }
    }
    fence_proxy_async_smem();
    __syncthreads();   // (C) the dQ tile is in shared memory
    if (tid == 0) {
      if constexpr (kDet) det_wait_turn(bp.dq_turn + bh * n_qtiles + i, (int)blockIdx.x);
      bulk_reduce_add_f32(bp.dq_acc + (bh * Lq_pad + (long long)i * kBM) * DP, smem_base + kOffDQ, kBM * DP * 4);
      bulk_commit();
      if constexpr (kDet) {
        bulk_wait_all();             // the reduction's writes are performed (not only its reads of shared memory) ...
        fence_proxy_async_global();  // ... and ordered before the generic-proxy release that passes the turn on
        red_release_gpu_add(bp.dq_turn + bh * n_qtiles + i, 1);
      }
    }
  }
  if (tid == 0) bulk_wait_all();   // shared memory must outlive the last store's and reduction's reads

  // ---- epilogue: dK_j, dV_j (rows = my two keys) ------------------------------------------------------------------
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const int key = half ? kr1 : kr0;
    if (key >= p.Lk) continue;
    T* dvg = reinterpret_cast<T*>(bp.dv) + (long long)b * bp.dv_sb + (long long)key * bp.dv_sl + (long long)h * bp.dv_sh;
    T* dkg = reinterpret_cast<T*>(bp.dk) + (long long)b * bp.dk_sb + (long long)key * bp.dk_sl + (long long)h * bp.dk_sh;
#pragma unroll
    for (int n = 0; n < DP / 8; ++n) {
      if (8 * n >= p.D) continue;   // columns 8n + 2c, +1 exist iff 8n < D (D % 8 == 0)
      const int e = 4 * n + 2 * half;
      *reinterpret_cast<uint32_t*>(dvg + 8 * n + 2 * c) = bwd_pack2<T>(dv[e] * keep_scale, dv[e + 1] * keep_scale);
      *reinterpret_cast<uint32_t*>(dkg + 8 * n + 2 * c) = bwd_pack2<T>(dk[e] * p.scale, dk[e + 1] * p.scale);
    }
  }
}

// dbias[n] = sum_b ds[b, n] (fp32 accumulate), n over H * Lq * Lk in 16-byte vectors.  kCausal: a vector whose 8 keys
// are all past its query lies in a dS tile the causal kernel skipped (never written); it is stored as 0 unread.
template <typename T, bool kCausal>
__global__ void __launch_bounds__(256) fmha_dbias_reduce_kernel(const T* __restrict__ ds, T* __restrict__ dbias, int B,
                                                                  long long nvec, int Lq, int Lk) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += stride) {
    if constexpr (kCausal) {
      const long long vpr = Lk / 8;   // vectors per row (Lk % 8 == 0)
      const int key = (int)(v % vpr) * 8, q = (int)((v / vpr) % Lq);
      if (key > q) {
        st_global_v4(dbias + v * 8, Vec16{});
        continue;
      }
    }
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int b0 = 0; b0 < B; b0 += 4) {
      Vec16 in[4];
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (b0 + u < B) in[u] = ld_global_nc_v4(ds + ((long long)(b0 + u) * nvec + v) * 8);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (b0 + u < B) {
          float x[8];
          unpack<T>(in[u], x);
#pragma unroll
          for (int e = 0; e < 8; ++e) acc[e] += x[e];
        }
      }
    }
    st_global_v4(dbias + v * 8, pack<T>(acc));
  }
}

int device_sms() {
  static int sms = [] {
    int dev = 0, n = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    return n > 0 ? n : 132;
  }();
  return sms;
}

template <typename T, int DP>
void run_bwd(const FmhaBwdParams& bp, cudaStream_t stream) {
  const FmhaFwdParams& p = bp.f;
  const long long nrows = (long long)p.B * p.Lq * p.H;
  const int n_qt = (p.Lq + kBM - 1) / kBM;
  const bool det = bp.dq_turn != nullptr;   // the turn counters follow dq_acc: one memset zeroes both
  cudaMemsetAsync(bp.dq_acc, 0, (size_t)p.B * p.H * n_qt * (kBM * DP * sizeof(float) + (det ? sizeof(int) : 0)), stream);
  fmha_delta_kernel<T><<<(unsigned)((nrows * 8 + 255) / 256), 256, 0, stream>>>(
      reinterpret_cast<const T*>(bp.dout), reinterpret_cast<const T*>(p.out), bp.delta, p.B, p.H, p.Lq, p.D);
  dim3 grid((p.Lk + kBN - 1) / kBN, p.H, p.B);
  auto run = [&](auto kern, uint32_t smem_bytes) {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes);
    kern<<<grid, kBwdThreads, smem_bytes, stream>>>(bp);
  };
  // causal + logits is refused by the binding (fmha_bind.cpp)
  if (det) {
    if (bp.dlogits != nullptr) run(fmha_bwd_kernel<T, DP, true, false, true>, BwdCfg<DP, true>::kSmemBytes);
    else if (p.causal) run(fmha_bwd_kernel<T, DP, false, true, true>, BwdCfg<DP, false>::kSmemBytes);
    else run(fmha_bwd_kernel<T, DP, false, false, true>, BwdCfg<DP, false>::kSmemBytes);
  } else if (bp.dlogits != nullptr) run(fmha_bwd_kernel<T, DP, true, false>, BwdCfg<DP, true>::kSmemBytes);
  else if (p.causal) run(fmha_bwd_kernel<T, DP, false, true>, BwdCfg<DP, false>::kSmemBytes);
  else run(fmha_bwd_kernel<T, DP, false, false>, BwdCfg<DP, false>::kSmemBytes);
  const long long cap = (long long)device_sms() * 16;
  if (bp.ds_buf != nullptr && bp.dbias != bp.ds_buf) {
    const long long nv = (long long)p.H * p.Lq * p.Lk / 8;
    const long long rb = std::min((nv + 255) / 256, cap);
    auto reduce = p.causal ? fmha_dbias_reduce_kernel<T, true> : fmha_dbias_reduce_kernel<T, false>;
    reduce<<<(unsigned)rb, 256, 0, stream>>>(reinterpret_cast<const T*>(bp.ds_buf), reinterpret_cast<T*>(bp.dbias), p.B,
                                             nv, p.Lq, p.Lk);
  }
  const long long nvec = nrows * (p.D / 8);
  const long long blocks = std::min((nvec + 255) / 256, cap);
  fmha_dq_convert_kernel<T><<<(unsigned)blocks, 256, 0, stream>>>(bp.dq_acc, reinterpret_cast<T*>(bp.dq), p.H, p.Lq,
                                                                  n_qt * kBM, p.D, DP, nvec, p.scale, bp.dq_sb, bp.dq_sl,
                                                                  bp.dq_sh);
}

}  // namespace

void launch_fmha_bwd(const FmhaBwdParams& bp, cudaStream_t stream) {
  if (bp.f.D <= 64) {
    if (bp.f.is_bf16) run_bwd<__nv_bfloat16, 64>(bp, stream);
    else run_bwd<__half, 64>(bp, stream);
  } else {
    if (bp.f.is_bf16) run_bwd<__nv_bfloat16, 128>(bp, stream);
    else run_bwd<__half, 128>(bp, stream);
  }
}

unsigned int fmha_det_timeouts_take() {
  unsigned int n = 0;
  const unsigned int zero = 0;
  cudaDeviceSynchronize();   // every backward launched so far has finished counting
  cudaMemcpyFromSymbol(&n, g_det_timeouts, sizeof(n));
  cudaMemcpyToSymbol(g_det_timeouts, &zero, sizeof(zero));
  return n;
}

}  // namespace ub
