// LayerNorm / RMSNorm forward + single-pass backward, and the fused
// "bias + dropout + residual + LayerNorm" block epilogue, for sm_90a.
//
// Replaces reference csrc/layernorm/layernorm.cu:25-148, layernorm_backward.cu:130-247, csrc/rmsnorm/rmsnorm.cu:25-125,
// rmsnorm_backward.cu:108-196:
//   * any hidden size that is a multiple of the 16-byte vector width (reference: 16 fixed sizes);
//   * a row is owned by a group of TPR threads (TPR = 1..256, power of two, picked from the hidden
//     size) that keeps the whole row in registers: VPT 16-byte vectors per thread; groups of <= 32
//     threads reduce with shuffles only;
//   * backward reads x and dy ONCE and emits dx plus per-CTA partial dgamma/dbeta (fp32), which a
//     small second kernel reduces deterministically (reference: x, dy read twice + 2 extra kernels);
//   * fp32 statistics, biased variance, rstd = rsqrt(var + eps).
#include <algorithm>
#include <type_traits>

#include "../api.h"
#include "../common.cuh"

namespace ub {

constexpr int kNormThreads = 256;

template <typename T>
UB_DEVICE Vec16 ldv(const T* p) { return ld_global_v4(p); }

// Reduce `v` over the TPR threads that own a row. TPR <= 32: shuffles; else via shared memory.
// `scratch` holds (kNormThreads/32) floats per reduced quantity slot.
template <int NVAL>
UB_DEVICE void group_sum(float (&v)[NVAL], int tpr, float* scratch) {
  const int lim = tpr < 32 ? tpr : 32;
#pragma unroll
  for (int k = 0; k < NVAL; ++k) {
    for (int o = lim >> 1; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
  }
  if (tpr > 32) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wpg = tpr >> 5;                 // warps per group
    const int gfirst = (warp / wpg) * wpg;    // first warp of my group
    __syncthreads();
    if (lane == 0) {
#pragma unroll
      for (int k = 0; k < NVAL; ++k) scratch[k * 8 + warp] = v[k];
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < NVAL; ++k) {
      float s = 0.f;
      for (int w = 0; w < wpg; ++w) s += scratch[k * 8 + gfirst + w];
      v[k] = s;
    }
  }
}

struct NormGeom {
  int rows, cols, tpr, nvec;  // nvec = cols / elems-per-vector
};

// ------------------------------------------------------------------------------------------------
// forward.  kRMS: RMSNorm (no mean / beta).  kFused: h = residual + dropout(x + bias) first.
// ------------------------------------------------------------------------------------------------
template <typename T, int VPT, bool kRMS, bool kFused>
__global__ void __launch_bounds__(kNormThreads) norm_fwd_kernel(
    const T* __restrict__ x, const T* __restrict__ gamma, const T* __restrict__ beta, T* __restrict__ y,
    float* __restrict__ mean_out, float* __restrict__ rstd_out, NormGeom g, float eps,
    // fused-only arguments
    const T* __restrict__ bias, const T* __restrict__ residual, T* __restrict__ summed, float p, float keep_scale,
    unsigned long long seed, unsigned long long offset) {
  constexpr int EPV = VecTraits<T>::kElems;
  __shared__ float scratch[2 * 8];
  const int tpr = g.tpr;
  const int rows_per_cta = kNormThreads / tpr;
  const int grp = threadIdx.x / tpr, j = threadIdx.x % tpr;
  const float inv_cols = 1.f / (float)g.cols;
  const uint32_t thresh = kFused ? dropout_thresh16(p) : 0u;

  // per-thread column slice of gamma / beta / bias (fixed for all rows)
  float gam[VPT][EPV], bet[VPT][EPV], bia[VPT][EPV];
#pragma unroll
  for (int k = 0; k < VPT; ++k) {
    const int vi = j + k * tpr;
    if (vi < g.nvec) {
      unpack<T>(ldv(gamma + vi * EPV), gam[k]);
      if (!kRMS) unpack<T>(ldv(beta + vi * EPV), bet[k]);
      if (kFused && bias != nullptr) unpack<T>(ldv(bias + vi * EPV), bia[k]);
    }
    if (!(kFused && bias != nullptr)) {
#pragma unroll
      for (int e = 0; e < EPV; ++e) bia[k][e] = 0.f;
    }
  }

  const int nrow_iters = (g.rows + gridDim.x * rows_per_cta - 1) / (gridDim.x * rows_per_cta);
  for (int it = 0; it < nrow_iters; ++it) {
    const int row = (it * gridDim.x + blockIdx.x) * rows_per_cta + grp;
    const bool active = row < g.rows;
    float xs[VPT][EPV];
    float acc[1] = {0.f};
#pragma unroll
    for (int k = 0; k < VPT; ++k) {
      const int vi = j + k * tpr;
      if (active && vi < g.nvec) {
        const size_t off = (size_t)row * g.cols + (size_t)vi * EPV;
        unpack<T>(ld_global_nc_v4(x + off), xs[k]);
        if (kFused) {
          float res[EPV];
          unpack<T>(ld_global_nc_v4(residual + off), res);
          uint32_t keep = 0xffu;
          if (p > 0.f) keep = dropout_keep8(seed, offset, off / 8, thresh);
#pragma unroll
          for (int e = 0; e < EPV; ++e) {
            const float h = (xs[k][e] + bia[k][e]) * (((keep >> e) & 1u) ? keep_scale : 0.f);
            // round the sum to T first: backward and the pre-LN consumer see exactly this value
            xs[k][e] = to_f32<T>(from_f32<T>(res[e] + h));
          }
          st_global_v4(summed + off, pack<T>(xs[k]));
        }
#pragma unroll
        for (int e = 0; e < EPV; ++e) acc[0] += kRMS ? xs[k][e] * xs[k][e] : xs[k][e];
      } else {
#pragma unroll
        for (int e = 0; e < EPV; ++e) xs[k][e] = 0.f;
      }
    }
    group_sum<1>(acc, tpr, scratch);
    float mu = 0.f, rs;
    if (kRMS) {
      rs = rsqrtf(acc[0] * inv_cols + eps);
    } else {
      mu = acc[0] * inv_cols;
      float var[1] = {0.f};
#pragma unroll
      for (int k = 0; k < VPT; ++k) {
        if (j + k * tpr < g.nvec) {
#pragma unroll
          for (int e = 0; e < EPV; ++e) {
            const float d = xs[k][e] - mu;
            var[0] += d * d;
          }
        }
      }
      group_sum<1>(var, tpr, scratch);
      rs = rsqrtf(var[0] * inv_cols + eps);
    }
    if (active) {
      if (j == 0) {
        if (!kRMS) mean_out[row] = mu;
        rstd_out[row] = rs;
      }
#pragma unroll
      for (int k = 0; k < VPT; ++k) {
        const int vi = j + k * tpr;
        if (vi < g.nvec) {
          float o[EPV];
#pragma unroll
          for (int e = 0; e < EPV; ++e) {
            const float xh = (xs[k][e] - mu) * rs;
            o[e] = kRMS ? xh * gam[k][e] : xh * gam[k][e] + bet[k][e];
          }
          st_global_v4(y + (size_t)row * g.cols + (size_t)vi * EPV, pack<T>(o));
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// backward: dx (+ optional dropout-masked copy for the fused op) and per-CTA dgamma/dbeta partials
// ------------------------------------------------------------------------------------------------
template <typename T, int VPT, bool kRMS, bool kFused, bool kDet = false>
__global__ void __launch_bounds__(kNormThreads) norm_bwd_kernel(
    const T* __restrict__ dy, const T* __restrict__ x, const float* __restrict__ mean,
    const float* __restrict__ rstd, const T* __restrict__ gamma, T* __restrict__ dx, float* __restrict__ dgamma_part,
    float* __restrict__ dbeta_part, NormGeom g,
    // fused-only: dx_drop = keep ? dx * keep_scale : 0
    T* __restrict__ dx_drop, float p, float keep_scale, unsigned long long seed, unsigned long long offset) {
  constexpr int EPV = VecTraits<T>::kElems;
  extern __shared__ float sm_acc[];  // [2][cols] cross-group accumulators (dgamma, dbeta)
  __shared__ float scratch[2 * 8];
  const int tpr = g.tpr;
  const int rows_per_cta = kNormThreads / tpr;
  const int grp = threadIdx.x / tpr, j = threadIdx.x % tpr;
  const float inv_cols = 1.f / (float)g.cols;
  const uint32_t thresh = kFused ? dropout_thresh16(p) : 0u;

  for (int c = threadIdx.x; c < (kRMS ? 1 : 2) * g.cols; c += kNormThreads) sm_acc[c] = 0.f;

  float gam[VPT][EPV], dg[VPT][EPV], db[VPT][EPV];
#pragma unroll
  for (int k = 0; k < VPT; ++k) {
    const int vi = j + k * tpr;
    if (vi < g.nvec) unpack<T>(ldv(gamma + vi * EPV), gam[k]);
#pragma unroll
    for (int e = 0; e < EPV; ++e) dg[k][e] = db[k][e] = 0.f;
  }

  const int nrow_iters = (g.rows + gridDim.x * rows_per_cta - 1) / (gridDim.x * rows_per_cta);
  for (int it = 0; it < nrow_iters; ++it) {
    const int row = (it * gridDim.x + blockIdx.x) * rows_per_cta + grp;
    const bool active = row < g.rows;
    const float mu = (active && !kRMS) ? mean[row] : 0.f;
    const float rs = active ? rstd[row] : 0.f;
    float xh[VPT][EPV], gy[VPT][EPV];
    float s[2] = {0.f, 0.f};
#pragma unroll
    for (int k = 0; k < VPT; ++k) {
      const int vi = j + k * tpr;
      if (active && vi < g.nvec) {
        const size_t off = (size_t)row * g.cols + (size_t)vi * EPV;
        float xv[EPV], dv[EPV];
        unpack<T>(ld_global_nc_v4(x + off), xv);
        unpack<T>(ld_global_nc_v4(dy + off), dv);
#pragma unroll
        for (int e = 0; e < EPV; ++e) {
          xh[k][e] = (xv[e] - mu) * rs;
          gy[k][e] = dv[e] * gam[k][e];
          s[0] += gy[k][e];
          s[1] += gy[k][e] * xh[k][e];
          dg[k][e] += dv[e] * xh[k][e];
          if (!kRMS) db[k][e] += dv[e];
        }
      } else {
#pragma unroll
        for (int e = 0; e < EPV; ++e) xh[k][e] = gy[k][e] = 0.f;
      }
    }
    group_sum<2>(s, tpr, scratch);
    const float m1 = kRMS ? 0.f : s[0] * inv_cols, m2 = s[1] * inv_cols;
    if (active) {
#pragma unroll
      for (int k = 0; k < VPT; ++k) {
        const int vi = j + k * tpr;
        if (vi < g.nvec) {
          const size_t off = (size_t)row * g.cols + (size_t)vi * EPV;
          float o[EPV];
#pragma unroll
          for (int e = 0; e < EPV; ++e) o[e] = rs * (gy[k][e] - m1 - xh[k][e] * m2);
          st_global_v4(dx + off, pack<T>(o));
          if (kFused) {
            uint32_t keep = 0xffu;
            if (p > 0.f) keep = dropout_keep8(seed, offset, off / 8, thresh);
#pragma unroll
            for (int e = 0; e < EPV; ++e) o[e] = ((keep >> e) & 1u) ? o[e] * keep_scale : 0.f;
            st_global_v4(dx_drop + off, pack<T>(o));
          }
        }
      }
    }
  }

  // combine the row groups of this CTA, then publish one fp32 partial row per CTA.  kDet: group 0, 1, ... add in turn
  // (each column belongs to one thread of a group), so the order is fixed; otherwise shared atomics in arrival order.
  __syncthreads();
  for (int r = 0; r < (kDet ? rows_per_cta : 1); ++r) {
    if (!kDet || grp == r) {
#pragma unroll
      for (int k = 0; k < VPT; ++k) {
        const int vi = j + k * tpr;
        if (vi < g.nvec) {
#pragma unroll
          for (int e = 0; e < EPV; ++e) {
            if constexpr (kDet) {
              sm_acc[vi * EPV + e] += dg[k][e];
              if (!kRMS) sm_acc[g.cols + vi * EPV + e] += db[k][e];
            } else {
              atomicAdd(&sm_acc[vi * EPV + e], dg[k][e]);
              if (!kRMS) atomicAdd(&sm_acc[g.cols + vi * EPV + e], db[k][e]);
            }
          }
        }
      }
    }
    __syncthreads();
  }
  for (int c = threadIdx.x; c < g.cols; c += kNormThreads) {
    dgamma_part[(size_t)blockIdx.x * g.cols + c] = sm_acc[c];
    if (!kRMS) dbeta_part[(size_t)blockIdx.x * g.cols + c] = sm_acc[g.cols + c];
  }
}

// partial rows -> dgamma / dbeta. block = (32 columns, 8 row slices)
template <typename T>
__global__ void __launch_bounds__(256) norm_param_grad_kernel(const float* __restrict__ dg_part,
                                                                const float* __restrict__ db_part, int parts,
                                                                int cols, T* __restrict__ dgamma,
                                                                T* __restrict__ dbeta, int acc_mask) {
  __shared__ float red[2][8][33];
  const int cx = threadIdx.x & 31, ry = threadIdx.x >> 5;
  const int col = blockIdx.x * 32 + cx;
  float a = 0.f, b = 0.f;
  if (col < cols) {
    for (int r = ry; r < parts; r += 8) {
      a += dg_part[(size_t)r * cols + col];
      if (db_part != nullptr) b += db_part[(size_t)r * cols + col];
    }
  }
  red[0][ry][cx] = a;
  red[1][ry][cx] = b;
  __syncthreads();
  if (ry == 0 && col < cols) {
    float sa = 0.f, sb = 0.f;
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      sa += red[0][r][cx];
      sb += red[1][r][cx];
    }
    if (acc_mask & 1) sa += to_f32<T>(dgamma[col]);
    dgamma[col] = from_f32<T>(sa);
    if (db_part != nullptr) {
      if (acc_mask & 2) sb += to_f32<T>(dbeta[col]);
      dbeta[col] = from_f32<T>(sb);
    }
  }
}

// ================================================================================================
// v2 kernels (rows of up to 384 16-byte vectors, i.e. every hidden size in practice).
//
// The v1 kernels above keep VPT vectors per thread, which for hidden = 768 costs 170 registers in
// the backward (dgamma/dbeta accumulators scale with VPT) -> 8 warps per SM and stop-and-go loads;
// ncu showed them at ~30 % of HBM bandwidth.  Here a thread owns exactly ONE vector column (so the
// accumulators are 8 floats each), a row is owned by ceil32(nvec) threads, and memory-level
// parallelism comes from R consecutive rows kept in flight per thread instead.
// ================================================================================================
constexpr int kNormV2Threads = 384;
constexpr int kNormStages = 4;  // bulk-copy input stages per CTA (<= ~25 KB each)
constexpr int kNormV2Warps = kNormV2Threads / 32;

struct NormGeom2 {
  int rows, cols, tpr, nvec, groups;  // blockDim.x = tpr * groups
};

template <int NVAL>
UB_DEVICE void group_sum2(float (&v)[NVAL], int tpr, float* scratch) {
  if (tpr >= 32) {  // whole warps: five unrolled butterfly steps (the runtime loop cost ~6 instructions per element)
#pragma unroll
    for (int k = 0; k < NVAL; ++k) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
    }
  } else {
#pragma unroll
    for (int k = 0; k < NVAL; ++k) {
      for (int o = tpr >> 1; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
    }
  }
  if (tpr > 32) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wpg = tpr >> 5;
    const int gfirst = (warp / wpg) * wpg;
    __syncthreads();
    if (lane == 0) {
#pragma unroll
      for (int k = 0; k < NVAL; ++k) scratch[k * kNormV2Warps + warp] = v[k];
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < NVAL; ++k) {
      float s = 0.f;
      for (int w = 0; w < wpg; ++w) s += scratch[k * kNormV2Warps + gfirst + w];
      v[k] = s;
    }
  }
}

template <typename T, int R, bool kRMS, bool kFused>
__global__ void __launch_bounds__(kNormV2Threads, 2) norm_fwd_v2_kernel(
    const T* __restrict__ x, const T* __restrict__ gamma, const T* __restrict__ beta, T* __restrict__ y,
    float* __restrict__ mean_out, float* __restrict__ rstd_out, NormGeom2 g, float eps,
    const T* __restrict__ bias, const T* __restrict__ residual, T* __restrict__ summed, float p, float keep_scale,
    unsigned long long seed, unsigned long long offset) {
  constexpr int EPV = VecTraits<T>::kElems;
  extern __shared__ __align__(128) uint8_t dyn_smem[];
  __shared__ float scratch[R * kNormV2Warps];
  const int tpr = g.tpr;
  const int grp = threadIdx.x / tpr, j = threadIdx.x - grp * tpr;
  const bool col_ok = j < g.nvec;
  const float inv_cols = 1.f / (float)g.cols;
  const uint32_t thresh = kFused ? dropout_thresh16(p) : 0u;

  // ---- input pipeline: tiles of (groups * R) consecutive rows arrive by bulk copy, kNormStages deep ----
  const int tile_rows = g.groups * R;
  const uint32_t row_bytes = (uint32_t)g.cols * (uint32_t)sizeof(T);
  const uint32_t tile_bytes = (uint32_t)tile_rows * row_bytes;
  const uint32_t stage_bytes = tile_bytes * (kFused ? 2u : 1u);
  const uint32_t stage_base = smem_addr_u32(dyn_smem);
  const uint32_t bar_base = stage_base + kNormStages * stage_bytes;
  const long long n_tiles = ((long long)g.rows + tile_rows - 1) / tile_rows;
  const int n_my = (int)((n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x);  // tiles blockIdx.x, +gridDim.x, ...
  auto issue = [&](int it) {  // one thread
    const uint32_t s = (uint32_t)(it % kNormStages);
    const long long trow0 = ((long long)it * gridDim.x + blockIdx.x) * tile_rows;
    const long long left = (long long)g.rows - trow0;
    const uint32_t bytes = (uint32_t)(left < tile_rows ? left : tile_rows) * row_bytes;
    bulk_expect_tx(bar_base + s * 8, bytes * (kFused ? 2u : 1u));
    bulk_g2s(stage_base + s * stage_bytes, x + trow0 * g.cols, bytes, bar_base + s * 8);
    if (kFused) bulk_g2s(stage_base + s * stage_bytes + tile_bytes, residual + trow0 * g.cols, bytes, bar_base + s * 8);
  };
  if (threadIdx.x == 0) {
    for (int s = 0; s < kNormStages; ++s) bulk_bar_init(bar_base + s * 8, 1);
    bulk_bar_init_fence();
    for (int it = 0; it < kNormStages && it < n_my; ++it) issue(it);
  }

  float gam[EPV], bet[EPV], bia[EPV];
#pragma unroll
  for (int e = 0; e < EPV; ++e) gam[e] = bet[e] = bia[e] = 0.f;
  if (col_ok) {
    unpack<T>(ldv(gamma + j * EPV), gam);
    if (!kRMS) unpack<T>(ldv(beta + j * EPV), bet);
    if (kFused && bias != nullptr) unpack<T>(ldv(bias + j * EPV), bia);
  }
  __syncthreads();  // barrier objects are initialised before anyone waits on them

  for (int it = 0; it < n_my; ++it) {
    const int row0 = ((it * gridDim.x + blockIdx.x) * g.groups + grp) * R;
    const uint32_t s = (uint32_t)(it % kNormStages);
    bulk_wait(bar_base + s * 8, (uint32_t)((it / kNormStages) & 1));
    const uint8_t* st = dyn_smem + s * stage_bytes + (size_t)(grp * R) * row_bytes + (size_t)j * 16;
    Vec16 xv[R], rv[R];
#pragma unroll
    for (int i = 0; i < R; ++i) {
      if (col_ok && row0 + i < g.rows) {
        xv[i] = *reinterpret_cast<const Vec16*>(st + (size_t)i * row_bytes);
        if (kFused) rv[i] = *reinterpret_cast<const Vec16*>(st + tile_bytes + (size_t)i * row_bytes);
      }
    }
    __syncthreads();  // the stage has been copied out by everybody: refill it
    if (threadIdx.x == 0 && it + kNormStages < n_my) issue(it + kNormStages);
    float xs[R][EPV];
    float acc[R];
#pragma unroll
    for (int i = 0; i < R; ++i) {
      acc[i] = 0.f;
      if (col_ok && row0 + i < g.rows) {
        unpack<T>(xv[i], xs[i]);
        if (kFused) {
          const size_t off = (size_t)(row0 + i) * g.cols + (size_t)j * EPV;
          float res[EPV];
          unpack<T>(rv[i], res);
          uint32_t keep = 0xffu;
          if (p > 0.f) keep = dropout_keep8(seed, offset, off / 8, thresh);
#pragma unroll
          for (int e = 0; e < EPV; ++e) {
            const float h = (xs[i][e] + bia[e]) * (((keep >> e) & 1u) ? keep_scale : 0.f);
            // round the sum to T first: backward and the pre-LN consumer see exactly this value
            xs[i][e] = to_f32<T>(from_f32<T>(res[e] + h));
          }
          st_global_v4(summed + off, pack<T>(xs[i]));
        }
#pragma unroll
        for (int e = 0; e < EPV; ++e) acc[i] += kRMS ? xs[i][e] * xs[i][e] : xs[i][e];
      } else {
#pragma unroll
        for (int e = 0; e < EPV; ++e) xs[i][e] = 0.f;
      }
    }
    group_sum2<R>(acc, tpr, scratch);
    float mu[R], rs[R];
    if (kRMS) {
#pragma unroll
      for (int i = 0; i < R; ++i) {
        mu[i] = 0.f;
        rs[i] = rsqrtf(acc[i] * inv_cols + eps);
      }
    } else {
      float var[R];
#pragma unroll
      for (int i = 0; i < R; ++i) {
        mu[i] = acc[i] * inv_cols;
        var[i] = 0.f;
        if (col_ok) {
#pragma unroll
          for (int e = 0; e < EPV; ++e) {
            const float d = xs[i][e] - mu[i];
            var[i] += d * d;
          }
        }
      }
      group_sum2<R>(var, tpr, scratch);
#pragma unroll
      for (int i = 0; i < R; ++i) rs[i] = rsqrtf(var[i] * inv_cols + eps);
    }
#pragma unroll
    for (int i = 0; i < R; ++i) {
      const int row = row0 + i;
      if (row < g.rows) {
        if (j == 0) {
          if (!kRMS) mean_out[row] = mu[i];
          rstd_out[row] = rs[i];
        }
        if (col_ok) {
          float o[EPV];
#pragma unroll
          for (int e = 0; e < EPV; ++e) {
            const float xh = (xs[i][e] - mu[i]) * rs[i];
            o[e] = kRMS ? xh * gam[e] : xh * gam[e] + bet[e];
          }
          st_global_v4(y + (size_t)row * g.cols + (size_t)j * EPV, pack<T>(o));
        }
      }
    }
  }
}

// Backward.  part = [3][gridDim.x][cols] fp32 partial column sums: dgamma, dbeta, and (fused op with a
// bias) dbias = column sums of the dropout-masked gradient, which saves a separate reduction pass.
template <typename T, int R, bool kRMS, bool kFused>
__global__ void __launch_bounds__(kNormV2Threads, 2) norm_bwd_v2_kernel(
    const T* __restrict__ dy, const T* __restrict__ x, const float* __restrict__ mean,
    const float* __restrict__ rstd, const T* __restrict__ gamma, T* __restrict__ dx, float* __restrict__ part,
    NormGeom2 g, T* __restrict__ dx_drop, int want_dbias, float p, float keep_scale, unsigned long long seed,
    unsigned long long offset) {
  constexpr int EPV = VecTraits<T>::kElems;
  extern __shared__ __align__(128) uint8_t dyn_smem[];
  float* sm_acc = reinterpret_cast<float*>(dyn_smem);  // [3][cols], then the input stages, then their barriers
  __shared__ float scratch[2 * R * kNormV2Warps];
  const int tpr = g.tpr;
  const int grp = threadIdx.x / tpr, j = threadIdx.x - grp * tpr;
  const bool col_ok = j < g.nvec;
  const float inv_cols = 1.f / (float)g.cols;
  const uint32_t thresh = kFused ? dropout_thresh16(p) : 0u;

  // ---- input pipeline (see norm_fwd_v2_kernel): every stage holds a dy tile and an x tile ----
  const int tile_rows = g.groups * R;
  const uint32_t row_bytes = (uint32_t)g.cols * (uint32_t)sizeof(T);
  const uint32_t tile_bytes = (uint32_t)tile_rows * row_bytes;
  const uint32_t stage_bytes = tile_bytes * 2u;
  const uint32_t acc_bytes = (3u * (uint32_t)g.cols * 4u + 127u) & ~127u;
  const uint32_t stage_base = smem_addr_u32(dyn_smem) + acc_bytes;
  const uint32_t bar_base = stage_base + kNormStages * stage_bytes;
  const long long n_tiles = ((long long)g.rows + tile_rows - 1) / tile_rows;
  const int n_my = (int)((n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x);
  auto issue = [&](int it) {  // one thread
    const uint32_t s = (uint32_t)(it % kNormStages);
    const long long trow0 = ((long long)it * gridDim.x + blockIdx.x) * tile_rows;
    const long long left = (long long)g.rows - trow0;
    const uint32_t bytes = (uint32_t)(left < tile_rows ? left : tile_rows) * row_bytes;
    bulk_expect_tx(bar_base + s * 8, bytes * 2u);
    bulk_g2s(stage_base + s * stage_bytes, dy + trow0 * g.cols, bytes, bar_base + s * 8);
    bulk_g2s(stage_base + s * stage_bytes + tile_bytes, x + trow0 * g.cols, bytes, bar_base + s * 8);
  };
  if (threadIdx.x == 0) {
    for (int s = 0; s < kNormStages; ++s) bulk_bar_init(bar_base + s * 8, 1);
    bulk_bar_init_fence();
    for (int it = 0; it < kNormStages && it < n_my; ++it) issue(it);
  }

  float gam[EPV], dg[EPV], db[EPV], dbi[EPV];
#pragma unroll
  for (int e = 0; e < EPV; ++e) gam[e] = dg[e] = db[e] = dbi[e] = 0.f;
  if (col_ok) unpack<T>(ldv(gamma + j * EPV), gam);
  __syncthreads();

  for (int it = 0; it < n_my; ++it) {
    const int row0 = ((it * gridDim.x + blockIdx.x) * g.groups + grp) * R;
    const uint32_t stg = (uint32_t)(it % kNormStages);
    bulk_wait(bar_base + stg * 8, (uint32_t)((it / kNormStages) & 1));
    const uint8_t* st = dyn_smem + acc_bytes + stg * stage_bytes + (size_t)(grp * R) * row_bytes + (size_t)j * 16;
    Vec16 xq[R], dq[R];
    float mu[R], rs[R];
#pragma unroll
    for (int i = 0; i < R; ++i) {
      const bool ok = row0 + i < g.rows;
      mu[i] = (ok && !kRMS) ? mean[row0 + i] : 0.f;
      rs[i] = ok ? rstd[row0 + i] : 0.f;
      if (ok && col_ok) {
        dq[i] = *reinterpret_cast<const Vec16*>(st + (size_t)i * row_bytes);
        xq[i] = *reinterpret_cast<const Vec16*>(st + tile_bytes + (size_t)i * row_bytes);
      } else {
        xq[i].w[0] = xq[i].w[1] = xq[i].w[2] = xq[i].w[3] = 0u;
        dq[i] = xq[i];
      }
    }
    __syncthreads();  // the stage has been copied out by everybody: refill it
    if (threadIdx.x == 0 && it + kNormStages < n_my) issue(it + kNormStages);
    float s[2 * R];
#pragma unroll
    for (int i = 0; i < R; ++i) {
      float xv[EPV], dv[EPV];
      unpack<T>(xq[i], xv);
      unpack<T>(dq[i], dv);
      float s0 = 0.f, s1 = 0.f;
#pragma unroll
      for (int e = 0; e < EPV; ++e) {
        const float xh = (xv[e] - mu[i]) * rs[i];
        const float gy = dv[e] * gam[e];
        s0 += gy;
        s1 += gy * xh;
        dg[e] += dv[e] * xh;
        if (!kRMS) db[e] += dv[e];
      }
      s[2 * i] = s0;
      s[2 * i + 1] = s1;
    }
    group_sum2<2 * R>(s, tpr, scratch);
#pragma unroll
    for (int i = 0; i < R; ++i) {
      if (col_ok && row0 + i < g.rows) {
        const float m1 = kRMS ? 0.f : s[2 * i] * inv_cols, m2 = s[2 * i + 1] * inv_cols;
        const size_t off = (size_t)(row0 + i) * g.cols + (size_t)j * EPV;
        float xv[EPV], dv[EPV], o[EPV];
        unpack<T>(xq[i], xv);
        unpack<T>(dq[i], dv);
#pragma unroll
        for (int e = 0; e < EPV; ++e) {
          const float xh = (xv[e] - mu[i]) * rs[i];
          o[e] = rs[i] * (dv[e] * gam[e] - m1 - xh * m2);
        }
        st_global_v4(dx + off, pack<T>(o));
        if (kFused) {
          uint32_t keep = 0xffu;
          if (p > 0.f) keep = dropout_keep8(seed, offset, off / 8, thresh);
#pragma unroll
          for (int e = 0; e < EPV; ++e) {
            o[e] = ((keep >> e) & 1u) ? o[e] * keep_scale : 0.f;
            dbi[e] += o[e];
          }
          if (dx_drop != dx) st_global_v4(dx_drop + off, pack<T>(o));
        }
      }
    }
  }

  // Column sums across the row groups of this CTA, without shared-memory float atomics (those are
  // CAS loops): groups that share a warp combine with shuffles, then one group (or warp) at a time
  // adds its registers into the shared row.
  const int narr = want_dbias ? 3 : (kRMS ? 1 : 2);
  if (tpr < 32) {
    for (int o = tpr; o < 32; o <<= 1) {
#pragma unroll
      for (int e = 0; e < EPV; ++e) {
        dg[e] += __shfl_xor_sync(0xffffffffu, dg[e], o);
        db[e] += __shfl_xor_sync(0xffffffffu, db[e], o);
        dbi[e] += __shfl_xor_sync(0xffffffffu, dbi[e], o);
      }
    }
  }
  const int n_owner = tpr < 32 ? (int)(blockDim.x >> 5) : g.groups;
  const int my_owner = tpr < 32 ? (int)(threadIdx.x >> 5) : grp;
  const bool writer = col_ok && (tpr >= 32 || (int)(threadIdx.x & 31) < tpr);
  __syncthreads();
  for (int w = 0; w < n_owner; ++w) {
    if (writer && my_owner == w) {
      float* a0 = sm_acc + j * EPV;
#pragma unroll
      for (int e = 0; e < EPV; ++e) {
        if (w == 0) {
          a0[e] = dg[e];
          a0[g.cols + e] = db[e];
          if (want_dbias) a0[2 * g.cols + e] = dbi[e];
        } else {
          a0[e] += dg[e];
          a0[g.cols + e] += db[e];
          if (want_dbias) a0[2 * g.cols + e] += dbi[e];
        }
      }
    }
    __syncthreads();
  }
  for (int a = 0; a < 3; ++a) {
    if (a == 1 && kRMS) continue;
    if (a == 2 && !want_dbias) continue;
    float* dst = part + ((size_t)a * gridDim.x + blockIdx.x) * g.cols;
    for (int c = threadIdx.x; c < g.cols; c += blockDim.x) dst[c] = sm_acc[a * g.cols + c];
  }
  (void)narr;
}

// partial rows -> 16-bit column sums.  block = (32 columns) x (32 row slices); grid.y picks the array.
// acc_mask bit a: array a is ADDED to what `out` already holds (parameter gradients written straight into the
// optimizer's flat gradient arena instead of into a temporary that autograd then adds with one more kernel)
template <typename T>
__global__ void __launch_bounds__(1024) colsum_finalize_kernel(const float* __restrict__ part, int parts, int cols,
                                                                 T* __restrict__ out0, T* __restrict__ out1,
                                                                 T* __restrict__ out2, int acc_mask) {
  __shared__ float red[32][33];
  T* out = blockIdx.y == 0 ? out0 : (blockIdx.y == 1 ? out1 : out2);
  if (out == nullptr) return;
  const float* src = part + (size_t)blockIdx.y * parts * cols;
  const int cx = threadIdx.x & 31, ry = threadIdx.x >> 5;
  const int col = blockIdx.x * 32 + cx;
  float a = 0.f;
  if (col < cols) {
#pragma unroll 4
    for (int r = ry; r < parts; r += 32) a += src[(size_t)r * cols + col];
  }
  red[ry][cx] = a;
  __syncthreads();
  if (ry == 0 && col < cols) {
    float s = 0.f;
#pragma unroll
    for (int r = 0; r < 32; ++r) s += red[r][cx];
    if ((acc_mask >> blockIdx.y) & 1) s += to_f32<T>(out[col]);
    out[col] = from_f32<T>(s);
  }
}

// ================================================================================================
// v3 kernels: ONE WARP PER ROW (or 32/LPR short rows per warp), no block-level synchronisation in the row loop.
//
// The v2 kernels spend their time in barriers: six __syncthreads per 8-row tile (stage hand-over plus the cross-warp
// row reductions of a 96-thread row group).  Here a
// row of up to 32 * VPL 16-byte vectors is held by one warp - lane l owns vectors l, l + 32, ... - so the row
// reductions are five shuffles, every load is a fully coalesced 512-byte warp request and nothing in the loop waits
// for another warp.  A warp works on R rows at a time and already has the NEXT R rows in flight (register double
// buffer, kPF).  Rows stay PACKED (16-bit) in registers and are converted again by each pass over them - conversions
// are cheap, registers are what limits the bytes in flight; gamma / beta / bias are held packed as well.  Rows shorter
// than 32 vectors are packed 32 / LPR to a warp (LPR = lanes per row, a power of two).  The backward keeps its
// dgamma / dbeta (/ dbias) column accumulators in registers for the whole persistent loop and combines the CTA's warps
// once at the end, in a fixed order (no atomics).
// ================================================================================================
constexpr int kNormV3Threads = 256;
constexpr int kNormV3Warps = kNormV3Threads / 32;
constexpr int kNormV3BwdThreads = 384;  // backward: 12 warps, one CTA per SM (168 registers: the column accumulators)
constexpr int kNormV3BwdWarps = kNormV3BwdThreads / 32;
constexpr int kNormV3MaxVPL = 4;  // longer rows (> 1024 16-bit elements) stay on the v2 kernels: the row no longer fits a warp's registers

struct NormGeom3 {
  int rows, cols, nvec;
};

template <int LPR>
UB_DEVICE float row_sum(float v) {
#pragma unroll
  for (int o = LPR >> 1; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Forward.  The current row lives in fp32 registers (every pass after the first is pure math), the NEXT row is already
// in flight as packed 16-bit vectors (kPF), gamma / beta / bias are NOT held in registers: they are re-read at their
// single use per row from L1 (a 1.5 KB working set that never leaves it), which is two issue slots per eight elements
// and frees 24-36 registers for occupancy.  kFull: the row is exactly 32 * VPL vectors - no per-vector predicates.
// (A first version that re-converted the packed row in every pass was instruction-bound.)
template <typename T, int VPL, int LPR, int R, bool kPF, bool kRMS, bool kFused, bool kFull>
__global__ void __launch_bounds__(kNormV3Threads, (VPL <= 3 ? 3 : (VPL == 4 ? 2 : 1))) norm_fwd_v3_kernel(
    const T* __restrict__ x, const T* __restrict__ gamma, const T* __restrict__ beta, T* __restrict__ y,
    float* __restrict__ mean_out, float* __restrict__ rstd_out, NormGeom3 g, float eps,
    const T* __restrict__ bias, const T* __restrict__ residual, T* __restrict__ summed, float p, float keep_scale,
    unsigned long long seed, unsigned long long offset) {
  constexpr int EPV = VecTraits<T>::kElems;
  constexpr int RW = 32 / LPR;  // short rows per warp
  static_assert(LPR == 32 || VPL == 1, "short rows use one vector per lane");
  static_assert(R == 1 || !kFused, "the fused variant works on one row group at a time");
  const int lane = threadIdx.x & 31;
  const int sub = lane / LPR, j = lane % LPR;
  const long long gw = (long long)blockIdx.x * kNormV3Warps + (threadIdx.x >> 5);
  const long long stride = (long long)gridDim.x * kNormV3Warps * (RW * R);
  const float inv_cols = 1.f / (float)g.cols;
  const uint32_t thresh = kFused ? dropout_thresh16(p) : 0u;
  const bool has_bias = kFused && bias != nullptr;

  bool ok[VPL];
#pragma unroll
  for (int k = 0; k < VPL; ++k) ok[k] = kFull || (j + k * LPR < g.nvec);
  const T* gam_p = gamma + (size_t)j * EPV;
  const T* bet_p = kRMS ? nullptr : beta + (size_t)j * EPV;
  const T* bia_p = has_bias ? bias + (size_t)j * EPV : nullptr;

  auto fetch = [&](long long base, Vec16 (&xd)[R][VPL], Vec16 (&rd)[kFused ? R : 1][VPL]) {
#pragma unroll
    for (int i = 0; i < R; ++i) {
      const long long r = base + i * RW + sub;
      if (r < g.rows) {
        const T* xp = x + (size_t)r * g.cols + (size_t)j * EPV;
        const T* rp = kFused ? residual + (size_t)r * g.cols + (size_t)j * EPV : nullptr;
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
          if (ok[k]) {
            xd[i][k] = ld_global_nc_v4(xp + k * (LPR * EPV));
            if (kFused) rd[kFused ? i : 0][k] = ld_global_nc_v4(rp + k * (LPR * EPV));
          }
        }
      }
    }
  };
  long long base = gw * (RW * R);
  Vec16 xv[R][VPL], rv[kFused ? R : 1][VPL];
  fetch(base, xv, rv);
  for (; base < g.rows; base += stride) {
    float xs[R][VPL][EPV];
    float acc[R];
    // pass 1: convert (fused: bias + dropout + residual, store the rounded sum), row sum
#pragma unroll
    for (int i = 0; i < R; ++i) {
      const long long row = base + i * RW + sub;
      acc[i] = 0.f;
#pragma unroll
      for (int k = 0; k < VPL; ++k) {
        if (row < g.rows && ok[k]) {
          unpack<T>(xv[i][k], xs[i][k]);
          if (kFused) {
            const size_t off = (size_t)row * g.cols + (size_t)(j + k * LPR) * EPV;
            float res[EPV];
            unpack<T>(rv[kFused ? i : 0][k], res);
            if (has_bias) {
              float bf[EPV];
              unpack<T>(ldv(bia_p + k * (LPR * EPV)), bf);
#pragma unroll
              for (int e = 0; e < EPV; ++e) xs[i][k][e] += bf[e];
            }
            uint32_t keep = 0xffu;
            if (p > 0.f) keep = dropout_keep8(seed, offset, off / 8, thresh);
#pragma unroll
            for (int e = 0; e < EPV; ++e)
              xs[i][k][e] = fmaf(xs[i][k][e], ((keep >> e) & 1u) ? keep_scale : 0.f, res[e]);
            // the sum is rounded to T first: backward and the pre-LN consumer see exactly this value
            const Vec16 sv = pack<T>(xs[i][k]);
            st_global_v4(summed + off, sv);
            unpack<T>(sv, xs[i][k]);
          }
#pragma unroll
          for (int e = 0; e < EPV; ++e) acc[i] += kRMS ? xs[i][k][e] * xs[i][k][e] : xs[i][k][e];
        } else {
#pragma unroll
          for (int e = 0; e < EPV; ++e) xs[i][k][e] = 0.f;
        }
      }
    }
    // the packed registers are free now: the next rows start their trip through the memory system
    if (kPF) fetch(base + stride, xv, rv);
#pragma unroll
    for (int i = 0; i < R; ++i) acc[i] = row_sum<LPR>(acc[i]);
    float mu[R], rs[R];
    if (kRMS) {
#pragma unroll
      for (int i = 0; i < R; ++i) {
        mu[i] = 0.f;
        rs[i] = rsqrtf(acc[i] * inv_cols + eps);
      }
    } else {
      float var[R];
#pragma unroll
      for (int i = 0; i < R; ++i) {
        mu[i] = acc[i] * inv_cols;
        var[i] = 0.f;
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
          if (kFull || ok[k]) {
#pragma unroll
            for (int e = 0; e < EPV; ++e) {
              xs[i][k][e] -= mu[i];  // centred values are what the output needs
              var[i] = fmaf(xs[i][k][e], xs[i][k][e], var[i]);
            }
          }
        }
      }
#pragma unroll
      for (int i = 0; i < R; ++i) rs[i] = rsqrtf(row_sum<LPR>(var[i]) * inv_cols + eps);
    }
    // pass 3: y = x_hat * gamma (+ beta); gamma / beta come from L1
#pragma unroll
    for (int k = 0; k < VPL; ++k) {
      if (kFull || ok[k]) {
        float gf[EPV], bf[EPV];
        unpack<T>(ldv(gam_p + k * (LPR * EPV)), gf);
        if (!kRMS) unpack<T>(ldv(bet_p + k * (LPR * EPV)), bf);
#pragma unroll
        for (int i = 0; i < R; ++i) {
          const long long row = base + i * RW + sub;
          if (row < g.rows) {
            float o[EPV];
#pragma unroll
            for (int e = 0; e < EPV; ++e) {
              const float xh = xs[i][k][e] * rs[i];
              o[e] = kRMS ? xh * gf[e] : fmaf(xh, gf[e], bf[e]);
            }
            st_global_v4(y + (size_t)row * g.cols + (size_t)(j + k * LPR) * EPV, pack<T>(o));
          }
        }
      }
    }
    if (j == 0) {
#pragma unroll
      for (int i = 0; i < R; ++i) {
        const long long row = base + i * RW + sub;
        if (row < g.rows) {
          if (!kRMS) mean_out[row] = mu[i];
          rstd_out[row] = rs[i];
        }
      }
    }
    if (!kPF) fetch(base + stride, xv, rv);
  }
}

// part = [3][gridDim.x][cols] fp32 partial column sums (dgamma, dbeta, dbias of the fused op) - the layout of the v2
// kernel, finished by colsum_finalize_kernel.  Dynamic shared memory: kNormV3BwdWarps * cols floats.
template <typename T, int VPL, int LPR, int R, bool kPF, bool kRMS, bool kFused, bool kFull>
__global__ void __launch_bounds__(kNormV3BwdThreads, (VPL <= 1 ? 2 : 1)) norm_bwd_v3_kernel(
    const T* __restrict__ dy, const T* __restrict__ x, const float* __restrict__ mean,
    const float* __restrict__ rstd, const T* __restrict__ gamma, T* __restrict__ dx, float* __restrict__ part,
    NormGeom3 g, T* __restrict__ dx_drop, int want_dbias, float p, float keep_scale, unsigned long long seed,
    unsigned long long offset) {
  constexpr int EPV = VecTraits<T>::kElems;
  constexpr int RW = 32 / LPR;
  static_assert(LPR == 32 || VPL == 1, "short rows use one vector per lane");
  extern __shared__ __align__(16) float sm_cols[];  // [kNormV3BwdWarps][cols]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int sub = lane / LPR, j = lane % LPR;
  const long long gw = (long long)blockIdx.x * kNormV3BwdWarps + warp;
  const long long stride = (long long)gridDim.x * kNormV3BwdWarps * (RW * R);
  const float inv_cols = 1.f / (float)g.cols;
  const uint32_t thresh = kFused ? dropout_thresh16(p) : 0u;

  bool ok[VPL];
  float dg[VPL][EPV], db[VPL][EPV], dbi[kFused ? VPL : 1][EPV];
#pragma unroll
  for (int k = 0; k < VPL; ++k) {
    ok[k] = kFull || (j + k * LPR < g.nvec);
#pragma unroll
    for (int e = 0; e < EPV; ++e) {
      dg[k][e] = db[k][e] = 0.f;
      if (kFused) dbi[kFused ? k : 0][e] = 0.f;
    }
  }
  const T* gam_p = gamma + (size_t)j * EPV;  // re-read from L1 at its use (see the forward kernel)

  auto fetch = [&](long long base, Vec16 (&xd)[R][VPL], Vec16 (&dd)[R][VPL], float (&mu)[R], float (&rs)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) {
      const long long r = base + i * RW + sub;
      mu[i] = 0.f;
      rs[i] = 0.f;
      if (r < g.rows) {
        if (!kRMS) mu[i] = __ldg(mean + r);
        rs[i] = __ldg(rstd + r);
        const T* dp = dy + (size_t)r * g.cols + (size_t)j * EPV;
        const T* xp = x + (size_t)r * g.cols + (size_t)j * EPV;
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
          if (ok[k]) {
            dd[i][k] = ld_global_nc_v4(dp + k * (LPR * EPV));
            xd[i][k] = ld_global_nc_v4(xp + k * (LPR * EPV));
          }
        }
      }
    }
  };
  long long base = gw * (RW * R);
  Vec16 xv[R][VPL], dv[R][VPL];
  float mu[R], rs[R];
  fetch(base, xv, dv, mu, rs);
  for (; base < g.rows; base += stride) {
    // pass 1: x_hat and dy * gamma in fp32 registers, row sums, column accumulators
    float xh[R][VPL][EPV], gy[R][VPL][EPV];
    float s0[R], s1[R], rs_c[R];
#pragma unroll
    for (int i = 0; i < R; ++i) s0[i] = s1[i] = 0.f;
#pragma unroll
    for (int k = 0; k < VPL; ++k) {
      float gf[EPV];
      if (kFull || ok[k]) unpack<T>(ldv(gam_p + k * (LPR * EPV)), gf);
#pragma unroll
      for (int i = 0; i < R; ++i) {
        const long long row = base + i * RW + sub;
        if (row < g.rows && ok[k]) {
          float xf[EPV], df[EPV];
          unpack<T>(xv[i][k], xf);
          unpack<T>(dv[i][k], df);
#pragma unroll
          for (int e = 0; e < EPV; ++e) {
            // subtract first: x * rstd - mean * rstd cancels two large products when |mean| >> std (loses ~|mean| / std
            // ulp of x_hat), x - mean is exact there
            xh[i][k][e] = (xf[e] - mu[i]) * rs[i];
            gy[i][k][e] = df[e] * gf[e];
            s0[i] += gy[i][k][e];
            s1[i] = fmaf(gy[i][k][e], xh[i][k][e], s1[i]);
            dg[k][e] = fmaf(df[e], xh[i][k][e], dg[k][e]);
            if (!kRMS) db[k][e] += df[e];
          }
        } else {
#pragma unroll
          for (int e = 0; e < EPV; ++e) xh[i][k][e] = gy[i][k][e] = 0.f;
        }
      }
    }
#pragma unroll
    for (int i = 0; i < R; ++i) rs_c[i] = rs[i];
    // the packed registers are free: the next rows start their trip through the memory system
    if (kPF) fetch(base + stride, xv, dv, mu, rs);
#pragma unroll
    for (int i = 0; i < R; ++i) {
      if (!kRMS) s0[i] = row_sum<LPR>(s0[i]);
      s1[i] = row_sum<LPR>(s1[i]);
    }
    // pass 2: dx = rstd * (gy - mean(gy) - x_hat * mean(gy * x_hat))
#pragma unroll
    for (int i = 0; i < R; ++i) {
      const long long row = base + i * RW + sub;
      if (row < g.rows) {
        const float b0 = kRMS ? 0.f : -s0[i] * inv_cols * rs_c[i], c0 = -s1[i] * inv_cols * rs_c[i];
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
          if (kFull || ok[k]) {
            const size_t off = (size_t)row * g.cols + (size_t)(j + k * LPR) * EPV;
            float o[EPV];
#pragma unroll
            for (int e = 0; e < EPV; ++e) o[e] = fmaf(xh[i][k][e], c0, fmaf(gy[i][k][e], rs_c[i], b0));
            st_global_v4(dx + off, pack<T>(o));
            if (kFused) {
              uint32_t keep = 0xffu;
              if (p > 0.f) keep = dropout_keep8(seed, offset, off / 8, thresh);
#pragma unroll
              for (int e = 0; e < EPV; ++e) {
                o[e] = ((keep >> e) & 1u) ? o[e] * keep_scale : 0.f;
                dbi[kFused ? k : 0][e] += o[e];
              }
              if (dx_drop != dx) st_global_v4(dx_drop + off, pack<T>(o));
            }
          }
        }
      }
    }
    if (!kPF) fetch(base + stride, xv, dv, mu, rs);
  }

  // column sums: sub-rows of a warp by shuffles, the CTA's warps through one shared-memory row each, then a fixed
  // order sum per column -> one fp32 partial row per CTA and array (deterministic: no atomics anywhere)
  const int narr = kFused && want_dbias ? 3 : (kRMS ? 1 : 2);
  for (int a = 0; a < narr; ++a) {
    if (a == 1 && kRMS) continue;
#pragma unroll
    for (int k = 0; k < VPL; ++k) {
      float v[EPV];
#pragma unroll
      for (int e = 0; e < EPV; ++e) {
        v[e] = a == 0 ? dg[k][e] : (a == 1 ? db[k][e] : dbi[kFused ? k : 0][e]);
#pragma unroll
        for (int o = LPR; o < 32; o <<= 1) v[e] += __shfl_xor_sync(0xffffffffu, v[e], o);
      }
      if ((kFull || ok[k]) && sub == 0) {
        float* dst = sm_cols + (size_t)warp * g.cols + (size_t)(j + k * LPR) * EPV;
#pragma unroll
        for (int e = 0; e < EPV; e += 4) *reinterpret_cast<float4*>(dst + e) = make_float4(v[e], v[e + 1], v[e + 2], v[e + 3]);
      }
    }
    __syncthreads();
    float* out = part + ((size_t)a * gridDim.x + blockIdx.x) * g.cols;
    for (int c = threadIdx.x; c < g.cols; c += kNormV3BwdThreads) {
      float s = 0.f;
#pragma unroll
      for (int w = 0; w < kNormV3BwdWarps; ++w) s += sm_cols[(size_t)w * g.cols + c];
      out[c] = s;
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
// set by the launch_* entry points for the duration of one call (the host side of a stream is single-threaded)
static thread_local int g_acc_mask = 0;
// deterministic mode (torch.use_deterministic_algorithms), set the same way: the gen-1 backward combines its row groups
// in a fixed order
static thread_local bool g_det = false;

static int sm_count() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms <= 0) sms = 132;
  }
  return sms;
}

static int pow2ceil(int v) {
  int p = 1;
  while (p < v) p <<= 1;
  return p;
}

constexpr int kFwdR = 2, kBwdR = 2;

static int dtype_epv(int dtype) { return dtype == kF32 ? 4 : 8; }

template <typename T>
constexpr int dtype_of() {
  return std::is_same<T, float>::value ? kF32 : (std::is_same<T, __half>::value ? kF16 : kBF16);
}

// (vectors per lane, lanes per row) -> rows per warp iteration R and whether the next R rows are prefetched: about four
// to six 16-byte vectors per lane and tensor in flight; very long rows (VPL >= 5) run without the register double buffer
#define UB_V3_CASE(V, L, RR, PF, ...)                                                                     \
  if (vpl == V && lpr == L) {                                                                             \
    constexpr int VPL = V; constexpr int LPR = L; constexpr int R = RR; constexpr bool kPF = PF;          \
    (void)VPL; (void)LPR; (void)R; (void)kPF;                                                             \
    __VA_ARGS__;                                                                                          \
    return true;                                                                                          \
  }
#define UB_DISPATCH_V3(...)                                                                               \
  UB_V3_CASE(1, 1, 1, true, __VA_ARGS__) UB_V3_CASE(1, 2, 1, true, __VA_ARGS__)                           \
  UB_V3_CASE(1, 4, 1, true, __VA_ARGS__) UB_V3_CASE(1, 8, 1, true, __VA_ARGS__)                           \
  UB_V3_CASE(1, 16, 1, true, __VA_ARGS__) UB_V3_CASE(1, 32, 2, true, __VA_ARGS__)                         \
  UB_V3_CASE(2, 32, 1, true, __VA_ARGS__) UB_V3_CASE(3, 32, 1, true, __VA_ARGS__)                         \
  UB_V3_CASE(4, 32, 1, true, __VA_ARGS__)

// true if UB_DISPATCH_V3 has a kernel for (vpl, lpr); r = its rows per warp iteration
static bool v3_case(int vpl, int lpr, int& r) {
  UB_DISPATCH_V3(r = R);
  return false;
}

// Persistent grids: v3 runs `per_sm` CTAs per SM (forward 8 warps, backward 12 warps; the backward emits one fp32
// partial row per CTA and array, so few CTAs keep the finalize pass short), v2 two CTAs per SM, v1 eight (forward)
// or two (backward) - fewer when the rows do not fill them.
NormPlan norm_plan(int rows, int cols, int dtype, int kind) {
  NormPlan p{};
  const int epv = dtype_epv(dtype);
  if (rows < 0 || cols < epv || cols % epv != 0) return p;
  const bool bwd = kind == kNormBwd;
  p.nvec = cols / epv;
  long long cap;
  if (p.nvec <= 32 * kNormV3MaxVPL && v3_case(p.nvec <= 32 ? 1 : (p.nvec + 31) / 32, p.nvec <= 32 ? pow2ceil(p.nvec) : 32, p.r)) {
    p.gen = 3;
    p.lpr = p.nvec <= 32 ? pow2ceil(p.nvec) : 32;
    p.vpl = (p.nvec + p.lpr - 1) / p.lpr;
    if (kind == kNormFusedFwd) p.r = 1;  // the fused forward works on one row group at a time
    p.full = p.nvec == p.vpl * p.lpr;
    const int warps = bwd ? kNormV3BwdWarps : kNormV3Warps;
    p.threads = warps * 32;
    p.tile_rows = (32 / p.lpr) * p.r;
    cap = (long long)sm_count() * (bwd ? (p.vpl <= 1 ? 2 : 1) : (p.vpl <= 3 ? 3 : (p.vpl == 4 ? 2 : 1)));
    const long long need = ((long long)rows + warps * p.tile_rows - 1) / (warps * p.tile_rows);
    p.grid = (int)std::max(1ll, std::min(need, cap));
    p.units = (long long)p.grid * warps;
  } else if (p.nvec <= kNormV2Threads) {
    p.gen = 2;
    p.tpr = p.nvec < 32 ? pow2ceil(p.nvec) : ((p.nvec + 31) / 32) * 32;
    p.groups = kNormV2Threads / p.tpr;
    p.r = bwd ? kBwdR : kFwdR;
    p.full = p.nvec == p.tpr;
    p.threads = p.tpr * p.groups;
    p.tile_rows = p.groups * p.r;
    const long long need = ((long long)rows + p.tile_rows - 1) / p.tile_rows;
    p.grid = (int)std::max(1ll, std::min(need, (long long)sm_count() * 2));
    p.units = p.grid;
  } else {
    p.tpr = p.nvec <= 128 ? std::min(pow2ceil(p.nvec), 32) : std::min(pow2ceil((p.nvec + 3) / 4), kNormThreads);
    p.vpt = (p.nvec + p.tpr - 1) / p.tpr;
    if (p.vpt > 4) return NormPlan{};
    p.gen = 1;
    p.groups = kNormThreads / p.tpr;
    p.full = p.nvec == p.vpt * p.tpr;
    p.threads = kNormThreads;
    p.tile_rows = p.groups;
    const long long need = bwd ? ((long long)rows + 7) / 8 : ((long long)rows + p.tile_rows - 1) / p.tile_rows;
    p.grid = (int)std::max(1ll, std::min(need, (long long)sm_count() * (bwd ? 2 : 8)));
    p.units = p.grid;
  }
  const long long tiles = ((long long)rows + p.tile_rows - 1) / p.tile_rows;
  p.rows_per_sweep = p.units * p.tile_rows;
  p.tiles_min = tiles / p.units;
  p.tiles_max = (tiles + p.units - 1) / p.units;
  return p;
}

bool norm_v2_supported(int cols, int dtype) { return norm_plan(1, cols, dtype, kNormBwd).gen >= 2; }

int norm_bwd_parts(int rows, int cols, int dtype) { return norm_plan(rows, cols, dtype, kNormBwd).grid; }

template <typename T, bool kRMS, bool kFused>
static bool run_fwd_v3(const NormPlan& pl, const void* x, const void* gamma, const void* beta, void* y, float* mean,
                       float* rstd, int rows, int cols, float eps, const void* bias, const void* residual, void* summed,
                       float p, float keep_scale, unsigned long long seed, unsigned long long offset,
                       cudaStream_t stream) {
  const NormGeom3 g{rows, cols, pl.nvec};
  const int vpl = pl.vpl, lpr = pl.lpr, grid = pl.grid;
  UB_DISPATCH_V3({
    constexpr int RF = kFused ? 1 : R;
    if (pl.full)
      norm_fwd_v3_kernel<T, VPL, LPR, RF, kPF, kRMS, kFused, true><<<grid, kNormV3Threads, 0, stream>>>(
          (const T*)x, (const T*)gamma, (const T*)beta, (T*)y, mean, rstd, g, eps, (const T*)bias, (const T*)residual,
          (T*)summed, p, keep_scale, seed, offset);
    else
      norm_fwd_v3_kernel<T, VPL, LPR, RF, kPF, kRMS, kFused, false><<<grid, kNormV3Threads, 0, stream>>>(
          (const T*)x, (const T*)gamma, (const T*)beta, (T*)y, mean, rstd, g, eps, (const T*)bias, (const T*)residual,
          (T*)summed, p, keep_scale, seed, offset);
  });
  return false;
}

template <typename T, bool kRMS, bool kFused>
static bool run_bwd_v3(const NormPlan& pl, const void* dy, const void* x, const float* mean, const float* rstd,
                       const void* gamma, void* dx, void* dgamma, void* dbeta, void* dbias, float* part, int rows,
                       int cols, void* dx_drop, float p, float keep_scale, unsigned long long seed,
                       unsigned long long offset, cudaStream_t stream) {
  const NormGeom3 g{rows, cols, pl.nvec};
  const int vpl = pl.vpl, lpr = pl.lpr, grid = pl.grid;
  const size_t smem = (size_t)kNormV3BwdWarps * cols * sizeof(float);
  auto finish = [&]() {
    colsum_finalize_kernel<T><<<dim3((cols + 31) / 32, 3), 1024, 0, stream>>>(part, grid, cols, (T*)dgamma, (T*)dbeta,
                                                                              (T*)dbias, g_acc_mask);
  };
  UB_DISPATCH_V3({
    auto kern = pl.full ? norm_bwd_v3_kernel<T, VPL, LPR, R, (kPF && VPL <= 3), kRMS, kFused, true>
                        : norm_bwd_v3_kernel<T, VPL, LPR, R, (kPF && VPL <= 3), kRMS, kFused, false>;
    if (smem > 48 * 1024) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    kern<<<grid, kNormV3BwdThreads, smem, stream>>>((const T*)dy, (const T*)x, mean, rstd, (const T*)gamma, (T*)dx, part, g,
                                                 (T*)dx_drop, dbias != nullptr ? 1 : 0, p, keep_scale, seed, offset);
    finish();
  });
  return false;
}

#define UB_DISPATCH_VPT(VPT_VALUE, ...)                                   \
  switch (VPT_VALUE) {                                                    \
    case 1: { constexpr int VPT = 1; __VA_ARGS__; break; }                \
    case 2: { constexpr int VPT = 2; __VA_ARGS__; break; }                \
    case 3: { constexpr int VPT = 3; __VA_ARGS__; break; }                \
    case 4: { constexpr int VPT = 4; __VA_ARGS__; break; }                \
    default: break;                                                       \
  }

#define UB_DISPATCH_DTYPE(DTYPE_VALUE, ...)                               \
  switch (DTYPE_VALUE) {                                                  \
    case kF32: { using T = float; __VA_ARGS__; break; }                   \
    case kF16: { using T = __half; __VA_ARGS__; break; }                  \
    case kBF16: { using T = __nv_bfloat16; __VA_ARGS__; break; }          \
    default: break;                                                       \
  }

template <typename T, bool kRMS, bool kFused>
static void run_fwd(const void* x, const void* gamma, const void* beta, void* y, float* mean, float* rstd, int rows,
                    int cols, float eps, const void* bias, const void* residual, void* summed, float p,
                    unsigned long long seed, unsigned long long offset, cudaStream_t stream) {
  const float keep_scale = p > 0.f ? 1.f / (1.f - p) : 1.f;
  const NormPlan pl = norm_plan(rows, cols, dtype_of<T>(), kFused ? kNormFusedFwd : kNormFwd);
  if (pl.gen == 3) {
    run_fwd_v3<T, kRMS, kFused>(pl, x, gamma, beta, y, mean, rstd, rows, cols, eps, bias, residual, summed, p,
                                keep_scale, seed, offset, stream);
  } else if (pl.gen == 2) {
    const NormGeom2 g2{rows, cols, pl.tpr, pl.nvec, pl.groups};
    auto fkern = norm_fwd_v2_kernel<T, kFwdR, kRMS, kFused>;
    const size_t fsmem = (size_t)kNormStages * pl.tile_rows * cols * sizeof(T) * (kFused ? 2 : 1) + 64;
    cudaFuncSetAttribute(fkern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fsmem);
    fkern<<<pl.grid, pl.threads, fsmem, stream>>>(
        (const T*)x, (const T*)gamma, (const T*)beta, (T*)y, mean, rstd, g2, eps, (const T*)bias, (const T*)residual,
        (T*)summed, p, keep_scale, seed, offset);
  } else if (pl.gen == 1) {
    const NormGeom g{rows, cols, pl.tpr, pl.nvec};
    UB_DISPATCH_VPT(pl.vpt, (norm_fwd_kernel<T, VPT, kRMS, kFused><<<pl.grid, kNormThreads, 0, stream>>>(
                                (const T*)x, (const T*)gamma, (const T*)beta, (T*)y, mean, rstd, g, eps,
                                (const T*)bias, (const T*)residual, (T*)summed, p, keep_scale, seed, offset)));
  }
}

template <typename T, bool kRMS, bool kFused>
static void run_bwd(const void* dy, const void* x, const float* mean, const float* rstd, const void* gamma, void* dx,
                    void* dgamma, void* dbeta, void* dbias, float* part, int rows, int cols, void* dx_drop, float p,
                    unsigned long long seed, unsigned long long offset, cudaStream_t stream) {
  const float keep_scale = p > 0.f ? 1.f / (1.f - p) : 1.f;
  const NormPlan pl = norm_plan(rows, cols, dtype_of<T>(), kNormBwd);
  if (pl.gen == 3) {
    run_bwd_v3<T, kRMS, kFused>(pl, dy, x, mean, rstd, gamma, dx, dgamma, dbeta, dbias, part, rows, cols, dx_drop, p,
                                keep_scale, seed, offset, stream);
  } else if (pl.gen == 2) {
    const NormGeom2 g2{rows, cols, pl.tpr, pl.nvec, pl.groups};
    const size_t smem2 = (((size_t)3 * cols * sizeof(float) + 127) & ~(size_t)127) +
                         (size_t)kNormStages * pl.tile_rows * cols * sizeof(T) * 2 + 64;
    auto kern = norm_bwd_v2_kernel<T, kBwdR, kRMS, kFused>;
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2);
    kern<<<pl.grid, pl.threads, smem2, stream>>>((const T*)dy, (const T*)x, mean, rstd, (const T*)gamma, (T*)dx, part,
                                                  g2, (T*)dx_drop, dbias != nullptr ? 1 : 0, p, keep_scale, seed,
                                                  offset);
    colsum_finalize_kernel<T><<<dim3((cols + 31) / 32, 3), 1024, 0, stream>>>(part, pl.grid, cols, (T*)dgamma,
                                                                              (T*)dbeta, (T*)dbias, g_acc_mask);
  } else if (pl.gen == 1) {
    const NormGeom g{rows, cols, pl.tpr, pl.nvec};
    const int parts = pl.grid;
    float* dg_part = part;
    float* db_part = part + (size_t)parts * cols;
    const size_t smem = (size_t)(kRMS ? 1 : 2) * cols * sizeof(float);
    UB_DISPATCH_VPT(pl.vpt, {
      auto kern = g_det ? norm_bwd_kernel<T, VPT, kRMS, kFused, true> : norm_bwd_kernel<T, VPT, kRMS, kFused>;
      if (smem > 48 * 1024) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      kern<<<parts, kNormThreads, smem, stream>>>((const T*)dy, (const T*)x, mean, rstd, (const T*)gamma, (T*)dx,
                                                  dg_part, db_part, g, (T*)dx_drop, p, keep_scale, seed, offset);
    });
    norm_param_grad_kernel<T><<<(cols + 31) / 32, 256, 0, stream>>>(dg_part, kRMS ? nullptr : db_part, parts, cols,
                                                                    (T*)dgamma, (T*)dbeta, g_acc_mask);
  }
}

void launch_layernorm_fwd(const void* x, const void* gamma, const void* beta, void* y, float* mean, float* rstd,
                          int rows, int cols, float eps, int dtype, cudaStream_t stream) {
  UB_DISPATCH_DTYPE(dtype, (run_fwd<T, false, false>(x, gamma, beta, y, mean, rstd, rows, cols, eps, nullptr, nullptr,
                                                     nullptr, 0.f, 0, 0, stream)));
}

void launch_layernorm_bwd(const void* dy, const void* x, const float* mean, const float* rstd, const void* gamma,
                          void* dx, void* dgamma, void* dbeta, float* part, int rows, int cols, int dtype,
                          cudaStream_t stream, int accumulate, bool deterministic) {
  g_acc_mask = accumulate;
  g_det = deterministic;
  UB_DISPATCH_DTYPE(dtype, (run_bwd<T, false, false>(dy, x, mean, rstd, gamma, dx, dgamma, dbeta, nullptr, part, rows,
                                                     cols, nullptr, 0.f, 0, 0, stream)));
  g_acc_mask = 0;
  g_det = false;
}

void launch_rmsnorm_fwd(const void* x, const void* gamma, void* y, float* rstd, int rows, int cols, float eps,
                        int dtype, cudaStream_t stream) {
  UB_DISPATCH_DTYPE(dtype, (run_fwd<T, true, false>(x, gamma, nullptr, y, nullptr, rstd, rows, cols, eps, nullptr,
                                                    nullptr, nullptr, 0.f, 0, 0, stream)));
}

void launch_rmsnorm_bwd(const void* dy, const void* x, const float* rstd, const void* gamma, void* dx, void* dgamma,
                        float* part, int rows, int cols, int dtype, cudaStream_t stream, int accumulate, bool deterministic) {
  g_acc_mask = accumulate;
  g_det = deterministic;
  UB_DISPATCH_DTYPE(dtype, (run_bwd<T, true, false>(dy, x, nullptr, rstd, gamma, dx, dgamma, nullptr, nullptr, part,
                                                    rows, cols, nullptr, 0.f, 0, 0, stream)));
  g_acc_mask = 0;
  g_det = false;
}

void launch_bias_dropout_add_ln_fwd(const void* x, const void* bias, const void* residual, const void* gamma,
                                    const void* beta, void* y, void* summed, float* mean, float* rstd, int rows,
                                    int cols, float p, float eps, unsigned long long seed, unsigned long long offset,
                                    int dtype, cudaStream_t stream) {
  if (dtype == kF16) {
    run_fwd<__half, false, true>(x, gamma, beta, y, mean, rstd, rows, cols, eps, bias, residual, summed, p, seed,
                                 offset, stream);
  } else if (dtype == kBF16) {
    run_fwd<__nv_bfloat16, false, true>(x, gamma, beta, y, mean, rstd, rows, cols, eps, bias, residual, summed, p,
                                        seed, offset, stream);
  }
}

void launch_bias_dropout_add_ln_bwd(const void* dy, const void* summed, const float* mean, const float* rstd,
                                    const void* gamma, void* dsum, void* dx, void* dgamma, void* dbeta,
                                    void* dbias, float* part, int rows, int cols, float p, unsigned long long seed,
                                    unsigned long long offset, int dtype, cudaStream_t stream, int accumulate, bool deterministic) {
  // dbias (optional, v2 geometries only): column sums of dx, produced by the same pass
  g_acc_mask = accumulate;
  g_det = deterministic;
  if (dtype == kF16) {
    run_bwd<__half, false, true>(dy, summed, mean, rstd, gamma, dsum, dgamma, dbeta, dbias, part, rows, cols, dx, p,
                                 seed, offset, stream);
  } else if (dtype == kBF16) {
    run_bwd<__nv_bfloat16, false, true>(dy, summed, mean, rstd, gamma, dsum, dgamma, dbeta, dbias, part, rows, cols,
                                        dx, p, seed, offset, stream);
  }
  g_acc_mask = 0;
  g_det = false;
}

}  // namespace ub
