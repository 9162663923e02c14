// Gaussian radial-basis pair features of Uni-Mol (unicore_b200/models/unimol.py GaussianLayer):
//   t = mul[edge] * d + bias[edge]                       (one scalar per atom pair, per-edge-type affine map)
//   y[n, k] = exp(-0.5 ((t - mean_k) / std_k)^2) / (sqrt(2 * 3.14159) * std_k),   std_k = |stds_k| + 1e-5
// The PyTorch formulation is two embedding look-ups over B*L*L indices, a broadcast and a TorchScript-fused
// expression: its backward sorts the 2 M indices for the (deterministic) embedding gradient on every step, and
// TorchScript re-specialises on every new padded length.  Here: one forward kernel that writes the [N, K] features
// once, and one backward kernel that recomputes y, reduces d mean / d std per column and scatters d mul / d bias
// through a per-CTA shared-memory histogram (the edge-type table is small: < 1024 entries).
#include <math_constants.h>

#include "../api.h"
#include "../common.cuh"

namespace ub {

constexpr int kGbfThreads = 256;
constexpr float kGbfA = 2.5066272f;  // (2 * 3.14159) ** 0.5, the constant of the reference formula

template <typename T>
__global__ void __launch_bounds__(kGbfThreads) gbf_fwd_kernel(const T* __restrict__ d, const long long* __restrict__ edge,
                                                               const T* __restrict__ mul_w, const T* __restrict__ bias_w,
                                                               const T* __restrict__ means, const T* __restrict__ stds,
                                                               T* __restrict__ y, long long n, int K) {
  const int kvec = K / 8;                  // 16-byte vectors per row
  const int rows_per_cta = kGbfThreads / kvec;
  const int j = threadIdx.x % kvec, rl = threadIdx.x / kvec;
  if (rl >= rows_per_cta) return;
  float m[8], inv_s[8], norm[8];
  {
    float sv[8];
    unpack<T>(ld_global_v4(means + j * 8), m);
    unpack<T>(ld_global_v4(stds + j * 8), sv);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float s = fabsf(sv[e]) + 1e-5f;
      inv_s[e] = 1.f / s;
      norm[e] = 1.f / (kGbfA * s);
    }
  }
  for (long long row = (long long)blockIdx.x * rows_per_cta + rl; row < n; row += (long long)gridDim.x * rows_per_cta) {
    const long long e_idx = edge[row];
    const float t = to_f32<T>(mul_w[e_idx]) * to_f32<T>(d[row]) + to_f32<T>(bias_w[e_idx]);
    float o[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float z = (t - m[e]) * inv_s[e];
      o[e] = __expf(-0.5f * z * z) * norm[e];
    }
    st_global_v4(y + row * K + j * 8, pack<T>(o));
  }
}

// part: float[gridDim.x][2 * K] (d mean, d std partial column sums); hist: float[2 * E] global (d mul, d bias), zeroed
// kDet (deterministic mode): no atomics.  hist is then float[n][2], each row's (dt * dist, dt), which
// gbf_edge_sum_kernel sums per edge type in a fixed order; shared memory holds every thread's column accumulators
// [rows_per_cta][2 * K], and each column of the CTA's partial row is their sum in row-group order.
template <typename T, bool kDet = false>
__global__ void __launch_bounds__(kGbfThreads) gbf_bwd_kernel(const T* __restrict__ dy, const T* __restrict__ d,
                                                               const long long* __restrict__ edge,
                                                               const T* __restrict__ mul_w, const T* __restrict__ bias_w,
                                                               const T* __restrict__ means, const T* __restrict__ stds,
                                                               float* __restrict__ part, float* __restrict__ hist,
                                                               long long n, int K, int E) {
  extern __shared__ float sm[];            // [2 * E] histogram, then [2 * K] column accumulators
  float* sm_hist = sm;
  float* sm_col = sm + 2 * E;
  if constexpr (!kDet) {
    for (int i = threadIdx.x; i < 2 * E + 2 * K; i += kGbfThreads) sm[i] = 0.f;
    __syncthreads();
  }
  const int kvec = K / 8;
  const int rows_per_cta = kGbfThreads / kvec;
  const int j = threadIdx.x % kvec, rl = threadIdx.x / kvec;
  const bool active = rl < rows_per_cta;
  float m[8], inv_s[8], norm[8], dm[8], ds[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) dm[e] = ds[e] = 0.f;
  if (active) {
    float sv[8];
    unpack<T>(ld_global_v4(means + j * 8), m);
    unpack<T>(ld_global_v4(stds + j * 8), sv);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float s = fabsf(sv[e]) + 1e-5f;
      inv_s[e] = 1.f / s;
      norm[e] = 1.f / (kGbfA * s);
    }
  }
  const long long n_iter = (n + (long long)gridDim.x * rows_per_cta - 1) / ((long long)gridDim.x * rows_per_cta);
  for (long long it = 0; it < n_iter; ++it) {
    const long long row = (it * gridDim.x + blockIdx.x) * rows_per_cta + rl;
    float dt = 0.f, dist = 0.f;
    long long e_idx = 0;
    if (active && row < n) {
      e_idx = edge[row];
      dist = to_f32<T>(d[row]);
      const float t = to_f32<T>(mul_w[e_idx]) * dist + to_f32<T>(bias_w[e_idx]);
      float g[8];
      unpack<T>(ld_global_nc_v4(dy + row * K + j * 8), g);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float z = (t - m[e]) * inv_s[e];               // (t - mean) / std
        const float yv = __expf(-0.5f * z * z) * norm[e];
        const float gy = g[e] * yv;
        const float zs = z * inv_s[e];                       // (t - mean) / std^2
        dt -= gy * zs;
        dm[e] += gy * zs;
        ds[e] += gy * (z * z - 1.f) * inv_s[e];              // y ((t-m)^2 / s^3 - 1 / s)
      }
    }
    // the kvec threads of a row sit in one warp segment (kvec is a power of two <= 32): reduce dt among them
    for (int o = kvec >> 1; o > 0; o >>= 1) dt += __shfl_xor_sync(0xffffffffu, dt, o);
    if (active && row < n && j == 0) {
      if constexpr (kDet) {
        *reinterpret_cast<float2*>(hist + 2 * row) = make_float2(dt * dist, dt);
      } else {
        atomicAdd(&sm_hist[e_idx], dt * dist);
        atomicAdd(&sm_hist[E + e_idx], dt);
      }
    }
  }
  if constexpr (kDet) {
    if (active) {
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        sm[(size_t)rl * 2 * K + j * 8 + e] = dm[e];
        sm[(size_t)rl * 2 * K + K + j * 8 + e] = ds[e];
      }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 2 * K; i += kGbfThreads) {
      float s = 0.f;
      for (int r = 0; r < rows_per_cta; ++r) s += sm[(size_t)r * 2 * K + i];
      part[(size_t)blockIdx.x * 2 * K + i] = s;
    }
    return;
  }
  if (active) {
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      atomicAdd(&sm_col[j * 8 + e], dm[e]);
      atomicAdd(&sm_col[K + j * 8 + e], ds[e]);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2 * K; i += kGbfThreads) part[(size_t)blockIdx.x * 2 * K + i] = sm_col[i];
  for (int i = threadIdx.x; i < 2 * E; i += kGbfThreads) {
    const float v = sm_hist[i];
    if (v != 0.f) atomicAdd(&hist[i], v);
  }
}

// Deterministic d mul / d bias: `rowg` [n][2] from gbf_bwd_kernel<T, true>; `sorted` / `perm` the stable-sorted edge
// types and their row indices.  A CTA per edge type e finds its run by binary search and sums (dt * dist, dt) over it
// in ascending row order, from 0: the CTA stages 256 rows in shared memory, thread 0 adds them in order.
// hist: float[2 * E], zeroed (types with no row, and ids outside [0, E), contribute nothing).
constexpr int kGbfSumThreads = 256;

__global__ void __launch_bounds__(kGbfSumThreads) gbf_edge_sum_kernel(const float* __restrict__ rowg,
                                                                       const long long* __restrict__ sorted,
                                                                       const long long* __restrict__ perm,
                                                                       float* __restrict__ hist, long long n, int E) {
  __shared__ long long run[2];
  __shared__ float2 stage[kGbfSumThreads];
  for (int e = blockIdx.x; e < E; e += gridDim.x) {
    if (threadIdx.x < 2) {
      long long lo = 0, hi = n;
      const long long key = e + threadIdx.x;
      while (lo < hi) {
        const long long mid = (lo + hi) >> 1;
        if (sorted[mid] < key) lo = mid + 1;
        else hi = mid;
      }
      run[threadIdx.x] = lo;
    }
    __syncthreads();
    const long long r0 = run[0], r1 = run[1];
    __syncthreads();   // run[] is rewritten for the next edge type
    float a = 0.f, b = 0.f;
    for (long long c = r0; c < r1; c += kGbfSumThreads) {
      const long long r = c + threadIdx.x;
      if (r < r1) stage[threadIdx.x] = *reinterpret_cast<const float2*>(rowg + 2 * perm[r]);
      __syncthreads();
      if (threadIdx.x == 0) {
        const int m = (int)(r1 - c < kGbfSumThreads ? r1 - c : kGbfSumThreads);
        for (int u = 0; u < m; ++u) {
          a += stage[u].x;
          b += stage[u].y;
        }
      }
      __syncthreads();
    }
    if (threadIdx.x == 0 && r1 > r0) {
      hist[e] = a;
      hist[E + e] = b;
    }
  }
}

GbfPlan gbf_plan(long long n, int K, int E) {
  GbfPlan p;
  p.kvec = K / 8;
  p.rows_per_cta = kGbfThreads / p.kvec;
  const SweepPlan s = sweep_plan(n, p.rows_per_cta, 4);
  p.grid = s.grid;
  p.rows_per_sweep = s.items_per_sweep;
  p.sweeps = s.sweeps;
  p.smem = (2 * E + 2 * K) * (int)sizeof(float);
  return p;
}

static int gbf_grid(long long n, int K) { return gbf_plan(n, K, 0).grid; }

// (no rows: no partial rows, their column sums are zero)
int gbf_parts(long long n, int K) { return gbf_grid(n, K); }

void launch_gbf_fwd(const void* d, const long long* edge, const void* mul_w, const void* bias_w, const void* means,
                    const void* stds, void* y, long long n, int K, int dtype, cudaStream_t stream) {
  if (n <= 0) return;
  const int grid = gbf_grid(n, K);
  UB_DISPATCH_16BIT(dtype, (gbf_fwd_kernel<T><<<grid, kGbfThreads, 0, stream>>>(
                               (const T*)d, edge, (const T*)mul_w, (const T*)bias_w, (const T*)means, (const T*)stds,
                               (T*)y, n, K)));
}

void launch_gbf_bwd(const void* dy, const void* d, const long long* edge, const void* mul_w, const void* bias_w,
                    const void* means, const void* stds, float* part, float* hist, long long n, int K, int E, int dtype,
                    cudaStream_t stream) {
  if (n <= 0) return;
  const GbfPlan plan = gbf_plan(n, K, E);
  const size_t smem = (size_t)plan.smem;
  UB_DISPATCH_16BIT(dtype, {
    auto kern = gbf_bwd_kernel<T>;
    if (smem > 48 * 1024) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    kern<<<plan.grid, kGbfThreads, smem, stream>>>((const T*)dy, (const T*)d, edge, (const T*)mul_w, (const T*)bias_w,
                                                   (const T*)means, (const T*)stds, part, hist, n, K, E);
  });
}

void launch_gbf_bwd_det(const void* dy, const void* d, const long long* edge, const void* mul_w, const void* bias_w,
                        const void* means, const void* stds, float* part, float* rowg, const long long* sorted,
                        const long long* perm, float* hist, long long n, int K, int E, int dtype, cudaStream_t stream) {
  if (n <= 0) return;
  const int grid = gbf_grid(n, K);
  const size_t smem = (size_t)kGbfThreads * 16 * sizeof(float);   // [rows_per_cta][2 * K] = 256 / (K / 8) * 2 * K
  UB_DISPATCH_16BIT(dtype, (gbf_bwd_kernel<T, true><<<grid, kGbfThreads, smem, stream>>>(
                               (const T*)dy, (const T*)d, edge, (const T*)mul_w, (const T*)bias_w, (const T*)means,
                               (const T*)stds, part, rowg, n, K, E)));
  const int egrid = sweep_plan(E, 1, 8).grid;
  if (egrid > 0) gbf_edge_sum_kernel<<<egrid, kGbfSumThreads, 0, stream>>>(rowg, sorted, perm, hist, n, E);
}

}  // namespace ub
