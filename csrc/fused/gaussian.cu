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
template <typename T>
__global__ void __launch_bounds__(kGbfThreads) gbf_bwd_kernel(const T* __restrict__ dy, const T* __restrict__ d,
                                                               const long long* __restrict__ edge,
                                                               const T* __restrict__ mul_w, const T* __restrict__ bias_w,
                                                               const T* __restrict__ means, const T* __restrict__ stds,
                                                               float* __restrict__ part, float* __restrict__ hist,
                                                               long long n, int K, int E) {
  extern __shared__ float sm[];            // [2 * E] histogram, then [2 * K] column accumulators
  float* sm_hist = sm;
  float* sm_col = sm + 2 * E;
  for (int i = threadIdx.x; i < 2 * E + 2 * K; i += kGbfThreads) sm[i] = 0.f;
  __syncthreads();
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
      atomicAdd(&sm_hist[e_idx], dt * dist);
      atomicAdd(&sm_hist[E + e_idx], dt);
    }
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

static int gbf_grid(long long n, int K) {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int rows_per_cta = kGbfThreads / (K / 8);
  const long long need = (n + rows_per_cta - 1) / rows_per_cta;
  const long long cap = (long long)sms * 4;
  return (int)(need < cap ? (need < 1 ? 1 : need) : cap);
}

int gbf_parts(long long n, int K) { return gbf_grid(n, K); }

void launch_gbf_fwd(const void* d, const long long* edge, const void* mul_w, const void* bias_w, const void* means,
                    const void* stds, void* y, long long n, int K, int dtype, cudaStream_t stream) {
  if (n <= 0) return;
  const int grid = gbf_grid(n, K);
  if (dtype == kF16)
    gbf_fwd_kernel<__half><<<grid, kGbfThreads, 0, stream>>>((const __half*)d, edge, (const __half*)mul_w,
                                                             (const __half*)bias_w, (const __half*)means,
                                                             (const __half*)stds, (__half*)y, n, K);
  else
    gbf_fwd_kernel<__nv_bfloat16><<<grid, kGbfThreads, 0, stream>>>(
        (const __nv_bfloat16*)d, edge, (const __nv_bfloat16*)mul_w, (const __nv_bfloat16*)bias_w,
        (const __nv_bfloat16*)means, (const __nv_bfloat16*)stds, (__nv_bfloat16*)y, n, K);
}

void launch_gbf_bwd(const void* dy, const void* d, const long long* edge, const void* mul_w, const void* bias_w,
                    const void* means, const void* stds, float* part, float* hist, long long n, int K, int E, int dtype,
                    cudaStream_t stream) {
  if (n <= 0) return;
  const int grid = gbf_grid(n, K);
  const size_t smem = (size_t)(2 * E + 2 * K) * sizeof(float);
  if (dtype == kF16) {
    auto kern = gbf_bwd_kernel<__half>;
    if (smem > 48 * 1024) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    kern<<<grid, kGbfThreads, smem, stream>>>((const __half*)dy, (const __half*)d, edge, (const __half*)mul_w,
                                              (const __half*)bias_w, (const __half*)means, (const __half*)stds, part,
                                              hist, n, K, E);
  } else {
    auto kern = gbf_bwd_kernel<__nv_bfloat16>;
    if (smem > 48 * 1024) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    kern<<<grid, kGbfThreads, smem, stream>>>((const __nv_bfloat16*)dy, (const __nv_bfloat16*)d, edge,
                                              (const __nv_bfloat16*)mul_w, (const __nv_bfloat16*)bias_w,
                                              (const __nv_bfloat16*)means, (const __nv_bfloat16*)stds, part, hist, n, K, E);
  }
}

}  // namespace ub
