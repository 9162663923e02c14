// Gradient of an embedding lookup  y[r, :] = W[token[r], :]  (unicore/modules of the reference use nn.Embedding; its
// backward in ATen is a radix sort of the indices + segmented reduction: ~30 launches per BERT-base step).
//
// Two kernels, no sort:
//   scatter : a warp per row adds dy[r, :] (as fp32) into scratch[token[r], :] with red.global.add.v4.f32 and marks
//             the vocabulary row as touched.  fp32 accumulation: a frequent token ([MASK], punctuation) sums thousands
//             of rows, which fp16 atomics would round after every add.
//   finalize: a warp per vocabulary row; touched rows are added to (or written into) the 16-bit gradient and their
//             scratch + flag are cleared again, so the scratch buffer is persistent and never needs a memset.
// The 16-bit gradient is the optimizer's flat arena view when the parameter is claimed (ops/grad_sink.py).
// The red-adds land in scheduler order, so the fp32 sums can differ in the last bits from run to run.  Under
// torch.use_deterministic_algorithms the binding sorts the ids instead and embedding_sorted_kernel sums each row's run
// in a fixed order (no scratch, no flags).
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "../api.h"
#include "../common.cuh"

namespace ub {
namespace {

UB_DEVICE void red_add_v4(float* addr, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

constexpr int kEmbThreads = 256;

template <typename T>
__global__ void __launch_bounds__(kEmbThreads) embedding_scatter_kernel(const T* __restrict__ dy,
                                                                        const long long* __restrict__ tokens,
                                                                        float* __restrict__ scratch,
                                                                        unsigned char* __restrict__ touched, long long rows,
                                                                        int cols, long long vocab, long long padding_idx) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * kEmbThreads + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * kEmbThreads) >> 5;
  const int vecs = cols >> 3;
  for (long long r = warp; r < rows; r += n_warps) {
    const long long tok = tokens[r];
    if (tok == padding_idx || tok < 0 || tok >= vocab) continue;
    if (lane == 0) touched[tok] = 1;
    const T* src = dy + r * cols;
    float* dst = scratch + tok * cols;
    for (int v = lane; v < vecs; v += 32) {
      float f[8];
      unpack<T>(ld_global_nc_v4(src + v * 8), f);
      red_add_v4(dst + v * 8, f[0], f[1], f[2], f[3]);
      red_add_v4(dst + v * 8 + 4, f[4], f[5], f[6], f[7]);
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(kEmbThreads) embedding_finalize_kernel(float* __restrict__ scratch,
                                                                         unsigned char* __restrict__ touched,
                                                                         T* __restrict__ grad, long long vocab, int cols,
                                                                         int accumulate) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * kEmbThreads + threadIdx.x) >> 5;
  const long long n_warps = ((long long)gridDim.x * kEmbThreads) >> 5;
  const int vecs = cols >> 3;
  for (long long row = warp; row < vocab; row += n_warps) {
    if (touched[row] == 0) continue;   // same byte for the whole warp: no divergence
    __syncwarp();
    if (lane == 0) touched[row] = 0;
    float* src = scratch + row * cols;
    T* dst = grad + row * cols;
    for (int v = lane; v < vecs; v += 32) {
      float4 a = *reinterpret_cast<const float4*>(src + v * 8);
      float4 b = *reinterpret_cast<const float4*>(src + v * 8 + 4);
      float f[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
      if (accumulate) {
        float g[8];
        unpack<T>(*reinterpret_cast<const Vec16*>(dst + v * 8), g);
#pragma unroll
        for (int e = 0; e < 8; ++e) f[e] += g[e];
      }
      *reinterpret_cast<Vec16*>(dst + v * 8) = pack<T>(f);
      const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
      *reinterpret_cast<float4*>(src + v * 8) = z;
      *reinterpret_cast<float4*>(src + v * 8 + 4) = z;
    }
  }
}

// Deterministic mode: `sorted` / `perm` are the token ids stable-sorted and their original row indices, so the rows of
// vocabulary row v are the run perm[lo .. hi) in ascending original order.  A CTA per vocabulary row, threads over
// 8-column vectors: each column is summed in fp32 strictly in that order, starting from 0.0f; with `accumulate` the
// existing 16-bit gradient is then added in fp32 and the result rounded once.  A float32 loop on the host over the rows
// in ascending order reproduces it bit for bit.
UB_DEVICE long long lower_bound_ll(const long long* __restrict__ a, long long n, long long key) {
  long long lo = 0, hi = n;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (a[mid] < key) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

constexpr int kEmbDetThreads = 128;

template <typename T>
__global__ void __launch_bounds__(kEmbDetThreads) embedding_sorted_kernel(const T* __restrict__ dy,
                                                                         const long long* __restrict__ sorted,
                                                                         const long long* __restrict__ perm,
                                                                         T* __restrict__ grad, long long rows, int cols,
                                                                         long long vocab, long long padding_idx,
                                                                         int accumulate) {
  __shared__ long long run[2];
  const int vecs = cols >> 3;
  for (long long row = blockIdx.x; row < vocab; row += gridDim.x) {
    if (row == padding_idx) continue;
    if (threadIdx.x < 2) run[threadIdx.x] = lower_bound_ll(sorted, rows, row + threadIdx.x);
    __syncthreads();
    const long long lo = run[0], hi = run[1];
    __syncthreads();   // run[] is rewritten for the next row
    if (lo == hi) continue;
    for (int v = threadIdx.x; v < vecs; v += kEmbDetThreads) {
      float f[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      long long r = lo;
      for (; r + 4 <= hi; r += 4) {   // four loads in flight, added in order
        Vec16 in[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) in[u] = ld_global_nc_v4(dy + perm[r + u] * cols + v * 8);
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          float x[8];
          unpack<T>(in[u], x);
#pragma unroll
          for (int e = 0; e < 8; ++e) f[e] += x[e];
        }
      }
      for (; r < hi; ++r) {
        float x[8];
        unpack<T>(ld_global_nc_v4(dy + perm[r] * cols + v * 8), x);
#pragma unroll
        for (int e = 0; e < 8; ++e) f[e] += x[e];
      }
      T* dst = grad + row * cols + v * 8;
      if (accumulate) {
        float g[8];
        unpack<T>(*reinterpret_cast<const Vec16*>(dst), g);
#pragma unroll
        for (int e = 0; e < 8; ++e) f[e] += g[e];
      }
      *reinterpret_cast<Vec16*>(dst) = pack<T>(f);
    }
  }
}

}  // namespace

void launch_embedding_bwd_sorted(const void* dy, const long long* sorted, const long long* perm, void* grad,
                                 long long rows, int cols, long long vocab, long long padding_idx, int accumulate,
                                 int dtype, cudaStream_t stream) {
  if (rows == 0 || vocab == 0) return;
  const unsigned grid = (unsigned)(vocab < 132 * 16 ? vocab : 132 * 16);
  if (dtype == kBF16)
    embedding_sorted_kernel<__nv_bfloat16><<<grid, kEmbDetThreads, 0, stream>>>(
        reinterpret_cast<const __nv_bfloat16*>(dy), sorted, perm, reinterpret_cast<__nv_bfloat16*>(grad), rows, cols,
        vocab, padding_idx, accumulate);
  else
    embedding_sorted_kernel<__half><<<grid, kEmbDetThreads, 0, stream>>>(reinterpret_cast<const __half*>(dy), sorted, perm,
                                                                         reinterpret_cast<__half*>(grad), rows, cols,
                                                                         vocab, padding_idx, accumulate);
}

void launch_embedding_bwd(const void* dy, const long long* tokens, float* scratch, unsigned char* touched, void* grad,
                          long long rows, int cols, long long vocab, long long padding_idx, int accumulate, int dtype,
                          cudaStream_t stream) {
  const int warps_per_block = kEmbThreads / 32;
  long long b1 = (rows + warps_per_block - 1) / warps_per_block;
  if (b1 > 132 * 16) b1 = 132 * 16;
  long long b2 = (vocab + warps_per_block - 1) / warps_per_block;
  if (b2 > 132 * 16) b2 = 132 * 16;
  if (rows == 0) b1 = 0;
  if (dtype == kBF16) {
    if (b1 > 0)
      embedding_scatter_kernel<__nv_bfloat16><<<(unsigned)b1, kEmbThreads, 0, stream>>>(
          reinterpret_cast<const __nv_bfloat16*>(dy), tokens, scratch, touched, rows, cols, vocab, padding_idx);
    embedding_finalize_kernel<__nv_bfloat16><<<(unsigned)b2, kEmbThreads, 0, stream>>>(
        scratch, touched, reinterpret_cast<__nv_bfloat16*>(grad), vocab, cols, accumulate);
  } else {
    if (b1 > 0)
      embedding_scatter_kernel<__half><<<(unsigned)b1, kEmbThreads, 0, stream>>>(
          reinterpret_cast<const __half*>(dy), tokens, scratch, touched, rows, cols, vocab, padding_idx);
    embedding_finalize_kernel<__half><<<(unsigned)b2, kEmbThreads, 0, stream>>>(scratch, touched, reinterpret_cast<__half*>(grad),
                                                                               vocab, cols, accumulate);
  }
}

}  // namespace ub
