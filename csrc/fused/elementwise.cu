// Fused element-wise / row-reduction kernels around the transformer GEMMs (sm_90a):
//   bias + exact GELU (fwd/bwd), and softmax cross-entropy over the vocabulary (fwd/bwd) that never
//   materialises fp32 log-probabilities.  All are pure HBM streams: 128-bit (or the widest legal)
//   accesses, fp32 math, grid sized to fill every SM with 8 CTAs.
// Reference formulation: separate ATen kernels - fc1 bias add + GELU (unicore/modules/transformer_encoder_layer.py:79-94),
// fp32 log_softmax + nll_loss over [n_masked, vocab] (unicore/losses/masked_lm.py:37-47).
#include <math_constants.h>

#include "../api.h"
#include "../common.cuh"

namespace ub {

// ================================================================================================
// bias + GELU
//
// exact (erf) GELU = x * Phi(x).  CUDA's erff costs ~40 issued instructions per element, which made
// the first version of this kernel issue-bound at 2x its HBM time.  Phi is evaluated instead with
// the classic 5-term rational/exponential form (Abramowitz-Stegun 26.2.17), on element pairs (common.cuh F2):
//   t = 1 / (1 + 0.2316419 |x|),  pdf = exp(-x^2/2) / sqrt(2 pi),
//   Q = pdf * t (b1 + t (b2 + t (b3 + t (b4 + t b5)))),  Phi(x) = 1 - Q for x >= 0,  Q for x < 0.
// The formula's absolute error is < 7.5e-8, but GELU's negative tail is far smaller than that in
// absolute terms, so what matters there is the relative error of Q: 0.16 % at x = -5, 0.36 % at -6,
// 1.0 % at -8, 3.7 % at -13 (under one bf16 ulp down to -6; |GELU| < 5e-15 below -8).  Forming the
// tail as 0.5 - (0.5 - Q) instead cancels to an absolute fp32 error of ~2^-25 and returns 0 for x < -5.75.
// Layout: a thread owns one 8-wide column vector (its bias slice lives in registers) and walks
// rows; the backward also accumulates the bias gradient (column sums of dx) in registers, so no
// separate reduction pass over dx is needed.
// ================================================================================================
struct PhiPdf {
  F2 phi, pdf;
};
UB_DEVICE PhiPdf normal_cdf_pdf2(F2 x) {
  const unsigned long long xb = f2_bits(x);
  const F2 ax = f2_from_bits(xb & 0x7fffffff7fffffffull);
  const F2 den = fma2(ax, f2(0.2316419f), f2(1.f));
  F2 t;
  t.x = rcp_approx(den.x);
  t.y = rcp_approx(den.y);
  const F2 arg = mul2(mul2(x, x), f2(-0.72134752044448170368f));  // -x^2/2 * log2(e)
  F2 e;
  e.x = ex2_approx(arg.x);
  e.y = ex2_approx(arg.y);
  F2 poly = fma2(t, f2(1.330274429f), f2(-1.821255978f));
  poly = fma2(poly, t, f2(1.781477937f));
  poly = fma2(poly, t, f2(-0.356563782f));
  poly = fma2(poly, t, f2(0.319381530f));
  poly = mul2(poly, t);
  PhiPdf r;
  r.pdf = mul2(e, f2(0.39894228040143267794f));
  const F2 q = mul2(r.pdf, poly);                      // upper tail of |x|, in (0, 0.5]
  const F2 d = fma2(q, f2(-1.f), f2(0.5f));             // 0.5 - Q >= 0
  const F2 p = add2(d, f2(0.5f));                       // x >= 0: 1 - Q
  r.phi.x = x.x < 0.f ? q.x : p.x;                       // x < 0: Q itself (see above)
  r.phi.y = x.y < 0.f ? q.y : p.y;
  return r;
}

constexpr int kGeluColsPerCta = 128;  // column vectors per CTA (x 2 row lanes = 256 threads)
constexpr int kGeluUnroll = 4;

template <typename T, bool kBwd>
__global__ void __launch_bounds__(256) bias_gelu_kernel(const T* __restrict__ dy, const T* __restrict__ x,
                                                          const T* __restrict__ bias, T* __restrict__ out,
                                                          float* __restrict__ part, int rows, int nvec) {
  constexpr int EPV = 8;
  __shared__ float red[kGeluColsPerCta][EPV + 1];
  const int cv = blockIdx.x * kGeluColsPerCta + (threadIdx.x & (kGeluColsPerCta - 1));
  const int rl = threadIdx.x / kGeluColsPerCta;  // 0 / 1
  const bool col_ok = cv < nvec;
  const int cols = nvec * EPV;
  F2 b2[4], acc[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) b2[k] = acc[k] = f2(0.f);
  if (col_ok && bias != nullptr) {
    float bs[EPV];
    unpack<T>(ld_global_v4(bias + (size_t)cv * EPV), bs);
#pragma unroll
    for (int k = 0; k < 4; ++k) b2[k] = F2{bs[2 * k], bs[2 * k + 1]};
  }
  const int row_step = gridDim.y * 2;
  if (col_ok) {
    for (int r0 = blockIdx.y * 2 + rl; r0 < rows; r0 += row_step * kGeluUnroll) {
      Vec16 xv[kGeluUnroll], gv[kGeluUnroll];
#pragma unroll
      for (int u = 0; u < kGeluUnroll; ++u) {
        const int r = r0 + u * row_step;
        if (r < rows) {
          const size_t off = (size_t)r * cols + (size_t)cv * EPV;
          xv[u] = ld_global_nc_v4(x + off);
          if (kBwd) gv[u] = ld_global_nc_v4(dy + off);
        }
      }
#pragma unroll
      for (int u = 0; u < kGeluUnroll; ++u) {
        const int r = r0 + u * row_step;
        if (r < rows) {
          float xs[EPV], g[EPV], o[EPV];
          unpack<T>(xv[u], xs);
          if (kBwd) unpack<T>(gv[u], g);
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const F2 xx = add2(F2{xs[2 * k], xs[2 * k + 1]}, b2[k]);
            const PhiPdf pp = normal_cdf_pdf2(xx);
            F2 res;
            if (kBwd) {
              // d gelu / dx = Phi(x) + x pdf(x)
              res = mul2(F2{g[2 * k], g[2 * k + 1]}, fma2(xx, pp.pdf, pp.phi));
              acc[k] = add2(acc[k], res);
            } else {
              res = mul2(xx, pp.phi);
            }
            o[2 * k] = res.x;
            o[2 * k + 1] = res.y;
          }
          st_global_v4(out + (size_t)r * cols + (size_t)cv * EPV, pack<T>(o));
        }
      }
    }
  }
  if (kBwd && part != nullptr) {
    // combine the two row lanes, publish one fp32 partial row per (column block, row slice)
    const int c = threadIdx.x & (kGeluColsPerCta - 1);
    if (rl == 1) {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        red[c][2 * k] = acc[k].x;
        red[c][2 * k + 1] = acc[k].y;
      }
    }
    __syncthreads();
    if (rl == 0 && col_ok) {
      float* dst = part + (size_t)blockIdx.y * cols + (size_t)cv * EPV;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        dst[2 * k] = acc[k].x + red[c][2 * k];
        dst[2 * k + 1] = acc[k].y + red[c][2 * k + 1];
      }
    }
  }
}

// Column sums of a [rows, cols] 16-bit matrix (bias gradient of a Linear layer: ATen runs a generic reduce at
// ~2 TB/s for these shapes).  Same geometry as bias_gelu_kernel: a thread owns one 16-byte column vector, two row
// lanes per CTA, kGeluUnroll rows in flight; fp32 partial rows, finished by launch_colsum_finalize.
template <typename T>
__global__ void __launch_bounds__(256) column_sum_kernel(const T* __restrict__ x, float* __restrict__ part, int rows,
                                                           int nvec) {
  constexpr int EPV = 8;
  __shared__ float red[kGeluColsPerCta][EPV + 1];
  const int c = threadIdx.x & (kGeluColsPerCta - 1);
  const int cv = blockIdx.x * kGeluColsPerCta + c;
  const int rl = threadIdx.x / kGeluColsPerCta;
  const bool col_ok = cv < nvec;
  const int cols = nvec * EPV;
  float acc[EPV];
#pragma unroll
  for (int e = 0; e < EPV; ++e) acc[e] = 0.f;
  const int row_step = gridDim.y * 2;
  if (col_ok) {
    for (int r0 = blockIdx.y * 2 + rl; r0 < rows; r0 += row_step * kGeluUnroll) {
      Vec16 xv[kGeluUnroll];
#pragma unroll
      for (int u = 0; u < kGeluUnroll; ++u) {
        const int r = r0 + u * row_step;
        if (r < rows) xv[u] = ld_global_nc_v4(x + (size_t)r * cols + (size_t)cv * EPV);
      }
#pragma unroll
      for (int u = 0; u < kGeluUnroll; ++u) {
        if (r0 + u * row_step < rows) {
          float xs[EPV];
          unpack<T>(xv[u], xs);
#pragma unroll
          for (int e = 0; e < EPV; ++e) acc[e] += xs[e];
        }
      }
    }
  }
  if (rl == 1) {
#pragma unroll
    for (int e = 0; e < EPV; ++e) red[c][e] = acc[e];
  }
  __syncthreads();
  if (rl == 0 && col_ok) {
    float* dst = part + (size_t)blockIdx.y * cols + (size_t)cv * EPV;
#pragma unroll
    for (int e = 0; e < EPV; ++e) dst[e] = acc[e] + red[c][e];
  }
}

ColumnPlan bias_gelu_plan(long long rows, int cols, bool fwd) {
  ColumnPlan p;
  p.nvec = cols / 8;
  p.col_blocks = (p.nvec + kGeluColsPerCta - 1) / kGeluColsPerCta;
  // The forward fits 5 CTAs per SM (48 registers): a grid of 16 CTAs per SM keeps the tail of the last wave short
  // (with 6, the 32 x 512 x 3072 fp16 forward ran 1.2 waves in 92 us, with 16 in 76 us: H100 80GB HBM3, 400 W limit).
  // The backward and the column sum keep 6 per SM: each slice adds a partial row to the final column pass.
  long long slices = ((long long)device_sm_count() * (fwd ? 16 : 6) + p.col_blocks - 1) / p.col_blocks;
  const long long max_slices = (rows + 2 * kGeluUnroll - 1) / (2 * kGeluUnroll);
  if (slices > max_slices) slices = max_slices;
  p.slices = (int)(slices < 1 ? 1 : slices);
  p.rows_per_sweep = 2LL * kGeluUnroll * p.slices;
  p.sweeps = (rows + p.rows_per_sweep - 1) / p.rows_per_sweep;
  return p;
}

int bias_gelu_parts(long long rows, int cols) { return bias_gelu_plan(rows, cols, false).slices; }

// out[cols] = column sums of x[rows, cols]; part = float[bias_gelu_parts(rows, cols) * cols] scratch
void launch_column_sum(const void* x, void* out, float* part, long long rows, int cols, int dtype, cudaStream_t stream,
                       int accumulate) {
  if (cols <= 0) return;
  const ColumnPlan p = bias_gelu_plan(rows, cols, false);
  const int parts = rows > 0 ? p.slices : 0;  // no rows: zero sums
  if (parts > 0)
    UB_DISPATCH_16BIT(dtype, (column_sum_kernel<T><<<dim3(p.col_blocks, parts), 256, 0, stream>>>((const T*)x, part,
                                                                                                (int)rows, p.nvec)));
  launch_colsum_finalize(part, parts, cols, out, accumulate, dtype, stream);
}

void launch_bias_gelu_fwd(const void* x, const void* bias, void* y, long long rows, int cols, int dtype,
                          cudaStream_t stream) {
  if (rows <= 0 || cols <= 0) return;
  const ColumnPlan p = bias_gelu_plan(rows, cols, true);
  UB_DISPATCH_16BIT(dtype, (bias_gelu_kernel<T, false><<<dim3(p.col_blocks, p.slices), 256, 0, stream>>>(
                               nullptr, (const T*)x, (const T*)bias, (T*)y, nullptr, (int)rows, p.nvec)));
}
// dbias (nullable): column sums of dx; part: float[bias_gelu_parts(rows, cols) * cols] scratch
void launch_bias_gelu_bwd(const void* dy, const void* x, const void* bias, void* dx, void* dbias, float* part,
                          long long rows, int cols, int dtype, cudaStream_t stream, int accumulate) {
  if (cols <= 0) return;
  const ColumnPlan p = bias_gelu_plan(rows, cols, false);
  const bool want = dbias != nullptr && part != nullptr;
  const int parts = rows > 0 ? p.slices : 0;  // no rows: zero sums
  if (parts > 0)
    UB_DISPATCH_16BIT(dtype, (bias_gelu_kernel<T, true><<<dim3(p.col_blocks, parts), 256, 0, stream>>>(
                                 (const T*)dy, (const T*)x, (const T*)bias, (T*)dx, want ? part : nullptr, (int)rows,
                                 p.nvec)));
  if (want) launch_colsum_finalize(part, parts, cols, dbias, accumulate, dtype, stream);
}

// ================================================================================================
// softmax cross entropy: one CTA per row, online (max, sum) in a single pass over the logits
// ================================================================================================
constexpr int kXentThreads = 512;

UB_DEVICE void online_merge(float& m, float& s, float m2, float s2) {
  const float mn = fmaxf(m, m2);
  if (mn == -CUDART_INF_F) {
    s = 0.f;
  } else {
    s = s * __expf(m - mn) + s2 * __expf(m2 - mn);
  }
  m = mn;
}

// The exponentials of the online sum are taken relative to the running max, or to 0 while that max is -inf (every
// element seen so far is -inf): exp(-inf - -inf) would be NaN, and a row with masked (-inf) logits is ordinary input.
// The state then stays (-inf, 0), as in online_merge; a NaN element still makes the sum NaN.
UB_DEVICE float online_ref(float mn) { return mn == -CUDART_INF_F ? 0.f : mn; }

UB_DEVICE void online_add(float& m, float& s, float v) {
  const float mn = fmaxf(m, v);
  const float r = online_ref(mn);
  s = s * __expf(m - r) + __expf(v - r);
  m = mn;
}

template <typename T>
UB_DEVICE void row_max_sum(const T* row, int cols, float& m, float& s) {
  // per-thread online softmax statistics, widest aligned access that the row start allows
  m = -CUDART_INF_F;
  s = 0.f;
  constexpr int EPV = VecTraits<T>::kElems;
  const uintptr_t addr = reinterpret_cast<uintptr_t>(row);
  int head = (int)(((16 - (addr & 15)) & 15) / sizeof(T));
  if (head > cols) head = cols;
  const int nvec = (cols - head) / EPV;
  const int tail_begin = head + nvec * EPV;
  for (int c = threadIdx.x; c < head; c += blockDim.x) online_add(m, s, to_f32<T>(row[c]));
  for (int vi = threadIdx.x; vi < nvec; vi += blockDim.x) {
    float xs[EPV];
    unpack<T>(ld_global_nc_v4(row + head + vi * EPV), xs);
    float lm = xs[0];
#pragma unroll
    for (int e = 1; e < EPV; ++e) lm = fmaxf(lm, xs[e]);
    const float mn = fmaxf(m, lm);
    const float r = online_ref(mn);
    float acc = 0.f;
#pragma unroll
    for (int e = 0; e < EPV; ++e) acc += __expf(xs[e] - r);
    s = s * __expf(m - r) + acc;
    m = mn;
  }
  for (int c = tail_begin + threadIdx.x; c < cols; c += blockDim.x) online_add(m, s, to_f32<T>(row[c]));
}

template <typename T>
__global__ void __launch_bounds__(kXentThreads) xent_fwd_kernel(const T* __restrict__ logits,
                                                                  const long long* __restrict__ target,
                                                                  float* __restrict__ loss_rows,
                                                                  float* __restrict__ lse_out, int cols,
                                                                  int stride, long long ignore_index) {
  __shared__ float sm_m[32], sm_s[32];
  const int rowi = blockIdx.x;
  const T* row = logits + (size_t)rowi * stride;
  float m, s;
  row_max_sum<T>(row, cols, m, s);
  // warp then block merge
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
    online_merge(m, s, m2, s2);
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  if (lane == 0) {
    sm_m[wid] = m;
    sm_s[wid] = s;
  }
  __syncthreads();
  if (wid == 0) {
    m = lane < nw ? sm_m[lane] : -CUDART_INF_F;
    s = lane < nw ? sm_s[lane] : 0.f;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
      online_merge(m, s, m2, s2);
    }
    if (lane == 0) {
      const float lse = m + __logf(s);
      lse_out[rowi] = lse;
      const long long t = target[rowi];
      loss_rows[rowi] = (t == ignore_index || t < 0 || t >= cols) ? 0.f : lse - to_f32<T>(row[t]);
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(kXentThreads) xent_bwd_kernel(const T* __restrict__ logits,
                                                                  const long long* __restrict__ target,
                                                                  const float* __restrict__ lse,
                                                                  const float* __restrict__ dloss,
                                                                  T* __restrict__ dlogits, int cols,
                                                                  int stride, long long ignore_index) {
  // rows are `stride` elements apart (a vocabulary padded for GEMM alignment); columns [cols, stride)
  // of the gradient are zero-filled so that it can feed the padded backward GEMMs directly
  constexpr int EPV = VecTraits<T>::kElems;
  const int rowi = blockIdx.x;
  const T* row = logits + (size_t)rowi * stride;
  T* drow = dlogits + (size_t)rowi * stride;
  const long long t = target[rowi];
  const bool ignored = (t == ignore_index || t < 0 || t >= cols);
  const float scale = ignored ? 0.f : __ldg(dloss);
  const float l = lse[rowi];
  const uintptr_t addr = reinterpret_cast<uintptr_t>(row);
  int head = (int)(((16 - (addr & 15)) & 15) / sizeof(T));
  if (head > cols) head = cols;
  const bool same_align = ((reinterpret_cast<uintptr_t>(drow) & 15) == (addr & 15));
  const int nvec = same_align ? (cols - head) / EPV : 0;
  if (!same_align) head = 0;
  const int tail_begin = head + nvec * EPV;
  for (int c = threadIdx.x; c < head; c += blockDim.x) {
    const float pr = __expf(to_f32<T>(row[c]) - l);
    drow[c] = from_f32<T>((pr - (c == t ? 1.f : 0.f)) * scale);
  }
  for (int vi = threadIdx.x; vi < nvec; vi += blockDim.x) {
    const int c0 = head + vi * EPV;
    float xs[EPV], o[EPV];
    unpack<T>(ld_global_nc_v4(row + c0), xs);
#pragma unroll
    for (int e = 0; e < EPV; ++e) o[e] = (__expf(xs[e] - l) - ((c0 + e) == t ? 1.f : 0.f)) * scale;
    st_global_v4(drow + c0, pack<T>(o));
  }
  for (int c = tail_begin + threadIdx.x; c < cols; c += blockDim.x) {
    const float pr = __expf(to_f32<T>(row[c]) - l);
    drow[c] = from_f32<T>((pr - (c == t ? 1.f : 0.f)) * scale);
  }
  for (int c = cols + threadIdx.x; c < stride; c += blockDim.x) drow[c] = from_f32<T>(0.f);
}

void launch_softmax_xent_fwd(const void* logits, const long long* target, float* loss_rows, float* lse, int rows,
                             int cols, int stride, long long ignore_index, int dtype, cudaStream_t stream) {
  if (rows <= 0) return;
  UB_DISPATCH_FLOAT(dtype, (xent_fwd_kernel<T><<<rows, kXentThreads, 0, stream>>>(
                               (const T*)logits, target, loss_rows, lse, cols, stride, ignore_index)));
}

void launch_softmax_xent_bwd(const void* logits, const long long* target, const float* lse, const float* dloss,
                             void* dlogits, int rows, int cols, int stride, long long ignore_index, int dtype,
                             cudaStream_t stream) {
  if (rows <= 0) return;
  UB_DISPATCH_FLOAT(dtype, (xent_bwd_kernel<T><<<rows, kXentThreads, 0, stream>>>(
                               (const T*)logits, target, lse, dloss, (T*)dlogits, cols, stride, ignore_index)));
}

}  // namespace ub
