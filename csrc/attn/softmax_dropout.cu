// softmax(x + mask + bias) followed by dropout, forward and backward, for sm_90a.
//
// Stand-alone counterpart of reference csrc/softmax_dropout/* (used when attention probabilities
// must be materialised, e.g. return_attn=True / head_dim 8 models; the BERT path uses the fused
// wgmma attention kernel instead).  Differences from the reference kernels:
//   * a row is owned by a group of 1..256 threads that keeps it in registers; 128-bit accesses;
//   * any row length that is a multiple of the vector width up to 8192 takes the fast path WITH
//     dropout (reference: dropout only for K <= 1024, block kernel on the default stream above);
//     other lengths use a scalar three-pass kernel;
//   * no dropout bit-mask tensor: keep/drop is recomputed from Philox(seed, offset, index) in
//     backward, which removes one output stream in forward and one input stream in backward;
//   * fully masked rows produce zeros instead of NaN.
// Contract kept: x is overwritten with the probabilities; mask row = row / mask_div; bias row =
// row % bias_rows; backward overwrites dy with dx = (d - sum(d*y)) * y, d = keep ? dy/(1-p) : 0.
//
// "Logits mode" (lse != nullptr) serves pair-representation models (Uni-Mol: the biased logits of one
// layer are the bias of the next, reference unicore/modules/multihead_attention.py:98-103 adds the bias
// in its own pass and clones before the softmax): the kernel writes z = x + mask + bias (rounded to the
// storage type, exactly what the unfused formulation feeds the softmax) to `logits`, the row
// log-sum-exp to `lse`, and the dropped-out probabilities to `out`; x is left untouched and no
// probability tensor is stored.  Backward rebuilds y = exp(z - lse) from the logits and adds the
// gradient that arrived for the logits output (`addend`) before its single store.
#include <math_constants.h>

#include <initializer_list>

#include "../api.h"
#include "../common.cuh"

namespace ub {

constexpr int kSmThreads = 256;

template <bool kMax>
UB_DEVICE float group_reduce(float v, int tpr, float* scratch) {
  if (tpr >= 32) {  // the common case, fully unrolled (the generic loop costs 7 instructions per step)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float other = __shfl_xor_sync(0xffffffffu, v, o);
      v = kMax ? fmaxf(v, other) : v + other;
    }
  } else {
    for (int o = tpr >> 1; o > 0; o >>= 1) {
      const float other = __shfl_xor_sync(0xffffffffu, v, o);
      v = kMax ? fmaxf(v, other) : v + other;
    }
  }
  if (tpr > 32) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int wpg = tpr >> 5, gfirst = (warp / wpg) * wpg;
    __syncthreads();
    if (lane == 0) scratch[warp] = v;
    __syncthreads();
    float r = scratch[gfirst];
    for (int w = 1; w < wpg; ++w) r = kMax ? fmaxf(r, scratch[gfirst + w]) : r + scratch[gfirst + w];
    v = r;
  }
  return v;
}

struct SmGeom {
  long long rows;
  int K, tpr, nvec;
  long long mask_div, bias_rows;
};

template <typename T, int VPT>
__global__ void __launch_bounds__(kSmThreads) softmax_dropout_fwd_kernel(
    const T* x, T* probs, T* __restrict__ out, const T* __restrict__ mask, const T* __restrict__ bias, SmGeom g, float p,
    float keep_scale, unsigned long long seed, unsigned long long offset, T* __restrict__ logits,
    float* __restrict__ lse) {
  // `probs` (what backward reads) may be x itself (the reference's in-place contract) or a separate buffer (non
  // in-place callers: no clone pass in front of the kernel)
  constexpr int EPV = VecTraits<T>::kElems;
  __shared__ float scratch[8];
  const int tpr = g.tpr, rows_per_cta = kSmThreads / tpr;
  const int grp = threadIdx.x / tpr, j = threadIdx.x % tpr;
  const uint32_t thresh = dropout_thresh14(p);
  const bool drop = p > 0.f;
  const bool logits_mode = lse != nullptr;
  // broadcast row lookups without 64-bit division (~100 emulated instructions each) in the common cases
  const bool bias_per_row = g.bias_rows >= g.rows, narrow = g.rows < (1ll << 31);
  const long long stride_rows = (long long)gridDim.x * rows_per_cta;
  const long long iters = (g.rows + stride_rows - 1) / stride_rows;
  for (long long it = 0; it < iters; ++it) {
    const long long row = (it * gridDim.x + blockIdx.x) * rows_per_cta + grp;
    const bool active = row < g.rows;
    float v[VPT][EPV];
    float mx = -CUDART_INF_F;
#pragma unroll
    for (int k = 0; k < VPT; ++k) {
      const int vi = j + k * tpr;
      if (active && vi < g.nvec) {
        unpack<T>(ld_global_nc_v4(x + row * g.K + (long long)vi * EPV), v[k]);
        if (mask != nullptr) {
          float t[EPV];
          const long long mrow = narrow ? (long long)((unsigned)row / (unsigned)g.mask_div) : row / g.mask_div;
          unpack<T>(ld_global_v4(mask + mrow * g.K + (long long)vi * EPV), t);
#pragma unroll
          for (int e = 0; e < EPV; ++e) v[k][e] += t[e];
        }
        if (bias != nullptr) {
          float t[EPV];
          const long long brow = bias_per_row ? row
                                 : narrow     ? (long long)((unsigned)row % (unsigned)g.bias_rows)
                                              : row % g.bias_rows;
          unpack<T>(ld_global_v4(bias + brow * g.K + (long long)vi * EPV), t);
#pragma unroll
          for (int e = 0; e < EPV; ++e) v[k][e] += t[e];
        }
        if (logits_mode) {
          const Vec16 z = pack<T>(v[k]);
          st_global_v4(logits + row * g.K + (long long)vi * EPV, z);
          unpack<T>(z, v[k]);  // the softmax sees the stored (rounded) logits
        }
#pragma unroll
        for (int e = 0; e < EPV; ++e) mx = fmaxf(mx, v[k][e]);
      } else {
#pragma unroll
        for (int e = 0; e < EPV; ++e) v[k][e] = -CUDART_INF_F;
      }
    }
    mx = group_reduce<true>(mx, tpr, scratch);
    if (mx == -CUDART_INF_F) mx = 0.f;  // fully masked row
    float sum = 0.f;
#pragma unroll
    for (int k = 0; k < VPT; ++k) {
#pragma unroll
      for (int e = 0; e < EPV; ++e) {
        v[k][e] = exp2f((v[k][e] - mx) * 1.4426950408889634f);
        sum += v[k][e];
      }
    }
    sum = group_reduce<false>(sum, tpr, scratch);
    const float inv = sum > 0.f ? 1.f / sum : 0.f;
    if (active) {
      if (logits_mode && j == 0) lse[row] = sum > 0.f ? mx + logf(sum) : CUDART_INF_F;
#pragma unroll
      for (int k = 0; k < VPT; ++k) {
        const int vi = j + k * tpr;
        if (vi < g.nvec) {
          const long long off = row * g.K + (long long)vi * EPV;
          float pr[EPV];
#pragma unroll
          for (int e = 0; e < EPV; ++e) pr[e] = v[k][e] * inv;
          const Vec16 packed = pack<T>(pr);
          if (!logits_mode) st_global_v4(probs + off, packed);
          else if (!drop) st_global_v4(out + off, packed);
          if (drop) {
            // out = keep ? p * keep_scale : 0, the scale applied in fp32 ahead of the single rounding
#pragma unroll
            for (int e = 0; e < EPV; ++e) pr[e] *= keep_scale;
            Vec16 o = pack<T>(pr);
            if constexpr (EPV == 8) {
              uint32_t m[4];
              dropout_lane_masks8(seed, offset, (unsigned long long)off >> 3, thresh, m);
#pragma unroll
              for (int w = 0; w < 4; ++w) o.w[w] &= m[w];
            } else {
              const uint32_t keep = dropout_keep8_14(seed, offset, (unsigned long long)off >> 3, thresh) >> (off & 7);
#pragma unroll
              for (int e = 0; e < EPV; ++e)
                if (!((keep >> e) & 1u)) o.w[e] = 0u;
            }
            st_global_v4(out + off, o);
          }
        }
      }
    }
  }
}

template <typename T, int VPT>
__global__ void __launch_bounds__(kSmThreads) softmax_dropout_bwd_kernel(
    const T* dy, T* dx, const T* __restrict__ probs, SmGeom g, float p, float keep_scale, unsigned long long seed,
    unsigned long long offset, const float* __restrict__ lse, const T* __restrict__ addend) {
  constexpr int EPV = VecTraits<T>::kElems;
  __shared__ float scratch[8];
  const int tpr = g.tpr, rows_per_cta = kSmThreads / tpr;
  const int grp = threadIdx.x / tpr, j = threadIdx.x % tpr;
  const uint32_t thresh = dropout_thresh14(p);
  const bool drop = p > 0.f;
  const long long stride_rows = (long long)gridDim.x * rows_per_cta;
  const long long iters = (g.rows + stride_rows - 1) / stride_rows;
  for (long long it = 0; it < iters; ++it) {
    const long long row = (it * gridDim.x + blockIdx.x) * rows_per_cta + grp;
    const bool active = row < g.rows;
    float d[VPT][EPV], y[VPT][EPV];
    float dot = 0.f;
    const float row_lse = (lse != nullptr && active) ? lse[row] : 0.f;
#pragma unroll
    for (int k = 0; k < VPT; ++k) {
      const int vi = j + k * tpr;
      if (active && vi < g.nvec) {
        const long long off = row * g.K + (long long)vi * EPV;
        Vec16 dyv = ld_global_nc_v4(dy + off);
        if (drop) {
          if constexpr (EPV == 8) {
            uint32_t m[4];
            dropout_lane_masks8(seed, offset, (unsigned long long)off >> 3, thresh, m);
#pragma unroll
            for (int w = 0; w < 4; ++w) dyv.w[w] &= m[w];
          } else {
            const uint32_t keep = dropout_keep8_14(seed, offset, (unsigned long long)off >> 3, thresh) >> (off & 7);
#pragma unroll
            for (int e = 0; e < EPV; ++e)
              if (!((keep >> e) & 1u)) dyv.w[e] = 0u;
          }
        }
        unpack<T>(dyv, d[k]);
        unpack<T>(ld_global_nc_v4(probs + off), y[k]);
        if (lse != nullptr) {  // `probs` holds logits: rebuild the (rounded) probabilities forward used
#pragma unroll
          for (int e = 0; e < EPV; ++e) y[k][e] = exp2f((y[k][e] - row_lse) * 1.4426950408889634f);
          unpack<T>(pack<T>(y[k]), y[k]);
        }
#pragma unroll
        for (int e = 0; e < EPV; ++e) {
          d[k][e] = d[k][e] * keep_scale * y[k][e];  // keep_scale is 1 without dropout
          dot += d[k][e];
        }
      } else {
#pragma unroll
        for (int e = 0; e < EPV; ++e) d[k][e] = y[k][e] = 0.f;
      }
    }
    dot = group_reduce<false>(dot, tpr, scratch);
    if (active) {
#pragma unroll
      for (int k = 0; k < VPT; ++k) {
        const int vi = j + k * tpr;
        if (vi < g.nvec) {
          const long long off = row * g.K + (long long)vi * EPV;
          float o[EPV];
#pragma unroll
          for (int e = 0; e < EPV; ++e) o[e] = d[k][e] - y[k][e] * dot;
          if (addend != nullptr) {
            float a[EPV];
            unpack<T>(ld_global_nc_v4(addend + off), a);
#pragma unroll
            for (int e = 0; e < EPV; ++e) o[e] += a[e];
          }
          st_global_v4(dx + off, pack<T>(o));
        }
      }
    }
  }
}

// ---- scalar fallback (row length not a multiple of the vector width): one warp per row ----------------
template <typename T>
__global__ void softmax_dropout_fwd_scalar(const T* x, T* probs, T* out, const T* mask, const T* bias, SmGeom g, float p,
                                           float keep_scale, unsigned long long seed, unsigned long long offset,
                                           T* logits, float* lse) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const uint32_t thresh = dropout_thresh14(p);
  const bool logits_mode = lse != nullptr;
  for (long long row = warp; row < g.rows; row += nwarps) {
    const T* xr = x + row * g.K;
    T* pr_row = probs + row * g.K;
    T* zr = logits_mode ? logits + row * g.K : nullptr;
    const T* mr = mask ? mask + (row / g.mask_div) * g.K : nullptr;
    const T* br = bias ? bias + (row % g.bias_rows) * g.K : nullptr;
    auto biased = [&](int c) { return to_f32<T>(xr[c]) + (mr ? to_f32<T>(mr[c]) : 0.f) + (br ? to_f32<T>(br[c]) : 0.f); };
    float mx = -CUDART_INF_F;
    for (int c = lane; c < g.K; c += 32) {
      float v = biased(c);
      if (logits_mode) {
        zr[c] = from_f32<T>(v);  // later passes re-read this thread's own stores
        v = to_f32<T>(zr[c]);
      }
      mx = fmaxf(mx, v);
    }
    mx = warp_max(mx);
    if (mx == -CUDART_INF_F) mx = 0.f;
    float sum = 0.f;
    for (int c = lane; c < g.K; c += 32) sum += expf((logits_mode ? to_f32<T>(zr[c]) : biased(c)) - mx);
    sum = warp_sum(sum);
    const float inv = sum > 0.f ? 1.f / sum : 0.f;
    if (logits_mode && lane == 0) lse[row] = sum > 0.f ? mx + logf(sum) : CUDART_INF_F;
    for (int c = lane; c < g.K; c += 32) {
      const float v = logits_mode ? to_f32<T>(zr[c]) : biased(c);
      const T pr = from_f32<T>(expf(v - mx) * inv);
      if (!logits_mode) pr_row[c] = pr;
      else if (p <= 0.f) out[row * g.K + c] = pr;
      if (p > 0.f) {
        const unsigned long long idx = (unsigned long long)(row * g.K + c);
        const uint32_t keep = dropout_keep8_14(seed, offset, idx >> 3, thresh);
        out[row * g.K + c] = ((keep >> (idx & 7)) & 1u) ? from_f32<T>(expf(v - mx) * inv * keep_scale) : from_f32<T>(0.f);
      }
    }
  }
}

template <typename T>
__global__ void softmax_dropout_bwd_scalar(const T* dy, T* dx, const T* probs, SmGeom g, float p, float keep_scale,
                                           unsigned long long seed, unsigned long long offset, const float* lse,
                                           const T* addend) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const uint32_t thresh = dropout_thresh14(p);
  for (long long row = warp; row < g.rows; row += nwarps) {
    const float row_lse = lse != nullptr ? lse[row] : 0.f;
    auto prob = [&](unsigned long long idx) {
      const float t = to_f32<T>(probs[idx]);
      return lse != nullptr ? to_f32<T>(from_f32<T>(expf(t - row_lse))) : t;
    };
    auto grad = [&](unsigned long long idx) {
      float d = to_f32<T>(dy[idx]);
      if (p > 0.f) {
        const uint32_t keep = dropout_keep8_14(seed, offset, idx >> 3, thresh);
        d = ((keep >> (idx & 7)) & 1u) ? d * keep_scale : 0.f;
      }
      return d;
    };
    float dot = 0.f;
    for (int c = lane; c < g.K; c += 32) {
      const unsigned long long idx = (unsigned long long)(row * g.K + c);
      dot += grad(idx) * prob(idx);
    }
    dot = warp_sum(dot);
    for (int c = lane; c < g.K; c += 32) {
      const unsigned long long idx = (unsigned long long)(row * g.K + c);
      float o = (grad(idx) - dot) * prob(idx);
      if (addend != nullptr) o += to_f32<T>(addend[idx]);
      dx[idx] = from_f32<T>(o);
    }
  }
}

// ---- host ------------------------------------------------------------------------------------------------------
static bool make_sm_geom(SmGeom& g, long long rows, int K, int epv, int& vpt) {
  g.rows = rows;
  g.K = K;
  if (K % epv != 0) return false;
  g.nvec = K / epv;
  return row_group_geom(g.nvec, g.tpr, vpt);
}

// The kernels are grid-stride loops over rows: launch exactly as many CTAs as fit on the machine at once.  (A fixed
// "8 per SM" left the register-limited kernels with 1.6 waves: the second wave ran on 60 % of the SMs.)
template <typename Kernel>
static int resident_per_sm(Kernel kernel) {
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kSmThreads, 0) != cudaSuccess || per_sm < 1) per_sm = 2;
  return per_sm;
}

template <typename T, int VPT>
static int resident_fwd() {
  static const int n = resident_per_sm(softmax_dropout_fwd_kernel<T, VPT>);
  return n;
}

template <typename T, int VPT>
static int resident_bwd() {
  static const int n = resident_per_sm(softmax_dropout_bwd_kernel<T, VPT>);
  return n;
}

template <typename T>
static SoftmaxPlan plan_sm(long long rows, int K, bool aligned, bool bwd, SmGeom& g) {
  SoftmaxPlan pl{};
  SweepPlan s;
  int vpt = 0;
  if (make_sm_geom(g, rows, K, VecTraits<T>::kElems, vpt) && aligned) {
    int per_sm = 0;
    UB_DISPATCH_VPT(vpt, per_sm = bwd ? resident_bwd<T, VPT>() : resident_fwd<T, VPT>());
    s = sweep_plan(rows, kSmThreads / g.tpr, per_sm);
    pl.vec = 1;
    pl.vpt = vpt;
    pl.tpr = g.tpr;
    pl.threads = kSmThreads;
  } else {  // scalar kernels: 8 warps per CTA, one row per warp
    s = sweep_plan(rows, 8, 8);
    pl.tpr = 32;
    pl.threads = 256;
  }
  pl.grid = s.grid;
  pl.rows_per_sweep = s.items_per_sweep;
  pl.sweeps = s.sweeps;
  return pl;
}

SoftmaxPlan softmax_plan(long long rows, int K, int dtype, bool aligned, bool bwd) {
  SmGeom g;
  UB_DISPATCH_FLOAT(dtype, return plan_sm<T>(rows, K, aligned, bwd, g));
  return SoftmaxPlan{};
}

// 1 / P(keep) for the 14-bit threshold the kernels compare against (mirrors dropout_thresh14)
static float keep_scale_for(float p) {
  if (!(p > 0.f)) return 1.f;
  const float t = p * 16384.f + 0.5f;
  const float t14 = t >= 16383.f ? 16383.f : (float)(unsigned)t;
  return 16384.f / (16384.f - t14);
}

static bool aligned16(std::initializer_list<const void*> ptrs) {
  uintptr_t bits = 0;
  for (const void* q : ptrs) bits |= reinterpret_cast<uintptr_t>(q);
  return (bits & 15) == 0;
}

template <typename T>
static void run_sm_fwd(void* x, void* out, const void* mask, const void* bias, long long rows, int K,
                       long long mask_div, long long bias_rows, float p, unsigned long long seed,
                       unsigned long long offset, void* logits, float* lse, cudaStream_t stream, void* probs) {
  SmGeom g;
  if (probs == nullptr) probs = x;
  const SoftmaxPlan pl = plan_sm<T>(rows, K, aligned16({x, out, probs, mask, bias, logits}), false, g);
  g.mask_div = mask_div > 0 ? mask_div : 1;
  g.bias_rows = bias_rows > 0 ? bias_rows : 1;
  const float keep_scale = keep_scale_for(p);
  if (pl.vec) {
    UB_DISPATCH_VPT(pl.vpt, {
      softmax_dropout_fwd_kernel<T, VPT><<<pl.grid, kSmThreads, 0, stream>>>(
          (const T*)x, (T*)probs, (T*)out, (const T*)mask, (const T*)bias, g, p, keep_scale, seed, offset, (T*)logits, lse);
    });
  } else {
    softmax_dropout_fwd_scalar<T><<<pl.grid, pl.threads, 0, stream>>>((const T*)x, (T*)probs, (T*)out, (const T*)mask,
                                                                      (const T*)bias, g, p, keep_scale, seed, offset,
                                                                      (T*)logits, lse);
  }
}

template <typename T>
static void run_sm_bwd(const void* dy, void* dx, const void* probs, long long rows, int K, float p, unsigned long long seed,
                       unsigned long long offset, const float* lse, const void* addend, cudaStream_t stream) {
  SmGeom g;
  const SoftmaxPlan pl = plan_sm<T>(rows, K, aligned16({dy, dx, probs, addend}), true, g);
  g.mask_div = 1;
  g.bias_rows = 1;
  const float keep_scale = keep_scale_for(p);
  if (pl.vec) {
    UB_DISPATCH_VPT(pl.vpt, {
      softmax_dropout_bwd_kernel<T, VPT><<<pl.grid, kSmThreads, 0, stream>>>(
          (const T*)dy, (T*)dx, (const T*)probs, g, p, keep_scale, seed, offset, lse, (const T*)addend);
    });
  } else {
    softmax_dropout_bwd_scalar<T><<<pl.grid, pl.threads, 0, stream>>>((const T*)dy, (T*)dx, (const T*)probs, g, p,
                                                                      keep_scale, seed, offset, lse, (const T*)addend);
  }
}

void launch_softmax_dropout_fwd(void* x, void* out, const void* mask, const void* bias, long long rows, int K,
                                long long mask_div, long long bias_rows, float p, unsigned long long seed,
                                unsigned long long offset, int dtype, cudaStream_t stream, void* logits, float* lse,
                                void* probs) {
  if (rows <= 0 || K <= 0) return;
  UB_DISPATCH_FLOAT(dtype, run_sm_fwd<T>(x, out, mask, bias, rows, K, mask_div, bias_rows, p, seed, offset, logits, lse,
                                         stream, probs));
}

void launch_softmax_dropout_bwd(const void* dy, void* dx, const void* probs, long long rows, int K, float p,
                                unsigned long long seed, unsigned long long offset, int dtype, cudaStream_t stream,
                                const float* lse, const void* addend) {
  if (rows <= 0 || K <= 0) return;
  UB_DISPATCH_FLOAT(dtype, run_sm_bwd<T>(dy, dx, probs, rows, K, p, seed, offset, lse, addend, stream));
}

}  // namespace ub
