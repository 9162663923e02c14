// Multi-tensor optimizer kernels for sm_90a: L2 norm, scale, Adam (+16-bit write-back,
// stochastic rounding, EMA, grad zeroing), fp32->bf16 stochastic rounding, EMA.
//
// Replaces reference csrc/adam/adam_kernel.cu:16-152 (scalar accesses, one launch per tensor),
// csrc/multi_tensor/multi_tensor_l2norm_kernel.cu:27-118 (chunk table by value + separate cleanup kernel) and
// csrc/rounding/fp32_to_bf16.cu:23-59 (curand_init per element).
//
// Design: up to 24 tensors per launch are described by value in the kernel parameter block.
// Work is cut into fixed chunks of kChunk elements; a persistent grid walks the chunk list
// (chunk -> tensor by scanning <= 24 prefix entries). Every thread moves 8 elements per iteration
// with 128-bit loads/stores; all math is fp32. HBM traffic per element (mixed precision step):
// g16 2B + p32 4B + m 4B + v 4B read, p32 4B + m 4B + v 4B + p16 2B + g16 2B (zero) write = 30 B.
#include "../api.h"
#include "../common.cuh"
#include "adam_math.cuh"

namespace ub {

constexpr int kThreads = 256;
constexpr long long kChunk = 8192;  // elements per chunk = 256 threads x 8 elems x 4 iterations

// ---- dtype-generic 8-element access (pointer 16B aligned, idx multiple of 8) -------------------
UB_DEVICE void load8(const void* base, int dtype, long long i, float* out) {
  if (dtype == kF32) {
    const float* p = reinterpret_cast<const float*>(base) + i;
    Vec16 a = ld_global_v4(p), b = ld_global_v4(p + 4);
    unpack<float>(a, out);
    unpack<float>(b, out + 4);
  } else if (dtype == kF16) {
    Vec16 a = ld_global_v4(reinterpret_cast<const __half*>(base) + i);
    unpack<__half>(a, out);
  } else {
    Vec16 a = ld_global_v4(reinterpret_cast<const __nv_bfloat16*>(base) + i);
    unpack<__nv_bfloat16>(a, out);
  }
}
UB_DEVICE void store8(void* base, int dtype, long long i, const float* in) {
  if (dtype == kF32) {
    float* p = reinterpret_cast<float*>(base) + i;
    st_global_v4(p, pack<float>(in));
    st_global_v4(p + 4, pack<float>(in + 4));
  } else if (dtype == kF16) {
    st_global_v4(reinterpret_cast<__half*>(base) + i, pack<__half>(in));
  } else {
    st_global_v4(reinterpret_cast<__nv_bfloat16*>(base) + i, pack<__nv_bfloat16>(in));
  }
}
UB_DEVICE float load1(const void* base, int dtype, long long i) {
  if (dtype == kF32) return reinterpret_cast<const float*>(base)[i];
  if (dtype == kF16) return __half2float(reinterpret_cast<const __half*>(base)[i]);
  return __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(base)[i]);
}
UB_DEVICE void store1(void* base, int dtype, long long i, float v) {
  if (dtype == kF32) reinterpret_cast<float*>(base)[i] = v;
  else if (dtype == kF16) reinterpret_cast<__half*>(base)[i] = __float2half_rn(v);
  else reinterpret_cast<__nv_bfloat16*>(base)[i] = __float2bfloat16_rn(v);
}
UB_DEVICE bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// chunk index -> (tensor, first element). Linear scan: count <= 24 and uniform per CTA.
template <typename Table>
UB_DEVICE bool locate_chunk(const Table& t, long long chunk, int& tensor, long long& begin) {
  long long c = chunk;
#pragma unroll 1
  for (int i = 0; i < t.count; ++i) {
    const long long nch = (t.numel[i] + kChunk - 1) / kChunk;
    if (c < nch) {
      tensor = i;
      begin = c * kChunk;
      return true;
    }
    c -= nch;
  }
  return false;
}
template <typename Table>
static long long total_chunks(const Table& t) {
  long long n = 0;
  for (int i = 0; i < t.count; ++i) n += (t.numel[i] + kChunk - 1) / kChunk;
  return n;
}
constexpr int kCtasPerSm = 8;  // 8 CTAs of 256 threads per SM = full occupancy
static int persistent_grid(long long chunks) { return sweep_plan(chunks, 1, kCtasPerSm).grid; }

// ================================================================================================
// L2 norm
// ================================================================================================
__global__ void __launch_bounds__(kThreads) l2norm_kernel(NormTensors t, long long nchunks, float* acc,
                                                            float* partials, unsigned* counter, float* out,
                                                            int finalize) {
  __shared__ float red[32];
  __shared__ bool is_last;
  float sum = 0.f;
  for (long long c = blockIdx.x; c < nchunks; c += gridDim.x) {
    int ti;
    long long begin;
    if (!locate_chunk(t, c, ti, begin)) break;
    const long long n = t.numel[ti];
    const long long end = begin + kChunk < n ? begin + kChunk : n;
    const void* base = t.ptr[ti];
    const int dt = t.dtype[ti];
    if (aligned16(base)) {
      const long long vend = begin + ((end - begin) & ~7LL);
      for (long long i = begin + (long long)threadIdx.x * 8; i < vend; i += kThreads * 8) {
        float x[8];
        load8(base, dt, i, x);
#pragma unroll
        for (int k = 0; k < 8; ++k) sum = fmaf(x[k], x[k], sum);
      }
      for (long long i = vend + threadIdx.x; i < end; i += kThreads) {
        const float x = load1(base, dt, i);
        sum = fmaf(x, x, sum);
      }
    } else {
      for (long long i = begin + threadIdx.x; i < end; i += kThreads) {
        const float x = load1(base, dt, i);
        sum = fmaf(x, x, sum);
      }
    }
  }
  sum = block_sum(sum, red);
  if (threadIdx.x == 0) {
    partials[blockIdx.x] = sum;
    __threadfence();
    const unsigned ticket = atomicAdd(counter, 1u);
    is_last = (ticket == gridDim.x - 1);
  }
  __syncthreads();
  if (is_last) {
    // deterministic final reduction: fixed order over the per-CTA partials
    __threadfence();
    float s = 0.f;
    for (int i = threadIdx.x; i < (int)gridDim.x; i += kThreads) s += __ldcg(partials + i);
    s = block_sum(s, red);
    if (threadIdx.x == 0) {
      const float total = *acc + s;
      *acc = total;
      if (finalize) out[0] = sqrtf(total);
      *counter = 0;  // ready for the next launch
    }
  }
}

int l2norm_max_ctas() { return device_sm_count() * kCtasPerSm; }

void launch_l2norm(const NormTensors& t, float* acc, float* partials, unsigned* counter, float* out, int finalize,
                   cudaStream_t stream) {
  const long long nchunks = total_chunks(t);
  int grid = persistent_grid(nchunks);
  if (grid < 1) grid = 1;
  l2norm_kernel<<<grid, kThreads, 0, stream>>>(t, nchunks, acc, partials, counter, out, finalize);
}

// ================================================================================================
// scale
// ================================================================================================
__global__ void __launch_bounds__(kThreads) scale_kernel(ScaleTensors t, long long nchunks, float scale,
                                                           const float* scale_dev) {
  const float s = scale * (scale_dev ? __ldg(scale_dev) : 1.f);
  for (long long c = blockIdx.x; c < nchunks; c += gridDim.x) {
    int ti;
    long long begin;
    if (!locate_chunk(t, c, ti, begin)) break;
    const long long n = t.numel[ti];
    const long long end = begin + kChunk < n ? begin + kChunk : n;
    void* base = t.ptr[ti];
    const int dt = t.dtype[ti];
    long long vend = begin;
    if (aligned16(base)) {
      vend = begin + ((end - begin) & ~7LL);
      for (long long i = begin + (long long)threadIdx.x * 8; i < vend; i += kThreads * 8) {
        float x[8];
        load8(base, dt, i, x);
#pragma unroll
        for (int k = 0; k < 8; ++k) x[k] *= s;
        store8(base, dt, i, x);
      }
    }
    for (long long i = vend + threadIdx.x; i < end; i += kThreads) store1(base, dt, i, load1(base, dt, i) * s);
  }
}

void launch_scale(const ScaleTensors& t, float scale, const float* scale_dev, cudaStream_t stream) {
  const long long nchunks = total_chunks(t);
  if (nchunks == 0) return;
  scale_kernel<<<persistent_grid(nchunks), kThreads, 0, stream>>>(t, nchunks, scale, scale_dev);
}

// ================================================================================================
// Adam
// ================================================================================================
__global__ void __launch_bounds__(kThreads) adam_kernel(AdamTensors t, long long nchunks, AdamLaunch cfg) {
  // A non-finite (or zero) device divisor means "the gradients overflowed": the update skips itself -
  // parameters, moments and EMA stay untouched, only the gradient clearing happens - so the host does
  // not have to read the gradient norm before it may launch this kernel (deferred overflow check).
  const float sdev = cfg.scale_dev ? __ldg(cfg.scale_dev) : 1.f;
  const bool skip = cfg.scale_dev != nullptr && !(isfinite(sdev) && sdev != 0.f);
  if (skip && !cfg.zero_grad) return;
  const float gmul = cfg.inv_scale / sdev;
  for (long long c = blockIdx.x; c < nchunks; c += gridDim.x) {
    int ti;
    long long begin;
    if (!locate_chunk(t, c, ti, begin)) break;
    const long long n = t.numel[ti];
    const long long end = begin + kChunk < n ? begin + kChunk : n;
    void* P = t.p[ti];
    void* G = t.g[ti];
    float* M = t.m[ti];
    float* V = t.v[ti];
    void* PH = t.p_half[ti];
    float* E = t.ema[ti];
    const int pdt = t.p_dtype[ti], gdt = t.g_dtype[ti], hdt = t.half_dtype[ti];
    const AdamHyper h{t.beta1[ti], t.beta2[ti], t.eps[ti], t.step_size[ti], t.decay_mul[ti]};
    const bool sr = cfg.stochastic_rounding && PH != nullptr && hdt == kBF16;
    const bool vec_ok = aligned16(P) && aligned16(G) && aligned16(M) && aligned16(V) &&
                        (PH == nullptr || aligned16(PH)) && (E == nullptr || aligned16(E));
    long long vend = begin;
    if (vec_ok) {
      vend = begin + ((end - begin) & ~7LL);
      for (long long i = begin + (long long)threadIdx.x * 8; i < vend; i += kThreads * 8) {
        if (skip) {
          float z[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
          store8(G, gdt, i, z);
          continue;
        }
        float g[8], p[8], m[8], v[8];
        load8(G, gdt, i, g);
        load8(P, pdt, i, p);
        load8(M, kF32, i, m);
        load8(V, kF32, i, v);
#pragma unroll
        for (int k = 0; k < 8; ++k) adam_math(p[k], m[k], v[k], g[k] * gmul, h);
        store8(P, pdt, i, p);
        store8(M, kF32, i, m);
        store8(V, kF32, i, v);
        if (PH != nullptr) {
          if (sr) {
            const Philox4 r = philox4x32_10(cfg.seed, cfg.offset, (t.elem_base[ti] + (unsigned long long)i) >> 3);
            const uint32_t rw[4] = {r.x, r.y, r.z, r.w};
            Vec16 o;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const uint32_t lo = bf16_sr_bits(p[2 * k], rw[k] & 0xffffu);
              const uint32_t hi = bf16_sr_bits(p[2 * k + 1], rw[k] >> 16);
              o.w[k] = lo | (hi << 16);
            }
            st_global_v4(reinterpret_cast<__nv_bfloat16*>(PH) + i, o);
          } else {
            store8(PH, hdt, i, p);
          }
        }
        if (E != nullptr) {
          float e[8];
          load8(E, kF32, i, e);
#pragma unroll
          for (int k = 0; k < 8; ++k) e[k] = ema_step(e[k], p[k], 1.f - cfg.ema_decay);
          store8(E, kF32, i, e);
        }
        if (cfg.zero_grad) {
          float z[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
          store8(G, gdt, i, z);
        }
      }
    }
    for (long long i = vend + threadIdx.x; i < end; i += kThreads) {
      if (skip) {
        store1(G, gdt, i, 0.f);
        continue;
      }
      float p = load1(P, pdt, i), m = M[i], v = V[i];
      const float g = load1(G, gdt, i) * gmul;
      adam_math(p, m, v, g, h);
      store1(P, pdt, i, p);
      M[i] = m;
      V[i] = v;
      if (PH != nullptr) {
        if (sr) {
          const unsigned long long gi = t.elem_base[ti] + (unsigned long long)i;
          const Philox4 r = philox4x32_10(cfg.seed, cfg.offset, gi >> 3);
          const uint32_t rw[4] = {r.x, r.y, r.z, r.w};
          const uint32_t w = rw[(gi & 7) >> 1];
          const uint32_t rnd = (gi & 1) ? (w >> 16) : (w & 0xffffu);
          reinterpret_cast<uint16_t*>(PH)[i] = bf16_sr_bits(p, rnd);
        } else {
          store1(PH, hdt, i, p);
        }
      }
      if (E != nullptr) E[i] = ema_step(E[i], p, 1.f - cfg.ema_decay);
      if (cfg.zero_grad) store1(G, gdt, i, 0.f);
    }
  }
}

void launch_adam(const AdamTensors& t, const AdamLaunch& cfg, cudaStream_t stream) {
  const long long nchunks = total_chunks(t);
  if (nchunks == 0) return;
  adam_kernel<<<persistent_grid(nchunks), kThreads, 0, stream>>>(t, nchunks, cfg);
}

// ================================================================================================
// fp32 -> bf16 stochastic rounding, EMA (stand-alone)
// ================================================================================================
__global__ void __launch_bounds__(kThreads) sr_kernel(const float* in, uint16_t* out, long long n,
                                                        unsigned long long seed, unsigned long long offset) {
  const bool vec_ok = aligned16(in) && aligned16(out);
  const long long vend = vec_ok ? (n & ~7LL) : 0;
  const long long stride = (long long)gridDim.x * kThreads * 8;
  for (long long i = ((long long)blockIdx.x * kThreads + threadIdx.x) * 8; i < vend; i += stride) {
    float x[8];
    load8(in, kF32, i, x);
    const Philox4 r = philox4x32_10(seed, offset, (unsigned long long)i >> 3);
    const uint32_t rw[4] = {r.x, r.y, r.z, r.w};
    Vec16 o;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint32_t lo = bf16_sr_bits(x[2 * k], rw[k] & 0xffffu);
      const uint32_t hi = bf16_sr_bits(x[2 * k + 1], rw[k] >> 16);
      o.w[k] = lo | (hi << 16);
    }
    st_global_v4(out + i, o);
  }
  for (long long i = vend + (long long)blockIdx.x * kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads) {
    const Philox4 r = philox4x32_10(seed, offset, (unsigned long long)i >> 3);
    const uint32_t rw[4] = {r.x, r.y, r.z, r.w};
    const uint32_t w = rw[(i & 7) >> 1];
    out[i] = bf16_sr_bits(in[i], (i & 1) ? (w >> 16) : (w & 0xffffu));
  }
}

void launch_fp32_to_bf16_sr(const float* in, void* out, long long n, unsigned long long seed,
                            unsigned long long offset, cudaStream_t stream) {
  if (n <= 0) return;
  const long long chunks = (n + kChunk - 1) / kChunk;
  sr_kernel<<<persistent_grid(chunks), kThreads, 0, stream>>>(in, reinterpret_cast<uint16_t*>(out), n, seed, offset);
}

__global__ void __launch_bounds__(kThreads) ema_kernel(float* ema, const float* p, long long n, float one_minus) {
  const bool vec_ok = aligned16(ema) && aligned16(p);
  const long long vend = vec_ok ? (n & ~7LL) : 0;
  const long long stride = (long long)gridDim.x * kThreads * 8;
  for (long long i = ((long long)blockIdx.x * kThreads + threadIdx.x) * 8; i < vend; i += stride) {
    float e[8], w[8];
    load8(ema, kF32, i, e);
    load8(p, kF32, i, w);
#pragma unroll
    for (int k = 0; k < 8; ++k) e[k] = ema_step(e[k], w[k], one_minus);
    store8(ema, kF32, i, e);
  }
  for (long long i = vend + (long long)blockIdx.x * kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads)
    ema[i] = ema_step(ema[i], p[i], one_minus);
}

void launch_ema(float* ema, const float* p, long long n, float decay, cudaStream_t stream) {
  if (n <= 0) return;
  const long long chunks = (n + kChunk - 1) / kChunk;
  ema_kernel<<<persistent_grid(chunks), kThreads, 0, stream>>>(ema, p, n, 1.f - decay);
}

}  // namespace ub
