// Shared device helpers for the unicore_b200 sm_90a kernels.
//   * 128-bit vector load/store wrappers and 16-bit <-> fp32 pack/unpack
//   * warp / block reductions
//   * counter-based Philox4x32-10 (no per-thread state, no curand_init)
//   * dtype tags shared with the host binding (csrc/api.h)
//   * host side: the SM count, grid-stride sweep plans, row-group geometry and dtype / VPT dispatch of the launchers
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <type_traits>

#include "api.h"

namespace ub {

#define UB_DEVICE __device__ __forceinline__
#define UB_HOST_DEVICE __host__ __device__ __forceinline__

// ------------------------------------------------------------------------------------------------
// 16-byte vector access
// ------------------------------------------------------------------------------------------------
struct alignas(16) Vec16 {
  uint32_t w[4];
};

UB_DEVICE Vec16 ld_global_v4(const void* p) {
  Vec16 v;
  asm volatile("ld.global.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.w[0]), "=r"(v.w[1]), "=r"(v.w[2]), "=r"(v.w[3])
               : "l"(p));
  return v;
}
// streaming load: read-once data, do not pollute L1
UB_DEVICE Vec16 ld_global_nc_v4(const void* p) {
  Vec16 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.w[0]), "=r"(v.w[1]), "=r"(v.w[2]), "=r"(v.w[3])
               : "l"(p));
  return v;
}
UB_DEVICE void st_global_v4(void* p, const Vec16& v) {
  asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.w[0]), "r"(v.w[1]), "r"(v.w[2]),
               "r"(v.w[3])
               : "memory");
}
UB_DEVICE void st_global_na_v4(void* p, const Vec16& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.w[0]), "r"(v.w[1]),
               "r"(v.w[2]), "r"(v.w[3])
               : "memory");
}

// ------------------------------------------------------------------------------------------------
// scalar conversions
// ------------------------------------------------------------------------------------------------
template <typename T>
UB_DEVICE float to_f32(T v);
template <>
UB_DEVICE float to_f32<float>(float v) { return v; }
template <>
UB_DEVICE float to_f32<__half>(__half v) { return __half2float(v); }
template <>
UB_DEVICE float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

template <typename T>
UB_DEVICE T from_f32(float v);
template <>
UB_DEVICE float from_f32<float>(float v) { return v; }
template <>
UB_DEVICE __half from_f32<__half>(float v) { return __float2half_rn(v); }
template <>
UB_DEVICE __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }

// elements per 16-byte vector
template <typename T>
struct VecTraits { static constexpr int kElems = 16 / sizeof(T); };

// unpack a 16-byte vector of T into fp32 lanes
template <typename T>
UB_DEVICE void unpack(const Vec16& v, float* out);
template <>
UB_DEVICE void unpack<float>(const Vec16& v, float* out) {
#pragma unroll
  for (int i = 0; i < 4; ++i) out[i] = __uint_as_float(v.w[i]);
}
template <>
UB_DEVICE void unpack<__half>(const Vec16& v, float* out) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    __half2 h = *reinterpret_cast<const __half2*>(&v.w[i]);
    float2 f = __half22float2(h);
    out[2 * i] = f.x;
    out[2 * i + 1] = f.y;
  }
}
template <>
UB_DEVICE void unpack<__nv_bfloat16>(const Vec16& v, float* out) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    // bf16 -> fp32 is a 16-bit shift
    out[2 * i] = __uint_as_float(v.w[i] << 16);
    out[2 * i + 1] = __uint_as_float(v.w[i] & 0xffff0000u);
  }
}

template <typename T>
UB_DEVICE Vec16 pack(const float* in);
template <>
UB_DEVICE Vec16 pack<float>(const float* in) {
  Vec16 v;
#pragma unroll
  for (int i = 0; i < 4; ++i) v.w[i] = __float_as_uint(in[i]);
  return v;
}
template <>
UB_DEVICE Vec16 pack<__half>(const float* in) {
  Vec16 v;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    __half2 h = __floats2half2_rn(in[2 * i], in[2 * i + 1]);
    v.w[i] = *reinterpret_cast<uint32_t*>(&h);
  }
  return v;
}
template <>
UB_DEVICE Vec16 pack<__nv_bfloat16>(const float* in) {
  Vec16 v;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    __nv_bfloat162 h = __floats2bfloat162_rn(in[2 * i], in[2 * i + 1]);
    v.w[i] = *reinterpret_cast<uint32_t*>(&h);
  }
  return v;
}

// one pair of 16-bit values <-> two fp32 (round to nearest)
template <typename T>
UB_DEVICE uint32_t pack2(float a, float b);
template <>
UB_DEVICE uint32_t pack2<__half>(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
template <>
UB_DEVICE uint32_t pack2<__nv_bfloat16>(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
template <typename T>
UB_DEVICE float2 unpack2(uint32_t w) {
  if constexpr (std::is_same<T, __half>::value) {
    return __half22float2(*reinterpret_cast<const __half2*>(&w));
  } else {
    return make_float2(__uint_as_float(w << 16), __uint_as_float(w & 0xffff0000u));
  }
}

// 14-bit dropout thresholds compared two at a time as fp16 bit patterns (HSET2): a random 16-bit
// lane masked to 14 bits is a finite non-negative half whose float order equals its integer order,
// so ONE instruction yields the 0xffff / 0x0000 select masks of a packed pair of probabilities.
// drop <=> u14 < T14; the effective rate is T14 / 16384 (|p - p_eff| < 3.1e-5) and the keep scale
// is computed from T14 so that forward and backward agree and the estimator stays unbiased.
UB_DEVICE uint32_t dropout_thresh14(float p) {
  const float t = p * 16384.f + 0.5f;
  return t <= 0.f ? 0u : (t >= 16383.f ? 16383u : (uint32_t)t);
}
UB_DEVICE float dropout_keep_scale14(uint32_t t14) { return 16384.f / (16384.f - (float)t14); }
// The same rule for the 16-bit threshold of dropout_keep8 (keep <=> u16 >= t16, P(keep) = (65536 - t16) / 65536), so
// that E[dropout(x)] = x exactly for the rate the kernels draw, not for the requested p.
UB_HOST_DEVICE float dropout_keep_scale16(uint32_t t16) { return 65536.f / (65536.f - (float)t16); }
UB_DEVICE uint32_t keep_mask2(uint32_t rnd, uint32_t t14x2) {
  const uint32_t u = rnd & 0x3fff3fffu;
  return __hge2_mask(*reinterpret_cast<const __half2*>(&u), *reinterpret_cast<const __half2*>(&t14x2));
}

// ------------------------------------------------------------------------------------------------
// fp32 pairs: the kernels keep their math on element pairs (two adjacent columns); sm_90 has no packed fp32x2
// instructions, so every operation is two scalar FFMA / FMUL / FADD.
// ------------------------------------------------------------------------------------------------
struct alignas(8) F2 {
  float x, y;
};
UB_DEVICE unsigned long long f2_bits(F2 a) { return *reinterpret_cast<unsigned long long*>(&a); }
UB_DEVICE F2 f2_from_bits(unsigned long long b) { return *reinterpret_cast<F2*>(&b); }
UB_DEVICE F2 f2(float a) { return F2{a, a}; }
UB_DEVICE F2 fma2(F2 a, F2 b, F2 c) { return F2{fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)}; }
UB_DEVICE F2 mul2(F2 a, F2 b) { return F2{a.x * b.x, a.y * b.y}; }
UB_DEVICE F2 add2(F2 a, F2 b) { return F2{a.x + b.x, a.y + b.y}; }
UB_DEVICE float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
UB_DEVICE float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// ------------------------------------------------------------------------------------------------
// 1-D bulk asynchronous copies (cp.async.bulk, the non-tensor form of TMA) + mbarrier completion:
// ONE instruction by ONE thread moves a contiguous block of up to tens of KB from global to shared
// memory with no register or LSU-issue cost; the bytes are counted on an mbarrier the consumers
// wait on.  Addresses and sizes must be multiples of 16 bytes.
// ------------------------------------------------------------------------------------------------
UB_DEVICE uint32_t smem_addr_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
UB_DEVICE void bulk_bar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
UB_DEVICE void bulk_bar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
UB_DEVICE void bulk_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
UB_DEVICE void bulk_g2s(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
UB_DEVICE void bulk_wait(uint32_t bar, uint32_t parity) {
  const long long t0 = clock64();
  uint32_t done = 0;
  while (!done) {
    asm volatile(
        "{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    if (!done && clock64() - t0 > 4000000000LL) __trap();  // ~2 s: never hang the GPU on a lost copy
  }
}

// ------------------------------------------------------------------------------------------------
// reductions
// ------------------------------------------------------------------------------------------------
UB_DEVICE float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
UB_DEVICE float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Sum across the whole CTA (blockDim.x multiple of 32, <= 1024). Result valid in ALL threads.
// `smem` must hold 32 floats.
UB_DEVICE float block_sum(float v, float* smem) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();  // protect smem reuse between consecutive calls
  if (lane == 0) smem[wid] = v;
  __syncthreads();
  float r = (lane < nw) ? smem[lane] : 0.f;
  return warp_sum(r);
}

// ------------------------------------------------------------------------------------------------
// Philox4x32-10, counter based.  philox(seed, offset, ctr) is a pure function: the same
// (seed, offset, element index) yields the same random bits in forward and backward kernels and on
// every data-parallel rank.
// ------------------------------------------------------------------------------------------------
struct Philox4 {
  uint32_t x, y, z, w;
};

template <int kRounds>
UB_DEVICE Philox4 philox4x32(uint64_t seed, uint64_t offset, uint64_t ctr) {
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
  uint32_t c0 = (uint32_t)ctr, c1 = (uint32_t)(ctr >> 32), c2 = (uint32_t)offset, c3 = (uint32_t)(offset >> 32);
#pragma unroll
  for (int r = 0; r < kRounds; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return Philox4{c0, c1, c2, c3};
}
// full-strength variant (stochastic rounding of the weights)
UB_DEVICE Philox4 philox4x32_10(uint64_t seed, uint64_t offset, uint64_t ctr) {
  return philox4x32<10>(seed, offset, ctr);
}

// Dropout decisions for 8 consecutive elements whose first linear index is `idx8*8`:
// one Philox call gives 8 x 16-bit uniforms; keep iff u16 >= thresh16 (thresh16 = round(p*65536)).
// Returns an 8-bit keep mask (bit i = element i kept).
UB_DEVICE uint32_t dropout_keep8(uint64_t seed, uint64_t offset, uint64_t idx8, uint32_t thresh16) {
  // 7 rounds: Philox4x32-7 already passes BigCrush and dropout only needs decorrelated bits
  const Philox4 r = philox4x32<7>(seed, offset, idx8);
  uint32_t m = 0;
  const uint32_t ws[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    m |= ((ws[i] & 0xffffu) >= thresh16 ? 1u : 0u) << (2 * i);
    m |= ((ws[i] >> 16) >= thresh16 ? 1u : 0u) << (2 * i + 1);
  }
  return m;
}

// 14-bit variant of dropout_keep8 (keep iff (u16 & 0x3fff) >= thresh14), in two forms that agree bit for bit:
// an 8-bit keep mask for scalar code, and four AND-masks (0xffff per kept 16-bit lane, one word per element
// pair - one HSET2 each) that are applied straight to packed fp16 / bf16 data.
UB_DEVICE uint32_t dropout_keep8_14(uint64_t seed, uint64_t offset, uint64_t idx8, uint32_t thresh14) {
  const Philox4 r = philox4x32<7>(seed, offset, idx8);
  uint32_t m = 0;
  const uint32_t ws[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    m |= ((ws[i] & 0x3fffu) >= thresh14 ? 1u : 0u) << (2 * i);
    m |= (((ws[i] >> 16) & 0x3fffu) >= thresh14 ? 1u : 0u) << (2 * i + 1);
  }
  return m;
}
UB_DEVICE void dropout_lane_masks8(uint64_t seed, uint64_t offset, uint64_t idx8, uint32_t thresh14, uint32_t (&m)[4]) {
  const Philox4 r = philox4x32<7>(seed, offset, idx8);
  const uint32_t t14x2 = thresh14 | (thresh14 << 16);
  m[0] = keep_mask2(r.x, t14x2);
  m[1] = keep_mask2(r.y, t14x2);
  m[2] = keep_mask2(r.z, t14x2);
  m[3] = keep_mask2(r.w, t14x2);
}

UB_HOST_DEVICE uint32_t dropout_thresh16(float p) {
  float t = p * 65536.f + 0.5f;
  return t >= 65535.f ? 65535u : (uint32_t)t;
}

// ------------------------------------------------------------------------------------------------
// host: launch geometry and dispatch
// ------------------------------------------------------------------------------------------------
// Streaming multiprocessors of the current device, queried once per device ordinal (132, an H100 SXM, when the query
// fails).
inline int device_sm_count() {
  constexpr int kMaxDevices = 64;
  static std::atomic<int> cache[kMaxDevices];  // 0: not queried yet
  int dev = 0;
  cudaGetDevice(&dev);
  std::atomic<int>* slot = dev >= 0 && dev < kMaxDevices ? &cache[dev] : nullptr;
  int sms = slot != nullptr ? slot->load(std::memory_order_relaxed) : 0;
  if (sms == 0) {
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
    if (slot != nullptr) slot->store(sms, std::memory_order_relaxed);
  }
  return sms;
}

// Plan of a grid-stride kernel over `items` work items, `per_cta` of them per CTA and pass: as many CTAs as the items
// need, at most `ctas_per_sm` per SM.  The grid is 0 exactly when there are no items.
inline SweepPlan sweep_plan(long long items, long long per_cta, int ctas_per_sm) {
  const long long need = (items + per_cta - 1) / per_cta, cap = (long long)device_sm_count() * ctas_per_sm;
  SweepPlan p;
  p.grid = (int)(need < cap ? need : cap);
  p.items = items;
  p.items_per_sweep = (long long)p.grid * per_cta;
  p.sweeps = p.grid > 0 ? (items + p.items_per_sweep - 1) / p.items_per_sweep : 0;
  return p;
}

// A row of `nvec` 16-byte vectors held in registers by a group of `tpr` threads (a power of two), `vpt` vectors each:
// rows up to 128 vectors take a vector per thread on at most 32 threads, longer rows about four per thread on at most
// 256.  False when that leaves more than 4 vectors per thread.
inline bool row_group_geom(int nvec, int& tpr, int& vpt) {
  const int want = nvec <= 128 ? nvec : (nvec + 3) / 4, max_tpr = nvec <= 128 ? 32 : 256;
  tpr = 1;
  while (tpr < want && tpr < max_tpr) tpr <<= 1;
  vpt = (nvec + tpr - 1) / tpr;
  return vpt <= 4;
}

// Host dispatch of a launcher body on a run-time value: the body is compiled once per case, with `T` the element type
// of a dtype tag or `VPT` the vectors per thread of row_group_geom.  Other values run nothing.
#define UB_DISPATCH_FLOAT(DTYPE_VALUE, ...)                               \
  switch (DTYPE_VALUE) {                                                  \
    case kF32: { using T = float; __VA_ARGS__; break; }                   \
    case kF16: { using T = __half; __VA_ARGS__; break; }                  \
    case kBF16: { using T = __nv_bfloat16; __VA_ARGS__; break; }          \
    default: break;                                                       \
  }
#define UB_DISPATCH_16BIT(DTYPE_VALUE, ...)                               \
  switch (DTYPE_VALUE) {                                                  \
    case kF16: { using T = __half; __VA_ARGS__; break; }                  \
    case kBF16: { using T = __nv_bfloat16; __VA_ARGS__; break; }          \
    default: break;                                                       \
  }
#define UB_DISPATCH_VPT(VPT_VALUE, ...)                                   \
  switch (VPT_VALUE) {                                                    \
    case 1: { constexpr int VPT = 1; __VA_ARGS__; break; }                \
    case 2: { constexpr int VPT = 2; __VA_ARGS__; break; }                \
    case 3: { constexpr int VPT = 3; __VA_ARGS__; break; }                \
    case 4: { constexpr int VPT = 4; __VA_ARGS__; break; }                \
    default: break;                                                       \
  }

}  // namespace ub
