// Pair-representation relayout for sm_90a:  head-major [B, H, M] <-> pair-major [B, M, H]  (M = Lq * Lk).
//
// Pair-bias models (Uni-Mol; reference usage in SURVEY App. E) keep the pair representation head-major while
// it is the attention bias ([B*H, L, L]) and pair-major ([B, L, L, H]) for the heads that consume it.  In
// PyTorch each crossing is a strided `permute().contiguous()` over B*H*L*L elements, and the encoder tail adds
// a subtraction, two masked_fill passes and an equality pass on top (and all of them again in backward).
//
// Here a thread owns an 8 x 8 tile of 16-bit elements: eight 16-byte loads along one layout, an in-register
// transpose (32 PRMT), eight 16-byte stores along the other.  Lanes are ordered (head-vector, then m) so both
// sides touch whole 32-byte sectors; no shared memory, no bank conflicts.  Two kernels build on the tile:
//   * pair_transpose:  plain relayout, either direction (each is the other's backward);
//   * pair_tail fwd:   pair  = transpose(z) with -inf -> 0
//                      delta = transpose(z - z0) with padded key columns -> 0        (one pass instead of six)
//     pair_tail bwd:   dz = [z != -inf] * T(d_pair) + T(d_delta * !pad),  dz0 = -T(d_delta * !pad).
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "../api.h"
#include "../common.cuh"

namespace ub {

namespace {

struct Tile {
  uint32_t w[8][4];  // 8 rows of 8 16-bit elements
};

UB_DEVICE void tile_load(Tile& t, const Vec16* base, long long row_stride_vec) {
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    const Vec16 v = ld_global_nc_v4(base + r * row_stride_vec);
#pragma unroll
    for (int j = 0; j < 4; ++j) t.w[r][j] = v.w[j];
  }
}

UB_DEVICE void tile_store(const Tile& t, Vec16* base, long long row_stride_vec) {
#pragma unroll
  for (int r = 0; r < 8; ++r) {
    Vec16 v;
#pragma unroll
    for (int j = 0; j < 4; ++j) v.w[j] = t.w[r][j];
    st_global_v4(base + r * row_stride_vec, v);
  }
}

UB_DEVICE void tile_zero(Tile& t) {
#pragma unroll
  for (int r = 0; r < 8; ++r)
#pragma unroll
    for (int j = 0; j < 4; ++j) t.w[r][j] = 0u;
}

// out[c][r] = in[r][c] for 16-bit elements: pair rows (2i, 2i+1), split every word into its low / high halves
UB_DEVICE void tile_transpose(const Tile& in, Tile& out) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      out.w[2 * j][i] = __byte_perm(in.w[2 * i][j], in.w[2 * i + 1][j], 0x5410);
      out.w[2 * j + 1][i] = __byte_perm(in.w[2 * i][j], in.w[2 * i + 1][j], 0x7632);
    }
  }
}

template <typename T2>
UB_DEVICE T2 as_pair(uint32_t w) {
  return *reinterpret_cast<T2*>(&w);
}
template <typename T2>
UB_DEVICE uint32_t as_word(T2 v) {
  return *reinterpret_cast<uint32_t*>(&v);
}

// the packed pair type of a 16-bit element type
template <typename T>
using Pair2 = std::conditional_t<std::is_same<T, __half>::value, __half2, __nv_bfloat162>;

template <typename T2>
struct NegInf;
template <>
struct NegInf<__half2> { static constexpr uint32_t kBits = 0xFC00FC00u; };
template <>
struct NegInf<__nv_bfloat162> { static constexpr uint32_t kBits = 0xFF80FF80u; };

// 0xFFFF in every 16-bit lane of `w` that holds -inf
template <typename T2>
UB_DEVICE uint32_t neg_inf_lanes(uint32_t w) {
  return __heq2_mask(as_pair<T2>(w), as_pair<T2>(NegInf<T2>::kBits));
}

struct PairGeom {
  int B, H, HV, L;       // HV = H / 8
  long long M, MV;       // M = Lq * Lk, MV = M / 8
};

// work item -> (b, hv, mq); lanes run over hv first so a warp covers whole pair-major rows
UB_DEVICE bool pair_item(const PairGeom& g, long long w, int& b, int& hv, long long& mq) {
  const long long total = (long long)g.B * g.HV * g.MV;
  if (w >= total) return false;
  hv = (int)(w % g.HV);
  w /= g.HV;
  mq = w % g.MV;
  b = (int)(w / g.MV);
  return true;
}

UB_DEVICE const Vec16* head_ptr(const void* base, const PairGeom& g, int b, int hv, long long mq) {
  return reinterpret_cast<const Vec16*>(base) + ((long long)b * g.H + hv * 8) * g.MV + mq;  // row stride: MV
}
UB_DEVICE const Vec16* pair_ptr(const void* base, const PairGeom& g, int b, int hv, long long mq) {
  return reinterpret_cast<const Vec16*>(base) + ((long long)b * g.M + mq * 8) * g.HV + hv;  // row stride: HV
}

// 8 key-padding flags of the pair rows m0 .. m0+7 (key index = m % L; L % 8 == 0 keeps them in one row of the mask)
UB_DEVICE unsigned long long pad_flags(const unsigned char* key_pad, const PairGeom& g, int b, long long mq) {
  if (key_pad == nullptr) return 0ull;
  const int k0 = (int)((mq * 8) % g.L);
  return *reinterpret_cast<const unsigned long long*>(key_pad + (long long)b * g.L + k0);
}

}  // namespace

template <bool kToPair>
__global__ void __launch_bounds__(256) pair_transpose_kernel(const void* in, void* out, PairGeom g) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x;; w += stride) {
    int b, hv;
    long long mq;
    if (!pair_item(g, w, b, hv, mq)) break;
    Tile a, t;
    if (kToPair) {
      tile_load(a, head_ptr(in, g, b, hv, mq), g.MV);
      tile_transpose(a, t);
      tile_store(t, const_cast<Vec16*>(pair_ptr(out, g, b, hv, mq)), g.HV);
    } else {
      tile_load(a, pair_ptr(in, g, b, hv, mq), g.HV);
      tile_transpose(a, t);
      tile_store(t, const_cast<Vec16*>(head_ptr(out, g, b, hv, mq)), g.MV);
    }
  }
}

template <typename T2>
__global__ void __launch_bounds__(256) pair_tail_fwd_kernel(const void* z, const void* z0, const unsigned char* key_pad,
                                                            void* pair, void* delta, PairGeom g) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x;; w += stride) {
    int b, hv;
    long long mq;
    if (!pair_item(g, w, b, hv, mq)) break;
    Tile a, a0, t;
    tile_load(a, head_ptr(z, g, b, hv, mq), g.MV);
    tile_load(a0, head_ptr(z0, g, b, hv, mq), g.MV);
#pragma unroll
    for (int r = 0; r < 8; ++r) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t zw = a.w[r][j];
        a0.w[r][j] = as_word<T2>(__hsub2(as_pair<T2>(zw), as_pair<T2>(a0.w[r][j])));  // delta (one rounding, as z - z0)
        a.w[r][j] = zw & ~neg_inf_lanes<T2>(zw);                                      // pair: -inf -> 0
      }
    }
    tile_transpose(a, t);
    tile_store(t, const_cast<Vec16*>(pair_ptr(pair, g, b, hv, mq)), g.HV);
    tile_transpose(a0, t);
    const unsigned long long pads = pad_flags(key_pad, g, b, mq);
#pragma unroll
    for (int r = 0; r < 8; ++r) {
      if ((pads >> (8 * r)) & 0xffull) {
#pragma unroll
        for (int j = 0; j < 4; ++j) t.w[r][j] = 0u;  // padded key column: no delta (also clears -inf - finite)
      }
    }
    tile_store(t, const_cast<Vec16*>(pair_ptr(delta, g, b, hv, mq)), g.HV);
  }
}

template <typename T2>
__global__ void __launch_bounds__(256) pair_tail_bwd_kernel(const void* d_pair, const void* d_delta, const void* z,
                                                            const unsigned char* key_pad, void* dz, void* dz0, PairGeom g) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x;; w += stride) {
    int b, hv;
    long long mq;
    if (!pair_item(g, w, b, hv, mq)) break;
    Tile gp, gd, t, zt;
    if (d_delta != nullptr) {
      tile_load(t, pair_ptr(d_delta, g, b, hv, mq), g.HV);
      const unsigned long long pads = pad_flags(key_pad, g, b, mq);
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        if ((pads >> (8 * r)) & 0xffull) {
#pragma unroll
          for (int j = 0; j < 4; ++j) t.w[r][j] = 0u;
        }
      }
      tile_transpose(t, gd);
    } else {
      tile_zero(gd);
    }
    if (d_pair != nullptr) {
      tile_load(t, pair_ptr(d_pair, g, b, hv, mq), g.HV);
      tile_transpose(t, gp);
    } else {
      tile_zero(gp);
    }
    tile_load(zt, head_ptr(z, g, b, hv, mq), g.MV);
#pragma unroll
    for (int r = 0; r < 8; ++r) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t live = gp.w[r][j] & ~neg_inf_lanes<T2>(zt.w[r][j]);
        gp.w[r][j] = as_word<T2>(__hadd2(as_pair<T2>(live), as_pair<T2>(gd.w[r][j])));
        gd.w[r][j] ^= 0x80008000u;  // dz0 = -d_delta
      }
    }
    tile_store(gp, const_cast<Vec16*>(head_ptr(dz, g, b, hv, mq)), g.MV);
    tile_store(gd, const_cast<Vec16*>(head_ptr(dz0, g, b, hv, mq)), g.MV);
  }
}

static PairGeom make_pair_geom(int B, int H, int L, long long M) {
  PairGeom g;
  g.B = B;
  g.H = H;
  g.HV = H / 8;
  g.L = L;
  g.M = M;
  g.MV = M / 8;
  return g;
}

SweepPlan pair_plan(int B, int H, long long M) { return sweep_plan((long long)B * (H / 8) * (M / 8), 256, 8); }

static int pair_grid(const PairGeom& g) { return pair_plan(g.B, g.H, g.M).grid; }

void launch_pair_transpose(const void* in, void* out, int B, int H, long long M, bool to_pair, cudaStream_t stream) {
  if (B <= 0 || H <= 0 || M <= 0) return;
  const PairGeom g = make_pair_geom(B, H, 8, M);
  if (to_pair) pair_transpose_kernel<true><<<pair_grid(g), 256, 0, stream>>>(in, out, g);
  else pair_transpose_kernel<false><<<pair_grid(g), 256, 0, stream>>>(in, out, g);
}

void launch_pair_tail_fwd(const void* z, const void* z0, const unsigned char* key_pad, void* pair, void* delta, int B,
                          int H, int Lq, int Lk, int dtype, cudaStream_t stream) {
  if (B <= 0 || H <= 0 || Lq <= 0 || Lk <= 0) return;
  const PairGeom g = make_pair_geom(B, H, Lk, (long long)Lq * Lk);
  UB_DISPATCH_16BIT(dtype,
                    (pair_tail_fwd_kernel<Pair2<T>><<<pair_grid(g), 256, 0, stream>>>(z, z0, key_pad, pair, delta, g)));
}

void launch_pair_tail_bwd(const void* d_pair, const void* d_delta, const void* z, const unsigned char* key_pad, void* dz,
                          void* dz0, int B, int H, int Lq, int Lk, int dtype, cudaStream_t stream) {
  if (B <= 0 || H <= 0 || Lq <= 0 || Lk <= 0) return;
  const PairGeom g = make_pair_geom(B, H, Lk, (long long)Lq * Lk);
  UB_DISPATCH_16BIT(dtype, (pair_tail_bwd_kernel<Pair2<T>><<<pair_grid(g), 256, 0, stream>>>(d_pair, d_delta, z,
                                                                                            key_pad, dz, dz0, g)));
}

}  // namespace ub
