// Rotary position embeddings (GPT-NeoX / LLaMA "rotate-half" form) over a packed projection, for sm_90a.
//
//   x    [B, L, N, D]  16-bit, last dim contiguous, head stride D, any token / batch stride (a strided q slice, or the
//                      whole packed [B, L, 3, H, D] / [B, L, H + 2 H_kv, D] projection viewed as N heads)
//   out  [B, L, N, D]  contiguous: heads 0 .. R-1 (q and k, the leading heads of both packed layouts) rotated on their
//                      first rd columns, every other element copied bitwise
//
// Pair i < rd/2 of a rotated head is (x[i], x[i + rd/2]); at position pos = l + offset[b] and angle
// theta = fl32(float(pos) * inv_freq[i]):  y1 = x1 cos - x2 sin,  y2 = x2 cos + x1 sin  (kInverse: sin -> -sin, the
// transpose, which is the backward).  The rotation runs in fp32 and rounds once to the storage type.
//
// Trig: the build uses --use_fast_math, under which sincosf becomes MUFU.SIN / MUFU.COS, whose absolute error grows
// with the argument (angles reach thousands of radians at long positions).  cos / sin are therefore the fp64 sincos
// of the fp32 angle, rounded to fp32; fast math leaves fp64 alone.  That costs tens of fp64 instructions, so it is done
// once per (token, frequency) and shared through shared memory by all N heads of the token.
//
// Structure: a CTA takes tiles of kTileTokens consecutive tokens in a grid-stride sweep (rotary_plan).  Phase 1 writes
// the tile's [tokens, rd/2] cos / sin to shared memory; phase 2 streams the (token, head, chunk) items.  Vector path:
// a rotated chunk is 8 pairs (two 16-byte loads at i and i + rd/2, two stores), a copied chunk one 16-byte vector.
// Narrow path (rd/2 % 8 != 0, or an operand off 16 bytes): a rotated item is one pair, a copied item one element.
// No atomics, allocation or host synchronisation: the result is bitwise reproducible and the launch is graph-safe.
#include "../api.h"
#include "../common.cuh"

namespace ub {

namespace {

constexpr int kRotaryThreads = 256;
constexpr int kTileTokens = 8;

struct RotaryArgs {
  const void* x;
  void* out;
  const float* inv_freq;
  const int* offsets;        // nullable: positions are l
  long long sb, sl;          // x strides of batch and token, elements
  int B, L, N, D, R, half;   // half = rd / 2
};

template <typename T, bool kVec, bool kInverse>
__global__ void __launch_bounds__(kRotaryThreads) rotary_kernel(RotaryArgs a) {
  extern __shared__ float4 rotary_smem[];
  float* cs = reinterpret_cast<float*>(rotary_smem);  // [kTileTokens][half] cos
  float* sn = cs + kTileTokens * a.half;               // [kTileTokens][half] sin
  const long long tokens = (long long)a.B * a.L;
  const long long tiles = (tokens + kTileTokens - 1) / kTileTokens;
  constexpr int E = kVec ? 8 : 1;   // elements per item: pairs of a rotated chunk, or elements of a copied one
  const int rot_items = a.half / E + (a.D - 2 * a.half) / E;   // per rotated head: pair chunks, then the copied tail
  const int copy_items = a.D / E;                               // per copied head
  const int per_token = a.R * rot_items + (a.N - a.R) * copy_items;
  const T* x = static_cast<const T*>(a.x);
  T* out = static_cast<T*>(a.out);
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const long long t0 = tile * kTileTokens;
    const int nt = (int)(tokens - t0 < kTileTokens ? tokens - t0 : kTileTokens);
    __syncthreads();   // the previous tile's phase 2 is done with cs / sn
    for (int i = threadIdx.x; i < nt * a.half; i += blockDim.x) {
      const int tok = i / a.half, f = i - tok * a.half;
      const long long t = t0 + tok;
      const int b = (int)(t / a.L), l = (int)(t - (long long)b * a.L);
      const int pos = l + (a.offsets != nullptr ? a.offsets[b] : 0);
      const float theta = __fmul_rn((float)pos, a.inv_freq[f]);
      double s, c;
      sincos((double)theta, &s, &c);
      cs[i] = (float)c;
      sn[i] = kInverse ? -(float)s : (float)s;
    }
    __syncthreads();
    for (int k = threadIdx.x; k < nt * per_token; k += blockDim.x) {
      const int tok = k / per_token;
      int r = k - tok * per_token;
      const long long t = t0 + tok;
      const long long b = t / a.L, l = t - b * a.L;
      int head, col;          // col: first element of the item
      bool rotate;
      if (r < a.R * rot_items) {
        head = r / rot_items;
        const int j = r - head * rot_items;
        rotate = j < a.half / E;
        col = rotate ? j * E : 2 * a.half + (j - a.half / E) * E;
      } else {
        r -= a.R * rot_items;
        head = a.R + r / copy_items;
        col = (r - (head - a.R) * copy_items) * E;
        rotate = false;
      }
      const T* src = x + b * a.sb + l * a.sl + (long long)head * a.D;
      T* dst = out + (t * a.N + head) * a.D;
      const float* c = cs + tok * a.half + col;
      const float* s = sn + tok * a.half + col;
      if constexpr (kVec) {
        if (!rotate) {
          st_global_v4(dst + col, ld_global_nc_v4(src + col));
          continue;
        }
        float x1[8], x2[8], cf[8], sf[8];
        unpack<T>(ld_global_nc_v4(src + col), x1);
        unpack<T>(ld_global_nc_v4(src + col + a.half), x2);
        *reinterpret_cast<float4*>(cf) = *reinterpret_cast<const float4*>(c);
        *reinterpret_cast<float4*>(cf + 4) = *reinterpret_cast<const float4*>(c + 4);
        *reinterpret_cast<float4*>(sf) = *reinterpret_cast<const float4*>(s);
        *reinterpret_cast<float4*>(sf + 4) = *reinterpret_cast<const float4*>(s + 4);
        float y1[8], y2[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          y1[e] = x1[e] * cf[e] - x2[e] * sf[e];
          y2[e] = x2[e] * cf[e] + x1[e] * sf[e];
        }
        st_global_v4(dst + col, pack<T>(y1));
        st_global_v4(dst + col + a.half, pack<T>(y2));
      } else {
        if (!rotate) {
          // raw 16-bit copy: NaN payloads and signalling NaNs pass unchanged
          reinterpret_cast<unsigned short*>(dst)[col] = reinterpret_cast<const unsigned short*>(src)[col];
          continue;
        }
        const float x1 = to_f32<T>(src[col]), x2 = to_f32<T>(src[col + a.half]);
        dst[col] = from_f32<T>(x1 * c[0] - x2 * s[0]);
        dst[col + a.half] = from_f32<T>(x2 * c[0] + x1 * s[0]);
      }
    }
  }
}

}  // namespace

RotaryPlan rotary_plan(int B, int L, int N, int D, int rd, int dtype, bool aligned) {
  RotaryPlan p;
  p.vec = aligned && (rd / 2) % 8 == 0 && D % 8 == 0;
  p.tile_tokens = kTileTokens;
  p.smem = 2 * kTileTokens * (rd / 2) * (int)sizeof(float);
  p.sweep = sweep_plan(((long long)B * L + kTileTokens - 1) / kTileTokens, 1, 8);
  return p;
}

void launch_rotary(const void* x, void* out, const float* inv_freq, const int* offsets, long long sb, long long sl,
                   int B, int L, int N, int D, int rd, int rotated_heads, bool aligned, bool inverse, int dtype,
                   cudaStream_t stream) {
  if (B <= 0 || L <= 0 || N <= 0 || D <= 0) return;
  const RotaryPlan p = rotary_plan(B, L, N, D, rd, dtype, aligned);
  RotaryArgs a{x, out, inv_freq, offsets, sb, sl, B, L, N, D, rotated_heads, rd / 2};
  UB_DISPATCH_16BIT(dtype, {
    auto kern = p.vec ? (inverse ? rotary_kernel<T, true, true> : rotary_kernel<T, true, false>)
                      : (inverse ? rotary_kernel<T, false, true> : rotary_kernel<T, false, false>);
    kern<<<p.sweep.grid, kRotaryThreads, p.smem, stream>>>(a);
  });
}

}  // namespace ub
