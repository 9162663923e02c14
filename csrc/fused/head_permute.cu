// Token-major <-> head-major relayout of packed projections, for sm_90a.
//
//   token-major  [B, L, T, H, D]   what `in_proj` writes (T = 3: q | k | v) and what `out_proj` reads (T = 1)
//   head-major   T x [B, H, L, D]  what the batched attention GEMMs need (one matrix per (b, h))
//
// The reference reaches head-major through `.view().transpose().contiguous()` chains (unicore/modules/
// multihead_attention.py:62-76, 105-110): four strided ATen copies and a multiply per layer in forward, and
// in backward three zero-fills + three slice copies + two adds to rebuild the packed gradient.  Here each
// direction is ONE kernel moving 16-byte vectors: head-major tensors are addressed through up to four base
// pointers, so the three gradients that autograd hands back separately are gathered straight into the packed
// [B, L, 3, H, D] gradient (absent ones read as zero), and the query scale rides along on slice 0.
//
// Access pattern: a thread moves one 16-byte vector; consecutive lanes cover (d-vector, 2 neighbouring
// tokens, head) in that order, so for head_dim 8 (one vector per head, Uni-Mol) every warp still reads two
// 256-byte runs on the token-major side and writes full 32-byte sectors on the head-major side.
#include "../api.h"
#include "../common.cuh"

namespace ub {

struct HeadPtrs {
  void* p[4];
};

template <typename T, bool kToHeads>
__global__ void __launch_bounds__(256) head_permute_kernel(void* token_major, HeadPtrs heads, int B, int L, int NT, int H,
                                                           int DV, float scale0) {
  const long long lp_count = (L + 1) >> 1;
  const long long total = (long long)B * NT * lp_count * H * 2 * DV;
  for (long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x; w < total; w += (long long)gridDim.x * blockDim.x) {
    long long r = w;
    const int dv = (int)(r % DV);
    r /= DV;
    const int l_sub = (int)(r & 1);
    r >>= 1;
    const int h = (int)(r % H);
    r /= H;
    const int l = (int)(r % lp_count) * 2 + l_sub;
    r /= lp_count;
    const int t = (int)(r % NT);
    const int b = (int)(r / NT);
    if (l >= L) continue;
    Vec16* tok = reinterpret_cast<Vec16*>(token_major) + ((((long long)b * L + l) * NT + t) * H + h) * DV + dv;
    Vec16* head = reinterpret_cast<Vec16*>(heads.p[t]);
    if (head != nullptr) head += (((long long)b * H + h) * L + l) * DV + dv;
    Vec16 v;
    if (kToHeads) {
      v = ld_global_nc_v4(reinterpret_cast<const T*>(tok));
    } else if (head != nullptr) {
      v = ld_global_nc_v4(reinterpret_cast<const T*>(head));
    } else {
      v.w[0] = v.w[1] = v.w[2] = v.w[3] = 0u;  // no gradient arrived for this slice
    }
    if (t == 0 && scale0 != 1.f) {
      float f[VecTraits<T>::kElems];
      unpack<T>(v, f);
#pragma unroll
      for (int e = 0; e < VecTraits<T>::kElems; ++e) f[e] *= scale0;
      v = pack<T>(f);
    }
    if (kToHeads) st_global_v4(reinterpret_cast<T*>(head), v);
    else st_global_v4(reinterpret_cast<T*>(tok), v);
  }
}

SweepPlan head_permute_plan(int B, int L, int T, int H, int D, int dtype) {
  const int dv = D / (dtype == kF32 ? 4 : 8);
  return sweep_plan((long long)B * T * ((L + 1) / 2) * H * 2 * dv, 256, 16);
}

void launch_head_permute(void* token_major, void* const* head_major, int B, int L, int NT, int H, int D, float scale0,
                         bool to_heads, int dtype, cudaStream_t stream) {
  if (B <= 0 || L <= 0 || NT <= 0 || H <= 0 || D <= 0) return;
  HeadPtrs heads;
  for (int t = 0; t < 4; ++t) heads.p[t] = t < NT ? head_major[t] : nullptr;
  const int grid = head_permute_plan(B, L, NT, H, D, dtype).grid;
  UB_DISPATCH_FLOAT(dtype, {
    auto kern = to_heads ? head_permute_kernel<T, true> : head_permute_kernel<T, false>;
    kern<<<grid, 256, 0, stream>>>(token_major, heads, B, L, NT, H, D / VecTraits<T>::kElems, scale0);
  });
}

}  // namespace ub
