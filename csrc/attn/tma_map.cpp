#include "tma_map.h"

#include <cstdio>
#include <mutex>

namespace ub {
namespace {

using EncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                              const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                              CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeFn encode_fn() {
  static EncodeFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeFn>(p);
  });
  return fn;
}

bool encode_sw128(CUtensorMap* map, const void* base, bool bf16, int rank, const cuuint64_t* dims, const cuuint64_t* strides,
                  const cuuint32_t* box) {
  EncodeFn fn = encode_fn();
  if (fn == nullptr) return false;
  const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  const CUresult r = fn(map, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank,
                        const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) fprintf(stderr, "cuTensorMapEncodeTiled (128B swizzle, rank %d) -> %d  base=%p\n", rank, (int)r, base);
  return r == CUDA_SUCCESS;
}

}  // namespace

bool make_head_tile_map_sw128(CUtensorMap* map, const void* base, bool bf16, int B, int L, int H, int D, long long sb,
                              long long sl, long long sh, int box_rows) {
  // columns D..127 of a box lie outside the tensor: the TMA unit fills them with zeros
  const cuuint64_t dims[4] = {(cuuint64_t)D, (cuuint64_t)H, (cuuint64_t)L, (cuuint64_t)B};
  const cuuint64_t strides[3] = {(cuuint64_t)sh * 2, (cuuint64_t)sl * 2, (cuuint64_t)sb * 2};
  const cuuint32_t box[4] = {64, 1, (cuuint32_t)box_rows, 1};
  return encode_sw128(map, base, bf16, 4, dims, strides, box);
}

bool make_bias_tile_map_sw128(CUtensorMap* map, const void* base, bool bf16, int NB, int Lq, int Lk) {
  const cuuint64_t dims[3] = {(cuuint64_t)Lk, (cuuint64_t)Lq, (cuuint64_t)NB};
  const cuuint64_t strides[2] = {(cuuint64_t)Lk * 2, (cuuint64_t)Lq * Lk * 2};
  const cuuint32_t box[3] = {64, 64, 1};
  return encode_sw128(map, base, bf16, 3, dims, strides, box);
}

}  // namespace ub
