// Helpers shared by the binding translation units (bind.cpp, attn/fmha_bind.cpp, comm/comm_bind.cpp).  They include
// the PyTorch headers, so no .cu file includes this one.
#pragma once
#include <ATen/cuda/CUDAContext.h>
#include <ATen/cuda/CUDAGeneratorImpl.h>
#include <torch/extension.h>

#include <algorithm>
#include <cstdint>
#include <initializer_list>
#include <mutex>
#include <optional>
#include <string>
#include <utility>

#include "api.h"

namespace ub_bind {

using torch::Tensor;
using OptTensor = std::optional<Tensor>;
using DTypes = std::initializer_list<at::ScalarType>;

inline bool has(const OptTensor& t) { return t.has_value() && t->defined(); }
inline const void* opt_ptr(const OptTensor& t) { return has(t) ? t->data_ptr() : nullptr; }
inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
inline cudaStream_t cur_stream() { return at::cuda::getCurrentCUDAStream().stream(); }

inline int dtype_tag(at::ScalarType s) {
  switch (s) {
    case at::kFloat: return ub::kF32;
    case at::kHalf: return ub::kF16;
    case at::kBFloat16: return ub::kBF16;
    default: TORCH_CHECK(false, "unsupported dtype ", s);
  }
  return -1;
}

// Reserve `increment` Philox counters from the default CUDA generator: (seed, offset).
inline std::pair<uint64_t, uint64_t> philox_reserve(uint64_t increment) {
  auto gen = at::get_generator_or_default<at::CUDAGeneratorImpl>(std::nullopt,
                                                                 at::cuda::detail::getDefaultCUDAGenerator());
  std::lock_guard<std::mutex> lock(gen->mutex_);
  at::PhiloxCudaState st = gen->philox_cuda_state(increment);
  TORCH_CHECK(!st.captured_, "unicore_b200 kernels do not support RNG under CUDA graph capture yet");
  return {st.seed_.val, st.offset_.val};
}

inline void check_launch(const char* what) {
  cudaError_t err = cudaGetLastError();
  TORCH_CHECK(err == cudaSuccess, what, " launch failed: ", cudaGetErrorString(err));
}

// What a kernel needs of an operand besides its device, dtype and sizes.
enum Need : unsigned {
  kContig = 1,   // indexed as one dense row-major array
  kAligned = 2,  // read or written with 16-byte vectors or bulk copies from the first element on
  kVec = kContig | kAligned,
  kNumel = 4,    // `sizes` is {element count}: any shape with that many elements
};
constexpr int64_t kAnySize = -1;  // an extent of `sizes` that any size matches

// `dim` extents of any size
inline at::IntArrayRef any_shape(size_t dim) {
  static constexpr int64_t any[4] = {kAnySize, kAnySize, kAnySize, kAnySize};
  return {any, dim};
}

inline const DTypes kFloating = {at::kFloat, at::kHalf, at::kBFloat16};
inline const DTypes k16Bit = {at::kHalf, at::kBFloat16};

// "fp16 / bf16": the dtypes as the messages name them
inline std::string dtype_names(DTypes dtypes) {
  std::string s;
  for (at::ScalarType d : dtypes) {
    if (!s.empty()) s += " / ";
    switch (d) {
      case at::kFloat: s += "fp32"; break;
      case at::kHalf: s += "fp16"; break;
      case at::kBFloat16: s += "bf16"; break;
      case at::kDouble: s += "fp64"; break;
      case at::kLong: s += "int64"; break;
      case at::kInt: s += "int32"; break;
      case at::kByte: s += "uint8"; break;
      case at::kBool: s += "bool"; break;
      default: s += c10::toString(d);
    }
  }
  return s;
}

inline bool sizes_match(at::IntArrayRef got, at::IntArrayRef want) {
  if (got.size() != want.size()) return false;
  for (size_t i = 0; i < got.size(); ++i)
    if (want[i] != kAnySize && want[i] != got[i]) return false;
  return true;
}

// The per-tensor check of every binding, run before its device guard, allocations and Philox reservation: `t` is a
// CUDA tensor on `dev` (the device the call runs on), of one of `dtypes`, of shape `sizes` (empty: any shape; kAnySize
// extents match anything) and has what `need` asks for.  The messages name the operand.
inline void check_operand(const Tensor& t, const char* name, const c10::Device& dev, DTypes dtypes,
                          at::IntArrayRef sizes = {}, unsigned need = kContig) {
  TORCH_CHECK(t.is_cuda(), name, " must be a CUDA tensor");
  TORCH_CHECK(t.device() == dev, name, " must be on ", dev, ", the device of the call, not on ", t.device());
  TORCH_CHECK(std::find(dtypes.begin(), dtypes.end(), t.scalar_type()) != dtypes.end(), name, " must be ",
              dtype_names(dtypes), ", not ", dtype_names({t.scalar_type()}));
  TORCH_CHECK(!(need & kNumel) || t.numel() == sizes[0], name, " must have ", sizes[0], " elements, not ", t.numel());
  TORCH_CHECK((need & kNumel) || sizes.empty() || sizes_match(t.sizes(), sizes), name, " must have sizes ", sizes,
              " (-1: any), not ", t.sizes());
  TORCH_CHECK(!(need & kContig) || t.is_contiguous(), name, " must be contiguous");
  TORCH_CHECK(!(need & kAligned) || aligned16(t.data_ptr()), name, " must be 16-byte aligned");
}

// The same for an optional operand, when it is given.
inline void check_operand(const OptTensor& t, const char* name, const c10::Device& dev, DTypes dtypes,
                          at::IntArrayRef sizes = {}, unsigned need = kContig) {
  if (has(t)) check_operand(*t, name, dev, dtypes, sizes, need);
}

// Grouped-query attention: the `kv_heads` key / value heads of operand `name` are shared by groups of G = heads /
// kv_heads query heads, so kv_heads must divide the query head count.  Returns G.
inline int kv_group(int64_t heads, int64_t kv_heads, const char* name) {
  TORCH_CHECK(kv_heads >= 1 && heads % kv_heads == 0, name, " has ", kv_heads,
              " key / value heads, which must divide the ", heads, " query heads");
  return (int)(heads / kv_heads);
}

}  // namespace ub_bind
