// Block allocator of paged key / value caches (contract in fmha_api.h): reserve hands blocks off a free stack to the
// table entries that need one, release pushes the blocks past each sequence's length back.  Each is one CTA that walks
// the B x M table entries in order, kThreads at a time, with a block-wide exclusive scan of a 0 / 1 flag per entry:
// the k-th flagged entry takes (or gives) stack slot k.  No atomics, so the result depends only on the inputs, and
// nothing is read on the host, so a CUDA graph can hold both.  Tables are small (B * M entries, a few thousand), so
// one CTA is far below a microsecond of a decoding step's work.
#include "../common.cuh"
#include "fmha_api.h"

namespace ub {
namespace {

constexpr int kThreads = 1024;
constexpr int kWarps = kThreads / 32;

// Exclusive prefix sum of `flag` over the CTA (thread order) and the CTA total.  `warp_sums` is kWarps ints of shared
// memory; the call ends with a barrier, so it can be called again at once.
UB_DEVICE int block_exclusive_scan(int flag, int* warp_sums, int& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int x = flag;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, d);
    if (lane >= d) x += y;
  }
  if (lane == 31) warp_sums[warp] = x;
  __syncthreads();
  if (warp == 0) {
    int w = warp_sums[lane];   // kWarps == 32
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, w, d);
      if (lane >= d) w += y;
    }
    warp_sums[lane] = w;   // inclusive sums of the warps
  }
  __syncthreads();
  const int before = warp > 0 ? warp_sums[warp - 1] : 0;
  total = warp_sums[kWarps - 1];
  __syncthreads();
  return before + x - flag;
}

// first table entry of sequence b that lies wholly at or past its clamped length: ceil(min(max(len, 0), C) / bs)
UB_DEVICE int blocks_needed(const KvBlocksParams& p, int b) {
  const long long cap = (long long)p.blocks_per_seq * p.block_size;
  long long n = p.lengths[b];
  n = n < 0 ? 0 : (n > cap ? cap : n);
  return (int)((n + p.block_size - 1) / p.block_size);
}

__global__ void __launch_bounds__(kThreads) kv_blocks_reserve_kernel(const KvBlocksParams p) {
  static_assert(kWarps == 32, "the scan's second level is one warp");
  __shared__ int warp_sums[kWarps];
  const int count = min(max(*p.free_count, 0), p.num_blocks);
  const long long entries = (long long)p.B * p.blocks_per_seq;
  int taken = 0;   // blocks handed out so far (may exceed count: the entries past it overflow)
  for (long long base = 0; base < entries; base += kThreads) {
    const long long e = base + threadIdx.x;
    bool need = false;
    if (e < entries) {
      const int b = (int)(e / p.blocks_per_seq), i = (int)(e % p.blocks_per_seq);
      need = i < blocks_needed(p, b) && p.block_table[e] < 0;
    }
    int total;
    const int k = taken + block_exclusive_scan(need ? 1 : 0, warp_sums, total);
    if (need) {
      if (k < count) p.block_table[e] = p.free_list[count - 1 - k];
      else *p.overflow = 1;   // every writer stores the same value
    }
    taken += total;
  }
  if (threadIdx.x == 0) *p.free_count = count - min(taken, count);
}

__global__ void __launch_bounds__(kThreads) kv_blocks_release_kernel(const KvBlocksParams p) {
  __shared__ int warp_sums[kWarps];
  const int count = min(max(*p.free_count, 0), p.num_blocks);
  const long long entries = (long long)p.B * p.blocks_per_seq;
  long long pushed = 0;
  for (long long base = 0; base < entries; base += kThreads) {
    const long long e = base + threadIdx.x;
    bool drop = false, push = false;
    int blk = -1;
    if (e < entries) {
      const int b = (int)(e / p.blocks_per_seq), i = (int)(e % p.blocks_per_seq);
      drop = i >= blocks_needed(p, b);
      blk = p.block_table[e];
      push = drop && blk >= 0 && blk < p.num_blocks;
    }
    int total;
    const long long slot = count + pushed + block_exclusive_scan(push ? 1 : 0, warp_sums, total);
    if (push && slot < p.num_blocks) p.free_list[slot] = blk;
    if (drop) p.block_table[e] = -1;
    pushed += total;
  }
  if (threadIdx.x == 0) *p.free_count = (int)min((long long)count + pushed, (long long)p.num_blocks);
}

}  // namespace

void launch_kv_blocks_reserve(const KvBlocksParams& p, cudaStream_t stream) {
  kv_blocks_reserve_kernel<<<1, kThreads, 0, stream>>>(p);
}

void launch_kv_blocks_release(const KvBlocksParams& p, cudaStream_t stream) {
  kv_blocks_release_kernel<<<1, kThreads, 0, stream>>>(p);
}

}  // namespace ub
