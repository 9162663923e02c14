// Gradient all-reduce over NVLink 4 / NVSwitch peer memory (sm_90a), replacing the NCCL all-reduce
// issued by DDP in the reference (unicore/models/distributed_unicore_model.py:37-46) on the
// gradient path.  The flat 16-bit gradient arena lives in symmetric memory (every rank maps every
// peer's buffer + an NVLS multicast alias), so the kernels below read/write peers with plain
// ld/st.global or multimem.* and synchronise with flags in a symmetric signal buffer:
//
//   one-shot : every rank reads the range from all peers and reduces locally (latency optimal,
//              used for small ranges / statistics vectors)
//   two-shot : rank r reduces its 1/N slice from all peers (reduce-scatter by peer loads) and
//              writes the result into every peer (all-gather by peer stores)
//   nvls     : rank r issues multimem.ld_reduce on its slice (reduction inside the NVSwitch, fp32
//              accumulate) and multimem.st to broadcast it - each byte crosses each link once
//
// Reduction order is the fixed rank order 0..N-1 with fp32 accumulation, so every replica ends up
// with bit-identical gradients.  An optional scale (1/world) is applied before the 16-bit store.
#include "comm_device.cuh"

namespace ub {

// Rendezvous of the ranks before a data kernel: ONE warp per GPU waits until every peer's stream has
// reached the same point (i.e. its producer kernels have finished).  Ranks are skewed by up to a few
// hundred microseconds inside a backward pass; parking that wait in a 32-thread kernel instead of in
// the data kernel's CTAs leaves the SMs to the compute kernels the reduction overlaps with.
__global__ void __launch_bounds__(32) symm_handshake_kernel(CommPeers peers) {
  slot_barrier(peers, kHandshakeSlot, /*release_first=*/false);
}

// Sum of squares of this CTA -> sq_out[blockIdx.x] (a plain store: the consumer adds the slots of all launches in a
// fixed order, so the gradient norm is bit-reproducible run to run - no floating-point atomics anywhere).
UB_DEVICE void publish_sq(float sq, float* sq_out) {
  if (sq_out == nullptr) return;
  const float v = comm_block_sum(sq);
  if (threadIdx.x == 0) sq_out[blockIdx.x] = v;
}

// ---- one-shot / two-shot ------------------------------------------------------------------------------------------
// Range = [begin_vec, end_vec) in 16-byte vectors relative to each buffer base.
constexpr int kCommUnroll = 4;  // vectors per thread in flight per peer (NVLink latency ~2-3 us)

// One-shot, in place: every rank reads the whole range from every peer, so nobody may store its result
// before all peers have finished reading - the grid covers the range with ONE vector per thread, the
// reduced value waits in registers across a second barrier.  (Host guarantees grid * 512 >= vectors.)
template <typename T>
__global__ void __launch_bounds__(kCommThreads) allreduce_oneshot_kernel(CommPeers peers, long long begin_vec,
                                                                          long long end_vec, float scale, float* sq_out) {
  constexpr int EPV = 16 / sizeof(T);
  // (the handshake kernel ahead of us in the stream established that every rank's producers finished)
  const long long v = begin_vec + (long long)blockIdx.x * kCommThreads + threadIdx.x;
  const bool active = v < end_vec;
  float acc[EPV];
#pragma unroll
  for (int e = 0; e < EPV; ++e) acc[e] = 0.f;
  if (active) {
    Vec16 in[kMaxPeers];
#pragma unroll
    for (int p = 0; p < kMaxPeers; ++p) {
      if (p < peers.world) in[p] = ld_global_v4(reinterpret_cast<const uint8_t*>(peers.buf[p]) + v * 16);
    }
#pragma unroll
    for (int p = 0; p < kMaxPeers; ++p) {
      if (p < peers.world) acc_add<T>(acc, in[p]);
    }
  }
  const bool healthy = block_barrier(peers, /*release_first=*/false);  // all peers hold their sums in registers
  float sq = 0.f;
  if (active && healthy) {
#pragma unroll
    for (int e = 0; e < EPV; ++e) acc[e] *= scale;
    st_global_v4(reinterpret_cast<uint8_t*>(peers.buf[peers.rank]) + v * 16, pack<T>(acc));
    // every rank holds the whole result here; each counts only "its" 1/world slice so that the ranks' sums add up
    const long long n = end_vec - begin_vec, per = (n + peers.world - 1) / peers.world;
    const long long lo = begin_vec + per * peers.rank;
    if (v >= lo && v < lo + per) {
#pragma unroll
      for (int e = 0; e < EPV; ++e) sq += acc[e] * acc[e];
    }
  }
  publish_sq(sq, sq_out);
}

// Two-shot: rank r owns slice r: reduce-scatter by peer loads, all-gather by peer stores.
// W = compile-time bound on the world size (2 / 4 / 8); W * kU = 16 peer vectors in flight per thread.
template <typename T, int W, bool kScatterOnly = false>
__global__ void __launch_bounds__(kCommThreads) allreduce_twoshot_kernel(CommPeers peers, long long begin_vec,
                                                                          long long end_vec, float scale, float* sq_out) {
  constexpr int EPV = 16 / sizeof(T);
  constexpr int kU = 16 / W;
  const long long n = end_vec - begin_vec;
  const long long per = (n + peers.world - 1) / peers.world;
  long long lo = begin_vec + per * peers.rank;
  const long long hi = lo + per < end_vec ? lo + per : end_vec;
  if (lo > end_vec) lo = end_vec;
  const long long stride = (long long)gridDim.x * kCommThreads;
  float sq = 0.f;
  for (long long v0 = lo + (long long)blockIdx.x * kCommThreads + threadIdx.x; v0 < hi; v0 += stride * kU) {
    Vec16 in[kU][W];
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const long long v = v0 + u * stride;
#pragma unroll
      for (int p = 0; p < W; ++p) {
        if (p < peers.world && v < hi) in[u][p] = ld_global_v4(reinterpret_cast<const uint8_t*>(peers.buf[p]) + v * 16);
      }
    }
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const long long v = v0 + u * stride;
      if (v < hi) {
        float acc[EPV];
#pragma unroll
        for (int e = 0; e < EPV; ++e) acc[e] = 0.f;
#pragma unroll
        for (int p = 0; p < W; ++p) {
          if (p < peers.world) acc_add<T>(acc, in[u][p]);
        }
#pragma unroll
        for (int e = 0; e < EPV; ++e) {
          acc[e] *= scale;
          sq += acc[e] * acc[e];
        }
        const Vec16 out = pack<T>(acc);
        if (kScatterOnly) {
          st_global_v4(reinterpret_cast<uint8_t*>(peers.buf[peers.rank]) + v * 16, out);
        } else {
#pragma unroll
          for (int p = 0; p < W; ++p) {
            if (p < peers.world) st_global_v4(reinterpret_cast<uint8_t*>(peers.buf[p]) + v * 16, out);
          }
        }
      }
    }
  }
  publish_sq(sq, sq_out);
  block_barrier(peers, /*release_first=*/true);  // my stores are visible at the peers before anyone proceeds
}

// ---- NVLS (multimem) --------------------------------------------------------------------------------------------------
template <typename T, bool kScatterOnly = false>
__global__ void __launch_bounds__(kCommThreads) allreduce_nvls_kernel(CommPeers peers, long long begin_vec,
                                                                        long long end_vec, float scale, float* sq_out) {
  constexpr int EPV = 16 / sizeof(T);
  const long long n = end_vec - begin_vec;
  const long long per = (n + peers.world - 1) / peers.world;
  long long lo = begin_vec + per * peers.rank;
  long long hi = lo + per < end_vec ? lo + per : end_vec;
  if (lo > end_vec) lo = end_vec;
  uint8_t* mc = reinterpret_cast<uint8_t*>(peers.multicast);
  const long long stride = (long long)gridDim.x * kCommThreads;
  float sq = 0.f;
  for (long long v0 = lo + (long long)blockIdx.x * kCommThreads + threadIdx.x; v0 < hi; v0 += stride * kCommUnroll) {
    Vec16 r[kCommUnroll];
#pragma unroll
    for (int u = 0; u < kCommUnroll; ++u) {
      const long long v = v0 + u * stride;
      if (v < hi) r[u] = multimem_ld_reduce<T>(mc + v * 16);
    }
#pragma unroll
    for (int u = 0; u < kCommUnroll; ++u) {
      const long long v = v0 + u * stride;
      if (v < hi) {
        if (scale != 1.f || sq_out != nullptr) {
          float acc[EPV];
          unpack<T>(r[u], acc);
#pragma unroll
          for (int e = 0; e < EPV; ++e) {
            acc[e] *= scale;
            sq += acc[e] * acc[e];
          }
          r[u] = pack<T>(acc);
        }
        if (kScatterOnly) st_global_v4(reinterpret_cast<uint8_t*>(peers.buf[peers.rank]) + v * 16, r[u]);
        else multimem_st(mc + v * 16, r[u]);
      }
    }
  }
  publish_sq(sq, sq_out);
  block_barrier(peers, true);
}

// ---- host --------------------------------------------------------------------------------------------------------------
template <typename T>
static void run_allreduce(const CommPeers& peers, long long begin_vec, long long end_vec, float scale, int algo,
                          int blocks, float* sq_out, cudaStream_t stream, bool scatter_only) {
  symm_handshake_kernel<<<1, 32, 0, stream>>>(peers);
  if (scatter_only) {  // reduce-scatter half only (sharded optimizer); one-shot has no such form
    if (algo == kAlgoNvls)
      allreduce_nvls_kernel<T, true><<<blocks, kCommThreads, 0, stream>>>(peers, begin_vec, end_vec, scale, sq_out);
    else if (peers.world <= 2)
      allreduce_twoshot_kernel<T, 2, true><<<blocks, kCommThreads, 0, stream>>>(peers, begin_vec, end_vec, scale, sq_out);
    else if (peers.world <= 4)
      allreduce_twoshot_kernel<T, 4, true><<<blocks, kCommThreads, 0, stream>>>(peers, begin_vec, end_vec, scale, sq_out);
    else
      allreduce_twoshot_kernel<T, 8, true><<<blocks, kCommThreads, 0, stream>>>(peers, begin_vec, end_vec, scale, sq_out);
    return;
  }
  if (algo == kAlgoNvls) {
    allreduce_nvls_kernel<T><<<blocks, kCommThreads, 0, stream>>>(peers, begin_vec, end_vec, scale, sq_out);
  } else if (algo == kAlgoTwoShot) {
    if (peers.world <= 2)
      allreduce_twoshot_kernel<T, 2><<<blocks, kCommThreads, 0, stream>>>(peers, begin_vec, end_vec, scale, sq_out);
    else if (peers.world <= 4)
      allreduce_twoshot_kernel<T, 4><<<blocks, kCommThreads, 0, stream>>>(peers, begin_vec, end_vec, scale, sq_out);
    else
      allreduce_twoshot_kernel<T, 8><<<blocks, kCommThreads, 0, stream>>>(peers, begin_vec, end_vec, scale, sq_out);
  } else {
    allreduce_oneshot_kernel<T><<<blocks, kCommThreads, 0, stream>>>(peers, begin_vec, end_vec, scale, sq_out);
  }
}

int pick_allreduce_algo(long long bytes, int world, bool has_multicast) {
  if (bytes <= 256 * 1024) return kAlgoOneShot;
  if (has_multicast && world > 2) return kAlgoNvls;
  return kAlgoTwoShot;
}

void launch_allreduce(const CommPeers& peers, long long byte_offset, long long bytes, int dtype, float scale, int algo,
                      int blocks, float* sq_out, cudaStream_t stream, bool scatter_only) {
  const long long begin_vec = byte_offset / 16, end_vec = (byte_offset + bytes) / 16;
  if (end_vec <= begin_vec) return;
  if (algo == kAlgoAuto) algo = pick_allreduce_algo(bytes, peers.world, peers.multicast != nullptr);
  if (scatter_only && algo == kAlgoOneShot) algo = peers.multicast != nullptr && peers.world > 2 ? kAlgoNvls : kAlgoTwoShot;
  if (algo == kAlgoNvls && peers.multicast == nullptr) algo = kAlgoTwoShot;
  const long long one_shot_blocks = (end_vec - begin_vec + kCommThreads - 1) / kCommThreads;
  if (algo == kAlgoOneShot && one_shot_blocks > kMaxDataBlocks) algo = kAlgoTwoShot;  // range too large
  if (algo == kAlgoOneShot) {
    blocks = (int)one_shot_blocks;  // exactly one vector per thread (see kernel)
  } else {
    if (blocks <= 0) blocks = 24;
    if (blocks > kMaxDataBlocks) blocks = kMaxDataBlocks;  // the last slots are reserved (handshake, tail, stats)
  }
  if (dtype == kF32) run_allreduce<float>(peers, begin_vec, end_vec, scale, algo, blocks, sq_out, stream, scatter_only);
  else if (dtype == kF16) run_allreduce<__half>(peers, begin_vec, end_vec, scale, algo, blocks, sq_out, stream, scatter_only);
  else run_allreduce<__nv_bfloat16>(peers, begin_vec, end_vec, scale, algo, blocks, sq_out, stream, scatter_only);
}

}  // namespace ub
