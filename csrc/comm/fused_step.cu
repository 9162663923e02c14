// The fused optimizer tail of --ddp-backend b200: ONE kernel after backward (sm_90a, NVLink 4 / NVSwitch peer memory).
//
// What the reference does between the end of backward and the next forward (unicore/trainer.py:700-760):
//   NCCL all-reduce of every gradient bucket (models/distributed_unicore_model.py:37-46)  ->  NCCL all-reduce of the
//   logging statistics (trainer.py:1011-1049)  ->  fp16->fp32 gradient copy, L2-norm kernels, host read of the norm,
//   clip, Adam, fp32->fp16 parameter copy, two gradient memsets (optim/fp16_optimizer.py:258-308)  ->  NCCL all-gather of
//   the per-rank norms for the consistency check (trainer.py:1051-1084)  ->  EMA pass (ema.py:44-60).
//
// Here the gradient buckets that become ready DURING backward are reduce-scattered by the bucket kernels of
// allreduce.cu (scatter_only: rank r ends up with the reduced 1/N slice of every bucket and the partial sum of its
// squares).  Everything else is this kernel, launched once per update on the communication stream:
//
//   P0  peer barrier: every rank's backward (and its earlier bucket kernels) has finished
//   P1  reduce-scatter of the buckets that could not overlap backward (multimem.ld_reduce through the switch, or peer
//       loads), sum of squares on the fly
//   P2  one exchange over peer memory: every rank stores {its partial sum of squares, its logging statistics} into
//       every peer's exchange row; one flag barrier; every rank adds the rows in rank order -> identical global norm,
//       identical statistics, no NCCL call.  The gradient multiplier (1/loss-scale * world/sample-size), the clip
//       coefficient and the overflow decision are computed right here on the device.
//   P3  Adam (+ EMA) on this rank's shard: 16-bit gradient slice in, compact fp32 master / moments (1/N of the state and
//       of the optimizer's HBM traffic), new 16-bit parameters stored straight into EVERY rank's parameter arena with
//       multimem.st (NVLS) or peer stores - the all-gather is the optimizer's own store.  The gradient arena is zeroed.
//   P4  peer barrier: all parameter shards have landed everywhere; the next forward may start.
//
// Only CTA 0 talks to the peers; the CTAs of one GPU meet at a counter barrier in local memory (cooperative launch).
#include "../optim/adam_math.cuh"
#include "comm_device.cuh"

namespace ub {

namespace {

// ---- grid barrier (all CTAs of this launch are co-resident: cooperative launch) ------------------------------------
UB_DEVICE void grid_barrier(unsigned int* gs) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    volatile unsigned int* gen_p = gs + 1;
    const unsigned int gen = *gen_p;
    if (atomicAdd(gs, 1u) == gridDim.x - 1) {
      gs[0] = 0u;
      __threadfence();
      atomicAdd(gs + 1, 1u);
    } else {
      while (*gen_p == gen) __nanosleep(64);
    }
    __threadfence();
  }
  __syncthreads();
}

// ---- P1: reduce-scatter of this rank's slice [lo_vec, hi_vec) (16-byte vectors) of a bucket ------------------------
template <typename T>
UB_DEVICE float tail_reduce_slice(const TailGroup& G, int rank, int world, long long lo_vec, long long hi_vec,
                                  float scale) {
  constexpr int EPV = 16 / sizeof(T);
  constexpr int kU = 4;
  uint8_t* local = reinterpret_cast<uint8_t*>(G.grad[rank]);
  const long long stride = (long long)gridDim.x * kCommThreads;
  float sq = 0.f;
  if (G.grad_mc != nullptr && world > 2) {
    const uint8_t* mc = reinterpret_cast<const uint8_t*>(G.grad_mc);
    for (long long v0 = lo_vec + (long long)blockIdx.x * kCommThreads + threadIdx.x; v0 < hi_vec; v0 += stride * kU) {
      Vec16 r[kU];
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        const long long v = v0 + u * stride;
        if (v < hi_vec) r[u] = multimem_ld_reduce<T>(mc + v * 16);
      }
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        const long long v = v0 + u * stride;
        if (v < hi_vec) {
          float acc[EPV];
          unpack<T>(r[u], acc);
#pragma unroll
          for (int e = 0; e < EPV; ++e) {
            acc[e] *= scale;
            sq += acc[e] * acc[e];
          }
          st_global_v4(local + v * 16, pack<T>(acc));
        }
      }
    }
  } else {
    // peer loads: one vector per thread and trip, `world` independent 16-byte loads in flight (132 x 512 threads keep
    // ~2 MB on the wire at 2 GPUs, the bandwidth-delay product of a link)
    for (long long v = lo_vec + (long long)blockIdx.x * kCommThreads + threadIdx.x; v < hi_vec; v += stride) {
      Vec16 in[kMaxPeers];
#pragma unroll
      for (int p = 0; p < kMaxPeers; ++p) {
        if (p < world) in[p] = ld_global_v4(reinterpret_cast<const uint8_t*>(G.grad[p]) + v * 16);
      }
      float acc[EPV];
#pragma unroll
      for (int e = 0; e < EPV; ++e) acc[e] = 0.f;
#pragma unroll
      for (int p = 0; p < kMaxPeers; ++p) {
        if (p < world) acc_add<T>(acc, in[p]);
      }
#pragma unroll
      for (int e = 0; e < EPV; ++e) {
        acc[e] *= scale;
        sq += acc[e] * acc[e];
      }
      st_global_v4(local + v * 16, pack<T>(acc));
    }
  }
  return sq;
}

// ---- P3: Adam on the slice [lo, hi) of a group (elements, multiples of 8) ----------------------------------------------
template <typename T>
UB_DEVICE void tail_adam_slice(const TailArgs& A, const TailGroup& G, const TailRange& R, float gmul) {
  const int rank = A.sync.rank, world = A.sync.world;
  T* g_local = reinterpret_cast<T*>(G.grad[rank]);
  const bool sr = A.stochastic_rounding != 0 && G.dtype == kBF16;
  const long long stride = (long long)gridDim.x * kCommThreads * 8;
  const float ema_w = 1.f - A.ema_decay;
  for (long long i = R.lo + ((long long)blockIdx.x * kCommThreads + threadIdx.x) * 8; i < R.hi; i += stride) {
    const long long c = R.compact_off + (i - R.lo);
    float g[8], p[8], m[8], v[8];
    const Vec16 gv = ld_global_v4(g_local + i);
    const Vec16 p0 = ld_global_v4(G.master + c), p1 = ld_global_v4(G.master + c + 4);
    const Vec16 m0 = ld_global_v4(G.exp_avg + c), m1 = ld_global_v4(G.exp_avg + c + 4);
    const Vec16 v0 = ld_global_v4(G.exp_avg_sq + c), v1 = ld_global_v4(G.exp_avg_sq + c + 4);
    unpack<T>(gv, g);
    unpack<float>(p0, p);
    unpack<float>(p1, p + 4);
    unpack<float>(m0, m);
    unpack<float>(m1, m + 4);
    unpack<float>(v0, v);
    unpack<float>(v1, v + 4);
#pragma unroll
    for (int k = 0; k < 8; ++k) adam_math(p[k], m[k], v[k], g[k] * gmul, G);
    st_global_v4(G.master + c, pack<float>(p));
    st_global_v4(G.master + c + 4, pack<float>(p + 4));
    st_global_v4(G.exp_avg + c, pack<float>(m));
    st_global_v4(G.exp_avg + c + 4, pack<float>(m + 4));
    st_global_v4(G.exp_avg_sq + c, pack<float>(v));
    st_global_v4(G.exp_avg_sq + c + 4, pack<float>(v + 4));
    if (G.ema != nullptr) {
      float e[8];
      unpack<float>(ld_global_v4(G.ema + i), e);
      unpack<float>(ld_global_v4(G.ema + i + 4), e + 4);
#pragma unroll
      for (int k = 0; k < 8; ++k) e[k] = ema_step(e[k], p[k], ema_w);
      st_global_v4(G.ema + i, pack<float>(e));
      st_global_v4(G.ema + i + 4, pack<float>(e + 4));
    }
    Vec16 o;
    if (sr) {
      const Philox4 r = philox4x32_10(A.seed, A.offset, (unsigned long long)i >> 3);
      const uint32_t rw[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t lo = bf16_sr_bits(p[2 * k], rw[k] & 0xffffu);
        const uint32_t hi = bf16_sr_bits(p[2 * k + 1], rw[k] >> 16);
        o.w[k] = lo | (hi << 16);
      }
    } else {
      o = pack<T>(p);
    }
    // the parameter all-gather IS this store: one instruction through the switch, or one store per peer
    if (G.param_mc != nullptr) {
      multimem_st(reinterpret_cast<T*>(G.param_mc) + i, o);
    } else {
#pragma unroll
      for (int r = 0; r < kMaxPeers; ++r) {
        if (r < world) st_global_v4(reinterpret_cast<T*>(G.param[r]) + i, o);
      }
    }
    Vec16 z;
    z.w[0] = z.w[1] = z.w[2] = z.w[3] = 0u;
    st_global_v4(g_local + i, z);
  }
}

template <typename T>
UB_DEVICE void tail_zero(T* base, long long lo, long long hi) {
  Vec16 z;
  z.w[0] = z.w[1] = z.w[2] = z.w[3] = 0u;
  const long long stride = (long long)gridDim.x * kCommThreads * 8;
  for (long long i = lo + ((long long)blockIdx.x * kCommThreads + threadIdx.x) * 8; i < hi; i += stride)
    st_global_v4(base + i, z);
}

constexpr int kXchgRow = 1 + kMaxStats;  // doubles per sender row: {sum of squares, statistics...}

UB_DEVICE bool range_pending(const TailArgs& A, int r) { return (A.pending_mask >> r) & 1ull; }

__global__ void __launch_bounds__(kCommThreads) fused_tail_kernel(TailArgs A) {
  const int rank = A.sync.rank, world = A.sync.world;
  __shared__ double tot_s[kXchgRow];
  __shared__ float bcast_s[4];
  bool healthy = true;  // block-uniform by construction (barrier results are broadcast through shared memory)

  // ---- P0: every rank has finished backward and its bucket kernels -------------------------------------------
  if (blockIdx.x == 0) {
    healthy = slot_barrier(A.sync, kTailSlot, /*release_first=*/false);
    if (threadIdx.x == 0) {
      A.grid_sync[2] = healthy ? 0u : 1u;  // the other CTAs learn about a broken communicator from local memory
      __threadfence();
    }
  }
  grid_barrier(A.grid_sync);
  if (threadIdx.x == 0) bcast_s[2] = *reinterpret_cast<volatile unsigned int*>(A.grid_sync + 2) != 0u ? 1.f : 0.f;
  __syncthreads();
  healthy = bcast_s[2] == 0.f;

  // ---- P1: reduce-scatter what did not overlap backward --------------------------------------------------------------
  float sq = 0.f;
  if (healthy && A.pending_mask != 0ull) {
    for (int r = 0; r < A.nranges; ++r) {
      if (!range_pending(A, r)) continue;
      const TailRange R = A.ranges[r];
      const TailGroup& G = A.groups[(int)R.group];
      if (G.dtype == kF16) sq += tail_reduce_slice<__half>(G, rank, world, R.lo / 8, R.hi / 8, A.rs_scale);
      else sq += tail_reduce_slice<__nv_bfloat16>(G, rank, world, R.lo / 8, R.hi / 8, A.rs_scale);
    }
  }
  {
    const float v = comm_block_sum(sq);
    if (threadIdx.x == 0) A.block_sq[blockIdx.x] = v;
  }
  grid_barrier(A.grid_sync);

  // ---- P2: norm + statistics exchange, multiplier / clip / overflow on the device ----------------------------------------
  if (blockIdx.x == 0) {
    // local sum of squares in a FIXED order: bucket-kernel slots, then this launch's CTAs (double accumulation)
    double local = 0.0;
    if (threadIdx.x < 32) {
      const int n_slots = A.nranges * kMaxCommBlocks;
      double part = 0.0;
      for (int i = threadIdx.x; i < n_slots; i += 32) part += (double)A.bucket_sq[i];
      for (int i = threadIdx.x; i < (int)gridDim.x; i += 32) part += (double)A.block_sq[i];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
      local = part;
    }
    if (threadIdx.x == 0) tot_s[0] = local;
    __syncthreads();
    local = tot_s[0];
    __syncthreads();
    const int nk = 1 + A.nstats;
    if (healthy) {
      for (int idx = threadIdx.x; idx < world * nk; idx += kCommThreads) {
        const int p = idx / nk, k = idx - p * nk;
        double* row = reinterpret_cast<double*>(A.sync.buf[p]) + ((size_t)A.parity * world + rank) * kXchgRow;
        row[k] = k == 0 ? local : A.stats_src[k - 1];
      }
      healthy = slot_barrier(A.sync, kTailSlot, /*release_first=*/true);
    }
    if (threadIdx.x < nk) {
      const volatile double* mine =
          reinterpret_cast<const volatile double*>(A.sync.buf[rank]) + (size_t)A.parity * world * kXchgRow;
      double s = 0.0;
      for (int r = 0; r < world; ++r) s += mine[(size_t)r * kXchgRow + threadIdx.x];
      tot_s[threadIdx.x] = s;
      if (threadIdx.x > 0 && A.stats_dst != nullptr) A.stats_dst[threadIdx.x - 1] = s;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      const double total_sq = tot_s[0];
      double denom = 1.0;
      if (A.denom_index >= 0 && A.denom_index < A.nstats && tot_s[1 + A.denom_index] > 0.0) denom = tot_s[1 + A.denom_index];
      const float gmul0 = (float)((double)A.factor / denom);
      const float norm = sqrtf((float)total_sq) * gmul0;  // the true (unscaled, normalised) gradient norm
      const bool overflow = !healthy || !isfinite(norm);
      float coef = 1.f;
      if (A.max_norm > 0.f && norm > A.max_norm) coef = A.max_norm / (norm + A.clip_eps);
      A.state[0] = norm;
      A.state[1] = gmul0 * coef;
      A.state[2] = overflow ? 1.f : 0.f;
      A.state[3] = (float)total_sq;
      __threadfence();
    }
    // the bucket kernels of the next update store (not accumulate) into their slots; slots of buckets that stay
    // pending next time must read as zero
    for (int i = threadIdx.x; i < A.nranges * kMaxCommBlocks; i += kCommThreads) A.bucket_sq[i] = 0.f;
  }
  grid_barrier(A.grid_sync);
  if (threadIdx.x == 0) {
    bcast_s[0] = *reinterpret_cast<volatile float*>(A.state + 1);
    bcast_s[1] = *reinterpret_cast<volatile float*>(A.state + 2);
  }
  __syncthreads();
  const float gmul = bcast_s[0];
  const bool overflow = bcast_s[1] != 0.f;

  // ---- P3: Adam (+EMA) on this rank's shard, parameters to every rank, gradient arena zeroed -----------------------------
  // (every peer passed the barrier of P2, i.e. nobody reads this rank's gradient arena any more)
  for (int r = 0; r < A.nranges; ++r) {
    const TailRange R = A.ranges[r];
    const TailGroup& G = A.groups[(int)R.group];
    if (G.dtype == kF16) {
      __half* gl = reinterpret_cast<__half*>(G.grad[rank]);
      if (!overflow) {
        tail_adam_slice<__half>(A, G, R, gmul);
        tail_zero(gl, R.bucket_lo, R.lo);
        tail_zero(gl, R.hi, R.bucket_hi);
      } else {
        tail_zero(gl, R.bucket_lo, R.bucket_hi);
      }
    } else {
      __nv_bfloat16* gl = reinterpret_cast<__nv_bfloat16*>(G.grad[rank]);
      if (!overflow) {
        tail_adam_slice<__nv_bfloat16>(A, G, R, gmul);
        tail_zero(gl, R.bucket_lo, R.lo);
        tail_zero(gl, R.hi, R.bucket_hi);
      } else {
        tail_zero(gl, R.bucket_lo, R.bucket_hi);
      }
    }
  }

  // ---- P4: all shards have landed everywhere --------------------------------------------------------------------------
  __threadfence_system();
  grid_barrier(A.grid_sync);
  if (blockIdx.x == 0) slot_barrier(A.sync, kTailSlot, /*release_first=*/true);  // (returns at once when broken)
}

// ---- stand-alone statistics reduction (validation steps, replicated-optimizer fallback) ------------------------------
__global__ void __launch_bounds__(kMaxStats) stats_allreduce_kernel(CommPeers x, const double* __restrict__ src,
                                                                    double* __restrict__ dst, int k, int parity) {
  const int rank = x.rank, world = x.world;
  for (int idx = threadIdx.x; idx < world * k; idx += kMaxStats) {
    const int p = idx / k, j = idx - p * k;
    double* row = reinterpret_cast<double*>(x.buf[p]) + ((size_t)parity * world + rank) * kXchgRow;
    row[1 + j] = src[j];
  }
  if (!slot_barrier(x, kStatsSlot, /*release_first=*/true)) return;
  if (threadIdx.x < k) {
    const volatile double* mine = reinterpret_cast<const volatile double*>(x.buf[rank]) + (size_t)parity * world * kXchgRow;
    double s = 0.0;
    for (int r = 0; r < world; ++r) s += mine[(size_t)r * kXchgRow + 1 + threadIdx.x];
    dst[threadIdx.x] = s;
  }
}

}  // namespace

// one CTA per SM: enough to saturate HBM and the links, always co-resident
int fused_tail_max_blocks() { return device_sm_count(); }

void launch_fused_tail(const TailArgs& a, int blocks, cudaStream_t stream) {
  const int cap = fused_tail_max_blocks();
  if (blocks <= 0 || blocks > cap) blocks = cap;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)blocks);
  cfg.blockDim = dim3(kCommThreads);
  cfg.dynamicSmemBytes = 0;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;  // all CTAs co-resident: the kernel contains a grid-wide barrier
  attr[0].val.cooperative = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  cudaLaunchKernelEx(&cfg, fused_tail_kernel, a);
}

void launch_stats_allreduce(const CommPeers& xchg, const double* src, double* dst, int k, int parity, cudaStream_t stream) {
  if (k <= 0) return;
  if (k > kMaxStats) k = kMaxStats;
  stats_allreduce_kernel<<<1, kMaxStats, 0, stream>>>(xchg, src, dst, k, parity);
}

}  // namespace ub
