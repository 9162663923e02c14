// Host launchers of the peer-memory collective kernels (csrc/comm/*.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace ub {

constexpr int kMaxPeers = 8;         // one NVSwitch domain (HGX H100: 8 GPUs)
constexpr int kMaxCommBlocks = 64;   // flag slots: [kMaxCommBlocks][kMaxPeers] uint32 per rank (last 3 reserved)

enum CommAlgo : int { kAlgoAuto = 0, kAlgoOneShot = 1, kAlgoTwoShot = 2, kAlgoNvls = 3 };

// Symmetric-memory view handed to the kernels by value.
struct CommPeers {
  void* buf[kMaxPeers];     // peer-mapped base address of every rank's data buffer
  void* flags[kMaxPeers];   // peer-mapped base address of every rank's flag buffer (zero-initialised)
  void* multicast;          // NVLS multicast alias of the data buffers (nullptr when unsupported)
  void* err;                // 4 x uint32 of pinned, device-mapped host memory: {code, detail, rank, -} (nullable)
  uint32_t tag;             // identifies the collective in the flag protocol (bucket index, kernel kind); 0 -> 1
  int rank, world;
};

int pick_allreduce_algo(long long bytes, int world, bool has_multicast);

// In-place sum over ranks of bytes [byte_offset, byte_offset + bytes) of the symmetric buffer
// (16-byte aligned range), fp32 accumulation in rank order, result scaled by `scale`.
// sq_out (nullable, local device memory, >= kMaxCommBlocks floats): CTA b STORES the sum of squares of the REDUCED,
// scaled values it produced for this rank's 1/world slice of the range at sq_out[b] - summed over CTAs and ranks that
// is the squared L2 norm of the result, so no separate gradient-norm pass reads the arena, and because the slots are
// added up in a fixed order by the consumer the norm is reproducible bit for bit.
// scatter_only: stop after the reduce-scatter half - rank r's 1/world slice of the range holds the result in ITS buffer
// only (slice = vectors [begin + r*per, begin + (r+1)*per), per = ceil(n/world)); the fused optimizer tail
// (fused_step.cu) consumes exactly these slices.
void launch_allreduce(const CommPeers& peers, long long byte_offset, long long bytes, int dtype, float scale, int algo,
                      int blocks, float* sq_out, cudaStream_t stream, bool scatter_only = false);

// ---- statistics vector: K doubles summed over ranks, one launch, one flag round trip -------------------------------
// xchg: symmetric buffer of 2 * world * kMaxStats doubles per rank ([parity][sender][k]); every rank stores its vector into
// every peer's [parity][rank] row, one barrier, then sums the rows in rank order (identical result everywhere).
// `parity` alternates per call so that a fast rank's next call cannot overwrite rows a slow rank still reads.
constexpr int kMaxStats = 64;
void launch_stats_allreduce(const CommPeers& xchg, const double* src, double* dst, int k, int parity, cudaStream_t stream);

// ---- the fused optimizer tail: ONE kernel after backward -------------------------------------------------------------
// (reduce-scatter of the buckets that did not overlap backward) -> squared-norm + statistics exchange over peer memory
// -> loss-scale / sample-size / clip coefficient and the overflow decision on the device -> Adam (+EMA) on this rank's
// shard of the fp32 master / moments -> new 16-bit parameters stored into EVERY rank's parameter arena (multimem.st or
// peer stores) -> gradient arena zeroed -> closing barrier.
constexpr int kMaxTailGroups = 4;
constexpr int kMaxTailRanges = 64;

struct TailGroup {              // one flat parameter group (one dtype arena pair)
  void* grad[kMaxPeers];        // symmetric GRADIENT arena (peer addresses) + multicast alias
  void* grad_mc;
  void* param[kMaxPeers];       // symmetric PARAMETER arena + multicast alias
  void* param_mc;
  float* master;                // COMPACT fp32 state of this rank's shard: owned ranges back to back
  float* exp_avg;
  float* exp_avg_sq;
  float* ema;                   // nullable: full-length fp32 EMA arena (indexed by absolute element)
  long long numel;              // arena length in elements (multiple of 8)
  float beta1, beta2, eps, step_size, decay_mul;
  int dtype;                    // kF16 / kBF16
};

struct TailRange {              // one gradient bucket of a group (six 64-bit words: uploaded from an int64 tensor)
  long long bucket_lo, bucket_hi;   // the bucket, in elements of the arena
  long long lo, hi;                 // this rank's slice of it (16-byte vectors [b + r*per, b + (r+1)*per))
  long long compact_off;            // where the slice starts in the compact state arrays
  long long group;
};

struct TailArgs {
  CommPeers sync;               // flags / err / rank / world (buf = the symmetric exchange buffer, see below)
  TailGroup groups[kMaxTailGroups];
  int ngroups, nranges;
  const TailRange* ranges;      // device array (nranges entries; uploaded once per bucket plan)
  unsigned long long pending_mask;  // bit r: bucket r has NOT been reduce-scattered yet - the tail does it first
  // norm / statistics exchange: sync.buf[r] = rank r's symmetric buffer of 2 * world * (1 + kMaxStats) doubles
  float* bucket_sq;             // [nranges][kMaxCommBlocks] partial sums of squares stored by the bucket kernels
  float* block_sq;              // [gridDim.x] scratch
  unsigned int* grid_sync;      // 4 x uint32, zero-initialised once (local grid barrier: count, generation, abort)
  const double* stats_src;      // nullable: nstats local doubles to be summed over ranks
  double* stats_dst;            // their sums (local)
  int nstats, parity;
  int denom_index;              // >= 0: gradients are additionally divided by stats sum #denom_index (sample size)
  float factor;                 // host part of the gradient multiplier (world / loss_scale ...)
  float max_norm;               // <= 0: no clipping
  float clip_eps;               // added to the norm in the clip quotient (reference: 0 for fp16, 1e-6 for bf16)
  float rs_scale;               // scale applied by the reduce-scatter (1 / world)
  float ema_decay;
  int stochastic_rounding;
  unsigned long long seed, offset;
  float* state;                 // device out: {grad_norm, grad_multiplier incl. clip, overflow (0/1), sum of squares}
};
int fused_tail_max_blocks();
void launch_fused_tail(const TailArgs& a, int blocks, cudaStream_t stream);

}  // namespace ub
