// Bindings of the peer-memory collective kernels.
#include <c10/cuda/CUDAGuard.h>

#include <vector>

#include "../api.h"
#include "../bind_util.h"
#include "comm_api.h"

namespace {
using namespace ub_bind;

// buffer_ptrs / flag_ptrs: integer device addresses of every rank's (peer-mapped) buffers as returned
// by the symmetric-memory rendezvous; multicast_ptr: NVLS alias or 0.
void symm_reduce_impl(const std::vector<int64_t>& buffer_ptrs, const std::vector<int64_t>& flag_ptrs,
                      int64_t multicast_ptr, int64_t rank, int64_t byte_offset, int64_t bytes, int64_t dtype,
                      double scale, int64_t algo, int64_t blocks, int64_t sq_acc_ptr, bool scatter_only,
                      int64_t err_ptr, int64_t tag) {
  const int world = (int)buffer_ptrs.size();
  TORCH_CHECK(world >= 1 && world <= ub::kMaxPeers, "world size must be in [1, ", ub::kMaxPeers, "]");
  TORCH_CHECK((int)flag_ptrs.size() == world && rank >= 0 && rank < world);
  TORCH_CHECK(byte_offset % 16 == 0 && bytes % 16 == 0, "range must be 16-byte aligned");
  ub::CommPeers peers{};
  for (int i = 0; i < world; ++i) {
    peers.buf[i] = reinterpret_cast<void*>(buffer_ptrs[i]);
    peers.flags[i] = reinterpret_cast<void*>(flag_ptrs[i]);
  }
  peers.multicast = reinterpret_cast<void*>(multicast_ptr);
  peers.err = reinterpret_cast<void*>(err_ptr);
  peers.tag = (uint32_t)tag;
  peers.rank = (int)rank;
  peers.world = world;
  ub::launch_allreduce(peers, byte_offset, bytes, (int)dtype, (float)scale, (int)algo, (int)blocks,
                       reinterpret_cast<float*>(sq_acc_ptr), cur_stream(), scatter_only);
  check_launch("symm_allreduce");
}

void symm_allreduce(const std::vector<int64_t>& buffer_ptrs, const std::vector<int64_t>& flag_ptrs,
                    int64_t multicast_ptr, int64_t rank, int64_t byte_offset, int64_t bytes, int64_t dtype,
                    double scale, int64_t algo, int64_t blocks, int64_t sq_out_ptr, int64_t err_ptr, int64_t tag) {
  symm_reduce_impl(buffer_ptrs, flag_ptrs, multicast_ptr, rank, byte_offset, bytes, dtype, scale, algo, blocks,
                   sq_out_ptr, false, err_ptr, tag);
}

// Reduce-scatter half only: afterwards rank r's buffer holds the reduced values of ITS slice of the range
// (16-byte vectors [begin + r*per, begin + (r+1)*per), per = ceil(n_vectors / world)); the rest is stale.
void symm_reduce_scatter(const std::vector<int64_t>& buffer_ptrs, const std::vector<int64_t>& flag_ptrs,
                         int64_t multicast_ptr, int64_t rank, int64_t byte_offset, int64_t bytes, int64_t dtype,
                         double scale, int64_t blocks, int64_t sq_out_ptr, int64_t err_ptr, int64_t tag) {
  symm_reduce_impl(buffer_ptrs, flag_ptrs, multicast_ptr, rank, byte_offset, bytes, dtype, scale, ub::kAlgoAuto, blocks,
                   sq_out_ptr, true, err_ptr, tag);
}

ub::CommPeers make_sync(const std::vector<int64_t>& buf_ptrs, const std::vector<int64_t>& flag_ptrs, int64_t err_ptr,
                        int64_t rank, int64_t tag) {
  const int world = (int)flag_ptrs.size();
  TORCH_CHECK(world >= 1 && world <= ub::kMaxPeers && rank >= 0 && rank < world, "bad rank / world size");
  TORCH_CHECK(buf_ptrs.empty() || (int)buf_ptrs.size() == world);
  ub::CommPeers peers{};
  for (int i = 0; i < world; ++i) {
    peers.buf[i] = buf_ptrs.empty() ? nullptr : reinterpret_cast<void*>(buf_ptrs[i]);
    peers.flags[i] = reinterpret_cast<void*>(flag_ptrs[i]);
  }
  peers.multicast = nullptr;
  peers.err = reinterpret_cast<void*>(err_ptr);
  peers.tag = (uint32_t)tag;
  peers.rank = (int)rank;
  peers.world = world;
  return peers;
}

// K doubles summed over ranks through the symmetric exchange buffer (see comm_api.h); src / dst are local tensors.
void symm_stats_allreduce(const std::vector<int64_t>& xchg_ptrs, const std::vector<int64_t>& flag_ptrs, int64_t err_ptr,
                          int64_t rank, int64_t tag, const at::Tensor& src, at::Tensor dst, int64_t parity) {
  check_operand(src, "src", src.device(), {at::kDouble});
  check_operand(dst, "dst", src.device(), {at::kDouble}, {src.numel()}, kContig | kNumel);
  TORCH_CHECK(src.numel() <= ub::kMaxStats, "at most SYMM_MAX_STATS statistics");
  const c10::cuda::CUDAGuard guard(src.device());
  ub::CommPeers x = make_sync(xchg_ptrs, flag_ptrs, err_ptr, rank, tag);
  ub::launch_stats_allreduce(x, src.data_ptr<double>(), dst.data_ptr<double>(), (int)src.numel(), (int)(parity & 1),
                             cur_stream());
  check_launch("symm_stats_allreduce");
}

// The fused optimizer tail (csrc/comm/fused_step.cu).  Per flat parameter group g: peer addresses + multicast alias of
// its symmetric gradient and parameter arenas, the COMPACT fp32 state of this rank's shard, optionally the full-length
// fp32 EMA arena, and the group's hyper-parameters hyper[g] = {beta1, beta2, eps, step_size, decay_mul}.
// `ranges`: int64 CUDA tensor [nranges, 6] = {bucket_lo, bucket_hi, lo, hi, compact_off, group} (elements).
void symm_fused_tail(const std::vector<int64_t>& xchg_ptrs, const std::vector<int64_t>& flag_ptrs, int64_t err_ptr,
                     int64_t rank, int64_t tag, const std::vector<std::vector<int64_t>>& grad_ptrs,
                     const std::vector<int64_t>& grad_mc, const std::vector<std::vector<int64_t>>& param_ptrs,
                     const std::vector<int64_t>& param_mc, const std::vector<at::Tensor>& master,
                     const std::vector<at::Tensor>& exp_avg, const std::vector<at::Tensor>& exp_avg_sq,
                     const std::vector<std::optional<at::Tensor>>& ema, const std::vector<int64_t>& numel,
                     const std::vector<int64_t>& dtypes, const std::vector<std::vector<double>>& hyper,
                     const at::Tensor& ranges, uint64_t pending_mask, at::Tensor bucket_sq, at::Tensor block_sq,
                     at::Tensor grid_sync, const std::optional<at::Tensor>& stats_src,
                     const std::optional<at::Tensor>& stats_dst, int64_t parity, int64_t denom_index, double factor,
                     double max_norm, double clip_eps, double rs_scale, double ema_decay, bool stochastic_rounding,
                     int64_t seed, int64_t offset, at::Tensor state, int64_t blocks) {
  const int ng = (int)grad_ptrs.size();
  TORCH_CHECK(ng >= 1 && ng <= ub::kMaxTailGroups, "between 1 and ", ub::kMaxTailGroups, " parameter groups");
  TORCH_CHECK((int)param_ptrs.size() == ng && (int)grad_mc.size() == ng && (int)param_mc.size() == ng &&
              (int)master.size() == ng && (int)exp_avg.size() == ng && (int)exp_avg_sq.size() == ng &&
              (int)ema.size() == ng && (int)numel.size() == ng && (int)dtypes.size() == ng && (int)hyper.size() == ng);
  const c10::Device dev = state.device();
  check_operand(state, "state", dev, {at::kFloat});
  check_operand(ranges, "ranges", dev, {at::kLong}, {kAnySize, 6});
  TORCH_CHECK(ranges.size(0) >= 1 && ranges.size(0) <= ub::kMaxTailRanges, "bad range table");
  const int nr = (int)ranges.size(0);
  const int cap = ub::fused_tail_max_blocks();
  if (blocks <= 0 || blocks > cap) blocks = cap;
  check_operand(bucket_sq, "bucket_sq", dev, {at::kFloat});
  check_operand(block_sq, "block_sq", dev, {at::kFloat});
  check_operand(grid_sync, "grid_sync", dev, {at::kInt});
  TORCH_CHECK(bucket_sq.numel() >= (int64_t)nr * ub::kMaxCommBlocks, "bucket_sq must hold SYMM_MAX_BLOCKS per range");
  TORCH_CHECK(block_sq.numel() >= blocks, "block_sq must hold one float per block");
  TORCH_CHECK(grid_sync.numel() >= 4, "grid_sync must hold 4 words");
  TORCH_CHECK(state.numel() >= 4, "state must hold 4 words");
  const bool stats = has(stats_src) && stats_src->numel() > 0;
  TORCH_CHECK(!stats || has(stats_dst), "stats_src needs stats_dst");
  if (stats) {
    check_operand(stats_src, "stats_src", dev, {at::kDouble});
    check_operand(stats_dst, "stats_dst", dev, {at::kDouble}, {stats_src->numel()}, kContig | kNumel);
    TORCH_CHECK(stats_src->numel() <= ub::kMaxStats, "at most SYMM_MAX_STATS statistics");
  }
  for (int g = 0; g < ng; ++g) {
    check_operand(master[g], "master", dev, {at::kFloat}, {}, kVec);
    check_operand(exp_avg[g], "exp_avg", dev, {at::kFloat}, {master[g].numel()}, kVec | kNumel);
    check_operand(exp_avg_sq[g], "exp_avg_sq", dev, {at::kFloat}, {master[g].numel()}, kVec | kNumel);
    // (the arena view may end a few elements before the padded length; its STORAGE must cover the padding)
    check_operand(ema[g], "ema", dev, {at::kFloat}, {}, kVec);
    if (has(ema[g])) {
      const int64_t room = (int64_t)(ema[g]->storage().nbytes() / sizeof(float)) - ema[g]->storage_offset();
      TORCH_CHECK(room >= numel[g], "ema must have storage for the padded arena length");
    }
    TORCH_CHECK(numel[g] % 8 == 0, "arena lengths must be multiples of 8 elements");
    TORCH_CHECK(dtypes[g] == ub::kF16 || dtypes[g] == ub::kBF16, "16-bit arenas expected");
    TORCH_CHECK(hyper[g].size() == 5, "hyper: {beta1, beta2, eps, step_size, decay_mul} per group");
  }
  const c10::cuda::CUDAGuard guard(dev);
  ub::TailArgs a{};
  a.sync = make_sync(xchg_ptrs, flag_ptrs, err_ptr, rank, tag);
  const int world = a.sync.world;
  for (int g = 0; g < ng; ++g) {
    ub::TailGroup& G = a.groups[g];
    TORCH_CHECK((int)grad_ptrs[g].size() == world && (int)param_ptrs[g].size() == world);
    for (int r = 0; r < world; ++r) {
      G.grad[r] = reinterpret_cast<void*>(grad_ptrs[g][r]);
      G.param[r] = reinterpret_cast<void*>(param_ptrs[g][r]);
      TORCH_CHECK(aligned16(G.grad[r]) && aligned16(G.param[r]), "arenas must be 16-byte aligned");
    }
    G.grad_mc = reinterpret_cast<void*>(grad_mc[g]);
    G.param_mc = reinterpret_cast<void*>(param_mc[g]);
    G.master = master[g].data_ptr<float>();
    G.exp_avg = exp_avg[g].data_ptr<float>();
    G.exp_avg_sq = exp_avg_sq[g].data_ptr<float>();
    G.ema = has(ema[g]) ? ema[g]->data_ptr<float>() : nullptr;
    G.numel = numel[g];
    G.dtype = (int)dtypes[g];
    G.beta1 = (float)hyper[g][0];
    G.beta2 = (float)hyper[g][1];
    G.eps = (float)hyper[g][2];
    G.step_size = (float)hyper[g][3];
    G.decay_mul = (float)hyper[g][4];
  }
  a.ngroups = ng;
  a.nranges = nr;
  a.ranges = reinterpret_cast<const ub::TailRange*>(ranges.data_ptr<int64_t>());
  a.pending_mask = pending_mask;
  a.bucket_sq = bucket_sq.data_ptr<float>();
  a.block_sq = block_sq.data_ptr<float>();
  a.grid_sync = reinterpret_cast<unsigned int*>(grid_sync.data_ptr<int>());
  a.stats_src = stats ? stats_src->data_ptr<double>() : nullptr;
  a.stats_dst = stats ? stats_dst->data_ptr<double>() : nullptr;
  a.nstats = stats ? (int)stats_src->numel() : 0;
  a.parity = (int)(parity & 1);
  a.denom_index = (int)denom_index;
  a.factor = (float)factor;
  a.max_norm = (float)max_norm;
  a.clip_eps = (float)clip_eps;
  a.rs_scale = (float)rs_scale;
  a.ema_decay = (float)ema_decay;
  a.stochastic_rounding = stochastic_rounding ? 1 : 0;
  a.seed = (unsigned long long)seed;
  a.offset = (unsigned long long)offset;
  a.state = state.data_ptr<float>();
  ub::launch_fused_tail(a, (int)blocks, cur_stream());
  check_launch("symm_fused_tail");
}

// Pinned, device-mapped host words for the communicator's error channel: returns (host tensor view, device address).
std::tuple<at::Tensor, int64_t> symm_error_channel() {
  uint32_t* host = nullptr;
  cudaError_t err = cudaHostAlloc(reinterpret_cast<void**>(&host), 4 * sizeof(uint32_t), cudaHostAllocMapped);
  TORCH_CHECK(err == cudaSuccess, "cudaHostAlloc failed: ", cudaGetErrorString(err));
  for (int i = 0; i < 4; ++i) host[i] = 0u;
  void* dev = nullptr;
  err = cudaHostGetDevicePointer(&dev, host, 0);
  TORCH_CHECK(err == cudaSuccess, "cudaHostGetDevicePointer failed: ", cudaGetErrorString(err));
  at::Tensor view = at::from_blob(host, {4}, [](void* p) { cudaFreeHost(p); }, at::TensorOptions().dtype(at::kInt));
  return {view, reinterpret_cast<int64_t>(dev)};
}

int64_t symm_pick_algo(int64_t bytes, int64_t world, bool has_multicast) {
  return ub::pick_allreduce_algo(bytes, (int)world, has_multicast);
}

}  // namespace

void register_comm(pybind11::module_& m) {
  m.def("symm_allreduce", &symm_allreduce);
  m.def("symm_reduce_scatter", &symm_reduce_scatter);
  m.def("symm_pick_algo", &symm_pick_algo);
  m.def("symm_fused_tail", &symm_fused_tail);
  m.def("symm_stats_allreduce", &symm_stats_allreduce);
  m.def("symm_error_channel", &symm_error_channel);
  m.def("symm_tail_max_blocks", []() { return (int64_t)ub::fused_tail_max_blocks(); });
  m.attr("SYMM_MAX_BLOCKS") = (int64_t)ub::kMaxCommBlocks;
  m.attr("SYMM_MAX_PEERS") = (int64_t)ub::kMaxPeers;
  m.attr("SYMM_MAX_TAIL_RANGES") = (int64_t)ub::kMaxTailRanges;
  m.attr("SYMM_MAX_TAIL_GROUPS") = (int64_t)ub::kMaxTailGroups;
  m.attr("SYMM_MAX_STATS") = (int64_t)ub::kMaxStats;
  m.attr("SYMM_XCHG_DOUBLES_PER_RANK") = (int64_t)(1 + ub::kMaxStats);
}
