#!/usr/bin/env python3
"""Gradient reduction + optimizer update per gradient size: three ways of doing the same work (BASELINE config 5).

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 \
        --master-port 29532 bench/fused_step_sweep.py [--max-mb 256]

For every size (1 MB .. --max-mb of 16-bit gradients, x4 steps, 25 MB buckets) it times, with CUDA events, max over
ranks, "local gradients are ready" -> "new 16-bit parameters on every rank, gradients zeroed, norm known":

  nccl    NCCL all-reduce per bucket + L2-norm kernel + replicated fused Adam kernel   (what --ddp-backend c10d runs)
  symm    our all-reduce kernels per bucket (one-shot / two-shot / NVLS, squared norm on the fly) + the 64-thread norm
          exchange + replicated fused Adam kernel                                       (b200 without the fused tail)
  fused   reduce-scatter bucket kernels for all buckets but the last + ONE fused tail kernel (last bucket's
          reduce-scatter, norm exchange, clip, Adam on the 1/N shard, parameter all-gather by multimem.st)  (b200 default)

and checks that the three leave the same 16-bit parameters behind.  Each line carries the roofline
max(36 B/param / HBM peak, gradient bytes / 450 GB/s per direction of H100 NVLink 4) and the SM clock record.  Rank 0 prints one JSON
object per size.
"""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from op_compare import Clocks, peaks  # noqa: E402


def timed(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    dist.barrier()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    t = torch.tensor([s.elapsed_time(e) / iters], device="cuda", dtype=torch.float64)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--max-mb", type=int, default=256)
    ap.add_argument("--dtype", default="bfloat16", choices=["bfloat16", "float16"])
    ap.add_argument("--bucket-mb", type=int, default=25)
    args = ap.parse_args()
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
    dist.init_process_group("nccl", init_method="env://")
    dist.all_reduce(torch.zeros(1, device="cuda"))

    from unicore import ops, utils
    from unicore_b200.parallel.comm import TAG_BUCKET, SymmComm
    from unicore_b200.parallel.fused_tail import FusedTail, adam_hyper, plan_buckets
    from unicore_b200.parallel.symm_dp import symm_available

    assert symm_available(), "symmetric memory / native kernels unavailable"
    dtype = getattr(torch, args.dtype)
    comm = SymmComm()
    hbm = peaks()
    clocks = Clocks() if rank == 0 else None
    hyper = dict(lr=1e-3, beta1=0.9, beta2=0.98, eps=1e-6, step=1, bias_correction=True, weight_decay=0.01)
    mb = 1
    while mb <= args.max_mb:
        n = mb * 1024 * 1024 // 2
        grads = comm.allocate(n, dtype)       # symmetric gradient arena
        params = comm.allocate(n, dtype)      # symmetric parameter arena
        torch.manual_seed(1)
        init = torch.randn(n, device="cuda") * 0.02
        local_grad = (torch.randn(n, device="cuda", generator=torch.Generator("cuda").manual_seed(100 + rank)) * 1e-2).to(dtype)
        tail = FusedTail(comm, [grads], [params], args.bucket_mb << 20)
        buckets = [(b.lo, b.hi, b.index) for b in tail.buckets]
        n_slots = comm.max_blocks
        slots = torch.zeros(len(buckets) * n_slots, dtype=torch.float32, device="cuda")
        state = {}

        def reset(which):
            full = init.clone()
            if which == "fused":
                state[which] = dict(master=tail.to_compact(full, 0))
                state[which]["m"] = torch.zeros_like(state[which]["master"])
                state[which]["v"] = torch.zeros_like(state[which]["master"])
            else:
                state[which] = dict(master=full, m=torch.zeros(n, device="cuda"), v=torch.zeros(n, device="cuda"))
            params.tensor.copy_(init.to(dtype))

        def work_item(st):
            return [dict(p=st["master"], g=grads.tensor, m=st["m"], v=st["v"], p_half=params.tensor, **hyper)]

        def clip_scale(norm):  # device-side: divisor = max(1, norm / max_norm)
            return torch.clamp(norm, min=1.0)

        def run_nccl():
            grads.tensor.copy_(local_grad)
            for lo, hi, _ in buckets:
                dist.all_reduce(grads.tensor[lo:hi])
            norm = utils.multi_tensor_total_norm([grads.tensor]) / world
            ops.fused_adam(work_item(state["nccl"]), grad_scale=clip_scale(norm) * world, zero_grad=True)

        def run_symm():
            grads.tensor.copy_(local_grad)
            for lo, hi, i in buckets:
                comm.all_reduce(grads, lo, hi - lo, scale=1.0 / world, sq_out=slots[i * n_slots:(i + 1) * n_slots],
                                tag=TAG_BUCKET + i)
            total = comm.stats_allreduce(slots.double().sum().reshape(1))
            slots.zero_()
            ops.fused_adam(work_item(state["symm"]), grad_scale=clip_scale(total[0].float().sqrt()), zero_grad=True)

        hyp = [adam_hyper(hyper["lr"], hyper["beta1"], hyper["beta2"], hyper["eps"], 1, True, hyper["weight_decay"])]

        def run_fused():
            grads.tensor.copy_(local_grad)
            for lo, hi, i in buckets[:-1]:
                comm.reduce_scatter(grads, lo, hi - lo, scale=1.0 / world, sq_out=tail.sq_slots(i), tag=TAG_BUCKET + i)
            st = state["fused"]
            tail.launch(masters=[st["master"]], exp_avgs=[st["m"]], exp_avg_sqs=[st["v"]], hypers=hyp,
                        pending=[buckets[-1][2]], factor=1.0, max_norm=1.0, clip_eps=0.0)

        results, finals = {}, {}
        mark = clocks.mark() if clocks is not None else 0
        for name, fn in (("nccl", run_nccl), ("symm", run_symm), ("fused", run_fused)):
            reset(name)
            fn()
            torch.cuda.synchronize()
            comm.check_health()
            dist.barrier()
            finals[name] = params.tensor.float().clone()
            reset(name)
            results[name] = timed(fn, iters=10 if mb <= 64 else 5)
        copy_ms = timed(lambda: grads.tensor.copy_(local_grad), iters=10)  # the sweep's own set-up cost, reported
        diff = max(float((finals["nccl"] - finals[k]).abs().max()) for k in ("symm", "fused"))
        d = torch.tensor([diff], device="cuda")
        dist.all_reduce(d, op=dist.ReduceOp.MAX)
        if rank == 0:
            roof_ms = max(n * 36 / (hbm * 1e9), (mb << 20) / 450e9) * 1e3
            net = {k: max(v - copy_ms, 1e-6) for k, v in results.items()}
            print(json.dumps({
                "grad_mb": mb, "params": n, "world": world, "dtype": args.dtype, "buckets": len(buckets),
                "ms": {k: round(v, 4) for k, v in results.items()}, "setup_copy_ms": round(copy_ms, 4),
                "ms_net_of_setup": {k: round(v, 4) for k, v in net.items()},
                "roofline_ms": round(roof_ms, 4), "frac_of_roofline": {k: round(roof_ms / v, 3) for k, v in net.items()},
                "fused_speedup_vs_nccl": round(net["nccl"] / net["fused"], 3),
                "max_param_diff_vs_nccl": float(d.item()), "provider": comm.provider, "nvls": bool(grads.multicast_ptr),
                "clocks": clocks.since(mark),
            }), flush=True)
        del grads, params, tail
        torch.cuda.empty_cache()
        mb *= 4
    if clocks is not None:
        clocks.stop()
    dist.barrier()
    dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
