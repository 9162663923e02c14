#!/usr/bin/env python3
"""All-reduce sweep: hand-written NVLink kernels (one-shot / two-shot / NVLS) vs NCCL.

Launch:  python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 \
             --master-port 29531 bench/allreduce_sweep.py [--check] [--max-mb 1024]

For every size (1 KB .. --max-mb, x4 steps) and dtype it verifies the result against
``torch.distributed.all_reduce`` (NCCL) on identical inputs, then times both with CUDA events
(max over ranks) and reports bus bandwidth ``bytes * 2(N-1)/N / t`` (BASELINE.md B3 / config 5) next to the NVLink
roofline (H100 SXM NVLink 4: 450 GB/s per direction nominal).  Every line
carries the SM clock / throttle record sampled while it was measured.  Rank 0 prints one JSON object per line.
"""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

NVLINK_GBS = 450.0   # H100 SXM, NVLink 4: 18 links, 450 GB/s per direction (data sheet)

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from op_compare import Clocks  # noqa: E402


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
    ap.add_argument("--max-mb", type=int, default=1024)
    ap.add_argument("--check", action="store_true")
    ap.add_argument("--stress", action="store_true", help="random per-rank delays before every collective")
    ap.add_argument("--dtypes", default="float16,bfloat16,float32")
    args = ap.parse_args()
    rank = int(os.environ["RANK"])
    world = int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
    dist.init_process_group("nccl", init_method="env://")
    dist.all_reduce(torch.zeros(1, device="cuda"))

    from unicore_b200.parallel.symm_dp import SymmAllReduce, symm_available

    assert symm_available(), "symmetric memory / native kernels unavailable"
    red = SymmAllReduce()
    algos = {"oneshot": 1, "twoshot": 2}
    failures = 0
    clocks = Clocks() if rank == 0 else None
    for dname in args.dtypes.split(","):
        dtype = getattr(torch, dname)
        max_elems = args.max_mb * 1024 * 1024 // torch.empty(0, dtype=dtype).element_size()
        buf = red.allocate(max_elems, dtype)
        if buf.multicast_ptr:
            algos["nvls"] = 3
        nbytes = 1024
        while nbytes <= args.max_mb * 1024 * 1024:
            n = nbytes // buf.tensor.element_size()
            torch.manual_seed(1234 + rank)
            src = (torch.randn(n, device="cuda") * 0.5).to(dtype)
            ref = src.clone()
            dist.all_reduce(ref)
            row = {"bytes": nbytes, "dtype": dname, "world": world, "provider": red.comm.provider}
            mark = clocks.mark() if clocks is not None else 0
            for name, algo in algos.items():
                if name == "oneshot" and nbytes > 8 * 1024 * 1024:
                    continue
                view = buf.tensor[:n]
                view.copy_(src)
                torch.cuda.synchronize()
                dist.barrier()
                slots = red.sq_slots()
                if args.stress:  # skew the ranks: the flag protocol must tolerate any arrival order
                    torch.cuda._sleep(int(torch.randint(0, 2_000_000, (1,)).item()))
                red(buf, 0, n, scale=1.0, algo=algo, sq_out=slots)
                torch.cuda.synchronize()
                red.comm.check_health()
                if args.check:
                    err = (view.float() - ref.float()).abs().max().item()
                    denom = max(1.0, ref.float().abs().max().item())
                    ok = err / denom < {torch.float32: 1e-6, torch.float16: 4e-3, torch.bfloat16: 1.6e-2}[dtype]  # one rounding step
                    # the kernels also store |result|^2 of each rank's slice per CTA: all slots of all ranks add up to it
                    sq = slots.double().sum().reshape(1)
                    dist.all_reduce(sq)
                    want = ref.float().pow(2).sum().item()
                    ok = ok and abs(sq.item() - want) <= (8e-3 if dtype == torch.bfloat16 else 2e-3) * max(want, 1e-6)
                    allsame = view.clone()
                    dist.broadcast(allsame, src=0)
                    identical = bool(torch.equal(allsame, view))
                    ok_t = torch.tensor([int(ok and identical)], device="cuda")
                    dist.all_reduce(ok_t, op=dist.ReduceOp.MIN)
                    row[name + "_ok"] = bool(ok_t.item())
                    failures += 0 if ok_t.item() else 1
                iters = 50 if nbytes <= 1 << 20 else (20 if nbytes <= 64 << 20 else 8)
                ms = timed(lambda: red(buf, 0, n, scale=1.0, algo=algo), iters)
                row[name + "_us"] = round(ms * 1e3, 2)
                row[name + "_busbw_GBs"] = round(nbytes * 2 * (world - 1) / world / (ms * 1e-3) / 1e9, 2)
            work = src.clone()
            ms = timed(lambda: dist.all_reduce(work), 50 if nbytes <= 1 << 20 else 10)
            row["nccl_us"] = round(ms * 1e3, 2)
            row["nccl_busbw_GBs"] = round(nbytes * 2 * (world - 1) / world / (ms * 1e-3) / 1e9, 2)
            best = max(row.get(k + "_busbw_GBs", 0.0) for k in algos)
            row["best_frac_of_nvlink"] = round(best / NVLINK_GBS, 3)
            if clocks is not None:
                row["clocks"] = clocks.since(mark)
            if rank == 0:
                print(json.dumps(row), flush=True)
            nbytes *= 4
    if clocks is not None:
        clocks.stop()
    if rank == 0:
        print(json.dumps({"summary": "allreduce_sweep", "failures": failures, "world": world}))
    dist.barrier()
    dist.destroy_process_group()
    return 1 if failures else 0


if __name__ == "__main__":
    sys.exit(main())
