#!/usr/bin/env python3
"""Uni-Mol (SE(3)-invariant molecular transformer) pre-training step benchmark — BASELINE.json config
"Uni-Mol SE(3) Transformer bf16 on 8 GPUs (softmax_dropout + LayerNorm hot path)".

Drives ``examples/unimol`` (arch ``unimol_base``: 15 layers, 512 dim, 64 heads, pair-bias attention, masked
atom-type / coordinate / distance heads) through the public ``Trainer.train_step`` on synthetic molecules
(``--task synthetic_unimol``: random atom types and coordinates, 64..254 atoms, padded to a multiple of 8).
One process per GPU under ``torch.distributed.run``; device-timed, max over ranks, one JSON line.
"""
import argparse
import importlib
import json
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch-size", type=int, default=32)
    ap.add_argument("--precision", default="bf16", choices=["fp16", "bf16"])
    ap.add_argument("--max-atoms", type=int, default=254)
    ap.add_argument("--ddp-backend", default=None)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"],
                    help="reference: the unmodified reference framework from baseline/_ref (BASELINE.md B6)")
    ap.add_argument("--ref-ext", action="store_true", help="reference arm: with its own CUDA extensions (sm_90 build)")
    ap.add_argument("--portable", action="store_true",
                    help="use examples/unimol_portable (public Uni-Core API only; the plug-in both frameworks can load) "
                         "instead of this framework's optimised examples/unimol; implied by --impl reference")
    a = ap.parse_args()
    a.portable = a.portable or a.impl == "reference"
    from op_compare import Clocks
    sys.path.insert(0, REPO)
    import bench as B

    why = B.setup_paths(a.impl, a.ref_ext)
    if why is not None:
        print(json.dumps({"impl": a.impl, "unavailable": why}))
        return 0
    sys.path.insert(0, os.path.join(REPO, "examples"))

    import torch
    import torch.distributed as dist

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local_rank)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group(backend="nccl", init_method="env://", world_size=world, rank=rank)
        dist.all_reduce(torch.zeros(1, device="cuda"))

    importlib.import_module("unimol_portable" if a.portable else "unimol")
    from unicore import options, tasks, utils
    from unicore.trainer import Trainer

    backend = a.ddp_backend or ("b200" if (world > 1 and a.impl == "ours") else "c10d")
    names = ("synthetic_unimol_portable", "unimol_portable", "unimol_portable_base") if a.portable else \
        ("synthetic_unimol", "unimol", "unimol_base")
    flags = [
        "--task", names[0], "--loss", names[1], "--arch", names[2],
        "--synthetic-num-samples", str(a.batch_size * 8), "--synthetic-max-atoms", str(a.max_atoms),
        "--optimizer", "adam", "--adam-betas", "(0.9, 0.99)", "--adam-eps", "1e-6", "--clip-norm", "1.0",
        "--lr", "1e-4", "--lr-scheduler", "polynomial_decay", "--warmup-updates", "100",
        "--total-num-update", "100000", "--max-update", "100000", "--batch-size", str(a.batch_size),
        "--update-freq", "1", "--seed", "1", "--no-save", "--disable-validation", "--log-format", "none",
        "--distributed-world-size", str(world), "--ddp-backend", backend, "--device-id", str(local_rank),
        "--distributed-rank", str(rank), "--" + a.precision,
    ]
    if a.impl == "ours":
        flags.append("--deferred-overflow-check")
    parser = options.get_training_parser()
    args = options.parse_args_and_arch(parser, input_args=flags)
    args.distributed_rank, args.device_id = rank, local_rank
    task = tasks.setup_task(args)
    model = task.build_model(args)
    loss = task.build_loss(args)
    trainer = Trainer(args, task, model, loss)
    trainer._total_train_steps = args.max_update
    task.load_dataset("train")
    ds = task.dataset("train")
    n = a.batch_size
    batches = [ds.collater([ds[(k * n + i) % len(ds)] for i in range(n)]) for k in range(4)]
    batches = [utils.move_to_cuda(b) for b in batches]
    atoms = sum(int(b["net_input"]["src_tokens"].numel()) for b in batches) / len(batches)

    for i in range(a.warmup):
        trainer.train_step([batches[i % 4]])
    torch.cuda.synchronize()
    if world > 1:
        dist.barrier()
    clocks = Clocks() if rank == 0 else None
    mark = clocks.mark() if clocks is not None else 0
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for i in range(a.steps):
        trainer.train_step([batches[i % 4]])
    e.record()
    torch.cuda.synchronize()
    ms = torch.tensor([s.elapsed_time(e) / a.steps], device="cuda", dtype=torch.float64)
    if world > 1:
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
    if rank == 0:
        t = float(ms.item())
        nparams = sum(p.numel() for p in model.parameters())
        print(json.dumps({
            "metric": "Uni-Mol pre-training throughput (molecules/s, whole job, device-timed, max over ranks)",
            "value": a.batch_size * world / t * 1e3, "unit": "molecules/s", "n_gpus": world, "ms_per_step": t,
            "steps": a.steps, "warmup": a.warmup, "dtype": a.precision, "data": "synthetic molecules",
            "impl": a.impl, "plugin": "examples/unimol_portable" if a.portable else "examples/unimol",
            "reference_cuda_ext": bool(a.ref_ext) if a.impl == "reference" else None,
            "config": {"model": "unimol_base", "params": nparams, "per_gpu_batch": a.batch_size,
                       "padded_atoms_per_batch": atoms, "ddp_backend": backend},
            "clocks": clocks.since(mark) if clocks is not None else None,
        }))
    if clocks is not None:
        clocks.stop()
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
