#!/usr/bin/env python3
"""Loss trajectory of N optimizer updates of a tiny BERT, fp32 on the CPU, for either implementation.

    python tools/loss_parity.py --impl ours      --init /tmp/init.pt --steps 6
    python tools/loss_parity.py --impl reference --init /tmp/init.pt --steps 6

The first arm that runs creates ``--init`` (the model's initial ``state_dict``); the other one loads it, so both
start from identical weights (the parameter names are the same by design).  Dropout is off, the batches are the
deterministic synthetic ones of ``bench.py``, the optimizer is Adam with clipping and a polynomial schedule.  One
process per arm: the reference lives in ``baseline/_ref`` under the same package name and cannot share an
interpreter with this repo.  Prints ``{"impl": ..., "losses": [...]}`` (the logged loss of every update).
"""
import argparse
import json
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import bench  # noqa: E402  (path / task helpers shared with the benchmark)


def zipf_batches(n, bsz, seq_len, vocab, pad_idx, mask_idx, special, seed):
    import numpy as np
    import torch

    rng = np.random.RandomState(seed)
    allowed = np.setdiff1d(np.arange(vocab), np.asarray(sorted(special)))
    prob = 1.0 / (np.arange(len(allowed)) + 10.0)
    prob /= prob.sum()
    n_mask = max(1, int(round(0.15 * seq_len)))
    out = []
    for _ in range(n):
        tokens = allowed[rng.choice(len(allowed), size=(bsz, seq_len), p=prob)]
        target = np.full((bsz, seq_len), pad_idx, dtype=np.int64)
        src = tokens.copy()
        for b in range(bsz):
            pos = rng.choice(seq_len, n_mask, replace=False)
            target[b, pos] = tokens[b, pos]
            src[b, pos] = mask_idx
        out.append({"net_input": {"src_tokens": torch.from_numpy(src.astype(np.int64))}, "target": torch.from_numpy(target)})
    return out


def gpu_main(a):
    """Loss curve of the flagship configuration on one GPU."""
    why = bench.setup_paths(a.impl)
    if why is not None:
        print(json.dumps({"impl": a.impl, "unavailable": why}))
        return 0
    import torch

    if a.impl == "reference":
        import bert  # noqa: F401  reference examples/bert
    else:
        import importlib

        sys.path.insert(0, os.path.join(REPO, "examples"))
        importlib.import_module("bert")
    from unicore import options, tasks
    from unicore.trainer import Trainer

    bench.register_bench_task(a.impl)
    flags = [
        "--task", "bench_mlm", "--loss", "masked_lm", "--arch", "bert_base", "--optimizer", "adam",
        "--adam-betas", "(0.9, 0.98)", "--adam-eps", "1e-6", "--clip-norm", "1.0", "--lr-scheduler", "polynomial_decay",
        "--lr", a.lr, "--warmup-updates", "10", "--total-num-update", "10000", "--max-update", "10000",
        "--batch-size", "32", "--seed", "1", "--num-workers", "0", "--log-format", "none", "--disable-validation",
        "--no-save", "--max-seq-len", "512", "--distributed-world-size", "1", "--fp16", "--fp16-init-scale", "4",
        "--fp16-scale-window", "256",
    ]
    if a.dropout is not None:
        for name in ("--dropout", "--emb-dropout", "--attention-dropout", "--activation-dropout", "--pooler-dropout"):
            flags += [name, str(a.dropout)]
    args = options.parse_args_and_arch(options.get_training_parser(), input_args=flags)
    torch.manual_seed(args.seed)
    torch.cuda.set_device(0)
    task = tasks.setup_task(args)
    model = task.build_model(args)
    if os.path.exists(a.init):
        model.load_state_dict(torch.load(a.init, map_location="cpu"))
    else:
        torch.save(model.state_dict(), a.init)
    trainer = Trainer(args, task, model, task.build_loss(args))
    trainer._total_train_steps = args.max_update
    d = task.dictionary
    # Zipf-distributed tokens: there is a unigram distribution to learn, so the curve falls from ln(V) = 10.3 towards the
    # entropy of the distribution and a divergence between the two implementations would show
    batches = zipf_batches(16, 32, 512, len(d), d.pad(), task.mask_idx,
                           special=[d.pad(), d.unk(), d.bos(), d.eos(), task.mask_idx], seed=123)
    batches = [{"net_input": {"src_tokens": b["net_input"]["src_tokens"].cuda()}, "target": b["target"].cuda()} for b in batches]
    losses = []
    for i in range(a.steps):
        out = trainer.train_step([batches[i % len(batches)]])
        v = out.get("loss", None) if out is not None else None
        losses.append(None if v is None else round(float(v), 4))   # None: update skipped (fp16 overflow)
    line = json.dumps({"impl": a.impl, "model": "bert_base", "precision": "fp16", "batch": [32, 512],
                       "dropout": a.dropout if a.dropout is not None else 0.1, "lr": float(a.lr), "steps": a.steps,
                       "device": torch.cuda.get_device_name(0), "losses": losses})
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")
    return 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--impl", choices=["ours", "reference"], required=True)
    ap.add_argument("--init", required=True)
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--gpu", action="store_true",
                    help="full BERT-base, fp16 mixed precision, batch 32 x 512 on cuda:0 (the bench.py configuration) "
                         "instead of the tiny fp32 CPU model")
    ap.add_argument("--dropout", type=float, default=None, help="--gpu only: all dropout rates (default: the model's 0.1)")
    ap.add_argument("--lr", default="1e-4", help="--gpu only")
    ap.add_argument("--out", default="", help="also write the JSON line to this file")
    a = ap.parse_args()
    if a.gpu:
        return gpu_main(a)
    why = bench.setup_paths(a.impl)
    if why is not None:
        print(json.dumps({"impl": a.impl, "unavailable": why}))
        return 0
    import torch

    if a.impl == "reference":
        import bert  # noqa: F401  reference examples/bert
    else:
        import importlib

        sys.path.insert(0, os.path.join(REPO, "examples"))
        importlib.import_module("bert")
    from unicore import options, tasks
    from unicore.trainer import Trainer

    bench.register_bench_task(a.impl)
    flags = [
        "--task", "bench_mlm", "--bench-vocab", "512", "--loss", "masked_lm", "--arch", "bert_base",
        "--encoder-layers", "2", "--encoder-embed-dim", "64", "--encoder-ffn-embed-dim", "128",
        "--encoder-attention-heads", "4", "--max-seq-len", "32", "--dropout", "0.0", "--emb-dropout", "0.0",
        "--attention-dropout", "0.0", "--activation-dropout", "0.0", "--pooler-dropout", "0.0",
        "--optimizer", "adam", "--adam-betas", "(0.9, 0.98)", "--adam-eps", "1e-6", "--weight-decay", "0.01",
        "--clip-norm", "1.0", "--lr-scheduler", "polynomial_decay", "--lr", "1e-3", "--warmup-updates", "2",
        "--total-num-update", "20", "--max-update", "20", "--batch-size", "4", "--seed", "1", "--num-workers", "0",
        "--log-format", "none", "--disable-validation", "--no-save", "--distributed-world-size", "1", "--cpu",
    ]
    args = options.parse_args_and_arch(options.get_training_parser(), input_args=flags)
    torch.manual_seed(args.seed)
    task = tasks.setup_task(args)
    model = task.build_model(args)
    if os.path.exists(a.init):
        model.load_state_dict(torch.load(a.init, map_location="cpu"))
    else:
        torch.save(model.state_dict(), a.init)
    trainer = Trainer(args, task, model, task.build_loss(args))
    trainer._total_train_steps = args.max_update
    d = task.dictionary
    batches = bench.make_batches(4, 4, 24, len(d), d.pad(), task.mask_idx,
                                 special=[d.pad(), d.unk(), d.bos(), d.eos(), task.mask_idx], seed=99)
    losses = []
    for i in range(a.steps):
        out = trainer.train_step([batches[i % len(batches)]])
        losses.append(float(out["loss"]))  # what the trainer logs: bits per masked token, 3 decimals
    print(json.dumps({"impl": a.impl, "losses": losses}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
