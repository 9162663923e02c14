#!/usr/bin/env python3
"""What deterministic mode (``torch.use_deterministic_algorithms(True)``, ``--deterministic``) costs.

In one process, times each workload with the switch off and on, alternating the two and warmed up, with CUDA events
(median over --rounds rounds of --iters calls each), and checks that the two modes agree: bitwise where only the
order of a reduction could change the result the other way round, else within the fp32-reorder bound of the 16-bit
output.  Workloads:
- fused attention backward at BERT-base (B 32, H 12, L 512, D 64, shared bias, padding, dropout 0.1), causal at
  (8, 12, 2048, 64), D = 128 at (32, 8, 512, 128), and Uni-Mol's logits mode (B 32, H 64, L 256, D 8, bf16, per-batch
  bias, incoming dz).  Deterministic mode orders the dQ reductions of the key tiles; the 8 key tiles per chain at
  L = 512 are where the serialisation could show.
- the embedding backward of BERT's 30522 x 768 table over 16k tokens (sort + ordered runs instead of red-adds)
- ``gbf_bwd`` at a Uni-Mol pair shape (32 x 128 x 128 pairs, K = 128, 900 edge types)
- a whole BERT-base ``train_step`` (fp16, batch 16 x 512)

CUBLAS_WORKSPACE_CONFIG=:4096:8 is set for both modes (the deterministic one needs it before cuBLAS starts).
Prints the card name and power limit, then one JSON line per workload.
"""
import argparse
import json
import math
import os
import subprocess
import sys

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")

import torch  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

UNIT = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}


def set_mode(on):
    torch.use_deterministic_algorithms(on)


def time_ms(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def compare_modes(name, fn, iters, rounds, check):
    res = {}
    for on in (False, True):   # warm-up of both modes
        set_mode(on)
        res[on] = fn()
        fn()
    torch.cuda.synchronize()
    times = {False: [], True: []}
    for r in range(rounds):
        for on in ((False, True) if r % 2 == 0 else (True, False)):
            set_mode(on)
            times[on].append(time_ms(fn, iters))
    set_mode(False)
    med = {on: sorted(t)[len(t) // 2] for on, t in times.items()}
    out = {"workload": name, "off_ms": round(med[False], 4), "on_ms": round(med[True], 4),
           "ratio": round(med[True] / med[False], 3), "agree": check(res[False], res[True])}
    print(json.dumps(out), flush=True)
    return out


def within_reorder(a, b, dtype):
    a, b = a.double(), b.double()
    bound = 2 * UNIT[dtype] * b.abs() + 2.0 ** -18 * b.abs().max()
    return bool(((a - b).abs() <= bound).all())


def attention(nat, B, H, L, D, dtype, bias_mode, causal, logits, iters, rounds):
    g = torch.Generator(device="cuda").manual_seed(0)
    q = (torch.randn(B, L, H, D, device="cuda", generator=g) * 0.6).to(dtype)
    k = (torch.randn(B, L, H, D, device="cuda", generator=g) * 0.6).to(dtype)
    v = torch.randn(B, L, H, D, device="cuda", generator=g).to(dtype)
    bias = None if bias_mode == "none" else torch.randn(B if bias_mode == "batch" else 1, H, L, L, device="cuda",
                                                        generator=g).to(dtype)
    kpm = torch.zeros(B, L, dtype=torch.bool, device="cuda")
    kpm[:, L - L // 8:] = True
    scale, p = 1.0 / math.sqrt(D), 0.1
    dz = None
    if logits:
        out, lse, bits, z = nat.fmha_fwd_logits(q, k, v, bias, kpm, p, scale)
        dz = (torch.randn(z.shape, device="cuda", generator=g) * 0.1).to(dtype)
    else:
        out, lse, bits = nat.fmha_fwd(q, k, v, bias, kpm, p, scale, causal=causal)
    dout = torch.randn(B, L, H, D, device="cuda", generator=g).to(dtype)

    def run():
        return nat.fmha_bwd(dout, q, k, v, out, lse, bias, kpm, p, scale, bits, bias is not None, False, dlogits=dz,
                            causal=causal)

    def check(off, on):
        same = all((a is None and b is None) or torch.equal(a, b) for a, b in zip(off[1:], on[1:]))
        return same and within_reorder(on[0], off[0], dtype)

    name = "fmha_bwd B{} H{} L{} D{} {}{}{}".format(B, H, L, D, str(dtype).split(".")[-1],
                                                   " causal" if causal else "", " logits" if logits else "")
    r = compare_modes(name, run, iters, rounds, check)
    print(json.dumps({"workload": name, "fmha_det_timeouts": nat.fmha_det_timeouts()}), flush=True)
    return r


def embedding(nat, iters, rounds):
    V, C, R = 30522, 768, 16384
    g = torch.Generator(device="cuda").manual_seed(1)
    tok = torch.randint(0, V, (R,), device="cuda", generator=g)
    tok[torch.rand(R, device="cuda", generator=g) < 0.15] = 103   # [MASK]: ~2.5k rows of one id
    dy = torch.randn(R, C, device="cuda", generator=g).half()
    scratch, touched = torch.zeros(V, C, device="cuda"), torch.zeros(V, dtype=torch.uint8, device="cuda")
    grad = torch.zeros(V, C, device="cuda", dtype=torch.half)

    def run():
        grad.zero_()
        nat.embedding_bwd(dy, tok, 0, scratch, touched, grad, False)
        return grad.clone()

    return compare_modes("embedding_bwd 30522x768, 16k tokens", run, iters, rounds,
                         lambda a, b: within_reorder(b, a, torch.float16))


def gaussian(nat, iters, rounds):
    B, L, K, E = 32, 128, 128, 900
    g = torch.Generator(device="cuda").manual_seed(2)
    dist = (torch.rand(B, L, L, device="cuda", generator=g) * 6).half()
    edge = torch.randint(0, E, (B, L, L), device="cuda", generator=g)
    mul_w = (1 + 0.2 * torch.randn(E, 1, device="cuda", generator=g)).half()
    bias_w = (0.2 * torch.randn(E, 1, device="cuda", generator=g)).half()
    means = (torch.rand(1, K, device="cuda", generator=g) * 3).half()
    stds = (torch.rand(1, K, device="cuda", generator=g) * 3 + 0.5).half()
    dy = torch.randn(B, L, L, K, device="cuda", generator=g).half()

    def run():
        return nat.gbf_bwd(dy, dist, edge, mul_w, bias_w, means, stds)

    def check(off, on):   # fp32 outputs: relative to the largest magnitude of each
        return all(bool(((a - b).abs() <= 1e-5 * b.abs().max()).all()) for a, b in zip(on, off))

    return compare_modes("gbf_bwd 32x128x128 K128 E900", run, iters, rounds, check)


def bert_step(iters, rounds):
    import importlib

    sys.path.insert(0, os.path.join(ROOT, "examples"))
    importlib.import_module("bert")
    from unicore import options, tasks
    from unicore.trainer import Trainer

    parser = options.get_training_parser()
    args = options.parse_args_and_arch(parser, input_args=[
        "--task", "synthetic_mlm", "--loss", "masked_lm", "--arch", "bert_base", "--synthetic-seq-len", "512",
        "--max-seq-len", "512", "--optimizer", "adam", "--lr", "1e-5", "--lr-scheduler", "fixed", "--batch-size", "16",
        "--fp16", "--clip-norm", "1.0", "--distributed-world-size", "1", "--no-save", "--disable-validation",
        "--log-format", "none", "--max-update", "100000"])
    task = tasks.setup_task(args)
    trainer = Trainer(args, task, task.build_model(args), task.build_loss(args))
    task.load_dataset("train")
    ds = task.dataset("train")
    batch = ds.collater([ds[i] for i in range(16)])

    def run():
        return trainer.train_step([batch])

    # the parameters move every step, so the two modes' outputs are not comparable: only finiteness is checked
    return compare_modes("BERT-base train_step fp16 16x512", run, iters, rounds,
                         lambda a, b: a is not None and b is not None and float(b["loss"]) == float(b["loss"]))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--skip-train-step", action="store_true")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the GPU"
    from unicore import ops

    assert ops.USE_NATIVE
    nat = ops.native()
    print(json.dumps({"card": card()}), flush=True)
    attention(nat, 32, 12, 512, 64, torch.float16, "shared", False, False, a.iters, a.rounds)
    attention(nat, 8, 12, 2048, 64, torch.float16, "none", True, False, a.iters, a.rounds)
    attention(nat, 32, 8, 512, 128, torch.float16, "shared", False, False, a.iters, a.rounds)
    attention(nat, 32, 64, 256, 8, torch.bfloat16, "batch", False, True, a.iters, a.rounds)
    embedding(nat, a.iters, a.rounds)
    gaussian(nat, a.iters, a.rounds)
    if not a.skip_train_step:
        bert_step(max(2, a.iters // 4), a.rounds)


if __name__ == "__main__":
    main()
