"""Packed (varlen) vs padded batches of the same sentences: fused attention forward + backward, a BERT-base encoder
forward + backward, and a whole BERT-base masked-LM ``Trainer.train_step`` (fp16, Adam).

Lengths are seeded: uniform on [64, L], and a skewed mix (most sentences short, a few at L).  Both arms run the same
sentences and alternate within one process, so that clock and neighbour noise fall on both.  The attention rate counts
the valid (query, key) pairs only: 4 * H * D * sum(len_b^2) FLOPs forward, 2.5x that for the backward.
Usage: python bench/varlen_bench.py [--iters 20] [--rounds 5]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from unicore import ops  # noqa: E402
from unicore.modules.transformer import TransformerEncoder  # noqa: E402


def lengths(kind, B, L, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "uniform":
        return torch.randint(64, L + 1, (B,), generator=g).tolist()
    short = torch.randint(16, 129, (B,), generator=g)   # skewed: 3/4 short, 1/4 at L
    return [L if i % 4 == 0 else int(x) for i, x in enumerate(short)]


def cu_of(lens):
    return torch.tensor([0] + lens, device="cuda").cumsum(0).to(torch.int32)


def scatter(x, lens, L):
    out = x.new_zeros(len(lens), L, *x.shape[1:])
    s = 0
    for b, n in enumerate(lens):
        out[b, :n] = x[s:s + n]
        s += n
    return out


def timed(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def alternate(arms, iters, rounds):
    for fn in arms.values():   # warm-up of every shape
        fn()
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            times[k].append(timed(fn, iters))
    return {k: sorted(v)[len(v) // 2] for k, v in times.items()}


def attention_case(kind, dtype, B, L, H, D, iters, rounds):
    lens = lengths(kind, B, L, 0)
    N = sum(lens)
    qkv = torch.randn(N, 3 * H, D, device="cuda", dtype=dtype, requires_grad=True)
    cu = cu_of(lens)
    qkvp = scatter(qkv.detach(), lens, L).view(B, L, 3, H, D).requires_grad_(True)
    kpm = torch.arange(L, device="cuda")[None, :] >= torch.tensor(lens, device="cuda")[:, None]
    do = torch.randn(N, H, D, device="cuda", dtype=dtype)
    dop = scatter(do, lens, L)

    def packed():
        ops.fused_attention_varlen_qkvpacked(qkv, cu, L, num_kv_heads=H).backward(do)

    def padded():
        ops.fused_attention_qkvpacked(qkvp, key_padding_mask=kpm).backward(dop)

    t = alternate({"packed": packed, "padded": padded}, iters, rounds)
    flops = 4 * H * D * sum(n * n for n in lens) * 3.5   # forward + backward (2.5x), valid pairs only
    return {"case": "attention", "lengths": kind, "dtype": str(dtype).split(".")[-1], "B": B, "L": L, "H": H, "D": D,
            "real_tokens": N, "packed_ms": round(t["packed"], 3), "padded_ms": round(t["padded"], 3),
            "speedup": round(t["padded"] / t["packed"], 3),
            "packed_tflops": round(flops / t["packed"] * 1e-9, 1), "padded_tflops": round(flops / t["padded"] * 1e-9, 1)}


def encoder_case(kind, dtype, B, L, iters, rounds):
    lens = lengths(kind, B, L, 1)
    N = sum(lens)
    torch.manual_seed(0)
    enc = TransformerEncoder(encoder_layers=12, embed_dim=768, ffn_embed_dim=3072, attention_heads=12,
                             max_seq_len=L, post_ln=True).cuda().to(dtype)
    emb = torch.randn(N, 768, device="cuda", dtype=dtype, requires_grad=True)
    embp = scatter(emb.detach(), lens, L).requires_grad_(True)
    kpm = torch.arange(L, device="cuda")[None, :] >= torch.tensor(lens, device="cuda")[:, None]
    cu = cu_of(lens)

    def packed():
        enc(emb, cu_seqlens=cu, max_seqlen=L).float().square().mean().backward()

    def padded():
        enc(embp, padding_mask=kpm).float().square().mean().backward()

    t = alternate({"packed": packed, "padded": padded}, iters, rounds)
    # the same sentences, dropout off: the two arms agree at the real rows
    enc.eval()
    with torch.no_grad():
        y = enc(emb, cu_seqlens=cu, max_seqlen=L)
        yp = enc(embp, padding_mask=kpm)
        yp = torch.cat([yp[b, :n] for b, n in enumerate(lens)])
        rel = ((y.double() - yp.double()).norm() / yp.double().norm()).item()
    return {"case": "bert_base_encoder_fwd_bwd", "lengths": kind, "dtype": str(dtype).split(".")[-1], "B": B, "L": L,
            "real_tokens": N, "packed_ms": round(t["packed"], 3), "padded_ms": round(t["padded"], 3),
            "speedup": round(t["padded"] / t["packed"], 3), "packed_samples_per_s": round(B / t["packed"] * 1e3, 1),
            "padded_samples_per_s": round(B / t["padded"] * 1e3, 1),
            "packed_real_tokens_per_s": round(N / t["packed"] * 1e3), "padded_real_tokens_per_s":
            round(N / t["padded"] * 1e3), "eval_output_rel_diff": rel}


def trainer_case(kind, B, L, iters, rounds):
    """BERT-base (12 layers) ``Trainer.train_step`` on one padded batch and on the same sentences packed.  The losses
    of the two batches are compared first, with dropout off (eval mode) on the same weights."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, os.path.join(root, "examples"))
    import importlib

    importlib.import_module("bert")
    from unicore import options, tasks, utils
    from unicore.trainer import Trainer

    args = options.parse_args_and_arch(options.get_training_parser(), input_args=[
        "--task", "synthetic_mlm", "--loss", "masked_lm", "--arch", "bert_base", "--synthetic-vocab-size", "30522",
        "--synthetic-seq-len", str(L), "--max-seq-len", str(L), "--optimizer", "adam", "--lr", "1e-4",
        "--lr-scheduler", "fixed", "--max-update", "100000", "--batch-size", str(B), "--fp16", "--clip-norm", "1.0",
        "--distributed-world-size", "1", "--no-save", "--disable-validation", "--log-format", "none", "--seed", "1",
    ])
    torch.manual_seed(0)
    task = tasks.setup_task(args)
    model = task.build_model(args)
    trainer = Trainer(args, task, model, task.build_loss(args))
    trainer._total_train_steps = args.max_update
    task.load_dataset("train")
    ds = task.dataset("train")
    padded = ds.collater([ds[i] for i in range(B)])
    pad = task.dictionary.pad()
    lens = lengths(kind, B, L, 2)
    for b, n in enumerate(lens):   # right-pad the sentences to their lengths
        padded["net_input"]["src_tokens"][b, n:] = pad
        padded["target"][b, n:] = pad
    src, tgt = padded["net_input"]["src_tokens"], padded["target"]
    packed = {"net_input": {"src_tokens": torch.cat([src[b, :n] for b, n in enumerate(lens)]),
                            "cu_seqlens": torch.tensor([0] + lens).cumsum(0).to(torch.int32), "max_seqlen": L},
              "target": torch.cat([tgt[b, :n] for b, n in enumerate(lens)])}
    trainer.model.eval()
    with torch.no_grad():
        losses = {k: float(trainer.loss(trainer.model, utils.move_to_cuda(v))[0]) for k, v in
                  (("packed", packed), ("padded", padded))}
    trainer.model.train()
    arms = {"packed": lambda: trainer.train_step([packed]), "padded": lambda: trainer.train_step([padded])}
    t = alternate(arms, iters, rounds)
    N = sum(lens)
    return {"case": "bert_base_trainer_train_step", "lengths": kind, "dtype": "float16", "B": B, "L": L,
            "real_tokens": N, "packed_ms": round(t["packed"], 3), "padded_ms": round(t["padded"], 3),
            "speedup": round(t["padded"] / t["packed"], 3), "packed_samples_per_s": round(B / t["packed"] * 1e3, 1),
            "padded_samples_per_s": round(B / t["padded"] * 1e3, 1),
            "packed_real_tokens_per_s": round(N / t["packed"] * 1e3), "padded_real_tokens_per_s":
            round(N / t["padded"] * 1e3), "eval_loss_packed": losses["packed"], "eval_loss_padded": losses["padded"],
            "eval_loss_rel_diff": abs(losses["packed"] - losses["padded"]) / abs(losses["padded"])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("varlen_bench needs a GPU")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": card}))
    for dtype in (torch.float16, torch.bfloat16):
        for kind in ("uniform", "skewed"):
            print(json.dumps(attention_case(kind, dtype, 32, 512, 12, 64, args.iters, args.rounds)), flush=True)
    for kind in ("uniform", "skewed"):
        print(json.dumps(encoder_case(kind, torch.float16, 32, 512, max(args.iters // 4, 3), args.rounds)), flush=True)
    for kind in ("uniform", "skewed"):
        print(json.dumps(trainer_case(kind, 32, 512, max(args.iters // 4, 3), args.rounds)), flush=True)


if __name__ == "__main__":
    main()
