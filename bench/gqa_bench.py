#!/usr/bin/env python3
"""Grouped-query attention: what sharing key / value heads saves in the decode step and in training.

Decode arm: device time per call of ``ops.attention_with_kv_cache`` (one query per (b, h), H = 32 query heads, D = 128,
fp16, appending the new key / value, every sequence at the same visible length n) for H_kv in {32, 8, 1}, at B in
{1, 8, 64} and n in {1024, 4096, 16384}.  The K + V bytes a step has to read are 2 * B * n * H_kv * D * 2 (from the
shapes: the cache holds each row once however many query heads share it); the achieved bandwidth is those bytes over
the kernel time, against the H100 SXM data-sheet 3.35 TB/s.

Training arm: forward + backward of ``ops.fused_attention`` at B = 8, L = 2048, H = 32, D = 128, fp16, no bias or
dropout, for the same H_kv values.  ``attn_tflops`` counts the 4 * B * H * L^2 * D forward and 10 * B * H * L^2 * D
forward + backward flops (two and five L x L x D products per query head), which do not depend on H_kv.

CUDA events, every arm warmed up, the arms of one shape alternating, median of --rounds rounds of --iters calls.
Prints the card name and power limit, then one JSON line per measurement.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "bench"))

from decode_bench import HBM_BYTES_PER_S, alternate, card  # noqa: E402

H, D = 32, 128
KV_HEADS = [32, 8, 1]


def decode_arm(ops, B, n, iters, rounds):
    g = torch.Generator(device="cuda").manual_seed(0)
    arms, kv_bytes = {}, {}
    for H_kv in KV_HEADS:
        k = torch.randn(B, n, H_kv, D, device="cuda", generator=g).half()
        v = torch.randn(B, n, H_kv, D, device="cuda", generator=g).half()
        q = torch.randn(B, 1, H, D, device="cuda", generator=g).half()
        kn = torch.randn(B, 1, H_kv, D, device="cuda", generator=g).half()
        vn = torch.randn(B, 1, H_kv, D, device="cuda", generator=g).half()
        seqlens = torch.full((B,), n - 1, dtype=torch.int32, device="cuda")   # the appended row makes n visible keys
        arms[H_kv] = (lambda q=q, k=k, v=v, s=seqlens, kn=kn, vn=vn:
                      ops.attention_with_kv_cache(q, k, v, s, n - 1, k_new=kn, v_new=vn))
        kv_bytes[H_kv] = 2 * B * n * H_kv * D * 2
    with torch.no_grad():
        med = alternate(arms, iters, rounds)
    for H_kv in KV_HEADS:
        bw = kv_bytes[H_kv] / (med[H_kv] * 1e-3)
        print(json.dumps({"arm": "decode", "B": B, "n": n, "H": H, "H_kv": H_kv, "D": D,
                          "splits": ops.native().fmha_decode_num_splits(B, H, n), "us": round(med[H_kv] * 1e3, 2),
                          "kv_bytes": kv_bytes[H_kv], "GBps": round(bw / 1e9, 1),
                          "of_3.35TBps": round(bw / HBM_BYTES_PER_S, 3),
                          "speedup_vs_mha": round(med[KV_HEADS[0]] / med[H_kv], 2)}), flush=True)


def train_arm(ops, B, L, iters, rounds):
    g = torch.Generator(device="cuda").manual_seed(1)
    arms = {}
    for H_kv in KV_HEADS:
        q = torch.randn(B, L, H, D, device="cuda", generator=g).half().requires_grad_()
        k = torch.randn(B, L, H_kv, D, device="cuda", generator=g).half().requires_grad_()
        v = torch.randn(B, L, H_kv, D, device="cuda", generator=g).half().requires_grad_()
        dout = torch.randn(B, L, H, D, device="cuda", generator=g).half()

        def step(q=q, k=k, v=v, dout=dout):
            out = ops.fused_attention(q, k, v, dropout_p=0.0)
            torch.autograd.grad(out, (q, k, v), dout)

        arms[H_kv] = step
    med = alternate(arms, iters, rounds)
    flops = 10 * B * H * L * L * D
    for H_kv in KV_HEADS:
        print(json.dumps({"arm": "train_fwd_bwd", "B": B, "L": L, "H": H, "H_kv": H_kv, "D": D,
                          "ms": round(med[H_kv], 3), "attn_tflops": round(flops / (med[H_kv] * 1e-3) / 1e12, 1),
                          "speedup_vs_mha": round(med[KV_HEADS[0]] / med[H_kv], 2)}), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--batch", type=int, nargs="*", default=[1, 8, 64])
    ap.add_argument("--lengths", type=int, nargs="*", default=[1024, 4096, 16384])
    ap.add_argument("--skip-train", action="store_true")
    args = ap.parse_args()
    from unicore import ops

    assert ops.USE_NATIVE, "the native kernels are not active"
    print("card:", card(), flush=True)
    for B in args.batch:
        for n in args.lengths:
            decode_arm(ops, B, n, args.iters, args.rounds)
            torch.cuda.empty_cache()
    if not args.skip_train:
        train_arm(ops, 8, 2048, max(2, args.iters // 4), args.rounds)


if __name__ == "__main__":
    main()
