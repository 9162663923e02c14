#!/usr/bin/env python3
"""Micro-benchmark of the wgmma fused attention vs the materialised PyTorch path.

BERT-base shape by default: B=32, H=12, L=512, D=64, fp16, rel-pos bias [1,H,L,L], dropout 0.1; --D sets the
head dim (softmax scale 1/sqrt(D)).
Times forward and forward+backward with CUDA events (L2 flushed between iterations by writing a
256 MB buffer) and prints one JSON line per variant with achieved TFLOP/s (4*B*H*L*L*D FLOPs forward,
2.5x that backward) and the fraction of the dense 16-bit peak (MEASURED_PEAKS.json if present, else the H100
data sheet).

--causal adds three variants with dropout 0.1: ``causal_dropout`` (no bias), ``causal_bias_mask_dropout`` (the kernels'
causal flag) and ``future_bias_mask_dropout`` (the same bias plus an explicit [L, L] -inf future mask, added once
outside the timed region, in the non-causal kernels).  Their FLOP/s count only the visible (query, key) pairs,
4*B*H*D*sum_i min(i+1, L), for all three, so that the numbers compare the work each path has to do.
"""
import argparse
import json
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def timeit(fn, iters, flush):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    total = 0.0
    for _ in range(iters):
        flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        total += s.elapsed_time(e)
    return total / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=32)
    ap.add_argument("--H", type=int, default=12)
    ap.add_argument("--L", type=int, default=512)
    ap.add_argument("--D", type=int, default=64)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--dtype", default="float16")
    ap.add_argument("--only", default="")
    ap.add_argument("--causal", action="store_true", help="also time the causal variants (FLOPs of visible pairs)")
    args = ap.parse_args()
    from unicore import ops

    assert ops.USE_NATIVE
    dtype = getattr(torch, args.dtype)
    B, H, L, D = args.B, args.H, args.L, args.D
    scale = 1.0 / math.sqrt(D)
    peak = 989.4   # H100 SXM data sheet, dense fp16 / bf16 TFLOP/s (700 W); a measured peak replaces it when present
    try:
        peak = json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")))["bf16_tflops"]
    except Exception:  # noqa: BLE001
        pass
    torch.manual_seed(0)
    qkv = (torch.randn(B, L, 3, H, D, device="cuda") * 0.5).to(dtype).requires_grad_(True)
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    bias = torch.randn(1, H, L, L, device="cuda").to(dtype).requires_grad_(True)
    kpm = torch.zeros(B, L, dtype=torch.bool, device="cuda")
    dout = torch.randn(B, L, H, D, device="cuda").to(dtype)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    dense_flops = 4.0 * B * H * L * L * D
    variants = {
        "plain": dict(bias=None, kpm=None, p=0.0),
        "bias": dict(bias=bias, kpm=None, p=0.0),
        "bias_mask": dict(bias=bias, kpm=kpm, p=0.0),
        "bias_mask_dropout": dict(bias=bias, kpm=kpm, p=0.1),
    }
    if args.causal:
        future = torch.full((L, L), float("-inf"), device="cuda").triu(1)
        future_bias = (bias.detach().float() + future).to(dtype).requires_grad_(True)
        variants.update({
            "causal_dropout": dict(bias=None, kpm=None, p=0.1, causal=True),
            "causal_bias_mask_dropout": dict(bias=bias, kpm=kpm, p=0.1, causal=True),
            "future_bias_mask_dropout": dict(bias=future_bias, kpm=kpm, p=0.1, visible=True),
        })
    for name, cfg in variants.items():
        if args.only and name != args.only:
            continue
        causal = cfg.get("causal", False)
        # visible (query, key) pairs only for the causal variants: sum_i min(i + 1, L) = L (L + 1) / 2
        fwd_flops = 4.0 * B * H * D * L * (L + 1) / 2 if causal or cfg.get("visible") else dense_flops

        def fwd():
            return ops.fused_attention(q, k, v, bias=cfg["bias"], key_padding_mask=cfg["kpm"], dropout_p=cfg["p"],
                                       training=True, scale=scale, causal=causal)

        def fwd_bwd():
            qkv.grad = None
            if cfg["bias"] is not None:
                cfg["bias"].grad = None
            fwd().backward(dout)

        with torch.no_grad():
            t_f = timeit(fwd, args.iters, flush)
        t_fb = timeit(fwd_bwd, args.iters, flush)
        t_b = t_fb - t_f
        print(json.dumps({
            "kernel": "fmha_sm90", "variant": name, "B": B, "H": H, "L": L, "D": D, "dtype": args.dtype,
            "fwd_ms": round(t_f, 4), "bwd_ms": round(t_b, 4),
            "fwd_tflops": round(fwd_flops / t_f / 1e9, 1), "bwd_tflops": round(2.5 * fwd_flops / t_b / 1e9, 1),
            "fwd_frac_of_peak": round(fwd_flops / t_f / 1e9 / peak, 4),
            "bwd_frac_of_peak": round(2.5 * fwd_flops / t_b / 1e9 / peak, 4),
        }), flush=True)
    fwd_flops = dense_flops
    if not args.only:
        # materialised reference path (what the reference framework executes)
        def ref_fwd():
            return ops.attention_reference(q, k, v, bias, kpm, 0.1, True, scale)

        def ref_fwd_bwd():
            qkv.grad = None
            bias.grad = None
            ref_fwd().backward(dout)

        with torch.no_grad():
            t_f = timeit(ref_fwd, max(2, args.iters // 3), flush)
        t_fb = timeit(ref_fwd_bwd, max(2, args.iters // 3), flush)
        t_b = t_fb - t_f
        print(json.dumps({"kernel": "pytorch_materialised", "variant": "bias_mask_dropout", "D": D,
                          "fwd_ms": round(t_f, 4), "bwd_ms": round(t_b, 4),
                          "fwd_tflops": round(fwd_flops / t_f / 1e9, 1),
                          "bwd_tflops": round(2.5 * fwd_flops / t_b / 1e9, 1)}), flush=True)


if __name__ == "__main__":
    main()
