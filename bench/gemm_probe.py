#!/usr/bin/env python3
"""cuBLAS settings probe for the GEMM shapes of one BERT-base training step (16384 tokens, fp16 / bf16).

A large share of the step is library GEMMs; this script times every distinct
(M, N, K, layout) of forward, dgrad and wgrad under a few library settings so that a better default can be chosen
with one short GPU run:

    python bench/gemm_probe.py [--dtype float16] [--tokens 16384]

settings: default | cublaslt (torch.backends.cuda.preferred_blas_library) | reduced-precision accumulation allowed |
TunableOp (torch.cuda.tunable, tuning enabled for the probe).  Prints one JSON line per setting with per-shape
microseconds, TFLOP/s and the step total (12 layers x shapes + LM head).
"""
import argparse
import json

import torch


def shapes(tokens, hidden=768, ffn=3072, vocab_pad=30528, masked=2458):
    # (name, M, N, K, count per step) for y = x @ W^T (fwd), dx = dy @ W (dgrad), dW = dy^T @ x (wgrad)
    out = []
    for name, n_out, n_in, count, rows in (
        ("qkv", 3 * hidden, hidden, 12, tokens), ("out", hidden, hidden, 12, tokens),
        ("fc1", ffn, hidden, 12, tokens), ("fc2", hidden, ffn, 12, tokens), ("lm_head", vocab_pad, hidden, 1, masked),
    ):
        out.append((name + ".fwd", rows, n_out, n_in, count, "nt"))
        out.append((name + ".dgrad", rows, n_in, n_out, count, "nn"))
        out.append((name + ".wgrad", n_out, n_in, rows, count, "tn"))
    return out


def time_mm(a, b, iters=20):
    for _ in range(3):
        torch.mm(a, b)
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        torch.mm(a, b)
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters * 1e3  # us


def run(dtype, tokens):
    res, total = {}, 0.0
    for name, m, n, k, count, layout in shapes(tokens):
        if layout == "nt":      # [m, k] @ [n, k]^T
            a, b = torch.randn(m, k, device="cuda", dtype=dtype), torch.randn(n, k, device="cuda", dtype=dtype).t()
        elif layout == "nn":    # [m, k] @ [k, n]
            a, b = torch.randn(m, k, device="cuda", dtype=dtype), torch.randn(k, n, device="cuda", dtype=dtype)
        else:                   # [k, m]^T @ [k, n]
            a, b = torch.randn(k, m, device="cuda", dtype=dtype).t(), torch.randn(k, n, device="cuda", dtype=dtype)
        us = time_mm(a, b)
        res[name] = {"us": round(us, 1), "tflops": round(2.0 * m * n * k / us / 1e6, 1)}
        total += us * count
    return res, total / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dtype", default="float16", choices=["float16", "bfloat16"])
    ap.add_argument("--tokens", type=int, default=16384)
    a = ap.parse_args()
    dtype = getattr(torch, a.dtype)
    settings = ["default", "cublaslt", "reduced_precision", "tunableop"]
    for setting in settings:
        torch.backends.cuda.preferred_blas_library("cublas")
        torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction = False
        torch.backends.cuda.matmul.allow_bf16_reduced_precision_reduction = False
        tunable = getattr(torch.cuda, "tunable", None)
        if tunable is not None:
            tunable.enable(False)
        try:
            if setting == "cublaslt":
                torch.backends.cuda.preferred_blas_library("cublaslt")
            elif setting == "reduced_precision":
                torch.backends.cuda.matmul.allow_fp16_reduced_precision_reduction = True
                torch.backends.cuda.matmul.allow_bf16_reduced_precision_reduction = True
            elif setting == "tunableop":
                if tunable is None:
                    raise RuntimeError("torch.cuda.tunable not available")
                tunable.enable(True)
                tunable.tuning_enable(True)
            res, total_ms = run(dtype, a.tokens)
            print(json.dumps({"setting": setting, "dtype": a.dtype, "gemm_ms_per_step": round(total_ms, 3), "shapes": res}))
        except Exception as exc:  # noqa: BLE001
            print(json.dumps({"setting": setting, "error": repr(exc)[:200]}))
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
