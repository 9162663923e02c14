#!/usr/bin/env python3
"""Achieved HBM bandwidth of the memory-bound kernels at the flagship (BERT-base, 32x512 tokens) shapes.

Each op is timed with CUDA events over ``--iters`` launches after warm-up; the operands of
consecutive launches rotate over enough distinct buffers to exceed the 50 MB L2.  Prints one JSON
line per op: microseconds, the minimum bytes the op must move, and the resulting GB/s (compare with
the 3.35 TB/s of HBM3 in the H100 SXM data sheet).
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from unicore_b200.ops._native import native  # noqa: E402


def timeit(fns, iters):
    for f in fns:
        f()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for i in range(iters):
        fns[i % len(fns)]()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters * 1e3  # us


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=32 * 512)
    ap.add_argument("--hidden", type=int, default=768)
    ap.add_argument("--ffn", type=int, default=3072)
    ap.add_argument("--iters", type=int, default=40)
    ap.add_argument("--dtype", default="float16")
    a = ap.parse_args()
    dt = getattr(torch, a.dtype)
    C = native()
    R, H, F = a.rows, a.hidden, a.ffn
    nbuf = 6
    es = 2
    out = []

    def report(name, us, nbytes):
        out.append({"op": name, "us": round(us, 2), "MB": round(nbytes / 1e6, 1), "GBps": round(nbytes / us / 1e3, 1)})
        print(json.dumps(out[-1]), flush=True)

    g = torch.randn(H, device="cuda", dtype=dt)
    b = torch.randn(H, device="cuda", dtype=dt)
    xs = [torch.randn(R, H, device="cuda", dtype=dt) for _ in range(nbuf)]
    rs = [torch.randn(R, H, device="cuda", dtype=dt) for _ in range(nbuf)]
    # LayerNorm
    us = timeit([lambda x=x: C.layernorm_fwd(x, g, b, 1e-5) for x in xs], a.iters)
    report("layernorm_fwd", us, 2 * R * H * es)
    y, mean, rstd = C.layernorm_fwd(xs[0], g, b, 1e-5)
    us = timeit([lambda x=x, d=d: C.layernorm_bwd(d, x, mean, rstd, g) for x, d in zip(xs, rs)], a.iters)
    report("layernorm_bwd(+dgamma,dbeta)", us, 3 * R * H * es)
    # fused bias + dropout + residual + LN
    for p in (0.0, 0.1):
        us = timeit([lambda x=x, r=r: C.bias_dropout_add_ln_fwd(x, b, r, g, b, p, 1e-5) for x, r in zip(xs, rs)], a.iters)
        report("bias_dropout_add_ln_fwd p=%.1f" % p, us, 4 * R * H * es)
        y, mean, rstd, summed, seed, off = C.bias_dropout_add_ln_fwd(xs[0], b, rs[0], g, b, p, 1e-5)
        us = timeit([lambda s=s, d=d: C.bias_dropout_add_ln_bwd(d, s, mean, rstd, g, p, seed, off, True) for s, d in zip(xs, rs)], a.iters)
        report("bias_dropout_add_ln_bwd(+dbias) p=%.1f" % p, us, (4 if p > 0 else 3) * R * H * es)
    del xs, rs
    # bias + GELU
    fb = torch.randn(F, device="cuda", dtype=dt)
    fx = [torch.randn(R, F, device="cuda", dtype=dt) for _ in range(3)]
    fd = [torch.randn(R, F, device="cuda", dtype=dt) for _ in range(3)]
    us = timeit([lambda x=x: C.bias_gelu_fwd(x, fb) for x in fx], a.iters)
    report("bias_gelu_fwd", us, 2 * R * F * es)
    us = timeit([lambda x=x, d=d: C.bias_gelu_bwd(d, x, fb) for x, d in zip(fx, fd)], a.iters)
    report("bias_gelu_bwd(+dbias)", us, 3 * R * F * es)
    del fx, fd
    # cross entropy over a padded vocabulary
    n, V, Vp = 2458, 30522, 30528
    lg = [torch.randn(n, Vp, device="cuda", dtype=dt) for _ in range(3)]
    tgt = torch.randint(0, V, (n,), device="cuda")
    us = timeit([lambda l=l: C.softmax_xent_fwd(l, tgt, 1, V) for l in lg], a.iters)
    report("softmax_xent_fwd", us, n * V * es)
    loss, lse = C.softmax_xent_fwd(lg[0], tgt, 1, V)
    one = torch.ones(1, device="cuda")
    us = timeit([lambda l=l: C.softmax_xent_bwd(l, tgt, lse, one, 1, V) for l in lg], a.iters)
    report("softmax_xent_bwd", us, 2 * n * V * es)
    # copy roofline for reference
    src = [torch.empty(256 << 20, device="cuda", dtype=torch.uint8) for _ in range(2)]
    dst = torch.empty(256 << 20, device="cuda", dtype=torch.uint8)
    us = timeit([lambda s=s: dst.copy_(s) for s in src], 20)
    report("torch copy 256MB (roofline)", us, 2 * (256 << 20))
    return 0


if __name__ == "__main__":
    sys.exit(main())
