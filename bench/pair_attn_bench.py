#!/usr/bin/env python3
"""Uni-Mol's pair-bias attention: the fused kernel in logits mode against the materialised chain.

Shape of one Uni-Mol layer's attention: H = 64, D = 8, bf16, a per-batch bias [B, H, L, L] with its gradient, key
padding, dropout 0.1, and an incoming gradient dz of the logits (they are the next layer's bias).  Arms:
* fused: ``ops.fused_attention_qkvpacked(..., return_logits=True)``;
* materialised: what ``SelfMultiheadAttention.attend(return_attn=True)`` runs with the probabilities requested:
  split_heads -> bmm -> softmax_dropout_with_logits -> bmm -> merge_heads.

Times forward and forward + backward with CUDA events, and prints one JSON line per (arm, L) with ms, the
achieved bandwidth of the pair traffic (bytes counted below, over the time) against 3.35 TB/s (H100 SXM data
sheet), and the peak memory allocated during forward + backward beyond the inputs.

Pair traffic, in 16-bit passes over one [B, H, L, L] tensor (the q/k/v traffic is small at D = 8):
  materialised forward:  bmm writes S; softmax reads S and bias, writes z and P_drop; bmm reads P_drop   = 6
  materialised backward: dP write, P_drop read (dV), softmax backward reads dP, z and dz and writes dx,
                         two bmm reads of dx                                                            = 8
  fused forward:  read bias, write z, write keep bits (1/16)                                           = 2 + 1/16
  fused backward: read bias, read dz, write dbias, read keep bits                                      = 3 + 1/16
"""
import argparse
import json
import math
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet (700 W)
PASSES = {"fused": (2 + 1 / 16, 3 + 1 / 16), "materialised": (6.0, 8.0)}


def timeit(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def peak_bytes(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=32)
    ap.add_argument("--H", type=int, default=64)
    ap.add_argument("--D", type=int, default=8)
    ap.add_argument("--L", type=int, nargs="+", default=[128, 256])
    ap.add_argument("--p", type=float, default=0.1)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    from unicore import ops
    from unicore.modules.attention import _materialised_attention

    assert ops.USE_NATIVE and torch.cuda.is_available(), "this benchmark needs the native kernels on a GPU"
    B, H, D, p = args.B, args.H, args.D, args.p
    dtype = torch.bfloat16
    scale = 1.0 / math.sqrt(D)
    for L in args.L:
        torch.manual_seed(0)
        qkv = (torch.randn(B, L, 3, H, D, device="cuda") * 0.5).to(dtype).requires_grad_(True)
        bias = torch.randn(B, H, L, L, device="cuda").to(dtype).requires_grad_(True)
        kpm = torch.zeros(B, L, dtype=torch.bool, device="cuda")
        kpm[:, L - L // 8:] = True
        dout = torch.randn(B, L, H * D, device="cuda").to(dtype)
        dz = torch.randn(B, H, L, L, device="cuda").to(dtype)
        assert ops.fused_attention_supported(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], bias, kpm)

        def fused():
            o, z = ops.fused_attention_qkvpacked(qkv, bias=bias, key_padding_mask=kpm, dropout_p=p, training=True,
                                                 scale=scale, return_logits=True)
            return o.reshape(B, L, H * D), z

        def materialised():
            qh, kh, vh = ops.split_heads(qkv.view(B, L, 3 * H * D), 3, H, scale)
            o, z, _ = _materialised_attention(qh, kh, vh, kpm, bias, p, True, True)
            return o, z.view(B, H, L, L)

        pair_bytes = B * H * L * L * 2
        for name, fn in (("fused", fused), ("materialised", materialised)):
            def fwd_bwd(fn=fn):
                qkv.grad = None
                bias.grad = None
                o, z = fn()
                torch.autograd.backward([o, z], [dout, dz])

            with torch.no_grad():
                t_f = timeit(fn, args.iters)
            t_fb = timeit(fwd_bwd, args.iters)
            qkv.grad = None
            bias.grad = None
            mem = peak_bytes(fwd_bwd)
            qkv.grad = None
            bias.grad = None
            pf, pb = PASSES[name]
            gbs_f = pf * pair_bytes / (t_f * 1e-3) / 1e9
            gbs_fb = (pf + pb) * pair_bytes / (t_fb * 1e-3) / 1e9
            print(json.dumps({
                "arm": name, "B": B, "H": H, "L": L, "D": D, "dtype": "bf16", "p": p,
                "fwd_ms": round(t_f, 4), "fwd_bwd_ms": round(t_fb, 4),
                "fwd_GBps": round(gbs_f, 1), "fwd_bwd_GBps": round(gbs_fb, 1),
                "fwd_frac_of_hbm": round(gbs_f * 1e9 / HBM_BYTES_PER_S, 3),
                "fwd_bwd_frac_of_hbm": round(gbs_fb * 1e9 / HBM_BYTES_PER_S, 3),
                "peak_fwd_bwd_MB": round(mem / 2 ** 20, 1), "pair_tensor_MB": round(pair_bytes / 2 ** 20, 1),
            }), flush=True)


if __name__ == "__main__":
    main()
