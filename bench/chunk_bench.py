#!/usr/bin/env python3
"""Multi-token steps into a key / value cache: one chunk call against T decode calls.

Kernel arm: device time of ``ops.attention_with_kv_cache`` with a chunk of T queries per (b, h) against a [B, C, H, D]
fp16 cache, appending the T new keys / values (the KV-cache mode of the wgmma forward, plus its append kernel), against
T successive appending single-query calls (``fmha_decode``, the path a chunk took before) and against the same chunk
in ``attention_with_kv_cache_reference`` (PyTorch).  T in {4, 16, 64, 256}, B in {1, 8, 64}, (H, D) in {(12, 64),
(8, 96)}, every sequence at n visible keys after the chunk, n in {1024, 4096}.  CUDA events, every arm warmed up,
alternating, median of --rounds rounds of --iters calls.  The achieved bandwidth counts the K and V bytes a chunk has
to read once (B * n * H * D * 2 bytes each, from the shapes) over the chunk's time, against the H100 SXM data-sheet
3.35 TB/s.  ``ctas`` is the chunk kernel's grid: B * H * ceil(T / 64) CTAs (no split-KV).

End-to-end arm: a 6-layer default ``TransformerDecoder`` (768 wide, 8 heads, fp16, eval), B = 8, a 128-token prompt
prefilled, then a given 256-token continuation fed in chunks of {1, 16, 64, 256} tokens.  Tokens/s count the B * 256
continuation tokens; ``max_rel_diff`` is the largest per-token relative difference of the outputs from the one-token
path.

Prints the card name and power limit, then one JSON line per measurement.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name()


def time_ms(fn, iters):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def alternate(arms, iters, rounds):
    for fn in arms.values():   # warm-up
        fn()
        fn()
    torch.cuda.synchronize()
    times = {name: [] for name in arms}
    names = list(arms)
    for r in range(rounds):
        for name in (names if r % 2 == 0 else names[::-1]):
            times[name].append(time_ms(arms[name], iters))
    return {name: sorted(t)[len(t) // 2] for name, t in times.items()}


def kernel_arm(ops, T, B, H, D, n, iters, rounds):
    g = torch.Generator(device="cuda").manual_seed(0)
    C = n
    k = torch.randn(B, C, H, D, device="cuda", generator=g).half()
    v = torch.randn(B, C, H, D, device="cuda", generator=g).half()
    qkv = torch.randn(B, T, 3, H, D, device="cuda", generator=g).half()
    q, k_new, v_new = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    p = n - T   # the T appended rows make n visible keys
    seqlens = torch.full((B,), p, dtype=torch.int32, device="cuda")
    steps_lens = [seqlens + i for i in range(T)]

    def chunk():
        return ops.attention_with_kv_cache(q, k, v, seqlens, p, k_new=k_new, v_new=v_new)

    def steps():
        return [ops.attention_with_kv_cache(q[:, i:i + 1], k, v, steps_lens[i], p + i, k_new=k_new[:, i:i + 1],
                                            v_new=v_new[:, i:i + 1]) for i in range(T)]

    def ref():
        return ops.attention_with_kv_cache_reference(q, k, v, seqlens, p, k_new=k_new, v_new=v_new)

    with torch.no_grad():
        a, s, r = chunk().float(), torch.cat(steps(), 1).float(), ref().float()
        err_ref = ((a - r).norm() / r.norm()).item()
        err_steps = ((a - s).norm() / s.norm()).item()
        med = alternate({"chunk": chunk, "steps": steps, "reference": ref}, iters, rounds)
    kv_bytes = 2 * B * n * H * D * 2
    bw = kv_bytes / (med["chunk"] * 1e-3)
    out = {"arm": "kernel", "T": T, "B": B, "H": H, "D": D, "n": n, "ctas": B * H * ((T + 63) // 64),
           "chunk_ms": round(med["chunk"], 4), "steps_ms": round(med["steps"], 4),
           "reference_ms": round(med["reference"], 4), "vs_steps": round(med["steps"] / med["chunk"], 2),
           "vs_reference": round(med["reference"] / med["chunk"], 2), "kv_bytes": kv_bytes,
           "chunk_GBps": round(bw / 1e9, 1), "of_3.35TBps": round(bw / HBM_BYTES_PER_S, 3),
           "rel_err_ref": err_ref, "rel_diff_steps": err_steps}
    print(json.dumps(out), flush=True)
    del k, v


def end_to_end(B, prompt_len, new_tokens, chunks, rounds):
    from unicore.modules import TransformerDecoder

    torch.manual_seed(0)
    total = prompt_len + new_tokens
    model = TransformerDecoder(max_seq_len=total).cuda().half().eval()
    g = torch.Generator(device="cuda").manual_seed(1)
    emb = torch.randn(B, total, 768, device="cuda", generator=g).half()

    def run(size):
        cache = model.new_cache(B, total)
        model(emb[:, :prompt_len], cache=cache)
        outs = [model(emb[:, t:t + size], cache=cache) for t in range(prompt_len, total, size)]
        return torch.cat(outs, 1)

    arms = {size: (lambda size=size: run(size)) for size in chunks}
    times = {size: [] for size in chunks}
    outs = {}
    with torch.no_grad():
        for fn in arms.values():   # warm-up
            fn()
        torch.cuda.synchronize()
        for r in range(rounds):
            for size in (chunks if r % 2 == 0 else chunks[::-1]):
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                outs[size] = arms[size]()
                e.record()
                torch.cuda.synchronize()
                times[size].append(s.elapsed_time(e) / 1e3)
    base = outs[1].float() if 1 in outs else None
    for size in chunks:
        med = sorted(times[size])[len(times[size]) // 2]
        out = {"arm": "end_to_end", "B": B, "prompt": prompt_len, "new_tokens": new_tokens, "chunk": size,
               "layers": len(model.layers), "tok_s": round(B * new_tokens / med, 1), "seconds": round(med, 4)}
        if base is not None:
            y = outs[size].float()
            out["max_rel_diff"] = ((y - base).norm(dim=-1) / base.norm(dim=-1)).max().item()
        print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--e2e-rounds", type=int, default=3)
    ap.add_argument("--T", type=int, nargs="*", default=[4, 16, 64, 256])
    ap.add_argument("--batch", type=int, nargs="*", default=[1, 8, 64])
    ap.add_argument("--lengths", type=int, nargs="*", default=[1024, 4096])
    ap.add_argument("--chunks", type=int, nargs="*", default=[1, 16, 64, 256])
    ap.add_argument("--skip-kernel", action="store_true")
    ap.add_argument("--skip-e2e", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("chunk_bench needs a GPU")
    from unicore import ops

    assert ops.USE_NATIVE, "native kernels are not active"
    print("card:", card(), flush=True)
    if not args.skip_kernel:
        for B in args.batch:
            for H, D in ((12, 64), (8, 96)):
                for n in args.lengths:
                    for T in args.T:
                        kernel_arm(ops, T, B, H, D, n, args.iters, args.rounds)
                        torch.cuda.empty_cache()
    if not args.skip_e2e:
        end_to_end(8, 128, 256, args.chunks, args.e2e_rounds)


if __name__ == "__main__":
    main()
