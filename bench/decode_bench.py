#!/usr/bin/env python3
"""Incremental decoding: the decode attention kernel and a whole greedy decode.

Kernel arm: device time per call of ``ops.attention_with_kv_cache`` (one query per (b, h) against a [B, C, H, D] fp16
cache, appending the new key / value, every sequence at the same visible length) against the same call in
``attention_with_kv_cache_reference`` (PyTorch), at B in {1, 8, 64}, (H, D) in {(12, 64), (8, 96)} and visible lengths
{256, 1024, 4096, 16384}.  CUDA events, both arms warmed up, alternating, median of --rounds rounds of --iters calls.
The achieved bandwidth counts the K and V bytes the step has to read (B * n * H * D * 2 bytes each, from the shapes)
over the kernel time, against the H100 SXM data-sheet 3.35 TB/s.  ``splits`` is the split count the kernel picked.

End-to-end arm: greedy decoding with a 6-layer default ``TransformerDecoder`` (768 wide, 8 heads, fp16, eval) under a
tied 1024-token embedding / output table, B = 8, a 128-token prompt, 256 new tokens.  Incremental decoding (prefill +
one cached step per token) against re-running the full forward over the prefix for every token.  Tokens/s count the
B * 256 generated tokens; ``same_tokens`` is the share of generated tokens on which the two arms agree.

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


def kernel_arm(ops, B, H, D, n, iters, rounds):
    g = torch.Generator(device="cuda").manual_seed(0)
    C = n
    k = torch.randn(B, C, H, D, device="cuda", generator=g).half()
    v = torch.randn(B, C, H, D, device="cuda", generator=g).half()
    qkv = torch.randn(B, 1, 3, H, D, device="cuda", generator=g).half()
    q, k_new, v_new = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    seqlens = torch.full((B,), n - 1, dtype=torch.int32, device="cuda")   # the appended row makes n visible keys

    def kern():
        return ops.attention_with_kv_cache(q, k, v, seqlens, n - 1, k_new=k_new, v_new=v_new)

    def ref():
        return ops.attention_with_kv_cache_reference(q, k, v, seqlens, n - 1, k_new=k_new, v_new=v_new)

    with torch.no_grad():
        a, b = kern().float(), ref().float()
        err = ((a - b).norm() / b.norm()).item()
        med = alternate({"kernel": kern, "reference": ref}, iters, rounds)
    kv_bytes = 2 * B * n * H * D * 2
    bw = kv_bytes / (med["kernel"] * 1e-3)
    out = {"arm": "kernel", "B": B, "H": H, "D": D, "n": n, "splits": ops.native().fmha_decode_num_splits(B, H, n),
           "kernel_ms": round(med["kernel"], 4), "reference_ms": round(med["reference"], 4),
           "speedup": round(med["reference"] / med["kernel"], 2), "kv_bytes": kv_bytes,
           "kernel_GBps": round(bw / 1e9, 1), "of_3.35TBps": round(bw / HBM_BYTES_PER_S, 3), "rel_err": err}
    print(json.dumps(out), flush=True)
    del k, v


def end_to_end(B, prompt_len, new_tokens, rounds):
    from unicore.modules import TransformerDecoder

    torch.manual_seed(0)
    total = prompt_len + new_tokens
    model = TransformerDecoder(max_seq_len=total).cuda().half().eval()
    table = (torch.randn(1024, 768, device="cuda") * 0.5).half()
    prompt = torch.randint(0, 1024, (B, prompt_len), device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))

    def next_token(y):   # y [B, E] -> greedy token ids [B]
        return (y.float() @ table.float().t()).argmax(-1)

    def incremental(n_new):
        cache = model.new_cache(B, prompt_len + n_new)
        y = model(table[prompt], cache=cache)[:, -1]
        toks = []
        for _ in range(n_new):
            tok = next_token(y)
            toks.append(tok)
            y = model(table[tok][:, None], cache=cache)[:, 0]
        return torch.stack(toks, 1)

    def recompute(n_new):
        seq = prompt
        toks = []
        for _ in range(n_new):
            tok = next_token(model(table[seq])[:, -1])
            toks.append(tok)
            seq = torch.cat([seq, tok[:, None]], 1)
        return torch.stack(toks, 1)

    arms = {"incremental": incremental, "recompute": recompute}
    times = {name: [] for name in arms}
    outs = {}
    with torch.no_grad():
        for fn in arms.values():   # warm-up, every prefix length of the recompute arm included
            fn(new_tokens)
        torch.cuda.synchronize()
        for r in range(rounds):
            for name in (list(arms) if r % 2 == 0 else list(arms)[::-1]):
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                outs[name] = arms[name](new_tokens)
                e.record()
                torch.cuda.synchronize()
                times[name].append(s.elapsed_time(e) / 1e3)
    med = {name: sorted(t)[len(t) // 2] for name, t in times.items()}
    same = (outs["incremental"] == outs["recompute"]).float().mean().item()
    out = {"arm": "end_to_end", "B": B, "prompt": prompt_len, "new_tokens": new_tokens, "layers": len(model.layers),
           "incremental_tok_s": round(B * new_tokens / med["incremental"], 1),
           "recompute_tok_s": round(B * new_tokens / med["recompute"], 1),
           "speedup": round(med["recompute"] / med["incremental"], 2), "same_tokens": round(same, 4)}
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--e2e-rounds", type=int, default=2)
    ap.add_argument("--batch", type=int, nargs="*", default=[1, 8, 64])
    ap.add_argument("--lengths", type=int, nargs="*", default=[256, 1024, 4096, 16384])
    ap.add_argument("--skip-e2e", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("decode_bench needs a GPU")
    from unicore import ops

    assert ops.USE_NATIVE, "native kernels are not active"
    print("card:", card(), flush=True)
    for B in args.batch:
        for H, D in ((12, 64), (8, 96)):
            for n in args.lengths:
                kernel_arm(ops, B, H, D, n, args.iters, args.rounds)
                torch.cuda.empty_cache()
    if not args.skip_e2e:
        end_to_end(8, 128, 256, args.e2e_rounds)


if __name__ == "__main__":
    main()
