#!/usr/bin/env python3
"""Paged key / value caches against contiguous ones: step time, captured decoding and memory.

Op arm: device time per call of ``ops.attention_with_kv_cache`` with a one-token step (the split-KV decode kernel) and
with a 16-token chunk (the KV-cache mode of the wgmma forward), each appending its rows, 12 heads of 64, fp16, every
sequence at the same visible length, at B in {1, 8, 64} and lengths {512, 2048}.  The paged arm reads pools of
128-row blocks through a shuffled block table (``B * capacity / 128`` blocks); the contiguous arm reads [B, C, H, D]
caches holding the same rows.  CUDA events, both arms warmed up, alternating, median of --rounds rounds of --iters
calls.

End-to-end arm: greedy decoding with a 6-layer default ``TransformerDecoder`` (768 wide, 8 heads, fp16, eval) under a
tied 1024-token embedding / output table, B = 8, a 128-token prompt, 256 new tokens, every step a captured CUDA graph
(``capture_step``); a paged cache (128-row blocks) against a contiguous one, alternating.  Tokens/s count the tokens of
the B * 255 steps after the first (which captures the graph); ``same_tokens`` says whether the two arms generated the
same tokens.

Memory arm: the cache bytes of each layout for B = 256 sequences of capacity 2048 whose lengths are uniform on
[1, 800], with the paged blocks counted from the block table the allocator kernels fill (``kv_blocks_reserve``).

Prints the card name and power limit, then one JSON line per measurement.
"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "bench"))

from decode_bench import alternate, card  # noqa: E402

BS = 128


def paged_copy(k, v, g):
    """Pools of 128-row blocks holding the rows of the [B, C, H, D] caches k / v, behind a shuffled block table."""
    B, C = k.shape[:2]
    M = C // BS
    table = torch.randperm(B * M, device=k.device, generator=g).view(B, M).to(torch.int32)
    kp = torch.empty(B * M, BS, *k.shape[2:], dtype=k.dtype, device=k.device)
    vp = torch.empty_like(kp)
    kp[table.long()] = k.view(B, M, BS, *k.shape[2:])
    vp[table.long()] = v.view(B, M, BS, *v.shape[2:])
    return kp, vp, table


def op_arm(args, ops):
    H, D = 12, 64
    g = torch.Generator(device="cuda").manual_seed(0)
    for T in (1, 16):
        for B in args.batch:
            for n in args.lengths:
                C = n + 128   # a whole number of blocks above the n visible rows and the appended ones
                k = (torch.randn(B, C, H, D, device="cuda", generator=g) * 0.5).half()
                v = torch.randn(B, C, H, D, device="cuda", generator=g).half()
                kp, vp, table = paged_copy(k, v, g)
                q = (torch.randn(B, T, H, D, device="cuda", generator=g) * 0.5).half()
                kn, vn = (torch.randn(B, T, H, D, device="cuda", generator=g).half() for _ in range(2))
                seqlens = torch.full((B,), n - T, dtype=torch.int32, device="cuda")
                with torch.no_grad():
                    ref = ops.attention_with_kv_cache(q, k, v, seqlens, n - T, kn, vn)
                    got = ops.attention_with_kv_cache(q, kp, vp, seqlens, n - T, kn, vn, block_table=table)
                    same = bool(torch.equal(ref, got))
                    t = alternate({
                        "contiguous": lambda: ops.attention_with_kv_cache(q, k, v, seqlens, n - T, kn, vn),
                        "paged": lambda: ops.attention_with_kv_cache(q, kp, vp, seqlens, n - T, kn, vn,
                                                                     block_table=table),
                    }, args.iters, args.rounds)
                out = {"arm": "op", "T": T, "B": B, "len": n, "contiguous_us": round(t["contiguous"] * 1e3, 2),
                       "paged_us": round(t["paged"] * 1e3, 2), "paged_over_contiguous": round(t["paged"] /
                                                                                               t["contiguous"], 3),
                       "bitwise_equal": same}
                print(json.dumps(out), flush=True)


def e2e_arm(args):
    from unicore.modules import TransformerDecoder

    B, P, N, V = 8, 128, 256, 1024
    torch.manual_seed(0)
    m = TransformerDecoder(max_seq_len=P + N).cuda().eval().half()
    g = torch.Generator(device="cuda").manual_seed(1)
    table = (torch.randn(V, m.embed_dim, device="cuda", generator=g) * 0.5).half()
    prompt = table[torch.randint(0, V, (B, P), device="cuda", generator=g)]
    cap = P + N

    def run(block_size):
        cache = m.new_cache(B, cap, block_size=block_size)
        toks = []
        with torch.no_grad():
            y = m(prompt, cache=cache)[:, -1:]
            step = m.capture_step(cache)
            for i in range(N):
                if i == 1:   # the first call captures the graph: the clock starts after it
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                tok = (y[:, 0].float() @ table.float().t()).argmax(-1)
                toks.append(tok)
                y = step(table[tok][:, None])
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
        return dt, torch.stack(toks, 1)

    res = {"contiguous": [], "paged": []}
    out_toks = {}
    for r in range(args.e2e_rounds + 1):   # round 0 warms up both arms
        for name in (["contiguous", "paged"] if r % 2 == 0 else ["paged", "contiguous"]):
            dt, toks = run(None if name == "contiguous" else BS)
            out_toks[name] = toks
            if r > 0:
                res[name].append(B * (N - 1) / dt)
    med = {k: sorted(v)[len(v) // 2] for k, v in res.items()}
    print(json.dumps({"arm": "captured_greedy", "B": B, "prompt": P, "new_tokens": N,
                      "contiguous_tok_s": round(med["contiguous"], 1), "paged_tok_s": round(med["paged"], 1),
                      "paged_over_contiguous": round(med["paged"] / med["contiguous"], 3),
                      "same_tokens": bool(torch.equal(out_toks["contiguous"], out_toks["paged"]))}), flush=True)


def memory_arm(ops):
    B, C, layers, H_kv, D = 256, 2048, 6, 12, 64
    g = torch.Generator().manual_seed(2)
    lengths = torch.randint(1, 801, (B,), generator=g, dtype=torch.int32).cuda()
    M = C // BS
    table = torch.full((B, M), -1, dtype=torch.int32, device="cuda")
    free = torch.arange(B * M - 1, -1, -1, dtype=torch.int32, device="cuda")
    count = torch.tensor([B * M], dtype=torch.int32, device="cuda")
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    ops.kv_blocks_reserve(table, free, count, lengths, BS, flag)
    blocks = int((table >= 0).sum())
    row = 2 * H_kv * D * 2 * layers   # K and V, fp16, every layer
    print(json.dumps({"arm": "memory", "B": B, "capacity": C, "mean_len": round(float(lengths.float().mean()), 1),
                      "contiguous_bytes": B * C * row, "paged_bytes": blocks * BS * row, "blocks": blocks,
                      "ratio": round(B * C / (blocks * BS), 2)}), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--e2e-rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, nargs="*", default=[1, 8, 64])
    ap.add_argument("--lengths", type=int, nargs="*", default=[512, 2048])
    ap.add_argument("--skip-e2e", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("paged_decode_bench.py measures on a GPU; none is available")
    from unicore import ops

    assert ops.USE_NATIVE, "the native kernels are not active"
    print("card:", card(), flush=True)
    op_arm(args, ops)
    if not args.skip_e2e:
        e2e_arm(args)
    memory_arm(ops)


if __name__ == "__main__":
    main()
