#!/usr/bin/env python3
"""Incremental decoding with the step captured in a CUDA graph (``TransformerDecoder.capture_step``).

End-to-end arm: greedy decoding with the model, table and prompt of ``bench/decode_bench.py``'s end-to-end arm (6-layer
default ``TransformerDecoder``, 768 wide, 8 heads, fp16, eval; a tied 1024-token table; 128-token prompts, 256 new
tokens) at B in {1, 8, 64}: eager incremental steps against captured steps.  Each arm keeps one cache (and the captured
arm one captured step) across its runs, and every run starts with a new prefill into it, as a server would.  Tokens/s
count the B * 256 generated tokens per run (median of --e2e-rounds alternating runs); ``same_tokens`` is the share of
generated tokens on which the two arms agree; ``step_ms`` is the median device time between the starts of two
consecutive steps (CUDA events recorded on the stream, so it includes the gaps where the GPU waits for the host).

Kernel arm: ``fmha_decode`` with the host bound at the capacity C in {4096, 16384} (as in a captured step), appending,
every sequence at n in {256, 1024, 4096} visible keys, B x H in {12, 96, 768} (H = 12, D = 64): the split ranges from
the host bound (``split_by_length=False``) against those from each sequence's device length (True).  Device time per
call (CUDA events, alternating, median of --rounds rounds of --iters calls) and the K + V bytes of the n visible keys
over it.

Prints the card name, power limit and max SM clock, then one JSON line per measurement.
"""
import argparse
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from decode_bench import alternate, card  # noqa: E402


def kernel_arm(ops, B, H, D, C, n, iters, rounds):
    g = torch.Generator(device="cuda").manual_seed(0)
    k = torch.randn(B, C, H, D, device="cuda", generator=g).half()
    v = torch.randn(B, C, H, D, device="cuda", generator=g).half()
    qkv = torch.randn(B, 1, 3, H, D, device="cuda", generator=g).half()
    q, k_new, v_new = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    seqlens = torch.full((B,), n - 1, dtype=torch.int32, device="cuda")   # the appended row makes n visible keys
    scale = D ** -0.5

    def call(by_length):
        return lambda: ops.native().fmha_decode(q, k, v, seqlens, C - 1, k_new, v_new, None, None, scale, 0,
                                                split_by_length=by_length)

    arms = {"bound": call(False), "length": call(True)}
    with torch.no_grad():
        diff = (arms["bound"]().float() - arms["length"]().float()).abs().max().item()
        med = alternate(arms, iters, rounds)
    kv_bytes = 2 * B * n * H * D * 2
    out = {"arm": "kernel", "B": B, "H": H, "D": D, "C": C, "n": n,
           "splits": ops.native().fmha_decode_num_splits(B, H, C),
           "bound_us": round(med["bound"] * 1e3, 1), "length_us": round(med["length"] * 1e3, 1),
           "speedup": round(med["bound"] / med["length"], 2), "kv_bytes": kv_bytes,
           "bound_GBps": round(kv_bytes / (med["bound"] * 1e-3) / 1e9, 1),
           "length_GBps": round(kv_bytes / (med["length"] * 1e-3) / 1e9, 1), "max_abs_diff": diff}
    print(json.dumps(out), flush=True)


def end_to_end(B, prompt_len, new_tokens, rounds):
    from unicore.modules import TransformerDecoder

    torch.manual_seed(0)
    total = prompt_len + new_tokens
    model = TransformerDecoder(max_seq_len=total).cuda().half().eval()
    table = (torch.randn(1024, 768, device="cuda") * 0.5).half()
    prompt = torch.randint(0, 1024, (B, prompt_len), device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))

    def next_token(y):   # y [B, E] -> greedy token ids [B]
        return (y.float() @ table.float().t()).argmax(-1)

    caches = {name: model.new_cache(B, total) for name in ("eager", "captured")}
    starts = {name: [torch.cuda.Event(enable_timing=True) for _ in range(new_tokens + 1)] for name in caches}
    step_fn = {}

    def decode(name):
        cache = caches[name]
        cache.rewind(cache.max_len)   # a new prefill into the same cache
        y = model(table[prompt], cache=cache)[:, -1]
        if name == "captured" and name not in step_fn:
            step_fn[name] = model.capture_step(cache)
        step = step_fn.get(name, lambda emb: model(emb, cache=cache))
        toks = []
        for i in range(new_tokens):
            starts[name][i].record()
            tok = next_token(y)
            toks.append(tok)
            y = step(table[tok][:, None])[:, 0]
        starts[name][new_tokens].record()
        return torch.stack(toks, 1)

    times = {name: [] for name in caches}
    step_ms = {name: [] for name in caches}
    outs = {}
    with torch.no_grad():
        for name in caches:   # warm-up (and the one capture)
            decode(name)
        torch.cuda.synchronize()
        for r in range(rounds):
            for name in (list(caches) if r % 2 == 0 else list(caches)[::-1]):
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                outs[name] = decode(name)
                e.record()
                torch.cuda.synchronize()
                times[name].append(s.elapsed_time(e) / 1e3)
                ev = starts[name]
                step_ms[name] += [ev[i].elapsed_time(ev[i + 1]) for i in range(new_tokens)]
    med = {name: sorted(t)[len(t) // 2] for name, t in times.items()}
    per_step = {name: sorted(t)[len(t) // 2] for name, t in step_ms.items()}
    same = (outs["eager"] == outs["captured"]).float().mean().item()
    out = {"arm": "end_to_end", "B": B, "prompt": prompt_len, "new_tokens": new_tokens, "layers": len(model.layers),
           "eager_tok_s": round(B * new_tokens / med["eager"], 1),
           "captured_tok_s": round(B * new_tokens / med["captured"], 1),
           "speedup": round(med["eager"] / med["captured"], 2),
           "eager_step_ms": round(per_step["eager"], 4), "captured_step_ms": round(per_step["captured"], 4),
           "captures": step_fn["captured"].captures, "same_tokens": round(same, 4)}
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--e2e-rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, nargs="*", default=[1, 8, 64])
    ap.add_argument("--capacities", type=int, nargs="*", default=[4096, 16384])
    ap.add_argument("--lengths", type=int, nargs="*", default=[256, 1024, 4096])
    ap.add_argument("--new-tokens", type=int, default=256)
    ap.add_argument("--skip-kernel", action="store_true")
    ap.add_argument("--skip-e2e", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("graph_decode_bench needs a GPU")
    from unicore import ops

    assert ops.USE_NATIVE, "native kernels are not active"
    print("card:", card(), flush=True)
    if not args.skip_e2e:
        for B in args.batch:
            end_to_end(B, 128, args.new_tokens, args.e2e_rounds)
            torch.cuda.empty_cache()
    if not args.skip_kernel:
        for C in args.capacities:
            for B in args.batch:
                for n in args.lengths:
                    if n <= C:
                        kernel_arm(ops, B, 12, 64, C, n, args.iters, args.rounds)
                torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
