#!/usr/bin/env python3
"""Packed variable-length steps into a key / value cache against the padded chunk of the same tokens.

Op arm: device time of ``ops.attention_with_kv_cache_varlen`` (packed ``[N, H, D]`` queries, each sequence its own T_b,
appending its T_b keys / values) against ``ops.attention_with_kv_cache`` on the same tokens padded to ``[B, max T_b,
H, D]`` (appending max T_b rows per sequence; at max T_b = 1 that is the split-KV decode kernel).  B = 16 sequences of
(H, D) = (12, 64), each at 1024 cached keys; T_b distributions: half the batch at 1 and half at a 512-token prompt,
uniform on [1, 64], and all 1.  CUDA events, every arm warmed up, alternating, median of --rounds rounds of --iters
calls.  ``rel_diff`` is the largest per-row relative difference between the arms at the real rows.

End-to-end arm, on the 6-layer default ``TransformerDecoder`` (768 wide, 8 heads, fp16, eval), B = 16:
  * prefill: prompts of lengths uniform on [32, 512], packed (``cu_seqlens``) against padded (``padding_mask``);
  * verification of ragged drafts: after a 256-token prefill, draft lengths uniform on [1, 8] per sequence, packed
    against padded to the longest draft plus ``rewind`` of the extra rows.
Tokens/s count the real tokens; ``max_rel_diff`` is the largest per-token relative difference of the outputs between
the arms.  Each timed call starts from the same cache state.

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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name()


def alternate(arms, iters, rounds):
    """Median milliseconds per call of each arm, the arms alternating in order every round."""
    for fn in arms.values():   # warm-up
        fn()
        fn()
    torch.cuda.synchronize()
    times = {name: [] for name in arms}
    names = list(arms)
    for r in range(rounds):
        for name in (names if r % 2 == 0 else names[::-1]):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(iters):
                arms[name]()
            e.record()
            torch.cuda.synchronize()
            times[name].append(s.elapsed_time(e) / iters)
    return {name: sorted(t)[len(t) // 2] for name, t in times.items()}


def _cu(sizes):
    return torch.tensor([0] + torch.tensor(sizes).cumsum(0).tolist(), dtype=torch.int32, device="cuda")


def _rel(a, b):
    return ((a.float() - b.float()).norm(dim=-1) / b.float().norm(dim=-1).clamp(min=1e-6)).max().item()


def op_arm(ops, name, sizes, H, D, n, iters, rounds):
    g = torch.Generator(device="cuda").manual_seed(0)
    B, T, N = len(sizes), max(sizes), sum(sizes)
    C = n + T
    k = torch.randn(B, C, H, D, device="cuda", generator=g).half()
    v = torch.randn(B, C, H, D, device="cuda", generator=g).half()
    qkv = torch.randn(B, T, 3, H, D, device="cuda", generator=g).half()   # padded; the packed arm takes its real rows
    real = torch.arange(T, device="cuda")[None, :] < torch.tensor(sizes, device="cuda")[:, None]
    packed = qkv[real].contiguous()   # [N, 3, H, D]
    cu = _cu(sizes)
    seqlens = torch.full((B,), n, dtype=torch.int32, device="cuda")

    def run_packed():
        return ops.attention_with_kv_cache_varlen(packed[:, 0], k, v, cu, T, seqlens, n, k_new=packed[:, 1],
                                                  v_new=packed[:, 2])

    def run_padded():
        return ops.attention_with_kv_cache(qkv[:, :, 0], k, v, seqlens, n, k_new=qkv[:, :, 1], v_new=qkv[:, :, 2])

    with torch.no_grad():
        # the padded arm appends rows past T_b that the packed one does not: compare on fresh copies
        k0, v0 = k.clone(), v.clone()
        a = run_packed()
        k.copy_(k0), v.copy_(v0)
        b = run_padded()[real]
        diff = _rel(a, b)
        med = alternate({"packed": run_packed, "padded": run_padded}, iters, rounds)
    out = {"arm": "op", "dist": name, "B": B, "H": H, "D": D, "cached": n, "tokens": N, "padded_tokens": B * T,
           "packed_ms": round(med["packed"], 4), "padded_ms": round(med["padded"], 4),
           "speedup": round(med["padded"] / med["packed"], 2), "rel_diff": diff}
    print(json.dumps(out), flush=True)


def _time(fn, rounds):
    times = []
    for _ in range(rounds):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        times.append(s.elapsed_time(e) / 1e3)
    return sorted(times)[len(times) // 2]


def end_to_end(B, rounds):
    from unicore.modules import TransformerDecoder

    torch.manual_seed(0)
    model = TransformerDecoder(max_seq_len=1024).cuda().half().eval()
    g = torch.Generator(device="cuda").manual_seed(1)
    emb = torch.randn(B, 1024, 768, device="cuda", generator=g).half()

    # ---- prefill of ragged prompts
    lens = torch.randint(32, 513, (B,), generator=torch.Generator().manual_seed(2)).tolist()
    L = max(lens)
    real = torch.arange(L, device="cuda")[None, :] < torch.tensor(lens, device="cuda")[:, None]
    packed_emb = emb[:, :L][real].contiguous()
    cu = _cu(lens)

    def prefill_packed():
        return model(packed_emb, cu_seqlens=cu, max_seqlen=L, cache=model.new_cache(B, 1024))

    def prefill_padded():
        return model(emb[:, :L], padding_mask=~real, cache=model.new_cache(B, 1024))

    # ---- verification of ragged drafts after a 256-token prefill
    drafts = torch.randint(1, 9, (B,), generator=torch.Generator().manual_seed(3)).tolist()
    Td = max(drafts)
    dreal = torch.arange(Td, device="cuda")[None, :] < torch.tensor(drafts, device="cuda")[:, None]
    step = emb[:, 256:256 + Td]
    packed_step = step[dreal].contiguous()
    dcu = _cu(drafts)
    extra = torch.tensor([Td - t for t in drafts], dtype=torch.int32, device="cuda")
    caches = {}
    with torch.no_grad():
        for arm in ("packed", "padded"):
            caches[arm] = model.new_cache(B, 1024)
            model(emb[:, :256], cache=caches[arm])
    start = caches["packed"].seqlens.clone()

    def verify(arm):
        cache = caches[arm]
        cache.seqlens.copy_(start)   # every call starts from the prefilled state
        cache.max_len = 256
        if arm == "packed":
            return model(packed_step, cu_seqlens=dcu, max_seqlen=Td, cache=cache)
        y = model(step, cache=cache)
        cache.rewind(extra)
        return y

    with torch.no_grad():
        results = {}
        for what, arms, tokens in (
                ("prefill", {"packed": prefill_packed, "padded": prefill_padded}, sum(lens)),
                ("verify", {"packed": lambda: verify("packed"), "padded": lambda: verify("padded")}, sum(drafts))):
            for fn in arms.values():   # warm-up
                fn()
            torch.cuda.synchronize()
            times = {name: [] for name in arms}
            for r in range(rounds):
                for name in (list(arms) if r % 2 == 0 else list(arms)[::-1]):
                    times[name].append(_time(arms[name], 1))
            med = {name: sorted(t)[len(t) // 2] for name, t in times.items()}
            yp, yq = arms["packed"](), arms["padded"]()
            mask = real if what == "prefill" else dreal
            results[what] = {"arm": "end_to_end", "what": what, "B": B, "layers": len(model.layers),
                             "tokens": tokens, "padded_tokens": mask.numel(),
                             "packed_tok_s": round(tokens / med["packed"], 1),
                             "padded_tok_s": round(tokens / med["padded"], 1),
                             "speedup": round(med["padded"] / med["packed"], 2),
                             "max_rel_diff": _rel(yp, yq[mask])}
            print(json.dumps(results[what]), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--e2e-rounds", type=int, default=7)
    ap.add_argument("--skip-op", action="store_true")
    ap.add_argument("--skip-e2e", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("packed_decode_bench needs a GPU")
    from unicore import ops

    assert ops.USE_NATIVE, "native kernels are not active"
    print("card:", card(), flush=True)
    B = 16
    rng = torch.Generator().manual_seed(0)
    dists = {"half_1_half_512": [1] * (B // 2) + [512] * (B // 2),
             "uniform_1_64": torch.randint(1, 65, (B,), generator=rng).tolist(),
             "all_1": [1] * B}
    if not args.skip_op:
        for name, sizes in dists.items():
            op_arm(ops, name, sizes, 12, 64, 1024, args.iters, args.rounds)
            torch.cuda.empty_cache()
    if not args.skip_e2e:
        end_to_end(B, args.e2e_rounds)


if __name__ == "__main__":
    main()
