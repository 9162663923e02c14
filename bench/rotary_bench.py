#!/usr/bin/env python3
"""Rotary position embeddings: the kernel, and what a bias-free decoder gains over the T5 relative-position bias.

Kernel arm: device time of ``ops.rotary_embedding`` (the sm_90a kernel) and of its backward (the inverse rotation)
against the PyTorch formula (``ops.rotary_embedding_reference``) on the same fp16 tensor, at
  * B 32 x L 512, H 12, D 64, the packed [B, L, 3 H, D] projection (q and k rotated, rd = D);
  * B 8 x L 2048, H 32, H_kv 8, D 128, the GQA projection [B, L, H + 2 H_kv, D] (rd = D);
  * a decode step, B 64 x T 1, H 8, D 96 (the default decoder's heads), offsets near 1000.
The kernel reads and writes every element once: 2 * B * L * N * D * 2 bytes over the kernel time is the achieved
bandwidth, reported as a share of the H100 SXM data-sheet 3.35 TB/s.

Decoder arm: greedy decoding with the 6-layer default ``TransformerDecoder`` (768 wide, 8 heads, fp16, eval; a 1024-token
table; 128-token prompts, --new-tokens new tokens) at B in {1, 8, 64}, eager steps and captured steps, for
``rel_pos=True`` (the T5 bias, gathered every step) against ``rel_pos=False, rotary_dim=96`` (no bias anywhere).
Tokens/s count the generated tokens per run, median of --e2e-rounds runs, the arms alternating.

Training arm: one fp16 forward + backward of the same decoder at B 8 x L 512 (dropout as constructed), in the same two
configurations; median of --rounds rounds of --iters steps.

CUDA events, every arm warmed up, alternating arms.  Prints the card name, power limit and max SM clock, then one JSON
line per measurement.
"""
import argparse
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

from decode_bench import HBM_BYTES_PER_S, alternate, card  # noqa: E402

E, HEADS = 768, 8
CONFIGS = {"rel_pos": dict(rel_pos=True), "rotary": dict(rel_pos=False, rotary_dim=E // HEADS)}


def kernel_arm(ops, name, B, L, N, R, D, offsets, iters, rounds):
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(B, L, N, D, device="cuda", generator=g).half()
    gy = torch.randn(B, L, N, D, device="cuda", generator=g).half()
    inv = ops.rotary_inv_freq(D, device="cuda")
    off = torch.full((B,), offsets, dtype=torch.int32, device="cuda") if offsets else None
    rot = ops.native().rotary
    arms = {
        "fwd_kernel": lambda: rot.rotary_embedding(x, inv, R, off, False),
        "fwd_torch": lambda: ops.rotary_embedding_reference(x, inv, R, off),
        "bwd_kernel": lambda: rot.rotary_embedding(gy, inv, R, off, True),
        "bwd_torch": lambda: ops.rotary_embedding_reference(gy, inv, R, off, inverse=True),
    }
    with torch.no_grad():
        diff = (arms["fwd_kernel"]().float() - arms["fwd_torch"]().float()).abs().max().item()
        med = alternate(arms, iters, rounds)
    nbytes = 2 * x.numel() * x.element_size()
    out = {"arm": "kernel", "shape": name, "B": B, "L": L, "N": N, "rotated_heads": R, "D": D, "rd": D,
           "plan": {k: v for k, v in rot.rotary_plan(B, L, N, D, D, torch.float16, True).items()
                    if k in ("grid", "sweeps", "vec")},
           "bytes": nbytes, "max_abs_diff_vs_torch": diff}
    for k in ("fwd", "bwd"):
        t = med[k + "_kernel"]
        out[k + "_kernel_us"] = round(t * 1e3, 2)
        out[k + "_torch_us"] = round(med[k + "_torch"] * 1e3, 2)
        out[k + "_of_3.35TBps"] = round(nbytes / (t * 1e-3) / HBM_BYTES_PER_S, 3)
        out[k + "_speedup_vs_torch"] = round(med[k + "_torch"] / t, 2)
    print(json.dumps(out), flush=True)


def _decoder(cfg, max_seq_len, dtype=torch.float16):
    from unicore.modules import TransformerDecoder

    torch.manual_seed(0)
    return TransformerDecoder(max_seq_len=max_seq_len, **CONFIGS[cfg]).cuda().to(dtype)


def decoder_arm(B, prompt_len, new_tokens, rounds):
    total = prompt_len + new_tokens
    models = {cfg: _decoder(cfg, total).eval() for cfg in CONFIGS}
    table = (torch.randn(1024, E, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2)) * 0.5).half()
    prompt = torch.randint(0, 1024, (B, prompt_len), device="cuda", generator=torch.Generator(device="cuda").manual_seed(1))
    arms = [(cfg, mode) for cfg in CONFIGS for mode in ("eager", "captured")]
    caches = {a: models[a[0]].new_cache(B, total) for a in arms}
    steps = {}

    def decode(arm):
        cfg, mode = arm
        model, cache = models[cfg], caches[arm]
        cache.rewind(cache.max_len)   # a new prefill into the same cache
        y = model(table[prompt], cache=cache)[:, -1]
        if mode == "captured" and arm not in steps:
            steps[arm] = model.capture_step(cache)
        step = steps.get(arm, lambda emb: model(emb, cache=cache))
        for _ in range(new_tokens):
            tok = (y.float() @ table.float().t()).argmax(-1)
            y = step(table[tok][:, None])[:, 0]

    times = {a: [] for a in arms}
    with torch.no_grad():
        for a in arms:   # warm-up (and the captures)
            decode(a)
        torch.cuda.synchronize()
        for r in range(rounds):
            for a in (arms if r % 2 == 0 else arms[::-1]):
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                decode(a)
                e.record()
                torch.cuda.synchronize()
                times[a].append(s.elapsed_time(e) / 1e3)
    tok_s = {a: B * new_tokens / sorted(t)[len(t) // 2] for a, t in times.items()}
    for mode in ("eager", "captured"):
        print(json.dumps({"arm": "decoder", "mode": mode, "B": B, "prompt": prompt_len, "new_tokens": new_tokens,
                          "layers": len(models["rel_pos"].layers),
                          "rel_pos_tok_s": round(tok_s[("rel_pos", mode)], 1),
                          "rotary_tok_s": round(tok_s[("rotary", mode)], 1),
                          "rotary_speedup": round(tok_s[("rotary", mode)] / tok_s[("rel_pos", mode)], 3)}), flush=True)


def train_arm(B, L, iters, rounds):
    models = {cfg: _decoder(cfg, L).train() for cfg in CONFIGS}
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(B, L, E, device="cuda", generator=g).half()
    gy = torch.randn(B, L, E, device="cuda", generator=g).half()

    def step(model):
        model(x).backward(gy)

    med = alternate({cfg: (lambda m=models[cfg]: step(m)) for cfg in CONFIGS}, iters, rounds)
    print(json.dumps({"arm": "train_fwd_bwd", "B": B, "L": L, "layers": len(models["rel_pos"].layers),
                      "rel_pos_ms": round(med["rel_pos"], 3), "rotary_ms": round(med["rotary"], 3),
                      "rotary_speedup": round(med["rel_pos"] / med["rotary"], 3)}), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--e2e-rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, nargs="*", default=[1, 8, 64])
    ap.add_argument("--new-tokens", type=int, default=128)
    ap.add_argument("--skip-kernel", action="store_true")
    ap.add_argument("--skip-decoder", action="store_true")
    ap.add_argument("--skip-train", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("rotary_bench needs a GPU")
    from unicore import ops

    assert ops.USE_NATIVE, "native kernels are not active"
    print("card:", card(), flush=True)
    if not args.skip_kernel:
        kernel_arm(ops, "mha_packed", 32, 512, 36, 24, 64, 0, args.iters, args.rounds)
        kernel_arm(ops, "gqa_packed", 8, 2048, 48, 40, 128, 0, args.iters, args.rounds)
        kernel_arm(ops, "decode_step", 64, 1, 24, 16, 96, 1000, args.iters, args.rounds)
    if not args.skip_decoder:
        for B in args.batch:
            decoder_arm(B, 128, args.new_tokens, args.e2e_rounds)
            torch.cuda.empty_cache()
    if not args.skip_train:
        train_arm(8, 512, max(2, args.iters // 4), args.rounds)


if __name__ == "__main__":
    main()
