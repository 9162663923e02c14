"""Packed (varlen) vs padded batches of the same sequence pairs through an encoder-decoder, and a decoder-only stack.

One training step = forward + backward + an Adam step over every parameter, fp16, dropout on (the default 0.1):
- encoder-decoder: a 6-layer ``TransformerEncoder`` and a 6-layer ``TransformerDecoder`` at BERT-base widths (768, 12
  heads, ffn 3072), B = 32 pairs, source lengths uniform on [64, 512], target lengths uniform on [16, 256].  The packed
  arm runs the decoder's cross-attention in the varlen kernels with separate key sequences (``cu_seqlens_k``);
- decoder-only: the 6-layer decoder alone (causal self-attention), B = 32, lengths uniform on [64, 512].
The inputs are the embeddings themselves (no token embedding layer); the loss is the mean square of the real output
rows.  Both arms run the same sequences and alternate within one process, so that clock and neighbour noise fall on
both; before timing, their losses are compared in eval mode (dropout off) on the same weights.
Usage: python bench/varlen_decoder_bench.py [--iters 10] [--rounds 5]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from unicore.modules.transformer import TransformerDecoder, TransformerEncoder  # noqa: E402

E, FFN, HEADS, LAYERS, B = 768, 3072, 12, 6, 32


def lengths(lo, hi, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(lo, hi + 1, (B,), generator=g).tolist()


def cu_of(lens):
    return torch.tensor([0] + lens, device="cuda").cumsum(0).to(torch.int32)


def pad_mask(lens, L):
    return torch.arange(L, device="cuda")[None, :] >= torch.tensor(lens, device="cuda")[:, None]


def real_rows(lens, L):
    """flat indices of the real rows of a [B, L] batch, in packed order"""
    return (~pad_mask(lens, L)).reshape(-1).nonzero().squeeze(1)


def scatter(x, lens, L):
    out = x.new_zeros(len(lens), L, *x.shape[1:])
    out.view(-1, *x.shape[1:])[real_rows(lens, L)] = x
    return out


def timed(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def alternate(arms, iters, rounds):
    for fn in arms.values():   # warm-up of every shape
        fn()
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            times[k].append(timed(fn, iters))
    return {k: sorted(v)[len(v) // 2] for k, v in times.items()}


def stack(cls, max_seq_len):
    kw = dict(embed_dim=E, ffn_embed_dim=FFN, attention_heads=HEADS, max_seq_len=max_seq_len)
    layers = {"encoder_layers": LAYERS} if cls is TransformerEncoder else {"decoder_layers": LAYERS}
    return cls(**layers, **kw).cuda().half()


def case(name, encoder, src_lens, Ls, tgt_lens, Lt, iters, rounds):
    torch.manual_seed(0)
    enc = stack(TransformerEncoder, Ls) if encoder else None
    dec = stack(TransformerDecoder, max(Ls, Lt))
    params = list(dec.parameters()) + (list(enc.parameters()) if encoder else [])
    opt = torch.optim.Adam(params, lr=1e-5, eps=1e-4)
    g = torch.Generator(device="cuda").manual_seed(1)
    tgt = torch.randn(sum(tgt_lens), E, device="cuda", generator=g, dtype=torch.float16)
    src = torch.randn(sum(src_lens), E, device="cuda", generator=g, dtype=torch.float16) if encoder else None
    cu_t, pad_t, rows_t = cu_of(tgt_lens), pad_mask(tgt_lens, Lt), real_rows(tgt_lens, Lt)
    tgtp = scatter(tgt, tgt_lens, Lt)
    if encoder:
        cu_s, pad_s = cu_of(src_lens), pad_mask(src_lens, Ls)
        srcp = scatter(src, src_lens, Ls)

    def loss_packed():
        kw = {}
        enc_out = None
        if encoder:
            enc_out = enc(src, cu_seqlens=cu_s, max_seqlen=Ls)
            kw = dict(encoder_cu_seqlens=cu_s, encoder_max_seqlen=Ls)
        y = dec(tgt, encoder_out=enc_out, cu_seqlens=cu_t, max_seqlen=Lt, **kw)
        return y.float().square().mean()

    def loss_padded():
        enc_out = enc(srcp, padding_mask=pad_s) if encoder else None
        y = dec(tgtp, encoder_out=enc_out, padding_mask=pad_t, encoder_padding_mask=pad_s if encoder else None)
        return y.reshape(-1, E)[rows_t].float().square().mean()

    modules = [dec] + ([enc] if encoder else [])
    for m in modules:
        m.eval()
    with torch.no_grad():
        losses = {"packed": float(loss_packed()), "padded": float(loss_padded())}
    for m in modules:
        m.train()

    def step(loss_fn):
        def run():
            opt.zero_grad(set_to_none=True)
            loss_fn().backward()
            opt.step()
        return run

    t = alternate({"packed": step(loss_packed), "padded": step(loss_padded)}, iters, rounds)
    N = sum(tgt_lens) + (sum(src_lens) if encoder else 0)
    return {"case": name, "dtype": "float16", "B": B, "src_L": Ls if encoder else None, "tgt_L": Lt,
            "real_tokens": N, "padded_tokens": B * (Lt + (Ls if encoder else 0)),
            "packed_ms": round(t["packed"], 3), "padded_ms": round(t["padded"], 3),
            "speedup": round(t["padded"] / t["packed"], 3),
            "packed_samples_per_s": round(B / t["packed"] * 1e3, 1), "padded_samples_per_s": round(B / t["padded"] * 1e3, 1),
            "eval_loss_packed": losses["packed"], "eval_loss_padded": losses["padded"],
            "eval_loss_rel_diff": abs(losses["packed"] - losses["padded"]) / abs(losses["padded"])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("varlen_decoder_bench needs a GPU")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": card}))
    print(json.dumps(case("encoder_decoder_train_step", True, lengths(64, 512, 0), 512, lengths(16, 256, 1), 256,
                          args.iters, args.rounds)), flush=True)
    print(json.dumps(case("decoder_only_train_step", False, None, 0, lengths(64, 512, 2), 512, args.iters,
                          args.rounds)), flush=True)


if __name__ == "__main__":
    main()
