"""Rotary position embeddings on the CPU (fp32: the PyTorch formula of ``ops.rotary_embedding`` and the module paths).

The formula is checked against an fp64 implementation on the same fp32 angles; attention with rotary depends on
relative positions only; the modules validate ``rotary_dim``, keep their ``state_dict`` keys, and decode incrementally
(prefill, one-token steps, chunks, ``reorder``, ``rewind``) to the outputs of the full forward."""
import pytest
import torch

from unicore import ops
from unicore.modules import SelfMultiheadAttention, TransformerDecoder
from unicore.modules.transformer import TransformerDecoderLayer, TransformerEncoder, TransformerEncoderLayer

E = 64


def rotary_fp64(x, inv_freq, R, offsets=None, inverse=False):
    """The rotate-half rotation in fp64 at the fp32 angles fl32(float(pos) * inv_freq[i])."""
    B, L, N, D = x.shape
    half = inv_freq.numel()
    pos = torch.arange(L).view(1, L) + (offsets.long().view(-1, 1) if offsets is not None else 0)
    theta = (pos.float()[..., None] * inv_freq.float()).double()[:, :, None, :]
    c, s = theta.cos(), theta.sin() * (-1 if inverse else 1)
    y = x.double().clone()
    x1, x2 = y[:, :, :R, :half].clone(), y[:, :, :R, half:2 * half].clone()
    y[:, :, :R, :half] = x1 * c - x2 * s
    y[:, :, :R, half:2 * half] = x2 * c + x1 * s
    return y


@pytest.mark.parametrize("N,R,D,rd", [(6, 4, 16, 16), (6, 4, 16, 6), (12, 10, 8, 8), (3, 3, 10, 2)],
                         ids=["mha_full", "mha_partial", "gqa", "all_heads_rd2"])
@pytest.mark.parametrize("offsets", [False, True], ids=["no_offsets", "offsets"])
def test_fallback_matches_fp64(N, R, D, rd, offsets):
    g = torch.Generator().manual_seed(N * 100 + D + rd)
    B, L = 3, 7
    x = torch.randn(B, L, N, D, generator=g)
    inv = ops.rotary_inv_freq(rd)
    off = torch.tensor([0, 5, 1000], dtype=torch.int32) if offsets else None
    y = ops.rotary_embedding(x, inv, R, off)
    want = rotary_fp64(x, inv, R, off)
    torch.testing.assert_close(y.double(), want, atol=1e-5, rtol=1e-5)
    assert torch.equal(y[:, :, R:], x[:, :, R:])                 # value heads untouched
    assert torch.equal(y[:, :, :R, rd:], x[:, :, :R, rd:])       # columns past rd untouched
    back = ops.rotary_embedding_reference(y, inv, R, off, inverse=True)
    torch.testing.assert_close(back, x, atol=1e-5, rtol=1e-5)


def test_inv_freq_and_gradient():
    inv = ops.rotary_inv_freq(8, base=500.0)
    assert inv.dtype == torch.float32
    assert torch.equal(inv, 1.0 / (500.0 ** (torch.arange(0, 8, 2, dtype=torch.float32) / 8)))
    x = torch.randn(2, 5, 3, 8, dtype=torch.float64, requires_grad=True)
    off = torch.tensor([3, 9], dtype=torch.int32)
    gy = torch.randn(2, 5, 3, 8, dtype=torch.float64)
    (gx,) = torch.autograd.grad(ops.rotary_embedding(x, inv, 2, off), x, gy)
    torch.testing.assert_close(gx, rotary_fp64(gy, inv, 2, off, inverse=True))


def test_attention_is_shift_invariant():
    """q . k after rotation depends on the position difference only: one offset added to every position leaves the
    attention output unchanged within fp32 rounding."""
    g = torch.Generator().manual_seed(0)
    B, L, H, D = 2, 9, 4, 16
    qkv = torch.randn(B, L, 3 * H, D, generator=g)
    inv = ops.rotary_inv_freq(D)
    outs = []
    for shift in (0, 37, 1000):
        r = ops.rotary_embedding(qkv, inv, 2 * H, torch.full((B,), shift, dtype=torch.int32))
        outs.append(ops.attention_reference(r[:, :, :H], r[:, :, H:2 * H], r[:, :, 2 * H:], dropout_p=0.0,
                                            causal=True))
    for o in outs[1:]:
        torch.testing.assert_close(o, outs[0], atol=2e-5, rtol=2e-5)


def test_invalid_arguments_raise():
    for rd in (3, 0, 18, -2):
        with pytest.raises(ValueError, match="rotary_dim"):
            SelfMultiheadAttention(E, 4, rotary_dim=rd)   # head_dim 16
    with pytest.raises(ValueError, match="rotary_dim"):
        TransformerDecoder(decoder_layers=1, embed_dim=E, attention_heads=4, rotary_dim=7)
    with pytest.raises(ValueError, match="rotary_dim"):
        TransformerEncoderLayer(embed_dim=E, attention_heads=4, rotary_dim=32)
    with pytest.raises(ValueError, match="rotary_dim"):
        ops.rotary_inv_freq(5)
    x = torch.randn(1, 2, 3, 8)
    with pytest.raises(ValueError, match="rotated_heads"):
        ops.rotary_embedding(x, ops.rotary_inv_freq(8), 4)
    with pytest.raises(ValueError, match="inv_freq"):
        ops.rotary_embedding(x, ops.rotary_inv_freq(10))
    with pytest.raises(ValueError, match="position_offsets"):
        ops.rotary_embedding(x, ops.rotary_inv_freq(8), 3, torch.zeros(2, dtype=torch.int32))
    with pytest.raises(ValueError, match=r"\[B, L, N, D\]"):
        ops.rotary_embedding(x[0], ops.rotary_inv_freq(8))


def test_state_dict_keys_unchanged_and_strict_load():
    kw = dict(embed_dim=E, ffn_embed_dim=2 * E, attention_heads=4, max_seq_len=32)
    for cls, n in ((TransformerDecoder, "decoder_layers"), (TransformerEncoder, "encoder_layers")):
        torch.manual_seed(0)
        plain = cls(**{n: 2}, **kw)
        torch.manual_seed(0)
        rot = cls(**{n: 2}, rotary_dim=8, **kw)
        assert plain.state_dict().keys() == rot.state_dict().keys()
        rot.load_state_dict(plain.state_dict(), strict=True)
        plain.load_state_dict(rot.state_dict(), strict=True)
        assert rot.layers[0].self_attn.inv_freq.dtype == torch.float32
    assert not hasattr(TransformerDecoderLayer(embed_dim=E, attention_heads=4).encoder_attn, "inv_freq")
    m = SelfMultiheadAttention(E, 4, rotary_dim=16).half()     # a dtype cast keeps the fp32 frequencies
    assert m.inv_freq.dtype == torch.float32 and torch.equal(m.inv_freq, ops.rotary_inv_freq(16))


def test_module_rotates_q_and_k_only():
    torch.manual_seed(0)
    H, H_kv, D = 8, 2, E // 8
    for kv in (None, H_kv):
        m = SelfMultiheadAttention(E, H, dropout=0.0, num_kv_heads=kv, rotary_dim=6)
        Hk = kv or H
        x = torch.randn(2, 7, E, requires_grad=True)
        out = m(x, causal=True)
        qkv = torch.nn.functional.linear(x, m.in_proj.weight, m.in_proj.bias).view(2, 7, H + 2 * Hk, D)
        r = rotary_fp64(qkv, m.inv_freq, H + Hk).float()
        ref = ops.attention_reference(r[:, :, :H], r[:, :, H:H + Hk], r[:, :, H + Hk:], dropout_p=0.0,
                                      scale=m.scaling, causal=True)
        ref = m.out_proj(ref.reshape(2, 7, E))
        torch.testing.assert_close(out, ref, atol=1e-5, rtol=1e-5)
        gy = torch.randn_like(out)
        got = torch.autograd.grad(out, [x, m.in_proj.weight], gy)
        r = ops.rotary_embedding_reference(qkv, m.inv_freq, H + Hk)
        ref = m.out_proj(ops.attention_reference(r[:, :, :H], r[:, :, H:H + Hk], r[:, :, H + Hk:], dropout_p=0.0,
                                                 scale=m.scaling, causal=True).reshape(2, 7, E))
        want = torch.autograd.grad(ref, [x, m.in_proj.weight], gy)
        for a, b in zip(got, want):
            torch.testing.assert_close(a, b, atol=1e-5, rtol=1e-5)


def _decoder(rel_pos, kv_heads, seed=0):
    torch.manual_seed(seed)
    m = TransformerDecoder(decoder_layers=2, embed_dim=E, ffn_embed_dim=2 * E, attention_heads=4, max_seq_len=64,
                           rel_pos=rel_pos, attention_kv_heads=kv_heads, rotary_dim=12).eval()
    with torch.no_grad():
        for p in m.parameters():
            p.add_(torch.randn_like(p) * 0.02)
    return m


@pytest.mark.parametrize("rel_pos,kv_heads", [(False, None), (True, None), (False, 2)],
                         ids=["rotary", "rotary_rel_pos", "rotary_gqa"])
def test_decoder_steps_match_full_forward(rel_pos, kv_heads):
    m = _decoder(rel_pos, kv_heads)
    g = torch.Generator().manual_seed(1)
    B, steps = 3, 4
    lens = [5, 3, 6]
    L = max(lens)
    tokens, enc = torch.randn(B, 32, E, generator=g), torch.randn(B, 6, E, generator=g)
    prompt = torch.zeros(B, L, E)
    pad = torch.ones(B, L, dtype=torch.bool)
    for b, n in enumerate(lens):
        prompt[b, :n] = tokens[b, :n]
        pad[b, :n] = False

    def full(b, upto, order=None):
        seq = tokens if order is None else tokens[order]
        e = enc if order is None else enc[order]
        return m(seq[b:b + 1, :upto], encoder_out=e[b:b + 1])

    with torch.no_grad():
        cache = m.new_cache(B, 32)
        y = m(prompt, encoder_out=enc, padding_mask=pad, cache=cache)
        for b, n in enumerate(lens):
            torch.testing.assert_close(y[b, :n], full(b, n)[0], atol=2e-5, rtol=2e-5)
        pos = list(lens)

        def feed(T, order=None):
            seq = tokens if order is None else tokens[order]
            emb = torch.stack([seq[b, pos[b]:pos[b] + T] for b in range(B)])
            y = m(emb, cache=cache)
            for b in range(B):
                pos[b] += T
                torch.testing.assert_close(y[b], full(b, pos[b], order)[0, -T:], atol=3e-5, rtol=3e-5)

        for _ in range(steps):
            feed(1)
        feed(3)                                   # a chunk
        cache.rewind(2)
        pos = [p - 2 for p in pos]
        feed(1)
        order = torch.tensor([2, 0, 1])
        cache.reorder(order)
        pos = [pos[i] for i in order.tolist()]
        feed(2, order)
        feed(1, order)
