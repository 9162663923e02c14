"""Grouped-query attention on the CPU (fp32, the PyTorch references and the materialised module paths).

The references expand the shared key / value heads with ``repeat_interleave``, so a call with ``H_kv`` heads equals
the same call on the expanded tensors.  The modules take ``num_kv_heads`` / ``attention_kv_heads``; the default keeps
every parameter, and a head count that does not divide raises ``ValueError``."""
import pytest
import torch

from unicore import ops
from unicore.modules import CrossMultiheadAttention, SelfMultiheadAttention, TransformerDecoder
from unicore.modules.transformer import TransformerEncoder

E = 64


def _expand(t, G):
    return t.repeat_interleave(G, dim=2)


@pytest.mark.parametrize("H,H_kv", [(12, 6), (12, 4), (12, 1), (8, 2)])
def test_reference_equals_explicit_expansion(H, H_kv):
    g = torch.Generator().manual_seed(H * 10 + H_kv)
    B, Lq, Lk, D = 2, 9, 11, 8
    q = torch.randn(B, Lq, H, D, generator=g)
    k, v = torch.randn(B, Lk, H_kv, D, generator=g), torch.randn(B, Lk, H_kv, D, generator=g)
    bias = torch.randn(1, H, Lq, Lk, generator=g)
    kpm = torch.zeros(B, Lk, dtype=torch.bool)
    kpm[1, -3:] = True
    G = H // H_kv
    for kw in ({}, {"bias": bias, "key_padding_mask": kpm}, {"causal": True}, {"bias": bias, "return_logits": True}):
        got = ops.attention_reference(q, k, v, dropout_p=0.0, **kw)
        want = ops.attention_reference(q, _expand(k, G), _expand(v, G), dropout_p=0.0, **kw)
        for a, b in zip(got if isinstance(got, tuple) else (got,), want if isinstance(want, tuple) else (want,)):
            assert torch.equal(a, b), kw
    torch.manual_seed(3)
    got = ops.attention_reference(q, k, v, dropout_p=0.3)
    torch.manual_seed(3)
    want = ops.attention_reference(q, _expand(k, G), _expand(v, G), dropout_p=0.3)
    assert torch.equal(got, want)


@pytest.mark.parametrize("T", [1, 5])
def test_kv_cache_reference_equals_explicit_expansion(T):
    g = torch.Generator().manual_seed(T)
    B, C, H, H_kv, D = 3, 16, 8, 2, 8
    q = torch.randn(B, T, H, D, generator=g)
    k, v = torch.randn(B, C, H_kv, D, generator=g), torch.randn(B, C, H_kv, D, generator=g)
    kn, vn = torch.randn(B, T, H_kv, D, generator=g), torch.randn(B, T, H_kv, D, generator=g)
    seqlens = torch.tensor([0, 4, 9], dtype=torch.int32)
    bias = torch.randn(1, H, T, C, generator=g)
    ke, ve = _expand(k, 4), _expand(v, 4)
    got = ops.attention_with_kv_cache(q, k, v, seqlens, 10, k_new=kn, v_new=vn, bias=bias)
    want = ops.attention_with_kv_cache(q, ke, ve, seqlens, 10, k_new=_expand(kn, 4), v_new=_expand(vn, 4), bias=bias)
    assert torch.equal(got, want)
    assert torch.equal(_expand(k, 4), ke) and torch.equal(_expand(v, 4), ve)   # the same rows were appended
    got = ops.attention_with_kv_cache(q, k, v)                                 # cross-attention: all C rows
    assert torch.equal(got, ops.attention_with_kv_cache(q, ke, ve))


def test_self_attention_fallback_matches_expanded_heads():
    torch.manual_seed(0)
    H, H_kv = 8, 2
    m = SelfMultiheadAttention(E, H, dropout=0.0, num_kv_heads=H_kv)
    D = E // H
    assert m.in_proj.weight.shape == ((H + 2 * H_kv) * D, E)
    x = torch.randn(2, 7, E, requires_grad=True)
    kpm = torch.zeros(2, 7, dtype=torch.bool)
    kpm[0, -2:] = True
    for causal in (False, True):
        out = m(x, key_padding_mask=kpm, causal=causal)
        qkv = torch.nn.functional.linear(x, m.in_proj.weight, m.in_proj.bias).view(2, 7, H + 2 * H_kv, D)
        q, k, v = qkv[:, :, :H], qkv[:, :, H:H + H_kv], qkv[:, :, H + H_kv:]
        ref = ops.attention_reference(q, k, v, key_padding_mask=kpm, dropout_p=0.0, scale=m.scaling, causal=causal)
        ref = m.out_proj(ref.reshape(2, 7, E))
        torch.testing.assert_close(out, ref, atol=1e-5, rtol=1e-5)
        gy = torch.randn_like(out)
        got = torch.autograd.grad(out, [x, m.in_proj.weight], gy)
        want = torch.autograd.grad(ref, [x, m.in_proj.weight], gy)
        for a, b in zip(got, want):
            torch.testing.assert_close(a, b, atol=1e-5, rtol=1e-5)
    o, logits, probs = m(x, return_attn=True)
    assert logits.shape == (2 * H, 7, 7) and probs.shape == (2 * H, 7, 7)


def test_cross_attention_fallback_matches_expanded_heads():
    torch.manual_seed(1)
    H, H_kv = 8, 1
    m = CrossMultiheadAttention(E, H, dropout=0.0, num_kv_heads=H_kv)
    D = E // H
    assert m.k_proj.weight.shape == (H_kv * D, E) and m.v_proj.weight.shape == (H_kv * D, E)
    x, enc = torch.randn(2, 5, E), torch.randn(2, 6, E, requires_grad=True)
    out = m(x, enc, enc)
    q = m.q_proj(x).view(2, 5, H, D)
    k, v = m.k_proj(enc).view(2, 6, H_kv, D), m.v_proj(enc).view(2, 6, H_kv, D)
    ref = m.out_proj(ops.attention_reference(q, k, v, dropout_p=0.0, scale=m.scaling).reshape(2, 5, E))
    torch.testing.assert_close(out, ref, atol=1e-5, rtol=1e-5)
    gy = torch.randn_like(out)
    torch.testing.assert_close(torch.autograd.grad(out, [enc, m.k_proj.weight], gy),
                               torch.autograd.grad(ref, [enc, m.k_proj.weight], gy), atol=1e-5, rtol=1e-5)


def _shapes(m):
    return {k: tuple(v.shape) for k, v in m.state_dict().items()}


def test_default_kv_heads_keep_state_dict():
    torch.manual_seed(0)
    base = _shapes(SelfMultiheadAttention(E, 4))
    assert base["in_proj.weight"] == (3 * E, E) and base["in_proj.bias"] == (3 * E,)
    assert _shapes(SelfMultiheadAttention(E, 4, num_kv_heads=4)) == base
    cross = _shapes(CrossMultiheadAttention(E, 4))
    assert cross["k_proj.weight"] == (E, E) and _shapes(CrossMultiheadAttention(E, 4, num_kv_heads=4)) == cross
    kw = dict(embed_dim=E, ffn_embed_dim=2 * E, attention_heads=4, max_seq_len=32)
    for cls, n in ((TransformerDecoder, "decoder_layers"), (TransformerEncoder, "encoder_layers")):
        torch.manual_seed(0)
        a = cls(**{n: 2}, **kw)
        torch.manual_seed(0)
        b = cls(**{n: 2}, attention_kv_heads=None, **kw)
        torch.manual_seed(0)
        c = cls(**{n: 2}, attention_kv_heads=4, **kw)
        assert _shapes(a) == _shapes(b) == _shapes(c)
        for k, v in a.state_dict().items():   # the same initialisation, parameter by parameter
            assert torch.equal(v, b.state_dict()[k]) and torch.equal(v, c.state_dict()[k]), k
    gqa = _shapes(TransformerDecoder(decoder_layers=1, attention_kv_heads=2, **kw))
    assert gqa["layers.0.self_attn.in_proj.weight"] == ((4 + 2 * 2) * 16, E)
    assert gqa["layers.0.encoder_attn.k_proj.weight"] == (2 * 16, E)


def test_non_dividing_head_count_raises():
    with pytest.raises(ValueError, match="divide"):
        SelfMultiheadAttention(E, 8, num_kv_heads=3)
    with pytest.raises(ValueError, match="divide"):
        CrossMultiheadAttention(E, 8, num_kv_heads=5)
    with pytest.raises(ValueError, match="divide"):
        TransformerDecoder(decoder_layers=1, embed_dim=E, attention_heads=4, attention_kv_heads=3)
    q, k = torch.randn(1, 8, 6, 8), torch.randn(1, 8, 4, 8)
    for fn in (ops.attention_reference, ops.fused_attention):
        with pytest.raises(ValueError, match="divide"):
            fn(q, k, k)
    with pytest.raises(ValueError, match="same number of heads"):
        ops.fused_attention(q, k, torch.randn(1, 8, 2, 8))
    with pytest.raises(ValueError, match="divide"):
        ops.attention_with_kv_cache(q[:, :1], k, k)
    with pytest.raises(ValueError, match="divide"):
        ops.attention_with_kv_cache_reference(q[:, :1], k, k)
    with pytest.raises(ValueError, match="divide"):
        ops.fused_attention_qkvpacked(torch.randn(1, 8, 12, 8), num_kv_heads=5)   # 2 query heads, 5 kv heads
    with pytest.raises(ValueError, match="num_kv_heads"):
        ops.fused_attention_qkvpacked(torch.randn(1, 8, 12, 8))


def test_packed_reference_path_slices_heads():
    g = torch.Generator().manual_seed(2)
    qkv = torch.randn(2, 8, 6 + 2 * 3, 8, generator=g)
    got = ops.fused_attention_qkvpacked(qkv, dropout_p=0.0, num_kv_heads=3)
    want = ops.attention_reference(qkv[:, :, :6], qkv[:, :, 6:9], qkv[:, :, 9:], dropout_p=0.0)
    assert torch.equal(got, want)


def _gqa_decoder(seed=0):
    torch.manual_seed(seed)
    m = TransformerDecoder(decoder_layers=2, embed_dim=E, ffn_embed_dim=2 * E, attention_heads=4, max_seq_len=64,
                           attention_kv_heads=2).eval()
    with torch.no_grad():
        for p in m.parameters():
            p.add_(torch.randn_like(p) * 0.02)
    return m


def test_gqa_decoder_steps_match_full_forward():
    m = _gqa_decoder()
    g = torch.Generator().manual_seed(1)
    B, L, steps = 2, 5, 6
    tokens, enc = torch.randn(B, L + steps + 4, E, generator=g), torch.randn(B, 6, E, generator=g)
    with torch.no_grad():
        cache = m.new_cache(B, 32)
        assert cache.layers[0].k.shape == (B, 32, 2, E // 4)
        m(tokens[:, :L], encoder_out=enc, cache=cache)
        for t in range(steps):
            y = m(tokens[:, L + t:L + t + 1], cache=cache)
            full = m(tokens[:, :L + t + 1], encoder_out=enc)
            torch.testing.assert_close(y[:, 0], full[:, -1], atol=2e-5, rtol=2e-5)
        y = m(tokens[:, L + steps:L + steps + 4], cache=cache)   # a chunk of 4
        full = m(tokens[:, :L + steps + 4], encoder_out=enc)
        torch.testing.assert_close(y, full[:, -4:], atol=2e-5, rtol=2e-5)
        cache.rewind(4)
        cache.reorder(torch.tensor([1, 0]))
        y = m(tokens[[1, 0], L + steps:L + steps + 1], cache=cache)
        full = m(tokens[[1, 0], :L + steps + 1], encoder_out=enc[[1, 0]])
        torch.testing.assert_close(y[:, 0], full[:, -1], atol=2e-5, rtol=2e-5)
