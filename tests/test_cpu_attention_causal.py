"""Causal attention on the CPU: ``attention_reference(causal=True)`` is the explicit future-mask formula (top-left
aligned for Lq != Lk, additive in logits mode), and the modules' ``causal`` flag equals passing the future mask as
``attn_bias``."""
import math

import pytest
import torch

from unicore import ops
from unicore.modules import SelfMultiheadAttention, TransformerDecoderLayer
from unicore.modules.transformer import bulid_future_mask


def _qkv(B, H, Lq, Lk, D, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, Lq, H, D, generator=g), torch.randn(B, Lk, H, D, generator=g),
            torch.randn(B, Lk, H, D, generator=g))


@pytest.mark.parametrize("return_logits", [False, True], ids=["plain", "logits"])
@pytest.mark.parametrize("Lq,Lk", [(24, 24), (40, 16), (16, 40)])
def test_reference_equals_explicit_future_mask(Lq, Lk, return_logits):
    B, H, D = 2, 3, 8
    q, k, v = _qkv(B, H, Lq, Lk, D)
    bias = torch.randn(1, H, Lq, Lk)
    kpm = torch.zeros(B, Lk, dtype=torch.bool)
    kpm[0, Lk - 4:] = True
    scale = 1.0 / math.sqrt(D)
    fm = torch.triu(torch.full((Lq, Lk), float("-inf")), 1)
    got = ops.attention_reference(q, k, v, bias, kpm, 0.0, False, scale, return_logits=return_logits, causal=True)
    want = ops.attention_reference(q, k, v, bias + fm, kpm, 0.0, False, scale, return_logits=return_logits)
    if return_logits:
        assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
        assert bool(torch.isinf(got[1][..., fm.isinf()]).all())
    else:
        assert torch.equal(got, want)


def test_reference_causal_logits_gradient_matches_explicit_mask():
    q, k, v = _qkv(1, 2, 16, 24, 8, seed=3)
    fm = torch.triu(torch.full((16, 24), float("-inf")), 1)
    grads = []
    for causal in (True, False):
        x = [t.clone().requires_grad_(True) for t in (q, k, v)]
        out, z = ops.attention_reference(*x, None if causal else fm.expand(1, 2, 16, 24), None, 0.0, False, None,
                                         return_logits=True, causal=causal)
        (out.sum() + z.masked_fill(z.isinf(), 0.0).square().sum()).backward()
        grads.append([t.grad for t in x])
    for a, b in zip(*grads):
        assert torch.equal(a, b)


@pytest.mark.parametrize("with_bias", [False, True], ids=["mask_only", "bias"])
@pytest.mark.parametrize("return_attn", [False, True])
def test_self_attention_causal_equals_future_mask_bias(return_attn, with_bias):
    torch.manual_seed(0)
    attn = SelfMultiheadAttention(32, 4, dropout=0.0).eval()
    L = 12
    x = torch.randn(2, L, 32)
    kpm = torch.zeros(2, L, dtype=torch.bool)
    kpm[1, L - 3:] = True
    bias = torch.randn(1, 4, L, L) if with_bias else None
    fm = bulid_future_mask(L)
    explicit = fm if bias is None else bias + fm
    got = attn(x, key_padding_mask=kpm, attn_bias=bias, return_attn=return_attn, causal=True)
    want = attn(x, key_padding_mask=kpm, attn_bias=explicit, return_attn=return_attn)
    if return_attn:
        for a, b in zip(got, want):
            assert torch.equal(a, b)
    else:
        assert torch.equal(got, want)


def test_decoder_layer_causal_equals_future_mask_bias():
    torch.manual_seed(1)
    layer = TransformerDecoderLayer(32, 64, 4, dropout=0.0, attention_dropout=0.0).eval()
    L, Le = 10, 6
    x, enc = torch.randn(2, L, 32), torch.randn(2, Le, 32)
    pad = torch.zeros(2, L, dtype=torch.bool)
    pad[0, L - 2:] = True
    enc_pad = torch.zeros(2, Le, dtype=torch.bool)
    enc_pad[1, Le - 1:] = True
    rel = torch.randn(1, 4, L, L)
    got = layer(x, encoder_out=enc, attn_bias=rel, padding_mask=pad, encoder_padding_mask=enc_pad, causal=True)
    want = layer(x, encoder_out=enc, attn_bias=rel + bulid_future_mask(L), padding_mask=pad,
                 encoder_padding_mask=enc_pad)
    assert torch.equal(got, want)
