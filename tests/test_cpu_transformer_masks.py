"""The stacks hand their layers one mask form on every path: the bias (relative positions ``[1, H, L, L]``, plus a user
``attn_mask`` as ``[B, H, L, L]``) with no ``-inf`` in it, the ``[B, L]`` key padding mask as it is, and for the
auto-regressive decoder ``causal=True``.  On the materialised path (CPU, fp32 / fp64) that form gives the result of the
reference's merged formulation, where everything is one ``[B*H, L, L]`` bias with ``-inf`` at padded keys."""
import copy

import pytest
import torch

from unicore.modules import SelfMultiheadAttention, TransformerDecoder, TransformerEncoder

B, L, E, H, LE = 3, 20, 32, 4, 7


def _stack(decoder, rel_pos, dtype, dropout=0.0):
    torch.manual_seed(1)
    kw = dict(embed_dim=E, ffn_embed_dim=64, attention_heads=H, emb_dropout=dropout, dropout=dropout,
              attention_dropout=dropout, max_seq_len=64, rel_pos=rel_pos)
    m = TransformerDecoder(decoder_layers=2, **kw) if decoder else TransformerEncoder(encoder_layers=2, **kw)
    with torch.no_grad():
        for p in m.parameters():   # non-trivial LayerNorm parameters and biases
            p.add_(torch.randn_like(p) * 0.05)
    return m.to(dtype)


def _padding():
    pad = torch.zeros(B, L, dtype=torch.bool)
    pad[1, L - 5:] = True
    pad[2, L - 1:] = True
    return pad


def _merged_reference(m, emb, attn_mask, pad, encoder):
    """The reference's formulation: ``attn_mask + rel (+ future mask)`` as ``[B*H, L, L]``, ``-inf`` written into the
    padded key columns, no key mask and no ``causal`` flag."""
    x = m._embed_prologue(emb, pad)
    bias = m.get_rel_pos_bias(x).repeat(B, 1, 1) if m.rel_pos else None
    if attn_mask is not None:
        bias = attn_mask.clone() if bias is None else attn_mask + bias
    decoder = isinstance(m, TransformerDecoder)
    if decoder:
        bias = m.get_future_mask(x, bias)
    if bias is not None and pad is not None:
        bias = bias.view(B, -1, L, L).masked_fill(pad[:, None, None, :], float("-inf")).view(-1, L, L)
        pad = None
    for layer in m.layers:
        if decoder:
            x = layer(x, encoder_out=encoder[0], attn_bias=bias, padding_mask=pad, encoder_padding_mask=encoder[1])
        else:
            x = layer(x, attn_bias=bias, padding_mask=pad)
    return m.final_layer_norm(x) if m.final_layer_norm is not None else x


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["fp32", "fp64"])
@pytest.mark.parametrize("padded", [False, True], ids=["no_pad", "pad"])
@pytest.mark.parametrize("with_mask", [False, True], ids=["no_mask", "attn_mask"])
@pytest.mark.parametrize("rel_pos", [False, True], ids=["no_rel", "rel"])
@pytest.mark.parametrize("decoder", [False, True], ids=["encoder", "decoder"])
def test_stack_equals_merged_reference(decoder, rel_pos, with_mask, padded, dtype):
    m = _stack(decoder, rel_pos, dtype)
    ref = copy.deepcopy(m)
    g = torch.Generator().manual_seed(7)
    emb = torch.randn(B, L, E, generator=g, dtype=dtype)
    attn_mask = torch.randn(B * H, L, L, generator=g, dtype=dtype) if with_mask else None
    pad = _padding() if padded else None
    enc = torch.randn(B, LE, E, generator=g, dtype=dtype)
    enc_pad = torch.zeros(B, LE, dtype=torch.bool)
    enc_pad[0, LE - 2:] = True
    dy = torch.randn(B, L, E, generator=g, dtype=dtype)

    e1 = emb.clone().requires_grad_(True)
    if decoder:
        y = m(e1, encoder_out=enc, padding_mask=pad, encoder_padding_mask=enc_pad, attn_mask=attn_mask)
    else:
        y = m(e1, attn_mask=attn_mask, padding_mask=pad)
    y.backward(dy)
    e2 = emb.clone().requires_grad_(True)
    y_ref = _merged_reference(ref, e2, attn_mask, pad, (enc, enc_pad))
    y_ref.backward(dy)

    assert torch.equal(y, y_ref)
    assert torch.equal(e1.grad, e2.grad)
    for (name, p), (_, r) in zip(m.named_parameters(), ref.named_parameters()):
        if p.grad is None:
            assert r.grad is None, name
        elif name == "relative_attention_bias.weight":
            # the batch sum of the bias gradient is the broadcast's here and repeat()'s backward there
            torch.testing.assert_close(p.grad, r.grad)
        else:
            assert torch.equal(p.grad, r.grad), name


@pytest.mark.parametrize("with_mask", [False, True], ids=["no_mask", "attn_mask"])
@pytest.mark.parametrize("decoder", [False, True], ids=["encoder", "decoder"])
def test_layers_get_one_mask_form(monkeypatch, decoder, with_mask):
    calls = []
    attend = SelfMultiheadAttention.attend

    def spy(self, query, key_padding_mask=None, attn_bias=None, return_attn=False, need_probs=True, causal=False,
            cache=None):
        calls.append((key_padding_mask, attn_bias, causal))
        return attend(self, query, key_padding_mask, attn_bias, return_attn, need_probs, causal, cache=cache)

    monkeypatch.setattr(SelfMultiheadAttention, "attend", spy)
    m = _stack(decoder, True, torch.float32)
    pad = _padding()
    attn_mask = torch.randn(B * H, L, L) if with_mask else None
    m(torch.randn(B, L, E), padding_mask=pad, attn_mask=attn_mask)
    assert len(calls) == len(m.layers)
    for kpm, bias, causal in calls:
        assert kpm is pad
        assert bias.shape == ((B if with_mask else 1), H, L, L) and not bool(torch.isinf(bias).any())
        assert causal == decoder


@pytest.mark.parametrize("decoder", [False, True], ids=["encoder", "decoder"])
def test_all_false_padding_equals_none(decoder):
    """With dropout on at a fixed seed: an all-False padding mask gives bitwise the output and gradients of none."""
    m = _stack(decoder, True, torch.float32, dropout=0.1).train()
    emb, dy = torch.randn(B, L, E), torch.randn(B, L, E)
    results = []
    for pad in (None, torch.zeros(B, L, dtype=torch.bool)):
        torch.manual_seed(5)
        e = emb.clone().requires_grad_(True)
        y = m(e, padding_mask=pad)
        y.backward(dy)
        results.append([y, e.grad] + [p.grad.clone() for p in m.parameters() if p.grad is not None])
        m.zero_grad(set_to_none=True)
    a, b = results
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
