"""The logits mode of the attention ops on the reference path (CPU): ``(out, logits)`` with an additive key mask whose
gradient reaches the masked keys, and ``need_probs=False`` on the attention module and the encoder layer."""
import copy
import math

import torch

from unicore import ops


def _inputs(B=2, H=3, Lq=10, Lk=12, D=8, seed=0, bias_batch=1):
    g = torch.Generator().manual_seed(seed)
    q, k, v = (torch.randn(B, L, H, D, generator=g).requires_grad_(True) for L in (Lq, Lk, Lk))
    bias = torch.randn(bias_batch, H, Lq, Lk, generator=g).requires_grad_(True)
    kpm = torch.zeros(B, Lk, dtype=torch.bool)
    kpm[0, 9:] = True
    return q, k, v, bias, kpm


def test_reference_returns_logits_with_additive_mask():
    q, k, v, bias, kpm = _inputs()
    scale = 1.0 / math.sqrt(q.shape[-1])
    out, z = ops.attention_reference(q, k, v, bias, kpm, 0.0, False, scale, return_logits=True)
    plain = ops.attention_reference(q, k, v, bias, kpm, 0.0, False, scale)
    assert torch.equal(out, plain)
    zf = torch.einsum("bqhd,bkhd->bhqk", q, k) * scale + bias
    assert z.shape == (2, 3, 10, 12)
    assert torch.isinf(z[0, :, :, 9:]).all() and torch.isfinite(z[0, :, :, :9]).all() and torch.isfinite(z[1]).all()
    fin = torch.isfinite(z)
    assert torch.allclose(z[fin], zf.expand_as(z)[fin], atol=1e-6)


def test_reference_logits_gradient_reaches_masked_keys():
    """dz flows through z = scale * q k^T + bias + mask at every position, masked keys included."""
    q, k, v, bias, kpm = _inputs(seed=1, bias_batch=2)
    scale = 0.3
    out, z = ops.attention_reference(q, k, v, bias, kpm, 0.0, False, scale, return_logits=True)
    dout, dz = torch.randn_like(out), torch.randn_like(z)
    torch.autograd.backward([out, z], [dout, dz])
    qr, kr, vr, br = (t.detach().clone().requires_grad_(True) for t in (q, k, v, bias))
    s = torch.einsum("bqhd,bkhd->bhqk", qr, kr) * scale + br
    pad = torch.zeros(kpm.shape).masked_fill(kpm, float("-inf"))[:, None, None, :]
    zr = s + pad
    o_r = torch.einsum("bhqk,bkhd->bqhd", torch.softmax(zr, -1), vr)
    torch.autograd.backward([o_r, zr], [dout, dz])
    for g, gr in ((q.grad, qr.grad), (k.grad, kr.grad), (v.grad, vr.grad), (bias.grad, br.grad)):
        assert torch.allclose(g, gr, atol=1e-5)
    # at masked keys the bias gradient is exactly dz (the softmax contributes nothing there)
    assert torch.equal(bias.grad[0, :, :, 9:], dz[0, :, :, 9:])


def test_fused_attention_falls_back_with_logits_on_cpu():
    q, k, v, bias, kpm = _inputs(seed=2)
    out, z = ops.fused_attention(q, k, v, bias=bias, key_padding_mask=kpm, dropout_p=0.0, training=False,
                                 return_logits=True)
    ref_out, ref_z = ops.attention_reference(q, k, v, bias, kpm, 0.0, False, None, return_logits=True)
    assert torch.equal(out, ref_out) and torch.equal(z, ref_z)
    qkv = torch.stack([q.detach(), k.detach()[:, :10], v.detach()[:, :10]], dim=2)
    out_p, z_p = ops.fused_attention_qkvpacked(qkv, bias=bias.detach()[..., :10], dropout_p=0.0, training=False,
                                               return_logits=True)
    assert out_p.shape == (2, 10, 3, 8) and z_p.shape == (2, 3, 10, 10)


def test_attention_module_need_probs_false():
    from unicore.modules import SelfMultiheadAttention

    torch.manual_seed(3)
    attn = SelfMultiheadAttention(32, 4, dropout=0.0).eval()
    x = torch.randn(2, 8, 32)
    bias = torch.randn(2 * 4, 8, 8)
    pad = torch.zeros(2, 8, dtype=torch.bool)
    pad[1, 6:] = True
    o, z, probs = attn(x, key_padding_mask=pad, attn_bias=bias, return_attn=True)
    o2, z2, probs2 = attn(x, key_padding_mask=pad, attn_bias=bias, return_attn=True, need_probs=False)
    assert probs is not None and probs2 is None
    assert torch.equal(o, o2) and torch.equal(z, z2)


def test_encoder_layer_need_probs_false():
    from unicore.modules import TransformerEncoderLayer

    torch.manual_seed(4)
    layer = TransformerEncoderLayer(32, 64, 4, dropout=0.0, attention_dropout=0.0).eval()
    ref = copy.deepcopy(layer)
    x = torch.randn(2, 8, 32, requires_grad=True)
    xr = x.detach().clone().requires_grad_(True)
    bias = torch.randn(2 * 4, 8, 8)
    y, z, probs = layer(x, attn_bias=bias, return_attn=True, need_probs=False)
    yr, zr, probs_r = ref(xr, attn_bias=bias, return_attn=True)
    assert probs is None and probs_r.shape == (8, 8, 8)
    assert torch.equal(y, yr) and torch.equal(z, zr)
    dz = torch.randn_like(z)
    torch.autograd.backward([y, z], [torch.ones_like(y), dz])
    torch.autograd.backward([yr, zr], [torch.ones_like(yr), dz])
    assert torch.equal(x.grad, xr.grad)
