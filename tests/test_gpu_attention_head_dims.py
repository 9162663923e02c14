"""Fused attention at every head dim the kernels take (D % 8 == 0, 8 <= D <= 128): forward, LSE and backward against
an fp32 reference, the packed entry point, the dropout keep mask, grids of more than one wave, the attention modules
and the encoder stack at head dims other than 64, and the head dims that must fall back to the reference."""
import copy
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

HEAD_DIMS = [8, 16, 32, 40, 64, 80, 96, 128]
DTYPES = [torch.float16, torch.bfloat16]


def _ops():
    from unicore import ops

    assert ops.USE_NATIVE
    return ops


def _ref(q, k, v, bias, kpm, scale, keep=None, p=0.0):
    """fp32 reference; q,k,v [B, L, H, D]; keep: optional [B, H, Lq, Lk] dropout keep mask. Returns (O, LSE)."""
    qf, kf, vf = q.float(), k.float(), v.float()
    s = torch.einsum("bqhd,bkhd->bhqk", qf, kf) * scale
    if bias is not None:
        s = s + bias.float()
    if kpm is not None:
        s = s.masked_fill(kpm[:, None, None, :], float("-inf"))
    pr = torch.softmax(s, dim=-1)
    lse = torch.logsumexp(s, dim=-1)
    if keep is not None:
        pr = pr * keep / (1 - p)
    return torch.einsum("bhqk,bkhd->bqhd", pr, vf), lse


def _qkv(B, H, Lq, Lk, D, dtype, seed, amp=0.8):
    g = torch.Generator(device="cuda").manual_seed(seed)

    def rnd(L):
        return (torch.randn(B, L, H, D, device="cuda", generator=g) * amp).to(dtype).requires_grad_(True)

    return rnd(Lq), rnd(Lk), rnd(Lk)


def _tol(dtype):
    return 1e-2 if dtype == torch.float16 else 6e-2


def _keep_mask_by_probes(q, k, p, scale, seed, bias=None, kpm=None):
    """The forward kernel's dropout keep mask [B, H, Lq, Lk], read back through value probes: with v = e_d at key
    blk * D + d, output column d is P_drop of that key (same seed -> same Philox stream).  D keys per probe pass."""
    ops = _ops()
    B, Lk, H, D = k.shape
    masks = []
    for blk in range((Lk + D - 1) // D):
        n = min(D, Lk - blk * D)
        eye = torch.zeros(B, Lk, H, D, device="cuda", dtype=q.dtype)
        idx = torch.arange(n, device="cuda")
        eye[:, blk * D + idx, :, idx] = 1
        torch.manual_seed(seed)
        pd = ops.fused_attention(q.detach(), k.detach(), eye, bias=None if bias is None else bias.detach(),
                                 key_padding_mask=kpm, dropout_p=p, training=True, scale=scale)
        masks.append(pd.permute(0, 2, 1, 3)[..., :n])
    return (torch.cat(masks, dim=-1) != 0).float()


@pytest.mark.parametrize("D", HEAD_DIMS)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("shape", [(2, 2, 200, 72), (1, 2, 640, 1000)])
@pytest.mark.parametrize("with_bias,with_mask", [(False, False), (True, False), (True, True)])
def test_forward_and_lse(D, dtype, shape, with_bias, with_mask):
    ops = _ops()
    B, H, Lq, Lk = shape
    q, k, v = _qkv(B, H, Lq, Lk, D, dtype, seed=D)
    bias = torch.randn(1, H, Lq, Lk, device="cuda").to(dtype) if with_bias else None
    kpm = None
    if with_mask:
        kpm = torch.zeros(B, Lk, dtype=torch.bool, device="cuda")
        kpm[0, Lk - Lk // 4:] = True
    assert ops.fused_attention_supported(q, k, v, bias, kpm)
    scale = 1.0 / math.sqrt(D)
    with torch.no_grad():
        out, lse, bits = ops.native().fmha_fwd(q, k, v, bias, kpm, 0.0, scale)
        ref, ref_lse = _ref(q, k, v, bias, kpm, scale)
    assert out.shape == (B, Lq, H, D) and out.is_contiguous() and bits is None
    assert (out.float() - ref).abs().max().item() < (4e-3 if dtype == torch.float16 else 2e-2)
    assert (lse - ref_lse).abs().max().item() < 1e-3 * max(1.0, ref_lse.abs().max().item())


@pytest.mark.parametrize("D", HEAD_DIMS)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("p", [0.0, 0.25])
def test_backward_ragged(D, dtype, p):
    """Lq != Lk, neither a multiple of the tiles; per-batch bias with its gradient, key padding, dropout."""
    ops = _ops()
    B, H, Lq, Lk = 2, 3, 200, 136
    q, k, v = _qkv(B, H, Lq, Lk, D, dtype, seed=100 + D)
    bias = torch.randn(B, H, Lq, Lk, device="cuda").to(dtype).requires_grad_(True)
    kpm = torch.zeros(B, Lk, dtype=torch.bool, device="cuda")
    kpm[0, Lk - 40:] = True
    scale = 1.0 / math.sqrt(D)
    keep = _keep_mask_by_probes(q, k, p, scale, 11, bias, kpm) if p > 0 else None
    torch.manual_seed(11)
    out = ops.fused_attention(q, k, v, bias=bias, key_padding_mask=kpm, dropout_p=p, training=True, scale=scale)
    dout = torch.randn_like(out)
    out.backward(dout)
    qr, kr, vr, br = (t.detach().float().requires_grad_(True) for t in (q, k, v, bias))
    ref, _ = _ref(qr, kr, vr, br, kpm, scale, keep=keep, p=p)
    ref.backward(dout.float())
    tol = _tol(dtype)
    assert (out.float() - ref).abs().max().item() < tol
    for name, g, gr in (("dq", q.grad, qr.grad), ("dk", k.grad, kr.grad), ("dv", v.grad, vr.grad),
                        ("dbias", bias.grad, br.grad)):
        assert g.shape == gr.shape, name
        err = (g.float() - gr).abs().max().item()
        assert err < tol * max(1.0, gr.abs().max().item()), (name, err)


@pytest.mark.parametrize("D", [32, 96, 128])
@pytest.mark.parametrize("dtype", DTYPES)
def test_qkvpacked_backward(D, dtype):
    """Packed entry point: the gradient is one contiguous [B, L, 3, H, D] tensor written by the kernels."""
    ops = _ops()
    B, H, L = 2, 3, 328
    g = torch.Generator(device="cuda").manual_seed(D)
    qkv = (torch.randn(B, L, 3, H, D, device="cuda", generator=g) * 0.8).to(dtype).requires_grad_(True)
    bias = torch.randn(1, H, L, L, device="cuda").to(dtype).requires_grad_(True)
    kpm = torch.zeros(B, L, dtype=torch.bool, device="cuda")
    kpm[0, 300:] = True
    scale = 1.0 / math.sqrt(D)
    assert ops.fused_attention_supported(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], bias, kpm)
    out = ops.fused_attention_qkvpacked(qkv, bias=bias, key_padding_mask=kpm, dropout_p=0.0, training=True,
                                        scale=scale)
    dout = torch.randn_like(out)
    out.backward(dout)
    assert qkv.grad.shape == qkv.shape and qkv.grad.is_contiguous()
    qkv_r = qkv.detach().float().requires_grad_(True)
    bias_r = bias.detach().float().requires_grad_(True)
    ref, _ = _ref(qkv_r[:, :, 0], qkv_r[:, :, 1], qkv_r[:, :, 2], bias_r, kpm, scale)
    ref.backward(dout.float())
    tol = _tol(dtype)
    assert (out.float() - ref).abs().max().item() < tol
    assert (qkv.grad.float() - qkv_r.grad).abs().max().item() < tol * max(1.0, qkv_r.grad.abs().max().item())
    assert (bias.grad.float() - bias_r.grad).abs().max().item() < tol * max(1.0, bias_r.grad.abs().max().item())


def test_keep_mask_independent_of_head_dim():
    """Same seed and (B, H, Lq, Lk): the same keep mask at every head dim (and so at every key-tile size)."""
    B, H, Lq, Lk, p = 2, 2, 136, 200, 0.25
    masks = {}
    for D in (32, 64, 128):
        q, k, _ = _qkv(B, H, Lq, Lk, D, torch.float16, seed=7, amp=0.3)
        masks[D] = _keep_mask_by_probes(q, k, p, 1.0 / math.sqrt(D), 23)
    frac = masks[64].mean().item()
    assert abs(frac - (1 - p)) < 0.01, frac
    assert torch.equal(masks[32], masks[64])
    assert torch.equal(masks[128], masks[64])


@pytest.mark.parametrize("dtype", DTYPES)
def test_d128_more_than_one_wave(dtype):
    """B = 4, H = 8, L = 1024 at D = 128: 512 CTAs in either direction (several per SM), 16 key tiles per CTA row."""
    ops = _ops()
    B, H, L, D = 4, 8, 1024, 128
    q, k, v = _qkv(B, H, L, L, D, dtype, seed=31)
    bias = (torch.randn(1, H, L, L, device="cuda") * 0.5).to(dtype).requires_grad_(True)
    kpm = torch.zeros(B, L, dtype=torch.bool, device="cuda")
    kpm[1, 900:] = True
    kpm[3, 77:] = True
    scale = 1.0 / math.sqrt(D)
    out = ops.fused_attention(q, k, v, bias=bias, key_padding_mask=kpm, dropout_p=0.0, training=True, scale=scale)
    dout = torch.randn_like(out)
    out.backward(dout)
    qr, kr, vr, br = (t.detach().float().requires_grad_(True) for t in (q, k, v, bias))
    ref, _ = _ref(qr, kr, vr, br, kpm, scale)
    ref.backward(dout.float())
    tol = _tol(dtype)
    assert (out.float() - ref).abs().max().item() < tol
    for name, g, gr in (("dq", q.grad, qr.grad), ("dk", k.grad, kr.grad), ("dv", v.grad, vr.grad),
                        ("dbias", bias.grad, br.grad)):
        err = (g.float() - gr).abs().max().item()
        assert err < tol * max(1.0, gr.abs().max().item()), (name, err)


def test_self_attention_module_head_dim_96():
    """SelfMultiheadAttention(768, 8): head dim 96 takes the fused kernel and matches the materialised path."""
    from unicore.modules import SelfMultiheadAttention

    ops = _ops()
    torch.manual_seed(3)
    attn = SelfMultiheadAttention(768, 8, dropout=0.0).cuda().half()
    x = torch.randn(2, 128, 768, device="cuda", dtype=torch.half)
    bias = torch.randn(1, 8, 128, 128, device="cuda", dtype=torch.half)
    mask = torch.zeros(2, 128, dtype=torch.bool, device="cuda")
    mask[1, 100:] = True
    qkv = torch.nn.functional.linear(x, attn.in_proj.weight, attn.in_proj.bias).view(2, 128, 3, 8, 96)
    assert ops.fused_attention_supported(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], bias, mask)
    fused = attn(x, key_padding_mask=mask, attn_bias=bias)
    o, _, probs = attn(x, key_padding_mask=mask, attn_bias=bias, return_attn=True)
    assert probs.shape == (16, 128, 128)
    assert (fused.float() - o.float()).abs().max().item() < 2e-2


def test_cross_attention_module_head_dim_128():
    from unicore.modules import CrossMultiheadAttention

    ops = _ops()
    torch.manual_seed(4)
    E, H, B, Lq, Lk = 1024, 8, 2, 136, 200
    attn = CrossMultiheadAttention(E, H, dropout=0.0).cuda().half()
    query = torch.randn(B, Lq, E, device="cuda", dtype=torch.half)
    key = torch.randn(B, Lk, E, device="cuda", dtype=torch.half)
    bias = torch.randn(1, H, Lq, Lk, device="cuda", dtype=torch.half)
    mask = torch.zeros(B, Lk, dtype=torch.bool, device="cuda")
    mask[0, 150:] = True
    out = attn.attend(query, key, key, key_padding_mask=mask, attn_bias=bias)
    q = attn.q_proj(query).view(B, Lq, H, 128).float()
    k = attn.k_proj(key).view(B, Lk, H, 128).float()
    v = attn.v_proj(key).view(B, Lk, H, 128).float()
    assert ops.fused_attention_supported(q.half(), k.half(), v.half(), bias, mask)
    ref = ops.attention_reference(q, k, v, bias.float(), mask, 0.0, False, attn.scaling).reshape(B, Lq, E)
    assert out.shape == ref.shape
    assert (out.float() - ref).abs().max().item() < 1e-2


def test_encoder_default_width_and_heads_matches_fp32_formulation():
    """TransformerEncoder() width and heads (768 / 8: head dim 96) with a padding mask: the stack passes the bias and
    the [B, L] padding mask separately to the fused kernel, and output and every gradient match plain fp32."""
    from unicore.modules import TransformerEncoder

    torch.manual_seed(21)
    B, L = 2, 128
    enc = TransformerEncoder(encoder_layers=2, emb_dropout=0.0, dropout=0.0, attention_dropout=0.0).cuda()
    E, H = enc.embed_dim, enc.attention_heads
    assert (E, H) == (768, 8)
    ref = copy.deepcopy(enc).float()
    enc = enc.half().train()
    emb = torch.randn(B, L, E, device="cuda").half().requires_grad_(True)
    pad = torch.zeros(B, L, dtype=torch.bool, device="cuda")
    pad[1, 100:] = True
    bias, kpm = enc._compose_bias(enc._embed_prologue(emb, pad), None, pad)
    assert kpm is pad and bias.shape == (1, H, L, L)
    y = enc(emb, padding_mask=pad)
    dy = torch.randn_like(y)
    y.backward(dy)

    def plain(m, emb):
        x = F.layer_norm(emb, (E,), m.emb_layer_norm.weight, m.emb_layer_norm.bias)
        x = x * (1 - pad.unsqueeze(-1).float())
        rel = F.embedding(m.rp_bucket[:L, :L].to(emb.device), m.relative_attention_bias.weight).permute(2, 0, 1)
        for layer in m.layers:
            sa = layer.self_attn
            h = F.layer_norm(x, (E,), layer.self_attn_layer_norm.weight, layer.self_attn_layer_norm.bias)
            qkv = F.linear(h, sa.in_proj.weight, sa.in_proj.bias).view(B, L, 3, H, E // H)
            q, k, v = (qkv[:, :, i].transpose(1, 2) for i in range(3))
            s = q @ k.transpose(-1, -2) * sa.scaling + rel
            s = s.masked_fill(pad[:, None, None, :], float("-inf"))
            o = (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(B, L, E)
            x = x + F.linear(o, sa.out_proj.weight, sa.out_proj.bias)
            h = F.layer_norm(x, (E,), layer.final_layer_norm.weight, layer.final_layer_norm.bias)
            x = x + F.linear(F.gelu(F.linear(h, layer.fc1.weight, layer.fc1.bias)), layer.fc2.weight, layer.fc2.bias)
        return F.layer_norm(x, (E,), m.final_layer_norm.weight, m.final_layer_norm.bias)

    er = emb.detach().float().requires_grad_(True)
    yr = plain(ref, er)
    yr.backward(dy.float())
    assert (y.float() - yr).abs().max().item() < 3e-2
    assert (emb.grad.float() - er.grad).abs().max().item() < 3e-2 * max(1.0, er.grad.abs().max().item())
    for (name, p), (_, pr) in zip(enc.named_parameters(), ref.named_parameters()):
        assert p.grad is not None, name
        tol = 4e-2 * max(1.0, pr.grad.abs().max().item())
        assert (p.grad.float() - pr.grad).abs().max().item() < tol, name


@pytest.mark.parametrize("D", [12, 136])
def test_unsupported_head_dims_use_the_reference(D):
    """D = 12 (rows not 16-byte aligned) and D = 136 (wider than the kernels) are not taken by the fused path."""
    ops = _ops()
    assert not ops.fused_head_dim_supported(D)
    B, H, Lq, Lk = 2, 2, 72, 136
    q, k, v = _qkv(B, H, Lq, Lk, D, torch.float16, seed=D)
    bias = torch.randn(1, H, Lq, Lk, device="cuda").half()
    kpm = torch.zeros(B, Lk, dtype=torch.bool, device="cuda")
    kpm[1, 100:] = True
    assert not ops.fused_attention_supported(q, k, v, bias, kpm)
    scale = 1.0 / math.sqrt(D)
    with torch.no_grad():
        out = ops.fused_attention(q, k, v, bias=bias, key_padding_mask=kpm, dropout_p=0.0, training=True, scale=scale)
        ref = ops.attention_reference(q, k, v, bias, kpm, 0.0, True, scale)
    assert torch.equal(out, ref)
    with pytest.raises(RuntimeError, match="head_dim must be"):   # the binding refuses it too
        ops.native().fmha_fwd(q.detach(), k.detach(), v.detach(), None, None, 0.0, scale)
