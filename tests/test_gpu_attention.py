"""wgmma fused attention (forward + backward) against an fp32 PyTorch reference."""

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _ops():
    from unicore import ops

    assert ops.USE_NATIVE
    return ops


def _ref(q, k, v, bias, kpm, scale, keep=None, p=0.0):
    """fp32 reference; q,k,v [B, L, H, D]; keep: optional [B, H, Lq, Lk] dropout keep mask."""
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


def _make(B, H, Lq, Lk, dtype, packed=True, seed=0):
    torch.manual_seed(seed)
    if packed and Lq == Lk:
        qkv = (torch.randn(B, Lq, 3, H, 64, device="cuda") * 0.8).to(dtype)
        qkv.requires_grad_(True)
        return qkv, qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    q = (torch.randn(B, Lq, H, 64, device="cuda") * 0.8).to(dtype).requires_grad_(True)
    k = (torch.randn(B, Lk, H, 64, device="cuda") * 0.8).to(dtype).requires_grad_(True)
    v = (torch.randn(B, Lk, H, 64, device="cuda") * 0.8).to(dtype).requires_grad_(True)
    return None, q, k, v


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("shape", [(2, 3, 128, 128), (2, 4, 512, 512), (1, 2, 256, 384), (2, 2, 200, 72), (1, 1, 8, 8), (1, 2, 640, 1000)])
@pytest.mark.parametrize("with_bias,with_mask", [(False, False), (True, False), (True, True)])
def test_fmha_forward(dtype, shape, with_bias, with_mask):
    ops = _ops()
    B, H, Lq, Lk = shape
    _, q, k, v = _make(B, H, Lq, Lk, dtype)
    bias = torch.randn(1, H, Lq, Lk, device="cuda").to(dtype) if with_bias else None
    kpm = None
    if with_mask:
        kpm = torch.zeros(B, Lk, dtype=torch.bool, device="cuda")
        kpm[0, Lk - Lk // 4:] = True
    assert ops.fused_attention_supported(q, k, v, bias, kpm)
    scale = 1.0 / 8.0
    out = ops.fused_attention(q, k, v, bias=bias, key_padding_mask=kpm, dropout_p=0.0, training=True, scale=scale)
    ref, _ = _ref(q, k, v, bias, kpm, scale)
    tol = 4e-3 if dtype == torch.float16 else 2e-2
    assert out.shape == ref.shape
    err = (out.float() - ref).abs().max().item()
    assert err < tol, err


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("bias_batch", [1, 2])
def test_fmha_backward(dtype, bias_batch):
    ops = _ops()
    B, H, L = 2, 3, 256
    qkv, q, k, v = _make(B, H, L, L, dtype, seed=1)
    bias = torch.randn(bias_batch, H, L, L, device="cuda").to(dtype).requires_grad_(True)
    kpm = torch.zeros(B, L, dtype=torch.bool, device="cuda")
    kpm[1, 200:] = True
    scale = 0.125
    out = ops.fused_attention(q, k, v, bias=bias, key_padding_mask=kpm, dropout_p=0.0, training=True, scale=scale)
    dout = torch.randn_like(out)
    out.backward(dout)
    qkv_r = qkv.detach().float().requires_grad_(True)
    bias_r = bias.detach().float().requires_grad_(True)
    ref, _ = _ref(qkv_r[:, :, 0], qkv_r[:, :, 1], qkv_r[:, :, 2], bias_r, kpm, scale)
    ref.backward(dout.float())
    tol = 1e-2 if dtype == torch.float16 else 6e-2
    assert (out.float() - ref).abs().max().item() < tol
    gerr = (qkv.grad.float() - qkv_r.grad).abs().max().item()
    assert gerr < tol * max(1.0, qkv_r.grad.abs().max().item()), gerr
    berr = (bias.grad.float() - bias_r.grad).abs().max().item()
    assert berr < tol * max(1.0, bias_r.grad.abs().max().item()), berr


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_fmha_qkvpacked_backward(dtype):
    """Packed entry point: gradients land in one [B, L, 3, H, D] tensor written by the kernels."""
    ops = _ops()
    B, H, L = 2, 4, 384
    qkv, _, _, _ = _make(B, H, L, L, dtype, seed=4)
    bias = torch.randn(1, H, L, L, device="cuda").to(dtype).requires_grad_(True)
    kpm = torch.zeros(B, L, dtype=torch.bool, device="cuda")
    kpm[0, 300:] = True
    out = ops.fused_attention_qkvpacked(qkv, bias=bias, key_padding_mask=kpm, dropout_p=0.0, training=True, scale=0.125)
    dout = torch.randn_like(out)
    out.backward(dout)
    assert qkv.grad.shape == qkv.shape and qkv.grad.is_contiguous()
    qkv_r = qkv.detach().float().requires_grad_(True)
    bias_r = bias.detach().float().requires_grad_(True)
    ref, _ = _ref(qkv_r[:, :, 0], qkv_r[:, :, 1], qkv_r[:, :, 2], bias_r, kpm, 0.125)
    ref.backward(dout.float())
    tol = 1e-2 if dtype == torch.float16 else 6e-2
    assert (out.float() - ref).abs().max().item() < tol
    assert (qkv.grad.float() - qkv_r.grad).abs().max().item() < tol * max(1.0, qkv_r.grad.abs().max().item())
    assert (bias.grad.float() - bias_r.grad).abs().max().item() < tol * max(1.0, bias_r.grad.abs().max().item())


def _keep_mask_by_probes(q, k, p, scale, seed, bias=None, kpm=None):
    """The forward kernel's dropout keep mask [B, H, Lq, Lk], read back through value probes: with v = e_d at key
    blk * 64 + d, output column d is P_drop of that key (same seed -> same Philox stream)."""
    from unicore import ops

    B, Lk, H, _ = k.shape
    masks = []
    for blk in range((Lk + 63) // 64):
        eye = torch.zeros(B, Lk, H, 64, device="cuda", dtype=q.dtype)
        n = min(64, Lk - blk * 64)
        for d in range(n):
            eye[:, blk * 64 + d, :, d] = 1
        torch.manual_seed(seed)
        pd = ops.fused_attention(q.detach(), k.detach(), eye, bias=None if bias is None else bias.detach(),
                                 key_padding_mask=kpm, dropout_p=p, training=True, scale=scale)
        masks.append(pd.permute(0, 2, 1, 3)[..., :n])
    return (torch.cat(masks, dim=-1) != 0).float()


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("shape", [(2, 3, 200, 136), (1, 2, 72, 328)])
@pytest.mark.parametrize("p", [0.0, 0.25])
def test_fmha_backward_ragged(dtype, shape, p):
    """Backward with Lq != Lk and lengths that are not multiples of the 64-row / 64-key tiles: query rows past Lq,
    keys past Lk, the last (partial) keep-bit word of a row and clipped dS stores, with a per-batch bias gradient,
    key padding and dropout."""
    ops = _ops()
    B, H, Lq, Lk = shape
    _, q, k, v = _make(B, H, Lq, Lk, dtype, packed=False, seed=5)
    bias = torch.randn(B, H, Lq, Lk, device="cuda").to(dtype).requires_grad_(True)
    kpm = torch.zeros(B, Lk, dtype=torch.bool, device="cuda")
    kpm[0, Lk - 40:] = True
    scale = 0.125
    keep = _keep_mask_by_probes(q, k, p, scale, 11, bias, kpm) if p > 0 else None
    torch.manual_seed(11)
    out = ops.fused_attention(q, k, v, bias=bias, key_padding_mask=kpm, dropout_p=p, training=True, scale=scale)
    dout = torch.randn_like(out)
    out.backward(dout)
    qr, kr, vr, br = (t.detach().float().requires_grad_(True) for t in (q, k, v, bias))
    ref, _ = _ref(qr, kr, vr, br, kpm, scale, keep=keep, p=p)
    ref.backward(dout.float())
    tol = 1e-2 if dtype == torch.float16 else 6e-2
    assert (out.float() - ref).abs().max().item() < tol
    for g, gr in ((q.grad, qr.grad), (k.grad, kr.grad), (v.grad, vr.grad), (bias.grad, br.grad)):
        assert (g.float() - gr).abs().max().item() < tol * max(1.0, gr.abs().max().item())


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_fmha_leading_masked_tile_with_very_negative_logits(dtype):
    """The first 128-key tile is entirely padding and every real logit is far below -87 (exp underflows in fp32
    without a proper offset): the softmax must still be the fp32 reference's, forward and backward."""
    ops = _ops()
    B, H, Lq, Lk = 2, 2, 64, 320
    _, q, k, v = _make(B, H, Lq, Lk, dtype, packed=False, seed=6)
    bias = (torch.randn(1, H, Lq, Lk, device="cuda") - 200.0).to(dtype)
    kpm = torch.zeros(B, Lk, dtype=torch.bool, device="cuda")
    kpm[:, :130] = True
    scale = 0.125
    out = ops.fused_attention(q, k, v, bias=bias, key_padding_mask=kpm, dropout_p=0.0, training=True, scale=scale)
    dout = torch.randn_like(out)
    out.backward(dout)
    qr, kr, vr = (t.detach().float().requires_grad_(True) for t in (q, k, v))
    ref, _ = _ref(qr, kr, vr, bias, kpm, scale)
    ref.backward(dout.float())
    tol = 1e-2 if dtype == torch.float16 else 6e-2
    assert ref.abs().max().item() > 0.1
    assert (out.float() - ref).abs().max().item() < tol
    for g, gr in ((q.grad, qr.grad), (k.grad, kr.grad), (v.grad, vr.grad)):
        assert (g.float() - gr).abs().max().item() < tol * max(1.0, gr.abs().max().item())


def test_fmha_dropout_consistency():
    """Dropout: keep-rate, and backward uses exactly the forward's mask (checked via a linear probe)."""
    ops = _ops()
    B, H, L, p = 2, 2, 256, 0.25
    dtype = torch.float16
    _, q, k, v = _make(B, H, L, L, dtype, packed=False, seed=2)
    scale = 0.125
    torch.manual_seed(10)
    out = ops.fused_attention(q, k, v, dropout_p=p, training=True, scale=scale)
    # recover the keep mask: with v = identity-like probes we can read P_drop directly
    eye = torch.zeros(B, L, H, 64, device="cuda", dtype=dtype)
    masks = []
    for blk in range(L // 64):
        eye.zero_()
        for d in range(64):
            eye[:, blk * 64 + d, :, d] = 1
        torch.manual_seed(10)
        pd = ops.fused_attention(q.detach(), k.detach(), eye, dropout_p=p, training=True, scale=scale)
        masks.append(pd.permute(0, 2, 1, 3))  # [B, H, Lq, 64 keys of this block]
    pdrop = torch.cat(masks, dim=-1).float()  # [B, H, Lq, Lk]
    keep = (pdrop != 0).float()
    frac = keep.mean().item()
    assert abs(frac - (1 - p)) < 0.01, frac
    ref, _ = _ref(q, k, v, None, None, scale, keep=keep, p=p)
    assert (out.float() - ref).abs().max().item() < 1e-2
    dout = torch.randn_like(out)
    torch.manual_seed(10)
    out2 = ops.fused_attention(q, k, v, dropout_p=p, training=True, scale=scale)
    out2.backward(dout)
    qr, kr, vr = (t.detach().float().requires_grad_(True) for t in (q, k, v))
    ref2, _ = _ref(qr, kr, vr, None, None, scale, keep=keep, p=p)
    ref2.backward(dout.float())
    for g, gr in ((q.grad, qr.grad), (k.grad, kr.grad), (v.grad, vr.grad)):
        assert (g.float() - gr).abs().max().item() < 2e-2 * max(1.0, gr.abs().max().item())


def test_self_attention_module_matches_materialised_path():
    from unicore.modules import SelfMultiheadAttention

    torch.manual_seed(3)
    attn = SelfMultiheadAttention(768, 12, dropout=0.0).cuda().half()
    x = torch.randn(2, 128, 768, device="cuda", dtype=torch.half)
    bias = torch.randn(1, 12, 128, 128, device="cuda", dtype=torch.half)
    mask = torch.zeros(2, 128, dtype=torch.bool, device="cuda")
    mask[1, 100:] = True
    fused = attn(x, key_padding_mask=mask, attn_bias=bias)
    o, logits, probs = attn(x, key_padding_mask=mask, attn_bias=bias, return_attn=True)
    assert (fused.float() - o.float()).abs().max().item() < 2e-2
    assert probs.shape == (24, 128, 128)


@pytest.mark.parametrize("post_ln", [False, True])
def test_encoder_layer_matches_fp32_formulation(post_ln):
    """Whole pre-LN or post-LN layer (wgmma attention, bias-GELU, column-sum bias gradients, and on the post-LN path
    the fused bias + dropout + residual + LayerNorm) against the plain fp32 formulation of the same layer, forward
    and all gradients (dropout off)."""
    import copy

    import torch.nn.functional as F

    from unicore.modules import TransformerEncoderLayer

    torch.manual_seed(21)
    E, H, L, B = 256, 4, 128, 3
    layer = TransformerEncoderLayer(embed_dim=E, ffn_embed_dim=4 * E, attention_heads=H, dropout=0.0,
                                    attention_dropout=0.0, activation_dropout=0.0, post_ln=post_ln).cuda()
    ref = copy.deepcopy(layer).float()
    layer = layer.half().train()
    x = torch.randn(B, L, E, device="cuda").half().requires_grad_(True)
    bias = (torch.randn(1, H, L, L, device="cuda") * 0.5).half()
    pad = torch.zeros(B, L, dtype=torch.bool, device="cuda")
    pad[2, 100:] = True
    y = layer(x, attn_bias=bias, padding_mask=pad)
    dy = torch.randn_like(y)
    y.backward(dy)

    def plain(m, x):
        def attn(h):
            qkv = F.linear(h, m.self_attn.in_proj.weight, m.self_attn.in_proj.bias).view(B, L, 3, H, E // H)
            q, k, v = (qkv[:, :, i].transpose(1, 2) for i in range(3))
            s = q @ k.transpose(-1, -2) * m.self_attn.scaling + bias.float()
            s = s.masked_fill(pad[:, None, None, :], float("-inf"))
            o = (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(B, L, E)
            return F.linear(o, m.self_attn.out_proj.weight, m.self_attn.out_proj.bias)

        def ffn(h):
            return F.linear(F.gelu(F.linear(h, m.fc1.weight, m.fc1.bias)), m.fc2.weight, m.fc2.bias)

        ln1 = lambda t: F.layer_norm(t, (E,), m.self_attn_layer_norm.weight, m.self_attn_layer_norm.bias)  # noqa: E731
        ln2 = lambda t: F.layer_norm(t, (E,), m.final_layer_norm.weight, m.final_layer_norm.bias)  # noqa: E731
        if post_ln:
            x = ln1(x + attn(x))
            return ln2(x + ffn(x))
        x = x + attn(ln1(x))
        return x + ffn(ln2(x))

    xr = x.detach().float().requires_grad_(True)
    yr = plain(ref, xr)
    yr.backward(dy.float())
    assert (y.float() - yr).abs().max().item() < 3e-2
    assert (x.grad.float() - xr.grad).abs().max().item() < 3e-2 * max(1.0, xr.grad.abs().max().item())
    for (name, p), (_, pr) in zip(layer.named_parameters(), ref.named_parameters()):
        assert p.grad is not None, name
        tol = 4e-2 * max(1.0, pr.grad.abs().max().item())
        assert (p.grad.float() - pr.grad).abs().max().item() < tol, name
