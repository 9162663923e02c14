"""Fused attention in logits mode (``return_logits=True``): the kernels also write z = scale * q k^T + bias + key mask
and take its gradient dz.  Logits against fp32, O / LSE / keep bits bitwise equal to the plain kernel, the backward
with dz against fp32 autograd (additive mask), dz = None against the plain backward, the packed entry point, the
attention module and Uni-Mol's pair encoder against the materialised path, the activation memory saved by a pair
stack, and the head dims that fall back to the reference."""
import copy
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]


def _ops():
    from unicore import ops

    assert ops.USE_NATIVE
    return ops


def _qkv(B, H, Lq, Lk, D, dtype, seed, amp=0.8):
    g = torch.Generator(device="cuda").manual_seed(seed)

    def rnd(L):
        return (torch.randn(B, L, H, D, device="cuda", generator=g) * amp).to(dtype).requires_grad_(True)

    return rnd(Lq), rnd(Lk), rnd(Lk)


def _bias(layout, B, H, Lq, Lk, dtype, grad=False):
    if layout is None:
        return None
    b = torch.randn(B if layout == "B" else 1, H, Lq, Lk, device="cuda").to(dtype)
    return b.requires_grad_(grad)


def _kpm(B, Lk):
    kpm = torch.zeros(B, Lk, dtype=torch.bool, device="cuda")
    kpm[0, Lk - Lk // 4:] = True
    kpm[-1, :8] = True
    return kpm


def _ref(q, k, v, bias, kpm, scale, keep=None, p=0.0):
    """fp32 reference with the logits contract: additive -inf key mask. Returns (O, z)."""
    qf, kf, vf = q.float(), k.float(), v.float()
    z = torch.einsum("bqhd,bkhd->bhqk", qf, kf) * scale
    if bias is not None:
        z = z + bias.float()
    if kpm is not None:
        z = z + torch.zeros(kpm.shape, device=kpm.device).masked_fill(kpm, float("-inf"))[:, None, None, :]
    pr = torch.softmax(z, dim=-1)
    if keep is not None:
        pr = pr * keep / (1 - p)
    return torch.einsum("bhqk,bkhd->bqhd", pr, vf), z


def _tol(dtype):
    return 1e-2 if dtype == torch.float16 else 6e-2


def _keep_mask_by_probes(q, k, p, scale, seed, bias=None, kpm=None):
    """The forward kernel's dropout keep mask [B, H, Lq, Lk], read back through value probes (as in
    test_gpu_attention_head_dims.py): with v = e_d at key blk * D + d, output column d is P_drop of that key."""
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


@pytest.mark.parametrize("D", [8, 64, 128])
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("shape", [(2, 2, 200, 72), (1, 2, 640, 1000)])
@pytest.mark.parametrize("layout", [None, "1", "B"])
@pytest.mark.parametrize("with_mask", [False, True])
def test_logits_match_fp32(D, dtype, shape, layout, with_mask):
    ops = _ops()
    B, H, Lq, Lk = shape
    q, k, v = _qkv(B, H, Lq, Lk, D, dtype, seed=D)
    bias = _bias(layout, B, H, Lq, Lk, dtype)
    kpm = _kpm(B, Lk) if with_mask else None
    assert ops.fused_attention_supported(q, k, v, bias, kpm)
    scale = 1.0 / math.sqrt(D)
    with torch.no_grad():
        out, z = ops.fused_attention(q, k, v, bias=bias, key_padding_mask=kpm, dropout_p=0.0, scale=scale,
                                     return_logits=True)
        ref, zr = _ref(q, k, v, bias, kpm, scale)
    assert z.shape == (B, H, Lq, Lk) and z.dtype == dtype and z.is_contiguous()
    masked = torch.zeros(B, 1, 1, Lk, dtype=torch.bool, device="cuda") if kpm is None else kpm[:, None, None, :]
    assert torch.equal(torch.isinf(z), masked.expand_as(z)) and bool((z[torch.isinf(z)] < 0).all())
    assert torch.isfinite(z[~masked.expand_as(z)]).all()
    fin = torch.isfinite(zr)
    eps = 2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -11   # one unit of 16-bit rounding, relative
    err = (z.float()[fin] - zr[fin]).abs()
    assert (err <= eps * zr[fin].abs() + 1e-3).all(), err.max().item()
    assert (out.float() - ref).abs().max().item() < (4e-3 if dtype == torch.float16 else 2e-2)


@pytest.mark.parametrize("D", [8, 64, 128])
@pytest.mark.parametrize("dtype", DTYPES)
def test_out_lse_and_keep_bits_bitwise_equal_to_plain_kernel(D, dtype):
    ops = _ops()
    B, H, Lq, Lk = 2, 2, 200, 328
    q, k, v = _qkv(B, H, Lq, Lk, D, dtype, seed=40 + D)
    bias = _bias("B", B, H, Lq, Lk, dtype)
    kpm = _kpm(B, Lk)
    scale = 1.0 / math.sqrt(D)
    with torch.no_grad():
        torch.manual_seed(5)
        out, lse, bits = ops.native().fmha_fwd(q, k, v, bias, kpm, 0.25, scale)
        torch.manual_seed(5)
        out2, lse2, bits2, z = ops.native().fmha_fwd_logits(q, k, v, bias, kpm, 0.25, scale)
    assert z.shape == (B, H, Lq, Lk)
    assert torch.equal(out, out2) and torch.equal(lse, lse2) and torch.equal(bits, bits2)


@pytest.mark.parametrize("D", [8, 64, 128])
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("p", [0.0, 0.25])
@pytest.mark.parametrize("layout", ["1", "B"])
def test_backward_with_logits_gradient(D, dtype, p, layout):
    """dS_total = P o (drop(dP) - delta) + dz feeds dq, dk and dbias; dz reaches the masked keys too."""
    ops = _ops()
    B, H, Lq, Lk = 2, 3, 200, 136
    q, k, v = _qkv(B, H, Lq, Lk, D, dtype, seed=100 + D)
    bias = _bias(layout, B, H, Lq, Lk, dtype, grad=True)
    kpm = _kpm(B, Lk)
    scale = 1.0 / math.sqrt(D)
    keep = _keep_mask_by_probes(q, k, p, scale, 11, bias, kpm) if p > 0 else None
    torch.manual_seed(11)
    out, z = ops.fused_attention(q, k, v, bias=bias, key_padding_mask=kpm, dropout_p=p, training=True, scale=scale,
                                 return_logits=True)
    dout = torch.randn_like(out)
    dz = torch.randn_like(z)
    torch.autograd.backward([out, z], [dout, dz])
    qr, kr, vr, br = (t.detach().float().requires_grad_(True) for t in (q, k, v, bias))
    ref, zr = _ref(qr, kr, vr, br, kpm, scale, keep=keep, p=p)
    torch.autograd.backward([ref, zr], [dout.float(), dz.float()])
    tol = _tol(dtype)
    assert (out.float() - ref).abs().max().item() < tol
    for name, g, gr in (("dq", q.grad, qr.grad), ("dk", k.grad, kr.grad), ("dv", v.grad, vr.grad),
                        ("dbias", bias.grad, br.grad)):
        assert g.shape == gr.shape, name
        err = (g.float() - gr).abs().max().item()
        assert err < tol * max(1.0, gr.abs().max().item()), (name, err)


@pytest.mark.parametrize("D", [8, 64, 128])
def test_no_logits_gradient_is_the_plain_backward(D):
    """dz = None means zero: dk, dv and dbias are bitwise the plain fused backward's, dq up to its bulk-reduction
    ordering."""
    ops = _ops()
    B, H, Lq, Lk = 2, 3, 200, 136
    dtype = torch.bfloat16
    q, k, v = _qkv(B, H, Lq, Lk, D, dtype, seed=200 + D)
    bias = _bias("B", B, H, Lq, Lk, dtype, grad=True)
    kpm = _kpm(B, Lk)
    scale = 1.0 / math.sqrt(D)
    dout = torch.randn(B, Lq, H, D, device="cuda").to(dtype)
    grads = []
    for logits in (False, True):
        for t in (q, k, v, bias):
            t.grad = None
        torch.manual_seed(3)
        res = ops.fused_attention(q, k, v, bias=bias, key_padding_mask=kpm, dropout_p=0.25, training=True,
                                  scale=scale, return_logits=logits)
        (res[0] if logits else res).backward(dout)
        grads.append([t.grad.clone() for t in (q, k, v, bias)])
    (dq0, dk0, dv0, db0), (dq1, dk1, dv1, db1) = grads
    assert torch.equal(dk0, dk1) and torch.equal(dv0, dv1) and torch.equal(db0, db1)
    assert (dq0.float() - dq1.float()).abs().max().item() <= 1e-2 * max(1.0, dq0.float().abs().max().item())


@pytest.mark.parametrize("D", [8, 64, 128])
@pytest.mark.parametrize("dtype", DTYPES)
def test_qkvpacked_with_logits(D, dtype):
    ops = _ops()
    B, H, L = 2, 3, 200
    g = torch.Generator(device="cuda").manual_seed(D)
    qkv = (torch.randn(B, L, 3, H, D, device="cuda", generator=g) * 0.8).to(dtype).requires_grad_(True)
    bias = _bias("1", B, H, L, L, dtype, grad=True)
    kpm = _kpm(B, L)
    scale = 1.0 / math.sqrt(D)
    out, z = ops.fused_attention_qkvpacked(qkv, bias=bias, key_padding_mask=kpm, dropout_p=0.0, training=True,
                                           scale=scale, return_logits=True)
    assert z.shape == (B, H, L, L)
    dout, dz = torch.randn_like(out), torch.randn_like(z)
    torch.autograd.backward([out, z], [dout, dz])
    assert qkv.grad.shape == qkv.shape and qkv.grad.is_contiguous()
    qkv_r = qkv.detach().float().requires_grad_(True)
    bias_r = bias.detach().float().requires_grad_(True)
    ref, zr = _ref(qkv_r[:, :, 0], qkv_r[:, :, 1], qkv_r[:, :, 2], bias_r, kpm, scale)
    torch.autograd.backward([ref, zr], [dout.float(), dz.float()])
    tol = _tol(dtype)
    fin = torch.isfinite(zr)
    assert torch.equal(torch.isfinite(z), fin)
    assert (z.float()[fin] - zr[fin]).abs().max().item() < tol * max(1.0, zr[fin].abs().max().item())
    assert (out.float() - ref).abs().max().item() < tol
    assert (qkv.grad.float() - qkv_r.grad).abs().max().item() < tol * max(1.0, qkv_r.grad.abs().max().item())
    assert (bias.grad.float() - bias_r.grad).abs().max().item() < tol * max(1.0, bias_r.grad.abs().max().item())


def _close(a, b, rel, name):
    assert a.shape == b.shape, name
    fa, fb = torch.isfinite(a), torch.isfinite(b)
    assert torch.equal(fa, fb), name
    err = (a.float()[fa] - b.float()[fb]).abs().max().item() if fa.any() else 0.0
    assert err <= rel * max(1.0, b.float()[fb].abs().max().item()), (name, err)


def test_self_attention_module_logits_without_probs():
    """SelfMultiheadAttention(512, 64): need_probs=False gives the fused o and logits of the materialised path."""
    from unicore.modules import SelfMultiheadAttention

    torch.manual_seed(6)
    B, L, E, H = 2, 96, 512, 64
    attn = SelfMultiheadAttention(E, H, dropout=0.0).cuda().bfloat16()
    ref = copy.deepcopy(attn)
    x = torch.randn(B, L, E, device="cuda").bfloat16().requires_grad_(True)
    xr = x.detach().clone().requires_grad_(True)
    bias = torch.randn(B * H, L, L, device="cuda").bfloat16().requires_grad_(True)
    br = bias.detach().clone().requires_grad_(True)
    pad = torch.zeros(B, L, dtype=torch.bool, device="cuda")
    pad[1, 70:] = True
    o, z, probs = attn(x, key_padding_mask=pad, attn_bias=bias, return_attn=True, need_probs=False)
    o_r, z_r, probs_r = ref(xr, key_padding_mask=pad, attn_bias=br, return_attn=True)
    assert probs is None and probs_r.shape == (B * H, L, L)
    assert z.shape == z_r.shape == (B * H, L, L)
    _close(o, o_r, 3e-2, "o")
    _close(z, z_r, 3e-2, "logits")
    do, dz = torch.randn_like(o), torch.randn_like(z)
    torch.autograd.backward([o, z], [do, dz])
    torch.autograd.backward([o_r, z_r], [do, dz])
    _close(x.grad, xr.grad, 3e-2, "dx")
    _close(bias.grad, br.grad, 3e-2, "dbias")
    for (name, p), (_, pr) in zip(attn.named_parameters(), ref.named_parameters()):
        _close(p.grad, pr.grad, 3e-2, name)


def _force_probs(enc):
    """Route every layer of a pair encoder through the materialised need_probs=True path."""
    for layer in enc.layers:
        fwd = layer.forward
        layer.forward = lambda *a, _f=fwd, **kw: _f(*a, **{**kw, "need_probs": True})
    return enc


def _pair_encoder(layers, E=512, H=64, ffn=1024, attention_dropout=0.0):
    from unicore_b200.models.unimol import TransformerEncoderWithPair

    return TransformerEncoderWithPair(encoder_layers=layers, embed_dim=E, ffn_embed_dim=ffn, attention_heads=H,
                                      emb_dropout=0.0, dropout=0.0, attention_dropout=attention_dropout,
                                      max_seq_len=512).cuda().bfloat16()


def test_unimol_pair_encoder_fused_matches_materialised():
    """3 layers, 512 wide, 64 heads, padded batch, bf16: outputs and all gradients of the fused logits path equal the
    same weights run layer by layer through the materialised path."""
    torch.manual_seed(8)
    B, L, E, H = 2, 64, 512, 64
    enc = _pair_encoder(3)
    ref = _force_probs(copy.deepcopy(enc))
    emb = torch.randn(B, L, E, device="cuda").bfloat16().requires_grad_(True)
    pair = torch.randn(B * H, L, L, device="cuda").bfloat16().requires_grad_(True)
    pad = torch.zeros(B, L, dtype=torch.bool, device="cuda")
    pad[0, 50:] = True
    emb_r, pair_r = (t.detach().clone().requires_grad_(True) for t in (emb, pair))
    outs = enc(emb, attn_mask=pair, padding_mask=pad)
    outs_r = ref(emb_r, attn_mask=pair_r, padding_mask=pad)
    names = ("x", "pair", "delta", "x_norm", "delta_norm")
    for name, a, b in zip(names, outs, outs_r):
        _close(a, b, 4e-2, name)
    weights = [torch.randn_like(t) for t in outs]
    torch.autograd.backward(list(outs), weights)
    torch.autograd.backward(list(outs_r), weights)
    _close(emb.grad, emb_r.grad, 4e-2, "demb")
    _close(pair.grad, pair_r.grad, 4e-2, "dpair")
    for (name, p), (_, pr) in zip(enc.named_parameters(), ref.named_parameters()):
        assert p.grad is not None, name
        _close(p.grad, pr.grad, 5e-2, name)


def test_pair_stack_peak_memory():
    """Forward + backward of a 4-layer pair stack: the fused path holds less activation memory than the materialised
    one by at least 3 [B, H, L, L] 16-bit tensors (the count predicts about 3.75: one P_drop per layer, less the keep
    bits)."""
    torch.manual_seed(9)
    B, L, E, H = 4, 128, 512, 64
    pair_bytes = B * H * L * L * 2
    enc = _pair_encoder(4, ffn=512, attention_dropout=0.1).train()
    ref = _force_probs(copy.deepcopy(enc)).train()
    emb = torch.randn(B, L, E, device="cuda").bfloat16()
    pair = torch.randn(B * H, L, L, device="cuda").bfloat16()
    pad = torch.zeros(B, L, dtype=torch.bool, device="cuda")
    pad[0, 100:] = True

    def peak(model):
        emb_g, pair_g = emb.clone().requires_grad_(True), pair.clone().requires_grad_(True)
        model.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        outs = model(emb_g, attn_mask=pair_g, padding_mask=pad)
        sum(o.float().sum() for o in outs).backward()
        torch.cuda.synchronize()
        used = torch.cuda.max_memory_allocated() - base
        del outs, emb_g, pair_g
        model.zero_grad(set_to_none=True)
        return used

    peak(enc), peak(ref)   # first calls allocate parameter gradients and workspaces
    fused, mat = peak(enc), peak(ref)
    saved = (mat - fused) / pair_bytes
    print("peak bytes: fused {} materialised {} saved {:.2f} x B*H*L*L*2".format(fused, mat, saved))
    assert saved >= 3.0, saved


def test_unsupported_head_dim_falls_back_with_logits():
    ops = _ops()
    D = 12
    B, H, Lq, Lk = 2, 2, 72, 136
    q, k, v = _qkv(B, H, Lq, Lk, D, torch.float16, seed=D)
    bias = torch.randn(1, H, Lq, Lk, device="cuda").half()
    kpm = torch.zeros(B, Lk, dtype=torch.bool, device="cuda")
    kpm[1, 100:] = True
    assert not ops.fused_attention_supported(q, k, v, bias, kpm)
    scale = 1.0 / math.sqrt(D)
    with torch.no_grad():
        out, z = ops.fused_attention(q, k, v, bias=bias, key_padding_mask=kpm, dropout_p=0.0, training=True,
                                     scale=scale, return_logits=True)
        ref, zr = ops.attention_reference(q, k, v, bias, kpm, 0.0, True, scale, return_logits=True)
    assert z.shape == (B, H, Lq, Lk)
    assert torch.equal(out, ref) and torch.equal(z, zr)
    assert torch.isinf(z[1, :, :, 100:]).all() and torch.isfinite(z[0]).all()
