"""Numerics of every hand-written sm_90a kernel against plain PyTorch fp32 references."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DTYPES = [torch.float32, torch.float16, torch.bfloat16]
TOL = {torch.float32: 2e-5, torch.float16: 2e-3, torch.bfloat16: 1.6e-2}


def _ops():
    from unicore import ops

    assert ops.USE_NATIVE, "native kernels must be active on the GPU box"
    return ops


def maxdiff(a, b):
    return (a.float() - b.float()).abs().max().item()


# ---------------------------------------------------------------------------------------------------
# optimizer ops
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_l2norm(dtype):
    ops = _ops()
    torch.manual_seed(0)
    ts = [torch.randn(n, device="cuda").to(dtype) for n in (1, 7, 8, 1023, 8192, 100003, 3_000_001)]
    ts.append(torch.randn(4099, device="cuda").to(dtype)[3:])  # misaligned view
    ref = torch.sqrt(sum(t.float().pow(2).sum() for t in ts))
    got = ops.multi_tensor_l2norm(ts)
    assert got.dtype == torch.float32 and got.dim() == 0
    assert abs(got.item() - ref.item()) / ref.item() < 1e-5
    many = [torch.randn(257, device="cuda").to(dtype) for _ in range(61)]  # > 24 tensors: several launches
    ref = torch.sqrt(sum(t.float().pow(2).sum() for t in many))
    assert abs(ops.multi_tensor_l2norm(many).item() - ref.item()) / ref.item() < 1e-5
    bad = [torch.ones(100, device="cuda", dtype=dtype), torch.full((5,), float("inf"), device="cuda", dtype=dtype)]
    assert math.isinf(ops.multi_tensor_l2norm(bad).item())


@pytest.mark.parametrize("dtype", DTYPES)
def test_scale(dtype):
    ops = _ops()
    ts = [torch.randn(n, device="cuda").to(dtype) for n in (5, 4096, 77777)]
    ref = [t.float() * 0.37 for t in ts]
    ops.multi_tensor_scale_(ts, 0.37)
    for t, r in zip(ts, ref):
        assert maxdiff(t, r) <= TOL[dtype] * 4
    ts2 = [t.clone() for t in ts]
    ops.multi_tensor_scale_(ts2, torch.tensor(2.0, device="cuda"))
    for a, b in zip(ts2, ts):
        assert maxdiff(a, b.float() * 2) <= TOL[dtype] * 4


def _adam_ref(p, g, m, v, lr, b1, b2, eps, step, wd, scale):
    g = g.float() / scale
    m = b1 * m + (1 - b1) * g
    v = b2 * v + (1 - b2) * g * g
    ss = lr * math.sqrt(1 - b2 ** step) / (1 - b1 ** step)
    p = p * (1 - ss * wd) - ss * m / (v.sqrt() + eps)
    return p, m, v


@pytest.mark.parametrize("gdtype", [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize("n", [1, 9, 8192, 100001])
def test_fused_adam(gdtype, n):
    ops = _ops()
    torch.manual_seed(1)
    p = torch.randn(n, device="cuda")
    g = (torch.randn(n, device="cuda") * 8).to(gdtype)
    m = torch.randn(n, device="cuda") * 0.1
    v = torch.rand(n, device="cuda") * 0.1
    half = torch.empty(n, device="cuda", dtype=torch.float16 if gdtype != torch.bfloat16 else torch.bfloat16)
    rp, rm, rv = _adam_ref(p.clone(), g, m.clone(), v.clone(), 1e-2, 0.9, 0.98, 1e-6, 3, 0.01, 8.0)
    work = [dict(p=p, g=g, m=m, v=v, p_half=half, lr=1e-2, beta1=0.9, beta2=0.98, eps=1e-6, step=3,
                 bias_correction=True, weight_decay=0.01)]
    ops.fused_adam(work, grad_scale=torch.tensor(8.0, device="cuda"), zero_grad=True)
    assert maxdiff(p, rp) < 1e-5 and maxdiff(m, rm) < 1e-5 and maxdiff(v, rv) < 1e-4
    assert maxdiff(half, rp) <= rp.abs().max().item() * 2 ** -7  # one 16-bit rounding of the fp32 result
    assert g.abs().max().item() == 0.0


def test_fused_adam_many_tensors_and_fp32_step():
    ops = _ops()
    torch.manual_seed(2)
    work, refs = [], []
    for i in range(40):
        n = 100 + 37 * i
        p, g = torch.randn(n, device="cuda"), torch.randn(n, device="cuda")
        m, v = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
        refs.append(_adam_ref(p.clone(), g, m.clone(), v.clone(), 1e-3, 0.9, 0.999, 1e-8, 1, 0.0, 1.0))
        work.append(dict(p=p, g=g, m=m, v=v, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, step=1,
                         bias_correction=True, weight_decay=0.0))
    ops.fused_adam(work, grad_scale=1.0)
    for w, (rp, rm, rv) in zip(work, refs):
        assert maxdiff(w["p"], rp) < 1e-5 and maxdiff(w["m"], rm) < 1e-6


def test_stochastic_rounding_unbiased():
    ops = _ops()
    x = torch.full((1 << 20,), 1.0 + 2 ** -10, device="cuda")  # between two bf16 values (spacing 2^-7)
    out = torch.empty_like(x, dtype=torch.bfloat16)
    ops.fp32_to_bf16_sr(x, out)
    vals = out.float().unique()
    assert set(vals.tolist()) <= {1.0, 1.0 + 2 ** -7}
    assert abs(out.float().mean().item() - x[0].item()) < 2e-4
    out2 = torch.empty_like(out)
    ops.fp32_to_bf16_sr(x, out2)
    assert not torch.equal(out, out2)  # fresh Philox offset each call


def test_ema_update():
    ops = _ops()
    ema, p = torch.randn(100003, device="cuda"), torch.randn(100003, device="cuda")
    ref = ema - (1 - 0.99) * (ema - p)
    ops.ema_update_(ema, p, 0.99)
    assert maxdiff(ema, ref) < 1e-6


# ---------------------------------------------------------------------------------------------------
# norms
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("dim", [8, 64, 128, 200, 512, 768, 1024, 1536, 4096, 8192])
def test_layer_norm(dtype, dim):
    ops = _ops()
    torch.manual_seed(3)
    rows = 257
    x = (torch.randn(rows, dim, device="cuda") * 2 + 0.5).to(dtype).requires_grad_(True)
    w = (torch.randn(dim, device="cuda") * 0.5 + 1).to(dtype).requires_grad_(True)
    b = torch.randn(dim, device="cuda").to(dtype).requires_grad_(True)
    dy = torch.randn(rows, dim, device="cuda").to(dtype)
    y = ops.layer_norm(x, (dim,), w, b, 1e-5)
    y.backward(dy)
    xr, wr, br = (t.detach().float().requires_grad_(True) for t in (x, w, b))
    yr = F.layer_norm(xr, (dim,), wr, br, 1e-5)
    yr.backward(dy.float())
    tol = TOL[dtype]
    assert maxdiff(y, yr) < tol * 8
    assert maxdiff(x.grad, xr.grad) < tol * 16
    scale = max(1.0, wr.grad.abs().max().item())
    assert maxdiff(w.grad, wr.grad) / scale < tol * 4
    assert maxdiff(b.grad, br.grad) / max(1.0, br.grad.abs().max().item()) < tol * 4


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("dim", [64, 768, 1000, 2048])
def test_rms_norm(dtype, dim):
    ops = _ops()
    torch.manual_seed(4)
    rows = 130
    x = torch.randn(rows, dim, device="cuda").to(dtype).requires_grad_(True)
    w = (torch.randn(dim, device="cuda") * 0.5 + 1).to(dtype).requires_grad_(True)
    dy = torch.randn(rows, dim, device="cuda").to(dtype)
    y = ops.rms_norm(x, (dim,), w, 1e-5)
    y.backward(dy)
    xr, wr = (t.detach().float().requires_grad_(True) for t in (x, w))
    yr = xr * torch.rsqrt(xr.pow(2).mean(-1, keepdim=True) + 1e-5) * wr
    yr.backward(dy.float())
    tol = TOL[dtype]
    assert maxdiff(y, yr) < tol * 8
    assert maxdiff(x.grad, xr.grad) < tol * 16
    assert maxdiff(w.grad, wr.grad) / max(1.0, wr.grad.abs().max().item()) < tol * 4


def test_layer_norm_3d_and_module():
    from unicore.modules import LayerNorm

    ln = LayerNorm(768).cuda().half()
    x = torch.randn(4, 33, 768, device="cuda", dtype=torch.half)
    y = ln(x)
    ref = F.layer_norm(x.float(), (768,), ln.weight.float(), ln.bias.float(), 1e-5)
    assert maxdiff(y, ref) < 1e-2


# ---------------------------------------------------------------------------------------------------
# softmax_dropout (shapes follow the reference test-suite: 4-D and 5-D "triangle" broadcasts)
# ---------------------------------------------------------------------------------------------------
def _gen_mask(shape, dtype):
    m = (torch.rand(shape, device="cuda") > 0.8).to(dtype) * -3e4
    return m


def _check_softmax(x_shape, mask_shape, bias_shape, dtype):
    ops = _ops()
    torch.manual_seed(5)
    x = torch.randn(x_shape, device="cuda").to(dtype)
    mask = _gen_mask(mask_shape, dtype) if mask_shape else None
    bias = torch.randn(bias_shape, device="cuda").to(dtype).requires_grad_(True) if bias_shape else None
    xin = x.clone().requires_grad_(True)
    out = ops.softmax_dropout(xin, 0.0, True, mask=mask, bias=bias, inplace=False)
    dy = torch.randn_like(out)
    out.backward(dy)
    xr = x.float().requires_grad_(True)
    br = bias.detach().float().requires_grad_(True) if bias is not None else None
    z = xr
    if mask is not None:
        z = z + mask.float()
    if br is not None:
        z = z + br
    ref = F.softmax(z, dim=-1)
    ref.backward(dy.float())
    tol = 1e-3 if dtype != torch.bfloat16 else 8e-3
    assert maxdiff(out, ref) < tol
    assert maxdiff(xin.grad, xr.grad) < tol
    if bias is not None:
        assert maxdiff(bias.grad, br.grad) / max(1.0, br.grad.abs().max().item()) < tol * 8


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("k", [8, 64, 128, 256, 512, 1024, 1536, 2048, 100])
def test_softmax_4d(dtype, k):
    _check_softmax((4, 8, 16, k), (4, 1, 1, k), (4, 8, 16, k), dtype)
    _check_softmax((4, 8, 16, k), None, (1, 8, 16, k), dtype)
    _check_softmax((4, 8, 16, k), (4, 8, 16, k), None, dtype)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("k", [64, 256])
def test_softmax_tri(dtype, k):
    _check_softmax((2, 8, 4, 16, k), (2, 8, 1, 1, k), (1, 1, 4, 16, k), dtype)
    _check_softmax((2, 8, 4, 16, k), (2, 8, 4, 1, k), (1, 8, 4, 16, k), dtype)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32])
@pytest.mark.parametrize("k", [128, 512, 2048, 100])
def test_softmax_dropout_statistics_and_backward(dtype, k):
    ops = _ops()
    torch.manual_seed(6)
    p = 0.25
    x = torch.randn(64, 32, k, device="cuda").to(dtype)
    probs_ref = F.softmax(x.float(), dim=-1)
    xin = x.clone().requires_grad_(True)
    out = ops.softmax_dropout(xin, p, True, inplace=False)
    kept = out != 0
    frac = kept.float().mean().item()
    assert abs(frac - (1 - p)) < 0.01, frac
    # kept values are probs / (1-p)
    err = ((out.float() - probs_ref / (1 - p)).abs() * kept).max().item()
    assert err < (2e-3 if dtype != torch.bfloat16 else 1.6e-2)
    dy = torch.randn_like(out)
    out.backward(dy)
    # reference backward with the SAME mask
    xr = x.float().requires_grad_(True)
    ref = F.softmax(xr, dim=-1) * kept.float() / (1 - p)
    ref.backward(dy.float())
    assert maxdiff(xin.grad, xr.grad) < (2e-3 if dtype != torch.bfloat16 else 1.6e-2)


def test_softmax_inplace_contract():
    ops = _ops()
    x = torch.randn(8, 16, 256, device="cuda", dtype=torch.half)
    ref = F.softmax(x.float(), -1)
    out = ops.softmax_dropout(x, 0.0, False)  # eval: result is the (overwritten) input buffer
    assert out.data_ptr() == x.data_ptr()
    assert maxdiff(x, ref) < 1e-3
    x2 = torch.randn(8, 16, 256, device="cuda", dtype=torch.half)
    ref2 = F.softmax(x2.float(), -1)
    out2 = ops.softmax_dropout(x2, 0.5, True)
    assert maxdiff(x2, ref2) < 1e-3  # input now holds probabilities
    assert out2.data_ptr() != x2.data_ptr()


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32])
@pytest.mark.parametrize("k,p", [(128, 0.0), (248, 0.2), (100, 0.2), (2048, 0.0)])
def test_softmax_dropout_with_logits(dtype, k, p):
    """Logits mode: z = x + mask + bias is an output with its own gradient; -inf bias entries (padding) included."""
    ops = _ops()
    torch.manual_seed(11)
    B, H, Q = 3, 4, 24
    x = torch.randn(B, H, Q, k, device="cuda").to(dtype)
    bias = torch.randn(B, H, Q, k, device="cuda").to(dtype)
    bias[1, :, :, k - 5:] = float("-inf")
    bias[2, 1, 3, :] = float("-inf")  # a fully masked row must give zeros, not NaN
    pad = torch.zeros(B, 1, 1, k, device="cuda", dtype=dtype)
    pad[0, :, :, :3] = float("-inf")
    xin, bin_ = x.clone().requires_grad_(True), bias.clone().requires_grad_(True)
    x_before = xin.detach().clone()
    out, z = ops.softmax_dropout_with_logits(xin, p, True, mask=pad, bias=bin_)
    assert torch.equal(xin.detach(), x_before), "input must not be overwritten"
    z_ref = (x + pad) + bias if dtype != torch.float32 else x + pad + bias
    finite = torch.isfinite(z_ref)
    assert torch.equal(torch.isfinite(z), finite)
    assert maxdiff(torch.where(finite, z, torch.zeros_like(z)), torch.where(finite, z_ref, torch.zeros_like(z))) <= TOL[dtype] * 4
    kept = (out != 0) if p > 0 else torch.ones_like(out, dtype=torch.bool)
    zr = z.detach().float().masked_fill(~finite, float("-inf"))
    probs_ref = torch.nan_to_num(F.softmax(zr, dim=-1), nan=0.0)
    assert not torch.isnan(out).any()
    assert ((out.float() - probs_ref / (1 - p)).abs() * kept).max().item() < (2e-3 if dtype != torch.bfloat16 else 1.6e-2)
    if p > 0:
        live = probs_ref > 1e-4
        assert abs((kept & live).float().sum().item() / live.float().sum().item() - (1 - p)) < 0.02
    # gradients: through the probabilities AND directly into the logits output
    dy, dz = torch.randn_like(out), torch.randn_like(z)
    torch.autograd.backward([out, z], [dy, dz])
    safe = z.detach().float().masked_fill(~finite, -1e4).requires_grad_(True)
    alive = finite.any(dim=-1, keepdim=True).float()  # fully masked rows: zero probabilities, gradient = dz only
    ref = F.softmax(safe, dim=-1) * kept.float() * alive / (1 - p)
    torch.autograd.backward([ref, safe * 1.0], [dy.float(), dz.float()])
    tol = 2e-3 if dtype == torch.float16 else (2e-2 if dtype == torch.bfloat16 else 1e-5)
    scale = max(1.0, dz.abs().max().item())
    assert maxdiff(xin.grad, safe.grad) < tol * scale
    assert maxdiff(bin_.grad, safe.grad) < tol * scale
    # only the probability path: no gradient arrives for the logits
    xin2 = x.clone().requires_grad_(True)
    out2, _ = ops.softmax_dropout_with_logits(xin2, 0.0, True, mask=pad, bias=bias)
    out2.backward(dy)
    safe2 = safe.detach().requires_grad_(True)
    (F.softmax(safe2, dim=-1) * alive).backward(dy.float())
    assert maxdiff(xin2.grad, safe2.grad) < tol


# ---------------------------------------------------------------------------------------------------
# head split / merge
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32])
@pytest.mark.parametrize("B,L,H,D", [(3, 37, 64, 8), (2, 128, 12, 64), (1, 1, 5, 16)])
def test_split_merge_heads(dtype, B, L, H, D):
    ops = _ops()
    torch.manual_seed(12)
    scale = D ** -0.5
    x = torch.randn(B, L, 3 * H * D, device="cuda").to(dtype).requires_grad_(True)
    q, k, v = ops.split_heads(x, 3, H, scale)
    ref = x.detach().view(B, L, 3, H, D).permute(2, 0, 3, 1, 4)
    assert q.shape == (B, H, L, D) and q.is_contiguous() and k.is_contiguous() and v.is_contiguous()
    assert maxdiff(q, ref[0].float() * scale) <= TOL[dtype] and torch.equal(k, ref[1]) and torch.equal(v, ref[2])
    # gradient gathered by one kernel; a slice nobody used reads as zeros
    gq, gv = torch.randn_like(q), torch.randn_like(v)
    torch.autograd.backward([q, v], [gq, gv])
    g = x.grad.view(B, L, 3, H, D)
    assert maxdiff(g[:, :, 0], gq.permute(0, 2, 1, 3).float() * scale) <= TOL[dtype] * 4
    assert g[:, :, 1].abs().max().item() == 0 and torch.equal(g[:, :, 2], gv.permute(0, 2, 1, 3))
    # merge is the inverse (and split its backward)
    o = torch.randn(B, H, L, D, device="cuda").to(dtype).requires_grad_(True)
    m = ops.merge_heads(o)
    assert m.shape == (B, L, H * D) and torch.equal(m, o.detach().permute(0, 2, 1, 3).reshape(B, L, H * D))
    gm = torch.randn_like(m)
    m.backward(gm)
    assert torch.equal(o.grad, gm.view(B, L, H, D).permute(0, 2, 1, 3))
    back = ops.merge_heads(q.detach(), k.detach(), v.detach(), scale0=1.0 / scale)
    assert maxdiff(back, x) <= TOL[dtype] * 4


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("B,H,L", [(3, 64, 40), (2, 8, 24), (1, 16, 8)])
def test_pair_layout_kernels(dtype, B, H, L):
    """Register-tile transposes between head-major and pair-major, and the fused encoder tail."""
    ops = _ops()
    torch.manual_seed(13)
    x = torch.randn(B, H, L, L, device="cuda").to(dtype).requires_grad_(True)
    y = ops.heads_to_pair(x)
    assert y.shape == (B, L, L, H) and y.is_contiguous() and torch.equal(y, x.detach().permute(0, 2, 3, 1))
    gy = torch.randn_like(y)
    y.backward(gy)
    assert torch.equal(x.grad, gy.permute(0, 3, 1, 2))
    assert torch.equal(ops.pair_to_heads(y.detach()), x.detach())
    # encoder tail: z carries -inf in padded key columns (and a stray one elsewhere), z0 is finite
    pad = torch.zeros(B, L, dtype=torch.bool, device="cuda")
    pad[0, L - 3:] = True
    z0 = torch.randn(B, H, L, L, device="cuda").to(dtype).requires_grad_(True)
    z = (z0.detach().float() + torch.randn(B, H, L, L, device="cuda")).to(dtype)
    z = z.masked_fill(pad[:, None, None, :], float("-inf"))
    z[-1, 0, 1, 2] = float("-inf")
    z.requires_grad_(True)
    pair, delta = ops.pair_tail(z, z0, pad)
    zr, z0r = z.detach().float().requires_grad_(True), z0.detach().float().requires_grad_(True)
    pair_ref = zr.masked_fill(zr == float("-inf"), 0).permute(0, 2, 3, 1)
    delta_ref = (zr - z0r).masked_fill(pad[:, None, None, :], 0).permute(0, 2, 3, 1)
    assert torch.equal(pair.float(), pair_ref.detach())
    stray = torch.isinf(delta_ref.detach())
    assert stray.sum().item() == 1 and torch.equal(torch.isinf(delta), stray)
    assert maxdiff(delta.masked_fill(stray, 0), delta_ref.detach().masked_fill(stray, 0)) <= TOL[dtype] * 4
    gp, gd = torch.randn_like(pair), torch.randn_like(delta)
    gd = gd.masked_fill(stray, 0)
    torch.autograd.backward([pair, delta], [gp, gd])
    torch.autograd.backward([pair_ref, delta_ref], [gp.float(), gd.float()])
    assert maxdiff(z.grad, zr.grad) <= TOL[dtype] * 4 and maxdiff(z0.grad, z0r.grad) <= TOL[dtype]
    # one of the two outputs unused
    z2 = z.detach().clone().requires_grad_(True)
    p2, _ = ops.pair_tail(z2, z0.detach(), None)
    p2.backward(gp)
    live = ~torch.isinf(z.detach())
    assert maxdiff(z2.grad, gp.float().permute(0, 3, 1, 2) * live) <= TOL[dtype]


# ---------------------------------------------------------------------------------------------------
# fused element-wise
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_bias_gelu(dtype):
    ops = _ops()
    torch.manual_seed(7)
    x = torch.randn(300, 3072, device="cuda").to(dtype).requires_grad_(True)
    b = torch.randn(3072, device="cuda").to(dtype).requires_grad_(True)
    dy = torch.randn(300, 3072, device="cuda").to(dtype)
    y = ops.bias_gelu(x, b)
    y.backward(dy)
    xr, br = x.detach().float().requires_grad_(True), b.detach().float().requires_grad_(True)
    yr = F.gelu(xr + br)
    yr.backward(dy.float())
    tol = TOL[dtype]
    assert maxdiff(y, yr) < tol * 8
    assert maxdiff(x.grad, xr.grad) < tol * 8
    assert maxdiff(b.grad, br.grad) / br.grad.abs().max().item() < tol * 4


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_relative_position_bias_as_one_hot_gemm(dtype):
    """The rel-pos bias computed as W^T E (cached one-hot of the bucket table) equals the embedding lookup bit for bit,
    and its weight gradient equals the fp32 scatter-add."""
    from unicore.modules import TransformerEncoder

    torch.manual_seed(5)
    enc = TransformerEncoder(encoder_layers=1, embed_dim=96, ffn_embed_dim=128, attention_heads=12, max_seq_len=256,
                             rel_pos=True).cuda().to(dtype)
    x = torch.zeros(2, 200, 96, device="cuda", dtype=dtype)
    w = enc.relative_attention_bias.weight
    bias = enc.get_rel_pos_bias(x)
    bucket = enc.rp_bucket[:200, :200]
    ref = F.embedding(bucket, w).permute(2, 0, 1)
    assert bias.shape == (12, 200, 200) and torch.equal(bias, ref)
    g = torch.randn_like(bias)
    bias.backward(g)
    want = torch.zeros(w.shape, device="cuda", dtype=torch.float32)
    want.index_add_(0, bucket.reshape(-1), g.permute(1, 2, 0).reshape(-1, 12).float())
    assert maxdiff(w.grad, want) / want.abs().max().item() < TOL[dtype]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("vocab,dim,shape", [(30522, 768, (32, 512)), (100, 64, (7, 13)), (5000, 512, (1, 1))])
def test_embedding_sort_free_backward(dtype, vocab, dim, shape):
    """fp32-accumulated red scatter + finalize == the fp32 reference; heavy duplicates, padding rows, two calls in a row
    (the persistent scratch must come back clean), accumulate-in-place mode."""
    ops = _ops()
    torch.manual_seed(21)
    pad = 1
    w = (torch.randn(vocab, dim, device="cuda") * 0.1).to(dtype).requires_grad_(True)
    tok = torch.randint(0, vocab, shape, device="cuda")
    tok.view(-1)[::5] = 3          # one very frequent token
    tok.view(-1)[1::7] = pad       # padding positions contribute nothing
    dy = torch.randn(*shape, dim, device="cuda").to(dtype)
    for _ in range(2):
        w.grad = None
        y = ops.embedding(tok, w, pad)
        assert torch.equal(y, F.embedding(tok, w, pad))
        y.backward(dy)
        ref = torch.zeros(vocab, dim, device="cuda", dtype=torch.float32)
        keep = tok.view(-1) != pad
        ref.index_add_(0, tok.view(-1)[keep], dy.view(-1, dim).float()[keep])
        scale = max(1.0, ref.abs().max().item())
        assert maxdiff(w.grad, ref) / scale < TOL[dtype]
        assert w.grad[pad].abs().max().item() == 0.0
    # accumulate into an existing gradient buffer (what the gradient arena does)
    native = ops.native()
    from unicore_b200.ops import fused_ops

    scratch, touched = fused_ops._scratch_for(w)
    assert scratch.abs().max().item() == 0.0 and touched.max().item() == 0
    base = torch.randn(vocab, dim, device="cuda").to(dtype)
    acc = base.clone()
    native.embedding_bwd(dy, tok, pad, scratch, touched, acc, True)
    assert maxdiff(acc, base.float() + ref) / scale < TOL[dtype] * 2
    assert scratch.abs().max().item() == 0.0 and touched.max().item() == 0


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("rows,din,dout", [(16384, 768, 2304), (4001, 512, 512), (37, 64, 256), (65536, 128, 64),
                                            (12288, 64, 128)])
def test_linear_with_column_sum_bias_grad(dtype, rows, din, dout):
    ops = _ops()
    torch.manual_seed(14)
    x = (torch.randn(rows, din, device="cuda") * 0.5).to(dtype).requires_grad_(True)
    w = (torch.randn(dout, din, device="cuda") * 0.05).to(dtype).requires_grad_(True)
    b = torch.randn(dout, device="cuda").to(dtype).requires_grad_(True)
    dy = torch.randn(rows, dout, device="cuda").to(dtype)
    y = ops.linear(x.view(1, rows, din), w, b)
    assert y.shape == (1, rows, dout)
    y.backward(dy.view(1, rows, dout))
    xr, wr, br = (t.detach().float().requires_grad_(True) for t in (x, w, b))
    yr = F.linear(xr, wr, br)
    yr.backward(dy.float())
    assert maxdiff(y[0], yr) < TOL[dtype] * 8
    # the bias gradient is accumulated in fp32 and rounded once: error relative to its magnitude (~sqrt(rows))
    assert maxdiff(b.grad, br.grad) <= TOL[dtype] * max(1.0, br.grad.abs().max().item())
    assert maxdiff(x.grad, xr.grad) < TOL[dtype] * 8
    assert maxdiff(w.grad, wr.grad) <= TOL[dtype] * 2 * max(1.0, wr.grad.abs().max().item())


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_bias_dropout_add_layer_norm(dtype, p):
    ops = _ops()
    torch.manual_seed(8)
    rows, dim = 515, 768
    x = torch.randn(rows, dim, device="cuda").to(dtype).requires_grad_(True)
    bias = torch.randn(dim, device="cuda").to(dtype).requires_grad_(True)
    res = torch.randn(rows, dim, device="cuda").to(dtype).requires_grad_(True)
    w = (torch.randn(dim, device="cuda") * 0.3 + 1).to(dtype).requires_grad_(True)
    b = torch.randn(dim, device="cuda").to(dtype).requires_grad_(True)
    dy = torch.randn(rows, dim, device="cuda").to(dtype)
    y = ops.bias_dropout_add_layer_norm(x, bias, res, w, b, p, 1e-5, True)
    y.backward(dy)
    # recover the dropout mask from dx (dx is zero exactly where the element was dropped)
    if p > 0:
        keep = (x.grad != 0).float()
        assert abs(keep.mean().item() - (1 - p)) < 0.01
    else:
        keep = torch.ones(rows, dim, device="cuda")
    xr, biasr, resr, wr, br = (t.detach().float().requires_grad_(True) for t in (x, bias, res, w, b))
    h = resr + (xr + biasr) * keep / (1 - p)
    yr = F.layer_norm(h, (dim,), wr, br, 1e-5)
    yr.backward(dy.float())
    tol = TOL[dtype]
    assert maxdiff(y, yr) < tol * 16
    assert maxdiff(res.grad, resr.grad) < tol * 16
    assert maxdiff(x.grad, xr.grad) < tol * 16
    assert maxdiff(w.grad, wr.grad) / wr.grad.abs().max().item() < tol * 4
    assert maxdiff(bias.grad, biasr.grad) / biasr.grad.abs().max().item() < tol * 4


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("vocab", [30522, 1000, 37])
def test_softmax_cross_entropy(dtype, vocab):
    ops = _ops()
    torch.manual_seed(9)
    n = 301
    logits = (torch.randn(n, vocab, device="cuda") * 3).to(dtype).requires_grad_(True)
    target = torch.randint(0, vocab, (n,), device="cuda")
    target[::7] = 0  # ignored rows
    loss = ops.softmax_cross_entropy(logits, target, ignore_index=0)
    (loss * 2.0).backward()
    lr = logits.detach().float().requires_grad_(True)
    ref = F.nll_loss(F.log_softmax(lr, dim=-1), target, ignore_index=0, reduction="sum")
    (ref * 2.0).backward()
    assert abs(loss.item() - ref.item()) / abs(ref.item()) < 1e-4
    assert maxdiff(logits.grad, lr.grad) < (1e-5 if dtype == torch.float32 else 4e-3)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_vocab_projection_padded_xent(dtype):
    """LM head with a vocabulary that is not a multiple of 8: padded GEMMs + strided cross entropy."""
    from unicore import ops

    torch.manual_seed(0)
    n, d, V = 333, 256, 30522
    x = (torch.randn(n, d, device="cuda") * 0.5).to(dtype).requires_grad_(True)
    w = (torch.randn(V, d, device="cuda") * 0.05).to(dtype).requires_grad_(True)
    b = (torch.randn(V, device="cuda") * 0.1).to(dtype).requires_grad_(True)
    tgt = torch.randint(0, V, (n,), device="cuda")
    tgt[::7] = 1  # ignored
    logits = ops.vocab_projection(x, w, b)
    assert logits.shape == (n, V) and not logits.is_contiguous()
    loss = ops.softmax_cross_entropy(logits, tgt, ignore_index=1)
    loss.backward()
    xr, wr, br = (t.detach().float().requires_grad_(True) for t in (x, w, b))
    ref_logits = F.linear(xr, wr, br)
    ref = F.nll_loss(F.log_softmax(ref_logits, dim=-1), tgt, ignore_index=1, reduction="sum")
    ref.backward()
    assert abs(loss.item() - ref.item()) < 2e-2 * abs(ref.item())
    for g, gr in ((x.grad, xr.grad), (w.grad, wr.grad), (b.grad, br.grad)):
        assert g.shape == gr.shape
        tol = (3e-2 if dtype == torch.float16 else 8e-2) * max(1e-3, gr.abs().max().item())
        assert (g.float() - gr).abs().max().item() < tol


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_gaussian_basis(dtype):
    """Uni-Mol pair features: fused kernels vs the embedding + broadcast formulation in fp32."""
    from unicore import ops

    torch.manual_seed(0)
    B, L, K, E = 3, 40, 128, 961
    dist = (torch.rand(B, L, L, device="cuda") * 6).to(dtype)
    edge = torch.randint(0, E, (B, L, L), device="cuda")
    mul_w = (1 + 0.2 * torch.randn(E, 1, device="cuda")).to(dtype).requires_grad_(True)
    bias_w = (0.2 * torch.randn(E, 1, device="cuda")).to(dtype).requires_grad_(True)
    means = (torch.rand(1, K, device="cuda") * 3).to(dtype).requires_grad_(True)
    stds = (torch.rand(1, K, device="cuda") * 3 - 0.5).to(dtype).requires_grad_(True)  # some negative: |.| path
    y = ops.gaussian_basis(dist, edge, mul_w, bias_w, means, stds)
    assert y.shape == (B, L, L, K) and y.dtype == dtype
    dy = torch.randn_like(y)
    y.backward(dy)
    ref_in = [t.detach().float().requires_grad_(True) for t in (mul_w, bias_w, means, stds)]
    t = (ref_in[0].view(-1)[edge] * dist.float() + ref_in[1].view(-1)[edge]).unsqueeze(-1)
    std = ref_in[3].view(-1).abs() + 1e-5
    yr = torch.exp(-0.5 * ((t - ref_in[2].view(-1)) / std) ** 2) / ((2 * 3.14159) ** 0.5 * std)
    yr.backward(dy.float())
    tol = 2e-2 if dtype == torch.bfloat16 else 4e-3
    assert (y.float() - yr).abs().max().item() < tol * max(1.0, yr.abs().max().item())
    for got, ref in zip((mul_w, bias_w, means, stds), ref_in):
        scale = max(1.0, ref.grad.abs().max().item())
        assert (got.grad.float() - ref.grad.view_as(got.grad)).abs().max().item() < 3e-2 * scale


# ---------------------------------------------------------------------------------------------------
# softmax_dropout on every launch path, past the first sweep of the grid, against fp64
# ---------------------------------------------------------------------------------------------------
E32 = 2.0 ** -24
UNIT = {torch.float32: 2.0 ** -24, torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}  # unit roundoff
# row lengths in 16-byte vectors: threads per row < 32 (8), = 32 with 1..4 vectors per thread (32, 64, 96, 128),
# 64 threads (160, 256: 3 and 4 vectors), 256 threads (640, 1024); the scalar kernels take K = 99 (not a multiple of
# the vector width) and K past the longest vector row
SM_NVECS = [8, 32, 64, 96, 128, 160, 256, 640, 1024]
SM_SCALAR_K = [99, "long"]


def _sm_k(spec, dtype):
    epv = 16 // torch.empty((), dtype=dtype).element_size()
    return 1024 * epv + epv if spec == "long" else spec


def _sm_case(plan):
    if not plan["vec"]:
        return ("scalar",)
    t = plan["tpr"]
    return ("vec", "<32" if t < 32 else ("32" if t == 32 else ("256" if t == 256 else "64-128")), plan["vpt"])


def _sm_keep_scale(p):
    """1 / P(keep): the kernels compare 14 random bits against round(p * 2^14), so p is quantised to 1 / 16384."""
    return 1.0 if p == 0 else 16384.0 / (16384.0 - round(p * 16384.0))


def _sm_rows(K, dtype, Q):
    """Rows (a multiple of Q) that make every CTA of both kernels take 3 sweeps or more, with a ragged last sweep.
    Rows past the longest vector row run one sweep only: three would take gigabytes; the scalar kernels' later
    sweeps are covered by K = 99."""
    nat = _ops().native()
    if K > 1024 * (16 // torch.empty((), dtype=dtype).element_size()):
        return Q * 17
    sweep = max(nat.softmax_plan(1 << 40, K, dtype, True, k)["rows_per_sweep"] for k in ("fwd", "bwd"))
    rows = -(-(3 * sweep + sweep // 2 + 1) // Q) * Q
    for k in ("fwd", "bwd"):
        pl = nat.softmax_plan(rows, K, dtype, True, k)
        while rows % pl["rows_per_sweep"] == 0:
            rows += Q
        assert pl["sweeps"] >= 4, pl
    return rows


def _sm_chunks(rows, K):
    step = max(1, (1 << 21) // K)
    for r0 in range(0, rows, step):
        yield slice(r0, min(rows, r0 + step))


def _within(got, ref, bound, what):
    err = (got.double() - ref).abs()
    bad = err > bound
    if bad.any():
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError("{}: {} elements out of bound, first at {}: got {}, want {} +- {}".format(
            what, int(bad.sum()), i, got[i].item(), ref[i].item(), bound[i].item()))


def _check_sm_forward(z, probs, out, p, dtype):
    """probs = softmax(z), out = keep * probs / P(keep), with keep read from out; returns (keep, live) counts.
    Bound: one rounding of the output type plus fp32 error relative to the probability: the exponent's argument
    (2 |z - max| ulp), exp2 and the row sum (< 80 ulp)."""
    u, tiny = UNIT[dtype], torch.finfo(dtype).tiny * UNIT[dtype]
    scale = _sm_keep_scale(p)
    kept = live = 0
    for s in _sm_chunks(*z.shape):
        zd = z[s].double()
        yr = torch.softmax(zd, -1)
        comp = yr * E32 * (2 * (zd - zd.max(-1, keepdim=True).values).abs() + 80)
        if probs is not None:
            _within(probs[s], yr, u * (yr + comp) + comp + tiny, "probs")
        keep = out[s] != 0 if p > 0 else torch.ones_like(yr, dtype=torch.bool)
        ref = yr * keep * scale
        _within(out[s], ref, u * (ref + comp * scale) + comp * scale + tiny, "out")
        alive = yr > 1e-3 / z.shape[1]  # probabilities that cannot round to zero
        kept += int((keep & alive).sum())
        live += int(alive.sum())
    return kept, live


def _check_sm_backward(dy, probs, out, dx, p, dtype, z=None, addend=None):
    """dx = y * (d - sum(d * y)) (+ addend), d = keep * dy / P(keep), keep read from the forward's `out`.  y: the
    stored probabilities `probs`, or (logits mode) softmax(z) rebuilt by backward from z and the row log-sum-exp,
    with error e_y: one rounding (absolute below the normal range), the exponent's argument and the log-sum-exp."""
    u, tiny = UNIT[dtype], torch.finfo(dtype).tiny * UNIT[dtype]
    scale = _sm_keep_scale(p)
    for s in _sm_chunks(*dy.shape):
        if z is None:
            yd, e_y = probs[s].double(), 0.0
        else:
            zd = z[s].double()
            yd = torch.softmax(zd, -1)
            lse = torch.logsumexp(zd, -1, keepdim=True)
            e_y = yd * (u + E32 * (2 * (zd - lse).abs() + 2 * lse.abs() + 80)) + tiny
        keep = (out[s] != 0) if p > 0 else 1.0
        d = dy[s].double() * keep * scale
        dot = (d * yd).sum(-1, keepdim=True)
        ref = yd * (d - dot)
        comp = ((d - dot).abs() * e_y + yd * ((d.abs() * e_y).sum(-1, keepdim=True)
                                               + 72 * E32 * (d * yd).abs().sum(-1, keepdim=True))
                + 4 * E32 * ((d * yd).abs() + (yd * dot).abs()))
        if addend is not None:
            ref = ref + addend[s].double()
            comp = comp + 2 * E32 * addend[s].double().abs()
        _within(dx[s], ref, u * (ref.abs() + comp) + comp + tiny, "dx")


def _sm_rate(kept, live, p):
    if p > 0:
        q = 1 - 1 / _sm_keep_scale(p)
        assert abs(kept / live - (1 - q)) < 6 * math.sqrt(q * (1 - q) / live), kept / live


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32])
@pytest.mark.parametrize("k", SM_NVECS + SM_SCALAR_K)
@pytest.mark.parametrize("mode", ["plain", "in_place", "logits"])
def test_softmax_dropout_all_paths(mode, k, dtype):
    """Every vector case (threads per row, vectors per thread) and the scalar kernels, plain / in-place / logits mode,
    p in {0, 0.2}; each CTA runs several sweeps, and backward must regenerate exactly the forward's keep mask."""
    nat = _ops().native()
    epv = 16 // torch.empty((), dtype=dtype).element_size()
    K = k * epv if isinstance(k, int) and k in SM_NVECS else _sm_k(k, dtype)
    Q = 16
    rows = _sm_rows(K, dtype, Q)
    assert _sm_case(nat.softmax_plan(rows, K, dtype, True, "fwd"))[0] == ("vec" if k in SM_NVECS else "scalar")
    g = torch.Generator(device="cuda").manual_seed(K)
    x = (torch.randn(rows // Q, Q, K, device="cuda", generator=g) * 2).to(dtype)
    bias = torch.randn(1, Q, K, device="cuda", generator=g).to(dtype)
    dy = torch.randn(rows // Q, Q, K, device="cuda", generator=g).to(dtype)
    addend = torch.randn(rows // Q, Q, K, device="cuda", generator=g).to(dtype)
    for p in (0.0, 0.2):
        if mode == "logits":
            out, z, lse, seed, off = nat.softmax_dropout_logits_fwd(x, None, bias, p, True)
            u = UNIT[dtype]
            for s in _sm_chunks(rows // Q, Q * K):
                zr = x[s].double() + bias.double()
                _within(z[s], zr, u * zr.abs() + 2 * E32 * zr.abs(), "logits")
            kept, live = _check_sm_forward(z.view(rows, K), None, out.view(rows, K), p, dtype)
            dx = nat.softmax_dropout_logits_bwd(dy, z, lse, addend, p, seed, off)
            _check_sm_backward(dy.view(rows, K), None, out.view(rows, K), dx.view(rows, K), p, dtype,
                               z=z.view(rows, K), addend=addend.view(rows, K))
        else:
            xin = x.clone()
            out, probs, seed, off = nat.softmax_dropout_fwd(xin, None, None, p, True, mode == "in_place")
            assert (probs.data_ptr() == xin.data_ptr()) == (mode == "in_place")
            kept, live = _check_sm_forward(x.view(rows, K), probs.view(rows, K), out.view(rows, K), p, dtype)
            dx = nat.softmax_dropout_bwd(dy, probs, p, seed, off)
            _check_sm_backward(dy.view(rows, K), probs.view(rows, K), out.view(rows, K), dx.view(rows, K), p, dtype)
        _sm_rate(kept, live, p)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32])
@pytest.mark.parametrize("nvec", [8, 128, 256])
def test_softmax_dropout_vector_and_scalar_paths_agree(dtype, nvec):
    """The same rows and Philox state through the vector kernels (aligned buffers) and the scalar kernels (a
    contiguous view at an odd element offset): identical keep masks, probabilities equal to rounding."""
    nat = _ops().native()
    epv = 16 // torch.empty((), dtype=dtype).element_size()
    K, Q = nvec * epv, 8
    rows = _sm_rows(K, dtype, Q)
    assert nat.softmax_plan(rows, K, dtype, True, "fwd")["vec"] and nat.softmax_plan(rows, K, dtype, True, "bwd")["vec"]
    assert not nat.softmax_plan(rows, K, dtype, False, "fwd")["vec"]
    assert not nat.softmax_plan(rows, K, dtype, False, "bwd")["vec"]
    g = torch.Generator(device="cuda").manual_seed(nvec)
    xbuf = (torch.randn(rows * K + 1, device="cuda", generator=g) * 2).to(dtype)
    dbuf = torch.randn(rows * K + 1, device="cuda", generator=g).to(dtype)
    xm, dym = xbuf[1:].view(rows // Q, Q, K), dbuf[1:].view(rows // Q, Q, K)
    assert xm.data_ptr() % 16 != 0
    res = []
    for xi, di in ((xm.clone(), dym.clone()), (xm, dym)):
        torch.cuda.manual_seed(5)
        out, probs, seed, off = nat.softmax_dropout_fwd(xi, None, None, 0.2, True, False)
        dx = nat.softmax_dropout_bwd(di, probs, 0.2, seed, off)
        res.append((out, probs, dx, (seed, off)))
    (oa, pa, da, sa), (om, pm, dm, sm) = res
    assert sa == sm
    assert torch.equal(oa != 0, om != 0)
    for probs, out, dx in ((pa, oa, da), (pm, om, dm)):
        kept, live = _check_sm_forward(xm.reshape(rows, K), probs.view(rows, K), out.view(rows, K), 0.2, dtype)
        _sm_rate(kept, live, 0.2)
        _check_sm_backward(dym.reshape(rows, K), probs.view(rows, K), out.view(rows, K), dx.view(rows, K), 0.2, dtype)


def test_softmax_dispatch_coverage():
    """The test row lengths reach every case the softmax launchers can dispatch to (launches no kernel)."""
    nat = _ops().native()
    for dtype in (torch.float16, torch.bfloat16, torch.float32):
        epv = 16 // torch.empty((), dtype=dtype).element_size()
        reachable = {_sm_case(nat.softmax_plan(64, K, dtype, True, kind))
                     for K in range(1, 1024 * epv + 2 * epv) for kind in ("fwd", "bwd")}
        tested = {_sm_case(nat.softmax_plan(64, n * epv, dtype, True, kind)) for n in SM_NVECS for kind in ("fwd", "bwd")}
        tested |= {_sm_case(nat.softmax_plan(64, _sm_k(k, dtype), dtype, True, "fwd")) for k in SM_SCALAR_K}
        assert tested == reachable, (dtype, sorted(reachable - tested))
        assert not nat.softmax_plan(64, 64 * epv, dtype, False, "fwd")["vec"]
