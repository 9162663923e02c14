"""Causal attention in the fused kernels (``causal=True``: key j is visible to query i iff j <= i, top-left aligned for
any Lq, Lk), and the decoder self-attention that runs on it.

Checked: O and LSE against an fp32 reference with the mask; bitwise agreement with the plain kernel given the future
mask as bias (O, LSE, dK, dV, dBias and the keep words of visible keys; dQ up to the order of its fp32 reduction); the
backward against fp64 with the keep bits the host derives from the Philox stream; exact zeros of dBias above the
diagonal and of dK / dV at keys no query sees; the packed entry point; rows whose visible keys are all padded; the
logits mode fallback; and the modules (SelfMultiheadAttention, TransformerDecoder) against their materialised paths.
"""
import copy
import math

import numpy as np
import pytest
import torch

from test_gpu_attention_dropout_stream import _assert_within, host_keep_words

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]
DT_IDS = ["fp16", "bf16"]
UNIT = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
HEAD_DIMS = [8, 32, 64, 96, 128]
P_DROP = 0.2
# (B, H, Lq, Lk): ragged against both key-tile sizes; one tile; Lq > Lk; Lq < Lk (key tiles no query sees); and a grid
# of more than one wave (4 * 12 * 16 = 768 CTAs)
SHAPES = {"ragged": (2, 3, 200, 200), "one_tile": (2, 2, 64, 64), "lq_gt_lk": (1, 2, 136, 72),
          "lq_lt_lk": (1, 2, 72, 200)}
BIG = (4, 12, 1024, 1024)


def _ops():
    from unicore import ops

    assert ops.USE_NATIVE, "native kernels must be active on the GPU box"
    return ops


def _inputs(B, H, Lq, Lk, D, dtype, seed, bias_batch=1):
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = (torch.randn(B, Lq, H, D, device="cuda", generator=g) * 0.6).to(dtype)
    k = (torch.randn(B, Lk, H, D, device="cuda", generator=g) * 0.6).to(dtype)
    v = torch.randn(B, Lk, H, D, device="cuda", generator=g).to(dtype)
    bias = torch.randn(bias_batch, H, Lq, Lk, device="cuda", generator=g).to(dtype)
    # trailing keys of batch 0 and a block of batch -1 are padded; every query still sees key 0
    kpm = torch.zeros(B, Lk, dtype=torch.bool, device="cuda")
    kpm[0, Lk - Lk // 4:] = True
    kpm[-1, 8:16] = True
    return q, k, v, bias, kpm


def _future(Lq, Lk, dtype=torch.float32):
    return torch.full((Lq, Lk), float("-inf"), device="cuda", dtype=dtype).triu(1)


def _visible(Lq, Lk):
    return torch.ones(Lq, Lk, dtype=torch.bool, device="cuda").tril()


def _fwd(q, k, v, bias, kpm, scale, causal, rng_seed, p=P_DROP):
    torch.cuda.manual_seed(rng_seed)
    gen = torch.cuda.default_generators[torch.cuda.current_device()]
    seed, offset = gen.initial_seed(), gen.get_offset()
    out, lse, bits = _ops().native().fmha_fwd(q, k, v, bias, kpm, p, scale, causal=causal)
    return out, lse, bits, seed, offset


# ---- 1. forward against fp32 ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("bias_mode", ["none", "shared", "batch"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("D", HEAD_DIMS)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_forward_against_fp32(shape, D, dtype, bias_mode):
    B, H, Lq, Lk = SHAPES[shape]
    q, k, v, bias, kpm = _inputs(B, H, Lq, Lk, D, dtype, seed=D, bias_batch=B if bias_mode == "batch" else 1)
    if bias_mode == "none":
        bias, kpm = None, None
    scale = 1.0 / math.sqrt(D)
    out, lse, _, _, _ = _fwd(q, k, v, bias, kpm, scale, True, 0, p=0.0)
    z = torch.einsum("bqhd,bkhd->bhqk", q.float(), k.float()) * scale + _future(Lq, Lk)
    if bias is not None:
        z = z + bias.float()
    if kpm is not None:
        z = z.masked_fill(kpm[:, None, None, :], float("-inf"))
    ref = torch.einsum("bhqk,bkhd->bqhd", torch.softmax(z, dim=-1), v.float())
    tol = 4e-3 if dtype == torch.float16 else 2e-2
    torch.testing.assert_close(out.float(), ref, atol=tol, rtol=tol)
    torch.testing.assert_close(lse, torch.logsumexp(z, dim=-1), atol=1e-3, rtol=1e-4)


# ---- 2. the same result as the explicit future mask ----------------------------------------------------------------
def _equal_to_explicit_mask(B, H, Lq, Lk, D, dtype, bias_mode):
    scale = 1.0 / math.sqrt(D)
    q, k, v, bias, kpm = _inputs(B, H, Lq, Lk, D, dtype, seed=3 + D, bias_batch=B if bias_mode == "batch" else 1)
    fm = _future(Lq, Lk, dtype)
    if bias_mode == "none":   # the mask alone is the explicit run's bias
        bias, masked = None, fm.view(1, 1, Lq, Lk).expand(1, H, Lq, Lk).contiguous()
    else:
        masked = (bias + fm).contiguous()
    nat = _ops().native()
    out_c, lse_c, bits_c, _, _ = _fwd(q, k, v, bias, kpm, scale, True, 77)
    out_n, lse_n, bits_n, _, _ = _fwd(q, k, v, masked, kpm, scale, False, 77)
    assert torch.equal(out_c, out_n) and torch.equal(lse_c, lse_n)
    # keep words holding at least one visible key: word w of row i is such a word iff 32 w <= i
    nw = bits_n.shape[-1]
    vis_w = (32 * torch.arange(nw, device="cuda"))[None, :] <= torch.arange(Lq, device="cuda")[:, None]
    assert torch.equal(bits_c[..., vis_w], bits_n[..., vis_w])

    dout = torch.randn(B, Lq, H, D, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5)).to(dtype)
    need = bias is not None
    dq_c, dk_c, dv_c, db_c = nat.fmha_bwd(dout, q, k, v, out_c, lse_c, bias, kpm, P_DROP, scale, bits_c, need, False,
                                          causal=True)
    dq_n, dk_n, dv_n, db_n = nat.fmha_bwd(dout, q, k, v, out_n, lse_n, masked, kpm, P_DROP, scale, bits_n, need, False)
    assert torch.equal(dk_c, dk_n) and torch.equal(dv_c, dv_n)
    if need:
        assert torch.equal(db_c, db_n)
    # dQ: the same fp32 terms (the skipped tiles add exact zeros), summed in another order, then rounded once
    u = UNIT[dtype]
    bound = 2 * u * dq_n.double().abs() + 2.0 ** -18 * dq_n.double().abs().max()
    _assert_within(dq_c, dq_n.double(), bound, "dQ")


@pytest.mark.parametrize("bias_mode", ["none", "shared", "batch"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("D", HEAD_DIMS)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_equal_to_explicit_future_mask(shape, D, dtype, bias_mode):
    _equal_to_explicit_mask(*SHAPES[shape], D, dtype, bias_mode)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("D", [64, 128])
def test_equal_to_explicit_future_mask_waves(D, dtype):
    _equal_to_explicit_mask(*BIG, D, dtype, "shared")


# ---- 3. backward against fp64 with the host keep bits --------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("D", HEAD_DIMS)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_backward_against_fp64_with_host_bits(shape, D, dtype):
    B, H, Lq, Lk = SHAPES[shape]
    u = UNIT[dtype]
    scale = 1.0 / math.sqrt(D)
    q, k, v, bias, kpm = _inputs(B, H, Lq, Lk, D, dtype, seed=11 + D, bias_batch=B)
    out, lse, bits, seed, offset = _fwd(q, k, v, bias, kpm, scale, True, 99 + D)
    host, keep_np, keep_scale = host_keep_words(seed, offset, B, H, Lq, Lk, P_DROP)
    vis_w = (32 * np.arange(host.shape[-1]))[None, :] <= np.arange(Lq)[:, None]
    assert np.array_equal(bits.cpu().numpy()[..., vis_w], host[..., vis_w])
    keep = torch.from_numpy(keep_np).to("cuda", torch.float64)

    qd, kd, vd = q.double(), k.double(), v.double()
    vis = _visible(Lq, Lk)
    z = torch.einsum("bqhd,bkhd->bhqk", qd, kd) * scale + bias.double()
    zabs = (torch.einsum("bqhd,bkhd->bhqk", qd.abs(), kd.abs()) * scale + bias.double().abs()).masked_fill(~vis, 0.0)
    z = z.masked_fill(~vis, float("-inf")).masked_fill(kpm[:, None, None, :], float("-inf"))
    lse_ref = torch.logsumexp(z, dim=-1)
    pr = torch.exp(z - lse_ref[..., None])
    pd = pr * keep * keep_scale
    o_ref = torch.einsum("bhqk,bkhd->bqhd", pd, vd)
    oabs = torch.einsum("bhqk,bkhd->bqhd", pd, vd.abs())
    rel_z = 2.0 ** -16 * zabs.amax(dim=-1) + 1e-5
    rz = rel_z.permute(0, 2, 1)[..., None]
    sub = 2.0 ** -25 if dtype == torch.float16 else 0.0
    _assert_within(out, o_ref, (2 * u + rz) * oabs + u * o_ref.abs() + sub * Lk * v.abs().max().item(), "O")
    _assert_within(lse, lse_ref, 2.0 ** -16 * zabs.amax(dim=-1) + 1e-5 * (1 + lse_ref.abs()), "LSE")

    dout = torch.randn(B, Lq, H, D, device="cuda", generator=torch.Generator(device="cuda").manual_seed(7 + D)).to(dtype)
    dq, dk, dv, dbias = _ops().native().fmha_bwd(dout, q, k, v, out, lse, bias, kpm, P_DROP, scale, bits, True, False,
                                                 causal=True)
    dod = dout.double()
    delta = (dod * out.double()).sum(-1).permute(0, 2, 1)[..., None]
    delta_abs = (dod.abs() * out.double().abs()).sum(-1).permute(0, 2, 1)[..., None]
    dp = torch.einsum("bqhd,bkhd->bhqk", dod, vd)
    dp_abs = torch.einsum("bqhd,bkhd->bhqk", dod.abs(), vd.abs())
    dpd = dp * keep * keep_scale
    ds = pr * (dpd - delta)
    e_ds = pr * (rel_z[..., None] * (dpd - delta).abs() + 2.0 ** -16 * (dp_abs * keep * keep_scale + delta_abs)) \
        + u * ds.abs()
    dv_ref = torch.einsum("bhqk,bqhd->bkhd", pd, dod)
    dv_bnd = torch.einsum("bhqk,bqhd->bkhd", pd * (u + rel_z[..., None]), dod.abs()) + u * dv_ref.abs()
    _assert_within(dv, dv_ref, dv_bnd + sub * Lq * keep_scale * dout.abs().max().item() + 1e-6, "dV")
    dk_ref = torch.einsum("bhqk,bqhd->bkhd", ds, qd) * scale
    dk_bnd = torch.einsum("bhqk,bqhd->bkhd", e_ds, qd.abs()) * scale + u * dk_ref.abs()
    _assert_within(dk, dk_ref, dk_bnd + sub * Lq * scale * q.abs().max().item() + 1e-6, "dK")
    dq_ref = torch.einsum("bhqk,bkhd->bqhd", ds, kd) * scale
    dq_bnd = torch.einsum("bhqk,bkhd->bqhd", e_ds, kd.abs()) * scale + u * dq_ref.abs()
    _assert_within(dq, dq_ref, dq_bnd + sub * Lk * scale * k.abs().max().item() + 1e-6, "dQ")
    _assert_within(dbias, ds, e_ds + sub + 1e-6, "dBias")


# ---- 4. exact zeros where no query looks ---------------------------------------------------------------------------
@pytest.mark.parametrize("bias_batch", ["shared", "batch"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_zero_gradients_where_no_query_looks(shape, dtype, bias_batch):
    B, H, Lq, Lk = SHAPES[shape]
    D, scale = 64, 0.125
    q, k, v, bias, kpm = _inputs(B, H, Lq, Lk, D, dtype, seed=21, bias_batch=B if bias_batch == "batch" else 1)
    out, lse, bits, _, _ = _fwd(q, k, v, bias, kpm, scale, True, 5)
    dout = torch.randn_like(out)
    # best effort against reads of unwritten dS: the allocator hands the freed NaN block to the backward's scratch
    poison = torch.full((B * H * Lq * Lk * 2,), float("nan"), dtype=dtype, device="cuda")
    del poison
    dq, dk, dv, dbias = _ops().native().fmha_bwd(dout, q, k, v, out, lse, bias, kpm, P_DROP, scale, bits, True, False,
                                                 causal=True)
    above = ~_visible(Lq, Lk)
    assert bool((dbias[..., above] == 0).all()), "dBias above the diagonal must be exactly 0"
    assert bool(torch.isfinite(dbias).all())
    if Lk > Lq:
        assert bool((dk[:, Lq:] == 0).all()) and bool((dv[:, Lq:] == 0).all())
    assert bool(torch.isfinite(dq).all() and torch.isfinite(dk).all() and torch.isfinite(dv).all())


# ---- 5. the packed entry point ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("D", [64, 96])
@pytest.mark.parametrize("shape", ["ragged", "one_tile"])
def test_packed_equals_unpacked(shape, D, dtype):
    ops = _ops()
    B, H, L, _ = SHAPES[shape]
    g = torch.Generator(device="cuda").manual_seed(D)
    qkv = (torch.randn(B, L, 3, H, D, device="cuda", generator=g) * 0.6).to(dtype)
    bias = torch.randn(1, H, L, L, device="cuda", generator=g).to(dtype)
    kpm = torch.zeros(B, L, dtype=torch.bool, device="cuda")
    kpm[0, L - 8:] = True
    dout = torch.randn(B, L, H, D, device="cuda", generator=g).to(dtype)

    def run(packed):
        x = qkv.clone().requires_grad_(True)
        b = bias.clone().requires_grad_(True)
        torch.cuda.manual_seed(3)
        if packed:
            o = ops.fused_attention_qkvpacked(x, b, kpm, P_DROP, True, None, causal=True)
        else:
            o = ops.fused_attention(x[:, :, 0], x[:, :, 1], x[:, :, 2], b, kpm, P_DROP, True, None, causal=True)
        o.backward(dout)
        return o, x.grad, b.grad

    o_p, g_p, b_p = run(True)
    o_u, g_u, b_u = run(False)
    assert torch.equal(o_p, o_u)
    assert torch.equal(g_p[:, :, 1:], g_u[:, :, 1:]) and torch.equal(b_p, b_u)
    u = UNIT[dtype]
    dq = g_u[:, :, 0].double()
    _assert_within(g_p[:, :, 0], dq, 2 * u * dq.abs() + 2.0 ** -18 * dq.abs().max(), "dQ")


# ---- 6. rows with no visible key --------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("D", [64, 128])
def test_rows_whose_visible_keys_are_all_padded(D, dtype):
    """The kernels' contract for a fully masked row: O = 0, LSE = -inf, and it contributes nothing to any gradient.
    Under the causal mask, rows 0..15 of batch 1 see keys 0..15 only, and those are padded."""
    ops = _ops()
    B, H, L = 2, 2, 136
    g = torch.Generator(device="cuda").manual_seed(1)
    q, k, v = [(torch.randn(B, L, H, D, device="cuda", generator=g) * 0.6).to(dtype).requires_grad_(True)
               for _ in range(3)]
    bias = torch.randn(1, H, L, L, device="cuda", generator=g).to(dtype).requires_grad_(True)
    kpm = torch.zeros(B, L, dtype=torch.bool, device="cuda")
    kpm[1, :16] = True
    o = ops.fused_attention(q, k, v, bias, kpm, 0.0, True, None, causal=True)
    assert bool((o[1, :16] == 0).all())
    o.backward(torch.randn_like(o))
    for t in (q.grad, k.grad, v.grad, bias.grad):
        assert bool(torch.isfinite(t).all())
    assert bool((q.grad[1, :16] == 0).all())
    ref = ops.attention_reference(q.detach().float(), k.detach().float(), v.detach().float(), bias.detach().float(),
                                  kpm, 0.0, False, None, causal=True)
    tol = 4e-3 if dtype == torch.float16 else 2e-2
    torch.testing.assert_close(o[0].float(), ref[0], atol=tol, rtol=tol)
    torch.testing.assert_close(o[1, 16:].float(), ref[1, 16:], atol=tol, rtol=tol)


# ---- 7. logits mode ------------------------------------------------------------------------------------------------
def test_causal_with_logits_is_the_reference():
    ops = _ops()
    q, k, v, bias, kpm = _inputs(2, 3, 200, 200, 64, torch.float16, seed=2)
    out, z = ops.fused_attention(q, k, v, bias, kpm, 0.0, True, None, return_logits=True, causal=True)
    ref, zr = ops.attention_reference(q, k, v, bias, kpm, 0.0, True, 0.125, return_logits=True, causal=True)
    assert torch.equal(out, ref) and torch.equal(z, zr)
    with pytest.raises(RuntimeError, match="causal"):
        ops.native().fmha_bwd(torch.zeros_like(q), q, k, v, torch.zeros_like(q),
                              torch.zeros(2, 3, 200, device="cuda"), None, None, 0.0, 0.125, None, False, False,
                              torch.zeros(2, 3, 200, 200, dtype=q.dtype, device="cuda"), causal=True)


# ---- 8. modules ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_self_attention_module_fused_matches_materialised(dtype):
    from unicore.modules import SelfMultiheadAttention

    torch.manual_seed(0)
    attn = SelfMultiheadAttention(768, 8, dropout=0.0).cuda().to(dtype)
    x = torch.randn(2, 136, 768, device="cuda").to(dtype)
    kpm = torch.zeros(2, 136, dtype=torch.bool, device="cuda")
    kpm[1, 120:] = True
    bias = torch.randn(1, 8, 136, 136, device="cuda").to(dtype)
    fused = attn(x, key_padding_mask=kpm, attn_bias=bias, causal=True)
    mat, logits, _ = attn(x, key_padding_mask=kpm, attn_bias=bias, return_attn=True, causal=True)
    tol = 4e-3 if dtype == torch.float16 else 3e-2
    torch.testing.assert_close(fused.float(), mat.float(), atol=tol, rtol=tol)
    assert bool(torch.isinf(logits.view(2, 8, 136, 136)[..., ~_visible(136, 136)]).all())


def _decoder_pair(dtype):
    from unicore.modules import TransformerDecoder

    torch.manual_seed(0)
    ref = TransformerDecoder().cuda().eval()
    with torch.no_grad():
        for p in ref.parameters():   # non-trivial LayerNorm and bias parameters
            p.add_(torch.randn_like(p) * 0.02)
    return ref, copy.deepcopy(ref).to(dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_decoder_matches_fp32_materialised_path(dtype):
    ref, model = _decoder_pair(dtype)
    B, L, Le = 2, 136, 72
    g = torch.Generator(device="cuda").manual_seed(4)
    emb = torch.randn(B, L, 768, device="cuda", generator=g)
    enc = torch.randn(B, Le, 768, device="cuda", generator=g)
    pad = torch.zeros(B, L, dtype=torch.bool, device="cuda")
    pad[1, L - 24:] = True
    enc_pad = torch.zeros(B, Le, dtype=torch.bool, device="cuda")
    enc_pad[0, Le - 8:] = True
    gout = torch.randn(B, L, 768, device="cuda", generator=g)
    y_ref = ref(emb, encoder_out=enc, padding_mask=pad, encoder_padding_mask=enc_pad)
    y_ref.backward(gout)
    y = model(emb.to(dtype), encoder_out=enc.to(dtype), padding_mask=pad, encoder_padding_mask=enc_pad)
    y.backward(gout.to(dtype))
    tol = 2e-2 if dtype == torch.float16 else 6e-2

    def rel(a, b):
        return ((a.float() - b).norm() / b.norm().clamp_min(1e-12)).item()

    assert rel(y, y_ref) < tol
    names = dict(ref.named_parameters())
    assert "relative_attention_bias.weight" in names
    bad = []
    for n, p in model.named_parameters():
        r = names[n]
        assert p.grad is not None and r.grad is not None, n
        a, b = p.grad, r.grad
        # a key-projection bias shifts every logit of a query row by the same amount: its exact gradient is 0, and
        # both paths return rounding noise there
        if n.endswith("k_proj.bias"):
            continue
        if n.endswith("self_attn.in_proj.bias"):
            a, b = torch.cat([a[:768], a[1536:]]), torch.cat([b[:768], b[1536:]])
        if not rel(a, b) < tol:
            bad.append((n, rel(a, b)))
    assert not bad, bad


def test_decoder_self_attention_calls_are_causal(monkeypatch):
    import unicore_b200.ops.attention_ops as attention_ops

    ops = _ops()
    _, model = _decoder_pair(torch.float16)
    real = ops.native()
    calls = []

    class Spy:
        def __getattr__(self, name):
            return getattr(real, name)

        def fmha_fwd(self, q, k, v, bias, kpm, p, scale, causal=False):
            calls.append((q.shape[1], k.shape[1], causal, bias, kpm))
            return real.fmha_fwd(q, k, v, bias, kpm, p, scale, causal=causal)

    monkeypatch.setattr(attention_ops, "native", lambda: Spy())
    B, L, Le = 2, 136, 72
    H = model.attention_heads
    emb = torch.randn(B, L, 768, device="cuda").half()
    enc = torch.randn(B, Le, 768, device="cuda").half()
    pad = torch.zeros(B, L, dtype=torch.bool, device="cuda")
    pad[1, L - 24:] = True
    # with an attn_mask as well, the padding still reaches the kernel as the [B, L] key mask, not as -inf in the bias
    for attn_mask in (None, torch.randn(B * H, L, L, device="cuda").half()):
        calls.clear()
        model(emb, encoder_out=enc, padding_mask=pad, attn_mask=attn_mask).float().sum().backward()
        self_calls = [c for c in calls if c[1] == L]
        cross_calls = [c for c in calls if c[1] == Le]
        assert len(self_calls) == len(model.layers) and len(cross_calls) == len(model.layers)
        for _, _, causal, bias, kpm in self_calls:
            assert causal and bias is not None and not bool(torch.isinf(bias).any())
            assert kpm is not None and torch.equal(kpm, pad)
        assert not any(c[2] for c in cross_calls)
