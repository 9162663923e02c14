"""Grouped-query attention in the wgmma forward, the backward and the decode kernels.

Query head h reads key / value head h // G.  Each query head does the arithmetic of the same call on K / V expanded
with ``repeat_interleave(G, dim=2)``, so the forward (O, LSE, keep bits, logits), dQ and dBias are bitwise those of
the expanded call; dK / dV are the group sums, checked against an fp64 reference.  Decode and chunk steps, the cache
append, the packed module path and a GQA ``TransformerDecoder`` (eager and captured steps) are covered as well."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]
DT_IDS = ["fp16", "bf16"]
UNIT = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
GRAD_TOL = {torch.float16: 1e-2, torch.bfloat16: 5e-2}   # relative norm error against fp64
STEP_TOL = {torch.float16: 2e-2, torch.bfloat16: 6e-2}   # relative norm per step, as the eager decoder tests
HEADS = [(12, 6), (12, 4), (12, 1), (8, 2)]
HEAD_IDS = ["12x6", "12x4", "12x1", "8x2"]
HEAD_DIMS = [8, 64, 96, 128]
P_DROP = 0.2


def _ops():
    from unicore import ops

    assert ops.USE_NATIVE, "native kernels must be active on the GPU box"
    return ops


def _bits(t):
    return t.view(torch.int16) if t.dtype in (torch.float16, torch.bfloat16) else t


def _eq(a, b, what):
    assert a.shape == b.shape and torch.equal(_bits(a), _bits(b)), what


def _rel(got, want):
    return ((got.double() - want.double()).norm() / want.double().norm().clamp(min=1e-30)).item()


def _x(g, dtype, *shape):
    return torch.randn(*shape, device="cuda", generator=g).to(dtype)


def _case(H, H_kv, D, dtype, seed, B=2, Lq=136, Lk=200):
    g = torch.Generator(device="cuda").manual_seed(seed)
    q, k, v = _x(g, dtype, B, Lq, H, D), _x(g, dtype, B, Lk, H_kv, D), _x(g, dtype, B, Lk, H_kv, D)
    bias = _x(g, dtype, B, H, Lq, Lk)
    kpm = torch.zeros(B, Lk, dtype=torch.bool, device="cuda")
    kpm[1, Lk - 37:] = True
    return q, k, v, bias, kpm


def _expand(t, G):
    return t.repeat_interleave(G, dim=2)


# ---- forward: bitwise the expanded call ----------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("D", HEAD_DIMS)
@pytest.mark.parametrize("H,H_kv", HEADS, ids=HEAD_IDS)
def test_forward_bitwise_equals_expanded(H, H_kv, D, dtype):
    nat = _ops().native()
    G = H // H_kv
    q, k, v, bias, kpm = _case(H, H_kv, D, dtype, H * 1000 + H_kv * 100 + D)
    ke, ve = _expand(k, G), _expand(v, G)
    scale = D ** -0.5
    cases = [("per-batch bias, padding, dropout", dict(bias=bias, kpm=kpm, p=P_DROP, causal=False)),
             ("shared bias, dropout, causal", dict(bias=bias[:1].contiguous(), kpm=None, p=P_DROP, causal=True)),
             ("padding, causal", dict(bias=None, kpm=kpm, p=0.0, causal=True)),
             ("plain", dict(bias=None, kpm=None, p=0.0, causal=False))]
    for what, c in cases:
        runs = []
        for kk, vv in ((k, v), (ke, ve)):
            torch.cuda.manual_seed(7)
            runs.append(nat.fmha_fwd(q, kk, vv, c["bias"], c["kpm"], c["p"], scale, causal=c["causal"]))
        (o, lse, bits), (oe, lsee, bitse) = runs
        _eq(o, oe, what + ": O")
        _eq(lse, lsee, what + ": LSE")
        if c["p"] > 0:
            if c["causal"]:   # the causal forward writes the keep words of the key tiles it walks: 32 w <= query
                rows = torch.arange(bits.shape[2], device="cuda")[:, None]
                walked = (32 * torch.arange(bits.shape[3], device="cuda"))[None, :] <= rows
                bits, bitse = bits[:, :, walked], bitse[:, :, walked]
            _eq(bits, bitse, what + ": keep bits")
    for b in (bias, bias[:1].contiguous()):   # logits mode
        runs = []
        for kk, vv in ((k, v), (ke, ve)):
            torch.cuda.manual_seed(9)
            runs.append(nat.fmha_fwd_logits(q, kk, vv, b, kpm, P_DROP, scale))
        for x, y, name in zip(runs[0], runs[1], ("O", "LSE", "keep bits", "logits")):
            _eq(x, y, "logits mode: " + name)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("D", HEAD_DIMS)
@pytest.mark.parametrize("H,H_kv", HEADS, ids=HEAD_IDS)
def test_kvcache_chunk_bitwise_equals_expanded(H, H_kv, D, dtype):
    ops = _ops()
    G = H // H_kv
    g = torch.Generator(device="cuda").manual_seed(H * 31 + H_kv * 7 + D)
    B, T, C = 3, 70, 300
    lens = torch.tensor([0, 57, 230], dtype=torch.int32, device="cuda")
    q = _x(g, dtype, B, T, H, D)
    kc, vc = _x(g, dtype, B, C, H_kv, D), _x(g, dtype, B, C, H_kv, D)
    kn, vn = _x(g, dtype, B, T, H_kv, D), _x(g, dtype, B, T, H_kv, D)
    bias = _x(g, dtype, 1, H, T, C)
    kce, vce = _expand(kc, G), _expand(vc, G)
    kc0, vc0 = kc.double(), vc.double()
    got = ops.attention_with_kv_cache(q, kc, vc, lens, 230, k_new=kn, v_new=vn, bias=bias)
    want = ops.attention_with_kv_cache(q, kce, vce, lens, 230, k_new=_expand(kn, G), v_new=_expand(vn, G), bias=bias)
    _eq(got, want, "chunk output")
    _eq(_expand(kc, G), kce, "appended keys")
    _eq(_expand(vc, G), vce, "appended values")
    ref = ops.attention_with_kv_cache_reference(q.double(), kc0, vc0, lens, 230, kn.double(), vn.double(),
                                                bias=bias.double())
    assert _rel(got, ref) < STEP_TOL[dtype]
    # without seqlens: every query sees all C rows (cross-attention)
    _eq(ops.attention_with_kv_cache(q, kc, vc), ops.attention_with_kv_cache(q, _expand(kc, G), _expand(vc, G)),
        "cross-attention chunk")


# ---- backward ---------------------------------------------------------------------------------------------------
def _bwd(nat, q, k, v, bias, kpm, p, causal, dout, seed):
    scale = q.shape[-1] ** -0.5
    torch.cuda.manual_seed(seed)
    out, lse, bits = nat.fmha_fwd(q, k, v, bias, kpm, p, scale, causal=causal)
    return nat.fmha_bwd(dout, q, k, v, out, lse, bias, kpm, p, scale, bits, bias is not None, False, causal=causal)


def _group_sum(t, G):
    B, L, H, D = t.shape
    return t.double().view(B, L, H // G, G, D).sum(3)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("H,H_kv", HEADS, ids=HEAD_IDS)
@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
def test_backward_deterministic_bitwise_dq_dbias(H, H_kv, D, dtype, causal):
    ops = _ops()
    nat = ops.native()
    G = H // H_kv
    q, k, v, bias, kpm = _case(H, H_kv, D, dtype, 5 + D + H_kv, Lq=136, Lk=136 if causal else 200)
    dout = _x(torch.Generator(device="cuda").manual_seed(1), dtype, *q.shape)
    nat.fmha_det_timeouts()
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        for b in (bias, bias[:1].contiguous()):
            gqa = _bwd(nat, q, k, v, b, kpm, P_DROP, causal, dout, 3)
            again = _bwd(nat, q, k, v, b, kpm, P_DROP, causal, dout, 3)
            exp = _bwd(nat, q, _expand(k, G), _expand(v, G), b, kpm, P_DROP, causal, dout, 3)
            _eq(gqa[0], exp[0], "dQ")
            _eq(gqa[3], exp[3], "dBias")
            for x, y, name in zip(gqa, again, ("dQ", "dK", "dV", "dBias")):
                _eq(x, y, "repeated deterministic backward: " + name)
            assert gqa[1].shape == k.shape and gqa[2].shape == v.shape
            for x, y, name in ((gqa[1], exp[1], "dK"), (gqa[2], exp[2], "dV")):   # the group sums of the expanded call
                assert _rel(x, _group_sum(y, G)) < 2 * UNIT[dtype] * G ** 0.5 + 4 * UNIT[dtype], name
    finally:
        torch.use_deterministic_algorithms(prev)
    assert nat.fmha_det_timeouts() == 0


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("H,H_kv", [(12, 4), (8, 1)], ids=["12x4", "8x1"])
def test_backward_default_mode_within_reorder_bound(H, H_kv, dtype):
    nat = _ops().native()
    G = H // H_kv
    q, k, v, bias, kpm = _case(H, H_kv, 64, dtype, 77)
    dout = _x(torch.Generator(device="cuda").manual_seed(2), dtype, *q.shape)
    gqa = _bwd(nat, q, k, v, bias[:1].contiguous(), kpm, P_DROP, False, dout, 4)
    exp = _bwd(nat, q, _expand(k, G), _expand(v, G), bias[:1].contiguous(), kpm, P_DROP, False, dout, 4)
    for x, y, name in ((gqa[0], exp[0], "dQ"), (gqa[3], exp[3], "dBias")):
        # the key tiles add their fp32 dQ shares in completion order: one 16-bit rounding apart at most
        err = (x.float() - y.float()).abs()
        assert bool((err <= 2 * UNIT[dtype] * y.float().abs() + 1e-3 * y.float().abs().max()).all()), name


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("D", [64, 96])
@pytest.mark.parametrize("causal", [False, True], ids=["full", "causal"])
def test_backward_dk_dv_against_fp64_group_sums(D, dtype, causal):
    ops = _ops()
    H, H_kv = 12, 4
    q, k, v, bias, kpm = _case(H, H_kv, D, dtype, 300 + D, Lq=136, Lk=136)
    dout = _x(torch.Generator(device="cuda").manual_seed(3), dtype, *q.shape)
    leaves = [t.detach().requires_grad_() for t in (q, k, v, bias)]
    out = ops.fused_attention(*leaves[:3], bias=leaves[3], key_padding_mask=kpm, dropout_p=0.0, causal=causal)
    got = torch.autograd.grad(out, leaves, dout)
    ref_leaves = [t.detach().double().requires_grad_() for t in (q, k, v, bias)]
    ref = ops.attention_reference(*ref_leaves[:3], bias=ref_leaves[3], key_padding_mask=kpm, dropout_p=0.0,
                                  causal=causal)
    want = torch.autograd.grad(ref, ref_leaves, dout.double())   # repeat_interleave's backward sums each group
    for x, y, name in zip(got, want, ("dQ", "dK", "dV", "dBias")):
        assert x.shape == y.shape, name
        assert _rel(x, y) < GRAD_TOL[dtype], (name, _rel(x, y))


def test_causal_key_tiles_past_the_queries_give_zero_dk_dv():
    nat = _ops().native()
    dtype, H, H_kv, D = torch.float16, 8, 2, 64
    q, k, v, bias, kpm = _case(H, H_kv, D, dtype, 11, Lq=64, Lk=200)
    dout = _x(torch.Generator(device="cuda").manual_seed(4), dtype, *q.shape)
    dq, dk, dv, dbias = _bwd(nat, q, k, v, bias, None, 0.0, True, dout, 5)
    assert torch.equal(dk[:, 64:], torch.zeros_like(dk[:, 64:])) and torch.equal(dv[:, 64:], torch.zeros_like(dv[:, 64:]))
    assert bool(dk[:, :64].abs().sum() > 0) and bool(dv[:, :64].abs().sum() > 0)
    fut = torch.ones(64, 200, dtype=torch.bool, device="cuda").triu(1)
    assert bool((dbias[:, :, fut] == 0).all())


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_packed_path_writes_one_gradient_tensor(dtype):
    ops = _ops()
    H, H_kv, D, B, L = 8, 2, 64, 2, 128
    g = torch.Generator(device="cuda").manual_seed(12)
    qkv = _x(g, dtype, B, L, H + 2 * H_kv, D).requires_grad_()
    dout = _x(g, dtype, B, L, H, D)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        out = ops.fused_attention_qkvpacked(qkv, dropout_p=0.0, causal=True, num_kv_heads=H_kv)
        out.backward(dout)
        split = qkv.detach().clone().requires_grad_()
        q, k, v = split[:, :, :H], split[:, :, H:H + H_kv], split[:, :, H + H_kv:]
        out2 = ops.fused_attention(q, k, v, dropout_p=0.0, causal=True)
        out2.backward(dout)
    finally:
        torch.use_deterministic_algorithms(prev)
    _eq(out, out2, "packed output")
    assert qkv.grad.shape == (B, L, H + 2 * H_kv, D)
    # equal values (the slice gradients of the split arm reach split.grad through autograd's adds, which turn -0 into 0)
    assert torch.equal(qkv.grad, split.grad), "packed gradient"
    # the module: in_proj of (H + 2 H_kv) * D rows, its gradient through the packed kernel
    from unicore.modules import SelfMultiheadAttention

    torch.manual_seed(0)
    m = SelfMultiheadAttention(H * D, H, dropout=0.0, num_kv_heads=H_kv).cuda().to(dtype)
    x = _x(g, dtype, B, L, H * D).requires_grad_()
    y = m(x)
    y.float().square().sum().backward()
    assert m.in_proj.weight.grad.shape == ((H + 2 * H_kv) * D, H * D) and bool(torch.isfinite(x.grad).all())


# ---- decode ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("H,H_kv", HEADS, ids=HEAD_IDS)
@pytest.mark.parametrize("splits", ["one", "several", "by_length"])
def test_decode_step_appends_once_and_matches_reference(H, H_kv, D, dtype, splits):
    ops = _ops()
    nat = ops.native()
    G = H // H_kv
    g = torch.Generator(device="cuda").manual_seed(H + H_kv + D)
    B, C = 4, 1100
    lens = torch.tensor([0, 5, 700, 1099], dtype=torch.int32, device="cuda")
    q = _x(g, dtype, B, 1, H, D)
    kc, vc = _x(g, dtype, B, C, H_kv, D), _x(g, dtype, B, C, H_kv, D)
    kn, vn = _x(g, dtype, B, 1, H_kv, D), _x(g, dtype, B, 1, H_kv, D)
    bias = _x(g, dtype, B, H, 1, C)
    kc0, vc0 = kc.clone(), vc.clone()
    kce, vce = _expand(kc, G), _expand(vc, G)
    n = {"one": 1, "several": 5, "by_length": 5}[splits]
    by_len = splits == "by_length"
    got = nat.fmha_decode(q, kc, vc, lens, C - 1, kn, vn, bias, None, D ** -0.5, n, by_len)
    want = nat.fmha_decode(q, kce, vce, lens, C - 1, _expand(kn, G), _expand(vn, G), bias, None, D ** -0.5, n, by_len)
    _eq(got, want, "decode output")
    for b, p in enumerate(lens.tolist()):   # the new row, bitwise, and nothing else
        kc0[b, p], vc0[b, p] = kn[b, 0], vn[b, 0]
    _eq(kc, kc0, "key cache after the append")
    _eq(vc, vc0, "value cache after the append")
    ref = ops.attention_with_kv_cache_reference(q.double(), kc.double(), vc.double(), lens + 1, C, bias=bias.double())
    assert _rel(got, ref) < STEP_TOL[dtype]


def test_decode_group_ctas_store_the_new_row_once():
    """Every query head of a group reads the new row from k_new / v_new: a cache row that held NaN before the append
    cannot reach any of them, whichever CTA stores it."""
    ops = _ops()
    H, H_kv, D, B, C = 16, 2, 128, 2, 600
    g = torch.Generator(device="cuda").manual_seed(21)
    q = _x(g, torch.float16, B, 1, H, D)
    kc, vc = _x(g, torch.float16, B, C, H_kv, D), _x(g, torch.float16, B, C, H_kv, D)
    kn, vn = _x(g, torch.float16, B, 1, H_kv, D), _x(g, torch.float16, B, 1, H_kv, D)
    lens = torch.tensor([100, 599], dtype=torch.int32, device="cuda")
    for b, p in enumerate(lens.tolist()):
        kc[b, p] = float("nan")
        vc[b, p] = float("nan")
    with torch.no_grad():
        out = ops.attention_with_kv_cache(q, kc, vc, lens, C - 1, k_new=kn, v_new=vn)
    assert bool(torch.isfinite(out).all())
    for b, p in enumerate(lens.tolist()):
        _eq(kc[b, p], kn[b, 0], "key row")
        _eq(vc[b, p], vn[b, 0], "value row")


# ---- a GQA decoder ------------------------------------------------------------------------------------------------
E, N_HEADS, N_KV = 256, 4, 2


def _decoder(dtype, seed=0):
    from unicore.modules import TransformerDecoder

    torch.manual_seed(seed)
    m = TransformerDecoder(decoder_layers=2, embed_dim=E, ffn_embed_dim=2 * E, attention_heads=N_HEADS,
                           max_seq_len=128, attention_kv_heads=N_KV).cuda().eval()
    with torch.no_grad():
        for p in m.parameters():
            p.add_(torch.randn_like(p) * 0.02)
    return m.to(dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_gqa_decoder_steps_match_full_forward(dtype):
    _ops()
    m = _decoder(dtype)
    g = torch.Generator(device="cuda").manual_seed(5)
    B, L = 3, 9
    tokens, enc = _x(g, dtype, B, L + 16, E), _x(g, dtype, B, 10, E)
    with torch.no_grad():
        cache = m.new_cache(B, 64)
        assert cache.layers[0].k.shape == (B, 64, N_KV, E // N_HEADS)
        m(tokens[:, :L], encoder_out=enc, cache=cache)
        pos = L
        for T in (1, 1, 4, 1, 7):
            y = m(tokens[:, pos:pos + T], cache=cache)
            pos += T
            full = m(tokens[:, :pos], encoder_out=enc)
            assert _rel(y, full[:, -T:]) < STEP_TOL[dtype], (T, pos)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_gqa_captured_steps_equal_eager_steps(dtype):
    import copy

    _ops()
    m = _decoder(dtype)
    g = torch.Generator(device="cuda").manual_seed(6)
    B, L = 3, 12
    prompt, enc = _x(g, dtype, B, L, E), _x(g, dtype, B, 10, E)
    toks = _x(g, dtype, 10, B, 1, E)
    cache = m.new_cache(B, 64)   # one split at this size, captured or not: the same arithmetic
    with torch.no_grad():
        m(prompt, encoder_out=enc, cache=cache)
    eager = copy.deepcopy(cache)
    step = m.capture_step(cache)
    with torch.no_grad():
        for t in range(10):
            want = m(toks[t], cache=eager)
            got = step(toks[t]).clone()
            _eq(got, want, "step {}".format(t))
    assert step.captures == 1
    for a, b in zip(cache.layers, eager.layers):
        _eq(a.k, b.k, "keys")
        _eq(a.v, b.v, "values")
