"""Packed cross-attention: separate key sequences (cu_seqlens_k) in the varlen mode of the wgmma forward and backward,
the op layer, CrossMultiheadAttention and the packed TransformerDecoder.

The varlen call with cu_seqlens_k must equal the padded kernel call on q scattered to ``[B, Lq]`` and k / v to
``[B, Lk]`` with ``key_padding_mask = (j >= n_k)`` and the same Philox seed: O, LSE and the keep bits bitwise at every
real row (and real key), dK / dV bitwise when dO is zero at the pad rows, and dQ / dBias too in deterministic mode.  A
sequence without keys gives O = 0, LSE = -inf and dQ = 0.  The self-attention call is unchanged when it passes its own
description as cu_seqlens_k, malformed key descriptions are clamped, and a packed encoder-decoder forward + backward
does not synchronise."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]
DT_IDS = ["fp16", "bf16"]
GRAD_TOL = {torch.float16: 1e-2, torch.bfloat16: 5e-2}   # relative norm error against fp64
HEAD_DIMS = [8, 64, 96, 128]
UNIT = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
P_DROP = 0.2
# (query lengths, Lq, key lengths, Lk): n_q = 0, n_k = 0 < n_q, 1, lengths that are not multiples of 8 or 64, and
# each max itself; Lq < Lk and Lq > Lk
CASES = {
    "lq_lt_lk": ([77, 0, 5, 120, 64, 13, 40], 120, [250, 31, 0, 129, 1, 256, 64], 256),
    "lq_gt_lk": ([200, 3, 17, 1, 129, 0, 64], 200, [13, 64, 0, 104, 72, 9, 1], 104),
}
# (H, H_kv, bias: None / "shared" / "batch", dropout)
MODES = {
    "plain": (12, 12, None, False),
    "shared_bias_dropout": (12, 12, "shared", True),
    "batch_bias": (12, 12, "batch", False),
    "gqa4_batch_bias_dropout": (12, 4, "batch", True),
    "mqa_dropout": (12, 1, None, True),
}


def _ops():
    from unicore import ops

    assert ops.USE_NATIVE, "native kernels must be active on the GPU box"
    return ops


def _vl():
    return _ops().native().varlen


def _eq(a, b, what):
    assert a.shape == b.shape and torch.equal(a, b), what


def _rel(got, want):
    return ((got.double() - want.double()).norm() / want.double().norm().clamp(min=1e-30)).item()


def _cu(lens):
    return torch.tensor([0] + lens, device="cuda").cumsum(0).to(torch.int32)


def _scatter(x, lens, L):
    """packed [N, ...] -> padded [B, L, ...] with zeros at the pad rows"""
    out = x.new_zeros(len(lens), L, *x.shape[1:])
    s = 0
    for b, n in enumerate(lens):
        out[b, :n] = x[s:s + n]
        s += n
    return out


def _gather(xp, lens):
    return torch.cat([xp[b, :n] for b, n in enumerate(lens)])


def _kpm(lens, L):
    return torch.arange(L, device="cuda")[None, :] >= torch.tensor(lens, device="cuda")[:, None]


def _case(case, mode, D, dtype, seed=0):
    lq, Lq, lk, Lk = CASES[case]
    H, H_kv, bias_kind, drop = MODES[mode]
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = torch.randn(sum(lq), H, D, device="cuda", generator=g).to(dtype)
    # k / v as head slices of one [N_k, 2 H_kv, D] projection, as the modules' separate k_proj / v_proj are not
    kv = torch.randn(sum(lk), 2 * H_kv, D, device="cuda", generator=g).to(dtype)
    bias = None
    if bias_kind is not None:
        bias = torch.randn(1 if bias_kind == "shared" else len(lq), H, Lq, Lk, device="cuda", generator=g).to(dtype)
    return q, kv[:, :H_kv], kv[:, H_kv:], bias, (P_DROP if drop else 0.0)


def _fwd_both(case, q, k, v, bias, p, scale):
    lq, Lq, lk, Lk = CASES[case]
    torch.cuda.manual_seed(11)
    out, lse, bits = _vl().fmha_varlen_fwd(q, k, v, _cu(lq), Lq, bias, p, scale, cu_seqlens_k=_cu(lk), max_seqlen_k=Lk)
    qp, kp, vp = _scatter(q, lq, Lq), _scatter(k, lk, Lk), _scatter(v, lk, Lk)
    torch.cuda.manual_seed(11)
    outp, lsep, bitsp = _ops().native().fmha_fwd(qp, kp, vp, bias, _kpm(lk, Lk), p, scale)
    return (out, lse, bits), (qp, kp, vp, outp, lsep, bitsp)


# the bits of the first m keys of a word (key 2i in bit i, key 2i + 1 in bit 16 + i), as int32
_FIRST = [sum(1 << (16 * (j & 1) + (j >> 1)) for j in range(m)) for m in range(33)]


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("D", HEAD_DIMS)
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_forward_is_bitwise_the_padded_call(dtype, D, mode, case):
    lq, Lq, lk, Lk = CASES[case]
    q, k, v, bias, p = _case(case, mode, D, dtype)
    (out, lse, bits), (_, _, _, outp, lsep, bitsp) = _fwd_both(case, q, k, v, bias, p, D ** -0.5)
    _eq(out, _gather(outp, lq), "O")
    first = torch.tensor([x - (1 << 32) if x >= 1 << 31 else x for x in _FIRST], dtype=torch.int32, device="cuda")
    s = 0
    for b, (nq, nk) in enumerate(zip(lq, lk)):
        _eq(lse[b, :, :nq], lsep[b, :, :nq], ("LSE", b))
        if nk == 0 and nq > 0:   # no keys: the fully-masked contract
            assert torch.count_nonzero(out[s:s + nq]) == 0
            assert bool((lse[b, :, :nq] == float("-inf")).all())
        if p > 0 and nq > 0 and nk > 0:   # the words of the keys every row sees (j < n_k)
            w = (nk + 31) // 32
            m = (nk - 32 * torch.arange(w, device="cuda")).clamp(0, 32)
            keep = first[m][None, None, :]
            _eq(bits[b, :, :nq, :w] & keep, bitsp[b, :, :nq, :w] & keep, ("keep bits", b))
        s += nq


def _bwd_both(case, mode, D, dtype, det):
    lq, Lq, lk, Lk = CASES[case]
    q, k, v, bias, p = _case(case, mode, D, dtype, seed=1)
    scale = D ** -0.5
    (out, lse, bits), (qp, kp, vp, outp, lsep, bitsp) = _fwd_both(case, q, k, v, bias, p, scale)
    dout = torch.randn_like(out)
    doutp = _scatter(dout, lq, Lq)
    need = bias is not None
    with torch.no_grad():
        torch.use_deterministic_algorithms(det)
        try:
            args = (dout, q, k, v, out, lse, _cu(lq), Lq, bias, p, scale, bits, need, False)
            kw = dict(cu_seqlens_k=_cu(lk), max_seqlen_k=Lk)
            got = _vl().fmha_varlen_bwd(*args, **kw)
            again = _vl().fmha_varlen_bwd(*args, **kw)
            want = _ops().native().fmha_bwd(doutp, qp, kp, vp, outp, lsep, bias, _kpm(lk, Lk), p, scale, bitsp, need,
                                            False, None)
        finally:
            torch.use_deterministic_algorithms(False)
    return got, again, want


def _check_empty_source_dq(case, dq):
    lq, _, lk, _ = CASES[case]
    s = 0
    for nq, nk in zip(lq, lk):
        if nk == 0:
            assert torch.count_nonzero(dq[s:s + nq]) == 0, "dQ of a sequence without keys"
        s += nq


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("mode", ["shared_bias_dropout", "batch_bias", "gqa4_batch_bias_dropout", "mqa_dropout"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_backward_is_bitwise_the_padded_call(dtype, D, mode, case):
    lq, _, lk, _ = CASES[case]
    got, _, want = _bwd_both(case, mode, D, dtype, det=False)
    _eq(got[1], _gather(want[1], lk), "dK")
    _eq(got[2], _gather(want[2], lk), "dV")
    _check_empty_source_dq(case, got[0])
    # default mode: the key tiles add their fp32 dQ shares in completion order, one 16-bit rounding apart at most
    pairs = [(got[0], _gather(want[0], lq), "dQ")] + ([(got[3], want[3], "dBias")] if got[3] is not None else [])
    for x, y, name in pairs:
        err = (x.float() - y.float()).abs()
        assert bool((err <= 2 * UNIT[dtype] * y.float().abs() + 1e-3 * y.float().abs().max()).all()), name


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("mode", ["shared_bias_dropout", "batch_bias", "gqa4_batch_bias_dropout"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_deterministic_backward_is_bitwise_the_padded_call_and_repeats(dtype, mode, case):
    lq, _, lk, _ = CASES[case]
    got, again, want = _bwd_both(case, mode, 64, dtype, det=True)
    for x, y, what in zip(got, again, ("dQ", "dK", "dV", "dBias")):
        _eq(x, y, ("repeat", what))
    _eq(got[0], _gather(want[0], lq), "dQ")
    _eq(got[1], _gather(want[1], lk), "dK")
    _eq(got[2], _gather(want[2], lk), "dV")
    _eq(got[3], want[3], "dBias")
    _check_empty_source_dq(case, got[0])
    assert _ops().native().fmha_det_timeouts() == 0


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_gradients_against_fp64_reference(dtype, mode, case):
    ops = _ops()
    lq, Lq, lk, Lk = CASES[case]
    q, k, v, bias, _ = _case(case, mode, 64, dtype, seed=2)
    k, v = k.contiguous(), v.contiguous()
    leaves = [t.requires_grad_(True) for t in (q, k, v) + (() if bias is None else (bias,))]
    kw = dict(cu_seqlens_k=_cu(lk), max_seqlen_k=Lk)
    assert ops.fused_attention_varlen_supported(q, k, v, _cu(lq), Lq, bias, **kw)
    out = ops.fused_attention_varlen(q, k, v, _cu(lq), Lq, bias, **kw)
    dout = torch.randn_like(out)
    out.backward(dout)
    ref_leaves = [t.detach().double().requires_grad_(True) for t in leaves]
    b64 = ref_leaves[3] if bias is not None else None
    ref = ops.attention_varlen_reference(*ref_leaves[:3], _cu(lq), Lq, b64, **kw)
    ref.backward(dout.double())
    assert _rel(out, ref) < GRAD_TOL[dtype]
    for got, want, name in zip(leaves, ref_leaves, ("dq", "dk", "dv", "dbias")):
        assert _rel(got.grad, want.grad) < GRAD_TOL[dtype], name
    _check_empty_source_dq(case, q.grad)


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("kind", ["shared", "batch"])
def test_dbias_is_zero_outside_every_block(kind, case):
    ops = _ops()
    lq, Lq, lk, Lk = CASES[case]
    mode = "shared_bias_dropout" if kind == "shared" else "gqa4_batch_bias_dropout"
    q, k, v, bias, p = _case(case, mode, 64, torch.float16, seed=3)
    bias.requires_grad_(True)
    out = ops.fused_attention_varlen(q, k, v, _cu(lq), Lq, bias, dropout_p=p, cu_seqlens_k=_cu(lk), max_seqlen_k=Lk)
    out.float().square().sum().backward()
    inside = torch.zeros(len(lq), 1, Lq, Lk, dtype=torch.bool, device="cuda")
    for b, (nq, nk) in enumerate(zip(lq, lk)):
        inside[b, :, :nq, :nk] = True
    if kind == "shared":
        inside = inside.any(0, keepdim=True)
    assert not bool(inside.all())
    assert torch.count_nonzero(bias.grad.masked_fill(inside, 0)) == 0
    assert torch.count_nonzero(bias.grad) > 0


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_self_description_is_the_self_call(dtype):
    """cu_seqlens_k = (a copy of) cu_seqlens with max_seqlen_k = max_seqlen is bitwise the call without them, forward
    and deterministic backward; causal self-attention, which reads the same key fields, is bitwise the padded causal
    call, and causal is refused together with cu_seqlens_k."""
    lens, L, H, D = [77, 0, 1, 200, 64, 129, 13], 200, 12, 64
    g = torch.Generator(device="cuda").manual_seed(7)
    q, k, v = (torch.randn(sum(lens), H, D, device="cuda", generator=g).to(dtype) for _ in range(3))
    bias = torch.randn(len(lens), H, L, L, device="cuda", generator=g).to(dtype)
    cu, scale = _cu(lens), D ** -0.5
    dout = torch.randn(sum(lens), H, D, device="cuda", generator=g).to(dtype)
    runs = []
    for kw in ({}, dict(cu_seqlens_k=cu.clone(), max_seqlen_k=L)):
        torch.cuda.manual_seed(3)
        out, lse, bits = _vl().fmha_varlen_fwd(q, k, v, cu, L, bias, P_DROP, scale, **kw)
        torch.use_deterministic_algorithms(True)
        try:
            grads = _vl().fmha_varlen_bwd(dout, q, k, v, out, lse, cu, L, bias, P_DROP, scale, bits, True, False, **kw)
        finally:
            torch.use_deterministic_algorithms(False)
        runs.append((out, lse, bits, grads))
    (out0, lse0, bits0, g0), (out1, lse1, bits1, g1) = runs
    _eq(out0, out1, "O")
    for x, y, what in zip(g0, g1, ("dQ", "dK", "dV", "dBias")):
        _eq(x, y, what)
    for b, n in enumerate(lens):   # the rows and keep words each sequence writes
        _eq(lse0[b, :, :n], lse1[b, :, :n], ("LSE", b))
        _eq(bits0[b, :, :n, :(n + 31) // 32], bits1[b, :, :n, :(n + 31) // 32], ("keep bits", b))
    assert _ops().native().fmha_det_timeouts() == 0
    # causal: the kernels read the key fields the binding set from cu_seqlens
    qp, kp, vp = (_scatter(t, lens, L) for t in (q, k, v))
    out, _, _ = _vl().fmha_varlen_fwd(q, k, v, cu, L, bias, 0.0, scale, causal=True)
    outp, _, _ = _ops().native().fmha_fwd(qp, kp, vp, bias, _kpm(lens, L), 0.0, scale, causal=True)
    _eq(out, _gather(outp, lens), "causal O")
    with pytest.raises(RuntimeError):
        _vl().fmha_varlen_fwd(q, k, v, cu, L, bias, 0.0, scale, causal=True, cu_seqlens_k=cu, max_seqlen_k=L)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_out_of_range_cu_seqlens_k_are_clamped(dtype):
    """Decreasing entries, entries past N_k, negative entries and lengths above max_seqlen_k: the kernels clamp every key
    sequence to s_k = clamp(cu_k[b], 0, N_k), n_k = clamp(cu_k[b + 1] - cu_k[b], 0, min(Lk, N_k - s_k)), stay inside
    the tensors and give the result of the reference, which applies the same clamps."""
    from unicore_b200.ops.attention_ops import _varlen_index

    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(4)
    lq, Lq = [10, 20, 30, 5, 8], 32
    Nq, Nk, H, D, Lk = sum(lq), 150, 4, 64, 64
    q = torch.randn(Nq, H, D, device="cuda", generator=g).to(dtype)
    k, v = (torch.randn(Nk, H, D, device="cuda", generator=g).to(dtype) for _ in range(2))
    # key sequences: rows 0 .. 34 (a negative start clamped to 0), none (decreasing), rows 20 .. 39, rows 40 .. 103
    # (140 rows clamped to Lk) and none (a start past N_k)
    cu_k = torch.tensor([-5, 30, 20, 40, 180, 1000], dtype=torch.int32, device="cuda")
    bias = torch.randn(len(lq), H, Lq, Lk, device="cuda", generator=g).to(dtype)
    rows, valid = _varlen_index(cu_k, Lk, Nk)
    covered = torch.zeros(Nk, dtype=torch.bool, device="cuda")
    covered[rows[valid]] = True
    assert not bool(covered.all())
    # canary: NaN in the key rows no sequence covers; the kernels must hide them by assignment and zero their V rows
    kn, vn = (t.masked_fill(~covered[:, None, None], float("nan")) for t in (k, v))
    kw = dict(cu_seqlens_k=cu_k, max_seqlen_k=Lk)
    out, lse, _ = _vl().fmha_varlen_fwd(q, kn, vn, _cu(lq), Lq, bias, 0.0, D ** -0.5, **kw)
    assert bool(torch.isfinite(out).all())
    ref = ops.attention_varlen_reference(q.double(), k.double(), v.double(), _cu(lq), Lq, bias.double(),
                                         scale=D ** -0.5, **kw)
    assert _rel(out, ref) < GRAD_TOL[dtype]
    dq, dk, dv, db = _vl().fmha_varlen_bwd(torch.ones_like(out), q, k, v, out, lse, _cu(lq), Lq, bias, 0.0,
                                           D ** -0.5, None, True, False, **kw)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(db).all()) and bool(torch.isfinite(dq).all())
    assert bool(torch.isfinite(dk[covered]).all()) and bool(torch.isfinite(dv[covered]).all())


def _valid():
    dt = torch.float16
    q = torch.randn(24, 2, 64, device="cuda", dtype=dt)
    k, v = (torch.randn(40, 2, 64, device="cuda", dtype=dt) for _ in range(2))
    cu = torch.tensor([0, 10, 24], dtype=torch.int32, device="cuda")
    cu_k = torch.tensor([0, 30, 40], dtype=torch.int32, device="cuda")
    bias = torch.randn(2, 2, 16, 40, device="cuda", dtype=dt)
    return [q, k, v, cu, 16, bias, 0.0, 0.125, False, cu_k, 40]


BAD = {
    "k / v rows differ": (2, lambda a: a[2][:32]),
    "cu_seqlens_k int64": (9, lambda a: a[9].long()),
    "cu_seqlens_k on the cpu": (9, lambda a: a[9].cpu()),
    "cu_seqlens_k another B": (9, lambda a: torch.tensor([0, 10, 20, 40], dtype=torch.int32, device="cuda")),
    "cu_seqlens_k strided": (9, lambda a: torch.zeros(6, dtype=torch.int32, device="cuda")[::2]),
    "max_seqlen_k not a multiple of 8": (10, lambda a: 12),
    "max_seqlen_k negative": (10, lambda a: -8),
    "bias columns": (5, lambda a: a[5][..., :32].contiguous()),
    "causal with cu_seqlens_k": (8, lambda a: True),
    "N_k != N_q without cu_seqlens_k": (9, lambda a: None),
}


def test_binding_rejects_bad_operands():
    _vl().fmha_varlen_fwd(*_valid())   # the builder is valid
    torch.cuda.synchronize()
    for label, (i, bad) in BAD.items():
        args = _valid()
        args[i] = bad(args)
        with pytest.raises(RuntimeError):
            _vl().fmha_varlen_fwd(*args)
        print("rejected:", label)
    q, k, v, cu, Lm, bias, p, scale, _, cu_k, Lk = _valid()
    with pytest.raises(RuntimeError):   # a key bound other than the queries' own without key sequences
        _vl().fmha_varlen_fwd(q, q, q, cu, Lm, None, 0.0, scale, max_seqlen_k=24)
    out, lse, bits = _vl().fmha_varlen_fwd(q, k, v, cu, Lm, bias, 0.1, scale, cu_seqlens_k=cu_k, max_seqlen_k=Lk)
    good = [out, q, k, v, out, lse, cu, Lm, bias, 0.1, scale, bits, True, False, False, cu_k, Lk]
    _vl().fmha_varlen_bwd(*good)
    bad_bwd = {
        "packed gradients with cu_seqlens_k": (13, True),
        "keep bits at max_seqlen": (11, torch.zeros(2, 2, 16, 1, dtype=torch.int32, device="cuda")),
        "cu_seqlens_k another B": (15, torch.tensor([0, 40], dtype=torch.int32, device="cuda")),
        "max_seqlen_k": (16, 24),
    }
    for label, (i, bad) in bad_bwd.items():
        args = list(good)
        args[i] = bad
        with pytest.raises(RuntimeError):
            _vl().fmha_varlen_bwd(*args)
        print("rejected:", label)
    torch.cuda.synchronize()


# ---- the modules -------------------------------------------------------------------------------------------------
class C:
    """the tolerances of tests/test_gpu_encoder_path.py (relative norm error against float64)"""
    OUT = {torch.float16: 1e-2, torch.bfloat16: 5e-2}
    GRAD = {torch.float16: 2e-2, torch.bfloat16: 8e-2}


DEC_LQ, DEC_LQ_MAX = [77, 0, 1, 200, 64, 129, 13], 200
DEC_LK, DEC_LK_MAX = [150, 33, 0, 256, 1, 64, 90], 256


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_cross_attention_module_against_fp64_and_the_padded_call(dtype):
    import copy

    from unicore.modules import CrossMultiheadAttention

    ops = _ops()
    torch.manual_seed(8)
    attn = CrossMultiheadAttention(256, 4, dropout=0.0, num_kv_heads=2).cuda().to(dtype)
    ref = copy.deepcopy(attn).double()
    g = torch.Generator(device="cuda").manual_seed(9)
    x = torch.randn(sum(DEC_LQ), 256, device="cuda", generator=g).to(dtype).requires_grad_(True)
    e = torch.randn(sum(DEC_LK), 256, device="cuda", generator=g).to(dtype).requires_grad_(True)
    bias = torch.randn(4, DEC_LQ_MAX, DEC_LK_MAX, device="cuda", generator=g).to(dtype)
    kw = dict(cu_seqlens=_cu(DEC_LQ), max_seqlen=DEC_LQ_MAX, encoder_cu_seqlens=_cu(DEC_LK),
              encoder_max_seqlen=DEC_LK_MAX)
    qh = torch.empty(sum(DEC_LQ), 4, 64, device="cuda", dtype=dtype)
    kh = torch.empty(sum(DEC_LK), 2, 64, device="cuda", dtype=dtype)
    assert ops.fused_attention_varlen_supported(qh, kh, kh, _cu(DEC_LQ), DEC_LQ_MAX, bias[None], _cu(DEC_LK),
                                                DEC_LK_MAX)
    y = attn(x, e, e, attn_bias=bias, **kw)
    dy = torch.randn_like(y)
    y.backward(dy)
    x64, e64 = (t.detach().double().requires_grad_(True) for t in (x, e))
    y64 = ref(x64, e64, e64, attn_bias=bias.double(), **kw)
    y64.backward(dy.double())
    assert _rel(y, y64) < C.OUT[dtype]
    assert _rel(x.grad, x64.grad) < C.GRAD[dtype]
    assert _rel(e.grad, e64.grad) < C.GRAD[dtype]
    # the weights (the key projection's bias has a zero gradient: it shifts every score of a query row alike)
    for (name, p), (_, q) in zip(attn.named_parameters(), ref.named_parameters()):
        if p.dim() == 2:
            assert _rel(p.grad, q.grad) < C.GRAD[dtype], name
    ep = _scatter(e.detach(), DEC_LK, DEC_LK_MAX)
    with torch.no_grad():
        yp = attn(_scatter(x.detach(), DEC_LQ, DEC_LQ_MAX), ep, ep, key_padding_mask=_kpm(DEC_LK, DEC_LK_MAX),
                  attn_bias=bias)
    assert _rel(y.detach(), _gather(yp, DEC_LQ)) < C.OUT[dtype]


def _decoder(dtype, rotary, post_ln=False):
    from unicore.modules import TransformerDecoder

    torch.manual_seed(5)
    dec = TransformerDecoder(decoder_layers=2, embed_dim=256, ffn_embed_dim=512, attention_heads=4, emb_dropout=0.0,
                             dropout=0.0, attention_dropout=0.0, max_seq_len=DEC_LK_MAX, rel_pos=not rotary,
                             post_ln=post_ln, attention_kv_heads=2, rotary_dim=32 if rotary else None)
    return dec.cuda().to(dtype)


@pytest.mark.parametrize("encoder", [False, True], ids=["decoder_only", "encoder_decoder"])
@pytest.mark.parametrize("rotary", [False, True], ids=["relpos", "rotary"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_packed_decoder_against_fp64_and_the_padded_stack(dtype, rotary, encoder):
    import copy

    dec = _decoder(dtype, rotary, post_ln=encoder)
    ref = copy.deepcopy(dec).double()
    g = torch.Generator(device="cuda").manual_seed(6)
    emb = torch.randn(sum(DEC_LQ), 256, device="cuda", generator=g).to(dtype).requires_grad_(True)
    enc = None
    kw = dict(cu_seqlens=_cu(DEC_LQ), max_seqlen=DEC_LQ_MAX)
    if encoder:
        enc = torch.randn(sum(DEC_LK), 256, device="cuda", generator=g).to(dtype).requires_grad_(True)
        kw.update(encoder_cu_seqlens=_cu(DEC_LK), encoder_max_seqlen=DEC_LK_MAX)
    y = dec(emb, encoder_out=enc, **kw)
    dy = torch.randn_like(y)
    y.backward(dy)
    e64 = emb.detach().double().requires_grad_(True)
    enc64 = None if enc is None else enc.detach().double().requires_grad_(True)
    y64 = ref(e64, encoder_out=enc64, **kw)
    y64.backward(dy.double())
    assert _rel(y, y64) < C.OUT[dtype]
    assert _rel(emb.grad, e64.grad) < C.GRAD[dtype]
    if encoder:
        assert _rel(enc.grad, enc64.grad) < C.GRAD[dtype]
    for (name, p), (_, q) in zip(dec.named_parameters(), ref.named_parameters()):
        if p.dim() == 2 and p.grad is not None:
            assert _rel(p.grad, q.grad) < C.GRAD[dtype], name
    # the padded stack on the same sentences, at the real rows
    with torch.no_grad():
        encp = None if enc is None else _scatter(enc.detach(), DEC_LK, DEC_LK_MAX)
        yp = dec(_scatter(emb.detach(), DEC_LQ, DEC_LQ_MAX), encoder_out=encp,
                 padding_mask=_kpm(DEC_LQ, DEC_LQ_MAX),
                 encoder_padding_mask=None if enc is None else _kpm(DEC_LK, DEC_LK_MAX))
    assert _rel(y.detach(), _gather(yp, DEC_LQ)) < C.OUT[dtype]


def test_packed_encoder_decoder_does_not_synchronise():
    dec = _decoder(torch.float16, rotary=True)
    emb = torch.randn(sum(DEC_LQ), 256, device="cuda", dtype=torch.float16, requires_grad=True)
    enc = torch.randn(sum(DEC_LK), 256, device="cuda", dtype=torch.float16, requires_grad=True)
    kw = dict(cu_seqlens=_cu(DEC_LQ), max_seqlen=DEC_LQ_MAX, encoder_cu_seqlens=_cu(DEC_LK),
              encoder_max_seqlen=DEC_LK_MAX)
    dec(emb, encoder_out=enc, **kw).float().sum().backward()   # warm-up: caches, kernels loaded
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        dec(emb, encoder_out=enc, **kw).float().sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
