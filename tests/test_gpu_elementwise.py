"""bias + GELU, the column sum behind ``ops.linear``, softmax cross entropy and the Gaussian basis against fp64.

Shapes come from the launch plans (``bias_gelu_plan``, ``gbf_plan``, the functions the launchers run), so that every
column-block and row-slice case of ``csrc/fused/elementwise.cu`` and every geometry of ``csrc/fused/gaussian.cu``
runs, with several grid sweeps and a ragged last one.

Error bounds are per element.  The kernels compute in fp32 and round each output once, so a bound is one rounding of
the output type (``UNIT[dtype] * |ref|``) plus the fp32 error of the computation, written as a small multiple of
``E32`` times the magnitudes that enter it.  The approximate instructions get their documented errors: ``rcp.approx``
and ``ex2.approx`` 1 ulp (2 E32) and 2 ulp, ``__expf(x)`` 2 + 1.173 |x| ulp, ``__logf`` 2^-21.41 absolute on
[0.5, 2] and 3 ulp elsewhere.  Everything runs flush-to-zero, so results below 2^-126 may read as 0.
"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

E32 = 2.0 ** -24
UNIT = {torch.float32: 2.0 ** -24, torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}  # unit roundoff
FTZ = 2.0 ** -126
HALF = [torch.float16, torch.bfloat16]
CHUNK = 1 << 21  # elements per fp64 reference chunk


def _native():
    from unicore import ops

    assert ops.USE_NATIVE, "native kernels must be active on the GPU box"
    return ops.native()


def _tiny(dtype):
    return torch.finfo(dtype).tiny * UNIT[dtype]  # half the spacing of the subnormals


def _chunks(rows, cols):
    step = max(1, CHUNK // max(1, cols))
    for r0 in range(0, rows, step):
        yield slice(r0, min(rows, r0 + step))


def _assert_within(got, ref, bound, what):
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)  # NaN fails too
    if bad.any():
        i = bad.nonzero()[0].tolist()
        worst = (err / bound.clamp_min(1e-300)).nan_to_num(math.inf).max().item()
        raise AssertionError("{}: {} elements out of bound, first at {}: got {}, want {} +- {} (worst {:.3g}x)".format(
            what, int(bad.sum()), i, got[tuple(i)].item(), ref[tuple(i)].item(), bound[tuple(i)].item(), worst))


def _nan_blocks(shape, dtype=torch.float32, n=4):
    """Leave `n` freed NaN blocks of `shape` in the caching allocator, so that an output or scratch buffer of that size
    which no kernel writes reads as NaN rather than as zeros by luck."""
    blocks = [torch.full(shape, math.nan, device="cuda", dtype=dtype) for _ in range(n)]
    del blocks


def _check_sum(got, ref, absum, comp_sum, dtype, chain, what, base=None):
    """A sum accumulated in fp32 and rounded once (onto `base` for a sink): the chain of additions behind it times
    the absolute sum, plus the per-term errors `comp_sum` of the fp32 terms."""
    if base is not None:
        ref = ref + base.double()
        absum = absum + base.double().abs()
    comp = chain * E32 * absum + comp_sum
    _assert_within(got, ref, UNIT[dtype] * (ref.abs() + comp) + comp + _tiny(dtype), what)


# ---------------------------------------------------------------------------------------------------
# bias + GELU
# ---------------------------------------------------------------------------------------------------
AS_B = [0.319381530, -0.356563782, 1.781477937, -1.821255978, 1.330274429]  # Abramowitz-Stegun 26.2.17
NVECS = [1, 127, 128, 129, 384]  # one partial / one full / full + partial / three full column blocks
SHORT_ROWS = [1, 7, 8, 9, 16]  # one slice: ragged (1, 7) or whole (8); two slices: ragged (9) or whole (16)


def column_case(plan, rows):
    """(last column block full, several slices, ragged last sweep) of a bias_gelu / column_sum launch."""
    return (plan["nvec"] % 128 == 0, plan["slices"] > 1, rows % plan["rows_per_sweep"] != 0)


def long_rows(nvec):
    """Rows with which every (slice, lane) of the forward and the backward plan loops three times or more and the
    last sweep of both is ragged."""
    nat = _native()
    sweep = nat.bias_gelu_plan(1 << 30, nvec * 8, "fwd")["rows_per_sweep"]
    rows = 3 * sweep + sweep // 2 + 1
    while any(rows % nat.bias_gelu_plan(rows, nvec * 8, k)["rows_per_sweep"] == 0 for k in ("fwd", "bwd")):
        rows += 1
    for k in ("fwd", "bwd"):
        p = nat.bias_gelu_plan(rows, nvec * 8, k)
        assert p["sweeps"] >= 4 and rows % p["rows_per_sweep"] != 0, (k, p)
    return rows


def column_chain(plan):
    """Longest chain of fp32 additions behind one column sum: 4 rows per sweep in a lane, the two lanes, the strided
    and the 32-way sums over the slices, the sink."""
    return 4 * plan["sweeps"] + 2 + -(-plan["slices"] // 32) + 32 + 2


def gelu_parts(x):
    """fp64 terms for GELU at x: exact Phi and pdf, the kernel's formula Phi_AS, and the fp32 error bound of Phi_AS
    as the kernel evaluates it."""
    ax = x.abs()
    pdf = torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)
    phi = 0.5 * torch.erfc(-x / math.sqrt(2.0))
    t = 1.0 / (1.0 + 0.2316419 * ax)
    poly = torch.zeros_like(x)
    absp = torch.zeros_like(x)
    dabsp = torch.zeros_like(x)
    tp = t.clone()
    for i, b in enumerate(AS_B):
        poly += b * tp
        absp += abs(b) * tp
        dabsp += (i + 1) * abs(b) * tp
        tp = tp * t
    q = pdf * poly
    phi_as = torch.where(x < 0, q, 1.0 - q)
    # t: fma + rcp.approx (+ the constant); Horner: 5 fma + 1 mul over partial sums <= absp; pdf: x*x*c feeds ex2
    # (relative error of the argument times |x^2/2|), ex2.approx, one product; q: one product
    rel_poly = (12 * absp + 4 * dabsp) * E32 / poly
    rel_q = rel_poly + (1.5 * x * x + 8) * E32 + 4 * E32
    phi_err = q * rel_q + (x >= 0).double() * 2 * E32  # x >= 0: 0.5 + (0.5 - Q), two roundings
    return phi, pdf, phi_as, phi_err, (1.5 * x * x + 12) * E32


def gelu_fwd_ref(xd, biased):
    """(ref, comp): x Phi(x) and the kernel's error without the output rounding."""
    phi, pdf, phi_as, phi_err, _ = gelu_parts(xd)
    ref = xd * phi
    comp = xd.abs() * ((phi_as - phi).abs() + phi_err) + E32 * (xd * phi_as).abs() + FTZ * (xd.abs() + 1)
    if biased:  # x + bias rounded to fp32 once
        comp += (phi + xd * pdf).abs() * E32 * xd.abs()
    return ref, comp


def gelu_bwd_ref(xd, dyd, biased):
    """(ref, comp): dy (Phi + x pdf) and the kernel's error without the output rounding."""
    phi, pdf, phi_as, phi_err, rel_pdf = gelu_parts(xd)
    inner = phi + xd * pdf
    ic = ((phi_as - phi).abs() + phi_err + xd.abs() * pdf * rel_pdf + E32 * (phi_as.abs() + (xd * pdf).abs())
          + FTZ * (xd.abs() + 2))
    if biased:
        ic += (pdf * (2 - xd * xd)).abs() * E32 * xd.abs()
    ref = dyd * inner
    comp = dyd.abs() * ic + E32 * ref.abs() + FTZ
    return ref, comp


def _gelu_inputs(rows, cols, dtype, seed):
    """x: every value of `dtype` in [-14, 14] (a random subset when the tensor is smaller), then random values."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    allv = torch.arange(-32768, 32768, dtype=torch.int32, device="cuda").to(torch.int16).view(dtype)
    grid = allv[torch.isfinite(allv) & (allv.float().abs() <= 14)]
    grid = grid[torch.randperm(grid.numel(), device="cuda", generator=g)]
    n = rows * cols
    extra = max(0, n - grid.numel())
    x = torch.cat([grid[:n], (torch.randn(extra, device="cuda", generator=g) * 4).to(dtype)]).view(rows, cols)
    dy = torch.randn(rows, cols, device="cuda", generator=g).to(dtype)
    bias = (torch.randn(cols, device="cuda", generator=g) * 0.5).to(dtype)
    return x, dy, bias


def check_bias_gelu(nat, x, dy, bias, mode, dtype):
    rows, cols = x.shape
    u, tiny = UNIT[dtype], _tiny(dtype)
    biased = mode != "none"
    b = bias if biased else None
    y = nat.bias_gelu_fwd(x, b)
    sink_base = None
    if mode == "sink":
        arena = torch.randn(cols + 64, device="cuda").to(dtype)
        before = arena.clone()
        sink = arena[32:32 + cols]
        sink_base = sink.clone()
        dx, db = nat.bias_gelu_bwd(dy, x, b, sink)
        assert db.data_ptr() == sink.data_ptr()
        outside = torch.ones_like(arena, dtype=torch.bool)
        outside[32:32 + cols] = False
        assert torch.equal(arena[outside], before[outside])
    else:
        dx, db = nat.bias_gelu_bwd(dy, x, b)
        assert (db is None) == (not biased)
    bd = bias.double() if biased else 0.0
    db_r = torch.zeros(cols, dtype=torch.float64, device="cuda")
    db_a, db_c = torch.zeros_like(db_r), torch.zeros_like(db_r)
    for s in _chunks(rows, cols):
        xd = x[s].double() + bd
        ref, comp = gelu_fwd_ref(xd, biased)
        _assert_within(y[s], ref, u * (ref.abs() + comp) + comp + tiny, "gelu")
        ref, comp = gelu_bwd_ref(xd, dy[s].double(), biased)
        _assert_within(dx[s], ref, u * (ref.abs() + comp) + comp + tiny, "gelu'")
        db_r += ref.sum(0)
        db_a += ref.abs().sum(0)
        db_c += comp.sum(0)
    if biased:
        chain = column_chain(nat.bias_gelu_plan(rows, cols, "bwd"))
        _check_sum(db, db_r, db_a, db_c, dtype, chain, "dbias", sink_base)


@pytest.mark.parametrize("mode", ["bias", "none", "sink"])
@pytest.mark.parametrize("rows", SHORT_ROWS + ["long"])
@pytest.mark.parametrize("nvec", NVECS)
@pytest.mark.parametrize("dtype", HALF)
def test_bias_gelu_all_paths(dtype, nvec, rows, mode):
    nat = _native()
    cols = nvec * 8
    rows = long_rows(nvec) if rows == "long" else rows
    x, dy, bias = _gelu_inputs(rows, cols, dtype, seed=nvec * 100 + rows % 97)
    check_bias_gelu(nat, x, dy, bias, mode, dtype)


@pytest.mark.parametrize("dtype", HALF)
def test_bias_gelu_op(dtype):
    """The autograd op equals the bindings: forward, dx and the bias gradient."""
    from unicore import ops

    nat = _native()
    rows, cols = 300, 1032
    x, dy, bias = _gelu_inputs(rows, cols, dtype, seed=5)
    xr = x.clone().requires_grad_(True)
    br = bias.clone().requires_grad_(True)
    y = ops.bias_gelu(xr, br)
    y.backward(dy)
    assert torch.equal(y, nat.bias_gelu_fwd(x, bias))
    dx, db = nat.bias_gelu_bwd(dy, x, bias)
    assert torch.equal(xr.grad, dx) and torch.equal(br.grad, db)


@pytest.mark.parametrize("dtype", HALF)
def test_bias_gelu_alignment_guards(dtype):
    """The bindings refuse operands the 16-byte kernels cannot read; the op copies a misaligned view once and gives
    exactly the result of the same values in an aligned buffer."""
    from unicore import ops

    nat = _native()
    rows, cols = 33, 264
    buf = torch.randn(rows * cols + 8, device="cuda").to(dtype)
    xm = buf[1:1 + rows * cols].view(rows, cols)
    assert xm.is_contiguous() and xm.data_ptr() % 16 != 0
    xa = xm.clone()
    bias = torch.randn(cols, device="cuda").to(dtype)
    bm = buf[3:3 + cols]
    dy = torch.randn(rows, cols, device="cuda").to(dtype)
    dym = buf[5:5 + rows * cols].view(rows, cols)
    outs = []
    for t in (xm, xa):
        t = t.detach().requires_grad_(True)
        bb = bias.clone().requires_grad_(True)
        y = ops.bias_gelu(t, bb)
        y.backward(dym)
        outs.append((y, t.grad, bb.grad))
    for u, v in zip(*outs):
        assert torch.equal(u, v)
    for call in (lambda: nat.bias_gelu_fwd(xm, bias), lambda: nat.bias_gelu_fwd(xa, bm),
                 lambda: nat.bias_gelu_bwd(dy, xm, bias), lambda: nat.bias_gelu_bwd(dym, xa, bias),
                 lambda: nat.bias_gelu_bwd(dy, xa, bm)):
        with pytest.raises(RuntimeError, match="16-byte aligned"):
            call()
    with pytest.raises(RuntimeError, match="multiple of 8"):
        nat.bias_gelu_fwd(torch.zeros(4, 12, device="cuda", dtype=dtype), None)
    with pytest.raises(RuntimeError, match="fp16 / bf16"):
        nat.bias_gelu_bwd(dy.float(), xa.float(), None)
    with pytest.raises(RuntimeError, match="dy must match x"):
        nat.bias_gelu_bwd(dy[:-1].contiguous(), xa, bias)


# ---------------------------------------------------------------------------------------------------
# column sum
# ---------------------------------------------------------------------------------------------------
def check_column_sum(got, x, dtype, chain, base=None, extra_rel=0.0):
    rows, cols = x.shape
    ref = torch.zeros(cols, dtype=torch.float64, device="cuda")
    absum = torch.zeros_like(ref)
    for s in _chunks(rows, cols):
        ref += x[s].double().sum(0)
        absum += x[s].double().abs().sum(0)
    _check_sum(got, ref, absum, extra_rel * absum, dtype, chain, "column sum", base)


@pytest.mark.parametrize("rows", SHORT_ROWS + ["long"])
@pytest.mark.parametrize("nvec", NVECS)
@pytest.mark.parametrize("dtype", HALF)
def test_column_sum_all_paths(dtype, nvec, rows):
    nat = _native()
    cols = nvec * 8
    rows = long_rows(nvec) if rows == "long" else rows
    g = torch.Generator(device="cuda").manual_seed(7000 + nvec)
    x = (torch.randn(rows, cols, device="cuda", generator=g) + 0.25).to(dtype)
    chain = column_chain(nat.bias_gelu_plan(rows, cols, "bwd"))
    check_column_sum(nat.column_sum(x), x, dtype, chain)
    arena = torch.randn(cols + 64, device="cuda").to(dtype)
    before = arena.clone()
    sink = arena[24:24 + cols]
    base = sink.clone()
    out = nat.column_sum(x, sink)
    assert out.data_ptr() == sink.data_ptr()
    check_column_sum(out, x, dtype, chain, base)
    outside = torch.ones_like(arena, dtype=torch.bool)
    outside[24:24 + cols] = False
    assert torch.equal(arena[outside], before[outside])


@pytest.mark.parametrize("shape", [(300, 3072), (8192, 8), (4096, 64), (12288, 200), (9, 129 * 8)])
@pytest.mark.parametrize("dtype", HALF)
def test_linear_bias_gradient(dtype, shape):
    """``ops.linear``'s bias gradient: the column kernel directly, or for narrow outputs (< 256 columns, >= 4096
    rows) folded into [rows / f, f * cols], summed by the kernel, rounded, and the f partials summed in fp32."""
    from unicore import ops
    from unicore_b200.ops.fused_ops import _narrow_fold

    nat = _native()
    rows, cols = shape
    g = torch.Generator(device="cuda").manual_seed(rows + cols)
    x = torch.randn(rows, 16, device="cuda", generator=g).to(dtype).requires_grad_(True)
    w = (torch.randn(cols, 16, device="cuda", generator=g) * 0.25).to(dtype).requires_grad_(True)
    b = torch.randn(cols, device="cuda", generator=g).to(dtype).requires_grad_(True)
    dy = (torch.randn(rows, cols, device="cuda", generator=g) + 0.1).to(dtype)
    ops.linear(x, w, b).backward(dy)
    fold = _narrow_fold(dy)
    assert (fold > 1) == (cols < 256 and rows >= 4096)
    plan = nat.bias_gelu_plan(rows // fold, cols * fold, "bwd")
    # folded: the f kernel sums are rounded to the dtype before they are added (UNIT per partial, <= UNIT * absum)
    check_column_sum(b.grad, dy, dtype, column_chain(plan) + fold, extra_rel=UNIT[dtype] if fold > 1 else 0.0)


@pytest.mark.parametrize("dtype", HALF)
def test_column_sums_of_no_rows(dtype):
    """Zero rows (a micro-batch without masked tokens): column_sum and bias_gelu_bwd return zero column sums and leave
    a sink as it was, and ``ops.linear``'s backward gives a zero bias gradient."""
    from unicore import ops

    nat = _native()
    cols = 768
    zeros = torch.zeros(cols, device="cuda", dtype=dtype)
    x = torch.empty(0, cols, device="cuda", dtype=dtype)
    bias = torch.randn(cols, device="cuda").to(dtype)
    _nan_blocks((cols,), dtype)
    assert torch.equal(nat.column_sum(x, None), zeros)
    _nan_blocks((cols,), dtype)
    dx, db = nat.bias_gelu_bwd(x, x, bias, None)
    assert dx.shape == x.shape and torch.equal(db, zeros)
    sink = torch.randn(cols, device="cuda").to(dtype)
    before = sink.clone()
    assert nat.column_sum(x, sink).data_ptr() == sink.data_ptr() and torch.equal(sink, before)
    nat.bias_gelu_bwd(x, x, bias, sink)
    assert torch.equal(sink, before)
    # 768 outputs take the column kernel; the bias is not claimed by a gradient arena
    xr = x.clone().requires_grad_(True)
    w = torch.randn(cols, cols, device="cuda").to(dtype).requires_grad_(True)
    b = bias.clone().requires_grad_(True)
    y = ops.linear(xr, w, b)
    _nan_blocks((cols,), dtype)
    y.backward(torch.empty_like(y))
    assert torch.equal(b.grad, zeros)


def test_column_dispatch_coverage():
    """The shapes above reach every (full / partial last column block) x (one slice / several) x (ragged or whole
    last sweep) case of the bias_gelu forward and backward / column_sum launch plans, and the long shapes loop several
    sweeps; none of this launches a kernel."""
    nat = _native()
    for kind in ("fwd", "bwd"):
        reachable = set()
        for nvec in range(1, 400):
            for rows in (1, 8, 9, 16, 100, 4096, 4097, 1 << 20):
                reachable.add(column_case(nat.bias_gelu_plan(rows, nvec * 8, kind), rows))
        tested = set()
        for nvec in NVECS:
            for rows in SHORT_ROWS + [long_rows(nvec)]:
                tested.add(column_case(nat.bias_gelu_plan(rows, nvec * 8, kind), rows))
        assert tested == reachable, (kind, sorted(reachable - tested))
        assert len(tested) == 8


# ---------------------------------------------------------------------------------------------------
# softmax cross entropy
# ---------------------------------------------------------------------------------------------------
XENT_COLS = [1, 7, 8, 9, 511, 512, 513, 4097, 30522]
XENT_ROWS = 24


def _exp_rel(d):
    """Relative error of __expf at d: 2 + 1.173 |d| ulp (one ulp <= 2 E32), plus the rounding of its argument."""
    return (2 + 1.2 * d.abs()) * 2 * E32 + E32 * d.abs()


def _xent_case(cols, dtype, seed, stride=None):
    g = torch.Generator(device="cuda").manual_seed(seed)
    stride = stride or cols
    full = (torch.randn(XENT_ROWS, stride, device="cuda", generator=g) * 3).to(dtype)
    if stride > cols:
        full[:, cols:] = 3e4  # padding that must never be read
    logits = full[:, :cols]
    target = torch.randint(0, cols, (XENT_ROWS,), device="cuda", generator=g)
    ninf = float("-inf")
    # rows 0-2: leading 1, 8 and >= 512 * 8 logits -inf; row 3: one stray -inf; row 4: all -inf (NaN, as PyTorch)
    for r, lead in ((0, 1), (1, 8), (2, 4099)):
        if lead < cols:
            logits[r, :lead] = ninf
            target[r] = cols - 1
    if cols > 2:
        c = (cols * 2) // 3
        logits[3, c] = ninf
        target[3] = (c + 1) % cols
    logits[4] = ninf
    target[5] = -100  # ignored
    target[6] = cols  # out of range
    target[7] = -3
    return full, target


def check_xent(nat, full, target, cols, dtype):
    stride = full.shape[1]
    valid = cols if stride > cols else 0
    loss, lse = nat.softmax_xent_fwd(full, target, -100, valid)
    dloss = torch.tensor([0.75], device="cuda")
    dl = nat.softmax_xent_bwd(full, target, lse, dloss, -100, valid)
    x = full[:, :cols].double()
    finite = torch.isfinite(x)
    m = x.masked_fill(~finite, -math.inf).amax(-1, keepdim=True)
    ref_lse = torch.logsumexp(x, -1, keepdim=True)
    rng = (m - x.masked_fill(~finite, math.inf).amin(-1, keepdim=True)).clamp_min(0)
    ok_rows = torch.isfinite(m).squeeze(1)
    valid_t = (target >= 0) & (target < cols)
    tt = target.clamp(0, cols - 1)
    # forward: s = sum exp(x - m) over <= cols / 512 + 8 additions per thread, rescaled by exp at most once per vector
    # and per merge level (10); every exp has the error of its argument, at most the row's range
    iters = -(-cols // 512) + 2
    rel_s = (iters * 9 + 12) * E32 + (iters + 11) * _exp_rel(rng)
    ls = ref_lse - m
    lse_err = rel_s + 2.0 ** -21.41 + 6 * E32 * ls.abs() + E32 * ref_lse.abs()
    okl = ok_rows[:, None]
    _assert_within(lse[:, None].where(okl, torch.zeros_like(lse[:, None])),
                   ref_lse.where(okl, torch.zeros_like(ref_lse)), lse_err.where(okl, torch.zeros_like(lse_err)), "lse")
    xt = x.gather(1, tt[:, None])
    ref_loss = ref_lse - xt
    counted = (valid_t & ok_rows)[:, None]
    bound = lse_err + E32 * (ref_loss.abs() + xt.abs())
    _assert_within(loss[:, None].where(counted, torch.zeros_like(loss[:, None])),
                   ref_loss.where(counted, torch.zeros_like(ref_loss)), bound.where(counted, torch.zeros_like(bound)),
                   "loss")
    assert bool((loss[~valid_t] == 0).all()), "ignored or out-of-range targets must give a zero loss"
    # all -inf: NaN, as PyTorch
    dead = ~ok_rows
    if dead.any():
        xr = full[dead, :cols].float().requires_grad_(True)
        tr = target[dead].clamp(0, cols - 1)
        ref_nan = F.cross_entropy(xr, tr, reduction="none")
        ref_nan.sum().backward()
        assert torch.equal(torch.isnan(loss[dead]), torch.isnan(ref_nan)) and bool(torch.isnan(loss[dead]).all())
        assert torch.equal(torch.isnan(dl[dead, :cols].float()), torch.isnan(xr.grad))
    # backward from the saved lse: (exp(x - lse) - [c == t]) * dloss, zero rows for ignored targets, exact 0 at -inf
    # and in the padding
    live = (valid_t & ok_rows)
    lz = lse.double()[:, None]
    d = x - lz
    p = torch.exp(d).where(finite, torch.zeros_like(d))
    onehot = torch.zeros_like(p).scatter_(1, tt[:, None], 1.0)
    ref = (p - onehot) * 0.75
    comp = 0.75 * (p * _exp_rel(d.where(finite, torch.zeros_like(d))) + E32 * (p + onehot)) + E32 * ref.abs() + FTZ
    got = dl[:, :cols]
    rows_ok = live[:, None].expand_as(got)
    _assert_within(got.where(rows_ok, torch.zeros_like(got)), ref.where(rows_ok, torch.zeros_like(ref)),
                   UNIT[dtype] * (ref.abs() + comp) + comp + _tiny(dtype), "dlogits")
    assert bool((dl[~valid_t] == 0).all()), "ignored rows must get a zero gradient"
    assert bool((got[ok_rows][~finite[ok_rows]] == 0).all()), "-inf logits must get a zero gradient"
    if stride > cols:
        assert bool((dl[:, cols:] == 0).all()), "padding columns of the gradient must be 0"
    return loss, lse, dl


@pytest.mark.parametrize("cols", XENT_COLS)
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_cross_entropy(dtype, cols):
    nat = _native()
    full, target = _xent_case(cols, dtype, seed=cols)
    check_xent(nat, full, target, cols, dtype)
    # rows at every offset from a 16-byte boundary: the same rows one element further into a buffer
    buf = torch.empty(XENT_ROWS * cols + 1, device="cuda", dtype=dtype)
    shifted = buf[1:].view(XENT_ROWS, cols)
    shifted.copy_(full)
    check_xent(nat, shifted, target, cols, dtype)


@pytest.mark.parametrize("cols", [7, 513, 30522])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_cross_entropy_padded_stride(dtype, cols):
    """`valid_cols` < stride (a vocabulary padded for the GEMMs): the padding is never read, its gradient is 0."""
    nat = _native()
    stride = -(-cols // 64) * 64 + 64
    full, target = _xent_case(cols, dtype, seed=cols + 1, stride=stride)
    check_xent(nat, full, target, cols, dtype)


# ---------------------------------------------------------------------------------------------------
# Gaussian basis
# ---------------------------------------------------------------------------------------------------
GBF_K = [8, 16, 32, 64, 128, 256]
GBF_E = [1, 961, 8192]
GBF_A = (2 * 3.14159) ** 0.5


def gbf_rows(K):
    """Rows with which every CTA runs three or more iterations and the last sweep is ragged."""
    nat = _native()
    sweep = nat.gbf_plan(1 << 30, K, 1)["rows_per_sweep"]
    n = 3 * sweep + sweep // 2 + 3
    p = nat.gbf_plan(n, K, 1)
    assert p["sweeps"] == 4 and n % p["rows_per_sweep"] != 0, p
    return n


def _gbf_inputs(n, K, E, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    d = (torch.rand(n, device="cuda", generator=g) * 8).to(dtype)
    edge = torch.randint(0, E, (n,), device="cuda", generator=g)
    mul = (torch.rand(E, device="cuda", generator=g) + 0.5).to(dtype)
    bias = (torch.randn(E, device="cuda", generator=g) * 0.5).to(dtype)
    means = (torch.rand(K, device="cuda", generator=g) * 6).to(dtype)
    stds = (torch.rand(K, device="cuda", generator=g) * 2 + 0.2).to(dtype)
    stds[1::3] = -stds[1::3]  # negative: |stds| is used
    stds[2] = 0.0  # std = 1e-5 exactly, the narrowest basis function
    stds[min(5, K - 1)] = 1e-3
    dy = torch.randn(n, K, device="cuda", generator=g).to(dtype)
    return d, edge, mul, bias, means, stds, dy


def gbf_reference(d, edge, mul, bias, means, stds, dy, rows):
    """fp64 y and gradient terms for `rows`, with the kernel's fp32 error of each."""
    dd = d[rows].double()
    e = edge[rows]
    md, bd = mul.double()[e], bias.double()[e]
    t = (md * dd + bd)[:, None]
    mean = means.double()[None, :]
    s = stds.double().abs()[None, :] + 1e-5
    z = (t - mean) / s
    y = torch.exp(-0.5 * z * z) / (GBF_A * s)
    # t: one fma (or a product and a sum); 1e-5 added to |stds| and 1/s, 1/(A s) (div.approx: 2 ulp) in fp32
    dt_abs = 2 * E32 * ((md * dd).abs() + bd.abs())[:, None]
    dz = (dt_abs + E32 * (t - mean).abs()) / s + z.abs() * 6 * E32
    # y: z*z*-0.5 (2 roundings), __expf of it, the product with the normaliser
    arg = 0.5 * z * z
    rel_y = z.abs() * dz + 2 * E32 * arg + _exp_rel(arg) + 6 * E32
    # __expf flushes results below 2^-126 to 0, which the normaliser 1 / (A s) then scales
    return t, z, s, y, dz, rel_y, FTZ * (1 + 1 / (GBF_A * s))


def check_gbf(nat, d, edge, mul, bias, means, stds, dy, dtype, det):
    n, K = dy.shape
    E = mul.numel()
    y = nat.gbf_fwd(d, edge, mul, bias, means, stds)
    u, tiny = UNIT[dtype], _tiny(dtype)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        dmul, dbias, dmean, dstd = nat.gbf_bwd(dy, d, edge, mul, bias, means, stds)
    finally:
        torch.use_deterministic_algorithms(prev)
    plan = nat.gbf_plan(n, K, E)
    acc = {k: torch.zeros(n_, dtype=torch.float64, device="cuda") for k, n_ in
           (("mul", E), ("bias", E), ("mean", K), ("std", K), ("mul_a", E), ("bias_a", E), ("mean_a", K), ("std_a", K),
            ("mul_c", E), ("bias_c", E), ("mean_c", K), ("std_c", K))}
    step = max(1, CHUNK // K)
    for r0 in range(0, n, step):
        rows = slice(r0, min(n, r0 + step))
        t, z, s, yr, dz, rel_y, ftz = gbf_reference(d, edge, mul, bias, means, stds, dy, rows)
        comp = yr * rel_y + ftz
        _assert_within(y[rows], yr, u * (yr.abs() + comp) + comp + tiny, "gaussian basis")
        g = dy[rows].double()
        gy = g * yr
        gyc = g.abs() * comp
        zs = z / s
        tm = gy * zs  # d mean term; dt = -sum_k tm
        tm_c = gyc * zs.abs() + gy.abs() * (dz / s + 4 * E32 * zs.abs())
        ts = gy * (z * z - 1) / s
        ts_c = gyc * (z * z + 1) / s + gy.abs() * (2 * z.abs() * dz + 6 * E32 * (z * z + 1)) / s
        dtr = -tm.sum(1)
        dta = tm.abs().sum(1)
        dtc = tm_c.sum(1) + 16 * E32 * dta  # 8 in-thread additions, <= 5 shuffle levels
        dist = d[rows].double()
        e = edge[rows]
        acc["mean"] += tm.sum(0)
        acc["mean_a"] += tm.abs().sum(0)
        acc["mean_c"] += tm_c.sum(0)
        acc["std"] += ts.sum(0)
        acc["std_a"] += ts.abs().sum(0)
        acc["std_c"] += ts_c.sum(0)
        acc["mul"].index_add_(0, e, dtr * dist)
        acc["mul_a"].index_add_(0, e, dta * dist.abs())
        acc["mul_c"].index_add_(0, e, (dtc + E32 * dta) * dist.abs())
        acc["bias"].index_add_(0, e, dtr)
        acc["bias_a"].index_add_(0, e, dta)
        acc["bias_c"].index_add_(0, e, dtc)
    # chains: a thread's rows, the CTA's row groups (shared atomics or the fixed-order sum), the sum over CTAs; per
    # edge type, every row of a CTA (atomics) or of the type (the sorted sum) and the CTAs
    per_type = torch.bincount(edge, minlength=E).max().item()
    col_chain = plan["sweeps"] + plan["rows_per_cta"] + plan["grid"] + 2
    edge_chain = (per_type if det else plan["sweeps"] * plan["rows_per_cta"] + plan["grid"]) + 2
    for got, k, chain in ((dmean, "mean", col_chain), (dstd, "std", col_chain), (dmul, "mul", edge_chain),
                          (dbias, "bias", edge_chain)):
        _check_sum(got, acc[k], acc[k + "_a"], acc[k + "_c"], torch.float32, chain, "d " + k)
    return y, (dmul, dbias, dmean, dstd)


@pytest.mark.parametrize("E", GBF_E)
@pytest.mark.parametrize("K", GBF_K)
@pytest.mark.parametrize("dtype", HALF)
def test_gaussian_basis_all_paths(dtype, K, E):
    nat = _native()
    n = gbf_rows(K)
    args = _gbf_inputs(n, K, E, dtype, seed=K * 10 + E)
    y, grads = check_gbf(nat, *args, dtype, det=False)
    y2, grads2 = check_gbf(nat, *args, dtype, det=True)
    assert torch.equal(y, y2)
    # the short end: one row, one partial CTA
    for short in (1, 37):
        sub = [a[:short] if i in (0, 1, 6) else a for i, a in enumerate(args)]
        check_gbf(nat, *sub, dtype, det=False)


@pytest.mark.parametrize("det", [False, True])
def test_gaussian_basis_no_pairs(det):
    """An empty distance tensor: every parameter gradient of ``ops.gaussian_basis`` is zero, in the default and in
    deterministic mode."""
    from unicore import ops

    K, E, dtype = 128, 64, torch.float16
    d, edge, mul, bias, means, stds, _ = _gbf_inputs(0, K, E, dtype, seed=11)
    params = [t.clone().requires_grad_(True) for t in (mul, bias, means, stds)]
    y = ops.gaussian_basis(d, edge, *params)
    assert y.shape == (0, K)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    try:
        _nan_blocks((1, 2 * K))  # the size of one CTA's partial (d mean, d std) row
        y.backward(torch.empty_like(y))
    finally:
        torch.use_deterministic_algorithms(prev)
    for p in params:
        assert torch.equal(p.grad, torch.zeros_like(p)), p.grad


def test_gaussian_dispatch_coverage():
    """Every K geometry (8 ... 256, kvec = 1 ... 32) with and without the > 48 KB shared-memory opt-in of the backward
    is run by the test shapes above; none of this launches a kernel."""
    nat = _native()
    tested = set()
    for K in GBF_K:
        n = gbf_rows(K)
        for E in GBF_E:
            p = nat.gbf_plan(n, K, E)
            assert p["sweeps"] >= 3 and n % p["rows_per_sweep"] != 0
            tested.add((p["kvec"], p["smem"] > 48 * 1024))
    reachable = {(nat.gbf_plan(1000, K, E)["kvec"], nat.gbf_plan(1000, K, E)["smem"] > 48 * 1024)
                 for K in (8 << i for i in range(6)) for E in (1, 100, 6000, 6200, 8192)}
    assert reachable == tested, sorted(reachable - tested)
    assert len(tested) == 12
