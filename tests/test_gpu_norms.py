"""LayerNorm, RMSNorm and the fused bias + dropout + residual + LayerNorm kernels against fp64 references.

Every width is chosen from the launch plan (``norm_plan``, the function the launchers run) so that each dispatch
case of ``csrc/norm/norm.cu`` runs, and every row count so that each loop unit (a warp for v3, a CTA for v2 and v1)
runs several tiles and the last sweep over the grid is ragged: the register prefetch of the next rows, the column
accumulators carried from tile to tile and the v2 bulk-copy ring only run from a unit's second tile on.

Error bounds are per element.  The kernels compute in fp32 and round each output once, so a bound is one rounding
of the output type (``UNIT[dtype] * |ref|``) plus the fp32 error of the computation, which is a small multiple of
``E32`` times the magnitudes that enter it.  The backward is checked against the statistics the forward saved (its
inputs), the forward against exact fp64 statistics.
"""
import math

import pytest
import torch

from test_gpu_elementwise import column_chain as column_sum_chain

pytestmark = pytest.mark.gpu

DTYPES = [torch.float32, torch.float16, torch.bfloat16]
E32 = 2.0 ** -24
UNIT = {torch.float32: 2.0 ** -24, torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}  # unit roundoff
EPS = 1e-5
CHUNK = 1 << 21  # elements per fp64 reference chunk (keeps the reference's memory small)

# Row widths in 16-byte vectors (cols = nvec * elements per vector):
#   v3 (one warp per row), every (VPL, LPR) case of UB_DISPATCH_V3, full and partial:
#     1 (1,1)  2 (1,2)  3/4 (1,4)  5/8 (1,8)  9/16 (1,16)  25/32 (1,32)  40/64 (2,32)  65/96 (3,32)  125/128 (4,32)
#   v2 (bulk-copy ring): 129 / 192 two row groups, partial / full last warp; 250 / 256 / 384 one row group
#   v1 (rows in registers): 500 (4 vectors per thread, 2 rows per CTA), 520 (3 vectors), 1024 (4 vectors)
V1_NVECS = [500, 520, 1024]
NVECS = [1, 2, 3, 4, 5, 8, 9, 16, 25, 32, 40, 64, 65, 96, 125, 128, 129, 192, 250, 256, 384] + V1_NVECS
MIN_TILES = {3: 3, 2: 9, 1: 3}  # v2: a ring stage is reused from the 5th tile on, its parity flips back at the 9th


def _native():
    from unicore import ops

    assert ops.USE_NATIVE, "native kernels must be active on the GPU box"
    return ops.native()


def _epv(dtype):
    return 16 // torch.empty((), dtype=dtype).element_size()


def _tiny(dtype):
    return torch.finfo(dtype).tiny * UNIT[dtype]  # half the spacing of the subnormals


def norm_case(plan):
    """The dispatch case a plan runs (None: no kernel)."""
    if plan["gen"] == 3:
        return (3, plan["vpl"], plan["lpr"], plan["full"])
    if plan["gen"] == 2:
        return (2, plan["groups"], plan["full"])
    if plan["gen"] == 1:
        return (1, plan["vpt"], plan["tpr"])
    return None


def plan_rows(cols, dtype, kinds):
    """Rows with which every loop unit of every kernel in `kinds` runs MIN_TILES tiles or more, and a ragged last sweep."""
    nat = _native()
    big = [nat.norm_plan(1 << 30, cols, dtype, k) for k in kinds]
    sweep = max(p["rows_per_sweep"] for p in big)
    rows = MIN_TILES[big[0]["gen"]] * sweep + sweep // 2 + 1
    for k in kinds:
        p = nat.norm_plan(rows, cols, dtype, k)
        assert p["tiles_min"] >= MIN_TILES[p["gen"]], (k, p)
        assert rows % p["rows_per_sweep"] != 0, (k, p)
    return rows


def _chunks(rows, cols):
    step = max(1, CHUNK // cols)
    for r0 in range(0, rows, step):
        yield slice(r0, min(rows, r0 + step))


def _assert_within(got, ref, bound, what):
    err = (got.double() - ref).abs()
    bad = err > bound
    if bad.any():
        i = bad.nonzero()[0].tolist()
        worst = (err / bound.clamp_min(1e-300)).max().item()
        raise AssertionError("{}: {} elements out of bound, first at {}: got {}, want {} +- {} (worst {:.3g}x)".format(
            what, int(bad.sum()), i, got[tuple(i)].item(), ref[tuple(i)].item(), bound[tuple(i)].item(), worst))


def check_forward(x, w, b, y, mean, rstd, rms):
    """y, mean and rstd of LayerNorm (RMSNorm if `rms`) of the rounded inputs x, w, b, in fp64."""
    dtype = x.dtype
    rows, cols = x.shape
    wd = w.double()
    bd = b.double() if b is not None else torch.zeros_like(wd)
    for s in _chunks(rows, cols):
        xd = x[s].double()
        if rms:
            mu = torch.zeros(xd.shape[0], 1, dtype=torch.float64, device=x.device)
            var = (xd * xd).mean(-1, keepdim=True)
        else:
            mu = xd.mean(-1, keepdim=True)
            var = ((xd - mu) ** 2).mean(-1, keepdim=True)
            # fp32 row sum: chains of at most 32 additions per thread plus at most 17 reduction levels (< 64)
            _assert_within(mean[s, None], mu, 64 * E32 * xd.abs().mean(-1, keepdim=True), "mean")
        rs = torch.rsqrt(var + EPS)
        dmu = 0.0 if rms else (mean[s, None].double() - mu).abs()
        # rstd: the same sum bound on the variance (its relative error halves under the square root), rsqrt's
        # approximation, and the mean's error, which adds dmu^2 to the variance of the centred values
        _assert_within(rstd[s, None], rs, rs * (72 * E32 + (dmu * rs) ** 2), "rstd")
        drs = (rstd[s, None].double() - rs).abs() / rs
        xh = (xd - mu) * rs
        yr = xh * wd + bd
        # the measured statistics errors carried through x_hat, a few fp32 roundings, one rounding to the output type
        comp = wd.abs() * (dmu * rs + xh.abs() * drs) + 4 * E32 * ((xh * wd).abs() + bd.abs())
        _assert_within(y[s], yr, UNIT[dtype] * (yr.abs() + comp) + comp + _tiny(dtype), "y")


def backward_ref(dy, x, mean, rstd, w, rms):
    """fp64 backward from the saved statistics, chunk by chunk: yields (rows, dx_ref, dx_comp_bound, dy_d, xh)."""
    rows, cols = x.shape
    wd = w.double()
    for s in _chunks(rows, cols):
        xd, dyd = x[s].double(), dy[s].double()
        mu = 0.0 if rms else mean[s, None].double()
        rs = rstd[s, None].double()
        xh = (xd - mu) * rs
        gy = dyd * wd
        m1 = torch.zeros_like(rs) if rms else gy.mean(-1, keepdim=True)
        m2 = (gy * xh).mean(-1, keepdim=True)
        dx = rs * (gy - m1 - xh * m2)
        # fp32 error: a few roundings per element (x_hat, dy * gamma, the combination) and the two row sums
        comp = rs * (4 * E32 * (gy.abs() + m1.abs() + (xh * m2).abs() + xh.abs() * m2.abs())
                     + 72 * E32 / cols * (gy.abs().sum(-1, keepdim=True) + xh.abs() * (gy * xh).abs().sum(-1, keepdim=True)))
        yield s, dx, comp, dyd, xh


def column_chain(plan):
    """Longest chain of fp32 additions behind one parameter-gradient column: one per row a thread visits plus the
    fixed-order sums across warps, CTAs and the finalize pass (< 80)."""
    return plan["tiles_max"] * plan["tile_rows"] + 80


def dbias_chain(nat, plan, rows, cols):
    """The chain behind the fused op's dbias: the norm kernel's column sums at v3 / v2 widths; at v1 widths the
    column sum of the rounded dx that runs after the norm kernel."""
    return column_sum_chain(nat.bias_gelu_plan(rows, cols, "bwd")) if plan["gen"] == 1 else column_chain(plan)


def check_param_grad(got, ref, absum, dtype, chain, what, base=None):
    """A column sum accumulated in fp32 and rounded once (onto `base` when the gradient went into a sink)."""
    if base is not None:
        ref = ref + base.double()
        absum = absum + base.double().abs()
    comp = chain * E32 * absum
    _assert_within(got, ref, UNIT[dtype] * (ref.abs() + comp) + comp + _tiny(dtype), what)


def _inputs(rows, cols, dtype, seed, offset=0.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = (torch.randn(rows, cols, device="cuda", generator=g) * 2 + 0.5 + offset).to(dtype)
    w = (torch.randn(cols, device="cuda", generator=g) * 0.5 + 1).to(dtype)
    b = torch.randn(cols, device="cuda", generator=g).to(dtype)
    dy = torch.randn(rows, cols, device="cuda", generator=g).to(dtype)
    return x, w, b, dy


def run_norm(nat, rms, x, w, b, dy, sinks=()):
    if rms:
        y, rstd = nat.rmsnorm_fwd(x, w, EPS)
        mean = None
        dx, dg = nat.rmsnorm_bwd(dy, x, rstd, w, *sinks)
        db = None
    else:
        y, mean, rstd = nat.layernorm_fwd(x, w, b, EPS)
        dx, dg, db = nat.layernorm_bwd(dy, x, mean, rstd, w, *sinks)
    return y, mean, rstd, dx, dg, db


def check_norm(nat, rms, x, w, b, dy, y, mean, rstd, dx, dg, db, chain, sinks=None):
    dtype, cols = x.dtype, x.shape[1]
    check_forward(x, w, None if rms else b, y, mean, rstd, rms)
    dg_r = torch.zeros(cols, dtype=torch.float64, device="cuda")
    db_r, dg_a, db_a = torch.zeros_like(dg_r), torch.zeros_like(dg_r), torch.zeros_like(dg_r)
    for s, dxr, comp, dyd, xh in backward_ref(dy, x, mean, rstd, w, rms):
        _assert_within(dx[s], dxr, UNIT[dtype] * (dxr.abs() + comp) + comp + _tiny(dtype), "dx")
        dg_r += (dyd * xh).sum(0)
        dg_a += (dyd * xh).abs().sum(0)
        db_r += dyd.sum(0)
        db_a += dyd.abs().sum(0)
    bases = sinks or (None, None)
    check_param_grad(dg, dg_r, dg_a, dtype, chain, "dgamma", bases[0])
    if not rms:
        check_param_grad(db, db_r, db_a, dtype, chain, "dbeta", bases[1])


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("nvec", NVECS)
@pytest.mark.parametrize("rms", [False, True], ids=["layer_norm", "rms_norm"])
def test_norm_all_paths(rms, nvec, dtype):
    nat = _native()
    cols = nvec * _epv(dtype)
    rows = plan_rows(cols, dtype, ("fwd", "bwd"))
    chain = column_chain(nat.norm_plan(rows, cols, dtype, "bwd"))
    x, w, b, dy = _inputs(rows, cols, dtype, seed=nvec)
    y, mean, rstd, dx, dg, db = run_norm(nat, rms, x, w, b, dy)
    check_norm(nat, rms, x, w, b, dy, y, mean, rstd, dx, dg, db, chain)
    # the backward is deterministic: fixed-order sums, no atomics
    dx2, dg2 = run_norm(nat, rms, x, w, b, dy)[3:5]
    assert torch.equal(dx, dx2) and torch.equal(dg, dg2)
    if not rms:
        assert torch.equal(db, nat.layernorm_bwd(dy, x, mean, rstd, w)[2])
    # the short end: one row, and a single partial sweep
    for short in (1, 31):
        ys, ms, rss, dxs, dgs, dbs = run_norm(nat, rms, x[:short], w, b, dy[:short])
        check_norm(nat, rms, x[:short], w, b, dy[:short], ys, ms, rss, dxs, dgs, dbs, 80)


@pytest.mark.parametrize("nvec", NVECS)
def test_layer_norm_large_common_offset(nvec):
    """fp32 rows with |mean| / std ~ 1e3: x_hat must be formed as (x - mean) * rstd; the forms that fold the mean into
    a product first lose ~1e3 ulp of x_hat to cancellation."""
    nat = _native()
    dtype = torch.float32
    cols = nvec * _epv(dtype)
    rows = plan_rows(cols, dtype, ("fwd", "bwd"))
    chain = column_chain(nat.norm_plan(rows, cols, dtype, "bwd"))
    x, w, b, dy = _inputs(rows, cols, dtype, seed=1000 + nvec, offset=2e3)
    y, mean, rstd, dx, dg, db = run_norm(nat, False, x, w, b, dy)
    check_norm(nat, False, x, w, b, dy, y, mean, rstd, dx, dg, db, chain)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("nvec", [96, 192, 520], ids=["v3", "v2", "v1"])
@pytest.mark.parametrize("rms", [False, True], ids=["layer_norm", "rms_norm"])
def test_norm_gradient_sinks(rms, nvec, dtype):
    """dgamma / dbeta written into sinks (views of the optimizer's gradient arena): sink = base + gradient with one
    rounding, the sink itself is returned, and nothing around it is written."""
    nat = _native()
    cols = nvec * _epv(dtype)
    rows = plan_rows(cols, dtype, ("fwd", "bwd"))
    chain = column_chain(nat.norm_plan(rows, cols, dtype, "bwd"))
    x, w, b, dy = _inputs(rows, cols, dtype, seed=2000 + nvec)
    arena = torch.randn(3 * cols + 64, device="cuda").to(dtype)
    before = arena.clone()
    sg, sb = arena[16:16 + cols], arena[32 + cols:32 + 2 * cols]
    bases = (sg.clone(), sb.clone())
    sinks = (sg,) if rms else (sg, sb)
    y, mean, rstd, dx, dg, db = run_norm(nat, rms, x, w, b, dy, sinks)
    assert dg.data_ptr() == sg.data_ptr() and (rms or db.data_ptr() == sb.data_ptr())
    check_norm(nat, rms, x, w, b, dy, y, mean, rstd, dx, dg, db, chain, sinks=bases)
    outside = torch.ones_like(arena, dtype=torch.bool)
    outside[16:16 + cols] = False
    if not rms:
        outside[32 + cols:32 + 2 * cols] = False
    assert torch.equal(arena[outside], before[outside])


# ---------------------------------------------------------------------------------------------------
# fused bias + dropout + residual + LayerNorm
# ---------------------------------------------------------------------------------------------------
def _fused_case(nat, x, bias, res, w, b, dy, p, sinks=()):
    y, mean, rstd, summed, seed, off = nat.bias_dropout_add_ln_fwd(x, bias, res, w, b, p, EPS)
    dsum, dx, dg, db, dbias = nat.bias_dropout_add_ln_bwd(dy, summed, mean, rstd, w, p, seed, off, True, *sinks)
    return y, mean, rstd, summed, dsum, dx, dg, db, dbias


# p = 0.5 puts the 16-bit threshold at the top bit of each random lane
FUSED_PS = [0.1, 0.0, 0.5]


@pytest.mark.parametrize("p", FUSED_PS)
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("nvec", [n for n in NVECS if n not in V1_NVECS])
def test_bias_dropout_add_ln_all_paths(nvec, dtype, p):
    check_fused_all_paths(nvec, dtype, p)


@pytest.mark.parametrize("p", FUSED_PS)
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("nvec", V1_NVECS)
def test_bias_dropout_add_ln_dbias_at_gen1_widths(nvec, dtype, p):
    """The v1 widths return dbias too: a column sum of the rounded dx that runs after the norm kernel, into a sink as
    well.  Every other check is the one of the v3 / v2 widths."""
    check_fused_all_paths(nvec, dtype, p)


def check_fused_all_paths(nvec, dtype, p):
    nat = _native()
    cols = nvec * 8
    rows = plan_rows(cols, dtype, ("fused", "bwd"))
    plan = nat.norm_plan(rows, cols, dtype, "bwd")
    chain, bias_chain = column_chain(plan), dbias_chain(nat, plan, rows, cols)
    g = torch.Generator(device="cuda").manual_seed(3000 + nvec)
    x = torch.randn(rows, cols, device="cuda", generator=g).to(dtype)
    res = torch.randn(rows, cols, device="cuda", generator=g).to(dtype)
    bias = torch.randn(cols, device="cuda", generator=g).to(dtype)
    w = (torch.randn(cols, device="cuda", generator=g) * 0.5 + 1).to(dtype)
    b = torch.randn(cols, device="cuda", generator=g).to(dtype)
    dy = torch.randn(rows, cols, device="cuda", generator=g).to(dtype)
    u, tiny = UNIT[dtype], _tiny(dtype)
    torch.cuda.manual_seed(11)  # the same Philox state for every run compared below
    y, mean, rstd, summed, dsum, dx, dg, db, dbias = _fused_case(nat, x, bias, res, w, b, dy, p)
    assert dbias is not None  # at every width
    # the keep mask, read from dx (zero where the element was dropped, or where dsum underflowed to zero: there
    # the forward's sum tells, it differs from the residual where x + bias was added); forward and backward agree
    keep = (dx != 0) | ((dsum == 0) & (summed != res)) if p > 0 else torch.ones_like(dx, dtype=torch.bool)
    if p > 0:
        rate = keep.double().mean().item()
        assert abs(rate - (1 - p)) < 6 * math.sqrt(p * (1 - p) / keep.numel()) + 2.0 ** -16, rate
    # kept elements are scaled by 1 / P(keep) of the 16-bit threshold the kernels compare against
    t16 = min(int(p * 65536 + 0.5), 65535)
    scale = 65536 / (65536 - t16)
    # summed = residual + keep * (x + bias) * scale: a few fp32 roundings, one rounding to the output type
    for s in _chunks(rows, cols):
        h = keep[s].double() * (x[s].double() + bias.double()) * scale
        ref = res[s].double() + h
        comp = 4 * E32 * (res[s].double().abs() + h.abs())
        _assert_within(summed[s], ref, u * (ref.abs() + comp) + comp + tiny, "summed")
    # LayerNorm of the stored (rounded) sum, and its backward from the saved statistics
    check_forward(summed, w, b, y, mean, rstd, False)
    dg_r = torch.zeros(cols, dtype=torch.float64, device="cuda")
    db_r, dg_a, db_a, dbi_r, dbi_a = (torch.zeros_like(dg_r) for _ in range(5))
    for s, dsr, comp, dyd, xh in backward_ref(dy, summed, mean, rstd, w, False):
        _assert_within(dsum[s], dsr, u * (dsr.abs() + comp) + comp + tiny, "dsum")
        k = keep[s].double() * scale
        dxr, dxc = dsr * k, (comp + 2 * E32 * dsr.abs()) * k
        _assert_within(dx[s], dxr, u * (dxr.abs() + dxc) + dxc + tiny, "dx")
        dg_r += (dyd * xh).sum(0)
        dg_a += (dyd * xh).abs().sum(0)
        db_r += dyd.sum(0)
        db_a += dyd.abs().sum(0)
        dbi_r += dxr.sum(0)
        # the per-element error of the dx terms enters the column sum: fp32 ones at v3 / v2 widths, the rounded dx
        # (the bound checked above) at v1 widths
        dxe = u * (dxr.abs() + dxc) + dxc + tiny if plan["gen"] == 1 else dxc
        dbi_a += (dxr.abs() + dxe / E32 / bias_chain).sum(0)
    check_param_grad(dg, dg_r, dg_a, dtype, chain, "dgamma")
    check_param_grad(db, db_r, db_a, dtype, chain, "dbeta")
    check_param_grad(dbias, dbi_r, dbi_a, dtype, bias_chain, "dbias")
    # deterministic backward
    torch.cuda.manual_seed(11)
    again = _fused_case(nat, x, bias, res, w, b, dy, p)
    assert torch.equal(summed, again[3])
    for got, rep in zip((dsum, dx, dg, db, dbias), again[4:]):
        assert torch.equal(got, rep)
    if nvec not in (96, 192, 520) or p == 0:
        return
    # gradient sinks (one width per generation): sink = base + gradient with one rounding, nothing else written
    arena = torch.randn(3 * cols + 64, device="cuda").to(dtype)
    before = arena.clone()
    views = (arena[16:16 + cols], arena[32 + cols:32 + 2 * cols], arena[48 + 2 * cols:48 + 3 * cols])
    bases = [v.clone() for v in views]
    torch.cuda.manual_seed(11)
    fw = nat.bias_dropout_add_ln_fwd(x, bias, res, w, b, p, EPS)
    assert torch.equal(fw[3], summed)
    out = nat.bias_dropout_add_ln_bwd(dy, fw[3], fw[1], fw[2], w, p, fw[4], fw[5], True, *views)
    assert torch.equal(out[0], dsum) and torch.equal(out[1], dx)  # same mask as the run above
    for got, view, base, ref, absum, ch, what in zip(out[2:], views, bases, (dg_r, db_r, dbi_r),
                                                     (dg_a, db_a, dbi_a), (chain, chain, bias_chain),
                                                     ("dgamma", "dbeta", "dbias")):
        assert got.data_ptr() == view.data_ptr()
        check_param_grad(got, ref, absum, dtype, ch, what + " sink", base)
    outside = torch.ones_like(arena, dtype=torch.bool)
    for v in views:
        outside[(v.data_ptr() - arena.data_ptr()) // arena.element_size():][:cols] = False
    assert torch.equal(arena[outside], before[outside])


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("nvec", [96, 192, 520], ids=["v3", "v2", "v1"])
def test_bias_dropout_add_layer_norm_op(nvec, dtype):
    """The autograd op equals the bindings, p = 0 and training=False included; the bias gradient comes from the
    binding at every width, also when it goes into a sink (a view of the optimizer's gradient arena)."""
    from unicore import ops
    from unicore_b200.ops import grad_sink

    nat = _native()
    cols = nvec * 8
    rows = plan_rows(cols, dtype, ("fused", "bwd"))
    plan = nat.norm_plan(rows, cols, dtype, "bwd")
    g = torch.Generator(device="cuda").manual_seed(4000 + nvec)
    x = torch.randn(rows, cols, device="cuda", generator=g).to(dtype).requires_grad_(True)
    res = torch.randn(rows, cols, device="cuda", generator=g).to(dtype).requires_grad_(True)
    bias = torch.randn(cols, device="cuda", generator=g).to(dtype).requires_grad_(True)
    w = (torch.randn(cols, device="cuda", generator=g) * 0.5 + 1).to(dtype).requires_grad_(True)
    b = torch.randn(cols, device="cuda", generator=g).to(dtype).requires_grad_(True)
    dy = torch.randn(rows, cols, device="cuda", generator=g).to(dtype)
    arena = torch.randn(cols + 64, device="cuda").to(dtype)
    for p, training, sink in ((0.1, True, False), (0.0, True, False), (0.1, False, False), (0.1, True, True)):
        for t in (x, res, bias, w, b):
            t.grad = None
        base = None
        if sink:
            bias.grad = arena[16:16 + cols]
            base = bias.grad.clone()
            grad_sink.enable([bias])
        torch.cuda.manual_seed(7)
        try:
            y = ops.bias_dropout_add_layer_norm(x, bias, res, w, b, p, EPS, training)
            y.backward(dy)
        finally:
            grad_sink.disable([bias])
        # the same computation through the bindings, same Philox state
        torch.cuda.manual_seed(7)
        pe = p if training else 0.0
        yk, mean, rstd, summed, dsum, dxk, dg, db, dbias = _fused_case(
            nat, x.detach(), bias.detach(), res.detach(), w.detach(), b.detach(), dy, pe)
        assert torch.equal(y, yk) and torch.equal(x.grad, dxk) and torch.equal(res.grad, dsum)
        assert torch.equal(w.grad, dg) and torch.equal(b.grad, db)
        keep = dxk != 0 if pe > 0 else torch.ones_like(dxk, dtype=torch.bool)
        if pe == 0:
            assert torch.equal(summed, (res.detach().float() + (x.detach().float() + bias.detach().float())).to(dtype))
        if sink:
            assert bias.grad.data_ptr() == arena[16:].data_ptr()
        else:
            assert torch.equal(bias.grad, dbias)
        # bias gradient: column sums of dx (fp32, one rounding; at v3 / v2 widths of the fp32 dx before its rounding)
        ref = torch.zeros(cols, dtype=torch.float64, device="cuda")
        absum = torch.zeros_like(ref)
        for s in _chunks(rows, cols):
            ref += dxk[s].double().sum(0)
            absum += dxk[s].double().abs().sum(0)
        chain = dbias_chain(nat, plan, rows, cols)
        check_param_grad(bias.grad, ref, absum * (1 + UNIT[dtype] / E32 / chain), dtype, chain, "dbias", base)
        if pe > 0:
            assert abs(keep.double().mean().item() - 0.9) < 0.01


# ---------------------------------------------------------------------------------------------------
# alignment, plans
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("nvec", [96, 192, 520], ids=["v3", "v2", "v1"])
def test_misaligned_rows_take_the_aligned_copy(nvec, dtype):
    """A contiguous view at an odd element offset gives exactly the result of the same rows in an aligned buffer; the
    bindings refuse it."""
    from unicore import ops

    nat = _native()
    cols = nvec * _epv(dtype)
    rows = 67
    buf = torch.randn(rows * cols + 1, device="cuda").to(dtype)
    xm = buf[1:].view(rows, cols)
    assert xm.is_contiguous() and xm.data_ptr() % 16 != 0
    xa = xm.clone()
    w = (torch.randn(cols, device="cuda") * 0.5 + 1).to(dtype)
    b = torch.randn(cols, device="cuda").to(dtype)
    dbuf = torch.randn(rows * cols + 1, device="cuda").to(dtype)
    dym = dbuf[1:].view(rows, cols)
    for fn in (lambda t: ops.layer_norm(t, (cols,), w, b, EPS), lambda t: ops.rms_norm(t, (cols,), w, EPS)):
        outs = []
        for t, d in ((xm, dym), (xa, dym.clone())):
            t = t.detach().requires_grad_(True)
            y = fn(t)
            y.backward(d)
            outs.append((y, t.grad))
        assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    for call in (lambda: nat.layernorm_fwd(xm, w, b, EPS), lambda: nat.rmsnorm_fwd(xm, w, EPS),
                 lambda: nat.layernorm_bwd(dym, xa, torch.zeros(rows, device="cuda"), torch.ones(rows, device="cuda"), w),
                 lambda: nat.layernorm_fwd(xa, buf[1:1 + cols], b, EPS)):
        with pytest.raises(RuntimeError, match="16-byte aligned"):
            call()
    if dtype == torch.float32:
        return
    res_m = dbuf[1:].view(rows, cols)
    bias = torch.randn(cols, device="cuda").to(dtype)
    outs = []
    for xi, ri in ((xm, res_m), (xa, res_m.clone())):
        xi, ri = xi.detach().requires_grad_(True), ri.detach().requires_grad_(True)
        torch.cuda.manual_seed(3)
        y = ops.bias_dropout_add_layer_norm(xi, bias, ri, w, b, 0.1, EPS, True)
        y.backward(dym)
        outs.append((y, xi.grad, ri.grad))
    for u, v in zip(*outs):
        assert torch.equal(u, v)
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        nat.bias_dropout_add_ln_fwd(xm, bias, xa, w, b, 0.1, EPS)


def test_norm_dispatch_coverage():
    """The test widths reach every case the norm launchers can dispatch to, for every dtype and kernel, and widths
    without a kernel are refused (launches nothing)."""
    nat = _native()
    for dtype in DTYPES:
        epv = _epv(dtype)
        for kind in ("fwd", "bwd", "fused"):
            reachable = {norm_case(nat.norm_plan(1, n * epv, dtype, kind)) for n in range(1, 1025)}
            assert None not in reachable
            tested = {norm_case(nat.norm_plan(1, n * epv, dtype, kind)) for n in NVECS}
            assert tested == reachable, (dtype, kind, sorted(reachable - tested))
        assert nat.norm_plan(1, 1025 * epv, dtype, "fwd")["gen"] == 0
        assert nat.norm_plan(1, 64 * epv + 1, dtype, "fwd")["gen"] == 0
        x = torch.zeros(2, 1025 * epv, device="cuda", dtype=dtype)
        with pytest.raises(RuntimeError, match="no norm kernel"):
            nat.layernorm_fwd(x, x[0].clone(), x[0].clone(), EPS)
