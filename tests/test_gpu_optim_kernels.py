"""The multi-tensor optimizer kernels (``csrc/optim/multi_tensor.cu``) against fp64, on every path.

Each tensor of a launch takes the 16-byte vector path when every buffer it touches is 16-byte aligned, else the scalar
path, and a chunk's last (numel % 8) elements always take the scalar path.  The tests offset one buffer at a time by
one element, use lengths around the 8-element vector and the 8192-element chunk, lists of more than 24 tensors (one
launch each 24) and lists long enough that every CTA of the persistent grid walks several chunks.

Error bounds are per element: one rounding of the output type plus the fp32 error of the update, propagated from the
magnitudes of its operands (``E32`` per rounding; fast-math division and square root 2 ulp).  The reference uses the
fp32 hyper-parameters exactly as the binding computes them (step size and weight-decay factor rounded once).
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

E32 = 2.0 ** -24
UNIT = {torch.float32: 2.0 ** -24, torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
FTZ = 2.0 ** -126
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
NUMELS = [1, 7, 8, 9, 8191, 8192, 8193]
CHUNK = 8192


def _native():
    from unicore import ops

    assert ops.USE_NATIVE, "native kernels must be active on the GPU box"
    return ops.native()


def _ops():
    from unicore import ops

    assert ops.USE_NATIVE
    return ops


def _f32(v):
    return float(torch.tensor(v, dtype=torch.float32))


def _tiny(dtype):
    return torch.finfo(dtype).tiny * UNIT[dtype]


def _assert_within(got, ref, bound, what):
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)
    if bad.any():
        i = bad.nonzero()[0].tolist()
        worst = (err / bound.clamp_min(1e-300)).nan_to_num(math.inf).max().item()
        raise AssertionError("{}: {} elements out of bound, first at {}: got {}, want {} +- {} (worst {:.3g}x)".format(
            what, int(bad.sum()), i, got[tuple(i)].item(), ref[tuple(i)].item(), bound[tuple(i)].item(), worst))


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _big_numel():
    """Elements with which every CTA of the persistent grid (8 per SM) walks three chunks or more, ragged."""
    return 3 * 8 * _sms() * CHUNK + CHUNK // 2 + 5


def _buf(n, dtype, misaligned, fill):
    """A contiguous tensor of n elements, at an odd element offset from a 16-byte boundary when `misaligned`."""
    base = torch.empty(n + 1, device="cuda", dtype=dtype)
    t = base[1:] if misaligned else base[:n]
    t.copy_(fill)
    assert (t.data_ptr() % 16 != 0) == misaligned
    return t


# ---------------------------------------------------------------------------------------------------
# Adam
# ---------------------------------------------------------------------------------------------------
def _hyper(i):
    """Per-tensor hyper-parameters, different for every tensor."""
    return dict(lr=1e-3 * (1 + 0.37 * (i % 7)), beta1=0.9 - 0.01 * (i % 5), beta2=0.999 - 0.003 * (i % 4),
                eps=10.0 ** -(6 + i % 3), step=1 + (i * 7) % 50, bias_correction=(i % 3 != 1),
                weight_decay=0.01 * (i % 4))


def _adam_item(n, gdt, pdt, hdt, mis, ema, seed, hp):
    g0 = torch.Generator(device="cuda").manual_seed(seed)
    p = torch.randn(n, device="cuda", generator=g0)
    g = torch.randn(n, device="cuda", generator=g0) * 4
    m = torch.randn(n, device="cuda", generator=g0) * 0.1
    v = torch.rand(n, device="cuda", generator=g0) * 0.1
    g[: n // 5] *= 1e-3  # small gradients: b1 m + (1 - b1) g cancels where m and g have opposite signs
    w = dict(hp, p=_buf(n, pdt, mis == "p", p), g=_buf(n, gdt, mis == "g", g), m=_buf(n, torch.float32, mis == "m", m),
             v=_buf(n, torch.float32, mis == "v", v))
    if hdt is not None:
        w["p_half"] = _buf(n, hdt, mis == "p_half", torch.zeros(n))
    if ema:
        w["ema"] = _buf(n, torch.float32, mis == "ema", torch.randn(n, device="cuda", generator=g0))
    return w


def adam_reference(w, inv_scale, rel_scale, ema_decay):
    """fp64 update of the (rounded) inputs with the binding's fp32 hyper-parameters; returns refs and error bounds
    (without the output rounding) of p, m, v and ema."""
    b1, b2, eps = _f32(w["beta1"]), _f32(w["beta2"]), _f32(w["eps"])
    ss = w["lr"]
    if w["bias_correction"]:
        ss = w["lr"] * math.sqrt(1 - w["beta2"] ** w["step"]) / (1 - w["beta1"] ** w["step"])
    dm = _f32(1.0 - ss * w["weight_decay"])
    ss = _f32(ss)
    g = w["g"].double() * inv_scale
    ge = g.abs() * rel_scale  # the gradient's error: the kernel's multiplier and the product
    m0, v0, p0 = w["m"].double(), w["v"].double(), w["p"].double()
    m = b1 * m0 + (1 - b1) * g
    me = 3 * E32 * (b1 * m0.abs() + (1 - b1) * g.abs()) + (1 - b1) * ge
    v = b2 * v0 + (1 - b2) * g * g
    ve = 4 * E32 * (b2 * v0 + (1 - b2) * g * g) + 2 * (1 - b2) * g.abs() * ge + FTZ
    sq = v.sqrt()
    den = sq + eps
    # |sqrt(v + e) - sqrt(v)| <= min(e / (2 sqrt(v)), sqrt(e)); sqrt.approx 2 ulp; the addition of eps
    dene = torch.minimum(ve / (2 * sq).clamp_min(1e-300), ve.sqrt()) + 2 * E32 * sq + E32 * den
    upd = m / den
    upde = upd.abs() * (4 * E32 + dene / den) + me / den
    p = p0 * dm - ss * upd
    pe = 3 * E32 * ((p0 * dm).abs() + ss * upd.abs()) + ss * upde + FTZ
    out = dict(p=(p, pe), m=(m, me), v=(v, ve))
    if "ema" in w and ema_decay is not None:
        e0 = w["ema"].double()
        a = 1 - _f32(ema_decay)
        a = _f32(a)
        e = e0 - a * (e0 - p)
        ee = 3 * E32 * (e0.abs() + a * (e0 - p).abs()) + a * pe + FTZ
        out["ema"] = (e, ee)
    return out


def check_adam(work, before, inv_scale, rel_scale, ema_decay, zero_grad, sr=False):
    for w, b in zip(work, before):
        ref = adam_reference(b, inv_scale, rel_scale, ema_decay)
        for k in ("p", "m", "v", "ema"):
            if k not in ref:
                continue
            r, comp = ref[k]
            dt = w[k].dtype
            _assert_within(w[k], r, UNIT[dt] * (r.abs() + comp) + comp + _tiny(dt), "adam " + k)
        if "p_half" in w:
            ph = w["p_half"]
            if w["p"].dtype == torch.float32 and not sr:
                assert torch.equal(ph, w["p"].to(ph.dtype)), "p_half must be the fp32 result rounded once"
            elif sr and ph.dtype == torch.bfloat16 and w["p"].dtype == torch.float32:
                check_sr(w["p"], ph)
            else:
                r, comp = ref["p"]
                dt = ph.dtype
                _assert_within(ph, r, UNIT[dt] * (r.abs() + comp) + comp + _tiny(dt), "adam p_half")
        if zero_grad:
            assert bool((w["g"] == 0).all())
        else:
            assert torch.equal(w["g"], b["g"])


def _snapshot(work):
    return [{k: (v.clone() if torch.is_tensor(v) else v) for k, v in w.items()} for w in work]


@pytest.mark.parametrize("mis", ["none", "p", "g", "m", "v", "p_half", "ema"])
@pytest.mark.parametrize("hdt", [None, torch.float16, torch.bfloat16], ids=["no_half", "half_f16", "half_bf16"])
@pytest.mark.parametrize("pdt", DTYPES, ids=["p32", "p16", "pbf16"])
@pytest.mark.parametrize("gdt", DTYPES, ids=["g32", "g16", "gbf16"])
def test_adam_all_paths(gdt, pdt, hdt, mis):
    if mis == "p_half" and hdt is None:
        pytest.skip("no p_half to offset")
    ops = _ops()
    numels = NUMELS + ([_big_numel()] if mis in ("none", "g") else [])
    work = [_adam_item(n, gdt, pdt, hdt, mis, True, seed=i + 17 * n, hp=_hyper(i)) for i, n in enumerate(numels)]
    before = _snapshot(work)
    zero_grad = mis in ("none", "m", "p_half")
    ops.fused_adam(work, grad_scale=torch.tensor(8.0, device="cuda"), zero_grad=zero_grad, ema_decay=0.999)
    # 1 / 8 is exact; the kernel divides 1.0 by the device scalar (2 ulp) and multiplies (1 rounding)
    check_adam(work, before, 1 / 8.0, 5 * E32, 0.999, zero_grad)


def test_adam_many_tensors_own_hyperparameters():
    """More than 24 tensors (two launches), each with its own lr, betas, eps, weight decay, step and bias correction;
    a host float scale."""
    ops = _ops()
    work = [_adam_item(NUMELS[i % 7] + i, DTYPES[i % 3], DTYPES[(i // 3) % 3], None, "none", i % 2 == 0, seed=i,
                       hp=_hyper(i)) for i in range(53)]
    before = _snapshot(work)
    ops.fused_adam(work, grad_scale=3.0, zero_grad=False, ema_decay=0.99)
    # inv_scale = fp32(1 / 3) (1 rounding), divided by 1.0 (2 ulp), the product (1 rounding)
    check_adam(work, before, 1 / 3.0, 6 * E32, 0.99, False)


@pytest.mark.parametrize("mis", ["none", "m"])
@pytest.mark.parametrize("zero_grad", [False, True])
@pytest.mark.parametrize("bad", [math.inf, -math.inf, math.nan, 0.0], ids=["inf", "-inf", "nan", "zero"])
def test_adam_overflow_skip(bad, zero_grad, mis):
    """A non-finite or zero device scale skips the update in every launch and on both paths: p, m, v, p_half and
    ema are bitwise unchanged, g is zeroed exactly when zero_grad is set.  A host float scale never skips."""
    ops = _ops()
    work = [_adam_item(NUMELS[i % 7] * (1 + i % 2), torch.float16, torch.float32, torch.bfloat16, mis, True, seed=i,
                       hp=_hyper(i)) for i in range(30)]
    for w in work:
        w["p_half"].copy_(w["p"])
    before = _snapshot(work)
    ops.fused_adam(work, grad_scale=torch.tensor(bad, device="cuda"), zero_grad=zero_grad, stochastic_rounding=True,
                   ema_decay=0.9)
    for w, b in zip(work, before):
        for k in ("p", "m", "v", "p_half", "ema"):
            assert torch.equal(w[k], b[k]), k
        if zero_grad:
            assert bool((w["g"] == 0).all())
        else:
            assert torch.equal(w["g"], b["g"])
    if bad == math.inf:
        # the same value as a host float: 1 / inf = 0, the update runs on zero gradients
        before = _snapshot(work)
        ops.fused_adam(work, grad_scale=bad, zero_grad=False, ema_decay=0.9)
        check_adam(work, before, 0.0, 0.0, 0.9, False)
        assert not torch.equal(work[0]["m"], before[0]["m"])


# ---------------------------------------------------------------------------------------------------
# stochastic rounding
# ---------------------------------------------------------------------------------------------------
def _bf16_neighbours(x):
    """(lo, hi): the bf16 values at or below and above fp32 x (truncation of the low 16 bits, and the next value)."""
    bits = x.view(torch.int32)
    lo = (bits & ~0xFFFF).view(torch.float32)
    hi = ((bits & ~0xFFFF) + 0x10000).view(torch.float32)
    lo, hi = torch.where(x >= 0, lo, hi), torch.where(x >= 0, hi, lo)  # magnitude truncation: swap for negatives
    return lo, hi


def check_sr(x, out):
    """Every output is one of the two bf16 neighbours of x, exactly x when x is representable, and rounds up at the
    rate given by x's position between the neighbours (binomial bound)."""
    xf = x.float()
    o = out.float()
    exact = (xf.view(torch.int32) & 0xFFFF) == 0
    assert torch.equal(o[exact], xf[exact]), "representable values must be kept"
    lo, hi = _bf16_neighbours(xf)
    inexact = ~exact
    assert bool(((o == lo) | (o == hi))[inexact].all()), "outputs must be a bf16 neighbour"
    frac = ((xf.double() - lo.double()) / (hi.double() - lo.double()))[inexact]
    up = (o == hi)[inexact].double()
    n = up.numel()
    if n > 1000:
        var = (frac * (1 - frac)).sum().item()
        assert abs(up.sum().item() - frac.sum().item()) < 6 * math.sqrt(var) + 1, (up.mean().item(), frac.mean().item())


@pytest.mark.parametrize("n", [7, 8193, 1 << 20])
def test_fp32_to_bf16_sr(n):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(n)
    x = torch.randn(n, device="cuda", generator=g) * 10
    x[::11] = x[::11].to(torch.bfloat16).float()  # representable values
    x[5::13] = 1.0 + 2.0 ** -10  # 1/8 of the bf16 step above 1.0
    outs = []
    for mis in (False, True):
        xi = _buf(n, torch.float32, mis, x)
        oi = _buf(n, torch.bfloat16, mis, torch.zeros(n))
        torch.cuda.manual_seed(123)
        ops.fp32_to_bf16_sr(xi, oi)
        check_sr(xi, oi)
        outs.append(oi.clone())
    # the vector and the scalar path draw the same random bits for the same element index
    assert torch.equal(outs[0], outs[1])
    if n >= 1 << 20:
        q = x[5::13]
        o = outs[0][5::13].float()
        rate = (o > 1.0).double().mean().item()
        assert abs(rate - 1 / 8) < 6 * math.sqrt(1 / 8 * 7 / 8 / q.numel())


def test_adam_stochastic_rounding():
    """bf16 p_half by stochastic rounding of the fp32 master: each output a neighbour of the stored fp32 weight at the
    rate of its position; the vector and the scalar path (misaligned m) choose the same direction wherever their fp32
    weights are equal, across launches (> 24 tensors): the element index counts from the start of the whole list."""
    ops = _ops()
    results = []
    for mis in ("none", "m"):
        work = [_adam_item(n, torch.float32, torch.float32, torch.bfloat16, mis, False, seed=i, hp=_hyper(0))
                for i, n in enumerate([8193, 1 << 18, 9] * 9)]
        before = _snapshot(work)
        torch.cuda.manual_seed(99)
        ops.fused_adam(work, grad_scale=1.0, zero_grad=False, stochastic_rounding=True)
        check_adam(work, before, 1.0, 3 * E32, None, False, sr=True)
        results.append(work)
    for a, b in zip(*results):
        same = a["p"] == b["p"]
        assert same.double().mean().item() > 0.5
        assert torch.equal(a["p_half"][same], b["p_half"][same])


# ---------------------------------------------------------------------------------------------------
# L2 norm, scale, EMA
# ---------------------------------------------------------------------------------------------------
def _norm_list(seed, count, big):
    g = torch.Generator(device="cuda").manual_seed(seed)
    ts = []
    for i in range(count):
        n = NUMELS[i % 7] + (i // 7)
        if big and i == 3:
            n = _big_numel()
        ts.append(_buf(n, DTYPES[i % 3], i % 4 == 1, torch.randn(n, device="cuda", generator=g) * (1 + i % 5)))
    return ts


def l2_chain(ts):
    """Longest chain of fp32 additions behind the norm: 32 fma per chunk a thread visits, the block and grid sums of
    the partials (fixed order), one addition per launch."""
    chunks = [sum(-(-t.numel() // CHUNK) for t in ts[i:i + 24]) for i in range(0, len(ts), 24)]
    grid = [min(c, 8 * _sms()) for c in chunks]
    per_cta = max(-(-c // gr) for c, gr in zip(chunks, grid))
    return 33 * per_cta + 16 + -(-max(grid) // 256) + 16 + len(chunks)


@pytest.mark.parametrize("big", [False, True])
@pytest.mark.parametrize("count", [5, 24, 61])
def test_l2norm(count, big):
    ops = _ops()
    ts = _norm_list(count + big, count, big)
    ref = math.sqrt(sum(t.double().pow(2).sum().item() for t in ts))
    got = ops.multi_tensor_l2norm(ts)
    # each square is summed with one rounding per addition; the square root halves the relative error
    bound = ref * (l2_chain(ts) * E32 / 2 + 2 * E32) + 1e-30
    assert abs(got.item() - ref) <= bound, (got.item(), ref, bound)
    # the ticket counter is back at zero: a second call is the same fixed-order sum
    assert torch.equal(ops.multi_tensor_l2norm(ts), got)


@pytest.mark.parametrize("bad", [math.inf, math.nan])
def test_l2norm_non_finite(bad):
    ops = _ops()
    ts = _norm_list(3, 30, False)
    ts[27][-1] = bad  # the second launch, a scalar tail
    got = ops.multi_tensor_l2norm(ts).item()
    assert (math.isinf(got) and got > 0) if bad == math.inf else math.isnan(got)
    ts[27][-1] = 0
    assert math.isfinite(ops.multi_tensor_l2norm(ts).item())


@pytest.mark.parametrize("device_scale", [False, True])
@pytest.mark.parametrize("big", [False, True])
def test_scale(big, device_scale):
    ops = _ops()
    ts = _norm_list(7 + big, 40, big)
    before = [t.clone() for t in ts]
    s = 0.37
    ops.multi_tensor_scale_(ts, torch.tensor(s, device="cuda") if device_scale else s)
    sf = _f32(s)
    for t, b in zip(ts, before):
        ref = b.double() * s
        comp = (3 * E32 + abs(sf - s) / s) * ref.abs() + FTZ
        _assert_within(t, ref, UNIT[t.dtype] * (ref.abs() + comp) + comp + _tiny(t.dtype), "scale")


@pytest.mark.parametrize("mis", ["none", "ema", "p"])
@pytest.mark.parametrize("n", [1, 7, 8, 9, 8193, 100003])
def test_ema_update(n, mis):
    """The vector path, its scalar tail, and the scalar path (either buffer misaligned)."""
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(n)
    e0 = torch.randn(n, device="cuda", generator=g)
    p = _buf(n, torch.float32, mis == "p", torch.randn(n, device="cuda", generator=g))
    ema = _buf(n, torch.float32, mis == "ema", e0)
    decay = 0.999
    ops.ema_update_(ema, p, decay)
    a = 1 - _f32(decay)  # the binding passes the decay as fp32; 1 - decay is then exact
    ref = e0.double() - a * (e0.double() - p.double())
    comp = 3 * E32 * (e0.double().abs() + a * (e0.double() - p.double()).abs()) + FTZ
    _assert_within(ema, ref, E32 * ref.abs() + comp, "ema")
