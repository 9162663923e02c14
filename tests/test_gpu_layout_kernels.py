"""Head relayout, pair relayout and embedding-gradient kernels against exact references on every launch path.

Shapes come from the launch plans (``head_permute_plan``, ``pair_plan``, ``embedding_plan``: the functions the
launchers run), so that every kernel runs one grid sweep, several, and a ragged last one.

These kernels move bits or round once, so the references are exact:
- ``split_heads`` / ``merge_heads``: a PyTorch view / permute, bitwise (NaN payloads and subnormals included).  The
  scaled query slice is bitwise ``(x.float() * float32(scale)).to(dtype)`` with the flush to zero of the fast-math
  build emulated: fp32 operands and products below 2^-126 become signed zeros (fp16 values never get there);
- pair transpose: bitwise ``permute().contiguous()``;
- pair tail: bitwise the 16-bit PyTorch ops of ``pair_tail``'s fallback.  The kernel's ``__hsub2`` / ``__hadd2``
  round once, PyTorch rounds through fp32 first, which is innocuous for one addition.  NaN payloads may differ, so
  the NaN masks are compared and the bits everywhere else;
- embedding gradient, scatter path: within one 16-bit ulp plus the fp32 error of its sum of fp64 ``index_add_``; a
  vocabulary row with a single contribution is that row of dy, bitwise;
- embedding gradient, deterministic sorted path: bitwise a float32 loop over each row's contributions in ascending
  original order.
"""
import contextlib

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

F32, F16, BF16 = torch.float32, torch.float16, torch.bfloat16
ALL = [F32, F16, BF16]
HALF = [F16, BF16]
BITS = {F32: torch.int32, F16: torch.int16, BF16: torch.int16}
FTZ = 2.0 ** -126
E32 = 2.0 ** -24
NEG_INF = float("-inf")

# NaNs with payloads (quiet and signalling), +-inf, +-0, the smallest and largest subnormal, the largest finite and
# the smallest normal value, as bit patterns
SPECIAL_BITS = {
    F32: [0x7FC00001, 0xFFC12345, 0x7F800001, 0x7F800000, 0xFF800000, 0x0, 0x80000000, 0x00000001, 0x807FFFFF,
          0x7F7FFFFF, 0x00800000],
    F16: [0x7E01, 0xFE55, 0x7C01, 0x7C00, 0xFC00, 0x0, 0x8000, 0x0001, 0x83FF, 0x7BFF, 0x0400],
    BF16: [0x7FC1, 0xFF85, 0x7F81, 0x7F80, 0xFF80, 0x0, 0x8000, 0x0001, 0x807F, 0x7F7F, 0x0080],
}


def _native():
    from unicore import ops

    assert ops.USE_NATIVE, "native kernels must be active on the GPU box"
    return ops.native()


def _ops():
    from unicore import ops

    assert ops.USE_NATIVE, "native kernels must be active on the GPU box"
    return ops


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _signed(v, bits):
    return v - (1 << bits) if v >= 1 << (bits - 1) else v


def special_values(shape, dtype, g, tiny=True):
    """Random normals of `dtype` with every eighth element a special value (NaN payloads, infinities, signed zeros,
    subnormals, extremes) and, with `tiny`, every eighth another one near 2^-126, where the scaled slice flushes."""
    n = 1
    for s in shape:
        n *= s
    x = torch.randn(n, device="cuda", generator=g).to(dtype)
    bits = x.view(BITS[dtype])
    width = 32 if dtype == F32 else 16
    sp = torch.tensor([_signed(v, width) for v in SPECIAL_BITS[dtype]], dtype=BITS[dtype], device="cuda")
    pos = torch.randperm(n, device="cuda", generator=g)
    k = n // 8
    bits[pos[:k]] = sp[torch.randint(0, sp.numel(), (k,), device="cuda", generator=g)]
    if tiny:
        small = (torch.rand(k, device="cuda", generator=g) - 0.5) * (16 * FTZ)
        x[pos[k:2 * k]] = small.to(dtype)
    return x.view(shape)


def assert_exact(got, want, what):
    """Bitwise equal, NaN payloads included."""
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape, got.dtype, want.dtype)
    bad = got.view(BITS[got.dtype]) != want.view(BITS[want.dtype])
    if bad.any():
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError("{}: {} elements differ, first at {}: got {!r}, want {!r}".format(
            what, int(bad.sum()), i, got[i].item(), want[i].item()))


def assert_bits(got, want, what):
    """NaN at the same places, bitwise equal everywhere else."""
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, want.shape, got.dtype, want.dtype)
    nan = torch.isnan(got)
    assert torch.equal(nan, torch.isnan(want)), "{}: NaN at other places ({} vs {})".format(
        what, int(nan.sum()), int(torch.isnan(want).sum()))
    bad = (got.view(BITS[got.dtype]) != want.view(BITS[want.dtype])) & ~nan
    if bad.any():
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError("{}: {} elements differ, first at {}: got {!r}, want {!r}".format(
            what, int(bad.sum()), i, got[i].item(), want[i].item()))


def _ragged(plan):
    return plan["items"] % plan["items_per_sweep"] != 0


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


# ---------------------------------------------------------------------------------------------------
# split_heads / merge_heads
# ---------------------------------------------------------------------------------------------------
# one 16-byte vector per head (fp32 D = 4, fp16 D = 8), an odd count (fp16 D = 24: 3, fp32 D = 12: 3), two (bf16)
HEAD_CASES = [(F32, 4), (F32, 12), (F16, 8), (F16, 24), (BF16, 16)]
HEAD_IDS = ["fp32-D4", "fp32-D12", "fp16-D8", "fp16-D24", "bf16-D16"]
HEAD_B, HEAD_H = 2, 3
SCALE = 0.3  # not a power of two: the product rounds


def scaled_ref(x, scale):
    """x * float32(scale) in fp32, rounded once to x's dtype, as the kernel computes slice 0.  The build runs with
    --use_fast_math, so fp32 operands and products below 2^-126 are signed zeros there (fp32 and bf16 inputs reach that
    range; fp16 values and their products with SCALE do not)."""
    xf = x.float()
    xf = torch.where(xf.abs() < FTZ, xf * 0, xf)
    y = xf * torch.tensor(scale, dtype=F32, device=x.device)
    y = torch.where(y.abs() < FTZ, y * 0, y)
    return y.to(x.dtype)


def check_split(outs, x, T, H, scale, what):
    B, L, W = x.shape
    ref = x.view(B, L, T, H, W // (T * H)).permute(2, 0, 3, 1, 4)
    assert len(outs) == T
    for t, o in enumerate(outs):
        assert o.shape == ref[t].shape and o.is_contiguous(), (what, t)
        if t == 0 and scale != 1.0:
            assert_bits(o, scaled_ref(ref[0], scale), "{} slice 0 scaled".format(what))
        else:
            assert_exact(o, ref[t], "{} slice {}".format(what, t))


def check_merge(out, heads, scale, what):
    """`heads`: T tensors [B, H, L, D] or None (reads as zeros)."""
    ref = next(h for h in heads if h is not None)
    B, H, L, D = ref.shape
    T = len(heads)
    assert out.shape == (B, L, T * H * D) and out.is_contiguous()
    got = out.view(B, L, T, H, D)
    for t, h in enumerate(heads):
        want = torch.zeros_like(ref) if h is None else h
        if t == 0 and scale != 1.0:
            assert_bits(got[:, :, 0], scaled_ref(want, scale).permute(0, 2, 1, 3), "{} slice 0 scaled".format(what))
        else:
            assert_exact(got[:, :, t], want.permute(0, 2, 1, 3), "{} slice {}".format(what, t))


def head_multi_shape(dtype):
    """(B, L, T, H, D) with which split / merge run three grid sweeps or more, the last one ragged; L is odd."""
    nat = _native()
    L, T, H, D = 257, 3, 8, (12 if dtype == F32 else 24)
    one = nat.head_permute_plan(1, L, T, H, D, dtype)["items"]
    sweep = _sms() * 16 * 256
    B = -(-5 * sweep // (2 * one))
    while not _ragged(nat.head_permute_plan(B, L, T, H, D, dtype)):
        B += 1
    return B, L, T, H, D


@pytest.mark.parametrize("L", [1, 7, 16])
@pytest.mark.parametrize("T", [1, 2, 3, 4])
@pytest.mark.parametrize("dtype,D", HEAD_CASES, ids=HEAD_IDS)
def test_head_permute_bindings(dtype, D, T, L):
    """split_heads and merge_heads, scale 1 and SCALE; merge_heads with an absent slice in every position."""
    nat = _native()
    B, H = HEAD_B, HEAD_H
    x = special_values((B, L, T * H * D), dtype, _gen(100 * T + L + D))
    for scale in (1.0, SCALE):
        outs = nat.split_heads(x, T, H, scale)
        check_split(outs, x, T, H, scale, "split_heads(scale={})".format(scale))
        heads = [o.clone() for o in outs]
        for absent in [None] + (list(range(T)) if T > 1 else []):
            hs = [None if t == absent else heads[t] for t in range(T)]
            check_merge(nat.merge_heads(hs, scale), hs, scale, "merge_heads(scale={}, absent={})".format(scale, absent))


@pytest.mark.parametrize("dtype,D", HEAD_CASES, ids=HEAD_IDS)
def test_head_permute_autograd(dtype, D):
    """ops.split_heads with each output in turn unused (its gradient reads as zero), and ops.merge_heads."""
    ops = _ops()
    B, L, T, H = 2, 9, 3, HEAD_H
    g = _gen(7 + D)
    x = special_values((B, L, T * H * D), dtype, g)
    grads = [special_values((B, H, L, D), dtype, g) for _ in range(T)]
    for unused in range(T):
        xr = x.clone().requires_grad_(True)
        outs = ops.split_heads(xr, T, H, SCALE)
        check_split([o.detach() for o in outs], x, T, H, SCALE, "ops.split_heads")
        used = [t for t in range(T) if t != unused]
        torch.autograd.backward([outs[t] for t in used], [grads[t] for t in used])
        check_merge(xr.grad, [None if t == unused else grads[t] for t in range(T)], SCALE,
                    "split_heads backward (slice {} unused)".format(unused))
    hs = [h.clone().requires_grad_(True) for h in grads]
    m = ops.merge_heads(*hs, scale0=SCALE)
    check_merge(m.detach(), grads, SCALE, "ops.merge_heads")
    gm = special_values(m.shape, dtype, g)
    m.backward(gm)
    check_split([h.grad for h in hs], gm, T, H, SCALE, "merge_heads backward")


@pytest.mark.parametrize("dtype", ALL)
def test_head_permute_several_sweeps(dtype):
    nat = _native()
    B, L, T, H, D = head_multi_shape(dtype)
    plan = nat.head_permute_plan(B, L, T, H, D, dtype)
    assert plan["sweeps"] >= 3 and _ragged(plan), plan
    x = special_values((B, L, T * H * D), dtype, _gen(31))
    outs = nat.split_heads(x, T, H, SCALE)
    check_split(outs, x, T, H, SCALE, "split_heads")
    hs = [outs[0], None, outs[2]]
    check_merge(nat.merge_heads(hs, SCALE), hs, SCALE, "merge_heads")


# ---------------------------------------------------------------------------------------------------
# pair transpose and pair tail
# ---------------------------------------------------------------------------------------------------
# (B, H, Lq, Lk): H = 8 is one vector per tile row; Lq != Lk; Lk % 8 != 0 with Lq * Lk % 8 == 0 (transpose only)
TRANSPOSE_SHAPES = [(2, 8, 4, 6), (3, 64, 3, 8), (2, 8, 7, 16), (1, 64, 16, 12), (2, 16, 10, 4)]
TAIL_SHAPES = [(2, 8, 3, 8), (3, 64, 5, 16), (2, 16, 8, 24)]


def pair_multi_shape():
    """(B, H, Lq, Lk) with which the pair kernels run three grid sweeps or more, the last one ragged."""
    nat = _native()
    H, Lq, Lk = 64, 96, 128
    sweep = _sms() * 8 * 256
    one = nat.pair_plan(1, H, Lq * Lk)["items"]
    B = -(-5 * sweep // (2 * one))
    while not _ragged(nat.pair_plan(B, H, Lq * Lk)):
        B += 1
    return B, H, Lq, Lk


def _pair_shape(shape):
    return pair_multi_shape() if shape == "multi" else shape


@pytest.mark.parametrize("shape", TRANSPOSE_SHAPES + ["multi"], ids=str)
@pytest.mark.parametrize("dtype", HALF)
def test_pair_transpose(dtype, shape):
    nat, ops = _native(), _ops()
    B, H, Lq, Lk = _pair_shape(shape)
    g = _gen(B + H + Lq + Lk)
    x = special_values((B, H, Lq, Lk), dtype, g, tiny=False)
    y = nat.pair_transpose(x, True)
    assert_exact(y, x.permute(0, 2, 3, 1).contiguous(), "heads -> pair")
    assert_exact(nat.pair_transpose(y, False), x, "pair -> heads")
    # the autograd ops: each direction is the other's backward
    xr = x.clone().requires_grad_(True)
    yo = ops.heads_to_pair(xr)
    assert_exact(yo.detach(), y, "ops.heads_to_pair")
    gy = special_values(y.shape, dtype, g, tiny=False)
    yo.backward(gy)
    assert_exact(xr.grad, gy.permute(0, 3, 1, 2).contiguous(), "heads_to_pair backward")
    yr = y.clone().requires_grad_(True)
    xo = ops.pair_to_heads(yr)
    assert_exact(xo.detach(), x, "ops.pair_to_heads")
    xo.backward(x)
    assert_exact(yr.grad, y, "pair_to_heads backward")


def tail_inputs(B, H, Lq, Lk, dtype, both_inf, g):
    """z, z0 [B, H, Lq, Lk] and the padding [B, Lk]: padded key columns are -inf in z (what unimol.py feeds) or in both
    z and z0 (the reference Uni-Mol's layout: z - z0 is NaN there until the pad clears it); stray -inf, +inf, NaN and
    -0.0 sit in live positions of both."""
    pad = torch.zeros(B, Lk, dtype=torch.bool, device="cuda")
    pad[0, Lk - 3:] = True
    pad[-1, 1] = True
    z0 = torch.randn(B, H, Lq, Lk, device="cuda", generator=g).to(dtype)
    z = (z0.float() + torch.randn(B, H, Lq, Lk, device="cuda", generator=g)).to(dtype)
    cols = pad[:, None, None, :]
    z = z.masked_fill(cols, NEG_INF)
    if both_inf:
        z0 = z0.masked_fill(cols, NEG_INF)
    for t, vals in ((z, (NEG_INF, float("inf"), float("nan"), -0.0)), (z0, (float("inf"), float("nan"), -0.0))):
        flat = t.view(-1)
        pick = torch.randint(0, flat.numel(), (64 * len(vals),), device="cuda", generator=g)
        pick = pick[~pad[pick // (H * Lq * Lk), pick % Lk]][:4 * len(vals)]  # live positions only
        for i, v in enumerate(vals):
            flat[pick[4 * i:4 * i + 4]] = v
    return z, z0, pad


def tail_fwd_ref(z, z0, pad):
    delta = z - z0
    if pad is not None:
        delta = delta.masked_fill(pad[:, None, None, :], 0)
    pair = z.masked_fill(z == NEG_INF, 0)
    return pair.permute(0, 2, 3, 1).contiguous(), delta.permute(0, 2, 3, 1).contiguous()


def tail_bwd_ref(d_pair, d_delta, z, pad):
    """dz = (d_pair masked where z == -inf) + (d_delta masked at pad), dz0 = -(d_delta masked at pad); an absent
    gradient reads as zeros."""
    zero = torch.zeros_like(z)
    gp = zero if d_pair is None else d_pair.permute(0, 3, 1, 2).masked_fill(z == NEG_INF, 0)
    gd = zero if d_delta is None else d_delta.permute(0, 3, 1, 2)
    if pad is not None:
        gd = gd.masked_fill(pad[:, None, None, :], 0)
    return (gp + gd).contiguous(), (-gd).contiguous()


@pytest.mark.parametrize("mask", ["none", "bool", "uint8"])
@pytest.mark.parametrize("both_inf", [False, True], ids=["inf_in_z", "inf_in_both"])
@pytest.mark.parametrize("shape", TAIL_SHAPES + ["multi"], ids=str)
@pytest.mark.parametrize("dtype", HALF)
def test_pair_tail(dtype, shape, both_inf, mask):
    nat = _native()
    B, H, Lq, Lk = _pair_shape(shape)
    g = _gen(B * H + Lq + Lk + both_inf)
    z, z0, pad = tail_inputs(B, H, Lq, Lk, dtype, both_inf, g)
    if mask == "none":
        key_pad, pad = None, None
    elif mask == "bool":
        key_pad = pad
    else:  # any nonzero byte pads
        key_pad = pad.to(torch.uint8) * torch.randint(1, 256, pad.shape, device="cuda", generator=g).to(torch.uint8)
    pair, delta = nat.pair_tail_fwd(z, z0, key_pad)
    pair_r, delta_r = tail_fwd_ref(z, z0, pad)
    assert_bits(pair, pair_r, "pair")
    assert_bits(delta, delta_r, "delta")
    d_pair = special_values(pair.shape, dtype, g, tiny=False)
    d_delta = special_values(pair.shape, dtype, g, tiny=False)
    for dp, dd, what in ((d_pair, d_delta, "both"), (d_pair, None, "d_pair only"), (None, d_delta, "d_delta only")):
        dz, dz0 = nat.pair_tail_bwd(dp, dd, z, key_pad)
        dz_r, dz0_r = tail_bwd_ref(dp, dd, z, pad)
        assert_bits(dz, dz_r, "dz ({})".format(what))
        assert_bits(dz0, dz0_r, "dz0 ({})".format(what))


@pytest.mark.parametrize("dtype", HALF)
def test_pair_tail_op(dtype):
    """ops.pair_tail forward and backward are the bindings', with both outputs used and with one unused."""
    ops, nat = _ops(), _native()
    g = _gen(5)
    z, z0, pad = tail_inputs(2, 16, 8, 24, dtype, False, g)
    pair_b, delta_b = nat.pair_tail_fwd(z, z0, pad)
    gp = special_values(pair_b.shape, dtype, g, tiny=False)
    gd = special_values(pair_b.shape, dtype, g, tiny=False)
    for grads in ((gp, gd), (gp, None)):
        zr, z0r = z.clone().requires_grad_(True), z0.clone().requires_grad_(True)
        pair, delta = ops.pair_tail(zr, z0r, pad)
        assert_exact(pair.detach(), pair_b, "pair")
        assert_exact(delta.detach(), delta_b, "delta")
        outs = [o for o, gr in zip((pair, delta), grads) if gr is not None]
        torch.autograd.backward(outs, [gr for gr in grads if gr is not None])
        dz, dz0 = nat.pair_tail_bwd(grads[0], grads[1], z, pad)
        assert_exact(zr.grad, dz, "dz")
        assert_exact(z0r.grad, dz0, "dz0")


def _misaligned(t):
    """A contiguous copy of `t` that starts one element past a 16-byte boundary."""
    buf = torch.empty(t.numel() + 16, dtype=t.dtype, device=t.device)
    v = buf[1:1 + t.numel()].view(t.shape)
    v.copy_(t)
    assert v.is_contiguous() and v.data_ptr() % 16 != 0
    return v


def _run_op(fn, inputs, grads):
    """fn(*inputs) with autograd; returns the outputs and the input gradients."""
    leaves = [t if t.dtype == torch.bool else t.detach().requires_grad_(True) for t in inputs]  # (views stay views)
    outs = fn(*leaves)
    outs = outs if isinstance(outs, (tuple, list)) else (outs,)
    torch.autograd.backward(list(outs), list(grads))
    return [o.detach() for o in outs] + [t.grad for t in leaves if t.dtype != torch.bool]


@pytest.mark.parametrize("dtype", HALF)
def test_layout_ops_copy_misaligned_views(dtype):
    """Contiguous views one element off a 16-byte boundary (inputs, the key padding mask and incoming gradients) are
    copied once by the layout ops: the results equal those of the same values in aligned buffers."""
    ops = _ops()
    g = _gen(9)
    B, H, L, D = 2, 8, 16, 8
    z, z0, pad = tail_inputs(B, H, L, L, dtype, False, g)
    pair_g = [special_values((B, L, L, H), dtype, g, tiny=False) for _ in range(2)]
    x = special_values((B, H, L, L), dtype, g, tiny=False)
    qkv = special_values((B, L, 3 * H * D), dtype, g, tiny=False)
    head_g = [special_values((B, H, L, D), dtype, g, tiny=False) for _ in range(3)]
    cases = {
        "pair_tail": (lambda a, b, m: ops.pair_tail(a, b, m), [z, z0, pad], pair_g),
        "heads_to_pair": (ops.heads_to_pair, [x], pair_g[:1]),
        "pair_to_heads": (ops.pair_to_heads, [pair_g[1]], [x]),
        "split_heads": (lambda t: ops.split_heads(t, 3, H, SCALE), [qkv], head_g),
        "merge_heads": (lambda a, b, c: ops.merge_heads(a, b, c, scale0=SCALE), head_g, [qkv]),
    }
    for name, (fn, inputs, grads) in cases.items():
        want = _run_op(fn, inputs, grads)
        got = _run_op(fn, [_misaligned(t) for t in inputs], [_misaligned(t) for t in grads])
        assert len(got) == len(want)
        for i, (a, b) in enumerate(zip(got, want)):
            assert_exact(a, b, "{} result {}".format(name, i))


# ---------------------------------------------------------------------------------------------------
# embedding gradient
# ---------------------------------------------------------------------------------------------------
MANT = {F16: 10, BF16: 7}
EMIN = {F16: -14, BF16: -126}


@contextlib.contextmanager
def deterministic():
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def ulp16(ref, dtype):
    """Spacing of `dtype` at |ref| (fp64), subnormals included."""
    _, e = torch.frexp(ref.abs())  # |ref| = m 2^e, 0.5 <= m < 1
    e = torch.where(ref == 0, torch.full_like(e, EMIN[dtype]), torch.clamp(e - 1, min=EMIN[dtype]))
    return torch.exp2((e - MANT[dtype]).double())


def emb_reference(dy, tok, vocab, pad):
    """fp64 sums, absolute sums and contribution counts per vocabulary row; ids < 0, >= vocab or == pad skipped."""
    cols = dy.shape[-1]
    dy2, tok1 = dy.reshape(-1, cols), tok.reshape(-1)
    keep = (tok1 >= 0) & (tok1 < vocab) & (tok1 != pad)
    ref = torch.zeros(vocab, cols, dtype=torch.float64, device="cuda")
    absum = torch.zeros_like(ref)
    step = max(1, (1 << 21) // cols)
    for r0 in range(0, tok1.numel(), step):
        s = slice(r0, r0 + step)
        k = keep[s]
        rows = dy2[s][k].double()
        ref.index_add_(0, tok1[s][k], rows)
        absum.index_add_(0, tok1[s][k], rows.abs())
    n = torch.bincount(tok1[keep], minlength=vocab)
    return ref, absum, n


def check_emb_grad(got, dy, tok, pad, base, accumulate, dtype, what, singles=False):
    """Scatter path: |got - ref| <= ulp16(|ref|) + (n + 1) 2^-24 A per element, A = |base| + sum |dy_i| over the n
    contributions; bf16 adds n 2^-126 (red.add.f32 flushes subnormal terms).  Rows without a contribution keep base.
    With `singles` (and without accumulate), a row with one contribution is that row of dy, bitwise."""
    vocab = got.shape[0]
    ref, absum, n = emb_reference(dy, tok, vocab, pad)
    nd = n.double()[:, None]
    b = base.double()
    if accumulate:
        ref, absum = ref + b, absum + b.abs()
    bound = ulp16(ref, dtype) + (nd + 1) * E32 * absum + (nd * FTZ if dtype == BF16 else 0.0)
    err = (got.double() - ref).abs()
    touched = n > 0
    bad = ~(err <= bound) & touched[:, None]
    if bad.any():
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError("{}: {} elements out of bound, first at {} (n = {}): got {}, want {} +- {}".format(
            what, int(bad.sum()), i, int(n[i[0]]), got[i].item(), ref[i].item(), bound[i].item()))
    assert_exact(got[~touched], base[~touched], "{}: rows without a contribution".format(what))
    if singles and not accumulate:
        single = (n == 1).nonzero().view(-1)
        assert single.numel() > 0
        tok1 = tok.reshape(-1)
        src = torch.full((vocab,), -1, dtype=torch.long, device="cuda")
        keep = (tok1 >= 0) & (tok1 < vocab) & (tok1 != pad)
        src[tok1[keep]] = keep.nonzero().view(-1)
        assert_exact(got[single], dy.reshape(-1, dy.shape[-1])[src[single]], "{}: single contributions".format(what))


def emb_multi(kind, vocab=None):
    """Rows (kind "rows") or a vocabulary (kind "vocab") for which the scatter or the finalize kernel runs two grid
    sweeps or more with a ragged last one."""
    nat = _native()
    sweep = _sms() * 16 * 8
    n = 2 * sweep + sweep // 2 + 1
    key = "scatter" if kind == "rows" else "finalize"
    plan = nat.embedding_plan(n, vocab or 1000) if kind == "rows" else nat.embedding_plan(1000, n)
    assert plan[key]["items_per_sweep"] == sweep and _ragged(plan[key]), plan
    return n


# name: (cols, rows, vocab).  A lane moves one vector for 8 and 264 columns past the first 256 (33 vectors), a
# BERT-base batch; "multi" rows / vocabulary take several scatter / finalize sweeps
EMB_CASES = {
    "w8-multi_rows-multi_vocab": (8, "multi", "multi"),
    "w264-multi_rows": (264, "multi", 1000),
    "w768-bert": (768, 32 * 512, 30522),
    "w1032-multi_rows": (1032, "multi", 3000),
}


def emb_case(name):
    cols, rows, vocab = EMB_CASES[name]
    vocab = emb_multi("vocab") if vocab == "multi" else vocab
    rows = emb_multi("rows", vocab) if rows == "multi" else rows
    return cols, rows, vocab


def emb_tokens(rows, vocab, g, pad=None, out_of_range=True):
    """Random ids with a token that takes a third of the rows, the padding id, ids outside [0, vocab) and eight ids
    that occur exactly once."""
    tok = torch.randint(0, vocab - 8, (rows,), device="cuda", generator=g)
    tok[::3] = 5
    if pad is not None:
        tok[1::11] = pad
    if out_of_range:
        tok[2::13] = -1
        tok[4::17] = -7
        tok[7::19] = vocab
        tok[8::23] = vocab + 5
    pos = torch.randperm(rows, device="cuda", generator=g)
    pos = pos[pos % 3 != 0][:8]
    tok[pos] = torch.arange(vocab - 8, vocab, device="cuda")
    return tok


@pytest.mark.parametrize("case", sorted(EMB_CASES))
@pytest.mark.parametrize("dtype", HALF)
def test_embedding_scatter(dtype, case):
    """The binding: padding id none (-1) or 2, accumulate off (over a random gradient: untouched rows keep it) and
    on; out-of-range and negative ids are skipped; scratch and flags are all zero again after every call."""
    nat = _native()
    cols, rows, vocab = emb_case(case)
    g = _gen(cols + rows)
    scratch = torch.zeros(vocab * cols, device="cuda")
    touched = torch.zeros(vocab, dtype=torch.uint8, device="cuda")
    dy = torch.randn(rows, cols, device="cuda", generator=g).to(dtype)
    for pad in (-1, 2):
        tok = emb_tokens(rows, vocab, g, pad=pad if pad >= 0 else None)
        for accumulate in (False, True):
            base = torch.randn(vocab, cols, device="cuda", generator=g).to(dtype)
            grad = base.clone()
            nat.embedding_bwd(dy, tok, pad, scratch, touched, grad, accumulate)
            check_emb_grad(grad, dy, tok, pad, base, accumulate, dtype,
                           "{} pad={} accumulate={}".format(case, pad, accumulate), singles=True)
            assert not scratch.any() and not touched.any(), "scratch / flags left dirty"


@pytest.mark.parametrize("deterministic_mode", [False, True], ids=["scatter", "sorted"])
@pytest.mark.parametrize("padding_idx", [None, 3, -1, -2])
@pytest.mark.parametrize("dtype", HALF)
def test_embedding_op_padding(dtype, padding_idx, deterministic_mode):
    """ops.embedding follows F.embedding: a negative padding_idx counts from the end (-1 is the last row), and the
    padding row gets no gradient."""
    ops = _ops()
    V, C = 50, 264
    g = _gen(V + (padding_idx or 0))
    w = torch.randn(V, C, device="cuda", generator=g).to(dtype).requires_grad_(True)
    tok = torch.randint(0, V, (40, 100), device="cuda", generator=g)
    tok.view(-1)[:V] = torch.arange(V, device="cuda")  # every row is used, the last ones included
    dy = torch.randn(40, 100, C, device="cuda", generator=g).to(dtype)
    ctx = deterministic() if deterministic_mode else contextlib.nullcontext()
    with ctx:
        y = ops.embedding(tok, w, padding_idx)
        assert_exact(y.detach(), F.embedding(tok, w.detach(), padding_idx), "forward")
        y.backward(dy)
    wr = w.detach().double().requires_grad_(True)
    F.embedding(tok, wr, padding_idx).backward(dy.double())
    p = -1 if padding_idx is None else padding_idx % V
    if p >= 0:
        assert not wr.grad[p].any() and not w.grad[p].any(), "the padding row got a gradient"
    check_emb_grad(w.grad, dy, tok, p, torch.zeros_like(w.grad), False, dtype, "ops.embedding")
    assert torch.allclose(emb_reference(dy, tok, V, p)[0], wr.grad, rtol=1e-12, atol=1e-12)  # same rows skipped


def sorted_loop_ref(dy, tok, vocab, pad, base, accumulate):
    """The deterministic kernel's sum: for each vocabulary row, fp32 from 0 over its rows in ascending original order,
    then (accumulate) + base in fp32, rounded once; rows without a contribution and the padding row keep base."""
    cols = dy.shape[-1]
    ids, perm = torch.sort(tok, stable=True)
    rank = torch.arange(ids.numel(), device="cuda") - torch.searchsorted(ids, ids)
    live = (ids >= 0) & (ids < vocab) & (ids != pad)
    acc = torch.zeros(vocab, cols, dtype=torch.float32, device="cuda")
    for k in range(int(rank.max()) + 1):
        sel = live & (rank == k)  # at most one row of every run: each vocabulary row gets one fp32 addition
        acc[ids[sel]] += dy[perm[sel]].float()
    has = torch.zeros(vocab, dtype=torch.bool, device="cuda")
    has[ids[live]] = True
    out = ((acc + base.float()) if accumulate else acc).to(base.dtype)
    return torch.where(has[:, None], out, base)


@pytest.mark.parametrize("accumulate", [False, True], ids=["write", "accumulate"])
@pytest.mark.parametrize("dtype", HALF)
def test_embedding_sorted(dtype, accumulate):
    """Deterministic mode: a vocabulary of more rows than the sorted kernel's grid, 1032 columns (129 vectors: a thread
    takes two), runs of every length 0 - 7 (the kernel adds four rows at a time, then the rest one by one), the padding
    row and out-of-range ids."""
    nat = _native()
    V, C, pad = 30522, 1032, 7
    g = _gen(accumulate + 2)
    ids = torch.arange(V, device="cuda")
    counts = torch.where((ids < 2048) | (ids % 13 == 0), ids % 8, torch.zeros_like(ids))
    counts[pad] = 5
    tok = torch.cat([torch.repeat_interleave(ids, counts), torch.tensor([-1, -3, V, V + 5], device="cuda")])
    tok = tok[torch.randperm(tok.numel(), device="cuda", generator=g)]
    plan = _native().embedding_plan(tok.numel(), V)["sorted"]
    assert plan["sweeps"] >= 2 and _ragged(plan), plan
    dy = torch.randn(tok.numel(), C, device="cuda", generator=g).to(dtype)
    base = torch.randn(V, C, device="cuda", generator=g).to(dtype)
    scratch = torch.zeros(V * C, device="cuda")
    touched = torch.zeros(V, dtype=torch.uint8, device="cuda")
    grad = base.clone()
    with deterministic():
        nat.embedding_bwd(dy, tok, pad, scratch, touched, grad, accumulate)
    assert_exact(grad, sorted_loop_ref(dy, tok, V, pad, base, accumulate), "sorted embedding gradient")


@pytest.mark.parametrize("first", [True, False], ids=["embedding_first", "after_a_2_element_parameter"])
def test_embedding_gradient_into_the_arena(first):
    """Flat arenas pad parameters to 2 elements, so an embedding behind a 2-element parameter has a 4-byte aligned
    gradient view: its gradient then arrives through AccumulateGrad (the post-accumulate hook fires, on_written does
    not).  An aligned view is written in place by the kernel and reported through on_written."""
    from unicore.optim.fp16_optimizer import flatten_parameters
    from unicore_b200.ops import grad_sink

    ops = _ops()
    V, C, dtype = 100, 64, F16
    g = _gen(first + 11)
    emb = torch.nn.Parameter(torch.randn(V, C, device="cuda", generator=g).to(dtype))
    small = torch.nn.Parameter(torch.randn(2, device="cuda", generator=g).to(dtype))
    params = [emb, small] if first else [small, emb]
    flatten_parameters(params)
    arena_view = emb.grad.data_ptr()
    assert (arena_view % 16 == 0) == first
    written, hooked = [], []
    grad_sink.enable(params, on_written=written.append)
    handle = emb.register_post_accumulate_grad_hook(hooked.append)
    tok = torch.randint(0, V, (8, 33), device="cuda", generator=g)
    dy = torch.randn(8, 33, C, device="cuda", generator=g).to(dtype)
    try:
        ops.embedding(tok, emb, 1).backward(dy)
    finally:
        handle.remove()
        grad_sink.disable(params)
    wr = emb.detach().double().requires_grad_(True)
    F.embedding(tok, wr, 1).backward(dy.double())
    check_emb_grad(emb.grad, dy, tok, 1, torch.zeros_like(emb.grad), False, dtype, "arena gradient")
    assert torch.allclose(emb_reference(dy, tok, V, 1)[0], wr.grad, rtol=1e-12, atol=1e-12)
    assert emb.grad.data_ptr() == arena_view, "the gradient left the arena"
    if first:
        assert written == [emb] and emb._ub_pending == 0
    else:
        assert written == [] and len(hooked) == 1 and hooked[0] is emb


# ---------------------------------------------------------------------------------------------------
# launch plans
# ---------------------------------------------------------------------------------------------------
def test_dispatch_coverage():
    """The plans mirror the launch geometry, and the shapes above run one sweep, several and a ragged last one of
    every kernel; nothing is launched."""
    nat = _native()
    sms = _sms()
    for dtype, D in HEAD_CASES:
        for T in (1, 4):
            p = nat.head_permute_plan(HEAD_B, 7, T, HEAD_H, D, dtype)
            dv = D * torch.finfo(dtype).bits // 128
            assert p["items"] == HEAD_B * T * 4 * HEAD_H * 2 * dv, p
            assert p["grid"] == -(-p["items"] // 256) and p["sweeps"] == 1, p
    for dtype in ALL:
        B, L, T, H, D = head_multi_shape(dtype)
        p = nat.head_permute_plan(B, L, T, H, D, dtype)
        assert p["grid"] == sms * 16 and p["items_per_sweep"] == sms * 16 * 256 and p["sweeps"] >= 3 and _ragged(p)
    for B, H, Lq, Lk in TRANSPOSE_SHAPES + TAIL_SHAPES:
        p = nat.pair_plan(B, H, Lq * Lk)
        assert p["items"] == B * (H // 8) * (Lq * Lk // 8) and p["sweeps"] == 1, p
    B, H, Lq, Lk = pair_multi_shape()
    p = nat.pair_plan(B, H, Lq * Lk)
    assert p["grid"] == sms * 8 and p["sweeps"] >= 3 and _ragged(p), p
    seen = {"scatter": set(), "finalize": set()}
    for name in EMB_CASES:
        cols, rows, vocab = emb_case(name)
        p = nat.embedding_plan(rows, vocab)
        for k in seen:
            assert p[k]["grid"] == min(-(-p[k]["items"] // 8), sms * 16), p
            seen[k].add((p[k]["sweeps"] > 1, _ragged(p[k])))
    # one whole sweep, and several with a ragged last one, of both kernels
    assert seen["scatter"] >= {(False, False), (True, True)}, seen
    assert seen["finalize"] >= {(False, False), (True, True)}, seen
    p = nat.embedding_plan(14000, 30522)["sorted"]
    assert p["grid"] == sms * 16 and p["sweeps"] >= 2 and _ragged(p), p
    assert nat.embedding_plan(0, 30522)["sorted"]["grid"] == 0  # no rows: nothing is launched
