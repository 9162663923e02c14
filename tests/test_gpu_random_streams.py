"""Every dropout and stochastic-rounding kernel outside fused attention against a host Philox, bit for bit.

The kernels promise that each random decision is a pure function of ``(seed, offset, element index)``: one
Philox4x32 block per 8 consecutive elements, keyed by the pair the launch reserved from the CUDA generator.  Backward
rebuilds the keep mask from that promise instead of storing it.  A mask read back from a kernel's output only shows
that forward and backward agree with each other; a stream that is wrong in a self-consistent way (a counter taken
from the row within a grid sweep, the two 16-bit halves of a word swapped, two tensors sharing counters) keeps the
rate and the consistency.  Here the bits come from a numpy Philox instead, and every output is held to float64
computed with those bits:

* ``softmax_dropout_fwd / _bwd`` and the logits mode (``csrc/attn/softmax_dropout.cu``): 14-bit rule, element
  ``(r, c)`` of the flattened ``[rows, K]`` input at index ``r * K + c``, on every launch case of ``softmax_plan``;
* ``bias_dropout_add_ln_fwd / _bwd`` (``csrc/norm/norm.cu``): 16-bit rule, index ``row * cols + col``, on every
  generation ``norm_plan`` picks for the fused op;
* ``fp32_to_bf16_sr`` and ``multi_tensor_adam`` with stochastic rounding (``csrc/optim/multi_tensor.cu``).

The one scaling rule: a kept element is scaled by ``1 / P(keep)`` of the quantised threshold the kernel compares
against, ``16384 / (16384 - t14)`` for the 14-bit rule and ``65536 / (65536 - t16)`` for the 16-bit one, so that
E[dropout(x)] = x for the rate the kernels actually draw.

The host generator is checked on the CPU against the published Philox4x32-10 known-answer vectors before any GPU
test relies on it.
"""
import math

import numpy as np
import pytest
import torch

E32 = 2.0 ** -24
UNIT = {torch.float32: 2.0 ** -24, torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}  # unit roundoff
FTZ = 2.0 ** -126  # the kernels' fp32 arithmetic flushes subnormal results to zero
EPS = 1e-5

# ---------------------------------------------------------------------------------------------------
# host Philox4x32 (csrc/common.cuh: philox4x32<R>)
# ---------------------------------------------------------------------------------------------------
M32 = 0xFFFFFFFF
PHILOX_M0, PHILOX_M1 = 0xD2511F53, 0xCD9E8D57
PHILOX_W0, PHILOX_W1 = 0x9E3779B9, 0xBB67AE85


def philox4x32(seed, offset, ctr, rounds):
    """Philox4x32-`rounds` of the uint64 counters `ctr` (array): words (c0, c1, c2, c3) = (ctr lo, ctr hi, offset lo,
    offset hi), key (k0, k1) = (seed lo, seed hi), as ``philox4x32<R>`` lays them out.  Returns uint32 [n, 4]."""
    ctr = np.asarray(ctr, dtype=np.uint64)
    m32 = np.uint64(M32)
    c0, c1 = ctr & m32, ctr >> np.uint64(32)
    c2 = np.full_like(c0, offset & M32)
    c3 = np.full_like(c0, (offset >> 32) & M32)
    k0, k1 = seed & M32, (seed >> 32) & M32
    for _ in range(rounds):
        p0 = c0 * np.uint64(PHILOX_M0)  # both factors < 2^32: the 64-bit product is exact
        p1 = c2 * np.uint64(PHILOX_M1)
        c0, c1, c2, c3 = ((p1 >> np.uint64(32)) ^ c1 ^ np.uint64(k0), p1 & m32,
                          (p0 >> np.uint64(32)) ^ c3 ^ np.uint64(k1), p0 & m32)
        k0, k1 = (k0 + PHILOX_W0) & M32, (k1 + PHILOX_W1) & M32
    return np.stack([c0, c1, c2, c3], axis=1).astype(np.uint32)


def philox4x32_scalar(seed, offset, ctr, rounds):
    """The round of ``philox4x32<R>`` transcribed line by line in plain Python (the vectorised version's check)."""
    k0, k1 = seed & M32, seed >> 32
    c0, c1, c2, c3 = ctr & M32, ctr >> 32, offset & M32, offset >> 32
    for _ in range(rounds):
        hi0, lo0 = (PHILOX_M0 * c0) >> 32, (PHILOX_M0 * c0) & M32
        hi1, lo1 = (PHILOX_M1 * c2) >> 32, (PHILOX_M1 * c2) & M32
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
        k0, k1 = (k0 + PHILOX_W0) & M32, (k1 + PHILOX_W1) & M32
    return c0, c1, c2, c3


def _lanes16(words):
    """The 8 16-bit lanes of each block in element order: word i gives element 2i (low half) and 2i+1 (high half)."""
    lanes = np.empty((words.shape[0], 8), dtype=np.uint32)
    lanes[:, 0::2] = words & 0xFFFF
    lanes[:, 1::2] = words >> 16
    return lanes


def dropout_thresh14(p):
    """``dropout_thresh14``: round(p * 16384) in fp32, clamped to [0, 16383]."""
    t = np.float32(p) * np.float32(16384) + np.float32(0.5)
    return 0 if t <= 0 else (16383 if t >= 16383 else int(t))


def dropout_thresh16(p):
    """``dropout_thresh16``: round(p * 65536) in fp32, at most 65535."""
    t = np.float32(p) * np.float32(65536) + np.float32(0.5)
    return 65535 if t >= 65535 else int(t)


def keep_scale14(p):
    return 1.0 if p <= 0 else 16384.0 / (16384 - dropout_thresh14(p))


def keep_scale16(p):
    return 1.0 if p <= 0 else 65536.0 / (65536 - dropout_thresh16(p))


def keep_mask16(seed, offset, n, p):
    """``dropout_keep8`` over elements 0..n-1: keep iff the element's 16-bit lane >= dropout_thresh16(p)."""
    if p <= 0:
        return np.ones(n, dtype=bool)
    words = philox4x32(seed, offset, np.arange((n + 7) // 8, dtype=np.uint64), 7)
    return (_lanes16(words) >= dropout_thresh16(p)).reshape(-1)[:n]


def keep_mask14(seed, offset, n, p):
    """``dropout_keep8_14`` / ``dropout_lane_masks8`` over elements 0..n-1: keep iff the lane's low 14 bits >=
    dropout_thresh14(p) (an integer compare; the vector form compares the same bits as fp16 patterns)."""
    if p <= 0:
        return np.ones(n, dtype=bool)
    words = philox4x32(seed, offset, np.arange((n + 7) // 8, dtype=np.uint64), 7)
    return ((_lanes16(words) & 0x3FFF) >= dropout_thresh14(p)).reshape(-1)[:n]


def sr_random16(seed, offset, index):
    """The 16 random bits of global element `index` (array) in ``multi_tensor.cu``: Philox4x32-10 of counter
    index >> 3, word (index & 7) >> 1, low half for even index and high half for odd."""
    index = np.asarray(index, dtype=np.uint64)
    words = philox4x32(seed, offset, index >> np.uint64(3), 10)
    w = words[np.arange(index.size), ((index & np.uint64(7)) >> np.uint64(1)).astype(np.int64)]
    return np.where((index & np.uint64(1)) == 1, w >> 16, w & 0xFFFF).astype(np.uint32)


def bf16_sr_bits(x_fp32, rnd16):
    """``bf16_sr_bits``: add the random bits to the fp32 pattern (inf / nan untouched) and keep the high half."""
    bits = np.ascontiguousarray(x_fp32, dtype=np.float32).view(np.uint32)
    finite = (bits & 0x7F800000) != 0x7F800000
    bits = np.where(finite, bits + rnd16.astype(np.uint32), bits)  # uint32 wrap-around as on the device
    return (bits >> 16).astype(np.uint16)


def rng_pair():
    """The (seed, offset) the next ``philox_reserve`` hands out: the CUDA generator's state is the seed and the
    Philox offset, two little-endian 64-bit words."""
    st = torch.cuda.get_rng_state().numpy()
    assert st.size == 16, st.size
    return int.from_bytes(st[:8].tobytes(), "little"), int.from_bytes(st[8:].tobytes(), "little")


def _u64(v):
    return v & 0xFFFFFFFFFFFFFFFF  # the bindings return the uint64 pair as int64


# ---------------------------------------------------------------------------------------------------
# CPU: the host generator against the published vectors and its own scalar transcription
# ---------------------------------------------------------------------------------------------------
# Random123 kat_vectors, philox4x32 with 10 rounds: (counter c0..c3, key k0 k1) -> output
PHILOX_KAT = [
    ((0x00000000, 0x00000000, 0x00000000, 0x00000000), (0x00000000, 0x00000000),
     (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF), (0xFFFFFFFF, 0xFFFFFFFF),
     (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
]


@pytest.mark.parametrize("case", range(len(PHILOX_KAT)))
def test_host_philox_known_answers(case):
    (c0, c1, c2, c3), (k0, k1), want = PHILOX_KAT[case]
    seed, offset, ctr = k0 | (k1 << 32), c2 | (c3 << 32), c0 | (c1 << 32)
    assert philox4x32_scalar(seed, offset, ctr, 10) == want
    assert tuple(int(w) for w in philox4x32(seed, offset, [ctr], 10)[0]) == want


def test_host_philox_vectorised_equals_scalar():
    rng = np.random.default_rng(0)
    for rounds in (7, 10):
        seed, offset = int(rng.integers(0, 2 ** 63)) * 2 + 1, int(rng.integers(0, 2 ** 63)) * 2
        ctr = np.concatenate([np.arange(40, dtype=np.uint64), rng.integers(0, 2 ** 63, 24, dtype=np.uint64) * 2 + 1])
        got = philox4x32(seed, offset, ctr, rounds)
        for i, c in enumerate(ctr.tolist()):
            assert tuple(int(w) for w in got[i]) == philox4x32_scalar(seed, offset, c, rounds)


def test_host_rules():
    """Thresholds, lane order and the rounding rule on hand-made bits."""
    assert dropout_thresh14(1e-6) == 0 and keep_scale14(1e-6) == 1.0
    assert dropout_thresh16(1e-6) == 0 and keep_scale16(1e-6) == 1.0
    assert dropout_thresh14(0.5) == 8192 and dropout_thresh16(0.5) == 32768
    assert dropout_thresh14(1 - 2 ** -14) == 16383 and dropout_thresh14(2.0) == 16383
    assert dropout_thresh16(0.01) == 655 and dropout_thresh14(0.01) == 164
    words = np.array([[0x0000FFFF, 0xFFFF0000, 0x40003FFF, 0x7FFF8000]], dtype=np.uint32)
    lanes = _lanes16(words)[0].tolist()
    assert lanes == [0xFFFF, 0x0000, 0x0000, 0xFFFF, 0x3FFF, 0x4000, 0x8000, 0x7FFF]
    assert ((_lanes16(words) & 0x3FFF) >= 1).tolist() == [[True, False, False, True, True, False, False, True]]
    x = np.array([1.0, 1.0, -1.5, np.inf, -np.inf, np.nan, 3.0e38, 1e-40], dtype=np.float32)
    r = np.array([0xFFFF, 0, 0x8000, 0xFFFF, 0xFFFF, 0xFFFF, 0xFFFF, 0xFFFF], dtype=np.uint32)
    out = bf16_sr_bits(x, r)
    xb = x.view(np.uint32)
    assert out[0] == 0x3F80 and out[1] == 0x3F80  # 1.0 is exact: no random bits move it
    assert out[2] == 0xBFC0  # -1.5 is exact as well
    assert (out[3:6] == (xb[3:6] >> 16)).all()  # inf / nan untouched
    assert out[6] == (xb[6] + 0xFFFF) >> 16
    assert out[7] == (xb[7] + 0xFFFF) >> 16
    # the SR lanes: element i takes word (i & 7) >> 1 of block i >> 3, low half for even i
    idx = np.arange(16, dtype=np.uint64)
    blocks = philox4x32(5, 9, np.arange(2, dtype=np.uint64), 10)
    assert (sr_random16(5, 9, idx) == _lanes16(blocks).reshape(-1)).all()


# ---------------------------------------------------------------------------------------------------
# shared GPU helpers
# ---------------------------------------------------------------------------------------------------
def _nat():
    from unicore import ops

    assert ops.USE_NATIVE, "native kernels must be active on the GPU box"
    return ops.native()


def _epv(dtype):
    return 16 // torch.empty((), dtype=dtype).element_size()


def _tiny(dtype):
    return torch.finfo(dtype).tiny * UNIT[dtype]


def _bits(t):
    return t.view({2: torch.int16, 4: torch.int32}[t.element_size()])


def _within(got, ref, bound, what):
    err = (got.double() - ref).abs()
    bad = err > bound
    if bad.any():
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError("{}: {} elements out of bound, first at {}: got {}, want {} +- {}".format(
            what, int(bad.sum()), i, got[i].item(), ref[i].item(), bound[i].item()))


def _assert_dropped_are_zero(out, keep, what):
    """Dropped elements are stored as +0 (all bits clear), whatever the value would have been."""
    bad = (_bits(out) != 0) & ~keep
    assert not bad.any(), "{}: {} dropped elements are not zero, first at {}".format(
        what, int(bad.sum()), bad.nonzero()[0].tolist())


def _assert_independent(a, b, q, what):
    """Two keep masks of the same length drawn from independent streams agree at (1-q)^2 + q^2, q the drawn rate."""
    n = a.numel()
    want = (1 - q) ** 2 + q ** 2
    got = (a == b).double().mean().item()
    assert abs(got - want) < 6 * math.sqrt(want * (1 - want) / n) + 1e-12, (what, got, want)


# ---------------------------------------------------------------------------------------------------
# softmax + dropout
# ---------------------------------------------------------------------------------------------------
# Row lengths in 16-byte vectors that reach every launch case of softmax_plan: threads per row < 32 (8), = 32 with
# 1..4 vectors per thread (32, 64, 96, 128), 64-128 threads (160, 256), 256 threads (640, 1024).  The scalar kernels
# take K = 99 (not a multiple of the vector width) and K one vector past the longest vector row.
SM_NVECS = [8, 32, 64, 96, 128, 160, 256, 640, 1024]
SM_SCALAR = [99, "long"]
SM_Q = 16


def _sm_k(k, dtype):
    epv = _epv(dtype)
    if k == "long":
        return 1024 * epv + epv
    return k * epv if k in SM_NVECS else k


def _sm_case(plan):
    if not plan["vec"]:
        return ("scalar",)
    t = plan["tpr"]
    return ("vec", "<32" if t < 32 else ("32" if t == 32 else ("256" if t == 256 else "64-128")), plan["vpt"])


def _sm_rows(K, dtype):
    """Rows (a multiple of SM_Q) with which every CTA of both kernels runs 3 sweeps or more and the last sweep is
    ragged.  Rows past the longest vector row take 17 * SM_Q rows: the scalar kernels' later sweeps run at K = 99."""
    nat = _nat()
    if K > 1024 * _epv(dtype):
        return SM_Q * 17
    sweep = max(nat.softmax_plan(1 << 40, K, dtype, True, k)["rows_per_sweep"] for k in ("fwd", "bwd"))
    rows = -(-(3 * sweep + sweep // 2 + 1) // SM_Q) * SM_Q
    for k in ("fwd", "bwd"):
        pl = nat.softmax_plan(rows, K, dtype, True, k)
        while rows % pl["rows_per_sweep"] == 0:
            rows += SM_Q
        assert pl["sweeps"] >= 4, pl
    return rows


def _sm_inputs(rows, K, dtype, seed):
    """x [B, Q, K] with every 7th column far below the rest (its probability underflows in the output type, fp32
    included: the kernels flush), a [B, 1, K] mask and a [1, Q, K] bias, dy and the logits-mode addend."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    B = rows // SM_Q
    x = torch.randn(B, SM_Q, K, device="cuda", generator=g) * 2
    x[..., 3::7] = -30.0 if dtype == torch.float16 else -110.0
    mask = torch.where(torch.rand(B, 1, K, device="cuda", generator=g) < 0.1, -4.0, 0.0)
    bias = torch.randn(1, SM_Q, K, device="cuda", generator=g)
    dy = torch.randn(B, SM_Q, K, device="cuda", generator=g)
    addend = torch.randn(B, SM_Q, K, device="cuda", generator=g)
    return [t.to(dtype) for t in (x, mask, bias, dy, addend)]


def _run_softmax(nat, mode, x, mask, bias, dy, addend, p):
    """Forward and backward through the bindings; returns (out, probs-or-None, z-or-None, dx, seed, offset)."""
    if mode == "logits":
        out, z, lse, seed, off = nat.softmax_dropout_logits_fwd(x, mask, bias, p, True)
        dx = nat.softmax_dropout_logits_bwd(dy, z, lse, addend, p, seed, off)
        return out, None, z, dx, _u64(seed), _u64(off)
    xin = x.clone() if mode == "in_place" else x  # the plain mode leaves x untouched (and keeps its alignment)
    out, probs, seed, off = nat.softmax_dropout_fwd(xin, mask, bias, p, True, mode == "in_place")
    assert (probs.data_ptr() == xin.data_ptr()) == (mode == "in_place")
    dx = nat.softmax_dropout_bwd(dy, probs, p, seed, off)
    return out, probs, None, dx, _u64(seed), _u64(off)


def _check_softmax(mode, x, mask, bias, dy, addend, p, res):
    """Output zero exactly where the host mask drops, forward and backward equal to fp64 with the host mask (every
    element, underflowed probabilities included).  Returns the host keep mask [rows, K]."""
    out, probs, z, dx, seed, off = res
    dtype = x.dtype
    B, Q, K = x.shape
    rows = B * Q
    u, tiny = UNIT[dtype], _tiny(dtype)
    keep = torch.from_numpy(keep_mask14(seed, off, rows * K, p)).to("cuda").view(rows, K)
    _assert_dropped_are_zero(out.view(rows, K), keep, "out")
    scale = keep_scale14(p)
    if z is None:
        zd = (x.double() + mask.double() + bias.double()).view(rows, K)
        zabs = (x.double().abs() + mask.double().abs() + bias.double().abs()).view(rows, K)  # the kernel's fp32 sum
    else:
        zr = x.double() + mask.double() + bias.double()
        zin = x.double().abs() + mask.double().abs() + bias.double().abs()  # two fp32 additions, one rounding to T
        _within(z, zr, u * zr.abs() + 2 * E32 * zin, "logits")
        zd = z.double().view(rows, K)
        zabs = zd.abs()
    yr = torch.softmax(zd, -1)
    comp = yr * E32 * (2 * (zd - zd.max(-1, keepdim=True).values).abs() + 4 * zabs + 80)
    if probs is not None:
        _within(probs.view(rows, K), yr, u * (yr + comp) + comp + tiny + FTZ, "probs")
    ref = yr * keep * scale
    _within(out.view(rows, K), ref, u * (ref + comp * scale) + comp * scale + tiny + FTZ * scale, "out")
    # backward: dx = y * (d - sum(d * y)) (+ addend), d = keep * dy * scale; y the stored probabilities, or (logits
    # mode) softmax(z) rebuilt from z and the row log-sum-exp
    if z is None:
        yd, e_y = probs.double().view(rows, K), 0.0
    else:
        yd = yr
        lse = torch.logsumexp(zd, -1, keepdim=True)
        e_y = yd * (u + E32 * (2 * (zd - lse).abs() + 2 * lse.abs() + 80)) + tiny + FTZ
    d = dy.double().view(rows, K) * keep * scale
    dot = (d * yd).sum(-1, keepdim=True)
    ref = yd * (d - dot)
    comp = ((d - dot).abs() * e_y + yd * ((d.abs() * e_y).sum(-1, keepdim=True)
                                           + 72 * E32 * (d * yd).abs().sum(-1, keepdim=True))
            + 4 * E32 * ((d * yd).abs() + (yd * dot).abs()))
    if z is not None:
        ref = ref + addend.double().view(rows, K)
        comp = comp + 2 * E32 * addend.double().view(rows, K).abs()
    _within(dx.view(rows, K), ref, u * (ref.abs() + comp) + comp + tiny + FTZ, "dx")
    return keep


def _softmax_ps(k, dtype):
    """p = 0.1 everywhere; p = 0.01 and 0.05 where the fp16 compare of dropout_lane_masks8 runs (vector kernels of
    16-bit types), whose thresholds (164, 819 < 1024) and many random lanes are fp16 subnormal patterns."""
    return (0.1, 0.01, 0.05) if k in SM_NVECS and _epv(dtype) == 8 else (0.1,)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32])
@pytest.mark.parametrize("k", SM_NVECS + SM_SCALAR)
@pytest.mark.parametrize("mode", ["plain", "in_place", "logits"])
def test_softmax_dropout_stream(mode, k, dtype):
    nat = _nat()
    K = _sm_k(k, dtype)
    rows = _sm_rows(K, dtype)
    for kind in ("fwd", "bwd"):
        case = _sm_case(nat.softmax_plan(rows, K, dtype, True, kind))
        assert case[0] == ("vec" if k in SM_NVECS else "scalar"), (kind, case)
    x, mask, bias, dy, addend = _sm_inputs(rows, K, dtype, 100 + K)
    for p in _softmax_ps(k, dtype):
        want = rng_pair()
        res = _run_softmax(nat, mode, x, mask, bias, dy, addend, p)
        assert res[4:] == want  # the decoded generator state is the pair the binding reserved
        _check_softmax(mode, x, mask, bias, dy, addend, p, res)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16, torch.float32])
@pytest.mark.parametrize("k", [8, 256, 99])
@pytest.mark.parametrize("p", [1e-6, 0.5, 1 - 2 ** -14])
def test_softmax_dropout_stream_extreme_p(p, k, dtype):
    """A threshold that rounds to 0 (nothing dropped, scale exactly 1), one half, and the largest threshold, 16383 (the
    bindings take any p; from here on the 14-bit rule keeps 1 element in 16384 and scales it by 16384)."""
    nat = _nat()
    K = _sm_k(k, dtype)
    rows = _sm_rows(K, dtype)
    x, mask, bias, dy, addend = _sm_inputs(rows, K, dtype, 200 + K)
    for mode in ("plain", "logits"):
        res = _run_softmax(nat, mode, x, mask, bias, dy, addend, p)
        keep = _check_softmax(mode, x, mask, bias, dy, addend, p, res)
        if p < 1e-5:
            assert bool(keep.all())


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("p", [0.01, 0.05, 0.2])
def test_softmax_vector_and_scalar_forms_agree_at_small_p(p, dtype):
    """The fp16-pattern compare (vector kernels, aligned) and the integer compare (scalar kernels, a view at an odd
    element offset) give the host mask at small p, where thresholds and lanes are fp16 subnormal patterns."""
    nat = _nat()
    K = 128 * _epv(dtype)
    rows = _sm_rows(K, dtype)
    x, mask, bias, dy, addend = _sm_inputs(rows, K, dtype, 300)
    xm, dym = (torch.empty(t.numel() + 1, device="cuda", dtype=dtype)[1:].view_as(t).copy_(t) for t in (x, dy))
    assert xm.data_ptr() % 16 != 0 and dym.data_ptr() % 16 != 0
    for kind in ("fwd", "bwd"):
        assert nat.softmax_plan(rows, K, dtype, True, kind)["vec"] and not nat.softmax_plan(rows, K, dtype, False, kind)["vec"]
    keeps = []
    for xi, di in ((x, dy), (xm, dym)):
        torch.cuda.manual_seed(9)
        res = _run_softmax(nat, "plain", xi, mask, bias, di, addend, p)
        keeps.append(_check_softmax("plain", x, mask, bias, dy, addend, p, res))
    assert torch.equal(keeps[0], keeps[1])


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_softmax_dropout_op_broadcast_index(dtype):
    """``ops.softmax_dropout`` on a 4-D input with a [B, 1, 1, K] mask and a [1, H, Q, K] bias: the keep bit of element
    (b, h, q, c) is that of its index in the flattened input, not of the broadcast operands."""
    from unicore import ops

    B, H, Q, K = 3, 4, 40, 96
    g = torch.Generator(device="cuda").manual_seed(17)
    x = (torch.randn(B, H, Q, K, device="cuda", generator=g) * 2).to(dtype).requires_grad_(True)
    mask = torch.zeros(B, 1, 1, K, device="cuda", dtype=dtype)
    mask[0, ..., 80:] = float("-inf")
    mask[2, ..., :5] = float("-inf")
    bias = torch.randn(1, H, Q, K, device="cuda", generator=g).to(dtype).requires_grad_(True)
    dy = torch.randn(B, H, Q, K, device="cuda", generator=g).to(dtype)
    p = 0.3
    x0 = x.detach().clone()  # the op works in place: x ends up holding the probabilities
    seed, off = rng_pair()
    out = ops.softmax_dropout(x, p, True, mask=mask, bias=bias)
    out.backward(dy)
    keep = torch.from_numpy(keep_mask14(seed, off, x.numel(), p)).to("cuda").view(B, H, Q, K)
    _assert_dropped_are_zero(out.detach().reshape(-1, K), keep.view(-1, K), "out")
    zd = x0.double() + mask.double() + bias.detach().double()
    zabs = (x0.double().abs() + bias.detach().double().abs()).expand_as(zd)
    yr = torch.softmax(zd, -1)
    zmax = zd.max(-1, keepdim=True).values
    # fp32 error of the probabilities (exponent argument, exp2, row sum), as in the kernel-level checks above
    comp = yr * E32 * (2 * (zd - zmax).nan_to_num(0, 0, 0).abs() + 4 * zabs + 80)
    scale = keep_scale14(p)
    u, tiny = UNIT[dtype], _tiny(dtype)
    ref = yr * keep * scale
    _within(out.detach(), ref, u * (ref + comp * scale) + comp * scale + tiny + FTZ * scale, "out")
    # backward reads the stored probabilities: yr within one rounding and the fp32 error above (e_y)
    e_y = u * (yr + comp) + comp + tiny + FTZ
    d = dy.double() * keep * scale
    dot = (d * yr).sum(-1, keepdim=True)
    dx = yr * (d - dot)
    comp = ((d - dot).abs() * e_y + yr * ((d.abs() * e_y).sum(-1, keepdim=True)
                                          + 72 * E32 * (d * yr).abs().sum(-1, keepdim=True))
            + 4 * E32 * ((d * yr).abs() + (yr * dot).abs()))
    dbound = u * (dx.abs() + comp) + comp + tiny + FTZ
    _within(x.grad, dx, dbound, "dx")
    _within(bias.grad[0], dx.sum(0), dbound.sum(0) + u * dx.sum(0).abs(), "dbias")


# ---------------------------------------------------------------------------------------------------
# bias + dropout + residual + LayerNorm
# ---------------------------------------------------------------------------------------------------
# Widths in 16-byte vectors that reach every generation and dispatch case norm_plan picks for the fused op: the v3 / v2
# widths and the v1 widths of the norm tests, and a ragged v1 width none of them has (777).
NORM_V1_NVECS = [500, 520, 1024]
NORM_NVECS = [1, 2, 3, 4, 5, 8, 9, 16, 25, 32, 40, 64, 65, 96, 125, 128, 129, 192, 250, 256, 384] + NORM_V1_NVECS + [777]


def _norm_case(plan):
    if plan["gen"] == 3:
        return (3, plan["vpl"], plan["lpr"], plan["full"])
    if plan["gen"] == 2:
        return (2, plan["groups"], plan["full"])
    if plan["gen"] == 1:
        return (1, plan["vpt"], plan["tpr"])
    return None


def _norm_rows(cols, dtype):
    """Rows past one grid sweep of the fused forward and the backward, with a ragged last sweep."""
    nat = _nat()
    sweep = max(nat.norm_plan(1 << 30, cols, dtype, k)["rows_per_sweep"] for k in ("fused", "bwd"))
    rows = sweep + sweep // 2 + 1
    for k in ("fused", "bwd"):
        pl = nat.norm_plan(rows, cols, dtype, k)
        assert pl["tiles_max"] >= 2 and rows % pl["rows_per_sweep"] != 0, (k, pl)
    return rows


def _norm_inputs(rows, cols, dtype, seed):
    """x, residual, bias, gamma, beta, dy; every 5th row of dy is tiny, so that dsum underflows in the output type
    there while dx = dsum * scale (computed from fp32) may not."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(rows, cols, device="cuda", generator=g)
    res = torch.randn(rows, cols, device="cuda", generator=g)
    bias = torch.randn(cols, device="cuda", generator=g)
    w = torch.randn(cols, device="cuda", generator=g) * 0.5 + 1
    b = torch.randn(cols, device="cuda", generator=g)
    dy = torch.randn(rows, cols, device="cuda", generator=g)
    dy[::5] *= 2.0 ** -20 if dtype == torch.float16 else 2.0 ** -125
    return [t.to(dtype) for t in (x, res, bias, w, b, dy)]


def _run_norm(nat, x, res, bias, w, b, dy, p):
    y, mean, rstd, summed, seed, off = nat.bias_dropout_add_ln_fwd(x, bias, res, w, b, p, EPS)
    dsum, dx, dg, db, dbias = nat.bias_dropout_add_ln_bwd(dy, summed, mean, rstd, w, p, seed, off, True, None, None, None)
    return y, mean, rstd, summed, dsum, dx, dbias, _u64(seed), _u64(off)


def _check_norm(x, res, bias, w, b, dy, p, out, chain):
    """summed, y, dsum, dx and dbias against fp64 with the host mask; dx is +0 exactly where the host mask drops, also
    where dsum underflowed.  Returns the host keep mask."""
    y, mean, rstd, summed, dsum, dx, dbias, seed, off = out
    dtype = x.dtype
    rows, cols = x.shape
    u, tiny = UNIT[dtype], _tiny(dtype)
    keep = torch.from_numpy(keep_mask16(seed, off, rows * cols, p)).to("cuda").view(rows, cols)
    scale = keep_scale16(p)
    # summed = residual + keep * (x + bias) * scale: a few fp32 roundings, one rounding to the output type
    h = keep * (x.double() + bias.double()) * scale
    ref = res.double() + h
    comp = 4 * E32 * (res.double().abs() + h.abs())
    _within(summed, ref, u * (ref.abs() + comp) + comp + tiny, "summed")
    # LayerNorm of the stored sum: exact statistics against the saved ones, y against the saved ones
    sd = summed.double()
    mu = sd.mean(-1, keepdim=True)
    rs = torch.rsqrt(((sd - mu) ** 2).mean(-1, keepdim=True) + EPS)
    _within(mean[:, None], mu, 64 * E32 * sd.abs().mean(-1, keepdim=True), "mean")
    dmu = (mean[:, None].double() - mu).abs()
    _within(rstd[:, None], rs, rs * (72 * E32 + (dmu * rs) ** 2), "rstd")
    wd, bd = w.double(), b.double()
    xh = (sd - mean[:, None].double()) * rstd[:, None].double()
    yr = xh * wd + bd
    comp = 4 * E32 * ((xh * wd).abs() + bd.abs() + (sd.abs() * rstd[:, None].double()) * wd.abs())
    _within(y, yr, u * (yr.abs() + comp) + comp + tiny, "y")
    # backward from the saved statistics
    rsk = rstd[:, None].double()
    gy = dy.double() * wd
    m1 = gy.mean(-1, keepdim=True)
    m2 = (gy * xh).mean(-1, keepdim=True)
    dsr = rsk * (gy - m1 - xh * m2)
    comp = rsk * (4 * E32 * (gy.abs() + m1.abs() + (xh * m2).abs() + xh.abs() * m2.abs())
                  + 72 * E32 / cols * (gy.abs().sum(-1, keepdim=True) + xh.abs() * (gy * xh).abs().sum(-1, keepdim=True)))
    comp = comp + (1 + rsk * (4 + 2 * xh.abs())) * FTZ  # flushed fp32 products and results in the rows of tiny dy
    _within(dsum, dsr, u * (dsr.abs() + comp) + comp + tiny, "dsum")
    _assert_dropped_are_zero(dx, keep, "dx")
    dxr = dsr * keep * scale
    dxc = (comp + 2 * E32 * dsr.abs()) * scale
    dxb = u * (dxr.abs() + dxc) + dxc + tiny
    _within(dx, dxr, dxb, "dx")
    # dbias: fp32 column sums of dx (of the fp32 values at v3 / v2 widths, of the rounded dx at v1 widths)
    ref = dxr.sum(0)
    absum = dxr.abs().sum(0) + dxb.sum(0)
    comp = chain * E32 * absum + dxb.sum(0)
    _within(dbias, ref, u * (ref.abs() + comp) + comp + tiny, "dbias")
    return keep


def _norm_chain(nat, rows, cols, dtype):
    """Longest chain of fp32 additions behind a dbias column: the rows one loop unit visits plus the fixed-order sums
    across units (v3 / v2), or, at v1 widths, the column sum over all rows that runs after the norm kernel."""
    pl = nat.norm_plan(rows, cols, dtype, "bwd")
    return rows + 80 if pl["gen"] == 1 else pl["tiles_max"] * pl["tile_rows"] + 80


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("nvec", NORM_NVECS)
def test_bias_dropout_add_ln_stream(nvec, dtype):
    nat = _nat()
    cols = nvec * 8
    rows = _norm_rows(cols, dtype)
    fused, bwd = nat.norm_plan(rows, cols, dtype, "fused"), nat.norm_plan(rows, cols, dtype, "bwd")
    assert fused["gen"] == bwd["gen"] == (3 if nvec <= 128 else (2 if nvec <= 384 else 1)), (fused, bwd)
    x, res, bias, w, b, dy = _norm_inputs(rows, cols, dtype, 500 + nvec)
    chain = _norm_chain(nat, rows, cols, dtype)
    for p in (0.1, 0.5) if nvec in (5, 96, 192, 520) else (0.1,):
        want = rng_pair()
        out = _run_norm(nat, x, res, bias, w, b, dy, p)
        assert out[-2:] == want
        _check_norm(x, res, bias, w, b, dy, p, out, chain)


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("nvec", [5, 96, 192, 520])
@pytest.mark.parametrize("p", [1e-6, 0.999])
def test_bias_dropout_add_ln_stream_extreme_p(p, nvec, dtype):
    """A 16-bit threshold that rounds to 0 (nothing dropped, scale exactly 1) and p = 0.999 (scale 1000 keeps the
    scaled fp16 values finite), one width per generation and v3 dispatch shape."""
    nat = _nat()
    cols = nvec * 8
    rows = _norm_rows(cols, dtype)
    x, res, bias, w, b, dy = _norm_inputs(rows, cols, dtype, 600 + nvec)
    out = _run_norm(nat, x, res, bias, w, b, dy, p)
    keep = _check_norm(x, res, bias, w, b, dy, p, out, _norm_chain(nat, rows, cols, dtype))
    if p < 1e-5:
        assert bool(keep.all())


# ---------------------------------------------------------------------------------------------------
# stochastic rounding
# ---------------------------------------------------------------------------------------------------
def _sr_input(n, seed):
    """fp32 values with random low halves, both signs, subnormals, and a few infs and nans."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(n, device="cuda", generator=g) * torch.exp2(torch.randint(-20, 20, (n,), device="cuda", generator=g))
    x[::97] = float("inf")
    x[5::97] = float("-inf")
    x[11::97] = float("nan")
    x[17::97] *= 2.0 ** -130  # subnormal
    return x


def _sr_check(x, out, seed, off, what):
    want = bf16_sr_bits(x.cpu().numpy(), sr_random16(seed, off, np.arange(x.numel(), dtype=np.uint64)))
    got = out.view(torch.int16).cpu().numpy().view(np.uint16)
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, "{}: {} elements differ, first at {}".format(what, bad.size, bad[:4].tolist())
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("n", [7, 8193, (1 << 20) + 3])
@pytest.mark.parametrize("aligned", [True, False], ids=["vector", "scalar"])
def test_fp32_to_bf16_sr_stream(n, aligned):
    """Aligned buffers take the vector loop up to the last multiple of 8 and the scalar loop after it; a view at an
    odd element offset takes the scalar loop throughout.  The index is the element's position in the view."""
    nat = _nat()
    x = _sr_input(n, n)
    if not aligned:
        buf = torch.empty(n + 1, device="cuda")
        buf[1:].copy_(x)
        x = buf[1:]
        assert x.data_ptr() % 16 != 0
    out = torch.empty(n, device="cuda", dtype=torch.bfloat16)
    seed, off = rng_pair()
    nat.fp32_to_bf16_sr(x, out)
    _sr_check(x, out, seed, off, "fp32_to_bf16_sr")


def _adam_work(sizes, misaligned, seed):
    """fp32 masters with bf16 copies; `misaligned` items get a p_half view at an odd element offset, which sends the
    whole tensor through the kernel's scalar loop."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    work = []
    for i, n in enumerate(sizes):
        p = torch.randn(n, device="cuda", generator=g)
        half = torch.empty(n + 1, device="cuda", dtype=torch.bfloat16)
        work.append(dict(
            p=p, g=torch.randn(n, device="cuda", generator=g) * 1e-2, m=torch.rand(n, device="cuda", generator=g) * 1e-3,
            v=torch.rand(n, device="cuda", generator=g) * 1e-4, p_half=half[1:] if i in misaligned else half[:n],
            lr=1e-3 * (1 + i % 3), beta1=0.9, beta2=0.999, eps=1e-8, step=3 + i, bias_correction=True,
            weight_decay=0.01))
    return work


def _adam_elem_base(sizes):
    """The contract of ``multi_tensor_adam``'s ``elem_base``: tensor i's first element is Philox element index
    elem_base[i], the sum over the tensors before it in the call's list - across the launches of up to 24 tensors
    that one call makes - of their element counts rounded up to a multiple of 8.  Every tensor thus starts at a
    fresh counter (8 elements per counter), and no two tensors of one call share a counter."""
    base, out = 0, []
    for n in sizes:
        out.append(base)
        base += (n + 7) // 8 * 8
    return out


def _check_adam_sr(work, sizes, seed, off):
    bases = _adam_elem_base(sizes)
    spans = [(bb // 8, (bb + n + 7) // 8) for bb, n in zip(bases, sizes)]
    for (a0, a1), (b0, b1) in zip(spans, spans[1:]):
        assert a0 < a1 <= b0 < b1  # counter ranges of the tensors are disjoint
    halves = []
    for i, (w, n, bb) in enumerate(zip(work, sizes, bases)):
        master = w["p"].cpu().numpy()  # the fp32 master the kernel stored; the bf16 copy is its rounding
        want = bf16_sr_bits(master, sr_random16(seed, off, bb + np.arange(n, dtype=np.uint64)))
        got = w["p_half"].contiguous().view(torch.int16).cpu().numpy().view(np.uint16)
        bad = np.nonzero(got != want)[0]
        assert bad.size == 0, "tensor {} ({} elements, elem_base {}): {} differ, first at {}".format(
            i, n, bb, bad.size, bad[:4].tolist())
        halves.append(got)
    return halves


# 5 tensors of odd sizes: 8193 and 16397 span chunk boundaries (8192 elements) with a scalar tail of 1 and 5; 7 is
# all tail; 30011 crosses three chunks; 20001 has its bf16 copy misaligned (scalar loop throughout).  The long list
# adds 25 more so that one call makes two launches (24 tensors each at most) and elem_base carries over.
ADAM_SIZES = [8193, 7, 16397, 30011, 20001]
ADAM_MISALIGNED = {4}


@pytest.mark.gpu
@pytest.mark.parametrize("long_list", [False, True], ids=["one_launch", "two_launches"])
def test_adam_stochastic_rounding_stream(long_list):
    from unicore import ops

    sizes = ADAM_SIZES + ([9 + 2 * i for i in range(20)] + [8191, 12, 1, 24577, 5] if long_list else [])
    work = _adam_work(sizes, ADAM_MISALIGNED | ({27} if long_list else set()), 41)
    seed, off = rng_pair()
    ops.fused_adam(work, grad_scale=1.0, zero_grad=False, stochastic_rounding=True)
    _check_adam_sr(work, sizes, seed, off)


# ---------------------------------------------------------------------------------------------------
# between calls
# ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("op", ["softmax", "norm", "sr", "adam"])
def test_back_to_back_calls(op):
    """Two calls in a row reserve different (seed, offset) pairs (the same seed, offsets at least 4 apart: no Philox
    block (ctr, offset) is used twice), each equals the host stream for its own pair, and their random decisions
    agree at the rate of independent draws.  torch.cuda.manual_seed(s) before a call reproduces its bits."""
    nat = _nat()
    p = 0.5
    if op == "softmax":
        dtype, K = torch.float16, 64 * 8
        rows = _sm_rows(K, dtype)
        args = _sm_inputs(rows, K, dtype, 700)

        def call():
            res = _run_softmax(nat, "plain", *args, p)
            return res[4:], _check_softmax("plain", *args, p, res), res[0]
        q_drawn = dropout_thresh14(p) / 16384
    elif op == "norm":
        dtype, cols = torch.bfloat16, 96 * 8
        rows = _norm_rows(cols, dtype)
        args = _norm_inputs(rows, cols, dtype, 701)
        chain = _norm_chain(nat, rows, cols, dtype)

        def call():
            out = _run_norm(nat, *args, p)
            return out[-2:], _check_norm(*args, p, out, chain), out[3]
        q_drawn = dropout_thresh16(p) / 65536
    elif op == "sr":
        n = (1 << 20) + 3
        x = _sr_input(n, 702)

        def call():
            pair = rng_pair()
            out = torch.empty(n, device="cuda", dtype=torch.bfloat16)
            nat.fp32_to_bf16_sr(x, out)
            return pair, torch.from_numpy(_sr_check(x, out, *pair, "fp32_to_bf16_sr").astype(np.int32)), out
    else:
        from unicore import ops

        sizes = ADAM_SIZES
        state = _adam_work(sizes, ADAM_MISALIGNED, 703)

        def call():
            work = [dict(w, p=w["p"].clone(), m=w["m"].clone(), v=w["v"].clone()) for w in state]
            pair = rng_pair()
            ops.fused_adam(work, grad_scale=1.0, zero_grad=False, stochastic_rounding=True)
            halves = np.concatenate(_check_adam_sr(work, sizes, *pair))
            return pair, torch.from_numpy(halves.astype(np.int32)), torch.cat([w["p_half"] for w in work])

    (pa, ma, oa), (pb, mb, ob) = call(), call()
    assert pa[0] == pb[0] and pb[1] - pa[1] >= 4, (pa, pb)
    if op in ("softmax", "norm"):
        _assert_independent(ma.view(-1), mb.view(-1), q_drawn, op)
    else:
        # each element rounds up with probability f = (low 16 bits) / 65536 of its master: two independent draws agree
        # with probability f^2 + (1 - f)^2 (1 where the value is exact, inf or nan)
        if op == "adam":  # both calls start from the same masters and store the same update
            work = [dict(w, p=w["p"].clone(), m=w["m"].clone(), v=w["v"].clone()) for w in state]
            ops.fused_adam(work, grad_scale=1.0, zero_grad=False, stochastic_rounding=False)
            x = torch.cat([w["p"] for w in work])
        xb = x.cpu().numpy().view(np.uint32)
        f = np.where((xb & 0x7F800000) != 0x7F800000, (xb & 0xFFFF) / 65536.0, 0.0)
        q = f * f + (1 - f) * (1 - f)
        agree = (ma.numpy() == mb.numpy()).sum()
        sd = math.sqrt((q * (1 - q)).sum())
        assert abs(agree - q.sum()) < 6 * sd + 1, (agree, q.sum(), sd)
    # manual_seed reproduces the bits
    runs = []
    for _ in range(2):
        torch.cuda.manual_seed(1234)
        runs.append(call())
    assert runs[0][0] == runs[1][0]
    assert torch.equal(_bits(runs[0][2]), _bits(runs[1][2]))


# ---------------------------------------------------------------------------------------------------
# coverage of the launch plans (launches nothing)
# ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_random_stream_dispatch_coverage():
    """The tested row lengths reach every case the softmax launchers can dispatch to, and the tested widths every
    case norm_plan picks for the fused op's forward and backward."""
    nat = _nat()
    for dtype in (torch.float16, torch.bfloat16, torch.float32):
        epv = _epv(dtype)
        reachable = {_sm_case(nat.softmax_plan(64, K, dtype, True, kind))
                     for K in range(1, 1024 * epv + 2 * epv) for kind in ("fwd", "bwd")}
        tested = {_sm_case(nat.softmax_plan(64, _sm_k(k, dtype), dtype, True, kind))
                  for k in SM_NVECS + SM_SCALAR for kind in ("fwd", "bwd")}
        assert tested == reachable, (dtype, sorted(reachable - tested, key=str))
    for dtype in (torch.float16, torch.bfloat16):
        for kind in ("fused", "bwd"):
            reachable = {_norm_case(nat.norm_plan(1, n * 8, dtype, kind)) for n in range(1, 1025)}
            tested = {_norm_case(nat.norm_plan(1, n * 8, dtype, kind)) for n in NORM_NVECS}
            assert None not in reachable and tested == reachable, (dtype, kind, sorted(reachable - tested, key=str))
            assert {t[0] for t in tested} == {1, 2, 3}
