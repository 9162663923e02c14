"""The fused attention's dropout stream, pinned independently of how the kernels compute it.

A numpy Philox4x32-7 (the generator of csrc/common.cuh) reproduces the forward's keep bits on the host from the seed
and offset that the default CUDA generator hands the kernel: element (lin, key) of row lin = (b * H + h) * Lq + q uses
call (lin * Lk + key) >> 3, word (key & 7) >> 1, low half for even keys and high half for odd ones, and is kept iff its
14 low bits are >= round(p * 16384).  The returned ``bits`` tensor must equal the host words bit for bit, and O, LSE,
the logits z and every gradient are checked against an fp64 reference that uses those host keep bits, with per-element
bounds built from the dtype's unit roundoff (as tests/test_gpu_norms.py does).

Covered: D in {32, 64, 96, 128} (both padded widths of the kernels), fp16 and bf16, plain and logits mode, ragged
Lq != Lk with Lk not a multiple of the key tile, a single key tile, and a grid of more than one wave.
"""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]
UNIT = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}   # unit roundoff of the 16-bit operands and results
HEAD_DIMS = [32, 64, 96, 128]
P_DROP = 0.2
# (B, H, Lq, Lk): ragged with Lk past a whole key tile; one key tile at either padded width (Lk <= 64); and a grid of
# more than one wave of CTAs (B * H * Lq / 64 = 768 forward CTAs, 2 per SM on 132 SMs)
SHAPES = {"ragged": (2, 3, 136, 200), "one_tile": (2, 2, 72, 40), "waves": (4, 12, 1024, 72)}
M32 = np.uint64(0xFFFFFFFF)


def _native():
    from unicore import ops

    assert ops.USE_NATIVE, "native kernels must be active on the GPU box"
    return ops.native()


def philox4x32_7(seed, offset, ctr):
    """Philox4x32 with 7 rounds, vectorised over uint64 counters; the word order of csrc/common.cuh."""
    k0, k1 = np.uint64(seed & 0xFFFFFFFF), np.uint64((seed >> 32) & 0xFFFFFFFF)
    c0, c1 = ctr & M32, ctr >> np.uint64(32)
    c2 = np.full_like(ctr, offset & 0xFFFFFFFF)
    c3 = np.full_like(ctr, (offset >> 32) & 0xFFFFFFFF)
    for _ in range(7):
        p0 = np.uint64(0xD2511F53) * c0
        p1 = np.uint64(0xCD9E8D57) * c2
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & M32, p1 >> np.uint64(32), p1 & M32
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
        k0 = (k0 + np.uint64(0x9E3779B9)) & M32
        k1 = (k1 + np.uint64(0xBB67AE85)) & M32
    return c0, c1, c2, c3


def host_keep_words(seed, offset, B, H, Lq, Lk, p):
    """[B, H, Lq, ceil(Lk / 32)] keep words in the layout of csrc/attn/fmha_api.h (key 32w + 2i in bit i, key
    32w + 2i + 1 in bit 16 + i), and the [B, H, Lq, Lk] keep mask they encode."""
    t14 = min(max(int(p * 16384.0 + 0.5), 0), 16383)
    nw = (Lk + 31) // 32
    lin = np.arange(B * H * Lq, dtype=np.uint64)[:, None]
    ctr = (lin * np.uint64(Lk) + np.arange(0, 32 * nw, 8, dtype=np.uint64)[None, :]) >> np.uint64(3)
    words = np.stack(philox4x32_7(seed, offset, ctr), axis=-1)   # [rows, 4 * nw calls, word c]: keys 8j + 2c, +1
    lo = (words & np.uint64(0x3FFF)) >= t14
    hi = ((words >> np.uint64(16)) & np.uint64(0x3FFF)) >= t14
    keep = np.stack([lo, hi], axis=-1).reshape(B * H * Lq, 32 * nw)   # key 8j + 2c + e
    bitpos = np.arange(32)
    shift = np.where(bitpos % 2 == 0, bitpos // 2, 16 + bitpos // 2).astype(np.uint64)   # bit of key 32w + bitpos
    kw = keep.reshape(B * H * Lq, nw, 32).astype(np.uint64) << shift
    packed = np.bitwise_or.reduce(kw, axis=-1).astype(np.uint32).view(np.int32).reshape(B, H, Lq, nw)
    mask = keep[:, :Lk].reshape(B, H, Lq, Lk)
    return packed, mask, 16384.0 / (16384.0 - t14)


def _inputs(B, H, Lq, Lk, D, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    q = (torch.randn(B, Lq, H, D, device="cuda", generator=g) * 0.6).to(dtype)
    k = (torch.randn(B, Lk, H, D, device="cuda", generator=g) * 0.6).to(dtype)
    v = torch.randn(B, Lk, H, D, device="cuda", generator=g).to(dtype)
    bias = torch.randn(1, H, Lq, Lk, device="cuda", generator=g).to(dtype)
    kpm = torch.zeros(B, Lk, dtype=torch.bool, device="cuda")
    kpm[0, Lk - Lk // 4:] = True
    kpm[-1, :8] = True
    return q, k, v, bias, kpm


def run_forward(q, k, v, bias, kpm, scale, logits, rng_seed):
    """Calls the binding directly; returns (out, lse, bits, z, seed, offset) with the generator state it used."""
    nat = _native()
    torch.cuda.manual_seed(rng_seed)
    gen = torch.cuda.default_generators[torch.cuda.current_device()]
    seed, offset = gen.initial_seed(), gen.get_offset()
    if logits:
        out, lse, bits, z = nat.fmha_fwd_logits(q, k, v, bias, kpm, P_DROP, scale)
    else:
        (out, lse, bits), z = nat.fmha_fwd(q, k, v, bias, kpm, P_DROP, scale), None
    return out, lse, bits, z, seed, offset


def _assert_within(got, ref, bound, what):
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)
    if bad.any():
        i = bad.nonzero()[0].tolist()
        worst = (err / bound.clamp_min(1e-300)).nan_to_num(float("inf")).max().item()
        raise AssertionError("{}: {} elements out of bound, first at {}: got {}, want {} +- {} (worst {:.3g}x)".format(
            what, int(bad.sum()), i, got[tuple(i)].item(), ref[tuple(i)].item(), bound[tuple(i)].item(), worst))


def _reference(q, k, v, bias, kpm, scale, keep, keep_scale):
    """fp64 forward with the host keep mask: logits z, |z| bound terms, P, dropped P, O, |O| terms, LSE."""
    qd, kd, vd = q.double(), k.double(), v.double()
    z = torch.einsum("bqhd,bkhd->bhqk", qd, kd) * scale + bias.double()
    zabs = torch.einsum("bqhd,bkhd->bhqk", qd.abs(), kd.abs()) * scale + bias.double().abs()
    madd = torch.zeros(kpm.shape, dtype=torch.float64, device="cuda").masked_fill(kpm, float("-inf"))
    z = z + madd[:, None, None, :]
    lse = torch.logsumexp(z, dim=-1)
    pr = torch.exp(z - lse[..., None])
    pd = pr * keep * keep_scale
    out = torch.einsum("bhqk,bkhd->bqhd", pd, vd)
    oabs = torch.einsum("bhqk,bkhd->bqhd", pd, vd.abs())
    # fp32 logits: D products accumulated in fp32 (D * 2^-24 <= 2^-17 relative to |q||k|), then exp / ex2.approx
    rel_z = 2.0 ** -16 * zabs.amax(dim=-1) + 1e-5   # [B, H, Lq]: relative error of the probabilities of a row
    return z, zabs, pr, pd, out, oabs, lse, rel_z


@pytest.mark.parametrize("logits", [False, True], ids=["plain", "logits"])
@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("D", HEAD_DIMS)
@pytest.mark.parametrize("shape", list(SHAPES), ids=list(SHAPES))
def test_keep_bits_equal_host_philox(shape, D, dtype, logits):
    B, H, Lq, Lk = SHAPES[shape]
    q, k, v, bias, kpm = _inputs(B, H, Lq, Lk, D, dtype, seed=11)
    out, lse, bits, z, seed, offset = run_forward(q, k, v, bias, kpm, 1.0 / math.sqrt(D), logits, rng_seed=1234 + D)
    host, _, _ = host_keep_words(seed, offset, B, H, Lq, Lk, P_DROP)
    got = bits.cpu().numpy()
    assert got.shape == host.shape
    diff = got != host
    assert not diff.any(), "{} of {} keep words differ, first at {}".format(int(diff.sum()), diff.size,
                                                                             np.argwhere(diff)[0].tolist())


@pytest.mark.parametrize("logits", [False, True], ids=["plain", "logits"])
@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("D", HEAD_DIMS)
@pytest.mark.parametrize("shape", ["ragged", "one_tile"])
def test_forward_and_backward_against_fp64_with_host_bits(shape, D, dtype, logits):
    B, H, Lq, Lk = SHAPES[shape]
    u = UNIT[dtype]
    scale = 1.0 / math.sqrt(D)
    q, k, v, bias, kpm = _inputs(B, H, Lq, Lk, D, dtype, seed=5 + D)
    out, lse, bits, z, seed, offset = run_forward(q, k, v, bias, kpm, scale, logits, rng_seed=99 + D)
    host, keep_np, keep_scale = host_keep_words(seed, offset, B, H, Lq, Lk, P_DROP)
    assert np.array_equal(bits.cpu().numpy(), host)
    keep = torch.from_numpy(keep_np).to("cuda", torch.float64)
    z_ref, zabs, pr, pd, o_ref, oabs, lse_ref, rel_z = _reference(q, k, v, bias, kpm, scale, keep, keep_scale)
    rz = rel_z.permute(0, 2, 1)[..., None]   # [B, Lq, H, 1]

    # O: P is rounded to the 16-bit type before P V (u), the fp32 row sum and accumulation, one rounding of O
    # fp16 has subnormals below 2^-14: a rounded probability or dS element may be off by up to 2^-25 absolutely
    sub = 2.0 ** -25 if dtype == torch.float16 else 0.0
    _assert_within(out, o_ref, (2 * u + rz) * oabs + u * o_ref.abs() + sub * Lk * v.abs().max().item(), "O")
    _assert_within(lse, lse_ref, 2.0 ** -16 * zabs.amax(dim=-1) + 1e-5 * (1 + lse_ref.abs()), "LSE")
    if logits:
        fin = torch.isfinite(z_ref)
        assert torch.equal(torch.isfinite(z), fin) and bool((z[~fin] < 0).all()), "z is -inf exactly at masked keys"
        _assert_within(z[fin], z_ref[fin], (u * z_ref.abs() + 2.0 ** -17 * zabs)[fin], "z")

    # ---- backward, with an incoming dz in logits mode -----------------------------------------------------------
    g = torch.Generator(device="cuda").manual_seed(7 + D)
    dout = torch.randn(B, Lq, H, D, device="cuda", generator=g).to(dtype)
    dz = (torch.randn(B, H, Lq, Lk, device="cuda", generator=g) * 0.1).to(dtype) if logits else None
    dq, dk, dv, dbias = _native().fmha_bwd(dout, q, k, v, out, lse, bias, kpm, P_DROP, scale, bits, True, False, dz)

    dod, vd, qd, kd = dout.double(), v.double(), q.double(), k.double()
    delta = (dod * out.double()).sum(-1).permute(0, 2, 1)[..., None]   # from the forward's 16-bit O, as the kernel
    delta_abs = (dod.abs() * out.double().abs()).sum(-1).permute(0, 2, 1)[..., None]
    dp = torch.einsum("bqhd,bkhd->bhqk", dod, vd)
    dp_abs = torch.einsum("bqhd,bkhd->bhqk", dod.abs(), vd.abs())
    dpd = dp * keep * keep_scale
    ds = pr * (dpd - delta) + (dz.double() if logits else 0.0)
    # dS error: fp32 probabilities (rel_z), fp32 dP and delta sums, then one rounding to the 16-bit type
    e_ds = (pr * (rel_z[..., None] * (dpd - delta).abs() + 2.0 ** -16 * (dp_abs * keep * keep_scale + delta_abs))
            + u * ds.abs())
    dv_ref = torch.einsum("bhqk,bqhd->bkhd", pd, dod)
    dv_bnd = torch.einsum("bhqk,bqhd->bkhd", pd * (u + rel_z[..., None]), dod.abs()) + u * dv_ref.abs()
    _assert_within(dv, dv_ref, dv_bnd + sub * Lq * keep_scale * dout.abs().max().item() + 1e-6, "dV")
    dk_ref = torch.einsum("bhqk,bqhd->bkhd", ds, qd) * scale
    dk_bnd = torch.einsum("bhqk,bqhd->bkhd", e_ds, qd.abs()) * scale + u * dk_ref.abs()
    _assert_within(dk, dk_ref, dk_bnd + sub * Lq * scale * q.abs().max().item() + 1e-6, "dK")
    dq_ref = torch.einsum("bhqk,bkhd->bqhd", ds, kd) * scale
    dq_bnd = torch.einsum("bhqk,bkhd->bqhd", e_ds, kd.abs()) * scale + u * dq_ref.abs()
    _assert_within(dq, dq_ref, dq_bnd + sub * Lk * scale * k.abs().max().item() + 1e-6, "dQ")
    # the bias is shared by the batch: the 16-bit dS tiles are summed over it in fp32, then rounded once
    db_ref = ds.sum(0, keepdim=True)
    _assert_within(dbias, db_ref, e_ds.sum(0, keepdim=True) + u * db_ref.abs() + sub * B + 1e-6, "dBias")
