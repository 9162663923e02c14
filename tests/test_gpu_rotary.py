"""Rotary position embeddings on the H100: the kernel behind ``ops.rotary_embedding`` (``csrc/fused/rotary.cu``) and the
modules that use it.

Shapes come from the launch plan (``rotary_plan``, the function the launcher runs): one grid sweep, several, and a
ragged last one; the 16-byte path and the narrow one; fp16 and bf16; head dims 8 .. 160 with ``rd = D`` and ``rd < D``;
the MHA and GQA packed layouts and a strided q slice.  Rotated values are checked against fp64 on the same fp32 angles
(also at positions near 2^20, where a fast-math sine fails), everything else bitwise (NaN payloads included).  Then the
backward, graph capture with device offsets, the operand checks, and encoder / decoder modules: training against the
fp32 module and incremental decoding (steps, chunks, captured steps, reorder, rewind) against the full forward.
"""
import re

import pytest
import torch

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]
DT_IDS = ["fp16", "bf16"]
UNIT = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
GRAD_TOL = {torch.float16: 1e-2, torch.bfloat16: 5e-2}   # relative norm error against the fp32 module
STEP_TOL = {torch.float16: 2e-2, torch.bfloat16: 6e-2}   # relative norm per step, as the eager decoder tests


def _ops():
    from unicore import ops

    assert ops.USE_NATIVE, "native kernels must be active on the GPU box"
    return ops


def _rot():
    return _ops().native().rotary


def _bits(t):
    return t.contiguous().view(torch.int16)


def _rel(got, want):
    return ((got.double() - want.double()).norm() / want.double().norm()).item()


def _fp64(x, inv_freq, R, offsets=None, inverse=False):
    """fp64 rotation at the kernel's fp32 angles fl32(float(pos) * inv_freq[i]), and the magnitude |x1| + |x2| of
    each rotated element's pair (for the fp32 product error)."""
    B, L, N, D = x.shape
    half = inv_freq.numel()
    pos = torch.arange(L, device=x.device).view(1, L)
    if offsets is not None:
        pos = pos + offsets.long().view(-1, 1)
    theta = (pos.float()[..., None] * inv_freq).double()[:, :, None, :]
    c, s = theta.cos(), theta.sin() * (-1 if inverse else 1)
    xd = x.double()
    y, mag = xd.clone(), torch.zeros_like(xd)
    x1, x2 = xd[:, :, :R, :half], xd[:, :, :R, half:2 * half]
    y[:, :, :R, :half] = x1 * c - x2 * s
    y[:, :, :R, half:2 * half] = x2 * c + x1 * s
    mag[:, :, :R, :half] = mag[:, :, :R, half:2 * half] = x1.abs() + x2.abs()
    return y, mag


def _assert_rotated(got, x, inv_freq, R, offsets, dtype, inverse=False, what=""):
    """Rotated elements within one rounding of the output type plus the fp32 error of the two products (and of the
    rounded cos / sin); every other element bitwise x."""
    ref, mag = _fp64(x, inv_freq, R, offsets, inverse)
    rd = 2 * inv_freq.numel()
    bound = UNIT[dtype] * ref.abs() + 2.0 ** -21 * mag + 2.0 ** -24
    err = (got.double() - ref).abs()
    rot = err[:, :, :R, :rd]
    bad = ~(rot <= bound[:, :, :R, :rd])
    if bad.any():
        i = bad.nonzero()[0].tolist()
        raise AssertionError("{}: {} rotated elements out of bound, first at {}: got {}, want {}".format(
            what, int(bad.sum()), i, got[:, :, :R, :rd][tuple(i)].item(), ref[:, :, :R, :rd][tuple(i)].item()))
    assert torch.equal(_bits(got[:, :, R:]), _bits(x[:, :, R:])), what
    assert torch.equal(_bits(got[:, :, :R, rd:]), _bits(x[:, :, :R, rd:])), what


def _inv(rd):
    return _ops().rotary_inv_freq(rd, device="cuda")


def _layout(kind, B, L, H, D, dtype, g, misalign=False):
    """(x [B, L, N, D] as the op gets it, rotated heads).  mha: [B, L, 3, H, D] viewed as 3H heads; gqa: [B, L, H +
    2 H_kv, D] with H_kv = H / 2; qslice: the q heads of a packed [B, L, 3, H, D] projection (token stride 3 H D).
    misalign: the same values one element into their buffer, which only the narrow path takes."""
    N = {"mha": 3 * H, "gqa": 2 * H, "qslice": 3 * H}[kind]
    n = B * L * N * D
    buf = torch.randn(n + 8, device="cuda", generator=g).to(dtype)
    base = buf[1:1 + n] if misalign else buf[:n]
    packed = base.view(B, L, N, D)
    if kind == "mha":
        return packed, 2 * H
    if kind == "gqa":
        return packed, H + H // 2
    return packed.view(B, L, 3, H, D)[:, :, 0], H


def _plan_tokens(N, D, rd, dtype, aligned, sweeps):
    """B, L for `sweeps` grid sweeps of rotary_plan with a ragged last one (sweeps = 0: one partial sweep)."""
    rot = _rot()
    p = rot.rotary_plan(1, 1 << 24, N, D, rd, dtype, aligned)
    per_sweep = p["items_per_sweep"] * p["tile_tokens"]
    tokens = 5 * p["tile_tokens"] + 3 if sweeps == 0 else sweeps * per_sweep - per_sweep // 2 + 3
    B = 2
    L = (tokens + B - 1) // B
    q = rot.rotary_plan(B, L, N, D, rd, dtype, aligned)
    assert q["sweeps"] == max(sweeps, 1), q
    assert (B * L) % per_sweep != 0
    return B, L


# ---- the kernel ---------------------------------------------------------------------------------------------------
CASES = [  # (D, rd): vector path where rd / 2 % 8 == 0, narrow path otherwise
    (8, 8), (64, 64), (64, 32), (64, 6), (96, 96), (96, 48), (128, 128), (128, 64), (160, 160), (160, 20)]


@pytest.mark.parametrize("kind", ["mha", "gqa", "qslice"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("D,rd", CASES, ids=["D{}_rd{}".format(*c) for c in CASES])
def test_kernel_against_fp64(D, rd, dtype, kind):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(D * 1000 + rd)
    x, R = _layout(kind, 3, 37, 4, D, dtype, g)
    inv = _inv(rd)
    off = torch.tensor([0, 17, (1 << 20) - 40], dtype=torch.int32, device="cuda")
    aligned = kind != "qslice" or (3 * 4 * D) % 8 == 0
    assert _rot().rotary_plan(3, 37, x.size(2), D, rd, dtype, aligned)["vec"] == ((rd // 2) % 8 == 0)
    for offsets in (None, off):
        y = ops.rotary_embedding(x, inv, R, offsets)
        assert y.shape == x.shape and y.is_contiguous()
        _assert_rotated(y, x, inv, R, offsets, dtype, what=(kind, offsets is not None))


@pytest.mark.parametrize("sweeps", [0, 1, 3], ids=["partial", "one", "three"])
@pytest.mark.parametrize("vec", [True, False], ids=["vec", "narrow"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_kernel_sweeps(sweeps, vec, dtype):
    ops = _ops()
    H, D, rd = 2, 16, 16
    B, L = _plan_tokens(3 * H, D, rd, dtype, vec, sweeps)
    g = torch.Generator(device="cuda").manual_seed(sweeps)
    x, R = _layout("mha", B, L, H, D, dtype, g, misalign=not vec)
    assert _rot().rotary_plan(B, L, 3 * H, D, rd, dtype, x.data_ptr() % 16 == 0)["vec"] == vec
    off = torch.tensor([3, 100000], dtype=torch.int32, device="cuda")
    _assert_rotated(ops.rotary_embedding(x, _inv(rd), R, off), x, _inv(rd), R, off, dtype, what=(sweeps, vec))


@pytest.mark.parametrize("vec", [True, False], ids=["vec", "narrow"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_copies_are_bitwise_with_nan_payloads(vec, dtype):
    ops = _ops()
    B, L, N, D, R, rd = 2, 19, 6, 64, 4, 32
    n = B * L * N * D
    buf = torch.randint(-(1 << 15), 1 << 15, (n + 8,), dtype=torch.int16, device="cuda")
    bits = buf[:n] if vec else buf[1:1 + n]
    x = bits.view(dtype).view(B, L, N, D)
    # quiet and signalling NaNs with payloads, infinities, negative zero and subnormals in the copied region
    special = torch.tensor([0x7c01, 0x7e55, -0x0001, 0x7c00, -0x8000, 0x0001, 0x7f81, 0x7fc3], dtype=torch.int16,
                           device="cuda")
    bits.view(B, L, N, D)[:, :, R:, :8] = special
    bits.view(B, L, N, D)[:, :, :R, rd:rd + 8] = special
    y = ops.rotary_embedding(x, _inv(rd), R)
    assert torch.equal(_bits(y[:, :, R:]), _bits(x[:, :, R:]))
    assert torch.equal(_bits(y[:, :, :R, rd:]), _bits(x[:, :, :R, rd:]))


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("D,rd", [(64, 64), (96, 20), (128, 64)])
def test_backward_is_the_inverse_rotation(D, rd, dtype):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(D + rd)
    x, R = _layout("gqa", 2, 33, 4, D, dtype, g)
    inv = _inv(rd)
    off = torch.tensor([5, 70000], dtype=torch.int32, device="cuda")
    xr = x.detach().clone().requires_grad_(True)
    y = ops.rotary_embedding(xr, inv, R, off)
    gy = torch.randn(y.shape, device="cuda", generator=g).to(dtype)
    gy_keep = gy.clone()
    (gx,) = torch.autograd.grad(y, xr, gy)
    assert torch.equal(gy, gy_keep)   # the incoming gradient is not written into
    _assert_rotated(gx, gy, inv, R, off, dtype, inverse=True, what="grad")
    back = _rot().rotary_embedding(y, inv, R, off, True)
    x1, x2 = x[:, :, :R, :rd // 2].double(), x[:, :, :R, rd // 2:rd].double()
    mag = torch.zeros_like(x, dtype=torch.float64)
    mag[:, :, :R, :rd // 2] = mag[:, :, :R, rd // 2:rd] = x1.abs() + x2.abs()
    assert bool(((back.double() - x.double()).abs() <= 4 * UNIT[dtype] * mag + 2.0 ** -24).all())
    assert torch.equal(_bits(back[:, :, R:]), _bits(x[:, :, R:]))


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_graph_replay_reads_new_offsets(dtype):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(9)
    x, R = _layout("mha", 4, 3, 4, 64, dtype, g)
    inv = _inv(64)
    off = torch.tensor([0, 1, 2, 3], dtype=torch.int32, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.rotary_embedding(x, inv, R, off)   # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = ops.rotary_embedding(x, inv, R, off)
    for new in ([0, 1, 2, 3], [100, 7, 65536, 1000000]):
        off.copy_(torch.tensor(new, dtype=torch.int32))
        graph.replay()
        eager = ops.rotary_embedding(x, inv, R, off)
        assert torch.equal(_bits(out), _bits(eager)), new
        _assert_rotated(out, x, inv, R, off, dtype, what=new)


def test_operands_are_checked():
    """The operand-rejection table of tests/test_gpu_bindings.py over _C.rotary.rotary_embedding."""
    rot = _rot()

    def nc(t):
        s = torch.empty(*t.shape, 2, dtype=t.dtype, device=t.device)[..., 0]
        s.copy_(t)
        return s

    mutate = {"cpu": lambda t: t.cpu(), "dtype": lambda t: t.to(torch.int16),
              "small": lambda t: t.reshape(-1)[:-1].clone(), "nc": nc}

    def valid():
        return [torch.randn(2, 5, 6, 16, device="cuda").half(), _inv(16), 4,
                torch.tensor([1, 2], dtype=torch.int32, device="cuda"), False]

    rot.rotary_embedding(*valid())
    for i, (label, kinds) in {0: ("x", ("cpu", "dtype", "small", "nc")), 1: ("inv_freq", ("cpu", "dtype", "nc")),
                              3: ("position_offsets", ("cpu", "dtype", "small", "nc"))}.items():
        for kind in kinds:
            args = valid()
            args[i] = mutate[kind](args[i])
            with pytest.raises(RuntimeError, match=r"\b" + re.escape(label) + " must"):
                rot.rotary_embedding(*args)
    args = valid()
    with pytest.raises(RuntimeError, match="rotated_heads"):
        rot.rotary_embedding(args[0], args[1], 7, None)
    with pytest.raises(RuntimeError, match="inv_freq must have"):
        rot.rotary_embedding(args[0], _inv(18), 4, None)
    with pytest.raises(RuntimeError, match="rotary_plan needs"):
        rot.rotary_plan(1, 8, 3, 16, 7, torch.float16)
    with pytest.raises(RuntimeError, match="rotary_plan needs"):
        rot.rotary_plan(1, 8, 3, 16, 16, torch.float32)
    assert rot.rotary_plan(1, 8, 3, 16, 16, torch.float16)["grid"] == 1


# ---- the modules ----------------------------------------------------------------------------------------------------
E, HEADS = 256, 4


def _stack(cls, dtype, rel_pos, kv_heads, seed=0, dropout=0.0):
    from unicore.modules import TransformerDecoder
    from unicore.modules.transformer import TransformerEncoder

    n = "decoder_layers" if cls is TransformerDecoder else "encoder_layers"
    torch.manual_seed(seed)
    m = (TransformerDecoder if cls is TransformerDecoder else TransformerEncoder)(
        **{n: 2}, embed_dim=E, ffn_embed_dim=2 * E, attention_heads=HEADS, max_seq_len=256, rel_pos=rel_pos,
        attention_kv_heads=kv_heads, rotary_dim=E // HEADS, emb_dropout=dropout, dropout=dropout,
        attention_dropout=dropout).cuda()
    with torch.no_grad():
        for p in m.parameters():
            p.add_(torch.randn_like(p) * 0.02)
    return m.to(dtype) if dtype is not None else m


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("rel_pos,kv_heads", [(False, None), (True, None), (False, 2)],
                         ids=["rotary", "rotary_rel_pos", "rotary_gqa"])
@pytest.mark.parametrize("stack", ["encoder", "decoder"])
def test_module_training_matches_fp32(stack, rel_pos, kv_heads, dtype):
    from unicore.modules import TransformerDecoder

    ops = _ops()
    cls = TransformerDecoder if stack == "decoder" else None
    ref = _stack(cls, None, rel_pos, kv_heads)
    m = _stack(cls, dtype, rel_pos, kv_heads)
    assert m.layers[0].self_attn.inv_freq.dtype == torch.float32
    g = torch.Generator(device="cuda").manual_seed(1)
    B, L = 3, 136
    x = torch.randn(B, L, E, device="cuda", generator=g)
    pad = torch.zeros(B, L, dtype=torch.bool, device="cuda")
    pad[1, -20:] = True
    calls = []
    real = ops.native()

    class Spy:
        class rotary:   # noqa: N801
            @staticmethod
            def rotary_embedding(*args, **kwargs):
                calls.append(args[4] if len(args) > 4 else False)
                return real.rotary.rotary_embedding(*args, **kwargs)

        def __getattr__(self, name):
            return getattr(real, name)

    import unicore_b200.ops.rotary_ops as rotary_ops
    saved = rotary_ops.native
    rotary_ops.native = lambda: Spy()
    try:
        xm = x.to(dtype).requires_grad_(True)
        y = m(xm, padding_mask=pad)
        gy = torch.randn(y.shape, device="cuda", generator=g)
        y.backward(gy.to(dtype))
    finally:
        rotary_ops.native = saved
    assert calls.count(False) == 2 and calls.count(True) == 2   # the kernel ran forward and backward in each layer
    xr = x.clone().requires_grad_(True)
    yr = ref(xr, padding_mask=pad)
    yr.backward(gy)
    keep = ~pad
    assert _rel(y[keep], yr[keep]) < GRAD_TOL[dtype]
    assert _rel(xm.grad[keep], xr.grad[keep]) < GRAD_TOL[dtype]
    for (name, p), (_, q) in zip(m.named_parameters(), ref.named_parameters()):
        if p.dim() == 2 and q.grad is not None:   # weight matrices (some bias gradients are rounding noise)
            assert _rel(p.grad, q.grad) < GRAD_TOL[dtype], name


def _prompts(dtype, lens, extra, g):
    B, L = len(lens), max(lens)
    tokens = torch.randn(B, L + extra, E, device="cuda", generator=g).to(dtype)
    prompt = torch.zeros(B, L, E, device="cuda", dtype=dtype)
    pad = torch.ones(B, L, dtype=torch.bool, device="cuda")
    for b, n in enumerate(lens):
        prompt[b, :n] = tokens[b, :n]
        pad[b, :n] = False
    enc = torch.randn(B, 10, E, device="cuda", generator=g).to(dtype)
    return tokens, prompt, pad, enc


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("rel_pos,kv_heads", [(False, None), (True, None), (False, 2)],
                         ids=["rotary", "rotary_rel_pos", "rotary_gqa"])
def test_decoding_matches_full_forward(rel_pos, kv_heads, dtype):
    from unicore.modules import TransformerDecoder

    _ops()
    m = _stack(TransformerDecoder, dtype, rel_pos, kv_heads).eval()
    lens = [12, 5, 9]
    g = torch.Generator(device="cuda").manual_seed(2)
    tokens, prompt, pad, enc = _prompts(dtype, lens, 40, g)
    pos = list(lens)
    order = None

    def check(y, T, what):
        seq = tokens if order is None else tokens[order]
        e = enc if order is None else enc[order]
        for b in range(len(lens)):
            full = m(seq[b:b + 1, :pos[b] + T], encoder_out=e[b:b + 1])
            assert _rel(y[b], full[0, -T:]) < STEP_TOL[dtype], (what, b)

    def emb(T):
        seq = tokens if order is None else tokens[order]
        return torch.stack([seq[b, pos[b]:pos[b] + T] for b in range(len(lens))])

    def advance(T):
        for b in range(len(lens)):
            pos[b] += T

    with torch.no_grad():
        cache = m.new_cache(3, 64)
        m(prompt, encoder_out=enc, padding_mask=pad, cache=cache)
        for t in range(4):                                   # eager one-token steps
            e = emb(1)
            check(m(e, cache=cache), 1, ("step", t))
            advance(1)
        e = emb(4)                                           # an eager chunk
        check(m(e, cache=cache), 4, "chunk")
        advance(4)
        step = m.capture_step(cache)
        for t in range(3):                                   # captured one-token steps
            e = emb(1)
            check(step(e).clone(), 1, ("replay", t))
            advance(1)
        cache.rewind(2)
        for b in range(3):
            pos[b] -= 2
        order = torch.tensor([2, 0, 1], device="cuda")
        cache.reorder(order)
        pos = [pos[i] for i in order.tolist()]
        for t in range(2):                                   # replays after rewind and reorder
            e = emb(1)
            check(step(e).clone(), 1, ("replay after reorder", t))
            advance(1)
        assert step.captures == 1
        chunk = m.capture_step(cache, T=3)                   # a captured chunk
        e = emb(3)
        check(chunk(e).clone(), 3, "captured chunk")
        advance(3)
