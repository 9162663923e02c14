"""Multi-token steps into a key / value cache on the GPU: the KV-cache mode of the wgmma forward
(``kvcache.fmha_kvcache_fwd``, ``ops.attention_with_kv_cache`` with T > 1) and ``TransformerDecoder`` chunks on it.

Checked: the op against the fp64 ``attention_with_kv_cache_reference`` for T from 2 to 200 at every head-dim tier in
fp16 / bf16, with ragged ``seqlens`` (0 .. 1000) in one batch, capacities that are not multiples of 8, shared and
per-batch bias rows wider than the visible keys, key padding with a fully masked query, and out-of-range ``seqlens``
(clamped as the reference clamps them); the append from strided views of a packed ``[B, T, 3, H, D]`` projection
(new rows bitwise equal, every other row bitwise untouched, NaN sentinels past the visible rows harmless);
cross-attention (``seqlens=None``); agreement with T successive ``fmha_decode`` steps; a decoder fed prefill + chunks +
single steps in fp16 / bf16 against an fp32 copy run on each sequence alone, which binding each step calls, and that a
chunk step does not synchronise; and the binding's operand checks.
"""
import copy
import re

import pytest
import torch

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]
DT_IDS = ["fp16", "bf16"]
UNIT = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
HEAD_DIMS = [8, 64, 96, 128]   # both padded widths, the narrowest and the widest
TS = [2, 3, 8, 63, 64, 65, 200]
LENS = [0, 1, 127, 128, 129, 1000]   # one batch, ragged


def _ops():
    from unicore import ops

    assert ops.USE_NATIVE, "native kernels must be active on the GPU box"
    return ops


def _kv():
    return _ops().native().kvcache


def _ref_mag(q, k, v, seqlens, max_len, k_new, v_new, bias, kpm, scale):
    """fp64 reference O and mag = sum_k p_k |v_k| with the exact probabilities.  The caches are copied, so the
    caller's are not appended to."""
    ops = _ops()
    d = lambda t: None if t is None else t.double()   # noqa: E731
    ref = ops.attention_with_kv_cache_reference(d(q), k.double(), v.double(), seqlens, max_len, d(k_new), d(v_new),
                                                d(bias), kpm, scale)
    mag = ops.attention_with_kv_cache_reference(d(q), k.double(), v.double().abs(), seqlens, max_len, d(k_new),
                                                None if v_new is None else v_new.double().abs(), d(bias), kpm, scale)
    return ref, mag


def _decode_bound(q, k, v, seqlens, max_len, bias, scale, dtype):
    """The bound of test_gpu_attention_kvcache.py for one decode step (fp32 P V on the CUDA cores): the 16-bit rounding
    of O plus fp32 terms of sum_k p_k |v_k|."""
    ref, mag = _ref_mag(q, k, v, seqlens, max_len, None, None, bias, None, scale)
    return ref, UNIT[dtype] * ref.abs() + 2.0 ** -13 * mag


def _bound(q, k, v, seqlens, max_len, k_new, v_new, bias, kpm, scale, dtype):
    """fp64 reference O and the error bound of a chunk, which runs in the wgmma forward: P is rounded to the 16-bit
    type before P V, so on top of the decode step's terms every p_k carries one rounding (2u sum_k p_k |v_k| in all, as
    the fused-forward tests of test_gpu_attention_causal.py count it), ex2 of a logit z is off by about 2^-16 |z|, and
    fp16 flushes probabilities below its subnormal range (2^-25 each, at most one per visible key)."""
    u = UNIT[dtype]
    ref, mag = _ref_mag(q, k, v, seqlens, max_len, k_new, v_new, bias, kpm, scale)
    qa = q.double().abs()
    keys = [torch.nan_to_num(k.double().abs(), nan=0.0)] + ([] if k_new is None else [k_new.double().abs()])
    zmax = scale * max(torch.einsum("bqhd,bkhd->bhqk", qa, t).max().item() for t in keys)
    if bias is not None:
        zmax += bias.double().abs().max().item()
    rz = 2.0 ** -16 * zmax + 1e-5
    vmax = torch.nan_to_num(v.double().abs(), nan=0.0).max().item()
    if v_new is not None:
        vmax = max(vmax, v_new.double().abs().max().item())
    sub = 2.0 ** -25 * k.shape[1] * vmax if dtype == torch.float16 else 0.0
    return ref, (2 * u + rz + 2.0 ** -13) * mag + u * ref.abs() + sub


def _assert_within(got, ref, bound, what):
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)
    if bad.any():
        i = bad.nonzero()[0].tolist()
        raise AssertionError("{}: {} elements out of bound, first at {}: got {}, want {} +- {}".format(
            what, int(bad.sum()), i, got[tuple(i)].item(), ref[tuple(i)].item(), bound[tuple(i)].item()))


def _inputs(B, T, C, H, D, dtype, g):
    k = (torch.randn(B, C, H, D, device="cuda", generator=g) * 0.6).to(dtype)
    v = torch.randn(B, C, H, D, device="cuda", generator=g).to(dtype)
    qkv = (torch.randn(B, T, 3, H, D, device="cuda", generator=g) * 0.6).to(dtype)
    return k, v, qkv


# ---- 1. op against fp64 --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["plain", "bias_shared_kpm", "bias_batch"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("D", HEAD_DIMS)
@pytest.mark.parametrize("T", TS)
def test_op_against_fp64(T, D, dtype, case):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(T * 1000 + D)
    B, H = len(LENS), 2
    max_len = max(LENS)
    C = max_len + T + 3   # not a multiple of 8 for odd T
    k, v, qkv = _inputs(B, T, C, H, D, dtype, g)
    for b, n in enumerate(LENS):   # stale rows past the visible keys
        k[b, n + T:] = float("nan")
        v[b, n + T:] = float("nan")
    q, k_new, v_new = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    seqlens = torch.tensor(LENS, dtype=torch.int32, device="cuda")
    bias = kpm = None
    if case != "plain":
        Lb = max_len + T + 11   # wider than the visible keys; the op pads it to a multiple of 8
        bias = torch.randn(B if case == "bias_batch" else 1, H, T, Lb, device="cuda", generator=g).to(dtype)
    if case == "bias_shared_kpm":
        kpm = torch.zeros(B, C, dtype=torch.bool, device="cuda")
        kpm[0, 0] = True            # length 0: query 0 sees only key 0, which is masked -> O = 0
        kpm[2, 3:90] = True
        kpm[5, 500:900] = True
    scale = D ** -0.5
    ref, bound = _bound(q, k, v, seqlens, max_len, k_new, v_new, bias, kpm, scale, dtype)
    out = ops.attention_with_kv_cache(q, k, v, seqlens, max_len, k_new=k_new, v_new=v_new, bias=bias,
                                      key_padding_mask=kpm, scale=scale)
    assert out.shape == (B, T, H, D) and out.dtype == dtype
    assert bool(torch.isfinite(out).all())
    _assert_within(out, ref, bound, "O")
    if case == "bias_shared_kpm":
        assert torch.equal(out[0, 0], torch.zeros_like(out[0, 0]))


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_out_of_range_seqlens_are_clamped(dtype):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(3)
    B, T, C, H, D = 4, 9, 77, 2, 64
    k, v, qkv = _inputs(B, T, C, H, D, dtype, g)
    q, k_new, v_new = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    seqlens = torch.tensor([-5, 72, 77, 1 << 30], dtype=torch.int32, device="cuda")   # partly or wholly past C
    ref, bound = _bound(q, k, v, seqlens, C - T, k_new, v_new, None, None, D ** -0.5, dtype)
    out = ops.attention_with_kv_cache(q, k, v, seqlens, C - T, k_new=k_new, v_new=v_new, scale=D ** -0.5)
    _assert_within(out, ref, bound, "O")


# ---- 2. append, from the packed projection --------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("D", [40, 128])
@pytest.mark.parametrize("T", [2, 17, 130])
def test_append_from_packed_projection(T, D, dtype):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(100 + T + D)
    lens = [0, 5, 64, 300, 1023 - T]
    B, H, C = len(lens), 3, 1023
    k, v, qkv = _inputs(B, T, C, H, D, dtype, g)
    for b, n in enumerate(lens):   # a NaN sentinel in every row that is not visible before the append
        k[b, n:] = float("nan")
        v[b, n:] = float("nan")
    k0, v0 = k.clone(), v.clone()
    q, k_new, v_new = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]   # strided views [B, T, H, D]
    assert not k_new.is_contiguous()
    seqlens = torch.tensor(lens, dtype=torch.int32, device="cuda")
    scale = D ** -0.5
    out = _kv().fmha_kvcache_fwd(q, k, v, seqlens, max(lens), k_new, v_new, None, None, scale)
    i16 = lambda t: t.view(torch.int16)   # noqa: E731
    for b, n in enumerate(lens):
        assert torch.equal(i16(k[b, n:n + T]), i16(k_new[b])) and torch.equal(i16(v[b, n:n + T]), i16(v_new[b]))
        k0[b, n:n + T], v0[b, n:n + T] = k_new[b], v_new[b]
    assert torch.equal(i16(k), i16(k0)) and torch.equal(i16(v), i16(v0))   # NaN rows included, bitwise
    assert bool(torch.isfinite(out).all())
    ref, bound = _bound(q, k, v, seqlens, max(lens), k_new, v_new, None, None, scale, dtype)
    _assert_within(out, ref, bound, "O")


# ---- 3. cross-attention ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("D", [16, 96])
def test_cross_attention_chunk(D, dtype):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(D)
    B, T, S, H = 3, 37, 203, 4
    k, v, qkv = _inputs(B, T, S, H, D, dtype, g)
    q = qkv[:, :, 0].contiguous()
    bias = torch.randn(B * H, T, S, device="cuda", generator=g).to(dtype).view(B, H, T, S)
    kpm = torch.zeros(B, S, dtype=torch.bool, device="cuda")
    kpm[0, 150:] = True
    kpm[2] = True   # every key masked: O = 0
    scale = D ** -0.5
    ref, bound = _bound(q, k, v, None, None, None, None, bias, kpm, scale, dtype)
    out = ops.attention_with_kv_cache(q, k, v, bias=bias, key_padding_mask=kpm, scale=scale)
    _assert_within(out, ref, bound, "O")
    assert torch.equal(out[2], torch.zeros_like(out[2]))


# ---- 4. agreement with the decode kernel ----------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_chunk_agrees_with_decode_steps(dtype):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(11)
    B, T, H, D, C = 3, 24, 4, 64, 700
    lens = [0, 333, 600]
    k, v, qkv = _inputs(B, T, C, H, D, dtype, g)
    q, k_new, v_new = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    bias = torch.randn(B, H, T, 632, device="cuda", generator=g).to(dtype)
    seqlens = torch.tensor(lens, dtype=torch.int32, device="cuda")
    k1, v1 = k.clone(), v.clone()
    chunk = ops.attention_with_kv_cache(q, k, v, seqlens, max(lens), k_new=k_new, v_new=v_new, bias=bias)
    for i in range(T):
        step = ops.native().fmha_decode(q[:, i:i + 1], k1, v1, seqlens + i, max(lens) + i, k_new[:, i:i + 1],
                                        v_new[:, i:i + 1], bias[:, :, i:i + 1], None, D ** -0.5, 0)
        # query i sees rows 0 .. seqlens[b] + i in both: one bound for each result
        args = (q[:, i:i + 1], k1, v1, seqlens + i + 1, max(lens) + i + 1)
        ref, b_step = _decode_bound(*args, bias[:, :, i:i + 1], D ** -0.5, dtype)
        _, b_chunk = _bound(*args, None, None, bias[:, :, i:i + 1], None, D ** -0.5, dtype)
        _assert_within(step, ref, b_step, "decode step {}".format(i))
        _assert_within(chunk[:, i:i + 1], ref, b_chunk, "chunk query {}".format(i))
        _assert_within(chunk[:, i:i + 1], step.double(), b_step + b_chunk, "chunk vs decode step {}".format(i))
    assert torch.equal(k.view(torch.int16), k1.view(torch.int16)) and torch.equal(v.view(torch.int16),
                                                                                 v1.view(torch.int16))


# ---- 5. decoder ---------------------------------------------------------------------------------------------------
def _decoder_pair(dtype, post_ln):
    from unicore.modules import TransformerDecoder

    torch.manual_seed(0)
    ref = TransformerDecoder(post_ln=post_ln).cuda().eval()
    with torch.no_grad():
        for p in ref.parameters():   # non-trivial LayerNorm and bias parameters
            p.add_(torch.randn_like(p) * 0.02)
    return ref, copy.deepcopy(ref).to(dtype)


def _prompts(lens, T, Le, g):
    B = len(lens)
    tokens = torch.randn(B, T, 768, device="cuda", generator=g)
    enc = torch.randn(B, Le, 768, device="cuda", generator=g)
    enc_pad = torch.zeros(B, Le, dtype=torch.bool, device="cuda")
    enc_pad[0, Le - 8:] = True
    L = max(lens)
    prompt = torch.zeros(B, L, 768, device="cuda")
    pad = torch.ones(B, L, dtype=torch.bool, device="cuda")
    for b, n in enumerate(lens):
        prompt[b, :n] = tokens[b, :n]
        pad[b, :n] = False
    return tokens, prompt, pad, enc, enc_pad


@pytest.mark.parametrize("post_ln", [False, True], ids=["pre_ln", "post_ln"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_decoder_chunks_match_fp32_full_forward(dtype, post_ln, monkeypatch):
    import unicore_b200.ops.attention_ops as attention_ops

    ops = _ops()
    ref, model = _decoder_pair(dtype, post_ln)
    real = ops.native()
    calls = []

    class KvSpy:
        def fmha_kvcache_fwd(self, *args, **kwargs):
            calls.append(("chunk", args[3] is not None))
            return real.kvcache.fmha_kvcache_fwd(*args, **kwargs)

    class Spy:
        kvcache = KvSpy()

        def __getattr__(self, name):
            return getattr(real, name)

        def fmha_decode(self, *args, **kwargs):
            calls.append(("decode", args[3] is not None))
            return real.fmha_decode(*args, **kwargs)

    monkeypatch.setattr(attention_ops, "native", lambda: Spy())
    lens, sizes, Le = [24, 13, 19], [5, 1, 16, 2, 1, 9], 37
    fed = sum(sizes)
    g = torch.Generator(device="cuda").manual_seed(5)
    tokens, prompt, pad, enc, enc_pad = _prompts(lens, max(lens) + fed, Le, g)
    got = []
    with torch.no_grad():
        cache = model.new_cache(len(lens), 100)
        model(prompt.to(dtype), encoder_out=enc.to(dtype), padding_mask=pad, encoder_padding_mask=enc_pad, cache=cache)
        t = 0
        for T in sizes:
            chunk = torch.stack([tokens[b, n + t:n + t + T] for b, n in enumerate(lens)])
            got.append(model(chunk.to(dtype), encoder_padding_mask=enc_pad, cache=cache))
            t += T
        want = [ref(tokens[b:b + 1, :n + fed], encoder_out=enc[b:b + 1], encoder_padding_mask=enc_pad[b:b + 1])[0, n:]
                for b, n in enumerate(lens)]
    layers = len(model.layers)
    expect = []
    for T in sizes:   # per layer: the self-attention (with seqlens), then the encoder attention
        expect += [("decode" if T == 1 else "chunk", True), ("decode" if T == 1 else "chunk", False)] * layers
    assert calls == expect
    tol = 2e-2 if dtype == torch.float16 else 6e-2
    y = torch.cat(got, 1)
    for b in range(len(lens)):
        for i in range(fed):
            rel = ((y[b, i].float() - want[b][i]).norm() / want[b][i].norm()).item()
            assert rel < tol, (b, i, rel)
    assert cache.seqlens.tolist() == [n + fed for n in lens] and cache.max_len == max(lens) + fed


def test_decoder_chunk_does_not_synchronise():
    _ops()
    _, model = _decoder_pair(torch.float16, False)
    lens = [24, 13, 19]
    g = torch.Generator(device="cuda").manual_seed(6)
    tokens, prompt, pad, enc, enc_pad = _prompts(lens, 40, 40, g)
    tokens, prompt, enc = tokens.half(), prompt.half(), enc.half()
    with torch.no_grad():
        cache = model.new_cache(len(lens), 64)
        model(prompt, encoder_out=enc, padding_mask=pad, encoder_padding_mask=enc_pad, cache=cache)
        model(tokens[:, :4], encoder_padding_mask=enc_pad, cache=cache)   # warm-up chunk
        r = torch.tensor([1, 2, 3], dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            y = model(tokens[:, 4:10], encoder_padding_mask=enc_pad, cache=cache)
            cache.rewind(r)
            cache.rewind(1)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    assert y.shape == (3, 6, 768) and bool(torch.isfinite(y).all())


# ---- 6. binding rejections ----------------------------------------------------------------------------------------
def _valid():
    q = torch.randn(2, 4, 2, 64, device="cuda").half()
    k = torch.randn(2, 21, 2, 64, device="cuda").half()
    lens = torch.tensor([3, 4], dtype=torch.int32, device="cuda")
    bias = torch.randn(2, 2, 4, 24, device="cuda").half()
    kpm = torch.zeros(2, 21, dtype=torch.bool, device="cuda")
    return [q, k, k.clone(), lens, 8, q.clone(), q.clone(), bias, kpm, 0.125]


def _nc(t):
    s = torch.empty(*t.shape, 2, dtype=t.dtype, device=t.device)[..., 0]
    s.copy_(t)
    return s


def _mis(t):
    buf = torch.empty(t.numel() + 16, dtype=t.dtype, device=t.device)
    v = buf[1:1 + t.numel()].view(t.shape)
    v.copy_(t)
    return v


MUTATE = {"cpu": lambda t: t.cpu(), "dtype": lambda t: t.to(torch.int16), "small": lambda t: t.reshape(-1)[:-1].clone(),
          "nc": _nc, "mis": _mis}
OPERANDS = {0: ("q", ("cpu", "dtype", "small", "mis")), 1: ("k_cache", ("cpu", "dtype", "small", "mis")),
            2: ("v_cache", ("cpu", "dtype", "small", "mis")), 3: ("seqlens", ("cpu", "dtype", "small", "nc")),
            5: ("k_new", ("cpu", "dtype", "small", "mis")), 6: ("v_new", ("cpu", "dtype", "small", "mis")),
            7: ("bias", ("cpu", "dtype", "small", "nc", "mis")),
            8: ("key_padding_mask", ("cpu", "dtype", "small", "nc"))}


def test_binding_rejects_bad_operands():
    _kv().fmha_kvcache_fwd(*_valid())   # the builder is valid
    torch.cuda.synchronize()
    for i, (label, kinds) in OPERANDS.items():
        for kind in kinds:
            args = _valid()
            args[i] = MUTATE[kind](args[i])
            with pytest.raises(RuntimeError, match=r"\b" + re.escape(label) + " must"):
                _kv().fmha_kvcache_fwd(*args)


def test_binding_rejects_bad_shapes_and_capacity():
    fn = _kv().fmha_kvcache_fwd
    q, k, v, lens, _, kn, vn, bias, kpm, scale = _valid()
    with pytest.raises(RuntimeError, match="T >= 2"):
        fn(q[:, :1], k, v, lens, 8, kn[:, :1], vn[:, :1], None, None, scale)
    with pytest.raises(RuntimeError, match="k_new must have sizes"):
        fn(q, k, v, lens, 8, kn[:, :3], vn, None, None, scale)
    with pytest.raises(RuntimeError, match="k_cache must have sizes"):
        fn(q, k[:, :, :1], v, lens, 8, kn, vn, None, None, scale)
    with pytest.raises(RuntimeError, match="capacity"):
        fn(q, k, v, lens, 18, kn, vn, None, None, scale)   # 18 + 4 > 21
    with pytest.raises(RuntimeError, match="multiple of 8"):
        fn(q, k, v, lens, 8, kn, vn, bias[..., :20].contiguous(), None, scale)
    with pytest.raises(RuntimeError, match="column for every key"):
        fn(q, k, v, lens, 8, kn, vn, bias[..., :8].contiguous(), None, scale)
    with pytest.raises(RuntimeError, match="append"):
        fn(q, k, v, lens, 8, None, None, None, None, scale)
    with pytest.raises(ValueError, match="capacity"):
        _ops().attention_with_kv_cache(q, k, v, lens, 18, k_new=kn, v_new=vn)
    with pytest.raises(ValueError, match="appends"):
        _ops().attention_with_kv_cache(q, k, v, lens, 8)
