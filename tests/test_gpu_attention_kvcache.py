"""Decode attention against a key / value cache (``fmha_decode``, ``ops.attention_with_kv_cache``) and incremental
decoding with ``TransformerDecoder`` on it.

Checked: the op against the fp64 ``attention_with_kv_cache_reference`` at every head-dim tier, ragged lengths from 1 to
4097 in one batch, shared and per-batch bias rows wider than the visible keys, key padding with a fully masked row;
the append (row ``seqlens[b]`` bitwise equal to the new key / value, every other row bitwise untouched, the new key
attended) from strided views of a packed ``[B, 1, 3, H, D]`` projection; forced split counts (agreement within the
fp32 combine, bitwise repeatable), a grid of several waves and a host bound far above the true lengths; a decoder step
without a host synchronisation; and whole decodes in fp16 / bf16 against an fp32 copy of the model run on each
sequence alone.
"""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]
DT_IDS = ["fp16", "bf16"]
UNIT = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
HEAD_DIMS = [8, 16, 40, 64, 96, 128]
LENS = [1, 2, 63, 64, 65, 127, 1000, 4097]   # one batch, ragged


def _ops():
    from unicore import ops

    assert ops.USE_NATIVE, "native kernels must be active on the GPU box"
    return ops


def _cache(B, C, H, D, dtype, g):
    k = (torch.randn(B, C, H, D, device="cuda", generator=g) * 0.6).to(dtype)
    v = torch.randn(B, C, H, D, device="cuda", generator=g).to(dtype)
    return k, v


def _bound(q, k, v, seqlens, max_len, k_new, v_new, bias, kpm, scale, dtype):
    """fp64 reference O and its error bound: the 16-bit rounding of O plus fp32 terms of sum_k p_k |v_k|."""
    ops = _ops()
    d = lambda t: None if t is None else t.double()   # noqa: E731
    kc, vc = k.double(), v.double()
    ref = ops.attention_with_kv_cache_reference(d(q), kc, vc, seqlens, max_len, d(k_new), d(v_new), d(bias), kpm,
                                                scale)
    kc, vc = k.double(), v.double()
    mag = ops.attention_with_kv_cache_reference(d(q), kc, vc.abs(), seqlens, max_len, d(k_new),
                                                None if v_new is None else v_new.double().abs(), d(bias), kpm, scale)
    return ref, UNIT[dtype] * ref.abs() + 2.0 ** -13 * mag


def _assert_within(got, ref, bound, what):
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)
    if bad.any():
        i = bad.nonzero()[0].tolist()
        raise AssertionError("{}: {} elements out of bound, first at {}: got {}, want {} +- {}".format(
            what, int(bad.sum()), i, got[tuple(i)].item(), ref[tuple(i)].item(), bound[tuple(i)].item()))


# ---- 1. op against fp64 --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("masked", [False, True], ids=["nomask", "kpm"])
@pytest.mark.parametrize("bias_mode", ["none", "shared", "batch"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("D", HEAD_DIMS)
def test_op_against_fp64(D, dtype, bias_mode, masked):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(D)
    B, H, C = len(LENS), 2, 4104
    max_len = max(LENS)
    k, v = _cache(B, C, H, D, dtype, g)
    q = (torch.randn(B, 1, H, D, device="cuda", generator=g) * 0.6).to(dtype)
    seqlens = torch.tensor(LENS, dtype=torch.int32, device="cuda")
    Lb = max_len + 5
    bias = None
    if bias_mode != "none":
        bias = torch.randn(B if bias_mode == "batch" else 1, H, 1, Lb, device="cuda", generator=g).to(dtype)
    kpm = None
    if masked:
        kpm = torch.zeros(B, C, dtype=torch.bool, device="cuda")
        kpm[0, 0] = True            # length 1, fully masked: O = 0
        kpm[5, 3:90] = True
        kpm[7, 1000:3000] = True
    scale = D ** -0.5
    out = ops.attention_with_kv_cache(q, k, v, seqlens, max_len, bias=bias, key_padding_mask=kpm, scale=scale)
    ref, bound = _bound(q, k, v, seqlens, max_len, None, None, bias, kpm, scale, dtype)
    assert out.shape == (B, 1, H, D) and out.dtype == dtype
    _assert_within(out, ref, bound, "O")
    if masked:
        assert torch.equal(out[0], torch.zeros_like(out[0]))


# ---- 2. append, from the packed projection --------------------------------------------------------------------------
@pytest.mark.parametrize("num_splits", [1, 3])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("D", HEAD_DIMS)
def test_append_from_packed_projection(D, dtype, num_splits):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(100 + D)
    lens = [0, 5, 64, 300, 1023]
    B, H, C = len(lens), 3, 1024
    k, v = _cache(B, C, H, D, dtype, g)
    for b, n in enumerate(lens):   # a NaN sentinel in every row that is not visible before the append
        k[b, n:] = float("nan")
        v[b, n:] = float("nan")
    k0, v0 = k.clone(), v.clone()
    qkv = (torch.randn(B, 1, 3, H, D, device="cuda", generator=g) * 0.6).to(dtype)
    q, k_new, v_new = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]   # strided views [B, 1, H, D]
    assert not q.is_contiguous()
    seqlens = torch.tensor(lens, dtype=torch.int32, device="cuda")
    scale = D ** -0.5
    out = ops.native().fmha_decode(q, k, v, seqlens, max(lens), k_new, v_new, None, None, scale, num_splits)
    for b, n in enumerate(lens):
        assert torch.equal(k[b, n].view(torch.int16), k_new[b, 0].view(torch.int16))
        assert torch.equal(v[b, n].view(torch.int16), v_new[b, 0].view(torch.int16))
        k0[b, n], v0[b, n] = k_new[b, 0], v_new[b, 0]
    assert torch.equal(k.view(torch.int16), k0.view(torch.int16)) and torch.equal(v.view(torch.int16), v0.view(torch.int16))
    # the reference on the appended caches: the new row is the last visible key
    ref, bound = _bound(q, k, v, seqlens + 1, None, None, None, None, None, scale, dtype)
    _assert_within(out, ref, bound, "O")
    # without the new key the result would differ (batch 0 sees nothing else)
    assert torch.allclose(out[0].double(), v_new[0].double(), atol=UNIT[dtype] * 4, rtol=UNIT[dtype] * 4)
    # the op appends the same way
    k2, v2 = k0.clone(), v0.clone()
    for b, n in enumerate(lens):
        k2[b, n] = v2[b, n] = float("nan")
    out2 = ops.attention_with_kv_cache(q, k2, v2, seqlens, max(lens), k_new=k_new, v_new=v_new, scale=scale)
    assert torch.equal(k2.view(torch.int16), k0.view(torch.int16))
    _assert_within(out2, ref, bound, "O (op)")


# ---- 3. split counts ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", ["ragged", "multi_wave", "loose_bound"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_split_counts(shape, dtype):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(7)
    D = 64
    if shape == "ragged":
        B, H, C, lens, max_len = 4, 2, 4200, [4097, 1, 650, 2000], 4097
    elif shape == "multi_wave":    # 64 * 12 * 7 CTAs: several waves on any H100
        B, H, C, max_len = 64, 12, 520, 512
        lens = torch.randint(1, 513, (B,), generator=torch.Generator().manual_seed(0)).tolist()
    else:                          # a host bound far above the true lengths: most splits are empty
        B, H, C, lens, max_len = 3, 4, 8192, [5, 40, 17], 8191
    k, v = _cache(B, C, H, D, dtype, g)
    q = (torch.randn(B, 1, H, D, device="cuda", generator=g) * 0.6).to(dtype)
    bias = torch.randn(1, H, 1, max_len, device="cuda", generator=g).to(dtype)
    seqlens = torch.tensor(lens, dtype=torch.int32, device="cuda")
    scale = D ** -0.5
    ref, bound = _bound(q, k, v, seqlens, max_len, None, None, bias, None, scale, dtype)
    outs = {}
    for s in [0, 1, 2, 7, ops.native().fmha_decode_max_splits()]:
        a = ops.native().fmha_decode(q, k, v, seqlens, max_len, None, None, bias, None, scale, s)
        b = ops.native().fmha_decode(q, k, v, seqlens, max_len, None, None, bias, None, scale, s)
        assert torch.equal(a.view(torch.int16), b.view(torch.int16)), "num_splits={} is not repeatable".format(s)
        _assert_within(a, ref, bound, "O, num_splits={}".format(s))
        outs[s] = a
    # any two split counts differ only by the fp32 combine: at most a few units of the 16-bit result
    for s, o in outs.items():
        _assert_within(o, outs[1].double(), 2 * bound + UNIT[dtype] * outs[1].double().abs(), "splits {} vs 1".format(s))


def test_bad_arguments():
    ops = _ops()
    q = torch.randn(2, 1, 2, 64, device="cuda").half()
    k = torch.randn(2, 16, 2, 64, device="cuda").half()
    lens = torch.tensor([3, 4], dtype=torch.int32, device="cuda")
    with pytest.raises(RuntimeError, match="capacity"):
        ops.native().fmha_decode(q, k, k.clone(), lens, 16, q, q, None, None, 0.125, 0)
    with pytest.raises(RuntimeError, match="num_splits"):
        ops.native().fmha_decode(q, k, k.clone(), lens, 8, None, None, None, None, 0.125, 100000)
    with pytest.raises(RuntimeError, match="bias"):
        ops.native().fmha_decode(q, k, k.clone(), lens, 8, None, None, torch.zeros(1, 2, 1, 4, device="cuda").half(),
                                 None, 0.125, 0)
    with pytest.raises(ValueError, match="capacity"):
        ops.attention_with_kv_cache(q, k, k.clone(), lens, 16, k_new=q, v_new=q)


# ---- 4. decoder ---------------------------------------------------------------------------------------------------
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
def test_decoder_steps_match_fp32_full_forward(dtype, post_ln, monkeypatch):
    import unicore_b200.ops.attention_ops as attention_ops

    ops = _ops()
    ref, model = _decoder_pair(dtype, post_ln)
    real = ops.native()
    calls = []

    class Spy:
        def __getattr__(self, name):
            return getattr(real, name)

        def fmha_decode(self, *args, **kwargs):
            calls.append(args[3] is not None)   # self-attention steps pass seqlens
            return real.fmha_decode(*args, **kwargs)

    monkeypatch.setattr(attention_ops, "native", lambda: Spy())
    lens, steps, Le = [24, 13, 19], 40, 40
    g = torch.Generator(device="cuda").manual_seed(5)
    tokens, prompt, pad, enc, enc_pad = _prompts(lens, max(lens) + steps, Le, g)
    got = []
    with torch.no_grad():
        cache = model.new_cache(len(lens), 128)
        model(prompt.to(dtype), encoder_out=enc.to(dtype), padding_mask=pad, encoder_padding_mask=enc_pad, cache=cache)
        for t in range(steps):
            tok = torch.stack([tokens[b, n + t] for b, n in enumerate(lens)])[:, None]
            got.append(model(tok.to(dtype), encoder_padding_mask=enc_pad, cache=cache)[:, 0])
        want = []
        for t in range(steps):
            want.append(torch.stack([
                ref(tokens[b:b + 1, :n + t + 1], encoder_out=enc[b:b + 1], encoder_padding_mask=enc_pad[b:b + 1])[0, -1]
                for b, n in enumerate(lens)]))
    assert len(calls) == steps * 2 * len(model.layers)
    assert sum(calls) == steps * len(model.layers)
    tol = 2e-2 if dtype == torch.float16 else 6e-2
    for t in range(steps):
        rel = ((got[t].float() - want[t]).norm() / want[t].norm()).item()
        assert rel < tol, (t, rel)
    assert cache.seqlens.tolist() == [n + steps for n in lens] and cache.max_len == max(lens) + steps


def test_decoder_step_does_not_synchronise():
    _ops()
    _, model = _decoder_pair(torch.float16, False)
    lens = [24, 13, 19]
    g = torch.Generator(device="cuda").manual_seed(6)
    tokens, prompt, pad, enc, enc_pad = _prompts(lens, 30, 40, g)
    tokens, prompt, enc = tokens.half(), prompt.half(), enc.half()
    with torch.no_grad():
        cache = model.new_cache(len(lens), 64)
        model(prompt, encoder_out=enc, padding_mask=pad, encoder_padding_mask=enc_pad, cache=cache)
        model(tokens[:, :1], encoder_padding_mask=enc_pad, cache=cache)   # warm-up step
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            y = model(tokens[:, 1:2], encoder_padding_mask=enc_pad, cache=cache)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    assert y.shape == (3, 1, 768) and bool(torch.isfinite(y).all())
