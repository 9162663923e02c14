"""Decoding steps captured in CUDA graphs: the length-split mode of ``fmha_decode`` and
``TransformerDecoder.capture_step``.

Checked: ``split_by_length`` against the fp64 ``attention_with_kv_cache_reference`` with a host bound at the capacity
(ragged lengths from 0 to C - 1, appending or not, bias and key mask, NaN in every row past n_b, forced and heuristic
split counts, a grid of several waves), bitwise repeatable, bitwise equal to the host-bound partition when every length
equals the bound, and the append (row n_b bitwise the new key / value, every other row untouched).  Then captured
steps of a 2-layer decoder with relative positions, cross-attention and an encoder padding mask against eager steps
from the same state: 24 one-token steps with greedy tokens, bitwise repeatable replays, ``reorder`` / ``rewind``
between replays, new prefills (same shapes: no new capture; another encoder length: one), 4-token chunks, a
decoder-only model, and a full cache that raises before the replay.
"""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]
DT_IDS = ["fp16", "bf16"]
UNIT = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
STEP_TOL = {torch.float16: 2e-2, torch.bfloat16: 6e-2}   # relative norm per step, as the eager decoder tests


def _ops():
    from unicore import ops

    assert ops.USE_NATIVE, "native kernels must be active on the GPU box"
    return ops


def _bits(t):
    return t.view(torch.int16)


def _bound(q, k, v, seqlens, max_len, k_new, v_new, bias, kpm, scale, dtype):
    """fp64 reference O and its error bound: the 16-bit rounding of O plus fp32 terms of sum_k p_k |v_k|."""
    ops = _ops()
    d = lambda t: None if t is None else t.double()   # noqa: E731
    ref = ops.attention_with_kv_cache_reference(d(q), k.double(), v.double(), seqlens, max_len, d(k_new), d(v_new),
                                                d(bias), kpm, scale)
    mag = ops.attention_with_kv_cache_reference(d(q), k.double(), v.double().abs(), seqlens, max_len, d(k_new),
                                                None if v_new is None else v_new.double().abs(), d(bias), kpm, scale)
    return ref, UNIT[dtype] * ref.abs() + 2.0 ** -13 * mag


def _assert_within(got, ref, bound, what):
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)
    if bad.any():
        i = bad.nonzero()[0].tolist()
        raise AssertionError("{}: {} elements out of bound, first at {}: got {}, want {} +- {}".format(
            what, int(bad.sum()), i, got[tuple(i)].item(), ref[tuple(i)].item(), bound[tuple(i)].item()))


def _decode_case(B, H, C, D, lens, dtype, seed, append):
    g = torch.Generator(device="cuda").manual_seed(seed)
    k = (torch.randn(B, C, H, D, device="cuda", generator=g) * 0.6).to(dtype)
    v = torch.randn(B, C, H, D, device="cuda", generator=g).to(dtype)
    for b, n in enumerate(lens):   # rows past the visible keys are never read: a NaN there must not matter
        k[b, n:] = float("nan")
        v[b, n:] = float("nan")
    qkv = (torch.randn(B, 1, 3, H, D, device="cuda", generator=g) * 0.6).to(dtype)
    q, k_new, v_new = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    bias = torch.randn(B, H, 1, C, device="cuda", generator=g).to(dtype)
    kpm = torch.rand(B, C, device="cuda", generator=g) < 0.2
    seqlens = torch.tensor(lens, dtype=torch.int32, device="cuda")
    return q, k, v, (k_new, v_new) if append else (None, None), bias, kpm, seqlens


# ---- 1. the length-split mode of the kernel -------------------------------------------------------------------------
@pytest.mark.parametrize("num_splits", [1, 3, 0], ids=["s1", "s3", "heuristic"])
@pytest.mark.parametrize("append", [False, True], ids=["read", "append"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("D", [8, 64, 96, 128])
def test_split_by_length_against_fp64(D, dtype, append, num_splits):
    ops = _ops()
    C = 1024
    lens = [0, 1, 100, 511, 700, C - 1]
    B, H = len(lens), 2
    q, k, v, (k_new, v_new), bias, kpm, seqlens = _decode_case(B, H, C, D, lens, dtype, D, append)
    max_len = C - 1 if append else C   # the bound a captured step runs with: the capacity
    k0, v0 = k.clone(), v.clone()
    scale = D ** -0.5
    ref, bound = _bound(q, k0.clone(), v0.clone(), seqlens, max_len, k_new, v_new, bias, kpm, scale, dtype)
    outs = []
    for _ in range(2):
        k1, v1 = k0.clone(), v0.clone()
        outs.append(ops.native().fmha_decode(q, k1, v1, seqlens, max_len, k_new, v_new, bias, kpm, scale, num_splits,
                                             split_by_length=True))
    assert torch.equal(_bits(outs[0]), _bits(outs[1])), "not bitwise repeatable"
    _assert_within(outs[0], ref, bound, "O")
    if append:   # row n_b is bitwise the new key / value, every other row is untouched
        for b, n in enumerate(lens):
            assert torch.equal(_bits(k1[b, n]), _bits(k_new[b, 0])) and torch.equal(_bits(v1[b, n]), _bits(v_new[b, 0]))
            k0[b, n], v0[b, n] = k_new[b, 0], v_new[b, 0]
    assert torch.equal(_bits(k1), _bits(k0)) and torch.equal(_bits(v1), _bits(v0))


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_split_by_length_multi_wave(dtype):
    ops = _ops()
    B, H, C, D = 64, 12, 520, 64   # 64 * 12 * 7 CTAs: several waves on any H100
    lens = torch.randint(0, C, (B,), generator=torch.Generator().manual_seed(0)).tolist()
    q, k, v, (k_new, v_new), bias, kpm, seqlens = _decode_case(B, H, C, D, lens, dtype, 11, True)
    scale = D ** -0.5
    ref, bound = _bound(q, k.clone(), v.clone(), seqlens, C - 1, k_new, v_new, bias, kpm, scale, dtype)
    out = ops.native().fmha_decode(q, k, v, seqlens, C - 1, k_new, v_new, bias, kpm, scale, 7, split_by_length=True)
    _assert_within(out, ref, bound, "O")


@pytest.mark.parametrize("append", [False, True], ids=["read", "append"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("D", [64, 128])
def test_split_by_length_equals_host_partition_at_the_bound(D, dtype, append):
    ops = _ops()
    B, H, C, n = 4, 3, 1500, 1234
    lens = [n - 1 if append else n] * B
    q, k, v, (k_new, v_new), bias, kpm, seqlens = _decode_case(B, H, C, D, lens, dtype, 3 + D, append)
    for s in [1, 3, 7, 0]:
        got = {}
        for mode in (False, True):
            k1, v1 = k.clone(), v.clone()
            got[mode] = ops.native().fmha_decode(q, k1, v1, seqlens, lens[0], k_new, v_new, bias, kpm, D ** -0.5, s,
                                                 split_by_length=mode)
        assert torch.equal(_bits(got[False]), _bits(got[True])), "num_splits={}".format(s)


# ---- 2. captured decoder steps --------------------------------------------------------------------------------------
E, HEADS, VOCAB = 256, 4, 16
LENS = [12, 5, 9]


def _decoder(dtype, layers=2, seed=0):
    from unicore.modules import TransformerDecoder

    torch.manual_seed(seed)
    m = TransformerDecoder(decoder_layers=layers, embed_dim=E, ffn_embed_dim=2 * E, attention_heads=HEADS,
                           max_seq_len=128).cuda().eval()
    with torch.no_grad():
        for p in m.parameters():   # non-trivial LayerNorm and bias parameters
            p.add_(torch.randn_like(p) * 0.02)
    return m.to(dtype)


def _inputs(dtype, seed, lens=LENS, Le=10):
    g = torch.Generator(device="cuda").manual_seed(seed)
    B, L = len(lens), max(lens)
    prompt = torch.randn(B, L, E, device="cuda", generator=g).to(dtype)
    pad = torch.ones(B, L, dtype=torch.bool, device="cuda")
    for b, n in enumerate(lens):
        pad[b, :n] = False
    enc = torch.randn(B, Le, E, device="cuda", generator=g).to(dtype)
    enc_pad = torch.zeros(B, Le, dtype=torch.bool, device="cuda")
    enc_pad[0, Le - 3:] = True
    table = (torch.randn(VOCAB, E, device="cuda", generator=g) * 0.5).to(dtype)
    return prompt, pad, enc, enc_pad, table


def _prefill(m, cache, prompt, pad, enc, enc_pad):
    with torch.no_grad():
        m(prompt, encoder_out=enc, padding_mask=pad, encoder_padding_mask=enc_pad, cache=cache)


def _assert_close_step(got, want, dtype, what):
    rel = ((got.float() - want.float()).norm() / want.float().norm()).item()
    assert rel < STEP_TOL[dtype], (what, rel)


def _cache_state(cache):
    return [cache.seqlens] + [t for lc in cache.layers for t in (lc.k, lc.v, lc.enc_k, lc.enc_v) if t is not None]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_captured_greedy_steps_match_eager(dtype):
    _ops()
    m = _decoder(dtype)
    prompt, pad, enc, enc_pad, table = _inputs(dtype, 1)
    cache = m.new_cache(3, 64)
    _prefill(m, cache, prompt, pad, enc, enc_pad)
    eager = copy.deepcopy(cache)
    step = m.capture_step(cache, encoder_padding_mask=enc_pad)
    y = torch.zeros(3, E, device="cuda", dtype=dtype)
    with torch.no_grad():
        for t in range(24):
            logits = (y.float() @ table.float().t()) if t else torch.zeros(3, VOCAB, device="cuda")
            tok = logits.argmax(-1)   # the eager arm's greedy token feeds both arms
            emb = table[tok][:, None]
            want = m(emb, encoder_padding_mask=enc_pad, cache=eager)[:, 0]
            got = step(emb)[:, 0].clone()
            _assert_close_step(got, want, dtype, t)
            lw, lg = want.float() @ table.float().t(), got.float() @ table.float().t()
            top2 = lw.topk(2, -1).values
            clear = (top2[:, 0] - top2[:, 1]) > 1e-2 * top2[:, 0].abs().clamp(min=1)   # not a near-tie
            assert torch.equal(lg.argmax(-1)[clear], lw.argmax(-1)[clear]), t
            y = want
    assert step.captures == 1
    assert cache.max_len == eager.max_len == max(LENS) + 24
    assert torch.equal(cache.seqlens, eager.seqlens)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_replays_are_bitwise_repeatable(dtype):
    _ops()
    m = _decoder(dtype)
    prompt, pad, enc, enc_pad, _ = _inputs(dtype, 2)
    cache = m.new_cache(3, 64)
    _prefill(m, cache, prompt, pad, enc, enc_pad)
    saved, max_len = [t.clone() for t in _cache_state(cache)], cache.max_len
    toks = torch.randn(8, 3, 1, E, device="cuda", generator=torch.Generator(device="cuda").manual_seed(3)).to(dtype)
    step = m.capture_step(cache, encoder_padding_mask=enc_pad)
    runs = []
    for _ in range(2):
        for t, s in zip(_cache_state(cache), saved):   # back to the same state, in place
            t.copy_(s)
        cache.max_len = max_len
        with torch.no_grad():
            runs.append(torch.stack([step(toks[i]).clone() for i in range(8)]))
    assert torch.equal(_bits(runs[0]), _bits(runs[1]))
    assert step.captures == 1


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_reorder_rewind_and_prefill_between_replays(dtype):
    _ops()
    m = _decoder(dtype)
    prompt, pad, enc, enc_pad, _ = _inputs(dtype, 4)
    cache = m.new_cache(3, 64)
    _prefill(m, cache, prompt, pad, enc, enc_pad)
    eager = copy.deepcopy(cache)
    step = m.capture_step(cache, encoder_padding_mask=enc_pad)
    g = torch.Generator(device="cuda").manual_seed(5)

    def run(n, mask, what):
        with torch.no_grad():
            for i in range(n):
                emb = torch.randn(3, 1, E, device="cuda", generator=g).to(dtype)
                want = m(emb, encoder_padding_mask=mask, cache=eager)
                _assert_close_step(step(emb, encoder_padding_mask=mask), want, dtype, (what, i))
        assert torch.equal(cache.seqlens, eager.seqlens) and cache.max_len == eager.max_len

    run(3, enc_pad, "start")
    index = torch.tensor([2, 0, 2], device="cuda")
    for c in (cache, eager):
        c.reorder(index)
    run(3, enc_pad[index], "reorder")
    for c in (cache, eager):
        c.rewind(2)
    run(2, enc_pad[index], "rewind int")
    back = torch.tensor([1, 0, 3], device="cuda")
    for c in (cache, eager):
        c.rewind(back)
    run(2, enc_pad[index], "rewind tensor")
    assert step.captures == 1
    # a new prefill of the same shapes writes into the same buffers: no new capture
    prompt2, pad2, enc2, enc_pad2, _ = _inputs(dtype, 6)
    for c in (cache, eager):
        c.rewind(c.max_len)
        _prefill(m, c, prompt2, pad2, enc2, enc_pad2)
    run(3, enc_pad2, "prefill")
    assert step.captures == 1
    # another encoder length: the encoder keys / values are new tensors, and the step captures once more
    prompt3, pad3, enc3, enc_pad3, _ = _inputs(dtype, 7, Le=14)
    for c in (cache, eager):
        c.rewind(c.max_len)
        _prefill(m, c, prompt3, pad3, enc3, enc_pad3)
    run(3, enc_pad3, "encoder length")
    assert step.captures == 2


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_captured_chunk_steps_match_eager(dtype):
    _ops()
    m = _decoder(dtype)
    prompt, pad, enc, enc_pad, _ = _inputs(dtype, 8)
    cache = m.new_cache(3, 61)   # a capacity that is not a multiple of 8: the chunk bias is 64 wide
    _prefill(m, cache, prompt, pad, enc, enc_pad)
    eager = copy.deepcopy(cache)
    step = m.capture_step(cache, T=4, encoder_padding_mask=enc_pad)
    g = torch.Generator(device="cuda").manual_seed(9)
    with torch.no_grad():
        for i in range(5):
            emb = torch.randn(3, 4, E, device="cuda", generator=g).to(dtype)
            want = m(emb, encoder_padding_mask=enc_pad, cache=eager)
            got = step(emb)
            assert got.shape == (3, 4, E)
            _assert_close_step(got, want, dtype, i)
    assert torch.equal(cache.seqlens, eager.seqlens) and cache.max_len == eager.max_len == max(LENS) + 20
    assert step.captures == 1


def test_decoder_only_model():
    _ops()
    dtype = torch.float16
    m = _decoder(dtype)
    prompt, pad, _, _, _ = _inputs(dtype, 10)
    cache = m.new_cache(3, 40)
    with torch.no_grad():
        m(prompt, padding_mask=pad, cache=cache)
    assert cache.layers[0].enc_k is None
    eager = copy.deepcopy(cache)
    step = m.capture_step(cache)
    g = torch.Generator(device="cuda").manual_seed(11)
    with torch.no_grad():
        for i in range(6):
            emb = torch.randn(3, 1, E, device="cuda", generator=g).to(dtype)
            _assert_close_step(step(emb), m(emb, cache=eager), dtype, i)


def test_full_cache_raises_before_the_replay():
    _ops()
    dtype = torch.float16
    m = _decoder(dtype)
    prompt, pad, enc, enc_pad, _ = _inputs(dtype, 12)
    C = max(LENS) + 3
    cache = m.new_cache(3, C)
    _prefill(m, cache, prompt, pad, enc, enc_pad)
    step = m.capture_step(cache, encoder_padding_mask=enc_pad)
    chunk = m.capture_step(cache, T=2, encoder_padding_mask=enc_pad)
    emb = torch.randn(3, 1, E, device="cuda", dtype=dtype)
    with torch.no_grad():
        step(emb)
        step(emb)   # max_len = C - 1: one more token fits, a chunk of two does not
        with pytest.raises(ValueError, match="capacity"):
            chunk(torch.randn(3, 2, E, device="cuda", dtype=dtype))
        assert chunk.captures == 0
        step(emb)
        assert cache.max_len == C
        before = [t.clone() for t in _cache_state(cache)]
        with pytest.raises(ValueError, match="capacity"):
            step(emb)
    assert cache.max_len == C and step.captures == 1
    assert all(torch.equal(a, b) for a, b in zip(_cache_state(cache), before))


def test_capture_step_refuses_dropout_and_an_empty_cache():
    _ops()
    m = _decoder(torch.float16)
    cache = m.new_cache(3, 32)
    with pytest.raises(ValueError, match="prefill"):
        m.capture_step(cache)
    prompt, pad, enc, enc_pad, _ = _inputs(torch.float16, 13)
    _prefill(m, cache, prompt, pad, enc, enc_pad)
    m.train()
    with pytest.raises(RuntimeError, match="dropout"):
        m.capture_step(cache, encoder_padding_mask=enc_pad)
