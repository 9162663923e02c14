"""Packed variable-length chunks into a key / value cache on the GPU: the KV-cache mode of the wgmma forward on packed
queries (``kvcache.fmha_kvcache_varlen_fwd``, ``ops.attention_with_kv_cache_varlen``) and ``TransformerDecoder``'s
packed prefill and steps on it.

Checked: the op against fp64 with the chunk tests' error bound at every head-dim tier, fp16 / bf16 and H_kv = H, H / 4,
1, with T_b from 0 to 200 and seqlens from 0 to near the capacity in one batch, a capacity that is not a multiple of 8,
shared and per-batch bias wider than the visible keys and a key mask with a fully masked query; every real row with
T_b >= 2 bitwise equal to ``attention_with_kv_cache`` on its sequence alone; the appended rows bitwise the new keys
and values and every other row bitwise untouched (NaN sentinels included, which reach no output); cross mode with a
key mask; out-of-range cu_seqlens / seqlens clamped as the reference clamps them; a decoder fed a packed prefill and
packed ragged steps in fp16 / bf16 against an fp32 copy run on each sequence alone, with the binding called once per
layer and attention; a captured step after a packed prefill giving the eager steps' tokens; a packed step that does not
synchronise; and the binding's operand checks.
"""
import re

import pytest
import torch

from test_gpu_attention_kvcache_chunk import DT_IDS, DTYPES, MUTATE, _assert_within, _bound, _decoder_pair

pytestmark = pytest.mark.gpu

HEAD_DIMS = [8, 64, 96, 128]
SIZES = [0, 1, 2, 63, 64, 65, 200]   # T_b of one batch
LENS = [5, 900, 0, 128, 1, 300, 777]  # seqlens of the same batch, up to max_len = C - max(T_b) - 3


def _ops():
    from unicore import ops

    assert ops.USE_NATIVE, "native kernels must be active on the GPU box"
    return ops


def _kv():
    return _ops().native().kvcache


def _cu(sizes, device="cuda"):
    return torch.tensor([0] + torch.tensor(sizes).cumsum(0).tolist(), dtype=torch.int32, device=device)


def _inputs(sizes, lens, C, H, H_kv, D, dtype, g, sentinel=True):
    """Caches with NaN rows from each sequence's length on, and the packed projection ``[N, H + 2 H_kv, D]`` whose head
    slices are q, k_new and v_new."""
    B, N = len(sizes), sum(sizes)
    k = (torch.randn(B, C, H_kv, D, device="cuda", generator=g) * 0.6).to(dtype)
    v = torch.randn(B, C, H_kv, D, device="cuda", generator=g).to(dtype)
    if sentinel:
        for b, n in enumerate(lens):
            k[b, n:] = float("nan")
            v[b, n:] = float("nan")
    qkv = (torch.randn(N, H + 2 * H_kv, D, device="cuda", generator=g) * 0.6).to(dtype)
    return k, v, qkv[:, :H], qkv[:, H:H + H_kv], qkv[:, H + H_kv:]


# ---- 1. op against fp64, bitwise against the padded call, cache contents ------------------------------------------
@pytest.mark.parametrize("case", ["plain", "bias_shared_kpm", "bias_batch"])
@pytest.mark.parametrize("kv_div", [1, 4, 0], ids=["mha", "gqa4", "mqa"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("D", HEAD_DIMS)
def test_op_against_fp64_and_padded_call(D, dtype, kv_div, case):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(D * 10 + kv_div)
    H = 8
    H_kv = H // kv_div if kv_div else 1
    B, T, max_len = len(SIZES), max(SIZES), max(LENS)
    C = max_len + T + 3   # not a multiple of 8
    k, v, q, k_new, v_new = _inputs(SIZES, LENS, C, H, H_kv, D, dtype, g)
    cu, seqlens = _cu(SIZES), torch.tensor(LENS, dtype=torch.int32, device="cuda")
    bias = kpm = None
    if case != "plain":
        Lb = max_len + T + 11   # wider than the visible keys; the op pads it to a multiple of 8
        bias = torch.randn(B if case == "bias_batch" else 1, H, T, Lb, device="cuda", generator=g).to(dtype)
    if case == "bias_shared_kpm":
        kpm = torch.zeros(B, C, dtype=torch.bool, device="cuda")
        kpm[2, 0] = True   # length 0: query 0 sees only key 0, which is masked -> O = 0
        kpm[3, 3:90] = True
        kpm[1, 500:900] = True
    scale = D ** -0.5
    k0, v0 = k.clone(), v.clone()
    out = ops.attention_with_kv_cache_varlen(q, k, v, cu, T, seqlens, max_len, k_new=k_new, v_new=v_new, bias=bias,
                                             key_padding_mask=kpm, scale=scale)
    assert out.shape == (sum(SIZES), H, D) and out.dtype == dtype
    assert bool(torch.isfinite(out).all())
    i16 = lambda t: t.view(torch.int16)   # noqa: E731
    for b, (n, t) in enumerate(zip(LENS, SIZES)):
        s = int(sum(SIZES[:b]))
        # cache contents: the T_b new rows bitwise, every other row (NaN sentinels included) untouched
        k0[b, n:n + t], v0[b, n:n + t] = k_new[s:s + t], v_new[s:s + t]
        if t == 0:
            continue
        bb = b if case == "bias_batch" else 0
        args = (q[None, s:s + t], k[b:b + 1], v[b:b + 1], seqlens[b:b + 1], max_len, k_new[None, s:s + t],
                v_new[None, s:s + t], None if bias is None else bias[bb:bb + 1, :, :t],
                None if kpm is None else kpm[b:b + 1])
        # the oracle appends again: the rows it writes are the ones already there.  Its bound takes K / V with one head
        # per query head, which gives the same reference
        x = lambda t: t.repeat_interleave(H // H_kv, dim=2)   # noqa: E731
        ref, bound = _bound(args[0], x(args[1]), x(args[2]), *args[3:5], x(args[5]), x(args[6]), *args[7:], scale,
                            dtype)
        _assert_within(out[None, s:s + t], ref, bound, "O of sequence {}".format(b))
        if t >= 2:   # the padded chunk kernel on this sequence alone, into copies of its caches
            kb, vb = k0[b:b + 1].clone(), v0[b:b + 1].clone()
            kb[0, n:n + t], vb[0, n:n + t] = float("nan"), float("nan")
            one = ops.attention_with_kv_cache(args[0], kb, vb, *args[3:], scale=scale)
            assert torch.equal(i16(out[s:s + t]), i16(one[0])), "sequence {} differs from the padded call".format(b)
    assert torch.equal(i16(k), i16(k0)) and torch.equal(i16(v), i16(v0))
    if case == "bias_shared_kpm":
        assert torch.equal(out[1], torch.zeros_like(out[1]))   # sequence 2's first query: every key masked


# ---- 2. cross mode, clamps --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("D", [16, 96])
def test_cross_attention_with_key_mask(D, dtype):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(D)
    sizes, S, H = [37, 0, 5, 70], 203, 4
    k, v, q, _, _ = _inputs(sizes, [S] * 4, S, H, H, D, dtype, g, sentinel=False)
    cu = _cu(sizes)
    bias = torch.randn(4, H, 70, 208, device="cuda", generator=g).to(dtype)
    kpm = torch.zeros(4, S, dtype=torch.bool, device="cuda")
    kpm[0, 150:] = True
    kpm[3] = True   # every key masked: O = 0
    scale = D ** -0.5
    out = ops.attention_with_kv_cache_varlen(q, k, v, cu, 70, bias=bias, key_padding_mask=kpm, scale=scale)
    for b, t in enumerate(sizes):
        s = int(sum(sizes[:b]))
        if t:
            ref, bound = _bound(q[None, s:s + t], k[b:b + 1], v[b:b + 1], None, None, None, None,
                                bias[b:b + 1, :, :t], kpm[b:b + 1], scale, dtype)
            _assert_within(out[None, s:s + t], ref, bound, "O of sequence {}".format(b))
    assert torch.equal(out[42:], torch.zeros_like(out[42:]))


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_out_of_range_lengths_are_clamped(dtype):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(3)
    C, H, D, N = 77, 2, 64, 30
    cu = torch.tensor([0, 12, 12, 1 << 20, 1 << 20], dtype=torch.int32, device="cuda")   # {0,9}, {12,0}, {12,9}, {30,0}
    seqlens = torch.tensor([-5, 72, 70, 1 << 30], dtype=torch.int32, device="cuda")   # partly or wholly past C
    k, v, q, k_new, v_new = _inputs([N], [0], C, H, H, D, dtype, g, sentinel=False)
    k, v = k.expand(4, C, H, D).clone(), v.expand(4, C, H, D).clone()
    kd, vd = k.double(), v.double()
    out = ops.attention_with_kv_cache_varlen(q, k, v, cu, 9, seqlens, C - 9, k_new=k_new, v_new=v_new,
                                             scale=D ** -0.5)
    ref = ops.attention_with_kv_cache_varlen_reference(q.double(), kd, vd, cu, 9, seqlens, C - 9,
                                                       k_new=k_new.double(), v_new=v_new.double(), scale=D ** -0.5)
    i16 = lambda t: t.view(torch.int16)   # noqa: E731
    assert torch.equal(i16(k), i16(kd.to(dtype))) and torch.equal(i16(v), i16(vd.to(dtype)))
    for rows in (slice(0, 9), slice(12, 21)):   # the rows of no sequence hold no defined value
        torch.testing.assert_close(out[rows].double(), ref[rows], atol=2e-2, rtol=2e-2)


# ---- 3. decoder --------------------------------------------------------------------------------------------------
def _packed(tokens, starts, sizes):
    emb = torch.cat([tokens[b, s:s + t] for b, (s, t) in enumerate(zip(starts, sizes))])
    return emb, _cu(sizes), max(max(sizes), 1)


STEPS = [[5, 1, 0], [1, 16, 2], [0, 1, 1], [9, 0, 4]]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_decoder_packed_steps_match_fp32(dtype, monkeypatch):
    import unicore_b200.ops.attention_ops as attention_ops

    ops = _ops()
    ref, model = _decoder_pair(dtype, False)
    real = ops.native()
    calls = []

    class KvSpy:
        def __getattr__(self, name):
            return getattr(real.kvcache, name)

        def fmha_kvcache_varlen_fwd(self, *args, **kwargs):
            calls.append(args[5] is not None)   # True: self-attention (seqlens), False: encoder attention
            return real.kvcache.fmha_kvcache_varlen_fwd(*args, **kwargs)

    class Spy:
        kvcache = KvSpy()

        def __getattr__(self, name):
            return getattr(real, name)

    monkeypatch.setattr(attention_ops, "native", lambda: Spy())
    lens, Le = [24, 13, 19], 37
    g = torch.Generator(device="cuda").manual_seed(5)
    tokens = torch.randn(3, 64, 768, device="cuda", generator=g)
    enc = torch.randn(3, Le, 768, device="cuda", generator=g)
    enc_pad = torch.zeros(3, Le, dtype=torch.bool, device="cuda")
    enc_pad[0, Le - 8:] = True
    got = []
    with torch.no_grad():
        cache = model.new_cache(3, 100)
        emb, cu, L = _packed(tokens, [0, 0, 0], lens)
        got.append((model(emb.to(dtype), encoder_out=enc.to(dtype), encoder_padding_mask=enc_pad, cu_seqlens=cu,
                          max_seqlen=L, cache=cache), [0, 0, 0], lens))
        done = list(lens)
        for sizes in STEPS:
            emb, cu, T = _packed(tokens, done, sizes)
            got.append((model(emb.to(dtype), encoder_padding_mask=enc_pad, cu_seqlens=cu, max_seqlen=T, cache=cache),
                        list(done), sizes))
            done = [n + t for n, t in zip(done, sizes)]
        want = [ref(tokens[b:b + 1, :n], encoder_out=enc[b:b + 1], encoder_padding_mask=enc_pad[b:b + 1])[0]
                for b, n in enumerate(done)]
    assert calls == [True, False] * len(model.layers) * (1 + len(STEPS))
    tol = 2e-2 if dtype == torch.float16 else 6e-2
    for y, starts, sizes in got:
        row = 0
        for b, (s, t) in enumerate(zip(starts, sizes)):
            for i in range(t):
                rel = ((y[row + i].float() - want[b][s + i]).norm() / want[b][s + i].norm()).item()
                assert rel < tol, (b, s + i, rel)
            row += t
    assert cache.seqlens.tolist() == done and cache.max_len == max(lens) + sum(max(s) for s in STEPS)


def test_captured_step_after_packed_prefill_gives_eager_tokens():
    _ops()
    _, model = _decoder_pair(torch.float16, False)
    lens, Le, steps = [24, 13, 19], 40, 6
    g = torch.Generator(device="cuda").manual_seed(8)
    tokens = torch.randn(3, 32, 768, device="cuda", generator=g).half()
    enc = torch.randn(3, Le, 768, device="cuda", generator=g).half()
    enc_pad = torch.zeros(3, Le, dtype=torch.bool, device="cuda")
    enc_pad[1, 30:] = True
    table = torch.randn(64, 768, device="cuda", generator=g).half()   # a toy vocabulary: token -> embedding
    emb, cu, L = _packed(tokens, [0, 0, 0], lens)
    runs = []
    with torch.no_grad():
        for captured in (False, True):
            cache = model.new_cache(3, 64)
            y = model(emb, encoder_out=enc, encoder_padding_mask=enc_pad, cu_seqlens=cu, max_seqlen=L, cache=cache)
            last = torch.stack([y[int(cu[b + 1]) - 1] for b in range(3)])[:, None]
            step = model.capture_step(cache, encoder_padding_mask=enc_pad) if captured else None
            ids = []
            for _ in range(steps):
                tok = (last[:, 0].float() @ table.float().t()).argmax(-1)   # greedy
                ids.append(tok)
                x = table[tok][:, None]
                last = step(x).clone() if captured else model(x, encoder_padding_mask=enc_pad, cache=cache)
            runs.append(torch.stack(ids, 1))
    assert torch.equal(runs[0], runs[1]), runs


def test_packed_step_does_not_synchronise():
    _ops()
    _, model = _decoder_pair(torch.float16, False)
    lens = [24, 13, 19]
    g = torch.Generator(device="cuda").manual_seed(6)
    tokens = torch.randn(3, 40, 768, device="cuda", generator=g).half()
    enc = torch.randn(3, 40, 768, device="cuda", generator=g).half()
    enc_pad = torch.zeros(3, 40, dtype=torch.bool, device="cuda")
    with torch.no_grad():
        cache = model.new_cache(3, 96)
        emb, cu, L = _packed(tokens, [0, 0, 0], lens)
        model(emb, encoder_out=enc, encoder_padding_mask=enc_pad, cu_seqlens=cu, max_seqlen=L, cache=cache)
        emb, cu, T = _packed(tokens, lens, [3, 1, 5])
        model(emb, encoder_padding_mask=enc_pad, cu_seqlens=cu, max_seqlen=T, cache=cache)   # warm-up
        emb, cu, T = _packed(tokens, [n + t for n, t in zip(lens, [3, 1, 5])], [2, 0, 6])
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            y = model(emb, encoder_padding_mask=enc_pad, cu_seqlens=cu, max_seqlen=T, cache=cache)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    assert y.shape == (8, 768) and bool(torch.isfinite(y).all())


# ---- 4. binding rejections ----------------------------------------------------------------------------------------
def _valid():
    q = torch.randn(7, 2, 64, device="cuda").half()
    k = torch.randn(2, 21, 2, 64, device="cuda").half()
    cu = torch.tensor([0, 3, 7], dtype=torch.int32, device="cuda")
    lens = torch.tensor([3, 4], dtype=torch.int32, device="cuda")
    bias = torch.randn(2, 2, 4, 24, device="cuda").half()
    kpm = torch.zeros(2, 21, dtype=torch.bool, device="cuda")
    return [q, k, k.clone(), cu, 4, lens, 8, q.clone(), q.clone(), bias, kpm, 0.125]


OPERANDS = {0: ("q", ("cpu", "dtype", "small", "mis")), 1: ("k_cache", ("cpu", "dtype", "small", "mis")),
            2: ("v_cache", ("cpu", "dtype", "small", "mis")), 3: ("cu_seqlens", ("cpu", "dtype", "nc")),
            5: ("seqlens", ("cpu", "dtype", "small", "nc")), 7: ("k_new", ("cpu", "dtype", "small", "mis")),
            8: ("v_new", ("cpu", "dtype", "small", "mis")), 9: ("bias", ("cpu", "dtype", "small", "nc", "mis")),
            10: ("key_padding_mask", ("cpu", "dtype", "small", "nc"))}


def test_binding_rejects_bad_operands():
    _kv().fmha_kvcache_varlen_fwd(*_valid())   # the builder is valid
    torch.cuda.synchronize()
    for i, (label, kinds) in OPERANDS.items():
        for kind in kinds:
            args = _valid()
            args[i] = MUTATE[kind](args[i])
            with pytest.raises(RuntimeError, match=r"\b" + re.escape(label) + " must"):
                _kv().fmha_kvcache_varlen_fwd(*args)


def test_binding_rejects_bad_shapes_and_capacity():
    fn = _kv().fmha_kvcache_varlen_fwd
    q, k, v, cu, L, lens, _, kn, vn, bias, kpm, scale = _valid()
    with pytest.raises(RuntimeError, match="k_new must have sizes"):
        fn(q, k, v, cu, L, lens, 8, kn[:6], vn, None, None, scale)
    with pytest.raises(RuntimeError, match="k_cache must have sizes"):
        fn(q, k[:, :, :1], v, cu, L, lens, 8, kn, vn, None, None, scale)
    with pytest.raises(RuntimeError, match="capacity"):
        fn(q, k, v, cu, L, lens, 18, kn, vn, None, None, scale)   # 18 + 4 > 21
    with pytest.raises(RuntimeError, match="multiple of 8"):
        fn(q, k, v, cu, L, lens, 8, kn, vn, bias[..., :20].contiguous(), None, scale)
    with pytest.raises(RuntimeError, match="column for every key"):
        fn(q, k, v, cu, L, lens, 8, kn, vn, bias[..., :8].contiguous(), None, scale)
    with pytest.raises(RuntimeError, match="append"):
        fn(q, k, v, cu, L, lens, 8, None, None, None, None, scale)
    with pytest.raises(RuntimeError, match="B \\+ 1 >= 2"):
        fn(q, k[:0], v[:0], cu[:1], L, None, 0, None, None, None, None, scale)
    with pytest.raises(RuntimeError, match="sizes"):   # cu_seqlens of another B than the caches
        fn(q, k[:1], v[:1], cu, L, lens[:1], 8, kn, vn, None, None, scale)
    with pytest.raises(RuntimeError, match="max_seqlen"):
        fn(q, k, v, cu, 0, lens, 8, kn, vn, None, None, scale)
    with pytest.raises(ValueError, match="capacity"):
        _ops().attention_with_kv_cache_varlen(q, k, v, cu, L, lens, 18, k_new=kn, v_new=vn)
