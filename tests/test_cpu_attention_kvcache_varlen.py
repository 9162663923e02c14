"""Packed variable-length steps into a decoder cache on the CPU (float64, ``attention_with_kv_cache_varlen_reference``):
the op equals ``attention_with_kv_cache_reference`` on each sequence alone with ``T = T_b`` (ragged ``T_b`` including 0
and 1, ragged ``seqlens``, cross mode); a decoder fed a packed prefill and packed ragged steps equals each sequence's
full forward alone and the padded path (relative positions and rotary, with and without an encoder, grouped-query
attention); a sequence rewound to 0 and re-prompted inside a packed step equals a fresh prefill of its new prompt; and
the error cases (capacity by the host bound, dropout in training, gradients through the op, a packed encoder output
with a cache)."""
import pytest
import torch

from unicore import ops
from unicore.modules import TransformerDecoder

E, HEADS, S = 64, 4, 6
LENS = [7, 3, 5]   # prompt lengths
F64 = torch.float64
# the cache references take their softmax in fp32, so the decoder's outputs agree to about 1e-7
TOL = dict(atol=1e-6, rtol=1e-6)


def _cu(lens):
    return torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32)


def _decoder(kind="relpos", kv_heads=None, seed=0):
    torch.manual_seed(seed)
    rotary = kind == "rotary"
    m = TransformerDecoder(decoder_layers=2, embed_dim=E, ffn_embed_dim=2 * E, attention_heads=HEADS, max_seq_len=64,
                           rel_pos=not rotary, rotary_dim=8 if rotary else None, attention_kv_heads=kv_heads).eval()
    with torch.no_grad():
        for p in m.parameters():   # non-trivial LayerNorm and bias parameters
            p.add_(torch.randn_like(p) * 0.02)
    return m.to(F64)


def _data(B=3, T=40, seed=1):
    g = torch.Generator().manual_seed(seed)
    tokens = torch.randn(B, T, E, generator=g, dtype=F64)   # sequence b is tokens[b, :n]
    enc = torch.randn(B, S, E, generator=g, dtype=F64)
    enc_pad = torch.zeros(B, S, dtype=torch.bool)
    enc_pad[1, S - 2:] = True
    return tokens, enc, enc_pad


def _packed(tokens, starts, sizes):
    """``(emb [N, E], cu_seqlens, max_seqlen)``: tokens ``starts[b] .. starts[b] + sizes[b] - 1`` of each sequence."""
    emb = torch.cat([tokens[b, s:s + t] for b, (s, t) in enumerate(zip(starts, sizes))])
    return emb, _cu(sizes), max(max(sizes), 1)


def _full(m, tokens, enc, enc_pad, b, upto):
    """The full forward of sequence b alone over its first ``upto`` tokens: ``[upto, E]``."""
    if enc is None:
        return m(tokens[b:b + 1, :upto])[0]
    return m(tokens[b:b + 1, :upto], encoder_out=enc[b:b + 1], encoder_padding_mask=enc_pad[b:b + 1])[0]


def _enc_args(enc, enc_pad, prefill):
    if enc is None:
        return {}
    return dict(encoder_out=enc if prefill else None, encoder_padding_mask=enc_pad)


# ---- the op ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kv_heads", [4, 2, 1])
def test_reference_equals_per_sequence_calls(kv_heads):
    g = torch.Generator().manual_seed(kv_heads)
    sizes, lens = [0, 1, 2, 5, 3], [0, 4, 9, 2, 20]
    B, C, H, D = len(sizes), 31, 4, 8
    N = sum(sizes) + 2   # two rows of no sequence
    T = max(sizes)
    q = torch.randn(N, H, D, generator=g, dtype=F64)
    kn, vn = (torch.randn(N, kv_heads, D, generator=g, dtype=F64) for _ in range(2))
    k, v = (torch.randn(B, C, kv_heads, D, generator=g, dtype=F64) for _ in range(2))
    bias = torch.randn(B, H, T, 40, generator=g, dtype=F64)
    kpm = torch.rand(B, C, generator=g) < 0.2
    seqlens = torch.tensor(lens, dtype=torch.int32)
    cu = _cu(sizes)
    k1, v1 = k.clone(), v.clone()
    out = ops.attention_with_kv_cache_varlen(q, k1, v1, cu, T, seqlens, max(lens), k_new=kn, v_new=vn, bias=bias,
                                             key_padding_mask=kpm)
    assert out.shape == (N, H, D)
    for b, (n, t) in enumerate(zip(lens, sizes)):
        s = int(cu[b])
        k2, v2 = k[b:b + 1].clone(), v[b:b + 1].clone()
        if t > 0:
            want = ops.attention_with_kv_cache_reference(q[None, s:s + t], k2, v2, seqlens[b:b + 1], max(lens),
                                                         k_new=kn[None, s:s + t], v_new=vn[None, s:s + t],
                                                         bias=bias[b:b + 1, :, :t], key_padding_mask=kpm[b:b + 1])
            torch.testing.assert_close(out[s:s + t], want[0], atol=1e-12, rtol=1e-12)
        assert torch.equal(k1[b], k2[0]) and torch.equal(v1[b], v2[0])   # T_b rows appended, the rest untouched
    assert torch.equal(out[-2:], torch.zeros(2, H, D))


def test_reference_cross_mode_and_clamps():
    g = torch.Generator().manual_seed(2)
    sizes = [3, 0, 4]
    B, C, H, D = 3, 9, 2, 8
    q = torch.randn(sum(sizes), H, D, generator=g, dtype=F64)
    k, v = (torch.randn(B, C, H, D, generator=g, dtype=F64) for _ in range(2))
    kpm = torch.zeros(B, C, dtype=torch.bool)
    kpm[0, 5:] = True
    kpm[2] = True   # every key masked: O = 0
    cu = _cu(sizes)
    out = ops.attention_with_kv_cache_varlen(q, k, v, cu, 4, key_padding_mask=kpm)
    torch.testing.assert_close(out[:3], ops.attention_reference(q[None, :3], k[:1], v[:1], key_padding_mask=kpm[:1],
                                                                dropout_p=0.0)[0])
    assert torch.equal(out[3:], torch.zeros(4, H, D))
    # out-of-range cu_seqlens / seqlens: clamped as the kernels clamp them
    k1, v1 = k.clone(), v.clone()
    kn = torch.randn(7, H, D, generator=g, dtype=F64)
    bad_cu = torch.tensor([0, 2, 2, 50], dtype=torch.int32)   # {s_b, T_b}: {0, 2}, {2, 0}, {2, min(48, 4, 7 - 2)}
    seqlens = torch.tensor([-5, 3, 1 << 30], dtype=torch.int32)
    out = ops.attention_with_kv_cache_varlen(q[:7], k1, v1, bad_cu, 4, seqlens, 5, k_new=kn, v_new=kn)
    want = ops.attention_with_kv_cache_reference(q[None, :2], k[:1].clone(), v[:1].clone(),
                                                 torch.zeros(1, dtype=torch.int32), 5, k_new=kn[None, :2],
                                                 v_new=kn[None, :2])
    torch.testing.assert_close(out[:2], want[0])
    assert torch.equal(k1[2], k[2]) and torch.equal(k1[1], k[1])   # p_2 = C: nothing fits; T_1 = 0
    assert torch.equal(k1[0, :2], kn[:2]) and torch.equal(k1[0, 2:], k[0, 2:])


# ---- the decoder --------------------------------------------------------------------------------------------------
STEPS = [[1, 0, 3], [2, 1, 1], [0, 4, 2], [1, 1, 1], [5, 0, 0]]


@pytest.mark.parametrize("encoder", [True, False], ids=["enc_dec", "dec_only"])
@pytest.mark.parametrize("kind,kv_heads", [("relpos", None), ("rotary", None), ("relpos", 2)],
                         ids=["relpos", "rotary", "gqa"])
def test_decoder_packed_steps_match_full_forward(kind, kv_heads, encoder):
    m = _decoder(kind, kv_heads)
    tokens, enc, enc_pad = _data()
    if not encoder:
        enc = enc_pad = None
    with torch.no_grad():
        cache = m.new_cache(3, 48)
        emb, cu, L = _packed(tokens, [0, 0, 0], LENS)
        y = m(emb, cu_seqlens=cu, max_seqlen=L, cache=cache, **_enc_args(enc, enc_pad, True))
        assert y.shape == (sum(LENS), E)
        for b, n in enumerate(LENS):
            torch.testing.assert_close(y[int(cu[b]):int(cu[b + 1])], _full(m, tokens, enc, enc_pad, b, n),
                                       **TOL)
        assert cache.seqlens.tolist() == LENS and cache.max_len == max(LENS)
        done = list(LENS)
        for sizes in STEPS:
            emb, cu, T = _packed(tokens, done, sizes)
            y = m(emb, cu_seqlens=cu, max_seqlen=T, cache=cache, **_enc_args(enc, enc_pad, False))
            for b, (n, t) in enumerate(zip(done, sizes)):
                if t:
                    full = _full(m, tokens, enc, enc_pad, b, n + t)
                    torch.testing.assert_close(y[int(cu[b]):int(cu[b + 1])], full[n:], **TOL)
            done = [n + t for n, t in zip(done, sizes)]
            assert cache.seqlens.tolist() == done
        assert cache.max_len == max(LENS) + sum(max(max(s), 1) for s in STEPS)


@pytest.mark.parametrize("kind", ["relpos", "rotary"])
def test_decoder_packed_equals_padded_path(kind):
    m = _decoder(kind)
    tokens, enc, enc_pad = _data()
    T = 3
    with torch.no_grad():
        padded = m.new_cache(3, 32)
        L = max(LENS)
        prompt = torch.zeros(3, L, E, dtype=F64)
        pad = torch.ones(3, L, dtype=torch.bool)
        for b, n in enumerate(LENS):
            prompt[b, :n] = tokens[b, :n]
            pad[b, :n] = False
        yp = m(prompt, encoder_out=enc, padding_mask=pad, encoder_padding_mask=enc_pad, cache=padded)
        packed = m.new_cache(3, 32)
        emb, cu, Lp = _packed(tokens, [0, 0, 0], LENS)
        y = m(emb, encoder_out=enc, encoder_padding_mask=enc_pad, cu_seqlens=cu, max_seqlen=Lp, cache=packed)
        for b, n in enumerate(LENS):
            torch.testing.assert_close(y[int(cu[b]):int(cu[b + 1])], yp[b, :n], **TOL)
            for lp, lq in zip(padded.layers, packed.layers):
                torch.testing.assert_close(lq.k[b, :n], lp.k[b, :n], **TOL)
                torch.testing.assert_close(lq.v[b, :n], lp.v[b, :n], **TOL)
        step = torch.stack([tokens[b, n:n + T] for b, n in enumerate(LENS)])
        yp = m(step, encoder_padding_mask=enc_pad, cache=padded)
        y = m(step.reshape(-1, E), encoder_padding_mask=enc_pad, cu_seqlens=_cu([T] * 3), max_seqlen=T, cache=packed)
        torch.testing.assert_close(y.view(3, T, E), yp, **TOL)
        assert packed.seqlens.tolist() == padded.seqlens.tolist()


@pytest.mark.parametrize("kind", ["relpos", "rotary"])
def test_slot_reuse_inside_a_packed_step(kind):
    m = _decoder(kind)
    tokens, enc, enc_pad = _data()
    fresh = _data(seed=7)[0]   # sequence 1's new prompt
    with torch.no_grad():
        cache = m.new_cache(3, 48)
        emb, cu, L = _packed(tokens, [0, 0, 0], LENS)
        m(emb, encoder_out=enc, encoder_padding_mask=enc_pad, cu_seqlens=cu, max_seqlen=L, cache=cache)
        emb, cu, T = _packed(tokens, LENS, [2, 2, 2])
        m(emb, encoder_padding_mask=enc_pad, cu_seqlens=cu, max_seqlen=T, cache=cache)
        cache.rewind(torch.tensor([0, LENS[1] + 2, 0]))   # sequence 1 is done: its slot is emptied
        done = [LENS[0] + 2, 0, LENS[2] + 2]
        sizes = [1, 6, 1]   # one token for the others, the new prompt for slot 1, in one call
        emb = torch.cat([tokens[0, done[0]:done[0] + 1], fresh[1, :6], tokens[2, done[2]:done[2] + 1]])
        cu = _cu(sizes)
        y = m(emb, encoder_padding_mask=enc_pad, cu_seqlens=cu, max_seqlen=6, cache=cache)
        torch.testing.assert_close(y[1:7], _full(m, fresh, enc, enc_pad, 1, 6), **TOL)
        for b in (0, 2):
            full = _full(m, tokens, enc, enc_pad, b, done[b] + 1)
            torch.testing.assert_close(y[int(cu[b]):int(cu[b + 1])], full[done[b]:], **TOL)
        assert cache.seqlens.tolist() == [done[0] + 1, 6, done[2] + 1]


# ---- errors ----------------------------------------------------------------------------------------------------
def test_capacity_by_host_bound_raises():
    m = _decoder()
    tokens, enc, enc_pad = _data()
    with torch.no_grad():
        cache = m.new_cache(3, 12)
        emb, cu, L = _packed(tokens, [0, 0, 0], LENS)
        m(emb, encoder_out=enc, encoder_padding_mask=enc_pad, cu_seqlens=cu, max_seqlen=L, cache=cache)   # max_len 7
        emb, cu, _ = _packed(tokens, LENS, [1, 1, 1])
        with pytest.raises(ValueError, match="capacity"):   # the bound, not the real lengths, decides
            m(emb, encoder_padding_mask=enc_pad, cu_seqlens=cu, max_seqlen=6, cache=cache)
        m(emb, encoder_padding_mask=enc_pad, cu_seqlens=cu, max_seqlen=5, cache=cache)   # exactly full
        assert cache.max_len == 12
    q = torch.randn(4, 2, 8)
    k, v = torch.randn(1, 10, 2, 8), torch.randn(1, 10, 2, 8)
    with pytest.raises(ValueError, match="capacity"):
        ops.attention_with_kv_cache_varlen(q, k, v, _cu([4]), 4, torch.tensor([3], dtype=torch.int32), 7, k_new=q,
                                           v_new=q)
    with pytest.raises(ValueError, match="append k_new"):
        ops.attention_with_kv_cache_varlen(q, k, v, _cu([4]), 4, torch.tensor([3], dtype=torch.int32), 3)


def test_packed_step_in_training_with_dropout_raises():
    m = _decoder()
    tokens, enc, enc_pad = _data()
    m.train()
    emb, cu, L = _packed(tokens, [0, 0, 0], LENS)
    with pytest.raises(RuntimeError, match="dropout"):
        m(emb, encoder_out=enc, encoder_padding_mask=enc_pad, cu_seqlens=cu, max_seqlen=L, cache=m.new_cache(3, 16))


def test_grad_through_op_raises():
    q = torch.randn(3, 2, 8, requires_grad=True)
    k, v = torch.randn(1, 8, 2, 8), torch.randn(1, 8, 2, 8)
    kn = torch.randn(3, 2, 8)
    lens = torch.tensor([2], dtype=torch.int32)
    with pytest.raises(RuntimeError, match="no backward"):
        ops.attention_with_kv_cache_varlen(q, k, v, _cu([3]), 3, lens, 2, k_new=kn, v_new=kn)
    with torch.no_grad():
        ops.attention_with_kv_cache_varlen(q, k, v, _cu([3]), 3, lens, 2, k_new=kn, v_new=kn)


def test_packed_encoder_output_with_cache_raises():
    m = _decoder()
    tokens, enc, _ = _data()
    emb, cu, L = _packed(tokens, [0, 0, 0], LENS)
    enc_packed, enc_cu, enc_L = _packed(enc, [0, 0, 0], [S, 4, 5])
    with torch.no_grad(), pytest.raises(ValueError, match="encoder_cu_seqlens"):
        m(emb, encoder_out=enc_packed, cu_seqlens=cu, max_seqlen=L, encoder_cu_seqlens=enc_cu,
          encoder_max_seqlen=enc_L, cache=m.new_cache(3, 16))
