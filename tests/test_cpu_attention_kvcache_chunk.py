"""Multi-token steps into a non-empty decoder cache on the CPU (fp32, ``attention_with_kv_cache_reference``): the op
with a chunk of T queries equals T single-query calls; a decoder fed a prefill, chunks of mixed sizes and single
steps equals the full forward of each sequence alone; ``DecoderCache.rewind`` after a chunk equals feeding only the
kept tokens; ``reorder`` after a chunk; and the error cases (capacity, a chunk with ``seqlens`` but nothing to append,
dropout in training mode, gradients through the op)."""
import pytest
import torch

from unicore import ops
from unicore.modules import TransformerDecoder

E, HEADS, S = 64, 4, 6
LENS = [7, 3, 5]   # right-padded prompts of different lengths


def _decoder(post_ln=False, seed=0):
    torch.manual_seed(seed)
    m = TransformerDecoder(decoder_layers=2, embed_dim=E, ffn_embed_dim=2 * E, attention_heads=HEADS, max_seq_len=64,
                           post_ln=post_ln).eval()
    with torch.no_grad():
        for p in m.parameters():   # non-trivial LayerNorm and bias parameters
            p.add_(torch.randn_like(p) * 0.02)
    return m


def _data(B=3, T=40, seed=1):
    g = torch.Generator().manual_seed(seed)
    tokens = torch.randn(B, T, E, generator=g)   # sequence b is tokens[b, :LENS[b] + fed]
    enc = torch.randn(B, S, E, generator=g)
    enc_pad = torch.zeros(B, S, dtype=torch.bool)
    enc_pad[1, S - 2:] = True
    return tokens, enc, enc_pad


def _prefill(m, tokens, enc, enc_pad, lens, capacity=48):
    L = max(lens)
    prompt = torch.zeros(tokens.shape[0], L, E)
    pad = torch.ones(tokens.shape[0], L, dtype=torch.bool)
    for b, n in enumerate(lens):
        prompt[b, :n] = tokens[b, :n]
        pad[b, :n] = False
    cache = m.new_cache(tokens.shape[0], capacity)
    m(prompt, encoder_out=enc, padding_mask=pad, encoder_padding_mask=enc_pad, cache=cache)
    return cache


def _next(tokens, starts, T):
    """``[B, T, E]``: tokens ``starts[b] .. starts[b] + T - 1`` of each sequence."""
    return torch.stack([tokens[b, s:s + T] for b, s in enumerate(starts)])


def _full(m, tokens, enc, enc_pad, b, upto):
    """The full forward of sequence b alone over its first ``upto`` tokens: ``[upto, E]``."""
    return m(tokens[b:b + 1, :upto], encoder_out=enc[b:b + 1], encoder_padding_mask=enc_pad[b:b + 1])[0]


def test_reference_chunk_equals_single_rows():
    B, C, H, D, T = 3, 21, 2, 8, 5
    g = torch.Generator().manual_seed(0)
    k = torch.randn(B, C, H, D, generator=g)
    v = torch.randn(B, C, H, D, generator=g)
    q, kn, vn = (torch.randn(B, T, H, D, generator=g) for _ in range(3))
    bias = torch.randn(B, H, T, C, generator=g)
    kpm = torch.rand(B, C, generator=g) < 0.2
    seqlens = torch.tensor([0, 9, 16], dtype=torch.int32)
    k1, v1 = k.clone(), v.clone()
    out = ops.attention_with_kv_cache(q, k, v, seqlens, 16, k_new=kn, v_new=vn, bias=bias, key_padding_mask=kpm)
    assert out.shape == (B, T, H, D)
    for i in range(T):
        want = ops.attention_with_kv_cache(q[:, i:i + 1], k1, v1, seqlens + i, 16 + i, k_new=kn[:, i:i + 1],
                                           v_new=vn[:, i:i + 1], bias=bias[:, :, i:i + 1], key_padding_mask=kpm)
        torch.testing.assert_close(out[:, i:i + 1], want, atol=1e-6, rtol=1e-6)
    assert torch.equal(k, k1) and torch.equal(v, v1)   # the same rows appended


def test_reference_chunk_skips_rows_past_capacity():
    B, C, H, D, T = 2, 10, 1, 8, 4
    k, v = torch.zeros(B, C, H, D), torch.zeros(B, C, H, D)
    q, kn, vn = torch.randn(B, T, H, D), torch.randn(B, T, H, D), torch.randn(B, T, H, D)
    seqlens = torch.tensor([8, 30], dtype=torch.int32)   # rows 8, 9 fit; nothing fits the second sequence
    out = ops.attention_with_kv_cache_reference(q, k, v, seqlens, 6, k_new=kn, v_new=vn)
    assert torch.equal(k[0, 8:], kn[0, :2]) and torch.equal(k[0, :8], torch.zeros(8, H, D))
    assert torch.equal(k[1], torch.zeros(C, H, D)) and bool(torch.isfinite(out).all())


def test_reference_cross_attention_chunk():
    q, k, v = torch.randn(2, 3, 2, 8), torch.randn(2, 5, 2, 8), torch.randn(2, 5, 2, 8)
    kpm = torch.zeros(2, 5, dtype=torch.bool)
    kpm[1, 3:] = True
    out = ops.attention_with_kv_cache(q, k, v, key_padding_mask=kpm)
    torch.testing.assert_close(out, ops.attention_reference(q, k, v, key_padding_mask=kpm, dropout_p=0.0))


@pytest.mark.parametrize("post_ln", [False, True], ids=["pre_ln", "post_ln"])
def test_decoder_chunks_match_full_forward(post_ln):
    m = _decoder(post_ln)
    tokens, enc, enc_pad = _data()
    sizes = [1, 2, 5, 8, 1, 1, 3]
    with torch.no_grad():
        cache = _prefill(m, tokens, enc, enc_pad, LENS)
        fed = 0
        for T in sizes:
            y = m(_next(tokens, [n + fed for n in LENS], T), encoder_padding_mask=enc_pad, cache=cache)
            assert y.shape == (3, T, E)
            for b, n in enumerate(LENS):
                full = _full(m, tokens, enc, enc_pad, b, n + fed + T)
                torch.testing.assert_close(y[b], full[n + fed:], atol=2e-5, rtol=2e-5)
            fed += T
        assert cache.max_len == max(LENS) + fed and cache.seqlens.tolist() == [n + fed for n in LENS]


@pytest.mark.parametrize("per_sequence", [False, True], ids=["int", "tensor"])
def test_rewind_after_chunk_equals_feeding_kept_tokens(per_sequence):
    m = _decoder()
    tokens, enc, enc_pad = _data()
    T = 6
    r = torch.tensor([2, 0, 5], dtype=torch.int32) if per_sequence else 3
    keep = [T - int(x) for x in r.tolist()] if per_sequence else [T - r] * 3
    with torch.no_grad():
        cache = _prefill(m, tokens, enc, enc_pad, LENS)
        m(_next(tokens, LENS, T), encoder_padding_mask=enc_pad, cache=cache)   # a draft chunk
        cache.rewind(r)
        assert cache.seqlens.tolist() == [n + kp for n, kp in zip(LENS, keep)]
        assert cache.max_len == max(LENS) + (T if per_sequence else T - r)
        # continue from each sequence's own position: the rewound rows are overwritten
        y = m(_next(tokens, [n + kp for n, kp in zip(LENS, keep)], 4), encoder_padding_mask=enc_pad, cache=cache)
        for b, (n, kp) in enumerate(zip(LENS, keep)):
            full = _full(m, tokens, enc, enc_pad, b, n + kp + 4)
            torch.testing.assert_close(y[b], full[n + kp:], atol=2e-5, rtol=2e-5)


def test_rewind_clamps_at_zero_and_rejects_negative():
    m = _decoder()
    cache = m.new_cache(2, 16)
    cache.seqlens.copy_(torch.tensor([3, 7], dtype=torch.int32))
    cache.max_len = 7
    cache.rewind(torch.tensor([5, 1]))
    assert cache.seqlens.tolist() == [0, 6] and cache.max_len == 7
    cache.rewind(9)
    assert cache.seqlens.tolist() == [0, 0] and cache.max_len == 0
    with pytest.raises(ValueError, match=">= 0"):
        cache.rewind(-1)


def test_reorder_after_chunk():
    m = _decoder()
    tokens, enc, enc_pad = _data()
    index = torch.tensor([2, 0, 2])
    lens_r = [LENS[i] for i in index.tolist()]
    with torch.no_grad():
        cache = _prefill(m, tokens, enc, enc_pad, LENS)
        m(_next(tokens, LENS, 5), encoder_padding_mask=enc_pad, cache=cache)
        cache.reorder(index)
        tok_r, enc_pad_r = tokens[index], enc_pad[index]
        y = m(_next(tok_r, [n + 5 for n in lens_r], 3), encoder_padding_mask=enc_pad_r, cache=cache)
        for b, n in enumerate(lens_r):
            full = _full(m, tok_r, enc[index], enc_pad_r, b, n + 8)
            torch.testing.assert_close(y[b], full[n + 5:], atol=2e-5, rtol=2e-5)


def test_chunk_capacity_overflow_raises():
    m = _decoder()
    tokens, enc, enc_pad = _data()
    with torch.no_grad():
        cache = _prefill(m, tokens, enc, enc_pad, LENS, capacity=12)   # max_len 7
        with pytest.raises(ValueError, match="capacity"):
            m(tokens[:, :6], encoder_padding_mask=enc_pad, cache=cache)
        m(tokens[:, :5], encoder_padding_mask=enc_pad, cache=cache)   # exactly full
        assert cache.max_len == 12
    q = torch.randn(1, 4, 2, 8)
    k, v = torch.randn(1, 10, 2, 8), torch.randn(1, 10, 2, 8)
    with pytest.raises(ValueError, match="capacity"):
        ops.attention_with_kv_cache(q, k, v, torch.tensor([3], dtype=torch.int32), 7, k_new=q, v_new=q)


def test_chunk_with_seqlens_needs_new_rows():
    q, k, v = torch.randn(1, 3, 2, 8), torch.randn(1, 10, 2, 8), torch.randn(1, 10, 2, 8)
    with pytest.raises(ValueError, match="appends"):
        ops.attention_with_kv_cache(q, k, v, torch.tensor([3], dtype=torch.int32), 3)
    with pytest.raises(ValueError, match="appends"):
        ops.attention_with_kv_cache_reference(q, k, v, torch.tensor([3], dtype=torch.int32), 3)


def test_chunk_in_training_with_dropout_raises():
    m = _decoder()
    tokens, enc, enc_pad = _data()
    with torch.no_grad():
        cache = _prefill(m, tokens, enc, enc_pad, LENS)
    m.train()
    with pytest.raises(RuntimeError, match="dropout"):
        m(tokens[:, :4], encoder_padding_mask=enc_pad, cache=cache)


def test_chunk_grad_through_op_raises():
    q = torch.randn(1, 3, 2, 8, requires_grad=True)
    k, v = torch.randn(1, 8, 2, 8), torch.randn(1, 8, 2, 8)
    kn = torch.randn(1, 3, 2, 8)
    lens = torch.tensor([2], dtype=torch.int32)
    with pytest.raises(RuntimeError, match="no backward"):
        ops.attention_with_kv_cache(q, k, v, lens, 2, k_new=kn, v_new=kn)
    with torch.no_grad():
        ops.attention_with_kv_cache(q, k, v, lens, 2, k_new=kn, v_new=kn)
