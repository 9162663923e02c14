"""Incremental decoding on the CPU (fp32, ``attention_with_kv_cache_reference``): a decoder run token by token against
its ``DecoderCache`` equals the full forward of each sequence alone; ``reorder`` equals decoding the reordered batch;
and the error cases (dropout in training mode, a step with ``attn_mask``, a full cache, gradients through the op)."""
import copy

import pytest
import torch

from unicore import ops
from unicore.modules import TransformerDecoder

E, HEADS, S = 64, 4, 6
LENS = [7, 3, 5]   # right-padded prompts of different lengths


def _decoder(post_ln, seed=0):
    torch.manual_seed(seed)
    m = TransformerDecoder(decoder_layers=2, embed_dim=E, ffn_embed_dim=2 * E, attention_heads=HEADS, max_seq_len=64,
                           post_ln=post_ln).eval()
    with torch.no_grad():
        for p in m.parameters():   # non-trivial LayerNorm and bias parameters
            p.add_(torch.randn_like(p) * 0.02)
    return m


def _data(B=3, T=24, seed=1):
    g = torch.Generator().manual_seed(seed)
    tokens = torch.randn(B, T, E, generator=g)   # sequence b is tokens[b, :LENS[b] + steps]
    enc = torch.randn(B, S, E, generator=g)
    enc_pad = torch.zeros(B, S, dtype=torch.bool)
    enc_pad[1, S - 2:] = True
    return tokens, enc, enc_pad


def _prompt(tokens, lens):
    L = max(lens)
    prompt = torch.zeros(tokens.shape[0], L, E)
    pad = torch.ones(tokens.shape[0], L, dtype=torch.bool)
    for b, n in enumerate(lens):
        prompt[b, :n] = tokens[b, :n]
        pad[b, :n] = False
    return prompt, pad


def _decode(m, tokens, enc, enc_pad, lens, steps, cache=None):
    """Prefill + ``steps`` single-token steps; returns the cache and the outputs of every step [B, E]."""
    prompt, pad = _prompt(tokens, lens)
    cache = cache or m.new_cache(tokens.shape[0], 40)
    m(prompt, encoder_out=enc, padding_mask=pad, encoder_padding_mask=enc_pad, cache=cache)
    outs = []
    for t in range(steps):
        tok = torch.stack([tokens[b, n + t] for b, n in enumerate(lens)])[:, None]
        outs.append(m(tok, encoder_padding_mask=enc_pad, cache=cache)[:, 0])
    return cache, outs


@pytest.mark.parametrize("post_ln", [False, True], ids=["pre_ln", "post_ln"])
def test_decoder_steps_match_full_forward(post_ln):
    m = _decoder(post_ln)
    tokens, enc, enc_pad = _data()
    steps = 12
    with torch.no_grad():
        cache, outs = _decode(m, tokens, enc, enc_pad, LENS, steps)
        assert cache.max_len == max(LENS) + steps
        assert cache.seqlens.tolist() == [n + steps for n in LENS]
        for t, y in enumerate(outs):
            for b, n in enumerate(LENS):
                full = m(tokens[b:b + 1, :n + t + 1], encoder_out=enc[b:b + 1], encoder_padding_mask=enc_pad[b:b + 1])
                torch.testing.assert_close(y[b], full[0, -1], atol=2e-5, rtol=2e-5)


def test_reorder_matches_reordered_batch():
    m = _decoder(False)
    tokens, enc, enc_pad = _data()
    index = torch.tensor([2, 0, 2])
    lens_r = [LENS[i] for i in index.tolist()]
    with torch.no_grad():
        cache, _ = _decode(m, tokens, enc, enc_pad, LENS, 3)
        cache.reorder(index)
        tok_r, enc_pad_r = tokens[index], enc_pad[index]
        got = [m(torch.stack([tok_r[b, n + 3 + t] for b, n in enumerate(lens_r)])[:, None],
                 encoder_padding_mask=enc_pad_r, cache=cache)[:, 0] for t in range(4)]
        _, want = _decode(m, tok_r, enc[index], enc_pad_r, lens_r, 7)
    for t in range(4):
        torch.testing.assert_close(got[t], want[3 + t], atol=2e-5, rtol=2e-5)


def test_reference_append_writes_one_row():
    B, C, H, D = 2, 9, 2, 8
    g = torch.Generator().manual_seed(0)
    k = torch.randn(B, C, H, D, generator=g)
    v = torch.randn(B, C, H, D, generator=g)
    k0, v0 = k.clone(), v.clone()
    q, kn, vn = (torch.randn(B, 1, H, D, generator=g) for _ in range(3))
    seqlens = torch.tensor([3, 8], dtype=torch.int32)
    out = ops.attention_with_kv_cache(q, k, v, seqlens, 8, k_new=kn, v_new=vn)
    for b, n in enumerate(seqlens.tolist()):
        assert torch.equal(k[b, n], kn[b, 0]) and torch.equal(v[b, n], vn[b, 0])
        k0[b, n], v0[b, n] = kn[b, 0], vn[b, 0]
        want = ops.attention_reference(q[b:b + 1], k0[b:b + 1, :n + 1], v0[b:b + 1, :n + 1], dropout_p=0.0)
        torch.testing.assert_close(out[b:b + 1], want)
    assert torch.equal(k, k0) and torch.equal(v, v0)


def test_fully_masked_row_gives_zero():
    q, k, v = torch.randn(2, 1, 2, 8), torch.randn(2, 5, 2, 8), torch.randn(2, 5, 2, 8)
    kpm = torch.zeros(2, 5, dtype=torch.bool)
    kpm[1] = True
    out = ops.attention_with_kv_cache(q, k, v, key_padding_mask=kpm)
    assert torch.equal(out[1], torch.zeros_like(out[1])) and bool(out[0].abs().sum() > 0)


def test_training_with_dropout_raises():
    m = _decoder(False)
    m.train()
    tokens, enc, enc_pad = _data()
    with pytest.raises(RuntimeError, match="dropout"):
        _decode(m, tokens, enc, enc_pad, LENS, 1)


def test_attn_mask_on_step_raises():
    m = _decoder(False)
    tokens, enc, enc_pad = _data()
    with torch.no_grad():
        cache, _ = _decode(m, tokens, enc, enc_pad, LENS, 1)
        with pytest.raises(NotImplementedError, match="not supported"):
            m(tokens[:, :1], attn_mask=torch.zeros(3 * HEADS, 1, 9), encoder_padding_mask=enc_pad, cache=cache)


def test_capacity_overflow_raises():
    m = _decoder(False)
    tokens, enc, enc_pad = _data()
    with torch.no_grad():
        with pytest.raises(ValueError, match="capacity"):
            m.new_cache(3, 65)
        cache = m.new_cache(3, 9)
        _decode(m, tokens, enc, enc_pad, LENS, 2, cache=cache)   # max_len 9 after two steps
        with pytest.raises(ValueError, match="capacity"):
            m(tokens[:, :1], encoder_padding_mask=enc_pad, cache=cache)
        with pytest.raises(ValueError, match="capacity"):
            _decode(m, torch.randn(3, 12, E), enc, enc_pad, [10, 10, 10], 0, cache=m.new_cache(3, 9))


def test_grad_through_op_raises():
    q = torch.randn(1, 1, 2, 8, requires_grad=True)
    k, v = torch.randn(1, 4, 2, 8), torch.randn(1, 4, 2, 8)
    with pytest.raises(RuntimeError, match="no backward"):
        ops.attention_with_kv_cache(q, k, v)
    with torch.no_grad():
        ops.attention_with_kv_cache(q, k, v)


def test_new_cache_shapes_and_default_path_unchanged():
    m = _decoder(False)
    cache = m.new_cache(2, 16)
    assert len(cache.layers) == 2 and cache.layers[0].k.shape == (2, 16, HEADS, E // HEADS)
    assert cache.seqlens.dtype == torch.int32 and cache.max_len == 0
    tokens, enc, enc_pad = _data(B=2)
    with torch.no_grad():
        a = m(tokens[:, :5], encoder_out=enc, encoder_padding_mask=enc_pad)
        b = copy.deepcopy(m)(tokens[:, :5], encoder_out=enc, encoder_padding_mask=enc_pad, cache=cache)
    assert torch.equal(a, b)
