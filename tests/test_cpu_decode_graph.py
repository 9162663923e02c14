"""What a captured decoding step relies on, checked on the CPU: ``DecoderCache.reorder`` and ``store_encoder`` write into
the buffers they already hold (a CUDA graph keeps their addresses), the relative-position bias of a step at a fixed
width equals the bias at the host bound on its first columns, and ``capture_step`` refuses to run without CUDA."""
import pytest
import torch

from unicore.modules import TransformerDecoder

E, HEADS, S = 64, 4, 6
LENS = [7, 3, 5]


def _decoder(seed=0):
    torch.manual_seed(seed)
    m = TransformerDecoder(decoder_layers=2, embed_dim=E, ffn_embed_dim=2 * E, attention_heads=HEADS,
                           max_seq_len=64).eval()
    with torch.no_grad():
        for p in m.parameters():
            p.add_(torch.randn_like(p) * 0.02)
    return m


def _prefilled(m, capacity=40, steps=2, seed=1):
    g = torch.Generator().manual_seed(seed)
    B, L = len(LENS), max(LENS)
    prompt = torch.randn(B, L, E, generator=g)
    pad = torch.ones(B, L, dtype=torch.bool)
    for b, n in enumerate(LENS):
        pad[b, :n] = False
    enc = torch.randn(B, S, E, generator=g)
    enc_pad = torch.zeros(B, S, dtype=torch.bool)
    enc_pad[1, S - 2:] = True
    cache = m.new_cache(B, capacity)
    with torch.no_grad():
        m(prompt, encoder_out=enc, padding_mask=pad, encoder_padding_mask=enc_pad, cache=cache)
        for _ in range(steps):
            m(torch.randn(B, 1, E, generator=g), encoder_padding_mask=enc_pad, cache=cache)
    return cache, enc, enc_pad


def test_reorder_writes_in_place():
    m = _decoder()
    cache, _, _ = _prefilled(m)
    index = torch.tensor([2, 0, 2])
    n = cache.max_len
    want_seqlens = cache.seqlens.index_select(0, index)
    want = [(lc.k.index_select(0, index)[:, :n], lc.v.index_select(0, index)[:, :n],
             lc.enc_k.index_select(0, index), lc.enc_v.index_select(0, index)) for lc in cache.layers]
    tensors = [cache.seqlens] + [t for lc in cache.layers for t in (lc.k, lc.v, lc.enc_k, lc.enc_v)]
    ptrs = [t.data_ptr() for t in tensors]
    cache.reorder(index)
    after = [cache.seqlens] + [t for lc in cache.layers for t in (lc.k, lc.v, lc.enc_k, lc.enc_v)]
    assert all(a is b for a, b in zip(after, tensors)) and [t.data_ptr() for t in after] == ptrs
    assert torch.equal(cache.seqlens, want_seqlens)
    for lc, (k, v, ek, ev) in zip(cache.layers, want):
        assert torch.equal(lc.k[:, :n], k) and torch.equal(lc.v[:, :n], v)
        assert torch.equal(lc.enc_k, ek) and torch.equal(lc.enc_v, ev)


def test_reorder_to_another_batch_size_rebinds():
    m = _decoder()
    cache, _, _ = _prefilled(m)
    index = torch.tensor([1, 1, 0, 2, 2])
    k0, seqlens0 = cache.layers[0].k.clone(), cache.seqlens.clone()
    cache.reorder(index)
    assert cache.seqlens.shape == (5,) and torch.equal(cache.seqlens, seqlens0.index_select(0, index))
    assert torch.equal(cache.layers[0].k, k0.index_select(0, index))


def test_store_encoder_reuses_tensors_of_the_same_shape():
    m = _decoder()
    cache, _, _ = _prefilled(m)
    lc = cache.layers[0]
    ek, ev = lc.enc_k, lc.enc_v
    k, v = torch.randn(ek.shape), torch.randn(ev.shape)
    lc.store_encoder(k, v)
    assert lc.enc_k is ek and lc.enc_v is ev
    assert torch.equal(lc.enc_k, k) and torch.equal(lc.enc_v, v)
    k2, v2 = torch.randn(3, S + 2, HEADS, E // HEADS), torch.randn(3, S + 2, HEADS, E // HEADS)
    lc.store_encoder(k2, v2)
    assert lc.enc_k is not ek and torch.equal(lc.enc_k, k2) and torch.equal(lc.enc_v, v2)


@pytest.mark.parametrize("T", [1, 4])
def test_fixed_width_rel_pos_bias_extends_the_bias_at_the_bound(T):
    m = _decoder()
    cache, _, _ = _prefilled(m)
    cache.seqlens.copy_(torch.tensor([9, 4, 6], dtype=torch.int32))
    like = torch.empty(0)
    cols = cache.capacity + (-cache.capacity % 8 if T > 1 else 0)
    with torch.no_grad():
        now = m._step_rel_pos_bias(cache, like, T)
        wide = m._step_rel_pos_bias(cache, like, T, cols)
    assert wide.shape == (3, HEADS, T, cols)
    assert now.shape[-1] >= cache.max_len + T
    assert torch.equal(wide[..., :now.shape[-1]], now)


def test_capture_step_needs_cuda():
    m = _decoder()
    cache, _, enc_pad = _prefilled(m)
    with pytest.raises(RuntimeError, match="CUDA"):
        m.capture_step(cache, encoder_padding_mask=enc_pad)
