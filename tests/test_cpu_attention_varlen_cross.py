"""Packed cross-attention (separate key sequences, ``cu_seqlens_k``) and the packed decoder on the CPU, in float64.

``attention_varlen_reference`` with ``cu_seqlens_k`` must be ``attention_reference`` on the scattered padded tensors
with the key-length mask at every real row, with 0 (and zero, finite gradients) at the rows of a sequence without
keys; and the packed ``TransformerDecoder`` must be the padded one at every real row, forward and every gradient."""
import pytest
import torch

from unicore import ops
from unicore.modules import CrossMultiheadAttention
from unicore.modules.transformer import TransformerDecoder

# (query lengths, Lq, key lengths, Lk): n_q = 0, n_k = 0 < n_q, 1, lengths that are not multiples of 8, each max itself
CASES = {
    "lq_lt_lk": ([5, 0, 3, 16, 1, 9], 16, [12, 7, 0, 24, 1, 3]),
    "lq_gt_lk": ([13, 0, 4, 24, 1, 7], 24, [5, 2, 0, 16, 11, 1]),
}


def _lk(case):
    return max(CASES[case][2]) + (-max(CASES[case][2]) % 8)


def _cu(lens):
    return torch.tensor([0] + lens).cumsum(0).to(torch.int32)


def _scatter(x, lens, L):
    out = x.new_zeros(len(lens), L, *x.shape[1:])
    s = 0
    for b, n in enumerate(lens):
        out[b, :n] = x[s:s + n]
        s += n
    return out


def _gather(xp, lens):
    return torch.cat([xp[b, :n] for b, n in enumerate(lens)])


def _qkv(case, H, H_kv, bias_batch, D=8, seed=0):
    lq, Lq, lk = CASES[case]
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(sum(lq), H, D, generator=g, dtype=torch.float64)
    k, v = (torch.randn(sum(lk), H_kv, D, generator=g, dtype=torch.float64) for _ in range(2))
    bias = None if bias_batch is None else torch.randn(bias_batch, H, Lq, _lk(case), generator=g, dtype=torch.float64)
    return q, k, v, bias


@pytest.mark.parametrize("bias_batch", [None, 1, 6])
@pytest.mark.parametrize("H,H_kv", [(4, 4), (4, 2), (4, 1)])
@pytest.mark.parametrize("case", list(CASES))
def test_reference_is_the_padded_call_with_the_key_length_mask(case, H, H_kv, bias_batch):
    lq, Lq, lk = CASES[case]
    Lk = _lk(case)
    q, k, v, bias = _qkv(case, H, H_kv, bias_batch)
    out = ops.attention_varlen_reference(q, k, v, _cu(lq), Lq, bias, cu_seqlens_k=_cu(lk), max_seqlen_k=Lk)
    assert out.shape == q.shape
    kpm = torch.arange(Lk)[None, :] >= torch.tensor(lk)[:, None]
    want = ops.attention_reference(_scatter(q, lq, Lq), _scatter(k, lk, Lk), _scatter(v, lk, Lk), bias, kpm)
    s = 0
    for b, (nq, nk) in enumerate(zip(lq, lk)):
        if nk > 0:
            torch.testing.assert_close(out[s:s + nq], want[b, :nq], rtol=1e-5, atol=1e-6)
        else:   # no keys: the kernels' fully-masked contract
            assert torch.count_nonzero(out[s:s + nq]) == 0
        s += nq


@pytest.mark.parametrize("H,H_kv", [(4, 4), (4, 2)])
@pytest.mark.parametrize("case", list(CASES))
def test_reference_gradients_are_per_sequence_attention(case, H, H_kv):
    """Gradients through the reference equal those of per-sequence attention; the rows of a sequence without keys get
    zero, finite gradients and contribute nothing to k, v or the bias."""
    lq, Lq, lk = CASES[case]
    Lk = _lk(case)
    q, k, v, bias = (t.requires_grad_(True) for t in _qkv(case, H, H_kv, 6, seed=1))
    out = ops.attention_varlen_reference(q, k, v, _cu(lq), Lq, bias, cu_seqlens_k=_cu(lk), max_seqlen_k=Lk)
    dout = torch.randn_like(out)
    out.backward(dout)
    q2, k2, v2, b2 = (t.detach().clone().requires_grad_(True) for t in (q, k, v, bias))
    parts, sq, sk = [], 0, 0
    for b, (nq, nk) in enumerate(zip(lq, lk)):
        if nk > 0:
            parts.append(ops.attention_reference(q2[None, sq:sq + nq], k2[None, sk:sk + nk], v2[None, sk:sk + nk],
                                                 b2[b:b + 1, :, :nq, :nk])[0])
        else:
            parts.append(q2.new_zeros(nq, H, q.shape[-1]))
        sq, sk = sq + nq, sk + nk
    want = torch.cat(parts)
    want.backward(dout)
    torch.testing.assert_close(out, want, rtol=1e-5, atol=1e-6)
    for got, ref in ((q, q2), (k, k2), (v, v2), (bias, b2)):
        assert bool(torch.isfinite(got.grad).all())
        torch.testing.assert_close(got.grad, ref.grad, rtol=1e-5, atol=1e-6)
    empty = [b for b, n in enumerate(lk) if n == 0 and lq[b] > 0]
    assert empty, "a sequence with queries and no keys"
    for b in empty:
        s = sum(lq[:b])
        assert torch.count_nonzero(q.grad[s:s + lq[b]]) == 0
        assert torch.count_nonzero(bias.grad[b]) == 0


def test_self_description_is_the_self_call():
    """cu_seqlens_k = cu_seqlens with max_seqlen_k = max_seqlen is the self-attention call."""
    lens, L = [5, 0, 1, 16, 9], 16
    g = torch.Generator().manual_seed(2)
    q, k, v = (torch.randn(sum(lens), 2, 8, generator=g, dtype=torch.float64) for _ in range(3))
    want = ops.attention_varlen_reference(q, k, v, _cu(lens), L)
    got = ops.attention_varlen_reference(q, k, v, _cu(lens), L, cu_seqlens_k=_cu(lens).clone(), max_seqlen_k=L)
    assert torch.equal(got, want)


def test_ops_reject_what_they_cannot_do():
    lq, Lq, lk = CASES["lq_lt_lk"]
    q, k, v, _ = _qkv("lq_lt_lk", 4, 4, None)
    for fn in (ops.fused_attention_varlen, ops.attention_varlen_reference):
        with pytest.raises(ValueError):   # causal is not defined with separate key sequences
            fn(q, k, v, _cu(lq), Lq, causal=True, cu_seqlens_k=_cu(lk), max_seqlen_k=24)
        with pytest.raises(ValueError):   # another B
            fn(q, k, v, _cu(lq), Lq, cu_seqlens_k=_cu(lk[:-1]), max_seqlen_k=24)
        with pytest.raises(ValueError):   # no bound on the key lengths
            fn(q, k, v, _cu(lq), Lq, cu_seqlens_k=_cu(lk))
        with pytest.raises(ValueError):   # a key bound without key sequences
            fn(q, q, q, _cu(lq), Lq, max_seqlen_k=24)
    assert not ops.fused_attention_varlen_supported(q, k, v, _cu(lq), Lq, cu_seqlens_k=_cu(lk), max_seqlen_k=24)


# ---- the modules -------------------------------------------------------------------------------------------------
DEC_LQ, DEC_LQ_MAX = [5, 1, 3, 16, 9], 16       # no empty sequence: the padded stack's fully-masked rows are NaN
DEC_LK, DEC_LK_MAX = [12, 7, 1, 20, 3], 24


def _decoder(post_ln, pos, kv_heads):
    torch.manual_seed(3)
    return TransformerDecoder(decoder_layers=2, embed_dim=32, ffn_embed_dim=64, attention_heads=4, emb_dropout=0.0,
                              dropout=0.0, attention_dropout=0.0, max_seq_len=DEC_LK_MAX, rel_pos=pos == "relpos",
                              post_ln=post_ln, attention_kv_heads=kv_heads,
                              rotary_dim=4 if pos == "rotary" else None).double()


@pytest.mark.parametrize("kv_heads", [None, 2], ids=["mha", "gqa"])
@pytest.mark.parametrize("pos", ["relpos", "rotary"])
@pytest.mark.parametrize("post_ln", [True, False], ids=["post_ln", "pre_ln"])
@pytest.mark.parametrize("encoder", [False, True], ids=["decoder_only", "encoder_decoder"])
def test_packed_decoder_is_the_padded_one_at_real_rows(encoder, post_ln, pos, kv_heads):
    dec = _decoder(post_ln, pos, kv_heads)
    g = torch.Generator().manual_seed(4)
    emb = torch.randn(sum(DEC_LQ), 32, generator=g, dtype=torch.float64, requires_grad=True)
    enc = torch.randn(sum(DEC_LK), 32, generator=g, dtype=torch.float64, requires_grad=True) if encoder else None
    packed = dict(cu_seqlens=_cu(DEC_LQ), max_seqlen=DEC_LQ_MAX)
    if encoder:
        packed.update(encoder_cu_seqlens=_cu(DEC_LK), encoder_max_seqlen=DEC_LK_MAX)
    y = dec(emb, encoder_out=enc, **packed)
    assert y.shape == emb.shape
    dy = torch.randn_like(y)
    y.backward(dy)
    grads = {n: p.grad.clone() for n, p in dec.named_parameters() if p.grad is not None}
    dec.zero_grad()

    embp = _scatter(emb.detach(), DEC_LQ, DEC_LQ_MAX).requires_grad_(True)
    pad = torch.arange(DEC_LQ_MAX)[None, :] >= torch.tensor(DEC_LQ)[:, None]
    encp = enc_pad = None
    if encoder:
        encp = _scatter(enc.detach(), DEC_LK, DEC_LK_MAX).requires_grad_(True)
        enc_pad = torch.arange(DEC_LK_MAX)[None, :] >= torch.tensor(DEC_LK)[:, None]
    yp = dec(embp, encoder_out=encp, padding_mask=pad, encoder_padding_mask=enc_pad)
    torch.testing.assert_close(y, _gather(yp, DEC_LQ), rtol=1e-5, atol=1e-6)
    _gather(yp, DEC_LQ).backward(dy)
    torch.testing.assert_close(emb.grad, _gather(embp.grad, DEC_LQ), rtol=1e-5, atol=1e-6)
    if encoder:
        torch.testing.assert_close(enc.grad, _gather(encp.grad, DEC_LK), rtol=1e-5, atol=1e-6)
    want = {n: p.grad for n, p in dec.named_parameters() if p.grad is not None}
    assert set(grads) == set(want)
    for name, gr in grads.items():
        torch.testing.assert_close(gr, want[name], rtol=1e-5, atol=1e-6, msg=name)


def test_packed_cross_attention_is_the_padded_one():
    torch.manual_seed(5)
    attn = CrossMultiheadAttention(32, 4, dropout=0.0, num_kv_heads=2).double()
    g = torch.Generator().manual_seed(6)
    x = torch.randn(sum(DEC_LQ), 32, generator=g, dtype=torch.float64)
    e = torch.randn(sum(DEC_LK), 32, generator=g, dtype=torch.float64)
    bias = torch.randn(len(DEC_LQ) * 4, DEC_LQ_MAX, DEC_LK_MAX, generator=g, dtype=torch.float64)
    y = attn(x, e, e, attn_bias=bias, cu_seqlens=_cu(DEC_LQ), max_seqlen=DEC_LQ_MAX, encoder_cu_seqlens=_cu(DEC_LK),
             encoder_max_seqlen=DEC_LK_MAX)
    ep = _scatter(e, DEC_LK, DEC_LK_MAX)
    enc_pad = torch.arange(DEC_LK_MAX)[None, :] >= torch.tensor(DEC_LK)[:, None]
    yp = attn(_scatter(x, DEC_LQ, DEC_LQ_MAX), ep, ep, key_padding_mask=enc_pad, attn_bias=bias)
    torch.testing.assert_close(y, _gather(yp, DEC_LQ), rtol=1e-5, atol=1e-6)


def test_packed_decoder_rejects_what_it_cannot_do():
    dec = _decoder(False, "relpos", None)
    emb = torch.randn(sum(DEC_LQ), 32, dtype=torch.float64)
    enc = torch.randn(sum(DEC_LK), 32, dtype=torch.float64)
    B = len(DEC_LQ)
    packed = dict(cu_seqlens=_cu(DEC_LQ), max_seqlen=DEC_LQ_MAX)
    packed_enc = dict(encoder_cu_seqlens=_cu(DEC_LK), encoder_max_seqlen=DEC_LK_MAX)
    with pytest.raises(ValueError):   # packed target, padded encoder_out
        dec(emb, encoder_out=torch.randn(B, DEC_LK_MAX, 32, dtype=torch.float64), **packed)
    with pytest.raises(ValueError):   # padded target, packed encoder_out
        dec(torch.randn(B, DEC_LQ_MAX, 32, dtype=torch.float64), encoder_out=enc, **packed_enc)
    with pytest.raises(ValueError):
        dec(emb, encoder_out=enc, padding_mask=torch.zeros(B, DEC_LQ_MAX, dtype=torch.bool), **packed, **packed_enc)
    with pytest.raises(ValueError):
        dec(emb, encoder_out=enc, encoder_padding_mask=torch.zeros(B, DEC_LK_MAX, dtype=torch.bool), **packed,
            **packed_enc)
    with pytest.raises(ValueError):
        dec(emb, encoder_out=enc, cache=dec.new_cache(B, 16), **packed, **packed_enc)
    with pytest.raises(ValueError):   # another B
        dec(emb, encoder_out=enc, encoder_cu_seqlens=_cu(DEC_LK[:-1]), encoder_max_seqlen=DEC_LK_MAX, **packed)
    attn = dec.layers[0].encoder_attn
    with pytest.raises(ValueError):   # mixed forms on the module
        attn(emb, enc, enc, **packed)
    with pytest.raises(ValueError):
        attn(emb, enc, enc, key_padding_mask=torch.zeros(B, DEC_LK_MAX, dtype=torch.bool), **packed, **packed_enc)
