"""Multi-head attention modules.

Parity: reference ``unicore/modules/multihead_attention.py`` - ``SelfMultiheadAttention:12``
(packed ``in_proj``, ``scaling = (head_dim * scaling_factor) ** -0.5``, additive ``attn_bias``,
boolean ``key_padding_mask``, ``return_attn`` yielding ``(out, pre-softmax logits incl. bias,
probabilities)``) and ``CrossMultiheadAttention:121``.

GPU path: the whole ``QK^T -> +bias/mask -> softmax -> dropout -> @V`` chain runs in the wgmma kernel
behind ``ops.fused_attention`` for every head dim the kernel takes (a multiple of 8 up to 128,
``ops.fused_head_dim_supported``); q/k/v are strided views of the projection output (no
transpose/contiguous copies) and the bias is *not* expanded over the batch.  ``return_attn=True,
need_probs=False`` (the caller wants the logits but not the probabilities, as Uni-Mol's pair stack does)
runs in the same kernel in its logits mode, which also writes the logits; its third result is ``None``.
With the probabilities requested (``return_attn`` and the default ``need_probs=True``), or another head
dim, or on the CPU, the materialised path (bmm + ``softmax_dropout`` kernel) is used.

``causal=True`` on ``SelfMultiheadAttention`` hides key ``j`` from query ``i`` when ``j > i``.  The fused path passes it
to the kernel as a flag (no mask tensor); the materialised path adds the future mask ``triu(-inf, 1)`` to the bias, so
its logits are those of the same call with that mask in ``attn_bias``.

``num_kv_heads`` (grouped-query attention): the keys and values have ``H_kv`` heads, each shared by ``H / H_kv``
consecutive query heads (``repeat_interleave`` order).  ``None`` or ``num_heads`` keeps the parameters and checkpoints
of plain multi-head attention; otherwise ``SelfMultiheadAttention.in_proj`` projects to ``(H + 2 * H_kv) * D`` (q, k, v
head slices in that order) and ``CrossMultiheadAttention.k_proj`` / ``v_proj`` to ``H_kv * D``.  The fused kernels read
the shared heads as they are; the materialised path expands them, and autograd sums the expanded gradients.

``rotary_dim`` (rotary position embeddings, ``ops.rotary_embedding``): ``SelfMultiheadAttention`` rotates the first
``rotary_dim`` columns of every query and key head right after ``in_proj`` (rotate-half form, frequencies
``1 / rotary_base ** (2i / rotary_dim)``), before anything reads the projection: the fused and materialised attention,
the prefill's ``store_prefix`` (the cache holds rotated keys) and a step's ``k_new``.  Positions are ``0 .. L-1`` on a
whole sequence or a prefill, ``seqlens[b] + i`` on a decoding step, read on the device.  ``None`` (the default) rotates
nothing; the frequencies are a non-persistent buffer, so ``state_dict`` keys are the same either way.  Cross-attention is
never rotated.

``cu_seqlens`` / ``max_seqlen`` on ``SelfMultiheadAttention``: the input is B sequences packed back to back, ``[N, E]``
with sequence ``b`` on rows ``cu_seqlens[b] .. cu_seqlens[b + 1] - 1`` (int ``[B + 1]`` on the device) and
``max_seqlen`` a host bound on the lengths; the output is packed too.  No row is padding, so the projections do no work
on pad rows, and the attention runs in the varlen mode of the fused kernels (``ops.fused_attention_varlen``; the
varlen reference elsewhere).  ``attn_bias`` is ``[1|B, H, max_seqlen, max_seqlen]`` (each sequence reads its top-left
block); rotary positions restart at 0 in every sequence.  No key padding mask, logits or probabilities.  With a
``cache`` the packed rows are each sequence's new tokens (a different count per sequence, 0 included): they are
appended at ``seqlens[b] + i``, rotated at those positions, and attend to the cache up to their own position
(``ops.attention_with_kv_cache_varlen``), ``attn_bias`` then holding ``[1|B, H, max_seqlen, Lb]`` rows of the new
queries.  On an empty cache this is the prefill; there is one packed path for both.
``CrossMultiheadAttention`` takes a packed query ``[N_q, E]`` (``cu_seqlens`` / ``max_seqlen``) with packed keys and
values ``[N_k, E]`` (``encoder_cu_seqlens`` / ``encoder_max_seqlen``, the same B sequences) and returns ``[N_q, E]``:
query ``i`` of sequence ``b`` sees the keys of source sequence ``b`` only, in the varlen mode of the fused kernels with
separate key sequences.  ``attn_bias`` is then ``[B*H | B | H, max_seqlen, encoder_max_seqlen]``; a sequence without
source rows gives 0.  No key padding mask.  A packed query with a ``cache`` and padded ``key`` / ``value [B, S, E]``
(no ``encoder_cu_seqlens``) is a decoding call: the prefill stores the projected keys / values as the padded path does,
and every packed call attends to them with ``key_padding_mask [B, S]`` (``ops.attention_with_kv_cache_varlen``).

``DecoderCache`` holds what incremental decoding keeps between steps: per layer the self-attention keys and values
``[B, C, H_kv, D]`` and the projected encoder keys and values, the device lengths and a host bound on them.  A step may
add one token or a chunk of several per sequence, and ``rewind`` drops tokens again.  A paged ``DecoderCache``
(``block_size`` set) keeps the self-attention keys and values in pools ``[num_blocks, block_size, H_kv, D]`` per layer
instead, with one block table, free stack and overflow flag shared by the layers: a sequence holds blocks only for the
rows it has, and gives them back when it is rewound.
"""
from typing import Optional

import torch
from torch import Tensor, nn

from unicore import ops
from unicore_b200.ops.attention_ops import _fused_attention, _fused_attention_varlen, _paged_gather, _split_packed


def _bias_as_4d(attn_bias: Optional[Tensor], bsz: int, heads: int, tgt: int, src: int) -> Optional[Tensor]:
    """Normalise the accepted bias layouts to ``[1|B, H, tgt, src]``."""
    if attn_bias is None:
        return None
    if attn_bias.dim() == 4:
        return attn_bias
    if attn_bias.dim() == 3:
        lead = attn_bias.shape[0]
        if lead == bsz * heads:
            return attn_bias.view(bsz, heads, tgt, src)
        if lead == heads:
            return attn_bias.view(1, heads, tgt, src)
    if attn_bias.dim() == 2:
        return attn_bias.view(1, 1, tgt, src).expand(1, heads, tgt, src)
    raise ValueError("unsupported attn_bias shape {}".format(tuple(attn_bias.shape)))


def _add_future_mask(bias4: Optional[Tensor], heads: int, seq_len: int, like: Tensor) -> Tensor:
    """``bias4`` (``[1|B, H, L, L]`` or None) plus the causal mask: ``-inf`` where key > query."""
    fm = torch.full((seq_len, seq_len), float("-inf"), dtype=like.dtype, device=like.device).triu(1)
    if bias4 is None:
        return fm.view(1, 1, seq_len, seq_len).expand(1, heads, seq_len, seq_len)
    return bias4 + fm


def _materialised_attention(qh, kh, vh, key_padding_mask, attn_bias4, dropout, training, return_attn):
    """qh, kh, vh: head-major ``[B, H, L, D]`` (contiguous, query already scaled).

    Returns ``(out [B, Lq, H*D], logits?, probs?)``; scores are materialised (``return_attn`` / head dims the
    wgmma kernel does not cover).  Parity: reference ``multihead_attention.py:78-118``.
    """
    bsz, heads, tgt_len, dim = qh.shape
    src_len = kh.shape[2]
    w4 = torch.bmm(qh.view(bsz * heads, tgt_len, dim), kh.view(bsz * heads, src_len, dim).transpose(1, 2))
    w4 = w4.view(bsz, heads, tgt_len, src_len)
    pad = None
    if key_padding_mask is not None:
        # additive [B, 1, 1, K] mask: consumed by the softmax kernel's broadcast instead of a masked_fill_ pass
        pad = torch.zeros(bsz, 1, 1, src_len, dtype=w4.dtype, device=w4.device)
        pad.masked_fill_(key_padding_mask[:, None, None, :].to(torch.bool), float("-inf"))
    bias = attn_bias4.to(w4.dtype) if attn_bias4 is not None else None
    if not return_attn:
        attn = ops.softmax_dropout(w4, dropout, training, mask=pad, bias=bias)
        logits = probs = None
    else:
        # logits (scores + mask + bias) are an output: the pair representation of the next layer
        attn, logits = ops.softmax_dropout_with_logits(w4, dropout, training, mask=pad, bias=bias)
        logits = logits.view(bsz * heads, tgt_len, src_len)
        probs = attn.view(bsz * heads, tgt_len, src_len)
    out = torch.bmm(attn.view(bsz * heads, tgt_len, src_len), vh.view(bsz * heads, src_len, dim))
    return ops.merge_heads(out.view(bsz, heads, tgt_len, dim)), logits, probs


def _kv_heads(num_heads, num_kv_heads):
    """The key / value head count: ``num_heads`` for ``None``; it must divide ``num_heads``."""
    if num_kv_heads is None:
        return num_heads
    if num_kv_heads < 1 or num_heads % num_kv_heads != 0:
        raise ValueError("num_kv_heads {} must divide num_heads {}".format(num_kv_heads, num_heads))
    return num_kv_heads


def _rotary_dim(rotary_dim, head_dim):
    """``rotary_dim`` checked: ``None`` (no rotation) or an even count of columns in ``[2, head_dim]``."""
    if rotary_dim is None:
        return None
    if int(rotary_dim) != rotary_dim or rotary_dim % 2 != 0 or not 2 <= rotary_dim <= head_dim:
        raise ValueError("rotary_dim {} must be even and in [2, head_dim = {}]".format(rotary_dim, head_dim))
    return int(rotary_dim)


def _expand_heads(x, groups):
    """``[B, H_kv, L, D]`` -> ``[B, H_kv * groups, L, D]``, each head repeated for the query heads of its group."""
    return x if groups == 1 else x.repeat_interleave(groups, dim=1)


class SelfMultiheadAttention(nn.Module):
    def __init__(self, embed_dim, num_heads, dropout=0.1, bias=True, scaling_factor=1, num_kv_heads=None,
                 rotary_dim=None, rotary_base=10000.0):
        super().__init__()
        self.embed_dim = embed_dim
        self.num_heads = num_heads
        self.num_kv_heads = _kv_heads(num_heads, num_kv_heads)
        self.dropout = dropout
        self.head_dim = embed_dim // num_heads
        if self.head_dim * num_heads != embed_dim:
            raise ValueError("embed_dim must be divisible by num_heads")
        self.scaling = (self.head_dim * scaling_factor) ** -0.5
        self.in_proj = nn.Linear(embed_dim, (num_heads + 2 * self.num_kv_heads) * self.head_dim, bias=bias)
        self.out_proj = nn.Linear(embed_dim, embed_dim, bias=bias)
        self.rotary_dim = _rotary_dim(rotary_dim, self.head_dim)
        self.rotary_base = rotary_base
        if self.rotary_dim is not None:
            self.register_buffer("inv_freq", ops.rotary_inv_freq(self.rotary_dim, rotary_base), persistent=False)

    def _apply(self, fn, *args, **kwargs):
        # .half() / .to(dtype) cast floating buffers too; the frequencies stay the fp32 values they were built as
        super()._apply(fn, *args, **kwargs)
        if self.rotary_dim is not None and self.inv_freq.dtype != torch.float32:
            self.inv_freq = ops.rotary_inv_freq(self.rotary_dim, self.rotary_base).to(self.inv_freq.device)
        return self

    def attend(self, query, key_padding_mask=None, attn_bias=None, return_attn=False, need_probs=True, causal=False,
               cache=None, cu_seqlens=None, max_seqlen=None):
        """Everything up to (not including) ``out_proj``: returns ``(o [B, L, E], logits, probs)``.

        ``need_probs=False`` returns ``probs = None``; with ``return_attn`` the fused kernel then also computes the
        logits ``[B*H, L, L]`` where it takes the shapes.  ``causal`` hides key j from query i when j > i (see the module
        docstring).  ``cache`` (a ``LayerKVCache`` of a ``DecoderCache``): on the prefill the keys and values of the L
        positions are also stored in it; on a decoding step (``query [B, T, E]``, one token or a chunk) the new tokens'
        keys and values are appended and their queries attend to the cached keys up to their own positions
        (``ops.attention_with_kv_cache``), with ``attn_bias`` the ``[B, H, T, Lb]`` rows of the new queries.
        ``cu_seqlens`` / ``max_seqlen``: packed sequences, ``query [N, E]`` -> ``o [N, E]`` (see the module
        docstring)."""
        if cu_seqlens is not None:
            return self._attend_packed(query, key_padding_mask, attn_bias, return_attn, causal, cache, cu_seqlens,
                                       max_seqlen)
        bsz, tgt_len, embed_dim = query.size()
        if embed_dim != self.embed_dim:
            raise ValueError("query dim {} != embed_dim {}".format(embed_dim, self.embed_dim))
        if key_padding_mask is not None and key_padding_mask.dim() == 0:
            key_padding_mask = None
        H, H_kv = self.num_heads, self.num_kv_heads
        qkv = ops.linear(query, self.in_proj.weight, self.in_proj.bias).view(bsz, tgt_len, H + 2 * H_kv, self.head_dim)
        if self.rotary_dim is not None:
            # q and k are the leading H + H_kv heads of the projection
            offsets = cache.seqlens if cache is not None and cache.stepping else None
            qkv = ops.rotary_embedding(qkv, self.inv_freq, H + H_kv, offsets)
        q, k, v = _split_packed(qkv, H_kv)   # strided views: q [B, L, H, D], k / v [B, L, H_kv, D]
        if cache is not None and cache.stepping:
            if return_attn:
                raise ValueError("a decoding step does not return attention weights")
            o = ops.attention_with_kv_cache(q, cache.k, cache.v, cache.seqlens, cache.max_len, k_new=k, v_new=v,
                                            bias=attn_bias, scale=self.scaling, block_table=cache.block_table)
            return o.reshape(bsz, tgt_len, embed_dim), None, None
        if cache is not None:
            cache.store_prefix(k, v)
        bias4 = _bias_as_4d(attn_bias, bsz, self.num_heads, tgt_len, tgt_len)
        if (not return_attn or not need_probs) and ops.fused_attention_supported(q, k, v, bias4, key_padding_mask):
            res = _fused_attention(q, k, v, bias4, key_padding_mask, self.dropout, self.training, self.scaling,
                                   return_attn, causal, qkv, supported=True)
            if not return_attn:
                return res.reshape(bsz, tgt_len, embed_dim), None, None
            o, logits = res
            return o.reshape(bsz, tgt_len, embed_dim), logits.view(bsz * self.num_heads, tgt_len, tgt_len), None
        if H_kv == H:
            qh, kh, vh = ops.split_heads(qkv.view(bsz, tgt_len, 3 * embed_dim), 3, self.num_heads, self.scaling)
        else:
            qh = (q * self.scaling).transpose(1, 2).contiguous()
            kh = _expand_heads(k.transpose(1, 2), H // H_kv).contiguous()
            vh = _expand_heads(v.transpose(1, 2), H // H_kv).contiguous()
        if causal:
            bias4 = _add_future_mask(bias4, self.num_heads, tgt_len, qh)
        o, logits, probs = _materialised_attention(qh, kh, vh, key_padding_mask, bias4, self.dropout, self.training,
                                                   return_attn)
        return o, logits, (probs if need_probs else None)

    def _attend_packed(self, query, key_padding_mask, attn_bias, return_attn, causal, cache, cu_seqlens, max_seqlen):
        if return_attn:
            raise ValueError("packed sequences (cu_seqlens) do not return attention weights")
        if key_padding_mask is not None:
            raise ValueError("packed sequences (cu_seqlens) take no key padding mask")
        if max_seqlen is None:
            raise ValueError("cu_seqlens needs max_seqlen, a host bound on the lengths")
        total, embed_dim = query.size()
        if embed_dim != self.embed_dim:
            raise ValueError("query dim {} != embed_dim {}".format(embed_dim, self.embed_dim))
        H, H_kv, D = self.num_heads, self.num_kv_heads, self.head_dim
        qkv = ops.linear(query, self.in_proj.weight, self.in_proj.bias).view(total, H + 2 * H_kv, D)
        if self.rotary_dim is not None:
            # one token per row of the rotary op, at its position inside its sequence (after the cached tokens)
            pos = ops.varlen_positions(cu_seqlens, total, None if cache is None else cache.seqlens)
            qkv = ops.rotary_embedding(qkv.view(total, 1, H + 2 * H_kv, D), self.inv_freq, H + H_kv, pos)
            qkv = qkv.view(total, H + 2 * H_kv, D)
        q, k, v = (t[:, 0] for t in _split_packed(qkv[:, None], H_kv))
        if cache is not None:   # the prefill (from seqlens = 0) and every step alike: append, then attend
            o = ops.attention_with_kv_cache_varlen(q, cache.k, cache.v, cu_seqlens, max_seqlen, cache.seqlens,
                                                   cache.max_len, k_new=k, v_new=v, bias=attn_bias, scale=self.scaling,
                                                   block_table=cache.block_table)
            return o.reshape(total, embed_dim), None, None
        bias4 = _bias_as_4d(attn_bias, cu_seqlens.numel() - 1, H, max_seqlen, max_seqlen)
        o = _fused_attention_varlen(q, k, v, cu_seqlens, max_seqlen, bias4, self.dropout, self.training, self.scaling,
                                    causal, qkv)
        return o.reshape(total, embed_dim), None, None

    def forward(
        self,
        query,
        key_padding_mask: Optional[Tensor] = None,
        attn_bias: Optional[Tensor] = None,
        return_attn: bool = False,
        need_probs: bool = True,
        causal: bool = False,
        cu_seqlens: Optional[Tensor] = None,
        max_seqlen: Optional[int] = None,
    ) -> Tensor:
        o, logits, probs = self.attend(query, key_padding_mask, attn_bias, return_attn, need_probs, causal,
                                       cu_seqlens=cu_seqlens, max_seqlen=max_seqlen)
        o = self.out_proj(o)
        return (o, logits, probs) if return_attn else o


class CrossMultiheadAttention(nn.Module):
    def __init__(self, embed_dim, num_heads, dropout=0.1, bias=True, scaling_factor=1, num_kv_heads=None):
        super().__init__()
        self.embed_dim = embed_dim
        self.num_heads = num_heads
        self.num_kv_heads = _kv_heads(num_heads, num_kv_heads)
        self.dropout = dropout
        self.head_dim = embed_dim // num_heads
        if self.head_dim * num_heads != embed_dim:
            raise ValueError("embed_dim must be divisible by num_heads")
        self.scaling = (self.head_dim * scaling_factor) ** -0.5
        kv_dim = self.num_kv_heads * self.head_dim
        self.q_proj = nn.Linear(embed_dim, embed_dim, bias=bias)
        self.k_proj = nn.Linear(embed_dim, kv_dim, bias=bias)
        self.v_proj = nn.Linear(embed_dim, kv_dim, bias=bias)
        self.out_proj = nn.Linear(embed_dim, embed_dim, bias=bias)

    def attend(self, query, key, value, key_padding_mask=None, attn_bias=None, cache=None, cu_seqlens=None,
               max_seqlen=None, encoder_cu_seqlens=None, encoder_max_seqlen=None):
        """Everything up to (not including) ``out_proj``.

        ``cache`` (a ``LayerKVCache``): the projected keys and values are computed once, on the prefill, and kept in
        it; a decoding step (``query [B, T, E]``, ``key`` / ``value`` unused) attends to them with
        ``ops.attention_with_kv_cache``, ``attn_bias`` holding the rows of the T new queries.
        ``cu_seqlens`` / ``max_seqlen`` and ``encoder_cu_seqlens`` / ``encoder_max_seqlen``: packed sequences, ``query
        [N_q, E]`` and ``key`` / ``value`` ``[N_k, E]`` -> ``o [N_q, E]`` (see the module docstring)."""
        if cu_seqlens is not None or encoder_cu_seqlens is not None:
            return self._attend_packed(query, key, value, key_padding_mask, attn_bias, cache, cu_seqlens, max_seqlen,
                                       encoder_cu_seqlens, encoder_max_seqlen)
        bsz, tgt_len, embed_dim = query.size()
        if embed_dim != self.embed_dim:
            raise ValueError("query dim {} != embed_dim {}".format(embed_dim, self.embed_dim))
        if key_padding_mask is not None and key_padding_mask.dim() == 0:
            key_padding_mask = None
        q = self.q_proj(query).view(bsz, tgt_len, self.num_heads, self.head_dim)
        if cache is not None and cache.stepping:
            src_len = cache.enc_k.size(1)
            bias4 = _bias_as_4d(attn_bias, bsz, self.num_heads, tgt_len, src_len)
            o = ops.attention_with_kv_cache(q, cache.enc_k, cache.enc_v, bias=bias4,
                                            key_padding_mask=key_padding_mask, scale=self.scaling)
            return o.reshape(bsz, tgt_len, embed_dim)
        src_len = key.size(1)
        H_kv = self.num_kv_heads
        k = self.k_proj(key).view(bsz, src_len, H_kv, self.head_dim)
        v = self.v_proj(value).view(bsz, src_len, H_kv, self.head_dim)
        if cache is not None:
            cache.store_encoder(k, v)
        bias4 = _bias_as_4d(attn_bias, bsz, self.num_heads, tgt_len, src_len)
        if ops.fused_attention_supported(q, k, v, bias4, key_padding_mask):
            return _fused_attention(q, k, v, bias4, key_padding_mask, self.dropout, self.training, self.scaling,
                                    False, False, supported=True).reshape(bsz, tgt_len, embed_dim)
        (qh,) = ops.split_heads(q.view(bsz, tgt_len, embed_dim), 1, self.num_heads, self.scaling)
        (kh,) = ops.split_heads(k.view(bsz, src_len, H_kv * self.head_dim), 1, H_kv)
        (vh,) = ops.split_heads(v.view(bsz, src_len, H_kv * self.head_dim), 1, H_kv)
        kh = _expand_heads(kh, self.num_heads // H_kv).contiguous()
        vh = _expand_heads(vh, self.num_heads // H_kv).contiguous()
        o, _, _ = _materialised_attention(qh, kh, vh, key_padding_mask, bias4, self.dropout, self.training, False)
        return o

    def _attend_packed(self, query, key, value, key_padding_mask, attn_bias, cache, cu_seqlens, max_seqlen,
                       encoder_cu_seqlens, encoder_max_seqlen):
        if cache is not None and cu_seqlens is not None and encoder_cu_seqlens is None:
            return self._attend_packed_cached(query, key, value, key_padding_mask, attn_bias, cache, cu_seqlens,
                                              max_seqlen)
        if cu_seqlens is None or encoder_cu_seqlens is None:
            raise ValueError("packed cross-attention takes a packed query (cu_seqlens) and packed keys / values "
                             "(encoder_cu_seqlens) together")
        if key_padding_mask is not None or cache is not None:
            raise ValueError("packed sequences (cu_seqlens) take neither a key padding mask nor a cache")
        if max_seqlen is None or encoder_max_seqlen is None:
            raise ValueError("cu_seqlens / encoder_cu_seqlens need max_seqlen / encoder_max_seqlen, host bounds on "
                             "the lengths")
        if encoder_cu_seqlens.dim() != 1 or encoder_cu_seqlens.numel() != cu_seqlens.numel():
            raise ValueError("encoder_cu_seqlens must describe the B = {} sequences of cu_seqlens, not {}".format(
                cu_seqlens.numel() - 1, tuple(encoder_cu_seqlens.shape)))
        total, embed_dim = query.size()
        if embed_dim != self.embed_dim:
            raise ValueError("query dim {} != embed_dim {}".format(embed_dim, self.embed_dim))
        if key.dim() != 2 or value.dim() != 2:
            raise ValueError("packed cross-attention takes key / value [N_k, E]")
        H, H_kv, D = self.num_heads, self.num_kv_heads, self.head_dim
        q = self.q_proj(query).view(total, H, D)
        k = self.k_proj(key).view(key.size(0), H_kv, D)
        v = self.v_proj(value).view(value.size(0), H_kv, D)
        bias4 = _bias_as_4d(attn_bias, cu_seqlens.numel() - 1, H, max_seqlen, encoder_max_seqlen)
        o = _fused_attention_varlen(q, k, v, cu_seqlens, max_seqlen, bias4, self.dropout, self.training, self.scaling,
                                    False, cu_seqlens_k=encoder_cu_seqlens, max_seqlen_k=encoder_max_seqlen)
        return o.reshape(total, embed_dim)

    def _attend_packed_cached(self, query, key, value, key_padding_mask, attn_bias, cache, cu_seqlens, max_seqlen):
        """A packed query ``[N, E]`` against the encoder keys / values of ``cache``: the prefill projects and stores the
        padded ``key`` / ``value [B, S, E]`` first.  ``key_padding_mask [B, S]``; ``attn_bias [B*H | B | H, max_seqlen,
        S]`` or ``[1|B, H, max_seqlen, S]``, row i for query i of every sequence."""
        if max_seqlen is None:
            raise ValueError("cu_seqlens needs max_seqlen, a host bound on the lengths")
        total, embed_dim = query.size()
        if embed_dim != self.embed_dim:
            raise ValueError("query dim {} != embed_dim {}".format(embed_dim, self.embed_dim))
        B, H, H_kv, D = cu_seqlens.numel() - 1, self.num_heads, self.num_kv_heads, self.head_dim
        if not cache.stepping:
            if key is None or key.dim() != 3 or key.size(0) != B:
                raise ValueError("the prefill of a packed query stores a padded encoder_out [B = {}, S, E]".format(B))
            src_len = key.size(1)
            cache.store_encoder(self.k_proj(key).view(B, src_len, H_kv, D), self.v_proj(value).view(B, src_len, H_kv, D))
        src_len = cache.enc_k.size(1)
        if attn_bias is not None and attn_bias.dim() == 3 and attn_bias.shape[0] not in (B * H, H):
            attn_bias = attn_bias.view(B, 1, max_seqlen, src_len)   # [B, ...]: the same rows for every head
        bias4 = _bias_as_4d(attn_bias, B, H, max_seqlen, src_len)
        q = self.q_proj(query).view(total, H, D)
        o = ops.attention_with_kv_cache_varlen(q, cache.enc_k, cache.enc_v, cu_seqlens, max_seqlen, bias=bias4,
                                               key_padding_mask=key_padding_mask, scale=self.scaling)
        return o.reshape(total, embed_dim)

    def forward(
        self,
        query,
        key,
        value,
        key_padding_mask: Optional[Tensor] = None,
        attn_bias: Optional[Tensor] = None,
        cu_seqlens: Optional[Tensor] = None,
        max_seqlen: Optional[int] = None,
        encoder_cu_seqlens: Optional[Tensor] = None,
        encoder_max_seqlen: Optional[int] = None,
    ) -> Tensor:
        return self.out_proj(self.attend(query, key, value, key_padding_mask, attn_bias, cu_seqlens=cu_seqlens,
                                         max_seqlen=max_seqlen, encoder_cu_seqlens=encoder_cu_seqlens,
                                         encoder_max_seqlen=encoder_max_seqlen))


def _same_layout(a: Tensor, b: Tensor) -> bool:
    return a.shape == b.shape and a.dtype == b.dtype and a.device == b.device


class LayerKVCache:
    """One decoder layer's share of a ``DecoderCache``: self-attention keys / values ``k``, ``v`` ``[B, C, H_kv, D]``
    (pools ``[num_blocks, block_size, H_kv, D]`` of a paged cache) and the projected encoder keys / values ``enc_k``,
    ``enc_v`` ``[B, S, H_kv, D]`` (None until the prefill stores them)."""

    def __init__(self, owner, k, v):
        self.owner = owner
        self.k, self.v = k, v
        self.enc_k = self.enc_v = None

    @property
    def stepping(self):
        """False on the prefill (the first call on an empty cache), True on every decoding step after it."""
        return self.owner.max_len > 0

    @property
    def seqlens(self):
        return self.owner.seqlens

    @property
    def max_len(self):
        return self.owner.max_len

    @property
    def block_table(self):
        """The paged cache's ``[B, M]`` block table, None for a contiguous cache."""
        return self.owner.block_table

    def store_prefix(self, k, v):
        """Rows ``0 .. L-1`` of the self-attention cache from the prefill's ``[B, L, H, D]`` keys and values (through
        the block table of a paged cache, whose rows without a block are skipped)."""
        with torch.no_grad():
            if self.block_table is not None:
                ops.kv_cache_append(k, v, self.k, self.v, torch.zeros_like(self.seqlens), self.block_table)
                return
            self.k[:, :k.size(1)].copy_(k)
            self.v[:, :v.size(1)].copy_(v)

    def store_encoder(self, k, v):
        """Keep the prefill's projected encoder keys / values.  A later prefill of the same shape writes into the
        tensors kept before, so that their addresses stay valid (a captured decoding step reads them)."""
        if self.enc_k is not None and _same_layout(self.enc_k, k) and _same_layout(self.enc_v, v):
            with torch.no_grad():
                self.enc_k.copy_(k)
                self.enc_v.copy_(v)
        else:
            self.enc_k, self.enc_v = k.detach(), v.detach()

    def _reorder_encoder(self, index):
        if self.enc_k is None:
            return
        if index.numel() != self.enc_k.size(0):
            self.enc_k, self.enc_v = self.enc_k.index_select(0, index), self.enc_v.index_select(0, index)
            return
        with torch.no_grad():
            for buf in (self.enc_k, self.enc_v):
                buf.copy_(buf.index_select(0, index))

    def reorder(self, index):
        """In place when ``index`` keeps the batch size: only the rows below the host bound ``max_len`` can be read,
        so only they are gathered (into a temporary) and written back.  A new batch size rebinds the buffers."""
        n = self.owner.max_len
        if index.numel() != self.k.size(0):
            self.k, self.v = self.k.index_select(0, index), self.v.index_select(0, index)
        else:
            with torch.no_grad():
                for buf in (self.k[:, :n], self.v[:, :n]):
                    buf.copy_(buf.index_select(0, index))
        self._reorder_encoder(index)


class DecoderCache:
    """State of incremental decoding for a ``TransformerDecoder`` (made by ``TransformerDecoder.new_cache``).

    ``layers``: one ``LayerKVCache`` per layer.  ``seqlens``: int32 ``[B]`` on the device, the tokens decoded so far per
    sequence (the position of the next one).  ``max_len``: a host-side upper bound on ``seqlens`` (0 = empty cache), so
    that no step has to read the device lengths.  ``capacity``: rows of the self-attention buffers per sequence.
    ``heads``: the key / value heads of the layers (``H_kv`` under grouped-query attention).

    Paged (``block_size`` set): every layer's ``k`` / ``v`` is a pool ``[num_blocks, block_size, H_kv, D]``, and the
    layers share ``block_table`` (int32 ``[B, capacity / block_size]``, -1 = no block), the free stack ``free_list``
    (int32 ``[num_blocks]``, top at ``free_count - 1``), ``free_count`` and ``overflow`` (int32 ``[1]`` each, on the
    device).  Every call that adds tokens reserves blocks for them first (``reserve``), ``rewind`` releases the blocks
    past the new lengths, and a pool that runs out sets ``overflow`` (the rows without a block are then not stored).
    The first blocks handed out are 0, 1, 2, ...  Otherwise the cache behaves as the contiguous one."""

    def __init__(self, num_layers, batch_size, capacity, heads, head_dim, dtype, device, block_size=None,
                 num_blocks=None):
        self.capacity = capacity
        self.seqlens = torch.zeros(batch_size, dtype=torch.int32, device=device)
        self.max_len = 0
        self.block_size = block_size
        self.block_table = self.free_list = self.free_count = self.overflow = None
        if block_size is None:
            shape = (batch_size, capacity, heads, head_dim)
        else:
            shape = (num_blocks, block_size, heads, head_dim)
            self.block_table = torch.full((batch_size, capacity // block_size), -1, dtype=torch.int32, device=device)
            self.free_list = torch.arange(num_blocks - 1, -1, -1, dtype=torch.int32, device=device)
            self.free_count = torch.full((1,), num_blocks, dtype=torch.int32, device=device)
            self.overflow = torch.zeros(1, dtype=torch.int32, device=device)
        self.layers = [
            LayerKVCache(self, torch.zeros(shape, dtype=dtype, device=device),
                         torch.zeros(shape, dtype=dtype, device=device))
            for _ in range(num_layers)
        ]

    @property
    def paged(self):
        return self.block_size is not None

    def reserve(self, lengths):
        """Paged: blocks for every row below ``lengths[b]`` (int ``[B]`` on the device) that has none, before a call
        stores those rows.  Nothing is read on the host.  A no-op for a contiguous cache."""
        if self.paged:
            ops.kv_blocks_reserve(self.block_table, self.free_list, self.free_count, lengths, self.block_size,
                                  self.overflow)

    def _release(self):
        """Paged: the blocks past ``seqlens`` back onto the free stack."""
        if self.paged:
            ops.kv_blocks_release(self.block_table, self.free_list, self.free_count, self.seqlens, self.block_size)

    def free_blocks(self):
        """Paged: the blocks on the free stack (reads the device, so it synchronises)."""
        return int(self.free_count.item())

    def overflowed(self):
        """Paged: whether a reservation has found the pool empty since the cache was made (reads the device)."""
        return bool(self.overflow.item())

    def reorder(self, index):
        """Select (and repeat) sequences of the batch along ``index`` in every buffer, as beam search does.  With as
        many entries as sequences it writes into the existing buffers (a captured decoding step keeps reading them).
        Paged: the rows below ``max_len`` are gathered through the table, every block is released, the sequences
        reserve blocks again in their new order and the rows are written back through the new table, so the contents
        are those of a contiguous cache's ``reorder``."""
        if self.paged:
            self._reorder_paged(index)
            return
        for layer in self.layers:
            layer.reorder(index)
        if index.numel() == self.seqlens.numel():
            self.seqlens.copy_(self.seqlens.index_select(0, index))
        else:
            self.seqlens = self.seqlens.index_select(0, index)

    def _reorder_paged(self, index):
        n, same = self.max_len, index.numel() == self.seqlens.numel()
        rows = []
        if n > 0:
            table = self.block_table[:, :-(-n // self.block_size)]   # the entries of the rows below max_len
            with torch.no_grad():
                for layer in self.layers:
                    k = _paged_gather(layer.k, table)[:, :n].index_select(0, index)
                    v = _paged_gather(layer.v, table)[:, :n].index_select(0, index)
                    rows.append((k, v))
        seqlens = self.seqlens.index_select(0, index)
        self.seqlens.zero_()
        self._release()
        if same:
            self.seqlens.copy_(seqlens)
        else:
            self.seqlens = seqlens
            self.block_table = torch.full((index.numel(), self.block_table.size(1)), -1, dtype=torch.int32,
                                          device=self.block_table.device)
        self.reserve(self.seqlens)
        for layer, (k, v) in zip(self.layers, rows):
            layer.store_prefix(k, v)
        for layer in self.layers:
            layer._reorder_encoder(index)

    def rewind(self, n):
        """Drop the last ``n`` tokens of every sequence (an int), or ``n[b]`` of sequence b (an integer ``[B]`` tensor
        on the device), as speculative decoding does after verifying a chunk of draft tokens: ``seqlens -= n``, clamped
        at 0, without a host synchronisation.  An int also lowers ``max_len``; a tensor leaves it, a valid bound.  The
        rows past ``seqlens`` are never read, so nothing else is reset; rewinding every token empties the cache, and
        the next call is a prefill again.  Paged: the blocks wholly past the new lengths go back to the free stack, so
        a sequence rewound to 0 holds no memory."""
        if isinstance(n, torch.Tensor):
            self.seqlens.sub_(n.to(device=self.seqlens.device, dtype=self.seqlens.dtype)).clamp_(min=0)
            self._release()
            return
        n = int(n)
        if n < 0:
            raise ValueError("rewind takes a count of tokens >= 0, not {}".format(n))
        self.seqlens.sub_(n).clamp_(min=0)
        self.max_len = max(self.max_len - n, 0)
        self._release()
