"""Fused multi-head attention: ``softmax(scale * q k^T + bias + key_padding) -> dropout -> @ v``.

The reference materialises the ``[B*H, L, L]`` score tensor three times per layer
(``unicore/modules/multihead_attention.py:47-114``: bmm -> softmax_dropout -> bmm, plus four
transpose+contiguous copies).  The sm_90a kernels (``csrc/attn/fmha_{fwd,bwd}_sm90.cu``) keep scores in
registers: ``wgmma`` computes S = QK^T, the softmax adds the bias tile / padding mask and applies Philox
dropout in registers, and P is the register operand of a second ``wgmma`` that accumulates O += PV.
q/k/v are consumed directly from the packed ``in_proj`` output through strides (no transposes) and O is
written as ``[B, L, H*D]``.  Backward recomputes P from the saved log-sum-exp (flash-attention style) and
reads the dropout keep bits the forward kernel stored.

The kernels take every head dim ``D`` with ``D % 8 == 0`` and ``8 <= D <= 128`` (``fused_head_dim_supported``);
other head dims, and callers that need the probabilities (``return_attn``), use ``attention_reference``.

``return_logits=True`` also returns the logits ``z = scale * q k^T + bias + key_mask`` as ``[B, H, Lq, Lk]`` (the
contract of ``softmax_dropout_with_logits``): the key padding mask is additive, so ``z`` is ``-inf`` at masked keys,
and the gradient ``dz`` of ``z`` is added to the softmax gradient at every position before it reaches q, k and the
bias.  The kernels write ``z`` from the forward pass and take ``dz`` in the backward pass; the probabilities are never
materialised.  Uni-Mol threads ``z`` through its layers as the pair representation.

``causal=True`` lets key ``j`` reach query ``i`` only when ``j <= i``, for any ``Lq`` and ``Lk``: the top-left aligned
mask ``torch.triu(full((Lq, Lk), -inf), 1)``, as the future mask of ``TransformerDecoder`` (not flash-attn's
bottom-right convention when ``Lq != Lk``).  It combines with the bias, the key padding mask and dropout.  The kernels
take it as a flag: no mask tensor is read, and the key tiles above the diagonal are never computed, in the forward or
the backward pass.  ``causal=True`` with ``return_logits=True`` runs ``attention_reference``.

``attention_with_kv_cache`` is the decoding step: T queries per sequence against a ``[B, C, H, D]`` key / value cache,
optionally appending the new tokens' keys and values first.  One query (T = 1) runs in
``csrc/attn/fmha_decode_sm90.cu`` (split-KV, fp32 on the CUDA cores).  A chunk (T > 1: a prompt continued after some
decoding, a chunked prefill, the candidates of speculative decoding) runs in the KV-cache mode of the wgmma forward
(``csrc/attn/fmha_fwd_sm90.cu``), after a small kernel that appends its rows: query ``i`` of sequence ``b`` sees the
cache rows up to ``seqlens[b] + i``, so K and V are streamed once per 64-query tile instead of once per token.  Both
take every head dim the fused kernels take and have no backward.

Paged caches: with ``block_table`` (int ``[B, M]`` on the device) the caches of ``attention_with_kv_cache`` and
``attention_with_kv_cache_varlen`` are pools ``[num_blocks, block_size, H_kv, D]`` shared by all sequences:
``block_table[b, i]`` is the block holding rows ``i * block_size .. (i + 1) * block_size - 1`` of sequence ``b`` (-1:
none), ``block_size`` is a multiple of 128 and the per-sequence capacity is ``C = M * block_size``.  The kernels read
and append through the table and compute bitwise what the contiguous call computes on the cache gathered through it.
An append into a row whose entry is outside ``[0, num_blocks)`` is skipped, and reading such a row gives an unspecified
value.  ``kv_blocks_reserve`` / ``kv_blocks_release`` hand blocks out of a free stack and back, on the device.

Grouped-query attention: every op takes k / v (and the caches) with ``H_kv`` heads where ``H_kv`` divides the ``H``
query heads.  Query head ``h`` reads key / value head ``h // G``, ``G = H // H_kv`` - the order of
``k.repeat_interleave(G, dim=2)`` - and everything else (bias, key mask, dropout, logits, causal) stays per query head,
so the result is that of the same call on K / V expanded that way.  ``G`` comes from the shapes; a head count that
does not divide raises ``ValueError``.  The kernels read each key / value head once per query head that shares it and
never expand it; the backward pass sums dK / dV over each group on chip.  Multi-query attention is ``H_kv = 1``.
"""
import math

import torch
import torch.nn.functional as F

from ._native import native, use_native

FUSED_MAX_HEAD_DIM = 128


def fused_head_dim_supported(head_dim: int) -> bool:
    """True when the fused attention kernels take this head dim: a multiple of 8 from 8 to 128."""
    return 8 <= head_dim <= FUSED_MAX_HEAD_DIM and head_dim % 8 == 0


def kv_group(q_heads, k, v=None):
    """``G = q_heads // H_kv``: the query heads that share each of the ``H_kv`` key / value heads of ``k`` (and ``v``,
    which must have as many).  Raises ``ValueError`` when ``H_kv`` does not divide ``q_heads``."""
    kv_heads = k.shape[2]
    if v is not None and v.shape[2] != kv_heads:
        raise ValueError("k and v must have the same number of heads, not {} and {}".format(kv_heads, v.shape[2]))
    if kv_heads < 1 or q_heads % kv_heads != 0:
        raise ValueError("{} key / value heads do not divide {} query heads".format(kv_heads, q_heads))
    return q_heads // kv_heads


def _expand_kv(q_heads, k, v):
    """k / v with one head per query head: ``repeat_interleave(G, dim=2)`` (unchanged when G = 1)."""
    G = kv_group(q_heads, k, v)
    if G == 1:
        return k, v
    return k.repeat_interleave(G, dim=2), v.repeat_interleave(G, dim=2)


def attention_reference(q, k, v, bias=None, key_padding_mask=None, dropout_p=0.0, training=True, scale=None,
                        return_logits=False, causal=False):
    """Plain PyTorch implementation with the same signature (fallback + test oracle).

    q: [B, Lq, H, D], k/v: [B, Lk, H_kv, D] (H_kv dividing H, expanded by ``repeat_interleave``); bias broadcastable
    to [B, H, Lq, Lk];
    key_padding_mask: [B, Lk] bool (True = masked); ``causal`` masks key j > query i. Returns [B, Lq, H, D], or with
    ``return_logits`` ``(out, z)`` with ``z [B, H, Lq, Lk]`` built with additive ``-inf`` masks (its gradient reaches
    masked keys).
    """
    B, Lq, H, D = q.shape
    k, v = _expand_kv(H, k, v)
    scale = scale if scale is not None else 1.0 / math.sqrt(D)
    scores = torch.einsum("bqhd,bkhd->bhqk", q, k) * scale
    if bias is not None:
        scores = scores + bias.to(scores.dtype)
    if key_padding_mask is not None:
        if return_logits:
            pad = torch.zeros(B, 1, 1, k.shape[1], dtype=scores.dtype, device=scores.device)
            scores = scores + pad.masked_fill(key_padding_mask[:, None, None, :].to(torch.bool), float("-inf"))
        else:
            scores = scores.masked_fill(key_padding_mask[:, None, None, :].to(torch.bool), float("-inf"))
    if causal:
        future = torch.ones(Lq, k.shape[1], dtype=torch.bool, device=scores.device).triu(1)
        if return_logits:
            scores = scores + torch.zeros(future.shape, dtype=scores.dtype, device=scores.device).masked_fill(
                future, float("-inf"))
        else:
            scores = scores.masked_fill(future, float("-inf"))
    probs = F.softmax(scores.float(), dim=-1).to(q.dtype)
    probs = F.dropout(probs, p=dropout_p, training=training)
    out = torch.einsum("bhqk,bkhd->bqhd", probs, v)
    return (out, scores) if return_logits else out


def _split_packed(qkv, num_kv_heads):
    """q, k, v views of a packed projection: ``[B, L, 3, H, D]``, or ``[B, L, H + 2 * H_kv, D]`` with
    ``num_kv_heads = H_kv`` (heads ``[0, H)``, ``[H, H + H_kv)`` and ``[H + H_kv, H + 2 * H_kv)``)."""
    if qkv.dim() == 5:
        return qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    if num_kv_heads is None:
        raise ValueError("a [B, L, H + 2 * H_kv, D] projection needs num_kv_heads")
    H = qkv.shape[2] - 2 * num_kv_heads
    if H < 1 or num_kv_heads < 1 or H % num_kv_heads != 0:
        raise ValueError("{} key / value heads do not divide the {} query heads of a packed projection of {} heads"
                         .format(num_kv_heads, H, qkv.shape[2]))
    return qkv[:, :, :H], qkv[:, :, H:H + num_kv_heads], qkv[:, :, H + num_kv_heads:]


class _FusedAttentionFn(torch.autograd.Function):
    """The fused kernels' forward and backward.  ``qkv``: None, or the contiguous packed projection that q, k and v
    are (detached) views of; the backward kernel then writes dq, dk and dv straight into one gradient of its layout,
    which spares autograd three zero-filled slice gradients and their sum."""

    @staticmethod
    def forward(ctx, qkv, q, k, v, bias, key_padding_mask, dropout_p, training, scale, return_logits, causal):
        p = float(dropout_p) if training else 0.0
        logits = None
        if return_logits:
            out, lse, bits, logits = native().fmha_fwd_logits(q, k, v, bias, key_padding_mask, p, float(scale))
            # a logits gradient that autograd never produced stays None (= zero) instead of a zero-filled [B, H, Lq, Lk]
            ctx.set_materialize_grads(False)
        else:
            out, lse, bits = native().fmha_fwd(q, k, v, bias, key_padding_mask, p, float(scale), causal=causal)
        ctx.p = p
        ctx.causal = causal
        ctx.scale = float(scale)
        ctx.need_dbias = bias is not None and bias.requires_grad
        ctx.packed_shape = None if qkv is None else qkv.shape
        ctx.save_for_backward(q, k, v, out, lse, bias, key_padding_mask, bits)
        return (out, logits) if return_logits else out

    @staticmethod
    def backward(ctx, dout, dlogits=None):
        q, k, v, out, lse, bias, kpm, bits = ctx.saved_tensors
        # a missing gradient is zero, and a missing dlogits runs the plain backward
        dout = torch.zeros_like(out) if dout is None else dout.contiguous()
        dlogits = None if dlogits is None else dlogits.contiguous()
        packed = ctx.packed_shape is not None
        dq, dk, dv, dbias = native().fmha_bwd(
            dout, q, k, v, out, lse, bias, kpm, ctx.p, ctx.scale, bits, ctx.need_dbias, packed, dlogits,
            causal=ctx.causal
        )
        if dbias is not None and dbias.dtype != bias.dtype:
            dbias = dbias.to(bias.dtype)
        if packed:   # the [B, L, H + 2 * H_kv, D] tensor the three gradients are views of, in the layout of qkv
            dqkv, dq, dk, dv = dq._base.view(ctx.packed_shape), None, None, None
        else:
            dqkv = None
        return dqkv, dq, dk, dv, dbias, None, None, None, None, None, None


def _kernel_tensors(q, *tensors) -> bool:
    """The kernels' rule for q and the key / value tensors that go with it (None entries are skipped): 4-d, fp16 or
    bf16 and all of the dtype of q, one head dim that ``fused_head_dim_supported`` takes, 16-byte aligned, strides
    that are multiples of 8 elements and a contiguous last dim."""
    if q.dtype not in (torch.float16, torch.bfloat16) or not fused_head_dim_supported(q.shape[-1]):
        return False
    for t in (q,) + tensors:
        if t is None:
            continue
        if t.dim() != 4 or t.dtype != q.dtype or t.shape[-1] != q.shape[-1] or t.stride(-1) != 1:
            return False
        if t.data_ptr() % 16 != 0 or any(s % 8 != 0 for s in t.stride()[:3]):
            return False
    return True


def fused_attention_supported(q, k, v, bias=None, key_padding_mask=None) -> bool:
    if not use_native(q, k, v, bias, key_padding_mask) or not hasattr(native(), "fmha_fwd"):
        return False
    if key_padding_mask is not None and key_padding_mask.dtype != torch.bool:
        return False
    if not _kernel_tensors(q, k, v):
        return False
    # the TMA maps take (head, 16-byte chunk) as one dimension: the heads of each tensor are contiguous
    if any(t.stride(2) != q.shape[-1] for t in (q, k, v)):
        return False
    if k.shape[2] != v.shape[2] or k.shape[2] < 1 or q.shape[2] % k.shape[2] != 0:
        return False
    if q.shape[1] % 8 != 0 or k.shape[1] % 8 != 0:
        return False
    if bias is not None:
        if bias.dim() != 4 or bias.shape[0] not in (1, q.shape[0]) or bias.shape[1] != q.shape[2]:
            return False
        if bias.shape[2] != q.shape[1] or bias.shape[3] != k.shape[1]:
            return False
        if bias.dtype not in (q.dtype, torch.float32):
            return False
        if bias.dtype == q.dtype and bias.is_contiguous() and bias.data_ptr() % 16 != 0:
            return False
    return True


def _fused_attention(q, k, v, bias, key_padding_mask, dropout_p, training, scale, return_logits, causal, qkv=None,
                     supported=None):
    """``fused_attention`` on q / k / v, which are the views of ``qkv`` (``_split_packed``) when it is given: a
    contiguous ``qkv`` then gets one packed gradient.  ``supported``: the answer of ``fused_attention_supported`` for
    these operands when the caller has it already (None: ask)."""
    if scale is None:
        scale = 1.0 / math.sqrt(q.shape[-1])
    if causal and return_logits:   # the kernels do not return the logits of causal attention
        supported = False
    elif supported is None:
        supported = fused_attention_supported(q, k, v, bias, key_padding_mask)
    if not supported:
        return attention_reference(q, k, v, bias, key_padding_mask, dropout_p, training, scale, return_logits, causal)
    if bias is not None:
        # the kernel stages the bias tile next to P in shared memory in the compute dtype
        bias = bias.to(q.dtype).contiguous()
    if key_padding_mask is not None:
        key_padding_mask = key_padding_mask.to(torch.bool).contiguous()
    if qkv is not None and qkv.is_contiguous():
        q, k, v = q.detach(), k.detach(), v.detach()   # autograd sees qkv alone
    else:
        qkv = None
    return _FusedAttentionFn.apply(qkv, q, k, v, bias, key_padding_mask, dropout_p, training, scale, return_logits,
                                   causal)


def fused_attention(q, k, v, bias=None, key_padding_mask=None, dropout_p=0.0, training=True, scale=None,
                    return_logits=False, causal=False):
    """Dispatch to the wgmma kernel when shapes/dtypes allow, else to the PyTorch reference.

    q: ``[B, Lq, H, D]``, k / v: ``[B, Lk, H_kv, D]`` with ``H_kv`` dividing ``H`` (grouped-query attention, see the
    module docstring).  Returns ``[B, Lq, H, D]``, or ``(out, z [B, H, Lq, Lk])`` with ``return_logits``.  ``causal``
    masks key j > query i; with ``return_logits`` it runs the reference."""
    kv_group(q.shape[2], k, v)
    return _fused_attention(q, k, v, bias, key_padding_mask, dropout_p, training, scale, return_logits, causal)


def fused_attention_qkvpacked(qkv, bias=None, key_padding_mask=None, dropout_p=0.0, training=True, scale=None,
                              return_logits=False, causal=False, num_kv_heads=None):
    """Self-attention on the packed in_proj output ``qkv [B, L, 3, H, D]``, or with grouped-query attention
    ``qkv [B, L, H + 2 * H_kv, D]`` (q, k, v the head slices in that order) and ``num_kv_heads = H_kv``.  Returns
    ``[B, L, H, D]``, or ``(out, z [B, H, L, L])`` with ``return_logits``; ``causal`` as in ``fused_attention``."""
    q, k, v = _split_packed(qkv, num_kv_heads)
    return _fused_attention(q, k, v, bias, key_padding_mask, dropout_p, training, scale, return_logits, causal, qkv)


def varlen_positions(cu_seqlens, total, offsets=None):
    """int32 ``[total]``: the position of each packed row inside its sequence (``cu_seqlens [B + 1]``), computed on
    the device, so that no length is read on the host.  ``offsets`` (int ``[B]`` on the device): added to the
    positions of sequence b's rows, as a packed step into a cache places them after the ``seqlens[b]`` cached ones."""
    cu = cu_seqlens.to(torch.long)
    rows = torch.arange(total, device=cu.device)
    seq = torch.searchsorted(cu[1:], rows, right=True).clamp(max=cu.numel() - 1)
    pos = rows - cu[seq]
    if offsets is not None:   # rows past the last sequence take its offset
        pos = pos + offsets.to(device=cu.device, dtype=torch.long)[seq.clamp(max=offsets.numel() - 1)]
    return pos.to(torch.int32)


def _varlen_lengths(cu_seqlens, max_seqlen, total):
    """``(s [B], n [B])``, int64 on the device: each sequence's first packed row and length with the kernels' clamps,
    ``s_b = clamp(cu[b], 0, N)`` and ``n_b = clamp(cu[b + 1] - cu[b], 0, min(L, N - s_b))``."""
    cu = cu_seqlens.to(torch.long)
    start = cu[:-1].clamp(0, total)
    return start, torch.minimum((cu[1:] - cu[:-1]).clamp(min=0), (total - start).clamp(max=max_seqlen))


def _varlen_index(cu_seqlens, max_seqlen, total):
    """``(rows [B, L], valid [B, L])``: the packed row of position ``i`` of sequence ``b`` and whether it exists, with
    the kernels' clamps (``_varlen_lengths``)."""
    start, n = _varlen_lengths(cu_seqlens, max_seqlen, total)
    pos = torch.arange(max_seqlen, device=start.device)
    valid = pos[None, :] < n[:, None]
    rows = torch.where(valid, start[:, None] + pos[None, :], torch.zeros_like(valid, dtype=torch.long))
    return rows, valid


def _varlen_keys(cu_seqlens, max_seqlen, bias, causal, cu_seqlens_k, max_seqlen_k):
    """``(L, Lk)``: the kernels' query and key widths of a varlen call, after the checks its arguments share.  Without
    ``cu_seqlens_k`` the keys are the queries' own rows and ``Lk = L``; with it ``max_seqlen_k`` bounds the key
    lengths, rounded up to a multiple of 8 without a bias as ``max_seqlen`` is."""
    L = _varlen_max_seqlen(max_seqlen, bias)
    if cu_seqlens_k is None:
        if max_seqlen_k is not None:
            raise ValueError("max_seqlen_k goes with cu_seqlens_k")
        return L, L
    if causal:
        raise ValueError("causal attention is not defined with separate key sequences (cu_seqlens_k)")
    if max_seqlen_k is None:
        raise ValueError("cu_seqlens_k needs max_seqlen_k, a host bound on the key lengths")
    if cu_seqlens_k.dim() != 1 or cu_seqlens_k.numel() != cu_seqlens.numel():
        raise ValueError("cu_seqlens_k must describe the B = {} sequences of cu_seqlens, not {}".format(
            cu_seqlens.numel() - 1, tuple(cu_seqlens_k.shape)))
    return L, _varlen_max_seqlen(max_seqlen_k, bias)


def attention_varlen_reference(q, k, v, cu_seqlens, max_seqlen, bias=None, dropout_p=0.0, training=True, scale=None,
                               causal=False, cu_seqlens_k=None, max_seqlen_k=None):
    """Plain PyTorch implementation of ``fused_attention_varlen`` (CPU path, fallback and test oracle): the packed
    rows are scattered to ``[B, max_seqlen]`` (k / v to ``[B, max_seqlen_k]`` by ``cu_seqlens_k`` when given),
    ``attention_reference`` runs with the length mask (key ``j`` of sequence ``b`` hidden when ``j >= n_k``), and the
    real rows are gathered back.  Packed rows that belong to no sequence give 0, and so do the rows of a sequence
    without keys, with zero gradients.  Differentiable in q, k, v and the bias.  Without a bias ``max_seqlen`` (and
    ``max_seqlen_k``) is rounded up to a multiple of 8, as on the kernel path, so that both clamp a length to the same
    bound."""
    N, H, D = q.shape
    L, Lk = _varlen_keys(cu_seqlens, max_seqlen, bias, causal, cu_seqlens_k, max_seqlen_k)
    rows, valid = _varlen_index(cu_seqlens.to(q.device), L, N)
    if cu_seqlens_k is None:
        rows_k, valid_k = rows, valid
    else:
        rows_k, valid_k = _varlen_index(cu_seqlens_k.to(q.device), Lk, k.shape[0])
    B = rows.shape[0]

    def scatter(x, rows, valid):
        return torch.where(valid[:, :, None, None], x[rows], torch.zeros((), dtype=x.dtype, device=x.device))

    # the length mask as an additive bias.  The rows past n_q, and the rows of a sequence without keys, see every
    # (padded) key, so that they stay finite: the former are dropped, the latter multiplied by 0
    n_k = valid_k.sum(1)
    has_keys = n_k > 0
    hide = (torch.arange(Lk, device=q.device)[None, None, :] >= n_k[:, None, None]) \
        & (valid & has_keys[:, None])[:, :, None]
    mask = torch.zeros(B, 1, L, Lk, dtype=q.dtype, device=q.device).masked_fill(hide[:, None], float("-inf"))
    bias = mask if bias is None else bias.to(q.dtype) + mask
    out = attention_reference(scatter(q, rows, valid), scatter(k, rows_k, valid_k), scatter(v, rows_k, valid_k), bias,
                              None, dropout_p, training, scale, causal=causal)
    out = out * has_keys[:, None, None, None].to(out.dtype)
    # gather back: the rows of no sequence (and the positions past n_q) write into a dropped row N
    dest = torch.where(valid, rows, torch.full_like(rows, N)).reshape(-1)
    packed = torch.zeros(N + 1, H, D, dtype=out.dtype, device=out.device).index_put((dest,), out.reshape(-1, H, D))
    return packed[:N]


class _FusedVarlenAttentionFn(torch.autograd.Function):
    """The varlen kernels' forward and backward (``_C.varlen``), shaped as ``_FusedAttentionFn``: ``qkv`` None or
    the contiguous ``[N, H + 2 * H_kv, D]`` projection that q, k and v are (detached) views of, which then gets one
    packed gradient.  ``cu_seqlens_k`` None (self-attention, ``max_seqlen_k`` 0) or the key sequences'
    description."""

    @staticmethod
    def forward(ctx, qkv, q, k, v, cu_seqlens, max_seqlen, bias, dropout_p, training, scale, causal, cu_seqlens_k,
                max_seqlen_k):
        p = float(dropout_p) if training else 0.0
        out, lse, bits = native().varlen.fmha_varlen_fwd(q, k, v, cu_seqlens, max_seqlen, bias, p, float(scale),
                                                         causal=causal, cu_seqlens_k=cu_seqlens_k,
                                                         max_seqlen_k=max_seqlen_k)
        ctx.p = p
        ctx.causal = causal
        ctx.scale = float(scale)
        ctx.max_seqlen = max_seqlen
        ctx.max_seqlen_k = max_seqlen_k
        ctx.need_dbias = bias is not None and bias.requires_grad
        ctx.packed_shape = None if qkv is None else qkv.shape
        ctx.save_for_backward(q, k, v, out, lse, cu_seqlens, bias, bits, cu_seqlens_k)
        return out

    @staticmethod
    def backward(ctx, dout):
        q, k, v, out, lse, cu_seqlens, bias, bits, cu_seqlens_k = ctx.saved_tensors
        packed = ctx.packed_shape is not None
        dq, dk, dv, dbias = native().varlen.fmha_varlen_bwd(
            dout.contiguous(), q, k, v, out, lse, cu_seqlens, ctx.max_seqlen, bias, ctx.p, ctx.scale, bits,
            ctx.need_dbias, packed, causal=ctx.causal, cu_seqlens_k=cu_seqlens_k, max_seqlen_k=ctx.max_seqlen_k
        )
        if dbias is not None and dbias.dtype != bias.dtype:
            dbias = dbias.to(bias.dtype)
        if packed:   # the [N, H + 2 * H_kv, D] tensor the three gradients are views of
            dqkv, dq, dk, dv = dq._base.view(ctx.packed_shape), None, None, None
        else:
            dqkv = None
        return dqkv, dq, dk, dv, None, None, dbias, None, None, None, None, None, None


def _varlen_max_seqlen(max_seqlen, bias):
    """The kernels' ``max_seqlen``: a multiple of 8.  Without a bias it is rounded up (the padded side layout is
    internal and the lengths stay below it); with one it must be the bias's own size."""
    L = int(max_seqlen)
    return L if bias is not None else L + (-L % 8)


def fused_attention_varlen_supported(q, k, v, cu_seqlens, max_seqlen, bias=None, cu_seqlens_k=None,
                                     max_seqlen_k=None) -> bool:
    if not use_native(q, k, v, cu_seqlens, bias, cu_seqlens_k) or not hasattr(native(), "varlen"):
        return False
    if q.dim() != 3 or k.dim() != 3 or v.dim() != 3 or q.shape[0] < 1 or cu_seqlens.dim() != 1 \
            or cu_seqlens.numel() < 2:
        return False
    if cu_seqlens_k is None:
        if k.shape[0] != q.shape[0] or v.shape[0] != q.shape[0] or max_seqlen_k is not None:
            return False
    elif k.shape[0] < 1 or v.shape[0] != k.shape[0] or cu_seqlens_k.dim() != 1 \
            or cu_seqlens_k.numel() != cu_seqlens.numel() or max_seqlen_k is None:
        return False
    if not _kernel_tensors(q.unsqueeze(0), k.unsqueeze(0), v.unsqueeze(0)):
        return False
    if any(t.stride(1) != q.shape[-1] for t in (q, k, v)):
        return False
    if k.shape[1] != v.shape[1] or k.shape[1] < 1 or q.shape[1] % k.shape[1] != 0:
        return False
    L = _varlen_max_seqlen(max_seqlen, bias)
    Lk = L if cu_seqlens_k is None else _varlen_max_seqlen(max_seqlen_k, bias)
    if L < 1 or L % 8 != 0 or Lk < 1 or Lk % 8 != 0:
        return False
    if bias is not None:
        if bias.dim() != 4 or bias.shape[0] not in (1, cu_seqlens.numel() - 1) or bias.shape[1] != q.shape[1]:
            return False
        if bias.shape[2] != L or bias.shape[3] != Lk or bias.dtype not in (q.dtype, torch.float32):
            return False
    return True


def _fused_attention_varlen(q, k, v, cu_seqlens, max_seqlen, bias, dropout_p, training, scale, causal, qkv=None,
                            cu_seqlens_k=None, max_seqlen_k=None):
    """``fused_attention_varlen`` on q / k / v, which are the views of ``qkv`` when it is given: a contiguous ``qkv``
    then gets one packed gradient."""
    if scale is None:
        scale = 1.0 / math.sqrt(q.shape[-1])
    L, Lk = _varlen_keys(cu_seqlens, max_seqlen, bias, causal, cu_seqlens_k, max_seqlen_k)
    if not fused_attention_varlen_supported(q, k, v, cu_seqlens, max_seqlen, bias, cu_seqlens_k, max_seqlen_k):
        return attention_varlen_reference(q, k, v, cu_seqlens, max_seqlen, bias, dropout_p, training, scale, causal,
                                          cu_seqlens_k, max_seqlen_k)
    cu_seqlens = cu_seqlens.to(torch.int32).contiguous()
    if cu_seqlens_k is not None:
        cu_seqlens_k = cu_seqlens_k.to(torch.int32).contiguous()
    if bias is not None:
        bias = bias.to(q.dtype).contiguous()
    if qkv is not None and qkv.is_contiguous():
        q, k, v = q.detach(), k.detach(), v.detach()   # autograd sees qkv alone
    else:
        qkv = None
    return _FusedVarlenAttentionFn.apply(qkv, q, k, v, cu_seqlens, L, bias, dropout_p, training, scale, causal,
                                         cu_seqlens_k, 0 if cu_seqlens_k is None else Lk)


def fused_attention_varlen(q, k, v, cu_seqlens, max_seqlen, bias=None, dropout_p=0.0, training=True, scale=None,
                           causal=False, cu_seqlens_k=None, max_seqlen_k=None):
    """Attention over packed variable-length sequences (no padding): q ``[N, H, D]``, k / v ``[N, H_kv, D]`` with
    ``H_kv`` dividing ``H``, the B sequences back to back; sequence ``b`` holds rows ``cu_seqlens[b] ..
    cu_seqlens[b + 1] - 1`` (int ``[B + 1]`` on the device, never read on the host).  ``max_seqlen``: a host bound
    on the lengths; without a bias it is rounded up to a multiple of 8.  ``bias``: ``[1|B, H, max_seqlen,
    max_seqlen]``, sequence b reading its top-left block; the kernels take it when ``max_seqlen`` is a multiple of 8
    (the rule of the padded call), other widths run ``attention_varlen_reference``.
    ``causal`` masks key j > query i within each sequence.  Returns ``[N, H, D]``: at every real row the result of
    the padded call with ``key_padding_mask = (j >= len_b)``.  Lengths are clamped to ``[0, max_seqlen]`` and the
    starts to ``[0, N]``.

    Cross-attention: ``cu_seqlens_k`` (int ``[B + 1]`` on the device, the same B) and ``max_seqlen_k`` describe
    separate key sequences, k / v ``[N_k, H_kv, D]`` (flash-attention's ``cu_seqlens_q`` / ``cu_seqlens_k``); the bias
    is then ``[1|B, H, max_seqlen, max_seqlen_k]`` and ``max_seqlen_k`` is rounded up like ``max_seqlen``.  Query i of
    sequence b sees its keys j < n_k; a sequence without keys gives 0 at its rows, with zero gradients.  Not with
    ``causal`` (``ValueError``)."""
    kv_group(q.shape[1], k.unsqueeze(0), v.unsqueeze(0))
    return _fused_attention_varlen(q, k, v, cu_seqlens, max_seqlen, bias, dropout_p, training, scale, causal,
                                   cu_seqlens_k=cu_seqlens_k, max_seqlen_k=max_seqlen_k)


def fused_attention_varlen_qkvpacked(qkv, cu_seqlens, max_seqlen, bias=None, dropout_p=0.0, training=True,
                                     scale=None, causal=False, num_kv_heads=None):
    """``fused_attention_varlen`` on the packed projection ``qkv [N, 3, H, D]``, or ``[N, H + 2 * H_kv, D]`` with
    ``num_kv_heads = H_kv``; a contiguous ``qkv`` gets one gradient tensor."""
    q, k, v = (t[:, 0] for t in _split_packed(qkv[:, None], num_kv_heads))
    return _fused_attention_varlen(q, k, v, cu_seqlens, max_seqlen, bias, dropout_p, training, scale, causal, qkv)


def _check_no_grad(*tensors):
    if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in tensors):
        raise RuntimeError("attention_with_kv_cache has no backward: call it under torch.no_grad() or "
                           "torch.inference_mode(), or detach the inputs")


PAGED_BLOCK_MULTIPLE = 128


def _check_block_table(block_table, k_cache, v_cache, B):
    """A paged cache's arguments checked: ``block_table`` an integer ``[B, M >= 1]`` and ``k_cache`` / ``v_cache``
    pools ``[num_blocks, block_size, H_kv, D]`` of one shape, ``block_size`` a multiple of 128."""
    if block_table.dim() != 2 or block_table.shape[0] != B or block_table.shape[1] < 1:
        raise ValueError("block_table must be [B = {}, M >= 1], not {}".format(B, tuple(block_table.shape)))
    if block_table.dtype not in (torch.int32, torch.int64):
        raise ValueError("block_table must be int32 or int64, not {}".format(block_table.dtype))
    if k_cache.dim() != 4 or k_cache.shape[:2] != v_cache.shape[:2] or k_cache.shape[0] < 1:
        raise ValueError("paged caches must be pools [num_blocks, block_size, H_kv, D] of one shape, not {} and {}"
                         .format(tuple(k_cache.shape), tuple(v_cache.shape)))
    if k_cache.shape[1] % PAGED_BLOCK_MULTIPLE != 0:
        raise ValueError("the block size of paged caches must be a multiple of {}, not {}".format(
            PAGED_BLOCK_MULTIPLE, k_cache.shape[1]))


def cache_capacity(k_cache, block_table=None):
    """Rows per sequence of a key / value cache: ``C`` of ``[B, C, H_kv, D]``, or ``M * block_size`` of a pool
    ``[num_blocks, block_size, H_kv, D]`` named by ``block_table [B, M]``."""
    return k_cache.shape[1] if block_table is None else block_table.shape[1] * k_cache.shape[1]


def _paged_gather(cache, block_table):
    """``[B, C, ...]``: the rows of every sequence gathered through the table from the pool (entries outside the pool
    clamped into it, as the kernels clamp their reads)."""
    idx = block_table.long().to(cache.device).clamp(0, cache.shape[0] - 1)
    return cache[idx].reshape(idx.shape[0], idx.shape[1] * cache.shape[1], *cache.shape[2:])


def _cache_store(cache, block_table, rows, write, values):
    """``cache`` row ``rows[b, i]`` of sequence b becomes ``values[b, i]`` where ``write [B, T]``: batch b of a
    contiguous cache, or through ``block_table`` into the pool, skipping the rows whose entry is outside it."""
    B = rows.shape[0]
    seq = torch.arange(B, device=cache.device)[:, None].expand_as(rows)
    rows = rows.clamp(0, cache_capacity(cache, block_table) - 1)
    if block_table is None:
        dst_b, dst_r = seq, rows
    else:
        bs = cache.shape[1]
        dst_b = block_table.long().to(cache.device)[seq, rows // bs]
        dst_r = rows % bs
        write = write & (dst_b >= 0) & (dst_b < cache.shape[0])
    cache[dst_b[write], dst_r[write]] = values[write].to(cache.dtype)


def _kv_cache_plan(q, k_cache, v_cache, seqlens, max_len, k_new, v_new, T=None, block_table=None, B=None):
    """The arguments of ``attention_with_kv_cache`` checked, as ``(T, append, max_len, bound)``: ``max_len`` the host
    bound on ``seqlens`` (by default the most the capacity allows; None without ``seqlens`` unless given) and
    ``bound`` the keys any query can see, ``max_len`` plus the appended rows, else the capacity C.  ``T``: the new
    queries per sequence (default ``q.shape[1]``; the host bound ``max_seqlen`` of packed chunks, whose q / k_new /
    v_new are ``[N, heads, D]``).  ``block_table``: the caches are pools (``_check_block_table``) of ``B`` sequences
    (default ``q.shape[0]``) and C is ``M * block_size``."""
    kv_group(q.shape[-2], k_cache, v_cache)
    if block_table is not None:
        _check_block_table(block_table, k_cache, v_cache, q.shape[0] if B is None else B)
    append = k_new is not None
    if append != (v_new is not None):
        raise ValueError("k_new and v_new go together")
    if append and seqlens is None:
        raise ValueError("appending needs seqlens (the row to write)")
    if append and (k_new.shape[-2] != k_cache.shape[2] or v_new.shape[-2] != k_cache.shape[2]):
        raise ValueError("k_new / v_new must have the {} heads of the caches".format(k_cache.shape[2]))
    T = q.shape[1] if T is None else int(T)
    if T > 1 and seqlens is not None and not append:
        raise ValueError("a chunk of T > 1 queries with seqlens appends k_new / v_new")
    C = cache_capacity(k_cache, block_table)
    new_rows = T if append else 0
    if seqlens is not None and max_len is None:
        max_len = C - new_rows
    if max_len is not None and int(max_len) + new_rows > C:
        raise ValueError("max_len {} {}exceeds the cache capacity {}".format(
            max_len, "+ {} ".format(new_rows) if append else "", C))
    return T, append, max_len, C if seqlens is None else int(max_len) + new_rows


def attention_with_kv_cache_reference(q, k_cache, v_cache, seqlens=None, max_len=None, k_new=None, v_new=None,
                                      bias=None, key_padding_mask=None, scale=None, block_table=None):
    """Plain PyTorch implementation of ``attention_with_kv_cache`` (CPU path, fallback and test oracle).

    Performs the append in place like the kernels.  One query (T = 1): row ``seqlens[b]`` (clamped to ``C - 1``) of the
    caches becomes ``k_new[b] / v_new[b]``.  A chunk (T > 1): rows ``p_b + i``, ``p_b = seqlens[b]`` clamped to
    ``[0, C]``, become ``k_new[b, i] / v_new[b, i]``, rows at or past ``C`` are skipped, and query ``i`` sees key ``j``
    only when ``j <= p_b + i``.  Keys past the visible length are masked; a row with no visible unmasked key gives 0.
    ``block_table``: the caches are pools; the call runs on the caches gathered through the table, and the appended
    rows are written back through it (rows whose entry is outside the pool are skipped).
    """
    if block_table is not None:
        T, append, _, _ = _kv_cache_plan(q, k_cache, v_cache, seqlens, max_len, k_new, v_new, block_table=block_table)
        kc, vc = _paged_gather(k_cache, block_table), _paged_gather(v_cache, block_table)
        out = attention_with_kv_cache_reference(q, kc, vc, seqlens, max_len, k_new, v_new, bias, key_padding_mask,
                                                scale)
        if append:
            C = kc.shape[1]
            if T == 1:
                start = seqlens.long().to(kc.device).clamp(0, C - 1)
            else:
                start = seqlens.long().to(kc.device).clamp(0, C)
            rows = start[:, None] + torch.arange(T, device=kc.device)[None, :]
            _write_back(k_cache, v_cache, kc, vc, block_table, rows, rows < C)
        return out
    T, append, _, K = _kv_cache_plan(q, k_cache, v_cache, seqlens, max_len, k_new, v_new)
    B, _, H, D = q.shape
    C = k_cache.shape[1]
    scale = scale if scale is not None else 1.0 / math.sqrt(D)
    future = None
    if T == 1 and append:
        pos = seqlens.long().clamp(0, C - 1)
        rows = torch.arange(B, device=k_cache.device)
        k_cache[rows, pos] = k_new[:, 0].to(k_cache.dtype)
        v_cache[rows, pos] = v_new[:, 0].to(v_cache.dtype)
        n = pos + 1
    elif append:
        p = seqlens.long().to(k_cache.device).clamp(0, C)
        pos = p[:, None] + torch.arange(T, device=k_cache.device)[None, :]   # [B, T]
        rows = torch.arange(B, device=k_cache.device)
        for i in range(T):   # one row per sequence at a time; a row at or past C keeps row C - 1 as it is
            at, keep = pos[:, i].clamp(max=C - 1), (pos[:, i] >= C)[:, None, None]
            k_cache[rows, at] = torch.where(keep, k_cache[rows, at], k_new[:, i].to(k_cache.dtype))
            v_cache[rows, at] = torch.where(keep, v_cache[rows, at], v_new[:, i].to(v_cache.dtype))
        n = (p + T).clamp(max=C)
        future = pos.to(q.device)   # query i of batch b sees keys j <= p_b + i
    elif seqlens is not None:
        n = seqlens.long().clamp(0, C)
    else:
        n = torch.full((B,), C, dtype=torch.long, device=q.device)
    return _kv_cache_attend_reference(q, k_cache, v_cache, n, future, K, bias, key_padding_mask, scale)


def _write_back(k_cache, v_cache, kc, vc, block_table, rows, write):
    """The rows ``rows [B, T]`` (where ``write``) of the gathered caches ``kc`` / ``vc`` stored back into the pools."""
    at = rows.clamp(0, kc.shape[1] - 1)
    seq = torch.arange(rows.shape[0], device=kc.device)[:, None]
    _cache_store(k_cache, block_table, rows, write, kc[seq, at])
    _cache_store(v_cache, block_table, rows, write, vc[seq, at])


def _kv_cache_attend_reference(q, k_cache, v_cache, n, future, K, bias, key_padding_mask, scale):
    """The attention of the cache references after their appends: q ``[B, T, H, D]`` against cache rows ``j < n_b``
    (``n [B]``) and ``j < K`` (the keys any query can see), and ``j <= future[b, i]`` when ``future [B, T]`` is given;
    the keys past the columns of the bias or of the key mask are hidden too."""
    H = q.shape[2]
    if bias is not None:
        K = min(K, bias.shape[-1])
    if key_padding_mask is not None:
        K = min(K, key_padding_mask.shape[-1])
    k, v = _expand_kv(H, k_cache[:, :K], v_cache[:, :K])
    scores = torch.einsum("bqhd,bkhd->bhqk", q, k) * scale   # [B, H, T, K]
    if bias is not None:
        scores = scores + bias[..., :K].to(scores.dtype)
    keys = torch.arange(K, device=q.device)
    hidden = keys[None, :] >= n.to(q.device)[:, None]   # [B, K]
    # rows past the visible length are never read by the kernel: whatever they hold (NaN included) must not matter
    v = v.masked_fill(hidden[:, :, None, None], 0)
    if key_padding_mask is not None:
        hidden = hidden | key_padding_mask[:, :K].to(torch.bool)
    hidden = hidden[:, None, None, :]   # [B, 1, 1, K]
    if future is not None:
        hidden = hidden | (keys[None, None, :] > future[:, :, None])[:, None]   # [B, 1, T, K]
    scores = scores.masked_fill(hidden, float("-inf"))
    probs = torch.nan_to_num(F.softmax(scores.float(), dim=-1), nan=0.0).to(q.dtype)   # all masked -> 0
    return torch.einsum("bhqk,bkhd->bqhd", probs, v)


def _decode_supported(q, k_cache, v_cache, seqlens, k_new, v_new, bias, key_padding_mask, block_table=None) -> bool:
    """True when ``fmha_decode`` (T = 1) or ``kvcache.fmha_kvcache_fwd`` (T > 1) takes the operands."""
    if not use_native(q, k_cache, v_cache, seqlens, k_new, v_new, bias, key_padding_mask, block_table) \
            or not hasattr(native(), "fmha_decode"):
        return False
    if q.dim() != 4 or q.shape[1] < 1 or (q.shape[1] > 1 and not hasattr(native(), "kvcache")):
        return False
    if not _kernel_tensors(q, k_cache, v_cache, k_new, v_new):
        return False
    if bias is not None and bias.stride(-1) != 1 and bias.shape[-1] > 1:
        return False
    return True


def _native_cache_operands(q, seqlens, bias, key_padding_mask, bound, B, T, chunk):
    """``seqlens``, the bias and the key mask as ``fmha_decode`` (one query per sequence) and the chunk kernel
    (``chunk``: ``fmha_kvcache_fwd`` or ``fmha_kvcache_varlen_fwd``, up to T queries) take them for B sequences:
    int32 lengths, a bool key mask and a bias in the dtype of q, each with a contiguous last dim.  A bias or key mask
    narrower than the ``bound`` visible keys is widened with -inf / True, which hides the keys past it as the
    reference's clamp to its columns does.  Operands that are already so are passed on as they are."""
    if seqlens is not None and (seqlens.dtype != torch.int32 or not seqlens.is_contiguous()):
        seqlens = seqlens.to(torch.int32).contiguous()
    if bias is not None:
        Lb = bias.shape[-1]
        width = max(Lb, bound)
        bias = bias.to(q.dtype)
        if chunk:   # read by TMA: a row for every query head, of a multiple of 8 columns
            bias = bias.expand(bias.shape[0], q.shape[-2], T, Lb)
            width += -width % 8
        if width != Lb:
            bias = F.pad(bias, (0, width - Lb), value=float("-inf"))
        if chunk or bias.stride(-1) != 1:
            bias = bias.contiguous()
    if key_padding_mask is not None:
        if key_padding_mask.dtype != torch.bool or key_padding_mask.stride(-1) != 1:
            key_padding_mask = key_padding_mask.to(torch.bool).contiguous()
        cols = key_padding_mask.shape[1]
        if cols < bound:
            key_padding_mask = torch.cat([key_padding_mask, key_padding_mask.new_ones(B, bound - cols)], 1)
        if chunk:
            key_padding_mask = key_padding_mask.contiguous()
    return seqlens, bias, key_padding_mask


def attention_with_kv_cache(q, k_cache, v_cache, seqlens=None, max_len=None, k_new=None, v_new=None, bias=None,
                            key_padding_mask=None, scale=None, block_table=None):
    """Attention of T new queries per sequence against a key / value cache: one decoding step (T = 1) or a chunk.

    q: ``[B, T, H, D]``; k_cache / v_cache: ``[B, C, H_kv, D]`` with ``H_kv`` dividing ``H`` (strided views are fine,
    the last dim contiguous).  ``k_new`` / ``v_new`` ``[B, T, H_kv, D]`` (needs ``seqlens``): the new tokens' keys and values, written bitwise into
    rows ``seqlens[b] .. seqlens[b] + T - 1`` of the caches before the attention.  Query ``i`` of batch b then sees
    rows ``0 .. seqlens[b] + i`` (the future mask of the whole sequence); with ``seqlens=None`` every query sees all C
    rows (cross-attention).  At T = 1, ``seqlens`` without ``k_new`` shows rows ``0 .. seqlens[b] - 1``; a chunk with
    ``seqlens`` must append.  ``max_len``: a host-side upper bound on ``seqlens`` (default: the most the capacity
    allows); ``max_len + T > C`` raises, and the device lengths are never read on the host, so a step does not
    synchronise.  bias: ``[1|B, H, T, Lb]``, row i for query i, ``Lb`` covering the visible keys (columns past them
    are ignored); key_padding_mask: bool ``[B, Lk]``, True = masked; a narrower bias or key mask hides the keys past
    its columns.  A query whose visible keys are all masked gives 0.  Returns ``[B, T, H, D]``.  No dropout and no
    backward.  Under CUDA-graph capture (``max_len`` then a fixed bound such as the capacity) a one-token step divides
    each sequence's device length over the split-KV splits.  ``block_table`` (int ``[B, M]`` on the device): the
    caches are pools ``[num_blocks, block_size, H_kv, D]`` and ``C = M * block_size`` (see the module docstring)."""
    _check_no_grad(q, k_cache, v_cache, k_new, v_new, bias)
    T, _, max_len, bound = _kv_cache_plan(q, k_cache, v_cache, seqlens, max_len, k_new, v_new,
                                          block_table=block_table)
    if scale is None:
        scale = 1.0 / math.sqrt(q.shape[-1])
    if not _decode_supported(q, k_cache, v_cache, seqlens, k_new, v_new, bias, key_padding_mask, block_table):
        return attention_with_kv_cache_reference(q, k_cache, v_cache, seqlens, max_len, k_new, v_new, bias,
                                                 key_padding_mask, scale, block_table)
    seqlens, bias, key_padding_mask = _native_cache_operands(q, seqlens, bias, key_padding_mask, bound, q.shape[0], T,
                                                             T > 1)
    block_table = _native_table(block_table)
    max_len = 0 if max_len is None else int(max_len)
    if T == 1:
        # A step captured in a CUDA graph runs with the capacity as its host bound, far above most true lengths: each
        # (b, h) then spreads its own device length over the splits, not the bound (or most splits would be empty).
        return native().fmha_decode(q, k_cache, v_cache, seqlens, max_len, k_new, v_new, bias, key_padding_mask,
                                    float(scale), split_by_length=torch.cuda.is_current_stream_capturing(),
                                    block_table=block_table)
    return native().kvcache.fmha_kvcache_fwd(q, k_cache, v_cache, seqlens, max_len, k_new, v_new, bias,
                                             key_padding_mask, float(scale), block_table=block_table)


def _native_table(block_table):
    """The block table as the kernels take it: int32 and contiguous (passed on as it is when it already is)."""
    if block_table is not None and (block_table.dtype != torch.int32 or not block_table.is_contiguous()):
        block_table = block_table.to(torch.int32).contiguous()
    return block_table


def _kv_cache_varlen_plan(q, k_cache, v_cache, cu_seqlens, max_seqlen, seqlens, max_len, k_new, v_new,
                          block_table=None):
    """``attention_with_kv_cache_varlen``'s arguments checked, as ``_kv_cache_plan``'s result for chunks of up to
    ``max_seqlen`` queries."""
    if q.dim() != 3 or (k_new is not None and k_new.dim() != 3) or (v_new is not None and v_new.dim() != 3):
        raise ValueError("packed chunks take q [N, H, D] and k_new / v_new [N, H_kv, D]")
    B = k_cache.shape[0] if block_table is None else block_table.shape[0]
    if cu_seqlens.dim() != 1 or cu_seqlens.numel() != B + 1:
        raise ValueError("cu_seqlens must have B + 1 = {} entries for the caches' B = {} sequences, not {}".format(
            B + 1, B, tuple(cu_seqlens.shape)))
    if int(max_seqlen) < 1:
        raise ValueError("max_seqlen must be positive, not {}".format(max_seqlen))
    if seqlens is not None and k_new is None:
        raise ValueError("packed chunks with seqlens append k_new / v_new")
    return _kv_cache_plan(q, k_cache, v_cache, seqlens, max_len, k_new, v_new, T=max_seqlen, block_table=block_table,
                          B=B)


def attention_with_kv_cache_varlen_reference(q, k_cache, v_cache, cu_seqlens, max_seqlen, seqlens=None, max_len=None,
                                             k_new=None, v_new=None, bias=None, key_padding_mask=None, scale=None,
                                             block_table=None):
    """Plain PyTorch implementation of ``attention_with_kv_cache_varlen`` (CPU path, fallback and test oracle).

    Performs the append in place like the kernels, ``T_b`` rows per sequence: rows ``p_b + i`` of the caches,
    ``p_b = seqlens[b]`` clamped to ``[0, C]``, become packed rows ``s_b + i`` of ``k_new / v_new``, and rows at or past
    ``C`` are skipped.  At every real row the result is what ``attention_with_kv_cache_reference`` gives for that
    sequence alone with ``T = T_b``; packed rows of no sequence give 0.  ``block_table``: pools, as in
    ``attention_with_kv_cache_reference``."""
    if block_table is not None:
        T, _, _, _ = _kv_cache_varlen_plan(q, k_cache, v_cache, cu_seqlens, max_seqlen, seqlens, max_len, k_new, v_new,
                                           block_table)
        kc, vc = _paged_gather(k_cache, block_table), _paged_gather(v_cache, block_table)
        out = attention_with_kv_cache_varlen_reference(q, kc, vc, cu_seqlens, max_seqlen, seqlens, max_len, k_new,
                                                       v_new, bias, key_padding_mask, scale)
        if seqlens is not None:
            C = kc.shape[1]
            _, n = _varlen_lengths(cu_seqlens.to(kc.device), T, q.shape[0])
            i = torch.arange(T, device=kc.device)[None, :]
            rows = seqlens.long().to(kc.device).clamp(0, C)[:, None] + i
            _write_back(k_cache, v_cache, kc, vc, block_table, rows, (i < n[:, None]) & (rows < C))
        return out
    T, _, _, K = _kv_cache_varlen_plan(q, k_cache, v_cache, cu_seqlens, max_seqlen, seqlens, max_len, k_new, v_new)
    N, H, D = q.shape
    B, C = k_cache.shape[:2]
    scale = scale if scale is not None else 1.0 / math.sqrt(D)
    rows, valid = _varlen_index(cu_seqlens.to(q.device), T, N)   # [B, T]: packed row of query i of sequence b
    future = None
    if seqlens is not None:
        dev = k_cache.device
        p = seqlens.long().to(dev).clamp(0, C)
        pos = p[:, None] + torch.arange(T, device=dev)[None, :]   # [B, T]
        write = valid.to(dev) & (pos < C)
        src, seq = rows.to(dev), torch.arange(B, device=dev)
        for i in range(T):   # one row per sequence at a time; a row not written keeps what it holds
            at, keep = pos[:, i].clamp(max=C - 1), ~write[:, i, None, None]
            k_cache[seq, at] = torch.where(keep, k_cache[seq, at], k_new[src[:, i]].to(k_cache.dtype))
            v_cache[seq, at] = torch.where(keep, v_cache[seq, at], v_new[src[:, i]].to(v_cache.dtype))
        n = (p + valid.sum(1).to(dev)).clamp(max=C)
        future = pos.to(q.device)   # query i of sequence b sees keys j <= p_b + i
    else:
        n = torch.full((B,), C, dtype=torch.long, device=q.device)
    qp = torch.where(valid[:, :, None, None], q[rows], torch.zeros((), dtype=q.dtype, device=q.device))
    out = _kv_cache_attend_reference(qp, k_cache, v_cache, n, future, K, bias, key_padding_mask, scale)
    # gather back: the positions past T_b write into a dropped row N
    dest = torch.where(valid, rows, torch.full_like(rows, N)).reshape(-1)
    packed = torch.zeros(N + 1, H, D, dtype=out.dtype, device=out.device).index_put((dest,), out.reshape(-1, H, D))
    return packed[:N]


def _kvcache_varlen_supported(q, k_cache, v_cache, cu_seqlens, seqlens, k_new, v_new, bias, key_padding_mask,
                              block_table=None) -> bool:
    """True when ``kvcache.fmha_kvcache_varlen_fwd`` takes the operands."""
    if not use_native(q, k_cache, v_cache, cu_seqlens, seqlens, k_new, v_new, bias, key_padding_mask, block_table) \
            or not hasattr(getattr(native(), "kvcache", None), "fmha_kvcache_varlen_fwd"):
        return False
    if q.shape[0] < 1 or q.stride(1) != q.shape[-1]:   # the q map takes (head, 16-byte chunk) as one dimension
        return False
    if not _kernel_tensors(q[None], k_cache, v_cache, None if k_new is None else k_new[None],
                           None if v_new is None else v_new[None]):
        return False
    if bias is not None and bias.stride(-1) != 1 and bias.shape[-1] > 1:
        return False
    return True


def attention_with_kv_cache_varlen(q, k_cache, v_cache, cu_seqlens, max_seqlen, seqlens=None, max_len=None,
                                   k_new=None, v_new=None, bias=None, key_padding_mask=None, scale=None,
                                   block_table=None):
    """``attention_with_kv_cache`` for packed chunks: each sequence brings its own number of new queries.

    q: ``[N, H, D]``, the B sequences' new queries back to back; sequence b's ``T_b`` queries are rows ``s_b .. s_b +
    T_b - 1`` with ``s_b = clamp(cu_seqlens[b], 0, N)`` and ``T_b = clamp(cu_seqlens[b + 1] - cu_seqlens[b], 0,
    min(max_seqlen, N - s_b))`` (``cu_seqlens`` int ``[B + 1]`` on the device; ``max_seqlen`` a host bound on ``T_b``,
    any value >= 1).  ``T_b = 0`` is allowed: that sequence adds nothing.  k_cache / v_cache: ``[B, C, H_kv, D]``.
    ``k_new`` / ``v_new`` ``[N, H_kv, D]`` (needed with ``seqlens``): rows ``s_b + i`` are written bitwise into cache
    rows ``p_b + i``, ``p_b = clamp(seqlens[b], 0, C)``, before the attention; rows at or past ``C`` are skipped.  Query
    ``i`` of sequence b then sees cache rows ``0 .. p_b + i``.  With ``seqlens=None`` every query sees all C rows
    (cross-attention against stored encoder keys).  ``max_len``: a host bound on ``seqlens`` (default: the most the
    capacity allows); ``max_len + max_seqlen > C`` raises.  bias: ``[1|B, H, max_seqlen, Lb]``, row i for query i of
    every sequence; key_padding_mask: bool ``[B, Lk]``; a narrower bias or key mask hides the keys past its columns.  A
    query with no visible unmasked key gives 0.  Returns ``[N, H, D]``; at every real row the result of
    ``attention_with_kv_cache`` on that sequence alone with ``T = T_b``.  Rows of q that belong to no sequence are not
    written by the kernel (0 on the reference path), as in ``fused_attention_varlen``.  No dropout and no backward, and
    no device value is read on the host, so a step does not synchronise.

    It runs in the KV-cache mode of the wgmma forward for every ``T_b``, one-token sequences included: the host cannot
    tell that every ``T_b`` is 1 without reading ``cu_seqlens``.  For pure one-token decoding a padded ``[B, 1, H, D]``
    step (``attention_with_kv_cache``, split-KV) or a captured step stays the fast path.  ``block_table``: paged
    caches, as in ``attention_with_kv_cache``."""
    _check_no_grad(q, k_cache, v_cache, k_new, v_new, bias)
    T, _, max_len, bound = _kv_cache_varlen_plan(q, k_cache, v_cache, cu_seqlens, max_seqlen, seqlens, max_len,
                                                 k_new, v_new, block_table)
    if scale is None:
        scale = 1.0 / math.sqrt(q.shape[-1])
    if not _kvcache_varlen_supported(q, k_cache, v_cache, cu_seqlens, seqlens, k_new, v_new, bias, key_padding_mask,
                                     block_table):
        return attention_with_kv_cache_varlen_reference(q, k_cache, v_cache, cu_seqlens, T, seqlens, max_len, k_new,
                                                        v_new, bias, key_padding_mask, scale, block_table)
    B = cu_seqlens.numel() - 1
    seqlens, bias, key_padding_mask = _native_cache_operands(q, seqlens, bias, key_padding_mask, bound, B, T, True)
    cu_seqlens = cu_seqlens.to(torch.int32).contiguous()
    return native().kvcache.fmha_kvcache_varlen_fwd(q, k_cache, v_cache, cu_seqlens, T, seqlens,
                                                    0 if max_len is None else int(max_len), k_new, v_new, bias,
                                                    key_padding_mask, float(scale),
                                                    block_table=_native_table(block_table))


# ---- paged caches: the append on its own and the block allocator ----------------------------------------------------
def kv_cache_append(k_new, v_new, k_cache, v_cache, seqlens, block_table=None):
    """Rows ``i`` of ``k_new`` / ``v_new [B, T, H_kv, D]`` written bitwise into rows ``p_b + i`` of the caches, ``p_b =
    clamp(seqlens[b], 0, C)``: ``[B, C, H_kv, D]``, or pools through ``block_table`` (``attention_with_kv_cache``).
    Rows at or past ``C``, and rows whose table entry is outside the pool, are skipped.  This is the append of a chunk
    step without its attention: a paged prefill stores its keys and values with it (``seqlens`` = 0)."""
    B, T = k_new.shape[:2]
    if block_table is not None:
        _check_block_table(block_table, k_cache, v_cache, B)
    if use_native(k_new, v_new, k_cache, v_cache, seqlens, block_table) and _kernel_tensors(k_new, v_new, k_cache,
                                                                                            v_cache):
        native().kvcache.kv_cache_append(k_new, v_new, k_cache, v_cache, seqlens.to(torch.int32).contiguous(),
                                         _native_table(block_table))
        return
    C = cache_capacity(k_cache, block_table)
    rows = seqlens.long().to(k_cache.device).clamp(0, C)[:, None] + torch.arange(T, device=k_cache.device)[None, :]
    _cache_store(k_cache, block_table, rows, rows < C, k_new)
    _cache_store(v_cache, block_table, rows, rows < C, v_new)


def _check_kv_blocks(block_table, free_list, free_count, lengths, block_size, overflow=None):
    for name, t in (("block_table", block_table), ("free_list", free_list), ("free_count", free_count),
                    ("overflow", overflow)):
        if t is not None and (t.dtype != torch.int32 or not t.is_contiguous()):
            raise ValueError("{} must be a contiguous int32 tensor (it is updated in place)".format(name))
    if block_table.dim() != 2 or free_list.dim() != 1 or free_list.numel() < 1 or free_count.numel() != 1 \
            or (overflow is not None and overflow.numel() != 1):
        raise ValueError("the allocator takes block_table [B, M], free_list [num_blocks >= 1], free_count [1] and "
                         "overflow [1]")
    if lengths.shape != (block_table.shape[0],):
        raise ValueError("lengths must be [B = {}], not {}".format(block_table.shape[0], tuple(lengths.shape)))
    if int(block_size) < 1:
        raise ValueError("block_size must be positive, not {}".format(block_size))
    return lengths.to(device=block_table.device, dtype=torch.int32).contiguous()


def _kv_blocks_flags(block_table, lengths, block_size):
    """``(kept [B, M], table [B * M] int64)``: the entries below ``ceil(clamp(lengths[b], 0, C) / block_size)``."""
    B, M = block_table.shape
    n = lengths.long().clamp(0, M * block_size)
    kept = torch.arange(M, device=block_table.device)[None, :] < ((n + block_size - 1) // block_size)[:, None]
    return kept, block_table.reshape(-1).long()


def kv_blocks_reserve(block_table, free_list, free_count, lengths, block_size, overflow):
    """Give every sequence b a block for each table entry below ``ceil(clamp(lengths[b], 0, C) / block_size)`` that
    has none (< 0), off the top of the free stack (``free_list[free_count - 1]`` first), in the order (b, i)
    ascending.  When the stack runs out the entry stays -1 and ``overflow`` (int32 ``[1]``) is set to 1.  All int32
    tensors on one device, updated in place; nothing is read on the host, so a CUDA graph can hold the call.  The
    block ids depend only on the inputs (``kv_blocks`` kernels, or the same result in PyTorch)."""
    lengths = _check_kv_blocks(block_table, free_list, free_count, lengths, block_size, overflow)
    if use_native(block_table, free_list, free_count, lengths, overflow):
        native().kvcache.kv_blocks_reserve(block_table, free_list, free_count, lengths, int(block_size), overflow)
        return
    kept, table = _kv_blocks_flags(block_table, lengths, block_size)
    NB = free_list.numel()
    need = kept.reshape(-1) & (table < 0)
    k = need.long().cumsum(0) - need.long()   # the stack slot each needing entry takes, counted from the top
    count = free_count.long().clamp(0, NB)
    give = need & (k < count)
    src = (count - 1 - k).clamp(0, NB - 1)
    block_table.copy_(torch.where(give, free_list.long()[src], table).view_as(block_table))
    overflow.copy_(torch.where((need & ~give).any(), torch.ones_like(overflow), overflow))
    free_count.copy_(count - torch.minimum(need.long().sum(), count))


def kv_blocks_release(block_table, free_list, free_count, lengths, block_size):
    """Push every block at or past entry ``ceil(clamp(lengths[b], 0, C) / block_size)`` of sequence b back onto the
    free stack, in the order (b, i) ascending, and set those entries to -1.  Entries outside ``[0, num_blocks)`` are
    dropped, not pushed.  In place and on the device, as ``kv_blocks_reserve``."""
    lengths = _check_kv_blocks(block_table, free_list, free_count, lengths, block_size)
    if use_native(block_table, free_list, free_count, lengths):
        native().kvcache.kv_blocks_release(block_table, free_list, free_count, lengths, int(block_size))
        return
    kept, table = _kv_blocks_flags(block_table, lengths, block_size)
    NB = free_list.numel()
    drop = ~kept.reshape(-1)
    push = drop & (table >= 0) & (table < NB)
    count = free_count.long().clamp(0, NB)
    slot = count + push.long().cumsum(0) - push.long()
    ok = push & (slot < NB)
    stack = torch.cat([free_list.long(), free_list.new_zeros(1, dtype=torch.long)])   # slot NB: dropped writes
    stack.scatter_(0, torch.where(ok, slot, torch.full_like(slot, NB)), table)
    free_list.copy_(stack[:NB])
    block_table.copy_(torch.where(drop, torch.full_like(table, -1), table).view_as(block_table))
    free_count.copy_(torch.minimum(count + push.long().sum(), torch.full_like(count, NB)))
