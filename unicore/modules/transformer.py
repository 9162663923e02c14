"""Transformer encoder / decoder stacks (BERT/XLM style, pre- or post-LN, T5 relative positions).

Parity: reference ``unicore/modules/transformer_encoder_layer.py:15``,
``transformer_encoder.py:16-162`` (``init_bert_params``, ``relative_position_bucket``,
``TransformerEncoder``), ``transformer_decoder_layer.py:15`` and ``transformer_decoder.py:19-169``.
Same constructor arguments, parameter names (=> identical ``state_dict`` keys) and forward
signatures, including ``return_attn`` on the encoder layer.

GPU execution plan for one layer (post-LN shown; pre-LN analogous):
  in_proj GEMM -> fused wgmma attention (bias tile + key padding + dropout inside) ->
  out_proj GEMM -> ONE kernel: bias + dropout + residual + LayerNorm ->
  fc1 GEMM -> ONE kernel: bias + GELU -> fc2 GEMM -> ONE kernel: bias + dropout + residual + LN.
The stacks hand every layer its masks in one form, whichever path the attention takes: the relative-position bias
as ``[1, H, L, L]`` (never repeated over the batch), plus a user ``attn_mask`` as ``[B, H, L, L]``, and the key padding
mask as ``[B, L]`` (never merged into the bias as ``-inf``).  The auto-regressive decoder's future mask is not a tensor
at all: its layers run self-attention with ``causal=True``.  The attention module alone chooses between the fused
kernels and the materialised path, and both take this form; the reference's merged ``[B*H, L, L]`` mask gives the same
result.
``attention_kv_heads`` (default ``None``: one key / value head per query head) makes every attention of the stack
grouped-query attention with that many key / value heads (``unicore/modules/attention.py``); the decoder's cache then
holds ``H_kv`` heads per layer.
``rotary_dim`` / ``rotary_base`` (default ``None``: off) give every layer's self-attention rotary position embeddings
(``SelfMultiheadAttention``); they are independent of ``rel_pos``, and with ``rel_pos=False`` no attention of the stack
has a bias.  A decoding step rotates its tokens at the cache lengths ``seqlens``, which ``_decode_step`` advances only
after every layer, so all layers see the same positions.
``TransformerEncoder`` and its layers also take packed sequences: ``emb [N, E]`` with ``cu_seqlens`` (int ``[B + 1]`` on
the device) and ``max_seqlen`` (a host bound on the lengths) instead of a padded batch and its padding mask.  Every
token-wise kernel then runs on the N real tokens only, the relative-position bias is built at ``max_seqlen``, and the
attention runs in the varlen mode of the fused kernels; the output is packed ``[N, E]``.  ``TransformerDecoder`` takes
packed targets the same way, decoder-only or with a packed ``encoder_out [N_k, E]`` described by
``encoder_cu_seqlens`` / ``encoder_max_seqlen``: its self-attention is causal per sequence and its encoder attention
sees each target sequence's own source rows (the varlen kernels with separate key sequences).  With a ``DecoderCache``
the packed decoder takes each sequence's new tokens, a different count per sequence, into the cache (the prefill on
an empty one), through ``ops.attention_with_kv_cache_varlen``.
"""
import math
from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from unicore import ops, utils
from unicore_b200.ops.attention_ops import _varlen_lengths

from .attention import CrossMultiheadAttention, DecoderCache, SelfMultiheadAttention
from .norm import LayerNorm


# ------------------------------------------------------------------------------------------------
# initialisation + relative positions
# ------------------------------------------------------------------------------------------------
def init_bert_params(module):
    """N(0, 0.02) for Linear/Embedding weights, zero biases and padding rows.

    Values are drawn from the CPU generator (like the reference, so a given seed yields the same
    initial weights) but in one shot per tensor in the tensor's own dtype/device afterwards.
    """
    if not getattr(module, "can_global_init", True):
        return

    def draw(weight):
        fresh = torch.empty(weight.shape, dtype=torch.float32, device="cpu").normal_(mean=0.0, std=0.02)
        weight.copy_(fresh.to(device=weight.device, dtype=weight.dtype))

    with torch.no_grad():
        if isinstance(module, nn.Linear):
            draw(module.weight.data)
            if module.bias is not None:
                module.bias.data.zero_()
        if isinstance(module, nn.Embedding):
            draw(module.weight.data)
            if module.padding_idx is not None:
                module.weight.data[module.padding_idx].zero_()


def relative_position_bucket(relative_position, num_buckets=32, max_distance=128):
    """Signed T5-style bucketing: exact buckets for small |d|, log-spaced up to ``max_distance``."""
    sign = torch.sign(relative_position)
    half = num_buckets // 2
    dist = torch.abs(relative_position)
    exact = half // 2
    top = half - 1 - exact
    log_bucket = exact + torch.ceil(
        torch.log(dist.float() / exact) / math.log((max_distance - 1) / exact) * top
    ).long()
    log_bucket = torch.clamp(log_bucket, max=half - 1)
    return torch.where(dist < exact, dist, log_bucket) * sign


def _build_rp_bucket(max_seq_len, bins, max_rel_pos):
    pos = torch.arange(max_seq_len, dtype=torch.long)
    bucket = relative_position_bucket(pos[None, :] - pos[:, None], num_buckets=bins, max_distance=max_rel_pos)
    return bucket - bucket.min()


def fill_with_neg_inf(t):
    return t.float().fill_(float("-inf")).type_as(t)


def bulid_future_mask(seq_len):  # (sic) name kept for API compatibility
    return torch.triu(fill_with_neg_inf(torch.zeros([seq_len, seq_len])), 1)


# ------------------------------------------------------------------------------------------------
# shared block pieces
# ------------------------------------------------------------------------------------------------
def _linear_no_bias(layer: nn.Linear, x):
    """GEMM only; the bias is applied by the fused epilogue kernel that follows."""
    return ops.linear(x, layer.weight, None)


class _BlockMixin:
    """Residual/FFN plumbing shared by encoder and decoder layers."""

    def _fused_ok(self, x):
        return ops.use_native(x) and x.dtype in (torch.float16, torch.bfloat16) and self._gelu

    def _attn_residual(self, attn_module, norm, residual, attn_in, **kw):
        """post-LN: LN(residual + drop(attn(x)));  pre-LN: residual + drop(attn(LN(x)))."""
        return_attn = kw.pop("return_attn", False)
        need_probs = kw.pop("need_probs", True)
        causal = kw.pop("causal", False)
        cache = kw.pop("cache", None)
        # packed sequences: passed on only when given, so that attend keeps its padded-batch signature otherwise
        packed = {} if kw.get("cu_seqlens") is None else {"cu_seqlens": kw["cu_seqlens"], "max_seqlen": kw["max_seqlen"]}
        kw.pop("cu_seqlens", None)
        kw.pop("max_seqlen", None)
        if kw.get("encoder_cu_seqlens") is not None:   # packed keys / values of the encoder attention
            packed.update(encoder_cu_seqlens=kw["encoder_cu_seqlens"], encoder_max_seqlen=kw["encoder_max_seqlen"])
        kw.pop("encoder_cu_seqlens", None)
        kw.pop("encoder_max_seqlen", None)
        h = attn_in if self.post_ln else norm(attn_in)
        extra = None
        if isinstance(attn_module, SelfMultiheadAttention):
            o, logits, probs = attn_module.attend(h, kw.get("key_padding_mask"), kw.get("attn_bias"), return_attn,
                                                  need_probs, causal, cache=cache, **packed)
            if return_attn:
                extra = (logits, probs)
        else:
            o = attn_module.attend(h, kw["key"], kw["value"], kw.get("key_padding_mask"), kw.get("attn_bias"),
                                   cache=cache, **packed)
        proj = attn_module.out_proj
        if self.post_ln and self._fused_ok(o):
            # out_proj bias + dropout + residual + LayerNorm in one pass over the GEMM output
            out = ops.bias_dropout_add_layer_norm(
                ops.linear(o, proj.weight, None), proj.bias, residual, norm.weight, norm.bias,
                self.dropout, norm.eps, self.training,
            )
            return out, extra
        out = residual + F.dropout(ops.linear(o, proj.weight, proj.bias), p=self.dropout, training=self.training)
        if self.post_ln:
            out = norm(out)
        return out, extra

    def _ffn_residual(self, x):
        residual = x
        if self._fused_ok(x):
            h = x if self.post_ln else self.final_layer_norm(x)
            h = ops.bias_gelu(_linear_no_bias(self.fc1, h), self.fc1.bias)
            h = F.dropout(h, p=self.activation_dropout, training=self.training)
            if self.post_ln:
                return ops.bias_dropout_add_layer_norm(
                    _linear_no_bias(self.fc2, h), self.fc2.bias, residual,
                    self.final_layer_norm.weight, self.final_layer_norm.bias,
                    self.dropout, self.final_layer_norm.eps, self.training,
                )
            h = ops.linear(h, self.fc2.weight, self.fc2.bias)
            return residual + F.dropout(h, p=self.dropout, training=self.training)
        h = x if self.post_ln else self.final_layer_norm(x)
        h = self.activation_fn(self.fc1(h))
        h = F.dropout(h, p=self.activation_dropout, training=self.training)
        h = self.fc2(h)
        h = residual + F.dropout(h, p=self.dropout, training=self.training)
        return self.final_layer_norm(h) if self.post_ln else h


class TransformerEncoderLayer(nn.Module, _BlockMixin):
    def __init__(
        self,
        embed_dim: int = 768,
        ffn_embed_dim: int = 3072,
        attention_heads: int = 8,
        dropout: float = 0.1,
        attention_dropout: float = 0.1,
        activation_dropout: float = 0.0,
        activation_fn: str = "gelu",
        post_ln=False,
        attention_kv_heads: Optional[int] = None,
        rotary_dim: Optional[int] = None,
        rotary_base: float = 10000.0,
    ) -> None:
        super().__init__()
        self.embed_dim = embed_dim
        self.attention_heads = attention_heads
        self.attention_dropout = attention_dropout
        self.dropout = dropout
        self.activation_dropout = activation_dropout
        self.activation_fn = utils.get_activation_fn(activation_fn)
        self._gelu = activation_fn == "gelu"
        self.self_attn = SelfMultiheadAttention(self.embed_dim, attention_heads, dropout=attention_dropout,
                                                num_kv_heads=attention_kv_heads, rotary_dim=rotary_dim,
                                                rotary_base=rotary_base)
        self.self_attn_layer_norm = LayerNorm(self.embed_dim)
        self.fc1 = nn.Linear(self.embed_dim, ffn_embed_dim)
        self.fc2 = nn.Linear(ffn_embed_dim, self.embed_dim)
        self.final_layer_norm = LayerNorm(self.embed_dim)
        self.post_ln = post_ln

    def forward(
        self,
        x: torch.Tensor,
        attn_bias: Optional[torch.Tensor] = None,
        padding_mask: Optional[torch.Tensor] = None,
        return_attn: bool = False,
        need_probs: bool = True,
        cu_seqlens: Optional[torch.Tensor] = None,
        max_seqlen: Optional[int] = None,
    ) -> torch.Tensor:
        """With ``return_attn`` returns ``(x, logits, probs)``; ``need_probs=False`` makes ``probs`` None and lets the
        fused attention kernel produce the logits.  ``cu_seqlens`` / ``max_seqlen``: ``x`` is packed ``[N, E]`` (see
        the module docstring)."""
        x, extra = self._attn_residual(
            self.self_attn, self.self_attn_layer_norm, x, x,
            key_padding_mask=padding_mask, attn_bias=attn_bias, return_attn=return_attn, need_probs=need_probs,
            cu_seqlens=cu_seqlens, max_seqlen=max_seqlen,
        )
        x = self._ffn_residual(x)
        if not return_attn:
            return x
        attn_weights, attn_probs = extra
        return x, attn_weights, attn_probs


class TransformerDecoderLayer(nn.Module, _BlockMixin):
    def __init__(
        self,
        embed_dim: int = 768,
        ffn_embed_dim: int = 3072,
        attention_heads: int = 8,
        dropout: float = 0.1,
        attention_dropout: float = 0.1,
        activation_dropout: float = 0.0,
        activation_fn: str = "gelu",
        post_ln=False,
        attention_kv_heads: Optional[int] = None,
        rotary_dim: Optional[int] = None,
        rotary_base: float = 10000.0,
    ) -> None:
        super().__init__()
        self.embed_dim = embed_dim
        self.attention_heads = attention_heads
        self.attention_dropout = attention_dropout
        self.dropout = dropout
        self.activation_dropout = activation_dropout
        self.activation_fn = utils.get_activation_fn(activation_fn)
        self._gelu = activation_fn == "gelu"
        self.self_attn = SelfMultiheadAttention(self.embed_dim, attention_heads, dropout=attention_dropout,
                                                num_kv_heads=attention_kv_heads, rotary_dim=rotary_dim,
                                                rotary_base=rotary_base)
        self.self_attn_layer_norm = LayerNorm(self.embed_dim)
        self.encoder_attn = CrossMultiheadAttention(self.embed_dim, attention_heads, dropout=attention_dropout,
                                                    num_kv_heads=attention_kv_heads)
        self.encoder_attn_layer_norm = LayerNorm(self.embed_dim)
        self.fc1 = nn.Linear(self.embed_dim, ffn_embed_dim)
        self.fc2 = nn.Linear(ffn_embed_dim, self.embed_dim)
        self.final_layer_norm = LayerNorm(self.embed_dim)
        self.post_ln = post_ln

    def forward(
        self,
        x: torch.Tensor,
        encoder_out: torch.Tensor = None,
        attn_bias: Optional[torch.Tensor] = None,
        padding_mask: Optional[torch.Tensor] = None,
        encoder_attn_bias: Optional[torch.Tensor] = None,
        encoder_padding_mask: Optional[torch.Tensor] = None,
        causal: bool = False,
        cache=None,
        cu_seqlens: Optional[torch.Tensor] = None,
        max_seqlen: Optional[int] = None,
        encoder_cu_seqlens: Optional[torch.Tensor] = None,
        encoder_max_seqlen: Optional[int] = None,
    ) -> torch.Tensor:
        """``causal`` masks future keys in the self-attention (key j > query i), without a mask tensor on the fused
        path; the encoder attention is unaffected.  ``cache``: this layer's ``LayerKVCache`` of a ``DecoderCache``
        (see ``TransformerDecoder.forward``); on a decoding step the encoder attention uses the encoder keys and values
        it stored on the prefill, and ``encoder_out`` may be None.  ``cu_seqlens`` / ``max_seqlen``: ``x`` is packed
        ``[N, E]``; ``encoder_cu_seqlens`` / ``encoder_max_seqlen``: ``encoder_out`` is packed ``[N_k, E]`` (see the
        module docstring)."""
        x, _ = self._attn_residual(
            self.self_attn, self.self_attn_layer_norm, x, x, key_padding_mask=padding_mask, attn_bias=attn_bias,
            causal=causal, cache=cache, cu_seqlens=cu_seqlens, max_seqlen=max_seqlen,
        )
        if encoder_out is not None or (cache is not None and cache.stepping and cache.enc_k is not None):
            x, _ = self._attn_residual(
                self.encoder_attn, self.encoder_attn_layer_norm, x, x,
                key=encoder_out, value=encoder_out,
                key_padding_mask=encoder_padding_mask, attn_bias=encoder_attn_bias, cache=cache,
                cu_seqlens=cu_seqlens, max_seqlen=max_seqlen, encoder_cu_seqlens=encoder_cu_seqlens,
                encoder_max_seqlen=encoder_max_seqlen,
            )
        return self._ffn_residual(x)


# ------------------------------------------------------------------------------------------------
# stacks
# ------------------------------------------------------------------------------------------------
class _StackMixin:
    def _init_rel_pos(self, rel_pos, rel_pos_bins, max_rel_pos):
        self.rel_pos = rel_pos
        if not rel_pos:
            return
        if rel_pos_bins % 2 != 0:
            raise ValueError("rel_pos_bins must be even")
        self.rel_pos_bins = rel_pos_bins
        self.max_rel_pos = max_rel_pos
        self.relative_attention_bias = nn.Embedding(rel_pos_bins, self.attention_heads)
        self.rp_bucket = _build_rp_bucket(self.max_seq_len, rel_pos_bins, max_rel_pos)

    def get_rel_pos_bias(self, x, seq_len=None):
        """``[H, L, L]`` bias from the bucket table (positions assumed ordered), ``L = seq_len`` or ``x.size(1)``."""
        if self.rp_bucket.device != x.device:
            self.rp_bucket = self.rp_bucket.to(x.device)
        seq_len = x.size(1) if seq_len is None else int(seq_len)
        weight = self.relative_attention_bias.weight
        one_hot_bytes = self.rel_pos_bins * seq_len * seq_len * 2
        if weight.is_cuda and weight.dtype in (torch.float16, torch.bfloat16) and one_hot_bytes <= (64 << 20):
            # The bucket table is a constant: with its one-hot matrix E [bins, L*L] (cached) the lookup is the GEMM
            # W^T E - it lands directly in [H, L, L] order (no permute copy), and autograd's backward is the GEMM
            # dBias E^T with fp32 accumulation instead of ATen's embedding backward (a radix sort of L*L indices plus
            # a segmented reduction: 12 launches per BERT-base step).  Same values: each output element is
            # one table entry times 1.
            return (weight.t() @ self._bucket_one_hot(seq_len, weight)).view(-1, seq_len, seq_len)
        values = F.embedding(self.rp_bucket[:seq_len, :seq_len], weight)
        return values.permute(2, 0, 1).contiguous()

    def _bucket_one_hot(self, seq_len, like):
        key = (seq_len, like.device, like.dtype)
        cache = getattr(self, "_rp_one_hot", None)
        if cache is None or cache[0] != key:
            idx = self.rp_bucket[:seq_len, :seq_len].reshape(1, -1)
            one_hot = torch.zeros(self.rel_pos_bins, idx.numel(), dtype=like.dtype, device=like.device)
            one_hot.scatter_(0, idx, 1.0)
            self._rp_one_hot = cache = (key, one_hot)
        return cache[1]

    def _embed_prologue(self, emb, padding_mask):
        x = self.emb_layer_norm(emb)
        x = F.dropout(x, p=self.emb_dropout, training=self.training)
        if padding_mask is not None:
            x = x * (1 - padding_mask.unsqueeze(-1).type_as(x))
        return x

    def _compose_bias(self, x, attn_mask, padding_mask, bsz=None, seq_len=None):
        """What the layers receive: ``(attn_bias, key_padding_mask)``.

        ``attn_bias`` is None, the relative-position bias ``[1, H, L, L]``, or ``attn_mask`` (the reference's
        ``[B*H, L, L]``, or ``[B, L, L]`` for every head) viewed as ``[B, H, L, L]`` plus that bias.  The key padding mask
        ``[B, L]`` is passed on as it is.  ``bsz`` / ``seq_len``: B and L of packed sequences (default: ``x [B, L, E]``)."""
        bsz = x.size(0) if bsz is None else bsz
        seq_len = x.size(1) if seq_len is None else seq_len
        bias = self.get_rel_pos_bias(x, seq_len).unsqueeze(0) if self.rel_pos else None  # [1, H, L, L]
        if attn_mask is not None:
            mask = attn_mask.view(bsz, -1, seq_len, seq_len).expand(bsz, self.attention_heads, seq_len, seq_len)
            bias = mask if bias is None else mask + bias
        return bias, padding_mask


class TransformerEncoder(nn.Module, _StackMixin):
    def __init__(
        self,
        encoder_layers: int = 6,
        embed_dim: int = 768,
        ffn_embed_dim: int = 3072,
        attention_heads: int = 8,
        emb_dropout: float = 0.1,
        dropout: float = 0.1,
        attention_dropout: float = 0.1,
        activation_dropout: float = 0.0,
        max_seq_len: int = 256,
        activation_fn: str = "gelu",
        rel_pos: bool = True,
        rel_pos_bins: int = 32,
        max_rel_pos: int = 128,
        post_ln: bool = False,
        attention_kv_heads: Optional[int] = None,
        rotary_dim: Optional[int] = None,
        rotary_base: float = 10000.0,
    ) -> None:
        super().__init__()
        self.emb_dropout = emb_dropout
        self.max_seq_len = max_seq_len
        self.embed_dim = embed_dim
        self.attention_heads = attention_heads
        self.emb_layer_norm = LayerNorm(self.embed_dim)
        self.final_layer_norm = None if post_ln else LayerNorm(self.embed_dim)
        self.layers = nn.ModuleList(
            [
                TransformerEncoderLayer(
                    embed_dim=self.embed_dim,
                    ffn_embed_dim=ffn_embed_dim,
                    attention_heads=attention_heads,
                    dropout=dropout,
                    attention_dropout=attention_dropout,
                    activation_dropout=activation_dropout,
                    activation_fn=activation_fn,
                    post_ln=post_ln,
                    attention_kv_heads=attention_kv_heads,
                    rotary_dim=rotary_dim,
                    rotary_base=rotary_base,
                )
                for _ in range(encoder_layers)
            ]
        )
        self._init_rel_pos(rel_pos, rel_pos_bins, max_rel_pos)

    def forward(
        self,
        emb: torch.Tensor,
        attn_mask: Optional[torch.Tensor] = None,
        padding_mask: Optional[torch.Tensor] = None,
        cu_seqlens: Optional[torch.Tensor] = None,
        max_seqlen: Optional[int] = None,
    ) -> torch.Tensor:
        """``emb [B, L, E]`` (right-padded as ``padding_mask`` says), or packed ``emb [N, E]`` with ``cu_seqlens`` and
        ``max_seqlen``; ``attn_mask`` is then ``[B*H | B, max_seqlen, max_seqlen]``.  Returns the input's layout.
        Without ``attn_mask``, ``max_seqlen`` is rounded up to a multiple of 8 (the row width of the kernels' bias and
        side tensors), which changes no result; an ``attn_mask`` whose width is not a multiple of 8 makes the attention
        take the materialised varlen reference, as a padded batch of that width does."""
        if cu_seqlens is not None:
            if padding_mask is not None:
                raise ValueError("packed sequences (cu_seqlens) have no padding_mask")
            if max_seqlen is None:
                raise ValueError("cu_seqlens needs max_seqlen, a host bound on the lengths")
            x = self._embed_prologue(emb, None)   # no pad rows to zero
            if attn_mask is None:
                max_seqlen = int(max_seqlen) + (-int(max_seqlen) % 8)
            attn_bias, _ = self._compose_bias(x, attn_mask, None, cu_seqlens.numel() - 1, max_seqlen)
            for layer in self.layers:
                x = layer(x, attn_bias=attn_bias, cu_seqlens=cu_seqlens, max_seqlen=max_seqlen)
            return x if self.final_layer_norm is None else self.final_layer_norm(x)
        x = self._embed_prologue(emb, padding_mask)
        attn_bias, key_padding = self._compose_bias(x, attn_mask, padding_mask)
        for layer in self.layers:
            x = layer(x, padding_mask=key_padding, attn_bias=attn_bias)
        if self.final_layer_norm is not None:
            x = self.final_layer_norm(x)
        return x


class TransformerDecoder(nn.Module, _StackMixin):
    def __init__(
        self,
        decoder_layers: int = 6,
        embed_dim: int = 768,
        ffn_embed_dim: int = 3072,
        attention_heads: int = 8,
        emb_dropout: float = 0.1,
        dropout: float = 0.1,
        attention_dropout: float = 0.1,
        activation_dropout: float = 0.0,
        max_seq_len: int = 256,
        activation_fn: str = "gelu",
        rel_pos: bool = True,
        rel_pos_bins: int = 32,
        max_rel_pos: int = 128,
        post_ln: bool = False,
        auto_regressive: bool = True,
        attention_kv_heads: Optional[int] = None,
        rotary_dim: Optional[int] = None,
        rotary_base: float = 10000.0,
    ) -> None:
        super().__init__()
        self.emb_dropout = emb_dropout
        self.max_seq_len = max_seq_len
        self.embed_dim = embed_dim
        self.attention_heads = attention_heads
        self.attention_kv_heads = attention_kv_heads
        self.emb_layer_norm = LayerNorm(self.embed_dim)
        self.auto_regressive = auto_regressive
        self.final_layer_norm = None if post_ln else LayerNorm(self.embed_dim)
        self.layers = nn.ModuleList(
            [
                TransformerDecoderLayer(
                    embed_dim=self.embed_dim,
                    ffn_embed_dim=ffn_embed_dim,
                    attention_heads=attention_heads,
                    dropout=dropout,
                    attention_dropout=attention_dropout,
                    activation_dropout=activation_dropout,
                    activation_fn=activation_fn,
                    post_ln=post_ln,
                    attention_kv_heads=attention_kv_heads,
                    rotary_dim=rotary_dim,
                    rotary_base=rotary_base,
                )
                for _ in range(decoder_layers)
            ]
        )
        self._init_rel_pos(rel_pos, rel_pos_bins, max_rel_pos)

    def get_future_mask(self, x, attn_mask):
        """Reference-format helper: returns ``[B*H, L, L]`` mask including the causal part."""
        if not self.auto_regressive:
            return attn_mask
        fm = bulid_future_mask(x.size(1)).to(x)
        if attn_mask is None:
            return fm.unsqueeze(0).repeat(x.size(0) * self.attention_heads, 1, 1)
        return attn_mask + fm

    def forward(
        self,
        emb,
        encoder_out: Optional[torch.Tensor] = None,
        padding_mask: Optional[torch.Tensor] = None,
        encoder_padding_mask: Optional[torch.Tensor] = None,
        attn_mask: Optional[torch.Tensor] = None,
        encoder_attn_mask: Optional[torch.Tensor] = None,
        cache: Optional[DecoderCache] = None,
        cu_seqlens: Optional[torch.Tensor] = None,
        max_seqlen: Optional[int] = None,
        encoder_cu_seqlens: Optional[torch.Tensor] = None,
        encoder_max_seqlen: Optional[int] = None,
    ) -> torch.Tensor:
        """Without ``cache`` the whole sequence is decoded at once: ``emb [B, L, E]`` right-padded as ``padding_mask``
        says, or packed ``emb [N, E]`` with ``cu_seqlens`` and ``max_seqlen`` (see ``_forward_packed``).  With a
        ``DecoderCache`` (``new_cache``):

        * the first call (the prefill) takes the prompts ``emb [B, L, E]``, right-padded as ``padding_mask`` says, runs
          exactly the path above and stores every layer's keys / values of the L positions and its projected encoder
          keys / values; the cache then holds the unpadded lengths;
        * every later call (a step) takes T tokens per sequence, ``emb [B, T, E]`` at positions ``seqlens[b] ..
          seqlens[b] + T - 1`` (one token, or a chunk: a prompt continued, a long prompt fed in pieces, draft tokens to
          verify), and returns ``[B, T, E]``.  Its self-attention appends the tokens' keys / values and each token
          attends to the cache up to its own position; the encoder attention uses the stored encoder keys / values
          (``encoder_out`` may be None) with ``encoder_padding_mask``, and ``encoder_attn_mask``, if given, holds the
          rows of the new queries ``[B*H, T, S]``.  ``padding_mask`` and ``attn_mask`` are not supported on a step.
          ``cache.rewind`` drops tokens again.
        """
        if cu_seqlens is not None or encoder_cu_seqlens is not None:
            return self._forward_packed(emb, encoder_out, padding_mask, encoder_padding_mask, attn_mask,
                                        encoder_attn_mask, cache, cu_seqlens, max_seqlen, encoder_cu_seqlens,
                                        encoder_max_seqlen)
        if cache is not None:
            return self._forward_cached(emb, encoder_out, padding_mask, encoder_padding_mask, attn_mask,
                                        encoder_attn_mask, cache)
        return self._forward_prefix(emb, encoder_out, padding_mask, encoder_padding_mask, attn_mask, encoder_attn_mask)

    def _forward_packed(self, emb, encoder_out, padding_mask, encoder_padding_mask, attn_mask, encoder_attn_mask,
                        cache, cu_seqlens, max_seqlen, encoder_cu_seqlens, encoder_max_seqlen):
        """Packed target sequences ``emb [N, E]`` (``cu_seqlens`` int ``[B + 1]`` on the device, ``max_seqlen`` a host
        bound on their lengths), and, for encoder-decoder use, a packed ``encoder_out [N_k, E]`` of the same B
        sequences (``encoder_cu_seqlens``, ``encoder_max_seqlen``).  ``attn_mask`` is ``[B*H | B, max_seqlen,
        max_seqlen]`` and ``encoder_attn_mask`` ``[B*H | B, max_seqlen, encoder_max_seqlen]``.  Without a mask of that
        width, ``max_seqlen`` / ``encoder_max_seqlen`` are rounded up to a multiple of 8, which changes no result.
        The self-attention is causal per sequence when ``auto_regressive``; every token-wise kernel runs on the real
        rows only.  Returns packed ``[N, E]``.  No padding masks.  With a ``cache``: ``_forward_packed_cached``."""
        if cu_seqlens is None:
            raise ValueError("a packed encoder_out (encoder_cu_seqlens) needs a packed target (cu_seqlens)")
        if max_seqlen is None:
            raise ValueError("cu_seqlens needs max_seqlen, a host bound on the lengths")
        if cache is not None:
            return self._forward_packed_cached(emb, encoder_out, padding_mask, encoder_padding_mask, attn_mask,
                                               encoder_attn_mask, cache, cu_seqlens, int(max_seqlen),
                                               encoder_cu_seqlens)
        if padding_mask is not None or encoder_padding_mask is not None:
            raise ValueError("packed sequences (cu_seqlens) have no padding_mask or encoder_padding_mask")
        if (encoder_out is None) != (encoder_cu_seqlens is None):
            raise ValueError("a packed target takes a packed encoder_out with encoder_cu_seqlens, or neither")
        if encoder_cu_seqlens is not None:
            if encoder_max_seqlen is None:
                raise ValueError("encoder_cu_seqlens needs encoder_max_seqlen, a host bound on the source lengths")
            if encoder_cu_seqlens.dim() != 1 or encoder_cu_seqlens.numel() != cu_seqlens.numel():
                raise ValueError("encoder_cu_seqlens must describe the B = {} sequences of cu_seqlens, not {}".format(
                    cu_seqlens.numel() - 1, tuple(encoder_cu_seqlens.shape)))
            if encoder_attn_mask is None:
                encoder_max_seqlen = int(encoder_max_seqlen) + (-int(encoder_max_seqlen) % 8)
        x = self._embed_prologue(emb, None)   # no pad rows to zero
        if attn_mask is None and encoder_attn_mask is None:
            max_seqlen = int(max_seqlen) + (-int(max_seqlen) % 8)
        attn_bias, _ = self._compose_bias(x, attn_mask, None, cu_seqlens.numel() - 1, max_seqlen)
        for layer in self.layers:
            x = layer(x, encoder_out=encoder_out, attn_bias=attn_bias, encoder_attn_bias=encoder_attn_mask,
                      causal=self.auto_regressive, cu_seqlens=cu_seqlens, max_seqlen=max_seqlen,
                      encoder_cu_seqlens=encoder_cu_seqlens, encoder_max_seqlen=encoder_max_seqlen)
        return x if self.final_layer_norm is None else self.final_layer_norm(x)

    def _forward_packed_cached(self, emb, encoder_out, padding_mask, encoder_padding_mask, attn_mask,
                               encoder_attn_mask, cache, cu_seqlens, max_seqlen, encoder_cu_seqlens):
        """Packed new tokens into a ``DecoderCache``: ``emb [N, E]``, sequence b's ``T_b`` tokens on rows
        ``cu_seqlens[b] ..`` (clamped as the varlen kernels clamp them, ``T_b <= max_seqlen``) at positions
        ``seqlens[b] .. seqlens[b] + T_b - 1``; ``T_b`` may differ per sequence and be 0.  On an empty cache the call is
        the prefill, which also stores the projected padded ``encoder_out [B, S, E]``; every call appends each layer's
        keys / values of its tokens, attends with ``encoder_padding_mask [B, S]`` and ``encoder_attn_mask [B*H | B,
        max_seqlen, S]``, then advances ``cache.seqlens`` by ``T_b`` on the device (clamped to the capacity) and
        ``cache.max_len`` by ``max_seqlen``.  Returns ``[N, E]``.  Nothing is read on the host."""
        self._check_no_dropout()
        if encoder_cu_seqlens is not None:
            raise ValueError("a packed encoder_out (encoder_cu_seqlens) does not go into a cache: give it padded, "
                             "[B, S, E] with encoder_padding_mask")
        if padding_mask is not None or attn_mask is not None:
            raise ValueError("packed sequences (cu_seqlens) into a cache take no padding_mask or attn_mask")
        if cu_seqlens.dim() != 1 or cu_seqlens.numel() != cache.seqlens.numel() + 1:
            raise ValueError("cu_seqlens must have B + 1 = {} entries for the cache's sequences, not {}".format(
                cache.seqlens.numel() + 1, tuple(cu_seqlens.shape)))
        _check_room(cache, max_seqlen)
        _, lengths = _varlen_lengths(cu_seqlens.to(cache.seqlens.device), max_seqlen, emb.size(0))
        new_lengths = (cache.seqlens.clamp(0, cache.capacity) + lengths).clamp(max=cache.capacity)
        cache.reserve(new_lengths)
        x = self._embed_prologue(emb, None)
        attn_bias = self._step_rel_pos_bias(cache, x, max_seqlen) if self.rel_pos else None
        for layer, lc in zip(self.layers, cache.layers):
            x = layer(x, encoder_out=encoder_out, attn_bias=attn_bias, encoder_padding_mask=encoder_padding_mask,
                      encoder_attn_bias=encoder_attn_mask, cache=lc, cu_seqlens=cu_seqlens, max_seqlen=max_seqlen)
        cache.seqlens.copy_(new_lengths)
        cache.max_len += max_seqlen
        return x if self.final_layer_norm is None else self.final_layer_norm(x)

    def _forward_prefix(self, emb, encoder_out, padding_mask, encoder_padding_mask, attn_mask, encoder_attn_mask,
                        cache=None):
        """The whole sequence in one pass, final LayerNorm included; with a ``cache`` (the prefill) every layer also
        stores its keys / values in it."""
        x = self._embed_prologue(emb, padding_mask)
        attn_bias, key_padding = self._compose_bias(x, attn_mask, padding_mask)
        layer_caches = cache.layers if cache is not None else [None] * len(self.layers)
        for layer, lc in zip(self.layers, layer_caches):
            x = layer(x, encoder_out=encoder_out, padding_mask=key_padding, attn_bias=attn_bias,
                      encoder_padding_mask=encoder_padding_mask, encoder_attn_bias=encoder_attn_mask,
                      causal=self.auto_regressive, cache=lc)
        if self.final_layer_norm is not None:
            x = self.final_layer_norm(x)
        return x

    # ---- incremental decoding ------------------------------------------------------------------------------------
    def new_cache(self, batch_size, capacity, dtype=None, device=None, block_size=None,
                  num_blocks=None) -> DecoderCache:
        """An empty ``DecoderCache`` for ``batch_size`` sequences of up to ``capacity`` tokens (prompt included).
        ``capacity <= max_seq_len``: the relative-position table ends there.

        ``block_size`` (a multiple of 128 that divides ``capacity``): a paged cache, whose layers keep their keys and
        values in pools of ``num_blocks`` blocks of ``block_size`` rows, handed to the sequences as they grow.
        ``num_blocks`` defaults to ``batch_size * capacity / block_size``, which never runs out; a smaller pool serves
        a batch whose lengths are mostly below the capacity.  ``None`` (the default) is the contiguous
        ``[batch_size, capacity, H_kv, D]`` cache."""
        if not self.auto_regressive:
            raise ValueError("incremental decoding needs an auto-regressive decoder")
        if capacity > self.max_seq_len:
            raise ValueError("capacity {} exceeds max_seq_len {}".format(capacity, self.max_seq_len))
        if block_size is None:
            if num_blocks is not None:
                raise ValueError("num_blocks goes with block_size (a paged cache)")
        else:
            if int(block_size) != block_size or block_size < 1 or block_size % ops.PAGED_BLOCK_MULTIPLE != 0:
                raise ValueError("block_size must be a positive multiple of {}, not {}".format(
                    ops.PAGED_BLOCK_MULTIPLE, block_size))
            if capacity < 1 or capacity % block_size != 0:
                raise ValueError("capacity {} must be a positive multiple of block_size {}".format(capacity,
                                                                                                  block_size))
            if num_blocks is None:
                num_blocks = batch_size * capacity // block_size
            if int(num_blocks) != num_blocks or num_blocks < 1:
                raise ValueError("num_blocks must be a positive integer, not {}".format(num_blocks))
            block_size, num_blocks = int(block_size), int(num_blocks)
        weight = self.emb_layer_norm.weight
        heads = self.attention_heads
        kv_heads = self.attention_kv_heads or heads   # grouped-query attention caches H_kv heads
        return DecoderCache(len(self.layers), batch_size, capacity, kv_heads, self.embed_dim // heads,
                            dtype or weight.dtype, device or weight.device, block_size, num_blocks)

    def _check_no_dropout(self):
        rates = [self.emb_dropout]
        for layer in self.layers:
            rates += [layer.dropout, layer.attention_dropout, layer.activation_dropout]
        if self.training and any(r > 0 for r in rates):
            raise RuntimeError("incremental decoding runs without dropout: call eval() or set the dropout rates to 0")

    def _step_rel_pos_bias(self, cache, like, T=1, cols=None):
        """``[B, H, T, Lb]``: the relative-position bias rows of each sequence's T new tokens, gathered on the device at
        their positions ``seqlens[b] + i`` (keys past them are not visible).  ``Lb`` is ``cols`` when given (a captured
        step fixes it), else ``max_len + 1`` for one token and ``max_len + T`` rounded up to 8 for a chunk (the row
        stride the chunk kernel reads); columns past the bucket table are 0.  A wider bias has the same first
        columns."""
        if self.rp_bucket.device != like.device:
            self.rp_bucket = self.rp_bucket.to(like.device)
        if cols is None:
            cols = cache.max_len + T
            if T > 1:
                cols += -cols % 8
        width = min(cols, self.max_seq_len)
        pos = cache.seqlens.long()[:, None] + torch.arange(T, device=like.device)   # [B, T]
        idx = self.rp_bucket[pos.clamp(max=self.max_seq_len - 1), :width]   # [B, T, width]
        values = F.embedding(idx, self.relative_attention_bias.weight)   # [B, T, width, H]
        bias = values.permute(0, 3, 1, 2)
        if cols > width:
            bias = F.pad(bias, (0, cols - width))
        return bias.to(like.dtype).contiguous()

    def _forward_cached(self, emb, encoder_out, padding_mask, encoder_padding_mask, attn_mask, encoder_attn_mask,
                        cache):
        self._check_no_dropout()
        if cache.max_len == 0:
            # prefill: the ordinary path, with every layer storing its keys / values on the way
            L = emb.size(1)
            if L > cache.capacity:
                raise ValueError("the prompt ({} tokens) exceeds the cache capacity {}".format(L, cache.capacity))
            if padding_mask is None:
                lengths = torch.full_like(cache.seqlens, L)
            else:
                lengths = L - padding_mask.to(device=cache.seqlens.device, dtype=torch.int32).sum(1)
            cache.reserve(lengths)   # paged: blocks for the unpadded rows, before the layers store them
            x = self._forward_prefix(emb, encoder_out, padding_mask, encoder_padding_mask, attn_mask,
                                     encoder_attn_mask, cache)
            cache.seqlens.copy_(lengths)
            cache.max_len = L
            return x
        T = emb.size(1)
        if attn_mask is not None:
            raise NotImplementedError("attn_mask is not supported on a decoding step")
        if padding_mask is not None:
            raise NotImplementedError("padding_mask is not supported on a decoding step")
        _check_room(cache, T)
        x = self._decode_step(emb, encoder_out, encoder_padding_mask, encoder_attn_mask, cache)
        cache.max_len += T
        return x

    def _decode_step(self, emb, encoder_out, encoder_padding_mask, encoder_attn_mask, cache, bias_cols=None):
        """A step of T tokens into a non-empty cache, final LayerNorm included: appends the tokens' keys / values,
        attends and advances ``cache.seqlens`` by T on the device.  Every host-side shape follows ``cache.max_len``
        (and ``bias_cols``), which the caller advances."""
        T = emb.size(1)
        cache.reserve(cache.seqlens + T)
        x = self._embed_prologue(emb, None)
        attn_bias = self._step_rel_pos_bias(cache, x, T, bias_cols) if self.rel_pos else None
        for layer, lc in zip(self.layers, cache.layers):
            x = layer(x, encoder_out=encoder_out, attn_bias=attn_bias, encoder_padding_mask=encoder_padding_mask,
                      encoder_attn_bias=encoder_attn_mask, cache=lc)
        cache.seqlens += T
        if self.final_layer_norm is not None:
            x = self.final_layer_norm(x)
        return x

    def capture_step(self, cache, T=1, encoder_padding_mask=None, encoder_attn_mask=None):
        """A decoding step of T tokens per sequence into ``cache`` as a CUDA graph: returns a ``CapturedDecoderStep``,
        ``step(emb [B, T, E]) -> [B, T, E]``, which does what ``self(emb, encoder_padding_mask=...,
        encoder_attn_mask=..., cache=cache)`` does on a step, with one graph launch instead of a chain of kernel
        launches from Python.  Make it after the prefill (which stays eager: prompt lengths vary); it captures on its
        first call.  Needs CUDA, the native kernels, a 16-bit cache and no active dropout."""
        return CapturedDecoderStep(self, cache, T, encoder_padding_mask, encoder_attn_mask)


def _check_room(cache, T):
    if cache.max_len + T > cache.capacity:
        raise ValueError("{} more tokens do not fit the cache: {} of capacity {} are in use".format(
            T, cache.max_len, cache.capacity))


def _static_copy(buf, src, dtype, device):
    """``src`` written into the static buffer ``buf`` when the shapes match, else a copy of its own (whose new address
    makes the next call capture again)."""
    if src is None:
        return buf
    if buf is not None and buf.shape == src.shape:
        return buf.copy_(src)
    return src.to(device=device, dtype=dtype).clone(memory_format=torch.contiguous_format)


class CapturedDecoderStep:
    """A ``TransformerDecoder`` decoding step of T tokens per sequence captured in a CUDA graph
    (``TransformerDecoder.capture_step``).

    ``step(emb [B, T, E])`` copies ``emb`` into the graph's static input, replays the graph (append, attention, every
    layer, ``seqlens += T``), advances ``cache.max_len`` by T on the host and returns the graph's static output
    ``[B, T, E]``: the next call overwrites it, so clone what has to outlive it.  A step past the capacity raises
    before the replay.  ``encoder_padding_mask`` / ``encoder_attn_mask`` given to a call replace those of the capture.

    The graph is built for the largest host bound, ``max_len = capacity - T``: the relative-position bias has
    ``capacity`` columns (rounded up to 8 for a chunk), and the one-token decode attention divides each sequence's
    device length over its splits.  So the same graph serves every step until the cache is full, and between calls
    ``cache.reorder``, ``cache.rewind`` (an int or a device tensor) and a new prefill of the same shapes need no new
    capture: they write into the buffers the graph reads.  Before each replay the addresses and shapes of those
    buffers are compared with the ones captured; when one differs (a prefill with another encoder length, a reorder
    to another batch size, a mask of another shape) the step is captured again.  ``captures`` counts the captures."""

    def __init__(self, model, cache, T=1, encoder_padding_mask=None, encoder_attn_mask=None):
        k = cache.layers[0].k if cache.layers else None
        if not torch.cuda.is_available() or k is None or not k.is_cuda:
            raise RuntimeError("capture_step needs a CUDA device and a DecoderCache on it")
        if not ops.USE_NATIVE or k.dtype not in (torch.float16, torch.bfloat16) \
                or not ops.fused_head_dim_supported(k.size(-1)):
            raise RuntimeError("capture_step needs the native sm_90a kernels, an fp16 / bf16 cache and a head dim the "
                               "fused attention kernels take")
        model._check_no_dropout()
        if cache.max_len == 0:
            raise ValueError("capture_step comes after the prefill: the cache is empty")
        if not 1 <= T < cache.capacity:
            raise ValueError("a captured step takes 1 <= T < capacity ({}) tokens, not {}".format(cache.capacity, T))
        self.model, self.cache, self.T = model, cache, T
        self.captures = 0
        self._graph = self._out = self._emb = self._key = None
        self._enc_pad = _static_copy(None, encoder_padding_mask, torch.bool, k.device)
        self._enc_bias = _static_copy(None, encoder_attn_mask, k.dtype, k.device)

    def _buffers(self):
        """Every tensor the graph reads or writes besides its own intermediates."""
        bufs = [self.cache.seqlens, self._emb, self._enc_pad, self._enc_bias, self.cache.block_table,
                self.cache.free_list, self.cache.free_count, self.cache.overflow]
        for lc in self.cache.layers:
            bufs += [lc.k, lc.v, lc.enc_k, lc.enc_v]
        return bufs

    def _layout_key(self):
        return tuple(None if t is None else (t.data_ptr(), tuple(t.shape), t.dtype) for t in self._buffers())

    def _capture(self):
        model, cache, T = self.model, self.cache, self.T
        k = cache.layers[0].k
        B, cap = cache.seqlens.numel(), cache.capacity   # a paged cache's k is a pool: its size(0) is not B
        self._graph = self._out = None   # the old graph's memory pool goes back to the allocator
        if self._emb is None or self._emb.size(0) != B:
            self._emb = torch.zeros(B, T, model.embed_dim, dtype=k.dtype, device=k.device)
        cols = cap + (-cap % 8 if T > 1 else 0)
        args = (self._emb, None, self._enc_pad, self._enc_bias, cache, cols)
        seqlens, max_len = cache.seqlens.clone(), cache.max_len
        cache.max_len = cap - T   # the host bound every shape of the graph follows
        try:
            with torch.no_grad():
                # the warm-up really runs (loads the modules, lets cuBLAS pick its kernels) on a side stream, as capture
                # requires; it writes rows seqlens[b] .. seqlens[b] + T - 1 of the caches, which are not visible yet
                side = torch.cuda.Stream(device=k.device)
                side.wait_stream(torch.cuda.current_stream(k.device))
                with torch.cuda.stream(side):
                    model._decode_step(*args)
                torch.cuda.current_stream(k.device).wait_stream(side)
                cache.seqlens.copy_(seqlens)
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    out = model._decode_step(*args)
        finally:
            cache.seqlens.copy_(seqlens)
            cache.max_len = max_len
        self._graph, self._out = graph, out
        self._key = self._layout_key()
        self.captures += 1

    def __call__(self, emb, encoder_padding_mask=None, encoder_attn_mask=None):
        cache = self.cache
        if cache.max_len == 0:
            raise ValueError("the cache is empty: run the prefill first")
        _check_room(cache, self.T)
        self.model._check_no_dropout()
        k = cache.layers[0].k
        self._enc_pad = _static_copy(self._enc_pad, encoder_padding_mask, torch.bool, k.device)
        self._enc_bias = _static_copy(self._enc_bias, encoder_attn_mask, k.dtype, k.device)
        if self._graph is None or self._layout_key() != self._key:
            self._capture()
        self._emb.copy_(emb)
        self._graph.replay()
        cache.max_len += self.T
        return self._out
