"""Token-major <-> head-major relayout (``csrc/fused/head_permute.cu``).

``split_heads`` turns a packed projection ``[B, L, T*H*D]`` (``T`` = 3 for q|k|v) into ``T`` contiguous
``[B, H, L, D]`` tensors with ONE kernel (the query scale folded in), ``merge_heads`` is the inverse; each is
the other's backward, so the packed gradient of the in-projection is gathered by one kernel from the three
gradients autograd hands back (reference formulation: ``unicore/modules/multihead_attention.py:62-76,105-110``
- view / transpose / contiguous chains whose backward zero-fills and adds three full-size tensors).
"""
from typing import Optional, Sequence, Tuple

import torch

from ._native import aligned_param, native, use_native


def _eligible(x: torch.Tensor, head_dim: int) -> bool:
    return (
        use_native(x)
        and x.dtype in (torch.float16, torch.bfloat16, torch.float32)
        and (head_dim * x.element_size()) % 16 == 0
        and x.numel() > 0
    )


def _split_reference(x, num_slices, num_heads, scale0):
    bsz, seq_len, width = x.shape
    parts = x.view(bsz, seq_len, num_slices, num_heads, width // (num_slices * num_heads)).permute(2, 0, 3, 1, 4)
    out = [parts[t].contiguous() for t in range(num_slices)]
    if scale0 != 1.0:
        out[0] = out[0] * scale0
    return tuple(out)


def _merge_reference(heads: Sequence[Optional[torch.Tensor]], scale0):
    ref = next(h for h in heads if h is not None)
    full = [torch.zeros_like(ref) if h is None else h for h in heads]
    if scale0 != 1.0:
        full[0] = full[0] * scale0
    bsz, num_heads, seq_len, dim = ref.shape
    return torch.stack(full, dim=0).permute(1, 3, 0, 2, 4).reshape(bsz, seq_len, len(full) * num_heads * dim)


class _SplitHeadsFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, num_slices, num_heads, scale0):
        ctx.scale0 = scale0
        return tuple(native().split_heads(x, num_slices, num_heads, scale0))

    @staticmethod
    def backward(ctx, *grads):
        return native().merge_heads([aligned_param(g) for g in grads], ctx.scale0), None, None, None


class _MergeHeadsFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, scale0, *heads):
        ctx.scale0 = scale0
        ctx.count = len(heads)
        ctx.num_heads = heads[0].shape[1]
        return native().merge_heads(list(heads), scale0)

    @staticmethod
    def backward(ctx, grad):
        parts = native().split_heads(aligned_param(grad), ctx.count, ctx.num_heads, ctx.scale0)
        return (None,) + tuple(parts)


def split_heads(x: torch.Tensor, num_slices: int, num_heads: int, scale0: float = 1.0) -> Tuple[torch.Tensor, ...]:
    """``[B, L, T*H*D] -> T x [B, H, L, D]`` (contiguous); slice 0 is multiplied by ``scale0``."""
    if x.dim() != 3 or x.shape[-1] % (num_slices * num_heads) != 0:
        raise ValueError("expected [B, L, T*H*D], got {}".format(tuple(x.shape)))
    head_dim = x.shape[-1] // (num_slices * num_heads)
    if 1 <= num_slices <= 4 and _eligible(x, head_dim):
        # the kernel moves 16-byte vectors: a view at an odd element offset is copied once (aligned_param), here and
        # for every tensor below that reaches a binding
        return _SplitHeadsFn.apply(aligned_param(x), num_slices, num_heads, float(scale0))
    return _split_reference(x.contiguous(), num_slices, num_heads, float(scale0))


def merge_heads(*heads: torch.Tensor, scale0: float = 1.0) -> torch.Tensor:
    """``T x [B, H, L, D] -> [B, L, T*H*D]``; slice 0 is multiplied by ``scale0``."""
    ref = heads[0]
    if ref.dim() != 4:
        raise ValueError("expected [B, H, L, D], got {}".format(tuple(ref.shape)))
    if 1 <= len(heads) <= 4 and _eligible(ref, ref.shape[-1]):
        return _MergeHeadsFn.apply(float(scale0), *[aligned_param(h) for h in heads])
    return _merge_reference(list(heads), float(scale0))


# ------------------------------------------------------------------------------------------------
# pair representation: head-major [B, H, Lq, Lk] <-> pair-major [B, Lq, Lk, H]
# ------------------------------------------------------------------------------------------------
def _pair_eligible(x: torch.Tensor, heads: int, lq: int, lk: int, need_lk8: bool) -> bool:
    return (
        use_native(x)
        and x.dtype in (torch.float16, torch.bfloat16)
        and heads % 8 == 0
        and (lq * lk) % 8 == 0
        and (lk % 8 == 0 or not need_lk8)
        and x.numel() > 0
    )


class _PairTransposeFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, to_pair):
        ctx.to_pair = to_pair
        return native().pair_transpose(x, to_pair)

    @staticmethod
    def backward(ctx, grad):
        return native().pair_transpose(aligned_param(grad), not ctx.to_pair), None


def heads_to_pair(x: torch.Tensor) -> torch.Tensor:
    """``[B, H, Lq, Lk] -> [B, Lq, Lk, H]`` (contiguous) - register-tile transpose, see ``csrc/fused/pair_layout.cu``."""
    if x.dim() == 4 and _pair_eligible(x, x.shape[1], x.shape[2], x.shape[3], False):
        return _PairTransposeFn.apply(aligned_param(x), True)
    return x.permute(0, 2, 3, 1).contiguous()


def pair_to_heads(x: torch.Tensor) -> torch.Tensor:
    """``[B, Lq, Lk, H] -> [B, H, Lq, Lk]`` (contiguous)."""
    if x.dim() == 4 and _pair_eligible(x, x.shape[3], x.shape[1], x.shape[2], False):
        return _PairTransposeFn.apply(aligned_param(x), False)
    return x.permute(0, 3, 1, 2).contiguous()


class _PairTailFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, z, z0, key_pad):
        pair, delta = native().pair_tail_fwd(z, z0, key_pad)
        ctx.save_for_backward(z, key_pad)
        ctx.need_z0 = z0.requires_grad
        return pair, delta

    @staticmethod
    def backward(ctx, d_pair, d_delta):
        z, key_pad = ctx.saved_tensors
        dz, dz0 = native().pair_tail_bwd(aligned_param(d_pair), aligned_param(d_delta), z, key_pad)
        return dz, (dz0 if ctx.need_z0 else None), None


def pair_tail(logits: torch.Tensor, input_bias: torch.Tensor, key_padding_mask: Optional[torch.Tensor] = None):
    """Tail of a pair-bias encoder in one pass over the ``[B, H, Lq, Lk]`` logits.

    Returns ``(pair, delta)``, both pair-major ``[B, Lq, Lk, H]``:
    ``pair = logits`` with ``-inf -> 0`` and ``delta = logits - input_bias`` with padded key columns set to 0
    (Uni-Mol's ``TransformerEncoderWithPair`` computes them with a subtraction, two ``masked_fill``, an equality
    pass and two ``permute().contiguous()`` copies - and the mirror image of all that in backward).
    """
    if logits.shape != input_bias.shape or logits.dim() != 4:
        raise ValueError("pair_tail expects two [B, H, Lq, Lk] tensors")
    bsz, heads, lq, lk = logits.shape
    if key_padding_mask is not None:
        key_padding_mask = key_padding_mask.to(torch.bool)
    if _pair_eligible(logits, heads, lq, lk, True) and input_bias.dtype == logits.dtype:
        # the mask is read 8 flags at a time: it is copied like the logits when its view is not 16-byte aligned
        return _PairTailFn.apply(aligned_param(logits), aligned_param(input_bias), aligned_param(key_padding_mask))
    delta = logits - input_bias
    if key_padding_mask is not None:
        delta = delta.masked_fill(key_padding_mask[:, None, None, :], 0)
    pair = logits.masked_fill(logits == float("-inf"), 0)
    return pair.permute(0, 2, 3, 1).contiguous(), delta.permute(0, 2, 3, 1).contiguous()
