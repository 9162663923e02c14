"""Rotary position embeddings, rotate-half (GPT-NeoX / LLaMA) form (``csrc/fused/rotary.cu``).

``rotary_embedding(x, inv_freq, rotated_heads, position_offsets)`` takes ``x [B, L, N, D]`` (a packed projection
viewed as N heads, or one head slice of it) and returns a new ``[B, L, N, D]`` tensor in which the first
``rotated_heads`` heads of every token are rotated on their first ``rd = 2 * inv_freq.numel()`` columns and everything
else is copied.  Pair ``i < rd / 2`` is ``(x[i], x[i + rd/2])``; at position ``pos = l + offset[b]`` the angle is
``theta = fl32(float(pos) * inv_freq[i])`` and

    y1 = x1 cos(theta) - x2 sin(theta),   y2 = x2 cos(theta) + x1 sin(theta)

with cos / sin evaluated accurately (fp64 of the fp32 angle) and rounded to fp32, the rotation in fp32, one rounding to
the storage type.  ``position_offsets`` (int32 ``[B]``) is read on the device, so a captured decoding step follows the
cache lengths.  The op is out of place on purpose: rotating the module's view of the linear output in place would make
autograd wrap the backward in ``CopySlices``, which clones the whole packed gradient; a new tensor costs one copy of the
unrotated (value) heads in each direction instead.  The backward is the inverse rotation (``-theta``) into a new
tensor.
"""
from typing import Optional

import torch

from ._native import native, use_native

# the kernel keeps the cos / sin of a tile of tokens in shared memory up to this rotary dim
_MAX_KERNEL_ROTARY_DIM = 512


def rotary_inv_freq(rotary_dim: int, base: float = 10000.0, device=None) -> torch.Tensor:
    """fp32 ``[rotary_dim / 2]`` frequencies ``1 / base ** (arange(0, rotary_dim, 2) / rotary_dim)``."""
    if rotary_dim < 2 or rotary_dim % 2 != 0:
        raise ValueError("rotary_dim must be even and >= 2, not {}".format(rotary_dim))
    return 1.0 / (base ** (torch.arange(0, rotary_dim, 2, dtype=torch.float32, device=device) / rotary_dim))


def rotary_embedding_reference(x, inv_freq, rotated_heads=None, position_offsets=None, inverse=False):
    """The formula in PyTorch (the CPU / fp32 path, differentiable through autograd): the same fp32 angles and
    accurately rounded cos / sin as the kernel, the rotation in fp32."""
    B, L, N, D = x.shape
    R = N if rotated_heads is None else rotated_heads
    half = inv_freq.numel()
    pos = torch.arange(L, device=x.device).view(1, L)
    if position_offsets is not None:
        pos = pos + position_offsets.to(device=x.device, dtype=torch.long).view(-1, 1)
    theta = pos.to(torch.float32)[..., None] * inv_freq.to(device=x.device, dtype=torch.float32)   # [B|1, L, half]
    cos = theta.double().cos().float()[:, :, None, :]
    sin = theta.double().sin().float()[:, :, None, :]
    if inverse:
        sin = -sin
    rot = x[:, :, :R]
    x1, x2 = rot[..., :half].float(), rot[..., half:2 * half].float()
    y = torch.cat([(x1 * cos - x2 * sin).to(x.dtype), (x2 * cos + x1 * sin).to(x.dtype), rot[..., 2 * half:]], dim=-1)
    return torch.cat([y, x[:, :, R:]], dim=2)


def _kernel_takes(x, inv_freq, position_offsets) -> bool:
    return (
        use_native(x, inv_freq, position_offsets)
        and x.dtype in (torch.float16, torch.bfloat16)
        and inv_freq.dtype == torch.float32 and inv_freq.is_contiguous()
        and 2 * inv_freq.numel() <= min(x.size(3), _MAX_KERNEL_ROTARY_DIM)
        and x.stride(3) == 1 and (x.size(2) == 1 or x.stride(2) == x.size(3))
        and (position_offsets is None or (position_offsets.dtype == torch.int32 and position_offsets.is_contiguous()))
    )


class _RotaryFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, inv_freq, rotated_heads, position_offsets):
        ctx.rotated_heads = rotated_heads
        ctx.save_for_backward(inv_freq, position_offsets)
        return native().rotary.rotary_embedding(x, inv_freq, rotated_heads, position_offsets, False)

    @staticmethod
    def backward(ctx, grad):
        inv_freq, position_offsets = ctx.saved_tensors
        if grad.stride(3) != 1 or (grad.size(2) > 1 and grad.stride(2) != grad.size(3)):
            grad = grad.contiguous()
        dx = native().rotary.rotary_embedding(grad, inv_freq, ctx.rotated_heads, position_offsets, True)
        return dx, None, None, None


def rotary_embedding(x: torch.Tensor, inv_freq: torch.Tensor, rotated_heads: Optional[int] = None,
                     position_offsets: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``x [B, L, N, D]`` with its first ``rotated_heads`` heads (all when None) rotated at positions
    ``l + position_offsets[b]`` (``l`` when None); see the module docstring.  Differentiable in ``x``."""
    if x.dim() != 4:
        raise ValueError("rotary_embedding takes x [B, L, N, D], not {}".format(tuple(x.shape)))
    B, L, N, D = x.shape
    R = N if rotated_heads is None else int(rotated_heads)
    if not 0 <= R <= N:
        raise ValueError("rotated_heads must be in [0, {}], not {}".format(N, R))
    if inv_freq.dim() != 1 or not 2 <= 2 * inv_freq.numel() <= D:
        raise ValueError("inv_freq must be [rotary_dim / 2] with 2 <= rotary_dim <= head_dim {}, not {}".format(
            D, tuple(inv_freq.shape)))
    if position_offsets is not None and tuple(position_offsets.shape) != (B,):
        raise ValueError("position_offsets must be [B] = [{}], not {}".format(B, tuple(position_offsets.shape)))
    if _kernel_takes(x, inv_freq, position_offsets):
        return _RotaryFn.apply(x, inv_freq, R, position_offsets)
    return rotary_embedding_reference(x, inv_freq, R, position_offsets)
