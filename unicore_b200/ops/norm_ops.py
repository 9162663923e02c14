"""LayerNorm / RMSNorm with hand-written sm_90a forward and single-pass backward kernels.

Replaces reference extensions N4-N7 (``csrc/layernorm/layernorm.cu:25-148``, ``layernorm_backward.cu:130-247``,
``csrc/rmsnorm/rmsnorm.cu:25-125``, ``rmsnorm_backward.cu:108-196``; Python callers ``unicore/modules/layer_norm.py:22-48``,
``rms_norm.py:24-56``): any hidden size
(the reference supports 16 sizes), 128-bit accesses, fp32 statistics, and ONE backward kernel that
reads ``x`` and ``dy`` once and produces ``dx`` plus ``dgamma``/``dbeta`` partials reduced by the
last CTA (the reference reads them twice: dx kernel + two gamma/beta kernels).
"""
from typing import Optional

import torch
import torch.nn.functional as F

from . import grad_sink
from ._native import aligned_param, aligned_rows, native, use_native


class _LayerNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, eps):
        shape = x.shape
        x2 = aligned_rows(x)
        y, mean, rstd = native().layernorm_fwd(x2, weight, bias, eps)
        ctx.save_for_backward(x2, weight, mean, rstd)
        ctx.has_bias = bias is not None
        need = ctx.needs_input_grad  # gradients go straight into the arena
        ctx.sinks = (grad_sink.claim(weight, need[1]), grad_sink.claim(bias, need[2]))
        return y.view(shape)

    @staticmethod
    def backward(ctx, dy):
        x2, weight, mean, rstd = ctx.saved_tensors
        dy2 = aligned_rows(dy)
        g_sink, b_sink = ctx.sinks
        dx, dgamma, dbeta = native().layernorm_bwd(dy2, x2, mean, rstd, weight, grad_sink.sink(g_sink), grad_sink.sink(b_sink))
        if g_sink is not None:
            grad_sink.done(g_sink)
            dgamma = None
        if b_sink is not None:
            grad_sink.done(b_sink)
            dbeta = None
        return dx.view(dy.shape), dgamma, (dbeta if ctx.has_bias else None), None


class _RMSNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, eps):
        shape = x.shape
        x2 = aligned_rows(x)
        y, rstd = native().rmsnorm_fwd(x2, weight, eps)
        ctx.save_for_backward(x2, weight, rstd)
        ctx.g_sink = grad_sink.claim(weight, ctx.needs_input_grad[1])
        return y.view(shape)

    @staticmethod
    def backward(ctx, dy):
        x2, weight, rstd = ctx.saved_tensors
        dy2 = aligned_rows(dy)
        dx, dgamma = native().rmsnorm_bwd(dy2, x2, rstd, weight, grad_sink.sink(ctx.g_sink))
        if ctx.g_sink is not None:
            grad_sink.done(ctx.g_sink)
            dgamma = None
        return dx.view(dy.shape), dgamma, None


def _norm_supported(x: torch.Tensor, weight: Optional[torch.Tensor]) -> bool:
    if weight is None or x.dtype not in (torch.float16, torch.bfloat16, torch.float32) or x.numel() == 0:
        return False
    cols = x.shape[-1]
    epv = 16 // x.element_size()  # elements per 128-bit vector
    # a row is held in registers by <= 256 threads x 4 vectors
    return cols == weight.numel() and cols % epv == 0 and cols // epv <= 1024


def layer_norm(x, normalized_shape, weight, bias, eps=1e-5):
    """LayerNorm over the last dimension (biased variance, ``rsqrt(var + eps)``)."""
    if use_native(x, weight, bias) and len(normalized_shape) == 1 and _norm_supported(x, weight):
        w = aligned_param(weight, x.dtype)
        b = aligned_param(bias, x.dtype)
        return _LayerNormFn.apply(x, w, b, eps)
    return F.layer_norm(
        x, normalized_shape,
        weight.to(x.dtype) if weight is not None else None,
        bias.to(x.dtype) if bias is not None else None,
        eps,
    )


def rms_norm(x, normalized_shape, weight, eps=1e-5):
    """``y = x * rsqrt(mean(x^2) + eps) * weight`` over the last dimension."""
    if use_native(x, weight) and len(normalized_shape) == 1 and _norm_supported(x, weight):
        w = aligned_param(weight, x.dtype)
        return _RMSNormFn.apply(x, w, eps)
    if hasattr(F, "rms_norm"):
        return F.rms_norm(x, normalized_shape, weight.to(x.dtype) if weight is not None else None, eps)
    var = x.float().pow(2).mean(dim=-1, keepdim=True)
    y = (x.float() * torch.rsqrt(var + eps)).to(x.dtype)
    return y * weight.to(x.dtype) if weight is not None else y
