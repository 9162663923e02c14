"""Optimizer-side ops: multi-tensor L2 norm / scale, fused Adam, stochastic rounding, EMA.

Native kernels: ``csrc/optim/*.cu`` (sm_90a, 128-bit vector accesses, any number of tensors per
launch through a device-side descriptor table).  Replaces reference extensions N1-N3
(``csrc/adam``, ``csrc/multi_tensor``, ``csrc/rounding``).  PyTorch fallbacks keep identical
math for CPU runs.
"""
import math
from typing import Dict, List, Sequence, Union

import torch

from ._native import native, use_native

Scalar = Union[float, torch.Tensor]


# ------------------------------------------------------------------------------------------------
# L2 norm / scale
# ------------------------------------------------------------------------------------------------
def multi_tensor_l2norm(tensors: Sequence[torch.Tensor], chunk_size: int = 2048 * 32) -> torch.Tensor:
    """``sqrt(sum_i ||t_i||^2)`` accumulated in fp32; returns a 0-dim fp32 tensor on the device.

    One launch for the whole list (reference: one launch per <=110 tensors + a cleanup kernel,
    ``multi_tensor_l2norm_kernel.cu:27-171``); the final sqrt is done by the last CTA to finish.
    Non-finite inputs propagate (inf/nan norm) - that is how fp16 overflow is detected.
    """
    tensors = [t for t in tensors if t is not None and t.numel() > 0]
    if len(tensors) == 0:
        return torch.zeros((), dtype=torch.float32)
    if use_native(*tensors):
        return native().multi_tensor_l2norm([t.detach() for t in tensors])
    total = None
    for t in tensors:
        sq = t.detach().float().pow(2).sum()
        total = sq if total is None else total + sq.to(total.device)
    return total.sqrt()


def multi_tensor_scale_(tensors: Sequence[torch.Tensor], scale: Scalar) -> None:
    """In-place ``t *= scale`` for every tensor; ``scale`` may be a device scalar (no host sync)."""
    tensors = [t for t in tensors if t is not None and t.numel() > 0]
    if len(tensors) == 0:
        return
    if use_native(*tensors):
        if torch.is_tensor(scale):
            native().multi_tensor_scale([t for t in tensors], 1.0, scale.detach().float().reshape(1))
        else:
            native().multi_tensor_scale([t for t in tensors], float(scale), None)
        return
    for t in tensors:
        if torch.is_tensor(scale):
            t.mul_(scale.to(device=t.device, dtype=t.dtype if t.is_floating_point() else None))
        else:
            t.mul_(scale)


# ------------------------------------------------------------------------------------------------
# Adam
# ------------------------------------------------------------------------------------------------
def _adam_reference_math(w: Dict, inv_scale, zero_grad: bool, stochastic_rounding: bool, ema_decay=None) -> None:
    """FusedAdam semantics in plain PyTorch (fp32 math), used on CPU."""
    p, g, m, v = w["p"], w["g"], w["m"], w["v"]
    beta1, beta2, eps, lr, wd, step = w["beta1"], w["beta2"], w["eps"], w["lr"], w["weight_decay"], w["step"]
    if w["bias_correction"]:
        step_size = lr * math.sqrt(1 - beta2 ** step) / (1 - beta1 ** step)
    else:
        step_size = lr
    grad = g.float() * inv_scale
    m.mul_(beta1).add_(grad, alpha=1 - beta1)
    v.mul_(beta2).addcmul_(grad, grad, value=1 - beta2)
    p32 = p.float() if p.dtype != torch.float32 else p
    p32.mul_(1 - step_size * wd).addcdiv_(m, v.sqrt().add_(eps), value=-step_size)
    if p32.data_ptr() != p.data_ptr():
        p.copy_(p32)
    half = w.get("p_half")
    if half is not None:
        if stochastic_rounding and half.dtype == torch.bfloat16:
            fp32_to_bf16_sr(p32, half)
        else:
            half.copy_(p32)
    if w.get("ema") is not None and ema_decay is not None:
        w["ema"].sub_(w["ema"] - p32, alpha=1.0 - ema_decay)
    if zero_grad:
        g.zero_()


@torch.no_grad()
def fused_adam(work: List[Dict], grad_scale: Scalar = 1.0, zero_grad: bool = False,
               stochastic_rounding: bool = False, ema_decay=None) -> None:
    """Adam update for a list of tensors in ONE launch.

    Each ``work`` item: ``p`` (fp32 master, or half/bf16 param), ``g`` (grad, any float dtype),
    ``m``/``v`` (fp32), optional ``p_half`` (16-bit copy to write), and scalars ``lr, beta1,
    beta2, eps, step, bias_correction, weight_decay``.  Gradients are divided by ``grad_scale``
    (python float or device scalar) inside the kernel; a device scalar that is non-finite or zero
    makes the whole update skip itself (overflowed gradients, see ``--deferred-overflow-check``).  ``zero_grad`` clears ``g`` in the same
    pass; ``stochastic_rounding`` applies to bf16 ``p_half`` outputs (Philox keyed by the CUDA
    generator's seed/offset so all data-parallel ranks round identically).  A work item may carry ``ema`` (fp32,
    same length as ``p``): with ``ema_decay`` given, ``ema -= (1 - decay) * (ema - p_new)`` happens in the same pass
    (reference: a separate three-kernel sweep, ``unicore/ema.py:44-60``).
    """
    if len(work) == 0:
        return
    tensors = [w["p"] for w in work]
    if use_native(*tensors):
        inv = None
        scale_f = 1.0
        if torch.is_tensor(grad_scale):
            inv = grad_scale.detach().float().reshape(1)  # kernel divides by *inv
        else:
            scale_f = float(grad_scale)
        native().multi_tensor_adam(
            [w["p"] for w in work], [w["g"] for w in work], [w["m"] for w in work], [w["v"] for w in work],
            [w.get("p_half") for w in work],
            [float(w["lr"]) for w in work], [float(w["beta1"]) for w in work], [float(w["beta2"]) for w in work],
            [float(w["eps"]) for w in work], [int(w["step"]) for w in work],
            [bool(w["bias_correction"]) for w in work], [float(w["weight_decay"]) for w in work],
            scale_f, inv, bool(zero_grad), bool(stochastic_rounding),
            [w.get("ema") for w in work] if ema_decay is not None else [], float(ema_decay or 0.0),
        )
        return
    if torch.is_tensor(grad_scale):
        gs = float(grad_scale)
        if not math.isfinite(gs) or gs == 0.0:  # same contract as the kernel: the update skips itself
            if zero_grad:
                for w in work:
                    w["g"].zero_()
            return
    inv_scale = (1.0 / grad_scale) if not torch.is_tensor(grad_scale) else grad_scale.reciprocal()
    for w in work:
        _adam_reference_math(w, inv_scale, zero_grad, stochastic_rounding, ema_decay)


# ------------------------------------------------------------------------------------------------
# stochastic rounding / EMA
# ------------------------------------------------------------------------------------------------
@torch.no_grad()
def fp32_to_bf16_sr(src: torch.Tensor, dst: torch.Tensor) -> None:
    """dst(bf16) = stochastic_round(src(fp32)): add 16 uniform random low bits, truncate."""
    if src.dtype != torch.float32 or dst.dtype != torch.bfloat16:
        raise TypeError("fp32_to_bf16_sr expects (float32, bfloat16)")
    if use_native(src, dst):
        native().fp32_to_bf16_sr(src.contiguous(), dst)
        return
    bits = src.contiguous().view(torch.int32)
    noise = torch.randint(0, 1 << 16, bits.shape, device=bits.device, dtype=torch.int32)
    finite = torch.isfinite(src)
    rounded = torch.where(finite, (bits + noise) & ~0xFFFF, bits & ~0xFFFF)
    dst.copy_(rounded.view(torch.float32))


@torch.no_grad()
def ema_update_(ema: torch.Tensor, param: torch.Tensor, decay: float) -> None:
    """``ema -= (1 - decay) * (ema - param)`` in one pass (reference: 3 kernels + a temporary)."""
    if use_native(ema, param) and ema.dtype == torch.float32 and param.dtype == torch.float32:
        native().ema_update(ema, param, float(decay))
        return
    ema.sub_((ema - param.to(ema.dtype)).mul_(1 - decay))
