"""``softmax_dropout``: ``dropout(softmax(input + mask + bias, dim=-1))`` with broadcast mask/bias.

Contract (reference ``unicore/modules/softmax_dropout.py:100-144`` + ``csrc/softmax_dropout``):
* works **in place** on ``input`` by default (the buffer ends up holding the softmax
  probabilities; the dropped-out result is returned);
* ``mask`` broadcasts as ``[..., 1|H, 1|Q, K]`` (row ``r`` of the flattened input uses mask row
  ``r // (rows / mask_rows)``); ``bias`` broadcasts over leading batch dims (row ``r`` uses bias
  row ``r % bias_rows``); anything else is pre-added in PyTorch;
* gradient flows to ``input`` and ``bias``.

sm_90a kernel (``csrc/attn/softmax_dropout.cu``): one warp per row with 128-bit loads, rows of any
length (dropout included for K > 1024, which the reference cannot fuse), current-stream launch,
and **no stored dropout mask**: keep/drop decisions are a pure function of
``(philox seed, offset, element index)`` and are regenerated in backward.
"""

import torch
import torch.nn.functional as F

from ._native import native, use_native


def _mask_plan(mask: torch.Tensor, x: torch.Tensor) -> bool:
    """True if ``mask`` fits the kernel's division-broadcast (else it must be pre-added)."""
    if mask.dtype != x.dtype or mask.dim() != x.dim() or mask.shape[-1] != x.shape[-1]:
        return False
    if x.dim() < 3:
        return False
    h_ok = mask.shape[-3] in (1, x.shape[-3])
    if not h_ok:
        return False
    if mask.shape[-3] == 1:
        if mask.shape[-2] != 1:
            return False
    elif mask.shape[-2] not in (1, x.shape[-2]):
        return False
    # leading dims must match exactly (division mapping assumes contiguous outer order)
    return tuple(mask.shape[:-3]) == tuple(x.shape[:-3])


def _bias_plan(bias: torch.Tensor, x: torch.Tensor) -> bool:
    """True if ``bias`` fits the kernel's modulo-broadcast."""
    if bias.dtype != x.dtype or bias.dim() != x.dim():
        return False
    if bias.shape[-1] != x.shape[-1] or bias.shape[-2] != x.shape[-2]:
        return False
    nd = x.dim()
    tail = 3 if nd > 3 else 2
    if nd > 3 and bias.shape[-3] != x.shape[-3]:
        return False
    # going outwards: once a dim is broadcast (1), all dims further out must be broadcast too
    inner_full = True
    for i in range(nd - tail - 1, -1, -1):
        if inner_full:
            if bias.shape[i] not in (1, x.shape[i]):
                return False
        elif bias.shape[i] != 1:
            return False
        inner_full = bias.shape[i] != 1 or x.shape[i] == 1
    return True


class _SoftmaxDropoutFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x3, mask3, bias3, p, training, in_place=True):
        out, probs, seed, offset = native().softmax_dropout_fwd(x3, mask3, bias3, float(p), bool(training), bool(in_place))
        ctx.p = float(p) if training else 0.0
        ctx.rng = (seed, offset)
        ctx.bias_rows = bias3.shape[0] if (bias3 is not None and bias3.requires_grad) else 0
        # the softmax probabilities: x3 itself when the kernel ran in place, else the kernel's own buffer
        ctx.save_for_backward(probs)
        return out

    @staticmethod
    def backward(ctx, dy):
        (probs,) = ctx.saved_tensors
        dy = dy.contiguous()
        if dy.data_ptr() == probs.data_ptr():
            dy = dy.clone()
        dx = native().softmax_dropout_bwd(dy, probs, ctx.p, ctx.rng[0], ctx.rng[1])
        return dx, None, _bias_grad(dx, ctx.bias_rows), None, None, None


def _bias_grad(dx3, bias_rows):
    """Gradient of a ``[bias_rows, Q, K]`` bias that was broadcast (modulo) over the rows of ``dx3``."""
    if bias_rows <= 0:
        return None
    if bias_rows == dx3.shape[0]:
        return dx3  # nothing was broadcast: the two gradients are the same tensor, no pass over it
    return dx3.view(-1, bias_rows, dx3.shape[-2], dx3.shape[-1]).sum(dim=0)


class _SoftmaxDropoutLogitsFn(torch.autograd.Function):
    """``z = x + mask + bias`` and ``dropout(softmax(z))`` from one kernel; ``z`` is an output (the pair
    representation handed to the next layer), its incoming gradient is folded into the backward kernel's store."""

    @staticmethod
    def forward(ctx, x3, mask3, bias3, p, training):
        out, logits, lse, seed, offset = native().softmax_dropout_logits_fwd(x3, mask3, bias3, float(p), bool(training))
        ctx.p = float(p) if training else 0.0
        ctx.rng = (seed, offset)
        ctx.bias_rows = bias3.shape[0] if (bias3 is not None and bias3.requires_grad) else 0
        ctx.save_for_backward(logits, lse)
        return out, logits

    @staticmethod
    def backward(ctx, dy, dlogits):
        logits, lse = ctx.saved_tensors
        if dy is None:
            dy = torch.zeros_like(logits)
        dx = native().softmax_dropout_logits_bwd(
            dy.contiguous(), logits, lse, None if dlogits is None else dlogits.contiguous(), ctx.p, ctx.rng[0], ctx.rng[1]
        )
        return dx, None, _bias_grad(dx, ctx.bias_rows), None, None


def _kernel_operands(input, mask, bias, may_overwrite):
    """Bring ``mask`` / ``bias`` into the kernel's 3-D broadcast forms (pre-adding whatever does not fit)."""
    if input.dim() == 2:
        input = input.unsqueeze(0)
        mask = mask.unsqueeze(0) if mask is not None and mask.dim() == 2 else mask
        bias = bias.unsqueeze(0) if bias is not None and bias.dim() == 2 else bias
    if mask is not None:
        if _mask_plan(mask, input):
            mask = mask.contiguous().view(-1, mask.shape[-2], mask.shape[-1])
        else:
            input = input.add_(mask) if may_overwrite and not input.requires_grad else input + mask
            mask = None
    if bias is not None:
        if _bias_plan(bias, input):
            bias = bias.contiguous().view(-1, bias.shape[-2], bias.shape[-1])
        else:
            input = input.add_(bias) if may_overwrite and not input.requires_grad else input + bias
            bias = None
    return input.view(-1, input.shape[-2], input.shape[-1]), mask, bias


def _kernel_eligible(input, mask, bias):
    return use_native(input, mask, bias) and input.dim() >= 2 and input.numel() > 0 and input.dtype in (
        torch.float16, torch.bfloat16, torch.float32
    )


def softmax_dropout(input, dropout_prob, is_training=True, mask=None, bias=None, inplace=True):
    """See module docstring. Returns a tensor shaped like ``input``."""
    input = input.contiguous()
    if _kernel_eligible(input, mask, bias):
        shape = input.shape
        x3, mask, bias = _kernel_operands(input, mask, bias, may_overwrite=inplace)
        # not in place (or a leaf that needs grad, which must not be overwritten): the kernel reads x and writes the
        # probabilities to its own buffer - no clone pass
        overwrite = inplace and not (x3.requires_grad and x3.is_leaf)
        out = _SoftmaxDropoutFn.apply(x3, mask, bias, dropout_prob, is_training, overwrite)
        return out.view(shape)
    if not inplace:
        input = input.clone()
    if mask is not None:
        input = input + mask
    if bias is not None:
        input = input + bias
    return F.dropout(F.softmax(input, dim=-1), p=dropout_prob, training=is_training)


def softmax_dropout_with_logits(input, dropout_prob, is_training=True, mask=None, bias=None):
    """``(dropout(softmax(z)), z)`` with ``z = input + mask + bias`` materialised once.

    The ``return_attn=True`` formulation of the reference (``unicore/modules/multihead_attention.py:98-103``:
    ``attn_weights += attn_bias`` then ``softmax_dropout(..., inplace=False)``) spends a pass on the bias add,
    a clone, and - in backward - an add of the two gradients that meet at ``z``.  Here ``z`` is a by-product
    of the softmax kernel, no probability tensor is kept (backward rebuilds it from ``z`` and the row
    log-sum-exp) and the gradient arriving for ``z`` is added inside the backward kernel.  ``input`` is not
    modified.
    """
    input = input.contiguous()
    if _kernel_eligible(input, mask, bias):
        shape = input.shape
        x3, mask, bias = _kernel_operands(input, mask, bias, may_overwrite=False)
        out, logits = _SoftmaxDropoutLogitsFn.apply(x3, mask, bias, dropout_prob, is_training)
        return out.view(shape), logits.view(shape)
    logits = input
    if mask is not None:
        logits = logits + mask
    if bias is not None:
        logits = logits + bias
    return F.dropout(F.softmax(logits, dim=-1), p=dropout_prob, training=is_training), logits
