"""Parameter gradients written straight into the optimizer's flat gradient arena.

With flat arenas (``unicore/optim/fp16_optimizer.py``) every parameter's ``.grad`` is a view of one 16-bit buffer.
Plain autograd still computes each parameter gradient into a temporary and then ADDS it to that view with one more
kernel per parameter (``AccumulateGrad``): for BERT-base that is ~155 extra launches and three passes over the gradient
bytes per step.

The backward kernels of this framework can accumulate in place instead: the weight-gradient GEMM runs with beta = 1 on
the arena view (``addmm_``), the bias / LayerNorm column-sum finalisers add to the view.  A custom autograd Function
"claims" a parameter in forward, writes into ``param.grad`` in backward and returns ``None`` for that input, so
autograd has nothing left to accumulate.

Because no ``AccumulateGrad`` node runs for such a parameter, gradient-ready hooks would not fire.  Engines that
schedule communication from those hooks register ``on_written`` here instead; a parameter counts as ready when every
claim of the current step has been written (a parameter used twice is claimed twice).  Direct sinks are switched on by
the trainer only for engines that cooperate (single process, ``--ddp-backend b200``); torch DDP keeps plain autograd.
"""
from typing import Callable, Iterable, Optional

import torch


def enable(params: Iterable[torch.nn.Parameter], on_written: Optional[Callable] = None) -> None:
    for p in params:
        p._ub_direct_grad = True
        p._ub_pending = 0
        p._ub_grad_written = on_written


def disable(params: Iterable[torch.nn.Parameter]) -> None:
    for p in params:
        p._ub_direct_grad = False
        p._ub_pending = 0
        p._ub_grad_written = None


def reset(params: Iterable[torch.nn.Parameter]) -> None:
    """New update: forget claims whose backward never ran (a forward without backward, an aborted step)."""
    for p in params:
        p._ub_pending = 0


def wants(p) -> bool:
    """Is ``p`` a parameter whose gradient may be accumulated in place?  (Grad mode is the caller's business: inside
    ``autograd.Function.forward`` it is always off - use ``ctx.needs_input_grad`` there.)"""
    return p is not None and getattr(p, "_ub_direct_grad", False) and p.requires_grad and p.grad is not None


def claim(p, needed: bool = True):
    """Forward (``needed`` = ``ctx.needs_input_grad[i]``): returns ``p`` when its gradient will be written in place by
    this node's backward, else ``None``."""
    if not needed or not wants(p):
        return None
    p._ub_pending += 1
    return p


def sink(p):
    """Backward: the tensor to accumulate into (``None`` when ``p`` was not claimed)."""
    return None if p is None else p.grad


def done(p) -> None:
    """Backward: this node's contribution to ``p.grad`` has been enqueued."""
    if p is None:
        return
    p._ub_pending -= 1
    if p._ub_pending <= 0:
        p._ub_pending = 0
        callback = getattr(p, "_ub_grad_written", None)
        if callback is not None:
            callback(p)
