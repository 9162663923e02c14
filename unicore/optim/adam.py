"""Adam (decoupled weight decay, i.e. AdamW-style) and its CLI wrapper.

``UnicoreAdam`` uses ``FusedAdam`` (one multi-tensor sm_90a launch per step) when the CUDA
extension is loaded and the params are on a GPU, else the pure-PyTorch ``Adam`` below.
Parity: reference ``unicore/optim/adam.py:22-204`` (flags ``--adam-betas``, ``--adam-eps``,
``--weight-decay``; python Adam decays with ``lr * wd``; amsgrad supported).
"""
import ast
import logging
import math
from collections.abc import Collection

import torch
import torch.optim

from unicore.optim import UnicoreOptimizer, register_optimizer
from unicore.optim.fused_adam import get_fused_adam_class

logger = logging.getLogger(__name__)


@register_optimizer("adam")
class UnicoreAdam(UnicoreOptimizer):
    def __init__(self, args, params):
        super().__init__(args)
        from unicore_b200.parallel import reference_tail_requested

        fused_cls = get_fused_adam_class()
        use_fused = (
            not getattr(args, "use_old_adam", False)
            and fused_cls is not None
            and torch.cuda.is_available()
            and not getattr(args, "cpu", False)
        )
        if reference_tail_requested() and not getattr(args, "use_old_adam", False):
            from unicore.optim.fused_adam import FusedAdam

            fused_cls, use_fused = FusedAdam, True  # (its kernel call has a PyTorch fallback)
        if use_fused:
            logger.info("using FusedAdam (sm_90a multi-tensor kernel)")
            self._optimizer = fused_cls(params, **self.optimizer_config)
        else:
            self._optimizer = Adam(params, **self.optimizer_config)

    @staticmethod
    def add_args(parser):
        parser.add_argument("--adam-betas", default="(0.9, 0.999)", metavar="B", help="betas for Adam optimizer")
        parser.add_argument("--adam-eps", type=float, default=1e-8, metavar="D", help="epsilon for Adam optimizer")
        parser.add_argument("--weight-decay", "--wd", default=0.0, type=float, metavar="WD", help="weight decay")

    @property
    def optimizer_config(self):
        lr = self.args.lr[0] if isinstance(self.args.lr, Collection) else self.args.lr
        betas = self.args.adam_betas
        if isinstance(betas, str):
            betas = ast.literal_eval(betas)
        return {"lr": lr, "betas": tuple(betas), "eps": self.args.adam_eps, "weight_decay": self.args.weight_decay}


class Adam(torch.optim.Optimizer):
    """Reference-semantics Adam in plain PyTorch (fp32 state regardless of param dtype)."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=amsgrad))

    @property
    def supports_memory_efficient_fp16(self):
        return True

    @property
    def supports_flat_params(self):
        return True

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            beta1, beta2 = group["betas"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                grad = p.grad
                if grad.is_sparse:
                    raise RuntimeError("Adam does not support sparse gradients, please consider SparseAdam instead")
                grad = grad.float() if grad.dtype != torch.float32 else grad
                work = p.data.float() if p.dtype != torch.float32 else p.data
                state = self.state[p]
                if len(state) == 0:
                    state["step"] = 0
                    state["exp_avg"] = torch.zeros_like(work)
                    state["exp_avg_sq"] = torch.zeros_like(work)
                    if group.get("amsgrad", False):
                        state["max_exp_avg_sq"] = torch.zeros_like(work)
                else:
                    for key in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq"):
                        if key in state:
                            state[key] = state[key].to(work)
                state["step"] += 1
                m, v = state["exp_avg"], state["exp_avg_sq"]
                m.mul_(beta1).add_(grad, alpha=1 - beta1)
                v.mul_(beta2).addcmul_(grad, grad, value=1 - beta2)
                if group.get("amsgrad", False):
                    vmax = state["max_exp_avg_sq"]
                    torch.max(vmax, v, out=vmax)
                    denom = vmax.sqrt().add_(group["eps"])
                else:
                    denom = v.sqrt().add_(group["eps"])
                correction1 = 1 - beta1 ** state["step"]
                correction2 = 1 - beta2 ** state["step"]
                step_size = group["lr"] * math.sqrt(correction2) / correction1
                if group["weight_decay"] != 0:
                    work.add_(work, alpha=-group["weight_decay"] * group["lr"])
                work.addcdiv_(m, denom, value=-step_size)
                if work.data_ptr() != p.data.data_ptr():
                    p.data.copy_(work)
        return loss
