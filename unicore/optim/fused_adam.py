"""FusedAdam: ``torch.optim.Optimizer`` whose ``step`` is a single multi-tensor kernel launch.

Math (reference kernel ``csrc/adam/adam_kernel.cu:38-78`` / wrapper ``optim/fused_adam.py:20-145``):
``step_size = lr*sqrt(1-b2^t)/(1-b1^t)`` (or ``lr`` without bias correction), ``g = grad/scale``,
``m = b1 m + (1-b1) g``, ``v = b2 v + (1-b2) g^2``, ``p = p (1 - step_size*wd) - step_size m/(sqrt(v)+eps)``.
Note the decay is scaled by the *bias-corrected* step size (differs from the python ``Adam``).

GPU design: all parameters of all groups go to ``unicore.ops.fused_adam`` as tensor lists with
per-tensor hyper-parameters, i.e. one launch per step irrespective of the number of tensors; the
kernel uses 128-bit accesses, accepts fp32 or half/bf16 params+grads with fp32 moments, and can
emit a 16-bit copy of the updated parameter (optionally stochastically rounded) and zero the
gradient in the same pass - see ``csrc/optim/adam.cu``.
"""
import torch


def get_fused_adam_class():
    """Return ``FusedAdam`` when the sm_90a extension is importable, else ``None``."""
    from unicore import ops

    return FusedAdam if ops.HAS_CUDA_EXT else None


class FusedAdam(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, bias_correction=True, betas=(0.9, 0.999), eps=1e-8,
                 weight_decay=0.0, amsgrad=False):
        if amsgrad:
            raise RuntimeError("FusedAdam does not support the AMSGrad variant.")
        defaults = dict(lr=lr, bias_correction=bias_correction, betas=betas, eps=eps, weight_decay=weight_decay)
        super().__init__(params, defaults)

    @property
    def supports_memory_efficient_fp16(self):
        return True

    @property
    def supports_flat_params(self):
        return True

    @property
    def supports_step_with_scale(self):
        return True

    def _state_for(self, p):
        state = self.state[p]
        if len(state) == 0:
            state["step"] = 0
            state["exp_avg"] = torch.zeros_like(p.data, dtype=torch.float)
            state["exp_avg_sq"] = torch.zeros_like(p.data, dtype=torch.float)
        elif state["exp_avg"].dtype != torch.float or state["exp_avg"].device != p.device:
            state["exp_avg"] = state["exp_avg"].to(device=p.device, dtype=torch.float)
            state["exp_avg_sq"] = state["exp_avg_sq"].to(device=p.device, dtype=torch.float)
        return state

    @torch.no_grad()
    def step(self, closure=None, scale=1.0):
        """``scale`` divides every gradient inside the kernel (loss-scale / clip folding)."""
        from unicore import ops

        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        work = []
        for group in self.param_groups:
            beta1, beta2 = group["betas"]
            for p in group["params"]:
                if p.grad is None:
                    continue
                if p.grad.is_sparse:
                    raise RuntimeError("FusedAdam does not support sparse gradients, please consider SparseAdam instead")
                state = self._state_for(p)
                state["step"] += 1
                work.append(dict(
                    p=p.data, g=p.grad.data, m=state["exp_avg"], v=state["exp_avg_sq"],
                    lr=group["lr"], beta1=beta1, beta2=beta2, eps=group["eps"], step=state["step"],
                    bias_correction=bool(group.get("bias_correction", True)), weight_decay=group["weight_decay"],
                ))
        if work:
            ops.fused_adam(work, grad_scale=scale)
        return loss
