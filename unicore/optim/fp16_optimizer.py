"""Mixed-precision optimisation: 16-bit model/grads in flat arenas + fp32 master weights.

Layout contract (checkpoint compatible with reference ``unicore/optim/fp16_optimizer.py:16-136``):
parameters are split into a decay and a no-decay group (``separate_decay_params``); inside a
group they are bucketed by dtype in first-seen order and concatenated in encounter order, each
tensor padded to an even element count.  Every model parameter's ``.data`` and ``.grad`` become
views into the group's flat 16-bit buffers; one flat fp32 master ``nn.Parameter`` per group is
what the inner optimizer (and therefore ``last_optimizer_state``) sees.

Step semantics follow ``_FP16OptimizerMixin`` (reference ``:139-308``): loss is multiplied by the
loss scale, every later gradient scaling (1/loss_scale, world/sample_size, clipping) is folded
into the scalar ``_multiply_factor`` and applied *inside* the optimizer kernel.

Fused tail (CUDA + FusedAdam): the reference runs
``grad16->grad32 copy, L2 norm, Adam, param32->param16 copy, zero_grad(2 memsets)`` as separate
passes (~86 B/param incl. EMA).  Here the norm (+ non-finite detection) is computed directly from
the 16-bit flat gradient (2 B/param) and ONE kernel then does unscale/clip + Adam on the fp32
master + 16-bit write-back (optionally stochastically rounded) + gradient zeroing (30 B/param);
no fp32 gradient buffer exists at all in that mode.  Bitwise result is identical to the unfused
path because fp16/bf16 -> fp32 conversion is exact and all math is fp32.
"""
import logging
from collections import OrderedDict
from typing import Callable, Optional

import torch

from unicore import utils

from .dynamic_loss_scaler import DynamicLossScaler
from .unicore_optimizer import UnicoreOptimizer

logger = logging.getLogger(__name__)


# ------------------------------------------------------------------------------------------------
# parameter partition + flat layout
# ------------------------------------------------------------------------------------------------
def separate_decay_params(args, params):
    """Split ``[(name, param), ...]`` into ``[{decay}, {no_decay, weight_decay: 0}]`` groups.

    Exempt from decay: names ending in ``.bias``, 1-D params, names containing any entry of
    ``--no-weight-decay-names``.  A single group when ``weight_decay <= 0``.
    """
    trainable = [(n, p) for n, p in params if p.requires_grad]
    if getattr(args, "weight_decay", 0.0) <= 0:
        return [{"params": [p for _, p in trainable]}]
    names = getattr(args, "no_weight_decay_names", "") or ""
    exempt_substrings = [s for s in names.split(",") if s] if names else []

    def exempt(name, p):
        return name.endswith(".bias") or p.ndim == 1 or any(s in name for s in exempt_substrings)

    decay = [p for n, p in trainable if not exempt(n, p)]
    no_decay = [p for n, p in trainable if exempt(n, p)]
    groups = []
    if decay:
        groups.append({"params": decay})
    if no_decay:
        groups.append({"params": no_decay, "weight_decay": 0.0})
    return groups


def check_param_device(params):
    devices = {p.device for p in params}
    if len(devices) > 1:
        raise ValueError("all parameters of a group must live on one device, got {}".format(devices))


def pad_numel(numel, multiplier=2):
    return -(-numel // multiplier) * multiplier


def flatten_orders(params):
    """Group params by dtype (first-seen order). Returns (dtype->params, dtype order, padded size)."""
    by_dtype: "OrderedDict[torch.dtype, list]" = OrderedDict()
    total = 0
    for p in params:
        by_dtype.setdefault(p.dtype, []).append(p)
        total += pad_numel(p.data.numel())
    return by_dtype, list(by_dtype.keys()), total


def _slots(params):
    """Yield ``(param, offset, numel)`` for the padded concatenation of ``params``."""
    offset = 0
    for p in params:
        n = p.data.numel()
        yield p, offset, n
        offset += pad_numel(n)


@torch.no_grad()
def flatten_parameters(params, grad_alloc: Optional[Callable[[int, torch.dtype, torch.device], torch.Tensor]] = None,
                       param_alloc: Optional[Callable[[int, torch.dtype, torch.device], Optional[torch.Tensor]]] = None):
    """Re-point ``p.data`` / ``p.grad`` of every param into one flat buffer per dtype.

    ``grad_alloc(numel, dtype, device)`` lets a communication engine provide the gradient buffer
    (e.g. NVLink peer-mapped symmetric memory) so gradients are produced in place where the
    reduction kernels read them - no staging copies.  ``param_alloc`` does the same for the flat
    parameter buffer (it may return ``None`` to decline): the sharded optimizer step stores new
    parameters straight into every rank's arena.
    Returns the flat ``nn.Parameter`` per dtype (with ``.grad`` = the flat grad buffer).
    """
    by_dtype, order, _ = flatten_orders(params)
    flats = []
    for dtype in order:
        members = by_dtype[dtype]
        total = sum(pad_numel(p.data.numel()) for p in members)
        device = members[0].device
        flat = param_alloc(total, dtype, device) if param_alloc is not None else None
        if flat is None:
            flat = torch.zeros(total, dtype=dtype, device=device)
        else:
            flat.zero_()
        for p, off, n in _slots(members):
            flat[off:off + n].copy_(p.data.reshape(-1))
            p.data = flat[off:off + n].view(p.shape)
        flat = torch.nn.Parameter(flat)
        if grad_alloc is not None:
            gbuf = grad_alloc(total, dtype, device)
            gbuf.zero_()
        else:
            gbuf = torch.zeros(total, dtype=dtype, device=device)
        flat.grad = gbuf
        for p, off, n in _slots(members):
            p.grad = gbuf[off:off + n].view(p.shape)
        flats.append(flat)
    if torch.cuda.is_available():
        torch.cuda.empty_cache()
    return flats


@torch.no_grad()
def flatten_parameters_fp32(params, set_to_param=False, set_grad=True):
    """One flat fp32 copy of ``params`` (dtype-major, same padding). With ``set_to_param`` the
    params themselves become views of it (used by the EMA shadow model)."""
    by_dtype, order, total = flatten_orders(params)
    # the storage is a whole number of 32-byte groups (8 floats): kernels that walk the arena in 8-element vectors may
    # touch the slack behind the last parameter
    flat = torch.zeros(pad_numel(total, 8), dtype=torch.float32, device=params[0].device)[:total]
    ordered = [p for dtype in order for p in by_dtype[dtype]]
    for p, off, n in _slots(ordered):
        flat[off:off + n].copy_(p.data.reshape(-1))
        if set_to_param:
            p.data = flat[off:off + n].view(p.shape)
            p.grad = None
    flat = torch.nn.Parameter(flat)
    if set_grad:
        flat.grad = torch.zeros_like(flat)
    if torch.cuda.is_available():
        torch.cuda.empty_cache()
    return flat


def get_fp16_params(args, params, grad_alloc=None, fp32_grads=True, param_alloc=None):
    """Build the per-group flat 16-bit params (+grads) and fp32 masters."""
    fp16_groups, fp32_groups = [], []
    for group in separate_decay_params(args, params):
        members = group["params"]
        check_param_device(members)
        flats16 = flatten_parameters(members, grad_alloc=grad_alloc, param_alloc=param_alloc)
        master = flatten_parameters_fp32(members, set_grad=fp32_grads)
        fp16_groups.append({"params": flats16})
        group = dict(group)
        group["params"] = [master]
        fp32_groups.append(group)
    return fp16_groups, fp32_groups


# ------------------------------------------------------------------------------------------------
# mixed-precision wrapper
# ------------------------------------------------------------------------------------------------
class _FP16OptimizerMixin(object):
    def __init__(self, args, **kwargs):
        super().__init__(args, **kwargs)
        self._multiply_factor = 1.0
        self.bf16_sr = getattr(args, "bf16_sr", False)
        self._grads_zeroed = False

    # -- fused tail (--ddp-backend b200): reduce-scatter tail + norm/stat exchange + clip + Adam(+EMA) on the shard +
    #    parameter all-gather in ONE kernel, see unicore_b200/parallel/fused_tail.py ------------------------------------
    _tail = None
    _tail_engine = None

    def enable_fused_tail(self, engine, tail) -> bool:
        """``tail`` (``FusedTail``) owns the shard geometry; ``engine.run_tail(**kw)`` launches the kernel behind the
        step's bucket kernels.  From here on the fp32 master weights and the Adam moments of this rank are COMPACT
        shards (1/world of the state); ``state_dict()`` re-assembles the reference layout with collectives."""
        if not self._fused or any(len(g["params"]) != 1 for g in self.fp16_params):
            return False
        inner = self.fp32_optimizer.optimizer
        if not hasattr(inner, "_state_for"):
            return False
        self._tail, self._tail_engine = tail, engine
        self._tail_full_numel = []
        for gi, (_flats16, master) in enumerate(self._pairs()):
            self._tail_full_numel.append(master.numel())
            state = inner.state.get(master, None)
            moments = None
            if state is not None and "exp_avg" in state:
                moments = (tail.to_compact(state["exp_avg"], gi), tail.to_compact(state["exp_avg_sq"], gi))
            master.data = tail.to_compact(master.data, gi)
            master.grad = None
            if moments is not None:
                state["exp_avg"], state["exp_avg_sq"] = moments
        self._tail_max_norm = 0.0
        self._tail_stats = None
        self._tail_stats_len = 0
        self._tail_denom_index = -1
        self._ema_flats, self._ema_decay = None, 0.0
        return True

    @property
    def uses_fused_tail(self) -> bool:
        return self._tail is not None

    def attach_ema(self, ema_flats, decay: float) -> bool:
        """Fused tail only: the EMA update (``ema -= (1-d)(ema - w)`` on the fp32 master) moves into the kernel.
        ``ema_flats[g]``: the full-length fp32 EMA arena of group g; a rank keeps ITS slices current."""
        if self._tail is None:
            return False
        self._ema_flats, self._ema_decay = list(ema_flats), float(decay)
        return True

    def set_step_stats(self, values, denom_index: int = -1) -> None:
        """Fused tail only: ``values`` (<= 64 numbers / device scalars) are summed over the ranks INSIDE the tail kernel;
        the gradients are divided by sum number ``denom_index`` (the sample size).  Read them with ``step_stats()``."""
        self._tail_stats, self._tail_denom_index = values, int(denom_index)
        self._tail_stats_len = int(values.numel()) if torch.is_tensor(values) else len(values)

    def step_stats(self):
        """fp64 device vector with the rank sums of the statistics handed to ``set_step_stats`` (valid after ``step``;
        a copy - the kernel's output buffer is overwritten by the next update)."""
        return self._tail.stats_dst[:self._tail_stats_len].clone()

    def step_grad_norm(self):
        """The gradient norm the last ``step`` computed on the device (a copy of the tail's state slot)."""
        return self._tail.state[0].clone()

    def attach_replicated_ema(self, ema_flats, decay: float) -> bool:
        """Replicated fused Adam: the EMA update rides in the Adam kernel's pass over the master weights instead of
        being a separate sweep (reference ``unicore/ema.py:44-60``)."""
        if self._tail is not None or not self._fused or any(len(g["params"]) != 1 for g in self.fp16_params):
            return False
        flats = list(ema_flats)
        if len(flats) != len(self.fp32_params) or any(
                f.numel() != g["params"][0].numel() for f, g in zip(flats, self.fp32_params)):
            return False
        self._replicated_ema = (flats, float(decay))
        return True

    @torch.no_grad()
    def gather_ema(self) -> None:
        """COLLECTIVE (fused tail): merge the ranks' slices of the EMA arenas so that every rank holds all of it."""
        if self._tail is None or self._ema_flats is None:
            return
        for gi, flat in enumerate(self._ema_flats):
            self._tail.scatter_owned_(flat.data, gi)

    @torch.no_grad()
    def sync_master_from_params(self) -> None:
        """Rebuild the fp32 master weights from the 16-bit model weights (after a checkpoint load)."""
        for gi, (flats16, master) in enumerate(self._pairs()):
            if self._tail is not None:
                master.data.copy_(self._tail.to_compact(flats16[0].data.float(), gi))
            else:
                offset = 0
                for f in flats16:
                    master.data[offset:offset + f.numel()].copy_(f.data)
                    offset += f.numel()

    @torch.no_grad()
    def consolidate_state(self) -> None:
        """COLLECTIVE - call on EVERY rank before the master rank takes ``state_dict()`` (``checkpoint_utils`` does):
        with the fused tail the ranks' shards of the Adam moments are assembled into the reference's full-length layout
        (kept until the next update) and the EMA slices are merged.  No-op for the replicated optimizers."""
        if self._tail is None:
            return
        self.resolve_pending_overflow()
        inner = self.fp32_optimizer.optimizer
        self._consolidated = {}
        for gi, (_f, master) in enumerate(self._pairs()):
            state = inner.state.get(master, None)
            if not state or "exp_avg" not in state:
                continue
            n = self._tail_full_numel[gi]
            self._consolidated[gi] = tuple(self._tail.to_full(state[name], gi, n) for name in ("exp_avg", "exp_avg_sq"))
        self.gather_ema()

    def _tail_full_state(self, state):
        """The inner optimizer's state dict with the full-length (reference layout) moments of ``consolidate_state``."""
        inner = self.fp32_optimizer.optimizer
        index = {id(master): gi for gi, (_f, master) in enumerate(self._pairs())}
        packed = state["state"]
        # torch packs state by parameter index in group order: one master per group, in order
        order = [p for g in inner.param_groups for p in g["params"]]
        full = getattr(self, "_consolidated", None)
        for key, p in enumerate(order):
            if key in packed and id(p) in index and "exp_avg" in packed[key]:
                gi = index[id(p)]
                if full is None or gi not in full:
                    raise RuntimeError("sharded optimizer state: call consolidate_state() on every rank before state_dict()")
                entry = dict(packed[key])
                entry["exp_avg"], entry["exp_avg_sq"] = full[gi]
                packed[key] = entry
        return state

    def _tail_reshard_loaded_state(self):
        inner = self.fp32_optimizer.optimizer
        for gi, (_f, master) in enumerate(self._pairs()):
            state = inner.state.get(master, None)
            if not state:
                continue
            for name in ("exp_avg", "exp_avg_sq"):
                t = state.get(name, None)
                if torch.is_tensor(t) and t.numel() != master.numel():
                    state[name] = self._tail.to_compact(t.to(device=master.device, dtype=torch.float32), gi)

    # -- state ----------------------------------------------------------------------------------
    def state_dict(self):
        """Reference schema (``unicore/optim/fp16_optimizer.py:163-178``).  With the fused tail the moments come from the
        preceding ``consolidate_state()`` (a collective that every rank runs; only the master goes on to save)."""
        self.resolve_pending_overflow()
        state = self.fp32_optimizer.state_dict()
        if self._tail is not None:
            state = self._tail_full_state(state)
        if self.scaler is not None:
            state["loss_scale"] = self.scaler.loss_scale
        return state

    def load_state_dict(self, state_dict, optimizer_overrides=None):
        if "loss_scale" in state_dict and self.scaler is not None:
            self.scaler.loss_scale = state_dict["loss_scale"]
        self.fp32_optimizer.load_state_dict(state_dict, optimizer_overrides)
        if self._tail is not None:
            self._tail_reshard_loaded_state()

    # -- backward -------------------------------------------------------------------------------
    def backward(self, loss):
        """Scale the loss (fp16 only) and back-propagate; grads accumulate in the flat arena."""
        # deferred overflow check: the previous update's gradient norm has long arrived on the host by now;
        # the loss scale must be settled before this loss is scaled
        self.resolve_pending_overflow()
        if self.scaler is not None:
            loss = self.scaler.scale(loss)
        loss.backward()
        self._needs_sync = True
        self._grads_zeroed = False

    # -- grad/param synchronisation between the 16-bit arena and the fp32 master ----------------------
    def _pairs(self):
        for g16, g32 in zip(self.fp16_params, self.fp32_params):
            yield g16["params"], g32["params"][0]

    def _sync_fp16_grads_to_fp32(self):
        if not self._needs_sync or self._fused:
            self._needs_sync = False
            return
        for flats16, master in self._pairs():
            offset = 0
            for f in flats16:
                n = f.numel()
                master.grad.data[offset:offset + n].copy_(f.grad.data)
                offset += n
        self._needs_sync = False

    def _add_fp16_grads_to_fp32(self, mul=0.0):
        """master.grad = mul * master.grad + grad16 (per-sample clipping accumulation)."""
        for flats16, master in self._pairs():
            offset = 0
            for f in flats16:
                n = f.numel()
                seg = master.grad.data[offset:offset + n]
                seg.mul_(mul).add_(f.grad.data.float())
                f.grad.zero_()
                offset += n
        self._needs_sync = False

    def _sync_fp32_params_to_fp16(self):
        for flats16, master in self._pairs():
            offset = 0
            for f in flats16:
                n = f.numel()
                src = master.data[offset:offset + n]
                if self.bf16_sr and f.dtype == torch.bfloat16:
                    utils.fp32_to_bf16_sr(src, f.data)
                else:
                    f.data.copy_(src)
                offset += n

    def _unscale_grads(self):
        self._sync_fp16_grads_to_fp32()
        factor = self._multiply_factor
        if torch.is_tensor(factor) or factor != 1.0:
            self.fp32_optimizer.multiply_grads(factor)
            self._multiply_factor = 1.0

    def multiply_grads(self, c):
        """Deferred: only the scalar factor changes, no kernel runs (applied inside ``step``)."""
        self._multiply_factor = self._multiply_factor * c

    def per_sample_clip_grad_norm(self, max_norm, aggregate_norm_fn=None):
        """Clip the current micro-batch's grads to ``max_norm`` and accumulate them in fp32."""
        if max_norm <= 0.0:
            return 0.0
        if self._fused:
            raise RuntimeError("--per-sample-clip-norm requires the unfused optimizer path")
        all_flats = [f for g in self.fp16_params for f in g["params"]]
        grad_norm = self._multiply_factor * utils.multi_tensor_total_norm([f.grad for f in all_flats])
        if aggregate_norm_fn is not None:
            grad_norm = aggregate_norm_fn(grad_norm)
        coef = (max_norm / (grad_norm + 1e-6)).clamp_(max=1.0) if torch.is_tensor(grad_norm) \
            else min(1.0, max_norm / (grad_norm + 1e-6))
        for f in all_flats:
            f.grad.mul_(coef.to(f.grad.dtype) if torch.is_tensor(coef) else coef)
        self._add_fp16_grads_to_fp32(mul=1.0 if self._has_accumulated else 0.0)
        self._has_accumulated = True
        return grad_norm

    # -- norm / clip ----------------------------------------------------------------------------
    def set_external_grad_sq_norm(self, fn) -> None:
        """``fn() -> squared L2 norm of the flat gradients (device scalar) or None``: the NVLink all-reduce kernels
        accumulate it while they reduce, which saves the separate norm pass over the arena."""
        self._external_sq_norm = fn

    def _raw_grad_norm(self) -> torch.Tensor:
        """L2 norm of the (still scaled) gradients as an fp32 device scalar."""
        fn = getattr(self, "_external_sq_norm", None)
        if fn is not None and self._fused:
            sq = fn()
            if sq is not None:
                return sq.float().sqrt()
        if self._fused:
            grads = [f.grad for g in self.fp16_params for f in g["params"]]
        else:
            self._sync_fp16_grads_to_fp32()
            grads = [g["params"][0].grad for g in self.fp32_params]
        return utils.multi_tensor_total_norm(grads)

    def clip_grad_norm(self, max_norm, aggregate_norm_fn=None):
        """Fold clipping into ``_multiply_factor``; returns the un-scaled, pre-clip grad norm."""
        if self._tail is not None:
            # norm, clip coefficient and overflow decision are taken inside the tail kernel; the returned device scalar
            # is filled in by ``step()`` (a "future": consumers read it after the update was launched)
            self._tail_max_norm = float(max_norm)
            return self._tail.state[0]
        raw = self._raw_grad_norm()
        grad_norm = self._multiply_factor * raw
        if aggregate_norm_fn is not None:
            grad_norm = aggregate_norm_fn(grad_norm)
        if self.scaler is not None and self._deferred_overflow_active(grad_norm):
            # no host read here: the clip coefficient stays on the device, the fused update skips itself if the
            # norm is not finite, and the scaler is told before the next backward (resolve_pending_overflow)
            self.resolve_pending_overflow()
            factor = self._multiply_factor
            if max_norm > 0.0:
                # fp16 path of the reference: ``if grad_norm > max_norm: factor *= max_norm / grad_norm`` (no epsilon)
                factor = factor * torch.where(grad_norm > max_norm, max_norm / grad_norm, torch.ones_like(grad_norm))
            factor = torch.as_tensor(factor, dtype=torch.float32, device=grad_norm.device)
            self._multiply_factor = factor
            self._device_grad_scale = torch.where(
                torch.isfinite(grad_norm), factor.reciprocal(), torch.full_like(factor, float("inf"))
            )
            self._pending_norm = utils.AsyncHostRead(grad_norm)
        elif self.scaler is not None:
            # ONE host read per step: needed for the overflow decision (skip / rescale)
            norm_host = float(utils.item(grad_norm))
            # downstream consumers (consistency check, gnorm/clip meters) get the host copy: no further
            # device reads or tiny kernels between this point and the optimizer launch
            grad_norm = torch.tensor(norm_host, dtype=torch.float32)
            if 0.0 < max_norm < norm_host:
                self._multiply_factor = self._multiply_factor * (max_norm / norm_host)
            self.scaler.check_overflow(norm_host)
        elif max_norm > 0.0:
            clip_coef = (max_norm / (grad_norm + 1e-6)).clamp_(max=1.0)
            self._multiply_factor = self._multiply_factor * clip_coef
        return grad_norm

    # -- deferred overflow check ---------------------------------------------------------------------
    def _deferred_overflow_active(self, grad_norm) -> bool:
        return (
            getattr(self, "_fused", False)
            and getattr(self.args, "deferred_overflow_check", False)
            and torch.is_tensor(grad_norm)
            and grad_norm.is_cuda
        )

    def add_late_overflow_handler(self, fn) -> None:
        """``fn(message)`` is called when an overflow is discovered after its update was already launched
        (and skipped on the device); the trainer uses it to take back the update count."""
        if not hasattr(self, "_late_overflow_handlers"):
            self._late_overflow_handlers = []
        self._late_overflow_handlers.append(fn)

    def resolve_pending_overflow(self) -> None:
        """Settle the update that was launched last: tell the loss scaler (exactly ONE tick per update: ``update()`` for a
        finite norm, ``check_overflow()`` otherwise) and take back the optimistic bookkeeping of a skipped update."""
        pending = getattr(self, "_pending_norm", None)
        if pending is None:
            return
        self._pending_norm = None
        value = pending.get()
        if self._tail is not None:  # the tail's state vector {grad_norm, multiplier, overflow, sum of squares}
            norm_host = float(value[0]) if float(value[2]) == 0.0 else float("inf")
        else:
            norm_host = float(value)
        self._last_grad_norm = norm_host
        if self.scaler is None:
            if norm_host != norm_host or abs(norm_host) == float("inf"):
                self._undo_skipped_update("gradients are Nan/Inf")
                raise FloatingPointError("gradients are Nan/Inf")
            return
        try:
            self.scaler.check_overflow(norm_host)
        except OverflowError as exc:
            self._undo_skipped_update(str(exc))
            return
        self.scaler.update()

    def _undo_skipped_update(self, message: str) -> None:
        # the device skipped that update (non-finite divisor): undo the optimistic host bookkeeping
        inner = self.fp32_optimizer.optimizer
        for _, master in self._pairs():
            state = inner.state.get(master, None)
            if state is not None and state.get("step", 0) > 0:
                state["step"] -= 1
        if getattr(self, "_grads_zeroed", False) and not self._has_accumulated and self.scaler is not None:
            self._multiply_factor = 1.0 / float(self.scaler.loss_scale)
        for fn in getattr(self, "_late_overflow_handlers", []):
            fn(message)

    # -- update ---------------------------------------------------------------------------------
    def step(self, closure=None, groups=None):
        if self._fused:
            self._fused_step()
        else:
            self._sync_fp16_grads_to_fp32()
            if getattr(self, "supports_step_with_scale", False):
                factor = self._multiply_factor
                scale = (1.0 / factor) if not torch.is_tensor(factor) else factor.reciprocal()
                self.fp32_optimizer.step(closure, scale=scale, groups=groups)
            else:
                self._unscale_grads()
                self.fp32_optimizer.step(closure, groups=groups)
            self._sync_fp32_params_to_fp16()
        if self.scaler is not None and getattr(self, "_pending_norm", None) is None:
            self.scaler.update()  # (deferred / tail mode: the scaler is ticked when the outcome is known)
        self._has_accumulated = False

    def _fused_step(self):
        """unscale+clip, Adam on fp32 master, 16-bit write-back (+SR) and grad zeroing: one launch."""
        from unicore import ops

        if self._tail is not None:
            return self._tail_step()
        inner = self.fp32_optimizer.optimizer
        ema = getattr(self, "_replicated_ema", None)  # [(flat per group)], decay: the EMA pass rides in the Adam kernel
        work = []
        for (flats16, master), group in zip(self._pairs(), inner.param_groups):
            state = inner._state_for(master)
            state["step"] += 1
            beta1, beta2 = group["betas"]
            offset = 0
            for f in flats16:
                n = f.numel()
                work.append(dict(
                    p=master.data[offset:offset + n], g=f.grad.data,
                    m=state["exp_avg"][offset:offset + n], v=state["exp_avg_sq"][offset:offset + n],
                    p_half=f.data, lr=group["lr"], beta1=beta1, beta2=beta2, eps=group["eps"],
                    step=state["step"], bias_correction=bool(group.get("bias_correction", True)),
                    weight_decay=group["weight_decay"],
                ))
                if ema is not None:
                    work[-1]["ema"] = ema[0][len(work) - 1].data
                offset += n
        factor = self._multiply_factor
        grad_scale = getattr(self, "_device_grad_scale", None)
        self._device_grad_scale = None
        if grad_scale is None:
            grad_scale = (1.0 / factor) if not torch.is_tensor(factor) else factor.reciprocal()
        ops.fused_adam(
            work,
            grad_scale=grad_scale,
            zero_grad=True,
            stochastic_rounding=self.bf16_sr,
            ema_decay=(ema[1] if ema is not None else None),
        )
        self._grads_zeroed = True
        self._needs_sync = False

    def _tail_step(self):
        """Same contract as ``_fused_step``, but the whole tail - including what is left of the gradient reduction, the
        norm, the clip / overflow decision and the statistics - is the ONE kernel of ``fused_tail.py``."""
        from unicore_b200.parallel.fused_tail import adam_hyper

        inner = self.fp32_optimizer.optimizer
        self._consolidated = None  # (a checkpoint's full-length copy of the moments is stale from here on)
        masters, avgs, sqs, hypers = [], [], [], []
        for (_flats16, master), group in zip(self._pairs(), inner.param_groups):
            state = inner._state_for(master)
            state["step"] += 1
            beta1, beta2 = group["betas"]
            masters.append(master.data)
            avgs.append(state["exp_avg"])
            sqs.append(state["exp_avg_sq"])
            hypers.append(adam_hyper(group["lr"], beta1, beta2, group["eps"], state["step"],
                                     bool(group.get("bias_correction", True)), group["weight_decay"]))
        factor = self._multiply_factor
        if torch.is_tensor(factor):
            raise RuntimeError("fused tail: device-side gradient factors go through set_step_stats(denom_index=...)")
        stats = self._tail_stats
        if stats is not None and not torch.is_tensor(stats):
            stats = utils.stack_scalars(stats, device=masters[0].device)
        state_vec = self._tail_engine.run_tail(
            masters=masters, exp_avgs=avgs, exp_avg_sqs=sqs, hypers=hypers, factor=float(factor),
            max_norm=self._tail_max_norm, clip_eps=0.0 if self.scaler is not None else 1e-6,
            emas=self._ema_flats, ema_decay=self._ema_decay, stats_src=stats, denom_index=self._tail_denom_index,
            stochastic_rounding=self.bf16_sr,
        )
        self._tail_stats, self._tail_denom_index = None, -1
        self._grads_zeroed = True
        self._needs_sync = False
        self._pending_norm = utils.AsyncHostRead(state_vec)
        if not getattr(self.args, "deferred_overflow_check", False):
            # reference behaviour: the caller learns about an overflow from this very call
            skipped = []
            self._late_overflow_handlers, saved = [skipped.append], getattr(self, "_late_overflow_handlers", [])
            try:
                self.resolve_pending_overflow()
            finally:
                self._late_overflow_handlers = saved
            if skipped:
                raise OverflowError(skipped[0])

    def zero_grad(self):
        """Zero the flat grads and reset the deferred factor to ``1/loss_scale``."""
        if not self._grads_zeroed:
            for g16 in self.fp16_params:
                for f in g16["params"]:
                    if f.grad is not None:
                        f.grad.zero_()
        if not self._fused:
            for g32 in self.fp32_params:
                for p in g32["params"]:
                    if p.grad is not None:
                        p.grad.zero_()
        self._grads_zeroed = True
        self._needs_sync = False
        self._has_accumulated = False
        self._device_grad_scale = None
        self._multiply_factor = 1.0 / float(self.scaler.loss_scale) if self.scaler is not None else 1.0


class FP16Optimizer(_FP16OptimizerMixin, UnicoreOptimizer):
    """Wraps an fp32 optimizer to train a pure fp16/bf16 model with fp32 master weights."""

    def __init__(self, args, params, fp32_optimizer, fp32_params, fused=False, **kwargs):
        super().__init__(args)
        self.fp16_params = params
        self.fp32_optimizer = fp32_optimizer
        self.fp32_params = fp32_params
        self.allreduce_fp32_grad = getattr(args, "allreduce_fp32_grad", False)
        self._fused = fused
        self._needs_sync = False
        self._has_accumulated = False

        if getattr(args, "fp16_scale_window", None) is None:
            if len(args.update_freq) > 1:
                raise ValueError("--fp16-scale-window must be given explicitly when using a custom --update-freq schedule")
            dp_world = int(args.distributed_world_size)
            scale_window = int(2 ** 14 / dp_world / args.update_freq[0])
        else:
            scale_window = args.fp16_scale_window

        if not getattr(args, "bf16", False):
            self.scaler = DynamicLossScaler(
                init_scale=args.fp16_init_scale,
                scale_window=scale_window,
                tolerance=args.fp16_scale_tolerance,
                threshold=args.threshold_loss_scale,
                min_loss_scale=args.min_loss_scale,
            )
        else:
            self.scaler = None  # bf16 has fp32's exponent range: no loss scaling

    @classmethod
    def build_optimizer(cls, args, params, grad_alloc=None, param_alloc=None, **kwargs):
        """``params``: list of ``(name, param)`` of the (already 16-bit) model."""
        from unicore import ops, optim

        if getattr(args, "fp16_no_flatten_grads", False):
            raise ValueError("--fp16-no-flatten-grads is not supported: flat arenas are the design")
        params = list(params)
        from unicore_b200.parallel import reference_tail_requested

        on_cuda = len(params) > 0 and params[0][1].is_cuda
        want_fused = (
            ((on_cuda and ops.HAS_CUDA_EXT) or reference_tail_requested())
            and getattr(args, "optimizer", "adam") == "adam"
            and not getattr(args, "use_old_adam", False)
            and not getattr(args, "allreduce_fp32_grad", False)
            and getattr(args, "per_sample_clip_norm", 0) <= 0
            and not getattr(args, "no_fused_optimizer_tail", False)
        )
        fp16_params, fp32_params = get_fp16_params(
            args, params, grad_alloc=grad_alloc, fp32_grads=not want_fused, param_alloc=param_alloc if want_fused else None
        )
        fp32_optimizer = optim.build_optimizer(args, fp32_params, separate=False)
        fused = want_fused and hasattr(fp32_optimizer.optimizer, "_state_for")
        if want_fused and not fused:  # inner optimizer is not FusedAdam after all
            for g in fp32_params:
                for p in g["params"]:
                    p.grad = torch.zeros_like(p)
        return cls(args, fp16_params, fp32_optimizer, fp32_params, fused=fused, **kwargs)

    # -- delegation ---------------------------------------------------------------------------------
    @property
    def optimizer(self):
        return self.fp32_optimizer.optimizer

    @optimizer.setter
    def optimizer(self, optimizer):
        self.fp32_optimizer.optimizer = optimizer

    @property
    def lr_scheduler(self):
        return getattr(self.fp32_optimizer, "lr_scheduler", None)

    @property
    def optimizer_config(self):
        return self.fp32_optimizer.optimizer_config

    def get_lr(self):
        return self.fp32_optimizer.get_lr()

    def set_lr(self, lr):
        self.fp32_optimizer.set_lr(lr)

    def all_reduce_grads(self, module):
        """``--allreduce-fp32-grad``: reduce the fp32 master grads instead of the 16-bit ones."""
        if self.allreduce_fp32_grad and hasattr(module, "all_reduce_params"):
            self._sync_fp16_grads_to_fp32()
            module.all_reduce_params([p for g in self.fp32_params for p in g["params"]])
        else:
            self.fp32_optimizer.all_reduce_grads(module)

    @property
    def supports_flat_params(self):
        return self.fp32_optimizer.supports_flat_params

    @property
    def supports_step_with_scale(self):
        return self.fp32_optimizer.supports_step_with_scale

    @property
    def is_fused(self):
        return self._fused
