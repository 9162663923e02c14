"""Framework-wide helpers (sample movement, grad-norm/clip, seeding, flag value parsing, tensor
trees, activation lookup, user-module import).

Parity map (reference ``unicore/utils.py``): ``apply_to_sample:43``, ``move_to_cuda:64``,
``move_to_cpu:75`` (half/bf16 -> fp32), ``multi_tensor_total_norm:87``, ``clip_grad_norm_:111``,
``import_user_module:138``, ``get_activation_fn:174``, ``torch_seed:220``, ``CudaEnvironment:245``,
``eval_str_list/dict/bool:278-303``, ``checkpoint_sequential:306``, tensor-tree helpers
``:336-411``, ``fp32_to_bf16_sr:414``, ``set_jit_fusion_options:426``, ``validate_with_ema:437``.

Differences: the grad-norm and stochastic-rounding helpers dispatch to the hand-written
sm_90a kernels in ``unicore.ops`` (single-launch multi-tensor L2 norm, counter-based Philox SR)
and fall back to plain PyTorch on CPU.
"""
import contextlib
import copy
import hashlib
import importlib
import logging
import os
import sys
import weakref
from functools import partial
from typing import Any, Callable, Dict, List, Sequence

import torch
import torch.nn.functional as F
import torch.utils.checkpoint

logger = logging.getLogger(__name__)


# --------------------------------------------------------------------------------------------
# nested-sample helpers
# --------------------------------------------------------------------------------------------
def apply_to_sample(fn: Callable[[torch.Tensor], Any], sample):
    """Apply ``fn`` to every tensor inside an arbitrarily nested dict/list/tuple/set."""
    if hasattr(sample, "__len__") and len(sample) == 0:
        return {}

    def walk(node):
        if torch.is_tensor(node):
            return fn(node)
        if isinstance(node, dict):
            return {k: walk(v) for k, v in node.items()}
        if isinstance(node, list):
            return [walk(v) for v in node]
        if isinstance(node, tuple):
            return tuple(walk(v) for v in node)
        if isinstance(node, set):
            return {walk(v) for v in node}
        return node

    return walk(sample)


def move_to_cuda(sample, device=None):
    """Host->device copy of a sample; ``non_blocking`` only overlaps when the source is pinned
    (see ``unicore.data.iterators.BufferedIterator(pin_memory=True)``)."""
    device = device if device is not None else torch.cuda.current_device()
    return apply_to_sample(lambda t: t.to(device=device, non_blocking=True), sample)


def move_to_cpu(sample):
    """Device->host copy; 16-bit floats are widened to fp32 (checkpoints are stored in fp32)."""

    def to_cpu(t):
        if t.dtype in (torch.float16, torch.bfloat16):
            t = t.to(dtype=torch.float32)
        return t.cpu()

    return apply_to_sample(to_cpu, sample)


def pin_sample(sample):
    """Page-lock every tensor of a sample (addition: makes ``move_to_cuda`` truly async)."""
    if not torch.cuda.is_available():
        return sample
    return apply_to_sample(lambda t: t.pin_memory() if not t.is_pinned() else t, sample)


# --------------------------------------------------------------------------------------------
# gradient norm / clipping
# --------------------------------------------------------------------------------------------
class _HostReader:
    """Device scalar(s) -> host without parking the thread in a blocking stream synchronize.

    ``tensor.item()`` sleeps in ``cudaStreamSynchronize``; waking up is slow on virtualised
    hosts, and the GPU sits idle that long after each such host read.  Here the value is copied
    asynchronously into a cached pinned buffer and the thread polls the completion event instead.
    """

    def __init__(self):
        self._bufs = {}

    def read(self, t: torch.Tensor) -> torch.Tensor:
        if not t.is_cuda:
            return t
        key = (t.device, t.dtype, t.numel())
        slot = self._bufs.get(key)
        if slot is None:
            slot = (torch.empty(t.numel(), dtype=t.dtype, pin_memory=True), torch.cuda.Event())
            self._bufs[key] = slot
        buf, event = slot
        buf.copy_(t.detach().reshape(-1), non_blocking=True)
        event.record(torch.cuda.current_stream(t.device))
        while not event.query():
            pass
        return buf


_host_reader = _HostReader()


class AsyncHostRead:
    """Device value(s) on their way to the host: the copy is enqueued now, ``get()`` is called later (normally long
    after the copy has completed, so it does not stall anything).  A one-element tensor yields a python number, a
    longer one a list."""

    def __init__(self, t: torch.Tensor):
        self._value = None
        self._scalar = t.numel() == 1
        if not t.is_cuda:
            flat = t.detach().reshape(-1)
            self._value = flat[0].item() if self._scalar else flat.tolist()
            return
        self._buf = torch.empty(t.numel(), dtype=t.dtype, pin_memory=True)
        self._buf.copy_(t.detach().reshape(-1), non_blocking=True)
        self._event = torch.cuda.Event()
        self._event.record(torch.cuda.current_stream(t.device))

    def ready(self) -> bool:
        return self._value is not None or self._event.query()

    def get(self):
        if self._value is None:
            while not self._event.query():
                pass
            self._value = self._buf[0].item() if self._scalar else self._buf.tolist()
        return self._value


class _PinnedRing:
    """A few page-locked staging vectors per device, reused round-robin: host numbers reach the device with ONE
    asynchronous copy and without allocating pinned memory on the step path.  A slot is reused only after the copy
    that read it has completed (an event per slot; the ring is deep enough that this never waits in practice)."""

    def __init__(self, device, capacity=128, depth=16):
        self.device = device
        self.slots = [torch.empty(capacity, dtype=torch.float64, pin_memory=True) for _ in range(depth)]
        self.events = [None] * depth
        self.cursor = 0

    def send(self, numbers):
        n = len(numbers)
        i = self.cursor
        self.cursor = (i + 1) % len(self.slots)
        if n > self.slots[i].numel():
            return torch.tensor(numbers, dtype=torch.float64).to(self.device)
        if self.events[i] is not None:
            self.events[i].synchronize()
        buf = self.slots[i]
        for k, v in enumerate(numbers):
            buf[k] = v
        out = buf[:n].to(self.device, non_blocking=True)
        if self.events[i] is None:
            self.events[i] = torch.cuda.Event()
        self.events[i].record(torch.cuda.current_stream(self.device))
        return out


_pinned_rings = {}


def stack_scalars(values, device=None, dtype=torch.float64) -> torch.Tensor:
    """A list of python numbers and 0-dim tensors as ONE 1-D tensor on ``device``, in order, without synchronising
    the host: host numbers travel together through a page-locked ring slot, device scalars are stacked per dtype; if
    device scalars are not already in front (grouped by dtype) the result is assembled by slice copies."""
    values = list(values)
    n = len(values)
    dev_idx = [i for i, v in enumerate(values) if torch.is_tensor(v) and v.is_cuda]
    if device is None:
        device = values[dev_idx[0]].device if dev_idx else torch.device("cpu")
    device = torch.device(device)
    on_dev = set(dev_idx)
    host_idx = [i for i in range(n) if i not in on_dev]
    host_vals = [float(values[i]) if not torch.is_tensor(values[i]) else float(values[i].item()) for i in host_idx]
    if device.type != "cuda":
        out = torch.empty(n, dtype=dtype)
        for i, v in zip(host_idx, host_vals):
            out[i] = v
        for i in dev_idx:
            out[i] = values[i].detach().to("cpu", dtype)
        return out.to(device)
    if device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    parts, order = [], []
    by_dtype = {}
    for i in dev_idx:
        by_dtype.setdefault(values[i].dtype, []).append(i)
    for _dt, idx in by_dtype.items():
        parts.append(torch.stack([values[i].detach().reshape(()) for i in idx]).to(dtype))
        order += idx
    if host_idx:
        ring = _pinned_rings.get(device)
        if ring is None:
            ring = _pinned_rings[device] = _PinnedRing(device)
        staged = ring.send(host_vals)
        parts.append(staged if dtype == torch.float64 else staged.to(dtype))
        order += host_idx
    packed = torch.cat(parts) if len(parts) > 1 else parts[0]
    if order == list(range(n)):
        return packed
    out = torch.empty(n, dtype=dtype, device=device)
    # (rare: callers that care order their entries device-first; runs of consecutive targets become one copy each)
    pos = 0
    while pos < n:
        end = pos + 1
        while end < n and order[end] == order[end - 1] + 1:
            end += 1
        out[order[pos]:order[pos] + (end - pos)].copy_(packed[pos:end])
        pos = end
    return out


def item(t):
    """``float(t)`` / ``t.item()`` for a device scalar via the polling reader; passes numbers through."""
    if not torch.is_tensor(t):
        return t
    if not t.is_cuda:
        return t.item()
    return _host_reader.read(t)[0].item()


def tolist(t: torch.Tensor) -> list:
    """``t.tolist()`` of a small device vector via the polling reader."""
    if not t.is_cuda:
        return t.tolist()
    return _host_reader.read(t).view(t.shape).tolist()


# ---- logging outputs on their way to the host -------------------------------------------------------------------------
_staged_logs = {}


def stage_logging_output(log, enabled=True) -> None:
    """Start copying the device scalars of one micro-batch's logging output to pinned host memory NOW - a loss calls
    this between its forward and the backward launch, so the copy sits in the stream right behind the forward pass.
    ``resolve_logging_output`` later swaps the host numbers in.  Reading ``train_step(...)["loss"]`` then waits for the
    end of the FORWARD pass instead of the end of the whole update: a caller that reads the loss every step (an
    end-to-end benchmark, a notebook) keeps the launch queue a full backward pass ahead of the device."""
    if not enabled or not isinstance(log, dict):
        return
    keys = [k for k, v in log.items() if torch.is_tensor(v) and v.is_cuda and v.numel() == 1]
    if not keys:
        return
    packed = torch.stack([log[k].detach().reshape(()).double() for k in keys])
    _staged_logs[id(log)] = (log, keys, AsyncHostRead(packed))
    if len(_staged_logs) > 64:   # logging outputs that were never resolved (aborted steps): do not grow forever
        for stale in list(_staged_logs)[:-32]:
            _staged_logs.pop(stale, None)


def resolve_logging_output(log):
    """The logging output with its staged device scalars replaced by python floats (waits for the staged copy, i.e. for
    the forward pass that produced them); unchanged when nothing was staged."""
    entry = _staged_logs.pop(id(log), None)
    if entry is None or entry[0] is not log:
        return log
    _, keys, pending = entry
    numbers = pending.get()
    numbers = numbers if isinstance(numbers, list) else [numbers]
    resolved = dict(log)
    for key, number in zip(keys, numbers):
        resolved[key] = number
    return resolved


_mask_index_cache = (None, None, None)   # (weakref of the mask, indices or None, pending count read or None)


def request_mask_index(mask: torch.Tensor) -> None:
    """Start resolving ``mask_to_index(mask)`` without waiting: the number of True entries is summed on the device and
    copied to pinned host memory asynchronously.  A masked-LM loss calls this BEFORE the model runs; by the time the LM
    head asks for the indices the copy - queued ahead of the whole encoder - has long completed, so the host neither
    stalls nor lets the launch queue run dry (a blocking read at this point idles the GPU every step)."""
    global _mask_index_cache
    ref = _mask_index_cache[0]
    if ref is not None and ref() is mask:
        return
    flat = mask.reshape(-1)
    pending = None
    if flat.is_cuda and hasattr(torch, "nonzero_static"):
        pending = AsyncHostRead(flat.sum())
    _mask_index_cache = (weakref.ref(mask), None, pending)


def mask_to_index(mask: torch.Tensor) -> torch.Tensor:
    """Flat indices of the True entries of a boolean mask.

    ``x[mask]`` synchronises inside ``nonzero`` and its backward sorts the indices; a masked-LM step
    indexes with the same mask twice (features and targets).  This computes the indices once per
    mask object: one host read of the count (started early by ``request_mask_index``), then
    ``nonzero_static`` (no further sync); use ``index_select`` with the result (its backward is a
    plain ``index_add``).
    """
    global _mask_index_cache
    ref, idx, pending = _mask_index_cache
    if ref is None or ref() is not mask:
        request_mask_index(mask)
        ref, idx, pending = _mask_index_cache
    if idx is not None:
        return idx
    flat = mask.reshape(-1)
    if pending is not None:
        try:
            idx = torch.nonzero_static(flat, size=int(pending.get())).squeeze(1)
        except (RuntimeError, NotImplementedError):
            idx = None
    if idx is None:
        idx = flat.nonzero(as_tuple=False).squeeze(1)
    _mask_index_cache = (ref, idx, None)
    return idx


def multi_tensor_total_norm(grads: Sequence[torch.Tensor], chunk_size: int = 2048 * 32) -> torch.Tensor:
    """Global L2 norm of a list of tensors as an fp32 scalar tensor (no host sync)."""
    from unicore import ops

    grads = list(grads)
    if len(grads) == 0:
        return torch.zeros((), dtype=torch.float32)
    return ops.multi_tensor_l2norm(grads, chunk_size=chunk_size)


@torch.no_grad()
def clip_grad_norm_(params, max_norm, aggregate_norm_fn=None) -> torch.Tensor:
    """Clip the global grad norm of ``params`` to ``max_norm``; returns the *pre-clip* norm.

    coefficient = clamp(max_norm / (norm + 1e-6), max=1) (reference ``utils.py:130-134``).
    The scaling is a single fused multi-tensor launch on GPU and never synchronises the host.
    """
    from unicore import ops

    if isinstance(params, torch.Tensor):
        params = [params]
    params = list(params)
    grads = [p.grad.detach() for p in params if getattr(p, "grad", None) is not None]
    if len(grads) == 0:
        if len(params) > 0:
            return params[0].new_tensor(0.0)
        return torch.tensor(0.0)
    total_norm = multi_tensor_total_norm(grads)
    if aggregate_norm_fn is not None:
        total_norm = aggregate_norm_fn(total_norm)
    if max_norm > 0:
        max_norm = float(max_norm)
        clip_coef = (max_norm / (total_norm + 1e-6)).clamp_(max=1.0)
        ops.multi_tensor_scale_(grads, clip_coef)
    return total_norm


# --------------------------------------------------------------------------------------------
# plug-ins
# --------------------------------------------------------------------------------------------
def import_user_module(args) -> None:
    """Import the package named by ``--user-dir`` so that its ``@register_*`` decorators run."""
    module_path = getattr(args, "user_dir", None)
    if module_path is None:
        return
    module_path = os.path.abspath(module_path)
    if not os.path.exists(module_path):
        # allow paths relative to the installed package (``unicore/../<user_dir>``)
        alt = os.path.join(os.path.dirname(os.path.dirname(__file__)), args.user_dir)
        if os.path.exists(alt):
            module_path = alt
        else:
            raise FileNotFoundError(module_path)
    registry = import_user_module.__dict__.setdefault("_seen", {})
    parent, name = os.path.split(module_path.rstrip(os.sep))
    if name in sys.modules and name not in registry:
        existing = getattr(sys.modules[name], "__file__", None) or ""
        if os.path.dirname(os.path.abspath(existing)) != module_path:
            raise ImportError(
                "Failed to import --user-dir={} because the module name ({}) is not globally "
                "unique. Please rename the directory.".format(module_path, name)
            )
    if name in registry:
        return
    registry[name] = module_path
    sys.path.insert(0, parent)
    try:
        importlib.import_module(name)
    finally:
        # keep parent on sys.path: plug-ins commonly do sibling imports lazily
        pass


# --------------------------------------------------------------------------------------------
# activations
# --------------------------------------------------------------------------------------------
_ACTIVATIONS: Dict[str, Callable] = {
    "relu": F.relu,
    "gelu": F.gelu,
    "tanh": torch.tanh,
    "linear": lambda x: x,
}


def get_activation_fn(activation: str) -> Callable:
    try:
        return _ACTIVATIONS[activation]
    except KeyError:
        raise RuntimeError("--activation-fn {} not supported".format(activation))


def get_available_activation_fns() -> List[str]:
    return list(_ACTIVATIONS.keys())


def has_parameters(module) -> bool:
    for _ in module.parameters():
        return True
    return False


# --------------------------------------------------------------------------------------------
# RNG discipline
# --------------------------------------------------------------------------------------------
def get_rng_state() -> dict:
    state = {"torch_rng_state": torch.get_rng_state()}
    if torch.cuda.is_available():
        state["cuda_rng_state"] = torch.cuda.get_rng_state()
    return state


def set_rng_state(state: dict) -> None:
    torch.set_rng_state(state["torch_rng_state"])
    if torch.cuda.is_available() and "cuda_rng_state" in state:
        torch.cuda.set_rng_state(state["cuda_rng_state"])


def _mix_seed(seed, addl) -> int:
    """Deterministically fold a tuple of ints into one 31-bit-ish seed (stable across runs —
    unlike Python's ``hash`` this does not depend on PYTHONHASHSEED)."""
    if len(addl) == 0:
        return int(seed)
    blob = ",".join(str(int(s)) for s in (seed,) + tuple(addl)).encode()
    return int.from_bytes(hashlib.blake2b(blob, digest_size=8).digest(), "little") % (2 ** 31 - 1)


def _active_generators():
    """The generators a training step draws from: CPU default + the current CUDA device's default."""
    gens = [torch.default_generator]
    if torch.cuda.is_available() and torch.cuda.is_initialized():
        gens.append(torch.cuda.default_generators[torch.cuda.current_device()])
    return gens


@contextlib.contextmanager
def torch_seed(seed, *addl_seeds):
    """Seed torch (CPU + current CUDA device) inside the block, restore the RNG state after.

    Used for per-(update, micro-batch, rank) dropout reproducibility and the rank-invariant
    optimizer-step stream that stochastic rounding relies on (reference ``trainer.py:602-607,712``).
    The generators are driven directly: ``torch.manual_seed`` walks every device backend (and queues
    a formatted stack trace per call for uninitialised ones), which sat on the critical path twice
    per training step.
    """
    if seed is None:
        yield
        return
    seed = _mix_seed(seed, addl_seeds)
    if torch.cuda.is_available() and not torch.cuda.is_initialized():
        saved = get_rng_state()
        torch.manual_seed(seed)  # CUDA not initialised yet: let torch queue the device seeding
        try:
            yield
        finally:
            set_rng_state(saved)
        return
    gens = _active_generators()
    saved = [g.get_state() for g in gens]
    for g in gens:
        g.manual_seed(seed)
    try:
        yield
    finally:
        for g, st in zip(gens, saved):
            g.set_state(st)


# --------------------------------------------------------------------------------------------
# environment report
# --------------------------------------------------------------------------------------------
class CudaEnvironment(object):
    """Snapshot of the local GPU, gathered from all ranks and printed once by rank 0."""

    def __init__(self):
        dev = torch.cuda.current_device()
        prop = torch.cuda.get_device_properties("cuda:{}".format(dev))
        self.name = prop.name
        self.major = prop.major
        self.minor = prop.minor
        self.total_memory_in_GB = prop.total_memory / 1024 / 1024 / 1024
        self.sm_count = prop.multi_processor_count

    @staticmethod
    def pretty_print_cuda_env_list(cuda_env_list):
        n = len(cuda_env_list)
        header = "CUDA environments for all {} workers".format(n)
        bar = "*" * (len(header) + 8)
        lines = [bar, "*** " + header + " ***"]
        for rank, env in enumerate(cuda_env_list):
            lines.append(
                "rank {:3d}: capabilities = {:2d}.{:<2d}; total memory = {:.3f} GB; SMs = {}; name = {}".format(
                    rank, env.major, env.minor, env.total_memory_in_GB,
                    getattr(env, "sm_count", -1), env.name,
                )
            )
        lines.append(bar)
        for line in lines:
            logger.info(line)


# --------------------------------------------------------------------------------------------
# flag value parsers (kept eval-compatible with the reference CLI: "--lr '[1e-3, 1e-4]'")
# --------------------------------------------------------------------------------------------
def csv_str_list(x):
    return x.split(",")


def _safe_eval(x):
    import ast

    try:
        return ast.literal_eval(x)
    except (ValueError, SyntaxError):
        return eval(x)  # noqa: S307 - parity with reference semantics for expressions like 2**7


def eval_str_list(x, type=float):
    if x is None:
        return None
    if isinstance(x, str):
        x = _safe_eval(x)
    try:
        return [type(v) for v in x]
    except TypeError:
        return [type(x)]


def eval_str_dict(x, type=dict):
    if x is None:
        return None
    if isinstance(x, str):
        x = _safe_eval(x)
    return x


def eval_bool(x, default=False):
    if x is None:
        return default
    try:
        return bool(_safe_eval(x)) if isinstance(x, str) else bool(x)
    except (TypeError, NameError):
        return default


# --------------------------------------------------------------------------------------------
# activation checkpointing over a list of callables
# --------------------------------------------------------------------------------------------
def checkpoint_sequential(functions: Sequence[Callable], input, enabled: bool = True):
    """Run ``functions`` in order, re-materialising each one's activations in backward.

    ``input`` may be a tensor or a tuple of tensors; each function receives the unpacked tuple and
    may return a tensor or a tuple.
    """

    def as_tuple(value):
        return value if isinstance(value, tuple) else (value,)

    def make_runner(fn):
        def runner(*packed):
            return as_tuple(fn(*packed))

        return runner

    packed = as_tuple(input)
    was_tuple = isinstance(input, tuple)
    for fn in functions:
        if enabled and torch.is_grad_enabled():
            packed = torch.utils.checkpoint.checkpoint(make_runner(fn), *packed, use_reentrant=False)
        else:
            packed = as_tuple(fn(*packed))
    if not was_tuple and len(packed) == 1:
        return packed[0]
    return packed


# --------------------------------------------------------------------------------------------
# tensor / tree utilities used by downstream structure models (Uni-Fold style)
# --------------------------------------------------------------------------------------------
def permute_final_dims(tensor: torch.Tensor, inds: List[int]):
    lead = tensor.dim() - len(inds)
    return tensor.permute(*range(lead), *[lead + i for i in inds])


def flatten_final_dims(t: torch.Tensor, num_dims: int):
    return t.reshape(*t.shape[: t.dim() - num_dims], -1)


def masked_mean(mask, value, dim, eps=1e-10):
    mask = mask.expand(*value.shape)
    return (mask * value).sum(dim=dim) / (mask.sum(dim=dim) + eps)


def dict_multimap(fn, dicts):
    head = dicts[0]
    out = {}
    for key, val in head.items():
        column = [d[key] for d in dicts]
        out[key] = dict_multimap(fn, column) if type(val) is dict else fn(column)
    return out


def one_hot(x, num_classes, dtype=torch.float32):
    out = torch.zeros(*x.shape, num_classes, dtype=dtype, device=x.device)
    return out.scatter_(-1, x.long().unsqueeze(-1), 1)


def batched_gather(data, inds, dim=0, num_batch_dims=0):
    if not (dim < 0 or dim - num_batch_dims >= 0):
        raise ValueError("dim must address a non-batch dimension")
    index = []
    for i, size in enumerate(data.shape[:num_batch_dims]):
        shape = [1] * inds.dim()
        shape[i] = -1
        index.append(torch.arange(size, device=inds.device).view(*shape))
    rest = [slice(None)] * (data.dim() - num_batch_dims)
    rest[dim - num_batch_dims if dim >= 0 else dim] = inds
    index.extend(rest)
    return data[tuple(index)]


def dict_map(fn, dic, leaf_type):
    return {
        k: (dict_map(fn, v, leaf_type) if type(v) is dict else tree_map(fn, v, leaf_type))
        for k, v in dic.items()
    }


def tree_map(fn, tree, leaf_type):
    if isinstance(tree, dict):
        return dict_map(fn, tree, leaf_type)
    if isinstance(tree, list):
        return [tree_map(fn, x, leaf_type) for x in tree]
    if isinstance(tree, tuple):
        return tuple(tree_map(fn, x, leaf_type) for x in tree)
    if isinstance(tree, leaf_type):
        try:
            return fn(tree)
        except Exception as exc:  # noqa: BLE001
            raise ValueError("cannot apply {} on {}.".format(fn, tree)) from exc
    raise ValueError("{} not supported".format(type(tree)))


tensor_tree_map = partial(tree_map, leaf_type=torch.Tensor)


# --------------------------------------------------------------------------------------------
# stochastic rounding, JIT switches, EMA validation swap
# --------------------------------------------------------------------------------------------
def fp32_to_bf16_sr(t: torch.Tensor, o: torch.Tensor) -> None:
    """Stochastically round fp32 ``t`` into bf16 ``o`` (unbiased: E[o] == t)."""
    from unicore import ops

    ops.fp32_to_bf16_sr(t, o)


def set_jit_fusion_options() -> None:
    """Kept for CLI parity. This build does not rely on TorchScript fusers: hot element-wise
    chains are explicit CUDA kernels, so we only make sure legacy fusers are off."""
    try:
        torch._C._jit_set_profiling_executor(True)
        torch._C._jit_set_profiling_mode(True)
        torch._C._jit_override_can_fuse_on_cpu(False)
        torch._C._jit_override_can_fuse_on_gpu(False)
        torch._C._jit_set_texpr_fuser_enabled(False)
        torch._C._jit_set_nvfuser_enabled(False)
    except Exception:  # noqa: BLE001 - private API, best effort
        pass


@contextlib.contextmanager
def validate_with_ema(trainer, ema=False):
    """Temporarily swap the trainer's model for (a half/bf16 copy of) the EMA weights."""
    if not ema:
        yield
        return
    sync = getattr(trainer, "sync_ema_shards", None)
    if sync is not None:
        sync()  # (collective: a sharded EMA is merged on every rank before it is evaluated)
    live_model = trainer._wrapped_model
    shadow = copy.deepcopy(trainer.ema.model_ema)
    if trainer.args.fp16:
        shadow.half()
    elif trainer.args.bf16:
        shadow.bfloat16()
    trainer._wrapped_model = shadow
    try:
        yield
    finally:
        del shadow
        trainer._wrapped_model = live_model
