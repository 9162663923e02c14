"""Loader for the in-tree sm_90a extension ``unicore_b200._C``.

The extension is built in-tree (``python setup.py build_ext --inplace`` or
``__graft_entry__.build()``) so the ``.so`` travels with the source snapshot.  Policy:

* CPU-only process (no CUDA device): the extension is optional, ops use PyTorch fallbacks.
* Hopper device (compute capability 9.x): a missing/unloadable extension is a hard error unless
  ``UNICORE_ALLOW_FALLBACK=1`` - silent eager fallbacks on a GPU box would hide that the native
  path is not running.
"""
import importlib
import logging
import os
import types

import torch

logger = logging.getLogger(__name__)

_C = None
_ERR = None
try:
    _C = importlib.import_module("unicore_b200._C")
except Exception as exc:  # noqa: BLE001 - ImportError, OSError (missing libs), ...
    _ERR = exc

HAS_CUDA_EXT = _C is not None


def _is_hopper() -> bool:
    try:
        return torch.cuda.is_available() and torch.cuda.get_device_capability()[0] == 9
    except Exception:  # noqa: BLE001
        return False


if _is_hopper() and _C is None and os.environ.get("UNICORE_ALLOW_FALLBACK", "0") != "1":
    # fail loudly where the kernels are the product
    raise ImportError(
        "unicore_b200._C (sm_90a kernels) failed to load on a CUDA machine: {!r}. Build it with "
        "`python setup.py build_ext --inplace` (or __graft_entry__.build()), or set "
        "UNICORE_ALLOW_FALLBACK=1 to run on PyTorch fallbacks.".format(_ERR)
    )

# kernels are compiled for sm_90a only (arch-specific code loads on no other GPU); elsewhere use the fallbacks
USE_NATIVE = HAS_CUDA_EXT and _is_hopper() and os.environ.get("UNICORE_DISABLE_NATIVE", "0") != "1"
if torch.cuda.is_available() and not USE_NATIVE:
    logger.warning(
        "unicore_b200: the sm_90a kernels are not in use on this machine (%s); PyTorch fallbacks run instead",
        "extension not built: {!r}".format(_ERR) if _C is None else "not a Hopper GPU or UNICORE_DISABLE_NATIVE=1")


# kernels launched per binding call (used for the benchmark's ``gpu_launches`` figure); bias_dropout_add_ln_bwd with a
# bias launches 4 on rows wider than 3072 16-bit columns, which no benchmark workload has
_LAUNCHES_PER_CALL = {
    "layernorm_bwd": 2, "rmsnorm_bwd": 2, "bias_dropout_add_ln_bwd": 2, "fmha_bwd": 4, "bias_gelu_bwd": 2, "symm_allreduce": 2,
    "column_sum": 2, "symm_reduce_scatter": 2, "symm_fused_tail": 1, "symm_stats_allreduce": 1,
    # not kernels: allocation / capability queries
    "SymmAllocation": 0, "symm_error_channel": 0, "symm_mem_supported": 0, "symm_multicast_supported": 0,
    "symm_tail_max_blocks": 0, "symm_pick_algo": 0,
    "norm_plan": 0, "softmax_plan": 0, "bias_gelu_plan": 0, "gbf_plan": 0, "head_permute_plan": 0, "pair_plan": 0,
    "embedding_plan": 0, "fmha_decode_max_splits": 0,
    "fmha_decode_num_splits": 0, "rotary_plan": 0,
}
_launch_count = 0


class _CountingProxy:
    """Forwards attribute access to the extension, counting kernel launches per call."""

    def __init__(self, mod):
        self._mod = mod
        self._cache = {}

    def __getattr__(self, name):
        fn = self._cache.get(name)
        if fn is None:
            target = getattr(self._mod, name)
            if isinstance(target, types.ModuleType):  # a submodule (_C.kvcache, _C.rotary): count its calls too
                fn = self._cache[name] = _CountingProxy(target)
                return fn
            if not callable(target):  # module constants (SYMM_MAX_PEERS, ...)
                return target
            n = _LAUNCHES_PER_CALL.get(name, 1)

            def fn(*args, __target=target, __n=n, **kwargs):
                global _launch_count
                _launch_count += __n
                return __target(*args, **kwargs)

            self._cache[name] = fn
        return fn


_PROXY = _CountingProxy(_C) if _C is not None else None


def launch_counter_reset():
    global _launch_count
    _launch_count = 0
    return 0


def launch_counter_read():
    return _launch_count


def native():
    """Return the extension module (raises if it is not loaded)."""
    if _C is None:
        raise RuntimeError("unicore_b200._C is not loaded: {!r}".format(_ERR))
    return _PROXY


def aligned_param(t, dtype=None):
    """Return ``t`` (cast to ``dtype``) as a 16-byte aligned, contiguous tensor.

    Parameters are views into flat arenas whose per-tensor padding is 2 elements (checkpoint layout
    contract), so a small 1-D parameter can start at a 4-byte boundary; the vectorised kernels need
    16-byte alignment.  The (differentiable) copy only happens for such misaligned vectors.
    """
    if t is None:
        return None
    if dtype is not None and t.dtype != dtype:
        t = t.to(dtype)
    if not t.is_contiguous() or t.data_ptr() % 16 != 0:
        t = t.clone(memory_format=torch.contiguous_format)
    return t


def aligned_rows(t):
    """``t`` as a contiguous, 16-byte aligned ``[rows, t.shape[-1]]`` tensor.

    The row kernels (norms, the fused bias + dropout + residual + LayerNorm) read with 16-byte vector loads and bulk
    copies from the first element on, so a contiguous view at an odd element offset (``buf[1:].view(n, d)``) must
    not reach them.  Such a view is copied once to a fresh (aligned) buffer: the kernel still runs, and the copy is
    the same pass an eager fallback would have to make anyway.  Aligned rows are returned as a view, without a copy.
    """
    return aligned_param(t.reshape(-1, t.shape[-1]))


def use_native(*tensors) -> bool:
    """True when the native kernels should handle these tensors."""
    if not USE_NATIVE:
        return False
    for t in tensors:
        if t is not None and not t.is_cuda:
            return False
    return True
