"""Data-parallel engine factory (``--ddp-backend``).

* ``c10d``   - torch DDP (bucketed NCCL/Gloo all-reduce overlapped with backward); also valid on
  CPU modules (the reference passes ``device_ids`` unconditionally and fails there).
* ``apex``   - apex DDP when installed.
* ``no_c10d`` / ``legacy_ddp`` - explicit flat-buffer all-reduce after backward.
* ``b200``   - symmetric-memory engine: gradients are reduced by hand-written sm_90a kernels over
  NVLink peer memory and fused with the optimizer (``unicore_b200.parallel``); needs CUDA + NCCL
  and falls back to ``c10d`` otherwise.
All engines are wrapped in ``ModuleProxyWrapper``.  Parity: reference
``unicore/models/distributed_unicore_model.py:20-67``.
"""
import logging

import torch.nn as nn

from unicore.distributed import LegacyDistributedDataParallel, ModuleProxyWrapper

logger = logging.getLogger(__name__)


def DistributedUnicoreModel(args, model, process_group, device):
    if not isinstance(model, nn.Module):
        raise TypeError("model must be an nn.Module")
    backend = args.ddp_backend
    on_cuda = device.type == "cuda"
    if backend == "b200":
        from unicore_b200.parallel import SymmDataParallel, reference_tail_requested, symm_available

        if reference_tail_requested():
            from unicore_b200.parallel.reference_tail import ReferenceTailEngine

            bucket_mb = float(getattr(args, "bucket_cap_mb", 25))
            return ModuleProxyWrapper(ReferenceTailEngine(model.to(device), process_group, bucket_cap_mb=bucket_mb))
        if on_cuda and symm_available():
            wrapped = SymmDataParallel(model.to(device), process_group, bucket_cap_mb=args.bucket_cap_mb)
            return ModuleProxyWrapper(wrapped)
        logger.warning("--ddp-backend b200 needs CUDA peer memory; falling back to c10d")
        backend = "c10d"
    if backend == "c10d":
        kwargs = dict(
            broadcast_buffers=args.broadcast_buffers,
            bucket_cap_mb=args.bucket_cap_mb,
            process_group=process_group,
            find_unused_parameters=args.find_unused_parameters,
        )
        if on_cuda:
            kwargs.update(device_ids=[args.device_id], output_device=args.device_id)
        wrapped = nn.parallel.DistributedDataParallel(module=model.to(device), **kwargs)
    elif backend == "apex":
        import apex

        wrapped = apex.parallel.DistributedDataParallel(module=model.to(device))
    elif backend in ("no_c10d", "legacy_ddp"):
        wrapped = LegacyDistributedDataParallel(module=model.to(device), buffer_size=2 ** 28, process_group=process_group)
    else:
        raise ValueError("Unknown --ddp-backend: " + backend)
    return ModuleProxyWrapper(wrapped)
