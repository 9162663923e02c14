"""Command-line flag system: argparse + registries, parsed in two passes.

Pass 1 discovers ``--arch``, ``--task`` and each registry choice; the selected classes then
contribute their own flags through ``add_args`` and pass 2 parses everything. Flag names,
defaults and semantics follow the reference CLI (``unicore/options.py:24-428``; complete list in
SURVEY.md Appendix A) so existing launch scripts work unchanged. The flag tables below are
declarative: ``(names, kwargs)`` rows consumed by ``_add_rows``.

Additions (all optional, defaults preserve reference behaviour):
``--ddp-backend b200`` (gradient all-reduce kernels over NVLink symmetric memory, bucketed and overlapped with
backward, gradient norm accumulated in the same pass; falls back to c10d when peer memory is unavailable),
``--pin-memory`` (pinned batches + non-blocking H2D) and ``--deferred-overflow-check`` (fp16: the overflow
decision stays on the device, no host read between backward and the optimizer).
"""
import argparse
from typing import Callable, List, Optional

import torch

from unicore.utils import csv_str_list, eval_bool, eval_str_dict, eval_str_list, import_user_module  # noqa: F401


# ------------------------------------------------------------------------------------------------
# flag tables
# ------------------------------------------------------------------------------------------------
def _flag(*names, **kw):
    return (names, kw)


def _add_rows(target, rows) -> None:
    for names, kw in rows:
        target.add_argument(*names, **kw)


def _global_rows():
    return [
        _flag("--no-progress-bar", action="store_true", help="disable progress bar"),
        _flag("--log-interval", type=int, default=1000, metavar="N",
              help="log progress every N updates (when progress bar is disabled)"),
        _flag("--log-format", default=None, choices=["json", "none", "simple", "tqdm"],
              help="log format to use"),
        _flag("--tensorboard-logdir", metavar="DIR", default="",
              help="path to save logs for tensorboard (default: no tensorboard logging)"),
        _flag("--wandb-project", metavar="DIR", default="", help="Weights&Biases project name"),
        _flag("--wandb-name", metavar="DIR", default="", help="Weights&Biases run name"),
        _flag("--seed", default=1, type=int, metavar="N", help="pseudo random number generator seed"),
        _flag("--deterministic", action="store_true",
              help="bitwise reproducible training on one GPU: torch.use_deterministic_algorithms(True), which also "
                   "switches the native kernels to their fixed-order reductions (slower backward)"),
        _flag("--cpu", action="store_true", help="use CPU instead of CUDA"),
        _flag("--fp16", action="store_true", help="fp16 model + fp32 master weights + dynamic loss scaling"),
        _flag("--bf16", action="store_true", help="bf16 model + fp32 master weights (no loss scaling)"),
        _flag("--bf16-sr", action="store_true", help="stochastic rounding when writing bf16 params"),
        _flag("--allreduce-fp32-grad", action="store_true",
              help="all-reduce the fp32 master grads instead of the 16-bit grads (--ddp-backend no_c10d)"),
        _flag("--fp16-no-flatten-grads", action="store_true", help="don't flatten FP16 grads tensor"),
        _flag("--fp16-init-scale", default=2 ** 7, type=int, help="default FP16 loss scale"),
        _flag("--fp16-scale-window", type=int, help="number of updates before increasing loss scale"),
        _flag("--deferred-overflow-check", action="store_true",
              help="fp16 + fused optimizer: do not read the gradient norm on the host before the update; the "
                   "fused Adam kernel skips itself when the norm is non-finite and the loss scaler learns about "
                   "the overflow before the next backward pass (removes the per-step pipeline drain)"),
        _flag("--no-grad-sinks", action="store_true",
              help="keep plain autograd accumulation of parameter gradients (default on CUDA with flat 16-bit arenas: the "
                   "backward kernels add weight / bias / LayerNorm gradients straight into the gradient arena)"),
        _flag("--fp16-scale-tolerance", default=0.0, type=float,
              help="pct of updates that can overflow before decreasing the loss scale"),
        _flag("--min-loss-scale", default=1e-4, type=float, metavar="D",
              help="minimum FP16 loss scale, after which training is stopped"),
        _flag("--threshold-loss-scale", type=float, help="threshold FP16 loss scale from below"),
        _flag("--user-dir", default=None,
              help="path to a python module containing custom extensions (tasks and/or architectures)"),
        _flag("--empty-cache-freq", default=0, type=int,
              help="how often to clear the PyTorch CUDA cache (0 to disable)"),
        _flag("--all-gather-list-size", default=16384, type=int,
              help="number of bytes reserved for gathering stats from workers"),
        _flag("--suppress-crashes", action="store_true",
              help="suppress crashes when training with the entry point"),
        _flag("--profile", action="store_true", help="emit NVTX ranges (autograd profiler emit_nvtx)"),
        _flag("--ema-decay", default=-1.0, type=float, help="enable moving average for model weights"),
        _flag("--validate-with-ema", action="store_true"),
    ]


def _dataset_rows():
    return [
        _flag("--num-workers", default=1, type=int, metavar="N", help="how many subprocesses to use for data loading"),
        _flag("--skip-invalid-size-inputs-valid-test", action="store_true",
              help="ignore too long or too short lines in valid and test set"),
        _flag("--batch-size", "--max-sentences", type=int, metavar="N", help="maximum number of sentences in a batch"),
        _flag("--required-batch-size-multiple", default=1, type=int, metavar="N",
              help="batch size will be a multiplier of this value"),
        _flag("--data-buffer-size", default=10, type=int, help="number of batches to preload"),
        _flag("--train-subset", default="train", metavar="SPLIT",
              choices=["train", "valid", "test", "train.small"],
              help="data subset to use for training (train, valid, test)"),
        _flag("--valid-subset", default="valid", metavar="SPLIT",
              help="comma separated list of data subsets to use for validation (train, valid, valid1, test, test1)"),
        _flag("--validate-interval", type=int, default=1, metavar="N", help="validate every N epochs"),
        _flag("--validate-interval-updates", type=int, default=0, metavar="N", help="validate every N updates"),
        _flag("--validate-after-updates", type=int, default=0, metavar="N",
              help="dont validate until reaching this many updates"),
        _flag("--fixed-validation-seed", default=None, type=int, metavar="N",
              help="specified random seed for validation"),
        _flag("--disable-validation", action="store_true", help="disable validation"),
        _flag("--batch-size-valid", type=int, metavar="N",
              help="maximum number of sentences in a validation batch (defaults to --max-sentences)"),
        _flag("--max-valid-steps", type=int, metavar="N", help="How many batches to evaluate"),
        _flag("--curriculum", default=0, type=int, metavar="N", help="don't shuffle batches for first N epochs"),
        # addition: page-locked host staging so the H2D copy overlaps compute
        _flag("--pin-memory", action="store_true",
              help="page-lock prefetched batches so host-to-device copies are asynchronous"),
    ]


def _distributed_rows():
    n_dev = max(1, torch.cuda.device_count())
    return [
        _flag("--distributed-world-size", type=int, metavar="N", default=n_dev,
              help="total number of GPUs across all nodes (default: all visible GPUs)"),
        _flag("--distributed-rank", default=0, type=int, help="rank of the current worker"),
        _flag("--distributed-backend", default="nccl", type=str, help="distributed backend"),
        _flag("--distributed-init-method", default=None, type=str,
              help="typically tcp://hostname:port that will be used to establish initial connetion"),
        _flag("--distributed-port", default=-1, type=int, help="port number (not required if using --distributed-init-method)"),
        _flag("--device-id", "--local_rank", default=0, type=int, help="which GPU to use (usually configured automatically)"),
        _flag("--distributed-no-spawn", action="store_true",
              help="do not spawn multiple processes even if multiple GPUs are visible"),
        _flag("--ddp-backend", default="c10d", type=str, choices=["c10d", "apex", "no_c10d", "legacy_ddp", "b200"],
              help="DistributedDataParallel backend (b200 = all-reduce kernels over NVLink symmetric memory)"),
        _flag("--bucket-cap-mb", default=25, type=int, metavar="MB", help="bucket size for reduction"),
        _flag("--fix-batches-to-gpus", action="store_true",
              help="don't shuffle batches between GPUs; this reduces overall randomness"),
        _flag("--find-unused-parameters", default=False, action="store_true",
              help="disable unused parameter detection (not applicable to no_c10d ddp-backend"),
        _flag("--fast-stat-sync", default=False, action="store_true",
              help="[deprecated] this is now defined per Loss"),
        _flag("--broadcast-buffers", default=False, action="store_true",
              help="Copy non-trainable parameters between GPUs, such as batchnorm population statistics"),
        _flag("--nprocs-per-node", default=n_dev, type=int,
              help="number of GPUs in each node"),
    ]


def _optimization_rows():
    return [
        _flag("--max-epoch", "--me", default=0, type=int, metavar="N", help="force stop training at specified epoch"),
        _flag("--max-update", "--mu", default=0, type=int, metavar="N", help="force stop training at specified update"),
        _flag("--stop-time-hours", default=0, type=float, help="force stop training after specified cumulative time"),
        _flag("--no-weight-decay-names", default="", type=str, help="names of parameters to not apply weight decay"),
        _flag("--clip-norm", default=0, type=float, metavar="NORM", help="clip threshold of gradients"),
        _flag("--per-sample-clip-norm", default=0, type=float, metavar="PNORM",
              help="clip threshold of gradients, before gradient sync over workers"),
        _flag("--update-freq", default="1", metavar="N1,N2,...,N_K",
              type=lambda uf: eval_str_list(uf, type=int),
              help="update parameters every N_i batches, when in epoch i"),
        _flag("--lr", "--learning-rate", default="0.25", type=eval_str_list, metavar="LR_1,LR_2,...,LR_N",
              help="learning rate for the first N epochs; all epochs >N using LR_N"),
        _flag("--stop-min-lr", default=-1, type=float, metavar="LR",
              help="stop training when the learning rate reaches this minimum"),
    ]


def _checkpoint_rows():
    return [
        _flag("--save-dir", metavar="DIR", default="checkpoints", help="path to save checkpoints"),
        _flag("--tmp-save-dir", metavar="DIR", default="./", help="path to temporarily save checkpoints"),
        _flag("--restore-file", default="checkpoint_last.pt",
              help="filename from which to load checkpoint (default: <save-dir>/checkpoint_last.pt"),
        _flag("--finetune-from-model", type=str,
              help="finetune from a pretrained model; note that meters and lr scheduler will be reset"),
        _flag("--load-from-ema", action="store_true", help="finetune from a pretrained model's EMA weights"),
        _flag("--reset-dataloader", action="store_true",
              help="if set, does not reload dataloader state from the checkpoint"),
        _flag("--reset-lr-scheduler", action="store_true",
              help="if set, does not load lr scheduler state from the checkpoint"),
        _flag("--reset-meters", action="store_true", help="if set, does not load meters from the checkpoint"),
        _flag("--reset-optimizer", action="store_true", help="if set, does not load optimizer state from the checkpoint"),
        _flag("--optimizer-overrides", default="{}", type=str, metavar="DICT",
              help="a dictionary used to override optimizer args when loading a checkpoint"),
        _flag("--save-interval", type=int, default=1, metavar="N", help="save a checkpoint every N epochs"),
        _flag("--save-interval-updates", type=int, default=0, metavar="N",
              help="save a checkpoint (and validate) every N updates"),
        _flag("--keep-interval-updates", type=int, default=-1, metavar="N",
              help="keep the last N checkpoints saved with --save-interval-updates"),
        _flag("--keep-last-epochs", type=int, default=-1, metavar="N", help="keep last N epoch checkpoints"),
        _flag("--keep-best-checkpoints", type=int, default=-1, metavar="N",
              help="keep best N checkpoints based on scores"),
        _flag("--no-save", action="store_true", help="don't save models or checkpoints"),
        _flag("--no-epoch-checkpoints", action="store_true", help="only store last and best checkpoints"),
        _flag("--no-last-checkpoints", action="store_true", help="don't store last checkpoints"),
        _flag("--no-save-optimizer-state", action="store_true",
              help="don't save optimizer-state as part of checkpoint"),
        _flag("--best-checkpoint-metric", type=str, default="loss", help='metric to use for saving "best" checkpoints'),
        _flag("--maximize-best-checkpoint-metric", action="store_true",
              help='select the largest metric value for saving "best" checkpoints'),
        _flag("--patience", type=int, default=-1, metavar="N",
              help="early stop training if valid performance doesn't improve for N consecutive validation runs"),
        _flag("--checkpoint-suffix", type=str, default="", help="suffix to add to the checkpoint file name"),
    ]


# ------------------------------------------------------------------------------------------------
# group builders (public names kept)
# ------------------------------------------------------------------------------------------------
def add_dataset_args(parser, train=False, gen=False):
    group = parser.add_argument_group("Dataset and data loading")
    _add_rows(group, _dataset_rows())
    return group


def add_distributed_training_args(parser):
    group = parser.add_argument_group("Distributed training")
    _add_rows(group, _distributed_rows())
    return group


def add_optimization_args(parser):
    group = parser.add_argument_group("Optimization")
    _add_rows(group, _optimization_rows())
    return group


def add_checkpoint_args(parser):
    group = parser.add_argument_group("Checkpointing")
    _add_rows(group, _checkpoint_rows())
    return group


def add_common_eval_args(group):
    _add_rows(group, [
        _flag("--path", metavar="FILE", help="path(s) to model file(s), colon separated"),
        _flag("--quiet", action="store_true", help="only print final scores"),
        _flag("--model-overrides", default="{}", type=str, metavar="DICT",
              help="a dictionary used to override model args at generation that were used during model training"),
        _flag("--results-path", metavar="RESDIR", type=str, default=None, help="path to save eval results (optional)"),
    ])


def add_model_args(parser):
    from unicore.models import ARCH_MODEL_REGISTRY

    group = parser.add_argument_group("Model configuration")
    group.add_argument("--arch", "-a", default="fconv", metavar="ARCH", required=True,
                       choices=ARCH_MODEL_REGISTRY.keys(), help="Model Architecture")
    return group


def _preimport_user_dir(input_args=None) -> None:
    probe = argparse.ArgumentParser(add_help=False, allow_abbrev=False)
    probe.add_argument("--user-dir", default=None)
    known, _ = probe.parse_known_args(input_args)
    import_user_module(known)


def get_parser(desc, default_task="test"):
    _preimport_user_dir()
    from unicore.registry import REGISTRIES
    from unicore.tasks import TASK_REGISTRY

    parser = argparse.ArgumentParser(allow_abbrev=False)
    _add_rows(parser, _global_rows())
    for key, reg in REGISTRIES.items():
        parser.add_argument("--" + key.replace("_", "-"), default=reg["default"], choices=reg["registry"].keys())
    parser.add_argument("--task", metavar="TASK", default=default_task, choices=TASK_REGISTRY.keys(), help="task")
    return parser


def get_training_parser(default_task="translation"):
    parser = get_parser("Trainer", default_task)
    add_dataset_args(parser, train=True)
    add_distributed_training_args(parser)
    add_model_args(parser)
    add_optimization_args(parser)
    add_checkpoint_args(parser)
    return parser


def get_validation_parser(default_task=None):
    parser = get_parser("Validation", default_task)
    add_dataset_args(parser, train=True)
    add_distributed_training_args(parser)
    add_common_eval_args(parser.add_argument_group("Evaluation"))
    return parser


# ------------------------------------------------------------------------------------------------
# two-pass parse
# ------------------------------------------------------------------------------------------------
def _parse_without_defaults(parser, input_args, parse_known):
    args = parse_args_and_arch(parser, input_args=input_args, parse_known=parse_known, suppress_defaults=False)
    if parse_known:
        args = args[0]
    shadow = argparse.ArgumentParser(add_help=False, parents=[parser])
    shadow.set_defaults(**{k: None for k in vars(args)})
    explicit = shadow.parse_args(input_args)
    return argparse.Namespace(**{k: v for k, v in vars(explicit).items() if v is not None})


def _postprocess(args) -> None:
    if getattr(args, "batch_size_valid", None) is None:
        args.batch_size_valid = getattr(args, "batch_size", None)
    args.bf16 = getattr(args, "bf16", False)
    if getattr(args, "seed", None) is None:
        args.seed = 1
        args.no_seed_provided = True
    else:
        args.no_seed_provided = False
    args.validate_with_ema = getattr(args, "validate_with_ema", False)


def parse_args_and_arch(
    parser: argparse.ArgumentParser,
    input_args: List[str] = None,
    parse_known: bool = False,
    suppress_defaults: bool = False,
    modify_parser: Optional[Callable[[argparse.ArgumentParser], None]] = None,
):
    """Parse ``input_args`` (default ``sys.argv``) with component-specific flags resolved.

    ``suppress_defaults`` returns only explicitly-given values; ``modify_parser`` lets callers
    change defaults before each pass (reference ``options.py:43-156``).
    """
    if suppress_defaults:
        return _parse_without_defaults(parser, input_args, parse_known)

    from unicore.models import ARCH_CONFIG_REGISTRY, ARCH_MODEL_REGISTRY, MODEL_REGISTRY
    from unicore.registry import REGISTRIES
    from unicore.tasks import TASK_REGISTRY

    _preimport_user_dir(input_args)
    if modify_parser is not None:
        modify_parser(parser)

    first, _ = parser.parse_known_args(input_args)

    if hasattr(first, "arch"):
        # SUPPRESS: model flags only materialise when given, so arch functions can fill the rest
        model_group = parser.add_argument_group("Model-specific configuration", argument_default=argparse.SUPPRESS)
        owner = ARCH_MODEL_REGISTRY.get(first.arch) or MODEL_REGISTRY.get(first.arch)
        if owner is None:
            raise RuntimeError("unknown architecture {!r}".format(first.arch))
        owner.add_args(model_group)
    if hasattr(first, "task"):
        TASK_REGISTRY[first.task].add_args(parser)
    for key, reg in REGISTRIES.items():
        choice = getattr(first, key, None)
        if choice is None:
            continue
        cls = reg["registry"][choice]
        if hasattr(cls, "add_args"):
            cls.add_args(parser)

    if modify_parser is not None:
        modify_parser(parser)

    extra = None
    if parse_known:
        args, extra = parser.parse_known_args(input_args)
    else:
        args = parser.parse_args(input_args)
    _postprocess(args)
    if hasattr(args, "arch") and args.arch in ARCH_CONFIG_REGISTRY:
        ARCH_CONFIG_REGISTRY[args.arch](args)
    return (args, extra) if parse_known else args
