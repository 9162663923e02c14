#!/usr/bin/env python3
"""``unicore-train``: train a registered model on one or many GPUs (one process per GPU).

Flow (reference ``unicore_cli/train.py``: ``cli_main:409`` -> ``call_main`` -> ``main:43`` ->
``train:178`` -> ``validate_and_save:251`` -> ``validate:337``): parse flags, start/join the
process group, build task/model/loss/Trainer, resume from ``checkpoint_last.pt`` when present and
loop over epochs; each update goes through ``Trainer.train_step``; validation/saving is decided
after every update (``--validate-interval[-updates]``, ``--save-interval[-updates]``, stop
conditions ``--max-update``, ``--max-epoch``, ``--stop-time-hours``, ``--stop-min-lr``,
``--patience``).  The loop is organised as a ``TrainingSession`` object instead of free functions
with function-attribute state.
"""
import argparse
import logging
import math
import os
import sys
from multiprocessing.pool import ThreadPool
from typing import Callable, Dict, List, Optional, Tuple

import numpy as np
import torch

if __package__ in (None, ""):  # started as a script from a source checkout: make the checkout importable
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from unicore import checkpoint_utils, options, tasks, utils
from unicore.data import iterators
from unicore.distributed import utils as distributed_utils
from unicore.logging import meters, metrics, progress_bar
from unicore.trainer import Trainer

logging.basicConfig(
    format="%(asctime)s | %(levelname)s | %(name)s | %(message)s",
    datefmt="%Y-%m-%d %H:%M:%S",
    level=os.environ.get("LOGLEVEL", "INFO").upper(),
    stream=sys.stdout,
)
logger = logging.getLogger("unicore_cli.train")


class EarlyStopper:
    """``--patience``: stop after N consecutive validations without improvement."""

    def __init__(self, patience: int, maximize: bool):
        self.patience = patience
        self.maximize = maximize
        self.best = None
        self.num_runs = 0

    def should_stop(self, valid_loss: Optional[float]) -> bool:
        if valid_loss is None or self.patience <= 0:
            return False
        improved = self.best is None or (valid_loss > self.best if self.maximize else valid_loss < self.best)
        if improved:
            self.best = valid_loss
            self.num_runs = 0
            return False
        self.num_runs += 1
        if self.num_runs >= self.patience:
            logger.info("early stop since valid performance hasn't improved for last {} runs".format(self.patience))
            return True
        return False


class TrainingSession:
    def __init__(self, args, trainer: Trainer, task, ckp_copy_thread):
        self.args = args
        self.trainer = trainer
        self.task = task
        self.ckp_copy_thread = ckp_copy_thread
        self.stopper = EarlyStopper(args.patience, args.maximize_best_checkpoint_metric)
        self.valid_subsets = args.valid_subset.split(",")

    # -- progress bars ------------------------------------------------------------------------------------
    def _bar(self, itr, epoch, prefix=None, master_only=True):
        args = self.args
        on_master = distributed_utils.is_master(args)
        return progress_bar.progress_bar(
            itr,
            log_format=args.log_format,
            log_interval=args.log_interval,
            epoch=epoch,
            prefix=prefix,
            tensorboard_logdir=(args.tensorboard_logdir if on_master else None),
            wandb_project=(args.wandb_project if on_master else None),
            wandb_name=(args.wandb_name if on_master else None),
            default_log_format=("tqdm" if not args.no_progress_bar else "simple"),
            args=args,
        )

    # -- one epoch ----------------------------------------------------------------------------------------
    @metrics.aggregate("train")
    def train_epoch(self, epoch_itr) -> Tuple[List[Optional[float]], bool]:
        args, trainer = self.args, self.trainer
        itr = epoch_itr.next_epoch_itr(
            fix_batches_to_gpus=args.fix_batches_to_gpus, shuffle=(epoch_itr.next_epoch_idx > args.curriculum)
        )
        update_freq = args.update_freq[min(epoch_itr.epoch, len(args.update_freq)) - 1]
        itr = iterators.GroupedIterator(itr, update_freq)
        progress = self._bar(itr, epoch_itr.epoch)
        trainer.begin_epoch(epoch_itr.epoch)

        valid_losses, should_stop = [None], False
        num_updates = trainer.get_num_updates()
        logger.info("Start iterating over samples")
        max_update = args.max_update or math.inf
        for i, samples in enumerate(progress):
            with metrics.aggregate("train_inner"), torch.autograd.profiler.record_function("train_step-%d" % i):
                log_output = trainer.train_step(samples)
            if log_output is not None:
                num_updates = trainer.get_num_updates()
                if num_updates % args.log_interval == 0:
                    stats = self._training_stats(metrics.get_smoothed_values("train_inner"))
                    progress.log(stats, tag="train_inner", step=num_updates)
                    metrics.reset_meters("train_inner")  # mid-epoch stats are per log window
            end_of_epoch = not itr.has_next()
            valid_losses, should_stop = self.validate_and_save(epoch_itr, end_of_epoch)
            if should_stop:
                break

        logger.info("end of epoch {} (average epoch stats below)".format(epoch_itr.epoch))
        stats = self._training_stats(metrics.get_smoothed_values("train"))
        progress.print(stats, tag="train", step=num_updates)
        metrics.reset_meters("train")
        return valid_losses, should_stop

    @staticmethod
    def _training_stats(stats: Dict) -> Dict:
        stats["wall"] = round(metrics.get_meter("default", "wall").elapsed_time, 0)
        return stats

    # -- validation / saving policy ----------------------------------------------------------------------
    def validate_and_save(self, epoch_itr, end_of_epoch: bool) -> Tuple[List[Optional[float]], bool]:
        args, trainer = self.args, self.trainer
        num_updates = trainer.get_num_updates()
        max_update = args.max_update or math.inf

        should_stop = False
        if num_updates >= max_update:
            should_stop = True
            logger.info(
                "Stopping training due to num_updates: {} >= max_update: {}".format(num_updates, max_update)
            )
        hours = trainer.cumulative_training_time() / (60 * 60)
        if args.stop_time_hours > 0 and hours > args.stop_time_hours:
            should_stop = True
            logger.info(
                "Stopping training due to cumulative_training_time: {} > stop_time_hours: {} hour(s)".format(
                    hours, args.stop_time_hours
                )
            )

        on_update_boundary = num_updates > 0
        do_save = (
            (end_of_epoch and epoch_itr.epoch % args.save_interval == 0 and not args.no_epoch_checkpoints)
            or should_stop
            or (
                args.save_interval_updates > 0
                and on_update_boundary
                and num_updates % args.save_interval_updates == 0
                and num_updates >= args.validate_after_updates
            )
        )
        do_validate = (
            (
                (not end_of_epoch and do_save)
                or (end_of_epoch and epoch_itr.epoch % args.validate_interval == 0 and not args.no_epoch_checkpoints)
                or should_stop
                or (
                    args.validate_interval_updates > 0
                    and on_update_boundary
                    and num_updates % args.validate_interval_updates == 0
                )
            )
            and not args.disable_validation
        )

        valid_losses = [None]
        if do_validate:
            with utils.validate_with_ema(trainer, ema=args.validate_with_ema):
                valid_losses = self.validate(epoch_itr)
        should_stop |= self.stopper.should_stop(valid_losses[0])
        checkpoint_utils.save_checkpoint(
            args, trainer, epoch_itr, valid_losses[0], self.ckp_copy_thread, do_save=(do_save or should_stop)
        )
        return valid_losses, should_stop

    def validate(self, epoch_itr) -> List[Optional[float]]:
        """Evaluate on every validation subset; returns the tracked metric per subset."""
        args, trainer, task = self.args, self.trainer, self.task
        seed = None
        if args.fixed_validation_seed is not None:
            seed = args.fixed_validation_seed  # same dropout/noise (if any) at every validation
        with utils.torch_seed(seed):
            trainer.begin_valid_epoch(epoch_itr.epoch)
            losses = []
            for subset in self.valid_subsets:
                logger.info('begin validation on "{}" subset'.format(subset))
                itr = trainer.get_valid_iterator(subset).next_epoch_itr(shuffle=False, set_dataset_epoch=False)
                progress = self._bar(itr, epoch_itr.epoch, prefix="valid on '{}' subset".format(subset))
                with metrics.aggregate(new_root=True) as agg:  # keep validation out of training meters
                    collected = []
                    for i, sample in enumerate(progress):
                        if args.max_valid_steps is not None and i > args.max_valid_steps:
                            break
                        collected.extend(trainer.valid_step(sample))
                    task.reduce_metrics(collected, trainer.get_loss(), subset)
                stats = self._valid_stats(agg.get_smoothed_values())
                progress.print(stats, tag=subset, step=trainer.get_num_updates())
                if args.best_checkpoint_metric in stats:
                    losses.append(stats[args.best_checkpoint_metric])
            return losses if losses else [None]

    def _valid_stats(self, stats: Dict) -> Dict:
        args = self.args
        stats["num_updates"] = self.trainer.get_num_updates()
        best = getattr(checkpoint_utils.save_checkpoint, "best", None)
        if best is not None and args.best_checkpoint_metric in stats:
            pick = max if args.maximize_best_checkpoint_metric else min
            stats["best_{}".format(args.best_checkpoint_metric)] = pick(best, stats[args.best_checkpoint_metric])
        return stats


def main(args) -> None:
    utils.set_deterministic(getattr(args, "deterministic", False))
    utils.import_user_module(args)
    utils.set_jit_fusion_options()
    if args.batch_size is None:
        raise ValueError("Must specify batch size with --batch-size")
    metrics.reset()

    np.random.seed(args.seed)
    torch.manual_seed(args.seed)
    if torch.cuda.is_available():
        torch.cuda.manual_seed(args.seed)

    ckp_copy_thread = None
    if distributed_utils.is_master(args):
        checkpoint_utils.verify_checkpoint_directory(args.save_dir)
        checkpoint_utils.verify_checkpoint_directory(args.tmp_save_dir)
        ckp_copy_thread = ThreadPool(processes=1)

    logger.info(args)
    task = tasks.setup_task(args)
    if not args.loss:
        raise ValueError("Please specify loss to train a model")
    model = task.build_model(args)
    loss = task.build_loss(args)
    if not args.disable_validation:
        for split in args.valid_subset.split(","):
            task.load_dataset(split, combine=False, epoch=1)

    logger.info(model)
    logger.info("task: {}".format(task.__class__.__name__))
    logger.info("model: {}".format(model.__class__.__name__))
    logger.info("loss: {}".format(loss.__class__.__name__))
    logger.info(
        "num. model params: {:,} (num. trained: {:,})".format(
            sum(p.numel() for p in model.parameters()),
            sum(p.numel() for p in model.parameters() if p.requires_grad),
        )
    )

    trainer = Trainer(args, task, model, loss)
    logger.info("training on {} devices (GPUs)".format(args.distributed_world_size))
    logger.info("batch size per device = {}".format(args.batch_size))

    extra_state, epoch_itr = checkpoint_utils.load_checkpoint(args, trainer, disable_iterator_cache=False)

    session = TrainingSession(args, trainer, task, ckp_copy_thread)
    max_epoch = args.max_epoch or math.inf
    lr = trainer.get_lr()
    stopwatch = meters.StopwatchMeter()
    stopwatch.start()
    while epoch_itr.next_epoch_idx <= max_epoch:
        if lr <= args.stop_min_lr:
            logger.info(
                "stopping training because current learning rate ({}) is smaller than or equal to minimum "
                "learning rate (--stop-min-lr={})".format(lr, args.stop_min_lr)
            )
            break
        valid_losses, should_stop = session.train_epoch(epoch_itr)
        if should_stop:
            break
        lr = trainer.lr_step(epoch_itr.epoch, valid_losses[0])  # first subset drives the schedule
        epoch_itr = trainer.get_train_iterator(
            epoch_itr.next_epoch_idx,
            load_dataset=task.has_sharded_data("train"),
            disable_iterator_cache=False,
        )
    stopwatch.stop()
    if ckp_copy_thread is not None:
        ckp_copy_thread.close()
        ckp_copy_thread.join()
    logger.info("done training in {:.1f} seconds".format(stopwatch.sum))


def cli_main(modify_parser: Optional[Callable[[argparse.ArgumentParser], None]] = None) -> None:
    parser = options.get_training_parser()
    args = options.parse_args_and_arch(parser, modify_parser=modify_parser)
    try:
        if args.profile:
            with torch.cuda.profiler.profile():
                with torch.autograd.profiler.emit_nvtx():
                    distributed_utils.call_main(args, main)
        else:
            distributed_utils.call_main(args, main)
    finally:
        if torch.distributed.is_available() and torch.distributed.is_initialized():
            try:
                torch.distributed.barrier()
            finally:
                torch.distributed.destroy_process_group()


if __name__ == "__main__":
    cli_main()
