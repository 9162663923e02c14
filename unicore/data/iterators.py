"""Epoch/batch iteration: counting, sharding, grouping, background prefetch, resumable epochs.

Parity: reference ``unicore/data/iterators.py`` (``CountingIterator:28``,
``EpochBatchIterator:151`` incl. ``state_dict:311`` / ``load_state_dict:326`` with position
re-scaling, ``GroupedIterator:406``, ``ShardedIterator:438``, ``BufferedIterator:496``).

Design difference: the reference's "GPU-CPU overlapping" loader only overlaps *collation*
(SURVEY D19 - batches stay pageable so the H2D copy is synchronous).  ``BufferedIterator`` here
can page-lock each prefetched batch in its producer thread (``pin_memory=True``) so that the
trainer's ``non_blocking`` copy is a real async DMA, and ``DevicePrefetcher`` stages the next
batch on a side CUDA stream while the current step computes.
"""
import itertools
import logging
import math
import os
import queue
import threading
import time

import numpy as np
import torch

from . import data_utils

logger = logging.getLogger(__name__)

_END = object()  # sentinel placed in the prefetch queue when the source is exhausted


class CountingIterator(object):
    """An iterator that keeps score: ``n`` items handed out so far out of ``total``.

    ``start`` lets a resumed iterator begin its count where the interrupted one stopped; a source that produces more
    than ``total`` items is a bug upstream (different sharding than the checkpoint) and is reported as such."""

    _TOO_LONG = (
        "Mismatch between actual and expected iterable length. This may be caused by resuming training from a "
        "checkpoint using a different number of GPUs, in which case you can try the --reset-dataloader option. "
        "Alternatively you may have a train or validation set that is smaller than the number of GPUs. If none of "
        "these apply, please report this."
    )

    def __init__(self, iterable, start=None, total=None):
        self.iterable = iterable
        self.n = getattr(iterable, "n", 0) if start is None else start
        self.total = self.n + len(iterable) if total is None else total
        self._stream = self._counted()

    def _counted(self):
        for item in self.iterable:
            if self.n >= self.total:
                raise RuntimeError(self._TOO_LONG)
            self.n += 1
            yield item

    def __iter__(self):
        return self._stream

    def __next__(self):
        return next(self._stream)

    def __len__(self):
        return self.total

    def has_next(self):
        return self.n < self.total

    def skip(self, num_to_skip):
        for _ in itertools.islice(self._stream, num_to_skip):
            pass
        return self

    def take(self, n):
        """Stop after ``n`` items in total (counting the ones already consumed)."""
        self.total = min(self.total, n)
        remaining = max(n - self.n, 0)
        if hasattr(self.iterable, "take"):
            self.iterable.take(remaining)
        else:
            self.iterable = itertools.islice(self.iterable, remaining)
        return self


class EpochBatchIterating(object):
    """Interface of multi-epoch batch iterators (what the trainer and the CLI rely on)."""

    def __len__(self) -> int:
        raise NotImplementedError

    @property
    def next_epoch_idx(self):
        raise NotImplementedError

    def next_epoch_itr(self, shuffle=True, fix_batches_to_gpus=False, set_dataset_epoch=True):
        raise NotImplementedError

    def end_of_epoch(self) -> bool:
        raise NotImplementedError

    @property
    def iterations_in_epoch(self) -> int:
        raise NotImplementedError

    def state_dict(self):
        raise NotImplementedError

    def load_state_dict(self, state_dict):
        raise NotImplementedError

    @property
    def first_batch(self):
        return "DUMMY"


class EpochBatchIterator(EpochBatchIterating):
    """Epoch after epoch over one fixed list of batches (lists of dataset indices).

    An epoch's order is a pure function of ``(seed, epoch)``: the batch list is shuffled with ``seed + epoch``, rank
    ``shard_id`` takes every ``num_shards``-th entry (a short shard is completed with empty batches so that all ranks
    step in lockstep), and the index lists drive a ``DataLoader``.  That makes the position checkpointable as two
    numbers - epoch and batches consumed - and restorable into a run with a different world size (the position is
    rescaled by the ratio of the shard lengths).
    """

    def __init__(self, dataset, collate_fn, batch_sampler, seed=1, num_shards=1, shard_id=0, num_workers=0, epoch=1,
                 buffer_size=0, timeout=0, disable_shuffling=False, pin_memory=False):
        if not isinstance(dataset, torch.utils.data.Dataset):
            raise TypeError("dataset must be a torch Dataset")
        self.dataset, self.collate_fn, self.batch_sampler = dataset, collate_fn, batch_sampler
        self.seed, self.num_shards, self.shard_id = seed, num_shards, shard_id
        self.num_workers, self.timeout, self.pin_memory = num_workers, timeout, pin_memory
        self.buffer_size = min(buffer_size, 32)  # politeness cap on shared hosts
        self.disable_shuffling = disable_shuffling
        self.shuffle = not disable_shuffling
        self.epoch = max(epoch, 1)  # epochs count from 1
        # a callable sampler is asked again every epoch; a plain list is frozen once
        self._batches = None if callable(batch_sampler) else tuple(batch_sampler)
        self._running = None   # the iterator of the epoch in progress
        self._restored = None  # an iterator prepared by load_state_dict, handed out by the next next_epoch_itr()
        self._prefetching_dataset = getattr(dataset, "supports_prefetch", False)

    # ---- the batch list ---------------------------------------------------------------------------------------
    @property
    def frozen_batches(self):
        if self._batches is None:
            self._batches = tuple(self.batch_sampler(self.dataset, self.epoch))
        return self._batches

    @property
    def first_batch(self):
        batches = self.frozen_batches
        if not batches:
            raise Exception(
                "The dataset is empty. This could indicate that all elements in the dataset have been skipped. "
                "Try increasing the max number of allowed tokens or using a larger dataset."
            )
        if not getattr(self.dataset, "supports_fetch_outside_dataloader", True):
            return "DUMMY"
        return self.collate_fn([self.dataset[i] for i in batches[0]])

    def __len__(self):
        return -(-len(self.frozen_batches) // self.num_shards)

    # ---- position ---------------------------------------------------------------------------------------------------
    @property
    def iterations_in_epoch(self):
        active = self._running if self._running is not None else self._restored
        return 0 if active is None else active.n

    n = iterations_in_epoch

    def end_of_epoch(self) -> bool:
        return not self._running.has_next()

    @property
    def next_epoch_idx(self):
        if self._restored is None and self._running is not None and self.end_of_epoch():
            return self.epoch + 1
        return self.epoch

    def next_epoch_itr(self, shuffle=True, fix_batches_to_gpus=False, set_dataset_epoch=True):
        shuffle = shuffle and not self.disable_shuffling
        self.epoch = self.next_epoch_idx
        if set_dataset_epoch and hasattr(self.dataset, "set_epoch"):
            self.dataset.set_epoch(self.epoch)
        if self._restored is not None:
            self._running, self._restored = self._restored, None
        else:
            if callable(self.batch_sampler):
                self._batches = None  # new epoch, new sample of batches
            self._running = self._get_iterator_for_epoch(self.epoch, shuffle, fix_batches_to_gpus=fix_batches_to_gpus)
        self.shuffle = shuffle
        return self._running

    # ---- checkpointing ------------------------------------------------------------------------------------------
    def state_dict(self):
        done = self.end_of_epoch()
        return {
            "epoch": self.epoch + (1 if done else 0),
            "iterations_in_epoch": 0 if done else self.iterations_in_epoch,
            "shuffle": self.shuffle,
            "len": len(self),
        }

    def load_state_dict(self, state_dict):
        self.epoch = state_dict["epoch"]
        self._restored = None
        consumed = state_dict.get("iterations_in_epoch", 0)
        if consumed <= 0:
            return
        then, now = state_dict.get("len", None), len(self)
        if then is not None and then != now:
            rescaled = int(consumed * now / then)
            logger.info(
                "Iterator size changed ({} -> {}; different world size or update_freq?). "
                "Position rescaled from {} to {}.".format(then, now, consumed, rescaled)
            )
            consumed = rescaled
        self._restored = self._get_iterator_for_epoch(self.epoch, shuffle=state_dict.get("shuffle", True), offset=consumed)
        if self._restored is None:
            raise RuntimeError(
                "Cannot resume training due to dataloader mismatch. You can relaunch "
                "training with `--reset-dataloader` and it should work."
            )

    # ---- one epoch ------------------------------------------------------------------------------------------------
    def _epoch_order(self, epoch, shuffle, fix_batches_to_gpus):
        """This rank's batches of ``epoch``, in order."""

        def shuffled(seq, seed):
            seq = list(seq)
            with data_utils.numpy_seed(seed):
                np.random.shuffle(seq)
            return seq

        def my_share(seq):
            return list(ShardedIterator(seq, self.num_shards, self.shard_id, fill_value=[]))

        batches = self.frozen_batches
        if not self._prefetching_dataset:
            return my_share(shuffled(batches, self.seed + epoch) if shuffle else batches)
        # datasets that load ahead of time: decide the shard first, tell the dataset what it will be asked for, and only
        # then (optionally) reorder within the shard so that a rank keeps "its" batches across epochs
        if shuffle and not fix_batches_to_gpus:
            batches = shuffled(batches, self.seed + epoch)
        mine = my_share(batches)
        self.dataset.prefetch([i for batch in mine for i in batch])
        if shuffle and fix_batches_to_gpus:
            mine = shuffled(mine, self.seed + epoch + self.shard_id)
        return mine

    def _get_iterator_for_epoch(self, epoch, shuffle, fix_batches_to_gpus=False, offset=0):
        order = self._epoch_order(epoch, shuffle, fix_batches_to_gpus)
        if 0 < offset and len(order) <= offset:
            return None
        if self.num_workers > 0:
            os.environ["PYTHONWARNINGS"] = "ignore:semaphore_tracker:UserWarning"
        loader = torch.utils.data.DataLoader(self.dataset, collate_fn=self.collate_fn, batch_sampler=order[offset:],
                                             num_workers=self.num_workers, timeout=self.timeout)
        if self.buffer_size > 0:
            loader = BufferedIterator(self.buffer_size, loader, pin_memory=self.pin_memory)
        return CountingIterator(loader, start=offset)


class GroupedIterator(CountingIterator):
    """Yield lists of ``chunk_size`` consecutive items (the micro-batches of one update)."""

    def __init__(self, iterable, chunk_size):
        def chunks():
            it = iter(iterable)
            while True:
                group = list(itertools.islice(it, chunk_size))
                if not group:
                    return
                yield group

        super().__init__(
            chunks(),
            start=int(math.ceil(getattr(iterable, "n", 0) / float(chunk_size))),
            total=int(math.ceil(len(iterable) / float(chunk_size))),
        )
        self.chunk_size = chunk_size


class ShardedIterator(CountingIterator):
    """Every ``num_shards``-th item starting at ``shard_id``; all shards have equal length
    (``ceil(len/num_shards)``), short ones are completed with ``fill_value``."""

    def __init__(self, iterable, num_shards, shard_id, fill_value=None):
        if not 0 <= shard_id < num_shards:
            raise ValueError("shard_id must be between 0 and num_shards")
        sharded_len = int(math.ceil(len(iterable) / float(num_shards)))
        picked = itertools.islice(iterable, shard_id, len(iterable), num_shards)
        padded = itertools.chain(picked, itertools.repeat(fill_value))
        super().__init__(
            itertools.islice(padded, sharded_len),
            start=int(math.ceil(getattr(iterable, "n", 0) / float(num_shards))),
            total=sharded_len,
        )


class BackgroundConsumer(threading.Thread):
    """Daemon thread: pulls items from ``source`` into ``out_queue`` (optionally pinning them)."""

    def __init__(self, out_queue, source, max_len, pin_memory=False):
        super().__init__(daemon=True)
        self._queue = out_queue
        self._source = source
        self._max_len = max_len
        self._pin = pin_memory and torch.cuda.is_available()
        self.count = 0

    def run(self):
        from unicore import utils

        try:
            for item in self._source:
                if self._pin:
                    item = utils.pin_sample(item)
                self._queue.put(item)
                self.count += 1
                if self._max_len is not None and self.count >= self._max_len:
                    break
            self._queue.put(_END)
        except Exception as exc:  # noqa: BLE001 - hand the failure to the consumer thread
            self._queue.put(exc)


class BufferedIterator(object):
    """Prefetch up to ``size`` collated batches in a background thread."""

    def __init__(self, size, iterable, pin_memory=False):
        self._queue = queue.Queue(size)
        self._iterable = iterable
        self._consumer = None
        self._pin_memory = pin_memory
        self.start_time = time.time()
        self.warning_time = None
        self.total = len(iterable)

    def _start(self):
        self._consumer = BackgroundConsumer(self._queue, self._iterable, self.total, self._pin_memory)
        self._consumer.start()

    def __iter__(self):
        return self

    def __len__(self):
        return self.total

    def take(self, n):
        self.total = min(self.total, n)
        if hasattr(self._iterable, "take"):
            self._iterable.take(n)
        return self

    def __next__(self):
        if self._consumer is None:
            self._start()
        # tell the user (at most every 15 min) when the input pipeline is the bottleneck
        if self._queue.qsize() < min(2, max(1, self._queue.maxsize // 2)):
            now = time.time()
            if now - self.start_time > 5 * 60 and (self.warning_time is None or now - self.warning_time > 15 * 60):
                logger.debug(
                    "Data loading buffer is empty or nearly empty. This may indicate a data loading "
                    "bottleneck, and increasing the number of workers (--num-workers) may help."
                )
                self.warning_time = now
        item = self._queue.get(True)
        if isinstance(item, Exception):
            raise item
        if item is _END:
            raise StopIteration()
        return item


class DevicePrefetcher(object):
    """Stage batch *i+1* on the device (side stream) while batch *i* is being consumed.

    Wraps any iterator of (nested) CPU samples; yields samples whose tensors already live on
    ``device``.  With pinned sources the copy is a true async DMA; the consumer stream waits on
    a CUDA event, never on the host.
    """

    def __init__(self, iterable, device=None):
        self._iterable = iterable
        self._device = device if device is not None else torch.cuda.current_device()
        self._stream = torch.cuda.Stream(device=self._device)

    def __len__(self):
        return len(self._iterable)

    def _stage(self, sample):
        from unicore import utils

        with torch.cuda.stream(self._stream):
            moved = utils.move_to_cuda(sample, device=self._device)
        event = torch.cuda.Event()
        event.record(self._stream)
        return moved, event

    def __iter__(self):
        from unicore import utils

        it = iter(self._iterable)
        try:
            staged = self._stage(next(it))
        except StopIteration:
            return
        for nxt in it:
            ready, event = staged
            staged = self._stage(nxt)
            torch.cuda.current_stream().wait_event(event)
            utils.apply_to_sample(lambda t: t.record_stream(torch.cuda.current_stream()), ready)
            yield ready
        ready, event = staged
        torch.cuda.current_stream().wait_event(event)
        utils.apply_to_sample(lambda t: t.record_stream(torch.cuda.current_stream()), ready)
        yield ready
