"""Composable dataset wrappers (token edits, padding/collation, ordering, bookkeeping, storage).

One module instead of the reference's one-class-per-file layout; the old module paths
(``unicore.data.pad_dataset`` ...) are aliased in ``unicore/data/__init__.py``.  Behavioural
parity per class is cited inline (paths relative to ``/root/reference/unicore/data``).
A tiny per-instance memo (``_Memo``) replaces the reference's ``functools.lru_cache`` on bound
methods (which keeps datasets alive globally and breaks on unhashable args - SURVEY D13).
"""
import logging
import os
import pickle
from collections import OrderedDict

import numpy as np
import torch
from torch.utils.data import default_collate

from . import data_utils
from .base import BaseWrapperDataset, UnicoreDataset
from .dictionary import Dictionary
from .record_store import RecordStoreReader, is_record_store

logger = logging.getLogger(__name__)


class _Memo:
    """Bounded per-instance LRU keyed by item index (picklable: dropped on pickling)."""

    def __init__(self, capacity=16):
        self.capacity = capacity
        self.store = OrderedDict()

    def get(self, key, producer):
        hit = self.store.get(key, self)
        if hit is not self:
            self.store.move_to_end(key)
            return hit
        value = producer(key)
        self.store[key] = value
        if len(self.store) > self.capacity:
            self.store.popitem(last=False)
        return value

    def __getstate__(self):
        return {"capacity": self.capacity}

    def __setstate__(self, state):
        self.capacity = state["capacity"]
        self.store = OrderedDict()


# ------------------------------------------------------------------------------------------------
# token-level edits
# ------------------------------------------------------------------------------------------------
class AppendTokenDataset(BaseWrapperDataset):
    """item -> [item, token] (``append_token_dataset.py:14``)."""

    def __init__(self, dataset, token=None):
        super().__init__(dataset)
        self.token = token
        self._memo = _Memo()

    def _build(self, idx):
        item = self.dataset[idx]
        if self.token is None:
            return item
        tail = torch.full_like(item[0], self.token).unsqueeze(0)
        return torch.cat([item, tail], dim=0)

    def __getitem__(self, idx):
        return self._memo.get(idx, self._build)


class PrependTokenDataset(BaseWrapperDataset):
    """item -> [token, item] (``prepend_token_dataset.py:14``)."""

    def __init__(self, dataset, token=None):
        super().__init__(dataset)
        self.token = token
        self._memo = _Memo()

    def _build(self, idx):
        item = self.dataset[idx]
        if self.token is None:
            return item
        head = torch.full_like(item[0], self.token).unsqueeze(0)
        return torch.cat([head, item], dim=0)

    def __getitem__(self, idx):
        return self._memo.get(idx, self._build)


class TokenizeDataset(BaseWrapperDataset):
    """Sequence of symbols -> LongTensor of dictionary indices (``tokenize_dataset.py:13``)."""

    def __init__(self, dataset, dictionary: Dictionary, max_seq_len: int = 512):
        super().__init__(dataset)
        self.dictionary = dictionary
        self.max_seq_len = max_seq_len
        self._memo = _Memo()

    def _build(self, index):
        raw = self.dataset[index]
        if not (0 < len(raw) < self.max_seq_len):
            raise ValueError("sequence length {} outside (0, {})".format(len(raw), self.max_seq_len))
        return torch.from_numpy(self.dictionary.vec_index(raw)).long()

    def __getitem__(self, index):
        return self._memo.get(index, self._build)


class BertTokenizeDataset(BaseWrapperDataset):
    """Raw text -> WordPiece ids via HF ``tokenizers`` (``bert_tokenize_dataset.py:14``);
    the tokenizer package is imported lazily so ``import unicore`` never needs it."""

    def __init__(self, dataset, dict_path: str, max_seq_len: int = 512):
        super().__init__(dataset)
        from tokenizers import BertWordPieceTokenizer

        self.tokenizer = BertWordPieceTokenizer(dict_path, lowercase=True)
        self.max_seq_len = max_seq_len

    @property
    def can_reuse_epoch_itr_across_epochs(self):
        return True

    def __getitem__(self, index: int):
        text = self.dataset[index].replace("<unk>", "[UNK]")
        ids = torch.tensor(self.tokenizer.encode(text).ids, dtype=torch.long)
        return ids[: self.max_seq_len]


# ------------------------------------------------------------------------------------------------
# padding collaters
# ------------------------------------------------------------------------------------------------
class PadDataset(BaseWrapperDataset):
    """Collate 1-D items into ``[B, T]`` padded to a multiple of 8 (``pad_dataset.py:12-19``)."""

    pad_to_multiple = 8

    def __init__(self, dataset, pad_idx, left_pad):
        super().__init__(dataset)
        self.pad_idx = pad_idx
        self.left_pad = left_pad

    def collater(self, samples):
        return data_utils.collate_tokens(
            samples, self.pad_idx, left_pad=self.left_pad, pad_to_multiple=self.pad_to_multiple
        )


class LeftPadDataset(PadDataset):
    def __init__(self, dataset, pad_idx):
        super().__init__(dataset, pad_idx, left_pad=True)


class RightPadDataset(PadDataset):
    def __init__(self, dataset, pad_idx):
        super().__init__(dataset, pad_idx, left_pad=False)


class PackedSequenceDataset(BaseWrapperDataset):
    """Collate 1-D items back to back, without padding: ``[N]`` with N the total length.  With ``tokens_key`` the
    batch is ``{tokens_key: [N], "cu_seqlens": int32 [B + 1] (the cumulative lengths), "max_seqlen": int}``, the
    ``net_input`` of a model that runs packed sequences; ``max_seqlen`` is the longest length rounded up to a
    multiple of 8, the width ``RightPadDataset`` pads the same batch to.  Without it the batch is the ``[N]`` tensor
    alone (the targets that go with such an input).  Every value is known on the host at collate time."""

    pad_to_multiple = 8

    def __init__(self, dataset, tokens_key=None):
        super().__init__(dataset)
        self.tokens_key = tokens_key

    def collater(self, samples):
        tokens = torch.cat(list(samples))
        if self.tokens_key is None:
            return tokens
        lens = torch.tensor([0] + [len(s) for s in samples], dtype=torch.int64)
        longest = int(lens.max())
        return {
            self.tokens_key: tokens,
            "cu_seqlens": lens.cumsum(0).to(torch.int32),
            "max_seqlen": longest + (-longest % self.pad_to_multiple),
        }


class RightPadDataset2D(BaseWrapperDataset):
    """Collate square pair tensors into ``[B, T, T]`` (``pad_dataset.py:32-38``)."""

    pad_to_multiple = 8

    def __init__(self, dataset, pad_idx, left_pad=False):
        super().__init__(dataset)
        self.pad_idx = pad_idx
        self.left_pad = left_pad

    def collater(self, samples):
        return data_utils.collate_tokens_2d(
            samples, self.pad_idx, left_pad=self.left_pad, pad_to_multiple=self.pad_to_multiple
        )


# ------------------------------------------------------------------------------------------------
# ordering
# ------------------------------------------------------------------------------------------------
class SortDataset(BaseWrapperDataset):
    """Order items by ``np.lexsort(sort_order)`` (last key is primary; ``sort_dataset.py:12``)."""

    def __init__(self, dataset, sort_order):
        super().__init__(dataset)
        if not isinstance(sort_order, (list, tuple)):
            sort_order = [sort_order]
        for key in sort_order:
            if len(key) != len(dataset):
                raise ValueError("sort key length {} != dataset length {}".format(len(key), len(dataset)))
        self.sort_order = sort_order

    def ordered_indices(self):
        return np.lexsort(self.sort_order)


class EpochShuffleDataset(BaseWrapperDataset):
    """A fresh permutation every epoch, seeded by ``seed + epoch - 1`` (``sort_dataset.py:25``)."""

    def __init__(self, dataset, size, seed):
        super().__init__(dataset)
        self.size = size
        self.seed = seed
        self.set_epoch(1)

    def set_epoch(self, epoch):
        super().set_epoch(epoch)
        with data_utils.numpy_seed(self.seed + epoch - 1):
            self.sort_order = np.random.permutation(self.size)

    def ordered_indices(self):
        return self.sort_order

    @property
    def can_reuse_epoch_itr_across_epochs(self):
        return False


# ------------------------------------------------------------------------------------------------
# bookkeeping
# ------------------------------------------------------------------------------------------------
class NumelDataset(BaseWrapperDataset):
    """Item -> its element count; batch -> tensor of counts or their sum (``numel_dataset.py:13``)."""

    def __init__(self, dataset, reduce=False):
        super().__init__(dataset)
        self.reduce = reduce

    def __getitem__(self, index):
        item = self.dataset[index]
        return torch.numel(item) if torch.is_tensor(item) else np.size(item)

    def collater(self, samples):
        return sum(samples) if self.reduce else torch.tensor(samples)


class NumSamplesDataset(UnicoreDataset):
    """Every item is 1; a batch collates to its size (``num_samples_dataset.py:10``)."""

    def __getitem__(self, index):
        return 1

    def __len__(self):
        return 0

    def collater(self, samples):
        return sum(samples)


class LRUCacheDataset(BaseWrapperDataset):
    """Memoise the last few items of the wrapped dataset (``lru_cache_dataset.py:12``)."""

    def __init__(self, dataset, token=None):
        super().__init__(dataset)
        self._memo = _Memo()

    def set_epoch(self, epoch):
        super().set_epoch(epoch)
        self._memo.store.clear()  # items may be epoch dependent (e.g. masking noise)

    def __getitem__(self, index):
        return self._memo.get(index, lambda i: self.dataset[i])


# ------------------------------------------------------------------------------------------------
# in-memory sources
# ------------------------------------------------------------------------------------------------
class FromNumpyDataset(BaseWrapperDataset):
    """numpy item -> tensor (``from_numpy_dataset.py:11``)."""

    def __init__(self, dataset):
        super().__init__(dataset)
        self._memo = _Memo()

    def __getitem__(self, idx):
        return self._memo.get(idx, lambda i: torch.from_numpy(self.dataset[i]))


class RawLabelDataset(UnicoreDataset):
    """Plain python labels; batch -> ``torch.tensor`` (``raw_dataset.py:11``)."""

    def __init__(self, labels):
        super().__init__()
        self.labels = labels

    def __getitem__(self, index):
        return self.labels[index]

    def __len__(self):
        return len(self.labels)

    def collater(self, samples):
        return torch.tensor(samples)


class RawArrayDataset(UnicoreDataset):
    """Any indexable; default-collated unless the source has a collater (``raw_dataset.py:27``)."""

    def __init__(self, dataset):
        super().__init__()
        self.dataset = dataset

    def __getitem__(self, index):
        return self.dataset[index]

    def __len__(self):
        return len(self.dataset)

    def collater(self, samples):
        inner = getattr(self.dataset, "collater", None)
        return inner(samples) if inner is not None else default_collate(samples)


class RawNumpyDataset(RawArrayDataset):
    """Like ``RawArrayDataset`` but converts numpy items to tensors (``raw_dataset.py:47``)."""

    def __getitem__(self, index):
        return torch.from_numpy(self.dataset[index])


# ------------------------------------------------------------------------------------------------
# on-disk source
# ------------------------------------------------------------------------------------------------
class LMDBDataset:
    """Pickled records in a single-file LMDB (``lmdb_dataset.py:16``).

    ``lmdb`` is imported on first use, so the package imports without it (SURVEY D3). The
    environment handle is opened lazily per process, which keeps the object picklable for
    DataLoader workers.  Files written by ``unicore.data.record_store`` (the dependency-free
    fallback format) are recognised by their magic and read through a memory map instead.
    """

    def __init__(self, db_path):
        self.db_path = db_path
        if not os.path.isfile(db_path):
            raise FileNotFoundError("{} not found".format(db_path))
        self._store = RecordStoreReader(db_path) if is_record_store(db_path) else None
        if self._store is None:
            with self._open().begin() as txn:
                self._keys = list(txn.cursor().iternext(values=False))
        else:
            self._keys = range(len(self._store))
        self._memo = _Memo()

    def _open(self):
        try:
            import lmdb
        except ImportError as e:
            raise ImportError(
                "{} is an LMDB file but the `lmdb` package is not installed; install it or rewrite the corpus "
                "with unicore.data.record_store.RecordStoreWriter".format(self.db_path)
            ) from e
        return lmdb.open(
            self.db_path, subdir=False, readonly=True, lock=False, readahead=False, meminit=False, max_readers=256
        )

    def connect_db(self, lmdb_path=None, save_to_self=False):
        """Open the environment; keep it on the instance when ``save_to_self`` (``lmdb_dataset.py:26``)."""
        if lmdb_path is not None:
            self.db_path = lmdb_path
        env = self._open()
        if save_to_self:
            self.env = env
            return None
        return env

    def __len__(self):
        return len(self._keys)

    def _read(self, idx):
        if self._store is not None:
            return self._store[idx]
        if self.__dict__.get("env") is None:
            self.connect_db(save_to_self=True)
        return pickle.loads(self.env.begin().get(self._keys[idx]))

    def __getitem__(self, idx):
        return self._memo.get(idx, self._read)

    def __getstate__(self):
        state = dict(self.__dict__)
        state.pop("env", None)
        return state


# ------------------------------------------------------------------------------------------------
# nested dictionaries of datasets
# ------------------------------------------------------------------------------------------------
def _flatten(tree, prefix=None):
    """{'a': {'b': x}, 'c': [y, z]} -> {'a.b': x, 'c.[0]': y, 'c.[1]': z}"""
    flat = OrderedDict()
    if isinstance(tree, dict):
        prefix = prefix + "." if prefix is not None else ""
        for k, v in tree.items():
            if v is None:
                continue
            flat.update(_flatten(v, prefix + k))
    elif isinstance(tree, list):
        for i, v in enumerate(tree):
            flat.update(_flatten(v, "{}.[{}]".format(prefix, i)))
    else:
        flat[prefix] = tree
    return flat


def _unflatten(flat):
    tree = OrderedDict()
    for path, value in flat.items():
        parts = path.split(".")
        node = tree
        for part in parts[:-1]:
            if part.startswith("[") and part.endswith("]"):
                part = int(part[1:-1])
            node = node.setdefault(part, OrderedDict())
        node[parts[-1]] = value
    return tree


class NestedDictionaryDataset(UnicoreDataset):
    """A (nested) dict of equally long datasets presented as one dataset whose batches are nested
    dicts collated leaf by leaf (``nested_dictionary_dataset.py:48``)."""

    def __init__(self, defn):
        super().__init__()
        self.defn = _flatten(defn)
        anchor = None
        for leaf in self.defn.values():
            if not isinstance(leaf, (UnicoreDataset, torch.utils.data.Dataset)):
                raise ValueError("Expected Dataset but found: {}".format(leaf.__class__))
            anchor = anchor or leaf
            if len(leaf) > 0 and len(leaf) != len(anchor):
                raise ValueError("dataset lengths must match")
        self._len = len(anchor)

    def __getitem__(self, index):
        return OrderedDict((k, ds[index]) for k, ds in self.defn.items())

    def __len__(self):
        return self._len

    def collater(self, samples):
        if len(samples) == 0:
            return {}
        batch = OrderedDict()
        for key, ds in self.defn.items():
            column = [s[key] for s in samples]
            try:
                batch[key] = ds.collater(column)
            except NotImplementedError:
                batch[key] = default_collate(column)
        return _unflatten(batch)

    @property
    def supports_prefetch(self):
        return any(getattr(ds, "supports_prefetch", False) for ds in self.defn.values())

    def prefetch(self, indices):
        for ds in self.defn.values():
            if getattr(ds, "supports_prefetch", False):
                ds.prefetch(indices)

    @property
    def can_reuse_epoch_itr_across_epochs(self):
        return all(ds.can_reuse_epoch_itr_across_epochs for ds in self.defn.values())

    def set_epoch(self, epoch):
        super().set_epoch(epoch)
        for ds in self.defn.values():
            ds.set_epoch(epoch)
