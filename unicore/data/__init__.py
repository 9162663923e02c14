"""Data pipeline: datasets, wrappers, dictionary, batching and resumable iterators.

Exports the same names as the reference package (``unicore/data/__init__.py:9-34``).  The
reference keeps one class per module; here related classes share a module and the historic
module paths are registered as aliases so ``from unicore.data.pad_dataset import RightPadDataset``
style imports in downstream code keep working.
"""
import sys as _sys
import types as _types

from . import data_utils, iterators  # noqa: F401
from .base import BaseWrapperDataset, EpochListening, UnicoreDataset
from .dictionary import Dictionary
from .iterators import (
    BufferedIterator,
    CountingIterator,
    DevicePrefetcher,
    EpochBatchIterator,
    GroupedIterator,
    ShardedIterator,
)
from .masking import MaskTokensDataset
from .wrappers import (
    AppendTokenDataset,
    BertTokenizeDataset,
    EpochShuffleDataset,
    FromNumpyDataset,
    LeftPadDataset,
    LMDBDataset,
    LRUCacheDataset,
    NestedDictionaryDataset,
    NumelDataset,
    NumSamplesDataset,
    PackedSequenceDataset,
    PadDataset,
    PrependTokenDataset,
    RawArrayDataset,
    RawLabelDataset,
    RawNumpyDataset,
    RightPadDataset,
    RightPadDataset2D,
    SortDataset,
    TokenizeDataset,
)

__all__ = [
    "UnicoreDataset", "BaseWrapperDataset", "EpochListening", "Dictionary", "data_utils", "iterators",
    "AppendTokenDataset", "PrependTokenDataset", "TokenizeDataset", "BertTokenizeDataset",
    "MaskTokensDataset", "NestedDictionaryDataset", "NumelDataset", "NumSamplesDataset",
    "LeftPadDataset", "PadDataset", "PackedSequenceDataset", "RightPadDataset", "RightPadDataset2D", "LRUCacheDataset",
    "RawLabelDataset", "RawArrayDataset", "RawNumpyDataset", "LMDBDataset", "SortDataset",
    "EpochShuffleDataset", "FromNumpyDataset", "CountingIterator", "EpochBatchIterator",
    "GroupedIterator", "ShardedIterator", "BufferedIterator", "DevicePrefetcher",
]

# historic module path -> names it used to define
_LEGACY_MODULES = {
    "unicore_dataset": ["UnicoreDataset", "EpochListening"],
    "base_wrapper_dataset": ["BaseWrapperDataset"],
    "append_token_dataset": ["AppendTokenDataset"],
    "prepend_token_dataset": ["PrependTokenDataset"],
    "tokenize_dataset": ["TokenizeDataset"],
    "bert_tokenize_dataset": ["BertTokenizeDataset"],
    "mask_tokens_dataset": ["MaskTokensDataset"],
    "nested_dictionary_dataset": ["NestedDictionaryDataset"],
    "numel_dataset": ["NumelDataset"],
    "num_samples_dataset": ["NumSamplesDataset"],
    "pad_dataset": ["PadDataset", "LeftPadDataset", "RightPadDataset", "RightPadDataset2D"],
    "lru_cache_dataset": ["LRUCacheDataset"],
    "raw_dataset": ["RawLabelDataset", "RawArrayDataset", "RawNumpyDataset"],
    "lmdb_dataset": ["LMDBDataset"],
    "sort_dataset": ["SortDataset", "EpochShuffleDataset"],
    "from_numpy_dataset": ["FromNumpyDataset"],
}


def _install_legacy_modules():
    here = _sys.modules[__name__]
    for mod_name, names in _LEGACY_MODULES.items():
        full = __name__ + "." + mod_name
        if full in _sys.modules:
            continue
        alias = _types.ModuleType(full, "compatibility alias; see unicore.data")
        for n in names:
            setattr(alias, n, getattr(here, n))
        _sys.modules[full] = alias
        setattr(here, mod_name, alias)


_install_legacy_modules()
