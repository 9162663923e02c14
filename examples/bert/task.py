"""``--task bert``: masked-language-model pre-training on a corpus of raw text lines.

Data directory layout (that of the reference example, ``examples/bert/task.py:31-124`` there, so existing corpora work
unchanged): ``dict.txt`` - one WordPiece per line - and one record file per split, ``<split>.lmdb`` (or the
dependency-free ``<split>.rec`` written by ``example_data/prepare_data.py --format records``).

The pipeline is a chain of lazy dataset views, each adding one thing:

    records -> WordPiece ids (truncated to --max-seq-len) -> (masked input, targets at the masked positions)
            -> right-padded batches {"net_input": {"src_tokens"}, "target"} -> one fixed random order

``--pack-sequences`` collates the same sentences back to back instead of right-padding them: ``src_tokens`` and
``target`` are ``[N]`` (N the real tokens of the batch), and ``net_input`` also holds ``cu_seqlens`` and
``max_seqlen`` (``PackedSequenceDataset``), so that no kernel of the model runs on pad rows.  The model follows the
form of the batch it is given; checkpoints are the same either way.

Masking follows BERT: ``--mask-prob`` of the positions are selected; of those ``--random-token-prob`` become a random
token, ``--leave-unmasked-prob`` stay as they are, the rest become ``[MASK]``; the draw is a function of (seed, epoch,
index), i.e. reproducible and different every epoch.
"""
import logging
import os

import numpy as np

from unicore import data as D
from unicore.tasks import UnicoreTask, register_task

logger = logging.getLogger(__name__)

VOCAB_FILE = "dict.txt"


@register_task("bert")
class BertTask(UnicoreTask):
    @staticmethod
    def add_args(parser):
        parser.add_argument("data", help="directory with dict.txt and <split>.lmdb files")
        masking = parser.add_argument_group("BERT masking")
        masking.add_argument("--mask-prob", type=float, default=0.15,
                             help="probability of replacing a token with mask")
        masking.add_argument("--leave-unmasked-prob", type=float, default=0.1,
                             help="probability that a masked token is unmasked")
        masking.add_argument("--random-token-prob", type=float, default=0.1,
                             help="probability of replacing a token with a random token")
        parser.add_argument("--pack-sequences", action="store_true", default=False,
                            help="batch the sentences back to back with cu_seqlens instead of right-padding them")

    @classmethod
    def setup_task(cls, args, **kwargs):
        vocab = D.Dictionary.load(os.path.join(args.data, VOCAB_FILE))
        logger.info("dictionary: {} types".format(len(vocab)))
        return cls(args, vocab)

    def __init__(self, args, dictionary):
        super().__init__(args)
        self.dictionary = dictionary
        self.seed = args.seed
        # the mask symbol is part of the model's vocabulary: registered before the model is built
        self.mask_idx = dictionary.add_symbol("[MASK]", is_special=True)

    def _token_ids(self, split):
        root = self.args.data
        lines = D.LMDBDataset(os.path.join(root, split + ".lmdb"))
        return D.BertTokenizeDataset(lines, os.path.join(root, VOCAB_FILE), max_seq_len=self.args.max_seq_len)

    def load_dataset(self, split, combine=False, **kwargs):
        a, vocab = self.args, self.dictionary
        noisy, targets = D.MaskTokensDataset.apply_mask(
            self._token_ids(split), vocab, pad_idx=vocab.pad(), mask_idx=self.mask_idx, seed=a.seed,
            mask_prob=a.mask_prob, leave_unmasked_prob=a.leave_unmasked_prob, random_token_prob=a.random_token_prob,
        )

        if getattr(a, "pack_sequences", False):
            layout = {"net_input": D.PackedSequenceDataset(noisy, tokens_key="src_tokens"),
                      "target": D.PackedSequenceDataset(targets)}
        else:
            layout = {"net_input": {"src_tokens": D.RightPadDataset(noisy, pad_idx=vocab.pad())},
                      "target": D.RightPadDataset(targets, pad_idx=vocab.pad())}
        batch_layout = D.NestedDictionaryDataset(layout)
        with D.data_utils.numpy_seed(a.seed):
            fixed_order = np.random.permutation(len(noisy))
        self.datasets[split] = D.SortDataset(batch_layout, sort_order=[fixed_order])

    def build_model(self, args):
        from unicore import models

        return models.build_model(args, self)
