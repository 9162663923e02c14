"""Masked-LM loss (reference ``unicore/losses/masked_lm.py:13-67``): only positions whose target is not padding count;
the model projects only those positions (``masked_tokens``); ``sample_size`` - what the gradients are normalised by - is
the device-resident number of masked tokens.

GPU path: log-softmax + NLL over the ``[n_masked, vocab]`` logits is one fused kernel
(``unicore.ops.softmax_cross_entropy``) that never materialises fp32 log-probabilities, and the masked positions are
resolved without a host stall (``utils.request_mask_index``).

Logged per batch: ``bsz`` (sentences), ``sample_size`` (masked tokens) and ``seq_len`` (token slots of the padded
batch, ``bsz * width``).  A packed batch (``target [N]``, ``cu_seqlens`` / ``max_seqlen`` in ``net_input``) logs the
values of the padded batch of the same sentences: ``bsz = cu_seqlens.numel() - 1`` (a shape, not a device read) and
``seq_len = bsz * max_seqlen``, ``max_seqlen`` being the width the padded batch has.
"""
import math

from unicore import metrics, ops, utils
from unicore.losses import UnicoreLoss, register_loss


def _total(logging_outputs, key):
    return sum(entry.get(key, 0) for entry in logging_outputs)


@register_loss("masked_lm")
class MaskedLMLoss(UnicoreLoss):
    def __init__(self, task):
        super().__init__(task)
        self.padding_idx = task.dictionary.pad()

    def forward(self, model, sample, reduce=True):
        target = sample["target"]
        masked_tokens = target.ne(self.padding_idx)
        sample_size = masked_tokens.int().sum()
        # the count read behind the index of the masked positions is queued AHEAD of the encoder: by the time the LM
        # head and the target gather below ask for the index nobody has to wait
        utils.request_mask_index(masked_tokens)
        logits = model(**sample["net_input"], masked_tokens=masked_tokens)
        wanted = target.reshape(-1).index_select(0, utils.mask_to_index(masked_tokens))
        loss = ops.softmax_cross_entropy(logits, wanted, ignore_index=self.padding_idx)
        net_input = sample["net_input"]
        if net_input.get("cu_seqlens") is not None:
            rows, width = net_input["cu_seqlens"].numel() - 1, int(net_input["max_seqlen"])
        else:
            rows, width = target.size(0), target.size(1)
        return loss, sample_size, {"loss": loss.data, "bsz": rows, "sample_size": sample_size, "seq_len": rows * width}

    @staticmethod
    def reduce_metrics(logging_outputs, split="valid") -> None:
        sample_size = _total(logging_outputs, "sample_size")
        bits_per_token = _total(logging_outputs, "loss") / sample_size / math.log(2)
        metrics.log_scalar("loss", bits_per_token, sample_size, round=3)
        metrics.log_scalar("seq_len", _total(logging_outputs, "seq_len") / _total(logging_outputs, "bsz"), 1, round=3)

    @staticmethod
    def logging_outputs_can_be_summed(is_train) -> bool:
        return True
