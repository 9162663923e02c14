"""Registers the Hopper-native BERT (``unicore_b200/models/bert.py``) under the names the
reference example uses (``examples/bert/model.py:18,223-260``)."""
from unicore.models import register_model, register_model_architecture
from unicore_b200.models.bert import BertModel as _BertImpl
from unicore_b200.models.bert import apply_arch


@register_model("bert")
class BertModel(_BertImpl):
    pass


@register_model_architecture("bert", "bert")
def base_architecture(args):
    apply_arch(args, "bert_base")


@register_model_architecture("bert", "bert_base")
def bert_base_architecture(args):
    apply_arch(args, "bert_base")


@register_model_architecture("bert", "bert_large")
def bert_large_architecture(args):
    apply_arch(args, "bert_large")


@register_model_architecture("bert", "xlm")
def xlm_architecture(args):
    apply_arch(args, "xlm")
