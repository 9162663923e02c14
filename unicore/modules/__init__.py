"""NN building blocks on top of the fused ops (same public names as the reference package,
``unicore/modules/__init__.py:3-14``; historic module paths are aliased)."""
import sys as _sys
import types as _types

from .norm import FusedLayerNormFastFunction, FusedRMSNormFastFunction, LayerNorm, RMSNorm
from .softmax_dropout import softmax_dropout
from .attention import CrossMultiheadAttention, DecoderCache, LayerKVCache, SelfMultiheadAttention
from .transformer import (
    TransformerDecoder,
    TransformerDecoderLayer,
    TransformerEncoder,
    TransformerEncoderLayer,
    bulid_future_mask,
    fill_with_neg_inf,
    init_bert_params,
    relative_position_bucket,
)

__all__ = [
    "LayerNorm", "RMSNorm", "softmax_dropout", "SelfMultiheadAttention", "CrossMultiheadAttention",
    "TransformerEncoderLayer", "TransformerEncoder", "init_bert_params", "relative_position_bucket",
    "TransformerDecoderLayer", "TransformerDecoder", "DecoderCache", "LayerKVCache",
]

_LEGACY = {
    "layer_norm": ["LayerNorm", "FusedLayerNormFastFunction"],
    "rms_norm": ["RMSNorm", "FusedRMSNormFastFunction"],
    "multihead_attention": ["SelfMultiheadAttention", "CrossMultiheadAttention"],
    "transformer_encoder_layer": ["TransformerEncoderLayer"],
    "transformer_encoder": ["TransformerEncoder", "init_bert_params", "relative_position_bucket"],
    "transformer_decoder_layer": ["TransformerDecoderLayer"],
    "transformer_decoder": ["TransformerDecoder", "bulid_future_mask", "fill_with_neg_inf"],
}
for _mod, _names in _LEGACY.items():
    _full = __name__ + "." + _mod
    if _full not in _sys.modules:
        _alias = _types.ModuleType(_full, "compatibility alias; see unicore.modules")
        for _n in _names:
            setattr(_alias, _n, globals()[_n])
        _sys.modules[_full] = _alias
        globals()[_mod] = _alias
