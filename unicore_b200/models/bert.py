"""BERT (masked-LM encoder) on the fused Hopper op set.

Architecture = the reference example (``examples/bert/model.py:19-260``): token embedding + learned
absolute positions, ``TransformerEncoder`` with T5-style relative-position bias (32 buckets, max
distance 128), post-LN by default, LM head (dense -> act -> LayerNorm -> tied projection + bias)
evaluated only at masked positions; parameter names are identical, so checkpoints interchange.
Architectures: bert/bert_base 12L-768-3072-12H, bert_large 24L-1024-4096-16H, xlm 16L-1280-5120-16H.

GPU notes: the padding mask goes to the encoder as ``[B, L]`` on every path (no host sync to test
whether the batch has padding: an all-False mask gives the same result as none, and no ``[B*H, L, L]``
``-inf`` tensor); the LM-head activation uses the fused bias+GELU kernel.

Packed batches (``--pack-sequences``): ``src_tokens [N]`` with ``cu_seqlens`` / ``max_seqlen`` in ``net_input``.  Each
token's position inside its sentence comes from ``cu_seqlens`` on the device, the encoder runs packed (no pad rows),
and the LM head selects the masked tokens of the flat ``[N]`` mask as it does for a padded batch.
"""
import logging

import torch
import torch.nn as nn
import torch.nn.functional as F

from unicore import ops, utils
from unicore.models import BaseUnicoreModel
from unicore.modules import LayerNorm, TransformerEncoder, init_bert_params

logger = logging.getLogger(__name__)

ARCHS = {
    "bert_base": dict(encoder_layers=12, encoder_embed_dim=768, encoder_ffn_embed_dim=3072, encoder_attention_heads=12),
    "bert_large": dict(encoder_layers=24, encoder_embed_dim=1024, encoder_ffn_embed_dim=4096, encoder_attention_heads=16),
    "xlm": dict(encoder_layers=16, encoder_embed_dim=1280, encoder_ffn_embed_dim=1280 * 4, encoder_attention_heads=16),
}
_COMMON = dict(
    dropout=0.1, emb_dropout=0.1, attention_dropout=0.1, activation_dropout=0.0, pooler_dropout=0.0,
    max_seq_len=512, activation_fn="gelu", pooler_activation_fn="tanh", post_ln=True,
)


def apply_arch(args, arch: str) -> None:
    """Fill every hyper-parameter that was not given explicitly (CLI values win)."""
    for key, value in {**ARCHS[arch], **_COMMON}.items():
        if getattr(args, key, None) is None:
            setattr(args, key, value)


class BertModel(BaseUnicoreModel):
    @staticmethod
    def add_args(parser):
        parser.add_argument("--encoder-layers", type=int, metavar="L", help="num encoder layers")
        parser.add_argument("--encoder-embed-dim", type=int, metavar="H", help="encoder embedding dimension")
        parser.add_argument("--encoder-ffn-embed-dim", type=int, metavar="F", help="encoder embedding dimension for FFN")
        parser.add_argument("--encoder-attention-heads", type=int, metavar="A", help="num encoder attention heads")
        parser.add_argument("--activation-fn", choices=utils.get_available_activation_fns(), help="activation function to use")
        parser.add_argument("--pooler-activation-fn", choices=utils.get_available_activation_fns(),
                            help="activation function to use for pooler layer")
        parser.add_argument("--emb-dropout", type=float, metavar="D", help="dropout probability for embeddings")
        parser.add_argument("--dropout", type=float, metavar="D", help="dropout probability")
        parser.add_argument("--attention-dropout", type=float, metavar="D", help="dropout probability for attention weights")
        parser.add_argument("--activation-dropout", type=float, metavar="D", help="dropout probability after activation in FFN")
        parser.add_argument("--pooler-dropout", type=float, metavar="D", help="dropout probability in the masked_lm pooler layers")
        parser.add_argument("--max-seq-len", type=int, help="number of positional embeddings to learn")
        parser.add_argument("--post-ln", type=utils.eval_bool, help="use post layernorm or pre layernorm")

    def __init__(self, args, dictionary):
        super().__init__()
        apply_arch(args, "bert_base")
        self.args = args
        self.padding_idx = dictionary.pad()
        self.embed_tokens = nn.Embedding(len(dictionary), args.encoder_embed_dim, self.padding_idx)
        self.embed_positions = nn.Embedding(args.max_seq_len, args.encoder_embed_dim)
        self.sentence_encoder = TransformerEncoder(
            encoder_layers=args.encoder_layers,
            embed_dim=args.encoder_embed_dim,
            ffn_embed_dim=args.encoder_ffn_embed_dim,
            attention_heads=args.encoder_attention_heads,
            emb_dropout=args.emb_dropout,
            dropout=args.dropout,
            attention_dropout=args.attention_dropout,
            activation_dropout=args.activation_dropout,
            max_seq_len=args.max_seq_len,
            activation_fn=args.activation_fn,
            rel_pos=True,
            rel_pos_bins=32,
            max_rel_pos=128,
            post_ln=args.post_ln,
        )
        self.lm_head = BertLMHead(
            embed_dim=args.encoder_embed_dim,
            output_dim=len(dictionary),
            activation_fn=args.activation_fn,
            weight=self.embed_tokens.weight,
        )
        self.classification_heads = nn.ModuleDict()
        self.apply(init_bert_params)

    @classmethod
    def build_model(cls, args, task):
        return cls(args, task.dictionary)

    def forward(self, src_tokens, masked_tokens=None, features_only=False, classification_head_name=None,
                cu_seqlens=None, max_seqlen=None, **kwargs):
        if classification_head_name is not None:
            features_only = True
        x = ops.embedding(src_tokens, self.embed_tokens.weight, self.embed_tokens.padding_idx)   # sort-free backward
        if cu_seqlens is not None:   # packed sentences [N]
            if classification_head_name is not None:
                raise ValueError("the classification heads take padded batches")
            pos = ops.varlen_positions(cu_seqlens, src_tokens.size(0))
            x = x + self.embed_positions.weight.index_select(0, pos)
            x = self.sentence_encoder(x, cu_seqlens=cu_seqlens, max_seqlen=max_seqlen)
        else:
            x = x + self.embed_positions.weight[: src_tokens.size(1), :]
            x = self.sentence_encoder(x, padding_mask=src_tokens.eq(self.padding_idx))
        if not features_only:
            x = self.lm_head(x, masked_tokens)
        if classification_head_name is not None:
            x = self.classification_heads[classification_head_name](x)
        return x

    def register_classification_head(self, name, num_classes=None, inner_dim=None, **kwargs):
        if name in self.classification_heads:
            prev = self.classification_heads[name]
            if num_classes != prev.out_proj.out_features or inner_dim != prev.dense.out_features:
                logger.warning(
                    're-registering head "{}" with num_classes {} (prev: {}) and inner_dim {} (prev: {})'.format(
                        name, num_classes, prev.out_proj.out_features, inner_dim, prev.dense.out_features
                    )
                )
        self.classification_heads[name] = BertClassificationHead(
            input_dim=self.args.encoder_embed_dim,
            inner_dim=inner_dim or self.args.encoder_embed_dim,
            num_classes=num_classes,
            activation_fn=self.args.pooler_activation_fn,
            pooler_dropout=self.args.pooler_dropout,
        )


class BertLMHead(nn.Module):
    """dense -> activation -> LayerNorm -> projection onto the (tied) embedding matrix + bias."""

    def __init__(self, embed_dim, output_dim, activation_fn, weight=None):
        super().__init__()
        self.dense = nn.Linear(embed_dim, embed_dim)
        self.activation_fn = utils.get_activation_fn(activation_fn)
        self._gelu = activation_fn == "gelu"
        self.layer_norm = LayerNorm(embed_dim)
        if weight is None:
            weight = nn.Linear(embed_dim, output_dim, bias=False).weight
        self.weight = weight
        self.bias = nn.Parameter(torch.zeros(output_dim))

    def forward(self, features, masked_tokens=None, **kwargs):
        if masked_tokens is not None:
            # project only what the loss looks at (indices shared with the loss: one host read per step)
            features = features.reshape(-1, features.size(-1)).index_select(0, utils.mask_to_index(masked_tokens))
        if self._gelu and ops.use_native(features) and features.dtype in (torch.float16, torch.bfloat16):
            x = ops.bias_gelu(F.linear(features, self.dense.weight), self.dense.bias)
        else:
            x = self.activation_fn(self.dense(features))
        x = self.layer_norm(x)
        return ops.vocab_projection(x, self.weight, self.bias)


class BertClassificationHead(nn.Module):
    """Sentence-level head on the first ([CLS]) position."""

    def __init__(self, input_dim, inner_dim, num_classes, activation_fn, pooler_dropout):
        super().__init__()
        self.dense = nn.Linear(input_dim, inner_dim)
        self.activation_fn = utils.get_activation_fn(activation_fn)
        self.dropout = nn.Dropout(p=pooler_dropout)
        self.out_proj = nn.Linear(inner_dim, num_classes)

    def forward(self, features, **kwargs):
        x = self.dropout(features[:, 0, :])
        x = self.activation_fn(self.dense(x))
        return self.out_proj(self.dropout(x))
