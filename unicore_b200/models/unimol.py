"""Uni-Mol style SE(3)-invariant molecular transformer (BASELINE.json config 4).

The reference tree does not contain this model (it names Uni-Mol as a downstream project,
``README.md:40-43``) but ships the hooks it needs: ``return_attn`` in the attention / encoder layer
(``unicore/modules/multihead_attention.py:95-118``, ``transformer_encoder_layer.py:61-98``), 2-D padded
collation (``data/pad_dataset.py:32-38``), LayerNorm sizes 64/512 and the ``softmax_dropout`` op with a
full ``[B*H, N, N]`` bias.  This file implements the publicly described architecture on those hooks:

* atom-type embedding (+ optional [CLS]) -> 15 pre-LN encoder layers, 512 dim, 64 heads (head_dim 8);
* pair representation = attention bias: Gaussian basis of inter-atomic distances with an
  edge-type specific affine map -> MLP -> ``[B, H, N, N]``; every layer returns its pre-softmax
  logits, which become the next layer's bias (pair update);
* heads: masked-atom LM, pair-distance regression, SE(3)-equivariant coordinate update.

Hot ops on the GPU: the fused wgmma attention in its logits mode (``ops.fused_attention_qkvpacked(...,
return_logits=True)``: head dim 8 runs on the 64-column kernels; each layer writes its logits and takes their
gradient, and the ``[B, H, N, N]`` probabilities are never materialised), LayerNorm(512) and LayerNorm(64)
kernels, bias+GELU; the GEMMs go to cuBLAS.
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from unicore import ops, utils
from unicore.models import BaseUnicoreModel
from unicore.modules import LayerNorm, TransformerEncoderLayer, init_bert_params

UNIMOL_BASE = dict(
    encoder_layers=15, encoder_embed_dim=512, encoder_ffn_embed_dim=2048, encoder_attention_heads=64,
    dropout=0.1, emb_dropout=0.1, attention_dropout=0.1, activation_dropout=0.0, pooler_dropout=0.0,
    max_seq_len=512, activation_fn="gelu", pooler_activation_fn="tanh", post_ln=False,
    masked_token_loss=1.0, masked_coord_loss=5.0, masked_dist_loss=10.0, x_norm_loss=0.01, delta_pair_repr_norm_loss=0.01,
    gaussian_kernels=128,
)


def apply_unimol_arch(args):
    for k, v in UNIMOL_BASE.items():
        if getattr(args, k, None) is None:
            setattr(args, k, v)


def _gaussian(x, mean, std):
    a = (2 * 3.14159) ** 0.5
    return torch.exp(-0.5 * (((x - mean) / std) ** 2)) / (a * std)


class GaussianLayer(nn.Module):
    """K Gaussian radial basis functions of ``mul[edge] * d + bias[edge]``."""

    def __init__(self, K=128, edge_types=1024):
        super().__init__()
        self.K = K
        self.means = nn.Embedding(1, K)
        self.stds = nn.Embedding(1, K)
        self.mul = nn.Embedding(edge_types, 1)
        self.bias = nn.Embedding(edge_types, 1)
        nn.init.uniform_(self.means.weight, 0, 3)
        nn.init.uniform_(self.stds.weight, 0, 3)
        nn.init.constant_(self.bias.weight, 0)
        nn.init.constant_(self.mul.weight, 1)

    def forward(self, x, edge_type):
        if ops.use_native(x, edge_type) and self.means.weight.dtype in (torch.float16, torch.bfloat16):
            # one fused kernel per direction instead of two embedding look-ups (whose backward sorts B*L*L indices)
            # and a TorchScript expression over [B, L, L, K] fp32 temporaries
            return ops.gaussian_basis(x, edge_type, self.mul.weight, self.bias.weight, self.means.weight,
                                      self.stds.weight)
        mul = self.mul(edge_type).type_as(x)
        bias = self.bias(edge_type).type_as(x)
        x = (mul * x.unsqueeze(-1) + bias).expand(-1, -1, -1, self.K)
        mean = self.means.weight.float().view(-1)
        std = self.stds.weight.float().view(-1).abs() + 1e-5
        return _gaussian(x.float(), mean, std).type_as(self.means.weight)


class NonLinearHead(nn.Module):
    def __init__(self, input_dim, out_dim, activation_fn, hidden=None):
        super().__init__()
        hidden = input_dim if not hidden else hidden
        self.linear1 = nn.Linear(input_dim, hidden)
        self.linear2 = nn.Linear(hidden, out_dim)
        self.activation_fn = utils.get_activation_fn(activation_fn)

    def forward(self, x):
        # (ops.linear: bias gradients of these pair-tensor layers - millions of rows, 64-128 columns - through the
        # column-sum kernel instead of ATen's generic reduction)
        h = self.activation_fn(ops.linear(x, self.linear1.weight, self.linear1.bias))
        return ops.linear(h, self.linear2.weight, self.linear2.bias)


class MaskLMHead(nn.Module):
    def __init__(self, embed_dim, output_dim, activation_fn, weight=None):
        super().__init__()
        self.dense = nn.Linear(embed_dim, embed_dim)
        self.activation_fn = utils.get_activation_fn(activation_fn)
        self.layer_norm = LayerNorm(embed_dim)
        if weight is None:
            weight = nn.Linear(embed_dim, output_dim, bias=False).weight
        self.weight = weight
        self.bias = nn.Parameter(torch.zeros(output_dim))

    def forward(self, features, masked_tokens=None, **kwargs):
        if masked_tokens is not None:
            features = features.reshape(-1, features.size(-1)).index_select(0, utils.mask_to_index(masked_tokens))
        x = self.layer_norm(self.activation_fn(self.dense(features)))
        return F.linear(x, self.weight) + self.bias


class DistanceHead(nn.Module):
    def __init__(self, heads, activation_fn):
        super().__init__()
        self.dense = nn.Linear(heads, heads)
        self.layer_norm = LayerNorm(heads)
        self.out_proj = nn.Linear(heads, 1)
        self.activation_fn = utils.get_activation_fn(activation_fn)

    def forward(self, x):
        bsz, seq_len, _, _ = x.size()
        x = self.activation_fn(ops.linear(x, self.dense.weight, self.dense.bias))
        x = self.out_proj(self.layer_norm(x)).view(bsz, seq_len, seq_len)
        return (x + x.transpose(-1, -2)) * 0.5


class TransformerEncoderWithPair(nn.Module):
    """Encoder whose attention logits are threaded through the layers as the pair representation."""

    def __init__(self, encoder_layers=15, embed_dim=512, ffn_embed_dim=2048, attention_heads=64, emb_dropout=0.1,
                 dropout=0.1, attention_dropout=0.1, activation_dropout=0.0, max_seq_len=512, activation_fn="gelu",
                 post_ln=False, no_final_head_layer_norm=False):
        super().__init__()
        self.emb_dropout = emb_dropout
        self.max_seq_len = max_seq_len
        self.embed_dim = embed_dim
        self.attention_heads = attention_heads
        self.emb_layer_norm = LayerNorm(embed_dim)
        self.final_layer_norm = None if post_ln else LayerNorm(embed_dim)
        self.final_head_layer_norm = None if no_final_head_layer_norm else LayerNorm(attention_heads)
        self.layers = nn.ModuleList([
            TransformerEncoderLayer(embed_dim=embed_dim, ffn_embed_dim=ffn_embed_dim, attention_heads=attention_heads,
                                    dropout=dropout, attention_dropout=attention_dropout,
                                    activation_dropout=activation_dropout, activation_fn=activation_fn, post_ln=post_ln)
            for _ in range(encoder_layers)
        ])

    def forward(self, emb, attn_mask=None, padding_mask=None):
        bsz, seq_len = emb.size(0), emb.size(1)
        x = self.emb_layer_norm(emb)
        x = F.dropout(x, p=self.emb_dropout, training=self.training)
        if padding_mask is not None:
            x = x * (1 - padding_mask.unsqueeze(-1).type_as(x))
        input_attn_mask = attn_mask
        input_padding_mask = padding_mask

        # The reference writes -inf into the padded key columns of the pair bias up front (a full pass over
        # [B, H, L, L] and another in backward).  Here the first layer's attention kernel adds the [B, 1, 1, L]
        # padding mask while it forms the logits; those logits ARE the next layer's bias, so the -inf columns
        # travel with the pair representation from then on.
        # Only the logits are threaded on (need_probs=False), so on the GPU each layer's attention runs fused.
        for layer in self.layers:
            x, attn_mask, _ = layer(x, padding_mask=padding_mask, attn_bias=attn_mask, return_attn=True,
                                    need_probs=False)
            padding_mask = None

        def norm_loss(t, tolerance=1.0):
            # |t|_2 accumulated in fp32 by the reduction itself (no fp32 copy of the pair tensor)
            norm = torch.linalg.vector_norm(t, dim=-1, dtype=torch.float32)
            return F.relu(torch.abs(norm - math.sqrt(t.shape[-1])) - tolerance)

        def masked_mean(mask, value, dim=-1, eps=1e-10):
            return (torch.sum(mask * value, dim=dim) / (eps + torch.sum(mask, dim=dim))).mean()

        x_norm = norm_loss(x)
        token_mask = 1.0 - input_padding_mask.float() if input_padding_mask is not None else torch.ones_like(x_norm)
        x_norm = masked_mean(token_mask, x_norm)
        if self.final_layer_norm is not None:
            x = self.final_layer_norm(x)

        # pair-major outputs in one pass: pair = logits with -inf -> 0 (what the heads consume), delta = change of
        # the pair representation through the stack with padded key columns zeroed
        attn_mask, delta = ops.pair_tail(
            attn_mask.view(bsz, -1, seq_len, seq_len), input_attn_mask.view(bsz, -1, seq_len, seq_len), input_padding_mask
        )
        pair_mask = token_mask[..., None] * token_mask[..., None, :]
        delta_norm = masked_mean(pair_mask, norm_loss(delta), dim=(-1, -2))
        if self.final_head_layer_norm is not None:
            delta = self.final_head_layer_norm(delta)
        return x, attn_mask, delta, x_norm, delta_norm


class UniMolModel(BaseUnicoreModel):
    @staticmethod
    def add_args(parser):
        parser.add_argument("--encoder-layers", type=int, metavar="L")
        parser.add_argument("--encoder-embed-dim", type=int, metavar="H")
        parser.add_argument("--encoder-ffn-embed-dim", type=int, metavar="F")
        parser.add_argument("--encoder-attention-heads", type=int, metavar="A")
        parser.add_argument("--activation-fn", choices=utils.get_available_activation_fns())
        parser.add_argument("--pooler-activation-fn", choices=utils.get_available_activation_fns())
        parser.add_argument("--emb-dropout", type=float, metavar="D")
        parser.add_argument("--dropout", type=float, metavar="D")
        parser.add_argument("--attention-dropout", type=float, metavar="D")
        parser.add_argument("--activation-dropout", type=float, metavar="D")
        parser.add_argument("--pooler-dropout", type=float, metavar="D")
        parser.add_argument("--max-seq-len", type=int)
        parser.add_argument("--post-ln", type=utils.eval_bool)
        parser.add_argument("--masked-token-loss", type=float, metavar="D")
        parser.add_argument("--masked-dist-loss", type=float, metavar="D")
        parser.add_argument("--masked-coord-loss", type=float, metavar="D")
        parser.add_argument("--x-norm-loss", type=float, metavar="D")
        parser.add_argument("--delta-pair-repr-norm-loss", type=float, metavar="D")
        parser.add_argument("--gaussian-kernels", type=int)

    def __init__(self, args, dictionary):
        super().__init__()
        apply_unimol_arch(args)
        self.args = args
        self.padding_idx = dictionary.pad()
        n_tok = len(dictionary)
        self.embed_tokens = nn.Embedding(n_tok, args.encoder_embed_dim, self.padding_idx)
        self.encoder = TransformerEncoderWithPair(
            encoder_layers=args.encoder_layers, embed_dim=args.encoder_embed_dim,
            ffn_embed_dim=args.encoder_ffn_embed_dim, attention_heads=args.encoder_attention_heads,
            emb_dropout=args.emb_dropout, dropout=args.dropout, attention_dropout=args.attention_dropout,
            activation_dropout=args.activation_dropout, max_seq_len=args.max_seq_len,
            activation_fn=args.activation_fn, post_ln=args.post_ln,
            no_final_head_layer_norm=args.delta_pair_repr_norm_loss < 0,
        )
        if args.masked_token_loss > 0:
            self.lm_head = MaskLMHead(args.encoder_embed_dim, n_tok, args.activation_fn, weight=None)
        K = args.gaussian_kernels
        self.gbf_proj = NonLinearHead(K, args.encoder_attention_heads, args.activation_fn)
        self.gbf = GaussianLayer(K, n_tok * n_tok)
        if args.masked_coord_loss > 0:
            self.pair2coord_proj = NonLinearHead(args.encoder_attention_heads, 1, args.activation_fn)
        if args.masked_dist_loss > 0:
            self.dist_head = DistanceHead(args.encoder_attention_heads, args.activation_fn)
        self.classification_heads = nn.ModuleDict()
        self.apply(init_bert_params)

    @classmethod
    def build_model(cls, args, task):
        return cls(args, task.dictionary)

    def forward(self, src_tokens, src_distance, src_coord, src_edge_type, encoder_masked_tokens=None,
                features_only=False, **kwargs):
        padding_mask = src_tokens.eq(self.padding_idx)
        x = ops.embedding(src_tokens, self.embed_tokens.weight, self.embed_tokens.padding_idx)
        n_node = src_distance.size(-1)
        gbf_feature = self.gbf(src_distance, src_edge_type)
        graph_attn_bias = ops.pair_to_heads(self.gbf_proj(gbf_feature)).view(-1, n_node, n_node)
        enc, pair, delta_pair, x_norm, delta_norm = self.encoder(x, padding_mask=padding_mask, attn_mask=graph_attn_bias)
        # (the encoder already returns the pair representation with its -inf entries zeroed)
        logits = coord = dist = None
        if not features_only:
            if self.args.masked_token_loss > 0:
                logits = self.lm_head(enc, encoder_masked_tokens)
            if self.args.masked_coord_loss > 0:
                atom_num = (torch.sum(1 - padding_mask.type_as(x), dim=1) - 1).view(-1, 1, 1, 1)
                delta_pos = src_coord.unsqueeze(1) - src_coord.unsqueeze(2)
                attn_probs = self.pair2coord_proj(delta_pair)
                coord = src_coord + torch.sum(delta_pos / atom_num * attn_probs, dim=2)
            if self.args.masked_dist_loss > 0:
                dist = self.dist_head(pair)
        return logits, dist, coord, x_norm, delta_norm
