"""Fused element-wise / reduction ops around the GEMMs of a transformer layer.

These fusions do not exist in the reference (it runs GELU, three dropouts, residual adds,
LayerNorm and the fp32 log-softmax as separate ATen kernels,
``unicore/modules/transformer_encoder_layer.py:79-94``, ``losses/masked_lm.py:31-36``); on the GPU
every one of them is HBM-bound, so they are merged into the minimum number of passes:

* ``bias_gelu(x, bias)``                      - GEMM-output bias add + exact GELU (erf), fwd/bwd;
* ``bias_dropout_add_layer_norm(...)``        - ``LN(residual + dropout(x + bias))`` (post-LN) in
  one pass, also returning the pre-LN sum when requested (pre-LN);
* ``softmax_cross_entropy(logits, target)``   - summed NLL of an fp32 log-softmax without
  materialising the ``[N, V]`` fp32 log-probabilities; backward writes the gradient in the
  logits' dtype in place of the logits buffer.
Kernels: ``csrc/fused/*.cu``.  PyTorch fallbacks are bit-for-bit the reference formulation.
"""
from typing import Optional

import torch
import torch.nn.functional as F

from . import grad_sink
from ._native import aligned_param, aligned_rows, native, use_native


# ------------------------------------------------------------------------------------------------
# bias + GELU
# ------------------------------------------------------------------------------------------------
class _BiasGeluFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, bias):
        ctx.save_for_backward(x, bias)
        ctx.bias_sink = grad_sink.claim(bias, ctx.needs_input_grad[1])
        return native().bias_gelu_fwd(x, bias)

    @staticmethod
    def backward(ctx, dy):
        x, bias = ctx.saved_tensors
        claimed = ctx.bias_sink
        dx, dbias = native().bias_gelu_bwd(aligned_param(dy), x, bias, grad_sink.sink(claimed))
        if claimed is not None:  # the bias gradient went straight into the arena
            grad_sink.done(claimed)
            dbias = None
        return dx, dbias


def bias_gelu(x: torch.Tensor, bias: Optional[torch.Tensor]) -> torch.Tensor:
    if use_native(x, bias) and x.dtype in (torch.float16, torch.bfloat16) and x.is_contiguous() and x.shape[-1] % 8 == 0 \
            and x.numel() > 0:
        # the kernels read 16-byte vectors: a view at an odd element offset is copied once (aligned_param)
        return _BiasGeluFn.apply(aligned_param(x), aligned_param(bias, x.dtype))
    return F.gelu(x + bias if bias is not None else x)


# ------------------------------------------------------------------------------------------------
# Linear with a fast bias gradient
# ------------------------------------------------------------------------------------------------
class _LinearFn(torch.autograd.Function):
    """``x @ W^T (+ b)`` - cuBLAS GEMMs both ways; the bias gradient is our column-sum kernel (fp32 accumulation, one
    pass at copy bandwidth) instead of ATen's generic reduction; weight and bias gradients accumulate straight into
    the optimizer's gradient arena when the parameters are claimed (``grad_sink``): the weight-gradient GEMM runs with
    beta = 1 on the arena view."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        ctx.save_for_backward(x, weight)
        ctx.w_sink = grad_sink.claim(weight, ctx.needs_input_grad[1])
        ctx.b_sink = grad_sink.claim(bias, ctx.needs_input_grad[2]) if bias is not None else None
        ctx.has_bias = bias is not None
        return F.linear(x, weight, bias)

    @staticmethod
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        dy = dy.contiguous()
        dy2 = dy.view(-1, dy.shape[-1])
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = dy.matmul(weight)
        if ctx.needs_input_grad[1]:
            x2 = x.reshape(-1, x.shape[-1])
            if ctx.w_sink is not None:
                if weight.numel() * 64 < dy2.shape[0] * dy2.shape[1]:
                    # tiny weight, very long reduction (pair-tensor heads: 64 x 128 outputs over millions of rows): the
                    # beta = 1 GEMM falls onto a slow non-split-K kernel; plain mm + a small add
                    ctx.w_sink.grad.add_(dy2.t().mm(x2))
                else:
                    ctx.w_sink.grad.addmm_(dy2.t(), x2)
                grad_sink.done(ctx.w_sink)
            else:
                dw = dy2.t().mm(x2)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            claimed = ctx.b_sink
            fold = _narrow_fold(dy2)
            if fold > 1:
                # narrow output (< 256 columns): the column kernel would leave most of its lanes idle, so f rows are
                # folded into one [rows / f, f * cols] row first (a view) and the f partial sums added afterwards
                rows, cols = dy2.shape
                wide = native().column_sum(dy2.view(rows // fold, cols * fold), None)
                db = wide.view(fold, cols).float().sum(dim=0).to(dy2.dtype)
                if claimed is not None:
                    claimed.grad.add_(db)
            elif dy2.data_ptr() % 16 == 0 and dy2.shape[-1] % 8 == 0 and dy2.dtype in (torch.float16, torch.bfloat16):
                db = native().column_sum(dy2, grad_sink.sink(claimed))
            else:
                db = dy2.sum(dim=0)
                if claimed is not None:
                    claimed.grad.add_(db)
            if claimed is not None:
                grad_sink.done(claimed)
                db = None
        return dx, dw, db


def _narrow_fold(dy2: torch.Tensor) -> int:
    """How many rows of a narrow 16-bit [rows, cols] gradient to fold into one for ``column_sum`` (1 = do not fold)."""
    rows, cols = dy2.shape
    if (cols >= 256 or cols % 8 != 0 or rows < 4096 or not dy2.is_contiguous() or dy2.data_ptr() % 16 != 0
            or dy2.dtype not in (torch.float16, torch.bfloat16)):
        return 1
    fold = 1
    while cols * fold * 2 <= 1024 and rows % (fold * 2) == 0:
        fold *= 2
    return fold


def linear(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``F.linear`` whose backward computes the bias gradient with ``column_sum`` (``csrc/fused/elementwise.cu``) and
    writes parameter gradients in place into the gradient arena when they are claimed (``grad_sink``)."""
    if not (use_native(x, weight, bias) and x.dtype in (torch.float16, torch.bfloat16) and weight.dtype == x.dtype
            and torch.is_grad_enabled()):
        return F.linear(x, weight, bias)
    direct = grad_sink.wants(weight) or grad_sink.wants(bias)  # (grad mode was checked above)
    fast_bias = (
        bias is not None and bias.dtype == x.dtype
        and weight.shape[0] % 8 == 0
        and (weight.shape[0] >= 256 or x.numel() // max(1, x.shape[-1]) >= 4096)  # (narrow outputs: rows are folded)
        and (x.requires_grad or weight.requires_grad or bias.requires_grad)
    )
    if direct or fast_bias:
        return _LinearFn.apply(x, weight, bias)
    return F.linear(x, weight, bias)


# ------------------------------------------------------------------------------------------------
# bias + dropout + residual add (+ LayerNorm)
# ------------------------------------------------------------------------------------------------
class _BiasDropoutAddLNFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, bias, residual, ln_weight, ln_bias, p, eps, training):
        p = float(p) if training else 0.0
        shape = x.shape
        x2 = aligned_rows(x)
        r2 = aligned_rows(residual)
        y, mean, rstd, summed, seed, offset = native().bias_dropout_add_ln_fwd(x2, bias, r2, ln_weight, ln_bias, p, eps)
        ctx.save_for_backward(summed, ln_weight, mean, rstd)
        ctx.p = p
        ctx.rng = (seed, offset)
        ctx.has_bias = bias is not None
        need = ctx.needs_input_grad
        ctx.sinks = (grad_sink.claim(bias, need[1]) if bias is not None else None, grad_sink.claim(ln_weight, need[3]),
                     grad_sink.claim(ln_bias, need[4]))
        return y.view(shape)

    @staticmethod
    def backward(ctx, dy):
        summed, ln_weight, mean, rstd = ctx.saved_tensors
        dy2 = aligned_rows(dy)
        # dsum: gradient w.r.t. (residual + dropout(x+bias)); dx = dropout-masked dsum
        b_sink, g_sink, be_sink = ctx.sinks
        dsum, dx, dgamma, dbeta, dbias = native().bias_dropout_add_ln_bwd(
            dy2, summed, mean, rstd, ln_weight, ctx.p, ctx.rng[0], ctx.rng[1], ctx.has_bias,
            grad_sink.sink(g_sink), grad_sink.sink(be_sink), grad_sink.sink(b_sink),
        )
        if g_sink is not None:
            grad_sink.done(g_sink)
            dgamma = None
        if be_sink is not None:
            grad_sink.done(be_sink)
            dbeta = None
        if b_sink is not None:
            grad_sink.done(b_sink)
            dbias = None
        return dx.view(dy.shape), dbias, dsum.view(dy.shape), dgamma, dbeta, None, None, None


def bias_dropout_add_layer_norm(x, bias, residual, ln_weight, ln_bias, p, eps, training):
    """``LayerNorm(residual + dropout(x + bias))`` - the post-LN block epilogue in one pass."""
    if (
        use_native(x, bias, residual, ln_weight, ln_bias)
        and x.dtype in (torch.float16, torch.bfloat16)
        and x.shape[-1] % 8 == 0
        and x.shape[-1] <= 8192
        and ln_weight is not None and ln_bias is not None
        and hasattr(native(), "bias_dropout_add_ln_fwd")
    ):
        w = aligned_param(ln_weight, x.dtype)
        b = aligned_param(ln_bias, x.dtype)
        bb = aligned_param(bias, x.dtype)
        return _BiasDropoutAddLNFn.apply(x, bb, residual, w, b, p, eps, training)
    from .norm_ops import layer_norm

    h = x + bias if bias is not None else x
    h = residual + F.dropout(h, p=p, training=training)
    return layer_norm(h, (h.shape[-1],), ln_weight, ln_bias, eps)


# ------------------------------------------------------------------------------------------------
# softmax cross entropy (sum reduction, fp32 math)
# ------------------------------------------------------------------------------------------------
class _SoftmaxXentFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, target, ignore_index, valid_cols):
        loss_rows, lse = native().softmax_xent_fwd(logits, target, int(ignore_index), int(valid_cols))
        ctx.save_for_backward(logits, target, lse)
        ctx.ignore_index = int(ignore_index)
        ctx.valid_cols = int(valid_cols)
        return loss_rows.sum()

    @staticmethod
    def backward(ctx, dloss):
        logits, target, lse = ctx.saved_tensors
        dlogits = native().softmax_xent_bwd(
            logits, target, lse, dloss.float().reshape(1), ctx.ignore_index, ctx.valid_cols
        )
        return dlogits, None, None, None


def _padded_base(logits):
    """If ``logits`` is the ``[:, :V]`` slice of a wider contiguous 2-D tensor (a vocabulary padded for
    GEMM alignment, see ``vocab_projection``) return that tensor, else None."""
    base = logits._base
    if (
        base is not None
        and base.dim() == 2
        and base.is_contiguous()
        and base.shape[0] == logits.shape[0]
        and logits.storage_offset() == base.storage_offset()
        and logits.stride() == (base.shape[1], 1)
        and base.dtype == logits.dtype
    ):
        return base
    return None


class _VocabProjFn(torch.autograd.Function):
    """Padded vocabulary projection with the parameter gradients written in place (``grad_sink``): the weight-gradient
    GEMM accumulates into the arena view of the UNPADDED weight (beta = 1), so neither the pad's backward slice nor an
    AccumulateGrad add (47 MB each way for BERT-base) runs; the bias gradient is the column-sum kernel."""

    @staticmethod
    def forward(ctx, x2, weight, bias, pad):
        w = F.pad(weight, (0, 0, 0, pad))
        b = F.pad(bias, (0, pad)) if bias is not None else None
        ctx.save_for_backward(x2, w)
        ctx.V = weight.shape[0]
        ctx.w_sink = grad_sink.claim(weight, ctx.needs_input_grad[1])
        ctx.b_sink = grad_sink.claim(bias, ctx.needs_input_grad[2]) if bias is not None else None
        ctx.has_bias = bias is not None
        return F.linear(x2, w, b)

    @staticmethod
    def backward(ctx, dout):
        x2, w = ctx.saved_tensors
        V = ctx.V
        dout = dout.contiguous()
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = dout.matmul(w)
        if ctx.needs_input_grad[1]:
            if ctx.w_sink is not None:
                ctx.w_sink.grad.addmm_(dout[:, :V].t(), x2)
                grad_sink.done(ctx.w_sink)
            else:
                dw = dout[:, :V].t().mm(x2)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            if dout.dtype in (torch.float16, torch.bfloat16) and dout.shape[1] % 8 == 0 and dout.data_ptr() % 16 == 0:
                db = native().column_sum(dout, None)[:V]
            else:
                db = dout.sum(dim=0)[:V]
            if ctx.b_sink is not None:
                ctx.b_sink.grad.add_(db)
                grad_sink.done(ctx.b_sink)
                db = None
        return dx, dw, db, None


def vocab_projection(x, weight, bias=None, multiple=64):
    """``F.linear(x, weight, bias)`` for an output dimension (vocabulary) that is not a multiple of 8.

    With V = 30522 the logits' rows are only 4-byte aligned, which sends all three GEMMs of the
    projection (fwd, dgrad, wgrad) down cuBLAS' slow element-aligned path.  The weight/bias are zero-padded to a multiple of ``multiple`` rows on the fly (47 MB
    copy for BERT-base, ~15 us) and the result is returned as the ``[:, :V]`` view of the padded
    logits; ``softmax_cross_entropy`` recognises such views and reads/writes the padded buffer in
    place, so no compaction copy is ever made.
    """
    V = weight.shape[0]
    pad = (-V) % multiple
    if pad == 0 or not x.is_cuda or x.dtype not in (torch.float16, torch.bfloat16):
        return F.linear(x, weight, bias)
    lead = x.shape[:-1]
    x2 = x.reshape(-1, x.shape[-1])
    if (torch.is_grad_enabled() and use_native(x, weight) and (grad_sink.wants(weight) or grad_sink.wants(bias))
            and hasattr(native(), "embedding_bwd")):   # (both in-place paths of the tied embedding came with that build)
        out = _VocabProjFn.apply(x2, weight, bias, pad)
    else:
        w = F.pad(weight, (0, 0, 0, pad))
        b = F.pad(bias, (0, pad)) if bias is not None else None
        out = F.linear(x2, w, b)
    return out[:, :V] if len(lead) == 1 else out[:, :V].unflatten(0, lead)


# ------------------------------------------------------------------------------------------------
# embedding lookup with a sort-free backward
# ------------------------------------------------------------------------------------------------
_embedding_scratch = {}


def _scratch_for(weight):
    """Persistent fp32 accumulator [V, D] + row flags [V] of ``embedding_bwd`` (left all-zero by every call)."""
    key = (weight.device, weight.shape[0], weight.shape[1])
    buf = _embedding_scratch.get(key)
    if buf is None:
        buf = (torch.zeros(weight.shape, dtype=torch.float32, device=weight.device),
               torch.zeros(weight.shape[0], dtype=torch.uint8, device=weight.device))
        _embedding_scratch[key] = buf
    return buf


class _EmbeddingFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, tokens, weight, padding_idx):
        ctx.save_for_backward(tokens, weight)
        ctx.padding_idx = -1 if padding_idx is None else int(padding_idx)
        # the kernels write the sink with 16-byte vectors; flat arenas pad parameters to 2 elements only, so an arena
        # view may start 4-byte aligned: its gradient then goes through autograd (AccumulateGrad adds it to the view)
        aligned = weight.grad is not None and weight.grad.data_ptr() % 16 == 0
        ctx.w_sink = grad_sink.claim(weight, ctx.needs_input_grad[1] and aligned)
        return F.embedding(tokens, weight, padding_idx)

    @staticmethod
    def backward(ctx, dy):
        tokens, weight = ctx.saved_tensors
        if not ctx.needs_input_grad[1]:
            return None, None, None
        dy = dy.contiguous()
        scratch, touched = _scratch_for(weight)
        tokens = tokens.contiguous()
        if ctx.w_sink is not None:
            native().embedding_bwd(dy, tokens, ctx.padding_idx, scratch, touched, ctx.w_sink.grad, True)
            grad_sink.done(ctx.w_sink)
            return None, None, None
        grad = torch.zeros_like(weight)
        native().embedding_bwd(dy, tokens, ctx.padding_idx, scratch, touched, grad, False)
        return None, grad, None


def embedding(tokens: torch.Tensor, weight: torch.Tensor, padding_idx: Optional[int] = None) -> torch.Tensor:
    """``F.embedding`` whose backward is two kernels (fp32 ``red`` scatter + finalize, ``csrc/fused/embedding.cu``)
    instead of ATen's radix sort + segmented reduction (~30 launches per BERT-base step), writing into the
    gradient arena when the weight is claimed."""
    if padding_idx is not None and padding_idx < 0:
        padding_idx += weight.shape[0]  # F.embedding's convention: -1 is the last row (an index < -V stays invalid)
    if (
        use_native(weight) and torch.is_grad_enabled() and weight.requires_grad
        and weight.dtype in (torch.float16, torch.bfloat16) and weight.dim() == 2 and weight.shape[1] % 8 == 0
        and weight.is_contiguous() and tokens.dtype == torch.long and hasattr(native(), "embedding_bwd")
    ):
        return _EmbeddingFn.apply(tokens, weight, padding_idx)
    return F.embedding(tokens, weight, padding_idx)


def softmax_cross_entropy(logits: torch.Tensor, target: torch.Tensor, ignore_index: int = -100) -> torch.Tensor:
    """``nll_loss(log_softmax(logits, fp32), target, reduction='sum', ignore_index=...)``; fp64 logits are reduced in
    fp64."""
    if (
        use_native(logits, target)
        and logits.dim() == 2
        and logits.dtype in (torch.float16, torch.bfloat16, torch.float32)
        and logits.numel() > 0
        and hasattr(native(), "softmax_xent_fwd")
    ):
        if logits.is_contiguous():
            return _SoftmaxXentFn.apply(logits, target.contiguous(), ignore_index, 0)
        base = _padded_base(logits)
        if base is not None:
            return _SoftmaxXentFn.apply(base, target.contiguous(), ignore_index, logits.shape[1])
        return _SoftmaxXentFn.apply(logits.contiguous(), target.contiguous(), ignore_index, 0)
    # fp32 math for 16-bit and fp32 logits; fp64 logits (a float64 reference model) stay in fp64
    return F.nll_loss(
        F.log_softmax(logits, dim=-1, dtype=torch.promote_types(logits.dtype, torch.float32)), target,
        ignore_index=ignore_index, reduction="sum"
    )


# ------------------------------------------------------------------------------------------------
# Gaussian radial basis of an edge-type dependent affine map of the distance (Uni-Mol pair features)
# ------------------------------------------------------------------------------------------------
class _GaussianBasisFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, dist, edge_type, mul_w, bias_w, means, stds):
        y = native().gbf_fwd(dist, edge_type, mul_w, bias_w, means, stds)
        ctx.save_for_backward(dist, edge_type, mul_w, bias_w, means, stds)
        return y

    @staticmethod
    def backward(ctx, dy):
        dist, edge_type, mul_w, bias_w, means, stds = ctx.saved_tensors
        dmul, dbias, dmean, dstd = native().gbf_bwd(dy.contiguous(), dist, edge_type, mul_w, bias_w, means, stds)
        dstd = dstd * torch.sign(stds.float())
        dt = mul_w.dtype
        return None, None, dmul.to(dt).view_as(mul_w), dbias.to(dt).view_as(bias_w), dmean.to(dt).view_as(means), \
            dstd.to(dt).view_as(stds)


def gaussian_basis_reference(dist, edge_type, mul_w, bias_w, means, stds):
    """``exp(-0.5 ((mul[e] d + bias[e] - mean) / std)^2) / (sqrt(2 * 3.14159) std)``, ``std = |stds| + 1e-5`` -> [..., K]."""
    t = (mul_w.view(-1)[edge_type].type_as(dist) * dist + bias_w.view(-1)[edge_type].type_as(dist)).unsqueeze(-1).float()
    mean = means.float().view(-1)
    std = stds.float().view(-1).abs() + 1e-5
    a = (2 * 3.14159) ** 0.5
    return (torch.exp(-0.5 * (((t - mean) / std) ** 2)) / (a * std)).to(means.dtype)


def gaussian_basis(dist, edge_type, mul_w, bias_w, means, stds):
    """Fused forward/backward of Uni-Mol's ``GaussianLayer`` (no index sort, no [N, K] fp32 temporaries)."""
    K = means.numel()
    if (
        use_native(dist, edge_type, mul_w, means)
        and hasattr(native(), "gbf_fwd")
        and means.dtype in (torch.float16, torch.bfloat16)
        and K % 8 == 0 and (K // 8) <= 32 and ((K // 8) & (K // 8 - 1)) == 0
        and mul_w.numel() <= 8192
    ):
        dt = means.dtype
        return _GaussianBasisFn.apply(
            dist.to(dt).contiguous(), edge_type.contiguous(), aligned_param(mul_w.view(-1), dt),
            aligned_param(bias_w.view(-1), dt), aligned_param(means.view(-1), dt), aligned_param(stds.view(-1), dt),
        )
    return gaussian_basis_reference(dist, edge_type, mul_w, bias_w, means, stds)
