"""The Uni-Mol path the benchmark trains, composed, against float64: the pair-bias stack with the kernels' own dropout
masks, and the whole model and loss through the Trainer against the portable plug-in (``examples/unimol_portable``).

Every kernel on the path has an exact test of its own; these tests check that they compose where Uni-Mol differs from
BERT:
* the padding contract.  The plug-in writes ``-inf`` into the padded key columns of the input pair bias up front, so
  that bias gets an exactly zero gradient there.  ``TransformerEncoderWithPair`` passes the ``[B, L]`` key mask to the
  first layer's kernel instead, and from the second layer on the ``-inf`` columns travel inside the bias (the previous
  layer's logits) with no key mask at all; whole 64-key tiles are then ``-inf`` through the bias alone;
* the logits threaded through the layers: layer l's ``z`` is layer l + 1's ``[B*H, N, N]`` bias, so ``dz`` flows back
  through every layer into ``gbf_proj`` and the Gaussian basis;
* the model code only Uni-Mol runs: ``pair_to_heads``, ``ops.linear`` with column-sum bias gradients over B*N*N rows,
  ``pair_tail``, the two norm losses, the distance head's symmetrisation, the coordinate head and the 5-term loss.

The model-level reference is independent code: the portable plug-in in float64 (``test_cpu_models.py::
test_unimol_matches_the_portable_plugin`` pins that the two formulations agree), run with the weights the Trainer's step
ran with.

Dropout is compared element for element with the kernels' own masks (the helpers of ``test_gpu_encoder_path.py``): the
keep bits of the fused attention forward, and torch's ``F.dropout`` in ``unicore.modules.transformer`` (pre-LN residual
dropout) and in ``unicore_b200.models.unimol`` (embedding dropout), replaced by a dropout that records its mask.

Every tensor meets ``max|got - ref| <= c * u * max|ref|``, ``u`` the unit roundoff of the 16-bit type (2^-11 for fp16,
2^-8 for bf16), with one ``c`` per class of tensor (``C``): the output (the five encoder outputs, the loss and its
terms, the masked-token logits), dx (the gradient of the embeddings), weight gradients (GEMM weights, LayerNorm gains,
embedding tables and the Gaussian basis parameters), bias gradients (GEMM and LayerNorm biases) and dbias (the gradient
of the ``[B*H, N, N]`` input pair bias).

Calibration: the worst ratio ``max|got - ref| / (u * max|ref|)`` observed per class over every test here at p = 0, on
an H100 80GB HBM3 (700 W power limit); each ``c`` is at most 4x the worst observed value.

    =========  ====  ====  ==
    class      fp16  bf16  c
    =========  ====  ====  ==
    output     3.27  3.08  12
    dx         2.07  2.17  8
    weight     3.61  2.92  12
    bias       2.62  2.59  10
    dbias      2.87  2.75  10
    =========  ====  ====  ==

Every entry is set by the pair stack; the model's own worst ratios are 1.61 (output), 2.90 (weight) and 2.46 (bias).
At p = 0.1 the worst ratios of the stack are output 3.17, dx 2.88, weight 2.92, bias 2.84 and dbias 3.11.
"""
import copy
import importlib
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

from test_gpu_encoder_path import _attention_keep, _check_keep_rate, _perturb, _spies

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "examples"))
UNIT = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
DTYPES = [torch.float16, torch.bfloat16]
C = {"output": 12, "dx": 8, "weight": 12, "bias": 10, "dbias": 10}
# worst ratio max|got - ref| / (u * max|ref|) per (class, dtype) seen in this process: what the table above is made of
OBSERVED = {}
NEG_INF = float("-inf")


def _ops():
    from unicore import ops

    assert ops.USE_NATIVE, "native kernels must be active on the GPU box"
    return ops


def _check(got, ref, dtype, cls, what):
    got, ref = torch.as_tensor(got).detach().double(), torch.as_tensor(ref).detach().double()
    assert got.shape == ref.shape, (what, tuple(got.shape), tuple(ref.shape))
    assert bool(torch.isfinite(got).all()), what + ": not finite"
    scale = UNIT[dtype] * ref.abs().max().item()
    err = (got.to(ref.device) - ref).abs().max().item()
    ratio = err / scale if scale > 0 else (0.0 if err == 0 else math.inf)
    key = (cls, str(dtype).replace("torch.", ""))
    OBSERVED[key] = max(OBSERVED.get(key, 0.0), ratio)
    assert ratio <= C[cls], "{}: max|got - ref| = {:.3g} = {:.3g} u max|ref| (bound {} u max|ref|)".format(
        what, err, ratio, C[cls])


def _param_class(name):
    return "bias" if name.endswith("bias") else "weight"


# ------------------------------------------------------------------------------------------------------------------
# float64 formulation of the pair-bias stack, as the portable plug-in writes it
# ------------------------------------------------------------------------------------------------------------------
def _pair_layer64(P, pre, x, z, H, eps, attn_drop, res_keeps, res_scale):
    """Pre-LN ``TransformerEncoderLayer`` (GELU, activation dropout 0) in float64 that returns ``(x, z)``, ``z = s *
    D^-1/2 + bias`` its logits ``[B, H, L, L]``.  There is no key mask: padded keys are ``-inf`` columns of ``z``."""
    B, L, E = x.shape
    D = E // H

    def w(name):
        return P[pre + name]

    def drop(t, i):
        return t if res_keeps[i] is None else t * res_keeps[i] * res_scale

    h = F.layer_norm(x, (E,), w("self_attn_layer_norm.weight"), w("self_attn_layer_norm.bias"), eps)
    q, k, v = F.linear(h, w("self_attn.in_proj.weight"), w("self_attn.in_proj.bias")).view(B, L, 3, H, D).unbind(2)
    z = torch.einsum("bqhd,bkhd->bhqk", q, k) * D ** -0.5 + z
    pr = torch.softmax(z, dim=-1)
    keep, scale = attn_drop
    if keep is not None:
        pr = pr * keep * scale
    o = torch.einsum("bhqk,bkhd->bqhd", pr, v).reshape(B, L, E)
    x = x + drop(F.linear(o, w("self_attn.out_proj.weight"), w("self_attn.out_proj.bias")), 0)
    h = F.layer_norm(x, (E,), w("final_layer_norm.weight"), w("final_layer_norm.bias"), eps)
    h = F.linear(F.gelu(F.linear(h, w("fc1.weight"), w("fc1.bias"))), w("fc2.weight"), w("fc2.bias"))
    return x + drop(h, 1), z


def _excess_norm(t, tolerance=1.0):
    return F.relu((t.norm(dim=-1) - math.sqrt(t.shape[-1])).abs() - tolerance)


def _pair_major(t):
    """``[B, H, L, L] -> [B, L, L, H]`` with ``-inf -> 0``."""
    return t.masked_fill(t == NEG_INF, 0).permute(0, 2, 3, 1)


def _pair_stack64(P, emb, bias, pad, H, layers, eps, emb_keep, attn, res, p):
    """``TransformerEncoderWithPair`` (pre-LN, head LayerNorm on) in float64 after ``PairBiasEncoder``: returns ``(x,
    pair, delta, x_norm, delta_norm)`` and the last logits ``[B, H, L, L]``.  ``emb_keep``, ``attn`` and ``res`` are
    the recovered masks (Nones without dropout)."""
    B, L, E = emb.shape
    keep = (~pad).double()
    scale = 1.0 / (1.0 - p) if p > 0 else 1.0
    x = F.layer_norm(emb, (E,), P["emb_layer_norm.weight"], P["emb_layer_norm.bias"], eps)
    if emb_keep is not None:
        x = x * emb_keep * scale
    x = x * keep[..., None]
    z0 = bias.view(B, H, L, L).masked_fill(pad[:, None, None, :], NEG_INF)
    z = z0
    for i in range(layers):
        x, z = _pair_layer64(P, "layers.{}.".format(i), x, z, H, eps, attn[i], res[2 * i:2 * i + 2], scale)
    x_norm = ((keep * _excess_norm(x)).sum(-1) / (1e-10 + keep.sum(-1))).mean()
    x = F.layer_norm(x, (E,), P["final_layer_norm.weight"], P["final_layer_norm.bias"], eps)
    pair = _pair_major(z)
    delta = pair - _pair_major(z0)
    pair_keep = keep[..., None] * keep[..., None, :]
    delta_norm = ((pair_keep * _excess_norm(delta)).sum((-1, -2)) / (1e-10 + pair_keep.sum((-1, -2)))).mean()
    delta = F.layer_norm(delta, (H,), P["final_head_layer_norm.weight"], P["final_head_layer_norm.bias"], eps)
    return (x, pair, delta, x_norm, delta_norm), z


# (B, N, {molecule: first padded position}).  tiles: molecule 1 is padded from 60, so keys 64..127 are a whole -inf
# tile from layer 2 on; small: one partial tile; bench: the benchmark's molecule sizes, padded off the 64 grid
STACK_SHAPES = {
    "tiles": (4, 136, {1: 60, 2: 97, 3: 129}),
    "small": (4, 24, {1: 13, 2: 19}),
    "bench": (8, 256, {1: 67, 2: 100, 3: 141, 4: 190, 5: 203, 6: 231}),
}
STACK_CASES = [(d, s) for s in STACK_SHAPES for d in DTYPES if s != "bench" or d == torch.bfloat16]
STACK_LAYERS = 3


@pytest.mark.parametrize("p", [0.0, 0.1], ids=["p0", "p0.1"])
@pytest.mark.parametrize("dtype,shape", STACK_CASES,
                         ids=["{}-{}".format("fp16" if d == torch.float16 else "bf16", s) for d, s in STACK_CASES])
def test_pair_stack_against_fp64(dtype, shape, p, monkeypatch):
    """Three pre-LN layers of ``TransformerEncoderWithPair`` at Uni-Mol widths (E = 512, 64 heads of dim 8, ffn 2048,
    head LayerNorm on), a per-molecule pair bias that requires grad, padded molecules, embedding, attention and residual
    dropout p: the five outputs and every gradient against float64 with the kernels' own masks, under random upstream
    gradients on all five outputs.  Exactly: the input pair bias gets a zero gradient at every padded key column, and
    ``pair`` is 0 where the reference's logits are ``-inf`` (exactly the padded key columns)."""
    import unicore_b200.models.unimol as unimol
    from unicore_b200.models.unimol import TransformerEncoderWithPair

    B, L, pads = STACK_SHAPES[shape]
    E, H = 512, 64
    torch.manual_seed(23)
    enc = TransformerEncoderWithPair(encoder_layers=STACK_LAYERS, embed_dim=E, ffn_embed_dim=4 * E, attention_heads=H,
                                     emb_dropout=p, dropout=p, attention_dropout=p, activation_dropout=0.0,
                                     max_seq_len=512).cuda()
    _perturb(enc)
    with torch.no_grad():   # an embedding norm above sqrt(E) + 1, so that the x-norm term and its gradient are not 0
        enc.emb_layer_norm.weight.mul_(1.5)
    enc = enc.to(dtype).train()
    emb = torch.randn(B, L, E, device="cuda").to(dtype).requires_grad_(True)
    bias = torch.randn(B * H, L, L, device="cuda").to(dtype).requires_grad_(True)
    pad = torch.zeros(B, L, dtype=torch.bool, device="cuda")
    for b, start in pads.items():
        pad[b, start:] = True

    spy, drop = _spies(monkeypatch)
    monkeypatch.setattr(unimol, "F", drop)
    outs = enc(emb, attn_mask=bias, padding_mask=pad)
    grads = [torch.randn(o.shape, device="cuda").to(o.dtype) for o in outs]
    torch.autograd.backward(list(outs), grads)

    assert len(spy.attn) == STACK_LAYERS and not spy.ln
    assert len(drop.keeps) == (1 + 2 * STACK_LAYERS if p > 0 else 0)
    attn = [_attention_keep(rec[0], rec[1], L) for rec in spy.attn]
    assert all((keep is None) == (p == 0) for keep, _ in attn)
    emb_keep, res = None, [None] * (2 * STACK_LAYERS)
    if p > 0:
        emb_keep, res = drop.keeps[0][1], [keep for _, keep, _ in drop.keeps[1:]]
        for i, (keep, _) in enumerate(attn):
            _check_keep_rate(keep, p, "attention {}".format(i))
        for i, keep in enumerate(res):
            _check_keep_rate(keep, p, "residual {}".format(i))
        _check_keep_rate(emb_keep, p, "embedding")
        streams = [rec[2] for rec in spy.attn] + [rec[2] for rec in drop.keeps]
        assert len(set(streams)) == len(streams), streams

    P = {n: t.detach().double().requires_grad_(True) for n, t in enc.named_parameters()}
    emb64 = emb.detach().double().requires_grad_(True)
    bias64 = bias.detach().double().requires_grad_(True)
    refs, z = _pair_stack64(P, emb64, bias64, pad, H, STACK_LAYERS, enc.emb_layer_norm.eps, emb_keep, attn, res, p)
    torch.autograd.backward(list(refs), [g.double() for g in grads])

    padded_keys = pad[:, None, None, :].expand(B, H, L, L)
    assert bool((bias.grad.view(B, H, L, L)[padded_keys] == 0).all()), \
        "the input pair bias must get an exactly zero gradient at padded key columns"
    ref_inf = torch.isinf(z).permute(0, 2, 3, 1)
    assert torch.equal(ref_inf, pad[:, None, :, None].expand(B, L, L, H))
    assert bool((outs[1][ref_inf] == 0).all()), "pair must be 0 where the logits are -inf"

    for name, got, ref in zip(("x", "pair", "delta", "x_norm", "delta_norm"), outs, refs):
        _check(got, ref, dtype, "output", name)
    _check(emb.grad, emb64.grad, dtype, "dx", "d emb")
    _check(bias.grad, bias64.grad, dtype, "dbias", "d pair-bias")
    for name, param in enc.named_parameters():
        assert param.grad is not None, name
        _check(param.grad, P[name].grad, dtype, _param_class(name), name)


# ------------------------------------------------------------------------------------------------------------------
# the Uni-Mol model and loss the benchmark trains, through the Trainer, against the portable plug-in in float64
# ------------------------------------------------------------------------------------------------------------------
TERMS = ("masked_token_loss", "masked_coord_loss", "masked_dist_loss", "x_norm_loss", "delta_pair_repr_norm_loss")


def _molecules(ds):
    """Four molecules whose collated batch is 136 wide (padded to a multiple of 8): the widest has 127 to 134 atoms
    (a count off the multiples of 8), one has at most 60 (keys 64..127 are a whole padded tile), two lie in between."""
    tokens = [len(ds[i]["src_tokens"]) for i in range(len(ds))]   # atoms + [CLS] + [SEP]
    wide = next(i for i, n in enumerate(tokens) if 129 <= n <= 136 and (n - 2) % 8)
    small = next(i for i, n in enumerate(tokens) if n - 2 <= 60)
    mid = [i for i, n in enumerate(tokens) if 62 < n <= 128][:2]
    return [wide, small] + mid


def _unimol_trainer(precision, extra):
    importlib.import_module("unimol")
    from unicore import options, tasks
    from unicore.trainer import Trainer

    parser = options.get_training_parser()
    args = options.parse_args_and_arch(parser, input_args=[
        "--task", "synthetic_unimol", "--loss", "unimol", "--arch", "unimol_base", "--encoder-layers", "2",
        "--synthetic-num-samples", "256", "--synthetic-min-atoms", "20", "--synthetic-max-atoms", "134",
        "--optimizer", "adam", "--lr", "1e-4", "--lr-scheduler", "fixed", "--max-update", "10", "--batch-size", "4",
        precision, "--seed", "5", "--dropout", "0.0", "--attention-dropout", "0.0", "--emb-dropout", "0.0",
        "--activation-dropout", "0.0",
        "--distributed-world-size", "1", "--no-save", "--disable-validation", "--log-format", "none",
    ] + extra)
    torch.manual_seed(0)
    task = tasks.setup_task(args)
    model = task.build_model(args)
    with torch.no_grad():
        # init_bert_params redraws the Gaussian basis from N(0, 0.02): widths down to 1e-4 make spikes whose
        # parameter gradients no 16-bit evaluation gets within hundreds of u of float64 (a plain PyTorch bf16 run of
        # the portable formulation is as far off as the kernels).  Widths from 0.5 keep the comparison conditioned.
        gbf = model.gbf
        gbf.means.weight.uniform_(0.0, 3.0)
        gbf.stds.weight.uniform_(0.5, 3.0)
        gbf.mul.weight.normal_(1.0, 0.1)
        gbf.bias.weight.normal_(0.0, 0.1)
    loss = task.build_loss(args)
    trainer = Trainer(args, task, model, loss)
    trainer._total_train_steps = args.max_update
    task.load_dataset("train")
    ds = task.dataset("train")
    batch = ds.collater([ds[i] for i in _molecules(ds)])
    return trainer, batch


def _unimol_step(trainer, batch):
    """Forward + backward of one batch through the Trainer's task step; returns the loss, the five logged terms, the
    masked-token logits and every parameter's gradient read from the flat arena, divided by the loss scale (fp16)."""
    from unicore import utils

    trainer.zero_grad()
    trainer.model.train()
    model = trainer.get_model()
    seen = []
    hook = model.lm_head.register_forward_hook(lambda m, i, out: seen.append(out.detach().clone()))
    try:
        loss, _, log = trainer.task.train_step(utils.move_to_cuda(batch), trainer.model, trainer.loss,
                                               trainer.optimizer, 0)
    finally:
        hook.remove()
    torch.cuda.synchronize()
    arenas = [f.grad for g in trainer.optimizer.fp16_params for f in g["params"]]
    scaler = trainer.optimizer.scaler
    scale = 1.0 if scaler is None else float(scaler.loss_scale)
    grads = {}
    for name, param in model.named_parameters():
        g = param.grad
        assert g is not None, name
        assert any(g.untyped_storage().data_ptr() == a.untyped_storage().data_ptr() for a in arenas), \
            name + ": the gradient is not in the flat arena"
        grads[name] = g.double() / scale
    terms = {k: torch.as_tensor(log[k]).double() for k in TERMS}
    return loss.detach().double(), terms, seen[0], grads


def _float64(sample):
    if isinstance(sample, dict):
        return {k: _float64(v) for k, v in sample.items()}
    return sample.double() if sample.is_floating_point() else sample


@pytest.mark.parametrize("precision", ["--bf16", "--fp16"], ids=["bf16", "fp16"])
def test_unimol_model_against_fp64(precision):
    """``unimol_base`` with 2 layers (E = 512, 64 heads, K = 128 Gaussians), dropout off, B = 4 molecules collated to
    N = 136 with one of at most 60 atoms, through the Trainer with the gradient sinks (parameter gradients written into
    the flat arena by the backward kernels) and without them: the loss, its five terms, the masked-token logits and
    every parameter gradient against the portable plug-in loaded from the same weights and run in float64 on no
    native kernel."""
    from unicore import utils
    from unicore_b200.ops._native import launch_counter_read

    _ops()
    importlib.import_module("unimol_portable")
    from unimol_portable.model import PortableUniMol, PortableUniMolLoss

    dtype = torch.bfloat16 if precision == "--bf16" else torch.float16
    runs = {}
    for mode, extra in (("sinks", []), ("no_sinks", ["--no-grad-sinks"])):
        trainer, batch = _unimol_trainer(precision, extra)
        assert batch["net_input"]["src_tokens"].shape == (4, 136)
        runs[mode] = _unimol_step(trainer, batch)
        model = trainer.get_model()
        assert next(model.parameters()).dtype == dtype
        sinks = sum(1 for p in model.parameters() if getattr(p, "_ub_direct_grad", False))
        assert (sinks > 0) == (mode == "sinks"), (mode, sinks)
        if mode == "sinks":
            ref = PortableUniMol(copy.copy(model.args), trainer.task.dictionary)
            ref.load_state_dict(model.state_dict(), strict=True)
            ref = ref.double().cuda()
            weights = {n: p.detach().clone() for n, p in model.named_parameters()}
            loss_fn, sample = PortableUniMolLoss(trainer.task), batch
        else:
            for n, p in model.named_parameters():
                assert torch.equal(p.detach(), weights[n]), n + ": the two runs must start from the same weights"
        del trainer, model

    ref.train()
    seen = []
    hook = ref.lm_head.register_forward_hook(lambda m, i, out: seen.append(out.detach()))
    before = launch_counter_read()
    try:
        loss64, _, log64 = loss_fn(ref, _float64(utils.move_to_cuda(sample)))
        loss64.backward()
    finally:
        hook.remove()
    assert launch_counter_read() == before, "the float64 reference must not reach a native kernel"
    assert loss64.dtype == torch.float64 and seen[0].dtype == torch.float64
    for k in TERMS:
        assert float(log64[k]) != 0, k + ": every term of the loss must take part"
    grads64 = dict((n, p.grad) for n, p in ref.named_parameters())
    for name in ("gbf.means.weight", "gbf.stds.weight", "gbf.mul.weight", "gbf.bias.weight", "gbf_proj.linear1.weight",
                 "pair2coord_proj.linear2.bias", "dist_head.out_proj.weight", "embed_tokens.weight"):
        assert grads64.get(name) is not None, name

    for mode, (loss, terms, logits, grads) in runs.items():
        _check(loss, loss64, dtype, "output", mode + ": loss")
        for k in TERMS:
            _check(terms[k], log64[k], dtype, "output", "{}: {}".format(mode, k))
        _check(logits, seen[0], dtype, "output", mode + ": masked-token logits")
        assert set(grads) == set(grads64), mode
        for name, g in grads.items():
            assert grads64[name] is not None, name
            _check(g, grads64[name], dtype, _param_class(name), "{}: {}".format(mode, name))
