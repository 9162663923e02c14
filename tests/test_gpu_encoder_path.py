"""The encoder path that BERT masked-LM training runs, composed, against float64 formulations of the same maths.

Every kernel on the path has its own exact test; these tests check that they compose: the residual each fused
``bias_dropout_add_layer_norm`` receives, the dropout masks its backward regenerates after the attention kernel has
reserved Philox counters in between, the batch-shared bias gradient and its way into ``relative_attention_bias`` through
the one-hot GEMM, padded rows, and parameter gradients written straight into the flat arena by the backward kernels.

Dropout is compared element for element, with the kernels' own masks:
* attention: the keep bits ``[B, H, Lq, ceil(Lk / 32)]`` the forward returns, in the layout of
  ``csrc/attn/fmha_api.h`` (key ``32w + 2i`` in bit ``i``, key ``32w + 2i + 1`` in bit ``16 + i``), kept elements scaled
  by ``16384 / (16384 - round(p * 16384))``;
* the fused bias + dropout + residual + LayerNorm: its ``(seed, offset)`` replayed on a probe (x = 1, bias = residual
  = 0), whose kept elements are the nonzeros of ``summed``; kept elements are scaled by ``1 / (1 - p)``;
* torch's ``F.dropout`` in ``unicore.modules.transformer`` (embedding dropout, pre-LN residual dropout): replaced by a
  dropout that draws its mask explicitly and records it.

Every tensor meets ``max|got - ref| <= c * u * max|ref|``, ``u`` the unit roundoff of the 16-bit type (2^-11 for fp16,
2^-8 for bf16), with one ``c`` per class of tensor (``C``).  The classes are the output (layer output, loss, logits),
dx (the gradient of the layer or stack input), weight gradients (GEMM weights, LayerNorm gains, the token embedding),
bias gradients (GEMM and LayerNorm biases) and dbias (the gradient of the ``[1, H, L, L]`` attention bias, or of the
relative-position table it is looked up from).

Calibration: the worst ratio ``max|got - ref| / (u * max|ref|)`` observed per class over every test here at p = 0, on
an H100 80GB HBM3 (700 W power limit); each ``c`` is at most 4x the worst observed value.

    =========  ====  ====  ==
    class      fp16  bf16  c
    =========  ====  ====  ==
    output     2.22  2.45  8
    dx         1.99  1.88  7
    weight     2.77  1.64  8
    bias       1.91  1.34  6
    dbias      2.27  2.14  8
    =========  ====  ====  ==

At p = 0.1 the worst ratios are below these, except in the two-layer stack with every dropout on (output 2.98, dx
3.69, dbias 3.24), which is still inside ``c``.  The fp16 weight, bias and dbias columns are set by the BERT model
(its token embedding, LM-head bias and relative-position table); the other entries by single layers.
"""
import copy
import importlib
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UNIT = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
DTYPES = [torch.float16, torch.bfloat16]
C = {"output": 8, "dx": 7, "weight": 8, "bias": 6, "dbias": 8}
# worst ratio max|got - ref| / (u * max|ref|) per (class, dtype) seen in this process: what the table above is made of
OBSERVED = {}

# (B, L, E, H, {sequence: first padded position}); the bench shape pads at positions off the 64-row tiles
SHAPES = {
    "bench": (4, 512, 768, 12, {1: 300, 3: 481}),
    "ragged": (3, 200, 768, 12, {2: 137}),
    "d128": (2, 264, 1024, 8, {1: 201}),
}


def _ops():
    from unicore import ops

    assert ops.USE_NATIVE, "native kernels must be active on the GPU box"
    return ops


def _check(got, ref, dtype, cls, what):
    got, ref = got.detach().double(), ref.detach().double()
    assert got.shape == ref.shape, (what, tuple(got.shape), tuple(ref.shape))
    assert bool(torch.isfinite(got).all()), what + ": not finite"
    scale = UNIT[dtype] * ref.abs().max().item()
    err = (got - ref).abs().max().item()
    ratio = err / scale if scale > 0 else (0.0 if err == 0 else math.inf)
    key = (cls, str(dtype).replace("torch.", ""))
    OBSERVED[key] = max(OBSERVED.get(key, 0.0), ratio)
    assert ratio <= C[cls], "{}: max|got - ref| = {:.3g} = {:.3g} u max|ref| (bound {} u max|ref|)".format(
        what, err, ratio, C[cls])


def _param_class(name):
    if "relative_attention_bias" in name:
        return "dbias"
    return "bias" if name.endswith("bias") else "weight"


def _padding(B, L, pads):
    pad = torch.zeros(B, L, dtype=torch.bool, device="cuda")
    for b, start in pads.items():
        pad[b, start:] = True
    return pad


def _perturb(module):
    """Non-trivial LayerNorm gains / shifts and biases (the modules start them at 1 and 0)."""
    with torch.no_grad():
        for name, p in module.named_parameters():
            p.add_(torch.randn_like(p) * (0.1 if "layer_norm" in name else 0.02))


# ------------------------------------------------------------------------------------------------------------------
# the kernels' own dropout masks
# ------------------------------------------------------------------------------------------------------------------
def _generator():
    return torch.cuda.default_generators[torch.cuda.current_device()]


class _KernelSpy:
    """Forwards to the extension; records the keep bits of every fused attention forward and the ``(seed, offset)`` of
    every fused bias + dropout + residual + LayerNorm forward."""

    def __init__(self, real):
        self._real = real
        self.attn = []   # (p, keep bits or None, (seed, offset) the call reserved)
        self.ln = []     # ((rows, cols), dtype, p, seed, offset)

    def __getattr__(self, name):
        return getattr(self._real, name)

    def _attention(self, fn, args, kwargs):
        gen = _generator()
        stream = (gen.initial_seed(), gen.get_offset())
        res = fn(*args, **kwargs)
        self.attn.append((float(args[5]), res[2], stream))
        return res

    def fmha_fwd(self, *args, **kwargs):
        return self._attention(self._real.fmha_fwd, args, kwargs)

    def fmha_fwd_logits(self, *args, **kwargs):
        return self._attention(self._real.fmha_fwd_logits, args, kwargs)

    def bias_dropout_add_ln_fwd(self, x, bias, residual, gamma, beta, p, eps):
        res = self._real.bias_dropout_add_ln_fwd(x, bias, residual, gamma, beta, p, eps)
        self.ln.append((tuple(x.shape), x.dtype, float(p), res[4], res[5]))
        return res


class _DropoutSpy:
    """``torch.nn.functional`` for ``unicore.modules.transformer``, with a dropout that draws its keep mask explicitly
    (``rand >= p``, kept elements scaled by ``1 / (1 - p)`` in fp32) and records it."""

    def __init__(self):
        self.keeps = []   # (p, keep mask, (seed, offset) the draw used)

    def __getattr__(self, name):
        return getattr(F, name)

    def dropout(self, input, p=0.5, training=True, inplace=False):
        if not training or p == 0:
            return F.dropout(input, p, training, inplace)
        gen = _generator()
        stream = (gen.initial_seed(), gen.get_offset())
        keep = torch.rand(input.shape, device=input.device) >= p
        self.keeps.append((float(p), keep, stream))
        return (input.float() * keep * (1.0 / (1.0 - p))).to(input.dtype)


def _spies(monkeypatch):
    import unicore.modules.transformer as transformer
    import unicore_b200.ops.attention_ops as attention_ops
    import unicore_b200.ops.fused_ops as fused_ops

    spy, drop = _KernelSpy(_ops().native()), _DropoutSpy()
    monkeypatch.setattr(attention_ops, "native", lambda: spy)
    monkeypatch.setattr(fused_ops, "native", lambda: spy)
    monkeypatch.setattr(transformer, "F", drop)
    return spy, drop


_BIT_OF_KEY = [j // 2 if j % 2 == 0 else 16 + j // 2 for j in range(32)]


def _attention_keep(p, bits, Lk):
    """``[B, H, Lq, Lk]`` keep mask of the forward's keep words, and the keep scale; (None, 1) without dropout."""
    if p == 0:
        return None, 1.0
    shift = torch.tensor(_BIT_OF_KEY, device=bits.device)
    words = bits.long() & 0xFFFFFFFF
    keep = ((words[..., None] >> shift) & 1).flatten(-2)[..., :Lk].bool()
    t14 = min(max(int(p * 16384.0 + 0.5), 0), 16383)
    return keep, 16384.0 / (16384.0 - t14)


def _residual_keep(rec):
    """Replays a fused bias + dropout + residual + LayerNorm forward's dropout on a probe: returns its ``[rows, cols]``
    keep mask (None without dropout)."""
    (rows, cols), dtype, p, seed, offset = rec
    if p == 0:
        return None
    real = _ops().native()
    gen = _generator()
    state = gen.get_state()
    try:
        gen.manual_seed(seed % 2 ** 64)
        gen.set_offset(offset)
        ones = torch.ones(rows, cols, dtype=dtype, device="cuda")
        zero_col = torch.zeros(cols, dtype=dtype, device="cuda")
        one_col = torch.ones(cols, dtype=dtype, device="cuda")
        _, _, _, summed, seed2, offset2 = real.bias_dropout_add_ln_fwd(ones, zero_col, torch.zeros_like(ones), one_col,
                                                                      zero_col, p, 1e-5)
    finally:
        gen.set_state(state)
    assert (seed2, offset2) == (seed, offset), "the probe must draw the stream of the call it replays"
    return summed != 0


def _residual_keeps(spy, drop, post_ln, shape, count):
    """Keep masks of the ``count`` residual dropouts in call order (Nones without dropout): the fused LayerNorm calls
    on the post-LN path, torch's dropout on the pre-LN path."""
    if post_ln:
        return [None if k is None else k.view(shape) for k in map(_residual_keep, spy.ln)]
    return [keep for _, keep, _ in drop.keeps] or [None] * count


def _check_keep_rate(keep, p, what):
    n = keep.numel()
    rate = keep.double().mean().item()
    sigma = math.sqrt(p * (1 - p) / n)
    assert abs(rate - (1 - p)) <= 6 * sigma, "{}: keep rate {:.6f}, want {} +- 6 x {:.2g}".format(what, rate, 1 - p,
                                                                                                  sigma)


# ------------------------------------------------------------------------------------------------------------------
# float64 formulation of one encoder layer
# ------------------------------------------------------------------------------------------------------------------
def _layer64(P, pre, x, bias, pad, H, post_ln, eps, attn_drop, res_keeps, res_scale):
    """``TransformerEncoderLayer`` (GELU, activation dropout 0) in float64.  ``P``: float64 parameters by name, ``pre``
    the name prefix of this layer; ``bias`` ``[1|B, H, L, L]``; ``pad`` ``[B, L]`` (True = padded key);
    ``attn_drop``: (keep ``[B, H, L, L]`` or None, keep scale); ``res_keeps``: two keep masks ``[B, L, E]`` or Nones."""
    B, L, E = x.shape
    D = E // H

    def w(name):
        return P[pre + name]

    def attn(h):
        qkv = F.linear(h, w("self_attn.in_proj.weight"), w("self_attn.in_proj.bias")).view(B, L, 3, H, D)
        q, k, v = qkv.unbind(2)
        s = torch.einsum("bqhd,bkhd->bhqk", q, k) * D ** -0.5 + bias
        s = s.masked_fill(pad[:, None, None, :], float("-inf"))
        pr = torch.softmax(s, dim=-1)
        keep, scale = attn_drop
        if keep is not None:
            pr = pr * keep * scale
        o = torch.einsum("bhqk,bkhd->bqhd", pr, v).reshape(B, L, E)
        return F.linear(o, w("self_attn.out_proj.weight"), w("self_attn.out_proj.bias"))

    def ffn(h):
        return F.linear(F.gelu(F.linear(h, w("fc1.weight"), w("fc1.bias"))), w("fc2.weight"), w("fc2.bias"))

    def drop(t, i):
        return t if res_keeps[i] is None else t * res_keeps[i] * res_scale

    def ln1(t):
        return F.layer_norm(t, (E,), w("self_attn_layer_norm.weight"), w("self_attn_layer_norm.bias"), eps)

    def ln2(t):
        return F.layer_norm(t, (E,), w("final_layer_norm.weight"), w("final_layer_norm.bias"), eps)

    if post_ln:
        x = ln1(x + drop(attn(x), 0))
        return ln2(x + drop(ffn(x), 1))
    x = x + drop(attn(ln1(x)), 0)
    return x + drop(ffn(ln2(x)), 1)


def _params64(module):
    return {n: p.detach().double().requires_grad_(True) for n, p in module.named_parameters()}


# ------------------------------------------------------------------------------------------------------------------
# one layer, forward and every gradient
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("p", [0.0, 0.1], ids=["p0", "p0.1"])
@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
@pytest.mark.parametrize("post_ln", [True, False], ids=["post_ln", "pre_ln"])
def test_encoder_layer_against_fp64(post_ln, dtype, p, shape, monkeypatch):
    """The fused path of ``TransformerEncoderLayer`` (wgmma attention with a ``[1, H, L, L]`` bias that requires grad,
    key padding, attention and residual dropout p, fused bias + dropout + residual + LayerNorm or pre-LN norms,
    bias-GELU, column-sum bias gradients) against float64 with the kernels' own masks."""
    from unicore.modules import TransformerEncoderLayer

    B, L, E, H, pads = SHAPES[shape]
    torch.manual_seed(17)
    layer = TransformerEncoderLayer(embed_dim=E, ffn_embed_dim=4 * E, attention_heads=H, dropout=p,
                                    attention_dropout=p, activation_dropout=0.0, post_ln=post_ln).cuda()
    _perturb(layer)
    layer = layer.to(dtype).train()
    x = torch.randn(B, L, E, device="cuda").to(dtype).requires_grad_(True)
    bias = (torch.randn(1, H, L, L, device="cuda") * 0.5).to(dtype).requires_grad_(True)
    pad = _padding(B, L, pads)
    dy = torch.randn(B, L, E, device="cuda").to(dtype)

    spy, drop = _spies(monkeypatch)
    y = layer(x, attn_bias=bias, padding_mask=pad)
    y.backward(dy)

    assert len(spy.attn) == 1 and len(spy.ln) == (2 if post_ln else 0)
    attn_drop = _attention_keep(spy.attn[0][0], spy.attn[0][1], L)
    res_keeps = _residual_keeps(spy, drop, post_ln, (B, L, E), 2)
    assert len(res_keeps) == 2 and all((k is None) == (p == 0) for k in res_keeps + [attn_drop[0]])

    P = _params64(layer)
    x64 = x.detach().double().requires_grad_(True)
    bias64 = bias.detach().double().requires_grad_(True)
    y64 = _layer64(P, "", x64, bias64, pad, H, post_ln, layer.final_layer_norm.eps, attn_drop, res_keeps,
                   1.0 / (1.0 - p) if p > 0 else 1.0)
    y64.backward(dy.double())

    _check(y, y64, dtype, "output", "y")
    _check(x.grad, x64.grad, dtype, "dx", "dx")
    _check(bias.grad, bias64.grad, dtype, "dbias", "dbias")
    for name, param in layer.named_parameters():
        assert param.grad is not None, name
        _check(param.grad, P[name].grad, dtype, _param_class(name), name)


# ------------------------------------------------------------------------------------------------------------------
# a post-LN stack with every dropout on: embedding dropout, relative-position bias, masks across layers
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=["fp16", "bf16"])
def test_encoder_stack_with_dropout_against_fp64(dtype, monkeypatch):
    """Two post-LN layers at BERT-base widths under ``TransformerEncoder`` (embedding LayerNorm + dropout, padded rows
    zeroed, relative-position bias from the one-hot GEMM shared by the batch and both layers), dropout 0.1 everywhere
    as in BERT, against float64 with the recovered masks.  The recovered masks keep at the configured rate, and no two
    dropouts of the step share a Philox stream."""
    from unicore.modules import TransformerEncoder

    B, L, E, H, pads = SHAPES["bench"]
    p = 0.1
    torch.manual_seed(29)
    enc = TransformerEncoder(encoder_layers=2, embed_dim=E, ffn_embed_dim=4 * E, attention_heads=H, emb_dropout=p,
                             dropout=p, attention_dropout=p, activation_dropout=0.0, max_seq_len=L, rel_pos=True,
                             post_ln=True).cuda()
    _perturb(enc)
    with torch.no_grad():   # the table starts at zero in the module; give the bias a size the softmax notices
        enc.relative_attention_bias.weight.normal_(0.0, 0.5)
    enc = enc.to(dtype).train()
    emb = torch.randn(B, L, E, device="cuda").to(dtype).requires_grad_(True)
    pad = _padding(B, L, pads)
    dy = torch.randn(B, L, E, device="cuda").to(dtype)

    spy, drop = _spies(monkeypatch)
    y = enc(emb, padding_mask=pad)
    y.backward(dy)

    assert len(spy.attn) == 2 and len(spy.ln) == 4 and len(drop.keeps) == 1
    attn = [_attention_keep(rec[0], rec[1], L) for rec in spy.attn]
    res = _residual_keeps(spy, drop, True, (B, L, E), 4)
    emb_keep = drop.keeps[0][1]
    for i, (keep, _) in enumerate(attn):
        _check_keep_rate(keep, p, "attention {}".format(i))
    for i, keep in enumerate(res):
        _check_keep_rate(keep, p, "residual {}".format(i))
    _check_keep_rate(emb_keep, p, "embedding")
    streams = [rec[2] for rec in spy.attn] + [(rec[3], rec[4]) for rec in spy.ln] + [drop.keeps[0][2]]
    assert len(set(streams)) == len(streams), streams

    P = _params64(enc)
    emb64 = emb.detach().double().requires_grad_(True)
    eps = enc.emb_layer_norm.eps
    x = F.layer_norm(emb64, (E,), P["emb_layer_norm.weight"], P["emb_layer_norm.bias"], eps)
    x = x * emb_keep / (1 - p)
    x = x * (~pad)[..., None]
    bucket = enc.rp_bucket[:L, :L].to("cuda")
    rel = F.embedding(bucket, P["relative_attention_bias.weight"]).permute(2, 0, 1).unsqueeze(0)
    for i in range(2):
        x = _layer64(P, "layers.{}.".format(i), x, rel, pad, H, True, eps, attn[i], res[2 * i:2 * i + 2], 1 / (1 - p))
    x.backward(dy.double())

    _check(y, x, dtype, "output", "y")
    _check(emb.grad, emb64.grad, dtype, "dx", "d emb")
    for name, param in enc.named_parameters():
        assert param.grad is not None, name
        _check(param.grad, P[name].grad, dtype, _param_class(name), name)


# ------------------------------------------------------------------------------------------------------------------
# the BERT model the benchmark trains, built through the Trainer
# ------------------------------------------------------------------------------------------------------------------
BERT_PADS = {1: 300, 3: 481}


def _bert_trainer(extra):
    sys.path.insert(0, os.path.join(ROOT, "examples"))
    importlib.import_module("bert")
    from unicore import options, tasks
    from unicore.trainer import Trainer

    parser = options.get_training_parser()
    args = options.parse_args_and_arch(parser, input_args=[
        "--task", "synthetic_mlm", "--loss", "masked_lm", "--arch", "bert_base", "--encoder-layers", "2",
        "--synthetic-vocab-size", "30522", "--synthetic-seq-len", "512", "--max-seq-len", "512",
        "--optimizer", "adam", "--lr", "1e-4", "--lr-scheduler", "fixed", "--max-update", "10", "--batch-size", "4",
        "--fp16", "--fp16-init-scale", "16", "--seed", "3", "--dropout", "0.0", "--attention-dropout", "0.0",
        "--emb-dropout", "0.0", "--activation-dropout", "0.0",
        "--distributed-world-size", "1", "--no-save", "--disable-validation", "--log-format", "none",
    ] + extra)
    torch.manual_seed(0)
    task = tasks.setup_task(args)
    model = task.build_model(args)
    loss = task.build_loss(args)
    trainer = Trainer(args, task, model, loss)
    trainer._total_train_steps = args.max_update
    task.load_dataset("train")
    ds = task.dataset("train")
    batch = ds.collater([ds[i] for i in range(4)])
    pad = task.dictionary.pad()
    for b, start in BERT_PADS.items():   # two padded sequences
        batch["net_input"]["src_tokens"][b, start:] = pad
        batch["target"][b, start:] = pad
    return trainer, batch


def _bert_step(trainer, batch):
    """Forward + backward of one batch through the Trainer's task step; returns the loss, the masked-token logits
    and every parameter's gradient read from the flat arena, divided by the loss scale."""
    from unicore import utils

    trainer.zero_grad()
    trainer.model.train()
    model = trainer.get_model()
    seen = []
    hook = model.lm_head.register_forward_hook(lambda m, i, out: seen.append(out.detach().clone()))
    try:
        loss, _, _ = trainer.task.train_step(utils.move_to_cuda(batch), trainer.model, trainer.loss, trainer.optimizer,
                                             0)
    finally:
        hook.remove()
    torch.cuda.synchronize()
    arenas = [f.grad for g in trainer.optimizer.fp16_params for f in g["params"]]
    scale = float(trainer.optimizer.scaler.loss_scale)
    grads = {}
    for name, param in model.named_parameters():
        g = param.grad
        assert g is not None, name
        assert any(g.untyped_storage().data_ptr() == a.untyped_storage().data_ptr() for a in arenas), \
            name + ": the gradient is not in the flat arena"
        grads[name] = g.double() / scale
    return loss.detach().double(), seen[0], grads


def test_bert_masked_lm_against_fp64():
    """BERT-base widths (E = 768, H = 12, vocab 30,522, L = 512, B = 4) with 2 layers, 15 % masked tokens, two padded
    sequences, dropout off, fp16 through the Trainer: the loss, the masked-token logits and every parameter gradient,
    with the gradient sinks (parameter gradients written into the flat arena by the backward kernels) and without
    them, against a float64 copy of the model that runs no native kernel."""
    from unicore_b200.ops._native import launch_counter_read

    _ops()
    dtype = torch.float16
    runs = {}
    for mode, extra in (("sinks", []), ("no_sinks", ["--no-grad-sinks"])):
        trainer, batch = _bert_trainer(extra)
        runs[mode] = _bert_step(trainer, batch)
        sinks = sum(1 for p in trainer.get_model().parameters() if getattr(p, "_ub_direct_grad", False))
        assert (sinks > 0) == (mode == "sinks"), (mode, sinks)
        if mode == "sinks":
            model = trainer.get_model()
            ref = copy.deepcopy(model).double()
            weights = {n: p.detach().clone() for n, p in model.named_parameters()}
            loss_fn, sample = trainer.loss, batch
        else:
            for n, p in trainer.get_model().named_parameters():
                assert torch.equal(p.detach(), weights[n]), n + ": the two runs must start from the same weights"
        del trainer

    from unicore import utils

    ref.train()
    seen = []
    hook = ref.lm_head.register_forward_hook(lambda m, i, out: seen.append(out.detach()))
    before = launch_counter_read()
    try:
        loss64, _, _ = loss_fn(ref, utils.move_to_cuda(sample))
        loss64.backward()
    finally:
        hook.remove()
    assert launch_counter_read() == before, "the float64 reference must not reach a native kernel"
    assert loss64.dtype == torch.float64 and seen[0].dtype == torch.float64
    grads64 = dict((n, p.grad) for n, p in ref.named_parameters())
    assert "embed_tokens.weight" in grads64 and "sentence_encoder.relative_attention_bias.weight" in grads64

    for mode, (loss, logits, grads) in runs.items():
        _check(loss, loss64, dtype, "output", mode + ": loss")
        _check(logits, seen[0], dtype, "output", mode + ": masked-token logits")
        assert set(grads) == set(grads64), mode
        for name, g in grads.items():
            assert grads64[name] is not None, name
            _check(g, grads64[name], dtype, _param_class(name), "{}: {}".format(mode, name))
