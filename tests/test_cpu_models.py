"""CPU tests of the model-side layers on their PyTorch fallbacks: pair-representation attention
(``return_attn``), decoder / cross attention, the Uni-Mol plug-in end to end through the Trainer,
Gaussian basis, NaN detector and progress bars (SURVEY.md section 4: the reference has no unit tests
for these; its example configs are the de-facto integration tests, mirrored here at toy size)."""
import importlib
import json
import logging
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "examples"))

from unicore import ops, options, tasks  # noqa: E402


def test_softmax_dropout_with_logits_matches_unfused_formulation():
    """z = x + mask + bias is an output with its own gradient path (reference multihead_attention.py:98-103)."""
    torch.manual_seed(0)
    x = torch.randn(2, 4, 6, 16, requires_grad=True)
    bias = torch.randn(2, 4, 6, 16, requires_grad=True)
    mask = torch.zeros(2, 1, 1, 16)
    mask[0, ..., -4:] = float("-inf")
    out, z = ops.softmax_dropout_with_logits(x, 0.0, True, mask=mask, bias=bias)
    zr = x + mask + bias
    assert torch.equal(z, zr)
    assert torch.allclose(out, torch.softmax(zr, -1), atol=1e-6)
    w = torch.randn_like(out)
    finite = torch.isfinite(z)
    (out * w).sum().backward(retain_graph=True)
    g_probs_only = x.grad.clone()
    x.grad = bias.grad = None
    ((out * w).sum() + z[finite].sum() * 0.5).backward()
    assert torch.allclose(x.grad, g_probs_only + 0.5 * finite.float(), atol=1e-6)
    assert torch.allclose(bias.grad, x.grad)
    # dropout keeps the expectation and the logits are unaffected by it
    out_d, z_d = ops.softmax_dropout_with_logits(x.detach(), 0.5, True, bias=bias.detach())
    assert torch.equal(z_d, x.detach() + bias.detach())
    kept = out_d != 0
    assert 0.3 < kept.float().mean().item() < 0.7
    assert torch.allclose(out_d[kept], 2.0 * torch.softmax(z_d, -1)[kept], atol=1e-6)


def test_pair_representation_threads_through_layers():
    """Logits of layer i are the bias of layer i+1; padding folded in once as -inf stays -inf."""
    from unicore.modules import TransformerEncoderLayer

    torch.manual_seed(1)
    layers = [TransformerEncoderLayer(embed_dim=32, ffn_embed_dim=64, attention_heads=4, dropout=0.0,
                                      attention_dropout=0.0, activation_dropout=0.0).eval() for _ in range(2)]
    x = torch.randn(2, 8, 32)
    pair = torch.randn(2 * 4, 8, 8, requires_grad=True)
    pad = torch.zeros(2, 8, dtype=torch.bool)
    pad[1, 6:] = True
    bias = pair.view(2, 4, 8, 8).masked_fill(pad[:, None, None, :], float("-inf")).view(8, 8, 8)
    h, b = x, bias
    for layer in layers:
        h, b, probs = layer(h, padding_mask=None, attn_bias=b, return_attn=True)
        assert b.shape == (8, 8, 8) and probs.shape == (8, 8, 8)
        assert torch.isinf(b.view(2, 4, 8, 8)[1, :, :, 6:]).all() and torch.isfinite(b.view(2, 4, 8, 8)[0]).all()
        assert probs.view(2, 4, 8, 8)[1, :, :, 6:].abs().max() == 0
        assert torch.allclose(probs.sum(-1), torch.ones(8, 8), atol=1e-5)
    delta = (b - bias).masked_fill(~torch.isfinite(bias), 0)
    (h.sum() + delta.sum()).backward()
    assert torch.isfinite(pair.grad).all() and pair.grad.abs().sum() > 0


def test_unimol_encoder_folds_padding_into_first_layer():
    """Padding enters through the first layer's softmax mask; result equals the reference's up-front -inf fill."""
    from unicore_b200.models.unimol import TransformerEncoderWithPair

    torch.manual_seed(4)
    enc = TransformerEncoderWithPair(encoder_layers=3, embed_dim=32, ffn_embed_dim=64, attention_heads=4, emb_dropout=0.0,
                                     dropout=0.0, attention_dropout=0.0, max_seq_len=16).eval()
    emb, pair = torch.randn(2, 8, 32), torch.randn(2 * 4, 8, 8)
    pad = torch.zeros(2, 8, dtype=torch.bool)
    pad[0, 5:] = True
    x, pair_out, delta, x_norm, delta_norm = enc(emb, attn_mask=pair, padding_mask=pad)
    h = enc.emb_layer_norm(emb) * (1 - pad.unsqueeze(-1).float())
    b = pair.view(2, 4, 8, 8).masked_fill(pad[:, None, None, :], float("-inf")).view(8, 8, 8)
    for layer in enc.layers:
        h, b, _ = layer(h, padding_mask=None, attn_bias=b, return_attn=True)
    ref_pair = b.view(2, 4, 8, 8).permute(0, 2, 3, 1)
    assert torch.isinf(ref_pair[0, :, 5:]).all() and (pair_out[0, :, 5:] == 0).all()  # -inf -> 0 on the way out
    assert torch.allclose(pair_out, ref_pair.masked_fill(torch.isinf(ref_pair), 0), atol=1e-5)
    ref_delta = (ref_pair - pair.view(2, 4, 8, 8).permute(0, 2, 3, 1)).masked_fill(pad[:, None, :, None], 0)
    if enc.final_head_layer_norm is not None:
        ref_delta = enc.final_head_layer_norm(ref_delta)
    assert torch.allclose(delta, ref_delta, atol=1e-4)
    assert torch.allclose(x, enc.final_layer_norm(h), atol=1e-5)
    assert torch.isfinite(delta).all() and torch.isfinite(x_norm) and torch.isfinite(delta_norm)


def test_decoder_is_causal_and_attends_to_encoder():
    from unicore.modules import CrossMultiheadAttention, TransformerDecoder

    torch.manual_seed(2)
    dec = TransformerDecoder(decoder_layers=2, embed_dim=32, ffn_embed_dim=64, attention_heads=4, emb_dropout=0.0,
                             dropout=0.0, attention_dropout=0.0, max_seq_len=16).eval()
    emb, enc = torch.randn(2, 10, 32), torch.randn(2, 7, 32)
    enc_pad = torch.zeros(2, 7, dtype=torch.bool)
    enc_pad[0, 5:] = True
    y = dec(emb, encoder_out=enc, encoder_padding_mask=enc_pad)
    assert y.shape == (2, 10, 32) and torch.isfinite(y).all()
    emb2 = emb.clone()
    emb2[:, 6:] += torch.randn(2, 4, 32)  # the future must not leak into positions < 6
    y2 = dec(emb2, encoder_out=enc, encoder_padding_mask=enc_pad)
    assert torch.allclose(y[:, :6], y2[:, :6], atol=1e-5) and not torch.allclose(y[:, 6:], y2[:, 6:], atol=1e-3)
    enc2 = enc.clone()
    enc2[0, 5:] += torch.randn(2, 32) * 3  # padded encoder positions are invisible
    assert torch.allclose(dec(emb, encoder_out=enc2, encoder_padding_mask=enc_pad)[0], y[0], atol=1e-5)
    fm = dec.get_future_mask(emb, None)
    assert fm.shape == (2 * 4, 10, 10) and torch.isinf(fm[0, 0, 1]) and fm[0, 1, 0] == 0
    cross = CrossMultiheadAttention(32, 4, dropout=0.0)
    q, kv = torch.randn(2, 5, 32), torch.randn(2, 9, 32)
    out = cross(q, kv, kv, attn_bias=torch.randn(8, 5, 9))
    assert out.shape == (2, 5, 32)
    names = set(dec.state_dict())
    assert {"layers.0.encoder_attn.q_proj.weight", "layers.0.encoder_attn_layer_norm.weight",
            "layers.1.self_attn.in_proj.bias"} <= names


def test_gaussian_basis_matches_reference_formula():
    """Fallback of the fused kernel against the closed form of Uni-Mol's GaussianLayer."""
    torch.manual_seed(3)
    B, L, K, T = 2, 6, 16, 5
    dist = torch.rand(B, L, L) * 8
    et = torch.randint(0, T * T, (B, L, L))
    mul = (torch.randn(T * T, 1) * 0.1 + 1).requires_grad_(True)
    bias = (torch.randn(T * T, 1) * 0.1).requires_grad_(True)
    mean = (torch.rand(K) * 3).requires_grad_(True)
    std = (torch.rand(K) * 3).requires_grad_(True)
    out = ops.gaussian_basis(dist, et, mul, bias, mean, std)
    x = (mul[et] * dist.unsqueeze(-1) + bias[et]).expand(-1, -1, -1, K)
    s = std.abs() + 1e-5
    ref = torch.exp(-0.5 * ((x - mean) / s) ** 2) / (((2 * 3.14159) ** 0.5) * s)
    assert out.shape == (B, L, L, K) and torch.allclose(out, ref, atol=1e-5, rtol=1e-4)
    g = torch.autograd.grad(out.sum(), [mul, bias, mean, std])
    gr = torch.autograd.grad(ref.sum(), [mul, bias, mean, std])
    for a, b in zip(g, gr):
        assert torch.allclose(a, b, atol=1e-4, rtol=1e-3)


def _unimol_trainer(extra=()):
    importlib.import_module("unimol")
    from unicore.trainer import Trainer

    parser = options.get_training_parser()
    args = options.parse_args_and_arch(parser, input_args=[
        "--task", "synthetic_unimol", "--loss", "unimol", "--arch", "unimol_base", "--encoder-layers", "2",
        "--encoder-embed-dim", "32", "--encoder-ffn-embed-dim", "64", "--encoder-attention-heads", "4",
        "--gaussian-kernels", "16", "--synthetic-num-samples", "16", "--synthetic-min-atoms", "6",
        "--synthetic-max-atoms", "14", "--optimizer", "adam", "--lr", "1e-3", "--lr-scheduler", "fixed",
        "--clip-norm", "1.0", "--max-update", "10", "--batch-size", "4", "--seed", "7", "--cpu",
        "--distributed-world-size", "1", "--no-save", "--disable-validation", "--log-format", "none",
    ] + list(extra))
    task = tasks.setup_task(args)
    model = task.build_model(args)
    loss = task.build_loss(args)
    trainer = Trainer(args, task, model, loss)
    trainer._total_train_steps = args.max_update
    task.load_dataset("train")
    ds = task.dataset("train")
    batches = [ds.collater([ds[k * 4 + i] for i in range(4)]) for k in range(3)]
    return trainer, model, batches


def test_unimol_plugin_trains_on_cpu():
    """Uni-Mol plug-in (pair-bias encoder, 3 heads, 5-term loss) through the public Trainer on CPU."""
    trainer, model, batches = _unimol_trainer()
    n_tok = batches[0]["net_input"]["src_tokens"]
    assert n_tok.shape[1] % 8 == 0
    before = [p.detach().clone() for p in model.parameters()]
    logs = []
    for i in range(4):
        out = trainer.train_step([batches[i % 3]])
        logs.append(float(out["loss"]))
    assert all(map(lambda v: v == v and abs(v) != float("inf"), logs))
    moved = sum(int(not torch.equal(a, p.detach())) for a, p in zip(before, model.parameters()))
    assert moved >= 0.9 * len(before), "almost every parameter (incl. the Gaussian basis) must receive gradient"
    assert trainer.get_num_updates() == 4
    # evaluation path: deterministic and finite
    model.eval()
    with torch.no_grad():
        a = model(**batches[0]["net_input"])
        b = model(**batches[0]["net_input"])
    for u, v in zip(a, b):
        if torch.is_tensor(u):
            assert torch.equal(u, v)


def _unimol_task(plugin):
    importlib.import_module(plugin)
    name = {"unimol": ("synthetic_unimol", "unimol", "unimol_base"),
            "unimol_portable": ("synthetic_unimol_portable", "unimol_portable", "unimol_portable_base")}[plugin]
    args = options.parse_args_and_arch(options.get_training_parser(), input_args=[
        "--task", name[0], "--loss", name[1], "--arch", name[2], "--encoder-layers", "2", "--encoder-embed-dim", "32",
        "--encoder-ffn-embed-dim", "64", "--encoder-attention-heads", "4", "--gaussian-kernels", "16",
        "--synthetic-num-samples", "16", "--synthetic-min-atoms", "6", "--synthetic-max-atoms", "14", "--seed", "7",
        "--dropout", "0.0", "--emb-dropout", "0.0", "--attention-dropout", "0.0", "--activation-dropout", "0.0",
        "--cpu", "--distributed-world-size", "1",
    ])
    task = tasks.setup_task(args)
    return task, task.build_model(args), task.build_loss(args)


def test_unimol_matches_the_portable_plugin():
    """``UniMolModel`` + ``UniMolLoss`` and the portable plug-in (``examples/unimol_portable``, the reference's
    formulation: ``-inf`` written into the padded key columns of the pair bias up front, no fused tail) have the same
    parameters, and with the same weights and batch the same five loss terms and gradients, up to fp32 rounding.  The
    GPU test of the model against float64 uses the plug-in as its reference."""
    torch.manual_seed(5)
    task, model, loss = _unimol_task("unimol")
    _, ref, ref_loss = _unimol_task("unimol_portable")
    with torch.no_grad():   # an atom representation longer than sqrt(E) + 1: the x-norm term and its gradient are not 0
        model.encoder.emb_layer_norm.weight.fill_(1.5)
    ref.load_state_dict(model.state_dict(), strict=True)
    task.load_dataset("train")
    ds = task.dataset("train")
    batch = ds.collater([ds[i] for i in range(4)])
    assert batch["net_input"]["src_tokens"].eq(task.dictionary.pad()).any(), "the batch must have padded atoms"
    model.train()
    ref.train()
    value, _, log = loss(model, batch)
    value.backward()
    ref_value, _, ref_log = ref_loss(ref, batch)
    ref_value.backward()
    for key in ("loss", "masked_token_loss", "masked_coord_loss", "masked_dist_loss", "x_norm_loss",
                "delta_pair_repr_norm_loss"):
        assert float(ref_log[key]) != 0, key
        assert abs(float(log[key]) - float(ref_log[key])) <= 1e-6 * abs(float(ref_log[key])), key
    ref_params = dict(ref.named_parameters())
    assert set(ref_params) == {n for n, _ in model.named_parameters()}
    for name, p in model.named_parameters():
        g, r = p.grad, ref_params[name].grad
        assert g is not None and r is not None, name
        assert (g - r).abs().max() <= 1e-5 * r.abs().max(), name


def test_nan_detector_names_the_first_bad_module(caplog):
    from unicore.nan_detector import NanDetector

    class Bad(torch.nn.Module):
        def forward(self, x):
            return x / (x - x)

    net = torch.nn.Sequential(torch.nn.Linear(4, 4), Bad(), torch.nn.Linear(4, 2))
    with caplog.at_level(logging.WARNING, logger="unicore.nan_detector"):
        with NanDetector(net) as det:
            net(torch.randn(3, 4)).sum().backward()
    text = caplog.text
    assert "detected in output of 1" in text and "forward" in text
    assert not det.fhooks and not det.bhooks  # hooks removed on exit


@pytest.mark.parametrize("fmt", ["json", "simple", "none", "tqdm"])
def test_progress_bars_emit_stats(fmt, caplog):
    from unicore.logging import progress_bar

    with caplog.at_level(logging.INFO):
        bar = progress_bar.progress_bar(list(range(6)), log_format=fmt, log_interval=2, epoch=3, prefix="train")
        seen = []
        for i, item in enumerate(bar):
            seen.append(item)
            bar.log({"loss": 1.0 / (i + 1), "ups": 2.5}, tag="train_inner", step=i)
        bar.print({"loss": 0.25}, tag="train", step=6)
    assert seen == list(range(6))
    if fmt == "json":
        rec = [r.getMessage() for r in caplog.records if r.getMessage().startswith("{")]
        assert rec and json.loads(rec[-1])["train_loss"] in ("0.25", 0.25)
    if fmt == "simple":
        assert any("loss" in r.getMessage() for r in caplog.records)


def test_trainer_recovers_from_oom_in_forward_backward():
    """Single process: an out-of-memory error inside fwd/bwd skips that step (gradients cleared, no update counted)
    and training continues; any other RuntimeError propagates (reference `trainer.py:630-645,959-965`)."""
    trainer, model, batches = _unimol_trainer()
    real = trainer.task.train_step
    calls = {"n": 0}

    def flaky(**kw):
        calls["n"] += 1
        if calls["n"] == 2:
            raise RuntimeError("CUDA out of memory. Tried to allocate 1.00 GiB")
        return real(**kw)

    trainer.task.train_step = flaky
    assert trainer.train_step([batches[0]]) is not None
    before = [p.detach().clone() for p in model.parameters()]
    assert trainer.train_step([batches[1]]) is None  # the OOM step
    assert trainer.get_num_updates() == 1
    assert all(torch.equal(a, p.detach()) for a, p in zip(before, model.parameters()))
    assert all(p.grad is None or not p.grad.abs().sum().item() for p in model.parameters())
    assert trainer.train_step([batches[2]]) is not None and trainer.get_num_updates() == 2

    def broken(**kw):
        raise RuntimeError("shape mismatch")

    trainer.task.train_step = broken
    with pytest.raises(RuntimeError, match="shape mismatch"):
        trainer.train_step([batches[0]])


def test_narrow_bias_gradient_fold_rule():
    """``ops.linear``'s rule for folding rows of a narrow gradient before the column-sum kernel."""
    import torch

    from unicore_b200.ops.fused_ops import _narrow_fold

    def fold(rows, cols, dtype=torch.float16):
        return _narrow_fold(torch.zeros(rows, cols, dtype=dtype))

    assert fold(65536, 64) == 16          # 64 x 16 = 1024 columns
    assert fold(12288, 128) == 8
    assert fold(4096 * 3, 8) == 128       # capped by 1024 / cols
    assert fold(4098, 64) == 2            # rows only divisible by 2
    assert fold(65536, 256) == 1          # wide enough as it is
    assert fold(1000, 64) == 1            # too few rows to matter
    assert fold(65536, 60) == 1           # not a multiple of 8 columns
    assert fold(65536, 64, torch.float32) == 1


def test_embedding_and_vocab_projection_fall_back_on_cpu():
    """Without the native extension in play both ops are the plain PyTorch formulations (same values and gradients)."""
    import torch
    import torch.nn.functional as F

    from unicore import ops

    torch.manual_seed(3)
    w = torch.randn(50, 16, requires_grad=True)
    tok = torch.randint(0, 50, (4, 7))
    y = ops.embedding(tok, w, 1)
    assert torch.equal(y, F.embedding(tok, w, 1))
    y.sum().backward()
    g = w.grad.clone()
    w.grad = None
    F.embedding(tok, w, 1).sum().backward()
    assert torch.equal(g, w.grad)
    x = torch.randn(5, 16)
    assert torch.allclose(ops.vocab_projection(x, w, None), F.linear(x, w))
