"""Deterministic mode: under ``torch.use_deterministic_algorithms`` the native backward kernels reduce in a fixed order.

Checked, each with the switch on only around the kernel calls (warn-only, which the kernels honour too):
- fused attention backward: repeated calls are bitwise equal; dK, dV and dBias are bitwise those of the default mode
  and dQ agrees with it up to the order of its fp32 sum; the gradients of one batch slice are bitwise those of a call
  on that slice alone (an entirely different schedule); no wait for a turn timed out;
- embedding gradient: bitwise equal to a float32 host loop over the rows in ascending order;
- Gaussian basis gradient and the gen-1 norm backward: repeated calls are bitwise equal; the norm backward's outputs
  are bitwise those of the default mode;
- end to end, in fresh interpreters: two ``unicore-train --deterministic`` BERT runs log the same losses and write
  bitwise identical checkpoints, and two Uni-Mol forward + backward passes leave bitwise identical gradients.
"""
import contextlib
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from test_gpu_attention_dropout_stream import _assert_within

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DTYPES = [torch.float16, torch.bfloat16]
DT_IDS = ["fp16", "bf16"]
UNIT = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
P_DROP = 0.1


@contextlib.contextmanager
def deterministic():
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def _nat():
    from unicore import ops

    assert ops.USE_NATIVE, "native kernels must be active on the GPU box"
    return ops.native()


# ---- 1. fused attention backward -----------------------------------------------------------------------------------
# ragged against the 64-row tiles; Lq > Lk; Lq < Lk; B = 2 everywhere so that a batch slice has another schedule
SHAPES = {"ragged": (2, 3, 200, 200), "lq_gt_lk": (2, 2, 136, 72), "lq_lt_lk": (2, 2, 72, 200)}
# shared bias / per-batch bias (padding, dropout), causal, logits mode with dz, packed q/k/v gradients
MODES = ["shared", "batch", "causal", "logits", "packed"]
CASES = [(s, m) for s in SHAPES for m in MODES if m != "packed" or SHAPES[s][2] == SHAPES[s][3]]


def _attention_case(shape, D, dtype, mode):
    B, H, Lq, Lk = shape
    nat = _nat()
    g = torch.Generator(device="cuda").manual_seed(D + 7 * Lq + Lk)
    scale = 1.0 / math.sqrt(D)
    if mode == "packed":
        qkv = (torch.randn(B, Lq, 3, H, D, device="cuda", generator=g) * 0.6).to(dtype)
        q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    else:
        q = (torch.randn(B, Lq, H, D, device="cuda", generator=g) * 0.6).to(dtype)
        k = (torch.randn(B, Lk, H, D, device="cuda", generator=g) * 0.6).to(dtype)
        v = torch.randn(B, Lk, H, D, device="cuda", generator=g).to(dtype)
    per_batch = mode in ("batch", "logits")
    bias = torch.randn(B if per_batch else 1, H, Lq, Lk, device="cuda", generator=g).to(dtype)
    kpm = torch.zeros(B, Lk, dtype=torch.bool, device="cuda")
    kpm[0, Lk - Lk // 4:] = True
    kpm[-1, 8:16] = True
    causal = mode == "causal"
    dz = None
    if mode == "logits":
        out, lse, bits, z = nat.fmha_fwd_logits(q, k, v, bias, kpm, P_DROP, scale)
        dz = (torch.randn(z.shape, device="cuda", generator=g) * 0.1).to(dtype)
    else:
        out, lse, bits = nat.fmha_fwd(q, k, v, bias, kpm, P_DROP, scale, causal=causal)
    dout = torch.randn(B, Lq, H, D, device="cuda", generator=g).to(dtype)

    def bwd(b=None):
        s = slice(None) if b is None else slice(b, b + 1)
        return nat.fmha_bwd(dout[s], q[s], k[s], v[s], out[s], lse[s], bias[s] if per_batch else bias, kpm[s], P_DROP,
                            scale, bits[s], True, mode == "packed", dlogits=None if dz is None else dz[s], causal=causal)

    ref = bwd()
    nat.fmha_det_timeouts()
    with deterministic():
        det = [bwd() for _ in range(3)]
        slices = [bwd(b) for b in range(B)]
    assert nat.fmha_det_timeouts() == 0
    # (a) repeated calls are bitwise equal
    for other in det[1:]:
        for a, c in zip(det[0], other):
            assert torch.equal(a, c)
    dq, dk, dv, db = det[0]
    # (b) only the order of the dQ sum changed
    assert torch.equal(dk, ref[1]) and torch.equal(dv, ref[2]) and torch.equal(db, ref[3])
    r = ref[0].double()
    _assert_within(dq, r, 2 * UNIT[dtype] * r.abs() + 2.0 ** -18 * r.abs().max(), "dQ")
    # (c) the sum of a batch slice does not depend on what else is in the grid
    for b, (sq, sk, sv, sdb) in enumerate(slices):
        assert torch.equal(sq, dq[b:b + 1]) and torch.equal(sk, dk[b:b + 1]) and torch.equal(sv, dv[b:b + 1])
        if per_batch:
            assert torch.equal(sdb, db[b:b + 1])


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("D", [8, 64, 96, 128])
@pytest.mark.parametrize("shape,mode", CASES)
def test_attention_backward_is_deterministic(shape, mode, D, dtype):
    _attention_case(SHAPES[shape], D, dtype, mode)


@pytest.mark.parametrize("mode", ["shared", "causal"])
@pytest.mark.parametrize("D", [64, 128])
def test_attention_backward_is_deterministic_across_waves(D, mode):
    """4 x 12 x 16 key-tile CTAs: more than one wave, so CTAs wait on CTAs of earlier waves."""
    _attention_case((4, 12, 1024, 1024), D, torch.float16, mode)


# ---- 2. embedding gradient -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("accumulate", [False, True], ids=["write", "accumulate"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_embedding_gradient_matches_a_host_loop(dtype, accumulate):
    nat = _nat()
    V, R, C, pad = 37, 65536, 768, 1
    g = torch.Generator(device="cuda").manual_seed(11)
    # heavy repetition, the padding index, and ids outside [0, V)
    tok = torch.randint(-2, V + 3, (R,), device="cuda", generator=g)
    tok[: R // 4] = 5
    tok = tok[torch.randperm(R, device="cuda", generator=g)]
    dy = torch.randn(R, C, device="cuda", generator=g).to(dtype)
    base = torch.randn(V, C, device="cuda", generator=g).to(dtype) if accumulate else torch.zeros(V, C, device="cuda",
                                                                                                      dtype=dtype)
    scratch = torch.zeros(V, C, device="cuda")
    touched = torch.zeros(V, dtype=torch.uint8, device="cuda")
    outs = []
    with deterministic():
        for _ in range(3):
            grad = base.clone()
            nat.embedding_bwd(dy, tok, pad, scratch, touched, grad, accumulate)
            outs.append(grad)
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])

    tok_h, dy_h = tok.cpu().numpy(), dy.float().cpu().numpy()
    want = base.float().cpu().numpy().copy()
    for row in range(V):
        if row == pad:
            continue
        rows = dy_h[tok_h == row]            # ascending original order
        if len(rows) == 0:
            continue
        acc = np.add.accumulate(np.concatenate([np.zeros((1, C), np.float32), rows]), axis=0, dtype=np.float32)[-1]
        want[row] = acc + want[row] if accumulate else acc
    assert torch.equal(outs[0].cpu(), torch.from_numpy(want).to(dtype))


# ---- 3. Gaussian basis gradient ------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_gaussian_basis_gradient_is_deterministic(dtype):
    nat = _nat()
    B, L, K, E = 32, 128, 128, 900
    g = torch.Generator(device="cuda").manual_seed(3)
    dist = (torch.rand(B, L, L, device="cuda", generator=g) * 6).to(dtype)
    edge = torch.randint(0, E, (B, L, L), device="cuda", generator=g)
    mul_w = (1 + 0.2 * torch.randn(E, 1, device="cuda", generator=g)).to(dtype)
    bias_w = (0.2 * torch.randn(E, 1, device="cuda", generator=g)).to(dtype)
    means = (torch.rand(1, K, device="cuda", generator=g) * 3).to(dtype)
    stds = (torch.rand(1, K, device="cuda", generator=g) * 3 + 0.5).to(dtype)
    dy = torch.randn(B, L, L, K, device="cuda", generator=g).to(dtype)
    with deterministic():
        runs = [nat.gbf_bwd(dy, dist, edge, mul_w, bias_w, means, stds) for _ in range(3)]
    for other in runs[1:]:
        for a, c in zip(runs[0], other):
            assert torch.equal(a, c)
    ref_in = [t.detach().double().requires_grad_(True) for t in (mul_w, bias_w, means, stds)]
    t = (ref_in[0].view(-1)[edge] * dist.double() + ref_in[1].view(-1)[edge]).unsqueeze(-1)
    std = ref_in[3].view(-1).abs() + 1e-5
    yr = torch.exp(-0.5 * ((t - ref_in[2].view(-1)) / std) ** 2) / ((2 * 3.14159) ** 0.5 * std)
    yr.backward(dy.double())
    for got, ref in zip(runs[0], ref_in):
        scale = max(1.0, ref.grad.abs().max().item())
        assert (got.double() - ref.grad.view(-1)).abs().max().item() < 3e-2 * scale


# ---- 4. norm backward, gen 1 (rows too wide for v2) ----------------------------------------------------------------
@pytest.mark.parametrize("rms", [False, True], ids=["layer_norm", "rms_norm"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_gen1_norm_backward_is_deterministic(dtype, rms):
    nat = _nat()
    rows, cols = 4096, 5120
    assert nat.norm_plan(rows, cols, dtype, "bwd")["gen"] == 1
    g = torch.Generator(device="cuda").manual_seed(5)
    x = (torch.randn(rows, cols, device="cuda", generator=g) * 2 + 0.5).to(dtype)
    w = (torch.randn(cols, device="cuda", generator=g) * 0.5 + 1).to(dtype)
    b = torch.randn(cols, device="cuda", generator=g).to(dtype)
    dy = torch.randn(rows, cols, device="cuda", generator=g).to(dtype)
    if rms:
        _, rstd = nat.rmsnorm_fwd(x, w, 1e-5)
        ref = nat.rmsnorm_bwd(dy, x, rstd, w)
        with deterministic():
            runs = [nat.rmsnorm_bwd(dy, x, rstd, w) for _ in range(3)]
    else:
        _, mean, rstd = nat.layernorm_fwd(x, w, b, 1e-5)
        ref = nat.layernorm_bwd(dy, x, mean, rstd, w)
        with deterministic():
            runs = [nat.layernorm_bwd(dy, x, mean, rstd, w) for _ in range(3)]
    for other in runs[1:]:
        for a, c in zip(runs[0], other):
            assert torch.equal(a, c)
    for a, r in zip(runs[0], ref):   # the row groups add in turn in both modes
        assert torch.equal(a, r)


# ---- 5. end to end -------------------------------------------------------------------------------------------------
def _env():
    return dict(os.environ, PYTHONPATH=ROOT, CUBLAS_WORKSPACE_CONFIG=":4096:8")


def _train_bert(save):
    cmd = [sys.executable, os.path.join(ROOT, "unicore_cli", "train.py"), "--user-dir", os.path.join(ROOT, "examples", "bert"),
           "--task", "synthetic_mlm", "--loss", "masked_lm", "--arch", "bert_base", "--encoder-layers", "2",
           "--encoder-embed-dim", "256", "--encoder-ffn-embed-dim", "512", "--encoder-attention-heads", "4",
           "--synthetic-vocab-size", "1024", "--synthetic-seq-len", "256", "--synthetic-num-samples", "128",
           "--max-seq-len", "256", "--optimizer", "adam", "--lr", "1e-4", "--lr-scheduler", "polynomial_decay",
           "--total-num-update", "100", "--max-update", "8", "--batch-size", "8", "--fp16", "--clip-norm", "1.0",
           "--distributed-world-size", "1", "--num-workers", "0", "--disable-validation", "--log-format", "simple",
           "--log-interval", "1", "--save-dir", save, "--tmp-save-dir", save, "--no-epoch-checkpoints",
           "--deterministic", "--seed", "5"]
    out = subprocess.run(cmd, env=_env(), cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
    losses = [ln.split("loss=")[1].split(",")[0] for ln in out.stdout.splitlines() if "train_inner" in ln and "loss=" in ln]
    assert len(losses) == 8, out.stdout[-3000:]
    return losses, torch.load(os.path.join(save, "checkpoint_last.pt"), map_location="cpu", weights_only=False)


def _assert_same_tree(a, b, path="ck"):
    if isinstance(a, torch.Tensor):
        assert isinstance(b, torch.Tensor) and a.dtype == b.dtype and torch.equal(a, b), path
    elif isinstance(a, dict):
        assert set(a) == set(b), path
        for key in a:
            _assert_same_tree(a[key], b[key], "{}.{}".format(path, key))
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), path
        for i, (x, y) in enumerate(zip(a, b)):
            _assert_same_tree(x, y, "{}[{}]".format(path, i))


def test_bert_training_runs_are_bitwise_identical(tmp_path):
    la, ca = _train_bert(str(tmp_path / "a"))
    lb, cb = _train_bert(str(tmp_path / "b"))
    assert la == lb
    _assert_same_tree(ca["model"], cb["model"], "model")
    _assert_same_tree(ca["last_optimizer_state"], cb["last_optimizer_state"], "optimizer")


UNIMOL_SCRIPT = r"""
import importlib, sys
import torch
from unicore import options, tasks, utils
sys.path.insert(0, sys.argv[2])
importlib.import_module("unimol")
utils.set_deterministic(True)
parser = options.get_training_parser()
args = options.parse_args_and_arch(parser, input_args=[
    "--task", "synthetic_unimol", "--loss", "unimol", "--arch", "unimol_base", "--encoder-layers", "2",
    "--encoder-embed-dim", "64", "--encoder-ffn-embed-dim", "128", "--encoder-attention-heads", "8",
    "--synthetic-num-samples", "16", "--synthetic-min-atoms", "20", "--synthetic-max-atoms", "60",
    "--optimizer", "adam", "--lr", "1e-3", "--batch-size", "8", "--seed", "7", "--fp16",
    "--distributed-world-size", "1", "--log-format", "none"])
torch.manual_seed(7)
task = tasks.setup_task(args)
model = task.build_model(args).cuda().half()
loss = task.build_loss(args)
task.load_dataset("train")
ds = task.dataset("train")
sample = utils.move_to_cuda(ds.collater([ds[i] for i in range(8)]))
model.train()
torch.manual_seed(11)
value, _, _ = loss(model, sample)
value.float().backward()
torch.save({n: p.grad for n, p in model.named_parameters() if p.grad is not None}, sys.argv[1])
"""


def test_unimol_gradients_are_bitwise_identical(tmp_path):
    grads = []
    for name in ("a.pt", "b.pt"):
        path = str(tmp_path / name)
        out = subprocess.run([sys.executable, "-c", UNIMOL_SCRIPT, path, os.path.join(ROOT, "examples")], env=_env(),
                             cwd=ROOT, capture_output=True, text=True, timeout=900)
        assert out.returncode == 0, out.stdout[-3000:] + out.stderr[-3000:]
        grads.append(torch.load(path))
    assert len(grads[0]) > 10 and set(grads[0]) == set(grads[1])
    for n in grads[0]:
        assert torch.equal(grads[0][n], grads[1][n]), n
