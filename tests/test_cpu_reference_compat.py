"""Compatibility proofs against the reference implementation (SURVEY.md section 7.1-4): checkpoints travel in both
directions, and a plug-in written against the public API trains to the same losses.  What the unmodified reference
computed for these runs is stored in ``tests/golden/reference_records.json``, and the checkpoint it wrote in
``tests/golden/checkpoint_interop_reference.pt``; both implementations build their initial weights from the same seed,
which the recorded checksum of those weights pins down."""
import hashlib
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PY = sys.executable
with open(os.path.join(ROOT, "tests", "golden", "reference_records.json")) as _f:
    GOLDEN = json.load(_f)


def init_sha256(path):
    import torch

    sd = torch.load(path, map_location="cpu")
    h = hashlib.sha256()
    for k in sorted(sd):
        h.update(k.encode())
        h.update(sd[k].detach().contiguous().numpy().tobytes())
    return h.hexdigest()


def _interop(impl, init, *extra):
    tool = os.path.join(ROOT, "tools", "checkpoint_interop.py")
    out = subprocess.run([PY, tool, "--impl", impl, "--init", init] + list(extra), env=dict(os.environ, OMP_NUM_THREADS="1"),
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-3000:]
    return json.loads([l for l in out.stdout.splitlines() if l.startswith("{")][-1])


def test_checkpoints_travel_between_the_reference_and_this_framework(tmp_path):
    """bf16 + weight decay (two flat optimizer groups) + clipping + EMA on the CPU, in both directions (flat layout,
    reference ``unicore/optim/fp16_optimizer.py:54-121``; schema ``unicore/trainer.py:224-284``):
    * this framework loads the checkpoint the reference wrote (``tests/golden/checkpoint_interop_reference.pt``) and
      continues with the reference's own next losses, learning rate and EMA;
    * this framework trains 3 updates from the same initial weights and saves: the file has the reference's schema, the
      losses are the reference's, and the reference continued from exactly this file to the recorded losses and EMA,
      which loading it here reproduces."""
    gold = GOLDEN["checkpoint_interop"]
    ref, ref_loads_ref, ref_loads_ours = gold["reference"], gold["reference_loads_reference"], gold["reference_loads_ours"]
    width = ["--embed-dim", str(gold["embed_dim"])]
    init = str(tmp_path / "init.pt")

    # reference -> this framework
    ref_ck = os.path.join(ROOT, "tests", "golden", "checkpoint_interop_reference.pt")
    got = _interop("ours", init, "--load", ref_ck, "--more", "2", *width)
    assert init_sha256(init) == gold["init_sha256"]
    assert got["loaded_updates"] == ref_loads_ref["loaded_updates"] == 3
    assert got["loaded_epoch"] == ref_loads_ref["loaded_epoch"] == 1
    assert got["lr_after_load"] == pytest.approx(ref_loads_ref["lr_after_load"], rel=1e-9)
    assert got["losses_after"] == pytest.approx(ref_loads_ref["losses_after"], abs=3e-3)
    assert got["ema_checksum"] == pytest.approx(ref_loads_ref["ema_checksum"], rel=1e-5)

    # this framework -> reference
    ours = _interop("ours", init, "--steps", "3", "--save", str(tmp_path / "ours.pt"), "--more", "2", *width)
    assert ours["saved_keys"] == ref["saved_keys"] and ours["saved_opt_state_numel"] == ref["saved_opt_state_numel"]
    assert ours["losses_before"] == pytest.approx(ref["losses_before"], abs=2e-3)
    assert ours["losses_after"] == pytest.approx(ref["losses_after"], abs=3e-3)
    assert ours["losses_after"] == pytest.approx(ref_loads_ours["losses_after"], abs=3e-3)
    assert ours["ema_checksum"] == pytest.approx(ref_loads_ours["ema_checksum"], rel=1e-5)
    got = _interop("ours", init, "--load", str(tmp_path / "ours.pt"), "--more", "2", *width)
    assert got["loaded_updates"] == ref_loads_ours["loaded_updates"] == 3
    assert got["loaded_epoch"] == ref_loads_ours["loaded_epoch"] == 1
    assert got["lr_after_load"] == pytest.approx(ref_loads_ours["lr_after_load"], rel=1e-9)
    assert got["losses_after"] == pytest.approx(ref_loads_ours["losses_after"], abs=3e-3)
    assert got["ema_checksum"] == pytest.approx(ref_loads_ours["ema_checksum"], rel=1e-5)


def test_portable_unimol_plugin_gives_the_same_losses_under_both_frameworks(tmp_path):
    """``examples/unimol_portable`` only uses the public Uni-Core API: the identical plug-in code trains under this
    framework, from the reference's initial weights, to the losses it reached under the reference (BASELINE.md B6)."""
    gold = GOLDEN["unimol_portable"]
    tool = os.path.join(ROOT, "tools", "unimol_portable_check.py")
    init = str(tmp_path / "u.pt")
    out = subprocess.run([PY, tool, "--impl", "ours", "--init", init, "--steps", "3"], env=dict(os.environ, OMP_NUM_THREADS="1"),
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert out.returncode == 0, out.stdout[-3000:]
    ours = json.loads([l for l in out.stdout.splitlines() if l.startswith("{")][-1])["losses"]
    assert init_sha256(init) == gold["init_sha256"]
    assert len(ours) == 3 and ours[-1] < ours[0]
    assert ours == pytest.approx(gold["losses"], abs=2e-3)
