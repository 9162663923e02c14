"""``--deterministic``: the flag parses (default off), the function the CLI applies it with turns on PyTorch's
deterministic algorithms and the cuBLAS workspace setting, and a CPU run with the flag still trains."""
import os

import torch

from unicore import options, utils
from test_cpu_training import losses_of, run_cli


def _parse(extra):
    parser = options.get_training_parser()
    return options.parse_args_and_arch(parser, input_args=[
        "--task", "synthetic_mlm", "--loss", "masked_lm", "--arch", "bert_base", "--user-dir",
        os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "examples", "bert"),
        "--optimizer", "adam", "--lr", "1e-3", "--batch-size", "2", "--cpu"] + extra)


def test_flag_parses_and_defaults_off():
    assert _parse([]).deterministic is False
    assert _parse(["--deterministic"]).deterministic is True


def test_set_deterministic_sets_the_switch_and_cublas_config(monkeypatch):
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    monkeypatch.delenv("CUBLAS_WORKSPACE_CONFIG", raising=False)
    try:
        utils.set_deterministic(False)
        assert "CUBLAS_WORKSPACE_CONFIG" not in os.environ
        assert torch.are_deterministic_algorithms_enabled() == prev
        utils.set_deterministic(True)
        assert torch.are_deterministic_algorithms_enabled()
        assert not torch.is_deterministic_algorithms_warn_only_enabled()
        assert os.environ["CUBLAS_WORKSPACE_CONFIG"] == ":4096:8"
        monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":16:8")   # a setting the user made is kept
        utils.set_deterministic(True)
        assert os.environ["CUBLAS_WORKSPACE_CONFIG"] == ":16:8"
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def test_cli_trains_with_the_flag():
    log = run_cli(["--deterministic", "--max-update", "2", "--no-save", "--disable-validation"])
    losses = losses_of(log)
    assert len(losses) == 2 and all(v == v for v in losses), losses
