"""Operand validation of every tensor-taking binding in ``unicore_b200._C``.

Each binding has one valid argument builder.  Each tensor operand in turn is then replaced by a CPU tensor, a tensor
of a dtype no kernel takes, a too-small tensor and, where the kernel needs it, a non-contiguous or an off-16-byte view;
the call must raise a RuntimeError that names the operand.  All of these are refused before the binding takes its
device guard, allocates or launches anything.
"""
import importlib
import re

import pytest
import torch

pytestmark = pytest.mark.gpu

F16, F32 = torch.float16, torch.float32
ALL, CONTIG, VEC = ("cpu", "dtype", "small"), ("cpu", "dtype", "small", "nc"), ("cpu", "dtype", "small", "nc", "mis")
NO_SMALL_C, NO_SMALL_V = ("cpu", "dtype", "nc"), ("cpu", "dtype", "nc", "mis")
# builds that raise this after every operand check passed (the comm entry points get no peer addresses here)
NO_PEERS = "bad rank / world size"


def _nat():
    from unicore import ops

    assert ops.USE_NATIVE, "native kernels must be active on the GPU box"
    return ops.native()


def _r(*shape, dtype=F16):
    return torch.randn(*shape, device="cuda").to(dtype)


def _nc(t):
    s = torch.empty(*t.shape, 2, dtype=t.dtype, device=t.device)[..., 0]
    s.copy_(t)
    return s


def _mis(t):
    buf = torch.empty(t.numel() + 16, dtype=t.dtype, device=t.device)
    v = buf[1:1 + t.numel()].view(t.shape)
    v.copy_(t)
    return v


MUTATE = {
    "cpu": lambda t: t.cpu(),
    "dtype": lambda t: t.to(torch.int16),  # no kernel takes int16
    "small": lambda t: t.reshape(-1)[:-1].clone(),
    "nc": _nc,
    "mis": _mis,
    "dev": lambda t: t.to("cuda:1"),
}


# ---- valid argument builders ---------------------------------------------------------------------------------------
def _adam():
    n = 24
    return [[_r(n, dtype=F32)], [_r(n)], [_r(n, dtype=F32)], [_r(n, dtype=F32).abs()], [_r(n)], [1e-3], [0.9], [0.999],
            [1e-8], [1], [True], [0.01], 1.0, torch.ones(1, device="cuda"), False, False, [_r(n, dtype=F32)], 0.99]


def _norm_bwd():
    x = _r(4, 64)
    return [_r(4, 64), x, x.float().mean(1), torch.ones(4, device="cuda"), _r(64), _r(64), _r(64)]


def _embedding():
    V = 10
    return [_r(6, 64), torch.randint(0, V, (6,), device="cuda"), 0, torch.zeros(V * 64, device="cuda"),
            torch.zeros(V, dtype=torch.uint8, device="cuda"), torch.zeros(V, 64, dtype=F16, device="cuda"), False]


def _bdaln_bwd():
    return [_r(4, 64), _r(4, 64), _r(4, dtype=F32), torch.ones(4, device="cuda"), _r(64), 0.1, 1, 0, True, _r(64),
            _r(64), _r(64)]


def _gbf(dy=False):
    d, E, K = _r(2, 8), 4, 16
    args = [d, torch.randint(0, E, (2, 8), device="cuda"), _r(E, 1), _r(E, 1), _r(1, K), _r(1, K).abs() + 1]
    return ([_r(2, 8, K)] + args) if dy else args


def _qkv(L=64):
    return [_r(1, L, 2, 64) for _ in range(3)] + [_r(1, 2, L, L), torch.zeros(1, L, dtype=torch.bool, device="cuda")]


def _fmha_bwd():
    q, k, v, bias, kpm = _qkv()
    out, lse, bits = _nat().fmha_fwd(q, k, v, bias, kpm, 0.1, 0.125)
    return [torch.randn_like(out), q, k, v, out, lse, bias, kpm, 0.1, 0.125, bits, True, False, _r(1, 2, 64, 64)]


def _decode():
    B, C, H, D = 2, 16, 2, 64
    return [_r(B, 1, H, D), _r(B, C, H, D), _r(B, C, H, D), torch.tensor([3, 4], dtype=torch.int32, device="cuda"), 8,
            _r(B, 1, H, D), _r(B, 1, H, D), _r(1, H, 1, C), torch.zeros(B, C, dtype=torch.bool, device="cuda"), 0.125, 0]


def _fused_tail():
    n = 64
    return [[], [], 0, 0, 0, [[0]], [0], [[0]], [0], [_r(n, dtype=F32)], [_r(n, dtype=F32)], [_r(n, dtype=F32)],
            [_r(n, dtype=F32)], [n], [1], [[0.9, 0.999, 1e-8, 1e-3, 1.0]],
            torch.tensor([[0, n, 0, n, 0, 0]], device="cuda"), 0, torch.zeros(_nat().SYMM_MAX_BLOCKS, device="cuda"),
            torch.zeros(_nat().symm_tail_max_blocks(), device="cuda"), torch.zeros(4, dtype=torch.int32, device="cuda"),
            torch.zeros(2, dtype=torch.float64, device="cuda"), torch.zeros(2, dtype=torch.float64, device="cuda"),
            0, 0, 1.0, 0.0, 1e-6, 1.0, 0.99, False, 0, 0, torch.zeros(4, device="cuda"), 0]


# binding -> (valid argument builder, {operand: (name in the messages, mutations)}).  An operand is an argument index,
# or (argument index, list index).  The first operand listed is the one whose device the call runs on.
CASES = {
    "multi_tensor_l2norm": (lambda: [[_r(24), _r(40, dtype=F32)]],
                            {(0, 0): ("l2norm input", NO_SMALL_C), (0, 1): ("l2norm input", NO_SMALL_C)}),
    "multi_tensor_scale": (lambda: [[_r(24), _r(40, dtype=F32)], 0.5, torch.ones(1, device="cuda")],
                           {(0, 0): ("scale input", NO_SMALL_C), (0, 1): ("scale input", NO_SMALL_C),
                            2: ("scale_dev", ALL)}),
    "multi_tensor_adam": (_adam, {(0, 0): ("p", NO_SMALL_C), (1, 0): ("g", CONTIG), (2, 0): ("m", CONTIG),
                                  (3, 0): ("v", CONTIG), (4, 0): ("p_half", CONTIG), 13: ("scale_dev", ALL),
                                  (16, 0): ("ema", CONTIG)}),
    "fp32_to_bf16_sr": (lambda: [_r(24, dtype=F32), torch.empty(24, dtype=torch.bfloat16, device="cuda")],
                        {0: ("in", NO_SMALL_C), 1: ("out", CONTIG)}),
    "ema_update": (lambda: [_r(24, dtype=F32), _r(24, dtype=F32), 0.9], {0: ("ema", NO_SMALL_C), 1: ("p", CONTIG)}),
    "layernorm_fwd": (lambda: [_r(4, 64), _r(64), _r(64), 1e-5], {0: ("x", VEC), 1: ("gamma", VEC), 2: ("beta", VEC)}),
    "layernorm_bwd": (_norm_bwd, {1: ("x", VEC), 0: ("dy", VEC), 2: ("mean", CONTIG), 3: ("rstd", CONTIG),
                                  4: ("gamma", VEC), 5: ("dgamma_sink", CONTIG), 6: ("dbeta_sink", CONTIG)}),
    "rmsnorm_fwd": (lambda: [_r(4, 64), _r(64), 1e-5], {0: ("x", VEC), 1: ("gamma", VEC)}),
    "rmsnorm_bwd": (lambda: [_r(4, 64), _r(4, 64), torch.ones(4, device="cuda"), _r(64), _r(64)],
                    {1: ("x", VEC), 0: ("dy", VEC), 2: ("rstd", CONTIG), 3: ("gamma", VEC), 4: ("dgamma_sink", CONTIG)}),
    "softmax_dropout_fwd": (lambda: [_r(2, 4, 64), _r(1, 4, 64), _r(1, 4, 64), 0.1, True, False],
                            {0: ("input", CONTIG), 1: ("mask", CONTIG), 2: ("bias", CONTIG)}),
    "softmax_dropout_bwd": (lambda: [_r(2, 4, 64), _r(2, 4, 64), 0.1, 1, 0],
                            {0: ("grad_output", CONTIG), 1: ("softmax_results", CONTIG)}),
    "softmax_dropout_logits_fwd": (lambda: [_r(2, 4, 64), _r(1, 4, 64), _r(1, 4, 64), 0.1, True],
                                   {0: ("input", CONTIG), 1: ("mask", CONTIG), 2: ("bias", CONTIG)}),
    "softmax_dropout_logits_bwd": (lambda: [_r(2, 4, 64), _r(2, 4, 64), _r(2, 4, dtype=F32), _r(2, 4, 64), 0.1, 1, 0],
                                   {0: ("grad_output", CONTIG), 1: ("logits", CONTIG), 2: ("lse", CONTIG),
                                    3: ("grad_logits", CONTIG)}),
    "bias_gelu_fwd": (lambda: [_r(4, 64), _r(64)], {0: ("x", NO_SMALL_V), 1: ("bias", VEC)}),
    "bias_gelu_bwd": (lambda: [_r(4, 64), _r(4, 64), _r(64), _r(64)],
                      {1: ("x", NO_SMALL_V), 0: ("dy", VEC), 2: ("bias", VEC), 3: ("dbias_sink", CONTIG)}),
    "embedding_bwd": (_embedding, {0: ("dy", NO_SMALL_V), 5: ("grad", VEC), 1: ("tokens", CONTIG),
                                   3: ("scratch", VEC), 4: ("touched", CONTIG)}),
    "column_sum": (lambda: [_r(4, 64), _r(64)], {0: ("x", NO_SMALL_V), 1: ("sink", CONTIG)}),
    "bias_dropout_add_ln_fwd": (lambda: [_r(4, 64), _r(64), _r(4, 64), _r(64), _r(64), 0.1, 1e-5],
                                {0: ("x", VEC), 1: ("bias", VEC), 2: ("residual", VEC), 3: ("gamma", VEC),
                                 4: ("beta", VEC)}),
    "bias_dropout_add_ln_bwd": (_bdaln_bwd, {1: ("summed", VEC), 0: ("dy", VEC), 2: ("mean", CONTIG),
                                             3: ("rstd", CONTIG), 4: ("gamma", VEC), 9: ("dgamma_sink", CONTIG),
                                             10: ("dbeta_sink", CONTIG), 11: ("dbias_sink", CONTIG)}),
    "softmax_xent_fwd": (lambda: [_r(4, 64), torch.randint(0, 60, (4,), device="cuda"), -100, 60],
                         {0: ("logits", CONTIG), 1: ("target", CONTIG)}),
    "softmax_xent_bwd": (lambda: [_r(4, 64), torch.randint(0, 60, (4,), device="cuda"), _r(4, dtype=F32),
                                  torch.ones(1, device="cuda"), -100, 60],
                         {0: ("logits", CONTIG), 1: ("target", CONTIG), 2: ("lse", CONTIG), 3: ("dloss", ALL)}),
    "split_heads": (lambda: [_r(2, 8, 96), 3, 2, 0.5], {0: ("input", VEC)}),
    "merge_heads": (lambda: [[_r(2, 2, 8, 16), None, _r(2, 2, 8, 16)], 0.5], {(0, 2): ("heads", VEC),
                                                                              (0, 0): ("heads", VEC)}),
    "pair_transpose": (lambda: [_r(1, 8, 8, 8), True], {0: ("input", VEC)}),
    "pair_tail_fwd": (lambda: [_r(1, 8, 8, 8), _r(1, 8, 8, 8), torch.zeros(1, 8, dtype=torch.bool, device="cuda")],
                      {0: ("logits", VEC), 1: ("input bias", VEC), 2: ("key_padding_mask", VEC)}),
    "pair_tail_bwd": (lambda: [_r(1, 8, 8, 8), _r(1, 8, 8, 8), _r(1, 8, 8, 8),
                               torch.zeros(1, 8, dtype=torch.bool, device="cuda")],
                      {2: ("logits", VEC), 0: ("d_pair", VEC), 1: ("d_delta", VEC), 3: ("key_padding_mask", VEC)}),
    "gbf_fwd": (_gbf, {0: ("d", NO_SMALL_C), 1: ("edge", CONTIG), 2: ("mul_w", NO_SMALL_C), 3: ("bias_w", CONTIG),
                       4: ("means", NO_SMALL_C), 5: ("stds", CONTIG)}),
    "gbf_bwd": (lambda: _gbf(dy=True), {1: ("d", NO_SMALL_C), 0: ("dy", CONTIG), 2: ("edge", CONTIG),
                                        3: ("mul_w", NO_SMALL_C), 4: ("bias_w", CONTIG), 5: ("means", NO_SMALL_C),
                                        6: ("stds", CONTIG)}),
    "fmha_fwd": (lambda: _qkv() + [0.1, 0.125], {0: ("q", ("cpu", "dtype", "small", "mis")),
                                               1: ("k", ("cpu", "dtype", "small", "mis")),
                                               2: ("v", ("cpu", "dtype", "small", "mis")), 3: ("bias", VEC),
                                               4: ("key_padding_mask", CONTIG)}),
    "fmha_fwd_logits": (lambda: _qkv() + [0.1, 0.125], {0: ("q", ("cpu", "dtype", "small", "mis")),
                                                      1: ("k", ("cpu", "dtype", "small", "mis")),
                                                      2: ("v", ("cpu", "dtype", "small", "mis")), 3: ("bias", VEC),
                                                      4: ("key_padding_mask", CONTIG)}),
    "fmha_bwd": (_fmha_bwd, {1: ("q", ("cpu", "dtype", "small", "mis")), 2: ("k", ("cpu", "dtype", "small", "mis")),
                             3: ("v", ("cpu", "dtype", "small", "mis")), 0: ("dout", VEC), 4: ("out", CONTIG),
                             5: ("lse", CONTIG), 6: ("bias", VEC), 7: ("key_padding_mask", CONTIG),
                             10: ("drop_bits", CONTIG), 13: ("dlogits", VEC)}),
    "fmha_decode": (_decode, {0: ("q", ("cpu", "dtype", "small", "mis")), 1: ("k_cache", ("cpu", "dtype", "small", "mis")),
                              2: ("v_cache", ("cpu", "dtype", "small", "mis")), 3: ("seqlens", CONTIG),
                              5: ("k_new", ("cpu", "dtype", "small", "mis")), 6: ("v_new", ("cpu", "dtype", "small", "mis")),
                              7: ("bias", ALL), 8: ("key_padding_mask", ALL)}),
    "symm_stats_allreduce": (lambda: [[], [], 0, 0, 0, torch.zeros(2, dtype=torch.float64, device="cuda"),
                                      torch.zeros(2, dtype=torch.float64, device="cuda"), 0],
                             {5: ("src", NO_SMALL_C), 6: ("dst", CONTIG)}),
    "symm_fused_tail": (_fused_tail, {33: ("state", NO_SMALL_C), 16: ("ranges", CONTIG), 18: ("bucket_sq", CONTIG),
                                      19: ("block_sq", CONTIG), 20: ("grid_sync", CONTIG), (9, 0): ("master", NO_SMALL_V),
                                      (10, 0): ("exp_avg", VEC), (11, 0): ("exp_avg_sq", VEC), (12, 0): ("ema", VEC),
                                      21: ("stats_src", NO_SMALL_C), 22: ("stats_dst", CONTIG)}),
}

# callables without tensor operands: launch plans and queries, the symmetric-memory allocation, and the collectives
# that take raw peer addresses only
EXEMPT = {"norm_plan", "softmax_plan", "bias_gelu_plan", "gbf_plan", "head_permute_plan", "pair_plan", "embedding_plan",
          "fmha_decode_max_splits", "fmha_decode_num_splits", "fmha_det_timeouts", "symm_allreduce", "symm_reduce_scatter",
          "symm_pick_algo", "symm_error_channel", "symm_tail_max_blocks", "symm_mem_supported", "symm_multicast_supported",
          "SymmAllocation"}


def _call(name, args):
    fn = getattr(_nat(), name)
    if name.startswith("symm_"):
        with pytest.raises(RuntimeError, match=re.escape(NO_PEERS)):
            fn(*args)
    else:
        fn(*args)


def _replace(args, key, fn):
    if isinstance(key, tuple):
        i, j = key
        args[i] = list(args[i])
        args[i][j] = fn(args[i][j])
    else:
        args[key] = fn(args[key])


def test_every_binding_has_negative_cases():
    _nat()
    mod = importlib.import_module("unicore_b200._C")
    names = {n for n in dir(mod) if not n.startswith("_") and callable(getattr(mod, n))}
    assert names - EXEMPT == set(CASES), (sorted(names - EXEMPT - set(CASES)), sorted(set(CASES) - names))


@pytest.mark.parametrize("name", sorted(CASES))
def test_binding_rejects_bad_operands(name):
    build, operands = CASES[name]
    _call(name, build())   # the builder is valid: every operand check passes
    torch.cuda.synchronize()
    fn = getattr(_nat(), name)
    for n, (key, (label, kinds)) in enumerate(operands.items()):
        if n > 0 and torch.cuda.device_count() > 1:
            kinds = kinds + ("dev",)
        for kind in kinds:
            args = build()
            _replace(args, key, MUTATE[kind])
            with pytest.raises(RuntimeError, match=r"\b" + re.escape(label) + " must") as e:
                fn(*args)
            assert NO_PEERS not in str(e.value), (name, label, kind)
    torch.cuda.synchronize()


# ---- the inputs that reached a kernel or crashed the host before every operand went through one check ------------
def test_adam_per_tensor_lists_must_all_be_full():
    args = _adam()
    for i in range(5, 12):   # lr, beta1, beta2, eps, step, bias_correction, weight_decay
        short = list(args)
        short[i] = []
        with pytest.raises(RuntimeError, match="one entry per parameter"):
            _nat().multi_tensor_adam(*short)


def test_norm_backward_checks_mean_and_rstd():
    nat = _nat()
    dy, x, mean, rstd, gamma, _, _ = _norm_bwd()
    for bad in (mean.half(), mean[:-1].clone()):
        with pytest.raises(RuntimeError, match="mean must"):
            nat.layernorm_bwd(dy, x, bad, rstd, gamma)
    for bad in (rstd.double(), torch.ones(5, device="cuda")):
        with pytest.raises(RuntimeError, match="rstd must"):
            nat.rmsnorm_bwd(dy, x, bad, gamma)
    a = _bdaln_bwd()
    a[3] = a[3][:2].clone()
    with pytest.raises(RuntimeError, match="rstd must"):
        nat.bias_dropout_add_ln_bwd(*a)


def test_xent_backward_checks_target_lse_and_width():
    nat = _nat()
    logits, target, lse, one = _r(4, 64), torch.randint(0, 60, (4,), device="cuda"), _r(4, dtype=F32), torch.ones(1, device="cuda")
    with pytest.raises(RuntimeError, match="target must"):
        nat.softmax_xent_bwd(logits, target.int(), lse, one, -100, 0)
    with pytest.raises(RuntimeError, match="lse must"):
        nat.softmax_xent_bwd(logits, target, lse[:3].clone(), one, -100, 0)
    with pytest.raises(RuntimeError, match="logits must"):
        nat.softmax_xent_bwd(logits.view(-1), target, lse, one, -100, 0)
    with pytest.raises(RuntimeError, match="valid_cols"):
        nat.softmax_xent_bwd(logits, target, lse, one, -100, 65)


def test_gbf_backward_checks_its_operands():
    nat = _nat()
    dy, d, edge, mul_w, bias_w, means, stds = _gbf(dy=True)
    with pytest.raises(RuntimeError, match="edge must"):
        nat.gbf_bwd(dy, d, edge.int(), mul_w, bias_w, means, stds)
    with pytest.raises(RuntimeError, match="stds must"):
        nat.gbf_bwd(dy, d, edge, mul_w, bias_w, means, stds[:, :8].clone())
    with pytest.raises(RuntimeError, match="K must be"):
        nat.gbf_bwd(_r(2, 8, 12), d, edge, mul_w, bias_w, _r(1, 12), _r(1, 12))


def test_fmha_backward_checks_lse_bits_and_dout():
    nat = _nat()
    args = _fmha_bwd()
    for i, bad, label in ((0, args[0].float(), "dout"), (4, args[4].bfloat16(), "out"), (5, args[5].half(), "lse"),
                          (5, args[5][:, :, :-1].clone(), "lse"), (10, args[10][..., :-1].clone(), "drop_bits"),
                          (10, args[10].long(), "drop_bits"), (10, None, "dropout bits missing")):
        a = list(args)
        a[i] = bad
        with pytest.raises(RuntimeError, match=label):
            nat.fmha_bwd(*a)


def test_layout_plans_reject_shapes_no_launcher_takes():
    """The exempt launch-plan queries of the relayout and embedding kernels check their sizes as the bindings do."""
    nat = _nat()
    for args in ((0, 8, 3, 2, 8, F16), (2, 8, 5, 2, 8, F16), (2, 8, 3, 2, 4, F16), (2, 8, 3, 2, 6, F32)):
        with pytest.raises(RuntimeError, match="head_permute_plan needs"):
            nat.head_permute_plan(*args)
    for args in ((0, 8, 64), (1, 12, 64), (1, 8, 60), (1, 8, 0)):
        with pytest.raises(RuntimeError, match="pair_plan needs"):
            nat.pair_plan(*args)
    for args in ((-1, 10), (10, 0)):
        with pytest.raises(RuntimeError, match="embedding_plan needs"):
            nat.embedding_plan(*args)


def test_zero_width_inputs_raise_instead_of_dividing_by_zero():
    nat = _nat()
    with pytest.raises(RuntimeError, match="multiple of 8 columns"):
        nat.column_sum(torch.zeros(4, 0, dtype=F16, device="cuda"), None)
    d, edge, mul_w, bias_w, _, _ = _gbf()
    empty = torch.zeros(1, 0, dtype=F16, device="cuda")
    with pytest.raises(RuntimeError, match="K must be"):
        nat.gbf_fwd(d, edge, mul_w, bias_w, empty, empty)
