"""The Python op layer over the attention kernels (``unicore_b200/ops/attention_ops.py``).

Checked: a one-token decoding step with a bias or key mask narrower than the visible keys gives the result of
``attention_with_kv_cache_reference``, as a chunk already does; the kernel calls (names and flags) of a
``SelfMultiheadAttention`` forward + backward in each mode, with one ``fused_attention_supported`` call per module call;
and, without a GPU, that the KV-cache op and its reference reject the same bad calls with the same messages.
"""
import pytest
import torch

UNIT = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}


def _ops():
    from unicore import ops

    assert ops.USE_NATIVE, "native kernels must be active on the GPU box"
    return ops


# ---- 1. one-token step with a narrow bias / key mask ----------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("narrow", ["bias", "kpm", "both"])
@pytest.mark.parametrize("step", ["cross", "self", "append"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
def test_step_with_narrow_bias_or_key_mask_matches_reference(dtype, step, narrow):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(3)
    B, H, H_kv, D, C = 3, 4, 2, 64, 64
    lens = [5, 20, 40]
    x = lambda *shape: torch.randn(*shape, device="cuda", generator=g).to(dtype)   # noqa: E731
    k, v, q = x(B, C, H_kv, D), x(B, C, H_kv, D), x(B, 1, H, D)
    k_new = v_new = seqlens = max_len = None
    if step != "cross":
        seqlens, max_len = torch.tensor(lens, dtype=torch.int32, device="cuda"), max(lens)
    if step == "append":
        k_new, v_new = x(B, 1, H_kv, D), x(B, 1, H_kv, D)
    # narrower than the visible keys: max_len (+ 1 when appending), or the capacity C without seqlens
    bias = x(B, H, 1, 24) if narrow in ("bias", "both") else None
    kpm = None
    if narrow in ("kpm", "both"):
        kpm = torch.zeros(B, 30, dtype=torch.bool, device="cuda")
        kpm[1, 2:9] = True
    scale = D ** -0.5
    kc, vc = k.clone(), v.clone()
    with torch.no_grad():
        out = ops.attention_with_kv_cache(q, kc, vc, seqlens, max_len, k_new, v_new, bias, kpm, scale)
    d = lambda t: None if t is None else t.double()   # noqa: E731
    kr, vr = k.double(), v.double()
    ref = ops.attention_with_kv_cache_reference(d(q), kr, vr, seqlens, max_len, d(k_new), d(v_new), d(bias), kpm,
                                                scale)
    mag = ops.attention_with_kv_cache_reference(d(q), k.double(), v.double().abs(), seqlens, max_len, d(k_new),
                                                None if v_new is None else v_new.double().abs(), d(bias), kpm, scale)
    assert torch.equal(kc.double(), kr) and torch.equal(vc.double(), vr)   # the same rows appended
    err = (out.double() - ref).abs()
    assert bool((err <= UNIT[dtype] * ref.abs() + 2.0 ** -13 * mag).all()), err.max().item()


# ---- 2. kernel calls of the attention module ------------------------------------------------------------------------
class _Recorder:
    """``native()`` that records each attention kernel call with the flags that select its variant."""

    def __init__(self, real):
        self.real, self.calls = real, []

    def __getattr__(self, name):
        target = getattr(self.real, name)

        def call(*args, **kwargs):
            if name == "fmha_fwd":
                self.calls.append((name, {"causal": kwargs.get("causal", False)}))
            elif name == "fmha_bwd":
                self.calls.append((name, {"need_dbias": args[11], "packed_grad": args[12],
                                          "dlogits": args[13] is not None, "causal": kwargs.get("causal", False)}))
            else:
                self.calls.append((name, {}))
            return target(*args, **kwargs)

        return call


def _fwd(causal=False):
    return ("fmha_fwd", {"causal": causal})


def _bwd(packed_grad=True, need_dbias=True, dlogits=False, causal=False):
    return ("fmha_bwd", {"need_dbias": need_dbias, "packed_grad": packed_grad, "dlogits": dlogits, "causal": causal})


MODES = {
    # mode: (module arguments, call arguments, kernel calls of forward + backward); the bias always needs a gradient
    "plain": ({}, {}, [_fwd(), _bwd()]),
    "causal": ({}, {"causal": True}, [_fwd(True), _bwd(causal=True)]),
    "logits": ({}, {"return_attn": True, "need_probs": False},
               [("fmha_fwd_logits", {}), _bwd(dlogits=True)]),
    # the kernels do not return the logits of causal attention: attention_reference runs, no kernel
    "causal_logits": ({}, {"return_attn": True, "need_probs": False, "causal": True}, []),
    "gqa_packed": ({"num_kv_heads": 1}, {}, [_fwd(), _bwd()]),
    "rotary": ({"rotary_dim": 32}, {"causal": True}, [_fwd(True), _bwd(causal=True)]),
}


def _count_predicate(monkeypatch):
    """Counts the calls of ``fused_attention_supported`` from the module (``unicore.ops``) and from the ops."""
    import unicore_b200.ops.attention_ops as attention_ops
    from unicore import ops

    real, count = attention_ops.fused_attention_supported, [0]

    def counted(*args, **kwargs):
        count[0] += 1
        return real(*args, **kwargs)

    monkeypatch.setattr(attention_ops, "fused_attention_supported", counted)
    monkeypatch.setattr(ops, "fused_attention_supported", counted)
    return count


@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(MODES))
def test_module_kernel_calls(mode, monkeypatch):
    import unicore_b200.ops.attention_ops as attention_ops
    from unicore.modules import SelfMultiheadAttention

    ops = _ops()
    module_args, call_args, want = MODES[mode]
    B, L, E, H = 2, 64, 256, 4
    torch.manual_seed(0)
    attn = SelfMultiheadAttention(E, H, dropout=0.1, **module_args).cuda().half().train()
    x = torch.randn(B, L, E, device="cuda").half().requires_grad_()
    kpm = torch.zeros(B, L, dtype=torch.bool, device="cuda")
    kpm[1, L - 8:] = True
    bias = torch.randn(B, H, L, L, device="cuda").half().requires_grad_()
    rec = _Recorder(ops.native())
    monkeypatch.setattr(attention_ops, "native", lambda: rec)
    count = _count_predicate(monkeypatch)
    res = attn(x, key_padding_mask=kpm, attn_bias=bias, **call_args)
    loss = res[0].float().sum() + res[1].float().nan_to_num(0.0, 0.0, 0.0).sum() if call_args.get("return_attn") \
        else res.float().sum()
    loss.backward()
    assert count[0] == 1
    assert rec.calls == want
    assert x.grad is not None and attn.in_proj.weight.grad is not None and bias.grad is not None


@pytest.mark.gpu
def test_non_contiguous_projection_runs_the_unpacked_backward(monkeypatch):
    import unicore_b200.ops.attention_ops as attention_ops

    ops = _ops()
    B, L, H, D = 2, 64, 4, 64
    buf = torch.randn(B, L, 4, H, D, device="cuda").half().requires_grad_()
    qkv = buf[:, :, :3]
    assert not qkv.is_contiguous()
    rec = _Recorder(ops.native())
    monkeypatch.setattr(attention_ops, "native", lambda: rec)
    count = _count_predicate(monkeypatch)
    ops.fused_attention_qkvpacked(qkv, dropout_p=0.1).float().sum().backward()
    assert count[0] == 1
    assert rec.calls == [_fwd(), _bwd(packed_grad=False, need_dbias=False)]
    assert bool((buf.grad[:, :, 3] == 0).all()) and bool(buf.grad[:, :, :3].abs().sum() > 0)


# ---- 3. the KV-cache argument plan (no GPU) -------------------------------------------------------------------------
def _bad_calls():
    B, C, H, H_kv, D = 2, 16, 4, 2, 8
    q1, q3 = torch.randn(B, 1, H, D), torch.randn(B, 3, H, D)
    k, v = torch.randn(B, C, H_kv, D), torch.randn(B, C, H_kv, D)
    new1, new3 = torch.randn(B, 1, H_kv, D), torch.randn(B, 3, H_kv, D)
    lens = torch.tensor([3, 4], dtype=torch.int32)
    return {
        "heads_do_not_divide": (q1, torch.randn(B, C, 3, D), torch.randn(B, C, 3, D)),
        "cache_heads_differ": (q1, k, torch.randn(B, C, 1, D)),
        "k_new_alone": (q1, k, v, lens, None, new1, None),
        "v_new_alone": (q1, k, v, lens, None, None, new1),
        "append_without_seqlens": (q1, k, v, None, None, new1, new1),
        "new_heads_differ": (q1, k, v, lens, None, torch.randn(B, 1, 1, D), torch.randn(B, 1, 1, D)),
        "chunk_with_seqlens_does_not_append": (q3, k, v, lens, 4),
        "step_past_capacity": (q1, k, v, lens, C, new1, new1),
        "chunk_past_capacity": (q3, k, v, lens, C - 2, new3, new3),
        "bound_past_capacity": (q1, k, v, lens, C + 1),
    }


@pytest.mark.parametrize("case", list(_bad_calls()))
def test_kv_cache_op_and_reference_reject_alike(case):
    from unicore import ops

    args = _bad_calls()[case]
    errors = []
    for fn in (ops.attention_with_kv_cache, ops.attention_with_kv_cache_reference):
        with torch.no_grad(), pytest.raises(ValueError) as info:
            fn(*[a.clone() if isinstance(a, torch.Tensor) else a for a in args])
        errors.append(str(info.value))
    assert errors[0] == errors[1]
