"""Packed variable-length sequences (cu_seqlens) in the wgmma forward and backward, the op layer and the encoder stack.

The varlen call must equal the padded kernel call on the same sequences scattered to ``[B, L]`` with
``key_padding_mask = (j >= len_b)`` and the same Philox seed: O, LSE and the keep bits bitwise at every real row (and
real key), dK / dV bitwise when dO is zero at the pad rows, and dQ / dBias too in deterministic mode.  Gradients are
also checked against the fp64 varlen reference, dBias is exactly 0 outside every sequence's block, malformed
cu_seqlens are clamped, and a packed encoder forward + backward does not synchronise."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]
DT_IDS = ["fp16", "bf16"]
GRAD_TOL = {torch.float16: 1e-2, torch.bfloat16: 5e-2}   # relative norm error against fp64
HEAD_DIMS = [8, 64, 96, 128]
LENS = [77, 0, 1, 200, 64, 129, 13]   # 0, 1, not multiples of 8 or 64, and max_seqlen itself
L = 200
SHORT = [77, 0, 1, 150, 64, 129, 13]   # every length below L: the union of the blocks is not the whole L x L
UNIT = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
P_DROP = 0.2
# (H, H_kv, bias: None / "shared" / "batch", dropout, causal)
MODES = {
    "plain": (12, 12, None, False, False),
    "shared_bias_dropout": (12, 12, "shared", True, False),
    "batch_bias_dropout_causal": (12, 12, "batch", True, True),
    "gqa4_dropout": (12, 4, "shared", True, False),
    "mqa_causal": (12, 1, None, False, True),
}


def _ops():
    from unicore import ops

    assert ops.USE_NATIVE, "native kernels must be active on the GPU box"
    return ops


def _vl():
    return _ops().native().varlen


def _eq(a, b, what):
    assert a.shape == b.shape and torch.equal(a, b), what


def _rel(got, want):
    return ((got.double() - want.double()).norm() / want.double().norm().clamp(min=1e-30)).item()


def _cu(lens):
    return torch.tensor([0] + lens, device="cuda").cumsum(0).to(torch.int32)


def _case(mode, D, dtype, seed=0, lens=LENS):
    H, H_kv, bias_kind, drop, causal = MODES[mode]
    g = torch.Generator(device="cuda").manual_seed(seed)
    N, B = sum(lens), len(lens)
    qkv = torch.randn(N, H + 2 * H_kv, D, device="cuda", generator=g).to(dtype)
    bias = None
    if bias_kind is not None:
        bias = torch.randn(1 if bias_kind == "shared" else B, H, L, L, device="cuda", generator=g).to(dtype)
    return qkv, bias, (P_DROP if drop else 0.0), causal, H, H_kv


def _split(qkv, H, H_kv):
    return qkv[:, :H], qkv[:, H:H + H_kv], qkv[:, H + H_kv:]


def _scatter(x):
    """packed [N, ...] -> padded [B, L, ...] with zeros at the pad rows; and the key mask j >= len_b"""
    out = x.new_zeros(len(LENS), L, *x.shape[1:])
    s = 0
    for b, n in enumerate(LENS):
        out[b, :n] = x[s:s + n]
        s += n
    kpm = torch.arange(L, device="cuda")[None, :] >= torch.tensor(LENS, device="cuda")[:, None]
    return out, kpm


def _gather(xp):
    return torch.cat([xp[b, :n] for b, n in enumerate(LENS)])


def _fwd_both(qkv, bias, p, causal, H, H_kv, scale):
    q, k, v = _split(qkv, H, H_kv)
    torch.cuda.manual_seed(11)
    out, lse, bits = _vl().fmha_varlen_fwd(q, k, v, _cu(LENS), L, bias, p, scale, causal=causal)
    qp, kpm = _scatter(q)
    kp, vp = _scatter(k)[0], _scatter(v)[0]
    torch.cuda.manual_seed(11)
    outp, lsep, bitsp = _ops().native().fmha_fwd(qp, kp, vp, bias, kpm, p, scale, causal=causal)
    return (q, k, v, out, lse, bits), (qp, kp, vp, kpm, outp, lsep, bitsp)


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("D", HEAD_DIMS)
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_forward_is_bitwise_the_padded_call(dtype, D, mode):
    qkv, bias, p, causal, H, H_kv = _case(mode, D, dtype)
    (_, _, _, out, lse, bits), (_, _, _, _, outp, lsep, bitsp) = _fwd_both(qkv, bias, p, causal, H, H_kv, D ** -0.5)
    _eq(out, _gather(outp), "O")
    # the bits of the first m keys of a word (key 2i in bit i, key 2i + 1 in bit 16 + i), as int32
    first = [sum(1 << (16 * (j & 1) + (j >> 1)) for j in range(m)) for m in range(33)]
    first = torch.tensor([x - (1 << 32) if x >= 1 << 31 else x for x in first], dtype=torch.int32, device="cuda")
    for b, n in enumerate(LENS):
        _eq(lse[b, :, :n], lsep[b, :, :n], ("LSE", b))
        if p > 0 and n > 0:
            # compared: the keys a row sees (j < n_b, and j <= i when causal); both forwards write those words
            w = (n + 31) // 32
            rows = torch.arange(n, device="cuda")
            seen = torch.minimum(rows + 1, torch.tensor(n, device="cuda")) if causal else torch.full_like(rows, n)
            m = (seen[:, None] - 32 * torch.arange(w, device="cuda")[None, :]).clamp(0, 32)
            keep = first[m]
            _eq(bits[b, :, :n, :w] & keep, bitsp[b, :, :n, :w] & keep, ("keep bits", b))


def _bwd_both(mode, D, dtype, det):
    qkv, bias, p, causal, H, H_kv = _case(mode, D, dtype, seed=1)
    scale = D ** -0.5
    (q, k, v, out, lse, bits), (qp, kp, vp, kpm, outp, lsep, bitsp) = _fwd_both(qkv, bias, p, causal, H, H_kv, scale)
    dout = torch.randn_like(out)
    doutp = _scatter(dout)[0]
    need = bias is not None
    with torch.no_grad():
        torch.use_deterministic_algorithms(det)
        try:
            got = _vl().fmha_varlen_bwd(dout, q, k, v, out, lse, _cu(LENS), L, bias, p, scale, bits, need, False,
                                        causal=causal)
            again = _vl().fmha_varlen_bwd(dout, q, k, v, out, lse, _cu(LENS), L, bias, p, scale, bits, need, False,
                                          causal=causal)
            want = _ops().native().fmha_bwd(doutp, qp, kp, vp, outp, lsep, bias, kpm, p, scale, bitsp, need, False,
                                            None, causal=causal)
        finally:
            torch.use_deterministic_algorithms(False)
    return got, again, want, bias


@pytest.mark.parametrize("mode", ["shared_bias_dropout", "batch_bias_dropout_causal", "gqa4_dropout"])
@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_backward_is_bitwise_the_padded_call(dtype, D, mode):
    got, _, want, _ = _bwd_both(mode, D, dtype, det=False)
    _eq(got[1], _gather(want[1]), "dK")
    _eq(got[2], _gather(want[2]), "dV")
    # default mode: the key tiles add their fp32 dQ shares in completion order, one 16-bit rounding apart at most (the
    # bound of test_gpu_attention_gqa.py)
    for x, y, name in ((got[0], _gather(want[0]), "dQ"), (got[3], want[3], "dBias")):
        err = (x.float() - y.float()).abs()
        assert bool((err <= 2 * UNIT[dtype] * y.float().abs() + 1e-3 * y.float().abs().max()).all()), name


@pytest.mark.parametrize("mode", ["shared_bias_dropout", "batch_bias_dropout_causal", "gqa4_dropout"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_deterministic_backward_is_bitwise_the_padded_call_and_repeats(dtype, mode):
    ops = _ops()
    got, again, want, bias = _bwd_both(mode, 64, dtype, det=True)
    for x, y, what in zip(got, again, ("dQ", "dK", "dV", "dBias")):
        _eq(x, y, ("repeat", what))
    _eq(got[0], _gather(want[0]), "dQ")
    _eq(got[1], _gather(want[1]), "dK")
    _eq(got[2], _gather(want[2]), "dV")
    _eq(got[3], want[3], "dBias")
    assert ops.native().fmha_det_timeouts() == 0


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_gradients_against_fp64_reference(dtype, mode):
    ops = _ops()
    qkv, bias, _, causal, H, H_kv = _case(mode, 64, dtype, seed=2)
    qkv.requires_grad_(True)
    if bias is not None:
        bias.requires_grad_(True)
    out = ops.fused_attention_varlen_qkvpacked(qkv, _cu(LENS), L, bias, causal=causal, num_kv_heads=H_kv)
    dout = torch.randn_like(out)
    out.backward(dout)
    assert qkv.grad is not None and qkv.grad.shape == qkv.shape   # one packed gradient
    q64 = qkv.detach().double().requires_grad_(True)
    b64 = None if bias is None else bias.detach().double().requires_grad_(True)
    ref = ops.attention_varlen_reference(*_split(q64, H, H_kv), _cu(LENS), L, b64, causal=causal)
    ref.backward(dout.double())
    assert _rel(out, ref) < GRAD_TOL[dtype]
    assert _rel(qkv.grad, q64.grad) < GRAD_TOL[dtype]
    if bias is not None:
        assert _rel(bias.grad, b64.grad) < GRAD_TOL[dtype]


@pytest.mark.parametrize("kind", ["shared", "batch"])
def test_dbias_is_zero_outside_every_block(kind):
    ops = _ops()
    mode = "shared_bias_dropout" if kind == "shared" else "batch_bias_dropout_causal"
    qkv, bias, p, causal, H, H_kv = _case(mode, 64, torch.float16, seed=3, lens=SHORT)
    bias.requires_grad_(True)
    out = ops.fused_attention_varlen_qkvpacked(qkv, _cu(SHORT), L, bias, dropout_p=p, causal=causal, num_kv_heads=H_kv)
    out.float().square().sum().backward()
    inside = torch.zeros(len(SHORT), 1, L, L, dtype=torch.bool, device="cuda")
    for b, n in enumerate(SHORT):
        inside[b, :, :n, :n] = True
    if kind == "shared":
        inside = inside.any(0, keepdim=True)
    assert not bool(inside.all())
    assert torch.count_nonzero(bias.grad.masked_fill(inside, 0)) == 0
    assert torch.count_nonzero(bias.grad) > 0


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_out_of_range_cu_seqlens_are_clamped(dtype):
    """Decreasing entries, entries past N and lengths above max_seqlen: the kernels clamp every sequence to
    s_b = clamp(cu[b], 0, N), n_b = clamp(cu[b + 1] - cu[b], 0, min(L, N - s_b)) and stay inside the tensors."""
    from unicore_b200.ops.attention_ops import _varlen_index

    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(4)
    N, H, D, Lm = 150, 4, 64, 64
    q, k, v = (torch.randn(N, H, D, device="cuda", generator=g).to(dtype) for _ in range(3))
    # lengths 0 (decreasing), 20, 64 (140 clamped to max_seqlen) and 0 (a start past N)
    cu = torch.tensor([50, 40, 60, 200, 1000], dtype=torch.int32, device="cuda")
    bias = torch.randn(4, H, Lm, Lm, device="cuda", generator=g).to(dtype)
    rows, valid = _varlen_index(cu, Lm, N)
    covered = torch.zeros(N, dtype=torch.bool, device="cuda")
    covered[rows[valid]] = True
    assert not bool(covered.all())
    # canary: NaN in the rows no sequence covers (the last key tile of a sequence reaches into them); the forward must
    # hide those keys by assignment and zero their V rows, so no NaN reaches a covered row
    qn, kn, vn = (t.masked_fill(~covered[:, None, None], float("nan")) for t in (q, k, v))
    out, lse, _ = _vl().fmha_varlen_fwd(qn, kn, vn, cu, Lm, bias, 0.0, D ** -0.5)
    assert bool(torch.isfinite(out[covered]).all())
    ref = ops.attention_varlen_reference(q.double(), k.double(), v.double(), cu, Lm, bias.double(), scale=D ** -0.5)
    # rows no clamped sequence covers are not written by the kernel; compare the covered ones
    assert _rel(out[covered], ref[covered]) < GRAD_TOL[dtype]
    dq, dk, dv, db = _vl().fmha_varlen_bwd(torch.ones_like(out), q, k, v, out, lse, cu, Lm, bias, 0.0, D ** -0.5, None,
                                           True, False)
    torch.cuda.synchronize()
    assert torch.isfinite(db).all()


def _valid():
    dt = torch.float16
    q, k, v = (torch.randn(24, 2, 64, device="cuda", dtype=dt) for _ in range(3))
    cu = torch.tensor([0, 10, 24], dtype=torch.int32, device="cuda")
    bias = torch.randn(2, 2, 16, 16, device="cuda", dtype=dt)
    return [q, k, v, cu, 16, bias, 0.0, 0.125]


BAD = {
    "q fp32": (0, lambda a: a[0].float()),
    "q on the cpu": (0, lambda a: a[0].cpu()),
    "q 4-d": (0, lambda a: a[0][None]),
    "q head dim 12": (0, lambda a: torch.randn(24, 2, 12, device="cuda", dtype=torch.float16)),
    "k rows": (1, lambda a: a[1][:16]),
    "v dtype": (2, lambda a: a[2].to(torch.bfloat16)),
    "kv heads not dividing": (2, lambda a: torch.randn(24, 3, 64, device="cuda", dtype=torch.float16)),
    "cu_seqlens int64": (3, lambda a: a[3].long()),
    "cu_seqlens on the cpu": (3, lambda a: a[3].cpu()),
    "cu_seqlens one entry": (3, lambda a: a[3][:1]),
    "cu_seqlens strided": (3, lambda a: torch.zeros(6, dtype=torch.int32, device="cuda")[::2]),
    "max_seqlen 0": (4, lambda a: 0),
    "max_seqlen not a multiple of 8": (4, lambda a: 12),
    "bias size": (5, lambda a: a[5][:, :, :8]),
    "bias batch": (5, lambda a: torch.randn(3, 2, 16, 16, device="cuda", dtype=torch.float16)),
    "bias dtype": (5, lambda a: a[5].float()),
}


def test_binding_rejects_bad_operands():
    _vl().fmha_varlen_fwd(*_valid())   # the builder is valid
    torch.cuda.synchronize()
    for label, (i, bad) in BAD.items():
        args = _valid()
        args[i] = bad(args)
        with pytest.raises(RuntimeError):
            _vl().fmha_varlen_fwd(*args)
        print("rejected:", label)
    q, k, v, cu, Lm, bias, p, scale = _valid()
    out, lse, bits = _vl().fmha_varlen_fwd(q, k, v, cu, Lm, bias, p, scale)
    good = [out, q, k, v, out, lse, cu, Lm, bias, 0.0, scale, None, True, False]
    _vl().fmha_varlen_bwd(*good)
    for i, bad in [(0, out[:, :1]), (4, out.float()), (5, lse[:, :, :8]), (5, lse.half())]:
        args = list(good)
        args[i] = bad
        with pytest.raises(RuntimeError):
            _vl().fmha_varlen_bwd(*args)
    with pytest.raises(RuntimeError):   # dropout without its keep bits
        _vl().fmha_varlen_bwd(*(good[:9] + [0.1] + good[10:]))


# ---- the encoder stack -----------------------------------------------------------------------------------------------
class C:
    """the tolerances of tests/test_gpu_encoder_path.py (relative norm error against float64)"""
    OUT = {torch.float16: 1e-2, torch.bfloat16: 5e-2}
    GRAD = {torch.float16: 2e-2, torch.bfloat16: 8e-2}


def _encoder(post_ln, rotary, dtype):
    from unicore.modules import TransformerEncoder

    torch.manual_seed(5)
    enc = TransformerEncoder(encoder_layers=2, embed_dim=256, ffn_embed_dim=512, attention_heads=4, emb_dropout=0.0,
                             dropout=0.0, attention_dropout=0.0, max_seq_len=L, rel_pos=not rotary, post_ln=post_ln,
                             rotary_dim=32 if rotary else None)
    return enc.cuda().to(dtype)


@pytest.mark.parametrize("rotary", [False, True], ids=["relpos", "rotary"])
@pytest.mark.parametrize("post_ln", [True, False], ids=["post_ln", "pre_ln"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_packed_encoder_against_fp64_and_the_padded_stack(dtype, post_ln, rotary):
    import copy

    enc = _encoder(post_ln, rotary, dtype)
    ref = copy.deepcopy(enc).double()
    g = torch.Generator(device="cuda").manual_seed(6)
    emb = torch.randn(sum(LENS), 256, device="cuda", generator=g).to(dtype).requires_grad_(True)
    cu = _cu(LENS)
    y = enc(emb, cu_seqlens=cu, max_seqlen=L)
    dy = torch.randn_like(y)
    y.backward(dy)
    e64 = emb.detach().double().requires_grad_(True)
    y64 = ref(e64, cu_seqlens=cu, max_seqlen=L)
    y64.backward(dy.double())
    assert _rel(y, y64) < C.OUT[dtype]
    assert _rel(emb.grad, e64.grad) < C.GRAD[dtype]
    for (name, p), (_, q) in zip(enc.named_parameters(), ref.named_parameters()):
        if p.dim() == 2:
            assert _rel(p.grad, q.grad) < C.GRAD[dtype], name
    # the padded stack on the same sentences, at the real rows
    embp, kpm = _scatter(emb.detach())
    with torch.no_grad():
        yp = enc(embp, padding_mask=kpm)
    assert _rel(y.detach(), _gather(yp)) < C.OUT[dtype]


def test_packed_encoder_does_not_synchronise():
    enc = _encoder(True, False, torch.float16)
    emb = torch.randn(sum(LENS), 256, device="cuda", dtype=torch.float16, requires_grad=True)
    cu = _cu(LENS)
    enc(emb, cu_seqlens=cu, max_seqlen=L).float().sum().backward()   # warm-up: caches, kernels loaded
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        enc(emb, cu_seqlens=cu, max_seqlen=L).float().sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


# ---- BERT through the Trainer --------------------------------------------------------------------------------------
def test_bert_packed_step_against_fp64_and_the_padded_step():
    """The batch of tests/test_gpu_encoder_path.py::test_bert_masked_lm_against_fp64 (BERT-base widths, 2 layers,
    L = 512, two padded sentences, dropout off, fp16), packed: one step through the Trainer's task step against a
    float64 copy of the model on the packed batch (loss, masked-token logits, every parameter gradient in the flat
    arena), and against the padded step of the same sentences, within the same bounds."""
    import copy

    import test_gpu_encoder_path as ep
    from unicore import utils

    _ops()
    trainer, batch = ep._bert_trainer([])
    lens = [ep.BERT_PADS.get(b, 512) for b in range(batch["target"].size(0))]
    src, tgt = batch["net_input"]["src_tokens"], batch["target"]
    packed = {
        "net_input": {"src_tokens": torch.cat([src[b, :n] for b, n in enumerate(lens)]),
                      "cu_seqlens": torch.tensor([0] + lens).cumsum(0).to(torch.int32), "max_seqlen": 512},
        "target": torch.cat([tgt[b, :n] for b, n in enumerate(lens)]),
    }
    got = ep._bert_step(trainer, packed)
    padded = ep._bert_step(trainer, batch)

    ref = copy.deepcopy(trainer.get_model()).double()
    ref.train()
    seen = []
    hook = ref.lm_head.register_forward_hook(lambda m, i, out: seen.append(out.detach()))
    try:
        loss64, _, log = trainer.loss(ref, utils.move_to_cuda(packed))
        loss64.backward()
    finally:
        hook.remove()
    assert log["bsz"] == len(lens) and log["seq_len"] == len(lens) * 512   # the padded batch's values
    grads64 = {n: p.grad for n, p in ref.named_parameters()}
    dtype = torch.float16
    for want, what in (((loss64.detach(), seen[0], grads64), "fp64"), (padded, "padded step")):
        ep._check(got[0], want[0], dtype, "output", what + ": loss")
        ep._check(got[1], want[1], dtype, "output", what + ": masked-token logits")
        assert set(got[2]) == set(want[2]), what
        for name, g in got[2].items():
            ep._check(g, want[2][name], dtype, ep._param_class(name), "{}: {}".format(what, name))
