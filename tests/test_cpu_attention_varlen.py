"""Packed variable-length sequences on the CPU (float64, the varlen reference and the materialised module paths).

``attention_varlen_reference`` must be per-sequence ``attention_reference``, and the packed encoder stack must be the
padded one at every real row.  ``attention_reference`` takes its softmax in fp32 whatever the input dtype, so the
tolerances are those of fp32 sums over different key counts."""
import pytest
import torch

from unicore import ops
from unicore.modules import SelfMultiheadAttention
from unicore.modules.transformer import TransformerEncoder

LENS = [5, 0, 1, 16, 9]
L = 16


def _cu(lens):
    return torch.tensor([0] + lens).cumsum(0).to(torch.int32)


def _scatter(x):
    out = x.new_zeros(len(LENS), L, *x.shape[1:])
    s = 0
    for b, n in enumerate(LENS):
        out[b, :n] = x[s:s + n]
        s += n
    return out, torch.arange(L)[None, :] >= torch.tensor(LENS)[:, None]


def _gather(xp):
    return torch.cat([xp[b, :n] for b, n in enumerate(LENS)])


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("bias_batch", [None, 1, len(LENS)])
@pytest.mark.parametrize("H,H_kv", [(4, 4), (4, 2)])
def test_reference_is_per_sequence_attention(H, H_kv, bias_batch, causal):
    g = torch.Generator().manual_seed(H_kv * 7 + (bias_batch or 0))
    N, D = sum(LENS), 8
    q = torch.randn(N, H, D, generator=g, dtype=torch.float64)
    k, v = (torch.randn(N, H_kv, D, generator=g, dtype=torch.float64) for _ in range(2))
    bias = None if bias_batch is None else torch.randn(bias_batch, H, L, L, generator=g, dtype=torch.float64)
    out = ops.attention_varlen_reference(q, k, v, _cu(LENS), L, bias, causal=causal)
    s = 0
    for b, n in enumerate(LENS):
        if n:
            bb = None if bias is None else bias[b if bias_batch > 1 else 0, :, :n, :n][None]
            want = ops.attention_reference(q[None, s:s + n], k[None, s:s + n], v[None, s:s + n], bb, causal=causal)
            torch.testing.assert_close(out[s:s + n], want[0], rtol=1e-5, atol=1e-6)
        s += n


def test_reference_clamps_like_the_kernels():
    """A decreasing entry gives a length of 0, a start past N an empty sequence, a length above max_seqlen is cut."""
    g = torch.Generator().manual_seed(1)
    N, H, D = 20, 2, 8
    q, k, v = (torch.randn(N, H, D, generator=g, dtype=torch.float64) for _ in range(3))
    out = ops.attention_varlen_reference(q, k, v, torch.tensor([6, 2, 30, 40], dtype=torch.int32), 8)
    want = ops.attention_reference(q[None, 2:10], k[None, 2:10], v[None, 2:10])[0]   # sequence 1: rows 2..9
    torch.testing.assert_close(out[2:10], want, rtol=1e-5, atol=1e-6)
    assert torch.count_nonzero(out[:2]) == 0 and torch.count_nonzero(out[10:]) == 0


def test_varlen_positions_restart_in_every_sequence():
    pos = ops.varlen_positions(_cu(LENS), sum(LENS))
    assert pos.tolist() == [i for n in LENS for i in range(n)]


@pytest.mark.parametrize("rotary", [False, True], ids=["relpos", "rotary"])
@pytest.mark.parametrize("post_ln", [True, False], ids=["post_ln", "pre_ln"])
def test_packed_encoder_is_the_padded_one_at_real_rows(post_ln, rotary):
    torch.manual_seed(2)
    enc = TransformerEncoder(encoder_layers=2, embed_dim=32, ffn_embed_dim=64, attention_heads=4, emb_dropout=0.0,
                             dropout=0.0, attention_dropout=0.0, max_seq_len=L, rel_pos=not rotary, post_ln=post_ln,
                             rotary_dim=4 if rotary else None).double()
    emb = torch.randn(sum(LENS), 32, dtype=torch.float64, requires_grad=True)
    y = enc(emb, cu_seqlens=_cu(LENS), max_seqlen=L)
    embp, kpm = _scatter(emb.detach())
    embp.requires_grad_(True)
    yp = enc(embp, padding_mask=kpm)
    torch.testing.assert_close(y, _gather(yp), rtol=1e-5, atol=1e-6)
    dy = torch.randn_like(y)
    y.backward(dy)
    _gather(yp).backward(dy)
    torch.testing.assert_close(emb.grad, _gather(embp.grad), rtol=1e-5, atol=1e-6)


def test_packed_attention_rejects_what_it_cannot_do():
    attn = SelfMultiheadAttention(16, 2).double()
    x = torch.randn(sum(LENS), 16, dtype=torch.float64)
    with pytest.raises(ValueError):
        attn(x, return_attn=True, cu_seqlens=_cu(LENS), max_seqlen=L)
    with pytest.raises(ValueError):
        attn(x, key_padding_mask=torch.zeros(len(LENS), L, dtype=torch.bool), cu_seqlens=_cu(LENS), max_seqlen=L)
    with pytest.raises(ValueError):
        attn(x, cu_seqlens=_cu(LENS))


# ---- BERT: the packing collater, the model and the CLI ---------------------------------------------------------------
def test_packing_collater():
    from unicore.data import PackedSequenceDataset, RawArrayDataset

    items = [torch.arange(1, 6), torch.arange(10, 22), torch.arange(30, 31)]   # lengths 5, 12, 1
    ds = RawArrayDataset(items)
    batch = PackedSequenceDataset(ds, tokens_key="src_tokens").collater([ds[i] for i in range(3)])
    assert batch["src_tokens"].tolist() == torch.cat(items).tolist()
    assert batch["cu_seqlens"].dtype == torch.int32 and batch["cu_seqlens"].tolist() == [0, 5, 17, 18]
    assert batch["max_seqlen"] == 16   # 12 rounded up to a multiple of 8: the padded batch's width
    targets = [t * 2 for t in items]
    flat = PackedSequenceDataset(RawArrayDataset(targets)).collater(targets)
    assert torch.equal(flat, torch.cat(targets))
    for b in range(3):   # targets stay aligned with their tokens
        s, e = batch["cu_seqlens"][b], batch["cu_seqlens"][b + 1]
        assert torch.equal(flat[s:e], batch["src_tokens"][s:e] * 2)


def _bert_cpu_model():
    import importlib
    import os
    import sys

    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "examples"))
    importlib.import_module("bert")
    from unicore import options, tasks

    args = options.parse_args_and_arch(options.get_training_parser(), input_args=[
        "--task", "synthetic_mlm", "--loss", "masked_lm", "--arch", "bert_base", "--encoder-layers", "2",
        "--encoder-embed-dim", "32", "--encoder-ffn-embed-dim", "64", "--encoder-attention-heads", "4",
        "--synthetic-vocab-size", "120", "--synthetic-seq-len", "16", "--max-seq-len", "16", "--optimizer", "adam",
        "--lr", "1e-3", "--cpu", "--dropout", "0", "--attention-dropout", "0", "--emb-dropout", "0",
    ])
    torch.manual_seed(0)
    task = tasks.setup_task(args)
    return task.build_model(args).double(), task.dictionary.pad()


def test_packed_bert_is_the_padded_one():
    model, pad = _bert_cpu_model()
    g = torch.Generator().manual_seed(4)
    B = len(LENS)
    src = torch.randint(pad + 5, 120, (B, L), generator=g)
    real = torch.arange(L)[None, :] < torch.tensor(LENS)[:, None]
    src = src.masked_fill(~real, pad)
    masked = real & (torch.rand(B, L, generator=g) < 0.3)
    out = model(src, masked_tokens=masked)
    packed_src, packed_mask = _gather(src), _gather(masked)
    got = model(packed_src, masked_tokens=packed_mask, cu_seqlens=_cu(LENS), max_seqlen=L)
    torch.testing.assert_close(got, out, rtol=1e-5, atol=1e-6)


def test_pack_sequences_cli_logs_the_padded_run(tmp_path):
    """``--pack-sequences`` trains a few updates on the text-corpus pipeline and logs the same bsz, seq_len and (with
    dropout off, on the same weights and masks) loss as the right-padded run."""
    pytest.importorskip("tokenizers")
    import os
    import random
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    rng = random.Random(0)
    words = ["alpha", "beta", "gamma", "delta", "epsilon", "zeta", "eta", "theta", "iota", "kappa"]
    with open(tmp_path / "train.txt", "w") as f:
        for _ in range(64):
            f.write(" ".join(rng.choice(words) for _ in range(rng.randint(3, 20))) + " .\n")
    data = tmp_path / "data"
    prep = os.path.join(root, "examples", "bert", "example_data", "prepare_data.py")
    out = subprocess.run([sys.executable, prep, "--train", str(tmp_path / "train.txt"), "--valid",
                          str(tmp_path / "train.txt"), "--out", str(data),
                          "--build-dict", "--min-count", "1", "--format", "records"],
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert out.returncode == 0, out.stdout
    env = dict(os.environ, PYTHONPATH=root, OMP_NUM_THREADS="1")
    cmd = [sys.executable, os.path.join(root, "unicore_cli", "train.py"), str(data), "--user-dir",
           os.path.join(root, "examples", "bert"), "--task", "bert", "--loss", "masked_lm", "--arch", "bert_base",
           "--encoder-layers", "2", "--encoder-embed-dim", "32", "--encoder-ffn-embed-dim", "64",
           "--encoder-attention-heads", "4", "--max-seq-len", "32", "--optimizer", "adam", "--lr", "1e-3",
           "--lr-scheduler", "fixed", "--batch-size", "8", "--max-update", "4", "--log-format", "simple",
           "--log-interval", "1", "--num-workers", "0", "--cpu", "--disable-validation", "--no-save",
           "--dropout", "0", "--attention-dropout", "0", "--emb-dropout", "0",
           "--distributed-world-size", "1", "--seed", "1"]
    logs = {}
    for mode, extra in (("padded", []), ("packed", ["--pack-sequences"])):
        run = subprocess.run(cmd + extra, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                             timeout=600)
        assert run.returncode == 0, run.stdout[-4000:]
        logs[mode] = [line for line in run.stdout.splitlines() if "train_inner" in line]
        assert len(logs[mode]) >= 4, run.stdout[-4000:]

    def field(line, key):
        return float(line.split(key + "=")[1].split(",")[0].split()[0])

    for a, b in zip(logs["padded"], logs["packed"]):
        assert field(a, "bsz") == field(b, "bsz")
        assert field(a, "seq_len") == field(b, "seq_len")
        assert abs(field(a, "loss") - field(b, "loss")) <= 2e-3 * abs(field(a, "loss"))
