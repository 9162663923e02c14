"""CPU tests of the Python layers: registries, options, schedulers, loss scaler, flat arenas,
metrics, data pipeline, EMA, modules (fallback paths)."""
import argparse
import math
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "examples"))

import unicore  # noqa: E402
from unicore import metrics, options, registry, utils  # noqa: E402
from unicore.data import (  # noqa: E402
    CountingIterator, Dictionary, EpochBatchIterator, GroupedIterator, MaskTokensDataset, NestedDictionaryDataset,
    NumelDataset, RawArrayDataset, RightPadDataset, RightPadDataset2D, ShardedIterator, SortDataset, UnicoreDataset,
    data_utils,
)
from unicore.logging import meters  # noqa: E402
from unicore.optim import lr_scheduler  # noqa: E402
from unicore.optim.dynamic_loss_scaler import DynamicLossScaler  # noqa: E402
from unicore.optim.fp16_optimizer import (  # noqa: E402
    flatten_parameters, flatten_parameters_fp32, pad_numel, separate_decay_params,
)


def bert_args(extra=()):
    import bert  # noqa: F401  (examples/bert plug-in)

    parser = options.get_training_parser()
    base = [
        "--task", "synthetic_mlm", "--loss", "masked_lm", "--arch", "bert_base", "--encoder-layers", "2",
        "--encoder-embed-dim", "32", "--encoder-ffn-embed-dim", "64", "--encoder-attention-heads", "4",
        "--synthetic-vocab-size", "120", "--synthetic-seq-len", "16", "--synthetic-num-samples", "64",
        "--max-seq-len", "32", "--optimizer", "adam", "--batch-size", "8", "--distributed-world-size", "1",
        "--cpu", "--num-workers", "0", "--log-format", "none",
    ]
    extra = list(extra)
    if "--lr" not in extra:
        extra += ["--lr", "1e-3"]
    if "--lr-scheduler" not in extra:
        extra += ["--lr-scheduler", "polynomial_decay", "--warmup-updates", "5", "--total-num-update", "40"]
    return options.parse_args_and_arch(parser, input_args=base + extra)


# ---------------------------------------------------------------------------------------------------
def test_registry_and_aliases():
    assert sorted(registry.REGISTRIES) == ["loss", "lr_scheduler", "optimizer"]
    assert set(registry.REGISTRIES["lr_scheduler"]["registry"]) == {
        "cosine", "exponential_decay", "fixed", "inverse_sqrt", "pass_through", "polynomial_decay",
        "reduce_lr_on_plateau", "tri_stage", "triangular",
    }
    assert set(registry.REGISTRIES["optimizer"]["registry"]) == {"adam", "sgd", "adagrad", "adadelta"}
    import unicore.distributed_utils as du  # alias module
    from unicore import progress_bar  # noqa: F401

    assert du is unicore.distributed.utils
    build, register, table = registry.setup_registry("--widget", default=None)

    @register("a")
    class A:
        @staticmethod
        def add_args(p):
            p.add_argument("--widget-size", type=int, default=7)

        def __init__(self, args):
            self.size = args.widget_size

    with pytest.raises(ValueError):
        register("a")(type("B", (), {}))
    ns = argparse.Namespace(widget="a")
    assert build(ns).size == 7  # defaults back-filled from add_args
    del registry.REGISTRIES["widget"]
    from unicore.data.pad_dataset import RightPadDataset as legacy  # legacy module path

    assert legacy is RightPadDataset


def test_options_two_pass_and_arch_defaults():
    args = bert_args(["--encoder-layers", "3", "--adam-betas", "(0.9, 0.98)", "--update-freq", "2,4"])
    assert args.encoder_layers == 3 and args.encoder_attention_heads == 4
    assert args.post_ln is True and args.activation_fn == "gelu" and args.dropout == 0.1
    assert args.update_freq == [2, 4] and args.lr == [1e-3]
    assert args.batch_size_valid == 8 and args.bf16 is False and args.ddp_backend == "c10d"
    assert args.fp16_init_scale == 128 and args.bucket_cap_mb == 25 and args.restore_file == "checkpoint_last.pt"


def _sched(name, extra, lr="1e-3", total=None):
    from unicore.optim import build_optimizer

    ns = bert_args(["--lr-scheduler", name, "--lr", lr] + extra)
    p = torch.nn.Parameter(torch.zeros(3))
    opt = build_optimizer(ns, [("w", p)])
    return lr_scheduler.build_lr_scheduler(ns, opt, total), opt


def test_lr_schedulers_closed_form():
    s, opt = _sched("polynomial_decay", ["--warmup-updates", "5", "--total-num-update", "40"])
    assert s.step_update(4) == pytest.approx(0.0008)
    assert s.step_update(8) == pytest.approx(0.000914286, rel=1e-5)
    assert s.step_update(12) == pytest.approx(0.0008)
    assert s.step_update(400) == 0.0
    s, _ = _sched("inverse_sqrt", ["--warmup-updates", "100"])
    assert s.step_update(50) == pytest.approx(5e-4)
    assert s.step_update(400) == pytest.approx(1e-3 * (100 / 400) ** 0.5)
    s, _ = _sched("fixed", ["--warmup-updates", "10"])
    s.step_begin_epoch(1)
    assert s.step_update(4) == pytest.approx(1e-3 * 5 / 10)
    assert s.step_update(100) == pytest.approx(1e-3)
    s, _ = _sched("cosine", ["--warmup-updates", "10", "--min-lr", "1e-5", "--lr-period-updates", "100"], total=1000)
    assert s.step_update(10) == pytest.approx(1e-3)
    assert s.step_update(60) == pytest.approx(1e-5 + 0.5 * (1e-3 - 1e-5) * (1 + math.cos(math.pi * 0.5)))
    s, _ = _sched("tri_stage", ["--warmup-steps", "10", "--hold-steps", "10", "--decay-steps", "10"])
    assert s.step_update(0) == pytest.approx(1e-5)
    assert s.step_update(15) == pytest.approx(1e-3)
    assert s.step_update(10_000) == pytest.approx(1e-5)
    s, _ = _sched("triangular", ["--max-lr", "1e-2", "--lr-period-updates", "100"])
    assert s.step_update(50) == pytest.approx(1e-2)
    assert s.step_update(100) == pytest.approx(1e-3)
    s, _ = _sched("exponential_decay", ["--warmup-updates", "10", "--decay-ratio", "0.5", "--decay-steps", "10"])
    assert s.step_update(5) == pytest.approx(5e-4)
    assert s.step_update(20) == pytest.approx(1e-3 * 0.5)
    s, opt = _sched("reduce_lr_on_plateau", ["--lr-shrink", "0.5"])
    s.step(1, 1.0)
    s.step(2, 2.0)
    assert opt.get_lr() == pytest.approx(5e-4)


def test_dynamic_loss_scaler_state_machine():
    sc = DynamicLossScaler(init_scale=4.0, scale_window=2, tolerance=0.0, min_loss_scale=0.5)
    sc.check_overflow(1.0)  # finite: nothing happens
    with pytest.raises(OverflowError):
        sc.check_overflow(float("inf"))
    assert sc.loss_scale == 2.0
    sc.update()
    sc.update()
    assert sc.loss_scale == 4.0  # grew after scale_window clean updates
    with pytest.raises(OverflowError):
        sc.check_overflow(float("nan"))
    with pytest.raises(OverflowError):
        sc.check_overflow(float("inf"))
    with pytest.raises(FloatingPointError):
        sc.check_overflow(float("inf"))  # would reach min_loss_scale
    assert sc.loss_scale == 1.0


def test_decay_partition_and_flat_layout():
    m = torch.nn.Sequential(torch.nn.Linear(3, 5), torch.nn.LayerNorm(5), torch.nn.Linear(5, 3, bias=False)).half()
    ns = argparse.Namespace(weight_decay=0.01, no_weight_decay_names="")
    groups = separate_decay_params(ns, list(m.named_parameters()))
    assert [len(g["params"]) for g in groups] == [2, 3] and groups[1]["weight_decay"] == 0.0
    ns0 = argparse.Namespace(weight_decay=0.0, no_weight_decay_names="")
    assert len(separate_decay_params(ns0, list(m.named_parameters()))) == 1
    params = groups[1]["params"]  # bias(5), ln.weight(5), ln.bias(5): each padded to 6
    before = [p.detach().clone() for p in params]
    flats = flatten_parameters(params)
    assert len(flats) == 1 and flats[0].numel() == 3 * pad_numel(5) == 18
    for i, (p, b) in enumerate(zip(params, before)):
        assert torch.equal(p.data, b)
        assert p.data.data_ptr() == flats[0].data.data_ptr() + i * 6 * 2  # views at padded offsets
        assert p.grad.data_ptr() == flats[0].grad.data_ptr() + i * 6 * 2
    master = flatten_parameters_fp32(params)
    assert master.dtype == torch.float32 and master.numel() == 18
    assert torch.equal(master.data[6:11], before[1].float())


def test_meters_and_metrics_roundtrip():
    metrics.reset()
    with metrics.aggregate("train"):
        metrics.log_scalar("loss", 2.0, weight=2)
        metrics.log_scalar("loss", 4.0, weight=2)
        with metrics.aggregate("inner"):
            metrics.log_scalar("x", 1.0)
        with metrics.aggregate(new_root=True) as agg:
            metrics.log_scalar("val", 7.0)
        assert "val" in agg and metrics.get_meter("train", "val") is None
    assert metrics.get_smoothed_value("train", "loss") == 3.0
    assert metrics.get_smoothed_value("default", "x") == 1.0
    state = metrics.state_dict()
    metrics.reset()
    metrics.load_state_dict(state)
    assert metrics.get_smoothed_value("train", "loss") == 3.0
    md = meters.MetersDict()
    md.add_meter("b", meters.AverageMeter(), 20)
    md.add_meter("a", meters.AverageMeter(), 10)
    assert list(md.keys()) == ["a", "b"]


class _ListDataset(UnicoreDataset):
    def __init__(self, n, length=5):
        self.items = [torch.arange(4, 4 + 1 + (i % length)) for i in range(n)]

    def __getitem__(self, i):
        return self.items[i]

    def __len__(self):
        return len(self.items)

    def collater(self, samples):
        return data_utils.collate_tokens(samples, 0, pad_to_multiple=8)


def test_data_utils_and_iterators():
    a, b = torch.tensor([1, 2, 3]), torch.tensor([4])
    out = data_utils.collate_tokens([a, b], 0, pad_to_multiple=8)
    assert out.shape == (2, 8) and out[1].tolist() == [4, 0, 0, 0, 0, 0, 0, 0]
    out = data_utils.collate_tokens([a, b], 9, left_pad=True)
    assert out[1].tolist() == [9, 9, 4]
    sq = data_utils.collate_tokens_2d([torch.ones(2, 2), torch.ones(3, 3)], 0)
    assert sq.shape == (2, 3, 3) and sq[0, 2].sum() == 0
    batches = data_utils.batch_by_size(np.arange(10), batch_size=4, required_batch_size_multiple=1)
    assert [len(x) for x in batches] == [4, 4, 2]
    with data_utils.numpy_seed(3, 4):
        x = np.random.rand()
    with data_utils.numpy_seed(3, 4):
        assert np.random.rand() == x
    it = CountingIterator(list(range(10)))
    assert next(it) == 0 and it.n == 1 and it.has_next()
    it.skip(3)
    assert next(it) == 4
    assert [list(g) for g in GroupedIterator(CountingIterator(list(range(5))), 2)] == [[0, 1], [2, 3], [4]]
    assert list(ShardedIterator(list(range(5)), 2, 1, fill_value=-1)) == [1, 3, -1]

    ds = _ListDataset(23)
    batches = ds.batch_by_size(ds.ordered_indices(), batch_size=4)

    def make(shard, num_shards=2):
        return EpochBatchIterator(ds, ds.collater, batches, seed=7, num_shards=num_shards, shard_id=shard)

    e0, e1 = make(0), make(1)
    assert len(e0) == len(e1) == 3
    seen = [b for e in (e0, e1) for b in e.next_epoch_itr(shuffle=True) if len(b) > 0]
    assert sum(x.shape[0] for x in seen) == 23
    # resume mid-epoch: the restored iterator yields exactly the remaining batches
    full = [x.clone() for x in make(0).next_epoch_itr(shuffle=True)]
    e = make(0)
    itr = e.next_epoch_itr(shuffle=True)
    next(itr)
    state = e.state_dict()
    assert state["iterations_in_epoch"] == 1 and state["epoch"] == 1
    r = make(0)
    r.load_state_dict(state)
    rest = list(r.next_epoch_itr(shuffle=True))
    assert len(rest) == 2 and all(torch.equal(x, y) for x, y in zip(rest, full[1:]))
    # epoch boundary
    while itr.has_next():
        next(itr)
    assert e.end_of_epoch() and e.state_dict()["epoch"] == 2 and e.next_epoch_idx == 2


def test_dictionary_and_masking(tmp_path):
    f = tmp_path / "dict.txt"
    f.write_text("[PAD]\n[UNK]\n[CLS]\n[SEP]\nhello 5\nworld 3\n")
    d = Dictionary.load(str(f))
    assert len(d) == 6 and d.pad() == 0 and d.index("nope") == d.unk() and d.index("world") == 5
    mask_idx = d.add_symbol("[MASK]", is_special=True)
    for i in range(30):
        d.add_symbol("w%d" % i)
    base = RawArrayDataset([torch.randint(7, len(d), (20,)) for _ in range(8)])
    src, tgt = MaskTokensDataset.apply_mask(base, d, pad_idx=d.pad(), mask_idx=mask_idx, seed=5, mask_prob=0.3)
    src.set_epoch(1)
    tgt.set_epoch(1)
    s0, t0 = src[0], tgt[0]
    masked = t0 != d.pad()
    assert 3 <= masked.sum() <= 8 and not masked[0] and not masked[-1]
    assert torch.equal(t0[masked], base[0][masked])          # targets hold the original tokens
    assert torch.equal(s0[~masked], base[0][~masked])        # unmasked positions untouched
    assert torch.equal(src[0], s0)                           # deterministic per (seed, epoch, index)
    src.set_epoch(2)
    tgt.set_epoch(2)
    assert not torch.equal(tgt[0], t0) or not torch.equal(src[0], s0)
    nested = NestedDictionaryDataset(
        {"net_input": {"src_tokens": RightPadDataset(src, pad_idx=0)}, "target": RightPadDataset(tgt, pad_idx=0),
         "n": NumelDataset(src, reduce=True)}
    )
    batch = nested.collater([nested[i] for i in range(3)])
    assert batch["net_input"]["src_tokens"].shape == (3, 24) and batch["n"] == 60
    order = SortDataset(nested, sort_order=[np.array([3, 1, 2, 0, 4, 5, 6, 7])]).ordered_indices()
    assert order[0] == 3 and order[1] == 1
    assert RightPadDataset2D(RawArrayDataset([torch.ones(3, 3)]), 0).collater([torch.ones(3, 3)]).shape == (1, 8, 8)


def test_softmax_dropout_fallback_and_modules():
    from unicore.modules import LayerNorm, RMSNorm, SelfMultiheadAttention, TransformerEncoder, softmax_dropout

    x = torch.randn(2, 4, 8, 16)
    mask = torch.zeros(2, 1, 1, 16)
    mask[..., -3:] = -1e4
    bias = torch.randn(1, 4, 8, 16)
    ref = torch.softmax(x + mask + bias, -1)
    out = softmax_dropout(x.clone(), 0.0, True, mask=mask, bias=bias)
    assert torch.allclose(out, ref, atol=1e-6)
    assert torch.allclose(LayerNorm(16)(x), torch.nn.functional.layer_norm(x, (16,)), atol=1e-6)
    assert RMSNorm(16)(x).shape == x.shape
    attn = SelfMultiheadAttention(32, 4, dropout=0.0)
    q = torch.randn(2, 8, 32)
    pad = torch.zeros(2, 8, dtype=torch.bool)
    pad[1, 6:] = True
    o, logits, probs = attn(q, key_padding_mask=pad, attn_bias=torch.randn(8, 8, 8), return_attn=True)
    assert o.shape == (2, 8, 32) and probs.shape == (8, 8, 8) and probs[4:, :, 6:].abs().max() == 0
    assert torch.allclose(attn(q, key_padding_mask=pad, attn_bias=None), attn(q, key_padding_mask=pad), atol=1e-6)
    enc = TransformerEncoder(encoder_layers=2, embed_dim=32, ffn_embed_dim=64, attention_heads=4, max_seq_len=16,
                             emb_dropout=0.0, dropout=0.0, attention_dropout=0.0, post_ln=True).eval()
    y = enc(torch.randn(2, 8, 32), padding_mask=pad)
    assert y.shape == (2, 8, 32) and torch.isfinite(y).all()
    keys = set(enc.state_dict().keys())
    assert "layers.0.self_attn.in_proj.weight" in keys and "relative_attention_bias.weight" in keys
    assert "emb_layer_norm.weight" in keys and "layers.1.final_layer_norm.bias" in keys


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_softmax_cross_entropy_fallback_keeps_at_least_fp32(dtype):
    """The fallback reduces fp32 logits in fp32 and fp64 logits (a float64 reference model) in fp64."""
    from unicore import ops

    torch.manual_seed(0)
    logits = (torch.randn(16, 50, dtype=torch.float64) * 4).to(dtype)
    target = torch.randint(0, 50, (16,))
    target[3] = 0
    loss = ops.softmax_cross_entropy(logits, target, ignore_index=0)
    keep = target != 0
    want = -torch.log_softmax(logits.double(), -1)[keep, target[keep]].sum()
    assert loss.dtype == dtype
    assert abs(loss.item() - want.item()) <= (1e-12 if dtype == torch.float64 else 1e-5) * want.item()


def test_bert_parameter_count_and_names():
    import bert  # noqa: F401
    from unicore.tasks.synthetic import build_synthetic_dictionary
    from unicore_b200.models.bert import BertModel, apply_arch

    ns = argparse.Namespace()
    apply_arch(ns, "bert_base")
    model = BertModel(ns, build_synthetic_dictionary(30522))
    n = sum(p.numel() for p in model.parameters())
    assert n == 109_513_146  # SURVEY section 6.4 / Appendix G
    names = [k for k, _ in model.named_parameters()]
    assert names[:4] == ["embed_tokens.weight", "embed_positions.weight", "sentence_encoder.emb_layer_norm.weight",
                         "sentence_encoder.emb_layer_norm.bias"]
    assert len(names) == 154 and len(model.state_dict()) == 155


def test_ema_and_utils():
    from unicore.ema import ExponentialMovingAverageModel

    ns = argparse.Namespace(weight_decay=0.0, no_weight_decay_names="")
    m = torch.nn.Linear(4, 4)
    ema = ExponentialMovingAverageModel(ns, m, 0.9)
    w0 = m.weight.detach().clone()
    with torch.no_grad():
        m.weight.add_(1.0)
    ema.update(m.named_parameters())
    assert torch.allclose(ema.model_ema.weight, w0 + 0.1)
    assert set(ema.state_dict()) == {"params", "decay"}
    with utils.torch_seed(1, 2, 3):
        a = torch.rand(3)
    with utils.torch_seed(1, 2, 3):
        assert torch.equal(torch.rand(3), a)
    assert utils.eval_str_list("1e-3,2e-3") == [1e-3, 2e-3] and utils.eval_str_list("[2,3]", int) == [2, 3]
    moved = utils.move_to_cpu({"a": torch.ones(2, dtype=torch.half), "b": [torch.ones(1)]})
    assert moved["a"].dtype == torch.float32
    g = [torch.full((4,), 3.0), torch.full((9,), 4.0)]
    assert utils.multi_tensor_total_norm(g).item() == pytest.approx(math.sqrt(36 + 144))
    out = torch.empty(4096, dtype=torch.bfloat16)
    utils.fp32_to_bf16_sr(torch.full((4096,), 1.0 + 2 ** -10), out)
    assert abs(out.float().mean().item() - (1 + 2 ** -10)) < 1e-3
    y = utils.checkpoint_sequential([torch.nn.Linear(4, 4), torch.tanh], torch.randn(2, 4, requires_grad=True))
    y.sum().backward()


def test_host_read_helpers_and_lazy_stats_cpu():
    """utils.item / tolist / AsyncHostRead / mask_to_index degrade gracefully on CPU tensors."""
    import torch

    from unicore import utils

    t = torch.tensor([3.5])
    assert utils.item(t) == 3.5 and utils.item(2) == 2
    assert utils.tolist(torch.tensor([1.0, 2.0])) == [1.0, 2.0]
    pending = utils.AsyncHostRead(torch.tensor(7.0))
    assert pending.ready() and pending.get() == 7.0
    mask = torch.tensor([[True, False, True], [False, False, True]])
    idx = utils.mask_to_index(mask)
    assert idx.tolist() == [0, 2, 5] and utils.mask_to_index(mask) is idx  # cached per mask object
    x = torch.arange(12.0).view(2, 3, 2)
    assert torch.equal(x[mask], x.reshape(-1, 2).index_select(0, idx))


def test_meters_localize_and_scheduler_module_aliases():
    import torch

    from unicore.logging import meters
    from unicore.optim.lr_scheduler.polynomial_decay_schedule import PolynomialDecayLRSchedule
    from unicore.optim.lr_scheduler import LR_SCHEDULER_REGISTRY

    assert LR_SCHEDULER_REGISTRY["polynomial_decay"] is PolynomialDecayLRSchedule
    md = meters.MetersDict()
    md.add_meter("loss", meters.AverageMeter(round=3), 10)
    md["loss"].update(torch.tensor(2.0), 4)
    md["loss"].update(torch.tensor(4.0), 4)
    md.localize()  # no CUDA tensors: a no-op that must not disturb the values
    assert abs(float(md.get_smoothed_values()["loss"]) - 3.0) < 1e-6


def test_torch_seed_is_scoped_and_reproducible():
    import torch

    from unicore import utils

    torch.manual_seed(11)
    outside_a = torch.rand(3)
    torch.manual_seed(11)
    with utils.torch_seed(5, 1, 2):
        inside_a = torch.rand(3)
    outside_b = torch.rand(3)
    with utils.torch_seed(5, 1, 2):
        inside_b = torch.rand(3)
    with utils.torch_seed(5, 1, 3):
        inside_c = torch.rand(3)
    assert torch.equal(outside_a, outside_b) and torch.equal(inside_a, inside_b) and not torch.equal(inside_a, inside_c)


def test_iterator_resume_with_a_different_world_size():
    """A position saved by a 2-rank run is rescaled when the job resumes on 1 rank (and back): the restored
    iterator has the remaining fraction of the epoch left (reference ``iterators.py:331-336``)."""
    ds = _ListDataset(64, length=1)
    batches = ds.batch_by_size(ds.ordered_indices(), batch_size=4)  # 16 batches

    def make(num_shards, shard):
        return EpochBatchIterator(ds, ds.collater, batches, seed=3, num_shards=num_shards, shard_id=shard)

    two = make(2, 0)
    assert len(two) == 8
    itr = two.next_epoch_itr(shuffle=True)
    for _ in range(2):
        next(itr)
    state = two.state_dict()
    assert state["iterations_in_epoch"] == 2 and state["len"] == 8
    one = make(1, 0)
    assert len(one) == 16
    one.load_state_dict(state)
    rest = list(one.next_epoch_itr(shuffle=True))
    assert len(rest) == 16 - 4  # a quarter of the epoch was consumed
    back = make(2, 1)
    one_state = {"epoch": 1, "iterations_in_epoch": 8, "shuffle": True, "len": 16}
    back.load_state_dict(one_state)
    assert len(list(back.next_epoch_itr(shuffle=True))) == 4
    fresh = make(2, 0)
    fresh.load_state_dict({"epoch": 3, "iterations_in_epoch": 0, "shuffle": True, "len": 8})
    assert fresh.next_epoch_idx == 3 and len(list(fresh.next_epoch_itr(shuffle=True))) == 8


def test_staged_logging_outputs_and_lazy_step_statistics():
    """CPU semantics of the early statistics path: nothing is staged for host tensors (the logging output comes back
    unchanged), and ``LazyStats`` answers single keys without materialising the rest."""
    import torch

    from unicore import metrics, utils
    from unicore.engine.update import LazyStats

    log = {"loss": torch.tensor(3.0), "bsz": 4}
    utils.stage_logging_output(log)                 # no CUDA scalars: a no-op
    assert utils.resolve_logging_output(log) is log
    with metrics.aggregate() as agg:
        metrics.log_scalar("loss", 2.5, 4, round=3)
        metrics.log_scalar("gnorm", torch.tensor(1.25), round=3)
        metrics.log_scalar("_hidden", 1.0)
    stats = LazyStats(agg, 4)
    assert stats["loss"] == 2.5 and stats._values is None
    assert stats.get("missing", "dflt") == "dflt" and "loss" in stats and "_hidden" not in stats
    assert stats["sample_size"] == 4
    full = dict(stats.items())
    assert full["loss"] == 2.5 and abs(float(full["gnorm"]) - 1.25) < 1e-6 and "_hidden" not in full
    assert stats._values is not None and stats["loss"] == 2.5


def test_norm_rows_are_16_byte_aligned():
    """The norm kernels read rows with 16-byte vector loads and bulk copies: a contiguous view at an odd element
    offset must reach them as an aligned copy, an aligned tensor as itself."""
    from unicore_b200.ops._native import aligned_rows

    for dtype in (torch.float32, torch.float16, torch.bfloat16):
        buf = torch.randn(3 * 5 * 64 + 1).to(dtype)
        for x in (buf[1:].view(3, 5, 64), buf[1:].view(15, 64)):
            assert x.is_contiguous() and x.data_ptr() % 16 != 0
            rows = aligned_rows(x)
            assert rows.shape == (15, 64) and rows.is_contiguous() and rows.data_ptr() % 16 == 0
            assert torch.equal(rows, x.reshape(15, 64))
        aligned = torch.randn(4, 3, 64).to(dtype)
        assert aligned.data_ptr() % 16 == 0 and aligned_rows(aligned).data_ptr() == aligned.data_ptr()
        strided = torch.randn(64, 30).to(dtype).t()  # not contiguous: copied
        assert torch.equal(aligned_rows(strided), strided) and aligned_rows(strided).is_contiguous()
