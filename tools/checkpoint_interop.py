#!/usr/bin/env python3
"""Checkpoint interchange with the reference implementation (SURVEY.md section 7.1-4), one process per side.

    # side A trains K updates, writes a checkpoint, trains M more and reports their losses
    python tools/checkpoint_interop.py --impl reference --init /tmp/i.pt --steps 3 --save /tmp/ck.pt --more 2
    # side B loads that checkpoint with ITS trainer (``Trainer.load_checkpoint``) and trains the same M updates
    python tools/checkpoint_interop.py --impl ours --init /tmp/i.pt --load /tmp/ck.pt --more 2

Both sides run the tiny BERT of ``tools/loss_parity.py`` on the CPU in bf16 with weight decay (two flat optimizer
groups), gradient clipping and an EMA - i.e. every part of the checkpoint schema is exercised: ``model``,
``optimizer_history`` (update count, LR-scheduler state), ``last_optimizer_state`` (flat fp32 Adam moments per group),
``ema``, ``extra_state.train_iterator``.  If the loaded state is complete and laid out identically, side B's next
losses equal side A's.  Prints one JSON line.
"""
import argparse
import json
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import bench  # noqa: E402


def register_task(impl):
    import torch

    from unicore.data import Dictionary, NestedDictionaryDataset, RightPadDataset, UnicoreDataset
    from unicore.tasks import TASK_REGISTRY, UnicoreTask, register_task

    if "interop_mlm" in TASK_REGISTRY:
        return

    class Rows(UnicoreDataset):
        def __init__(self, rows):
            self.rows = rows

        def __getitem__(self, i):
            return self.rows[i]

        def __len__(self):
            return len(self.rows)

    @register_task("interop_mlm")
    class InteropTask(UnicoreTask):
        def __init__(self, args, dictionary):
            super().__init__(args)
            self.dictionary = dictionary
            self.mask_idx = dictionary.add_symbol("[MASK]", is_special=True)

        @classmethod
        def setup_task(cls, args, **kwargs):
            d = Dictionary()
            for i in range(512):
                d.add_symbol({0: "[PAD]", 100: "[UNK]", 101: "[CLS]", 102: "[SEP]"}.get(i, "t{}".format(i)))
            return cls(args, d)

        def batches(self, n):
            d = self.dictionary
            return bench.make_batches(n, 4, 24, len(d), d.pad(), self.mask_idx,
                                      special=[d.pad(), d.unk(), d.bos(), d.eos(), self.mask_idx], seed=99)

        def load_dataset(self, split, **kwargs):
            src, tgt = [], []
            for b in self.batches(4):
                src += list(b["net_input"]["src_tokens"])
                tgt += list(b["target"])
            pad = self.dictionary.pad()
            self.datasets[split] = NestedDictionaryDataset(
                {"net_input": {"src_tokens": RightPadDataset(Rows(src), pad_idx=pad)},
                 "target": RightPadDataset(Rows(tgt), pad_idx=pad)})

    _ = torch


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--impl", choices=["ours", "reference"], required=True)
    ap.add_argument("--init", required=True)
    ap.add_argument("--steps", type=int, default=0, help="updates before --save")
    ap.add_argument("--save", default="")
    ap.add_argument("--load", default="")
    ap.add_argument("--more", type=int, default=2, help="updates after the save / load whose losses are reported")
    ap.add_argument("--precision", default="bf16", choices=["bf16", "fp32"])
    ap.add_argument("--embed-dim", type=int, default=64, help="encoder width (the FFN is twice as wide)")
    a = ap.parse_args()
    why = bench.setup_paths(a.impl)
    if why is not None:
        print(json.dumps({"impl": a.impl, "unavailable": why}))
        return 0
    import torch

    if a.impl == "reference":
        import bert  # noqa: F401
    else:
        import importlib

        sys.path.insert(0, os.path.join(REPO, "examples"))
        importlib.import_module("bert")
    from unicore import options, tasks
    from unicore.trainer import Trainer

    register_task(a.impl)
    flags = [
        "--task", "interop_mlm", "--loss", "masked_lm", "--arch", "bert_base", "--encoder-layers", "2",
        "--encoder-embed-dim", str(a.embed_dim), "--encoder-ffn-embed-dim", str(2 * a.embed_dim),
        "--encoder-attention-heads", "4",
        "--max-seq-len", "32", "--dropout", "0.0", "--emb-dropout", "0.0", "--attention-dropout", "0.0",
        "--activation-dropout", "0.0", "--pooler-dropout", "0.0", "--optimizer", "adam", "--adam-betas", "(0.9, 0.98)",
        "--adam-eps", "1e-6", "--weight-decay", "0.01", "--clip-norm", "1.0", "--lr-scheduler", "polynomial_decay",
        "--lr", "1e-3", "--warmup-updates", "2", "--total-num-update", "20", "--max-update", "20", "--batch-size", "4",
        "--seed", "1", "--num-workers", "0", "--log-format", "none", "--disable-validation", "--no-save",
        "--distributed-world-size", "1", "--cpu", "--ema-decay", "0.9", "--train-subset", "train",
    ]
    if a.precision == "bf16":
        flags.append("--bf16")
    args = options.parse_args_and_arch(options.get_training_parser(), input_args=flags)
    torch.manual_seed(args.seed)
    task = tasks.setup_task(args)
    model = task.build_model(args)
    if os.path.exists(a.init):
        model.load_state_dict(torch.load(a.init, map_location="cpu"))
    else:
        torch.save(model.state_dict(), a.init)
    trainer = Trainer(args, task, model, task.build_loss(args))
    report = {"impl": a.impl}
    if a.load:
        extra, epoch_itr = trainer.load_checkpoint(a.load)
        report["loaded_updates"] = trainer.get_num_updates()
        report["loaded_epoch"] = epoch_itr.epoch
        report["lr_after_load"] = float(trainer.get_lr())
    else:
        epoch_itr = trainer.get_train_iterator(epoch=1)
        trainer.init_total_train_steps(epoch_itr)
        trainer.lr_step(epoch_itr.epoch)
        epoch_itr.next_epoch_itr(shuffle=False)
    batches = task.batches(4)

    def run(n, first):
        out = []
        for i in range(first, first + n):
            res = trainer.train_step([batches[i % len(batches)]])
            out.append(float(res["loss"]))
        return out

    done = trainer.get_num_updates()
    if a.steps:
        report["losses_before"] = run(a.steps, done)
        done += a.steps
    if a.save:
        if hasattr(trainer, "consolidate_optimizer_state"):
            trainer.consolidate_optimizer_state()
        trainer.save_checkpoint(a.save, {"train_iterator": epoch_itr.state_dict(), "val_loss": None})
        ck = torch.load(a.save, map_location="cpu", weights_only=False)
        report["saved_keys"] = sorted(ck.keys())
        report["saved_opt_state_numel"] = [int(v["exp_avg"].numel()) for v in ck["last_optimizer_state"]["state"].values()]
    report["losses_after"] = run(a.more, done)
    ema = trainer.ema.state_dict()["params"]
    report["ema_checksum"] = float(sum(v.double().abs().sum() for v in ema.values() if torch.is_floating_point(v)))
    print(json.dumps(report))
    return 0


if __name__ == "__main__":
    sys.exit(main())
