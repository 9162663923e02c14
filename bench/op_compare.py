#!/usr/bin/env python3
"""Per-op comparison (BASELINE.md B4): our sm_90a kernels vs the reference's own CUDA extensions built for
sm_90 (``baseline/_ref_ext``, see ``baseline/build_ref_ext.sh``) vs PyTorch natives - same shapes, same script.

    python bench/op_compare.py --impl ours      >  gpurun_out/op_ours.jsonl
    python bench/op_compare.py --impl reference >  gpurun_out/op_ref.jsonl     # imports baseline/_ref + _ref_ext ONLY
    python bench/op_compare.py --impl torch     >  gpurun_out/op_torch.jsonl
    python bench/op_compare.py --merge gpurun_out/op_ours.jsonl gpurun_out/op_ref.jsonl gpurun_out/op_torch.jsonl

Both frameworks expose the same public API (``unicore.modules.LayerNorm`` / ``RMSNorm`` / ``softmax_dropout``,
``unicore.optim.fused_adam``, ``unicore.utils.multi_tensor_total_norm`` / ``fp32_to_bf16_sr``), so each arm is the same
code with a different ``sys.path``.  Every measurement: the op on rotating operands (working set > the 50 MB L2)
captured ONCE in a CUDA graph (so neither arm pays Python / allocator time), replayed after warm-up, timed with CUDA
events.  forward is timed under ``no_grad``; backward = (forward + backward) - forward.  One JSON line per op with the
minimum bytes the op has to move, GB/s, the fraction of the HBM peak (MEASURED_PEAKS.json if present, else the H100 data sheet) and the SM clock /
throttle record sampled while it ran.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import threading

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def peaks():
    try:
        with open(os.path.join(REPO, "MEASURED_PEAKS.json")) as f:
            return float(json.load(f)["hbm_gbs"])
    except Exception:  # noqa: BLE001
        return 3350.0  # H100 SXM data sheet: 3.35 TB/s of HBM3


class Clocks:
    FIELDS = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
              "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
              "clocks_event_reasons.sw_power_cap")

    def __init__(self):
        self.lines, self.proc = [], None
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "--query-gpu=" + self.FIELDS, "--format=csv,noheader,nounits",
                                          "-lms", "50", "-i", "0"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL,
                                         text=True)
            threading.Thread(target=self._pump, daemon=True).start()
        except Exception:  # noqa: BLE001
            self.proc = None

    def _pump(self):
        for line in self.proc.stdout:
            self.lines.append(line.strip())

    def mark(self):
        return len(self.lines)

    def since(self, mark):
        sm, smax, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for line in self.lines[mark:]:
            parts = [p.strip() for p in line.split(",")]
            if len(parts) < 7:
                continue
            try:
                sm.append(float(parts[0]))
                smax.append(float(parts[1]))
            except ValueError:
                continue
            for n, v in zip(names, parts[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(n)
        return {"sm_mhz": statistics.median(sm) if sm else None, "sm_max_mhz": max(smax) if smax else None,
                "reasons": sorted(reasons)}

    def stop(self):
        if self.proc is not None:
            self.proc.terminate()


def setup(impl):
    if impl == "reference":
        ref = os.path.join(REPO, "baseline", "_ref")
        ext = os.path.join(REPO, "baseline", "_ref_ext")
        for p in (os.path.join(REPO, "baseline", "stubs"), ref, ext):
            sys.path.insert(0, p)
        sys.path[:] = [p for p in sys.path if os.path.abspath(p or ".") != REPO]
    else:
        sys.path.insert(0, REPO)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--impl", default="ours", choices=["ours", "reference", "torch"])
    ap.add_argument("--merge", nargs="*", default=None)
    ap.add_argument("--only", default="", help="comma-separated op-name prefixes")
    ap.add_argument("--reps", type=int, default=5, help="graph replays per measurement")
    a = ap.parse_args()
    if a.merge is not None:
        return merge(a.merge)
    setup("ours" if a.impl == "torch" else a.impl)

    import torch
    import torch.nn.functional as F

    import unicore
    from unicore import utils as uutils
    from unicore.modules import LayerNorm, softmax_dropout
    try:
        from unicore.modules import RMSNorm
    except ImportError:
        from unicore.modules.rms_norm import RMSNorm

    loaded = sorted({os.path.basename(l.split()[-1]) for l in open("/proc/self/maps")
                     if ("unicore_fused" in l or "unicore_b200/_C" in l) and l.rstrip().endswith(".so")})
    dev = torch.device("cuda")
    hbm = peaks()
    clocks = Clocks()
    only = [s for s in a.only.split(",") if s]

    def want(name):
        return not only or any(name.startswith(s) for s in only)

    def measure(fns, inner):
        """fns: closures over distinct operand sets; returns us per call."""
        seq = [fns[i % len(fns)] for i in range(inner)]
        for f in fns:
            f()
        torch.cuda.synchronize()
        graph, used_graph = torch.cuda.CUDAGraph(), True
        try:
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for f in fns:
                    f()
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            with torch.cuda.graph(graph):
                for f in seq:
                    f()
        except Exception:  # noqa: BLE001  (an op that cannot be captured: time it eagerly)
            used_graph = False
            torch.cuda.synchronize()
        run = graph.replay if used_graph else (lambda: [f() for f in seq])
        run()
        torch.cuda.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        best = None
        for _ in range(a.reps):
            s.record()
            run()
            e.record()
            torch.cuda.synchronize()
            t = s.elapsed_time(e) * 1e3 / inner
            best = t if best is None else min(best, t)
        return best, used_graph

    def report(name, us, nbytes, graph, mark, note=None):
        rec = {"op": name, "impl": a.impl, "us": round(us, 2), "MB": round(nbytes / 1e6, 2),
               "GBps": round(nbytes / us / 1e3, 1), "frac_of_hbm_peak": round(nbytes / us / 1e3 / hbm, 3),
               "graph": graph, "clocks": clocks.since(mark), "native_so": loaded}
        if note:
            rec["note"] = note
        print(json.dumps(rec), flush=True)

    def fwd_bwd(name, make_module, make_inputs, bytes_fwd, bytes_bwd, nset, inner):
        """times forward (no_grad) and forward+backward of ``y = module(x)``; reports fwd and bwd separately."""
        if not want(name):
            return
        mod = make_module()
        sets = [make_inputs() for _ in range(nset)]

        def f_only(x, dy):
            with torch.no_grad():
                return mod(x)

        def f_b(x, dy):
            x.grad = None
            y = mod(x)
            y.backward(dy)

        mark = clocks.mark()
        t_f, g1 = measure([lambda s=s: f_only(*s) for s in sets], inner)
        report(name + "_fwd", t_f, bytes_fwd, g1, mark)
        mark = clocks.mark()
        t_fb, g2 = measure([lambda s=s: f_b(*s) for s in sets], inner)
        report(name + "_bwd", max(t_fb - t_f, 1e-3), bytes_bwd, g1 and g2, mark, note="(fwd+bwd) - fwd")

    dt = torch.float16
    es = 2
    total = 16384 * 768  # elements per operand: the BERT-base activation (25 MB in fp16)

    # ---- LayerNorm / RMSNorm --------------------------------------------------------------------------------------
    for D in (64, 512, 768, 1024):
        rows = total // D
        nset = 8  # 8 x (x, dy) x 25 MB + outputs: ~ 600 MB rotating, far beyond L2

        def mk_inputs(rows=rows, D=D):
            return (torch.randn(rows, D, device=dev, dtype=dt, requires_grad=True), torch.randn(rows, D, device=dev, dtype=dt))

        if a.impl == "torch":
            class TorchLN(torch.nn.Module):
                def __init__(self, D):
                    super().__init__()
                    self.w = torch.nn.Parameter(torch.ones(D, device=dev, dtype=dt))
                    self.b = torch.nn.Parameter(torch.zeros(D, device=dev, dtype=dt))

                def forward(self, x):
                    return F.layer_norm(x, (x.shape[-1],), self.w, self.b, 1e-5)

            class TorchRMS(torch.nn.Module):
                def __init__(self, D):
                    super().__init__()
                    self.w = torch.nn.Parameter(torch.ones(D, device=dev, dtype=dt))

                def forward(self, x):
                    return F.rms_norm(x, (x.shape[-1],), self.w, 1e-5)

            mk_ln, mk_rms = (lambda D=D: TorchLN(D)), (lambda D=D: TorchRMS(D))
        else:
            mk_ln = lambda D=D: LayerNorm(D).to(dev).to(dt)  # noqa: E731
            mk_rms = lambda D=D: RMSNorm(D).to(dev).to(dt)  # noqa: E731
        n = rows * D
        fwd_bwd("layernorm_D%d" % D, mk_ln, mk_inputs, 2 * n * es, 3 * n * es, nset, 16)
        fwd_bwd("rmsnorm_D%d" % D, mk_rms, mk_inputs, 2 * n * es, 3 * n * es, nset, 16)

    # ---- softmax_dropout ------------------------------------------------------------------------------------------
    for shape in ((32 * 12, 512, 512), (32 * 64, 256, 256)):
        for p in (0.0, 0.1):
            name = "softmax_dropout_%dx%dx%d_p%.1f" % (shape[0], shape[1], shape[2], p)
            if not want(name):
                continue
            n = shape[0] * shape[1] * shape[2]

            class SD(torch.nn.Module):
                def forward(self, x, p=p):
                    if a.impl == "torch":
                        return F.dropout(torch.softmax(x, dim=-1), p, True)
                    return softmax_dropout(x, p, True, inplace=False)

            def mk_inputs(shape=shape):
                return (torch.randn(*shape, device=dev, dtype=dt, requires_grad=True), torch.randn(*shape, device=dev, dtype=dt))

            # non-inplace contract: read x, write y (+ clone inside the reference); backward reads dy, y(/mask) writes dx
            fwd_bwd(name, SD, mk_inputs, 2 * n * es, 3 * n * es, 2, 4)

    # ---- optimizer tail ------------------------------------------------------------------------------------------------
    for nparam, tag in ((109_513_146, "109.5M"), (335_172_922, "335.2M")):
        nparam = (nparam + 7) // 8 * 8
        name = "fused_adam_" + tag
        if want(name):
            p32 = torch.randn(nparam, device=dev) * 0.02
            if a.impl == "ours":
                from unicore import ops

                g16 = (torch.randn(nparam, device=dev) * 1e-2).to(dt)
                p16 = p32.to(dt)
                m, v = torch.zeros_like(p32), torch.zeros_like(p32)
                work = [dict(p=p32, g=g16, m=m, v=v, p_half=p16, lr=1e-4, beta1=0.9, beta2=0.98, eps=1e-6, step=1,
                             bias_correction=True, weight_decay=0.01)]
                fn = lambda: ops.fused_adam(work, grad_scale=4.0, zero_grad=False, stochastic_rounding=False)  # noqa: E731
                nbytes = nparam * (4 * 3 * 2 + 2 + 2)
                note = "ONE kernel: 16-bit grad in, unscale, Adam on fp32 p/m/v, 16-bit weight out (30 B/param incl. zeroing off)"
            elif a.impl == "reference":
                from unicore.optim.fused_adam import FusedAdam

                prm = torch.nn.Parameter(p32)
                prm.grad = torch.randn(nparam, device=dev) * 1e-2
                opt = FusedAdam([prm], lr=1e-4, betas=(0.9, 0.98), eps=1e-6, weight_decay=0.01)
                fn = lambda: opt.step(scale=4.0)  # noqa: E731
                nbytes = nparam * (4 * 3 * 2 + 4)
                note = "reference adam kernel alone (fp32 grad in; its fp16 copy passes are separate, see adam_tail)"
            else:
                prm = torch.nn.Parameter(p32)
                prm.grad = torch.randn(nparam, device=dev) * 1e-2
                opt = torch.optim.Adam([prm], lr=1e-4, betas=(0.9, 0.98), eps=1e-6, weight_decay=0.01, fused=True)
                fn = opt.step
                nbytes = nparam * (4 * 3 * 2 + 4)
                note = "torch.optim.Adam(fused=True)"
            mark = clocks.mark()
            t, g = measure([fn], 3)
            report(name, t, nbytes, g, mark, note)
            del fn
            torch.cuda.empty_cache()
        # the whole mixed-precision tail: grad norm + unscale/clip + update + 16-bit weights + zeroed grads
        name = "adam_tail_" + tag
        if want(name):
            g16 = (torch.randn(nparam, device=dev) * 1e-2).to(dt)
            p16 = (torch.randn(nparam, device=dev) * 0.02).to(dt)
            p32 = p16.float()
            if a.impl == "ours":
                from unicore import ops

                m, v = torch.zeros_like(p32), torch.zeros_like(p32)
                work = [dict(p=p32, g=g16, m=m, v=v, p_half=p16, lr=1e-4, beta1=0.9, beta2=0.98, eps=1e-6, step=1,
                             bias_correction=True, weight_decay=0.01)]

                def fn():
                    norm = uutils.multi_tensor_total_norm([g16])
                    scale = torch.clamp(norm * 0.25, min=1.0) * 4.0  # clip to 1.0 after the 1/4 unscale, on device
                    ops.fused_adam(work, grad_scale=scale, zero_grad=True, stochastic_rounding=False)
            else:
                prm = torch.nn.Parameter(p32)
                prm.grad = torch.zeros_like(p32)
                if a.impl == "reference":
                    from unicore.optim.fused_adam import FusedAdam

                    opt = FusedAdam([prm], lr=1e-4, betas=(0.9, 0.98), eps=1e-6, weight_decay=0.01)
                else:
                    opt = torch.optim.Adam([prm], lr=1e-4, betas=(0.9, 0.98), eps=1e-6, weight_decay=0.01, fused=True)

                def fn():  # the reference FP16Optimizer sequence (fp16_optimizer.py:180-291) on flat buffers
                    prm.grad.copy_(g16)                                       # _sync_fp16_grads_to_fp32
                    norm = uutils.multi_tensor_total_norm([prm.grad]) if a.impl == "reference" else torch.norm(prm.grad)
                    scale = torch.clamp(norm * 0.25, min=1.0) * 4.0
                    if a.impl == "reference":
                        opt.step(scale=float(4.0))                            # (host scalar in the reference)
                    else:
                        prm.grad.div_(scale)
                        opt.step()
                    p16.copy_(prm.data)                                       # _sync_fp32_params_to_fp16
                    g16.zero_()
                    prm.grad.zero_()
            mark = clocks.mark()
            t, g = measure([fn], 3)
            report(name, t, nparam * 36, g, mark, "bytes = 36 B/param (the fused minimum); the unfused sequence moves ~86")
            del fn
            torch.cuda.empty_cache()

    # ---- multi-tensor L2 norm -----------------------------------------------------------------------------------
    name = "l2norm_109.5M_fp16"
    if want(name):
        n = 109_513_152
        gs = [(torch.randn(n, device=dev) * 1e-2).to(dt) for _ in range(2)]
        # the reference groups tensors per dtype and needs > 1 tensor to take its kernel: split into 12 chunks
        chunks = [list(g.split(n // 12)) for g in gs]
        if a.impl == "torch":
            fns = [lambda c=c: torch.norm(torch.stack([torch.norm(t, p=2, dtype=torch.float32) for t in c])) for c in chunks]
        else:
            fns = [lambda c=c: uutils.multi_tensor_total_norm(c) for c in chunks]
        mark = clocks.mark()
        t, g = measure(fns, 4)
        report(name, t, n * es, g, mark)
        del gs, chunks
        torch.cuda.empty_cache()

    # ---- fp32 -> bf16 stochastic rounding ------------------------------------------------------------------------
    name = "fp32_to_bf16_sr_109.5M"
    if want(name) and a.impl != "torch":
        n = 109_513_152
        srcs = [torch.randn(n, device=dev) for _ in range(2)]
        dst = torch.empty(n, device=dev, dtype=torch.bfloat16)
        fns = [lambda s=s: uutils.fp32_to_bf16_sr(s, dst) for s in srcs]
        mark = clocks.mark()
        t, g = measure(fns, 4)
        report(name, t, n * 6, g, mark)

    # ---- copy roofline, same harness --------------------------------------------------------------------------------
    if want("copy"):
        srcs = [torch.empty(256 << 20, device=dev, dtype=torch.uint8) for _ in range(2)]
        dst = torch.empty(256 << 20, device=dev, dtype=torch.uint8)
        mark = clocks.mark()
        t, g = measure([lambda s=s: dst.copy_(s) for s in srcs], 4)
        report("copy_256MB", t, 2 * (256 << 20), g, mark)
    clocks.stop()
    return 0


def merge(paths):
    rows = {}
    for p in paths:
        for line in open(p):
            line = line.strip()
            if not line.startswith("{"):
                continue
            r = json.loads(line)
            rows.setdefault(r["op"], {})[r["impl"]] = r
    print("| op | ours us (GB/s, % of copy peak) | reference ext (sm_90 build) us | torch native us | ours / reference |")
    print("|---|---|---|---|---|")
    for op, by in rows.items():
        def cell(k):
            r = by.get(k)
            return "-" if r is None else "%.1f (%.0f, %.0f %%)" % (r["us"], r["GBps"], 100 * r["frac_of_hbm_peak"])
        ratio = "-"
        if "ours" in by and "reference" in by:
            ratio = "%.2fx" % (by["reference"]["us"] / by["ours"]["us"])
        print("| %s | %s | %s | %s | %s |" % (op, cell("ours"), cell("reference"), cell("torch"), ratio))
    return 0


if __name__ == "__main__":
    sys.exit(main())
