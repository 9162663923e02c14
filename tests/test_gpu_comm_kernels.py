"""The peer-memory collectives (``csrc/comm/allreduce.cu``) and the fused optimizer tail (``csrc/comm/fused_step.cu``)
on one GPU, against exact and fp64 references.

The bindings take raw device addresses, so ordinary CUDA tensors stand in for the symmetric buffers of W ranks.  Rank
r's collective runs ALONE: before the call the test plants the other W - 1 ranks' arrival tags in rank r's own flag
buffer (``uint32 [slot][sender]``, stride W) at exactly the slots that collective uses - the handshake slot and one data
slot per CTA of an all-reduce, the statistics slot of the statistics reduction - and fills the other ranks' data.  No
two ranks ever run concurrently.  After every call all four error words must be 0, rank r's flag buffer must be all
zero, and every peer's flag buffer must hold r's tag at [slot][r] for exactly the used slots (then it is cleared).  A
harness that planted the wrong slots would see the kernel give up after ~10 s and report a timeout, not hang.

All-reduce results are compared bitwise with the exact reference of the kernels: the ranks summed in rank order in fp32
from 0.0f, times fp32(scale), rounded once to the output type.  The statistics sums are compared bitwise with the
rank-order fp64 sum.  The fused tail (W = 1: its one peer slot is used three times per launch) is driven through
``FusedTail`` and checked against an fp64 re-derivation of the norm, the multiplier and the Adam update (with the
per-element bounds of tests/test_gpu_optim_kernels.py), and bitwise against ``multi_tensor_adam`` on the same inputs.
"""
import math

import numpy as np
import pytest
import torch

import test_gpu_optim_kernels as ok

pytestmark = pytest.mark.gpu

E32 = 2.0 ** -24
SLOTS = 64                 # SYMM_MAX_BLOCKS flag slots per rank
HANDSHAKE, STATS = SLOTS - 1, SLOTS - 3     # (slot SLOTS - 2 is the fused tail's)
MAX_DATA = SLOTS - 3       # data CTAs of one collective
THREADS = 512
XROW = 65                  # doubles per sender row of an exchange buffer: {sum of squares, 64 statistics}
ALGO = {"auto": 0, "oneshot": 1, "twoshot": 2, "nvls": 3}
DT = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}
BITS = {torch.float32: torch.int32, torch.float16: torch.int16, torch.bfloat16: torch.int16}
CANARY = {torch.float32: 0x7FC01234, torch.float16: 0x7E5A, torch.bfloat16: 0x7FA5}   # NaN payloads
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
DT_IDS = ["fp32", "fp16", "bf16"]
TAG_BUCKET, TAG_STATS = 0x100, 0x7002


def _nat():
    from unicore import ops

    assert ops.USE_NATIVE, "native kernels must be active on the GPU box"
    return ops.native()


def _f32(v):
    return float(np.float32(v))


def _same_bits(a, b):
    return torch.equal(a.view(BITS.get(a.dtype, torch.int64)), b.view(BITS.get(b.dtype, torch.int64)))


# ---- the peer emulator ---------------------------------------------------------------------------------------------
class Peers:
    """The flag buffers of W ranks and a fresh error channel."""

    def __init__(self, world):
        self.world = world
        self.flags = [torch.zeros(SLOTS * world, dtype=torch.int32, device="cuda") for _ in range(world)]
        self.ptrs = [f.data_ptr() for f in self.flags]
        self.err_host, self.err_dev = _nat().symm_error_channel()

    def plant(self, r, slots, tag):
        """The arrival tags of every rank but r at `slots` of rank r's flag buffer."""
        idx = [s * self.world + p for s in slots for p in range(self.world) if p != r]
        if idx:
            self.flags[r][torch.tensor(idx, device="cuda")] = tag if tag != 0 else 1

    def check_and_clear(self, r, slots, tag):
        torch.cuda.synchronize()
        assert self.err_host.tolist() == [0, 0, 0, 0], "error channel: {}".format(self.err_host.tolist())
        assert not bool(self.flags[r].any()), "rank {} took every planted tag".format(r)
        want = torch.zeros(SLOTS * self.world, dtype=torch.int32, device="cuda")
        want[torch.tensor([s * self.world + r for s in slots], device="cuda")] = tag if tag != 0 else 1
        for p in range(self.world):
            if p != r:
                assert torch.equal(self.flags[p], want), "rank {}'s tags in rank {}'s flags".format(r, p)
                self.flags[p].zero_()


# ---- all-reduce / reduce-scatter ----------------------------------------------------------------------------------
def plan(kind, nvec, blocks):
    """(algorithm, CTAs) of launch_allreduce's host rules for a range of nvec vectors, with no multicast address."""
    scatter = kind == "rs"
    algo = ALGO["auto"] if scatter else ALGO[kind]
    if algo == ALGO["auto"]:
        algo = ALGO["oneshot"] if nvec * 16 <= 256 * 1024 else ALGO["twoshot"]
    if scatter and algo == ALGO["oneshot"]:
        algo = ALGO["twoshot"]
    if algo == ALGO["nvls"]:
        algo = ALGO["twoshot"]
    one_shot_blocks = -(-nvec // THREADS)
    if algo == ALGO["oneshot"] and one_shot_blocks > MAX_DATA:
        algo = ALGO["twoshot"]
    if algo == ALGO["oneshot"]:
        return algo, one_shot_blocks
    return algo, min(24 if blocks <= 0 else blocks, MAX_DATA)


def _sweep(world, blocks):
    """Vectors one grid sweep of the two-shot kernel covers (W * kU = 16 vectors in flight per thread)."""
    wt = 2 if world <= 2 else 4 if world <= 4 else 8
    return blocks * THREADS * (16 // wt)


def sizes(world):
    """(vectors, blocks): one vector; fewer vectors than ranks; around one CTA; the one-shot limit and one past it;
    two-shot ranges of several grid sweeps per rank at 1 and 61 CTAs; 100 CTAs requested (clamped to 61)."""
    out = [(1, 0), (2, 0), (511, 0), (512, 0), (513, 0), (MAX_DATA * THREADS, 0), (MAX_DATA * THREADS + 1, 0)]
    out += [(int(2.5 * world * _sweep(world, 1)) + 3, 1), (int(2.5 * world * _sweep(world, MAX_DATA)) + 5, MAX_DATA),
            (100 * THREADS * world + 7, 100)]
    return out


def _ranks(world):
    return [0, 3, 7] if world == 8 else list(range(world))


def _slice(nvec, world, r):
    """Rank r's vectors of the range (per = ceil(n / W), the formula of SymmComm.slice_of)."""
    per = -(-nvec // world)
    return min(nvec, per * r), min(nvec, per * (r + 1))


def _run_reduce(peers, kind, dtype, r, nvec, blocks, scale, tag, seed):
    nat, world = _nat(), peers.world
    epv = 128 // torch.finfo(dtype).bits
    pre, post = 3, 2  # canary vectors on both sides: the range starts 48 bytes into every buffer
    gen = torch.Generator(device="cuda").manual_seed(seed)
    bufs = []
    for p in range(world):
        b = torch.empty((pre + nvec + post) * epv, dtype=dtype, device="cuda")
        b.view(BITS[dtype]).fill_(CANARY[dtype])
        b[pre * epv:(pre + nvec) * epv] = (torch.randn(nvec * epv, device="cuda", generator=gen) * (1 + p)).to(dtype)
        bufs.append(b)
    before = [b.clone() for b in bufs]
    algo, nb = plan(kind, nvec, blocks)
    slots = [HANDSHAKE] + list(range(nb))
    sq = torch.full((SLOTS,), -7.0, device="cuda")
    peers.plant(r, slots, tag)
    args = ([b.data_ptr() for b in bufs], peers.ptrs, 0, r, pre * 16, nvec * 16, DT[dtype], scale)
    if kind == "rs":
        nat.symm_reduce_scatter(*args, blocks, sq.data_ptr(), peers.err_dev, tag)
    else:
        nat.symm_allreduce(*args, ALGO[kind], blocks, sq.data_ptr(), peers.err_dev, tag)
    peers.check_and_clear(r, slots, tag)

    # the exact reference: rank order from 0.0f in fp32, one fp32 product, one rounding
    rng = slice(pre * epv, (pre + nvec) * epv)
    acc = torch.zeros(nvec * epv, dtype=torch.float32, device="cuda")
    for p in range(world):
        acc = acc + before[p][rng].float()
    acc = acc * torch.tensor(_f32(scale), dtype=torch.float32, device="cuda")
    red = acc.to(dtype)
    lo, hi = _slice(nvec, world, r)
    own = slice((pre + lo) * epv, (pre + hi) * epv)
    want = [b.clone() for b in before]
    if algo == ALGO["oneshot"]:
        want[r][rng] = red
    elif kind == "rs":
        want[r][own] = red[lo * epv:hi * epv]
    else:
        for w in want:
            w[own] = red[lo * epv:hi * epv]
    what = "{} W={} rank {} {} vectors {} CTAs ({})".format(kind, world, r, nvec, nb,
                                                           "one-shot" if algo == ALGO["oneshot"] else "two-shot")
    for p in range(world):
        assert _same_bits(bufs[p], want[p]), "{}: buffer of rank {}".format(what, p)

    # the CTAs' sums of squares of rank r's slice of the scaled fp32 values; the slots past the grid untouched
    ref = acc[lo * epv:hi * epv].double().pow(2).sum().item()
    got = sq[:nb].double().sum().item()
    chain = epv * -(-(hi - lo) // (nb * THREADS)) + 12   # a thread's additions, then the CTA's tree
    assert abs(got - ref) <= 2 * chain * E32 * ref + 1e-30, (what, got, ref)
    assert bool((sq[nb:] == -7.0).all()), what
    return algo


@pytest.mark.parametrize("world", [1, 2, 3, 4, 5, 8], ids=lambda w: "W{}".format(w))
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("kind", ["oneshot", "twoshot", "auto", "nvls", "rs"])
def test_allreduce_against_exact_reference(kind, dtype, world):
    """symm_allreduce (one-shot, two-shot, auto, NVLS requested without a multicast address) and symm_reduce_scatter,
    rank by rank: one-shot leaves rank r's whole range reduced in its own buffer, two-shot rank r's slice in EVERY
    buffer, reduce-scatter rank r's slice in its own buffer only; nothing else changes, canaries included."""
    peers = Peers(world)
    ran = set()
    scales = [1.0, 1.0 / world, 0.37]
    for r in _ranks(world):
        for i, (nvec, blocks) in enumerate(sizes(world)):
            tag = 0 if (r == 0 and i == 0) else TAG_BUCKET + i
            algo = _run_reduce(peers, kind, dtype, r, nvec, blocks, scales[i % 3], tag, seed=1000 * world + 10 * r + i)
            ran.add("one-shot" if algo == ALGO["oneshot"] else "two-shot")
    print("{} {} W={} ranks {}: ran {}".format(kind, dtype, world, _ranks(world), sorted(ran)))
    if kind in ("twoshot", "nvls", "rs"):
        assert ran == {"two-shot"}
    else:
        assert ran == {"one-shot", "two-shot"}


# ---- statistics reduction ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("parity", [0, 1])
@pytest.mark.parametrize("k", [1, 7, 64])
@pytest.mark.parametrize("world", [1, 2, 8], ids=lambda w: "W{}".format(w))
def test_stats_allreduce(world, k, parity):
    """Rank r's row lands at [parity][r] of every peer's exchange buffer, the other parity half is untouched, and dst
    is the rank-order fp64 sum bitwise."""
    nat = _nat()
    peers = Peers(world)
    gen = torch.Generator(device="cuda").manual_seed(17 * world + k + parity)
    for r in _ranks(world):
        xchg = [torch.randn(2 * world * XROW, dtype=torch.float64, device="cuda", generator=gen) * 1e3
                for _ in range(world)]
        before = [x.clone() for x in xchg]
        src = torch.randn(k, dtype=torch.float64, device="cuda", generator=gen) * 1e5
        dst = torch.full((k,), math.nan, dtype=torch.float64, device="cuda")
        peers.plant(r, [STATS], TAG_STATS)
        nat.symm_stats_allreduce([x.data_ptr() for x in xchg], peers.ptrs, peers.err_dev, r, TAG_STATS, src, dst,
                                 parity)
        peers.check_and_clear(r, [STATS], TAG_STATS)
        row = lambda p: slice((parity * world + p) * XROW + 1, (parity * world + p) * XROW + 1 + k)  # noqa: E731
        for p in range(world):
            want = before[p].clone()
            want[row(r)] = src
            assert _same_bits(xchg[p], want), "W={} rank {}: exchange buffer of rank {}".format(world, r, p)
        rows = [src.tolist() if p == r else before[r][row(p)].tolist() for p in range(world)]
        ref = []
        for j in range(k):
            s = 0.0
            for p in range(world):
                s += rows[p][j]
            ref.append(s)
        assert _same_bits(dst, torch.tensor(ref, dtype=torch.float64, device="cuda")), (world, r, k, parity)


# ---- the fused optimizer tail at W = 1 -------------------------------------------------------------------------------
class _Buf:
    def __init__(self, t):
        self.tensor, self.ptrs, self.multicast_ptr = t, [t.data_ptr()], 0


class OneRankComm:
    """What FusedTail needs of a communicator, for one rank on ordinary CUDA tensors.  The kernel always runs as rank 0
    of 1; `slice_of` may cut the buckets as rank `own` of `of` ranks, so that the tail owns only slices of them."""

    def __init__(self, own=0, of=1):
        nat = _nat()
        self.native, self.device, self.rank, self.world = nat, torch.device("cuda"), 0, 1
        self.max_blocks, self.max_stats = int(nat.SYMM_MAX_BLOCKS), int(nat.SYMM_MAX_STATS)
        self.own, self.of = own, of
        self.flags = _Buf(torch.zeros(SLOTS, dtype=torch.int32, device="cuda"))
        self.xchg_tail = _Buf(torch.zeros(2 * XROW, dtype=torch.float64, device="cuda"))
        self.err_host, self.err_dev = nat.symm_error_channel()

    def slice_of(self, lo, hi, elem_size, rank=None):
        epv = 16 // elem_size
        nvec = (hi - lo) // epv
        per = -(-nvec // self.of)
        return lo + min(nvec, per * self.own) * epv, lo + min(nvec, per * (self.own + 1)) * epv

    def check(self):
        torch.cuda.synchronize()
        assert self.err_host.tolist() == [0, 0, 0, 0], self.err_host.tolist()
        assert not bool(self.flags.tensor.any())


def philox4x32_10(seed, offset, ctr):
    """Philox4x32 with 10 rounds, vectorised over uint64 counters; the word order of csrc/common.cuh."""
    m32 = np.uint64(0xFFFFFFFF)
    k0, k1 = np.uint64(seed & 0xFFFFFFFF), np.uint64((seed >> 32) & 0xFFFFFFFF)
    c0, c1 = ctr & m32, ctr >> np.uint64(32)
    c2 = np.full_like(ctr, offset & 0xFFFFFFFF)
    c3 = np.full_like(ctr, (offset >> 32) & 0xFFFFFFFF)
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c0
        p1 = np.uint64(0xCD9E8D57) * c2
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & m32, p1 >> np.uint64(32), p1 & m32
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
        k0 = (k0 + np.uint64(0x9E3779B9)) & m32
        k1 = (k1 + np.uint64(0xBB67AE85)) & m32
    return c0, c1, c2, c3


def bf16_sr(master, idx, seed, offset):
    """bf16 bits of fp32 `master` at absolute arena elements `idx` by the tail's stochastic rounding: Philox call
    (seed, offset, i >> 3), word (i & 7) >> 1, its low half for even i and its high half for odd i; the 16 random bits
    are added to the fp32 bits (not to inf / nan) and the sum truncated."""
    i = idx.cpu().numpy().astype(np.uint64)
    words = np.stack(philox4x32_10(seed, offset, i >> np.uint64(3)), axis=-1)
    w = np.take_along_axis(words, ((i & np.uint64(7)) >> np.uint64(1)).astype(np.int64)[:, None], axis=1)[:, 0]
    rnd = np.where((i & np.uint64(1)) == 1, w >> np.uint64(16), w & np.uint64(0xFFFF))
    bits = master.cpu().numpy().view(np.uint32).astype(np.uint64)
    finite = (bits & np.uint64(0x7F800000)) != np.uint64(0x7F800000)
    bits = np.where(finite, (bits + rnd) & np.uint64(0xFFFFFFFF), bits)
    return torch.from_numpy((bits >> np.uint64(16)).astype(np.uint16).view(np.int16)).cuda()


class TailCase:
    """Arenas, compact state and a FusedTail over them; `update()` runs one update and checks it against fp64."""

    def __init__(self, dtype, numels, bucket_bytes, own=0, of=1, stats=0, ema="off", blocks=0, sr=False, seed=0):
        self.dtype, self.numels, self.sr = dtype, numels, sr
        self.esz = torch.finfo(dtype).bits // 8
        self.comm = OneRankComm(own, of)
        self.full = of == 1
        self.gen = torch.Generator(device="cuda").manual_seed(seed)
        self.grads = [_Buf(torch.zeros(n, dtype=dtype, device="cuda")) for n in numels]
        self.params = [_Buf(self._randn(n).to(dtype)) for n in numels]
        from unicore_b200.parallel.fused_tail import FusedTail

        self.tail = FusedTail(self.comm, self.grads, self.params, bucket_bytes, seed=0x1234_5678_9ABC + seed)
        if blocks > 0:
            self.tail.blocks = blocks
        t = self.tail
        self.masters = [self._randn(n) for n in t.compact_numels]
        self.exp_avgs = [self._randn(n) * 0.1 for n in t.compact_numels]
        self.exp_avg_sqs = [torch.rand(n, device="cuda", generator=self.gen) * 0.1 for n in t.compact_numels]
        # the EMA arenas: full length, or a view that ends before the padded arena (its storage covers the padding)
        self.ema_base = [self._randn(n) for n in numels] if ema != "off" else None
        self.emas = None
        if ema == "full":
            self.emas = list(self.ema_base)
        elif ema == "short":
            self.emas = [e[:n - 3] for e, n in zip(self.ema_base, numels)]
        self.nstats = stats
        # per group: the element indices this rank owns in compact order
        self.owned = []
        for g in range(len(numels)):
            parts = [torch.arange(lo, hi, device="cuda") for lo, hi in t.owned_ranges(g)]
            self.owned.append(torch.cat(parts) if parts else torch.zeros(0, dtype=torch.int64, device="cuda"))
        self.step = 0

    def _randn(self, n):
        return torch.randn(n, device="cuda", generator=self.gen)

    def hyper(self, g):
        return ok._hyper(g + 3 * self.step)

    def update(self, pending, factor=0.125, max_norm=0.0, clip="none", clip_eps=0.0, denom_index=-1, denom_zero=False,
               bad=None, ema_decay=0.999):
        """One update.  `clip`: "below" / "above" sets max_norm to half / twice the fp64 norm.  `bad` = (bucket,
        value) puts a non-finite gradient into that bucket."""
        nat, t = _nat(), self.tail
        self.step += 1
        for g, b in enumerate(self.grads):
            b.tensor.copy_((self._randn(b.tensor.numel()) * 2).to(self.dtype))
        if bad is not None:
            bk = t.buckets[bad[0]]
            self.grads[bk.group].tensor[bk.own_lo + 3] = bad[1]
        stats_src = None
        if self.nstats:
            stats_src = torch.rand(self.nstats, dtype=torch.float64, device="cuda", generator=self.gen) * 100 + 1
            if 0 <= denom_index < self.nstats:
                stats_src[denom_index] = 0.0 if denom_zero else 37.0
        grads0 = [b.tensor.clone() for b in self.grads]
        params0 = [b.tensor.clone() for b in self.params]
        masters0 = [m.clone() for m in self.masters]
        m0 = [m.clone() for m in self.exp_avgs]
        v0 = [v.clone() for v in self.exp_avg_sqs]
        ema0 = [e.clone() for e in self.ema_base] if self.ema_base is not None else None

        # fp64: the sum of squares over the owned slices, the multiplier, the norm and the clip coefficient
        total = sum(grads0[g][self.owned[g]].double().pow(2).sum().item() for g in range(len(self.numels)))
        denom = 1.0
        if stats_src is not None and 0 <= denom_index < self.nstats and stats_src[denom_index].item() > 0:
            denom = stats_src[denom_index].item()
        mul = _f32(factor) / denom
        norm = math.sqrt(total) * mul
        if clip == "below":
            max_norm = 0.5 * norm
        elif clip == "above":
            max_norm = 2.0 * norm
        coef = max_norm / (norm + clip_eps) if (max_norm > 0 and norm > max_norm) else 1.0
        mult = mul * coef

        # the buckets that are not pending: their bucket kernel (full ownership only) before the tail
        for b in t.buckets:
            if b.index not in pending:
                assert self.full, "rank r of W > 1: every bucket is pending"
                nat.symm_reduce_scatter(self.grads[b.group].ptrs, self.comm.flags.ptrs, 0, 0, b.lo * self.esz,
                                        (b.hi - b.lo) * self.esz, DT[self.dtype], 1.0, 0,
                                        t.sq_slots(b.index).data_ptr(), self.comm.err_dev, TAG_BUCKET + b.index)
        from unicore_b200.parallel.fused_tail import adam_hyper

        hypers = []
        for g in range(len(self.numels)):
            h = self.hyper(g)
            hypers.append(adam_hyper(h["lr"], h["beta1"], h["beta2"], h["eps"], h["step"], h["bias_correction"],
                                     h["weight_decay"]))
        state = t.launch(masters=self.masters, exp_avgs=self.exp_avgs, exp_avg_sqs=self.exp_avg_sqs, hypers=hypers,
                         pending=list(pending), factor=factor, max_norm=max_norm, clip_eps=clip_eps, emas=self.emas,
                         ema_decay=ema_decay, stats_src=stats_src, denom_index=denom_index,
                         stochastic_rounding=self.sr)
        self.comm.check()
        st = state.tolist()
        what = "update {} pending {}".format(self.step, sorted(pending))

        # every whole bucket of the gradient arena is zero; the statistics are summed even on overflow
        for b in self.grads:
            assert not bool(b.tensor.any()), what + ": gradient arena not zeroed"
        if stats_src is not None:
            assert _same_bits(t.stats_dst[:self.nstats], stats_src), what
        if bad is not None:
            assert st[2] == 1.0, what + ": overflow not flagged"
            for a, b in [(self.masters, masters0), (self.exp_avgs, m0), (self.exp_avg_sqs, v0),
                         ([p.tensor for p in self.params], params0)] + ([(self.ema_base, ema0)] if ema0 else []):
                for x, y in zip(a, b):
                    assert _same_bits(x, y), what + ": state changed on overflow"
            return st
        assert st[2] == 0.0, what

        # the state vector within the fp32 error of its computation
        owned_vecs = sum(int(o.numel()) for o in self.owned) // (16 // self.esz)
        chain = (16 // self.esz) * -(-owned_vecs // (min(t.blocks, 24) * THREADS)) + 24
        sq_rel = chain * E32
        assert abs(st[3] - total) <= (2 * sq_rel + E32) * total, (what, st[3], total)
        norm_rel = sq_rel / 2 + 4 * E32
        assert abs(st[0] - norm) <= 2 * norm_rel * norm, (what, st[0], norm)
        mult_rel = 2 * (norm_rel + 4 * E32) if coef != 1.0 else E32
        assert abs(st[1] - mult) <= mult_rel * mult, (what, st[1], mult)

        # compact master / moments and EMA within the bounds of the one-GPU optimizer; parameters = round(master)
        for g in range(len(self.numels)):
            idx = self.owned[g]
            w = dict(self.hyper(g), p=masters0[g], m=m0[g], v=v0[g], g=grads0[g][idx])
            if ema0 is not None:
                w["ema"] = ema0[g][idx]
            ref = ok.adam_reference(w, mult, mult_rel + E32, ema_decay if ema0 is not None else None)
            got = dict(p=self.masters[g], m=self.exp_avgs[g], v=self.exp_avg_sqs[g])
            if ema0 is not None:
                got["ema"] = self.ema_base[g][idx]
            for k, x in got.items():
                r, comp = ref[k]
                ok._assert_within(x, r, E32 * (r.abs() + comp) + comp + ok._tiny(torch.float32),
                                  "{} group {} {}".format(what, g, k))
            p = self.params[g].tensor
            if self.sr:
                assert _same_bits(p[idx], bf16_sr(self.masters[g], idx, t.seed, t.calls).view(self.dtype)), \
                    what + ": stochastic rounding"
            else:
                assert _same_bits(p[idx], self.masters[g].to(self.dtype)), what + ": parameters != round(master)"
            outside = torch.ones(p.numel(), dtype=torch.bool, device="cuda")
            outside[idx] = False
            assert _same_bits(p[outside], params0[g][outside]), what + ": parameters outside the shard changed"
            if ema0 is not None:
                assert _same_bits(self.ema_base[g][outside], ema0[g][outside]), what + ": EMA outside the shard"
        return st


def _every(n, k, phase=0):
    return {i for i in range(n) if i % k == phase}


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
def test_tail_full_ownership_pending_subsets(dtype):
    """Rank 0 of 1 owns every bucket.  Updates with no bucket pending, all pending, and mixtures whose buckets were
    reduced by their bucket kernel in the update before (their slots must have been cleared); 1 to 4 groups (one only
    8 elements long), 0 or 64 statistics, every kind of denominator, clipping off / not reached / reached, EMA on and
    off (a short EMA view), 1, 3 and all CTAs."""
    cases = [
        dict(numels=[4096, 1304, 8], bucket_bytes=1024, stats=0, ema="off", blocks=1),
        dict(numels=[2048, 520], bucket_bytes=512, stats=64, ema="short", blocks=3),
        dict(numels=[3000, 808, 8, 1600], bucket_bytes=800, stats=64, ema="full", blocks=0),
        dict(numels=[40000], bucket_bytes=4096, stats=64, ema="full", blocks=3),
    ]
    for ci, c in enumerate(cases):
        case = TailCase(dtype, seed=ci, **c)
        n = len(case.tail.buckets)
        case.update(set(), max_norm=0.0)
        case.update(set(range(n)), clip="below", clip_eps=1e-6, denom_index=5 if c["stats"] else -1)
        case.update(_every(n, 3), clip="above", denom_index=7 if c["stats"] else -1, denom_zero=True)
        case.update(_every(n, 3, 1), clip="below", denom_index=70)   # out of range: no denominator
        case.update({n - 1}, clip="below", clip_eps=1e-6, denom_index=0)
        print("tail {} groups {} buckets {} CTAs {}: 5 updates".format(dtype, len(c["numels"]), n, case.tail.blocks))


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
def test_tail_rank_one_of_three(dtype):
    """The tail owns rank 1 of 3's slices of every bucket, all pending: slices start inside their buckets and end before
    them, compact offsets are not the arena offsets, the rest of every bucket is zeroed but not updated."""
    for ci, (numels, bucket_bytes, stats, ema, blocks) in enumerate([
            ([2400, 96, 8], 1024, 64, "short", 3), ([1000, 5000], 2048, 0, "off", 1), ([8, 16, 24, 4096], 512, 64,
                                                                                      "full", 0)]):
        case = TailCase(dtype, numels, bucket_bytes, own=1, of=3, stats=stats, ema=ema, blocks=blocks, seed=10 + ci)
        n = len(case.tail.buckets)
        assert any(b.own_lo > b.lo and b.own_hi < b.hi for b in case.tail.buckets)
        for k, clip in enumerate(["below", "none", "above"]):
            case.update(set(range(n)), clip=clip, clip_eps=1e-6, denom_index=[3, -1, 64][k])
    print("tail {} rank 1 of 3: 3 plans x 3 updates".format(dtype))


def test_tail_overflow():
    """An inf in a pending bucket, then a NaN in a bucket reduced by its bucket kernel: the overflow flag is set, the
    master, the moments, the EMA and the parameters are bitwise unchanged, the gradients are zeroed and the statistics
    still summed; the next update is a normal one."""
    for dtype in (torch.float16, torch.bfloat16):
        case = TailCase(dtype, [2048, 808], 1024, stats=64, ema="full", blocks=3, seed=20)
        n = len(case.tail.buckets)
        case.update(_every(n, 2))
        case.update(_every(n, 2), bad=(0, math.inf), denom_index=2)
        case.update(_every(n, 2), bad=(1, math.nan), denom_index=2)
        case.update(_every(n, 2), clip="below", denom_index=2)


def test_tail_stochastic_rounding():
    """bf16 parameters by stochastic rounding of the new master, bitwise the host Philox4x32-10 keyed (seed, call count,
    element >> 3), over three updates (the call count moves the stream)."""
    for own, of in ((0, 1), (1, 3)):
        case = TailCase(torch.bfloat16, [4096, 1304, 8], 1024, own=own, of=of, stats=64, ema="full", sr=True, seed=30)
        n = len(case.tail.buckets)
        for k in range(3):
            case.update(set(range(n)) if of > 1 else _every(n, 2, k % 2), clip="below", denom_index=1)


def test_tail_64_buckets():
    """A plan of exactly 64 buckets with the last one pending: the pending mask is 2**63."""
    for dtype in (torch.float16, torch.bfloat16):
        case = TailCase(dtype, [64 * 64], 64 * 2, stats=64, ema="full", blocks=3, seed=40)
        assert len(case.tail.buckets) == 64
        for _ in range(3):
            case.update({63}, clip="below", denom_index=0)
        case.update(set(range(64)), clip="above")


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["fp16", "bf16"])
def test_tail_trains_like_multi_tensor_adam(dtype):
    """Under full ownership the tail's update is the one-GPU optimizer's bit for bit (csrc/optim/adam_math.cuh): the
    same fp32 multiplier as multi_tensor_adam's host scale, and the same master, moments, parameters and EMA."""
    case = TailCase(dtype, [3000, 808, 8], 1024, stats=64, ema="full", blocks=3, seed=50)
    t = case.tail
    n = len(t.buckets)
    for k in range(3):
        masters = [m.clone() for m in case.masters]
        m0, v0 = [m.clone() for m in case.exp_avgs], [v.clone() for v in case.exp_avg_sqs]
        ema0 = [e.clone() for e in case.ema_base]
        step = case.step + 1
        # the gradients this update will draw: replay the generator
        state_gen = case.gen.get_state()
        grads = [(case._randn(b.tensor.numel()) * 2).to(dtype) for b in case.grads]
        case.gen.set_state(state_gen)
        st = case.update(_every(n, 2, k % 2), clip="below" if k != 1 else "none", clip_eps=1e-6, denom_index=4)
        grad_scale = 1.0 / st[1]
        assert _f32(1.0 / grad_scale) == st[1], "multi_tensor_adam's fp32 multiplier must equal the tail's"
        work = []
        for b in t.buckets:
            g = b.group
            sl = slice(b.compact_off, b.compact_off + b.hi - b.lo)
            h = ok._hyper(g + 3 * step)
            work.append(dict(h, p=masters[g][sl].clone(), g=grads[g][b.lo:b.hi].clone(), m=m0[g][sl].clone(),
                             v=v0[g][sl].clone(), p_half=torch.zeros(b.hi - b.lo, dtype=dtype, device="cuda"),
                             ema=ema0[g][b.lo:b.hi].clone()))
        ok._ops().fused_adam(work, grad_scale=grad_scale, zero_grad=False, ema_decay=0.999)
        for b, w in zip(t.buckets, work):
            g = b.group
            sl = slice(b.compact_off, b.compact_off + b.hi - b.lo)
            for name, mine, theirs in (("master", case.masters[g][sl], w["p"]),
                                       ("exp_avg", case.exp_avgs[g][sl], w["m"]),
                                       ("exp_avg_sq", case.exp_avg_sqs[g][sl], w["v"]),
                                       ("parameters", case.params[g].tensor[b.lo:b.hi], w["p_half"]),
                                       ("ema", case.ema_base[g][b.lo:b.hi], w["ema"])):
                assert _same_bits(mine, theirs), "update {} bucket {}: {} differs from multi_tensor_adam".format(
                    k, b.index, name)
