"""Paged key / value caches on the GPU: the decode kernel (one split, the split heuristic, the ``chunk == 0`` path of
captured steps), the chunk and the packed-chunk KV-cache modes of the wgmma forward with a block table, the append
kernel and the block allocator kernels.

Checked: at D 8 / 64 / 96 / 128, fp16 / bf16, H_kv = H, H / 4, 1 and block sizes 128 / 256, with no bias, a shared bias
with a key mask and a per-batch bias, every output is ``torch.equal`` to the contiguous call on the cache gathered
through a shuffled table; the appended rows are bitwise in their blocks and every other pool row is untouched, with
NaN in every row no sequence holds (which reaches no output) and -1 entries past each sequence's rows; the allocator
kernels equal the PyTorch fallback bit for bit over a random series of reserve / release calls, pool exhaustion and more
entries than one scan pass included, and never hand out a block twice; greedy decoding with a paged decoder (eager,
captured, chunks, packed ragged steps, rewind and refill, reorder) gives bitwise the outputs and tokens of a contiguous
cache; a paged step does not synchronise; and the bindings reject malformed tables and pools."""
import pytest
import torch

pytestmark = pytest.mark.gpu

DTYPES = [torch.float16, torch.bfloat16]
DT_IDS = ["fp16", "bf16"]
HEAD_DIMS = [8, 64, 96, 128]
B, C = 4, 1024
LENS = [0, 127, 300, 900]   # the cached rows of each sequence
T_CHUNK, SIZES = 5, [0, 1, 17, 64]   # a padded chunk, and the T_b of a packed one
MAX_NEW = 64   # the most rows any call appends


def _ops():
    from unicore import ops

    assert ops.USE_NATIVE, "native kernels must be active on the GPU box"
    return ops


def _bits(t):
    return t.view(torch.int16)


def _paged_inputs(bs, H_kv, D, dtype, g):
    """Pools with the cached rows of LENS and NaN everywhere else, a shuffled table with -1 past each sequence's
    reach, and the contiguous caches gathered through it."""
    M = C // bs
    NB = B * M + 3
    k = (torch.randn(NB, bs, H_kv, D, device="cuda", generator=g) * 0.6).to(dtype)
    v = torch.randn(NB, bs, H_kv, D, device="cuda", generator=g).to(dtype)
    perm = torch.randperm(NB, device="cuda", generator=g)
    table = perm[:B * M].view(B, M).to(torch.int32)
    held = torch.zeros(NB, bs, dtype=torch.bool, device="cuda")
    for b, n in enumerate(LENS):
        reach = -(-(n + MAX_NEW) // bs)
        table[b, reach:] = -1
        for i in range(M):
            lo = i * bs
            if table[b, i] >= 0 and lo < n:
                held[table[b, i], :min(bs, n - lo)] = True
    k[~held] = float("nan")
    v[~held] = float("nan")
    return k, v, table


def _gather(pool, table):
    idx = table.long().clamp(min=0)
    return pool[idx].reshape(B, -1, *pool.shape[2:]).clone()


def _expected_pool(pool, table, starts, counts, rows):
    out = pool.clone()
    bs = pool.shape[1]
    for b in range(B):
        for i in range(counts[b]):
            r = starts[b] + i
            if r < C and table[b, r // bs] >= 0:
                out[table[b, r // bs], r % bs] = rows[b][i]
    return out


def _bias_kpm(case, T, H, dtype, g):
    if case == "plain":
        return None, None
    nb = 1 if case == "bias_shared_kpm" else B
    bias = torch.randn(nb, H, T, C, device="cuda", generator=g).to(dtype)
    kpm = None
    if case == "bias_shared_kpm":
        kpm = torch.rand(B, C, device="cuda", generator=g) < 0.2
    return bias, kpm


def _check(out, ref, k1, v1, kexp, vexp, what):
    assert torch.equal(out, ref), what
    assert bool(torch.isfinite(out).all()), what
    assert torch.equal(_bits(k1), _bits(kexp)), what
    assert torch.equal(_bits(v1), _bits(vexp)), what


@pytest.mark.parametrize("bs", [128, 256])
@pytest.mark.parametrize("kv_div", [1, 4, 0], ids=["mha", "gqa4", "mqa"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
@pytest.mark.parametrize("D", HEAD_DIMS)
def test_paged_calls_equal_contiguous_on_gathered(D, dtype, kv_div, bs):
    ops = _ops()
    nat = ops.native()
    H = 8
    H_kv = 1 if kv_div == 0 else H // kv_div
    g = torch.Generator(device="cuda").manual_seed(D * 7 + kv_div + bs)
    k, v, table = _paged_inputs(bs, H_kv, D, dtype, g)
    seqlens = torch.tensor(LENS, dtype=torch.int32, device="cuda")
    max_len = C - MAX_NEW
    scale = D ** -0.5
    for case in ["plain", "bias_shared_kpm", "bias_batch"]:
        # one-token decode: one split, the heuristic, and each (b, h) splitting its own length (captured steps)
        bias, kpm = _bias_kpm(case, 1, H, dtype, g)
        q = (torch.randn(B, 1, H, D, device="cuda", generator=g) * 0.6).to(dtype)
        kn, vn = ((torch.randn(B, 1, H_kv, D, device="cuda", generator=g) * 0.6).to(dtype) for _ in range(2))
        for splits, by_len in [(1, False), (0, False), (0, True), (7, True)]:
            k1, v1, kc, vc = k.clone(), v.clone(), _gather(k, table), _gather(v, table)
            ref = nat.fmha_decode(q, kc, vc, seqlens, max_len, kn, vn, bias, kpm, scale, num_splits=splits,
                                  split_by_length=by_len)
            out = nat.fmha_decode(q, k1, v1, seqlens, max_len, kn, vn, bias, kpm, scale, num_splits=splits,
                                  split_by_length=by_len, block_table=table)
            _check(out, ref, k1, v1, _expected_pool(k, table, LENS, [1] * B, kn),
                   _expected_pool(v, table, LENS, [1] * B, vn), (case, "decode", splits, by_len))
        # a padded chunk
        bias, kpm = _bias_kpm(case, T_CHUNK, H, dtype, g)
        q = (torch.randn(B, T_CHUNK, H, D, device="cuda", generator=g) * 0.6).to(dtype)
        kn, vn = ((torch.randn(B, T_CHUNK, H_kv, D, device="cuda", generator=g) * 0.6).to(dtype) for _ in range(2))
        k1, v1, kc, vc = k.clone(), v.clone(), _gather(k, table), _gather(v, table)
        ref = ops.attention_with_kv_cache(q, kc, vc, seqlens, max_len, kn, vn, bias, kpm, scale)
        out = ops.attention_with_kv_cache(q, k1, v1, seqlens, max_len, kn, vn, bias, kpm, scale, block_table=table)
        _check(out, ref, k1, v1, _expected_pool(k, table, LENS, [T_CHUNK] * B, kn),
               _expected_pool(v, table, LENS, [T_CHUNK] * B, vn), (case, "chunk"))
        # packed chunks of T_b in SIZES
        T = max(SIZES)
        bias, kpm = _bias_kpm(case, T, H, dtype, g)
        N = sum(SIZES)
        q = (torch.randn(N, H, D, device="cuda", generator=g) * 0.6).to(dtype)
        kn, vn = ((torch.randn(N, H_kv, D, device="cuda", generator=g) * 0.6).to(dtype) for _ in range(2))
        cu = torch.tensor([0] + torch.tensor(SIZES).cumsum(0).tolist(), dtype=torch.int32, device="cuda")
        k1, v1, kc, vc = k.clone(), v.clone(), _gather(k, table), _gather(v, table)
        ref = ops.attention_with_kv_cache_varlen(q, kc, vc, cu, T, seqlens, max_len, kn, vn, bias, kpm, scale)
        out = ops.attention_with_kv_cache_varlen(q, k1, v1, cu, T, seqlens, max_len, kn, vn, bias, kpm, scale,
                                                 block_table=table)
        starts = cu[:-1].tolist()
        rows_k = [kn[s:s + t] for s, t in zip(starts, SIZES)]
        rows_v = [vn[s:s + t] for s, t in zip(starts, SIZES)]
        _check(out, ref, k1, v1, _expected_pool(k, table, LENS, SIZES, rows_k),
               _expected_pool(v, table, LENS, SIZES, rows_v), (case, "packed"))


def test_append_skips_rows_without_a_block():
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(5)
    k = torch.randn(6, 128, 2, 64, device="cuda", generator=g).half()
    v = torch.randn(6, 128, 2, 64, device="cuda", generator=g).half()
    table = torch.tensor([[3, -1, 5], [0, 1, 9]], dtype=torch.int32, device="cuda")   # 9 is not a block of the pool
    kn = torch.randn(2, 300, 2, 64, device="cuda", generator=g).half()
    vn = torch.randn(2, 300, 2, 64, device="cuda", generator=g).half()
    seqlens = torch.tensor([40, 50], dtype=torch.int32, device="cuda")
    k1, v1 = k.clone(), v.clone()
    ops.kv_cache_append(kn, vn, k1, v1, seqlens, table)
    ke, ve = k.cpu(), v.cpu()   # the PyTorch fallback on the CPU
    ops.kv_cache_append(kn.cpu(), vn.cpu(), ke, ve, seqlens.cpu(), table.cpu())
    assert torch.equal(_bits(k1.cpu()), _bits(ke)) and torch.equal(_bits(v1.cpu()), _bits(ve))
    assert torch.equal(_bits(k1[[2, 4]]), _bits(k[[2, 4]]))   # blocks of no sequence are untouched
    assert torch.equal(_bits(k1[3, :40]), _bits(k[3, :40])) and torch.equal(_bits(k1[3, 40:]), _bits(kn[0, :88]))


# ---- the allocator ----------------------------------------------------------------------------------------------
def _state(Bn, M, NB, device):
    return [torch.full((Bn, M), -1, dtype=torch.int32, device=device),
            torch.arange(NB - 1, -1, -1, dtype=torch.int32, device=device),
            torch.tensor([NB], dtype=torch.int32, device=device), torch.zeros(1, dtype=torch.int32, device=device)]


@pytest.mark.parametrize("Bn,M,NB", [(5, 4, 12), (37, 9, 200), (300, 8, 1500)])
def test_allocator_kernels_equal_the_fallback(Bn, M, NB):
    ops = _ops()
    bs = 128
    g = torch.Generator().manual_seed(Bn)
    gpu, cpu = _state(Bn, M, NB, "cuda"), _state(Bn, M, NB, "cpu")
    for step in range(40):
        lengths = torch.randint(-10, M * bs + 50, (Bn,), generator=g, dtype=torch.int32)
        lengths[torch.rand(Bn, generator=g) < 0.3] = 0
        if step % 3 == 2:
            ops.kv_blocks_release(gpu[0], gpu[1], gpu[2], lengths.cuda(), bs)
            ops.kv_blocks_release(cpu[0], cpu[1], cpu[2], lengths, bs)
        else:
            ops.kv_blocks_reserve(*gpu[:3], lengths.cuda(), bs, gpu[3])
            ops.kv_blocks_reserve(*cpu[:3], lengths, bs, cpu[3])
        for a, b in zip(gpu, cpu):
            assert torch.equal(a.cpu(), b), step
        held = gpu[0][gpu[0] >= 0]
        assert held.numel() == held.unique().numel(), step   # no block is held twice
        count = int(gpu[2].item())
        assert held.numel() + count == NB, step   # every block is held or on the stack
        assert torch.equal(torch.cat([held, gpu[1][:count]]).sort().values,
                           torch.arange(NB, dtype=torch.int32, device="cuda")), step
    assert int(cpu[3].item()) == 1   # the random lengths exhaust every pool at some point


def test_allocator_in_a_graph():
    ops = _ops()
    table, free, count, flag = _state(3, 4, 12, "cuda")
    lengths = torch.tensor([200, 0, 513], dtype=torch.int32, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            ops.kv_blocks_reserve(table, free, count, lengths, 128, flag)
            ops.kv_blocks_release(table, free, count, lengths - 100, 128)
    torch.cuda.current_stream().wait_stream(side)
    graph.replay()
    cpu = _state(3, 4, 12, "cpu")
    ops.kv_blocks_reserve(*cpu[:3], lengths.cpu(), 128, cpu[3])
    ops.kv_blocks_release(*cpu[:3], lengths.cpu() - 100, 128)
    for a, b in zip([table, free, count, flag], cpu):
        assert torch.equal(a.cpu(), b)


# ---- the decoder ------------------------------------------------------------------------------------------------
E, VOCAB, CAP, BSZ = 256, 97, 512, 4


def _decoder(dtype):
    from unicore.modules import TransformerDecoder

    torch.manual_seed(0)
    m = TransformerDecoder(decoder_layers=2, embed_dim=E, ffn_embed_dim=2 * E, attention_heads=4,
                           max_seq_len=CAP).cuda().eval()
    with torch.no_grad():
        for p in m.parameters():
            p.add_(torch.randn_like(p) * 0.02)
    return m.to(dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_IDS)
def test_greedy_decoding_paged_equals_contiguous(dtype):
    _ops()
    m = _decoder(dtype)
    g = torch.Generator(device="cuda").manual_seed(11)
    lens = [130, 20, 1, 77]
    L, Le = max(lens), 9
    prompt = torch.randn(BSZ, L, E, device="cuda", generator=g).to(dtype)
    pad = torch.ones(BSZ, L, dtype=torch.bool, device="cuda")
    for b, n in enumerate(lens):
        pad[b, :n] = False
    enc = torch.randn(BSZ, Le, E, device="cuda", generator=g).to(dtype)
    enc_pad = torch.zeros(BSZ, Le, dtype=torch.bool, device="cuda")
    enc_pad[2, 6:] = True
    table = (torch.randn(VOCAB, E, device="cuda", generator=g) * 0.5).to(dtype)
    contig = m.new_cache(BSZ, CAP)
    paged = m.new_cache(BSZ, CAP, block_size=128, num_blocks=9)   # 16 blocks would hold every sequence at capacity
    caches = [contig, paged]

    def both(fn):
        outs = [fn(c) for c in caches]
        assert torch.equal(_bits(outs[0]), _bits(outs[1]))
        return outs[0]

    def tokens(y):
        return table[(y.float() @ table.float().t()).argmax(-1)]

    with torch.no_grad():
        y = both(lambda c: m(prompt, encoder_out=enc, padding_mask=pad, encoder_padding_mask=enc_pad, cache=c))
        y = y[torch.arange(BSZ), torch.tensor(lens) - 1][:, None]
        for _ in range(6):   # eager one-token steps
            y = both(lambda c: m(tokens(y), encoder_padding_mask=enc_pad, cache=c))
        steps = [m.capture_step(c, encoder_padding_mask=enc_pad) for c in caches]
        for _ in range(10):   # captured one-token steps
            emb = tokens(y)
            outs = [s(emb).clone() for s in steps]
            assert torch.equal(_bits(outs[0]), _bits(outs[1]))
            y = outs[0]
        y = both(lambda c: m(torch.cat([tokens(y)] * 3, 1), encoder_padding_mask=enc_pad, cache=c))[:, -1:]
        # sequence 1 finishes: its slot is emptied (its blocks go back) and re-prompted in a packed ragged step
        for c in caches:
            c.rewind(torch.tensor([0, 10_000, 2, 0], dtype=torch.int32, device="cuda"))
        emb = torch.cat([tokens(y)[0], prompt[1, :40], tokens(y)[3].expand(3, E)])
        cu = torch.tensor([0, 1, 41, 41, 44], dtype=torch.int32, device="cuda")   # T_b = 1, 40, 0, 3
        both(lambda c: m(emb, encoder_padding_mask=enc_pad, cu_seqlens=cu, max_seqlen=40, cache=c))
        for c in caches:
            c.rewind(1)
        for _ in range(3):
            emb = tokens(y)
            outs = [s(emb).clone() for s in steps]
            assert torch.equal(_bits(outs[0]), _bits(outs[1]))
            y = outs[0]
        # beam-style reorder in place (the captured step keeps its graph), then to a smaller batch
        idx = torch.tensor([3, 0, 1, 1], device="cuda")
        for c in caches:
            c.reorder(idx)
        emb = tokens(y)[idx]
        outs = [s(emb, encoder_padding_mask=enc_pad[idx]).clone() for s in steps]
        assert torch.equal(_bits(outs[0]), _bits(outs[1]))
        assert [s.captures for s in steps] == [1, 1]
        idx2 = torch.tensor([2, 0], device="cuda")
        for c in caches:
            c.reorder(idx2)
        both(lambda c: m(tokens(outs[0])[idx2], encoder_padding_mask=enc_pad[idx][idx2], cache=c))
    assert torch.equal(contig.seqlens, paged.seqlens)
    assert not paged.overflowed()


def test_paged_step_does_not_synchronise():
    _ops()
    m = _decoder(torch.float16)
    cache = m.new_cache(2, CAP, block_size=128, num_blocks=4)
    x = torch.randn(2, 100, E, device="cuda").half()
    with torch.no_grad():
        m(x, cache=cache)
        step = torch.randn(2, 1, E, device="cuda").half()
        chunk = torch.randn(2, 40, E, device="cuda").half()
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            y = m(step, cache=cache)
            z = m(chunk, cache=cache)   # crosses into a second block: reserves on the device
            cache.rewind(30)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    assert bool(torch.isfinite(y).all()) and bool(torch.isfinite(z).all())
    assert cache.free_blocks() == 2 and not cache.overflowed()


# ---- binding rejections -----------------------------------------------------------------------------------------
def _valid_decode():
    q = torch.randn(2, 1, 2, 64, device="cuda").half()
    pool = torch.randn(5, 128, 2, 64, device="cuda").half()
    lens = torch.tensor([3, 130], dtype=torch.int32, device="cuda")
    table = torch.tensor([[0, 1], [2, 3]], dtype=torch.int32, device="cuda")
    return q, pool, lens, table


def test_bindings_reject_malformed_tables_and_pools():
    nat = _ops().native()
    q, pool, lens, table = _valid_decode()
    nat.fmha_decode(q, pool, pool.clone(), lens, 200, None, None, None, None, 0.125, block_table=table)
    torch.cuda.synchronize()
    bad_tables = {"must be int32": table.long(), "must be a CUDA": table.cpu(), "must have sizes": table[:1],
                  "must be contiguous": table.t().contiguous().t(), "M >= 1": table[:, :0]}
    for msg, t in bad_tables.items():
        with pytest.raises(RuntimeError, match=msg):
            nat.fmha_decode(q, pool, pool.clone(), lens, 200, None, None, None, None, 0.125, block_table=t)
    small = torch.randn(5, 64, 2, 64, device="cuda").half()
    with pytest.raises(RuntimeError, match="multiple of 128"):
        nat.fmha_decode(q, small, small.clone(), lens, 100, None, None, None, None, 0.125, block_table=table)
    with pytest.raises(RuntimeError, match="same shape"):
        nat.fmha_decode(q, pool, pool[:4].clone(), lens, 200, None, None, None, None, 0.125, block_table=table)
    with pytest.raises(RuntimeError, match="v_cache"):
        nat.fmha_decode(q, pool, pool[:, :, :, :32].clone(), lens, 200, None, None, None, None, 0.125,
                        block_table=table)
    with pytest.raises(RuntimeError, match="capacity"):   # C = 2 * 128
        nat.fmha_decode(q, pool, pool.clone(), lens, 257, None, None, None, None, 0.125, block_table=table)
    qc = torch.randn(2, 4, 2, 64, device="cuda").half()
    kn = torch.randn(2, 4, 2, 64, device="cuda").half()
    with pytest.raises(RuntimeError, match="block_table must have sizes"):
        nat.kvcache.fmha_kvcache_fwd(qc, pool, pool.clone(), lens, 200, kn, kn.clone(), None, None, 0.125,
                                     block_table=table[:1])
    with pytest.raises(RuntimeError, match="multiple of 128"):
        nat.kvcache.fmha_kvcache_fwd(qc, small, small.clone(), lens, 100, kn, kn.clone(), None, None, 0.125,
                                     block_table=table)
    qp = torch.randn(6, 2, 64, device="cuda").half()
    cu = torch.tensor([0, 2, 6], dtype=torch.int32, device="cuda")
    with pytest.raises(RuntimeError, match="block_table must be int32"):
        nat.kvcache.fmha_kvcache_varlen_fwd(qp, pool, pool.clone(), cu, 4, lens, 200, qp.clone(), qp.clone(), None,
                                            None, 0.125, block_table=table.long())
    tbl, free, count, flag = _state(2, 2, 4, "cuda")
    for msg, args in {"free_count must have 1 elements": (tbl, free, free, lens, 128, flag),
                      "lengths must have sizes": (tbl, free, count, lens[:1], 128, flag),
                      "block_table must be int32": (tbl.long(), free, count, lens, 128, flag),
                      "block_size must be positive": (tbl, free, count, lens, 0, flag)}.items():
        with pytest.raises(RuntimeError, match=msg):
            nat.kvcache.kv_blocks_reserve(*args)
    with pytest.raises(RuntimeError, match="free_list must have"):
        nat.kvcache.kv_blocks_release(tbl, free[:0], count, lens, 128)
    with pytest.raises(RuntimeError, match="lengths must be a CUDA"):
        nat.kvcache.kv_blocks_release(tbl, free, count, lens.cpu(), 128)
