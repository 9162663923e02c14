"""Paged key / value caches on the CPU: the cache references with a shuffled block table equal the contiguous
references on the cache gathered through it (one token, a chunk, packed chunks), with the appended rows in their blocks
and the rows of missing blocks skipped; the allocator fallbacks give exact tables, stacks, counts and flags through a
scripted series of calls, pool exhaustion included; a decoder with a pool smaller than B x capacity gives the outputs
of a contiguous cache through a prefill, one-token steps, chunks, packed ragged steps, rewinds, an emptied and refilled
slot and reorders; and ``new_cache`` rejects bad arguments."""
import pytest
import torch

from unicore import ops
from unicore.modules import TransformerDecoder

F64 = torch.float64
BS = 128


def _cu(lens):
    return torch.tensor([0] + torch.tensor(lens).cumsum(0).tolist(), dtype=torch.int32)


def _pool_and_table(g, B, M, NB, heads, D, missing=()):
    """A pool of NB blocks filled with noise, and a table naming distinct shuffled blocks (-1 at ``missing``)."""
    k, v = (torch.randn(NB, BS, heads, D, generator=g, dtype=F64) for _ in range(2))
    perm = torch.randperm(NB, generator=g)[:B * M].to(torch.int32).view(B, M)
    for b, i in missing:
        perm[b, i] = -1
    return k, v, perm


def _gathered(pool, table):
    idx = table.long().clamp(min=0)
    return pool[idx].reshape(table.shape[0], table.shape[1] * BS, *pool.shape[2:])


def _expect_rows(pool, table, seqlens_start, counts, new_rows):
    """The pool after an append of ``new_rows[b][i]`` at rows ``start_b + i`` through the table."""
    out = pool.clone()
    for b in range(table.shape[0]):
        for i in range(counts[b]):
            r = int(seqlens_start[b]) + i
            if r >= table.shape[1] * BS:
                continue
            blk = int(table[b, r // BS])
            if blk >= 0:
                out[blk, r % BS] = new_rows[b][i]
    return out


@pytest.mark.parametrize("T", [1, 3])
def test_reference_equals_contiguous_on_gathered(T):
    g = torch.Generator().manual_seed(T)
    B, M, NB, H, H_kv, D = 3, 2, 8, 4, 2, 8
    k, v, table = _pool_and_table(g, B, M, NB, H_kv, D, missing=[(2, 1)])
    q = torch.randn(B, T, H, D, generator=g, dtype=F64)
    kn, vn = (torch.randn(B, T, H_kv, D, generator=g, dtype=F64) for _ in range(2))
    bias = torch.randn(B, H, T, 2 * BS, generator=g, dtype=F64)
    kpm = torch.rand(B, 2 * BS, generator=g) < 0.2
    # sequence 2 writes across into its missing second block (T = 3): those rows are skipped
    seqlens = torch.tensor([5, 130, 127], dtype=torch.int32)
    kc, vc = _gathered(k, table), _gathered(v, table)
    ref = ops.attention_with_kv_cache_reference(q, kc, vc, seqlens, 200, kn, vn, bias, kpm)
    k1, v1 = k.clone(), v.clone()
    out = ops.attention_with_kv_cache(q, k1, v1, seqlens, 200, kn, vn, bias, kpm, block_table=table)
    assert torch.equal(out, ref)
    assert torch.equal(k1, _expect_rows(k, table, seqlens, [T] * B, kn))
    assert torch.equal(v1, _expect_rows(v, table, seqlens, [T] * B, vn))


def test_reference_varlen_equals_contiguous_on_gathered():
    g = torch.Generator().manual_seed(7)
    B, M, NB, H, H_kv, D = 4, 2, 9, 4, 1, 8
    k, v, table = _pool_and_table(g, B, M, NB, H_kv, D, missing=[(3, 1)])
    sizes = [0, 1, 4, 3]
    N, T = sum(sizes) + 1, max(sizes)
    q = torch.randn(N, H, D, generator=g, dtype=F64)
    kn, vn = (torch.randn(N, H_kv, D, generator=g, dtype=F64) for _ in range(2))
    seqlens = torch.tensor([9, 60, 126, 127], dtype=torch.int32)
    cu = _cu(sizes)
    kc, vc = _gathered(k, table), _gathered(v, table)
    ref = ops.attention_with_kv_cache_varlen_reference(q, kc, vc, cu, T, seqlens, 200, kn, vn)
    k1, v1 = k.clone(), v.clone()
    out = ops.attention_with_kv_cache_varlen(q, k1, v1, cu, T, seqlens, 200, kn, vn, block_table=table)
    assert torch.equal(out, ref)
    starts = cu[:-1].tolist()
    rows_k = [kn[s:s + t] for s, t in zip(starts, sizes)]
    rows_v = [vn[s:s + t] for s, t in zip(starts, sizes)]
    assert torch.equal(k1, _expect_rows(k, table, seqlens, sizes, rows_k))
    assert torch.equal(v1, _expect_rows(v, table, seqlens, sizes, rows_v))


def test_kv_cache_append_through_table():
    g = torch.Generator().manual_seed(3)
    k, v, table = _pool_and_table(g, 2, 2, 5, 2, 8, missing=[(1, 1)])
    kn, vn = (torch.randn(2, 140, 2, 8, generator=g, dtype=F64) for _ in range(2))
    k1, v1 = k.clone(), v.clone()
    ops.kv_cache_append(kn, vn, k1, v1, torch.zeros(2, dtype=torch.int32), table)
    assert torch.equal(k1, _expect_rows(k, table, [0, 0], [140, 140], kn))
    assert torch.equal(v1, _expect_rows(v, table, [0, 0], [140, 140], vn))


def test_paged_argument_errors():
    q = torch.zeros(2, 1, 4, 8, dtype=F64)
    pool = torch.zeros(4, 64, 4, 8, dtype=F64)
    with pytest.raises(ValueError, match="multiple of 128"):
        ops.attention_with_kv_cache(q, pool, pool, block_table=torch.zeros(2, 1, dtype=torch.int32))
    pool = torch.zeros(4, 128, 4, 8, dtype=F64)
    with pytest.raises(ValueError, match="block_table"):
        ops.attention_with_kv_cache(q, pool, pool, block_table=torch.zeros(3, 1, dtype=torch.int32))
    with pytest.raises(ValueError, match="capacity"):
        ops.attention_with_kv_cache(q, pool, pool, torch.zeros(2, dtype=torch.int32), 128,
                                    torch.zeros(2, 1, 4, 8, dtype=F64), torch.zeros(2, 1, 4, 8, dtype=F64),
                                    block_table=torch.zeros(2, 1, dtype=torch.int32))


# ---- the allocator ---------------------------------------------------------------------------------------------
def _alloc(B, M, NB):
    return (torch.full((B, M), -1, dtype=torch.int32), torch.arange(NB - 1, -1, -1, dtype=torch.int32),
            torch.tensor([NB], dtype=torch.int32), torch.zeros(1, dtype=torch.int32))


def test_allocator_scripted_series():
    table, free, count, flag = _alloc(3, 3, 5)
    lens = lambda *x: torch.tensor(x, dtype=torch.int32)   # noqa: E731

    ops.kv_blocks_reserve(table, free, count, lens(130, 0, 1), BS, flag)
    assert table.tolist() == [[0, 1, -1], [-1, -1, -1], [2, -1, -1]]
    assert count.item() == 2 and flag.item() == 0

    # sequence 1 asks for 3 blocks (300 clamps to C = 384); 2 are left: its third entry stays -1, the flag is set
    ops.kv_blocks_reserve(table, free, count, lens(130, 300, 1), BS, flag)
    assert table.tolist() == [[0, 1, -1], [3, 4, -1], [2, -1, -1]]
    assert count.item() == 0 and flag.item() == 1

    # releases in (b, i) order: block 1 (sequence 0, entry 1), then block 2 (sequence 2)
    ops.kv_blocks_release(table, free, count, lens(1, 129, 0), BS)
    assert table.tolist() == [[0, -1, -1], [3, 4, -1], [-1, -1, -1]]
    assert count.item() == 2 and free[:2].tolist() == [1, 2]

    ops.kv_blocks_reserve(table, free, count, lens(0, 129, 200), BS, flag)   # lengths below the held blocks keep them
    assert table.tolist() == [[0, -1, -1], [3, 4, -1], [2, 1, -1]]
    assert count.item() == 0 and flag.item() == 1

    ops.kv_blocks_release(table, free, count, lens(0, -5, 0), BS)
    assert table.tolist() == [[-1] * 3] * 3
    assert count.item() == 5 and free.tolist() == [0, 3, 4, 2, 1]

    # the flag is never cleared by the allocator; blocks come off the top again
    ops.kv_blocks_reserve(table, free, count, lens(1, 1, 1), BS, flag)
    assert table.tolist() == [[1, -1, -1], [2, -1, -1], [4, -1, -1]]
    assert count.item() == 2 and flag.item() == 1


def test_allocator_drops_foreign_entries():
    table, free, count, flag = _alloc(2, 2, 3)
    table.copy_(torch.tensor([[7, -3], [1, 2]], dtype=torch.int32))   # 7 and -3 are not blocks of the pool
    count.fill_(1)
    ops.kv_blocks_release(table, free, count, torch.tensor([0, 0], dtype=torch.int32), BS)
    assert table.tolist() == [[-1, -1], [-1, -1]]
    assert count.item() == 3 and free.tolist() == [2, 1, 2]


# ---- the decoder -----------------------------------------------------------------------------------------------
E, HEADS, CAP = 64, 4, 2 * BS


def _decoder(kv_heads=None, rotary=False):
    torch.manual_seed(0)
    m = TransformerDecoder(decoder_layers=2, embed_dim=E, ffn_embed_dim=2 * E, attention_heads=HEADS,
                           max_seq_len=CAP, rel_pos=not rotary, rotary_dim=8 if rotary else None,
                           attention_kv_heads=kv_heads).eval()
    with torch.no_grad():
        for p in m.parameters():
            p.add_(torch.randn_like(p) * 0.02)
    return m.to(F64)


@pytest.mark.parametrize("kind", ["relpos", "rotary_gqa"])
def test_decoder_paged_equals_contiguous(kind):
    m = _decoder(kv_heads=2 if kind == "rotary_gqa" else None, rotary=kind == "rotary_gqa")
    g = torch.Generator().manual_seed(1)
    B, S = 3, 6
    enc = torch.randn(B, S, E, generator=g, dtype=F64)
    enc_pad = torch.zeros(B, S, dtype=torch.bool)
    enc_pad[1, 4:] = True
    # 4 blocks of 128 rows for 3 sequences of capacity 256: less than B x capacity
    caches = [m.new_cache(B, CAP), m.new_cache(B, CAP, block_size=BS, num_blocks=4)]
    paged = caches[1]
    assert paged.layers[0].k.shape == (4, BS, m.layers[0].self_attn.num_kv_heads, E // HEADS)

    def run(fn):
        outs = [fn(c) for c in caches]
        assert torch.equal(outs[0], outs[1])
        return outs[0]

    with torch.no_grad():
        L = 130
        prompt = torch.randn(B, L, E, generator=g, dtype=F64)
        pad = torch.zeros(B, L, dtype=torch.bool)
        pad[1, 20:] = True
        pad[2, 60:] = True
        run(lambda c: m(prompt, encoder_out=enc, padding_mask=pad, encoder_padding_mask=enc_pad, cache=c))
        assert paged.free_blocks() == 0 and not paged.overflowed()   # 2 + 1 + 1 blocks
        for _ in range(2):
            x = torch.randn(B, 1, E, generator=g, dtype=F64)
            run(lambda c: m(x, encoder_padding_mask=enc_pad, cache=c))
        x = torch.randn(B, 4, E, generator=g, dtype=F64)
        run(lambda c: m(x, encoder_padding_mask=enc_pad, cache=c))
        # a per-sequence rewind: sequence 0 drops back into its first block, which frees its second
        n = torch.tensor([10, 0, 2], dtype=torch.int32)
        for c in caches:
            c.rewind(n)
        assert paged.free_blocks() == 1
        # sequence 1 is emptied and re-prompted inside a packed ragged step; the others add 0 and 3 tokens
        for c in caches:
            c.rewind(torch.tensor([0, 1000, 0], dtype=torch.int32))
        assert paged.free_blocks() == 2
        sizes = [0, 7, 3]
        emb = torch.randn(sum(sizes), E, generator=g, dtype=F64)
        run(lambda c: m(emb, encoder_padding_mask=enc_pad, cache=c, cu_seqlens=_cu(sizes), max_seqlen=7))
        x = torch.randn(B, 1, E, generator=g, dtype=F64)
        run(lambda c: m(x, encoder_padding_mask=enc_pad, cache=c))
        for c in caches:
            c.rewind(1)
        x = torch.randn(B, 2, E, generator=g, dtype=F64)
        run(lambda c: m(x, encoder_padding_mask=enc_pad, cache=c))
        # reorder to the same batch size, then to a new one
        for c in caches:
            c.reorder(torch.tensor([2, 0, 1]))
        assert torch.equal(caches[0].seqlens, paged.seqlens)
        x = torch.randn(B, 1, E, generator=g, dtype=F64)
        run(lambda c: m(x, encoder_padding_mask=enc_pad[[2, 0, 1]], cache=c))
        assert paged.free_blocks() == 0
        for c in caches:
            c.reorder(torch.tensor([1, 1]))   # a repeated sequence gets blocks of its own
        x = torch.randn(2, 3, E, generator=g, dtype=F64)
        run(lambda c: m(x, encoder_padding_mask=enc_pad[[0, 0]], cache=c))
        assert not paged.overflowed()
        # the gathered rows below the lengths equal the contiguous cache's
        for lc, lp in zip(caches[0].layers, paged.layers):
            kg = _gathered(lp.k, paged.block_table)
            for b, n_b in enumerate(paged.seqlens.tolist()):
                assert torch.equal(kg[b, :n_b], lc.k[b, :n_b])


def test_decoder_pool_exhaustion_sets_the_flag():
    m = _decoder()
    cache = m.new_cache(2, CAP, block_size=BS, num_blocks=1)
    with torch.no_grad():
        m(torch.randn(2, 5, E, dtype=F64), cache=cache)
    assert cache.overflowed() and cache.free_blocks() == 0
    assert cache.block_table.tolist() == [[0, -1], [-1, -1]]


def test_new_cache_errors():
    m = _decoder()
    with pytest.raises(ValueError, match="multiple of 128"):
        m.new_cache(2, CAP, block_size=64)
    with pytest.raises(ValueError, match="multiple of block_size"):
        m.new_cache(2, 200, block_size=BS)
    with pytest.raises(ValueError, match="max_seq_len"):
        m.new_cache(2, 2 * CAP, block_size=BS)
    with pytest.raises(ValueError, match="num_blocks"):
        m.new_cache(2, CAP, block_size=BS, num_blocks=0)
    with pytest.raises(ValueError, match="num_blocks goes with block_size"):
        m.new_cache(2, CAP, num_blocks=4)
    cache = m.new_cache(3, CAP, block_size=BS)
    assert cache.free_blocks() == 6 and cache.block_table.shape == (3, 2)
