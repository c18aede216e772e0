"""ymp.engine.KVCache's row table on the CPU (no kernel involved): the table the single-token decoding steps read keys
through, `reindex` (a beam permutation that gathers the table and moves no K/V row), the batched prefill's shared first
slot, and `reorder` (the physical permutation) after a history of reindexes.

The K/V writes of the decoding kernels are simulated: position p of sequence b goes into cache row b * max_len + p.
The logical cache of a sequence is its rows gathered through the table; it must equal the cache that the all-moving
reorder history produces."""
import torch

from oracle import port


def _cache(B, ML):
    from ymp import engine
    return engine.KVCache(dict(port.GCFG_TINY), B, ML, torch.device("cpu"))


def _identity(B, ML):
    return torch.arange(B * ML, dtype=torch.int32).view(B, ML)


def _append(caches, n, gen, stride=1):
    """n new positions for every sequence, as the kernels write them: stride > 1 is gpt_decode's seq_stride prefill
    (only slot c * stride of each group is written; the moving reference, `caches[1:]`, gets every slot of the group,
    which is what each beam's cache must hold)."""
    c0 = caches[0]
    B, ML, off = c0.B, c0.max_len, c0.len
    vals = torch.randn(c0.store.shape[0], B // stride, n, c0.store.shape[2], generator=gen).to(c0.store.dtype)
    for i, c in enumerate(caches):
        st = c.store.view(c.store.shape[0], B, ML, -1)
        if i == 0:
            st[:, ::stride, off:off + n] = vals
        else:
            st[:, :, off:off + n] = vals.repeat_interleave(stride, 1)
        c._set_len(off + n)
    caches[0].share_prefill(stride)


def _logical(cache):
    """[layers, B, len, 3H]: position p of sequence b read through the row table."""
    idx = cache.rows[:, :cache.len].reshape(-1).long()
    return cache.store.index_select(1, idx).view(cache.store.shape[0], cache.B, cache.len, -1)


def _physical(cache):
    return cache.store.view(cache.store.shape[0], cache.B, cache.max_len, -1)[:, :, :cache.len]


def test_rows_identity_after_construction_and_reset():
    B, ML = 4, 7
    c = _cache(B, ML)
    assert c.rows.dtype == torch.int32 and c.rows.shape == (B, ML)
    assert torch.equal(c.rows, _identity(B, ML))
    ptrs = (c.rows.data_ptr(), c.store.data_ptr())
    c._set_len(3)
    c.reindex(torch.tensor([3, 3, 0, 1]))
    assert not torch.equal(c.rows, _identity(B, ML))
    c.reset()
    assert c.len == 0 and torch.equal(c.rows, _identity(B, ML))
    assert (c.rows.data_ptr(), c.store.data_ptr()) == ptrs     # the captured step holds both pointers


def test_reindex_touches_cached_columns_only_and_moves_no_row():
    B, ML, n = 5, 9, 4
    c = _cache(B, ML)
    g = torch.Generator().manual_seed(0)
    c.store.copy_(torch.randn(c.store.shape, generator=g).to(c.store.dtype))
    store0 = c.store.clone()
    ptrs = (c.rows.data_ptr(), c.store.data_ptr())
    c._set_len(n)
    idx = torch.tensor([4, 4, 1, 0, 2])
    c.reindex(idx)
    ident = _identity(B, ML)
    assert torch.equal(c.rows[:, :n], ident[idx, :n])
    assert torch.equal(c.rows[:, n:], ident[:, n:])             # where the next positions go: each sequence's own slot
    assert torch.equal(c.store, store0)                          # no K/V byte moved
    c._set_len(n + 1)
    idx2 = torch.tensor([1, 0, 0, 3, 3])
    before = c.rows.clone()
    c.reindex(idx2)
    assert torch.equal(c.rows[:, :n + 1], before[idx2, :n + 1])
    assert torch.equal(c.rows[:, n + 1:], ident[:, n + 1:])
    assert (c.rows.data_ptr(), c.store.data_ptr()) == ptrs
    empty = _cache(B, ML)
    empty.reindex(idx)                                           # nothing cached: nothing to permute
    assert torch.equal(empty.rows, ident)


def test_seq_stride_prefill_table():
    B, ML, beam, n = 6, 8, 3, 5
    c = _cache(B, ML)
    c._set_len(n)
    c.share_prefill(beam)
    ident = _identity(B, ML)
    for b in range(B):
        first = (b // beam) * beam
        assert torch.equal(c.rows[b, :n], ident[first, :n]), b   # every beam reads its clip's first slot
        assert torch.equal(c.rows[b, n:], ident[b, n:]), b
    c1 = _cache(B, ML)
    c1._set_len(n)
    c1.share_prefill(1)
    assert torch.equal(c1.rows, ident)


def _history(seed, B, ML, stride, n_ops):
    """Random appends and beam permutations on an indexed cache and on the all-moving reference."""
    g = torch.Generator().manual_seed(seed)
    idx_c, mov = _cache(B, ML), _cache(B, ML)
    n0 = int(torch.randint(1, 4, (1,), generator=g))
    _append([idx_c, mov], n0, g, stride=stride)
    ops = []
    while idx_c.len < ML and len(ops) < n_ops:
        idx = torch.randint(0, B, (B,), generator=g)
        idx_c.reindex(idx)
        mov.reorder(idx)
        _append([idx_c, mov], 1, g)
        ops.append(idx)
    return idx_c, mov, g


def test_reindex_history_equals_moving_reorder():
    for seed, (B, ML, stride) in enumerate([(5, 12, 1), (6, 10, 3), (15, 9, 5), (4, 6, 2)]):
        idx_c, mov, _ = _history(seed, B, ML, stride, n_ops=20)
        assert idx_c.len == mov.len
        assert torch.equal(_logical(idx_c), _physical(mov)), (seed, B, ML, stride)
        # every entry names a valid row, also past len
        assert int(idx_c.rows.min()) >= 0 and int(idx_c.rows.max()) < B * ML


def test_reorder_after_reindex_equals_moving_history():
    """reorder materialises the table first (physical row b := logical row b, table := identity), then permutes."""
    for seed, (B, ML, stride) in enumerate([(5, 12, 1), (6, 10, 3)]):
        idx_c, mov, g = _history(100 + seed, B, ML, stride, n_ops=5)
        ptrs = (idx_c.rows.data_ptr(), idx_c.store.data_ptr())
        idx = torch.randint(0, B, (B,), generator=g)
        idx_c.reorder(idx)
        mov.reorder(idx)
        assert torch.equal(idx_c.rows, _identity(B, ML))
        assert torch.equal(_physical(idx_c), _physical(mov))
        assert (idx_c.rows.data_ptr(), idx_c.store.data_ptr()) == ptrs
        # and the history can go on mixing both
        _append([idx_c, mov], 1, g)
        idx = torch.randint(0, B, (B,), generator=g)
        idx_c.reindex(idx)
        mov.reorder(idx)
        assert torch.equal(_logical(idx_c), _physical(mov))


def test_reorder_right_after_seq_stride_prefill_copies_the_first_slot():
    """swap_key_value_dict straight after the batched prefill: the reference's per-beam rows, physically."""
    g = torch.Generator().manual_seed(7)
    B, ML, beam = 6, 8, 3
    idx_c, mov = _cache(B, ML), _cache(B, ML)
    _append([idx_c, mov], 4, g, stride=beam)
    idx = torch.tensor([0, 0, 0, 3, 3, 3])
    idx_c.reorder(idx)
    mov.reorder(idx)
    assert torch.equal(_physical(idx_c), _physical(mov))
