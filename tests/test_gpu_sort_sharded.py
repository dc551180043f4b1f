"""GPU: sort / sort_desc over rows sharded across ranks (b2p_sort_shard_* and b2p_sort_cells_allgather_dev).  R ranks
are simulated on one GPU, one context each: every rank counts its valid cells, the counts are stacked into the table,
every rank packs its block, the blocks are laid back to back in rank order, and every rank merges them; one more merge
takes the table and the blocks rotated.  Every merge's out_cells must equal b2p_sort_cells_dev over the global grid
bit for bit, and out_vals the grid's value bits at those cells."""
import contextlib

import numpy as np
import pytest

from tests import select_keys as sk
from tests.ranks import one_rank_comm

pytestmark = pytest.mark.gpu

I64_MIN, I64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max


def dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def words_with_junk(ok):
    """validity words with every bit past T in the last word set (the calls must ignore them)"""
    w = sk.words(ok).copy()
    T = ok.shape[1]
    if T % 32:
        w[:, -1] |= np.uint32((0xFFFFFFFF << (T % 32)) & 0xFFFFFFFF)
    return w


class Rank:
    """One simulated rank: its own context and rows (global row ids `rows`, increasing) of the global grid"""
    def __init__(self, rows, grids, valid, T, i64=False):
        from greptimedb_b200 import Context
        self.ctx = Context(0)
        self.ctx.use_torch_stream()
        self.rows, self.T, self.i64 = rows, T, i64
        n = max(rows.size, 1)
        pad = lambda a: np.concatenate([a[rows], np.zeros((n - rows.size,) + a.shape[1:], a.dtype)])
        self.vals = [dev(pad(g)) for g in grids]
        self.valid = dev(pad(valid).view(np.int32))
        self.row_id = dev(np.concatenate([rows, np.zeros(n - rows.size, np.int64)]).astype(np.int32))

    @property
    def F(self):
        return len(self.vals)

    def grid(self):
        return self.vals[0] if self.i64 else (self.vals if self.F > 1 else self.vals[0])

    def count(self):
        return self.ctx.sort_shard_counts_dev(self.valid, self.rows.size, self.T)

    def pack(self, desc, count):
        import torch
        block = torch.full((max(int(count) * (self.F + 1), 1),), -1, dtype=torch.int64, device="cuda")
        self.ctx.sort_shard_pack_dev(desc, self.grid(), self.valid, self.row_id, self.rows.size, self.T, count, block,
                                     i64=self.i64)
        return block

    def merge(self, desc, counts, blocks):
        import torch
        N = int(np.asarray(counts, np.int64).sum())
        cells = torch.full((max(N, 1),), -1, dtype=torch.int64, device="cuda")
        dt = torch.int64 if self.i64 else torch.float64
        outs = [torch.full((max(N, 1),), -7, dtype=dt, device="cuda") for _ in range(self.F)]
        self.ctx.sort_shard_merge_dev(desc, counts, blocks, cells, outs if self.F > 1 else outs[0], i64=self.i64)
        torch.cuda.synchronize()
        return cells.cpu().numpy()[:N].view(np.uint64), [o.cpu().numpy()[:N] for o in outs]

    def close(self):
        self.ctx.close()


def single_sort(desc, grids, valid, T, i64=False):
    """b2p_sort_cells_dev (_fields_dev, _i64_dev) over the global grid -> cells u64"""
    import torch
    from greptimedb_b200 import Context
    R = valid.shape[0]
    with Context(0) as ctx:
        ctx.use_torch_stream()
        out = torch.full((max(R * T, 1),), -1, dtype=torch.int64, device="cuda")
        n = torch.zeros(1, dtype=torch.int64, device="cuda")
        vs, vw = [dev(g) for g in grids], dev(valid.view(np.int32))
        if i64:
            ctx.sort_cells_i64_dev(desc, vs[0], vw, R, T, out, n)
        elif len(vs) > 1:
            ctx.sort_cells_fields_dev(desc, vs, vw, R, T, out, n)
        else:
            ctx.sort_cells_dev(desc, vs[0], vw, R, T, out, n)
        torch.cuda.synchronize()
        return out.cpu().numpy()[:int(n.item())].view(np.uint64)


def run_sharded(desc, owner, n_ranks, grids, ok, T, i64=False):
    """every rank's (cells, values) and the rotated merge's, the counts and the bytes each rank reported"""
    import torch
    valid = words_with_junk(ok)
    ranks = [Rank(np.flatnonzero(owner == r), grids, valid, T, i64) for r in range(n_ranks)]
    try:
        counts = np.concatenate([r.count() for r in ranks])
        blocks, sent = [], []
        for r, c in zip(ranks, counts):
            blocks.append(r.pack(desc, c))
            sent.append(r.ctx.last_exchange_bytes())
        F = len(grids)
        laid = lambda order: torch.cat([blocks[i][:int(counts[i]) * (F + 1)] for i in order] +
                                       [torch.zeros(1, dtype=torch.int64, device="cuda")])
        outs = [r.merge(desc, counts, laid(range(n_ranks))) for r in ranks]
        rot = [(j + 1) % n_ranks for j in range(n_ranks)]
        outs.append(ranks[-1].merge(desc, counts[rot], laid(rot)))
        return outs, counts, sent
    finally:
        for r in ranks:
            r.close()


def check(desc, owner, n_ranks, grids, ok, T, i64=False):
    outs, counts, sent = run_sharded(desc, owner, n_ranks, grids, ok, T, i64)
    exp = single_sort(desc, grids, words_with_junk(ok), T, i64)
    assert exp.size == ok.sum() == counts.sum()
    F = len(grids)
    for cells, vals in outs:
        assert np.array_equal(cells, exp)
        for f in range(F):
            want = np.ascontiguousarray(grids[f]).reshape(-1)[exp.astype(np.int64)]
            assert np.array_equal(vals[f].view(np.uint64), want.view(np.uint64))
    assert [int(c) for c in counts] == [int(ok[owner == r].sum()) for r in range(n_ranks)]
    assert sent == [int(c) * 8 * (F + 1) for c in counts]


def hashed(n_rows, n_ranks, seed=0):
    from greptimedb_b200 import distributed as D
    own = D.shard_of_series(np.arange(n_rows, dtype=np.uint32) + np.uint32(seed), n_ranks)
    if n_ranks == 3:
        own[own == 2] = 0  # a rank with no rows
    return own


def specials(R, T, seed, p=0.7):
    from tests.test_sort_oracle import TOTAL_ORDER
    rng = np.random.default_rng(seed)
    return np.array(TOTAL_ORDER)[rng.integers(0, len(TOTAL_ORDER), (R, T))], rng.random((R, T)) < p


@pytest.mark.parametrize("n_ranks", [1, 2, 3, 8])
@pytest.mark.parametrize("desc", [False, True])
def test_simulated_ranks_match_the_single_rank_sort(n_ranks, desc):
    vals, ok = specials(700, 37, n_ranks)
    check(desc, hashed(700, n_ranks), n_ranks, [vals], ok, 37)


@pytest.mark.parametrize("T", [1, 37, 1000])
def test_step_counts(T):
    R = {1: 20000, 37: 900, 1000: 60}[T]
    rng = np.random.default_rng(T)
    vals = rng.normal(size=(R, T))
    vals[rng.random((R, T)) < 0.3] = 0.5  # ties across ranks
    ok = rng.random((R, T)) < 0.8
    for desc in (False, True):
        check(desc, hashed(R, 3, T), 3, [vals], ok, T)


def test_contiguous_shards():
    vals, ok = specials(5000, 3, 9)
    owner = np.minimum(np.arange(5000) // 1250, 3)
    check(False, owner, 4, [vals], ok, 3)
    check(True, owner[::-1].copy(), 4, [vals], ok, 3)


def test_many_merge_tiles():
    rng = np.random.default_rng(4)
    R, T = 300_000, 1
    vals = rng.normal(size=(R, T))
    vals[rng.random((R, T)) < 0.5] = np.nan  # one key shared by half the cells, in every tile of every round
    ok = rng.random((R, T)) < 0.9
    check(False, hashed(R, 8, 1), 8, [vals], ok, T)
    check(True, hashed(R, 5, 2), 5, [vals], ok, T)


def test_no_valid_cells_anywhere():
    vals, _ = specials(100, 37, 3)
    ok = np.zeros((100, 37), bool)
    for n_ranks in (1, 3):
        check(False, hashed(100, n_ranks), n_ranks, [vals], ok, 37)


@pytest.mark.parametrize("n_fields", [2, 3])
def test_fields(n_fields):
    rng = np.random.default_rng(n_fields)
    R, T = 800, 37
    grids = [rng.choice([1.0, -0.0, 0.0], (R, T)), rng.choice([3.0, np.nan, -np.inf, 2.0], (R, T)),
             specials(R, T, 5)[0]][:n_fields]
    ok = rng.random((R, T)) < 0.85
    for n_ranks in (2, 3, 8):
        for desc in (False, True):
            check(desc, hashed(R, n_ranks, 7), n_ranks, grids, ok, T)


def test_one_field_list_is_the_one_field_form():
    vals, ok = specials(300, 40, 12)
    check(True, hashed(300, 2), 2, [vals], ok, 40)


@pytest.mark.parametrize("n_ranks", [1, 2, 3, 8])
def test_int64(n_ranks):
    rng = np.random.default_rng(n_ranks + 40)
    R, T = 600, 37
    iv = rng.choice(np.array([I64_MIN, I64_MAX, -1, 0, 1, 7, 1 << 62], np.int64), (R, T))
    ok = rng.random((R, T)) < 0.8
    for desc in (False, True):
        check(desc, hashed(R, n_ranks, 3), n_ranks, [iv], ok, T, i64=True)


def composed(desc, grids, ok, T, i64=False, comm=False):
    """the composed call over every row on one context (without a communicator, or over a one-rank one)"""
    import torch
    valid = words_with_junk(ok)
    r = Rank(np.arange(ok.shape[0]), grids, valid, T, i64)
    try:
        with one_rank_comm(r.ctx) if comm else contextlib.nullcontext():
            counts = r.ctx.sort_shard_counts_dev(r.valid, r.rows.size, T)
            N = int(counts.sum())
            cells = torch.full((max(N, 1),), -1, dtype=torch.int64, device="cuda")
            dt = torch.int64 if i64 else torch.float64
            outs = [torch.full((max(N, 1),), -7, dtype=dt, device="cuda") for _ in grids]
            r.ctx.sort_cells_allgather_dev(desc, r.grid(), r.valid, r.row_id, r.rows.size, T, counts, cells,
                                           outs if len(grids) > 1 else outs[0], i64=i64)
            torch.cuda.synchronize()
            sent = r.ctx.last_exchange_bytes()
    finally:
        r.close()
    exp = single_sort(desc, grids, valid, T, i64)
    assert np.array_equal(cells.cpu().numpy()[:N].view(np.uint64), exp)
    for g, o in zip(grids, outs):
        want = np.ascontiguousarray(g).reshape(-1)[exp.astype(np.int64)]
        assert np.array_equal(o.cpu().numpy()[:N].view(np.uint64), want.view(np.uint64))
    assert sent == N * 8 * (len(grids) + 1)


@pytest.mark.parametrize("comm", [False, True])
def test_composed_call(comm):
    vals, ok = specials(2000, 37, 21)
    rng = np.random.default_rng(22)
    for desc in (False, True):
        composed(desc, [vals], ok, 37, comm=comm)
    composed(True, [vals, specials(2000, 37, 23)[0]], ok, 37, comm=comm)
    iv = rng.choice(np.array([I64_MIN, I64_MAX, 0, 5], np.int64), (2000, 37))
    composed(False, [iv], ok, 37, i64=True, comm=comm)
    composed(False, [vals], np.zeros_like(ok), 37, comm=comm)


def test_argument_errors():
    import torch
    from greptimedb_b200 import B2PError
    vals, ok = specials(200, 37, 31)
    r = Rank(np.arange(200), [vals], sk.words(ok), 37)
    try:
        n = int(r.count()[0])
        blk = torch.zeros(2 * n, dtype=torch.int64, device="cuda")
        out = torch.zeros(n, dtype=torch.int64, device="cuda")
        ov = torch.zeros(n, dtype=torch.float64, device="cuda")
        ctx = r.ctx
        with pytest.raises(B2PError):  # counts[rank] is not the rank's own count
            ctx.sort_cells_allgather_dev(False, r.grid(), r.valid, r.row_id, 200, 37, [n - 1], out, ov)
        with pytest.raises(B2PError):
            ctx.sort_shard_pack_dev(False, r.grid(), r.valid, r.row_id, 200, 37, n + 1, blk)
        bad = np.arange(200, dtype=np.int32)
        bad[100] = bad[99]  # not strictly increasing
        with pytest.raises(B2PError):
            ctx.sort_cells_allgather_dev(False, r.grid(), r.valid, dev(bad), 200, 37, [n], out, ov)
        with pytest.raises(B2PError):
            ctx.sort_shard_pack_dev(False, r.grid(), r.valid, dev(bad[::-1].copy()), 200, 37, n, blk)
        with pytest.raises(B2PError):  # NULL arguments
            ctx.sort_cells_allgather_dev(False, r.grid(), r.valid, None, 200, 37, [n], out, ov)
        with pytest.raises(B2PError):
            ctx.sort_cells_allgather_dev(False, r.grid(), r.valid, r.row_id, 200, 37, [n], None, ov)
        with pytest.raises(B2PError):
            ctx.sort_shard_pack_dev(False, r.grid(), r.valid, r.row_id, 200, 37, n, None)
        with pytest.raises(B2PError):
            ctx.sort_shard_merge_dev(False, [n], None, out, ov)
        with pytest.raises(B2PError):
            ctx.sort_shard_counts_dev(None, 200, 37)
        with pytest.raises(B2PError) as e:  # T > 2^32
            ctx.sort_shard_counts_dev(r.valid, 0, (1 << 32) + 1)
        assert e.value.code == -5
        with pytest.raises(B2PError):
            ctx.sort_shard_pack_dev(False, r.grid(), r.valid, r.row_id, 0, (1 << 32) + 1, 0, blk)
        ctx.sort_shard_pack_dev(False, r.grid(), r.valid, r.row_id, 200, 37, n, blk)
        assert ctx.last_exchange_bytes() == n * 16
    finally:
        r.close()
