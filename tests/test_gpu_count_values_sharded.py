"""GPU: count_values by label over rows sharded across ranks (b2p_count_values_shard_* and
b2p_count_values_allgather_dev).  R ranks are simulated on one GPU, one context each: every rank runs
b2p_count_values_dev over its own rows and measures its heights, the heights are stacked into the table, and per batch
each rank packs its block; the blocks are gathered section by section, and every rank merges them in its own rotation
(with the heights table's rows rotated the same way).  Every rank's rows out_goff[g] .. out_goff[g] + U_g must equal the
first U_g rows of group g of b2p_count_values_dev over all rows, bit for bit, and the single-rank rows past U_g must
all have count 0."""
import numpy as np
import pytest

from tests import select_keys as sk
from tests.ranks import one_rank_comm

pytestmark = pytest.mark.gpu

ENTRY = 12  # bytes of one (key u64, count u32) entry
MAX_NAN = 0x7FFFFFFFFFFFFFFF
I64_MAX, I64_MIN = np.iinfo(np.int64).max, np.iinfo(np.int64).min


def dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


class Rank:
    """One simulated rank: its own context, rows, group index and count_values output"""
    def __init__(self, rows, vals, valid, gid, n_groups, T, i64=False):
        import torch
        from greptimedb_b200 import Context
        self.ctx = Context(0)
        self.ctx.use_torch_stream()
        self.rows, self.T, self.n_groups, self.i64 = rows, T, n_groups, i64
        n = max(rows.size, 1)
        self.vals, self.valid = dev(vals[rows]), dev(valid[rows].view(np.int32))
        self.ix = self.ctx.group_index_create_dev(dev(gid[rows].view(np.int32)), rows.size, n_groups)
        self.lv = torch.full((n * T,), -7, dtype=torch.int64 if i64 else torch.float64, device="cuda")
        self.lc = torch.full((n * T,), -1, dtype=torch.int32, device="cuda")
        if rows.size and T:
            f = self.ctx.count_values_i64_dev if i64 else self.ctx.count_values_dev
            f(self.vals, self.valid, self.ix, T, self.lv, self.lc)

    def heights(self):
        return self.ctx.count_values_shard_heights_dev(self.lc, self.ix, self.T, self.n_groups)

    def close(self):
        self.ctx.group_index_destroy(self.ix)
        self.ctx.close()


def make_ranks(owner, n_ranks, vals, ok, gid, n_groups, T, i64=False):
    valid = sk.words(ok)
    return [Rank(np.flatnonzero(owner == r), vals, valid, gid, n_groups, T, i64) for r in range(n_ranks)]


def hashed(n_rows, n_ranks, seed):
    """hashed rows, except that with three ranks the last one holds nothing"""
    from greptimedb_b200 import distributed as D
    own = D.shard_of_series(np.arange(n_rows, dtype=np.uint32) + np.uint32(seed), n_ranks)
    if n_ranks == 3:
        own[own == 2] = 0
    return own


def run_sharded(ranks, n_groups, T):
    """heights, plan, then per batch every rank's block and every rank's merge over the gathered blocks in its own
    rotation -> ([(out_val, out_cnt)] per rank [U, T], heights [R, G], out_goff, plan, bytes sent per rank)"""
    import torch
    from greptimedb_b200 import Context
    R, i64 = len(ranks), ranks[0].i64
    H = np.concatenate([r.heights() for r in ranks]) if n_groups else np.zeros((R, 0), np.uint32)
    plan = ranks[0].ctx.count_values_shard_plan(H, T)
    out_goff = Context.count_values_shard_rows(H)
    U = int(out_goff[-1])
    blocks = [torch.zeros(max(plan["block_bytes"], 16), dtype=torch.uint8, device="cuda") for _ in ranks]
    outs = [(torch.full((max(U, 1) * T,), -7, dtype=torch.int64 if i64 else torch.float64, device="cuda"),
             torch.full((max(U, 1) * T,), -1, dtype=torch.int32, device="cuda")) for _ in ranks]
    sent = [0] * R
    for b in range(plan["n_batches"]):
        nbytes = None
        for i, (r, blk) in enumerate(zip(ranks, blocks)):
            r.ctx.count_values_shard_pack_dev(r.lv, r.lc, r.ix, T, H, i, b, blk, i64=i64)
            got = r.ctx.last_exchange_bytes()
            assert nbytes in (None, got), "ranks disagree on the block size"
            nbytes = got
            sent[i] += got
        assert 0 < nbytes <= plan["block_bytes"] and nbytes % ENTRY == 0
        P = nbytes // ENTRY
        for i, (r, (ov, oc)) in enumerate(zip(ranks, outs)):
            order = [(i + j) % R for j in range(R)]
            gathered = torch.cat([blocks[o][:8 * P] for o in order] + [blocks[o][8 * P:12 * P] for o in order])
            r.ctx.count_values_shard_merge_dev(H[order], T, b, gathered, ov, oc, i64=i64)
    torch.cuda.synchronize()
    res = [(ov.cpu().numpy()[:U * T].reshape(U, T), oc.cpu().numpy().view(np.uint32)[:U * T].reshape(U, T))
           for ov, oc in outs]
    return res, H, out_goff, plan, sent


def single_rank(full):
    n = full.rows.size
    val = full.lv.cpu().numpy()[:n * full.T].reshape(n, full.T)
    return val, full.lc.cpu().numpy().view(np.uint32)[:n * full.T].reshape(n, full.T)


def same(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint64), np.ascontiguousarray(b).view(np.uint64))


def check_case(ranks, full, vals, ok, gid, n_groups, T):
    """-> (heights, plan, bytes sent per rank)"""
    outs, H, out_goff, plan, sent = run_sharded(ranks, n_groups, T)
    one, one_cnt = single_rank(full)
    if not full.i64:
        exp, exp_cnt = sk.count_values(vals, ok, gid, n_groups)
        assert same(one, exp) and (one_cnt == exp_cnt).all()
    _, goff = sk._groups(gid, n_groups)
    for r, h in zip(ranks, H):  # the device heights are the rows with a count, per group
        cnt = single_rank(r)[1] if r.rows.size else np.zeros((0, T), np.uint32)
        _, lg = sk._groups(gid[r.rows], n_groups)
        for g in range(n_groups):
            nz = np.flatnonzero(cnt[lg[g]:lg[g + 1]].any(axis=1))
            assert h[g] == (nz[-1] + 1 if nz.size else 0), (len(ranks), g)
    for out, cnt in outs:
        for g in range(n_groups):
            U = out_goff[g + 1] - out_goff[g]
            assert U <= goff[g + 1] - goff[g]
            assert same(out[out_goff[g]:out_goff[g + 1]], one[goff[g]:goff[g] + U]), (len(ranks), g)
            assert (cnt[out_goff[g]:out_goff[g + 1]] == one_cnt[goff[g]:goff[g] + U]).all(), (len(ranks), g)
            assert (one_cnt[goff[g] + U:goff[g + 1]] == 0).all(), (len(ranks), g)
    assert len(set(sent)) == 1
    return H, plan, sent[0]


def mixed_grid(seed, T, sizes=(300, 150, 1, 1, 3, 0, 9, 40, 2, 65, 1, 7)):
    """select_keys' classes (payloads, ±0, the largest positive NaN among the sentinels), repeated values, groups
    absent on some ranks, empty groups, rows of no group and rows without a valid cell"""
    rng = np.random.default_rng(seed)
    vals, ok, gid, n_groups, _ = sk.grid(list(sizes), T, 0.5, rng, drop=0.2, gid_gap=2, stray=6)
    rep = rng.random(vals.shape) < 0.3
    vals[rep] = np.array([1.5, -0.0, 0.0, np.uint64(MAX_NAN).view(np.float64)])[rng.integers(0, 4, int(rep.sum()))]
    ok[rng.random(gid.size) < 0.03] = False
    return vals, ok, gid, n_groups


def run_case(owner, n_ranks, vals, ok, gid, n_groups, T):
    full = Rank(np.arange(gid.size), vals, sk.words(ok), gid, n_groups, T)
    ranks = make_ranks(owner, n_ranks, vals, ok, gid, n_groups, T)
    try:
        return check_case(ranks, full, vals, ok, gid, n_groups, T)
    finally:
        for r in ranks + [full]:
            r.close()


@pytest.mark.parametrize("n_ranks", [1, 2, 3, 8])
def test_simulated_ranks_match_the_single_rank_count(n_ranks):
    T = 37
    vals, ok, gid, n_groups = mixed_grid(n_ranks, T)
    H, plan, sent = run_case(hashed(gid.size, n_ranks, n_ranks), n_ranks, vals, ok, gid, n_groups, T)
    assert plan["n_batches"] == 1
    assert sent == T * int(H.astype(np.int64).sum(axis=1).max()) * ENTRY  # one batch: W = T


@pytest.mark.parametrize("T", [1, 1000])
def test_step_counts(T):
    rng = np.random.default_rng(T)
    vals, ok, gid, n_groups, _ = sk.grid([300, 20, 1, 0, 4], T, 0.5, rng, drop=0.1, stray=2)
    vals[rng.random(vals.shape) < 0.5] = 2.0
    run_case(hashed(gid.size, 2, T), 2, vals, ok, gid, n_groups, T)


def test_value_classes_split_across_ranks():
    """the same values on both ranks and disjoint values, ±0.0 and NaN payloads split across ranks, the largest
    positive NaN on one rank only (and alone), a group on one rank only, uneven and empty shards"""
    from tests.test_count_values_sharded_gloo import cases
    for name, vals, ok, gid, n_groups, owner in cases():
        run_case(owner, 2, vals, ok, gid, n_groups, vals.shape[1])


def test_largest_nan_beside_fillers_in_every_order():
    """one rank's only value is the largest positive NaN at a step where the other rank has fillers: the run of key ~0
    mixes entries of count 0 and real counts, in whatever order the sort leaves them"""
    T = 40
    R = 24
    gid = np.zeros(R, np.uint32)
    own = (np.arange(R) % 2).astype(np.int64)
    vals = np.tile(np.arange(R, dtype=np.float64)[:, None], (1, T))  # rank 0: many distinct values -> many fillers
    vals[own == 1] = np.uint64(MAX_NAN).view(np.float64)
    ok = np.random.default_rng(3).random((R, T)) < 0.6
    for n_ranks, owner in ((2, own), (2, 1 - own), (3, np.where(own == 1, 2, 0))):
        run_case(owner, n_ranks, vals, ok, gid, 1, T)


def test_no_groups():
    import torch
    T = 40
    vals, ok = np.random.default_rng(2).standard_normal((5, T)), np.ones((5, T), bool)
    gid = np.full(5, 3, np.uint32)  # rows of no group
    full = Rank(np.arange(5), vals, sk.words(ok), gid, 0, T)
    try:
        H = full.heights()
        assert H.shape == (1, 0)
        assert full.ctx.count_values_shard_plan(H, T) == {"n_batches": 0, "block_bytes": 0}
        out = torch.zeros(1, dtype=torch.float64, device="cuda")
        cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
        full.ctx.count_values_allgather_dev(full.lv, full.lc, full.ix, T, H, out, cnt)
        assert full.ctx.last_exchange_bytes() == 0
    finally:
        full.close()


def composed_check(full, vals, ok, gid, n_groups, T):
    """the composed call over one rank: the first U_g rows of each group of the single-rank count, and the bytes of
    the same batches run step by step"""
    import torch
    H = full.heights()
    out_goff = full.ctx.count_values_shard_rows(H)
    U = int(out_goff[-1])
    ov = torch.full((max(U, 1) * T,), -7, dtype=torch.int64 if full.i64 else torch.float64, device="cuda")
    oc = torch.full((max(U, 1) * T,), -1, dtype=torch.int32, device="cuda")
    full.ctx.count_values_allgather_dev(full.lv, full.lc, full.ix, T, H, ov, oc, i64=full.i64)
    torch.cuda.synchronize()
    sent = full.ctx.last_exchange_bytes()
    outs, _, _, _, step_sent = run_sharded([full], n_groups, T)
    assert sent == step_sent[0]
    ov, oc = ov.cpu().numpy()[:U * T].reshape(U, T), oc.cpu().numpy().view(np.uint32)[:U * T].reshape(U, T)
    assert same(ov, outs[0][0]) and (oc == outs[0][1]).all()
    one, one_cnt = single_rank(full)
    _, goff = sk._groups(gid, n_groups)
    for g in range(n_groups):
        u = out_goff[g + 1] - out_goff[g]
        assert same(ov[out_goff[g]:out_goff[g + 1]], one[goff[g]:goff[g] + u]), g
        assert (oc[out_goff[g]:out_goff[g + 1]] == one_cnt[goff[g]:goff[g] + u]).all(), g
    return sent


@pytest.mark.parametrize("n_ranks", [2, 3])
def test_int64_against_the_single_rank_int64_count(n_ranks):
    T = 37
    rng = np.random.default_rng(40 + n_ranks)
    _, ok, gid, n_groups, _ = sk.grid([120, 33, 5, 1, 0, 64], T, 0.5, rng, drop=0.2, gid_gap=2, stray=3)
    pool = np.array([I64_MAX, I64_MIN, 0, -1, 1, 7, I64_MAX - 1, -(1 << 52)], np.int64)
    ivals = pool[rng.integers(0, pool.size, ok.shape)]
    wide = rng.random(ok.shape) < 0.2
    ivals[wide] = rng.integers(I64_MIN, I64_MAX, int(wide.sum()), dtype=np.int64)
    ivals[:, 0] = I64_MAX  # INT64_MAX, whose key is the filler's, at every group's first step
    valid = sk.words(ok)
    owner = hashed(gid.size, n_ranks, 5)
    full = Rank(np.arange(gid.size), ivals, valid, gid, n_groups, T, i64=True)
    ranks = [Rank(np.flatnonzero(owner == r), ivals, valid, gid, n_groups, T, i64=True) for r in range(n_ranks)]
    try:
        check_case(ranks, full, ivals, ok, gid, n_groups, T)
        composed_check(full, ivals, ok, gid, n_groups, T)
        v, c = single_rank(full)
        assert (v[:, 0][c[:, 0] > 0] == I64_MAX).any()
    finally:
        for r in ranks + [full]:
            r.close()


def test_batches_under_a_small_exchange_cap(monkeypatch):
    """a cap of 64 KB cuts the groups and steps into batches, and the group of 900 members is a batch of its own over
    32 steps; the result does not change, and the composed call sends what the steps send"""
    monkeypatch.setenv("B2P_TOPK_EXCHANGE_BYTES", str(64 << 10))
    T = 200
    vals, ok, gid, n_groups = mixed_grid(9, T, sizes=(900, 150, 1, 3, 0, 9, 40, 2, 65, 1, 7))
    vals[rng_cells(vals.shape, 9)] = 4.0
    H, plan, sent = run_case(hashed(gid.size, 2, 9), 2, vals, ok, gid, n_groups, T)
    assert plan["n_batches"] > T // 32
    full = Rank(np.arange(gid.size), vals, sk.words(ok), gid, n_groups, T)
    try:
        assert full.ctx.count_values_shard_plan(full.heights(), T)["n_batches"] > 1
        composed_check(full, vals, ok, gid, n_groups, T)
    finally:
        full.close()


def rng_cells(shape, seed):
    return np.random.default_rng(seed).random(shape) < 0.3


def test_composed_call_without_communicator_is_the_single_rank_count():
    T = 70
    vals, ok, gid, n_groups = mixed_grid(3, T, sizes=(3000, 150, 1, 1, 3, 0, 9))
    full = Rank(np.arange(gid.size), vals, sk.words(ok), gid, n_groups, T)
    try:
        sent = composed_check(full, vals, ok, gid, n_groups, T)
        assert sent == T * int(full.heights().astype(np.int64).sum()) * ENTRY
    finally:
        full.close()


def test_single_rank_communicator_round_trips_the_blocks():
    """Over a one-rank communicator, the heights' all-gather and the composed call over NCCL's all-gathers"""
    T = 70
    vals, ok, gid, n_groups = mixed_grid(4, T, sizes=(3000, 150, 1, 1, 3, 0, 9))
    full = Rank(np.arange(gid.size), vals, sk.words(ok), gid, n_groups, T)
    try:
        with one_rank_comm(full.ctx):
            composed_check(full, vals, ok, gid, n_groups, T)
    finally:
        full.close()


def test_argument_errors():
    import torch
    from greptimedb_b200 import B2PError
    T = 33
    vals, ok, gid, n_groups = mixed_grid(5, T, sizes=(300, 20, 4))
    full = Rank(np.arange(gid.size), vals, sk.words(ok), gid, n_groups, T)
    try:
        H = full.heights()
        plan = full.ctx.count_values_shard_plan(H, T)
        blk = torch.zeros(plan["block_bytes"], dtype=torch.uint8, device="cuda")
        U = int(H.astype(np.int64).sum())
        ov = torch.zeros(U * T, dtype=torch.float64, device="cuda")
        oc = torch.zeros(U * T, dtype=torch.int32, device="cuda")
        pack = full.ctx.count_values_shard_pack_dev
        with pytest.raises(B2PError):  # batch out of range
            pack(full.lv, full.lc, full.ix, T, H, 0, plan["n_batches"], blk)
        with pytest.raises(B2PError):
            full.ctx.count_values_shard_merge_dev(H, T, plan["n_batches"], blk, ov, oc)
        with pytest.raises(B2PError):  # NULL block, NULL output
            pack(full.lv, full.lc, full.ix, T, H, 0, 0, None)
        with pytest.raises(B2PError):
            full.ctx.count_values_shard_merge_dev(H, T, 0, blk, None, oc)
        with pytest.raises(B2PError):  # rank outside the table
            pack(full.lv, full.lc, full.ix, T, H, 1, 0, blk)
        big = H.copy()
        big[0, 2] = 21  # more rows than the rank's 20 members of group 2
        with pytest.raises(B2PError):
            pack(full.lv, full.lc, full.ix, T, big, 0, 0, blk)
        with pytest.raises(B2PError):
            full.ctx.count_values_allgather_dev(full.lv, full.lc, full.ix, T, big, ov, oc)
        pack(full.lv, full.lc, full.ix, T, H, 0, 0, blk)
        assert full.ctx.last_exchange_bytes() > 0
    finally:
        full.close()
