"""GPU: topk / bottomk over rows sharded across ranks (b2p_topk_shard_* and b2p_topk_allgather_dev).  R ranks are
simulated on one GPU, one context each, through the per-rank and merge entry points: each rank writes its candidate
block, the blocks are concatenated section by section as the all-gather lays them, the merge runs once, then each rank
marks its words.  The union of the kept cells must equal b2p_topk_dev over all rows and select_keys.topk, bit for bit."""
import math

import numpy as np
import pytest

from tests import select_keys as sk
from tests.ranks import one_rank_comm

pytestmark = pytest.mark.gpu

NAN_NEG = np.array([0xFFF8000000000000], np.uint64).view(np.float64)[0]
KS = [0, 0.5, 1, 2.7, 5, 32, 33, 100, math.inf, math.nan, NAN_NEG, "largest"]
# NaN payloads of both signs, ±0, ±inf, repeated ordinary numbers (value ties within and across ranks)
VALS = np.concatenate([
    np.array([0x7FF8000000000001, 0xFFF800000000BEEF, 0x7FF4000000000000, 0x8000000000000000, 0x7FF0000000000000,
              0xFFF0000000000000, 0x0000000000000001], np.uint64).view(np.float64),
    np.array([0.0, 1.0, 1.0, -2.5, 1e300, 7.0]),
])


def ranks_of(k):
    """topk_ranks of b2p_aggregation.cu"""
    if math.isnan(k):
        return 0 if math.copysign(1.0, k) < 0 else 2 ** 32 - 1
    if not k >= 1.0:
        return 0
    return 2 ** 32 - 1 if k >= 4294967295.0 else int(math.floor(k))


def grid(seed, T, big=2500):
    """One group of `big` rows (several chunks on one rank), one of 150, 40 groups of 0..9 rows, empty ids between them,
    rows without a valid cell and rows of no group."""
    rng = np.random.default_rng(seed)
    sizes = [big, 150] + list(rng.integers(0, 10, 40))
    gid = np.concatenate([np.full(s, 2 * g, np.uint32) for g, s in enumerate(sizes)])
    n_groups = 2 * len(sizes)
    gid[rng.random(gid.size) < 0.01] = n_groups + 3
    rng.shuffle(gid)
    R = gid.size
    vals = VALS[rng.integers(0, VALS.size, (R, T))]
    spread = rng.random((R, T)) < 0.5
    vals[spread] = rng.standard_normal(int(spread.sum()))
    ok = rng.random((R, T)) < 0.8
    ok[rng.random(R) < 0.05] = False
    tie = rng.permutation(R).astype(np.uint32)
    return vals, ok, gid, n_groups, tie


def owners(n_rows, n_ranks, seed):
    """hashed rows, except that with three ranks the last one holds nothing"""
    from greptimedb_b200 import distributed as D
    own = D.shard_of_series(np.arange(n_rows, dtype=np.uint32) + np.uint32(seed), n_ranks)
    if n_ranks == 3:
        own[own == 2] = 0
    return own


def dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


class Rank:
    """One simulated rank: its own context, rows and group index"""
    def __init__(self, rows, vals, valid, gid, n_groups, tie):
        from greptimedb_b200 import Context
        self.ctx = Context(0)
        self.ctx.use_torch_stream()
        self.rows = rows
        self.vals, self.valid = dev(vals[rows]), dev(valid[rows].view(np.int32))
        self.tie = dev(tie[rows].view(np.int32))
        self.ix = self.ctx.group_index_create_dev(dev(gid[rows].view(np.int32)), rows.size, n_groups)

    def close(self):
        self.ctx.group_index_destroy(self.ix)
        self.ctx.close()


def run_sharded(ranks, op, k, sizes, T):
    """the per-rank / merge / mark steps over the simulated ranks -> (out words per rank, plan, block bytes sent)"""
    import torch
    R = len(ranks)
    c0 = ranks[0].ctx
    plan = c0.topk_shard_plan(k, sizes, T, R)
    state = torch.zeros(max(plan["state_bytes"], 16), dtype=torch.uint8, device="cuda")
    blocks = [torch.zeros(max(plan["block_bytes"], 16), dtype=torch.uint8, device="cuda") for _ in ranks]
    gathered = torch.zeros(max(plan["block_bytes"], 16) * R, dtype=torch.uint8, device="cuda")
    outs = [torch.full_like(r.valid, -1) for r in ranks]
    K = plan["slots"]
    sent = 0
    for b in range(plan["n_batches"]):
        for rnd in range(plan["n_rounds"]):
            nbytes = None
            for r, blk in zip(ranks, blocks):
                r.ctx.topk_shard_candidates_dev(op, k, r.vals, r.valid, r.ix, r.tie, T, sizes, R, b, rnd, state, blk)
                got = r.ctx.last_exchange_bytes()
                assert nbytes in (None, got), "ranks disagree on the block size"
                nbytes = got
            sent += nbytes
            units = nbytes // (32 * (12 * K + 4))
            assert units * 32 * (12 * K + 4) == nbytes and nbytes <= plan["block_bytes"]
            cuts = np.cumsum([0, units * K * 32 * 8, units * K * 32 * 4, units * 32 * 4])
            parts = [blk[cuts[s]:cuts[s + 1]] for s in range(3) for blk in blocks]
            gathered[:R * nbytes] = torch.cat(parts)
            c0.topk_shard_merge_dev(k, sizes, T, R, b, rnd, gathered, state)
        for r, out in zip(ranks, outs):
            r.ctx.topk_shard_mark_dev(op, k, r.vals, r.valid, r.ix, r.tie, T, sizes, R, b, state, out)
    torch.cuda.synchronize()
    return [o.cpu().numpy().view(np.uint32) for o in outs], plan, sent


def expected_bytes(kk, sizes, T):
    """b2p_last_exchange_bytes' formula: rounds x G_x x 32 ceil(T / 32) x (12 slots + 4), 0 without exchanged groups"""
    if kk == 0 or kk >= sizes.max():
        return 0
    X = int((sizes > kk).sum())
    slots = min(kk, 32)
    rounds = 1 if kk <= 32 else -(-kk // 32)
    return rounds * X * 32 * ((T + 31) // 32) * (12 * slots + 4)


def check_case(ranks, full, op, k, vals, ok, gid, n_groups, tie, T):
    import torch
    sizes = np.bincount(gid[gid < n_groups], minlength=n_groups).astype(np.uint32)
    kk = ranks_of(k)
    outs, plan, sent = run_sharded(ranks, op, k, sizes, T)
    union = np.zeros((gid.size, (T + 31) // 32), np.uint32)
    for r, out in zip(ranks, outs):
        union[r.rows] = out
    exp = sk.words(sk.topk(op == "bottomk", kk, vals, ok, gid, n_groups, tie))
    assert (union == exp).all(), (op, k, len(ranks))
    one = torch.full_like(full.valid, -1)
    full.ctx.topk_dev(op, k, full.vals, full.valid, full.ix, full.tie, T, one)
    torch.cuda.synchronize()
    assert (one.cpu().numpy().view(np.uint32) == union).all(), (op, k, len(ranks))
    assert sent == expected_bytes(kk, sizes, T), (op, k)
    assert plan["n_rounds"] == (0 if expected_bytes(kk, sizes, T) == 0 else (1 if kk <= 32 else -(-kk // 32)))


def make_ranks(n_ranks, seed, vals, ok, gid, n_groups, tie):
    valid = sk.words(ok)
    own = owners(gid.size, n_ranks, seed)
    return [Rank(np.flatnonzero(own == r), vals, valid, gid, n_groups, tie) for r in range(n_ranks)]


@pytest.mark.parametrize("n_ranks", [1, 2, 3, 8])
def test_simulated_ranks_match_the_single_rank_selection(n_ranks):
    T = 65
    vals, ok, gid, n_groups, tie = grid(n_ranks, T)
    largest = int(np.bincount(gid[gid < n_groups]).max())
    full = Rank(np.arange(gid.size), vals, sk.words(ok), gid, n_groups, tie)
    ranks = make_ranks(n_ranks, n_ranks, vals, ok, gid, n_groups, tie)
    try:
        for op in ("topk", "bottomk"):
            for k in KS:
                check_case(ranks, full, op, float(largest) if k == "largest" else k, vals, ok, gid, n_groups, tie, T)
    finally:
        for r in ranks + [full]:
            r.close()


def test_adversarial_keys_with_value_ties_across_ranks():
    """select_keys' total-order classes (equal keys, ±0, NaN payloads, sentinels): ties in value across ranks are
    decided by the tie alone"""
    rng = np.random.default_rng(17)
    classes = ("equal", "signed-zero", "payloads", "sentinel-lo0", "sentinel-onlymax", "ulps-inf", "depth7-last")
    T = 40
    vals, ok, gid, n_groups, _ = sk.grid([400, 60, 33, 5, 0, 1], T, 0.5, rng, classes=classes, drop=0.2, gid_gap=2,
                                         stray=4)
    tie = rng.permutation(gid.size).astype(np.uint32)
    full = Rank(np.arange(gid.size), vals, sk.words(ok), gid, n_groups, tie)
    ranks = make_ranks(3, 5, vals, ok, gid, n_groups, tie)
    try:
        for op in ("topk", "bottomk"):
            for k in (1, 2, 5, 32, 33, 70):
                check_case(ranks, full, op, k, vals, ok, gid, n_groups, tie, T)
    finally:
        for r in ranks + [full]:
            r.close()


def test_batches_under_a_small_exchange_cap(monkeypatch):
    """a cap of 64 KB cuts the exchange into batches of groups and tiles; the result does not change"""
    monkeypatch.setenv("B2P_TOPK_EXCHANGE_BYTES", str(64 << 10))
    T = 200
    vals, ok, gid, n_groups, tie = grid(9, T, big=600)
    full = Rank(np.arange(gid.size), vals, sk.words(ok), gid, n_groups, tie)
    ranks = make_ranks(2, 9, vals, ok, gid, n_groups, tie)
    try:
        sizes = np.bincount(gid[gid < n_groups], minlength=n_groups).astype(np.uint32)
        for op, k in (("topk", 1), ("bottomk", 5), ("topk", 33), ("bottomk", 100)):
            assert ranks[0].ctx.topk_shard_plan(k, sizes, T, 2)["n_batches"] > 1, k
            check_case(ranks, full, op, k, vals, ok, gid, n_groups, tie, T)
    finally:
        for r in ranks + [full]:
            r.close()


def composed_check(full, vals, ok, gid, n_groups, tie, T):
    import torch
    sizes = np.bincount(gid[gid < n_groups], minlength=n_groups)
    largest = int(sizes.max())
    for op in ("topk", "bottomk"):
        for k in (0, 1, 5, 33, 100, float(largest), math.inf):
            a = torch.full_like(full.valid, -1)
            b = torch.full_like(full.valid, -1)
            full.ctx.topk_allgather_dev(op, k, full.vals, full.valid, full.ix, full.tie, T, a)
            full.ctx.topk_dev(op, k, full.vals, full.valid, full.ix, full.tie, T, b)
            full.ctx.sync()
            torch.cuda.synchronize()
            assert torch.equal(a, b), (op, k)
            assert full.ctx.last_exchange_bytes() == expected_bytes(ranks_of(k), sizes, T), (op, k)
        inplace = full.valid.clone()
        full.ctx.topk_allgather_dev(op, 5, full.vals, inplace, full.ix, full.tie, T, inplace)
        b = torch.full_like(full.valid, -1)
        full.ctx.topk_dev(op, 5, full.vals, full.valid, full.ix, full.tie, T, b)
        torch.cuda.synchronize()
        assert torch.equal(inplace, b), op


def test_composed_call_without_communicator_is_the_single_rank_topk():
    T = 70
    vals, ok, gid, n_groups, tie = grid(3, T)
    full = Rank(np.arange(gid.size), vals, sk.words(ok), gid, n_groups, tie)
    try:
        composed_check(full, vals, ok, gid, n_groups, tie, T)
        # every group within kk: nothing is exchanged
        full.ctx.topk_allgather_dev("topk", 3000, full.vals, full.valid, full.ix, full.tie, T, full.valid.clone())
        assert full.ctx.last_exchange_bytes() == 0
    finally:
        full.close()


def test_single_rank_communicator_round_trips_the_candidates():
    """Over a one-rank communicator, the composed call over NCCL's all-reduce and all-gather: the words of b2p_topk_dev"""
    T = 70
    vals, ok, gid, n_groups, tie = grid(4, T)
    full = Rank(np.arange(gid.size), vals, sk.words(ok), gid, n_groups, tie)
    try:
        with one_rank_comm(full.ctx):
            composed_check(full, vals, ok, gid, n_groups, tie, T)
    finally:
        full.close()


def test_argument_errors():
    from greptimedb_b200 import B2PError
    vals, ok, gid, n_groups, tie = grid(5, 33)
    full = Rank(np.arange(gid.size), vals, sk.words(ok), gid, n_groups, tie)
    sizes = np.bincount(gid[gid < n_groups], minlength=n_groups).astype(np.uint32)
    try:
        plan = full.ctx.topk_shard_plan(5, sizes, 33, 2)
        with pytest.raises(B2PError):
            full.ctx.topk_shard_merge_dev(5, sizes, 33, 2, plan["n_batches"], 0, full.vals, full.vals)
        with pytest.raises(B2PError):
            full.ctx.topk_shard_merge_dev(5, sizes, 33, 2, 0, plan["n_rounds"], full.vals, full.vals)
        with pytest.raises(B2PError):
            full.ctx.topk_shard_plan(5, sizes, 33, 0)
    finally:
        full.close()
