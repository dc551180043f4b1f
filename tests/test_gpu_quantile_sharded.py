"""GPU: quantile(phi) by label over rows sharded across ranks (b2p_quantile_shard_* and b2p_quantile_allreduce_dev).  R
ranks are simulated on one GPU, one context each, through the per-rank and merge entry points: per batch and pass each
rank writes its block, the blocks are concatenated (each rank merges them in its own order), and every rank advances
its own state from them.  Every rank's result must equal b2p_group_quantile_dev over all rows, bit for bit, and
select_keys.quantile."""
import math

import numpy as np
import pytest

from tests import nibble_keys as nk
from tests import select_keys as sk
from tests.ranks import one_rank_comm

pytestmark = pytest.mark.gpu

PHIS = (math.nan, -0.5, 1.5, 0.0, 1.0, 0.5, 0.99)
PASSES = 17        # sixteen 4-bit digits and the extreme pass
UNIT_BYTES = 2560  # block bytes per (group, 32-step tile) unit and pass


def dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


class Rank:
    """One simulated rank: its own context, rows and group index"""
    def __init__(self, rows, vals, valid, gid, n_groups):
        from greptimedb_b200 import Context
        self.ctx = Context(0)
        self.ctx.use_torch_stream()
        self.rows = rows
        self.vals, self.valid = dev(vals[rows]), dev(valid[rows].view(np.int32))
        self.ix = self.ctx.group_index_create_dev(dev(gid[rows].view(np.int32)), rows.size, n_groups)

    def close(self):
        self.ctx.group_index_destroy(self.ix)
        self.ctx.close()


def make_ranks(owner, n_ranks, vals, ok, gid, n_groups):
    valid = sk.words(ok)
    return [Rank(np.flatnonzero(owner == r), vals, valid, gid, n_groups) for r in range(n_ranks)]


def hashed(n_rows, n_ranks, seed):
    """hashed rows, except that with three ranks the last one holds nothing"""
    from greptimedb_b200 import distributed as D
    own = D.shard_of_series(np.arange(n_rows, dtype=np.uint32) + np.uint32(seed), n_ranks)
    if n_ranks == 3:
        own[own == 2] = 0
    return own


def run_sharded(ranks, phi, n_groups, T):
    """plan -> per batch and pass: every rank's block, then every rank's advance over the concatenated blocks.
    -> ([(out_val, out_cnt)] per rank, passes run per batch, [block bytes] per batch, plan)"""
    import torch
    R = len(ranks)
    plan = ranks[0].ctx.quantile_shard_plan(n_groups, T)
    blocks = [torch.zeros(max(plan["block_bytes"], 16), dtype=torch.uint8, device="cuda") for _ in ranks]
    outs = [(torch.full((n_groups * T,), math.nan, dtype=torch.float64, device="cuda"),
             torch.full((n_groups * T,), -1, dtype=torch.int32, device="cuda")) for _ in ranks]
    passes, sizes = [], []
    for b in range(plan["n_batches"]):
        for p in range(PASSES):
            nbytes = None
            for r, blk in zip(ranks, blocks):
                r.ctx.quantile_shard_pass_dev(phi, r.vals, r.valid, r.ix, T, b, p, blk)
                got = r.ctx.last_exchange_bytes()
                assert nbytes in (None, got), "ranks disagree on the block size"
                nbytes = got
            assert nbytes % UNIT_BYTES == 0 and 0 < nbytes <= plan["block_bytes"]
            lives = []
            for i, (r, (ov, oc)) in enumerate(zip(ranks, outs)):
                order = [blocks[(i + j) % R][:nbytes] for j in range(R)]  # each rank merges in its own order
                lives.append(r.ctx.quantile_shard_advance_dev(phi, n_groups, T, b, p, torch.cat(order), R, ov, oc))
            assert len(set(lives)) == 1, lives
            if lives[0] == 0:
                passes.append(p + 1)
                sizes.append(nbytes)
                break
        else:
            pytest.fail(f"batch {b} did not finish in {PASSES} passes")
    torch.cuda.synchronize()
    return [(ov.cpu().numpy().reshape(n_groups, T), oc.cpu().numpy().view(np.uint32).reshape(n_groups, T))
            for ov, oc in outs], passes, sizes, plan


def single_rank(full, phi, n_groups, T):
    import torch
    ov = torch.full((n_groups * T,), math.nan, dtype=torch.float64, device="cuda")
    oc = torch.full((n_groups * T,), -1, dtype=torch.int32, device="cuda")
    full.ctx.group_quantile_dev(phi, full.vals, full.valid, full.ix, T, ov, oc)
    torch.cuda.synchronize()
    return ov.cpu().numpy().reshape(n_groups, T), oc.cpu().numpy().view(np.uint32).reshape(n_groups, T)


def check_case(ranks, full, phi, vals, ok, gid, n_groups, T, finite=False):
    """-> passes run per batch"""
    outs, passes, sizes, plan = run_sharded(ranks, phi, n_groups, T)
    one, one_cnt = single_rank(full, phi, n_groups, T)
    exp, exp_cnt = sk.quantile(phi, vals, ok, gid, n_groups)
    assert (one_cnt == exp_cnt).all() and sk.same_or_nan(one, exp), phi
    for out, cnt in outs:
        assert (cnt == exp_cnt).all(), (phi, len(ranks))
        assert sk.same_bits(out, one), (phi, len(ranks))
        if finite:  # no NaN from the arithmetic: the reference's bits too
            assert sk.same_bits(out, exp), (phi, len(ranks))
    assert len(passes) == plan["n_batches"] and all(1 <= p <= PASSES for p in passes)
    assert sum(s // UNIT_BYTES for s in sizes) == n_groups * ((T + 31) // 32)  # every unit in one batch
    if not 0.0 <= phi <= 1.0:
        assert set(passes) == {1}, passes
    return passes, sizes


def mixed_grid(seed, T, big=5000):
    """one group large enough for several chunks on each of 8 ranks, groups absent on some ranks, groups of one
    member, empty groups, rows of no group and rows without a valid cell; every select_keys class"""
    rng = np.random.default_rng(seed)
    sizes = [big, 150, 1, 1, 3, 0, 9, 40, 2, 65, 1, 7]
    vals, ok, gid, n_groups, _ = sk.grid(sizes, T, 0.5, rng, drop=0.2, gid_gap=2, stray=6)
    ok[rng.random(gid.size) < 0.03] = False
    return vals, ok, gid, n_groups


@pytest.mark.parametrize("n_ranks", [1, 2, 3, 8])
def test_simulated_ranks_match_the_single_rank_select(n_ranks):
    T = 37
    vals, ok, gid, n_groups = mixed_grid(n_ranks, T)
    full = Rank(np.arange(gid.size), vals, sk.words(ok), gid, n_groups)
    ranks = make_ranks(hashed(gid.size, n_ranks, n_ranks), n_ranks, vals, ok, gid, n_groups)
    try:
        for phi in PHIS:
            check_case(ranks, full, phi, vals, ok, gid, n_groups, T)
    finally:
        for r in ranks + [full]:
            r.close()


@pytest.mark.parametrize("T", [1, 1000])
def test_step_counts(T):
    rng = np.random.default_rng(T)
    vals, ok, gid, n_groups, _ = sk.grid([300, 20, 1, 0, 4], T, 0.5, rng, drop=0.1, stray=2)
    full = Rank(np.arange(gid.size), vals, sk.words(ok), gid, n_groups)
    ranks = make_ranks(hashed(gid.size, 2, T), 2, vals, ok, gid, n_groups)
    try:
        for phi in (math.nan, 0.0, 0.5, 0.99, 1.0):
            check_case(ranks, full, phi, vals, ok, gid, n_groups, T)
    finally:
        for r in ranks + [full]:
            r.close()


def test_no_groups():
    import torch
    rng = np.random.default_rng(2)
    vals, ok = rng.standard_normal((5, 40)), np.ones((5, 40), bool)
    gid = np.full(5, 3, np.uint32)  # rows of no group
    full = Rank(np.arange(5), vals, sk.words(ok), gid, 0)
    try:
        assert full.ctx.quantile_shard_plan(0, 40) == {"n_batches": 0, "block_bytes": 0, "state_bytes": 0}
        out = torch.zeros(1, dtype=torch.float64, device="cuda")
        cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
        full.ctx.quantile_allreduce_dev(0.5, full.vals, full.valid, full.ix, 40, out, cnt)
        assert full.ctx.last_exchange_bytes() == 0
    finally:
        full.close()


@pytest.mark.parametrize("n_ranks", [2, 8])
def test_nibble_depth_classes_split_across_ranks(n_ranks):
    """every 4-bit depth 0-15 x adjacent / gap / first / last, s[lo] and s[hi] on different ranks and the rest of
    their bins on every rank: one bin's count at the cum == k and cum + c == k + 1 boundaries comes from several ranks"""
    T = 6
    for phi in (0.0, 0.5, 0.99, 1.0):
        rng = np.random.default_rng(int(phi * 100) + n_ranks)
        vals, ok, gid, n_groups, owner = nk.grid(16, T, phi, lambda r: r % n_ranks, rng)
        full = Rank(np.arange(gid.size), vals, sk.words(ok), gid, n_groups)
        ranks = make_ranks(owner, n_ranks, vals, ok, gid, n_groups)
        try:
            check_case(ranks, full, phi, vals, ok, gid, n_groups, T, finite=True)
        finally:
            for r in ranks + [full]:
                r.close()


def test_pass_counts():
    """equal keys run every one of the 16 digit passes; a phi outside [0, 1] exactly one"""
    rng = np.random.default_rng(11)
    T = 33
    vals, ok, gid, n_groups, _ = sk.grid([50, 7, 2], T, 0.5, rng, classes=("equal",))
    full = Rank(np.arange(gid.size), vals, sk.words(ok), gid, n_groups)
    ranks = make_ranks(hashed(gid.size, 2, 1), 2, vals, ok, gid, n_groups)
    try:
        passes, _ = check_case(ranks, full, 0.5, vals, ok, gid, n_groups, T, finite=True)
        assert passes == [16]
        for phi in (math.nan, -0.5, 1.5):
            assert check_case(ranks, full, phi, vals, ok, gid, n_groups, T)[0] == [1]
    finally:
        for r in ranks + [full]:
            r.close()


def test_batches_under_a_small_exchange_cap(monkeypatch):
    """a cap of 64 KB cuts the units into batches of groups and tiles; the result does not change"""
    monkeypatch.setenv("B2P_TOPK_EXCHANGE_BYTES", str(64 << 10))
    T = 200
    vals, ok, gid, n_groups = mixed_grid(9, T, big=700)
    full = Rank(np.arange(gid.size), vals, sk.words(ok), gid, n_groups)
    ranks = make_ranks(hashed(gid.size, 2, 9), 2, vals, ok, gid, n_groups)
    try:
        assert ranks[0].ctx.quantile_shard_plan(n_groups, T)["n_batches"] > 1
        for phi in (0.5, 0.99, math.nan):
            passes, sizes = check_case(ranks, full, phi, vals, ok, gid, n_groups, T)
            assert len(passes) > 1
    finally:
        for r in ranks + [full]:
            r.close()


def composed_check(full, vals, ok, gid, n_groups, T):
    import torch
    for phi in PHIS:
        ov = torch.full((n_groups * T,), math.nan, dtype=torch.float64, device="cuda")
        oc = torch.full((n_groups * T,), -1, dtype=torch.int32, device="cuda")
        full.ctx.quantile_allreduce_dev(phi, full.vals, full.valid, full.ix, T, ov, oc)
        torch.cuda.synchronize()
        one, one_cnt = single_rank(full, phi, n_groups, T)
        assert sk.same_bits(ov.cpu().numpy().reshape(n_groups, T), one), phi
        assert (oc.cpu().numpy().view(np.uint32).reshape(n_groups, T) == one_cnt).all(), phi
        sent = full.ctx.last_exchange_bytes()
        _, passes, sizes, _ = run_sharded([full], phi, n_groups, T)  # the same passes, step by step
        assert sent == sum(p * s for p, s in zip(passes, sizes)), phi


def test_composed_call_without_communicator_is_the_single_rank_quantile():
    T = 70
    vals, ok, gid, n_groups = mixed_grid(3, T, big=3000)
    full = Rank(np.arange(gid.size), vals, sk.words(ok), gid, n_groups)
    try:
        composed_check(full, vals, ok, gid, n_groups, T)
    finally:
        full.close()


def test_single_rank_communicator_round_trips_the_counts():
    """Over a one-rank communicator, the composed call over NCCL's all-reduces: the output of b2p_group_quantile_dev"""
    T = 70
    vals, ok, gid, n_groups = mixed_grid(4, T, big=3000)
    full = Rank(np.arange(gid.size), vals, sk.words(ok), gid, n_groups)
    try:
        with one_rank_comm(full.ctx):
            composed_check(full, vals, ok, gid, n_groups, T)
    finally:
        full.close()


def test_argument_errors():
    import torch
    from greptimedb_b200 import B2PError
    T = 33
    vals, ok, gid, n_groups = mixed_grid(5, T, big=300)
    full = Rank(np.arange(gid.size), vals, sk.words(ok), gid, n_groups)
    try:
        plan = full.ctx.quantile_shard_plan(n_groups, T)
        blk = torch.zeros(plan["block_bytes"], dtype=torch.uint8, device="cuda")
        ov = torch.zeros(n_groups * T, dtype=torch.float64, device="cuda")
        oc = torch.zeros(n_groups * T, dtype=torch.int32, device="cuda")
        with pytest.raises(B2PError):  # before any pass 0 on this context
            full.ctx.quantile_shard_advance_dev(0.5, n_groups, T, 0, 0, blk, 1, ov, oc)
        with pytest.raises(B2PError):
            full.ctx.quantile_shard_pass_dev(0.5, full.vals, full.valid, full.ix, T, plan["n_batches"], 0, blk)
        with pytest.raises(B2PError):
            full.ctx.quantile_shard_pass_dev(0.5, full.vals, full.valid, full.ix, T, 0, PASSES, blk)
        full.ctx.quantile_shard_pass_dev(0.5, full.vals, full.valid, full.ix, T, 0, 0, blk)
        with pytest.raises(B2PError):
            full.ctx.quantile_shard_advance_dev(0.5, n_groups, T, 0, 0, blk, 0, ov, oc)
        with pytest.raises(B2PError):
            full.ctx.quantile_shard_advance_dev(0.5, n_groups, T, plan["n_batches"], 0, blk, 1, ov, oc)
    finally:
        full.close()
