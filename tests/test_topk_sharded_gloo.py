"""World-size-2 gloo test (CPU) of the sharded topk / bottomk exchange: every rank holds whole series, the host mirror
of b2p_topk_allgather_dev (distributed.merge_topk_candidates) exchanges candidates, and the union of the ranks' kept
cells equals select_keys.topk over all rows.  The grids hold adversarial total-order keys (NaN payloads of both signs,
±0, ±inf, sentinel and equal-key columns) with value ties across ranks; the shards are hashed, uneven, and empty."""
import numpy as np

from tests.ranks import spawn_gloo

KKS = (0, 1, 2, 5, 32, 33, 70)


def cases():
    """(name, vals, ok, gid, n_groups, tie, owner [R] rank of each row, slots_max)"""
    from greptimedb_b200 import distributed as D
    from tests import select_keys as sk
    out = []
    rng = np.random.default_rng(0x70B)
    classes = ("equal", "signed-zero", "payloads", "sentinel-lo0", "sentinel-onlymax", "ulps-inf", "depth3-adjacent",
               "depth7-last", "top")
    sizes = [300, 90, 40, 33, 6, 1, 0, 70]
    vals, ok, gid, n_groups, _ = sk.grid(sizes, 37, 0.5, rng, classes=classes, drop=0.2, gid_gap=2, stray=5)
    R = gid.size
    tie = rng.permutation(R).astype(np.uint32)
    hashed = D.shard_of_series(np.arange(R, dtype=np.uint32), 2)
    out.append(("hashed", vals, ok, gid, n_groups, tie, hashed, 32))
    out.append(("hashed-3-slots", vals, ok, gid, n_groups, tie, hashed, 3))
    uneven = (rng.random(R) < 0.1).astype(np.int64)          # rank 1 holds a tenth
    out.append(("uneven", vals, ok, gid, n_groups, tie, uneven, 32))
    out.append(("rank-1-empty", vals, ok, gid, n_groups, tie, np.zeros(R, np.int64), 32))
    # equal values on both ranks: only the tie decides
    vals2 = np.where(rng.random(vals.shape) < 0.7, 1.0, vals)
    out.append(("value-ties", vals2, ok, gid, n_groups, tie, hashed, 32))
    return out


def _worker(rank, world):
    from greptimedb_b200 import distributed as D
    res = {}
    for name, vals, ok, gid, n_groups, tie, owner, slots in cases():
        mine = np.flatnonzero(owner == rank)
        for bottom in (False, True):
            largest = int(np.bincount(gid[gid < n_groups], minlength=n_groups).max())
            for kk in KKS + (largest,):
                kept, X, rounds, K = D.merge_topk_candidates(bottom, kk, vals[mine], ok[mine], gid[mine], n_groups,
                                                             tie[mine], slots_max=slots)
                res[(name, bottom, kk)] = (mine, kept, X, rounds, K)
    return res


def test_sharded_topk_union_equals_the_unsharded_selection():
    from tests import select_keys as sk
    world = 2
    got = spawn_gloo(_worker, world, timeout=300)
    checked = 0
    for name, vals, ok, gid, n_groups, tie, owner, slots in cases():
        sizes = np.bincount(gid[gid < n_groups], minlength=n_groups)
        for bottom in (False, True):
            for kk in KKS + (int(sizes.max()),):
                exp = sk.topk(bottom, kk, vals, ok, gid, n_groups, tie)
                union = np.zeros_like(exp)
                for r in range(world):
                    mine, kept, X, rounds, K = got[r][(name, bottom, kk)]
                    union[mine] |= kept
                    assert X == (int((sizes > kk).sum()) if 0 < kk < sizes.max() else 0), (name, kk)
                    assert rounds == (0 if X == 0 else -(-kk // slots)), (name, kk)
                assert (union == exp).all(), (name, bottom, kk)
                checked += 1
    assert checked == 5 * 2 * 8
