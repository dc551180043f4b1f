"""World-size-2 gloo test (CPU) of the sharded quantile: every rank holds whole series, the host mirror of
b2p_quantile_allreduce_dev (distributed.merge_quantile_digits) all-reduces each pass's 4-bit digit counts, and both
ranks' results equal select_keys.quantile over all rows, bit for bit.  The grids hold select_keys' adversarial classes
and the nibble-depth classes (s[lo] and s[hi] on different ranks), rows of no group and rows without a valid cell; the
shards are hashed, uneven, and one is empty."""
import math

import numpy as np

from tests.ranks import spawn_gloo

PHIS = (math.nan, -0.5, 1.5, 0.0, 1.0, 0.5, 0.99)


def cases():
    """(name, phi, vals, ok, gid, n_groups, owner [R] rank of each row)"""
    from greptimedb_b200 import distributed as D
    from tests import nibble_keys as nk
    from tests import select_keys as sk
    out = []
    for i, phi in enumerate(PHIS):
        rng = np.random.default_rng(0x9A1 + i)
        vals, ok, gid, n_groups, _ = sk.grid([70, 40, 33, 9, 2, 1, 0, 120], 37, phi, rng, drop=0.2, gid_gap=2, stray=5)
        ok[rng.random(gid.size) < 0.05] = False   # rows without a valid cell
        R = gid.size
        hashed = D.shard_of_series(np.arange(R, dtype=np.uint32), 2)
        out.append(("hashed", phi, vals, ok, gid, n_groups, hashed))
        out.append(("uneven", phi, vals, ok, gid, n_groups, (rng.random(R) < 0.1).astype(np.int64)))
        out.append(("rank-1-empty", phi, vals, ok, gid, n_groups, np.zeros(R, np.int64)))
        kphi = phi if 0.0 <= phi <= 1.0 else 0.5
        nv, nok, ngid, ng, nown = nk.grid(6, 4, kphi, lambda r: r % 2, rng)
        out.append(("nibbles", phi, nv, nok, ngid, ng, nown))
    return out


def _worker(rank, world):
    from greptimedb_b200 import distributed as D
    res = []
    for name, phi, vals, ok, gid, n_groups, owner in cases():
        mine = np.flatnonzero(owner == rank)
        res.append(D.merge_quantile_digits(phi, vals[mine], ok[mine], gid[mine], n_groups))
    return res


def test_sharded_quantile_equals_the_unsharded_select():
    from greptimedb_b200 import distributed as D
    from tests import select_keys as sk
    world = 2
    got = spawn_gloo(_worker, world, timeout=600)
    all_cases = cases()
    assert len(all_cases) == 4 * len(PHIS)
    for i, (name, phi, vals, ok, gid, n_groups, owner) in enumerate(all_cases):
        exp, exp_cnt = sk.quantile(phi, vals, ok, gid, n_groups)
        (o0, c0, p0, b0), (o1, c1, p1, b1) = got[0][i], got[1][i]
        assert sk.same_bits(o0, o1) and (c0 == c1).all() and p0 == p1 and b0 == b1, (name, phi)
        assert sk.same_bits(o0, exp), (name, phi)
        assert (c0 == exp_cnt).all(), (name, phi)
        assert 1 <= p0 <= D.QUANT_SHARD_PASSES, (name, phi)
        if not 0.0 <= phi <= 1.0:
            assert p0 == 1, (name, phi)
        assert b0 == p0 * n_groups * ((vals.shape[1] + 31) // 32) * D.QUANT_UNIT_BYTES
