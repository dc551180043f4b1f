"""World-size-2 gloo test (CPU) of the sharded sort: every rank holds some rows of one global grid, in global order, with
their global row ids; the host mirror of b2p_sort_cells_allgather_dev (distributed.merge_sorted_runs) sorts each
rank's valid cells, all-gathers the runs and merges them, and both ranks' global cells and values equal the sort of the
whole grid bit for bit (select_keys.sort and sort_oracle.value_order for one Float64 field, a lexicographic stable sort
for several, signed order for Int64).  Classes: both directions; the total-order specials split across ranks; equal
values on both ranks, whose order the row ids decide; hashed, uneven and empty shards; two and three fields with ties
in field 0 across ranks; Int64 with INT64_MIN and INT64_MAX."""
import numpy as np

from tests.ranks import spawn_gloo

I64_MIN, I64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max


def cases():
    """(name, vals [R, T] or [F grids], ok [R, T], owner [R] rank of each row)"""
    from greptimedb_b200 import distributed as D
    from tests.test_sort_oracle import TOTAL_ORDER
    rng = np.random.default_rng(0x50)
    out = []
    R, T = 90, 37
    spec = np.array(TOTAL_ORDER)[rng.integers(0, len(TOTAL_ORDER), (R, T))]
    ok = rng.random((R, T)) < 0.7
    out.append(("specials-hashed", spec, ok, D.shard_of_series(np.arange(R, dtype=np.uint32), 2)))
    out.append(("specials-uneven", spec, ok, (rng.random(R) < 0.1).astype(np.int64)))
    out.append(("specials-rank-1-empty", spec, ok, np.zeros(R, np.int64)))
    out.append(("specials-alternate", spec, ok, np.arange(R) % 2))
    few = rng.choice([-1.0, 0.0, 2.5], (R, T))                      # equal values on both ranks
    out.append(("equal-values", few, rng.random((R, T)) < 0.9, np.arange(R) // 3 % 2))
    out.append(("no-valid-cell", few, np.zeros((R, T), bool), np.arange(R) % 2))
    R, T = 40, 1
    out.append(("one-step", rng.normal(size=(R, T)), rng.random((R, T)) < 0.8, np.arange(R) % 2))
    # two and three fields, field 0 from few values so its ties span both ranks
    R, T = 60, 9
    f0 = rng.choice([1.0, -0.0, 0.0], (R, T))
    f1 = rng.choice([3.0, np.nan, -np.inf], (R, T))
    f2 = np.array(TOTAL_ORDER)[rng.integers(0, len(TOTAL_ORDER), (R, T))]
    ok = rng.random((R, T)) < 0.85
    own = D.shard_of_series(np.arange(R, dtype=np.uint32) + np.uint32(5), 2)
    out.append(("two-fields", [f0, f1], ok, own))
    out.append(("three-fields", [f0, f1, f2], ok, own))
    # Int64
    R, T = 50, 33
    iv = rng.choice(np.array([I64_MIN, I64_MAX, -1, 0, 1, 7], np.int64), (R, T))
    out.append(("int64-extremes", iv, rng.random((R, T)) < 0.8, D.shard_of_series(np.arange(R, dtype=np.uint32), 2)))
    return out


def expected(desc, vals, ok):
    """(cells, values) of the whole grid, sorted"""
    from tests import select_keys as sk
    from tests import sort_oracle as so
    many = isinstance(vals, list)
    grids = vals if many else [vals]
    cells = np.flatnonzero(ok.reshape(-1))
    if grids[0].dtype == np.int64:
        k = grids[0].reshape(-1)[cells].view(np.uint64) ^ np.uint64(1 << 63)
        order = cells[np.argsort(~k if desc else k, kind="stable")].astype(np.uint64)
    elif not many:
        order = sk.sort(desc, vals, ok)
        assert np.array_equal(order, so.value_order(vals, ok, desc))
    else:
        keys = [sk.keys_of_values(g.reshape(-1)[cells]) for g in grids]
        keys = [~k if desc else k for k in keys]
        order = cells[np.lexsort(keys[::-1])].astype(np.uint64)
    return order, [g.reshape(-1)[order.astype(np.int64)] for g in grids]


def _worker(rank, world):
    from greptimedb_b200 import distributed as D
    res = []
    for name, vals, ok, owner in cases():
        mine = np.flatnonzero(owner == rank)
        local = [v[mine] for v in vals] if isinstance(vals, list) else vals[mine]
        for desc in (False, True):
            res.append(D.merge_sorted_runs(desc, local, ok[mine], mine.astype(np.uint32)))
    return res


def test_sharded_sort_equals_the_sort_of_the_union():
    world = 2
    got = spawn_gloo(_worker, world, timeout=600)
    i = 0
    for name, vals, ok, owner in cases():
        F = len(vals) if isinstance(vals, list) else 1
        for desc in (False, True):
            exp_cells, exp_vals = expected(desc, vals, ok)
            (c0, v0, b0), (c1, v1, b1) = got[0][i], got[1][i]
            i += 1
            v0 = v0 if isinstance(v0, list) else [v0]
            v1 = v1 if isinstance(v1, list) else [v1]
            assert np.array_equal(c0, exp_cells) and np.array_equal(c1, exp_cells), (name, desc)
            for f in range(F):
                assert np.array_equal(v0[f].view(np.uint64), exp_vals[f].view(np.uint64)), (name, desc, f)
                assert np.array_equal(v1[f].view(np.uint64), exp_vals[f].view(np.uint64)), (name, desc, f)
            n = [int(ok[owner == r].sum()) for r in range(world)]
            assert (b0, b1) == (n[0] * 8 * (F + 1), n[1] * 8 * (F + 1)), (name, desc)
    assert i == 2 * len(cases())
