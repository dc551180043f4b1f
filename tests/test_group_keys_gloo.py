"""World-size-2 gloo test (CPU) of a sharded plan node's group-label agreement: each rank holds whole series, takes
group_rows' table over its own rows, and the host mirror (distributed.agree_group_keys: the 8-byte sizes all-gathered,
one broadcast per rank) gives both ranks the same table, equal to group_rows over the union, with each rank's groups
mapped to their place in it.  Classes: hashed, uneven and empty shards; a group on one rank only; NULL against "";
id-keyed children (ids as decimal strings); multi-byte UTF-8; `by` and `without`; __tsid carried."""
import zlib

import numpy as np

from tests.ranks import spawn_gloo

NAMES = ["host", "idc", "zone"]


def cases():
    """(name, series label tuples over NAMES, owner rank of each series, group columns)"""
    from greptimedb_b200 import distributed as D
    rng = np.random.default_rng(0x6B)
    pool = [None, "", "a", "é", "日本", "\U0001F600", "b"]
    series = [tuple(pool[rng.integers(len(pool))] for _ in NAMES) for _ in range(300)]
    hashed = D.shard_of_series(np.arange(len(series), dtype=np.uint32), 2)
    out = []
    for cols in ([0], [1, 0], [0, 1, 2], [], [1, 2]):  # by (host), by (idc, host), all, no modifier, without (host)
        out.append((f"hashed-{cols}", series, hashed, cols))
    out.append(("uneven", series, (rng.random(len(series)) < 0.05).astype(np.int64), [0, 2]))
    out.append(("rank-1-empty", series, np.zeros(len(series), np.int64), [1]))
    out.append(("rank-0-empty", series, np.ones(len(series), np.int64), []))
    one = [("x", "", None), ("x", None, None), ("y", "only-on-1", "z")]
    out.append(("one-rank-only-and-null-vs-empty", one, np.array([0, 0, 1]), [0, 1]))
    ids = [(str(i),) for i in rng.integers(0, 40, 120)]  # an id-keyed child: "10" sorts before "9"
    out.append(("id-keyed", ids, D.shard_of_series(np.arange(len(ids), dtype=np.uint32), 2), [0]))
    return out


def _worker(rank, world):
    from greptimedb_b200 import distributed as D
    res = []
    for name, series, owner, cols in cases():
        mine = D.group_tuples([tuple(series[i][c] for c in cols) for i in np.flatnonzero(owner == rank)])
        res.append((mine,) + D.agree_group_keys(mine, len(cols)))
        ids = [zlib.crc32(repr(t).encode()) for t in mine]  # one id per full tuple, whichever rank holds it
        res.append((mine,) + D.agree_group_keys(mine, len(cols), ids))
    return res


def test_agreement_equals_group_rows_over_the_union():
    from greptimedb_b200 import distributed as D
    world = 2
    got = spawn_gloo(_worker, world, timeout=600)
    for i, (name, series, owner, cols) in enumerate(cases()):
        union = D.group_tuples([tuple(t[c] for c in cols) for t in series])
        for j in (2 * i, 2 * i + 1):
            (m0, t0, i0, l0, b0), (m1, t1, i1, l1, b1) = got[0][j], got[1][j]
            assert t0 == t1 == union, name
            assert i0 == i1, name
            if j % 2:
                assert i0 == [zlib.crc32(repr(t).encode()) for t in union], name
            assert [union[g] for g in l0] == m0 and [union[g] for g in l1] == m1, name
            assert b0 == len(D.serialize_group_keys(m0, len(cols), None if j % 2 == 0 else [0] * len(m0))), name
