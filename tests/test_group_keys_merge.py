"""CPU: b2p_group_keys_merge, the host merge of a sharded plan node's group-label agreement, over 1, 2, 3 and 8 simulated
ranks with the shards assigned to the ranks in every rotation.  Every rank's call gives the same table, equal to the host
mirror's (distributed.merge_group_keys) and to group_rows over the union, and maps its own groups to their place in it.
The table carries the rows of all ranks and the field types of the ranks with rows (an empty rank's default types give
way); ranks with rows whose types differ, and malformed blocks, are refused."""
import ctypes as C

import numpy as np
import pytest

from greptimedb_b200 import _lib
from greptimedb_b200 import distributed as D


def rows_of(seed, n):
    """label tuples over (a, b): NULL against "", multi-byte UTF-8, decimal-string ids"""
    rng = np.random.default_rng(seed)
    pool = [None, "", "a", "b", "é", "日本", "\U0001F600", "10", "9", "a\x00b", "zz"]
    return [(pool[rng.integers(len(pool))], pool[rng.integers(len(pool))]) for _ in range(n)]


def merge(blocks, rank):
    L = _lib.load()
    arr = (C.c_void_p * len(blocks))(*[C.cast(C.c_char_p(b), C.c_void_p) for b in blocks])
    keep = list(blocks)  # (the buffers stay alive during the call)
    sizes = (C.c_uint64 * len(blocks))(*[len(b) for b in blocks])
    out = C.create_string_buffer(max(1, sum(len(b) for b in blocks)))
    nbytes, ng = C.c_uint64(), C.c_uint32()
    n_local = int.from_bytes(blocks[rank][:4], "little") if len(blocks[rank]) >= 4 else 0
    l2g = (C.c_uint32 * max(1, n_local))()
    rc = L.b2p_group_keys_merge(arr, sizes, len(blocks), rank, out, C.byref(nbytes), C.byref(ng), l2g)
    del keep
    if rc != 0:
        raise ValueError(L.b2p_plan_last_error().decode())
    return out.raw[:nbytes.value], ng.value, list(l2g)[:n_local]


@pytest.mark.parametrize("R", [1, 2, 3, 8])
@pytest.mark.parametrize("tsid", [False, True])
def test_every_rank_derives_the_same_table(R, tsid):
    rows = rows_of(R, 400)
    ids = {t: i * 7 + 3 for i, t in enumerate(D.group_tuples(rows))}  # one id per tuple, as the metric engine gives
    rng = np.random.default_rng(R)
    owner = D.shard_of_series(np.arange(len(rows), dtype=np.uint32), R)
    owner[rng.random(len(rows)) < 0.2] = 0  # uneven
    if R > 2:
        owner[owner == R - 1] = 0  # and one empty shard
    shards = [D.group_tuples([rows[i] for i in np.flatnonzero(owner == r)]) for r in range(R)]
    union = D.group_tuples(rows)
    for rot in range(R):
        order = [shards[(r + rot) % R] for r in range(R)]
        # a rank with rows read Int64 fields; an empty one kept the Float64 default
        blocks = [D.serialize_group_keys(s, 2, [ids[t] for t in s] if tsid else None, n_rows=3 * len(s),
                                         types=(1, 0) if s else (0, 0)) for s in order]
        tables = set()
        for rank in range(R):
            table, ng, l2g = merge(blocks, rank)
            tables.add(table)
            mt, mids, ml2g, mrows, mtypes = D.merge_group_keys(blocks, rank)
            assert mrows == 3 * sum(len(s) for s in shards) and mtypes == (1, 0)
            assert table == D.serialize_group_keys(mt, 2, mids, n_rows=mrows, types=mtypes)
            assert mt == union and ng == len(union)
            assert [union[g] for g in l2g] == order[rank] and l2g == ml2g
            if tsid:
                assert mids == [ids[t] for t in union]
        assert len(tables) == 1


def test_no_group_columns_and_empty_ranks():
    blocks = [D.serialize_group_keys([()], 0, n_rows=5), D.serialize_group_keys([], 0),
              D.serialize_group_keys([()], 0, n_rows=2)]
    for rank in range(3):
        table, ng, l2g = merge(blocks, rank)
        assert ng == 1 and table == D.serialize_group_keys([()], 0, n_rows=7)
        assert l2g == ([] if rank == 1 else [0])


def test_malformed_blocks_are_refused():
    good = D.serialize_group_keys([("a",), ("b",)], 1)
    unsorted = D.serialize_group_keys([("b",), ("a",)], 1)
    dup = D.serialize_group_keys([("a",), ("a",)], 1)
    other = D.serialize_group_keys([("a", "b")], 2)
    for blocks, text in [([good[:-1]], "truncated"), ([good + b"\0"], "longer"), ([unsorted], "label order"),
                         ([dup], "label order"), ([good, other], "unlike block 0"),
                         ([D.serialize_group_keys([("a",)], 1, [5]), good], "unlike block 0"),
                         ([good, D.serialize_group_keys([("a",)], 1, types=(0,))], "unlike block 0"),
                         ([D.serialize_group_keys([("a",)], 1, types=(1,)), D.serialize_group_keys([("b",)], 1, types=(0,))],
                          "different value types"),
                         ([D.serialize_group_keys([("a",)], 1, n_rows=0)], "rows without groups")]:
        with pytest.raises(ValueError, match=text):
            merge(blocks, 0)


def test_an_empty_rank_takes_the_types_of_the_ranks_with_rows():
    blocks = [D.serialize_group_keys([], 1, types=(0,)), D.serialize_group_keys([("a",)], 1, n_rows=4, types=(1,))]
    for rank in range(2):
        table, ng, _ = merge(blocks, rank)
        assert ng == 1 and table == D.serialize_group_keys([("a",)], 1, n_rows=4, types=(1,))
