"""CPU: the references of tests/shard_edges.py against select_keys and the oracles, and every edge class landing on its
edge by the restated host arithmetic of the sort merge, the count_values plan and cut_batches."""
import collections
import math

import numpy as np

from tests import int64_oracle as i64o
from tests import select_keys as sk
from tests import shard_edges as se
from tests import sort_oracle as so


def test_sort_items_cover_every_tile_size():
    items = {F: se.sort_items(F) for F in se.SORT_FIELDS}
    assert items == {1: 8, 2: 8, 4: 8, 5: 7, 6: 6, 8: 5, 9: 4, 12: 3, 16: 2, 31: 1, 64: 1}
    assert set(items.values()) == set(range(1, 9))
    assert [se.sort_items(F) for F in (10, 11, 14, 15, 22, 23)] == [4, 3, 3, 2, 2, 1]
    # the largest dynamic shared memory request, F = 64, and every request within the 227 KB an H100 CTA may use
    assert se.sort_smem(64) == 134144 == max(se.sort_smem(F) for F in range(1, se.MAX_FIELDS + 1))
    assert all(se.sort_smem(F) <= 227 << 10 for F in range(1, se.MAX_FIELDS + 1))


def test_merge_rounds():
    assert se.merge_rounds([0, 0], 256) == []
    assert se.merge_rounds([5], 256) == [[(5, 0, 0)]]  # one run: one round, a copy
    assert [len(r) for r in se.merge_rounds([1] * 17, 256)] == [9, 5, 3, 2, 1]
    r = se.merge_rounds([300, 0, 256, 1], 256)
    assert r == [[(300, 256, 0), (1, 0, 3)], [(556, 1, 0)]]


def test_sort_cases_reach_every_edge():
    rounds_per_F = collections.defaultdict(set)
    edges, wheres, keys = set(), collections.Counter(), collections.Counter()
    for c in se.sort_cases():
        cap = se.sort_cap(c["F"])
        rounds = se.merge_rounds(c["counts"], cap)
        rounds_per_F[c["F"]].add(len(rounds))
        edges |= {(min(k, 1), e) for k, e in se.tile_edges(rounds, cap)}
        edges |= {(4, e) for k, e in se.tile_edges(rounds, cap) if k == 4}
        assert set(c["counts"]) - {0} <= {1, cap - 1, cap, cap + 1, 2 * cap + 1}
        nz = [i for i, x in enumerate(c["counts"]) if x == 0]
        wheres[("first" if 0 in nz else "") + ("last" if len(c["counts"]) - 1 in nz else "") +
               ("middle" if any(0 < i < len(c["counts"]) - 1 for i in nz) else "")] += 1
        keys[c["keys"], c["desc"]] += 1
    assert all(rounds_per_F[F] == {1, 2, 3, 4, 5} for F in se.SORT_FIELDS)
    for e in ("end-of-a", "past-b", "at-b", "empty-b"):
        assert (0, e) in edges and (1, e) in edges, e  # in the first round and in a later one
    assert (4, "past-b") in edges  # a merge in the fifth round
    assert {"first", "middle", "last", ""} <= set(wheres)
    assert {k for k, _ in keys} == set(se.SORT_KEYS) and all((k, d) in keys for k in se.SORT_KEYS for d in (0, 1))


def test_sort_grids_hold_their_counts():
    for c in se.sort_cases()[::7]:
        grids, ok, owner = se.sort_grid(c)
        assert [int(ok[owner == r].sum()) for r in range(len(c["counts"]))] == c["counts"]
        assert len(grids) == c["F"]


def test_sort_ref_is_the_oracles_order():
    rng = np.random.default_rng(1)
    for c in se.sort_cases()[:40]:
        grids, ok, _ = se.sort_grid(c)
        exp = se.sort_ref(c["desc"], grids, ok, c["keys"] == "i64")
        if c["keys"] == "i64":
            assert exp.tolist() == i64o.value_order(grids[0], ok, c["desc"])
        elif c["F"] == 1:
            assert np.array_equal(exp, so.value_order(grids[0], ok, c["desc"]))
            assert np.array_equal(exp, sk.sort(c["desc"], grids[0], ok))
    # several fields: a stable sort by each field from the last to the first is the lexicographic order
    v = [rng.choice([0.0, -0.0, np.nan, 1.0], (40, 3)) for _ in range(3)]
    ok = rng.random((40, 3)) < 0.8
    for desc in (False, True):
        cells = np.flatnonzero(ok.reshape(-1)).astype(np.uint64)
        for g in v[::-1]:
            k = sk.keys_of_values(g.reshape(-1)[cells.astype(np.int64)])
            cells = cells[np.argsort(~k if desc else k, kind="stable")]
        assert np.array_equal(se.sort_ref(desc, v, ok), cells)


def test_cv_ref_is_select_keys_and_the_int64_oracle():
    for R, T in ((5, 33), (16, 1)):
        vals, ok, gid, G, _ = se.cv_grid(R, T, 3)
        out, cnt = se.cv_ref(vals, ok, gid, G)
        e_out, e_cnt = sk.count_values(vals, ok, gid, G)
        assert sk.same_bits(out, e_out) and (cnt == e_cnt).all()
        ivals, iok, igid, G, _ = se.cv_grid(R, T, 3, i64=True)
        out, cnt = se.cv_ref(ivals, iok, igid, G, i64=True)
        exp = i64o.count_values(ivals, iok, igid, G)
        _, goff = sk._groups(igid, G)
        for (g, k), pairs in exp.items():
            n = goff[g + 1] - goff[g]
            assert [(int(out[goff[g] + j, k]), int(cnt[goff[g] + j, k])) for j in range(len(pairs))] == pairs
            assert (cnt[goff[g] + len(pairs):goff[g] + n, k] == 0).all()


def test_cv_plan_restatement():
    H = np.array([[1, 0, 3], [2, 0, 1]], np.uint32)
    assert se.cv_plan(H, 40, se.DEFAULT_CAP) == [(0, 3, 0, 40, 4 * 40, 7)]  # one window of every step; P from rank 0
    assert se.cv_plan(np.zeros((2, 3), np.uint32), 40, se.DEFAULT_CAP) == []
    b = se.cv_plan(H, 40, 1)  # one group per batch (the empty one left out), windows of 32
    assert b == [(0, 1, 0, 32, 64, 3), (2, 3, 0, 32, 96, 4), (0, 1, 32, 8, 16, 3), (2, 3, 32, 8, 24, 4)]


def test_cv_cases_reach_every_edge():
    seen = collections.defaultdict(set)
    for cap in se.CV_CAPS:
        for s, (R, T) in enumerate(se.cv_cases(cap)):
            for i64 in (False, True):
                vals, ok, gid, G, owner = se.cv_grid(R, T, s, i64)
                H = se.cv_heights(vals, ok, gid, G, owner, R, i64)
                full = 3
                assert H[R - 1, full] == (owner[gid == full] == R - 1).sum()  # height = the rank's member count
                seen[cap, i64] |= se.cv_edges(H, T, cap)
                top = se.I64_MAX if i64 else se.f64([se.MAX_NAN])[0]
                only = gid == 8
                assert (np.ascontiguousarray(vals[only][ok[only]]).view(np.uint64) ==
                        np.array([top]).view(np.uint64)[0]).all()
    for i64 in (False, True):
        assert {"one-rank-first", "one-rank-middle", "one-rank-last", "U=1", "empty-between",
                "mostly-zero-heights"} <= seen[se.DEFAULT_CAP, i64]
        assert {"k0>0", "short-last-window"} <= seen[64 << 10, i64]
        assert {"k0>0", "short-last-window", "one-group-batch"} <= seen[1, i64]
        assert "k0>0" not in seen[se.DEFAULT_CAP, i64]


def test_cut_batches():
    assert se.cut_batches(3, 4, 12) == (3, 4, "all")
    assert se.cut_batches(3, 4, 11) == (3, 3, "tiles")
    assert se.cut_batches(3, 4, 3) == (3, 1, "tiles")
    assert se.cut_batches(3, 4, 2) == (2, 1, "items")


def test_topk_cases_take_every_branch():
    seen = collections.defaultdict(set)
    for R, kk, T, branch in se.topk_cases():
        vals, ok, gid, G, tie, owner = se.topk_grid(R, kk, T, 0)
        sizes = np.bincount(gid, minlength=G)
        X, tiles = int((sizes > kk).sum()), -(-T // 32)
        fit = se.topk_fit(branch, X, tiles)
        plan = se.topk_plan(kk, sizes, T, R, fit * se.topk_unit(R, kk))
        assert plan["branch"] == branch
        xb, tb, _ = se.cut_batches(X, tiles, fit)
        if branch == "tiles" and X > 1:
            assert math.ceil(fit / X) != fit // X  # rounding fit / X up changes the cut
        if branch == "items":
            assert X % xb  # a short last batch of groups
        seen["branch"].add(branch)
        seen["rounds"].add(se.topk_rounds(kk))
        seen["nonzero-tile0"].add(tb < tiles)
        # the group classes: more than kk, at most kk on every rank; exactly kk; kk + 1; ranks without a member
        per_rank = np.bincount(owner[gid == 0], minlength=R).max()
        assert sizes[0] > kk >= per_rank and sizes[1] == kk and sizes[2] == kk + 1 and sizes[4] == 0
        assert sizes[3] > kk and set(owner[gid == 3]) <= {0, 1}
        assert tie.size == np.unique(tie).size
    assert seen["branch"] == set(se.BRANCHES) and seen["rounds"] == {1, 2, 3, 4} and True in seen["nonzero-tile0"]
    assert {(kk, T) for _, kk, T, _ in se.topk_cases()} == {(kk, T) for kk in se.TOPK_KK for T in se.TOPK_STEPS}


def test_quantile_placements():
    for R in (5, 16):
        for per_place in (1, 4):
            vals, ok, gid, G, owner = se.quant_grid(R, 33, 0.5, 1, per_place)
            spans = [np.unique(owner[gid == g]).size for g in range(G)]
            assert spans == [1] * per_place + [R - 1] * per_place + [R] * per_place
            assert (np.bincount(owner[gid == G - 1], minlength=R) == 1).all()
            assert np.isfinite(vals).all()
        assert se.quant_plan(3, 65, se.QUANT_UNIT) == dict(n_batches=9, block_bytes=2560, branch="items")
        assert se.quant_plan(12, 65, se.DEFAULT_CAP)["n_batches"] == 1
