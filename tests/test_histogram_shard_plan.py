"""CPU-only: the host steps of the sharded histogram_quantile (b2p_histogram_shard_owners, b2p_histogram_shard_index)
over 1, 2, 3 and 8 simulated ranks, in every rotation of the ranks.  The owner's index, built from the headers of its
own and its received bucket rows in any arrival order, must be the unsharded index over the ranks' rows concatenated in
rank order: histograms in order, bounds ascending with NaN last, ties in (rank, row) order."""
import math

import numpy as np
import pytest

from greptimedb_b200 import B2PError, Context
from greptimedb_b200.distributed import histogram_owners
from oracle.oracle import parse_f64_rust

LE = ["0.1", "0.5", "1", "1.0", "5", "+Inf", "Inf", None, "bogus", "-1", "2.5e0"]


def owners_ref(counts):
    """the rank with the most buckets, the lowest on a tie"""
    R, H = counts.shape
    out = np.zeros(H, np.int64)
    for h in range(H):
        for r in range(R):
            if counts[r, h] > counts[out[h], h]:
                out[h] = r
    return out


def unsharded_order(hist, le):
    """the plan layer's histogram_index order before it was shared: a stable sort of the rows by (histogram, NaN last,
    bound)"""
    def key(i):
        return (hist[i], math.isnan(le[i]), 0.0 if math.isnan(le[i]) else le[i])
    return sorted(range(len(hist)), key=key)


def shards(rng, n_ranks, n_hist, layout):
    """each rank's bucket rows as (histogram, le label): by series hash (a histogram's buckets spread over the ranks) or
    by histogram (each histogram whole on one rank); some ranks may hold nothing"""
    rows = [[] for _ in range(n_ranks)]
    for h in range(n_hist):
        whole = int(rng.integers(n_ranks))
        for le in rng.choice(LE, size=int(rng.integers(1, 7)), replace=True):
            r = whole if layout == "histogram" else int(rng.integers(n_ranks))
            rows[r].append((h, le))
    if n_ranks > 2:
        rows[int(rng.integers(n_ranks))] = []  # a rank without rows
    return rows


def counts_of(rows, n_hist):
    return np.array([np.bincount([h for h, _ in rr], minlength=n_hist) for rr in rows], np.uint32).reshape(len(rows),
                                                                                                           n_hist)


@pytest.mark.parametrize("n_ranks", [1, 2, 3, 8])
@pytest.mark.parametrize("layout", ["series", "histogram"])
def test_owners_and_owner_index_in_every_rotation(n_ranks, layout):
    rng = np.random.default_rng(100 * n_ranks + (layout == "series"))
    H = 23
    base = shards(rng, n_ranks, H, layout)
    for rot in range(n_ranks):
        rows = base[rot:] + base[:rot]
        counts = counts_of(rows, H)
        owner = Context.histogram_shard_owners(counts)
        assert owner.tolist() == owners_ref(counts).tolist() == histogram_owners(counts).tolist()
        # the concatenation in rank order, and the unsharded index over it
        cat = [(h, le, r, i) for r, rr in enumerate(rows) for i, (h, le) in enumerate(rr)]
        c_hist = np.array([c[0] for c in cat], np.uint32)
        c_le = np.array([parse_f64_rust(c[1]) for c in cat], np.float64)
        off, bs, ble = Context.histogram_shard_index(c_hist, c_le, np.zeros(len(cat)), np.arange(len(cat)), H)
        assert bs.tolist() == unsharded_order(c_hist.tolist(), c_le.tolist())
        assert np.array_equal(ble, c_le[bs], equal_nan=True)
        assert off.tolist() == np.concatenate([[0], np.cumsum(np.bincount(c_hist, minlength=H))]).tolist()
        moved = 0
        for me in range(n_ranks):
            # the owner's buckets: its own rows first, then the received ones in an arbitrary arrival order
            own = [c for c in cat if c[2] == me and owner[c[0]] == me]
            got = [c for c in cat if c[2] != me and owner[c[0]] == me]
            moved += len(got)
            rng.shuffle(got)
            buf = own + got
            mh = sorted({int(h) for h in np.flatnonzero(owner == me)})
            local = {h: i for i, h in enumerate(mh)}
            o_off, o_bs, o_le = Context.histogram_shard_index(
                [local[c[0]] for c in buf], [parse_f64_rust(c[1]) for c in buf], [c[2] for c in buf],
                [c[3] for c in buf], len(mh))
            # ... is the unsharded index restricted to this owner's histograms
            want = [(c_hist[j], cat[j][2], cat[j][3]) for j in bs if owner[c_hist[j]] == me]
            assert [(mh[local[buf[k][0]]], buf[k][2], buf[k][3]) for k in o_bs] == [(int(h), r, i) for h, r, i in want]
            assert np.array_equal(o_le, np.array([c_le[j] for j in bs if owner[c_hist[j]] == me]), equal_nan=True)
            assert o_off[-1] == len(buf)
        if layout == "histogram":
            assert moved == 0  # whole histograms: no bucket row leaves its rank


def test_owner_ties_go_to_the_lowest_rank():
    counts = np.array([[2, 0, 1, 0], [2, 3, 1, 0], [1, 3, 1, 0]], np.uint32)
    assert Context.histogram_shard_owners(counts).tolist() == [0, 1, 0, 0]


def test_equal_bounds_on_different_ranks_order_by_rank_then_row():
    # "1" and "1.0" parse alike; -0.0 ties +0.0; NULL and unparsable are NaN, last, still in (rank, row) order
    le = [parse_f64_rust(x) for x in ["1.0", "1", "+Inf", None, "0", "-0", "bogus", "1"]]
    rank = [1, 0, 0, 2, 1, 0, 0, 0]
    row = [0, 5, 1, 0, 3, 2, 9, 0]
    off, bs, _ = Context.histogram_shard_index(np.zeros(8), le, rank, row, 1)
    assert off.tolist() == [0, 8]
    assert [(rank[i], row[i]) for i in bs] == [(0, 2), (1, 3), (0, 0), (0, 5), (1, 0), (0, 1), (0, 9), (2, 0)]


def test_missing_inf_and_empty_histograms_keep_their_place():
    le = [parse_f64_rust(x) for x in ["5", "1"]]
    off, bs, ble = Context.histogram_shard_index([2, 2], le, [0, 0], [0, 1], 4)
    assert off.tolist() == [0, 0, 0, 2, 2]
    assert bs.tolist() == [1, 0] and ble.tolist() == [1.0, 5.0]
    off, bs, ble = Context.histogram_shard_index([], [], [], [], 3)
    assert off.tolist() == [0, 0, 0, 0] and bs.size == 0


def test_index_and_owners_refuse_bad_arguments():
    with pytest.raises(B2PError):
        Context.histogram_shard_index([3], [1.0], [0], [0], 3)
    with pytest.raises(B2PError):
        Context.histogram_shard_owners(np.zeros((0, 4), np.uint32))
