"""World-size-2 gloo test (CPU) of the sharded histogram_quantile: the host mirror of b2p_histogram_fold_allgather
(distributed.histogram_fold_sharded) over bucket rows sharded by series hash (histograms split across the ranks) and
by histogram (each whole on one rank) gives both ranks the same rows, equal to oracle.histogram_fold_rows over the
ranks' rows concatenated in rank order.  By histogram, no bucket row is sent: a rank's bytes are its result block."""
import numpy as np
import pytest

from tests.ranks import spawn_gloo

BOUNDS = ["0.05", "0.1", "0.25", "0.5", "1", "2.5", "5", "+Inf"]
T = 37


def table(seed):
    """[(tags, le label, counters [T], ok [T])]: 11 histograms over (job, instance) with their bucket series; a few
    cells missing on every bucket at once (the fold then has no row at that step)"""
    rng = np.random.default_rng(seed)
    rows = []
    for h in range(11):
        tags = (f"job{h % 3}", f"i{h}")
        gap = rng.random(T) < 0.1
        base = np.sort(rng.random((len(BOUNDS), T)) * 100, axis=0)
        for b, le in enumerate(BOUNDS):
            rows.append((tags, le, base[b], ~gap))
    return rows


def sharding(rows, hid, layout, world):
    """each row's rank: by series hash, or by histogram"""
    from greptimedb_b200 import distributed as D
    if layout == "series":
        return D.shard_of_series(np.arange(len(rows), dtype=np.uint32), world)
    return np.array([hid[r[0]] % world for r in rows])


def _worker(rank, world, layout, seed):
    from greptimedb_b200 import distributed as D
    from oracle.oracle import parse_f64_rust
    rows = table(seed)
    hists = sorted({r[0] for r in rows})
    hid = {t: i for i, t in enumerate(hists)}
    owner = sharding(rows, hid, layout, world)
    mine = [r for r, o in zip(rows, owner) if o == rank]
    rates = np.array([r[2] for r in mine]).reshape(len(mine), T)
    ok = np.array([r[3] for r in mine]).reshape(len(mine), T)
    return D.histogram_fold_sharded(0.9, rates, ok, [hid[r[0]] for r in mine], [parse_f64_rust(r[1]) for r in mine],
                                    len(hists))


@pytest.mark.parametrize("layout", ["series", "histogram"])
def test_mirror_equals_the_fold_over_the_concatenation(layout):
    from greptimedb_b200 import distributed as D
    from oracle.oracle import histogram_fold_rows, parse_f64_rust
    seed = 7
    got = spawn_gloo(_worker, 2, args=(layout, seed))
    assert np.array_equal(got[0][0], got[1][0], equal_nan=True) and np.array_equal(got[0][1], got[1][1])
    rows = table(seed)
    hists = sorted({r[0] for r in rows})
    # scan order of the reference: (tags, ts, le); a step without any bucket has no row
    scan = sorted(((r[0], k, r[1], float(r[2][k])) for r in rows for k in range(T) if r[3][k]),
                  key=lambda x: (x[0], x[1], parse_f64_rust(x[2])))
    want = {(t, k): v for t, k, v in histogram_fold_rows(scan, 0.9)}
    out, ok = got[0][0], got[0][1]
    for h, tags in enumerate(hists):
        for k in range(T):
            assert ok[h, k] == ((tags, k) in want)
            if ok[h, k]:
                assert out[h, k] == pytest.approx(want[(tags, k)], rel=1e-12, nan_ok=True)
    # bytes sent: each rank's rows of histograms it does not own with their headers, and its result block
    hid = {t: i for i, t in enumerate(hists)}
    rank_of_row = sharding(rows, hid, layout, 2)
    row_hist = np.array([hid[r[0]] for r in rows])
    counts = np.stack([np.bincount(row_hist[rank_of_row == r], minlength=len(hists)) for r in range(2)])
    owners = D.histogram_owners(counts)
    block, row = 8 * T + 4 * ((T + 31) // 32), 8 * T + 4 * ((T + 31) // 32) + D.HIST_HEADER_BYTES
    for r in range(2):
        n_sent = int(np.count_nonzero((rank_of_row == r) & (owners[row_hist] != r)))
        assert got[r][2] == n_sent * row + int(np.count_nonzero(owners == r)) * block
        if layout == "histogram":
            assert n_sent == 0  # whole histograms: only the result block
        else:
            assert n_sent > 0
