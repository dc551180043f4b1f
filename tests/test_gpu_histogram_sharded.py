"""GPU: histogram_quantile over series sharded across ranks.  Over a one-rank communicator the sharded node and the
sharded leaf export the unsharded bytes, and the composed b2p_histogram_fold_allgather equals b2p_histogram_fold.  R = 2,
3 and 8 simulated ranks on one GPU, through the step entry points (owners, the row move, the owner's index) with torch
copies standing in for NCCL, give bit for bit the fold over the ranks' rows concatenated in rank order, sharded by series
hash (histograms split) and by histogram (whole).  The row-move kernel at its edges, and the refusals."""
import numpy as np
import pyarrow as pa
import pytest
import torch

from tests.binary_oracle import _words
from tests.ranks import one_rank_comm
from tests.test_gpu_histogram_node import END, HISTS, LES, START, STEP, histograms, leaf, table_batch
from tests.test_gpu_plan_sharded import same_export

pytestmark = pytest.mark.gpu
LE_CHOICES = ["0.1", "0.5", "1", "1.0", "2.5", "10", "+Inf", "Inf", "+Inf", None, "bogus"]


@pytest.fixture(scope="module")
def ctxs():
    """(plain context, context with a one-rank communicator)"""
    from greptimedb_b200 import Context
    plain, comm = Context(0), Context(0)
    with one_rank_comm(comm):
        yield plain, comm
    comm.close()
    plain.close()


def bucket_rows(rng, n_hist=40, T=45):
    """a [rows x T] grid of bucket counters with each row's histogram and parsed bound: 1 to 70 buckets per histogram
    (past 64: K5's wide walk), duplicate bounds ("1" and "1.0"), NULL and unparsable bounds, sometimes no +Inf, cells
    missing at some steps, NaN counters; rows in a shuffled order"""
    from oracle.oracle import parse_f64_rust
    hist, le = [], []
    for h in range(n_hist):
        n = int(rng.choice([1, 2, 5, 12, 64, 65, 70])) if h % 4 == 0 else int(rng.integers(1, 14))
        hist += [h] * n
        le += [parse_f64_rust(x) for x in rng.choice(LE_CHOICES, size=n)]
    R = len(hist)
    rates = np.cumsum(rng.random((R, T)) * 3.0, axis=1)
    rates[rng.random((R, T)) < 0.03] = np.nan
    ok = rng.random((R, T)) < 0.9
    ok[:, 7] = False  # a step no bucket has
    rates[~ok] = 0.0
    perm = rng.permutation(R)
    return rates[perm], _words(ok[perm]), np.array(hist, np.uint32)[perm], np.array(le, np.float64)[perm]


def unsharded_fold(ctx, phi, rates, words, hist, le, n_hist):
    """the unsharded node's fold: b2p_histogram_fold with the index over the rows in their order"""
    off, bs, ble = ctx.histogram_shard_index(hist, le, np.zeros(hist.size), np.arange(hist.size), n_hist)
    return ctx.histogram_fold(phi, off, bs, ble, rates, words)


def simulate(ctx, phi, rates, words, hist, le, n_hist, rank_of_row, R):
    """R ranks on one GPU through the step entry points; a torch copy stands in for each ncclSend / ncclRecv and for
    the gather of the results.  Rank r holds the rows with rank_of_row == r, in their order."""
    T, Tw = rates.shape[1], words.shape[1]
    dev = torch.device("cuda", 0)
    ranks = [np.flatnonzero(rank_of_row == r) for r in range(R)]
    counts = np.stack([np.bincount(hist[rows], minlength=n_hist) for rows in ranks]).astype(np.uint32)
    owner = ctx.histogram_shard_owners(counts)
    g_val = [torch.from_numpy(rates[rows].reshape(-1)).to(dev) for rows in ranks]
    g_w = [torch.from_numpy(words[rows].reshape(-1).view(np.int32)).to(dev) for rows in ranks]
    inbox = [[] for _ in range(R)]  # owner -> [(values, words, headers)] in sender rank order
    for q in range(R):
        lh = hist[ranks[q]]
        sel = sorted((i for i in range(lh.size) if owner[lh[i]] != q), key=lambda i: (owner[lh[i]], lh[i], i))
        n = len(sel)
        s_val = torch.zeros(max(n, 1) * T, dtype=torch.float64, device=dev)
        s_w = torch.zeros(max(n, 1) * Tw, dtype=torch.int32, device=dev)
        src = torch.tensor(sel + [0], dtype=torch.int32, device=dev)
        dst = torch.arange(n + 1, dtype=torch.int32, device=dev)
        ctx.row_move_dev(g_val[q], g_w[q], src, dst, n, T, s_val, s_w)
        a = 0
        for o in range(R):
            part = [i for i in sel if owner[lh[i]] == o]
            if part:
                b = a + len(part)
                inbox[o].append((s_val[a * T:b * T], s_w[a * Tw:b * Tw],
                                 [(int(lh[i]), float(le[ranks[q][i]]), q, i) for i in part]))
                a = b
    torch.cuda.synchronize()
    blocks_val, blocks_ok = [], []
    for me in range(R):
        mh = [int(h) for h in np.flatnonzero(owner == me)]
        local = {h: i for i, h in enumerate(mh)}
        lh = hist[ranks[me]]
        entries = [(int(lh[i]), float(le[ranks[me][i]]), me, i, i) for i in range(lh.size) if owner[lh[i]] == me]
        n_rows = lh.size
        buf_val, buf_w = [g_val[me]], [g_w[me]]
        at = n_rows  # received rows follow the owner's own
        for vals, wds, hdr in inbox[me]:
            for h, b, q, i in hdr:
                entries.append((h, b, q, i, at))
                at += 1
            buf_val.append(vals)
            buf_w.append(wds)
        grid = torch.cat(buf_val).cpu().numpy().reshape(-1, T)
        grid_w = torch.cat(buf_w).cpu().numpy().view(np.uint32).reshape(-1, Tw)
        off, bs, ble = ctx.histogram_shard_index([local[e[0]] for e in entries], [e[1] for e in entries],
                                                 [e[2] for e in entries], [e[3] for e in entries], len(mh))
        buf_row = np.array([e[4] for e in entries], np.uint32)
        if mh:
            out, ov = ctx.histogram_fold(phi, off, buf_row[bs], ble, grid, grid_w)
        else:
            out, ov = np.zeros((0, T)), np.zeros((0, Tw), np.uint32)
        blocks_val.append(out)
        blocks_ok.append(ov)
    # every owner's block to every rank, then placed in histogram order by the row move
    a_val = torch.from_numpy(np.concatenate(blocks_val).reshape(-1)).to(dev)
    a_w = torch.from_numpy(np.concatenate(blocks_ok).reshape(-1).view(np.int32)).to(dev)
    dst = np.concatenate([np.flatnonzero(owner == r) for r in range(R)]).astype(np.int32)
    out = torch.zeros(n_hist * T, dtype=torch.float64, device=dev)
    ov = torch.zeros(n_hist * Tw, dtype=torch.int32, device=dev)
    ctx.row_move_dev(a_val, a_w, torch.arange(n_hist, dtype=torch.int32, device=dev), torch.from_numpy(dst).to(dev),
                     n_hist, T, out, ov)
    torch.cuda.synchronize()
    moved = sum(len(h) for box in inbox for _, _, h in box)
    return out.cpu().numpy().reshape(n_hist, T), ov.cpu().numpy().view(np.uint32).reshape(n_hist, Tw), moved


@pytest.mark.parametrize("R", [2, 3, 8])
@pytest.mark.parametrize("layout", ["series", "histogram"])
def test_simulated_ranks_equal_the_fold_over_the_concatenation(ctxs, R, layout):
    plain, _ = ctxs
    rng = np.random.default_rng(R * 31 + (layout == "series"))
    rates, words, hist, le = bucket_rows(rng)
    H = int(hist.max()) + 1
    if layout == "series":
        rank_of_row = rng.integers(0, R, hist.size)
    else:
        rank_of_row = rng.integers(0, R, H)[hist]
    if R > 2:
        rank_of_row[rank_of_row == 1] = 0  # rank 1 holds no rows
    order = np.argsort(rank_of_row, kind="stable")  # the concatenation in rank order
    want_v, want_w = unsharded_fold(plain, 0.9, rates[order], words[order], hist[order], le[order], H)
    got_v, got_w, moved = simulate(plain, 0.9, rates, words, hist, le, H, rank_of_row, R)
    assert np.array_equal(got_w, want_w)
    assert np.array_equal(got_v.view(np.uint64), want_v.view(np.uint64))
    if layout == "histogram":
        assert moved == 0
    else:
        assert moved > 0


def test_composed_call_over_one_rank_equals_the_fold(ctxs):
    plain, comm = ctxs
    rates, words, hist, le = bucket_rows(np.random.default_rng(5))
    H = int(hist.max()) + 2  # the last histogram has no bucket: no rows
    want_v, want_w = unsharded_fold(plain, 0.75, rates, words, hist, le, H)
    for c in (plain, comm):
        got_v, got_w = c.histogram_fold_allgather(0.75, rates, words, hist, le, H)
        assert np.array_equal(got_w, want_w) and np.array_equal(got_v.view(np.uint64), want_v.view(np.uint64))
        T = rates.shape[1]
        assert c.last_exchange_bytes() == H * (8 * T + 4 * ((T + 31) // 32))  # its result block, no bucket row
    # a rank without rows
    got_v, got_w = comm.histogram_fold_allgather(0.5, np.zeros((0, 45)), np.zeros((0, 2), np.uint32), [], [], 3)
    assert not got_w.any() and not got_v.any()


# ---- the plan layer over a one-rank communicator -------------------------------------------------------------------------
def bucket_batch(seed, missing=0.1):
    return histograms(np.random.default_rng(seed), HISTS, LES, 90, missing=missing)


def test_sharded_node_and_leaf_export_the_unsharded_bytes(ctxs):
    from greptimedb_b200.plan import AggregatePlan, HistogramQuantilePlan
    plain, comm = ctxs
    batch = bucket_batch(3)
    tags = ["job", "instance", "le"]
    want = HistogramQuantilePlan(plain, 0.9, leaf(plain, batch, tags, START, END, STEP)).execute()
    got = HistogramQuantilePlan(comm, 0.9, leaf(comm, batch, tags, START, END, STEP)).sharded().execute()
    assert same_export(got, want)
    want = leaf(plain, batch, tags, START, END, STEP, histogram_quantile=0.5).execute()
    got = leaf(comm, batch, tags, START, END, STEP, histogram_quantile=0.5).sharded().execute()
    assert same_export(got, want)
    # a node above sees the replicated result
    want = AggregatePlan(plain, "max", HistogramQuantilePlan(plain, 0.9, leaf(plain, batch, tags, START, END, STEP)),
                         by=["job"]).execute()
    got = AggregatePlan(comm, "max", HistogramQuantilePlan(comm, 0.9, leaf(comm, batch, tags, START, END, STEP)).sharded(),
                        by=["job"]).execute()
    assert same_export(got, want)


def test_sharded_node_over_a_leaf_without_rows(ctxs):
    from greptimedb_b200.plan import HistogramQuantilePlan
    _, comm = ctxs
    empty = leaf(comm, histograms(np.random.default_rng(0), HISTS[:2], LES, 5, t0=10**9), ["job", "instance", "le"],
                 START, END, STEP)
    b = HistogramQuantilePlan(comm, 0.5, empty).sharded().execute()
    assert b.num_rows == 0


def test_refusals(ctxs):
    from greptimedb_b200 import B2PError
    from greptimedb_b200.plan import AggregatePlan, CountValuesPlan, HistogramQuantilePlan, PromRangeExec
    _, comm = ctxs
    tags = ["job", "instance", "le"]
    node = HistogramQuantilePlan(comm, 0.9, leaf(comm, bucket_batch(4), tags, START, END, STEP)).sharded()
    with pytest.raises(B2PError, match="below a sharded node"):
        AggregatePlan(comm, "sum", node).sharded().execute()
    with pytest.raises(B2PError, match="histogram_quantile"):
        HistogramQuantilePlan(comm, 0.9, HistogramQuantilePlan(comm, 0.9, leaf(comm, bucket_batch(4), tags, START,
                                                                                   END, STEP))).sharded().execute()
    cv = CountValuesPlan(comm, "le", leaf(comm, bucket_batch(5), tags, START, END, STEP), by=["job"])
    with pytest.raises(B2PError, match="count_values"):
        HistogramQuantilePlan(comm, 0.5, cv).sharded().execute()
    ids = leaf(comm, table_batch([({"__tsid": 7}, [START], [1.0])], ["__tsid"], string_tags=False), ["__tsid"],
               START, START, STEP, instant=True)
    with pytest.raises(B2PError, match="id-keyed"):
        HistogramQuantilePlan(comm, 0.5, ids).sharded().execute()
    # an Int64 value column read from the batch: decided on the agreed types
    i64 = pa.RecordBatch.from_pydict({"ts": pa.array([START, START], pa.timestamp("ms")),
                                      "val": pa.array([1, 2], pa.int64()), "job": ["a", "a"], "le": ["1", "+Inf"]})
    ex = PromRangeExec(comm, "", START, START, STEP, 0, "ts", "val", ["job", "le"], lookback_delta=STEP)
    ex.push(i64)
    with pytest.raises(B2PError, match="Int64"):
        HistogramQuantilePlan(comm, 0.5, ex).sharded().execute()
    two = pa.RecordBatch.from_pydict({"ts": pa.array([START], pa.timestamp("ms")), "a": [1.0], "b": [2.0],
                                      "job": ["x"], "le": ["1"]})
    mf = PromRangeExec(comm, "", START, START, STEP, 0, "ts", ["a", "b"], ["job", "le"], lookback_delta=STEP)
    mf.push(two)
    with pytest.raises(B2PError, match="multi-field"):
        HistogramQuantilePlan(comm, 0.5, mf).sharded().execute()
    no_le = leaf(comm, histograms(np.random.default_rng(42), HISTS[:2], LES, 60, tags=("job", "instance", "bucket")),
                 ["job", "instance", "bucket"], START, END, STEP)
    b = HistogramQuantilePlan(comm, 0.5, no_le).sharded().execute()
    assert b.num_rows == 0 and b.num_columns == 0
    with pytest.raises(B2PError, match="sharded form"):
        leaf(comm, bucket_batch(6), tags, START, END, STEP).sharded()


# ---- the row-move kernel ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T", [1, 31, 32, 33, 64, 1000])
@pytest.mark.parametrize("n", [0, 1, 77])
@pytest.mark.parametrize("shift", [0, 1])
def test_row_move_kernel(ctxs, T, n, shift):
    """out[dst[i]] = in[src[i]]; shift 1 puts both grids 8 bytes off 16-byte alignment (the scalar copy)"""
    plain, _ = ctxs
    dev = torch.device("cuda", 0)
    rng = np.random.default_rng(T * 7 + n)
    Tw = (T + 31) // 32
    rows_in, rows_out = 90, 100
    vin = torch.from_numpy(rng.standard_normal(rows_in * T + 1)).to(dev)
    win = torch.from_numpy(rng.integers(-2**31, 2**31, rows_in * Tw, dtype=np.int64).astype(np.int32)).to(dev)
    vout = torch.full((rows_out * T + 1,), -7.0, dtype=torch.float64, device=dev)
    wout = torch.full((rows_out * Tw,), 5, dtype=torch.int32, device=dev)
    src = rng.integers(0, rows_in, max(n, 1)).astype(np.int32)
    dst = rng.permutation(rows_out)[:max(n, 1)].astype(np.int32)
    plain.row_move_dev(vin.data_ptr() + 8 * shift, win, torch.from_numpy(src).to(dev), torch.from_numpy(dst).to(dev),
                       n, T, vout.data_ptr() + 8 * shift, wout)
    torch.cuda.synchronize()
    want_v = np.full(rows_out * T + 1, -7.0)
    want_w = np.full(rows_out * Tw, 5, np.int32)
    hv, hw = vin.cpu().numpy(), win.cpu().numpy()
    for i in range(n):
        want_v[shift + dst[i] * T: shift + (dst[i] + 1) * T] = hv[shift + src[i] * T: shift + (src[i] + 1) * T]
        want_w[dst[i] * Tw:(dst[i] + 1) * Tw] = hw[src[i] * Tw:(src[i] + 1) * Tw]
    assert np.array_equal(vout.cpu().numpy(), want_v) and np.array_equal(wout.cpu().numpy(), want_w)


# ---- the range form: the range function's grid stays on the device -------------------------------------------------
def bucket_series(rng, n_hist=30, n=60):
    """counter samples of each histogram's bucket series (1 to 70 buckets, the bounds of bucket_rows), series after
    series -> (ts, val, offsets [S+1], row_hist [S], row_le [S], params of rate over them)"""
    from greptimedb_b200 import make_params
    from oracle.oracle import parse_f64_rust
    ts, val, offsets, hist, le = [], [], [0], [], []
    for h in range(n_hist):
        nb = int(rng.choice([1, 2, 5, 12, 64, 65, 70])) if h % 4 == 0 else int(rng.integers(1, 14))
        for b in rng.choice(LE_CHOICES, size=nb):
            keep = rng.random(n) >= 0.1
            t = (15_000 * np.arange(n, dtype=np.int64))[keep]
            ts.append(t)
            val.append(np.cumsum(rng.random(n) * 4.0)[keep])
            offsets.append(offsets[-1] + t.size)
            hist.append(h)
            le.append(parse_f64_rust(b))
    p = make_params("rate", 300_000, 15_000 * (n - 1), 15_000, 120_000)
    return (np.concatenate(ts), np.concatenate(val), np.array(offsets, np.uint64), np.array(hist, np.uint32),
            np.array(le, np.float64), p)


def series_subset(ts, val, offsets, rows):
    """the samples and offsets of the series `rows`, in that order"""
    parts = [np.arange(offsets[s], offsets[s + 1], dtype=np.int64) for s in rows]
    take = np.concatenate(parts) if parts else np.zeros(0, np.int64)
    return ts[take], val[take], np.r_[0, np.cumsum([x.size for x in parts])].astype(np.uint64)


def test_range_form_over_one_rank_equals_the_unsharded_fold(ctxs):
    plain, comm = ctxs
    ts, val, offsets, hist, le, p = bucket_series(np.random.default_rng(8))
    H = int(hist.max()) + 1
    grid, words, _ = plain.range_eval(p, ts, val, offsets=offsets)
    want_v, want_w = unsharded_fold(plain, 0.9, grid, words, hist, le, H)
    for c in (plain, comm):
        got_v, got_w = c.range_histogram_fold_allgather(p, 0.9, ts, val, offsets, hist, le, H)
        assert np.array_equal(got_w, want_w) and np.array_equal(got_v.view(np.uint64), want_v.view(np.uint64))
        T = grid.shape[1]
        assert c.last_exchange_bytes() == H * (8 * T + 4 * ((T + 31) // 32))  # no bucket row, the results only
    # a rank without series takes part with its empty grid
    got_v, got_w = comm.range_histogram_fold_allgather(p, 0.9, ts[:0], val[:0], np.zeros(1, np.uint64), [], [], 4)
    assert not got_w.any()


@pytest.mark.parametrize("R", [2, 3, 8])
@pytest.mark.parametrize("layout", ["series", "histogram"])
def test_range_form_over_simulated_ranks(ctxs, R, layout):
    """By histogram (nothing split): every simulated rank's range form over its own series, one rank of one each, folds
    its own histograms and the union of those results is the fold over the concatenation.  By series hash (split):
    the step entry points over each rank's range grid give it too."""
    plain, _ = ctxs
    rng = np.random.default_rng(R + 100 * (layout == "series"))
    ts, val, offsets, hist, le, p = bucket_series(rng)
    H = int(hist.max()) + 1
    rank_of_row = rng.integers(0, R, hist.size) if layout == "series" else rng.integers(0, R, H)[hist]
    if R > 2:
        rank_of_row[rank_of_row == 1] = 0  # rank 1 holds no series
    order = np.argsort(rank_of_row, kind="stable")
    grid, words, _ = plain.range_eval(p, ts, val, offsets=offsets)
    want_v, want_w = unsharded_fold(plain, 0.9, grid[order], words[order], hist[order], le[order], H)
    if layout == "histogram":
        got_v, got_w = np.zeros_like(want_v), np.zeros_like(want_w)
        for r in range(R):
            rows = np.flatnonzero(rank_of_row == r)
            r_ts, r_val, r_off = series_subset(ts, val, offsets, rows)
            v, w = plain.range_histogram_fold_allgather(p, 0.9, r_ts, r_val, r_off, hist[rows], le[rows], H)
            held = np.unique(hist[rows])
            got_v[held], got_w[held] = v[held], w[held]
            assert not w[np.setdiff1d(np.arange(H), held)].any()  # a histogram it holds no bucket of: no row
    else:
        got_v, got_w, moved = simulate(plain, 0.9, grid, words, hist, le, H, rank_of_row, R)
        assert moved > 0
    assert np.array_equal(got_w, want_w) and np.array_equal(got_v.view(np.uint64), want_v.view(np.uint64))
