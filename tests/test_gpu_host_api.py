"""GPU: every synchronous host-pointer entry point against its device-API route, bit for bit (the host API stages
the columns, runs the same kernels and copies the results back), its NULL-argument checks, and a device-API call
that keeps its own scratch while a host call runs behind it."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

T0, STEP = 1_700_000_000_000, 15_000
E_INVALID = -1


def _ctx(torch_stream=False):
    from greptimedb_b200 import Context
    c = Context(0)
    if torch_stream:
        c.use_torch_stream()
    return c


@pytest.fixture
def pair():
    """(host-API context, device-API context): two fresh contexts, so that the adaptive tiering of each sees the same
    sequence of range calls"""
    h, d = _ctx(), _ctx(torch_stream=True)
    yield h, d
    h.close()
    d.close()


def dev(x):
    """flat device copy of a column; an empty one still has an address (one element), as an empty numpy array has"""
    import torch
    x = np.ascontiguousarray(x)
    signed = {np.dtype(np.uint32): np.int32, np.dtype(np.uint64): np.int64}.get(x.dtype)
    t = torch.from_numpy(x.view(signed) if signed else x)
    d = torch.zeros(max(t.numel(), 1), dtype=t.dtype, device="cuda")
    d[:t.numel()].copy_(t.reshape(-1))
    return d


def zeros(n, dtype):
    import torch
    return torch.zeros(max(n, 1), dtype=dtype, device="cuda")


def host(t, dtype, shape):
    import torch
    torch.cuda.synchronize()
    return t.cpu().numpy().view(dtype)[:int(np.prod(shape))].reshape(shape)


def words_to_bool(words, T):
    from greptimedb_b200 import valid_to_bool
    return valid_to_bool(words.reshape(-1, words.shape[-1]) if words.size else np.zeros((0, 1), np.uint32), T)


def same(out_h, valid_h, out_d, valid_d, T):
    """identical validity and identical bits in every valid cell"""
    np.testing.assert_array_equal(valid_h, valid_d)
    if out_h.size:
        mask = words_to_bool(valid_h, T)
        np.testing.assert_array_equal(out_h.view(np.uint64)[mask], out_d.view(np.uint64)[mask])


def samples(seed, S, max_rows=60):
    """S series of jittered 15 s scrapes with counter resets; every fifth series is empty"""
    rng = np.random.default_rng(seed)
    counts = rng.integers(1, max_rows, S)
    counts[::5] = 0
    ts, val = [], []
    for n in counts:
        ts.append(T0 + np.cumsum(rng.integers(STEP - 2000, STEP + 2000, n)))
        v = np.cumsum(rng.random(n) * 10.0)
        v[rng.random(n) < 0.05] = 0.0
        val.append(v)
    ts = np.concatenate(ts or [np.zeros(0)]).astype(np.int64)
    val = np.concatenate(val or [np.zeros(0)]).astype(np.float64)
    offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.uint64)
    sid = np.repeat(np.arange(S, dtype=np.uint32), counts)
    return ts, val, sid, offsets


def grid_end(T, interval=30_000):
    return T0 + (T - 1) * interval if T > 0 else T0 - 1


def dev_offsets(d, sid, offsets, n_rows, S):
    if offsets is not None:
        return dev(offsets)
    d_off = zeros(S + 1, __import__("torch").int64)
    d.series_offsets_dev(dev(sid), n_rows, S, d_off)
    return d_off


# ---- range_eval / instant_select / range_histogram_fold: the series input by ids or by offsets ------------------------

SHAPES = [(40, 31), (40, 32), (40, 0), (0, 32), ("empty", 33)]


@pytest.mark.parametrize("fn", ["rate", "sum_over_time", "quantile_over_time"])
@pytest.mark.parametrize("by", ["ids", "offsets"])
@pytest.mark.parametrize("S,T", SHAPES)
def test_range_eval(pair, fn, by, S, T):
    import torch
    from greptimedb_b200 import make_params
    h, d = pair
    if S == "empty":  # series without a single row: n_rows = 0
        S = 12
        ts, val = np.zeros(0, np.int64), np.zeros(0, np.float64)
        sid, offsets = np.zeros(0, np.uint32), np.zeros(S + 1, np.uint64)
    else:
        ts, val, sid, offsets = samples(1 + S + T, S)
    p = make_params(fn, T0, grid_end(T), 30_000, 120_000, param0=0.9)
    sid_h, off_h = (sid, None) if by == "ids" else (None, offsets)
    out_h, valid_h, ets = h.range_eval_n(p, ts, val, sid_h, off_h, S)
    np.testing.assert_array_equal(ets, T0 + np.arange(max(T, 0)) * 30_000)
    Tw = (T + 31) // 32
    out_d, valid_d = zeros(S * T, torch.float64), zeros(S * Tw, torch.int32)
    d.range_eval_dev(p, dev(ts), dev(val), dev_offsets(d, sid_h, off_h, ts.size, S), ts.size, S, out_d, valid_d)
    d.sync()
    same(out_h, valid_h, host(out_d, np.float64, (S, T)), host(valid_d, np.uint32, (S, Tw)), T)
    assert h.last_h2d_bytes() == ts.size * 16 + ((S + 1) * 8 if by == "offsets" else ts.size * 4) or S == 0 or T == 0


@pytest.mark.parametrize("by", ["ids", "offsets"])
@pytest.mark.parametrize("S,T", SHAPES)
def test_instant_select(pair, by, S, T):
    import torch
    h, d = pair
    if S == "empty":
        S = 12
        ts, val = np.zeros(0, np.int64), np.zeros(0, np.float64)
        sid, offsets = np.zeros(0, np.uint32), np.zeros(S + 1, np.uint64)
    else:
        ts, val, sid, offsets = samples(7 + S + T, S)
    from greptimedb_b200.engine import _ptr
    sid_h, off_h = (sid, None) if by == "ids" else (None, offsets)
    args = (T0, grid_end(T), 30_000, 300_000, 5_000)
    Tw = (T + 31) // 32
    out_h, valid_h = np.zeros((S, T)), np.zeros((S, Tw), np.uint32)
    rc = h._L.b2p_instant_select(h._h, *args, _ptr(ts), _ptr(val), _ptr(sid_h), _ptr(off_h), ts.size, S, _ptr(out_h),
                                 _ptr(valid_h))
    assert rc == 0, h._L.b2p_last_error().decode()
    out_d, valid_d = zeros(S * T, torch.float64), zeros(S * Tw, torch.int32)
    d.instant_select_dev(*args, dev(ts), dev(val), dev_offsets(d, sid_h, off_h, ts.size, S), ts.size, S, out_d,
                         valid_d)
    d.sync()
    same(out_h, valid_h, host(out_d, np.float64, (S, T)), host(valid_d, np.uint32, (S, Tw)), T)


def fold_index(n_hist, n_buckets):
    """histograms of n_buckets consecutive bucket series each, le bounds ascending, the last +Inf"""
    hist_off = (np.arange(n_hist + 1) * n_buckets).astype(np.uint32)
    bucket_series = np.arange(n_hist * n_buckets, dtype=np.uint32)
    les = np.concatenate([np.geomspace(0.01, 10.0, n_buckets - 1), [np.inf]])
    return hist_off, bucket_series, np.tile(les, n_hist)


def range_histogram_fold_host(ctx, p, ts, val, sid, offsets, S, phi, hist_off, bucket_series, bucket_le, T):
    from greptimedb_b200 import _lib
    from greptimedb_b200.engine import _ptr
    H, Tw = hist_off.size - 1, (T + 31) // 32
    out, ov = np.zeros((H, T)), np.zeros((H, Tw), np.uint32)
    rc = _lib.load().b2p_range_histogram_fold(ctx._h, C.byref(p), _ptr(ts), _ptr(val), _ptr(sid), _ptr(offsets),
                                              ts.size, S, phi, _ptr(hist_off), _ptr(bucket_series), _ptr(bucket_le),
                                              H, _ptr(out), _ptr(ov))
    return rc, out, ov


@pytest.mark.parametrize("by", ["ids", "offsets"])
@pytest.mark.parametrize("T", [31, 32, 0])
def test_range_histogram_fold(pair, by, T):
    import torch
    from greptimedb_b200 import make_params
    h, d = pair
    H, B = 8, 6
    S = H * B
    ts, val, sid, offsets = samples(20 + T, S)
    hist_off, bucket_series, bucket_le = fold_index(H, B)
    p = make_params("rate", T0, grid_end(T), 30_000, 120_000)
    sid_h, off_h = (sid, None) if by == "ids" else (None, offsets)
    rc, out_h, valid_h = range_histogram_fold_host(h, p, ts, val, sid_h, off_h, S, 0.9, hist_off, bucket_series,
                                                   bucket_le, T)
    assert rc == 0, h._L.b2p_last_error().decode()
    Tw = (T + 31) // 32
    rates, rvalid = zeros(S * T, torch.float64), zeros(S * Tw, torch.int32)
    d.range_eval_dev(p, dev(ts), dev(val), dev_offsets(d, sid_h, off_h, ts.size, S), ts.size, S, rates, rvalid)
    d.sync()
    out_d, valid_d = zeros(H * T, torch.float64), zeros(H * Tw, torch.int32)
    d.histogram_fold_dev(0.9, dev(hist_off), dev(bucket_series), dev(bucket_le), H, rates, rvalid, T, out_d, valid_d)
    d.sync()
    same(out_h, valid_h, host(out_d, np.float64, (H, T)), host(valid_d, np.uint32, (H, Tw)), T)


# ---- range_udf: explicit windows, eval_ts given or omitted ----------------------------------------------------------

@pytest.mark.parametrize("fn", ["rate", "delta", "holt_winters", "quantile_over_time"])
@pytest.mark.parametrize("with_eval_ts", [True, False])
@pytest.mark.parametrize("n_rows", [500, 0])
def test_range_udf(pair, fn, with_eval_ts, n_rows):
    import torch
    from greptimedb_b200 import pack_ranges
    from greptimedb_b200.engine import FN_IDS
    h, d = pair
    rng = np.random.default_rng(n_rows + len(fn))
    ts = T0 + np.cumsum(rng.integers(1, 20_000, n_rows)).astype(np.int64)
    val = np.cumsum(rng.random(n_rows) * 5.0)
    starts = rng.integers(0, max(n_rows, 1), 97)
    lens = np.minimum(rng.integers(0, 30, 97), max(n_rows, 0) - starts) if n_rows else np.zeros(97, np.int64)
    ranges = np.stack([starts if n_rows else np.zeros(97, np.int64), lens], axis=1)
    eval_ts = (T0 + np.arange(97) * 7_000).astype(np.int64) if with_eval_ts else None
    out_h, valid_h = h.range_udf(fn, ts, val, ranges, eval_ts, 60_000, 0.5, 0.3)
    packed = pack_ranges(ranges)
    out_d, valid_d = zeros(97, torch.float64), zeros(97, torch.uint8)
    from greptimedb_b200.engine import _ptr
    # (the device columns are held until the kernel has run: a freed block would be handed to the next copy)
    cols = [dev(ts), dev(val), dev(packed), None if eval_ts is None else dev(eval_ts)]
    rc = d._L.b2p_range_udf_dev(d._h, FN_IDS[fn], _ptr(cols[0]), _ptr(cols[1]), n_rows, _ptr(cols[2]), _ptr(cols[3]),
                                97, 60_000, 0.5, 0.3, _ptr(out_d), _ptr(valid_d))
    assert rc == 0, d._L.b2p_last_error().decode()
    vd = host(valid_d, np.uint8, (97,)).astype(bool)
    od = host(out_d, np.float64, (97,))
    np.testing.assert_array_equal(valid_h, vd)
    np.testing.assert_array_equal(out_h.view(np.uint64)[vd], od.view(np.uint64)[vd])


# ---- by-label aggregate, histogram_quantile ----------------------------------------------------------------------------

def dense(seed, S, T):
    rng = np.random.default_rng(seed)
    vals = rng.normal(size=(S, T)) * 100.0
    ok = rng.random((S, T)) < 0.7
    Tw = (T + 31) // 32
    words = np.zeros((S, Tw * 32), bool)
    words[:, :T] = ok
    return vals, np.packbits(words, axis=1, bitorder="little").view(np.uint32).reshape(S, Tw)


@pytest.mark.parametrize("agg", ["sum", "avg", "count", "min", "max", "stddev", "stdvar"])
@pytest.mark.parametrize("S,G,T", [(50, 7, 31), (50, 7, 32), (0, 3, 32), (50, 0, 32), (50, 7, 0)])
def test_group_aggregate(pair, agg, S, G, T):
    import torch
    h, d = pair
    vals, words = dense(S * 3 + T, S, T)
    gid = (np.arange(S) % max(G, 1)).astype(np.uint32)
    out_h, cnt_h = h.group_aggregate(agg, vals, words, gid, G)
    out_d, cnt_d = zeros(G * T, torch.float64), zeros(G * T, torch.int32)
    d.group_aggregate_dev(agg, dev(vals), dev(words), dev(gid), S, G, T, out_d, cnt_d)
    d.sync()
    cd = host(cnt_d, np.uint32, (G, T))
    np.testing.assert_array_equal(cnt_h, cd)
    np.testing.assert_array_equal(out_h.view(np.uint64)[cd > 0], host(out_d, np.float64, (G, T)).view(np.uint64)[cd > 0])


@pytest.mark.parametrize("H,T", [(9, 31), (9, 32), (9, 0), (0, 32)])
def test_histogram_quantile(pair, H, T):
    import torch
    h, d = pair
    B = 5
    les = np.array([0.1, 0.5, 1.0, 5.0, np.inf])
    rates, words = dense(H + T, H * B, T)
    rates = np.abs(rates)
    out_h, valid_h = h.histogram_quantile(0.75, les, rates, words)
    Tw = (T + 31) // 32
    out_d, valid_d = zeros(H * T, torch.float64), zeros(H * Tw, torch.int32)
    d.histogram_quantile_dev(0.75, dev(les), B, dev(rates), dev(words), H, T, out_d, valid_d)
    d.sync()
    same(out_h, valid_h, host(out_d, np.float64, (H, T)), host(valid_d, np.uint32, (H, Tw)), T)


# ---- binary and set operators --------------------------------------------------------------------------------------

@pytest.mark.parametrize("op,return_bool", [("+", False), ("/", False), (">", False), ("<=", True)])
@pytest.mark.parametrize("L,R,P,T", [(30, 20, 45, 31), (30, 20, 45, 32), (30, 0, 0, 32), (30, 20, 45, 0)])
def test_binary_op(pair, op, return_bool, L, R, P, T):
    import torch
    h, d = pair
    rng = np.random.default_rng(L + R + P + T)
    lhs, lv = dense(1 + T, L, T)
    rhs, rv = dense(2 + T, R, T)
    lrow = rng.integers(0, L, P).astype(np.uint32)
    rrow = rng.integers(0, max(R, 1), P).astype(np.uint32)
    out_h, valid_h = h.binary_op(op, lhs, lv, lrow, rhs, rv, rrow, return_bool=return_bool)
    Tw = (T + 31) // 32
    out_d, valid_d = zeros(P * T, torch.float64), zeros(P * Tw, torch.int32)
    d.binary_op_dev(op, dev(lhs), dev(lv), dev(lrow), L, dev(rhs), dev(rv), dev(rrow), R, P, T, out_d, valid_d,
                    return_bool=return_bool)
    d.sync()
    same(out_h, valid_h, host(out_d, np.float64, (P, T)), host(valid_d, np.uint32, (P, Tw)), T)


@pytest.mark.parametrize("op,return_bool", [("-", False), ("^", False), ("==", False), (">", True)])
@pytest.mark.parametrize("scalar_on_left", [False, True])
@pytest.mark.parametrize("S,T", [(25, 31), (25, 32), (0, 32), (25, 0)])
def test_scalar_op(pair, op, return_bool, scalar_on_left, S, T):
    import torch
    h, d = pair
    vals, words = dense(S + T, S, T)
    kw = dict(scalar_on_left=scalar_on_left, return_bool=return_bool)
    out_h, valid_h = h.scalar_op(op, 2.5, vals, words, **kw)
    Tw = (T + 31) // 32
    out_d, valid_d = zeros(S * T, torch.float64), zeros(S * Tw, torch.int32)
    d.scalar_op_dev(op, 2.5, dev(vals), dev(words), S, T, out_d, valid_d, **kw)
    d.sync()
    same(out_h, valid_h, host(out_d, np.float64, (S, T)), host(valid_d, np.uint32, (S, Tw)), T)


@pytest.mark.parametrize("op", ["and", "or", "unless"])
@pytest.mark.parametrize("L,R,K,T", [(40, 30, 12, 31), (40, 30, 12, 32), (40, 30, 0, 32), (0, 30, 12, 32),
                                     (40, 0, 12, 33), (40, 30, 12, 0)])
def test_setop(pair, op, L, R, K, T):
    import torch
    from greptimedb_b200.engine import NO_KEY
    h, d = pair
    rng = np.random.default_rng(L + R + K + T)
    lhs, lv = dense(3 + T, L, T)
    rhs, rv = dense(4 + T, R, T)
    keys = lambda n: np.where(rng.random(n) < 0.1, NO_KEY, rng.integers(0, max(K, 1), n)).astype(np.uint32) \
        if K else np.full(n, NO_KEY, np.uint32)
    lk, rk = keys(L), keys(R)
    out_h, valid_h = h.setop(op, lhs, lv, lk, rhs, rv, rk, K)
    n = L + R if op == "or" else L
    Tw = (T + 31) // 32
    out_d, valid_d = zeros(n * T, torch.float64), zeros(n * Tw, torch.int32)
    d.setop_dev(op, dev(lhs), dev(lv), dev(lk), L, dev(rhs), dev(rv), dev(rk), R, K, T, out_d, valid_d)
    d.sync()
    same(out_h, valid_h, host(out_d, np.float64, (n, T)), host(valid_d, np.uint32, (n, Tw)), T)


# ---- a NULL host column where there is work -------------------------------------------------------------------------

def host_calls(ctx):
    """name -> (C entry point, arguments before the outputs, index of the input column to pass as NULL, the output
    columns as (shape, dtype, initial value), index of the output column to pass as NULL)"""
    from greptimedb_b200 import make_params, pack_ranges
    from greptimedb_b200.engine import _ptr as P
    ts, val, sid, offsets = samples(99, 20)
    S, T, Tw = 20, 32, 1
    p = make_params("rate", T0, grid_end(T), 30_000, 120_000)
    p_sub = make_params("sum_over_time", T0, grid_end(T), 30_000, 120_000, filter_nan=False)
    vals, words = dense(5, S, T)
    rates = np.abs(vals)
    gid = (np.arange(S) % 4).astype(np.uint32)
    rows = np.arange(S, dtype=np.uint32)
    keys = (np.arange(S) % 6).astype(np.uint32)
    tie = rows[::-1].copy()
    hist_off, bucket_series, bucket_le = fold_index(4, 5)
    packed = pack_ranges(np.stack([np.arange(10) * 3, np.full(10, 5)], axis=1))
    H = ctx._h
    f8, u4 = np.float64, np.uint32
    grid = lambda n, m=Tw: [((n, T), f8, -1.0), ((n, m), u4, 7)]
    calls = {
        "range_eval": ("b2p_range_eval", [H, C.byref(p), P(ts), P(val), P(sid), None, ts.size, S], 2, grid(S), 0),
        "range_udf": ("b2p_range_udf", [H, 0, P(ts), P(val), ts.size, P(packed), None, 10, 60_000, 0.0, 0.0], 2,
                      [((10,), f8, -1.0), ((10,), np.uint8, 7)], 1),
        "instant_select": ("b2p_instant_select", [H, T0, grid_end(T), 30_000, 300_000, 0, P(ts), P(val), None,
                                                  P(offsets), ts.size, S], 6, grid(S), 0),
        "group_aggregate": ("b2p_group_aggregate", [H, 0, P(vals), P(words), P(gid), S, 4, T], 2, grid(4, T), 1),
        "histogram_quantile": ("b2p_histogram_quantile", [H, 0.5, P(bucket_le), 5, P(rates), P(words), 4,
                                                          T], 4, grid(4), 0),
        "histogram_fold": ("b2p_histogram_fold", [H, 0.5, P(hist_off), P(bucket_series), P(bucket_le), 4, P(rates),
                                                  P(words), S, T], 6, grid(4), 1),
        "range_histogram_fold": ("b2p_range_histogram_fold", [H, C.byref(p), P(ts), P(val), P(sid), None, ts.size, S,
                                                              0.5, P(hist_off), P(bucket_series), P(bucket_le), 4],
                                 11, grid(4), 0),
        "binary_op": ("b2p_binary_op", [H, 0, 0, P(vals), P(words), P(rows), S, P(vals), P(words), P(rows), S, S, T],
                      8, grid(S), 1),
        "scalar_op": ("b2p_scalar_op", [H, 0, 0, 0, 1.5, P(vals), P(words), S, T], 6, grid(S), 0),
        "setop": ("b2p_setop", [H, 0, P(vals), P(words), P(keys), S, P(vals), P(words), P(keys), S, 6, T], 4, grid(S),
                  1),
        "instant_fn": ("b2p_instant_fn", [H, 3, 0.0, 0.0, P(rates), P(words), S, T], 4, grid(S), 1),
        "scalar_calculate": ("b2p_scalar_calculate", [H, P(vals), P(words), P(rows), S, T], 3,
                             [((T,), f8, -1.0), ((Tw,), u4, 7)], 0),
        "topk": ("b2p_topk", [H, 0, 3.0, P(vals), P(words), P(gid), S, 4, P(tie), T], 5, [((S, Tw), u4, 7)], 0),
        "group_quantile": ("b2p_group_quantile", [H, 0.25, P(vals), P(words), P(gid), S, 4, T], 2, grid(4, T), 1),
        "count_values": ("b2p_count_values", [H, P(vals), P(words), P(gid), S, 4, T], 3, grid(S, T), 0),
        "subquery": ("b2p_subquery", [H, C.byref(p_sub), T0 - 60_000, 15_000, P(vals), P(words), S, T], 4, grid(S),
                     1),
        # (the cell count starts at 0: a rejected call may leave an empty result's count)
        "sort_cells": ("b2p_sort_cells", [H, 0, P(vals), P(words), S, T], 3,
                       [((S * T,), np.uint64, 7), ((1,), np.uint64, 0)], 1),
    }
    keep = (ts, val, sid, offsets, vals, rates, words, gid, rows, keys, tie, hist_off, bucket_series, bucket_le, packed,
            p, p_sub)
    return calls, keep


def run(ctx, fn, args, outs, null_out=None):
    """one call with fresh output columns, output `null_out` passed as NULL -> (rc, the output columns)"""
    from greptimedb_b200.engine import _ptr
    cols = [np.full(shape, init, dtype) for shape, dtype, init in outs]
    ptrs = [None if i == null_out else _ptr(col) for i, col in enumerate(cols)]
    tail = [None] if fn == "b2p_range_eval" else []  # (out_ts)
    return getattr(ctx._L, fn)(*args, *ptrs, *tail), cols


HOST_FORMS = ["range_eval", "range_udf", "instant_select", "group_aggregate", "histogram_quantile",
              "range_histogram_fold", "binary_op", "scalar_op", "setop", "instant_fn", "scalar_calculate", "topk",
              "group_quantile", "count_values", "subquery", "histogram_fold", "sort_cells"]


@pytest.mark.parametrize("name", HOST_FORMS + [f"{n}:out" for n in HOST_FORMS])
def test_null_host_column_is_rejected_and_the_context_stays_usable(name):
    """a call with one NULL input column (`<form>:out`: output column) where there is work fails with B2P_E_INVALID
    and writes nothing; the same call with every column then gives the same bits as before it"""
    form, _, output = name.partition(":")
    ctx = _ctx()
    try:
        calls, _keep = host_calls(ctx)
        fn, args, null_in, outs, null_out = calls[form]
        rc, good = run(ctx, fn, args, outs)
        assert rc == 0, ctx._L.b2p_last_error().decode()
        bad = list(args)
        if not output:
            bad[null_in] = None
        rc, cols = run(ctx, fn, bad, outs, null_out if output else None)
        assert rc == E_INVALID and "NULL" in ctx._L.b2p_last_error().decode()
        for col, (_, _, init) in zip(cols, outs):
            assert (col == init).all()  # nothing was written
        rc, again = run(ctx, fn, args, outs)
        assert rc == 0, ctx._L.b2p_last_error().decode()
        for a, b in zip(again, good):
            np.testing.assert_array_equal(a.view(f"u{a.itemsize}"), b.view(f"u{b.itemsize}"))
    finally:
        ctx.close()


# ---- the device forms check the sample columns themselves ------------------------------------------------------------

@pytest.mark.parametrize("column", ["ts", "val"])
def test_null_sample_column_of_a_device_form_is_rejected(column):
    """range_udf / instant_select on the device with a NULL sample column and rows to read: B2P_E_INVALID, no launch"""
    import torch
    from greptimedb_b200 import pack_ranges
    from greptimedb_b200.engine import _ptr
    ctx = _ctx(torch_stream=True)
    try:
        ts, val, _sid, offsets = samples(3, 8)
        cols = {"ts": dev(ts), "val": dev(val)}
        cols[column] = None
        packed = dev(pack_ranges(np.stack([np.arange(4) * 2, np.full(4, 3)], axis=1)))
        out, valid = zeros(4, torch.float64), zeros(4, torch.uint8)
        rc = ctx._L.b2p_range_udf_dev(ctx._h, 0, _ptr(cols["ts"]), _ptr(cols["val"]), ts.size, _ptr(packed), None, 4,
                                      60_000, 0.0, 0.0, _ptr(out), _ptr(valid))
        assert rc == E_INVALID and "NULL" in ctx._L.b2p_last_error().decode()
        out, valid = zeros(8 * 32, torch.float64), zeros(8, torch.int32)
        rc = ctx._L.b2p_instant_select_dev(ctx._h, T0, grid_end(32), 30_000, 300_000, 0, _ptr(cols["ts"]),
                                           _ptr(cols["val"]), _ptr(dev(offsets)), ts.size, 8, _ptr(out), _ptr(valid))
        assert rc == E_INVALID and "NULL" in ctx._L.b2p_last_error().decode()
        assert ctx._L.b2p_sync(ctx._h) == 0, ctx._L.b2p_last_error().decode()
    finally:
        ctx.close()


# ---- a device-API call's scratch is its own --------------------------------------------------------------------------

def test_unfused_group_sum_survives_a_host_call_issued_behind_it():
    """the by-label sum of a function without a fused tier evaluates the range function into scratch and folds it by an
    asynchronous kernel; a host call on another stream right behind it must not write into that scratch"""
    import torch
    from greptimedb_b200 import make_params
    S, G, T = 4096, 64, 400
    ts, val, sid, offsets = samples(5, S, max_rows=400)
    p = make_params("sum_over_time", T0, grid_end(T, 15_000), 15_000, 60_000)
    gid = (np.arange(S) % G).astype(np.uint32)
    Tw = (T + 31) // 32

    ref = _ctx(torch_stream=True)
    out, valid = zeros(S * T, torch.float64), zeros(S * Tw, torch.int32)
    ref.range_eval_dev(p, dev(ts), dev(val), dev(offsets), ts.size, S, out, valid)
    ref.sync()
    e_sum, e_cnt = zeros(G * T, torch.float64), zeros(G * T, torch.int32)
    ref.group_aggregate_dev("sum", out, valid, dev(gid), S, G, T, e_sum, e_cnt)
    ref.sync()
    e_sum, e_cnt = host(e_sum, np.float64, (G, T)), host(e_cnt, np.uint32, (G, T))
    ref.close()

    ctx = _ctx(torch_stream=True)
    try:
        ix = ctx.group_index_create_dev(dev(gid), S, G)
        assert not ctx.range_group_sum_fused(p, ix)
        d_ts, d_val, d_off = dev(ts), dev(val), dev(offsets)
        g_sum, g_cnt = zeros(G * T, torch.float64), zeros(G * T, torch.int32)
        ctx.range_group_sum_indexed_dev(p, d_ts, d_val, d_off, ts.size, S, ix, 0, G, g_sum, g_cnt)
        ctx.use_own_stream()  # the host call runs on the context's own stream, beside the aggregate
        junk, junk_valid = dense(11, S, T)
        ctx.group_aggregate("max", junk * 1e6, junk_valid, gid, G)
        torch.cuda.synchronize()
        np.testing.assert_array_equal(host(g_cnt, np.uint32, (G, T)), e_cnt)
        np.testing.assert_array_equal(host(g_sum, np.float64, (G, T)), e_sum)
        ctx.group_index_destroy(ix)
    finally:
        ctx.close()
