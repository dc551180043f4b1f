"""GPU: SeriesDivide (K0) and the host-pointer range call at their edges (run with -m gpu).

  - K0's device form on every layout of tests/series_divide_edges.py, exact against the reference; every bad column is
    B2P_E_UNSORTED at b2p_sync and leaves all-zero offsets, so a range call queued on them reads no row; the
    context's next call is exact.
  - The one-shot host entries (range, instant, timestamp, both multi-field forms, histogram fold) by ids and by
    offsets give the same bits; the range call matches the oracle's rescan restatement.
  - The chunked pipeline of b2p_range_eval over more than 6 291 456 rows, by ids with the host scan, by ids without it
    and by offsets, with pageable and with pinned buffers: every cell against b2p_range_eval_dev over the whole column,
    sampled series against the oracle, and b2p_last_h2d_bytes against the chunk table, which names each chunk's route.
  - Offsets that decrease or run past n_rows are B2P_E_INVALID from every host entry before any copy; bad id columns
    are B2P_E_UNSORTED from every host entry and both chunked id routes.
Offsets start as all ones with a 64-entry guard tail; outputs as a NaN pattern and validity words as all ones, each
with a guard tail that must stay untouched.
"""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle as orc
from tests import series_divide_edges as sd

pytestmark = pytest.mark.gpu

T0, SC = 1_700_000_000_000, 15_000
GUARD = 64
NAN_BITS = np.uint64(0x7FF4DEADBEEF0BAD)
FN = "sum_over_time"   # every sample of a window changes the sum, and every tier gives the oracle's bits


@pytest.fixture(scope="module")
def torch():
    import torch
    return torch


@pytest.fixture(scope="module")
def ctx():
    from greptimedb_b200 import Context
    c = Context(0)
    c.use_torch_stream()   # ordered after the torch copies and fills that set up its inputs
    yield c
    c.close()


@pytest.fixture(scope="module")
def sms(torch):
    return torch.cuda.get_device_properties(0).multi_processor_count


def _err(f):
    from greptimedb_b200 import B2PError
    try:
        f()
    except B2PError as e:
        return e.code
    return 0


# ---- K0 device form ---------------------------------------------------------------------------------------------
def _k0(torch, ctx, ids, S):
    d_sid = torch.from_numpy(ids.view(np.int32)).cuda() if ids.size else torch.empty(0, dtype=torch.int32, device="cuda")
    d_off = torch.full((S + 1 + GUARD,), -1, dtype=torch.int64, device="cuda")
    ctx.series_offsets_dev(d_sid, ids.size, S, d_off)
    return d_sid, d_off


def _guard_ok(d_off, S):
    return bool((d_off[S + 1:].cpu().numpy() == -1).all())


def test_k0_on_every_layout(torch, ctx, sms):
    from greptimedb_b200 import make_params
    seen = set()
    good_prev = None
    for lay in sd.layout_cases(sms):
        seen |= lay.classes
        S, n = lay.n_series, lay.ids.size
        d_sid, d_off = _k0(torch, ctx, lay.ids, S)
        if not lay.bad:
            ctx.sync()
            ref, _ = sd.offsets_fast(lay.ids, S)
            got = d_off[:S + 1].cpu().numpy().view(np.uint64)
            bad = np.flatnonzero(got != ref)
            assert not bad.size, f"{lay.name}: offsets differ at {bad[:5].tolist()}: {got[bad[:5]]} vs {ref[bad[:5]]}"
            assert _guard_ok(d_off, S), lay.name
            good_prev = (lay, ref)
            continue
        # a range call queued on the flagged column's offsets reads no row: every cell invalid
        T = 8
        p = make_params(FN, T0, T0 + 7 * SC, SC, 60_000)
        d_ts = torch.arange(n, dtype=torch.int64, device="cuda") * SC + T0
        d_val = torch.ones(n, dtype=torch.float64, device="cuda")
        out = torch.full((S * T,), float("nan"), dtype=torch.float64, device="cuda")
        valid = torch.full((S,), -1, dtype=torch.int32, device="cuda")
        ctx.range_eval_dev(p, d_ts, d_val, d_off, n, S, out, valid)
        assert _err(ctx.sync) == sd.E_UNSORTED, lay.name
        assert (d_off[:S + 1].cpu().numpy() == 0).all() and _guard_ok(d_off, S), lay.name
        assert (valid.cpu().numpy() == 0).all(), lay.name
        # the context's next call is exact
        glay, gref = good_prev
        _, d_off2 = _k0(torch, ctx, glay.ids, glay.n_series)
        ctx.sync()
        assert (d_off2[:glay.n_series + 1].cpu().numpy().view(np.uint64) == gref).all(), lay.name
    assert seen >= sd.CLASSES, sorted(sd.CLASSES - seen)


def test_k0_refuses_a_misaligned_id_column(torch, ctx):
    from greptimedb_b200 import B2PError
    d_sid = torch.zeros(1024, dtype=torch.int32, device="cuda")
    d_off = torch.full((3 + GUARD,), -1, dtype=torch.int64, device="cuda")
    before = ctx.launch_count()
    with pytest.raises(B2PError) as ei:
        ctx.series_offsets_dev(d_sid[1:], 1023, 2, d_off)
    assert ei.value.code == sd.E_INVALID and ctx.launch_count() == before
    ctx.sync()
    assert (d_off.cpu().numpy() == -1).all()


# ---- host entries -----------------------------------------------------------------------------------------------
def _series_columns(offs, seed, regular=True, t0s=None):
    """ts (15 s cadence from each series' t0; one row 1 ms late in every irregular series) and random values"""
    rng = np.random.default_rng(seed)
    offs = np.asarray(offs, np.uint64)
    S = offs.size - 1
    t0s = np.full(S, T0, np.int64) if t0s is None else t0s
    ts = sd.timestamps(offs, np.full(S, SC, np.int64), t0s)
    lens = np.diff(offs.astype(np.int64))
    reg = np.broadcast_to(np.asarray(regular), (S,))
    for s in np.flatnonzero(~reg & (lens >= 3)):
        ts[int(offs[s]) + 1: int(offs[s + 1])] += 1   # the cadence holds from row 1 on, but not at row 1
    val = rng.standard_normal(ts.size) * 100
    return ts, val


def _pad(a, fill):
    """a with a guard tail of GUARD entries of `fill` (bits), and the view of its first a.size entries"""
    buf = np.empty(a.size + GUARD, a.dtype)
    buf.view(np.uint64 if a.itemsize == 8 else np.uint32)[:] = fill
    return buf


def _outs(S, T, n=1):
    Tw = (T + 31) // 32
    outs = [_pad(np.empty(S * T), NAN_BITS) for _ in range(n)]
    valid = _pad(np.empty(S * Tw, np.uint32), 0xFFFFFFFF)
    return outs, valid


def _guards(outs, valid, S, T):
    Tw = (T + 31) // 32
    for o in outs:
        assert (o[S * T:].view(np.uint64) == NAN_BITS).all(), "a write past the output"
    assert (valid[S * Tw:] == 0xFFFFFFFF).all(), "a write past the validity words"


def _p(a):
    return None if a is None else C.c_void_p(a.ctypes.data)


def _ptrs(cols):
    arr = (C.c_void_p * len(cols))(*[c.ctypes.data for c in cols])
    return C.cast(arr, C.c_void_p), arr


GRID = dict(start=T0 + 30_000, end=T0 + 30_000 + 40 * 60_000, interval=60_000, lookback=300_000)


def host_entries(ctx, ts, val, sid, offs, S, n_rows=None):
    """every one-shot host entry over one batch -> {name: (rc, results)}"""
    from greptimedb_b200 import make_params
    L, h = ctx._L, ctx._h
    n = ts.size if n_rows is None else n_rows
    g = GRID
    T = orc.num_steps(g["start"], g["end"], g["interval"])
    p = make_params(FN, g["start"], g["end"], g["interval"], g["lookback"])
    res = {}
    outs, valid = _outs(S, T)
    rc = L.b2p_range_eval(h, C.byref(p), _p(ts), _p(val), _p(sid), _p(offs), n, S, _p(outs[0]), _p(valid), None)
    res["range_eval"] = (rc, outs, valid)
    args = (g["start"], g["end"], g["interval"], g["lookback"], 0)
    outs, valid = _outs(S, T)
    rc = L.b2p_instant_select(h, *args, _p(ts), _p(val), _p(sid), _p(offs), n, S, _p(outs[0]), _p(valid))
    res["instant_select"] = (rc, outs, valid)
    outs, valid = _outs(S, T)
    rc = L.b2p_instant_timestamp(h, *args, _p(ts), _p(sid), _p(offs), n, S, _p(outs[0]), _p(valid))
    res["instant_timestamp"] = (rc, outs, valid)
    vals = [val, -val]
    vp, _k1 = _ptrs(vals)
    outs, valid = _outs(S, T, 2)
    op, _k2 = _ptrs(outs)
    rc = L.b2p_range_eval_fields(h, C.byref(p), _p(ts), vp, None, 2, _p(sid), _p(offs), n, S, op, _p(valid))
    res["range_eval_fields"] = (rc, outs, valid)
    outs, valid = _outs(S, T, 2)
    op, _k3 = _ptrs(outs)
    rc = L.b2p_instant_select_fields(h, *args, _p(ts), vp, None, 2, _p(sid), _p(offs), n, S, op, _p(valid))
    res["instant_select_fields"] = (rc, outs, valid)
    # one histogram over every series as a bucket
    hist_off = np.array([0, S], np.uint32)
    bucket_series = np.arange(S, dtype=np.uint32)
    le = np.arange(1, S + 1, dtype=np.float64)
    le[-1] = np.inf
    outs, valid = _outs(1, T)
    rc = L.b2p_range_histogram_fold(h, C.byref(p), _p(ts), _p(val), _p(sid), _p(offs), n, S, 0.9, _p(hist_off),
                                    _p(bucket_series), _p(le), 1, _p(outs[0]), _p(valid))
    res["range_histogram_fold"] = (rc, outs, valid)
    for name, (rc, outs, valid) in res.items():
        _guards(outs, valid, 1 if name == "range_histogram_fold" else S, T)
    return res, T, p


def _one_shot_layouts(sms):
    keep = ("gaps=", "one_row_series", "boundaries")
    for lay in sd.layout_cases(sms, big=False):
        n = lay.ids.size
        if not lay.bad and n >= 8 and any(k in lay.name for k in keep) and (n % 4 or "gaps=" in lay.name) and n < 50_000:
            yield lay


def test_one_shot_host_entries_by_ids_and_by_offsets(ctx, sms):
    ran = 0
    for i, lay in enumerate(_one_shot_layouts(sms)):
        S = lay.n_series
        offs, _ = sd.offsets_fast(lay.ids, S)
        # series start staggered by up to a minute so that the steps fall at different rows of each
        ts, val = _series_columns(offs, i, regular=True, t0s=T0 + (np.arange(S) * 7919 % 60_000))
        by_ids, T, p = host_entries(ctx, ts, val, lay.ids, None, S)
        by_off, _, _ = host_entries(ctx, ts, val, None, offs, S)
        for name in by_ids:
            rc_i, outs_i, valid_i = by_ids[name]
            rc_o, outs_o, valid_o = by_off[name]
            assert rc_i == rc_o == 0, (lay.name, name, rc_i, rc_o)
            assert (valid_i == valid_o).all(), (lay.name, name)
            for a, b in zip(outs_i, outs_o):
                assert (a.view(np.uint64) == b.view(np.uint64)).all(), (lay.name, name)
        _, outs, valid = by_ids["range_eval"]
        e_out, e_valid = orc.range_query(orc.make_params(FN, p.start, p.end, p.interval, p.range), ts, val, None, offs,
                                         threads=4, rescan=True)
        Tw = (T + 31) // 32
        assert (valid[:S * Tw].reshape(S, Tw) == e_valid).all(), lay.name
        g = outs[0][:S * T].reshape(S, T)
        assert ((g.view(np.uint64) == e_out.view(np.uint64)) | (np.isnan(g) & np.isnan(e_out))).all(), lay.name
        assert e_valid.any(), lay.name
        ran += 1
    assert ran >= 20


def test_host_entries_refuse_bad_offsets_and_bad_ids_then_run_exact(ctx, sms):
    """offsets that decrease or end past n_rows: B2P_E_INVALID before any copy; a bad id column: B2P_E_UNSORTED from
    every entry; after each, the context's next call gives the same bits as before"""
    n = 4096 + 15
    ids = sd.ids_from_cuts(n, set(range(100, n, 100)))
    S = int(ids[-1]) + 1
    offs, _ = sd.offsets_fast(ids, S)
    ts, val = _series_columns(offs, 1)
    good, _, _ = host_entries(ctx, ts, val, None, offs, S)
    bad_offs = []
    o = offs.copy(); o[7] = o[8] + 1; bad_offs.append(o)                    # a decrease inside
    o = offs.copy(); o[-1] = n + 1; bad_offs.append(o)                      # past the rows
    o = offs.copy(); o[0] = o[1] + 5; bad_offs.append(o)                    # the first entry past the second
    for o in bad_offs:
        res, _, _ = host_entries(ctx, ts, val, None, o, S)
        for name, (rc, outs, valid) in res.items():
            assert rc == sd.E_INVALID, (name, rc)
            assert (valid[:-GUARD] == 0xFFFFFFFF).all(), f"{name}: results copied back after a refusal"
        again, _, _ = host_entries(ctx, ts, val, None, offs, S)
        for name in good:
            assert again[name][0] == 0 and (again[name][2] == good[name][2]).all(), name
    for lay in sd.bad_cases(sms):
        S2 = lay.n_series
        offs2 = np.linspace(0, lay.ids.size, S2 + 1).astype(np.uint64)
        ts2, val2 = _series_columns(offs2, 2)
        res, _, _ = host_entries(ctx, ts2, val2, lay.ids, None, S2)
        for name, (rc, outs, valid) in res.items():
            assert rc == sd.E_UNSORTED, (lay.name, name, rc)
        again, _, _ = host_entries(ctx, ts, val, ids, None, S)
        for name in good:
            assert again[name][0] == 0 and (again[name][2] == good[name][2]).all(), (lay.name, name)
            for a, b in zip(again[name][1], good[name][1]):
                assert (a.view(np.uint64) == b.view(np.uint64)).all(), (lay.name, name)


# ---- chunked pipeline -------------------------------------------------------------------------------------------
def chunk_layouts():
    """(name, lens, regular per series, grid) of the chunked matrix; lens: rows per series"""
    n_chunk = sd.ONE_SHOT_ROWS + 1
    out = []
    # 6600 series of 1000 rows: two chunks, all described / none described
    out.append(("all_described", np.full(6600, 1000), True))
    out.append(("none_described", np.full(6600, 1000), False))
    # four chunks (C = 4 194 304 // 801 series each), the first and last regular, the middle two not: each buffer pair
    # takes both routes
    C_ = (4 << 20) // 801
    S = 3 * C_ + 100
    reg = np.ones(S, bool)
    reg[C_:3 * C_] = False
    out.append(("alternating", np.full(S, 800), reg))
    # one series longer than a chunk target, among shorter ones: the chunk holding it exceeds the target
    lens = np.full(200, 12_000)
    lens[70] = (4 << 20) + 77
    out.append(("longer_than_a_chunk", lens, True))
    # a chunk whose series are all empty, empty series at chunk starts and ends, trailing empty series; the rows they
    # lose go to other series, so the chunk table (C = 4 194 304 // 701) stays put
    S, C_ = 21000, (4 << 20) // 701
    lens = np.full(S, 700)
    for lo, hi in ((C_, 2 * C_), (0, 5), (C_ - 3, C_), (2 * C_, 2 * C_ + 4), (S - 40, S)):
        lens[lo:hi] = 0
    moved = 700 * S - int(lens.sum())
    lens[3 * C_:3 * C_ + 1000] += moved // 1000
    lens[3 * C_] += moved % 1000
    out.append(("empty_chunk_and_edges", lens, True))
    # the one-shot edge: 6 291 456 against 6 291 457 rows, 63 against 64 series
    lens = np.full(64, sd.ONE_SHOT_ROWS // 64)
    out.append(("rows_at_one_shot", lens, True))
    lens = lens.copy(); lens[-1] += 1
    out.append(("rows_past_one_shot", lens, True))
    lens = np.full(63, n_chunk // 63 + 1)
    out.append(("63_series", lens, True))
    lens = np.full(64, n_chunk // 64 + 1)
    out.append(("64_series", lens, True))
    # the long regular series (i * 15 s past 2^31 ms) inside a described chunk
    lens = np.full(64, 150_000)
    out.append(("long_regular", lens, True))
    return out


def _grid_for(lens):
    """Short series: 16 steps over the first minutes.  Series of more than 4 000 rows: a step every 30 minutes (120
    samples) up to the end of the longest, past row 143 167 where i * 15 s > 2^31 ms.  The steps follow such a series
    to its end, so no sample piles up in the warp tier's ring behind the last step: the series stays off the slow path,
    whose arena would have to hold it whole in each of its warps' regions."""
    from greptimedb_b200 import make_params
    if lens.max() <= 4000:
        return make_params(FN, T0 + 60_000, T0 + 15 * 60_000, 48_000, 120_000)
    return make_params(FN, T0 + 60_000, T0 + int(lens.max()) * SC, 1_800_000, 300_000)


def _offsets(lens):
    return np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)


def _dev_reference(torch, ctx, p, ts, val, offs, S, T):
    d_ts, d_val = torch.from_numpy(ts).cuda(), torch.from_numpy(val).cuda()
    d_off = torch.from_numpy(offs.view(np.int64)).cuda()
    Tw = (T + 31) // 32
    out = torch.zeros(S * T, dtype=torch.float64, device="cuda")
    valid = torch.zeros(S * Tw, dtype=torch.int32, device="cuda")
    ctx.range_eval_dev(p, d_ts, d_val, d_off, ts.size, S, out, valid)
    ctx.sync()
    return out.cpu().numpy().reshape(S, T), valid.cpu().numpy().view(np.uint32).reshape(S, Tw)


def _host_call(torch, c, p, ts, val, sid, offs, S, T, pinned, n_rows=None):
    """b2p_range_eval as bench.py calls it -> (rc, out [S,T], valid [S,Tw], h2d bytes); outputs with guards"""
    Tw = (T + 31) // 32
    n = ts.size if n_rows is None else n_rows

    def buf(a):
        if a is None or not pinned:
            return a
        t = torch.empty(a.size, dtype={8: torch.int64, 4: torch.int32}[a.itemsize], pin_memory=True)
        h = t.numpy().view(a.dtype)
        h[:] = a
        return h
    ts_, val_, sid_, off_ = buf(ts), buf(val), buf(sid), buf(offs)
    outs, valid = _outs(S, T)
    out = outs[0]
    if pinned:
        out = buf(out)
        valid = buf(valid)
    rc = c._L.b2p_range_eval(c._h, C.byref(p), _p(ts_), _p(val_), _p(sid_), _p(off_), n, S, _p(out), _p(valid), None)
    _guards([out], valid, S, T)
    return rc, out[:S * T].reshape(S, T).copy(), valid[:S * Tw].reshape(S, Tw).copy(), c.last_h2d_bytes()


def _same(a, b, what):
    (oa, va), (ob, vb) = a, b
    assert (va == vb).all(), f"{what}: validity differs"
    same = (oa.view(np.uint64) == ob.view(np.uint64)) | (np.isnan(oa) & np.isnan(ob))
    bad = np.argwhere(~same)
    assert not bad.size, f"{what}: {len(bad)} cells differ, first at {bad[:3].tolist()}"


def _oracle_sample(p, ts, val, offs, series, got, what):
    """the rescan oracle over the sampled series alone"""
    series = sorted(set(series))
    lens = np.diff(offs.astype(np.int64))
    rows = np.concatenate([np.arange(int(offs[s]), int(offs[s + 1])) for s in series])
    sub = np.concatenate([[0], np.cumsum(lens[series])]).astype(np.uint64)
    e_out, e_valid = orc.range_query(orc.make_params(FN, p.start, p.end, p.interval, p.range), ts[rows], val[rows],
                                     None, sub, threads=4, rescan=True)
    _same((got[0][series], got[1][series]), (e_out, e_valid), what + " vs oracle")


def _contexts(monkeypatch, scan):
    """a fresh context with the host scan on or off"""
    from greptimedb_b200 import Context
    monkeypatch.setenv("B2P_HOST_TS_SCAN", "1" if scan else "0")
    c = Context(0)
    monkeypatch.delenv("B2P_HOST_TS_SCAN")
    return c


@pytest.mark.parametrize("layout", [x[0] for x in chunk_layouts()])
def test_chunk_pipeline_matrix(torch, ctx, monkeypatch, layout):
    name, lens, regular = next(x for x in chunk_layouts() if x[0] == layout)
    S = lens.size
    offs = _offsets(lens)
    ids = np.repeat(np.arange(S, dtype=np.uint32), lens)
    ts, val = _series_columns(offs, S, regular)
    n = ts.size
    p = _grid_for(lens)
    T = orc.num_steps(p.start, p.end, p.interval)
    ref = _dev_reference(torch, ctx, p, ts, val, offs, S, T)
    assert ref[1].any()
    chunks = sd.plan_chunks(n, S, ids=ids)
    if chunks is not None:
        sd.mark_regular(chunks, ts, ids)
        assert [k.r1 for k in chunks] == [k.r1 for k in sd.plan_chunks(n, S, offsets=offs)]
    if name in ("rows_at_one_shot", "63_series"):
        assert chunks is None
    elif name != "longer_than_a_chunk":
        assert chunks is not None
    if name == "alternating":
        assert [k.regular for k in chunks] == [True, False, False, True]
    if name == "empty_chunk_and_edges":
        assert any(k.r1 == k.r0 for k in chunks)
    sample = [0, S - 1] + [k.s0 for k in chunks or []] + [k.s1 - 1 for k in chunks or []]
    sample += np.random.default_rng(S).integers(0, S, 6).tolist()
    sample = [s for s in sample if lens[s] < 300_000]
    for route in ("scan", "ids", "offsets"):
        c = _contexts(monkeypatch, route == "scan")
        try:
            for pinned in (False, True):
                what = f"{name}/{route}/{'pinned' if pinned else 'pageable'}"
                rc, out, valid, h2d = _host_call(torch, c, p, ts, val, None if route == "offsets" else ids,
                                                 offs if route == "offsets" else None, S, T, pinned)
                assert rc == 0, (what, ctx._L.b2p_last_error())
                _same((out, valid), ref, what)
                # exact: no chunk was redone from its host columns (a redo restages the timestamps and would hide
                # what ts_expand_kernel rebuilt)
                assert h2d == sd.h2d_bytes(n, S, chunks, route), (what, h2d, sd.h2d_bytes(n, S, chunks, route))
            if sample:
                _oracle_sample(p, ts, val, offs, sample, (out, valid), name)
        finally:
            c.close()


def test_rows_outside_every_series_through_offsets(torch, ctx):
    """offsets_host[0] > 0 and offsets_host[n] < n_rows, chunked and one-shot: the same bits as the ids route over the
    rows inside the series, and as the device form"""
    S = 6600
    lens = np.full(S, 1000)
    inner = _offsets(lens)
    head, tail = 4096 + 3, 1001
    offs = inner + np.uint64(head)
    ts_in, val_in = _series_columns(inner, 5, regular=np.arange(S) % 2 == 0)
    rng = np.random.default_rng(3)
    ts = np.concatenate([rng.integers(0, 1 << 62, head), ts_in, rng.integers(0, 1 << 62, tail)]).astype(np.int64)
    val = np.concatenate([np.full(head, 1e300), val_in, np.full(tail, -1e300)])
    ids = np.repeat(np.arange(S, dtype=np.uint32), lens)
    p = _grid_for(lens)
    T = orc.num_steps(p.start, p.end, p.interval)
    ref = _dev_reference(torch, ctx, p, ts, val, offs, S, T)
    chunks = sd.plan_chunks(ts.size, S, offsets=offs)
    assert chunks is not None and chunks[0].r0 == 0 and chunks[-1].r1 == ts.size - tail
    for pinned in (False, True):
        rc, out, valid, h2d = _host_call(torch, ctx, p, ts, val, None, offs, S, T, pinned)
        assert rc == 0
        _same((out, valid), ref, f"offsets/{pinned}")
        assert h2d == sd.h2d_bytes(ts.size, S, chunks, "offsets")
        rc, out2, valid2, _ = _host_call(torch, ctx, p, ts_in, val_in, ids, None, S, T, pinned)
        assert rc == 0
        _same((out2, valid2), ref, f"ids/{pinned}")
    # one shot: the same offsets over a column short enough
    S1 = 600
    offs1 = offs[:S1 + 1]
    ref1 = _dev_reference(torch, ctx, p, ts, val, offs1, S1, T)
    rc, out, valid, _ = _host_call(torch, ctx, p, ts, val, None, offs1, S1, T, False, n_rows=int(offs1[-1]) + 7)
    assert rc == 0
    _same((out, valid), ref1, "one-shot offsets")


def test_chunked_call_refuses_bad_offsets_and_bad_ids(torch, ctx, monkeypatch):
    S, N = 6600, 1000
    offs = _offsets(np.full(S, N))
    ts, val = _series_columns(offs, 9)
    ids = np.repeat(np.arange(S, dtype=np.uint32), N)
    p = _grid_for(np.full(S, N))
    T = orc.num_steps(p.start, p.end, p.interval)
    good = _host_call(torch, ctx, p, ts, val, None, offs, S, T, False)
    assert good[0] == 0
    for k in (5, 4190):   # a decrease inside a chunk, then one at the chunk edge (C = 4190)
        o = offs.copy()
        o[k] = o[k + 1] + 3
        rc, out, valid, _ = _host_call(torch, ctx, p, ts, val, None, o, S, T, True)
        assert rc == sd.E_INVALID and (valid == 0xFFFFFFFF).all()
    o = offs.copy()
    o[-1] = ts.size + 1
    assert _host_call(torch, ctx, p, ts, val, None, o, S, T, False)[0] == sd.E_INVALID
    again = _host_call(torch, ctx, p, ts, val, None, offs, S, T, False)
    _same(again[1:3], good[1:3], "after refusals")
    for scan in (True, False):
        c = _contexts(monkeypatch, scan)
        try:
            for where in ("inside", "tail", "top"):
                bad = ids.copy()
                if where == "inside":
                    bad[10 * N + 5] = 11   # 10, 11, 10: a decrease inside the first chunk
                elif where == "tail":
                    bad[-3:] = S
                else:
                    bad[-1] = 0xFFFFFFFF
                rc = _host_call(torch, c, p, ts, val, bad, None, S, T, scan)[0]
                assert rc == sd.E_UNSORTED, (scan, where, rc)
                rc, out, valid, _ = _host_call(torch, c, p, ts, val, ids, None, S, T, False)
                assert rc == 0
                _same((out, valid), good[1:3], f"after {where}")
        finally:
            c.close()


def test_chunk_redone_beside_described_chunks(torch, monkeypatch):
    """windows longer than the 1024-sample ring over 4000-row jittered series send them to the slow path, which
    overflows a fresh context's arena: their chunk is redone, while the regular short series' chunk goes over as
    descriptors.  The redo's restaging is counted on top."""
    from greptimedb_b200 import make_params
    lens = np.concatenate([np.full(42000, 100), np.full(800, 4000)])
    S = lens.size
    offs = _offsets(lens)
    reg = np.arange(S) < 42000
    ts, val = _series_columns(offs, 4, regular=reg)
    ids = np.repeat(np.arange(S, dtype=np.uint32), lens)
    p = make_params(FN, T0 + 1600 * SC, T0 + 3999 * SC, 750_000, 24_000_000)
    T = orc.num_steps(p.start, p.end, p.interval)
    chunks = sd.mark_regular(sd.plan_chunks(ts.size, S, ids=ids), ts, ids)
    assert chunks[0].regular and not chunks[-1].regular
    c0 = _contexts(monkeypatch, True)
    c0.use_torch_stream()
    try:
        ref = _dev_reference(torch, c0, p, ts, val, offs, S, T)
    finally:
        c0.close()
    c = _contexts(monkeypatch, True)
    try:
        rc, out, valid, h2d = _host_call(torch, c, p, ts, val, ids, None, S, T, True)
        assert rc == 0 and c.last_slow_series() >= 800
        _same((out, valid), ref, "redo")
        long_chunks = [i for i, k in enumerate(chunks) if k.s1 > 42000]
        assert h2d == sd.h2d_bytes(ts.size, S, chunks, "scan", redone=long_chunks), h2d
    finally:
        c.close()


def test_chunked_call_on_the_callers_stream(torch, ctx):
    from greptimedb_b200 import Context
    S, N = 6600, 1000
    offs = _offsets(np.full(S, N))
    ts, val = _series_columns(offs, 12, regular=np.arange(S) % 3 != 0)
    ids = np.repeat(np.arange(S, dtype=np.uint32), N)
    p = _grid_for(np.full(S, N))
    T = orc.num_steps(p.start, p.end, p.interval)
    ref = _dev_reference(torch, ctx, p, ts, val, offs, S, T)
    s = torch.cuda.Stream()
    c = Context(0)
    try:
        with torch.cuda.stream(s):
            c.use_torch_stream()
            rc, out, valid, _ = _host_call(torch, c, p, ts, val, ids, None, S, T, True)
        assert rc == 0
        _same((out, valid), ref, "caller's stream")
    finally:
        c.close()
