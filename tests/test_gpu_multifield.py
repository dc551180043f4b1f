"""GPU: the selectors over several field columns (b2p_range_eval_fields[_dev], b2p_instant_select_fields[_dev]; K16-K18
in b2p_fields.cuh) against the CPU restatement in tests/multifield_oracle.py, bit for bit, and against the single-field
entry points they extend."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import oracle as orc
from tests import multifield_oracle as mf

pytestmark = pytest.mark.gpu

T0 = 1_700_000_000_000
STEP = 15_000
PARAMS = {"predict_linear": (600.0, 0.0), "quantile_over_time": (0.9, 0.0), "holt_winters": (0.3, 0.1)}


@pytest.fixture(scope="module")
def ctx():
    from greptimedb_b200 import Context
    c = Context(0)
    yield c
    c.close()


def table(rows, F, seed, nan_rate=0.03, jitter=4000):
    """`rows` rows over a few series (series 1 empty when there are several), F fields with NaNs sprinkled into single
    fields -> (ts, vals, offsets)"""
    rng = np.random.default_rng(seed)
    S = 1 if rows <= 1 else max(3, rows // 100)
    cuts = np.sort(rng.integers(0, rows + 1, S - 1)) if S > 1 else np.array([], np.int64)
    if S > 1:
        cuts[0] = cuts[1] if S > 2 else cuts[0]  # series 1 has no rows
    offsets = np.concatenate([[0], cuts, [rows]]).astype(np.uint64)
    ts = np.zeros(rows, np.int64)
    for s in range(S):
        a, b = int(offsets[s]), int(offsets[s + 1])
        ts[a:b] = T0 + np.arange(b - a) * STEP + (rng.integers(0, jitter, b - a) if jitter else 0)
    vals = []
    for f in range(F):
        v = np.cumsum(rng.uniform(0, 5, rows)) if f % 2 == 0 else rng.normal(0, 10, rows)
        v[rng.random(rows) < nan_rate / F] = np.nan
        vals.append(v)
    return ts, vals, offsets


def grid(T):
    return T0, T0 + (T - 1) * 20_000, 20_000


def same_bits(a, b):
    """equal cell for cell; NaNs match as NaNs"""
    a, b = np.asarray(a), np.asarray(b)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint64), b[~nb].view(np.uint64))


def tail_clear(valid, T):
    return T % 32 == 0 or not (valid[:, -1] >> np.uint32(T % 32)).any()


def params(fn, T, rng=60_000, filter_nan=True):
    from greptimedb_b200 import make_params
    p0, p1 = PARAMS.get(fn, (0.0, 0.0))
    start, end, itv = grid(T)
    return (make_params(fn, start, end, itv, rng, filter_nan=filter_nan, param0=p0, param1=p1),
            orc.make_params(fn, start, end, itv, rng, filter_nan=filter_nan, param0=p0, param1=p1))


def expect_range(op, ts, vals, offsets):
    outs, valid = mf.range_query_fields(op, ts, vals, offsets, rescan=True)
    return outs, valid


def check_range(outs, valid, e_outs, e_valid, T):
    assert np.array_equal(valid, e_valid)
    assert tail_clear(valid, T)
    ok = orc.valid_to_bool(valid, T)
    for f in range(len(e_outs)):
        assert same_bits(outs[f][ok], e_outs[f][ok]), f"field {f}"


# ---- K16 + range tiers + K18, host form -------------------------------------------------------------------------------
@pytest.mark.parametrize("T", [1, 31, 32, 33, 1000])
@pytest.mark.parametrize("rows", [0, 1, 5, 10_000])
@pytest.mark.parametrize("F", [1, 2, 3, 8])
def test_range_fields_shapes(ctx, T, rows, F):
    ts, vals, offsets = table(rows, F, seed=T * 7 + rows + F)
    p, op = params("sum_over_time", T)
    outs, valid = ctx.range_eval_fields(p, ts, vals, offsets=offsets)
    check_range(outs, valid, *expect_range(op, ts, vals, offsets), T)


@pytest.mark.parametrize("T", [1, 31, 32, 33, 1000])
@pytest.mark.parametrize("rows", [0, 1, 5, 10_000])
@pytest.mark.parametrize("F", [1, 2, 3, 8])
def test_instant_fields_shapes(ctx, T, rows, F):
    ts, vals, offsets = table(rows, F, seed=T * 11 + rows + F, nan_rate=0.2)
    start, end, itv = grid(T)
    outs, valid = ctx.instant_select_fields(ts, vals, start, end, itv, 45_000, offsets=offsets)
    e_outs, e_valid = mf.instant_query_fields(ts, vals, offsets, start, end, itv, 45_000)
    assert np.array_equal(valid, e_valid) and tail_clear(valid, T)
    assert np.array_equal(outs.view(np.uint64), e_outs.view(np.uint64))  # gathered bits, NaN payloads included


# ---- every range function on the range tiers ---------------------------------------------------------------------------
TIERS = {"default": {}, "warp": {"B2P_DISABLE_LEAN_TIER": "1"}, "flags": {"B2P_LEAN_FORCE_FLAGS": "1",
                                                                          "B2P_LEAN_ADAPTIVE": "0"}}


@pytest.fixture(scope="module", params=list(TIERS))
def tier_ctx(request):
    from greptimedb_b200 import Context
    env = TIERS[request.param]
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        c = Context(0)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    yield c
    c.close()


@pytest.mark.parametrize("fn", list(orc.FN_IDS))
@pytest.mark.parametrize("jitter", [0, 4000])
def test_every_function_on_every_tier(tier_ctx, fn, jitter):
    """NaNs in single fields; regular scrapes reach the first tier's uniform-cadence form, jittered ones its general
    form; long windows (range 40 scrapes) the 1024-sample ring"""
    ts, vals, offsets = table(20_000, 3, seed=5 + jitter, jitter=jitter)
    for rng in (60_000, 600_000):
        p, op = params(fn, 120, rng=rng)
        outs, valid = tier_ctx.range_eval_fields(p, ts, vals, offsets=offsets)
        check_range(outs, valid, *expect_range(op, ts, vals, offsets), 120)


def test_nans_in_single_fields_without_filter(ctx):
    """filter_nan = 0: a field's NaN stays a sample of that field only; the cell is still conjoined"""
    ts, vals, offsets = table(5_000, 3, seed=9, nan_rate=0.1)
    p, op = params("max_over_time", 200, filter_nan=False)
    outs, valid = ctx.range_eval_fields(p, ts, vals, offsets=offsets)
    check_range(outs, valid, *expect_range(op, ts, vals, offsets), 200)


# ---- against the single-field entry points -----------------------------------------------------------------------------
def dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def run_dev(ctx, kind, ts, vals, offsets, T, p=None, start=None):
    import torch
    S = offsets.size - 1
    Tw = (T + 31) // 32
    d_vals = [dev(v) for v in vals]
    outs = [torch.full((S, T), -1.0, dtype=torch.float64, device="cuda") for _ in vals]
    valid = torch.zeros((S, Tw), dtype=torch.int32, device="cuda")
    if kind == "range":
        ctx.range_eval_fields_dev(p, dev(ts), d_vals, dev(offsets), ts.size, S, outs, valid)
    else:
        s, e, itv = grid(T)
        ctx.instant_select_fields_dev(s, e, itv, 45_000, 0, dev(ts), d_vals, dev(offsets), ts.size, S, outs, valid)
    ctx.sync()
    torch.cuda.synchronize()
    return [o.cpu().numpy() for o in outs], valid.cpu().numpy().view(np.uint32), [v.cpu().numpy() for v in d_vals]


def run_single_dev(ctx, kind, ts, val, offsets, T, p=None):
    import torch
    S = offsets.size - 1
    out = torch.full((S, T), -1.0, dtype=torch.float64, device="cuda")
    valid = torch.zeros((S, (T + 31) // 32), dtype=torch.int32, device="cuda")
    if kind == "range":
        ctx.range_eval_dev(p, dev(ts), dev(val), dev(offsets), ts.size, S, out, valid)
    else:
        s, e, itv = grid(T)
        ctx.instant_select_dev(s, e, itv, 45_000, 0, dev(ts), dev(val), dev(offsets), ts.size, S, out, valid)
    ctx.sync()
    torch.cuda.synchronize()
    return out.cpu().numpy(), valid.cpu().numpy().view(np.uint32)


@pytest.mark.parametrize("kind", ["range", "instant"])
def test_one_field_is_the_single_field_call(ctx, kind):
    ts, vals, offsets = table(10_000, 1, seed=21, nan_rate=0.05)
    p, _ = params("rate", 300)
    outs, valid, _ = run_dev(ctx, kind, ts, vals, offsets, 300, p)
    out1, valid1 = run_single_dev(ctx, kind, ts, vals[0], offsets, 300, p)
    assert np.array_equal(valid, valid1)
    assert np.array_equal(outs[0].view(np.uint64), out1.view(np.uint64))


@pytest.mark.parametrize("kind", ["range", "instant"])
def test_identical_fields_give_identical_grids(ctx, kind):
    ts, vals, offsets = table(10_000, 1, seed=22, nan_rate=0.05)
    p, _ = params("rate", 300)
    outs, valid, _ = run_dev(ctx, kind, ts, [vals[0], vals[0].copy()], offsets, 300, p)
    out1, valid1 = run_single_dev(ctx, kind, ts, vals[0], offsets, 300, p)
    assert np.array_equal(valid, valid1)
    ok = orc.valid_to_bool(valid, 300)
    for o in outs:
        assert np.array_equal(o[ok].view(np.uint64), out1[ok].view(np.uint64))


@pytest.mark.parametrize("kind", ["range", "instant"])
def test_host_and_device_forms_agree(ctx, kind):
    ts, vals, offsets = table(10_000, 4, seed=23, nan_rate=0.1)
    p, _ = params("delta", 300)
    outs, valid, d_vals_after = run_dev(ctx, kind, ts, vals, offsets, 300, p)
    if kind == "range":
        h_outs, h_valid = ctx.range_eval_fields(p, ts, vals, offsets=offsets)
        sid = np.repeat(np.arange(offsets.size - 1, dtype=np.uint32), np.diff(offsets).astype(np.int64))
        s_outs, s_valid = ctx.range_eval_fields(p, ts, vals, sid=sid)
    else:
        s, e, itv = grid(300)
        h_outs, h_valid = ctx.instant_select_fields(ts, vals, s, e, itv, 45_000, offsets=offsets)
        sid = np.repeat(np.arange(offsets.size - 1, dtype=np.uint32), np.diff(offsets).astype(np.int64))
        s_outs, s_valid = ctx.instant_select_fields(ts, vals, s, e, itv, 45_000, sid=sid)
    assert np.array_equal(valid, h_valid) and np.array_equal(valid, s_valid)
    ok = orc.valid_to_bool(valid, 300)
    for f in range(4):
        assert np.array_equal(outs[f][ok].view(np.uint64), h_outs[f][ok].view(np.uint64))
        assert np.array_equal(outs[f][ok].view(np.uint64), s_outs[f][ok].view(np.uint64))
        assert np.array_equal(d_vals_after[f].view(np.uint64), vals[f].view(np.uint64))  # the caller's columns stay


def test_instant_staleness_reads_field_zero_only(ctx):
    ts = np.array([T0, T0 + 20_000, T0 + 40_000], np.int64)
    f0 = np.array([1.0, 2.0, np.nan])
    f1 = np.array([10.0, np.nan, 30.0])
    offsets = np.array([0, 3], np.uint64)
    outs, valid = ctx.instant_select_fields(ts, [f0, f1], T0, T0 + 40_000, 20_000, 45_000, offsets=offsets)
    assert orc.valid_to_bool(valid, 3)[0].tolist() == [True, True, False]
    assert outs[0][0].tolist() == [1.0, 2.0, 0.0]
    assert outs[1][0, 0] == 10.0 and np.isnan(outs[1][0, 1]) and outs[1][0, 2] == 0.0


def test_nan_in_one_field_drops_the_row_from_every_field(ctx):
    """last_over_time over one series: the NaN in field 1 at the last row makes every field read the row before"""
    ts = np.array([T0, T0 + 10_000, T0 + 20_000], np.int64)
    f0 = np.array([1.0, 2.0, 3.0])
    f1 = np.array([10.0, 20.0, np.nan])
    from greptimedb_b200 import make_params
    p = make_params("last_over_time", T0 + 20_000, T0 + 20_000, 10_000, 60_000)
    outs, valid = ctx.range_eval_fields(p, ts, [f0, f1], offsets=np.array([0, 3], np.uint64))
    assert valid[0, 0] == 1 and outs[0][0, 0] == 2.0 and outs[1][0, 0] == 20.0


# ---- refusals -----------------------------------------------------------------------------------------------------------
def test_null_and_out_of_range_arguments(ctx):
    from greptimedb_b200 import make_params
    from greptimedb_b200.engine import _ptr
    L = ctx._L
    ts = np.array([T0, T0 + 15_000], np.int64)
    a = np.array([1.0, 2.0])
    b = np.array([3.0, 4.0])
    off = np.array([0, 2], np.uint64)
    out = [np.full(4, -7.0), np.full(4, -7.0)]
    valid = np.full(1, 7, np.uint32)
    p = make_params("sum_over_time", T0, T0 + 45_000, 15_000, 60_000)
    arr = lambda cols: (C.c_void_p * 2)(*[_ptr(x) for x in cols])
    good_v, good_o = arr([a, b]), arr(out)

    def calls(vals, n, outs, h=ctx._h):
        yield L.b2p_range_eval_fields(h, C.byref(p), _ptr(ts), vals, None, n, None, _ptr(off), 2, 1, outs, _ptr(valid))
        yield L.b2p_instant_select_fields(h, T0, T0 + 45_000, 15_000, 60_000, 0, _ptr(ts), vals, None, n, None,
                                          _ptr(off), 2, 1, outs, _ptr(valid))

    for vals, n, outs in [(good_v, 0, good_o), (good_v, 65, good_o), (None, 2, good_o), (good_v, 2, None),
                          (arr([a, None]), 2, good_o), (arr([a, b]), 2, arr([out[0], None]))]:
        v = C.cast(vals, C.c_void_p) if vals is not None else None
        o = C.cast(outs, C.c_void_p) if outs is not None else None
        for rc in calls(v, n, o):
            assert rc == -1
    for rc in calls(C.cast(good_v, C.c_void_p), 2, C.cast(good_o, C.c_void_p), h=None):
        assert rc == -1
    assert all((o == -7.0).all() for o in out) and valid.tolist() == [7]  # a refused call writes nothing
    # device forms: NULL pointer arrays and NULL columns
    d_ts, d_off = dev(ts), dev(off)
    import torch
    d_out = [torch.zeros(4, dtype=torch.float64, device="cuda") for _ in range(2)]
    d_valid = torch.zeros(1, dtype=torch.int32, device="cuda")
    dv, do = arr([dev(a), dev(b)]), arr(d_out)
    assert L.b2p_range_eval_fields_dev(ctx._h, C.byref(p), _ptr(d_ts), None, None, 2, _ptr(d_off), 2, 1,
                                       C.cast(do, C.c_void_p), _ptr(d_valid)) == -1
    assert L.b2p_range_eval_fields_dev(ctx._h, C.byref(p), _ptr(d_ts), C.cast(dv, C.c_void_p), None, 2,
                                       _ptr(d_off), 2, 1,
                                       C.cast(do, C.c_void_p), None) == -1
    assert L.b2p_instant_select_fields_dev(ctx._h, T0, T0 + 45_000, 15_000, 60_000, 0, None, C.cast(dv, C.c_void_p),
                                           None, 2, _ptr(d_off), 2, 1, C.cast(do, C.c_void_p), _ptr(d_valid)) == -1
    assert L.b2p_instant_select_fields_dev(ctx._h, T0, T0 + 45_000, 15_000, 60_000, 0, _ptr(d_ts),
                                           C.cast(arr([dev(a), None]), C.c_void_p), None, 2, _ptr(d_off), 2, 1,
                                           C.cast(do, C.c_void_p), _ptr(d_valid)) == -1
    assert "NULL" in L.b2p_last_error().decode()


# ---- NULL field slots -------------------------------------------------------------------------------------------------
def null_table(seed):
    """NaN-free fields with NULL slots in field 1: the slots' buffer values are 0.0, as arrow's builders leave them"""
    ts, vals, offsets = table(10_000, 3, seed=seed, nan_rate=0.0)
    present = [None, np.random.default_rng(seed).random(ts.size) > 0.05, None]
    vals[1][~present[1]] = 0.0
    return ts, vals, offsets, present


@pytest.mark.parametrize("fn", sorted(mf.BUFFER_FNS))
def test_null_slots_of_buffer_reading_functions_read_the_buffer(ctx, fn):
    ts, vals, offsets, present = null_table(31)
    p, op = params(fn, 300)
    outs, valid = ctx.range_eval_fields(p, ts, vals, offsets=offsets, present=present)
    check_range(outs, valid, *mf.range_query_fields(op, ts, vals, offsets, present=present, rescan=True), 300)
    plain = ctx.range_eval_fields(p, ts, vals, offsets=offsets)
    assert np.array_equal(valid, plain[1]) and np.array_equal(outs.view(np.uint64), plain[0].view(np.uint64))


@pytest.mark.parametrize("fn", sorted(mf.NULL_FNS))
def test_null_slots_of_null_skipping_functions_are_refused(ctx, fn):
    from greptimedb_b200 import B2PError
    ts, vals, offsets, present = null_table(32)
    p, _ = params(fn, 300)
    with pytest.raises(B2PError, match="field 1 has NULL slots"):
        ctx.range_eval_fields(p, ts, vals, offsets=offsets, present=present)
    # the device form reads the bitmaps on the device
    S = offsets.size - 1
    import torch
    outs = [torch.zeros((S, 300), dtype=torch.float64, device="cuda") for _ in vals]
    valid = torch.zeros((S, 10), dtype=torch.int32, device="cuda")
    bms = [None, dev(np.packbits(present[1], bitorder="little")), None]
    with pytest.raises(B2PError, match="field 1 has NULL slots"):
        ctx.range_eval_fields_dev(p, dev(ts), [dev(v) for v in vals], dev(offsets), ts.size, S, outs, valid,
                                  field_valid=bms)
    # bitmaps without a NULL slot in rows [0, n_rows) (stray bits past the last row ignored) are accepted
    full = [np.ones(ts.size, bool)] * 3
    a = ctx.range_eval_fields(p, ts, vals, offsets=offsets, present=full)
    b = ctx.range_eval_fields(p, ts, vals, offsets=offsets)
    assert np.array_equal(a[1], b[1]) and np.array_equal(a[0].view(np.uint64), b[0].view(np.uint64))


def test_one_field_with_null_slots_follows_the_same_rule(ctx):
    from greptimedb_b200 import B2PError
    ts, vals, offsets, present = null_table(33)
    p, _ = params("avg_over_time", 300)
    with pytest.raises(B2PError, match="field 0 has NULL slots"):
        ctx.range_eval_fields(p, ts, [vals[1]], offsets=offsets, present=[present[1]])
    p, _ = params("rate", 300)
    ctx.range_eval_fields(p, ts, [vals[1]], offsets=offsets, present=[present[1]])


def test_instant_selection_with_null_slots_is_refused(ctx):
    from greptimedb_b200 import B2PError
    ts, vals, offsets, present = null_table(34)
    s, e, itv = grid(300)
    with pytest.raises(B2PError, match="field 1 has NULL slots"):
        ctx.instant_select_fields(ts, vals, s, e, itv, 45_000, offsets=offsets, present=present)
    full = [np.ones(ts.size, bool)] * 3
    a = ctx.instant_select_fields(ts, vals, s, e, itv, 45_000, offsets=offsets, present=full)
    b = ctx.instant_select_fields(ts, vals, s, e, itv, 45_000, offsets=offsets)
    assert np.array_equal(a[1], b[1]) and np.array_equal(a[0].view(np.uint64), b[0].view(np.uint64))
