"""CPU: the multi-field restatement (tests/multifield_oracle.py) against independent statements of the same rules."""
import numpy as np
import pytest

from oracle import oracle as orc
from tests import multifield_oracle as mf

T0 = 1_700_000_000_000
FNS = list(orc.FN_IDS)
PARAMS = {"predict_linear": (600.0, 0.0), "quantile_over_time": (0.9, 0.0), "holt_winters": (0.3, 0.1)}


def table(seed, S=6, n=40, F=3, jitter=True):
    """S series of n rows 15 s apart (jittered), F NaN-free gauge / counter fields"""
    rng = np.random.default_rng(seed)
    ts = np.concatenate([T0 + np.arange(n) * 15_000 + (rng.integers(0, 4000, n) if jitter else 0) for _ in range(S)])
    offsets = np.arange(S + 1, dtype=np.uint64) * n
    vals = [np.cumsum(rng.uniform(0, 5, S * n)) if f % 2 == 0 else rng.normal(0, 10, S * n) for f in range(F)]
    return ts.astype(np.int64), vals, offsets


def params(fn, filter_nan=True):
    p0, p1 = PARAMS.get(fn, (0.0, 0.0))
    return orc.make_params(fn, T0 + 60_000, T0 + 600_000, 30_000, 120_000, filter_nan=filter_nan, param0=p0, param1=p1)


def test_nan_union_marks_every_field_of_a_row():
    a = np.array([1.0, np.nan, 3.0, 4.0])
    b = np.array([np.nan, 2.0, 3.0, 4.0])
    c = np.array([1.0, 2.0, 3.0, -np.nan])
    u = mf.nan_union([a, b, c])
    for v in u:
        assert np.isnan(v).tolist() == [True, True, False, True]
    assert np.isnan(a).tolist() == [False, True, False, False]  # the inputs stay as they were


@pytest.mark.parametrize("fn", FNS)
def test_nan_free_fields_are_the_single_field_results(fn):
    """F NaN-free fields: each field is exactly its single-field query, and the windows (so the validity) are shared."""
    ts, vals, offsets = table(1)
    p = params(fn)
    outs, valid = mf.range_query_fields(p, ts, vals, offsets)
    for f, v in enumerate(vals):
        o, w = orc.range_query(p, ts, v, None, offsets)
        ok = orc.valid_to_bool(valid, o.shape[1])
        assert np.array_equal(o[ok].view(np.uint64), outs[f][ok].view(np.uint64))
        assert (w & valid == valid).all()
    o0, w0 = orc.range_query(p, ts, vals[0], None, offsets)
    assert (valid == w0).all()


@pytest.mark.parametrize("fn", FNS)
@pytest.mark.parametrize("j", [0, 2])
def test_one_nan_removes_the_sample_from_every_field(fn, j):
    """A NaN in field j at row r: every field's result is the single-field query over the table without row r."""
    ts, vals, offsets = table(2)
    r = 47  # series 1, row 7
    vals[j][r] = np.nan
    p = params(fn)
    outs, valid = mf.range_query_fields(p, ts, vals, offsets)
    keep = np.arange(ts.size) != r
    off2 = offsets.copy()
    off2[2:] -= 1
    cut = [orc.range_query(p, ts[keep], v[keep], None, off2) for v in vals]
    exp_valid = cut[0][1].copy()
    for _, w in cut[1:]:
        exp_valid &= w
    assert (valid == exp_valid).all()
    ok = orc.valid_to_bool(valid, outs.shape[2])
    for f in range(len(vals)):
        a, b = outs[f][ok], cut[f][0][ok]
        assert np.array_equal(np.isnan(a), np.isnan(b))
        assert np.array_equal(a[~np.isnan(a)].view(np.uint64), b[~np.isnan(b)].view(np.uint64))


def test_without_filter_nan_fields_do_not_couple():
    ts, vals, offsets = table(3)
    vals[1][10] = np.nan
    p = params("sum_over_time", filter_nan=False)
    outs, _ = mf.range_query_fields(p, ts, vals, offsets)
    o0, w0 = orc.range_query(p, ts, vals[0], None, offsets)
    ok = orc.valid_to_bool(w0, o0.shape[1])
    assert np.array_equal(outs[0][ok], o0[ok])


def test_instant_selection_reads_staleness_from_field_zero():
    # one series: rows at 0, 10, 20 s; field 0 is NaN (stale) at 20 s, field 1 is NaN at 10 s
    ts = np.array([T0, T0 + 10_000, T0 + 20_000], np.int64)
    f0 = np.array([1.0, 2.0, np.nan])
    f1 = np.array([10.0, np.nan, 30.0])
    offsets = np.array([0, 3], np.uint64)
    outs, valid = mf.instant_query_fields(ts, [f0, f1], offsets, T0, T0 + 20_000, 10_000, 300_000)
    assert orc.valid_to_bool(valid, 3)[0].tolist() == [True, True, False]
    assert outs[0][0, :2].tolist() == [1.0, 2.0]
    assert outs[1][0, 0] == 10.0 and np.isnan(outs[1][0, 1])  # field 1's NaN is a value, not a stale marker
    # swapping the fields moves the staleness test with field 0
    outs2, valid2 = mf.instant_query_fields(ts, [f1, f0], offsets, T0, T0 + 20_000, 10_000, 300_000)
    assert orc.valid_to_bool(valid2, 3)[0].tolist() == [True, False, True]
    assert outs2[1][0, 0] == 1.0 and np.isnan(outs2[1][0, 2])


def test_instant_fields_pick_field_zeros_row():
    ts, vals, offsets = table(4, jitter=True)
    vals[0][::7] = np.nan
    outs, valid = mf.instant_query_fields(ts, vals, offsets, T0, T0 + 600_000, 20_000, 45_000)
    o0, w0 = orc.instant_query(ts, vals[0], offsets, T0, T0 + 600_000, 20_000, 45_000)
    assert (valid == w0).all() and np.array_equal(outs[0], o0)


def test_null_slot_families_cover_every_function():
    assert mf.NULL_FNS.isdisjoint(mf.BUFFER_FNS) and mf.NULL_FNS | mf.BUFFER_FNS == set(orc.FN_IDS)


@pytest.mark.parametrize("fn", FNS)
def test_null_slots_read_the_buffer_or_are_refused(fn):
    """(4): with a NULL slot, a buffer-reading function gives what the buffer gives; a NULL-skipping one is refused"""
    ts, vals, offsets = table(5)
    present = [None, np.arange(ts.size) % 11 != 3, None]
    p = params(fn)
    if fn in mf.NULL_FNS:
        with pytest.raises(mf.NullSlotRefused, match="field 1"):
            mf.range_query_fields(p, ts, vals, offsets, present=present)
    else:
        a = mf.range_query_fields(p, ts, vals, offsets, present=present)
        b = mf.range_query_fields(p, ts, vals, offsets)
        assert np.array_equal(a[1], b[1]) and np.array_equal(a[0].view(np.uint64), b[0].view(np.uint64))
    full = [np.ones(ts.size, bool)] * 3
    mf.range_query_fields(p, ts, vals, offsets, present=full)  # no NULL slot: never refused
