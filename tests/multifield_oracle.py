"""CPU restatement of PromQL selectors over a table with several Float64 field columns, over the single-field oracle.

GreptimeDB plans every field of such a table at once:
  (1) SeriesNormalize with need_filter_out_nan drops a row when ANY Float64 column is NaN (normalize.rs:415-428), so a
      NaN in one field removes that sample from the windows of every field;
  (2) RangeManipulate carries all field columns (range_manipulate.rs:70-153) with windows from the timestamps alone,
      the prom_* UDF is projected once per field (planner.rs:2180) and the closing Filter is the conjunction of
      `IS NOT NULL` over every field (planner.rs:2774-2791): a (series, step) cell is kept only where every field's
      result is;
  (3) InstantManipulate is handed the first field only (planner.rs:922): its lookback walk and stale-NaN test read
      field 0 (instant_manipulate.rs:555-575) and every field is then taken from the chosen row;
  (4) NULL field slots: the NaN filter reads the buffer value (`value(i)`), and so do the range functions in
      BUFFER_FNS (`values()`: extrapolate_rate.rs, idelta.rs, resets.rs, changes.rs, last_over_time, quantile.rs,
      double_exponential_smoothing.rs) or they read only the window's length (count / present / absent_over_time).
      The functions in NULL_FNS see NULL slots: arrow's null-skipping sum / min / max (sum, avg, min, max_over_time;
      avg divides by the length, NULLs included), `value.unwrap()` (stdvar / stddev_over_time panic) and
      linear_regression_slices' `is_null` skip (deriv, predict_linear; functions.rs:126-144).  The device reproduces
      the first family from the buffers and refuses the second over a NULL slot, as it refuses any NULL slot in an
      instant selection (the reference exports it as a NULL in that field of an emitted row).
"""
import numpy as np

from oracle import oracle as orc

NULL_FNS = {"sum_over_time", "avg_over_time", "min_over_time", "max_over_time", "stdvar_over_time", "stddev_over_time",
            "deriv", "predict_linear"}
BUFFER_FNS = {"rate", "increase", "delta", "irate", "idelta", "resets", "changes", "last_over_time",
              "quantile_over_time", "holt_winters", "count_over_time", "present_over_time", "absent_over_time"}


class NullSlotRefused(ValueError):
    pass


def check_null_slots(fn, present):
    """(4): the refusal of a call over NULL slots (fn None: an instant selection); present: per-field masks or None"""
    if present is None:
        return
    for f, m in enumerate(present):
        if m is not None and not np.asarray(m, bool).all() and (fn is None or fn in NULL_FNS):
            raise NullSlotRefused(f"field {f} has NULL slots")


def nan_union(vals):
    """(1): every field of a row in which any field is NaN becomes NaN (the row is dropped from all of them)."""
    vals = [np.array(v, np.float64) for v in vals]
    if not vals:
        return vals
    bad = np.zeros(vals[0].shape, bool)
    for v in vals:
        bad |= np.isnan(v)
    for v in vals:
        v[bad & ~np.isnan(v)] = np.nan
    return vals


def range_query_fields(p, ts, vals, offsets, present=None, **kw):
    """(1) + (2) + (4) -> (outs [F, S, T], valid_words [S, Tw]): one single-field range query per field over the shared
    windows (the value buffers as they are, NULL slots included), then the conjunction of the per-field validity."""
    check_null_slots({v: k for k, v in orc.FN_IDS.items()}[p.fn_id], present)
    cols = nan_union(vals) if p.filter_nan else [np.asarray(v, np.float64) for v in vals]
    res = [orc.range_query(p, ts, v, None, offsets, **kw) for v in cols]
    valid = res[0][1].copy()
    for _, w in res[1:]:
        valid &= w
    return np.stack([o for o, _ in res]), valid


def instant_query_fields(ts, vals, offsets, start, end, interval, lookback, offset=0, present=None):
    """(3) -> (outs [F, S, T], valid_words [S, Tw]): the cells and rows of field 0's instant query; every other field
    is read from the row field 0's query chose (a NaN there is exported as it is)."""
    check_null_slots(None, present)
    ts = np.asarray(ts, np.int64)
    offsets = np.asarray(offsets, np.uint64)
    out0, valid = orc.instant_query(ts, vals[0], offsets, start, end, interval, lookback, offset)
    # the chosen row: the single-field query over the row index as the value column picks the same row wherever field
    # 0's cell is valid (field 0 decides staleness, so a row index stands in for every other field)
    rows = np.arange(ts.size, dtype=np.float64)
    idx_cells, idx_valid = orc.instant_query(ts, np.where(np.isnan(vals[0]), np.nan, rows), offsets, start, end,
                                             interval, lookback, offset)
    assert (idx_valid == valid).all()
    ok = orc.valid_to_bool(valid, out0.shape[1])
    outs = []
    for v in vals:
        v = np.asarray(v, np.float64)
        o = np.zeros(out0.shape, np.float64)
        o[ok] = v[idx_cells[ok].astype(np.int64)]
        outs.append(o)
    return np.stack(outs), valid
