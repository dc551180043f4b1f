"""Row-literal restatement of a PromQL subquery fn(<expr>[range:step]) (prom_subquery_expr_to_plan,
src/query/src/promql/planner.rs:292-332): the inner expression is evaluated on its own grid, every valid cell of a child
row is one sample of that row's series (RangeManipulate sits directly on the child: no SeriesNormalize, so NaN is a
sample), and the CPU oracle's range query evaluates the windows over those rows with filter_nan off."""
import numpy as np

from oracle import oracle as orc


def inner_grid(start, end, interval, range_ms, step=None):
    """The inner expression's grid: (start', step', T') with step' = step or the outer interval and
    start' = start - range + step'; the end is the outer end."""
    step = interval if step is None else step
    s = start - range_ms + step
    return s, step, orc.num_steps(s, end, step)


def grid_to_rows(vals, valid_words, inner_start, inner_interval):
    """child grid -> (ts, val, offsets): row r's valid cells k, in step order, as samples (start' + k * step', cell)"""
    vals = np.asarray(vals, np.float64)
    R, T = vals.shape
    bits = orc.valid_to_bool(np.ascontiguousarray(valid_words, np.uint32).reshape(R, -1), T)
    ts, val, offsets = [], [], [0]
    for r in range(R):
        for k in range(T):
            if bits[r, k]:
                ts.append(inner_start + k * inner_interval)
                val.append(vals[r, k])
        offsets.append(len(ts))
    return np.array(ts, np.int64), np.array(val, np.float64), np.array(offsets, np.uint64)


def subquery(fn, start, end, interval, range_ms, inner_start, inner_interval, vals, valid_words, param0=0.0, param1=0.0):
    """-> (out [R x T], valid words [R x Tw]) of fn over the rows of the child grid"""
    ts, val, offsets = grid_to_rows(vals, valid_words, inner_start, inner_interval)
    p = orc.make_params(fn, start, end, interval, range_ms, filter_nan=False, param0=param0, param1=param1)
    return orc.range_query(p, ts, val, None, offsets)


def instant_child(ts, val, start, end, interval, lookback):
    """The instant selector of one series on a grid (InstantManipulate): (vals [1 x T], valid words [1 x Tw])"""
    offsets = np.array([0, len(ts)], np.uint64)
    return orc.instant_query(np.asarray(ts, np.int64), np.asarray(val, np.float64), offsets, start, end, interval,
                             lookback)
