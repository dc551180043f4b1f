"""Plain restatement of the reference's time functions, for the CPU and GPU tests of K19, the timestamp mode of K4 and
the plan nodes above them.

- time(): `CAST(CAST(ts AS Int64) AS Float64) / 1000.0` (build_special_time_expr, empty_metric.rs:393-402): a
  round-to-nearest conversion, then one IEEE division (not a multiplication by 0.001).
- The calendar functions: DataFusion's date_part on a UTC millisecond timestamp (planner.rs:2222-2300, 3994-4009),
  restated over integer days with floor division (so negative epochs work): minute, hour, day, dow (Sunday = 0),
  doy (from 1), month, year, and days_in_month = the day of date_trunc('month', t) + 1 month - 1 day.
- EmptyMetric's grid: start, start + interval, .. <= end, none when start > end (empty_metric.rs).
- timestamp(<selector>): InstantManipulate (instant_manipulate.rs:473-585) over the sample timestamps without the
  stale-NaN test, the value being the chosen sample's ts + offset over 1000.

Everything works on numpy int64 arrays (or Python ints) elementwise.
"""
import numpy as np

PARTS = ["time", "minute", "hour", "day_of_month", "day_of_week", "day_of_year", "month", "year", "days_in_month"]
# the date_part field each calendar function asks DataFusion for
DATE_PART_FIELD = {"minute": "minute", "hour": "hour", "day_of_month": "day", "day_of_week": "dow",
                   "day_of_year": "doy", "month": "month", "year": "year"}
MAX_YEAR = 262143  # chrono's NaiveDate range; beyond it the library refuses the step
MS_PER_DAY = 86_400_000


def time_value(ts):
    """time() / timestamp() value of a millisecond timestamp: (double)ts / 1000.0"""
    return np.asarray(ts, np.int64).astype(np.float64) / 1000.0


def civil(days):
    """days since 1970-01-01 -> (year, month, day), proleptic Gregorian (H. Hinnant's civil_from_days)"""
    z = np.asarray(days, np.int64) + 719468
    era = z // 146097
    doe = z - era * 146097
    yoe = (doe - doe // 1460 + doe // 36524 - doe // 146096) // 365
    doy = doe - (365 * yoe + yoe // 4 - yoe // 100)
    mp = (5 * doy + 2) // 153
    d = doy - (153 * mp + 2) // 5 + 1
    m = np.where(mp < 10, mp + 3, mp - 9)
    y = yoe + era * 400 + (m <= 2)
    return y, m, d


def days_from_civil(y, m, d):
    y = np.asarray(y, np.int64) - (np.asarray(m) <= 2)
    era = y // 400
    yoe = y - era * 400
    doy = (153 * np.where(m > 2, m - 3, m + 9) + 2) // 5 + d - 1
    doe = yoe * 365 + yoe // 4 - yoe // 100 + doy
    return era * 146097 + doe - 719468


def is_leap(y):
    y = np.asarray(y, np.int64)
    return ((y % 4 == 0) & (y % 100 != 0)) | (y % 400 == 0)


def in_range(ts):
    """the steps the library computes (the others are refused)"""
    y, _, _ = civil(np.asarray(ts, np.int64) // MS_PER_DAY)
    return (y >= -MAX_YEAR) & (y <= MAX_YEAR)


def step_value(part, ts):
    """f(ts) of one part (a name of PARTS) as the Float64 a grid cell holds"""
    ts = np.asarray(ts, np.int64)
    if part == "time":
        return time_value(ts)
    days = ts // MS_PER_DAY
    ms = ts - days * MS_PER_DAY
    y, m, d = civil(days)
    if part == "minute":
        v = ms // 60_000 % 60
    elif part == "hour":
        v = ms // 3_600_000
    elif part == "day_of_month":
        v = d
    elif part == "day_of_week":
        v = (days + 4) % 7  # 1970-01-01 was a Thursday
    elif part == "day_of_year":
        v = days - days_from_civil(y, 1, 1) + 1
    elif part == "month":
        v = m
    elif part == "year":
        v = y
    elif part == "days_in_month":
        v = np.where(m == 2, np.where(is_leap(y), 29, 28), np.where(np.isin(m, [4, 6, 9, 11]), 30, 31))
    else:
        raise KeyError(part)
    return np.asarray(v, np.int64).astype(np.float64)


def step_fn(part, eval_ts, ok):
    """K19 over a grid: f(eval_ts[k]) where ok[r, k], 0.0 elsewhere"""
    v = step_value(part, eval_ts)
    return np.where(ok, v[None, :], 0.0)


def empty_metric_grid(start, end, interval):
    return np.arange(start, end + 1, interval, dtype=np.int64) if start <= end else np.zeros(0, np.int64)


def instant_timestamp(ts, offsets, start, end, interval, lookback, offset=0):
    """timestamp(<selector>) over series offsets -> (out [S,T] f64, ok [S,T] bool): per step the newest sample with
    t - lookback < ts + offset <= t (ts + offset == t when lookback is 0), the first of several rows sharing that
    timestamp, valued (ts + offset) / 1000; no stale-NaN test"""
    ts = np.asarray(ts, np.int64)
    grid = empty_metric_grid(start, end, interval)
    S, T = len(offsets) - 1, grid.size
    out = np.zeros((S, T))
    ok = np.zeros((S, T), bool)
    for s in range(S):
        t = ts[offsets[s]:offsets[s + 1]] + offset
        for k, te in enumerate(grid):
            j = int(np.searchsorted(t, te, side="right")) - 1
            if j < 0:
                continue
            fresh = t[j] + lookback > te if lookback > 0 else t[j] == te
            if fresh:
                ok[s, k] = True
                out[s, k] = float(t[j]) / 1000.0
    return out, ok
