"""CPU: tests/time_fn_oracle.py against the reference's goldens (time_fn, timestamp_fn, binary_time_fn and the
EmptyMetric unit vectors) and against Python's datetime over 1900-2100, negative epochs, leap days and years 1 / 9999."""
import calendar
import datetime
import json
import os

import numpy as np
import pytest

from tests import time_fn_oracle as to

GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "reference_time_fn_vectors.json")))
EPOCH = datetime.datetime(1970, 1, 1)


def stamp(ms):
    """a timestamp as the reference's tables print it"""
    t = EPOCH + datetime.timedelta(milliseconds=int(ms))
    s = t.strftime("%Y-%m-%dT%H:%M:%S")
    return s + (f".{t.microsecond // 1000:03d}" if t.microsecond else "")


def printed(v):
    """a Float64 cell as the reference's tables print it (shortest round-trip digits, .0 for integers)"""
    return repr(float(v))


def calendar_cases():
    for c in GOLDEN["cases"]:
        q = c["query"]
        if q.endswith("()") and q[:-2] in to.PARTS and q != "time()":
            yield c


def test_fixture_holds_every_table():
    files = {c["file"] for c in GOLDEN["cases"]}
    assert files == {"time_fn.result", "timestamp_fn.result", "binary_time_fn.result"}
    assert len(GOLDEN["cases"]) == 56 and len(GOLDEN["empty_metric"]) == 5
    assert sum(1 for _ in calendar_cases()) == 22


@pytest.mark.parametrize("case", list(calendar_cases()), ids=lambda c: f"{c['query']}@{c['start_ms']}")
def test_calendar_goldens(case):
    part = case["query"][:-2]
    grid = to.empty_metric_grid(case["start_ms"], case["end_ms"], case["step_ms"])
    want = [(r[0], int(r[1])) for r in case["rows"]]
    got = [(stamp(t), int(to.step_value(part, t))) for t in grid]
    assert got == want
    field = "day" if part == "days_in_month" else to.DATE_PART_FIELD[part]
    assert case["columns"][1].startswith(f'date_part(Utf8("{field}")')


def test_time_goldens():
    for c in GOLDEN["cases"]:
        if c["query"] == "time()":
            grid = to.empty_metric_grid(c["start_ms"], c["end_ms"], c["step_ms"])
            assert [[stamp(t), printed(to.time_value(t))] for t in grid] == c["rows"]
            assert c["columns"] == ["time", "time / Float64(1000)"]


def test_time_is_a_division_not_a_multiplication():
    ts = np.arange(1, 200_000, dtype=np.int64)
    div = to.time_value(ts)
    assert (div == ts.astype(np.float64) / 1000.0).all()
    assert (div != ts.astype(np.float64) * 0.001).any()  # the two differ in the last bit somewhere


def test_empty_metric_unit_vectors():
    for v in GOLDEN["empty_metric"]:
        grid = to.empty_metric_grid(v["start"], v["end"], v["interval"])
        if v["field_expr"] is None:
            assert [[stamp(t)] for t in grid] == v["rows"]
        else:
            assert [[stamp(t), printed(to.time_value(t))] for t in grid] == v["rows"], v["name"]


def test_timestamp_goldens():
    tab = GOLDEN["tables"]["timestamp_test"]["rows"]
    ts = np.array([r[0] for r in tab], np.int64)
    for c in GOLDEN["cases"]:
        if c["query"] not in ("timestamp(timestamp_test)", "-timestamp(timestamp_test)"):
            continue
        out, ok = to.instant_timestamp(ts, [0, ts.size], c["start_ms"], c["end_ms"], c["step_ms"], 300_000)
        grid = to.empty_metric_grid(c["start_ms"], c["end_ms"], c["step_ms"])
        sign = -1.0 if c["query"].startswith("-") else 1.0
        got = [[stamp(grid[k]), printed(np.negative(out[0, k]) if sign < 0 else out[0, k])] for k in range(grid.size) if ok[0, k]]
        assert got == c["rows"], c["query"]
    assert printed(np.negative(to.time_value(0))) == "-0.0"


def test_weekend_golden_steps():
    c = next(c for c in GOLDEN["cases"] if c["file"] == "binary_time_fn.result")
    grid = to.empty_metric_grid(c["start_ms"], c["end_ms"], c["step_ms"])
    dow = to.step_value("day_of_week", grid)
    weekend = {stamp(t) for t, d in zip(grid, dow) if d in (0.0, 6.0)}
    assert {r[0] for r in c["rows"]} <= weekend
    assert stamp(to.days_from_civil(2023, 10, 28) * to.MS_PER_DAY) in weekend  # a Saturday


def _datetime_parts(ms):
    t = EPOCH + datetime.timedelta(milliseconds=int(ms))
    return {"minute": t.minute, "hour": t.hour, "day_of_month": t.day, "day_of_week": (t.weekday() + 1) % 7,
            "day_of_year": t.timetuple().tm_yday, "month": t.month, "year": t.year,
            "days_in_month": calendar.monthrange(t.year, t.month)[1]}


def _check_against_datetime(ms):
    ms = np.asarray(ms, np.int64)
    want = [_datetime_parts(x) for x in ms]
    for part in to.PARTS[1:]:
        got = to.step_value(part, ms)
        assert got.tolist() == [float(w[part]) for w in want], part


def test_every_midnight_1900_2100_against_datetime():
    d0 = (datetime.datetime(1900, 1, 1) - EPOCH).days
    d1 = (datetime.datetime(2100, 12, 31) - EPOCH).days
    mid = np.arange(d0, d1 + 1, dtype=np.int64) * to.MS_PER_DAY
    ms = np.concatenate([mid - 1, mid, mid + 1])[1:]  # (1899-12-31T23:59:59.999 is before the sweep)
    want = {}
    for part, fn in (("year", lambda t: t.year), ("month", lambda t: t.month), ("day_of_month", lambda t: t.day),
                     ("day_of_week", lambda t: (t.weekday() + 1) % 7), ("day_of_year", lambda t: t.timetuple().tm_yday),
                     ("hour", lambda t: t.hour), ("minute", lambda t: t.minute)):
        want[part] = [float(fn(EPOCH + datetime.timedelta(milliseconds=int(x)))) for x in ms]
        assert to.step_value(part, ms).tolist() == want[part], part
    ym = [((EPOCH + datetime.timedelta(milliseconds=int(x))).year, (EPOCH + datetime.timedelta(milliseconds=int(x))).month)
          for x in ms]
    assert to.step_value("days_in_month", ms).tolist() == [float(calendar.monthrange(y, m)[1]) for y, m in ym]


def test_negative_epochs():
    _check_against_datetime([-1, -999, -1000, -86_400_000, -86_400_001, -2_208_988_800_000, -62_135_596_800_000])
    assert to.step_value("hour", -1).item() == 23.0 and to.step_value("minute", -1).item() == 59.0
    assert to.step_value("day_of_week", -1).item() == 3.0  # 1969-12-31 was a Wednesday
    assert to.time_value(-1).item() == -0.001


def test_leap_days():
    for y, leap in ((2000, True), (2100, False), (2400, True)):
        feb = to.days_from_civil(y, 2, 1) * to.MS_PER_DAY
        assert to.step_value("days_in_month", feb).item() == (29.0 if leap else 28.0)
        d = to.days_from_civil(y, 3, 1) * to.MS_PER_DAY - 1  # the last millisecond of February
        assert to.step_value("day_of_month", d).item() == (29.0 if leap else 28.0)
        assert to.step_value("day_of_year", d).item() == (60.0 if leap else 59.0)
    _check_against_datetime([to.days_from_civil(2000, 2, 29) * to.MS_PER_DAY])


def test_years_1_and_9999():
    first = (datetime.datetime(1, 1, 1) - EPOCH).days * to.MS_PER_DAY
    last = (datetime.datetime(9999, 12, 31, 23, 59, 59, 999000) - EPOCH) // datetime.timedelta(milliseconds=1)
    _check_against_datetime([first, first + 1, first + 86_399_999, last, last - 86_400_000])
    assert to.step_value("year", first).item() == 1.0 and to.step_value("year", last).item() == 9999.0
    assert to.step_value("day_of_year", last).item() == 365.0


def test_out_of_range_years():
    edge = to.days_from_civil(to.MAX_YEAR + 1, 1, 1) * to.MS_PER_DAY
    assert to.in_range(edge - 1) and not to.in_range(edge)
    low = to.days_from_civil(-to.MAX_YEAR, 1, 1) * to.MS_PER_DAY
    assert to.in_range(low) and not to.in_range(low - 1)
    assert to.in_range(np.int64(0)) and not to.in_range(np.iinfo(np.int64).max)


def test_instant_timestamp_keeps_the_first_of_equal_timestamps_and_honours_offset():
    ts = np.array([0, 1000, 1000, 5000], np.int64)
    out, ok = to.instant_timestamp(ts, [0, 4], 0, 6000, 1000, 2000, offset=500)
    assert ok[0].tolist() == [False, True, True, True, False, False, True]
    assert out[0, 2] == 1.5 and out[0, 6] == 5.5
    out0, ok0 = to.instant_timestamp(ts, [0, 4], 0, 6000, 1000, 0)
    assert ok0[0].tolist() == [True, True, False, False, False, True, False]


def test_rust_shim_time_enum_layout_compiles():
    """rust-shim/tests/layout_time.c static-asserts the enums ffi.rs mirrors: B2pIfn::Neg, B2pStepPart and
    B2pEmptyMetricKind."""
    import re
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    subprocess.check_call(["gcc", "-std=c11", "-fsyntax-only", "-I" + os.path.join(root, "include"),
                           os.path.join(root, "rust-shim", "tests", "layout_time.c")])
    ffi = open(os.path.join(root, "rust-shim", "src", "ffi.rs")).read()
    assert "Neg = 28," in ffi
    for enum, n in (("B2pStepPart", 9), ("B2pEmptyMetricKind", 3)):
        body = ffi[ffi.index(f"pub enum {enum} {{"):]
        body = body[:body.index("}")]
        assert [int(v) for v in re.findall(r"= (\d+),", body)] == list(range(n)), enum
