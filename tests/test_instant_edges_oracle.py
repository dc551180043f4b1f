"""The instant selector's edge cases on the CPU: the literal interpreter of the reference's cursor walk
(tests/instant_edges.py) against the C oracle's restatement (orc.instant_query) and the Int64 selector of
tests/int64_oracle.py on every generated case, and against the committed goldens that pin InstantManipulate.  No
device is needed."""
import numpy as np
import pytest

from oracle import oracle as orc
from tests import instant_edges as ie
from tests import int64_oracle as io
from tests.helpers import farr, fnum, load_sqlness, load_unit, pack_series

CASES = ie.cases()
UNIT = load_unit()
SQL = load_sqlness()


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.name)
def test_interpreter_matches_the_c_oracle(case):
    out, valid = orc.instant_query(case.ts, case.val, case.offsets, case.start, case.end, case.interval, case.lookback,
                                   case.offset)
    want, want_valid = ie.expected_values(case, [case.val])
    why = ie.first_difference(out.view(np.uint64), want[0], valid, want_valid, case.T)
    assert not why, f"{case.describe()}: C oracle vs interpreter: {why}"


@pytest.mark.parametrize("case", [c for c in CASES if c.offset == 0], ids=lambda c: c.name)
def test_interpreter_matches_the_int64_selector(case):
    """no staleness test (an Int64 field 0, whatever its bits): every NaN pattern is taken"""
    outs, ok = io.instant_select(case.ts, [case.val.view(np.int64)], case.offsets, case.start, case.end,
                                 case.interval, case.lookback)
    want, want_valid = ie.expected_values(case, [case.val], stale=False)
    why = ie.first_difference(outs.view(np.uint64), want, ie.valid_words(ok), want_valid, case.T)
    assert not why, f"{case.describe()}: Int64 selector vs interpreter: {why}"


def test_every_class_runs():
    ran = set().union(*(c.classes for c in CASES))
    assert ran == ie.CLASSES, f"classes no case hits: {sorted(ie.CLASSES - ran)}"


def test_the_large_cases_are_large():
    """the binary search runs at least 17 levels, and warps stride over the series"""
    sizes = np.concatenate([np.diff(c.offsets.astype(np.int64)) for c in CASES])
    assert sizes.max() >= 1 << 17
    big = max(CASES, key=lambda c: c.S)
    strided = np.diff(big.offsets.astype(np.int64))[ie.WARPS_LAUNCHED:]
    assert (strided > 0).sum() >= ie.STRIDED - 1, "series a warp takes on its second pass hold rows"


def test_stale_and_timestamp_selections_differ_only_at_nan_rows():
    """value mode drops exactly the NaN rows timestamp mode takes"""
    for c in CASES:
        a, b = c.rows(stale=True), c.rows(stale=False)
        kept = a >= 0
        assert (a[kept] == b[kept]).all(), c.describe()
        dropped = (b >= 0) & ~kept
        assert np.isnan(c.val[b[dropped]]).all(), c.describe()


def _grid_rows(names, ts, val, offsets, start, end, interval, lookback, offset):
    """{(series name, step ts): value} of the interpreter's walk over packed series"""
    got = {}
    for s, name in enumerate(names):
        r0, r1 = int(offsets[s]), int(offsets[s + 1])
        shifted = [int(t) + offset for t in ts[r0:r1]]
        for t, j in ie.interpret(shifted, val[r0:r1].tolist(), start, end, interval, lookback):
            got[(name, t)] = float(val[r0 + j])
    return got


@pytest.mark.parametrize("case", SQL["instant_cases"] + SQL.get("instant_offset_direction_cases", []),
                         ids=lambda c: c["name"])
def test_interpreter_reproduces_the_sqlness_goldens(case):
    names, ts, val, sid, offsets = pack_series(case["series"])
    got = _grid_rows(names, ts, val, offsets, case["start"], case["end"], case["interval"], case["lookback"],
                     case["offset"])
    assert got == {(n, t): fnum(v) for n, t, v in case["expected"]}


@pytest.mark.parametrize("case", UNIT["instant_manipulate"]["cases"], ids=lambda c: c["name"])
def test_interpreter_reproduces_the_unit_goldens(case):
    g = UNIT["instant_manipulate"]
    d = g["data_nan"] if case["nan"] else g["data"]
    val = farr(d["val"])
    taken = ie.interpret(list(d["ts"]), val.tolist(), case["start"], case["end"], case["interval"], case["lookback"])
    assert [t for t, _ in taken] == case["out_ts"]
    if "out_val" in case:
        assert [float(val[j]) for _, j in taken] == case["out_val"]


def test_interpreter_takes_the_first_row_of_a_run_on_the_step():
    """rows sharing the eval timestamp: the first is taken, or nothing when it is NaN, whatever the later rows hold;
    between steps the last row of the run is taken"""
    nan = float("nan")
    ts = [1000, 2000, 2000, 2000, 2500, 2500]
    for v, want in (([0.0, 1.0, 2.0, 3.0, 4.0, 5.0], [(1000, 0), (2000, 1), (3000, 5)]),
                    ([0.0, nan, 2.0, 3.0, 4.0, nan], [(1000, 0)]),
                    ([0.0, 1.0, nan, nan, nan, 5.0], [(1000, 0), (2000, 1), (3000, 5)])):
        assert ie.interpret(ts, v, 1000, 3000, 1000, 1000) == want
    assert ie.interpret(ts, [nan] * 6, 1000, 3000, 1000, 1000, stale=False) == [(1000, 0), (2000, 1), (3000, 5)]


def test_interpreter_lookback_edges():
    """a sample exactly `lookback` before the step is too old, `lookback - 1` before is taken; lookback 0 takes only
    a sample on the step"""
    assert ie.interpret([0, 10_000], [1.0, 2.0], 5000, 15_000, 5000, 5000) == [(10_000, 1)]
    assert ie.interpret([0, 10_000], [1.0, 2.0], 4999, 14_999, 5000, 5000) == [(4999, 0), (14_999, 1)]
    assert ie.interpret([0, 10_000], [1.0, 2.0], 0, 20_000, 5000, 0) == [(0, 0), (10_000, 1)]
    assert ie.interpret([-7, 3], [1.0, 2.0], -10, 10, 1, 1) == [(-7, 0), (3, 1)]
