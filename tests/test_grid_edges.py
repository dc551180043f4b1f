"""CPU: the references and layout cases of tests/grid_edges.py — each reference against the existing oracle of its
kernel on the cases they both cover, the calendar against datetime and against time_fn_oracle over the whole
+-262143-year range, time() and i64_to_f64 against exact rational arithmetic, and every layout class present."""
import datetime
from fractions import Fraction

import numpy as np
import pytest

from tests import absent_oracle as ao
from tests import binary_oracle as bor
from tests import grid_edges as ge
from tests import instant_fn_oracle as ifo
from tests import set_oracle as so
from tests import time_fn_oracle as to

CASES = ge.grid_cases()


def bits(x):
    return np.ascontiguousarray(x, np.float64).view(np.uint64)


def test_every_layout_class_runs():
    want = {f"T={T}" for T in ge.T_LIST} | {f"valid:{p}" for p in ge.PATTERNS} | {
        "junk_past_T", "invalid:nan_both_signs", "invalid:inf_both_signs", "route:vec", "route:scalar_odd",
        "route:scalar_even_unaligned", "inplace", "outofplace", "k19:rows_per_warp", "k19:W=96", "k19:W=160",
        "k19:W=192", "k19:W=224", "k19:second_y_pass", "k15:shared", "k15:rows", "k15:columns", "k15:T=1_over_2^20_rows",
        "scalar:one_key_disjoint", "scalar:one_key_overlap", "scalar:no_key_one_cell", "scalar:no_key_two_cells",
        "scalar:two_keys"}
    for sms in (132, 114, 78):  # the grid-stride and geometry classes hold for any SM count
        got = ge.all_classes(sms)
        assert want <= got, sorted(want - got)


def test_T_list_covers_the_unit_residues():
    assert {T % 64 for T in ge.T_LIST if T % 2 == 0} >= {0, 2, 30, 32, 34, 62}
    assert {T % 32 for T in ge.T_LIST if T % 2} >= {1, 31}  # a word with only its first step, or all but its last
    assert {ge.step_fn_geometry(132, T, 1)["W"] for T in (65, 129, 161, 193)} == {96, 160, 192, 224}


def test_cases_hold_their_classes():
    for c in CASES:
        T, ok, valid = c["T"], c["ok"], c["valid"]
        assert (ge.ok_of(valid, T) == ok).all()
        m = ge.past_t_mask(T)
        if m:
            assert (valid[:, -1] & np.uint32(m)).all(), "every row's last word carries junk past T"
        assert not (ge.words_of(ok)[:, -1] & np.uint32(m)).any()
        inv = bits(c["vals"][~ok])
        assert np.isin(inv, bits(ge.INVALID_FILL)).all()


def test_geometry_sizes_force_a_second_pass():
    for sms in (132, 114):
        for T, rows in ge.K19_SHAPES(sms)[-4:]:
            assert ge.step_fn_geometry(sms, T, rows)["second_pass"]
        for T, steps in ((1000, 64), (999, 32), (1000, 32)):
            assert ge.rows_past_warp_grid(sms, T, steps) * -(-T // steps) > sms * 16 * 8
        assert ge.absent_regime(sms, 2 ** 20, 1) == "shared"


# ---- references against the existing oracles ------------------------------------------------------------------------
@pytest.mark.parametrize("op,rb", [("+", False), ("-", False), ("*", False), ("/", False), ("%", False), ("^", False),
                                   ("atan2", False), (">", False), ("==", True), ("<=", False), ("!=", True)])
def test_binary_ref_matches_binary_oracle(op, rb):
    for i, c in enumerate(CASES):
        other = CASES[(i + 5) % len(CASES)]
        if other["T"] != c["T"]:
            other = c
        lrow = np.array([0, 3, 1, 2], np.uint32)
        rrow = np.array([2, 0, 3, 1], np.uint32)
        x, y = c["vals"][lrow], other["vals"][rrow]
        exp, ev = ge.binary_ref(op, x, y, c["ok"][lrow] & other["ok"][rrow], x, rb)
        got, gv = bor.binary_op(op, c["vals"], c["valid"], lrow, other["vals"], other["valid"], rrow, return_bool=rb)
        assert (gv == ev).all()
        same = (bits(got) == bits(exp)) | (np.isnan(got) & np.isnan(exp))
        assert same.all(), op
        for left in (False, True):
            s = 0.5
            xs, ys = (np.full_like(c["vals"], s), c["vals"]) if left else (c["vals"], np.full_like(c["vals"], s))
            exp, ev = ge.binary_ref(op, xs, ys, c["ok"], c["vals"], rb)
            got, gv = bor.scalar_op(op, s, c["vals"], c["valid"], scalar_on_left=left, return_bool=rb)
            assert (gv == ev).all()
            assert ((bits(got) == bits(exp)) | (np.isnan(got) & np.isnan(exp))).all(), op


@pytest.mark.parametrize("op", ["and", "or", "unless"])
def test_setop_ref_matches_set_oracle(op):
    keys = {"and": ([0, so.NO_KEY, 1, 0], [1, 0, 2, 1]), "unless": ([0, so.NO_KEY, 1, 2], [1, 0, 2, 1]),
            "or": ([0, 1, so.NO_KEY, 0], [1, 2, 0, so.NO_KEY])}[op]
    lk, rk = np.array(keys[0], np.uint32), np.array(keys[1], np.uint32)
    for i, c in enumerate(CASES):
        other = CASES[(i + 1) % len(CASES)]
        if other["T"] != c["T"]:
            continue
        exp, ev = ge.setop_ref(op, c["vals"], c["ok"], lk, other["vals"], other["ok"], rk, 3)
        got, gv = so.setop(op, c["vals"], c["valid"], lk, other["vals"], other["valid"], rk, 3)
        assert (gv == ev).all() and (bits(got) == bits(exp)).all(), (op, c["T"], c["pattern"])


@pytest.mark.parametrize("fn", ["abs", "sgn", "clamp", "floor"])
def test_instant_fn_ref_matches_instant_fn_oracle(fn):
    a0, a1, _, keeps_nan = ge.INSTANT_FNS[fn]
    for c in CASES:
        exp = ge.instant_fn_ref(fn, c["vals"], c["ok"])
        got, gv = ifo.instant_fn(fn, c["vals"], c["valid"], a0, a1)
        assert (gv == c["valid"]).all()
        same = bits(got) == bits(exp)
        if not keeps_nan:
            same |= np.isnan(got) & np.isnan(exp)
        assert same.all(), fn
    v = ge.VALID_FILL
    assert (bits(ge.instant_fn_ref("neg", v[None, :], np.ones((1, v.size), bool))[0]) ==
            (bits(v) ^ np.uint64(1 << 63))).all()


def test_scalar_ref_matches_instant_fn_oracle():
    for name, vals, ok, valid, key, overlap in ge.scalar_cases():
        exp, ev, ov = ge.scalar_ref(vals, ok, key)
        assert ov == overlap, name
        if overlap:
            with pytest.raises(ValueError):
                ifo.scalar_calculate(vals, valid, key)
            continue
        got, gv = ifo.scalar_calculate(vals, valid, key)
        assert (gv == ev).all() and (bits(got) == bits(exp)).all(), name


def test_absent_and_count_valid_refs():
    for c in CASES:
        out, words = ge.absent_ref(c["ok"])
        o2, w2 = ao.absent_words(c["ok"], c["T"])
        assert (words == w2).all() and (bits(out) == bits(o2)).all()
        cnt = np.where(c["ok"], np.arange(1, c["ok"].size + 1).reshape(c["ok"].shape), 0)
        assert (ge.count_valid_ref(cnt) == ge.words_of(c["ok"])).all()
    # the K15 shapes: per-row stripes leave steps no row claims
    for rows, T in ge.ABSENT_SHAPES[:2]:
        ok = np.zeros((rows, T), bool)
        for r in range(rows):
            ok[r, r::rows + 1] = True
        out, _ = ge.absent_ref(ok)
        assert out.any() and not out.all()
        assert ao.absent_steps(0, T - 1, 1, ok) == [k for k in range(T) if out[k] == 1.0]


def test_subquery_rows():
    ok = np.array([[1, 0, 1, 1, 0], [0, 0, 0, 0, 0], [0, 0, 0, 0, 1]], bool)
    vals = np.arange(15.0).reshape(3, 5)
    ts, val, off = ge.subquery_rows(vals, ok, -5_000, 1000)
    assert ts.tolist() == [-5_000, -3_000, -2_000, -1_000] and val.tolist() == [0.0, 2.0, 3.0, 14.0]
    assert off.tolist() == [0, 3, 3, 4]


# ---- calendar, time() and i64_to_f64 --------------------------------------------------------------------------------------
def test_calendar_walk_agrees_with_datetime():
    rng = np.random.default_rng(1)
    ords = np.concatenate([rng.integers(1, datetime.date.max.toordinal() + 1, 20_000),
                           [1, 59, 60, 365, 366, datetime.date.max.toordinal()]])
    for o in ords.tolist():
        d = datetime.date.fromordinal(o)
        assert ge.civil_walk(o) == (d.year, d.month, d.day, d.timetuple().tm_yday), o


def test_calendar_agrees_with_time_fn_oracle_over_the_year_range():
    rng = np.random.default_rng(2)
    lo, hi = ge.ms_of(-ge.MAX_YEAR, 1, 1), ge.ms_of(ge.MAX_YEAR + 1, 1, 1) - 1
    ts = np.concatenate([rng.integers(lo, hi, 20_000, dtype=np.int64), ge.calendar_steps(),
                         ge.calendar_edge_steps()["in"]])
    ts[::3] = ts[::3] // ge.MS_PER_DAY * ge.MS_PER_DAY + rng.integers(-1, 2, ts[::3].size)
    ts = ts[(ts >= lo) & (ts <= hi)]
    for part in to.PARTS:
        want = to.step_value(part, ts)
        got = np.array([ge.calendar(part, t) for t in ts.tolist()], np.float64)
        assert (bits(got) == bits(want)).all(), part
    assert to.in_range(ts).all()
    out = ge.calendar_edge_steps()["out"]
    assert all(ge.calendar("year", t) is None for t in out.tolist()) and not to.in_range(out).any()


def test_calendar_fixed_dates():
    ms = lambda y, m, d: ge.ms_of(y, m, d)
    assert ms(1970, 1, 1) == 0 and ms(2000, 3, 1) - ms(2000, 2, 28) == 2 * ge.MS_PER_DAY
    assert ms(1900, 3, 1) - ms(1900, 2, 28) == ge.MS_PER_DAY and ms(2100, 3, 1) - ms(2100, 2, 28) == ge.MS_PER_DAY
    assert ms(2400, 3, 1) - ms(2400, 2, 28) == 2 * ge.MS_PER_DAY and ms(-400, 3, 1) - ms(-400, 2, 28) == 2 * ge.MS_PER_DAY
    assert ge.calendar("days_in_month", ms(-400, 2, 10)) == 29.0 and ge.calendar("days_in_month", ms(-100, 2, 10)) == 28.0
    assert ge.calendar("day_of_year", ms(2000, 12, 31)) == 366.0 and ge.calendar("day_of_year", ms(-1, 1, 1)) == 1.0
    assert ge.calendar("day_of_week", ms(2024, 6, 9)) == 0.0  # a Sunday
    assert ge.calendar("year", ms(0, 6, 1)) == 0.0 and ge.calendar("day_of_year", ms(0, 12, 31)) == 366.0
    last = ms(ge.MAX_YEAR + 1, 1, 1) - 1
    assert ge.calendar("month", last) == 12.0 and ge.calendar("minute", last) == 59.0
    assert ge.calendar("year", last + 1) is None and ge.calendar("year", ms(-ge.MAX_YEAR, 1, 1) - 1) is None


def test_time_and_i64_to_f64_are_correctly_rounded():
    for t in ge.TIME_EDGES.tolist():
        assert ge.time_correctly_rounded(t)
        assert ge.calendar("time", t) == float(Fraction(float(t)) / 1000)
    assert ge.calendar("time", np.iinfo(np.int64).max) == float(2 ** 63) / 1000.0
    want = ge.i64_to_f64_ref(ge.I64_EDGES)
    for v, w in zip(ge.I64_EDGES.tolist(), want.tolist()):
        f = Fraction(v)
        lo, hi = np.nextafter(w, -np.inf), np.nextafter(w, np.inf)
        assert abs(Fraction(w) - f) <= abs(Fraction(lo) - f) and abs(Fraction(w) - f) <= abs(Fraction(hi) - f), v
    assert (bits(want) == bits(ge.I64_EDGES.astype(np.float64))).all()
    assert ge.i64_to_f64_ref([2 ** 53 + 1])[0] == 2.0 ** 53 and ge.i64_to_f64_ref([2 ** 54 + 2])[0] == 2.0 ** 54
    assert ge.i64_to_f64_ref([2 ** 54 + 6])[0] == 2.0 ** 54 + 8
