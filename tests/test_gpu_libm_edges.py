"""GPU: the results this library takes from CUDA's libm — K9's transcendental functions and K7's `^` / `atan2` — on the
operand classes of tests/libm_cases.py, through every route that reaches them: the host API, the device API in place
and out of place with even T (128-bit path) and odd T, and K7's vector form and both scalar forms.

  exact classes      bit for bit equal to glibc;
  threshold classes  ±inf exactly where glibc has it, the same zero / subnormal / normal outcome, and the same sign of
                     every zero and every infinity;
  every other class  within ULP_BOUND / POW_ATAN2_ULPS of glibc (tests/ulp_bounds.py).
The exceptions are named in tests/ulp_bounds.py with their measured sizes: CLASS_ULPS (cos / tan at the worst argument
reduction, where glibc is the one off) and UNDERFLOW_TO_ZERO (exp / pow give +0 where glibc gives 2^-1074).

With $B2P_LIBM_REPORT set, the largest distance from glibc and from the correctly rounded result per (function, class)
is written there as JSON.  A plan-layer check holds the exported Float64 of log2, log10, x ^ 2 and 2 ^ x to glibc's, so
that log2(8) prints 3."""
import json
import math
import os

import numpy as np
import pytest

from tests import instant_fn_oracle as ifo
from tests import libm_cases as lc
from tests.instant_fn_helpers import same_value
from tests.ulp_bounds import CLASS_ULPS, POW_ATAN2_ULPS, ULP_BOUND, UNDERFLOW_TO_ZERO, ulp_distance

pytestmark = pytest.mark.gpu
CASES = lc.cases()
UNARY = [c for c in CASES if c.fn in lc.UNARY]
BINARY = [c for c in CASES if c.fn in lc.BINARY]
OP = {"pow": "^", "atan2": "atan2"}
REPORT = {}


def _id(c):
    return f"{c.fn}-{c.cls}"


def bits(x):
    return np.ascontiguousarray(x, np.float64).view(np.uint64)


@pytest.fixture(scope="module")
def ctx():
    from greptimedb_b200 import Context
    c = Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    path = os.environ.get("B2P_LIBM_REPORT")
    if not path:
        return
    out = {}
    for c in CASES:
        if _id(c) not in REPORT:
            continue
        got = REPORT[_id(c)]
        cr = lc.correctly_rounded(c.fn, c.x, c.y)
        g = lc.glibc(c.fn, c.x, c.y)
        out[_id(c)] = {"fn": c.fn, "class": c.cls, "kind": c.kind, "n": int(c.x.size),
                       "glibc_ulps": max(float(ulp_distance(r, g).max(initial=0)) for r in got),
                       "cr_ulps": max(float(ulp_distance(r, cr).max(initial=0)) for r in got),
                       "glibc_cr_ulps": float(ulp_distance(g, cr).max(initial=0))}
    with open(path, "w") as f:
        json.dump(out, f, indent=1)


def check(c, got, route):
    """got: the device's results for c's operands, in order."""
    REPORT.setdefault(_id(c), []).append(np.array(got, np.float64))
    g = lc.glibc(c.fn, c.x, c.y)
    where = f"{_id(c)} via {route}"
    assert (np.isnan(got) == np.isnan(g)).all(), f"{where}: NaN at {c.x[np.isnan(got) != np.isnan(g)][:4]}"
    if c.kind == "exact":
        bad = bits(got) != bits(g)
        assert not bad.any(), f"{where}: {got[bad][:4]} where glibc gives {g[bad][:4]} (x = {c.x[bad][:4]})"
    elif c.kind == "threshold":
        assert (np.isinf(got) == np.isinf(g)).all(), f"{where}: overflows elsewhere than glibc: {got} vs {g}"
        differ = lc.outcome(got) != lc.outcome(g)
        if (c.fn, c.cls) in UNDERFLOW_TO_ZERO:   # +0 only where glibc gives the smallest subnormal
            assert (bits(got[differ]) == 0).all() and (g[differ] == lc.TINY).all(), f"{where}: {got} vs glibc {g}"
            differ[:] = False
        assert not differ.any(), f"{where}: {lc.outcome(got)} vs glibc {lc.outcome(g)}"
        edge = (got == 0) | np.isinf(got) | (g == 0) | np.isinf(g)
        assert (np.signbit(got[edge]) == np.signbit(g[edge])).all(), f"{where}: the sign of a zero or an infinity"
    else:
        bound = CLASS_ULPS.get((c.fn, c.cls), POW_ATAN2_ULPS if c.fn in lc.BINARY else ULP_BOUND[c.fn])
        d = ulp_distance(got, g)
        assert d.max(initial=0) <= bound, \
            f"{where}: {d.max()} ulps from glibc at x = {c.x[d > bound][:4]}" + ("" if c.y is None else f", y = {c.y[d > bound][:4]}")


def padded(x, parity):
    """x as one row of T cells with T % 2 == parity (a trailing 1.0 pads it), and its all-valid words."""
    x = np.asarray(x, np.float64)
    row = x if x.size % 2 == parity else np.append(x, 1.0)
    return row.reshape(1, -1), ifo._words(np.ones((1, row.size), bool))


@pytest.mark.parametrize("c", UNARY, ids=_id)
def test_instant_fn_host_api(ctx, c):
    for parity in (0, 1):
        vals, words = padded(c.x, parity)
        out, _ = ctx.instant_fn(c.fn, vals, words)
        check(c, out[0, :c.x.size], f"host API, T % 2 = {parity}")


@pytest.mark.parametrize("c", UNARY, ids=_id)
def test_instant_fn_device_api(ctx, c):
    """Out of place and in place, even T (the 128-bit path) and odd T, over three rows."""
    import torch
    for parity in (0, 1):
        row, _ = padded(c.x, parity)
        vals = np.repeat(row, 3, axis=0)
        T = vals.shape[1]
        words = ifo._words(np.ones(vals.shape, bool))
        dv = torch.from_numpy(vals.copy()).cuda()
        dw = torch.from_numpy(words.view(np.int32).copy()).cuda()
        out = torch.full_like(dv, 7.0)
        ow = torch.zeros_like(dw)
        ctx.instant_fn_dev(c.fn, dv, dw, 3, T, out, ow)
        ctx.instant_fn_dev(c.fn, dv, dw, 3, T, dv, dw)
        ctx.sync()
        for r in range(3):
            check(c, out.cpu().numpy()[r, :c.x.size], f"device API out of place, T % 2 = {parity}")
            check(c, dv.cpu().numpy()[r, :c.x.size], f"device API in place, T % 2 = {parity}")
        assert (ow.cpu().numpy() == dw.cpu().numpy()).all()


@pytest.mark.parametrize("c", BINARY, ids=_id)
def test_binary_vector_form(ctx, c):
    for parity in (0, 1):
        lhs, words = padded(c.x, parity)
        rhs, _ = padded(c.y, parity)
        out, _ = ctx.binary_op(OP[c.fn], lhs, words, [0], rhs, words, [0])
        check(c, out[0, :c.x.size], f"vector form, T % 2 = {parity}")


@pytest.mark.parametrize("c", BINARY, ids=_id)
@pytest.mark.parametrize("left", [True, False], ids=["scalar_left", "scalar_right"])
def test_binary_scalar_forms(ctx, c, left):
    """`s op v` with each distinct lhs as the scalar, and `v op s` with each distinct rhs."""
    scalar, vector = (c.x, c.y) if left else (c.y, c.x)
    got = np.full(c.x.size, np.nan)
    for s in np.unique(bits(scalar)):
        idx = np.flatnonzero(bits(scalar) == s)
        vals, words = padded(vector[idx], idx.size % 2)
        out, _ = ctx.scalar_op(OP[c.fn], float(np.uint64(s).view(np.float64)), vals, words, scalar_on_left=left)
        got[idx] = out[0, :idx.size]
    check(c, got, "scalar " + ("left" if left else "right"))


def test_plan_layer_prints_glibc(ctx):
    """log2 of powers of two, log10 of powers of ten, x ^ 2 of integers and 2 ^ x of integers through an instant leaf:
    each exported Float64 is glibc's exact value, compared as the goldens' printed values are, so log2(8) prints 3."""
    import pyarrow as pa
    from greptimedb_b200.plan import PromRangeExec

    def exported(xs, stage):
        n = xs.size
        node = PromRangeExec(ctx, "", 0, (n - 1) * 5000, 5000, 0, "ts", "val", ["host"], lookback_delta=1000)
        node.push(pa.RecordBatch.from_pydict({"ts": pa.array(np.arange(n) * 5000, pa.timestamp("ms")),
                                              "val": pa.array(xs, pa.float64()),
                                              "host": pa.array(["a"] * n, pa.utf8())}))
        b = stage(node).execute()
        v = [f for f in b.schema if pa.types.is_float64(f.type)]
        assert len(v) == 1 and b.num_rows == n
        order = np.argsort(b.column("ts").cast(pa.int64()).to_numpy())
        return np.array(b.column(v[0].name).to_pylist())[order]

    p2 = np.concatenate([[8.0], np.ldexp(1.0, np.arange(-1074, 1024, 7))])
    ints = np.arange(-40.0, 41.0)
    for name, xs, stage, want in (
            ("log2", p2, lambda n: n.function("log2"), ifo.apply("log2", p2)),
            ("log10", 10.0 ** np.arange(0, 23), lambda n: n.function("log10"), np.arange(0.0, 23.0)),
            ("x ^ 2", ints, lambda n: n.scalar_op("^", 2.0), lc.glibc("pow", ints, np.full(ints.size, 2.0))),
            ("2 ^ x", np.arange(-1074.0, 1024.0, 13), lambda n: n.scalar_op("^", 2.0, scalar_on_left=True),
             np.ldexp(1.0, np.arange(-1074, 1024, 13)))):
        got = exported(xs, stage)
        for x, g, w in zip(xs, got, want):
            assert same_value(repr(float(w)), g), f"{name}({x!r}) exports {g!r}, glibc prints {w!r}"
        assert (bits(got) == bits(want)).all(), name
    assert exported(np.array([8.0]), lambda n: n.function("log2"))[0] == 3.0


def test_pow_atan2_ulp_bound_over_a_million_operands(ctx):
    """The largest distance from glibc of `^` and `atan2` over 2^20 seeded random pairs each (the measurement behind
    POW_ATAN2_ULPS; in $B2P_LIBM_REPORT under "random pow" / "random atan2")."""
    n = 1 << 20
    rng = np.random.default_rng(0xA7A2)
    sign = np.where(rng.random(n) < 0.15, -1.0, 1.0)
    y = rng.uniform(-30, 30, n)
    pairs = {"pow": (sign * np.exp(rng.uniform(-20, 20, n)), np.where(sign < 0, np.round(y), y)),
             "atan2": (np.exp(rng.uniform(-700, 700, n)) * np.where(rng.random(n) < 0.5, -1.0, 1.0),
                       np.exp(rng.uniform(-700, 700, n)) * np.where(rng.random(n) < 0.5, -1.0, 1.0))}
    measured = {}
    for fn, (a, b) in pairs.items():
        words = ifo._words(np.ones((1024, 1024), bool))
        out, _ = ctx.binary_op(OP[fn], a.reshape(1024, 1024), words, np.arange(1024), b.reshape(1024, 1024), words,
                               np.arange(1024))
        measured[fn] = float(ulp_distance(out.ravel(), lc.glibc(fn, a, b)).max())
    path = os.environ.get("B2P_LIBM_REPORT")
    if path:
        with open(path + ".random.json", "w") as f:
            json.dump(measured, f, indent=1)
    for fn, d in measured.items():
        assert d <= POW_ATAN2_ULPS, f"{fn}: {d} ulps from glibc"
