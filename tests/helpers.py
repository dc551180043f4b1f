"""Shared helpers for the parity tests (golden loading, special-value parsing)."""
import json
import math
import os

import numpy as np

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def fnum(x):
    if x is None:
        return None
    if isinstance(x, str):
        return {"nan": math.nan, "inf": math.inf, "-inf": -math.inf}[x]
    return float(x)


def farr(xs):
    return np.array([fnum(x) for x in xs], dtype=np.float64)


def load_unit():
    with open(os.path.join(GOLDEN_DIR, "reference_unit_vectors.json")) as f:
        return json.load(f)


def load_sqlness():
    with open(os.path.join(GOLDEN_DIR, "reference_sqlness_vectors.json")) as f:
        return json.load(f)


def udf_case_inputs(case, unit):
    if "fixture" in case:
        fx = unit["fixtures"][case["fixture"]]
        ts, val, ranges = fx["ts"], fx["val"], fx["ranges"]
    else:
        ts, val, ranges = case["ts"], case["val"], case["ranges"]
    return np.array(ts, np.int64), farr(val), np.array(ranges, np.uint32).reshape(-1, 2)


def check_expected(out, valid, expected, tol, what=""):
    assert len(out) == len(expected), what
    for i, e in enumerate(expected):
        if e is None:
            assert not valid[i], f"{what}: window {i} expected null, got {out[i]}"
            continue
        e = fnum(e)
        assert valid[i], f"{what}: window {i} expected {e}, got null"
        if math.isnan(e):
            assert math.isnan(out[i]), f"{what}: window {i}"
        elif tol == 0 or math.isinf(e):
            assert out[i] == e, f"{what}: window {i}: {out[i]!r} != {e!r}"
        else:
            assert abs(out[i] - e) < tol, f"{what}: window {i}: {out[i]!r} vs {e!r}"


def pack_series(series_dict):
    """{name: {ts, val}} -> (names, ts, val, sid, offsets) in dict order (series sorted rows)."""
    names, ts, val, sid, offsets = [], [], [], [], [0]
    for i, (name, d) in enumerate(series_dict.items()):
        names.append(name)
        ts.extend(d["ts"])
        val.extend(fnum(v) for v in d["val"])
        sid.extend([i] * len(d["ts"]))
        offsets.append(len(ts))
    return (names, np.array(ts, np.int64), np.array(val, np.float64), np.array(sid, np.uint32),
            np.array(offsets, np.uint64))


# Members whose order under f64::total_cmp differs from IEEE min / max: NaN of both signs (one with a payload), the two
# zeros, and ordinary values around them.
SPECIALS = np.array([0x7FF8000000000000, 0xFFF8000000000000, 0x7FF8000000000123, 0x8000000000000000, 0x0000000000000000,
                     0x4008000000000000, 0xC008000000000000, 0x7FF0000000000000, 0xFFF0000000000000],
                    dtype=np.uint64).view(np.float64)   # +NaN, -NaN, +NaN payload, -0.0, +0.0, 3.0, -3.0, +inf, -inf


def total_order_case():
    """One group per ordered pair of SPECIALS, its first member in the first half of the series and its second in the
    second half (one half per rank or shard, so every placement order occurs), at T = 3 steps: both members valid at
    step 0, only the first-half member at step 1, none at step 2.
    -> (vals [2G x T], valid words [2G x 1], gid [2G], G); rows 0..G-1 are the first half, rows G..2G-1 the second."""
    pairs = [(a, b) for a in range(SPECIALS.size) for b in range(SPECIALS.size)]
    G, T = len(pairs), 3
    vals = np.zeros((2 * G, T))
    valid = np.zeros((2 * G, 1), np.uint32)
    for g, (a, b) in enumerate(pairs):
        vals[g, :] = SPECIALS[a]
        vals[G + g, :] = SPECIALS[b]
        valid[g, 0] = 0b011
        valid[G + g, 0] = 0b001
    gid = np.concatenate([np.arange(G), np.arange(G)]).astype(np.uint32)
    return vals, valid, gid, G


def promql_series(spec):
    """Prometheus test-series notation 'a+bxN a-bxN ...' (double_exponential_smoothing.rs:466-494)."""
    out = []
    for part in spec.split(" "):
        head, n = part.split("x")
        n = int(n)
        if "+" in head:
            a, b = head.split("+")
            a, b = int(a), int(b)
            out.extend(float(x) for x in range(a, b * n + a + 1, b))
        else:
            a, b = head.split("-")
            a, b = int(a), int(b)
            lo = -b * n + a
            seq = list(range(lo, a + 1))[::-1][::b]
            out.extend(float(x) for x in seq)
    return np.array(out, np.float64)
