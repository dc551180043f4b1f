"""A plain reference for `sum by` over a per-series grid, and a checker of a device's group sums against it.

The input is a per-series grid (values [S, T] and validity words [S, Tw]), in the suite always the oracle's rescan grid
(orc.range_query(..., rescan=True)), which every range tier reproduces bit for bit, and one group id per series.  For
every cell (g, k) the reference holds

  cnt    the number of valid members;
  seq    orc.group_aggregate("sum"): the members added in series-id order, starting from +0.0 (DataFusion's `+=`, and
         the order of the fused first tier, whose CSR members are sorted by series id);
  exact  math.fsum of the members (correctly rounded);
  mag    the sum of their magnitudes;
  the non-finite class: NaN when a member is NaN or both infinities occur, else +inf / -inf when one occurs.

Two modes compare a device grid (sum, cnt) with it:

  bits   counts equal, and every sum has seq's bits (+0.0 and -0.0 differ); a NaN only has to be a NaN;
  bound  counts equal, and |got - exact| <= gamma(n - 1) * mag, with gamma(m) = m u / (1 - m u), u = 2^-53: the error
         bound of recursive summation in any order (Higham, Accuracy and Stability of Numerical Algorithms, 4.2).
         Non-finite cells must match their class.  Whether a partial sum overflows depends on the order: every partial
         sum lies within [-(1 + gamma) neg, (1 + gamma) pos], pos / neg the sums of the positive / negative members, so
         a cell may also be +inf where that upper end reaches f64::MAX, and -inf where the lower end does (for members
         of one sign: where exact + bound reaches it).

Cells whose members could overflow a partial sum of fsum are evaluated scaled by a power of two; the scaling loses at
most the last bit of subnormal members, a slack of n * 2^-1074 that is added to their bound only.
"""
import math
from dataclasses import dataclass

import numpy as np

from oracle import oracle as orc

U = 2.0 ** -53
F64_MAX = float(np.finfo(np.float64).max)
TINY = 2.0 ** -1074


def gamma(m):
    """gamma(m) = m u / (1 - m u) for an array or a scalar of addend counts minus one (m >= 0)"""
    m = np.asarray(m, np.float64)
    return m * U / (1.0 - m * U)


@dataclass
class Reference:
    groups: np.ndarray   # the group ids the rows below describe
    cnt: np.ndarray      # [len(groups), T] u32
    seq: np.ndarray      # [len(groups), T] f64
    exact: np.ndarray    # [len(groups), T] f64, scaled by `scale`
    mag: np.ndarray      # [len(groups), T] f64, scaled by `scale`
    pos: np.ndarray      # [len(groups), T] f64: the sum of the positive members, scaled by `scale`
    neg: np.ndarray      # [len(groups), T] f64: minus the sum of the negative members, scaled by `scale`
    scale: np.ndarray    # [len(groups), T] f64: 1.0, or the power of two exact / mag were taken at
    cls: np.ndarray      # [len(groups), T] f64: 0.0 finite, NaN, +inf or -inf


def _cell(xs):
    """-> (exact, mag, pos, neg, scale, cls) of the valid members xs of one cell"""
    nan = bool(np.isnan(xs).any())
    pinf, ninf = bool((xs == np.inf).any()), bool((xs == -np.inf).any())
    if nan or (pinf and ninf):
        return 0.0, 0.0, 0.0, 0.0, 1.0, math.nan
    if pinf or ninf:
        return 0.0, 0.0, 0.0, 0.0, 1.0, (math.inf if pinf else -math.inf)
    vals = xs.tolist()
    s = 1.0
    if max(abs(x) for x in vals) * len(vals) >= F64_MAX / 2:
        s = 2.0 ** -(math.ceil(math.log2(len(vals))) + 2)
    v = [x * s for x in vals]
    return (math.fsum(v), math.fsum(abs(x) for x in v), math.fsum(x for x in v if x > 0),
            -math.fsum(x for x in v if x < 0), s, 0.0)


def reference(out, valid_words, gid, n_groups, groups=None):
    """The reference of sum by over the grid (out [S, T], valid_words [S, Tw]) with group ids gid (a series whose id is
    >= n_groups belongs to no group); `groups`: the group ids to describe (default: all)."""
    out = np.ascontiguousarray(out, np.float64)
    valid_words = np.ascontiguousarray(valid_words, np.uint32)
    gid = np.ascontiguousarray(gid, np.uint32)
    S, T = out.shape
    groups = np.arange(n_groups) if groups is None else np.asarray(groups)
    seq_all, cnt_all = orc.group_aggregate("sum", out, valid_words, gid, n_groups)
    vb = orc.valid_to_bool(valid_words, T) if S else np.zeros((0, T), bool)
    G = groups.size
    exact, mag, pos, neg = np.zeros((G, T)), np.zeros((G, T)), np.zeros((G, T)), np.zeros((G, T))
    scale, cls = np.ones((G, T)), np.zeros((G, T))
    for i, g in enumerate(groups):
        members = np.flatnonzero(gid == g)
        if not members.size:
            continue
        rows, ok = out[members], vb[members]
        for k in np.flatnonzero(ok.any(0)):
            exact[i, k], mag[i, k], pos[i, k], neg[i, k], scale[i, k], cls[i, k] = _cell(rows[ok[:, k], k])
    return Reference(groups, cnt_all[groups], seq_all[groups], exact, mag, pos, neg, scale, cls)


def _where(mask):
    return np.argwhere(mask)[:4].tolist()


def check(ref, got, cnt, mode, what="", bound_factor=1.0):
    """Compares the device's sums / counts of ref.groups (arrays [len(groups), T], or the whole [n_groups, T] grid when
    ref describes every group) with the reference.  mode: "bits" or "bound".  bound_factor scales the bound (2 for two
    device results that each hold it).  Raises AssertionError naming the first offending cells."""
    got = np.asarray(got, np.float64)
    cnt = np.asarray(cnt).view(np.uint32) if np.asarray(cnt).dtype == np.int32 else np.asarray(cnt, np.uint32)
    if got.shape != ref.seq.shape:
        got, cnt = got[ref.groups], cnt[ref.groups]
    assert cnt.shape == ref.cnt.shape, f"{what}: shape {cnt.shape} vs {ref.cnt.shape}"
    bad = cnt != ref.cnt
    assert not bad.any(), f"{what}: {int(bad.sum())} counts differ at {_where(bad)}: " \
                          f"{cnt[bad][:4].tolist()} vs {ref.cnt[bad][:4].tolist()}"
    if mode == "bits":
        gb, eb = got.view(np.uint64), ref.seq.view(np.uint64)
        bad = np.where(np.isnan(ref.seq), ~np.isnan(got), gb != eb)
        assert not bad.any(), f"{what}: {int(bad.sum())} sums differ from the series-order sum at {_where(bad)}: " \
                              f"{got[bad][:4].tolist()} vs {ref.seq[bad][:4].tolist()}"
        return
    assert mode == "bound", mode
    empty = ref.cnt == 0
    bad = empty & (got != 0.0)
    assert not bad.any(), f"{what}: empty cells hold {got[bad][:4].tolist()} at {_where(bad)}"
    nonfin = ~empty & (ref.cls != 0.0)
    bad = nonfin & ~(np.isnan(ref.cls) & np.isnan(got)) & ~(got == ref.cls)
    assert not bad.any(), f"{what}: {int(bad.sum())} non-finite sums of the wrong class at {_where(bad)}: " \
                          f"{got[bad][:4].tolist()} vs {ref.cls[bad][:4].tolist()}"
    fin = ~empty & (ref.cls == 0.0)
    n = ref.cnt.astype(np.float64)
    bound = bound_factor * gamma(np.maximum(n - 1.0, 0.0)) * ref.mag + np.where(ref.scale < 1.0, n * TINY, 0.0)
    with np.errstate(over="ignore", invalid="ignore"):
        err = np.abs(got * ref.scale - ref.exact)
        ok = err <= bound
        # an order whose partial sum overflows: +inf where the largest partial sum can reach f64::MAX, -inf where the
        # smallest can
        g1 = 1.0 + gamma(n)
        ok |= (got == np.inf) & (ref.pos * g1 >= F64_MAX * ref.scale)
        ok |= (got == -np.inf) & (ref.neg * g1 >= F64_MAX * ref.scale)
    bad = fin & ~ok
    if bad.any():
        i = tuple(np.argwhere(bad)[0])
        with np.errstate(over="ignore"):
            raise AssertionError(f"{what}: {int(bad.sum())} sums outside the summation error bound at {_where(bad)}; "
                                 f"first: got {got[i]!r}, exact {ref.exact[i] / ref.scale[i]!r}, "
                                 f"bound {bound[i] / ref.scale[i]!r}, {int(ref.cnt[i])} members")


def check_pair(a, b, ref, what=""):
    """Two device results of the same sums: equal counts, and sums within 2 gamma(n - 1) mag of each other (each holds
    the bound against exact) and of the same non-finite class."""
    check(ref, a[0], a[1], "bound", what + " (first)")
    check(ref, b[0], b[1], "bound", what + " (second)")
    x, y = np.asarray(a[0], np.float64), np.asarray(b[0], np.float64)
    if x.shape != ref.seq.shape:
        x, y = x[ref.groups], y[ref.groups]
    fin = (ref.cnt > 0) & (ref.cls == 0.0) & np.isfinite(x) & np.isfinite(y)
    bound = 2.0 * gamma(np.maximum(ref.cnt.astype(np.float64) - 1.0, 0.0)) * ref.mag
    with np.errstate(over="ignore", invalid="ignore"):
        bad = fin & ~(np.abs(x * ref.scale - y * ref.scale) <= bound + np.where(ref.scale < 1.0, 2 * ref.cnt * TINY, 0))
    assert not bad.any(), f"{what}: the two routes differ by more than 2 gamma(n-1) mag at {_where(bad)}"
