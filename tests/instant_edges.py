"""The instant selector (InstantManipulate) at its edges: a literal interpreter of the reference's cursor walk and a
seeded generator of cases that place samples and steps where the kernels' bounds, searches and tests turn.

interpret() restates InstantManipulateStream::manipulate (instant_manipulate.rs:473-585) statement by statement, in
Python integers, over one series whose timestamps already carry the offset (SeriesNormalize adds it before the
selector, planner.rs:886-928):
  - last_useful = last_ts + lookback - 1 when lookback > 0, else last_ts (:501-505); max_start / min_end and the
    aligned bounds with Rust's truncating division (:507-511);
  - per aligned step, the cursor runs forward; a row equal to the step stops it: that row is taken, or dropped when
    field 0 is NaN, and the step ends without looking at later rows of the same timestamp (:523-541);
  - a cursor that ran off the end steps back one row and ends the walk when that row is too old (:542-548);
  - otherwise the row in front of the cursor is taken when it is fresh (ts + lookback > step), stale when NaN
    (:550-580).
The staleness test reads field 0 only, through a Float64 downcast: stale=False models an Int64 field 0 (the downcast
fails, so nothing is stale) and timestamp(<selector>), whose value column is the projected timestamp.
It never calls the C oracle: it is the second, independent judge of the kernels.

cases() yields the seeded cases; each carries the classes it hits (classes_of, read from the data and the walk's
result, not declared), so a test can assert that every class of CLASSES ran.
"""
import functools
import math
from dataclasses import dataclass, field

import numpy as np

MS_2_40 = 1 << 40
MS_2_50 = 1 << 50
# the warps capped_grid(c, n_series, 8, 8) launches on the 132-SM H100 SXM (8 CTAs of 8 warps per SM): series s and
# s + WARPS_LAUNCHED share a warp.  A part with fewer SMs (the 114-SM H100 PCIe) strides over more series.
WARPS_LAUNCHED = 132 * 8 * 8
STRIDED = 64  # series past WARPS_LAUNCHED in the largest case
BIG_SERIES = (1 << 17) + 3    # the binary search over it runs 18 levels

# special Float64 values by their bits
SPECIAL_BITS = {
    "nan_pos_payload": 0x7FF8DEADBEEF0001,
    "nan_neg_payload": 0xFFF80000000ABCDE,
    "snan": 0x7FF0000000000BAD,
    "pos_zero": 0x0000000000000000,
    "neg_zero": 0x8000000000000000,
    "pos_inf": 0x7FF0000000000000,
    "neg_inf": 0xFFF0000000000000,
    "subnormal": 0x000000000000BEEF,
    "neg_subnormal": 0x800FFFFFFFFFFFFF,
    "pos_max": 0x7FEFFFFFFFFFFFFF,
    "neg_max": 0xFFEFFFFFFFFFFFFF,
}
QNAN_BITS = 0x7FF8000000000000

LOOKBACK_KINDS = ("0", "1", "interval-1", "interval", "interval+1", "gt_span", "2^40")
T_CLASSES = (1, 31, 32, 33, 63, 64, 65, 1000)
OFFSET_KINDS = ("0", "+1", "-1", "+interval", "-interval", "+gt_span", "-gt_span")

CLASSES = frozenset(
    [f"lookback={k}" for k in LOOKBACK_KINDS]
    + ["lookback_edge_excluded", "lookback_edge_included"]
    + ["dup_on_step_first_nan", "dup_on_step_later_nan", "dup_on_step_all_nan", "dup_on_step_none_nan",
       "dup_between_steps"]
    + [f"value_{k}" for k in ("nan_pos_payload", "nan_neg_payload", "snan", "pos_zero", "neg_zero", "pos_inf",
                              "neg_inf", "subnormal", "pos_max", "neg_max")]
    + [f"T={t}" for t in T_CLASSES]
    + ["start_off_lattice", "start_before_first", "start_after_last_useful", "end_before_first",
       "interval_gt_span", "start_eq_end", "negative_epoch", "epoch_near_+2^50", "epoch_near_-2^50"]
    + [f"offset={k}" for k in OFFSET_KINDS]
    + ["series_empty_first", "series_empty_middle", "series_empty_last", "series_n1", "series_n2",
       "series_2^17", "series_more_than_warps"])


def tdiv(a, b):
    """Rust's `/` on i64: truncates toward zero (Python's // floors)"""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b >= 0) else -q


def num_steps(start, end, interval):
    return 0 if end < start else (end - start) // interval + 1


# ---- the interpreter -----------------------------------------------------------------------------------------------
def interpret(ts, field0, start, end, interval, lookback, stale=True):
    """One series: ts (shifted timestamps, ascending, ties allowed) and field0 (its Float64 values).
    -> [(expected_ts, row)], the reference's aligned_ts and take_indices."""
    taken = []
    n = len(ts)
    if n == 0:  # :485-487
        return taken
    is_stale = (lambda i: math.isnan(field0[i])) if stale else (lambda i: False)
    first_ts = ts[0]
    last_ts = ts[n - 1]
    if lookback > 0:
        last_useful = last_ts + lookback - 1
    else:
        last_useful = last_ts
    max_start = max(first_ts, start)
    min_end = min(last_useful, end)
    aligned_start = start + tdiv(max_start - start, interval) * interval
    aligned_end = end - tdiv(end - min_end, interval) * interval
    cursor = 0
    expected_ts = aligned_start
    while expected_ts <= aligned_end:  # (aligned_start..=aligned_end).step_by(interval)
        step_done = False
        while cursor < n:
            curr = ts[cursor]
            if curr == expected_ts:
                if not is_stale(cursor):
                    taken.append((expected_ts, cursor))
                step_done = True  # continue 'next
                break
            if curr > expected_ts:
                break
            cursor += 1
        if not step_done:
            if cursor == n:
                cursor -= 1
                if ts[cursor] + lookback <= expected_ts:
                    break
            curr_ts = ts[cursor]
            if curr_ts + lookback <= expected_ts:
                pass  # continue
            elif curr_ts > expected_ts:
                if cursor >= 1:  # cursor.checked_sub(1)
                    prev_cursor = cursor - 1
                    prev_ts = ts[prev_cursor]
                    if prev_ts + lookback > expected_ts:
                        if not is_stale(prev_cursor):
                            taken.append((expected_ts, prev_cursor))
            elif is_stale(cursor):
                pass
            else:
                taken.append((expected_ts, cursor))
        expected_ts += interval
    return taken


# ---- cases ---------------------------------------------------------------------------------------------------------
@dataclass
class Case:
    name: str
    seed: int
    ts: np.ndarray       # int64 [n_rows], unshifted
    val: np.ndarray      # float64 [n_rows], field 0
    offsets: np.ndarray  # uint64 [S + 1]
    start: int
    end: int
    interval: int
    lookback: int
    offset: int
    lookback_kind: str = ""
    offset_kind: str = ""
    tags: tuple = ()     # classes the data cannot show (where the samples' lattice lies)
    classes: frozenset = field(default_factory=frozenset)
    _rows: dict = field(default_factory=dict, repr=False)

    @property
    def S(self):
        return self.offsets.size - 1

    @property
    def T(self):
        return num_steps(self.start, self.end, self.interval)

    @property
    def Tw(self):
        return (self.T + 31) // 32

    def series(self, s):
        r0, r1 = int(self.offsets[s]), int(self.offsets[s + 1])
        return r0, r1

    def rows(self, stale=True):
        """[S, T] int64: the global row each (series, step) takes, -1 for none (the interpreter's walk)"""
        if stale not in self._rows:
            out = np.full((self.S, self.T), -1, np.int64)
            ts = (self.ts + self.offset).tolist()
            v = self.val.tolist()
            for s in range(self.S):
                r0, r1 = self.series(s)
                for t, j in interpret(ts[r0:r1], v[r0:r1], self.start, self.end, self.interval, self.lookback, stale):
                    k, rem = divmod(t - self.start, self.interval)
                    assert rem == 0 and 0 <= k < self.T, (self.name, s, t)
                    out[s, k] = r0 + j
            self._rows[stale] = out
        return self._rows[stale]

    def describe(self):
        return (f"case {self.name} (seed {self.seed}; start={self.start} end={self.end} interval={self.interval} "
                f"lookback={self.lookback} offset={self.offset} S={self.S} T={self.T}; classes "
                f"{sorted(self.classes)})")


def bits(values):
    return np.asarray(values, np.float64).view(np.uint64)


def from_bits(b):
    return np.asarray(b, np.uint64).view(np.float64)


def _values(rng, n, special_share):
    """n Float64 values: normals of several magnitudes, and specials by their bits"""
    v = rng.normal(size=n) * 10.0 ** rng.integers(-3, 6, n)
    pick = rng.random(n) < special_share
    keys = list(SPECIAL_BITS.values()) + [QNAN_BITS]
    sb = np.array(keys, np.uint64)[rng.integers(0, len(keys), n)]
    return np.where(pick, from_bits(sb), v)


def _resolve_lookback(kind, interval, span):
    return {"0": 0, "1": 1, "interval-1": interval - 1, "interval": interval, "interval+1": interval + 1,
            "gt_span": span + interval + 7, "2^40": MS_2_40}[kind]


def _resolve_offset(kind, interval, span):
    return {"0": 0, "+1": 1, "-1": -1, "+interval": interval, "-interval": -interval,
            "+gt_span": span + 3 * interval + 11, "-gt_span": -(span + 3 * interval + 11)}[kind]


def _anchor_series(rng, start, interval, T, lookback, shift, n_anchor, dup_share, special_share, window):
    """One series built around eval steps: for each anchor step k a sample `d` ms before it, with d one of the
    lookback's edges (lookback, lookback - 1, 0, lookback + 1) or any value below the lookback, some of them repeated
    in runs of equal timestamps; plus samples between steps.  The anchors lie in a random window of `window` steps.
    Timestamps are stored `shift` ms early, so that the offset `shift` brings them onto the anchors.
    -> (ts unshifted, values)"""
    w = min(window or T, T)
    k0 = int(rng.integers(0, T - w + 1))
    ks = np.sort(rng.integers(k0, k0 + w, n_anchor))
    t_list = []
    for k in ks:
        te = start + int(k) * interval
        choice = rng.integers(0, 6)
        d = [lookback, lookback - 1, 0, lookback + 1, int(rng.integers(0, max(lookback, 1))),
             int(rng.integers(0, interval))][choice]
        t_list.append(te - max(d, 0))
    t_list += [start + int(rng.integers((k0 - 2) * interval, (k0 + w + 1) * interval + 1))
               for _ in range(n_anchor // 3)]
    t_list.sort()
    ts, vals = [], []
    for t in t_list:
        reps = 1 if rng.random() >= dup_share else int(rng.integers(2, 5))
        v = _values(rng, reps, special_share)
        if reps > 1:  # the NaN pattern of the run: first row, a later row, all rows or none
            pattern = rng.integers(0, 4)
            if pattern == 0:
                v[0] = np.nan
            elif pattern == 1:
                v[int(rng.integers(1, reps))] = np.nan
            elif pattern == 2:
                v[:] = np.nan
            else:
                v[np.isnan(v)] = 1.5
        ts += [t - shift] * reps
        vals += v.tolist()
    return np.array(ts, np.int64), np.array(vals, np.float64)


def _pack(series):
    sizes = [s[0].size for s in series]
    offsets = np.zeros(len(series) + 1, np.uint64)
    offsets[1:] = np.cumsum(sizes)
    ts = np.concatenate([s[0] for s in series]) if series else np.zeros(0, np.int64)
    val = np.concatenate([s[1] for s in series]) if series else np.zeros(0, np.float64)
    return ts.astype(np.int64), val.astype(np.float64), offsets


def _empty():
    return np.zeros(0, np.int64), np.zeros(0, np.float64)


def anchor_case(name, seed, T, lookback_kind, offset_kind="0", start=1_000_000, interval=1000, S=40, n_anchor=12,
                dup_share=0.15, special_share=0.3, empties=(0, "mid", -1), short=True, extra=(), window=None):
    """S series of anchor samples around the grid [start, start + (T-1) interval]; the even series are stored
    `offset` early, so that the offset brings them onto their anchors, the odd ones are not (an offset longer than
    the span moves them wholly off the grid).  Empty series at the positions in `empties` ("mid": S // 2), a 1-sample
    and a 2-sample series when `short`; `extra`: more (ts, val) series, as stored."""
    rng = np.random.default_rng(seed)
    span = (T + 2) * interval
    lookback = _resolve_lookback(lookback_kind, interval, span)
    offset = _resolve_offset(offset_kind, interval, span)
    series = []
    for s in range(S):
        series.append(_anchor_series(rng, start, interval, T, lookback, 0 if s % 2 else offset, n_anchor, dup_share,
                                     special_share, window))
    if short:
        series[1] = (series[1][0][:1], series[1][1][:1]) if series[1][0].size else series[1]
        series[2] = (series[2][0][:2], series[2][1][:2]) if series[2][0].size >= 2 else series[2]
    for pos in empties:
        series[S // 2 if pos == "mid" else pos] = _empty()
    series += list(extra)
    ts, val, offsets = _pack(series)
    return Case(name, seed, ts, val, offsets, start, start + (T - 1) * interval, interval, lookback, offset,
                lookback_kind, offset_kind)


def regular_case(name, seed, T, lookback, start, interval, cadence, phase, n, S=12, offset=0, tags=()):
    """S regular series (sample i at t0 + i cadence, t0 = start + phase + s), values with specials; the grid
    [start, start + (T-1) interval] over them"""
    rng = np.random.default_rng(seed)
    series = []
    for s in range(S):
        t0 = start + phase + s * 3
        series.append((np.arange(n, dtype=np.int64) * cadence + t0 - offset, _values(rng, n, 0.1)))
    ts, val, offsets = _pack(series)
    return Case(name, seed, ts, val, offsets, start, start + (T - 1) * interval, interval, lookback, offset,
                tags=tags)


@functools.lru_cache(maxsize=None)
def cases():
    """the seeded cases, classes attached (built once per process)"""
    out = []
    seed = 1000
    # the lookback boundary for every lookback kind, across the T classes
    for i, kind in enumerate(LOOKBACK_KINDS):
        for T in (T_CLASSES[i % 7], T_CLASSES[(i + 3) % 7]):
            seed += 1
            out.append(anchor_case(f"lookback_{kind}_T{T}", seed, T, kind, interval=1000 + 7 * i))
    # offsets, at a lookback that straddles a step
    for i, kind in enumerate(OFFSET_KINDS):
        seed += 1
        out.append(anchor_case(f"offset_{kind}", seed, 65 if i % 2 else 33, "interval+1", offset_kind=kind))
    # T = 1000 with the lookback edges, and the grid's epochs: negative, near +2^50 and near -2^50
    seed += 1
    out.append(anchor_case("T1000_interval", seed, 1000, "interval", S=20, n_anchor=300))
    for name, start in (("negative_epoch", -7_000_003), ("epoch_near_+2^50", MS_2_50 - 5_000_000 + 13),
                        ("epoch_near_-2^50", -MS_2_50 + 17)):
        for kind in ("interval-1", "2^40"):
            seed += 1
            out.append(anchor_case(f"{name}_{kind}", seed, 64, kind, offset_kind="-interval", start=start,
                                   interval=997))
    # start off the samples' lattice, before the first sample; start == end; interval longer than the span
    seed += 1
    out.append(regular_case("start_off_lattice", seed, 63, 30_000, 1_000_000, 15_000, 15_000, 7_001, 70,
                            tags=("start_off_lattice",)))
    seed += 1
    out.append(regular_case("start_before_first", seed, 65, 45_000, 1_000_000, 10_000, 10_000, 123_457, 40))
    for lb in (0, 1, 300_000):
        seed += 1
        out.append(regular_case(f"start_eq_end_lookback{lb}", seed, 1, lb, 1_000_000 + 15_000 * 4, 1000, 15_000,
                                -15_000 * 3 if lb else 0, 9))
    seed += 1
    out.append(regular_case("interval_gt_span", seed, 3, 500_000, 1_000_000, 1_000_000, 1000, 500_123, 30))
    # series wholly after the grid (no step: end before the first sample) and wholly before it (start after
    # last_useful), beside ordinary ones
    seed += 1
    rng = np.random.default_rng(seed)
    late = (np.arange(5, dtype=np.int64) * 1000 + 2_000_000, _values(rng, 5, 0.2))
    early = (np.arange(5, dtype=np.int64) * 1000 + 100_000, _values(rng, 5, 0.2))
    out.append(anchor_case("series_outside_the_grid", seed, 32, "interval", extra=(late, early, _empty())))
    # one long series (the binary search over 2^17 rows), beside short ones
    seed += 1
    rng = np.random.default_rng(seed)
    big_ts = 1_000_000 + np.cumsum(rng.integers(0, 4, BIG_SERIES)).astype(np.int64)  # zero steps: equal timestamps
    big = (big_ts, _values(rng, BIG_SERIES, 0.05))
    for kind in ("0", "interval-1", "interval+1"):
        seed += 1
        out.append(anchor_case(f"series_2^17_lookback_{kind}", seed, 1000, kind, interval=331, S=6,
                               extra=(big,)))
    # more series than the kernels launch warps
    seed += 1
    # the warps of series 0 .. STRIDED - 1 take a second series past WARPS_LAUNCHED, with anchors in another window:
    # non-empty after non-empty, after an empty one (series 3) and an empty one after a non-empty one (series 5)
    out.append(anchor_case("series_more_than_warps", seed, 1000, "interval", S=WARPS_LAUNCHED + STRIDED, n_anchor=6,
                           empties=(3, "mid", WARPS_LAUNCHED + 5), window=24))
    for c in out:
        c.classes = classes_of(c)
    return out


# ---- classes -------------------------------------------------------------------------------------------------------
def classes_of(c):
    """the classes of CLASSES case c hits, read from its data, its grid and the interpreter's walk"""
    got = set(c.tags)
    if c.lookback_kind:
        got.add(f"lookback={c.lookback_kind}")
    if c.offset_kind:
        got.add(f"offset={c.offset_kind}")
    T, S = c.T, c.S
    if T in T_CLASSES:
        got.add(f"T={T}")
    if c.start == c.end:
        got.add("start_eq_end")
    sts = c.ts + c.offset
    sizes = np.diff(c.offsets.astype(np.int64))
    nonempty = np.flatnonzero(sizes > 0)
    if S and sizes[0] == 0:
        got.add("series_empty_first")
    if S and sizes[-1] == 0:
        got.add("series_empty_last")
    if S > 2 and (sizes[1:-1] == 0).any():
        got.add("series_empty_middle")
    if (sizes == 1).any():
        got.add("series_n1")
    if (sizes == 2).any():
        got.add("series_n2")
    if (sizes >= 1 << 17).any():
        got.add("series_2^17")
    if (sizes[WARPS_LAUNCHED:] > 0).any():
        got.add("series_more_than_warps")
    if sts.size:
        lo, hi = int(sts.min()), int(sts.max())
        if c.interval > hi - lo:
            got.add("interval_gt_span")
        if c.start < 0 and lo < 0:
            got.add("negative_epoch")
        if c.start > MS_2_50 - (1 << 40) and lo > MS_2_50 - (1 << 40):
            got.add("epoch_near_+2^50")
        if c.start < -MS_2_50 + (1 << 40) and hi < -MS_2_50 + (1 << 40):
            got.add("epoch_near_-2^50")
    for s in nonempty:
        r0, r1 = c.series(s)
        first, last = int(sts[r0]), int(sts[r1 - 1])
        last_useful = last + c.lookback - 1 if c.lookback > 0 else last
        if c.start < first <= c.end:
            got.add("start_before_first")
        if last_useful < c.start:
            got.add("start_after_last_useful")
        if c.end < first:
            got.add("end_before_first")
    # the walk: lookback edges, runs of equal timestamps, the values of taken rows
    rows = c.rows(stale=False)
    steps = c.start + np.arange(T, dtype=np.int64) * c.interval
    for s in nonempty:
        r0, r1 = c.series(s)
        t = sts[r0:r1]
        last_le = np.searchsorted(t, steps, side="right") - 1  # the row in front of each step
        has = last_le >= 0
        if not has.any():
            continue
        age = np.where(has, steps - t[np.maximum(last_le, 0)], -1)
        if c.lookback > 0 and (has & (age == c.lookback)).any():
            got.add("lookback_edge_excluded")
        if c.lookback > 0 and (has & (age == c.lookback - 1)).any():
            got.add("lookback_edge_included")
        # runs of equal timestamps
        same = np.flatnonzero(t[1:] == t[:-1])
        for i in same:
            if i > 0 and t[i - 1] == t[i]:
                continue  # not the start of its run
            tt = int(t[i])
            j = i + 1
            while j + 1 < t.size and t[j + 1] == tt:
                j += 1
            run = c.val[r0 + i:r0 + j + 1]
            on_step = c.start <= tt <= c.end and (tt - c.start) % c.interval == 0
            if on_step:
                nan = np.isnan(run)
                got.add("dup_on_step_all_nan" if nan.all() else "dup_on_step_first_nan" if nan[0]
                        else "dup_on_step_later_nan" if nan.any() else "dup_on_step_none_nan")
            elif (rows[s] == r0 + j).any():
                got.add("dup_between_steps")
    taken = rows[rows >= 0]
    tb = set(bits(c.val[taken]).tolist())
    for k, b in SPECIAL_BITS.items():
        if b in tb:
            got.add("value_" + {"neg_subnormal": "subnormal"}.get(k, k))
    return frozenset(got & CLASSES)


# ---- expected grids ------------------------------------------------------------------------------------------------
def valid_words(ok):
    """[S, T] bool -> [S, Tw] uint32 validity words, bits past T zero"""
    S, T = ok.shape
    pad = np.pad(ok, ((0, 0), (0, (-T) % 32)))
    return np.packbits(pad, axis=1, bitorder="little").view(np.uint32).reshape(S, (T + 31) // 32)


def unpack_words(words, T):
    """[S, Tw] uint32 validity words -> [S, T] bool"""
    w = np.ascontiguousarray(words, np.uint32)
    return np.unpackbits(w.view(np.uint8), axis=1, bitorder="little")[:, :T].astype(bool)


def gather(col, rows):
    """[S, T] cells of an 8-byte column at the taken rows (as uint64 bits), 0 where no row is taken"""
    b = np.ascontiguousarray(col).view(np.uint64)
    return np.where(rows >= 0, b[np.maximum(rows, 0)] if b.size else np.uint64(0), np.uint64(0))


def expected_values(c, cols, stale=True):
    """value mode over the columns `cols` -> ([F, S, T] uint64 bits, [S, Tw] uint32 words)"""
    rows = c.rows(stale)
    return np.stack([gather(col, rows) for col in cols]), valid_words(rows >= 0)


def expected_timestamps(c):
    """timestamp(<selector>): (double)(ts + offset) / 1000.0 of the row taken without the staleness test"""
    rows = c.rows(stale=False)
    out = np.zeros(rows.shape, np.float64)
    ok = rows >= 0
    out[ok] = (c.ts[rows[ok]] + c.offset).astype(np.float64) / 1000.0
    return out.view(np.uint64), valid_words(ok)


def extra_fields(c, F):
    """F - 1 Float64 columns beside field 0: random 64-bit patterns (NaNs with payloads, infinities, subnormals and
    signed zeros among them), a NaN in every fourth row"""
    rng = np.random.default_rng(c.seed + 77)
    cols = []
    for f in range(1, F):
        b = rng.integers(0, 1 << 64, c.ts.size, dtype=np.uint64, endpoint=False)
        b[f % 4::4] = np.uint64(0xFFF0000000000000 | (f * 0x1111))  # -NaN with a payload
        cols.append(b.view(np.float64))
    return cols


def first_difference(got_bits, exp_bits, got_words, exp_words, T):
    """'' when equal, else where the first cell differs: (series, step) and both sides"""
    gw, ew = np.asarray(got_words, np.uint32), np.asarray(exp_words, np.uint32)
    if gw.shape != ew.shape:
        return f"validity shape {gw.shape} != {ew.shape}"
    bad = np.argwhere(gw != ew)
    if bad.size:
        s, w = bad[0]
        diff = int(gw[s, w] ^ ew[s, w])
        k = int(w) * 32 + (diff & -diff).bit_length() - 1
        return (f"validity differs first at (series {s}, step {k}{' past T' if k >= T else ''}): got "
                f"{bool(gw[s, w] >> (k % 32) & 1)}, expected {bool(ew[s, w] >> (k % 32) & 1)}")
    g, e = np.asarray(got_bits, np.uint64), np.asarray(exp_bits, np.uint64)
    bad = np.argwhere(g != e)
    if bad.size:
        idx = tuple(bad[0])
        return (f"value differs first at (series {idx[-2]}, step {idx[-1]})"
                f"{' field %d' % idx[0] if g.ndim == 3 else ''}: got 0x{int(g[idx]):016x}, expected "
                f"0x{int(e[idx]):016x}")
    return ""
