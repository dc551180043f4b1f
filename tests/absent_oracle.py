"""CPU restatement of PromQL absent(): AbsentStream's cursor walk (GreptimeDB src/promql/src/extension_plan/absent.rs,
process_input_batch / process_remaining_absent_timestamps) over the child's timestamps, and the same result as "no
valid cell at step k" over a dense [rows x T] grid, which is what K15 computes.  Fake labels as Absent::try_new keeps
them: collected into a map (the last value of a name wins) and sorted by name."""
import re

import numpy as np


def absent_stream(start, end, step, present):
    """The timestamps AbsentStream emits for sorted input timestamps `present` (one batch; its split into batches of the
    session's batch size does not change them)."""
    out = []
    cursor = start
    for ts in present:
        # generate absent timestamps up to this input timestamp
        while cursor < ts and cursor <= end:
            out.append(cursor)
            cursor += step
        # skip the input timestamp if it matches the cursor
        if cursor == ts:
            cursor += step
    while cursor <= end:
        out.append(cursor)
        cursor += step
    return out


def grid(start, end, step):
    """The eval timestamps start + k * step <= end (none when start > end)."""
    return list(range(start, end + 1, step)) if start <= end else []


def absent_steps(start, end, step, ok):
    """The grid steps at which no row of ok [rows x T] (bool) has a valid cell (every step when there is no row)."""
    ts = grid(start, end, step)
    ok = np.asarray(ok, bool)
    assert ok.ndim == 2 and ok.shape[1] == len(ts)
    return [t for t, any_row in zip(ts, ok.any(axis=0)) if not any_row]


def absent_words(ok, T):
    """K15's output over ok [rows x T]: (out [T] f64, words [Tw] u32)."""
    ok = np.asarray(ok, bool)
    assert ok.ndim == 2 and ok.shape[1] == T
    gone = ~ok.any(axis=0)
    Tw = (T + 31) // 32
    padded = np.zeros(Tw * 32, np.uint8)
    padded[:T] = gone
    words = np.packbits(padded, bitorder="little").view(np.uint32).copy()
    return np.where(gone, 1.0, 0.0), words


def fake_labels(matchers):
    """The equality matchers of a selector as Absent::try_new keeps them: [(name, value)], one per name (the last one
    given), ordered by name (bytes)."""
    kept = {}
    for name, op, value in matchers:
        if op == "=":
            kept[name] = value
    return sorted(kept.items(), key=lambda nv: nv[0].encode())


def matches(labels, matchers):
    """A series' labels against PromQL label matchers (a missing label reads as ""; regexes are anchored)."""
    for name, op, value in matchers:
        v = labels.get(name, "")
        if op == "=" and v != value or op == "!=" and v == value:
            return False
        if op == "=~" and not re.fullmatch(value, v) or op == "!~" and re.fullmatch(value, v):
            return False
    return True


def present_steps(series, start, end, step, lookback):
    """The grid steps at which an instant selector over `series` ([{"ts": [..]}]) has a sample: one at or before the
    step, at most `lookback` before it."""
    out = []
    for k in grid(start, end, step):
        if any(any(t <= k and k - t <= lookback for t in s["ts"]) for s in series):
            out.append(k)
    return out
