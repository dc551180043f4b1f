"""A plain restatement of what the reference computes over an Int64 (BIGINT) value column, for the tests of the Int64
device calls and plan nodes: the instant selector over a table given as rows, sort, topk, count_values and the
aggregates, with the type of every printed column.  Int64 arithmetic wraps at 64 bits (DataFusion's Int64 Sum
accumulator); an Int64 is never NaN, whatever its bits; a Float64 result prints with a decimal point."""
import numpy as np

INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
LOOKBACK = 300_000


def wrap(x):
    """x as two's-complement Int64"""
    return (int(x) + (1 << 63)) % (1 << 64) - (1 << 63)


def fold(op, values):
    """one (group, step) of the by-label aggregate over Int64 values in member order -> (value, "Int64" | "Float64")"""
    if op == "sum":
        acc = 0
        for v in values:
            acc = wrap(acc + int(v))
        return acc, "Int64"
    if op == "min":
        return min(int(v) for v in values), "Int64"
    if op == "max":
        return max(int(v) for v in values), "Int64"
    if op == "count":
        return float(len(values)), "Float64"
    xs = [float(int(v)) for v in values]
    if op == "avg":
        s = 0.0
        for x in xs:
            s += x
        return s / len(xs), "Float64"
    mean = m2 = 0.0
    for n, x in enumerate(xs, 1):  # Welford, as the Float64 path
        d1 = x - mean
        mean = d1 / float(n) + mean
        m2 += d1 * (x - mean)
    return (m2 / len(xs) if op == "stdvar" else float(np.sqrt(m2 / len(xs)))), "Float64"


def group_aggregate(op, vals, ok, gid, n_groups):
    """[G x T] results and counts of fold() over an int64 grid"""
    R, T = vals.shape
    out, cnt = [[0] * T for _ in range(n_groups)], np.zeros((n_groups, T), np.uint32)
    for g in range(n_groups):
        for k in range(T):
            xs = [vals[r, k] for r in range(R) if gid[r] == g and ok[r, k]]
            cnt[g, k] = len(xs)
            if xs:
                out[g][k] = fold(op, xs)[0]
    return out, cnt


def value_order(vals, ok, desc):
    """sort / sort_desc over an int64 grid: valid cells r * T + k by signed value, ties in row-major order"""
    R, T = vals.shape
    cells = [r * T + k for r in range(R) for k in range(T) if ok[r, k]]
    flat = vals.reshape(-1)
    return sorted(cells, key=lambda c: -int(flat[c]) if desc else int(flat[c]))  # (stable)


def topk_keep(bottom, kk, vals, ok, gid, n_groups, tie):
    """the kept cells of topk / bottomk(kk) over an int64 grid: per (group, step) the best by (value, tie)"""
    R, T = vals.shape
    keep = np.zeros((R, T), bool)
    for g in range(n_groups):
        for k in range(T):
            rows = [r for r in range(R) if gid[r] == g and ok[r, k]]
            rows.sort(key=lambda r: (int(vals[r, k]), int(tie[r])), reverse=not bottom)
            for r in rows[:kk]:
                keep[r, k] = True
    return keep


def count_values(vals, ok, gid, n_groups):
    """per (group, step): the distinct Int64 values ascending with their multiplicities"""
    R, T = vals.shape
    out = {}
    for g in range(n_groups):
        for k in range(T):
            xs = sorted(int(vals[r, k]) for r in range(R) if gid[r] == g and ok[r, k])
            out[g, k] = [(v, xs.count(v)) for v in sorted(set(xs))]
    return out


# ---- the golden tables --------------------------------------------------------------------------------------------
def printed(v, typ):
    """a cell as the reference's table prints it: an Int64 without a decimal point, a Float64 with one"""
    if typ == "Int64":
        return str(int(v))
    return "NaN" if np.isnan(v) else repr(float(v))


def instant(rows, t, pred=lambda row: True):
    """InstantManipulate at eval time t over (ts, host, idc, val) rows: each series' latest row within the lookback"""
    best = {}
    for ts, host, idc, val in rows:
        if pred((ts, host, idc, val)) and t - LOOKBACK < ts <= t:
            key = (host, idc)
            if key not in best or best[key][0] <= ts:
                best[key] = (ts, val)
    return {k: v[1] for k, v in sorted(best.items())}


STEPS = [0, 5000, 10000, 15000]


def stamp(t):
    return "1970-01-01T00:00:%02d" % (t // 1000)


def evaluate(case, table):
    """the printed rows of one golden case, restated from its table"""
    rows = table["rows"]
    q = case["query"]
    if q.startswith("sort") and "sum(" not in q:
        desc = q.startswith("sort_desc")
        cells = [(t, k, v) for t in STEPS for k, v in instant(rows, t, lambda r: r[1] == "host1").items()]
        cells.sort(key=lambda c: -c[2] if desc else c[2])
        return [[stamp(t), printed(v, "Int64"), k[0], k[1]] for t, k, v in cells]
    if q.startswith("sort"):
        desc = q.startswith("sort_desc")
        cells = []
        for t in STEPS:
            sel = instant(rows, t, lambda r: r[1] == "host2")
            by = {}
            for (host, idc), v in sel.items():
                by[idc] = wrap(by.get(idc, 0) + v)
            cells += [(t, idc, v) for idc, v in sorted(by.items())]
        cells.sort(key=lambda c: -c[2] if desc else c[2])
        return [["timestamp", printed(v, "Int64"), idc] for t, idc, v in cells]
    if q.startswith("count_values"):
        by_idc = q.endswith("by (idc)")
        out = []
        groups = ["idc1", "idc2"] if by_idc else [None]
        for g in groups:
            for t in STEPS:
                xs = [v for (h, i), v in instant(rows, t).items() if g is None or i == g]
                for v in sorted(set(xs)):
                    out.append([printed(xs.count(v), "Int64")] + ([g] if g else []) + [stamp(t), printed(v, "Int64")])
        return out
    if q.startswith("quantile"):
        def quantile(xs, phi=0.5):
            s = sorted(float(x) for x in xs)
            rank = phi * (len(s) - 1)
            lo = int(np.floor(rank))
            hi = min(len(s) - 1, lo + 1)
            w = rank - lo
            return s[lo] * (1 - w) + s[hi] * w
        out = []
        if q == "quantile(0.5, test)":
            for t in STEPS:
                out.append([stamp(t), printed(quantile(instant(rows, t).values()), "Float64")])
        elif q == "quantile(0.5, test) by (idc)":
            for g in ("idc1", "idc2"):
                for t in STEPS:
                    xs = [v for (h, i), v in instant(rows, t).items() if i == g]
                    out.append([g, stamp(t), printed(quantile(xs), "Float64")])
        else:
            for t in STEPS:
                sums = {}
                for (h, i), v in instant(rows, t).items():
                    sums[i] = wrap(sums.get(i, 0) + v)
                out.append([stamp(t), printed(quantile(sums.values()), "Float64")])
        return out
    if q.startswith("topk"):
        kk = int(q[len("topk("):q.index(",")])
        out = []
        for t in STEPS:
            sel = instant(rows, t)
            # the window orders by value, then the tags descending
            ranked = sorted(sel.items(), key=lambda kv: (kv[1], kv[0]), reverse=True)[:kk]
            out += [[printed(v, "Int64"), h, i, stamp(t)] for (h, i), v in ranked]
        return out
    raise KeyError(q)


# ---- expression cases: {"expr": [...]} over a table {"tags", "fields", "rows": [ts, tags.., fields..]} -------------
# A node is (tags, {tag tuple: {t: (value, type)}}); `run` evaluates one, `print_rows` prints it as the reference does.
def run(expr, tables):
    kind = expr[0]
    if kind == "sel":
        _, name, field, match = expr
        tab = tables[name]
        tags, fi = tab["tags"], 1 + len(tab["tags"]) + tab["fields"].index(field)
        out = {}
        for t in STEPS:
            best = {}
            for row in tab["rows"]:
                key = tuple(row[1:1 + len(tags)])
                if any(row[1 + tags.index(k)] != v for k, v in match.items()):
                    continue
                if t - LOOKBACK < row[0] <= t and (key not in best or best[key][0] <= row[0]):
                    best[key] = (row[0], row[fi])
            for key, (_, v) in best.items():
                out.setdefault(key, {})[t] = (int(v), "Int64")
        return tags, out
    if kind == "sum_by":
        tags, series = run(expr[2], tables)
        by = expr[1]
        out = {}
        for key, cells in series.items():
            g = tuple(key[tags.index(b)] for b in by)
            for t, (v, _) in cells.items():
                old = out.setdefault(g, {}).get(t, (0, "Int64"))[0]
                out[g][t] = (wrap(old + v), "Int64")
        return list(by), out
    if kind == "scalar":
        tags, series = run(expr[1], tables)
        live = [k for k, c in series.items() if c]
        one = series[live[0]] if len(live) == 1 else {}
        return [], {(): {t: (float(one[t][0]) if t in one else float("nan"), "Float64") for t in STEPS}}
    if kind == "op":
        _, op, c, left, child = expr
        tags, series = run(child, tables)
        return tags, {k: {t: ((c + float(v)) if left else (float(v) + c), "Float64") for t, (v, _) in cells.items()}
                      for k, cells in series.items()}
    if kind == "bin":
        _, op, lhs, rhs, side = expr
        (lt, ls), (rt, rs) = run(lhs, tables), run(rhs, tables)
        out, tags = {}, lt if side == "lhs" else rt
        for lk, lc in ls.items():
            for rk, rc in rs.items():
                key = lk if side == "lhs" else rk
                for t in STEPS:
                    if t in lc and t in rc:
                        out.setdefault(key, {})[t] = (float(lc[t][0]) + float(rc[t][0]), "Float64")
        return tags, out
    if kind == "fn":
        _, name, args, child = expr
        tags, series = run(child, tables)
        lo = -np.finfo(np.float64).max if name == "clamp_max" else args[0]
        hi = args[1] if name == "clamp" else np.finfo(np.float64).max if name == "clamp_min" else args[0]
        return tags, {k: {t: (lo if float(v) < lo else hi if float(v) > hi else float(v), "Float64")
                          for t, (v, _) in cells.items()} for k, cells in series.items()}
    raise KeyError(kind)


def print_rows(expr, tables):
    """the rows of `expr` in the reference's column order: topk {value, tags.., ts} per step by rank; scalar() and an
    operator on it {ts, value}; a vector binary operator {tags.., ts, value}; a function {ts, value, tags..}"""
    kind = expr[0]
    if kind == "topk":
        _, kk, bottom, child = expr
        tags, series = run(child, tables)
        out = []
        for t in STEPS:
            cells = [(v, key, typ) for key, c in series.items() if t in c for v, typ in [c[t]]]
            # value, then the tags: descending for topk, ascending for bottomk (the window's order)
            cells.sort(key=lambda x: (x[0], x[1]), reverse=not bottom)
            out += [[printed(v, typ)] + list(key) + [stamp(t)] for v, key, typ in cells[:kk]]
        return out
    tags, series = run(expr, tables)
    out = []
    for key, cells in series.items():
        for t, (v, typ) in cells.items():
            if kind in ("scalar", "op"):
                out.append([stamp(t), printed(v, typ)])
            elif kind == "bin":
                out.append(list(key) + [stamp(t), printed(v, typ)])
            else:
                out.append([stamp(t), printed(v, typ)] + list(key))
    return out


def instant_select(ts, vals, offsets, start, end, interval, lookback):
    """InstantManipulate over F field columns with an Int64 field 0: at each step t the row in front of t is chosen,
    the last row with ts <= t or, where rows share ts == t, the first of them (instant_manipulate.rs:523-541), when
    it is fresh: ts + lookback > t, or ts == t at lookback 0; no stale-NaN test.  Rows sorted by ts.
    -> (outs [F,S,T] int64 bits, ok [S,T])"""
    T = (end - start) // interval + 1
    S = len(offsets) - 1
    steps = start + np.arange(T, dtype=np.int64) * interval
    cols = [np.ascontiguousarray(v).view(np.int64) for v in vals]
    outs = np.zeros((len(vals), S, T), np.int64)
    ok = np.zeros((S, T), bool)
    for s in range(S):
        r0, r1 = int(offsets[s]), int(offsets[s + 1])
        t_s = np.asarray(ts[r0:r1], np.int64)
        if t_s.size == 0:
            continue
        j = np.searchsorted(t_s, steps, side="right") - 1
        has = j >= 0
        at = t_s[np.maximum(j, 0)]
        on_step = has & (at == steps)
        j = np.where(on_step, np.searchsorted(t_s, steps, side="left"), j)
        ok[s] = on_step if lookback <= 0 else has & (at + lookback > steps)
        for f, col in enumerate(cols):
            outs[f, s] = np.where(ok[s], col[r0 + np.maximum(j, 0)], 0)
    return outs, ok
