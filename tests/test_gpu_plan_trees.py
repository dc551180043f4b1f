"""GPU: random PromQL expression trees through the plan layer, bit for bit against the row-literal interpreter of
tests/plan_tree_oracle.py, which composes the single-node oracles from the tables' raw rows up to the root.

Each seed draws a grid (T in {1, 31, 32, 33, 64, 65, 200}, start not aligned to the samples), three tables of seeded value
classes (NaNs with payloads, ±0, ±inf, subnormals, values near ±f64::MAX, counters with resets, duplicate timestamps,
series that start mid-grid or never reach it, NULL and empty labels) and a tree of depth <= 4 with <= 8 nodes.  The
device's rows must equal the interpreter's as a multiset of (labels, ts), in order where the reference pins it, with the
same value bits (-0.0 != +0.0); an unpinned cell (a computed NaN, or one an ordering read) only has to be a NaN where the
interpreter has one, and a `maybe` row only may exist.  At most 5 % of the compared cells may be unpinned.  Building the
same tree again in the same context must give the same rows and bits (a computed NaN as a NaN).  A failing tree is reported with its seed, its PromQL and
the lowest subtree whose device result differs.  PLAN_TREES_SEEDS=<n> draws n seeds instead of the default."""
import math
import os
import struct

import pyarrow as pa
import pytest

from tests import plan_tree_oracle as pto

pytestmark = pytest.mark.gpu

SEEDS = int(os.environ.get("PLAN_TREES_SEEDS", "300"))
MAX_UNPINNED = 0.05


@pytest.fixture(scope="module")
def ctx():
    from greptimedb_b200 import Context
    c = Context(0)
    yield c
    c.close()


def _bits(x):
    return struct.unpack("<Q", struct.pack("<d", float(x)))[0]


def device_rows(b):
    """-> (tag names, value type, [(value, {tag: label}, ts)] in the batch's order)"""
    if b.num_columns == 0:
        return [], None, []
    ti = next(i for i, f in enumerate(b.schema) if pa.types.is_timestamp(f.type))
    vi = next(i for i, f in enumerate(b.schema) if i != ti and not pa.types.is_string(f.type))
    names = b.schema.names
    tags = [n for i, n in enumerate(names) if i not in (vi, ti)]
    ts = b.column(ti).cast(pa.int64()).to_pylist()
    vals = b.column(vi).to_pylist()
    cols = {t: b.column(names.index(t)).to_pylist() for t in tags}
    return tags, str(b.schema.types[vi]), [(vals[r], {t: cols[t][r] for t in tags}, ts[r]) for r in range(b.num_rows)]


def _key(labels, ts):
    return tuple(sorted((k, (0, "") if v is None else (1, v)) for k, v in labels.items())), ts


def diff(batch, res: pto.Result):
    """the first difference between a device batch and the interpreter's result, or None"""
    tags, vtype, got = device_rows(batch)
    exp = res.export
    if exp and sorted(tags) != sorted(res.tags):
        return f"tags {tags} != {res.tags}"
    if exp and vtype != "double":
        return f"value type {vtype}"
    by_key = {}
    for r in exp:
        by_key.setdefault(_key(r.labels, r.ts), []).append(r)
    seen = {}
    for v, lab, ts in got:
        seen.setdefault(_key(lab, ts), []).append(v)
    for k in set(by_key) | set(seen):
        want, have = by_key.get(k, []), sorted(seen.get(k, []), key=_bits)
        sure = [r for r in want if not r.maybe]
        if not (len(sure) <= len(have) <= len(want)):
            return f"row {k}: device {len(have)} rows, interpreter {len(sure)}..{len(want)}: " \
                   f"{have[:4]} vs {[(r.value, r.pin, r.maybe) for r in want[:4]]}"
        left = list(have)
        for r in sorted(want, key=lambda r: (r.pin != pto.BITS, r.maybe)):
            if r.pin == pto.BITS:
                hit = next((i for i, x in enumerate(left) if _bits(x) == _bits(r.value)), None)
            elif r.pin == pto.NAN:
                hit = next((i for i, x in enumerate(left) if math.isnan(x)), None)
            else:
                hit = 0 if left else None
            if hit is None:
                if r.maybe:
                    continue
                return f"row {k}: value {r.value!r} ({r.pin}) not among the device's {have}"
            left.pop(hit)
        if left:
            return f"row {k}: device values {left} left over"
    if res.ordered and not any(r.maybe for r in exp):
        want = [_key(r.labels, r.ts) for r in exp]
        have = [_key(lab, ts) for _, lab, ts in got]
        if want != have:
            i = next(i for i, (a, b) in enumerate(zip(want, have)) if a != b)
            return f"order differs at row {i}: device {have[i]} vs {want[i]}"
    return None


def localise(ctx, tree, tables, grid):
    """the lowest subtree whose device result differs from the interpreter's, with the difference"""
    for sub in tree.subtrees():
        d = diff(pto.build(ctx, sub, tables, grid).execute(), pto.evaluate(sub, tables, grid))
        if d:
            return sub, d
    return None, None


def check_tree(ctx, seed, tree, tables, grid, stats):
    from greptimedb_b200 import B2PError
    res = pto.evaluate(tree, tables, grid)
    try:
        out = pto.build(ctx, tree, tables, grid).execute()
    except B2PError as e:
        pytest.fail(f"seed {seed}: the plan refused a drawn tree: {pto.promql(tree)}: {e}")
    d = diff(out, res)
    if d:
        sub, sd = localise(ctx, tree, tables, grid)
        where = f"lowest differing subtree: {pto.promql(sub)}: {sd}" if sub is not None else "no subtree differs alone"
        pytest.fail(f"seed {seed} grid {grid}: {pto.promql(tree)}: {d}; {where}")
    again = pto.build(ctx, tree, tables, grid).execute()
    d = repeat_diff(again, out, res)
    assert d is None, f"seed {seed}: a second build differs: {pto.promql(tree)}: {d}"
    stats["trees"] += 1
    stats["nodes"] += tree.size()
    stats["cells"] += len(res.export)
    stats["unpinned"] += sum(1 for r in res.export if r.pin != pto.BITS or r.maybe)


def repeat_diff(a, b, res):
    """the first difference between two executes of one tree, or None.  Columns equal, floating-point cells by their
    bits; a NaN the interpreter does not pin by its bits only has to be a NaN again, because the route of a range call
    depends on the context's earlier calls (DESIGN.md §2, "NaN payloads across tiers")."""
    if a.schema != b.schema:
        return f"schema {a.schema} != {b.schema}"
    pinned = {_key(r.labels, r.ts) for r in res.export if r.pin == pto.BITS}
    _, _, ra = device_rows(a)
    _, _, rb = device_rows(b)
    for i, f in enumerate(a.schema):
        x, y = a.column(i).to_pylist(), b.column(i).to_pylist()
        for r, (u, v) in enumerate(zip(x, y)):
            if pa.types.is_floating(f.type) and u is not None and v is not None:
                if _bits(u) == _bits(v) or (math.isnan(u) and math.isnan(v) and _key(ra[r][1], ra[r][2]) not in pinned):
                    continue
            elif u == v:
                continue
            return f"column {f.name} row {r}: {u!r} vs {v!r}"
    return None


def test_random_trees(ctx):
    stats = {"trees": 0, "nodes": 0, "cells": 0, "unpinned": 0}
    for seed in range(SEEDS):
        tree, tables, grid = pto.draw_case(seed)
        check_tree(ctx, seed, tree, tables, grid, stats)
    print(f"plan trees: {stats}")
    assert stats["cells"] > 0
    assert stats["unpinned"] <= MAX_UNPINNED * stats["cells"], stats
