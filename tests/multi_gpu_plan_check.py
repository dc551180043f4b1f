"""Multi-rank check of sharded plan nodes over the library's communicator (run under torchrun, one rank per GPU; started
by tests/test_multi_gpu.py when at least two GPUs are visible): every rank regenerates the same table from a seed,
pushes the series distributed.shard_of_series gives it into a sharded aggregate node (and, over Float64, a leaf with a
sharded aggregate stage) and a sharded count_values node, and its export must equal the unsharded node over the whole table on
its own GPU: bit for bit for count, group, min, max, quantile, count_values and Int64 sum; the Float64 sum and avg bit
for bit at two ranks against the host mirror (each rank's partials from the unsharded node over its shard, added in
rank order), and within 1e-9 relative otherwise, as stddev and stdvar (the ranks' partials add in another order).  A
second pass puts every series on rank 0, so the other ranks read no batch and must take rank 0's Int64 types.  Every
rank's export must be the same bytes.  torch.distributed only carries the
128-byte communicator id, the export digests and the verdict."""
import hashlib
import os
import sys

import numpy as np
import pyarrow as pa
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.ranks import rank_session  # noqa: E402

EXACT = {"count", "group", "min", "max", "quantile"}


def table(seed, i64, keep=None):
    """series s: labels (host, idc, sid), 60 steps of samples; keep(s) selects this rank's series"""
    rng = np.random.default_rng(seed)
    hosts = [None, "", "h1", "é", "日本"]
    cols = {"ts": [], "host": [], "idc": [], "sid": [], "v": []}
    series = sorted(range(400), key=lambda s: (hosts[s % 5] is not None, hosts[s % 5] or "", f"dc{s % 7}", f"s{s:04d}"))
    for s in series:
        vals = rng.integers(-1000, 1000, 60) if i64 else rng.normal(size=60) * 1e3
        if keep is not None and not keep(s):
            continue
        for t in range(60):
            if (s * 31 + t) % 5 == 0:
                continue
            cols["ts"].append(t * 1000)
            cols["host"].append(hosts[s % 5])
            cols["idc"].append(f"dc{s % 7}")
            cols["sid"].append(f"s{s:04d}")
            cols["v"].append(int(vals[t]) if i64 else float(vals[t]))
    return pa.record_batch([pa.array(cols["ts"], pa.timestamp("ms")), pa.array(cols["host"], pa.utf8()),
                            pa.array(cols["idc"], pa.utf8()), pa.array(cols["sid"], pa.utf8()),
                            pa.array(cols["v"], pa.int64() if i64 else pa.float64())],
                           names=["ts", "host", "idc", "sid", "v"])


def leaf(ctx, batch, aggregate=None, by=()):
    from greptimedb_b200.plan import PromRangeExec
    ex = PromRangeExec(ctx, "", 0, 59_000, 1000, 0, "ts", "v", ["host", "idc", "sid"], lookback_delta=2000,
                       aggregate=aggregate, by_columns=by)
    if batch.num_rows:  # (a rank whose regions hold no series reads no batch)
        ex.push(batch)
    return ex


def digest(b):
    sink = pa.BufferOutputStream()
    with pa.ipc.new_stream(sink, b.schema) as w:
        w.write_batch(b)
    return hashlib.sha256(sink.getvalue().to_pybytes()).hexdigest()


def agree(got, exp, exact):
    if got.schema != exp.schema or got.num_rows != exp.num_rows:
        return False
    for x, y in zip(got.columns, exp.columns):
        if pa.types.is_floating(x.type):
            a, b = x.to_numpy(zero_copy_only=False), y.to_numpy(zero_copy_only=False)
            if exact and not (a.view(np.uint64) == b.view(np.uint64)).all():
                return False
            if not exact and not np.allclose(a, b, rtol=1e-9, atol=0, equal_nan=True):
                return False
        elif not x.equals(y):
            return False
    return True


def keyed(b):
    """{(every column but the value, as a tuple): the value} of an aggregate export {labels.., ts, value}"""
    cols = [c.to_pylist() for c in b.columns]
    return {tuple(c[i] for c in cols[:-1]): cols[-1][i] for i in range(b.num_rows)}


def mirror(plain, world, op, by, i64, owner_of):
    """sum / avg of two ranks as the sharded node merges them: each rank's (sum, count) partials over its own shard,
    absent groups 0, added in rank order -> {key: value}"""
    from greptimedb_b200.plan import AggregatePlan
    kw = {"by": by} if by else {}
    parts = [(keyed(AggregatePlan(plain, "sum", leaf(plain, table(5, i64, lambda s, r=r: owner_of(s) == r)), **kw).execute()),
              keyed(AggregatePlan(plain, "count", leaf(plain, table(5, i64, lambda s, r=r: owner_of(s) == r)), **kw).execute()))
             for r in range(world)]
    out = {}
    for k in set().union(*(p[0] for p in parts)):
        s = np.float64(parts[0][0].get(k, 0.0))
        for p in parts[1:]:
            s = s + np.float64(p[0].get(k, 0.0))
        c = sum(p[1].get(k, 0.0) for p in parts)
        out[k] = float(s) if op == "sum" else float(s / np.float64(c))
    return out


def main(s):
    rank, world, ctx = s.rank, s.world, s.ctx
    from greptimedb_b200 import Context
    from greptimedb_b200 import distributed as D
    from greptimedb_b200.plan import AggregatePlan, CountValuesPlan
    plain = Context(ctx.device)
    owner_of = lambda s: int(D.shard_of_series(np.array([s], np.uint32), world)[0])  # noqa: E731
    mine = lambda s: owner_of(s) == rank  # noqa: E731
    bad, digests = [], []
    for i64 in (False, True):
        whole, shard = table(5, i64), table(5, i64, mine)
        for by in (["idc"], None):
            kw = {"by": by} if by else {}
            exp = CountValuesPlan(plain, "value", leaf(plain, whole), **kw).execute()
            got = CountValuesPlan(ctx, "value", leaf(ctx, shard), **kw).sharded().execute()
            if not agree(got, exp, True):
                bad.append(("count_values", i64, by))
            digests.append(digest(got))
        if world == 2 and not i64:
            for op in ("sum", "avg"):
                for by in (["idc"], ["host"], None):
                    kw = {"by": by} if by else {}
                    got = keyed(AggregatePlan(ctx, op, leaf(ctx, shard), **kw).sharded().execute())
                    exp = mirror(plain, world, op, by, i64, owner_of)
                    if got.keys() != exp.keys() or any(
                            np.float64(got[k]).view(np.uint64) != np.float64(exp[k]).view(np.uint64) for k in exp):
                        bad.append(("two-rank mirror", op, by))
        for op in ("sum", "avg", "count", "min", "max", "stddev", "stdvar", "group", "quantile"):
            for by in (["idc"], ["host"], None):
                kw = {"by": by} if by else {}
                param = 0.25 if op == "quantile" else None
                exp = AggregatePlan(plain, op, leaf(plain, whole), param=param, **kw).execute()
                got = AggregatePlan(ctx, op, leaf(ctx, shard), param=param, **kw).sharded().execute()
                exact = op in EXACT or (i64 and op in ("sum", "min", "max"))
                if not agree(got, exp, exact):
                    bad.append((op, i64, by))
                digests.append(digest(got))
        for op in ("sum", "max") if not i64 else ():  # (a leaf's aggregate stage reads Float64 fields only)
            exp = leaf(plain, whole, op, ["idc"]).execute()
            got = leaf(ctx, shard, op, ["idc"]).sharded().execute()
            if not agree(got, exp, op == "max"):
                bad.append(("leaf-" + op, i64))
            digests.append(digest(got))
    # every series on rank 0: the other ranks read no batch (their default types are Float64)
    for op in ("sum", "min", "max"):
        whole, shard = table(5, True), table(5, True, lambda s: rank == 0)
        exp = AggregatePlan(plain, op, leaf(plain, whole), by=["idc"]).execute()
        got = AggregatePlan(ctx, op, leaf(ctx, shard), by=["idc"]).sharded().execute()
        if not agree(got, exp, True):
            bad.append(("empty ranks", op))
        digests.append(digest(got))
    exp = CountValuesPlan(plain, "value", leaf(plain, table(5, True))).execute()
    got = CountValuesPlan(ctx, "value", leaf(ctx, table(5, True, lambda s: rank == 0))).sharded().execute()
    if not agree(got, exp, True):
        bad.append(("empty ranks", "count_values"))
    digests.append(digest(got))
    every = [None] * world
    dist.all_gather_object(every, digests)
    if any(d != every[0] for d in every):
        bad.append("exports differ across ranks")
    plain.close()
    return bad


if __name__ == "__main__":
    rank_session("MULTI_GPU_PLAN_CHECK", main)
