"""GPU: the instant selector at its edges, on every route, bit for bit against the literal interpreter of the
reference's cursor walk (tests/instant_edges.py):
  K4 value mode      b2p_instant_select by offsets and by sid; b2p_instant_select_dev
  K4 timestamp mode  b2p_instant_timestamp, b2p_instant_timestamp_dev: (double)(ts + offset) / 1000.0, no staleness
  K17 Float64        b2p_instant_select_fields[_dev] at F = 1, 2, 3, 8, 64 (B2P_MAX_FIELDS); one Float64 field is
                     handed to K4 (instant_select_fields in b2p_range.cu), so K17<true> runs from F = 2 on; a NaN in
                     a field past 0 is moved by its bits, never tested
  K17 Int64          b2p_instant_select_fields_i64: K17<false> at every F, field 0 never stale whatever its bits
  plan layer         the PromRangeExec instant leaf, one and three fields
and K17 against K4 on the same rows: K17<true> over [field 0, field 0] gives K4's grid twice, and K17<false> over the
timestamp column as an Int64 field takes the rows K4's timestamp mode takes.

Bit for bit: the validity words are equal, bits past T included (zero); invalid cells hold +0.0; values compare by
their bits (-0.0 != +0.0, NaN payloads kept).  The device forms write into buffers filled with a NaN pattern, so a
cell the kernel leaves unwritten fails.  F = 8 and 64 run on the cases of at most 2^20 and 2^16 cells.
"""
import numpy as np
import pytest

from tests import instant_edges as ie

pytestmark = pytest.mark.gpu

CASES = ie.cases()
POISON = 0x7FF4DEADDEADBEEF  # a signalling NaN no route writes
FIELD_COUNTS = (1, 2, 3, 8, 64)
MAX_CELLS = {8: 1 << 20, 64: 1 << 16}
PLAN_CELLS = 1 << 18


@pytest.fixture(scope="module")
def ctx():
    from greptimedb_b200 import Context
    c = Context(0)
    yield c
    c.close()


def ids(c):
    return c.name


def check(case, route, got_bits, got_words, exp_bits, exp_words):
    why = ie.first_difference(got_bits, exp_bits, got_words, exp_words, case.T)
    assert not why, f"{route}: {case.describe()}: {why}"


def dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).to("cuda")


def poisoned(shape):
    import torch
    return dev(np.full(shape, POISON, np.uint64).view(np.float64)), torch.full((shape[0], (shape[1] + 31) // 32), -1,
                                                                               dtype=torch.int32, device="cuda")


def host(t):
    import torch
    torch.cuda.synchronize()
    return t.cpu().numpy()


def sid_of(case):
    return np.repeat(np.arange(case.S, dtype=np.uint32), np.diff(case.offsets.astype(np.int64)))


def grid_args(case):
    return case.start, case.end, case.interval, case.lookback, case.offset


def test_the_largest_case_strides_on_this_device():
    """warps take a second series: the largest case holds rows past the warps capped_grid launches here (8 CTAs of 8
    warps per SM)"""
    import torch
    warps = torch.cuda.get_device_properties(0).multi_processor_count * 8 * 8
    big = max(CASES, key=lambda c: c.S)
    assert (np.diff(big.offsets.astype(np.int64))[warps:] > 0).any(), f"{big.name}: no series past warp {warps}"


# ---- K4 ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES, ids=ids)
def test_k4_value_host(ctx, case):
    want, words = ie.expected_values(case, [case.val])
    out, valid = ctx.instant_select(case.ts, case.val, *grid_args(case), offsets=case.offsets)
    check(case, "K4 host by offsets", out.view(np.uint64), valid, want[0], words)
    # by sid: the series count is the largest sid + 1, so trailing empty series are not rows of the result
    out, valid = ctx.instant_select(case.ts, case.val, *grid_args(case), sid=sid_of(case))
    S = out.shape[0]
    assert not words[S:].any()
    check(case, "K4 host by sid", out.view(np.uint64), valid, want[0][:S], words[:S])


@pytest.mark.parametrize("case", CASES, ids=ids)
def test_k4_value_device(ctx, case):
    import torch
    want, words = ie.expected_values(case, [case.val])
    out, valid = poisoned((case.S, case.T))
    d_ts, d_val, d_off = dev(case.ts), dev(case.val), dev(case.offsets.view(np.int64))
    torch.cuda.synchronize()
    ctx.instant_select_dev(*grid_args(case), d_ts, d_val, d_off, case.ts.size, case.S, out, valid)
    ctx.sync()
    check(case, "K4 device", host(out).view(np.uint64), host(valid).view(np.uint32), want[0], words)


@pytest.mark.parametrize("case", CASES, ids=ids)
def test_k4_timestamp(ctx, case):
    import torch
    want, words = ie.expected_timestamps(case)
    out, valid = ctx.instant_timestamp(case.ts, *grid_args(case), offsets=case.offsets)
    check(case, "K4 timestamp host", out.view(np.uint64), valid, want, words)
    d_out, d_valid = poisoned((case.S, case.T))
    d_ts, d_off = dev(case.ts), dev(case.offsets.view(np.int64))
    torch.cuda.synchronize()
    ctx.instant_timestamp_dev(*grid_args(case), d_ts, d_off, case.ts.size, case.S, d_out, d_valid)
    ctx.sync()
    check(case, "K4 timestamp device", host(d_out).view(np.uint64), host(d_valid).view(np.uint32), want, words)


# ---- K17 -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case,F", [(c, F) for c in CASES for F in FIELD_COUNTS
                                    if c.S * c.T <= MAX_CELLS.get(F, 1 << 62)],
                         ids=lambda x: x.name if isinstance(x, ie.Case) else f"F{x}")
def test_k17_float64(ctx, case, F):
    import torch
    cols = [case.val] + ie.extra_fields(case, F)
    want, words = ie.expected_values(case, cols)
    outs, valid = ctx.instant_select_fields(case.ts, cols, *grid_args(case), offsets=case.offsets)
    check(case, f"K17 host F={F}", outs.view(np.uint64), valid, want, words)
    d_outs = [poisoned((case.S, case.T))[0] for _ in range(F)]
    d_valid = poisoned((case.S, case.T))[1]
    d_cols = [dev(c) for c in cols]
    d_ts, d_off = dev(case.ts), dev(case.offsets.view(np.int64))
    torch.cuda.synchronize()
    ctx.instant_select_fields_dev(*grid_args(case), d_ts, d_cols, d_off, case.ts.size, case.S, d_outs, d_valid)
    ctx.sync()
    got = np.stack([host(o).view(np.uint64) for o in d_outs])
    check(case, f"K17 device F={F}", got, host(d_valid).view(np.uint32), want, words)


@pytest.mark.parametrize("F", (1, 3))
@pytest.mark.parametrize("case", CASES, ids=ids)
def test_k17_int64(ctx, case, F):
    """field 0 is the value column's bits as an Int64: its NaN patterns are values, never stale"""
    cols = [case.val.view(np.int64)] + ie.extra_fields(case, F)
    want, words = ie.expected_values(case, cols, stale=False)
    outs, valid = ctx.instant_select_fields_i64(case.ts, cols, *grid_args(case), offsets=case.offsets)
    check(case, f"K17 Int64 F={F}", outs.view(np.uint64), valid, want, words)


@pytest.mark.parametrize("case", CASES, ids=ids)
def test_k17_agrees_with_k4_on_the_same_rows(ctx, case):
    """K17<true> over [field 0, field 0] is K4's value grid twice; K17<false> over the timestamp column takes the rows
    K4's timestamp mode takes"""
    out, valid = ctx.instant_select(case.ts, case.val, *grid_args(case), offsets=case.offsets)
    outs, valid2 = ctx.instant_select_fields(case.ts, [case.val, case.val], *grid_args(case), offsets=case.offsets)
    for f in range(2):
        check(case, f"K17 field {f} vs K4", outs[f].view(np.uint64), valid2, out.view(np.uint64), valid)
    t_out, t_valid = ctx.instant_timestamp(case.ts, *grid_args(case), offsets=case.offsets)
    i_outs, i_valid = ctx.instant_select_fields_i64(case.ts, [case.ts], *grid_args(case), offsets=case.offsets)
    ok = ie.unpack_words(i_valid, case.T)
    as_ts = np.where(ok, (i_outs[0] + case.offset).astype(np.float64) / 1000.0, 0.0)
    check(case, "K17 Int64 timestamp column vs K4 timestamp mode", as_ts.view(np.uint64), i_valid,
          t_out.view(np.uint64), t_valid)


# ---- the plan layer ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("F", (1, 3))
@pytest.mark.parametrize("case", [c for c in CASES if c.S * c.T <= PLAN_CELLS], ids=ids)
def test_plan_instant_leaf(ctx, case, F):
    """the PromRangeExec instant leaf: one series per host tag (empty series have no rows, so no series), one row per
    valid cell, series by series, step by step"""
    import pyarrow as pa
    from greptimedb_b200.plan import PromRangeExec
    cols = [case.val] + ie.extra_fields(case, F)
    names = [f"f{f}" for f in range(F)]
    sizes = np.diff(case.offsets.astype(np.int64))
    hosts = np.repeat(np.array([f"h{s:05d}" for s in range(case.S)]), sizes)
    batch = pa.record_batch([pa.array(case.ts, pa.timestamp("ms"))] + [pa.array(c, pa.float64()) for c in cols]
                            + [pa.array(hosts)], names=["ts"] + names + ["host"])
    ex = PromRangeExec(ctx, "", case.start, case.end, case.interval, 0, "ts", names if F > 1 else names[0],
                       ["host"], offset=case.offset, lookback_delta=case.lookback)
    ex.push(batch)
    got = ex.execute()
    want, words = ie.expected_values(case, cols)
    ok = ie.unpack_words(words, case.T)
    s_idx, k_idx = np.nonzero(ok)
    route = f"plan instant leaf F={F}"
    assert got.num_rows == s_idx.size, f"{route}: {case.describe()}: {got.num_rows} rows, expected {s_idx.size}"
    g_ts = got.column("ts").cast(pa.int64()).to_numpy()
    e_ts = case.start + k_idx * case.interval
    bad = np.flatnonzero(g_ts != e_ts)
    assert not bad.size, f"{route}: {case.describe()}: row {bad[0]} at ts {g_ts[bad[0]]}, expected {e_ts[bad[0]]}"
    g_host = np.array(got.column("host").to_pylist())
    bad = np.flatnonzero(g_host != np.array([f"h{s:05d}" for s in s_idx]))
    assert not bad.size, f"{route}: {case.describe()}: row {bad[0]} of series {g_host[bad[0]]}"
    for f, name in enumerate(names):
        g = got.column(name).to_numpy(zero_copy_only=False).view(np.uint64)
        e = want[f][s_idx, k_idx]
        bad = np.flatnonzero(g != e)
        assert not bad.size, (f"{route}: {case.describe()}: field {f} differs first at (series {s_idx[bad[0]]}, step "
                              f"{k_idx[bad[0]]}): got 0x{int(g[bad[0]]):016x}, expected 0x{int(e[bad[0]]):016x}")
