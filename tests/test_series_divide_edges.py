"""CPU: the SeriesDivide reference of tests/series_divide_edges.py against np.searchsorted and the oracle, and the
library's host-side SeriesDivide and cadence scan (b2p_host_scan_series, no device work) on every layout and
timestamp class, by ids at several sid_base values and by offsets that start past row 0.  Every class must run."""
import ctypes as C

import numpy as np
import pytest

from oracle import oracle as orc
from tests import series_divide_edges as sd


@pytest.fixture(scope="module")
def L():
    from greptimedb_b200 import _lib
    return _lib.load()


def _scan(L, ts, sid, offs, n_series, base=0):
    ts = np.ascontiguousarray(ts, np.int64)
    out = np.full(n_series + 1, 0xFFFFFFFFFFFFFFFF, np.uint64)
    t0 = np.zeros(n_series, np.int64)
    cad = np.zeros(n_series, np.int64)
    reg = C.c_int32(-1)
    p = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
    sid = None if sid is None else np.ascontiguousarray(sid, np.uint32)
    offs = None if offs is None else np.ascontiguousarray(offs, np.uint64)
    n = ts.size if sid is None else sid.size
    rc = L.b2p_host_scan_series(p(ts), p(sid), p(offs), n, n_series, base, p(out), p(t0), p(cad), C.addressof(reg))
    return rc, out, t0, cad, reg.value


def _ts_for(offs, seed, irregular):
    """regular timestamps per series (cadences 0, 1, 15 s, 2^40 ms in turn), one row off when `irregular`"""
    S = len(offs) - 1
    cads = np.array([0, 1, 15000, 1 << 40], np.int64)[np.arange(S) % 4]
    ts = sd.timestamps(offs, cads, np.arange(S, dtype=np.int64) * 7 - (1 << 41))
    if irregular and ts.size >= 3:
        r = int(np.random.default_rng(seed).integers(1, ts.size))
        ts[r:] += 1   # non-decreasing still
    return ts


def test_reference_matches_searchsorted_and_the_oracle():
    ran = 0
    for lay in sd.layout_cases(big=False):
        if lay.ids.size > 20000:
            continue
        ref, verdict = sd.offsets_ref(lay.ids, lay.n_series)
        fast, v2 = sd.offsets_fast(lay.ids, lay.n_series)
        assert verdict == v2 == (sd.E_UNSORTED if lay.bad else 0), lay.name
        if ref is None:
            continue
        assert (ref == fast).all(), lay.name
        assert ref[-1] == lay.ids.size and ref[0] == 0, lay.name
        ids = lay.ids.astype(np.int64)
        gap_free = ids.size and ids[0] == 0 and ids[-1] == lay.n_series - 1 and (np.diff(ids) <= 1).all()
        if gap_free:   # the oracle restates find_first_diff_row: one series per run of equal ids
            assert (orc.series_divide(lay.ids) == ref).all(), lay.name
            ran += 1
    assert ran > 30
    # a column that never changes is one series; ids below sid_base wrap past n_series
    assert sd.offsets_ref(np.array([5, 5, 5], np.uint32), 6)[0].tolist() == [0, 0, 0, 0, 0, 0, 3]
    assert sd.offsets_ref(np.array([4, 5], np.uint32), 3, sid_base=5)[1] == sd.E_UNSORTED


def test_host_scan_on_every_layout_and_sid_base(L):
    seen = set()
    for i, lay in enumerate(sd.layout_cases()):
        seen |= lay.classes
        ref, verdict = sd.offsets_fast(lay.ids, lay.n_series)
        if lay.bad:
            assert _scan(L, np.zeros(lay.ids.size, np.int64), lay.ids, None, lay.n_series)[0] == sd.E_UNSORTED, lay.name
            continue
        ts = _ts_for(ref, i, irregular=i % 3 == 0)
        t0, cad, reg = sd.scan_ref(ts, ref) if ts.size < 20000 else (None, None, sd.chunk_regular(ts, ref))
        big = lay.ids.size > 20000
        for base in (0, 1, 1 << 31, (1 << 32) - lay.n_series - 1):
            if big and base not in (0, 1 << 31):
                continue
            sid = (lay.ids.astype(np.uint64) + base).astype(np.uint32)
            rc, off, g_t0, g_cad, g_reg = _scan(L, ts, sid, None, lay.n_series, base)
            assert rc == 0 and (off == ref).all(), (lay.name, base)
            assert g_reg == int(reg), (lay.name, base)
            if t0 is not None:
                assert (g_t0 == t0).all() and (g_cad == cad).all(), (lay.name, base)
            if lay.ids.size and base:   # an id below sid_base is refused, wherever it is
                bad = sid.copy()
                bad[-1] = base - 1
                assert _scan(L, ts, bad, None, lay.n_series, base)[0] == sd.E_UNSORTED, (lay.name, base)
                bad = sid.copy()
                bad[0] = base - 1
                assert _scan(L, ts, bad, None, lay.n_series, base)[0] == sd.E_UNSORTED, (lay.name, base)
        # the offsets form, offsets_in[0] > 0: rebased to the batch, whose first row is offsets_in[0]
        if not big:
            rc, off, g_t0, g_cad, g_reg = _scan(L, ts, None, ref + np.uint64(40), lay.n_series)
            assert rc == 0 and (off == ref).all() and g_reg == int(reg), lay.name
            assert (g_t0 == t0).all() and (g_cad == cad).all(), lay.name
    assert seen >= sd.CLASSES, sorted(sd.CLASSES - seen)


def test_host_scan_on_every_timestamp_class(L):
    seen = set()
    for name, ts, offs, regular in sd.ts_cases():
        seen.add(name.split("/")[0])
        if name.endswith("negative_epoch"):
            seen.add("negative_epoch")
        S = len(offs) - 1
        t0, cad, reg = sd.scan_ref(ts, offs)
        assert reg == regular, name
        sid = np.repeat(np.arange(S, dtype=np.uint32), np.diff(offs).astype(np.int64))
        lens = np.diff(offs)
        seen |= {"one_row"} if (lens == 1).any() else set()
        seen |= {"empty"} if (lens == 0).any() else set()
        for by_ids in (True, False):
            rc, off, g_t0, g_cad, g_reg = _scan(L, ts, sid if by_ids else None, None if by_ids else offs, S)
            assert rc == 0 and (off == offs).all(), name
            assert (g_t0 == t0).all() and (g_cad == cad).all() and g_reg == int(regular), name
    assert seen >= set(sd.TS_CLASSES), sorted(set(sd.TS_CLASSES) - seen)


def test_host_scan_refuses_offsets_that_decrease_or_run_past_the_rows(L):
    ts = np.arange(10, dtype=np.int64)
    assert _scan(L, ts, None, np.array([0, 3, 2, 10], np.uint64), 3)[0] == sd.E_INVALID
    assert _scan(L, ts, None, np.array([0, 3, 5, 11], np.uint64), 3)[0] == sd.E_INVALID
    assert _scan(L, ts, None, np.array([0, 3, 5, 10], np.uint64), 3)[0] == 0


def test_chunk_table_covers_every_series_and_row():
    """the restated chunk planning: one shot at or below 6 291 456 rows or under 64 series; otherwise chunks of whole
    series, contiguous in rows, the last ending at the last series' end"""
    assert sd.plan_chunks(sd.ONE_SHOT_ROWS, 1000, offsets=np.zeros(1001)) is None
    assert sd.plan_chunks(sd.ONE_SHOT_ROWS + 1, 63, offsets=np.zeros(64)) is None
    n, S = sd.ONE_SHOT_ROWS + 1, 64
    offs = np.linspace(0, n, S + 1).astype(np.uint64)
    ch = sd.plan_chunks(n, S, offsets=offs)
    assert len(ch) == 1 and (ch[0].s0, ch[0].s1, ch[0].r0, ch[0].r1) == (0, 64, 0, n)
    S = 9000
    offs = np.linspace(0, 9_000_000, S + 1).astype(np.uint64)
    ids = np.repeat(np.arange(S, dtype=np.uint32), np.diff(offs).astype(np.int64))
    a, b = sd.plan_chunks(ids.size, S, ids=ids), sd.plan_chunks(ids.size, S, offsets=offs)
    assert [(k.s0, k.s1, k.r0, k.r1) for k in a] == [(k.s0, k.s1, k.r0, k.r1) for k in b]
    C_ = 4194304 // (1000 + 1)
    assert [k.s0 for k in a] == list(range(0, S, C_)) and a[-1].r1 == ids.size
    assert all(k.r1 == n.r0 for k, n in zip(a, a[1:]))
    assert sd.h2d_bytes(ids.size, S, a, "ids") == 20 * ids.size
    assert sd.h2d_bytes(ids.size, S, b, "offsets") == 16 * ids.size + 8 * (S + len(b))
