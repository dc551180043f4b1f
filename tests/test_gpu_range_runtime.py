"""GPU: the range-call runtime around the kernels on the chunked host path (b2p_range_eval over more than 6 M rows):
a chunk redone after its slow path ran out of arena, series ids the host or K0 rejects, and the hand-off counters and
the adaptive back-off of a call made of several chunks."""
import numpy as np
import pytest

from oracle import oracle as orc

pytestmark = pytest.mark.gpu

T0, SC = 1_700_000_000_000, 15_000
E_UNSORTED = -3


def _ctx():
    from greptimedb_b200 import Context
    return Context(0)


def _same_bits(a, b):
    """two (out, valid) results agree bit for bit in every valid slot"""
    (out_a, valid_a), (out_b, valid_b) = a, b
    assert (valid_a == valid_b).all()
    vb = orc.valid_to_bool(valid_a, out_a.shape[1])
    assert (out_a.view(np.uint64)[vb] == out_b.view(np.uint64)[vb]).all()


def test_chunk_redone_after_arena_overflow_through_host_offsets():
    """Windows longer than the 1024-sample ring send every series to the slow path, and a 4000-row series does not fit
    a warp's region of the default arena: every chunk is redone from its host columns, here with the offsets rebased
    to the chunk.  The redo's copy is counted on top of the call's."""
    from greptimedb_b200 import make_params
    S, N = 1600, 4000   # 6.4 M rows: two chunks
    ts, val, sid = orc.synth_fill(0, S, N, T0, SC, 1000, 1, 0x5EED)
    val[::1013] = np.nan
    offsets = np.arange(S + 1, dtype=np.uint64) * N
    end, step, rng = T0 + (N - 1) * SC, 750_000, 24_000_000   # 1600-sample windows
    p = make_params("sum_over_time", T0, end, step, rng)
    results = {}
    for route in ("offsets", "ids"):
        c = _ctx()   # a fresh context: the default arena
        try:
            by_offsets = route == "offsets"
            out, valid, ets = c.range_eval_n(p, ts, val, None if by_offsets else sid, offsets if by_offsets else None, S)
            assert c.last_slow_series() == S
            if by_offsets:
                assert c.last_h2d_bytes() >= 16 * ts.size
            results[route] = (out, valid)
        finally:
            c.close()
    _same_bits(results["offsets"], results["ids"])
    op = orc.make_params("sum_over_time", T0, end, step, rng)
    e_out, e_valid = orc.range_query(op, ts, val, sid, offsets, threads=8)
    out, valid = results["offsets"]
    gv, ev = orc.valid_to_bool(valid, ets.size), orc.valid_to_bool(e_valid, ets.size)
    assert (gv == ev).all()
    g, e = out[ev], e_out[ev]
    assert (np.isnan(g) == np.isnan(e)).all()
    g, e = g[~np.isnan(e)], e[~np.isnan(e)]
    assert ((g == e) | (np.abs(g - e) <= 1e-9 * np.maximum(np.abs(g), np.abs(e)))).all()
    assert (out[~ev] == 0.0).all()


def test_bad_ids_in_a_chunked_call_fail_and_the_next_call_is_correct():
    """Two rows swapped inside a chunk (K0 finds them on the device) and trailing rows with id == n_series (the host's
    chunk bounds find them) each fail with B2P_E_UNSORTED; the context's next call gives the same bits as before."""
    from greptimedb_b200 import B2PError, make_params
    S, N = 6500, 1000
    ts, val, sid = orc.synth_fill(0, S, N, T0, SC, 1000, 1, 11)
    p = make_params("rate", T0, T0 + 999 * SC, 60_000, 300_000)
    swapped = sid.copy()
    swapped[[10 * N + N - 1, 11 * N]] = swapped[[11 * N, 10 * N + N - 1]]
    trailing = sid.copy()
    trailing[-5:] = S
    c = _ctx()
    try:
        good = c.range_eval_n(p, ts, val, sid, None, S)[:2]
        for bad in (swapped, trailing):
            with pytest.raises(B2PError) as ei:
                c.range_eval_n(p, ts, val, bad, None, S)
            assert ei.value.code == E_UNSORTED
            _same_bits(c.range_eval_n(p, ts, val, sid, None, S)[:2], good)
    finally:
        c.close()


def test_first_tier_backs_off_after_a_chunked_call_it_mostly_declined():
    """Every counter resets: the first tier hands every series of every chunk on, and the call's hand-off count is the
    sum over its chunks.  The verdict, taken once over the whole call, makes the next chunked call run the first tier
    with reset bit words, which hands nothing on; the bits are the same."""
    from greptimedb_b200 import make_params
    S, N = 9000, 1000
    ts, val, sid = orc.synth_fill(0, S, N, T0, SC, 1000, 1, 0x5EED)
    p = make_params("rate", T0, T0 + 999 * SC, SC, 300_000)
    c = _ctx()
    try:
        first = c.range_eval_n(p, ts, val, sid, None, S)[:2]
        assert c.last_warp_tier_series() == S
        second = c.range_eval_n(p, ts, val, sid, None, S)[:2]
        assert c.last_warp_tier_series() == 0
        _same_bits(first, second)
    finally:
        c.close()
