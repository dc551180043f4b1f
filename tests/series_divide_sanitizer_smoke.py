"""Small end-to-end run of SeriesDivide and the host-pointer range call for compute-sanitizer memcheck: K0 on columns
that end in a partial quad and run a second grid-stride pass, one chunked call whose chunks go over as descriptors,
and every refusal (bad offsets, bad ids) with the context's next call.  An over-read past a device buffer seldom
changes a value; memcheck sees it.  Not collected by pytest (no test_ prefix); run on a GPU box:
  compute-sanitizer --tool memcheck python tests/series_divide_sanitizer_smoke.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from greptimedb_b200 import B2PError, Context, make_params  # noqa: E402
from tests import series_divide_edges as sd  # noqa: E402

T0, SC = 1_700_000_000_000, 15_000


def k0(ctx, ids, S):
    d_sid = torch.from_numpy(ids.view(np.int32)).cuda()
    d_off = torch.full((S + 1,), -1, dtype=torch.int64, device="cuda")
    ctx.series_offsets_dev(d_sid, ids.size, S, d_off)
    return d_off


def main():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ctx = Context(0)
    ctx.use_torch_stream()   # ordered after the torch copies and fills that set up its inputs
    for n in (4096 + 15, 4096 * 2 + 1, 513):
        ids = sd.ids_from_cuts(n, sd.boundary_rows(n, sms))
        S = int(ids[-1]) + 1
        d_off = k0(ctx, ids, S)
        ctx.sync()
        assert (d_off.cpu().numpy().view(np.uint64) == sd.offsets_fast(ids, S)[0]).all(), n
    for lay in sd.bad_cases(sms):
        n, S = lay.ids.size, lay.n_series
        d_off = k0(ctx, lay.ids, S)
        p = make_params("rate", T0, T0 + 7 * SC, SC, 60_000)
        d_ts = torch.arange(n, dtype=torch.int64, device="cuda") * SC + T0
        out = torch.empty(S * 8, dtype=torch.float64, device="cuda")
        valid = torch.empty(S, dtype=torch.int32, device="cuda")
        ctx.range_eval_dev(p, d_ts, torch.ones(n, dtype=torch.float64, device="cuda"), d_off, n, S, out, valid)
        try:
            ctx.sync()
            raise AssertionError(lay.name)
        except B2PError as e:
            assert e.code == sd.E_UNSORTED, lay.name
    # one chunked call of regular series (every chunk described), then refusals and the same call again
    S, N = 6600, 1000
    ts, val, sid = (np.repeat(T0 + np.zeros(S, np.int64), N) + np.tile(np.arange(N) * SC, S),
                    np.random.default_rng(1).standard_normal(S * N), np.repeat(np.arange(S, dtype=np.uint32), N))
    offs = np.arange(S + 1, dtype=np.uint64) * N
    p = make_params("sum_over_time", T0, T0 + 999 * SC, 60_000, 300_000)
    first = ctx.range_eval_n(p, ts, val, sid, None, S)[:2]
    assert ctx.last_h2d_bytes() < 20 * S * N
    for n_series in (S, 600):   # chunked, one shot
        for where in ("decrease", "past_rows"):
            o = offs[:n_series + 1].copy()
            if where == "decrease":
                o[7] = o[8] + 1
            else:
                o[-1] = n_series * N + 1
            try:
                ctx.range_eval_n(p, ts[:n_series * N], val[:n_series * N], None, o, n_series)
                raise AssertionError("bad offsets accepted")
            except B2PError as e:
                assert e.code == sd.E_INVALID
        bad = sid[:n_series * N].copy()
        bad[-3:] = 0xFFFFFFFF
        try:
            ctx.range_eval_n(p, ts[:bad.size], val[:bad.size], bad, None, n_series)
            raise AssertionError("bad ids accepted")
        except B2PError as e:
            assert e.code == sd.E_UNSORTED
    again = ctx.range_eval_n(p, ts, val, sid, None, S)[:2]
    assert (again[1] == first[1]).all() and (again[0].view(np.uint64) == first[0].view(np.uint64)).all()
    ctx.close()
    print("series divide sanitizer smoke ok")


if __name__ == "__main__":
    main()
