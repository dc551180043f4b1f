"""One small call per kernel path of the multi-field selectors (K16-K18 in b2p_fields.cuh), for a compute-sanitizer run
on a GPU machine:

    compute-sanitizer --tool memcheck python tests/multifield_sanitizer_smoke.py

Paths: the range form with filter_nan (context copies, K16, the range tiers per field, K18) and without it (K18 only);
the instant form (K17); each through the device form, plus the host form of the range call.  Each result is checked
against tests/multifield_oracle.py."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch

    from greptimedb_b200 import Context, make_params
    from oracle import oracle as orc
    from tests import multifield_oracle as mf

    rng = np.random.default_rng(16)
    S, n, F, T, T0 = 7, 50, 3, 45, 1_700_000_000_000
    ts = np.concatenate([T0 + np.arange(n) * 15_000 + rng.integers(0, 3000, n) for _ in range(S)]).astype(np.int64)
    offsets = np.arange(S + 1, dtype=np.uint64) * n
    vals = [np.cumsum(rng.uniform(0, 5, S * n)) for _ in range(F)]
    for v in vals:
        v[rng.random(S * n) < 0.05] = np.nan
    ctx = Context(0)
    cuda = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    d_ts, d_off, d_vals = cuda(ts), cuda(offsets), [cuda(v) for v in vals]
    Tw = (T + 31) // 32
    for filter_nan in (True, False):
        p = make_params("rate", T0, T0 + (T - 1) * 20_000, 20_000, 60_000, filter_nan=filter_nan)
        op = orc.make_params("rate", T0, T0 + (T - 1) * 20_000, 20_000, 60_000, filter_nan=filter_nan)
        outs = [torch.zeros((S, T), dtype=torch.float64, device="cuda") for _ in range(F)]
        valid = torch.zeros((S, Tw), dtype=torch.int32, device="cuda")
        ctx.range_eval_fields_dev(p, d_ts, d_vals, d_off, ts.size, S, outs, valid)
        ctx.sync()
        e_outs, e_valid = mf.range_query_fields(op, ts, vals, offsets, rescan=True)
        assert np.array_equal(valid.cpu().numpy().view(np.uint32), e_valid)
        if filter_nan:
            h_outs, h_valid = ctx.range_eval_fields(p, ts, vals, offsets=offsets)
            assert np.array_equal(h_valid, e_valid)
    outs = [torch.zeros((S, T), dtype=torch.float64, device="cuda") for _ in range(F)]
    valid = torch.zeros((S, Tw), dtype=torch.int32, device="cuda")
    ctx.instant_select_fields_dev(T0, T0 + (T - 1) * 20_000, 20_000, 45_000, 0, d_ts, d_vals, d_off, ts.size, S, outs,
                                  valid)
    ctx.sync()
    e_outs, e_valid = mf.instant_query_fields(ts, vals, offsets, T0, T0 + (T - 1) * 20_000, 20_000, 45_000)
    assert np.array_equal(valid.cpu().numpy().view(np.uint32), e_valid)
    assert np.array_equal(np.stack([o.cpu().numpy() for o in outs]).view(np.uint64), e_outs.view(np.uint64))
    ctx.close()
    print("multifield sanitizer smoke ok")


if __name__ == "__main__":
    main()
