"""One small subquery call per path of K13 (b2p_subquery.cuh), for a compute-sanitizer run on a GPU machine:

    compute-sanitizer --tool memcheck  python tests/subquery_sanitizer_smoke.py
    compute-sanitizer --tool racecheck python tests/subquery_sanitizer_smoke.py

Paths: a grid with holes, an empty row, NaN cells and a T' that is not a multiple of 32 (the count kernel, CUB's scan,
the scatter and the range tiers); the same call through the host-pointer form; a grid with no inner step (the output
is only cleared).  Each result is checked against the row-literal oracle."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch

    from greptimedb_b200 import Context, make_params
    from tests import subquery_oracle as sqo
    from tests.binary_oracle import _words

    rng = np.random.default_rng(13)
    R, start, end, interval, rng_ms, step = 5, 0, 600_000, 60_000, 300_000, 15_000
    s, step, T_in = sqo.inner_grid(start, end, interval, rng_ms, step)
    ok = rng.random((R, T_in)) < 0.8
    ok[1] = False
    vals = np.cumsum(rng.random((R, T_in)), axis=1)
    vals[2, ::3] = np.nan
    valid = _words(ok)
    p = make_params("sum_over_time", start, end, interval, rng_ms, filter_nan=False)
    ctx = Context(0)
    T = (end - start) // interval + 1
    out = torch.zeros((R, T), dtype=torch.float64, device="cuda")
    ov = torch.zeros((R, (T + 31) // 32), dtype=torch.int32, device="cuda")
    before = ctx.launch_count()
    ctx.subquery_dev(p, s, step, torch.from_numpy(vals).cuda(), torch.from_numpy(valid.view(np.int32)).cuda(), R, T_in,
                     out, ov)
    ctx.sync()
    assert ctx.launch_count() - before >= 2
    e_out, e_ov = sqo.subquery("sum_over_time", start, end, interval, rng_ms, s, step, vals, valid)
    assert (ov.cpu().numpy().view(np.uint32) == e_ov).all()
    assert np.allclose(out.cpu().numpy(), e_out, rtol=1e-12, atol=0, equal_nan=True)
    h_out, h_ov = ctx.subquery(p, s, step, vals, valid)
    assert (h_ov == e_ov).all() and np.allclose(h_out, e_out, rtol=1e-12, atol=0, equal_nan=True)
    z_out, z_ov = ctx.subquery(p, s, step, np.zeros((R, 0)), np.zeros((R, 0), np.uint32))
    assert not z_ov.any()
    ctx.close()
    print("subquery sanitizer smoke ok")


if __name__ == "__main__":
    main()
