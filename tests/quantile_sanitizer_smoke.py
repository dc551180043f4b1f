"""One small quantile call per path of K11 (b2p_quantile.cuh), for a compute-sanitizer run on a GPU machine:

    compute-sanitizer --tool memcheck  python tests/quantile_sanitizer_smoke.py
    compute-sanitizer --tool racecheck python tests/quantile_sanitizer_smoke.py
    compute-sanitizer --tool initcheck python tests/quantile_sanitizer_smoke.py

Paths: resident groups (at most 64 members), a multi-pass group finished by one warp (65 .. 256 members here: the chunk
size is at least 256), a group of several chunks (histograms summed across chunks, the advance kernel), and a special φ
(count only).  Each call's launch count shows that it took its path, and each result is checked against the dense
oracle."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch

    from greptimedb_b200 import Context
    from tests import aggregate_oracle as ago
    from tests import binary_oracle as bor

    rng = np.random.default_rng(12)
    T = 65
    # launches of the call: the resident kernel; + one pass kernel (whole groups); + 9 x (pass, advance) (chunked)
    for sizes, phi, launches in [([5, 64, 0, 2], 0.5, 1), ([200, 7], 0.3, 2), ([60_000, 3], 0.99, 19),
                                 ([200, 7], float("nan"), 1)]:
        gid = np.concatenate([np.full(s, g, np.uint32) for g, s in enumerate(sizes)] + [np.full(3, 99, np.uint32)])
        R, G = gid.size, len(sizes)
        vals = rng.standard_normal((R, T))
        vals[rng.random((R, T)) < 0.2] = 1.0
        valid = bor._words(rng.random((R, T)) < 0.8)
        dev = torch.device("cuda:0")
        ctx = Context(0)
        d_vals = torch.from_numpy(vals).to(dev)
        d_valid = torch.from_numpy(valid.view(np.int32).copy()).to(dev)
        ix = ctx.group_index_create_dev(torch.from_numpy(gid.view(np.int32)).to(dev), R, G)
        out = torch.zeros((G, T), dtype=torch.float64, device=dev)
        cnt = torch.zeros((G, T), dtype=torch.int32, device=dev)
        before = ctx.launch_count()
        ctx.group_quantile_dev(phi, d_vals, d_valid, ix, T, out, cnt)
        ctx.sync()
        assert ctx.launch_count() - before == launches, (sizes, ctx.launch_count() - before)
        exp, ecnt = ago.group_quantile(phi, vals, valid, gid, G)
        got = out.cpu().numpy()
        assert (cnt.cpu().numpy().view(np.uint32) == ecnt).all(), sizes
        assert ((np.isnan(got) & np.isnan(exp)) | (got.view(np.uint64) == exp.view(np.uint64))).all(), sizes
        ctx.group_index_destroy(ix)
        ctx.close()
    print("quantile sanitizer smoke ok")


if __name__ == "__main__":
    main()
