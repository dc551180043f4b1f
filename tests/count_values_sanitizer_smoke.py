"""One small count_values call per path of K12 (b2p_count_values.cuh), for a compute-sanitizer run on a GPU machine:

    compute-sanitizer --tool memcheck  python tests/count_values_sanitizer_smoke.py
    compute-sanitizer --tool racecheck python tests/count_values_sanitizer_smoke.py
    compute-sanitizer --tool initcheck python tests/count_values_sanitizer_smoke.py

Paths: groups of every size in one batch (the member-group, segment, scatter, head, rank and count kernels around CUB's
segmented sort and scan), with empty groups, invalid cells and rows of no group; and a call whose rows all lie outside
the groups (the rows are only cleared).  A batch of more groups or a window of fewer steps runs the same kernels.  Each
call's launch count shows that it took its path, and each result is checked against the dense oracle."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch

    from greptimedb_b200 import Context
    from tests import binary_oracle as bor
    from tests import count_values_oracle as cvo

    rng = np.random.default_rng(12)
    T = 65
    # launches of the call: the member-group kernel, then per batch five kernels (CUB's are not counted); none when no
    # row is in a group
    for sizes, n_groups, launches in [([5, 64, 0, 2, 300, 1], 6, 6), ([4, 3], 0, 0)]:
        gid = np.concatenate([np.full(s, g, np.uint32) for g, s in enumerate(sizes)] + [np.full(3, 99, np.uint32)])
        R = gid.size
        vals = rng.choice(np.array([1.0, -0.0, 0.0, np.nan, 2.5]), (R, T))
        vals[rng.random((R, T)) < 0.3] = rng.standard_normal(1)[0]
        valid = bor._words(rng.random((R, T)) < 0.8)
        dev = torch.device("cuda:0")
        ctx = Context(0)
        d_vals = torch.from_numpy(vals).to(dev)
        d_valid = torch.from_numpy(valid.view(np.int32).copy()).to(dev)
        ix = ctx.group_index_create_dev(torch.from_numpy(gid.view(np.int32)).to(dev), R, n_groups)
        out = torch.zeros((R, T), dtype=torch.float64, device=dev)
        cnt = torch.zeros((R, T), dtype=torch.int32, device=dev)
        before = ctx.launch_count()
        ctx.count_values_dev(d_vals, d_valid, ix, T, out, cnt)
        ctx.sync()
        assert ctx.launch_count() - before == launches, (sizes, ctx.launch_count() - before)
        exp, ecnt = cvo.count_values(vals, valid, gid, n_groups)
        assert (cnt.cpu().numpy().view(np.uint32) == ecnt).all(), sizes
        assert (out.cpu().numpy().view(np.uint64) == exp.view(np.uint64)).all(), sizes
        ctx.group_index_destroy(ix)
        ctx.close()
    print("count_values sanitizer smoke ok")


if __name__ == "__main__":
    main()
