"""One small topk / bottomk call per path of K10 (b2p_topk.cuh), for a compute-sanitizer run on a GPU machine:

    compute-sanitizer --tool memcheck  python tests/topk_sanitizer_smoke.py
    compute-sanitizer --tool racecheck python tests/topk_sanitizer_smoke.py

Paths: the fast path with single-chunk groups, the fast path with a group of several chunks (candidate lists, merge,
mark), the general path (k > 32) with both kinds of group, the copy (k >= the largest group), k < 1, and rows whose
group id is out of range.  Each result is checked against the dense oracle."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch

    from greptimedb_b200 import Context
    from tests import topk_oracle as tko

    rng = np.random.default_rng(11)
    T = 65
    gid = np.concatenate([np.zeros(700, np.uint32), np.full(100, 1, np.uint32), np.full(5, 2, np.uint32),
                          np.full(3, 9, np.uint32)])   # several chunks, one chunk, a small group, no group
    R = gid.size
    vals = rng.standard_normal((R, T))
    vals[rng.random((R, T)) < 0.2] = 1.0
    valid = tko._words(rng.random((R, T)) < 0.8)
    tie = rng.permutation(R).astype(np.uint32)
    dev = torch.device("cuda:0")
    ctx = Context(0)
    d_vals = torch.from_numpy(vals).to(dev)
    d_valid = torch.from_numpy(valid.view(np.int32).copy()).to(dev)
    d_tie = torch.from_numpy(tie.view(np.int32)).to(dev)
    ix = ctx.group_index_create_dev(torch.from_numpy(gid.view(np.int32)).to(dev), R, 3)
    for op, k in [("topk", 3), ("bottomk", 32), ("topk", 40), ("bottomk", 150), ("topk", 700), ("topk", 0.5)]:
        out = torch.zeros_like(d_valid)
        ctx.topk_dev(op, k, d_vals, d_valid, ix, d_tie, T, out)
        ctx.sync()
        exp = tko.topk(op == "bottomk", k, vals, valid, gid, 3, tie)
        assert (out.cpu().numpy().view(np.uint32) == exp).all(), (op, k)
    ctx.group_index_destroy(ix)
    ctx.close()
    print("topk sanitizer smoke ok")


if __name__ == "__main__":
    main()
