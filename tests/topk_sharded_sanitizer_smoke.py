"""One small sharded topk / bottomk per path (b2p_topk_shard_* over three simulated ranks, one context each), for a
compute-sanitizer run on a GPU machine:

    compute-sanitizer --tool memcheck  python tests/topk_sharded_sanitizer_smoke.py
    compute-sanitizer --tool racecheck python tests/topk_sharded_sanitizer_smoke.py

Paths: the exchange with one round (k <= 32) and with rounds (k > 32), a group of several chunks on one rank, a rank
with no rows, the copy (k >= the largest group), k < 1, and rows whose group id is out of range.  Each union of kept
cells is checked against select_keys.topk."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    from tests import select_keys as sk
    from tests.test_gpu_topk_sharded import Rank, ranks_of, run_sharded

    rng = np.random.default_rng(11)
    T = 65
    gid = np.concatenate([np.zeros(700, np.uint32), np.full(100, 1, np.uint32), np.full(5, 2, np.uint32),
                          np.full(3, 9, np.uint32)])
    R = gid.size
    vals = rng.standard_normal((R, T))
    vals[rng.random((R, T)) < 0.2] = 1.0
    ok = rng.random((R, T)) < 0.8
    tie = rng.permutation(R).astype(np.uint32)
    own = np.where(np.arange(R) < 650, 0, 1)          # rank 0 holds most of group 0; rank 2 holds nothing
    ranks = [Rank(np.flatnonzero(own == r), vals, sk.words(ok), gid, 3, tie) for r in range(3)]
    sizes = np.bincount(gid[gid < 3], minlength=3).astype(np.uint32)
    for op, k in [("topk", 3), ("bottomk", 32), ("topk", 40), ("bottomk", 150), ("topk", 700), ("topk", 0.5)]:
        outs, _, _ = run_sharded(ranks, op, k, sizes, T)
        union = np.zeros((R, (T + 31) // 32), np.uint32)
        for r, out in zip(ranks, outs):
            union[r.rows] = out
        assert (union == sk.words(sk.topk(op == "bottomk", ranks_of(k), vals, ok, gid, 3, tie))).all(), (op, k)
    for r in ranks:
        r.close()
    print("topk sharded sanitizer smoke ok")


if __name__ == "__main__":
    main()
