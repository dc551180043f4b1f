"""One small sharded quantile per path (b2p_quantile_shard_* over three simulated ranks, one context each), for a
compute-sanitizer run on a GPU machine:

    compute-sanitizer --tool memcheck  python tests/quantile_sharded_sanitizer_smoke.py
    compute-sanitizer --tool racecheck python tests/quantile_sharded_sanitizer_smoke.py

Paths: digit passes and the extreme pass, a group of several chunks on one rank, a group on one rank only, a rank with
no rows, groups without members, rows whose group id is out of range, a step count that is not a multiple of 32, and
phi outside [0, 1] (one counting pass).  Each rank's result is checked against b2p_group_quantile_dev."""
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    from tests import select_keys as sk
    from tests.test_gpu_quantile_sharded import Rank, run_sharded, single_rank

    rng = np.random.default_rng(11)
    T = 65
    gid = np.concatenate([np.zeros(700, np.uint32), np.full(100, 1, np.uint32), np.full(5, 2, np.uint32),
                          np.full(3, 9, np.uint32)])
    R = gid.size
    vals = rng.standard_normal((R, T))
    vals[rng.random((R, T)) < 0.2] = 1.0
    ok = rng.random((R, T)) < 0.8
    own = np.where(np.arange(R) < 650, 0, 1)          # rank 0 holds most of group 0; rank 2 holds nothing
    ranks = [Rank(np.flatnonzero(own == r), vals, sk.words(ok), gid, 4) for r in range(3)]
    full = Rank(np.arange(R), vals, sk.words(ok), gid, 4)
    for phi in (0.0, 0.5, 0.99, 1.0, math.nan):
        outs, _, _, _ = run_sharded(ranks, phi, 4, T)
        one, one_cnt = single_rank(full, phi, 4, T)
        for out, cnt in outs:
            assert sk.same_bits(out, one) and (cnt == one_cnt).all(), phi
    for r in ranks + [full]:
        r.close()
    print("quantile sharded sanitizer smoke ok")


if __name__ == "__main__":
    main()
