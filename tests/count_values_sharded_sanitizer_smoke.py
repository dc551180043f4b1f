"""One small sharded count_values per path (b2p_count_values_shard_* over three simulated ranks, one context each, and
the composed call over one rank), for a compute-sanitizer run on a GPU machine:

    compute-sanitizer --tool memcheck  python tests/count_values_sharded_sanitizer_smoke.py
    compute-sanitizer --tool racecheck python tests/count_values_sharded_sanitizer_smoke.py

Paths: a group on one rank only, a rank with no rows, groups without members, rows whose group id is out of range, a
step count that is not a multiple of 32, the largest positive NaN beside fillers, the Int64 form, and batches under a
small exchange cap.  Each rank's result is checked against b2p_count_values_dev over all rows."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    from tests import select_keys as sk
    from tests.test_gpu_count_values_sharded import MAX_NAN, Rank, check_case, composed_check

    rng = np.random.default_rng(11)
    T = 65
    gid = np.concatenate([np.zeros(300, np.uint32), np.full(100, 1, np.uint32), np.full(5, 2, np.uint32),
                          np.full(3, 9, np.uint32)])
    R = gid.size
    vals = rng.integers(0, 40, (R, T)).astype(np.float64)
    top = rng.random((R, T)) < 0.05
    ivals = vals.astype(np.int64)
    ivals[top] = np.iinfo(np.int64).max                # the filler's key in both forms
    vals[top] = np.uint64(MAX_NAN).view(np.float64)
    ok = rng.random((R, T)) < 0.8
    own = np.where(np.arange(R) < 250, 0, 1)          # rank 0 holds most of group 0; rank 2 holds nothing
    for i64 in (False, True):
        v = ivals if i64 else vals
        valid = sk.words(ok)
        ranks = [Rank(np.flatnonzero(own == r), v, valid, gid, 4, T, i64) for r in range(3)]
        full = Rank(np.arange(R), v, valid, gid, 4, T, i64)
        check_case(ranks, full, v, ok, gid, 4, T)
        composed_check(full, v, ok, gid, 4, T)
        for r in ranks + [full]:
            r.close()
    os.environ["B2P_TOPK_EXCHANGE_BYTES"] = str(32 << 10)
    ranks = [Rank(np.flatnonzero(own == r), vals, sk.words(ok), gid, 4, T) for r in range(3)]
    full = Rank(np.arange(R), vals, sk.words(ok), gid, 4, T)
    _, plan, _ = check_case(ranks, full, vals, ok, gid, 4, T)
    assert plan["n_batches"] > 1
    for r in ranks + [full]:
        r.close()
    print("count_values sharded sanitizer smoke ok")


if __name__ == "__main__":
    main()
