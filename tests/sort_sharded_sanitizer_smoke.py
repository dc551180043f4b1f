"""One small sharded sort per path (b2p_sort_shard_* over three simulated ranks, one context each, and the composed
call over one rank), for a compute-sanitizer run on a GPU machine:

    compute-sanitizer --tool memcheck  python tests/sort_sharded_sanitizer_smoke.py
    compute-sanitizer --tool racecheck python tests/sort_sharded_sanitizer_smoke.py

Paths: a rank with no rows, a step count that is not a multiple of 32 with bits past it set, one, two and three
merge rounds, two fields (the general merge), and the Int64 form.  Each result is checked against b2p_sort_cells_dev
over all rows."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    from tests.test_gpu_sort_sharded import check, composed, hashed, specials

    vals, ok = specials(3000, 37, 1)
    for n_ranks in (1, 2, 3, 5):
        check(True, hashed(3000, n_ranks), n_ranks, [vals], ok, 37)
    check(False, hashed(3000, 3), 3, [vals, specials(3000, 37, 2)[0]], ok, 37)
    iv = np.random.default_rng(3).integers(-5, 5, (3000, 37)).astype(np.int64)
    check(False, hashed(3000, 3), 3, [iv], ok, 37, i64=True)
    composed(False, [vals], ok, 37)
    print("sort sharded sanitizer smoke ok")


if __name__ == "__main__":
    main()
