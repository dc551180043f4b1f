"""One small call per path of the multi-key sort (b2p_sort_cells_fields[_dev]; sort_rekey_kernel in b2p_sort.cuh), for
a compute-sanitizer run on a GPU machine:

    compute-sanitizer --tool memcheck  python tests/multifield_plan_sanitizer_smoke.py
    compute-sanitizer --tool racecheck python tests/multifield_plan_sanitizer_smoke.py
    compute-sanitizer --tool initcheck python tests/multifield_plan_sanitizer_smoke.py

Paths: F = 1 (the scatter and one radix sort), 2 and 8 (one rekey and radix sort per earlier field) over a grid with
holes, special values and stray bits past T in each row's last validity word, ascending and descending, through the
device form and the host-pointer form; an all-valid grid; an all-invalid grid (no cell: nothing is sorted).  Each result
is checked against tests/multifield_plan_oracle.py."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch

    from greptimedb_b200 import Context
    from tests import multifield_plan_oracle as mp
    from tests.select_keys import words

    rng = np.random.default_rng(16)
    R, T = 5, 45
    ctx = Context(0)
    for F in (1, 2, 8):
        vals = rng.choice([0.0, -0.0, 1.0, np.inf, -np.inf, np.nan], (F, R, T))
        for ok in (rng.random((R, T)) < 0.7, np.ones((R, T), bool)):
            valid = words(ok)
            valid[:, -1] |= np.uint32(0xFFFFFFFF) << np.uint32(T % 32)  # stray bits past T
            d_vals = [torch.from_numpy(np.ascontiguousarray(v)).cuda() for v in vals]
            d_valid = torch.from_numpy(valid.view(np.int32)).cuda()
            for desc in (False, True):
                cells = torch.zeros(R * T, dtype=torch.int64, device="cuda")
                n = torch.zeros(1, dtype=torch.int64, device="cuda")
                ctx.sort_cells_fields_dev(desc, d_vals, d_valid, R, T, cells, n)
                ctx.sync()
                got = cells[: int(n.item())].cpu().numpy().view(np.uint64)
                assert got.tolist() == mp.sort(desc, vals, ok).tolist()
                assert ctx.sort_cells_fields(desc, vals, valid).tolist() == got.tolist()
        assert ctx.sort_cells_fields(False, vals, np.zeros((R, (T + 31) // 32), np.uint32)).size == 0
    ctx.close()
    print("multi-field sort sanitizer smoke ok")


if __name__ == "__main__":
    main()
