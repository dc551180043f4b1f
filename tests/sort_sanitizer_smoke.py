"""One small sort call per path of K14 (b2p_sort.cuh), for a compute-sanitizer run on a GPU machine:

    compute-sanitizer --tool memcheck  python tests/sort_sanitizer_smoke.py
    compute-sanitizer --tool racecheck python tests/sort_sanitizer_smoke.py

Paths: a grid with holes, an empty row, special values and a T that is not a multiple of 32, with stray bits past T in
each row's last validity word (K13's count kernel, CUB's scan, the scatter, CUB's radix sort), ascending and
descending, through the device form and the host-pointer form; an all-invalid grid (no cell: the sort is skipped);
a grid with no row.  Each result is checked against the oracle."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch

    from greptimedb_b200 import Context
    from tests import sort_oracle as so
    from tests.binary_oracle import _words

    rng = np.random.default_rng(14)
    R, T = 5, 45
    ok = rng.random((R, T)) < 0.7
    ok[1] = False
    vals = rng.integers(0, 4, (R, T)).astype(np.float64)
    vals[2, ::3] = np.nan
    vals[3, ::4] = -0.0
    valid = _words(ok)
    valid[:, -1] |= np.uint32(0xFFFFFFFF) << np.uint32(T % 32)  # stray bits past T
    ctx = Context(0)
    d_vals = torch.from_numpy(vals).cuda()
    d_valid = torch.from_numpy(valid.view(np.int32)).cuda()
    for desc in (False, True):
        cells = torch.zeros(R * T, dtype=torch.int64, device="cuda")
        n = torch.zeros(1, dtype=torch.int64, device="cuda")
        ctx.sort_cells_dev(desc, d_vals, d_valid, R, T, cells, n)
        ctx.sync()
        got = cells[: int(n.item())].cpu().numpy().view(np.uint64)
        assert got.tolist() == so.value_order(vals, ok, desc).tolist()
        assert ctx.sort_cells(desc, vals, valid).tolist() == got.tolist()
    assert ctx.sort_cells(False, vals, np.zeros_like(valid)).size == 0
    assert ctx.sort_cells(True, np.zeros((0, T)), np.zeros((0, (T + 31) // 32), np.uint32)).size == 0
    ctx.close()
    print("sort sanitizer smoke ok")


if __name__ == "__main__":
    main()
