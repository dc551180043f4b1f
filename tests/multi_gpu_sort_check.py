"""Multi-rank check of the sharded sort over the library's communicator (run under torchrun, one rank per GPU; started
by tests/test_multi_gpu.py when at least two GPUs are visible): every rank regenerates the same grid from a seed
(the total-order specials, T = 1 and T = 37, and two fields), keeps the rows distributed.shard_rows gives it with their
global row ids, counts its cells, and runs b2p_sort_cells_allgather_dev in both directions; every rank's cells and
values == b2p_sort_cells_dev (_fields_dev) over all rows on its own GPU, bit for bit.  torch.distributed only carries
the 128-byte communicator id and the verdict."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests.ranks import rank_session  # noqa: E402


def main(s):
    rank, world, dev, ctx = s.rank, s.world, s.dev, s.ctx
    from greptimedb_b200 import distributed as D
    from tests import select_keys as sk
    from tests.test_sort_oracle import TOTAL_ORDER
    bad = []
    for R, T, F in ((200_000, 1, 1), (3000, 37, 1), (3000, 37, 2)):
        rng = np.random.default_rng(R + T + F)
        grids = [np.array(TOTAL_ORDER)[rng.integers(0, len(TOTAL_ORDER), (R, T))] for _ in range(F)]
        ok = rng.random((R, T)) < 0.8
        _, rows, _ = D.shard_rows(np.arange(R + 1, dtype=np.uint64), world, rank)
        n = max(rows.size, 1)
        pad = lambda a: torch.from_numpy(np.concatenate([a[rows], np.zeros((n - rows.size,) + a.shape[1:], a.dtype)])).to(dev)
        valid = pad(sk.words(ok).view(np.int32))
        vals = [pad(g) for g in grids]
        row_id = pad(np.arange(R, dtype=np.int32))
        all_valid = torch.from_numpy(sk.words(ok).view(np.int32)).to(dev)
        all_vals = [torch.from_numpy(g).to(dev) for g in grids]
        torch.cuda.synchronize()
        counts = ctx.sort_shard_counts_dev(valid, rows.size, T, world)
        N = int(counts.sum())
        for desc in (False, True):
            cells = torch.full((max(N, 1),), -1, dtype=torch.int64, device=dev)
            outs = [torch.zeros(max(N, 1), dtype=torch.float64, device=dev) for _ in range(F)]
            ctx.sort_cells_allgather_dev(desc, vals if F > 1 else vals[0], valid, row_id, rows.size, T, counts, cells,
                                         outs if F > 1 else outs[0])
            sent = ctx.last_exchange_bytes()
            exp = torch.full((R * T,), -1, dtype=torch.int64, device=dev)
            en = torch.zeros(1, dtype=torch.int64, device=dev)
            if F > 1:
                ctx.sort_cells_fields_dev(desc, all_vals, all_valid, R, T, exp, en)
            else:
                ctx.sort_cells_dev(desc, all_vals[0], all_valid, R, T, exp, en)
            ctx.sync()
            torch.cuda.synchronize()
            e = exp.cpu().numpy()[:int(en.item())]
            got = cells.cpu().numpy()[:N]
            if N != int(ok.sum()) or not np.array_equal(got, e):
                bad.append(f"cells differ: R={R} T={T} F={F} desc={desc} rank={rank}")
                continue
            for f in range(F):
                if not np.array_equal(outs[f].cpu().numpy()[:N].view(np.uint64), grids[f].reshape(-1)[e].view(np.uint64)):
                    bad.append(f"values differ: R={R} T={T} F={F} desc={desc} field {f} rank={rank}")
            if sent != int(counts[rank]) * 8 * (F + 1):
                bad.append(f"exchange bytes {sent} on rank {rank}")
    return bad


if __name__ == "__main__":
    rank_session("MULTI_GPU_SORT_CHECK", main)
