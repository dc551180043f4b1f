"""One small absent() call per path of K15 (b2p_absent.cuh), for a compute-sanitizer run on a GPU machine:

    compute-sanitizer --tool memcheck  python tests/absent_sanitizer_smoke.py
    compute-sanitizer --tool racecheck python tests/absent_sanitizer_smoke.py

Paths: words shared by the threads of a CTA (Tw < 256: the shared-memory fold), with stray bits past T; one word per
thread (Tw >= 256, fewer words than threads); word columns that a thread walks row by row (more words than threads in
the grid); a grid with no row (the OR pass is skipped); all of them through the device form, and the first through the
host-pointer form.  Each result is checked against the numpy OR."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch

    from greptimedb_b200 import Context
    from tests import absent_oracle as ao
    from tests.binary_oracle import _words

    rng = np.random.default_rng(15)
    ctx = Context(0)
    # (rows, T): Tw = 2 (shared words); Tw = 300 over 6 CTAs (one word per thread); Tw = 9000 over 18 CTAs (a thread
    # walks word columns); no row
    for rows, T in ((37, 45), (20, 9600), (2, 288_000), (0, 70)):
        ok = rng.random((rows, T)) < 0.01
        valid = _words(ok)
        if T % 32 and rows:
            valid[:, -1] |= np.uint32(0xFFFFFFFF) << np.uint32(T % 32)  # stray bits past T
        e_out, e_words = ao.absent_words(ok, T)
        Tw = (T + 31) // 32
        out = torch.zeros(T, dtype=torch.float64, device="cuda")
        ov = torch.zeros(Tw, dtype=torch.int32, device="cuda")
        d_valid = torch.from_numpy(valid.view(np.int32)).cuda() if rows else None
        ctx.absent_dev(d_valid, rows, T, out, ov)
        ctx.sync()
        assert out.cpu().numpy().tolist() == e_out.tolist()
        assert ov.cpu().numpy().view(np.uint32).tolist() == e_words.tolist()
        if rows == 37:
            h_out, h_words = ctx.absent(valid, T)
            assert h_out.tolist() == e_out.tolist() and h_words.tolist() == e_words.tolist()
    ctx.close()
    print("absent sanitizer smoke ok")


if __name__ == "__main__":
    main()
