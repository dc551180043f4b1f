"""CPU checks of bench.py's contract pieces that do not need a GPU: --dump-outputs writes the validity bit words as a
0/1 grid and invalid cells as 0.0 from a fixed row sample, and the reference arm (--impl reference: the oracle port
timed on the host cores) prints one JSON line with the keys a reader of the result expects."""
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_dump_outputs_grid_unpacks_validity_words_and_samples_rows_reproducibly(tmp_path):
    sys.path.insert(0, ROOT)
    import bench
    R, T = 5, 40
    Tw = (T + 31) // 32
    vals = np.arange(R * T, dtype=np.float64).reshape(R, T)
    vals[:, 5] = np.nan   # what an invalid cell may hold in the library's output
    words = np.zeros((R, Tw), np.uint32)
    words[:, 0] = 0x80000001   # steps 0 and 31
    words[:, 1] = 0x00000080   # step 39
    rows = bench.Dump.rows(R, 3, 7)
    assert rows.tolist() == bench.Dump.rows(R, 3, 7).tolist() and len(set(rows.tolist())) == 3
    d = bench.Dump(str(tmp_path / "out"))
    d.grid("g", vals, words.view(np.int32), T, rows)
    v, ok = np.load(tmp_path / "out" / "g.npy"), np.load(tmp_path / "out" / "g_valid.npy")
    assert v.dtype == np.float64 and ok.dtype == np.float32 and v.shape == ok.shape == (3, T)
    assert (np.flatnonzero(ok[0]) == [0, 31, 39]).all() and (ok == ok[0]).all()
    assert (v[:, [0, 31, 39]] == vals[rows][:, [0, 31, 39]]).all() and (v[:, 1:31] == 0.0).all() and np.isfinite(v).all()
    bench.Dump(None).save("x", vals)   # without --dump-outputs nothing is written


def test_reference_arm_prints_one_contract_line():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "0"],
                         capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-2000:]
    lines = [l for l in out.stdout.strip().splitlines() if l.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["unit"] == "samples/s" and d["higher_is_better"] is True
    assert d["value"] > 0 and d["steps"] == 1
    assert d["cpu_baseline"]["kind"] == "port" and d["cpu_baseline"]["cores"] >= 1
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["e2e"]["d2h_bytes_per_step"] == 0
    assert d["config"]["workload"]
