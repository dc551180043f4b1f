"""CPU-only: the C-ABI library loads and exports every symbol include/b200promql.h declares."""
import ctypes
import os
import re

import pytest

from greptimedb_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "b200promql.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b2p_[a-z0-9_]+)\s*\(", src)))


def test_header_and_binding_agree():
    assert _declared_symbols() == sorted(_lib.EXPORTED_SYMBOLS)


def test_library_exports_every_declared_symbol():
    if not os.path.exists(_lib.LIB_PATH):
        pytest.fail(f"{_lib.LIB_PATH} not built — run __graft_entry__.build()")
    L = ctypes.CDLL(_lib.LIB_PATH)
    for name in _declared_symbols():
        assert hasattr(L, name), f"symbol {name} missing from libb200promql.so"
    _lib.load()  # signatures bind


def test_pure_host_entry_points():
    L = _lib.load()
    assert L.b2p_num_steps(0, 310_000, 30_000) == 11
    assert L.b2p_num_steps(10, 0, 5) == 0
    assert b"sm_90a" in L.b2p_version()


def test_params_struct_layout_matches_oracle():
    from oracle import oracle as orc
    assert ctypes.sizeof(_lib.RangeParams) == ctypes.sizeof(orc.Params) == 64
    for (n1, _), (n2, _) in zip(_lib.RangeParams._fields_, orc.Params._fields_):
        assert n1 == n2


def test_no_cpu_fallback_without_device():
    """On a box without a GPU the product must fail loudly instead of computing on the CPU."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from greptimedb_b200 import B2PError, Context
    with pytest.raises(B2PError) as ei:
        Context(0)
    assert "no CPU fallback" in str(ei.value) or "CUDA" in str(ei.value)


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "greptimedb_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h")):
                txt = open(os.path.join(dp, f)).read()
                assert "oracle/" not in txt.replace("oracle/promql_oracle.c:orc_synth_fill", "") or f.endswith(".cuh"), f
                assert "import oracle" not in txt and "from oracle" not in txt, f


def test_rust_shim_layout_assertions_compile():
    """rust-shim/tests/layout.c static-asserts every layout rust-shim/src/ffi.rs assumes about the header."""
    import subprocess
    subprocess.check_call(["gcc", "-std=c11", "-fsyntax-only", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "rust-shim", "tests", "layout.c")])


def test_rust_ffi_declares_every_header_symbol():
    src = open(os.path.join(ROOT, "rust-shim", "src", "ffi.rs")).read()
    declared = set(re.findall(r"pub fn (b2p_[a-z0-9_]+)\s*\(", src))
    assert sorted(declared) == _declared_symbols()


def test_host_scan_series_divides_and_describes_regular_series():
    """b2p_host_scan_series (no device work): SeriesDivide's boundaries on the host plus, per series, (first timestamp,
    cadence) and whether ts[i] == t0 + i * cadence for every row — what b2p_range_eval sends instead of the timestamp
    and id columns when it holds."""
    import ctypes as C
    import numpy as np
    from greptimedb_b200 import _lib
    L = _lib.load()

    def scan(ts, sid, offs, n_series, base=0):
        ts = np.ascontiguousarray(ts, np.int64)
        out = np.zeros(n_series + 1, np.uint64)
        t0 = np.zeros(n_series, np.int64)
        cad = np.zeros(n_series, np.int64)
        reg = C.c_int32(-1)
        p = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
        sid = None if sid is None else np.ascontiguousarray(sid, np.uint32)
        offs = None if offs is None else np.ascontiguousarray(offs, np.uint64)
        rc = L.b2p_host_scan_series(p(ts), p(sid), p(offs), ts.size, n_series, base, p(out), p(t0), p(cad), C.addressof(reg))
        return rc, out, t0, cad, reg.value

    # series 5 (3 rows), 6 (empty), 7 (1 row), 8 (4 rows, step 0: duplicate timestamps), 9 (2 rows); ids start at 5
    ts = np.array([100, 115, 130, 7, 50, 50, 50, 50, -3, 9], np.int64)
    sid = np.array([5, 5, 5, 7, 8, 8, 8, 8, 9, 9], np.uint32)
    rc, off, t0, cad, reg = scan(ts, sid, None, 5, base=5)
    assert rc == 0 and off.tolist() == [0, 3, 3, 4, 8, 10]
    assert t0.tolist() == [100, 0, 7, 50, -3] and cad.tolist() == [15, 0, 0, 0, 12] and reg == 1
    # the same through offsets (rebased to the batch), one row off the cadence
    ts2 = ts.copy(); ts2[2] += 1
    rc, off2, _, cad2, reg2 = scan(ts2, None, np.array([40, 43, 43, 44, 48, 50], np.uint64), 5)
    assert rc == 0 and off2.tolist() == off.tolist() and cad2.tolist() == cad.tolist() and reg2 == 0
    # ids out of order / out of range are errors (B2P_E_UNSORTED = -3)
    assert scan(ts, np.array([5, 5, 6, 5, 8, 8, 8, 8, 9, 9]), None, 5, base=5)[0] == -3
    assert scan(ts, sid, None, 4, base=5)[0] == -3
    assert scan(ts, sid, None, 5, base=6)[0] == -3


def test_host_scan_series_on_the_reference_series_divide_fixture():
    """series_divide.rs:668-905 through the library's host-side SeriesDivide: the same 7 boundaries."""
    import ctypes as C
    import numpy as np
    from greptimedb_b200 import _lib
    from tests.helpers import load_unit
    from tests.test_oracle_golden import _series_divide_ids
    g = load_unit()["series_divide"]
    _, ids = _series_divide_ids(g)
    ts = np.array([t for b in g["batches"] for t in b["ts"]], np.int64)
    out = np.zeros(8, np.uint64)
    reg = C.c_int32(-1)
    L = _lib.load()
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    assert L.b2p_host_scan_series(p(ts), p(ids), None, ts.size, 7, 0, p(out), None, None, C.addressof(reg)) == 0
    assert out.tolist() == g["expected_offsets"] and reg.value == 1   # (its timestamps are 1 s apart throughout)
