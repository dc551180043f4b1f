"""GPU: the dense-grid kernels at their layout edges on every route, bit for bit against the references of
tests/grid_edges.py:
  K7   binary_op_kernel (vector-vector, scalar left / right; in place and out of place) and count_valid_kernel;
  K8   setop_copy / mask / dedupe / key_check (`and`, `or`, `unless`; `and` / `unless` in place);
  K9   instant_fn_kernel over the exact functions and unary minus (in place with out_valid == valid, and out of place),
       scalar_reduce / scalar_write, i64_to_f64;
  K13  subquery_count / scatter, seen through last_over_time and count_over_time windows;
  K15  absent_or / absent_write in each of its three OR regimes;
  K18  valid_and_kernel under a multi-field range call;
  K19  step_fn_kernel over its CTA geometries, against a calendar that does not share the kernel's algorithm.
Routes: the host form and the `_dev` form; the 128-bit variants of K7 / K8 / K9 (T even, 16-byte aligned pointers),
and their scalar variants by T odd or by an output (and input) pointer 8 bytes off.  Every `_dev` output starts filled
with a NaN sentinel and carries a guard tail of 128 cells and 4 validity words, which must be untouched afterwards.
Validity words are compared exactly; bits past T must be zero wherever the header promises it (all but K9, whose
words are copied through, junk included).  Sizes that force a second grid-stride pass are computed from the device's
SM count and each launcher's capped_grid arguments (b2p_elementwise.cu, b2p_range.cu)."""
import numpy as np
import pytest

from tests import grid_edges as ge
from tests.ulp_bounds import POW_ATAN2_ULPS

pytestmark = pytest.mark.gpu

GUARD_CELLS, GUARD_WORDS = 128, 4
SENTINEL = np.uint64(0x7FF4_5E47_1E17_0001)  # a NaN no kernel computes
WORD_SENTINEL = np.uint32(0xA5A5_5A5A)
CASES = ge.grid_cases()
BY_T = {T: [c for c in CASES if c["T"] == T] for T in ge.T_LIST}
BIN_OPS = [("+", False), ("^", False), (">", False), ("==", True)]
SCALARS = [0.5, -0.0]


@pytest.fixture(scope="module")
def ctx():
    from greptimedb_b200 import Context
    c = Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def bits(x):
    return np.ascontiguousarray(x, np.float64).view(np.uint64)


def total_key(x):
    return ge.total_key(x)


class Slab:
    """A device buffer of n items (f64 cells, u32 words, i64 / u32 inputs) `off` items in, filled with the sentinel
    before and after (the guard tail), or with `data` in its body.  ptr is the body's address."""

    def __init__(self, n, kind, off=0, data=None):
        import torch
        self.kind, self.n, self.off = kind, n, off
        guard = GUARD_CELLS if kind in ("f64", "i64") else GUARD_WORDS
        if kind in ("f64", "i64"):
            host = np.full(off + n + guard, SENTINEL, np.uint64).view(np.int64)
        else:
            host = np.full(off + n + guard, WORD_SENTINEL, np.uint32).view(np.int32)
        if data is not None:
            host[off:off + n] = np.ascontiguousarray(data).reshape(-1).view(host.dtype)
        self.t = torch.from_numpy(host).cuda()
        self.ptr = self.t.data_ptr() + off * host.itemsize

    def read(self):
        h = self.t.cpu().numpy()
        return h.view(np.uint64 if self.kind in ("f64", "i64") else np.uint32)

    def body(self):
        b = self.read()[self.off:self.off + self.n]
        return b.view(np.float64) if self.kind == "f64" else b

    def assert_guards(self, what):
        h = self.read()
        s = SENTINEL if self.kind in ("f64", "i64") else WORD_SENTINEL
        assert (h[:self.off] == s).all() and (h[self.off + self.n:] == s).all(), f"{what}: a write outside the output"


def launches(ctx, f):
    n0 = ctx.launch_count()
    f()
    ctx.sync()
    return ctx.launch_count() - n0


def check_cells(got, gv, exp, ev, arith_nan=False, ulp_bound=None):
    """validity words exactly; invalid cells 0.0; values by bits (arith_nan: a NaN that arithmetic produced counts as
    a NaN; ulp_bound: cells off the special values within that many ulps)"""
    assert (np.asarray(gv, np.uint32) == np.asarray(ev, np.uint32)).all(), "validity words differ"
    T = got.shape[-1]
    ok = ge.ok_of(np.asarray(ev, np.uint32).reshape(got.shape[0], -1), T)
    assert (bits(got[~ok]) == 0).all(), "an invalid cell does not hold 0.0"
    g, e = got[ok], exp[ok]
    if arith_nan:
        assert (np.isnan(g) == np.isnan(e)).all(), "NaN where the reference has none, or the reverse"
        keep = ~np.isnan(e)
        g, e = g[keep], e[keep]
    if ulp_bound is not None:
        exact = ~np.isfinite(e) | (e == 0) | (np.abs(e) == 1.0)
        assert (bits(g[exact]) == bits(e[exact])).all(), "a special case differs"
        assert np.abs(total_key(g) - total_key(e)).max(initial=0) <= ulp_bound
        return
    assert (bits(g) == bits(e)).all(), "a cell differs from the reference"


# ---- K7 -------------------------------------------------------------------------------------------------------------------
def bin_expect(op, rb, form, lhs, lok, rhs, rok, lrow, rrow, s):
    if form == "vector":
        x, y = lhs[lrow], rhs[rrow]
        return ge.binary_ref(op, x, y, lok[lrow] & rok[rrow], x, rb)
    x, y = (np.full_like(lhs, s), lhs) if form == "left" else (lhs, np.full_like(lhs, s))
    return ge.binary_ref(op, x, y, lok, lhs, rb)


def bin_check(op, got, gv, exp, ev):
    arith = op in ("+", "^")
    check_cells(got, gv, exp, ev, arith_nan=arith, ulp_bound=POW_ATAN2_ULPS if op == "^" else None)


@pytest.mark.parametrize("T", ge.T_LIST)
def test_k7_binary_every_route(ctx, T):
    Tw = (T + 31) // 32
    cases = BY_T[T]
    for i, c in enumerate(cases):
        other = cases[(i + 2) % len(cases)]
        lhs, lv, lok = c["vals"], c["valid"], c["ok"]
        rhs, rv, rok = other["vals"], other["valid"], other["ok"]
        L, R = lhs.shape[0], rhs.shape[0]
        lrow = np.array([0, 3, 1, 1, 2, 0], np.uint32)
        rrow = np.array([2, 0, 3, 1, 0, 0], np.uint32)
        P = lrow.size
        for op, rb in BIN_OPS:
            exp, ev = bin_expect(op, rb, "vector", lhs, lok, rhs, rok, lrow, rrow, None)
            got, gv = ctx.binary_op(op, lhs, lv, lrow, rhs, rv, rrow, return_bool=rb)
            bin_check(op, got, gv, exp, ev)
            for off in (0, 1):  # aligned: the 128-bit variant when T is even; 8 bytes off: the scalar variant
                dl, dlv = Slab(L * T, "f64", off, lhs), Slab(L * Tw, "u32", 0, lv)
                dr, drv = Slab(R * T, "f64", off, rhs), Slab(R * Tw, "u32", 0, rv)
                dlr, drr = Slab(P, "u32", 0, lrow), Slab(P, "u32", 0, rrow)
                out, ov = Slab(P * T, "f64", off), Slab(P * Tw, "u32", off)
                n = launches(ctx, lambda: ctx.binary_op_dev(op, dl.ptr, dlv.ptr, dlr.ptr, L, dr.ptr, drv.ptr, drr.ptr, R,
                                                            P, T, out.ptr, ov.ptr, return_bool=rb))
                assert n == 1
                out.assert_guards("K7 cells")
                ov.assert_guards("K7 words")
                bin_check(op, out.body().reshape(P, T), ov.body().reshape(P, Tw), exp, ev)
            for form in ("left", "right"):
                for s in SCALARS:
                    exp, ev = bin_expect(op, rb, form, lhs, lok, None, None, None, None, s)
                    got, gv = ctx.scalar_op(op, s, lhs, lv, scalar_on_left=form == "left", return_bool=rb)  # in place
                    bin_check(op, got, gv, exp, ev)
                    for off, in_place in ((0, False), (1, False), (0, True), (1, True)):
                        dv, dvv = Slab(L * T, "f64", off, lhs), Slab(L * Tw, "u32", off, lv)
                        out, ov = (dv, dvv) if in_place else (Slab(L * T, "f64", off), Slab(L * Tw, "u32", off))
                        n = launches(ctx, lambda: ctx.scalar_op_dev(op, s, dv.ptr, dvv.ptr, L, T, out.ptr, ov.ptr,
                                                                    scalar_on_left=form == "left", return_bool=rb))
                        assert n == 1
                        out.assert_guards("K7 scalar cells")
                        ov.assert_guards("K7 scalar words")
                        bin_check(op, out.body().reshape(L, T), ov.body().reshape(L, Tw), exp, ev)


@pytest.mark.parametrize("T,steps", [(1000, 64), (999, 32), (1000, 32)])
def test_k7_k9_second_grid_stride_pass(ctx, sms, T, steps):
    """more (row, tile) units than the capped grid has warps: 1000 steps on the 128-bit route, 999 on the scalar one,
    and 1000 steps 8 bytes off (scalar)"""
    rng = np.random.default_rng(T + steps)
    rows = ge.rows_past_warp_grid(sms, T, steps)
    assert rows * -(-T // steps) > sms * 16 * 8
    Tw = (T + 31) // 32
    ok = rng.random((rows, T)) < 0.7
    vals = np.where(ok, ge.VALID_FILL[rng.integers(0, ge.VALID_FILL.size, (rows, T))], ge.INVALID_FILL[0])
    valid = ge.add_junk(ge.words_of(ok), T, rng)
    off = 1 if (T % 2 == 0 and steps == 32) else 0
    dv, dvv = Slab(rows * T, "f64", off, vals), Slab(rows * Tw, "u32", off, valid)
    out, ov = Slab(rows * T, "f64", off), Slab(rows * Tw, "u32", off)
    assert launches(ctx, lambda: ctx.scalar_op_dev(">", 0.0, dv.ptr, dvv.ptr, rows, T, out.ptr, ov.ptr)) == 1
    out.assert_guards("K7 cells")
    ov.assert_guards("K7 words")
    exp, ev = ge.binary_ref(">", vals, 0.0, ok, vals)
    check_cells(out.body().reshape(rows, T), ov.body().reshape(rows, Tw), exp, ev)
    out2, ov2 = Slab(rows * T, "f64", off), Slab(rows * Tw, "u32", off)
    assert launches(ctx, lambda: ctx.instant_fn_dev("neg", dv.ptr, dvv.ptr, rows, T, out2.ptr, ov2.ptr)) == 1
    out2.assert_guards("K9 cells")
    ov2.assert_guards("K9 words")
    assert (bits(out2.body().reshape(rows, T)) == bits(ge.instant_fn_ref("neg", vals, ok))).all()
    assert (ov2.body().reshape(rows, Tw) == valid).all()


@pytest.mark.parametrize("T", [1, 31, 32, 33, 64, 65, 1000])
def test_count_valid_words(ctx, sms, T):
    rng = np.random.default_rng(T)
    Tw = (T + 31) // 32
    for rows in (1, 5, sms * 16 * 8 // Tw + 3):  # the last: more (row, word) units than the capped grid's warps
        cnt = rng.integers(0, 3, (rows, T)).astype(np.uint32)
        cnt[rng.random((rows, T)) < 0.1] = 0xFFFFFFFF
        dc = Slab(rows * T, "u32", 0, cnt)
        ov = Slab(rows * Tw, "u32", 0)
        assert launches(ctx, lambda: ctx.count_valid_words_dev(dc.ptr, rows, T, ov.ptr)) == 1
        ov.assert_guards("count_valid words")
        assert (ov.body().reshape(rows, Tw) == ge.count_valid_ref(cnt)).all()


# ---- K8 -------------------------------------------------------------------------------------------------------------------
SET_KEYS = {  # (lhs keys, rhs keys, n_keys): repeated keys, NO_KEY on either side, a key out of range on neither
    "and": ([0, ge.NO_KEY, 1, 0], [1, 0, 2, 1], 3),
    "unless": ([0, ge.NO_KEY, 1, 2], [1, 0, 2, 1], 3),
    "or": ([0, 1, ge.NO_KEY, 0], [1, 2, 0, ge.NO_KEY], 3),
}


@pytest.mark.parametrize("op", ["and", "or", "unless"])
@pytest.mark.parametrize("T", ge.T_LIST)
def test_k8_setop_every_route(ctx, op, T):
    Tw = (T + 31) // 32
    cases = BY_T[T]
    lk, rk, nk = np.array(SET_KEYS[op][0], np.uint32), np.array(SET_KEYS[op][1], np.uint32), SET_KEYS[op][2]
    for i, c in enumerate(cases):
        other = cases[(i + 1) % len(cases)]
        lhs, lv, lok = c["vals"], c["valid"], c["ok"]
        rhs, rv, rok = other["vals"], other["valid"], other["ok"]
        L, R = lhs.shape[0], rhs.shape[0]
        exp, ev = ge.setop_ref(op, lhs, lok, lk, rhs, rok, rk, nk)
        n_out = exp.shape[0]
        got, gv = ctx.setop(op, lhs, lv, lk, rhs, rv, rk, nk)
        check_cells(got, gv, exp, ev)
        routes = [(0, False), (1, False)] + ([(0, True), (1, True)] if op != "or" else [])
        for off, in_place in routes:
            dl, dlv = Slab(L * T, "f64", off, lhs), Slab(L * Tw, "u32", off, lv)
            dr, drv = Slab(R * T, "f64", off, rhs), Slab(R * Tw, "u32", 0, rv)
            dlk, drk = Slab(L, "u32", 0, lk), Slab(R, "u32", 0, rk)
            out, ov = (dl, dlv) if in_place else (Slab(n_out * T, "f64", off), Slab(n_out * Tw, "u32", off))
            ctx.setop_dev(op, dl.ptr, dlv.ptr, dlk.ptr, L, dr.ptr, drv.ptr, drk.ptr, R, nk, T, out.ptr, ov.ptr)
            ctx.sync()
            out.assert_guards("K8 cells")
            ov.assert_guards("K8 words")
            check_cells(out.body().reshape(n_out, T), ov.body().reshape(n_out, Tw), exp, ev)


@pytest.mark.parametrize("op", ["and", "or"])
def test_k8_second_grid_stride_pass(ctx, sms, op):
    rng = np.random.default_rng(8)
    for T, off in ((1000, 0), (1000, 1), (999, 0)):
        Tw = (T + 31) // 32
        rows = ge.rows_past_warp_grid(sms, T, 64 if (T % 2 == 0 and off == 0) else 32)
        lok, rok = rng.random((rows, T)) < 0.5, rng.random((rows, T)) < 0.5
        lhs = np.where(lok, ge.VALID_FILL[rng.integers(0, ge.VALID_FILL.size, (rows, T))], ge.INVALID_FILL[1])
        rhs = np.where(rok, -lhs, ge.INVALID_FILL[2])
        lv, rv = ge.add_junk(ge.words_of(lok), T, rng), ge.add_junk(ge.words_of(rok), T, rng)
        nk = rows // 3
        lk = rng.integers(0, nk, rows).astype(np.uint32)
        rk = rng.integers(0, nk, rows).astype(np.uint32)
        exp, ev = ge.setop_ref(op, lhs, lok, lk, rhs, rok, rk, nk)
        n_out = exp.shape[0]
        dl, dlv = Slab(rows * T, "f64", off, lhs), Slab(rows * Tw, "u32", off, lv)
        dr, drv = Slab(rows * T, "f64", off, rhs), Slab(rows * Tw, "u32", 0, rv)
        dlk, drk = Slab(rows, "u32", 0, lk), Slab(rows, "u32", 0, rk)
        out, ov = Slab(n_out * T, "f64", off), Slab(n_out * Tw, "u32", off)
        ctx.setop_dev(op, dl.ptr, dlv.ptr, dlk.ptr, rows, dr.ptr, drv.ptr, drk.ptr, rows, nk, T, out.ptr, ov.ptr)
        ctx.sync()
        out.assert_guards("K8 cells")
        ov.assert_guards("K8 words")
        check_cells(out.body().reshape(n_out, T), ov.body().reshape(n_out, Tw), exp, ev)


# ---- K9 -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T", ge.T_LIST)
def test_k9_instant_fn_every_route(ctx, T):
    Tw = (T + 31) // 32
    for c in BY_T[T]:
        vals, valid, ok = c["vals"], c["valid"], c["ok"]
        rows = vals.shape[0]
        for fn, (a0, a1, _, keeps_nan) in ge.INSTANT_FNS.items():
            exp = ge.instant_fn_ref(fn, vals, ok)
            ev = ge.words_of(ok)

            def same(got):
                if keeps_nan:
                    assert (bits(got) == bits(exp)).all(), fn
                else:
                    assert (np.isnan(got) == np.isnan(exp)).all() and \
                        (bits(got[~np.isnan(exp)]) == bits(exp[~np.isnan(exp)])).all(), fn
                assert (bits(got[~ok]) == 0).all(), fn

            got, gv = ctx.instant_fn(fn, vals, valid, a0, a1)  # in place on the device, out_valid == valid
            same(got)
            assert (gv == valid).all()
            for off, in_place in ((0, False), (1, False), (0, True), (1, True)):
                dv, dvv = Slab(rows * T, "f64", off, vals), Slab(rows * Tw, "u32", off, valid)
                out, ov = (dv, dvv) if in_place else (Slab(rows * T, "f64", off), Slab(rows * Tw, "u32", off))
                assert launches(ctx, lambda: ctx.instant_fn_dev(fn, dv.ptr, dvv.ptr, rows, T, out.ptr, ov.ptr,
                                                                a0, a1)) == 1
                out.assert_guards("K9 cells")
                ov.assert_guards("K9 words")
                same(out.body().reshape(rows, T))
                # out of place the words are copied, bits past T included; in place they are left as they were
                assert (ov.body().reshape(rows, Tw) == valid).all(), fn
                assert (ge.ok_of(ov.body(), T) == ok).all() and (ev == ge.words_of(ok)).all()


def test_i64_to_f64_rounding_and_grid_stride(ctx, sms):
    edges = ge.I64_EDGES
    assert (bits(ctx.i64_to_f64(edges)) == bits(ge.i64_to_f64_ref(edges))).all()
    rng = np.random.default_rng(64)
    n = sms * 16 * 256 + 7  # past the threads of the capped grid
    v = rng.integers(np.iinfo(np.int64).min, np.iinfo(np.int64).max, n, dtype=np.int64)
    v[1::7] = (v[1::7] >> 9) | 1  # odd values around 2^54: ties and near-ties
    v[:edges.size] = edges
    v[-edges.size:] = edges
    want = v.astype(np.float64)  # numpy's int64 -> f64 cast rounds to nearest, ties to even
    assert (bits(want[:edges.size]) == bits(ge.i64_to_f64_ref(edges))).all()
    for in_place in (False, True):
        dv = Slab(n, "i64", 0, v)
        out = dv if in_place else Slab(n, "f64", 0)
        assert launches(ctx, lambda: ctx._check(ctx._L.b2p_i64_to_f64_dev(ctx._h, dv.ptr, n, out.ptr))) == 1
        out.assert_guards("i64_to_f64")
        assert (out.read()[:n] == bits(want)).all()


# ---- scalar() --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", range(len(ge.scalar_cases())), ids=[c[0] + f"-T{c[1].shape[1]}"
                                                                       for c in ge.scalar_cases()])
def test_scalar_calculate_layouts(ctx, case):
    from greptimedb_b200 import B2PError
    name, vals, ok, valid, key, overlap = ge.scalar_cases()[case]
    rows, T = vals.shape
    Tw = (T + 31) // 32
    exp, ev, ov_ref = ge.scalar_ref(vals, ok, key)
    assert ov_ref == overlap
    if overlap:
        with pytest.raises(B2PError) as ei:
            ctx.scalar_calculate(vals, valid, key)
        assert ei.value.code == -1
    else:
        got, gv = ctx.scalar_calculate(vals, valid, key)
        check_cells(got[None, :], gv[None, :], exp[None, :], ev[None, :])
    dv, dvv, dk = Slab(rows * T, "f64", 0, vals), Slab(rows * Tw, "u32", 0, valid), Slab(rows, "u32", 0, key)
    out, ov = Slab(T, "f64", 0), Slab(Tw, "u32", 0)
    n0 = ctx.launch_count()
    ctx.scalar_calculate_dev(dv.ptr, dvv.ptr, dk.ptr, rows, T, out.ptr, ov.ptr)
    if overlap:
        with pytest.raises(B2PError):
            ctx.sync()
        return
    ctx.sync()
    assert ctx.launch_count() - n0 == 2  # reduce, write
    out.assert_guards("scalar() cells")
    ov.assert_guards("scalar() words")
    check_cells(out.body()[None, :], ov.body()[None, :], exp[None, :], ev[None, :])


def test_scalar_calculate_grid_strides(ctx, sms):
    """rows past the reduce's capped warps (dead rows carry junk past T, which must not make them live), and steps past
    the write's capped warps"""
    rng = np.random.default_rng(5)
    T = 33
    rows = sms * 16 * 8 + 5
    ok = np.zeros((rows, T), bool)
    ok[0, :16], ok[rows - 1, 16:] = True, True  # one key, first and last row, disjoint steps
    vals = np.where(ok, ge.VALID_FILL[rng.integers(0, ge.VALID_FILL.size, (rows, T))], ge.INVALID_FILL[3])
    valid = ge.add_junk(ge.words_of(ok), T, rng)
    key = rng.integers(0, rows, rows).astype(np.uint32)
    key[0] = key[rows - 1] = 77  # (every key below the row count)
    exp, ev, _ = ge.scalar_ref(vals, ok, key)
    dv, dvv, dk = Slab(vals.size, "f64", 0, vals), Slab(valid.size, "u32", 0, valid), Slab(rows, "u32", 0, key)
    out, ov = Slab(T, "f64", 0), Slab(valid.shape[1], "u32", 0)
    assert launches(ctx, lambda: ctx.scalar_calculate_dev(dv.ptr, dvv.ptr, dk.ptr, rows, T, out.ptr, ov.ptr)) == 2
    out.assert_guards("scalar() cells")
    ov.assert_guards("scalar() words")
    check_cells(out.body()[None, :], ov.body()[None, :], exp[None, :], ev[None, :])
    T = 32 * sms * 16 * 8 + 45  # output words past the write's capped warps
    Tw = (T + 31) // 32
    ok = np.zeros((2, T), bool)
    ok[0, ::2], ok[1, 1::2] = True, True
    vals = np.where(ok, rng.standard_normal((2, T)), ge.INVALID_FILL[0])
    valid = ge.add_junk(ge.words_of(ok), T, rng)
    for key in (np.array([1, 1], np.uint32), np.array([0, 1], np.uint32)):
        exp, ev, _ = ge.scalar_ref(vals, ok, key)
        got, gv = ctx.scalar_calculate(vals, valid, key)
        check_cells(got[None, :], gv[None, :], exp[None, :], ev[None, :])
        dv, dvv, dk = Slab(2 * T, "f64", 0, vals), Slab(2 * Tw, "u32", 0, valid), Slab(2, "u32", 0, key)
        out, ov = Slab(T, "f64", 0), Slab(Tw, "u32", 0)
        assert launches(ctx, lambda: ctx.scalar_calculate_dev(dv.ptr, dvv.ptr, dk.ptr, 2, T, out.ptr, ov.ptr)) == 2
        out.assert_guards("scalar() cells")
        ov.assert_guards("scalar() words")
        check_cells(out.body()[None, :], ov.body()[None, :], exp[None, :], ev[None, :])


# ---- K15 ------------------------------------------------------------------------------------------------------------------
def absent_run(ctx, ok, valid, T):
    rows = ok.shape[0]
    Tw = (T + 31) // 32
    exp, ev = ge.absent_ref(ok)
    got, gv = ctx.absent(valid.reshape(rows, Tw), T)
    check_cells(got[None, :], gv[None, :], exp[None, :], ev[None, :])
    dvv = Slab(rows * Tw, "u32", 0, valid)
    out, ov = Slab(T, "f64", 0), Slab(Tw, "u32", 0)
    assert launches(ctx, lambda: ctx.absent_dev(dvv.ptr, rows, T, out.ptr, ov.ptr)) == (2 if rows else 1)
    out.assert_guards("absent cells")
    ov.assert_guards("absent words")
    check_cells(out.body()[None, :], ov.body()[None, :], exp[None, :], ev[None, :])


@pytest.mark.parametrize("T", ge.T_LIST)
def test_k15_absent_layouts(ctx, T):
    for c in BY_T[T]:
        absent_run(ctx, c["ok"], c["valid"], T)
        absent_run(ctx, c["ok"][:1], c["valid"][:1], T)
    absent_run(ctx, np.zeros((0, T), bool), np.zeros((0, (T + 31) // 32), np.uint32), T)


@pytest.mark.parametrize("rows,T", ge.ABSENT_SHAPES + [(2 ** 20, 1)])
def test_k15_absent_regimes(ctx, sms, rows, T):
    """Tw < 256 (the shared-memory fold), Tw >= 256 read as whole rows, 1 to 3 rows with Tw above the grid's threads
    (the column walk), and T = 1 over 2^20 rows"""
    rng = np.random.default_rng(rows * 31 + T)
    want = "shared" if (rows, T) in ((5, 33), (2 ** 20, 1)) else ("rows" if rows == 4 else "columns")
    assert ge.absent_regime(sms, rows, T) == want
    ok = np.zeros((rows, T), bool)
    if T == 1:
        ok[rows - 1, 0] = True  # only the last row has the step
    else:
        for r in range(rows):  # each row claims its own stripe, some steps are claimed by no row
            ok[r, r::rows + 1] = True
        ok[:, T - 1] = False
    absent_run(ctx, ok, ge.add_junk(ge.words_of(ok), T, rng), T)
    if T == 1:
        ok[rows - 1, 0] = False
        absent_run(ctx, ok, ge.add_junk(ge.words_of(ok), T, rng), T)


# ---- K13 ------------------------------------------------------------------------------------------------------------------
EXTRA = 40  # outer steps past the inner grid's last step: no sample lies there, junk bits past T included


def subquery_params(T_out, step, fn, range_ms, start=-5_000):
    from greptimedb_b200 import make_params
    return make_params(fn, start, start + (T_out - 1) * step, step, range_ms, filter_nan=False)


def subquery_cases(ctx, vals, ok, start, step):
    """(params, (out, words)) over the outer grid, the inner grid's steps and EXTRA steps past them: last_over_time over
    windows of one inner step (each valid cell comes back as itself) and count_over_time over four.  The expected grid
    is a leaf range call over the sample rows K13 must produce (subquery_rows); the range tiers are held to the oracle
    elsewhere, so a difference here is K13's."""
    ts, val, off = ge.subquery_rows(vals, ok, start, step)
    T_out = ok.shape[1] + EXTRA
    out = []
    for fn, rng_ms in (("last_over_time", step - 1), ("count_over_time", 4 * step - 1)):
        p = subquery_params(T_out, step, fn, rng_ms, start)
        e, ev, _ = ctx.range_eval(p, ts, val, offsets=off)
        out.append((p, (e, ev)))
    return out


def subquery_dev_run(ctx, p, start, step, vals, valid, T_out):
    rows, T = vals.shape
    Tw, Tw_out = (T + 31) // 32, (T_out + 31) // 32
    dv, dvv = Slab(rows * T, "f64", 0, vals), Slab(rows * Tw, "u32", 0, valid)
    out, ov = Slab(rows * T_out, "f64", 0), Slab(rows * Tw_out, "u32", 0)
    ctx.subquery_dev(p, start, step, dv.ptr, dvv.ptr, rows, T, out.ptr, ov.ptr)
    ctx.sync()
    out.assert_guards("K13 cells")
    ov.assert_guards("K13 words")
    return out.body().reshape(rows, T_out), ov.body().reshape(rows, Tw_out)


@pytest.mark.parametrize("T", ge.T_LIST)
def test_k13_subquery_layouts(ctx, T):
    """every pattern's sample rows, junk past T included in the words, through both routes"""
    step, start, T_out = 1000, -5_000, T + EXTRA
    for c in BY_T[T]:
        vals, valid, ok = c["vals"], c["valid"], c["ok"]
        for p, (exp, ev) in subquery_cases(ctx, vals, ok, start, step):
            got, gv = ctx.subquery(p, start, step, vals, valid)
            check_cells(got, gv, exp, ev)
            check_cells(*subquery_dev_run(ctx, p, start, step, vals, valid, T_out), exp, ev)


def test_k13_rows_past_the_warp_grid(ctx, sms):
    """K13's count and scatter take one warp per row on cell_rows_grid (8 warps per CTA, 8 CTAs per SM): rows past it"""
    rng = np.random.default_rng(13)
    T, step = 65, 1000
    rows = sms * 8 * 8 + 9
    ok = rng.random((rows, T)) < 0.5
    vals = np.where(ok, ge.VALID_FILL[rng.integers(0, ge.VALID_FILL.size, (rows, T))], ge.INVALID_FILL[4])
    valid = ge.add_junk(ge.words_of(ok), T, rng)
    for p, (exp, ev) in subquery_cases(ctx, vals, ok, -5_000, step):
        check_cells(*subquery_dev_run(ctx, p, -5_000, step, vals, valid, T + EXTRA), exp, ev)


# ---- K18 ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("F", [2, 3])
def test_k18_valid_and_past_the_grid(ctx, sms, F):
    """a multi-field range call whose validity words outnumber the threads of K18's capped grid: the conjunction equals
    the AND of each field's own range call, and no bit past T is set"""
    import torch
    from greptimedb_b200 import make_params
    rng = np.random.default_rng(18 + F)
    T, step = 65, 1000
    Tw = (T + 31) // 32
    S = sms * 16 * 256 // Tw + 11
    n = rng.integers(0, 3, S)
    offsets = np.concatenate([[0], np.cumsum(n)]).astype(np.int64)
    ts = np.concatenate([np.sort(rng.choice(T * step, k, replace=False)) for k in n]).astype(np.int64)
    vals = [rng.standard_normal(ts.size) for _ in range(F)]
    p = make_params("last_over_time", 0, (T - 1) * step, step, 3 * step)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    dts, doff = d(ts), d(offsets)
    dvals = [d(v) for v in vals]
    outs = [torch.zeros(S * T, dtype=torch.float64, device="cuda") for _ in range(F)]
    vw = Slab(S * Tw, "u32", 0, np.full(S * Tw, 0xFFFFFFFF, np.uint32))
    ctx.range_eval_fields_dev(p, dts, dvals, doff, ts.size, S, outs, vw.ptr)
    ctx.sync()
    vw.assert_guards("K18 words")
    want = np.full((S, Tw), 0xFFFFFFFF, np.uint32)
    for f in range(F):
        o1 = torch.zeros(S * T, dtype=torch.float64, device="cuda")
        v1 = torch.zeros(S * Tw, dtype=torch.int32, device="cuda")
        ctx.range_eval_dev(p, dts, dvals[f], doff, ts.size, S, o1, v1)
        ctx.sync()
        want &= v1.cpu().numpy().view(np.uint32).reshape(S, Tw)
    got = vw.body().reshape(S, Tw)
    assert (got == want).all()
    assert not (got[:, -1] & np.uint32(ge.past_t_mask(T))).any()


# ---- K19 ------------------------------------------------------------------------------------------------------------------
STEPS = ge.calendar_steps()
PARTS = ["time", "minute", "hour", "day_of_month", "day_of_week", "day_of_year", "month", "year", "days_in_month"]


def step_expect(part, ets):
    return np.array([ge.calendar(part, t) for t in ets], np.float64)


@pytest.mark.parametrize("shape", range(len(ge.K19_SHAPES(1))))
def test_k19_step_fn_geometries(ctx, sms, shape):
    shapes = ge.K19_SHAPES(sms)
    T, rows = shapes[shape]
    rng = np.random.default_rng(shape)
    Tw = (T + 31) // 32
    ets = STEPS[(np.arange(T) * 7 + shape) % STEPS.size]
    ok = rng.random((rows, T)) < 0.6
    valid = ge.add_junk(ge.words_of(ok), T, rng)
    dts, dvv = Slab(T, "i64", 0, ets), Slab(rows * Tw, "u32", 0, valid)
    big = rows * T > 200_000
    for part in (["time", "day_of_year", "day_of_week"] if big else PARTS):
        exp = np.where(ok, step_expect(part, ets)[None, :], 0.0)
        if not big:
            assert (bits(ctx.step_fn(part, ets, valid)) == bits(exp)).all(), part
        out = Slab(rows * T, "f64", 0)
        assert launches(ctx, lambda: ctx.step_fn_dev(part, dts.ptr, dvv.ptr, rows, T, out.ptr)) == 1
        out.assert_guards("K19 cells")
        assert (out.body().reshape(rows, T).view(np.uint64) == bits(exp)).all(), part
    assert (dvv.body().reshape(rows, Tw) == valid).all()  # validity is not changed


def test_k19_calendar_edges(ctx):
    """every month end of the sampled years, 29 February, both ends of the year range"""
    T = STEPS.size
    ok = np.ones((2, T), bool)
    ok[1, ::3] = False
    valid = ge.add_junk(ge.words_of(ok), T, np.random.default_rng(1))
    for part in PARTS:
        exp = np.where(ok, step_expect(part, STEPS)[None, :], 0.0)
        assert (bits(ctx.step_fn(part, STEPS, valid)) == bits(exp)).all(), part


def test_k19_range_ends_and_time_extremes(ctx):
    from greptimedb_b200 import B2PError
    e = ge.calendar_edge_steps()
    valid = np.full((2, 1), 0xFFFFFFFF, np.uint32)
    for part in PARTS[1:]:
        got = ctx.step_fn(part, e["in"], valid)
        assert (bits(got) == bits(np.tile(step_expect(part, e["in"]), (2, 1)))).all(), part
        for t in e["out"]:
            with pytest.raises(B2PError):
                ctx.step_fn(part, np.array([0, t], np.int64), valid)
            dts, dvv = Slab(2, "i64", 0, np.array([0, t], np.int64)), Slab(2, "u32", 0, valid[:, 0])
            out = Slab(4, "f64", 0)
            ctx.step_fn_dev(part, dts.ptr, dvv.ptr, 2, 2, out.ptr)
            with pytest.raises(B2PError):
                ctx.sync()
            cells = out.body().reshape(2, 2)
            assert (bits(cells[:, 1]) == 0).all(), "a refused step's cells hold 0.0"
            assert (bits(cells[:, 0]) == bits(np.full(2, ge.calendar(part, 0)))).all()
    for t in ge.TIME_EDGES:
        assert ge.time_correctly_rounded(t)
    got = ctx.step_fn("time", ge.TIME_EDGES, np.full((1, 1), 0xFFFFFFFF, np.uint32))
    assert (bits(got[0]) == bits(step_expect("time", ge.TIME_EDGES))).all()


def test_abs_clears_a_nan_sign_before_a_comparison(ctx):
    """abs(-NaN) is +NaN (Rust's f64::abs clears the sign bit), so `abs(v) > 5` keeps it: +NaN is above +inf in the
    total order comparisons use, where -NaN is below -inf"""
    v = np.array([[np.uint64(0xFFF8000000000001).view(np.float64), -7.0, 3.0, -np.inf]])
    valid = np.array([[0xF]], np.uint32)
    a, av = ctx.instant_fn("abs", v, valid)
    want = np.array([np.uint64(0x7FF8000000000001).view(np.float64), 7.0, 3.0, np.inf])
    assert (bits(a[0]) == bits(want)).all()
    out, ov = ctx.scalar_op(">", 5.0, a, av)
    assert int(ov[0, 0]) == 0b1011
