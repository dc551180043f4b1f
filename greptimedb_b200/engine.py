"""Thin Python handle on the C ABI (include/b200promql.h).

`Context` owns one b2p_ctx (one device, one stream).  Two call families, mirroring the header:
  * host API  — numpy arrays in, numpy arrays out (H2D / kernels / D2H inside the library);
  * device API — torch CUDA tensors (or raw pointers) in place, asynchronous until `sync()`.
torch is used only to hold device memory and the current stream; all arithmetic is in the CUDA
library.  Function names follow the reference's UDF names (prom_rate -> "rate", ...).
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np

from . import _lib
from ._lib import RangeParams

FN_IDS = {
    "rate": 0, "increase": 1, "delta": 2, "irate": 3, "idelta": 4, "resets": 5, "changes": 6,
    "count_over_time": 7, "sum_over_time": 8, "avg_over_time": 9, "min_over_time": 10,
    "max_over_time": 11, "last_over_time": 12, "present_over_time": 13, "absent_over_time": 14,
    "stdvar_over_time": 15, "stddev_over_time": 16, "deriv": 17, "predict_linear": 18,
    "quantile_over_time": 19, "holt_winters": 20,
}
AGG_IDS = {"sum": 0, "avg": 1, "count": 2, "min": 3, "max": 4, "stddev": 5, "stdvar": 6}
# enum b2p_binop: PromQL binary operators, arithmetic first, then the comparisons
OP_IDS = {"+": 0, "-": 1, "*": 2, "/": 3, "%": 4, "^": 5, "atan2": 6,
          "==": 7, "!=": 8, ">": 9, "<": 10, ">=": 11, "<=": 12}


# enum b2p_setop, and the key of a row that matches nothing on the other side
SETOP_IDS = {"and": 0, "or": 1, "unless": 2}
NO_KEY = 0xFFFFFFFF


# enum b2p_ifn: instant-vector math functions under their PromQL names
IFN_IDS = {"abs": 0, "ceil": 1, "floor": 2, "sqrt": 3, "exp": 4, "ln": 5, "log2": 6, "log10": 7, "sin": 8, "cos": 9,
           "tan": 10, "asin": 11, "acos": 12, "atan": 13, "sinh": 14, "cosh": 15, "tanh": 16, "asinh": 17,
           "acosh": 18, "atanh": 19, "round": 20, "deg": 21, "rad": 22, "sgn": 23, "clamp": 24, "clamp_min": 25,
           "clamp_max": 26, "neg": 28}

# enum b2p_step_part: time() and the calendar functions under their PromQL names
STEP_PARTS = {"time": 0, "minute": 1, "hour": 2, "day_of_month": 3, "day_of_week": 4, "day_of_year": 5, "month": 6,
              "year": 7, "days_in_month": 8}


def step_part(part) -> int:
    return STEP_PARTS[part] if isinstance(part, str) else int(part)


def ifn_id(fn) -> int:
    return IFN_IDS[fn] if isinstance(fn, str) else int(fn)


def op_id(op) -> int:
    return OP_IDS[op] if isinstance(op, str) else int(op)


def setop_id(op) -> int:
    return SETOP_IDS[op] if isinstance(op, str) else int(op)


def topk_bottom(op) -> int:
    """"topk" -> 0, "bottomk" -> 1 (the `bottom` argument of b2p_topk)"""
    if isinstance(op, str):
        return {"topk": 0, "bottomk": 1}[op]
    return int(op)

E_UNSORTED = -3


class B2PError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"b200promql error {code}: {msg}")
        self.code = code


def _ptr(x):
    """numpy array / torch tensor / int / None -> void*"""
    if x is None:
        return None
    if isinstance(x, int):
        return C.c_void_p(x)
    if isinstance(x, np.ndarray):
        return C.c_void_p(x.ctypes.data)
    return C.c_void_p(x.data_ptr())  # torch tensor


def num_steps(start: int, end: int, interval: int) -> int:
    return int(_lib.load().b2p_num_steps(start, end, interval))


def make_params(fn, start, end, interval, range_ms, offset=0, filter_nan=True, param0=0.0, param1=0.0) -> RangeParams:
    fid = FN_IDS[fn] if isinstance(fn, str) else int(fn)
    return RangeParams(fid, int(bool(filter_nan)), int(start), int(end), int(interval), int(range_ms), int(offset),
                       float(param0), float(param1))


def pack_ranges(ranges) -> np.ndarray:
    """[(offset, len)] -> RangeArray keys, offset | len<<32 (range_array.rs:247-254)."""
    r = np.asarray(ranges, dtype=np.uint64).reshape(-1, 2)
    return (r[:, 0] | (r[:, 1] << np.uint64(32))).astype(np.int64)


def valid_to_bool(valid_words: np.ndarray, T: int) -> np.ndarray:
    bits = np.unpackbits(np.ascontiguousarray(valid_words).view(np.uint8), axis=1, bitorder="little")
    return bits[:, :T].astype(bool)


class Context:
    def __init__(self, device: int = 0):
        self._L = _lib.load()
        self._h = self._L.b2p_create(int(device))
        if not self._h:
            raise B2PError(-2, self._L.b2p_last_error().decode())
        self.device = int(device)

    def close(self):
        if getattr(self, "_h", None):
            self._L.b2p_destroy(self._h)
            self._h = None

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    # -- plumbing ---------------------------------------------------------------------------
    def _check(self, rc: int):
        if rc != 0:
            raise B2PError(rc, self._L.b2p_last_error().decode())

    def set_stream(self, cuda_stream_ptr: Optional[int]):
        """Enqueue on the given cudaStream_t; 0/None is the legacy default stream."""
        self._check(self._L.b2p_set_stream(self._h, C.c_void_p(cuda_stream_ptr) if cuda_stream_ptr else None))

    def use_own_stream(self):
        self._check(self._L.b2p_use_own_stream(self._h))

    def use_torch_stream(self):
        import torch
        self.set_stream(torch.cuda.current_stream(self.device).cuda_stream)

    def sync(self):
        self._check(self._L.b2p_sync(self._h))

    def last_slow_series(self) -> int:
        return int(self._L.b2p_last_slow_series(self._h))

    def last_h2d_bytes(self) -> int:
        return int(self._L.b2p_last_h2d_bytes(self._h))

    def last_warp_tier_series(self) -> int:
        return int(self._L.b2p_last_warp_tier_series(self._h))

    def kernel_ms(self, stage: int) -> float:
        return float(self._L.b2p_last_kernel_ms(self._h, stage))

    def launch_count(self) -> int:
        return int(self._L.b2p_launch_count(self._h))

    # -- host API (numpy) --------------------------------------------------------------------
    def range_eval(self, p: RangeParams, ts, val, sid=None, offsets=None):
        """-> (out [S,T] f64, valid_words [S,Tw] u32, eval_ts [T] i64)"""
        ts = np.ascontiguousarray(ts, np.int64)
        val = np.ascontiguousarray(val, np.float64)
        if offsets is not None:
            offsets = np.ascontiguousarray(offsets, np.uint64)
            S = offsets.size - 1
        else:
            sid = np.ascontiguousarray(sid, np.uint32)
            S = int(sid.max()) + 1 if sid.size else 0
        return self.range_eval_n(p, ts, val, sid, offsets, S)

    def range_eval_n(self, p, ts, val, sid, offsets, n_series):
        T = num_steps(p.start, p.end, p.interval)
        Tw = (T + 31) // 32
        out = np.zeros((n_series, T), np.float64)
        valid = np.zeros((n_series, Tw), np.uint32)
        ets = np.zeros(T, np.int64)
        self._check(self._L.b2p_range_eval(self._h, C.byref(p), _ptr(ts), _ptr(val), _ptr(sid), _ptr(offsets),
                                           ts.size, n_series, _ptr(out), _ptr(valid), _ptr(ets)))
        return out, valid, ets

    def range_udf(self, fn, ts, val, ranges, eval_ts=None, range_length=0, param0=0.0, param1=0.0):
        """One prom_* UDF call over explicit windows -> (out f64[], valid bool[])."""
        ts = np.ascontiguousarray(ts, np.int64)
        val = np.ascontiguousarray(val, np.float64)
        packed = pack_ranges(ranges)
        n = packed.size
        ets = None if eval_ts is None else np.ascontiguousarray(eval_ts, np.int64)
        out = np.zeros(n, np.float64)
        valid = np.zeros(n, np.uint8)
        fid = FN_IDS[fn] if isinstance(fn, str) else int(fn)
        self._check(self._L.b2p_range_udf(self._h, fid, _ptr(ts), _ptr(val), ts.size, _ptr(packed), _ptr(ets), n,
                                          int(range_length), float(param0), float(param1), _ptr(out), _ptr(valid)))
        return out, valid.astype(bool)

    def instant_select(self, ts, val, start, end, interval, lookback, offset=0, sid=None, offsets=None):
        ts = np.ascontiguousarray(ts, np.int64)
        val = np.ascontiguousarray(val, np.float64)
        if offsets is not None:
            offsets = np.ascontiguousarray(offsets, np.uint64)
            S = offsets.size - 1
        else:
            sid = np.ascontiguousarray(sid, np.uint32)
            S = int(sid.max()) + 1 if sid.size else 0
        T = num_steps(start, end, interval)
        Tw = (T + 31) // 32
        out = np.zeros((S, T), np.float64)
        valid = np.zeros((S, Tw), np.uint32)
        self._check(self._L.b2p_instant_select(self._h, start, end, interval, lookback, offset, _ptr(ts), _ptr(val),
                                               _ptr(sid), _ptr(offsets), ts.size, S, _ptr(out), _ptr(valid)))
        return out, valid

    @staticmethod
    def _ptr_array(cols):
        """a host array of the columns' pointers (const double* const* / double* const*)"""
        arr = (C.c_void_p * max(1, len(cols)))(*[_ptr(x) for x in cols])
        return C.cast(arr, C.c_void_p), arr

    def _series_count(self, sid, offsets):
        if offsets is not None:
            offsets = np.ascontiguousarray(offsets, np.uint64)
            return None, offsets, offsets.size - 1
        sid = np.ascontiguousarray(sid, np.uint32)
        return sid, None, (int(sid.max()) + 1 if sid.size else 0)

    @classmethod
    def _field_bitmaps(cls, present):
        """per-field bool masks (True = a value; None: no NULL slot) -> (void* to the Arrow validity bitmaps, keep-alive)"""
        if present is None:
            return None, None
        bms = [None if m is None else np.packbits(np.asarray(m, bool), bitorder="little") for m in present]
        ptr, arr = cls._ptr_array(bms)
        return ptr, (bms, arr)

    def range_eval_fields(self, p: RangeParams, ts, vals, sid=None, offsets=None, present=None):
        """A range selector over F field columns of the same rows (vals: F value columns, their buffers as they are;
        present: per-field bool masks of the non-NULL slots, or None) -> (outs [F,S,T] f64, valid_words [S,Tw] u32):
        one validity bitmap, a cell valid only where every field's result is."""
        ts = np.ascontiguousarray(ts, np.int64)
        vals = [np.ascontiguousarray(v, np.float64) for v in vals]
        nb, _keep3 = self._field_bitmaps(present)
        sid, offsets, S = self._series_count(sid, offsets)
        T = num_steps(p.start, p.end, p.interval)
        outs = np.zeros((len(vals), S, T), np.float64)
        valid = np.zeros((S, (T + 31) // 32), np.uint32)
        vp, _keep = self._ptr_array(vals)
        op, _keep2 = self._ptr_array(list(outs))
        self._check(self._L.b2p_range_eval_fields(self._h, C.byref(p), _ptr(ts), vp, nb, len(vals), _ptr(sid),
                                                  _ptr(offsets), ts.size, S, op, _ptr(valid)))
        return outs, valid

    def instant_select_fields(self, ts, vals, start, end, interval, lookback, offset=0, sid=None, offsets=None,
                              present=None):
        """The instant selector over F field columns -> (outs [F,S,T] f64, valid_words [S,Tw] u32): the row of each
        step is chosen by field 0 (its stale-NaN test included) and every field is read from it."""
        ts = np.ascontiguousarray(ts, np.int64)
        vals = [np.ascontiguousarray(v, np.float64) for v in vals]
        nb, _keep3 = self._field_bitmaps(present)
        sid, offsets, S = self._series_count(sid, offsets)
        T = num_steps(start, end, interval)
        outs = np.zeros((len(vals), S, T), np.float64)
        valid = np.zeros((S, (T + 31) // 32), np.uint32)
        vp, _keep = self._ptr_array(vals)
        op, _keep2 = self._ptr_array(list(outs))
        self._check(self._L.b2p_instant_select_fields(self._h, start, end, interval, lookback, offset, _ptr(ts), vp, nb,
                                                      len(vals), _ptr(sid), _ptr(offsets), ts.size, S, op,
                                                      _ptr(valid)))
        return outs, valid

    def group_aggregate(self, agg, vals, valid, gid, n_groups):
        vals = np.ascontiguousarray(vals, np.float64)
        valid = np.ascontiguousarray(valid, np.uint32)
        gid = np.ascontiguousarray(gid, np.uint32)
        S, T = vals.shape
        out = np.zeros((n_groups, T), np.float64)
        cnt = np.zeros((n_groups, T), np.uint32)
        aid = AGG_IDS[agg] if isinstance(agg, str) else int(agg)
        self._check(self._L.b2p_group_aggregate(self._h, aid, _ptr(vals), _ptr(valid), _ptr(gid), S, n_groups, T,
                                                _ptr(out), _ptr(cnt)))
        return out, cnt

    def histogram_quantile(self, phi, le, rates, valid):
        le = np.ascontiguousarray(le, np.float64)
        rates = np.ascontiguousarray(rates, np.float64)
        valid = np.ascontiguousarray(valid, np.uint32)
        B = le.size
        S, T = rates.shape
        H = S // B
        Tw = (T + 31) // 32
        out = np.zeros((H, T), np.float64)
        ov = np.zeros((H, Tw), np.uint32)
        self._check(self._L.b2p_histogram_quantile(self._h, float(phi), _ptr(le), B, _ptr(rates), _ptr(valid), H, T,
                                                   _ptr(out), _ptr(ov)))
        return out, ov

    def histogram_fold(self, phi, hist_off, bucket_series, bucket_le, rates, valid):
        """HistogramFold over any grid rates [R,T] / valid [R,Tw] u32 through the index hist_off [H+1], bucket_series /
        bucket_le [hist_off[H]] (each histogram's buckets in ascending le order, NaN bounds last) -> (out [H,T] f64,
        valid_words [H,Tw] u32).  A malformed index is rejected on the host (B2P_E_INVALID)."""
        hist_off = np.ascontiguousarray(hist_off, np.uint32)
        bucket_series = np.ascontiguousarray(bucket_series, np.uint32)
        bucket_le = np.ascontiguousarray(bucket_le, np.float64)
        rates = np.ascontiguousarray(rates, np.float64)
        valid = np.ascontiguousarray(valid, np.uint32)
        R, T = rates.shape
        if valid.shape != (R, (T + 31) // 32):
            raise ValueError(f"valid must be [{R}, {(T + 31) // 32}] u32 words, got {valid.shape}")
        if hist_off.ndim != 1 or hist_off.size == 0:
            raise ValueError("hist_off must hold n_hist + 1 >= 1 offsets")
        H = hist_off.size - 1
        if bucket_series.size < hist_off[-1] or bucket_le.size < hist_off[-1]:
            raise ValueError(f"bucket_series / bucket_le must hold hist_off[-1] = {int(hist_off[-1])} entries")
        out = np.zeros((H, T), np.float64)
        ov = np.zeros((H, (T + 31) // 32), np.uint32)
        self._check(self._L.b2p_histogram_fold(self._h, float(phi), _ptr(hist_off), _ptr(bucket_series),
                                               _ptr(bucket_le), H, _ptr(rates), _ptr(valid), R, T, _ptr(out), _ptr(ov)))
        return out, ov

    def binary_op(self, op, lhs, lhs_valid, lhs_row, rhs, rhs_valid, rhs_row, return_bool=False):
        """lhs[lhs_row[p]] op rhs[rhs_row[p]] for every pair p -> (out [P,T] f64, valid_words [P,Tw] u32)."""
        lhs = np.ascontiguousarray(lhs, np.float64)
        rhs = np.ascontiguousarray(rhs, np.float64)
        lhs_valid = np.ascontiguousarray(lhs_valid, np.uint32)
        rhs_valid = np.ascontiguousarray(rhs_valid, np.uint32)
        lhs_row = np.ascontiguousarray(lhs_row, np.uint32)
        rhs_row = np.ascontiguousarray(rhs_row, np.uint32)
        T = lhs.shape[1] if lhs.ndim == 2 else rhs.shape[1]
        P = lhs_row.size
        out = np.zeros((P, T), np.float64)
        ov = np.zeros((P, (T + 31) // 32), np.uint32)
        self._check(self._L.b2p_binary_op(self._h, op_id(op), int(bool(return_bool)), _ptr(lhs), _ptr(lhs_valid),
                                          _ptr(lhs_row), lhs.shape[0], _ptr(rhs), _ptr(rhs_valid), _ptr(rhs_row),
                                          rhs.shape[0], P, T, _ptr(out), _ptr(ov)))
        return out, ov

    def scalar_op(self, op, scalar, vals, valid, scalar_on_left=False, return_bool=False):
        """`vals op scalar` (or `scalar op vals`) -> (out [S,T] f64, valid_words [S,Tw] u32)."""
        vals = np.ascontiguousarray(vals, np.float64)
        valid = np.ascontiguousarray(valid, np.uint32)
        S, T = vals.shape
        out = np.zeros((S, T), np.float64)
        ov = np.zeros((S, (T + 31) // 32), np.uint32)
        self._check(self._L.b2p_scalar_op(self._h, op_id(op), int(bool(return_bool)), int(bool(scalar_on_left)),
                                          float(scalar), _ptr(vals), _ptr(valid), S, T, _ptr(out), _ptr(ov)))
        return out, ov

    def setop(self, op, lhs, lhs_valid, lhs_key, rhs, rhs_valid, rhs_key, n_keys):
        """`lhs op rhs` for op in and / or / unless, rows keyed by dense match-key ids (NO_KEY: no match)
        -> (out f64, valid_words u32): [L,T] / [L,Tw] for and / unless, [L+R,T] / [L+R,Tw] (lhs rows first) for or."""
        lhs = np.ascontiguousarray(lhs, np.float64)
        rhs = np.ascontiguousarray(rhs, np.float64)
        lhs_valid = np.ascontiguousarray(lhs_valid, np.uint32)
        rhs_valid = np.ascontiguousarray(rhs_valid, np.uint32)
        lhs_key = np.ascontiguousarray(lhs_key, np.uint32)
        rhs_key = np.ascontiguousarray(rhs_key, np.uint32)
        T = lhs.shape[1] if lhs.ndim == 2 else rhs.shape[1]
        L, R = lhs_key.size, rhs_key.size
        n = L + R if setop_id(op) == SETOP_IDS["or"] else L
        out = np.zeros((n, T), np.float64)
        ov = np.zeros((n, (T + 31) // 32), np.uint32)
        self._check(self._L.b2p_setop(self._h, setop_id(op), _ptr(lhs), _ptr(lhs_valid), _ptr(lhs_key), L, _ptr(rhs),
                                      _ptr(rhs_valid), _ptr(rhs_key), R, int(n_keys), T, _ptr(out), _ptr(ov)))
        return out, ov

    def instant_fn(self, fn, vals, valid, arg0=0.0, arg1=0.0):
        """fn(vals) where valid (round: arg0 = to_nearest; clamp: arg0, arg1 = lo, hi; clamp_min / clamp_max: arg0)
        -> (out [S,T] f64, valid_words [S,Tw] u32, unchanged)."""
        vals = np.ascontiguousarray(vals, np.float64)
        valid = np.ascontiguousarray(valid, np.uint32)
        S, T = vals.shape
        out = np.zeros((S, T), np.float64)
        ov = np.zeros((S, (T + 31) // 32), np.uint32)
        self._check(self._L.b2p_instant_fn(self._h, ifn_id(fn), float(arg0), float(arg1), _ptr(vals), _ptr(valid), S, T,
                                           _ptr(out), _ptr(ov)))
        return out, ov

    def step_fn(self, part, eval_ts, valid):
        """K19: f(eval_ts[k]) at every valid cell of a [S,T] grid (part: "time", "hour", ... or enum b2p_step_part)
        -> out [S,T] f64 (0.0 where invalid); validity is unchanged."""
        eval_ts = np.ascontiguousarray(eval_ts, np.int64)
        valid = np.ascontiguousarray(valid, np.uint32)
        S, T = valid.shape[0], eval_ts.size
        out = np.zeros((S, T), np.float64)
        self._check(self._L.b2p_step_fn(self._h, step_part(part), _ptr(eval_ts), _ptr(valid), S, T, _ptr(out)))
        return out

    def instant_timestamp(self, ts, start, end, interval, lookback, offset=0, sid=None, offsets=None):
        """timestamp(<selector>): the instant selector's rows with the chosen sample's (ts + offset) / 1000 as the
        value and no stale-NaN test -> (out [S,T] f64, valid_words [S,Tw] u32)."""
        ts = np.ascontiguousarray(ts, np.int64)
        sid, offsets, S = self._series_count(sid, offsets)
        T = num_steps(start, end, interval)
        out = np.zeros((S, T), np.float64)
        valid = np.zeros((S, (T + 31) // 32), np.uint32)
        self._check(self._L.b2p_instant_timestamp(self._h, start, end, interval, lookback, offset, _ptr(ts), _ptr(sid),
                                                  _ptr(offsets), ts.size, S, _ptr(out), _ptr(valid)))
        return out, valid

    def scalar_calculate(self, vals, valid, row_key):
        """scalar() over a grid whose rows carry dense series keys (NO_KEY: a label tuple with a NULL)
        -> (out [T] f64, valid_words [Tw] u32)."""
        vals = np.ascontiguousarray(vals, np.float64)
        valid = np.ascontiguousarray(valid, np.uint32)
        row_key = np.ascontiguousarray(row_key, np.uint32)
        S, T = vals.shape
        out = np.zeros(T, np.float64)
        ov = np.zeros((T + 31) // 32, np.uint32)
        self._check(self._L.b2p_scalar_calculate(self._h, _ptr(vals), _ptr(valid), _ptr(row_key), S, T, _ptr(out),
                                                 _ptr(ov)))
        return out, ov

    def topk(self, op, k, vals, valid, gid, n_groups, tie):
        """topk / bottomk (op) of k per (group, step): rows grouped by gid (>= n_groups: no group), ranked by (value in the
        f64 total order, tie) -> the kept cells' validity words [S,Tw] u32 (the values are not touched)."""
        vals = np.ascontiguousarray(vals, np.float64)
        valid = np.ascontiguousarray(valid, np.uint32)
        gid = np.ascontiguousarray(gid, np.uint32)
        tie = np.ascontiguousarray(tie, np.uint32)
        S, T = vals.shape
        ov = np.zeros((S, (T + 31) // 32), np.uint32)
        self._check(self._L.b2p_topk(self._h, topk_bottom(op), float(k), _ptr(vals), _ptr(valid), _ptr(gid), S,
                                     int(n_groups), _ptr(tie), T, _ptr(ov)))
        return ov

    def group_quantile(self, phi, vals, valid, gid, n_groups):
        """quantile(phi) per (group, step): rows grouped by gid (>= n_groups: no group) -> (out [G,T] f64, cnt [G,T]
        u32); cnt 0 is "no row" (value 0.0)."""
        vals = np.ascontiguousarray(vals, np.float64)
        valid = np.ascontiguousarray(valid, np.uint32)
        gid = np.ascontiguousarray(gid, np.uint32)
        S, T = vals.shape
        out = np.zeros((n_groups, T), np.float64)
        cnt = np.zeros((n_groups, T), np.uint32)
        self._check(self._L.b2p_group_quantile(self._h, float(phi), _ptr(vals), _ptr(valid), _ptr(gid), S,
                                               int(n_groups), T, _ptr(out), _ptr(cnt)))
        return out, cnt

    def count_values(self, vals, valid, gid, n_groups):
        """count_values per (group, step): rows grouped by gid (>= n_groups: no group) -> (out [R,T] f64, cnt [R,T] u32)
        with rows in the order of a stable sort of the rows by gid: at each step a group's j-th row holds its j-th
        smallest distinct value (by bits, in the f64 total order) and its multiplicity; cnt 0 past the last."""
        vals = np.ascontiguousarray(vals, np.float64)
        valid = np.ascontiguousarray(valid, np.uint32)
        gid = np.ascontiguousarray(gid, np.uint32)
        S, T = vals.shape
        out = np.zeros((S, T), np.float64)
        cnt = np.zeros((S, T), np.uint32)
        self._check(self._L.b2p_count_values(self._h, _ptr(vals), _ptr(valid), _ptr(gid), S, int(n_groups), T,
                                             _ptr(out), _ptr(cnt)))
        return out, cnt

    def instant_select_fields_i64(self, ts, vals, start, end, interval, lookback, offset=0, sid=None, offsets=None,
                                  present=None):
        """The instant selector with an Int64 field 0 (int64 column; the other fields int64 or float64, moved bit for
        bit) -> (outs [F,S,T] as int64 bits, valid_words [S,Tw] u32): no stale-NaN test."""
        ts = np.ascontiguousarray(ts, np.int64)
        vals = [np.ascontiguousarray(v) for v in vals]
        if any(v.dtype.itemsize != 8 for v in vals):
            raise ValueError("field columns must be 8-byte (int64 or float64)")
        nb, _keep3 = self._field_bitmaps(present)
        sid, offsets, S = self._series_count(sid, offsets)
        T = num_steps(start, end, interval)
        outs = np.zeros((len(vals), S, T), np.int64)
        valid = np.zeros((S, (T + 31) // 32), np.uint32)
        vp, _keep = self._ptr_array(vals)
        op, _keep2 = self._ptr_array(list(outs))
        self._check(self._L.b2p_instant_select_fields_i64(self._h, start, end, interval, lookback, offset, _ptr(ts), vp,
                                                          nb, len(vals), _ptr(sid), _ptr(offsets), ts.size, S, op,
                                                          _ptr(valid)))
        return outs, valid

    def sort_cells_i64_dev(self, desc, vals, valid, n_rows, T, out_cells, out_n):
        """b2p_sort_cells_i64_dev over device tensors (int64 grid, int32 words; out_cells / out_n int64)."""
        self._check(self._L.b2p_sort_cells_i64_dev(self._h, int(bool(desc)), _ptr(vals), _ptr(valid), n_rows, T,
                                                   _ptr(out_cells), _ptr(out_n)))

    def group_aggregate_i64_dev(self, agg, vals, valid, gid, n_series, n_groups, T, out_val, out_cnt):
        """b2p_group_aggregate_i64_dev over device tensors."""
        aid = AGG_IDS[agg] if isinstance(agg, str) else int(agg)
        self._check(self._L.b2p_group_aggregate_i64_dev(self._h, aid, _ptr(vals), _ptr(valid), _ptr(gid), n_series,
                                                        n_groups, T, _ptr(out_val), _ptr(out_cnt)))

    # ---- Int64 (BIGINT) value grids: int64 cells in the same layout; the calls that read a value as a number ----------
    def group_aggregate_i64(self, agg, vals, valid, gid, n_groups):
        """group_aggregate over an int64 grid -> (out [G,T], cnt [G,T] u32): sum (wrapping), min and max as int64, the
        other aggregators as float64 over (double)i64."""
        vals = np.ascontiguousarray(vals, np.int64)
        valid = np.ascontiguousarray(valid, np.uint32)
        gid = np.ascontiguousarray(gid, np.uint32)
        S, T = vals.shape
        out = np.zeros((n_groups, T), np.float64)
        cnt = np.zeros((n_groups, T), np.uint32)
        aid = AGG_IDS[agg] if isinstance(agg, str) else int(agg)
        self._check(self._L.b2p_group_aggregate_i64(self._h, aid, _ptr(vals), _ptr(valid), _ptr(gid), S, n_groups, T,
                                                    _ptr(out), _ptr(cnt)))
        return (out.view(np.int64) if aid in (AGG_IDS["sum"], AGG_IDS["min"], AGG_IDS["max"]) else out), cnt

    def topk_i64(self, op, k, vals, valid, gid, n_groups, tie):
        """topk over an int64 grid (signed order) -> the kept cells' validity words [S,Tw] u32."""
        vals = np.ascontiguousarray(vals, np.int64)
        valid = np.ascontiguousarray(valid, np.uint32)
        gid = np.ascontiguousarray(gid, np.uint32)
        tie = np.ascontiguousarray(tie, np.uint32)
        S, T = vals.shape
        ov = np.zeros((S, (T + 31) // 32), np.uint32)
        self._check(self._L.b2p_topk_i64(self._h, topk_bottom(op), float(k), _ptr(vals), _ptr(valid), _ptr(gid), S,
                                         int(n_groups), _ptr(tie), T, _ptr(ov)))
        return ov

    def count_values_i64(self, vals, valid, gid, n_groups):
        """count_values over an int64 grid -> (out [R,T] int64, cnt [R,T] u32), distinct values in signed order."""
        vals = np.ascontiguousarray(vals, np.int64)
        valid = np.ascontiguousarray(valid, np.uint32)
        gid = np.ascontiguousarray(gid, np.uint32)
        S, T = vals.shape
        out = np.zeros((S, T), np.int64)
        cnt = np.zeros((S, T), np.uint32)
        self._check(self._L.b2p_count_values_i64(self._h, _ptr(vals), _ptr(valid), _ptr(gid), S, int(n_groups), T,
                                                 _ptr(out), _ptr(cnt)))
        return out, cnt

    def sort_cells_i64(self, desc, vals, valid):
        """sort / sort_desc over an int64 grid (signed order, ties in row-major order) -> u64 [n valid cells]."""
        vals = np.ascontiguousarray(vals, np.int64)
        valid = np.ascontiguousarray(valid, np.uint32)
        R, T = vals.shape
        out = np.zeros(max(R * T, 1), np.uint64)
        n = C.c_uint64(0)
        self._check(self._L.b2p_sort_cells_i64(self._h, int(bool(desc)), _ptr(vals), _ptr(valid), R, T, _ptr(out),
                                               C.byref(n)))
        return out[:n.value].copy()

    def i64_to_f64(self, vals):
        """(double)i64 of every cell, on the device."""
        vals = np.ascontiguousarray(vals, np.int64)
        out = np.zeros(vals.shape, np.float64)
        self._check(self._L.b2p_i64_to_f64(self._h, _ptr(vals), vals.size, _ptr(out)))
        return out

    def subquery(self, p: RangeParams, inner_start, inner_interval, vals, valid):
        """fn(<child>[range:step]): vals [R,T'] / valid [R,Tw'] u32 are the child's grid on the inner steps
        inner_start + k * inner_interval; every valid cell of a row is a sample of its series (NaN included).  p is the
        outer grid, range and function (offset 0, filter_nan False).  -> (out [R,T] f64, valid_words [R,Tw] u32)."""
        vals = np.ascontiguousarray(vals, np.float64)
        valid = np.ascontiguousarray(valid, np.uint32)
        R, T_in = vals.shape
        T = num_steps(p.start, p.end, p.interval)
        out = np.zeros((R, T), np.float64)
        ov = np.zeros((R, (T + 31) // 32), np.uint32)
        self._check(self._L.b2p_subquery(self._h, C.byref(p), int(inner_start), int(inner_interval), _ptr(vals),
                                         _ptr(valid), R, T_in, _ptr(out), _ptr(ov)))
        return out, ov

    def sort_cells(self, desc, vals, valid):
        """sort / sort_desc (desc) over any grid vals [R,T] / valid [R,Tw] u32: the valid cells' indices r * T + k in
        value order (the f64 total order; equal values in row-major order) -> u64 [n valid cells]."""
        vals = np.ascontiguousarray(vals, np.float64)
        valid = np.ascontiguousarray(valid, np.uint32)
        R, T = vals.shape
        if valid.shape != (R, (T + 31) // 32):
            raise ValueError(f"valid must be [{R}, {(T + 31) // 32}] u32 words, got {valid.shape}")
        out = np.zeros(max(R * T, 1), np.uint64)
        n = C.c_uint64(0)
        self._check(self._L.b2p_sort_cells(self._h, int(bool(desc)), _ptr(vals), _ptr(valid), R, T, _ptr(out),
                                           C.byref(n)))
        return out[:n.value].copy()

    def sort_cells_fields(self, desc, vals, valid):
        """sort / sort_desc over F fields: vals [F,R,T] (or F grids [R,T]) sharing valid [R,Tw] u32 -> u64 [n valid
        cells], ordered lexicographically by the fields' values (field 0 first, the f64 total order), equal tuples in
        row-major order."""
        vals = [np.ascontiguousarray(v, np.float64) for v in vals]
        valid = np.ascontiguousarray(valid, np.uint32)
        R, T = vals[0].shape
        if any(v.shape != (R, T) for v in vals):
            raise ValueError(f"every field must be [{R}, {T}]")
        if valid.shape != (R, (T + 31) // 32):
            raise ValueError(f"valid must be [{R}, {(T + 31) // 32}] u32 words, got {valid.shape}")
        out = np.zeros(max(R * T, 1), np.uint64)
        n = C.c_uint64(0)
        vp, _keep = self._ptr_array(vals)
        self._check(self._L.b2p_sort_cells_fields(self._h, int(bool(desc)), vp, len(vals), _ptr(valid), R, T,
                                                  _ptr(out), C.byref(n)))
        return out[:n.value].copy()

    def absent(self, valid, T):
        """absent() over any grid's validity valid [R,Tw] u32 with T steps -> (out [T] f64, out_valid [Tw] u32): the steps
        at which no row has a valid cell (bits past T ignored), with the value 1.0; 0.0 and a clear bit elsewhere."""
        valid = np.ascontiguousarray(valid, np.uint32)
        Tw = (T + 31) // 32
        if valid.ndim != 2 or valid.shape[1] != Tw:
            raise ValueError(f"valid must be [rows, {Tw}] u32 words, got {valid.shape}")
        out = np.zeros(T, np.float64)
        ov = np.zeros(Tw, np.uint32)
        self._check(self._L.b2p_absent(self._h, _ptr(valid), valid.shape[0], T, _ptr(out), _ptr(ov)))
        return out, ov

    # -- device API (torch tensors or raw pointers; asynchronous) ----------------------------------
    def series_offsets_dev(self, sid, n_rows, n_series, offsets):
        self._check(self._L.b2p_series_offsets_dev(self._h, _ptr(sid), n_rows, n_series, _ptr(offsets)))

    def range_eval_dev(self, p, ts, val, offsets, n_rows, n_series, out, valid):
        self._check(self._L.b2p_range_eval_dev(self._h, C.byref(p), _ptr(ts), _ptr(val), _ptr(offsets), n_rows,
                                               n_series, _ptr(out), _ptr(valid)))

    def instant_select_dev(self, start, end, interval, lookback, offset, ts, val, offsets, n_rows, n_series, out, valid):
        self._check(self._L.b2p_instant_select_dev(self._h, start, end, interval, lookback, offset, _ptr(ts), _ptr(val),
                                                   _ptr(offsets), n_rows, n_series, _ptr(out), _ptr(valid)))

    def range_eval_fields_dev(self, p, ts, vals, offsets, n_rows, n_series, outs, valid, field_valid=None):
        """vals / outs: sequences of F device columns / grids (tensors or pointers); field_valid: None, or F device
        Arrow validity bitmaps (None entries: no NULL slot)"""
        vp, _keep = self._ptr_array(vals)
        op, _keep2 = self._ptr_array(outs)
        nb, _keep3 = self._ptr_array(field_valid) if field_valid is not None else (None, None)
        self._check(self._L.b2p_range_eval_fields_dev(self._h, C.byref(p), _ptr(ts), vp, nb, len(vals), _ptr(offsets),
                                                      n_rows, n_series, op, _ptr(valid)))

    def instant_select_fields_dev(self, start, end, interval, lookback, offset, ts, vals, offsets, n_rows, n_series,
                                  outs, valid, field_valid=None):
        vp, _keep = self._ptr_array(vals)
        op, _keep2 = self._ptr_array(outs)
        nb, _keep3 = self._ptr_array(field_valid) if field_valid is not None else (None, None)
        self._check(self._L.b2p_instant_select_fields_dev(self._h, start, end, interval, lookback, offset, _ptr(ts), vp,
                                                          nb, len(vals), _ptr(offsets), n_rows, n_series, op, _ptr(valid)))

    def group_aggregate_dev(self, agg, vals, valid, gid, n_series, n_groups, T, out_val, out_cnt):
        aid = AGG_IDS[agg] if isinstance(agg, str) else int(agg)
        self._check(self._L.b2p_group_aggregate_dev(self._h, aid, _ptr(vals), _ptr(valid), _ptr(gid), n_series,
                                                    n_groups, T, _ptr(out_val), _ptr(out_cnt)))

    def range_group_sum_dev(self, p, ts, val, offsets, n_rows, n_series, gid, n_groups, out_sum, out_cnt):
        self._check(self._L.b2p_range_group_sum_dev(self._h, C.byref(p), _ptr(ts), _ptr(val), _ptr(offsets), n_rows,
                                                    n_series, _ptr(gid), n_groups, _ptr(out_sum), _ptr(out_cnt)))

    # group index: an opaque handle (ctypes void pointer) owned by the caller; destroy it with group_index_destroy
    def group_index_create_dev(self, gid, n_series, n_groups):
        h = C.c_void_p()
        self._check(self._L.b2p_group_index_create_dev(self._h, _ptr(gid), n_series, n_groups, C.byref(h)))
        return h

    def group_index_destroy(self, index):
        self._L.b2p_group_index_destroy(self._h, index)

    def group_aggregate_indexed_dev(self, agg, vals, valid, index, T, out_val, out_cnt):
        aid = AGG_IDS[agg] if isinstance(agg, str) else int(agg)
        self._check(self._L.b2p_group_aggregate_indexed_dev(self._h, aid, _ptr(vals), _ptr(valid), index, T,
                                                            _ptr(out_val), _ptr(out_cnt)))

    def range_group_sum_indexed_dev(self, p, ts, val, offsets, n_rows, n_series, index, g_lo, g_hi, out_sum, out_cnt):
        self._check(self._L.b2p_range_group_sum_indexed_dev(self._h, C.byref(p), _ptr(ts), _ptr(val), _ptr(offsets),
                                                            n_rows, n_series, index, g_lo, g_hi, _ptr(out_sum),
                                                            _ptr(out_cnt)))

    def range_group_sum_fused(self, p, index) -> bool:
        return bool(self._L.b2p_range_group_sum_fused(self._h, C.byref(p), index))

    def group_aggregate_partial_dev(self, agg, vals, valid, gid, n_series, n_groups, T, out_val, out_cnt, out_mean=None):
        aid = AGG_IDS[agg] if isinstance(agg, str) else int(agg)
        self._check(self._L.b2p_group_aggregate_partial_dev(self._h, aid, _ptr(vals), _ptr(valid), _ptr(gid), n_series,
                                                            n_groups, T, _ptr(out_val), _ptr(out_cnt), _ptr(out_mean)))

    # multi-GPU: NCCL communicator owned by the context (rank 0 makes the id, every rank calls comm_init)
    def comm_unique_id(self) -> bytes:
        buf = C.create_string_buffer(128)
        self._check(self._L.b2p_comm_unique_id(buf, 128))
        return buf.raw

    def comm_init(self, id_bytes: bytes, n_ranks: int, rank: int):
        buf = C.create_string_buffer(bytes(id_bytes), 128)
        self._check(self._L.b2p_comm_init(self._h, buf, 128, n_ranks, rank))

    def comm_destroy(self):
        self._check(self._L.b2p_comm_destroy(self._h))

    def allreduce_partials_dev(self, agg, val, cnt, mean, n):
        aid = AGG_IDS[agg] if isinstance(agg, str) else int(agg)
        self._check(self._L.b2p_allreduce_partials_dev(self._h, aid, _ptr(val), _ptr(cnt), _ptr(mean), n))

    def range_group_sum_allreduce_dev(self, p, ts, val, offsets, n_rows, n_series, index, n_tiles, out_sum, out_cnt):
        self._check(self._L.b2p_range_group_sum_allreduce_dev(self._h, C.byref(p), _ptr(ts), _ptr(val), _ptr(offsets),
                                                              n_rows, n_series, index, n_tiles, _ptr(out_sum),
                                                              _ptr(out_cnt)))

    def allreduce_columns_dev(self, col_sum, col_cnt, n_cols):
        self._check(self._L.b2p_allreduce_columns_dev(self._h, _ptr(col_sum), _ptr(col_cnt), n_cols))

    def group_finalize_dev(self, agg, val, cnt, n):
        aid = AGG_IDS[agg] if isinstance(agg, str) else int(agg)
        self._check(self._L.b2p_group_finalize_dev(self._h, aid, _ptr(val), _ptr(cnt), n))

    def histogram_quantile_dev(self, phi, le, n_buckets, rates, valid, n_hist, T, out, out_valid):
        self._check(self._L.b2p_histogram_quantile_dev(self._h, float(phi), _ptr(le), n_buckets, _ptr(rates),
                                                       _ptr(valid), n_hist, T, _ptr(out), _ptr(out_valid)))

    def histogram_fold_dev(self, phi, hist_off, bucket_series, bucket_le, n_hist, rates, valid, T, out, out_valid):
        self._check(self._L.b2p_histogram_fold_dev(self._h, float(phi), _ptr(hist_off), _ptr(bucket_series),
                                                   _ptr(bucket_le), n_hist, _ptr(rates), _ptr(valid), T, _ptr(out),
                                                   _ptr(out_valid)))

    def column_reduce_dev(self, col_ptrs, n_cols, n_rows, out_sum, out_cnt):
        self._check(self._L.b2p_column_reduce_dev(self._h, _ptr(col_ptrs), n_cols, n_rows, _ptr(out_sum), _ptr(out_cnt)))

    def binary_op_dev(self, op, lhs, lhs_valid, lhs_row, n_lhs_rows, rhs, rhs_valid, rhs_row, n_rhs_rows, n_pairs, T,
                      out, out_valid, return_bool=False):
        self._check(self._L.b2p_binary_op_dev(self._h, op_id(op), int(bool(return_bool)), _ptr(lhs), _ptr(lhs_valid),
                                              _ptr(lhs_row), n_lhs_rows, _ptr(rhs), _ptr(rhs_valid), _ptr(rhs_row),
                                              n_rhs_rows, n_pairs, T, _ptr(out), _ptr(out_valid)))

    def scalar_op_dev(self, op, scalar, vals, valid, n_rows, T, out, out_valid, scalar_on_left=False, return_bool=False):
        self._check(self._L.b2p_scalar_op_dev(self._h, op_id(op), int(bool(return_bool)), int(bool(scalar_on_left)),
                                              float(scalar), _ptr(vals), _ptr(valid), n_rows, T, _ptr(out),
                                              _ptr(out_valid)))

    def setop_dev(self, op, lhs, lhs_valid, lhs_key, n_lhs_rows, rhs, rhs_valid, rhs_key, n_rhs_rows, n_keys, T, out,
                  out_valid):
        self._check(self._L.b2p_setop_dev(self._h, setop_id(op), _ptr(lhs), _ptr(lhs_valid), _ptr(lhs_key), n_lhs_rows,
                                          _ptr(rhs), _ptr(rhs_valid), _ptr(rhs_key), n_rhs_rows, int(n_keys), T,
                                          _ptr(out), _ptr(out_valid)))

    def instant_fn_dev(self, fn, vals, valid, n_rows, T, out, out_valid, arg0=0.0, arg1=0.0):
        self._check(self._L.b2p_instant_fn_dev(self._h, ifn_id(fn), float(arg0), float(arg1), _ptr(vals), _ptr(valid),
                                               n_rows, T, _ptr(out), _ptr(out_valid)))

    def step_fn_dev(self, part, eval_ts, valid, n_rows, T, out):
        """Device form of step_fn(): eval_ts [T] (int64), valid [n_rows,Tw] into out [n_rows,T]."""
        self._check(self._L.b2p_step_fn_dev(self._h, step_part(part), _ptr(eval_ts), _ptr(valid), n_rows, T, _ptr(out)))

    def instant_timestamp_dev(self, start, end, interval, lookback, offset, ts, offsets, n_rows, n_series, out, valid):
        self._check(self._L.b2p_instant_timestamp_dev(self._h, start, end, interval, lookback, offset, _ptr(ts),
                                                      _ptr(offsets), n_rows, n_series, _ptr(out), _ptr(valid)))

    def scalar_calculate_dev(self, vals, valid, row_key, n_rows, T, out, out_valid):
        self._check(self._L.b2p_scalar_calculate_dev(self._h, _ptr(vals), _ptr(valid), _ptr(row_key), n_rows, T,
                                                     _ptr(out), _ptr(out_valid)))

    def topk_dev(self, op, k, vals, valid, index, tie, T, out_valid):
        """topk / bottomk over the rows of a group index (group_index_create_dev); out_valid may be valid."""
        self._check(self._L.b2p_topk_dev(self._h, topk_bottom(op), float(k), _ptr(vals), _ptr(valid), index, _ptr(tie),
                                         T, _ptr(out_valid)))

    def topk_allgather_dev(self, op, k, vals, valid, index, tie, T, out_valid):
        """topk / bottomk over rows sharded across the ranks of the context's communicator (or one rank without one):
        this rank's kept cells into out_valid; tie must be distinct across every rank."""
        self._check(self._L.b2p_topk_allgather_dev(self._h, topk_bottom(op), float(k), _ptr(vals), _ptr(valid), index,
                                                   _ptr(tie), T, _ptr(out_valid)))

    def last_exchange_bytes(self) -> int:
        return int(self._L.b2p_last_exchange_bytes(self._h))

    def topk_shard_plan(self, k, group_sizes, T, n_ranks) -> dict:
        """The exchange of a sharded topk from the global member count of every group (host u32 [n_groups])."""
        sizes = np.ascontiguousarray(group_sizes, np.uint32)
        out = [C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_uint64(), C.c_uint64()]
        self._check(self._L.b2p_topk_shard_plan(self._h, float(k), _ptr(sizes), sizes.size, T, n_ranks,
                                                *[C.byref(o) for o in out]))
        names = ("n_batches", "n_rounds", "slots", "block_bytes", "state_bytes")
        return {n: int(o.value) for n, o in zip(names, out)}

    def topk_shard_candidates_dev(self, op, k, vals, valid, index, tie, T, group_sizes, n_ranks, batch, rnd, state,
                                  block):
        sizes = np.ascontiguousarray(group_sizes, np.uint32)
        self._check(self._L.b2p_topk_shard_candidates_dev(self._h, topk_bottom(op), float(k), _ptr(vals), _ptr(valid),
                                                          index, _ptr(tie), T, _ptr(sizes), n_ranks, batch, rnd,
                                                          _ptr(state), _ptr(block)))

    def topk_shard_merge_dev(self, k, group_sizes, T, n_ranks, batch, rnd, blocks, state):
        sizes = np.ascontiguousarray(group_sizes, np.uint32)
        self._check(self._L.b2p_topk_shard_merge_dev(self._h, float(k), _ptr(sizes), sizes.size, T, n_ranks, batch, rnd,
                                                     _ptr(blocks), _ptr(state)))

    def topk_shard_mark_dev(self, op, k, vals, valid, index, tie, T, group_sizes, n_ranks, batch, state, out_valid):
        sizes = np.ascontiguousarray(group_sizes, np.uint32)
        self._check(self._L.b2p_topk_shard_mark_dev(self._h, topk_bottom(op), float(k), _ptr(vals), _ptr(valid), index,
                                                    _ptr(tie), T, _ptr(sizes), n_ranks, batch, _ptr(state),
                                                    _ptr(out_valid)))

    def group_quantile_dev(self, phi, vals, valid, index, T, out_val, out_cnt):
        """quantile(phi) over the rows of a group index (group_index_create_dev) into out_val / out_cnt [G,T]."""
        self._check(self._L.b2p_group_quantile_dev(self._h, float(phi), _ptr(vals), _ptr(valid), index, T,
                                                   _ptr(out_val), _ptr(out_cnt)))

    def quantile_allreduce_dev(self, phi, vals, valid, index, T, out_val, out_cnt):
        """quantile(phi) by label over rows sharded across the ranks of the context's communicator (or one rank without
        one): every rank's out_val / out_cnt [G,T] receive the result over the union of the ranks' rows."""
        self._check(self._L.b2p_quantile_allreduce_dev(self._h, float(phi), _ptr(vals), _ptr(valid), index, T,
                                                       _ptr(out_val), _ptr(out_cnt)))

    def quantile_shard_plan(self, n_groups, T) -> dict:
        """The batches of a sharded quantile: n_batches and the largest block and state of a batch in bytes."""
        out = [C.c_uint32(), C.c_uint64(), C.c_uint64()]
        self._check(self._L.b2p_quantile_shard_plan(self._h, n_groups, T, *[C.byref(o) for o in out]))
        return {n: int(o.value) for n, o in zip(("n_batches", "block_bytes", "state_bytes"), out)}

    def quantile_shard_pass_dev(self, phi, vals, valid, index, T, batch, pss, block):
        """This rank's block of one pass of a batch (pass 0 also clears the context's state of the batch)."""
        self._check(self._L.b2p_quantile_shard_pass_dev(self._h, float(phi), _ptr(vals), _ptr(valid), index, T, batch,
                                                        pss, _ptr(block)))

    def quantile_shard_advance_dev(self, phi, n_groups, T, batch, pss, blocks, n_blocks, out_val, out_cnt) -> int:
        """Merges n_blocks blocks, advances the context's state and writes the finished cells -> cells left."""
        live = C.c_uint64()
        self._check(self._L.b2p_quantile_shard_advance_dev(self._h, float(phi), n_groups, T, batch, pss, _ptr(blocks),
                                                           n_blocks, _ptr(out_val), _ptr(out_cnt), C.byref(live)))
        return int(live.value)

    def count_values_dev(self, vals, valid, index, T, out_val, out_cnt):
        """count_values over the rows of a group index (group_index_create_dev) into out_val / out_cnt [rows,T], rows in
        the index's member order."""
        self._check(self._L.b2p_count_values_dev(self._h, _ptr(vals), _ptr(valid), index, T, _ptr(out_val),
                                                 _ptr(out_cnt)))

    def count_values_i64_dev(self, vals, valid, index, T, out_val, out_cnt):
        """count_values over an int64 grid and the rows of a group index into out_val (int64) / out_cnt [rows,T]."""
        self._check(self._L.b2p_count_values_i64_dev(self._h, _ptr(vals), _ptr(valid), index, T, _ptr(out_val),
                                                     _ptr(out_cnt)))

    def count_values_shard_heights_dev(self, local_cnt, index, T, n_groups, n_ranks=1) -> np.ndarray:
        """h_r(g) of this rank's count_values output (rows in member order): with a communicator of n_ranks ranks every
        rank's row, the same table everywhere; without one (n_ranks 1) this rank's.  -> host u32 [n_ranks, n_groups].
        Synchronises the context's stream."""
        heights = np.zeros((n_ranks, n_groups), np.uint32)
        self._check(self._L.b2p_count_values_shard_heights_dev(self._h, _ptr(local_cnt), index, T, _ptr(heights)))
        return heights

    @staticmethod
    def count_values_shard_rows(heights) -> np.ndarray:
        """out_goff [n_groups + 1] of a sharded count_values: group g's rows from out_goff[g], sum over ranks of h_r(g)"""
        u = np.asarray(heights, np.int64).sum(axis=0)
        return np.concatenate([[0], np.cumsum(u)]).astype(np.int64)

    def count_values_allgather_dev(self, local_val, local_cnt, index, T, heights, out_val, out_cnt, i64=False):
        """count_values by label over rows sharded across the ranks of the context's communicator (or one rank without
        one): this rank's count_values output and the heights table -> every rank's out_val / out_cnt
        [out_goff[G], T] (count_values_shard_rows) receive the merged rows."""
        h = np.ascontiguousarray(heights, np.uint32)
        f = self._L.b2p_count_values_allgather_i64_dev if i64 else self._L.b2p_count_values_allgather_dev
        self._check(f(self._h, _ptr(local_val), _ptr(local_cnt), index, T, _ptr(h), _ptr(out_val), _ptr(out_cnt)))

    def count_values_shard_plan(self, heights, T) -> dict:
        """The batches of a sharded count_values from the heights table [n_ranks, n_groups]: n_batches and the largest
        rank block in bytes."""
        h = np.ascontiguousarray(heights, np.uint32)
        out = [C.c_uint32(), C.c_uint64()]
        self._check(self._L.b2p_count_values_shard_plan(self._h, _ptr(h), h.shape[0], h.shape[1], T,
                                                        *[C.byref(o) for o in out]))
        return {n: int(o.value) for n, o in zip(("n_batches", "block_bytes"), out)}

    def count_values_shard_pack_dev(self, local_val, local_cnt, index, T, heights, rank, batch, block, i64=False):
        """This rank's block of one batch: [keys P u64][counts P u32]; last_exchange_bytes() gives P x 12."""
        h = np.ascontiguousarray(heights, np.uint32)
        f = self._L.b2p_count_values_shard_pack_i64_dev if i64 else self._L.b2p_count_values_shard_pack_dev
        self._check(f(self._h, _ptr(local_val), _ptr(local_cnt), index, T, _ptr(h), h.shape[0], rank, batch,
                      _ptr(block)))

    def count_values_shard_merge_dev(self, heights, T, batch, blocks, out_val, out_cnt, i64=False):
        """Merges the gathered blocks of one batch ([keys of rank 0 .. R-1][counts of rank 0 .. R-1], rank r's block
        from row r of heights) into the batch's rows of out_val / out_cnt."""
        h = np.ascontiguousarray(heights, np.uint32)
        f = self._L.b2p_count_values_shard_merge_i64_dev if i64 else self._L.b2p_count_values_shard_merge_dev
        self._check(f(self._h, _ptr(h), h.shape[0], h.shape[1], T, batch, _ptr(blocks), _ptr(out_val), _ptr(out_cnt)))

    def subquery_dev(self, p, inner_start, inner_interval, vals, valid, n_rows, T_inner, out, out_valid):
        """Device form of subquery(): vals [n_rows,T_inner] / valid [n_rows,Tw'] into out [n_rows,T] / out_valid."""
        self._check(self._L.b2p_subquery_dev(self._h, C.byref(p), int(inner_start), int(inner_interval), _ptr(vals),
                                             _ptr(valid), n_rows, T_inner, _ptr(out), _ptr(out_valid)))

    def sort_cells_dev(self, desc, vals, valid, n_rows, T, out_cells, out_n):
        """Device form of sort_cells(): vals [n_rows,T] / valid [n_rows,Tw] into out_cells (room for n_rows * T u64, the
        first out_n written) and out_n (one device u64).  Synchronises the context's stream once (the cell count)."""
        self._check(self._L.b2p_sort_cells_dev(self._h, int(bool(desc)), _ptr(vals), _ptr(valid), n_rows, T,
                                               _ptr(out_cells), _ptr(out_n)))

    def sort_cells_fields_dev(self, desc, vals, valid, n_rows, T, out_cells, out_n):
        """Device form of sort_cells_fields(): vals a sequence of F device grids [n_rows,T] sharing valid [n_rows,Tw].
        Synchronises the context's stream once (the cell count)."""
        vp, _keep = self._ptr_array(vals)
        self._check(self._L.b2p_sort_cells_fields_dev(self._h, int(bool(desc)), vp, len(vals), _ptr(valid), n_rows, T,
                                                      _ptr(out_cells), _ptr(out_n)))

    def absent_dev(self, valid, n_rows, T, out, out_valid):
        """Device form of absent(): valid [n_rows,Tw] into out [T] / out_valid [Tw].  No host round trip."""
        self._check(self._L.b2p_absent_dev(self._h, _ptr(valid), n_rows, T, _ptr(out), _ptr(out_valid)))

    def count_valid_words_dev(self, cnt, n_rows, T, valid_words):
        self._check(self._L.b2p_count_valid_words_dev(self._h, _ptr(cnt), n_rows, T, _ptr(valid_words)))

    def synth_fill_dev(self, series_begin, n_series, n_samples, t0, scrape_ms, jitter_ms, with_resets, seed, ts, val, sid):
        self._check(self._L.b2p_synth_fill_dev(self._h, series_begin, n_series, n_samples, t0, scrape_ms, jitter_ms,
                                               int(with_resets), seed, _ptr(ts), _ptr(val), _ptr(sid)))
