"""Inputs in key space for the selection kernels (quantile, topk / bottomk, count_values, sort), and a plain reference
for the four of them (test infrastructure only).

Every selection kernel ranks a cell by the same unsigned 64-bit key u = total_key(v) ^ 2^63 (`quant_key` in
b2p_quantile.cuh): -NaN < -inf < .. < -0.0 < +0.0 < .. < +inf < +NaN, every bit pattern its own key.  Key 0 is the
-NaN 0xFFFFFFFFFFFFFFFF and key ~0 the +NaN 0x7FFFFFFFFFFFFFFF.  K11's radix select reads the key as eight 8-bit digits
from the top; the digit where two keys first differ is how deep the select has to go to tell them apart.

`column(cls, n, phi, rng)` lays out the n keys of one (group, step) from a named class.  `lo = floor(phi (n - 1))` and
`hi = min(n - 1, lo + 1)` are the order statistics quantile(phi) reads.  The classes place the pair (a, b) = (lo, hi),
or (lo - 1, lo) when lo = n - 1, of the sorted keys s:
  depth{d}-adjacent  s[a] and s[b] first differ at digit d (0 = the top byte), in neighbouring bins;
  depth{d}-gap       the same, with empty bins between them;
  depth{d}-first     every other key under their shared d-digit prefix, in bins below s[a]'s and above s[b]'s: rank a
                     is the first key of its bin at level d (cum == k);
  depth{d}-last      every key below s[a] in s[a]'s bin at level d: rank a is the last key of a full bin
                     (cum + c == k + 1);
  equal              every key identical: the select runs to level 8;
  top                many keys one digit-7 step apart, the largest at rank n - 1 (what phi = 1 selects);
  sentinel-lo0       s[0..a] = key 0, s[b..] = key ~0;
  sentinel-lomax     s[a..] = key ~0;
  sentinel-hi0       s[..b] = key 0;
  sentinel-only0 / sentinel-onlymax   every key 0 / ~0 (a group of one member holds exactly that key);
  ulps-zero / ulps-subnormal / ulps-inf   keys at most three ulps from ±0, from the smallest normals, from ±inf;
  signed-zero        +0.0 and -0.0 side by side;
  payloads           NaNs of both signs with distinct payloads.
The depth and top classes stay finite (top digit 1 .. 254), so a wrong order statistic shows in the result's bits.

The reference is written from the operations' definitions only: sort the keys (np.sort / np.lexsort / np.unique /
np.argsort), then index.  It is vectorised across steps.
"""
import numpy as np

SIGN = np.uint64(1 << 63)
ALL = np.uint64(0xFFFFFFFFFFFFFFFF)
DEPTHS = range(8)
DEPTH_VARIANTS = ("adjacent", "gap", "first", "last")
OTHER = ("equal", "top", "sentinel-lo0", "sentinel-lomax", "sentinel-hi0", "sentinel-only0", "sentinel-onlymax",
         "ulps-zero", "ulps-subnormal", "ulps-inf", "signed-zero", "payloads")
CLASSES = tuple(f"depth{d}-{v}" for d in DEPTHS for v in DEPTH_VARIANTS) + OTHER
SENTINELS = tuple(c for c in CLASSES if c.startswith("sentinel"))


# ---- the key ---------------------------------------------------------------------------------------------------------
def key_of(bits):
    """f64 bit patterns (uint64) -> u = total_key ^ 2^63: a negative value's bits inverted, a positive one's sign set"""
    b = np.asarray(bits, np.uint64)
    return np.where(b >> np.uint64(63) != 0, ~b, b | SIGN)


def value_of(u):
    """u -> the f64 bit pattern (uint64), the exact inverse of key_of"""
    u = np.asarray(u, np.uint64)
    return np.where(u >> np.uint64(63) != 0, u ^ SIGN, ~u)


def keys_of_values(v):
    return key_of(np.ascontiguousarray(v, np.float64).view(np.uint64))


def values_of_keys(u):
    return np.ascontiguousarray(value_of(u), np.uint64).view(np.float64)


def digit(u, d):
    """digit d (0 = the top byte) of keys u"""
    return (np.asarray(u, np.uint64) >> np.uint64(56 - 8 * d)) & np.uint64(255)


def first_diff_digit(x, y):
    """the first digit at which keys x != y differ"""
    z = int(x) ^ int(y)
    assert z, "equal keys"
    return (63 - z.bit_length() + 1) // 8


def order_stats(n, phi):
    """(lo, hi) of quantile(phi) over n >= 1 keys, phi in [0, 1]"""
    lo = min(int(np.floor(np.float64(phi) * np.float64(n - 1))), n - 1)
    return lo, min(n - 1, lo + 1)


def pair(n, phi):
    """the ranks (a, b) a class lays out: (lo, hi), or (lo - 1, lo) when lo = n - 1"""
    lo, hi = order_stats(n, phi)
    return (lo, hi) if lo < hi else (lo - 1, lo)


# ---- one column ------------------------------------------------------------------------------------------------------
def _u(x):
    return np.uint64(x & 0xFFFFFFFFFFFFFFFF)


def _rand(rng, lo, hi, size):
    """uniform keys in [lo, hi] (Python ints, lo <= hi)"""
    span = hi - lo
    if span == 0:
        return np.full(size, _u(lo), np.uint64)
    r = rng.integers(0, 1 << 63, size, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size, dtype=np.uint64)
    if span < (1 << 64) - 1:
        r = r % np.uint64(span + 1)
    return r + np.uint64(lo)


KMIN, KMAX = 1 << 56, (255 << 56) - 1  # the finite keys the depth classes use: top digit 1 .. 254


def _depth(variant, d, n, a, b, rng):
    shift = 56 - 8 * d
    low_mask = (1 << shift) - 1
    # the shared prefix (digits 0 .. d-1) and the two bins x < y at digit d
    if d == 0:
        prefix = 0
        x = int(rng.integers(2, 200))
    else:
        prefix = int(_rand(rng, KMIN, KMAX, 1)[0]) >> (shift + 8) << (shift + 8)
        x = int(rng.integers(2, 200))
    y = x + 1 if variant in ("adjacent", "last") else x + int(rng.integers(2, 40))
    A = prefix | x << shift | (int(_rand(rng, 0, low_mask, 1)[0]) if shift else 0)
    B = prefix | y << shift | (int(_rand(rng, 0, low_mask, 1)[0]) if shift else 0)
    if variant == "last":  # s[a] as large as its bin allows, so the keys below it fit in the bin
        A = prefix | x << shift | low_mask
    p_lo, p_hi = prefix | 0, prefix | (1 << (shift + 8)) - 1 if d else (1 << 64) - 1
    n_below, n_above = a, n - 1 - b
    if variant in ("adjacent", "gap"):  # the others outside the prefix where there is room, else anywhere
        below = _rand(rng, KMIN, p_lo - 1, n_below) if d and p_lo > KMIN else _rand(rng, KMIN, A, n_below)
        above = _rand(rng, p_hi + 1, KMAX, n_above) if d and p_hi < KMAX else _rand(rng, B, KMAX, n_above)
    elif variant == "first":  # under the prefix, bins below x and above y
        below = _rand(rng, max(p_lo, KMIN), (prefix | x << shift) - 1, n_below)
        above = _rand(rng, (prefix | (y + 1) << shift), min(p_hi, KMAX), n_above)
    else:  # "last": s[a]'s bin, below it
        below = _rand(rng, prefix | x << shift, A, n_below)
        above = _rand(rng, B, min(p_hi, KMAX), n_above)
    return np.concatenate([below, [_u(A)], [_u(B)], above]).astype(np.uint64)


def _near(rng, centres, n, lo_off, hi_off):
    c = np.array([_u(k) for k in centres], np.uint64)[rng.integers(0, len(centres), n)]
    off = rng.integers(lo_off, hi_off + 1, n)
    return (c.astype(object) + off.astype(object)).astype(np.uint64)


def column(cls, n, phi, rng):
    """n keys of class `cls` for quantile(phi), in random order (see the module docstring)"""
    if n == 0:
        return np.zeros(0, np.uint64)
    kphi = phi if 0.0 <= phi <= 1.0 else 0.5
    if cls.startswith("depth"):
        if n == 1:
            return _rand(rng, KMIN, KMAX, 1)
        a, b = pair(n, kphi)
        d, variant = int(cls[5]), cls.split("-")[1]
        s = _depth(variant, d, n, a, b, rng)
    elif cls == "equal":
        s = np.full(n, _rand(rng, KMIN, KMAX, 1)[0], np.uint64)
    elif cls == "top":
        base = int(_rand(rng, KMIN, KMAX, 1)[0]) >> 8 << 8
        s = np.sort(_rand(rng, base, base + 254, n))
        s[-1] = _u(base + 255)  # the largest key, once
    elif cls.startswith("sentinel"):
        s = _rand(rng, KMIN, KMAX, n)
        s.sort()
        a, b = pair(n, kphi) if n > 1 else (0, 0)
        if cls == "sentinel-lo0":
            s[:a + 1], s[b:] = 0, ALL
            if n == 1:
                s[:] = 0
        elif cls == "sentinel-lomax":
            s[a:] = ALL
        elif cls == "sentinel-hi0":
            s[:b + 1] = 0
        elif cls == "sentinel-only0":
            s[:] = 0
        else:
            s[:] = ALL
    elif cls == "ulps-zero":  # -0.0 = 0x7FFF..FF, +0.0 = 0x8000..00
        s = _near(rng, [0x8000000000000000], n, -3, 2)
    elif cls == "ulps-subnormal":  # the largest subnormal / smallest normal of both signs
        s = _near(rng, [0x8010000000000000, key_of_int(0x8010000000000000)], n, -2, 1)
    elif cls == "ulps-inf":  # +inf and the largest finite below it; -inf and the ones above
        up = _near(rng, [key_of_int(0x7FF0000000000000)], n, -3, 0)
        down = _near(rng, [key_of_int(0xFFF0000000000000)], n, 0, 3)
        s = np.where(rng.random(n) < 0.5, up, down)
    elif cls == "signed-zero":
        s = np.where(rng.random(n) < 0.5, _u(0x8000000000000000), _u(0x7FFFFFFFFFFFFFFF)).astype(np.uint64)
    elif cls == "payloads":
        pay = rng.integers(1, 1 << 51, n, dtype=np.uint64) | (rng.integers(0, 2, n, dtype=np.uint64) << np.uint64(51))
        sign = rng.integers(0, 2, n, dtype=np.uint64) << np.uint64(63)
        s = key_of(np.uint64(0x7FF0000000000000) | pay | sign)
    else:
        raise ValueError(cls)
    return rng.permutation(np.asarray(s, np.uint64))


def key_of_int(bits):
    return int(key_of(np.array([bits], np.uint64))[0])


# ---- a grid ----------------------------------------------------------------------------------------------------------
def grid(sizes, T, phi, rng, classes=None, drop=0.0, gid_gap=1, stray=0):
    """Groups of `sizes` members over T steps, group g at id gid_gap * g (the ids between are empty groups), plus
    `stray` rows whose group id is out of range, all rows shuffled.  At step k, group g's valid cells hold a column of
    class classes[(g + k) % len(classes)]: the 32 steps of a tile take different classes, so lanes finish after
    different numbers of passes.  A share `drop` of each group's cells is invalid (every cell of a group of one member
    stays valid) and holds garbage the kernels must not read.
    -> (vals [R, T] f64, ok [R, T] bool, gid [R] u32, n_groups, cls [G, T] class names)"""
    classes = CLASSES if classes is None else classes
    G = len(sizes)
    n_groups = gid_gap * G
    gid = np.concatenate([np.full(s, gid_gap * g, np.uint32) for g, s in enumerate(sizes)] +
                         [np.full(stray, n_groups + 7, np.uint32)])
    gid = gid[rng.permutation(gid.size)]
    R = gid.size
    keys = _rand(rng, 0, (1 << 64) - 1, R * T).reshape(R, T)  # garbage in the invalid cells
    ok = np.zeros((R, T), bool)
    names = np.empty((G, T), object)
    for g, s in enumerate(sizes):
        rows = np.flatnonzero(gid == gid_gap * g)
        for k in range(T):
            n = s - int(rng.binomial(s, drop)) if drop and s > 1 else s
            cls = classes[(g + k) % len(classes)]
            names[g, k] = cls
            pick = rows[rng.permutation(s)[:n]]
            keys[pick, k] = column(cls, n, phi, rng)
            ok[pick, k] = True
    return values_of_keys(keys), ok, gid, n_groups, names


def words(ok):
    """[R, T] bool -> [R, Tw] u32 validity words, no bit at or past T"""
    R, T = ok.shape
    Tw = (T + 31) // 32
    pad = np.zeros((R, Tw * 32), np.uint8)
    pad[:, :T] = ok
    return np.packbits(pad, axis=1, bitorder="little").view(np.uint32).reshape(R, Tw)


def bits_of(valid_words, T):
    w = np.ascontiguousarray(valid_words, np.uint32)
    return np.unpackbits(w.view(np.uint8).reshape(w.shape[0], -1), axis=1, bitorder="little")[:, :T].astype(bool)


def _groups(gid, n_groups):
    gid = np.asarray(gid, np.int64)
    order = np.argsort(gid, kind="stable")
    goff = np.searchsorted(gid[order], np.arange(n_groups + 1))
    return order, goff


# ---- the reference ---------------------------------------------------------------------------------------------------
def quantile(phi, vals, ok, gid, n_groups):
    """quantile(phi) per (group, step) -> (out [G, T] f64, cnt [G, T] u32): the valid keys sorted, lo = floor(phi (n -
    1)), hi = min(n - 1, lo + 1), s[lo] (1 - w) + s[hi] w in separate f64 operations; NaN / -inf / +inf for phi NaN /
    < 0 / > 1; value 0.0 and count 0 without a cell."""
    vals = np.asarray(vals, np.float64)
    R, T = vals.shape
    out = np.zeros((n_groups, T), np.float64)
    cnt = np.zeros((n_groups, T), np.uint32)
    order, goff = _groups(gid, n_groups)
    keys = keys_of_values(vals)
    phi = np.float64(phi)
    for g in range(n_groups):
        rows = order[goff[g]:goff[g + 1]]
        if rows.size == 0:
            continue
        v = ok[rows]
        n = v.sum(axis=0)
        cnt[g] = n
        has = n > 0
        if np.isnan(phi) or phi < 0 or phi > 1:
            out[g, has] = np.nan if np.isnan(phi) else (-np.inf if phi < 0 else np.inf)
            continue
        s = np.sort(np.where(v, keys[rows], ALL), axis=0)  # invalid cells last (as the largest key)
        nm1 = np.maximum(n, 1) - 1
        rank = phi * nm1.astype(np.float64)
        lo = np.minimum(np.floor(rank).astype(np.int64), nm1)
        hi = np.minimum(nm1, lo + 1)
        t = np.arange(T)
        w = rank - np.floor(rank)
        a = values_of_keys(s[lo, t])
        b = values_of_keys(s[hi, t])
        with np.errstate(invalid="ignore", over="ignore"):
            res = a * (np.float64(1.0) - w) + b * w
        out[g] = np.where(has, res, 0.0)
    return out, cnt


def topk(bottom, kk, vals, ok, gid, n_groups, tie):
    """kept cells [R, T] bool: per (group, step) the min(kk, n) best valid cells by (key, tie), the largest for topk,
    the smallest for bottomk; nothing on rows of no group"""
    vals = np.asarray(vals, np.float64)
    R, T = vals.shape
    kept = np.zeros((R, T), bool)
    order, goff = _groups(gid, n_groups)
    keys = keys_of_values(vals)
    tie = np.asarray(tie, np.uint32)
    for g in range(n_groups):
        rows = order[goff[g]:goff[g + 1]]
        if rows.size == 0 or kk == 0:
            continue
        v = ok[rows]
        kh, kl = keys[rows], np.broadcast_to(tie[rows][:, None], v.shape)
        if bottom:  # the smallest first: rank by the inverted key
            kh, kl = ~kh, ~kl
        rank = np.lexsort((kl, kh, v), axis=0)  # ascending; invalid cells first, the best last
        take = np.minimum(v.sum(axis=0), kk)
        pos = np.empty_like(rank)
        np.put_along_axis(pos, rank, np.arange(rows.size)[:, None].repeat(T, axis=1), axis=0)
        kept[rows] = (pos >= rows.size - take) & v
    return kept


def count_values(vals, ok, gid, n_groups):
    """-> (out [R, T] f64, cnt [R, T] u32) in member order (rows stably sorted by gid): at step k, group g's j-th row
    holds its j-th smallest distinct valid key's value and multiplicity; 0.0 / 0 past them and on rows of no group"""
    vals = np.asarray(vals, np.float64)
    R, T = vals.shape
    out = np.zeros((R, T), np.float64)
    cnt = np.zeros((R, T), np.uint32)
    order, goff = _groups(gid, n_groups)
    keys = keys_of_values(vals)
    for g in range(n_groups):
        rows = order[goff[g]:goff[g + 1]]
        r, k = np.nonzero(ok[rows])
        if r.size == 0:
            continue
        pairs, n = np.unique(np.stack([k.astype(np.uint64), keys[rows][r, k]], axis=1), axis=0, return_counts=True)
        step = pairs[:, 0].astype(np.int64)
        first = np.searchsorted(step, step)  # each step's first distinct key
        j = np.arange(step.size) - first
        out[goff[g] + j, step] = values_of_keys(pairs[:, 1])
        cnt[goff[g] + j, step] = n
    return out, cnt


def sort(desc, vals, ok):
    """valid cells as indices r * T + k, stably sorted by key (sort) or ~key (sort_desc)"""
    cells = np.flatnonzero(np.asarray(ok, bool).reshape(-1))
    k = keys_of_values(np.asarray(vals, np.float64).reshape(-1)[cells])
    return cells[np.argsort(~k if desc else k, kind="stable")].astype(np.uint64)


def same_bits(a, b):
    return np.array_equal(np.ascontiguousarray(a, np.float64).view(np.uint64),
                          np.ascontiguousarray(b, np.float64).view(np.uint64))


def same_or_nan(a, b):
    """bits equal, or both NaN (every quantile result passes through arithmetic, which leaves a NaN's payload open)"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return bool(((np.isnan(a) & np.isnan(b)) | (a.view(np.uint64) == b.view(np.uint64))).all())
