"""Inputs in key space for the sharded quantile's 4-bit select (test infrastructure only).

The sharded select reads the key u = total_key(v) ^ 2^63 (select_keys.key_of) as sixteen 4-bit digits from the top.
`column(variant, d, n, phi, rng)` lays out the n sorted keys of one (group, step) for quantile(phi), with the pair
(a, b) = select_keys.pair(n, phi) placed as select_keys' depth classes place it, but at 4-bit digit d (0 = the top
nibble):
  adjacent  s[a] and s[b] first differ at digit d, in neighbouring bins;
  gap       the same, with empty bins between them;
  first     every other key under their shared d-digit prefix, in bins below s[a]'s and above s[b]'s: rank a is the
            first key of its bin at level d (cum == k);
  last      every key below s[a] in s[a]'s bin at level d: rank a is the last key of a full bin (cum + c == k + 1).
`place` spreads a column over a group's rows so that s[a] and s[b] lie on rows of different ranks and the other keys
(the rest of their bins included) on rows of every rank.  The keys stay finite (top byte 1 .. 254).
"""
import numpy as np

from tests import select_keys as sk

VARIANTS = ("adjacent", "gap", "first", "last")
CLASSES = tuple(f"nibble{d}-{v}" for d in range(16) for v in VARIANTS)


def column(cls, n, phi, rng):
    """-> (sorted keys [n] u64, a, b) of class `cls` ("nibble{d}-{variant}"), n >= 2"""
    d, variant = int(cls[6:cls.index("-")]), cls.split("-")[1]
    a, b = sk.pair(n, phi)
    shift = 60 - 4 * d
    low_mask = (1 << shift) - 1
    prefix = 0 if d == 0 else int(sk._rand(rng, sk.KMIN, sk.KMAX, 1)[0]) >> (shift + 4) << (shift + 4)
    x = int(rng.integers(2, 10))                  # room for keys below x's bin and above y's
    y = x + 1 if variant in ("adjacent", "last") else x + int(rng.integers(2, 5))
    A = prefix | x << shift | (int(sk._rand(rng, 0, low_mask, 1)[0]) if shift else 0)
    B = prefix | y << shift | (int(sk._rand(rng, 0, low_mask, 1)[0]) if shift else 0)
    if variant == "last":  # s[a] as large as its bin allows, so the keys below it fit in the bin
        A = prefix | x << shift | low_mask
    p_lo, p_hi = prefix, (prefix | (1 << (shift + 4)) - 1) if d else (1 << 64) - 1
    n_below, n_above = a, n - 1 - b
    if variant in ("adjacent", "gap"):  # the others outside the prefix where there is room, else anywhere
        below = sk._rand(rng, sk.KMIN, p_lo - 1, n_below) if d and p_lo > sk.KMIN else sk._rand(rng, sk.KMIN, A, n_below)
        above = sk._rand(rng, p_hi + 1, sk.KMAX, n_above) if d and p_hi < sk.KMAX else sk._rand(rng, B, sk.KMAX, n_above)
    elif variant == "first":  # under the prefix, bins below x and above y
        below = sk._rand(rng, max(p_lo, sk.KMIN), (prefix | x << shift) - 1, n_below)
        above = sk._rand(rng, prefix | (y + 1) << shift, min(p_hi, sk.KMAX), n_above)
    else:  # "last": s[a]'s bin, below it
        below = sk._rand(rng, prefix | x << shift, A, n_below)
        above = sk._rand(rng, B, min(p_hi, sk.KMAX), n_above)
    s = np.concatenate([np.sort(below), [sk._u(A)], [sk._u(B)], np.sort(above)]).astype(np.uint64)
    assert (np.diff(s.astype(object)) >= 0).all() and s[a] == sk._u(A) and s[b] == sk._u(B)
    return s, a, b


def place(keys, a, b, rows, owner, rng):
    """-> the rows [n] that receive keys[0 .. n): keys[a] and keys[b] on rows of two different ranks, the rest on a
    random permutation of the other rows.  rows: the group's rows (n of them), owner: their ranks (two at least)."""
    ranks = rng.permutation(np.unique(owner))
    ra = rng.choice(rows[owner == ranks[0]])
    rb = rng.choice(rows[owner == ranks[1]])
    rest = rng.permutation(rows[(rows != ra) & (rows != rb)])
    at = np.empty(rows.size, rows.dtype)
    others = [i for i in range(rows.size) if i not in (a, b)]
    at[a], at[b] = ra, rb
    at[others] = rest
    return at


def grid(n_members, T, phi, owner_of, rng, classes=CLASSES):
    """One group per class, each of n_members rows, step k holding a column of class classes[(g + k) % len]; every
    cell valid.  owner_of(rows) -> the rank of each row (each group must span two ranks at least).
    -> (vals [R, T] f64, ok [R, T] bool, gid [R] u32, n_groups, owner [R])"""
    G = len(classes)
    gid = np.repeat(np.arange(G, dtype=np.uint32), n_members)
    R = gid.size
    owner = owner_of(np.arange(R))
    keys = np.zeros((R, T), np.uint64)
    for g in range(G):
        rows = np.arange(g * n_members, (g + 1) * n_members)
        for k in range(T):
            s, a, b = column(classes[(g + k) % G], n_members, phi, rng)
            keys[place(s, a, b, rows, owner[rows], rng), k] = s
    return sk.values_of_keys(keys), np.ones((R, T), bool), gid, G, owner
