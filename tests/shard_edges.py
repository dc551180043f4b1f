"""Edge classes of the sharded exchange kernels, and their plain references (test infrastructure only).

The sharded operators run a rank's part of the work, exchange blocks, and merge the blocks on every rank.  The host
cuts that work into tiles, rounds and batches, and the cut decides which code a shape reaches.  This module restates
each cut in Python, generates inputs that land on its edges, and holds the references the GPU tests compare with.

  sort (b2p_sort.cu, shard_merge): each thread of a merge tile places `items` outputs, items = 8 for one field and
      min(8, 98304 / (256 (8F + 12))) (at least 1) for F fields, so a tile is cap = 256 items outputs.  The non-empty
      runs merge pairwise in ceil(log2 runs) rounds (one round, a copy, for one run); a round with an odd run count
      passes its last run through with an empty partner.  Round k writes run buffer k % 2, so rounds 4 and 5 (9 to 17
      runs) are the first to overwrite a buffer a round has read.  A tile starting at output d of a pair (a, b) finds
      its split by a binary search over [max(0, d - len b), min(d, len a)].
  count_values (b2p_aggregation.cu, cv_shard_plan): windows of W steps (every step when the costliest group fits the
      exchange cap over all steps, else a multiple of 32), each cut into runs of whole groups that fit the cap.
  topk and quantile (cut_batches): X items x `tiles` 32-step tiles cut into batches of at most `fit` units: every
      unit (branch "all"), every item x fit / X tiles ("tiles"), or fit items x 1 tile ("items").

The references sort keys only (np.lexsort over select_keys' total-order keys and the global cell), so they share no
arithmetic with the kernels.
"""
import math

import numpy as np

from tests import nibble_keys as nk
from tests import select_keys as sk

MAX_FIELDS = 64                    # B2P_MAX_FIELDS
DEFAULT_CAP = 128 << 20            # the context's exchange cap without B2P_TOPK_EXCHANGE_BYTES
I64_MIN, I64_MAX = int(np.iinfo(np.int64).min), int(np.iinfo(np.int64).max)
MAX_NAN = 0x7FFFFFFFFFFFFFFF       # +NaN with every payload bit: key ~0
MIN_NAN = 0xFFFFFFFFFFFFFFFF       # -NaN with every payload bit: key 0


def f64(bits):
    return np.array(bits, np.uint64).view(np.float64)


# ---- sort: the merge's layout ------------------------------------------------------------------------------------------
# every items value: 8 (F <= 4), 7, 6, 5 (F = 7, 8), 4 (F = 9, 10), 3 (F = 11 .. 14), 2 (F = 15 .. 22), 1 (F >= 23)
SORT_FIELDS = (1, 2, 4, 5, 6, 8, 9, 12, 16, 31, 64)
SORT_KEYS = ("equal", "last-field", "sentinels", "nan-zero", "banded", "i64")


def sort_items(F):
    return 8 if F == 1 else max(1, min(8, 98304 // (256 * (8 * F + 12))))


def sort_cap(F):
    return 256 * sort_items(F)


def sort_smem(F):
    """dynamic shared memory of one merge CTA: F + 1 u64 columns and one u32 column of cap entries"""
    return (F + 1) * sort_cap(F) * 8 + sort_cap(F) * 4


def merge_rounds(counts, cap):
    """-> per round, its pairs (len a, len b, first tile); the merge makes one launch per round"""
    runs = [int(c) for c in counts if c]
    if not runs:
        return []
    n_rounds = max(1, math.ceil(math.log2(len(runs))))
    rounds = []
    for _ in range(n_rounds):
        pairs, tiles, nxt = [], 0, []
        for j in range(0, len(runs), 2):
            a, b = runs[j], runs[j + 1] if j + 1 < len(runs) else 0
            pairs.append((a, b, tiles))
            tiles += -(-(a + b) // cap)
            nxt.append(a + b)
        rounds.append(pairs)
        runs = nxt
    return rounds


def tile_edges(rounds, cap):
    """The edges the tiles of a merge reach, as (round, edge) pairs: 'end-of-a' (a tile boundary d = len a, hi clamps
    to len a), 'past-b' (d > len b, the lower bound is d - len b), 'at-b' (d = len b, the lower bound 0 exactly),
    'empty-b' (a run passed through with no partner)"""
    out = set()
    for k, pairs in enumerate(rounds):
        for a, b, _ in pairs:
            if b == 0:
                out.add((k, "empty-b"))
                continue
            for d in range(cap, a + b, cap):
                if d == a:
                    out.add((k, "end-of-a"))
                if d > b:
                    out.add((k, "past-b"))
                if d == b:
                    out.add((k, "at-b"))
    return out


def sort_lengths(F, n_runs, seed):
    """run lengths from {1, cap - 1, cap, cap + 1, 2 cap + 1}; the pattern rotates with n_runs so that a tile boundary
    meets a run's end in the first round and in later ones"""
    cap = sort_cap(F)
    pool = (1, cap - 1, cap, cap + 1, 2 * cap + 1)
    return [pool[(seed + 2 * i + (i >> 2)) % 5] for i in range(n_runs)]


def with_empties(lengths, where):
    """empty ranks first, in the middle or last (or none)"""
    if where == "first":
        return [0, 0] + lengths
    if where == "middle":
        h = len(lengths) // 2
        return lengths[:h] + [0] + lengths[h:]
    if where == "last":
        return lengths + [0]
    return list(lengths)


def sort_cases():
    """every F, run counts 1 .. 17 with empty ranks placed in turn, both orders and every key class"""
    wheres = ("first", "middle", "last", "none")
    cases = []
    for fi, F in enumerate(SORT_FIELDS):
        for n in range(1, 18):
            i = fi * 17 + n
            keys = SORT_KEYS[i % (len(SORT_KEYS) - (F > 1))]  # Int64 is one field
            if F == 1 and keys == "last-field":
                keys = "i64" if n % 2 else "banded"
            cases.append(dict(F=F, counts=with_empties(sort_lengths(F, n, i), wheres[i % 4]), desc=bool(i % 3 == 1),
                              keys=keys, seed=i))
    return cases


def sort_grid(case, T=3):
    """-> (grids [F] of [rows, T] (f64, or one i64), ok [rows, T], owner [rows]) with exactly counts[r] valid cells on
    rank r's rows; a rank's rows interleave with the others' in the global order.  An empty rank holds either no row or
    rows with no valid cell."""
    rng = np.random.default_rng(case["seed"])
    F, counts, keys = case["F"], case["counts"], case["keys"]
    per = [-(-c // T) if c else (r % 2) for r, c in enumerate(counts)]
    owner = rng.permutation(np.repeat(np.arange(len(counts)), per))
    rows = owner.size
    ok = np.zeros((rows, T), bool)
    for r, c in enumerate(counts):
        mine = np.flatnonzero(owner == r)
        if c:
            cells = rng.choice(mine.size * T, c, replace=False)
            ok[mine[cells // T], cells % T] = True
    shape = (rows, T)
    if keys == "i64":
        pool = np.array([I64_MIN, I64_MAX, I64_MIN + 1, I64_MAX - 1, -1, 0], np.int64)
        return [pool[rng.integers(0, pool.size, shape)]], ok, owner
    if keys == "equal":
        grids = [np.full(shape, 2.5) for _ in range(F)]
    elif keys == "last-field":
        grids = [np.full(shape, -1.0) for _ in range(F - 1)] + [rng.choice([0.0, 1.0, 3.0], shape)]
    elif keys == "sentinels":  # key 0 and key ~0, which the desc flip swaps, and ±inf beside them
        pool = f64([MIN_NAN, MAX_NAN, 0x7FF0000000000000, 0xFFF0000000000000])
        grids = [pool[rng.integers(0, 4, shape)] for _ in range(F)]
    elif keys == "nan-zero":  # NaN payloads of both signs and ±0
        pool = f64([0x7FF8000000000001, 0xFFF8000000000001, 0x7FF4000000000000, 0xFFFC00000000BEEF,
                    0x0000000000000000, 0x8000000000000000])
        grids = [pool[rng.integers(0, pool.size, shape)] for _ in range(F)]
    elif keys == "banded":  # rank r's first field in its own band, the later ranks lower: whole runs precede others
        grids = [(-owner[:, None] * 10.0 + rng.integers(0, 3, shape)).astype(np.float64)]
        grids += [rng.choice([0.0, -0.0, np.nan], shape) for _ in range(F - 1)]
    else:
        raise ValueError(keys)
    return grids, ok, owner


def int_keys(bits):
    """I64Key: the two's-complement bits with the sign bit flipped"""
    return np.asarray(bits, np.int64).view(np.uint64) ^ sk.SIGN


def sort_ref(desc, grids, ok, i64=False):
    """the valid cells r * T + k in the order of (field keys .., cell), each key flipped for desc -> u64 cells"""
    T = ok.shape[1]
    cells = np.flatnonzero(ok.reshape(-1)).astype(np.uint64)
    flip = sk.ALL if desc else np.uint64(0)
    keys = [(int_keys(g.reshape(-1)[cells.astype(np.int64)]) if i64 else
             sk.keys_of_values(g.reshape(-1)[cells.astype(np.int64)])) ^ flip for g in grids]
    assert T >= 1
    return cells[np.lexsort([cells] + keys[::-1])]


# ---- count_values: the merge's layout ------------------------------------------------------------------------------------
CV_ENTRY, CV_MERGE_ENTRY, CV_MERGE_SEGMENT = 12, 28, 4
CV_RANKS = (1, 2, 5, 16, 33)
CV_STEPS = (1, 33, 65, 1000)
CV_CAPS = (DEFAULT_CAP, 64 << 10, 1)   # every step in one window; windows of 32 steps; one group per batch


def cv_ref(vals, ok, gid, n_groups, i64=False):
    """select_keys.count_values over Float64 or Int64 keys -> (out [rows, T], cnt [rows, T] u32) in member order"""
    if not i64:
        return sk.count_values(vals, ok, gid, n_groups)
    R, T = vals.shape
    out, cnt = np.zeros((R, T), np.int64), np.zeros((R, T), np.uint32)
    order, goff = sk._groups(gid, n_groups)
    keys = int_keys(vals)
    for g in range(n_groups):
        rows = order[goff[g]:goff[g + 1]]
        r, k = np.nonzero(ok[rows])
        if r.size == 0:
            continue
        pairs, n = np.unique(np.stack([k.astype(np.uint64), keys[rows][r, k]], axis=1), axis=0, return_counts=True)
        step = pairs[:, 0].astype(np.int64)
        j = np.arange(step.size) - np.searchsorted(step, step)
        out[goff[g] + j, step] = (pairs[:, 1] ^ sk.SIGN).view(np.int64)
        cnt[goff[g] + j, step] = n
    return out, cnt


def cv_cases(cap):
    """(R, T) of the count_values runs under `cap`: every rank count with every step count, but with one group per
    batch the 1 000 steps only up to five ranks (32 windows x every group x every rank of calls)"""
    return [(R, T) for R in CV_RANKS for T in CV_STEPS if not (cap == 1 and T == 1000 and R > 5)]


def cv_heights(vals, ok, gid, n_groups, owner, R, i64=False):
    """h_r(g): the rows of group g with a count in rank r's own count_values, i.e. its most distinct values at a step"""
    H = np.zeros((R, n_groups), np.uint32)
    for r in range(R):
        rows = np.flatnonzero(owner == r)
        _, cnt = cv_ref(vals[rows], ok[rows], gid[rows], n_groups, i64)
        _, goff = sk._groups(gid[rows], n_groups)
        for g in range(n_groups):
            nz = np.flatnonzero(cnt[goff[g]:goff[g + 1]].any(axis=1))
            H[r, g] = nz[-1] + 1 if nz.size else 0
    return H


def cv_plan(H, T, cap):
    """cv_shard_plan: H [R, G] heights -> batches [(g0, g1, k0, W, P, rows)]"""
    H = np.asarray(H, np.int64)
    R, G = H.shape
    u = H.sum(axis=0)
    worst = 0
    for g in range(G):
        if u[g]:
            worst = max(worst, (R + 1) * CV_ENTRY * int(H[:, g].max()) + CV_MERGE_ENTRY * int(u[g]) + CV_MERGE_SEGMENT)
    if T == 0 or G == 0 or u.sum() == 0:
        return []
    W = min(-(-T // 32) * 32, max(32, cap // worst // 32 * 32))
    out = []
    for k0 in range(0, T, W):
        Wb = min(W, T - k0)
        g = 0
        while g < G:
            g0, run, pmax, rows = g, np.zeros(R, np.int64), 0, 0
            while g < G:
                pm = max(pmax, int((run + H[:, g]).max()))
                nbytes = ((R + 1) * CV_ENTRY * pm + CV_MERGE_ENTRY * (rows + int(u[g])) +
                          CV_MERGE_SEGMENT * (g + 1 - g0)) * Wb
                if g > g0 and nbytes > cap:
                    break
                run += H[:, g]
                pmax, rows = pm, rows + int(u[g])
                g += 1
            if rows:
                out.append((g0, g, k0, Wb, pmax * Wb, rows))
    return out


def cv_edges(H, T, cap):
    """the edges a count_values case reaches"""
    H = np.asarray(H, np.int64)
    R, G = H.shape
    b = cv_plan(H, T, cap)
    e = set()
    if any(k0 > 0 for _, _, k0, _, _, _ in b):
        e.add("k0>0")
    if b and T % b[0][3] and len({W for _, _, _, W, _, _ in b}) > 1:
        e.add("short-last-window")
    if any(g1 - g0 == 1 for g0, g1, _, _, _, _ in b) and len(b) > 1:
        e.add("one-group-batch")
    u = H.sum(axis=0)
    for g in range(G):
        on = np.flatnonzero(H[:, g])
        if on.size == 1 and R > 2:
            e.add({0: "one-rank-first", R - 1: "one-rank-last"}.get(int(on[0]), "one-rank-middle"))
        if u[g] == 1:
            e.add("U=1")
        if 0 < g < G - 1 and u[g] == 0 and u[:g].any() and u[g + 1:].any():
            e.add("empty-between")
    if R > 8 and (H == 0).mean() > 0.5:
        e.add("mostly-zero-heights")
    return e


def cv_grid(R, T, seed, i64=False):
    """count_values inputs over R ranks -> (vals [rows, T], ok, gid, n_groups, owner, full_group).  Groups, in id order:
    one on rank 0 only, one in the middle rank only, one on the last rank only, a group whose every member holds its
    own value at step 0 on one rank (height = its member count there), an empty group, a group whose members have no
    valid cell, a group of one member with one value everywhere (U = 1), a group with ~0 keys beside real ones on
    every rank, a group whose only real value is ~0, and one spread over every rank."""
    rng = np.random.default_rng(seed)
    top = I64_MAX if i64 else f64([MAX_NAN])[0]
    pool = np.array([I64_MIN, -1, 0, 5, I64_MAX - 1], np.int64) if i64 else np.array([1.5, -0.0, 0.0, -2.0, 1e300])
    mid, last = R // 2, R - 1
    groups = []  # (member ranks, kind)
    groups.append(([0] * 3, "plain"))
    groups.append(([mid] * 4, "plain"))
    groups.append(([last] * 2, "plain"))
    groups.append(([last] * 6 + [0] * 2, "full"))
    groups.append(([], "empty"))
    groups.append(([mid, last], "invalid"))
    groups.append(([0], "one"))
    groups.append((list(range(R)) * 2, "top-beside"))
    groups.append(([mid] * 3, "top-only"))
    groups.append((list(rng.integers(0, R, 3 * R)), "plain"))
    gid, owner, kinds = [], [], []
    for g, (ranks, kind) in enumerate(groups):
        gid += [g] * len(ranks)
        owner += list(ranks)
        kinds += [kind] * len(ranks)
    gid, owner, kinds = np.array(gid, np.uint32), np.array(owner, np.int64), np.array(kinds)
    rows = gid.size
    vals = pool[rng.integers(0, pool.size, (rows, T))]
    ok = rng.random((rows, T)) < 0.7
    full = (kinds == "full") & (owner == last)
    vals[full, 0] = (np.arange(int(full.sum())) * 3 + 1).astype(vals.dtype)  # a distinct value per member there
    ok[full, 0] = True
    ok[kinds == "invalid"] = False
    vals[kinds == "one"] = pool[3]
    ok[kinds == "one"] = True
    beside = kinds == "top-beside"
    vals[beside[:, None] & (rng.random((rows, T)) < 0.5)] = top
    only = kinds == "top-only"
    vals[only] = top
    ok[only] = rng.random((int(only.sum()), T)) < 0.5
    return vals, ok, gid, len(groups), owner


# ---- topk / bottomk: the batch cut -------------------------------------------------------------------------------------------
TOPK_KK = (1, 31, 32, 33, 64, 65, 97)
TOPK_STEPS = (1, 32, 33, 65, 1000)
TOPK_RANKS = (5, 16)
BRANCHES = ("all", "tiles", "items")
STATE_UNIT = 32 * 20


def cut_batches(X, tiles, fit):
    """-> (items per batch, tiles per batch, branch)"""
    if X * tiles <= fit:
        return X, tiles, "all"
    if X <= fit:
        return X, fit // X, "tiles"
    return fit, 1, "items"


def topk_slots(kk):
    return min(kk, 32)


def topk_rounds(kk):
    return 1 if kk <= 32 else -(-kk // 32)


def topk_unit(R, kk):
    """send, gathered and state bytes of one (group, tile) unit"""
    return (R + 1) * 32 * (topk_slots(kk) * 12 + 4) + STATE_UNIT


def topk_plan(kk, sizes, T, R, cap):
    """the sharded topk's plan -> dict(n_batches, block_bytes, branch), exchanged groups only"""
    X = int((np.asarray(sizes) > kk).sum())
    tiles = -(-T // 32)
    xb, tb, branch = cut_batches(X, tiles, max(1, cap // topk_unit(R, kk)))
    n_batches = -(-X // xb) * -(-tiles // tb)
    return dict(n_batches=n_batches, block_bytes=xb * tb * 32 * (topk_slots(kk) * 12 + 4), branch=branch)


def topk_fit(branch, X, tiles):
    """a fit that takes `branch`, with a remainder in the division the branch makes where there is one"""
    if branch == "all":
        return X * tiles
    if branch == "tiles":  # X m + X - 1 < X (m + 1) <= X tiles: m tiles per batch, m + 1 if fit / X rounded up
        return X * min(tiles - 1, 3) + X - 1
    return max(1, X - 1)


def topk_cases():
    """(R, kk, T, branch): every kk with every T, the branches and rank counts in turn (no "tiles" where one tile
    leaves nothing to cut, no "items" with one exchanged group)"""
    cases = []
    for i, kk in enumerate(TOPK_KK):
        for j, T in enumerate(TOPK_STEPS):
            branch = BRANCHES[(i + j) % 3]
            if branch == "tiles" and T <= 32:
                branch = "items"
            cases.append((TOPK_RANKS[(i + j) % 2], kk, T, branch))
    return cases


def topk_grid(R, kk, T, seed):
    """-> (vals, ok, gid, n_groups, tie, owner).  Groups: more than kk members in all but at most kk on every rank;
    exactly kk; kk + 1; more than kk on ranks 0 and 1 only (the others hold no member); an empty group; a small group."""
    rng = np.random.default_rng(seed)
    spread = min(R * kk, kk + 1 + R)
    plan = [
        np.arange(spread) % R,                    # at most ceil(spread / R) <= kk per rank
        rng.integers(0, R, kk),
        rng.integers(0, R, kk + 1),
        rng.integers(0, 2, kk + 3),
        np.zeros(0, np.int64),
        rng.integers(0, R, 2),
    ]
    gid = np.concatenate([np.full(p.size, g, np.uint32) for g, p in enumerate(plan)])
    owner = np.concatenate(plan).astype(np.int64)
    n = gid.size
    pool = np.concatenate([f64([0x7FF8000000000001, 0xFFF800000000BEEF, 0x8000000000000000, MAX_NAN, MIN_NAN]),
                           [0.0, 1.0, 1.0, -2.5, 7.0]])
    vals = pool[rng.integers(0, pool.size, (n, T))]
    ok = rng.random((n, T)) < 0.9
    tie = rng.permutation(n).astype(np.uint32)
    return vals, ok, gid, len(plan), tie, owner


# ---- quantile: the batch cut -------------------------------------------------------------------------------------------
QUANT_UNIT = 2560 + 32 * 56          # block and state of one (group, tile) unit
QUANT_PHIS = (0.0, 1.0, 0.5, math.nan, -0.1, 1.1)
QUANT_PLACES = ("one-rank", "all-but-one", "one-per-rank")
QUANT_CLASSES = ("nibble0-gap", "nibble3-first", "nibble9-last", "nibble15-adjacent")


def quant_plan(n_groups, T, cap):
    tiles = -(-T // 32)
    gb, tb, branch = cut_batches(n_groups, tiles, max(1, cap // QUANT_UNIT))
    return dict(n_batches=-(-n_groups // gb) * -(-tiles // tb), block_bytes=gb * tb * 2560, branch=branch)


def quant_grid(R, T, phi, seed, per_place=4, members=12):
    """groups of nibble_keys' depth classes, each placed on one rank, on every rank but one, or one member per rank
    -> (vals, ok, gid, n_groups, owner)"""
    rng = np.random.default_rng(seed)
    phi = phi if 0.0 <= phi <= 1.0 else 0.5  # outside [0, 1] only the counts are read
    gid, owner, keys = [], [], []
    g = 0
    for place in QUANT_PLACES:
        for cls in QUANT_CLASSES[:per_place]:
            n = {"one-rank": members, "all-but-one": max(members, R - 1), "one-per-rank": R}[place]
            if place == "one-rank":
                own = np.full(n, g % R)
            elif place == "all-but-one":
                others = np.delete(np.arange(R), g % R)
                own = others[np.arange(n) % others.size]
            else:
                own = np.arange(R)
            col = np.zeros((n, T), np.uint64)
            for k in range(T):
                s, _, _ = nk.column(QUANT_CLASSES[(QUANT_CLASSES.index(cls) + k) % len(QUANT_CLASSES)], n, phi, rng)
                col[:, k] = rng.permutation(s)
            gid.append(np.full(n, g, np.uint32))
            owner.append(own)
            keys.append(col)
            g += 1
    keys = np.concatenate(keys)
    return sk.values_of_keys(keys), np.ones(keys.shape, bool), np.concatenate(gid), g, np.concatenate(owner)
