"""SeriesDivide and the host-pointer range call at their edges: a plain reference of the series offsets, seeded id
columns that put series boundaries where K0's loads, shuffles and carries turn, timestamp classes for the host cadence
scan and ts_expand_kernel, and a restatement of b2p_range_eval's chunk planning with the bytes each chunk sends.

The reference is the header's contract, not the kernel's quad logic:
  - offsets[s] is the first row whose id is >= s, and offsets[n_series] = n_rows;
  - the verdict is B2P_E_UNSORTED iff the ids decrease somewhere or an id (less sid_base, in u32 arithmetic, so an id
    below sid_base wraps past n_series) is >= n_series.

K0's geometry (b2p_range.cu, series_offsets_impl): capped_grid(c, n_rows / 16, 256, 16) CTAs of 8 warps; a warp takes
512 ids per grid-stride pass (4 quad rows of 32 lanes x 4 ids).  A CTA covers 4096 ids, a pass grid * 4096.

layout_cases() yields the seeded columns; each carries the classes its data hit (classes_of, read from the ids), so a
test can assert that every class of CLASSES ran.
"""
from dataclasses import dataclass, field

import numpy as np

E_INVALID, E_UNSORTED = -1, -3
H100_SXM_SMS = 132
IDS_PER_WARP, IDS_PER_CTA, CTAS_PER_SM = 512, 4096, 16
CHUNK_ROWS = 4 << 20          # b2p_range_eval's chunk target (kChunkRows)
ONE_SHOT_ROWS = CHUNK_ROWS + CHUNK_ROWS // 2   # 6 291 456: at or below, one shot
ONE_SHOT_SERIES = 64          # fewer series: one shot
GAPS = (1, 31, 32, 33, 1000)


# ---- reference ------------------------------------------------------------------------------------------------
def offsets_ref(ids, n_series, sid_base=0):
    """(offsets or None, verdict): a plain loop over the rows, from the contract."""
    n = len(ids)
    bad = False
    for r in range(n):
        local = (int(ids[r]) - sid_base) & 0xFFFFFFFF
        if local >= n_series or (r and int(ids[r]) < int(ids[r - 1])):
            bad = True
    if bad:
        return None, E_UNSORTED
    offs = [n] * (n_series + 1)
    s = 0
    for r in range(n):
        local = int(ids[r]) - sid_base
        while s <= local:
            offs[s] = r
            s += 1
    return np.array(offs, np.uint64), 0


def offsets_fast(ids, n_series, sid_base=0):
    """offsets_ref by np.searchsorted, for columns too long for the loop (test_series_divide_edges checks the two agree
    on every small layout)."""
    ids = np.asarray(ids, np.uint32)
    local = ids.astype(np.int64) - sid_base
    if ids.size and ((local < 0).any() or (local >= n_series).any() or (np.diff(ids.astype(np.int64)) < 0).any()):
        return None, E_UNSORTED
    return np.searchsorted(local, np.arange(n_series + 1), side="left").astype(np.uint64), 0


# ---- K0 geometry ------------------------------------------------------------------------------------------------
def k0_grid(n_rows, sms):
    blocks = min(-(-(n_rows // 16) // 256), sms * CTAS_PER_SM)
    return max(blocks, 1)


def k0_pass(n_rows, sms):
    """ids one grid-stride pass covers"""
    return k0_grid(n_rows, sms) * IDS_PER_CTA


def cap_rows(sms):
    """the row count at which K0's grid stops growing"""
    return sms * CTAS_PER_SM * IDS_PER_CTA


def n_rows_list(sms):
    small = [0, 1, 2, 3, 4, 5, 7, 8, 127, 128, 129, 511, 512, 513, 4095, 4096, 4097]
    passes = [4096 * k + r for k in (1, 2, 5) for r in (1, 15)]
    big = [cap_rows(sms) + d for d in (-1, 0, 1, 4, 513)]
    return small + passes + big


# ---- classes read from the data ---------------------------------------------------------------------------------
BOUNDARY_CLASSES = (
    [f"boundary_quad_pos={k}" for k in range(4)]
    + ["boundary_lane0", "boundary_lane31"]
    + [f"boundary_quad_row={j}" for j in range(1, 4)]
    + ["boundary_warp", "boundary_cta", "boundary_second_pass", "boundary_row1", "boundary_last_row",
       "boundary_tail_quad"])
SHAPE_CLASSES = (
    ["one_series", "every_row_own_series", "one_row_series", "zero_rows_with_series", "partial_tail_quad",
     "second_pass"]
    + [f"gap_{w}={g}" for w in ("start", "middle", "end") for g in GAPS])
BAD_CLASSES = ["decrease_in_quad", "decrease_across_lanes", "decrease_across_quad_rows", "decrease_across_passes",
               "out_of_range_row0", "out_of_range_in_run", "out_of_range_last_row", "out_of_range_tail_quad",
               "id_0x80000000", "id_0xFFFFFFFF"]
N_ROWS_CLASSES = ["n_rows_small", "n_rows_4096k+r", "n_rows_past_cap"]
CLASSES = frozenset(BOUNDARY_CLASSES + SHAPE_CLASSES + BAD_CLASSES + N_ROWS_CLASSES)


def classes_of(ids, n_series, sms):
    ids = np.asarray(ids, np.uint32)
    n = ids.size
    c = set()
    if n == 0:
        if n_series >= 1:
            c.add("zero_rows_with_series")
        return c
    if n % 4:
        c.add("partial_tail_quad")
    P = k0_pass(n, sms)
    if n > P:
        c.add("second_pass")
    i64 = ids.astype(np.int64)
    d = np.diff(i64)
    for r in (np.nonzero(d < 0)[0] + 1).tolist():
        if r % 4:
            c.add("decrease_in_quad")
        elif r % 128:
            c.add("decrease_across_lanes")
        elif r % P:
            c.add("decrease_across_quad_rows")
        else:
            c.add("decrease_across_passes")
    oor = np.nonzero(i64 >= n_series)[0]
    if oor.size:
        if oor[0] == 0:
            c.add("out_of_range_row0")
        if ((oor > 0) & (oor < n - 1)).any() and (ids[oor[0]] == ids[min(oor[0] + 1, n - 1)]):
            c.add("out_of_range_in_run")
        if oor.tolist() == [n - 1]:
            c.add("out_of_range_last_row")
        if n % 4 and oor[0] >= n - n % 4:
            c.add("out_of_range_tail_quad")
        if (ids == 0x80000000).any():
            c.add("id_0x80000000")
        if (ids == 0xFFFFFFFF).any():
            c.add("id_0xFFFFFFFF")
    if (d < 0).any() or oor.size:
        return c
    changes = (np.nonzero(d)[0] + 1).tolist()
    for r in changes:
        c.add(f"boundary_quad_pos={r % 4}")
        if r % 128 == 0:
            c.add("boundary_lane0")
        if 124 <= r % 128 <= 127:
            c.add("boundary_lane31")
        if r % 512 and r % 128 == 0:
            c.add(f"boundary_quad_row={(r % 512) // 128}")
        if r % 512 == 0:
            c.add("boundary_warp")
        if r % 4096 == 0:
            c.add("boundary_cta")
        if r == P:
            c.add("boundary_second_pass")
        if r == 1:
            c.add("boundary_row1")
        if r == n - 1:
            c.add("boundary_last_row")
        if n % 4 and r >= n - n % 4:
            c.add("boundary_tail_quad")
    lengths = np.diff(np.asarray(changes + [n]))
    if not changes:
        c.add("one_series")
    elif len(changes) == n - 1:
        c.add("every_row_own_series")
    if (lengths == 1).any() or (changes and changes[0] == 1):
        c.add("one_row_series")
    if ids[0] in GAPS:
        c.add(f"gap_start={int(ids[0])}")
    for g in set((d[d > 1] - 1).tolist()) & set(GAPS):
        c.add(f"gap_middle={g}")
    if n_series - 1 - int(ids[-1]) in GAPS:
        c.add(f"gap_end={n_series - 1 - int(ids[-1])}")
    return c


# ---- layouts ----------------------------------------------------------------------------------------------------
@dataclass
class Layout:
    name: str
    ids: np.ndarray
    n_series: int
    bad: bool = False
    classes: set = field(default_factory=set)


def ids_from_cuts(n, cuts, first=0, jumps=None):
    """ids of n rows whose id grows at each row of `cuts` (by jumps[cut], default 1: gaps of jumps - 1 empty series)"""
    cuts = sorted(set(r for r in cuts if 0 < r < n))
    inc = np.zeros(n, np.int64)
    for r in cuts:
        inc[r] = (jumps or {}).get(r, 1)
    return (first + np.cumsum(inc)).astype(np.uint32)


def boundary_rows(n, sms):
    """every boundary position K0 treats differently, below n"""
    P = k0_pass(n, sms)
    rows = {1, 2, 3, 5, 6, 7, 124, 125, 126, 127, 128, 129, 256, 384, 512, 640, 4096, 4096 + 128, P, P + 1, n - 1}
    rows |= {n - n % 4 + i for i in range(n % 4)}       # inside the partial tail quad
    rows |= {r for r in (8192, 8192 + 512) if r < n}
    return {r for r in rows if 0 < r < n}


def layout_cases(sms=H100_SXM_SMS, seed=0x5D1D, big=True):
    """the good columns, then bad_cases(); generated one at a time (the past-the-cap columns are 35 MB each)"""
    rng = np.random.default_rng(seed)

    def lay(name, ids, n_series, bad=False):
        ids = np.asarray(ids, np.uint32)
        n = ids.size
        cls = classes_of(ids, n_series, sms)
        cls.add("n_rows_past_cap" if n >= cap_rows(sms) - 1 else
                "n_rows_4096k+r" if n > 4096 and n % 4096 in (1, 15) else "n_rows_small")
        return Layout(name, ids, int(n_series), bad, cls)

    for n in n_rows_list(sms):
        if not big and n >= cap_rows(sms) - 1:
            continue
        yield lay(f"n={n}/one_series", np.zeros(n, np.uint32), 1 if n else 3)
        if n <= 8192:
            yield lay(f"n={n}/every_row", np.arange(n, dtype=np.uint32), n)
        cuts = boundary_rows(n, sms)
        ids = ids_from_cuts(n, cuts)
        yield lay(f"n={n}/boundaries", ids, int(ids[-1]) + 1 if n else 1)
        # one-row series at each boundary: a cut at r and at r + 1
        ids = ids_from_cuts(n, cuts | {r + 1 for r in cuts})
        yield lay(f"n={n}/one_row_series", ids, int(ids[-1]) + 1 if n else 1)
    # empty runs at the start, in the middle and at the end
    for n in (129, 4097, 4096 * 2 + 15):
        for g in GAPS:
            cuts = boundary_rows(n, sms)
            mid = sorted(cuts)[len(cuts) // 2]
            ids = ids_from_cuts(n, cuts, first=g, jumps={mid: g + 1})
            yield lay(f"n={n}/gaps={g}", ids, int(ids[-1]) + 1 + g)
    # a seeded random layout over several passes, with a few empty runs
    n = 4096 * 3 + 13
    cuts = set(rng.choice(np.arange(1, n), 400, replace=False).tolist())
    yield lay("random", ids_from_cuts(n, cuts, jumps={r: int(rng.integers(1, 4)) for r in cuts}), 2000)
    for b in bad_cases(sms):
        yield lay(b.name, b.ids, b.n_series, True)


def bad_cases(sms=H100_SXM_SMS):
    """columns K0 must flag: a decrease at each boundary class, an id >= n_series at each place, the top ids"""
    out = []
    n = 4096 * 2 + 15
    P = k0_pass(n, sms)
    base = ids_from_cuts(n, set(range(64, n, 64)))  # ids 0 .. 128
    S = int(base[-1]) + 1
    for name, r in (("in_quad", 1026), ("across_lanes", 1028), ("across_quad_rows", 1024 + 128), ("across_passes", P)):
        ids = base.copy()
        ids[r] = ids[r - 1] - 1   # the one decrease: ids[r + 1] >= ids[r - 1]
        out.append(Layout(f"bad/decrease_{name}", ids, S, True))
    for name, rows in (("row0", [0]), ("in_run", range(640, 700)), ("last_row", [n - 1]),
                       ("tail_quad", [n - 3])):
        ids = base.copy()
        for r in rows:
            ids[r] = S
        if name == "in_run":
            ids[700:] = S
        elif name == "tail_quad":
            ids[n - 3:] = S
        out.append(Layout(f"bad/out_of_range_{name}", ids, S, True))
    for top in (0x80000000, 0xFFFFFFFF):
        ids = base.copy()
        ids[-9:] = top
        out.append(Layout(f"bad/id_{top:#x}", ids, S, True))
        ids = base.copy()
        ids[:1] = top  # a decrease after it as well
        out.append(Layout(f"bad/id_{top:#x}_row0", ids, S, True))
    return out


# ---- timestamp classes ------------------------------------------------------------------------------------------
TS_CLASSES = ("cadence=0", "cadence=1", "cadence=15000", "cadence=2^40", "negative_epoch", "off_first_pair",
              "off_middle", "off_last_row", "long_regular", "one_row", "empty")
LONG_ROWS = 143_167   # 143 167 * 15 000 > 2^31


def timestamps(offsets, cadences, t0s):
    """per series t0 + i * cadence (wrapping, as int64)"""
    offsets = np.asarray(offsets, np.int64)
    lens = np.diff(offsets)
    n = int(offsets[-1])
    idx = np.arange(n, dtype=np.int64) - np.repeat(offsets[:-1], lens)
    cad = np.repeat(np.asarray(cadences, np.int64), lens).astype(np.uint64)
    t0 = np.repeat(np.asarray(t0s, np.int64), lens).astype(np.uint64)
    ts = np.zeros(int(offsets[0]), np.uint64)
    return np.concatenate([ts, t0 + idx.astype(np.uint64) * cad]).view(np.int64)


def ts_cases(seed=0x75C):
    """(name, ts, offsets, regular) for the host scan: every series non-decreasing; `regular` as the scan must say"""
    rng = np.random.default_rng(seed)
    out = []
    lens = [3, 1, 0, 5, 2, 0, 7]
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
    S = len(lens)
    for cad, name in ((0, "cadence=0"), (1, "cadence=1"), (15000, "cadence=15000"), (1 << 40, "cadence=2^40")):
        for t0, epoch in ((1_700_000_000_000, "pos"), (-(1 << 41) - 7, "negative_epoch")):
            ts = timestamps(offs, [cad] * S, rng.integers(-5, 5, S) + t0)
            out.append((f"{name}/{epoch}", ts, offs, True))
    base = timestamps(offs, [15000] * S, [-123_456] * S)
    for name, r in (("off_first_pair", 1), ("off_middle", 7), ("off_last_row", int(offs[-1]) - 1)):
        ts = base.copy()
        ts[r] += 1   # (still non-decreasing within its series)
        out.append((name, ts, offs, False))
    long_offs = np.array([0, 2, LONG_ROWS + 2, LONG_ROWS + 3], np.uint64)
    out.append(("long_regular", timestamps(long_offs, [15000] * 3, [7, 1_700_000_000_000, 0]), long_offs, True))
    return out


def scan_ref(ts, offsets):
    """(t0, cadence, all_regular) of the host scan over rebased offsets, in Python integers mod 2^64"""
    M = 1 << 64
    ts = [int(t) % M for t in np.asarray(ts, np.int64)]
    t0, cad, regular = [], [], True
    for s in range(len(offsets) - 1):
        r0, r1 = int(offsets[s]), int(offsets[s + 1])
        first = ts[r0] if r1 > r0 else 0
        step = (ts[r0 + 1] - first) % M if r1 - r0 >= 2 else 0
        t0.append(first)
        cad.append(step)
        regular = regular and all(ts[r0 + i] == (first + i * step) % M for i in range(r1 - r0))
    signed = lambda v: np.array(v, np.uint64).view(np.int64)
    return signed(t0), signed(cad), regular


# ---- chunk planning of b2p_range_eval ---------------------------------------------------------------------------
@dataclass
class Chunk:
    s0: int
    s1: int
    r0: int
    r1: int
    regular: bool = False


def plan_chunks(n_rows, n_series, ids=None, offsets=None):
    """b2p_range_eval's chunk table (None: one shot)"""
    if n_rows <= ONE_SHOT_ROWS or n_series < ONE_SHOT_SERIES:
        return None
    C = max(64, CHUNK_ROWS // (n_rows // n_series + 1))
    chunks = []
    for s0 in range(0, n_series, C):
        s1 = min(s0 + C, n_series)
        r0 = chunks[-1].r1 if chunks else 0
        r1 = int(offsets[s1]) if offsets is not None else int(np.searchsorted(ids, s1, side="left"))
        chunks.append(Chunk(s0, s1, r0, r1))
    return chunks


def mark_regular(chunks, ts, ids):
    """each chunk's host-scan verdict (ids route): every series in it equally spaced"""
    for k in chunks:
        offs, _ = offsets_fast(ids[k.r0:k.r1], k.s1 - k.s0, k.s0)
        k.regular = offs is not None and chunk_regular(ts[k.r0:k.r1], offs)
    return chunks


def chunk_regular(ts, offs):
    """ts[i] == t0 + i * (ts[1] - ts[0]) (wrapping) in every series: scan_ref(...)[2], vectorised"""
    ts = np.asarray(ts, np.int64).view(np.uint64)
    if ts.size == 0:
        return True
    offs = np.asarray(offs, np.int64)
    starts, lens = offs[:-1], np.diff(offs)
    s0 = np.minimum(starts, ts.size - 1)
    s1 = np.minimum(starts + 1, ts.size - 1)
    step = np.where(lens >= 2, ts[s1] - ts[s0], np.uint64(0)).astype(np.uint64)
    idx = (np.arange(ts.size, dtype=np.int64) - np.repeat(starts, lens)).astype(np.uint64)
    return bool((ts == np.repeat(ts[s0], lens) + idx * np.repeat(step, lens)).all())


def h2d_bytes(n_rows, n_series, chunks, route, redone=()):
    """what b2p_last_h2d_bytes reports: route in {"scan", "ids", "offsets"}; `redone` = indices of chunks redone"""
    by_off = route == "offsets"
    if chunks is None:
        return 16 * n_rows + (8 * (n_series + 1) if by_off else 4 * n_rows)
    total = 0
    for i, k in enumerate(chunks):
        nr, ns = k.r1 - k.r0, k.s1 - k.s0
        if route == "scan" and k.regular:
            total += 8 * nr + 8 * (ns + 1) + 16 * ns
        else:
            total += 16 * nr + (8 * (ns + 1) if by_off else 4 * nr)
        if i in redone:
            total += 16 * nr + (8 * (ns + 1) if by_off else 4 * nr)
    return total
