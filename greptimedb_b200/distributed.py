"""Multi-GPU plumbing for the by-label aggregate: series are hash-sharded across ranks (one process
per GPU), every rank reduces its shard into [n_groups x T] (sum f64, cnt u32) partials, and ONE
all-reduce per buffer merges them — the analogue of the reference's __sum_state (datanode) /
__sum_merge (frontend) split, src/query/src/dist_plan/commutativity.rs:85-113,158-176.
rate() alone needs no collective.  torch.distributed is plumbing only (NCCL over NVLink on GPUs,
gloo in the CPU tests); the arithmetic before and after the collective is in libb200promql.so.
"""
from __future__ import annotations

import numpy as np


def mix32(x: np.ndarray) -> np.ndarray:
    """murmur3 fmix32 — the series -> shard / series -> synthetic group hash."""
    x = np.asarray(x, dtype=np.uint32).copy()
    x ^= x >> np.uint32(16)
    x *= np.uint32(0x85EBCA6B)
    x ^= x >> np.uint32(13)
    x *= np.uint32(0xC2B2AE35)
    x ^= x >> np.uint32(16)
    return x


def shard_of_series(series_id: np.ndarray, world: int) -> np.ndarray:
    """Owner rank of every (dense, global) series id: hash(series key) mod n_gpu (SURVEY §8e)."""
    return (mix32(series_id) % np.uint32(world)).astype(np.int64)


def shard_rows(offsets: np.ndarray, world: int, rank: int):
    """Rows and local offsets of the series owned by `rank`.
    -> (series_idx[int64] global ids owned, row_index[int64] gather list, local_offsets[uint64])"""
    offsets = np.asarray(offsets, dtype=np.uint64)
    n_series = offsets.size - 1
    owned = np.flatnonzero(shard_of_series(np.arange(n_series, dtype=np.uint32), world) == rank)
    lens = (offsets[owned + 1] - offsets[owned]).astype(np.int64)
    local_offsets = np.zeros(owned.size + 1, np.uint64)
    np.cumsum(lens, out=local_offsets[1:].view(np.int64))
    rows = np.concatenate([np.arange(int(offsets[s]), int(offsets[s + 1]), dtype=np.int64) for s in owned]) \
        if owned.size else np.zeros(0, np.int64)
    return owned, rows, local_offsets


def allreduce_group_partials(sum_t, cnt_t, group=None):
    """In-place SUM all-reduce of the (sum, cnt) partial matrices (torch tensors, CPU/gloo or CUDA/NCCL).
    cnt is reduced as int64 on gloo-safe dtypes; on CUDA it stays int32."""
    import torch
    import torch.distributed as dist
    dist.all_reduce(sum_t, op=dist.ReduceOp.SUM, group=group)
    if cnt_t.dtype in (torch.int32, torch.int64):
        dist.all_reduce(cnt_t, op=dist.ReduceOp.SUM, group=group)
    else:
        tmp = cnt_t.to(torch.int64)
        dist.all_reduce(tmp, op=dist.ReduceOp.SUM, group=group)
        cnt_t.copy_(tmp.to(cnt_t.dtype))
    return sum_t, cnt_t


def finalize_host(agg: str, sum_a: np.ndarray, cnt_a: np.ndarray) -> np.ndarray:
    """Host mirror of b2p_group_finalize_dev (used by the gloo tests): avg = sum/cnt, count = cnt."""
    out = sum_a.copy()
    nz = cnt_a > 0
    if agg == "avg":
        out[nz] = sum_a[nz] / cnt_a[nz]
    elif agg == "count":
        out = cnt_a.astype(np.float64)
    out[~nz] = 0.0
    return out


_SIGN = np.uint64(1 << 63)


def _key(x):
    """u64 total-order key of float64 values: unsigned order of the keys is f64::total_cmp order"""
    b = np.ascontiguousarray(x, np.float64).view(np.uint64)
    return np.where(b >> np.uint64(63) != 0, ~b, b | _SIGN)


def _value(u):
    """float64 values of u64 total-order keys (the inverse of _key)"""
    return np.ascontiguousarray(np.where(u >> np.uint64(63) != 0, u ^ _SIGN, ~u), np.uint64).view(np.float64)


def _all_gather(arr, group):
    """every rank's numpy array `arr` (the same shape and dtype on every rank), in rank order"""
    import torch
    import torch.distributed as dist
    t = torch.from_numpy(np.ascontiguousarray(arr))
    out = [torch.empty_like(t) for _ in range(dist.get_world_size(group))]
    dist.all_gather(out, t, group=group)
    return [o.numpy() for o in out]


def total_key(x):
    """f64::total_cmp key of a float64 tensor as int64: the bit pattern with the 63 low bits flipped where the sign bit
    is set.  Applied to the int64 keys (or their bit patterns) it gives the bit patterns back: an involution."""
    import torch
    b = x.view(torch.int64)
    return b ^ ((b >> 63) & torch.iinfo(torch.int64).max)


def merge_partials(agg: str, val_t, cnt_t, mean_t=None, group=None):
    """Host mirror of b2p_allreduce_partials_dev (same formulas, torch.distributed instead of the library's NCCL
    communicator; used by the gloo tests): in-place merge of every rank's by-label partials.
      sum / avg / count : val and cnt are added                       (commutativity.rs:85-113)
      min / max         : val is reduced as f64::total_cmp keys (int64 min / max), the order of the single-pass
                          aggregate (+NaN greatest, -NaN least, -0.0 < +0.0); groups absent on a rank (cnt == 0) get
                          the neutral key, cnt is added, groups absent everywhere read 0.0 again
      stddev / stdvar   : per-rank (cnt, mean, M2 = val) states; global mean from an all-reduce of cnt * mean,
                          M2 = sum_r [M2_r + cnt_r (mean_r - mean)^2]  (commutativity.rs:158-191)"""
    import torch
    import torch.distributed as dist
    cnt64 = cnt_t.to(torch.int64)
    if agg in ("min", "max"):
        key = total_key(val_t.contiguous())
        key[cnt64 == 0] = torch.iinfo(torch.int64).max if agg == "min" else torch.iinfo(torch.int64).min
        dist.all_reduce(key, op=dist.ReduceOp.MIN if agg == "min" else dist.ReduceOp.MAX, group=group)
        dist.all_reduce(cnt64, op=dist.ReduceOp.SUM, group=group)
        val_t.copy_(total_key(key).view(torch.float64))
        val_t[cnt64 == 0] = 0.0
    elif agg in ("stddev", "stdvar"):
        cnt_r = cnt64.clone()
        wsum = cnt_r.to(torch.float64) * mean_t
        dist.all_reduce(wsum, op=dist.ReduceOp.SUM, group=group)
        dist.all_reduce(cnt64, op=dist.ReduceOp.SUM, group=group)
        mg = torch.where(cnt64 > 0, wsum / cnt64.clamp_min(1).to(torch.float64), torch.zeros_like(wsum))
        d = mean_t - mg
        val_t.copy_(torch.where(cnt_r > 0, val_t + cnt_r.to(torch.float64) * d * d, torch.zeros_like(val_t)))
        mean_t.copy_(mg)
        dist.all_reduce(val_t, op=dist.ReduceOp.SUM, group=group)
    else:
        dist.all_reduce(val_t, op=dist.ReduceOp.SUM, group=group)
        dist.all_reduce(cnt64, op=dist.ReduceOp.SUM, group=group)
    cnt_t.copy_(cnt64.to(cnt_t.dtype))
    return val_t, cnt_t


def topk_key_host(bottom: bool, vals: np.ndarray, tie: np.ndarray):
    """The rank key of every cell of K10, (hi, lo) = (f64 total-order key as u64, tie), both bit-inverted for bottomk so
    that better is always larger."""
    hi = _key(vals)
    lo = np.broadcast_to(np.asarray(tie, np.uint32)[:, None], hi.shape)
    return (~hi, ~lo) if bottom else (hi, lo.copy())


def merge_topk_candidates(bottom: bool, kk: int, vals: np.ndarray, ok: np.ndarray, gid: np.ndarray, n_groups: int,
                          tie: np.ndarray, group=None, slots_max: int = 32):
    """Host mirror of b2p_topk_allgather_dev (same exchange, torch.distributed instead of the library's NCCL
    communicator; used by the gloo tests): this rank's rows [R, T] (ok: valid cells, gid >= n_groups: no group, tie
    distinct across every rank) -> (kept [R, T] bool, exchanged group count, rounds, slots).
      - the per-group member counts are all-reduced; kk = 0 keeps nothing, kk >= the largest group every valid cell, a
        group of at most kk members every valid cell;
      - every other group is exchanged: per round and step each rank sends its best min(kk, slots_max) keys below the
        bound and their count, all-gathered; the merge's verdict is "all" (fewer than that many left, within what is
        still to take), the threshold (the rem-th best), or the next bound (the smallest of the slots taken);
      - each rank keeps its own valid cells at or above the threshold, or every one below the bounds taken ("all")."""
    import torch
    import torch.distributed as dist
    R, T = vals.shape
    gid = np.asarray(gid, np.int64)
    ing = gid < n_groups
    local = np.bincount(gid[ing], minlength=n_groups).astype(np.int64)
    sizes_t = torch.from_numpy(local.copy())
    dist.all_reduce(sizes_t, op=dist.ReduceOp.SUM, group=group)
    sizes = sizes_t.numpy()
    kept = np.zeros((R, T), bool)
    if kk == 0 or n_groups == 0:
        return kept, 0, 0, 0
    if kk >= sizes.max():
        kept[ing] = ok[ing]
        return kept, 0, 0, 0
    small = ing & (sizes[np.where(ing, gid, 0)] <= kk)
    kept[small] = ok[small]
    xg = np.flatnonzero(sizes > kk)
    K = min(kk, slots_max)
    rounds = -(-kk // slots_max) if kk > slots_max else 1
    hi, lo = topk_key_host(bottom, vals, tie)
    X = xg.size
    rem = np.full((X, T), kk, np.int64)
    done = np.zeros((X, T), bool)                   # "all": every cell below the bound is kept
    th_hi = np.zeros((X, T), np.uint64)             # bound (rounds) / threshold (rem == 0)
    th_lo = np.zeros((X, T), np.uint32)
    bounded = np.zeros((X, T), bool)
    members = [np.flatnonzero(gid == g) for g in xg]

    def below(h, l, i):  # cells strictly below the bound of group i
        return ~bounded[i] | (h < th_hi[i]) | ((h == th_hi[i]) & (l < th_lo[i]))

    for _ in range(rounds):
        s_hi = np.zeros((X, T, K), np.uint64)
        s_lo = np.zeros((X, T, K), np.uint32)
        s_n = np.zeros((X, T), np.int64)
        for i, rows in enumerate(members):
            if rows.size == 0:
                continue
            h, l = hi[rows], lo[rows]
            live = ok[rows] & below(h, l, i) & ~done[i] & (rem[i] > 0)
            order = np.lexsort((l, h, live), axis=0)[::-1]   # live first, then the best
            n = np.minimum(live.sum(axis=0), K)
            take = min(K, rows.size)
            s_hi[i, :, :take] = np.take_along_axis(h, order[:take], axis=0).T
            s_lo[i, :, :take] = np.take_along_axis(l, order[:take], axis=0).T
            s_n[i] = n
        parts = [_all_gather(a, group) for a in (s_hi.view(np.int64), s_lo.astype(np.int64), s_n)]
        g_hi = np.concatenate([p.view(np.uint64) for p in parts[0]], axis=2)      # [X, T, world * K]
        g_lo = np.concatenate([p.astype(np.uint32) for p in parts[1]], axis=2)
        g_on = np.concatenate([np.arange(K)[None, None, :] < p[:, :, None] for p in parts[2]], axis=2)
        order = np.lexsort((g_lo, g_hi, g_on), axis=2)[:, :, ::-1]
        n = np.minimum(g_on.sum(axis=2), K)
        active = ~done & (rem > 0)
        fits = active & (n < K) & (n <= rem)
        cut = active & ~fits & (rem <= n)
        more = active & ~fits & ~cut
        done |= fits
        j = np.clip(np.where(cut, rem, K) - 1, 0, None)[:, :, None]
        pick_hi = np.take_along_axis(np.take_along_axis(g_hi, order, axis=2), j, axis=2)[:, :, 0]
        pick_lo = np.take_along_axis(np.take_along_axis(g_lo, order, axis=2), j, axis=2)[:, :, 0]
        upd = cut | more
        th_hi[upd], th_lo[upd] = pick_hi[upd], pick_lo[upd]
        bounded |= more
        rem[cut] = 0
        rem[more] -= K
    for i, rows in enumerate(members):
        h, l = hi[rows], lo[rows]
        at_or_above = (h > th_hi[i]) | ((h == th_hi[i]) & (l >= th_lo[i]))
        kept[rows] = ok[rows] & np.where(done[i], True, at_or_above)
    return kept, X, rounds, K


def partial_state_host(agg: str, vals: np.ndarray, valid: np.ndarray, gid: np.ndarray, n_groups: int):
    """Host mirror of b2p_group_aggregate_partial_dev for stddev / stdvar: (M2, cnt, mean) per (group, step), Welford in
    series order like the by-label kernel."""
    S, T = vals.shape
    Tw = valid.shape[1]
    m2 = np.zeros((n_groups, T))
    mean = np.zeros((n_groups, T))
    cnt = np.zeros((n_groups, T), np.int64)
    bits = ((valid[:, :, None] >> np.arange(32, dtype=np.uint32)) & 1).reshape(S, Tw * 32)[:, :T].astype(bool)
    for s in range(S):
        g = int(gid[s])
        if g >= n_groups:
            continue
        k = np.flatnonzero(bits[s])
        x = vals[s, k]
        n1 = cnt[g, k] + 1.0
        d1 = x - mean[g, k]
        nm = d1 / n1 + mean[g, k]
        m2[g, k] += d1 * (x - nm)
        mean[g, k] = nm
        cnt[g, k] += 1
    return m2, cnt, mean


QUANT_SHARD_PASSES = 17                       # sixteen 4-bit digits, then one extreme pass
QUANT_UNIT_BYTES = 16 * 32 * 4 + 2 * 32 * 8   # block bytes per (group, 32-step tile) and pass


def merge_quantile_digits(phi, vals: np.ndarray, ok: np.ndarray, gid: np.ndarray, n_groups: int, group=None):
    """Host mirror of b2p_quantile_allreduce_dev (same select, torch.distributed instead of the library's NCCL
    communicator; used by the gloo tests): this rank's rows [R, T] (ok: valid cells, gid >= n_groups: no group) ->
    (out [G, T] f64, cnt [G, T] u32, passes run, block bytes sent), the same on every rank.
      - per (group, step) the state is a prefix of `level` fixed 4-bit digits of the key u = total_key ^ 2^63 and lo's
        rank k among the keys under it; each pass every rank counts the next digit of its keys under the prefix (16
        bins), or takes its largest key under p_lo and smallest under p_hi (the extreme pass);
      - the counts are all-reduced by SUM as int64, the extremes by MAX / MIN as int64 after XOR with 2^63 (which keeps
        the unsigned order), and every rank advances the same state from the merged block;
      - the passes stop when no cell is left, at most 17; phi outside [0, 1] or NaN stops after the count."""
    import math
    import torch
    import torch.distributed as dist
    sign, full = np.uint64(1 << 63), np.uint64(0xFFFFFFFFFFFFFFFF)
    vals = np.ascontiguousarray(vals, np.float64)
    R, T = vals.shape
    G = int(n_groups)
    out = np.zeros((G, T), np.float64)
    cnt = np.zeros((G, T), np.uint32)
    if G == 0 or T == 0:
        return out, cnt, 0, 0
    keys = _key(vals)
    gid = np.asarray(gid, np.int64)
    rr, rt = np.nonzero(np.asarray(ok, bool) & (gid < G)[:, None])
    rg, rk = gid[rr], keys[rr, rt]
    count_only = not (0.0 <= phi <= 1.0)
    mode = np.zeros((G, T), np.int64)             # 0 select, 1 extreme, 2 done
    level = np.zeros((G, T), np.int64)
    k = np.zeros((G, T), np.int64)
    eq = np.zeros((G, T), bool)
    p_lo = np.zeros((G, T), np.uint64)
    p_hi = np.zeros((G, T), np.uint64)

    def under(p, lv):
        sh = np.minimum(64 - 4 * lv, 63).astype(np.uint64)
        return (lv == 0) | ((rk >> sh) == (p >> sh))

    passes = 0
    for _ in range(QUANT_SHARD_PASSES):
        passes += 1
        cm, lv = mode[rg, rt], level[rg, rt]
        sel = (cm == 0) & under(p_lo[rg, rt], lv)
        dig = ((rk >> np.maximum(60 - 4 * lv, 0).astype(np.uint64)) & np.uint64(15)).astype(np.int64)
        hist = np.zeros((G, T, 16), np.int64)
        np.add.at(hist, (rg[sel], rt[sel], dig[sel]), 1)
        lo_m = (cm == 1) & under(p_lo[rg, rt], lv)
        hi_m = (cm == 1) & ~eq[rg, rt] & under(p_hi[rg, rt], lv)
        r_lo = np.zeros((G, T), np.uint64)
        r_hi = np.full((G, T), full, np.uint64)
        np.maximum.at(r_lo, (rg[lo_m], rt[lo_m]), rk[lo_m])
        np.minimum.at(r_hi, (rg[hi_m], rt[hi_m]), rk[hi_m])
        h_t = torch.from_numpy(hist)
        lo_t = torch.from_numpy((r_lo ^ sign).view(np.int64))
        hi_t = torch.from_numpy((r_hi ^ sign).view(np.int64))
        dist.all_reduce(h_t, op=dist.ReduceOp.SUM, group=group)
        dist.all_reduce(lo_t, op=dist.ReduceOp.MAX, group=group)
        dist.all_reduce(hi_t, op=dist.ReduceOp.MIN, group=group)
        hist = h_t.numpy()
        r_lo = lo_t.numpy().view(np.uint64) ^ sign
        r_hi = hi_t.numpy().view(np.uint64) ^ sign
        for g, t in zip(*np.nonzero(mode != 2)):
            if mode[g, t] == 1:                   # the extremes are s[lo] and s[hi]
                p_lo[g, t] = r_lo[g, t]
                p_hi[g, t] = r_lo[g, t] if eq[g, t] else r_hi[g, t]
                mode[g, t] = 2
                continue
            bins = [int(c) for c in hist[g, t]]
            if level[g, t] == 0:
                n = sum(bins)
                cnt[g, t] = n
                if n == 0 or count_only:
                    mode[g, t] = 2
                    continue
                k[g, t] = min(math.floor(phi * float(n - 1)), n - 1)
                if k[g, t] == n - 1:              # hi = lo: the largest key
                    mode[g, t], eq[g, t] = 1, True
                    continue
            kk, cum, blo, bhi, klo = int(k[g, t]), 0, 16, 15, 0
            for b, c in enumerate(bins):
                if blo == 16 and cum + c > kk:
                    blo, klo = b, kk - cum
                if cum + c > kk + 1:
                    bhi = b
                    break
                cum += c
            shift = np.uint64(60 - 4 * int(level[g, t]))
            p_hi[g, t] = p_lo[g, t] | (np.uint64(bhi) << shift)
            p_lo[g, t] |= np.uint64(blo) << shift
            k[g, t] = klo
            level[g, t] += 1
            if blo == bhi:
                if level[g, t] == 16:
                    p_hi[g, t] = p_lo[g, t]
                    mode[g, t] = 2
            else:
                mode[g, t] = 2 if level[g, t] == 16 else 1
        if (mode != 2).sum() == 0:
            break
    has = cnt > 0
    if count_only:
        out[has] = np.nan if math.isnan(phi) else (-np.inf if phi < 0 else np.inf)
    else:  # s[lo] (1 - w) + s[hi] w, each operation rounded (no FMA), one group's row at a time
        for g in range(G):
            rank = np.float64(phi) * (np.maximum(cnt[g], 1) - 1).astype(np.float64)
            w = rank - np.floor(rank)
            with np.errstate(invalid="ignore", over="ignore"):
                res = _value(p_lo[g]) * (np.float64(1.0) - w) + _value(p_hi[g]) * w
            out[g] = np.where(has[g], res, 0.0)
    return out, cnt, passes, passes * G * ((T + 31) // 32) * QUANT_UNIT_BYTES


CV_ENTRY_BYTES = 12                           # one (key u64, count u32) entry of a count_values block


def merge_count_values(vals: np.ndarray, cnt: np.ndarray, gid: np.ndarray, n_groups: int, group=None):
    """Host mirror of b2p_count_values_allgather_dev (same exchange, torch.distributed instead of the library's NCCL
    communicator; used by the gloo tests): this rank's count_values output (vals / cnt [R, T], rows in member order:
    rows stably sorted by gid, rows of gid >= n_groups last) -> (out [U, T] f64, cnt [U, T] u32, out_goff [G + 1],
    block bytes sent), the same on every rank.
      - h_r(g) = the number of leading rows of group g with a count at some step; the heights are all-gathered and
        group g gets U_g = sum over ranks of h_r(g) rows from out_goff[g];
      - each rank sends the first h_r(g) rows of each group as (key u64, count u32) entries, a cell without a count as
        the largest key with count 0, padded to the largest rank's rows; the blocks are all-gathered;
      - per (group, step) the entries of every rank are sorted by key, each run of equal keys is one value with the sum
        of its counts, and a run whose counts add up to 0 is no value."""
    import torch.distributed as dist
    world = dist.get_world_size(group)
    vals = np.ascontiguousarray(vals, np.float64)
    cnt = np.asarray(cnt, np.uint32)
    R, T = vals.shape
    G = int(n_groups)
    gid = np.asarray(gid, np.int64)
    goff = np.searchsorted(np.sort(gid), np.arange(G + 1))
    has = (cnt != 0).any(axis=1) if T else np.zeros(R, bool)
    h = np.zeros(G, np.int64)
    for g in range(G):
        rows = np.flatnonzero(has[goff[g]:goff[g + 1]])
        h[g] = rows[-1] + 1 if rows.size else 0
    parts = _all_gather(h, group)
    heights = np.stack(parts) if G else np.zeros((world, 0), np.int64)
    U = heights.sum(axis=0)
    out_goff = np.concatenate([[0], np.cumsum(U)]).astype(np.int64)
    P = int(heights.sum(axis=1).max()) if G else 0
    keys = _key(vals)
    mine = np.concatenate([np.arange(goff[g], goff[g] + h[g]) for g in range(G)] + [np.zeros(0, np.int64)])
    s_key = np.full((P, T), np.uint64(0xFFFFFFFFFFFFFFFF), np.uint64)
    s_cnt = np.zeros((P, T), np.int64)
    s_key[:mine.size] = np.where(cnt[mine] != 0, keys[mine], np.uint64(0xFFFFFFFFFFFFFFFF))
    s_cnt[:mine.size] = cnt[mine]
    got = [_all_gather(a, group) for a in (s_key.view(np.int64), s_cnt)]
    e_g, e_k, e_key, e_cnt = [], [], [], []
    for r in range(world):
        row_g = np.repeat(np.arange(G), heights[r])
        e_g.append(np.repeat(row_g, T))
        e_k.append(np.tile(np.arange(T), row_g.size))
        e_key.append(got[0][r][:row_g.size].view(np.uint64).reshape(-1))
        e_cnt.append(got[1][r][:row_g.size].reshape(-1))
    e_g, e_k, e_key, e_cnt = (np.concatenate(x) for x in (e_g, e_k, e_key, e_cnt))
    U_all = int(out_goff[-1])
    out_v = np.zeros((U_all, T), np.float64)
    out_c = np.zeros((U_all, T), np.uint32)
    if e_g.size:
        order = np.lexsort((e_key, e_k, e_g))
        g_s, k_s, key_s, c_s = e_g[order], e_k[order], e_key[order], e_cnt[order]
        head = np.ones(g_s.size, bool)
        head[1:] = (g_s[1:] != g_s[:-1]) | (k_s[1:] != k_s[:-1]) | (key_s[1:] != key_s[:-1])
        starts = np.flatnonzero(head)
        sums = np.add.reduceat(c_s, starts)
        keep = starts[sums > 0]
        sums = sums[sums > 0]
        g_r, k_r = g_s[keep], k_s[keep]
        seg = g_r * T + k_r
        first = np.searchsorted(seg, seg)              # each (group, step)'s first value
        j = np.arange(seg.size) - first
        u = key_s[keep]
        out_v[out_goff[g_r] + j, k_r] = _value(u)
        out_c[out_goff[g_r] + j, k_r] = sums
    return out_v, out_c, out_goff, P * T * CV_ENTRY_BYTES


def merge_sorted_runs(desc: bool, vals, ok: np.ndarray, row_id: np.ndarray, group=None):
    """Host mirror of b2p_sort_cells_allgather_dev (same blocks, torch.distributed instead of the library's NCCL
    communicator; used by the gloo tests): this rank's grid vals [R, T] (float64, or int64 for the Int64 form; a
    sequence of F float64 grids for several fields), ok [R, T] bool and row_id [R] (strictly increasing, distinct
    across ranks) -> (global cells u64 [N], values [N] (a list of F arrays for several fields), bytes sent), the same on
    every rank.
      - each rank's valid cells become (key of field 0 .. F-1, global cell row_id[r] * T + k) entries, the key
        total_key ^ 2^63 (Int64: bits ^ 2^63), inverted for desc, sorted: its run;
      - the counts are all-gathered, every run is padded to the largest and all-gathered;
      - the runs are merged by (keys, cell) ascending, and the values decoded from the keys."""
    many = isinstance(vals, (list, tuple))
    grids = [np.asarray(v) for v in vals] if many else [np.asarray(vals)]
    i64 = grids[0].dtype == np.int64
    ok = np.asarray(ok, bool)
    R, T = ok.shape
    F = len(grids)
    row_id = np.asarray(row_id, np.uint64)
    if R > 1 and not (row_id[1:] > row_id[:-1]).all():
        raise ValueError("row_id must be strictly increasing along the rank's rows")
    sign = np.uint64(1 << 63)
    flip = np.uint64(0xFFFFFFFFFFFFFFFF) if desc else np.uint64(0)
    cells = np.flatnonzero(ok.reshape(-1)).astype(np.uint64)
    keys = []
    for g in grids:
        b = np.ascontiguousarray(g).reshape(-1)[cells]
        k = b.view(np.uint64) ^ sign if i64 else _key(b)
        keys.append(k ^ flip)
    glob = row_id[cells // np.uint64(T)] * np.uint64(T) + cells % np.uint64(T) if T else cells
    ns = [int(x[0]) for x in _all_gather(np.array([cells.size], np.int64), group)]
    P = max(ns)
    block = np.zeros((F + 1, P), np.uint64)
    if cells.size:
        order = np.lexsort([glob] + keys[::-1])
        block[:F, :cells.size] = np.stack(keys)[:, order]
        block[F, :cells.size] = glob[order]
    got = _all_gather(block.view(np.int64), group)
    runs = np.concatenate([g.view(np.uint64)[:, :m] for g, m in zip(got, ns)], axis=1)
    merged = runs[:, np.lexsort([runs[F]] + [runs[f] for f in range(F - 1, -1, -1)])]
    out = []
    for f in range(F):
        u = merged[f] ^ flip
        out.append((u ^ sign).view(np.int64) if i64 else _value(u))
    return merged[F].copy(), (out if many else out[0]), int(cells.size) * 8 * (F + 1)


# ---- group-label agreement of a sharded plan node (b2p_plan_set_sharded; block layout of b2p_group_keys_merge) ----
GK_NULL = 0xFFFFFFFF   # the length tag of a NULL label
GK_FLAG_TSID = 1       # every group carries its u64 __tsid


def label_order_key(v):
    """The plan layer's order of one label value (Labels::less): "" first, then NULL, then the other strings by their
    UTF-8 bytes."""
    if v is None:
        return (1, b"")
    return (0, b"") if v == "" else (2, v.encode())


def tuple_order_key(t):
    return tuple(label_order_key(v) for v in t)


def group_tuples(tuples):
    """group_rows' table over rows labelled `tuples` (each a tuple of str / None): the distinct tuples in label order."""
    return sorted(set(tuple(t) for t in tuples), key=tuple_order_key)


def serialize_group_keys(tuples, n_labels: int, ids=None, n_rows=None, types=()) -> bytes:
    """One rank's block: its groups (distinct, in label order) with their __tsid when `ids` is given, its row count
    (default: one per group; 0 exactly when there is no group) and its field types (0 Float64, 1 Int64, 2 Int32,
    3 a count)."""
    import struct
    n_rows = len(tuples) if n_rows is None else n_rows
    out = [struct.pack("<IIIIQ", len(tuples), n_labels, GK_FLAG_TSID if ids is not None else 0, len(types), n_rows),
           bytes(bytearray(types))]
    for g, t in enumerate(tuples):
        if ids is not None:
            out.append(struct.pack("<Q", int(ids[g])))
        for v in t:
            if v is None:
                out.append(struct.pack("<I", GK_NULL))
            else:
                b = v.encode()
                out.append(struct.pack("<I", len(b)) + b)
    return b"".join(out)


def parse_group_keys(buf: bytes):
    """-> (tuples, ids or None, n_labels, n_rows, types) of one block"""
    import struct
    G, L, flags, F, n_rows = struct.unpack_from("<IIIIQ", buf, 0)
    types = tuple(buf[24:24 + F])
    at, tuples, ids = 24 + F, [], [] if flags & GK_FLAG_TSID else None
    for _ in range(G):
        if ids is not None:
            ids.append(struct.unpack_from("<Q", buf, at)[0])
            at += 8
        t = []
        for _ in range(L):
            n = struct.unpack_from("<I", buf, at)[0]
            at += 4
            if n == GK_NULL:
                t.append(None)
            else:
                t.append(bytes(buf[at:at + n]).decode())
                at += n
        tuples.append(tuple(t))
    assert at == len(buf), "block longer than its groups"
    return tuples, ids, L, n_rows, types


def merge_group_keys(blocks, rank: int):
    """Host mirror of b2p_group_keys_merge: the R-way merge of the blocks (rank order) into the global table without
    duplicates (a duplicate keeps the lowest rank's id) -> (table tuples, table ids or None, local_to_global of block
    `rank`, rows of all blocks, the field types of the blocks with rows)."""
    parsed = [parse_group_keys(b) for b in blocks]
    typed = [p[4] for p in parsed if p[3]]
    assert all(t == typed[0] for t in typed), "the ranks with rows read different value types"
    types = typed[0] if typed else parsed[0][4]
    heads = [0] * len(parsed)
    table, ids, l2g = [], [] if parsed[0][1] is not None else None, [0] * len(parsed[rank][0])
    while True:
        m = None
        for r, p in enumerate(parsed):
            t = p[0]
            if heads[r] < len(t) and (m is None or tuple_order_key(t[heads[r]]) < tuple_order_key(parsed[m][0][heads[m]])):
                m = r
        if m is None:
            return table, ids, l2g, sum(p[3] for p in parsed), types
        t = parsed[m][0][heads[m]]
        if ids is not None:
            ids.append(parsed[m][1][heads[m]])
        for r, p in enumerate(parsed):
            ts = p[0]
            if heads[r] < len(ts) and ts[heads[r]] == t:
                if r == rank:
                    l2g[heads[r]] = len(table)
                heads[r] += 1
        table.append(t)


def agree_group_keys(tuples, n_labels: int, ids=None, group=None):
    """Host mirror of a sharded node's group-label agreement (the same exchange as b2p_group_keys_sizes /
    b2p_group_keys_allgather, torch.distributed instead of the library's NCCL communicator; used by the gloo tests):
    this rank's groups (distinct, label order, with their __tsid when `ids` is given) -> (global table, its ids or
    None, local_to_global, this rank's block bytes), the same table on every rank.  One all-gather of the 8-byte block
    sizes, then one broadcast per rank with bytes."""
    import torch
    import torch.distributed as dist
    me = dist.get_rank(group)
    mine = serialize_group_keys(tuples, n_labels, ids)  # (no field types: the mirror agrees the labels)
    blocks = []
    for r, n in enumerate(int(s[0]) for s in _all_gather(np.array([len(mine)], np.int64), group)):
        buf = torch.frombuffer(bytearray(mine), dtype=torch.uint8) if r == me else torch.zeros(n, dtype=torch.uint8)
        if n:
            dist.broadcast(buf, src=r, group=group)
        blocks.append(buf.numpy().tobytes())
    table, table_ids, l2g, _, _ = merge_group_keys(blocks, me)
    return table, table_ids, l2g, len(mine)


HIST_HEADER_BYTES = 24  # (bound f64, histogram u32, rank u32, row u32, pad u32) with each shuffled bucket row


def histogram_owners(counts):
    """The owner of each histogram from the counts table [n_ranks, n_hist]: the rank with the most of its buckets, the
    lowest on a tie (b2p_histogram_shard_owners)"""
    counts = np.asarray(counts)
    return np.argmax(counts, axis=0).astype(np.int64) if counts.size else np.zeros(counts.shape[1], np.int64)


def _fold_cells(phi, bounds, counters):
    """K5 over one (histogram, step): the present buckets' bounds (ascending, NaN last) and counters -> its value
    (None: no bucket present)"""
    import math
    n = len(bounds)
    if n == 0:
        return None
    if n < 2 or not (math.isinf(bounds[-1]) and bounds[-1] > 0):
        return math.nan
    cnt, prev = [], 0.0
    for i, v in enumerate(counters):  # non-finite -> previous, decreasing -> previous (histogram_fold.rs:1074-1092)
        c = v if math.isfinite(v) else prev
        if i > 0 and c < prev:
            c = prev
        prev = c
        cnt.append(c)
    if phi < 0:
        return -math.inf
    if phi > 1:
        return math.inf
    if math.isnan(phi) or not all(a <= b for a, b in zip(bounds, bounds[1:])):
        return math.nan
    expected = cnt[-1] * phi
    fit = next((i for i, c in enumerate(cnt) if not c < expected), n)  # n: no counter reaches it (negative counters)
    if fit >= n - 1:
        return bounds[n - 2]
    uc, ub = cnt[fit], bounds[fit]
    lb, lc = (0.0 if math.isnan(bounds[0]) else min(bounds[0], 0.0)), 0.0  # f64::min ignores NaN
    if fit > 0:
        lb, lc = bounds[fit - 1], cnt[fit - 1]
    if abs(uc - lc) < 1e-10:
        return math.nan
    return lb + (ub - lb) / (uc - lc) * (expected - lc)


def histogram_fold_sharded(phi, rates, ok, row_hist, row_le, n_hist: int, group=None):
    """Host mirror of b2p_histogram_fold_allgather (the same owners and shuffle, torch.distributed instead of the
    library's NCCL communicator; used by the gloo tests): this rank's bucket rows rates / ok [R, T] (ok: the cell has a
    value), each row's global histogram id row_hist [R] and parsed bound row_le [R] -> (out [n_hist, T] f64,
    ok [n_hist, T] bool, bytes this rank sent), the same on every rank.
      - each rank's bucket count per histogram is all-gathered; a histogram's owner is the rank with the most of them,
        the lowest on a tie;
      - each rank sends its rows of histograms it does not own, with their headers (bound, histogram, rank, row), to
        the owner (here: an all-gather of every rank's sent rows, padded to the largest, from which each owner takes its
        own);
      - the owner folds each of its histograms over its buckets ordered by (bound ascending, NaN last, rank, row);
      - every owner's results are all-gathered and placed in histogram order."""
    import torch.distributed as dist
    world, me = dist.get_world_size(group), dist.get_rank(group)
    rates = np.ascontiguousarray(rates, np.float64)
    ok = np.asarray(ok, bool)
    R, T = rates.shape
    H = int(n_hist)
    Tw = (T + 31) // 32
    row_hist = np.asarray(row_hist, np.int64)
    row_le = np.asarray(row_le, np.float64)
    counts = np.stack(_all_gather(np.bincount(row_hist, minlength=H).astype(np.int64), group))
    owner = histogram_owners(counts)
    mine = np.flatnonzero(owner[row_hist] == me) if R else np.zeros(0, np.int64)
    sent = np.flatnonzero(owner[row_hist] != me) if R else np.zeros(0, np.int64)
    sent = sent[np.lexsort((sent, row_hist[sent]))] if sent.size else sent
    P = int(max(_all_gather(np.array([sent.size], np.int64), group))[0])
    s_val, s_ok, s_hdr = np.zeros((P, T)), np.zeros((P, T), bool), np.full((P, 3), -1, np.int64)
    s_le = np.zeros(P)
    s_val[:sent.size], s_ok[:sent.size], s_le[:sent.size] = rates[sent], ok[sent], row_le[sent]
    s_hdr[:sent.size] = np.stack([row_hist[sent], np.full(sent.size, me), sent], axis=1)
    got = [_all_gather(a, group) for a in (s_val, s_ok, s_le, s_hdr)]
    # the owner's buckets: (histogram, bound, rank, row, values, cells)
    buckets = [(int(row_hist[i]), float(row_le[i]), me, int(i), rates[i], ok[i]) for i in mine]
    for r in range(world):
        for j in range(P):
            h, src, row = (int(x) for x in got[3][r][j])
            if h >= 0 and owner[h] == me:
                buckets.append((h, float(got[2][r][j]), src, row, got[0][r][j], got[1][r][j]))
    buckets.sort(key=lambda b: (b[0], np.isnan(b[1]), 0.0 if np.isnan(b[1]) else b[1], b[2], b[3]))
    own = np.flatnonzero(owner == me)
    o_val, o_ok = np.zeros((own.size, T)), np.zeros((own.size, T), bool)
    place = {int(h): i for i, h in enumerate(own)}
    by_hist = {}
    for b in buckets:
        by_hist.setdefault(b[0], []).append(b)
    for h, bs in by_hist.items():
        for k in range(T):
            present = [b for b in bs if b[5][k]]
            v = _fold_cells(phi, [b[1] for b in present], [float(b[4][k]) for b in present])
            if v is not None:
                o_val[place[h], k], o_ok[place[h], k] = v, True
    n_own = np.bincount(owner, minlength=world)
    Q = int(n_own.max()) if H else 0
    p_val, p_ok = np.zeros((Q, T)), np.zeros((Q, T), bool)
    p_val[:own.size], p_ok[:own.size] = o_val, o_ok
    all_val, all_ok = _all_gather(p_val, group), _all_gather(p_ok, group)
    out, out_ok = np.zeros((H, T)), np.zeros((H, T), bool)
    for r in range(world):
        hs = np.flatnonzero(owner == r)
        out[hs], out_ok[hs] = all_val[r][:hs.size], all_ok[r][:hs.size]
    return out, out_ok, sent.size * (8 * T + 4 * Tw + HIST_HEADER_BYTES) + own.size * (8 * T + 4 * Tw)
