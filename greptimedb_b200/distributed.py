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
    b = np.ascontiguousarray(vals, np.float64).view(np.uint64)
    hi = np.where(b >> np.uint64(63) != 0, ~b, b | np.uint64(1 << 63))
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
    world = dist.get_world_size(group)
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
        parts = []
        for t in (torch.from_numpy(s_hi.view(np.int64)), torch.from_numpy(s_lo.astype(np.int64)), torch.from_numpy(s_n)):
            out = [torch.empty_like(t) for _ in range(world)]
            dist.all_gather(out, t, group=group)
            parts.append([o.numpy() for o in out])
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
    bits = vals.view(np.uint64)
    keys = np.where(bits >> np.uint64(63) != 0, ~bits, bits | sign)
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

    def value(u):  # keys -> f64
        return np.ascontiguousarray(np.where(u >> np.uint64(63) != 0, u ^ sign, ~u), np.uint64).view(np.float64)

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
                res = value(p_lo[g]) * (np.float64(1.0) - w) + value(p_hi[g]) * w
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
    import torch
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
    parts = [torch.empty(G, dtype=torch.int64) for _ in range(world)]
    dist.all_gather(parts, torch.from_numpy(h.copy()), group=group)
    heights = np.stack([p.numpy() for p in parts]) if G else np.zeros((world, 0), np.int64)
    U = heights.sum(axis=0)
    out_goff = np.concatenate([[0], np.cumsum(U)]).astype(np.int64)
    P = int(heights.sum(axis=1).max()) if G else 0
    bits = vals.view(np.uint64)
    keys = np.where(bits >> np.uint64(63) != 0, ~bits, bits | np.uint64(1 << 63))
    mine = np.concatenate([np.arange(goff[g], goff[g] + h[g]) for g in range(G)] + [np.zeros(0, np.int64)])
    s_key = np.full((P, T), np.uint64(0xFFFFFFFFFFFFFFFF), np.uint64)
    s_cnt = np.zeros((P, T), np.int64)
    s_key[:mine.size] = np.where(cnt[mine] != 0, keys[mine], np.uint64(0xFFFFFFFFFFFFFFFF))
    s_cnt[:mine.size] = cnt[mine]
    got = []
    for t in (torch.from_numpy(s_key.view(np.int64)), torch.from_numpy(s_cnt)):
        out = [torch.empty_like(t) for _ in range(world)]
        dist.all_gather(out, t, group=group)
        got.append([o.numpy() for o in out])
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
        out_v[out_goff[g_r] + j, k_r] = np.where(u >> np.uint64(63) != 0, u ^ np.uint64(1 << 63), ~u).view(np.float64)
        out_c[out_goff[g_r] + j, k_r] = sums
    return out_v, out_c, out_goff, P * T * CV_ENTRY_BYTES
