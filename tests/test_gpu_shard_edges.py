"""GPU: the sharded exchange kernels at their layout edges (tests/shard_edges.py), R ranks simulated on one GPU
through the step entry points with torch copies in place of the collectives.

  sort:          every merge tile size (items 8 .. 1, F up to 64), 1 .. 17 runs (rounds 1 .. 5) with empty ranks
                 first, in the middle and last, runs of 1, cap - 1, cap, cap + 1 and 2 cap + 1 entries; the merge's
                 cells and values against np.lexsort over (keys, cell) and the single-rank sort, its launches against
                 the round count.
  count_values:  1 .. 33 ranks, groups on one rank only, full heights, empty groups, U = 1, ~0 keys beside the
                 fillers, under three exchange caps (one window; windows of 32 steps; one group per batch); both merge
                 orders against select_keys and the single-rank count, the plan against its Python restatement.
  topk:          5 and 16 ranks, kk 1 .. 97 (one to four rounds), every cut_batches branch; both directions against
                 select_keys.topk and the single-rank topk, the plan against its Python restatement.
  quantile:      5 and 16 ranks, groups on one rank, on all but one and one per rank, one (group, tile) unit per batch;
                 against select_keys.quantile and the single-rank quantile, every batch ending with no live cell.

Every output starts as a sentinel and has a guard tail that must stay untouched; everything is compared by bits.
Contexts come from one module pool of 17 (rank r on context r mod 16, the merge and the single-rank call on the
17th), remade only when the exchange cap under test changes."""
import math

import numpy as np
import pytest

from tests import select_keys as sk
from tests import shard_edges as se

pytestmark = pytest.mark.gpu

GUARD = 64
SENTINEL = 0x7FF80000DEADBEEF  # a NaN no kernel writes
WORD_SENTINEL = 0x5A5A5A5A
PASSES = 17


def dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


class Pool:
    SIZE = 17

    def __init__(self):
        self.cap, self.ctxs = None, []

    def get(self, cap=se.DEFAULT_CAP):
        if cap != self.cap:
            from greptimedb_b200 import Context
            self.close()
            with pytest.MonkeyPatch.context() as mp:
                if cap == se.DEFAULT_CAP:
                    mp.delenv("B2P_TOPK_EXCHANGE_BYTES", raising=False)
                else:
                    mp.setenv("B2P_TOPK_EXCHANGE_BYTES", str(cap))
                self.ctxs = [Context(0) for _ in range(self.SIZE)]
            for c in self.ctxs:
                c.use_torch_stream()
            self.cap = cap
        return self.ctxs

    def close(self):
        for c in self.ctxs:
            c.close()
        self.cap, self.ctxs = None, []


@pytest.fixture(scope="module")
def pool():
    p = Pool()
    yield p
    p.close()


def rank_ctx(ctxs, r):
    return ctxs[r % (len(ctxs) - 1)]


def tail_ok(t, n):
    a = np.ascontiguousarray(t.cpu().numpy()).view(np.uint64 if t.element_size() == 8 else np.uint32)
    want = SENTINEL if t.element_size() == 8 else WORD_SENTINEL
    return bool((a[n:] == a.dtype.type(want)).all()) and a.size == n + GUARD


def guarded(n, dtype):
    import torch
    if dtype == torch.int32:
        return torch.full((n + GUARD,), WORD_SENTINEL, dtype=torch.int32, device="cuda")
    return torch.full((n + GUARD,), np.uint64(SENTINEL).view(np.int64).item(), dtype=torch.int64,
                      device="cuda").view(dtype)


# ---- sort -------------------------------------------------------------------------------------------------------------
def check_sort(ctxs, case):
    import torch
    F, counts, desc, i64 = case["F"], case["counts"], case["desc"], case["keys"] == "i64"
    grids, ok, owner = se.sort_grid(case)
    T = ok.shape[1]
    valid = sk.words(ok)
    blocks = []
    for r, c in enumerate(counts):
        ctx = rank_ctx(ctxs, r)
        rows = np.flatnonzero(owner == r)
        n = max(rows.size, 1)
        pad = lambda a: np.concatenate([a[rows], np.zeros((n - rows.size,) + a.shape[1:], a.dtype)])
        vs = [dev(pad(g)) for g in grids]
        w = dev(pad(valid).view(np.int32))
        rid = dev(pad(np.arange(owner.size, dtype=np.int32)))
        assert int(ctx.sort_shard_counts_dev(w, rows.size, T)[0]) == c
        blk = torch.full((max(c * (F + 1), 1),), -1, dtype=torch.int64, device="cuda")
        ctx.sort_shard_pack_dev(desc, vs[0] if F == 1 else vs, w, rid, rows.size, T, c, blk, i64=i64)
        blocks.append(blk[:c * (F + 1)])
    N = sum(counts)
    m = ctxs[-1]
    laid = torch.cat(blocks + [torch.zeros(1, dtype=torch.int64, device="cuda")])
    cells = guarded(N, torch.int64)
    outs = [guarded(N, torch.int64 if i64 else torch.float64) for _ in range(F)]
    before = m.launch_count()
    m.sort_shard_merge_dev(desc, counts, laid, cells, outs if F > 1 else outs[0], i64=i64)
    torch.cuda.synchronize()
    what = (F, counts, case["keys"], desc)
    assert m.launch_count() - before == len(se.merge_rounds(counts, se.sort_cap(F))), what
    exp = se.sort_ref(desc, grids, ok, i64)
    assert tail_ok(cells, N) and all(tail_ok(o, N) for o in outs), what
    got = cells.cpu().numpy()[:N].view(np.uint64)
    assert np.array_equal(got, exp), what
    for g, o in zip(grids, outs):
        want = np.ascontiguousarray(g).reshape(-1)[exp.astype(np.int64)].view(np.uint64)
        assert np.array_equal(o.cpu().numpy()[:N].view(np.uint64), want), what
    # the single-rank sort over the concatenation
    one = torch.full((max(ok.size, 1),), -1, dtype=torch.int64, device="cuda")
    n1 = torch.zeros(1, dtype=torch.int64, device="cuda")
    vs, w = [dev(g) for g in grids], dev(valid.view(np.int32))
    if i64:
        m.sort_cells_i64_dev(desc, vs[0], w, ok.shape[0], T, one, n1)
    elif F > 1:
        m.sort_cells_fields_dev(desc, vs, w, ok.shape[0], T, one, n1)
    else:
        m.sort_cells_dev(desc, vs[0], w, ok.shape[0], T, one, n1)
    torch.cuda.synchronize()
    assert int(n1.item()) == N and np.array_equal(one.cpu().numpy()[:N].view(np.uint64), exp), what


@pytest.mark.parametrize("F", se.SORT_FIELDS)
def test_sort_merge(pool, F):
    ctxs = pool.get()
    for case in se.sort_cases():
        if case["F"] == F:
            check_sort(ctxs, case)


# ---- count_values -------------------------------------------------------------------------------------------------------
def check_count_values(ctxs, cap, R, T, i64, seed):
    import torch
    from greptimedb_b200 import Context
    vals, ok, gid, G, owner = se.cv_grid(R, T, seed, i64)
    valid = sk.words(ok)
    vdt = torch.int64 if i64 else torch.float64
    made = []
    try:
        locs = []
        for r in range(R):
            ctx = rank_ctx(ctxs, r)
            rows = np.flatnonzero(owner == r)
            n = max(rows.size, 1)
            v, w = dev(vals[rows]), dev(valid[rows].view(np.int32))
            ix = ctx.group_index_create_dev(dev(gid[rows].view(np.int32)), rows.size, G)
            made.append((ctx, ix))
            lv = torch.zeros(n * T, dtype=vdt, device="cuda")
            lc = torch.zeros(n * T, dtype=torch.int32, device="cuda")
            if rows.size:
                (ctx.count_values_i64_dev if i64 else ctx.count_values_dev)(v, w, ix, T, lv, lc)
            locs.append((ctx, ix, lv, lc))
        H = np.concatenate([ctx.count_values_shard_heights_dev(lc, ix, T, G) for ctx, ix, _, lc in locs])
        what = (cap, R, T, i64)
        assert np.array_equal(H, se.cv_heights(vals, ok, gid, G, owner, R, i64)), what
        m = ctxs[-1]
        plan = m.count_values_shard_plan(H, T)
        batches = se.cv_plan(H, T, cap)
        assert plan["n_batches"] == len(batches), what
        assert plan["block_bytes"] == max([b[4] for b in batches], default=0) * se.CV_ENTRY, what
        out_goff = Context.count_values_shard_rows(H)
        U = int(out_goff[-1])
        outs = []
        for rot in (0, R // 2):
            order = [(rot + j) % R for j in range(R)]
            ov, oc = guarded(U * T, vdt), guarded(U * T, torch.int32)
            for b, bt in enumerate(batches):
                P = bt[4]
                blks = []
                for o in order:
                    ctx, ix, lv, lc = locs[o]
                    blk = torch.zeros(max(P * se.CV_ENTRY, 16), dtype=torch.uint8, device="cuda")
                    ctx.count_values_shard_pack_dev(lv, lc, ix, T, H, o, b, blk, i64=i64)
                    assert ctx.last_exchange_bytes() == P * se.CV_ENTRY, what
                    blks.append(blk)
                gathered = torch.cat([k[:8 * P] for k in blks] + [k[8 * P:12 * P] for k in blks] +
                                     [torch.zeros(16, dtype=torch.uint8, device="cuda")])
                m.count_values_shard_merge_dev(H[order], T, b, gathered, ov, oc, i64=i64)
            torch.cuda.synchronize()
            assert tail_ok(ov, U * T) and tail_ok(oc, U * T), what
            outs.append((ov.cpu().numpy()[:U * T].reshape(U, T), oc.cpu().numpy()[:U * T].view(np.uint32).reshape(U, T)))
        exp, exp_cnt = se.cv_ref(vals, ok, gid, G, i64)
        full = m.group_index_create_dev(dev(gid.view(np.int32)), gid.size, G)
        made.append((m, full))
        one = torch.zeros(gid.size * T, dtype=vdt, device="cuda")
        one_cnt = torch.zeros(gid.size * T, dtype=torch.int32, device="cuda")
        (m.count_values_i64_dev if i64 else m.count_values_dev)(dev(vals), dev(valid.view(np.int32)), full, T, one,
                                                                one_cnt)
        torch.cuda.synchronize()
        one = one.cpu().numpy().reshape(-1, T)
        one_cnt = one_cnt.cpu().numpy().view(np.uint32).reshape(-1, T)
        assert sk.same_bits(one.view(np.float64), exp.view(np.float64)) and (one_cnt == exp_cnt).all(), what
        _, goff = sk._groups(gid, G)
        for out, cnt in outs:
            for g in range(G):
                u = out_goff[g + 1] - out_goff[g]
                a, e = out[out_goff[g]:out_goff[g + 1]], exp[goff[g]:goff[g] + u]
                assert np.array_equal(a.view(np.uint64), np.ascontiguousarray(e).view(np.uint64)), (what, g)
                assert (cnt[out_goff[g]:out_goff[g + 1]] == exp_cnt[goff[g]:goff[g] + u]).all(), (what, g)
                assert (exp_cnt[goff[g] + u:goff[g + 1]] == 0).all(), (what, g)
    finally:
        for ctx, ix in made:
            ctx.group_index_destroy(ix)


@pytest.mark.parametrize("i64", [False, True])
@pytest.mark.parametrize("cap", se.CV_CAPS)
def test_count_values_merge(pool, cap, i64):
    ctxs = pool.get(cap)
    for s, (R, T) in enumerate(se.cv_cases(cap)):
        check_count_values(ctxs, cap, R, T, i64, s)


# ---- topk / bottomk ------------------------------------------------------------------------------------------------------
def run_topk(ctxs, ranks, op, kk, sizes, T):
    import torch
    R = len(ranks)
    m = ctxs[-1]
    plan = m.topk_shard_plan(kk, sizes, T, R)
    state = torch.zeros(max(plan["state_bytes"], 16), dtype=torch.uint8, device="cuda")
    blocks = [torch.zeros(max(plan["block_bytes"], 16), dtype=torch.uint8, device="cuda") for _ in ranks]
    outs = [guarded(max(r["n"], 1) * ((T + 31) // 32), torch.int32) for r in ranks]
    K = plan["slots"]
    for b in range(plan["n_batches"]):
        for rnd in range(plan["n_rounds"]):
            nbytes = None
            for r, blk in zip(ranks, blocks):
                r["ctx"].topk_shard_candidates_dev(op, kk, r["vals"], r["valid"], r["ix"], r["tie"], T, sizes, R, b, rnd,
                                                   state, blk)
                got = r["ctx"].last_exchange_bytes()
                assert nbytes in (None, got)
                nbytes = got
            units = nbytes // (32 * (12 * K + 4))
            cuts = np.cumsum([0, units * K * 32 * 8, units * K * 32 * 4, units * 32 * 4])
            gathered = torch.cat([blk[cuts[s]:cuts[s + 1]] for s in range(3) for blk in blocks])
            m.topk_shard_merge_dev(kk, sizes, T, R, b, rnd, gathered, state)
        for r, out in zip(ranks, outs):
            r["ctx"].topk_shard_mark_dev(op, kk, r["vals"], r["valid"], r["ix"], r["tie"], T, sizes, R, b, state, out)
    torch.cuda.synchronize()
    return outs, plan


@pytest.mark.parametrize("case", se.topk_cases(), ids=lambda c: "R%d-kk%d-T%d-%s" % c)
def test_topk_exchange(pool, case):
    import torch
    R, kk, T, branch = case
    vals, ok, gid, G, tie, owner = se.topk_grid(R, kk, T, kk * 1000 + T)
    sizes = np.bincount(gid, minlength=G).astype(np.uint32)
    X, tiles = int((sizes > kk).sum()), (T + 31) // 32
    cap = se.topk_fit(branch, X, tiles) * se.topk_unit(R, kk)
    exp_plan = se.topk_plan(kk, sizes, T, R, cap)
    assert exp_plan["branch"] == branch
    ctxs = pool.get(cap)
    valid = sk.words(ok)
    ranks = []
    try:
        for r in range(R):
            rows = np.flatnonzero(owner == r)
            ctx = ctxs[r]
            ranks.append(dict(ctx=ctx, rows=rows, n=rows.size, vals=dev(vals[rows]),
                              valid=dev(valid[rows].view(np.int32)), tie=dev(tie[rows].view(np.int32)),
                              ix=ctx.group_index_create_dev(dev(gid[rows].view(np.int32)), rows.size, G)))
        m = ctxs[-1]
        full = m.group_index_create_dev(dev(gid.view(np.int32)), gid.size, G)
        try:
            for op in ("topk", "bottomk"):
                outs, plan = run_topk(ctxs, ranks, op, kk, sizes, T)
                assert plan["n_batches"] == exp_plan["n_batches"], (case, plan)
                assert plan["block_bytes"] == exp_plan["block_bytes"], (case, plan)
                assert plan["n_rounds"] == se.topk_rounds(kk)
                Tw = (T + 31) // 32
                union = np.zeros((gid.size, Tw), np.uint32)
                for r, out in zip(ranks, outs):
                    assert tail_ok(out, max(r["n"], 1) * Tw), (case, op)
                    union[r["rows"]] = out.cpu().numpy()[:r["n"] * Tw].view(np.uint32).reshape(r["n"], Tw)
                exp = sk.words(sk.topk(op == "bottomk", kk, vals, ok, gid, G, tie))
                assert (union == exp).all(), (case, op)
                one = torch.full((gid.size * Tw,), -1, dtype=torch.int32, device="cuda")
                m.topk_dev(op, kk, dev(vals), dev(valid.view(np.int32)), full, dev(tie.view(np.int32)), T, one)
                torch.cuda.synchronize()
                assert (one.cpu().numpy().view(np.uint32).reshape(-1, Tw) == exp).all(), (case, op)
        finally:
            m.group_index_destroy(full)
    finally:
        for r in ranks:
            r["ctx"].group_index_destroy(r["ix"])


# ---- quantile ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("unit_batches", [False, True], ids=["one-batch", "unit-batches"])
@pytest.mark.parametrize("T", [33, 65])
@pytest.mark.parametrize("R", [5, 16])
def test_quantile_exchange(pool, R, T, unit_batches):
    import torch
    cap = se.QUANT_UNIT if unit_batches else se.DEFAULT_CAP
    ctxs = pool.get(cap)
    for phi in se.QUANT_PHIS:
        vals, ok, gid, G, owner = se.quant_grid(R, T, phi, R * 100 + T, per_place=1 if unit_batches else 4)
        valid = sk.words(ok)
        what = (R, T, unit_batches, phi)
        exp_plan = se.quant_plan(G, T, cap)
        ranks = []
        try:
            for r in range(R):
                rows = np.flatnonzero(owner == r)
                ctx = ctxs[r]
                ranks.append((ctx, dev(vals[rows]), dev(valid[rows].view(np.int32)),
                              ctx.group_index_create_dev(dev(gid[rows].view(np.int32)), rows.size, G)))
            m = ctxs[-1]
            plan = m.quantile_shard_plan(G, T)
            assert plan["n_batches"] == exp_plan["n_batches"] and plan["block_bytes"] == exp_plan["block_bytes"], what
            if unit_batches:
                assert exp_plan["branch"] == "items" and plan["block_bytes"] == 2560, what
            blocks = [torch.zeros(plan["block_bytes"], dtype=torch.uint8, device="cuda") for _ in ranks]
            outs = [(guarded(G * T, torch.float64), guarded(G * T, torch.int32)) for _ in ranks]
            for b in range(plan["n_batches"]):
                for p in range(PASSES):
                    for (ctx, v, w, ix), blk in zip(ranks, blocks):
                        ctx.quantile_shard_pass_dev(phi, v, w, ix, T, b, p, blk)
                    nbytes = ranks[0][0].last_exchange_bytes()
                    lives = {ctx.quantile_shard_advance_dev(phi, G, T, b, p,
                                                            torch.cat([blocks[(i + j) % R][:nbytes] for j in range(R)]),
                                                            R, ov, oc)
                             for i, ((ctx, _, _, _), (ov, oc)) in enumerate(zip(ranks, outs))}
                    assert len(lives) == 1, what
                    if lives == {0}:
                        break
                else:
                    pytest.fail(f"{what}: batch {b} has live cells after {PASSES} passes")
                if not 0.0 <= phi <= 1.0:
                    assert p == 0, what
            torch.cuda.synchronize()
            exp, exp_cnt = sk.quantile(phi, vals, ok, gid, G)
            full = m.group_index_create_dev(dev(gid.view(np.int32)), gid.size, G)
            one, one_cnt = guarded(G * T, torch.float64), guarded(G * T, torch.int32)
            m.group_quantile_dev(phi, dev(vals), dev(valid.view(np.int32)), full, T, one, one_cnt)
            torch.cuda.synchronize()
            m.group_index_destroy(full)
            one = one.cpu().numpy()[:G * T].reshape(G, T)
            for ov, oc in outs:
                assert tail_ok(ov, G * T) and tail_ok(oc, G * T), what
                out = ov.cpu().numpy()[:G * T].reshape(G, T)
                assert (oc.cpu().numpy()[:G * T].view(np.uint32).reshape(G, T) == exp_cnt).all(), what
                assert sk.same_bits(out, one), what
                assert sk.same_or_nan(out, exp) if math.isnan(phi) else sk.same_bits(out, exp), what
        finally:
            for ctx, _, _, ix in ranks:
                ctx.group_index_destroy(ix)
