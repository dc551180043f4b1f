"""GPU: the selection kernels on adversarial total-order keys and on every route, bit for bit against the plain
reference of tests/select_keys.py:
  K11 quantile       the resident sort (groups of at most 64 members), the whole-chunk radix select, the multi-chunk
                     select (nine pass + advance launches), count-only (phi outside [0, 1] or NaN);
  K10 topk/bottomk   the per-lane heap, chunk lists merged and marked, the general path in rounds of 32, the copy when
                     kk >= the largest group, and rows whose group id is out of range;
  K12 count_values   one batch, and a group whose cells exceed a batch, cut into step windows;
  K14 sort           sort and sort_desc over keys that differ in one bit, sentinels and payloads.
Each call asserts its route from Context.launch_count() around it (the group index is built before the first
reading).  The counts restate quantile_run / topk_run / count_values_run / sort_run (b2p_aggregation.cu, b2p_sort.cu):
  quantile   1 (resident only, or count-only), 2 (+ the pass kernel over whole-group chunks), 1 + 9 x 2 (a group of
             several chunks: nine pass + advance launches);
  topk       0 (kk = 0), 1 (copy, kk >= the largest group), else + 1 copy for out-of-range rows, then per round the
             chunk kernel (+ the merge kernel with multi-chunk groups), then the mark kernel (fast path with
             multi-chunk groups) or the select kernel (general path);
  count_values  1 + 5 per batch;  sort  1 (count) + 1 (scatter, when a cell is valid).
The chunk size C is max(256, ceil(members x tiles / U)) (quantile: members of groups above 64, capped at 32 768; topk:
every in-group member), with U 7/8 of the warps that stay resident.  U lies between 7/8 of one CTA of four warps per
SM and 7/8 of what the shared memory per SM (228 KB) and 64 warps per SM allow, so each call's route is computed from
both bounds; the calls at the route boundaries are sized so that both give the same route.
"""
import math

import numpy as np
import pytest

from tests import select_keys as sk

pytestmark = pytest.mark.gpu

SMEM_PER_SM = 228 * 1024
WARPS_PER_SM = 64
QUANT_CTA = 4 * 64 * 32 * 8  # kQuantWarps x kQuantWarpBytes
QUANT_CHUNK_MAX = 32768
NAN = float("nan")


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


def free_gb():
    import torch
    return torch.cuda.mem_get_info(0)[0] / 2 ** 30


# ---- routes ----------------------------------------------------------------------------------------------------------
def u_bounds(sms, cta_bytes):
    """(least, largest) U: 7/8 of the resident warps of a four-warp CTA, one CTA per SM up to what fits"""
    most = min(WARPS_PER_SM // 4, SMEM_PER_SM // cta_bytes)
    u = lambda per_sm: 4 * sms * per_sm - 4 * sms * per_sm // 8
    return u(1), u(most)


def chunk_bounds(member_tiles, sms, cta_bytes, cap=None):
    u_lo, u_hi = u_bounds(sms, cta_bytes)
    c = [max(256, -(-member_tiles // u)) for u in (u_hi, u_lo)]
    return [min(cap, x) for x in c] if cap else c


def floor_bound(sms):
    """member x tiles at or below which C is 256 whatever U is"""
    return 256 * math.floor(3.5 * sms)


def quantile_routes(sizes, T, phi, sms):
    if not (0.0 <= phi <= 1.0) or max(sizes) <= 64:
        return {1}
    tiles = (T + 31) // 32
    large = sum(s for s in sizes if s > 64)
    return {19 if any(s > C for s in sizes) else 2
            for C in chunk_bounds(large * tiles, sms, QUANT_CTA, QUANT_CHUNK_MAX)}


def topk_warp_bytes(K):
    return K * 32 * 16 + 512 * 4


def topk_routes(sizes, kk, T, stray, sms):
    """sizes: every in-range group (0 for an empty one)"""
    if kk == 0:
        return {0}
    if kk >= max(sizes):
        return {1}
    base = 1 if stray else 0
    if not any(sizes):
        return {base}
    general = kk > 32
    K = 32 if general else kk
    tiles = (T + 31) // 32
    out = set()
    for C in chunk_bounds(sum(sizes) * tiles, sms, 4 * topk_warp_bytes(K)):
        multi = any(s > C and not (general and s <= kk) for s in sizes)
        rounds = -(-kk // 32) if general else 1
        out.add(base + rounds * (1 + multi) + (1 if general or multi else 0))
    return out


def launches(ctx, f):
    before = ctx.launch_count()
    r = f()
    ctx.sync()
    return ctx.launch_count() - before, r


def dev(x, dtype=None):
    import torch
    x = np.ascontiguousarray(x)
    return torch.from_numpy(x.view(dtype) if dtype is not None else x).cuda()


def to_np(t, dtype):
    return t.cpu().numpy().view(dtype)


# ---- quantile --------------------------------------------------------------------------------------------------------
Q_SIZES = [1, 2, 63, 64, 65, 255, 256, 257, 512, 513, 4097]  # slots of 2, 2, 3 and 17 chunks at C = 256
Q_PHIS = [0.0, -0.0, 1.0, 0.5, 1 / 3, 0.25, float(np.nextafter(0.25, 0.0))]  # 0.25 (n - 1) is exact for n = 4j + 1
COUNT_ONLY = [NAN, -0.5, 1.5, -math.inf, math.inf]


def quantile_dev(ctx, phi, vals, ok, gid, n_groups):
    """the device form over a prebuilt index -> (launches, out, cnt)"""
    import torch
    T = vals.shape[1]
    d_vals, d_valid = dev(vals), dev(sk.words(ok), np.int32)
    ix = ctx.group_index_create_dev(dev(gid, np.int32), gid.size, n_groups)
    out = torch.full((n_groups, T), 12345.0, dtype=torch.float64, device="cuda")  # every cell is written
    cnt = torch.full((n_groups, T), 777, dtype=torch.int32, device="cuda")
    try:
        n, _ = launches(ctx, lambda: ctx.group_quantile_dev(phi, d_vals, d_valid, ix, T, out, cnt))
    finally:
        ctx.group_index_destroy(ix)
    return n, out.cpu().numpy(), to_np(cnt, np.uint32)


def check_quantile(ctx, sms, phi, vals, ok, gid, n_groups, sizes, host=False, routes=None):
    T = vals.shape[1]
    exp, ecnt = sk.quantile(phi, vals, ok, gid, n_groups)
    want = routes or quantile_routes(sizes, T, phi, sms)
    n, out, cnt = quantile_dev(ctx, phi, vals, ok, gid, n_groups)
    assert n in want, (phi, T, n, want)
    assert (cnt == ecnt).all(), (phi, T)
    bad = ~((np.isnan(out) & np.isnan(exp)) | (out.view(np.uint64) == exp.view(np.uint64)))
    assert not bad.any(), (phi, T, np.argwhere(bad)[:5])
    if host:
        n, (hout, hcnt) = launches(ctx, lambda: ctx.group_quantile(phi, vals, sk.words(ok), gid, n_groups))
        assert n - 2 in want, (phi, T, n)  # + the index the host form builds
        assert (hcnt == ecnt).all() and sk.same_or_nan(hout, exp), (phi, T)
    return n


@pytest.mark.parametrize("T", [1, 31, 32, 33, 64, 65, 1000])
def test_quantile_every_class_and_route(ctx, sms, T):
    """Groups of 1 .. 4 097 members (resident, whole-chunk and four multi-chunk slots in one call), each step of a tile
    a different class, 5 % of the cells invalid, empty groups between, rows out of range."""
    rng = np.random.default_rng(1000 + T)
    phis = Q_PHIS if T <= 65 else [0.5, 1.0, 0.25, float(np.nextafter(0.25, 0.0))]
    for i, phi in enumerate(phis):
        vals, ok, gid, G, _ = sk.grid(Q_SIZES, T, phi, rng, drop=0.05, gid_gap=2, stray=3)
        assert quantile_routes(Q_SIZES, T, phi, sms) == {19}
        check_quantile(ctx, sms, phi, vals, ok, gid, G, Q_SIZES, host=i < 2)
    for phi in COUNT_ONLY:
        check_quantile(ctx, sms, phi, vals, ok, gid, G, Q_SIZES, host=phi != phi)


@pytest.mark.parametrize("phi", [0.5, 1.0, 0.0, 0.25])
def test_quantile_route_boundaries_at_the_chunk_floor(ctx, sms, phi):
    """Group sizes on both sides of 64 and of the 256-member chunk floor, each call alone so that its launch count
    names its route: 257 members must take the multi-chunk route."""
    T = 33
    rng = np.random.default_rng(7)
    for sizes, want in [([1, 63, 64], 1), ([65], 2), ([65, 255, 256], 2), ([257], 19), ([512], 19), ([513], 19),
                        ([256, 257, 2], 19), ([64, 4097], 19)]:
        assert sum(s for s in sizes if s > 64) * 2 <= floor_bound(sms)
        assert quantile_routes(sizes, T, phi, sms) == {want}
        vals, ok, gid, G, _ = sk.grid(sizes, T, phi, rng, drop=0.02, stray=1)
        check_quantile(ctx, sms, phi, vals, ok, gid, G, sizes, routes={want})


def test_quantile_lanes_of_one_class_each(ctx, sms):
    """Every class alone over a whole tile of a multi-chunk group and of a whole-chunk group, with every cell valid:
    each (group, step) runs exactly the passes its class needs."""
    T = 64
    rng = np.random.default_rng(11)
    for phi in (0.5, 1.0, 1 / 3):
        for cls in sk.CLASSES:
            sizes = [200, 600, 40]
            vals, ok, gid, G, _ = sk.grid(sizes, T, phi, rng, classes=[cls])
            check_quantile(ctx, sms, phi, vals, ok, gid, G, sizes, routes={19})


def test_quantile_whole_chunk_at_the_counter_ceiling(ctx, sms):
    """One whole-chunk group of kQuantChunkMax (32 768) members whose keys at a step all fall in one bin at every
    level: the 16-bit per-lane counter at its ceiling.  C reaches 32 768 only when the large groups' members x tiles
    reach 32 768 U, so the call carries groups of 32 768 members with no valid cell."""
    import torch
    _, u_hi = u_bounds(sms, QUANT_CTA)
    n_groups = u_hi + 1
    R, T = n_groups * QUANT_CHUNK_MAX, 32
    if free_gb() < 24 or R * T * 8 / 2 ** 30 > free_gb() - 8:
        pytest.skip("needs 24 GB of free device memory")
    assert chunk_bounds((R - QUANT_CHUNK_MAX) * 1, sms, QUANT_CTA, QUANT_CHUNK_MAX) == [QUANT_CHUNK_MAX] * 2
    rng = np.random.default_rng(12)
    head_vals, head_ok, _, _, _ = sk.grid([QUANT_CHUNK_MAX], T, 0.5, rng, classes=["equal", "depth7-last", "top"])
    vals = torch.empty((R, T), dtype=torch.float64, device="cuda")  # never read past the first group
    vals[:QUANT_CHUNK_MAX] = dev(head_vals)
    valid = torch.zeros((R, 1), dtype=torch.int32, device="cuda")
    valid[:QUANT_CHUNK_MAX] = dev(sk.words(head_ok), np.int32)
    gid = (torch.arange(R, dtype=torch.int32, device="cuda") // QUANT_CHUNK_MAX).contiguous()
    ix = ctx.group_index_create_dev(gid, R, n_groups)
    try:
        for phi in (0.5, 1.0, 0.0):
            out = torch.full((n_groups, T), 12345.0, dtype=torch.float64, device="cuda")
            cnt = torch.full((n_groups, T), 777, dtype=torch.int32, device="cuda")
            n, _ = launches(ctx, lambda: ctx.group_quantile_dev(phi, vals, valid, ix, T, out, cnt))
            assert n == 2, n  # every group one whole chunk
            exp, ecnt = sk.quantile(phi, head_vals, head_ok, np.zeros(QUANT_CHUNK_MAX, np.uint32), 1)
            assert (to_np(cnt[:1], np.uint32) == ecnt).all()
            assert sk.same_or_nan(out[:1].cpu().numpy(), exp)
            assert not cnt[1:].any().item() and not out[1:].any().item()
    finally:
        ctx.group_index_destroy(ix)


# ---- topk / bottomk --------------------------------------------------------------------------------------------------
KKS = [1, 31, 32, 33, 64, 65, 96, 97]


def topk_grid(rng, sizes, T, stray):
    # value ties decided by the ordinals: equal keys, ±0, sentinels, and the other classes
    classes = ("equal", "signed-zero", "sentinel-only0", "sentinel-onlymax", "payloads", "equal") + sk.CLASSES
    vals, ok, gid, G, _ = sk.grid(sizes, T, 0.5, rng, classes=classes, drop=0.3, gid_gap=2, stray=stray)
    ok[:, ::3] |= gid[:, None] < G  # every member's cell on every third step: counts of exactly kk and kk + 1
    tie = np.arange(gid.size, dtype=np.uint32)
    rng.shuffle(tie)
    tie[tie == 1] = 0xFFFFFFFF  # ordinals stay distinct and include 0 and 0xFFFFFFFF
    return vals, ok, gid, G, tie


def topk_case(ctx, sms, op, kk, vals, ok, gid, G, tie, sizes, stray, host=False):
    import torch
    T = vals.shape[1]
    bottom = op == "bottomk"
    exp = sk.words(sk.topk(bottom, kk, vals, ok, gid, G, tie))
    want = topk_routes(sizes, kk, T, stray, sms)
    d_vals, d_valid, d_tie = dev(vals), dev(sk.words(ok), np.int32), dev(tie, np.int32)
    ix = ctx.group_index_create_dev(dev(gid, np.int32), gid.size, G)
    try:
        out = torch.full_like(d_valid, -1)
        n, _ = launches(ctx, lambda: ctx.topk_dev(op, float(kk), d_vals, d_valid, ix, d_tie, T, out))
        assert n in want, (op, kk, n, want)
        assert (to_np(out, np.uint32) == exp).all(), (op, kk)
        inplace = d_valid.clone()
        n, _ = launches(ctx, lambda: ctx.topk_dev(op, float(kk), d_vals, inplace, ix, d_tie, T, inplace))
        assert n in want and (to_np(inplace, np.uint32) == exp).all(), (op, kk, "in place")
    finally:
        ctx.group_index_destroy(ix)
    if host:
        n, got = launches(ctx, lambda: ctx.topk(op, float(kk), vals, sk.words(ok), gid, G, tie))
        assert n - 2 in want and (got == exp).all(), (op, kk, "host")
    return want


@pytest.mark.parametrize("kk", KKS)
def test_topk_every_kk_and_route(ctx, sms, kk):
    """Groups of kk and kk + 1 members, small groups, a group of 700 (three chunks at C = 256), empty groups and rows
    out of range; a third of the steps with every cell valid, the others thinned, so a warp's lanes take their verdicts
    (bound, threshold, every cell) in different rounds."""
    rng = np.random.default_rng(2000 + kk)
    T = 65
    sizes = [kk, kk + 1, 1, 2, 40, 700]
    vals, ok, gid, G, tie = topk_grid(rng, sizes, T, stray=5)
    all_sizes = [s for g in sizes for s in (g, 0)]
    assert sum(sizes) * 3 <= floor_bound(sms)
    for op in ("topk", "bottomk"):
        want = topk_case(ctx, sms, op, kk, vals, ok, gid, G, tie, all_sizes, 5, host=op == "topk")
        rounds = -(-kk // 32) if kk > 32 else 1
        assert want == {1 + rounds * 2 + 1}  # copy + chunk & merge per round + mark / select
    # the copy route (kk >= the largest group) and kk = 0
    for k in (700, 10 ** 6, 0):
        want = topk_case(ctx, sms, "topk", k, vals, ok, gid, G, tie, all_sizes, 5)
        assert want == ({0} if k == 0 else {1})


def test_topk_single_chunk_routes_and_the_middle_rounds(ctx, sms):
    """Without multi-chunk groups (fast path: the chunk kernel alone; general path: the rounds and the select kernel),
    with a group of 98 members whose steps hold 33 .. 98 valid cells: under kk = 97 some lanes keep every cell after
    round 1 or 2 while their neighbours still bound the next round."""
    rng = np.random.default_rng(21)
    T = 96
    sizes = [98, 33, 256, 3]
    vals, ok, gid, G, tie = topk_grid(rng, sizes, T, stray=0)
    rows = np.flatnonzero(gid == 0)
    for k in range(T):  # 33 + k % 66 valid cells at step k
        ok[rows, k] = False
        ok[rows[rng.permutation(98)[:33 + k % 66]], k] = True
    all_sizes = [s for g in sizes for s in (g, 0)]
    for op in ("topk", "bottomk"):
        for kk in (32, 33, 64, 65, 97):
            want = topk_case(ctx, sms, op, kk, vals, ok, gid, G, tie, all_sizes, 0)
            rounds = -(-kk // 32)
            assert want == ({1} if kk <= 32 else {rounds + 1}), (kk, want)


def test_topk_single_chunk_groups_straddle_the_mark_block(ctx, sms):
    """Single-chunk groups of 511, 512, 513 and 1 025 members write their words in 512-word blocks.  C > 1 025 needs
    more in-group members x tiles than 1 025 U, so the call carries groups of 1 000 members with no valid cell; the
    launch count shows that no merge or mark kernel ran."""
    import torch
    sizes = [511, 512, 513, 1025]
    T = 32
    u_most = 4 * sms * min(WARPS_PER_SM // 4, SMEM_PER_SM // (4 * topk_warp_bytes(1)))
    n_fill = -(-1026 * u_most // 1000)
    R = sum(sizes) + 1000 * n_fill
    if free_gb() < 8 or R * T * 8 / 2 ** 30 > free_gb() - 4:
        pytest.skip("needs 8 GB of free device memory")
    rng = np.random.default_rng(22)
    vals, ok, gid, G, tie = topk_grid(rng, sizes, T, stray=0)
    n_head = gid.size
    d_vals = torch.zeros((R, T), dtype=torch.float64, device="cuda")
    d_vals[:n_head] = dev(vals)
    d_valid = torch.zeros((R, 1), dtype=torch.int32, device="cuda")
    d_valid[:n_head] = dev(sk.words(ok), np.int32)
    d_gid = torch.empty(R, dtype=torch.int32, device="cuda")
    d_gid[:n_head] = dev(gid, np.int32)
    d_gid[n_head:] = G + torch.arange(R - n_head, dtype=torch.int32, device="cuda") // 1000
    d_tie = torch.arange(R, dtype=torch.int32, device="cuda")
    d_tie[:n_head] = dev(tie, np.int32)
    all_sizes = [s for g in sizes for s in (g, 0)][:G] + [1000] * n_fill
    ix = ctx.group_index_create_dev(d_gid, R, G + n_fill)
    try:
        for op in ("topk", "bottomk"):
            for kk in (1, 32, 33):
                want = topk_routes(all_sizes, kk, T, 0, sms)
                assert want == ({1} if kk <= 32 else {3}), want  # chunk kernel alone / two rounds + select
                exp = sk.words(sk.topk(op == "bottomk", kk, vals, ok, gid, G, tie))
                out = torch.full_like(d_valid, -1)
                n, _ = launches(ctx, lambda: ctx.topk_dev(op, float(kk), d_vals, d_valid, ix, d_tie, T, out))
                assert n in want, (op, kk, n)
                assert (to_np(out[:n_head], np.uint32) == exp).all(), (op, kk)
                assert not out[n_head:].any().item(), (op, kk)
    finally:
        ctx.group_index_destroy(ix)


# ---- count_values ----------------------------------------------------------------------------------------------------
CV_SIZES = [1, 2, 63, 64, 65, 300]


def check_count_values(ctx, vals, ok, gid, G, want_launches, host=True):
    import torch
    T = vals.shape[1]
    exp, ecnt = sk.count_values(vals, ok, gid, G)
    ix = ctx.group_index_create_dev(dev(gid, np.int32), gid.size, G)
    out = torch.full(vals.shape, 12345.0, dtype=torch.float64, device="cuda")  # every cell is written
    cnt = torch.full(vals.shape, 777, dtype=torch.int32, device="cuda")
    try:
        d_vals, d_valid = dev(vals), dev(sk.words(ok), np.int32)
        n, _ = launches(ctx, lambda: ctx.count_values_dev(d_vals, d_valid, ix, T, out, cnt))
    finally:
        ctx.group_index_destroy(ix)
    assert n == want_launches, n
    assert (to_np(cnt, np.uint32) == ecnt).all() and sk.same_bits(out.cpu().numpy(), exp)
    if host:
        n, (hout, hcnt) = launches(ctx, lambda: ctx.count_values(vals, sk.words(ok), gid, G))
        assert n - 2 == want_launches and (hcnt == ecnt).all() and sk.same_bits(hout, exp)


@pytest.mark.parametrize("T", [1, 33, 65, 1000])
def test_count_values_every_class_as_a_segment(ctx, T):
    """Every class as a (group, step) segment beside invalid cells, whose key is the largest, ~0: a valid ~0 (+NaN
    0x7FFF..F) must count as a value and the invalid cells must not.  One batch: 1 + 5 launches."""
    rng = np.random.default_rng(3000 + T)
    vals, ok, gid, G, _ = sk.grid(CV_SIZES, T, 0.5, rng, drop=0.25, gid_gap=2, stray=4)
    check_count_values(ctx, vals, ok, gid, G, 6, host=T <= 65)
    # the sentinel classes alone
    vals, ok, gid, G, _ = sk.grid(CV_SIZES, T, 0.5, rng, classes=sk.SENTINELS, drop=0.25, stray=2)
    check_count_values(ctx, vals, ok, gid, G, 6, host=False)


def test_count_values_group_beyond_a_batch_in_step_windows(ctx):
    """One group of 1.2 M members over 200 steps: its cells exceed kCvBatchCells (2^27), so the call runs in windows of
    2^27 / 1.2 M rounded down to 96 steps: 96, 96 and a short 8, one batch each (1 + 3 x 5 launches).  The class groups
    share the windows and are checked against the reference; the large group's values are 10 k + row % 5 at step k, so
    its distinct values and counts are known."""
    import torch
    M, T = 1_200_000, 200
    if free_gb() < 10:
        pytest.skip("needs 10 GB of free device memory")
    rng = np.random.default_rng(31)
    vals, ok, gid, G, _ = sk.grid(CV_SIZES, T, 0.5, rng, drop=0.25, stray=3)
    n_small = gid.size
    R = n_small + M
    Tw = (T + 31) // 32
    d_vals = torch.empty((R, T), dtype=torch.float64, device="cuda")
    d_vals[:n_small] = dev(vals)
    r = torch.arange(M, dtype=torch.float64, device="cuda")
    d_vals[n_small:] = (r % 5)[:, None] + 10.0 * torch.arange(T, dtype=torch.float64, device="cuda")[None, :]
    d_valid = torch.full((R, Tw), -1, dtype=torch.int32, device="cuda")  # (bits past T are ignored)
    d_valid[:n_small] = dev(sk.words(ok), np.int32)
    d_gid = torch.full((R,), G, dtype=torch.int32, device="cuda")  # the large group is the last in range
    d_gid[:n_small] = dev(gid, np.int32)
    out = torch.full((R, T), 12345.0, dtype=torch.float64, device="cuda")
    cnt = torch.full((R, T), 777, dtype=torch.int32, device="cuda")
    ix = ctx.group_index_create_dev(d_gid, R, G + 1)
    try:
        n, _ = launches(ctx, lambda: ctx.count_values_dev(d_vals, d_valid, ix, T, out, cnt))
    finally:
        ctx.group_index_destroy(ix)
    assert n == 1 + 3 * 5, n
    exp, ecnt = sk.count_values(vals, ok, gid, G)
    in_small = int((gid < G).sum())  # member order: the class groups, the large group, then the stray rows
    assert (to_np(cnt[:in_small], np.uint32) == ecnt[:in_small]).all()
    assert sk.same_bits(out[:in_small].cpu().numpy(), exp[:in_small])
    big_c, big_v = cnt[in_small:in_small + M], out[in_small:in_small + M]
    per = torch.tensor([(M - j + 4) // 5 for j in range(5)], dtype=torch.int32, device="cuda")
    assert torch.equal(big_c[:5], per[:, None].expand(5, T).contiguous())
    assert torch.equal(big_v[:5], torch.arange(5, dtype=torch.float64, device="cuda")[:, None]
                       + 10.0 * torch.arange(T, dtype=torch.float64, device="cuda")[None, :])
    assert not big_c[5:].any().item() and not big_v[5:].any().item()
    assert not cnt[in_small + M:].any().item() and not out[in_small + M:].any().item()


# ---- sort / sort_desc ------------------------------------------------------------------------------------------------
def sort_grid(rng, R, T):
    """Rows of keys that differ only in bit 0, only in bit 63, sentinels, payloads, and runs of equal keys across rows"""
    base = sk._rand(rng, sk.KMIN, sk.KMAX, 1)[0]
    keys = np.empty((R, T), np.uint64)
    kinds = ["bit0", "bit63", "equal-run"] + list(sk.SENTINELS) + ["payloads"]
    for k in range(T):
        kind = kinds[k % len(kinds)]
        if kind == "bit0":
            keys[:, k] = (base & ~np.uint64(1)) | rng.integers(0, 2, R, dtype=np.uint64)
        elif kind == "bit63":
            keys[:, k] = (base & ~sk.SIGN) | (rng.integers(0, 2, R, dtype=np.uint64) << np.uint64(63))
        elif kind == "equal-run":
            keys[:, k] = base
        else:
            keys[:, k] = sk.column(kind, R, 0.5, rng)
    keys[rng.random((R, T)) < 0.1] = 0  # key 0 (the -NaN of every payload bit) anywhere, ~0 too
    keys[rng.random((R, T)) < 0.1] = sk.ALL
    ok = rng.random((R, T)) < 0.85
    return sk.values_of_keys(keys), ok


@pytest.mark.parametrize("T", [1, 32, 45])
def test_sort_bit_edges_sentinels_and_ties(ctx, T):
    import torch
    rng = np.random.default_rng(4000 + T)
    R = 70
    vals, ok = sort_grid(rng, R, T)
    d_vals, d_valid = dev(vals), dev(sk.words(ok), np.int32)
    for desc in (False, True):
        exp = sk.sort(desc, vals, ok)
        cells = torch.zeros(R * T, dtype=torch.int64, device="cuda")
        n_out = torch.zeros(1, dtype=torch.int64, device="cuda")
        n, _ = launches(ctx, lambda: ctx.sort_cells_dev(desc, d_vals, d_valid, R, T, cells, n_out))
        assert n == 2, n  # count + scatter (CUB's scan and sort are not counted)
        got = to_np(cells, np.uint64)[:int(n_out.item())]
        assert got.size == exp.size and (got == exp).all(), desc
        n, host = launches(ctx, lambda: ctx.sort_cells(desc, vals, sk.words(ok)))
        assert n == 2 and (host == exp).all(), desc
