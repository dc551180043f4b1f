// b2p_aggregation.cu — by-label selections of the C ABI over a group index: topk / bottomk, quantile and count_values.
#include <algorithm>
#include <cmath>
#include <vector>

#include <cub/device/device_scan.cuh>
#include <cub/device/device_segmented_sort.cuh>

#include "b2p_runtime.cuh"
#include "b2p_topk.cuh"
#include "b2p_quantile.cuh"
#include "b2p_count_values.cuh"

using namespace b2p;

namespace {
// k -> the number of ranks kept: row_number <= k in the f64 total order (the reference's Filter compares the UInt64
// row number coerced to Float64 with the Float64 literal k): floor(k) for finite k >= 1; none for k < 1, -inf and
// -NaN; every rank for +inf and +NaN
uint32_t topk_ranks(double k) {
  if (std::isnan(k)) return std::signbit(k) ? 0u : UINT32_MAX;
  if (!(k >= 1.0)) return 0u;
  if (k >= 4294967295.0) return UINT32_MAX;
  return (uint32_t)std::floor(k);
}

// Scratch (context buffers t_table / t_cand / t_state), with C the chunk size below and U 7/8 of the warps of
// topk_chunk_kernel that stay resident (1 386 at K = 32, 3 234 at K = 10 on a 132-SM H100):
//   tables:     16 B per chunk and per multi-chunk group;
//   candidates: (K * 32 * 16 + 128) B per (chunk of a multi-chunk group, tile).  Such chunks hold more than C / 2
//               members and C >= members * tiles / U, so there are at most 2 * U of these units: 46 MB at K = 32,
//               34 MB at K = 10 on a 132-SM H100, whatever the input;
//   state:      640 B per (group with a state, tile), i.e. 20 B per (group, step): multi-chunk groups, and on the
//               general path every group of more than kk >= 33 members, so at most 0.61 B per input cell.
// i64: the grid is Int64 (I64Key).
int topk_run(b2p_ctx* c, int bottom, uint32_t kk, const double* vals, const uint32_t* valid, const b2p_group_index* ix,
             const uint32_t* tie, uint64_t T, uint32_t* out_valid, bool i64) {
  int rc;
  auto* const chunk_kernel = i64 ? topk_chunk_kernel<I64Key> : topk_chunk_kernel<F64Key>;
  auto* const select_kernel = i64 ? topk_select_kernel<I64Key> : topk_select_kernel<F64Key>;
  const uint32_t R = ix->n_series, G = ix->n_groups;
  const uint32_t Tw = (uint32_t)((T + 31) / 32), tiles = Tw;
  const size_t words = (size_t)R * Tw;
  auto copy = [&](int mode) {
    topk_copy_kernel<<<capped_grid(c, words, 256, 16), 256, 0, c->stream>>>(valid, ix->gid, G, R, T, Tw, mode, out_valid);
    c->launches++;
    CU(cudaGetLastError());
    return B2P_OK;
  };
  if (kk == 0) {
    CU(cudaMemsetAsync(out_valid, 0, words * 4, c->stream));
    return B2P_OK;
  }
  if (kk >= ix->max_members) return copy(0);  // every valid cell of every group is kept
  const uint32_t in_groups = G ? ix->goff_host[G] : 0;
  if (in_groups < R && (rc = copy(1))) return rc;  // rows whose group id is out of range keep nothing
  const bool general = kk > kTopkMax;
  const uint32_t K = general ? kTopkMax : kk;
  // chunk size: at most about one warp unit per resident warp (a second, partial wave would double the time; the 1/8
  // slack absorbs the rounding of the chunk counts), and at least 256 members
  const size_t smem = kTopkWarps * topk_warp_bytes(K);
  unsigned cap = 0;
  if ((rc = persistent_grid(c, chunk_kernel, smem, kTopkWarps, kAllResident, &cap))) return rc;
  const uint64_t resident = (uint64_t)cap * kTopkWarps;
  const uint64_t U = resident - resident / 8;
  const uint64_t C = std::max<uint64_t>(256, ((uint64_t)in_groups * tiles + U - 1) / U);
  std::vector<TopkChunk> chunks;
  std::vector<TopkMerge> merges;
  uint32_t n_cand = 0, n_state = 0;
  for (uint32_t g = 0; g < G; ++g) {
    const uint32_t b = ix->goff_host[g], e = ix->goff_host[g + 1], s = e - b;
    if (s == 0) continue;
    if (general && s <= kk) {  // keeps every valid cell
      chunks.push_back(TopkChunk{b, e, kTopkNone, kTopkNone});
    } else if (s <= C) {
      chunks.push_back(TopkChunk{b, e, kTopkNone, general ? n_state++ : kTopkNone});
    } else {
      const uint32_t nc = (uint32_t)((s + C - 1) / C);
      merges.push_back(TopkMerge{n_cand, n_cand + nc, n_state, 0});
      for (uint32_t i = 0; i < nc; ++i)
        chunks.push_back(TopkChunk{b + (uint32_t)((uint64_t)s * i / nc), b + (uint32_t)((uint64_t)s * (i + 1) / nc),
                                   n_cand++, n_state});
      ++n_state;
    }
  }
  if (chunks.empty()) return B2P_OK;
  const size_t tb_chunks = chunks.size() * sizeof(TopkChunk), tb_merges = merges.size() * sizeof(TopkMerge);
  if ((rc = c->t_table.ensure(tb_chunks + tb_merges + 16))) return rc;
  CU(cudaMemcpyAsync(c->t_table.p, chunks.data(), tb_chunks, cudaMemcpyHostToDevice, c->stream));
  if (tb_merges)
    CU(cudaMemcpyAsync(c->t_table.as<char>() + tb_chunks, merges.data(), tb_merges, cudaMemcpyHostToDevice, c->stream));
  const size_t cand_units = (size_t)n_cand * tiles, state_cells = (size_t)n_state * tiles * 32;
  const size_t cand_slots = cand_units * K * 32;
  if ((rc = c->t_cand.ensure(cand_slots * 16 + cand_units * 32 * 4 + 64))) return rc;
  if ((rc = c->t_state.ensure(state_cells * 20 + 64))) return rc;
  TopkArgs a{};
  a.vals = vals; a.valid = valid; a.members = ix->members; a.tie = tie;
  a.chunks = c->t_table.as<TopkChunk>(); a.n_chunks = (uint32_t)chunks.size();
  a.merges = reinterpret_cast<const TopkMerge*>(c->t_table.as<char>() + tb_chunks); a.n_merges = (uint32_t)merges.size();
  a.T = T; a.Tw = Tw; a.tiles = tiles; a.K = K; a.kk = kk; a.bottom = bottom ? 1 : 0; a.general = general ? 1 : 0;
  a.c_hi = c->t_cand.as<unsigned long long>();
  a.c_lo = reinterpret_cast<uint32_t*>(a.c_hi + cand_slots);
  a.c_pos = a.c_lo + cand_slots;
  a.c_n = a.c_pos + cand_slots;
  a.s_hi = c->t_state.as<unsigned long long>();
  a.s_lo = reinterpret_cast<uint32_t*>(a.s_hi + state_cells);
  a.s_rem = a.s_lo + state_cells;
  a.s_flags = a.s_rem + state_cells;
  a.out_valid = out_valid;
  const uint64_t chunk_units = (uint64_t)chunks.size() * tiles, merge_units = (uint64_t)merges.size() * tiles;
  unsigned g_chunk = 0, g_merge = 0, g_mark = 0;
  if ((rc = persistent_grid(c, chunk_kernel, smem, kTopkWarps, chunk_units, &g_chunk))) return rc;
  if (merge_units && (rc = persistent_grid(c, topk_merge_kernel, smem, kTopkWarps, merge_units, &g_merge))) return rc;
  const uint32_t rounds = general ? (kk + kTopkMax - 1) / kTopkMax : 1;
  for (uint32_t r = 0; r < rounds; ++r) {
    a.round = (int)r;
    chunk_kernel<<<g_chunk, kTopkWarps * 32, smem, c->stream>>>(a);
    c->launches++;
    CU(cudaGetLastError());
    if (merge_units) {
      topk_merge_kernel<<<g_merge, kTopkWarps * 32, smem, c->stream>>>(a);
      c->launches++;
      CU(cudaGetLastError());
    }
  }
  if (general) {
    select_kernel<<<capped_grid(c, chunk_units, 8, 16), 256, 0, c->stream>>>(a);
  } else if (merge_units) {
    if ((rc = persistent_grid(c, topk_mark_kernel, 0, kTopkWarps, chunk_units, &g_mark))) return rc;
    topk_mark_kernel<<<g_mark, kTopkWarps * 32, 0, c->stream>>>(a);
  } else {
    return B2P_OK;
  }
  c->launches++;
  CU(cudaGetLastError());
  return B2P_OK;
}

template <class Kern>
int quantile_launch(b2p_ctx* c, Kern* kern, uint64_t units, const QuantArgs& a) {
  const size_t smem = kQuantWarps * kQuantWarpBytes;
  unsigned grid = 0;
  if (int rc = persistent_grid(c, kern, smem, kQuantWarps, units, &grid)) return rc;
  if (grid == 0) return B2P_OK;
  kern<<<grid, kQuantWarps * 32, smem, c->stream>>>(a);
  c->launches++;
  CU(cudaGetLastError());
  return B2P_OK;
}

// Resident limit: groups of at most kQuantResident (64) members are read once and finished in shared memory.  A larger
// group takes at most kQuantPasses (9) reads of its cells: one per 8-bit digit of the key, one for the extremes; a
// (group, step) stops as soon as both order statistics are known, a warp as soon as its 32 steps are.  Such a group is
// cut into chunks of C members, C about its share of one wave of the pass kernel's resident warps (U below) and at
// most kQuantChunkMax; a group of one chunk is finished by one warp in one launch.
// Scratch (context buffers q_table / q_state / q_hist) for the groups of several chunks: 16 B per chunk and 4 B per
// such group; 56 B of state per (group, step); 32 KB of histogram per (group, tile).  Each such group has more than
// C >= min(members * tiles / U, kQuantChunkMax) members, so there are at most max(U, members * tiles / kQuantChunkMax)
// of these (group, tile) units: 44 MB of histograms with the 1 386 warps U is on a 132-SM H100 (three 64 KB CTAs of
// four warps per SM), until the large groups' members times tiles pass 45 M.
int quantile_run(b2p_ctx* c, double phi, const double* vals, const uint32_t* valid, const b2p_group_index* ix,
                 uint64_t T, double* out_val, uint32_t* out_cnt) {
  int rc;
  const uint32_t G = ix->n_groups, Tw = (uint32_t)((T + 31) / 32);
  QuantArgs a{};
  a.vals = vals; a.valid = valid; a.goff = ix->goff; a.members = ix->members; a.n_groups = G;
  a.T = T; a.Tw = Tw; a.tiles = Tw; a.phi = phi;
  a.count_only = !(phi >= 0.0 && phi <= 1.0) ? 1 : 0;
  a.out_val = out_val; a.out_cnt = out_cnt;
  if ((rc = quantile_launch(c, quantile_resident_kernel, (uint64_t)G * Tw, a))) return rc;
  if (a.count_only || ix->max_members <= kQuantResident) return B2P_OK;
  unsigned cap = 0;
  if ((rc = persistent_grid(c, quantile_pass_kernel, kQuantWarps * kQuantWarpBytes, kQuantWarps, kAllResident, &cap)))
    return rc;
  const uint64_t resident = (uint64_t)cap * kQuantWarps, U = resident - resident / 8;
  uint64_t large = 0;
  for (uint32_t g = 0; g < G; ++g) {
    const uint32_t s = ix->goff_host[g + 1] - ix->goff_host[g];
    if (s > kQuantResident) large += s;
  }
  const uint64_t C = std::min<uint64_t>(kQuantChunkMax, std::max<uint64_t>(256, (large * Tw + U - 1) / U));
  std::vector<QuantChunk> chunks;
  std::vector<uint32_t> slot_group;
  for (uint32_t g = 0; g < G; ++g) {
    const uint32_t b = ix->goff_host[g], e = ix->goff_host[g + 1], s = e - b;
    if (s <= kQuantResident) continue;
    if (s <= C) {
      chunks.push_back(QuantChunk{b, e, g, kQuantNone});
      continue;
    }
    const uint32_t nc = (uint32_t)((s + C - 1) / C), slot = (uint32_t)slot_group.size();
    slot_group.push_back(g);
    for (uint32_t i = 0; i < nc; ++i)
      chunks.push_back(QuantChunk{b + (uint32_t)((uint64_t)s * i / nc), b + (uint32_t)((uint64_t)s * (i + 1) / nc), g, slot});
  }
  const size_t tb_chunks = chunks.size() * sizeof(QuantChunk), tb_slots = slot_group.size() * 4;
  if ((rc = c->q_table.ensure(tb_chunks + tb_slots + 16))) return rc;
  CU(cudaMemcpyAsync(c->q_table.p, chunks.data(), tb_chunks, cudaMemcpyHostToDevice, c->stream));
  if (tb_slots)
    CU(cudaMemcpyAsync(c->q_table.as<char>() + tb_chunks, slot_group.data(), tb_slots, cudaMemcpyHostToDevice, c->stream));
  a.chunks = c->q_table.as<QuantChunk>(); a.n_chunks = (uint32_t)chunks.size();
  a.slot_group = reinterpret_cast<const uint32_t*>(c->q_table.as<char>() + tb_chunks);
  a.n_slots = (uint32_t)slot_group.size();
  if (a.n_slots) {
    const size_t state_bytes = (size_t)a.n_slots * T * sizeof(QuantState);
    const size_t hist_bytes = (size_t)a.n_slots * Tw * 256 * 32 * 4;
    if ((rc = c->q_state.ensure(state_bytes))) return rc;
    if ((rc = c->q_hist.ensure(hist_bytes))) return rc;
    CU(cudaMemsetAsync(c->q_state.p, 0, state_bytes, c->stream));
    CU(cudaMemsetAsync(c->q_hist.p, 0, hist_bytes, c->stream));
    a.state = c->q_state.as<QuantState>();
    a.hist = c->q_hist.as<uint32_t>();
  }
  const uint64_t units = (uint64_t)chunks.size() * Tw;
  for (uint32_t p = 0; p < (a.n_slots ? kQuantPasses : 1u); ++p) {
    a.pass = (int)p;
    if ((rc = quantile_launch(c, quantile_pass_kernel, units, a))) return rc;
    if (!a.n_slots) break;
    quantile_advance_kernel<<<capped_grid(c, (uint64_t)a.n_slots * T, 256, 8), 256, 0, c->stream>>>(a);
    c->launches++;
    CU(cudaGetLastError());
  }
  return B2P_OK;
}

// A run of groups [g0, g1) over steps [k0, k0 + W) (b2p_count_values.cuh)
struct CvBatch {
  uint32_t g0, g1, k0, W;
  uint64_t cells, segments;
};

// Batches: windows of W steps (every step when the largest group's cells fit kCvBatchCells, else a multiple of 32),
// each cut into runs of whole groups whose cells (members x W) and segments (groups x W) fit kCvBatchCells; a group
// too large for that alone is a batch of its own.  Per batch: the segment table, the scatter, CUB's segmented sort, the
// head flags, CUB's scan over them, the rank and count passes; no host round trip.
// Scratch (context buffers v_*): 20 B per cell of a batch (8 B key, 8 B sorted key, 4 B rank; the start table reuses
// the key buffer once the sort has left it), so at most 20 B x kCvBatchCells = 2.7 GB unless one group alone has more
// than kCvBatchCells / 32 = 4.2 M members (then 20 B x its members x 32); 8 B per (group, step) of a batch; 4 B per
// in-range row; CUB's temp storage for the sort and the scan.
// i64: the grid is Int64 (I64Key), and so are the distinct values out_val receives.
int count_values_run(b2p_ctx* c, const double* vals, const uint32_t* valid, const b2p_group_index* ix, uint64_t T,
                     double* out_val, uint32_t* out_cnt, bool i64) {
  int rc;
  const uint32_t R = ix->n_series, G = ix->n_groups, Tw = (uint32_t)((T + 31) / 32);
  const uint32_t in_rows = G ? ix->goff_host[G] : 0u;
  if (in_rows < R) {  // rows whose group id is out of range take part in nothing: count 0
    CU(cudaMemsetAsync(out_val + (uint64_t)in_rows * T, 0, (uint64_t)(R - in_rows) * T * 8, c->stream));
    CU(cudaMemsetAsync(out_cnt + (uint64_t)in_rows * T, 0, (uint64_t)(R - in_rows) * T * 4, c->stream));
  }
  if (in_rows == 0) return B2P_OK;
  const uint64_t W = std::min<uint64_t>((T + 31) / 32 * 32, std::max<uint64_t>(32, kCvBatchCells / ix->max_members / 32 * 32));
  if ((uint64_t)ix->max_members * std::min<uint64_t>(W, T) > (uint64_t)INT32_MAX)
    return fail(B2P_E_TOO_LARGE, "count_values: a group of %u members is too large", ix->max_members);
  std::vector<CvBatch> batches;
  uint64_t max_cells = 0, max_segs = 0;
  for (uint64_t k0 = 0; k0 < T; k0 += W) {
    const uint64_t Wb = std::min<uint64_t>(W, T - k0);
    for (uint32_t g = 0; g < G;) {
      const uint32_t g0 = g;
      uint64_t members = 0;
      for (; g < G; ++g) {
        const uint64_t s = ix->goff_host[g + 1] - ix->goff_host[g];
        if (g > g0 && std::max<uint64_t>(members + s, g + 1 - g0) * Wb > kCvBatchCells) break;
        members += s;
      }
      if (members == 0) continue;  // empty groups only: no output row
      batches.push_back(CvBatch{g0, g, (uint32_t)k0, (uint32_t)Wb, members * Wb, (uint64_t)(g - g0) * Wb});
      max_cells = std::max(max_cells, members * Wb);
      max_segs = std::max(max_segs, (uint64_t)(g - g0) * Wb);
    }
  }
  size_t tmp = 16;
  for (const CvBatch& b : batches) {
    size_t sort_bytes = 0, scan_bytes = 0;
    cub::DoubleBuffer<unsigned long long> db(nullptr, nullptr);
    CU(cub::DeviceSegmentedSort::SortKeys(nullptr, sort_bytes, db, (int)b.cells, (int)b.segments, (const uint32_t*)nullptr,
                                          (const uint32_t*)nullptr, c->stream));
    CU(cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, (uint32_t*)nullptr, (uint32_t*)nullptr, (int)b.cells, c->stream));
    tmp = std::max({tmp, sort_bytes, scan_bytes});
  }
  if ((rc = c->v_keys.ensure(max_cells * 8)) || (rc = c->v_alt.ensure(max_cells * 8)) ||
      (rc = c->v_rank.ensure(max_cells * 4)) || (rc = c->v_seg.ensure((2 * max_segs + 1) * 4)) ||
      (rc = c->v_group.ensure((size_t)in_rows * 4)) || (rc = c->v_tmp.ensure(tmp)))
    return rc;
  count_values_member_group_kernel<<<capped_grid(c, in_rows, 256, 16), 256, 0, c->stream>>>(
      ix->gid, ix->members, in_rows, c->v_group.as<uint32_t>());
  c->launches++;
  CU(cudaGetLastError());
  CvArgs a{};
  a.vals = vals; a.valid = valid; a.members = ix->members; a.goff = ix->goff; a.mgroup = c->v_group.as<uint32_t>();
  a.T = T; a.Tw = Tw;
  a.seg_off = c->v_seg.as<uint32_t>(); a.seg_n = a.seg_off + max_segs + 1;
  a.rank = c->v_rank.as<uint32_t>();
  a.out_val = out_val; a.out_cnt = out_cnt;
  for (const CvBatch& b : batches) {
    a.g0 = b.g0; a.g1 = b.g1; a.m0 = ix->goff_host[b.g0]; a.m1 = ix->goff_host[b.g1]; a.k0 = b.k0; a.W = b.W;
    a.cells = (uint32_t)b.cells;
    a.keys = c->v_keys.as<unsigned long long>();
    const unsigned cell_grid = capped_grid(c, b.cells, 256, 8);
    count_values_segments_kernel<<<capped_grid(c, b.segments, 256, 8), 256, 0, c->stream>>>(a);
    const uint64_t tiles = (uint64_t)((a.m1 - a.m0 + 31) / 32) * ((b.W + 31) / 32);
    (i64 ? count_values_scatter_kernel<I64Key> : count_values_scatter_kernel<F64Key>)<<<capped_grid(c, tiles, 1, 8), 256, 0, c->stream>>>(a);
    c->launches += 2;
    CU(cudaGetLastError());
    cub::DoubleBuffer<unsigned long long> db(c->v_keys.as<unsigned long long>(), c->v_alt.as<unsigned long long>());
    size_t bytes = c->v_tmp.cap;
    CU(cub::DeviceSegmentedSort::SortKeys(c->v_tmp.p, bytes, db, (int)b.cells, (int)b.segments, a.seg_off, a.seg_off + 1,
                                          c->stream));
    a.sorted = db.Current();
    a.start = reinterpret_cast<uint32_t*>(db.Alternate());
    count_values_head_kernel<<<cell_grid, 256, 0, c->stream>>>(a);
    c->launches++;
    CU(cudaGetLastError());
    bytes = c->v_tmp.cap;
    CU(cub::DeviceScan::InclusiveSum(c->v_tmp.p, bytes, a.rank, a.rank, (int)b.cells, c->stream));
    (i64 ? count_values_rank_kernel<I64Key> : count_values_rank_kernel<F64Key>)<<<cell_grid, 256, 0, c->stream>>>(a);
    count_values_count_kernel<<<cell_grid, 256, 0, c->stream>>>(a);
    c->launches += 2;
    CU(cudaGetLastError());
  }
  return B2P_OK;
}

// The end of a host call over a group index: stages gid, builds a temporary index of it, runs `dev(ix)`, finishes `s`
// and destroys the index once the copies have completed.
template <class Dev>
int end_indexed(Staging& s, const uint32_t* gid, uint32_t n_rows, uint32_t n_groups, Dev&& dev) {
  const uint32_t* d_gid = s.in(gid, (size_t)n_rows * 4);
  b2p_group_index* ix = nullptr;
  const int rc = s.end([&] {
    const int r = b2p_group_index_create_dev(s.c, d_gid, n_rows, n_groups, &ix);
    return r ? r : dev(ix);
  });
  b2p_group_index_destroy(s.c, ix);
  return rc;
}

// The device and host forms of topk / bottomk and count_values; i64: the grid is Int64
int topk_dev(b2p_ctx* c, int32_t bottom, double k, const double* vals, const uint32_t* valid, const b2p_group_index* ix,
             const uint32_t* tie, uint64_t T, uint32_t* out_valid, bool i64) {
  if (!c || !ix) return fail(B2P_E_INVALID, "NULL argument");
  if (ix->n_series == 0 || T == 0) return B2P_OK;
  if (!vals || !valid || !tie || !out_valid) return fail(B2P_E_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  stage_begin(c, 3);
  const int rc = topk_run(c, bottom, topk_ranks(k), vals, valid, ix, tie, T, out_valid, i64);
  stage_end(c, 3);
  return rc;
}

int topk_host(b2p_ctx* c, int32_t bottom, double k, const double* vals, const uint32_t* valid, const uint32_t* gid,
              uint32_t n_rows, uint32_t n_groups, const uint32_t* tie, uint64_t T, uint32_t* out_valid, bool i64) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  if (n_rows == 0 || T == 0) return B2P_OK;  // (no group index to build)
  DeviceGuard g(c->device);
  const size_t Tw = (size_t)((T + 31) / 32);
  Staging s{c};
  const double* d_vals = s.in(vals, (size_t)n_rows * T * 8);
  uint32_t* d_valid = s.in(valid, (size_t)n_rows * Tw * 4);
  const uint32_t* d_tie = s.in(tie, (size_t)n_rows * 4);
  uint32_t* d_out = s.copy_back(out_valid, d_valid, (size_t)n_rows * Tw * 4);  // topk runs in place
  return end_indexed(s, gid, n_rows, n_groups, [&](const b2p_group_index* ix) {
    return topk_dev(c, bottom, k, d_vals, d_valid, ix, d_tie, T, d_out, i64);
  });
}

int count_values_dev(b2p_ctx* c, const double* vals, const uint32_t* valid, const b2p_group_index* ix, uint64_t T,
                     double* out_val, uint32_t* out_cnt, bool i64) {
  if (!c || !ix) return fail(B2P_E_INVALID, "NULL argument");
  if (ix->n_series == 0 || T == 0) return B2P_OK;
  if (!vals || !valid || !out_val || !out_cnt) return fail(B2P_E_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  stage_begin(c, 3);
  const int rc = count_values_run(c, vals, valid, ix, T, out_val, out_cnt, i64);
  stage_end(c, 3);
  return rc;
}

int count_values_host(b2p_ctx* c, const double* vals, const uint32_t* valid, const uint32_t* gid, uint32_t n_rows,
                      uint32_t n_groups, uint64_t T, double* out_val, uint32_t* out_cnt, bool i64) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  if (n_rows == 0 || T == 0) return B2P_OK;  // (no group index to build)
  DeviceGuard g(c->device);
  const size_t Tw = (size_t)((T + 31) / 32);
  Staging s{c};
  const double* d_vals = s.in(vals, (size_t)n_rows * T * 8);
  const uint32_t* d_valid = s.in(valid, (size_t)n_rows * Tw * 4);
  double* d_out = s.out(out_val, (size_t)n_rows * T * 8);
  uint32_t* d_cnt = s.out(out_cnt, (size_t)n_rows * T * 4);
  return end_indexed(s, gid, n_rows, n_groups, [&](const b2p_group_index* ix) {
    return count_values_dev(c, d_vals, d_valid, ix, T, d_out, d_cnt, i64);
  });
}
}  // namespace

extern "C" {

/* ---- topk / bottomk ------------------------------------------------------------------------------------------ */

int b2p_topk_dev(b2p_ctx* c, int32_t bottom, double k, const double* vals, const uint32_t* valid,
                 const b2p_group_index* ix, const uint32_t* tie, uint64_t T, uint32_t* out_valid) {
  return topk_dev(c, bottom, k, vals, valid, ix, tie, T, out_valid, false);
}

int b2p_topk_i64_dev(b2p_ctx* c, int32_t bottom, double k, const int64_t* vals, const uint32_t* valid,
                     const b2p_group_index* ix, const uint32_t* tie, uint64_t T, uint32_t* out_valid) {
  return topk_dev(c, bottom, k, reinterpret_cast<const double*>(vals), valid, ix, tie, T, out_valid, true);
}

/* ---- quantile ------------------------------------------------------------------------------------------------ */

int b2p_group_quantile_dev(b2p_ctx* c, double phi, const double* vals, const uint32_t* valid, const b2p_group_index* ix,
                           uint64_t T, double* out_val, uint32_t* out_cnt) {
  if (!c || !ix) return fail(B2P_E_INVALID, "NULL argument");
  if (ix->n_groups == 0 || T == 0) return B2P_OK;
  if ((ix->n_series && (!vals || !valid)) || !out_val || !out_cnt) return fail(B2P_E_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  stage_begin(c, 3);
  const int rc = quantile_run(c, phi, vals, valid, ix, T, out_val, out_cnt);
  stage_end(c, 3);
  return rc;
}

/* ---- count_values -------------------------------------------------------------------------------------------- */

int b2p_count_values_dev(b2p_ctx* c, const double* vals, const uint32_t* valid, const b2p_group_index* ix, uint64_t T,
                         double* out_val, uint32_t* out_cnt) {
  return count_values_dev(c, vals, valid, ix, T, out_val, out_cnt, false);
}

int b2p_count_values_i64_dev(b2p_ctx* c, const int64_t* vals, const uint32_t* valid, const b2p_group_index* ix,
                             uint64_t T, int64_t* out_val, uint32_t* out_cnt) {
  return count_values_dev(c, reinterpret_cast<const double*>(vals), valid, ix, T, reinterpret_cast<double*>(out_val),
                          out_cnt, true);
}

/* ---- host-pointer API ------------------------------------------------------------------------ */

int b2p_topk(b2p_ctx* c, int32_t bottom, double k, const double* vals, const uint32_t* valid, const uint32_t* gid,
             uint32_t n_rows, uint32_t n_groups, const uint32_t* tie, uint64_t T, uint32_t* out_valid) {
  return topk_host(c, bottom, k, vals, valid, gid, n_rows, n_groups, tie, T, out_valid, false);
}

int b2p_topk_i64(b2p_ctx* c, int32_t bottom, double k, const int64_t* vals, const uint32_t* valid, const uint32_t* gid,
                 uint32_t n_rows, uint32_t n_groups, const uint32_t* tie, uint64_t T, uint32_t* out_valid) {
  return topk_host(c, bottom, k, reinterpret_cast<const double*>(vals), valid, gid, n_rows, n_groups, tie, T, out_valid,
                   true);
}

int b2p_group_quantile(b2p_ctx* c, double phi, const double* vals, const uint32_t* valid, const uint32_t* gid,
                       uint32_t n_rows, uint32_t n_groups, uint64_t T, double* out_val, uint32_t* out_cnt) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  if (n_groups == 0 || T == 0) return B2P_OK;  // (no group index to build)
  DeviceGuard g(c->device);
  const size_t Tw = (size_t)((T + 31) / 32);
  Staging s{c};
  const double* d_vals = s.in(vals, (size_t)n_rows * T * 8);
  const uint32_t* d_valid = s.in(valid, (size_t)n_rows * Tw * 4);
  double* d_out = s.out(out_val, (size_t)n_groups * T * 8);
  uint32_t* d_cnt = s.out(out_cnt, (size_t)n_groups * T * 4);
  return end_indexed(s, gid, n_rows, n_groups, [&](const b2p_group_index* ix) {
    return b2p_group_quantile_dev(c, phi, d_vals, d_valid, ix, T, d_out, d_cnt);
  });
}

int b2p_count_values(b2p_ctx* c, const double* vals, const uint32_t* valid, const uint32_t* gid, uint32_t n_rows,
                     uint32_t n_groups, uint64_t T, double* out_val, uint32_t* out_cnt) {
  return count_values_host(c, vals, valid, gid, n_rows, n_groups, T, out_val, out_cnt, false);
}

int b2p_count_values_i64(b2p_ctx* c, const int64_t* vals, const uint32_t* valid, const uint32_t* gid, uint32_t n_rows,
                         uint32_t n_groups, uint64_t T, int64_t* out_val, uint32_t* out_cnt) {
  return count_values_host(c, reinterpret_cast<const double*>(vals), valid, gid, n_rows, n_groups, T,
                           reinterpret_cast<double*>(out_val), out_cnt, true);
}

}  // extern "C"
