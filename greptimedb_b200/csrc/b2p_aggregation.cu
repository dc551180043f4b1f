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
      merges.push_back(TopkMerge{n_cand, n_cand + nc, n_state, 1});
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

// Cuts X items x `tiles` tiles into batches of at most `fit` (item, tile) units: every tile of every item when they fit,
// else every item x as many tiles as fit, else `fit` items x 1 tile -> xb items and tb tiles per batch
void cut_batches(uint64_t X, uint32_t tiles, uint64_t fit, uint32_t& xb, uint32_t& tb) {
  if (X * tiles <= fit) {
    xb = (uint32_t)X; tb = tiles;
  } else if (X <= fit) {
    xb = (uint32_t)X; tb = (uint32_t)(fit / X);
  } else {
    xb = (uint32_t)fit; tb = 1;
  }
}

// ---- sharded topk / bottomk: the rows of every rank, one exchange of candidates ---------------------------------------
// The exchange is derived from kk, T, the rank count and the global group sizes only, so every rank derives the same
// batches and block sizes.  Exchanged groups (G_x) are the groups of more than kk members globally, in id order.  The
// (exchanged group, tile) units are cut into batches whose blocks and state fit topk_exchange_cap: all the tiles of as
// many groups as fit, or groups x1 tile when one tile of every group does not fit.  Batch b covers tiles
// [t0, t0 + nt) of groups [x0, x0 + nx).
struct TopkShard {
  uint32_t kk = 0, K = 0, rounds = 0;
  int mode = 0;                   // 0: nothing kept; 1: every valid cell kept; 2: exchange
  std::vector<uint32_t> xg;       // exchanged group ids, ascending
  uint32_t tiles = 0, tb = 1, xb = 1, n_tb = 1, n_xb = 1, n_batches = 1;
  uint32_t n_ranks = 1;
  struct Batch { uint32_t x0, nx, t0, nt; };
  Batch batch(uint32_t b) const {
    const uint32_t x0 = (b % n_xb) * xb, t0 = (b / n_xb) * tb;
    return Batch{x0, std::min<uint32_t>(xb, (uint32_t)xg.size() - x0), t0, std::min(tb, tiles - t0)};
  }
  uint64_t slot_bytes() const { return (uint64_t)K * 12 + 4; }  // per (group, step): K keys (8 B + 4 B tie) and a count
  uint64_t block_bytes(const Batch& bt) const { return (uint64_t)bt.nx * bt.nt * 32 * slot_bytes(); }
  uint64_t state_bytes(const Batch& bt) const { return (uint64_t)bt.nx * bt.nt * 32 * 20; }
};

int shard_plan(const b2p_ctx* c, double k, const uint32_t* sizes, uint32_t n_groups, uint64_t T, int32_t n_ranks,
               TopkShard& sh) {
  if (n_ranks < 1) return fail(B2P_E_INVALID, "n_ranks %d < 1", n_ranks);
  if (n_groups && !sizes) return fail(B2P_E_INVALID, "NULL argument");
  sh.n_ranks = (uint32_t)n_ranks;
  sh.kk = topk_ranks(k);
  sh.tiles = (uint32_t)((T + 31) / 32);
  uint32_t largest = 0;
  for (uint32_t g = 0; g < n_groups; ++g) largest = std::max(largest, sizes[g]);
  sh.mode = sh.kk == 0 ? 0 : (sh.kk >= largest ? 1 : 2);
  if (sh.mode != 2 || T == 0) return B2P_OK;  // one batch without rounds: the words alone
  for (uint32_t g = 0; g < n_groups; ++g)
    if (sizes[g] > sh.kk) sh.xg.push_back(g);
  sh.K = std::min(sh.kk, kTopkMax);
  sh.rounds = sh.kk > kTopkMax ? (sh.kk + kTopkMax - 1) / kTopkMax : 1;
  const uint64_t X = sh.xg.size();
  const uint64_t unit = (uint64_t)(sh.n_ranks + 1) * 32 * sh.slot_bytes() + 32 * 20;  // send, gathered, state
  cut_batches(X, sh.tiles, std::max<uint64_t>(1, c->topk_exchange_cap / unit), sh.xb, sh.tb);
  sh.n_xb = (uint32_t)((X + sh.xb - 1) / sh.xb);
  sh.n_tb = (sh.tiles + sh.tb - 1) / sh.tb;
  sh.n_batches = sh.n_xb * sh.n_tb;
  return B2P_OK;
}

// This rank's chunks of the batch's exchanged groups (each chunk leaves a candidate list; state = the group's place in
// the batch) and one merge per exchanged group, with no chunk where the rank holds no member; the tables go to t_table
// and a is set up over them (candidate lists in t_cand).  The same inputs give the same tables, so the mark of a batch
// finds the lists its candidates step left.
int shard_local(b2p_ctx* c, const TopkShard& sh, const TopkShard::Batch& bt, const b2p_group_index* ix, TopkArgs& a) {
  int rc;
  const size_t smem = kTopkWarps * topk_warp_bytes(sh.K);
  unsigned cap = 0;
  if ((rc = persistent_grid(c, topk_chunk_kernel<F64Key>, smem, kTopkWarps, kAllResident, &cap))) return rc;
  const uint64_t resident = (uint64_t)cap * kTopkWarps, U = resident - resident / 8;
  uint64_t members = 0;
  for (uint32_t i = 0; i < bt.nx; ++i) {
    const uint32_t g = sh.xg[bt.x0 + i];
    if (g < ix->n_groups) members += ix->goff_host[g + 1] - ix->goff_host[g];
  }
  const uint64_t C = std::max<uint64_t>(256, (members * bt.nt + U - 1) / U);
  std::vector<TopkChunk> chunks;
  std::vector<TopkMerge> merges;
  uint32_t n_cand = 0;
  for (uint32_t i = 0; i < bt.nx; ++i) {
    const uint32_t g = sh.xg[bt.x0 + i];
    const uint32_t b = g < ix->n_groups ? ix->goff_host[g] : 0, e = g < ix->n_groups ? ix->goff_host[g + 1] : 0;
    const uint32_t s = e - b, nc = (uint32_t)((s + C - 1) / C);
    merges.push_back(TopkMerge{n_cand, n_cand + nc, i, 1});
    for (uint32_t j = 0; j < nc; ++j)
      chunks.push_back(TopkChunk{b + (uint32_t)((uint64_t)s * j / nc), b + (uint32_t)((uint64_t)s * (j + 1) / nc),
                                 n_cand++, i});
  }
  const size_t tb_chunks = chunks.size() * sizeof(TopkChunk), tb_merges = merges.size() * sizeof(TopkMerge);
  if ((rc = c->t_table.ensure(tb_chunks + tb_merges + 16))) return rc;
  if (tb_chunks) CU(cudaMemcpyAsync(c->t_table.p, chunks.data(), tb_chunks, cudaMemcpyHostToDevice, c->stream));
  CU(cudaMemcpyAsync(c->t_table.as<char>() + tb_chunks, merges.data(), tb_merges, cudaMemcpyHostToDevice, c->stream));
  const size_t cand_units = (size_t)n_cand * bt.nt, cand_slots = cand_units * sh.K * 32;
  if ((rc = c->t_cand.ensure(cand_slots * 16 + cand_units * 32 * 4 + 64))) return rc;
  a.members = ix->members;
  a.chunks = c->t_table.as<TopkChunk>(); a.n_chunks = (uint32_t)chunks.size();
  a.merges = reinterpret_cast<const TopkMerge*>(c->t_table.as<char>() + tb_chunks); a.n_merges = (uint32_t)merges.size();
  a.c_hi = c->t_cand.as<unsigned long long>();
  a.c_lo = reinterpret_cast<uint32_t*>(a.c_hi + cand_slots);
  a.c_pos = a.c_lo + cand_slots;
  a.c_n = a.c_pos + cand_slots;
  return B2P_OK;
}

// The arguments every shard step shares; state: the batch's selection state, [unit][lane] sections hi, lo, rem, flags
TopkArgs shard_args(const TopkShard& sh, const TopkShard::Batch& bt, uint64_t T, void* state) {
  TopkArgs a{};
  a.T = T; a.Tw = sh.tiles; a.tiles = bt.nt; a.tile0 = bt.t0;
  a.K = sh.K; a.kk = sh.kk; a.general = sh.rounds > 1 ? 1 : 0;
  const size_t cells = (size_t)bt.nx * bt.nt * 32;
  a.s_hi = static_cast<unsigned long long*>(state);
  a.s_lo = reinterpret_cast<uint32_t*>(a.s_hi + cells);
  a.s_rem = a.s_lo + cells;
  a.s_flags = a.s_rem + cells;
  return a;
}

template <class Kern>
int topk_launch(b2p_ctx* c, Kern* kern, size_t smem, uint64_t units, const TopkArgs& a) {
  unsigned grid = 0;
  if (int rc = persistent_grid(c, kern, smem, kTopkWarps, units, &grid)) return rc;
  if (grid == 0) return B2P_OK;
  kern<<<grid, kTopkWarps * 32, smem, c->stream>>>(a);
  c->launches++;
  CU(cudaGetLastError());
  return B2P_OK;
}

// A block of bt's units: [hi: units x K x 32 u64][lo: units x K x 32 u32][n: units x 32 u32]; the gathered blocks of R
// ranks: each section of every rank in rank order, [hi of rank 0 .. R-1][lo ..][n ..], as three all-gathers lay them
struct ShardBlock {
  unsigned long long* hi;
  uint32_t* lo;
  uint32_t* n;
};
ShardBlock shard_block(const TopkShard& sh, const TopkShard::Batch& bt, void* p, uint32_t ranks) {
  const size_t slots = (size_t)bt.nx * bt.nt * sh.K * 32 * ranks;
  ShardBlock k;
  k.hi = static_cast<unsigned long long*>(p);
  k.lo = reinterpret_cast<uint32_t*>(k.hi + slots);
  k.n = k.lo + slots;
  return k;
}

// Per-rank step: this rank's best K keys below the bound of every (exchanged group, step) of the batch -> block
int shard_candidates(b2p_ctx* c, const TopkShard& sh, uint32_t b, uint32_t round, int bottom, const double* vals,
                     const uint32_t* valid, const b2p_group_index* ix, const uint32_t* tie, uint64_t T, void* state,
                     void* block) {
  const TopkShard::Batch bt = sh.batch(b);
  TopkArgs a = shard_args(sh, bt, T, state);
  int rc;
  if ((rc = shard_local(c, sh, bt, ix, a))) return rc;
  a.vals = vals; a.valid = valid; a.tie = tie; a.bottom = bottom ? 1 : 0; a.round = (int)round;
  const size_t smem = kTopkWarps * topk_warp_bytes(sh.K);
  if ((rc = topk_launch(c, topk_chunk_kernel<F64Key>, smem, (uint64_t)a.n_chunks * bt.nt, a))) return rc;
  const ShardBlock x = shard_block(sh, bt, block, 1);
  a.x_hi = x.hi; a.x_lo = x.lo; a.x_n = x.n;
  if ((rc = topk_launch(c, topk_merge_kernel, smem, (uint64_t)bt.nx * bt.nt, a))) return rc;
  c->last_exchange_bytes += (long long)sh.block_bytes(bt);
  return B2P_OK;
}

// Merge step: the verdict of the round over the gathered blocks of every rank -> state
int shard_merge(b2p_ctx* c, const TopkShard& sh, uint32_t b, uint32_t round, const void* blocks, void* state, uint64_t T) {
  const TopkShard::Batch bt = sh.batch(b);
  TopkArgs a = shard_args(sh, bt, T, state);
  std::vector<TopkMerge> merges(bt.nx);
  for (uint32_t i = 0; i < bt.nx; ++i) merges[i] = TopkMerge{i, i + sh.n_ranks * bt.nx, i, bt.nx};
  int rc;
  if ((rc = c->x_table.ensure(merges.size() * sizeof(TopkMerge)))) return rc;
  CU(cudaMemcpyAsync(c->x_table.p, merges.data(), merges.size() * sizeof(TopkMerge), cudaMemcpyHostToDevice, c->stream));
  const ShardBlock x = shard_block(sh, bt, const_cast<void*>(blocks), sh.n_ranks);
  a.merges = c->x_table.as<TopkMerge>(); a.n_merges = bt.nx;
  a.c_hi = x.hi; a.c_lo = x.lo; a.c_n = x.n;
  a.round = (int)round;
  return topk_launch(c, topk_merge_kernel, kTopkWarps * topk_warp_bytes(sh.K), (uint64_t)bt.nx * bt.nt, a);
}

// Mark step: this rank's words of the batch from the state after the last round.  Batch 0 first writes the words of
// every row the exchange does not decide: 0 when nothing is kept and for rows of no group, the valid cells otherwise
// (the exchanged groups' rows are overwritten by their batches).
int shard_mark(b2p_ctx* c, const TopkShard& sh, uint32_t b, int bottom, const double* vals, const uint32_t* valid,
               const b2p_group_index* ix, const uint32_t* tie, uint64_t T, const void* state, uint32_t* out_valid) {
  const uint32_t R = ix->n_series;
  const size_t words = (size_t)R * sh.tiles;
  if (b == 0 && words) {
    if (sh.mode == 0) {
      CU(cudaMemsetAsync(out_valid, 0, words * 4, c->stream));
    } else {
      topk_copy_kernel<<<capped_grid(c, words, 256, 16), 256, 0, c->stream>>>(valid, ix->gid, ix->n_groups, R, T,
                                                                              sh.tiles, 0, out_valid);
      c->launches++;
      CU(cudaGetLastError());
    }
  }
  if (sh.mode != 2) return B2P_OK;
  const TopkShard::Batch bt = sh.batch(b);
  TopkArgs a = shard_args(sh, bt, T, const_cast<void*>(state));
  int rc;
  if ((rc = shard_local(c, sh, bt, ix, a))) return rc;
  if (a.n_chunks == 0) return B2P_OK;
  a.vals = vals; a.valid = valid; a.tie = tie; a.bottom = bottom ? 1 : 0; a.out_valid = out_valid;
  const uint64_t units = (uint64_t)a.n_chunks * bt.nt;
  if (sh.rounds > 1) {
    topk_select_kernel<F64Key><<<capped_grid(c, units, 8, 16), 256, 0, c->stream>>>(a);
    c->launches++;
    CU(cudaGetLastError());
    return B2P_OK;
  }
  return topk_launch(c, topk_mark_kernel, 0, units, a);
}

// The composed call: the global group sizes (one all-reduce and one read-back), then per batch the rounds of
// candidates, all-gather and merge, and the mark.  Without a communicator (one rank) the block is its own gather.
int topk_allgather_run(b2p_ctx* c, int bottom, double k, const double* vals, const uint32_t* valid,
                       const b2p_group_index* ix, const uint32_t* tie, uint64_t T, uint32_t* out_valid) {
  int rc;
  const uint32_t G = ix->n_groups;
  std::vector<uint32_t> sizes(G);
  for (uint32_t g = 0; g < G; ++g) sizes[g] = ix->goff_host[g + 1] - ix->goff_host[g];
  if (c->comm && G) {
    if ((rc = c->x_size.ensure((size_t)G * 4))) return rc;
    CU(cudaMemcpyAsync(c->x_size.p, sizes.data(), (size_t)G * 4, cudaMemcpyHostToDevice, c->stream));
    NCCL_TRY(g_nccl.AllReduce(c->x_size.p, c->x_size.p, G, Nccl::kUint32, Nccl::kSum, c->comm, c->stream));
    CU(cudaMemcpyAsync(sizes.data(), c->x_size.p, (size_t)G * 4, cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
  }
  TopkShard sh;
  if ((rc = shard_plan(c, k, sizes.data(), G, T, c->comm_ranks, sh))) return rc;
  c->last_exchange_bytes = 0;
  if (sh.mode == 2) {
    const TopkShard::Batch b0 = sh.batch(0);  // the largest block
    if ((rc = c->x_send.ensure(sh.block_bytes(b0))) || (rc = c->x_state.ensure(sh.state_bytes(b0)))) return rc;
    if (c->comm && (rc = c->x_recv.ensure(sh.block_bytes(b0) * sh.n_ranks))) return rc;
  }
  for (uint32_t b = 0; b < sh.n_batches; ++b) {
    for (uint32_t r = 0; r < sh.rounds; ++r) {
      if ((rc = shard_candidates(c, sh, b, r, bottom, vals, valid, ix, tie, T, c->x_state.p, c->x_send.p))) return rc;
      const void* gathered = c->x_send.p;
      if (c->comm) {
        const TopkShard::Batch bt = sh.batch(b);
        const size_t n_slots = (size_t)bt.nx * bt.nt * sh.K * 32, n_units = (size_t)bt.nx * bt.nt * 32;
        const ShardBlock s = shard_block(sh, bt, c->x_send.p, 1), g = shard_block(sh, bt, c->x_recv.p, sh.n_ranks);
        NCCL_TRY(g_nccl.GroupStart());
        NCCL_TRY(g_nccl.AllGather(s.hi, g.hi, n_slots, Nccl::kUint64, c->comm, c->stream));
        NCCL_TRY(g_nccl.AllGather(s.lo, g.lo, n_slots, Nccl::kUint32, c->comm, c->stream));
        NCCL_TRY(g_nccl.AllGather(s.n, g.n, n_units, Nccl::kUint32, c->comm, c->stream));
        NCCL_TRY(g_nccl.GroupEnd());
        gathered = c->x_recv.p;
      }
      if ((rc = shard_merge(c, sh, b, r, gathered, c->x_state.p, T))) return rc;
    }
    if ((rc = shard_mark(c, sh, b, bottom, vals, valid, ix, tie, T, c->x_state.p, out_valid))) return rc;
  }
  return B2P_OK;
}

// Argument checks of the per-rank steps: the exchange of (k, sizes, T, n_ranks), and batch / round inside it
int shard_check(b2p_ctx* c, double k, const uint32_t* sizes, uint32_t n_groups, uint64_t T, int32_t n_ranks,
                uint32_t batch, uint32_t round, bool rounds, TopkShard& sh) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  if (int rc = shard_plan(c, k, sizes, n_groups, T, n_ranks, sh)) return rc;
  if (batch >= sh.n_batches) return fail(B2P_E_INVALID, "batch %u of %u", batch, sh.n_batches);
  if (rounds && round >= sh.rounds) return fail(B2P_E_INVALID, "round %u of %u", round, sh.rounds);
  return B2P_OK;
}

template <class Kern>
int quantile_launch(b2p_ctx* c, Kern* kern, size_t smem, uint64_t units, const QuantArgs& a) {
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
  const size_t smem = kQuantWarps * kQuantWarpBytes;
  if ((rc = quantile_launch(c, quantile_resident_kernel, smem, (uint64_t)G * Tw, a))) return rc;
  if (a.count_only || ix->max_members <= kQuantResident) return B2P_OK;
  unsigned cap = 0;
  if ((rc = persistent_grid(c, quantile_pass_kernel<8>, smem, kQuantWarps, kAllResident, &cap))) return rc;
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
    if ((rc = quantile_launch(c, quantile_pass_kernel<8>, smem, units, a))) return rc;
    if (!a.n_slots) break;
    quantile_advance_kernel<8><<<capped_grid(c, (uint64_t)a.n_slots * T, 256, 8), 256, 0, c->stream>>>(a);
    c->launches++;
    CU(cudaGetLastError());
  }
  return B2P_OK;
}

// ---- sharded quantile: the rows of every rank, one all-reduce of digit counts per pass ----------------------------------
// The 4-bit select of b2p_quantile.cuh over the union of the ranks' rows.  Every rank derives the same batches from
// (n_groups, T, topk_exchange_cap): the (group, tile) units are cut into batches whose block (kUnitBlock per unit) and
// state (kUnitState per unit) fit the cap.  Batch b covers tiles [t0, t0 + nt) of groups [g0, g0 + ng).  Its block is
// [counts: units x 16 x 32 u32][r_lo: units x 32 u64][r_hi: units x 32 u64]; its state [units x 32] QuantState.
struct QuantShard {
  static constexpr uint64_t kCountBytes = (1u << kQuantShardBits) * 32 * 4;
  static constexpr uint64_t kUnitBlock = kCountBytes + 2 * 32 * 8;  // 2 560 B
  static constexpr uint64_t kUnitState = 32 * sizeof(QuantState);   // 1 792 B
  uint32_t n_groups = 0, tiles = 0, gb = 1, tb = 1, n_gb = 0, n_batches = 0;
  struct Batch {
    uint32_t g0, ng, t0, nt;
    uint64_t units() const { return (uint64_t)ng * nt; }
  };
  Batch batch(uint32_t b) const {
    const uint32_t g0 = (b % n_gb) * gb, t0 = (b / n_gb) * tb;
    return Batch{g0, std::min(gb, n_groups - g0), t0, std::min(tb, tiles - t0)};
  }
};
static_assert(QuantShard::kUnitBlock == 2560, "b200promql.h states 2 560 B per (group, tile) unit and pass");

QuantShard quantile_shard_plan(const b2p_ctx* c, uint32_t n_groups, uint64_t T) {
  QuantShard sh;
  sh.n_groups = n_groups;
  sh.tiles = (uint32_t)((T + 31) / 32);
  if (n_groups == 0 || T == 0) return sh;  // no batch
  const uint64_t fit = std::max<uint64_t>(1, c->topk_exchange_cap / (QuantShard::kUnitBlock + QuantShard::kUnitState));
  cut_batches(n_groups, sh.tiles, fit, sh.gb, sh.tb);
  sh.n_gb = (n_groups + sh.gb - 1) / sh.gb;
  sh.n_batches = sh.n_gb * ((sh.tiles + sh.tb - 1) / sh.tb);
  return sh;
}

// The arguments both steps share: the batch, the state and the sections of a block
QuantArgs quantile_shard_args(const QuantShard& sh, const QuantShard::Batch& bt, double phi, uint64_t T, void* state,
                              void* block) {
  QuantArgs a{};
  a.T = T; a.Tw = sh.tiles; a.tiles = bt.nt; a.tile0 = bt.t0; a.group0 = bt.g0; a.n_slots = bt.ng;
  a.phi = phi;
  a.count_only = !(phi >= 0.0 && phi <= 1.0) ? 1 : 0;
  a.state = static_cast<QuantState*>(state);
  a.hist = static_cast<uint32_t*>(block);
  a.r_lo = reinterpret_cast<unsigned long long*>(static_cast<char*>(block) + bt.units() * QuantShard::kCountBytes);
  a.r_hi = a.r_lo + bt.units() * 32;
  return a;
}

// Per-rank step: zeroes the block (counts and r_lo 0, r_hi ~0; pass 0 also clears the batch's state), then this rank's
// chunks of the batch's groups add one pass's counts or extremes into it.  Chunks are cut as quantile_run cuts them.
int quantile_shard_pass(b2p_ctx* c, const QuantShard& sh, uint32_t b, uint32_t pass, double phi, const double* vals,
                        const uint32_t* valid, const b2p_group_index* ix, uint64_t T, void* block) {
  int rc;
  const QuantShard::Batch bt = sh.batch(b);
  const uint64_t units = bt.units();
  if (pass == 0) {
    if ((rc = c->qx_state.ensure(units * QuantShard::kUnitState))) return rc;
    CU(cudaMemsetAsync(c->qx_state.p, 0, units * QuantShard::kUnitState, c->stream));
  }
  char* blk = static_cast<char*>(block);
  CU(cudaMemsetAsync(blk, 0, units * (QuantShard::kCountBytes + 32 * 8), c->stream));
  CU(cudaMemsetAsync(blk + units * (QuantShard::kCountBytes + 32 * 8), 0xFF, units * 32 * 8, c->stream));
  c->last_exchange_bytes += (long long)(units * QuantShard::kUnitBlock);
  const size_t smem = kQuantWarps * quant_pass_warp_bytes<kQuantShardBits>();
  unsigned cap = 0;
  if ((rc = persistent_grid(c, quantile_pass_kernel<kQuantShardBits>, smem, kQuantWarps, kAllResident, &cap))) return rc;
  const uint64_t resident = (uint64_t)cap * kQuantWarps, U = resident - resident / 8;
  uint64_t members = 0;
  for (uint32_t g = bt.g0; g < bt.g0 + bt.ng; ++g) members += ix->goff_host[g + 1] - ix->goff_host[g];
  const uint64_t C = std::min<uint64_t>(kQuantChunkMax, std::max<uint64_t>(256, (members * bt.nt + U - 1) / U));
  std::vector<QuantChunk> chunks;
  for (uint32_t i = 0; i < bt.ng; ++i) {
    const uint32_t g = bt.g0 + i, gb = ix->goff_host[g], s = ix->goff_host[g + 1] - gb;
    const uint32_t nc = (uint32_t)((s + C - 1) / C);
    for (uint32_t j = 0; j < nc; ++j)
      chunks.push_back(QuantChunk{gb + (uint32_t)((uint64_t)s * j / nc), gb + (uint32_t)((uint64_t)s * (j + 1) / nc), g, i});
  }
  if (chunks.empty()) return B2P_OK;  // no member of the batch's groups on this rank: its block stays zero
  const size_t tb_chunks = chunks.size() * sizeof(QuantChunk);
  if ((rc = c->qx_table.ensure(tb_chunks))) return rc;
  CU(cudaMemcpyAsync(c->qx_table.p, chunks.data(), tb_chunks, cudaMemcpyHostToDevice, c->stream));
  QuantArgs a = quantile_shard_args(sh, bt, phi, T, c->qx_state.p, block);
  a.vals = vals; a.valid = valid; a.members = ix->members;
  a.chunks = c->qx_table.as<QuantChunk>(); a.n_chunks = (uint32_t)chunks.size();
  return quantile_launch(c, quantile_pass_kernel<kQuantShardBits>, smem, (uint64_t)a.n_chunks * bt.nt, a);
}

// Merge step: the n_blocks blocks of the batch (the batch's block size apart) advance this context's state; finished
// cells are written to out_val / out_cnt, and *live receives the count of the others (read back: synchronises)
int quantile_shard_advance(b2p_ctx* c, const QuantShard& sh, uint32_t b, double phi, uint64_t T, const void* blocks,
                           uint32_t n_blocks, double* out_val, uint32_t* out_cnt, uint64_t* live) {
  int rc;
  const QuantShard::Batch bt = sh.batch(b);
  const uint64_t units = bt.units();
  if (c->qx_state.cap < units * QuantShard::kUnitState)
    return fail(B2P_E_INVALID, "no selection state for batch %u: its pass 0 runs first on this context", b);
  if ((rc = c->qx_live.ensure(8))) return rc;
  QuantArgs a = quantile_shard_args(sh, bt, phi, T, c->qx_state.p, const_cast<void*>(blocks));
  a.block_stride = units * QuantShard::kUnitBlock;
  a.n_blocks = n_blocks;
  a.live = c->qx_live.as<unsigned long long>();
  a.out_val = out_val; a.out_cnt = out_cnt;
  CU(cudaMemsetAsync(a.live, 0, 8, c->stream));
  quantile_advance_kernel<kQuantShardBits><<<capped_grid(c, units * 32, 256, 8), 256, 0, c->stream>>>(a);
  c->launches++;
  CU(cudaGetLastError());
  unsigned long long left = 0;
  CU(cudaMemcpyAsync(&left, a.live, 8, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  *live = left;
  return B2P_OK;
}

// The composed call: per batch and pass, this rank's block, one group of three in-place all-reduces (counts SUM, r_lo
// MAX, r_hi MIN), and the advance over the one merged block, until no cell is left.  Without a communicator (one rank)
// the block is its own merge.
int quantile_allreduce_run(b2p_ctx* c, double phi, const double* vals, const uint32_t* valid, const b2p_group_index* ix,
                           uint64_t T, double* out_val, uint32_t* out_cnt) {
  int rc;
  const QuantShard sh = quantile_shard_plan(c, ix->n_groups, T);
  if (sh.n_batches && (rc = c->x_send.ensure(sh.batch(0).units() * QuantShard::kUnitBlock))) return rc;
  for (uint32_t b = 0; b < sh.n_batches; ++b) {
    const uint64_t units = sh.batch(b).units();
    for (uint32_t p = 0; p < kQuantShardPasses; ++p) {
      if ((rc = quantile_shard_pass(c, sh, b, p, phi, vals, valid, ix, T, c->x_send.p))) return rc;
      if (c->comm) {
        char* blk = c->x_send.as<char>();
        void* r_lo = blk + units * QuantShard::kCountBytes;
        void* r_hi = blk + units * (QuantShard::kCountBytes + 32 * 8);
        NCCL_TRY(g_nccl.GroupStart());
        NCCL_TRY(g_nccl.AllReduce(blk, blk, units * (1u << kQuantShardBits) * 32, Nccl::kUint32, Nccl::kSum, c->comm, c->stream));
        NCCL_TRY(g_nccl.AllReduce(r_lo, r_lo, units * 32, Nccl::kUint64, Nccl::kMax, c->comm, c->stream));
        NCCL_TRY(g_nccl.AllReduce(r_hi, r_hi, units * 32, Nccl::kUint64, Nccl::kMin, c->comm, c->stream));
        NCCL_TRY(g_nccl.GroupEnd());
      }
      uint64_t live = 0;
      if ((rc = quantile_shard_advance(c, sh, b, phi, T, c->x_send.p, 1, out_val, out_cnt, &live))) return rc;
      if (live == 0) break;  // from the merged state alone, so every rank stops after the same pass
    }
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

// ---- sharded count_values: every rank's distinct values and counts, one all-gather per batch ----------------------
// The exchange is derived from (heights, n_ranks, n_groups, T, topk_exchange_cap) only, so every rank derives the same
// batches.  Group g has U_g = sum over ranks of h_r(g) output rows from uoff[g].  Windows of W steps (every step when
// the costliest group fits the cap over all of them, else a multiple of 32, at least 32), each cut into runs of whole
// groups whose send block, gathered blocks and merge scratch fit the cap; a group too large for the cap alone is a
// batch of its own.  Batches without an output row are left out.  Per step of a batch: (R + 1) x P' x 12 B of blocks
// (P' = max over ranks of its summed heights), 28 B of merge scratch per merged entry (arranged and sorted key and
// count, the run rank; the start and sum tables reuse the sort's alternate buffers) and 4 B per segment.
struct CvShard {
  static constexpr uint64_t kEntry = 12;        // key u64 and count u32
  static constexpr uint64_t kMergeEntry = 28;
  static constexpr uint64_t kMergeSegment = 4;
  uint32_t n_ranks = 1, n_groups = 0;
  uint64_t T = 0;
  const uint32_t* h = nullptr;   // [n_ranks x n_groups], host
  std::vector<uint32_t> uoff;    // [n_groups + 1]
  struct Batch {
    uint32_t g0, g1, k0, W;
    uint64_t P;                  // entries of each rank's block: W x max over ranks of the batch's summed heights
    uint64_t rows;               // output rows of the batch: sum of U_g
  };
  std::vector<Batch> batches;
  uint32_t height(uint32_t r, uint32_t g) const { return h[(uint64_t)r * n_groups + g]; }
  uint64_t max_block() const {
    uint64_t p = 0;
    for (const Batch& b : batches) p = std::max(p, b.P);
    return p * kEntry;
  }
};

int cv_shard_plan(const b2p_ctx* c, const uint32_t* heights, int32_t n_ranks, uint32_t n_groups, uint64_t T,
                  CvShard& sh) {
  if (n_ranks < 1) return fail(B2P_E_INVALID, "n_ranks %d < 1", n_ranks);
  if (n_groups && !heights) return fail(B2P_E_INVALID, "NULL argument");
  const uint32_t R = (uint32_t)n_ranks, G = n_groups;
  sh.n_ranks = R; sh.n_groups = G; sh.T = T; sh.h = heights;
  sh.uoff.assign(G + 1, 0u);
  uint64_t worst = 0;
  for (uint32_t g = 0; g < G; ++g) {
    uint64_t u = 0, hm = 0;
    for (uint32_t r = 0; r < R; ++r) {
      u += sh.height(r, g);
      hm = std::max<uint64_t>(hm, sh.height(r, g));
    }
    if (sh.uoff[g] + u > UINT32_MAX) return fail(B2P_E_TOO_LARGE, "count_values: more than 2^32 - 1 output rows");
    if (u * std::min<uint64_t>(32, T) > (uint64_t)INT32_MAX)
      return fail(B2P_E_TOO_LARGE, "count_values: a group of %llu merged rows is too large", (unsigned long long)u);
    sh.uoff[g + 1] = sh.uoff[g] + (uint32_t)u;
    if (u) worst = std::max(worst, (R + 1) * CvShard::kEntry * hm + CvShard::kMergeEntry * u + CvShard::kMergeSegment);
  }
  if (T == 0 || G == 0 || sh.uoff[G] == 0) return B2P_OK;  // no batch
  const uint64_t cap = c->topk_exchange_cap;
  const uint64_t W = std::min<uint64_t>((T + 31) / 32 * 32, std::max<uint64_t>(32, cap / worst / 32 * 32));
  std::vector<uint64_t> run(R);
  for (uint64_t k0 = 0; k0 < T; k0 += W) {
    const uint64_t Wb = std::min<uint64_t>(W, T - k0);
    for (uint32_t g = 0; g < G;) {
      const uint32_t g0 = g;
      std::fill(run.begin(), run.end(), 0);
      uint64_t pmax = 0, rows = 0;
      for (; g < G; ++g) {
        uint64_t pm = pmax;
        for (uint32_t r = 0; r < R; ++r) pm = std::max(pm, run[r] + sh.height(r, g));
        const uint64_t u = sh.uoff[g + 1] - sh.uoff[g];
        const uint64_t bytes = ((R + 1) * CvShard::kEntry * pm + CvShard::kMergeEntry * (rows + u) +
                                CvShard::kMergeSegment * (g + 1 - g0)) * Wb;
        if (g > g0 && bytes > cap) break;
        for (uint32_t r = 0; r < R; ++r) run[r] += sh.height(r, g);
        pmax = pm;
        rows += u;
      }
      if (rows == 0) continue;  // groups without a value on any rank: no output row
      if (std::max<uint64_t>(rows, g - g0) * Wb > (uint64_t)INT32_MAX)
        return fail(B2P_E_TOO_LARGE, "count_values: a batch of %llu merged rows is too large", (unsigned long long)rows);
      sh.batches.push_back(CvShard::Batch{g0, g, (uint32_t)k0, (uint32_t)Wb, pmax * Wb, rows});
    }
  }
  return B2P_OK;
}

// This rank's row of heights against its own index: h_r(g) <= its member count of g
int cv_shard_check_rank(const CvShard& sh, const b2p_group_index* ix, uint32_t rank) {
  if (ix->n_groups != sh.n_groups) return fail(B2P_E_INVALID, "index of %u groups, heights of %u", ix->n_groups, sh.n_groups);
  if (rank >= sh.n_ranks) return fail(B2P_E_INVALID, "rank %u of %u", rank, sh.n_ranks);
  for (uint32_t g = 0; g < sh.n_groups; ++g)
    if (sh.height(rank, g) > ix->goff_host[g + 1] - ix->goff_host[g])
      return fail(B2P_E_INVALID, "heights: %u rows of group %u on rank %u, which has %u", sh.height(rank, g), g, rank,
                  ix->goff_host[g + 1] - ix->goff_host[g]);
  return B2P_OK;
}

// h_r(g) of this rank into `heights` (host): [n_groups], or with a communicator every rank's row [n_ranks x n_groups]
// (one in-place all-gather).  Reads the table back, so it synchronises the stream.
int cv_shard_heights(b2p_ctx* c, const uint32_t* cnt, const b2p_group_index* ix, uint64_t T, uint32_t* heights) {
  int rc;
  const uint32_t G = ix->n_groups, R = c->comm ? (uint32_t)c->comm_ranks : 1u;
  if (G == 0) return B2P_OK;
  if ((rc = c->x_size.ensure((size_t)R * G * 4))) return rc;
  uint32_t* mine = c->x_size.as<uint32_t>() + (c->comm ? (size_t)c->comm_rank * G : 0);
  CU(cudaMemsetAsync(mine, 0, (size_t)G * 4, c->stream));
  const uint32_t in_rows = ix->goff_host[G];
  if (in_rows && T) {
    count_values_heights_kernel<<<capped_grid(c, in_rows, 8, 16), 256, 0, c->stream>>>(cnt, ix->gid, ix->members,
                                                                                        ix->goff, in_rows, T, mine);
    c->launches++;
    CU(cudaGetLastError());
  }
  if (c->comm)
    NCCL_TRY(g_nccl.AllGather(mine, c->x_size.p, G, Nccl::kUint32, c->comm, c->stream));
  CU(cudaMemcpyAsync(heights, c->x_size.p, (size_t)R * G * 4, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  return B2P_OK;
}

// Per-rank step: this rank's block of batch b, [keys: P u64][counts: P u32] (P the batch's padded entry count; the
// entries past the rank's own are not written and never read).  i64: the grid is Int64 (I64Key).
int cv_shard_pack(b2p_ctx* c, const CvShard& sh, uint32_t b, uint32_t rank, const double* vals, const uint32_t* cnt,
                  const b2p_group_index* ix, void* block, bool i64) {
  int rc;
  const CvShard::Batch& bt = sh.batches[b];
  const uint32_t ng = bt.g1 - bt.g0;
  std::vector<uint32_t> hoff(ng + 1, 0u);
  for (uint32_t q = 0; q < ng; ++q) hoff[q + 1] = hoff[q] + sh.height(rank, bt.g0 + q);
  c->last_exchange_bytes += (long long)(bt.P * CvShard::kEntry);
  if (hoff[ng] == 0) return B2P_OK;  // no entry of this rank in the batch
  if ((rc = c->x_table.ensure((ng + 1) * 4))) return rc;
  CU(cudaMemcpyAsync(c->x_table.p, hoff.data(), (ng + 1) * 4, cudaMemcpyHostToDevice, c->stream));
  CvShardArgs a{};
  a.T = sh.T; a.k0 = bt.k0; a.W = bt.W; a.g0 = bt.g0; a.ng = ng;
  a.off = c->x_table.as<uint32_t>();
  a.vals = vals; a.cnt = cnt; a.goff = ix->goff;
  a.bkeys = static_cast<unsigned long long*>(block);
  a.bcnt = reinterpret_cast<uint32_t*>(a.bkeys + bt.P);
  (i64 ? count_values_pack_kernel<I64Key> : count_values_pack_kernel<F64Key>)
      <<<capped_grid(c, (uint64_t)hoff[ng] * bt.W, 256, 8), 256, 0, c->stream>>>(a);
  c->launches++;
  CU(cudaGetLastError());
  return B2P_OK;
}

// Merge step: the n_ranks gathered blocks of batch b, [keys of rank 0 .. R-1][counts of rank 0 .. R-1] (each rank's
// section P entries), into the batch's rows of out_val / out_cnt.  Per batch: the tables, the segment offsets, the
// arrange, CUB's segmented sort of (key, count) pairs, the head flags, CUB's scans of the flags and of the counts, the
// run starts and the output; no host round trip.
int cv_shard_merge(b2p_ctx* c, const CvShard& sh, uint32_t b, const void* blocks, double* out_val, uint32_t* out_cnt,
                   bool i64) {
  int rc;
  const CvShard::Batch& bt = sh.batches[b];
  const uint32_t ng = bt.g1 - bt.g0, R = sh.n_ranks;
  // tables: uoff relative to the batch [ng + 1], the prefix over ranks of each group's heights [ng x (R + 1)], and
  // each rank's entry offset of each group within its block [ng x R]
  std::vector<uint32_t> tab((size_t)(ng + 1) + (size_t)ng * (R + 1) + (size_t)ng * R, 0u);
  uint32_t* uo = tab.data();
  uint32_t* pre = uo + ng + 1;
  uint32_t* hoffs = pre + (size_t)ng * (R + 1);
  std::vector<uint32_t> run(R, 0u);
  for (uint32_t q = 0; q < ng; ++q) {
    const uint32_t g = bt.g0 + q;
    uo[q + 1] = sh.uoff[g + 1] - sh.uoff[bt.g0];
    for (uint32_t r = 0; r < R; ++r) {
      pre[(size_t)q * (R + 1) + r + 1] = pre[(size_t)q * (R + 1) + r] + sh.height(r, g);
      hoffs[(size_t)q * R + r] = run[r];
      run[r] += sh.height(r, g);
    }
  }
  const uint32_t cells = (uint32_t)(bt.rows * bt.W), n_seg = ng * bt.W;
  size_t sort_bytes = 0, scan_bytes = 0;
  {
    cub::DoubleBuffer<unsigned long long> dk(nullptr, nullptr);
    cub::DoubleBuffer<uint32_t> dv(nullptr, nullptr);
    CU(cub::DeviceSegmentedSort::SortPairs(nullptr, sort_bytes, dk, dv, (int)cells, (int)n_seg, (const uint32_t*)nullptr,
                                           (const uint32_t*)nullptr, c->stream));
    CU(cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, (uint32_t*)nullptr, (uint32_t*)nullptr, (int)cells, c->stream));
  }
  if ((rc = c->x_table.ensure(tab.size() * 4)) || (rc = c->v_keys.ensure((size_t)cells * 8)) ||
      (rc = c->v_alt.ensure((size_t)cells * 8)) || (rc = c->vx_cnt.ensure((size_t)cells * 4)) ||
      (rc = c->vx_alt.ensure((size_t)cells * 4)) || (rc = c->v_rank.ensure((size_t)cells * 4)) ||
      (rc = c->v_seg.ensure(((size_t)n_seg + 1) * 4)) || (rc = c->v_tmp.ensure(std::max<size_t>({16, sort_bytes, scan_bytes}))))
    return rc;
  CU(cudaMemcpyAsync(c->x_table.p, tab.data(), tab.size() * 4, cudaMemcpyHostToDevice, c->stream));
  CvShardArgs a{};
  a.T = sh.T; a.k0 = bt.k0; a.W = bt.W; a.g0 = bt.g0; a.ng = ng;
  a.off = c->x_table.as<uint32_t>();
  a.hpre = a.off + ng + 1;
  a.hoffs = a.hpre + (size_t)ng * (R + 1);
  a.n_ranks = R; a.P = bt.P;
  a.gkeys = static_cast<const unsigned long long*>(blocks);
  a.gcnt = reinterpret_cast<const uint32_t*>(a.gkeys + (uint64_t)R * bt.P);
  a.cells = cells;
  a.seg_off = c->v_seg.as<uint32_t>();
  a.keys = c->v_keys.as<unsigned long long>();
  a.kcnt = c->vx_cnt.as<uint32_t>();
  a.rank = c->v_rank.as<uint32_t>();
  a.out_val = out_val; a.out_cnt = out_cnt; a.out_row0 = sh.uoff[bt.g0];
  const unsigned cell_grid = capped_grid(c, cells, 256, 8);
  count_values_merge_segments_kernel<<<capped_grid(c, n_seg, 256, 8), 256, 0, c->stream>>>(a);
  count_values_merge_arrange_kernel<<<cell_grid, 256, 0, c->stream>>>(a);
  c->launches += 2;
  CU(cudaGetLastError());
  cub::DoubleBuffer<unsigned long long> dk(c->v_keys.as<unsigned long long>(), c->v_alt.as<unsigned long long>());
  cub::DoubleBuffer<uint32_t> dv(c->vx_cnt.as<uint32_t>(), c->vx_alt.as<uint32_t>());
  size_t bytes = c->v_tmp.cap;
  CU(cub::DeviceSegmentedSort::SortPairs(c->v_tmp.p, bytes, dk, dv, (int)cells, (int)n_seg, a.seg_off, a.seg_off + 1,
                                         c->stream));
  a.sorted = dk.Current();
  a.scnt = dv.Current();
  a.csum = dv.Alternate();
  a.start = reinterpret_cast<uint32_t*>(dk.Alternate());
  count_values_merge_head_kernel<<<cell_grid, 256, 0, c->stream>>>(a);
  c->launches++;
  CU(cudaGetLastError());
  bytes = c->v_tmp.cap;
  CU(cub::DeviceScan::InclusiveSum(c->v_tmp.p, bytes, a.rank, a.rank, (int)cells, c->stream));
  bytes = c->v_tmp.cap;
  CU(cub::DeviceScan::InclusiveSum(c->v_tmp.p, bytes, a.scnt, a.csum, (int)cells, c->stream));
  count_values_merge_rank_kernel<<<cell_grid, 256, 0, c->stream>>>(a);
  (i64 ? count_values_merge_count_kernel<I64Key> : count_values_merge_count_kernel<F64Key>)
      <<<cell_grid, 256, 0, c->stream>>>(a);
  c->launches += 2;
  CU(cudaGetLastError());
  return B2P_OK;
}

// The composed call: per batch this rank's block, two all-gathers (keys, counts) in one group and the merge.  Without
// a communicator (one rank) the block is its own gather.
int cv_allgather_run(b2p_ctx* c, const CvShard& sh, const double* vals, const uint32_t* cnt, const b2p_group_index* ix,
                     double* out_val, uint32_t* out_cnt, bool i64) {
  int rc;
  if (sh.batches.empty()) return B2P_OK;
  const uint64_t block = sh.max_block();
  if ((rc = c->x_send.ensure(block))) return rc;
  if (c->comm && (rc = c->x_recv.ensure(block * sh.n_ranks))) return rc;
  for (uint32_t b = 0; b < (uint32_t)sh.batches.size(); ++b) {
    if ((rc = cv_shard_pack(c, sh, b, (uint32_t)c->comm_rank, vals, cnt, ix, c->x_send.p, i64))) return rc;
    const void* gathered = c->x_send.p;
    if (c->comm) {
      const uint64_t P = sh.batches[b].P;
      const unsigned long long* sk = c->x_send.as<unsigned long long>();
      unsigned long long* gk = c->x_recv.as<unsigned long long>();
      NCCL_TRY(g_nccl.GroupStart());
      NCCL_TRY(g_nccl.AllGather(sk, gk, P, Nccl::kUint64, c->comm, c->stream));
      NCCL_TRY(g_nccl.AllGather(sk + P, gk + P * sh.n_ranks, P, Nccl::kUint32, c->comm, c->stream));
      NCCL_TRY(g_nccl.GroupEnd());
      gathered = c->x_recv.p;
    }
    if ((rc = cv_shard_merge(c, sh, b, gathered, out_val, out_cnt, i64))) return rc;
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

// The device forms of the sharded count_values; i64: the grid is Int64
int cv_allgather_dev(b2p_ctx* c, const double* vals, const uint32_t* cnt, const b2p_group_index* ix, uint64_t T,
                     const uint32_t* heights, double* out_val, uint32_t* out_cnt, bool i64) {
  if (!c || !ix) return fail(B2P_E_INVALID, "NULL argument");
  if (ix->n_series && T && (!vals || !cnt)) return fail(B2P_E_INVALID, "NULL argument");
  if (!c->comm && c->comm_ranks != 1) return fail(B2P_E_INVALID, "no communicator: call b2p_comm_init first");
  c->last_exchange_bytes = 0;
  CvShard sh;
  if (int rc = cv_shard_plan(c, heights, c->comm_ranks, ix->n_groups, T, sh)) return rc;
  if (int rc = cv_shard_check_rank(sh, ix, (uint32_t)c->comm_rank)) return rc;
  if (!sh.batches.empty() && (!out_val || !out_cnt)) return fail(B2P_E_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  stage_begin(c, 3);
  const int rc = cv_allgather_run(c, sh, vals, cnt, ix, out_val, out_cnt, i64);
  stage_end(c, 3);
  return rc;
}

int cv_shard_pack_dev(b2p_ctx* c, const double* vals, const uint32_t* cnt, const b2p_group_index* ix, uint64_t T,
                      const uint32_t* heights, int32_t n_ranks, int32_t rank, uint32_t batch, void* block, bool i64) {
  if (!c || !ix || !block) return fail(B2P_E_INVALID, "NULL argument");
  if (ix->n_series && (!vals || !cnt)) return fail(B2P_E_INVALID, "NULL argument");
  if (rank < 0) return fail(B2P_E_INVALID, "rank %d < 0", rank);
  CvShard sh;
  if (int rc = cv_shard_plan(c, heights, n_ranks, ix->n_groups, T, sh)) return rc;
  if (int rc = cv_shard_check_rank(sh, ix, (uint32_t)rank)) return rc;
  if (batch >= sh.batches.size()) return fail(B2P_E_INVALID, "batch %u of %zu", batch, sh.batches.size());
  DeviceGuard g(c->device);
  c->last_exchange_bytes = 0;
  return cv_shard_pack(c, sh, batch, (uint32_t)rank, vals, cnt, ix, block, i64);
}

int cv_shard_merge_dev(b2p_ctx* c, const uint32_t* heights, int32_t n_ranks, uint32_t n_groups, uint64_t T,
                       uint32_t batch, const void* blocks, double* out_val, uint32_t* out_cnt, bool i64) {
  if (!c || !blocks || !out_val || !out_cnt) return fail(B2P_E_INVALID, "NULL argument");
  CvShard sh;
  if (int rc = cv_shard_plan(c, heights, n_ranks, n_groups, T, sh)) return rc;
  if (batch >= sh.batches.size()) return fail(B2P_E_INVALID, "batch %u of %zu", batch, sh.batches.size());
  DeviceGuard g(c->device);
  return cv_shard_merge(c, sh, batch, blocks, out_val, out_cnt, i64);
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

/* ---- topk / bottomk over sharded rows ------------------------------------------------------------------------- */

int b2p_topk_shard_plan(b2p_ctx* c, double k, const uint32_t* group_sizes, uint32_t n_groups, uint64_t T,
                        int32_t n_ranks, uint32_t* n_batches, uint32_t* n_rounds, uint32_t* slots,
                        uint64_t* block_bytes, uint64_t* state_bytes) {
  TopkShard sh;
  if (int rc = shard_check(c, k, group_sizes, n_groups, T, n_ranks, 0, 0, false, sh)) return rc;
  if (!n_batches || !n_rounds || !slots || !block_bytes || !state_bytes) return fail(B2P_E_INVALID, "NULL argument");
  *n_batches = sh.n_batches; *n_rounds = sh.rounds; *slots = sh.K;
  *block_bytes = sh.mode == 2 ? sh.block_bytes(sh.batch(0)) : 0;
  *state_bytes = sh.mode == 2 ? sh.state_bytes(sh.batch(0)) : 0;
  return B2P_OK;
}

int b2p_topk_shard_candidates_dev(b2p_ctx* c, int32_t bottom, double k, const double* vals, const uint32_t* valid,
                                  const b2p_group_index* ix, const uint32_t* tie, uint64_t T,
                                  const uint32_t* group_sizes, int32_t n_ranks, uint32_t batch, uint32_t round,
                                  void* state, void* block) {
  if (!ix) return fail(B2P_E_INVALID, "NULL argument");
  TopkShard sh;
  if (int rc = shard_check(c, k, group_sizes, ix->n_groups, T, n_ranks, batch, round, true, sh)) return rc;
  if ((ix->n_series && (!vals || !valid || !tie)) || !state || !block) return fail(B2P_E_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  c->last_exchange_bytes = 0;
  return shard_candidates(c, sh, batch, round, bottom, vals, valid, ix, tie, T, state, block);
}

int b2p_topk_shard_merge_dev(b2p_ctx* c, double k, const uint32_t* group_sizes, uint32_t n_groups, uint64_t T,
                             int32_t n_ranks, uint32_t batch, uint32_t round, const void* blocks, void* state) {
  TopkShard sh;
  if (int rc = shard_check(c, k, group_sizes, n_groups, T, n_ranks, batch, round, true, sh)) return rc;
  if (!blocks || !state) return fail(B2P_E_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  return shard_merge(c, sh, batch, round, blocks, state, T);
}

int b2p_topk_shard_mark_dev(b2p_ctx* c, int32_t bottom, double k, const double* vals, const uint32_t* valid,
                            const b2p_group_index* ix, const uint32_t* tie, uint64_t T, const uint32_t* group_sizes,
                            int32_t n_ranks, uint32_t batch, const void* state, uint32_t* out_valid) {
  if (!ix) return fail(B2P_E_INVALID, "NULL argument");
  TopkShard sh;
  if (int rc = shard_check(c, k, group_sizes, ix->n_groups, T, n_ranks, batch, 0, false, sh)) return rc;
  if (ix->n_series && (!vals || !valid || !tie || !out_valid)) return fail(B2P_E_INVALID, "NULL argument");
  if (sh.mode == 2 && !state) return fail(B2P_E_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  return shard_mark(c, sh, batch, bottom, vals, valid, ix, tie, T, state, out_valid);
}

int b2p_topk_allgather_dev(b2p_ctx* c, int32_t bottom, double k, const double* vals, const uint32_t* valid,
                           const b2p_group_index* ix, const uint32_t* tie, uint64_t T, uint32_t* out_valid) {
  if (!c || !ix) return fail(B2P_E_INVALID, "NULL argument");
  if (ix->n_series && (!vals || !valid || !tie || !out_valid)) return fail(B2P_E_INVALID, "NULL argument");
  if (!c->comm && c->comm_ranks != 1) return fail(B2P_E_INVALID, "no communicator: call b2p_comm_init first");
  c->last_exchange_bytes = 0;
  if (T == 0) return B2P_OK;  // (every rank has the same T)
  DeviceGuard g(c->device);
  stage_begin(c, 3);
  const int rc = topk_allgather_run(c, bottom, k, vals, valid, ix, tie, T, out_valid);
  stage_end(c, 3);
  return rc;
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

/* ---- quantile over sharded rows ------------------------------------------------------------------------------ */

int b2p_quantile_shard_plan(b2p_ctx* c, uint32_t n_groups, uint64_t T, uint32_t* n_batches, uint64_t* block_bytes,
                            uint64_t* state_bytes) {
  if (!c || !n_batches || !block_bytes || !state_bytes) return fail(B2P_E_INVALID, "NULL argument");
  const QuantShard sh = quantile_shard_plan(c, n_groups, T);
  *n_batches = sh.n_batches;
  *block_bytes = sh.n_batches ? sh.batch(0).units() * QuantShard::kUnitBlock : 0;
  *state_bytes = sh.n_batches ? sh.batch(0).units() * QuantShard::kUnitState : 0;
  return B2P_OK;
}

int b2p_quantile_shard_pass_dev(b2p_ctx* c, double phi, const double* vals, const uint32_t* valid,
                                const b2p_group_index* ix, uint64_t T, uint32_t batch, uint32_t pass, void* block) {
  if (!c || !ix || !block) return fail(B2P_E_INVALID, "NULL argument");
  if (ix->n_series && (!vals || !valid)) return fail(B2P_E_INVALID, "NULL argument");
  const QuantShard sh = quantile_shard_plan(c, ix->n_groups, T);
  if (batch >= sh.n_batches) return fail(B2P_E_INVALID, "batch %u of %u", batch, sh.n_batches);
  if (pass >= kQuantShardPasses) return fail(B2P_E_INVALID, "pass %u of at most %u", pass, kQuantShardPasses);
  DeviceGuard g(c->device);
  c->last_exchange_bytes = 0;
  return quantile_shard_pass(c, sh, batch, pass, phi, vals, valid, ix, T, block);
}

int b2p_quantile_shard_advance_dev(b2p_ctx* c, double phi, uint32_t n_groups, uint64_t T, uint32_t batch, uint32_t pass,
                                   const void* blocks, uint32_t n_blocks, double* out_val, uint32_t* out_cnt,
                                   uint64_t* live) {
  if (!c || !blocks || !out_val || !out_cnt || !live) return fail(B2P_E_INVALID, "NULL argument");
  if (n_blocks == 0) return fail(B2P_E_INVALID, "n_blocks is 0");
  const QuantShard sh = quantile_shard_plan(c, n_groups, T);
  if (batch >= sh.n_batches) return fail(B2P_E_INVALID, "batch %u of %u", batch, sh.n_batches);
  if (pass >= kQuantShardPasses) return fail(B2P_E_INVALID, "pass %u of at most %u", pass, kQuantShardPasses);
  DeviceGuard g(c->device);
  return quantile_shard_advance(c, sh, batch, phi, T, blocks, n_blocks, out_val, out_cnt, live);
}

int b2p_quantile_allreduce_dev(b2p_ctx* c, double phi, const double* vals, const uint32_t* valid,
                               const b2p_group_index* ix, uint64_t T, double* out_val, uint32_t* out_cnt) {
  if (!c || !ix) return fail(B2P_E_INVALID, "NULL argument");
  if ((ix->n_series && (!vals || !valid)) || (ix->n_groups && T && (!out_val || !out_cnt)))
    return fail(B2P_E_INVALID, "NULL argument");
  if (!c->comm && c->comm_ranks != 1) return fail(B2P_E_INVALID, "no communicator: call b2p_comm_init first");
  c->last_exchange_bytes = 0;
  if (ix->n_groups == 0 || T == 0) return B2P_OK;  // (every rank has the same n_groups and T)
  DeviceGuard g(c->device);
  stage_begin(c, 3);
  const int rc = quantile_allreduce_run(c, phi, vals, valid, ix, T, out_val, out_cnt);
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

/* ---- count_values over sharded rows -------------------------------------------------------------------------- */

int b2p_count_values_shard_heights_dev(b2p_ctx* c, const uint32_t* local_cnt, const b2p_group_index* ix, uint64_t T,
                                       uint32_t* heights) {
  if (!c || !ix) return fail(B2P_E_INVALID, "NULL argument");
  if ((ix->n_series && T && !local_cnt) || (ix->n_groups && !heights)) return fail(B2P_E_INVALID, "NULL argument");
  if (!c->comm && c->comm_ranks != 1) return fail(B2P_E_INVALID, "no communicator: call b2p_comm_init first");
  DeviceGuard g(c->device);
  return cv_shard_heights(c, local_cnt, ix, T, heights);
}

int b2p_count_values_allgather_dev(b2p_ctx* c, const double* local_val, const uint32_t* local_cnt,
                                   const b2p_group_index* ix, uint64_t T, const uint32_t* heights, double* out_val,
                                   uint32_t* out_cnt) {
  return cv_allgather_dev(c, local_val, local_cnt, ix, T, heights, out_val, out_cnt, false);
}

int b2p_count_values_allgather_i64_dev(b2p_ctx* c, const int64_t* local_val, const uint32_t* local_cnt,
                                       const b2p_group_index* ix, uint64_t T, const uint32_t* heights, int64_t* out_val,
                                       uint32_t* out_cnt) {
  return cv_allgather_dev(c, reinterpret_cast<const double*>(local_val), local_cnt, ix, T, heights,
                          reinterpret_cast<double*>(out_val), out_cnt, true);
}

int b2p_count_values_shard_plan(b2p_ctx* c, const uint32_t* heights, int32_t n_ranks, uint32_t n_groups, uint64_t T,
                                uint32_t* n_batches, uint64_t* block_bytes) {
  if (!c || !n_batches || !block_bytes) return fail(B2P_E_INVALID, "NULL argument");
  CvShard sh;
  if (int rc = cv_shard_plan(c, heights, n_ranks, n_groups, T, sh)) return rc;
  *n_batches = (uint32_t)sh.batches.size();
  *block_bytes = sh.max_block();
  return B2P_OK;
}

int b2p_count_values_shard_pack_dev(b2p_ctx* c, const double* local_val, const uint32_t* local_cnt,
                                    const b2p_group_index* ix, uint64_t T, const uint32_t* heights, int32_t n_ranks,
                                    int32_t rank, uint32_t batch, void* block) {
  return cv_shard_pack_dev(c, local_val, local_cnt, ix, T, heights, n_ranks, rank, batch, block, false);
}

int b2p_count_values_shard_pack_i64_dev(b2p_ctx* c, const int64_t* local_val, const uint32_t* local_cnt,
                                        const b2p_group_index* ix, uint64_t T, const uint32_t* heights, int32_t n_ranks,
                                        int32_t rank, uint32_t batch, void* block) {
  return cv_shard_pack_dev(c, reinterpret_cast<const double*>(local_val), local_cnt, ix, T, heights, n_ranks, rank,
                           batch, block, true);
}

int b2p_count_values_shard_merge_dev(b2p_ctx* c, const uint32_t* heights, int32_t n_ranks, uint32_t n_groups,
                                     uint64_t T, uint32_t batch, const void* blocks, double* out_val, uint32_t* out_cnt) {
  return cv_shard_merge_dev(c, heights, n_ranks, n_groups, T, batch, blocks, out_val, out_cnt, false);
}

int b2p_count_values_shard_merge_i64_dev(b2p_ctx* c, const uint32_t* heights, int32_t n_ranks, uint32_t n_groups,
                                         uint64_t T, uint32_t batch, const void* blocks, int64_t* out_val,
                                         uint32_t* out_cnt) {
  return cv_shard_merge_dev(c, heights, n_ranks, n_groups, T, batch, blocks, reinterpret_cast<double*>(out_val),
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
