// b2p_sort.cu — sort / sort_desc of the C ABI (K14, b2p_sort.cuh): the valid cells of a [rows x T] grid as cell
// indices in value order, over one field or lexicographically over several.
#include <algorithm>

#include <cub/device/device_radix_sort.cuh>
#include <vector>

#include "b2p_runtime.cuh"
#include "b2p_sort.cuh"

using namespace b2p;

namespace {
// K13's count and scan (scan_valid_cells), a read-back of the total (the radix sort takes its item count on the host:
// the one synchronisation of the call), K14's scatter into (keys, out_cells) keyed on the last field, then CUB's stable
// radix sort of the pairs over all 64 key bits; for every earlier field, last but one first, sort_rekey_kernel and one
// more stable radix sort.  The keys and the cell indices ping-pong between their two buffers (the cells between out_cells
// and the context's so_cells); if the cells end in the latter they are copied back.  Scratch (context buffers so_*):
// 8 B per row plus one (offsets), 24 B per valid cell (two key buffers, one cell buffer) and CUB's temp storage.
// *n_host is the number of valid cells.  i64: the cells are Int64 (I64Key).
// A shard pack (`shard`) reads its row-id flag back with the count, and refuses the call before the scatter when the
// flag is set or the count is not the one the caller sized the block for.
struct ShardCheck {
  const uint32_t* bad;  // device flag of sort_shard_rows_kernel
  uint64_t expect;      // the rank's count in the caller's table
};

int sort_run(b2p_ctx* c, int desc, const double* const* vals, int32_t n_fields, const uint32_t* valid, uint32_t rows,
             uint64_t T, uint64_t* out_cells, uint64_t* out_n, uint64_t* n_host, bool i64,
             const ShardCheck* shard = nullptr) {
  int rc;
  if ((rc = c->so_off.ensure(((size_t)rows + 1) * 8))) return rc;
  unsigned long long* off = c->so_off.as<unsigned long long>();
  if ((rc = scan_valid_cells(c, valid, T, rows, off, c->so_tmp))) return rc;
  CU(cudaMemcpyAsync(out_n, off + rows, 8, cudaMemcpyDeviceToDevice, c->stream));
  uint64_t n = 0;
  uint32_t bad = 0;
  CU(cudaMemcpyAsync(&n, off + rows, 8, cudaMemcpyDeviceToHost, c->stream));
  if (shard) CU(cudaMemcpyAsync(&bad, shard->bad, 4, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  *n_host = n;
  if (shard && bad) return fail(B2P_E_INVALID, "sort: row_id is not strictly increasing along the rank's rows");
  if (shard && n != shard->expect)
    return fail(B2P_E_INVALID, "sort: this rank has %llu valid cells, its entry in counts says %llu",
                (unsigned long long)n, (unsigned long long)shard->expect);
  if (n == 0) return B2P_OK;
  if ((rc = c->so_keys.ensure(n * 16)) || (rc = c->so_cells.ensure(n * 8))) return rc;
  SortArgs a{};
  a.vals = vals[n_fields - 1]; a.valid = valid; a.T = T; a.Tw = (uint32_t)((T + 31) / 32); a.rows = rows;
  a.desc = desc ? 1 : 0;
  a.offsets = off;
  a.keys = c->so_keys.as<unsigned long long>();
  a.cells = reinterpret_cast<unsigned long long*>(out_cells);
  (i64 ? sort_scatter_kernel<I64Key> : sort_scatter_kernel<F64Key>)<<<cell_rows_grid(c, rows), 256, 0, c->stream>>>(a);
  c->launches++;
  CU(cudaGetLastError());
  cub::DoubleBuffer<unsigned long long> keys(a.keys, a.keys + n);
  cub::DoubleBuffer<unsigned long long> cells(a.cells, c->so_cells.as<unsigned long long>());
  size_t bytes = 0;
  CU(cub::DeviceRadixSort::SortPairs(nullptr, bytes, keys, cells, n, 0, 64, c->stream));
  if ((rc = c->so_tmp.ensure(std::max<size_t>(bytes, 16)))) return rc;
  bytes = c->so_tmp.cap;
  CU(cub::DeviceRadixSort::SortPairs(c->so_tmp.p, bytes, keys, cells, n, 0, 64, c->stream));
  for (int32_t f = n_fields - 2; f >= 0; --f) {
    (i64 ? sort_rekey_kernel<I64Key> : sort_rekey_kernel<F64Key>)<<<capped_grid(c, n, 256, 8), 256, 0, c->stream>>>(
        vals[f], cells.Current(), keys.Current(), n, a.desc);
    c->launches++;
    CU(cudaGetLastError());
    bytes = c->so_tmp.cap;
    CU(cub::DeviceRadixSort::SortPairs(c->so_tmp.p, bytes, keys, cells, n, 0, 64, c->stream));
  }
  if (cells.Current() != a.cells)
    CU(cudaMemcpyAsync(a.cells, cells.Current(), n * 8, cudaMemcpyDeviceToDevice, c->stream));
  return B2P_OK;
}

int check_sort_shape(uint32_t n_rows, uint64_t T) {
  if (n_rows >= (uint32_t)INT32_MAX) return fail(B2P_E_TOO_LARGE, "sort: %u rows, at most %d", n_rows, INT32_MAX - 1);
  if (T > 0 && n_rows > UINT64_MAX / 8 / T) return fail(B2P_E_TOO_LARGE, "sort: %u rows x %llu steps", n_rows,
                                                        (unsigned long long)T);
  return B2P_OK;
}

int check_sort_fields(const double* const* vals, int32_t n_fields) {
  if (n_fields < 1 || n_fields > B2P_MAX_FIELDS)
    return fail(B2P_E_INVALID, "n_fields must be in [1, %d] (got %d)", B2P_MAX_FIELDS, (int)n_fields);
  if (!vals) return fail(B2P_E_INVALID, "NULL argument");
  return B2P_OK;
}

// the device and host forms of every sort entry point; i64: the grid is Int64 (one field)
int sort_cells_dev(b2p_ctx* c, int32_t desc, const double* const* vals, int32_t n_fields, const uint32_t* valid,
                   uint32_t n_rows, uint64_t T, uint64_t* out_cells, uint64_t* out_n, bool i64) {
  if (!c || !out_n) return fail(B2P_E_INVALID, "NULL argument");
  if (int rc = check_sort_fields(vals, n_fields)) return rc;
  if (int rc = check_sort_shape(n_rows, T)) return rc;
  DeviceGuard g(c->device);
  if (n_rows == 0 || T == 0) {
    CU(cudaMemsetAsync(out_n, 0, 8, c->stream));
    return B2P_OK;
  }
  if (!valid || !out_cells) return fail(B2P_E_INVALID, "NULL argument");
  for (int32_t f = 0; f < n_fields; ++f)
    if (!vals[f]) return fail(B2P_E_INVALID, "NULL argument (field %d)", (int)f);
  uint64_t n = 0;
  stage_begin(c, 3);
  const int rc = sort_run(c, desc, vals, n_fields, valid, n_rows, T, out_cells, out_n, &n, i64);
  stage_end(c, 3);
  return rc;
}

int sort_cells_host(b2p_ctx* c, int32_t desc, const double* const* vals, int32_t n_fields, const uint32_t* valid,
                    uint32_t n_rows, uint64_t T, uint64_t* out_cells, uint64_t* out_n, bool i64) {
  if (!c) return fail(B2P_E_INVALID, "NULL argument");
  if (int rc = check_sort_fields(vals, n_fields)) return rc;
  if (int rc = check_sort_shape(n_rows, T)) return rc;  // (before the cell column is sized)
  DeviceGuard g(c->device);
  const uint64_t cells = (uint64_t)n_rows * T, Tw = (T + 31) / 32;
  Staging s{c};
  const double* d_vals[B2P_MAX_FIELDS];
  s.in_cols(vals, n_fields, cells * 8, d_vals);
  const uint32_t* d_valid = s.in(valid, (size_t)n_rows * Tw * 4);
  uint64_t* d_cells = out_cells ? static_cast<uint64_t*>(s.buf(cells * 8)) : nullptr;
  uint64_t* d_n = s.out(out_n, 8);
  if (int rc = s.end([&] { return sort_cells_dev(c, desc, d_vals, n_fields, d_valid, n_rows, T, d_cells, d_n, i64); }))
    return rc;
  s.copy_back(out_cells, d_cells, *out_n * 8);  // only the valid cells' entries, now that their count is here
  return s.finish();
}

// ---- sort over rows sharded across ranks --------------------------------------------------------------------------

int check_shard_steps(uint64_t T) {
  if (T > (1ull << 32)) return fail(B2P_E_TOO_LARGE, "sort: %llu steps, at most 2^32 (global cells are row_id * T + k)",
                                    (unsigned long long)T);
  return B2P_OK;
}

int check_shard_grid(const double* const* vals, int32_t n_fields, const uint32_t* valid, const uint32_t* row_id,
                     uint32_t n_rows, uint64_t T) {
  if (int rc = check_sort_fields(vals, n_fields)) return rc;
  if (int rc = check_sort_shape(n_rows, T)) return rc;
  if (int rc = check_shard_steps(T)) return rc;
  if (n_rows == 0 || T == 0) return B2P_OK;
  if (!valid || !row_id) return fail(B2P_E_INVALID, "NULL argument");
  for (int32_t f = 0; f < n_fields; ++f)
    if (!vals[f]) return fail(B2P_E_INVALID, "NULL argument (field %d)", (int)f);
  return B2P_OK;
}

// This rank's valid cells (K13's count) into counts[0], or with a communicator every rank's into counts[n_ranks] (one
// in-place all-gather of 8 B per rank).  Reads the table back, so it synchronises the stream.
int shard_counts(b2p_ctx* c, const uint32_t* valid, uint32_t n_rows, uint64_t T, uint64_t* counts) {
  return rank_table(c, 1, Nccl::kUint64, counts, [&](void* mine) {
    if (n_rows && T) {
      if (int rc = c->so_off.ensure(((size_t)n_rows + 1) * 8)) return rc;
      unsigned long long* off = c->so_off.as<unsigned long long>();
      if (int rc = scan_valid_cells(c, valid, T, n_rows, off, c->so_tmp)) return rc;
      CU(cudaMemcpyAsync(mine, off + n_rows, 8, cudaMemcpyDeviceToDevice, c->stream));
    } else {
      CU(cudaMemsetAsync(mine, 0, 8, c->stream));
    }
    return B2P_OK;
  });
}

// Per-rank step: K14 over the rank's rows with its cells written into the block's last section, then the pack in
// place.  `count` is the rank's entry of the counts table, which sized the block; the row-id check and the count are
// read back together (K14's one synchronisation).  The block is [F x count keys][count global cells].
int shard_pack(b2p_ctx* c, int desc, const double* const* vals, int32_t F, const uint32_t* valid,
               const uint32_t* row_id, uint32_t n_rows, uint64_t T, uint64_t count, unsigned long long* block,
               bool i64) {
  int rc;
  if (n_rows == 0 || T == 0) {
    if (count) return fail(B2P_E_INVALID, "sort: this rank has no valid cell, its entry in counts says %llu",
                           (unsigned long long)count);
    return B2P_OK;
  }
  if ((rc = c->sx_flag.ensure(16))) return rc;
  uint32_t* bad = c->sx_flag.as<uint32_t>();
  uint64_t* n_dev = c->sx_flag.as<uint64_t>() + 1;
  CU(cudaMemsetAsync(bad, 0, 4, c->stream));
  if (n_rows > 1) {
    sort_shard_rows_kernel<<<capped_grid(c, n_rows, 256, 8), 256, 0, c->stream>>>(row_id, n_rows, bad);
    c->launches++;
    CU(cudaGetLastError());
  }
  const ShardCheck chk{bad, count};
  uint64_t n = 0;
  if ((rc = sort_run(c, desc, vals, F, valid, n_rows, T, reinterpret_cast<uint64_t*>(block + (uint64_t)F * count), n_dev,
                     &n, i64, &chk)))
    return rc;
  if (n == 0) return B2P_OK;
  SortPackArgs a{};
  for (int32_t f = 0; f < F; ++f) a.vals[f] = vals[f];
  a.F = F; a.row_id = row_id; a.T = T; a.n = n; a.flip = desc ? ~0ull : 0ull; a.block = block;
  (i64 ? sort_shard_pack_kernel<I64Key> : sort_shard_pack_kernel<F64Key>)<<<capped_grid(c, n, 256, 8), 256, 0,
                                                                            c->stream>>>(a);
  c->launches++;
  CU(cudaGetLastError());
  return B2P_OK;
}

// Merge step over the n_ranks blocks laid back to back (block r: counts[r] entries): ceil(log2 runs) rounds of pairwise
// merge-path merges over the non-empty runs (one round, a copy, for one run), ping-ponging between the context's two
// run buffers (N x 8 (F + 1) B each, the second only from three rounds on); the last round writes out_cells and the
// values decoded from the keys.  Every round's pair table goes to the device in one copy; no host round trip.
int shard_merge(b2p_ctx* c, int desc, int32_t F, const uint64_t* counts, uint32_t R, const unsigned long long* blocks,
                unsigned long long* out_cells, double* const* out_vals, bool i64) {
  int rc;
  std::vector<SortRun> runs;
  uint64_t N = 0, off = 0;
  for (uint32_t r = 0; r < R; ++r) {
    if (counts[r]) runs.push_back(SortRun{blocks + off, counts[r], counts[r]});
    off += counts[r] * (uint64_t)(F + 1);
    N += counts[r];
  }
  if (runs.empty()) return B2P_OK;
  int rounds = 1;
  while (((size_t)1 << rounds) < runs.size()) ++rounds;
  const uint32_t items = F == 1 ? 8u : (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(8, 98304 / (256 * (8 * (uint64_t)F + 12))));
  const uint32_t cap = 256 * items;
  const size_t smem = (size_t)(F + 1) * cap * 8 + (size_t)cap * 4;
  const size_t run_bytes = N * 8 * (uint64_t)(F + 1);
  if (rounds >= 2 && (rc = c->sx_run[0].ensure(run_bytes))) return rc;
  if (rounds >= 3 && (rc = c->sx_run[1].ensure(run_bytes))) return rc;
  std::vector<SortPair> pairs;
  std::vector<size_t> first(rounds + 1, 0);
  std::vector<uint64_t> tiles(rounds, 0);
  for (int k = 0; k < rounds; ++k) {
    const bool last = k == rounds - 1;
    const unsigned long long* dest = last ? nullptr : c->sx_run[k % 2].as<unsigned long long>();
    std::vector<SortRun> next;
    uint64_t out = 0;
    for (size_t j = 0; j < runs.size(); j += 2) {
      const SortRun a = runs[j], b = j + 1 < runs.size() ? runs[j + 1] : SortRun{a.base, a.stride, 0};
      const uint64_t len = a.len + b.len;
      pairs.push_back(SortPair{a, b, out, tiles[k]});
      tiles[k] += (len + cap - 1) / cap;
      if (!last) next.push_back(SortRun{dest + out, N, len});
      out += len;
    }
    if (tiles[k] > (uint64_t)INT32_MAX) return fail(B2P_E_TOO_LARGE, "sort: %llu merged entries", (unsigned long long)N);
    first[k + 1] = pairs.size();
    runs.swap(next);
  }
  if ((rc = c->x_table.ensure(pairs.size() * sizeof(SortPair)))) return rc;
  CU(cudaMemcpyAsync(c->x_table.p, pairs.data(), pairs.size() * sizeof(SortPair), cudaMemcpyHostToDevice, c->stream));
  SortMergeArgs a{};
  a.F = F; a.cap = cap; a.flip = desc ? ~0ull : 0ull;
  a.ostride = N;
  a.out_cells = out_cells;
  for (int32_t f = 0; f < F; ++f) a.out_vals[f] = out_vals[f];
  for (int k = 0; k < rounds; ++k) {
    const bool last = k == rounds - 1;
    a.pairs = c->x_table.as<SortPair>() + first[k];
    a.n_pairs = (uint32_t)(first[k + 1] - first[k]);
    a.obase = last ? nullptr : c->sx_run[k % 2].as<unsigned long long>();
    void (*kern)(const SortMergeArgs);
    if (F == 1)
      kern = last ? (i64 ? sort_shard_merge_kernel<true, true, I64Key> : sort_shard_merge_kernel<true, true, F64Key>)
                  : sort_shard_merge_kernel<true, false, F64Key>;
    else
      kern = last ? (i64 ? sort_shard_merge_kernel<false, true, I64Key> : sort_shard_merge_kernel<false, true, F64Key>)
                  : sort_shard_merge_kernel<false, false, F64Key>;
    if (smem > 48 * 1024) CU(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<(unsigned)tiles[k], 256, smem, c->stream>>>(a);
    c->launches++;
    CU(cudaGetLastError());
  }
  return B2P_OK;
}

// The composed call: this rank's block packed in place into the gathered buffer (x_recv, N x 8 (F + 1) B), one
// ncclBroadcast per rank with cells, in one group, each from that rank's block, then the merge.  Without a communicator
// (one rank) the block is its own gather.
int sort_allgather(b2p_ctx* c, int desc, const double* const* vals, int32_t F, const uint32_t* valid,
                   const uint32_t* row_id, uint32_t n_rows, uint64_t T, const uint64_t* counts,
                   unsigned long long* out_cells, double* const* out_vals, bool i64) {
  if (!c || !counts || !out_vals) return fail(B2P_E_INVALID, "NULL argument");
  if (int rc = check_shard_grid(vals, F, valid, row_id, n_rows, T)) return rc;
  const uint32_t R = (uint32_t)c->comm_ranks, me = (uint32_t)c->comm_rank;
  uint64_t N = 0, mine = 0;
  for (uint32_t r = 0; r < R; ++r) {
    if (r == me) mine = N;
    N += counts[r];
  }
  if (N && !out_cells) return fail(B2P_E_INVALID, "NULL argument");
  for (int32_t f = 0; N && f < F; ++f)
    if (!out_vals[f]) return fail(B2P_E_INVALID, "NULL argument (output field %d)", (int)f);
  c->last_exchange_bytes = 0;
  DeviceGuard g(c->device);
  int rc;
  const uint64_t E = (uint64_t)(F + 1);
  if ((rc = c->x_recv.ensure(std::max<uint64_t>(N * E * 8, 16)))) return rc;
  unsigned long long* all = c->x_recv.as<unsigned long long>();
  stage_begin(c, 3);
  if ((rc = shard_pack(c, desc, vals, F, valid, row_id, n_rows, T, counts[me], all + mine * E, i64))) return rc;
  if (N && (rc = gather_blocks(c, all, counts, E * 8, Nccl::kUint64))) return rc;
  rc = shard_merge(c, desc, F, counts, R, all, out_cells, out_vals, i64);
  stage_end(c, 3);
  c->last_exchange_bytes = (long long)(counts[me] * E * 8);
  return rc;
}

int sort_shard_pack_dev(b2p_ctx* c, int desc, const double* const* vals, int32_t F, const uint32_t* valid,
                        const uint32_t* row_id, uint32_t n_rows, uint64_t T, uint64_t count, void* block, bool i64) {
  if (!c) return fail(B2P_E_INVALID, "NULL argument");
  if (int rc = check_shard_grid(vals, F, valid, row_id, n_rows, T)) return rc;
  if (count && !block) return fail(B2P_E_INVALID, "NULL argument");
  c->last_exchange_bytes = 0;
  DeviceGuard g(c->device);
  if (int rc = shard_pack(c, desc, vals, F, valid, row_id, n_rows, T, count, static_cast<unsigned long long*>(block),
                          i64))
    return rc;
  c->last_exchange_bytes = (long long)(count * 8 * (uint64_t)(F + 1));
  return B2P_OK;
}

int sort_shard_merge_dev(b2p_ctx* c, int desc, int32_t F, const uint64_t* counts, int32_t n_ranks, const void* blocks,
                         uint64_t* out_cells, double* const* out_vals, bool i64) {
  if (!c || !counts || !out_vals) return fail(B2P_E_INVALID, "NULL argument");
  if (F < 1 || F > B2P_MAX_FIELDS)
    return fail(B2P_E_INVALID, "n_fields must be in [1, %d] (got %d)", B2P_MAX_FIELDS, (int)F);
  if (n_ranks < 1) return fail(B2P_E_INVALID, "n_ranks %d < 1", (int)n_ranks);
  uint64_t N = 0;
  for (int32_t r = 0; r < n_ranks; ++r) N += counts[r];
  if (N == 0) return B2P_OK;
  if (!blocks || !out_cells) return fail(B2P_E_INVALID, "NULL argument");
  for (int32_t f = 0; f < F; ++f)
    if (!out_vals[f]) return fail(B2P_E_INVALID, "NULL argument (output field %d)", (int)f);
  DeviceGuard g(c->device);
  return shard_merge(c, desc, F, counts, (uint32_t)n_ranks, static_cast<const unsigned long long*>(blocks),
                     reinterpret_cast<unsigned long long*>(out_cells), out_vals, i64);
}
}  // namespace

extern "C" {

int b2p_sort_cells_fields_dev(b2p_ctx* c, int32_t desc, const double* const* vals, int32_t n_fields,
                              const uint32_t* valid, uint32_t n_rows, uint64_t T, uint64_t* out_cells,
                              uint64_t* out_n) {
  return sort_cells_dev(c, desc, vals, n_fields, valid, n_rows, T, out_cells, out_n, false);
}

int b2p_sort_cells_dev(b2p_ctx* c, int32_t desc, const double* vals, const uint32_t* valid, uint32_t n_rows,
                       uint64_t T, uint64_t* out_cells, uint64_t* out_n) {
  return b2p_sort_cells_fields_dev(c, desc, &vals, 1, valid, n_rows, T, out_cells, out_n);
}

int b2p_sort_cells_i64_dev(b2p_ctx* c, int32_t desc, const int64_t* vals, const uint32_t* valid, uint32_t n_rows,
                           uint64_t T, uint64_t* out_cells, uint64_t* out_n) {
  const double* v = reinterpret_cast<const double*>(vals);
  return sort_cells_dev(c, desc, &v, 1, valid, n_rows, T, out_cells, out_n, true);
}

int b2p_sort_shard_counts_dev(b2p_ctx* c, const uint32_t* valid, uint32_t n_rows, uint64_t T, uint64_t* counts) {
  if (!c || !counts) return fail(B2P_E_INVALID, "NULL argument");
  if (int rc = check_sort_shape(n_rows, T)) return rc;
  if (int rc = check_shard_steps(T)) return rc;
  if (n_rows && T && !valid) return fail(B2P_E_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  return shard_counts(c, valid, n_rows, T, counts);
}

int b2p_sort_cells_allgather_fields_dev(b2p_ctx* c, int32_t desc, const double* const* vals, int32_t n_fields,
                                        const uint32_t* valid, const uint32_t* row_id, uint32_t n_rows, uint64_t T,
                                        const uint64_t* counts, uint64_t* out_cells, double* const* out_vals) {
  return sort_allgather(c, desc, vals, n_fields, valid, row_id, n_rows, T, counts,
                        reinterpret_cast<unsigned long long*>(out_cells), out_vals, false);
}

int b2p_sort_cells_allgather_dev(b2p_ctx* c, int32_t desc, const double* vals, const uint32_t* valid,
                                 const uint32_t* row_id, uint32_t n_rows, uint64_t T, const uint64_t* counts,
                                 uint64_t* out_cells, double* out_vals) {
  return b2p_sort_cells_allgather_fields_dev(c, desc, &vals, 1, valid, row_id, n_rows, T, counts, out_cells,
                                             &out_vals);
}

int b2p_sort_cells_allgather_i64_dev(b2p_ctx* c, int32_t desc, const int64_t* vals, const uint32_t* valid,
                                     const uint32_t* row_id, uint32_t n_rows, uint64_t T, const uint64_t* counts,
                                     uint64_t* out_cells, int64_t* out_vals) {
  const double* v = reinterpret_cast<const double*>(vals);
  double* o = reinterpret_cast<double*>(out_vals);
  return sort_allgather(c, desc, &v, 1, valid, row_id, n_rows, T, counts,
                        reinterpret_cast<unsigned long long*>(out_cells), &o, true);
}

int b2p_sort_shard_pack_dev(b2p_ctx* c, int32_t desc, const double* const* vals, int32_t n_fields,
                            const uint32_t* valid, const uint32_t* row_id, uint32_t n_rows, uint64_t T, uint64_t count,
                            void* block) {
  return sort_shard_pack_dev(c, desc, vals, n_fields, valid, row_id, n_rows, T, count, block, false);
}

int b2p_sort_shard_pack_i64_dev(b2p_ctx* c, int32_t desc, const int64_t* vals, const uint32_t* valid,
                                const uint32_t* row_id, uint32_t n_rows, uint64_t T, uint64_t count, void* block) {
  const double* v = reinterpret_cast<const double*>(vals);
  return sort_shard_pack_dev(c, desc, &v, 1, valid, row_id, n_rows, T, count, block, true);
}

int b2p_sort_shard_merge_dev(b2p_ctx* c, int32_t desc, int32_t n_fields, const uint64_t* counts, int32_t n_ranks,
                             const void* blocks, uint64_t* out_cells, double* const* out_vals) {
  return sort_shard_merge_dev(c, desc, n_fields, counts, n_ranks, blocks, out_cells, out_vals, false);
}

int b2p_sort_shard_merge_i64_dev(b2p_ctx* c, int32_t desc, const uint64_t* counts, int32_t n_ranks,
                                 const void* blocks, uint64_t* out_cells, int64_t* out_vals) {
  double* o = reinterpret_cast<double*>(out_vals);
  return sort_shard_merge_dev(c, desc, 1, counts, n_ranks, blocks, out_cells, &o, true);
}

/* ---- host-pointer API ------------------------------------------------------------------------ */

int b2p_sort_cells_fields(b2p_ctx* c, int32_t desc, const double* const* vals, int32_t n_fields, const uint32_t* valid,
                          uint32_t n_rows, uint64_t T, uint64_t* out_cells, uint64_t* out_n) {
  return sort_cells_host(c, desc, vals, n_fields, valid, n_rows, T, out_cells, out_n, false);
}

int b2p_sort_cells(b2p_ctx* c, int32_t desc, const double* vals, const uint32_t* valid, uint32_t n_rows, uint64_t T,
                   uint64_t* out_cells, uint64_t* out_n) {
  return b2p_sort_cells_fields(c, desc, &vals, 1, valid, n_rows, T, out_cells, out_n);
}

int b2p_sort_cells_i64(b2p_ctx* c, int32_t desc, const int64_t* vals, const uint32_t* valid, uint32_t n_rows, uint64_t T,
                       uint64_t* out_cells, uint64_t* out_n) {
  const double* v = reinterpret_cast<const double*>(vals);
  return sort_cells_host(c, desc, &v, 1, valid, n_rows, T, out_cells, out_n, true);
}

}  // extern "C"
