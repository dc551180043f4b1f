// b2p_sort.cu — sort / sort_desc of the C ABI (K14, b2p_sort.cuh): the valid cells of a [rows x T] grid as cell
// indices in value order, over one field or lexicographically over several.
#include <algorithm>

#include <cub/device/device_radix_sort.cuh>

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
int sort_run(b2p_ctx* c, int desc, const double* const* vals, int32_t n_fields, const uint32_t* valid, uint32_t rows,
             uint64_t T, uint64_t* out_cells, uint64_t* out_n, uint64_t* n_host, bool i64) {
  int rc;
  if ((rc = c->so_off.ensure(((size_t)rows + 1) * 8))) return rc;
  unsigned long long* off = c->so_off.as<unsigned long long>();
  if ((rc = scan_valid_cells(c, valid, T, rows, off, c->so_tmp))) return rc;
  CU(cudaMemcpyAsync(out_n, off + rows, 8, cudaMemcpyDeviceToDevice, c->stream));
  uint64_t n = 0;
  CU(cudaMemcpyAsync(&n, off + rows, 8, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  *n_host = n;
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
