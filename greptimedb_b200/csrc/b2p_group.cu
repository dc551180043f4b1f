// b2p_group.cu — by-label entry points of the C ABI: the group index, by-label aggregates and their partials, the
// all-reduce of partials over NCCL, HistogramFold / histogram_quantile and the column reduce.
#include <new>
#include <vector>

#include <cub/device/device_radix_sort.cuh>

#include "b2p_runtime.cuh"
#include "b2p_aggregate.cuh"

using namespace b2p;

int build_group_csr(b2p_ctx* c, const uint32_t* gid, uint32_t n_series, uint32_t n_groups, uint32_t* goff,
                    uint32_t* members) {
  int rc;
  const size_t ns = n_series ? n_series : 1;
  if ((rc = c->g_vals_in.ensure(ns * 4))) return rc;
  if ((rc = c->g_keys_out.ensure(ns * 4))) return rc;
  iota_kernel<<<(unsigned)((ns + 255) / 256 < 1024 ? (ns + 255) / 256 : 1024), 256, 0, c->stream>>>(
      c->g_vals_in.as<uint32_t>(), n_series);
  c->launches++;
  size_t tmp_bytes = 0;
  CU(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, gid, c->g_keys_out.as<uint32_t>(), c->g_vals_in.as<uint32_t>(),
                                     members, (int)n_series, 0, 32, c->stream));
  if ((rc = c->g_tmp.ensure(tmp_bytes ? tmp_bytes : 16))) return rc;
  if (n_series > 0)
    CU(cub::DeviceRadixSort::SortPairs(c->g_tmp.p, tmp_bytes, gid, c->g_keys_out.as<uint32_t>(),
                                       c->g_vals_in.as<uint32_t>(), members, (int)n_series, 0, 32, c->stream));
  group_offsets_kernel<<<(n_groups + 1 + 255) / 256, 256, 0, c->stream>>>(c->g_keys_out.as<uint32_t>(), n_series,
                                                                          n_groups, goff);
  c->launches++;
  CU(cudaGetLastError());
  return B2P_OK;
}

// accumulate = 1 (SUM / COUNT partials only, Float64 only): out_val / out_cnt are added to instead of overwritten;
// i64: the cells hold Int64
int group_aggregate_csr(b2p_ctx* c, int32_t agg, const double* vals, const uint32_t* valid_words, const uint32_t* goff,
                        const uint32_t* members, uint32_t n_groups, uint64_t T, double* out_val, uint32_t* out_cnt,
                        int accumulate, double* out_mean, bool i64) {
  GroupArgs a{};
  a.out_mean = out_mean;
  a.agg = agg; a.vals = vals; a.valid = valid_words; a.goff = goff;
  a.members = members; a.n_groups = n_groups; a.T = T; a.Tw = (uint32_t)((T + 31) / 32);
  a.out_val = out_val; a.out_cnt = out_cnt; a.accumulate = accumulate;
  const unsigned blocks = capped_grid(c, (uint64_t)n_groups * ((T + 31) / 32), 8, 32);
  return with_id<B2P_AGG_STDVAR + 1>(agg, "aggregator", [&](auto k) {
    if (i64) group_aggregate_kernel<decltype(k)::value, true><<<blocks, 256, 0, c->stream>>>(a);
    else group_aggregate_kernel<decltype(k)::value><<<blocks, 256, 0, c->stream>>>(a);
    c->launches++;
    CU(cudaGetLastError());
    return B2P_OK;
  });
}

namespace {
int group_aggregate_impl(b2p_ctx* c, int32_t agg, const double* vals, const uint32_t* valid_words, const uint32_t* gid,
                         uint32_t n_series, uint32_t n_groups, uint64_t T, double* out_val, uint32_t* out_cnt,
                         int accumulate, double* out_mean = nullptr, bool i64 = false) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  if (agg < 0 || agg > B2P_AGG_STDVAR) return fail(B2P_E_INVALID, "unknown aggregator %d", agg);
  if (n_groups == 0 || T == 0) return B2P_OK;
  if (!vals || !valid_words || !gid || !out_val || !out_cnt) return fail(B2P_E_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  int rc;
  const size_t ns = n_series ? n_series : 1;
  if ((rc = c->g_vals_out.ensure(ns * 4))) return rc;
  if ((rc = c->g_goff.ensure(((size_t)n_groups + 1) * 4))) return rc;
  stage_begin(c, 3);
  if ((rc = build_group_csr(c, gid, n_series, n_groups, c->g_goff.as<uint32_t>(), c->g_vals_out.as<uint32_t>()))) return rc;
  rc = group_aggregate_csr(c, agg, vals, valid_words, c->g_goff.as<uint32_t>(), c->g_vals_out.as<uint32_t>(), n_groups, T,
                           out_val, out_cnt, accumulate, out_mean, i64);
  stage_end(c, 3);
  return rc;
}
}  // namespace

extern "C" {

int b2p_group_aggregate_dev(b2p_ctx* c, int32_t agg, const double* vals, const uint32_t* valid_words,
                            const uint32_t* gid, uint32_t n_series, uint32_t n_groups, uint64_t T, double* out_val,
                            uint32_t* out_cnt) {
  return group_aggregate_impl(c, agg, vals, valid_words, gid, n_series, n_groups, T, out_val, out_cnt, 0);
}

int b2p_group_aggregate_i64_dev(b2p_ctx* c, int32_t agg, const int64_t* vals, const uint32_t* valid_words,
                                const uint32_t* gid, uint32_t n_series, uint32_t n_groups, uint64_t T, double* out_val,
                                uint32_t* out_cnt) {
  return group_aggregate_impl(c, agg, reinterpret_cast<const double*>(vals), valid_words, gid, n_series, n_groups, T,
                              out_val, out_cnt, 0, nullptr, true);
}

int b2p_group_aggregate_partial_dev(b2p_ctx* c, int32_t agg, const double* vals, const uint32_t* valid_words,
                                    const uint32_t* gid, uint32_t n_series, uint32_t n_groups, uint64_t T,
                                    double* out_val, uint32_t* out_cnt, double* out_mean) {
  const bool var = agg == B2P_AGG_STDDEV || agg == B2P_AGG_STDVAR;
  if (var && !out_mean) return fail(B2P_E_INVALID, "stddev / stdvar partials need out_mean");
  if (agg == B2P_AGG_AVG) agg = B2P_AGG_SUM;  // the partial of an average is (sum, count)
  return group_aggregate_impl(c, agg, vals, valid_words, gid, n_series, n_groups, T, out_val, out_cnt, 0,
                              var ? out_mean : nullptr);
}

int b2p_group_aggregate_partial_i64_dev(b2p_ctx* c, int32_t agg, const int64_t* vals, const uint32_t* valid_words,
                                        const uint32_t* gid, uint32_t n_series, uint32_t n_groups, uint64_t T,
                                        double* out_val, uint32_t* out_cnt) {
  if (agg != B2P_AGG_SUM && agg != B2P_AGG_MIN && agg != B2P_AGG_MAX)
    return fail(B2P_E_INVALID, "Int64 partials exist for sum, min and max only (aggregator %d)", agg);
  return group_aggregate_impl(c, agg, reinterpret_cast<const double*>(vals), valid_words, gid, n_series, n_groups, T,
                              out_val, out_cnt, 0, nullptr, true);
}

int b2p_group_index_create_dev(b2p_ctx* c, const uint32_t* gid, uint32_t n_series, uint32_t n_groups,
                               b2p_group_index** out_index) {
  if (!c || !out_index || (!gid && n_series)) return fail(B2P_E_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  b2p_group_index* ix = new (std::nothrow) b2p_group_index();
  if (!ix) return fail(B2P_E_NOMEM, "out of host memory");
  ix->n_series = n_series; ix->n_groups = n_groups;
  const size_t ns = n_series ? n_series : 1;
  bool ok = cudaMalloc(&ix->gid, ns * 4) == cudaSuccess && cudaMalloc(&ix->members, ns * 4) == cudaSuccess &&
            cudaMalloc(&ix->goff, ((size_t)n_groups + 1) * 4) == cudaSuccess;
  int rc = ok ? B2P_OK : fail(B2P_E_NOMEM, "cudaMalloc failed for the group index");
  if (!rc && n_series) {
    cudaMemcpyAsync(ix->gid, gid, (size_t)n_series * 4, cudaMemcpyDeviceToDevice, c->stream);
    rc = build_group_csr(c, ix->gid, n_series, n_groups, ix->goff, ix->members);
  } else if (!rc) {  // no rows: every group is empty (a rank of a sharded topk may hold none)
    const cudaError_t e = cudaMemsetAsync(ix->goff, 0, ((size_t)n_groups + 1) * 4, c->stream);
    if (e != cudaSuccess) rc = fail(B2P_E_CUDA, "group index offsets: %s", cudaGetErrorString(e));
  }
  if (!rc) {
    // largest group (host-side scan of the offsets: the index is built once per label assignment)
    std::vector<uint32_t> h((size_t)n_groups + 1);
    cudaError_t e = cudaMemcpyAsync(h.data(), ix->goff, h.size() * 4, cudaMemcpyDeviceToHost, c->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
    if (e != cudaSuccess) rc = fail(B2P_E_CUDA, "group index read-back: %s", cudaGetErrorString(e));
    for (uint32_t i = 0; !rc && i < n_groups; ++i)
      if (h[i + 1] - h[i] > ix->max_members) ix->max_members = h[i + 1] - h[i];
    if (!rc) ix->goff_host = std::move(h);
  }
  if (rc) {
    b2p_group_index_destroy(c, ix);
    return rc;
  }
  *out_index = ix;
  return B2P_OK;
}

void b2p_group_index_destroy(b2p_ctx* c, b2p_group_index* ix) {
  if (!ix) return;
  if (c) {
    DeviceGuard g(c->device);
    cudaStreamSynchronize(c->stream);
    if (ix->gid) cudaFree(ix->gid);
    if (ix->goff) cudaFree(ix->goff);
    if (ix->members) cudaFree(ix->members);
  }
  delete ix;
}

int b2p_group_aggregate_indexed_dev(b2p_ctx* c, int32_t agg, const double* vals, const uint32_t* valid_words,
                                    const b2p_group_index* ix, uint64_t T, double* out_val, uint32_t* out_cnt) {
  if (!c || !ix) return fail(B2P_E_INVALID, "NULL argument");
  if (agg < 0 || agg > B2P_AGG_STDVAR) return fail(B2P_E_INVALID, "unknown aggregator %d", agg);
  if (ix->n_groups == 0 || T == 0) return B2P_OK;
  if (!vals || !valid_words || !out_val || !out_cnt) return fail(B2P_E_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  stage_begin(c, 3);
  int rc = group_aggregate_csr(c, agg, vals, valid_words, ix->goff, ix->members, ix->n_groups, T, out_val, out_cnt, 0);
  stage_end(c, 3);
  return rc;
}

// One all-reduce of the by-label partials [n] of every rank, enqueued on the context's stream (asynchronous).
//   SUM / AVG / COUNT   val (plain sums) and cnt are added (the __sum_state / __sum_merge split of the reference,
//                       src/query/src/dist_plan/commutativity.rs:85-113); finalise afterwards (b2p_group_finalize_dev)
//   MIN / MAX           cnt is added; val is reduced as f64::total_cmp keys (int64 min / max), the order of the
//                       single-pass fold (+NaN greatest, -NaN least, -0.0 < +0.0), after groups absent on a rank
//                       (cnt == 0) were set to the neutral key; groups absent everywhere end up 0.0 again
//   STDDEV / STDVAR     inputs are per-rank (cnt, mean, M2 = val): the global mean comes from an all-reduce of
//                       cnt*mean, then M2 = sum_r [M2_r + cnt_r (mean_r - mean)^2] (commutativity.rs:158-191 merges
//                       the same state pairwise); on return mean / val hold the merged state on every rank
int b2p_allreduce_partials_dev(b2p_ctx* c, int32_t agg, double* val, uint32_t* cnt, double* mean, uint64_t n) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  if (agg < 0 || agg > B2P_AGG_STDVAR) return fail(B2P_E_INVALID, "unknown aggregator %d", agg);
  if (n == 0) return B2P_OK;
  if (!val || !cnt) return fail(B2P_E_INVALID, "NULL argument");
  const bool var = agg == B2P_AGG_STDDEV || agg == B2P_AGG_STDVAR;
  if (var && !mean) return fail(B2P_E_INVALID, "stddev / stdvar partials need the per-group means");
  if (!c->comm) return B2P_OK;  // single rank: nothing to merge
  DeviceGuard g(c->device);
  const unsigned blocks = capped_grid(c, n, 256, 16);
  if (agg == B2P_AGG_MIN || agg == B2P_AGG_MAX) {
    minmax_neutral_kernel<<<(unsigned)blocks, 256, 0, c->stream>>>(agg == B2P_AGG_MIN, val, cnt, n, 0);
    const int op = agg == B2P_AGG_MIN ? Nccl::kMin : Nccl::kMax;
    if (int rc = allreduce_with_counts(c, val, Nccl::kInt64, op, cnt, n, c->stream)) return rc;
    minmax_neutral_kernel<<<(unsigned)blocks, 256, 0, c->stream>>>(agg == B2P_AGG_MIN, val, cnt, n, 1);
    c->launches += 2;
  } else if (var) {
    int rc;
    if ((rc = c->m_tmp0.ensure(n * 8)) || (rc = c->m_tmp1.ensure(n * 4))) return rc;
    double* wsum = c->m_tmp0.as<double>();    // cnt_r * mean_r -> global sum
    uint32_t* cnt_r = c->m_tmp1.as<uint32_t>();  // this rank's counts (cnt itself becomes the global count)
    variance_merge_kernel<<<(unsigned)blocks, 256, 0, c->stream>>>(0, val, cnt, mean, wsum, cnt_r, n);
    if ((rc = allreduce_with_counts(c, wsum, Nccl::kFloat64, Nccl::kSum, cnt, n, c->stream))) return rc;
    variance_merge_kernel<<<(unsigned)blocks, 256, 0, c->stream>>>(1, val, cnt, mean, wsum, cnt_r, n);
    NCCL_TRY(g_nccl.AllReduce(val, val, n, Nccl::kFloat64, Nccl::kSum, c->comm, c->stream));
    c->launches += 2;
  } else {
    stage_begin(c, 4);
    if (int rc = allreduce_with_counts(c, val, Nccl::kFloat64, Nccl::kSum, cnt, n, c->stream)) return rc;
    stage_end(c, 4);
  }
  CU(cudaGetLastError());
  return B2P_OK;
}

// The Int64 partials of SUM / MIN / MAX (b2p_group_aggregate_partial_i64_dev), merged in place on the context's stream.
//   SUM        val is added as uint64: modular addition is the wrapping sum in any rank order (a signed NCCL sum is not
//              promised to wrap)
//   MIN / MAX  val is reduced as int64 after groups absent on a rank (cnt == 0) took INT64_MAX / INT64_MIN; groups absent
//              everywhere read 0 again
// cnt is added in both.
int b2p_allreduce_partials_i64_dev(b2p_ctx* c, int32_t agg, double* val, uint32_t* cnt, uint64_t n) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  if (agg != B2P_AGG_SUM && agg != B2P_AGG_MIN && agg != B2P_AGG_MAX)
    return fail(B2P_E_INVALID, "Int64 partials exist for sum, min and max only (aggregator %d)", agg);
  if (n == 0) return B2P_OK;
  if (!val || !cnt) return fail(B2P_E_INVALID, "NULL argument");
  if (!c->comm) return B2P_OK;
  DeviceGuard g(c->device);
  const unsigned blocks = capped_grid(c, n, 256, 16);
  const bool minmax = agg != B2P_AGG_SUM;
  if (minmax) {
    minmax_neutral_kernel<<<blocks, 256, 0, c->stream>>>(agg == B2P_AGG_MIN, val, cnt, n, 0, true);
    c->launches++;
  }
  const int op = agg == B2P_AGG_MIN ? Nccl::kMin : agg == B2P_AGG_MAX ? Nccl::kMax : Nccl::kSum;
  if (int rc = allreduce_with_counts(c, val, minmax ? Nccl::kInt64 : Nccl::kUint64, op, cnt, n, c->stream)) return rc;
  if (minmax) {
    minmax_neutral_kernel<<<blocks, 256, 0, c->stream>>>(agg == B2P_AGG_MIN, val, cnt, n, 1, true);
    c->launches++;
  }
  CU(cudaGetLastError());
  return B2P_OK;
}

// This rank's byte count into sizes[0], or with a communicator every rank's into sizes[n_ranks] (one all-gather of 8 B
// per rank); reads the table back, so it synchronises the stream.
int b2p_group_keys_sizes(b2p_ctx* c, uint64_t bytes, uint64_t* sizes) {
  if (!c || !sizes) return fail(B2P_E_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  const unsigned long long b = bytes;
  return rank_table(c, 1, Nccl::kUint64, sizes, [&](void* mine) {
    CU(cudaMemcpyAsync(mine, &b, 8, cudaMemcpyHostToDevice, c->stream));
    return B2P_OK;
  });
}

// Every rank's block, laid back to back in rank order into the host buffer `out` (sum of sizes bytes): this rank's block
// goes to its place in one device buffer, then one ncclBroadcast per rank with bytes, in one group, each from that
// rank's place (no block is padded), and the buffer comes back.  Synchronises the stream.
int b2p_group_keys_allgather(b2p_ctx* c, const void* block, const uint64_t* sizes, void* out) {
  if (!c || !sizes) return fail(B2P_E_INVALID, "NULL argument");
  const uint32_t R = (uint32_t)c->comm_ranks, me = (uint32_t)c->comm_rank;
  uint64_t N = 0, mine = 0;
  for (uint32_t r = 0; r < R; ++r) {
    if (r == me) mine = N;
    N += sizes[r];
  }
  if ((sizes[me] && !block) || (N && !out)) return fail(B2P_E_INVALID, "NULL argument");
  c->last_group_keys_bytes = (long long)sizes[me];
  if (N == 0) return B2P_OK;
  DeviceGuard g(c->device);
  int rc;
  if ((rc = c->x_recv.ensure(N))) return rc;
  unsigned char* all = static_cast<unsigned char*>(c->x_recv.p);
  if (sizes[me]) CU(cudaMemcpyAsync(all + mine, block, sizes[me], cudaMemcpyHostToDevice, c->stream));
  if ((rc = gather_blocks(c, all, sizes, 1, Nccl::kUint8))) return rc;
  CU(cudaMemcpyAsync(out, all, N, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  return B2P_OK;
}

// config 5 (wide avg_over_time): per-column (sum f64, count u64) of every rank added in place
int b2p_allreduce_columns_dev(b2p_ctx* c, double* sum, uint64_t* cnt, uint32_t n_cols) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  if (n_cols == 0) return B2P_OK;
  if (!sum || !cnt) return fail(B2P_E_INVALID, "NULL argument");
  if (!c->comm) return B2P_OK;
  DeviceGuard g(c->device);
  stage_begin(c, 4);
  if (int rc = nccl_group([&] {
        NCCL_TRY(g_nccl.AllReduce(sum, sum, n_cols, Nccl::kFloat64, Nccl::kSum, c->comm, c->stream));
        NCCL_TRY(g_nccl.AllReduce(cnt, cnt, n_cols, Nccl::kUint64, Nccl::kSum, c->comm, c->stream));
        return B2P_OK;
      })) return rc;
  stage_end(c, 4);
  return B2P_OK;
}

int b2p_group_finalize_dev(b2p_ctx* c, int32_t agg, double* val, const uint32_t* cnt, uint64_t n) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  if (n == 0) return B2P_OK;
  DeviceGuard g(c->device);
  group_finalize_kernel<<<capped_grid(c, n, 256, 16), 256, 0, c->stream>>>(agg, val, cnt, n);
  c->launches++;
  CU(cudaGetLastError());
  return B2P_OK;
}

// HistogramFold over an explicit (histogram -> buckets in le order) index; every pointer is a device pointer.
int b2p_histogram_fold_dev(b2p_ctx* c, double phi, const uint32_t* hist_off, const uint32_t* bucket_series,
                           const double* bucket_le, uint32_t n_hist, const double* rates, const uint32_t* valid_words,
                           uint64_t T, double* out, uint32_t* out_valid_words) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  if (n_hist == 0 || T == 0) return B2P_OK;
  if (!hist_off || !bucket_series || !bucket_le || !rates || !valid_words || !out || !out_valid_words)
    return fail(B2P_E_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  HistFoldArgs a{};
  a.phi = phi; a.hist_off = hist_off; a.bucket_series = bucket_series; a.bucket_le = bucket_le; a.n_hist = n_hist;
  a.rates = rates; a.valid = valid_words; a.T = T; a.Tw = (uint32_t)((T + 31) / 32); a.out = out; a.out_valid = out_valid_words;
  constexpr size_t smem = (size_t)kHistWarps * kHistSmemBuckets * 32 * (8 + 1);  // 72 KB: three CTAs per SM
  unsigned blocks = 0;
  int rc = persistent_grid(c, histogram_fold_kernel, smem, kHistWarps, (uint64_t)n_hist * ((T + 31) / 32), &blocks);
  if (rc) return rc;
  stage_begin(c, 3);
  histogram_fold_kernel<<<blocks, kHistWarps * 32, smem, c->stream>>>(a);
  c->launches++;
  stage_end(c, 3);
  CU(cudaGetLastError());
  return B2P_OK;
}

// Uniform layout: bucket b of histogram h is series h * n_buckets + b and every histogram has the bounds le[].
int b2p_histogram_quantile_dev(b2p_ctx* c, double phi, const double* le, uint32_t n_buckets, const double* rates,
                               const uint32_t* valid_words, uint32_t n_hist, uint64_t T, double* out,
                               uint32_t* out_valid_words) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  if (n_hist == 0 || T == 0) return B2P_OK;
  if (!le || !rates || !valid_words || !out || !out_valid_words || n_buckets == 0)
    return fail(B2P_E_INVALID, "NULL argument");
  if ((uint64_t)n_hist * n_buckets > 0xffffffffull) return fail(B2P_E_TOO_LARGE, "more than 2^32 bucket series");
  DeviceGuard g(c->device);
  int rc;
  const size_t nb = (size_t)n_hist * n_buckets;
  {  // the fold index of the uniform layout (12 B per bucket series, rebuilt per call: microseconds)
    if ((rc = c->hq_off.ensure(((size_t)n_hist + 1) * 4)) || (rc = c->hq_series.ensure(nb * 4)) || (rc = c->hq_les.ensure(nb * 8)))
      return rc;
    const unsigned blocks = capped_grid(c, nb, 256, 16);
    histogram_uniform_index_kernel<<<blocks, 256, 0, c->stream>>>(le, n_buckets, n_hist, c->hq_off.as<uint32_t>(),
                                                                            c->hq_series.as<uint32_t>(), c->hq_les.as<double>());
    c->launches++;
    CU(cudaGetLastError());
  }
  return b2p_histogram_fold_dev(c, phi, c->hq_off.as<uint32_t>(), c->hq_series.as<uint32_t>(), c->hq_les.as<double>(), n_hist,
                                rates, valid_words, T, out, out_valid_words);
}

int b2p_column_reduce_dev(b2p_ctx* c, const double* const* cols, uint32_t n_cols, uint64_t n_rows, double* out_sum,
                          uint64_t* out_cnt) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  if (n_cols == 0 || n_rows == 0) return B2P_OK;
  if (!cols || !out_sum || !out_cnt) return fail(B2P_E_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  unsigned bpc = (unsigned)((c->num_sms * 8 + n_cols - 1) / n_cols);
  if (bpc < 1) bpc = 1;
  const uint64_t max_useful = (n_rows + 511) / 512;
  if (bpc > max_useful) bpc = (unsigned)max_useful;
  int rc;
  if ((rc = c->c_psum.ensure((size_t)n_cols * bpc * 8))) return rc;
  if ((rc = c->c_pcnt.ensure((size_t)n_cols * bpc * 8))) return rc;
  stage_begin(c, 3);
  column_reduce_stage1<<<dim3(bpc, n_cols), 256, 0, c->stream>>>(cols, n_rows, c->c_psum.as<double>(),
                                                                 c->c_pcnt.as<unsigned long long>());
  column_reduce_stage2<<<n_cols, 32, 0, c->stream>>>(c->c_psum.as<double>(), c->c_pcnt.as<unsigned long long>(), bpc,
                                                     out_sum, reinterpret_cast<unsigned long long*>(out_cnt));
  c->launches += 2;
  stage_end(c, 3);
  CU(cudaGetLastError());
  return B2P_OK;
}

/* ---- host-pointer API ------------------------------------------------------------------------ */

namespace {
int group_aggregate_host(b2p_ctx* c, int32_t agg, const double* vals, const uint32_t* valid_words, const uint32_t* gid,
                         uint32_t n_series, uint32_t n_groups, uint64_t T, double* out_val, uint32_t* out_cnt, bool i64) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  DeviceGuard g(c->device);
  const uint32_t Tw = (uint32_t)((T + 31) / 32);
  Staging s{c};
  const double* d_vals = s.in(vals, (size_t)n_series * T * 8);
  const uint32_t* d_valid = s.in(valid_words, (size_t)n_series * Tw * 4);
  const uint32_t* d_gid = s.in(gid, (size_t)n_series * 4);
  double* d_out = s.out(out_val, (size_t)n_groups * T * 8);
  uint32_t* d_cnt = s.out(out_cnt, (size_t)n_groups * T * 4);
  return s.end([&] {
    return group_aggregate_impl(c, agg, d_vals, d_valid, d_gid, n_series, n_groups, T, d_out, d_cnt, 0, nullptr, i64);
  });
}

// The sharded by-label aggregate from host columns: this rank's partials over the global group ids, the all-reduce of
// every rank's, then the finalise (Float64; an Int64 sum / min / max needs none).  A rank without rows still takes part.
int group_allreduce_host(b2p_ctx* c, int32_t agg, const double* vals, const uint32_t* valid_words, const uint32_t* gid,
                         uint32_t n_series, uint32_t n_groups, uint64_t T, double* out_val, uint32_t* out_cnt, bool i64) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  if (n_groups == 0 || T == 0) return B2P_OK;  // (every rank has the same n_groups and T)
  if ((n_series && (!vals || !valid_words || !gid)) || !out_val || !out_cnt) return fail(B2P_E_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  const uint32_t Tw = (uint32_t)((T + 31) / 32);
  const uint64_t n = (uint64_t)n_groups * T;
  const bool var = agg == B2P_AGG_STDDEV || agg == B2P_AGG_STDVAR;
  Staging s{c};
  auto in = [&](const auto* host, size_t bytes) {  // (a rank without rows stages an empty buffer, never NULL)
    return n_series ? s.in(host, bytes) : static_cast<decltype(host)>(s.buf(0));
  };
  const double* d_vals = in(vals, (size_t)n_series * T * 8);
  const uint32_t* d_valid = in(valid_words, (size_t)n_series * Tw * 4);
  const uint32_t* d_gid = in(gid, (size_t)n_series * 4);
  double* d_out = s.out(out_val, n * 8);
  uint32_t* d_cnt = s.out(out_cnt, n * 4);
  double* d_mean = var ? static_cast<double*>(s.buf(n * 8)) : nullptr;
  return s.end([&] {
    int rc = i64 ? b2p_group_aggregate_partial_i64_dev(c, agg, reinterpret_cast<const int64_t*>(d_vals), d_valid, d_gid,
                                                       n_series, n_groups, T, d_out, d_cnt)
                 : b2p_group_aggregate_partial_dev(c, agg, d_vals, d_valid, d_gid, n_series, n_groups, T, d_out, d_cnt,
                                                   d_mean);
    if (!rc) rc = i64 ? b2p_allreduce_partials_i64_dev(c, agg, d_out, d_cnt, n)
                      : b2p_allreduce_partials_dev(c, agg, d_out, d_cnt, d_mean, n);
    if (!rc && !i64) rc = b2p_group_finalize_dev(c, agg, d_out, d_cnt, n);
    return rc;
  });
}
}  // namespace

int b2p_group_aggregate_allreduce(b2p_ctx* c, int32_t agg, const double* vals, const uint32_t* valid_words,
                                  const uint32_t* gid, uint32_t n_series, uint32_t n_groups, uint64_t T, double* out_val,
                                  uint32_t* out_cnt) {
  return group_allreduce_host(c, agg, vals, valid_words, gid, n_series, n_groups, T, out_val, out_cnt, false);
}

int b2p_group_aggregate_allreduce_i64(b2p_ctx* c, int32_t agg, const int64_t* vals, const uint32_t* valid_words,
                                      const uint32_t* gid, uint32_t n_series, uint32_t n_groups, uint64_t T,
                                      double* out_val, uint32_t* out_cnt) {
  return group_allreduce_host(c, agg, reinterpret_cast<const double*>(vals), valid_words, gid, n_series, n_groups, T,
                              out_val, out_cnt, true);
}

int b2p_group_aggregate(b2p_ctx* c, int32_t agg, const double* vals, const uint32_t* valid_words, const uint32_t* gid,
                        uint32_t n_series, uint32_t n_groups, uint64_t T, double* out_val, uint32_t* out_cnt) {
  return group_aggregate_host(c, agg, vals, valid_words, gid, n_series, n_groups, T, out_val, out_cnt, false);
}

int b2p_group_aggregate_i64(b2p_ctx* c, int32_t agg, const int64_t* vals, const uint32_t* valid_words,
                            const uint32_t* gid, uint32_t n_series, uint32_t n_groups, uint64_t T, double* out_val,
                            uint32_t* out_cnt) {
  return group_aggregate_host(c, agg, reinterpret_cast<const double*>(vals), valid_words, gid, n_series, n_groups, T,
                              out_val, out_cnt, true);
}

int b2p_histogram_quantile(b2p_ctx* c, double phi, const double* le, uint32_t n_buckets, const double* rates,
                           const uint32_t* valid_words, uint32_t n_hist, uint64_t T, double* out,
                           uint32_t* out_valid_words) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  DeviceGuard g(c->device);
  const uint32_t Tw = (uint32_t)((T + 31) / 32);
  const size_t ns = (size_t)n_hist * n_buckets;
  Staging s{c};
  const double* d_rates = s.in(rates, ns * T * 8);
  const uint32_t* d_valid = s.in(valid_words, ns * Tw * 4);
  const double* d_le = s.in(le, (size_t)n_buckets * 8);
  double* d_out = s.out(out, (size_t)n_hist * T * 8);
  uint32_t* d_out_valid = s.out(out_valid_words, (size_t)n_hist * Tw * 4);
  return s.end([&] {
    return b2p_histogram_quantile_dev(c, phi, d_le, n_buckets, d_rates, d_valid, n_hist, T, d_out, d_out_valid);
  });
}

// HistogramFold over any [n_rows x T] grid: the index is checked on the host, so a bad one never reaches K5; then the
// grid, its bitmap and the index go to the device, and [n_hist x T] comes back.
int b2p_histogram_fold(b2p_ctx* c, double phi, const uint32_t* hist_off, const uint32_t* bucket_series,
                       const double* bucket_le, uint32_t n_hist, const double* rates, const uint32_t* valid_words,
                       uint32_t n_rows, uint64_t T, double* out, uint32_t* out_valid_words) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  if (n_hist == 0 || T == 0) return B2P_OK;  // (no fold: the index is not read)
  if (!hist_off || !bucket_series) return fail(B2P_E_INVALID, "NULL argument");
  if (hist_off[0] != 0) return fail(B2P_E_INVALID, "hist_off[0] is %u, not 0", hist_off[0]);
  for (uint32_t h = 0; h < n_hist; ++h)
    if (hist_off[h + 1] < hist_off[h]) return fail(B2P_E_INVALID, "hist_off decreases at histogram %u", h);
  const size_t nb = hist_off[n_hist];
  for (size_t i = 0; i < nb; ++i)
    if (bucket_series[i] >= n_rows)
      return fail(B2P_E_INVALID, "bucket_series[%zu] = %u is not a row (n_rows = %u)", i, bucket_series[i], n_rows);
  DeviceGuard g(c->device);
  const uint32_t Tw = (uint32_t)((T + 31) / 32);
  Staging s{c};
  const double* d_rates = s.in(rates, (size_t)n_rows * T * 8);
  const uint32_t* d_valid = s.in(valid_words, (size_t)n_rows * Tw * 4);
  const uint32_t* d_hist_off = s.in(hist_off, ((size_t)n_hist + 1) * 4);
  const uint32_t* d_bucket_series = s.in(bucket_series, nb * 4);
  const double* d_bucket_le = s.in(bucket_le, nb * 8);
  double* d_out = s.out(out, (size_t)n_hist * T * 8);
  uint32_t* d_out_valid = s.out(out_valid_words, (size_t)n_hist * Tw * 4);
  return s.end([&] {
    return b2p_histogram_fold_dev(c, phi, d_hist_off, d_bucket_series, d_bucket_le, n_hist, d_rates, d_valid, T, d_out,
                                  d_out_valid);
  });
}

// histogram_quantile(phi, fn(bucket_series[range])) from host buffers to host rows without the dense [n_series x T]
// matrix ever leaving the device: H2D of the samples, series offsets, the range function into context scratch, the
// HistogramFold over the caller's (histogram -> buckets in le order) index, D2H of [n_hist x T] only.
int b2p_range_histogram_fold(b2p_ctx* c, const b2p_range_params* p, const int64_t* ts, const double* val,
                             const uint32_t* sid, const uint64_t* offsets_host, uint64_t n_rows, uint32_t n_series,
                             double phi, const uint32_t* hist_off, const uint32_t* bucket_series, const double* bucket_le,
                             uint32_t n_hist, double* out, uint32_t* out_valid_words) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  int64_t T = 0;
  int rc = check_grid(p, n_series, &T);
  if (rc) return rc;
  if (n_hist == 0 || T == 0) return B2P_OK;  // (no range evaluation whose rates nothing folds)
  if (!hist_off) return fail(B2P_E_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  if (!c->pending.empty() && (rc = b2p_sync(c))) return rc;
  const uint32_t Tw = (uint32_t)((T + 31) / 32);
  const size_t nb = hist_off[n_hist];
  Staging s{c};
  const SeriesIn in = stage_series(s, ts, val, sid, 0u, offsets_host, n_rows, n_series);
  const uint32_t* d_hist_off = s.in(hist_off, ((size_t)n_hist + 1) * 4);
  const uint32_t* d_bucket_series = s.in(bucket_series, nb * 4);
  const double* d_bucket_le = s.in(bucket_le, nb * 8);
  double* d_rates = static_cast<double*>(s.buf((size_t)n_series * (size_t)T * 8));
  uint32_t* d_rates_valid = static_cast<uint32_t*>(s.buf((size_t)n_series * Tw * 4));
  double* d_out = s.out(out, (size_t)n_hist * (size_t)T * 8);
  uint32_t* d_out_valid = s.out(out_valid_words, (size_t)n_hist * Tw * 4);
  return s.end([&] {
    int r = b2p_range_eval_dev(c, p, in.ts, in.val, in.offsets, n_rows, n_series, d_rates, d_rates_valid);
    if (!r) r = b2p_sync(c);  // slow-path fix-ups land before the fold reads
    return r ? r : b2p_histogram_fold_dev(c, phi, d_hist_off, d_bucket_series, d_bucket_le, n_hist, d_rates,
                                          d_rates_valid, (uint64_t)T, d_out, d_out_valid);
  });
}

}  // extern "C"
