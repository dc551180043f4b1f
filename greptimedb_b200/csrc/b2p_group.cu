// b2p_group.cu — by-label entry points of the C ABI: the group index, by-label aggregates and their partials, the
// all-reduce of partials over NCCL, HistogramFold / histogram_quantile and the column reduce.
#include <algorithm>
#include <cmath>
#include <new>
#include <numeric>
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

}  // extern "C"

namespace {
// out row dst[i] = in row src[i] for i < n, values and validity words (row_move_kernel); device pointers
int row_move(b2p_ctx* c, const double* in, const uint32_t* in_valid, const uint32_t* src, const uint32_t* dst, uint32_t n,
             uint64_t T, double* out, uint32_t* out_valid) {
  if (n == 0 || T == 0) return B2P_OK;
  const RowMoveArgs a{in, in_valid, src, dst, n, T, (uint32_t)((T + 31) / 32), out, out_valid};
  const unsigned blocks = capped_grid(c, (uint64_t)n * 32, 256, 8);
  if (T % 2 == 0 && aligned16(in) && aligned16(out)) row_move_kernel<true><<<blocks, 256, 0, c->stream>>>(a);
  else row_move_kernel<false><<<blocks, 256, 0, c->stream>>>(a);
  c->launches++;
  CU(cudaGetLastError());
  return B2P_OK;
}
}  // namespace

extern "C" {

int b2p_row_move_dev(b2p_ctx* c, const double* in, const uint32_t* in_valid, const uint32_t* src, const uint32_t* dst,
                     uint32_t n, uint64_t T, double* out, uint32_t* out_valid) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  if (n == 0 || T == 0) return B2P_OK;
  if (!in || !in_valid || !src || !dst || !out || !out_valid) return fail(B2P_E_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  return row_move(c, in, in_valid, src, dst, n, T, out, out_valid);
}

// A histogram's owner: the rank with the most of its buckets, the lowest on a tie (a function of the table alone).
int b2p_histogram_shard_owners(const uint32_t* counts, int32_t n_ranks, uint32_t n_hist, uint32_t* owner) {
  if (n_ranks < 1) return fail(B2P_E_INVALID, "n_ranks %d < 1", n_ranks);
  if (n_hist && (!counts || !owner)) return fail(B2P_E_INVALID, "NULL argument");
  for (uint32_t h = 0; h < n_hist; ++h) {
    uint32_t best = 0;
    for (uint32_t r = 1; r < (uint32_t)n_ranks; ++r)
      if (counts[(size_t)r * n_hist + h] > counts[(size_t)best * n_hist + h]) best = r;
    owner[h] = best;
  }
  return B2P_OK;
}

// The HistogramFold index over n buckets: histogram, then bound ascending with NaN last (-0.0 ties +0.0), then (rank,
// row).  The keys are distinct wherever (rank, row) is, so the order is total and any sort gives it.  The plan layer's
// unsharded index is this call with rank 0 and row = the row itself.
int b2p_histogram_shard_index(const uint32_t* hist, const double* le, const uint32_t* rank, const uint32_t* row,
                              uint32_t n, uint32_t n_hist, uint32_t* hist_off, uint32_t* bucket_series, double* bucket_le) {
  if (!hist_off || (n && (!hist || !le || !rank || !row || !bucket_series || !bucket_le)))
    return fail(B2P_E_INVALID, "NULL argument");
  std::fill(hist_off, hist_off + (size_t)n_hist + 1, 0u);
  for (uint32_t i = 0; i < n; ++i) {
    if (hist[i] >= n_hist) return fail(B2P_E_INVALID, "hist[%u] = %u is not a histogram (n_hist = %u)", i, hist[i], n_hist);
    hist_off[hist[i] + 1]++;
  }
  for (uint32_t h = 0; h < n_hist; ++h) hist_off[h + 1] += hist_off[h];
  {  // the buckets by histogram (a counting sort), then each histogram's by (bound, rank, row)
    std::vector<uint32_t> at(hist_off, hist_off + n_hist);
    for (uint32_t i = 0; i < n; ++i) bucket_series[at[hist[i]]++] = i;
  }
  const auto less = [&](uint32_t x, uint32_t y) {
    const bool nx = std::isnan(le[x]), ny = std::isnan(le[y]);
    if (nx != ny) return ny;
    if (!nx && le[x] != le[y]) return le[x] < le[y];
    if (rank[x] != rank[y]) return rank[x] < rank[y];
    return row[x] < row[y];
  };
  for (uint32_t h = 0; h < n_hist; ++h) std::sort(bucket_series + hist_off[h], bucket_series + hist_off[h + 1], less);
  for (uint32_t j = 0; j < n; ++j) bucket_le[j] = le[bucket_series[j]];
  return B2P_OK;
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

namespace {
// What travels with each shuffled bucket row of the sharded HistogramFold
struct BucketHeader {
  double le;
  uint32_t hist, rank, row, pad;
};
static_assert(sizeof(BucketHeader) == 24, "the bucket header is 24 bytes on every rank");

size_t align16(size_t b) { return (b + 15) & ~(size_t)15; }

// The sharded HistogramFold's plan, from the counts table alone (so every rank derives the same one): owners, each
// histogram's place among its owner's, the batches of contiguous histograms, this rank's largest batch send and
// receive, and its rows by (histogram, row).
struct HistShard {
  uint32_t H = 0, R = 1, me = 0, Tw = 0, n_rows = 0;
  uint64_t T = 0;
  const double* row_le = nullptr;
  std::vector<uint32_t> counts;          // [R x H]
  std::vector<uint32_t> owner, pos;      // [H]
  std::vector<uint64_t> own_n;           // [R] histograms each rank owns
  std::vector<uint32_t> cut;             // batch b: histograms cut[b] .. cut[b + 1]
  uint64_t send_max = 0, recv_max = 0, mine_off = 0;
  std::vector<uint32_t> loff, lrows;     // this rank's rows of histogram h: lrows[loff[h] .. loff[h + 1]]
  uint64_t cnt(uint32_t r, uint32_t h) const { return counts[(size_t)r * H + h]; }
  uint64_t grid_rows() const { return (uint64_t)n_rows + recv_max; }  // the fold's grid: own rows, then a batch's received
};

// Step 1 to 3 of b2p_histogram_fold_allgather (collective: one all-gather).  The table carries one more column per rank,
// set where that rank's row_hist names no histogram, so such a rank fails on every rank alike, after the collective.
int hist_shard_plan(b2p_ctx* c, const uint32_t* row_hist, const double* row_le, uint32_t n_rows, uint32_t n_hist,
                    uint64_t T, HistShard& sh) {
  const uint32_t H = n_hist, R = (uint32_t)c->comm_ranks, me = (uint32_t)c->comm_rank;
  sh.H = H; sh.R = R; sh.me = me; sh.T = T; sh.Tw = (uint32_t)((T + 31) / 32); sh.n_rows = n_rows;
  sh.row_le = row_le;
  std::vector<uint32_t> mine((size_t)H + 1, 0u);
  for (uint32_t i = 0; i < n_rows; ++i) {
    if (row_hist[i] >= H) mine[H] = 1;
    else ++mine[row_hist[i]];
  }
  std::vector<uint32_t> table((size_t)R * (H + 1));
  if (int rc = rank_table(c, (size_t)H + 1, Nccl::kUint32, table.data(), [&](void* slot) {
        CU(cudaMemcpyAsync(slot, mine.data(), ((size_t)H + 1) * 4, cudaMemcpyHostToDevice, c->stream));
        return B2P_OK;
      }))
    return rc;
  sh.counts.resize((size_t)R * H);
  uint64_t total = 0;
  for (uint32_t r = 0; r < R; ++r) {
    if (table[(size_t)r * (H + 1) + H])
      return fail(B2P_E_INVALID, "histogram_quantile: rank %u passed a row_hist entry >= n_hist (%u)", r, H);
    for (uint32_t h = 0; h < H; ++h) total += sh.counts[(size_t)r * H + h] = table[(size_t)r * (H + 1) + h];
  }
  if (total > UINT32_MAX) return fail(B2P_E_TOO_LARGE, "histogram_quantile: more than 2^32 - 1 bucket rows over the ranks");
  // 2. owners, and each histogram's place among its owner's
  sh.owner.resize(H);
  sh.pos.resize(H);
  sh.own_n.assign(R, 0);
  b2p_histogram_shard_owners(sh.counts.data(), (int32_t)R, H, sh.owner.data());
  for (uint32_t h = 0; h < H; ++h) sh.pos[h] = (uint32_t)sh.own_n[sh.owner[h]]++;
  for (uint32_t r = 0; r < me; ++r) sh.mine_off += sh.own_n[r];
  // 3. batches: a histogram joins the batch while every rank's sent and received rows of the batch fit the cap
  const uint64_t row_bytes = T * 8 + (uint64_t)sh.Tw * 4 + sizeof(BucketHeader);
  sh.cut.assign(1, 0u);
  std::vector<uint64_t> load(R, 0);
  uint64_t send_b = 0, recv_b = 0;  // this rank's rows of the current batch
  for (uint32_t h = 0; h < H; ++h) {
    const uint32_t o = sh.owner[h];
    uint64_t moved = 0;
    for (uint32_t r = 0; r < R; ++r) moved += r == o ? 0 : sh.cnt(r, h);
    bool over = false;
    for (uint32_t r = 0; r < R && h > sh.cut.back(); ++r)
      over = over || (load[r] + (r == o ? moved : sh.cnt(r, h))) * row_bytes > c->topk_exchange_cap;
    if (over) {
      sh.cut.push_back(h);
      std::fill(load.begin(), load.end(), 0);
      send_b = recv_b = 0;
    }
    for (uint32_t r = 0; r < R; ++r) load[r] += r == o ? moved : sh.cnt(r, h);
    if (o == me) recv_b += moved;
    else send_b += sh.cnt(me, h);
    sh.send_max = std::max(sh.send_max, send_b);
    sh.recv_max = std::max(sh.recv_max, recv_b);
  }
  sh.cut.push_back(H);
  // this rank's rows by (histogram, row)
  sh.loff.assign((size_t)H + 1, 0u);
  sh.lrows.resize(n_rows);
  for (uint32_t i = 0; i < n_rows; ++i) ++sh.loff[row_hist[i] + 1];
  std::partial_sum(sh.loff.begin(), sh.loff.end(), sh.loff.begin());
  std::vector<uint32_t> at(sh.loff.begin(), sh.loff.end() - 1);
  for (uint32_t i = 0; i < n_rows; ++i) sh.lrows[at[row_hist[i]]++] = i;
  return B2P_OK;
}

// Steps 4 to 7 over this rank's rows in g_val / g_valid (sh.grid_rows() rows of room): the shuffle, the owners' folds
// into a_val / a_valid [H] (every owner's results, rank by rank), their gather and placement into out / out_valid.
// Where no histogram is split across ranks no row is packed or sent and no point-to-point group is opened: each rank
// folds its own histograms over its own rows, and only the results travel.
int hist_shard_run(b2p_ctx* c, const HistShard& sh, double phi, double* g_val, uint32_t* g_valid, double* a_val,
                   uint32_t* a_valid, double* d_out, uint32_t* d_out_valid) {
  int rc;
  const uint32_t H = sh.H, R = sh.R, me = sh.me, Tw = sh.Tw, n_rows = sh.n_rows;
  const uint64_t T = sh.T, G = sh.grid_rows(), send_max = sh.send_max, recv_max = sh.recv_max, mine_off = sh.mine_off;
  const uint64_t row_bytes = T * 8 + (uint64_t)Tw * 4 + sizeof(BucketHeader);
  const std::vector<uint32_t>&owner = sh.owner, &pos = sh.pos, &cut = sh.cut, &loff = sh.loff, &lrows = sh.lrows;
  const std::vector<uint64_t>& own_n = sh.own_n;
  const double* row_le = sh.row_le;
  auto cnt = [&](uint32_t r, uint32_t h) { return sh.cnt(r, h); };
  const size_t sv = align16(send_max * T * 8), sw = align16(send_max * Tw * 4);
  const size_t tab = std::max<size_t>(align16(((size_t)H + 1) * 4) + align16(G * 4) + G * 8, 2 * align16((size_t)std::max<uint64_t>(send_max, H) * 4));
  if ((rc = c->x_send.ensure(sv + sw + send_max * sizeof(BucketHeader))) || (rc = c->x_recv.ensure(recv_max * sizeof(BucketHeader))) ||
      (rc = c->x_table.ensure(tab)))
    return rc;
  char* xs = c->x_send.as<char>();
  double* s_val = reinterpret_cast<double*>(xs);
  uint32_t* s_valid = reinterpret_cast<uint32_t*>(xs + sv);
  char* s_hdr = xs + sv + sw;
  char* r_hdr = c->x_recv.as<char>();
  uint32_t* t_u32 = c->x_table.as<uint32_t>();
  // the two u32 columns of a move (src, dst), uploaded and moved
  auto move = [&](const std::vector<uint32_t>& src, const std::vector<uint32_t>& dst, const double* in,
                  const uint32_t* in_valid, double* o_val, uint32_t* o_valid) {
    const size_t n = src.size(), half = align16(n * 4) / 4;
    if (n == 0) return B2P_OK;
    CU(cudaMemcpyAsync(t_u32, src.data(), n * 4, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(t_u32 + half, dst.data(), n * 4, cudaMemcpyHostToDevice, c->stream));
    return row_move(c, in, in_valid, t_u32, t_u32 + half, (uint32_t)n, T, o_val, o_valid);
  };
  uint64_t sent = 0;
  for (size_t b = 0; b + 1 < cut.size(); ++b) {
    const uint32_t h0 = cut[b], h1 = cut[b + 1];
    // 4. this rank's rows of histograms it does not own, grouped by owner, in (histogram, row) order
    std::vector<uint64_t> send_n(R, 0), recv_n(R, 0);
    std::vector<uint32_t> src, dst;
    std::vector<BucketHeader> hdr;
    for (uint32_t q = 0; q < R; ++q)
      for (uint32_t h = h0; h < h1; ++h) {
        if (owner[h] != q) continue;
        if (q == me) {
          for (uint32_t r = 0; r < R; ++r) recv_n[r] += r == me ? 0 : cnt(r, h);
          continue;
        }
        send_n[q] += cnt(me, h);
        for (uint32_t j = loff[h]; j < loff[h + 1]; ++j) {
          src.push_back(lrows[j]);
          hdr.push_back(BucketHeader{row_le[lrows[j]], h, me, lrows[j], 0u});
        }
      }
    dst.resize(src.size());
    std::iota(dst.begin(), dst.end(), 0u);
    if (!hdr.empty()) CU(cudaMemcpyAsync(s_hdr, hdr.data(), hdr.size() * sizeof(BucketHeader), cudaMemcpyHostToDevice, c->stream));
    if ((rc = move(src, dst, g_val, g_valid, s_val, s_valid))) return rc;
    sent += src.size();
    uint64_t n_recv = 0;
    for (uint32_t r = 0; r < R; ++r) n_recv += recv_n[r];
    // 5. the shuffle: one group of point-to-point calls, rows into the grid after this rank's own
    if (c->comm && (n_recv || !src.empty()) && (rc = nccl_group([&] {
          uint64_t so = 0, ro = 0;
          for (uint32_t q = 0; q < R; ++q) {
            if (send_n[q]) {
              NCCL_TRY(g_nccl.Send(s_val + so * T, send_n[q] * T, Nccl::kFloat64, (int)q, c->comm, c->stream));
              NCCL_TRY(g_nccl.Send(s_valid + so * Tw, send_n[q] * Tw, Nccl::kUint32, (int)q, c->comm, c->stream));
              NCCL_TRY(g_nccl.Send(s_hdr + so * sizeof(BucketHeader), send_n[q] * sizeof(BucketHeader), Nccl::kUint8,
                                   (int)q, c->comm, c->stream));
            }
            if (recv_n[q]) {
              const uint64_t at = n_rows + ro;
              NCCL_TRY(g_nccl.Recv(g_val + at * T, recv_n[q] * T, Nccl::kFloat64, (int)q, c->comm, c->stream));
              NCCL_TRY(g_nccl.Recv(g_valid + at * Tw, recv_n[q] * Tw, Nccl::kUint32, (int)q, c->comm, c->stream));
              NCCL_TRY(g_nccl.Recv(r_hdr + ro * sizeof(BucketHeader), recv_n[q] * sizeof(BucketHeader), Nccl::kUint8,
                                   (int)q, c->comm, c->stream));
            }
            so += send_n[q];
            ro += recv_n[q];
          }
          return B2P_OK;
        })))
      return rc;
    // 6. the owner's index over [its rows | the received rows] and K5 into its results
    uint32_t p0 = UINT32_MAX, nh = 0;
    for (uint32_t h = h0; h < h1; ++h)
      if (owner[h] == me) {
        if (p0 == UINT32_MAX) p0 = pos[h];
        ++nh;
      }
    if (nh == 0) continue;
    std::vector<BucketHeader> rh(n_recv);
    if (n_recv) {
      CU(cudaMemcpyAsync(rh.data(), r_hdr, n_recv * sizeof(BucketHeader), cudaMemcpyDeviceToHost, c->stream));
      CU(cudaStreamSynchronize(c->stream));
    }
    std::vector<uint32_t> ih, irank, irow, buf_row;
    std::vector<double> ile;
    auto entry = [&](uint32_t h, double le, uint32_t r, uint32_t row, uint32_t at) {
      ih.push_back(pos[h] - p0);
      ile.push_back(le);
      irank.push_back(r);
      irow.push_back(row);
      buf_row.push_back(at);
    };
    for (uint32_t h = h0; h < h1; ++h)
      if (owner[h] == me)
        for (uint32_t j = loff[h]; j < loff[h + 1]; ++j) entry(h, row_le[lrows[j]], me, lrows[j], lrows[j]);
    for (uint64_t i = 0; i < n_recv; ++i) {
      const BucketHeader& x = rh[i];
      if (x.hist < h0 || x.hist >= h1 || owner[x.hist] != me)
        return fail(B2P_E_INVALID, "histogram_quantile: received a bucket of histogram %u, not one of this rank's", x.hist);
      entry(x.hist, x.le, x.rank, x.row, (uint32_t)(n_rows + i));
    }
    const uint32_t ne = (uint32_t)ih.size();
    std::vector<uint32_t> hoff(nh + 1), bs(ne);
    std::vector<double> ble(ne);
    if ((rc = b2p_histogram_shard_index(ih.data(), ile.data(), irank.data(), irow.data(), ne, nh, hoff.data(), bs.data(),
                                        ble.data())))
      return rc;
    for (uint32_t& x : bs) x = buf_row[x];
    uint32_t* d_hoff = t_u32;
    uint32_t* d_bs = t_u32 + align16((size_t)(nh + 1) * 4) / 4;
    double* d_ble = reinterpret_cast<double*>(reinterpret_cast<char*>(d_bs) + align16((size_t)ne * 4));
    CU(cudaMemcpyAsync(d_hoff, hoff.data(), (size_t)(nh + 1) * 4, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(d_bs, bs.data(), (size_t)ne * 4, cudaMemcpyHostToDevice, c->stream));
    CU(cudaMemcpyAsync(d_ble, ble.data(), (size_t)ne * 8, cudaMemcpyHostToDevice, c->stream));
    if ((rc = b2p_histogram_fold_dev(c, phi, d_hoff, d_bs, d_ble, nh, g_val, g_valid, T, a_val + (mine_off + p0) * T,
                                     a_valid + (mine_off + p0) * Tw)))
      return rc;
  }
  // 7. every owner's results to every rank, then placed in global order
  if ((rc = gather_blocks(c, a_val, own_n.data(), T * 8, Nccl::kFloat64)) ||
      (rc = gather_blocks(c, a_valid, own_n.data(), (size_t)Tw * 4, Nccl::kUint32)))
    return rc;
  c->last_exchange_bytes = (long long)(sent * row_bytes + own_n[me] * (T * 8 + (uint64_t)Tw * 4));
  std::vector<uint32_t> src(H), dst;
  std::iota(src.begin(), src.end(), 0u);
  for (uint32_t r = 0; r < R; ++r)
    for (uint32_t h = 0; h < H; ++h)
      if (owner[h] == r) dst.push_back(h);
  return move(src, dst, a_val, a_valid, d_out, d_out_valid);
}

int hist_shard_check(b2p_ctx* c, uint32_t n_rows, uint64_t T, const uint32_t* row_hist, const double* row_le,
                     uint32_t n_hist, double* out, uint32_t* out_valid_words) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  c->last_exchange_bytes = 0;
  if (n_hist == 0 || T == 0) return B2P_OK;
  if ((n_rows && (!row_hist || !row_le)) || !out || !out_valid_words) return fail(B2P_E_INVALID, "NULL argument");
  return B2P_OK;
}

// b2p_histogram_fold_allgather: this rank's host grid staged into the fold's grid, then the plan and the run
int histogram_fold_allgather_host(b2p_ctx* c, double phi, const double* rates, const uint32_t* valid_words,
                                  uint32_t n_rows, uint64_t T, const uint32_t* row_hist, const double* row_le,
                                  uint32_t n_hist, double* out, uint32_t* out_valid_words) {
  if (int rc = hist_shard_check(c, n_rows, T, row_hist, row_le, n_hist, out, out_valid_words)) return rc;
  if (n_hist == 0 || T == 0) return B2P_OK;  // (every rank has the same n_hist and T)
  if (n_rows && (!rates || !valid_words)) return fail(B2P_E_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  HistShard sh;
  if (int rc = hist_shard_plan(c, row_hist, row_le, n_rows, n_hist, T, sh)) return rc;
  const uint64_t G = sh.grid_rows(), Tw = sh.Tw;
  Staging s{c};
  double* g_val = static_cast<double*>(s.buf(G * T * 8));
  uint32_t* g_valid = static_cast<uint32_t*>(s.buf(G * Tw * 4));
  if (n_rows && g_val && g_valid) {
    s.cuda(cudaMemcpyAsync(g_val, rates, (size_t)n_rows * T * 8, cudaMemcpyHostToDevice, c->stream), "host-to-device copy");
    s.cuda(cudaMemcpyAsync(g_valid, valid_words, (size_t)n_rows * Tw * 4, cudaMemcpyHostToDevice, c->stream),
           "host-to-device copy");
  }
  double* a_val = static_cast<double*>(s.buf((size_t)n_hist * T * 8));
  uint32_t* a_valid = static_cast<uint32_t*>(s.buf((size_t)n_hist * Tw * 4));
  double* d_out = s.out(out, (size_t)n_hist * T * 8);
  uint32_t* d_out_valid = s.out(out_valid_words, (size_t)n_hist * Tw * 4);
  return s.end([&] { return hist_shard_run(c, sh, phi, g_val, g_valid, a_val, a_valid, d_out, d_out_valid); });
}

// b2p_range_histogram_fold_allgather: the range function writes this rank's series straight into the fold's grid, so
// the dense matrix never leaves the device, whether or not any histogram is split
int range_histogram_fold_allgather_host(b2p_ctx* c, const b2p_range_params* p, const int64_t* ts, const double* val,
                                        const uint32_t* sid, const uint64_t* offsets_host, uint64_t n_samples,
                                        uint32_t n_series, double phi, const uint32_t* row_hist, const double* row_le,
                                        uint32_t n_hist, double* out, uint32_t* out_valid_words) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  int64_t T = 0;
  if (int rc = check_grid(p, n_series, &T)) return rc;
  if (int rc = hist_shard_check(c, n_series, (uint64_t)T, row_hist, row_le, n_hist, out, out_valid_words)) return rc;
  if (n_hist == 0 || T == 0) return B2P_OK;  // (every rank has the same n_hist and T)
  DeviceGuard g(c->device);
  int rc;
  if (!c->pending.empty() && (rc = b2p_sync(c))) return rc;
  HistShard sh;
  if ((rc = hist_shard_plan(c, row_hist, row_le, n_series, n_hist, (uint64_t)T, sh))) return rc;
  const uint64_t G = sh.grid_rows(), Tw = sh.Tw;
  Staging s{c};
  const SeriesIn in = n_series ? stage_series(s, ts, val, sid, 0u, offsets_host, n_samples, n_series) : SeriesIn{};
  double* g_val = static_cast<double*>(s.buf(G * (uint64_t)T * 8));
  uint32_t* g_valid = static_cast<uint32_t*>(s.buf(G * Tw * 4));
  double* a_val = static_cast<double*>(s.buf((size_t)n_hist * (size_t)T * 8));
  uint32_t* a_valid = static_cast<uint32_t*>(s.buf((size_t)n_hist * Tw * 4));
  double* d_out = s.out(out, (size_t)n_hist * (size_t)T * 8);
  uint32_t* d_out_valid = s.out(out_valid_words, (size_t)n_hist * Tw * 4);
  return s.end([&] {
    int r = n_series ? b2p_range_eval_dev(c, p, in.ts, in.val, in.offsets, n_samples, n_series, g_val, g_valid) : B2P_OK;
    if (!r && n_series) r = b2p_sync(c);  // slow-path fix-ups land before the fold reads
    return r ? r : hist_shard_run(c, sh, phi, g_val, g_valid, a_val, a_valid, d_out, d_out_valid);
  });
}
}  // namespace

extern "C" {

int b2p_histogram_fold_allgather(b2p_ctx* c, double phi, const double* rates, const uint32_t* valid_words,
                                 uint32_t n_rows, uint64_t T, const uint32_t* row_hist, const double* row_le,
                                 uint32_t n_hist, double* out, uint32_t* out_valid_words) {
  return histogram_fold_allgather_host(c, phi, rates, valid_words, n_rows, T, row_hist, row_le, n_hist, out,
                                       out_valid_words);
}

int b2p_range_histogram_fold_allgather(b2p_ctx* c, const b2p_range_params* p, const int64_t* ts, const double* val,
                                       const uint32_t* sid, const uint64_t* offsets_host, uint64_t n_samples,
                                       uint32_t n_series, double phi, const uint32_t* row_hist, const double* row_le,
                                       uint32_t n_hist, double* out, uint32_t* out_valid_words) {
  return range_histogram_fold_allgather_host(c, p, ts, val, sid, offsets_host, n_samples, n_series, phi, row_hist,
                                             row_le, n_hist, out, out_valid_words);
}

}  // extern "C"
