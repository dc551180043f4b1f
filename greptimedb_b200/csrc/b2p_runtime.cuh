// b2p_runtime.cuh — host-side runtime shared by the translation units of libb200promql.so: errors, the context and its
// device scratch, the group index, the launch helpers and the staging of synchronous host calls.  No kernels here:
// each kernel header is included by the one .cu file that launches its kernels.
//   b2p_context.cu      create / destroy, streams, counters, errors, NCCL communicator
//   b2p_range.cu        range tiers, series offsets, range / instant selectors, fused sum by, subqueries
//   b2p_group.cu        group index, by-label aggregates, all-reduce of partials, HistogramFold, column reduce
//   b2p_elementwise.cu  binary operators, instant-vector functions, scalar(), absent(), set operators
//   b2p_aggregation.cu  topk / bottomk, quantile, count_values
//   b2p_sort.cu         sort / sort_desc, and over rows sharded across ranks
// There is NO CPU fallback anywhere: every entry point either launches the CUDA kernels or returns an error.
#pragma once
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <cstdint>
#include <cstdlib>
#include <map>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "../../include/b200promql.h"
#include "b2p_status.cuh"

// Sets the calling thread's b2p_last_error() message and returns `code`.
int fail(int code, const char* fmt, ...);

#define CU(x)                                                                                   \
  do {                                                                                          \
    cudaError_t e__ = (x);                                                                      \
    if (e__ != cudaSuccess) return fail(B2P_E_CUDA, "%s: %s (%s:%d)", #x, cudaGetErrorString(e__), __FILE__, __LINE__); \
  } while (0)

// error of a non-zero Status::k0_errors word
int k0_fail(uint32_t k0);

// NCCL, bound at run time: libnccl.so.2 is not a link dependency (single-GPU users never need it), and inside a
// process that already loaded an NCCL (e.g. the one bundled with torch) dlopen hands back that same library.
// Only the entry points the by-label all-reduce and the sharded operators need, called through nccl_group (every
// group), allreduce_with_counts (partials and their counts), rank_table (a per-rank table) and gather_blocks
// (variable-size blocks); Send / Recv are the sharded HistogramFold's point-to-point shuffle.  Enum values are NCCL's
// ABI (nccl.h).
struct Nccl {
  typedef struct ncclComm* comm_t;
  struct unique_id { char internal[128]; };
  enum { kSum = 0, kMax = 2, kMin = 3 };
  enum { kUint8 = 1, kUint32 = 3, kInt64 = 4, kUint64 = 5, kFloat64 = 8 };
  static size_t bytes(int type) { return type == kUint8 ? 1 : type == kUint32 ? 4 : 8; }  // of one element
  int (*GetUniqueId)(unique_id*) = nullptr;
  int (*CommInitRank)(comm_t*, int, unique_id, int) = nullptr;
  int (*CommDestroy)(comm_t) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, comm_t, cudaStream_t) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, comm_t, cudaStream_t) = nullptr;
  int (*Broadcast)(const void*, void*, size_t, int, int, comm_t, cudaStream_t) = nullptr;
  int (*Send)(const void*, size_t, int, int, comm_t, cudaStream_t) = nullptr;
  int (*Recv)(void*, size_t, int, int, comm_t, cudaStream_t) = nullptr;
  int (*GroupStart)() = nullptr;
  int (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  void* handle = nullptr;
  bool load() {
    if (handle) return true;
    const char* names[] = {getenv("B2P_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
    for (const char* n : names) {
      if (!n || !*n) continue;
      handle = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
      if (handle) break;
    }
    if (!handle) return false;
    bool ok = true;
    auto sym = [&](const char* n) { void* p = dlsym(handle, n); ok = ok && p; return p; };
    GetUniqueId = reinterpret_cast<decltype(GetUniqueId)>(sym("ncclGetUniqueId"));
    CommInitRank = reinterpret_cast<decltype(CommInitRank)>(sym("ncclCommInitRank"));
    CommDestroy = reinterpret_cast<decltype(CommDestroy)>(sym("ncclCommDestroy"));
    AllReduce = reinterpret_cast<decltype(AllReduce)>(sym("ncclAllReduce"));
    AllGather = reinterpret_cast<decltype(AllGather)>(sym("ncclAllGather"));
    Broadcast = reinterpret_cast<decltype(Broadcast)>(sym("ncclBroadcast"));
    Send = reinterpret_cast<decltype(Send)>(sym("ncclSend"));
    Recv = reinterpret_cast<decltype(Recv)>(sym("ncclRecv"));
    GroupStart = reinterpret_cast<decltype(GroupStart)>(sym("ncclGroupStart"));
    GroupEnd = reinterpret_cast<decltype(GroupEnd)>(sym("ncclGroupEnd"));
    GetErrorString = reinterpret_cast<decltype(GetErrorString)>(sym("ncclGetErrorString"));
    if (!ok) { handle = nullptr; }
    return ok;
  }
};
extern Nccl g_nccl;

#define NCCL_TRY(x)                                                                                          \
  do {                                                                                                       \
    int r__ = (x);                                                                                           \
    if (r__ != 0) return fail(B2P_E_CUDA, "%s: %s", #x, g_nccl.GetErrorString ? g_nccl.GetErrorString(r__) : "NCCL error"); \
  } while (0)

// ncclGroupStart, body() (which enqueues collectives and returns a status), then ncclGroupEnd on every path: NCCL's
// group depth is per thread, so a group left open by a failed enqueue would defer every later collective of the
// thread.  Returns the first error.
template <class Body>
int nccl_group(Body&& body) {
  NCCL_TRY(g_nccl.GroupStart());
  const int rc = body(), end = g_nccl.GroupEnd();
  if (!rc && end) return fail(B2P_E_CUDA, "ncclGroupEnd: %s", g_nccl.GetErrorString(end));
  return rc;
}

// A device allocation that grows on demand and is freed with its owner (the context).
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(DevBuf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() {
    if (p) cudaFree(p);
  }
  int ensure(size_t bytes) {
    if (bytes <= cap) return B2P_OK;
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
    size_t want = bytes + bytes / 8 + 256;
    cudaError_t e = cudaMalloc(&p, want);
    if (e != cudaSuccess) {
      e = cudaMalloc(&p, bytes);
      want = bytes;
    }
    if (e != cudaSuccess) {
      cudaGetLastError();
      return fail(B2P_E_NOMEM, "cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e));
    }
    cap = want;
    return B2P_OK;
  }
  template <class T>
  T* as() const { return reinterpret_cast<T*>(p); }
};

constexpr int kStatusSlots = 32;      // range calls that may be outstanding between two b2p_sync
constexpr int kStageSlots = 11;       // device buffers of one host call, at most: b2p_range_histogram_fold's

// group -> member-series CSR of one gid[] assignment (b2p_group_index_create_dev), reusable across calls
struct b2p_group_index {
  uint32_t n_series = 0, n_groups = 0;
  uint32_t max_members = 0;      // size of the largest group
  uint32_t* gid = nullptr;       // [n_series] device copy
  uint32_t* goff = nullptr;      // [n_groups + 1]
  uint32_t* members = nullptr;   // [n_series] series ids ordered by (group, series id)
  std::vector<uint32_t> goff_host;  // host copy of goff (topk's chunk table)
};

// Device scratch is held in DevBuf members: it lives as long as the context and is freed when b2p_destroy deletes it.
struct b2p_ctx {
  int device = 0;
  int num_sms = 132;
  cudaStream_t own_stream = nullptr, stream = nullptr;
  // Device-side status.  Every range call owns one slot of d_ring until b2p_sync has read it back, so any number
  // (<= kStatusSlots, then the library synchronises by itself) of *_dev range calls may be outstanding; the verdict
  // of the series-id scan (K0) is sticky in d_k0 until the next b2p_sync.
  b2p::Status* d_ring = nullptr;  // [kStatusSlots]
  b2p::Status* h_ring = nullptr;  // pinned mirror
  b2p::Status* d_k0 = nullptr;
  b2p::Status* h_k0 = nullptr;    // pinned
  int next_slot = 0;
  // The tiers a range call starts with: the thread tier (K2T), or the first tier (K2L) in `lean_mode` (0 plain, 1 with
  // reset bit words; 2: the adaptive back-off skips it), and then the warp-per-series and slow tiers.
  struct Tiers {
    bool thread_tier = false;
    bool first_tier = false;
    int lean_mode = 0;
  };
  // The record of an admitted range call, until b2p_sync (or the host pipeline) has read its Status: enough to take its
  // verdict and to run it again.
  struct Pending {
    enum Kind {
      kPlain,
      kFused,   // by-label partials were added in place: only the slow kernel may be repeated
      kMerged,  // ... and already all-reduced (or tiled): nothing can be repeated, an arena overflow is an error
    };
    int slot;
    int fn;
    b2p::RangeArgs args;  // as admitted (use_w_list = 0)
    Tiers tiers;
    uint32_t n_series;
    Kind kind;
  };
  std::vector<Pending> pending;
  DevBuf slow_list, w_list, b_list, arena_ts, arena_val, win_scratch;
  // multi-GPU (one process per GPU): communicator of the by-label all-reduce, its stream and join event.  Invariant:
  // comm == nullptr => comm_ranks == 1 && comm_rank == 0, so without a communicator a context is rank 0 of one.
  Nccl::comm_t comm = nullptr;
  int comm_ranks = 1, comm_rank = 0;
  long long comm_headstart_cycles = 60000;  // ~30 us at 1.98 GHz, the H100's top SM clock (B2P_COMM_HEADSTART_US overrides)
  // SMs the fused tier leaves to the tile all-reduce (B2P_COMM_RESERVE_SMS).  Off: SMs left free do not make the
  // all-reduce of a tile run beside the next tile's kernel, the step only loses them (DESIGN.md section 7)
  int comm_reserve_sms = 0;
  int comm_reserve_now = 0;                 // ... in effect for the launch being issued
  cudaStream_t s_comm = nullptr;
  cudaEvent_t ev_comm_in = nullptr, ev_comm_done = nullptr, ev_comm_go = nullptr;
  DevBuf m_tmp0, m_tmp1;             // scratch of the variance merge
  DevBuf w_skip, b_skip, slow_skip;  // fused by-label partials: steps already added, parallel to the work lists
  bool fused_pending = false;        // a fused call is outstanding: its work lists must survive until b2p_sync
  // K2T (thread per series) in front of K2 for rate/increase/delta.  Slower than K2 on the benchmark shape, so it
  // is opt-in: B2P_ENABLE_THREAD_TIER=1.
  bool thread_tier = false;
  // K2L, the lean warp-per-series tier in front of K2 (default on; B2P_DISABLE_LEAN_TIER=1 turns it off)
  bool lean_tier = true;
  // adaptive tiering: when K2L handed more than half of the series of a call to K2 (e.g. every counter has resets),
  // the next calls skip it for a while; the verdict is taken wherever the status block is read back
  bool lean_force_flags = false;  // B2P_LEAN_FORCE_FLAGS=1: rate / increase always take the bit-word variant (tests)
  bool lean_adaptive = true;    // B2P_LEAN_ADAPTIVE=0 switches the back-off off (tests that pin the tier)
  // per range function: 0 = plain K2L; 1 = K2L with reset bit words (rate / increase after a call that handed most
  // series on); 2 = skip K2L.  `lean_backoff` counts the calls a non-zero mode still lasts.
  int lean_mode[B2P_FN__COUNT] = {};
  int lean_backoff[B2P_FN__COUNT] = {};
  // first-tier variant for equally spaced samples (rate / increase / delta): -1 = cadence_probe_kernel decides per call
  // on the device, 0 / 1 = forced (B2P_UNIFORM)
  int uniform_mode = -1;
  size_t arena_rows = 0;
  size_t arena_rows_wanted = 0;  // B2P_ARENA_ROWS: initial size of the slow-path arena (default kArenaDefaultRows)
  cudaEvent_t ev[5][2] = {};  // 0 K0, 1 range tiers, 2 slow kernel, 3 by-label aggregate, 4 all-reduce (last tile)
  bool ev_used[5] = {false, false, false, false, false};
  long long launches = 0;
  long long last_slow = 0;
  long long last_w = 0;
  // host-API staging: buffer i holds the i-th device copy a synchronous host call hands out (struct Staging)
  DevBuf stage[kStageSlots];
  // host-API pipeline (double-buffered staging, separate copy streams)
  bool pipe_ready = false;
  cudaStream_t s_h2d = nullptr, s_d2h = nullptr;
  cudaEvent_t ev_h2d[2] = {}, ev_comp[2] = {}, ev_d2h[2] = {};
  DevBuf p_ts[2], p_val[2], p_sid[2], p_off[2], p_out[2], p_valid[2], p_status;
  DevBuf p_t0[2], p_cad[2];  // per-series (first timestamp, cadence) of a chunk whose timestamp column stays on the host
  // b2p_range_eval: scan every chunk on the host (worker threads, ahead of the copies) and, where all of its series are
  // equally spaced, send (offsets, t0, cadence) instead of the timestamp and id columns (B2P_HOST_TS_SCAN=0: never)
  bool host_ts_scan = true;
  long long last_h2d_bytes = 0;
  // uniform histogram layout -> fold index (b2p_histogram_quantile_dev)
  DevBuf hq_off, hq_series, hq_les;
  // [n_series x T] range results of a by-label sum that cannot run fused (b2p_range_group_sum_indexed_dev)
  DevBuf rg_out, rg_valid;
  // group aggregate scratch
  DevBuf g_keys_in, g_keys_out, g_vals_in, g_vals_out, g_goff, g_tmp;
  // column reduce scratch
  DevBuf c_psum, c_pcnt;
  // set operators: the key -> member-row CSR of each side and the per-key validity mask
  DevBuf s_goff[2], s_members[2], s_mask;
  // scalar(): the reduction's verdict (struct ScalarState), read by the write pass on the device
  DevBuf sc_state;
  // absent(): the OR over rows of each validity word of the child's grid (b2p_absent.cuh; bound in absent_run)
  DevBuf ab_acc;
  // topk / bottomk: chunk and merge tables, candidate lists, selection state (b2p_topk.cuh; bound in topk_run)
  DevBuf t_table, t_cand, t_state;
  // sharded topk (b2p_aggregation.cu, shard_*): the merge table over the ranks' blocks, the group sizes all-reduced by
  // b2p_topk_allgather_dev, its candidate block, the gathered blocks and the selection state of one batch
  DevBuf x_table, x_size, x_send, x_recv, x_state;
  // bytes of blocks and state per batch of the sharded topk, quantile and count_values (B2P_TOPK_EXCHANGE_BYTES; the
  // sharded sort's exchange is its answer, N x 8 (F + 1) B on every rank, and is not cut into batches)
  size_t topk_exchange_cap = size_t(128) << 20;
  long long last_exchange_bytes = 0;  // bytes of this rank's blocks in the last sharded topk, quantile, count_values or sort
  long long last_group_keys_bytes = 0;  // bytes of this rank's block in the last group-label agreement
  // quantile: chunk table, state and histograms of the groups of several chunks (b2p_quantile.cuh; bound in quantile_run)
  DevBuf q_table, q_state, q_hist;
  // sharded quantile (b2p_aggregation.cu, quantile_shard_*): this rank's chunk table of a batch, the batch's selection
  // state (kept from pass to pass) and the count of cells left after an advance; the composed call's block is x_send
  DevBuf qx_table, qx_state, qx_live;
  // count_values: key and sorted-key buffers, ranks and starts, segment tables, member groups, CUB's temp (bound in
  // count_values_run)
  DevBuf v_keys, v_alt, v_rank, v_seg, v_group, v_tmp;
  // sharded count_values (b2p_aggregation.cu, cv_shard_*): the merge's counts and their sort buffer; its keys, runs,
  // segment table and CUB's temp are K12's v_keys / v_alt / v_rank / v_seg / v_tmp, its tables x_table, its block
  // x_send, the gathered blocks x_recv and the heights x_size
  DevBuf vx_cnt, vx_alt;
  // subquery: the sample rows of one batch of child rows (ts, val, offsets) and CUB's temp (bound in subquery_run)
  DevBuf sq_ts, sq_val, sq_off, sq_tmp;
  // multi-field range call: the value columns with K16's NaN union applied, and the validity bitmaps of fields 1.. before
  // K18's conjunction (bound in b2p_range_eval_fields_dev)
  DevBuf fd_val, fd_valid;
  DevBuf fd_null;  // one NULL-slot flag per field (null_slots_kernel)
  // sort / sort_desc: row offsets, keys (double-buffered), the alternate cell buffer and CUB's temp (bound in sort_run)
  DevBuf so_off, so_keys, so_cells, so_tmp;
  // sharded sort (b2p_sort.cu, shard_*): the row-id flag and K14's device count of a pack, and the merge's two run
  // buffers (ping-pong between rounds); its pair table is x_table, the gathered blocks x_recv and the counts x_size
  DevBuf sx_flag, sx_run[2];
  // resident CTAs per SM of each persistent kernel instantiation and dynamic shared-memory size (persistent_grid)
  std::map<std::pair<const void*, size_t>, int> blocks_per_sm;
};

struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    cudaGetDevice(&prev);
    if (prev != dev) cudaSetDevice(dev);
  }
  ~DeviceGuard() {
    int cur = -1;
    cudaGetDevice(&cur);
    if (prev >= 0 && cur != prev) cudaSetDevice(prev);
  }
};

// The per-rank table [n_ranks x count] of NCCL `type` in x_size: fill(mine) enqueues this rank's slot, the slots are
// all-gathered in place (with a communicator) and the table is copied to `host`.  Synchronises the stream.
template <class Fill>
int rank_table(b2p_ctx* c, size_t count, int type, void* host, Fill&& fill) {
  const size_t bytes = count * Nccl::bytes(type), table = (size_t)c->comm_ranks * bytes;
  if (int rc = c->x_size.ensure(table)) return rc;
  char* mine = c->x_size.as<char>() + (size_t)c->comm_rank * bytes;
  if (int rc = fill(mine)) return rc;
  if (c->comm) NCCL_TRY(g_nccl.AllGather(mine, c->x_size.p, count, type, c->comm, c->stream));
  CU(cudaMemcpyAsync(host, c->x_size.p, table, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  return B2P_OK;
}

// b2p_context.cu: one group of two in-place all-reduces on `s`: n partials of NCCL `type` by `op`, and their n u32
// counts added
int allreduce_with_counts(b2p_ctx* c, void* val, int type, int op, uint32_t* cnt, uint64_t n, cudaStream_t s);
// b2p_context.cu: the blocks of `buf`, back to back in rank order (block r: sizes[r] entries of `entry_bytes`), this
// rank's in place: with a communicator, one ncclBroadcast of NCCL `type` per rank with entries, in one group.
int gather_blocks(b2p_ctx* c, void* buf, const uint64_t* sizes, size_t entry_bytes, int type);

// the CUDA events around a stage's kernels, on `s` (default: the context's stream)
inline void stage_begin(b2p_ctx* c, int stage, cudaStream_t s = nullptr) {
  cudaEventRecord(c->ev[stage][0], s ? s : c->stream);
}
inline void stage_end(b2p_ctx* c, int stage, cudaStream_t s = nullptr) {
  cudaEventRecord(c->ev[stage][1], s ? s : c->stream);
  c->ev_used[stage] = true;
}

// CTAs for `units` work units, `per_block` per CTA, at most `per_sm` CTAs per SM (grid-stride beyond)
inline unsigned capped_grid(const b2p_ctx* c, uint64_t units, uint64_t per_block, uint64_t per_sm) {
  const uint64_t blocks = (units + per_block - 1) / per_block, cap = (uint64_t)c->num_sms * per_sm;
  return (unsigned)(blocks < cap ? blocks : cap);
}

constexpr uint64_t kAllResident = ~0ull;  // persistent_grid units: every CTA that stays resident

// Grid of a persistent kernel over `units` warp units, `warps` per CTA: at most the CTAs that stay resident.  The
// occupancy is queried once per context, kernel instantiation and dynamic shared-memory size.  The kernel's dynamic
// shared-memory limit is only ever raised, so a kernel launched with several sizes (topk's) stays launchable at each.
template <class Kern>
int persistent_grid(b2p_ctx* c, Kern* kern, size_t smem, int warps, uint64_t units, unsigned* grid) {
  int& per_sm = c->blocks_per_sm[{reinterpret_cast<const void*>(kern), smem}];
  if (per_sm == 0) {
    cudaFuncAttributes fa;
    int nb = 0;
    CU(cudaFuncGetAttributes(&fa, kern));
    if ((size_t)fa.maxDynamicSharedSizeBytes < smem)
      CU(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kern, warps * 32, smem));
    per_sm = nb > 0 ? nb : 1;
  }
  const uint64_t need = units / warps + (units % warps != 0), cap = (uint64_t)c->num_sms * per_sm;
  *grid = (unsigned)(need < cap ? need : cap);
  return B2P_OK;
}

// f(std::integral_constant<int, ID>{}) for the run-time id `id` in [0, COUNT): one instantiation of f per id
template <int COUNT, int ID = 0, class F>
int with_id(int id, const char* what, F&& f) {
  if constexpr (ID == COUNT) {
    return fail(B2P_E_INVALID, "unknown %s %d", what, id);
  } else {
    return id == ID ? f(std::integral_constant<int, ID>{}) : with_id<COUNT, ID + 1>(id, what, f);
  }
}
// range function id -> compile-time FN
template <class F>
int with_fn(int fn, F&& f) { return with_id<B2P_FN__COUNT>(fn, "fn_id", f); }

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// The eval-step count T of a range grid, after checking the grid (and n_series x T) is one the device can hold.
int check_grid(const b2p_range_params* p, uint32_t n_series, int64_t* T_out);

// Device copies of one synchronous host call's columns, in the context's staging buffers: the i-th buffer handed out
// is c->stage[i].  Inputs are copied to the device as they are handed out; the results noted by out() / copy_back()
// go back to the host, in that order, in download().  The first failure sticks in `rc` (later calls hand out NULL).
// An absent (NULL) host column is handed out as NULL and queues nothing, so the device form's argument check rejects
// it.  A host call reads: stage the inputs, stage the outputs, end() with the device form.
struct Staging {
  b2p_ctx* c;
  int next = 0, rc = B2P_OK;
  struct Back { void* host; const void* dev; size_t bytes; };
  std::vector<Back> back;

  void cuda(cudaError_t e, const char* what) {  // a failed CUDA call becomes the sticky error
    if (e != cudaSuccess && !rc) rc = fail(B2P_E_CUDA, "%s: %s", what, cudaGetErrorString(e));
  }
  void* buf(size_t bytes) {  // (16 bytes more: never NULL, even for an empty column)
    if (!rc && next == kStageSlots) rc = fail(B2P_E_INVALID, "host call stages more than %d buffers", kStageSlots);
    if (!rc) rc = c->stage[next].ensure(bytes + 16);
    return rc ? nullptr : c->stage[next++].p;
  }
  // device copy of a host column; NULL for an absent one
  template <class T>
  T* in(const T* host, size_t bytes) {
    if (!host) return nullptr;
    void* d = buf(bytes);
    if (d && bytes) cuda(cudaMemcpyAsync(d, host, bytes, cudaMemcpyHostToDevice, c->stream), "host-to-device copy");
    return static_cast<T*>(d);
  }
  // `dev` as the result buffer of `host` (copied there by download()); NULL for an absent one
  template <class T>
  T* copy_back(T* host, T* dev, size_t bytes) {
    if (!host) return nullptr;
    if (!rc) back.push_back(Back{host, dev, bytes});
    return dev;
  }
  // a result buffer, copied to `host` by download(); NULL for an absent one
  template <class T>
  T* out(T* host, size_t bytes) {
    return host ? copy_back(host, static_cast<T*>(buf(bytes)), bytes) : nullptr;
  }
  // n columns of `bytes` each in one buffer (each at a 16-byte aligned offset): device copies of the host columns, or
  // result columns copied back to them; dev[i] is NULL for an absent host column
  template <class T>
  void in_cols(const T* const* hosts, int n, size_t bytes, const T** dev) {
    const size_t stride = (bytes + 15) & ~(size_t)15;
    char* d = static_cast<char*>(buf(stride * (size_t)n));
    for (int i = 0; i < n; ++i) {
      dev[i] = d && hosts[i] ? reinterpret_cast<const T*>(d + stride * (size_t)i) : nullptr;
      if (dev[i] && bytes)
        cuda(cudaMemcpyAsync(const_cast<T*>(dev[i]), hosts[i], bytes, cudaMemcpyHostToDevice, c->stream), "host-to-device copy");
    }
  }
  template <class T>
  void out_cols(T* const* hosts, int n, size_t bytes, T** dev) {
    const size_t stride = (bytes + 15) & ~(size_t)15;
    char* d = static_cast<char*>(buf(stride * (size_t)n));
    for (int i = 0; i < n; ++i)
      dev[i] = d && hosts[i] ? copy_back(hosts[i], reinterpret_cast<T*>(d + stride * (size_t)i), bytes) : nullptr;
  }
  int download() {  // the results noted since the last download()
    for (size_t i = 0; !rc && i < back.size(); ++i)
      if (back[i].bytes)
        cuda(cudaMemcpyAsync(back[i].host, back[i].dev, back[i].bytes, cudaMemcpyDeviceToHost, c->stream),
             "device-to-host copy");
    back.clear();
    return rc;
  }
  int finish() {  // download() and wait for it
    if (!download()) cuda(cudaStreamSynchronize(c->stream), "cudaStreamSynchronize");
    return rc;
  }
  // The end of a host call: `dev()` (the device form, and whatever has to follow it before the results are read),
  // skipped once staging has failed so that its error stands; then finish(), or only download() when `wait` is false
  // and the caller synchronises by itself.  Returns the first error.
  template <class Dev>
  int end(Dev&& dev, bool wait = true) {
    if (!rc) rc = dev();
    return wait ? finish() : download();
  }
};

// The series columns of a host call: ts and val, then the offsets, or the id column and K0 (ids rebased by sid_base)
struct SeriesIn {
  const int64_t* ts;
  const double* val;
  uint64_t* offsets;
};
SeriesIn stage_series(Staging& s, const int64_t* ts, const double* val, const uint32_t* sid, uint32_t sid_base,
                      const uint64_t* offsets_host, uint64_t n_rows, uint32_t n_series);

// ---- internals of one file that another one calls -----------------------------------------------------------------
// b2p_range.cu: uploads the reciprocal table of the thread tier (b2p_kernel_t.cuh) to this module's constant memory
int upload_rcp_table();
// b2p_range.cu: K13's per-row count of the valid cells of a [rows x T] grid (bits past T ignored), then CUB's exclusive
// scan in place: offsets[r] = the valid cells of the rows before r, offsets[rows] = the total.  `tmp` grows to CUB's temp.
int scan_valid_cells(b2p_ctx* c, const uint32_t* valid, uint64_t T, uint32_t rows, unsigned long long* offsets,
                     DevBuf& tmp);
// the grid of a warp-per-row kernel over the rows of such a grid (256 threads per CTA)
inline unsigned cell_rows_grid(const b2p_ctx* c, uint32_t rows) {
  const unsigned g = capped_grid(c, (uint64_t)rows * 32, 256, 8);
  return g ? g : 1u;
}
// b2p_group.cu: group -> member series CSR: stable radix sort of (gid, series index), then lower bounds per group
int build_group_csr(b2p_ctx* c, const uint32_t* gid, uint32_t n_series, uint32_t n_groups, uint32_t* goff,
                    uint32_t* members);
// b2p_group.cu: the by-label aggregate over a CSR; accumulate = 1 (SUM / COUNT partials only): out_val / out_cnt are
// added to instead of overwritten
int group_aggregate_csr(b2p_ctx* c, int32_t agg, const double* vals, const uint32_t* valid_words, const uint32_t* goff,
                        const uint32_t* members, uint32_t n_groups, uint64_t T, double* out_val, uint32_t* out_cnt,
                        int accumulate, double* out_mean = nullptr, bool i64 = false);
