// b2p_range.cu — range-query entry points of the C ABI: the range tiers (first tier, warp per series, long windows,
// exact slow path) and their completion in b2p_sync, series offsets, range_eval (device columns, and host columns
// through the chunked copy pipeline and the host timestamp scan), prom_* UDF calls, the instant selector, the fused and
// all-reduced sum by, subqueries and the synthetic data generator.
#include <algorithm>
#include <atomic>
#include <cstring>
#include <memory>
#include <string>
#include <thread>
#include <vector>

#include <cub/device/device_scan.cuh>

#include "b2p_runtime.cuh"
#include "b2p_subquery.cuh"
#include "b2p_kernel_t.cuh"
#include "b2p_kernel_lean.cuh"
#include "b2p_kernels.cuh"
#include "b2p_fields.cuh"

using namespace b2p;

namespace {

constexpr int kRing = 256;
constexpr int kBigRing = 1024;        // long-window instantiation of the warp-per-series kernel (one CTA per SM)
constexpr int kSlowCtas = 132;        // slow-path grid (4 warps per CTA): one CTA per SM of an H100
constexpr int kSlowWarps = kSlowCtas * 4;
constexpr size_t kArenaDefaultRows = 1u << 21;  // 32 MB: regions of 3 971 rows for the 528 slow-path warps

// rate / increase / delta: the functions of the thread tier and of the fused by-label first tier
constexpr bool rate_like(int fn) { return fn == B2P_FN_RATE || fn == B2P_FN_INCREASE || fn == B2P_FN_DELTA; }

// 32-bit relative timestamps when the whole query span (plus one lookback) fits 31 bits of ms.
bool fits_ts32(const RangeArgs& a) {
  const double span = (double)a.end - (double)a.start + (double)a.range;
  return span >= 0 && span < 2147483000.0 && a.interval < 2147483000ll && a.range < 2147483000ll;
}

// Adaptive tiering verdict of a finished range call that started with K2L in `mode`: more than half of the series
// handed on -> the next 32 calls of this function use the next mode (plain -> bit words for rate / increase -> skip).
void lean_verdict(b2p_ctx* c, int fn, int mode, uint64_t handed, uint64_t n_series) {
  if (!c->lean_adaptive || handed * 2 <= n_series) return;
  const bool counter = (fn == B2P_FN_RATE || fn == B2P_FN_INCREASE);
  c->lean_mode[fn] = (mode == 0 && counter) ? 1 : 2;
  c->lean_backoff[fn] = 32;
}

bool lean_supported(int fn) {
  bool supported = false;
  if (fn >= 0 && fn < B2P_FN__COUNT)
    with_fn(fn, [&](auto k) { supported = LeanTraits<decltype(k)::value>::kSupported; return B2P_OK; });
  return supported;
}

// Lean first tier (K2L): rate / increase / delta in the 32-bit time domain.  The gates are what the kernel
// relies on: exact reciprocal division by range/1000, range >= interval (steps evaluated before the end of a
// series are below the trimmed end), start >= 0 (truncating division == floor in the end trim), and window
// ends of the 31 steps past the grid still below the 0xFFFFFFFF end sentinel.
bool lean_ok(const b2p_ctx* c, int fn, const RangeArgs& a) {
  if (!c->lean_tier || !lean_supported(fn)) return false;
  if (!fits_ts32(a) || a.range < a.interval || a.start < 0) return false;
  if (fn == B2P_FN_RATE && a.rcp_rs == 0.0) return false;
  return (double)a.rel_max + 64.0 * (double)a.interval < 4294967295.0;
}

// The tiers a range call of `fn` over the geometry `a` starts with (changes no state).  Tier 1 (rate / increase /
// delta, 32-bit time domain) is the thread tier (opt-in) or the lean warp-per-series kernel; what it declines goes to
// tier 2 (warp per series) through w_list, long windows from there to the 1024-sample instantiation through b_list,
// and what that declines to the exact slow kernel.  While a back-off lasts the first tier runs in the mode the last
// verdict chose (mode 2: not at all).
b2p_ctx::Tiers choose_tiers(const b2p_ctx* c, int fn, const RangeArgs& a) {
  b2p_ctx::Tiers t;
  t.thread_tier = c->thread_tier && fits_ts32(a) && rate_like(fn);
  if (t.thread_tier || !lean_ok(c, fn, a)) return t;
  if (c->lean_backoff[fn] > 0) t.lean_mode = c->lean_mode[fn];
  t.first_tier = t.lean_mode != 2;
  if (t.lean_mode == 0 && c->lean_force_flags) t.lean_mode = 1;
  return t;
}

// One launch of a range kernel on the context's stream; a zero grid launches nothing.
template <class Kern>
int launch_kernel(b2p_ctx* c, Kern* kern, unsigned grid, unsigned threads, size_t smem, const RangeArgs& a) {
  if (grid == 0) return B2P_OK;
  kern<<<grid, threads, smem, c->stream>>>(a);
  c->launches++;
  CU(cudaGetLastError());
  return B2P_OK;
}

// The warp-per-series tier (K2): RING = kRing over the series (w_list after a first tier), or its long-window
// instantiation RING = kBigRing (32-bit time domain only), one CTA per SM, over RangeArgs::b_list, whose length is
// known on the device only.
template <int FN, int RING, bool TS32>
int launch_warp_tier(b2p_ctx* c, RangeArgs a) {
  constexpr bool kBig = RING == kBigRing;
  static_assert(!kBig || TS32, "the long-window instantiation is 32-bit only");
  constexpr size_t smem = (size_t)kWarpsPerCta * (2 * RING * (8 + (TS32 ? 4 : 8)) + RING / 8) + kRcpTable * 8;
  auto kern = range_fast_kernel<FN, RING, TS32>;
  if (kBig) a.use_w_list = 2;
  unsigned grid = 0;
  if (int rc = persistent_grid(c, kern, smem, kWarpsPerCta, kBig ? kAllResident : a.n_series, &grid)) return rc;
  return launch_kernel(c, kern, grid, kWarpsPerCta * 32, smem, a);
}

// Functions whose first tier has a uniform-cadence variant: the probe (or B2P_UNIFORM) writes Status::uniform, then
// both variants are launched and the one the verdict does not name returns at once — no host round trip.
int cadence_verdict(b2p_ctx* c, const RangeArgs& a) {
  if (c->uniform_mode < 0) return launch_kernel(c, cadence_probe_kernel, 1, kProbeThreads, 0, a);
  CU(cudaMemsetAsync(&a.status->uniform, c->uniform_mode ? 1 : 0, sizeof(uint32_t), c->stream));
  return B2P_OK;
}

// One variant of the first tier (range_lean_kernel).  Plain: a persistent grid over the series.  GROUPED (the fused
// by-label SUM: rate / increase / delta walk the series group by group and add into gsum / gcnt): one CTA per SM that
// takes its groups from a counter, so the grid can be any size; while tiles are being all-reduced a few SMs are left
// to the collective's CTAs (they cannot be placed beside a resident 24-warp CTA).
template <int FN, bool FLAGS, bool GROUPED, bool UNI>
int launch_first_variant(b2p_ctx* c, const RangeArgs& a) {
  constexpr size_t smem = GROUPED ? lean_grouped_smem_bytes(UNI) : lean_smem_bytes(UNI);
  auto kern = range_lean_kernel<FN, FLAGS, GROUPED, UNI>;
  unsigned grid = 0;
  if (int rc = persistent_grid(c, kern, smem, kLeanWarps, GROUPED ? kAllResident : a.n_series, &grid)) return rc;
  if constexpr (GROUPED) {
    const unsigned need = (a.g_hi - a.g_lo + kLeanWarps - 1) / kLeanWarps;
    if (c->comm_reserve_now > 0 && grid > (unsigned)c->comm_reserve_now + 8u) grid -= (unsigned)c->comm_reserve_now;
    if (need < grid) grid = need;
  }
  return launch_kernel(c, kern, grid, kLeanWarps * 32, smem, a);
}

// Both uniform-cadence variants of the first tier where FN has them (cadence_verdict names one on the device), else
// the one variant.
template <int FN, bool GROUPED, bool FLAGS>
int launch_first_pair(b2p_ctx* c, const RangeArgs& a) {
  if constexpr (kLeanUniform<FN, FLAGS>) {
    int rc = cadence_verdict(c, a);
    if (!rc && c->uniform_mode != 0) rc = launch_first_variant<FN, FLAGS, GROUPED, true>(c, a);
    if (!rc && c->uniform_mode != 1) rc = launch_first_variant<FN, FLAGS, GROUPED, false>(c, a);
    return rc;
  } else {
    return launch_first_variant<FN, FLAGS, GROUPED, false>(c, a);
  }
}

// The first tier (K2L) of FN, plain or GROUPED.  `with_flags`: the variant whose ring carries the reset / change bit
// words (always for resets() / changes(); for rate / increase when the adaptive policy picked it; never for the other
// functions).
template <int FN, bool GROUPED>
int launch_first_tier(b2p_ctx* c, const RangeArgs& a, bool with_flags) {
  if constexpr (GROUPED ? !rate_like(FN) : !LeanTraits<FN>::kSupported) {
    return fail(B2P_E_INVALID, GROUPED ? "fn_id %d has no fused by-label tier" : "fn_id %d has no lean tier", FN);
  } else if constexpr (LeanTraits<FN>::kNeedsFlags) {
    return launch_first_pair<FN, GROUPED, true>(c, a);
  } else if constexpr (LeanTraits<FN>::kHasFlagsVariant) {
    return with_flags ? launch_first_pair<FN, GROUPED, true>(c, a) : launch_first_pair<FN, GROUPED, false>(c, a);
  } else {
    return launch_first_pair<FN, GROUPED, false>(c, a);
  }
}

template <int FN>
int launch_thread_tier(b2p_ctx* c, const RangeArgs& a) {
  if constexpr (!rate_like(FN)) {
    return fail(B2P_E_INVALID, "fn_id %d has no thread tier", FN);
  } else {  // at most the 1-warp CTAs whose rings fit in shared memory
    const unsigned grid = capped_grid(c, a.n_series, 32, 220 * 1024 / (kTRing * 32 * 12 + 512));
    return launch_kernel(c, range_thread_kernel<FN>, grid, 32, 0, a);
  }
}

int dispatch_slow(b2p_ctx* c, int fn, const RangeArgs& a) {
  return with_fn(fn, [&](auto k) { return launch_kernel(c, range_slow_kernel<decltype(k)::value>, kSlowCtas, 128, 0, a); });
}

// The window and time-domain fields of a range call over T steps (check_grid has accepted p); the first tier's gates
// (lean_ok) read them.
RangeArgs range_geometry(const b2p_range_params* p, int64_t T) {
  RangeArgs a{};
  a.start = p->start; a.end = p->end; a.interval = p->interval; a.range = p->range;
  a.T = T; a.Tw = (uint32_t)((T + 31) / 32);
  a.tb = p->start - p->range;
  if (fits_ts32(a)) a.rel_max = (uint32_t)(p->range + (T - 1) * p->interval + 1);
  // exact two-FMA division by range/1000 needs RN(1/b) and a significand that is not all ones
  const double rs = (double)p->range / 1000.0;
  uint64_t bits;
  memcpy(&bits, &rs, 8);
  const bool all_ones = (bits & 0x000fffffffffffffull) == 0x000fffffffffffffull;
  a.rcp_rs = (p->range > 0 && !all_ones) ? 1.0 / rs : 0.0;
  a.range_secs = rs;
  a.rcp_interval = 1.0 / (double)p->interval;
  a.start_mod = p->start >= 0 ? (uint32_t)(p->start % p->interval) : 0u;
  return a;
}

int ensure_slow_scratch(b2p_ctx* c, uint32_t n_series, int64_t T) {
  int rc;
  if ((rc = c->slow_list.ensure((size_t)(n_series ? n_series : 1) * 4))) return rc;
  if ((rc = c->w_list.ensure((size_t)(n_series ? n_series : 1) * 4))) return rc;
  if ((rc = c->b_list.ensure((size_t)(n_series ? n_series : 1) * 4))) return rc;
  if ((rc = c->win_scratch.ensure((size_t)kSlowWarps * (size_t)(T > 0 ? T : 1) * 8))) return rc;
  if (c->arena_rows == 0) {
    const size_t rows = c->arena_rows_wanted > kArenaDefaultRows ? c->arena_rows_wanted : kArenaDefaultRows;
    if ((rc = c->arena_ts.ensure(rows * 8))) return rc;
    if ((rc = c->arena_val.ensure(rows * 8))) return rc;
    c->arena_rows = rows;
  }
  return B2P_OK;
}

}  // namespace

int check_grid(const b2p_range_params* p, uint32_t n_series, int64_t* T_out) {
  if (!p) return fail(B2P_E_INVALID, "params is NULL");
  if (p->interval <= 0) return fail(B2P_E_INVALID, "interval must be > 0 (got %lld)", (long long)p->interval);
  if (p->range < 0) return fail(B2P_E_INVALID, "range must be >= 0");
  if (p->fn_id < 0 || p->fn_id >= B2P_FN__COUNT) return fail(B2P_E_INVALID, "unknown fn_id %d", p->fn_id);
  const int64_t T = b2p_num_steps(p->start, p->end, p->interval);
  if (T > (int64_t)0x7fffff00) return fail(B2P_E_TOO_LARGE, "%lld eval steps: trim [start,end] to the data extent first", (long long)T);
  if ((double)T * (double)n_series > 1.0e12) return fail(B2P_E_TOO_LARGE, "dense grid %lld x %u too large", (long long)T, n_series);
  *T_out = T;
  return B2P_OK;
}

// The thread tier's reciprocal table is a __constant__ of b2p_kernel_t.cuh, so it exists in this module only, where
// range_thread_kernel is launched; b2p_create fills it through this function.
int upload_rcp_table() {
  double tab[kRcpTable];
  tab[0] = 0.0;
  for (int i = 1; i < kRcpTable; ++i) tab[i] = 1.0 / (double)i;
  if (cudaMemcpyToSymbol(c_rcp_table, tab, sizeof tab) != cudaSuccess)
    return fail(B2P_E_CUDA, "constant table upload failed: %s", cudaGetErrorString(cudaGetLastError()));
  return B2P_OK;
}

extern "C" {

__global__ void comm_marker_kernel() {}
// a tiled call's counters before the next tile resets them: what b2p_last_*_series and the adaptive verdict read
__global__ void tile_counts_kernel(Status* st) {
  st->slow_tiles += st->slow_count;
  st->w_tiles += st->w_count;
}
// holds the compute stream back for a few microseconds so that the all-reduce released at the same instant on the
// communication stream has its CTAs placed before the persistent range kernel asks for every SM
__global__ void comm_headstart_kernel(long long cycles) {
  const long long t0 = clock64();
  while (clock64() - t0 < cycles) {}
}

// Launches every tier of a range call (its first tier or thread tier, warp-per-series kernel, long-window
// instantiation, exact slow kernel) on the context's stream.
static int launch_range_tiers(b2p_ctx* c, const b2p_ctx::Pending& pc, bool later_tile = false) {
  RangeArgs a = pc.args;
  int rc;
  if (!later_tile) {
    CU(cudaMemsetAsync(a.status, 0, sizeof(Status), c->stream));
  } else {  // a further tile of the same fused call: new work lists, same verdict (overflow / arena fields stay)
    tile_counts_kernel<<<1, 1, 0, c->stream>>>(a.status);
    c->launches++;
    CU(cudaGetLastError());
    CU(cudaMemsetAsync(&a.status->slow_count, 0, sizeof(uint32_t), c->stream));
    CU(cudaMemsetAsync(&a.status->w_count, 0, 3 * sizeof(uint32_t), c->stream));  // w_count, b_count, g_next
  }
  stage_begin(c, 1);
  if (pc.tiers.thread_tier || pc.tiers.first_tier) {
    rc = with_fn(pc.fn, [&](auto k) {
      constexpr int FN = decltype(k)::value;
      if (pc.tiers.thread_tier) return launch_thread_tier<FN>(c, a);
      const bool with_flags = pc.tiers.lean_mode == 1;
      return a.gsum ? launch_first_tier<FN, true>(c, a, with_flags) : launch_first_tier<FN, false>(c, a, with_flags);
    });
    if (rc) return rc;
    a.use_w_list = 1;
  }
  rc = with_fn(pc.fn, [&](auto k) {
    constexpr int FN = decltype(k)::value;
    const int r = fits_ts32(a) ? launch_warp_tier<FN, kRing, true>(c, a) : launch_warp_tier<FN, kRing, false>(c, a);
    return (r || !a.b_list) ? r : launch_warp_tier<FN, kBigRing, true>(c, a);
  });
  stage_end(c, 1);
  if (rc) return rc;
  stage_begin(c, 2);
  rc = dispatch_slow(c, pc.fn, a);
  stage_end(c, 2);
  return rc;
}

// The sticky verdict of the series-id scan (K0): read back (with whatever the stream has queued before it), cleared,
// and returned as an error.
static int take_k0(b2p_ctx* c) {
  CU(cudaMemcpyAsync(c->h_k0, c->d_k0, sizeof(Status), cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  if (const uint32_t k0 = c->h_k0->k0_errors) {
    CU(cudaMemsetAsync(c->d_k0, 0, sizeof(Status), c->stream));
    return k0_fail(k0);
  }
  return B2P_OK;
}

// The arena rows a call whose slow path ran out of arena needs to be redone (0: it fit).
static size_t redo_rows(const Status& st) { return st.arena_overflow ? (size_t)st.arena_needed + 1024 : 0; }

// The outcome of one range call from the Status of each of its `n` records (one; or one per chunk of a host call):
// the hand-off counters (summed over the records, and over the tiles of a tiled call) and the adaptive verdict, taken
// over all of them with the tiers of the last — unless `redo`: a redo is not a new call.  Returns the arena rows the
// largest record that ran out of arena needs (0: every one fit).
static size_t read_outcome(b2p_ctx* c, const b2p_ctx::Pending* recs, const Status* st, size_t n, bool redo) {
  size_t need = 0;
  long long slow = 0, handed = 0;
  uint64_t series = 0;
  for (size_t i = 0; i < n; ++i) {
    slow += (long long)st[i].slow_tiles + st[i].slow_count;
    handed += (long long)st[i].w_tiles + st[i].w_count;
    series += recs[i].n_series;
    need = std::max(need, redo_rows(st[i]));
  }
  if (!redo) {
    c->last_slow = slow;
    c->last_w = handed;
    const b2p_ctx::Pending& last = recs[n - 1];
    if (last.tiers.first_tier) lean_verdict(c, last.fn, last.tiers.lean_mode, (uint64_t)handed, series);
  }
  return need;
}

// Runs again the calls in `redo`, whose slow path ran out of arena, after the arena has grown to `need` rows, until
// every one fits.  They run one at a time, as they were admitted: they share the arena from offset 0.  A fused call
// repeats its slow kernel only, over its intact work list (a series that did not fit the arena added nothing; no
// other range call was admitted while it was outstanding); a merged call cannot be repeated.
static int redo_calls(b2p_ctx* c, std::vector<b2p_ctx::Pending> redo, size_t need) {
  for (int round = 0; round < 3 && !redo.empty(); ++round) {
    int rc;
    if ((rc = c->arena_ts.ensure(need * 8)) || (rc = c->arena_val.ensure(need * 8))) return rc;
    c->arena_rows = need;
    for (b2p_ctx::Pending& pc : redo) {
      if (pc.kind == b2p_ctx::Pending::kMerged)
        return fail(B2P_E_TOO_LARGE, "a series of %llu+ rows needs the exact slow path but does not fit its arena region; "
                    "the merged partials are incomplete — set B2P_ARENA_ROWS >= %zu and repeat the query",
                    (unsigned long long)(need / (size_t)kSlowWarps), need);
      pc.args.arena_ts = c->arena_ts.as<int64_t>();
      pc.args.arena_val = c->arena_val.as<double>();
      pc.args.arena_cap = need;
      if (pc.kind == b2p_ctx::Pending::kFused) {
        Status& patch = c->h_ring[pc.slot];
        patch.arena_overflow = 0; patch.arena_used = 0; patch.arena_needed = 0;
        CU(cudaMemcpyAsync(c->d_ring + pc.slot, c->h_ring + pc.slot, sizeof(Status), cudaMemcpyHostToDevice, c->stream));
        rc = dispatch_slow(c, pc.fn, pc.args);
      } else {
        rc = launch_range_tiers(c, pc);
      }
      if (rc) return rc;
      CU(cudaStreamSynchronize(c->stream));
    }
    CU(cudaMemcpyAsync(c->h_ring, c->d_ring, kStatusSlots * sizeof(Status), cudaMemcpyDeviceToHost, c->stream));
    CU(cudaStreamSynchronize(c->stream));
    std::vector<b2p_ctx::Pending> again;
    need = 0;
    for (const b2p_ctx::Pending& pc : redo)
      if (const size_t rows = read_outcome(c, &pc, &c->h_ring[pc.slot], 1, true)) {
        again.push_back(pc);
        need = std::max(need, rows);
      }
    redo.swap(again);
  }
  return redo.empty() ? B2P_OK : fail(B2P_E_NOMEM, "slow-path arena could not be sized");
}

int b2p_sync(b2p_ctx* c) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  DeviceGuard g(c->device);
  CU(cudaMemcpyAsync(c->h_ring, c->d_ring, kStatusSlots * sizeof(Status), cudaMemcpyDeviceToHost, c->stream));
  std::vector<b2p_ctx::Pending> calls;
  calls.swap(c->pending);
  c->fused_pending = false;
  if (int rc = take_k0(c)) return rc;
  // the outstanding range calls, oldest first; those whose slow path ran out of arena are redone
  std::vector<b2p_ctx::Pending> redo;
  size_t need = 0;
  for (const b2p_ctx::Pending& pc : calls)
    if (const size_t rows = read_outcome(c, &pc, &c->h_ring[pc.slot], 1, false)) {
      redo.push_back(pc);
      need = std::max(need, rows);
    }
  return redo_calls(c, std::move(redo), need);
}

/* ---- device-pointer API ---------------------------------------------------------------------- */

static int series_offsets_impl(b2p_ctx* c, const uint32_t* sid, uint64_t n_rows, uint32_t n_series, uint32_t sid_base,
                               uint64_t* offsets);

int b2p_series_offsets_dev(b2p_ctx* c, const uint32_t* sid, uint64_t n_rows, uint32_t n_series, uint64_t* offsets) {
  return series_offsets_impl(c, sid, n_rows, n_series, 0u, offsets);
}

static int series_offsets_impl(b2p_ctx* c, const uint32_t* sid, uint64_t n_rows, uint32_t n_series, uint32_t sid_base,
                               uint64_t* offsets) {
  if (!c || !offsets || (!sid && n_rows)) return fail(B2P_E_INVALID, "NULL argument");
  if (!aligned16(sid)) return fail(B2P_E_INVALID, "sid must be 16-byte aligned");
  DeviceGuard g(c->device);
  unsigned blocks = capped_grid(c, n_rows / 16, 256, 16);
  if (blocks == 0) blocks = 1;
  stage_begin(c, 0);
  series_offsets_kernel<<<blocks, 256, 0, c->stream>>>(sid, n_rows, n_series, sid_base, offsets, c->d_k0);
  series_offsets_clear_kernel<<<capped_grid(c, (uint64_t)n_series + 1, 256, 1), 256, 0, c->stream>>>(offsets, n_series,
                                                                                                    c->d_k0);
  c->launches += 2;
  stage_end(c, 0);
  CU(cudaGetLastError());
  return B2P_OK;
}

// Target of a fused by-label SUM / COUNT (b2p_range_group_sum*_dev): groups [g_lo, g_hi) of an index.
struct GroupTarget {
  const b2p_group_index* idx;
  uint32_t g_lo, g_hi;
  double* gsum;
  uint32_t* gcnt;
  // > 0: the group range is processed in this many tiles and every tile's rows of gsum / gcnt are all-reduced over
  // the context's communicator as soon as the tile is complete, on the (high-priority) communication stream, while
  // the next tile computes
  int allreduce_tiles;
};

// Can this range call add its results straight into by-label partials?  (the first tier runs for the function and
// the query shape, not switched off by the adaptive policy; groups balanced enough for group-exclusive warps)
static bool fused_group_ok(b2p_ctx* c, const b2p_range_params* p, int64_t T, const b2p_group_index* idx) {
  if (!rate_like(p->fn_id)) return false;
  if (T > 32 * (int64_t)kLeanFullWords) return false;  // per-warp word counters of the first tier
  if (!choose_tiers(c, p->fn_id, range_geometry(p, T)).first_tier) return false;
  // a group is walked by ONE warp: the largest group may not exceed a few times a warp's fair share
  const uint64_t warps = (uint64_t)c->num_sms * B2P_LEAN_MIN_BLOCKS * kLeanWarps;
  const uint64_t share = idx->n_series / warps + 1;
  return (uint64_t)idx->max_members <= 8 * share + 64;
}

// A fused call whose partials are all-reduced: its group range in `n_tiles` tiles, each tile's rows of gsum / gcnt
// all-reduced over the context's communicator as soon as the tile is complete, on the (high-priority) communication
// stream, while the next tile computes.
static int launch_allreduce_tiles(b2p_ctx* c, const b2p_ctx::Pending& pc, uint32_t n_tiles) {
  const RangeArgs& a = pc.args;
  const uint64_t span = (uint64_t)a.g_hi - a.g_lo;
  c->comm_reserve_now = (c->comm && n_tiles > 1) ? c->comm_reserve_sms : 0;
  bool launched = false;  // (with more tiles than groups the first tiles are empty: the first one run resets Status)
  for (uint32_t t = 0; t < n_tiles; ++t) {
    b2p_ctx::Pending tile = pc;
    tile.args.g_lo = a.g_lo + (uint32_t)(span * t / n_tiles);
    tile.args.g_hi = a.g_lo + (uint32_t)(span * (t + 1) / n_tiles);
    if (tile.args.g_hi == tile.args.g_lo) continue;
    if (int rc = launch_range_tiers(c, tile, launched)) return rc;
    launched = true;
    if (c->comm) {
      const size_t off = (size_t)tile.args.g_lo * (size_t)a.T, cnt_n = (size_t)(tile.args.g_hi - tile.args.g_lo) * (size_t)a.T;
      CU(cudaEventRecord(c->ev_comm_in, c->stream));
      CU(cudaStreamWaitEvent(c->s_comm, c->ev_comm_in, 0));
      // The next tile's kernels are released by a marker that sits directly IN FRONT of the all-reduce on the
      // communication stream: when they become runnable the (few) NCCL CTAs are already next in line on the
      // high-priority stream and get their SMs first; the persistent first-tier kernel fills what is left and its
      // dynamic group counter keeps late CTAs from becoming a tail.
      comm_marker_kernel<<<1, 32, 0, c->s_comm>>>();
      CU(cudaEventRecord(c->ev_comm_go, c->s_comm));
      CU(cudaStreamWaitEvent(c->stream, c->ev_comm_go, 0));
      if (c->comm_headstart_cycles > 0) comm_headstart_kernel<<<1, 32, 0, c->stream>>>(c->comm_headstart_cycles);
      stage_begin(c, 4, c->s_comm);
      if (int rc = allreduce_with_counts(c, a.gsum + off, Nccl::kFloat64, Nccl::kSum, a.gcnt + off, cnt_n, c->s_comm))
        return rc;
      stage_end(c, 4, c->s_comm);
    }
  }
  c->comm_reserve_now = 0;
  if (c->comm) {  // everything after this call on the context's stream sees the merged partials
    CU(cudaEventRecord(c->ev_comm_done, c->s_comm));
    CU(cudaStreamWaitEvent(c->stream, c->ev_comm_done, 0));
  }
  return B2P_OK;
}

static int range_call(b2p_ctx* c, const b2p_range_params* p, const int64_t* ts, const double* val,
                      const uint64_t* offsets, uint64_t n_rows, uint32_t n_series, double* out, uint32_t* valid_words,
                      const GroupTarget* gt);

int b2p_range_eval_dev(b2p_ctx* c, const b2p_range_params* p, const int64_t* ts, const double* val,
                       const uint64_t* offsets, uint64_t n_rows, uint32_t n_series, double* out,
                       uint32_t* valid_words) {
  return range_call(c, p, ts, val, offsets, n_rows, n_series, out, valid_words, nullptr);
}

static int range_call(b2p_ctx* c, const b2p_range_params* p, const int64_t* ts, const double* val,
                      const uint64_t* offsets, uint64_t n_rows, uint32_t n_series, double* out, uint32_t* valid_words,
                      const GroupTarget* gt) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  int64_t T = 0;
  int rc = check_grid(p, n_series, &T);
  if (rc) return rc;
  if (n_series == 0 || T == 0) return B2P_OK;
  if (!offsets || (!gt && (!out || !valid_words)) || ((!ts || !val) && n_rows)) return fail(B2P_E_INVALID, "NULL argument");
  if (!aligned16(ts) || !aligned16(val)) return fail(B2P_E_INVALID, "ts/val must be 16-byte aligned");
  DeviceGuard g(c->device);
  if ((rc = ensure_slow_scratch(c, n_series, T))) return rc;
  RangeArgs a = range_geometry(p, T);
  a.offset = p->offset; a.p0 = p->param0; a.p1 = p->param1; a.filter_nan = p->filter_nan;
  a.ts = ts; a.val = val; a.offsets = offsets; a.n_rows = n_rows; a.n_series = n_series;
  a.out = out; a.valid = valid_words;
  // a fused call keeps the work lists until its verdict is in: nothing else is admitted before that
  if (c->fused_pending && (rc = b2p_sync(c))) return rc;
  if (gt) {
    if (!c->pending.empty() && (rc = b2p_sync(c))) return rc;
    const size_t ns = n_series;
    if ((rc = c->w_skip.ensure(ns * 4)) || (rc = c->b_skip.ensure(ns * 4)) || (rc = c->slow_skip.ensure(ns * 4))) return rc;
    a.gsum = gt->gsum; a.gcnt = gt->gcnt; a.gid = gt->idx->gid; a.g_off = gt->idx->goff; a.g_members = gt->idx->members;
    a.n_groups = gt->idx->n_groups; a.g_lo = gt->g_lo; a.g_hi = gt->g_hi;
    a.w_skip = c->w_skip.as<uint32_t>(); a.b_skip = c->b_skip.as<uint32_t>(); a.slow_skip = c->slow_skip.as<uint32_t>();
  }
  // every call owns a status slot until b2p_sync has read it; with all slots taken the library synchronises itself
  if ((int)c->pending.size() >= kStatusSlots && (rc = b2p_sync(c))) return rc;
  const int slot = c->next_slot;
  c->next_slot = (c->next_slot + 1) % kStatusSlots;
  a.status = c->d_ring + slot; a.slow_list = c->slow_list.as<uint32_t>();
  a.w_list = c->w_list.as<uint32_t>();
  a.b_list = fits_ts32(a) ? c->b_list.as<uint32_t>() : nullptr;  // long windows: the 1024-sample ring (32-bit domain)
  a.use_w_list = 0;
  a.arena_ts = c->arena_ts.as<int64_t>(); a.arena_val = c->arena_val.as<double>(); a.arena_cap = c->arena_rows;
  a.win_scratch = c->win_scratch.as<unsigned long long>();
  b2p_ctx::Pending pc{};
  pc.slot = slot; pc.fn = p->fn_id; pc.args = a; pc.n_series = n_series;
  pc.tiers = choose_tiers(c, p->fn_id, a);
  // the choice read the back-off where the first tier applies: it runs, or mode 2 skips it
  if ((pc.tiers.first_tier || pc.tiers.lean_mode == 2) && c->lean_backoff[p->fn_id] > 0) c->lean_backoff[p->fn_id]--;
  if (gt && !pc.tiers.first_tier) return fail(B2P_E_INVALID, "fused by-label call without its first tier (internal)");
  pc.kind = !gt ? b2p_ctx::Pending::kPlain : gt->allreduce_tiles > 0 ? b2p_ctx::Pending::kMerged : b2p_ctx::Pending::kFused;
  rc = pc.kind == b2p_ctx::Pending::kMerged ? launch_allreduce_tiles(c, pc, (uint32_t)gt->allreduce_tiles)
                                            : launch_range_tiers(c, pc);
  if (rc) return rc;
  c->pending.push_back(pc);
  if (gt) c->fused_pending = true;
  return B2P_OK;
}

int b2p_range_udf_dev(b2p_ctx* c, int32_t fn_id, const int64_t* ts, const double* val, uint64_t n_rows,
                      const int64_t* packed_ranges, const int64_t* eval_ts, uint64_t n_win, int64_t range_length,
                      double param0, double param1, double* out, uint8_t* valid) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  if (n_win == 0) return B2P_OK;
  if (!packed_ranges || !out || !valid || ((!ts || !val) && n_rows)) return fail(B2P_E_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  stage_begin(c, 1);
  const int rc = with_fn(fn_id, [&](auto k) {
    range_udf_kernel<decltype(k)::value><<<capped_grid(c, n_win, 128, 32), 128, 0, c->stream>>>(
        ts, val, packed_ranges, eval_ts, n_win, range_length, param0, param1, out, valid);
    c->launches++;
    CU(cudaGetLastError());
    return B2P_OK;
  });
  stage_end(c, 1);
  return rc;
}

}  // extern "C"

// The grid of an instant selector: check_grid over lookback windows, and the grid fields of its kernel arguments.
static int instant_grid(int64_t start, int64_t end, int64_t interval, int64_t lookback, int64_t offset,
                        uint32_t n_series, InstantArgs* a) {
  b2p_range_params p{};
  p.start = start; p.end = end; p.interval = interval; p.range = lookback;
  int64_t T = 0;
  if (int rc = check_grid(&p, n_series, &T)) return rc;
  *a = InstantArgs{};
  a->start = start; a->end = end; a->interval = interval; a->lookback = lookback; a->offset = offset;
  a->T = T; a->Tw = (uint32_t)((T + 31) / 32); a->n_series = n_series;
  return B2P_OK;
}

extern "C" {

}  // extern "C"

// K4 over the grid `a`; `val` is not read (and may be NULL) in timestamp mode
static int instant_select_run(b2p_ctx* c, InstantArgs& a, const int64_t* ts, const double* val, const uint64_t* offsets,
                              uint64_t n_rows, double* out, uint32_t* valid_words, bool timestamp) {
  if (a.n_series == 0 || a.T == 0) return B2P_OK;
  if (!offsets || !out || !valid_words || ((!ts || (!val && !timestamp)) && n_rows))
    return fail(B2P_E_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  a.ts = ts; a.val = val; a.offsets = offsets; a.out = out; a.valid = valid_words;
  stage_begin(c, 1);
  (timestamp ? instant_kernel<true> : instant_kernel<false>)<<<capped_grid(c, a.n_series, kWarpsPerCta, 8),
                                                               kWarpsPerCta * 32, 0, c->stream>>>(a);
  c->launches++;
  stage_end(c, 1);
  CU(cudaGetLastError());
  return B2P_OK;
}

extern "C" {

int b2p_instant_select_dev(b2p_ctx* c, int64_t start, int64_t end, int64_t interval, int64_t lookback, int64_t offset,
                           const int64_t* ts, const double* val, const uint64_t* offsets, uint64_t n_rows,
                           uint32_t n_series, double* out, uint32_t* valid_words) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  InstantArgs a;
  if (int rc = instant_grid(start, end, interval, lookback, offset, n_series, &a)) return rc;
  return instant_select_run(c, a, ts, val, offsets, n_rows, out, valid_words, false);
}

int b2p_instant_timestamp_dev(b2p_ctx* c, int64_t start, int64_t end, int64_t interval, int64_t lookback,
                              int64_t offset, const int64_t* ts, const uint64_t* offsets, uint64_t n_rows,
                              uint32_t n_series, double* out, uint32_t* valid_words) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  InstantArgs a;
  if (int rc = instant_grid(start, end, interval, lookback, offset, n_series, &a)) return rc;
  return instant_select_run(c, a, ts, nullptr, offsets, n_rows, out, valid_words, true);
}

// n_fields and the two pointer arrays of a multi-field call; they must hold before the host form sizes its staging
static int check_fields(const void* vals, const void* outs, int32_t n_fields) {
  if (n_fields < 1 || n_fields > B2P_MAX_FIELDS)
    return fail(B2P_E_INVALID, "n_fields must be in [1, %d] (got %d)", B2P_MAX_FIELDS, (int)n_fields);
  if (!vals || !outs) return fail(B2P_E_INVALID, "NULL argument");
  return B2P_OK;
}

// NULL / alignment checks of the F columns and grids of a call that has rows and a non-empty grid
static int check_field_columns(const double* const* vals, double* const* outs, int32_t n_fields, uint64_t n_rows) {
  for (int32_t f = 0; f < n_fields; ++f) {
    if ((!vals[f] && n_rows) || !outs[f]) return fail(B2P_E_INVALID, "NULL argument (field %d)", (int)f);
    if (!aligned16(vals[f])) return fail(B2P_E_INVALID, "field %d column must be 16-byte aligned", (int)f);
  }
  return B2P_OK;
}

// Range functions that test is_null or go through arrow's null-skipping aggregates in the reference: sum / avg / min /
// max_over_time (compute::sum / min / max; avg divides by the window's length, NULL slots included), stdvar /
// stddev_over_time (`value.unwrap()` on each slot: a NULL panics), deriv and predict_linear (linear_regression_slices
// skips is_null slots, functions.rs:126-144).  Every other function reads the value buffer as it is (`values()`: rate /
// increase / delta, irate / idelta, resets, changes, last_over_time, quantile_over_time, holt_winters) or only the
// window's length (count / present / absent_over_time), as SeriesNormalize's NaN filter reads `value(i)`
// (normalize.rs:415-428): over NULL slots a multi-field call reproduces those from the buffer values alone.
static bool reads_nulls(int fn) {
  switch (fn) {
    case B2P_FN_SUM_OVER_TIME: case B2P_FN_AVG_OVER_TIME: case B2P_FN_MIN_OVER_TIME: case B2P_FN_MAX_OVER_TIME:
    case B2P_FN_STDVAR_OVER_TIME: case B2P_FN_STDDEV_OVER_TIME: case B2P_FN_DERIV: case B2P_FN_PREDICT_LINEAR:
      return true;
    default:
      return false;
  }
}

// The first field whose validity bitmap has a NULL slot in rows [0, n_rows), or -1 (field_valid or an entry NULL: none).
// Synchronises once when a bitmap is given.
static int first_null_field(b2p_ctx* c, const uint8_t* const* field_valid, int32_t n_fields, uint64_t n_rows, int* out) {
  *out = -1;
  if (!field_valid || n_rows == 0) return B2P_OK;
  bool any = false;
  for (int32_t f = 0; f < n_fields; ++f) any |= field_valid[f] != nullptr;
  if (!any) return B2P_OK;
  if (int rc = c->fd_null.ensure((size_t)kMaxFields * 4)) return rc;
  uint32_t* flags = c->fd_null.as<uint32_t>();
  CU(cudaMemsetAsync(flags, 0, (size_t)n_fields * 4, c->stream));
  for (int32_t f = 0; f < n_fields; ++f) {
    if (!field_valid[f]) continue;
    null_slots_kernel<<<capped_grid(c, (n_rows + 7) / 8, 256, 8), 256, 0, c->stream>>>(field_valid[f], n_rows, flags + f);
    c->launches++;
    CU(cudaGetLastError());
  }
  uint32_t h[kMaxFields];
  CU(cudaMemcpyAsync(h, flags, (size_t)n_fields * 4, cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->stream));
  for (int32_t f = 0; f < n_fields; ++f)
    if (h[f]) { *out = f; break; }
  return B2P_OK;
}

// An outstanding range call reads or writes `b`, and b2p_sync may run it again there: `b` must not change before that.
static bool pending_reads(const b2p_ctx* c, const DevBuf& b) {
  const char* lo = b.as<char>();
  auto in = [&](const void* p) { return lo && static_cast<const char*>(p) >= lo && static_cast<const char*>(p) < lo + b.cap; };
  for (const b2p_ctx::Pending& pc : c->pending) {
    const RangeArgs& a = pc.args;
    if (in(a.ts) || in(a.val) || in(a.offsets) || in(a.out) || in(a.valid)) return true;
  }
  return false;
}

int b2p_range_eval_fields_dev(b2p_ctx* c, const b2p_range_params* p, const int64_t* ts, const double* const* vals,
                              const uint8_t* const* field_valid, int32_t n_fields, const uint64_t* offsets,
                              uint64_t n_rows, uint32_t n_series, double* const* outs, uint32_t* valid_words) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  int rc = check_fields(vals, outs, n_fields);
  if (rc) return rc;
  if (p && p->fn_id >= 0 && p->fn_id < B2P_FN__COUNT && reads_nulls(p->fn_id)) {
    DeviceGuard g(c->device);
    int f = -1;
    if ((rc = first_null_field(c, field_valid, n_fields, n_rows, &f))) return rc;
    if (f >= 0)
      return fail(B2P_E_INVALID, "field %d has NULL slots: range function %d skips NULL slots in the reference, which a "
                  "multi-field call does not reproduce", f, (int)p->fn_id);
  }
  if (n_fields == 1) return b2p_range_eval_dev(c, p, ts, vals[0], offsets, n_rows, n_series, outs[0], valid_words);
  int64_t T = 0;
  if ((rc = check_grid(p, n_series, &T))) return rc;
  if (n_series == 0 || T == 0) return B2P_OK;
  if (!offsets || !valid_words || (!ts && n_rows)) return fail(B2P_E_INVALID, "NULL argument");
  if ((rc = check_field_columns(vals, outs, n_fields, n_rows))) return rc;
  DeviceGuard g(c->device);
  const int F = n_fields;
  const uint32_t Tw = (uint32_t)((T + 31) / 32);
  const uint64_t words = (uint64_t)n_series * Tw;
  const double* fv[kMaxFields];
  for (int f = 0; f < F; ++f) fv[f] = vals[f];
  if ((pending_reads(c, c->fd_val) || pending_reads(c, c->fd_valid)) && (rc = b2p_sync(c))) return rc;
  if (p->filter_nan && n_rows) {
    const uint64_t stride = (n_rows + 1) & ~1ull;  // 16-byte aligned columns
    if ((rc = c->fd_val.ensure((size_t)F * stride * 8))) return rc;
    double* base = c->fd_val.as<double>();
    for (int f = 0; f < F; ++f) {
      CU(cudaMemcpyAsync(base + f * stride, vals[f], n_rows * 8, cudaMemcpyDeviceToDevice, c->stream));
      fv[f] = base + f * stride;
    }
    stage_begin(c, 0);
    nan_union_kernel<<<capped_grid(c, n_rows, 256, 8), 256, 0, c->stream>>>(base, stride, F, n_rows);
    c->launches++;
    stage_end(c, 0);
    CU(cudaGetLastError());
  }
  if ((rc = c->fd_valid.ensure((size_t)(F - 1) * words * 4))) return rc;
  ValidAndArgs va{};
  va.F = F; va.out = valid_words; va.n_words = words; va.Tw = Tw; va.T = (uint64_t)T;
  va.in[0] = valid_words;
  for (int f = 1; f < F; ++f) va.in[f] = c->fd_valid.as<uint32_t>() + (uint64_t)(f - 1) * words;
  for (int f = 0; f < F; ++f)
    if ((rc = range_call(c, p, ts, fv[f], offsets, n_rows, n_series, outs[f], const_cast<uint32_t*>(va.in[f]), nullptr)))
      return rc;
  if ((rc = b2p_sync(c))) return rc;  // slow-path fix-ups (and repeated calls) land before the conjunction reads
  stage_begin(c, 3);
  valid_and_kernel<<<capped_grid(c, words, 256, 16), 256, 0, c->stream>>>(va);
  c->launches++;
  stage_end(c, 3);
  CU(cudaGetLastError());
  return B2P_OK;
}

}  // extern "C"

namespace {
// b2p_instant_select_fields_dev, and with i64 its Int64 form (field 0 is Int64: no staleness test, K17 for every F)
int instant_select_fields(b2p_ctx* c, int64_t start, int64_t end, int64_t interval, int64_t lookback, int64_t offset,
                          const int64_t* ts, const double* const* vals, const uint8_t* const* field_valid,
                          int32_t n_fields, const uint64_t* offsets, uint64_t n_rows, uint32_t n_series,
                          double* const* outs, uint32_t* valid_words, bool i64) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  int rc = check_fields(vals, outs, n_fields);
  if (rc) return rc;
  {  // the reference exports a NULL slot of the chosen row as a NULL in that field of an emitted row: one validity
     // bitmap for all fields cannot carry it
    DeviceGuard g(c->device);
    int f = -1;
    if ((rc = first_null_field(c, field_valid, n_fields, n_rows, &f))) return rc;
    if (f >= 0 && i64 && n_fields == 1)
      return fail(B2P_E_INVALID, "Int64 field has NULL slots: the instant selector exports a chosen NULL slot as a NULL "
                  "value (no stale-NaN test reads it), which the dense grid does not carry");
    if (f >= 0)
      return fail(B2P_E_INVALID, "field %d has NULL slots: the instant selector exports them as NULL in that field "
                  "only, which a multi-field call does not reproduce", f);
  }
  if (n_fields == 1 && !i64)
    return b2p_instant_select_dev(c, start, end, interval, lookback, offset, ts, vals[0], offsets, n_rows, n_series,
                                  outs[0], valid_words);
  FieldsInstantArgs fa{};
  InstantArgs& a = fa.g;
  if ((rc = instant_grid(start, end, interval, lookback, offset, n_series, &a))) return rc;
  if (n_series == 0 || a.T == 0) return B2P_OK;
  if (!offsets || !valid_words || (!ts && n_rows)) return fail(B2P_E_INVALID, "NULL argument");
  if ((rc = check_field_columns(vals, outs, n_fields, n_rows))) return rc;
  DeviceGuard g(c->device);
  a.ts = ts; a.val = vals[0]; a.offsets = offsets; a.out = outs[0]; a.valid = valid_words;
  fa.F = n_fields;
  for (int f = 0; f < n_fields; ++f) { fa.vals[f] = vals[f]; fa.outs[f] = outs[f]; }
  stage_begin(c, 1);
  (i64 ? instant_fields_kernel<false> : instant_fields_kernel<true>)<<<capped_grid(c, n_series, kWarpsPerCta, 8),
                                                                      kWarpsPerCta * 32, 0, c->stream>>>(fa);
  c->launches++;
  stage_end(c, 1);
  CU(cudaGetLastError());
  return B2P_OK;
}
}  // namespace

extern "C" {

int b2p_instant_select_fields_dev(b2p_ctx* c, int64_t start, int64_t end, int64_t interval, int64_t lookback,
                                  int64_t offset, const int64_t* ts, const double* const* vals,
                                  const uint8_t* const* field_valid, int32_t n_fields, const uint64_t* offsets,
                                  uint64_t n_rows, uint32_t n_series, double* const* outs, uint32_t* valid_words) {
  return instant_select_fields(c, start, end, interval, lookback, offset, ts, vals, field_valid, n_fields, offsets,
                               n_rows, n_series, outs, valid_words, false);
}

int b2p_instant_select_fields_i64_dev(b2p_ctx* c, int64_t start, int64_t end, int64_t interval, int64_t lookback,
                                      int64_t offset, const int64_t* ts, const double* const* vals,
                                      const uint8_t* const* field_valid, int32_t n_fields, const uint64_t* offsets,
                                      uint64_t n_rows, uint32_t n_series, double* const* outs, uint32_t* valid_words) {
  return instant_select_fields(c, start, end, interval, lookback, offset, ts, vals, field_valid, n_fields, offsets,
                               n_rows, n_series, outs, valid_words, true);
}

// sum by (..)(fn(..)) partials of groups [g_lo, g_hi) added into out_sum / out_cnt [n_groups x T].
// Fused (no [n_series x T] intermediate) for rate / increase / delta whenever the first tier applies; otherwise the
// range function is evaluated into context scratch and folded by the by-label kernel (two passes, synchronous).
int b2p_range_group_sum_indexed_dev(b2p_ctx* c, const b2p_range_params* p, const int64_t* ts, const double* val,
                                    const uint64_t* offsets, uint64_t n_rows, uint32_t n_series,
                                    const b2p_group_index* ix, uint32_t g_lo, uint32_t g_hi, double* out_sum,
                                    uint32_t* out_cnt) {
  if (!c || !ix) return fail(B2P_E_INVALID, "NULL argument");
  if (ix->n_series != n_series) return fail(B2P_E_INVALID, "group index was built for %u series, call has %u", ix->n_series, n_series);
  if (g_hi > ix->n_groups) g_hi = ix->n_groups;
  int64_t T = 0;
  int rc = check_grid(p, n_series, &T);
  if (rc) return rc;
  if (n_series == 0 || T == 0 || g_lo >= g_hi) return B2P_OK;
  if (!out_sum || !out_cnt) return fail(B2P_E_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  if (fused_group_ok(c, p, T, ix)) {
    GroupTarget gt{ix, g_lo, g_hi, out_sum, out_cnt, 0};
    return range_call(c, p, ts, val, offsets, n_rows, n_series, nullptr, nullptr, &gt);
  }
  if (g_lo != 0 || g_hi != ix->n_groups)
    return fail(B2P_E_INVALID, "group ranges need the fused tier (rate / increase / delta in the 32-bit time domain)");
  const uint32_t Tw = (uint32_t)((T + 31) / 32);
  if ((rc = c->rg_out.ensure((size_t)n_series * (size_t)T * 8))) return rc;
  if ((rc = c->rg_valid.ensure((size_t)n_series * Tw * 4))) return rc;
  if ((rc = b2p_range_eval_dev(c, p, ts, val, offsets, n_rows, n_series, c->rg_out.as<double>(),
                               c->rg_valid.as<uint32_t>())))
    return rc;
  if ((rc = b2p_sync(c))) return rc;  // slow-path fix-ups must land before the aggregate reads
  stage_begin(c, 3);
  rc = group_aggregate_csr(c, B2P_AGG_SUM, c->rg_out.as<double>(), c->rg_valid.as<uint32_t>(), ix->goff, ix->members,
                           ix->n_groups, (uint64_t)T, out_sum, out_cnt, 1);
  stage_end(c, 3);
  return rc;
}

// sum by over all ranks: the fused partials of this rank's series, tile by tile, each tile all-reduced over the
// communicator while the next one computes.  Falls back to partials + one all-reduce when the call cannot run fused.
int b2p_range_group_sum_allreduce_dev(b2p_ctx* c, const b2p_range_params* p, const int64_t* ts, const double* val,
                                      const uint64_t* offsets, uint64_t n_rows, uint32_t n_series,
                                      const b2p_group_index* ix, int32_t n_tiles, double* out_sum, uint32_t* out_cnt) {
  if (!c || !ix) return fail(B2P_E_INVALID, "NULL argument");
  if (ix->n_series != n_series) return fail(B2P_E_INVALID, "group index was built for %u series, call has %u", ix->n_series, n_series);
  int64_t T = 0;
  int rc = check_grid(p, n_series, &T);
  if (rc) return rc;
  if (T == 0 || ix->n_groups == 0) return B2P_OK;
  if (!out_sum || !out_cnt) return fail(B2P_E_INVALID, "NULL argument");
  if (n_tiles < 1) n_tiles = 1;
  DeviceGuard g(c->device);
  if (n_series > 0 && fused_group_ok(c, p, T, ix)) {
    GroupTarget gt{ix, 0, ix->n_groups, out_sum, out_cnt, n_tiles};
    return range_call(c, p, ts, val, offsets, n_rows, n_series, nullptr, nullptr, &gt);
  }
  if (n_series > 0 &&
      (rc = b2p_range_group_sum_indexed_dev(c, p, ts, val, offsets, n_rows, n_series, ix, 0, ix->n_groups, out_sum, out_cnt)))
    return rc;
  return b2p_allreduce_partials_dev(c, B2P_AGG_SUM, out_sum, out_cnt, nullptr, (uint64_t)ix->n_groups * (uint64_t)T);
}

int b2p_range_group_sum_fused(b2p_ctx* c, const b2p_range_params* p, const b2p_group_index* ix) {
  if (!c || !ix || !p || p->interval <= 0) return 0;  // (a grid the range call itself would reject)
  int64_t T = b2p_num_steps(p->start, p->end, p->interval);
  return fused_group_ok(c, p, T, ix) ? 1 : 0;
}

int b2p_range_group_sum_dev(b2p_ctx* c, const b2p_range_params* p, const int64_t* ts, const double* val,
                            const uint64_t* offsets, uint64_t n_rows, uint32_t n_series, const uint32_t* gid,
                            uint32_t n_groups, double* out_sum, uint32_t* out_cnt) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  if (n_series == 0 || n_groups == 0) return B2P_OK;
  b2p_group_index* ix = nullptr;
  int rc = b2p_group_index_create_dev(c, gid, n_series, n_groups, &ix);
  if (rc) return rc;
  rc = b2p_range_group_sum_indexed_dev(c, p, ts, val, offsets, n_rows, n_series, ix, 0, n_groups, out_sum, out_cnt);
  if (!rc) rc = b2p_sync(c);  // the temporary index must outlive the kernels that read it
  b2p_group_index_destroy(c, ix);
  return rc;
}

/* ---- subqueries ---------------------------------------------------------------------------------------------- */
}  // extern "C"

// K13's count kernel, then CUB's exclusive scan of the counts in place (declared in b2p_runtime.cuh; K14 uses it too)
int scan_valid_cells(b2p_ctx* c, const uint32_t* valid, uint64_t T, uint32_t rows, unsigned long long* offsets,
                     DevBuf& tmp) {
  size_t bytes = 0;
  CU(cub::DeviceScan::ExclusiveSum(nullptr, bytes, offsets, offsets, (int)rows + 1, c->stream));
  if (int rc = tmp.ensure(std::max<size_t>(bytes, 16))) return rc;
  SubqueryArgs a{};
  a.valid = valid; a.T = T; a.Tw = (uint32_t)((T + 31) / 32); a.rows = rows; a.offsets = offsets;
  subquery_count_kernel<<<cell_rows_grid(c, rows), 256, 0, c->stream>>>(a);
  c->launches++;
  CU(cudaGetLastError());
  bytes = tmp.cap;
  CU(cub::DeviceScan::ExclusiveSum(tmp.p, bytes, offsets, offsets, (int)rows + 1, c->stream));
  return B2P_OK;
}

namespace {
// Rows are processed in batches of at most kSqBatchCells / T_inner rows (one row when a row alone is larger).  Per
// batch: K13's count kernel, CUB's exclusive scan of the counts, K13's scatter, then the range call over the batch's
// sample rows into its rows of out / out_valid.  The range call is given the batch's cell count as its row count: the
// extent of the scratch, which the tiers only use to bound their paired loads, so the sample total is never read back.
// A batch waits (b2p_sync) for the verdict of the range call before it, since the scratch is rewritten; so does the
// first batch for that of an earlier call.  A grid of one batch makes no host round trip.
// Scratch (context buffers sq_*): 16 B per grid cell of a batch (8 B timestamp, 8 B value: at most 2.1 GB unless one
// row alone has more than kSqBatchCells steps), 8 B per row of a batch plus one for the offsets, and CUB's scan temp.
int subquery_run(b2p_ctx* c, const b2p_range_params* p, int64_t inner_start, int64_t inner_interval, const double* vals,
                 const uint32_t* valid, uint32_t n_rows, uint64_t T_inner, int64_t T, double* out, uint32_t* out_valid) {
  int rc;
  const uint32_t Tw_in = (uint32_t)((T_inner + 31) / 32), Tw = (uint32_t)((T + 31) / 32);
  const uint32_t batch_rows = (uint32_t)std::min<uint64_t>(n_rows, std::max<uint64_t>(1, kSqBatchCells / T_inner));
  const uint64_t cells = (uint64_t)batch_rows * T_inner;
  // a range call of an earlier batch or call may still be run again from the scratch (it reads its timestamps there)
  if (pending_reads(c, c->sq_ts) && (rc = b2p_sync(c))) return rc;
  if ((rc = c->sq_ts.ensure(cells * 8)) || (rc = c->sq_val.ensure(cells * 8)) ||
      (rc = c->sq_off.ensure(((size_t)batch_rows + 1) * 8)))
    return rc;
  b2p_range_params q = *p;
  for (uint32_t r0 = 0; r0 < n_rows; r0 += batch_rows) {
    const uint32_t nb = std::min(batch_rows, n_rows - r0);
    if (r0 > 0 && (rc = b2p_sync(c))) return rc;
    SubqueryArgs a{};
    a.vals = vals + (uint64_t)r0 * T_inner; a.valid = valid + (uint64_t)r0 * Tw_in;
    a.T = T_inner; a.Tw = Tw_in; a.rows = nb;
    a.start = inner_start; a.interval = inner_interval;
    a.offsets = c->sq_off.as<unsigned long long>(); a.ts = c->sq_ts.as<int64_t>(); a.val = c->sq_val.as<double>();
    stage_begin(c, 3);
    if ((rc = scan_valid_cells(c, a.valid, T_inner, nb, a.offsets, c->sq_tmp))) return rc;
    subquery_scatter_kernel<<<cell_rows_grid(c, nb), 256, 0, c->stream>>>(a);
    c->launches++;
    CU(cudaGetLastError());
    stage_end(c, 3);
    if ((rc = range_call(c, &q, a.ts, a.val, c->sq_off.as<uint64_t>(), (uint64_t)nb * T_inner, nb,
                         out + (uint64_t)r0 * T, out_valid + (uint64_t)r0 * Tw, nullptr)))
      return rc;
  }
  return B2P_OK;
}
}  // namespace

extern "C" {

int b2p_subquery_dev(b2p_ctx* c, const b2p_range_params* p, int64_t inner_start, int64_t inner_interval,
                     const double* vals, const uint32_t* valid, uint32_t n_rows, uint64_t T_inner, double* out,
                     uint32_t* out_valid) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  int64_t T = 0;
  int rc = check_grid(p, n_rows, &T);
  if (rc) return rc;
  if (p->range == 0) return fail(B2P_E_INVALID, "subquery: zero range");
  if (p->offset != 0 || p->filter_nan != 0) return fail(B2P_E_INVALID, "subquery: offset and filter_nan must be 0");
  if (inner_interval <= 0) return fail(B2P_E_INVALID, "subquery: inner interval must be > 0 (got %lld)", (long long)inner_interval);
  if (n_rows == 0 || T == 0) return B2P_OK;
  if (!out || !out_valid || (T_inner && (!vals || !valid))) return fail(B2P_E_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  if (T_inner == 0) {  // no inner steps: no samples, no cell
    CU(cudaMemsetAsync(out, 0, (size_t)n_rows * (size_t)T * 8, c->stream));
    CU(cudaMemsetAsync(out_valid, 0, (size_t)n_rows * (size_t)((T + 31) / 32) * 4, c->stream));
    return B2P_OK;
  }
  return subquery_run(c, p, inner_start, inner_interval, vals, valid, n_rows, T_inner, T, out, out_valid);
}

int b2p_synth_fill_dev(b2p_ctx* c, uint64_t series_begin, uint64_t n_series, uint32_t n_samples, int64_t t0,
                       int64_t scrape_ms, uint32_t jitter_ms, int32_t with_resets, uint64_t seed, int64_t* ts,
                       double* val, uint32_t* sid) {
  if (!c || !ts || !val) return fail(B2P_E_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  const uint64_t total = n_series * (uint64_t)n_samples;
  if (total == 0) return B2P_OK;
  synth_fill_kernel<<<capped_grid(c, total, 256, 32), 256, 0, c->stream>>>(series_begin, n_series, n_samples, t0,
                                                                           scrape_ms, jitter_ms, with_resets, seed, ts,
                                                                           val, sid);
  c->launches++;
  CU(cudaGetLastError());
  return B2P_OK;
}

/* ---- host-pointer API ------------------------------------------------------------------------ */
}  // extern "C"

// A host offsets column as every tier reads it, offsets[s] .. offsets[s + 1] without a clamp: non-decreasing, its last
// entry <= n_rows (rows before its first entry or past its last belong to no series).  The rule b2p_host_scan_series
// applies; B2P_E_INVALID, checked before anything is copied.
static int check_host_offsets(const uint64_t* offsets, uint64_t n_rows, uint32_t n_series) {
  for (uint32_t s = 0; s < n_series; ++s)
    if (offsets[s + 1] < offsets[s])
      return fail(B2P_E_INVALID, "offsets decrease at series %u (%llu -> %llu)", s, (unsigned long long)offsets[s],
                  (unsigned long long)offsets[s + 1]);
  if (offsets[n_series] > n_rows)
    return fail(B2P_E_INVALID, "offsets[n_series] = %llu exceeds n_rows = %llu", (unsigned long long)offsets[n_series],
                (unsigned long long)n_rows);
  return B2P_OK;
}

SeriesIn stage_series(Staging& s, const int64_t* ts, const double* val, const uint32_t* sid, uint32_t sid_base,
                      const uint64_t* offsets_host, uint64_t n_rows, uint32_t n_series) {
  if (!sid && !offsets_host && !s.rc) s.rc = fail(B2P_E_INVALID, "need sid or offsets_host");
  if (offsets_host && !s.rc) s.rc = check_host_offsets(offsets_host, n_rows, n_series);
  SeriesIn in{s.in(ts, n_rows * 8), s.in(val, n_rows * 8), nullptr};
  if (offsets_host) {
    in.offsets = s.in(offsets_host, ((size_t)n_series + 1) * 8);
  } else {
    const uint32_t* d_sid = s.in(sid, n_rows * 4);
    in.offsets = static_cast<uint64_t*>(s.buf(((size_t)n_series + 1) * 8));
    if (!s.rc) s.rc = series_offsets_impl(s.c, d_sid, n_rows, n_series, sid_base, in.offsets);
  }
  return in;
}

extern "C" {

// Host-side SeriesDivide + cadence scan (see the header).  Plain sequential passes, memory bound;
// b2p_range_eval runs one of these per chunk on a few worker threads while earlier chunks are on the bus.
static int host_scan_series(const int64_t* ts, const uint32_t* sid, const uint64_t* offsets_in, uint64_t n_rows,
                            uint32_t n_series, uint32_t sid_base, uint64_t* offsets_out, int64_t* t0, int64_t* cadence,
                            int32_t* all_regular) {
  if (sid) {
    uint64_t r = 0;
    uint32_t prev = sid_base;
    offsets_out[0] = 0;
    uint32_t next = 0;  // next local series whose start is still to be written (offsets_out[next + 1 ..] pending)
    for (; r < n_rows; ++r) {
      const uint32_t id = sid[r];
      if (id < prev || id - sid_base >= n_series) return B2P_E_UNSORTED;
      const uint32_t local = id - sid_base;
      while (next < local) offsets_out[++next] = r;  // series without rows in between start (and end) here
      prev = id;
    }
    while (next < n_series) offsets_out[++next] = n_rows;
  } else {
    for (uint32_t s = 0; s <= n_series; ++s) offsets_out[s] = offsets_in[s] - offsets_in[0];
    for (uint32_t s = 0; s < n_series; ++s)
      if (offsets_out[s + 1] < offsets_out[s] || offsets_out[s + 1] > n_rows) return B2P_E_INVALID;
  }
  bool regular = true;
  for (uint32_t s = 0; s < n_series; ++s) {
    const uint64_t r0 = offsets_out[s], r1 = offsets_out[s + 1];
    const int64_t first = r1 > r0 ? ts[r0] : 0;
    // (wrapping arithmetic: the device rebuilds the column with the same operations)
    const int64_t step = r1 - r0 >= 2 ? (int64_t)((uint64_t)ts[r0 + 1] - (uint64_t)first) : 0;
    if (t0) t0[s] = first;
    if (cadence) cadence[s] = step;
    if (regular) {
      uint64_t expect = (uint64_t)first;
      for (uint64_t r = r0; r < r1; ++r) {
        if ((uint64_t)ts[r] != expect) { regular = false; break; }
        expect += (uint64_t)step;
      }
    }
    if (!regular && !t0 && !cadence) break;
  }
  if (all_regular) *all_regular = regular ? 1 : 0;
  return B2P_OK;
}

int b2p_host_scan_series(const int64_t* ts, const uint32_t* sid, const uint64_t* offsets_in, uint64_t n_rows,
                         uint32_t n_series, uint32_t sid_base, uint64_t* offsets_out, int64_t* t0, int64_t* cadence,
                         int32_t* all_regular) {
  if (!offsets_out || (!sid && !offsets_in) || (!ts && n_rows)) return fail(B2P_E_INVALID, "NULL argument");
  const int rc = host_scan_series(ts, sid, offsets_in, n_rows, n_series, sid_base, offsets_out, t0, cadence, all_regular);
  if (rc == B2P_E_UNSORTED) return fail(rc, "series-id column is not non-decreasing or out of range");
  if (rc) return fail(rc, "offsets are not non-decreasing or exceed n_rows");
  return rc;
}

// A call small enough for one shot, no overlap: H2D -> K0/K2 -> D2H on the context stream.
static int range_eval_host_simple(b2p_ctx* c, const b2p_range_params* p, const int64_t* ts, const double* val,
                                  const uint32_t* sid, const uint64_t* offsets_host, uint64_t n_rows, uint32_t n_series,
                                  int64_t T, double* out, uint32_t* valid_words) {
  int rc;
  const uint32_t Tw = (uint32_t)((T + 31) / 32);
  c->last_h2d_bytes = (long long)(n_rows * 16 + (offsets_host ? ((size_t)n_series + 1) * 8 : n_rows * 4));
  Staging s{c};
  const SeriesIn in = stage_series(s, ts, val, sid, 0u, offsets_host, n_rows, n_series);
  double* d_out = s.out(out, (size_t)n_series * (size_t)T * 8);
  uint32_t* d_valid = s.out(valid_words, (size_t)n_series * Tw * 4);
  if ((rc = s.rc) || (rc = b2p_range_eval_dev(c, p, in.ts, in.val, in.offsets, n_rows, n_series, d_out, d_valid)) ||
      (rc = b2p_sync(c)))
    return rc;
  return s.finish();
}

// first row whose id is >= key in a non-decreasing id column
static uint64_t lower_bound_sid(const uint32_t* sid, uint64_t n, uint64_t key) {
  uint64_t lo = 0, hi = n;
  while (lo < hi) {
    const uint64_t mid = (lo + hi) >> 1;
    if ((uint64_t)sid[mid] < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

}  // extern "C"

namespace {
// One chunk of b2p_range_eval's pipeline: series [s0, s1), rows [r0, r1) of the host columns.
struct Chunk {
  uint32_t s0, s1;
  uint64_t r0, r1;
};

// pinned host memory, freed with its owner
struct FreeHost {
  void operator()(void* p) const { cudaFreeHost(p); }
};
template <class T>
using Pinned = std::unique_ptr<T[], FreeHost>;
template <class T>
int alloc_pinned(Pinned<T>& p, size_t n) {
  T* raw = nullptr;
  CU(cudaMallocHost(&raw, n * sizeof(T)));
  p.reset(raw);
  return B2P_OK;
}

// the host scan's worker threads, stopped and joined when their owner goes (before the pinned arrays they fill)
struct ScanWorkers {
  std::atomic<bool> stop{false};
  std::vector<std::thread> threads;
  void join() {
    stop.store(true);
    for (auto& t : threads)
      if (t.joinable()) t.join();
  }
  ~ScanWorkers() { join(); }
};
}  // namespace

extern "C" {

int b2p_range_eval(b2p_ctx* c, const b2p_range_params* p, const int64_t* ts, const double* val, const uint32_t* sid,
                   const uint64_t* offsets_host, uint64_t n_rows, uint32_t n_series, double* out,
                   uint32_t* valid_words, int64_t* out_ts) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  int64_t T = 0;
  int rc = check_grid(p, n_series, &T);
  if (rc) return rc;
  if (out_ts)
    for (int64_t k = 0; k < T; ++k) out_ts[k] = p->start + k * p->interval;
  if (n_series == 0 || T == 0) return B2P_OK;
  if (!sid && !offsets_host) return fail(B2P_E_INVALID, "need sid or offsets_host");
  if (!out || !valid_words || ((!ts || !val) && n_rows)) return fail(B2P_E_INVALID, "NULL argument");
  DeviceGuard g(c->device);
  if (!c->pending.empty() && (rc = b2p_sync(c))) return rc;  // earlier asynchronous calls finish first
  const uint32_t Tw = (uint32_t)((T + 31) / 32);

  // ---- small inputs: one shot -------------------------------------------------------------------
  constexpr uint64_t kChunkRows = 4u << 20;  // ~84 MB of H2D per chunk
  if (n_rows <= kChunkRows + kChunkRows / 2 || n_series < 64)
    return range_eval_host_simple(c, p, ts, val, sid, offsets_host, n_rows, n_series, T, out, valid_words);

  // ---- large inputs: series chunks, double-buffered; H2D(i+1) | K0+K2(i) | D2H(i-1) overlap -----------
  if (offsets_host && (rc = check_host_offsets(offsets_host, n_rows, n_series))) return rc;
  const uint64_t avg_rows = n_rows / n_series + 1;
  uint32_t C = (uint32_t)(kChunkRows / avg_rows);
  if (C < 64) C = 64;
  const uint32_t n_chunks = (n_series + C - 1) / C;
  if (!c->pipe_ready) {
    bool ok = cudaStreamCreateWithFlags(&c->s_h2d, cudaStreamNonBlocking) == cudaSuccess;
    ok = ok && cudaStreamCreateWithFlags(&c->s_d2h, cudaStreamNonBlocking) == cudaSuccess;
    for (int i = 0; ok && i < 2; ++i) {
      ok = ok && cudaEventCreateWithFlags(&c->ev_h2d[i], cudaEventDisableTiming) == cudaSuccess;
      ok = ok && cudaEventCreateWithFlags(&c->ev_comp[i], cudaEventDisableTiming) == cudaSuccess;
      ok = ok && cudaEventCreateWithFlags(&c->ev_d2h[i], cudaEventDisableTiming) == cudaSuccess;
    }
    if (!ok) return fail(B2P_E_CUDA, "pipeline stream/event creation failed");
    c->pipe_ready = true;
  }
  if ((rc = c->p_status.ensure((size_t)n_chunks * sizeof(Status)))) return rc;  // device copies of each chunk's status
  Pinned<Status> h_stat;
  Pinned<uint64_t> h_offs[2];
  if ((rc = alloc_pinned(h_stat, n_chunks))) return rc;
  for (int i = 0; offsets_host && i < 2; ++i)
    if ((rc = alloc_pinned(h_offs[i], (size_t)C + 1))) return rc;

  // the chunk table (chunks are whole series) and the worst-case chunk row count
  std::vector<Chunk> chunks(n_chunks);
  uint64_t max_rows = 0;
  for (uint32_t i = 0; i < n_chunks; ++i) {
    Chunk& k = chunks[i];
    k.s0 = i * C;
    k.s1 = (uint64_t)k.s0 + C < n_series ? k.s0 + C : n_series;
    k.r0 = i ? chunks[i - 1].r1 : 0;
    k.r1 = offsets_host ? offsets_host[k.s1] : lower_bound_sid(sid, n_rows, k.s1);
    if (k.r1 < k.r0) return fail(B2P_E_UNSORTED, "series-id column is not non-decreasing");  // (offsets: checked above)
    max_rows = std::max(max_rows, k.r1 - k.r0);
  }
  if (!offsets_host && chunks.back().r1 != n_rows) return fail(B2P_E_UNSORTED, "series id >= n_series");
  // Host scan of every chunk, ahead of the copies (worker k takes chunks k, k + W, ..): 0 = not scanned yet, 1 = every
  // series of the chunk is equally spaced (its rebased offsets, first timestamps and cadences are in the pinned
  // descriptor arrays), 2 = take the ordinary route (ids out of order included: K0 reports those as before)
  // (only when the batch comes with its id column: then the descriptors replace 12 of the 20 B/row and K0; with offsets
  // handed over the call is already at 16 B/row, and the scan's per-call cost — pinned descriptor arrays, worker
  // threads — costs more than the 8 B/row it saves)
  const bool scan = c->host_ts_scan && !offsets_host;
  Pinned<uint64_t> h_doff;
  Pinned<int64_t> h_t0, h_cad;
  std::unique_ptr<std::atomic<int>[]> scan_state;
  ScanWorkers workers;
  if (scan) {
    if ((rc = alloc_pinned(h_doff, (size_t)n_series + n_chunks)) || (rc = alloc_pinned(h_t0, n_series)) ||
        (rc = alloc_pinned(h_cad, n_series)))
      return rc;
    scan_state.reset(new std::atomic<int>[n_chunks]);
    for (uint32_t i = 0; i < n_chunks; ++i) scan_state[i].store(0);
    unsigned hw = std::thread::hardware_concurrency();
    unsigned W = hw >= 64 ? 16u : (hw >= 8 ? hw / 4 : 1u);
    if (W > n_chunks) W = n_chunks;
    std::atomic<int>* state = scan_state.get();
    const Chunk* table = chunks.data();
    uint64_t* doff = h_doff.get();
    int64_t *t0 = h_t0.get(), *cad = h_cad.get();
    std::atomic<bool>& stop = workers.stop;
    try {
      for (unsigned w = 0; w < W; ++w) {
        workers.threads.emplace_back([=, &stop]() {
          for (uint32_t i = w; i < n_chunks && !stop.load(std::memory_order_relaxed); i += W) {
            const Chunk& k = table[i];
            int32_t regular = 0;
            const int rc_scan = host_scan_series(ts + k.r0, sid + k.r0, nullptr, k.r1 - k.r0, k.s1 - k.s0, k.s0,
                                                 doff + k.s0 + i, t0 + k.s0, cad + k.s0, &regular);
            state[i].store((rc_scan == B2P_OK && regular) ? 1 : 2, std::memory_order_release);
          }
        });
      }
    } catch (...) {  // no threads to be had: every chunk the started workers do not reach takes the ordinary route
      workers.join();
      for (uint32_t i = 0; i < n_chunks; ++i) {
        int zero = 0;
        state[i].compare_exchange_strong(zero, 2);
      }
    }
  }
  for (int i = 0; i < 2; ++i) {
    if (scan && (rc = c->p_t0[i].ensure((size_t)C * 8))) return rc;
    if (scan && (rc = c->p_cad[i].ensure((size_t)C * 8))) return rc;
    if ((rc = c->p_ts[i].ensure(max_rows * 8 + 16))) return rc;
    if ((rc = c->p_val[i].ensure(max_rows * 8 + 16))) return rc;
    if (!offsets_host && (rc = c->p_sid[i].ensure(max_rows * 4 + 16))) return rc;
    if ((rc = c->p_off[i].ensure(((size_t)C + 1) * 8))) return rc;
    if ((rc = c->p_out[i].ensure((size_t)C * (size_t)T * 8))) return rc;
    if ((rc = c->p_valid[i].ensure((size_t)C * Tw * 4))) return rc;
  }
  CU(cudaStreamSynchronize(c->stream));
  c->last_h2d_bytes = 0;
  std::vector<b2p_ctx::Pending> recs;  // each chunk's range call, read below with all the others
  recs.reserve(n_chunks);
  for (uint32_t i = 0; i < n_chunks; ++i) {
    const int b = (int)(i & 1);
    const Chunk& k = chunks[i];
    const uint32_t ns = k.s1 - k.s0;
    const uint64_t nr = k.r1 - k.r0;
    int described = 2;  // 1: the chunk's timestamp (and id) column is described by (offsets, t0, cadence)
    if (scan)
      while ((described = scan_state[i].load(std::memory_order_acquire)) == 0) std::this_thread::yield();
    // H2D of chunk i may start once chunk i-2's kernels no longer read this buffer pair
    if (i >= 2) CU(cudaStreamWaitEvent(c->s_h2d, c->ev_comp[b], 0));
    CU(cudaMemcpyAsync(c->p_val[b].p, val + k.r0, nr * 8, cudaMemcpyHostToDevice, c->s_h2d));
    c->last_h2d_bytes += (long long)(nr * 8);
    if (described == 1) {
      c->last_h2d_bytes += (long long)(((size_t)ns + 1) * 8 + (size_t)ns * 16);
      CU(cudaMemcpyAsync(c->p_off[b].p, h_doff.get() + k.s0 + i, ((size_t)ns + 1) * 8, cudaMemcpyHostToDevice, c->s_h2d));
      CU(cudaMemcpyAsync(c->p_t0[b].p, h_t0.get() + k.s0, (size_t)ns * 8, cudaMemcpyHostToDevice, c->s_h2d));
      CU(cudaMemcpyAsync(c->p_cad[b].p, h_cad.get() + k.s0, (size_t)ns * 8, cudaMemcpyHostToDevice, c->s_h2d));
    } else {
      c->last_h2d_bytes += (long long)(nr * 8 + (offsets_host ? ((size_t)ns + 1) * 8 : nr * 4));
      CU(cudaMemcpyAsync(c->p_ts[b].p, ts + k.r0, nr * 8, cudaMemcpyHostToDevice, c->s_h2d));
      if (offsets_host) {
        if (i >= 2) CU(cudaEventSynchronize(c->ev_h2d[b]));  // the pinned rebase buffer is free again
        for (uint32_t q = 0; q <= ns; ++q) h_offs[b][q] = offsets_host[k.s0 + q] - k.r0;
        CU(cudaMemcpyAsync(c->p_off[b].p, h_offs[b].get(), ((size_t)ns + 1) * 8, cudaMemcpyHostToDevice, c->s_h2d));
      } else {
        CU(cudaMemcpyAsync(c->p_sid[b].p, sid + k.r0, nr * 4, cudaMemcpyHostToDevice, c->s_h2d));
      }
    }
    CU(cudaEventRecord(c->ev_h2d[b], c->s_h2d));
    // compute: after its inputs landed and after chunk i-2's results left the output buffers
    CU(cudaStreamWaitEvent(c->stream, c->ev_h2d[b], 0));
    if (i >= 2) CU(cudaStreamWaitEvent(c->stream, c->ev_d2h[b], 0));
    if (described == 1) {
      ts_expand_kernel<<<capped_grid(c, ns, 8, 8), 256, 0, c->stream>>>(
          c->p_off[b].as<uint64_t>(), c->p_t0[b].as<int64_t>(), c->p_cad[b].as<int64_t>(), ns, c->p_ts[b].as<int64_t>());
      c->launches++;
      CU(cudaGetLastError());
    } else if (!offsets_host &&
               (rc = series_offsets_impl(c, c->p_sid[b].as<uint32_t>(), nr, ns, k.s0, c->p_off[b].as<uint64_t>()))) {
      return rc;
    }
    if ((rc = b2p_range_eval_dev(c, p, c->p_ts[b].as<int64_t>(), c->p_val[b].as<double>(), c->p_off[b].as<uint64_t>(),
                                 nr, ns, c->p_out[b].as<double>(), c->p_valid[b].as<uint32_t>())))
      return rc;
    // the chunk's call leaves the pending queue: its Status is copied aside, its buffer pair reused
    recs.push_back(c->pending.back());
    c->pending.pop_back();
    CU(cudaMemcpyAsync(c->p_status.as<Status>() + i, c->d_ring + recs.back().slot, sizeof(Status),
                       cudaMemcpyDeviceToDevice, c->stream));
    CU(cudaEventRecord(c->ev_comp[b], c->stream));
    // D2H
    CU(cudaStreamWaitEvent(c->s_d2h, c->ev_comp[b], 0));
    CU(cudaMemcpyAsync(out + (size_t)k.s0 * (size_t)T, c->p_out[b].p, (size_t)ns * (size_t)T * 8, cudaMemcpyDeviceToHost,
                       c->s_d2h));
    CU(cudaMemcpyAsync(valid_words + (size_t)k.s0 * Tw, c->p_valid[b].p, (size_t)ns * Tw * 4, cudaMemcpyDeviceToHost,
                       c->s_d2h));
    CU(cudaEventRecord(c->ev_d2h[b], c->s_d2h));
  }
  CU(cudaMemcpyAsync(h_stat.get(), c->p_status.p, (size_t)n_chunks * sizeof(Status), cudaMemcpyDeviceToHost, c->stream));
  CU(cudaStreamSynchronize(c->s_d2h));
  if ((rc = take_k0(c))) return rc;
  // one verdict over all chunks; a chunk whose slow path ran out of arena is redone alone, with its own tiers, from
  // its host columns (its device buffers have been reused)
  const size_t need = read_outcome(c, recs.data(), h_stat.get(), n_chunks, false);
  for (uint32_t i = 0; need && i < n_chunks; ++i) {
    if (!redo_rows(h_stat[i])) continue;
    const Chunk& k = chunks[i];
    const uint32_t ns = k.s1 - k.s0;
    const uint64_t nr = k.r1 - k.r0;
    std::vector<uint64_t> offs;
    if (offsets_host)
      for (uint32_t q = 0; q <= ns; ++q) offs.push_back(offsets_host[k.s0 + q] - k.r0);
    c->last_h2d_bytes += (long long)(nr * 16 + (offsets_host ? ((size_t)ns + 1) * 8 : nr * 4));
    Staging s{c};
    const SeriesIn in = stage_series(s, ts + k.r0, val + k.r0, sid ? sid + k.r0 : nullptr, k.s0,
                                     offsets_host ? offs.data() : nullptr, nr, ns);
    b2p_ctx::Pending redo = recs[i];
    redo.args.ts = in.ts; redo.args.val = in.val; redo.args.offsets = in.offsets;
    redo.args.out = s.out(out + (size_t)k.s0 * (size_t)T, (size_t)ns * (size_t)T * 8);
    redo.args.valid = s.out(valid_words + (size_t)k.s0 * Tw, (size_t)ns * Tw * 4);
    if ((rc = s.end([&] { return redo_calls(c, {redo}, need); }))) return rc;
  }
  return B2P_OK;
}

int b2p_range_udf(b2p_ctx* c, int32_t fn_id, const int64_t* ts, const double* val, uint64_t n_rows,
                  const int64_t* packed_ranges, const int64_t* eval_ts, uint64_t n_win, int64_t range_length,
                  double param0, double param1, double* out, uint8_t* valid) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  DeviceGuard g(c->device);
  Staging s{c};
  const int64_t* d_ts = s.in(ts, n_rows * 8);
  const double* d_val = s.in(val, n_rows * 8);
  const int64_t* d_packed = s.in(packed_ranges, n_win * 8);
  const int64_t* d_eval_ts = s.in(eval_ts, n_win * 8);
  double* d_out = s.out(out, n_win * 8);
  uint8_t* d_valid = s.out(valid, n_win);
  return s.end([&] {
    return b2p_range_udf_dev(c, fn_id, d_ts, d_val, n_rows, d_packed, d_eval_ts, n_win, range_length, param0, param1,
                             d_out, d_valid);
  });
}

}  // extern "C"

// the host forms of b2p_instant_select_dev and b2p_instant_timestamp_dev (val NULL: no value column is staged)
static int instant_select_host(b2p_ctx* c, int64_t start, int64_t end, int64_t interval, int64_t lookback,
                               int64_t offset, const int64_t* ts, const double* val, const uint32_t* sid,
                               const uint64_t* offsets_host, uint64_t n_rows, uint32_t n_series, double* out,
                               uint32_t* valid_words, bool timestamp) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  InstantArgs grid;
  if (int rc = instant_grid(start, end, interval, lookback, offset, n_series, &grid)) return rc;
  if (n_series == 0 || grid.T == 0) return B2P_OK;  // (no sample copies, no series offsets)
  DeviceGuard g(c->device);
  Staging s{c};
  const SeriesIn in = stage_series(s, ts, val, sid, 0u, offsets_host, n_rows, n_series);
  double* d_out = s.out(out, (size_t)n_series * (size_t)grid.T * 8);
  uint32_t* d_valid = s.out(valid_words, (size_t)n_series * grid.Tw * 4);
  return s.end([&] {
    const int rc = timestamp ? b2p_instant_timestamp_dev(c, start, end, interval, lookback, offset, in.ts, in.offsets,
                                                         n_rows, n_series, d_out, d_valid)
                             : b2p_instant_select_dev(c, start, end, interval, lookback, offset, in.ts, in.val,
                                                      in.offsets, n_rows, n_series, d_out, d_valid);
    return rc ? rc : b2p_sync(c);
  });
}

extern "C" {

int b2p_instant_select(b2p_ctx* c, int64_t start, int64_t end, int64_t interval, int64_t lookback, int64_t offset,
                       const int64_t* ts, const double* val, const uint32_t* sid, const uint64_t* offsets_host,
                       uint64_t n_rows, uint32_t n_series, double* out, uint32_t* valid_words) {
  return instant_select_host(c, start, end, interval, lookback, offset, ts, val, sid, offsets_host, n_rows, n_series,
                             out, valid_words, false);
}

int b2p_instant_timestamp(b2p_ctx* c, int64_t start, int64_t end, int64_t interval, int64_t lookback, int64_t offset,
                          const int64_t* ts, const uint32_t* sid, const uint64_t* offsets_host, uint64_t n_rows,
                          uint32_t n_series, double* out, uint32_t* valid_words) {
  return instant_select_host(c, start, end, interval, lookback, offset, ts, nullptr, sid, offsets_host, n_rows,
                             n_series, out, valid_words, true);
}

}  // extern "C"

namespace {
// The device copies of a multi-field host call over a [n_series x T] grid: the timestamps and series offsets, the value
// columns, their NULL bitmaps (none when field_valid is NULL), the result grids and the validity bitmap.
struct FieldsIn {
  SeriesIn series;
  const double* vals[kMaxFields];
  const uint8_t* nulls[kMaxFields] = {};
  double* outs[kMaxFields];
  uint32_t* valid;
};
FieldsIn stage_fields(Staging& s, const int64_t* ts, const double* const* vals, const uint8_t* const* field_valid,
                      int32_t n_fields, const uint32_t* sid, const uint64_t* offsets_host, uint64_t n_rows,
                      uint32_t n_series, int64_t T, double* const* outs, uint32_t* valid_words) {
  FieldsIn f;
  f.series = stage_series(s, ts, nullptr, sid, 0u, offsets_host, n_rows, n_series);
  s.in_cols(vals, n_fields, n_rows * 8, f.vals);
  if (field_valid) s.in_cols(field_valid, n_fields, (n_rows + 7) / 8, f.nulls);
  s.out_cols(outs, n_fields, (size_t)n_series * (size_t)T * 8, f.outs);
  f.valid = s.out(valid_words, (size_t)n_series * (size_t)((T + 31) / 32) * 4);
  return f;
}
}  // namespace

extern "C" {

int b2p_range_eval_fields(b2p_ctx* c, const b2p_range_params* p, const int64_t* ts, const double* const* vals,
                          const uint8_t* const* field_valid, int32_t n_fields, const uint32_t* sid,
                          const uint64_t* offsets_host, uint64_t n_rows, uint32_t n_series, double* const* outs, uint32_t* valid_words) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  int64_t T = 0;
  if (int rc = check_grid(p, n_series, &T)) return rc;
  if (int rc = check_fields(vals, outs, n_fields)) return rc;
  if (n_series == 0 || T == 0) return B2P_OK;  // (no sample copies, no series offsets)
  DeviceGuard g(c->device);
  Staging s{c};
  const FieldsIn f =
      stage_fields(s, ts, vals, field_valid, n_fields, sid, offsets_host, n_rows, n_series, T, outs, valid_words);
  return s.end([&] {
    const int rc = b2p_range_eval_fields_dev(c, p, f.series.ts, f.vals, field_valid ? f.nulls : nullptr, n_fields,
                                             f.series.offsets, n_rows, n_series, f.outs, f.valid);
    return rc ? rc : b2p_sync(c);
  });
}

}  // extern "C"

namespace {
int instant_select_fields_host(b2p_ctx* c, int64_t start, int64_t end, int64_t interval, int64_t lookback,
                               int64_t offset, const int64_t* ts, const double* const* vals,
                               const uint8_t* const* field_valid, int32_t n_fields, const uint32_t* sid,
                               const uint64_t* offsets_host, uint64_t n_rows, uint32_t n_series, double* const* outs,
                               uint32_t* valid_words, bool i64) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  InstantArgs grid;
  if (int rc = instant_grid(start, end, interval, lookback, offset, n_series, &grid)) return rc;
  if (int rc = check_fields(vals, outs, n_fields)) return rc;
  if (n_series == 0 || grid.T == 0) return B2P_OK;  // (no sample copies, no series offsets)
  DeviceGuard g(c->device);
  Staging s{c};
  const FieldsIn f =
      stage_fields(s, ts, vals, field_valid, n_fields, sid, offsets_host, n_rows, n_series, grid.T, outs, valid_words);
  return s.end([&] {
    const int rc = instant_select_fields(c, start, end, interval, lookback, offset, f.series.ts, f.vals,
                                         field_valid ? f.nulls : nullptr, n_fields, f.series.offsets, n_rows, n_series,
                                         f.outs, f.valid, i64);
    return rc ? rc : b2p_sync(c);
  });
}
}  // namespace

extern "C" {

int b2p_instant_select_fields(b2p_ctx* c, int64_t start, int64_t end, int64_t interval, int64_t lookback,
                              int64_t offset, const int64_t* ts, const double* const* vals,
                              const uint8_t* const* field_valid, int32_t n_fields, const uint32_t* sid,
                              const uint64_t* offsets_host, uint64_t n_rows, uint32_t n_series, double* const* outs, uint32_t* valid_words) {
  return instant_select_fields_host(c, start, end, interval, lookback, offset, ts, vals, field_valid, n_fields, sid,
                                    offsets_host, n_rows, n_series, outs, valid_words, false);
}

int b2p_instant_select_fields_i64(b2p_ctx* c, int64_t start, int64_t end, int64_t interval, int64_t lookback,
                                  int64_t offset, const int64_t* ts, const double* const* vals,
                                  const uint8_t* const* field_valid, int32_t n_fields, const uint32_t* sid,
                                  const uint64_t* offsets_host, uint64_t n_rows, uint32_t n_series,
                                  double* const* outs, uint32_t* valid_words) {
  return instant_select_fields_host(c, start, end, interval, lookback, offset, ts, vals, field_valid, n_fields, sid,
                                    offsets_host, n_rows, n_series, outs, valid_words, true);
}

int b2p_subquery(b2p_ctx* c, const b2p_range_params* p, int64_t inner_start, int64_t inner_interval, const double* vals,
                 const uint32_t* valid, uint32_t n_rows, uint64_t T_inner, double* out, uint32_t* out_valid) {
  if (!c) return fail(B2P_E_INVALID, "ctx is NULL");
  int64_t T = 0;
  if (int rc = check_grid(p, n_rows, &T)) return rc;
  DeviceGuard g(c->device);
  const size_t Tw_in = (size_t)((T_inner + 31) / 32), Tw = (size_t)((T + 31) / 32);
  Staging s{c};
  const double* d_vals = s.in(vals, (size_t)n_rows * T_inner * 8);
  const uint32_t* d_valid = s.in(valid, (size_t)n_rows * Tw_in * 4);
  double* d_out = s.out(out, (size_t)n_rows * (size_t)T * 8);
  uint32_t* d_valid_out = s.out(out_valid, (size_t)n_rows * Tw * 4);
  return s.end([&] {
    const int rc = b2p_subquery_dev(c, p, inner_start, inner_interval, d_vals, d_valid, n_rows, T_inner, d_out,
                                    d_valid_out);
    return rc ? rc : b2p_sync(c);
  });
}

}  // extern "C"
