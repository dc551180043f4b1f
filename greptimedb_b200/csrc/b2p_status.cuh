// b2p_status.cuh — the device-side status block and the argument block of a range call: plain structs, no kernels, so
// that every kernel header and the host runtime can include them.
#pragma once
#include <cstdint>

namespace b2p {

// Device-side status block, reset before every range/instant call.
struct Status {
  uint32_t slow_count;      // series deferred to the slow path          (reset per range call)
  uint32_t arena_overflow;  // slow-path arena too small                 (reset per range call)
  uint32_t k0_errors;       // bit0: sid not sorted, bit1: sid >= n_series (reset per K0 call); the bits below
  uint32_t w_count;         // series the first tier handed to the warp-per-series kernel
  uint32_t b_count;         // series the warp-per-series kernel handed to its long-window (big ring) instantiation
  uint32_t g_next;          // fused by-label partials: next group (relative to g_lo) a first-tier warp takes
  uint32_t uniform;         // cadence_probe_kernel's verdict: != 0 => the uniform-cadence variant of the first tier runs
  unsigned long long arena_used;    // (unused since the arena is split into per-warp regions)
  unsigned long long arena_needed;  // arena rows that make a region large enough for the longest deferred series
  // a tiled call (all-reduced sum by) resets slow_count / w_count per tile: the counts of its earlier tiles
  uint32_t slow_tiles;
  uint32_t w_tiles;
};

// Status::k0_errors bits of the operators above the range functions
constexpr uint32_t kBinRowError = 4u;          // binary operator: a pair's row index >= the operand's row count
constexpr uint32_t kSetKeyError = 8u;          // set operator: a row's key is >= n_keys and not B2P_NO_KEY
constexpr uint32_t kScalarKeyError = 16u;      // scalar(): a row key >= n_rows and not B2P_NO_KEY
constexpr uint32_t kScalarOverlapError = 32u;  // scalar(): two rows of one key have a cell at one step
constexpr uint32_t kStepRangeError = 64u;      // step function (K19): an eval timestamp outside the calendar's years

struct RangeArgs {
  // query
  int64_t start, end, interval, range, offset;
  double p0, p1;
  int32_t filter_nan;
  int64_t T;    // global eval steps
  uint32_t Tw;  // validity words per series
  // derived (host): 32-bit time domain of the fast kernel and exact-division helper
  int64_t tb;        // start - range: origin of the uint32 timestamps
  uint32_t rel_max;  // range + (T-1)*interval + 1: clamp for samples after `end`
  double rcp_rs;     // RN(1/(range/1000)) when the Markstein division is exact for it, else 0
  double range_secs; // (double)range / 1000.0
  double rcp_interval; // 1.0 / interval
  uint32_t start_mod;  // start mod interval (lean tier's end trim; valid when start >= 0)
  // input
  const int64_t* ts;
  const double* val;
  const uint64_t* offsets;
  uint64_t n_rows;
  uint32_t n_series;
  // output
  double* out;
  uint32_t* valid;
  // tier hand-off: when use_w_list != 0 the warp-per-series kernel only runs the series in w_list
  uint32_t* w_list;
  int32_t use_w_list;  // 0: all series; 1: the series in w_list (w_count); 2: the series in b_list (b_count)
  uint32_t* b_list;    // long-window hand-off: series whose windows do not fit the 256-sample ring
  // Fused by-label SUM / COUNT partials (sum by (..)(rate(..)) without the [n_series x T] intermediate): when gsum
  // != nullptr results are not stored per series but added into gsum / gcnt [n_groups x T].  The first tier walks
  // the series group by group (CSR g_off / g_members, groups [g_lo, g_hi) dealt round-robin to the warps), so a
  // group's rows belong to one warp and are updated by plain read-modify-write in member order; the later tiers
  // add the series handed to them with atomics (group of series s = gid[s]).
  double* gsum;
  uint32_t* gcnt;
  const uint32_t* gid;
  const uint32_t* g_off;      // [n_groups + 1]
  const uint32_t* g_members;  // [n_series] series ids ordered by (group, series id)
  uint32_t n_groups, g_lo, g_hi;
  // a tier that hands a series on after it has already added some of its steps to the partials passes the number of
  // steps it committed along (parallel to the work lists); the next tier evaluates the series but only adds the rest
  uint32_t* w_skip;
  uint32_t* b_skip;
  uint32_t* slow_skip;
  // slow path plumbing
  Status* status;
  uint32_t* slow_list;
  int64_t* arena_ts;
  double* arena_val;
  unsigned long long arena_cap;
  unsigned long long* win_scratch;  // [slow warps][T] packed (off | len<<32)
};

}  // namespace b2p
