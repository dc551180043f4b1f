// b2p_quantile.cuh — PromQL `quantile(φ, v)` over a dense [rows x T] grid whose rows are grouped by a b2p_group_index:
//   K11 quantile_resident_kernel  per (group of at most kQuantResident members, 32-step tile), lane = step: one read,
//                                 each lane's keys stashed in shared memory and sorted there.  With a φ outside
//                                 [0, 1] (or NaN) it takes every group and only counts.
//       quantile_pass_kernel      larger groups, per (member chunk, 32-step tile): one MSB radix-select pass
//       quantile_advance_kernel   groups of several chunks, per (group, step): the pass's summed histogram -> the next
//                                 prefix, and the result once both order statistics are known
// The digit width B is a template parameter of the select: 8 bits on one GPU (each pass is a read of the cells, so
// few passes win), 4 bits over sharded rows (each pass all-reduces 2^B counters per (group, step), so few bins win; see
// "Sharded rows" below).
//
// The reference's QuantileAccumulator::evaluate (src/promql/src/functions/quantile_aggr.rs:110-116) calls
// quantile_with_scratch (quantile.rs:201-225): NaN for φ NaN, -inf for φ < 0, +inf for φ > 1; otherwise the n valid
// cells sorted by f64::total_cmp, rank = φ (n - 1), lo = floor(rank), hi = min(n - 1, lo + 1), w = rank - floor(rank),
// result s[lo] (1 - w) + s[hi] w.  That expression is evaluated as written, with no shortcut at w == 0 (so
// quantile(0, {1, +inf}) is NaN, as inf * 0 is) and no fused multiply-add.  The two order statistics are selected
// exactly on the 64-bit total-order key, so the result is the reference's bit for bit.
//
// Selection on the unsigned key u = total_key(v) ^ 2^63, 64 / B B-bit digits from the top.  Per (group, step) the state
// is a prefix of `level` fixed digits and lo's rank k among the keys under it:
//   kQSelect   s[lo] and s[hi] lie under the same prefix: a pass histograms the next digit of the keys under it, the
//              scan places rank k and k + 1.  Same bin: one more digit is fixed.  Different bins: s[lo] is the largest
//              key of its bin and s[hi] the smallest of the next non-empty one (kQExtreme).  lo = n - 1 (hi = lo) is
//              kQExtreme at once: s[lo] is the largest key.
//   kQExtreme  a pass takes the largest key under p_lo and the smallest under p_hi (registers, atomicMax / atomicMin
//              across chunks): kQDone.
// So a (group, step) is done after at most 64 / B + 1 passes; a group split into chunks sums 16-bit per-warp histograms
// into 32-bit integer counters, so every order of the atomics gives the same bits.
//
// Sharded rows (B = kQuantShardBits): a rank is one more set of chunks.  Every group of a batch of (group, tile) units
// has a slot, with or without local members, and no rank finishes a group alone (no whole-chunk path): each pass the
// rank's chunks add their counts into the batch's block ([unit][16][32] u32 counts, then [unit][32] u64 largest key
// under p_lo and [unit][32] u64 smallest key under p_hi), the blocks of every rank are summed / maxed / minned (an
// all-reduce, or the advance over n_blocks blocks), and every rank advances an identical state from the merged block.
// Counts add in any order, so the result is the bits of the single-rank select over the union of the rows.
#pragma once
#include <cstdint>

#include "b2p_window.cuh"

namespace b2p {

constexpr uint32_t kQuantResident = 64;     // largest group of the resident path (keys per lane in shared memory)
constexpr uint32_t kQuantWarps = 4;         // warps per CTA of the resident and pass kernels
constexpr uint32_t kQuantChunkMax = 32768;  // members per chunk: a lane's 16-bit bin counter cannot overflow
constexpr uint32_t kQuantNone = 0xFFFFFFFFu;
constexpr uint32_t kQuantPasses = 9;        // eight 8-bit digits, then one extreme pass
constexpr uint32_t kQuantShardBits = 4;     // digit width of the sharded select: 16 bins
constexpr uint32_t kQuantShardPasses = 17;  // sixteen 4-bit digits, then one extreme pass
static_assert(kQuantPasses == 64 / 8 + 1 && kQuantShardPasses == 64 / kQuantShardBits + 1,
              "a (group, step) takes at most one pass per digit and one extreme pass");
constexpr uint32_t kQSelect = 0, kQExtreme = 1, kQDone = 2;

// A run [begin, end) of one large group's member positions; slot: the group's state block (groups of several chunks)
// or kQuantNone (the chunk is the whole group and is finished by one warp in one launch)
struct QuantChunk { uint32_t begin, end, group, slot; };

// Selection state of one (group, step).  At kQDone p_lo / p_hi are the keys of s[lo] / s[hi].
struct QuantState {
  unsigned long long p_lo, p_hi;
  unsigned long long r_lo, r_hi;  // kQExtreme across chunks: largest key under p_lo, smallest under p_hi
  uint32_t k, level, n, mode, eq, pad;
};
static_assert(sizeof(QuantState) == 56, "quantile_run states the scratch bound with 56 B per (group, step)");

struct QuantArgs {
  const double* vals;      // [rows x T]
  const uint32_t* valid;   // [rows x Tw]
  const uint32_t* goff;    // [G + 1]
  const uint32_t* members; // [n_series]
  uint32_t n_groups;
  const QuantChunk* chunks;
  uint32_t n_chunks;
  const uint32_t* slot_group;  // [slot] its group
  uint32_t n_slots;
  uint64_t T;
  uint32_t Tw, tiles;
  double phi;
  int count_only;          // φ NaN, < 0 or > 1: the result depends on the count alone
  int pass;
  QuantState* state;       // [slot][T]
  uint32_t* hist;          // [slot][tile][256][32]
  double* out_val;         // [G x T]
  uint32_t* out_cnt;       // [G x T]
  // sharded select only (B = kQuantShardBits): slot s is group group0 + s and covers tiles [tile0, tile0 + tiles); the
  // state is [slot][tile][32], hist / r_lo / r_hi are the block's sections; the advance reads n_blocks blocks
  // block_stride bytes apart and adds the cells it leaves unfinished to *live
  uint32_t tile0, group0;
  unsigned long long* r_lo;  // [unit][32] largest key under p_lo (reduced by MAX)
  unsigned long long* r_hi;  // [unit][32] smallest key under p_hi (reduced by MIN)
  uint64_t block_stride;
  uint32_t n_blocks;
  unsigned long long* live;
};

// Shared memory per warp: the resident stash [kQuantResident][32] keys, or the pass histogram [128][32] words of two
// 16-bit bins each (bin b of a lane: word (b >> 1) * 32 + lane, half b & 1)
constexpr size_t kQuantWarpBytes = (size_t)kQuantResident * 32 * 8;
static_assert(kQuantWarpBytes >= 128 * 32 * 4, "the histogram must fit the warp's shared memory");
// Shared memory per warp of quantile_pass_kernel<B>: the sharded select needs only its 2^B / 2 histogram words per lane
template <uint32_t B>
__host__ __device__ constexpr size_t quant_pass_warp_bytes() { return B == 8 ? kQuantWarpBytes : (size_t)(1u << B) / 2 * 32 * 4; }

__device__ __forceinline__ unsigned long long quant_key(double v) { return F64Key::key(v); }
__device__ __forceinline__ double quant_value(unsigned long long u) { return F64Key::value(u); }
// lo = floor(φ (n - 1)), n >= 1 and 0 <= φ <= 1
__device__ __forceinline__ uint32_t quant_lo(double phi, uint32_t n) {
  const double f = floor(__dmul_rn(phi, (double)(n - 1)));
  return min((uint32_t)f, n - 1);
}
// s[lo] (1 - w) + s[hi] w as the reference evaluates it (no contraction into FMA); φ outside [0, 1] or NaN
// gives -inf / +inf / NaN
__device__ __forceinline__ double quant_result(double phi, uint32_t n, unsigned long long klo, unsigned long long khi) {
  if (phi != phi) return __longlong_as_double(0x7ff8000000000000ll);
  if (phi < 0.0) return -__longlong_as_double(0x7ff0000000000000ll);
  if (phi > 1.0) return __longlong_as_double(0x7ff0000000000000ll);
  const double rank = __dmul_rn(phi, (double)(n - 1));
  const double w = __dsub_rn(rank, floor(rank));
  return __dadd_rn(__dmul_rn(quant_value(klo), __dsub_rn(1.0, w)), __dmul_rn(quant_value(khi), w));
}

// Streams the keys of the valid cells of members [begin, end) at this lane's step of `tile` into f(key): 32 member ids
// and validity words per coalesced load, kAhead 256-byte value segments in flight.  Warp-uniform.
template <class F>
__device__ __forceinline__ void quant_stream(const QuantArgs& a, uint32_t begin, uint32_t end, uint32_t tile, int lane,
                                             bool want, F f) {
  constexpr uint32_t kAhead = 8;
  const uint64_t step = (uint64_t)tile * 32 + lane;
  for (uint32_t m0 = begin; m0 < end; m0 += 32) {
    const uint32_t j = m0 + lane;
    const bool in = j < end;
    const uint32_t row = in ? __ldg(a.members + j) : 0u;
    const uint32_t w = in ? __ldg(a.valid + (uint64_t)row * a.Tw + tile) : 0u;
    const uint32_t nb = min(32u, end - m0);
    for (uint32_t i0 = 0; i0 < nb; i0 += kAhead) {
      double v[kAhead];
      bool on[kAhead];
#pragma unroll
      for (uint32_t q = 0; q < kAhead; ++q) {
        const uint32_t i = i0 + q;
        const uint32_t r = __shfl_sync(0xFFFFFFFFu, row, i & 31);
        const uint32_t wq = __shfl_sync(0xFFFFFFFFu, w, i & 31);
        on[q] = want && i < nb && ((wq >> lane) & 1u);
        v[q] = on[q] ? __ldg(a.vals + (uint64_t)r * a.T + step) : 0.0;
      }
#pragma unroll
      for (uint32_t q = 0; q < kAhead; ++q)
        if (on[q]) f(quant_key(v[q]));
    }
  }
}

// u shares the first `level` B-bit digits of p
template <uint32_t B>
__device__ __forceinline__ bool quant_under(unsigned long long u, unsigned long long p, uint32_t level) {
  return level == 0 || (u >> (64 - B * level)) == (p >> (64 - B * level));
}

// One pass's work on a key: the digit's bin (kQSelect) or the extremes (kQExtreme).  h: the lane's histogram words.
template <uint32_t B>
__device__ __forceinline__ void quant_visit(const QuantState& st, unsigned long long u, uint32_t* h,
                                            unsigned long long& mx, unsigned long long& mn) {
  if (st.mode == kQSelect) {
    if (quant_under<B>(u, st.p_lo, st.level)) {
      const uint32_t b = (uint32_t)(u >> (64 - B - B * st.level)) & ((1u << B) - 1);
      h[(b >> 1) * 32] += 1u << ((b & 1u) * 16);
    }
  } else if (st.mode == kQExtreme) {
    if (quant_under<B>(u, st.p_lo, st.level) && u > mx) mx = u;
    if (!st.eq && quant_under<B>(u, st.p_hi, st.level) && u < mn) mn = u;
  }
}

// After a kQSelect pass at st.level with the lane's histogram bin(b): the next state (see the top of the file)
template <uint32_t B, class Bin>
__device__ __forceinline__ void quant_advance(QuantState& st, double phi, Bin bin) {
  constexpr uint32_t kBins = 1u << B, kLevels = 64 / B;
  if (st.level == 0) {
    uint32_t n = 0;
    for (uint32_t b = 0; b < kBins; ++b) n += bin(b);
    st.n = n;
    if (n == 0) { st.mode = kQDone; return; }
    st.k = quant_lo(phi, n);
    if (st.k == n - 1) {  // hi = lo: the largest key
      st.mode = kQExtreme; st.eq = 1; st.r_lo = 0ull; st.r_hi = ~0ull;
      return;
    }
  }
  const uint32_t k1 = st.k + 1;
  uint32_t cum = 0, blo = kBins, bhi = kBins - 1, klo = 0;
  for (uint32_t b = 0; b < kBins; ++b) {
    const uint32_t c = bin(b);
    if (blo == kBins && cum + c > st.k) { blo = b; klo = st.k - cum; }
    if (cum + c > k1) { bhi = b; break; }
    cum += c;
  }
  const uint32_t shift = 64 - B - B * st.level;
  st.p_hi = st.p_lo | ((unsigned long long)bhi << shift);
  st.p_lo |= (unsigned long long)blo << shift;
  st.k = klo;
  ++st.level;
  if (blo == bhi) {
    if (st.level == kLevels) { st.p_hi = st.p_lo; st.mode = kQDone; }
  } else {
    st.mode = st.level == kLevels ? kQDone : kQExtreme;
    st.r_lo = 0ull; st.r_hi = ~0ull;
  }
}
__device__ __forceinline__ void quant_finish_extreme(QuantState& st, unsigned long long mx, unsigned long long mn) {
  st.p_lo = mx;
  st.p_hi = st.eq ? mx : mn;
  st.mode = kQDone;
}
__device__ __forceinline__ void quant_write(const QuantArgs& a, uint32_t g, uint64_t step, const QuantState& st) {
  const uint64_t o = (uint64_t)g * a.T + step;
  a.out_val[o] = st.n ? quant_result(a.phi, st.n, st.p_lo, st.p_hi) : 0.0;
  a.out_cnt[o] = st.n;
}

// One warp per (group, tile) over every group of at most kQuantResident members (every group when count_only).
// Lane = step: the lane's keys go to its stash column in member order, an insertion sort orders them.
__global__ void __launch_bounds__(kQuantWarps * 32) quantile_resident_kernel(const QuantArgs a) {
  extern __shared__ __align__(16) unsigned char quant_smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned long long* s = reinterpret_cast<unsigned long long*>(quant_smem + (size_t)warp * kQuantWarpBytes) + lane;
  const uint64_t units = (uint64_t)a.n_groups * a.tiles;
  const uint64_t n_warps = (uint64_t)gridDim.x * kQuantWarps;
  for (uint64_t u = (uint64_t)blockIdx.x * kQuantWarps + warp; u < units; u += n_warps) {
    const uint32_t g = (uint32_t)(u / a.tiles), tile = (uint32_t)(u - (uint64_t)g * a.tiles);
    const uint32_t b = __ldg(a.goff + g), e = __ldg(a.goff + g + 1);
    if (!a.count_only && e - b > kQuantResident) continue;
    const uint64_t step = (uint64_t)tile * 32 + lane;
    const bool live = step < a.T;
    uint32_t n = 0;
    quant_stream(a, b, e, tile, lane, live, [&](unsigned long long key) {
      if (!a.count_only) s[n * 32] = key;
      ++n;
    });
    if (!live) continue;
    QuantState st{};
    st.n = n;
    if (n && !a.count_only) {
      for (uint32_t i = 1; i < n; ++i) {
        const unsigned long long x = s[i * 32];
        uint32_t j = i;
        for (; j > 0 && s[(j - 1) * 32] > x; --j) s[j * 32] = s[(j - 1) * 32];
        s[j * 32] = x;
      }
      const uint32_t lo = quant_lo(a.phi, n);
      st.p_lo = s[lo * 32];
      st.p_hi = s[min(lo + 1, n - 1) * 32];
    }
    quant_write(a, g, step, st);
  }
}

// One warp per (chunk of a group of more than kQuantResident members, tile).  A whole-group chunk (slot kQuantNone)
// runs every pass here in registers at pass 0 and writes its result; a chunk of a larger group does pass a.pass on the
// group's state and adds its histogram (or its extremes) into the group's counters for quantile_advance_kernel.
// Sharded (B = kQuantShardBits): every chunk is of the second kind, its slot a group of the batch, its tile a tile of
// the batch, and the counters are the rank's block.
template <uint32_t B>
__global__ void __launch_bounds__(kQuantWarps * 32, 1) quantile_pass_kernel(const QuantArgs a) {
  constexpr bool kShard = B == kQuantShardBits;
  constexpr uint32_t kBins = 1u << B;
  extern __shared__ __align__(16) unsigned char quant_smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t* h = reinterpret_cast<uint32_t*>(quant_smem + (size_t)warp * quant_pass_warp_bytes<B>()) + lane;
  const uint64_t units = (uint64_t)a.n_chunks * a.tiles;
  const uint64_t n_warps = (uint64_t)gridDim.x * kQuantWarps;
  for (uint64_t u = (uint64_t)blockIdx.x * kQuantWarps + warp; u < units; u += n_warps) {
    const uint32_t c = (uint32_t)(u / a.tiles), tile = (uint32_t)(u - (uint64_t)c * a.tiles);
    const QuantChunk ch = a.chunks[c];
    const bool whole = !kShard && ch.slot == kQuantNone;
    if (whole && a.pass != 0) continue;
    const uint32_t gtile = kShard ? a.tile0 + tile : tile;  // the tile of the grid
    const uint64_t step = (uint64_t)gtile * 32 + lane;
    const bool live = step < a.T;
    const uint64_t si = kShard ? ((uint64_t)ch.slot * a.tiles + tile) * 32 + lane
                               : (uint64_t)(whole ? 0u : ch.slot) * a.T + step;
    QuantState st{};
    if (!live) st.mode = kQDone;
    else if (!whole) st = a.state[si];
#pragma unroll 1
    for (uint32_t p = 0; p < kQuantPasses; ++p) {
      const bool active = st.mode != kQDone;
      if (!__any_sync(0xFFFFFFFFu, active)) break;
      if (st.mode == kQSelect)
        for (uint32_t i = 0; i < kBins / 2; ++i) h[i * 32] = 0u;
      unsigned long long mx = 0ull, mn = ~0ull;
      quant_stream(a, ch.begin, ch.end, gtile, lane, active,
                   [&](unsigned long long key) { quant_visit<B>(st, key, h, mx, mn); });
      if (!whole) {  // into the group's counters
        if (st.mode == kQSelect) {
          uint32_t* gh = a.hist + ((uint64_t)ch.slot * a.tiles + tile) * kBins * 32 + lane;
          for (uint32_t i = 0; i < kBins / 2; ++i) {
            const uint32_t w = h[i * 32];
            if (w & 0xFFFFu) atomicAdd(gh + (2 * i) * 32, w & 0xFFFFu);
            if (w >> 16) atomicAdd(gh + (2 * i + 1) * 32, w >> 16);
          }
        } else if (st.mode == kQExtreme) {
          atomicMax(kShard ? a.r_lo + si : &a.state[si].r_lo, mx);
          if (!st.eq) atomicMin(kShard ? a.r_hi + si : &a.state[si].r_hi, mn);
        }
        break;
      }
      if (st.mode == kQSelect) quant_advance<B>(st, a.phi, [&](uint32_t b) { return (h[(b >> 1) * 32] >> ((b & 1u) * 16)) & 0xFFFFu; });
      else if (st.mode == kQExtreme) quant_finish_extreme(st, mx, mn);
    }
    if (whole && live) quant_write(a, ch.group, step, st);
  }
}

// One thread per (slot, step) of the groups of several chunks, after each pass: the summed histogram (cleared for the
// next pass) or extremes advance the state; a finished (group, step) writes its result.
// Sharded (B = kQuantShardBits): one thread per (slot, batch step); the counts are summed and the extremes maxed /
// minned over the n_blocks blocks (the ranks' blocks, or one all-reduced block), which read nothing of the rank, so
// every rank reaches the same state.  φ outside [0, 1] finishes at the level-0 count.  The unfinished cells are
// counted into *live.
template <uint32_t B>
__global__ void __launch_bounds__(256) quantile_advance_kernel(const QuantArgs a) {
  constexpr bool kShard = B == kQuantShardBits;
  constexpr uint32_t kBins = 1u << B;
  const uint64_t n = (uint64_t)a.n_slots * (kShard ? (uint64_t)a.tiles * 32 : a.T);
  uint32_t left = 0;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    QuantState st = a.state[i];
    if (st.mode == kQDone) continue;
    if constexpr (kShard) {
      const uint64_t unit = i / 32;
      const uint32_t slot = (uint32_t)(unit / a.tiles), tile = (uint32_t)(unit - (uint64_t)slot * a.tiles);
      const uint64_t step = (uint64_t)(a.tile0 + tile) * 32 + (i & 31);
      if (step >= a.T) continue;
      const char* blk = reinterpret_cast<const char*>(a.hist);
      if (st.mode == kQSelect) {
        const uint64_t h0 = (unit * kBins * 32 + (i & 31)) * 4;
        auto bin = [&](uint32_t b) {
          uint32_t s = 0;
          for (uint32_t k = 0; k < a.n_blocks; ++k)
            s += *reinterpret_cast<const uint32_t*>(blk + k * a.block_stride + h0 + (uint64_t)b * 32 * 4);
          return s;
        };
        if (a.count_only) {
          for (uint32_t b = 0; b < kBins; ++b) st.n += bin(b);
          st.mode = kQDone;
        } else {
          quant_advance<B>(st, a.phi, bin);
        }
      } else {
        const uint64_t lo0 = reinterpret_cast<const char*>(a.r_lo + i) - blk, hi0 = reinterpret_cast<const char*>(a.r_hi + i) - blk;
        unsigned long long mx = 0ull, mn = ~0ull;
        for (uint32_t k = 0; k < a.n_blocks; ++k) {
          mx = max(mx, *reinterpret_cast<const unsigned long long*>(blk + k * a.block_stride + lo0));
          mn = min(mn, *reinterpret_cast<const unsigned long long*>(blk + k * a.block_stride + hi0));
        }
        quant_finish_extreme(st, mx, mn);
      }
      a.state[i] = st;
      if (st.mode == kQDone) quant_write(a, a.group0 + slot, step, st);
      else ++left;
    } else {
      const uint32_t slot = (uint32_t)(i / a.T);
      const uint64_t step = i - (uint64_t)slot * a.T;
      if (st.mode == kQSelect) {
        uint32_t* gh = a.hist + ((uint64_t)slot * a.tiles + step / 32) * kBins * 32 + (step & 31);
        quant_advance<B>(st, a.phi, [&](uint32_t b) { return gh[b * 32]; });
        for (uint32_t b = 0; b < kBins; ++b) gh[b * 32] = 0u;
      } else {
        quant_finish_extreme(st, st.r_lo, st.r_hi);
      }
      a.state[i] = st;
      if (st.mode == kQDone) quant_write(a, a.slot_group[slot], step, st);
    }
  }
  if constexpr (kShard) {
    left = __reduce_add_sync(0xFFFFFFFFu, left);
    if ((threadIdx.x & 31) == 0 && left) atomicAdd(a.live, (unsigned long long)left);
  }
}

}  // namespace b2p
