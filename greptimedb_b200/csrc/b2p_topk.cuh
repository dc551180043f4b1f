// b2p_topk.cuh — PromQL `topk` / `bottomk` over a dense [rows x T] grid whose rows are grouped by a b2p_group_index:
//   K10 topk_chunk_kernel   per (member chunk, 32-step tile), lane = step: the chunk's best cells in a per-lane heap
//       topk_merge_kernel   per (group spanning several chunks, tile): merges the chunks' candidate lists
//       topk_mark_kernel    per (chunk of such a group, tile): the kept candidates -> the chunk's validity words
//       topk_select_kernel  general path (kk > kTopkMax): per (chunk, tile), the words from the selected threshold
//       topk_copy_kernel    kk >= largest group (every valid cell is kept), and rows whose group id is out of range
//
// The reference plans topk / bottomk as Window(row_number() OVER (PARTITION BY group labels, ts ORDER BY value, tags))
// -> Filter(row_number <= k) (src/query/src/promql/planner.rs:454-541, 2963-3016).  Per (group, step) the cells are
// ranked by (value in the f64 total order, tie), descending for topk and ascending for bottomk, where tie [rows] is one
// distinct ordinal per row that the caller derives from the label tuples (b2p_plan.cpp).  That is a strict total
// order, so the kept set of a (group, step) is exactly its min(kk, valid cells) best cells.  Inside the kernels a
// cell's key is (hi, lo) = (total key, tie), bit-inverted for bottomk, so that "better" is always "larger".  The two
// kernels that read values take the key as a template parameter: F64Key, or I64Key for an Int64 grid (b2p_topk_i64).
//
// Only validity words are written: topk is a filter and every consumer reads a cell only where its bit is set.  The
// last pass of a (chunk, tile) writes the tile's word of every member row of the chunk, so no word has two writers and
// out_valid may be valid.  Bits at or past step T come out 0.
//
// Fast path (kk <= kTopkMax): each lane keeps a binary min-heap of its kk best (hi, lo, member position) in shared
// memory, laid out [slot][lane]; the heap's root sits in registers, so a cell that does not make the list costs one
// compare.  Members are streamed like K3 streams them: 32 member ids, validity words and ties per coalesced load,
// eight 256-byte value segments in flight.  A group whose only chunk is the whole group is finished in that pass.
// A larger group is split into chunks (about one warp unit per resident warp in all, so one group of 100 k rows does
// not run as 32 serial warps); each chunk leaves its list in scratch, topk_merge_kernel finds the kk-th best key of the
// group, and topk_mark_kernel turns the candidates at or above it into words, without reading the values again.
//
// General path (kTopkMax < kk < largest group): selection in rounds of kTopkMax.  Round j finds, per (group, step),
// the kTopkMax best keys below the previous round's smallest (the same chunk / merge kernels with a bound); after
// ceil(kk / kTopkMax) rounds the kk-th best key is known, and topk_select_kernel reads the values once more and keeps
// every cell at or above it.  Groups of at most kk members keep every valid cell and take no part in the rounds.
// Cost: ceil(kk / 32) + 1 reads of the group's cells; measured in DESIGN.md section 4.
//
// Sharded (b2p_topk_shard_*, b2p_topk_allgather_dev): a rank is one more kind of chunk.  The chunk kernel leaves each
// local chunk's list, topk_merge_kernel in export mode (x_hi set) writes the rank's best K of a group below the bound
// into a candidate block instead of taking a verdict, the blocks of every rank are gathered, and topk_merge_kernel
// with a stride (the groups of one block apart) takes the verdict over the ranks' blocks.  tile0 shifts every kernel
// to tiles [tile0, tile0 + tiles), so scratch and blocks cover one batch of tiles at a time.
#pragma once
#include <cstdint>

#include "b2p_window.cuh"

namespace b2p {

constexpr uint32_t kTopkMax = 32;          // largest kk of the fast path; the heap size of the general path's rounds
constexpr uint32_t kTopkWarps = 4;         // warps per CTA of the heap kernels
constexpr uint32_t kTopkMarkBlock = 512;   // member words a warp assembles in shared memory at a time
constexpr uint32_t kTopkNone = 0xFFFFFFFFu;
constexpr uint32_t kTopkBound = 1u;        // state flag: keys at or above (s_hi, s_lo) are taken, the rest is below
constexpr uint32_t kTopkAll = 2u;          // state flag: every valid cell of the (group, step) is kept

// A run [begin, end) of one group's member positions (b2p_group_index::members).  cand: the chunk's candidate block
// (groups of several chunks) or kTopkNone; state: the group's selection state (several chunks, or the general path)
// or kTopkNone.
struct TopkChunk { uint32_t begin, end, cand, state; };
// A group of several chunks: candidate blocks cand_begin, cand_begin + stride, .. below cand_end
struct TopkMerge { uint32_t cand_begin, cand_end, state, stride; };

struct TopkArgs {
  const double* vals;      // [rows x T]
  const uint32_t* valid;   // [rows x Tw]
  const uint32_t* members; // [n_series] member rows, grouped
  const uint32_t* tie;     // [rows]
  const TopkChunk* chunks;
  uint32_t n_chunks;
  const TopkMerge* merges;
  uint32_t n_merges;
  uint64_t T;
  uint32_t Tw, tiles;
  uint32_t tile0;          // the tiles run are [tile0, tile0 + tiles); scratch is indexed by tile - tile0
  uint32_t K;              // heap slots per lane: kk on the fast path, kTopkMax on the general path
  uint32_t kk;
  int bottom;
  int general;
  int round;               // general path: the round (the fast path is round 0 of one)
  // candidate lists of the chunks of multi-chunk groups: [cand][tile][slot][lane], counts [cand][tile][lane]
  unsigned long long* c_hi;
  uint32_t* c_lo;
  uint32_t* c_pos;
  uint32_t* c_n;
  // selection state per (state, tile, lane): the bound / threshold key, the count still to take, flags
  unsigned long long* s_hi;
  uint32_t* s_lo;
  uint32_t* s_rem;
  uint32_t* s_flags;
  uint32_t* out_valid;     // [rows x Tw]; may be valid
  // export mode of topk_merge_kernel (sharded): a merge's best K below the bound, [merge][tile][slot][lane], and their
  // count [merge][tile][lane], written instead of the verdict
  unsigned long long* x_hi;
  uint32_t* x_lo;
  uint32_t* x_n;
};

template <class Key>
__device__ __forceinline__ void topk_key(double v, uint32_t tie, int bottom, unsigned long long& hi, uint32_t& lo) {
  const unsigned long long k = Key::key(v);  // unsigned, order kept
  hi = bottom ? ~k : k;
  lo = bottom ? ~tie : tie;
}
__device__ __forceinline__ bool key_less(unsigned long long ah, uint32_t al, unsigned long long bh, uint32_t bl) {
  return ah < bh || (ah == bh && al < bl);
}

// One lane's min-heap of (hi, lo, pos) in shared memory, slot s at [s * 32] (the pointers are offset by the lane)
struct TopkHeap {
  unsigned long long* hi;
  uint32_t* lo;
  uint32_t* pos;
  __device__ __forceinline__ void put(uint32_t s, unsigned long long h, uint32_t l, uint32_t p) {
    hi[s * 32] = h; lo[s * 32] = l; pos[s * 32] = p;
  }
  __device__ __forceinline__ void move(uint32_t to, uint32_t from) { put(to, hi[from * 32], lo[from * 32], pos[from * 32]); }
  // places (h, l, p) at or below slot s of a heap of n entries whose slot s is free
  __device__ void sift_down(uint32_t s, uint32_t n, unsigned long long h, uint32_t l, uint32_t p) {
    for (;;) {
      uint32_t c = 2 * s + 1;
      if (c >= n) break;
      if (c + 1 < n && key_less(hi[(c + 1) * 32], lo[(c + 1) * 32], hi[c * 32], lo[c * 32])) ++c;
      if (!key_less(hi[c * 32], lo[c * 32], h, l)) break;
      move(s, c);
      s = c;
    }
    put(s, h, l, p);
  }
  __device__ void push(uint32_t& n, unsigned long long h, uint32_t l, uint32_t p) {
    uint32_t s = n++;
    while (s > 0) {
      const uint32_t up = (s - 1) / 2;
      if (!key_less(h, l, hi[up * 32], lo[up * 32])) break;
      move(s, up);
      s = up;
    }
    put(s, h, l, p);
  }
  __device__ void pop(uint32_t& n) {  // drops the smallest entry
    --n;
    if (n > 0) sift_down(0, n, hi[n * 32], lo[n * 32], pos[n * 32]);
  }
  // keeps (h, l, p) if it is among the K best seen; (th, tl) mirrors the root once the heap is full
  __device__ __forceinline__ void offer(uint32_t& n, uint32_t K, unsigned long long& th, uint32_t& tl,
                                        unsigned long long h, uint32_t l, uint32_t p) {
    if (n < K) {
      push(n, h, l, p);
      if (n == K) { th = hi[0]; tl = lo[0]; }
    } else if (key_less(th, tl, h, l)) {
      sift_down(0, n, h, l, p);
      th = hi[0]; tl = lo[0];
    }
  }
};

__device__ __forceinline__ TopkHeap topk_heap(unsigned char* smem, uint32_t K, size_t warp_bytes, int warp, int lane) {
  unsigned char* base = smem + (size_t)warp * warp_bytes;
  TopkHeap h;
  h.hi = reinterpret_cast<unsigned long long*>(base) + lane;
  h.lo = reinterpret_cast<uint32_t*>(base + (size_t)K * 32 * 8) + lane;
  h.pos = h.lo + (size_t)K * 32;
  return h;
}

// The selection state of one lane before a round: rem still to take, flags, the bound (hi, lo)
struct TopkState {
  uint32_t rem, flags;
  unsigned long long hi;
  uint32_t lo;
  __device__ __forceinline__ bool done() const { return rem == 0 || (flags & kTopkAll); }
};
__device__ __forceinline__ TopkState topk_state_load(const TopkArgs& a, uint64_t si) {
  if (a.round == 0) return TopkState{a.kk, 0u, 0ull, 0u};
  return TopkState{a.s_rem[si], a.s_flags[si], a.s_hi[si], a.s_lo[si]};
}
// The verdict of a round over the heap of the n (<= K) best keys below the bound: every remaining cell fits (All), or
// the rem-th best is the threshold (rem = 0), or all K are taken and the smallest of them bounds the next round
__device__ void topk_verdict(const TopkArgs& a, uint64_t si, TopkState st, TopkHeap& h, uint32_t n) {
  if (!st.done()) {
    if (n < a.K && n <= st.rem) {
      st.flags |= kTopkAll;
    } else if (st.rem <= n) {
      while (n > st.rem) h.pop(n);
      st.hi = h.hi[0]; st.lo = h.lo[0]; st.rem = 0;
    } else {
      st.rem -= a.K;
      st.hi = h.hi[0]; st.lo = h.lo[0]; st.flags |= kTopkBound;
    }
  }
  a.s_rem[si] = st.rem; a.s_flags[si] = st.flags; a.s_hi[si] = st.hi; a.s_lo[si] = st.lo;
}

// The words of members [begin, end) for one tile of the grid from a list of n kept-or-not entries (pos at [s * 32],
// lane-offset): keep(s) decides; a word has the bit of every lane whose list holds the member and keeps it
template <class Keep>
__device__ void topk_write_words(const TopkArgs& a, uint32_t* sw, const uint32_t* pos, uint32_t n, uint32_t begin,
                                 uint32_t end, uint32_t tile, int lane, Keep keep) {
  for (uint32_t b0 = begin; b0 < end; b0 += kTopkMarkBlock) {
    const uint32_t nb = min(kTopkMarkBlock, end - b0);
    for (uint32_t j = lane; j < nb; j += 32) sw[j] = 0u;
    __syncwarp();
    for (uint32_t s = 0; s < n; ++s) {
      const uint32_t p = pos[s * 32];
      if (p >= b0 && p - b0 < nb && keep(s)) atomicOr(&sw[p - b0], 1u << lane);
    }
    __syncwarp();
    for (uint32_t j = lane; j < nb; j += 32) a.out_valid[(uint64_t)__ldg(a.members + b0 + j) * a.Tw + tile] = sw[j];
    __syncwarp();
  }
}

// Streams the members of `ch` for one tile into the lane's heap (cells with want and below the bound, if any)
template <class Key>
__device__ __forceinline__ uint32_t topk_stream(const TopkArgs& a, const TopkChunk& ch, uint32_t tile, int lane,
                                                bool want, const TopkState& st, TopkHeap& h) {
  constexpr uint32_t kAhead = 8;
  const uint32_t gt = a.tile0 + tile;
  const uint64_t step = (uint64_t)gt * 32 + lane;
  const bool bounded = (st.flags & kTopkBound) != 0;
  uint32_t n = 0;
  unsigned long long th = 0;
  uint32_t tl = 0;
  if (!__any_sync(0xFFFFFFFFu, want)) return 0;
  for (uint32_t m0 = ch.begin; m0 < ch.end; m0 += 32) {
    const uint32_t j = m0 + lane;
    const bool in = j < ch.end;
    const uint32_t row = in ? __ldg(a.members + j) : 0u;
    const uint32_t w = in ? __ldg(a.valid + (uint64_t)row * a.Tw + gt) : 0u;
    const uint32_t t = in ? __ldg(a.tie + row) : 0u;
    const uint32_t nb = min(32u, ch.end - m0);
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
      for (uint32_t q = 0; q < kAhead; ++q) {
        const uint32_t tq = __shfl_sync(0xFFFFFFFFu, t, (i0 + q) & 31);
        if (!on[q]) continue;
        unsigned long long kh;
        uint32_t kl;
        topk_key<Key>(v[q], tq, a.bottom, kh, kl);
        if (bounded && !key_less(kh, kl, st.hi, st.lo)) continue;
        h.offer(n, a.K, th, tl, kh, kl, m0 + i0 + q);
      }
    }
  }
  return n;
}

// Dynamic shared memory per warp of topk_chunk_kernel / topk_merge_kernel
__host__ __device__ constexpr size_t topk_warp_bytes(uint32_t K) { return (size_t)K * 32 * 16 + kTopkMarkBlock * 4; }

// One warp per (chunk, tile).  Fast path: a single-chunk group writes its words here; a chunk of a larger group
// leaves its list.  General path: chunks of groups of at most kk members are skipped (topk_select_kernel copies their
// words), a single-chunk group takes its round's verdict here, a chunk of a larger group leaves its list.
template <class Key = F64Key>
__global__ void __launch_bounds__(kTopkWarps * 32) topk_chunk_kernel(const TopkArgs a) {
  extern __shared__ __align__(16) unsigned char topk_smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const size_t wb = topk_warp_bytes(a.K);
  TopkHeap h = topk_heap(topk_smem, a.K, wb, warp, lane);
  uint32_t* sw = reinterpret_cast<uint32_t*>(topk_smem + (size_t)warp * wb + (size_t)a.K * 32 * 16);
  const uint64_t units = (uint64_t)a.n_chunks * a.tiles;
  const uint64_t n_warps = (uint64_t)gridDim.x * kTopkWarps;
  for (uint64_t u = (uint64_t)blockIdx.x * kTopkWarps + warp; u < units; u += n_warps) {
    const uint32_t c = (uint32_t)(u / a.tiles), tile = (uint32_t)(u - (uint64_t)c * a.tiles);
    const TopkChunk ch = a.chunks[c];
    if (a.general && ch.state == kTopkNone) continue;
    const bool live = (uint64_t)(a.tile0 + tile) * 32 + lane < a.T;
    const uint64_t si = ch.state != kTopkNone ? ((uint64_t)ch.state * a.tiles + tile) * 32 + lane : 0;
    const TopkState st = ch.state != kTopkNone ? topk_state_load(a, si) : TopkState{a.kk, 0u, 0ull, 0u};
    const uint32_t n = topk_stream<Key>(a, ch, tile, lane, live && !st.done(), st, h);
    if (ch.cand != kTopkNone) {  // a chunk of a larger group: its list, for topk_merge_kernel
      const uint64_t cb = (uint64_t)ch.cand * a.tiles + tile;
      for (uint32_t s = 0; s < n; ++s) {
        const uint64_t i = (cb * a.K + s) * 32 + lane;
        a.c_hi[i] = h.hi[s * 32]; a.c_lo[i] = h.lo[s * 32]; a.c_pos[i] = h.pos[s * 32];
      }
      a.c_n[cb * 32 + lane] = n;
    } else if (a.general) {
      if (live) topk_verdict(a, si, st, h, n);
    } else {  // the whole group: every listed cell is kept
      topk_write_words(a, sw, h.pos, n, ch.begin, ch.end, a.tile0 + tile, lane, [](uint32_t) { return true; });
    }
    __syncwarp();  // the heap is reused by the next unit
  }
}

// One warp per (multi-chunk group, tile): the best K of the chunks' lists, then the round's verdict, or in export mode
// the best K themselves
__global__ void __launch_bounds__(kTopkWarps * 32) topk_merge_kernel(const TopkArgs a) {
  extern __shared__ __align__(16) unsigned char topk_smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  TopkHeap h = topk_heap(topk_smem, a.K, topk_warp_bytes(a.K), warp, lane);
  const uint64_t units = (uint64_t)a.n_merges * a.tiles;
  const uint64_t n_warps = (uint64_t)gridDim.x * kTopkWarps;
  for (uint64_t u = (uint64_t)blockIdx.x * kTopkWarps + warp; u < units; u += n_warps) {
    const uint32_t m = (uint32_t)(u / a.tiles), tile = (uint32_t)(u - (uint64_t)m * a.tiles);
    if ((uint64_t)(a.tile0 + tile) * 32 + lane >= a.T) {  // (no shuffles below)
      if (a.x_n) a.x_n[((uint64_t)m * a.tiles + tile) * 32 + lane] = 0u;
      continue;
    }
    const TopkMerge g = a.merges[m];
    const uint64_t si = ((uint64_t)g.state * a.tiles + tile) * 32 + lane;
    const TopkState st = topk_state_load(a, si);
    uint32_t n = 0;
    unsigned long long th = 0;
    uint32_t tl = 0;
    if (!st.done()) {
      // kAhead candidates (and the next list's count) are loaded before any is offered: one memory latency per batch
      constexpr uint32_t kAhead = 16;
      uint32_t cn = g.cand_begin < g.cand_end ? a.c_n[((uint64_t)g.cand_begin * a.tiles + tile) * 32 + lane] : 0u;
      for (uint32_t c = g.cand_begin; c < g.cand_end; c += g.stride) {
        const uint64_t cb = (uint64_t)c * a.tiles + tile;
        const uint32_t cn_next = c + g.stride < g.cand_end ? a.c_n[(cb + (uint64_t)g.stride * a.tiles) * 32 + lane] : 0u;
        for (uint32_t s0 = 0; s0 < cn; s0 += kAhead) {
          unsigned long long ch[kAhead];
          uint32_t cl[kAhead];
#pragma unroll
          for (uint32_t q = 0; q < kAhead; ++q) {
            const uint64_t i = (cb * a.K + s0 + q) * 32 + lane;
            const bool in = s0 + q < cn;
            ch[q] = in ? a.c_hi[i] : 0ull;
            cl[q] = in ? a.c_lo[i] : 0u;
          }
#pragma unroll
          for (uint32_t q = 0; q < kAhead; ++q)  // (a verdict reads keys only: the member position is not carried)
            if (s0 + q < cn) h.offer(n, a.K, th, tl, ch[q], cl[q], 0u);
        }
        cn = cn_next;
      }
    }
    if (a.x_hi) {
      const uint64_t xb = (uint64_t)m * a.tiles + tile;
      for (uint32_t s = 0; s < n; ++s) {
        a.x_hi[(xb * a.K + s) * 32 + lane] = h.hi[s * 32];
        a.x_lo[(xb * a.K + s) * 32 + lane] = h.lo[s * 32];
      }
      a.x_n[xb * 32 + lane] = n;
    } else {
      topk_verdict(a, si, st, h, n);
    }
  }
}

// Fast path, one warp per (chunk of a multi-chunk group, tile): the chunk's candidates at or above the group's
// threshold (all of them when the group keeps every cell) become the members' words
__global__ void __launch_bounds__(kTopkWarps * 32) topk_mark_kernel(const TopkArgs a) {
  __shared__ uint32_t sw_all[kTopkWarps][kTopkMarkBlock];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint64_t units = (uint64_t)a.n_chunks * a.tiles;
  const uint64_t n_warps = (uint64_t)gridDim.x * kTopkWarps;
  for (uint64_t u = (uint64_t)blockIdx.x * kTopkWarps + warp; u < units; u += n_warps) {
    const uint32_t c = (uint32_t)(u / a.tiles), tile = (uint32_t)(u - (uint64_t)c * a.tiles);
    const TopkChunk ch = a.chunks[c];
    if (ch.cand == kTopkNone) continue;
    const bool live = (uint64_t)(a.tile0 + tile) * 32 + lane < a.T;
    const uint64_t si = ((uint64_t)ch.state * a.tiles + tile) * 32 + lane;
    const uint64_t cb = (uint64_t)ch.cand * a.tiles + tile;
    const uint32_t n = live ? a.c_n[cb * 32 + lane] : 0u;
    const bool all = live && (a.s_flags[si] & kTopkAll);
    const unsigned long long th = live ? a.s_hi[si] : 0ull;
    const uint32_t tl = live ? a.s_lo[si] : 0u;
    const uint64_t base = cb * a.K * 32 + lane;
    topk_write_words(a, sw_all[warp], a.c_pos + base, n, ch.begin, ch.end, a.tile0 + tile, lane, [&](uint32_t s) {
      return all || !key_less(a.c_hi[base + (uint64_t)s * 32], a.c_lo[base + (uint64_t)s * 32], th, tl);
    });
  }
}

// General path, one warp per (chunk, tile): a member's word has the valid cells at or above the (group, step)'s
// threshold, or every valid cell (groups of at most kk members, and steps with fewer than kk cells)
template <class Key = F64Key>
__global__ void __launch_bounds__(256, 1) topk_select_kernel(const TopkArgs a) {
  constexpr uint32_t kAhead = 8;
  const int lane = threadIdx.x & 31;
  const uint64_t units = (uint64_t)a.n_chunks * a.tiles;
  const uint64_t n_warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t u = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; u < units; u += n_warps) {
    const uint32_t c = (uint32_t)(u / a.tiles), tile = (uint32_t)(u - (uint64_t)c * a.tiles);
    const TopkChunk ch = a.chunks[c];
    const uint32_t gt = a.tile0 + tile;
    const uint64_t step = (uint64_t)gt * 32 + lane;
    const bool live = step < a.T;
    bool all = true;
    unsigned long long th = 0;
    uint32_t tl = 0;
    if (ch.state != kTopkNone && live) {
      const uint64_t si = ((uint64_t)ch.state * a.tiles + tile) * 32 + lane;
      all = (a.s_flags[si] & kTopkAll) != 0;
      th = a.s_hi[si]; tl = a.s_lo[si];
    }
    const uint32_t live_bits = a.T - (uint64_t)gt * 32 >= 32 ? 0xFFFFFFFFu : (1u << (a.T - (uint64_t)gt * 32)) - 1u;
    for (uint32_t m0 = ch.begin; m0 < ch.end; m0 += 32) {
      const uint32_t j = m0 + lane;
      const bool in = j < ch.end;
      const uint32_t row = in ? __ldg(a.members + j) : 0u;
      const uint32_t w = in ? a.valid[(uint64_t)row * a.Tw + gt] & live_bits : 0u;
      const uint32_t t = in ? __ldg(a.tie + row) : 0u;
      const uint32_t nb = min(32u, ch.end - m0);
      uint32_t mine = w;  // groups that keep every cell
      if (ch.state != kTopkNone) {
        for (uint32_t i0 = 0; i0 < nb; i0 += kAhead) {
          double v[kAhead];
          uint32_t on = 0;  // bit q: member i0 + q has a cell at this lane's step
#pragma unroll
          for (uint32_t q = 0; q < kAhead; ++q) {
            const uint32_t i = i0 + q;
            const uint32_t r = __shfl_sync(0xFFFFFFFFu, row, i & 31);
            const uint32_t wq = __shfl_sync(0xFFFFFFFFu, w, i & 31);
            const bool cell = i < nb && ((wq >> lane) & 1u);
            on |= (uint32_t)cell << q;
            v[q] = cell && !all ? __ldg(a.vals + (uint64_t)r * a.T + step) : 0.0;
          }
#pragma unroll
          for (uint32_t q = 0; q < kAhead; ++q) {
            const uint32_t tq = __shfl_sync(0xFFFFFFFFu, t, (i0 + q) & 31);
            bool keep = (on >> q) & 1u;
            if (keep && !all) {
              unsigned long long kh;
              uint32_t kl;
              topk_key<Key>(v[q], tq, a.bottom, kh, kl);
              keep = !key_less(kh, kl, th, tl);
            }
            const uint32_t word = __ballot_sync(0xFFFFFFFFu, keep);
            if (lane == (int)((i0 + q) & 31)) mine = word;
          }
        }
      }
      __syncwarp();
      if (in) a.out_valid[(uint64_t)row * a.Tw + gt] = mine;
    }
  }
}

// Per (row, word): mode 0 (kk >= largest group): valid & live for a row of a group, 0 for a row whose group id is out
// of range; mode 1: only the rows whose group id is out of range are written (0)
__global__ void __launch_bounds__(256) topk_copy_kernel(const uint32_t* valid, const uint32_t* gid, uint32_t n_groups,
                                                        uint64_t n_rows, uint64_t T, uint32_t Tw, int mode,
                                                        uint32_t* out_valid) {
  const uint64_t n = n_rows * Tw;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t r = i / Tw;
    const uint32_t w = (uint32_t)(i - r * Tw);
    const bool in = gid[r] < n_groups;
    if (mode == 1 && in) continue;
    const uint64_t left = T - (uint64_t)w * 32;
    const uint32_t live = left >= 32 ? 0xFFFFFFFFu : (1u << left) - 1u;
    out_valid[i] = in ? (valid[i] & live) : 0u;
  }
}

}  // namespace b2p
