// b2p_absent.cuh — PromQL absent(<expr>) (K15): the steps of a dense [rows x T] grid at which no row has a valid cell,
// the steps the reference's AbsentStream emits when its cursor walks the grid past the child's timestamps (absent.rs).
// Only the validity words are read: one bit per cell, never a value.
//   absent_or_kernel     acc[w] = the OR over rows of validity word w (bits past T masked, grid_word).  Thread t of the
//                        P in the grid reads word w = t mod Tw of rows t / Tw, t / Tw + P / Tw, ..: each sweep reads
//                        P / Tw whole rows, one contiguous run of words, and every thread stays on its word.  When Tw > P
//                        a thread reads the words t, t + P, .. of every row, the grid reading one contiguous run of a
//                        row at a time.  A thread stops reading a word once it holds every step.  When Tw < 256 the
//                        threads of a CTA share words: they fold them in shared memory first.  Either way a CTA ORs
//                        each non-zero word into acc with one global atomic.
//   absent_write_kernel  one warp per output word w: out_valid[w] = ~acc[w] & the grid's bits, out[k] = 1.0 where the
//                        bit of step k is set, else 0.0
#pragma once
#include <cstdint>

#include "b2p_cells.cuh"

namespace b2p {

constexpr int kAbsentThreads = 256;  // per CTA of the OR pass; a word column shared by the CTA fits its shared array

struct AbsentArgs {
  const uint32_t* valid;  // [rows x Tw]
  uint32_t rows, Tw;
  uint64_t T;
  uint32_t* acc;          // [Tw], zeroed before the OR pass
  double* out;            // [T]
  uint32_t* out_valid;    // [Tw]
};

__global__ void __launch_bounds__(kAbsentThreads) absent_or_kernel(const AbsentArgs a) {
  __shared__ uint32_t s_or[kAbsentThreads];
  const uint64_t P = (uint64_t)gridDim.x * kAbsentThreads;
  const uint64_t t = (uint64_t)blockIdx.x * kAbsentThreads + threadIdx.x;
  const bool shared_words = a.Tw < kAbsentThreads;  // (then Tw < P: each thread has at most one word)
  if (shared_words) {
    if (threadIdx.x < a.Tw) s_or[threadIdx.x] = 0u;
    __syncthreads();
  }
  const uint64_t per = a.Tw <= P ? P / a.Tw : 1;  // rows read side by side
  const uint64_t span = per * a.Tw;               // words of one sweep, a multiple of Tw
  for (uint64_t f = t; f < span; f += P) {
    const uint32_t w = (uint32_t)(f % a.Tw);
    const uint32_t full = grid_mask(a.Tw, w, a.T);
    uint32_t o = 0u;
    uint64_t r = f / a.Tw;
    for (; r + 3 * per < a.rows && o != full; r += 4 * per)  // four independent loads in flight
      o |= grid_word(a.valid, r, a.Tw, w, a.T) | grid_word(a.valid, r + per, a.Tw, w, a.T) |
           grid_word(a.valid, r + 2 * per, a.Tw, w, a.T) | grid_word(a.valid, r + 3 * per, a.Tw, w, a.T);
    for (; r < a.rows && o != full; r += per) o |= grid_word(a.valid, r, a.Tw, w, a.T);
    if (!o) continue;
    if (shared_words) atomicOr(&s_or[w], o);
    else atomicOr(a.acc + w, o);  // (Tw >= 256: no other thread of the CTA has word w)
  }
  if (!shared_words) return;
  __syncthreads();
  if (threadIdx.x < a.Tw && s_or[threadIdx.x]) atomicOr(a.acc + threadIdx.x, s_or[threadIdx.x]);
}

__global__ void __launch_bounds__(256) absent_write_kernel(const AbsentArgs a) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warp0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint64_t n_warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t w = warp0; w < a.Tw; w += n_warps) {
    const uint32_t word = ~a.acc[w] & grid_mask(a.Tw, (uint32_t)w, a.T);
    const uint64_t k = w * 32 + lane;
    if (k < a.T) a.out[k] = ((word >> lane) & 1u) ? 1.0 : 0.0;
    if (lane == 0) a.out_valid[w] = word;
  }
}

}  // namespace b2p
