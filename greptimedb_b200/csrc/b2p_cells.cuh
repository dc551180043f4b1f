// b2p_cells.cuh — the validity words of a dense [rows x T] grid as the compacting kernels read them (K13's count and
// scatter, K14's scatter, K15's OR).  Device functions only: the header may be included by several translation units.
#pragma once
#include <cstdint>

namespace b2p {

// the bits of validity word w that are steps of the grid: all of them but in the last word when T is not a multiple of 32
__device__ __forceinline__ uint32_t grid_mask(uint32_t Tw, uint32_t w, uint64_t T) {
  const uint32_t tail = (uint32_t)(T & 31);
  return (w == Tw - 1 && tail) ? (1u << tail) - 1u : 0xFFFFFFFFu;
}

// bits of validity word w of row `row` that are steps of the grid (the last word of a row may carry stray bits past T)
__device__ __forceinline__ uint32_t grid_word(const uint32_t* valid, uint64_t row, uint32_t Tw, uint32_t w, uint64_t T) {
  return __ldg(valid + row * Tw + w) & grid_mask(Tw, w, T);
}

}  // namespace b2p
