// b2p_cells.cuh — the validity words of a dense [rows x T] grid as the compacting kernels read them (K13's count and
// scatter, K14's scatter).  Device functions only: the header may be included by several translation units.
#pragma once
#include <cstdint>

namespace b2p {

// bits of validity word w of row `row` that are steps of the grid (the last word of a row may carry stray bits past T)
__device__ __forceinline__ uint32_t grid_word(const uint32_t* valid, uint64_t row, uint32_t Tw, uint32_t w, uint64_t T) {
  const uint32_t word = __ldg(valid + row * Tw + w);
  const uint32_t tail = (uint32_t)(T & 31);
  return (w == Tw - 1 && tail) ? word & ((1u << tail) - 1u) : word;
}

}  // namespace b2p
