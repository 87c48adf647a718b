// The definition of a word's expanded value m (expand_as, heatmap.py:77-93): every word-list kernel builds m from it.
#pragma once

#include <math.h>

#include "daam_b200.h"

namespace daam {

constexpr int kWordChunks = 32;                       // min / max chunks of a plane (one (map, word) pair) at most
constexpr int kWordPartialFloats = 2 * kWordChunks;   // a plane's partials: (min, max) of v per chunk
static_assert(kWordPartialFloats == DAAM_EXPAND_SCRATCH_FLOATS, "expand's scratch holds one plane's partials per word");

// The word map at pixel i: the mean of rows[r0 .. r1) of maps [*][xx] (heatmap.py:121-123)
__device__ __forceinline__ float word_mean(const float* __restrict__ maps, const int* rows, int r0, int r1, int xx, int i) {
  float s = 0.f;
  for (int r = r0; r < r1; ++r) s += __ldg(maps + (long long)rows[r] * xx + i);
  return s / (float)(r1 - r0);
}

// min / max of v from a plane's partials slots[chunks][2], in chunk order. `chunks` is a reference to the params'
// count, read where the loop tests it: passed by value, nvcc hoists it and overlay_kernel spills.
__device__ __forceinline__ void partial_bounds(const float* slots, const int& chunks, float& lo, float& hi) {
  lo = INFINITY; hi = -INFINITY;
  for (int c = 0; c < chunks; ++c) { lo = fminf(lo, slots[2 * c]); hi = fmaxf(hi, slots[2 * c + 1]); }
}

// expand_as's min-max normalisation (heatmap.py:88-89)
__device__ __forceinline__ float minmax_normalize(float v, float lo, float hi) { return (v - lo) / (hi - lo + 1e-8f); }

}  // namespace daam
