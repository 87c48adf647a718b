// The bicubic interpolation both the finalize and the word-list kernels use: torch's `upsample_bicubic2d` with
// align_corners=False. Source index (dst + 0.5) * in/out - 0.5 (not clamped), Keys' cubic convolution with A = -0.75 on
// the 4 taps floor-1..floor+2, taps clamped to the border; rows are combined horizontally first, then vertically, all in
// fp32.
#pragma once

namespace daam {

struct Taps {
  int idx[4];
  float w[4];
};

__device__ __forceinline__ float cubic_near(float t, float a) { return ((a + 2.f) * t - (a + 3.f)) * t * t + 1.f; }
__device__ __forceinline__ float cubic_far(float t, float a) { return ((a * t - 5.f * a) * t + 8.f * a) * t - 4.f * a; }

__device__ __forceinline__ Taps make_taps(int dst, int n_in, int n_out) {
  const float a = -0.75f;
  const float scale = (float)n_in / (float)n_out;
  const float src = scale * ((float)dst + 0.5f) - 0.5f;
  const float fl = floorf(src);
  const float t = src - fl;
  const int base = (int)fl;
  Taps r;
  r.w[0] = cubic_far(t + 1.f, a);
  r.w[1] = cubic_near(t, a);
  r.w[2] = cubic_near(1.f - t, a);
  r.w[3] = cubic_far(2.f - t, a);
#pragma unroll
  for (int i = 0; i < 4; ++i) r.idx[i] = min(max(base - 1 + i, 0), n_in - 1);
  return r;
}

// from global memory, through the read-only cache
__device__ __forceinline__ float bicubic_at(const float* __restrict__ src, int w, const Taps& ty, const Taps& tx) {
  float v = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float* row = src + ty.idx[i] * w;
    float r = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) r += tx.w[j] * __ldg(row + tx.idx[j]);
    v += ty.w[i] * r;
  }
  return v;
}

// the same arithmetic with plain loads, for a map in shared memory
__device__ __forceinline__ float bicubic_shared(const float* sm, int w, const Taps& ty, const Taps& tx) {
  float v = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float* row = sm + ty.idx[i] * w;
    float r = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) r += tx.w[j] * row[tx.idx[j]];
    v += ty.w[i] * r;
  }
  return v;
}

}  // namespace daam
