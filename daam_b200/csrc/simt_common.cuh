// Code shared by the SIMT kernels (accumulate_simt.cu, probs.cu): each CTA's contiguous range of tiles, 16-byte staged
// loads of the K^T / Q tiles into shared memory, the one-thread-per-pixel logits + softmax, and the host-side
// shared-memory attribute of the kernels.
#pragma once

#include "common.cuh"

namespace daam {
namespace simt {

template <typename T> struct Vec;  // 16-byte global loads converted to fp32
template <> struct Vec<float> {
  static constexpr int kElems = 4;
  static __device__ __forceinline__ void load(const float* p, float* out) {
    float4 v = __ldg(reinterpret_cast<const float4*>(p));
    out[0] = v.x; out[1] = v.y; out[2] = v.z; out[3] = v.w;
  }
  static __device__ __forceinline__ float one(const float* p) { return __ldg(p); }
};
template <> struct Vec<__half> {
  static constexpr int kElems = 8;
  static __device__ __forceinline__ void load(const __half* p, float* out) {
    uint4 v = __ldg(reinterpret_cast<const uint4*>(p));
    const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
    for (int i = 0; i < 4; ++i) { float2 f = __half22float2(h[i]); out[2 * i] = f.x; out[2 * i + 1] = f.y; }
  }
  static __device__ __forceinline__ float one(const __half* p) { return __half2float(__ldg(p)); }
};
template <> struct Vec<__nv_bfloat16> {
  static constexpr int kElems = 8;
  static __device__ __forceinline__ void load(const __nv_bfloat16* p, float* out) {
    uint4 v = __ldg(reinterpret_cast<const uint4*>(p));
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
    for (int i = 0; i < 4; ++i) { float2 f = __bfloat1622float2(h[i]); out[2 * i] = f.x; out[2 * i + 1] = f.y; }
  }
  static __device__ __forceinline__ float one(const __nv_bfloat16* p) { return __bfloat162float(__ldg(p)); }
};

// This CTA's share of the launch's tiles, [first, first + count): contiguous, so consecutive tiles share (layer, prompt,
// head) and K^T is staged once per run.
struct TileSpan {
  int first, count;
};
__device__ __forceinline__ TileSpan cta_tiles(int total_tiles) {
  const int per = total_tiles / gridDim.x, rem = total_tiles % gridDim.x;
  const int first = blockIdx.x * per + min((int)blockIdx.x, rem);
  return {first, per + ((int)blockIdx.x < rem ? 1 : 0)};
}

// Stage K^T of context rows [77 chunk, 77 chunk + 77) (ks[dim][token], tokens padded to 80 with zeros) and the Q tile
// (qs[pixel][dim], row stride d+1: odd, hence bank-conflict free for the per-thread row walk) into shared memory with
// coalesced 16-byte global loads.
template <typename T>
__device__ __forceinline__ void stage_tile(const LayerParams& L, int prompt, int head, int pixel0, int chunk, float* ks,
                                           float* qs, bool load_k, bool load_q) {
  const int d = L.head_dim;
  const T* kbase = static_cast<const T*>(L.k) + prompt * L.ks_prompt + head * L.ks_head +
                   (long long)chunk * kTokens * L.ks_token;
  const T* qbase = static_cast<const T*>(L.q) + prompt * L.qs_prompt + head * L.qs_head;
  constexpr int V = Vec<T>::kElems;
  const int qstride = d + 1;
  if (L.vec_ok) {
    const int vec_per_row = d / V;
    for (int c = threadIdx.x; load_k && c < kTokensPad * vec_per_row; c += blockDim.x) {
      const int t = c / vec_per_row, v = c - t * vec_per_row;
      float f[V];
      if (t < kTokens) {
        Vec<T>::load(kbase + t * L.ks_token + v * V, f);
      } else {
#pragma unroll
        for (int i = 0; i < V; ++i) f[i] = 0.f;
      }
#pragma unroll
      for (int i = 0; i < V; ++i) ks[(v * V + i) * kTokensPad + t] = f[i];
    }
    for (int c = threadIdx.x; load_q && c < kTilePixels * vec_per_row; c += blockDim.x) {
      const int r = c / vec_per_row, v = c - r * vec_per_row;
      float f[V];
      if (pixel0 + r < L.hw) {
        Vec<T>::load(qbase + (long long)(pixel0 + r) * L.qs_pixel + v * V, f);
      } else {
#pragma unroll
        for (int i = 0; i < V; ++i) f[i] = 0.f;
      }
#pragma unroll
      for (int i = 0; i < V; ++i) qs[r * qstride + v * V + i] = f[i];
    }
  } else {  // unaligned views: scalar loads
    for (int c = threadIdx.x; load_k && c < kTokensPad * d; c += blockDim.x) {
      const int t = c / d, e = c - t * d;
      ks[e * kTokensPad + t] = t < kTokens ? Vec<T>::one(kbase + t * L.ks_token + e) : 0.f;
    }
    for (int c = threadIdx.x; load_q && c < kTilePixels * d; c += blockDim.x) {
      const int r = c / d, e = c - r * d;
      qs[r * qstride + e] = pixel0 + r < L.hw ? Vec<T>::one(qbase + (long long)(pixel0 + r) * L.qs_pixel + e) : 0.f;
    }
  }
}


// Decodes a tile index of a launch into (layer, prompt, head, first pixel); `li` is a monotone cursor.
struct TileRef {
  int li, prompt, head, pixel0, run;
};
__device__ __forceinline__ TileRef decode_tile(const LaunchParams& P, int tile, int& li) {
  while (li + 1 < P.n_layers && tile >= P.layer[li + 1].tile_begin) ++li;
  const LayerParams& L = P.layer[li];
  const int local = tile - L.tile_begin;
  const int ptile = local % L.tiles_per_head;
  const int ph = local / L.tiles_per_head;
  TileRef t;
  t.li = li;
  t.head = ph % L.heads;
  t.prompt = ph / L.heads;
  t.pixel0 = ptile * kTilePixels;
  t.run = L.tile_begin + ph;                  // unique per (layer, prompt, head) within the launch
  return t;
}

__device__ __forceinline__ void stage_any(const LayerParams& L, const TileRef& t, int chunk, float* ks, float* qs,
                                          bool load_k, bool load_q) {
  if (L.dtype == DAAM_F32) stage_tile<float>(L, t.prompt, t.head, t.pixel0, chunk, ks, qs, load_k, load_q);
  else if (L.dtype == DAAM_F16) stage_tile<__half>(L, t.prompt, t.head, t.pixel0, chunk, ks, qs, load_k, load_q);
  else stage_tile<__nv_bfloat16>(L, t.prompt, t.head, t.pixel0, chunk, ks, qs, load_k, load_q);
}

// This thread's pixel: the raw logits <q, k> of the staged tokens in s[0..79] (columns 77..79 are padding).
__device__ __forceinline__ void pixel_logits(int d, const float* ks, const float* qs, float* s) {
#pragma unroll
  for (int t = 0; t < kTokensPad; ++t) s[t] = 0.f;
  const float* qrow = qs + threadIdx.x * (d + 1);
#pragma unroll 2
  for (int e = 0; e < d; ++e) {
    const float qv = qrow[e];
    const float4* kr = reinterpret_cast<const float4*>(ks + e * kTokensPad);
#pragma unroll
    for (int j = 0; j < kTokensPad / 4; ++j) {
      const float4 kv = kr[j];
      s[4 * j + 0] = fmaf(qv, kv.x, s[4 * j + 0]);
      s[4 * j + 1] = fmaf(qv, kv.y, s[4 * j + 1]);
      s[4 * j + 2] = fmaf(qv, kv.z, s[4 * j + 2]);
      s[4 * j + 3] = fmaf(qv, kv.w, s[4 * j + 3]);
    }
  }
}

// This thread's pixel: 77 un-normalised probabilities exp2(scale*log2e*(s - max)) in s[0..76]; returns 1 / sum.
__device__ __forceinline__ float pixel_softmax(const LayerParams& L, const float* ks, const float* qs, float* s) {
  pixel_logits(L.head_dim, ks, qs, s);
  // softmax over the 77 real tokens (columns 77..79 are padding and never read)
  float m = s[0];
#pragma unroll
  for (int t = 1; t < kTokens; ++t) m = fmaxf(m, s[t]);
  const float c = L.scale_log2e, mc = m * c;
  float sum = 0.f;
#pragma unroll
  for (int t = 0; t < kTokens; ++t) { s[t] = fast_exp2(fmaf(s[t], c, -mc)); sum += s[t]; }
  return 1.0f / sum;
}

inline size_t tile_smem_floats(int head_dim) { return (size_t)head_dim * kTokensPad + (size_t)kTilePixels * (head_dim + 1); }

// Raises `kernel`'s dynamic shared-memory limit on the current device (`device`) to at least `smem` bytes; the attribute
// is per kernel and device, and each (kernel, device) pair is set once per size it grows to.
int reserve_dynamic_smem(const void* kernel, int device, size_t smem);

}  // namespace simt
}  // namespace daam
