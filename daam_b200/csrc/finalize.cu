// Finalize kernels: per-key bicubic upsample -> clamp -> mean over keys (-> normalise), word-map row mean,
// and the image-size expansion of a word map.
//
// Replaces DiffusionHeatMapHooker.compute_global_heat_map (daam/trace.py:109-130), GlobalHeatMap.
// compute_word_heat_map (daam/heatmap.py:121-123) and WordHeatMap.expand_as (daam/heatmap.py:77-93).
// The interpolation is torch's `upsample_bicubic2d` with align_corners=False: source index
// (dst + 0.5) * in/out - 0.5 (not clamped), Keys' cubic convolution with A = -0.75 on the 4 taps floor-1..floor+2,
// taps clamped to the border; rows are combined horizontally first, then vertically, all in fp32.
#include <cooperative_groups.h>
#include <math.h>
#include <stdlib.h>

#include <algorithm>
#include <mutex>

#include "common.cuh"

namespace daam {
namespace {

constexpr int kMaxGroups = 160;   // key groups (layer x prompt slices) per finalize launch
constexpr int kMaxRows = 128;     // selected rows of a word map
constexpr int kMaxMaps = DAAM_FINALIZE_MAX_MAPS;   // output maps per finalize launch

// One output map of a finalize launch: blocks [block_begin, block_begin + block_count) of every group, i.e. the keys
// of the expanded group list `for g: for b: {acc_g + b * heads_g * tokens_g * h_g * w_g, heads_g, head_sel_g}`.
struct MapSel {
  float* out;                             // [n_rows][oh][ow]
  int block_begin, block_count, n_rows, n_keys;
  int band_rows;                          // fast kernel only: 8 or 4 (daam_finalize's rule for this map's n_rows)
};

struct FinalizeParams {
  int n_groups, oh, ow, n_maps;           // output maps [oh][ow]
  daam_key_group g[kMaxGroups];
  MapSel map[kMaxMaps];                   // blockIdx.z selects the map
};

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

// grid: (ceil(oh*ow / 256), max n_rows, n_maps). One thread = one output element (map, row t, pixel o); it walks every
// selected key: group by group, block by block, head by head.
__global__ void __launch_bounds__(256) finalize_kernel(const __grid_constant__ FinalizeParams P) {
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  const int t = blockIdx.y;
  const int oh = P.oh, ow = P.ow;
  const MapSel& M = P.map[blockIdx.z];
  if (o >= oh * ow || t >= M.n_rows) return;
  const int oy = o / ow, ox = o - oy * ow;
  float sum = 0.f;
  int ch = -1, cw = -1;
  Taps ty, tx;
  for (int g = 0; g < P.n_groups; ++g) {
    const daam_key_group& G = P.g[g];
    const int hw = G.h * G.w;
    const int h0 = G.head_sel < 0 ? 0 : G.head_sel;
    const int h1 = G.head_sel < 0 ? G.heads : G.head_sel + 1;
    const bool same = (G.h == oh && G.w == ow);
    if (!same && (G.h != ch || G.w != cw)) {
      ty = make_taps(oy, G.h, oh);
      tx = make_taps(ox, G.w, ow);
      ch = G.h; cw = G.w;
    }
    const long long head_stride = (long long)G.tokens * hw;
    for (int b = M.block_begin; b < M.block_begin + M.block_count; ++b) {
      const float* base = G.acc + (long long)b * G.heads * head_stride + (long long)t * hw;
      if (same) {   // scale 1: the cubic weights are exactly (0, 1, 0, 0)
#pragma unroll 4
        for (int head = h0; head < h1; ++head) sum += fmaxf(__ldg(base + head * head_stride + o), 0.f);
      } else {
#pragma unroll 2
        for (int head = h0; head < h1; ++head) sum += fmaxf(bicubic_at(base + head * head_stride, G.w, ty, tx), 0.f);
      }
    }
  }
  M.out[(long long)t * oh * ow + o] = sum / (float)M.n_keys;
}


// ---- fast path: integer upsampling factors 1 / 2 / 4 -------------------------------------------------------------
// One CTA owns one output band (BR = 8 or 4 rows x ow columns; the last band is partial when BR does not divide oh) of
// one token row and walks the key classes (distinct (kh, kw) source sizes) one after the other. A class has one integer
// factor F on both axes (oh = F kh, ow = F kw), so the cubic weights depend only on the output phase (F distinct weight
// sets per axis), and the F x F outputs under one source pixel read the same 5 x 5 source window: a thread owns ONE
// source pixel and emits its F x F outputs from one window (25 values, 9-14 FMAs per output).
// The windows come from shared memory: the band's source rows (+2 halo rows each side, clamped at the borders) of a
// CHUNK of keys are streamed in with cp.async -- 16-byte units, or 8- / 4-byte units when a key row is not a multiple of
// 4 floats (every thread has several independent copies in flight, two chunks double-buffered) -- so the key loop is no
// longer a chain of dependent global loads -- the round-1 kernel's bound (34.8 us for the 175-key SD-2.1 case, 222
// registers, 0.86 waves) -- and the kernel fits two CTAs per SM.
// When a class has fewer source pixels per band than threads, the spare thread groups take every kg-th key and the
// groups are merged through the shared-memory band in a fixed order (deterministic sums). Arithmetic per key is
// bit-identical to bicubic_at (same taps, same weights, same order).
constexpr int kMaxClassKeys = 2048;        // key pointers of one class staged in shared memory
constexpr int kStageFloats = 4096;         // one chunk buffer (16 KB); two of them

template <int F>
struct PhaseWeights {
  float w[F][4];
  __device__ __forceinline__ void init() {
    const float a = -0.75f;
#pragma unroll
    for (int p = 0; p < F; ++p) {
      const float src = (1.0f / (float)F) * ((float)p + 0.5f) - 0.5f;   // source coordinate relative to the block's pixel
      const float t = src - floorf(src);
      w[p][0] = cubic_far(t + 1.f, a);
      w[p][1] = cubic_near(t, a);
      w[p][2] = cubic_near(1.f - t, a);
      w[p][3] = cubic_far(2.f - t, a);
    }
  }
};

template <int F>
__device__ __forceinline__ void add_key(const PhaseWeights<F>& pw, const float (&v)[5][5], float (&acc)[F][F]) {
  float r[5][F];                                       // horizontal pass, per source row and output phase
#pragma unroll
  for (int i = 0; i < 5; ++i)
#pragma unroll
    for (int px = 0; px < F; ++px) {
      const int off = px < F / 2 ? 0 : 1;
      float q = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) q += pw.w[px][j] * v[i][off + j];
      r[i][px] = q;
    }
#pragma unroll
  for (int py = 0; py < F; ++py) {
    const int off = py < F / 2 ? 0 : 1;
#pragma unroll
    for (int px = 0; px < F; ++px) {
      float o = 0.f;
#pragma unroll
      for (int i = 0; i < 4; ++i) o += pw.w[py][i] * r[off + i][px];
      acc[py][px] += fmaxf(o, 0.f);
    }
  }
}

__device__ __forceinline__ void cp_async16(float* smem_dst, const float* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gsrc)
               : "memory");
}
// 8- and 4-byte units (key rows that are not a multiple of 4 floats); .cg takes 16-byte copies only
__device__ __forceinline__ void cp_async8(float* smem_dst, const float* gsrc) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gsrc)
               : "memory");
}
__device__ __forceinline__ void cp_async4(float* smem_dst, const float* gsrc) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gsrc)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// Streams chunk `chunk` of a factor-2 / factor-4 class into `buf` (one commit group): the band's source rows (+2 halo rows
// each side, border rows replicated like the clamped taps) of up to kc keys. Every thread copies fixed units (16, 8 or 4
// bytes: the widest that divides a key row) of every keys_par-th key; a key with more units than threads is copied by
// all threads, 256 units apart. Shared by the class passes and by the cross-class prefetch (next class's first chunk).
struct ChunkGeom {
  int region, kc, n_src, kg, VR, unit;
  __device__ __forceinline__ ChunkGeom(int kw, int f, int br) {
    const int R = br / f;                              // source rows under the band
    VR = R + 4;                                        // + 2 halo rows above and below
    region = VR * kw;                                  // floats of one key's staged rows
    n_src = R * kw;                                    // source pixels under the band (<= 256, checked by the host)
    kg = 256 / n_src;                                  // thread groups that split the keys
    kc = kStageFloats / region;                        // keys per chunk, a multiple of kg so every group keeps its stride
    kc -= kc % kg;
    unit = kw % 4 == 0 ? 4 : (kw % 2 == 0 ? 2 : 1);    // floats per cp.async
  }
};
__device__ __forceinline__ void issue_chunk(int kh, int kw, int f, int band, int br, const float* const* keys, int nk,
                                            int chunk, float* buf) {
  const ChunkGeom G(kw, f, br);
  const int u = G.unit, row_units = kw / u, key_units = G.VR * row_units;
  const int keys_par = key_units <= 256 ? 256 / key_units : 1, copy_k = (int)threadIdx.x / key_units;
  const int k0 = chunk * G.kc, kn = min(G.kc, nk - k0);
  if (copy_k < keys_par) {
    for (int pos = (int)threadIdx.x - copy_k * key_units; pos < key_units; pos += 256) {
      const int vr = pos / row_units, c = pos - vr * row_units;
      const int src = min(max(band * (br / f) - 2 + vr, 0), kh - 1) * kw + u * c;
      float* dst = buf + vr * kw + u * c;
      if (u == 4) {
        for (int k = copy_k; k < kn; k += keys_par) cp_async16(dst + k * G.region, keys[k0 + k] + src);
      } else if (u == 2) {
        for (int k = copy_k; k < kn; k += keys_par) cp_async8(dst + k * G.region, keys[k0 + k] + src);
      } else {
        for (int k = copy_k; k < kn; k += keys_par) cp_async4(dst + k * G.region, keys[k0 + k] + src);
      }
    }
  }
  cp_async_commit();
}

// What to prefetch while a class is being merged: the first chunk of the next factor-2 / factor-4 class (into chunk
// buffer 1; the merge parks the key groups in buffer 0).
struct NextClass {
  int kh, kw, f, nk;                                   // f == 0: nothing to prefetch
  const float* const* keys;
};

// `first_buf`: the chunk buffer holding this class's chunk 0 (1 when the previous class prefetched it, else 0 and the
// chunk is issued here).
template <int F>
__device__ __forceinline__ void class_pass(const FinalizeParams& P, int kh, int kw, int nk, int band, int br, float* tile,
                                           const float* const* keys, float* stage, bool prefetched, const NextClass& next) {
  const int ow = P.ow;
  const ChunkGeom G(kw, F, br);
  const int region = G.region, n_src = G.n_src, kg = G.kg, kc = G.kc;
  const int n_chunks = (nk + kc - 1) / kc;
  const int first_buf = prefetched ? 1 : 0;
  auto issue = [&](int c) { issue_chunk(kh, kw, F, band, br, keys, nk, c, stage + ((c + first_buf) & 1) * kStageFloats); };

  const int group = (int)threadIdx.x / n_src;
  const int s = (int)threadIdx.x - group * n_src;
  const bool live = group < kg;
  const int ly = s / kw, sx = s - ly * kw;
  int ix[5];
#pragma unroll
  for (int j = 0; j < 5; ++j) ix[j] = min(max(sx - 2 + j, 0), kw - 1);
  PhaseWeights<F> pw;
  pw.init();
  float acc[F][F];
#pragma unroll
  for (int py = 0; py < F; ++py)
#pragma unroll
    for (int px = 0; px < F; ++px) acc[py][px] = 0.f;

  if (!prefetched) issue(0);
  for (int c = 0; c < n_chunks; ++c) {
    if (c + 1 < n_chunks) { issue(c + 1); cp_async_wait<1>(); } else { cp_async_wait<0>(); }
    __syncthreads();                                   // chunk c has landed for every thread
    if (live) {
      const float* buf = stage + ((c + first_buf) & 1) * kStageFloats + ly * kw;
      const int kn = min(kc, nk - c * kc);
      for (int k = group; k < kn; k += kg) {
        const float* src = buf + k * region;
        float v[5][5];
#pragma unroll
        for (int i = 0; i < 5; ++i)
#pragma unroll
          for (int j = 0; j < 5; ++j) v[i][j] = src[i * kw + ix[j]];
        add_key<F>(pw, v, acc);
      }
    }
    __syncthreads();                                   // buffer (c & 1) may be overwritten by chunk c + 2
  }
  // both chunk buffers are free now: the next class's first chunk streams into buffer 1 while this class is merged
  if (next.f) issue_chunk(next.kh, next.kw, next.f, band, br, next.keys, next.nk, 0, stage + kStageFloats);
  // merge the key groups in a fixed order (deterministic sums): every group parks its band in the (now free) first
  // chunk buffer, then each band element is summed over the groups by one thread. Source rows past the map's last row
  // (a partial last band) were staged from the clamped border row: their outputs land in band rows that are never
  // written out.
  const int band_elems = br * ow;
  if (live) {
    float* mine = stage + group * band_elems + (ly * F) * ow + sx * F;
#pragma unroll
    for (int py = 0; py < F; ++py)
#pragma unroll
      for (int px = 0; px < F; ++px) mine[py * ow + px] = acc[py][px];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < band_elems; i += blockDim.x) {
    float sum = tile[i];
    for (int g = 0; g < kg; ++g) sum += stage[g * band_elems + i];
    tile[i] = sum;
  }
  __syncthreads();
}

// factor 1: bicubic at scale 1 is the identity, the class contributes clamp(src) -- coalesced float4 reads over the
// band's `rows` valid rows (rows * ow is a multiple of 4: ow * br is, and a partial last band ends at h * w, which the
// host checks); when the band has fewer float4s than threads, the spare thread groups take every kg-th key (merged in a
// fixed order)
__device__ __forceinline__ void class_pass_identity(const FinalizeParams& P, int nk, int band, int br, int rows, float* tile,
                                                    const float* const* keys, float* stage, const NextClass& next) {
  const int ow = P.ow;
  // this pass reads its keys straight from global memory: the next class's first chunk streams in underneath it
  if (next.f) issue_chunk(next.kh, next.kw, next.f, band, br, next.keys, next.nk, 0, stage + kStageFloats);
  const int n_el = rows * ow, n4 = n_el / 4;
  const int kg = n4 >= 256 ? 1 : 256 / n4;
  const int passes = (n4 + 255) / 256;
  for (int pass = 0; pass < passes; ++pass) {
    const int group = n4 >= 256 ? 0 : (int)threadIdx.x / n4;
    const int i = n4 >= 256 ? pass * 256 + (int)threadIdx.x : (int)threadIdx.x % n4;
    const bool live = i < n4 && group < kg;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (live) {
      const long long off = (long long)band * br * ow + 4 * i;
#pragma unroll 8
      for (int k = group; k < nk; k += kg) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(keys[k] + off));
        acc.x += fmaxf(v.x, 0.f); acc.y += fmaxf(v.y, 0.f); acc.z += fmaxf(v.z, 0.f); acc.w += fmaxf(v.w, 0.f);
      }
    }
    if (kg == 1) {                                       // every float4 of the band has one owner
      if (live) {
        float4* dst = reinterpret_cast<float4*>(tile + 4 * i);
        float4 cur = *dst;
        cur.x += acc.x; cur.y += acc.y; cur.z += acc.z; cur.w += acc.w;
        *dst = cur;
      }
      __syncthreads();
    } else {                                             // park the groups' bands, then sum them in a fixed order
      if (live) *reinterpret_cast<float4*>(stage + group * n_el + 4 * i) = acc;
      __syncthreads();
      for (int e = threadIdx.x; e < n_el; e += blockDim.x) {
        float sum = tile[e];
        for (int g = 0; g < kg; ++g) sum += stage[g * n_el + e];
        tile[e] = sum;
      }
      __syncthreads();
    }
  }
}

struct ClassList {
  int n;
  int kh[8], kw[8];         // distinct source sizes, each (oh / F, ow / F) with F = 1, 2 or 4
  // per block: keys[] is ordered class by class, and class c owns [key_begin[c], key_begin[c + 1]) times the map's
  // block count; group g's keys start at key_slot[g] times the block count, block by block, head by head
  int key_begin[9];
  int key_slot[kMaxGroups];
};

// grid: (ceil(oh / 4) bands, max n_rows, n_maps); a CTA past its map's bands or rows returns at once. Dynamic smem: two
// chunk buffers + the band tile (the largest band_rows of the launch * ow floats)
__global__ void __launch_bounds__(256, 2) finalize_fast_kernel(const __grid_constant__ FinalizeParams P,
                                                               const __grid_constant__ ClassList C) {
  extern __shared__ __align__(16) float dyn[];
  __shared__ const float* keys[kMaxClassKeys];
  float* stage = dyn;                                  // 2 x kStageFloats
  float* tile = dyn + 2 * kStageFloats;
  const MapSel& M = P.map[blockIdx.z];
  const int band = blockIdx.x, t = blockIdx.y, oh = P.oh, ow = P.ow, br = M.band_rows, nb = M.block_count;
  if (t >= M.n_rows || band * br >= oh) return;
  const int rows = min(br, oh - band * br);            // valid output rows of this band
  // key pointers (token row t) of every selected key, class by class; one thread per key group
  for (int g = threadIdx.x; g < P.n_groups; g += blockDim.x) {
    const daam_key_group& G = P.g[g];
    const int per_block = G.head_sel < 0 ? G.heads : 1;
    const long long hw = (long long)G.h * G.w;
    const float** dst = keys + C.key_slot[g] * nb;
    // key j of the group: head (block_begin * heads + j) of all heads, or head_sel of block block_begin + j
    const long long first = G.head_sel < 0 ? (long long)M.block_begin * G.heads : (long long)M.block_begin * G.heads + G.head_sel;
    const long long step = G.head_sel < 0 ? 1 : G.heads;
    for (int j = 0; j < per_block * nb; ++j) dst[j] = G.acc + ((first + j * step) * G.tokens + t) * hw;
  }
  for (int i = threadIdx.x; i < br * ow; i += blockDim.x) tile[i] = 0.f;
  __syncthreads();
  bool prefetched = false;                             // chunk 0 of class c is already streaming into buffer 1
  for (int c = 0; c < C.n; ++c) {
    const int kh = C.kh[c], kw = C.kw[c], f = ow / kw, nk = (C.key_begin[c + 1] - C.key_begin[c]) * nb;
    const float* const* ck = keys + C.key_begin[c] * nb;
    NextClass next = {0, 0, 0, 0, nullptr};
    if (c + 1 < C.n && C.kw[c + 1] != ow)
      next = {C.kh[c + 1], C.kw[c + 1], ow / C.kw[c + 1], (C.key_begin[c + 2] - C.key_begin[c + 1]) * nb,
              keys + C.key_begin[c + 1] * nb};
    if (f == 1) class_pass_identity(P, nk, band, br, rows, tile, ck, stage, next);
    else if (f == 2) class_pass<2>(P, kh, kw, nk, band, br, tile, ck, stage, prefetched, next);
    else class_pass<4>(P, kh, kw, nk, band, br, tile, ck, stage, prefetched, next);
    prefetched = next.f != 0;
  }
  __syncthreads();
  float* dst = M.out + (long long)t * oh * ow + (long long)band * br * ow;
  for (int i = threadIdx.x; i < rows * ow; i += blockDim.x) dst[i] = tile[i] / (float)M.n_keys;
}

// One output map per selected key (no mean): out[key][row][oh][ow] = clamp(bicubic(key[row])). grid: (ceil(oh*ow/256),
// n_rows, n_keys); key k belongs to group g with first_key[g] <= k < first_key[g + 1].
struct PerKeyParams {
  int n_groups, oh, ow, n_rows, n_keys;
  int first_key[kMaxGroups + 1];
  daam_key_group g[kMaxGroups];
};

__global__ void __launch_bounds__(256) finalize_per_key_kernel(const __grid_constant__ PerKeyParams P, float* __restrict__ out) {
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  const int t = blockIdx.y, key = blockIdx.z;
  const int oh = P.oh, ow = P.ow;
  if (o >= oh * ow) return;
  int g = 0;
  while (g + 1 < P.n_groups && key >= P.first_key[g + 1]) ++g;
  const daam_key_group& G = P.g[g];
  const int head = (G.head_sel < 0 ? 0 : G.head_sel) + (key - P.first_key[g]);
  const int hw = G.h * G.w;
  const float* src = G.acc + ((long long)head * G.tokens + t) * hw;
  float v;
  if (G.h == oh && G.w == ow) {
    v = __ldg(src + o);
  } else {
    const int oy = o / ow, ox = o - oy * ow;
    v = bicubic_at(src, G.w, make_taps(oy, G.h, oh), make_taps(ox, G.w, ow));
  }
  out[((long long)key * P.n_rows + t) * oh * ow + o] = fmaxf(v, 0.f);
}

// maps / (maps[1:-1].sum(0) + 1e-6), in place (daam/trace.py:129-130), at pixel o of one [n_rows][xx] map
__device__ __forceinline__ void normalize_pixel(float* __restrict__ maps, int n_rows, int xx, int o) {
  float s = 0.f;
  for (int t = 1; t < n_rows - 1; ++t) s += maps[(long long)t * xx + o];
  s += 1e-6f;
  for (int t = 0; t < n_rows; ++t) maps[(long long)t * xx + o] = maps[(long long)t * xx + o] / s;
}

__global__ void normalize_kernel(float* __restrict__ maps, int n_rows, int xx) {
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= xx) return;
  // blockIdx.y: independent map stacks (per-key finalize)
  normalize_pixel(maps + (long long)blockIdx.y * n_rows * xx, n_rows, xx, o);
}

// the finalize launches' normalisation: blockIdx.y selects the map, each with its own output and row count
struct MapOuts {
  float* out[kMaxMaps];
  int n_rows[kMaxMaps];
};

__global__ void normalize_maps_kernel(const __grid_constant__ MapOuts P, int xx) {
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= xx) return;
  normalize_pixel(P.out[blockIdx.y], P.n_rows[blockIdx.y], xx, o);
}

struct RowSel {
  int n;
  int rows[kMaxRows];
};

__global__ void word_map_kernel(const float* __restrict__ maps, const __grid_constant__ RowSel sel, int xx,
                                float* __restrict__ out) {
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= xx) return;
  float s = 0.f;
  for (int i = 0; i < sel.n; ++i) s += __ldg(maps + (long long)sel.rows[i] * xx + o);
  out[o] = s / (float)sel.n;
}

// ---- fused word list -> image-size masks -------------------------------------------------------------------------
// One cooperative launch for a LIST of words: gather-mean of the word's rows of the [mh][mw] global map
// (heatmap.py:121-123) -> bicubic to (out_h, out_w), taps mh -> out_h and mw -> out_w -> min / max over the image ->
// normalise / threshold (heatmap.py:77-93). CTA = (word, chunk of output pixels). The word map lives in shared memory;
// the min/max pass and the write pass both interpolate from it (16 shared loads + 20 FMAs per pixel), so nothing but
// the final image is written and nothing is read back: per-chunk
// partial min/max go through `scratch`, one grid-wide barrier separates the passes. With `absolute` there is no
// min/max pass and no barrier. Deterministic (no atomics).
constexpr int kMaxWords = 96;
constexpr int kMaxWordRows = 320;       // selected rows over all words of a launch
constexpr int kMaxChunks = 32;          // CTAs per word; scratch holds 2 floats per (word, chunk)

struct ExpandWordsParams {
  const float* maps;                    // [n_map_rows][mh][mw]
  float* word_maps;                     // optional [n_words][mh][mw]
  float* out;                           // [n_words][oh][ow]
  float* scratch;                       // [n_words][chunks][2]
  int mh, mw, oh, ow, n_words, chunks, absolute, use_threshold;
  float threshold;
  int row_begin[kMaxWords + 1];
  int rows[kMaxWordRows];
};

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

// The word map at pixel i: the mean of rows[r0 .. r1) of maps [*][xx] (heatmap.py:121-123). Shared by the expand and
// segment kernels, so that their word maps are the same bits.
__device__ __forceinline__ float word_mean(const float* __restrict__ maps, const int* rows, int r0, int r1, int xx, int i) {
  float s = 0.f;
  for (int r = r0; r < r1; ++r) s += __ldg(maps + (long long)rows[r] * xx + i);
  return s / (float)(r1 - r0);
}

// expand_as's min-max normalisation (heatmap.py:88-89)
__device__ __forceinline__ float minmax_normalize(float v, float lo, float hi) { return (v - lo) / (hi - lo + 1e-8f); }

__global__ void __launch_bounds__(256) expand_words_kernel(const __grid_constant__ ExpandWordsParams P) {
  extern __shared__ __align__(16) float wm[];          // the word map [mh][mw]
  __shared__ float red_lo[8], red_hi[8];
  const int word = blockIdx.x / P.chunks, chunk = blockIdx.x - word * P.chunks;
  const int mh = P.mh, mw = P.mw, xx = mh * mw, n = P.oh * P.ow;
  const int r0 = P.row_begin[word], r1 = P.row_begin[word + 1];
  for (int i = threadIdx.x; i < xx; i += blockDim.x) {
    const float s = word_mean(P.maps, P.rows, r0, r1, xx, i);
    wm[i] = s;
    if (chunk == 0 && P.word_maps) P.word_maps[(long long)word * xx + i] = s;
  }
  __syncthreads();
  const int per = (n + P.chunks - 1) / P.chunks;
  const int begin = chunk * per, end = min(n, begin + per);
  float lo = 0.f, hi = 0.f;
  if (!P.absolute) {
    lo = INFINITY; hi = -INFINITY;
    for (int o = begin + threadIdx.x; o < end; o += blockDim.x) {
      const int oy = o / P.ow, ox = o - oy * P.ow;
      const float v = bicubic_shared(wm, mw, make_taps(oy, mh, P.oh), make_taps(ox, mw, P.ow));
      lo = fminf(lo, v); hi = fmaxf(hi, v);
    }
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
      lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, s));
      hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, s));
    }
    if ((threadIdx.x & 31) == 0) { red_lo[threadIdx.x >> 5] = lo; red_hi[threadIdx.x >> 5] = hi; }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int i = 1; i < (int)blockDim.x / 32; ++i) { lo = fminf(lo, red_lo[i]); hi = fmaxf(hi, red_hi[i]); }
      float* slot = P.scratch + 2 * ((long long)word * P.chunks + chunk);
      slot[0] = lo; slot[1] = hi;
      __threadfence();
    }
    cooperative_groups::this_grid().sync();
    if (threadIdx.x == 0) {
      lo = INFINITY; hi = -INFINITY;
      const volatile float* slots = P.scratch + 2 * (long long)word * P.chunks;
      for (int c = 0; c < P.chunks; ++c) { lo = fminf(lo, slots[2 * c]); hi = fmaxf(hi, slots[2 * c + 1]); }
      red_lo[0] = lo; red_hi[0] = hi;
    }
    __syncthreads();
    lo = red_lo[0]; hi = red_hi[0];
  }
  float* dst = P.out + (long long)word * n;
  for (int o = begin + threadIdx.x; o < end; o += blockDim.x) {
    const int oy = o / P.ow, ox = o - oy * P.ow;
    float v = bicubic_shared(wm, mw, make_taps(oy, mh, P.oh), make_taps(ox, mw, P.ow));
    if (!P.absolute) v = minmax_normalize(v, lo, hi);
    if (P.use_threshold) v = v > P.threshold ? 1.f : 0.f;
    dst[o] = v;
  }
}

// ---- word segmentation: a per-pixel word label for a word list --------------------------------------------------
// labels[p] = 1 + argmax_w m[w][p] (lowest w on ties), or 0 where use_threshold and the max is not > threshold;
// scores[p] = max_w m[w][p], with m[w] what expand_words_kernel writes for word w without threshold. For n_maps global
// maps back to back (one, or every step of a time-resolved history) in two launches whatever n_maps and n_words:
//  1. segment_minmax_kernel, CTA = (map, word, chunk of output pixels): the word map (word_mean) goes to `word_maps`
//     and, unless `absolute`, the chunk's min / max of the interpolated map to `scratch`;
//  2. segment_label_kernel, CTA = (output tile, map): every word's min / max is reduced from its chunks, the source
//     window under the tile of a pass of words is staged in shared memory from `word_maps`, and each pixel keeps the
//     running max / argmax in registers while the words are interpolated.
// Same taps, bicubic_shared, word_mean and minmax_normalize as expand_words_kernel: the scores are its values. The
// [n_words][out_h][out_w] stack is never written. Deterministic (no atomics).
constexpr int kSegTileH = 16, kSegTileW = 64;      // output tile of one label CTA
constexpr int kSegPix = kSegTileH * kSegTileW / 256;   // output pixels per thread
constexpr int kSegStageFloats = 12288;              // staged windows per pass when they fit (48 KB)

struct SegmentParams {
  const float* maps;                    // [n_maps][n_map_rows][mh][mw]
  float* word_maps;                     // [n_maps][n_words][mh][mw]
  unsigned char* labels;                // [n_maps][oh][ow]
  float* scores;                        // [n_maps][oh][ow]
  float* scratch;                       // [n_maps][n_words][chunks][2]
  long long map_stride;                 // n_map_rows * mh * mw
  int mh, mw, oh, ow, n_words, chunks, absolute, use_threshold;
  float threshold;
  int words_per_pass;                   // words whose windows are staged at once
  int row_begin[kMaxWords + 1];
  int rows[kMaxWordRows];
};

// grid: n_maps * n_words * chunks; dynamic smem: the word map [mh][mw]
__global__ void __launch_bounds__(256) segment_minmax_kernel(const __grid_constant__ SegmentParams P) {
  extern __shared__ __align__(16) float wm[];
  __shared__ float red_lo[8], red_hi[8];
  const int chunk = blockIdx.x % P.chunks, mword = blockIdx.x / P.chunks;   // mword = map * n_words + word
  const int word = mword % P.n_words, map = mword / P.n_words;
  const int mh = P.mh, mw = P.mw, xx = mh * mw, n = P.oh * P.ow;
  const int r0 = P.row_begin[word], r1 = P.row_begin[word + 1];
  const float* maps = P.maps + (long long)map * P.map_stride;
  float* word_map = P.word_maps + (long long)mword * xx;
  for (int i = threadIdx.x; i < xx; i += blockDim.x) {
    const float s = word_mean(maps, P.rows, r0, r1, xx, i);
    wm[i] = s;
    if (chunk == 0) word_map[i] = s;
  }
  if (P.absolute) return;
  __syncthreads();
  const int per = (n + P.chunks - 1) / P.chunks;
  const int begin = chunk * per, end = min(n, begin + per);
  float lo = INFINITY, hi = -INFINITY;
  for (int o = begin + threadIdx.x; o < end; o += blockDim.x) {
    const int oy = o / P.ow, ox = o - oy * P.ow;
    const float v = bicubic_shared(wm, mw, make_taps(oy, mh, P.oh), make_taps(ox, mw, P.ow));
    lo = fminf(lo, v); hi = fmaxf(hi, v);
  }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) {
    lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, s));
    hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, s));
  }
  if ((threadIdx.x & 31) == 0) { red_lo[threadIdx.x >> 5] = lo; red_hi[threadIdx.x >> 5] = hi; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < (int)blockDim.x / 32; ++i) { lo = fminf(lo, red_lo[i]); hi = fmaxf(hi, red_hi[i]); }
    float* slot = P.scratch + 2 * ((long long)mword * P.chunks + chunk);
    slot[0] = lo; slot[1] = hi;
  }
}

// grid: (tiles of kSegTileH x kSegTileW output pixels, n_maps); dynamic smem: words_per_pass source windows
__global__ void __launch_bounds__(256) segment_label_kernel(const __grid_constant__ SegmentParams P) {
  extern __shared__ __align__(16) float win[];
  __shared__ float s_lo[kMaxWords], s_hi[kMaxWords];
  const int map = blockIdx.y, mh = P.mh, mw = P.mw, oh = P.oh, ow = P.ow, n_words = P.n_words;
  const int tiles_x = (ow + kSegTileW - 1) / kSegTileW;
  const int y0 = (blockIdx.x / tiles_x) * kSegTileH, x0 = (blockIdx.x % tiles_x) * kSegTileW;
  const int th = min(kSegTileH, oh - y0), tw = min(kSegTileW, ow - x0);
  // the source rows / columns the tile's taps read: taps move monotonically with the output index
  const int wy = make_taps(y0, mh, oh).idx[0], wx = make_taps(x0, mw, ow).idx[0];
  const int wh = make_taps(y0 + th - 1, mh, oh).idx[3] - wy + 1, ww = make_taps(x0 + tw - 1, mw, ow).idx[3] - wx + 1;
  const int wn = wh * ww;
  if (!P.absolute) {
    for (int w = threadIdx.x; w < n_words; w += blockDim.x) {   // chunks in a fixed order
      const float* slots = P.scratch + 2 * ((long long)map * n_words + w) * P.chunks;
      float lo = INFINITY, hi = -INFINITY;
      for (int c = 0; c < P.chunks; ++c) { lo = fminf(lo, slots[2 * c]); hi = fmaxf(hi, slots[2 * c + 1]); }
      s_lo[w] = lo; s_hi[w] = hi;
    }
  }
  const float* word_maps = P.word_maps + (long long)map * n_words * mh * mw;
  float best[kSegPix];
  int arg[kSegPix];
#pragma unroll
  for (int k = 0; k < kSegPix; ++k) { best[k] = -INFINITY; arg[k] = 0; }
  for (int w0 = 0; w0 < n_words; w0 += P.words_per_pass) {
    const int nw = min(P.words_per_pass, n_words - w0);
    __syncthreads();                                   // the previous pass has read its windows
    for (int i = threadIdx.x; i < nw * wn; i += blockDim.x) {
      const int wi = i / wn, r = i - wi * wn, y = r / ww, x = r - y * ww;
      win[i] = __ldg(word_maps + ((long long)(w0 + wi) * mh + wy + y) * mw + wx + x);
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kSegPix; ++k) {
      const int p = threadIdx.x + 256 * k;
      if (p < th * tw) {
        const int py = p / tw;
        Taps ty = make_taps(y0 + py, mh, oh), tx = make_taps(x0 + p - py * tw, mw, ow);
#pragma unroll
        for (int j = 0; j < 4; ++j) { ty.idx[j] -= wy; tx.idx[j] -= wx; }
        for (int wi = 0; wi < nw; ++wi) {
          const int w = w0 + wi;
          float v = bicubic_shared(win + wi * wn, ww, ty, tx);
          if (!P.absolute) v = minmax_normalize(v, s_lo[w], s_hi[w]);
          if (w == 0 || v > best[k]) { best[k] = v; arg[k] = w; }   // strict: the lowest word wins a tie
        }
      }
    }
  }
  const long long base = (long long)map * oh * ow;
#pragma unroll
  for (int k = 0; k < kSegPix; ++k) {
    const int p = threadIdx.x + 256 * k;
    if (p < th * tw) {
      const int py = p / tw;
      const long long o = base + (long long)(y0 + py) * ow + x0 + p - py * tw;
      P.scores[o] = best[k];
      P.labels[o] = (!P.use_threshold || best[k] > P.threshold) ? (unsigned char)(arg[k] + 1) : (unsigned char)0;
    }
  }
}

// ---- word-region overlap: sums of a word list's expanded maps over binary image regions -------------------------
// With m[w] what expand_words_kernel writes for word w (0/1 when use_threshold) and R[r] = (regions[r] != 0):
//   intersection[map][r][w] = sum_p R[r](p) m[w](p),   word_area[map][w] = sum_p m[w](p)
// in three launches whatever n_maps, n_words and n_regions:
//  1. segment_minmax_kernel (unchanged): word maps and per-chunk min / max partials;
//  2. region_tile_kernel, CTA = (16 x 64 output tile, map): stages the source windows of a pass of words as
//     segment_label_kernel does, computes m[w] per pixel with the same taps, bicubic_shared, minmax_normalize and
//     threshold compare as expand_words_kernel, and reduces every (word, slot) over the tile in a fixed order -- slot 0
//     is the word's area, slot 1 + r its sum inside region r -- into one partial per tile;
//  3. region_reduce_kernel: one warp per (map, word, slot) sums the tiles' partials in a fixed order.
// The [n_words][out_h][out_w] stack is never written; no atomics, so the sums are the same bits on every call. With a
// threshold every value is 0 or 1 and every partial an integer below 2^24, so the sums are exact counts.
constexpr int kMaxRegions = DAAM_REGION_MAX_REGIONS;   // 63 + the area slot: 64 slots per word, two groups of 32
constexpr int kRegionSlots = kMaxRegions + 1;

struct RegionParams {
  SegmentParams s;                      // maps, word_maps, scratch (min / max partials), sizes, rows, words_per_pass
  const unsigned char* regions;         // [n_regions][oh][ow]
  float* partials;                      // [n_maps][n_words][n_regions + 1][tiles]
  int n_regions, tiles;
};

// Lane l returns the warp's sum of s[l]. Five halving exchange rounds (31 shuffles for 32 values); the order of every
// add is fixed.
// One round: lanes with bit H set keep s[H .. 2H), the others s[0 .. H); each sends the other half to lane ^ H. The
// round count is a template argument so that every index is a constant and s[] stays in registers.
template <int H>
__device__ __forceinline__ void reduce_scatter_round(float (&s)[32], int lane) {
  const bool upper = (lane & H) != 0;
#pragma unroll
  for (int i = 0; i < H; ++i) {
    const float send = upper ? s[i] : s[i + H];
    const float keep = upper ? s[i + H] : s[i];
    s[i] = keep + __shfl_xor_sync(0xffffffffu, send, H);
  }
}

__device__ __forceinline__ float warp_reduce_scatter32(float (&s)[32]) {
  const int lane = threadIdx.x & 31;
  reduce_scatter_round<16>(s, lane);
  reduce_scatter_round<8>(s, lane);
  reduce_scatter_round<4>(s, lane);
  reduce_scatter_round<2>(s, lane);
  reduce_scatter_round<1>(s, lane);
  return s[0];
}

// grid: (tiles of kSegTileH x kSegTileW output pixels, n_maps); dynamic smem: words_per_pass source windows
__global__ void __launch_bounds__(256) region_tile_kernel(const __grid_constant__ RegionParams R) {
  extern __shared__ __align__(16) float win[];
  __shared__ float s_lo[kMaxWords], s_hi[kMaxWords];
  __shared__ float red[2][8][kRegionSlots];          // per-warp sums of a word, double-buffered across words
  __shared__ int tyi[4][kSegTileH], txi[4][kSegTileW];   // the tile's taps, relative to the staged window
  __shared__ float tyw[4][kSegTileH], txw[4][kSegTileW];
  const SegmentParams& P = R.s;
  const int map = blockIdx.y, mh = P.mh, mw = P.mw, oh = P.oh, ow = P.ow, n_words = P.n_words;
  const int tiles_x = (ow + kSegTileW - 1) / kSegTileW;
  const int y0 = (blockIdx.x / tiles_x) * kSegTileH, x0 = (blockIdx.x % tiles_x) * kSegTileW;
  const int th = min(kSegTileH, oh - y0), tw = min(kSegTileW, ow - x0);
  const int wy = make_taps(y0, mh, oh).idx[0], wx = make_taps(x0, mw, ow).idx[0];
  const int wh = make_taps(y0 + th - 1, mh, oh).idx[3] - wy + 1, ww = make_taps(x0 + tw - 1, mw, ow).idx[3] - wx + 1;
  const int wn = wh * ww;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_slots = R.n_regions + 1;
  if (!P.absolute) {
    for (int w = threadIdx.x; w < n_words; w += blockDim.x) {   // chunks in a fixed order
      const float* slots = P.scratch + 2 * ((long long)map * n_words + w) * P.chunks;
      float lo = INFINITY, hi = -INFINITY;
      for (int c = 0; c < P.chunks; ++c) { lo = fminf(lo, slots[2 * c]); hi = fmaxf(hi, slots[2 * c + 1]); }
      s_lo[w] = lo; s_hi[w] = hi;
    }
  }
  if (threadIdx.x < th) {
    const Taps t = make_taps(y0 + threadIdx.x, mh, oh);
#pragma unroll
    for (int j = 0; j < 4; ++j) { tyi[j][threadIdx.x] = t.idx[j] - wy; tyw[j][threadIdx.x] = t.w[j]; }
  } else if (threadIdx.x >= kSegTileH && threadIdx.x < kSegTileH + tw) {
    const int x = threadIdx.x - kSegTileH;
    const Taps t = make_taps(x0 + x, mw, ow);
#pragma unroll
    for (int j = 0; j < 4; ++j) { txi[j][x] = t.idx[j] - wx; txw[j][x] = t.w[j]; }
  }
  // slot bits of the thread's pixels: bit j of mask[g][k] says pixel k counts towards slot 32 g + j (slot 0: every
  // pixel of the tile, slot 1 + r: the pixels inside region r); each region byte is read once
  const long long n = (long long)oh * ow;
  unsigned mask[2][kSegPix];
#pragma unroll
  for (int k = 0; k < kSegPix; ++k) {
    const int p = threadIdx.x + 256 * k;
    mask[0][k] = 0u; mask[1][k] = 0u;
    if (p < th * tw) {
      const int py = p / tw;
      const unsigned char* reg = R.regions + (long long)(y0 + py) * ow + x0 + p - py * tw;
      unsigned m0 = 1u, m1 = 0u;
      for (int r = 0; r < R.n_regions; ++r) {
        const unsigned bit = __ldg(reg + r * n) != 0 ? 1u : 0u;
        if (r < 31) m0 |= bit << (r + 1); else m1 |= bit << (r - 31);
      }
      mask[0][k] = m0; mask[1][k] = m1;
    }
  }
  const float* word_maps = P.word_maps + (long long)map * n_words * mh * mw;
  float* partials = R.partials + (long long)map * n_words * n_slots * R.tiles + blockIdx.x;
  for (int w0 = 0; w0 < n_words; w0 += P.words_per_pass) {
    const int nw = min(P.words_per_pass, n_words - w0);
    __syncthreads();                                   // the previous pass has read its windows (and the taps are set)
    for (int i = threadIdx.x; i < nw * wn; i += blockDim.x) {
      const int wi = i / wn, r = i - wi * wn, y = r / ww, x = r - y * ww;
      win[i] = __ldg(word_maps + ((long long)(w0 + wi) * mh + wy + y) * mw + wx + x);
    }
    __syncthreads();
    for (int wi = 0; wi < nw; ++wi) {
      const int w = w0 + wi;
      float v[kSegPix];
#pragma unroll
      for (int k = 0; k < kSegPix; ++k) {
        const int p = threadIdx.x + 256 * k;
        v[k] = 0.f;
        if (p < th * tw) {
          const int py = p / tw, px = p - py * tw;
          Taps ty, tx;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            ty.idx[j] = tyi[j][py]; ty.w[j] = tyw[j][py]; tx.idx[j] = txi[j][px]; tx.w[j] = txw[j][px];
          }
          float x = bicubic_shared(win + wi * wn, ww, ty, tx);
          if (!P.absolute) x = minmax_normalize(x, s_lo[w], s_hi[w]);
          if (P.use_threshold) x = x > P.threshold ? 1.f : 0.f;
          v[k] = x;
        }
      }
      float (*buf)[kRegionSlots] = red[w & 1];
#pragma unroll
      for (int g = 0; g < 2; ++g) {
        if (g * 32 < n_slots) {
          float s[32];
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            float a = 0.f;
#pragma unroll
            for (int k = 0; k < kSegPix; ++k) a += (mask[g][k] >> j) & 1u ? v[k] : 0.f;
            s[j] = a;
          }
          buf[warp][32 * g + lane] = warp_reduce_scatter32(s);
        }
      }
      // one barrier per word: red[w & 1] is rewritten two words later, after every warp has passed the next barrier
      __syncthreads();
      if (warp == (w & 7)) {
        for (int slot = lane; slot < n_slots; slot += 32) {
          float a = 0.f;
#pragma unroll
          for (int i = 0; i < 8; ++i) a += buf[i][slot];
          partials[((long long)w * n_slots + slot) * R.tiles] = a;
        }
      }
    }
  }
}

// grid: ceil(n_out / 8), 256 threads; one warp per output o = (map * n_words + word) * (n_regions + 1) + slot sums
// the tiles' partials (lane-strided, then a butterfly) in a fixed order
__global__ void __launch_bounds__(256) region_reduce_kernel(const float* __restrict__ partials, long long n_out,
                                                            int tiles, int n_words, int n_regions,
                                                            float* __restrict__ intersection, float* __restrict__ area) {
  const long long o = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (o >= n_out) return;                              // whole warps
  const int lane = threadIdx.x & 31;
  const float* src = partials + o * tiles;
  float s = 0.f;
  for (int t = lane; t < tiles; t += 32) s += __ldg(src + t);
#pragma unroll
  for (int h = 16; h > 0; h >>= 1) s += __shfl_xor_sync(0xffffffffu, s, h);
  if (lane == 0) {
    const int n_slots = n_regions + 1;
    const int slot = (int)(o % n_slots);
    const long long mword = o / n_slots;               // map * n_words + word
    if (slot == 0) {
      area[mword] = s;
    } else {
      const long long map = mword / n_words, word = mword - map * n_words;
      intersection[(map * n_regions + slot - 1) * n_words + word] = s;
    }
  }
}

// ---- heat-map overlays: the jet-coloured word map blended onto the image -----------------------------------------
// The reference's plot_overlay (heatmap.py:20-53, 66-75) as pixels: with m[w] what expand_words_kernel writes for word
// w, for every byte of frames [n_maps][n_words][oh][ow][3]:
//   c = color_normalize ? (hi == lo ? 0 : (m - lo) / (hi - lo)) : clamp(m, 0, 1)   (lo / hi: min / max of m[w])
//   k = min(int(c * 256), 255)                                                      (matplotlib's Colormap, N = 256)
//   a = clamp(m, 0, 1)                                                              (the image drawn with alpha 1 - a)
//   out = uint8(clamp(rne((1 - a) * image + a * jet[k]), 0, 255))                   (every operation rounded in fp32)
// in two launches whatever n_maps and n_words:
//  1. segment_minmax_kernel (unchanged): word maps and the per-chunk min / max of the interpolated map v;
//  2. overlay_kernel, CTA = (16 x 64 output tile, map): stages the source windows of a pass of words as
//     segment_label_kernel does, computes m[w] with the same taps, bicubic_shared, minmax_normalize and threshold
//     compare as expand_words_kernel, and writes every word's RGB bytes through shared memory in aligned 4- and 16-byte
//     stores. v -> m is monotone non-decreasing in fp32 (subtract, divide by a positive constant, `>` threshold), so
//     lo / hi of m are m at the min / max of v: no pass over m.
// The [n_words][out_h][out_w] stack is never written. A 4-byte word of frames belongs to the CTA that owns its first
// byte; when it reaches past the tile row, that CTA computes the one next pixel in memory order (the next tile, row,
// word or map) from the global word maps, with the same arithmetic.

// matplotlib's `jet` segment data (_cm.py): piecewise linear through (x, y) in each channel
struct JetSegments { int n; double x[6], y[6]; };
constexpr JetSegments kJet[3] = {
    {5, {0., 0.35, 0.66, 0.89, 1.}, {0., 0., 1., 1., 0.5}},
    {6, {0., 0.125, 0.375, 0.64, 0.91, 1.}, {0., 0., 1., 1., 0., 0.}},
    {5, {0., 0.11, 0.34, 0.65, 1.}, {0.5, 1., 1., 0., 0.}},
};

constexpr double jet_channel(int ch, double x) {
  const JetSegments& s = kJet[ch];
  int i = 0;
  while (i + 2 < s.n && x > s.x[i + 1]) ++i;
  const double t = (x - s.x[i]) / (s.x[i + 1] - s.x[i]);
  const double d = (s.y[i + 1] - s.y[i]) * t;
  return s.y[i] + d;
}

struct JetTable { float v[256 * 3]; };
constexpr JetTable make_jet_table() {
  JetTable t{};
  for (int k = 0; k < 256; ++k)
    for (int ch = 0; ch < 3; ++ch) t.v[3 * k + ch] = (float)(255.0 * jet_channel(ch, k / 255.0));
  return t;
}
constexpr JetTable kJetTable = make_jet_table();
static_assert(kJetTable.v[0] == 0.f && kJetTable.v[1] == 0.f && kJetTable.v[2] == 127.5f, "jet(0) = (0, 0, 0.5)");
static_assert(kJetTable.v[765] == 127.5f && kJetTable.v[766] == 0.f && kJetTable.v[767] == 0.f, "jet(1) = (0.5, 0, 0)");

// L[k][ch] = fp32(255 * jet_ch(k / 255)): the one copy of the table; daam_jet_colormap reads it back
__constant__ JetTable c_jet = kJetTable;

constexpr int kOverlayRowBytes = 16 + 3 * kSegTileW + 16;   // a tile row's bytes from its 16-byte aligned base, + 1 pixel

struct OverlayParams {
  SegmentParams s;                      // maps, word_maps, scratch, sizes, rows, words_per_pass; s.absolute: no min / max
  const unsigned char* image;           // [oh][ow][3], map i at image + i * image_map_stride
  long long image_map_stride;           // bytes; 0: one image for every map
  unsigned char* frames;                // [n_maps][n_words][oh][ow][3], 4-byte aligned, padded to a 4-byte multiple
  int absolute, color_normalize, n_maps;
};

// min / max of the interpolated map v of (map, word), reduced from segment_minmax_kernel's chunks
__device__ __forceinline__ void overlay_v_bounds(const SegmentParams& P, int map, int w, float& lo, float& hi) {
  lo = 0.f; hi = 0.f;
  if (P.absolute) return;                              // no min / max was computed: neither is needed
  const float* slots = P.scratch + 2 * ((long long)map * P.n_words + w) * P.chunks;
  lo = INFINITY; hi = -INFINITY;
  for (int c = 0; c < P.chunks; ++c) { lo = fminf(lo, slots[2 * c]); hi = fmaxf(hi, slots[2 * c + 1]); }
}

// v -> m as expand_words_kernel does it
__device__ __forceinline__ float overlay_m(const OverlayParams& O, float v, float vlo, float vhi) {
  if (!O.absolute) v = minmax_normalize(v, vlo, vhi);
  if (O.s.use_threshold) v = v > O.s.threshold ? 1.f : 0.f;
  return v;
}

// one pixel's three bytes from m, the word's lo / hi of m, the image pixel and the staged table
__device__ __forceinline__ void overlay_rgb(float m, float lo, float hi, int color_normalize, const unsigned char* im,
                                            const float* lut, unsigned char* out) {
  float c;
  if (color_normalize) c = hi == lo ? 0.f : __fdiv_rn(__fsub_rn(m, lo), __fsub_rn(hi, lo));
  else c = fminf(fmaxf(m, 0.f), 1.f);
  const int k = min((int)__fmul_rn(c, 256.f), 255);
  const float a = fminf(fmaxf(m, 0.f), 1.f), na = __fsub_rn(1.f, a);
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    const float v = __fadd_rn(__fmul_rn(na, (float)im[ch]), __fmul_rn(a, lut[3 * k + ch]));
    out[ch] = (unsigned char)min(max(__float2int_rn(v), 0), 255);
  }
}

// The bytes of output pixel (oy, ox) of (map, word), computed from the global word map: the same taps and
// bicubic_shared over the whole map as the tile path over its staged window. Zeros past the last map.
__device__ void overlay_pixel_global(const OverlayParams& O, const float* lut, int map, int w, int oy, int ox,
                                     unsigned char* out) {
  const SegmentParams& P = O.s;
  if (map >= O.n_maps) { out[0] = out[1] = out[2] = 0; return; }
  float vlo, vhi;
  overlay_v_bounds(P, map, w, vlo, vhi);
  const float lo = overlay_m(O, vlo, vlo, vhi), hi = overlay_m(O, vhi, vlo, vhi);
  const float* wm = P.word_maps + ((long long)map * P.n_words + w) * P.mh * P.mw;
  const float v = bicubic_shared(wm, P.mw, make_taps(oy, P.mh, P.oh), make_taps(ox, P.mw, P.ow));
  const unsigned char* im = O.image + map * O.image_map_stride + ((long long)oy * P.ow + ox) * 3;
  const unsigned char px[3] = {__ldg(im), __ldg(im + 1), __ldg(im + 2)};
  overlay_rgb(overlay_m(O, v, vlo, vhi), lo, hi, O.color_normalize, px, lut, out);
}

// grid: (tiles of kSegTileH x kSegTileW output pixels, n_maps); dynamic smem: words_per_pass source windows
__global__ void __launch_bounds__(256) overlay_kernel(const __grid_constant__ OverlayParams O) {
  extern __shared__ __align__(16) float win[];
  __shared__ float s_vlo[kMaxWords], s_vhi[kMaxWords], s_lo[kMaxWords], s_hi[kMaxWords];
  __shared__ int tyi[4][kSegTileH], txi[4][kSegTileW];   // the tile's taps, relative to the staged window
  __shared__ float tyw[4][kSegTileH], txw[4][kSegTileW];
  __shared__ float lut[256 * 3];
  __shared__ unsigned char img[kSegTileH * kSegTileW * 3];
  __shared__ __align__(16) unsigned char rows[2][kSegTileH][kOverlayRowBytes];   // double-buffered across words
  const SegmentParams& P = O.s;
  const int map = blockIdx.y, mh = P.mh, mw = P.mw, oh = P.oh, ow = P.ow, n_words = P.n_words;
  const int tiles_x = (ow + kSegTileW - 1) / kSegTileW;
  const int y0 = (blockIdx.x / tiles_x) * kSegTileH, x0 = (blockIdx.x % tiles_x) * kSegTileW;
  const int th = min(kSegTileH, oh - y0), tw = min(kSegTileW, ow - x0);
  const int wy = make_taps(y0, mh, oh).idx[0], wx = make_taps(x0, mw, ow).idx[0];
  const int wh = make_taps(y0 + th - 1, mh, oh).idx[3] - wy + 1, ww = make_taps(x0 + tw - 1, mw, ow).idx[3] - wx + 1;
  const int wn = wh * ww;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int w = threadIdx.x; w < n_words; w += blockDim.x) {
    float vlo, vhi;
    overlay_v_bounds(P, map, w, vlo, vhi);
    s_vlo[w] = vlo; s_vhi[w] = vhi;
    s_lo[w] = overlay_m(O, vlo, vlo, vhi); s_hi[w] = overlay_m(O, vhi, vlo, vhi);
  }
  for (int i = threadIdx.x; i < 256 * 3; i += blockDim.x) lut[i] = c_jet.v[i];
  if (threadIdx.x < th) {
    const Taps t = make_taps(y0 + threadIdx.x, mh, oh);
#pragma unroll
    for (int j = 0; j < 4; ++j) { tyi[j][threadIdx.x] = t.idx[j] - wy; tyw[j][threadIdx.x] = t.w[j]; }
  } else if (threadIdx.x >= kSegTileH && threadIdx.x < kSegTileH + tw) {
    const int x = threadIdx.x - kSegTileH;
    const Taps t = make_taps(x0 + x, mw, ow);
#pragma unroll
    for (int j = 0; j < 4; ++j) { txi[j][x] = t.idx[j] - wx; txw[j][x] = t.w[j]; }
  }
  // the tile's image bytes, read once for every word
  const unsigned char* image = O.image + map * O.image_map_stride;
  for (int i = threadIdx.x; i < th * tw * 3; i += blockDim.x) {
    const int r = i / (tw * 3), b = i - r * tw * 3;
    img[i] = __ldg(image + ((long long)(y0 + r) * ow + x0) * 3 + b);
  }
  const float* word_maps = P.word_maps + (long long)map * n_words * mh * mw;
  const unsigned long long frames = (unsigned long long)O.frames;   // byte addresses: the alignment of the stores
  for (int w0 = 0; w0 < n_words; w0 += P.words_per_pass) {
    const int nw = min(P.words_per_pass, n_words - w0);
    __syncthreads();                                   // the previous pass has read its windows (and the tables are set)
    for (int i = threadIdx.x; i < nw * wn; i += blockDim.x) {
      const int wi = i / wn, r = i - wi * wn, y = r / ww, x = r - y * ww;
      win[i] = __ldg(word_maps + ((long long)(w0 + wi) * mh + wy + y) * mw + wx + x);
    }
    __syncthreads();
    for (int wi = 0; wi < nw; ++wi) {
      const int w = w0 + wi;
      const float vlo = s_vlo[w], vhi = s_vhi[w], lo = s_lo[w], hi = s_hi[w];
      // row py of the tile starts at byte g0(py) of frames; rows[w & 1][py][g0 & 15] holds that byte
      const long long row0 = (((long long)map * n_words + w) * oh + y0) * ow + x0;
#pragma unroll
      for (int k = 0; k < kSegPix; ++k) {
        const int p = threadIdx.x + 256 * k;
        if (p < th * tw) {
          const int py = p / tw, px = p - py * tw;
          Taps ty, tx;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            ty.idx[j] = tyi[j][py]; ty.w[j] = tyw[j][py]; tx.idx[j] = txi[j][px]; tx.w[j] = txw[j][px];
          }
          const float m = overlay_m(O, bicubic_shared(win + wi * wn, ww, ty, tx), vlo, vhi);
          const unsigned shift = (unsigned)((frames + 3 * (row0 + (long long)py * ow)) & 15);
          overlay_rgb(m, lo, hi, O.color_normalize, img + 3 * p, lut, &rows[w & 1][py][shift + 3 * px]);
        }
      }
      // a row whose last 4-byte word reaches past it: the next pixel in memory order
      if (threadIdx.x < th) {
        const int py = threadIdx.x;
        const unsigned long long g1 = frames + 3 * (row0 + (long long)py * ow + tw);
        if (g1 & 3) {
          int nm = map, nwd = w, ny = y0 + py, nx = x0 + tw;
          if (nx == ow) { nx = 0; ++ny; }
          if (ny == oh) { ny = 0; ++nwd; }
          if (nwd == n_words) { nwd = 0; ++nm; }
          const unsigned shift = (unsigned)((g1 - 3 * tw) & 15);
          overlay_pixel_global(O, lut, nm, nwd, ny, nx, &rows[w & 1][py][shift + 3 * tw]);
        }
      }
      // one barrier per word: rows[w & 1] is rewritten two words later, after every warp has passed the next barrier
      __syncthreads();
      for (int py = warp; py < th; py += 8) {
        const unsigned long long g0 = frames + 3 * (row0 + (long long)py * ow), g1 = g0 + 3 * tw;
        const unsigned long long base = g0 & ~15ull, a0 = (g0 + 3) & ~3ull, a1 = (g1 + 3) & ~3ull;
        // the owned words [a0, a1): 4-byte words up to a 16-byte boundary, 16-byte stores, 4-byte words
        const unsigned long long b0 = min((a0 + 15) & ~15ull, a1), b1 = max(b0, a1 & ~15ull);
        const int n_head = (int)((b0 - a0) >> 2), n_body = (int)((b1 - b0) >> 4), n_tail = (int)((a1 - b1) >> 2);
        const unsigned char* src = rows[w & 1][py];
        for (int j = lane; j < n_head + n_body + n_tail; j += 32) {
          if (j < n_head) {
            const unsigned long long a = a0 + 4 * j;
            *reinterpret_cast<unsigned*>(O.frames + (a - frames)) = *reinterpret_cast<const unsigned*>(src + (a - base));
          } else if (j < n_head + n_body) {
            const unsigned long long a = b0 + 16 * (j - n_head);
            *reinterpret_cast<uint4*>(O.frames + (a - frames)) = *reinterpret_cast<const uint4*>(src + (a - base));
          } else {
            const unsigned long long a = b1 + 4 * (j - n_head - n_body);
            *reinterpret_cast<unsigned*>(O.frames + (a - frames)) = *reinterpret_cast<const unsigned*>(src + (a - base));
          }
        }
      }
    }
  }
}

}  // namespace
}  // namespace daam

using namespace daam;

// DAAM_FINALIZE_GENERIC=1 forces the generic gather kernel (tests compare the two paths)
static bool force_generic_finalize() {
  const char* e = getenv("DAAM_FINALIZE_GENERIC");
  return e && e[0] == '1';
}

// The checks daam_finalize and daam_finalize_per_key share (arguments, device, every key group); `name` is the entry
// point that was called. *n_keys: the keys the groups select.
static int check_key_groups(const char* name, const daam_key_group* groups, int32_t n_groups, int32_t oh, int32_t ow,
                            int32_t n_rows, const float* out, DeviceInfo* dev, int* n_keys) {
  if (!groups || !out || oh <= 0 || ow <= 0 || n_rows <= 0) { set_error("%s: null pointer or non-positive size", name); return DAAM_E_INVALID; }
  if (n_groups <= 0) { set_error("%s: no key selected", name); return DAAM_E_INVALID; }
  if (n_groups > kMaxGroups) { set_error("%s: %d key groups > %d", name, n_groups, kMaxGroups); return DAAM_E_UNSUPPORTED; }
  if (int rc = get_device_info(dev)) return rc;
  *n_keys = 0;
  for (int i = 0; i < n_groups; ++i) {
    const daam_key_group& g = groups[i];
    if (!g.acc || g.heads <= 0 || g.h <= 0 || g.w <= 0 || g.tokens < n_rows || g.head_sel >= g.heads) {
      set_error("%s: bad key group %d (heads %d, h %d, w %d, tokens %d, head_sel %d, n_rows %d)", name, i, g.heads,
                g.h, g.w, g.tokens, g.head_sel, n_rows);
      return DAAM_E_INVALID;
    }
    *n_keys += g.head_sel < 0 ? g.heads : 1;
  }
  return DAAM_OK;
}

// daam_finalize and daam_finalize_maps, after validation: `maps` are MapSel with out, blocks and n_rows set, and every
// map is reduced exactly as daam_finalize reduces the map's expanded group list. The kernel choice and the band height
// are daam_finalize's rule applied per map, so the maps of one call take at most two launches (fast and generic, one
// per kind present) plus one normalisation launch.
static int launch_finalize(const daam_key_group* groups, int32_t n_groups, int32_t oh, int32_t ow, MapSel* maps,
                           int n_maps, int keys_per_block, int32_t normalize, const DeviceInfo& dev, cudaStream_t stream) {
  static thread_local FinalizeParams p;
  p.n_groups = n_groups; p.oh = oh; p.ow = ow;
  for (int i = 0; i < n_groups; ++i) p.g[i] = groups[i];
  const int xx = oh * ow;
  // fast path: every key has one integer factor F = 1 / 2 / 4 on both axes (all SD / SDXL layers that are ever traced)
  // and 16-byte-aligned key bases (cp.async / float4: an aligned slab and h * w a multiple of 4, which keeps every block
  // of a group aligned too). A square map keeps the rule it always had (side a multiple of 16), so its kernel choice
  // and bits do not move. The map's key count (at most kMaxClassKeys) is checked per map below.
  ClassList cls;
  cls.n = 0;
  bool fast_groups = (oh != ow || oh % 16 == 0) && ow <= 256 && !force_generic_finalize();
  for (int i = 0; i < n_groups && fast_groups; ++i) {
    const daam_key_group& g = groups[i];
    const int f = oh / g.h;
    if (oh % g.h != 0 || ow % g.w != 0 || ow / g.w != f || (f != 1 && f != 2 && f != 4) ||
        reinterpret_cast<uintptr_t>(g.acc) % 16 != 0 || (g.h * g.w) % 4 != 0) { fast_groups = false; break; }
    bool seen = false;
    for (int c = 0; c < cls.n; ++c) seen = seen || (cls.kh[c] == g.h && cls.kw[c] == g.w);
    if (!seen) {
      if (cls.n == 8) { fast_groups = false; break; }
      cls.kh[cls.n] = g.h; cls.kw[cls.n] = g.w; ++cls.n;
    }
  }
  if (fast_groups) {
    int next = 0;
    for (int c = 0; c < cls.n; ++c) {                   // keys[] of the kernel: class by class, groups in call order
      cls.key_begin[c] = next;
      for (int i = 0; i < n_groups; ++i)
        if (groups[i].h == cls.kh[c] && groups[i].w == cls.kw[c]) {
          cls.key_slot[i] = next;
          next += groups[i].head_sel < 0 ? groups[i].heads : 1;
        }
    }
    cls.key_begin[cls.n] = next;
  }
  for (int pass = 0; pass < 2; ++pass) {                 // pass 0: the maps on the fast kernel, pass 1: the others
    int n = 0, max_rows = 0, max_br = 4;
    for (int m = 0; m < n_maps; ++m) {
      MapSel s = maps[m];
      s.n_keys = keys_per_block * s.block_count;
      if ((fast_groups && s.n_keys <= kMaxClassKeys) != (pass == 0)) continue;
      // 8-row bands unless that leaves the machine under-filled (< 2 CTAs per SM) or a band's source pixels of the
      // factor-2 class would exceed one CTA's 256 threads (ow > 128); forcing either height measured the same within
      // 1 % for the 175-key SD-2.1 case
      s.band_rows = (((oh + 7) / 8) * s.n_rows >= 2 * dev.sm_count && ow <= 128) ? 8 : 4;
      max_rows = std::max(max_rows, s.n_rows);
      max_br = std::max(max_br, s.band_rows);
      p.map[n++] = s;
    }
    if (n == 0) continue;
    p.n_maps = n;
    if (pass == 0) {
      int bands = 0;
      for (int m = 0; m < n; ++m) bands = std::max(bands, (oh + p.map[m].band_rows - 1) / p.map[m].band_rows);
      const size_t smem = (2 * kStageFloats + (size_t)max_br * ow) * sizeof(float);
      static std::once_flag attr_once[64];
      cudaError_t attr_err = cudaSuccess;
      std::call_once(attr_once[dev.device & 63], [&] {
        attr_err = cudaFuncSetAttribute(finalize_fast_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)((2 * kStageFloats + 8 * 256) * sizeof(float)));
      });
      DAAM_CUDA_TRY(attr_err);
      finalize_fast_kernel<<<dim3(bands, max_rows, n), 256, smem, stream>>>(p, cls);
    } else {
      finalize_kernel<<<dim3((xx + 255) / 256, max_rows, n), 256, 0, stream>>>(p);
    }
    DAAM_CUDA_TRY(cudaGetLastError());
    count_launch();
  }
  if (normalize) {
    MapOuts outs;
    for (int m = 0; m < n_maps; ++m) { outs.out[m] = maps[m].out; outs.n_rows[m] = maps[m].n_rows; }
    normalize_maps_kernel<<<dim3((xx + 255) / 256, n_maps), 256, 0, stream>>>(outs, xx);
    DAAM_CUDA_TRY(cudaGetLastError());
    count_launch();
  }
  return DAAM_OK;
}

extern "C" int daam_finalize(const daam_key_group* groups, int32_t n_groups, int32_t oh, int32_t ow, int32_t n_rows,
                             int32_t normalize, float* out, void* stream_) {
  DeviceInfo dev;
  int n_keys;
  if (int rc = check_key_groups("daam_finalize", groups, n_groups, oh, ow, n_rows, out, &dev, &n_keys)) return rc;
  MapSel map = {out, 0, 1, n_rows, 0, 0};             // block 0 of every group: the groups as given
  return launch_finalize(groups, n_groups, oh, ow, &map, 1, n_keys, normalize, dev, static_cast<cudaStream_t>(stream_));
}

extern "C" int daam_finalize_maps(const daam_key_group* groups, int32_t n_groups, const daam_map_sel* maps,
                                  int32_t n_maps, int32_t oh, int32_t ow, int32_t normalize, void* stream_) {
  const char* name = "daam_finalize_maps";
  if (!maps || n_maps <= 0) { set_error("%s: no output map", name); return DAAM_E_INVALID; }
  if (n_maps > kMaxMaps) { set_error("%s: %d maps > %d", name, n_maps, kMaxMaps); return DAAM_E_UNSUPPORTED; }
  MapSel sel[kMaxMaps];
  int max_rows = 0;
  for (int m = 0; m < n_maps; ++m) {
    const daam_map_sel& s = maps[m];
    if (!s.out || s.n_rows <= 0 || s.block_begin < 0 || s.block_count <= 0) {
      set_error("%s: bad map %d (out %p, n_rows %d, blocks [%d, +%d))", name, m, (void*)s.out, s.n_rows, s.block_begin,
                s.block_count);
      return DAAM_E_INVALID;
    }
    sel[m] = {s.out, s.block_begin, s.block_count, s.n_rows, 0, 0};
    max_rows = std::max(max_rows, s.n_rows);
  }
  DeviceInfo dev;
  int keys_per_block;
  if (int rc = check_key_groups(name, groups, n_groups, oh, ow, max_rows, maps[0].out, &dev, &keys_per_block)) return rc;
  for (int i = 0; i < n_groups; ++i)
    for (int m = 0; m < n_maps; ++m)
      if ((long long)maps[m].block_begin + maps[m].block_count > groups[i].n_blocks) {
        set_error("%s: map %d reads blocks [%d, %lld) but key group %d holds %d", name, m, maps[m].block_begin,
                  (long long)maps[m].block_begin + maps[m].block_count, i, groups[i].n_blocks);
        return DAAM_E_INVALID;
      }
  for (int m = 0; m < n_maps; ++m)
    if ((long long)keys_per_block * maps[m].block_count > (1 << 30)) {
      set_error("%s: map %d selects more than 2^30 keys", name, m);
      return DAAM_E_UNSUPPORTED;
    }
  return launch_finalize(groups, n_groups, oh, ow, sel, n_maps, keys_per_block, normalize, dev,
                         static_cast<cudaStream_t>(stream_));
}

extern "C" int daam_finalize_per_key(const daam_key_group* groups, int32_t n_groups, int32_t oh, int32_t ow,
                                     int32_t n_rows, int32_t normalize, float* out, void* stream_) {
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DeviceInfo dev;
  static thread_local PerKeyParams p;
  if (int rc = check_key_groups("daam_finalize_per_key", groups, n_groups, oh, ow, n_rows, out, &dev, &p.n_keys)) return rc;
  if (p.n_keys > 65535) { set_error("daam_finalize_per_key: %d keys > 65535", p.n_keys); return DAAM_E_UNSUPPORTED; }
  p.n_groups = n_groups; p.oh = oh; p.ow = ow; p.n_rows = n_rows;
  for (int i = 0, first = 0; i < n_groups; ++i) {
    p.g[i] = groups[i];
    p.first_key[i] = first;
    first += groups[i].head_sel < 0 ? groups[i].heads : 1;
  }
  p.first_key[n_groups] = p.n_keys;
  const int xx = oh * ow;
  dim3 grid((xx + 255) / 256, n_rows, p.n_keys);
  finalize_per_key_kernel<<<grid, 256, 0, stream>>>(p, out);
  DAAM_CUDA_TRY(cudaGetLastError());
  count_launch();
  if (normalize) {   // every key's map is an independent [n_rows, oh, ow] block
    normalize_kernel<<<dim3((xx + 255) / 256, p.n_keys), 256, 0, stream>>>(out, n_rows, xx);
    DAAM_CUDA_TRY(cudaGetLastError());
    count_launch();
  }
  return DAAM_OK;
}

extern "C" int daam_normalize_maps(float* maps, int32_t n_maps, int32_t n_rows, int32_t mh, int32_t mw, void* stream_) {
  if (!maps || n_maps < 0 || n_rows <= 0 || mh <= 0 || mw <= 0) { set_error("daam_normalize_maps: null pointer or bad size"); return DAAM_E_INVALID; }
  if (n_maps > 65535) { set_error("daam_normalize_maps: %d maps > 65535", n_maps); return DAAM_E_UNSUPPORTED; }
  if (n_maps == 0) return DAAM_OK;
  DeviceInfo dev;
  if (int rc = get_device_info(&dev)) return rc;
  const int xx = mh * mw;
  normalize_kernel<<<dim3((xx + 255) / 256, n_maps), 256, 0, static_cast<cudaStream_t>(stream_)>>>(maps, n_rows, xx);
  DAAM_CUDA_TRY(cudaGetLastError());
  count_launch();
  return DAAM_OK;
}

extern "C" int daam_word_heat_map(const float* global_maps, int32_t n_rows, int32_t mh, int32_t mw, const int32_t* rows,
                                  int32_t n_sel, float* out, void* stream_) {
  if (!global_maps || !rows || !out || mh <= 0 || mw <= 0 || n_sel <= 0) { set_error("daam_word_heat_map: null pointer or empty selection"); return DAAM_E_INVALID; }
  if (n_sel > kMaxRows) { set_error("daam_word_heat_map: %d rows > %d", n_sel, kMaxRows); return DAAM_E_UNSUPPORTED; }
  DeviceInfo dev;
  if (int rc = get_device_info(&dev)) return rc;
  RowSel sel;
  sel.n = n_sel;
  for (int i = 0; i < n_sel; ++i) {
    int r = rows[i];
    if (r < 0) r += n_rows;   // torch-style negative index
    if (r < 0 || r >= n_rows) { set_error("daam_word_heat_map: row %d out of range [0, %d)", rows[i], n_rows); return DAAM_E_INVALID; }
    sel.rows[i] = r;
  }
  const int xx = mh * mw;
  word_map_kernel<<<(xx + 255) / 256, 256, 0, static_cast<cudaStream_t>(stream_)>>>(global_maps, sel, xx, out);
  DAAM_CUDA_TRY(cudaGetLastError());
  count_launch();
  return DAAM_OK;
}

static int launch_expand_words(ExpandWordsParams& p, const DeviceInfo& dev, cudaStream_t stream) {
  const size_t smem = (size_t)p.mh * p.mw * sizeof(float);
  static std::mutex mu;
  static size_t configured_dev[64] = {};
  static int blocks_per_sm[64] = {};
  int per_sm;
  {
    std::lock_guard<std::mutex> lock(mu);
    size_t& configured = configured_dev[dev.device & 63];
    if (smem > configured) {
      if (smem > 48 * 1024)
        DAAM_CUDA_TRY(cudaFuncSetAttribute(expand_words_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      configured = smem;
      blocks_per_sm[dev.device & 63] = 0;
    }
    if (blocks_per_sm[dev.device & 63] == 0) {
      int occ = 0;
      DAAM_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, expand_words_kernel, 256, configured));
      blocks_per_sm[dev.device & 63] = occ < 1 ? 1 : occ;
    }
    per_sm = blocks_per_sm[dev.device & 63];
  }
  const int capacity = per_sm * dev.sm_count;          // a cooperative grid must be co-resident
  const int n = p.oh * p.ow;
  int done = 0;
  const int total = p.n_words;
  ExpandWordsParams q = p;
  while (done < total) {                                // more words than the device holds at once: several launches
    const int batch = total - done < capacity ? total - done : capacity;
    int chunks = capacity / batch;
    if (chunks > kMaxChunks) chunks = kMaxChunks;
    if (chunks > (n + 255) / 256) chunks = (n + 255) / 256;
    if (chunks < 1) chunks = 1;
    q.n_words = batch;
    q.chunks = chunks;
    q.out = p.out + (long long)done * n;
    q.word_maps = p.word_maps ? p.word_maps + (long long)done * p.mh * p.mw : nullptr;
    q.scratch = p.scratch + 2LL * kMaxChunks * done;
    for (int i = 0; i <= batch; ++i) q.row_begin[i] = p.row_begin[done + i];
    void* args[] = {&q};
    DAAM_CUDA_TRY(cudaLaunchCooperativeKernel((const void*)expand_words_kernel, dim3(batch * chunks), dim3(256), args, smem,
                                              stream));
    count_launch();
    done += batch;
  }
  return DAAM_OK;
}

// behind daam_expand_words and daam_expand_as; `name` is the entry point that was called
static int expand_words_impl(const char* name, const float* global_maps, int32_t n_rows, int32_t mh, int32_t mw,
                             const int32_t* rows, const int32_t* row_begin, int32_t n_words, int32_t out_h, int32_t out_w,
                             int32_t absolute, int32_t use_threshold, float threshold, float* word_maps, float* out,
                             float* scratch, void* stream) {
  if (!global_maps || !rows || !row_begin || !out || !scratch || mh <= 0 || mw <= 0 || out_h <= 0 || out_w <= 0 || n_rows <= 0) { set_error("%s: null pointer or non-positive size", name); return DAAM_E_INVALID; }
  if (n_words <= 0) { set_error("%s: empty word list", name); return DAAM_E_INVALID; }
  if (n_words > kMaxWords) { set_error("%s: %d words > %d", name, n_words, kMaxWords); return DAAM_E_UNSUPPORTED; }
  if (row_begin[0] != 0 || row_begin[n_words] > kMaxWordRows) { set_error("%s: row_begin must start at 0 and select at most %d rows", name, kMaxWordRows); return DAAM_E_UNSUPPORTED; }
  if ((size_t)mh * mw * sizeof(float) > 200 * 1024) { set_error("%s: a %d x %d map does not fit shared memory", name, mh, mw); return DAAM_E_UNSUPPORTED; }
  DeviceInfo dev;
  if (int rc = get_device_info(&dev)) return rc;
  static thread_local ExpandWordsParams p;
  p.maps = global_maps; p.word_maps = word_maps; p.out = out; p.scratch = scratch;
  p.mh = mh; p.mw = mw; p.oh = out_h; p.ow = out_w; p.n_words = n_words; p.chunks = 1;
  p.absolute = absolute ? 1 : 0; p.use_threshold = use_threshold ? 1 : 0; p.threshold = threshold;
  for (int w = 0; w < n_words; ++w) {
    if (row_begin[w + 1] <= row_begin[w]) { set_error("%s: word %d selects no row", name, w); return DAAM_E_INVALID; }
    p.row_begin[w] = row_begin[w];
  }
  p.row_begin[n_words] = row_begin[n_words];
  for (int i = 0; i < row_begin[n_words]; ++i) {
    int r = rows[i];
    if (r < 0) r += n_rows;   // torch-style negative index
    if (r < 0 || r >= n_rows) { set_error("%s: row %d out of range [0, %d)", name, rows[i], n_rows); return DAAM_E_INVALID; }
    p.rows[i] = r;
  }
  return launch_expand_words(p, dev, static_cast<cudaStream_t>(stream));
}

extern "C" int daam_expand_words(const float* global_maps, int32_t n_rows, int32_t mh, int32_t mw, const int32_t* rows,
                                 const int32_t* row_begin, int32_t n_words, int32_t out_h, int32_t out_w,
                                 int32_t absolute, int32_t use_threshold, float threshold, float* word_maps, float* out,
                                 float* scratch, void* stream) {
  return expand_words_impl("daam_expand_words", global_maps, n_rows, mh, mw, rows, row_begin, n_words, out_h, out_w,
                           absolute, use_threshold, threshold, word_maps, out, scratch, stream);
}

// What daam_segment_words, daam_region_overlap and daam_overlay_words share once their own pointers are checked: the word-list, map and
// size checks, `p` (all but labels / scores) and the shared memory of both launches (`*smem1`: one word map for
// segment_minmax_kernel, `*smem2`: words_per_pass staged source windows for the tile kernel). Launches nothing.
static int segment_prepare(const char* name, const float* global_maps, int32_t n_maps, int32_t n_rows, int32_t mh,
                           int32_t mw, const int32_t* rows, const int32_t* row_begin, int32_t n_words, int32_t out_h,
                           int32_t out_w, int32_t absolute, int32_t use_threshold, float threshold, float* word_maps,
                           float* scratch, SegmentParams& p, DeviceInfo* dev, size_t* smem1, size_t* smem2) {
  if (n_words <= 0) { set_error("%s: empty word list", name); return DAAM_E_INVALID; }
  if (n_words > kMaxWords) { set_error("%s: %d words > %d", name, n_words, kMaxWords); return DAAM_E_UNSUPPORTED; }
  if (row_begin[0] != 0 || row_begin[n_words] > kMaxWordRows) { set_error("%s: row_begin must start at 0 and select at most %d rows", name, kMaxWordRows); return DAAM_E_UNSUPPORTED; }
  if ((size_t)mh * mw * sizeof(float) > 200 * 1024) { set_error("%s: a %d x %d map does not fit shared memory", name, mh, mw); return DAAM_E_UNSUPPORTED; }
  if (n_maps > 65535) { set_error("%s: %d maps > 65535", name, n_maps); return DAAM_E_UNSUPPORTED; }
  if ((long long)out_h * out_w > (1LL << 30)) { set_error("%s: a %d x %d output is more than 2^30 pixels", name, out_h, out_w); return DAAM_E_UNSUPPORTED; }
  if (int rc = get_device_info(dev)) return rc;
  for (int w = 0; w < n_words; ++w) {
    if (row_begin[w + 1] <= row_begin[w]) { set_error("%s: word %d selects no row", name, w); return DAAM_E_INVALID; }
    p.row_begin[w] = row_begin[w];
  }
  p.row_begin[n_words] = row_begin[n_words];
  for (int i = 0; i < row_begin[n_words]; ++i) {
    int r = rows[i];
    if (r < 0) r += n_rows;   // torch-style negative index
    if (r < 0 || r >= n_rows) { set_error("%s: row %d out of range [0, %d)", name, rows[i], n_rows); return DAAM_E_INVALID; }
    p.rows[i] = r;
  }
  p.maps = global_maps; p.word_maps = word_maps; p.labels = nullptr; p.scores = nullptr; p.scratch = scratch;
  p.map_stride = (long long)n_rows * mh * mw;
  p.mh = mh; p.mw = mw; p.oh = out_h; p.ow = out_w; p.n_words = n_words;
  p.absolute = absolute ? 1 : 0; p.use_threshold = use_threshold ? 1 : 0; p.threshold = threshold;
  // launch 1: enough (map, word, chunk) CTAs for a few waves, at most kMaxChunks per word and one per 256 pixels
  const long long n = (long long)out_h * out_w, mwords = (long long)n_maps * n_words;
  long long chunks = (4LL * dev->sm_count + mwords - 1) / mwords;
  if (chunks > kMaxChunks) chunks = kMaxChunks;
  if (chunks > (n + 255) / 256) chunks = (n + 255) / 256;
  if (chunks < 1 || p.absolute) chunks = 1;
  p.chunks = (int)chunks;
  // launch 2: a tile's source window is at most ceil(tile * map / out) + 4 rows (columns), and no more than the map
  const int win_h = std::min<int>(mh, (int)ceil((double)kSegTileH * mh / out_h) + 5);
  const int win_w = std::min<int>(mw, (int)ceil((double)kSegTileW * mw / out_w) + 5);
  const int win = win_h * win_w;
  p.words_per_pass = std::max(1, std::min(n_words, kSegStageFloats / win));
  *smem1 = (size_t)mh * mw * sizeof(float);
  *smem2 = (size_t)p.words_per_pass * win * sizeof(float);
  static std::once_flag attr_once[64];
  cudaError_t attr_err = cudaSuccess;
  std::call_once(attr_once[dev->device & 63], [&] {
    attr_err = cudaFuncSetAttribute(segment_minmax_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    if (attr_err == cudaSuccess)
      attr_err = cudaFuncSetAttribute(segment_label_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    if (attr_err == cudaSuccess)
      attr_err = cudaFuncSetAttribute(region_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    if (attr_err == cudaSuccess)
      attr_err = cudaFuncSetAttribute(overlay_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  });
  DAAM_CUDA_TRY(attr_err);
  return DAAM_OK;
}

static int launch_segment_minmax(const SegmentParams& p, int n_maps, size_t smem1, cudaStream_t stream) {
  segment_minmax_kernel<<<(unsigned)((long long)n_maps * p.n_words * p.chunks), 256, smem1, stream>>>(p);
  DAAM_CUDA_TRY(cudaGetLastError());
  count_launch();
  return DAAM_OK;
}

extern "C" int daam_segment_words(const float* global_maps, int32_t n_maps, int32_t n_rows, int32_t mh, int32_t mw,
                                  const int32_t* rows, const int32_t* row_begin, int32_t n_words, int32_t out_h,
                                  int32_t out_w, int32_t absolute, int32_t use_threshold, float threshold,
                                  float* word_maps, uint8_t* labels, float* scores, float* scratch, void* stream_) {
  const char* name = "daam_segment_words";
  if (!global_maps || !rows || !row_begin || !word_maps || !labels || !scores || !scratch || n_maps <= 0 || mh <= 0 ||
      mw <= 0 || out_h <= 0 || out_w <= 0 || n_rows <= 0) { set_error("%s: null pointer or non-positive size", name); return DAAM_E_INVALID; }
  static thread_local SegmentParams p;
  DeviceInfo dev;
  size_t smem1, smem2;
  if (int rc = segment_prepare(name, global_maps, n_maps, n_rows, mh, mw, rows, row_begin, n_words, out_h, out_w,
                               absolute, use_threshold, threshold, word_maps, scratch, p, &dev, &smem1, &smem2)) return rc;
  p.labels = labels; p.scores = scores;
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (int rc = launch_segment_minmax(p, n_maps, smem1, stream)) return rc;
  const int tiles = ((out_h + kSegTileH - 1) / kSegTileH) * ((out_w + kSegTileW - 1) / kSegTileW);
  segment_label_kernel<<<dim3(tiles, n_maps), 256, smem2, stream>>>(p);
  DAAM_CUDA_TRY(cudaGetLastError());
  count_launch();
  return DAAM_OK;
}

extern "C" int daam_region_overlap(const float* global_maps, int32_t n_maps, int32_t n_rows, int32_t mh, int32_t mw,
                                   const int32_t* rows, const int32_t* row_begin, int32_t n_words, int32_t out_h,
                                   int32_t out_w, int32_t absolute, int32_t use_threshold, float threshold,
                                   float* word_maps, const uint8_t* regions, int32_t n_regions, float* intersection,
                                   float* word_area, float* scratch, void* stream_) {
  const char* name = "daam_region_overlap";
  if (!global_maps || !rows || !row_begin || !word_maps || !regions || !intersection || !word_area || !scratch ||
      n_maps <= 0 || mh <= 0 || mw <= 0 || out_h <= 0 || out_w <= 0 || n_rows <= 0 || n_regions <= 0) { set_error("%s: null pointer or non-positive size", name); return DAAM_E_INVALID; }
  if (n_regions > kMaxRegions) { set_error("%s: %d regions > %d", name, n_regions, kMaxRegions); return DAAM_E_UNSUPPORTED; }
  // fp32 partial sums of 0/1 values stay exact integers up to 2^24
  if ((long long)out_h * out_w > (1LL << 24)) { set_error("%s: a %d x %d output is more than 2^24 pixels", name, out_h, out_w); return DAAM_E_UNSUPPORTED; }
  static thread_local RegionParams p;
  DeviceInfo dev;
  size_t smem1, smem2;
  if (int rc = segment_prepare(name, global_maps, n_maps, n_rows, mh, mw, rows, row_begin, n_words, out_h, out_w,
                               absolute, use_threshold, threshold, word_maps, scratch, p.s, &dev, &smem1, &smem2)) return rc;
  const int tiles = ((out_h + kSegTileH - 1) / kSegTileH) * ((out_w + kSegTileW - 1) / kSegTileW);
  p.regions = regions; p.n_regions = n_regions; p.tiles = tiles;
  p.partials = scratch + 64LL * n_maps * n_words;     // after segment_minmax_kernel's min / max partials
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (int rc = launch_segment_minmax(p.s, n_maps, smem1, stream)) return rc;
  region_tile_kernel<<<dim3(tiles, n_maps), 256, smem2, stream>>>(p);
  DAAM_CUDA_TRY(cudaGetLastError());
  count_launch();
  const long long n_out = (long long)n_maps * n_words * (n_regions + 1);
  region_reduce_kernel<<<(unsigned)((n_out + 7) / 8), 256, 0, stream>>>(p.partials, n_out, tiles, n_words, n_regions,
                                                                        intersection, word_area);
  DAAM_CUDA_TRY(cudaGetLastError());
  count_launch();
  return DAAM_OK;
}

extern "C" int daam_overlay_words(const float* global_maps, int32_t n_maps, int32_t n_rows, int32_t mh, int32_t mw,
                                  const int32_t* rows, const int32_t* row_begin, int32_t n_words, int32_t out_h,
                                  int32_t out_w, int32_t absolute, int32_t use_threshold, float threshold,
                                  int32_t color_normalize, float* word_maps, const uint8_t* image,
                                  int64_t image_map_stride, uint8_t* frames, float* scratch, void* stream_) {
  const char* name = "daam_overlay_words";
  if (!global_maps || !rows || !row_begin || !word_maps || !image || !frames || !scratch || n_maps <= 0 || mh <= 0 ||
      mw <= 0 || out_h <= 0 || out_w <= 0 || n_rows <= 0 || image_map_stride < 0) { set_error("%s: null pointer or non-positive size", name); return DAAM_E_INVALID; }
  if ((uintptr_t)frames & 3) { set_error("%s: frames must be 4-byte aligned", name); return DAAM_E_INVALID; }
  static thread_local OverlayParams p;
  DeviceInfo dev;
  size_t smem1, smem2;
  // segment_minmax_kernel computes the min / max of v unless neither the normalisation nor the colour scale needs it
  const int skip_minmax = absolute && !color_normalize;
  if (int rc = segment_prepare(name, global_maps, n_maps, n_rows, mh, mw, rows, row_begin, n_words, out_h, out_w,
                               skip_minmax, use_threshold, threshold, word_maps, scratch, p.s, &dev, &smem1, &smem2)) return rc;
  p.image = image; p.image_map_stride = image_map_stride; p.frames = frames;
  p.absolute = absolute ? 1 : 0; p.color_normalize = color_normalize ? 1 : 0; p.n_maps = n_maps;
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (int rc = launch_segment_minmax(p.s, n_maps, smem1, stream)) return rc;
  const int tiles = ((out_h + kSegTileH - 1) / kSegTileH) * ((out_w + kSegTileW - 1) / kSegTileW);
  overlay_kernel<<<dim3(tiles, n_maps), 256, smem2, stream>>>(p);
  DAAM_CUDA_TRY(cudaGetLastError());
  count_launch();
  return DAAM_OK;
}

extern "C" int daam_jet_colormap(float* out) {
  if (!out) { set_error("daam_jet_colormap: null pointer"); return DAAM_E_INVALID; }
  DAAM_CUDA_TRY(cudaMemcpyFromSymbol(out, c_jet, sizeof(JetTable)));
  return DAAM_OK;
}

// one word whose "rows" are the word map itself
extern "C" int daam_expand_as(const float* word_map, int32_t mh, int32_t mw, int32_t out_h, int32_t out_w,
                              int32_t absolute, int32_t use_threshold, float threshold, float* out, float* scratch,
                              void* stream) {
  const int32_t rows[1] = {0}, row_begin[2] = {0, 1};
  return expand_words_impl("daam_expand_as", word_map, 1, mh, mw, rows, row_begin, 1, out_h, out_w, absolute,
                           use_threshold, threshold, nullptr, out, scratch, stream);
}
