// Finalize kernels: the key reductions behind a global heat map -- per-key bicubic upsample (bicubic.cuh) -> clamp
// -> mean over keys -- and the normalisation of finished maps.
//
// Replaces DiffusionHeatMapHooker.compute_global_heat_map (daam/trace.py:109-130).
#include <math.h>
#include <stdlib.h>

#include <algorithm>
#include <mutex>

#include "bicubic.cuh"
#include "common.cuh"

namespace daam {
namespace {

constexpr int kMaxGroups = 160;   // key groups (layer x prompt slices) per finalize launch
constexpr int kMaxMaps = DAAM_FINALIZE_MAX_MAPS;   // output maps per finalize launch

// One output map of a finalize launch: blocks [block_begin, block_begin + block_count) of the groups [group_begin,
// group_begin + group_count), i.e. the keys of the expanded group list `for g: for b: {acc_g + b * heads_g * tokens_g *
// h_g * w_g, heads_g, head_sel_g}`. daam_finalize_maps selects blocks of every group, daam_finalize_parts groups.
struct MapSel {
  float* out;                             // [n_rows][oh][ow]
  int block_begin, block_count, n_rows, n_keys;
  int band_rows;                          // fast kernel only: 8 or 4 (daam_finalize's rule for this map's n_rows)
  int group_begin, group_count;
  // Fast kernel only (n_classes 0: the map takes the generic kernel): the map's OWN key classes. A fast key has one
  // integer factor 1 / 2 / 4 on both axes, so a class is a source size (kh, kw) = (oh / F, ow / F) and a map has at most
  // three, kept in the order its groups first show them. Per block: keys[] is ordered class by class, class c owns
  // [key_begin[c], key_begin[c + 1]) times the map's block count, and a group g of class c starts at (key_slot0[c] +
  // FinalizeParams::class_keys_before[g]) times the block count, block by block, head by head.
  int n_classes;
  int kh[3], kw[3];
  int key_begin[4];
  int key_slot0[3];                       // key_begin[c] less the class's keys in the groups before group_begin
};

MapSel make_map(float* out, int block_begin, int block_count, int n_rows, int group_begin, int group_count) {
  MapSel s = {};
  s.out = out; s.block_begin = block_begin; s.block_count = block_count; s.n_rows = n_rows;
  s.group_begin = group_begin; s.group_count = group_count;
  return s;
}

struct FinalizeParams {
  int n_groups, oh, ow, n_maps;           // output maps [oh][ow]
  daam_key_group g[kMaxGroups];
  // fast kernel only: keys per block of the groups before g that have g's size (the same for every map of the launch)
  int class_keys_before[kMaxGroups];
  MapSel map[kMaxMaps];                   // blockIdx.z selects the map
  // weighted instances only: the [n_blocks][heads][tokens] weights of group g (its acc layout with h * w = 1), or null.
  // Last, so that the fields the plain instances read keep their offsets.
  const float* w[kMaxGroups];
};

// grid: (ceil(oh*ow / 256), max n_rows, n_maps). One thread = one output element (map, row t, pixel o); it walks every
// selected key: group by group, block by block, head by head. kWeighted: each clamped key value is scaled by its weight,
// `sum = fmaf(w, clamp(v), sum)`, instead of added.
template <bool kWeighted>
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
  for (int g = M.group_begin; g < M.group_begin + M.group_count; ++g) {
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
      if constexpr (kWeighted) {
        const float* wb = P.w[g] + ((long long)b * G.heads) * G.tokens + t;
        if (same) {
#pragma unroll 4
          for (int head = h0; head < h1; ++head)
            sum = fmaf(__ldg(wb + head * G.tokens), fmaxf(__ldg(base + head * head_stride + o), 0.f), sum);
        } else {
#pragma unroll 2
          for (int head = h0; head < h1; ++head)
            sum = fmaf(__ldg(wb + head * G.tokens), fmaxf(bicubic_at(base + head * head_stride, G.w, ty, tx), 0.f), sum);
        }
      } else if (same) {   // scale 1: the cubic weights are exactly (0, 1, 0, 0)
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

template <int F, bool kWeighted>
__device__ __forceinline__ void add_key(const PhaseWeights<F>& pw, const float (&v)[5][5], float (&acc)[F][F],
                                        float weight) {
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
      if constexpr (kWeighted) acc[py][px] = fmaf(weight, fmaxf(o, 0.f), acc[py][px]);
      else acc[py][px] += fmaxf(o, 0.f);
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
// chunk is issued here). `weights`: the class's key weights, parallel to `keys` (kWeighted only).
template <int F, bool kWeighted>
__device__ __forceinline__ void class_pass(const FinalizeParams& P, int kh, int kw, int nk, int band, int br, float* tile,
                                           const float* const* keys, const float* weights, float* stage, bool prefetched,
                                           const NextClass& next) {
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
        add_key<F, kWeighted>(pw, v, acc, kWeighted ? weights[c * kc + k] : 1.f);
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
template <bool kWeighted>
__device__ __forceinline__ void class_pass_identity(const FinalizeParams& P, int nk, int band, int br, int rows, float* tile,
                                                    const float* const* keys, const float* weights, float* stage,
                                                    const NextClass& next) {
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
        if constexpr (kWeighted) {
          const float wk = weights[k];
          acc.x = fmaf(wk, fmaxf(v.x, 0.f), acc.x); acc.y = fmaf(wk, fmaxf(v.y, 0.f), acc.y);
          acc.z = fmaf(wk, fmaxf(v.z, 0.f), acc.z); acc.w = fmaf(wk, fmaxf(v.w, 0.f), acc.w);
        } else {
          acc.x += fmaxf(v.x, 0.f); acc.y += fmaxf(v.y, 0.f); acc.z += fmaxf(v.z, 0.f); acc.w += fmaxf(v.w, 0.f);
        }
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

// grid: (ceil(oh / 4) bands, max n_rows, n_maps); a CTA past its map's bands or rows returns at once. Dynamic smem: two
// chunk buffers + the band tile (the largest band_rows of the launch * ow floats). kWeighted: every key's weight for row
// t is staged next to its pointer (8 KB more static smem; still two CTAs per SM).
template <bool kWeighted>
__global__ void __launch_bounds__(256, 2) finalize_fast_kernel(const __grid_constant__ FinalizeParams P) {
  extern __shared__ __align__(16) float dyn[];
  __shared__ const float* keys[kMaxClassKeys];
  float* wts = nullptr;
  if constexpr (kWeighted) {
    __shared__ float key_weights[kMaxClassKeys];
    wts = key_weights;
  }
  float* stage = dyn;                                  // 2 x kStageFloats
  float* tile = dyn + 2 * kStageFloats;
  const MapSel& M = P.map[blockIdx.z];
  const int band = blockIdx.x, t = blockIdx.y, oh = P.oh, ow = P.ow, br = M.band_rows, nb = M.block_count;
  if (t >= M.n_rows || band * br >= oh) return;
  const int rows = min(br, oh - band * br);            // valid output rows of this band
  // key pointers (token row t) of every selected key, class by class; one thread per key group of the map
  for (int g = M.group_begin + threadIdx.x; g < M.group_begin + M.group_count; g += blockDim.x) {
    const daam_key_group& G = P.g[g];
    const int per_block = G.head_sel < 0 ? G.heads : 1;
    const long long hw = (long long)G.h * G.w;
    const int slot0 = G.w == M.kw[0] ? M.key_slot0[0] : (G.w == M.kw[1] ? M.key_slot0[1] : M.key_slot0[2]);
    const float** dst = keys + (slot0 + P.class_keys_before[g]) * nb;
    // key j of the group: head (block_begin * heads + j) of all heads, or head_sel of block block_begin + j
    const long long first = G.head_sel < 0 ? (long long)M.block_begin * G.heads : (long long)M.block_begin * G.heads + G.head_sel;
    const long long step = G.head_sel < 0 ? 1 : G.heads;
    for (int j = 0; j < per_block * nb; ++j) dst[j] = G.acc + ((first + j * step) * G.tokens + t) * hw;
    if constexpr (kWeighted) {
      float* wdst = wts + (dst - keys);
      for (int j = 0; j < per_block * nb; ++j) wdst[j] = __ldg(P.w[g] + (first + j * step) * G.tokens + t);
    }
  }
  for (int i = threadIdx.x; i < br * ow; i += blockDim.x) tile[i] = 0.f;
  __syncthreads();
  bool prefetched = false;                             // chunk 0 of class c is already streaming into buffer 1
  for (int c = 0; c < M.n_classes; ++c) {                // the map's own classes: maps of one launch differ in them
    const int kh = M.kh[c], kw = M.kw[c], f = ow / kw, nk = (M.key_begin[c + 1] - M.key_begin[c]) * nb;
    const float* const* ck = keys + M.key_begin[c] * nb;
    const float* cw = kWeighted ? wts + M.key_begin[c] * nb : nullptr;
    NextClass next = {0, 0, 0, 0, nullptr};
    if (c + 1 < M.n_classes && M.kw[c + 1] != ow)
      next = {M.kh[c + 1], M.kw[c + 1], ow / M.kw[c + 1], (M.key_begin[c + 2] - M.key_begin[c + 1]) * nb,
              keys + M.key_begin[c + 1] * nb};
    if (f == 1) class_pass_identity<kWeighted>(P, nk, band, br, rows, tile, ck, cw, stage, next);
    else if (f == 2) class_pass<2, kWeighted>(P, kh, kw, nk, band, br, tile, ck, cw, stage, prefetched, next);
    else class_pass<4, kWeighted>(P, kh, kw, nk, band, br, tile, ck, cw, stage, prefetched, next);
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

// The fast kernel's dynamic shared memory opt-in, once per device and instance.
template <bool kWeighted>
static cudaError_t allow_fast_smem(int device) {
  static std::once_flag once[64];
  cudaError_t err = cudaSuccess;
  std::call_once(once[device & 63], [&] {
    err = cudaFuncSetAttribute(finalize_fast_kernel<kWeighted>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                               (int)((2 * kStageFloats + 8 * 256) * sizeof(float)));
  });
  return err;
}

// daam_finalize, daam_finalize_maps, daam_finalize_parts and daam_finalize_parts_weighted, after validation: `maps` are
// MapSel with out, blocks, groups and n_rows set, and every map is reduced exactly as daam_finalize reduces the map's
// expanded group list. The kernel choice and the band height are daam_finalize's rule applied per map, to the map's own
// groups, so the maps of one call take at most two launches (fast and generic, one per kind present) plus one
// normalisation launch. `weights` (one device pointer per group, or null): the weighted instances, same choice.
static int launch_finalize(const char* name, const daam_key_group* groups, int32_t n_groups, int32_t oh, int32_t ow,
                           MapSel* maps, int n_maps, int32_t normalize, const DeviceInfo& dev, cudaStream_t stream,
                           const float* const* weights = nullptr) {
  static thread_local FinalizeParams p;
  p.n_groups = n_groups; p.oh = oh; p.ow = ow;
  for (int i = 0; i < n_groups; ++i) p.g[i] = groups[i];
  for (int i = 0; i < n_groups; ++i) p.w[i] = weights ? weights[i] : nullptr;
  const int xx = oh * ow;
  // fast path: every key of the map has one integer factor F = 1 / 2 / 4 on both axes (all SD / SDXL layers that are
  // ever traced) and a 16-byte-aligned key base (cp.async / float4: an aligned slab and h * w a multiple of 4, which
  // keeps every block of a group aligned too). A square map keeps the rule it always had (side a multiple of 16), so its
  // kernel choice and bits do not move. Such keys have one of three sizes, (oh / F, ow / F), so the limit of 8 key sizes
  // a map may show can never bind. The map's key count (at most kMaxClassKeys) is checked per map below.
  const bool fast_grid = (oh != ow || oh % 16 == 0) && ow <= 256 && !force_generic_finalize();
  int factor[kMaxGroups];                                // of a group the fast kernel can read, else 0
  int seen[5] = {0, 0, 0, 0, 0};                         // keys per block so far of the class with factor F
  for (int i = 0; i < n_groups; ++i) {
    const daam_key_group& g = groups[i];
    const int f = oh / g.h;
    const bool ok = fast_grid && oh % g.h == 0 && ow % g.w == 0 && ow / g.w == f && (f == 1 || f == 2 || f == 4) &&
                    reinterpret_cast<uintptr_t>(g.acc) % 16 == 0 && (g.h * g.w) % 4 == 0;
    factor[i] = ok ? f : 0;
    p.class_keys_before[i] = seen[factor[i]];
    seen[factor[i]] += g.head_sel < 0 ? g.heads : 1;
  }
  for (int m = 0; m < n_maps; ++m) {                     // the map's keys and, if it can take the fast kernel, classes
    MapSel& s = maps[m];
    long long per_block = 0;
    int keys_of[5] = {0, 0, 0, 0, 0}, nc = 0;            // nc: the map's classes so far, -1 once a group is not fast
    for (int i = s.group_begin; i < s.group_begin + s.group_count; ++i) {
      const int k = groups[i].head_sel < 0 ? groups[i].heads : 1, f = factor[i];
      per_block += k;
      if (f == 0 || nc < 0) { nc = -1; continue; }
      if (keys_of[f] == 0) {                             // first seen: the class's keys before the map, for key_slot0
        s.kh[nc] = groups[i].h; s.kw[nc] = groups[i].w;
        s.key_slot0[nc++] = p.class_keys_before[i];
      }
      keys_of[f] += k;
    }
    if (per_block * s.block_count > (1 << 30)) {
      set_error("%s: map %d selects more than 2^30 keys", name, m);
      return DAAM_E_UNSUPPORTED;
    }
    s.n_keys = (int)per_block * s.block_count;
    if (s.n_keys > kMaxClassKeys) nc = -1;
    s.n_classes = std::max(nc, 0);
    for (int c = 0, next = 0; c < s.n_classes; ++c) {    // keys[] of the kernel: class by class, groups in call order
      s.key_begin[c] = next;
      s.key_slot0[c] = next - s.key_slot0[c];
      next += keys_of[oh / s.kh[c]];
      s.key_begin[c + 1] = next;
    }
    for (int c = s.n_classes; c < 3; ++c) s.kh[c] = s.kw[c] = 0;
  }
  for (int pass = 0; pass < 2; ++pass) {                 // pass 0: the maps on the fast kernel, pass 1: the others
    int n = 0, max_rows = 0, max_br = 4;
    for (int m = 0; m < n_maps; ++m) {
      MapSel s = maps[m];
      if ((s.n_classes > 0) != (pass == 0)) continue;
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
      const dim3 grid(bands, max_rows, n);
      if (weights) {
        DAAM_CUDA_TRY(allow_fast_smem<true>(dev.device));
        finalize_fast_kernel<true><<<grid, 256, smem, stream>>>(p);
      } else {
        DAAM_CUDA_TRY(allow_fast_smem<false>(dev.device));
        finalize_fast_kernel<false><<<grid, 256, smem, stream>>>(p);
      }
    } else if (weights) {
      finalize_kernel<true><<<dim3((xx + 255) / 256, max_rows, n), 256, 0, stream>>>(p);
    } else {
      finalize_kernel<false><<<dim3((xx + 255) / 256, max_rows, n), 256, 0, stream>>>(p);
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
  MapSel map = make_map(out, 0, 1, n_rows, 0, n_groups);   // block 0 of every group: the groups as given
  return launch_finalize("daam_finalize", groups, n_groups, oh, ow, &map, 1, normalize, dev,
                         static_cast<cudaStream_t>(stream_));
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
    sel[m] = make_map(s.out, s.block_begin, s.block_count, s.n_rows, 0, n_groups);
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
  return launch_finalize(name, groups, n_groups, oh, ow, sel, n_maps, normalize, dev, static_cast<cudaStream_t>(stream_));
}

// daam_finalize_parts and daam_finalize_parts_weighted (`weights` null: the plain reduction)
static int finalize_parts(const char* name, const daam_key_group* groups, int32_t n_groups, const daam_map_part* maps,
                          int32_t n_maps, int32_t oh, int32_t ow, int32_t normalize, const float* const* weights,
                          void* stream_) {
  if (!maps || n_maps <= 0) { set_error("%s: no output map", name); return DAAM_E_INVALID; }
  if (n_maps > kMaxMaps) { set_error("%s: %d maps > %d", name, n_maps, kMaxMaps); return DAAM_E_UNSUPPORTED; }
  auto bad_map = [&](int m) {
    set_error("%s: bad map %d (out %p, n_rows %d, groups [%d, +%d) of %d)", name, m, (void*)maps[m].out, maps[m].n_rows,
              maps[m].group_begin, maps[m].group_count, n_groups);
    return DAAM_E_INVALID;
  };
  for (int m = 0; m < n_maps; ++m)
    if (!maps[m].out || maps[m].n_rows <= 0 || maps[m].group_begin < 0 || maps[m].group_count <= 0) return bad_map(m);
  DeviceInfo dev;
  int n_keys;                                            // every group is checked, read by a map or not
  if (int rc = check_key_groups(name, groups, n_groups, oh, ow, 1, maps[0].out, &dev, &n_keys)) return rc;
  MapSel sel[kMaxMaps];
  for (int m = 0; m < n_maps; ++m) {
    const daam_map_part& s = maps[m];
    if ((long long)s.group_begin + s.group_count > n_groups) return bad_map(m);
    for (int i = s.group_begin; i < s.group_begin + s.group_count; ++i)
      if (groups[i].tokens < s.n_rows) {
        set_error("%s: map %d reads %d rows but key group %d holds %d", name, m, s.n_rows, i, groups[i].tokens);
        return DAAM_E_INVALID;
      }
    sel[m] = make_map(s.out, 0, 1, s.n_rows, s.group_begin, s.group_count);
  }
  return launch_finalize(name, groups, n_groups, oh, ow, sel, n_maps, normalize, dev, static_cast<cudaStream_t>(stream_),
                         weights);
}

extern "C" int daam_finalize_parts(const daam_key_group* groups, int32_t n_groups, const daam_map_part* maps,
                                   int32_t n_maps, int32_t oh, int32_t ow, int32_t normalize, void* stream_) {
  return finalize_parts("daam_finalize_parts", groups, n_groups, maps, n_maps, oh, ow, normalize, nullptr, stream_);
}

extern "C" int daam_finalize_parts_weighted(const daam_key_group* groups, int32_t n_groups, const daam_map_part* maps,
                                            int32_t n_maps, int32_t oh, int32_t ow, int32_t normalize,
                                            const float* const* weights, void* stream_) {
  const char* name = "daam_finalize_parts_weighted";
  if (!weights) { set_error("%s: null weights", name); return DAAM_E_INVALID; }
  for (int i = 0; i < n_groups && i < kMaxGroups; ++i)
    if (!weights[i]) { set_error("%s: null weights of key group %d", name, i); return DAAM_E_INVALID; }
  return finalize_parts(name, groups, n_groups, maps, n_maps, oh, ow, normalize, weights, stream_);
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
