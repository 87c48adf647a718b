// Word-list kernels: a word's heat map (the mean of its rows of a global map), and one pipeline that takes a list of
// words from the global map to image-size results without writing the [n_words][out_h][out_w] stack of expanded maps.
//
// Replaces GlobalHeatMap.compute_word_heat_map (daam/heatmap.py:121-123) and WordHeatMap.expand_as
// (daam/heatmap.py:77-93) over a word list. Every consumer runs the same steps:
//  1. word map: the gather-mean of the word's rows (word_mean) into shared memory;
//  2. min / max of the bicubic-interpolated word map v over the image, per chunk of output pixels, then over the
//     chunks in a fixed order (partial_bounds);
//  3. the tile kernels stage the source window under a 16 x 64 output tile for a pass of words;
//  4. per pixel: interpolate (bicubic.cuh), normalise and threshold: m = word_value(v), what expand_as returns.
// The consumers differ only in what they do with m:
//  - expand_words_kernel writes it (one cooperative launch, steps 1, 2 and 4 in one kernel);
//  - segment_label_kernel keeps each pixel's max / argmax over the words;
//  - region_tile_kernel sums it over binary image regions (then region_reduce_kernel);
//  - region_sweep_tile_kernel counts, per region, the pixels where it passes each of a list of thresholds (then
//    region_sweep_reduce_kernel);
//  - overlay_kernel blends its jet colour onto the image;
//  - word_pair_tile_kernel sums m[a] * m[b] over every pair of words (then word_pair_reduce_kernel);
//  - instance_mask_kernel writes it without threshold for components.cu, which labels the mask m > threshold, and
//    for ranking.cu, which sorts it and scores it against regions (daam_region_ranking), and for boundary.cu, which
//    measures the boundary of m > threshold against the regions' boundaries (daam_region_boundary), and for
//    distance.cu, which takes the signed distance transform of m > threshold (daam_word_distance);
//  - refine.cu recomputes it from segment_minmax_kernel's word maps and partials and filters it with the image as
//    guide (daam_refine_words);
//  - crf.cu recomputes it the same way as the unary logits of a Potts CRF with the image as bilateral guide
//    (daam_segment_crf);
//  - superpixels.cu recomputes it the same way and averages it over each SLIC superpixel of the image, whose words
//    then compete per superpixel (daam_segment_superpixels).
// word_value.cuh defines m's pieces (word_mean, partial_bounds, minmax_normalize): every consumer's m, here and in
// refine.cu, crf.cu and superpixels.cu, is built from them and is expand_words_kernel's value bit for bit. The tile kernels run after
// segment_minmax_kernel (steps 1 and 2, the word maps and min / max partials to global memory) and share the tile
// helpers (block_tile / tile_at, word_bounds, stage_windows, tap tables, and tile_value in the two that also run
// without staged windows). expand_words_kernel, segment_minmax_kernel and segment_label_kernel keep their steps
// inline: written with the helpers, nvcc scheduled them differently and they measured slower. Deterministic: the only
// atomics here are region_sweep_tile_kernel's integer adds (and components.cu's are integer atomics), whose results do
// not depend on their order.
#include <cooperative_groups.h>
#include <math.h>

#include <algorithm>
#include <mutex>

#include "bicubic.cuh"
#include "boundary.cuh"
#include "common.cuh"
#include "components.cuh"
#include "crf.cuh"
#include "distance.cuh"
#include "ranking.cuh"
#include "refine.cuh"
#include "superpixels.cuh"
#include "word_value.cuh"

namespace daam {
namespace {

constexpr int kMaxRows = 128;                       // selected rows of daam_word_heat_map
constexpr int kMaxWords = 96;
constexpr int kMaxWordRows = 320;                   // selected rows over all words of a launch
constexpr int kMaxSmem = 200 * 1024;                // dynamic shared memory: a word map, or a tile kernel's windows
constexpr int kSegTileH = 16, kSegTileW = 64;       // output tile of one tile-kernel CTA
constexpr int kSegPix = kSegTileH * kSegTileW / 256;   // output pixels per thread
constexpr int kSegStageFloats = 12288;              // staged windows per pass when they fit (48 KB)

struct RowSel {
  int n;
  int rows[kMaxRows];
};

__global__ void word_map_kernel(const float* __restrict__ maps, const __grid_constant__ RowSel sel, int xx,
                                float* __restrict__ out) {
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= xx) return;
  out[o] = word_mean(maps, sel.rows, 0, sel.n, xx, o);
}

// What every word-list kernel reads; each kernel's params add its outputs.
struct WordListParams {
  const float* maps;                    // [n_maps][n_map_rows][mh][mw]
  float* word_maps;                     // [n_maps][n_words][mh][mw] (optional for expand_words_kernel)
  float* scratch;                       // min / max partials [n_maps][n_words][chunks][2]
  long long map_stride;                 // n_map_rows * mh * mw
  int mh, mw, oh, ow, n_words, chunks, absolute, use_threshold;
  float threshold;
  int words_per_pass;                   // tile kernels: words whose windows are staged at once
  int minmax;                           // the min / max partials are computed and read
  int row_begin[kMaxWords + 1];
  int rows[kMaxWordRows];
};

// v at output pixel (oy, ox), from a whole word map
__device__ __forceinline__ float word_map_at(const WordListParams& P, const float* wm, int oy, int ox) {
  return bicubic_shared(wm, P.mw, make_taps(oy, P.mh, P.oh), make_taps(ox, P.mw, P.ow));
}

// v -> m, for a word whose v has min / max lo / hi
__device__ __forceinline__ float word_value(const WordListParams& P, float v, float lo, float hi) {
  if (!P.absolute) v = minmax_normalize(v, lo, hi);
  if (P.use_threshold) v = v > P.threshold ? 1.f : 0.f;
  return v;
}

// ---- expand: the word list's m written out ----------------------------------------------------------------------
// CTA = (word, chunk of output pixels). The word map lives in shared memory; the min/max pass and the write pass both
// interpolate from it (16 shared loads + 20 FMAs per pixel), so nothing but the final image is written and nothing is
// read back. The chunks' min / max go through `scratch` across one grid-wide barrier; with `absolute` there is no
// min/max pass and no barrier.
struct ExpandParams {
  WordListParams s;                     // one map
  float* out;                           // [n_words][oh][ow]
};

__global__ void __launch_bounds__(256) expand_words_kernel(const __grid_constant__ ExpandParams E) {
  const WordListParams& P = E.s;
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
  float* dst = E.out + (long long)word * n;
  for (int o = begin + threadIdx.x; o < end; o += blockDim.x) {
    const int oy = o / P.ow, ox = o - oy * P.ow;
    dst[o] = word_value(P, word_map_at(P, wm, oy, ox), lo, hi);
  }
}

// ---- the tile kernels' first launch and the helpers they share ------------------------------------------------
// grid: n_maps * n_words * chunks, CTA = (map, word, chunk of output pixels); dynamic smem: the word map [mh][mw].
// Chunk 0 writes the word map; with `minmax` every chunk writes its min / max of v to `scratch`.
__global__ void __launch_bounds__(256) segment_minmax_kernel(const __grid_constant__ WordListParams P) {
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
  if (!P.minmax) return;
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

// A tile kernel's CTA: output rows [y0, y0 + th) and columns [x0, x0 + tw) of map blockIdx.y, and the source window
// [wy, wy + wh) x [wx, wx + ww) (wn floats) its taps read: taps move monotonically with the output index
struct Tile {
  int y0, x0, th, tw, wy, wx, wh, ww, wn;
};

__device__ __forceinline__ Tile tile_at(const WordListParams& P, unsigned tile) {
  const int tiles_x = (P.ow + kSegTileW - 1) / kSegTileW;
  Tile t;
  t.y0 = (tile / tiles_x) * kSegTileH; t.x0 = (tile % tiles_x) * kSegTileW;
  t.th = min(kSegTileH, P.oh - t.y0); t.tw = min(kSegTileW, P.ow - t.x0);
  t.wy = make_taps(t.y0, P.mh, P.oh).idx[0]; t.wx = make_taps(t.x0, P.mw, P.ow).idx[0];
  t.wh = make_taps(t.y0 + t.th - 1, P.mh, P.oh).idx[3] - t.wy + 1;
  t.ww = make_taps(t.x0 + t.tw - 1, P.mw, P.ow).idx[3] - t.wx + 1;
  t.wn = t.wh * t.ww;
  return t;
}

__device__ __forceinline__ Tile block_tile(const WordListParams& P) { return tile_at(P, blockIdx.x); }

// min / max of v of (map, word w), reduced from segment_minmax_kernel's chunks in a fixed order; 0 / 0 without minmax
__device__ __forceinline__ void word_bounds(const WordListParams& P, int map, int w, float& lo, float& hi) {
  lo = 0.f; hi = 0.f;
  if (P.minmax) partial_bounds(P.scratch + 2 * ((long long)map * P.n_words + w) * P.chunks, P.chunks, lo, hi);
}

// The source windows of words [w0, w0 + nw) of `word_maps` (one map's) into `win`, one after the other. Barriers on
// both sides: the previous pass has read `win`, and every thread sees this one.
__device__ __forceinline__ void stage_windows(const WordListParams& P, const Tile& T, const float* word_maps, int w0,
                                              int nw, float* win) {
  __syncthreads();
  for (int i = threadIdx.x; i < nw * T.wn; i += blockDim.x) {
    const int wi = i / T.wn, r = i - wi * T.wn, y = r / T.ww, x = r - y * T.ww;
    win[i] = __ldg(word_maps + ((long long)(w0 + wi) * P.mh + T.wy + y) * P.mw + T.wx + x);
  }
  __syncthreads();
}

// The tile's taps per output row and column, relative to the staged window: filled once per CTA (visible after the
// first stage_windows), read back per pixel by tile_taps
struct TapTables {
  int yi[4][kSegTileH], xi[4][kSegTileW];
  float yw[4][kSegTileH], xw[4][kSegTileW];
};

__device__ __forceinline__ void fill_tap_tables(const WordListParams& P, const Tile& T, TapTables& tt) {
  if (threadIdx.x < T.th) {
    const Taps t = make_taps(T.y0 + threadIdx.x, P.mh, P.oh);
#pragma unroll
    for (int j = 0; j < 4; ++j) { tt.yi[j][threadIdx.x] = t.idx[j] - T.wy; tt.yw[j][threadIdx.x] = t.w[j]; }
  } else if (threadIdx.x >= kSegTileH && threadIdx.x < kSegTileH + T.tw) {
    const int x = threadIdx.x - kSegTileH;
    const Taps t = make_taps(T.x0 + x, P.mw, P.ow);
#pragma unroll
    for (int j = 0; j < 4; ++j) { tt.xi[j][x] = t.idx[j] - T.wx; tt.xw[j][x] = t.w[j]; }
  }
}

__device__ __forceinline__ void tile_taps(const TapTables& tt, int py, int px, Taps& ty, Taps& tx) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    ty.idx[j] = tt.yi[j][py]; ty.w[j] = tt.yw[j][py]; tx.idx[j] = tt.xi[j][px]; tx.w[j] = tt.xw[j][px];
  }
}

// m of word w at tile pixel p < T.th * T.tw: from window wi of the pass, or with words_per_pass 0 (no window fits
// beside the kernel's own shared memory) from word w of `word_maps` (one map's), with the same taps
__device__ __forceinline__ float tile_value(const WordListParams& P, const Tile& T, const TapTables& tt,
                                            const float* win, const float* word_maps, int w, int wi, int p, float lo,
                                            float hi) {
  const int py = p / T.tw;
  Taps ty, tx;
  tile_taps(tt, py, p - py * T.tw, ty, tx);
  float v;
  if (P.words_per_pass > 0) {
    v = bicubic_shared(win + wi * T.wn, T.ww, ty, tx);
  } else {
#pragma unroll
    for (int j = 0; j < 4; ++j) { ty.idx[j] += T.wy; tx.idx[j] += T.wx; }
    v = bicubic_at(word_maps + (long long)w * P.mh * P.mw, P.mw, ty, tx);
  }
  return word_value(P, v, lo, hi);
}

// ---- segmentation: a per-pixel word label -----------------------------------------------------------------------
// labels[p] = 1 + argmax_w m[w][p] (lowest w on ties), or 0 where use_threshold and the max is not > threshold;
// scores[p] = max_w m[w][p], with m[w] taken without threshold. Each pixel keeps the running max / argmax in registers
// while the words are interpolated; its taps are computed per pixel.
struct SegmentParams {
  WordListParams s;
  unsigned char* labels;                // [n_maps][oh][ow]
  float* scores;                        // [n_maps][oh][ow]
};

// grid: (tiles of kSegTileH x kSegTileW output pixels, n_maps); dynamic smem: words_per_pass source windows
__global__ void __launch_bounds__(256) segment_label_kernel(const __grid_constant__ SegmentParams S) {
  const WordListParams& P = S.s;
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
    for (int w = threadIdx.x; w < n_words; w += blockDim.x) {
      float lo, hi;
      partial_bounds(P.scratch + 2 * ((long long)map * n_words + w) * P.chunks, P.chunks, lo, hi);
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
      S.scores[o] = best[k];
      S.labels[o] = (!P.use_threshold || best[k] > P.threshold) ? (unsigned char)(arg[k] + 1) : (unsigned char)0;
    }
  }
}

// ---- word-region overlap: sums of m over binary image regions ---------------------------------------------------
// With R[r] = (regions[r] != 0):
//   intersection[map][r][w] = sum_p R[r](p) m[w](p),   word_area[map][w] = sum_p m[w](p)
// region_tile_kernel reduces every (word, slot) over its tile in a fixed order -- slot 0 is the word's area, slot 1 + r
// its sum inside region r -- into one partial per tile; region_reduce_kernel sums the tiles' partials in a fixed order.
// With a threshold every value is 0 or 1 and every partial an integer below 2^24, so the sums are exact counts.
constexpr int kMaxRegions = DAAM_REGION_MAX_REGIONS;   // 63 + the area slot: 64 slots per word, two groups of 32
constexpr int kRegionSlots = kMaxRegions + 1;

struct RegionParams {
  WordListParams s;
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

// Slot bits of the thread's pixels: bit j of mask[g][k] says tile pixel threadIdx.x + 256 k counts towards slot
// 32 g + j (slot 0: every pixel of the tile, slot 1 + r: the pixels inside region r of `regions` [n_regions][oh][ow]);
// each region byte is read once
__device__ __forceinline__ void region_slot_masks(const unsigned char* regions, int n_regions, int oh, int ow,
                                                  const Tile& T, unsigned (&mask)[2][kSegPix]) {
  const long long n = (long long)oh * ow;
#pragma unroll
  for (int k = 0; k < kSegPix; ++k) {
    const int p = threadIdx.x + 256 * k;
    mask[0][k] = 0u; mask[1][k] = 0u;
    if (p < T.th * T.tw) {
      const int py = p / T.tw;
      const unsigned char* reg = regions + (long long)(T.y0 + py) * ow + T.x0 + p - py * T.tw;
      unsigned m0 = 1u, m1 = 0u;
      for (int r = 0; r < n_regions; ++r) {
        const unsigned bit = __ldg(reg + r * n) != 0 ? 1u : 0u;
        if (r < 31) m0 |= bit << (r + 1); else m1 |= bit << (r - 31);
      }
      mask[0][k] = m0; mask[1][k] = m1;
    }
  }
}

// grid: (tiles of kSegTileH x kSegTileW output pixels, n_maps); dynamic smem: words_per_pass source windows
__global__ void __launch_bounds__(256) region_tile_kernel(const __grid_constant__ RegionParams R) {
  extern __shared__ __align__(16) float win[];
  __shared__ float s_lo[kMaxWords], s_hi[kMaxWords];
  __shared__ float red[2][8][kRegionSlots];          // per-warp sums of a word, double-buffered across words
  __shared__ TapTables taps;
  const WordListParams& P = R.s;
  const int map = blockIdx.y, oh = P.oh, ow = P.ow, n_words = P.n_words;
  const Tile T = block_tile(P);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_slots = R.n_regions + 1;
  for (int w = threadIdx.x; w < n_words; w += blockDim.x) word_bounds(P, map, w, s_lo[w], s_hi[w]);
  fill_tap_tables(P, T, taps);
  unsigned mask[2][kSegPix];
  region_slot_masks(R.regions, R.n_regions, oh, ow, T, mask);
  const float* word_maps = P.word_maps + (long long)map * n_words * P.mh * P.mw;
  float* partials = R.partials + (long long)map * n_words * n_slots * R.tiles + blockIdx.x;
  for (int w0 = 0; w0 < n_words; w0 += P.words_per_pass) {
    const int nw = min(P.words_per_pass, n_words - w0);
    stage_windows(P, T, word_maps, w0, nw, win);
    for (int wi = 0; wi < nw; ++wi) {
      const int w = w0 + wi;
      float v[kSegPix];
#pragma unroll
      for (int k = 0; k < kSegPix; ++k) {
        const int p = threadIdx.x + 256 * k;
        v[k] = 0.f;
        if (p < T.th * T.tw) {
          const int py = p / T.tw;
          Taps ty, tx;
          tile_taps(taps, py, p - py * T.tw, ty, tx);
          v[k] = word_value(P, bicubic_shared(win + wi * T.wn, T.ww, ty, tx), s_lo[w], s_hi[w]);
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

// ---- threshold sweeps of word-region overlap: exact counts at up to 64 thresholds in one pass ----------------------
// With m[w] taken without threshold, R[r] as above and ascending thresholds tau[0 .. T):
//   intersection[map][k][r][w] = #{p : R[r](p) and m[w](p) > tau[k]},   word_area[map][k][w] = #{p : m[w](p) > tau[k]}
// A pixel's bucket b = #{k : m > tau[k]} says it passes exactly thresholds 0 .. b - 1, so one histogram of b per
// (map, word, slot) holds every count: count[k] = sum_{b > k} hist[b]. region_sweep_tile_kernel builds the
// histograms; pixels of bucket 0 pass nothing and are not counted. Per word and pixel row of a warp (the warp's 32
// pixels k), the lanes of one bucket meet in __match_any_sync and their leader adds, per slot present in the warp,
// the popcount of those lanes inside the slot into the CTA's shared histogram of the word. After one barrier per word
// the CTA adds its nonzero bins to the global histograms `counts` (zeroed before the launch) with integer atomics;
// region_sweep_reduce_kernel takes the suffix sums. Every count is an integer, so the bits do not depend on the order
// of the atomics, and below 2^24 pixels every count is exact in fp32.
constexpr int kMaxThresholds = DAAM_REGION_SWEEP_MAX_THRESHOLDS;

struct SweepParams {
  WordListParams s;                     // use_threshold 0; words_per_pass 0: m is read from the word maps
  const unsigned char* regions;         // [n_regions][oh][ow]
  unsigned* counts;                     // [n_maps][n_words][n_regions + 1][T]: bin b - 1 holds bucket b
  int n_regions, n_thresholds;
  float thresholds[kMaxThresholds];     // strictly ascending, finite
};

// The dynamic shared memory region_sweep_tile_kernel keeps before its windows, in floats: two histograms of a word
// (double-buffered across words), T bins per slot
__host__ __device__ __forceinline__ int sweep_smem_floats(int n_regions, int n_thresholds) {
  return 2 * (n_regions + 1) * n_thresholds;
}

// grid: (tiles of kSegTileH x kSegTileW output pixels, n_maps); dynamic smem: sweep_smem_floats, then words_per_pass
// source windows
__global__ void __launch_bounds__(256) region_sweep_tile_kernel(const __grid_constant__ SweepParams S) {
  extern __shared__ __align__(16) float smem[];
  __shared__ float s_lo[kMaxWords], s_hi[kMaxWords];
  __shared__ float s_tau[kMaxThresholds];
  __shared__ unsigned lanes[8][kSegPix][kRegionSlots];   // per warp and pixel row: the lanes inside each slot
  __shared__ TapTables taps;
  const WordListParams& P = S.s;
  const int map = blockIdx.y, mh = P.mh, mw = P.mw, n_words = P.n_words, n_thr = S.n_thresholds;
  const Tile T = block_tile(P);
  const int n_pix = T.th * T.tw;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_slots = S.n_regions + 1, n_bins = n_slots * n_thr;
  unsigned* hist = reinterpret_cast<unsigned*>(smem);                       // [2][n_slots][T]
  float* win = smem + sweep_smem_floats(S.n_regions, n_thr);
  for (int w = threadIdx.x; w < n_words; w += blockDim.x) word_bounds(P, map, w, s_lo[w], s_hi[w]);
  for (int i = threadIdx.x; i < n_thr; i += blockDim.x) s_tau[i] = S.thresholds[i];
  for (int i = threadIdx.x; i < 2 * n_bins; i += blockDim.x) hist[i] = 0u;
  fill_tap_tables(P, T, taps);
  // the tile's slot masks as lane masks, and which slots each pixel row of the warp touches at all
  unsigned present[2][kSegPix];
  {
    unsigned mask[2][kSegPix];
    region_slot_masks(S.regions, S.n_regions, P.oh, P.ow, T, mask);
#pragma unroll
    for (int k = 0; k < kSegPix; ++k) {
#pragma unroll
      for (int g = 0; g < 2; ++g) {
        present[g][k] = __reduce_or_sync(0xffffffffu, mask[g][k]);
        for (int j = 0; j < 32 && 32 * g + j < n_slots; ++j) {
          const unsigned in = __ballot_sync(0xffffffffu, (mask[g][k] >> j) & 1u);
          if (lane == j) lanes[warp][k][32 * g + j] = in;
        }
      }
    }
  }
  __syncthreads();                                     // histograms zeroed, tap tables and lane masks visible
  const float* word_maps = P.word_maps + (long long)map * n_words * mh * mw;
  unsigned* counts = S.counts + (long long)map * n_words * n_bins;
  const bool staged = P.words_per_pass > 0;
  const int per_pass = staged ? P.words_per_pass : n_words;
  for (int w0 = 0; w0 < n_words; w0 += per_pass) {
    const int nw = min(per_pass, n_words - w0);
    if (staged) stage_windows(P, T, word_maps, w0, nw, win);
    for (int wi = 0; wi < nw; ++wi) {
      const int w = w0 + wi;
      unsigned* h = hist + (w & 1) * n_bins;
#pragma unroll
      for (int k = 0; k < kSegPix; ++k) {
        const int p = threadIdx.x + 256 * k;
        int b = 0;
        if (p < n_pix) {
          const float m = tile_value(P, T, taps, win, word_maps, w, wi, p, s_lo[w], s_hi[w]);
          // b = #{k : m > tau[k]}: the passing thresholds are a prefix of the ascending list
#pragma unroll
          for (int step = kMaxThresholds; step > 0; step >>= 1)
            if (b + step <= n_thr && m > s_tau[b + step - 1]) b += step;
        }
        const unsigned counted = __ballot_sync(0xffffffffu, b > 0);
        if (b > 0) {
          const unsigned peers = __match_any_sync(counted, b);
          if (lane == __ffs(peers) - 1) {
            unsigned* bin = h + b - 1;
#pragma unroll
            for (int g = 0; g < 2; ++g) {
              for (unsigned bits = present[g][k]; bits; bits &= bits - 1) {
                const int slot = 32 * g + __ffs(bits) - 1;
                const unsigned c = __popc(peers & lanes[warp][k][slot]);
                if (c) atomicAdd(bin + slot * n_thr, c);
              }
            }
          }
        }
      }
      // one barrier per word: hist[w & 1] is counted into again two words later, after every thread has passed the
      // next barrier, so it is flushed and zeroed by then
      __syncthreads();
      for (int i = threadIdx.x; i < n_bins; i += blockDim.x) {
        const unsigned c = h[i];
        if (c) { atomicAdd(counts + (long long)w * n_bins + i, c); h[i] = 0u; }
      }
    }
  }
}

// grid: ceil(n_out / 256), 256 threads; thread o = (map * n_words + word) * (n_regions + 1) + slot turns its histogram
// into the counts at every threshold (suffix sums, exact integers)
__global__ void __launch_bounds__(256) region_sweep_reduce_kernel(const unsigned* __restrict__ counts, long long n_out,
                                                                  int n_thresholds, int n_words, int n_regions,
                                                                  float* __restrict__ intersection,
                                                                  float* __restrict__ area) {
  const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= n_out) return;
  const int n_slots = n_regions + 1, slot = (int)(o % n_slots);
  const long long mword = o / n_slots, map = mword / n_words, word = mword - map * n_words;
  const unsigned* hist = counts + o * n_thresholds;
  // threshold k of (map, word, slot): area[map][k][word] or intersection[map][k][slot - 1][word]
  const long long stride = slot == 0 ? n_words : (long long)n_regions * n_words;
  float* dst = slot == 0 ? area + map * n_thresholds * n_words + word
                         : intersection + (map * n_thresholds * n_regions + slot - 1) * n_words + word;
  unsigned s = 0;
  for (int k = n_thresholds - 1; k >= 0; --k) {
    s += __ldg(hist + k);
    dst[k * stride] = (float)s;
  }
}

// ---- word-pair overlap: sums of m[a] * m[b] over the image --------------------------------------------------------
//   intersection[map][a][b] = intersection[map][b][a] = sum_p m[a](p) m[b](p),   word_area[map][a] = sum_p m[a](p)
// Slots: the n_words (n_words + 1) / 2 pairs a <= b row by row, then the n_words areas. CTA c of a map reduces tiles
// c, c + ctas, ... (ctas = min(tiles, kPairCtas): the same for every map count, so that a map's sums do not depend on
// the other maps of the call) into one partial per slot, kept in shared memory and owned by one thread (with a threshold) or one
// warp (without); word_pair_reduce_kernel sums the CTAs' partials in a fixed order and writes each pair twice.
//  - with a threshold every m is 0 or 1: each word's tile mask is 32 ballot words, and a pair's count is the popcount
//    of their AND. The counts are integers, so the sums are exact.
//  - without: the m of every word over 256 of the tile's pixels at a time go to shared memory; a warp's lanes take 8
//    of those pixels each per slot, in pixel order, then a butterfly.
constexpr int kPairChunk = 256;                     // pixels per step without a threshold: one per thread
constexpr int kPairMaskStride = 33;                 // a word's 32 ballot words, padded: the words' masks on other banks
constexpr int kPairCtas = DAAM_WORD_OVERLAP_CTAS;   // CTAs per map, at most one per tile

struct PairParams {
  WordListParams s;                     // words_per_pass 0: windows are not staged, m is read from the word maps
  float* partials;                      // [n_maps][slots][ctas]
  int tiles, ctas;                      // tiles of a map; CTAs per map
};

__host__ __device__ __forceinline__ int pair_count(int n_words) { return n_words * (n_words + 1) / 2; }

// pair slot s < pair_count(n_words) -> words a <= b
__host__ __device__ __forceinline__ void pair_words(int s, int n_words, int& a, int& b) {
  a = 0;
  while (s >= n_words - a) { s -= n_words - a; ++a; }
  b = a + s;
}

// the dynamic shared memory word_pair_tile_kernel keeps before its windows, in floats: the pair table (two bytes a
// pair), the slots' partials, and the masks or the values of a chunk
__host__ __device__ __forceinline__ int pair_smem_floats(int n_words, int use_threshold) {
  const int pairs = pair_count(n_words);
  return (pairs + 1) / 2 + pairs + n_words + n_words * (use_threshold ? kPairMaskStride : kPairChunk);
}

// grid: (ctas, n_maps); dynamic smem: pair_smem_floats, then words_per_pass source windows
__global__ void __launch_bounds__(256) word_pair_tile_kernel(const __grid_constant__ PairParams Q) {
  extern __shared__ __align__(16) float smem[];
  __shared__ float s_lo[kMaxWords], s_hi[kMaxWords];
  __shared__ TapTables taps;
  const WordListParams& P = Q.s;
  const int map = blockIdx.y, n_words = P.n_words, mh = P.mh, mw = P.mw;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int pairs = pair_count(n_words), n_slots = pairs + n_words;
  unsigned short* pair_ab = reinterpret_cast<unsigned short*>(smem);          // a << 8 | b
  float* acc = smem + (pairs + 1) / 2;                                        // [n_slots]
  unsigned* counts = reinterpret_cast<unsigned*>(acc);                        // acc, with a threshold
  unsigned* masks = reinterpret_cast<unsigned*>(acc + n_slots);               // [n_words][kPairMaskStride]
  float* vals = acc + n_slots;                                                // [n_words][kPairChunk]
  float* win = smem + pair_smem_floats(n_words, P.use_threshold);
  for (int w = threadIdx.x; w < n_words; w += blockDim.x) word_bounds(P, map, w, s_lo[w], s_hi[w]);
  for (int s = threadIdx.x; s < pairs; s += blockDim.x) {
    int a, b;
    pair_words(s, n_words, a, b);
    pair_ab[s] = (unsigned short)(a << 8 | b);
  }
  for (int s = threadIdx.x; s < n_slots; s += blockDim.x) acc[s] = 0.f;     // also counts = 0
  const float* word_maps = P.word_maps + (long long)map * n_words * mh * mw;
  const bool staged = P.words_per_pass > 0;
  const int per_pass = staged ? P.words_per_pass : n_words;
  for (int tile = blockIdx.x; tile < Q.tiles; tile += Q.ctas) {
    const Tile T = tile_at(P, tile);
    const int n_pix = T.th * T.tw;
    __syncthreads();                                   // the previous tile has read the tap tables and buffers
    fill_tap_tables(P, T, taps);
    if (!staged) __syncthreads();                      // (stage_windows' barriers publish them otherwise)
    if (P.use_threshold) {
      for (int w0 = 0; w0 < n_words; w0 += per_pass) {
        const int nw = min(per_pass, n_words - w0);
        if (staged) stage_windows(P, T, word_maps, w0, nw, win);
        for (int wi = 0; wi < nw; ++wi) {
          const int w = w0 + wi;
#pragma unroll
          for (int k = 0; k < kSegPix; ++k) {
            const int p = threadIdx.x + 256 * k;
            const bool in = p < n_pix && tile_value(P, T, taps, win, word_maps, w, wi, p, s_lo[w], s_hi[w]) != 0.f;
            const unsigned bits = __ballot_sync(0xffffffffu, in);
            if (lane == 0) masks[w * kPairMaskStride + 8 * k + warp] = bits;
          }
        }
      }
      __syncthreads();
      for (int s = threadIdx.x; s < n_slots; s += blockDim.x) {
        unsigned c = 0;
        if (s < pairs) {
          const unsigned* ma = masks + (pair_ab[s] >> 8) * kPairMaskStride;
          const unsigned* mb = masks + (pair_ab[s] & 255) * kPairMaskStride;
#pragma unroll 8
          for (int j = 0; j < 32; ++j) c += __popc(ma[j] & mb[j]);
        } else {
          const unsigned* ma = masks + (s - pairs) * kPairMaskStride;
#pragma unroll 8
          for (int j = 0; j < 32; ++j) c += __popc(ma[j]);
        }
        counts[s] += c;
      }
    } else {
      const bool restage = staged && per_pass < n_words;   // one pass: the windows stay for every chunk
      for (int c0 = 0; c0 < n_pix; c0 += kPairChunk) {
        const int p = c0 + threadIdx.x;
        for (int w0 = 0; w0 < n_words; w0 += per_pass) {
          const int nw = min(per_pass, n_words - w0);
          if (staged && (c0 == 0 || restage)) stage_windows(P, T, word_maps, w0, nw, win);
          for (int wi = 0; wi < nw; ++wi) {
            const int w = w0 + wi;
            vals[w * kPairChunk + threadIdx.x] =
                p < n_pix ? tile_value(P, T, taps, win, word_maps, w, wi, p, s_lo[w], s_hi[w]) : 0.f;
          }
        }
        __syncthreads();
        for (int s = warp; s < n_slots; s += 8) {
          float x = 0.f;
          if (s < pairs) {
            const float* va = vals + (pair_ab[s] >> 8) * kPairChunk + lane;
            const float* vb = vals + (pair_ab[s] & 255) * kPairChunk + lane;
#pragma unroll
            for (int i = 0; i < kPairChunk / 32; ++i) x = fmaf(va[32 * i], vb[32 * i], x);
          } else {
            const float* va = vals + (s - pairs) * kPairChunk + lane;
#pragma unroll
            for (int i = 0; i < kPairChunk / 32; ++i) x += va[32 * i];
          }
#pragma unroll
          for (int h = 16; h > 0; h >>= 1) x += __shfl_xor_sync(0xffffffffu, x, h);
          if (lane == 0) acc[s] += x;
        }
        __syncthreads();                                 // the next chunk rewrites vals
      }
    }
  }
  __syncthreads();
  float* partials = Q.partials + (long long)map * n_slots * Q.ctas + blockIdx.x;
  for (int s = threadIdx.x; s < n_slots; s += blockDim.x)
    partials[(long long)s * Q.ctas] = P.use_threshold ? (float)counts[s] : acc[s];
}

// grid: ceil(n_out / 8), 256 threads; one warp per output o = map * slots + slot sums the CTAs' partials (lane-strided,
// then a butterfly) in a fixed order; a pair's sum goes to both of its intersection elements
__global__ void __launch_bounds__(256) word_pair_reduce_kernel(const float* __restrict__ partials, long long n_out,
                                                               int ctas, int n_words, float* __restrict__ intersection,
                                                               float* __restrict__ area) {
  const long long o = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (o >= n_out) return;                              // whole warps
  const int lane = threadIdx.x & 31;
  const float* src = partials + o * ctas;
  float s = 0.f;
  for (int c = lane; c < ctas; c += 32) s += __ldg(src + c);
#pragma unroll
  for (int h = 16; h > 0; h >>= 1) s += __shfl_xor_sync(0xffffffffu, s, h);
  if (lane == 0) {
    const int pairs = pair_count(n_words), n_slots = pairs + n_words;
    const long long map = o / n_slots;
    const int slot = (int)(o - map * n_slots);
    if (slot < pairs) {
      int a, b;
      pair_words(slot, n_words, a, b);
      float* out = intersection + map * n_words * n_words;
      out[a * n_words + b] = s;
      out[b * n_words + a] = s;
    } else {
      area[map * n_words + slot - pairs] = s;
    }
  }
}

// ---- heat-map overlays: the jet-coloured m blended onto the image -----------------------------------------------
// The reference's plot_overlay (heatmap.py:20-53, 66-75) as pixels: for every byte of frames [n_maps][n_words][oh][ow][3]:
//   c = color_normalize ? (hi == lo ? 0 : (m - lo) / (hi - lo)) : clamp(m, 0, 1)   (lo / hi: min / max of m[w])
//   k = min(int(c * 256), 255)                                                      (matplotlib's Colormap, N = 256)
//   a = clamp(m, 0, 1)                                                              (the image drawn with alpha 1 - a)
//   out = uint8(clamp(rne((1 - a) * image + a * jet[k]), 0, 255))                   (every operation rounded in fp32)
// v -> m is monotone non-decreasing in fp32 (subtract, divide by a positive constant, `>` threshold), so lo / hi of m
// are m at the min / max of v: no pass over m. Every word's RGB bytes go through shared memory to aligned 4- and
// 16-byte stores. A 4-byte word of frames belongs to the CTA that owns its first byte; when it reaches past the tile
// row, that CTA computes the one next pixel in memory order (the next tile, row, word or map) from the global word
// maps, with the same arithmetic.

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
  WordListParams s;                     // minmax also when only color_normalize needs it
  const unsigned char* image;           // [oh][ow][3], map i at image + i * image_map_stride
  long long image_map_stride;           // bytes; 0: one image for every map
  unsigned char* frames;                // [n_maps][n_words][oh][ow][3], 4-byte aligned, padded to a 4-byte multiple
  int color_normalize, n_maps;
};

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
  const WordListParams& P = O.s;
  if (map >= O.n_maps) { out[0] = out[1] = out[2] = 0; return; }
  float vlo, vhi;
  word_bounds(P, map, w, vlo, vhi);
  const float lo = word_value(P, vlo, vlo, vhi), hi = word_value(P, vhi, vlo, vhi);
  const float v = word_map_at(P, P.word_maps + ((long long)map * P.n_words + w) * P.mh * P.mw, oy, ox);
  const unsigned char* im = O.image + map * O.image_map_stride + ((long long)oy * P.ow + ox) * 3;
  const unsigned char px[3] = {__ldg(im), __ldg(im + 1), __ldg(im + 2)};
  overlay_rgb(word_value(P, v, vlo, vhi), lo, hi, O.color_normalize, px, lut, out);
}

// grid: (tiles of kSegTileH x kSegTileW output pixels, n_maps); dynamic smem: words_per_pass source windows
__global__ void __launch_bounds__(256) overlay_kernel(const __grid_constant__ OverlayParams O) {
  extern __shared__ __align__(16) float win[];
  __shared__ float s_vlo[kMaxWords], s_vhi[kMaxWords], s_lo[kMaxWords], s_hi[kMaxWords];
  __shared__ TapTables taps;
  __shared__ float lut[256 * 3];
  __shared__ unsigned char img[kSegTileH * kSegTileW * 3];
  __shared__ __align__(16) unsigned char rows[2][kSegTileH][kOverlayRowBytes];   // double-buffered across words
  const WordListParams& P = O.s;
  const int map = blockIdx.y, oh = P.oh, ow = P.ow, n_words = P.n_words;
  const Tile T = block_tile(P);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int w = threadIdx.x; w < n_words; w += blockDim.x) {
    float vlo, vhi;
    word_bounds(P, map, w, vlo, vhi);
    s_vlo[w] = vlo; s_vhi[w] = vhi;
    s_lo[w] = word_value(P, vlo, vlo, vhi); s_hi[w] = word_value(P, vhi, vlo, vhi);
  }
  for (int i = threadIdx.x; i < 256 * 3; i += blockDim.x) lut[i] = c_jet.v[i];
  fill_tap_tables(P, T, taps);
  // the tile's image bytes, read once for every word
  const unsigned char* image = O.image + map * O.image_map_stride;
  for (int i = threadIdx.x; i < T.th * T.tw * 3; i += blockDim.x) {
    const int r = i / (T.tw * 3), b = i - r * T.tw * 3;
    img[i] = __ldg(image + ((long long)(T.y0 + r) * ow + T.x0) * 3 + b);
  }
  const float* word_maps = P.word_maps + (long long)map * n_words * P.mh * P.mw;
  const unsigned long long frames = (unsigned long long)O.frames;   // byte addresses: the alignment of the stores
  for (int w0 = 0; w0 < n_words; w0 += P.words_per_pass) {
    const int nw = min(P.words_per_pass, n_words - w0);
    stage_windows(P, T, word_maps, w0, nw, win);
    for (int wi = 0; wi < nw; ++wi) {
      const int w = w0 + wi;
      const float vlo = s_vlo[w], vhi = s_vhi[w], lo = s_lo[w], hi = s_hi[w];
      // row py of the tile starts at byte g0(py) of frames; rows[w & 1][py][g0 & 15] holds that byte
      const long long row0 = (((long long)map * n_words + w) * oh + T.y0) * ow + T.x0;
#pragma unroll
      for (int k = 0; k < kSegPix; ++k) {
        const int p = threadIdx.x + 256 * k;
        if (p < T.th * T.tw) {
          const int py = p / T.tw, px = p - py * T.tw;
          Taps ty, tx;
          tile_taps(taps, py, px, ty, tx);
          const float m = word_value(P, bicubic_shared(win + wi * T.wn, T.ww, ty, tx), vlo, vhi);
          const unsigned shift = (unsigned)((frames + 3 * (row0 + (long long)py * ow)) & 15);
          overlay_rgb(m, lo, hi, O.color_normalize, img + 3 * p, lut, &rows[w & 1][py][shift + 3 * px]);
        }
      }
      // a row whose last 4-byte word reaches past it: the next pixel in memory order
      if (threadIdx.x < T.th) {
        const int py = threadIdx.x;
        const unsigned long long g1 = frames + 3 * (row0 + (long long)py * ow + T.tw);
        if (g1 & 3) {
          int nm = map, nwd = w, ny = T.y0 + py, nx = T.x0 + T.tw;
          if (nx == ow) { nx = 0; ++ny; }
          if (ny == oh) { ny = 0; ++nwd; }
          if (nwd == n_words) { nwd = 0; ++nm; }
          const unsigned shift = (unsigned)((g1 - 3 * T.tw) & 15);
          overlay_pixel_global(O, lut, nm, nwd, ny, nx, &rows[w & 1][py][shift + 3 * T.tw]);
        }
      }
      // one barrier per word: rows[w & 1] is rewritten two words later, after every warp has passed the next barrier
      __syncthreads();
      for (int py = warp; py < T.th; py += 8) {
        const unsigned long long g0 = frames + 3 * (row0 + (long long)py * ow), g1 = g0 + 3 * T.tw;
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

// ---- word instances: m without threshold, for the connected components of m > threshold ---------------------------
// Writes every pixel's m (use_threshold 0: what daam_expand_words writes without threshold) to a plane per (map, word);
// components.cu labels the plane's mask m > threshold and reduces its components.
struct InstanceMaskParams {
  WordListParams s;
  float* pre;                           // [n_maps][n_words][oh][ow]
};

// grid: (tiles of kSegTileH x kSegTileW output pixels, n_maps); dynamic smem: words_per_pass source windows
__global__ void __launch_bounds__(256) instance_mask_kernel(const __grid_constant__ InstanceMaskParams I) {
  extern __shared__ __align__(16) float win[];
  __shared__ float s_lo[kMaxWords], s_hi[kMaxWords];
  __shared__ TapTables taps;
  const WordListParams& P = I.s;
  const int map = blockIdx.y, ow = P.ow, n_words = P.n_words;
  const Tile T = block_tile(P);
  for (int w = threadIdx.x; w < n_words; w += blockDim.x) word_bounds(P, map, w, s_lo[w], s_hi[w]);
  fill_tap_tables(P, T, taps);
  const float* word_maps = P.word_maps + (long long)map * n_words * P.mh * P.mw;
  const long long n = (long long)P.oh * ow;
  for (int w0 = 0; w0 < n_words; w0 += P.words_per_pass) {
    const int nw = min(P.words_per_pass, n_words - w0);
    stage_windows(P, T, word_maps, w0, nw, win);
    for (int wi = 0; wi < nw; ++wi) {
      const int w = w0 + wi;
      float* dst = I.pre + ((long long)map * n_words + w) * n + (long long)T.y0 * ow + T.x0;
#pragma unroll
      for (int k = 0; k < kSegPix; ++k) {
        const int p = threadIdx.x + 256 * k;
        if (p < T.th * T.tw) {
          const int py = p / T.tw, px = p - py * T.tw;
          Taps ty, tx;
          tile_taps(taps, py, px, ty, tx);
          dst[(long long)py * ow + px] = word_value(P, bicubic_shared(win + wi * T.wn, T.ww, ty, tx), s_lo[w], s_hi[w]);
        }
      }
    }
  }
}

}  // namespace
}  // namespace daam

using namespace daam;

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

// The word-list checks every word-list entry point makes once its own pointers and sizes are checked, in the order
// they are reported, then `p` from the arguments (one chunk). `tiled`: the tile entry points' limits of 65535 maps
// and 2^30 output pixels, checked before the device is queried.
static int word_list_prepare(const char* name, const float* global_maps, int32_t n_maps, int32_t n_rows, int32_t mh,
                             int32_t mw, const int32_t* rows, const int32_t* row_begin, int32_t n_words, int32_t out_h,
                             int32_t out_w, int32_t absolute, bool minmax, int32_t use_threshold, float threshold,
                             float* word_maps, float* scratch, bool tiled, WordListParams& p, DeviceInfo* dev) {
  if (n_words <= 0) { set_error("%s: empty word list", name); return DAAM_E_INVALID; }
  if (n_words > kMaxWords) { set_error("%s: %d words > %d", name, n_words, kMaxWords); return DAAM_E_UNSUPPORTED; }
  if (row_begin[0] != 0 || row_begin[n_words] > kMaxWordRows) { set_error("%s: row_begin must start at 0 and select at most %d rows", name, kMaxWordRows); return DAAM_E_UNSUPPORTED; }
  if ((size_t)mh * mw * sizeof(float) > kMaxSmem) { set_error("%s: a %d x %d map does not fit shared memory", name, mh, mw); return DAAM_E_UNSUPPORTED; }
  if (tiled && n_maps > 65535) { set_error("%s: %d maps > 65535", name, n_maps); return DAAM_E_UNSUPPORTED; }
  if (tiled && (long long)out_h * out_w > (1LL << 30)) { set_error("%s: a %d x %d output is more than 2^30 pixels", name, out_h, out_w); return DAAM_E_UNSUPPORTED; }
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
  p.maps = global_maps; p.word_maps = word_maps; p.scratch = scratch;
  p.map_stride = (long long)n_rows * mh * mw;
  p.mh = mh; p.mw = mw; p.oh = out_h; p.ow = out_w; p.n_words = n_words; p.chunks = 1; p.words_per_pass = 1;
  p.absolute = absolute ? 1 : 0; p.use_threshold = use_threshold ? 1 : 0; p.threshold = threshold;
  p.minmax = minmax ? 1 : 0;
  return DAAM_OK;
}

static int launch_expand_words(ExpandParams& p, const DeviceInfo& dev, cudaStream_t stream) {
  const size_t smem = (size_t)p.s.mh * p.s.mw * sizeof(float);
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
  const int n = p.s.oh * p.s.ow;
  int done = 0;
  const int total = p.s.n_words;
  ExpandParams q = p;
  while (done < total) {                                // more words than the device holds at once: several launches
    const int batch = total - done < capacity ? total - done : capacity;
    int chunks = capacity / batch;
    if (chunks > kWordChunks) chunks = kWordChunks;
    if (chunks > (n + 255) / 256) chunks = (n + 255) / 256;
    if (chunks < 1) chunks = 1;
    q.s.n_words = batch;
    q.s.chunks = chunks;
    q.out = p.out + (long long)done * n;
    q.s.word_maps = p.s.word_maps ? p.s.word_maps + (long long)done * p.s.mh * p.s.mw : nullptr;
    q.s.scratch = p.s.scratch + (long long)kWordPartialFloats * done;
    for (int i = 0; i <= batch; ++i) q.s.row_begin[i] = p.s.row_begin[done + i];
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
  static thread_local ExpandParams p;
  DeviceInfo dev;
  if (int rc = word_list_prepare(name, global_maps, 1, n_rows, mh, mw, rows, row_begin, n_words, out_h, out_w, absolute,
                                 !absolute, use_threshold, threshold, word_maps, scratch, false, p.s, &dev)) return rc;
  p.out = out;
  return launch_expand_words(p, dev, static_cast<cudaStream_t>(stream));
}

extern "C" int daam_expand_words(const float* global_maps, int32_t n_rows, int32_t mh, int32_t mw, const int32_t* rows,
                                 const int32_t* row_begin, int32_t n_words, int32_t out_h, int32_t out_w,
                                 int32_t absolute, int32_t use_threshold, float threshold, float* word_maps, float* out,
                                 float* scratch, void* stream) {
  return expand_words_impl("daam_expand_words", global_maps, n_rows, mh, mw, rows, row_begin, n_words, out_h, out_w,
                           absolute, use_threshold, threshold, word_maps, out, scratch, stream);
}

// one word whose "rows" are the word map itself
extern "C" int daam_expand_as(const float* word_map, int32_t mh, int32_t mw, int32_t out_h, int32_t out_w,
                              int32_t absolute, int32_t use_threshold, float threshold, float* out, float* scratch,
                              void* stream) {
  const int32_t rows[1] = {0}, row_begin[2] = {0, 1};
  return expand_words_impl("daam_expand_as", word_map, 1, mh, mw, rows, row_begin, 1, out_h, out_w, absolute,
                           use_threshold, threshold, nullptr, out, scratch, stream);
}

static int tile_count(const WordListParams& p) {
  return ((p.oh + kSegTileH - 1) / kSegTileH) * ((p.ow + kSegTileW - 1) / kSegTileW);
}

// Launch 1 of the tile entry points, and all of it for daam_refine_words, daam_segment_crf and daam_segment_superpixels:
// segment_minmax_kernel over (map, word, chunk)
// with enough CTAs for a few waves, at most kWordChunks per word and one per 256 pixels. Sets p.chunks.
static int launch_word_maps(WordListParams& p, int n_maps, const DeviceInfo& dev, cudaStream_t stream) {
  const long long n = (long long)p.oh * p.ow, mwords = (long long)n_maps * p.n_words;
  long long chunks = (4LL * dev.sm_count + mwords - 1) / mwords;
  if (chunks > kWordChunks) chunks = kWordChunks;
  if (chunks > (n + 255) / 256) chunks = (n + 255) / 256;
  if (chunks < 1 || !p.minmax) chunks = 1;
  p.chunks = (int)chunks;
  static std::once_flag attr_once[64];
  cudaError_t attr_err = cudaSuccess;
  std::call_once(attr_once[dev.device & 63], [&] {
    const void* kernels[] = {(const void*)segment_minmax_kernel, (const void*)segment_label_kernel,
                             (const void*)region_tile_kernel, (const void*)overlay_kernel,
                             (const void*)word_pair_tile_kernel, (const void*)instance_mask_kernel,
                             (const void*)region_sweep_tile_kernel};
    for (const void* f : kernels)
      if (attr_err == cudaSuccess) attr_err = cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem);
  });
  DAAM_CUDA_TRY(attr_err);
  segment_minmax_kernel<<<(unsigned)(mwords * p.chunks), 256, (size_t)p.mh * p.mw * sizeof(float), stream>>>(p);
  DAAM_CUDA_TRY(cudaGetLastError());
  count_launch();
  return DAAM_OK;
}

// The tile entry points' launches after word_list_prepare: launch_word_maps, then `kernel` over (tile, map), or over
// (CTA, map) with `ctas` CTAs per map. `smem_before`: the bytes of dynamic shared memory the kernel keeps before its
// windows; such a kernel stages as many words' windows as fit beside them (it stages them again per pixel chunk when
// they take several passes). Sets k.s.chunks and k.s.words_per_pass; words_per_pass 0 (only with smem_before): not
// one window fits, and the kernel reads the word maps instead.
template <class Params>
static int launch_tiles(void (*kernel)(Params), Params& k, int n_maps, const DeviceInfo& dev, cudaStream_t stream,
                        int ctas = 0, size_t smem_before = 0) {
  WordListParams& p = k.s;
  if (int rc = launch_word_maps(p, n_maps, dev, stream)) return rc;
  // launch 2: a tile's source window is at most ceil(tile * map / out) + 4 rows (columns), and no more than the map
  const int win_h = std::min<int>(p.mh, (int)ceil((double)kSegTileH * p.mh / p.oh) + 5);
  const int win_w = std::min<int>(p.mw, (int)ceil((double)kSegTileW * p.mw / p.ow) + 5);
  const int win = win_h * win_w;
  if (smem_before)
    p.words_per_pass = (int)std::min<size_t>(p.n_words, (kMaxSmem - smem_before) / (win * sizeof(float)));
  else
    p.words_per_pass = std::max(1, std::min(p.n_words, kSegStageFloats / win));
  const size_t smem = smem_before + (size_t)p.words_per_pass * win * sizeof(float);
  kernel<<<dim3(ctas ? ctas : tile_count(p), n_maps), 256, smem, stream>>>(k);
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
  if (int rc = word_list_prepare(name, global_maps, n_maps, n_rows, mh, mw, rows, row_begin, n_words, out_h, out_w,
                                 absolute, !absolute, use_threshold, threshold, word_maps, scratch, true, p.s, &dev)) return rc;
  p.labels = labels; p.scores = scores;
  return launch_tiles(segment_label_kernel, p, n_maps, dev, static_cast<cudaStream_t>(stream_));
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
  if (int rc = word_list_prepare(name, global_maps, n_maps, n_rows, mh, mw, rows, row_begin, n_words, out_h, out_w,
                                 absolute, !absolute, use_threshold, threshold, word_maps, scratch, true, p.s, &dev)) return rc;
  p.regions = regions; p.n_regions = n_regions; p.tiles = tile_count(p.s);
  p.partials = scratch + (long long)kWordPartialFloats * n_maps * n_words;   // after the min / max partials
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (int rc = launch_tiles(region_tile_kernel, p, n_maps, dev, stream)) return rc;
  const long long n_out = (long long)n_maps * n_words * (n_regions + 1);
  region_reduce_kernel<<<(unsigned)((n_out + 7) / 8), 256, 0, stream>>>(p.partials, n_out, p.tiles, n_words, n_regions,
                                                                        intersection, word_area);
  DAAM_CUDA_TRY(cudaGetLastError());
  count_launch();
  return DAAM_OK;
}

extern "C" int daam_region_sweep(const float* global_maps, int32_t n_maps, int32_t n_rows, int32_t mh, int32_t mw,
                                 const int32_t* rows, const int32_t* row_begin, int32_t n_words, int32_t out_h,
                                 int32_t out_w, int32_t absolute, const float* thresholds, int32_t n_thresholds,
                                 float* word_maps, const uint8_t* regions, int32_t n_regions, float* intersection,
                                 float* word_area, float* scratch, void* stream_) {
  const char* name = "daam_region_sweep";
  if (!global_maps || !rows || !row_begin || !thresholds || !word_maps || !regions || !intersection || !word_area ||
      !scratch || n_maps <= 0 || mh <= 0 || mw <= 0 || out_h <= 0 || out_w <= 0 || n_rows <= 0 || n_regions <= 0 ||
      n_thresholds <= 0) { set_error("%s: null pointer or non-positive size", name); return DAAM_E_INVALID; }
  if (n_thresholds > kMaxThresholds) { set_error("%s: %d thresholds > %d", name, n_thresholds, kMaxThresholds); return DAAM_E_UNSUPPORTED; }
  if (n_regions > kMaxRegions) { set_error("%s: %d regions > %d", name, n_regions, kMaxRegions); return DAAM_E_UNSUPPORTED; }
  // the counts are exact in fp32 up to 2^24
  if ((long long)out_h * out_w > (1LL << 24)) { set_error("%s: a %d x %d output is more than 2^24 pixels", name, out_h, out_w); return DAAM_E_UNSUPPORTED; }
  for (int k = 0; k < n_thresholds; ++k) {
    if (!isfinite(thresholds[k])) { set_error("%s: threshold %d is not finite", name, k); return DAAM_E_INVALID; }
    if (k > 0 && !(thresholds[k] > thresholds[k - 1])) { set_error("%s: thresholds %d and %d are not strictly ascending", name, k - 1, k); return DAAM_E_INVALID; }
  }
  static thread_local SweepParams p;
  DeviceInfo dev;
  if (int rc = word_list_prepare(name, global_maps, n_maps, n_rows, mh, mw, rows, row_begin, n_words, out_h, out_w,
                                 absolute, !absolute, 0, 0.f, word_maps, scratch, true, p.s, &dev)) return rc;
  p.regions = regions; p.n_regions = n_regions; p.n_thresholds = n_thresholds;
  for (int k = 0; k < n_thresholds; ++k) p.thresholds[k] = thresholds[k];
  // after the min / max partials
  p.counts = reinterpret_cast<unsigned*>(scratch + (long long)kWordPartialFloats * n_maps * n_words);
  const long long n_out = (long long)n_maps * n_words * (n_regions + 1);
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DAAM_CUDA_TRY(cudaMemsetAsync(p.counts, 0, (size_t)n_out * n_thresholds * sizeof(unsigned), stream));
  if (int rc = launch_tiles(region_sweep_tile_kernel, p, n_maps, dev, stream, 0,
                            (size_t)sweep_smem_floats(n_regions, n_thresholds) * sizeof(float))) return rc;
  region_sweep_reduce_kernel<<<(unsigned)((n_out + 255) / 256), 256, 0, stream>>>(p.counts, n_out, n_thresholds,
                                                                                  n_words, n_regions, intersection,
                                                                                  word_area);
  DAAM_CUDA_TRY(cudaGetLastError());
  count_launch();
  return DAAM_OK;
}

extern "C" int daam_word_overlap(const float* global_maps, int32_t n_maps, int32_t n_rows, int32_t mh, int32_t mw,
                                 const int32_t* rows, const int32_t* row_begin, int32_t n_words, int32_t out_h,
                                 int32_t out_w, int32_t absolute, int32_t use_threshold, float threshold,
                                 float* word_maps, float* intersection, float* word_area, float* scratch,
                                 void* stream_) {
  const char* name = "daam_word_overlap";
  if (!global_maps || !rows || !row_begin || !word_maps || !intersection || !word_area || !scratch || n_maps <= 0 ||
      mh <= 0 || mw <= 0 || out_h <= 0 || out_w <= 0 || n_rows <= 0) { set_error("%s: null pointer or non-positive size", name); return DAAM_E_INVALID; }
  // fp32 partial sums of 0/1 values stay exact integers up to 2^24
  if ((long long)out_h * out_w > (1LL << 24)) { set_error("%s: a %d x %d output is more than 2^24 pixels", name, out_h, out_w); return DAAM_E_UNSUPPORTED; }
  static thread_local PairParams p;
  DeviceInfo dev;
  if (int rc = word_list_prepare(name, global_maps, n_maps, n_rows, mh, mw, rows, row_begin, n_words, out_h, out_w,
                                 absolute, !absolute, use_threshold, threshold, word_maps, scratch, true, p.s, &dev)) return rc;
  p.tiles = tile_count(p.s);
  p.ctas = std::min(p.tiles, kPairCtas);
  p.partials = scratch + (long long)kWordPartialFloats * n_maps * n_words;   // after the min / max partials
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (int rc = launch_tiles(word_pair_tile_kernel, p, n_maps, dev, stream, p.ctas,
                            (size_t)pair_smem_floats(n_words, p.s.use_threshold) * sizeof(float))) return rc;
  const long long n_out = (long long)n_maps * (pair_count(n_words) + n_words);
  word_pair_reduce_kernel<<<(unsigned)((n_out + 7) / 8), 256, 0, stream>>>(p.partials, n_out, p.ctas, n_words,
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
  // the min / max of v is computed when the normalisation or the colour scale needs it
  if (int rc = word_list_prepare(name, global_maps, n_maps, n_rows, mh, mw, rows, row_begin, n_words, out_h, out_w,
                                 absolute, !absolute || color_normalize, use_threshold, threshold, word_maps, scratch,
                                 true, p.s, &dev)) return rc;
  p.image = image; p.image_map_stride = image_map_stride; p.frames = frames;
  p.color_normalize = color_normalize ? 1 : 0; p.n_maps = n_maps;
  return launch_tiles(overlay_kernel, p, n_maps, dev, static_cast<cudaStream_t>(stream_));
}

extern "C" int daam_jet_colormap(float* out) {
  if (!out) { set_error("daam_jet_colormap: null pointer"); return DAAM_E_INVALID; }
  DAAM_CUDA_TRY(cudaMemcpyFromSymbol(out, c_jet, sizeof(JetTable)));
  return DAAM_OK;
}

extern "C" int daam_word_instances(const float* global_maps, int32_t n_maps, int32_t n_rows, int32_t mh, int32_t mw,
                                   const int32_t* rows, const int32_t* row_begin, int32_t n_words, int32_t out_h,
                                   int32_t out_w, int32_t absolute, float threshold, int32_t max_instances,
                                   float* word_maps, int32_t* count, int32_t* area, int32_t* box, int64_t* sum_yx,
                                   float* peak, int32_t* peak_yx, void* scratch, int64_t scratch_bytes, void* stream_) {
  const char* name = "daam_word_instances";
  if (!global_maps || !rows || !row_begin || !word_maps || !count || !area || !box || !sum_yx || !peak || !peak_yx ||
      !scratch || n_maps <= 0 || mh <= 0 || mw <= 0 || out_h <= 0 || out_w <= 0 || n_rows <= 0 || max_instances <= 0) { set_error("%s: null pointer or non-positive size", name); return DAAM_E_INVALID; }
  if (max_instances > kMaxInstances) { set_error("%s: max_instances %d > %d", name, max_instances, kMaxInstances); return DAAM_E_UNSUPPORTED; }
  if ((long long)out_h * out_w > (1LL << 24)) { set_error("%s: a %d x %d output is more than 2^24 pixels", name, out_h, out_w); return DAAM_E_UNSUPPORTED; }
  const long long plane_bytes = instance_plane_bytes(out_h, out_w);
  if (scratch_bytes < plane_bytes) { set_error("%s: %lld scratch bytes < %lld, one %d x %d plane", name, (long long)scratch_bytes, plane_bytes, out_h, out_w); return DAAM_E_INVALID; }
  static thread_local InstanceMaskParams p, q;
  DeviceInfo dev;
  if (int rc = word_list_prepare(name, global_maps, n_maps, n_rows, mh, mw, rows, row_begin, n_words, out_h, out_w,
                                 absolute, !absolute, 0, 0.f, word_maps, nullptr, true, p.s, &dev)) return rc;
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  // a round: whole maps while a map's planes fit the scratch, else the words of one map in groups
  const int cap = (int)std::min<long long>(scratch_bytes / plane_bytes, 65535);
  const int maps_per_round = std::max(1, cap / n_words), words_per_round = std::min(cap, (int)n_words);
  for (int map0 = 0; map0 < n_maps; map0 += maps_per_round) {
    const int nm = std::min(maps_per_round, n_maps - map0);
    for (int w0 = 0; w0 < n_words; w0 += words_per_round) {
      const int nw = std::min(words_per_round, n_words - w0);
      q = p;
      q.s.maps = global_maps + map0 * p.s.map_stride;
      q.s.n_words = nw;
      for (int i = 0; i <= nw; ++i) q.s.row_begin[i] = p.s.row_begin[w0 + i];
      const long long plane0 = (long long)map0 * n_words + w0;
      q.s.word_maps = word_maps + plane0 * mh * mw;
      InstancePlanes c;
      instance_planes_in(scratch, nm * nw, out_h, out_w, c);
      q.s.scratch = c.minmax;
      q.pre = c.pre;
      if (int rc = launch_tiles(instance_mask_kernel, q, nm, dev, stream)) return rc;
      c.k = max_instances; c.threshold = threshold;
      c.count = count + plane0;
      c.out_area = area + plane0 * max_instances;
      c.out_box = box + plane0 * max_instances * 4;
      c.out_sum = reinterpret_cast<long long*>(sum_yx) + plane0 * max_instances * 2;
      c.out_peak = peak + plane0 * max_instances;
      c.out_peak_yx = peak_yx + plane0 * max_instances * 2;
      if (int rc = launch_components(c, stream)) return rc;
    }
  }
  return DAAM_OK;
}

extern "C" int daam_region_ranking(const float* global_maps, int32_t n_maps, int32_t n_rows, int32_t mh, int32_t mw,
                                   const int32_t* rows, const int32_t* row_begin, int32_t n_words, int32_t out_h,
                                   int32_t out_w, int32_t absolute, float* word_maps, const uint8_t* regions,
                                   int32_t n_regions, int64_t* u2, double* ap, void* scratch, int64_t scratch_bytes,
                                   void* stream_) {
  const char* name = "daam_region_ranking";
  if (!global_maps || !rows || !row_begin || !word_maps || !regions || !u2 || !ap || !scratch || n_maps <= 0 ||
      mh <= 0 || mw <= 0 || out_h <= 0 || out_w <= 0 || n_rows <= 0 || n_regions <= 0) { set_error("%s: null pointer or non-positive size", name); return DAAM_E_INVALID; }
  if (n_regions > kMaxRegions) { set_error("%s: %d regions > %d", name, n_regions, kMaxRegions); return DAAM_E_UNSUPPORTED; }
  if ((long long)out_h * out_w > (1LL << 24)) { set_error("%s: a %d x %d output is more than 2^24 pixels", name, out_h, out_w); return DAAM_E_UNSUPPORTED; }
  // the region masks once per call, then the planes of each round
  const long long mask_bytes = 8LL * out_h * out_w, plane_bytes = ranking_plane_bytes(out_h, out_w);
  if (scratch_bytes < mask_bytes + plane_bytes) { set_error("%s: %lld scratch bytes < %lld, the masks and one %d x %d plane", name, (long long)scratch_bytes, mask_bytes + plane_bytes, out_h, out_w); return DAAM_E_INVALID; }
  static thread_local InstanceMaskParams p, q;
  DeviceInfo dev;
  if (int rc = word_list_prepare(name, global_maps, n_maps, n_rows, mh, mw, rows, row_begin, n_words, out_h, out_w,
                                 absolute, !absolute, 0, 0.f, word_maps, nullptr, true, p.s, &dev)) return rc;
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (int rc = launch_region_masks(regions, n_regions, out_h, out_w, scratch, stream)) return rc;
  // a round: whole maps while a map's planes fit the scratch, else the words of one map in groups
  const int cap = (int)std::min<long long>((scratch_bytes - mask_bytes) / plane_bytes, 65535);
  const int maps_per_round = std::max(1, cap / n_words), words_per_round = std::min(cap, (int)n_words);
  for (int map0 = 0; map0 < n_maps; map0 += maps_per_round) {
    const int nm = std::min(maps_per_round, n_maps - map0);
    for (int w0 = 0; w0 < n_words; w0 += words_per_round) {
      const int nw = std::min(words_per_round, n_words - w0);
      q = p;
      q.s.maps = global_maps + map0 * p.s.map_stride;
      q.s.n_words = nw;
      for (int i = 0; i <= nw; ++i) q.s.row_begin[i] = p.s.row_begin[w0 + i];
      q.s.word_maps = word_maps + ((long long)map0 * n_words + w0) * mh * mw;
      RankingPlanes c;
      ranking_planes_in(scratch, nm * nw, out_h, out_w, c);
      q.s.scratch = c.minmax;
      q.pre = c.pre;
      if (int rc = launch_tiles(instance_mask_kernel, q, nm, dev, stream)) return rc;
      c.n_regions = n_regions; c.u2 = reinterpret_cast<long long*>(u2); c.ap = ap;
      c.n_words_round = nw; c.n_words = n_words; c.map0 = map0; c.w0 = w0;
      if (int rc = launch_ranking(c, stream)) return rc;
    }
  }
  return DAAM_OK;
}

extern "C" int daam_region_boundary(const float* global_maps, int32_t n_maps, int32_t n_rows, int32_t mh, int32_t mw,
                                    const int32_t* rows, const int32_t* row_begin, int32_t n_words, int32_t out_h,
                                    int32_t out_w, int32_t absolute, float threshold, const float* tolerances,
                                    int32_t n_tolerances, float* word_maps, const uint8_t* regions, int32_t n_regions,
                                    int32_t* word_boundary, int32_t* region_boundary, int32_t* word_hits,
                                    int32_t* region_hits, int64_t* max_d2, double* sum_dist, void* scratch,
                                    int64_t scratch_bytes, void* stream_) {
  const char* name = "daam_region_boundary";
  if (!global_maps || !rows || !row_begin || !tolerances || !word_maps || !regions || !word_boundary ||
      !region_boundary || !word_hits || !region_hits || !max_d2 || !sum_dist || !scratch || n_maps <= 0 || mh <= 0 ||
      mw <= 0 || out_h <= 0 || out_w <= 0 || n_rows <= 0 || n_regions <= 0 || n_tolerances <= 0) { set_error("%s: null pointer or non-positive size", name); return DAAM_E_INVALID; }
  if (n_tolerances > kBoundaryMaxTolerances) { set_error("%s: %d tolerances > %d", name, n_tolerances, kBoundaryMaxTolerances); return DAAM_E_UNSUPPORTED; }
  if (n_regions > kMaxRegions) { set_error("%s: %d regions > %d", name, n_regions, kMaxRegions); return DAAM_E_UNSUPPORTED; }
  if ((long long)out_h * out_w > (1LL << 24)) { set_error("%s: a %d x %d output is more than 2^24 pixels", name, out_h, out_w); return DAAM_E_UNSUPPORTED; }
  BoundaryPlanes c;
  if (int rc = boundary_check_tolerances(name, tolerances, n_tolerances, c)) return rc;
  if (!isfinite(threshold)) { set_error("%s: threshold %g is not finite", name, (double)threshold); return DAAM_E_INVALID; }
  if (int rc = boundary_check_scratch(name, scratch, scratch_bytes, n_regions, out_h, out_w)) return rc;
  static thread_local InstanceMaskParams p, q;
  DeviceInfo dev;
  if (int rc = word_list_prepare(name, global_maps, n_maps, n_rows, mh, mw, rows, row_begin, n_words, out_h, out_w,
                                 absolute, !absolute, 0, 0.f, word_maps, nullptr, true, p.s, &dev)) return rc;
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  c.word_boundary = word_boundary; c.region_boundary = region_boundary; c.word_hits = word_hits;
  c.region_hits = region_hits; c.max_d2 = reinterpret_cast<long long*>(max_d2); c.sum_dist = sum_dist;
  c.n_words = n_words;
  boundary_planes_in(scratch, n_regions, 1, out_h, out_w, c);
  if (int rc = launch_boundary_regions(regions, c, n_maps, stream)) return rc;
  // a round: whole maps while a map's planes fit the scratch, else the words of one map in groups
  const int cap = (int)std::min<long long>(
      (scratch_bytes - boundary_call_bytes(n_regions, out_h, out_w)) / boundary_plane_bytes(out_h, out_w), 65535);
  const int maps_per_round = std::max(1, cap / n_words), words_per_round = std::min(cap, (int)n_words);
  for (int map0 = 0; map0 < n_maps; map0 += maps_per_round) {
    const int nm = std::min(maps_per_round, n_maps - map0);
    for (int w0 = 0; w0 < n_words; w0 += words_per_round) {
      const int nw = std::min(words_per_round, n_words - w0);
      q = p;
      q.s.maps = global_maps + map0 * p.s.map_stride;
      q.s.n_words = nw;
      for (int i = 0; i <= nw; ++i) q.s.row_begin[i] = p.s.row_begin[w0 + i];
      q.s.word_maps = word_maps + ((long long)map0 * n_words + w0) * mh * mw;
      boundary_planes_in(scratch, n_regions, nm * nw, out_h, out_w, c);
      q.s.scratch = c.minmax;
      q.pre = c.pre;
      if (int rc = launch_tiles(instance_mask_kernel, q, nm, dev, stream)) return rc;
      c.n_words_round = nw; c.map0 = map0; c.w0 = w0;
      if (int rc = launch_boundary_round(c, threshold, nullptr, stream)) return rc;
    }
  }
  return DAAM_OK;
}

extern "C" int daam_word_distance(const float* global_maps, int32_t n_maps, int32_t n_rows, int32_t mh, int32_t mw,
                                  const int32_t* rows, const int32_t* row_begin, int32_t n_words, int32_t out_h,
                                  int32_t out_w, int32_t absolute, float threshold, float* word_maps,
                                  int32_t* signed_d2, void* scratch, int64_t scratch_bytes, void* stream_) {
  const char* name = "daam_word_distance";
  if (!global_maps || !rows || !row_begin || !word_maps || !signed_d2 || !scratch || n_maps <= 0 || mh <= 0 ||
      mw <= 0 || out_h <= 0 || out_w <= 0 || n_rows <= 0) { set_error("%s: null pointer or non-positive size", name); return DAAM_E_INVALID; }
  if (out_h > kDistanceMaxSide || out_w > kDistanceMaxSide) { set_error("%s: a %d x %d output has a side > %d", name, out_h, out_w, kDistanceMaxSide); return DAAM_E_UNSUPPORTED; }
  if ((long long)out_h * out_w > (1LL << 24)) { set_error("%s: a %d x %d output is more than 2^24 pixels", name, out_h, out_w); return DAAM_E_UNSUPPORTED; }
  if (!isfinite(threshold)) { set_error("%s: threshold %g is not finite", name, (double)threshold); return DAAM_E_INVALID; }
  if (int rc = distance_check_scratch(name, scratch, scratch_bytes, out_h, out_w)) return rc;
  static thread_local InstanceMaskParams p, q;
  DeviceInfo dev;
  if (int rc = word_list_prepare(name, global_maps, n_maps, n_rows, mh, mw, rows, row_begin, n_words, out_h, out_w,
                                 absolute, !absolute, 0, 0.f, word_maps, nullptr, true, p.s, &dev)) return rc;
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const long long n = (long long)out_h * out_w;
  // a round: whole maps while a map's planes fit the scratch, else the words of one map in groups; either way the
  // round's planes are consecutive in signed_d2
  const int cap = (int)std::min<long long>(scratch_bytes / distance_plane_bytes(out_h, out_w), 65535);
  const int maps_per_round = std::max(1, cap / n_words), words_per_round = std::min(cap, (int)n_words);
  for (int map0 = 0; map0 < n_maps; map0 += maps_per_round) {
    const int nm = std::min(maps_per_round, n_maps - map0);
    for (int w0 = 0; w0 < n_words; w0 += words_per_round) {
      const int nw = std::min(words_per_round, n_words - w0);
      q = p;
      q.s.maps = global_maps + map0 * p.s.map_stride;
      q.s.n_words = nw;
      for (int i = 0; i <= nw; ++i) q.s.row_begin[i] = p.s.row_begin[w0 + i];
      const long long plane0 = (long long)map0 * n_words + w0;
      q.s.word_maps = word_maps + plane0 * mh * mw;
      DistancePlanes c;
      distance_planes_in(scratch, nm * nw, out_h, out_w, c);
      q.s.scratch = c.minmax;
      q.pre = c.pre;
      if (int rc = launch_tiles(instance_mask_kernel, q, nm, dev, stream)) return rc;
      if (int rc = launch_distance(c.pre, threshold, nullptr, nm * nw, out_h, out_w, signed_d2 + plane0 * n, stream))
        return rc;
    }
  }
  return DAAM_OK;
}

extern "C" int daam_refine_words(const float* global_maps, int32_t n_maps, int32_t n_rows, int32_t mh, int32_t mw,
                                 const int32_t* rows, const int32_t* row_begin, int32_t n_words, int32_t out_h,
                                 int32_t out_w, int32_t absolute, int32_t use_threshold, float threshold,
                                 int32_t radius, float eps, float* word_maps, const uint8_t* image,
                                 int64_t image_map_stride, float* out, void* scratch, int64_t scratch_bytes,
                                 void* stream_) {
  const char* name = "daam_refine_words";
  if (!global_maps || !rows || !row_begin || !word_maps || !image || !out || !scratch || n_maps <= 0 || mh <= 0 ||
      mw <= 0 || out_h <= 0 || out_w <= 0 || n_rows <= 0 || image_map_stride < 0) { set_error("%s: null pointer or non-positive size", name); return DAAM_E_INVALID; }
  if (radius < 1 || radius > kRefineMaxRadius) { set_error("%s: radius %d is not in [1, %d]", name, radius, kRefineMaxRadius); return DAAM_E_INVALID; }
  if (!(eps > 0.f) || !isfinite(eps)) { set_error("%s: eps %g is not finite and > 0", name, (double)eps); return DAAM_E_INVALID; }
  if ((uintptr_t)scratch & 3) { set_error("%s: scratch must be 4-byte aligned", name); return DAAM_E_INVALID; }
  // the statistics of one image, then the planes of each round
  const long long guide_bytes = refine_guide_bytes(out_h, out_w), plane_bytes = refine_plane_bytes(out_h, out_w);
  if (scratch_bytes < guide_bytes + plane_bytes) { set_error("%s: %lld scratch bytes < %lld, one image's statistics and one %d x %d plane", name, (long long)scratch_bytes, guide_bytes + plane_bytes, out_h, out_w); return DAAM_E_INVALID; }
  static thread_local WordListParams p, q;
  DeviceInfo dev;
  if (int rc = word_list_prepare(name, global_maps, n_maps, n_rows, mh, mw, rows, row_begin, n_words, out_h, out_w,
                                 absolute, !absolute, 0, 0.f, word_maps, nullptr, true, p, &dev)) return rc;
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  // a round: whole maps while a map's planes (and with one image per map, its statistics) fit the scratch, else the
  // words of one map in groups
  const bool per_map = image_map_stride != 0;
  const long long map_bytes = (per_map ? guide_bytes : 0) + n_words * plane_bytes;
  const long long whole = std::min<long long>((scratch_bytes - (per_map ? 0 : guide_bytes)) / map_bytes, 65535 / n_words);
  const int maps_per_round = (int)std::max<long long>(1, std::min<long long>(whole, n_maps));
  const int words_per_round = whole >= 1 ? (int)n_words
                                         : (int)std::min<long long>((scratch_bytes - guide_bytes) / plane_bytes, n_words);
  RefinePlanes c;
  refine_planes_in(scratch, per_map ? maps_per_round : 1, maps_per_round * words_per_round, out_h, out_w, c);
  c.image_map_stride = image_map_stride;
  c.mh = mh; c.mw = mw; c.absolute = p.absolute; c.use_threshold = use_threshold ? 1 : 0; c.threshold = threshold;
  c.radius = radius; c.eps = eps;
  const long long n = (long long)out_h * out_w;
  for (int map0 = 0; map0 < n_maps; map0 += maps_per_round) {
    const int nm = std::min(maps_per_round, n_maps - map0);
    for (int w0 = 0; w0 < n_words; w0 += words_per_round) {
      const int nw = std::min(words_per_round, n_words - w0);
      q = p;
      q.maps = global_maps + map0 * p.map_stride;
      q.n_words = nw;
      for (int i = 0; i <= nw; ++i) q.row_begin[i] = p.row_begin[w0 + i];
      const long long plane0 = (long long)map0 * n_words + w0;
      q.word_maps = word_maps + plane0 * mh * mw;
      q.scratch = c.minmax;
      if (int rc = launch_word_maps(q, nm, dev, stream)) return rc;
      c.word_maps = q.word_maps; c.chunks = q.chunks;
      c.image = image + map0 * image_map_stride;
      c.planes = nm * nw; c.words_per_map = nw; c.out = out + plane0 * n;
      // the statistics of the round's images, kept while the words of one map take several rounds
      if (w0 == 0 && (per_map || map0 == 0)) {
        c.guides = per_map ? nm : 1;
        if (int rc = launch_refine_guides(c, stream)) return rc;
      }
      if (int rc = launch_refine(c, dev.device, stream)) return rc;
    }
  }
  return DAAM_OK;
}

extern "C" int daam_segment_crf(const float* global_maps, int32_t n_maps, int32_t n_rows, int32_t mh, int32_t mw,
                                const int32_t* rows, const int32_t* row_begin, int32_t n_words, int32_t out_h,
                                int32_t out_w, int32_t absolute, int32_t use_threshold, float threshold, float scale,
                                int32_t iterations, int32_t radius, float appearance, float sigma_xy, float sigma_rgb,
                                float smoothness, float sigma_smooth, float* word_maps, const uint8_t* image,
                                int64_t image_map_stride, uint8_t* labels, float* scores, float* probs, void* scratch,
                                int64_t scratch_bytes, void* stream_) {
  const char* name = "daam_segment_crf";
  if (!global_maps || !rows || !row_begin || !word_maps || !image || !labels || !scores || !scratch || n_maps <= 0 ||
      mh <= 0 || mw <= 0 || out_h <= 0 || out_w <= 0 || n_rows <= 0 || image_map_stride < 0) { set_error("%s: null pointer or non-positive size", name); return DAAM_E_INVALID; }
  if (radius < 1 || radius > kCrfMaxRadius) { set_error("%s: radius %d is not in [1, %d]", name, radius, kCrfMaxRadius); return DAAM_E_INVALID; }
  if (iterations < 0 || iterations > kCrfMaxIterations) { set_error("%s: iterations %d is not in [0, %d]", name, iterations, kCrfMaxIterations); return DAAM_E_INVALID; }
  const float positive[] = {scale, sigma_xy, sigma_rgb, sigma_smooth};
  const char* positive_names[] = {"scale", "sigma_xy", "sigma_rgb", "sigma_smooth"};
  for (int i = 0; i < 4; ++i)
    if (!(positive[i] > 0.f) || !isfinite(positive[i])) { set_error("%s: %s %g is not finite and > 0", name, positive_names[i], (double)positive[i]); return DAAM_E_INVALID; }
  if (!(appearance >= 0.f) || !isfinite(appearance)) { set_error("%s: appearance %g is not finite and >= 0", name, (double)appearance); return DAAM_E_INVALID; }
  if (!(smoothness >= 0.f) || !isfinite(smoothness)) { set_error("%s: smoothness %g is not finite and >= 0", name, (double)smoothness); return DAAM_E_INVALID; }
  if (use_threshold && !isfinite(threshold)) { set_error("%s: threshold %g is not finite", name, (double)threshold); return DAAM_E_INVALID; }
  if ((uintptr_t)scratch & 3) { set_error("%s: scratch must be 4-byte aligned", name); return DAAM_E_INVALID; }
  const int n_labels = n_words + (use_threshold ? 1 : 0);
  const long long map_bytes = crf_map_bytes(n_labels, out_h, out_w);
  if (scratch_bytes < map_bytes) { set_error("%s: %lld scratch bytes < %lld, one %d-label %d x %d map", name, (long long)scratch_bytes, map_bytes, n_labels, out_h, out_w); return DAAM_E_INVALID; }
  static thread_local WordListParams p, q;
  DeviceInfo dev;
  if (int rc = word_list_prepare(name, global_maps, n_maps, n_rows, mh, mw, rows, row_begin, n_words, out_h, out_w,
                                 absolute, !absolute, 0, 0.f, word_maps, nullptr, true, p, &dev)) return rc;
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  // a round: as many whole maps as the scratch holds (a map's labels are coupled: it is never split)
  const int maps_per_round = (int)std::min<long long>(std::min<long long>(scratch_bytes / map_bytes, 65535), n_maps);
  static thread_local CrfParams c;
  crf_tables(radius, appearance, sigma_xy, sigma_rgb, smoothness, sigma_smooth, c);
  c.image_map_stride = image_map_stride;
  c.n_words = n_words; c.n_labels = n_labels; c.mh = mh; c.mw = mw; c.oh = out_h; c.ow = out_w;
  c.absolute = p.absolute; c.use_threshold = use_threshold ? 1 : 0; c.threshold = use_threshold ? threshold : 0.f;
  c.scale = scale; c.radius = radius; c.q_in = nullptr;
  const long long n = (long long)out_h * out_w;
  float* minmax = static_cast<float*>(scratch);
  float* q_a = minmax + (long long)kWordPartialFloats * n_labels * maps_per_round;
  float* q_b = q_a + (long long)n_labels * n * maps_per_round;
  for (int map0 = 0; map0 < n_maps; map0 += maps_per_round) {
    const int nm = std::min(maps_per_round, n_maps - map0);
    q = p;
    q.maps = global_maps + map0 * p.map_stride;
    q.word_maps = word_maps + (long long)map0 * n_words * mh * mw;
    q.scratch = minmax;
    if (int rc = launch_word_maps(q, nm, dev, stream)) return rc;
    c.word_maps = q.word_maps; c.minmax = minmax; c.chunks = q.chunks; c.maps = nm;
    c.image = image + map0 * image_map_stride;
    c.labels = labels + map0 * n; c.scores = scores + map0 * n;
    if (int rc = launch_crf(c, iterations, q_a, q_b, probs ? probs + (long long)map0 * n_labels * n : nullptr,
                            dev.device, stream)) return rc;
  }
  return DAAM_OK;
}

extern "C" int daam_segment_superpixels(const float* global_maps, int32_t n_maps, int32_t n_rows, int32_t mh,
                                        int32_t mw, const int32_t* rows, const int32_t* row_begin, int32_t n_words,
                                        int32_t out_h, int32_t out_w, int32_t absolute, int32_t use_threshold,
                                        float threshold, int32_t n_segments, float compactness, int32_t iterations,
                                        float* word_maps, const uint8_t* image, int64_t image_map_stride,
                                        uint8_t* labels, float* scores, int32_t* superpixels, void* scratch,
                                        int64_t scratch_bytes, void* stream_) {
  const char* name = "daam_segment_superpixels";
  if (!global_maps || !rows || !row_begin || !word_maps || !image || !labels || !scores || !superpixels || !scratch ||
      n_maps <= 0 || mh <= 0 || mw <= 0 || out_h <= 0 || out_w <= 0 || n_rows <= 0 || image_map_stride < 0) { set_error("%s: null pointer or non-positive size", name); return DAAM_E_INVALID; }
  if ((long long)out_h * out_w > (1LL << 24)) { set_error("%s: a %d x %d output is more than 2^24 pixels", name, out_h, out_w); return DAAM_E_UNSUPPORTED; }
  if (n_segments < 1) { set_error("%s: n_segments %d < 1", name, n_segments); return DAAM_E_INVALID; }
  if (!(compactness > 0.f) || !isfinite(compactness)) { set_error("%s: compactness %g is not finite and > 0", name, (double)compactness); return DAAM_E_INVALID; }
  if (iterations < 1 || iterations > kSuperpixelMaxIterations) { set_error("%s: iterations %d is not in [1, %d]", name, iterations, kSuperpixelMaxIterations); return DAAM_E_INVALID; }
  const SlicGrid g = slic_grid(out_h, out_w, n_segments, compactness);
  if (g.cells > kSuperpixelMaxCells) { set_error("%s: a %d x %d grid of cells is more than %d", name, g.ny, g.nx, kSuperpixelMaxCells); return DAAM_E_UNSUPPORTED; }
  if ((uintptr_t)scratch & 7) { set_error("%s: scratch must be 8-byte aligned", name); return DAAM_E_INVALID; }
  const long long image_bytes = superpixel_image_bytes(g.cells), map_bytes = superpixel_map_bytes(n_words, g);
  if (scratch_bytes < image_bytes + map_bytes) { set_error("%s: %lld scratch bytes < %lld, one image and one %d-word map", name, (long long)scratch_bytes, image_bytes + map_bytes, n_words); return DAAM_E_INVALID; }
  static thread_local WordListParams p, q;
  DeviceInfo dev;
  if (int rc = word_list_prepare(name, global_maps, n_maps, n_rows, mh, mw, rows, row_begin, n_words, out_h, out_w,
                                 absolute, !absolute, 0, 0.f, word_maps, nullptr, true, p, &dev)) return rc;
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  // a round: as many whole maps as the scratch holds (a superpixel's pixels are pooled in one pass); one image's
  // partition serves every map, or each map has its own
  const bool per_map = image_map_stride != 0;
  const long long whole = per_map ? scratch_bytes / (image_bytes + map_bytes) : (scratch_bytes - image_bytes) / map_bytes;
  const int maps_per_round = (int)std::min<long long>(std::min<long long>(whole, 65535), n_maps);
  SlicParams s;
  PoolParams c;
  s.g = c.g = g;
  superpixel_scratch_in(scratch, per_map ? maps_per_round : 1, maps_per_round, n_words, g, s, c);
  float* minmax = const_cast<float*>(c.minmax);
  s.image_stride = image_map_stride;
  c.per_map = per_map ? 1 : 0; c.n_words = n_words; c.mh = mh; c.mw = mw; c.absolute = p.absolute;
  c.use_threshold = use_threshold ? 1 : 0; c.threshold = use_threshold ? threshold : 0.f;
  const long long n = (long long)out_h * out_w;
  for (int map0 = 0; map0 < n_maps; map0 += maps_per_round) {
    const int nm = std::min(maps_per_round, n_maps - map0);
    q = p;
    q.maps = global_maps + map0 * p.map_stride;
    q.word_maps = word_maps + (long long)map0 * n_words * mh * mw;
    q.scratch = minmax;
    if (int rc = launch_word_maps(q, nm, dev, stream)) return rc;
    if (per_map || map0 == 0) {
      s.images = per_map ? nm : 1;
      s.image = image + map0 * image_map_stride;
      s.superpixels = superpixels + (per_map ? map0 * n : 0);
      if (int rc = launch_slic(s, iterations, dev.device, stream)) return rc;
    }
    c.word_maps = q.word_maps; c.chunks = q.chunks; c.maps = nm; c.superpixels = s.superpixels;
    c.labels = labels + map0 * n; c.scores = scores + map0 * n;
    if (int rc = launch_pool(c, stream)) return rc;
  }
  return DAAM_OK;
}
