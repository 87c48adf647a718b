// Superpixel word segmentation (daam_image_superpixels, daam_segment_superpixels). SLIC over the RGB bytes, with the
// cell grid, centres and distances defined exactly (include/daam_b200.h), then the mean of each word's m over each
// superpixel and the word with the highest mean:
//  1. slic_init_kernel: each cluster's sums from the pixel at the middle of its cell;
//  2. slic_assign_kernel, once per pass: a 16 x 64 pixel tile stages the centres of the cells its pixels can reach in
//     shared memory; each pixel takes the nearest of the (up to) 9 centres around its cell, in float64 without FMA, the
//     lowest cluster on ties; the tile's integer sums per cluster go to `accum` with integer atomics;
//  3. slic_update_kernel, between passes: a cluster that has pixels takes their sums as its new state;
//  4. pool_tile_kernel: per tile and word, the float64 sum of m over each cell of the tile's box, each sum walking the
//     pixels in row-major order;
//  5. pool_cell_kernel: per superpixel, each word's sum over the tiles whose box holds it, in a fixed order, over its
//     pixel count, then the argmax over the words;
//  6. pool_paint_kernel: every pixel takes its superpixel's label and score.
// The only atomics are integer adds, whose results do not depend on their order, and every float sum has a fixed
// order: the results are the same bits on every call and however the maps are split into rounds.
#include <math.h>

#include <algorithm>
#include <mutex>

#include "bicubic.cuh"
#include "superpixels.cuh"
#include "word_value.cuh"

namespace daam {
namespace {

constexpr int kMaxBox = 19 * 67;     // box_h <= 15 + 4, box_w <= 63 + 4
constexpr int kPoolWords = 8;        // words whose m a pooling tile holds at once

__device__ __forceinline__ int cell_of(int y, int ny, int h) { return (int)(((long long)(y + 1) * ny - 1) / h); }
__device__ __forceinline__ int cell_begin(int c, int ny, int h) { return (int)((long long)c * h / ny); }

// grid: (clusters / 256, images); thread: one cluster's sums from its seed pixel, and zero sums
__global__ void __launch_bounds__(256) slic_init_kernel(const __grid_constant__ SlicParams P) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x, img = blockIdx.y;
  if (k >= P.g.cells) return;
  const int cy = k / P.g.nx, cx = k - cy * P.g.nx;
  const int y = (cell_begin(cy, P.g.ny, P.g.h) + cell_begin(cy + 1, P.g.ny, P.g.h) - 1) / 2;
  const int x = (cell_begin(cx, P.g.nx, P.g.w) + cell_begin(cx + 1, P.g.nx, P.g.w) - 1) / 2;
  const unsigned char* px = P.image + img * P.image_stride + ((long long)y * P.g.w + x) * 3;
  long long* s = P.state + ((long long)img * P.g.cells + k) * 6;
  unsigned long long* a = P.accum + ((long long)img * P.g.cells + k) * 6;
  s[0] = px[0]; s[1] = px[1]; s[2] = px[2]; s[3] = y; s[4] = x; s[5] = 1;
#pragma unroll
  for (int i = 0; i < 6; ++i) a[i] = 0;
}

// grid: (tiles of kSlicTileH x kSlicTileW pixels, images); dynamic smem: the centres [box][5] (float64) and the tile's
// sums [6][box] (int32, coordinates relative to the tile's corner) of the cells in the tile's box
__global__ void __launch_bounds__(256) slic_assign_kernel(const __grid_constant__ SlicParams P) {
  extern __shared__ __align__(16) double centres[];
  const SlicGrid& g = P.g;
  const int img = blockIdx.y, tiles_x = (g.w + kSlicTileW - 1) / kSlicTileW;
  const int y0 = (blockIdx.x / tiles_x) * kSlicTileH, x0 = (blockIdx.x % tiles_x) * kSlicTileW;
  const int th = min(kSlicTileH, g.h - y0), tw = min(kSlicTileW, g.w - x0);
  const int by0 = max(cell_of(y0, g.ny, g.h) - 1, 0), by1 = min(cell_of(y0 + th - 1, g.ny, g.h) + 1, g.ny - 1);
  const int bx0 = max(cell_of(x0, g.nx, g.w) - 1, 0), bx1 = min(cell_of(x0 + tw - 1, g.nx, g.w) + 1, g.nx - 1);
  const int bw = bx1 - bx0 + 1, box = (by1 - by0 + 1) * bw;
  int* sums = reinterpret_cast<int*>(centres + 5 * box);
  const long long* state = P.state + (long long)img * g.cells * 6;
  for (int j = threadIdx.x; j < box; j += blockDim.x) {
    const long long* s = state + ((long long)(by0 + j / bw) * g.nx + bx0 + j % bw) * 6;
    const double n = (double)s[5];
#pragma unroll
    for (int c = 0; c < 5; ++c) centres[5 * j + c] = __ddiv_rn((double)s[c], n);
  }
  for (int i = threadIdx.x; i < 6 * box; i += blockDim.x) sums[i] = 0;
  __syncthreads();
  const unsigned char* im = P.image + img * P.image_stride;
  for (int p = threadIdx.x; p < th * tw; p += blockDim.x) {
    const int ty = p / tw, tx = p - ty * tw, y = y0 + ty, x = x0 + tx;
    const unsigned char* px = im + ((long long)y * g.w + x) * 3;
    const double r = px[0], gr = px[1], b = px[2], fy = y, fx = x;
    const int cy = cell_of(y, g.ny, g.h), cx = cell_of(x, g.nx, g.w);
    double best = INFINITY;
    int arg = 0;
    // (cy + dy, cx + dx) in row-major order is ascending k: a strict < keeps the lowest cluster on ties
    for (int dy = -1; dy <= 1; ++dy) {
      const int ky = cy + dy;
      if (ky < 0 || ky >= g.ny) continue;
      for (int dx = -1; dx <= 1; ++dx) {
        const int kx = cx + dx;
        if (kx < 0 || kx >= g.nx) continue;
        const int j = (ky - by0) * bw + kx - bx0;
        const double* c = centres + 5 * j;
        const double er = __dsub_rn(r, c[0]), eg = __dsub_rn(gr, c[1]), eb = __dsub_rn(b, c[2]);
        const double ey = __dsub_rn(fy, c[3]), ex = __dsub_rn(fx, c[4]);
        const double colour = __dadd_rn(__dadd_rn(__dmul_rn(er, er), __dmul_rn(eg, eg)), __dmul_rn(eb, eb));
        const double d = __dadd_rn(colour, __dmul_rn(g.wxy, __dadd_rn(__dmul_rn(ey, ey), __dmul_rn(ex, ex))));
        if (d < best) { best = d; arg = j; }
      }
    }
    const int k = (by0 + arg / bw) * g.nx + bx0 + arg % bw;
    P.superpixels[(long long)img * g.h * g.w + (long long)y * g.w + x] = k;
    atomicAdd(&sums[arg], (int)px[0]);
    atomicAdd(&sums[box + arg], (int)px[1]);
    atomicAdd(&sums[2 * box + arg], (int)px[2]);
    atomicAdd(&sums[3 * box + arg], ty);
    atomicAdd(&sums[4 * box + arg], tx);
    atomicAdd(&sums[5 * box + arg], 1);
  }
  __syncthreads();
  for (int j = threadIdx.x; j < box; j += blockDim.x) {
    const int n = sums[5 * box + j];
    if (n == 0) continue;
    unsigned long long* a = P.accum + ((long long)img * g.cells + (long long)(by0 + j / bw) * g.nx + bx0 + j % bw) * 6;
    atomicAdd(a + 0, (unsigned long long)sums[j]);
    atomicAdd(a + 1, (unsigned long long)sums[box + j]);
    atomicAdd(a + 2, (unsigned long long)sums[2 * box + j]);
    atomicAdd(a + 3, (unsigned long long)((long long)sums[3 * box + j] + (long long)n * y0));
    atomicAdd(a + 4, (unsigned long long)((long long)sums[4 * box + j] + (long long)n * x0));
    atomicAdd(a + 5, (unsigned long long)n);
  }
}

// grid: (clusters / 256, images); thread: a cluster with pixels takes their sums; the sums restart from zero
__global__ void __launch_bounds__(256) slic_update_kernel(const __grid_constant__ SlicParams P) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= P.g.cells) return;
  const long long o = ((long long)blockIdx.y * P.g.cells + k) * 6;
  unsigned long long* a = P.accum + o;
  if (a[5]) {
#pragma unroll
    for (int i = 0; i < 6; ++i) P.state[o + i] = (long long)a[i];
  }
#pragma unroll
  for (int i = 0; i < 6; ++i) a[i] = 0;
}

// The first row (column) of the tile row (column) holding cell c's neighbourhood: cells c - 1 .. c + 1
__device__ __forceinline__ int box_origin(int t, int tile, int n_cells, int n) {
  return max(cell_of(t * tile, n_cells, n) - 1, 0);
}

// grid: (tiles of kSlicTileH x kSlicTileW pixels, maps); thread: m of the tile's pixels for a pass of words, then the
// sum of m over one (word, cell of the box) pair's pixels, in row-major order over the rows and columns of the cell's
// neighbourhood (the only pixels SLIC can give it)
__global__ void __launch_bounds__(256) pool_tile_kernel(const __grid_constant__ PoolParams P) {
  __shared__ float mv[kPoolWords][kSlicTileH * kSlicTileW];
  __shared__ short local[kSlicTileH * kSlicTileW];
  __shared__ float s_lo[kSuperpixelMaxWords], s_hi[kSuperpixelMaxWords];
  const SlicGrid& g = P.g;
  const int map = blockIdx.y, tiles_x = (g.w + kSlicTileW - 1) / kSlicTileW, tiles = gridDim.x;
  const int y0 = (blockIdx.x / tiles_x) * kSlicTileH, x0 = (blockIdx.x % tiles_x) * kSlicTileW;
  const int th = min(kSlicTileH, g.h - y0), tw = min(kSlicTileW, g.w - x0), tn = th * tw;
  const int by0 = box_origin(blockIdx.x / tiles_x, kSlicTileH, g.ny, g.h);
  const int bx0 = box_origin(blockIdx.x % tiles_x, kSlicTileW, g.nx, g.w);
  const int box = g.box_h * g.box_w, n_words = P.n_words;
  if (!P.absolute) {
    for (int w = threadIdx.x; w < n_words; w += blockDim.x) {
      float lo, hi;
      partial_bounds(P.minmax + 2LL * ((long long)map * n_words + w) * P.chunks, P.chunks, lo, hi);
      s_lo[w] = lo; s_hi[w] = hi;
    }
  }
  const int* sp = P.superpixels + (long long)map * P.per_map * g.h * g.w;
  for (int p = threadIdx.x; p < tn; p += blockDim.x) {
    const int ty = p / tw, k = sp[(long long)(y0 + ty) * g.w + x0 + p - ty * tw], ky = k / g.nx;
    local[p] = (short)((ky - by0) * g.box_w + k - ky * g.nx - bx0);
  }
  const float* word_maps = P.word_maps + (long long)map * n_words * P.mh * P.mw;
  for (int w0 = 0; w0 < n_words; w0 += kPoolWords) {
    const int nw = min(kPoolWords, n_words - w0);
    __syncthreads();                                     // the previous pass has read mv (and s_lo, local are written)
    for (int i = threadIdx.x; i < nw * tn; i += blockDim.x) {
      const int wi = i / tn, p = i - wi * tn, ty = p / tw, w = w0 + wi;
      float v = bicubic_shared(word_maps + (long long)w * P.mh * P.mw, P.mw, make_taps(y0 + ty, P.mh, g.h),
                               make_taps(x0 + p - ty * tw, P.mw, g.w));
      if (!P.absolute) v = minmax_normalize(v, s_lo[w], s_hi[w]);
      mv[wi][p] = v;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < nw * box; i += blockDim.x) {
      const int wi = i / box, j = i - wi * box, cy = by0 + j / g.box_w, cx = bx0 + j % g.box_w;
      double s = -0.0;                                   // the identity of +: a one-pixel sum keeps m's bits
      if (cy < g.ny && cx < g.nx) {
        const int r0 = max(cell_begin(max(cy - 1, 0), g.ny, g.h), y0) - y0;
        const int r1 = min(cell_begin(min(cy + 2, g.ny), g.ny, g.h), y0 + th) - y0;
        const int c0 = max(cell_begin(max(cx - 1, 0), g.nx, g.w), x0) - x0;
        const int c1 = min(cell_begin(min(cx + 2, g.nx), g.nx, g.w), x0 + tw) - x0;
        for (int r = r0; r < r1; ++r)
          for (int c = c0; c < c1; ++c)
            if (local[r * tw + c] == j) s = __dadd_rn(s, (double)mv[wi][r * tw + c]);
      }
      P.partials[(((long long)map * n_words + w0 + wi) * tiles + blockIdx.x) * box + j] = s;
    }
  }
}

// grid: (map, cluster) pairs / 8; warp: one superpixel's means over the words, its label and score
__global__ void __launch_bounds__(256) pool_cell_kernel(const __grid_constant__ PoolParams P) {
  const SlicGrid& g = P.g;
  const long long pair = (long long)blockIdx.x * 8 + threadIdx.x / 32;
  const int lane = threadIdx.x & 31;
  if (pair >= (long long)P.maps * g.cells) return;
  const int map = (int)(pair / g.cells), k = (int)(pair - (long long)map * g.cells);
  const unsigned long long n = P.accum[((long long)map * P.per_map * g.cells + k) * 6 + 5];
  if (n == 0) return;                                    // an empty cluster: no pixel takes its id
  const int cy = k / g.nx, cx = k - cy * g.nx, tiles_x = (g.w + kSlicTileW - 1) / kSlicTileW;
  const int tiles = tiles_x * ((g.h + kSlicTileH - 1) / kSlicTileH), box = g.box_h * g.box_w;
  // the tiles whose pixels meet the rows / columns of cells cy - 1 .. cy + 1, cx - 1 .. cx + 1: those whose box holds k
  const int ty0 = cell_begin(max(cy - 1, 0), g.ny, g.h) / kSlicTileH;
  const int ty1 = (cell_begin(min(cy + 2, g.ny), g.ny, g.h) - 1) / kSlicTileH;
  const int tx0 = cell_begin(max(cx - 1, 0), g.nx, g.w) / kSlicTileW;
  const int tx1 = (cell_begin(min(cx + 2, g.nx), g.nx, g.w) - 1) / kSlicTileW;
  const int ntc = tx1 - tx0 + 1, nt = (ty1 - ty0 + 1) * ntc;
  float best = -INFINITY;
  int arg = 0;
  for (int w = 0; w < P.n_words; ++w) {
    const double* part = P.partials + ((long long)map * P.n_words + w) * tiles * box;
    double s = -0.0;
    for (int i = lane; i < nt; i += 32) {
      const int tr = ty0 + i / ntc, tc = tx0 + i % ntc;
      const int j = (cy - box_origin(tr, kSlicTileH, g.ny, g.h)) * g.box_w + cx - box_origin(tc, kSlicTileW, g.nx, g.w);
      s = __dadd_rn(s, part[(long long)(tr * tiles_x + tc) * box + j]);
    }
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) s = __dadd_rn(s, __shfl_xor_sync(0xffffffffu, s, m));   // same bits in every lane
    const float mean = (float)__ddiv_rn(s, (double)n);
    if (w == 0 || mean > best) { best = mean; arg = w; }   // strict: the lowest word wins a tie
  }
  if (lane == 0) {
    P.cell_score[(long long)map * g.cells + k] = best;
    P.cell_label[(long long)map * g.cells + k] = (!P.use_threshold || best > P.threshold) ? arg + 1 : 0;
  }
}

// grid: (pixels / 256, maps); thread: one pixel's label and score, its superpixel's
__global__ void __launch_bounds__(256) pool_paint_kernel(const __grid_constant__ PoolParams P) {
  const long long n = (long long)P.g.h * P.g.w, o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= n) return;
  const int map = blockIdx.y, k = P.superpixels[(long long)map * P.per_map * n + o];
  P.labels[(long long)map * n + o] = (unsigned char)P.cell_label[(long long)map * P.g.cells + k];
  P.scores[(long long)map * n + o] = P.cell_score[(long long)map * P.g.cells + k];
}

long long tile_count(const SlicGrid& g) {
  return (long long)((g.h + kSlicTileH - 1) / kSlicTileH) * ((g.w + kSlicTileW - 1) / kSlicTileW);
}

}  // namespace

SlicGrid slic_grid(int out_h, int out_w, int n_segments, float compactness) {
  SlicGrid g;
  g.h = out_h; g.w = out_w;
  const double hw = (double)out_h * out_w, s = sqrt(hw / (double)n_segments);
  g.ny = (int)std::min<double>(std::max<double>(floor(out_h / s + 0.5), 1.0), out_h);
  g.nx = (int)std::min<double>(std::max<double>(floor(out_w / s + 0.5), 1.0), out_w);
  g.cells = (long long)g.ny * g.nx > kSuperpixelMaxCells ? kSuperpixelMaxCells + 1 : g.ny * g.nx;
  g.box_h = std::min(g.ny, (int)(15LL * g.ny / out_h) + 4);
  g.box_w = std::min(g.nx, (int)(63LL * g.nx / out_w) + 4);
  const double c = compactness;
  g.wxy = c * c * (double)((long long)g.ny * g.nx) / hw;
  return g;
}

long long superpixel_image_bytes(int cells) { return 96LL * cells; }

long long superpixel_map_bytes(int n_words, const SlicGrid& g) {
  return 4LL * kWordPartialFloats * n_words + 8LL * g.cells + 8LL * n_words * tile_count(g) * g.box_h * g.box_w;
}

void superpixel_scratch_in(void* scratch, int images, int maps, int n_words, const SlicGrid& g, SlicParams& s,
                           PoolParams& p) {
  char* b = static_cast<char*>(scratch);
  s.state = reinterpret_cast<long long*>(b);
  s.accum = reinterpret_cast<unsigned long long*>(b + 48LL * images * g.cells);
  b += superpixel_image_bytes(g.cells) * images;
  p.partials = reinterpret_cast<double*>(b);
  b += 8LL * maps * n_words * tile_count(g) * g.box_h * g.box_w;
  p.minmax = reinterpret_cast<float*>(b);
  b += 4LL * kWordPartialFloats * maps * n_words;
  p.cell_score = reinterpret_cast<float*>(b);
  p.cell_label = reinterpret_cast<int*>(b + 4LL * maps * g.cells);
  p.accum = s.accum;
}

int launch_slic(SlicParams& p, int iterations, int device, cudaStream_t stream) {
  static std::once_flag attr_once[64];
  cudaError_t attr_err = cudaSuccess;
  std::call_once(attr_once[device & 63], [&] {
    attr_err = cudaFuncSetAttribute(slic_assign_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)((5 * sizeof(double) + 6 * sizeof(int)) * kMaxBox));
  });
  DAAM_CUDA_TRY(attr_err);
  const dim3 cells((unsigned)((p.g.cells + 255) / 256), (unsigned)p.images);
  const dim3 tiles((unsigned)tile_count(p.g), (unsigned)p.images);
  const size_t smem = (5 * sizeof(double) + 6 * sizeof(int)) * (size_t)p.g.box_h * p.g.box_w;
  slic_init_kernel<<<cells, 256, 0, stream>>>(p);
  DAAM_CUDA_TRY(cudaGetLastError());
  count_launch();
  for (int it = 0; it < iterations; ++it) {
    if (it > 0) {
      slic_update_kernel<<<cells, 256, 0, stream>>>(p);
      DAAM_CUDA_TRY(cudaGetLastError());
      count_launch();
    }
    slic_assign_kernel<<<tiles, 256, smem, stream>>>(p);
    DAAM_CUDA_TRY(cudaGetLastError());
    count_launch();
  }
  return DAAM_OK;
}

int launch_pool(PoolParams& p, cudaStream_t stream) {
  pool_tile_kernel<<<dim3((unsigned)tile_count(p.g), (unsigned)p.maps), 256, 0, stream>>>(p);
  DAAM_CUDA_TRY(cudaGetLastError());
  pool_cell_kernel<<<(unsigned)(((long long)p.maps * p.g.cells + 7) / 8), 256, 0, stream>>>(p);
  DAAM_CUDA_TRY(cudaGetLastError());
  const long long n = (long long)p.g.h * p.g.w;
  pool_paint_kernel<<<dim3((unsigned)((n + 255) / 256), (unsigned)p.maps), 256, 0, stream>>>(p);
  DAAM_CUDA_TRY(cudaGetLastError());
  count_launch(3);
  return DAAM_OK;
}

}  // namespace daam

using namespace daam;

extern "C" int daam_image_superpixels(const uint8_t* image, int32_t n_images, int32_t out_h, int32_t out_w,
                                      int32_t n_segments, float compactness, int32_t iterations, int32_t* superpixels,
                                      void* scratch, int64_t scratch_bytes, void* stream_) {
  const char* name = "daam_image_superpixels";
  if (!image || !superpixels || !scratch || n_images <= 0 || out_h <= 0 || out_w <= 0) { set_error("%s: null pointer or non-positive size", name); return DAAM_E_INVALID; }
  if ((long long)out_h * out_w > (1LL << 24)) { set_error("%s: a %d x %d image is more than 2^24 pixels", name, out_h, out_w); return DAAM_E_UNSUPPORTED; }
  if (n_segments < 1) { set_error("%s: n_segments %d < 1", name, n_segments); return DAAM_E_INVALID; }
  if (!(compactness > 0.f) || !isfinite(compactness)) { set_error("%s: compactness %g is not finite and > 0", name, (double)compactness); return DAAM_E_INVALID; }
  if (iterations < 1 || iterations > kSuperpixelMaxIterations) { set_error("%s: iterations %d is not in [1, %d]", name, iterations, kSuperpixelMaxIterations); return DAAM_E_INVALID; }
  SlicParams p;
  p.g = slic_grid(out_h, out_w, n_segments, compactness);
  if (p.g.cells > kSuperpixelMaxCells) { set_error("%s: a %d x %d grid of cells is more than %d", name, p.g.ny, p.g.nx, kSuperpixelMaxCells); return DAAM_E_UNSUPPORTED; }
  if ((uintptr_t)scratch & 7) { set_error("%s: scratch must be 8-byte aligned", name); return DAAM_E_INVALID; }
  const long long image_bytes = superpixel_image_bytes(p.g.cells);
  if (scratch_bytes < image_bytes) { set_error("%s: %lld scratch bytes < %lld, one image of %d cells", name, (long long)scratch_bytes, image_bytes, p.g.cells); return DAAM_E_INVALID; }
  DeviceInfo dev;
  if (int rc = get_device_info(&dev)) return rc;
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  const long long n = (long long)out_h * out_w;
  const int per_round = (int)std::min<long long>(std::min<long long>(scratch_bytes / image_bytes, 65535), n_images);
  PoolParams unused;
  superpixel_scratch_in(scratch, per_round, 0, 0, p.g, p, unused);
  p.image_stride = 3 * n;
  for (int i0 = 0; i0 < n_images; i0 += per_round) {
    p.images = std::min(per_round, n_images - i0);
    p.image = image + i0 * 3 * n;
    p.superpixels = superpixels + i0 * n;
    if (int rc = launch_slic(p, iterations, dev.device, stream)) return rc;
  }
  return DAAM_OK;
}
