// Superpixel word segmentation: SLIC superpixels of the image (Achanta et al., "SLIC Superpixels Compared to
// State-of-the-Art Superpixel Methods", TPAMI 2012, in the pixel-centric form on the RGB bytes) and one word label per
// superpixel, behind daam_image_superpixels (superpixels.cu) and daam_segment_superpixels (words.cu). words.cu's
// segment_minmax_kernel writes the word maps and their min / max partials; the pooling kernels here recompute m from
// them, as crf.cu does, and never write the [n_words][out_h][out_w] stack of m.
#pragma once

#include "common.cuh"

namespace daam {

constexpr int kSuperpixelMaxCells = DAAM_SUPERPIXEL_MAX_CELLS;
constexpr int kSuperpixelMaxIterations = 64;
constexpr int kSuperpixelMaxWords = 96;
constexpr int kSlicTileH = 16, kSlicTileW = 64;   // the output tile of the assignment and pooling kernels

// The cell grid of an out_h x out_w image for n_segments superpixels (S = sqrt(H W / K) in float64; ny, nx its rows
// and columns) and the bound box_h x box_w on the cells a tile's pixels can be assigned to: the cells its rows and
// columns span, widened by one on each side.
struct SlicGrid {
  int h, w, ny, nx, cells, box_h, box_w;
  double wxy;                          // c * c * (ny * nx) / (H * W), left to right in float64
};
SlicGrid slic_grid(int out_h, int out_w, int n_segments, float compactness);

// One round of images: what the SLIC kernels read and write.
struct SlicParams {
  const unsigned char* image;         // [images][h][w][3]: image i at image + i * image_stride
  long long image_stride;             // bytes
  long long* state;                   // [images][cells][6]: (sum r, g, b, y, x, n) of the current centres
  unsigned long long* accum;          // [images][cells][6]: the same sums over the pass's assignment
  int* superpixels;                   // [images][h][w]
  int images;
  SlicGrid g;
};

// DAAM_SUPERPIXEL_IMAGE_BYTES: one image's state and sums
long long superpixel_image_bytes(int cells);
// DAAM_SUPERPIXEL_MAP_BYTES: one map's min / max partials, per-tile partial sums and per-superpixel label and score
long long superpixel_map_bytes(int n_words, const SlicGrid& g);
// The partition of p.images images: 2 * iterations launches. After it, accum's n is each superpixel's pixel count.
int launch_slic(SlicParams& p, int iterations, int device, cudaStream_t stream);

// One round of maps: what the pooling kernels read and write.
struct PoolParams {
  const float* word_maps;             // [maps][n_words][mh][mw]: the round's word maps (segment_minmax_kernel's)
  const float* minmax;                // [maps][n_words][chunks][2]: their min / max partials (unused with absolute)
  const int* superpixels;             // [images][h][w]: map i's partition at superpixels + i * per_map * h * w
  const unsigned long long* accum;    // [images][cells][6]: launch_slic's sums (n: the pixel count)
  double* partials;                   // [maps][n_words][tiles][box_h * box_w]: each tile's sum of m per cell of its box
  float* cell_score;                  // [maps][cells]
  int* cell_label;                    // [maps][cells]
  unsigned char* labels;              // [maps][h][w] of the round
  float* scores;                      // [maps][h][w] of the round
  int maps, per_map, n_words, mh, mw, chunks, absolute, use_threshold;
  float threshold;
  SlicGrid g;
};

// The pooled labels of the round's maps, after segment_minmax_kernel and launch_slic: 3 launches.
int launch_pool(PoolParams& p, cudaStream_t stream);
// The scratch layout of daam_segment_superpixels: `images` images' SLIC state, then `maps` maps' pooling buffers.
void superpixel_scratch_in(void* scratch, int images, int maps, int n_words, const SlicGrid& g, SlicParams& s,
                           PoolParams& p);

}  // namespace daam
