// Edge-aware word maps: the guided filter (He, Sun and Tang, "Guided Image Filtering", TPAMI 2013, colour guide) of
// each word's map m with the image as guide, behind daam_refine_words (refine.cu). words.cu's segment_minmax_kernel
// writes the word maps and their min / max partials; the kernels here recompute m from them, as the tile kernels do,
// and never write the [n_words][out_h][out_w] stack of m.
#pragma once

#include "common.cuh"

namespace daam {

constexpr int kRefineMaxRadius = 64;

// One round of planes (a plane: one (map, word) pair) of n = oh * ow pixels: the scratch buffers, laid out by
// refine_planes_in, and what the kernels read and write.
struct RefinePlanes {
  const float* word_maps;             // [planes][mh][mw]: the round's word maps (segment_minmax_kernel's)
  float* minmax;                      // [planes][chunks][2]: their min / max partials (unused with absolute)
  const unsigned char* image;         // [oh][ow][3] of the round's first map; map i at image + i * image_map_stride
  long long image_map_stride;         // bytes; 0: one image for every map
  float* guide;                       // [guides][9][n]: mu_r, mu_g, mu_b, then (Sigma + eps Id)^-1 rr, rg, rb, gg, gb, bb
  float* buf;                         // [planes][8][n]: window sums (channels 0-3), a_r, a_g, a_b, b (channels 4-7);
                                      // a guide's integer row sums while its statistics are built (guide g in plane g)
  float* out;                         // [planes][n] of the round: q, or q > threshold as 1 / 0
  int planes, words_per_map, guides;  // plane p is word p % words_per_map of map p / words_per_map of the round
  int mh, mw, oh, ow, chunks, absolute, use_threshold, radius;
  float threshold, eps;
};

// DAAM_REFINE_GUIDE_BYTES / DAAM_REFINE_PLANE_BYTES: one image's statistics, one plane's buffers and partials
long long refine_guide_bytes(int h, int w);
long long refine_plane_bytes(int h, int w);
// Points the buffers of `p` into `scratch` for `guides` guides and `planes` planes of h x w pixels.
void refine_planes_in(void* scratch, int guides, int planes, int h, int w, RefinePlanes& p);
// The guide statistics of the round's first p.guides images (two launches).
int launch_refine_guides(const RefinePlanes& p, cudaStream_t stream);
// The filter over the round's planes, after segment_minmax_kernel and the guides (four launches).
int launch_refine(const RefinePlanes& p, int device, cudaStream_t stream);

}  // namespace daam
