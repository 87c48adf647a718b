// CRF-refined word segmentation: mean-field inference of a Potts CRF over the word maps with the image as a bilateral
// guide (Kraehenbuehl and Koltun, NeurIPS 2011, in the exact windowed form of Teichmann and Cipolla's ConvCRF, BMVC
// 2019), behind daam_segment_crf (crf.cu). words.cu's segment_minmax_kernel writes the word maps and their min / max
// partials; the kernels here recompute m from them, as refine.cu does, and never write the [n_words][out_h][out_w]
// stack of m.
#pragma once

#include "common.cuh"

namespace daam {

constexpr int kCrfMaxRadius = DAAM_CRF_MAX_RADIUS;
constexpr int kCrfTaps = (2 * kCrfMaxRadius + 1) * (2 * kCrfMaxRadius + 1);
constexpr int kCrfMaxIterations = 64;
constexpr int kCrfMaxWords = 96;

// One round of whole maps: what the kernels read and write. Label l's logit is z_l = scale * s_l with s_0 = threshold
// (use_threshold only) and s_{w + use_threshold} = m[w]; the output label of l is l + 1 - use_threshold.
struct CrfParams {
  const float* word_maps;             // [maps][n_words][mh][mw]: the round's word maps (segment_minmax_kernel's)
  const float* minmax;                // [maps][n_words][chunks][2]: their min / max partials (unused with absolute)
  const unsigned char* image;         // [oh][ow][3] of the round's first map; map i at image + i * image_map_stride
  long long image_map_stride;         // bytes; 0: one image for every map
  const float* q_in;                  // [maps][n_labels][n]: Q of the previous update (crf_step_kernel)
  float* q_out;                       // [maps][n_labels][n]: the logits, then Q in place
  unsigned char* labels;              // [maps][n] of the round, written by the last launch
  float* scores;                      // [maps][n] of the round, written by the last launch
  int maps, n_words, n_labels, mh, mw, oh, ow, chunks, absolute, use_threshold, radius, last;
  float threshold, scale, rgb_coef;   // rgb_coef = fp32(1 / (2 sigma_rgb^2))
  float A[kCrfTaps], S[kCrfTaps];     // [(2r+1)^2] tables, row-major over (o_y, o_x); the centre entry is unused
};

// DAAM_CRF_MAP_BYTES: one map's two Q buffers and its min / max partials
long long crf_map_bytes(int n_labels, int h, int w);
// The appearance and smoothness tables of `p`, in float64 rounded once to fp32, and rgb_coef.
void crf_tables(int radius, float appearance, float sigma_xy, float sigma_rgb, float smoothness, float sigma_smooth,
                CrfParams& p);
// Q^0 and `iterations` mean-field updates over the round's maps, after segment_minmax_kernel (1 + iterations
// launches). q_a / q_b: the round's two Q buffers; probs: the round's [maps][n_labels][n] output, or nullptr.
int launch_crf(CrfParams& p, int iterations, float* q_a, float* q_b, float* probs, int device, cudaStream_t stream);

}  // namespace daam
