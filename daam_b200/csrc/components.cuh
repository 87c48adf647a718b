// Connected components of thresholded word maps: the labelling and per-component statistics behind
// daam_word_instances (components.cu). words.cu's instance_mask_kernel writes each plane's values `pre`; the kernels
// here label the mask pre > threshold (8-connected) and reduce each component to its statistics.
#pragma once

#include "common.cuh"

namespace daam {

constexpr int kMaxInstances = DAAM_WORD_INSTANCES_MAX;   // max_instances: the instances kept per plane

// One round of planes (a plane: one (map, word) pair): the scratch buffers, laid out by instance_planes_in, and the
// outputs of the round's first plane. A slot is a 2 x 2 pixel block: an 8-connected component owns every pixel of a
// block it touches, so a block holds at most one component's first pixel, and the slot of a component is the block
// of its first pixel.
struct InstancePlanes {
  unsigned long long* peak;   // [planes][slots]: orderable bits of the max of pre << 32 | (0xFFFFFFFF - its pixel)
  unsigned long long* sums;   // [planes][slots][2]: sums of the row and column indices
  float* pre;                 // [planes][h][w]
  int* label;                 // [planes][h][w]: a union-find parent, then the component's first pixel; -1 background
  int* area;                  // [planes][slots]
  int* box;                   // [planes][slots][4]: min row, min column, max row, max column
  int* roots;                 // [planes][slots]: the first pixels of the components, in no particular order
  int* n_roots;               // [planes]
  float* minmax;              // [planes][64]: segment_minmax_kernel's partials
  int planes, h, w, k;
  float threshold;
  int* count;                 // outputs from the round's first plane: [planes]
  int* out_area;              // [planes][k]
  int* out_box;               // [planes][k][4], half-open
  long long* out_sum;         // [planes][k][2]
  float* out_peak;            // [planes][k]
  int* out_peak_yx;           // [planes][k][2]
};

// DAAM_WORD_INSTANCES_PLANE_BYTES: the scratch one plane takes
long long instance_plane_bytes(int h, int w);
// Points the scratch buffers of `p` into `scratch` for `planes` planes of h x w pixels.
void instance_planes_in(void* scratch, int planes, int h, int w, InstancePlanes& p);
// The labelling and statistics launches over the planes of `p` (five launches).
int launch_components(const InstancePlanes& p, cudaStream_t stream);

}  // namespace daam
