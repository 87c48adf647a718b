// Word distance maps: the exact signed squared Euclidean distance transform of a mask, behind daam_word_distance
// (words.cu, whose instance_mask_kernel writes each plane's values `pre`) and daam_mask_distance (distance.cu, masks
// given on the device).
#pragma once

#include "common.cuh"

namespace daam {

constexpr int kDistanceMaxSide = DAAM_DISTANCE_MAX_SIDE;

// One round of daam_word_distance's planes in its scratch, laid out by distance_planes_in.
struct DistancePlanes {
  float* pre;                    // [planes][n]: the values
  float* minmax;                 // [planes][64]: segment_minmax_kernel's partials
};

// DAAM_DISTANCE_PLANE_BYTES
long long distance_plane_bytes(int h, int w);
// The scratch check of daam_word_distance: DAAM_E_INVALID with the error set, or DAAM_OK.
int distance_check_scratch(const char* name, const void* scratch, long long scratch_bytes, int h, int w);
// Points the buffers of `p` into `scratch` for `planes` planes of h x w pixels.
void distance_planes_in(void* scratch, int planes, int h, int w, DistancePlanes& p);
// The signed transform of `planes` planes of h x w pixels into signed_d2 [planes][h][w], from pre > threshold (masks
// null) or from masks != 0: the column pass, then the row pass in place (two launches per 65535 planes).
int launch_distance(const float* pre, float threshold, const unsigned char* masks, int planes, int h, int w,
                    int* signed_d2, cudaStream_t stream);

}  // namespace daam
