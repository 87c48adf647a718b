// Boundary scores of word masks against image regions: the boundaries, their column distances and the nearest-boundary
// queries behind daam_region_boundary (words.cu, whose instance_mask_kernel writes each plane's values `pre`) and
// daam_mask_boundary (boundary.cu, masks given on the device).
#pragma once

#include "common.cuh"

namespace daam {

constexpr int kBoundaryMaxTolerances = DAAM_BOUNDARY_MAX_TOLERANCES;

// One round of planes (a plane: one (map, word) pair, or one mask) of n = h * w pixels: the scratch buffers, laid out
// by boundary_planes_in, and the outputs. A column distance g(y, x) is the distance from (y, x) to the nearest boundary
// pixel in column x (0 on a boundary pixel), or kBoundaryNone when the column has none.
struct BoundaryPlanes {
  int* g_region;                 // [n_regions][n]: the regions' column distances (shared by every round)
  char* partials;                // [planes][tiles]: one query tile's hit bins, maxima and sums (kBoundaryTileBytes)
  float* pre;                    // [planes][n]: the values (region entry)
  int* g_plane;                  // [planes][n]: the planes' column distances
  float* minmax;                 // [planes][64]: segment_minmax_kernel's partials
  int planes, h, w, n_regions, tiles, tile_rows, n_tolerances;
  double tol2[kBoundaryMaxTolerances];   // theta_k^2, exact in float64
  // outputs of the call: plane p = map_local * n_words_round + word_local goes to map map0 + map_local, word
  // w0 + word_local; the mask entry has one word per map
  int* word_boundary;            // [n_maps][n_words]: zeroed per call, then counted by the column kernel
  int* region_boundary;          // [n_regions]: likewise
  int* word_hits;                // [n_maps][T][n_regions][n_words]
  int* region_hits;              // same shape
  long long* max_d2;             // [n_maps][n_regions][n_words][2]
  double* sum_dist;              // same shape
  int n_words_round, n_words, map0, w0;
};

// DAAM_BOUNDARY_CALL_BYTES / DAAM_BOUNDARY_PLANE_BYTES
long long boundary_call_bytes(int n_regions, int h, int w);
long long boundary_plane_bytes(int h, int w);
// The checks both entry points make on the tolerances (fills p.tol2 and p.n_tolerances) and on the scratch, in that
// order; DAAM_E_INVALID with the error set, or DAAM_OK.
int boundary_check_tolerances(const char* name, const float* tolerances, int n_tolerances, BoundaryPlanes& p);
int boundary_check_scratch(const char* name, const void* scratch, long long scratch_bytes, int n_regions, int h, int w);
// Points the buffers of `p` into `scratch` for `planes` planes of h x w pixels after the regions' state, and sets the
// tile geometry.
void boundary_planes_in(void* scratch, int n_regions, int planes, int h, int w, BoundaryPlanes& p);
// Zeroes the boundary counts of n_maps x n_words planes and of the regions, then the regions' boundaries and column
// distances from `regions` [n_regions][h][w] (two memsets, one launch).
int launch_boundary_regions(const unsigned char* regions, const BoundaryPlanes& p, int n_maps, cudaStream_t stream);
// One round: the planes' boundaries and column distances, from pre > threshold (masks null) or from masks != 0, then
// the queries and their reduction (three launches).
int launch_boundary_round(const BoundaryPlanes& p, float threshold, const unsigned char* masks, cudaStream_t stream);

}  // namespace daam
