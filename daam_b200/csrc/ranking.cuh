// Threshold-free ranking scores of word maps against image regions: the sort and the counts behind
// daam_region_ranking (ranking.cu). words.cu's instance_mask_kernel writes each plane's values `pre`; the kernels here
// sort every plane's values, descending, and turn the sorted order into twice the Mann-Whitney U and the average
// precision of each region.
#pragma once

#include "common.cuh"

namespace daam {

// One round of planes (a plane: one (map, word) pair) over n = h * w pixels: the scratch buffers, laid out by
// ranking_planes_in, and the outputs of the round's first plane. The sorted order is cut into segments of
// kRankSegment positions, one warp each.
struct RankingPlanes {
  const unsigned long long* masks;   // [n]: bit r set where regions[r] is nonzero (shared by every round)
  unsigned long long* part_s;        // [planes][segs][64]: per segment, sum of tp_g (FP_< + FP_<=) over its groups
  double* part_ap;                   // [planes][segs][64]: per segment, sum of tp_g TP_<= / (TP_<= + FP_<=)
  float* pre;                        // [planes][n]: the values; the sort's first key buffer
  unsigned* keys;                    // [planes][n]: the other key buffer
  unsigned* idx[2];                  // [planes][n] each: pixel indices carried by the sort
  unsigned* digits;                  // [planes][256][tiles]: digit counts, then their exclusive scan
  unsigned* seg_cnt;                 // [planes][segs][64]: positives per segment, then the count before it
  unsigned* seg_pre;                 // [planes][segs][64]: positives before the segment's last group start, then the
                                     // count at the start of the group open before the segment
  int* seg_start;                    // [planes][segs]: the segment's last group start (-1: none), then the start of
                                     // the group open before it
  unsigned* n_pos;                   // [planes][64]: pixels inside each region
  float* minmax;                     // [planes][64]: segment_minmax_kernel's partials
  int planes, n, tiles, segs, n_regions;
  // outputs of the round: plane p = map_local * n_words_round + word_local goes to map map0 + map_local, word
  // w0 + word_local of u2 / ap [n_maps][n_regions][n_words]
  long long* u2;
  double* ap;
  int n_words_round, n_words, map0, w0;
};

// DAAM_REGION_RANKING_PLANE_BYTES: the scratch one plane takes (the region masks come on top, once per call)
long long ranking_plane_bytes(int h, int w);
// Points the buffers of `p` into `scratch` for `planes` planes of h x w pixels, after the region masks.
void ranking_planes_in(void* scratch, int planes, int h, int w, RankingPlanes& p);
// The region masks of `regions` [n_regions][h][w] into the start of `scratch` (one launch).
int launch_region_masks(const unsigned char* regions, int n_regions, int h, int w, void* scratch, cudaStream_t stream);
// The sort and the counts over the planes of `p` (sixteen launches).
int launch_ranking(const RankingPlanes& p, cudaStream_t stream);

}  // namespace daam
