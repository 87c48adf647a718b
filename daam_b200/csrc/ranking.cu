// Region ranking: per plane (one (map, word) pair) and region r, twice the Mann-Whitney U and the average precision of
// the plane's values `pre` (words.cu's instance_mask_kernel) against the region's pixels (daam_region_ranking).
// With the values sorted descending and cut into tie groups g, tp_g / fp_g the group's pixels inside / outside the
// region, TP_< / FP_< those above the group and TP_<= = TP_< + tp_g, FP_<= = FP_< + fp_g:
//   u2 = sum_g tp_g (2 (n_n - FP_<=) + fp_g) = 2 n_p n_n - sum_g tp_g (FP_< + FP_<=)
//   ap = sum_g tp_g / n_p * TP_<= / (TP_<= + FP_<=)
// Sixteen launches over the planes of a round:
//  1-12. a least-significant-digit radix sort of every plane at once, 8 bits a pass: per pass the digit counts of
//        each 4096-key tile (rank_digits_kernel), their exclusive scan per plane in (digit, tile) order
//        (rank_scan_kernel), and a stable scatter (rank_scatter_kernel). The keys are the fp32 bits made orderable,
//        -0 folded onto +0, and inverted, so ascending keys are descending values; each key carries its pixel index.
//  13. rank_segments_kernel: one warp per segment of kRankSegment sorted positions counts the positives of every
//      region (the pixel's bit in the region masks, one ballot per region and 32 positions) and those before the
//      segment's last tie-group start;
//  14. rank_carry_kernel: per plane, in segment order, the positives before each segment and, for the tie group open
//      at its start, that group's first position and the positives before it; the totals are n_p;
//  15. rank_groups_kernel: one warp per segment walks its positions in order, lane l holding regions l and l + 32,
//      and adds every group that ends in the segment to the segment's sums of tp_g (FP_< + FP_<=) (integers) and of
//      tp_g TP_<= / (TP_<= + FP_<=) (float64, in position order: the exact product times the rounded reciprocal);
//  16. rank_reduce_kernel: per (plane, region) the segments' sums, lane-strided and then a butterfly: u2 and ap.
// No float atomics anywhere, and the only atomics are integer adds to shared digit counts: the results are the same
// bits on every call, and they do not depend on how the planes are split into rounds.
#include <math.h>

#include "ranking.cuh"
#include "word_value.cuh"

namespace daam {
namespace {

constexpr int kSortThreads = 256;
constexpr int kSortItems = 16;                       // keys per thread and tile
constexpr int kSortTile = kSortThreads * kSortItems;  // 4096 keys per tile
constexpr int kRankSegment = 1024;                    // sorted positions per warp of the group kernels

// The sort key of a value: orderable fp32 bits (-0 taken as +0), inverted so that ascending keys are descending values
__device__ __forceinline__ unsigned descending_key(float f) {
  const unsigned u = f == 0.f ? 0u : __float_as_uint(f);
  return ~((u & 0x80000000u) ? ~u : u | 0x80000000u);
}

__device__ __forceinline__ unsigned key_at(const unsigned* src, bool first, long long i) {
  return first ? descending_key(reinterpret_cast<const float*>(src)[i]) : src[i];
}

// grid: (tiles, planes), kSortThreads threads: the digit counts of one tile. A warp's lanes of one digit add once.
__global__ void __launch_bounds__(kSortThreads) rank_digits_kernel(const __grid_constant__ RankingPlanes P,
                                                                   const unsigned* __restrict__ keys_in, int first,
                                                                   int shift) {
  __shared__ unsigned hist[256];
  const int t = threadIdx.x, lane = t & 31, plane = blockIdx.y, n = P.n;
  hist[t] = 0u;
  __syncthreads();
  const unsigned* src = keys_in + (long long)plane * n;
  unsigned keys[kSortItems];                            // every load of the tile in flight at once
#pragma unroll
  for (int k = 0; k < kSortItems; ++k) {
    const int i = blockIdx.x * kSortTile + k * kSortThreads + t;
    keys[k] = i < n ? key_at(src, first, i) : 0u;
  }
#pragma unroll
  for (int k = 0; k < kSortItems; ++k) {
    const int i = blockIdx.x * kSortTile + k * kSortThreads + t;
    const bool valid = i < n;
    const unsigned d = valid ? (keys[k] >> shift) & 255u : 256u + lane;
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    if (valid && lane == __ffs(peers) - 1) atomicAdd(hist + d, (unsigned)__popc(peers));
  }
  __syncthreads();
  P.digits[((long long)plane * 256 + t) * P.tiles + blockIdx.x] = hist[t];
}

// grid: planes, 1024 threads: the exclusive scan of a plane's digit counts in (digit, tile) order, in place; each
// thread takes 4 consecutive counts per step of 4096
__global__ void __launch_bounds__(1024) rank_scan_kernel(const __grid_constant__ RankingPlanes P) {
  __shared__ unsigned sums[32];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  unsigned* a = P.digits + (long long)blockIdx.x * 256 * P.tiles;
  const int total = 256 * P.tiles;
  unsigned carry = 0u;
  for (int base = 0; base < total; base += 4096) {
    const int i0 = base + 4 * t;
    unsigned v[4], s = 0u;
#pragma unroll
    for (int j = 0; j < 4; ++j) { v[j] = i0 + j < total ? a[i0 + j] : 0u; s += v[j]; }
    unsigned x = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) sums[warp] = x;
    __syncthreads();
    if (warp == 0) {
      unsigned w = sums[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned y = __shfl_up_sync(0xffffffffu, w, o);
        if (lane >= o) w += y;
      }
      sums[lane] = w;
    }
    __syncthreads();
    unsigned run = carry + (warp ? sums[warp - 1] : 0u) + x - s;
#pragma unroll
    for (int j = 0; j < 4; ++j) if (i0 + j < total) { a[i0 + j] = run; run += v[j]; }
    carry += sums[31];
    __syncthreads();                                  // sums is rewritten by the next step
  }
}

// grid: (tiles, planes), kSortThreads threads: the stable scatter of one tile. Its keys go in kSortItems steps of
// 256 in position order; in each step a key's place is the tile's running offset of its digit, plus the keys of that
// digit in earlier warps, plus its rank among its warp's peers (__match_any_sync).
__global__ void __launch_bounds__(kSortThreads) rank_scatter_kernel(const __grid_constant__ RankingPlanes P,
                                                                    const unsigned* __restrict__ keys_in,
                                                                    const unsigned* __restrict__ idx_in,
                                                                    unsigned* __restrict__ keys_out,
                                                                    unsigned* __restrict__ idx_out, int first,
                                                                    int shift) {
  __shared__ unsigned offset[256];                     // per digit: where the tile's next key of that digit goes
  __shared__ unsigned count[kSortThreads / 32][256];   // per warp and digit: keys of this step
  __shared__ unsigned before[kSortThreads / 32][256];  // per warp and digit: where the warp's first such key goes
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5, plane = blockIdx.y, n = P.n;
  offset[t] = P.digits[((long long)plane * 256 + t) * P.tiles + blockIdx.x];
#pragma unroll
  for (int w = 0; w < kSortThreads / 32; ++w) count[w][t] = 0u;
  __syncthreads();
  const long long base = (long long)plane * n;
  const unsigned* src = keys_in + base;
  unsigned keys[kSortItems], ids[kSortItems];           // every load of the tile in flight at once
#pragma unroll
  for (int k = 0; k < kSortItems; ++k) {
    const int i = blockIdx.x * kSortTile + k * kSortThreads + t;
    keys[k] = i < n ? key_at(src, first, i) : 0u;
    ids[k] = i < n ? (first ? (unsigned)i : idx_in[base + i]) : 0u;
  }
#pragma unroll
  for (int k = 0; k < kSortItems; ++k) {
    const int i = blockIdx.x * kSortTile + k * kSortThreads + t;
    const bool valid = i < n;
    const unsigned key = keys[k], id = ids[k];
    const unsigned d = valid ? (key >> shift) & 255u : 256u + lane;
    const unsigned peers = __match_any_sync(0xffffffffu, d);
    const int rank = __popc(peers & ((1u << lane) - 1u));
    if (valid && rank == 0) count[warp][d] = __popc(peers);
    __syncthreads();
    {                                                  // thread t: digit t over the warps, in warp order
      unsigned acc = offset[t];
#pragma unroll
      for (int w = 0; w < kSortThreads / 32; ++w) {
        const unsigned c = count[w][t];
        count[w][t] = 0u;
        before[w][t] = acc;
        acc += c;
      }
      offset[t] = acc;
    }
    __syncthreads();
    if (valid) {
      const long long o = base + before[warp][d] + rank;
      keys_out[o] = key;
      idx_out[o] = id;
    }
  }
}

// 32 sorted positions [c0, c0 + 32) of a plane, clipped to `end`: which start and which end a tie group, and lane l's
// ballots of regions l (lo) and l + 32 (hi) over them
struct Chunk {
  unsigned starts, ends, lo, hi;
};

__device__ __forceinline__ Chunk load_chunk(const RankingPlanes& P, const unsigned* keys, const unsigned* idx, int c0,
                                            int end) {
  const int lane = threadIdx.x & 31, i = c0 + lane, n = P.n;
  const bool valid = i < end;
  unsigned long long m = 0ull;
  bool start = false, stop = false;
  if (valid) {
    const unsigned key = keys[i];
    start = i == 0 || keys[i - 1] != key;
    stop = i == n - 1 || keys[i + 1] != key;
    m = __ldg(P.masks + idx[i]);
  }
  Chunk c;
  c.starts = __ballot_sync(0xffffffffu, start);
  c.ends = __ballot_sync(0xffffffffu, stop);
  c.lo = 0u; c.hi = 0u;
  for (int r = 0; r < P.n_regions; ++r) {
    const unsigned b = __ballot_sync(0xffffffffu, (m >> r) & 1ull);
    if (r < 32) { if (lane == r) c.lo = b; }
    else if (lane == r - 32) c.hi = b;
  }
  return c;
}

// the planes' sorted keys and pixel indices after the four passes
__device__ __forceinline__ const unsigned* sorted_keys(const RankingPlanes& P, int plane) {
  return reinterpret_cast<const unsigned*>(P.pre) + (long long)plane * P.n;
}
__device__ __forceinline__ const unsigned* sorted_idx(const RankingPlanes& P, int plane) {
  return P.idx[1] + (long long)plane * P.n;
}

// grid: (ceil(segs / 8), planes), 256 threads: warp = segment
__global__ void __launch_bounds__(256) rank_segments_kernel(const __grid_constant__ RankingPlanes P) {
  const int lane = threadIdx.x & 31, seg = blockIdx.x * 8 + (threadIdx.x >> 5), plane = blockIdx.y;
  if (seg >= P.segs) return;                           // whole warps
  const unsigned* keys = sorted_keys(P, plane);
  const unsigned* idx = sorted_idx(P, plane);
  const int begin = seg * kRankSegment, end = min(P.n, begin + kRankSegment);
  unsigned cnt_lo = 0u, cnt_hi = 0u, pre_lo = 0u, pre_hi = 0u;
  int last = -1;
  for (int c0 = begin; c0 < end; c0 += 32) {
    const Chunk c = load_chunk(P, keys, idx, c0, end);
    if (c.starts) {
      const int j = 31 - __clz(c.starts);
      const unsigned lt = (1u << j) - 1u;
      last = c0 + j;
      pre_lo = cnt_lo + __popc(c.lo & lt); pre_hi = cnt_hi + __popc(c.hi & lt);
    }
    cnt_lo += __popc(c.lo); cnt_hi += __popc(c.hi);
  }
  const long long o = ((long long)plane * P.segs + seg) * 64;
  P.seg_cnt[o + lane] = cnt_lo; P.seg_cnt[o + 32 + lane] = cnt_hi;
  P.seg_pre[o + lane] = pre_lo; P.seg_pre[o + 32 + lane] = pre_hi;
  if (lane == 0) P.seg_start[(long long)plane * P.segs + seg] = last;
}

// grid: planes, 32 threads (lane l: regions l and l + 32); in place over the segment arrays. Segment s + 1 is loaded
// before segment s is written back, so the loop does not wait on a load per segment.
__global__ void __launch_bounds__(32) rank_carry_kernel(const __grid_constant__ RankingPlanes P) {
  const int lane = threadIdx.x, plane = blockIdx.x;
  unsigned run_lo = 0u, run_hi = 0u, open_lo = 0u, open_hi = 0u;
  int open = 0;                                        // position 0 starts a group
  unsigned* cnt = P.seg_cnt + (long long)plane * P.segs * 64;
  unsigned* pre = P.seg_pre + (long long)plane * P.segs * 64;
  int* start = P.seg_start + (long long)plane * P.segs;
  unsigned c_lo = cnt[lane], c_hi = cnt[32 + lane], p_lo = pre[lane], p_hi = pre[32 + lane];
  int last = start[0];
  for (int s = 0; s < P.segs; ++s) {
    const long long o = (long long)s * 64, q = s + 1 < P.segs ? o + 64 : o;
    const unsigned nc_lo = cnt[q + lane], nc_hi = cnt[q + 32 + lane], np_lo = pre[q + lane], np_hi = pre[q + 32 + lane];
    const int next = start[s + 1 < P.segs ? s + 1 : s];
    __syncwarp();                                      // every lane has read start[s + 1] before lane 0 writes start[s]
    cnt[o + lane] = run_lo; cnt[o + 32 + lane] = run_hi;
    pre[o + lane] = open_lo; pre[o + 32 + lane] = open_hi;
    if (lane == 0) start[s] = open;
    if (last >= 0) { open = last; open_lo = run_lo + p_lo; open_hi = run_hi + p_hi; }
    run_lo += c_lo; run_hi += c_hi;
    c_lo = nc_lo; c_hi = nc_hi; p_lo = np_lo; p_hi = np_hi; last = next;
  }
  P.n_pos[plane * 64 + lane] = run_lo;
  P.n_pos[plane * 64 + 32 + lane] = run_hi;
}

// A group that ends at `pos` - 1 and started at `open`: TP_<= = tp_le, positives before it `open_cnt`; rcp = 1 / pos
__device__ __forceinline__ void add_group(unsigned tp_le, unsigned open_cnt, int pos, int open, double rcp,
                                          unsigned long long& s, double& ap) {
  const unsigned tp = tp_le - open_cnt;
  if (tp == 0u) return;
  const unsigned fp = (unsigned)(pos - open) - tp, fp_le = (unsigned)pos - tp_le;
  s += (unsigned long long)tp * (2u * fp_le - fp);     // tp (FP_< + FP_<=)
  ap += (double)((unsigned long long)tp * tp_le) * rcp;   // the product is exact: below 2^48
}

// grid: (ceil(segs / 8), planes), 256 threads: warp = segment
__global__ void __launch_bounds__(256) rank_groups_kernel(const __grid_constant__ RankingPlanes P) {
  const int lane = threadIdx.x & 31, seg = blockIdx.x * 8 + (threadIdx.x >> 5), plane = blockIdx.y;
  if (seg >= P.segs) return;                           // whole warps
  const unsigned* keys = sorted_keys(P, plane);
  const unsigned* idx = sorted_idx(P, plane);
  const long long o = ((long long)plane * P.segs + seg) * 64;
  unsigned base_lo = P.seg_cnt[o + lane], base_hi = P.seg_cnt[o + 32 + lane];
  unsigned open_lo = P.seg_pre[o + lane], open_hi = P.seg_pre[o + 32 + lane];
  int open = P.seg_start[(long long)plane * P.segs + seg];
  unsigned long long s_lo = 0ull, s_hi = 0ull;
  double ap_lo = 0.0, ap_hi = 0.0;
  const int begin = seg * kRankSegment, end = min(P.n, begin + kRankSegment);
  const bool hi = P.n_regions > 32;
  for (int c0 = begin; c0 < end; c0 += 32) {
    const Chunk c = load_chunk(P, keys, idx, c0, end);
    const double rcp = 1.0 / (double)(c0 + lane + 1);  // 1 / (TP_<= + FP_<=) at each of the chunk's positions
    for (unsigned ev = c.starts | c.ends; ev; ev &= ev - 1u) {   // warp-uniform, in position order
      const int j = __ffs(ev) - 1;
      const unsigned bit = 1u << j;
      if (c.starts & bit) {
        open = c0 + j;
        open_lo = base_lo + __popc(c.lo & (bit - 1u)); open_hi = base_hi + __popc(c.hi & (bit - 1u));
      }
      if (c.ends & bit) {
        const unsigned le = bit | (bit - 1u);
        const double r = __shfl_sync(0xffffffffu, rcp, j);
        add_group(base_lo + __popc(c.lo & le), open_lo, c0 + j + 1, open, r, s_lo, ap_lo);
        if (hi) add_group(base_hi + __popc(c.hi & le), open_hi, c0 + j + 1, open, r, s_hi, ap_hi);
      }
    }
    base_lo += __popc(c.lo); base_hi += __popc(c.hi);
  }
  P.part_s[o + lane] = s_lo; P.part_s[o + 32 + lane] = s_hi;
  P.part_ap[o + lane] = ap_lo; P.part_ap[o + 32 + lane] = ap_hi;
}

// grid: ceil(planes * n_regions / 8), 256 threads: one warp per (plane, region) sums the segments' partials
// (lane-strided, then a butterfly) in a fixed order
__global__ void __launch_bounds__(256) rank_reduce_kernel(const __grid_constant__ RankingPlanes P) {
  const long long o = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (o >= (long long)P.planes * P.n_regions) return;  // whole warps
  const int lane = threadIdx.x & 31;
  const int plane = (int)(o / P.n_regions), r = (int)(o - (long long)plane * P.n_regions);
  unsigned long long s = 0ull;
  double a = 0.0;
  for (int g = lane; g < P.segs; g += 32) {
    const long long i = ((long long)plane * P.segs + g) * 64 + r;
    s += P.part_s[i];
    a += P.part_ap[i];
  }
#pragma unroll
  for (int h = 16; h > 0; h >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, h);
    a += __shfl_xor_sync(0xffffffffu, a, h);
  }
  if (lane == 0) {
    const unsigned long long n_p = P.n_pos[plane * 64 + r], n_n = (unsigned long long)P.n - n_p;
    const int map = plane / P.n_words_round, word = plane - map * P.n_words_round;
    const long long out = ((long long)(P.map0 + map) * P.n_regions + r) * P.n_words + P.w0 + word;
    P.u2[out] = (long long)(2ull * n_p * n_n - s);
    P.ap[out] = n_p ? a / (double)n_p : nan("");
  }
}

// grid: ceil(n / 256): bit r of masks[p] is regions[r][p] != 0
__global__ void __launch_bounds__(256) region_mask_kernel(const unsigned char* __restrict__ regions, int n_regions,
                                                          int n, unsigned long long* __restrict__ masks) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  unsigned long long m = 0ull;
  for (int r = 0; r < n_regions; ++r)
    if (__ldg(regions + (long long)r * n + p)) m |= 1ull << r;
  masks[p] = m;
}

int tiles_of(long long n) { return (int)((n + kSortTile - 1) / kSortTile); }
int segs_of(long long n) { return (int)((n + kRankSegment - 1) / kRankSegment); }

}  // namespace

long long ranking_plane_bytes(int h, int w) {
  const long long n = (long long)h * w;
  // segs_of: ceil(n / 1024); then n_pos and the min / max partials
  return 16 * n + 1024LL * tiles_of(n) + 1540LL * segs_of(n) + 4 * 64 + 4 * kWordPartialFloats;
}

void ranking_planes_in(void* scratch, int planes, int h, int w, RankingPlanes& p) {
  const long long n = (long long)h * w, tiles = tiles_of(n), segs = segs_of(n);
  char* c = static_cast<char*>(scratch);             // the 8-byte arrays first
  p.masks = reinterpret_cast<const unsigned long long*>(c); c += 8 * n;
  p.part_s = reinterpret_cast<unsigned long long*>(c); c += 8 * planes * segs * 64;
  p.part_ap = reinterpret_cast<double*>(c); c += 8 * planes * segs * 64;
  p.pre = reinterpret_cast<float*>(c); c += 4 * planes * n;
  p.keys = reinterpret_cast<unsigned*>(c); c += 4 * planes * n;
  p.idx[0] = reinterpret_cast<unsigned*>(c); c += 4 * planes * n;
  p.idx[1] = reinterpret_cast<unsigned*>(c); c += 4 * planes * n;
  p.digits = reinterpret_cast<unsigned*>(c); c += 4 * planes * 256 * tiles;
  p.seg_cnt = reinterpret_cast<unsigned*>(c); c += 4 * planes * segs * 64;
  p.seg_pre = reinterpret_cast<unsigned*>(c); c += 4 * planes * segs * 64;
  p.seg_start = reinterpret_cast<int*>(c); c += 4 * planes * segs;
  p.n_pos = reinterpret_cast<unsigned*>(c); c += 4LL * planes * 64;
  p.minmax = reinterpret_cast<float*>(c);
  p.planes = planes; p.n = (int)n; p.tiles = (int)tiles; p.segs = (int)segs;
}

int launch_region_masks(const unsigned char* regions, int n_regions, int h, int w, void* scratch, cudaStream_t stream) {
  const int n = h * w;
  region_mask_kernel<<<(n + 255) / 256, 256, 0, stream>>>(regions, n_regions, n,
                                                          static_cast<unsigned long long*>(scratch));
  DAAM_CUDA_TRY(cudaGetLastError());
  count_launch();
  return DAAM_OK;
}

int launch_ranking(const RankingPlanes& p, cudaStream_t stream) {
  // pre -> keys -> pre -> keys -> pre; idx[0] -> idx[1] -> idx[0] -> idx[1]
  unsigned* keys[2] = {reinterpret_cast<unsigned*>(p.pre), p.keys};
  const dim3 tiles(p.tiles, p.planes), segs((p.segs + 7) / 8, p.planes);
  for (int pass = 0; pass < 4; ++pass) {
    const unsigned* k_in = keys[pass & 1];
    const int first = pass == 0, shift = 8 * pass;
    rank_digits_kernel<<<tiles, kSortThreads, 0, stream>>>(p, k_in, first, shift);
    DAAM_CUDA_TRY(cudaGetLastError());
    rank_scan_kernel<<<p.planes, 1024, 0, stream>>>(p);
    DAAM_CUDA_TRY(cudaGetLastError());
    rank_scatter_kernel<<<tiles, kSortThreads, 0, stream>>>(p, k_in, first ? nullptr : p.idx[(pass + 1) & 1],
                                                            keys[(pass + 1) & 1], p.idx[pass & 1], first, shift);
    DAAM_CUDA_TRY(cudaGetLastError());
  }
  rank_segments_kernel<<<segs, 256, 0, stream>>>(p);
  DAAM_CUDA_TRY(cudaGetLastError());
  rank_carry_kernel<<<p.planes, 32, 0, stream>>>(p);
  DAAM_CUDA_TRY(cudaGetLastError());
  rank_groups_kernel<<<segs, 256, 0, stream>>>(p);
  DAAM_CUDA_TRY(cudaGetLastError());
  const long long n_out = (long long)p.planes * p.n_regions;
  rank_reduce_kernel<<<(unsigned)((n_out + 7) / 8), 256, 0, stream>>>(p);
  DAAM_CUDA_TRY(cudaGetLastError());
  count_launch(16);
  return DAAM_OK;
}

}  // namespace daam
