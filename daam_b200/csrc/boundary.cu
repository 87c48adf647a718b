// Boundary scores: per plane (one (map, word) pair, or one mask) and region r, the distances between the plane's mask
// boundary dA and the region's boundary dB_r, each boundary pixel to the nearest pixel of the other boundary
// (daam_region_boundary, daam_mask_boundary). A full 2-D distance transform is not needed: distances are only read at
// boundary pixels of the other set, and with g_S(y, x) the vertical distance from (y, x) to the nearest pixel of S in
// column x,
//   d2(p, S) = min_dx dx^2 + g_S(p_y, p_x +- dx)^2,
// which a warp scans outward along p's row, 32 columns a step, until dx^2 reaches the best value found: exact, and
// every read coalesced along the row.
//  - boundary_columns_kernel, once per call over the regions and once per round over the planes: one thread per column
//    marks the boundary (a pixel inside whose 4-neighbours are not all inside the image and the mask) in a down sweep
//    that also takes the distance to the boundary above, then an up sweep takes the distance to the one below; it
//    counts the boundary pixels into word_boundary / region_boundary with integer atomics;
//  - boundary_query_kernel, grid (row tiles, planes): each warp takes rows of its tile; per row, every dA pixel (in x
//    order) is queried against every nonempty region's g, and every dB_r pixel against the plane's g. Lane 0 adds the
//    pixel's first tolerance that holds to a shared bin (integer atomics), its d2 to a shared maximum and sqrt(d2) to
//    its warp's float64 sum, in position order; the tile's partials are the bins, maxima and the warps' sums in warp
//    order;
//  - boundary_reduce_kernel: per (plane, region, direction), the tiles' partials in tile order, the bins summed into
//    cumulative hit counts.
// No float atomics, and every float64 sum runs in an order fixed by pixel positions: the results are the same bits on
// every call and whatever the split of the planes into rounds.
#include <limits.h>
#include <math.h>

#include <algorithm>

#include "boundary.cuh"
#include "word_value.cuh"

namespace daam {
namespace {

constexpr int kBoundaryNone = 1 << 30;              // column distance where the column has no boundary pixel
constexpr int kBoundaryRegions = DAAM_REGION_MAX_REGIONS;
constexpr int kColumnThreads = 128;
constexpr int kQueryWarps = 8;
// one tile's partials: int bins [63][2][16], uint64 maxima [63][2], float64 sums [63][2]
constexpr int kBinBytes = kBoundaryRegions * 2 * kBoundaryMaxTolerances * 4;
constexpr int kMaxBytes = kBoundaryRegions * 2 * 8;
constexpr int kBoundaryTileBytes = kBinBytes + 2 * kMaxBytes;
static_assert(kBoundaryTileBytes == 10080, "DAAM_BOUNDARY_PLANE_BYTES counts 10080 bytes per tile");
static_assert(DAAM_BOUNDARY_PLANE_BYTES(0, 1) == kWordPartialFloats * sizeof(float),
              "DAAM_BOUNDARY_PLANE_BYTES counts one plane's min / max partials");

struct MaskIn {
  const unsigned char* m;
  __device__ __forceinline__ bool at(long long i) const { return m[i] != 0; }
};
struct ValueIn {
  const float* m;
  float threshold;
  __device__ __forceinline__ bool at(long long i) const { return m[i] > threshold; }
};

// grid: (ceil(w / kColumnThreads), planes): one thread per column of a plane. Plane p's count goes to
// count[(p / per_map) * map_stride + p % per_map].
template <class In>
__global__ void __launch_bounds__(kColumnThreads) boundary_columns_kernel(const In in, int h, int w,
                                                                          int* __restrict__ g, int* __restrict__ count,
                                                                          int per_map, int map_stride) {
  const int x = blockIdx.x * kColumnThreads + threadIdx.x, plane = blockIdx.y;
  const long long n = (long long)h * w, base = plane * n;
  int found = 0;
  if (x < w) {
    bool up = false, c = in.at(base + x);
    int last = -1;                                   // the row of the last boundary pixel above
#pragma unroll 4
    for (int y = 0; y < h; ++y) {
      const long long i = base + (long long)y * w + x;
      const bool dn = y + 1 < h && in.at(i + w);
      const bool l = x > 0 && in.at(i - 1), r = x + 1 < w && in.at(i + 1);
      const bool b = c && !(up && dn && l && r);
      if (b) { last = y; ++found; }
      g[i] = b ? 0 : last >= 0 ? y - last : kBoundaryNone;
      up = c; c = dn;
    }
    int next = -1;                                   // the row of the last boundary pixel below
#pragma unroll 4
    for (int y = h - 1; y >= 0; --y) {
      const long long i = base + (long long)y * w + x;
      const int v = g[i];
      if (v == 0) next = y;
      else if (next >= 0 && next - y < v) g[i] = next - y;
    }
  }
  for (int s = 16; s; s >>= 1) found += __shfl_xor_sync(0xffffffffu, found, s);
  if ((threadIdx.x & 31) == 0 && found) atomicAdd(count + (plane / per_map) * map_stride + plane % per_map, found);
}

// d2 from (y, x) to the nearest pixel of the set whose column distances of row y are `row` (at least one column of the
// image has one): the warp scans 32 columns a step on each side, until the next step's dx^2 reaches the best value.
// Every lane returns it.
__device__ __forceinline__ long long nearest_d2(const int* __restrict__ row, int w, int x, int lane) {
  long long best = LLONG_MAX;
  const int reach = max(x, w - 1 - x);
  for (int off = 0; off <= reach; off += 32) {
    const int dx = off + lane;
    const long long dx2 = (long long)dx * dx;
    long long v = LLONG_MAX;
    if (x + dx < w) {
      const long long g = row[x + dx];
      if (g != kBoundaryNone) v = dx2 + g * g;
    }
    if (x - dx >= 0) {
      const long long g = row[x - dx];
      if (g != kBoundaryNone) v = min(v, dx2 + g * g);
    }
    for (int s = 16; s; s >>= 1) v = min(v, __shfl_xor_sync(0xffffffffu, v, s));
    best = min(best, v);
    const long long next = off + 32;
    if (next * next >= best) break;
  }
  return best;
}

__device__ __forceinline__ void add_query(const BoundaryPlanes& P, int* bins, unsigned long long* mx, double& sum,
                                          long long d2) {
  const double d = (double)d2;
  int k = 0;
  while (k < P.n_tolerances && d > P.tol2[k]) ++k;
  if (k < P.n_tolerances) atomicAdd(bins + k, 1);
  atomicMax(mx, (unsigned long long)d2);
  sum += sqrt(d);
}

// grid: (tiles, planes), kQueryWarps warps: warp v takes rows tile * tile_rows + v, + kQueryWarps, ... of its tile
__global__ void __launch_bounds__(kQueryWarps * 32) boundary_query_kernel(const __grid_constant__ BoundaryPlanes P) {
  __shared__ int s_bins[kBoundaryRegions][2][kBoundaryMaxTolerances];
  __shared__ unsigned long long s_max[kBoundaryRegions][2];
  __shared__ double s_sum[kQueryWarps][kBoundaryRegions][2];
  __shared__ int s_has[kBoundaryRegions];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5, tile = blockIdx.x, plane = blockIdx.y;
  const int R = P.n_regions, T = P.n_tolerances, w = P.w;
  for (int i = t; i < R * 2 * kBoundaryMaxTolerances; i += blockDim.x) (&s_bins[0][0][0])[i] = 0;
  for (int i = t; i < R * 2; i += blockDim.x) (&s_max[0][0])[i] = 0ull;
  for (int i = t; i < kQueryWarps * kBoundaryRegions * 2; i += blockDim.x) (&s_sum[0][0][0])[i] = 0.0;
  for (int r = t; r < R; r += blockDim.x) s_has[r] = P.region_boundary[r] > 0;
  __syncthreads();
  const int ml = plane / P.n_words_round, wl = plane - ml * P.n_words_round;
  const bool has_a = P.word_boundary[(long long)(P.map0 + ml) * P.n_words + P.w0 + wl] > 0;
  const long long n = (long long)P.h * w;
  const int* g_a = P.g_plane + plane * n;
  const int y_end = min(P.h, (tile + 1) * P.tile_rows);
  for (int y = tile * P.tile_rows + warp; has_a && y < y_end; y += kQueryWarps) {
    const int* row_a = g_a + (long long)y * w;
    // every dA pixel against every region
    for (int xb = 0; xb < w; xb += 32) {
      unsigned bits = __ballot_sync(0xffffffffu, xb + lane < w && row_a[xb + lane] == 0);
      while (bits) {
        const int x = xb + __ffs(bits) - 1;
        bits &= bits - 1;
        for (int r = 0; r < R; ++r) {
          if (!s_has[r]) continue;
          const long long d2 = nearest_d2(P.g_region + r * n + (long long)y * w, w, x, lane);
          if (lane == 0) add_query(P, s_bins[r][0], &s_max[r][0], s_sum[warp][r][0], d2);
        }
      }
    }
    // every dB_r pixel against the plane
    for (int r = 0; r < R; ++r) {
      if (!s_has[r]) continue;
      const int* row_b = P.g_region + r * n + (long long)y * w;
      for (int xb = 0; xb < w; xb += 32) {
        unsigned bits = __ballot_sync(0xffffffffu, xb + lane < w && row_b[xb + lane] == 0);
        while (bits) {
          const int x = xb + __ffs(bits) - 1;
          bits &= bits - 1;
          const long long d2 = nearest_d2(row_a, w, x, lane);
          if (lane == 0) add_query(P, s_bins[r][1], &s_max[r][1], s_sum[warp][r][1], d2);
        }
      }
    }
  }
  __syncthreads();
  char* part = P.partials + ((long long)plane * P.tiles + tile) * kBoundaryTileBytes;
  int* p_bins = reinterpret_cast<int*>(part);
  unsigned long long* p_max = reinterpret_cast<unsigned long long*>(part + kBinBytes);
  double* p_sum = reinterpret_cast<double*>(part + kBinBytes + kMaxBytes);
  for (int i = t; i < R * 2 * kBoundaryMaxTolerances; i += blockDim.x)
    if ((i & (kBoundaryMaxTolerances - 1)) < T) p_bins[i] = (&s_bins[0][0][0])[i];
  for (int i = t; i < R * 2; i += blockDim.x) {
    p_max[i] = (&s_max[0][0])[i];
    double s = (&s_sum[0][0][0])[i];
    for (int v = 1; v < kQueryWarps; ++v) s += (&s_sum[v][0][0])[i];
    p_sum[i] = s;
  }
}

// one thread per (plane, region, direction): the tiles' partials in tile order
__global__ void __launch_bounds__(256) boundary_reduce_kernel(const __grid_constant__ BoundaryPlanes P) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int R = P.n_regions, T = P.n_tolerances;
  if (idx >= (long long)P.planes * R * 2) return;
  const int dir = (int)(idx & 1), r = (int)((idx >> 1) % R), plane = (int)((idx >> 1) / R);
  const int ml = plane / P.n_words_round, wl = plane - ml * P.n_words_round;
  const long long mi = P.map0 + ml, wi = P.w0 + wl, W = P.n_words;
  const int n_a = P.word_boundary[mi * W + wi], n_b = P.region_boundary[r];
  const char* part = P.partials + (long long)plane * P.tiles * kBoundaryTileBytes;
  const int slot = r * 2 + dir;
  int* hits = dir ? P.region_hits : P.word_hits;
  int acc = 0;
  for (int k = 0; k < T; ++k) {
    for (int tile = 0; tile < P.tiles; ++tile)
      acc += reinterpret_cast<const int*>(part + (long long)tile * kBoundaryTileBytes)[slot * kBoundaryMaxTolerances + k];
    hits[((mi * T + k) * R + r) * W + wi] = acc;
  }
  unsigned long long mx = 0ull;
  double s = 0.0;
  for (int tile = 0; tile < P.tiles; ++tile) {
    const char* p = part + (long long)tile * kBoundaryTileBytes;
    mx = max(mx, reinterpret_cast<const unsigned long long*>(p + kBinBytes)[slot]);
    s += reinterpret_cast<const double*>(p + kBinBytes + kMaxBytes)[slot];
  }
  const long long o = ((mi * R + r) * W + wi) * 2 + dir;
  const bool empty = n_a == 0 || n_b == 0;
  P.max_d2[o] = empty ? -1 : (long long)mx;
  P.sum_dist[o] = empty ? 0.0 : s;
}

template <class In>
int launch_columns(const In& in, int planes, int h, int w, int* g, int* count, int per_map, int map_stride,
                   cudaStream_t stream) {
  boundary_columns_kernel<<<dim3((w + kColumnThreads - 1) / kColumnThreads, planes), kColumnThreads, 0, stream>>>(
      in, h, w, g, count, per_map, map_stride);
  DAAM_CUDA_TRY(cudaGetLastError());
  count_launch();
  return DAAM_OK;
}

}  // namespace

long long boundary_call_bytes(int n_regions, int h, int w) { return DAAM_BOUNDARY_CALL_BYTES(n_regions, h, w); }
long long boundary_plane_bytes(int h, int w) { return DAAM_BOUNDARY_PLANE_BYTES(h, w); }

int boundary_check_tolerances(const char* name, const float* tolerances, int n_tolerances, BoundaryPlanes& p) {
  for (int k = 0; k < n_tolerances; ++k) {
    if (!isfinite(tolerances[k]) || !(tolerances[k] >= 0.f)) { set_error("%s: tolerance %d is not finite and >= 0", name, k); return DAAM_E_INVALID; }
    if (k > 0 && !(tolerances[k] > tolerances[k - 1])) { set_error("%s: tolerances %d and %d are not strictly ascending", name, k - 1, k); return DAAM_E_INVALID; }
    p.tol2[k] = (double)tolerances[k] * (double)tolerances[k];
  }
  p.n_tolerances = n_tolerances;
  return DAAM_OK;
}

int boundary_check_scratch(const char* name, const void* scratch, long long scratch_bytes, int n_regions, int h, int w) {
  if ((uintptr_t)scratch & 7) { set_error("%s: scratch must be 8-byte aligned", name); return DAAM_E_INVALID; }
  const long long need = boundary_call_bytes(n_regions, h, w) + boundary_plane_bytes(h, w);
  if (scratch_bytes < need) { set_error("%s: %lld scratch bytes < %lld, the regions and one %d x %d plane", name, scratch_bytes, need, h, w); return DAAM_E_INVALID; }
  return DAAM_OK;
}

void boundary_planes_in(void* scratch, int n_regions, int planes, int h, int w, BoundaryPlanes& p) {
  const long long n = (long long)h * w;
  p.tile_rows = (int)DAAM_BOUNDARY_TILE_ROWS(w);
  p.tiles = (h + p.tile_rows - 1) / p.tile_rows;
  char* c = static_cast<char*>(scratch);             // the 8-byte arrays first
  p.g_region = reinterpret_cast<int*>(c); c += boundary_call_bytes(n_regions, h, w);
  p.partials = c; c += (long long)planes * p.tiles * kBoundaryTileBytes;
  p.pre = reinterpret_cast<float*>(c); c += 4 * planes * n;
  p.g_plane = reinterpret_cast<int*>(c); c += 4 * planes * n;
  p.minmax = reinterpret_cast<float*>(c);
  p.planes = planes; p.h = h; p.w = w; p.n_regions = n_regions;
}

int launch_boundary_regions(const unsigned char* regions, const BoundaryPlanes& p, int n_maps, cudaStream_t stream) {
  DAAM_CUDA_TRY(cudaMemsetAsync(p.word_boundary, 0, (size_t)n_maps * p.n_words * sizeof(int), stream));
  DAAM_CUDA_TRY(cudaMemsetAsync(p.region_boundary, 0, (size_t)p.n_regions * sizeof(int), stream));
  return launch_columns(MaskIn{regions}, p.n_regions, p.h, p.w, p.g_region, p.region_boundary, 1, 1, stream);
}

int launch_boundary_round(const BoundaryPlanes& p, float threshold, const unsigned char* masks, cudaStream_t stream) {
  int* count = p.word_boundary + (long long)p.map0 * p.n_words + p.w0;
  if (int rc = masks ? launch_columns(MaskIn{masks}, p.planes, p.h, p.w, p.g_plane, count, p.n_words_round, p.n_words, stream)
                     : launch_columns(ValueIn{p.pre, threshold}, p.planes, p.h, p.w, p.g_plane, count,
                                      p.n_words_round, p.n_words, stream)) return rc;
  boundary_query_kernel<<<dim3(p.tiles, p.planes), kQueryWarps * 32, 0, stream>>>(p);
  DAAM_CUDA_TRY(cudaGetLastError());
  count_launch();
  const long long outs = (long long)p.planes * p.n_regions * 2;
  boundary_reduce_kernel<<<(unsigned)((outs + 255) / 256), 256, 0, stream>>>(p);
  DAAM_CUDA_TRY(cudaGetLastError());
  count_launch();
  return DAAM_OK;
}

}  // namespace daam

using namespace daam;

extern "C" int daam_mask_boundary(const uint8_t* masks, int32_t n_planes, int32_t out_h, int32_t out_w,
                                  const uint8_t* regions, int32_t n_regions, const float* tolerances,
                                  int32_t n_tolerances, int32_t* word_boundary, int32_t* region_boundary,
                                  int32_t* word_hits, int32_t* region_hits, int64_t* max_d2, double* sum_dist,
                                  void* scratch, int64_t scratch_bytes, void* stream_) {
  const char* name = "daam_mask_boundary";
  if (!masks || !regions || !tolerances || !word_boundary || !region_boundary || !word_hits || !region_hits ||
      !max_d2 || !sum_dist || !scratch || n_planes <= 0 || out_h <= 0 || out_w <= 0 || n_regions <= 0 ||
      n_tolerances <= 0) { set_error("%s: null pointer or non-positive size", name); return DAAM_E_INVALID; }
  if (n_tolerances > kBoundaryMaxTolerances) { set_error("%s: %d tolerances > %d", name, n_tolerances, kBoundaryMaxTolerances); return DAAM_E_UNSUPPORTED; }
  if (n_regions > DAAM_REGION_MAX_REGIONS) { set_error("%s: %d regions > %d", name, n_regions, DAAM_REGION_MAX_REGIONS); return DAAM_E_UNSUPPORTED; }
  if ((long long)out_h * out_w > (1LL << 24)) { set_error("%s: a %d x %d output is more than 2^24 pixels", name, out_h, out_w); return DAAM_E_UNSUPPORTED; }
  BoundaryPlanes c;
  if (int rc = boundary_check_tolerances(name, tolerances, n_tolerances, c)) return rc;
  if (int rc = boundary_check_scratch(name, scratch, scratch_bytes, n_regions, out_h, out_w)) return rc;
  const cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  c.word_boundary = word_boundary; c.region_boundary = region_boundary; c.word_hits = word_hits;
  c.region_hits = region_hits; c.max_d2 = reinterpret_cast<long long*>(max_d2); c.sum_dist = sum_dist;
  c.n_words = 1; c.n_words_round = 1; c.w0 = 0;
  boundary_planes_in(scratch, n_regions, 1, out_h, out_w, c);
  if (int rc = launch_boundary_regions(regions, c, n_planes, stream)) return rc;
  const long long n = (long long)out_h * out_w;
  const int cap = (int)std::min<long long>(
      (scratch_bytes - boundary_call_bytes(n_regions, out_h, out_w)) / boundary_plane_bytes(out_h, out_w), 65535);
  for (int p0 = 0; p0 < n_planes; p0 += cap) {
    boundary_planes_in(scratch, n_regions, std::min(cap, n_planes - p0), out_h, out_w, c);
    c.map0 = p0;
    if (int rc = launch_boundary_round(c, 0.f, masks + p0 * n, stream)) return rc;
  }
  return DAAM_OK;
}
