// Word instances: the 8-connected components of the mask pre > threshold of every plane (one (map, word) pair), with
// each component's area, box, index sums and peak, and the K largest per plane (daam_word_instances; words.cu's
// instance_mask_kernel writes `pre`). Five launches over the planes of a round:
//  1. cc_local_kernel: each 32 x 32 tile is labelled in shared memory by union-find; every foreground pixel's label
//     is the tile-local component's first pixel (its smallest raster index);
//  2. cc_seam_kernel: the pixels on tile edges unite, in global memory, with their neighbours in other tiles (the
//     diagonal ones across tile corners included);
//  3. cc_flatten_kernel: every pixel's label becomes its root by pointer jumping; a root opens its component's slot
//     and appends itself to the plane's root list;
//  4. cc_stats_kernel: area, box, index sums and peak per component with integer atomics;
//  5. cc_select_kernel: the K largest components per plane by (area desc, first pixel asc), by radix select.
// Union (Playne & Hawick): the larger of two roots is hooked under the smaller with atomicMin, so a label never
// increases and every root is the smallest raster index of its tree: after the flatten, a component's label is its
// first pixel. Every statistic is an integer sum, min or max, and the peak a 64-bit max of (orderable fp32 bits of
// pre, 0xFFFFFFFF - pixel), which keeps the first pixel of a tie: the results do not depend on the order the atomics
// land in, nor on how planes are split into rounds.
#include <limits.h>

#include "components.cuh"
#include "word_value.cuh"

namespace daam {
namespace {

constexpr int kCcTile = 32;                          // labelling tile: 32 x 32 pixels, a thread each
constexpr int kCcStatsPix = 8;                       // consecutive pixels per cc_stats_kernel thread
constexpr int kCcSelectThreads = 1024;

__device__ __forceinline__ int slot_of(int p, int w) {
  const int y = p / w, x = p - y * w;
  return (y >> 1) * ((w + 1) >> 1) + (x >> 1);
}

// The root of p's tree. Path splitting on the way: each node passed is pointed at its grandparent with atomicMin, so
// a label still never increases and trees stay shallow while many threads unite at once.
__device__ __forceinline__ int find_root(volatile int* L, int p) {
  int q = L[p];
  while (q != p) {
    const int r = L[q];
    if (r != q) atomicMin(const_cast<int*>(L + p), r);
    p = q;
    q = r;
  }
  return p;
}

// the trees of a and b become one: the larger root is hooked under the smaller
__device__ void unite(volatile int* L, int a, int b) {
  while (true) {
    a = find_root(L, a);
    b = find_root(L, b);
    if (a == b) return;
    if (a > b) { const int t = a; a = b; b = t; }
    const int old = atomicMin(const_cast<int*>(L + b), a);
    if (old == b) return;                             // b was still a root: hooked
    b = old;                                          // b was hooked meanwhile: unite a with its new parent
  }
}

// fp32 bits whose unsigned order is the float order (-0 taken as +0)
__device__ __forceinline__ unsigned orderable(float f) {
  const unsigned u = f == 0.f ? 0u : __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : u | 0x80000000u;
}

__device__ __forceinline__ float from_orderable(unsigned u) {
  return __uint_as_float((u & 0x80000000u) ? u & 0x7fffffffu : ~u);
}

// grid: (tiles, planes), 1024 threads: thread (ly, lx) of the tile's 32 x 32 pixels
__global__ void __launch_bounds__(1024) cc_local_kernel(const __grid_constant__ InstancePlanes P) {
  __shared__ int L[kCcTile * kCcTile];
  const int plane = blockIdx.y, h = P.h, w = P.w, t = threadIdx.x;
  const int tiles_x = (w + kCcTile - 1) / kCcTile;
  const int ty0 = (blockIdx.x / tiles_x) * kCcTile, tx0 = (blockIdx.x % tiles_x) * kCcTile;
  const int ly = t / kCcTile, lx = t % kCcTile, y = ty0 + ly, x = tx0 + lx;
  const long long base = (long long)plane * h * w;
  const bool fg = y < h && x < w && P.pre[base + (long long)y * w + x] > P.threshold;
  L[t] = fg ? t : -1;
  if (blockIdx.x == 0 && t == 0) P.n_roots[plane] = 0;
  __syncthreads();
  if (fg) {                                           // the neighbours before the pixel in raster order: W, NW, N, NE
    if (lx > 0 && L[t - 1] >= 0) unite(L, t, t - 1);
    if (ly > 0) {
      if (lx > 0 && L[t - kCcTile - 1] >= 0) unite(L, t, t - kCcTile - 1);
      if (L[t - kCcTile] >= 0) unite(L, t, t - kCcTile);
      if (lx < kCcTile - 1 && L[t - kCcTile + 1] >= 0) unite(L, t, t - kCcTile + 1);
    }
  }
  __syncthreads();
  if (y < h && x < w) {
    const int r = fg ? find_root(L, t) : 0;
    P.label[base + (long long)y * w + x] = fg ? (ty0 + r / kCcTile) * w + tx0 + r % kCcTile : -1;
  }
}

// grid: (tiles, planes), 96 threads: the tile's top row, left column and right column. Each edge pixel unites with
// its W, NW, N and NE neighbours that lie in another tile; every 8-adjacent pair across tiles is one of those.
__global__ void __launch_bounds__(96) cc_seam_kernel(const __grid_constant__ InstancePlanes P) {
  const int plane = blockIdx.y, h = P.h, w = P.w, t = threadIdx.x;
  const int tiles_x = (w + kCcTile - 1) / kCcTile;
  const int ty0 = (blockIdx.x / tiles_x) * kCcTile, tx0 = (blockIdx.x % tiles_x) * kCcTile;
  int y, x;
  if (t < kCcTile) { y = ty0; x = tx0 + t; }
  else if (t < 2 * kCcTile) { y = ty0 + t - kCcTile; x = tx0; }
  else { y = ty0 + t - 2 * kCcTile; x = tx0 + kCcTile - 1; }
  if (y >= h || x >= w) return;
  int* L = P.label + (long long)plane * h * w;
  const int p = y * w + x;
  if (L[p] < 0) return;
  const int dy[4] = {0, -1, -1, -1}, dx[4] = {-1, -1, 0, 1};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int qy = y + dy[j], qx = x + dx[j];
    if (qy < 0 || qx < 0 || qx >= w) continue;
    if (qy / kCcTile == y / kCcTile && qx / kCcTile == x / kCcTile) continue;   // same tile: cc_local_kernel's
    const int q = qy * w + qx;
    if (L[q] >= 0) unite(L, p, q);
  }
}

// grid: (ceil(h w / 256), planes)
__global__ void __launch_bounds__(256) cc_flatten_kernel(const __grid_constant__ InstancePlanes P) {
  const int plane = blockIdx.y, w = P.w, n = P.h * P.w;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= n) return;
  int* L = P.label + (long long)plane * n;
  if (L[p] < 0) return;
  const int r = find_root(L, p);
  L[p] = r;                                           // a root: every walk through p still ends there
  if (r == p) {
    const long long s = (long long)plane * (((P.h + 1) >> 1) * ((w + 1) >> 1)) + slot_of(p, w);
    P.area[s] = 0;
    P.box[4 * s] = INT_MAX; P.box[4 * s + 1] = INT_MAX; P.box[4 * s + 2] = -1; P.box[4 * s + 3] = -1;
    P.sums[2 * s] = 0; P.sums[2 * s + 1] = 0;
    P.peak[s] = 0;
    P.roots[(long long)plane * (((P.h + 1) >> 1) * ((w + 1) >> 1)) + atomicAdd(P.n_roots + plane, 1)] = p;
  }
}

// One thread's running statistics of a component over its pixels
struct Agg {
  int root, n, y0, x0, y1, x1;
  unsigned long long sy, sx, peak;
};

__device__ __forceinline__ void agg_flush(const InstancePlanes& P, long long slot_base, const Agg& a) {
  const long long s = slot_base + slot_of(a.root, P.w);
  atomicAdd(P.area + s, a.n);
  atomicMin(P.box + 4 * s, a.y0); atomicMin(P.box + 4 * s + 1, a.x0);
  atomicMax(P.box + 4 * s + 2, a.y1); atomicMax(P.box + 4 * s + 3, a.x1);
  atomicAdd(P.sums + 2 * s, a.sy); atomicAdd(P.sums + 2 * s + 1, a.sx);
  atomicMax(P.peak + s, a.peak);
}

// grid: (ceil(h w / 2048), planes), 256 threads: each thread kCcStatsPix consecutive pixels. A thread folds a run of
// one component into registers and flushes it with atomics when the component changes; the last runs of a warp are
// reduced per component across the warp first, so a component that covers the warp's pixels costs one set of atomics.
__global__ void __launch_bounds__(256) cc_stats_kernel(const __grid_constant__ InstancePlanes P) {
  const int plane = blockIdx.y, w = P.w, n = P.h * P.w;
  const long long base = (long long)plane * n;
  const long long slot_base = (long long)plane * (((P.h + 1) >> 1) * ((w + 1) >> 1));
  const int* L = P.label + base;
  const float* pre = P.pre + base;
  Agg a = {-1, 0, 0, 0, 0, 0, 0ull, 0ull, 0ull};
  const long long p0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * kCcStatsPix;
  for (int j = 0; j < kCcStatsPix; ++j) {
    const long long pl = p0 + j;
    if (pl >= n) break;
    const int p = (int)pl, r = L[p];
    if (r < 0) continue;
    const int y = p / w, x = p - y * w;
    const unsigned long long key = (unsigned long long)orderable(pre[p]) << 32 | (0xffffffffu - (unsigned)p);
    if (r != a.root) {
      if (a.root >= 0) agg_flush(P, slot_base, a);
      a = {r, 1, y, x, y, x, (unsigned long long)y, (unsigned long long)x, key};
    } else {
      ++a.n;
      a.y0 = min(a.y0, y); a.x0 = min(a.x0, x); a.y1 = max(a.y1, y); a.x1 = max(a.x1, x);
      a.sy += y; a.sx += x;
      a.peak = max(a.peak, key);
    }
  }
  const int lane = threadIdx.x & 31;
  unsigned pending = __ballot_sync(0xffffffffu, a.root >= 0);
  while (pending) {
    const int leader = __ffs(pending) - 1;
    const int root = __shfl_sync(0xffffffffu, a.root, leader);
    const bool mine = a.root == root;
    pending &= ~__ballot_sync(0xffffffffu, mine);
    Agg g;
    g.root = root;
    g.n = (int)__reduce_add_sync(0xffffffffu, mine ? (unsigned)a.n : 0u);
    g.y0 = (int)__reduce_min_sync(0xffffffffu, mine ? (unsigned)a.y0 : 0xffffffffu);
    g.x0 = (int)__reduce_min_sync(0xffffffffu, mine ? (unsigned)a.x0 : 0xffffffffu);
    g.y1 = (int)__reduce_max_sync(0xffffffffu, mine ? (unsigned)a.y1 : 0u);
    g.x1 = (int)__reduce_max_sync(0xffffffffu, mine ? (unsigned)a.x1 : 0u);
    g.sy = mine ? a.sy : 0ull; g.sx = mine ? a.sx : 0ull; g.peak = mine ? a.peak : 0ull;
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
      g.sy += __shfl_xor_sync(0xffffffffu, g.sy, s);
      g.sx += __shfl_xor_sync(0xffffffffu, g.sx, s);
      g.peak = max(g.peak, __shfl_xor_sync(0xffffffffu, g.peak, s));
    }
    if (lane == leader) agg_flush(P, slot_base, g);
  }
}

// grid: planes, kCcSelectThreads threads. The key of a component, (area << 32 | 0xFFFFFFFF - first pixel), is unique
// and orders the instances; the K-th largest key is found one byte at a time (radix select: a histogram of the byte
// over the keys that match the bytes found so far), then the at most K keys not below it are ranked in shared memory.
__global__ void __launch_bounds__(kCcSelectThreads) cc_select_kernel(const __grid_constant__ InstancePlanes P) {
  __shared__ unsigned hist[256];
  __shared__ unsigned long long s_prefix, sel[kMaxInstances];
  __shared__ int s_rank, s_m;
  const int plane = blockIdx.x, w = P.w, K = P.k, t = threadIdx.x;
  const long long slot_base = (long long)plane * (((P.h + 1) >> 1) * ((w + 1) >> 1));
  const int* roots = P.roots + slot_base;
  const int n = P.n_roots[plane];
  auto key_of = [&](int i) {
    const int p = roots[i];
    return (unsigned long long)(unsigned)P.area[slot_base + slot_of(p, w)] << 32 | (0xffffffffu - (unsigned)p);
  };
  unsigned long long prefix = 0;
  if (n > K) {
    unsigned long long mask = 0;
    int rank = K;                                     // the rank of the wanted key among those matching `prefix`
    for (int shift = 56; shift >= 0; shift -= 8) {
      for (int i = t; i < 256; i += blockDim.x) hist[i] = 0;
      __syncthreads();
      for (int i = t; i < n; i += blockDim.x) {
        const unsigned long long key = key_of(i);
        if ((key & mask) == prefix) atomicAdd(hist + ((key >> shift) & 255), 1u);
      }
      __syncthreads();
      if (t == 0) {
        int above = 0;
        for (int d = 255; d >= 0; --d) {
          if (above + (int)hist[d] >= rank) { s_prefix = prefix | (unsigned long long)d << shift; s_rank = rank - above; break; }
          above += hist[d];
        }
      }
      __syncthreads();
      prefix = s_prefix; rank = s_rank; mask |= 0xffull << shift;
    }
  }
  if (t == 0) s_m = 0;
  __syncthreads();
  for (int i = t; i < n; i += blockDim.x) {           // the min(n, K) keys not below the K-th
    const unsigned long long key = key_of(i);
    if (key >= prefix) sel[atomicAdd(&s_m, 1)] = key;
  }
  __syncthreads();
  const int m = s_m;
  const long long out = (long long)plane * K;
  if (t == 0) P.count[plane] = n;
  if (t < m) {
    const unsigned long long key = sel[t];
    int r = 0;
    for (int j = 0; j < m; ++j) r += sel[j] > key;
    const int p = (int)(0xffffffffu - (unsigned)key);
    const long long s = slot_base + slot_of(p, w), o = out + r;
    const unsigned long long pk = P.peak[s];
    const int pp = (int)(0xffffffffu - (unsigned)pk);
    P.out_area[o] = P.area[s];
    P.out_box[4 * o] = P.box[4 * s]; P.out_box[4 * o + 1] = P.box[4 * s + 1];
    P.out_box[4 * o + 2] = P.box[4 * s + 2] + 1; P.out_box[4 * o + 3] = P.box[4 * s + 3] + 1;
    P.out_sum[2 * o] = (long long)P.sums[2 * s]; P.out_sum[2 * o + 1] = (long long)P.sums[2 * s + 1];
    P.out_peak[o] = from_orderable((unsigned)(pk >> 32));
    P.out_peak_yx[2 * o] = pp / w; P.out_peak_yx[2 * o + 1] = pp % w;
  } else if (t < K) {                                 // padding past the count
    const long long o = out + t;
    P.out_area[o] = 0;
    P.out_box[4 * o] = 0; P.out_box[4 * o + 1] = 0; P.out_box[4 * o + 2] = 0; P.out_box[4 * o + 3] = 0;
    P.out_sum[2 * o] = 0; P.out_sum[2 * o + 1] = 0;
    P.out_peak[o] = 0.f;
    P.out_peak_yx[2 * o] = 0; P.out_peak_yx[2 * o + 1] = 0;
  }
}

long long slots(int h, int w) { return (long long)((h + 1) / 2) * ((w + 1) / 2); }

}  // namespace

long long instance_plane_bytes(int h, int w) {
  return 8LL * h * w + 48 * slots(h, w) + 4 + kWordPartialFloats * sizeof(float);
}

void instance_planes_in(void* scratch, int planes, int h, int w, InstancePlanes& p) {
  const long long n = (long long)planes * h * w, s = planes * slots(h, w);
  char* c = static_cast<char*>(scratch);             // the 8-byte arrays first
  p.peak = reinterpret_cast<unsigned long long*>(c); c += 8 * s;
  p.sums = reinterpret_cast<unsigned long long*>(c); c += 16 * s;
  p.pre = reinterpret_cast<float*>(c); c += 4 * n;
  p.label = reinterpret_cast<int*>(c); c += 4 * n;
  p.area = reinterpret_cast<int*>(c); c += 4 * s;
  p.box = reinterpret_cast<int*>(c); c += 16 * s;
  p.roots = reinterpret_cast<int*>(c); c += 4 * s;
  p.n_roots = reinterpret_cast<int*>(c); c += 4LL * planes;
  p.minmax = reinterpret_cast<float*>(c);
  p.planes = planes; p.h = h; p.w = w;
}

int launch_components(const InstancePlanes& p, cudaStream_t stream) {
  const unsigned tiles = ((p.h + kCcTile - 1) / kCcTile) * ((p.w + kCcTile - 1) / kCcTile);
  const long long n = (long long)p.h * p.w;
  cc_local_kernel<<<dim3(tiles, p.planes), kCcTile * kCcTile, 0, stream>>>(p);
  DAAM_CUDA_TRY(cudaGetLastError());
  cc_seam_kernel<<<dim3(tiles, p.planes), 3 * kCcTile, 0, stream>>>(p);
  DAAM_CUDA_TRY(cudaGetLastError());
  cc_flatten_kernel<<<dim3((unsigned)((n + 255) / 256), p.planes), 256, 0, stream>>>(p);
  DAAM_CUDA_TRY(cudaGetLastError());
  cc_stats_kernel<<<dim3((unsigned)((n + 256 * kCcStatsPix - 1) / (256 * kCcStatsPix)), p.planes), 256, 0, stream>>>(p);
  DAAM_CUDA_TRY(cudaGetLastError());
  cc_select_kernel<<<p.planes, kCcSelectThreads, 0, stream>>>(p);
  DAAM_CUDA_TRY(cudaGetLastError());
  count_launch(5);
  return DAAM_OK;
}

}  // namespace daam
