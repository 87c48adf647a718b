// Word distance maps: per plane (one (map, word) pair, or one mask) the exact signed squared Euclidean distance
// transform of its mask M (daam_word_distance, daam_mask_distance): d2 from each pixel outside M to the nearest pixel
// of M, and minus d2 from each pixel of M to the nearest pixel outside M. With g(y, x') the vertical distance from
// (y, x') to the nearest pixel of the other class in column x' (0 when (y, x') is of the other class itself),
//   d2(y, x) = min_x' (x - x')^2 + g(y, x')^2,
// the lower envelope of one parabola per column, evaluated along the row (Felzenszwalb and Huttenlocher, "Distance
// Transforms of Sampled Functions", Theory of Computing 2012). Two launches over the planes, O(h * w) work each:
//  - distance_columns_kernel: one thread per column, coalesced across columns. A down sweep and an up sweep give each
//    pixel its g to the other class, written to signed_d2 as +g outside M and -g inside it; kColumnNone marks a
//    column without a pixel of the other class. g is never 0, so the sign is the pixel's class;
//  - distance_rows_kernel: a CTA stages kRowsPerCta rows of g as int16 in shared memory, coalesced, then one thread
//    per row builds the envelope of each class in turn (a stack of sites in shared memory) and writes the row's
//    signed_d2 in place. For the outside pixels a pixel of M is a site of height 0 and an outside pixel one of height
//    g^2; likewise the other way. Every intersection is compared as an exact fraction in 64-bit integers.
// Integer arithmetic only: the results are the same bits on every call and whatever the split of the planes into
// rounds.
#include <math.h>

#include <algorithm>
#include <mutex>

#include "distance.cuh"
#include "word_value.cuh"

namespace daam {
namespace {

constexpr int kColumnNone = 32767;                  // |g| where the column has no pixel of the other class
constexpr int kColumnThreads = 128;
constexpr int kRowThreads = 32;                     // one warp per CTA: it stages the rows, then a thread per row
constexpr int kRowSmem = 48 * 1024;                 // rows per CTA: as many as fit, at most kRowThreads
constexpr int kMaxRowSmem = 4 * kDistanceMaxSide;   // one row of the widest plane: its g and its stack, int16 each
static_assert(kColumnNone == kDistanceMaxSide && kColumnNone <= 32767, "g and the column of a site fit an int16");

struct MaskIn {
  const unsigned char* m;
  __device__ __forceinline__ bool at(long long i) const { return m[i] != 0; }
};
struct ValueIn {
  const float* m;
  float threshold;
  __device__ __forceinline__ bool at(long long i) const { return m[i] > threshold; }
};

// grid: (ceil(w / kColumnThreads), planes): one thread per column of a plane
template <class In>
__global__ void __launch_bounds__(kColumnThreads) distance_columns_kernel(const In in, int h, int w,
                                                                          int* __restrict__ d) {
  const int x = blockIdx.x * kColumnThreads + threadIdx.x;
  if (x >= w) return;
  const long long base = blockIdx.y * (long long)h * w + x;
  // down: the distance to the other class above; a row of -kColumnNone - 1 is "none yet", clamped to kColumnNone
  int last_in = -kColumnNone - 1, last_out = -kColumnNone - 1;
#pragma unroll 4
  for (int y = 0; y < h; ++y) {
    const long long i = base + (long long)y * w;
    if (in.at(i)) { d[i] = -min(y - last_out, kColumnNone); last_in = y; }
    else          { d[i] = min(y - last_in, kColumnNone); last_out = y; }
  }
  // up: the distance to the other class below, if nearer
  int next_in = h + kColumnNone, next_out = h + kColumnNone;
#pragma unroll 4
  for (int y = h - 1; y >= 0; --y) {
    const long long i = base + (long long)y * w;
    const int v = d[i];
    if (v < 0) { d[i] = -min(-v, next_out - y); next_in = y; }
    else       { d[i] = min(v, next_in - y); next_out = y; }
  }
}

// F(x) = f(x) + x^2 of the site in column x, for the pixels of class `cls` (+1 outside, -1 inside): f = 0 where the
// pixel is of the other class, g^2 where it is of class cls. `c` is the staged signed g.
__device__ __forceinline__ long long site_F(int c, int x, int cls) {
  const long long g = c * cls > 0 ? c : 0;
  return g * g + (long long)x * x;
}

// One row, one class: every pixel of class cls gets cls * min_x' (x - x')^2 + f(x'). `row` and `v` step by R (the
// rows of the CTA are interleaved); `v` holds up to w sites.
__device__ __forceinline__ void row_envelope(const short* __restrict__ row, short* __restrict__ v, int R, int w,
                                             int cls, int* __restrict__ out) {
  int k = -1;                                         // the top of the stack of sites
  long long Fk = 0;                                   // F(v[k])
  bool any = false;                                   // the row has a pixel of class cls
  for (int q = 0; q < w; ++q) {
    const int c = row[q * R], g = c * cls;
    any |= g > 0;
    if (g == kColumnNone) continue;                   // no pixel of the other class in column q: no site
    const long long Fq = site_F(c, q, cls);
    // pop v[k] while q's parabola meets it at or left of where v[k] starts: (Fq - Fk) / 2(q - p) <= (Fk - Fpp) /
    // 2(p - pp), cross-multiplied (both denominators > 0)
    while (k > 0) {
      const int p = v[k * R], pp = v[(k - 1) * R];
      const long long Fpp = site_F(row[pp * R], pp, cls);
      if ((Fq - Fk) * (p - pp) > (Fk - Fpp) * (q - p)) break;
      --k;
      Fk = Fpp;
    }
    v[++k * R] = (short)q;
    Fk = Fq;
  }
  if (!any) return;
  if (k < 0) {                                        // the other class is empty: the whole image is class cls
    for (int x = 0; x < w; ++x) out[x] = cls * DAAM_DISTANCE_NONE;
    return;
  }
  int j = 0, vj = v[0], vn = 0;
  long long Fj = site_F(row[vj * R], vj, cls), Fn = 0;
  if (k > 0) { vn = v[R]; Fn = site_F(row[vn * R], vn, cls); }
  for (int x = 0; x < w; ++x) {
    // move to the next parabola while it starts left of x: (Fn - Fj) / 2(vn - vj) < x
    while (j < k && Fn - Fj < 2LL * x * (vn - vj)) {
      ++j; vj = vn; Fj = Fn;
      if (j < k) { vn = v[(j + 1) * R]; Fn = site_F(row[vn * R], vn, cls); }
    }
    if (row[x * R] * cls > 0) {
      const long long dx = x - vj;
      out[x] = cls * (int)(dx * dx + Fj - (long long)vj * vj);
    }
  }
}

// grid: (ceil(h / R), planes), kRowThreads threads; dynamic smem: R rows of staged g and R stacks, int16, element x of
// row r at [x * R + r]
__global__ void __launch_bounds__(kRowThreads) distance_rows_kernel(int* __restrict__ d, int h, int w, int R) {
  extern __shared__ short s_rows[];
  short* s_stack = s_rows + (long long)R * w;
  const int y0 = blockIdx.x * R, nr = min(R, h - y0);
  int* rows = d + (blockIdx.y * (long long)h + y0) * w;
  for (int i = threadIdx.x; i < nr * w; i += kRowThreads) {
    const int r = i / w, x = i - r * w;
    s_rows[x * R + r] = (short)rows[i];
  }
  __syncthreads();
  const int r = threadIdx.x;
  if (r >= nr) return;
  int* out = rows + (long long)r * w;
  row_envelope(s_rows + r, s_stack + r, R, w, 1, out);    // outside pixels: d2 to M
  row_envelope(s_rows + r, s_stack + r, R, w, -1, out);   // pixels of M: -d2 to the outside
}

int rows_per_cta(int w) { return std::max(1, std::min(kRowThreads, kRowSmem / (4 * w))); }

template <class In>
int launch_planes(const In& in, int planes, int h, int w, int* d, cudaStream_t stream) {
  distance_columns_kernel<<<dim3((w + kColumnThreads - 1) / kColumnThreads, planes), kColumnThreads, 0, stream>>>(
      in, h, w, d);
  DAAM_CUDA_TRY(cudaGetLastError());
  count_launch();
  const int R = rows_per_cta(w);
  const size_t smem = 4 * (size_t)R * w;
  if (smem > 48 * 1024) {
    static std::once_flag attr_once[64];
    int device = 0;
    DAAM_CUDA_TRY(cudaGetDevice(&device));
    cudaError_t attr_err = cudaSuccess;
    std::call_once(attr_once[device & 63], [&] {
      attr_err = cudaFuncSetAttribute(distance_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxRowSmem);
    });
    DAAM_CUDA_TRY(attr_err);
  }
  distance_rows_kernel<<<dim3((h + R - 1) / R, planes), kRowThreads, smem, stream>>>(d, h, w, R);
  DAAM_CUDA_TRY(cudaGetLastError());
  count_launch();
  return DAAM_OK;
}

}  // namespace

long long distance_plane_bytes(int h, int w) { return DAAM_DISTANCE_PLANE_BYTES(h, w); }
static_assert(DAAM_DISTANCE_PLANE_BYTES(0, 0) == kWordPartialFloats * sizeof(float),
              "DAAM_DISTANCE_PLANE_BYTES counts one plane's min / max partials");

int distance_check_scratch(const char* name, const void* scratch, long long scratch_bytes, int h, int w) {
  if ((uintptr_t)scratch & 3) { set_error("%s: scratch must be 4-byte aligned", name); return DAAM_E_INVALID; }
  const long long need = distance_plane_bytes(h, w);
  if (scratch_bytes < need) { set_error("%s: %lld scratch bytes < %lld, one %d x %d plane", name, scratch_bytes, need, h, w); return DAAM_E_INVALID; }
  return DAAM_OK;
}

void distance_planes_in(void* scratch, int planes, int h, int w, DistancePlanes& p) {
  p.pre = static_cast<float*>(scratch);
  p.minmax = p.pre + (long long)planes * h * w;
}

int launch_distance(const float* pre, float threshold, const unsigned char* masks, int planes, int h, int w,
                    int* signed_d2, cudaStream_t stream) {
  const long long n = (long long)h * w;
  for (int p0 = 0; p0 < planes; p0 += 65535) {
    const int np = std::min(65535, planes - p0);
    if (int rc = masks ? launch_planes(MaskIn{masks + p0 * n}, np, h, w, signed_d2 + p0 * n, stream)
                       : launch_planes(ValueIn{pre + p0 * n, threshold}, np, h, w, signed_d2 + p0 * n, stream))
      return rc;
  }
  return DAAM_OK;
}

}  // namespace daam

using namespace daam;

extern "C" int daam_mask_distance(const uint8_t* masks, int32_t n_planes, int32_t out_h, int32_t out_w,
                                  int32_t* signed_d2, void* stream_) {
  const char* name = "daam_mask_distance";
  if (!masks || !signed_d2 || n_planes <= 0 || out_h <= 0 || out_w <= 0) { set_error("%s: null pointer or non-positive size", name); return DAAM_E_INVALID; }
  if (out_h > kDistanceMaxSide || out_w > kDistanceMaxSide) { set_error("%s: a %d x %d output has a side > %d", name, out_h, out_w, kDistanceMaxSide); return DAAM_E_UNSUPPORTED; }
  if ((long long)out_h * out_w > (1LL << 24)) { set_error("%s: a %d x %d output is more than 2^24 pixels", name, out_h, out_w); return DAAM_E_UNSUPPORTED; }
  return launch_distance(nullptr, 0.f, masks, n_planes, out_h, out_w, signed_d2, static_cast<cudaStream_t>(stream_));
}
