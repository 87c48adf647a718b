// Edge-aware word maps (daam_refine_words): the guided filter of each plane's m (one (map, word) pair) with the
// map's image I = RGB / 255 as guide. With mean_f(x) the mean of f over the (2r+1)^2 window around x clipped to the
// image (border windows shrink), mu = mean(I), Sigma = mean(I I^T) - mu mu^T:
//   p = mean(m),  c = mean(I m) - mu p,  a = (Sigma + eps Id)^-1 c,  b = p - a . mu,  q = mean(a) . I + mean(b)
// Two launches per distinct image build its statistics, exact up to one rounding:
//  1. guide_row_kernel: per pixel, the integer window sums along the row of I_c and I_c I_d (bytes, so exact);
//  2. guide_col_kernel: the same along the column, then in int64 N S_cd - S_c S_d = N^2 255^2 Sigma_cd exactly, and
//     mu and the inverse of Sigma + eps Id in float64 (adjugate over determinant), stored as fp32.
// Four launches per round of planes, each a separable pass of direct window sums -- every output sums its at most
// 2r+1 staged inputs from 0 in ascending order, never a running sum, so the rounding does not depend on where the
// pixel is or how the work is cut:
//  3. refine_row_kernel<true>: m recomputed from the word map (the bits of expand_words), then the row sums of m and
//     I_c m;
//  4. refine_col_kernel<true>: their column sums, divided by the window's pixel count N, then a and b;
//  5. refine_row_kernel<false>: the row sums of a and b;
//  6. refine_col_kernel<false>: their column sums over N, then q (or q > threshold as 1 / 0) to the output.
// No atomics: the results are the same bits on every call and however the planes are split into rounds.
#include <math.h>

#include <mutex>

#include "bicubic.cuh"
#include "refine.cuh"
#include "word_value.cuh"

namespace daam {
namespace {

constexpr int kRowSeg = 256;                          // outputs of a row-pass CTA, one per thread
constexpr int kRowStage = kRowSeg + 2 * kRefineMaxRadius;
constexpr int kColW = 32, kColRows = 64;              // outputs of a column-pass CTA: 32 columns x 64 rows
constexpr int kColPer = 8;                            // rows per thread (8 row groups of 32 threads)
constexpr int kGuideRows = 8;                         // guide_col_kernel: 32 columns x 8 rows, one output per thread

__device__ __forceinline__ const unsigned char* plane_image(const RefinePlanes& P, int plane) {
  return P.image + (long long)(plane / P.words_per_map) * P.image_map_stride;
}

// grid: (row segments x rows, guides); thread x: S_r, S_g, S_b and the six S_cd over the row window, as integers
// (S_c <= 129 * 255 fits 16 bits: S_r and S_g share a word), into the 8 channels of plane g's buffer
__global__ void __launch_bounds__(256) guide_row_kernel(const __grid_constant__ RefinePlanes P) {
  __shared__ int px[3][kRowStage];
  const int ow = P.ow, r = P.radius, g = blockIdx.y;
  const int segs = (ow + kRowSeg - 1) / kRowSeg, y = blockIdx.x / segs, x0 = (blockIdx.x - y * segs) * kRowSeg;
  const int lo = max(0, x0 - r), hi = min(ow, x0 + kRowSeg + r);   // staged columns [lo, hi)
  const unsigned char* im = P.image + g * P.image_map_stride + ((long long)y * ow + lo) * 3;
  for (int i = threadIdx.x; i < 3 * (hi - lo); i += blockDim.x) px[i % 3][i / 3] = __ldg(im + i);
  __syncthreads();
  const int x = x0 + threadIdx.x;
  if (x >= ow) return;
  int s[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int k = max(0, x - r) - lo, k1 = min(ow - 1, x + r) - lo; k <= k1; ++k) {
    const int R = px[0][k], G = px[1][k], B = px[2][k];
    s[0] += R; s[1] += G; s[2] += B;
    s[3] += R * R; s[4] += R * G; s[5] += R * B; s[6] += G * G; s[7] += G * B; s[8] += B * B;
  }
  const long long n = (long long)P.oh * ow;
  unsigned* dst = reinterpret_cast<unsigned*>(P.buf) + (long long)g * 8 * n + (long long)y * ow + x;
  dst[0] = (unsigned)s[0] | ((unsigned)s[1] << 16);
#pragma unroll
  for (int j = 1; j < 8; ++j) dst[j * n] = (unsigned)s[j + 1];
}

// grid: (tiles of 32 x kGuideRows pixels, guides); thread (x, y): the column sums of guide_row_kernel's sums, then mu
// and (Sigma + eps Id)^-1 from exact integers. S_cd <= 129^2 * 255^2 < 2^31.
__global__ void __launch_bounds__(256) guide_col_kernel(const __grid_constant__ RefinePlanes P) {
  const int oh = P.oh, ow = P.ow, r = P.radius, g = blockIdx.y;
  const int tiles_x = (ow + kColW - 1) / kColW, tyi = blockIdx.x / tiles_x;
  const int x = (blockIdx.x - tyi * tiles_x) * kColW + (threadIdx.x & 31), y = tyi * kGuideRows + (threadIdx.x >> 5);
  if (x >= ow || y >= oh) return;
  const long long n = (long long)oh * ow;
  const unsigned* src = reinterpret_cast<const unsigned*>(P.buf) + (long long)g * 8 * n + x;
  const int y0 = max(0, y - r), y1 = min(oh - 1, y + r);
  int s[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int k = y0; k <= y1; ++k) {
    const unsigned* row = src + (long long)k * ow;
    const unsigned rg = __ldg(row);
    s[0] += (int)(rg & 0xffffu); s[1] += (int)(rg >> 16);
#pragma unroll
    for (int j = 1; j < 8; ++j) s[j + 1] += (int)__ldg(row + j * n);
  }
  const long long N = (long long)(min(ow - 1, x + r) - max(0, x - r) + 1) * (y1 - y0 + 1);
  // Sigma_cd = (N S_cd - S_c S_d) / (255 N)^2: an exact integer over an exact double, one rounding
  const double scale = 1.0 / (65025.0 * (double)(N * N));
  const long long S0 = s[0], S1 = s[1], S2 = s[2];
  const double e = (double)P.eps;
  const double a00 = (double)(N * s[3] - S0 * S0) * scale + e, a01 = (double)(N * s[4] - S0 * S1) * scale,
               a02 = (double)(N * s[5] - S0 * S2) * scale, a11 = (double)(N * s[6] - S1 * S1) * scale + e,
               a12 = (double)(N * s[7] - S1 * S2) * scale, a22 = (double)(N * s[8] - S2 * S2) * scale + e;
  const double c00 = a11 * a22 - a12 * a12, c01 = a02 * a12 - a01 * a22, c02 = a01 * a12 - a02 * a11;
  const double c11 = a00 * a22 - a02 * a02, c12 = a01 * a02 - a00 * a12, c22 = a00 * a11 - a01 * a01;
  const double inv_det = 1.0 / (a00 * c00 + a01 * c01 + a02 * c02);
  float* dst = P.guide + (long long)g * 9 * n + (long long)y * ow + x;
  const double mu_scale = 1.0 / (255.0 * (double)N);
  dst[0] = (float)(S0 * mu_scale); dst[n] = (float)(S1 * mu_scale); dst[2 * n] = (float)(S2 * mu_scale);
  dst[3 * n] = (float)(c00 * inv_det); dst[4 * n] = (float)(c01 * inv_det); dst[5 * n] = (float)(c02 * inv_det);
  dst[6 * n] = (float)(c11 * inv_det); dst[7 * n] = (float)(c12 * inv_det); dst[8 * n] = (float)(c22 * inv_det);
}

// grid: (row segments x rows, planes); thread x: the row window sums of four channels. kFirst: m and I_c m, from the
// word map; else a_r, a_g, a_b and b (buffer channels 4-7). To buffer channels 0-3.
template <bool kFirst>
__global__ void __launch_bounds__(256) refine_row_kernel(const __grid_constant__ RefinePlanes P) {
  __shared__ float st[4][kRowStage];
  __shared__ float s_lo, s_hi;
  const int ow = P.ow, r = P.radius, p = blockIdx.y;
  const int segs = (ow + kRowSeg - 1) / kRowSeg, y = blockIdx.x / segs, x0 = (blockIdx.x - y * segs) * kRowSeg;
  const int lo = max(0, x0 - r), hi = min(ow, x0 + kRowSeg + r);   // staged columns [lo, hi)
  const long long n = (long long)P.oh * ow, row = (long long)y * ow;
  float* buf = P.buf + (long long)p * 8 * n;
  if (kFirst) {
    // m = expand_words' m, from the word map and its min / max partials
    if (threadIdx.x == 0) {
      float vlo = 0.f, vhi = 0.f;
      if (!P.absolute) partial_bounds(P.minmax + 2LL * p * P.chunks, P.chunks, vlo, vhi);
      s_lo = vlo; s_hi = vhi;
    }
    __syncthreads();
    const float vlo = s_lo, vhi = s_hi;
    const float* wm = P.word_maps + (long long)p * P.mh * P.mw;
    const Taps ty = make_taps(y, P.mh, P.oh);
    const unsigned char* im = plane_image(P, p) + row * 3;
    for (int x = lo + threadIdx.x; x < hi; x += blockDim.x) {
      float m = bicubic_shared(wm, P.mw, ty, make_taps(x, P.mw, ow));
      if (!P.absolute) m = minmax_normalize(m, vlo, vhi);
      const int i = x - lo;
      st[0][i] = m;
#pragma unroll
      for (int c = 0; c < 3; ++c) st[1 + c][i] = ((float)__ldg(im + 3 * x + c) / 255.f) * m;
    }
  } else {
    for (int x = lo + threadIdx.x; x < hi; x += blockDim.x) {
#pragma unroll
      for (int c = 0; c < 4; ++c) st[c][x - lo] = buf[(4 + c) * n + row + x];
    }
  }
  __syncthreads();
  const int x = x0 + threadIdx.x;
  if (x >= ow) return;
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
  for (int k = max(0, x - r) - lo, k1 = min(ow - 1, x + r) - lo; k <= k1; ++k) {
    s0 += st[0][k]; s1 += st[1][k]; s2 += st[2][k]; s3 += st[3][k];
  }
  buf[row + x] = s0; buf[n + row + x] = s1; buf[2 * n + row + x] = s2; buf[3 * n + row + x] = s3;
}

// grid: (tiles of kColW x kColRows pixels, planes); dynamic smem: buffer channels 0-3 of rows [y0 - r, y0 + kColRows
// + r) of the tile's columns. Thread (column, row group) walks the staged rows once and adds each to those of its
// kColPer outputs whose window holds it: every output still sums its window from 0 in ascending row order.
// kFirst: means of m and I m -> a, b (channels 4-7); else means of a and b -> q.
template <bool kFirst>
__global__ void __launch_bounds__(256) refine_col_kernel(const __grid_constant__ RefinePlanes P) {
  extern __shared__ float cs[];                          // [4][rows][kColW]
  const int oh = P.oh, ow = P.ow, r = P.radius, p = blockIdx.y;
  const int tiles_x = (ow + kColW - 1) / kColW, tyi = blockIdx.x / tiles_x;
  const int x0 = (blockIdx.x - tyi * tiles_x) * kColW, y0 = tyi * kColRows;
  const int lo = max(0, y0 - r), rows = min(oh, y0 + kColRows + r) - lo, tw = min(kColW, ow - x0);
  const long long n = (long long)oh * ow;
  float* buf = P.buf + (long long)p * 8 * n;
  for (int c = 0; c < 4; ++c) {
    for (int i = threadIdx.x; i < rows * kColW; i += blockDim.x) {
      const int k = i / kColW, xx = i % kColW;
      cs[c * rows * kColW + i] = xx < tw ? buf[c * n + (long long)(lo + k) * ow + x0 + xx] : 0.f;
    }
  }
  __syncthreads();
  const int tx = threadIdx.x % kColW, x = x0 + tx, yb = y0 + (threadIdx.x / kColW) * kColPer;
  if (x >= ow || yb >= oh) return;
  float s[kColPer][4];
#pragma unroll
  for (int j = 0; j < kColPer; ++j) s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
  const int plane_floats = rows * kColW;
  for (int k = max(0, yb - r), k1 = min(oh - 1, yb + kColPer - 1 + r); k <= k1; ++k) {
    const float* v = cs + (k - lo) * kColW + tx;
    const float v0 = v[0], v1 = v[plane_floats], v2 = v[2 * plane_floats], v3 = v[3 * plane_floats];
#pragma unroll
    for (int j = 0; j < kColPer; ++j) {
      if ((unsigned)(k - (yb + j) + r) <= (unsigned)(2 * r)) {
        s[j][0] += v0; s[j][1] += v1; s[j][2] += v2; s[j][3] += v3;
      }
    }
  }
  const int nx = min(ow - 1, x + r) - max(0, x - r) + 1;
#pragma unroll
  for (int j = 0; j < kColPer; ++j) {
    const int y = yb + j;
    if (y >= oh) break;
    const float N = (float)(nx * (min(oh - 1, y + r) - max(0, y - r) + 1));
    const long long o = (long long)y * ow + x;
    if (kFirst) {
      const float pm = s[j][0] / N, mr = s[j][1] / N, mg = s[j][2] / N, mb = s[j][3] / N;
      const float* G = P.guide + (long long)(P.image_map_stride ? p / P.words_per_map : 0) * 9 * n + o;
      const float mu_r = G[0], mu_g = G[n], mu_b = G[2 * n];
      const float i_rr = G[3 * n], i_rg = G[4 * n], i_rb = G[5 * n], i_gg = G[6 * n], i_gb = G[7 * n], i_bb = G[8 * n];
      const float cr = mr - mu_r * pm, cg = mg - mu_g * pm, cb = mb - mu_b * pm;
      const float ar = i_rr * cr + i_rg * cg + i_rb * cb;
      const float ag = i_rg * cr + i_gg * cg + i_gb * cb;
      const float ab = i_rb * cr + i_gb * cg + i_bb * cb;
      buf[4 * n + o] = ar; buf[5 * n + o] = ag; buf[6 * n + o] = ab;
      buf[7 * n + o] = pm - (ar * mu_r + ag * mu_g + ab * mu_b);
    } else {
      const unsigned char* im = plane_image(P, p) + 3 * o;
      float q = (s[j][0] / N) * ((float)__ldg(im) / 255.f) + (s[j][1] / N) * ((float)__ldg(im + 1) / 255.f) +
                (s[j][2] / N) * ((float)__ldg(im + 2) / 255.f) + s[j][3] / N;
      if (P.use_threshold) q = q > P.threshold ? 1.f : 0.f;
      P.out[(long long)p * n + o] = q;
    }
  }
}

size_t col_smem(int radius) { return sizeof(float) * 4 * kColW * (kColRows + 2 * radius); }

}  // namespace

long long refine_guide_bytes(int h, int w) { return 36LL * h * w; }

long long refine_plane_bytes(int h, int w) { return 32LL * h * w + 4 * kWordPartialFloats; }

void refine_planes_in(void* scratch, int guides, int planes, int h, int w, RefinePlanes& p) {
  const long long n = (long long)h * w;
  float* f = static_cast<float*>(scratch);
  p.guide = f;
  f += 9 * n * guides;
  p.minmax = f;
  f += (long long)kWordPartialFloats * planes;
  p.buf = f;
  p.guides = guides; p.planes = planes; p.oh = h; p.ow = w;
}

int launch_refine_guides(const RefinePlanes& p, cudaStream_t stream) {
  const unsigned segs = (p.ow + kRowSeg - 1) / kRowSeg;
  guide_row_kernel<<<dim3(segs * p.oh, p.guides), 256, 0, stream>>>(p);
  DAAM_CUDA_TRY(cudaGetLastError());
  count_launch();
  const unsigned tiles = ((p.ow + kColW - 1) / kColW) * ((p.oh + kGuideRows - 1) / kGuideRows);
  guide_col_kernel<<<dim3(tiles, p.guides), 256, 0, stream>>>(p);
  DAAM_CUDA_TRY(cudaGetLastError());
  count_launch();
  return DAAM_OK;
}

int launch_refine(const RefinePlanes& p, int device, cudaStream_t stream) {
  static std::once_flag attr_once[64];
  cudaError_t attr_err = cudaSuccess;
  std::call_once(attr_once[device & 63], [&] {
    const int most = (int)col_smem(kRefineMaxRadius);
    attr_err = cudaFuncSetAttribute(refine_col_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, most);
    if (attr_err == cudaSuccess)
      attr_err = cudaFuncSetAttribute(refine_col_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, most);
  });
  DAAM_CUDA_TRY(attr_err);
  const dim3 rows((unsigned)((p.ow + kRowSeg - 1) / kRowSeg) * p.oh, p.planes);
  const dim3 tiles((unsigned)(((p.ow + kColW - 1) / kColW) * ((p.oh + kColRows - 1) / kColRows)), p.planes);
  const size_t smem = col_smem(p.radius);
  refine_row_kernel<true><<<rows, 256, 0, stream>>>(p);
  DAAM_CUDA_TRY(cudaGetLastError());
  refine_col_kernel<true><<<tiles, 256, smem, stream>>>(p);
  DAAM_CUDA_TRY(cudaGetLastError());
  refine_row_kernel<false><<<rows, 256, 0, stream>>>(p);
  DAAM_CUDA_TRY(cudaGetLastError());
  refine_col_kernel<false><<<tiles, 256, smem, stream>>>(p);
  DAAM_CUDA_TRY(cudaGetLastError());
  count_launch(4);
  return DAAM_OK;
}

}  // namespace daam
