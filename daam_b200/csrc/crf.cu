// CRF-refined word segmentation (daam_segment_crf): mean-field inference of a Potts CRF whose unary logits are the
// word maps and whose pairwise kernel joins pixels that are close and alike in colour. With m[w] what expand_words
// gives without threshold, L labels (label 0 the background with score threshold when use_threshold, word w label
// w + use_threshold with score m[w]), z_l = scale * s_l in fp32, W(x) the (2r+1)^2 window around x clipped to the image
// (not renormalised) and I the RGB bytes:
//   k(x, y) = A[y - x] exp(-|I_x - I_y|^2 rgb_coef) + S[y - x]         (A, S: normalised Gaussian tables, crf_tables)
//   Q^0 = softmax(z),  Q^{t+1} = softmax(z + msg),  msg_l(x) = sum_{y in W(x), y != x} k(x, y) Q^t_l(y)
// labels = argmax of the last logits (lowest label on ties), scores = Q of that label.
//  1. crf_init_kernel: z from the word maps (the bits of expand_words), Q^0 = softmax(z);
//  2. crf_step_kernel, one launch per update: a 32 x 8 pixel tile stages the image bytes of the tile plus an r-pixel
//     halo and Q in label chunks in shared memory; each thread owns one pixel, computes each pair's weight once per
//     chunk (once per update when the labels fit one chunk) and applies it to every label of the chunk, then writes
//     z + msg and, after the last chunk, the softmax in place.
// Every window sum walks the window in one fixed order (rows, then columns, ascending) and the softmax sums in label
// order; there are no atomics, so the results are the same bits on every call and however the maps are split into
// rounds.
#include <math.h>

#include <mutex>

#include "bicubic.cuh"
#include "crf.cuh"
#include "word_value.cuh"

namespace daam {
namespace {

constexpr int kTileW = 32, kTileH = 8;   // one warp per tile row: conflict-free shared loads at every window offset

// min / max of v per word of map `map`, from segment_minmax_kernel's partials
__device__ __forceinline__ void crf_bounds(const CrfParams& P, int map, float* lo, float* hi) {
  if (P.absolute) return;
  for (int w = threadIdx.x; w < P.n_words; w += blockDim.x) {
    float vlo, vhi;
    partial_bounds(P.minmax + 2LL * ((long long)map * P.n_words + w) * P.chunks, P.chunks, vlo, vhi);
    lo[w] = vlo; hi[w] = vhi;
  }
}

// z_l at pixel (y, x) of map `map`: scale * s_l, rounded once (never fused into a later add)
__device__ __forceinline__ float crf_logit(const CrfParams& P, int map, int l, int y, int x, const float* lo,
                                           const float* hi) {
  float s;
  if (P.use_threshold && l == 0) {
    s = P.threshold;
  } else {
    const int w = l - P.use_threshold;
    const float* wm = P.word_maps + ((long long)map * P.n_words + w) * P.mh * P.mw;
    s = bicubic_shared(wm, P.mw, make_taps(y, P.mh, P.oh), make_taps(x, P.mw, P.ow));
    if (!P.absolute) s = minmax_normalize(s, lo[w], hi[w]);
  }
  return __fmul_rn(P.scale, s);
}

// The logits t_l at q[l * n] -> softmax in place: max, then expf(t - max) summed in label order, then each over the
// sum. Returns the argmax of t (lowest label on ties).
__device__ __forceinline__ int crf_softmax(float* q, long long n, int n_labels) {
  float mx = q[0];
  int arg = 0;
  for (int l = 1; l < n_labels; ++l) {
    const float t = q[l * n];
    if (t > mx) { mx = t; arg = l; }
  }
  float sum = 0.f;
  for (int l = 0; l < n_labels; ++l) {
    const float e = expf(q[l * n] - mx);
    q[l * n] = e;
    sum += e;
  }
  for (int l = 0; l < n_labels; ++l) q[l * n] = q[l * n] / sum;
  return arg;
}

__device__ __forceinline__ void crf_write_label(const CrfParams& P, int map, long long o, long long n, const float* q,
                                                int arg) {
  P.labels[(long long)map * n + o] = (unsigned char)(arg + 1 - P.use_threshold);
  P.scores[(long long)map * n + o] = q[arg * n];
}

// grid: (pixel blocks of 256, maps); thread: z and Q^0 of one pixel
__global__ void __launch_bounds__(256) crf_init_kernel(const __grid_constant__ CrfParams P) {
  __shared__ float s_lo[kCrfMaxWords], s_hi[kCrfMaxWords];
  const int map = blockIdx.y;
  crf_bounds(P, map, s_lo, s_hi);
  __syncthreads();
  const long long n = (long long)P.oh * P.ow, o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= n) return;
  const int y = (int)(o / P.ow), x = (int)(o - (long long)y * P.ow);
  float* q = P.q_out + (long long)map * P.n_labels * n + o;
  for (int l = 0; l < P.n_labels; ++l) q[l * n] = crf_logit(P, map, l, y, x, s_lo, s_hi);
  const int arg = crf_softmax(q, n, P.n_labels);
  if (P.last) crf_write_label(P, map, o, n, q, arg);
}

// grid: (tiles of kTileW x kTileH pixels, maps); dynamic smem: the tile's halo of (kTileH + 2r) x (kTileW + 2r) pixels,
// as packed RGB words, then kC label planes of Q over it. Labels go in chunks of at most kC.
template <int kC>
__global__ void __launch_bounds__(256) crf_step_kernel(const __grid_constant__ CrfParams P) {
  extern __shared__ __align__(16) float sm[];
  __shared__ float s_lo[kCrfMaxWords], s_hi[kCrfMaxWords];
  const int map = blockIdx.y, r = P.radius, oh = P.oh, ow = P.ow, L = P.n_labels;
  const int tiles_x = (ow + kTileW - 1) / kTileW;
  const int y0 = (blockIdx.x / tiles_x) * kTileH, x0 = (blockIdx.x % tiles_x) * kTileW;
  const int hc = kTileW + 2 * r, hn = (kTileH + 2 * r) * hc;
  unsigned* px = reinterpret_cast<unsigned*>(sm);
  float* qs = sm + hn;
  crf_bounds(P, map, s_lo, s_hi);
  const unsigned char* im = P.image + map * P.image_map_stride;
  for (int i = threadIdx.x; i < hn; i += blockDim.x) {
    const int gy = y0 - r + i / hc, gx = x0 - r + i % hc;
    unsigned v = 0;
    if (gy >= 0 && gy < oh && gx >= 0 && gx < ow) {
      const unsigned char* p = im + ((long long)gy * ow + gx) * 3;
      v = (unsigned)__ldg(p) | ((unsigned)__ldg(p + 1) << 8) | ((unsigned)__ldg(p + 2) << 16);
    }
    px[i] = v;
  }
  const int tx = threadIdx.x % kTileW, ty = threadIdx.x / kTileW, x = x0 + tx, y = y0 + ty;
  const bool inside = x < ow && y < oh;
  const long long n = (long long)oh * ow, o = (long long)y * ow + x;
  const float* qin = P.q_in + (long long)map * L * n;
  float* q = P.q_out + (long long)map * L * n + o;
  // the window clipped to the image; offsets relative to the pixel
  const int dy0 = max(-r, -y), dy1 = min(r, oh - 1 - y), dx0 = max(-r, -x), dx1 = min(r, ow - 1 - x);
  const int centre = (ty + r) * hc + tx + r, taps = 2 * r + 1;
  const float coef = P.rgb_coef;
  for (int c0 = 0; c0 < L; c0 += kC) {
    const int nc = min(kC, L - c0);
    __syncthreads();                                   // the previous chunk has been read (and px, s_lo written)
    for (int i = threadIdx.x; i < kC * hn; i += blockDim.x) {   // planes past the last label are zeros
      const int c = i / hn, j = i - c * hn;
      const int gy = y0 - r + j / hc, gx = x0 - r + j % hc;
      qs[i] = (c < nc && gy >= 0 && gy < oh && gx >= 0 && gx < ow)
                  ? qin[(long long)(c0 + c) * n + (long long)gy * ow + gx] : 0.f;
    }
    __syncthreads();
    if (!inside) continue;
    float acc[kC];
#pragma unroll
    for (int c = 0; c < kC; ++c) acc[c] = 0.f;
    const unsigned me = px[centre];
    const int mr = me & 255, mg = (me >> 8) & 255, mb = me >> 16;
    for (int dy = dy0; dy <= dy1; ++dy) {
      const int row = centre + dy * hc, trow = (dy + r) * taps + r;
#pragma unroll 1
      for (int dx = dx0; dx <= dx1; ++dx) {
        if (dy == 0 && dx == 0) continue;
        const unsigned v = px[row + dx];
        const int er = mr - (int)(v & 255), eg = mg - (int)((v >> 8) & 255), eb = mb - (int)(v >> 16);
        const float d2 = (float)(er * er + eg * eg + eb * eb);           // exact: at most 3 * 255^2
        const float k = fmaf(P.A[trow + dx], expf(-d2 * coef), P.S[trow + dx]);
        const float* qp = qs + row + dx;
#pragma unroll
        for (int c = 0; c < kC; ++c) acc[c] = fmaf(k, qp[c * hn], acc[c]);
      }
    }
#pragma unroll
    for (int c = 0; c < kC; ++c)
      if (c < nc) q[(c0 + c) * n] = __fadd_rn(crf_logit(P, map, c0 + c, y, x, s_lo, s_hi), acc[c]);
  }
  if (!inside) return;
  const int arg = crf_softmax(q, n, L);
  if (P.last) crf_write_label(P, map, o, n, q, arg);
}

// labels per chunk: the fewest chunks of at most 16, each padded to a multiple of 4
int chunk_size(int n_labels) {
  const int chunks = (n_labels + 15) / 16, per = (n_labels + chunks - 1) / chunks;
  return (per + 3) / 4 * 4;
}

size_t step_smem(int radius, int kc) {
  return sizeof(float) * (size_t)(kc + 1) * (kTileH + 2 * radius) * (kTileW + 2 * radius);
}

template <int kC>
int launch_step(const CrfParams& p, size_t smem, cudaStream_t stream) {
  const unsigned tiles = (unsigned)(((p.ow + kTileW - 1) / kTileW) * ((p.oh + kTileH - 1) / kTileH));
  crf_step_kernel<kC><<<dim3(tiles, p.maps), 256, smem, stream>>>(p);
  DAAM_CUDA_TRY(cudaGetLastError());
  count_launch();
  return DAAM_OK;
}

}  // namespace

long long crf_map_bytes(int n_labels, int h, int w) {
  return 8LL * n_labels * h * w + 4LL * kWordPartialFloats * n_labels;
}

void crf_tables(int radius, float appearance, float sigma_xy, float sigma_rgb, float smoothness, float sigma_smooth,
                CrfParams& p) {
  const int taps = 2 * radius + 1;
  const double cxy = 1.0 / (2.0 * (double)sigma_xy * sigma_xy), cs = 1.0 / (2.0 * (double)sigma_smooth * sigma_smooth);
  double sum_a = 0.0, sum_s = 0.0;
  for (int oy = -radius; oy <= radius; ++oy)
    for (int ox = -radius; ox <= radius; ++ox)
      if (oy || ox) { sum_a += exp(-(oy * oy + ox * ox) * cxy); sum_s += exp(-(oy * oy + ox * ox) * cs); }
  for (int oy = -radius; oy <= radius; ++oy)
    for (int ox = -radius; ox <= radius; ++ox) {
      const int i = (oy + radius) * taps + ox + radius;
      const double d = oy * oy + ox * ox;
      p.A[i] = (oy || ox) ? (float)((double)appearance * exp(-d * cxy) / sum_a) : 0.f;
      p.S[i] = (oy || ox) ? (float)((double)smoothness * exp(-d * cs) / sum_s) : 0.f;
    }
  p.rgb_coef = (float)(1.0 / (2.0 * (double)sigma_rgb * sigma_rgb));
}

int launch_crf(CrfParams& p, int iterations, float* q_a, float* q_b, float* probs, int device, cudaStream_t stream) {
  static std::once_flag attr_once[64];
  cudaError_t attr_err = cudaSuccess;
  std::call_once(attr_once[device & 63], [&] {
    const void* kernels[] = {(const void*)crf_step_kernel<4>, (const void*)crf_step_kernel<8>,
                             (const void*)crf_step_kernel<12>, (const void*)crf_step_kernel<16>};
    const int sizes[] = {4, 8, 12, 16};
    for (int i = 0; i < 4 && attr_err == cudaSuccess; ++i)
      attr_err = cudaFuncSetAttribute(kernels[i], cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      (int)step_smem(kCrfMaxRadius, sizes[i]));
  });
  DAAM_CUDA_TRY(attr_err);
  const long long n = (long long)p.oh * p.ow;
  // Q^0, or with no update the final Q (into probs when asked) and the labels
  p.last = iterations == 0;
  p.q_out = (p.last && probs) ? probs : q_a;
  crf_init_kernel<<<dim3((unsigned)((n + 255) / 256), p.maps), 256, 0, stream>>>(p);
  DAAM_CUDA_TRY(cudaGetLastError());
  count_launch();
  const int kc = chunk_size(p.n_labels);
  const size_t smem = step_smem(p.radius, kc);
  for (int it = 0; it < iterations; ++it) {
    p.q_in = p.q_out;
    p.last = it == iterations - 1;
    p.q_out = (p.last && probs) ? probs : (p.q_in == q_a ? q_b : q_a);
    int rc;
    switch (kc) {
      case 4: rc = launch_step<4>(p, smem, stream); break;
      case 8: rc = launch_step<8>(p, smem, stream); break;
      case 12: rc = launch_step<12>(p, smem, stream); break;
      default: rc = launch_step<16>(p, smem, stream); break;
    }
    if (rc) return rc;
  }
  return DAAM_OK;
}

}  // namespace daam
