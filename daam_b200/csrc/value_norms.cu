// Value norms: n[b][h][j] = || W_h v_{b,h,j} ||_2, what context row j contributes through head h after the output
// projection (norm-based attention analysis). The weights of daam_finalize_parts_weighted.
//
// One CTA per (sample, head) and 77-token chunk of the context: it stages the chunk's [77][d] value block in shared
// memory, transposed so that consecutive threads read consecutive tokens, and streams W_h = W[:, h d : (h + 1) d] through
// shared memory kRows output rows at a time. Every y_c = sum_e W_h[c][e] v[e] is one thread's fmaf chain over e
// ascending; then thread j folds the chunk's y_c^2 into its token's sum, c ascending. So the arithmetic is the fixed
// order include/daam_b200.h states, whatever the launch geometry.
#include "common.cuh"

namespace daam {
namespace {

constexpr int kChunk = 77;     // tokens per CTA (one CLIP chunk)
constexpr int kRows = 32;      // output rows of W_h per shared-memory pass
constexpr int kThreads = 256;

__device__ __forceinline__ float load_f(const void* p, long long i, int dtype) {
  if (dtype == DAAM_F16) return __half2float(__ldg(static_cast<const __half*>(p) + i));
  if (dtype == DAAM_BF16) return __bfloat162float(__ldg(static_cast<const __nv_bfloat16*>(p) + i));
  return __ldg(static_cast<const float*>(p) + i);
}

struct NormParams {
  const void* v;
  const void* w;
  float* out;
  long long vs_sample, vs_token, vs_head, w_row;
  int v_dtype, w_dtype, heads, tokens, d, out_dim;
};

// grid: (n_samples * heads, tokens / 77). Dynamic smem: v^T [d][77], W rows [kRows][d + 1], y [kRows][77].
__global__ void __launch_bounds__(kThreads) value_norms_kernel(const __grid_constant__ NormParams P) {
  extern __shared__ float sm[];
  const int d = P.d, ldw = d + 1;
  float* vt = sm;                                      // vt[e * kChunk + j]
  float* ws = vt + d * kChunk;                         // ws[c * ldw + e]
  float* ys = ws + kRows * ldw;                        // ys[c * kChunk + j]
  const int sample = blockIdx.x / P.heads, head = blockIdx.x - sample * P.heads;
  const int t0 = blockIdx.y * kChunk;
  const long long vbase = sample * P.vs_sample + head * P.vs_head + t0 * P.vs_token;
  for (int i = threadIdx.x; i < kChunk * d; i += kThreads) {
    const int j = i / d, e = i - j * d;
    vt[e * kChunk + j] = load_f(P.v, vbase + j * P.vs_token + e, P.v_dtype);
  }
  float s = 0.f;                                       // thread j < 77: token t0 + j's sum of squares
  for (int c0 = 0; c0 < P.out_dim; c0 += kRows) {
    const int cn = min(kRows, P.out_dim - c0);
    __syncthreads();                                   // vt is staged / the previous pass's ws and ys are consumed
    for (int i = threadIdx.x; i < kRows * d; i += kThreads) {
      const int c = i / d, e = i - c * d;
      ws[c * ldw + e] = c < cn ? load_f(P.w, (long long)(c0 + c) * P.w_row + (long long)head * d + e, P.w_dtype) : 0.f;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < (kRows / 4) * kChunk; i += kThreads) {
      const int g = i / kChunk, j = i - g * kChunk;
      const float* w0 = ws + 4 * g * ldw;
      float y0 = 0.f, y1 = 0.f, y2 = 0.f, y3 = 0.f;
      for (int e = 0; e < d; ++e) {
        const float x = vt[e * kChunk + j];
        y0 = fmaf(w0[e], x, y0);
        y1 = fmaf(w0[ldw + e], x, y1);
        y2 = fmaf(w0[2 * ldw + e], x, y2);
        y3 = fmaf(w0[3 * ldw + e], x, y3);
      }
      float* y = ys + 4 * g * kChunk + j;
      y[0] = y0; y[kChunk] = y1; y[2 * kChunk] = y2; y[3 * kChunk] = y3;
    }
    __syncthreads();
    if (threadIdx.x < kChunk)
      for (int c = 0; c < cn; ++c) {
        const float y = ys[c * kChunk + threadIdx.x];
        s = fmaf(y, y, s);
      }
  }
  if (threadIdx.x < kChunk) P.out[(long long)blockIdx.x * P.tokens + t0 + threadIdx.x] = sqrtf(s);
}

}  // namespace
}  // namespace daam

using namespace daam;

extern "C" int daam_value_norms(const void* value, int32_t value_dtype, int64_t v_stride_sample, int64_t v_stride_token,
                                int64_t v_stride_head, const void* w, int32_t w_dtype, int64_t w_stride_row,
                                int32_t n_samples, int32_t heads, int32_t tokens, int32_t head_dim, int32_t out_dim,
                                float* out, void* stream) {
  const char* name = "daam_value_norms";
  if (!value || !w || !out || n_samples <= 0 || heads <= 0 || head_dim <= 0 || out_dim <= 0) {
    set_error("%s: null pointer or non-positive size", name);
    return DAAM_E_INVALID;
  }
  for (int32_t dt : {value_dtype, w_dtype})
    if (dt != DAAM_F32 && dt != DAAM_F16 && dt != DAAM_BF16) { set_error("%s: unknown dtype %d", name, dt); return DAAM_E_INVALID; }
  if (tokens != 77 && tokens != 154 && tokens != 231) {
    set_error("%s: %d context tokens (77, 154 or 231)", name, tokens);
    return DAAM_E_UNSUPPORTED;
  }
  if (head_dim > DAAM_MAX_HEAD_DIM || out_dim > 4096 || (long long)n_samples * heads > 65535) {
    set_error("%s: head_dim %d (<= %d), out_dim %d (<= 4096) or %d samples x %d heads (<= 65535) out of range", name,
              head_dim, DAAM_MAX_HEAD_DIM, out_dim, n_samples, heads);
    return DAAM_E_UNSUPPORTED;
  }
  DeviceInfo dev;
  if (int rc = get_device_info(&dev)) return rc;
  NormParams p;
  p.v = value; p.w = w; p.out = out;
  p.vs_sample = v_stride_sample; p.vs_token = v_stride_token; p.vs_head = v_stride_head; p.w_row = w_stride_row;
  p.v_dtype = value_dtype; p.w_dtype = w_dtype; p.heads = heads; p.tokens = tokens; p.d = head_dim; p.out_dim = out_dim;
  const size_t smem = ((size_t)head_dim * kChunk + (size_t)kRows * (head_dim + 1) + (size_t)kRows * kChunk) * sizeof(float);
  DAAM_CUDA_TRY(cudaFuncSetAttribute(value_norms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  value_norms_kernel<<<dim3(n_samples * heads, tokens / kChunk), kThreads, smem, static_cast<cudaStream_t>(stream)>>>(p);
  DAAM_CUDA_TRY(cudaGetLastError());
  count_launch();
  return DAAM_OK;
}
