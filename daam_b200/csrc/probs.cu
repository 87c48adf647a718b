// Materialised attention probabilities: the compatibility path behind the reference's save_heads / load_heads.
//
//  * attention_probs_kernel  -- P[(sample*heads + head)][pixel][token] = softmax_t(scale * q.k) for EVERY sample of
//    the batch, in the dtype of q: the tensor the reference saves with torch.save at daam/trace.py:246-247, 279-280
//    (the output of diffusers' get_attention_scores called at trace.py:276). Same one-thread-per-pixel SIMT tile as
//    accumulate_simt.cu; the 128 x 77 block of a tile is contiguous in P and written out coalesced through shared memory.
//  * accumulate_probs_kernel -- heat-map accumulation from supplied probabilities (load_heads, trace.py:281-294):
//    acc[r][token][pixel] += P[first_row + r][pixel][token]  (= _unravel_attn + update).
#include "simt_common.cuh"

namespace daam {
namespace {

template <typename T> __device__ __forceinline__ T from_float(float v);
template <> __device__ __forceinline__ float from_float<float>(float v) { return v; }
template <> __device__ __forceinline__ __half from_float<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 from_float<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <typename T> __device__ __forceinline__ float to_float(T v);
template <> __device__ __forceinline__ float to_float<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_float<__half>(__half v) { return __half2float(v); }
template <> __device__ __forceinline__ float to_float<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

template <typename T>
__device__ __forceinline__ void write_tile(const float* sp, T* out, int n) {
  for (int i = threadIdx.x; i < n; i += blockDim.x) out[i] = from_float<T>(sp[i]);
}

// One layer per launch; L.acc is unused, `probs` receives [n_prompts*heads][hw][77].
__global__ void __launch_bounds__(kTilePixels, 3) attention_probs_kernel(const __grid_constant__ LaunchParams P,
                                                                         void* __restrict__ probs) {
  extern __shared__ __align__(16) float smem[];
  const simt::TileSpan span = simt::cta_tiles(P.total_tiles);
  int li = 0, last_run = -1;
  for (int tile = span.first; tile < span.first + span.count; ++tile) {
    const simt::TileRef t = simt::decode_tile(P, tile, li);
    const LayerParams& L = P.layer[t.li];
    float* ks = smem;
    float* qs = smem + L.head_dim * kTokensPad;
    float* sp = qs;                                   // staged probabilities alias the Q tile once it has been consumed
    const bool load_k = t.run != last_run;
    last_run = t.run;
    __syncthreads();
    simt::stage_any(L, t, 0, ks, qs, load_k, /*load_q=*/true);
    __syncthreads();
    float s[kTokensPad];
    const float inv = simt::pixel_softmax(L, ks, qs, s);
    __syncthreads();                                  // every thread is done reading qs
#pragma unroll
    for (int j = 0; j < kTokens; ++j) sp[threadIdx.x * kTokens + j] = s[j] * inv;   // stride 77: conflict-free
    __syncthreads();
    const int rows = min(kTilePixels, L.hw - t.pixel0);
    const long long base = ((long long)(t.prompt * L.heads + t.head) * L.hw + t.pixel0) * kTokens;
    if (L.dtype == DAAM_F32) write_tile(sp, static_cast<float*>(probs) + base, rows * kTokens);
    else if (L.dtype == DAAM_F16) write_tile(sp, static_cast<__half*>(probs) + base, rows * kTokens);
    else write_tile(sp, static_cast<__nv_bfloat16*>(probs) + base, rows * kTokens);
  }
}

struct ProbsParams {
  const void* probs;
  float* acc;
  int dtype, first_row, n_rows, hw, tiles_per_row;
};

template <typename T>
__device__ __forceinline__ void read_tile(float* sp, const T* in, int n) {
  for (int i = threadIdx.x; i < n; i += blockDim.x) sp[i] = to_float<T>(in[i]);
}

// grid.x = n_rows * tiles_per_row; one CTA transposes one [128 pixels x 77] block through shared memory.
__global__ void __launch_bounds__(kTilePixels) accumulate_probs_kernel(const ProbsParams p) {
  __shared__ float sp[kTilePixels * kTokens];
  const int row = blockIdx.x / p.tiles_per_row, ptile = blockIdx.x % p.tiles_per_row;
  const int pixel0 = ptile * kTilePixels;
  const int rows = min(kTilePixels, p.hw - pixel0);
  const long long src = ((long long)(p.first_row + row) * p.hw + pixel0) * kTokens;
  if (p.dtype == DAAM_F32) read_tile(sp, static_cast<const float*>(p.probs) + src, rows * kTokens);
  else if (p.dtype == DAAM_F16) read_tile(sp, static_cast<const __half*>(p.probs) + src, rows * kTokens);
  else read_tile(sp, static_cast<const __nv_bfloat16*>(p.probs) + src, rows * kTokens);
  __syncthreads();
  if ((int)threadIdx.x < rows) {
    float* a = p.acc + (long long)row * kTokens * p.hw + pixel0 + threadIdx.x;
#pragma unroll 7
    for (int j = 0; j < kTokens; ++j) a[(long long)j * p.hw] += sp[threadIdx.x * kTokens + j];
  }
}

}  // namespace

int make_layer_params(const daam_layer& in, int index, LayerParams* out, bool need_acc);

}  // namespace daam

using namespace daam;

extern "C" int daam_attention_probs(const daam_layer* layer, void* probs, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!layer || !probs) { set_error("daam_attention_probs: null pointer"); return DAAM_E_INVALID; }
  DeviceInfo dev;
  if (int rc = get_device_info(&dev)) return rc;
  static thread_local LaunchParams p;
  if (int rc = make_layer_params(*layer, 0, &p.layer[0], /*need_acc=*/false)) return rc;
  if (layer->tokens != kTokens) { set_error("daam_attention_probs: tokens = %d, only %d-token contexts are materialised (the save_heads file format)", layer->tokens, kTokens); return DAAM_E_UNSUPPORTED; }
  p.n_layers = 1;
  p.layer[0].tile_begin = 0;
  p.total_tiles = p.layer[0].tiles_per_head * p.layer[0].heads * p.layer[0].n_prompts;
  p.rmw_mode = 0;
  p.pdl = 0;
  p.early_loads = 0;
  p.total_weight = p.total_tiles;
  size_t floats = simt::tile_smem_floats(p.layer[0].head_dim);
  const size_t need = (size_t)p.layer[0].head_dim * kTokensPad + (size_t)kTilePixels * kTokens;   // K^T + staged P
  if (need > floats) floats = need;
  const size_t smem = floats * sizeof(float);
  if (int rc = simt::reserve_dynamic_smem((const void*)attention_probs_kernel, dev.device, smem)) return rc;
  int grid = dev.sm_count * 3;
  if (grid > p.total_tiles) grid = p.total_tiles;
  attention_probs_kernel<<<grid, kTilePixels, smem, stream>>>(p, probs);
  DAAM_CUDA_TRY(cudaGetLastError());
  count_launch();
  return DAAM_OK;
}

extern "C" int daam_accumulate_probs(const void* probs, int32_t dtype, int32_t first_row, int32_t n_rows, int32_t hw,
                                     int32_t tokens, float* acc, void* stream_) {
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  if (!probs || !acc || first_row < 0 || n_rows <= 0 || hw <= 0) { set_error("daam_accumulate_probs: null pointer or bad size"); return DAAM_E_INVALID; }
  if (tokens != kTokens) { set_error("daam_accumulate_probs: tokens = %d, only %d-token probabilities are accumulated (the load_heads file format)", tokens, kTokens); return DAAM_E_UNSUPPORTED; }
  if (dtype != DAAM_F32 && dtype != DAAM_F16 && dtype != DAAM_BF16) { set_error("daam_accumulate_probs: unknown dtype %d", dtype); return DAAM_E_INVALID; }
  DeviceInfo dev;
  if (int rc = get_device_info(&dev)) return rc;
  ProbsParams p;
  p.probs = probs; p.acc = acc; p.dtype = dtype; p.first_row = first_row; p.n_rows = n_rows; p.hw = hw;
  p.tiles_per_row = (hw + kTilePixels - 1) / kTilePixels;
  accumulate_probs_kernel<<<n_rows * p.tiles_per_row, kTilePixels, 0, stream>>>(p);
  DAAM_CUDA_TRY(cudaGetLastError());
  count_launch();
  return DAAM_OK;
}
