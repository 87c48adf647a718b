// Fused softmax(QK^T) -> unravel -> accumulate for 154- / 231-token contexts (2 or 3 CLIP chunks of 77 tokens), SIMT.
//
// Serves every long-context layer the wgmma kernel does not take: fp32 projections (the wgmma kernel's split form has
// no long-context instances), unaligned rows, pixel counts that are not a multiple of 4, and DAAM_ACC_FORCE_SIMT. As in
// accumulate_simt.cu one thread owns one pixel and its registers hold 80 logits, here those of ONE 77-token chunk. K^T
// is staged one chunk at a time (all 231 tokens at head_dim 160 plus the Q tile would not fit in shared memory), and
// every tile takes two passes over the chunks:
//   pass 1: a chunk's logits, then the running max m and sum l of exp2(scale log2e (s - m)) (l rescaled when m grows);
//   pass 2: last staged chunk first, the chunk's logits again (same code, same bits), p = exp2(...) / l added to the
//           chunk's 77 accumulator rows, with the update mode of the plain kernel (RED, or load / add / store).
// Its own translation unit, so that the plain SIMT kernels are compiled exactly as before.
#include <mutex>

#include "simt_common.cuh"

namespace daam {
namespace {

// K^T of context rows [77 chunk, 77 chunk + 77) of (prompt, head) -> ks[dim][80], columns 77..79 zero.
template <typename T>
__device__ __forceinline__ void stage_k_chunk(const LayerParams& L, int prompt, int head, int chunk, float* ks) {
  const int d = L.head_dim;
  const T* kbase = static_cast<const T*>(L.k) + prompt * L.ks_prompt + head * L.ks_head +
                   (long long)chunk * kTokens * L.ks_token;
  constexpr int V = simt::Vec<T>::kElems;
  if (L.vec_ok) {
    const int vec_per_row = d / V;
    for (int c = threadIdx.x; c < kTokensPad * vec_per_row; c += blockDim.x) {
      const int t = c / vec_per_row, v = c - t * vec_per_row;
      float f[V];
      if (t < kTokens) {
        simt::Vec<T>::load(kbase + t * L.ks_token + v * V, f);
      } else {
#pragma unroll
        for (int i = 0; i < V; ++i) f[i] = 0.f;
      }
#pragma unroll
      for (int i = 0; i < V; ++i) ks[(v * V + i) * kTokensPad + t] = f[i];
    }
  } else {  // unaligned views: scalar loads
    for (int c = threadIdx.x; c < kTokensPad * d; c += blockDim.x) {
      const int t = c / d, e = c - t * d;
      ks[e * kTokensPad + t] = t < kTokens ? simt::Vec<T>::one(kbase + t * L.ks_token + e) : 0.f;
    }
  }
}

__device__ __forceinline__ void stage_k_any(const LayerParams& L, const simt::TileRef& t, int chunk, float* ks) {
  if (L.dtype == DAAM_F32) stage_k_chunk<float>(L, t.prompt, t.head, chunk, ks);
  else if (L.dtype == DAAM_F16) stage_k_chunk<__half>(L, t.prompt, t.head, chunk, ks);
  else stage_k_chunk<__nv_bfloat16>(L, t.prompt, t.head, chunk, ks);
}

// This thread's pixel: the raw logits <q, k> of the staged chunk in s[0..79] (columns 77..79 are padding).
__device__ __forceinline__ void chunk_logits(int d, const float* ks, const float* qs, float* s) {
#pragma unroll
  for (int t = 0; t < kTokensPad; ++t) s[t] = 0.f;
  const float* qrow = qs + threadIdx.x * (d + 1);
#pragma unroll 2
  for (int e = 0; e < d; ++e) {
    const float qv = qrow[e];
    const float4* kr = reinterpret_cast<const float4*>(ks + e * kTokensPad);
#pragma unroll
    for (int j = 0; j < kTokensPad / 4; ++j) {
      const float4 kv = kr[j];
      s[4 * j + 0] = fmaf(qv, kv.x, s[4 * j + 0]);
      s[4 * j + 1] = fmaf(qv, kv.y, s[4 * j + 1]);
      s[4 * j + 2] = fmaf(qv, kv.z, s[4 * j + 2]);
      s[4 * j + 3] = fmaf(qv, kv.w, s[4 * j + 3]);
    }
  }
}

__global__ void __launch_bounds__(kTilePixels, 3) accumulate_simt_long_kernel(const __grid_constant__ LaunchParams P) {
  extern __shared__ __align__(16) float smem[];
  const int per = P.total_tiles / gridDim.x, rem = P.total_tiles % gridDim.x;
  const int first = blockIdx.x * per + min((int)blockIdx.x, rem);
  const int count = per + ((int)blockIdx.x < rem ? 1 : 0);

  int li = 0;
  for (int tile = first; tile < first + count; ++tile) {
    const simt::TileRef t = simt::decode_tile(P, tile, li);
    const LayerParams& L = P.layer[t.li];
    float* ks = smem;                                 // [d][80]: one chunk of K^T
    float* qs = smem + L.head_dim * kTokensPad;       // [128][d + 1]
    const int chunks = L.tokens / kTokens;
    const float sc = L.scale_log2e;

    __syncthreads();                                  // previous tile's readers are done
    simt::stage_any(L, t, ks, qs, /*load_k=*/false);  // the Q tile
    stage_k_any(L, t, 0, ks);
    __syncthreads();

    float s[kTokensPad];
    float m = -INFINITY, l = 0.f;                     // running max and sum over the chunks seen so far
    for (int c = 0; c < chunks; ++c) {
      if (c > 0) {
        __syncthreads();
        stage_k_any(L, t, c, ks);
        __syncthreads();
      }
      chunk_logits(L.head_dim, ks, qs, s);
      float mc = s[0];
#pragma unroll
      for (int j = 1; j < kTokens; ++j) mc = fmaxf(mc, s[j]);
      const float mn = fmaxf(m, mc), mcn = mn * sc;
      float part = 0.f;
#pragma unroll
      for (int j = 0; j < kTokens; ++j) part += fast_exp2(fmaf(s[j], sc, -mcn));
      l = fmaf(l, fast_exp2(m * sc - mcn), part);    // (first chunk: exp2(-inf) = 0)
      m = mn;
    }
    const float inv = 1.0f / l, mcs = m * sc;

    const int pixel = t.pixel0 + threadIdx.x;
    const long long hw = L.hw;
    for (int c = chunks - 1; c >= 0; --c) {           // the last chunk is still staged
      if (c < chunks - 1) {
        __syncthreads();
        stage_k_any(L, t, c, ks);
        __syncthreads();
      }
      chunk_logits(L.head_dim, ks, qs, s);
#pragma unroll
      for (int j = 0; j < kTokens; ++j) s[j] = fast_exp2(fmaf(s[j], sc, -mcs));
      if (pixel >= L.hw) continue;
      float* a = L.acc + ((long long)(t.prompt * L.heads + t.head) * L.tokens + c * kTokens) * hw + pixel;
      if (P.rmw_mode == 1) {
#pragma unroll
        for (int j = 0; j < kTokens; ++j) atomicAdd(a + j * hw, s[j] * inv);     // result unused -> RED
      } else {
        constexpr int kChunk = 11;                    // 77 = 7 x 11 loads in flight per thread
#pragma unroll
        for (int j0 = 0; j0 < kTokens; j0 += kChunk) {
          float old[kChunk];
#pragma unroll
          for (int i = 0; i < kChunk; ++i) old[i] = a[(j0 + i) * hw];
#pragma unroll
          for (int i = 0; i < kChunk; ++i) a[(j0 + i) * hw] = fmaf(s[j0 + i], inv, old[i]);
        }
      }
    }
  }
}

}  // namespace

int prepare_accumulate_simt_long(const LaunchParams& p, const DeviceInfo& dev, int* grid_out, size_t* smem_out) {
  int dmax = 0;
  for (int i = 0; i < p.n_layers; ++i) {
    const int t = p.layer[i].tokens;
    if (t != 2 * kTokens && t != 3 * kTokens) {
      set_error("the long-context SIMT kernel takes 154- or 231-token contexts (got %d)", t);
      return DAAM_E_UNSUPPORTED;
    }
    dmax = p.layer[i].head_dim > dmax ? p.layer[i].head_dim : dmax;
  }
  const size_t smem = sizeof(float) * simt::tile_smem_floats(dmax);
  static std::mutex mu;
  static size_t configured_dev[64] = {};              // the attribute is per device
  {
    std::lock_guard<std::mutex> lock(mu);
    size_t& configured = configured_dev[dev.device & 63];
    if (smem > configured) {
      DAAM_CUDA_TRY(cudaFuncSetAttribute(accumulate_simt_long_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)smem));
      configured = smem;
    }
  }
  int occ = 0;
  DAAM_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, accumulate_simt_long_kernel, kTilePixels, smem));
  if (occ < 1) occ = 1;
  int grid = dev.sm_count * occ;
  if (grid > p.total_tiles) grid = p.total_tiles;
  *grid_out = grid;
  *smem_out = smem;
  return DAAM_OK;
}

int launch_prepared_simt_long(const LaunchParams& p, int grid, size_t smem, cudaStream_t stream) {
  accumulate_simt_long_kernel<<<grid, kTilePixels, smem, stream>>>(p);
  DAAM_CUDA_TRY(cudaGetLastError());
  count_launch();
  return DAAM_OK;
}

}  // namespace daam
