// Fused softmax(QK^T) -> unravel -> accumulate, SIMT fp32 variant ("warp dot" path).
//
// Serves fp32 projections (BASELINE config 1: the reference's own fp32 numerics, which tensor cores cannot give)
// and every layer the wgmma variant does not take (unaligned rows). One thread owns one pixel: its 77
// logits live in registers, K^T sits in shared memory and is read as warp-wide broadcasts, so softmax needs no
// shuffles and the accumulator update `acc[t][pixel] += p[t]` is one fully coalesced 128-byte access per warp and
// token. Replaces daam/trace.py:276 (get_attention_scores), :219-244 (_unravel_attn) and :293-294 (update loop).
//
// The step-slab kernel (daam_accumulate_steps) is the same body with kSlabStore: next to every add it stores the addend
// into the layer's step slab, again one coalesced 128-byte access per warp and token (flushed like RED in reduce mode;
// in load / add / store mode the add is an fma, so the stored value is the rounded product, i.e. fma(p, inv, 0)).
// The range-slab kernel (daam_accumulate_range) adds the addend into the layer's range slab with the arithmetic of the
// accumulator update: a second RED in reduce mode, fma(p, inv, old) in load / add / store mode.
#include <mutex>

#include "simt_common.cuh"

namespace daam {
namespace {

template <int kSlab>
__device__ __forceinline__ void accumulate_simt_body(const LaunchParams& P, const SecondSlabs* S) {
  extern __shared__ __align__(16) float smem[];
  // contiguous chunk of tiles per CTA: consecutive tiles share (layer, prompt, head), so K^T is staged once per run
  const int per = P.total_tiles / gridDim.x, rem = P.total_tiles % gridDim.x;
  const int first = blockIdx.x * per + min((int)blockIdx.x, rem);
  const int count = per + ((int)blockIdx.x < rem ? 1 : 0);

  int li = 0, last_run = -1;
  for (int tile = first; tile < first + count; ++tile) {
    const simt::TileRef t = simt::decode_tile(P, tile, li);
    const LayerParams& L = P.layer[t.li];
    float* ks = smem;                                 // [d][80]
    float* qs = smem + L.head_dim * kTokensPad;       // [128][d + 1]
    const bool load_k = t.run != last_run;
    last_run = t.run;

    __syncthreads();                                  // previous tile's readers are done
    simt::stage_any(L, t, ks, qs, load_k);
    __syncthreads();

    float s[kTokensPad];
    const float inv = simt::pixel_softmax(L, ks, qs, s);

    const int pixel = t.pixel0 + threadIdx.x;
    if (pixel < L.hw) {
      const long long off = ((long long)(t.prompt * L.heads + t.head) * kTokens) * L.hw + pixel;
      float* a = L.acc + off;
      const long long hw = L.hw;
      if (P.rmw_mode == 1) {
#pragma unroll
        for (int j = 0; j < kTokens; ++j) {
          atomicAdd(a + j * hw, s[j] * inv);          // result unused -> RED
          if constexpr (kSlab == kSlabStore) S->slab[t.li][off + j * hw] = add_ftz(0.f, s[j] * inv);
          if constexpr (kSlab == kSlabAdd) atomicAdd(S->slab[t.li] + off + j * hw, s[j] * inv);
        }
      } else {
        constexpr int kChunk = 11;                    // 77 = 7 x 11 loads in flight per thread
#pragma unroll
        for (int j0 = 0; j0 < kTokens; j0 += kChunk) {
          float old[kChunk];
#pragma unroll
          for (int i = 0; i < kChunk; ++i) old[i] = a[(j0 + i) * hw];
          if constexpr (kSlab == kSlabAdd) {
            float* r = S->slab[t.li] + off;
            float old_r[kChunk];
#pragma unroll
            for (int i = 0; i < kChunk; ++i) old_r[i] = r[(j0 + i) * hw];
#pragma unroll
            for (int i = 0; i < kChunk; ++i) r[(j0 + i) * hw] = fmaf(s[j0 + i], inv, old_r[i]);
          }
#pragma unroll
          for (int i = 0; i < kChunk; ++i) a[(j0 + i) * hw] = fmaf(s[j0 + i], inv, old[i]);
          if constexpr (kSlab == kSlabStore) {
#pragma unroll
            for (int i = 0; i < kChunk; ++i) S->slab[t.li][off + (j0 + i) * hw] = fmaf(s[j0 + i], inv, 0.f);
          }
        }
      }
    }
  }
}

__global__ void __launch_bounds__(kTilePixels, 3) accumulate_simt_kernel(const __grid_constant__ LaunchParams P) {
  accumulate_simt_body<kSlabNone>(P, nullptr);
}

// (defined before the step kernel: in this order nvcc keeps the step kernel at its register count, 150 instead of 151)
__global__ void __launch_bounds__(kTilePixels, 3)
accumulate_simt_range_kernel(const __grid_constant__ LaunchParams P, const __grid_constant__ SecondSlabs S) {
  accumulate_simt_body<kSlabAdd>(P, &S);
}

__global__ void __launch_bounds__(kTilePixels, 3)
accumulate_simt_step_kernel(const __grid_constant__ LaunchParams P, const __grid_constant__ SecondSlabs S) {
  accumulate_simt_body<kSlabStore>(P, &S);
}

// The three kernels, indexed by SlabMode.
const void* const kSimtInstances[] = {(const void*)accumulate_simt_kernel, (const void*)accumulate_simt_step_kernel,
                                    (const void*)accumulate_simt_range_kernel};

}  // namespace

int prepare_accumulate_simt(const LaunchParams& p, SlabMode mode, const DeviceInfo& dev, int* grid_out,
                            size_t* smem_out) {
  int dmax = 0;
  for (int i = 0; i < p.n_layers; ++i) dmax = p.layer[i].head_dim > dmax ? p.layer[i].head_dim : dmax;
  const size_t smem = sizeof(float) * simt::tile_smem_floats(dmax);
  static std::mutex mu;
  static size_t configured_dev[3][64] = {};           // the attribute is per device (and per kernel)
  const void* fn = kSimtInstances[mode];
  {
    std::lock_guard<std::mutex> lock(mu);
    size_t& configured = configured_dev[mode][dev.device & 63];
    if (smem > configured) {
      DAAM_CUDA_TRY(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      configured = smem;
    }
  }
  int occ = 0;
  DAAM_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, fn, kTilePixels, smem));
  if (occ < 1) occ = 1;
  int grid = dev.sm_count * occ;
  if (grid > p.total_tiles) grid = p.total_tiles;
  *grid_out = grid;
  *smem_out = smem;
  return DAAM_OK;
}

int launch_prepared_simt(const LaunchParams& p, const SecondSlabs* slabs, SlabMode mode, int grid, size_t smem,
                         cudaStream_t stream) {
  void* args[] = {const_cast<LaunchParams*>(&p), const_cast<SecondSlabs*>(slabs)};   // (the plain kernel reads args[0])
  DAAM_CUDA_TRY(cudaLaunchKernel(kSimtInstances[mode], dim3(grid), dim3(kTilePixels), args, smem, stream));
  count_launch();
  return DAAM_OK;
}

}  // namespace daam
