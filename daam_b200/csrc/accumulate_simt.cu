// Fused softmax(QK^T) -> unravel -> accumulate, SIMT fp32 variant ("warp dot" path).
//
// Serves fp32 projections (BASELINE config 1: the reference's own fp32 numerics, which tensor cores cannot give)
// and every layer the wgmma variant does not take (unaligned rows). One thread owns one pixel: its 77
// logits live in registers, K^T sits in shared memory and is read as warp-wide broadcasts, so softmax needs no
// shuffles and the accumulator update `acc[t][pixel] += p[t]` is one fully coalesced 128-byte access per warp and
// token. Replaces daam/trace.py:276 (get_attention_scores), :219-244 (_unravel_attn) and :293-294 (update loop).
//
// The four kernels are instances of one body, accumulate_simt_body<kSlab, kLong>: the plain kernel (daam_accumulate) and
//  * the step-slab kernel (daam_accumulate_steps, kSlabStore): next to every add it stores the addend into the layer's
//    step slab, again one coalesced 128-byte access per warp and token (flushed like RED in reduce mode; in load / add /
//    store mode the add is an fma, so the stored value is the rounded product, i.e. fma(p, inv, 0));
//  * the range-slab kernel (daam_accumulate_range, kSlabAdd): adds the addend into the layer's range slab with the
//    arithmetic of the accumulator update: a second RED in reduce mode, fma(p, inv, old) in load / add / store mode;
//  * the long-context kernel (kLong: 154- / 231-token contexts, 2 or 3 CLIP chunks of 77 tokens; every such layer the
//    wgmma kernel does not take, fp32 projections included). The registers hold the logits of ONE 77-token chunk, and
//    K^T is staged one chunk at a time (all 231 tokens at head_dim 160 plus the Q tile would not fit in shared memory),
//    so every tile takes two passes over the chunks:
//      pass 1: a chunk's logits, then the running max m and sum l of exp2(scale log2e (s - m)) (l rescaled when m grows);
//      pass 2: last staged chunk first, the chunk's logits again (same code, same bits), p = exp2(...) / l added to the
//              chunk's 77 accumulator rows with the update of the plain kernel.
#include <map>
#include <mutex>
#include <utility>

#include "simt_common.cuh"

namespace daam {
namespace {

// Adds p[j] = s[j] * inv to the 77 accumulator rows acc[off + j * hw] and, as kSlab asks, stores it into or adds it to
// the second slab's rows slab[off + j * hw]: red.global.add (`reduce`) or load / add / store.
template <int kSlab>
__device__ __forceinline__ void accumulate_rows(bool reduce, float* acc, float* slab, long long off, long long hw,
                                                const float* s, float inv) {
  float* a = acc + off;
  if (reduce) {
#pragma unroll
    for (int j = 0; j < kTokens; ++j) {
      atomicAdd(a + j * hw, s[j] * inv);              // result unused -> RED
      if constexpr (kSlab == kSlabStore) slab[off + j * hw] = add_ftz(0.f, s[j] * inv);
      if constexpr (kSlab == kSlabAdd) atomicAdd(slab + off + j * hw, s[j] * inv);
    }
  } else {
    constexpr int kChunk = 11;                        // 77 = 7 x 11 loads in flight per thread
#pragma unroll
    for (int j0 = 0; j0 < kTokens; j0 += kChunk) {
      float old[kChunk];
#pragma unroll
      for (int i = 0; i < kChunk; ++i) old[i] = a[(j0 + i) * hw];
      if constexpr (kSlab == kSlabAdd) {
        float* r = slab + off;
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
        for (int i = 0; i < kChunk; ++i) slab[off + (j0 + i) * hw] = fmaf(s[j0 + i], inv, 0.f);
      }
    }
  }
}

template <int kSlab, bool kLong>
__device__ __forceinline__ void accumulate_simt_body(const LaunchParams& P, const SecondSlabs* S) {
  static_assert(!kLong || kSlab == kSlabNone, "second slabs take 77-token contexts only");
  extern __shared__ __align__(16) float smem[];
  const simt::TileSpan span = simt::cta_tiles(P.total_tiles);

  int li = 0, last_run = -1;
  for (int tile = span.first; tile < span.first + span.count; ++tile) {
    const simt::TileRef t = simt::decode_tile(P, tile, li);
    const LayerParams& L = P.layer[t.li];
    float* ks = smem;                                 // [d][80] (long contexts: one 77-token chunk)
    float* qs = smem + L.head_dim * kTokensPad;       // [128][d + 1]
    const bool load_k = kLong || t.run != last_run;   // long contexts: chunk 0 of K^T at every tile
    last_run = t.run;

    __syncthreads();                                  // previous tile's readers are done
    simt::stage_any(L, t, 0, ks, qs, load_k, /*load_q=*/true);
    __syncthreads();

    float s[kTokensPad];
    if constexpr (!kLong) {
      const float inv = simt::pixel_softmax(L, ks, qs, s);
      const int pixel = t.pixel0 + threadIdx.x;
      if (pixel < L.hw) {
        const long long off = ((long long)(t.prompt * L.heads + t.head) * kTokens) * L.hw + pixel;
        accumulate_rows<kSlab>(P.rmw_mode == 1, L.acc, kSlab == kSlabNone ? nullptr : S->slab[t.li], off, L.hw, s,
                               inv);
      }
    } else {
      const int chunks = L.tokens / kTokens;
      const float sc = L.scale_log2e;
      float m = -INFINITY, l = 0.f;                   // running max and sum over the chunks seen so far
      for (int c = 0; c < chunks; ++c) {
        if (c > 0) {
          __syncthreads();
          simt::stage_any(L, t, c, ks, qs, /*load_k=*/true, /*load_q=*/false);
          __syncthreads();
        }
        simt::pixel_logits(L.head_dim, ks, qs, s);
        float mc = s[0];
#pragma unroll
        for (int j = 1; j < kTokens; ++j) mc = fmaxf(mc, s[j]);
        const float mn = fmaxf(m, mc), mcn = mn * sc;
        float part = 0.f;
#pragma unroll
        for (int j = 0; j < kTokens; ++j) part += fast_exp2(fmaf(s[j], sc, -mcn));
        l = fmaf(l, fast_exp2(m * sc - mcn), part);  // (first chunk: exp2(-inf) = 0)
        m = mn;
      }
      const float inv = 1.0f / l, mcs = m * sc;
      const int pixel = t.pixel0 + threadIdx.x;
      const long long hw = L.hw;

      for (int c = chunks - 1; c >= 0; --c) {         // the last chunk is still staged
        if (c < chunks - 1) {
          __syncthreads();
          simt::stage_any(L, t, c, ks, qs, /*load_k=*/true, /*load_q=*/false);
          __syncthreads();
        }
        simt::pixel_logits(L.head_dim, ks, qs, s);
#pragma unroll
        for (int j = 0; j < kTokens; ++j) s[j] = fast_exp2(fmaf(s[j], sc, -mcs));
        if (pixel >= L.hw) continue;
        const long long off = ((long long)(t.prompt * L.heads + t.head) * L.tokens + c * kTokens) * hw + pixel;
        accumulate_rows<kSlabNone>(P.rmw_mode == 1, L.acc, nullptr, off, hw, s, inv);
      }
    }
  }
}

__global__ void __launch_bounds__(kTilePixels, 3) accumulate_simt_kernel(const __grid_constant__ LaunchParams P) {
  accumulate_simt_body<kSlabNone, false>(P, nullptr);
}

// (defined before the step kernel: in this order nvcc keeps the step kernel at its register count, 150 instead of 151)
__global__ void __launch_bounds__(kTilePixels, 3)
accumulate_simt_range_kernel(const __grid_constant__ LaunchParams P, const __grid_constant__ SecondSlabs S) {
  accumulate_simt_body<kSlabAdd, false>(P, &S);
}

__global__ void __launch_bounds__(kTilePixels, 3)
accumulate_simt_step_kernel(const __grid_constant__ LaunchParams P, const __grid_constant__ SecondSlabs S) {
  accumulate_simt_body<kSlabStore, false>(P, &S);
}

__global__ void __launch_bounds__(kTilePixels, 3) accumulate_simt_long_kernel(const __grid_constant__ LaunchParams P) {
  accumulate_simt_body<kSlabNone, true>(P, nullptr);
}

// The four kernels: indexed by SlabMode for 77-token contexts, then the long-context kernel.
constexpr int kSimtLong = 3;
const void* const kSimtInstances[] = {(const void*)accumulate_simt_kernel, (const void*)accumulate_simt_step_kernel,
                                    (const void*)accumulate_simt_range_kernel,
                                    (const void*)accumulate_simt_long_kernel};

// The kernel of a pack: every layer of `p` has the context length of its first layer.
const void* simt_instance(const LaunchParams& p, SlabMode mode) {
  return kSimtInstances[p.layer[0].tokens == kTokens ? (int)mode : kSimtLong];
}

}  // namespace

int simt::reserve_dynamic_smem(const void* kernel, int device, size_t smem) {
  static std::mutex mu;
  static std::map<std::pair<const void*, int>, size_t> configured;
  std::lock_guard<std::mutex> lock(mu);
  size_t& have = configured[{kernel, device}];
  if (smem > have) {
    DAAM_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    have = smem;
  }
  return DAAM_OK;
}

int prepare_accumulate_simt(const LaunchParams& p, SlabMode mode, const DeviceInfo& dev, int* grid_out,
                            size_t* smem_out) {
  const int tokens = p.layer[0].tokens;
  if (tokens != kTokens && mode != kSlabNone) {
    set_error("the SIMT step and range kernels take %d-token contexts only (got %d)", kTokens, tokens);
    return DAAM_E_UNSUPPORTED;
  }
  int dmax = 0;
  for (int i = 0; i < p.n_layers; ++i) {
    if (p.layer[i].tokens != tokens) {
      set_error("a SIMT launch takes one context length (layers of %d and %d tokens)", tokens, p.layer[i].tokens);
      return DAAM_E_UNSUPPORTED;
    }
    dmax = p.layer[i].head_dim > dmax ? p.layer[i].head_dim : dmax;
  }
  const size_t smem = sizeof(float) * simt::tile_smem_floats(dmax);
  const void* fn = simt_instance(p, mode);
  if (int rc = simt::reserve_dynamic_smem(fn, dev.device, smem)) return rc;
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
  void* args[] = {const_cast<LaunchParams*>(&p), const_cast<SecondSlabs*>(slabs)};   // (plain, long: args[0] only)
  DAAM_CUDA_TRY(cudaLaunchKernel(simt_instance(p, mode), dim3(grid), dim3(kTilePixels), args, smem, stream));
  count_launch();
  return DAAM_OK;
}

}  // namespace daam
