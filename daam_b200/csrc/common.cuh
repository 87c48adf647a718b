// Shared declarations of libdaam_b200.so (host-side plumbing + the kernel parameter blocks).
#pragma once

#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

#include "daam_b200.h"

namespace daam {

constexpr int kTokens = DAAM_TOKENS;      // 77
constexpr int kTokensPad = 80;            // token axis padded to a multiple of 16 (UMMA N, float4 rows)
constexpr int kTilePixels = 128;          // pixels per tile == threads that own one pixel row each
constexpr int kMaxLayersPerLaunch = 32;   // layer descriptors carried in the kernel parameter block

// One layer call, device view. tile_begin is the exclusive prefix of tiles over the launch's layers.
struct LayerParams {
  const void* q;
  const void* k;
  float* acc;
  long long qs_prompt, qs_pixel, qs_head;
  long long ks_prompt, ks_token, ks_head;
  int n_prompts, heads, hw, head_dim;
  int dtype;
  float scale_log2e;        // attn.scale * log2(e): softmax is evaluated with exp2
  int tiles_per_head;       // ceil(hw / kTilePixels)
  int tile_begin;
  int vec_ok;               // 1: q/k rows are 16-byte aligned -> vector loads
  int weight;               // relative cost of one tile of this layer (wgmma kernel, K-chunked launches)
  int weight_begin;         // exclusive prefix of tiles x weight over the launch's layers
  int tokens;               // context rows: 77, or 154 / 231 (long-context instances); the accumulator's token extent
};

struct LaunchParams {
  int n_layers;
  int total_tiles;
  int rmw_mode;             // 0: load/add/store, 1: reduce-add (SIMT kernel, wgmma fp32 form)
  int pdl;                  // 1: launch with programmatic stream serialization (prologue overlaps the previous kernel)
  int early_loads;          // 1: only the accumulator updates wait for the previous kernel (DAAM_ACC_EARLY_LOADS)
  int total_weight;         // sum of tiles x weight (K-chunked launches partition by weight, not by tile count)
  LayerParams layer[kMaxLayersPerLaunch];
};

// exp2 on the SFU (ex2.approx: ~2 ulp, inputs here are <= 0 so no range handling is needed)
__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// The bulk-tensor reduce-add (cp.reduce.async.bulk .add.f32) and red.global.add.f32 flush subnormal inputs and results
// to zero; the accumulator updates done in shared memory use the same arithmetic, so both give the same bits.
// add_ftz(0.f, p) is the addend as such an add sees it: what the step-slab instances store.
__device__ __forceinline__ float add_ftz(float a, float b) {
  float r;
  asm("add.rn.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}

// Second slabs of one launch (daam_accumulate_steps: step slabs, daam_accumulate_range: range slabs): slab[i] has the
// layout of layer i's accumulator.
struct SecondSlabs {
  float* slab[kMaxLayersPerLaunch];
};
// What the accumulate kernels do to the second slab next to the add: nothing (daam_accumulate), store the addend
// (daam_accumulate_steps), or add it with the accumulator's arithmetic (daam_accumulate_range).
enum SlabMode : int { kSlabNone = 0, kSlabStore = 1, kSlabAdd = 2 };

// ---- error plumbing ---------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what);
#define DAAM_CUDA_TRY(expr)                                        \
  do {                                                             \
    cudaError_t e_ = (expr);                                       \
    if (e_ != cudaSuccess) return ::daam::cuda_fail(e_, #expr);    \
  } while (0)

struct DeviceInfo {
  int device = -1;
  int sm_count = 0;
  int cc_major = 0, cc_minor = 0;
};
int get_device_info(DeviceInfo* out);   // cached per device
void count_launch(int n = 1);

// ---- kernel launchers (one per translation unit) ----------------------------------------------------------------
// Preparation (tensor maps, grid, shared-memory size) is split from the launch so that api.cu can cache it per
// distinct daam_layer[] input: the steady state of a trace replays the same layer calls every denoising step.
// `slabs`: the launch's second slabs, nullptr exactly when `mode` is kSlabNone; `mode` selects the kernel instances
// (kSlabStore: daam_accumulate_steps, kSlabAdd: daam_accumulate_range).
// SIMT: every layer of `p` has one context length; 154- / 231-token contexts take the long-context kernel and no slabs.
int prepare_accumulate_simt(const LaunchParams& p, SlabMode mode, const DeviceInfo& dev, int* grid, size_t* smem);
int launch_prepared_simt(const LaunchParams& p, const SecondSlabs* slabs, SlabMode mode, int grid, size_t smem,
                         cudaStream_t stream);
void* prepared_mma_new();
void prepared_mma_delete(void* prepared);
int prepare_accumulate_mma(const LaunchParams& p, const SecondSlabs* slabs, SlabMode mode, const DeviceInfo& dev,
                           void* prepared);
int launch_prepared_mma(const void* prepared, cudaStream_t stream);
bool mma_supported(const LayerParams& l);

}  // namespace daam
