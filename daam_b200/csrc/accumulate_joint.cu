// Joint-attention heat maps (daam_accumulate_joint, include/daam_b200.h): for every (sample, head, context row, pixel)
// of every layer call,
//   acc[p][head][t][pixel] += exp2(fmaf(<q, k>, scale log2e, -lse log2e))
// where lse is the joint softmax's log-sum-exp over all image and context keys, taken from the attention that ran
// anyway. No softmax crosses a tile, so every (pixel tile, token tile) is independent and the cost is the accumulator's
// read-modify-write.
//
// Two kernels over one tile walk (a tile is one (layer, sample, head, pixel run); a CTA takes tiles blockIdx.x,
// blockIdx.x + gridDim.x, ...):
//  * 16-bit q / k: mma.sync m16n8k16 on tensor cores. A tile is 64 pixels; its queries are staged once in shared
//    memory, then the context is walked 64 tokens at a time, each of the 4 warps computing S^T = K Q^T for 16 tokens x
//    64 pixels. The C fragment gives each thread two adjacent pixels of a token row, so the accumulator moves as float2
//    loads and stores, every 32-byte sector whole; the loads are issued before the MMAs so that their latency hides
//    under them.
//  * fp32 q / k: SIMT, one thread per pixel of a 128-pixel tile, the context staged 32 tokens at a time and read as
//    warp-wide broadcasts; the dot product is an fmaf chain over the head dim in order.
// Every accumulator element of a launch is read and written by one thread once: no atomics, no order to vary.
#include <map>
#include <mutex>
#include <tuple>
#include <vector>

#include "common.cuh"

namespace daam {
namespace {

constexpr int kJointMaxLayers = DAAM_JOINT_MAX_LAYERS;
constexpr int kMmaPixels = 64;      // pixels per 16-bit tile
constexpr int kMmaTokens = 64;      // context rows per pass of a 16-bit tile (4 warps x 16)
constexpr int kSimtPixels = 128;    // pixels per fp32 tile (one per thread)
constexpr int kSimtTokens = 32;     // context rows per pass of an fp32 tile
constexpr float kLog2e = 1.4426950408889634f;

struct JointParams {
  const void* q;
  const void* k;
  float* acc;
  const float* lse;
  long long qs_prompt, qs_pixel, qs_head;
  long long ks_prompt, ks_token, ks_head;
  long long ls_prompt, ls_head, ls_pixel;
  int n_prompts, heads, hw, tokens, head_dim, dtype;
  int vec_ok;               // q / k rows and strides 16-byte aligned: staged with 16-byte loads
  float c;                  // fp32(scale * log2(e))
  int tiles_per_head;
  int tile_begin;           // exclusive prefix of tiles over the launch's layers
};

struct JointLaunch {
  int n_layers;
  int total_tiles;
  JointParams layer[kJointMaxLayers];
};

struct TileRef {
  int li, prompt, head, pixel0;
};

// Tiles of one CTA are increasing, so the layer index only moves forward.
__device__ __forceinline__ TileRef decode_tile(const JointLaunch& P, int tile, int& li, int tile_pixels) {
  while (li + 1 < P.n_layers && tile >= P.layer[li + 1].tile_begin) ++li;
  const JointParams& L = P.layer[li];
  const int local = tile - L.tile_begin;
  const int ptile = local % L.tiles_per_head, rest = local / L.tiles_per_head;
  return TileRef{li, rest / L.heads, rest % L.heads, ptile * tile_pixels};
}

// lse * log2(e) of the tile's pixels (0 past hw) into l2[0, n).
__device__ __forceinline__ void stage_lse(const JointParams& L, const TileRef& t, int n, float* l2) {
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int pixel = t.pixel0 + i;
    l2[i] = pixel < L.hw
                ? L.lse[t.prompt * L.ls_prompt + t.head * L.ls_head + pixel * L.ls_pixel] * kLog2e
                : 0.f;
  }
}

// ---- 16-bit: tensor cores ---------------------------------------------------------------------------------------

// Rows [0, 64) of a [rows][d] 16-bit matrix (row r at base + r * row_stride) into shared memory [64][ld], zero past
// `valid` rows and past column d (up to dpad, the head dim rounded up to 16).
__device__ __forceinline__ void stage16(const uint16_t* base, long long row_stride, int valid, int d, int dpad, int ld,
                                        bool vec, uint16_t* s) {
  const int cpr = dpad / 8;     // 16-byte chunks per row
  for (int i = threadIdx.x; i < 64 * cpr; i += blockDim.x) {
    const int r = i / cpr, c = (i % cpr) * 8;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (r < valid && c < d) {
      const uint16_t* src = base + r * row_stride + c;
      if (vec) {
        v = *reinterpret_cast<const uint4*>(src);
      } else {
        uint32_t w[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) w[j] = (uint32_t)src[2 * j] | ((uint32_t)src[2 * j + 1] << 16);
        v = make_uint4(w[0], w[1], w[2], w[3]);
      }
    }
    *reinterpret_cast<uint4*>(s + r * ld + c) = v;
  }
}

template <bool kBf16>
__device__ __forceinline__ void mma16816(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
  if constexpr (kBf16) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                 "{%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  } else {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                 "{%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  }
}

__device__ __forceinline__ uint32_t lds32(const uint16_t* p) { return *reinterpret_cast<const uint32_t*>(p); }

// The accumulate of one 16-token x 64-pixel block of a warp: `old` holds the accumulator values loaded before the
// MMAs, c the logits; rows t >= tokens and pixels >= hw are neither read nor written.
template <bool kPair>
__device__ __forceinline__ void load_block(const float* acc, int hw, int tokens, int row, int px, float (*old)[4]) {
#pragma unroll
  for (int nt = 0; nt < 8; ++nt) {
    const int pixel = px + nt * 8;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int t = row + 8 * half;
      float* o = old[nt] + 2 * half;
      o[0] = o[1] = 0.f;
      if (t < tokens) {
        const float* a = acc + (long long)t * hw + pixel;
        if constexpr (kPair) {
          if (pixel < hw) {
            const float2 v = *reinterpret_cast<const float2*>(a);
            o[0] = v.x;
            o[1] = v.y;
          }
        } else {
          if (pixel < hw) o[0] = a[0];
          if (pixel + 1 < hw) o[1] = a[1];
        }
      }
    }
  }
}

template <bool kPair>
__device__ __forceinline__ void store_block(float* acc, int hw, int tokens, int row, int px, const float (*old)[4],
                                            const float (*s)[4], float c, const float* l2, int lpx) {
#pragma unroll
  for (int nt = 0; nt < 8; ++nt) {
    const int pixel = px + nt * 8;
    const float l0 = l2[lpx + nt * 8], l1 = l2[lpx + nt * 8 + 1];
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int t = row + 8 * half;
      if (t >= tokens) continue;
      const float v0 = old[nt][2 * half] + fast_exp2(fmaf(s[nt][2 * half], c, -l0));
      const float v1 = old[nt][2 * half + 1] + fast_exp2(fmaf(s[nt][2 * half + 1], c, -l1));
      float* a = acc + (long long)t * hw + pixel;
      if constexpr (kPair) {
        if (pixel < hw) *reinterpret_cast<float2*>(a) = make_float2(v0, v1);
      } else {
        if (pixel < hw) a[0] = v0;
        if (pixel + 1 < hw) a[1] = v1;
      }
    }
  }
}

template <bool kBf16>
__global__ void __launch_bounds__(128, 4) accumulate_joint_mma_kernel(const __grid_constant__ JointLaunch P) {
  extern __shared__ __align__(16) uint16_t smem16[];
  __shared__ float l2[kMmaPixels];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, tig = lane & 3;
  int li = 0;
  for (int tile = blockIdx.x; tile < P.total_tiles; tile += gridDim.x) {
    const TileRef t = decode_tile(P, tile, li, kMmaPixels);
    const JointParams& L = P.layer[t.li];
    const int d = L.head_dim, dpad = (d + 15) & ~15, ld = dpad + 8;
    uint16_t* qs = smem16;
    uint16_t* ks = smem16 + kMmaPixels * ld;
    const bool vec = L.vec_ok != 0;
    const uint16_t* qb = static_cast<const uint16_t*>(L.q) + t.prompt * L.qs_prompt + t.head * L.qs_head +
                         (long long)t.pixel0 * L.qs_pixel;
    const uint16_t* kb = static_cast<const uint16_t*>(L.k) + t.prompt * L.ks_prompt + t.head * L.ks_head;
    float* acc = L.acc + (long long)(t.prompt * L.heads + t.head) * L.tokens * L.hw;
    const bool pair = (L.hw & 1) == 0;                 // float2 accesses stay 8-byte aligned
    const int px = t.pixel0 + 2 * tig;                 // this thread's first pixel, n-tile 0

    __syncthreads();                                   // the previous tile's readers are done with qs / l2
    stage16(qb, L.qs_pixel, L.hw - t.pixel0, d, dpad, ld, vec, qs);
    stage_lse(L, t, kMmaPixels, l2);
    for (int t0 = 0; t0 < L.tokens; t0 += kMmaTokens) {
      if (t0 > 0) __syncthreads();                     // every warp is done with the previous K tile
      stage16(kb + t0 * L.ks_token, L.ks_token, L.tokens - t0, d, dpad, ld, vec, ks);
      __syncthreads();
      const int row = t0 + 16 * warp + g;
      if (t0 + 16 * warp >= L.tokens) continue;        // (no barrier follows inside the pass)
      float old[8][4], s[8][4];
      if (pair) load_block<true>(acc, L.hw, L.tokens, row, px, old);
      else load_block<false>(acc, L.hw, L.tokens, row, px, old);
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
      const uint16_t* ka = ks + (16 * warp + g) * ld + 2 * tig;
      const uint16_t* qa = qs + g * ld + 2 * tig;
      for (int k0 = 0; k0 < dpad; k0 += 16) {
        uint32_t a[4];
        a[0] = lds32(ka + k0);
        a[1] = lds32(ka + 8 * ld + k0);
        a[2] = lds32(ka + k0 + 8);
        a[3] = lds32(ka + 8 * ld + k0 + 8);
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
          const uint16_t* qn = qa + nt * 8 * ld + k0;
          mma16816<kBf16>(s[nt], a, lds32(qn), lds32(qn + 8));
        }
      }
      if (pair) store_block<true>(acc, L.hw, L.tokens, row, px, old, s, L.c, l2, 2 * tig);
      else store_block<false>(acc, L.hw, L.tokens, row, px, old, s, L.c, l2, 2 * tig);
    }
  }
}

size_t mma_smem_bytes(int dmax) {
  const int dpad = (dmax + 15) & ~15;
  return sizeof(uint16_t) * 2 * kMmaPixels * (dpad + 8);
}

// ---- fp32: SIMT -------------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(kSimtPixels) accumulate_joint_simt_kernel(const __grid_constant__ JointLaunch P) {
  extern __shared__ __align__(16) float smem32[];
  __shared__ float l2[kSimtPixels];
  int li = 0;
  for (int tile = blockIdx.x; tile < P.total_tiles; tile += gridDim.x) {
    const TileRef t = decode_tile(P, tile, li, kSimtPixels);
    const JointParams& L = P.layer[t.li];
    const int d = L.head_dim;
    float* qs = smem32;                                // [128][d + 1]
    float* ks = smem32 + kSimtPixels * (d + 1);        // [32][d]
    const float* qb = static_cast<const float*>(L.q) + t.prompt * L.qs_prompt + t.head * L.qs_head;
    const float* kb = static_cast<const float*>(L.k) + t.prompt * L.ks_prompt + t.head * L.ks_head;
    float* acc = L.acc + (long long)(t.prompt * L.heads + t.head) * L.tokens * L.hw;
    const int pixel = t.pixel0 + threadIdx.x;
    const bool live = pixel < L.hw;

    __syncthreads();
    for (int i = threadIdx.x; i < kSimtPixels * d; i += kSimtPixels) {
      const int r = i / d, e = i % d, x = t.pixel0 + r;
      qs[r * (d + 1) + e] = x < L.hw ? qb[x * L.qs_pixel + e] : 0.f;
    }
    stage_lse(L, t, kSimtPixels, l2);
    for (int t0 = 0; t0 < L.tokens; t0 += kSimtTokens) {
      __syncthreads();
      for (int i = threadIdx.x; i < kSimtTokens * d; i += kSimtPixels) {
        const int r = i / d, e = i % d;
        ks[i] = t0 + r < L.tokens ? kb[(t0 + r) * L.ks_token + e] : 0.f;
      }
      __syncthreads();
      const float l = l2[threadIdx.x];
      const float* qrow = qs + threadIdx.x * (d + 1);
      for (int j0 = 0; j0 < kSimtTokens && t0 + j0 < L.tokens; j0 += 8) {
        float old[8], s[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          s[i] = 0.f;
          old[i] = live && t0 + j0 + i < L.tokens ? acc[(long long)(t0 + j0 + i) * L.hw + pixel] : 0.f;
        }
        for (int e = 0; e < d; ++e) {
          const float qv = qrow[e];
#pragma unroll
          for (int i = 0; i < 8; ++i) s[i] = fmaf(qv, ks[(j0 + i) * d + e], s[i]);
        }
#pragma unroll
        for (int i = 0; i < 8; ++i)
          if (live && t0 + j0 + i < L.tokens)
            acc[(long long)(t0 + j0 + i) * L.hw + pixel] = old[i] + fast_exp2(fmaf(s[i], L.c, -l));
      }
    }
  }
}

size_t simt_smem_bytes(int dmax) { return sizeof(float) * (kSimtPixels * (dmax + 1) + kSimtTokens * dmax); }

// ---- host -------------------------------------------------------------------------------------------------------

int validate(const daam_joint_layer& in, int i, JointParams* out) {
  static const char* fn = "daam_accumulate_joint";
  if (!in.q || !in.k || !in.acc || !in.lse) { set_error("%s: layer %d has a null pointer", fn, i); return DAAM_E_INVALID; }
  if (in.dtype != DAAM_F32 && in.dtype != DAAM_F16 && in.dtype != DAAM_BF16) { set_error("%s: layer %d: unknown dtype %d", fn, i, in.dtype); return DAAM_E_INVALID; }
  if (in.n_prompts <= 0 || in.heads <= 0 || in.hw <= 0) { set_error("%s: layer %d: non-positive n_prompts / heads / hw", fn, i); return DAAM_E_INVALID; }
  if (reinterpret_cast<uintptr_t>(in.acc) % 16 != 0) { set_error("%s: layer %d: acc is not 16-byte aligned", fn, i); return DAAM_E_INVALID; }
  if (!(in.scale > 0.f)) { set_error("%s: layer %d: scale must be positive", fn, i); return DAAM_E_INVALID; }
  if (in.tokens < 1 || in.tokens > DAAM_JOINT_MAX_TOKENS) { set_error("%s: layer %d: tokens = %d, must be in [1, %d]", fn, i, in.tokens, DAAM_JOINT_MAX_TOKENS); return DAAM_E_UNSUPPORTED; }
  if (in.head_dim <= 0 || in.head_dim % 8 != 0 || in.head_dim > DAAM_MAX_HEAD_DIM) { set_error("%s: layer %d: head_dim = %d must be a multiple of 8 in (0, %d]", fn, i, in.head_dim, DAAM_MAX_HEAD_DIM); return DAAM_E_UNSUPPORTED; }
  const long long slab = (long long)in.n_prompts * in.heads * in.tokens * in.hw;
  if (slab > (1ll << 40)) { set_error("%s: layer %d: accumulator of %lld elements is too large", fn, i, slab); return DAAM_E_INVALID; }
  JointParams& L = *out;
  L.q = in.q; L.k = in.k; L.acc = in.acc; L.lse = in.lse;
  L.qs_prompt = in.q_stride_prompt; L.qs_pixel = in.q_stride_pixel; L.qs_head = in.q_stride_head;
  L.ks_prompt = in.k_stride_prompt; L.ks_token = in.k_stride_token; L.ks_head = in.k_stride_head;
  L.ls_prompt = in.lse_stride_prompt; L.ls_head = in.lse_stride_head; L.ls_pixel = in.lse_stride_pixel;
  L.n_prompts = in.n_prompts; L.heads = in.heads; L.hw = in.hw; L.tokens = in.tokens; L.head_dim = in.head_dim;
  L.dtype = in.dtype;
  L.c = in.scale * kLog2e;
  const long long es = in.dtype == DAAM_F32 ? 4 : 2;
  auto aligned = [&](long long stride) { return (stride * es) % 16 == 0; };
  L.vec_ok = reinterpret_cast<uintptr_t>(in.q) % 16 == 0 && reinterpret_cast<uintptr_t>(in.k) % 16 == 0 &&
             aligned(in.q_stride_prompt) && aligned(in.q_stride_pixel) && aligned(in.q_stride_head) &&
             aligned(in.k_stride_prompt) && aligned(in.k_stride_token) && aligned(in.k_stride_head);
  const int tile = in.dtype == DAAM_F32 ? kSimtPixels : kMmaPixels;
  L.tiles_per_head = (in.hw + tile - 1) / tile;
  L.tile_begin = 0;
  return DAAM_OK;
}

size_t slab_bytes(const JointParams& l) { return sizeof(float) * (size_t)l.n_prompts * l.heads * l.tokens * l.hw; }

bool overlap(const JointParams& a, const JointParams& b) {
  const char *pa = reinterpret_cast<const char*>(a.acc), *pb = reinterpret_cast<const char*>(b.acc);
  return pa < pb + slab_bytes(b) && pb < pa + slab_bytes(a);
}

// Grid of one launch of `kernel` with `smem` bytes of dynamic shared memory: every SM full, at most one CTA per tile.
int grid_for(const void* kernel, int device, int sm_count, size_t smem, int tiles, int* grid) {
  static std::mutex mu;
  static std::map<std::tuple<const void*, int, size_t>, int> occupancy;
  static std::map<std::pair<const void*, int>, size_t> reserved;   // the kernel's largest dynamic smem so far
  int occ;
  {
    std::lock_guard<std::mutex> lock(mu);
    size_t& have = reserved[{kernel, device}];
    if (smem > have) {                                 // only ever raised: a smaller launch must not shrink it
      DAAM_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      have = smem;
    }
    auto it = occupancy.find({kernel, device, smem});
    if (it == occupancy.end()) {
      int n = 0;
      DAAM_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kernel, 128, smem));
      it = occupancy.emplace(std::make_tuple(kernel, device, smem), n < 1 ? 1 : n).first;
    }
    occ = it->second;
  }
  *grid = tiles < sm_count * occ ? tiles : sm_count * occ;
  return DAAM_OK;
}

int launch(JointLaunch& p, bool simt, const DeviceInfo& dev, cudaStream_t stream) {
  if (p.n_layers == 0) return DAAM_OK;
  int dmax = 0;
  for (int i = 0; i < p.n_layers; ++i) dmax = p.layer[i].head_dim > dmax ? p.layer[i].head_dim : dmax;
  const void* kernel = simt ? (const void*)accumulate_joint_simt_kernel
                            : p.layer[0].dtype == DAAM_BF16 ? (const void*)accumulate_joint_mma_kernel<true>
                                                            : (const void*)accumulate_joint_mma_kernel<false>;
  const size_t smem = simt ? simt_smem_bytes(dmax) : mma_smem_bytes(dmax);
  int grid = 0;
  if (int rc = grid_for(kernel, dev.device, dev.sm_count, smem, p.total_tiles, &grid)) return rc;
  void* args[] = {&p};
  DAAM_CUDA_TRY(cudaLaunchKernel(kernel, dim3(grid), dim3(128), args, smem, stream));
  count_launch();
  p.n_layers = 0;
  p.total_tiles = 0;
  return DAAM_OK;
}

}  // namespace
}  // namespace daam

using namespace daam;

extern "C" int daam_accumulate_joint(const daam_joint_layer* layers, int32_t n_layers, uint32_t flags, void* stream_) {
  if (n_layers < 0 || (n_layers > 0 && !layers)) { set_error("daam_accumulate_joint: bad layer array"); return DAAM_E_INVALID; }
  if (flags != 0) { set_error("daam_accumulate_joint: flags = %u, none are defined (pass 0)", flags); return DAAM_E_INVALID; }
  std::vector<JointParams> all((size_t)n_layers);
  for (int i = 0; i < n_layers; ++i)
    if (int rc = validate(layers[i], i, &all[i])) return rc;
  if (n_layers == 0) return DAAM_OK;
  DeviceInfo dev;
  if (int rc = get_device_info(&dev)) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  // Class by class (16-bit on tensor cores: fp16 and bf16 are separate kernels; then fp32), each layer in call order;
  // a layer whose accumulator overlaps one already in the launch, or a full launch, starts the next launch.
  static thread_local JointLaunch p;
  for (int cls : {DAAM_F16, DAAM_BF16, DAAM_F32}) {
    p.n_layers = 0;
    p.total_tiles = 0;
    for (const JointParams& L : all) {
      if (L.dtype != cls) continue;
      bool full = p.n_layers == kJointMaxLayers;
      for (int m = 0; m < p.n_layers && !full; ++m) full = overlap(p.layer[m], L);
      if (full)
        if (int rc = launch(p, cls == DAAM_F32, dev, stream)) return rc;
      JointParams& slot = p.layer[p.n_layers++];
      slot = L;
      slot.tile_begin = p.total_tiles;
      p.total_tiles += L.tiles_per_head * L.heads * L.n_prompts;
    }
    if (int rc = launch(p, cls == DAAM_F32, dev, stream)) return rc;
  }
  return DAAM_OK;
}
