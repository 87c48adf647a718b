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
//
// Head-reduced form (daam_accumulate_joint_heads): acc[p][t][pixel] += (sum over heads h ascending of v_h) / heads,
// v_h exactly the value above. A tile is (layer, sample, pixel run, token block), the token blocks of a pixel run
// adjacent in the walk (their CTAs read the same queries, from L2 after the first). The CTA walks the heads of its
// block and keeps the head sum in registers, so the accumulator is read and written once per tile:
//  * 16-bit: 64 pixels x 64 tokens, the mma.sync fragments of the per-head kernel; Q_h, K_h and lse_h of head h + 1
//    are staged by cp.async into the second of two buffers while head h computes.
//  * fp32: 128 pixels x 32 tokens, one thread per pixel, the per-head kernel's fmaf chain.
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
constexpr int kMeanMmaTokens = 64;  // context rows per head-reduced 16-bit tile
constexpr int kMeanSimtTokens = 32; // context rows per head-reduced fp32 tile

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
  int tiles_per_head;       // pixel runs per (sample, head)
  int token_blocks;         // head-reduced only: context blocks per pixel run
  int acc_heads;            // head axis of acc: heads, or 1 when the heads are reduced
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

// ---- head-reduced: one accumulator row per sample -----------------------------------------------------------------

struct MeanTile {
  int li, prompt, pixel0, token0;
};

// Tiles of one CTA are increasing, so the layer index only moves forward. Token blocks vary fastest.
__device__ __forceinline__ MeanTile decode_mean_tile(const JointLaunch& P, int tile, int& li, int tile_pixels,
                                                     int tile_tokens) {
  while (li + 1 < P.n_layers && tile >= P.layer[li + 1].tile_begin) ++li;
  const JointParams& L = P.layer[li];
  const int local = tile - L.tile_begin;
  const int block = local % L.token_blocks, rest = local / L.token_blocks;
  return MeanTile{li, rest / L.tiles_per_head, (rest % L.tiles_per_head) * tile_pixels, block * tile_tokens};
}

__device__ __forceinline__ void cp_async16(void* dst, const void* src) {
  const unsigned d = static_cast<unsigned>(__cvta_generic_to_shared(dst));
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(src) : "memory");
}

__device__ __forceinline__ void cp_async4(void* dst, const void* src) {
  const unsigned d = static_cast<unsigned>(__cvta_generic_to_shared(dst));
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(d), "l"(src) : "memory");
}

__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }

template <int kPending>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(kPending) : "memory"); }

// stage16 through cp.async when rows are 16-byte aligned; otherwise with plain loads, complete on return.
__device__ __forceinline__ void stage16_async(const uint16_t* base, long long row_stride, int valid, int d, int dpad,
                                              int ld, bool vec, uint16_t* s) {
  if (!vec) {
    stage16(base, row_stride, valid, d, dpad, ld, false, s);
    return;
  }
  const int cpr = dpad / 8;
  for (int i = threadIdx.x; i < 64 * cpr; i += blockDim.x) {
    const int r = i / cpr, c = (i % cpr) * 8;
    uint16_t* dst = s + r * ld + c;
    if (r < valid && c < d) cp_async16(dst, base + r * row_stride + c);
    else *reinterpret_cast<uint4*>(dst) = make_uint4(0u, 0u, 0u, 0u);
  }
}

// Raw lse (natural log, not yet times log2(e)) of pixels [pixel0, pixel0 + n) of (prompt, head) into l, 0 past hw.
__device__ __forceinline__ void stage_lse_async(const JointParams& L, int prompt, int head, int pixel0, int n,
                                                float* l) {
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int pixel = pixel0 + i;
    if (pixel < L.hw) cp_async4(l + i, L.lse + prompt * L.ls_prompt + head * L.ls_head + pixel * L.ls_pixel);
    else l[i] = 0.f;
  }
}

template <bool kPair>
__device__ __forceinline__ void store_mean_block(float* acc, int hw, int tokens, int row, int px, const float (*old)[4],
                                                 const float (*sum)[4], float heads) {
#pragma unroll
  for (int nt = 0; nt < 8; ++nt) {
    const int pixel = px + nt * 8;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int t = row + 8 * half;
      if (t >= tokens) continue;
      const float v0 = old[nt][2 * half] + __fdiv_rn(sum[nt][2 * half], heads);
      const float v1 = old[nt][2 * half + 1] + __fdiv_rn(sum[nt][2 * half + 1], heads);
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
__global__ void __launch_bounds__(128, 4) accumulate_joint_mean_mma_kernel(const __grid_constant__ JointLaunch P) {
  extern __shared__ __align__(16) uint16_t smem16[];
  __shared__ float lse_s[2][kMmaPixels];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, tig = lane & 3;
  int li = 0;
  for (int tile = blockIdx.x; tile < P.total_tiles; tile += gridDim.x) {
    const MeanTile t = decode_mean_tile(P, tile, li, kMmaPixels, kMeanMmaTokens);
    const JointParams& L = P.layer[t.li];
    const int d = L.head_dim, dpad = (d + 15) & ~15, ld = dpad + 8, buffer = 2 * kMmaPixels * ld;
    const bool vec = L.vec_ok != 0;
    const uint16_t* qb = static_cast<const uint16_t*>(L.q) + t.prompt * L.qs_prompt + (long long)t.pixel0 * L.qs_pixel;
    const uint16_t* kb = static_cast<const uint16_t*>(L.k) + t.prompt * L.ks_prompt + (long long)t.token0 * L.ks_token;
    float* acc = L.acc + (long long)t.prompt * L.tokens * L.hw;
    const bool pair = (L.hw & 1) == 0;
    const int px = t.pixel0 + 2 * tig;
    const int row = t.token0 + 16 * warp + g;          // this thread's first token row, in the sample
    const bool live = t.token0 + 16 * warp < L.tokens; // the warp has a row to accumulate
    auto stage_head = [&](int h, int buf) {
      uint16_t* qs = smem16 + buf * buffer;
      stage16_async(qb + h * L.qs_head, L.qs_pixel, L.hw - t.pixel0, d, dpad, ld, vec, qs);
      stage16_async(kb + h * L.ks_head, L.ks_token, L.tokens - t.token0, d, dpad, ld, vec, qs + kMmaPixels * ld);
      stage_lse_async(L, t.prompt, h, t.pixel0, kMmaPixels, lse_s[buf]);
      cp_async_commit();
    };
    float sum[8][4], old[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) sum[nt][0] = sum[nt][1] = sum[nt][2] = sum[nt][3] = 0.f;

    __syncthreads();                                   // the previous tile's readers are done with both buffers
    stage_head(0, 0);
    for (int h = 0; h < L.heads; ++h) {
      if (h + 1 < L.heads) {
        stage_head(h + 1, (h + 1) & 1);
        cp_async_wait<1>();
      } else {
        cp_async_wait<0>();
      }
      __syncthreads();                                 // head h's buffer is complete for every thread
      if (live) {
        const uint16_t* qs = smem16 + (h & 1) * buffer;
        const uint16_t* ks = qs + kMmaPixels * ld;
        if (h == L.heads - 1) {                        // the accumulator's latency hides under the last head
          if (pair) load_block<true>(acc, L.hw, L.tokens, row, px, old);
          else load_block<false>(acc, L.hw, L.tokens, row, px, old);
        }
        float s[8][4];
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
        const float* l = lse_s[h & 1] + 2 * tig;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
          const float l0 = l[nt * 8] * kLog2e, l1 = l[nt * 8 + 1] * kLog2e;
          sum[nt][0] += fast_exp2(fmaf(s[nt][0], L.c, -l0));
          sum[nt][1] += fast_exp2(fmaf(s[nt][1], L.c, -l1));
          sum[nt][2] += fast_exp2(fmaf(s[nt][2], L.c, -l0));
          sum[nt][3] += fast_exp2(fmaf(s[nt][3], L.c, -l1));
        }
      }
      __syncthreads();                                 // every warp is done with buffer h & 1: head h + 2 goes there
    }
    if (live) {
      if (pair) store_mean_block<true>(acc, L.hw, L.tokens, row, px, old, sum, (float)L.heads);
      else store_mean_block<false>(acc, L.hw, L.tokens, row, px, old, sum, (float)L.heads);
    }
  }
}

size_t mean_mma_smem_bytes(int dmax) { return 2 * mma_smem_bytes(dmax); }

__global__ void __launch_bounds__(kSimtPixels) accumulate_joint_mean_simt_kernel(const __grid_constant__ JointLaunch P) {
  extern __shared__ __align__(16) float smem32[];
  __shared__ float l2[kSimtPixels];
  int li = 0;
  for (int tile = blockIdx.x; tile < P.total_tiles; tile += gridDim.x) {
    const MeanTile t = decode_mean_tile(P, tile, li, kSimtPixels, kMeanSimtTokens);
    const JointParams& L = P.layer[t.li];
    const int d = L.head_dim;
    float* qs = smem32;                                // [128][d + 1]
    float* ks = smem32 + kSimtPixels * (d + 1);        // [32][d]
    const float* qb = static_cast<const float*>(L.q) + t.prompt * L.qs_prompt;
    const float* kb = static_cast<const float*>(L.k) + t.prompt * L.ks_prompt + (long long)t.token0 * L.ks_token;
    float* acc = L.acc + ((long long)t.prompt * L.tokens + t.token0) * L.hw;
    const int pixel = t.pixel0 + threadIdx.x;
    const bool live = pixel < L.hw;
    const int n = min(kMeanSimtTokens, L.tokens - t.token0);
    float sum[kMeanSimtTokens];
#pragma unroll
    for (int j = 0; j < kMeanSimtTokens; ++j) sum[j] = 0.f;
    for (int h = 0; h < L.heads; ++h) {
      __syncthreads();                                 // every thread is done with the previous head's operands
      for (int i = threadIdx.x; i < kSimtPixels * d; i += kSimtPixels) {
        const int r = i / d, e = i % d, x = t.pixel0 + r;
        qs[r * (d + 1) + e] = x < L.hw ? qb[h * L.qs_head + x * L.qs_pixel + e] : 0.f;
      }
      for (int i = threadIdx.x; i < kMeanSimtTokens * d; i += kSimtPixels) {
        const int r = i / d, e = i % d;
        ks[i] = r < n ? kb[h * L.ks_head + r * L.ks_token + e] : 0.f;
      }
      stage_lse(L, TileRef{t.li, t.prompt, h, t.pixel0}, kSimtPixels, l2);
      __syncthreads();
      const float l = l2[threadIdx.x];
      const float* qrow = qs + threadIdx.x * (d + 1);
#pragma unroll
      for (int j0 = 0; j0 < kMeanSimtTokens; j0 += 8) {
        if (j0 >= n) break;
        float s[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) s[i] = 0.f;
        for (int e = 0; e < d; ++e) {
          const float qv = qrow[e];
#pragma unroll
          for (int i = 0; i < 8; ++i) s[i] = fmaf(qv, ks[(j0 + i) * d + e], s[i]);
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) sum[j0 + i] += fast_exp2(fmaf(s[i], L.c, -l));
      }
    }
    if (live) {
      const float heads = (float)L.heads;
#pragma unroll
      for (int j = 0; j < kMeanSimtTokens; ++j)
        if (j < n) acc[(long long)j * L.hw + pixel] = acc[(long long)j * L.hw + pixel] + __fdiv_rn(sum[j], heads);
    }
  }
}

static_assert(kMeanSimtTokens == kSimtTokens, "the head-reduced fp32 kernel stages K like the per-head one");

// ---- host -------------------------------------------------------------------------------------------------------

// `reduce`: the head-reduced form, acc [n_prompts][tokens][hw].
int validate(const daam_joint_layer& in, int i, bool reduce, const char* fn, JointParams* out) {
  if (!in.q || !in.k || !in.acc || !in.lse) { set_error("%s: layer %d has a null pointer", fn, i); return DAAM_E_INVALID; }
  if (in.dtype != DAAM_F32 && in.dtype != DAAM_F16 && in.dtype != DAAM_BF16) { set_error("%s: layer %d: unknown dtype %d", fn, i, in.dtype); return DAAM_E_INVALID; }
  if (in.n_prompts <= 0 || in.heads <= 0 || in.hw <= 0) { set_error("%s: layer %d: non-positive n_prompts / heads / hw", fn, i); return DAAM_E_INVALID; }
  if (reinterpret_cast<uintptr_t>(in.acc) % 16 != 0) { set_error("%s: layer %d: acc is not 16-byte aligned", fn, i); return DAAM_E_INVALID; }
  if (!(in.scale > 0.f)) { set_error("%s: layer %d: scale must be positive", fn, i); return DAAM_E_INVALID; }
  if (in.tokens < 1 || in.tokens > DAAM_JOINT_MAX_TOKENS) { set_error("%s: layer %d: tokens = %d, must be in [1, %d]", fn, i, in.tokens, DAAM_JOINT_MAX_TOKENS); return DAAM_E_UNSUPPORTED; }
  if (in.head_dim <= 0 || in.head_dim % 8 != 0 || in.head_dim > DAAM_MAX_HEAD_DIM) { set_error("%s: layer %d: head_dim = %d must be a multiple of 8 in (0, %d]", fn, i, in.head_dim, DAAM_MAX_HEAD_DIM); return DAAM_E_UNSUPPORTED; }
  const long long slab = (long long)in.n_prompts * (reduce ? 1 : in.heads) * in.tokens * in.hw;
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
  const int block = in.dtype == DAAM_F32 ? kMeanSimtTokens : kMeanMmaTokens;
  L.tiles_per_head = (in.hw + tile - 1) / tile;
  L.token_blocks = reduce ? (in.tokens + block - 1) / block : 1;
  L.acc_heads = reduce ? 1 : in.heads;
  L.tile_begin = 0;
  return DAAM_OK;
}

// Tiles of one layer: (sample, head, pixel run), or head-reduced (sample, pixel run, token block).
int layer_tiles(const JointParams& l, bool reduce) {
  return l.n_prompts * l.tiles_per_head * (reduce ? l.token_blocks : l.heads);
}

size_t slab_bytes(const JointParams& l) { return sizeof(float) * (size_t)l.n_prompts * l.acc_heads * l.tokens * l.hw; }

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

int launch(JointLaunch& p, bool simt, bool reduce, const DeviceInfo& dev, cudaStream_t stream) {
  if (p.n_layers == 0) return DAAM_OK;
  int dmax = 0;
  for (int i = 0; i < p.n_layers; ++i) dmax = p.layer[i].head_dim > dmax ? p.layer[i].head_dim : dmax;
  const bool bf16 = p.layer[0].dtype == DAAM_BF16;
  const void* kernel;
  if (reduce)
    kernel = simt ? (const void*)accumulate_joint_mean_simt_kernel
                  : bf16 ? (const void*)accumulate_joint_mean_mma_kernel<true>
                         : (const void*)accumulate_joint_mean_mma_kernel<false>;
  else
    kernel = simt ? (const void*)accumulate_joint_simt_kernel
                  : bf16 ? (const void*)accumulate_joint_mma_kernel<true> : (const void*)accumulate_joint_mma_kernel<false>;
  const size_t smem = simt ? simt_smem_bytes(dmax) : reduce ? mean_mma_smem_bytes(dmax) : mma_smem_bytes(dmax);
  int grid = 0;
  if (int rc = grid_for(kernel, dev.device, dev.sm_count, smem, p.total_tiles, &grid)) return rc;
  void* args[] = {&p};
  DAAM_CUDA_TRY(cudaLaunchKernel(kernel, dim3(grid), dim3(128), args, smem, stream));
  count_launch();
  p.n_layers = 0;
  p.total_tiles = 0;
  return DAAM_OK;
}

// Both entry points: validate every layer, then class by class (16-bit on tensor cores: fp16 and bf16 are separate
// kernels; then fp32), each layer in call order; a layer whose accumulator overlaps one already in the launch, or a
// full launch, starts the next launch.
int accumulate_joint(const daam_joint_layer* layers, int32_t n_layers, uint32_t flags, void* stream_, bool reduce,
                     const char* fn) {
  if (n_layers < 0 || (n_layers > 0 && !layers)) { set_error("%s: bad layer array", fn); return DAAM_E_INVALID; }
  if (flags != 0) { set_error("%s: flags = %u, none are defined (pass 0)", fn, flags); return DAAM_E_INVALID; }
  std::vector<JointParams> all((size_t)n_layers);
  for (int i = 0; i < n_layers; ++i)
    if (int rc = validate(layers[i], i, reduce, fn, &all[i])) return rc;
  if (n_layers == 0) return DAAM_OK;
  DeviceInfo dev;
  if (int rc = get_device_info(&dev)) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  static thread_local JointLaunch p;
  for (int cls : {DAAM_F16, DAAM_BF16, DAAM_F32}) {
    p.n_layers = 0;
    p.total_tiles = 0;
    for (const JointParams& L : all) {
      if (L.dtype != cls) continue;
      bool full = p.n_layers == kJointMaxLayers;
      for (int m = 0; m < p.n_layers && !full; ++m) full = overlap(p.layer[m], L);
      if (full)
        if (int rc = launch(p, cls == DAAM_F32, reduce, dev, stream)) return rc;
      JointParams& slot = p.layer[p.n_layers++];
      slot = L;
      slot.tile_begin = p.total_tiles;
      p.total_tiles += layer_tiles(L, reduce);
    }
    if (int rc = launch(p, cls == DAAM_F32, reduce, dev, stream)) return rc;
  }
  return DAAM_OK;
}

}  // namespace
}  // namespace daam

using namespace daam;

extern "C" int daam_accumulate_joint(const daam_joint_layer* layers, int32_t n_layers, uint32_t flags, void* stream) {
  return daam::accumulate_joint(layers, n_layers, flags, stream, false, "daam_accumulate_joint");
}

extern "C" int daam_accumulate_joint_heads(const daam_joint_layer* layers, int32_t n_layers, uint32_t flags,
                                           void* stream) {
  return daam::accumulate_joint(layers, n_layers, flags, stream, true, "daam_accumulate_joint_heads");
}
