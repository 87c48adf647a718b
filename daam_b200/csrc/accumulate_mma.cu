// Fused softmax(QK^T) -> unravel -> accumulate, Hopper wgmma / TMA variant (head_dim up to 256 in 64-wide K chunks).
//
// One tile = 128 pixels x 77 tokens of one (layer, prompt, head). Per tile:
//   TMA        Q tile [128 x 64] and K [77(+3 zero rows) x 64] -> shared memory, 128B-swizzled K-major (the wgmma
//              canonical layout), straight from the strided `to_q`/`to_k` outputs via 4-D tensor maps
//              {dim, head, row, prompt}; partial tiles and the 3 padding token rows are zero-filled by the TMA unit.
//   wgmma      S = Q K^T: each of the two consumer warpgroups issues wgmma.m64n80k16 (fp32 accumulate) over its 64
//              pixel rows of the tile, K^T shared; the 64 x 80 logits land in registers (40 per thread).
//   epilogue   softmax over the 77 tokens of each pixel row (a row lives in the 4 threads of a quad: two shuffles per
//              reduction), then the probabilities are added into the tile's block of the fp32 accumulator
//              acc[head][token][pixel] ([77][128]) in shared memory: a separate loader warp has already brought that
//              block in by TMA, up to kAccStages tiles ahead, and one bulk-tensor store writes it back. The accumulator
//              is read from HBM well before the tile needs it, and the SM never waits for an L2 read-modify-write.
// Warp roles: 0-7 consumers (two warpgroups: MMA + softmax + accumulate), 8 Q/K TMA producer (one elected thread) that
// runs up to two K chunks ahead through a two-stage ring, 9 accumulator loader (one elected thread). Persistent, one CTA
// per SM (the rings fill its shared memory): in the single-chunk 16-bit instances CTA b takes tiles b, b + grid, ...,
// so the tiles in flight at any moment are consecutive (whole accumulator rows and the heads of a Q row move together);
// the others walk contiguous chunks of the launch's tiles. Accumulator loads and stores carry an L2 evict_first hint:
// each block is read and written once per launch, and the hint keeps them from pushing out the Q/K lines below.
//
// fp32 projections (the reference's default dtype for SD-1.x/2.x, daam/run/generate.py:205) take the same kernel in
// "split" form. Tensor cores have no fp32 operand type and a plain tf32 product would drop 13 mantissa bits, so every
// value is used as two tf32 terms, x = hi + lo with hi = trunc_tf32(x) and lo = rna_tf32(x - hi) (22 significand bits),
// and q.k = q_lo.k_hi + q_hi.k_lo + q_hi.k_hi (the dropped terms are ~2^-22 relative): the fp32 Q/K tiles arrive by TMA
// exactly like the 16-bit ones (two 128-byte-wide swizzled sub-tiles per 64 dims); the consumer threads rewrite them
// in place as hi and emit `lo` into a second buffer (a shared-memory -> shared-memory elementwise pass, swizzle-
// agnostic), then issue 3 x 8 wgmma.m64n80k8 tf32 per chunk. One CTA per SM (two 52 KB raw stages + one lo buffer +
// the staged probabilities). Its shared memory has no room for an accumulator ring, so the staged probabilities go to
// the accumulator either
//   red mode : as ONE bulk-tensor reduce-add (cp.reduce.async.bulk.tensor .add.f32): the read-modify-write happens in
//              L2, the SM never loads the accumulator;
//   ldst mode: coalesced 16-byte load / add / store of the staged tile by all consumer threads.
//
// head_dim other than 64 (SD-1.x: 40 / 80 / 160): the contraction runs in 64-wide K chunks, one chunk per smem stage,
// accumulated into the same registers; the last chunk is zero-filled beyond head_dim by the TMA unit.
//
// Step-slab instances (kSlab == kSlabStore, daam_accumulate_steps): every form also STORES what it adds into a second
// fp32 slab of the accumulator's layout, flushed like the add, so that a caller gets one denoising step's maps next to
// the time sum.
//   16-bit form: one more [77][128] shared block sS; the consumers write p there in the pass that adds into the ring
//                slot, and the thread that stores the accumulator tile issues a second bulk-tensor store from sS in the
//                same bulk group. Before sS is rewritten, that thread waits for the previous group's reads.
//   split form : red mode stages the flushed p in sP (the reduce flushes its inputs anyway) and bulk-stores sP next to
//                the reduce; ldst mode writes p to the step slab in its coalesced load / add / store pass.
// Range-slab instances (kSlab == kSlabAdd, daam_accumulate_range): every form also ADDS what it adds into a second slab,
// with the arithmetic it applies to the accumulator, so that a slab zeroed before a span of steps ends up holding
// exactly the accumulator a trace of only those steps would hold.
//   16-bit form: sS as in the step form (p flushed, as add.rn.ftz sees it); in place of the step store, a bulk-tensor
//                reduce-add from sS into the range slab, in the same bulk group (the reduce flushes like add.rn.ftz).
//   split form : red mode issues a second reduce-add from sP; ldst mode loads, adds and stores the range slab in its
//                coalesced pass, like the accumulator.
//
// Long-context instances (kC = 2 or 3 chunks of 77 tokens: 154- / 231-token contexts, 16-bit form, plain slab mode):
// a stage holds the Q box and kC K boxes [80 x 64], loaded at token rows 77c of the same 4-D map (token extent = the
// context); columns 77-79 of a box hold the next chunk's first tokens (or TMA zeros after the last one), which the
// column masks exclude exactly as they exclude the zero rows of a 77-token box. The consumers issue kC sets of
// wgmma.m64n80k16 into kC fragments, take max and sum over all of them, then add chunk c's probabilities into one ring
// slot per chunk (accumulator rows (p H + h) 77 kC + 77 c): a tile consumes kC consecutive slots of the same 3-slot
// ring, each with the single-chunk epilogue.
//
// Replaces daam/trace.py:276 (get_attention_scores), :219-244 (_unravel_attn) and :293-294 (update loop).
#include <cuda.h>

#include <mutex>
#include <type_traits>
#include <unordered_map>
#include <string>

#include "common.cuh"

namespace daam {
namespace {

constexpr int kStages = 2;                            // Q/K chunk ring
constexpr int kAccStages = 3;                         // 16-bit form: accumulator tile ring
constexpr int kPrefetchTiles = 6;                     // 16-bit form, early loads: tiles whose Q/K go to L2 before the wait
constexpr int kQBytes = kTilePixels * 128;            // 128 rows x 128 B (64 x 16-bit, or 32 x fp32: one swizzle span)
constexpr int kKBytes = kTokensPad * 128;             // 80 rows x 128 B
constexpr int kStageBytes = kQBytes + kKBytes;        // 26624 = 26 x 1024 (keeps every tile 1024-byte aligned)
constexpr int kPBytes = kTokens * kTilePixels * 4;    // one accumulator / probability tile [77][128] fp32 (128 x 308 B)
constexpr int kConsumers = 256;                       // two warpgroups, 64 pixel rows each
constexpr int kThreads = kConsumers + 32;             // split form: + the TMA producer warp
constexpr int kThreads16 = kConsumers + 64;           // 16-bit form: + the Q/K producer warp + the accumulator loader warp
constexpr int kBarBytes = 64;                         // split form: mbarriers
constexpr int kBarBytes16 = 8 * 2 * (kStages + kAccStages);
constexpr int kSmemBytes = 1024 + kStages * kStageBytes + kAccStages * kPBytes + kBarBytes16;
constexpr int kSlabSmemBytes = kSmemBytes + kPBytes;  // 16-bit form with a second slab: + the sS block (207.5 KB)
// split (fp32) form: a raw stage holds the fp32 tiles as [Q sub0][Q sub1][K sub0][K sub1] (sub-tile = 32 floats = one
// 128-byte swizzle span per row); one more buffer of the same shape holds the lo terms
constexpr int kSplitStageBytes = 2 * kStageBytes;     // 53248 = 52 x 1024
constexpr int kSplitSmemBytes = 1024 + (kStages + 1) * kSplitStageBytes + kPBytes + kBarBytes;
static_assert(kSmemBytes <= 232448, "16-bit form exceeds the 227 KB shared-memory limit");
static_assert(kSplitSmemBytes <= 232448, "split form exceeds the 227 KB shared-memory limit");
static_assert(kSlabSmemBytes <= 232448, "16-bit second-slab form exceeds the 227 KB shared-memory limit");
// 16-bit long-context form: kC K boxes per stage (kC = 3: 2 x 46 KB of stages + 3 x 38.5 KB of ring, 208.6 KB)
constexpr int long_smem_bytes(int chunks) {
  return 1024 + kStages * (kQBytes + chunks * kKBytes) + kAccStages * kPBytes + kBarBytes16;
}
static_assert(long_smem_bytes(3) <= 232448, "16-bit long-context form exceeds the 227 KB shared-memory limit");

struct MmaParams {
  LaunchParams base;
  CUtensorMap qmap[kMaxLayersPerLaunch];
  CUtensorMap kmap[kMaxLayersPerLaunch];
  CUtensorMap amap[kMaxLayersPerLaunch];
};
// Parameter block of the second-slab instances (about 20 KB): the second slab of every layer as a tensor map shaped
// like amap (bulk stores and reduces) and as a plain pointer (split form, ldst mode).
struct MmaSlabParams : MmaParams {
  CUtensorMap smap[kMaxLayersPerLaunch];
  float* slab[kMaxLayersPerLaunch];
};
template <bool kSecond>
using MmaParamsT = std::conditional_t<kSecond, MmaSlabParams, MmaParams>;

// ---- PTX wrappers -------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug traps (reported as a CUDA error) instead of hanging the GPU. The bound is ~10 s of SM
// clocks, far beyond any legitimate wait on a dedicated GPU; where a context can be descheduled for longer (MPS,
// time-slicing, a debugger) build with -DDAAM_MBAR_TIMEOUT_CYCLES=0 to wait without a bound.
#ifndef DAAM_MBAR_TIMEOUT_CYCLES
#define DAAM_MBAR_TIMEOUT_CYCLES 20000000000LL
#endif
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try(bar, parity)) return;
#if DAAM_MBAR_TIMEOUT_CYCLES > 0
  const long long t0 = clock64();
  while (!mbar_try(bar, parity)) {
    if (clock64() - t0 > DAAM_MBAR_TIMEOUT_CYCLES) __trap();
  }
#else
  while (!mbar_try(bar, parity)) {}
#endif
}

__device__ __forceinline__ void tma_load_4d(const CUtensorMap* map, uint32_t bar, uint32_t dst, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, uint32_t src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(map)),
               "r"(src), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_reduce_add_2d(const CUtensorMap* map, uint32_t src, int c0, int c1) {
  asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(map)),
               "r"(src), "r"(c0), "r"(c1)
               : "memory");
}
// L2 eviction-priority policies for the .L2::cache_hint forms below
__device__ __forceinline__ uint64_t l2_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t l2_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
// The box a tma_load_4d with the same coordinates would fetch, into L2 only (no shared memory, no barrier)
__device__ __forceinline__ void tma_prefetch_4d(const CUtensorMap* map, int c0, int c1, int c2, int c3, uint64_t pol) {
  asm volatile("cp.async.bulk.prefetch.tensor.4d.L2.global.tile.L2::cache_hint [%0, {%1, %2, %3, %4}], %5;"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "l"(pol)
               : "memory");
}
__device__ __forceinline__ void tma_load_2d_hint(const CUtensorMap* map, uint32_t bar, uint32_t dst, int c0, int c1,
                                                 uint64_t pol) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4}], "
      "[%2], %5;"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1), "l"(pol)
      : "memory");
}
__device__ __forceinline__ void tma_store_2d_hint(const CUtensorMap* map, uint32_t src, int c0, int c1, uint64_t pol) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group.L2::cache_hint [%0, {%2, %3}], [%1], %4;" ::"l"(
                   reinterpret_cast<uint64_t>(map)),
               "r"(src), "r"(c0), "r"(c1), "l"(pol)
               : "memory");
}
__device__ __forceinline__ void prefetch_tensormap(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read1() { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void consumer_barrier() { asm volatile("bar.sync 1, %0;" ::"n"(kConsumers) : "memory"); }

// wgmma shared-memory descriptor: K-major operand tile, 128B swizzle, rows of 128 bytes, 8-row groups 1024 B apart.
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t smem_addr) {
  return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | (1ull << 16) /* LBO (unused with swizzle) */ |
         ((uint64_t)(1024 >> 4) << 32) /* SBO */ | (1ull << 62) /* SWIZZLE_128B */;
}

// The 64 x 80 fp32 accumulator fragment of one warpgroup: thread (warp w, lane l) holds rows 16w + l/4 (+ 8) and
// columns 8j + 2(l%4) (+ 1) as d[4j + {0, 1}] (row r0) and d[4j + {2, 3}] (row r0 + 8), j = 0..9.
using Frag = float[40];

__device__ __forceinline__ void frag_fence(Frag& d) {
#pragma unroll
  for (int i = 0; i < 40; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

#define DAAM_FRAG_OPERANDS                                                                                          \
  "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),         \
      "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),          \
      "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),         \
      "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),         \
      "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
#define DAAM_FRAG_REGS                                                                                              \
  "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, " \
  "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39}"

// d += A[64 x 16] B[80 x 16]^T, both K-major in shared memory; 16-bit operands (fp16 or bf16)
template <bool kBf16>
__device__ __forceinline__ void wgmma_16bit(Frag& d, uint64_t adesc, uint64_t bdesc) {
  if constexpr (kBf16)
    asm volatile("wgmma.mma_async.sync.aligned.m64n80k16.f32.bf16.bf16 " DAAM_FRAG_REGS ", %40, %41, 1, 1, 1, 0, 0;"
                 : DAAM_FRAG_OPERANDS
                 : "l"(adesc), "l"(bdesc)
                 : "memory");
  else
    asm volatile("wgmma.mma_async.sync.aligned.m64n80k16.f32.f16.f16 " DAAM_FRAG_REGS ", %40, %41, 1, 1, 1, 0, 0;"
                 : DAAM_FRAG_OPERANDS
                 : "l"(adesc), "l"(bdesc)
                 : "memory");
}
// d += A[64 x 8] B[80 x 8]^T with tf32 operands (32-bit containers, K = 8 = 32 bytes along the swizzled row)
__device__ __forceinline__ void wgmma_tf32(Frag& d, uint64_t adesc, uint64_t bdesc) {
  asm volatile("wgmma.mma_async.sync.aligned.m64n80k8.f32.tf32.tf32 " DAAM_FRAG_REGS ", %40, %41, 1, 1, 1;"
               : DAAM_FRAG_OPERANDS
               : "l"(adesc), "l"(bdesc)
               : "memory");
}

struct Tile {
  int li, prompt, head, pixel0;
};
__device__ __forceinline__ Tile decode_tile(const LaunchParams& P, int tile, int& li) {
  while (li + 1 < P.n_layers && tile >= P.layer[li + 1].tile_begin) ++li;
  const LayerParams& L = P.layer[li];
  const int local = tile - L.tile_begin;
  const int ptile = local % L.tiles_per_head;
  const int ph = local / L.tiles_per_head;
  Tile t;
  t.li = li;
  t.head = ph % L.heads;
  t.prompt = ph / L.heads;
  t.pixel0 = ptile * kTilePixels;
  return t;
}

// First tile whose weight offset (tiles before it x their weights) is >= w; total_tiles for w >= total_weight.
__device__ __forceinline__ int tile_at_weight(const LaunchParams& P, long long w) {
  if (w >= P.total_weight) return P.total_tiles;
  int li = 0;
  while (li + 1 < P.n_layers && w >= P.layer[li + 1].weight_begin) ++li;
  const LayerParams& L = P.layer[li];
  return L.tile_begin + (int)((w - L.weight_begin + L.weight - 1) / L.weight);
}

__device__ __forceinline__ float rna_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}
__device__ __forceinline__ float trunc_tf32(float x) { return __uint_as_float(__float_as_uint(x) & 0xffffe000u); }

// Split pass (fp32 form): for a landed fp32 region [begin, end) of a raw stage (16-byte units, any swizzle -- the pass
// is elementwise) write hi = trunc_tf32(x) in place and lo = rna_tf32(x - hi) to the same offsets of the lo buffer.
// Both are exact tf32 values, so the product does not depend on how the tensor core reads the low 13 bits of a
// container. x - trunc_tf32(x) is exact in fp32 (13 significant bits), so hi + lo carries 22 significand bits of x.
// Four units per thread are loaded before the first is processed.
__device__ __forceinline__ void split_region(uint8_t* raw, uint8_t* lo, int begin, int end, int ctid, int n_conv) {
  const int stride = n_conv * 16;
  for (int off = begin + ctid * 16; off < end; off += 4 * stride) {
    float4 x[4];
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (off + u * stride < end) x[u] = *reinterpret_cast<const float4*>(raw + off + u * stride);
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (off + u * stride < end) {
        float4 h, l;
        h.x = trunc_tf32(x[u].x); h.y = trunc_tf32(x[u].y); h.z = trunc_tf32(x[u].z); h.w = trunc_tf32(x[u].w);
        l.x = rna_tf32(x[u].x - h.x); l.y = rna_tf32(x[u].y - h.y);
        l.z = rna_tf32(x[u].z - h.z); l.w = rna_tf32(x[u].w - h.w);
        *reinterpret_cast<float4*>(raw + off + u * stride) = h;
        *reinterpret_cast<float4*>(lo + off + u * stride) = l;
      }
  }
}

// One 64-wide K chunk of 16-bit operands: 4 x wgmma.m64n80k16, committed and waited for as one group.
template <bool kBf16>
__device__ __forceinline__ void wgmma_chunk_16bit(Frag& d, uint32_t a_src, uint32_t k_src) {
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < 4; ++k) wgmma_16bit<kBf16>(d, wgmma_desc_sw128(a_src + 32 * k), wgmma_desc_sw128(k_src + 32 * k));
  wgmma_commit();
  wgmma_wait0();
}
// The same over the kC K boxes of a long-context stage (box c at k_src + c * kKBytes), into kC fragments, one group.
template <bool kBf16, int kC>
__device__ __forceinline__ void wgmma_chunk_16bit_long(Frag (&d)[kC], uint32_t a_src, uint32_t k_src) {
  wgmma_fence();
#pragma unroll
  for (int c = 0; c < kC; ++c)
#pragma unroll
    for (int k = 0; k < 4; ++k)
      wgmma_16bit<kBf16>(d[c], wgmma_desc_sw128(a_src + 32 * k), wgmma_desc_sw128(k_src + c * kKBytes + 32 * k));
  wgmma_commit();
  wgmma_wait0();
}

__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// kChunked: some layer of the launch has head_dim > 64 (several K chunks per tile); the common single-chunk case keeps
// its simpler loops (one load iteration per tile). kSlab: also store (kSlabStore) or add (kSlabAdd) each tile's
// probabilities into the second slab. kC: 77-token chunks of the context (1, or 2 / 3 in the long-context instances).
template <bool kSplit, bool kChunked, int kSlab, int kC = 1>
__global__ void __launch_bounds__(kSplit ? kThreads : kThreads16, 1)
accumulate_mma_kernel(const __grid_constant__ MmaParamsT<kSlab != kSlabNone> MP) {
  static_assert(kC == 1 || (!kSplit && kSlab == kSlabNone), "long contexts: 16-bit form, plain slab mode only");
  constexpr bool kSecond = kSlab != kSlabNone;        // a second slab (store or add)
  constexpr int kCtx = kC * kTokens;                  // context rows: the accumulator's token extent
  constexpr int kStageBytesT = kSplit ? kSplitStageBytes : kQBytes + kC * kKBytes;
  constexpr int kOperandBytes = (kSplit ? kStages + 1 : kStages) * kStageBytesT;     // stages (+ the lo buffer)
  // staged probabilities (split) / the accumulator ring (16-bit), + sS (16-bit form with a second slab)
  constexpr int kPTiles = kSplit ? 1 : kAccStages + (kSecond ? 1 : 0);
  const LaunchParams& P = MP.base;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;                       // 1024-byte alignment for the swizzled tiles
  uint8_t* gen = smem_raw + (base - raw);
  float* sP = reinterpret_cast<float*>(gen + kOperandBytes);
  const uint32_t sP_u32 = base + kOperandBytes;
  float* sS = sP + kAccStages * (kTokens * kTilePixels);              // 16-bit second-slab form: the tile's p
  const uint32_t sS_u32 = sP_u32 + kAccStages * kPBytes;
  const uint32_t bars = sP_u32 + kPTiles * kPBytes;
  const uint32_t full0 = bars, empty0 = bars + 8 * kStages;           // Q/K ring
  const uint32_t afull0 = bars + 16 * kStages, aempty0 = afull0 + 8 * kAccStages;   // accumulator ring (16-bit form)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int first, count, stride = 1;                        // the CTA's tiles: first + i * stride, i < count (increasing)
  if constexpr (!kChunked && !kSplit) {               // equal tiles, interleaved: the grid works on consecutive tiles
    first = blockIdx.x;
    stride = gridDim.x;
    count = (P.total_tiles - (int)blockIdx.x + stride - 1) / stride;
  } else if constexpr (!kChunked) {                    // equal tiles: contiguous ranges of per / per + 1 tiles
    const int per = P.total_tiles / gridDim.x, rem = P.total_tiles % gridDim.x;
    first = blockIdx.x * per + min((int)blockIdx.x, rem);
    count = per + ((int)blockIdx.x < rem ? 1 : 0);
  } else {                                             // tiles of several K-chunk counts: contiguous ranges of equal WEIGHT
    first = tile_at_weight(P, (long long)P.total_weight * blockIdx.x / gridDim.x);
    count = tile_at_weight(P, (long long)P.total_weight * (blockIdx.x + 1) / gridDim.x) - first;
  }

  if (threadIdx.x == 0) {
#pragma unroll
    for (int s = 0; s < kStages; ++s) {
      mbar_init(full0 + 8 * s, 1);
      mbar_init(empty0 + 8 * s, kConsumers / 32);    // one arrival per consumer warp
    }
    if constexpr (!kSplit) {
#pragma unroll
      for (int s = 0; s < kAccStages; ++s) {
        mbar_init(afull0 + 8 * s, 1);
        mbar_init(aempty0 + 8 * s, 1);               // the consumer thread that stored the tile
      }
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // descriptor fetches of the first tile overlap the barrier set-up (and, under PDL, the previous kernel's tail)
  if (count > 0 && lane == 0 && (warp == (kSplit ? 0 : 9) || warp == 8)) {
    int li0 = 0;
    const Tile t0 = decode_tile(P, first, li0);
    if (warp != 8) {
      prefetch_tensormap(&MP.amap[t0.li]);
      if constexpr (kSecond) prefetch_tensormap(&MP.smap[t0.li]);
    } else {
      prefetch_tensormap(&MP.qmap[t0.li]);
      prefetch_tensormap(&MP.kmap[t0.li]);
    }
  }
  __syncthreads();
  // Programmatic dependent launch: everything above (barrier init, descriptor prefetch) may overlap the tail of the
  // previous kernel on the stream. By default nothing below starts before that kernel has completed and flushed.
  // With `early_loads` (the caller vouches that Q/K were complete before the previous kernel started, DAAM_ACC_EARLY_LOADS)
  // only the accumulator traffic waits (16-bit form: the accumulator loader's first load; split form: the first
  // reduce): Q/K loads, MMAs and the first tiles' softmax overlap the previous kernel's tail. The same promise makes
  // the 16-bit producer's L2 prefetch of its next tiles' Q/K legal before the wait: the previous kernel only writes
  // accumulators, so those bytes are final, and a prefetch reads nothing into shared memory that could go stale.
  // Our own dependents may be scheduled as soon as every CTA of this grid is past this point.
  if (!P.early_loads) griddep_wait();
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");

  if (warp == 9) {
    // ===== accumulator loader (16-bit form): the CTA's accumulator tiles, in order, through the kAccStages ring =====
    if constexpr (!kSplit) {
      if (lane == 0 && count > 0) {
        if (P.early_loads) griddep_wait();           // everything the previous kernel added is complete and visible
        const uint64_t pol = l2_evict_first();
        int li = 0;
        for (int i = 0; i < count; ++i) {
          const Tile t = decode_tile(P, first + i * stride, li);
#pragma unroll
          for (int c = 0; c < kC; ++c) {             // one ring slot per 77-token chunk of the tile
            const int n = i * kC + c;
            const int a = n % kAccStages;
            mbar_wait(aempty0 + 8 * a, ((uint32_t)(n / kAccStages) & 1u) ^ 1u);   // its previous tile's store has read it
            mbar_expect_tx(afull0 + 8 * a, kPBytes);   // (a partial tile's out-of-range pixels land as zeros)
            tma_load_2d_hint(&MP.amap[t.li], afull0 + 8 * a, sP_u32 + a * kPBytes, t.pixel0,
                             (t.prompt * P.layer[t.li].heads + t.head) * kCtx + c * kTokens, pol);
          }
        }
      }
    }
  } else if (warp == 8) {
    // ===== TMA producer =====
    if (lane == 0) {
      int li = 0, j = 0;
      for (int i = 0; i < count; ++i) {
        if (!kSplit && P.early_loads && i == (kChunked ? 1 : kStages)) {
          // the first tiles' stages are loaded; before waiting for a free stage (and, on a CTA that starts early, for
          // the previous launch), pull the Q boxes of the next kPrefetchTiles tiles and the K box of every new head
          // into L2 at evict_last priority, with the coordinates of the loads that will read them
          const uint64_t pol = l2_evict_last();
          const int end = min(count, i + kPrefetchTiles);
          int pli = 0;
          Tile prev = decode_tile(P, first + (i - 1) * stride, pli);         // its K is loaded already
          for (int p = i; p < end; ++p) {
            const Tile u = decode_tile(P, first + p * stride, pli);
            const bool new_head = u.li != prev.li || u.prompt != prev.prompt || u.head != prev.head;
            const int nc = kChunked ? (P.layer[u.li].head_dim + 63) >> 6 : 1;
            for (int c = 0; c < nc; ++c) {
              tma_prefetch_4d(&MP.qmap[u.li], 64 * c, u.head, u.pixel0, u.prompt, pol);
              if (new_head)
#pragma unroll
                for (int kc = 0; kc < kC; ++kc) tma_prefetch_4d(&MP.kmap[u.li], 64 * c, u.head, kc * kTokens, u.prompt, pol);
            }
            prev = u;
          }
        }
        const Tile t = decode_tile(P, first + i * stride, li);
        const int n_chunks = kChunked ? (P.layer[t.li].head_dim + 63) >> 6 : 1;
        for (int c = 0; c < n_chunks; ++c, ++j) {      // one load iteration = one 64-wide K chunk of one tile
          const int s = j % kStages;
          const uint32_t ph = (uint32_t)(j / kStages) & 1u;
          mbar_wait(empty0 + 8 * s, ph ^ 1u);
          const uint32_t q_dst = base + s * kStageBytesT;
          if constexpr (kSplit) {                      // fp32: two 32-float-wide boxes per operand
            const uint32_t k_dst = q_dst + 2 * kQBytes;          // (a box wholly beyond head_dim lands as zeros)
            mbar_expect_tx(full0 + 8 * s, kStageBytesT);
            tma_load_4d(&MP.qmap[t.li], full0 + 8 * s, q_dst, 64 * c, t.head, t.pixel0, t.prompt);
            tma_load_4d(&MP.kmap[t.li], full0 + 8 * s, k_dst, 64 * c, t.head, 0, t.prompt);
            tma_load_4d(&MP.qmap[t.li], full0 + 8 * s, q_dst + kQBytes, 64 * c + 32, t.head, t.pixel0, t.prompt);
            tma_load_4d(&MP.kmap[t.li], full0 + 8 * s, k_dst + kKBytes, 64 * c + 32, t.head, 0, t.prompt);
          } else {
            const uint32_t k_dst = q_dst + kQBytes;
            mbar_expect_tx(full0 + 8 * s, kStageBytesT);
            tma_load_4d(&MP.qmap[t.li], full0 + 8 * s, q_dst, 64 * c, t.head, t.pixel0, t.prompt);
#pragma unroll
            for (int kc = 0; kc < kC; ++kc)            // K box kc: token rows 77 kc .. 77 kc + 79
              tma_load_4d(&MP.kmap[t.li], full0 + 8 * s, k_dst + kc * kKBytes, 64 * c, t.head, kc * kTokens, t.prompt);
          }
        }
      }
    }
  } else {
    // ===== consumer warpgroups: MMA + softmax + accumulate =====
    const int tid = threadIdx.x;                       // 0..255
    const int wg = warp >> 2;                          // pixel rows 64 wg .. 64 wg + 63 of the tile
    const int quad = lane & 3;
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);            // this thread's rows: r0 and r0 + 8
    int li = 0, j = 0;
    bool issued = false;
    for (int i = 0; i < count; ++i) {
      const Tile t = decode_tile(P, first + i * stride, li);
      const LayerParams& L = P.layer[t.li];
      const int n_chunks = kChunked ? (L.head_dim + 63) >> 6 : 1;
      Frag dd[kC];                                     // the logits of 77-token chunk c in dd[c]
      Frag& d = dd[0];
#pragma unroll
      for (int kc = 0; kc < kC; ++kc)
#pragma unroll
        for (int e = 0; e < 40; ++e) dd[kc][e] = 0.f;
      for (int c = 0; c < n_chunks; ++c, ++j) {
        const int s = j % kStages;
        mbar_wait(full0 + 8 * s, (uint32_t)(j / kStages) & 1u);        // the chunk's operand tiles have landed
        const uint32_t q_src = base + s * kStageBytesT;
#pragma unroll
        for (int kc = 0; kc < kC; ++kc) frag_fence(dd[kc]);
        if constexpr (kSplit) {
          uint8_t* stage = gen + s * kStageBytesT;
          uint8_t* lo = gen + kStages * kStageBytesT;
          consumer_barrier();                          // both warpgroups' MMAs of the previous chunk have read lo
          split_region(stage, lo, 0, kSplitStageBytes, tid, kConsumers);
          fence_proxy_async();                         // generic-proxy stores -> visible to the tensor core's reads
          consumer_barrier();
          wgmma_fence();
          // q.k = q_lo.k_hi + q_hi.k_lo + q_hi.k_hi, smallest first; K = 8 floats = 32 bytes per instruction. Columns
          // beyond head_dim are zeros in both buffers, so all 24 MMAs run: the compiler serialises a wgmma that sits
          // behind a per-thread condition.
          const uint32_t q_lo = base + kStages * kStageBytesT;
          const uint32_t qa[3] = {q_lo, q_src, q_src};
          const uint32_t kb[3] = {q_src + 2 * kQBytes, q_lo + 2 * kQBytes, q_src + 2 * kQBytes};
#pragma unroll
          for (int p = 0; p < 3; ++p)
#pragma unroll
            for (int k = 0; k < 8; ++k)
              wgmma_tf32(d, wgmma_desc_sw128(qa[p] + (k >> 2) * kQBytes + wg * 64 * 128 + 32 * (k & 3)),
                         wgmma_desc_sw128(kb[p] + (k >> 2) * kKBytes + 32 * (k & 3)));
          wgmma_commit();
          wgmma_wait0();
        } else {
          // K 16 = 32 bytes along the swizzled row; columns beyond head_dim are zero-filled by TMA
          const uint32_t a_src = q_src + wg * 64 * 128, k_src = q_src + kQBytes;
          if constexpr (kC == 1) {
            if (L.dtype == DAAM_BF16)
              wgmma_chunk_16bit<true>(d, a_src, k_src);
            else
              wgmma_chunk_16bit<false>(d, a_src, k_src);
          } else {
            if (L.dtype == DAAM_BF16)
              wgmma_chunk_16bit_long<true, kC>(dd, a_src, k_src);
            else
              wgmma_chunk_16bit_long<false, kC>(dd, a_src, k_src);
          }
        }
#pragma unroll
        for (int kc = 0; kc < kC; ++kc) frag_fence(dd[kc]);
        __syncwarp();
        if (lane == 0) mbar_arrive(empty0 + 8 * s);    // this warp is done with the stage
      }

      // softmax over the 77 live columns of rows r0 (d[4j], d[4j+1]) and r0 + 8 (d[4j+2], d[4j+3]); columns 77..79
      // (zero-filled token rows) sit in j = 9 of quads 2 (odd column) and 3. Long contexts: the same over every chunk's
      // fragment (there columns 77..79 hold the next chunk's first tokens, masked alike).
      float m0 = d[0], m1 = d[2];
#pragma unroll
      for (int kc = 0; kc < kC; ++kc)
#pragma unroll
      for (int jj = 0; jj < 10; ++jj) {
        const bool l0 = jj < 9 || quad <= 2, l1 = jj < 9 || quad < 2;   // column 8jj+2q (+1) < 77
        if (l0) { m0 = fmaxf(m0, dd[kc][4 * jj]); m1 = fmaxf(m1, dd[kc][4 * jj + 2]); }
        if (l1) { m0 = fmaxf(m0, dd[kc][4 * jj + 1]); m1 = fmaxf(m1, dd[kc][4 * jj + 3]); }
      }
      m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 1));
      m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, 2));
      m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 1));
      m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, 2));
      const float sc = L.scale_log2e, mc0 = m0 * sc, mc1 = m1 * sc;
      float sum0 = 0.f, sum1 = 0.f;
#pragma unroll
      for (int kc = 0; kc < kC; ++kc)
#pragma unroll
      for (int jj = 0; jj < 10; ++jj) {
        const bool l0 = jj < 9 || quad <= 2, l1 = jj < 9 || quad < 2;
        float* f = dd[kc];
        f[4 * jj] = l0 ? fast_exp2(fmaf(f[4 * jj], sc, -mc0)) : 0.f;
        f[4 * jj + 2] = l0 ? fast_exp2(fmaf(f[4 * jj + 2], sc, -mc1)) : 0.f;
        f[4 * jj + 1] = l1 ? fast_exp2(fmaf(f[4 * jj + 1], sc, -mc0)) : 0.f;
        f[4 * jj + 3] = l1 ? fast_exp2(fmaf(f[4 * jj + 3], sc, -mc1)) : 0.f;
        sum0 += f[4 * jj] + f[4 * jj + 1];
        sum1 += f[4 * jj + 2] + f[4 * jj + 3];
      }
      sum0 += __shfl_xor_sync(0xffffffffu, sum0, 1);
      sum0 += __shfl_xor_sync(0xffffffffu, sum0, 2);
      sum1 += __shfl_xor_sync(0xffffffffu, sum1, 1);
      sum1 += __shfl_xor_sync(0xffffffffu, sum1, 2);
      const float inv0 = 1.0f / sum0, inv1 = 1.0f / sum1;

      if constexpr (!kSplit) {
        // Add the probabilities to the landed accumulator tile sA[token][pixel], then store it back with one bulk-tensor
        // store (clipped to the map for a partial tile). Quads 0-1 update row r0 while quads 2-3 update row r0 + 8 (and
        // then the other way round), so one access touches 16 banks instead of 8. All old values are loaded before the
        // first store: the compiler cannot tell the two rows apart and would otherwise serialise every load behind the
        // previous store. Long contexts: chunk kc of the tile goes through ring slot n = i kC + kc, with this epilogue.
#pragma unroll
        for (int kc = 0; kc < kC; ++kc) {
        const int n = i * kC + kc;
        const int a = n % kAccStages;
        float* sA = sP + a * (kTokens * kTilePixels);
        const bool lowq = quad < 2;
        const int ra = lowq ? r0 : r0 + 8, rb = lowq ? r0 + 8 : r0;
        mbar_wait(afull0 + 8 * a, (uint32_t)(n / kAccStages) & 1u);
        float old[40];
#pragma unroll
        for (int jj = 0; jj < 10; ++jj) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = 8 * jj + 2 * quad + e;
            if (col < kTokens) {
              old[4 * jj + e] = sA[col * kTilePixels + ra];
              old[4 * jj + 2 + e] = sA[col * kTilePixels + rb];
            }
          }
        }
        if constexpr (kSecond) {                       // the previous tile's second-slab store / reduce has read sS
          if (tid == 0 && i > 0) bulk_wait_read0();
          consumer_barrier();
        }
        const float* f = dd[kc];
#pragma unroll
        for (int jj = 0; jj < 10; ++jj) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int col = 8 * jj + 2 * quad + e;
            if (col < kTokens) {
              const float pa = f[4 * jj + e] * inv0, pb = f[4 * jj + 2 + e] * inv1;
              sA[col * kTilePixels + ra] = add_ftz(old[4 * jj + e], lowq ? pa : pb);
              sA[col * kTilePixels + rb] = add_ftz(old[4 * jj + 2 + e], lowq ? pb : pa);
              if constexpr (kSecond) {
                sS[col * kTilePixels + ra] = add_ftz(0.f, lowq ? pa : pb);
                sS[col * kTilePixels + rb] = add_ftz(0.f, lowq ? pb : pa);
              }
            }
          }
        }
        fence_proxy_async();                           // generic-proxy writes -> visible to the bulk-async proxy
        consumer_barrier();
        if (tid == 0) {
          tma_store_2d_hint(&MP.amap[t.li], sP_u32 + a * kPBytes, t.pixel0,
                            (t.prompt * L.heads + t.head) * kCtx + kc * kTokens, l2_evict_first());
          if constexpr (kSlab == kSlabStore)           // same bulk group: the waits below cover both stores
            tma_store_2d(&MP.smap[t.li], sS_u32, t.pixel0, (t.prompt * L.heads + t.head) * kTokens);
          if constexpr (kSlab == kSlabAdd)             // (and the range reduce: its reads of sS)
            tma_reduce_add_2d(&MP.smap[t.li], sS_u32, t.pixel0, (t.prompt * L.heads + t.head) * kTokens);
          bulk_commit();
          if (n > 0) {                                 // one store of slack: the previous tile's store has read its slot
            bulk_wait_read1();
            mbar_arrive(aempty0 + 8 * ((n - 1) % kAccStages));
          }
        }
        }
        continue;
      }

      // ---- split form: the probabilities are staged and reduce-added (or load/add/stored) into the accumulator ----
      // the first accumulator update of this CTA: everything the previous kernel added must be complete and visible
      if (i == 0 && P.early_loads) griddep_wait();

      // stage the probabilities token-major: sP[token][pixel]. Quads 0-1 store row r0 while quads 2-3 store row r0 + 8
      // (and then the other way round), so one store instruction touches 16 banks instead of 8.
      if (tid == 0 && issued) bulk_wait_read0();       // the previous reduce has finished reading sP
      consumer_barrier();                              // ... and (ldst mode) every thread has read the previous tile
      const bool lowq = quad < 2;
      // step form, red mode: stage p as the reduce sees it (flushed), so that one buffer serves the reduce and the store
      const bool stage_ftz = kSlab == kSlabStore && P.rmw_mode == 1;
#pragma unroll
      for (int jj = 0; jj < 10; ++jj) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int col = 8 * jj + 2 * quad + e;
          if (col < kTokens) {
            float a = d[4 * jj + e] * inv0, b = d[4 * jj + 2 + e] * inv1;
            if constexpr (kSecond) {
              if (stage_ftz) { a = add_ftz(0.f, a); b = add_ftz(0.f, b); }
            }
            sP[col * kTilePixels + (lowq ? r0 : r0 + 8)] = lowq ? a : b;
            sP[col * kTilePixels + (lowq ? r0 + 8 : r0)] = lowq ? b : a;
          }
        }
      }
      if (P.rmw_mode == 1) {
        fence_proxy_async();                           // generic-proxy writes -> visible to the bulk-async proxy
        consumer_barrier();
        if (tid == 0) {
          tma_reduce_add_2d(&MP.amap[t.li], sP_u32, t.pixel0, (t.prompt * L.heads + t.head) * kTokens);
          if constexpr (kSlab == kSlabStore)
            tma_store_2d(&MP.smap[t.li], sP_u32, t.pixel0, (t.prompt * L.heads + t.head) * kTokens);
          if constexpr (kSlab == kSlabAdd)
            tma_reduce_add_2d(&MP.smap[t.li], sP_u32, t.pixel0, (t.prompt * L.heads + t.head) * kTokens);
          bulk_commit();
        }
        issued = true;
      } else {
        consumer_barrier();
        const long long hw = L.hw;
        float* acc = L.acc + ((long long)(t.prompt * L.heads + t.head) * kTokens) * hw + t.pixel0;
        const int live = min(kTilePixels, L.hw - t.pixel0) >> 2;       // float4 columns inside the map (hw % 4 == 0)
        for (int u = tid; u < kTokens * (kTilePixels / 4); u += kConsumers) {
          const int tok = u / (kTilePixels / 4), c4 = u % (kTilePixels / 4);
          if (c4 < live) {
            float4* g = reinterpret_cast<float4*>(acc + tok * hw) + c4;
            const float4 p = reinterpret_cast<const float4*>(sP + tok * kTilePixels)[c4];
            float4 o = *g;
            o.x += p.x; o.y += p.y; o.z += p.z; o.w += p.w;
            *g = o;
            if constexpr (kSlab == kSlabStore)
              reinterpret_cast<float4*>(MP.slab[t.li] + (acc - L.acc) + tok * hw)[c4] = p;
            if constexpr (kSlab == kSlabAdd) {
              float4* r = reinterpret_cast<float4*>(MP.slab[t.li] + (acc - L.acc) + tok * hw) + c4;
              float4 ro = *r;
              ro.x += p.x; ro.y += p.y; ro.z += p.z; ro.w += p.w;
              *r = ro;
            }
          }
        }
      }
    }
    // shared memory must outlive the last store's / reduce's reads; the global writes complete with the grid
    if (tid == 0 && (kSplit ? issued : count > 0)) bulk_wait_read0();
  }
}

// ---- host: tensor maps ----------------------------------------------------------------------------------------------
using EncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                              const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                              CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeFn get_encode() {
  static EncodeFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeFn>(p);
  });
  return fn;
}

struct MapKey {
  const void* ptr;
  long long s1, s2, s3;
  int d1, d2, d3, kind;     // kind: 0 q/k 16-bit (dtype in bit 4), 1 accumulator
  bool operator==(const MapKey& o) const {
    return ptr == o.ptr && s1 == o.s1 && s2 == o.s2 && s3 == o.s3 && d1 == o.d1 && d2 == o.d2 && d3 == o.d3 &&
           kind == o.kind;
  }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    size_t h = reinterpret_cast<size_t>(k.ptr);
    auto mix = [&h](long long v) { h ^= (size_t)v + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2); };
    mix(k.s1); mix(k.s2); mix(k.s3); mix(k.d1); mix(k.d2); mix(k.d3); mix(k.kind);
    return h;
  }
};

// Tensor maps are pure functions of (pointer, shape, strides): cache them, the allocator hands the same Q/K
// addresses back every denoising step.
std::unordered_map<MapKey, CUtensorMap, MapKeyHash>& map_cache() {
  static std::unordered_map<MapKey, CUtensorMap, MapKeyHash> c;
  return c;
}
std::mutex g_map_mu;

// {head_dim, heads, rows, prompts} view of a projection; box = [box_rows x one 128-byte swizzle span] of one head (64
// 16-bit or 32 fp32 dims), 128B-swizzled; columns beyond head_dim are zero-filled.
int make_qk_map(const void* ptr, int dtype, int head_dim, int heads, int rows, int prompts, long long s_head,
                long long s_row, long long s_prompt, int box_rows, CUtensorMap* out) {
  MapKey key{ptr, s_head, s_row, s_prompt, heads, rows, prompts * 1024 + box_rows, (dtype << 4) | (head_dim << 8)};
  {
    std::lock_guard<std::mutex> lock(g_map_mu);
    auto it = map_cache().find(key);
    if (it != map_cache().end()) { *out = it->second; return DAAM_OK; }
  }
  EncodeFn enc = get_encode();
  if (!enc) { set_error("cuTensorMapEncodeTiled is not available from this driver"); return DAAM_E_CUDA; }
  const cuuint64_t es = dtype == DAAM_F32 ? 4 : 2;
  const cuuint64_t dims[4] = {(cuuint64_t)head_dim, (cuuint64_t)heads, (cuuint64_t)rows, (cuuint64_t)prompts};
  // (a stride <= 0 only reaches here for an axis of extent 1, which the map never steps along: mma_supported)
  auto bytes = [es](long long s) { return (cuuint64_t)(s > 0 ? s : 8) * es; };
  const cuuint64_t strides[3] = {bytes(s_head), bytes(s_row), bytes(s_prompt)};
  const cuuint32_t box[4] = {(cuuint32_t)(128 / es), 1, (cuuint32_t)box_rows, 1};
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  const CUtensorMapDataType type = dtype == DAAM_F32    ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
                                   : dtype == DAAM_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                                        : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  CUresult r = enc(out, type, 4, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(q/k) failed with CUresult %d", (int)r); return DAAM_E_CUDA; }
  std::lock_guard<std::mutex> lock(g_map_mu);
  if (map_cache().size() > 8192) map_cache().clear();
  map_cache()[key] = *out;
  return DAAM_OK;
}

// accumulator as a 2-D fp32 tensor {hw, prompts*heads*77}; box = [77 tokens x 128 pixels], no swizzle.
int make_acc_map(float* acc, int hw, int rows, CUtensorMap* out) {
  MapKey key{acc, 0, 0, 0, hw, rows, 0, 1};
  {
    std::lock_guard<std::mutex> lock(g_map_mu);
    auto it = map_cache().find(key);
    if (it != map_cache().end()) { *out = it->second; return DAAM_OK; }
  }
  EncodeFn enc = get_encode();
  if (!enc) { set_error("cuTensorMapEncodeTiled is not available from this driver"); return DAAM_E_CUDA; }
  const cuuint64_t dims[2] = {(cuuint64_t)hw, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)hw * 4};
  const cuuint32_t box[2] = {(cuuint32_t)kTilePixels, (cuuint32_t)kTokens};
  const cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, acc, dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(acc) failed with CUresult %d", (int)r); return DAAM_E_CUDA; }
  std::lock_guard<std::mutex> lock(g_map_mu);
  if (map_cache().size() > 8192) map_cache().clear();
  map_cache()[key] = *out;
  return DAAM_OK;
}

// Every wgmma instance and its dynamic shared memory, indexed by PreparedMma::variant: bit 0 split (fp32), bit 1
// chunked (head_dim > 64), bits 2-3 the SlabMode.
struct MmaInstance {
  const void* fn;
  int smem;
};
const MmaInstance kMmaInstances[] = {
    {(const void*)accumulate_mma_kernel<false, false, kSlabNone>, kSmemBytes},
    {(const void*)accumulate_mma_kernel<true, false, kSlabNone>, kSplitSmemBytes},
    {(const void*)accumulate_mma_kernel<false, true, kSlabNone>, kSmemBytes},
    {(const void*)accumulate_mma_kernel<true, true, kSlabNone>, kSplitSmemBytes},
    {(const void*)accumulate_mma_kernel<false, false, kSlabStore>, kSlabSmemBytes},
    {(const void*)accumulate_mma_kernel<true, false, kSlabStore>, kSplitSmemBytes},
    {(const void*)accumulate_mma_kernel<false, true, kSlabStore>, kSlabSmemBytes},
    {(const void*)accumulate_mma_kernel<true, true, kSlabStore>, kSplitSmemBytes},
    {(const void*)accumulate_mma_kernel<false, false, kSlabAdd>, kSlabSmemBytes},
    {(const void*)accumulate_mma_kernel<true, false, kSlabAdd>, kSplitSmemBytes},
    {(const void*)accumulate_mma_kernel<false, true, kSlabAdd>, kSlabSmemBytes},
    {(const void*)accumulate_mma_kernel<true, true, kSlabAdd>, kSplitSmemBytes},
    // long contexts (16-bit, plain slab mode), from kLongVariant0: bit 0 chunked, bit 1 three 77-token chunks (else two)
    {(const void*)accumulate_mma_kernel<false, false, kSlabNone, 2>, long_smem_bytes(2)},
    {(const void*)accumulate_mma_kernel<false, true, kSlabNone, 2>, long_smem_bytes(2)},
    {(const void*)accumulate_mma_kernel<false, false, kSlabNone, 3>, long_smem_bytes(3)},
    {(const void*)accumulate_mma_kernel<false, true, kSlabNone, 3>, long_smem_bytes(3)},
};
constexpr int kLongVariant0 = 12;

std::once_flag g_attr_once[64];                       // the shared-memory attribute is per device

}  // namespace

// Parameter block of one wgmma launch, opaque to api.cu (which caches prepared launches by their daam_layer[] input).
struct PreparedMma {
  MmaSlabParams mp;                                   // the plain instances are launched with its MmaParams part
  int grid, block, variant;                           // variant: index into kMmaInstances
  bool second;                                        // a second-slab instance (takes the whole MmaSlabParams)
};
void* prepared_mma_new() { return new PreparedMma; }                 // (aligned new: CUtensorMap is alignas(64))
void prepared_mma_delete(void* p) { delete static_cast<PreparedMma*>(p); }

// hw % 4 == 0: the accumulator / second-slab tensor maps (make_acc_map) need a row pitch of hw * 4 bytes that is a
// multiple of 16, and the split form's load / add / store epilogue moves float4 columns. Other layers (odd-sized keys
// such as 19 x 25) take the SIMT kernel, which updates the accumulator one element at a time.
// Strides: a tensor map takes positive byte strides only, so every stride make_qk_map encodes must be positive. The
// prompt stride is one of them once there are two or more prompts: a zero stride (a sample broadcast with expand()) or
// a negative one (samples stored in reverse) takes the SIMT kernel, which indexes any int64 stride.
bool mma_supported(const LayerParams& L) {
  const bool prompts_ok = L.n_prompts == 1 || (L.qs_prompt > 0 && L.ks_prompt > 0);
  return L.head_dim % 8 == 0 && L.head_dim <= DAAM_MAX_HEAD_DIM && L.vec_ok && L.qs_head > 0 && L.qs_pixel > 0 &&
         L.ks_head > 0 && L.ks_token > 0 && prompts_ok && L.hw % 4 == 0;
}

// Tensor maps, grid and kernel variant of one pack of layers (all fp32, or all 16-bit). `out`: prepared_mma_new().
int prepare_accumulate_mma(const LaunchParams& p, const SecondSlabs* slabs, SlabMode mode, const DeviceInfo& dev,
                           void* out) {
  if (dev.cc_major != 9) { set_error("the wgmma kernel needs an sm_90 device (found sm_%d%d)", dev.cc_major, dev.cc_minor); return DAAM_E_UNSUPPORTED; }
  PreparedMma& pm = *static_cast<PreparedMma*>(out);
  MmaSlabParams& mp = pm.mp;
  mp.base = p;
  const bool split = p.n_layers > 0 && p.layer[0].dtype == DAAM_F32;     // a pack holds one operand class (api.cu)
  const int ctx = p.n_layers > 0 ? p.layer[0].tokens : kTokens;          // ... and one context length
  if ((ctx != kTokens && ctx != 2 * kTokens && ctx != 3 * kTokens) || (ctx != kTokens && (split || slabs))) {
    set_error("the wgmma kernel takes %d-token contexts, or 154 / 231 tokens for 16-bit layers without a second slab "
              "(got %d)", kTokens, ctx);
    return DAAM_E_UNSUPPORTED;
  }
  bool chunked = false;
  for (int i = 0; i < p.n_layers; ++i) {
    const LayerParams& L = p.layer[i];
    if ((L.dtype == DAAM_F32) != split) { set_error("mixed fp32 / 16-bit layers in one wgmma pack"); return DAAM_E_INVALID; }
    if (L.tokens != ctx) { set_error("mixed context lengths in one wgmma pack"); return DAAM_E_INVALID; }
    if (int rc = make_qk_map(L.q, L.dtype, L.head_dim, L.heads, L.hw, L.n_prompts, L.qs_head, L.qs_pixel, L.qs_prompt, kTilePixels, &mp.qmap[i])) return rc;
    if (int rc = make_qk_map(L.k, L.dtype, L.head_dim, L.heads, ctx, L.n_prompts, L.ks_head, L.ks_token, L.ks_prompt, kTokensPad, &mp.kmap[i])) return rc;
    if (int rc = make_acc_map(L.acc, L.hw, L.n_prompts * L.heads * ctx, &mp.amap[i])) return rc;
    if (slabs) {                                      // the second slab has the accumulator's shape: same map, other base
      if (int rc = make_acc_map(slabs->slab[i], L.hw, L.n_prompts * L.heads * kTokens, &mp.smap[i])) return rc;
      mp.slab[i] = slabs->slab[i];
    }
    chunked = chunked || L.head_dim > 64;
  }
  cudaError_t attr_err = cudaSuccess;
  std::call_once(g_attr_once[dev.device & 63], [&] {
    for (const MmaInstance& k : kMmaInstances)
      if (cudaError_t e = cudaFuncSetAttribute(k.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, k.smem)) attr_err = e;
  });
  DAAM_CUDA_TRY(attr_err);
  pm.grid = dev.sm_count;                             // one CTA per SM (both forms fill its shared memory)
  if (pm.grid > p.total_tiles) pm.grid = p.total_tiles;
  pm.block = split ? kThreads : kThreads16;
  pm.variant = ctx == kTokens ? (split ? 1 : 0) | (chunked ? 2 : 0) | (mode << 2)
                              : kLongVariant0 + (chunked ? 1 : 0) + (ctx == 3 * kTokens ? 2 : 0);
  pm.second = mode != kSlabNone;
  return DAAM_OK;
}

int launch_prepared_mma(const void* prepared, cudaStream_t stream) {
  const PreparedMma& pm = *static_cast<const PreparedMma*>(prepared);
  const MmaInstance& k = kMmaInstances[pm.variant];
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(pm.grid);
  cfg.blockDim = dim3(pm.block);
  cfg.dynamicSmemBytes = k.smem;
  cfg.stream = stream;
  // Programmatic stream serialization also inside a stream capture: the launch becomes a kernel node with a programmatic
  // edge from its predecessor (CUDA >= 12.3).
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = pm.mp.base.pdl ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  // the one kernel argument: the whole block for the second-slab instances, its MmaParams part for the plain ones
  const MmaParams* plain = &pm.mp;
  void* args[] = {pm.second ? (void*)&pm.mp : (void*)plain};
  DAAM_CUDA_TRY(cudaLaunchKernelExC(&cfg, k.fn, args));
  DAAM_CUDA_TRY(cudaGetLastError());
  count_launch();
  return DAAM_OK;
}

}  // namespace daam
