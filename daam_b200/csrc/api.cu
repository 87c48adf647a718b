// C ABI entry points of libdaam_b200.so (include/daam_b200.h): argument validation, packing of layer calls into
// persistent launches, error strings. The kernels live in accumulate_simt.cu, accumulate_mma.cu, finalize.cu, words.cu
// and probs.cu.
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <memory>
#include <mutex>
#include <vector>

#include "common.cuh"

namespace daam {

static thread_local char g_error[512] = "";
static std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_error, sizeof(g_error), fmt, ap);
  va_end(ap);
}

int cuda_fail(cudaError_t e, const char* what) {
  set_error("CUDA error %d (%s) in %s", (int)e, cudaGetErrorString(e), what);
  return DAAM_E_CUDA;
}

void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int get_device_info(DeviceInfo* out) {
  static std::mutex mu;
  static DeviceInfo cache[64];
  int dev = 0;
  DAAM_CUDA_TRY(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lock(mu);
  if (dev < 0 || dev >= 64) { set_error("device index %d out of range", dev); return DAAM_E_CUDA; }
  if (cache[dev].device != dev) {
    cudaDeviceProp prop;
    DAAM_CUDA_TRY(cudaGetDeviceProperties(&prop, dev));
    cache[dev].device = dev;
    cache[dev].sm_count = prop.multiProcessorCount;
    cache[dev].cc_major = prop.major;
    cache[dev].cc_minor = prop.minor;
  }
  *out = cache[dev];
  return DAAM_OK;
}

static size_t dtype_size(int dtype) { return dtype == DAAM_F32 ? 4 : 2; }

// Validates one layer call and fills the device-side descriptor (tile_begin is set by the packer).
int make_layer_params(const daam_layer& in, int index, LayerParams* out, bool need_acc);
int make_layer_params(const daam_layer& in, int index, LayerParams* out, bool need_acc) {
  if (!in.q || !in.k || (need_acc && !in.acc)) { set_error("daam_accumulate: layer %d has a null pointer", index); return DAAM_E_INVALID; }
  if (in.dtype != DAAM_F32 && in.dtype != DAAM_F16 && in.dtype != DAAM_BF16) { set_error("daam_accumulate: layer %d: unknown dtype %d", index, in.dtype); return DAAM_E_INVALID; }
  if (in.tokens != kTokens && in.tokens != 2 * kTokens && in.tokens != 3 * kTokens) { set_error("daam_accumulate: layer %d: tokens = %d, only %d, %d or %d (one to three %d-token CLIP chunks) are traced", index, in.tokens, kTokens, 2 * kTokens, 3 * kTokens, kTokens); return DAAM_E_UNSUPPORTED; }
  if (in.head_dim <= 0 || in.head_dim % 8 != 0 || in.head_dim > DAAM_MAX_HEAD_DIM) { set_error("daam_accumulate: layer %d: head_dim = %d must be a multiple of 8 in (0, %d]", index, in.head_dim, DAAM_MAX_HEAD_DIM); return DAAM_E_UNSUPPORTED; }
  if (in.n_prompts <= 0 || in.heads <= 0 || in.hw <= 0) { set_error("daam_accumulate: layer %d: non-positive n_prompts/heads/hw", index); return DAAM_E_INVALID; }
  if (need_acc && reinterpret_cast<uintptr_t>(in.acc) % 16 != 0) { set_error("daam_accumulate: layer %d: acc is not 16-byte aligned", index); return DAAM_E_INVALID; }
  if (!(in.scale > 0.f)) { set_error("daam_accumulate: layer %d: scale must be positive", index); return DAAM_E_INVALID; }
  LayerParams& L = *out;
  L.q = in.q; L.k = in.k; L.acc = in.acc;
  L.qs_prompt = in.q_stride_prompt; L.qs_pixel = in.q_stride_pixel; L.qs_head = in.q_stride_head;
  L.ks_prompt = in.k_stride_prompt; L.ks_token = in.k_stride_token; L.ks_head = in.k_stride_head;
  L.n_prompts = in.n_prompts; L.heads = in.heads; L.hw = in.hw; L.head_dim = in.head_dim;
  L.dtype = in.dtype;
  L.scale_log2e = in.scale * 1.4426950408889634f;
  L.tiles_per_head = (in.hw + kTilePixels - 1) / kTilePixels;
  L.tile_begin = 0;
  const size_t es = dtype_size(in.dtype);
  auto aligned = [&](long long stride) { return (stride * (long long)es) % 16 == 0; };
  L.weight = 1;
  L.weight_begin = 0;
  L.vec_ok = reinterpret_cast<uintptr_t>(in.q) % 16 == 0 && reinterpret_cast<uintptr_t>(in.k) % 16 == 0 &&
             aligned(in.q_stride_prompt) && aligned(in.q_stride_pixel) && aligned(in.q_stride_head) &&
             aligned(in.k_stride_prompt) && aligned(in.k_stride_token) && aligned(in.k_stride_head);
  L.tokens = in.tokens;
  return DAAM_OK;
}

}  // namespace daam

using namespace daam;

namespace daam {
namespace {

// One kernel launch of a plan: a pack of layers for the wgmma kernel (prepared block, opaque) or a SIMT kernel.
struct PlannedLaunch {
  bool is_mma = false;
  LaunchParams simt;                     // SIMT: the parameter block itself
  SlabMode mode = kSlabNone;             // SIMT: the step- or range-slab kernel, with these slabs
  SecondSlabs slabs;
  int grid = 0;
  size_t smem = 0;
  struct MmaDeleter { void operator()(void* p) const { prepared_mma_delete(p); } };
  std::unique_ptr<void, MmaDeleter> mma; // wgmma: PreparedMma (tensor maps + parameter block), opaque here
};

// Everything daam_accumulate derives from its input: the packs, their tensor maps, grids. A trace replays the same
// layer calls (same pointers: the caching allocator hands the projections the same addresses) every denoising step,
// so plans are cached by the verbatim daam_layer[] input; a hit costs one memcmp instead of ~3 hash lookups per layer.
struct Plan {
  std::vector<uint8_t> key;              // the caller's daam_layer[n] bytes (+ its step_acc[n] / range_acc[n] pointers)
  uint32_t flags = 0;
  int device = -1;
  SlabMode mode = kSlabNone;             // daam_accumulate_steps stores into the slabs, daam_accumulate_range adds
  std::vector<PlannedLaunch> launches;
  uint64_t stamp = 0;
};
constexpr size_t kMaxPlans = 32;

// Bytes of a layer's accumulator slab [n_prompts][heads][tokens][hw] (fp32).
size_t slab_bytes(const LayerParams& l) { return (size_t)l.n_prompts * l.heads * l.tokens * l.hw * sizeof(float); }

// Whether [a, a + na) and [b, b + nb) share bytes.
bool spans_overlap(const void* a, size_t na, const void* b, size_t nb) {
  const char *pa = static_cast<const char*>(a), *pb = static_cast<const char*>(b);
  return pa < pb + nb && pb < pa + na;
}

bool acc_overlap(const LayerParams& a, const LayerParams& b) {
  return spans_overlap(a.acc, slab_bytes(a), b.acc, slab_bytes(b));
}

// The word the messages of daam_accumulate_steps / daam_accumulate_range use for their second slabs.
const char* slab_word(SlabMode mode) { return mode == kSlabAdd ? "range" : "step"; }

// daam_accumulate_steps / daam_accumulate_range (`fn`): every second slab is non-null, 16-byte aligned, and shares no
// byte with an accumulator or with another second slab of the call (the kernels store or add it tile by tile, in any
// order, next to the accumulator update).
int validate_second_slabs(const char* fn, const daam_layer* layers, float* const* slabs, int n_layers, SlabMode mode) {
  const char* what = slab_word(mode);
  std::vector<LayerParams> all((size_t)n_layers);
  for (int i = 0; i < n_layers; ++i) {
    if (int rc = make_layer_params(layers[i], i, &all[i], /*need_acc=*/true)) return rc;
    if (all[i].tokens != kTokens) { set_error("%s: layer %d: tokens = %d, the %s slabs take %d-token contexts only", fn, i, all[i].tokens, what, kTokens); return DAAM_E_UNSUPPORTED; }
  }
  for (int i = 0; i < n_layers; ++i) {
    if (!slabs[i]) { set_error("%s: layer %d has a null %s slab", fn, i, what); return DAAM_E_INVALID; }
    if (reinterpret_cast<uintptr_t>(slabs[i]) % 16 != 0) { set_error("%s: layer %d: the %s slab is not 16-byte aligned", fn, i, what); return DAAM_E_INVALID; }
  }
  for (int i = 0; i < n_layers; ++i) {
    const size_t n = slab_bytes(all[i]);
    for (int j = 0; j < n_layers; ++j) {
      if (spans_overlap(slabs[i], n, all[j].acc, slab_bytes(all[j]))) {
        set_error("%s: the %s slab of layer %d overlaps the accumulator of layer %d", fn, what, i, j);
        return DAAM_E_INVALID;
      }
      if (j != i && spans_overlap(slabs[i], n, slabs[j], slab_bytes(all[j]))) {
        set_error("%s: the %s slabs of layers %d and %d overlap", fn, what, i, j);
        return DAAM_E_INVALID;
      }
    }
  }
  return DAAM_OK;
}

int build_plan(const daam_layer* layers, float* const* slabs, SlabMode mode, int n_layers, uint32_t flags,
               const DeviceInfo& dev, Plan* plan) {
  const uint32_t path = flags & 3u, rmw = flags & DAAM_ACC_RMW_MASK;
  // Three packs of 77-token layers: 16-bit layers for the wgmma kernel (TMA form), fp32 layers for its split form, and
  // the rest for the SIMT kernel. Long contexts (154 / 231 tokens) take four more, one per context length and kernel:
  // a long-context layer never shares a launch with a layer of another length or class. Each pack is closed when its
  // parameter block is full.
  constexpr int kPacks = 7;
  LaunchParams packs[kPacks];            // 0: wgmma 16-bit, 1: wgmma fp32, 2: SIMT; 3 / 4: wgmma 16-bit at 154 / 231
  SecondSlabs pack_slabs[kPacks];        // tokens; 5 / 6: long-context SIMT at 154 / 231 tokens
                                         // steps / range: the second slab of every layer of a pack
  for (LaunchParams& p : packs) {
    p.n_layers = p.total_tiles = 0;
    p.rmw_mode = (rmw == DAAM_ACC_RMW_LDST) ? 0 : 1;     // default: reduce-add
    p.pdl = (flags & DAAM_ACC_NO_PDL) ? 0 : 1;
    p.early_loads = (flags & DAAM_ACC_EARLY_LOADS) && p.pdl ? 1 : 0;
    p.total_weight = 0;
  }
  // The fp32 split form holds a whole SM per CTA (196 KB of shared memory): its CTAs only become resident as the previous
  // launch's CTAs exit, so there is no tail to overlap and its loads wait at the top.
  packs[1].early_loads = 0;
  auto close = [&](int which) -> int {
    LaunchParams& p = packs[which];
    if (p.n_layers == 0) return DAAM_OK;
    plan->launches.emplace_back();
    PlannedLaunch& l = plan->launches.back();
    l.is_mma = which != 2 && which < 5;
    const SecondSlabs* st = slabs ? &pack_slabs[which] : nullptr;
    int rc;
    if (l.is_mma) {
      l.mma.reset(prepared_mma_new());
      rc = prepare_accumulate_mma(p, st, mode, dev, l.mma.get());
    } else {
      l.simt = p;
      l.mode = mode;
      if (st) l.slabs = *st;
      rc = prepare_accumulate_simt(p, mode, dev, &l.grid, &l.smem);
    }
    p.n_layers = 0;
    p.total_tiles = 0;
    p.total_weight = 0;
    return rc;
  };
  for (int i = 0; i < n_layers; ++i) {
    LayerParams L;
    if (int rc = make_layer_params(layers[i], i, &L, /*need_acc=*/true)) return rc;
    const int ctx_chunks = L.tokens / kTokens;          // 1, or 2 / 3 for a long context
    // (the wgmma kernel's fp32 split form has no long-context instances: such layers take the SIMT kernel)
    const bool use_mma = path != DAAM_ACC_FORCE_SIMT && dev.cc_major == 9 && mma_supported(L) &&
                         (ctx_chunks == 1 || L.dtype != DAAM_F32);
    if (path == DAAM_ACC_FORCE_MMA && !use_mma) {
      set_error("daam_accumulate: layer %d cannot take the wgmma path (dtype %d, head_dim %d, alignment %d, hw = %d, "
                "tokens = %d, %d prompts with prompt strides q %lld / k %lld, sm_%d%d)", i, L.dtype, L.head_dim,
                L.vec_ok, L.hw, L.tokens, L.n_prompts, L.qs_prompt, L.ks_prompt, dev.cc_major, dev.cc_minor);
      return DAAM_E_UNSUPPORTED;
    }
    const int which = ctx_chunks > 1 ? (use_mma ? 1 : 3) + ctx_chunks : use_mma ? (L.dtype == DAAM_F32 ? 1 : 0) : 2;
    LaunchParams& p = packs[which];
    // Two layers of one launch must not share accumulator elements: their tiles run concurrently, and the 16-bit wgmma
    // form and the LDST mode read, add and store them (lost updates), while RED would add in timing order (results not
    // deterministic). A layer whose slab overlaps one already in its pack starts that pack's next launch; stream order
    // then applies the two in call order.
    for (int m = 0; m < p.n_layers; ++m)
      if (acc_overlap(p.layer[m], L)) {
        if (int rc = close(which)) return rc;
        break;
      }
    L.tile_begin = p.total_tiles;
    // Cost of a tile relative to the launch's other layers (SD-1.5's 40 / 80 / 160 head dims): every 64-wide K chunk is
    // one load -> (convert ->) MMA round through the two-stage ring. In the fp32 split form that chain is the whole cost
    // of a tile (weight = chunks); in the 16-bit form the softmax and accumulator update of the tile add a fixed part
    // (weight = 1 + 4 * chunks).
    const int n_chunks = (L.head_dim + 63) / 64;
    L.weight = which == 1 ? n_chunks : 1 + 4 * n_chunks;
    L.weight_begin = p.total_weight;
    if (slabs) pack_slabs[which].slab[p.n_layers] = slabs[i];
    p.layer[p.n_layers++] = L;
    p.total_tiles += L.tiles_per_head * L.heads * L.n_prompts;
    p.total_weight += L.tiles_per_head * L.heads * L.n_prompts * L.weight;
    if (p.n_layers == kMaxLayersPerLaunch)
      if (int rc = close(which)) return rc;
  }
  for (int which = 0; which < kPacks; ++which)
    if (int rc = close(which)) return rc;
  return DAAM_OK;
}

}  // namespace
}  // namespace daam

namespace daam {
namespace {

// daam_accumulate (slabs == nullptr, kSlabNone), daam_accumulate_steps (kSlabStore) and daam_accumulate_range
// (kSlabAdd), with the argument checks they share; `fn`: the entry point, as its messages name it.
int accumulate_impl(const char* fn, const daam_layer* layers, float* const* slabs, SlabMode mode, int32_t n_layers,
                    uint32_t flags, void* stream_) {
  if (n_layers < 0 || (n_layers > 0 && !layers)) { set_error("%s: bad layer array", fn); return DAAM_E_INVALID; }
  if (n_layers == 0) return DAAM_OK;
  const bool with_slabs = mode != kSlabNone;
  if (with_slabs && !slabs) { set_error("%s: %s_acc is a null array", fn, slab_word(mode)); return DAAM_E_INVALID; }
  cudaStream_t stream = static_cast<cudaStream_t>(stream_);
  DeviceInfo dev;
  if (int rc = get_device_info(&dev)) return rc;

  static thread_local std::vector<std::unique_ptr<Plan>> plans;    // per calling thread: no locking on the hot path
  static thread_local uint64_t clock = 0;
  const size_t layer_bytes = sizeof(daam_layer) * (size_t)n_layers;
  const size_t slab_ptr_bytes = with_slabs ? sizeof(float*) * (size_t)n_layers : 0;
  const size_t bytes = layer_bytes + slab_ptr_bytes;
  Plan* plan = nullptr;
  for (auto& c : plans)
    if (c->key.size() == bytes && c->flags == flags && c->device == dev.device && c->mode == mode &&
        memcmp(c->key.data(), layers, layer_bytes) == 0 &&
        (!with_slabs || memcmp(c->key.data() + layer_bytes, slabs, slab_ptr_bytes) == 0)) {
      plan = c.get();
      break;
    }
  if (!plan) {
    if (with_slabs)
      if (int rc = validate_second_slabs(fn, layers, slabs, n_layers, mode)) return rc;
    std::unique_ptr<Plan> fresh(new Plan);
    fresh->key.assign(reinterpret_cast<const uint8_t*>(layers), reinterpret_cast<const uint8_t*>(layers) + layer_bytes);
    if (with_slabs)
      fresh->key.insert(fresh->key.end(), reinterpret_cast<const uint8_t*>(slabs),
                        reinterpret_cast<const uint8_t*>(slabs) + slab_ptr_bytes);
    fresh->flags = flags;
    fresh->device = dev.device;
    fresh->mode = mode;
    if (int rc = build_plan(layers, slabs, mode, n_layers, flags, dev, fresh.get())) return rc;     // failed plans are not cached
    if (plans.size() >= kMaxPlans) {                                                   // evict the least recently used
      size_t oldest = 0;
      for (size_t i = 1; i < plans.size(); ++i)
        if (plans[i]->stamp < plans[oldest]->stamp) oldest = i;
      plans[oldest] = std::move(fresh);
      plan = plans[oldest].get();
    } else {
      plans.push_back(std::move(fresh));
      plan = plans.back().get();
    }
  }
  plan->stamp = ++clock;
  for (const PlannedLaunch& l : plan->launches) {
    const int rc = l.is_mma ? launch_prepared_mma(l.mma.get(), stream)
                            : launch_prepared_simt(l.simt, l.mode != kSlabNone ? &l.slabs : nullptr, l.mode, l.grid,
                                                   l.smem, stream);
    if (rc) return rc;
  }
  return DAAM_OK;
}

}  // namespace
}  // namespace daam

extern "C" int daam_accumulate(const daam_layer* layers, int32_t n_layers, uint32_t flags, void* stream) {
  return accumulate_impl("daam_accumulate", layers, nullptr, kSlabNone, n_layers, flags, stream);
}

extern "C" int daam_accumulate_steps(const daam_layer* layers, float* const* step_acc, int32_t n_layers, uint32_t flags,
                                     void* stream) {
  return accumulate_impl("daam_accumulate_steps", layers, step_acc, kSlabStore, n_layers, flags, stream);
}

extern "C" int daam_accumulate_range(const daam_layer* layers, float* const* range_acc, int32_t n_layers, uint32_t flags,
                                     void* stream) {
  return accumulate_impl("daam_accumulate_range", layers, range_acc, kSlabAdd, n_layers, flags, stream);
}

// ---- side-stream launcher ------------------------------------------------------------------------------------------
struct daam_side_launcher {
  cudaEvent_t ready = nullptr, done = nullptr;
  int device = -1;
  bool launched = false;
};

extern "C" int daam_side_launcher_create(daam_side_launcher** out) {
  if (!out) { set_error("daam_side_launcher_create: null pointer"); return DAAM_E_INVALID; }
  DeviceInfo dev;
  if (int rc = get_device_info(&dev)) return rc;
  std::unique_ptr<daam_side_launcher> h(new daam_side_launcher);
  h->device = dev.device;
  DAAM_CUDA_TRY(cudaEventCreateWithFlags(&h->ready, cudaEventDisableTiming));
  if (cudaError_t e = cudaEventCreateWithFlags(&h->done, cudaEventDisableTiming)) {
    cudaEventDestroy(h->ready);
    return cuda_fail(e, "cudaEventCreateWithFlags");
  }
  *out = h.release();
  return DAAM_OK;
}

extern "C" void daam_side_launcher_destroy(daam_side_launcher* h) {
  if (!h) return;
  if (h->ready) cudaEventDestroy(h->ready);
  if (h->done) cudaEventDestroy(h->done);
  delete h;
}

extern "C" int daam_side_launcher_launch(daam_side_launcher* h, const daam_layer* layers, int32_t n_layers, uint32_t flags,
                                         void* producer_stream, void* side_stream) {
  if (!h) { set_error("daam_side_launcher_launch: null launcher"); return DAAM_E_INVALID; }
  cudaStream_t producer = static_cast<cudaStream_t>(producer_stream), side = static_cast<cudaStream_t>(side_stream);
  DAAM_CUDA_TRY(cudaEventRecord(h->ready, producer));          // the projections were produced on `producer`
  DAAM_CUDA_TRY(cudaStreamWaitEvent(side, h->ready, 0));
  if (int rc = daam_accumulate(layers, n_layers, flags, side_stream)) return rc;
  DAAM_CUDA_TRY(cudaEventRecord(h->done, side));
  h->launched = true;
  return DAAM_OK;
}

extern "C" int daam_side_launcher_join(daam_side_launcher* h, void* stream) {
  if (!h) { set_error("daam_side_launcher_join: null launcher"); return DAAM_E_INVALID; }
  if (h->launched) DAAM_CUDA_TRY(cudaStreamWaitEvent(static_cast<cudaStream_t>(stream), h->done, 0));
  return DAAM_OK;
}

extern "C" int daam_side_launcher_idle(daam_side_launcher* h) {
  if (!h) { set_error("daam_side_launcher_idle: null launcher"); return DAAM_E_INVALID; }
  if (!h->launched) return 1;
  const cudaError_t e = cudaEventQuery(h->done);
  if (e == cudaSuccess) return 1;
  if (e == cudaErrorNotReady) return 0;
  return cuda_fail(e, "cudaEventQuery");
}

extern "C" int daam_abi_version(void) { return DAAM_ABI_VERSION; }
extern "C" const char* daam_last_error(void) { return g_error; }
extern "C" int64_t daam_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

extern "C" int daam_device_info(int32_t* sm_count, int32_t* cc_major, int32_t* cc_minor) {
  DeviceInfo dev;
  if (int rc = get_device_info(&dev)) return rc;
  if (sm_count) *sm_count = dev.sm_count;
  if (cc_major) *cc_major = dev.cc_major;
  if (cc_minor) *cc_minor = dev.cc_minor;
  return DAAM_OK;
}
