/*
 * daam_b200.h -- C ABI of libdaam_b200.so: the H100 (sm_90a) cross-attention heat-map hot path.
 *
 * The reference (castorini/daam, paths below relative to its checkout) is pure Python/torch and has no FFI. The
 * entry points here are what a binding for its hot path replaces; each one cites the reference interface it stands
 * in for. INTEGRATION.md shows the ctypes stub a maintainer of the reference would add.
 *
 * Conventions
 *  - plain pointers and sizes only; every pointer named *device* is CUDA device memory owned by the caller (torch
 *    tensors on the Python side); the library never allocates or frees caller-visible memory;
 *  - `stream` is a cudaStream_t passed as void*; all work is enqueued asynchronously on it; the caller keeps the
 *    buffers alive until the stream has passed the call;
 *  - every function returns 0 on success and a negative DAAM_E_* code otherwise; daam_last_error() gives the message
 *    of the calling thread's last failure (the Python host raises RuntimeError / ValueError like the reference does,
 *    daam/hook.py:36-37, daam/trace.py:120-124);
 *  - there is no CPU fallback: without a CUDA device every compute entry point fails with DAAM_E_CUDA.
 */
#ifndef DAAM_B200_H
#define DAAM_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DAAM_ABI_VERSION 4          /* 2: + daam_attention_probs, daam_accumulate_probs, daam_finalize_per_key
                                       3: + DAAM_ACC_EARLY_LOADS, daam_expand_words, daam_side_launcher_*
                                          (later, additive: daam_accumulate_steps, daam_normalize_maps,
                                          daam_accumulate_range)
                                       4: the finalize family takes (map_h, map_w); the _rect names are gone
                                          (later, additive: layers with hw not a multiple of 4 are accepted) */
#define DAAM_TOKENS 77          /* context length the reference traces (daam/trace.py:194, guard at :289) */
#define DAAM_MAX_HEAD_DIM 256   /* any multiple of 8 up to here (SD-1.x deepest level: 1280 channels / 8 heads = 160) */

enum daam_status {
  DAAM_OK = 0,
  DAAM_E_INVALID = -1,          /* bad argument (shape, alignment, null pointer) */
  DAAM_E_UNSUPPORTED = -2,      /* tokens != 77, head_dim not a multiple of 8 or > DAAM_MAX_HEAD_DIM, ... */
  DAAM_E_CUDA = -3              /* a CUDA runtime call failed (including: no device) */
};

enum daam_dtype { DAAM_F32 = 0, DAAM_F16 = 1, DAAM_BF16 = 2 };

/* daam_accumulate flags */
#define DAAM_ACC_AUTO        0u  /* wgmma path whenever rows are 16-byte aligned (any dtype, head_dim % 8 == 0) and
                                    hw % 4 == 0, SIMT fp32 path otherwise */
#define DAAM_ACC_FORCE_SIMT  1u  /* always the SIMT fp32 ("warp dot") kernel */
#define DAAM_ACC_FORCE_MMA   2u  /* wgmma kernel or DAAM_E_UNSUPPORTED */
/* Accumulator update of the SIMT kernel and of the wgmma kernel's fp32 form. The wgmma kernel's 16-bit (fp16 / bf16)
   form ignores these flags: it always adds in shared memory, into accumulator tiles loaded ahead by TMA, and stores
   them back, with the same arithmetic as RED. */
#define DAAM_ACC_RMW_MASK   0x30u
#define DAAM_ACC_RMW_AUTO   0x00u /* = RED on both paths (one add per element per launch -- layers whose
                                     accumulators overlap go to separate launches -- so results stay deterministic) */
#define DAAM_ACC_RMW_LDST   0x10u /* coalesced load / add / store of the accumulator tile */
#define DAAM_ACC_RMW_RED    0x20u /* red.global.add.f32 (SIMT) / bulk-async reduce-add from shared memory (MMA) */
#define DAAM_ACC_NO_PDL     0x100u /* launch without programmatic dependent launch (measurement / debugging) */
#define DAAM_ACC_EARLY_LOADS 0x200u /* The caller vouches that q and k of every layer were complete BEFORE the previous
                                     kernel on `stream` started (they were produced on another stream and joined through
                                     an event, or are resident inputs). Then only the kernel's accumulator updates wait
                                     for the previous kernel (programmatic dependent launch); its loads, MMAs and first
                                     softmax overlap that kernel's tail. Never set it when the producer of q/k may be the
                                     immediately preceding kernel on `stream`. Ordering of the accumulator updates, and
                                     therefore the result, is unchanged. */

/*
 * One traced cross-attention layer call: the conditional half of the projections `to_q(hidden_states)` and
 * `to_k(encoder_hidden_states)` as the attention module emits them (daam/trace.py:262-270), *before* the reference's
 * head_to_batch_dim permute (trace.py:272-273) -- the strides below express that permute, nothing is copied.
 *
 * Replaces, fused in one kernel: Attention.get_attention_scores = softmax(scale * Q K^T) (called at trace.py:276),
 * UNetCrossAttentionHooker._unravel_attn (trace.py:219-244: token-major transpose, (h, w) reshape, "second half of the
 * batch*heads axis" = conditional samples) and the per-head RawHeatMapCollection.update loop (trace.py:293-294,
 * heatmap.py:153-156).
 *
 *   acc[p][head][t][pixel] += softmax_t( scale * <q[p][pixel][head][:], k[p][t][head][:]> )
 *
 * `acc` is fp32, contiguous [n_prompts][heads][tokens][hw]: acc[p][head] is exactly the reference's per-key
 * [77, h, w] heat map for key (factor, layer, head). n_prompts > 1 is the batched mode (independent single-prompt
 * traces run in one launch); the reference itself is single-prompt (trace.py:172-173).
 */
typedef struct daam_layer {
  const void* q;             /* device; element (prompt 0, pixel 0, head 0, dim 0) of the CONDITIONAL half */
  const void* k;             /* device; element (prompt 0, token 0, head 0, dim 0) of the conditional half */
  float* acc;                /* device; fp32 [n_prompts][heads][tokens][hw], 16-byte aligned */
  int64_t q_stride_prompt, q_stride_pixel, q_stride_head;   /* in elements; the head_dim axis is contiguous */
  int64_t k_stride_prompt, k_stride_token, k_stride_head;
  int32_t n_prompts, heads, hw, tokens, head_dim;   /* hw: any positive pixel count; the wgmma path needs hw % 4 == 0
                                                       (DAAM_ACC_AUTO sends other layers to the SIMT kernel) */
  int32_t dtype;             /* enum daam_dtype of q and k */
  float scale;               /* attn.scale = head_dim ** -0.5 */
  int32_t reserved;
} daam_layer;

/* Enqueue the fused softmax(QK^T) -> unravel -> accumulate kernel over `n_layers` layer calls (any number; the
 * library packs them into as few persistent launches as possible). `layers` is host memory, read before returning.
 * Layers may share accumulator elements (the same or overlapping slabs): such a layer starts a new launch, so on every
 * path and in every update mode each one adds, and layers of one operand class are applied in call order. Layers of
 * different classes (16-bit wgmma, fp32 wgmma, SIMT) go to different launches, issued class by class. */
int daam_accumulate(const daam_layer* layers, int32_t n_layers, uint32_t flags, void* stream);

/*
 * Time-resolved heat maps (daam_b200/trace.py, trace(..., time_resolved=True)): daam_accumulate, and also
 *   step_acc[i][p][head][t][pixel] = the value added (flushed like the add)
 * so that one denoising step's per-key maps exist next to the time sum. With acc == 0 beforehand, step_acc equals acc
 * afterwards bit for bit. Every element of every step slab is written; nothing else is.
 * step_acc: host array of n_layers device pointers, fp32, 16-byte aligned, same shape as layers[i].acc. A step slab
 * must not overlap any accumulator or any other step slab of the call (DAAM_E_INVALID). Same flags and packing as
 * daam_accumulate; with DAAM_ACC_EARLY_LOADS the step-slab stores, too, wait for the previous kernel.
 */
int daam_accumulate_steps(const daam_layer* layers, float* const* step_acc, int32_t n_layers, uint32_t flags,
                          void* stream);

/*
 * Step-range heat maps (daam_b200/trace.py, trace(..., step_ranges=[...])): daam_accumulate, and also
 *   range_acc[i][p][head][t][pixel] += the value added
 * with the arithmetic daam_accumulate applies to acc in the same update mode (16-bit wgmma form: add.rn.ftz, as the
 * accumulator tile; fp32 split form and SIMT: the reduce-add or load / add / store the flags select). So a range slab
 * zeroed before a span of calls holds afterwards, bit for bit, what an accumulator that received only those calls
 * would hold. Same validation, flags and packing as daam_accumulate_steps (range_acc: host array of n_layers device
 * pointers, fp32, 16-byte aligned, shaped like layers[i].acc, overlapping no accumulator and no other range slab).
 */
int daam_accumulate_range(const daam_layer* layers, float* const* range_acc, int32_t n_layers, uint32_t flags,
                          void* stream);

/*
 * The tracer's optional side-stream launch (daam_b200/trace.py flush, launch='overlap'): the reference's hook does its
 * heat-map work inline on the pipeline's stream (daam/trace.py:276-294), and so does the tracer by default (one
 * daam_accumulate per denoising step on the forward's own stream). With launch='overlap' that one launch runs on a
 * side stream so that it also overlaps the next step's first kernels; this helper does the stream plumbing in one
 * foreign call:
 *   launch: record an event on `producer_stream` (where to_q / to_k ran), make `side_stream` wait for it,
 *           daam_accumulate(layers, n_layers, flags, side_stream), record the launcher's `done` event on side_stream;
 *   join:   make `stream` wait for the last launch (before anything reads the accumulators or frees the projections);
 *   idle:   1 if the last launch has completed (the caller may then drop its references to that step's q / k), 0 if
 *           it is still running, negative on error.
 * The launcher owns two CUDA events and nothing else. Not thread-safe; one launcher per tracer.
 */
typedef struct daam_side_launcher daam_side_launcher;
int daam_side_launcher_create(daam_side_launcher** out);
void daam_side_launcher_destroy(daam_side_launcher* launcher);
int daam_side_launcher_launch(daam_side_launcher* launcher, const daam_layer* layers, int32_t n_layers, uint32_t flags,
                              void* producer_stream, void* side_stream);
int daam_side_launcher_join(daam_side_launcher* launcher, void* stream);
int daam_side_launcher_idle(daam_side_launcher* launcher);

/*
 * Compatibility path of the reference's save_heads: materialise what Attention.get_attention_scores returns
 * (daam/trace.py:276) so that it can be saved like daam/trace.py:246-247, 279-280 do:
 *   probs[(p*heads + head)][pixel][t] = softmax_t(scale * <q, k>)   for every sample p in [0, n_prompts)
 * in the dtype of q (device, contiguous [n_prompts*heads][hw][77]). `layer` describes the WHOLE batch here (q/k point
 * at sample 0, n_prompts = batch size); layer->acc is ignored. Runs the SIMT fp32 kernel for every dtype.
 */
int daam_attention_probs(const daam_layer* layer, void* probs, void* stream);

/*
 * Compatibility path of the reference's load_heads (daam/trace.py:281-294): heat maps from supplied probabilities,
 *   acc[r][t][pixel] += probs[first_row + r][pixel][t]     for r in [0, n_rows)
 * i.e. _unravel_attn + the update loop with rows = kept (sample, head) pairs; probs is [*][hw][77] of `dtype`,
 * acc fp32 [n_rows][77][hw].
 */
int daam_accumulate_probs(const void* probs, int32_t dtype, int32_t first_row, int32_t n_rows, int32_t hw,
                          int32_t tokens, float* acc, void* stream);

/*
 * All (or one) heads of one traced layer: `acc` points at [heads][tokens][h*w] fp32 (one prompt's slice of the
 * accumulator daam_accumulate fills). head_sel = -1 selects every head, otherwise one head index.
 */
typedef struct daam_key_group {
  const float* acc;          /* device */
  int32_t heads, h, w, tokens;
  int32_t head_sel;
  int32_t reserved;
} daam_key_group;

/*
 * Replaces DiffusionHeatMapHooker.compute_global_heat_map (daam/trace.py:83-132) after its Python-side key filter:
 * per selected key bicubic upsample (align_corners=False, A=-0.75, no antialias) to the [map_h][map_w] grid, taps key
 * h -> map_h and key w -> map_w, clamp(min=0), mean over the keys, keep rows [0, n_rows), and if `normalize` divide by
 * (sum of rows 1..n_rows-2 + 1e-6) per pixel. out: device fp32 [n_rows][map_h][map_w]. `groups` is host memory, at most
 * 160 groups. Fails with DAAM_E_INVALID when no key is selected (the host turns that into the reference's "No heat maps
 * found" RuntimeError, trace.py:120-124).
 * The banded fast kernel runs when every key has one integer factor 1, 2 or 4 on both axes and a 16-byte-aligned base
 * (aligned slab, h * w a multiple of 4), map_w <= 256, there are at most 8 key sizes and 2048 keys, and, for a square
 * map only, side % 16 == 0; anything else, or DAAM_FINALIZE_GENERIC=1, runs the generic gather kernel (DESIGN.md
 * section 4.3).
 */
int daam_finalize(const daam_key_group* groups, int32_t n_groups, int32_t map_h, int32_t map_w, int32_t n_rows,
                  int32_t normalize, float* out, void* stream);

/*
 * The reference's --all-heads sweep calls compute_global_heat_map(layer_idx=l, head_idx=h) once per (layer, head)
 * (daam/run/generate.py:239-255): each call reduces exactly one key, i.e. bicubic + clamp (+ normalise) of that key.
 * This entry point produces all of them in one launch: out [n_keys][n_rows][map_h][map_w] (device fp32), taps key
 * h -> map_h and key w -> map_w, keys enumerated group by group, head by head, in the order given. Limits: 160 groups,
 * 65535 keys.
 */
int daam_finalize_per_key(const daam_key_group* groups, int32_t n_groups, int32_t map_h, int32_t map_w, int32_t n_rows,
                          int32_t normalize, float* out, void* stream);

/*
 * The `normalize` step of daam_finalize on its own, in place, for n_maps <= 65535 independent [n_rows][map_h][map_w]
 * heat maps stored back to back (e.g. the per-step global maps of a time-resolved trace): maps / (sum of rows
 * 1..n_rows-2 + 1e-6) per pixel, the same arithmetic as daam_finalize(normalize = 1).
 */
int daam_normalize_maps(float* maps, int32_t n_maps, int32_t n_rows, int32_t map_h, int32_t map_w, void* stream);

/*
 * Replaces GlobalHeatMap.compute_word_heat_map's tensor part (daam/heatmap.py:121-123): mean over the rows
 * `rows[0..n_sel)` (host array, n_sel <= 128, already offset by +1 for SOS as daam/utils.py:91 does) of global_maps
 * [n_rows][map_h][map_w] -> out [map_h][map_w] (both device fp32).
 */
int daam_word_heat_map(const float* global_maps, int32_t n_rows, int32_t map_h, int32_t map_w, const int32_t* rows,
                       int32_t n_sel, float* out, void* stream);

/*
 * Replaces WordHeatMap.expand_as's tensor part (daam/heatmap.py:77-93): bicubic upsample of word_map [map_h][map_w] to
 * [out_h][out_w], taps map_h -> out_h and map_w -> out_w, then unless `absolute` (im - min) / (max - min + 1e-8), then
 * if `use_threshold` binarise (im > threshold) (the reference's `if threshold:` -- Python truthiness -- is resolved by
 * the host). out: device fp32 [out_h][out_w]; scratch: device, >= DAAM_EXPAND_SCRATCH_FLOATS floats, owned by the
 * caller. Limit: map_h * map_w * 4 bytes <= 200 KB (the map lives in shared memory). One launch (the n_words = 1 case
 * of daam_expand_words).
 */
#define DAAM_EXPAND_SCRATCH_FLOATS 64   /* per word: partial min/max of up to 32 pixel chunks */
int daam_expand_as(const float* word_map, int32_t map_h, int32_t map_w, int32_t out_h, int32_t out_w, int32_t absolute,
                   int32_t use_threshold, float threshold, float* out, float* scratch, void* stream);

/*
 * The per-word loop a user of the reference writes -- `for word in prompt: global_heat_map.compute_word_heat_map(word)
 * .expand_as(image)` (daam/heatmap.py:121-123 then :77-93; e.g. daam/run/generate.py, the README example) -- for a LIST
 * of words in one cooperative launch: word w averages rows[row_begin[w] .. row_begin[w+1]) of global_maps
 * [n_rows][map_h][map_w] (rows already offset by +1 for SOS, daam/utils.py:91), the [map_h][map_w] mean is
 * bicubic-upsampled to [out_h][out_w] (taps map_h -> out_h and map_w -> out_w), min-max normalised unless `absolute`,
 * binarised if `use_threshold`.
 * out: device fp32 [n_words][out_h][out_w]; word_maps: optional device fp32 [n_words][map_h][map_w] (the word heat maps
 * themselves, NULL to skip); scratch: device, >= DAAM_EXPAND_SCRATCH_FLOATS * n_words floats; rows / row_begin: host.
 * Limits: n_words <= 96, row_begin[n_words] <= 320, map_h * map_w * 4 bytes <= 200 KB. Nothing is copied to the host:
 * the caller reads `out` back once.
 */
int daam_expand_words(const float* global_maps, int32_t n_rows, int32_t map_h, int32_t map_w, const int32_t* rows,
                      const int32_t* row_begin, int32_t n_words, int32_t out_h, int32_t out_w, int32_t absolute,
                      int32_t use_threshold, float threshold, float* word_maps, float* out, float* scratch,
                      void* stream);

/* Library / device introspection. */
int daam_abi_version(void);
const char* daam_last_error(void);
/* sm_count, compute capability and the number of kernels this library has launched since load (bench.py's
 * gpu_launches). Any out pointer may be NULL. Returns DAAM_E_CUDA without a device. */
int daam_device_info(int32_t* sm_count, int32_t* cc_major, int32_t* cc_minor);
int64_t daam_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* DAAM_B200_H */
