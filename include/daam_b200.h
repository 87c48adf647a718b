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
                                          (later, additive: layers with hw not a multiple of 4 are accepted;
                                          daam_segment_words, daam_finalize_maps; daam_key_group.reserved is
                                          n_blocks; daam_accumulate takes 154- and 231-token contexts; layers with
                                          several prompts and a prompt stride <= 0 take the SIMT kernel;
                                          daam_region_overlap; daam_overlay_words, daam_jet_colormap;
                                          daam_finalize_parts; daam_word_overlap;
                                          daam_word_instances; daam_region_sweep;
                                          daam_region_ranking; daam_refine_words;
                                          daam_region_boundary, daam_mask_boundary;
                                          daam_segment_crf;
                                          daam_word_distance, daam_mask_distance;
                                          daam_image_superpixels, daam_segment_superpixels;
                                          daam_value_norms, daam_finalize_parts_weighted;
                                          daam_joint_layer, daam_accumulate_joint; a key group's acc may point at
                                          any row of a slab, see daam_key_group;
                                          daam_accumulate_joint_heads) */
#define DAAM_TOKENS 77          /* context length the reference traces (daam/trace.py:194, guard at :289) */
#define DAAM_MAX_TOKENS 231     /* daam_accumulate: long contexts of 2 or 3 CLIP chunks of 77 tokens (154, 231) */
#define DAAM_MAX_HEAD_DIM 256   /* any multiple of 8 up to here (SD-1.x deepest level: 1280 channels / 8 heads = 160) */

enum daam_status {
  DAAM_OK = 0,
  DAAM_E_INVALID = -1,          /* bad argument (shape, alignment, null pointer) */
  DAAM_E_UNSUPPORTED = -2,      /* tokens not 77 / 154 / 231 (77 only outside daam_accumulate), head_dim not a
                                   multiple of 8 or > DAAM_MAX_HEAD_DIM, ... */
  DAAM_E_CUDA = -3              /* a CUDA runtime call failed (including: no device) */
};

enum daam_dtype { DAAM_F32 = 0, DAAM_F16 = 1, DAAM_BF16 = 2 };

/* daam_accumulate flags */
#define DAAM_ACC_AUTO        0u  /* wgmma path whenever rows are 16-byte aligned (any dtype, head_dim % 8 == 0),
                                    hw % 4 == 0, the head and pixel / token strides are positive and, with
                                    n_prompts > 1, so are both prompt strides; SIMT fp32 path otherwise */
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
 *
 * Long contexts (daam_accumulate only): tokens may be 77, 154 or 231 (one to three CLIP chunks of 77 tokens, e.g.
 * chunked prompt embeddings); the softmax runs over all `tokens` columns and every row is accumulated. Any other count
 * is DAAM_E_UNSUPPORTED. 16-bit layers the wgmma path takes run its long-context instances; fp32 layers and the rest
 * run a two-pass SIMT kernel. A long-context layer never shares a launch with a layer of another context length.
 * daam_accumulate_steps, daam_accumulate_range, daam_attention_probs and daam_accumulate_probs take 77 tokens only.
 */
typedef struct daam_layer {
  const void* q;             /* device; element (prompt 0, pixel 0, head 0, dim 0) of the CONDITIONAL half */
  const void* k;             /* device; element (prompt 0, token 0, head 0, dim 0) of the conditional half */
  float* acc;                /* device; fp32 [n_prompts][heads][tokens][hw], 16-byte aligned */
  int64_t q_stride_prompt, q_stride_pixel, q_stride_head;   /* in elements; the head_dim axis is contiguous */
  int64_t k_stride_prompt, k_stride_token, k_stride_head;   /* Any int64 value, in any order: head-major
                                                               ([B, H, N, d]), padded heads, fused projections
                                                               (qkv / kv buffers), padding between samples. A zero
                                                               prompt stride repeats sample 0 (expand()), a negative
                                                               one walks back from it; with n_prompts > 1 such a
                                                               layer takes the SIMT kernel (DAAM_ACC_AUTO) and
                                                               DAAM_ACC_FORCE_MMA refuses it (DAAM_E_UNSUPPORTED).
                                                               The wgmma path needs every other stride positive and
                                                               a multiple of 16 bytes. */
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
 * Joint attention (MM-DiT, Stable Diffusion 3 / 3.5: daam_b200/trace.py traces pipe.transformer's
 * transformer_blocks[i].attn; FLUX.1: also single_transformer_blocks[j].attn, whose sequences are text-first,
 * [context, image], so q and lse point at row T of the sequence and k at row 0, and every sample is kept since the
 * batch has no CFG half). Image and context tokens go through ONE softmax over all hw + T keys, so the image-query x
 * context-key block is not a softmax over the context alone. Its normaliser is the joint attention's log-sum-exp, which
 * the attention itself returns (SDPA's logsumexp), so the heat map of one layer call is
 *
 *   acc[p][head][t][pixel] += exp(scale * <q[p][pixel][head][:], k[p][t][head][:]> - lse[p][head][pixel])
 *
 * q: the conditional IMAGE queries (after norm_q where the block has it); k: the conditional CONTEXT keys (after
 * norm_added_k); lse: fp32, natural-log units, element (p, head, pixel) at lse + p * lse_stride_prompt +
 * head * lse_stride_head + pixel * lse_stride_pixel, pointing at image query 0 of the first kept sample. Every other
 * field, stride and rule is daam_layer's (n_prompts counts samples: prompts x images per prompt; the head_dim axis is
 * contiguous; any int64 strides), except:
 *  - tokens: any count in [1, DAAM_JOINT_MAX_TOKENS] (SD3: 77 CLIP rows + max_sequence_length T5 rows, 333 or 589);
 *  - hw: any positive count (SD3 maps are (H / 16) x (W / 16));
 *  - head_dim: a multiple of 8 up to DAAM_MAX_HEAD_DIM (DAAM_E_UNSUPPORTED otherwise).
 *
 * Arithmetic (every element of every layer, every dtype):
 *   s  = <q, k> in fp32: fp16 / bf16 operands on tensor cores (mma.sync m16n8k16, products exact in fp32, the sum in
 *        an unspecified order, |s - <q, k>| <= head_dim * 2^-23 * sum_e |q_e k_e| is the bound to test against);
 *        fp32 operands: an fmaf chain over e ascending from 0 (SIMT kernel);
 *   c  = fp32(scale * log2(e)),  l = fp32(lse * log2(e))   (log2(e) = 1.4426950408889634f);
 *   v  = ex2.approx.ftz.f32(fmaf(s, c, -l))                 (relative error <= 2^-22 for v not subnormal);
 *   acc = acc + v                                            (add.rn.f32).
 * Each launch adds every element of every layer exactly once, with no atomics. The layers of a call fall into three
 * kernel classes by dtype, issued in this order: fp16 (tensor cores), bf16 (tensor cores, a kernel of its own) and
 * fp32 (SIMT); within a class the layers are applied in call order. So layers of different dtypes that share
 * accumulator bytes add fp16 first, then bf16, then fp32, whatever their call order, and the result does not depend
 * on timing. The layers of one class share a launch until one of them shares accumulator bytes with a layer already
 * in it, or the launch holds DAAM_JOINT_MAX_LAYERS: that layer starts the class's next launch.
 * Errors: DAAM_E_INVALID for a null layer array, a null q / k / acc / lse, a misaligned acc (16 bytes), a non-positive
 * n_prompts / heads / hw, an unknown dtype or a scale that is not positive; DAAM_E_UNSUPPORTED for tokens or head_dim
 * outside the limits. `flags` is reserved: pass 0. Arguments are checked before the device is touched.
 */
#define DAAM_JOINT_MAX_TOKENS 1024
#define DAAM_JOINT_MAX_LAYERS 64
typedef struct daam_joint_layer {
  const void* q;
  const void* k;
  float* acc;
  int64_t q_stride_prompt, q_stride_pixel, q_stride_head;
  int64_t k_stride_prompt, k_stride_token, k_stride_head;
  int32_t n_prompts, heads, hw, tokens, head_dim;
  int32_t dtype;
  float scale;
  int32_t reserved;
  const float* lse;          /* device fp32 */
  int64_t lse_stride_prompt, lse_stride_head, lse_stride_pixel;   /* in elements */
} daam_joint_layer;
int daam_accumulate_joint(const daam_joint_layer* layers, int32_t n_layers, uint32_t flags, void* stream);

/*
 * Head-reduced joint attention (daam_b200/trace.py, trace(pipe, reduce_heads=True)): daam_accumulate_joint with the
 * heads of every sample summed before anything reaches the accumulator,
 *
 *   acc[p][t][pixel] += fp32(sum_h v_h) / heads
 *
 * with v_h = ex2.approx.ftz.f32(fmaf(s_h, c, -l_h)) exactly the value daam_accumulate_joint adds for head h of the
 * same element (the same dot product, c and l). `acc` is fp32, contiguous [n_prompts][tokens][hw]: one slab row per
 * kept sample, no head axis. Arithmetic of the head sum and the update:
 *   sum = v_0;  sum = sum + v_h for h = 1, 2, .., heads - 1    (add.rn.f32, heads ascending, in registers);
 *   acc = acc + div.rn.f32(sum, heads)                        (add.rn.f32).
 * A joint key has its grid's own size (factor 1), so the finalize's bicubic taps are 0, 1, 0, 0 and its clamp does
 * nothing (every value is positive): the global map is linear in the keys, and the mean over the slab rows of the
 * layers that keep the same head count is the mean over their keys.
 * Every element is read and written once per launch by one thread, with no atomics, so the bits are the same on every
 * call and however the layers are split into calls. Layer array, strides, lse, dtypes, kernel classes and their order
 * (fp16, bf16, fp32), call order within a class, DAAM_JOINT_MAX_LAYERS per launch and the overlap rule (on the
 * head-free slab) are daam_accumulate_joint's, and so are its checks and error codes; a null or not 16-byte aligned
 * `acc` is DAAM_E_INVALID. `flags` is reserved: pass 0.
 */
int daam_accumulate_joint_heads(const daam_joint_layer* layers, int32_t n_layers, uint32_t flags, void* stream);

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
 * daam_finalize_maps reads a group as `n_blocks` such blocks back to back ([n_blocks][heads][tokens][h*w] from acc:
 * e.g. a whole slab [prompts][images * heads] with `heads` the heads per image) and head_sel applies inside each block;
 * the other entry points ignore n_blocks (it was `reserved`, callers set it to 0).
 * `acc` may point at row r0 of such a block instead of row 0, with `tokens` still the block's row count (the head
 * stride): the group's row t is then the slab's row r0 + t, and the rows a call reads, r0 + [0, n_rows), must lie in
 * the slab's rows (the caller's condition; the call checks n_rows <= tokens only). The joint-attention T5 read does
 * this with r0 = 76.
 */
typedef struct daam_key_group {
  const float* acc;          /* device */
  int32_t heads, h, w, tokens;
  int32_t head_sel;
  int32_t n_blocks;
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
 * Several daam_finalize maps over one group list in one launch (e.g. every image's map of a prompt, or every map a
 * time-resolved step writes). Each group is read as n_blocks blocks (see daam_key_group); map m reduces blocks
 * [block_begin, block_begin + block_count) of EVERY group, and is bit for bit what daam_finalize gives for the expanded
 * group list `for g: for b in those blocks: {acc_g + b * heads_g * tokens_g * h_g * w_g, heads_g, head_sel_g}` with
 * maps[m].n_rows and maps[m].out (same key order, kernel choice and band height; with head_sel = -1 that is one group
 * per layer with heads_g * block_count heads). `normalize` applies per map over its own rows. `groups` and `maps` are
 * host memory. One launch per kind of kernel the maps take (fast / generic: one when every map is alike, which is the
 * case whenever their key counts are on the same side of 2048) plus one normalisation launch.
 * Limits: n_groups <= 160 and n_maps <= DAAM_FINALIZE_MAX_MAPS (DAAM_E_UNSUPPORTED). DAAM_E_INVALID: what
 * daam_finalize refuses, no map, a map without output, rows or blocks, a negative block_begin, or a block range past
 * a group's n_blocks.
 */
#define DAAM_FINALIZE_MAX_MAPS 64
typedef struct daam_map_sel {
  int32_t block_begin, block_count;   /* blocks [block_begin, block_begin + block_count) of every group */
  int32_t n_rows, reserved;           /* rows [0, n_rows) of the map; reserved: 0 */
  float* out;                         /* device fp32 [n_rows][map_h][map_w] */
} daam_map_sel;
int daam_finalize_maps(const daam_key_group* groups, int32_t n_groups, const daam_map_sel* maps, int32_t n_maps,
                       int32_t map_h, int32_t map_w, int32_t normalize, void* stream);

/*
 * Several daam_finalize maps over SUBSETS of one group list in one launch (e.g. one map per UNet layer, or one per
 * resolution): map m reduces groups [group_begin, group_begin + group_count) of the call's list and is bit for bit what
 *   daam_finalize(groups + group_begin, group_count, map_h, map_w, n_rows, normalize, out, stream)
 * writes: same key order, kernel choice and band height. The kernel choice is daam_finalize's rule applied to the map's
 * own groups: only their factors, base alignment and key count (2048) decide, so a map whose groups the banded kernel
 * cannot read goes to the generic kernel while its neighbours stay on the fast one. Ranges may overlap, leave groups
 * unused, or cover every group, so the all-layers map and the per-layer maps can come out of one call. n_blocks is
 * ignored, as in daam_finalize. `groups` and `maps` are host memory. One launch per kind of kernel the maps take plus
 * one normalisation launch.
 * Limits: n_groups <= 160 and n_maps <= DAAM_FINALIZE_MAX_MAPS (DAAM_E_UNSUPPORTED). DAAM_E_INVALID: what daam_finalize
 * refuses (a group with fewer tokens than a map that reads it has rows included), no map, a map without output, rows or
 * groups, a negative group_begin, or a group range past n_groups.
 */
typedef struct daam_map_part {
  int32_t group_begin, group_count;   /* groups [group_begin, group_begin + group_count) of the call's list */
  int32_t n_rows, reserved;           /* rows [0, n_rows) of the map; reserved: 0 */
  float* out;                         /* device fp32 [n_rows][map_h][map_w] */
} daam_map_part;
int daam_finalize_parts(const daam_key_group* groups, int32_t n_groups, const daam_map_part* maps, int32_t n_maps,
                        int32_t map_h, int32_t map_w, int32_t normalize, void* stream);

/*
 * daam_finalize_parts with one weight per key and row (value-weighted heat maps, daam_b200/trace.py
 * trace(..., value_norms=True)): map m is
 *   (1 / K) sum_k weight_k[t] * clamp(bicubic(key_k[t]), 0)     (then normalised like daam_finalize if asked)
 * over the K keys daam_finalize_parts selects for it, in the same key order, kernel choice, band height, group-merge
 * order and final division by K. The only change is the per-key add: the plain `acc += clamp(o)` becomes
 * `acc = fmaf(w, clamp(o), acc)`. So weights of 1.0 give daam_finalize_parts' bits, and weights of 2^k give 2^k times
 * them (without `normalize`, which adds 1e-6 to its denominator).
 * weights: host array of n_groups device pointers; weights[g] is fp32 [heads][tokens] (the group's acc layout with
 * h * w = 1), read with the key's head index (head_sel included) at rows [0, n_rows). Weights must be finite and >= 0:
 * the call cannot check device memory. Limits and errors: those of daam_finalize_parts, and DAAM_E_INVALID for a null
 * weights array or a null entry.
 */
int daam_finalize_parts_weighted(const daam_key_group* groups, int32_t n_groups, const daam_map_part* maps,
                                 int32_t n_maps, int32_t map_h, int32_t map_w, int32_t normalize,
                                 const float* const* weights, void* stream);

/*
 * Value norms (norm-based attention analysis: Kobayashi et al., EMNLP 2020): for sample b, head h and context row j of
 * one cross-attention layer,
 *   n[b][h][j] = || W_h v ||_2,   v = value[b][j][h d .. (h + 1) d),   W_h = W[:, h d .. (h + 1) d)
 * with W = attn.to_out[0].weight ([out_dim][heads * d], row stride w_stride_row elements, columns contiguous) and
 * `value` what attn.to_v produced: element (b, j, h, e) at value + b * v_stride_sample + j * v_stride_token +
 * h * v_stride_head + e (elements; the channel axis is contiguous). Point `value` and `w` at head 0 of the first sample
 * kept, as daam_layer does for K: e.g. the conditional half of a CFG batch, or sample 0 for the whole batch. Both
 * operands are converted to fp32 (value_dtype and w_dtype: enum daam_dtype, independently).
 * Arithmetic: y_c = sum_e W_h[c][e] v[e] as an fmaf chain over e ascending from 0, s = sum_c y_c^2 as an fmaf chain
 * over c ascending from 0, n = sqrtf(s). out: device fp32 [n_samples][heads][tokens].
 * Limits (DAAM_E_UNSUPPORTED): tokens 77, 154 or 231, head_dim <= DAAM_MAX_HEAD_DIM, out_dim <= 4096,
 * n_samples * heads <= 65535. DAAM_E_INVALID: a null pointer, a non-positive size or an unknown dtype.
 */
int daam_value_norms(const void* value, int32_t value_dtype, int64_t v_stride_sample, int64_t v_stride_token,
                     int64_t v_stride_head, const void* w, int32_t w_dtype, int64_t w_stride_row, int32_t n_samples,
                     int32_t heads, int32_t tokens, int32_t head_dim, int32_t out_dim, float* out, void* stream);

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

/*
 * Word segmentation: one label per pixel for a word list, on each of n_maps global maps stored back to back
 * (global_maps [n_maps][n_rows][map_h][map_w]; e.g. every step of a time-resolved history). With m[w] what
 * daam_expand_words writes for word w without threshold (same rows / row_begin, host arrays shared by all maps):
 *   scores[i][p] = max_w m[w][p]                                  (bit-identical to daam_expand_words' values)
 *   labels[i][p] = 1 + argmax_w m[w][p], the lowest w on ties; 0 (background) where use_threshold and
 *                  !(scores[i][p] > threshold)
 * min / max run per (map, word). word_maps: device fp32 [n_maps][n_words][map_h][map_w] (required: the second kernel
 * reads them); labels: device uint8 [n_maps][out_h][out_w]; scores: device fp32 [n_maps][out_h][out_w]; scratch:
 * device, >= DAAM_SEGMENT_SCRATCH_FLOATS(n_maps, n_words) floats. Two launches whatever n_maps and n_words; the
 * [n_words][out_h][out_w] stack is never written. Deterministic.
 * Limits (DAAM_E_UNSUPPORTED): n_words <= 96 (labels 1..96 plus background fit a byte), row_begin[n_words] <= 320,
 * map_h * map_w * 4 bytes <= 200 KB, n_maps <= 65535, out_h * out_w <= 2^30. Any output size, smaller than the map
 * included. DAAM_E_INVALID: null pointer, non-positive size, empty word list, a word without rows, a row out of range.
 */
#define DAAM_SEGMENT_SCRATCH_FLOATS(n_maps, n_words) (64 * (n_maps) * (n_words))
int daam_segment_words(const float* global_maps, int32_t n_maps, int32_t n_rows, int32_t map_h, int32_t map_w,
                       const int32_t* rows, const int32_t* row_begin, int32_t n_words, int32_t out_h, int32_t out_w,
                       int32_t absolute, int32_t use_threshold, float threshold, float* word_maps, uint8_t* labels,
                       float* scores, float* scratch, void* stream);

/*
 * Word-region overlap: how much of each word's expanded map lies inside each of n_regions binary image regions, on
 * each of n_maps global maps stored back to back -- the sums behind the reference's evaluation (daam/evaluate.py:14-35:
 * compute_iou / compute_ioa of every (word mask, region) pair). With m[w] what daam_expand_words writes for word w with
 * the same arguments (0/1 when use_threshold) and R[r](p) = (regions[r][p] != 0):
 *   intersection[i][r][w] = sum_p R[r](p) * m[w](p)          (fp32 [n_maps][n_regions][n_words])
 *   word_area[i][w]       = sum_p m[w](p)                    (fp32 [n_maps][n_words])
 * Arguments as daam_segment_words, plus regions: device uint8 [n_regions][out_h][out_w], shared by every map (any
 * nonzero byte is inside). scratch: device, >= DAAM_REGION_SCRATCH_FLOATS(n_maps, n_words, n_regions, out_h, out_w)
 * floats. Three launches whatever n_maps, n_words and n_regions; the [n_words][out_h][out_w] stack is never written.
 * The sums run in a fixed order without atomics, so repeated calls give the same bits; with use_threshold every
 * sum is an exact pixel count.
 * Limits (DAAM_E_UNSUPPORTED): n_words <= 96, row_begin[n_words] <= 320, n_regions <= 63 (DAAM_REGION_MAX_REGIONS),
 * map_h * map_w * 4 bytes <= 200 KB, n_maps <= 65535, out_h * out_w <= 2^24 (counts stay exact in fp32). DAAM_E_INVALID:
 * null pointer, non-positive size (n_regions included), empty word list, a word without rows, a row out of range.
 */
#define DAAM_REGION_MAX_REGIONS 63
#define DAAM_REGION_SCRATCH_FLOATS(n_maps, n_words, n_regions, out_h, out_w)                                        \
  ((int64_t)(n_maps) * (n_words) * (64 + ((int64_t)(n_regions) + 1) * (((out_h) + 15) / 16) * (((out_w) + 63) / 64)))
int daam_region_overlap(const float* global_maps, int32_t n_maps, int32_t n_rows, int32_t map_h, int32_t map_w,
                        const int32_t* rows, const int32_t* row_begin, int32_t n_words, int32_t out_h, int32_t out_w,
                        int32_t absolute, int32_t use_threshold, float threshold, float* word_maps,
                        const uint8_t* regions, int32_t n_regions, float* intersection, float* word_area, float* scratch,
                        void* stream);

/*
 * Threshold sweep of word-region overlap: daam_region_overlap's pixel counts at n_thresholds thresholds in one pass --
 * IoU, precision and recall of the reference's evaluation (daam/evaluate.py) as functions of the binarisation
 * threshold. With m[w] what daam_expand_words writes for word w WITHOUT threshold (same rows / row_begin / absolute)
 * and R[r](p) = (regions[r][p] != 0), for every map i and threshold k:
 *   intersection[i][k][r][w] = #{p : R[r](p) and m[w](p) > thresholds[k]}    (fp32 [n_maps][n_thresholds][n_regions][n_words])
 *   word_area[i][k][w]       = #{p : m[w](p) > thresholds[k]}                 (fp32 [n_maps][n_thresholds][n_words])
 * compared in fp32 with the very m daam_expand_words thresholds, so for every nonzero thresholds[k] slice k equals what
 * daam_region_overlap(..., use_threshold = 1, threshold = thresholds[k]) writes, bit for bit. Every entry is a real
 * threshold: 0 and negative values count m > 0 and m > t (there is no "0 means none"). Arguments as
 * daam_region_overlap, with use_threshold / threshold replaced by thresholds: host fp32 [n_thresholds], finite and
 * strictly ascending. scratch: device, >= DAAM_REGION_SWEEP_SCRATCH_FLOATS(...) floats: the 64 min / max floats per
 * (map, word), then a (n_regions + 1) x n_thresholds histogram per (map, word); it does not grow with the image.
 * One memset and three launches whatever n_thresholds, n_maps, n_words and n_regions; the [n_words][out_h][out_w]
 * stack is never written. Every count is an integer sum, so repeated calls give the same bits.
 * Limits (DAAM_E_UNSUPPORTED): those of daam_region_overlap, and n_thresholds <= 64
 * (DAAM_REGION_SWEEP_MAX_THRESHOLDS). DAAM_E_INVALID: as daam_region_overlap, plus n_thresholds <= 0, null thresholds,
 * a threshold that is not finite, thresholds not strictly ascending.
 */
#define DAAM_REGION_SWEEP_MAX_THRESHOLDS 64
#define DAAM_REGION_SWEEP_SCRATCH_FLOATS(n_maps, n_words, n_regions, n_thresholds, out_h, out_w)                     \
  ((int64_t)(n_maps) * (n_words) * (64 + ((int64_t)(n_regions) + 1) * (n_thresholds)))
int daam_region_sweep(const float* global_maps, int32_t n_maps, int32_t n_rows, int32_t map_h, int32_t map_w,
                      const int32_t* rows, const int32_t* row_begin, int32_t n_words, int32_t out_h, int32_t out_w,
                      int32_t absolute, const float* thresholds, int32_t n_thresholds, float* word_maps,
                      const uint8_t* regions, int32_t n_regions, float* intersection, float* word_area,
                      float* scratch, void* stream);

/*
 * Word-pair overlap: how much each word's expanded map overlaps every other word's, on each of n_maps global maps
 * stored back to back -- the sums behind the DAAM paper's head / dependent analysis (the reference's
 * WordHeatMap.compute_ioa, daam/heatmap.py:95-96, and compute_iou / compute_ioa of every pair of word masks). With m[w]
 * what daam_expand_words writes for word w with the same arguments (0/1 when use_threshold):
 *   intersection[i][a][b] = sum_p m[a](p) * m[b](p)           (fp32 [n_maps][n_words][n_words])
 *   word_area[i][a]       = sum_p m[a](p)                     (fp32 [n_maps][n_words])
 * Each pair a <= b is summed once and written to [a][b] and [b][a], so the matrix is symmetric bit for bit; with
 * use_threshold the diagonal equals word_area. out_h x out_w = map_h x map_w sums over the heat-map grid itself
 * (there the bicubic taps are the identity, so m is the word heat map). Arguments as daam_segment_words; scratch:
 * device, >= DAAM_WORD_OVERLAP_SCRATCH_FLOATS(n_maps, n_words, out_h, out_w) floats: per map 64 n_words plus
 * n_words (n_words + 3) / 2 partials for each of min(tiles, DAAM_WORD_OVERLAP_CTAS) CTAs (tiles of 16 x 64 output
 * pixels), e.g. 47 KB at 8 words and 4.9 MB at 96 words for a 512 x 512 or larger image. A map's sums are the same bits
 * whatever n_maps. Three launches whatever n_maps and n_words; the [n_words][out_h][out_w] stack is never written. The sums run
 * in a fixed order without atomics, so repeated calls give the same bits; with use_threshold every sum is an exact
 * pixel count.
 * Limits (DAAM_E_UNSUPPORTED): n_words <= 96, row_begin[n_words] <= 320, map_h * map_w * 4 bytes <= 200 KB,
 * n_maps <= 65535, out_h * out_w <= 2^24 (counts stay exact in fp32). DAAM_E_INVALID: null pointer, non-positive size,
 * empty word list, a word without rows, a row out of range.
 */
#define DAAM_WORD_OVERLAP_CTAS 256   /* CTAs per map, at most one per 16 x 64 output tile */
#define DAAM_WORD_OVERLAP_SCRATCH_FLOATS(n_maps, n_words, out_h, out_w)                                               \
  ((int64_t)(n_maps) * ((n_words) * 64 + ((n_words) * ((n_words) + 3) / 2) *                                         \
       ((((out_h) + 15) / 16) * (((out_w) + 63) / 64) < DAAM_WORD_OVERLAP_CTAS                                       \
            ? (((out_h) + 15) / 16) * (((out_w) + 63) / 64) : DAAM_WORD_OVERLAP_CTAS)))
int daam_word_overlap(const float* global_maps, int32_t n_maps, int32_t n_rows, int32_t map_h, int32_t map_w,
                      const int32_t* rows, const int32_t* row_begin, int32_t n_words, int32_t out_h, int32_t out_w,
                      int32_t absolute, int32_t use_threshold, float threshold, float* word_maps,
                      float* intersection, float* word_area, float* scratch, void* stream);

/*
 * Word instances: the 8-connected components of each word's mask, on each of n_maps global maps stored back to back
 * -- where a word is and how many blobs it makes (the weakly supervised localisation protocol: threshold the map, take
 * the largest component, score its box). With pre[w] what daam_expand_words writes for word w without threshold
 * (same rows / row_begin / absolute), the mask is pre[w] > threshold: what daam_expand_words writes with it. For plane
 * (i, w) and its components sorted by area, largest first, ties to the component whose first pixel comes first in
 * raster order (scipy.ndimage.label's order), instance j < K = max_instances:
 *   count[i][w]              number of components, all of them                            int32 [n_maps][n_words]
 *   area[i][w][j]            pixels                                                       int32 [...][K]
 *   box[i][w][j]             (y0, x0, y1, x1), half-open: scipy.ndimage.find_objects      int32 [...][K][4]
 *   sum_yx[i][w][j]          sums of the row and of the column indices of its pixels      int64 [...][K][2]
 *   peak[i][w][j]            max of pre over the component                                fp32  [...][K]
 *   peak_yx[i][w][j]         the first pixel in raster order where pre == peak            int32 [...][K][2]
 * Slots j >= count are 0 in every field. Arguments as daam_word_overlap without use_threshold (the threshold is always
 * in effect); outputs on the device. scratch: device, 8-byte aligned; as many (map, word) planes are labelled per round
 * as scratch_bytes holds at DAAM_WORD_INSTANCES_PLANE_BYTES(out_h, out_w) each (about 20 bytes a pixel), whole maps
 * while a map's planes fit, and the call loops over the rounds: seven launches a round. The results are the same bits
 * whatever the scratch, and on every call (integer atomics only).
 * Limits (DAAM_E_UNSUPPORTED): those of daam_word_overlap, and max_instances <= 64 (DAAM_WORD_INSTANCES_MAX).
 * DAAM_E_INVALID: as daam_word_overlap, plus max_instances <= 0 and scratch_bytes below one plane.
 */
#define DAAM_WORD_INSTANCES_MAX 64
#define DAAM_WORD_INSTANCES_PLANE_BYTES(out_h, out_w)                                                                 \
  (8 * (int64_t)(out_h) * (out_w) + 48 * (int64_t)(((out_h) + 1) / 2) * (((out_w) + 1) / 2) + 260)
int daam_word_instances(const float* global_maps, int32_t n_maps, int32_t n_rows, int32_t map_h, int32_t map_w,
                        const int32_t* rows, const int32_t* row_begin, int32_t n_words, int32_t out_h, int32_t out_w,
                        int32_t absolute, float threshold, int32_t max_instances, float* word_maps, int32_t* count,
                        int32_t* area, int32_t* box, int64_t* sum_yx, float* peak, int32_t* peak_yx, void* scratch,
                        int64_t scratch_bytes, void* stream);

/*
 * Region ranking: threshold-free scores of each word's expanded map against each of n_regions binary image regions, on
 * each of n_maps global maps stored back to back -- pixel ROC-AUC and average precision of an attribution map against
 * a ground-truth mask, which no threshold sweep gives exactly. With m[w] what daam_expand_words writes for word w
 * WITHOUT threshold (same rows / row_begin / absolute), values compared as fp32 numbers (-0 and +0 tie), P = {p :
 * regions[r][p] != 0}, N the other pixels, n_p = |P| and n_n = out_h * out_w - n_p:
 *   u2[i][r][w] = sum_{p in P} sum_{q in N} (2 [m_p > m_q] + [m_p == m_q])      (int64 [n_maps][n_regions][n_words])
 * twice the Mann-Whitney U with ties counted half, an exact integer: ROC-AUC = u2 / (2 n_p n_n), undefined when n_p or
 * n_n is 0. With v_1 > v_2 > ... > v_K the distinct values of m[w], TP_k = #{p in P : m_p >= v_k} and FP_k the same
 * count over N (TP_0 = 0):
 *   ap[i][r][w] = sum_k (TP_k - TP_{k-1}) / n_p * TP_k / (TP_k + FP_k)        (double, same shape; NaN when n_p = 0)
 * sklearn's average_precision_score. Arguments as daam_region_overlap without use_threshold / threshold; u2 and ap on
 * the device. scratch: device, 8-byte aligned, at least DAAM_REGION_RANKING_SCRATCH_BYTES(1, out_h, out_w): one
 * uint64 region mask per pixel for the call, then DAAM_REGION_RANKING_PLANE_BYTES(out_h, out_w) (about 18 bytes a
 * pixel) per (map, word) plane of a round. As many planes go in a round as the scratch holds, whole maps while a map's
 * planes fit, and the call loops over the rounds: one launch, then eighteen a round (the values, a four-pass radix
 * sort of every plane of the round, the tie-group counts). The results are the same bits whatever the scratch and on
 * every call: no float atomics, every sum in a fixed order.
 * Limits (DAAM_E_UNSUPPORTED): those of daam_region_overlap. DAAM_E_INVALID: as daam_region_overlap, plus
 * scratch_bytes below DAAM_REGION_RANKING_SCRATCH_BYTES(1, out_h, out_w).
 */
#define DAAM_REGION_RANKING_PLANE_BYTES(out_h, out_w)                                                                 \
  (16 * (int64_t)(out_h) * (out_w) + 1024 * (((int64_t)(out_h) * (out_w) + 4095) / 4096) +                           \
   1540 * (((int64_t)(out_h) * (out_w) + 1023) / 1024) + 512)
#define DAAM_REGION_RANKING_SCRATCH_BYTES(n_planes, out_h, out_w)                                                     \
  (8 * (int64_t)(out_h) * (out_w) + (int64_t)(n_planes) * DAAM_REGION_RANKING_PLANE_BYTES(out_h, out_w))
int daam_region_ranking(const float* global_maps, int32_t n_maps, int32_t n_rows, int32_t map_h, int32_t map_w,
                        const int32_t* rows, const int32_t* row_begin, int32_t n_words, int32_t out_h, int32_t out_w,
                        int32_t absolute, float* word_maps, const uint8_t* regions, int32_t n_regions, int64_t* u2,
                        double* ap, void* scratch, int64_t scratch_bytes, void* stream);

/*
 * Heat-map overlays: the reference's plot_overlay (daam/heatmap.py:20-53, :66-75 -- the word map coloured with
 * matplotlib's `jet` under the image drawn with alpha 1 - heat) as RGB pixels, for a word list on each of n_maps global
 * maps stored back to back. With m[w] what daam_expand_words writes for word w with the same arguments, for every map,
 * word, pixel and channel:
 *   c   = color_normalize ? (hi == lo ? 0 : (m - lo) / (hi - lo)) : min(max(m, 0), 1)   (lo, hi: min / max of m[w])
 *   k   = min(int(c * 256), 255)                              (matplotlib's Colormap with N = 256)
 *   a   = min(max(m, 0), 1)
 *   out = uint8(clamp(rne((1 - a) * image + a * L[k]), 0, 255))   (each operation rounded in fp32, no fused multiply-add)
 * with L the table daam_jet_colormap returns.
 * Arguments as daam_segment_words, plus color_normalize; image: device uint8 [out_h][out_w][3], map i's image at
 * image + i * image_map_stride bytes (0: one image for every map); frames: device uint8
 * [n_maps][n_words][out_h][out_w][3], 4-byte aligned, in a buffer of DAAM_OVERLAY_FRAMES_BYTES(...) bytes (the frames
 * rounded up to whole 4-byte words: the bytes past them are overwritten); scratch: device, >=
 * DAAM_SEGMENT_SCRATCH_FLOATS(n_maps, n_words) floats. Two launches whatever n_maps and n_words; the
 * [n_words][out_h][out_w] fp32 stack is never written. Deterministic.
 * Limits (DAAM_E_UNSUPPORTED): as daam_segment_words. DAAM_E_INVALID: as daam_segment_words, plus a negative
 * image_map_stride or frames not 4-byte aligned.
 */
#define DAAM_OVERLAY_FRAMES_BYTES(n_maps, n_words, out_h, out_w)                                                      \
  (((int64_t)(n_maps) * (n_words) * (out_h) * (out_w) * 3 + 3) / 4 * 4)
int daam_overlay_words(const float* global_maps, int32_t n_maps, int32_t n_rows, int32_t map_h, int32_t map_w,
                       const int32_t* rows, const int32_t* row_begin, int32_t n_words, int32_t out_h, int32_t out_w,
                       int32_t absolute, int32_t use_threshold, float threshold, int32_t color_normalize,
                       float* word_maps, const uint8_t* image, int64_t image_map_stride, uint8_t* frames,
                       float* scratch, void* stream);

/*
 * The 256 x 3 colour table daam_overlay_words reads: L[k][ch] = fp32(255 * jet_ch(k / 255)), jet_ch evaluated in
 * float64, piecewise linear through matplotlib's `jet` segment points. out: host fp32 [256][3].
 */
int daam_jet_colormap(float* out);

/*
 * Edge-aware word maps: the guided filter (He, Sun and Tang, "Guided Image Filtering", TPAMI 2013, colour-guide form)
 * of each word's expanded map with the image as guide, on each of n_maps global maps stored back to back. With m[w]
 * what daam_expand_words writes for word w WITHOUT threshold (same rows / row_begin / absolute), I = image / 255 in
 * [0, 1]^3, W(x) the (2 radius + 1)^2 window around x clipped to the image, N(x) = |W(x)| and mean_f(x) = sum_{y in
 * W(x)} f(y) / N(x) (border windows shrink):
 *   mu = mean(I),  Sigma = mean(I I^T) - mu mu^T,  p = mean(m),  c = mean(I m) - mu p,
 *   a = (Sigma + eps Id)^-1 c,  b = p - a^T mu,  q(x) = mean(a)(x)^T I(x) + mean(b)(x)
 * out[i][w] = q, not clamped (it can overshoot [0, 1] slightly), or with use_threshold (q > threshold) as 1.0 / 0.0.
 * Arguments as daam_overlay_words with color_normalize replaced by radius (1 <= radius <= 64) and eps (finite, > 0, in
 * the units of I^2); out: device fp32 [n_maps][n_words][out_h][out_w]. scratch: device, 4-byte aligned, at least
 * DAAM_REFINE_SCRATCH_BYTES(1, 1, out_h, out_w): DAAM_REFINE_GUIDE_BYTES(out_h, out_w) of statistics per image of a
 * round (mu and the inverse, one image when image_map_stride is 0), then DAAM_REFINE_PLANE_BYTES(out_h, out_w) per
 * (map, word) plane of a round. As many planes go in a round as the scratch holds, whole maps while a map's planes fit,
 * and the call loops over the rounds: two launches per image for its statistics (built from exact integer window
 * sums), then five a round (the word maps, and two separable passes of direct fp32 window sums of at most 2 radius + 1
 * values each). The [n_words][out_h][out_w] stack of m is never written. The results are the same bits whatever the
 * scratch and on every call: no atomics.
 * Limits (DAAM_E_UNSUPPORTED): as daam_overlay_words. DAAM_E_INVALID: as daam_overlay_words, plus radius or eps out of
 * range, scratch not 4-byte aligned or scratch_bytes below DAAM_REFINE_SCRATCH_BYTES(1, 1, out_h, out_w).
 */
#define DAAM_REFINE_MAX_RADIUS 64
#define DAAM_REFINE_GUIDE_BYTES(out_h, out_w) (36 * (int64_t)(out_h) * (out_w))
#define DAAM_REFINE_PLANE_BYTES(out_h, out_w) (32 * (int64_t)(out_h) * (out_w) + 256)
#define DAAM_REFINE_SCRATCH_BYTES(n_images, n_planes, out_h, out_w)                                                    \
  ((int64_t)(n_images) * DAAM_REFINE_GUIDE_BYTES(out_h, out_w) + (int64_t)(n_planes) * DAAM_REFINE_PLANE_BYTES(out_h, out_w))
int daam_refine_words(const float* global_maps, int32_t n_maps, int32_t n_rows, int32_t map_h, int32_t map_w,
                      const int32_t* rows, const int32_t* row_begin, int32_t n_words, int32_t out_h, int32_t out_w,
                      int32_t absolute, int32_t use_threshold, float threshold, int32_t radius, float eps,
                      float* word_maps, const uint8_t* image, int64_t image_map_stride, float* out, void* scratch,
                      int64_t scratch_bytes, void* stream);

/*
 * Boundary scores: where each word's mask boundary lies against each of n_regions binary image regions, on each of
 * n_maps global maps stored back to back -- the boundary F-measure at pixel tolerances (DAVIS's contour accuracy,
 * Csurka et al.'s BF score), the Hausdorff distance and the average symmetric surface distance. With A the mask
 * m[w] > threshold (m what daam_expand_words writes for word w WITHOUT threshold, same rows / row_begin / absolute:
 * exactly daam_expand_words' thresholded mask), B_r = {p : regions[r][p] != 0}, the boundary of a mask M
 * dM = {p in M : a 4-neighbour of p is outside M or outside the image}, d2(p, S) = min_{q in S} (p_y - q_y)^2 +
 * (p_x - q_x)^2 (an exact integer between pixel centres) and theta_k = tolerances[k] (host fp32, compared as
 * d2 <= theta_k^2 in float64, exactly):
 *   word_boundary[i][w]      = |dA|                                                 (int32 [n_maps][n_words])
 *   region_boundary[r]       = |dB_r|                                               (int32 [n_regions])
 *   word_hits[i][k][r][w]    = #{p in dA : d2(p, dB_r) <= theta_k^2}    (int32 [n_maps][n_tolerances][n_regions][n_words])
 *   region_hits[i][k][r][w]  = #{q in dB_r : d2(q, dA) <= theta_k^2}    (int32, same shape)
 *   max_d2[i][r][w][0 / 1]   = max over dA of d2(., dB_r) / over dB_r of d2(., dA); -1 in both when dA or dB_r is
 *                              empty                                     (int64 [n_maps][n_regions][n_words][2])
 *   sum_dist[i][r][w][0 / 1] = the same two directions, sum of sqrt(d2), each root in float64; 0 when dA or dB_r is
 *                              empty                                     (double, same shape)
 * Boundary precision is word_hits / |dA|, recall region_hits / |dB_r|, the Hausdorff distance sqrt(max of max_d2) and
 * the ASSD (sum of sum_dist) / (|dA| + |dB_r|). Arguments as daam_region_ranking, plus threshold (finite, always in
 * effect) and 1 <= n_tolerances <= 16 tolerances, finite, >= 0 and strictly ascending; the outputs on the device.
 * scratch: device, 8-byte aligned, at least DAAM_BOUNDARY_SCRATCH_BYTES(n_regions, 1, out_h, out_w):
 * DAAM_BOUNDARY_CALL_BYTES(n_regions, out_h, out_w) for the regions' column distances (about 4 bytes a pixel per
 * region), then DAAM_BOUNDARY_PLANE_BYTES(out_h, out_w) (about 8 bytes a pixel) per (map, word) plane of a round. As
 * many planes go in a round as the scratch holds, whole maps while a map's planes fit, and the call loops over the
 * rounds: two memsets and one launch (the regions' boundaries and column distances), then five launches a round (the
 * values, the planes' boundaries and column distances, one query pass that finds every boundary pixel's nearest
 * boundary pixel of the other set, and a fixed-order reduction). The results are the same bits whatever the scratch
 * and on every call: no float atomics, every sum in an order fixed by pixel positions.
 * Limits (DAAM_E_UNSUPPORTED): those of daam_region_ranking, plus n_tolerances <= 16. DAAM_E_INVALID: as
 * daam_region_ranking, plus a bad tolerance list, a non-finite threshold, scratch not 8-byte aligned or scratch_bytes
 * below DAAM_BOUNDARY_SCRATCH_BYTES(n_regions, 1, out_h, out_w).
 */
#define DAAM_BOUNDARY_MAX_TOLERANCES 16
/* rows of one query tile: 16, or enough for 4096 pixels on narrow images; one tile's partials take 10080 bytes */
#define DAAM_BOUNDARY_TILE_ROWS(out_w) ((out_w) >= 256 ? 16 : (4096 + (int64_t)(out_w) - 1) / (out_w))
#define DAAM_BOUNDARY_CALL_BYTES(n_regions, out_h, out_w)                                                             \
  (8 * (int64_t)(n_regions) * (((int64_t)(out_h) * (out_w) + 1) / 2))
#define DAAM_BOUNDARY_PLANE_BYTES(out_h, out_w)                                                                       \
  (16 * (((int64_t)(out_h) * (out_w) + 1) / 2) + 256 +                                                                \
   10080 * (((int64_t)(out_h) + DAAM_BOUNDARY_TILE_ROWS(out_w) - 1) / DAAM_BOUNDARY_TILE_ROWS(out_w)))
#define DAAM_BOUNDARY_SCRATCH_BYTES(n_regions, n_planes, out_h, out_w)                                                \
  (DAAM_BOUNDARY_CALL_BYTES(n_regions, out_h, out_w) + (int64_t)(n_planes) * DAAM_BOUNDARY_PLANE_BYTES(out_h, out_w))
int daam_region_boundary(const float* global_maps, int32_t n_maps, int32_t n_rows, int32_t map_h, int32_t map_w,
                         const int32_t* rows, const int32_t* row_begin, int32_t n_words, int32_t out_h, int32_t out_w,
                         int32_t absolute, float threshold, const float* tolerances, int32_t n_tolerances,
                         float* word_maps, const uint8_t* regions, int32_t n_regions, int32_t* word_boundary,
                         int32_t* region_boundary, int32_t* word_hits, int32_t* region_hits, int64_t* max_d2,
                         double* sum_dist, void* scratch, int64_t scratch_bytes, void* stream);

/*
 * Boundary scores of n_planes device masks: daam_region_boundary with A = {p : masks[i][p] != 0} (masks: device uint8
 * [n_planes][out_h][out_w]) and n_maps * n_words replaced by n_planes in every output shape (word_boundary [n_planes],
 * word_hits [n_planes][n_tolerances][n_regions], max_d2 [n_planes][n_regions][2], ...). Scratch as daam_region_boundary
 * with n_planes planes; one launch per call and three a round. Limits: n_regions <= 63, out_h * out_w <= 2^24,
 * n_tolerances <= 16. DAAM_E_INVALID: a null pointer or non-positive size, a bad tolerance list, scratch not 8-byte
 * aligned or below DAAM_BOUNDARY_SCRATCH_BYTES(n_regions, 1, out_h, out_w).
 */
int daam_mask_boundary(const uint8_t* masks, int32_t n_planes, int32_t out_h, int32_t out_w, const uint8_t* regions,
                       int32_t n_regions, const float* tolerances, int32_t n_tolerances, int32_t* word_boundary,
                       int32_t* region_boundary, int32_t* word_hits, int32_t* region_hits, int64_t* max_d2,
                       double* sum_dist, void* scratch, int64_t scratch_bytes, void* stream);

/*
 * CRF-refined word segmentation: mean-field inference of a Potts CRF over a word list's maps with the image as a
 * bilateral guide (Kraehenbuehl and Koltun, "Efficient Inference in Fully Connected CRFs with Gaussian Edge Potentials",
 * NeurIPS 2011, in the exact windowed form of Teichmann and Cipolla, "Convolutional CRFs for Semantic Segmentation",
 * BMVC 2019), on each of n_maps global maps stored back to back. With m[w] what daam_expand_words writes for word w
 * WITHOUT threshold (same rows / row_begin / absolute):
 *   labels: with use_threshold L = n_words + 1 and label 0 the background with score s_0 = threshold; without it
 *           L = n_words and no background; word w is always label w + 1 with score s_{w+1} = m[w];
 *   logits: z_l = scale * s_l in fp32;
 *   tables: over the window offsets o != 0 with |o_y|, |o_x| <= radius, computed once per call in float64 and rounded
 *           once to fp32, each normalised over the full window (logit units, whatever the radius):
 *           A[o] = appearance exp(-|o|^2 / 2 sigma_xy^2) / sum_{o' != 0} exp(-|o'|^2 / 2 sigma_xy^2)
 *           S[o] = smoothness exp(-|o|^2 / 2 sigma_smooth^2) / sum_{o' != 0} exp(-|o'|^2 / 2 sigma_smooth^2)
 *   kernel: k(x, y) = A[y - x] exp(-|I_x - I_y|^2 / 2 sigma_rgb^2) + S[y - x], I the RGB bytes (|I_x - I_y|^2 is an
 *           exact integer), over the window W(x) clipped to the image and not renormalised at the border;
 *   mean field (parallel updates): Q^0 = softmax_l(z); each of `iterations` updates takes
 *           msg_l(x) = sum_{y in W(x), y != x} k(x, y) Q_l(y), then Q' = softmax_l(z + msg).
 * labels[i]: uint8 [n_maps][out_h][out_w], the output label (1 + w for word w, 0 for the background) of the argmax of
 * the last logits (z when iterations = 0), the lowest label on ties; scores[i]: fp32, the final Q of that label;
 * probs (may be NULL): fp32 [n_maps][L][out_h][out_w], the final Q. With iterations = 0, or appearance = smoothness =
 * 0, and scale a power of two, labels equal daam_segment_words' bit for bit. The window walk has a fixed order, the
 * softmax subtracts the max, takes expf and sums in label order, and there are no atomics: the results are the same
 * bits on every call and whatever the scratch.
 * Arguments as daam_overlay_words with color_normalize replaced by the CRF's, plus labels / scores / probs on the
 * device. scratch: device, 4-byte aligned, at least DAAM_CRF_SCRATCH_BYTES(1, L, out_h, out_w): two fp32 Q buffers and
 * the min / max partials per map (DAAM_CRF_MAP_BYTES). A map's labels are coupled, so a round takes as many whole maps
 * as the scratch holds and the call loops over the rounds: 2 + iterations launches a round (the word maps, Q^0, one
 * fused launch per update).
 * Limits (DAAM_E_UNSUPPORTED): as daam_overlay_words. DAAM_E_INVALID: as daam_overlay_words, plus radius not in
 * [1, DAAM_CRF_MAX_RADIUS], iterations not in [0, 64], scale or a sigma not finite and > 0, appearance or smoothness not
 * finite and >= 0, a threshold in effect that is not finite, scratch not 4-byte aligned or scratch_bytes below one map.
 * Checked in that order after the null pointers and sizes, and before the word list.
 */
#define DAAM_CRF_MAX_RADIUS 16
#define DAAM_CRF_MAP_BYTES(n_labels, out_h, out_w) (8 * (int64_t)(n_labels) * (out_h) * (out_w) + 256 * (int64_t)(n_labels))
#define DAAM_CRF_SCRATCH_BYTES(n_maps, n_labels, out_h, out_w) ((int64_t)(n_maps) * DAAM_CRF_MAP_BYTES(n_labels, out_h, out_w))
int daam_segment_crf(const float* global_maps, int32_t n_maps, int32_t n_rows, int32_t map_h, int32_t map_w,
                     const int32_t* rows, const int32_t* row_begin, int32_t n_words, int32_t out_h, int32_t out_w,
                     int32_t absolute, int32_t use_threshold, float threshold, float scale, int32_t iterations,
                     int32_t radius, float appearance, float sigma_xy, float sigma_rgb, float smoothness,
                     float sigma_smooth, float* word_maps, const uint8_t* image, int64_t image_map_stride,
                     uint8_t* labels, float* scores, float* probs, void* scratch, int64_t scratch_bytes, void* stream);

/*
 * Word distance maps: the exact signed squared Euclidean distance transform of each word's mask, on each of n_maps
 * global maps stored back to back. With M the mask m[w] > threshold (m what daam_expand_words writes for word w
 * WITHOUT threshold, same rows / row_begin / absolute: exactly daam_expand_words' thresholded mask) and d2 the squared
 * distance between pixel centres (an exact integer):
 *   signed_d2[i][w][p] =  min_{q in M} d2(p, q)        (>= 1)  for p outside M,
 *                      = -min_{q not in M} d2(p, q)    (<= -1) for p in M, q over the image's pixels only: the border
 *                                                              is not background;
 *   every pixel is +DAAM_DISTANCE_NONE for an empty mask and -DAAM_DISTANCE_NONE for a mask that fills the image.
 * signed_d2: int32 [n_maps][n_words][out_h][out_w] on the device. signed_d2 <= r^2 is the mask dilated by the disk of
 * radius r, signed_d2 < -r^2 the mask eroded by it. Each plane takes a column pass (one thread per column: each
 * pixel's vertical distance to the nearest pixel of the other class in its column, signed by its class, written to
 * signed_d2) and a row pass in place (the lower envelope of parabolas of Felzenszwalb and Huttenlocher, "Distance
 * Transforms of Sampled Functions", Theory of Computing 2012, once per class over each row, every comparison exact in
 * 64-bit integers): O(out_h * out_w) work per plane, whatever the distances. Integer arithmetic only: the results are
 * the same bits on every call and whatever the scratch.
 * Arguments as daam_word_instances without max_instances. scratch: device, 4-byte aligned, at least
 * DAAM_DISTANCE_PLANE_BYTES(out_h, out_w): the values `pre` and the min / max partials of one (map, word) plane. As
 * many planes go in a round as the scratch holds, whole maps while a map's planes fit, and the call loops over the
 * rounds: four launches a round (the word maps, the values, the column pass, the row pass).
 * Limits (DAAM_E_UNSUPPORTED): those of daam_word_instances, plus out_h, out_w <= 32767 (every d2 stays below
 * DAAM_DISTANCE_NONE). DAAM_E_INVALID: a null pointer or non-positive size, a non-finite threshold, scratch not 4-byte
 * aligned or scratch_bytes below DAAM_DISTANCE_PLANE_BYTES(out_h, out_w), then the word list as daam_word_instances.
 */
#define DAAM_DISTANCE_NONE INT32_MAX
#define DAAM_DISTANCE_MAX_SIDE 32767
#define DAAM_DISTANCE_PLANE_BYTES(out_h, out_w) (4 * (int64_t)(out_h) * (out_w) + 256)
int daam_word_distance(const float* global_maps, int32_t n_maps, int32_t n_rows, int32_t map_h, int32_t map_w,
                       const int32_t* rows, const int32_t* row_begin, int32_t n_words, int32_t out_h, int32_t out_w,
                       int32_t absolute, float threshold, float* word_maps, int32_t* signed_d2, void* scratch,
                       int64_t scratch_bytes, void* stream);

/*
 * The signed distance transform of n_planes device masks: daam_word_distance with M = {p : masks[i][p] != 0} (masks:
 * device uint8 [n_planes][out_h][out_w]; signed_d2: int32 [n_planes][out_h][out_w]). No scratch: the column distances
 * live in signed_d2. Two launches per 65535 planes. Limits (DAAM_E_UNSUPPORTED): out_h, out_w <= 32767, out_h * out_w
 * <= 2^24. DAAM_E_INVALID: a null pointer or non-positive size.
 */
int daam_mask_distance(const uint8_t* masks, int32_t n_planes, int32_t out_h, int32_t out_w, int32_t* signed_d2,
                       void* stream);

/*
 * SLIC superpixels (Achanta et al., "SLIC Superpixels Compared to State-of-the-Art Superpixel Methods", TPAMI 2012) of
 * n_images uint8 RGB images [n_images][out_h][out_w][3] stored back to back, in the pixel-centric form on the RGB bytes,
 * every step defined exactly:
 *   grid:   S = sqrt(H W / K) in float64 (K = n_segments), ny = clamp(floor(H / S + 0.5), 1, H), nx likewise with W;
 *           cell row cy holds the pixel rows [floor(cy H / ny), floor((cy + 1) H / ny)), so pixel row y lies in cell row
 *           floor(((y + 1) ny - 1) / H); columns likewise; cluster k = cy nx + cx, ny nx <= DAAM_SUPERPIXEL_MAX_CELLS;
 *   start:  each cluster's sums (r, g, b, y, x, n), int64, are those of the one pixel ((y0 + y1 - 1) // 2,
 *           (x0 + x1 - 1) // 2) of its cell [y0, y1) x [x0, x1) (no gradient perturbation);
 *   pass:   each pixel takes, among the up to 9 clusters whose cells are within one cell row and column of its own,
 *           the lowest D = ((dr dr + dg dg) + db db) + wxy ((dy dy) + (dx dx)), the differences to the centre
 *           sum / n, every operation rounded separately in float64 (no FMA); wxy = c c (ny nx) / (H W) left to right
 *           in float64, c = compactness (the RGB channels are 0..255); the lowest cluster wins a tie;
 *   update: between the `iterations` passes each cluster's sums become the integer sums over its pixels; a cluster
 *           without pixels keeps its sums.
 * superpixels: int32 [n_images][out_h][out_w], each pixel's cluster after the last pass. Superpixels may be disconnected
 * and an empty cluster leaves its id unused. The sums are integers (integer atomics, exact whatever their order) and
 * the distances exact float64 operations: the results are the same bits on every call and whatever the scratch.
 * scratch: device, 8-byte aligned, at least DAAM_SUPERPIXEL_IMAGE_BYTES(ny, nx): as many images go in a round as it
 * holds, 2 * iterations launches a round (the start, one launch per pass, one update between passes).
 * Limits (DAAM_E_UNSUPPORTED): out_h * out_w <= 2^24, ny nx <= DAAM_SUPERPIXEL_MAX_CELLS. DAAM_E_INVALID: a null
 * pointer or non-positive size, then n_segments < 1, compactness not finite and > 0, iterations not in [1, 64], then
 * (after the cell limit) scratch not 8-byte aligned or below one image.
 */
#define DAAM_SUPERPIXEL_MAX_CELLS 65536
#define DAAM_SUPERPIXEL_IMAGE_BYTES(ny, nx) (96 * (int64_t)(ny) * (nx))
/* the cells a 16 x 64 pixel tile's pixels can be assigned to lie in a box of at most this many */
#define DAAM_SUPERPIXEL_BOX(ny, nx, out_h, out_w)                                                     \
  ((int64_t)((ny) < 15 * (ny) / (out_h) + 4 ? (ny) : 15 * (ny) / (out_h) + 4) *                         \
   ((nx) < 63 * (nx) / (out_w) + 4 ? (nx) : 63 * (nx) / (out_w) + 4))
#define DAAM_SUPERPIXEL_MAP_BYTES(n_words, ny, nx, out_h, out_w)                                        \
  (256 * (int64_t)(n_words) + 8 * (int64_t)(ny) * (nx) +                                                \
   8 * (int64_t)(n_words) * (((out_h) + 15) / 16) * (((out_w) + 63) / 64) * DAAM_SUPERPIXEL_BOX(ny, nx, out_h, out_w))
#define DAAM_SUPERPIXEL_SCRATCH_BYTES(n_images, n_maps, n_words, ny, nx, out_h, out_w)                  \
  ((int64_t)(n_images) * DAAM_SUPERPIXEL_IMAGE_BYTES(ny, nx) +                                          \
   (int64_t)(n_maps) * DAAM_SUPERPIXEL_MAP_BYTES(n_words, ny, nx, out_h, out_w))
int daam_image_superpixels(const uint8_t* image, int32_t n_images, int32_t out_h, int32_t out_w, int32_t n_segments,
                           float compactness, int32_t iterations, int32_t* superpixels, void* scratch,
                           int64_t scratch_bytes, void* stream);

/*
 * Superpixel word segmentation: the words compete per SLIC superpixel of the image rather than per pixel, on each of
 * n_maps global maps stored back to back. The partition is daam_image_superpixels' of the image, made inside the call:
 * one for every map with image_map_stride 0, else one per map (map i's image at image + i * image_map_stride). With
 * m[w] what daam_expand_words writes for word w WITHOUT threshold (same rows / row_begin / absolute) and n_s the
 * pixel count of superpixel s:
 *   mean[w][s] = fp32(sum_{p in s} m[w](p) / n_s), the sum in float64 in a fixed order (no float atomics);
 *   labels[i][p] = 1 + argmax_w mean[w][s(p)] (the lowest word on ties), or 0 (background) where use_threshold and
 *                  !(max_w mean[w][s(p)] > threshold); scores[i][p] = max_w mean[w][s(p)].
 * labels: uint8 and scores: fp32 [n_maps][out_h][out_w]; superpixels: int32 [out_h][out_w] with one image, [n_maps]
 * [out_h][out_w] with one per map. With one-pixel cells (n_segments = out_h * out_w) every superpixel is its pixel and
 * labels / scores equal daam_segment_words' bit for bit. Each sum of m runs in an order fixed by pixel positions (per
 * 16 x 64 tile in row-major order, then over the tiles in a fixed order) and the SLIC state is integer: the results
 * are the same bits on every call and whatever the scratch.
 * Arguments as daam_segment_crf without its CRF arguments, plus n_segments / compactness / iterations as
 * daam_image_superpixels and the superpixels output. scratch: device, 8-byte aligned, at least
 * DAAM_SUPERPIXEL_SCRATCH_BYTES(1, 1, n_words, ny, nx, out_h, out_w): each image's SLIC state
 * (DAAM_SUPERPIXEL_IMAGE_BYTES) and each map's min / max partials, per-tile sums and per-superpixel results
 * (DAAM_SUPERPIXEL_MAP_BYTES). A round takes as many whole maps (and with one image per map, their images) as the
 * scratch holds and the call loops over the rounds: 4 launches a round (the word maps, the tile sums, the
 * per-superpixel means, the labels), plus 2 * iterations for each round's partitions (the first round's only, with
 * one image).
 * Limits (DAAM_E_UNSUPPORTED): out_h * out_w <= 2^24 and ny nx <= DAAM_SUPERPIXEL_MAX_CELLS, then the word list's
 * (n_words <= 96, as daam_segment_words). DAAM_E_INVALID: a null pointer or non-positive size, then n_segments < 1,
 * compactness not finite and > 0, iterations not in [1, 64], then (after the cell limit) scratch not 8-byte aligned
 * or below one image and one map, then the word list as daam_segment_words.
 */
int daam_segment_superpixels(const float* global_maps, int32_t n_maps, int32_t n_rows, int32_t map_h, int32_t map_w,
                             const int32_t* rows, const int32_t* row_begin, int32_t n_words, int32_t out_h,
                             int32_t out_w, int32_t absolute, int32_t use_threshold, float threshold,
                             int32_t n_segments, float compactness, int32_t iterations, float* word_maps,
                             const uint8_t* image, int64_t image_map_stride, uint8_t* labels, float* scores,
                             int32_t* superpixels, void* scratch, int64_t scratch_bytes, void* stream);

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
