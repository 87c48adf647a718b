"""The tracer: ``with trace(pipe) as tc: pipe(prompt); tc.compute_global_heat_map()`` on H100-native kernels.

Mirror of the reference's L1 (``daam/trace.py``): same classes, constructor arguments, methods and
exceptions; what differs is what runs underneath.

* The attention processor (:class:`UNetCrossAttentionHooker`, reference trace.py:189-315) owns the whole attn2 forward
  like the reference's, but never materialises the probabilities: the layer output comes from SDPA, and the
  heat-map side of the call -- ``get_attention_scores`` + ``_unravel_attn`` + the per-head ``update`` loop (trace.py:
  276, 219-244, 293-294) -- is one fused CUDA kernel (``daam_accumulate``) reading the Q/K projections in place.
* Kernel work is queued per denoising step and issued as ONE persistent launch covering every traced layer of the step
  at the end of the UNet forward, on the forward's own stream (``launch='step'``, default: one CUDA call per step, the
  kernel is 0.2 % of a step) or on a side stream so that it also overlaps the next step's first kernels
  (``launch='overlap'``: four CUDA calls per step); ``launch='layer'`` issues it immediately per layer.
* ``compute_global_heat_map`` (trace.py:83-132) keeps the Python-side key filter and error messages and runs the
  bicubic-upsample / clamp / mean / normalise reduction as one kernel (``daam_finalize``).
* ``time_resolved=True`` also answers *when* a word's attribution forms: the step launch becomes
  ``daam_accumulate_steps`` (the kernel also stores what it adds into a second slab per layer) followed by one
  ``daam_finalize`` per prompt over those step slabs, into that step's slot of a device history
  (``compute_time_heat_maps``).
* ``step_ranges=[(a, b), ...]`` answers what DAAM attributes during chosen spans of steps: every traced layer gets one
  more zeroed slab per declared range, and while the UNet forward index lies in range ``i`` the step launch becomes
  ``daam_accumulate_range``, which also adds what it adds into range ``i``'s slabs. Each range slab then is the
  accumulator a trace of only those steps would hold, so every read (``step_range=i``) reduces it exactly as the full
  run's accumulator is reduced.
* ``negative=True`` also keeps the map of the unconditional half of the CFG batch: the model attending to the negative
  prompt (or the empty one). Every layer's slab is twice as tall, ``[uncond x N, cond x N]`` like the batch, and its
  one descriptor covers the whole batch from sample 0, so the launches stay as they are with twice the tiles. Every read
  takes ``negative=True`` and then reduces the lower half against the negative text.
* ``value_norms=True`` also keeps, per traced layer, ``||W_h v||`` of every (sample, head, context row): what that row
  carries through that head after the output projection (``daam_value_norms``, once per layer and generation: the
  context does not change between steps). ``value_weighted=True`` reads then weight every key's clamped map by it
  (``daam_finalize_parts_weighted``); the accumulate launches do not change.

Accumulators are fp32 regardless of the pipeline dtype (the reference accumulates in the pipeline dtype, SURVEY.md
section 5); parity is stated against the fp32 oracle fed the same Q/K.
"""
from __future__ import annotations

import inspect
import math
import weakref
from pathlib import Path
from typing import Dict, List, Optional, Tuple, Type, Union

import torch
import torch.nn.functional as F

from . import _native, ops
from .geometry import FluxGeometry, JointGeometry, LatentGeometry
from .heatmap import (FactorHeatMaps, GlobalHeatMap, HeadHeatMaps, ImageHeatMaps, LayerHeatMaps, LayerSlab,
                      RawHeatMapCollection, TimeHeatMaps)
from .hook import AggregateHooker, ObjectHooker, UNetCrossAttentionLocator
from .locate import JointAttentionLocator
from .utils import T5Pieces, cache_dir, context_rows, t5_rows

__all__ = ['trace', 'DiffusionHeatMapHooker', 'GlobalHeatMap', 'UNetCrossAttentionHooker', 'JointAttentionHooker',
           'FluxAttentionHooker', 'PipelineHooker', 'ImageProcessorHooker']

class DiffusionHeatMapHooker(AggregateHooker):
    """Context manager that traces every located cross-attention layer of ``pipeline.unet`` (trace.py:22-59).

    Extra keyword-only options (not in the reference): ``launch`` ('step' | 'overlap' | 'layer', see module docstring),
    ``batch_prompts`` (accept several prompts per generation: N independent single-prompt traces sharing each launch;
    the reference rejects this, trace.py:172-173), ``locate_middle_block`` (also locate the mid block without
    enabling save/load of heads -- BASELINE config 5 "all 16+70 layers"), ``time_resolved`` (also keep one global
    heat map per denoising step, see :meth:`compute_time_heat_maps`) and ``step_ranges`` (a list of half-open
    ``(start, stop)`` tuples or ``range`` objects over UNet-forward indices of a generation, counted as
    :class:`TimeHeatMaps` counts them: also keep the per-key sums over each of those spans; read them with
    ``step_range=i`` in :meth:`compute_global_heat_map`, :meth:`compute_per_head_heat_maps` and
    ``all_heat_maps.items``), ``negative`` (also keep the maps of the unconditional half of the guidance batch, the
    negative prompt's; read them with ``negative=True`` in every read) and ``long_prompts`` (also trace contexts of 154
    and 231 tokens, two or three CLIP chunks such as chunked ``prompt_embeds`` give: every context row is accumulated,
    and every read returns the compact ``n_tokens + 2`` rows that :func:`~daam_b200.utils.context_rows` names; any
    other context length raises at the layer call; not with ``time_resolved``, ``step_ranges``, ``save_heads`` or
    ``load_heads``) and ``value_norms`` (also keep every key's value norms, for the ``value_weighted=True`` reads and
    :meth:`compute_value_norms`; not with ``save_heads`` / ``load_heads`` or CUDA-graph capture).

    A pipeline whose denoiser is an MM-DiT ``transformer`` and that has no ``unet`` (Stable Diffusion 3 / 3.5) is traced
    through the joint attention of every ``transformer.transformer_blocks[i].attn`` (:class:`JointAttentionHooker`):
    a map is the image-query x text-key block of each joint softmax, summed over steps (``daam_accumulate_joint``).
    Reads return the CLIP rows by default and the T5 rows with ``encoder='t5'``. Such a trace refuses the options it
    does not implement (see :data:`JOINT_REFUSED`) with a ``ValueError``.

    A FLUX.1 pipeline (a ``transformer`` with ``single_transformer_blocks``) is traced through the double-stream
    ``transformer_blocks[i].attn`` and then the single-stream ``single_transformer_blocks[j].attn``
    (:class:`FluxAttentionHooker`), whose sequences are ``[text, image]``. Every sample of its guidance-distilled batch
    is kept with all heads, reads return the T5 rows of ``prompt_2`` (or of the prompt), and it refuses what an SD3
    trace refuses, negative prompts included.

    ``reduce_heads=True`` (SD3 and FLUX traces only) keeps each layer's mean over heads instead of every head: the
    accumulate kernel (``daam_accumulate_joint_heads``) sums a sample's heads before anything reaches memory, so a
    layer's slab is ``[prompts, images, T, hw]``, 1/heads of the per-head one. A joint key has its grid's own size, so
    the finalize neither resamples nor clamps it, and every read that averages over heads returns the same maps up to
    rounding: the global, layer, factor and image maps, ``to_experiment`` and the word-list calls. Reads of single
    heads (``head_idx``, :meth:`compute_per_head_heat_maps`, :meth:`compute_head_heat_maps`, ``all_heat_maps.items``)
    raise. Every traced layer must have the same number of heads. A UNet trace refuses it: there every key is
    upsampled and clamped before the mean over keys, so the head sum cannot be taken first.
    """

    def __init__(self, pipeline, low_memory: bool = False, load_heads: bool = False, save_heads: bool = False,
                 data_dir: str = None, *, launch: str = 'step', batch_prompts: bool = False,
                 locate_middle_block: bool = False, kernel_flags: int = _native.ACC_AUTO, time_resolved: bool = False,
                 step_ranges=None, negative: bool = False, long_prompts: bool = False, value_norms: bool = False,
                 reduce_heads: bool = False):
        if launch not in ('step', 'overlap', 'layer'):
            raise ValueError("launch must be 'step', 'overlap' or 'layer'")
        if value_norms and (save_heads or load_heads):
            raise ValueError('value_norms=True does not support save_heads / load_heads: those layer calls replay '
                             'stored probabilities, not the value projection')
        if long_prompts:
            for name, on in (('time_resolved=True', time_resolved), ('step_ranges', step_ranges is not None),
                             ('save_heads', save_heads), ('load_heads', load_heads)):
                if on:
                    raise ValueError(f'long_prompts=True does not support {name}: it traces 77-token contexts only')
        modes = []                             # the enabled second-slab modes, and why each needs the step launch
        if step_ranges is not None:
            step_ranges = _normalize_step_ranges(step_ranges)
            modes.append(('step_ranges', 'which range a launch adds into depends on the UNet forward it ends'))
        if time_resolved:
            modes.append(('time_resolved=True', "the per-step heat map is finalized right after the step's launch"))
        for name, why in modes:
            if launch != 'step':
                raise ValueError(f"{name} needs launch='step': {why}, on the forward's own stream")
            if save_heads or load_heads:
                raise ValueError(f'{name} does not support save_heads / load_heads')
        if len(modes) > 1:
            raise ValueError('step_ranges cannot be combined with time_resolved=True')
        self.joint = getattr(pipeline, 'unet', None) is None and getattr(pipeline, 'transformer', None) is not None
        # FLUX.1: a joint trace whose transformer also has single-stream blocks (text-first, no CFG half)
        self.flux = self.joint and getattr(pipeline.transformer, 'single_transformer_blocks', None) is not None
        if reduce_heads and not self.joint:
            raise ValueError('reduce_heads=True needs a joint-attention (SD3 / FLUX) trace: a UNet layer upsamples and '
                             'clamps every key before the mean over keys, so the heads cannot be summed first')
        if self.joint:
            model = 'a FLUX' if self.flux else 'an SD3'
            options = dict(time_resolved=time_resolved, step_ranges=step_ranges is not None, negative=negative,
                           long_prompts=long_prompts, value_norms=value_norms, save_heads=save_heads,
                           load_heads=load_heads, low_memory=low_memory, locate_middle_block=locate_middle_block)
            for name in JOINT_REFUSED:
                if options[name]:
                    raise ValueError(f'{name} is not supported when tracing the joint attention of {model} '
                                     f'transformer')
            if launch == 'overlap':
                raise ValueError(f"launch='overlap' is not supported when tracing the joint attention of {model} "
                                 f"transformer: use 'step' or 'layer'")
        _native.load()   # fail here, loudly, if the CUDA library is missing
        self.all_heat_maps = RawHeatMapCollection()
        self.all_heat_maps.joint = self.joint
        self.reduce_heads = reduce_heads
        self.all_heat_maps.reduce_heads = reduce_heads
        if self.flux:
            # FLUX: the grid is the image size check_inputs receives, in 2 x 2 packed latent patches
            self.latent_hw = self._sample_size = None
            self.geometry = FluxGeometry(pipeline.vae_scale_factor)
            self.locator = JointAttentionLocator()
        elif self.joint:
            # joint mode: the grid is the latent in patches, known from the first transformer forward
            self.latent_hw = self._sample_size = None
            self.geometry = JointGeometry(pipeline.transformer.config.patch_size)
            self.locator = JointAttentionLocator()
        else:
            side = pipeline.unet.config.sample_size * pipeline.vae_scale_factor
            self.latent_hw = 4096 if side in (512, 1024) else 9216   # 64x64, or 96x96 for the 768-pixel models
            # the heat-map grid and every layer's (h, w, factor): square until the first UNet forward shows the latent
            # (a forward pre-hook on the UNet re-derives it whenever the latent's (H, W) changes)
            self._sample_size = pipeline.unet.config.sample_size
            self.geometry = LatentGeometry(self.latent_hw, self._sample_size)
            self.locator = UNetCrossAttentionLocator(restrict={0} if low_memory else None,
                                                     locate_middle_block=locate_middle_block or load_heads or save_heads)
        self.last_prompts_3: List[Optional[str]] = []   # joint mode: the T5 text (prompt_3) of every prompt, or None
        self.last_prompts_2: List[Optional[str]] = []   # FLUX: the T5 text (prompt_2) of every prompt, or None
        self._flux_tokens: Optional[int] = None   # FLUX: the context rows T of the running transformer forward
        self._joint_pending: List[_native.DaamJointLayer] = []   # joint mode: the layer calls of the running forward
        self.last_prompt: str = ''
        self.last_prompts: List[str] = []
        self.last_negative_prompts: List[str] = []   # negative=True: the negative text of every prompt ('' for none)
        self.negative = negative
        self.all_heat_maps.negative = negative
        self.long_prompts = long_prompts
        self.value_norms = value_norms
        self.all_heat_maps.value_norms = value_norms
        # value-norm mode: layer -> (slab, weakref to the context, (data_ptr, shape, strides, _version)) of the call
        # whose norms the slab holds; emptied at every generation's check_inputs
        self._norms_seen: Dict[int, tuple] = {}
        self.last_image = None
        self.last_images: list = []   # every image of the last generation, prompt-major (``out.images[p * n + i]``)
        self.time_idx = 0
        self._gen_idx = 0
        self.launch = launch
        self.batch_prompts = batch_prompts
        self.kernel_flags = kernel_flags
        # step queue: the layer calls of the running UNet forward, kept as one reusable host-side daam_layer[] whose slots
        # are rewritten in place (in the steady state a layer only stores two pointers into its slot)
        self._packed = _native.PackedLayers([_native.DaamLayer()] * 64)
        self._slots = [self._packed.array[i] for i in range(64)]      # ctypes proxies into the array, created once
        self._n_pending = 0
        self._refs: List[torch.Tensor] = []    # the queued projections, kept alive until their launch has run
        self._parked: List[list] = []          # projections of launches that may still be running
        self._layer_state: Dict[int, tuple] = {}   # layer -> (q shape, dtype, position, slot, slab, q_off, k_off, device, own)
        self._queued: Dict[int, int] = {}      # layer -> id of the step it was last queued in
        self._step_id = 1
        self._epoch_seen = -1                  # RawHeatMapCollection.epoch the cached layer states belong to
        self._device = None
        self._launcher: Optional[_native.SideLauncher] = None
        self._stream: Optional[torch.cuda.Stream] = None
        self._dirty = False                    # side-stream work not yet ordered before the current stream
        self.all_heat_maps.bind(self.synchronize, self._zero_slabs)
        # time-resolved mode: device histories [capacity, n_rows, xh, xw] of per-step global heat maps (grown by
        # doubling, restarted every generation), keyed by `negative` (the negative histories exist with the mode only)
        # and then by (prompt, None) for a prompt's map over all its images, or by (prompt, image) for one image's map
        # (kept only when a generation has several images per prompt)
        self.time_resolved = time_resolved
        self.all_heat_maps.time_resolved = time_resolved
        self._history: Dict[bool, Dict[Tuple[int, Optional[int]], torch.Tensor]] = {False: {}, True: {}}
        self._time_steps = 0
        self._history_rows: Optional[Dict[bool, List[int]]] = None   # n_rows of every prompt of the running generation
        # step-range mode: the UNet forward index of the running generation
        self.step_ranges: Optional[List[Tuple[int, int]]] = step_ranges
        self.all_heat_maps.n_ranges = len(step_ranges) if step_ranges else 0
        self.all_heat_maps.range_steps = [0] * self.all_heat_maps.n_ranges
        self._forward_idx = 0
        # the second slab of every slot of the step array (LayerSlab.second): one array of step slabs in time-resolved
        # mode, one array of range slabs per declared range in step-range mode, none otherwise
        self._slab_ptrs = [_native.StepPointers([0] * 64)
                           for _ in range(1 if time_resolved else self.all_heat_maps.n_ranges)]

        if self.joint:
            hooker = FluxAttentionHooker if self.flux else JointAttentionHooker
            modules = [hooker(m, self, layer_idx=idx) for idx, m in enumerate(self.locator.locate(pipeline.transformer))]
        else:
            modules = [
                UNetCrossAttentionHooker(m, self, layer_idx=idx, latent_hw=self.latent_hw, load_heads=load_heads,
                                         save_heads=save_heads, data_dir=data_dir)
                for idx, m in enumerate(self.locator.locate(pipeline.unet))
            ]
        self._attn_hookers = list(modules)
        modules.append(PipelineHooker(pipeline, self))
        if (self.joint or type(pipeline).__name__ == 'StableDiffusionXLPipeline') \
                and getattr(pipeline, 'image_processor', None):
            modules.append(ImageProcessorHooker(pipeline.image_processor, self))
        super().__init__(modules)
        self.pipe = pipeline

    # -- small reference API ------------------------------------------------------------------------------------------
    def time_callback(self, *args, **kwargs):
        self.time_idx += 1

    @property
    def layer_names(self):
        return self.locator.layer_names

    def to_experiment(self, path, seed=None, id='.', subtype='.', **compute_kwargs):
        """Exports the last generation call to a serializable generation experiment (trace.py:68-81). With
        ``negative=True`` it records the negative map and the text it belongs to; with ``image_idx=i`` image ``i``'s map
        and image ``i`` of the prompt (``prompt_idx``)."""
        from .experiment import GenerationExperiment
        heat_map = self.compute_global_heat_map(**compute_kwargs)
        image = self.last_image
        if compute_kwargs.get('image_idx') is not None:
            per_prompt = len(self.last_images) // max(1, len(self._texts()))
            image = self.last_images[compute_kwargs.get('prompt_idx', 0) * per_prompt + compute_kwargs['image_idx']]
        if self.flux:   # a T5 map: its own text (prompt_2 when given) and piece lookup
            return GenerationExperiment(image, heat_map.heat_maps, heat_map.prompt, seed=seed, id=id, subtype=subtype,
                                        path=path, tokenizer=heat_map.tokenizer)
        return GenerationExperiment(
            image,
            heat_map.heat_maps,
            heat_map.prompt if compute_kwargs.get('negative') else self.last_prompt,
            seed=seed, id=id, subtype=subtype, path=path, tokenizer=self.pipe.tokenizer,
        )

    def _hook_impl(self):
        super()._hook_impl()
        unet = self.pipe.transformer if self.joint else self.pipe.unet   # the denoiser: one forward per step
        self._forward_hook = None
        self._pre_hook = None
        if self.launch != 'layer' and hasattr(unet, 'register_forward_hook'):
            # end of every UNet forward = end of the step's layer calls: issue the step launch right away
            self._forward_hook = unet.register_forward_hook(lambda *_: self.flush())
        if hasattr(unet, 'register_forward_pre_hook'):
            # start of every UNet forward: the latent's (H, W) decides the heat-map geometry (one shape comparison)
            self._pre_hook = unet.register_forward_pre_hook(self._see_sample, with_kwargs=True)

    def _unhook_impl(self):
        self.synchronize()      # issue what is queued and order it (and the parked projections) before the caller's stream
        if getattr(self, '_forward_hook', None) is not None:
            self._forward_hook.remove()
            self._forward_hook = None
        if getattr(self, '_pre_hook', None) is not None:
            self._pre_hook.remove()
            self._pre_hook = None
        super()._unhook_impl()

    # -- geometry -----------------------------------------------------------------------------------------------------
    def _see_sample(self, _module, args, kwargs):
        """UNet forward pre-hook: the latent ``sample`` (``args[0]`` or ``kwargs['sample']``) fixes the geometry; in
        joint mode the transformer's ``hidden_states``. FLUX: the context rows ``T`` of ``encoder_hidden_states``,
        which the single-stream blocks cannot see (the grid comes from ``check_inputs``)."""
        if self.flux:
            ctx = kwargs.get('encoder_hidden_states', args[1] if len(args) > 1 else None)
            if ctx is not None:
                self._flux_tokens = ctx.shape[1]
            return
        if self.joint:
            sample = args[0] if args else kwargs.get('hidden_states')
            if sample is not None and tuple(sample.shape[-2:]) != self.geometry.latent_shape:
                self.geometry = JointGeometry(self.geometry.patch_size, tuple(sample.shape[-2:]))
            return
        sample = args[0] if args else kwargs.get('sample')
        if sample is not None and tuple(sample.shape[-2:]) != self.geometry.latent_shape:
            self.set_latent_shape(tuple(sample.shape[-2:]))

    def set_latent_shape(self, shape: Tuple[int, int]):
        """Re-derive the heat-map geometry for a latent of spatial size ``shape = (H, W)``. When the layer rule changes
        (e.g. 512x768 after 768x512: same query counts, transposed keys) every cached layer descriptor and factor is
        dropped, so the next call of each layer re-tags its slab with the new ``(h, w)``."""
        geometry = LatentGeometry(self.latent_hw, self._sample_size, shape)
        if geometry.key != self.geometry.key:
            self._layer_state.clear()
            for hooker in self._attn_hookers:
                hooker._geom = None
        self.geometry = geometry

    # -- kernel queue -------------------------------------------------------------------------------------------------
    def _side_stream(self, device) -> torch.cuda.Stream:
        if self._stream is None or self._stream.device != torch.device(device):
            self._stream = torch.cuda.Stream(device=device)
        return self._stream

    def _enqueue(self, layer_idx: int, factor: int, q: torch.Tensor, k: torch.Tensor, heads: int, scale: float):
        """Register one traced layer call: ``q [B, hw, C]``, ``k [B, 77, C]`` straight from ``to_q`` / ``to_k``.

        This runs once per layer per step on the host's critical path, so the steady state does as little as possible:
        when the projections are contiguous, shaped like the layer's previous call and the layer arrives at the same
        position of the step as last time, only the two data pointers of its slot in the step's ``daam_layer[]`` change."""
        if self._queued.get(layer_idx) == self._step_id:   # the layer comes round again: a new UNet forward has started
            self.flush()
        heat_maps = self.all_heat_maps
        if heat_maps.epoch != self._epoch_seen:            # a slab was (re)allocated: cached descriptors may be stale
            self._layer_state.clear()
            self._epoch_seen = heat_maps.epoch
        pos = self._n_pending if self.launch != 'layer' else 0
        st = self._layer_state.get(layer_idx)
        if st is not None and q.shape == st[0] and q.dtype is st[1] and st[2] == pos and q.is_contiguous() \
                and k.is_contiguous() and q.get_device() == st[7]:
            slot, slab = st[3], st[4]
            slot.q = q.data_ptr() + st[5]
            slot.k = k.data_ptr() + st[6]
            if not slab.touched:
                heat_maps.mark_live(slab)
        else:
            st, q, k = self._describe(layer_idx, factor, q, k, heads, scale, pos)    # (q, k: contiguous copies if it made any)
            slab = st[4]
        if self.launch == 'layer':
            if torch.cuda.is_current_stream_capturing():
                slab.captured = True
            self._launch_now(st[8], q.device)
            return
        self._refs.append(q)                               # kept alive until the step's launch has run
        self._refs.append(k)
        self._queued[layer_idx] = self._step_id
        self._n_pending = pos + 1

    def _describe(self, layer_idx: int, factor: int, q: torch.Tensor, k: torch.Tensor, heads: int, scale: float, pos: int):
        """Slow path of :meth:`_enqueue`: (re)build the layer's slab and descriptor and cache them. Returns the state and
        the tensors the descriptor points into (the caller keeps those alive, not the originals)."""
        if not q.is_cuda:
            raise RuntimeError('daam_b200 traces pipelines that live on a CUDA device only (there is no CPU '
                               'fallback)')
        if q.stride(-1) != 1 or k.stride(-1) != 1:
            q, k = q.contiguous(), k.contiguous()
        bsz, hw, _ = q.shape
        h, w, _ = self.geometry.level(hw, layer_idx)
        if h is None:
            raise RuntimeError(f'layer {layer_idx}: {hw} query positions are not a square map')
        self._check_guidance(layer_idx, bsz)
        # "second half of the batch*heads axis" (trace.py:240): the conditional samples of a CFG batch
        _, n_samples, head0, n_heads = ops.cond_half(bsz, heads)
        n_real, images = self._prompt_layout(layer_idx, n_samples)
        slab = self.all_heat_maps.slab_for(layer_idx, factor, n_real, images * n_heads, h, w, q.device, head0, images,
                                           k.shape[1])
        self._epoch_seen = self.all_heat_maps.epoch        # (this call may have bumped it; the other layers' slabs stand)
        if self.negative:                                  # one descriptor over the whole batch, into the whole slab
            desc = ops.make_layer_desc(q, k, slab.storage.view(bsz, n_heads, slab.acc.shape[2], hw), heads, scale,
                                       whole_batch=True)
        else:
            desc = ops.make_layer_desc(q, k, slab.acc.view(n_samples, n_heads, slab.acc.shape[2], hw), heads, scale)
        if self.launch != 'layer':
            if pos >= len(self._slots):                    # grow the step array (SDXL: 70 layers)
                grown = _native.PackedLayers([_native.DaamLayer()] * (2 * len(self._slots)))
                for i in range(pos):
                    grown.array[i] = self._packed.array[i]
                self._packed = grown
                self._slots = [grown.array[i] for i in range(len(grown.array))]
                self._layer_state.clear()                  # cached slot proxies point into the old array
                self._slab_ptrs = [_native.StepPointers(list(p.array) + [0] * (len(grown.array) - len(p.array)))
                                   for p in self._slab_ptrs]
            self._packed.array[pos] = desc
            for ptrs, second in zip(self._slab_ptrs, slab.second):
                ptrs.array[pos] = second.data_ptr()
            slot, own = self._slots[pos], None
        else:
            own = _native.PackedLayers([desc])             # 'layer' mode: every layer launches its own 1-element array
            slot = own.array[0]
        # the fast path is only valid for contiguous projections (strides implied by the shape)
        shape_key = q.shape if (q.is_contiguous() and k.is_contiguous()) else None
        state = (shape_key, q.dtype, pos, slot, slab, desc.q - q.data_ptr(), desc.k - k.data_ptr(), q.get_device(), own)
        self._layer_state[layer_idx] = state
        self._device = q.device
        return state, q, k

    def _prompt_layout(self, layer_idx: int, n_samples: int) -> Tuple[int, int]:
        """``(prompts, images per prompt)`` of a layer call's ``n_samples`` conditional samples.

        Samples vs prompts: diffusers repeats every prompt num_images_per_prompt times (prompt-major), and the
        reference's keys then enumerate images x heads of its single prompt (the "head" index of a key runs over the
        whole kept axis, trace.py:240, 293-294). A slab is therefore [prompts][images * heads]; the kernel sees the same
        memory as [samples][heads]."""
        n_real = len(self.last_prompts) if self.last_prompts else (n_samples if self.batch_prompts else 1)
        if n_real > 1 and not self.batch_prompts:
            raise ValueError('Only single prompt generation is supported for heat map computation.')
        if n_samples % n_real != 0:
            raise RuntimeError(f'layer {layer_idx}: {n_samples} conditional samples for {n_real} prompts')
        return n_real, n_samples // n_real

    def _check_guidance(self, layer_idx: int, bsz: int):
        """``negative=True`` keeps the unconditional half of a CFG batch: a batch without one is an error."""
        if self.negative and bsz % 2:
            raise RuntimeError(f'layer {layer_idx}: negative=True needs classifier-free guidance, but a batch of {bsz} '
                               f'is not a CFG pair batch [uncond x N, cond x N]')

    def _see_values(self, layer_idx: int, ctx: torch.Tensor, value: torch.Tensor, weight: torch.Tensor, heads: int):
        """Value-norm mode, after the layer's call was queued: the first call of a generation writes the layer's norms
        into its slab. A later call whose context is the same tensor, unmodified, does nothing (the norms are a function
        of the context); one with another context recomputes them into scratch and sets the slab's device flag if they
        differ from the stored ones, with no host synchronisation. A value-weighted read raises on that flag."""
        slab = self.all_heat_maps.slabs[layer_idx]
        ident = (ctx.data_ptr(), tuple(ctx.shape), ctx.stride(), ctx._version)
        seen = self._norms_seen.get(layer_idx)
        if seen is not None and seen[0] is slab and seen[1]() is ctx and seen[2] == ident:
            return
        if seen is None or seen[0] is not slab:            # first call of the generation, or a new slab
            out = slab.norms.view(-1, slab.heads // slab.images, slab.tokens)
            ops.value_norms(value, weight, heads, out, whole_batch=self.negative)
            slab.norms_changed.zero_()
        else:
            fresh = ops.value_norms(value, weight, heads, whole_batch=self.negative)
            slab.norms_changed.logical_or_((fresh.view_as(slab.norms) != slab.norms).any())
        self._norms_seen[layer_idx] = (slab, weakref.ref(ctx), ident)

    def _enqueue_joint(self, layer_idx: int, q: torch.Tensor, k: torch.Tensor, lse: torch.Tensor, n_image: int,
                       heads: int, scale: float):
        """Joint mode: register one layer call, ``q`` / ``k`` ``[B, heads, n_image + T, d]`` (image tokens, then the
        context; FLUX: the context, then the image tokens) and the attention's ``lse``. Queued for the step launch at
        the end of the transformer forward, or launched now with ``launch='layer'``.

        FLUX keeps every sample of the batch with every head (it has no CFG half). With ``reduce_heads`` the slab
        keeps each sample's mean over its kept heads, one row per sample."""
        if not q.is_cuda:
            raise RuntimeError('daam_b200 traces pipelines that live on a CUDA device only (there is no CPU '
                               'fallback)')
        if layer_idx in self._queued:                      # the layer comes round again: a new forward has started
            self.flush()
        h, w, factor = self.geometry.level(n_image, layer_idx)
        if self.flux:
            n_samples, head0, n_heads = q.shape[0], 0, heads
        else:
            _, n_samples, head0, n_heads = ops.cond_half(q.shape[0], heads)
        n_real, images = self._prompt_layout(layer_idx, n_samples)
        tokens = k.shape[2] - n_image
        if self.reduce_heads:
            slab = self.all_heat_maps.slab_for(layer_idx, factor, n_real, images, h, w, q.device, head0, images,
                                               tokens, head_mean=n_heads)
            acc = slab.acc.view(n_samples, tokens, n_image)
        else:
            slab = self.all_heat_maps.slab_for(layer_idx, factor, n_real, images * n_heads, h, w, q.device, head0,
                                               images, tokens)
            acc = slab.acc.view(n_samples, n_heads, tokens, n_image)
        desc = ops.make_joint_desc(q, k, lse, n_image, acc, heads, scale, text_first=self.flux, whole_batch=self.flux,
                                   reduce_heads=self.reduce_heads)
        self._device = q.device
        if self.launch == 'layer':
            self._accumulate_joint([desc], q.device)
            return
        self._joint_pending.append(desc)
        self._refs += [q, k, lse]                          # kept alive until the step's launch has been issued
        self._queued[layer_idx] = self._step_id

    def _accumulate_joint(self, descs, device):
        """The joint launch of ``descs``: per head, or with ``reduce_heads`` each sample's head mean."""
        (ops.accumulate_joint_heads if self.reduce_heads else ops.accumulate_joint)(descs, device)

    def _launch_now(self, own, device):
        """``launch='layer'``: the layer's kernel right away on the current stream (the producer of Q/K may be the
        immediately preceding kernel there, so no EARLY_LOADS)."""
        ops._run_on(device, None, lambda stream: _native.accumulate(own, stream, self.kernel_flags))

    def _accumulate_probs(self, layer_idx: int, factor: int, probs: torch.Tensor, bsz: int, heads: int):
        """Heat maps from materialised probabilities (save_heads / load_heads compatibility path)."""
        h, w, _ = self.geometry.level(probs.shape[1], layer_idx)
        if h is None:
            raise RuntimeError(f'layer {layer_idx}: {probs.shape[1]} query positions are not a square map')
        self._check_guidance(layer_idx, bsz)
        _, n_samples, head0, n_heads = ops.cond_half(bsz, heads)
        n_real, images = self._prompt_layout(layer_idx, n_samples)
        slab = self.all_heat_maps.slab_for(layer_idx, factor, n_real, images * n_heads, h, w, probs.device, head0,
                                           images)
        self.synchronize()
        if self.negative:                                  # rows [0, N*H) into neg, the rest into acc, in one launch
            ops.accumulate_probs(probs, slab.storage, whole_batch=True)
        else:
            ops.accumulate_probs(probs, slab.acc)

    def flush(self):
        """Issue the queued layer calls as one persistent launch (per pack of 32 layers)."""
        if self._joint_pending:
            descs, self._joint_pending = self._joint_pending, []
            self._accumulate_joint(descs, self._device)   # on the forward's own stream: the projections may go now
            self._refs = []
            self._queued.clear()
            return
        n = self._n_pending
        if n == 0:
            return
        device = self._device
        index = device.index if device.index is not None else torch.cuda.current_device()
        packed = self._packed
        packed.n = n
        flags = self.kernel_flags | _native.ACC_EARLY_LOADS
        current = torch.cuda.current_stream(index).cuda_stream
        previous = torch.cuda.current_device()
        switch = index != previous
        if switch:
            torch.cuda.set_device(index)
        try:
            capturing = torch.cuda.is_current_stream_capturing()
            if capturing:
                if self._slab_ptrs:                            # drop the step: its projections live in the graph's pool
                    self._refs, self._n_pending = [], 0
                    what, why = ('time_resolved=True', 'every step writes its heat map into another history slot') \
                        if self.time_resolved else \
                        ('step_ranges', 'which range slabs a step adds into depends on the step index')
                    raise RuntimeError(f'{what} cannot be captured into a CUDA graph: {why}, which a graph replay '
                                       f'cannot follow')
                # CUDA-graph capture of the UNet step: the launch becomes a node of the captured stream; replays bypass the
                # Python hook, so the layers of this launch stay live across per-generation resets
                step = self._step_id
                for layer_idx, st in self._layer_state.items():
                    if self._queued.get(layer_idx) == step:
                        st[4].captured = True
            if capturing or self.launch == 'step':
                # On the forward's own stream: the predecessor there is the tail of the UNet forward, never a producer of
                # the queued Q/K, so only the accumulator updates have to wait for it (EARLY_LOADS). Stream order also
                # makes it safe to drop the projections right after the launch. The second-slab modes need this launch
                # (checked at construction): time-resolved mode stores into the step slabs, then reduces them to the
                # step's global heat maps in stream order behind it; step-range mode adds into the slabs of the range
                # this forward lies in, if any.
                r = self._range_of(self._forward_idx) if self.step_ranges is not None else None
                if self.time_resolved:
                    _native.accumulate_steps(packed, self._slab_ptrs[0], current, flags)
                    self._finalize_step(device, current)
                elif r is not None:
                    _native.accumulate_range(packed, self._slab_ptrs[r], current, flags)
                    self.all_heat_maps.range_steps[r] += 1
                else:
                    _native.accumulate(packed, current, flags)
                self._forward_idx += 1
            else:
                side = self._side_stream(device)
                if self._launcher is None:
                    self._launcher = _native.SideLauncher()
                if self._parked and self._launcher.idle():     # the previous launches have run: drop their projections
                    self._parked = []
                elif len(self._parked) >= 8:                   # the host runs many steps ahead of the device: do not let
                    side.synchronize()                         # parked projections pile up (they pin allocator blocks)
                    self._parked = []
                # One foreign call: event on the current stream (Q/K were produced there) -> the side stream waits ->
                # launch -> `done` event. The side stream carries nothing but these launches and the projections are
                # complete before the previous one could have started (EARLY_LOADS holds here too).
                self._launcher.launch(packed, flags, current, side.cuda_stream)
                self._parked.append(self._refs)                # alive until a later idle() / join says the kernel has run
                self._dirty = True
        finally:
            if switch:
                torch.cuda.set_device(previous)
        self._refs = []
        self._n_pending = 0
        self._step_id += 1

    def _finalize_step(self, device, stream: int):
        """Time-resolved mode, right after the step's launch on ``stream``: ONE ``daam_finalize_maps`` launch writes,
        for every prompt, the global heat map of the step slabs this step wrote -- the same reduction, key order
        (live-slab order) and row count as :meth:`compute_global_heat_map` -- into the next slot of the prompt's
        history; with several images per prompt also every image's map (``image_idx``) into that image's history; and
        with ``negative=True`` the same again over the unconditional halves of the step slabs, into the negative
        histories."""
        queued = {idx for idx, step in self._queued.items() if step == self._step_id}
        slabs = [s for s in self.all_heat_maps.live_slabs() if s.layer_idx in queued]
        grid = self.geometry.grid
        t = self._time_steps
        halves = (False, True) if self.negative else (False,)
        if self._history_rows is None:
            self._history_rows = {negative: [self._n_rows(text) for text in self._texts(negative)]
                                  for negative in halves}
        n_prompts, images = slabs[0].n_prompts, slabs[0].images
        maps = []
        for negative in halves:
            rows, history = self._history_rows[negative], self._history[negative]
            first = n_prompts if self.negative and not negative else 0    # step slabs: [uncond x N, cond x N]
            for p in range(n_prompts):
                n_rows = rows[p] if p < len(rows) else rows[0]
                block = (first + p) * images
                for image, begin, count in [(None, block, images)] + \
                        ([(i, block + i, 1) for i in range(images)] if images > 1 else []):
                    hist = _history_slot(history, (p, image), n_rows, grid, t, device)
                    maps.append(_native.DaamMapSel(block_begin=begin, block_count=count, n_rows=n_rows,
                                                   out=hist[t].data_ptr()))
        _native.finalize_maps([_block_group(s.step, s) for s in slabs], maps, grid, False, stream)
        self._time_steps = t + 1

    def _texts(self, negative: bool = False) -> List[str]:
        """The text of every prompt of the running / last generation, or with ``negative`` its negative text."""
        if negative:
            return self.last_negative_prompts or ['']
        return self.last_prompts or [self.last_prompt]

    def _n_rows(self, text: str) -> int:
        return min(len(self.pipe.tokenizer.tokenize(text)) + 2, _native.TOKENS)   # 1 for SOS and 1 for padding

    def _restart_history(self):
        """A new generation: a new per-step history (maps handed out earlier stay valid: they are other tensors), and
        the UNet forward count of the step ranges starts again (their slabs were zeroed with the accumulators)."""
        self._history = {False: {}, True: {}}
        self._time_steps = 0
        self._history_rows = None
        self._forward_idx = 0

    def _range_of(self, forward_idx: int) -> Optional[int]:
        for i, (start, stop) in enumerate(self.step_ranges):
            if start <= forward_idx < stop:
                return i
        return None

    @property
    def step_range_counts(self) -> List[int]:
        """How many UNet forwards of the running / last generation each declared step range has received."""
        self.synchronize()
        return list(self.all_heat_maps.range_steps)

    def synchronize(self):
        """Make every accumulate issued so far visible to work enqueued on the current stream afterwards."""
        self.flush()
        if self._dirty and self._stream is not None:
            self._launcher.join(torch.cuda.current_stream(self._stream.device).cuda_stream)
            self._dirty = False
            # parked projections: their memory may only be reused by the current stream after the side stream is done
            # with them, which the wait above now guarantees for everything issued so far
            self._parked = []

    def _zero_slabs(self, slabs: List[LayerSlab]):
        if not slabs:
            return
        self.synchronize()
        for slab in slabs:
            slab.zero_()
        if self._stream is not None:   # later side-stream launches must see the zeroed slabs
            self._stream.wait_stream(torch.cuda.current_stream(slabs[0].acc.device))

    # -- finalize -------------------------------------------------------------------------------------------------------
    def compute_global_heat_map(self, prompt=None, factors=None, head_idx=None, layer_idx=None, normalize=False,
                                prompt_idx: int = 0, *, step_range: Optional[int] = None, negative: bool = False,
                                image_idx: Optional[int] = None, value_weighted: bool = False,
                                encoder: Optional[str] = None) -> GlobalHeatMap:
        """Aggregate across time (already summed in the slabs) and across layers/heads (trace.py:83-132).

        Args mirror the reference: ``factors`` restricts the spatial factors, ``head_idx`` / ``layer_idx`` restrict to one
        head / layer, ``normalize`` divides by the per-pixel sum over the real tokens. ``prompt_idx`` selects the prompt in
        ``batch_prompts`` mode. ``step_range=i`` aggregates over the steps of declared range ``i`` only
        (``trace(pipe, step_ranges=[...])``): the DAAM map a trace of only those steps would give. ``negative=True``
        (``trace(pipe, negative=True)``): the map of the unconditional half of the batch, whose text (and so row count
        and word lookup) is the prompt's negative prompt unless ``prompt`` is given.

        With several images per prompt (``num_images_per_prompt``) the map is, as in the reference, the mean over every
        image's keys, and ``head_idx`` indexes images x heads. ``image_idx=i`` keeps image ``i``'s keys only (``head_idx``
        then counts that image's heads); an un-guided batch has only the kept images (see ``ops.cond_half``).

        ``value_weighted=True`` (``trace(pipe, value_norms=True)``): every key's clamped map is scaled by its value norm
        ``||W_h v||`` for that row before the mean over keys (``daam_finalize_parts_weighted``; same keys, order, rows
        and normalisation).

        ``encoder='t5'`` (a joint-attention trace of an SD3 pipeline): the map of the T5 rows of ``prompt_3`` (or of
        the prompt), in the CLIP map's layout: row 0 is zeros (T5 has no start token), rows ``1 .. n`` the
        sentencepiece pieces and row ``n + 1`` the T5 EOS, so the word lookup (``pipe.tokenizer_3``, case kept) and
        every word-list call apply unchanged. The default (``encoder=None``) is the trace's own encoder: the CLIP rows
        with ``pipe.tokenizer``, or on a FLUX trace, whose context is T5 rows only, the T5 rows of ``prompt_2`` (or of
        the prompt) with ``pipe.tokenizer_2``, in the same layout (map row ``r >= 1`` is context row ``r - 1``).
        """
        encoder = self._encoder(encoder)
        prompt, grid, rows, groups, slabs = self._read_groups(prompt, factors, prompt_idx, step_range, layer_idx,
                                                              head_idx, negative, image_idx, encoder)
        tokenizer = self._map_tokenizer(encoder, rows)
        if value_weighted:
            weights = self._weight_ptrs(slabs, prompt_idx, negative, image_idx)
            maps = self._finalize_parts(groups, [(0, len(groups))], grid, rows, normalize, slabs, weights)[0]
            return GlobalHeatMap(tokenizer, prompt, maps)
        device = slabs[0].acc.device
        n_fin = _finalized_rows(rows)
        maps = torch.empty((n_fin,) + grid, dtype=torch.float32, device=device)
        with torch.cuda.device(device):
            _native.finalize(groups, grid, n_fin, normalize and n_fin == len(rows), maps.data_ptr(),
                             torch.cuda.current_stream(device).cuda_stream)
        return GlobalHeatMap(tokenizer, prompt, _t5_start_row(_compact(maps, rows, normalize), encoder))

    def compute_image_heat_maps(self, prompt_idx: int = 0, factors=None, layer_idx=None, head_idx=None,
                                normalize: bool = False, *, step_range: Optional[int] = None,
                                negative: bool = False, prompt: Optional[str] = None) -> ImageHeatMaps:
        """Every image's map of prompt ``prompt_idx`` in one launch (``daam_finalize_maps``): ``heat_maps[i]`` is
        ``compute_global_heat_map(image_idx=i, ...)`` with the same arguments, bit for bit (``head_idx`` counts one
        image's heads). ``prompt``: the text, when it is not the generation's (e.g. one driven by ``prompt_embeds``).
        Returns an :class:`ImageHeatMaps` ``[images, n_rows, xh, xw]``. The rows are those of the trace's own encoder
        (a FLUX trace: T5)."""
        encoder = self._encoder(None)
        prompt, grid, rows, _, slabs = self._read_groups(prompt, factors, prompt_idx, step_range, layer_idx, head_idx,
                                                         negative, 0, encoder)
        images, n_prompts = slabs[0].images, slabs[0].n_prompts
        if not 0 <= prompt_idx < n_prompts:
            raise IndexError(f'prompt_idx {prompt_idx} is out of range for {n_prompts} prompt(s)')
        groups = [_block_group(s.source(step_range, negative), s, -1 if head_idx is None else head_idx) for s in slabs]
        device = slabs[0].acc.device
        n_fin = _finalized_rows(rows)
        out = torch.empty((images, n_fin) + grid, dtype=torch.float32, device=device)
        maps = [_native.DaamMapSel(block_begin=prompt_idx * images + i, block_count=1, n_rows=n_fin,
                                   out=out[i].data_ptr()) for i in range(images)]
        with torch.cuda.device(device):
            _native.finalize_maps(groups, maps, grid, normalize and n_fin == len(rows),
                                  torch.cuda.current_stream(device).cuda_stream)
        return ImageHeatMaps(self._map_tokenizer(encoder, rows), prompt,
                             _t5_start_row(_compact(out, rows, normalize), encoder))

    def compute_time_heat_maps(self, prompt_idx: int = 0, normalize: bool = False, *,
                               negative: bool = False, image_idx: Optional[int] = None) -> TimeHeatMaps:
        """One global heat map per traced denoising step (UNet forward) of the running / last generation; needs
        ``trace(pipe, time_resolved=True)``. ``heat_maps[t]`` is what :meth:`compute_global_heat_map` would return had
        only step ``t`` been traced, with every key and layer; ``normalize`` applies the reference's normalisation to
        each step. Summing the steps does not give the all-steps map: there the clamp comes after the time sum.
        ``negative=True``: the same for the unconditional half, against the negative text. ``image_idx=i``: image
        ``i``'s map after every step (``compute_global_heat_map(image_idx=i)`` of a trace of that step only).

        Costs: a second fp32 slab per traced layer (as large as its accumulator) and ``steps x n_rows x xh x xw`` fp32
        of history per prompt (``heat_maps`` is ``[steps, n_rows, xh, xw]``, the grid of :attr:`geometry`), and as much
        again per image when a generation has several images per prompt."""
        if not self.time_resolved:
            raise RuntimeError('per-step heat maps need trace(pipe, time_resolved=True)')
        if negative:
            self.all_heat_maps.check_negative()
        self.synchronize()
        history = self._history[negative]
        if self._time_steps == 0 or (prompt_idx, None) not in history:
            raise RuntimeError('No heat maps found. Did you forget to call `with trace(...)` during generation?')
        if image_idx is not None:
            _check_image_idx(image_idx, max(1, sum(1 for p, i in history if p == prompt_idx and i is not None)))
        texts = self._texts(negative)
        prompt = texts[prompt_idx] if prompt_idx < len(texts) else texts[0]
        # one image per prompt: its map is the prompt's map (same keys, same order)
        key = (prompt_idx, image_idx) if (prompt_idx, image_idx) in history else (prompt_idx, None)
        maps = history[key][:self._time_steps]
        if normalize:
            maps = maps.clone()
            with torch.cuda.device(maps.device):
                _native.normalize_maps(maps.data_ptr(), maps.shape[0], maps.shape[1], maps.shape[-2:],
                                       torch.cuda.current_stream(maps.device).cuda_stream)
        return TimeHeatMaps(self.pipe.tokenizer, prompt, maps)


    def compute_per_head_heat_maps(self, prompt=None, factors=None, normalize=False, prompt_idx: int = 0, *,
                                   step_range: Optional[int] = None, negative: bool = False,
                                   image_idx: Optional[int] = None, value_weighted: bool = False,
                                   encoder: Optional[str] = None):
        """Every ``compute_global_heat_map(layer_idx=l, head_idx=h)`` of the reference's ``--all-heads`` sweep
        (daam/run/generate.py:239-255) in one launch. Returns ``(keys, maps)``: ``keys[i] = (factor, layer, head)`` and
        ``maps[i]`` the ``[n_tokens + 2, xh, xw]`` heat map the reference computes for that single key. ``step_range=i``
        and ``negative=True`` select the slabs as in :meth:`compute_global_heat_map`; ``image_idx=i`` keeps image
        ``i``'s keys, whose ``head`` then counts that image's heads. ``value_weighted=True``: ``maps[i]`` is the
        value-weighted global map of key ``i`` alone, bit for bit. ``encoder``: as in :meth:`compute_global_heat_map`."""
        return self._per_head(prompt, factors, normalize, prompt_idx, step_range, negative, image_idx,
                              value_weighted, encoder)[1:3]

    def _per_head(self, prompt, factors, normalize, prompt_idx, step_range, negative, image_idx, value_weighted=False,
                  encoder: Optional[str] = None):
        """``(prompt, keys, maps)`` of :meth:`compute_per_head_heat_maps`. Weighted: the per-key maps unnormalised,
        times each key's norm per row on the device, then normalised -- a single key's weighted global map. Also
        returns the map's tokenizer."""
        self.all_heat_maps.check_heads('per-head heat maps')
        encoder = self._encoder(encoder)
        prompt, grid, rows, groups, slabs = self._read_groups(prompt, factors, prompt_idx, step_range,
                                                              negative=negative, image_idx=image_idx, encoder=encoder)
        keys = [(slab.factor, slab.layer_idx, head) for slab, g in zip(slabs, groups) for head in range(g.heads)]
        device = slabs[0].acc.device
        n_fin = _finalized_rows(rows)
        norms = self._key_norms(slabs, prompt_idx, negative, image_idx)[:, :n_fin] if value_weighted else None
        maps = torch.empty((len(keys), n_fin) + grid, dtype=torch.float32, device=device)
        norm_here = normalize and n_fin == len(rows)
        with torch.cuda.device(device):
            stream = torch.cuda.current_stream(device).cuda_stream
            _native.finalize_per_key(groups, grid, n_fin, norm_here and norms is None, maps.data_ptr(), stream)
            if norms is not None:
                maps.mul_(norms[:, :, None, None])
                if norm_here:
                    _native.normalize_maps(maps.data_ptr(), len(keys), n_fin, grid, stream)
        return prompt, keys, _t5_start_row(_compact(maps, rows, normalize), encoder), self._map_tokenizer(encoder, rows)

    def compute_value_norms(self, prompt=None, prompt_idx: int = 0, *, negative: bool = False,
                            image_idx: Optional[int] = None, factors=None):
        """Which heads carry each word: ``(keys, norms)`` with ``keys`` those of :meth:`compute_per_head_heat_maps`
        and ``norms[i]`` ``[n_tokens + 2]`` (device fp32) key ``i``'s value norm ``||W_h v||`` of every row of the map
        (the compact rows of a long context). Needs ``trace(pipe, value_norms=True)``."""
        prompt, _, rows, groups, slabs = self._read_groups(prompt, factors, prompt_idx, None, negative=negative,
                                                           image_idx=image_idx)
        keys = [(slab.factor, slab.layer_idx, head) for slab, g in zip(slabs, groups) for head in range(g.heads)]
        norms = self._key_norms(slabs, prompt_idx, negative, image_idx)
        return keys, norms.index_select(1, torch.tensor(rows, dtype=torch.long).to(norms.device))

    def _check_weighted(self, slabs):
        """Raises unless every slab of a read holds value norms that stayed valid for the whole generation."""
        if not self.value_norms or any(s.norms is None for s in slabs):
            raise RuntimeError('value-weighted heat maps need a trace declared with trace(pipe, value_norms=True)')
        changed = torch.stack([s.norms_changed for s in slabs]).cpu()
        if bool(changed.any()):
            layer = slabs[int(changed.to(torch.uint8).argmax())].layer_idx
            raise ValueError(f'layer {layer}: the cross-attention context changed during the generation, so its value '
                             f'norms are not one set per key: a value-weighted read is undefined (plain reads work)')

    def _weight_ptrs(self, slabs, prompt_idx: int, negative: bool, image_idx: Optional[int]) -> List[int]:
        """The weights of the key groups ``_read_groups`` made from ``slabs``: each group's acc offset with the pixel
        axis dropped, in the slab's norms."""
        self._check_weighted(slabs)
        out = []
        for s in slabs:
            n = s.norm_source(negative)
            out.append((n[prompt_idx] if image_idx is None else n[prompt_idx, image_idx * s.heads_per_image]).data_ptr())
        return out

    def _key_norms(self, slabs, prompt_idx: int, negative: bool, image_idx: Optional[int]) -> torch.Tensor:
        """``[keys, tokens]``: the norms of every key of a per-head read over ``slabs``, in its key order."""
        self._check_weighted(slabs)
        parts = []
        for s in slabs:
            n = s.norm_source(negative)[prompt_idx]
            parts.append(n if image_idx is None else n[image_idx * s.heads_per_image:(image_idx + 1) * s.heads_per_image])
        return torch.cat(parts)

    def compute_head_heat_maps(self, prompt=None, factors=None, normalize=False, prompt_idx: int = 0, *,
                               step_range: Optional[int] = None, negative: bool = False,
                               image_idx: Optional[int] = None, value_weighted: bool = False,
                               encoder: Optional[str] = None) -> HeadHeatMaps:
        """:meth:`compute_per_head_heat_maps` as a stack the word-list calls work on: a :class:`HeadHeatMaps` whose
        ``keys[i] = (factor, layer, head)`` labels ``heat_maps[i]``. The stack takes ``keys x rows x xh x xw x 4`` bytes
        (SD-2.1, 175 keys, 12 rows, 64 x 64: 34 MB; the 1100 keys of SDXL's 60 layers: 216 MB); ``factors`` and ``image_idx`` narrow
        it."""
        prompt, keys, maps, tokenizer = self._per_head(prompt, factors, normalize, prompt_idx, step_range, negative,
                                                       image_idx, value_weighted, encoder)
        return HeadHeatMaps(tokenizer, prompt, maps, keys)

    def compute_layer_heat_maps(self, prompt=None, factors=None, head_idx=None, normalize=False, prompt_idx: int = 0, *,
                                step_range: Optional[int] = None, negative: bool = False,
                                image_idx: Optional[int] = None, value_weighted: bool = False,
                                encoder: Optional[str] = None) -> LayerHeatMaps:
        """Every traced layer's map in one launch (``daam_finalize_parts``): ``heat_maps[i]`` is
        ``compute_global_heat_map(layer_idx=layers[i], ...)`` with the same arguments, bit for bit. One map per layer
        that passes the filters (``head_idx``: the layers that have that head), in the order the layers were traced.
        Returns a :class:`LayerHeatMaps` ``[layers, n_rows, xh, xw]``. ``encoder``: as in
        :meth:`compute_global_heat_map`."""
        encoder = self._encoder(encoder)
        prompt, grid, rows, groups, slabs = self._read_groups(prompt, factors, prompt_idx, step_range, None, head_idx,
                                                              negative, image_idx, encoder)
        weights = self._weight_ptrs(slabs, prompt_idx, negative, image_idx) if value_weighted else None
        maps = self._finalize_parts(groups, [(i, 1) for i in range(len(groups))], grid, rows, normalize, slabs, weights)
        names = self.layer_names
        return LayerHeatMaps(self._map_tokenizer(encoder, rows), prompt, _t5_start_row(maps, encoder), [s.layer_idx for s in slabs],
                             [names[s.layer_idx] if s.layer_idx < len(names) else None for s in slabs],
                             [s.factor for s in slabs])

    def compute_factor_heat_maps(self, prompt=None, factors=None, head_idx=None, layer_idx=None, normalize=False,
                                 prompt_idx: int = 0, *, step_range: Optional[int] = None, negative: bool = False,
                                 image_idx: Optional[int] = None, value_weighted: bool = False) -> FactorHeatMaps:
        """Every traced resolution's map in one launch (``daam_finalize_parts``): ``heat_maps[j]`` is
        ``compute_global_heat_map(factors={stack.factors[j]}, ...)`` with the same arguments, bit for bit; ``factors``
        keeps some of them. Returns a :class:`FactorHeatMaps` ``[factors, n_rows, xh, xw]``, factors ascending. The
        rows are those of the trace's own encoder (a FLUX trace: T5)."""
        encoder = self._encoder(None)
        prompt, grid, rows, groups, slabs = self._read_groups(prompt, factors, prompt_idx, step_range, layer_idx,
                                                              head_idx, negative, image_idx, encoder)
        order, found, parts = _factor_parts([s.factor for s in slabs])
        weights = self._weight_ptrs(slabs, prompt_idx, negative, image_idx) if value_weighted else None
        maps = self._finalize_parts([groups[i] for i in order], parts, grid, rows, normalize, slabs,
                                    None if weights is None else [weights[i] for i in order])
        return FactorHeatMaps(self._map_tokenizer(encoder, rows), prompt, _t5_start_row(maps, encoder), found)

    def _finalize_parts(self, groups, parts, grid, rows, normalize, slabs, weights=None) -> torch.Tensor:
        """One ``daam_finalize_parts`` over ``groups``: map ``m`` reduces groups ``[begin, begin + count)`` of
        ``parts[m] = (begin, count)`` as a read of those groups alone does. Returns ``[len(parts), len(rows), xh, xw]``.
        ``weights``: one norms pointer per group, ``daam_finalize_parts_weighted``."""
        device = slabs[0].acc.device
        n_fin = _finalized_rows(rows)
        out = torch.empty((len(parts), n_fin) + grid, dtype=torch.float32, device=device)
        sel = [_native.DaamMapPart(group_begin=begin, group_count=count, n_rows=n_fin, out=out[m].data_ptr())
               for m, (begin, count) in enumerate(parts)]
        with torch.cuda.device(device):
            _native.finalize_parts(groups, sel, grid, normalize and n_fin == len(rows),
                                   torch.cuda.current_stream(device).cuda_stream, weights)
        return _compact(out, rows, normalize)

    def _read_groups(self, prompt, factors, prompt_idx: int, step_range: Optional[int], layer_idx=None, head_idx=None,
                     negative: bool = False, image_idx: Optional[int] = None, encoder: str = 'clip'):
        """What the heat-map reads share: the prompt (default: the generation's, or with ``negative`` its negative
        text), the map grid ``(xh, xw)``, the context rows the map reads (``utils.context_rows``: ``[0, n_tokens + 2)``
        for a 77-token context), and the key groups of prompt ``prompt_idx`` over the live slabs (with ``step_range``:
        over that range's slabs; with ``negative``: their unconditional halves) that pass the filters, with the slabs
        behind them; with ``image_idx`` the groups hold image ``image_idx``'s heads only, and ``head_idx`` counts those.
        Raises when no slab passes, ``IndexError`` for a bad ``image_idx`` and ``ValueError`` when the generation was
        driven by embeddings and no ``prompt`` text is given.

        A joint-attention trace reads the CLIP rows ``[0, n_tokens + 2)`` of its context, or with ``encoder='t5'`` the
        T5 rows: the groups then start at context row 76, so that map row ``r`` is context row ``76 + r`` (row 0, the
        last CLIP row, is zeroed by the read), and the text is ``prompt_3`` when the generation had one. A FLUX trace
        reads T5 rows only and its rows are ``[-1, 0, .., n]``: the finalize reads context rows ``[0, n + 1)`` from
        row 0 of each key, and ``_compact`` puts the zero row -1 stands for ahead of them, so that map row ``r >= 1``
        is context row ``r - 1`` (T5 has no start token); the text is ``prompt_2`` when the generation had one."""
        if encoder not in ('clip', 't5'):
            raise ValueError(f"encoder must be 'clip' or 't5', got {encoder!r}")
        if head_idx is not None and self.reduce_heads:
            raise ValueError('head_idx selects one head, but a trace(pipe, reduce_heads=True) keeps the mean over '
                             'heads only')
        if encoder == 't5':
            if not self.joint:
                raise ValueError("encoder='t5' reads the T5 rows of a joint-attention (SD3) trace; this trace has "
                                 "CLIP contexts only")
            name = 'tokenizer_2' if self.flux else 'tokenizer_3'
            if getattr(self.pipe, name, None) is None:
                raise ValueError(f"encoder='t5' needs the pipeline's T5 tokenizer (pipe.{name})")
            texts = self.last_prompts_2 if self.flux else self.last_prompts_3
            if prompt is None and prompt_idx < len(texts):
                prompt = texts[prompt_idx]
        if negative:
            self.all_heat_maps.check_negative()
        if prompt is None:
            if negative:
                prompt = self.last_negative_prompts[prompt_idx] if self.last_negative_prompts else ''
            else:
                prompt = self.last_prompts[prompt_idx] if self.last_prompts else self.last_prompt
            if prompt is None:
                raise ValueError(f'the generation was driven by {"negative_" if negative else ""}prompt_embeds, so '
                                 f'its text is unknown: pass the text it encodes as prompt=...')
        factors = {0, 1, 2, 4, 8, 16, 32, 64} if factors is None else set(factors)
        read = self.all_heat_maps.read_slabs(step_range, negative)
        if image_idx is not None and read:
            images = {s.images for s in read}
            if len(images) > 1:
                raise RuntimeError(f'image_idx needs every traced layer to hold the same images per prompt, got '
                                   f'{sorted(images)}')
            _check_image_idx(image_idx, images.pop())
        groups, slabs = [], []
        for slab in read:
            if slab.factor not in factors or (layer_idx is not None and layer_idx != slab.layer_idx):
                continue
            heads = slab.heads if image_idx is None else slab.heads_per_image
            if head_idx is not None and not 0 <= head_idx < heads:
                continue
            src = slab.source(step_range, negative)
            if image_idx is None:
                groups.append(_key_group(src[prompt_idx], slab, -1 if head_idx is None else head_idx))
            else:                                          # image i: heads [i * H, (i + 1) * H) of the prompt
                groups.append(_native.DaamKeyGroup(acc=src[prompt_idx, image_idx * heads].data_ptr(), heads=heads,
                                                   h=slab.h, w=slab.w, tokens=src.shape[2],
                                                   head_sel=-1 if head_idx is None else head_idx, n_blocks=1))
            slabs.append(slab)
        if not groups:
            if head_idx is not None or layer_idx is not None:
                raise RuntimeError('No heat maps found for the given parameters.')
            raise RuntimeError('No heat maps found. Did you forget to call `with trace(...)` during generation?')
        tokens = {s.tokens for s in slabs}
        if len(tokens) > 1:
            raise RuntimeError(f'the traced layers hold contexts of {sorted(tokens)} tokens: one read reduces one '
                               f'context length')
        tokens = tokens.pop()
        if not self.joint:
            return prompt, self.geometry.grid, context_rows(len(self.pipe.tokenizer.tokenize(prompt)), tokens), \
                groups, slabs
        if encoder == 'clip':
            return prompt, self.geometry.grid, context_rows(len(self.pipe.tokenizer.tokenize(prompt))), groups, slabs
        if self.flux:                                      # T5 rows only: pieces at context rows [0, n), EOS at n
            n = t5_rows(len(self.pipe.tokenizer_2.tokenize(prompt)), tokens, clip_tokens=0)
            return prompt, self.geometry.grid, [-1] + list(range(n + 1)), groups, slabs
        if tokens < _T5_FIRST_ROW + 2:
            raise RuntimeError(f'a context of {tokens} rows has no T5 rows after the {_T5_FIRST_ROW + 1} CLIP rows')
        n = t5_rows(len(self.pipe.tokenizer_3.tokenize(prompt)), tokens)
        for g, slab in zip(groups, slabs):
            g.acc += _T5_FIRST_ROW * slab.h * slab.w * 4
        return prompt, self.geometry.grid, list(range(n + 2)), groups, slabs

    def _encoder(self, encoder: Optional[str]) -> str:
        """A read's ``encoder``: ``None`` is the trace's own, ``'t5'`` on a FLUX trace (whose context is T5 rows only)
        and ``'clip'`` otherwise."""
        if encoder is None:
            return 't5' if self.flux else 'clip'
        if self.flux and encoder == 'clip':
            raise ValueError("encoder='clip': the context of a FLUX transformer holds T5 rows only; read them with "
                             "encoder='t5' (the default)")
        return encoder

    def _map_tokenizer(self, encoder: str, rows: List[int]):
        """The tokenizer of a read's map: the pipeline's CLIP tokenizer, or for a T5 read the T5 tokenizer
        (``pipe.tokenizer_3``; FLUX: ``pipe.tokenizer_2``) cut to the map's ``len(rows) - 2`` pieces."""
        if encoder != 't5':
            return self.pipe.tokenizer
        return T5Pieces(self.pipe.tokenizer_2 if self.flux else self.pipe.tokenizer_3, len(rows) - 2)


# trace() options a joint-attention (SD3) trace refuses, besides launch='overlap'
JOINT_REFUSED = ('time_resolved', 'step_ranges', 'negative', 'long_prompts', 'value_norms', 'save_heads', 'load_heads',
                 'low_memory', 'locate_middle_block')
# the context row a T5 read's group starts at: the last of the 77 CLIP rows, so that map row r + 1 is T5 row r
_T5_FIRST_ROW = 76


def _t5_start_row(maps: torch.Tensor, encoder: str) -> torch.Tensor:
    """A T5 read's maps ``[..., rows, xh, xw]`` with row 0 (the last CLIP row the group starts at) set to zeros: T5
    has no start token."""
    if encoder == 't5':
        maps[..., 0, :, :] = 0
    return maps


def _check_value_norms(layer_idx: int, attn):
    """Value-norm mode, at a traced layer call: the norms read ``attn.to_out[0].weight``, so that module must apply
    exactly that weight (a plain ``nn.Linear``: no unmerged LoRA, no hooks), and the call must run eagerly, since a
    CUDA-graph replay bypasses the hook that computes them."""
    proj = attn.to_out[0]
    plain = isinstance(proj, torch.nn.Linear) and not proj._forward_hooks and not proj._forward_pre_hooks and \
        (type(proj).forward is torch.nn.Linear.forward or
         (hasattr(proj, 'lora_layer') and getattr(proj, 'lora_layer') is None))
    if not plain:
        raise RuntimeError(f'layer {layer_idx}: value_norms=True needs the output projection to be a plain nn.Linear '
                           f'(its .weight is what the layer applies), got {type(proj).__name__}; merge any LoRA first')
    if torch.cuda.is_available() and torch.cuda.is_current_stream_capturing():
        raise RuntimeError('value_norms=True cannot be captured into a CUDA graph: the norms are computed by the '
                           'layer hook, which a graph replay bypasses')


def _factor_parts(factors: List[int]) -> Tuple[List[int], List[int], List[Tuple[int, int]]]:
    """The groups of a read, whose factors are ``factors``, partitioned by factor: ``(order, found, parts)`` with
    ``order`` the stable sort of the group indices by factor (each factor's groups contiguous, in the order a read of
    that factor alone passes them), ``found`` the distinct factors ascending and ``parts[j] = (begin, count)`` the run
    of ``found[j]`` in ``order``."""
    order = sorted(range(len(factors)), key=lambda i: factors[i])
    found, parts = [], []
    for pos, i in enumerate(order):
        if not found or found[-1] != factors[i]:
            found.append(factors[i])
            parts.append((pos, 0))
        parts[-1] = (parts[-1][0], parts[-1][1] + 1)
    return order, found, parts


def _finalized_rows(rows: List[int]) -> int:
    """The leading context rows a read finalizes: through its EOS row, ``rows[-1]``. For a 77-token context that is
    ``len(rows)``, the reference's truncation, and the finalize kernels return the map itself."""
    return rows[-1] + 1


def _compact(maps: torch.Tensor, rows: List[int], normalize: bool) -> torch.Tensor:
    """The compact map of a long context from the finalized prefix ``maps`` ``[..., rows[-1] + 1, xh, xw]``: its
    ``rows`` gathered on the device in order (SOS, every prompt token, EOS), then with ``normalize`` divided by the sum
    of compact rows ``1 .. n`` plus 1e-6 (``daam_normalize_maps``: the reference's ``rows[1:-1]`` rule on the compact
    map). When the rows are the prefix itself (every 77-token read, and a long context whose prompt fits its first
    chunk) the finalize call has normalised already and ``maps`` is returned as it is.

    Row -1 (only as ``rows[0]``) stands for a row of zeros: a FLUX T5 map, whose rows are ``[-1, 0, .., n]``, puts it
    ahead of the ``n + 1`` finalized context rows (T5 has no start token)."""
    if maps.shape[-3] == len(rows):
        return maps
    if rows[0] < 0:
        maps = F.pad(maps, (0, 0, 0, 0, 1, 0))
        rows = [r + 1 for r in rows]
    if maps.shape[-3] == len(rows):                        # (the rows are the padded prefix: nothing to gather)
        out = maps
    else:
        out = maps.index_select(maps.dim() - 3, torch.tensor(rows, dtype=torch.long).to(maps.device))
    if normalize:
        grid = tuple(out.shape[-2:])
        with torch.cuda.device(out.device):
            _native.normalize_maps(out.data_ptr(), out.numel() // (len(rows) * grid[0] * grid[1]), len(rows), grid,
                                   torch.cuda.current_stream(out.device).cuda_stream)
    return out


def _key_group(acc: torch.Tensor, slab: LayerSlab, head_sel: int = -1) -> _native.DaamKeyGroup:
    """The finalize input of one prompt's ``[heads, 77, hw]`` slab of ``slab``'s layer (its accumulator, step slab or a
    range slab); ``head_sel``: one head, or -1 for all."""
    return _native.DaamKeyGroup(acc=acc.data_ptr(), heads=slab.heads, h=slab.h, w=slab.w, tokens=acc.shape[1],
                                head_sel=head_sel, n_blocks=0)


def _block_group(src: torch.Tensor, slab: LayerSlab, head_sel: int = -1) -> _native.DaamKeyGroup:
    """The ``daam_finalize_maps`` input of a whole ``[prompts, images * heads, 77, hw]`` slab ``src`` of ``slab``'s layer
    (accumulator, step, range or negative slab): one block per (prompt, image), block ``p * images + i``; ``head_sel``
    one head within each image, or -1 for all."""
    return _native.DaamKeyGroup(acc=src.data_ptr(), heads=slab.heads_per_image, h=slab.h, w=slab.w, tokens=src.shape[2],
                                head_sel=head_sel, n_blocks=src.shape[0] * slab.images)


def _check_image_idx(image_idx, images: int):
    if not isinstance(image_idx, int) or isinstance(image_idx, bool) or not 0 <= image_idx < images:
        raise IndexError(f'image_idx {image_idx!r} is out of range for {images} image(s) per prompt')


def _history_slot(history: dict, key, n_rows: int, grid, t: int, device) -> torch.Tensor:
    """The time-resolved history ``history[key]`` ``[capacity, n_rows, xh, xw]`` with room for step ``t``: created
    with 16 slots, grown by doubling (in stream order between two steps)."""
    hist = history.get(key)
    if hist is None:
        hist = history[key] = torch.empty((16, n_rows) + tuple(grid), dtype=torch.float32, device=device)
    if t == hist.shape[0]:
        grown = torch.empty((2 * t,) + tuple(hist.shape[1:]), dtype=torch.float32, device=device)
        grown[:t].copy_(hist)
        history[key] = hist = grown
    return hist


def _normalize_step_ranges(step_ranges) -> List[Tuple[int, int]]:
    """``trace(step_ranges=...)``: a non-empty list of half-open ``(start, stop)`` tuples or step-1 ``range`` objects
    over UNet-forward indices, none empty or negative, no two overlapping. Returns ``[(start, stop), ...]`` in the
    given order (the order ``step_range=i`` indexes)."""
    if isinstance(step_ranges, (range, tuple)) or not hasattr(step_ranges, '__iter__'):
        raise ValueError(f'step_ranges is a list of (start, stop) tuples or ranges, got {step_ranges!r}')
    out = []
    for r in step_ranges:
        if isinstance(r, range):
            if r.step != 1:
                raise ValueError(f'step range {r!r} must have step 1')
            start, stop = r.start, r.stop
        elif isinstance(r, tuple) and len(r) == 2 and all(isinstance(v, int) and not isinstance(v, bool) for v in r):
            start, stop = r
        else:
            raise ValueError(f'a step range is a (start, stop) tuple of ints or a range, got {r!r}')
        if start < 0 or stop <= start:
            raise ValueError(f'step range [{start}, {stop}) must have 0 <= start < stop')
        out.append((start, stop))
    if not out:
        raise ValueError('step_ranges must declare at least one range')
    spans = sorted(out)
    for (a0, a1), (b0, b1) in zip(spans, spans[1:]):
        if b0 < a1:
            raise ValueError(f'step ranges [{a0}, {a1}) and [{b0}, {b1}) overlap')
    return out


class ImageProcessorHooker(ObjectHooker):
    """Remembers the first post-processed image of an SDXL pipeline (trace.py:135-147), and all of them in
    ``last_images``."""

    def __init__(self, processor, parent_trace: 'trace'):
        super().__init__(processor)
        self.parent_trace = parent_trace

    def _hooked_postprocess(hk_self, _, *args, **kwargs):
        images = hk_self.monkey_super('postprocess', *args, **kwargs)
        hk_self.parent_trace.last_image = images[0]
        hk_self.parent_trace.last_images = list(images)
        return images

    def _hook_impl(self):
        self.monkey_patch('postprocess', self._hooked_postprocess)


class PipelineHooker(ObjectHooker):
    """Per-generation reset + prompt capture at ``check_inputs``; image capture at the safety checker (trace.py:150-186):
    ``last_image`` is the last image, as in the reference, and ``last_images`` all of them."""

    def __init__(self, pipeline, parent_trace: 'trace'):
        super().__init__(pipeline)
        self.heat_maps = parent_trace.all_heat_maps
        self.parent_trace = parent_trace

    def _hooked_run_safety_checker(hk_self, self, image, *args, **kwargs):
        image, has_nsfw = hk_self.monkey_super('run_safety_checker', image, *args, **kwargs)
        processor = getattr(self, 'image_processor', None)
        if processor:
            images = processor.postprocess(image, output_type='pil') if torch.is_tensor(image) \
                else processor.numpy_to_pil(image)
        else:
            images = self.numpy_to_pil(image)
        hk_self.parent_trace.last_image = images[len(images) - 1]
        hk_self.parent_trace.last_images = list(images)      # prompt-major, as the pipeline returns them
        return image, has_nsfw

    def _hooked_check_inputs(hk_self, _, prompt: Union[str, List[str], None], *args, **kwargs):
        tr = hk_self.parent_trace
        if tr.flux:
            hk_self._see_flux_inputs(prompt, args, kwargs)
        if prompt is None:
            # a generation driven by prompt_embeds (e.g. chunked long-prompt embeddings): the prompt count comes from
            # them, and no text is recorded (a read then needs prompt=...)
            prompts = [None] * hk_self._embeds_count(prompt, args, kwargs)
            if len(prompts) > 1 and not tr.batch_prompts:
                raise ValueError('Only single prompt generation is supported for heat map computation.')
            if tr.time_resolved:
                raise ValueError('time_resolved=True needs the prompt text (the per-step heat map has one row per '
                                 'token): a generation driven by prompt_embeds alone cannot be traced with it')
        elif isinstance(prompt, str):
            prompts = [prompt]
        else:
            prompts = list(prompt)
            if len(prompts) > 1 and not tr.batch_prompts:
                raise ValueError('Only single prompt generation is supported for heat map computation.')
        negatives = hk_self._negative_prompts(prompt, args, kwargs, len(prompts)) if tr.negative else []
        hk_self.heat_maps.clear()
        tr._restart_history()
        tr._norms_seen.clear()                       # the value norms of the new generation are computed afresh
        if len(prompts) != len(tr.last_prompts):    # slabs are laid out [prompts][images * heads]: re-derive them
            tr._layer_state.clear()
        tr.last_prompt = prompts[0]
        tr.last_prompts = prompts
        tr.last_negative_prompts = negatives
        if tr.joint and not tr.flux:                 # SD3: the T5 encoder reads prompt_3 when one is given
            bound = inspect.signature(hk_self._replaced['check_inputs']).bind(prompt, *args, **kwargs)
            third = bound.arguments.get('prompt_3', kwargs.get('prompt_3'))
            tr.last_prompts_3 = [third] * len(prompts) if third is None or isinstance(third, str) else list(third)
        return hk_self.monkey_super('check_inputs', prompt, *args, **kwargs)

    def _see_flux_inputs(hk_self, prompt, args, kwargs):
        """FLUX, at ``check_inputs(prompt, prompt_2, height, width, negative_prompt=None, negative_prompt_2=None,
        prompt_embeds=None, negative_prompt_embeds=None, ...)``: refuses negative prompts (with them, true CFG runs a
        second transformer forward per step that the trace cannot tell from the conditional one), records the T5 text
        of every prompt (``prompt_2``, else the prompt) and sets the grid from ``height`` / ``width``."""
        tr = hk_self.parent_trace
        bound = inspect.signature(hk_self._replaced['check_inputs']).bind(prompt, *args, **kwargs).arguments
        for name in ('negative_prompt', 'negative_prompt_2', 'negative_prompt_embeds'):
            if bound.get(name, kwargs.get(name)) is not None:
                raise ValueError(f'{name} is not supported when tracing the joint attention of a FLUX transformer: '
                                 f'true CFG runs a second transformer forward per step, which the trace cannot tell '
                                 f'apart from the conditional one')
        second = bound.get('prompt_2', kwargs.get('prompt_2'))
        n = hk_self._embeds_count(prompt, args, kwargs) if prompt is None else \
            (1 if isinstance(prompt, str) else len(prompt))
        texts = [prompt] * n if prompt is None or isinstance(prompt, str) else list(prompt)
        if second is None:
            tr.last_prompts_2 = texts
        else:
            tr.last_prompts_2 = [second] * n if isinstance(second, str) else list(second)
        height, width = bound.get('height', kwargs.get('height')), bound.get('width', kwargs.get('width'))
        tr.geometry = FluxGeometry(tr.geometry.vae_scale_factor,
                                   None if height is None or width is None else (height, width))

    def _embeds_count(hk_self, prompt, args, kwargs) -> int:
        """The number of prompts of a ``check_inputs`` call without text: the batch of its ``prompt_embeds`` argument
        ``[N, T, C]``, bound by name like ``negative_prompt`` (1 when absent)."""
        bound = inspect.signature(hk_self._replaced['check_inputs']).bind(prompt, *args, **kwargs)
        embeds = bound.arguments.get('prompt_embeds', kwargs.get('prompt_embeds'))
        return int(embeds.shape[0]) if embeds is not None else 1

    def _negative_prompts(hk_self, prompt, args, kwargs, n: int) -> List[str]:
        """The negative text of each of the ``n`` prompts, from the ``negative_prompt`` argument of the
        ``check_inputs`` call: bound by name to the wrapped method's signature, because pipelines pass it positionally
        at different places (diffusers' SD: ``(prompt, height, width, callback_steps, negative_prompt, ...)``; SDXL has
        ``prompt_2`` before it). None or absent is the empty prompt, which is what the pipeline encodes then."""
        bound = inspect.signature(hk_self._replaced['check_inputs']).bind(prompt, *args, **kwargs)
        negative = bound.arguments.get('negative_prompt', kwargs.get('negative_prompt'))
        if negative is None:
            return [''] * n
        if isinstance(negative, str):
            return [negative] * n
        negatives = list(negative)
        if len(negatives) != n:
            raise ValueError(f'negative_prompt has {len(negatives)} entries for {n} prompts')
        return negatives

    def _hook_impl(self):
        self.monkey_patch('run_safety_checker', self._hooked_run_safety_checker, strict=False)  # absent in SDXL
        self.monkey_patch('check_inputs', self._hooked_check_inputs)


class UNetCrossAttentionHooker(ObjectHooker):
    """The attention processor installed on one ``attn2`` module (trace.py:189-315)."""

    def __init__(self, module, parent_trace: 'trace', context_size: int = 77, layer_idx: int = 0,
                 latent_hw: int = 9216, load_heads: bool = False, save_heads: bool = False,
                 data_dir: Union[str, Path] = None):
        super().__init__(module)
        self.heat_maps = parent_trace.all_heat_maps
        self.context_size = context_size
        self.layer_idx = layer_idx
        self.latent_hw = latent_hw             # kept for the reference's signature; the factor comes from trace.geometry
        self.load_heads = load_heads
        self.save_heads = save_heads
        self.trace = parent_trace
        self._geom = None
        self.data_dir = Path(data_dir) if data_dir is not None else cache_dir() / 'heads'
        if load_heads or save_heads:
            self.data_dir.mkdir(parents=True, exist_ok=True)

    def _save_attn(self, attn_slice: torch.Tensor):
        torch.save(attn_slice, self.data_dir / f'{self.trace._gen_idx}.pt')

    def _load_attn(self) -> torch.Tensor:
        return torch.load(self.data_dir / f'{self.trace._gen_idx}.pt')

    def _materialised_call(self, attn, query, key, value):
        """save_heads / load_heads (trace.py:276-302): the probabilities exist as a tensor -- written to / replaced
        from ``data_dir/{gen_idx}.pt`` -- heat maps and the layer output are both computed from that tensor."""
        bsz, n, _ = query.shape
        heads, tokens = attn.heads, key.shape[1]
        if self.save_heads:
            probs = ops.attention_probs(query, key, heads, attn.scale)     # [B*H, hw, 77], dtype of the pipeline
            self._save_attn(probs)
        else:
            probs = self._load_attn().to(query.device)
        factor = self.trace.geometry.level(probs.shape[1], self.layer_idx)[2]
        self.trace._gen_idx += 1
        if probs.shape[-1] == self.context_size and factor != 8:
            self.trace._accumulate_probs(self.layer_idx, factor, probs, bsz, heads)
        d = value.shape[-1] // heads
        v = value.view(bsz, tokens, heads, d).permute(0, 2, 1, 3).reshape(bsz * heads, tokens, d)
        out = torch.bmm(probs.to(v.dtype), v)
        out = out.view(bsz, heads, n, d).permute(0, 2, 1, 3).reshape(bsz, n, heads * d)
        return attn.to_out[1](attn.to_out[0](out))

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None):
        """attn2 forward: projections -> (heat-map kernel on Q/K) -> SDPA -> output projection."""
        if attention_mask is not None:
            raise RuntimeError('the heat-map kernel does not take an attention mask (SD cross-attention passes none)')
        bsz, n, _ = hidden_states.shape
        query = attn.to_q(hidden_states)
        if encoder_hidden_states is None:
            encoder_hidden_states = hidden_states
        elif attn.norm_cross is not None:
            encoder_hidden_states = attn.norm_cross(encoder_hidden_states)
        key = attn.to_k(encoder_hidden_states)
        value = attn.to_v(encoder_hidden_states)

        if self.save_heads or self.load_heads:
            return self._materialised_call(attn, query, key, value)

        heads = attn.heads
        tokens = key.shape[1]
        tr = self.trace
        geom = self._geom                                    # (n, tokens) -> factor and the trace / skip decision
        if geom is None or geom[0] != n or geom[1] != tokens:
            # trace.py:285-289; the tracer's geometry gives the factor (and drops this cache when the latent changes)
            traced = tokens == self.context_size
            if tr.long_prompts and not traced:
                if tokens not in _native.CONTEXT_TOKENS:
                    raise ValueError(f'layer {self.layer_idx}: a context of {tokens} tokens cannot be traced; '
                                     f'long_prompts=True traces {", ".join(map(str, _native.CONTEXT_TOKENS))} tokens '
                                     f'(1-3 CLIP chunks of 77)')
                traced = True
            if geom is not None and geom[1] != tokens:     # another context length: re-derive the layer's slab
                tr._layer_state.pop(self.layer_idx, None)
            factor = tr.geometry.level(n, self.layer_idx)[2] if traced else None
            geom = self._geom = (n, tokens, factor, traced and factor != 8)
        tr._gen_idx += 1
        if geom[3]:                                          # skip if too large (trace.py:289)
            if tr.value_norms:
                _check_value_norms(self.layer_idx, attn)
            tr._enqueue(self.layer_idx, geom[2], query, key, heads, attn.scale)
            if tr.value_norms:
                tr._see_values(self.layer_idx, encoder_hidden_states, value, attn.to_out[0].weight, heads)

        d = query.shape[-1] // heads
        q4 = query.view(bsz, n, heads, d).transpose(1, 2)
        k4 = key.view(bsz, tokens, heads, d).transpose(1, 2)
        v4 = value.view(bsz, tokens, heads, d).transpose(1, 2)
        out = F.scaled_dot_product_attention(q4, k4, v4, scale=attn.scale)
        out = out.transpose(1, 2).reshape(bsz, n, heads * d)
        out = attn.to_out[0](out)    # linear proj
        return attn.to_out[1](out)   # dropout

    def _hook_impl(self):
        self.original_processor = self.module.processor
        self.module.set_processor(self)

    def _unhook_impl(self):
        self.module.set_processor(self.original_processor)

    @property
    def num_heat_maps(self):
        return len(self.heat_maps)


class JointAttentionHooker(ObjectHooker):
    """The attention processor installed on one joint attention ``transformer_blocks[i].attn`` of an SD3 transformer,
    in place of diffusers' ``JointAttnProcessor2_0``. It computes what that processor computes, op for op, except that
    the attention runs through the SDPA op that also returns its log-sum-exp (flash for fp16 / bf16, memory-efficient
    for fp32): that is the normaliser of the image-query x text-key block the heat map keeps, and the attention had to
    compute it anyway. The layer call is then queued for ``daam_accumulate_joint``."""

    def __init__(self, module, parent_trace: 'trace', layer_idx: int = 0):
        super().__init__(module)
        self.heat_maps = parent_trace.all_heat_maps
        self.layer_idx = layer_idx
        self.trace = parent_trace

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, *args, **kwargs):
        if attention_mask is not None:
            raise ValueError(f'layer {self.layer_idx}: the joint-attention heat map does not take an attention mask '
                             f'(SD3 passes none)')
        if encoder_hidden_states is None:                  # no context, no text attention: the block as it was
            return self.original_processor(attn, hidden_states, encoder_hidden_states, attention_mask, *args,
                                           **kwargs)
        if torch.cuda.is_available() and torch.cuda.is_current_stream_capturing():
            raise RuntimeError('joint-attention heat maps cannot be captured into a CUDA graph: the layer hook, '
                               'which a graph replay bypasses, queues every call')
        residual = hidden_states
        bsz, heads = hidden_states.shape[0], attn.heads
        query = attn.to_q(hidden_states)
        key = attn.to_k(hidden_states)
        value = attn.to_v(hidden_states)
        d = key.shape[-1] // heads
        query = query.view(bsz, -1, heads, d).transpose(1, 2)
        key = key.view(bsz, -1, heads, d).transpose(1, 2)
        value = value.view(bsz, -1, heads, d).transpose(1, 2)
        if attn.norm_q is not None:
            query = attn.norm_q(query)
        if attn.norm_k is not None:
            key = attn.norm_k(key)
        ctx_q = attn.add_q_proj(encoder_hidden_states).view(bsz, -1, heads, d).transpose(1, 2)
        ctx_k = attn.add_k_proj(encoder_hidden_states).view(bsz, -1, heads, d).transpose(1, 2)
        ctx_v = attn.add_v_proj(encoder_hidden_states).view(bsz, -1, heads, d).transpose(1, 2)
        if attn.norm_added_q is not None:
            ctx_q = attn.norm_added_q(ctx_q)
        if attn.norm_added_k is not None:
            ctx_k = attn.norm_added_k(ctx_k)
        query = torch.cat([query, ctx_q], dim=2)
        key = torch.cat([key, ctx_k], dim=2)
        value = torch.cat([value, ctx_v], dim=2)
        out, lse = _attention_with_lse(query, key, value)
        n_image = residual.shape[1]
        self.trace._gen_idx += 1
        # the scale SDPA applies when none is given: 1 / sqrt(d), computed in double and used as a float
        self.trace._enqueue_joint(self.layer_idx, query, key, lse, n_image, heads, 1.0 / math.sqrt(d))
        hidden_states = out.transpose(1, 2).reshape(bsz, -1, heads * d).to(query.dtype)
        hidden_states, encoder_hidden_states = hidden_states[:, :n_image], hidden_states[:, n_image:]
        if not attn.context_pre_only:
            encoder_hidden_states = attn.to_add_out(encoder_hidden_states)
        hidden_states = attn.to_out[0](hidden_states)
        hidden_states = attn.to_out[1](hidden_states)
        return hidden_states, encoder_hidden_states

    def _hook_impl(self):
        self.original_processor = self.module.processor
        self.module.set_processor(self)

    def _unhook_impl(self):
        self.module.set_processor(self.original_processor)


class FluxAttentionHooker(JointAttentionHooker):
    """The attention processor installed on one attention of a FLUX.1 transformer, double-stream
    (``transformer_blocks[i].attn``, with a context) or single-stream (``single_transformer_blocks[j].attn``, on the
    joined sequence, ``encoder_hidden_states=None``), in place of diffusers' ``FluxAttnProcessor2_0`` /
    ``FluxAttnProcessor``. It computes what that processor computes, op for op: projections, q / k norms, for a double
    block the context projections and norms concatenated ahead of the image as ``[context, image]``, RoPE on q and k,
    one attention, then ``to_out`` and ``to_add_out`` (double) or the attention output alone (single, ``pre_only``).
    The attention runs through the SDPA op that also returns the log-sum-exp, as :class:`JointAttentionHooker`'s does.
    It reads only the submodules both diffusers' ``Attention`` and ``FluxAttention`` have, and ``attn.heads``."""

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None, image_rotary_emb=None,
                 *args, **kwargs):
        if attention_mask is not None:
            raise ValueError(f'layer {self.layer_idx}: the joint-attention heat map does not take an attention mask '
                             f'(FLUX passes none)')
        extra = [f'argument {i + 5}' for i, a in enumerate(args) if a is not None] + \
            [name for name, value in kwargs.items() if value is not None]
        if extra:                                          # e.g. an IP-Adapter's ip_hidden_states: not computed here
            raise ValueError(f'layer {self.layer_idx}: the FLUX heat-map hook computes the plain FLUX attention only, '
                             f'so it cannot take {", ".join(extra)} (the output would silently differ)')
        if torch.cuda.is_available() and torch.cuda.is_current_stream_capturing():
            raise RuntimeError('FLUX joint-attention heat maps cannot be captured into a CUDA graph: the layer hook, '
                               'which a graph replay bypasses, queues every call')
        bsz, heads = hidden_states.shape[0], attn.heads
        query = attn.to_q(hidden_states)
        key = attn.to_k(hidden_states)
        value = attn.to_v(hidden_states)
        d = key.shape[-1] // heads
        query = query.view(bsz, -1, heads, d).transpose(1, 2)
        key = key.view(bsz, -1, heads, d).transpose(1, 2)
        value = value.view(bsz, -1, heads, d).transpose(1, 2)
        if attn.norm_q is not None:
            query = attn.norm_q(query)
        if attn.norm_k is not None:
            key = attn.norm_k(key)
        if encoder_hidden_states is not None:              # double stream: [context, image]
            tokens = encoder_hidden_states.shape[1]
            ctx_q = attn.add_q_proj(encoder_hidden_states).view(bsz, -1, heads, d).transpose(1, 2)
            ctx_k = attn.add_k_proj(encoder_hidden_states).view(bsz, -1, heads, d).transpose(1, 2)
            ctx_v = attn.add_v_proj(encoder_hidden_states).view(bsz, -1, heads, d).transpose(1, 2)
            if attn.norm_added_q is not None:
                ctx_q = attn.norm_added_q(ctx_q)
            if attn.norm_added_k is not None:
                ctx_k = attn.norm_added_k(ctx_k)
            query = torch.cat([ctx_q, query], dim=2)
            key = torch.cat([ctx_k, key], dim=2)
            value = torch.cat([ctx_v, value], dim=2)
        else:                                              # single stream: the text rows come from the forward
            tokens = self.trace._flux_tokens
            if tokens is None:
                raise RuntimeError(f'layer {self.layer_idx}: a single-stream FLUX block was called outside a '
                                   f'transformer forward, so its context length is unknown')
        if image_rotary_emb is not None:
            query = _apply_rotary_emb(query, image_rotary_emb)
            key = _apply_rotary_emb(key, image_rotary_emb)
        out, lse = _attention_with_lse(query, key, value)
        self.trace._gen_idx += 1
        # the scale SDPA applies when none is given: 1 / sqrt(d), computed in double and used as a float
        self.trace._enqueue_joint(self.layer_idx, query, key, lse, query.shape[2] - tokens, heads, 1.0 / math.sqrt(d))
        hidden_states = out.transpose(1, 2).reshape(bsz, -1, heads * d).to(query.dtype)
        if encoder_hidden_states is None:
            return hidden_states
        encoder_hidden_states, hidden_states = hidden_states[:, :tokens], hidden_states[:, tokens:]
        hidden_states = attn.to_out[0](hidden_states)
        hidden_states = attn.to_out[1](hidden_states)
        encoder_hidden_states = attn.to_add_out(encoder_hidden_states)
        return hidden_states, encoder_hidden_states


def _apply_rotary_emb(x: torch.Tensor, freqs) -> torch.Tensor:
    """diffusers' ``apply_rotary_emb(x, (cos, sin), use_real=True, use_real_unbind_dim=-1)`` on ``x``
    ``[B, heads, L, d]`` with ``cos`` / ``sin`` ``[L, d]``: the interleaved pairs ``(x0, x1)`` rotate as
    ``(x0 cos - x1 sin, x1 cos + x0 sin)``, computed in fp32 and cast back."""
    cos, sin = freqs
    cos, sin = cos[None, None].to(x.device), sin[None, None].to(x.device)
    x_real, x_imag = x.reshape(*x.shape[:-1], -1, 2).unbind(-1)
    x_rotated = torch.stack([-x_imag, x_real], dim=-1).flatten(3)
    return (x.float() * cos + x_rotated.float() * sin).to(x.dtype)


def _attention_with_lse(query: torch.Tensor, key: torch.Tensor, value: torch.Tensor):
    """``(out, lse)``: SDPA of ``[B, heads, L, d]`` operands with the default scale, and its log-sum-exp (natural log,
    fp32 ``[B, heads, >= L]``). fp16 / bf16 take the flash kernel, fp32 the memory-efficient one (whose lse is padded
    to a multiple of 32 queries): the kernels ``F.scaled_dot_product_attention`` picks under the matching
    ``sdpa_kernel`` backend, so the output has their bits."""
    if query.dtype in (torch.float16, torch.bfloat16):
        res = torch.ops.aten._scaled_dot_product_flash_attention(query, key, value, 0.0, False, False)
    else:
        res = torch.ops.aten._scaled_dot_product_efficient_attention(query, key, value, None, True, 0.0, False)
    return res[0], res[1]


trace: Type[DiffusionHeatMapHooker] = DiffusionHeatMapHooker
