"""Heat-map store and algebra: the accumulator slabs the CUDA kernel sums into, and the global / word heat maps.

Mirror of the reference's L2 (``daam/heatmap.py``) for the hot-path rows of SURVEY.md section 8a:

* :class:`RawHeatMapCollection` (heatmap.py:148-172) -- same interface (``update``, ``factors``, ``layers``, ``heads``,
  iteration over ``((factor, layer, head), tensor[77, h, w])``, ``clear``), but backed by one fp32 device slab per traced
  layer, laid out ``[prompts][heads][77][h*w]``: the slab *is* the reference's per-key tensors (each key a contiguous
  view), and it is what ``daam_accumulate`` adds into, so nothing is copied or re-laid-out between kernel and API.
  A trace with ``negative=True`` keeps the unconditional half of the CFG batch in the same slab, below it.
* :class:`GlobalHeatMap` (heatmap.py:114-142) / :class:`WordHeatMap` (heatmap.py:56-96) -- ``compute_word_heat_map``
  and ``expand_as`` run the native kernels (``daam_word_heat_map``, ``daam_expand_as``).

The spaCy-parsed iterators and matplotlib overlays of the reference are out of scope (SURVEY.md section 2 row 2);
``plot_overlay`` is kept as a thin optional-matplotlib helper because ``expand_as(plot=True)`` calls it.
"""
from __future__ import annotations

import ctypes
import math
import numbers
from dataclasses import dataclass
from functools import lru_cache
from types import SimpleNamespace
from typing import Dict, Iterator, List, Optional, Set, Tuple, Union

import torch

from . import _native
from .utils import compute_token_merge_indices

__all__ = ['GlobalHeatMap', 'RawHeatMapCollection', 'WordHeatMap', 'LayerSlab', 'GlobalHeatMapStack', 'TimeHeatMaps',
           'ImageHeatMaps', 'LayerHeatMaps', 'FactorHeatMaps', 'HeadHeatMaps', 'RegionOverlap', 'RegionRanking', 'RegionBoundary', 'WordOverlap', 'RelationOverlap', 'WordInstances',
           'WordDistance']

RawHeatMapKey = Tuple[int, int, int]  # factor, layer, head


def _stream_ptr(device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def _require_cuda(t: torch.Tensor, what: str):
    if not t.is_cuda:
        raise RuntimeError(f'{what}: daam_b200 computes on CUDA tensors only (there is no CPU fallback)')


def _image_size(image, map_h: int, map_w: int) -> Tuple[int, int]:
    """``(out_h, out_w)`` a ``[map_h, map_w]`` map expands to over ``image``. A square map keeps the reference's
    ``size=(image.size[0], image.size[1])`` (heatmap.py:80; the same thing for the square images such maps come from);
    a non-square map comes from a non-square image and expands to ``(image.height, image.width)``."""
    if map_h == map_w:
        return int(image.size[0]), int(image.size[1])
    if hasattr(image, 'height') and hasattr(image, 'width'):
        return int(image.height), int(image.width)
    return int(image.size[1]), int(image.size[0])      # PIL-like ``size = (width, height)``


@dataclass
class LayerSlab:
    """Accumulators of one traced layer: ``acc[prompt][head]`` is the reference's ``[77, h, w]`` map of key
    ``(factor, layer_idx, head)``."""
    layer_idx: int
    factor: int
    heads: int
    h: int
    w: int
    acc: torch.Tensor            # fp32 [n_prompts, heads, 77, h*w]
    touched: bool = False        # a key exists only once it has been updated (defaultdict semantics)
    head_offset: int = 0         # first real head behind key head 0 (non-zero only for the un-guided B=1 quirk)
    captured: bool = False       # the layer's kernel launch is part of a CUDA graph: replays update it without the hook
    step: Optional[torch.Tensor] = None   # time-resolved traces only: what the last step added, shaped like ``acc``
    # step-range traces only: ``ranges[i]`` is shaped like ``acc`` and holds the sum over the steps of declared range i
    ranges: Optional[List[torch.Tensor]] = None
    # negative traces only: ``storage`` [2 * n_prompts, heads, 77, h*w] is what the layer's descriptor covers, the CFG
    # batch in its order; ``neg = storage[:n_prompts]`` (the unconditional half) and ``acc = storage[n_prompts:]``. The
    # step and range slabs then have ``storage``'s height too.
    storage: Optional[torch.Tensor] = None
    neg: Optional[torch.Tensor] = None
    # images per prompt: a prompt's ``heads`` keys are ``images`` runs of ``heads_per_image`` heads, image-major (key
    # head ``i * heads_per_image + h`` is head h of image i); 1 for slabs that ``RawHeatMapCollection.update`` creates
    images: int = 1
    # value-norm traces only (trace(pipe, value_norms=True)): ``norms`` [storage rows, heads, tokens] fp32 holds
    # ``||W_h v||`` of every key and context row, laid out like ``storage`` (or ``acc``) without the pixel axis;
    # ``norms_changed`` is a device bool, set when a later call of the generation saw other norms than the stored ones
    norms: Optional[torch.Tensor] = None
    norms_changed: Optional[torch.Tensor] = None
    # head-reduced joint traces only (trace(pipe, reduce_heads=True)): the number of heads whose mean each row of ``acc``
    # holds; ``acc`` is then [n_prompts, images, tokens, h*w], one key per image (``heads == images``); 0 otherwise
    head_mean: int = 0

    @property
    def n_prompts(self) -> int:
        return self.acc.shape[0]

    @property
    def tokens(self) -> int:
        """Context rows of every key: 77, or 154 / 231 in a ``long_prompts`` trace."""
        return self.acc.shape[2]

    @property
    def heads_per_image(self) -> int:
        return self.heads // self.images

    @property
    def second(self) -> List[torch.Tensor]:
        """The slabs the accumulate launches write next to ``acc``: the step slab, the range slabs, or none."""
        return [self.step] if self.step is not None else (self.ranges or [])

    def zero_(self):
        """Zero the accumulator and the range slabs (a step slab needs no zeroing: every step rewrites it whole)."""
        (self.acc if self.storage is None else self.storage).zero_()
        for r in self.ranges or ():
            r.zero_()

    def half(self, t: torch.Tensor, negative: bool = False) -> torch.Tensor:
        """The ``[n_prompts, heads, 77, h*w]`` half of a step or range slab that belongs to ``acc`` (or with
        ``negative`` to ``neg``); the slab itself when the trace keeps no negative half."""
        if self.storage is None:
            return t
        n = self.n_prompts
        return t[:n] if negative else t[n:]

    def source(self, step_range: Optional[int] = None, negative: bool = False) -> torch.Tensor:
        """What a read reduces: ``acc`` or ``neg``, or the matching half of range slab ``step_range``."""
        if step_range is None:
            return self.neg if negative else self.acc
        return self.half(self.ranges[step_range], negative)

    def norm_source(self, negative: bool = False) -> torch.Tensor:
        """The ``[n_prompts, heads, tokens]`` value norms of the keys ``source(..., negative)`` holds."""
        return self.half(self.norms, negative)

    def key_view(self, head: int, prompt: int = 0, step_range: Optional[int] = None,
                 negative: bool = False) -> torch.Tensor:
        src = self.source(step_range, negative)
        return src[prompt, head].view(src.shape[2], self.h, self.w)


class RawHeatMapCollection:
    """Per-(factor, layer, head) time-sums of attention maps, resident in HBM as fp32 slabs."""

    def __init__(self):
        self.slabs: Dict[int, LayerSlab] = {}
        self._order: List[int] = []          # layer indices in first-update order (the reference's dict order)
        self.epoch = 0                        # bumped whenever a slab object is (re)allocated (descriptor caches key on it)
        self._sync = None                     # callable making pending kernel work visible to the current stream
        self._zero = None                     # callable(slabs) zeroing slabs in accumulate-stream order
        self.time_resolved = False            # allocate a step slab next to every accumulator (trace(time_resolved=True))
        self.n_ranges = 0                     # range slabs next to every accumulator (trace(step_ranges=[...]))
        self.range_steps: List[int] = []      # UNet forwards each range has received since the last clear()
        self.negative = False                 # slabs also hold the unconditional half (trace(negative=True))
        self.value_norms = False              # slabs also hold every key's value norms (trace(value_norms=True))
        self.joint = False                    # joint-attention slabs: any context of 1 .. 1024 rows (SD3 traces)
        self.reduce_heads = False             # slabs hold each sample's head mean (trace(reduce_heads=True))

    # -- wiring from the tracer -------------------------------------------------------------------------------------
    def bind(self, sync, zero):
        self._sync, self._zero = sync, zero

    def _synchronize(self):
        if self._sync is not None:
            self._sync()

    def slab_for(self, layer_idx: int, factor: int, n_prompts: int, heads: int, h: int, w: int, device,
                 head_offset: int = 0, images: int = 1, tokens: int = _native.TOKENS, head_mean: int = 0) -> LayerSlab:
        """Returns (allocating or re-shaping on demand) the zero-initialised slab of a layer and marks it live.
        ``heads`` counts every image's heads of one prompt (``images`` runs of ``heads // images``); ``tokens`` is the
        context length (77, or 154 / 231 in a ``long_prompts`` trace): every context row is accumulated.
        ``head_mean``: the slab holds the mean of that many heads per image (``heads == images``), and every live
        layer must average the same number, or the mean of their rows is not the mean over their keys."""
        if tokens not in _native.CONTEXT_TOKENS and not (self.joint and 1 <= tokens <= _native.JOINT_MAX_TOKENS):
            raise ValueError(f'a slab holds a context of {_native.CONTEXT_TOKENS} tokens, not {tokens}')
        if head_mean:
            for other in self.live_slabs():
                if other.layer_idx != layer_idx and other.head_mean != head_mean:
                    raise RuntimeError(f'layer {layer_idx}: {head_mean} heads, but layer {other.layer_idx} of the '
                                       f'same trace has {other.head_mean}: reduce_heads=True averages each layer\'s '
                                       f'heads, which is the mean over keys only when every layer has as many')
        slab = self.slabs.get(layer_idx)
        shape = (n_prompts, heads, tokens, h * w)
        if slab is None or tuple(slab.acc.shape) != shape or slab.acc.device != torch.device(device) \
                or slab.factor != factor or (self.time_resolved and slab.step is None) \
                or (self.n_ranges and slab.ranges is None) or (self.negative and slab.neg is None) \
                or (self.value_norms and slab.norms is None):
            if torch.cuda.is_available() and torch.cuda.is_current_stream_capturing():
                raise RuntimeError('accumulator slabs cannot be created inside a CUDA-graph capture: run one eager '
                                   'UNet step under trace() before capturing')
            full = (2 * n_prompts,) + shape[1:] if self.negative else shape
            storage = torch.zeros(full, dtype=torch.float32, device=device)
            # the kernel writes every element of a step slab each step: no zeroing needed
            step = torch.empty(full, dtype=torch.float32, device=device) if self.time_resolved else None
            ranges = [torch.zeros(full, dtype=torch.float32, device=device) for _ in range(self.n_ranges)] \
                if self.n_ranges else None
            halves = dict(acc=storage[n_prompts:], storage=storage, neg=storage[:n_prompts]) if self.negative \
                else dict(acc=storage)
            if self.value_norms:
                halves.update(norms=torch.zeros(full[:3], dtype=torch.float32, device=device),
                              norms_changed=torch.zeros((), dtype=torch.bool, device=device))
            slab = LayerSlab(layer_idx, factor, heads, h, w, head_offset=head_offset, step=step, ranges=ranges,
                             images=images, **halves)
            self.slabs[layer_idx] = slab
            self.epoch += 1
        elif (slab.h, slab.w) != (h, w):      # same pixel count, other key shape (a transposed latent): re-tag
            slab.h, slab.w = h, w
        slab.images = images                  # (same key count, other split into images: only the tag changes)
        slab.head_mean = head_mean
        if not slab.touched:
            slab.touched = True
            self._order.append(layer_idx)
        return slab

    def mark_live(self, slab: LayerSlab):
        if not slab.touched:
            slab.touched = True
            self._order.append(slab.layer_idx)

    # -- reference interface ------------------------------------------------------------------------------------------
    def update(self, factor: int, layer_idx: int, head_idx: int, heatmap: torch.Tensor):
        """``acc[key] += heatmap`` for an externally produced ``[77, h, w]`` map (heatmap.py:153-156). The traced path
        never calls this -- the kernel accumulates in place -- it exists for API compatibility (e.g. merging maps)."""
        _require_cuda(heatmap, 'RawHeatMapCollection.update')
        self._synchronize()
        t, h, w = heatmap.shape
        slab = self.slabs.get(layer_idx)
        heads = max(head_idx + 1, slab.heads if slab is not None and slab.touched else 0)
        if slab is None or not slab.touched or slab.heads < heads or (slab.h, slab.w) != (h, w):
            old = slab if slab is not None and slab.touched and (slab.h, slab.w) == (h, w) else None
            acc = torch.zeros((1, heads, t, h * w), dtype=torch.float32, device=heatmap.device)
            if old is not None:
                acc[:, :old.heads] = old.acc[:1]
            new = LayerSlab(layer_idx, factor, heads, h, w, acc, touched=True)
            self.slabs[layer_idx] = new
            self.epoch += 1
            if layer_idx not in self._order:
                self._order.append(layer_idx)
            slab = new
        slab.acc[0, head_idx] += heatmap.reshape(t, h * w).float()

    def live_slabs(self) -> List[LayerSlab]:
        return [self.slabs[i] for i in self._order]

    def factors(self) -> Set[int]:
        return {s.factor for s in self.live_slabs()}

    def layers(self) -> Set[int]:
        return {s.layer_idx for s in self.live_slabs()}

    def heads(self) -> Set[int]:
        return {h for s in self.live_slabs() for h in range(s.heads)}

    def items(self, prompt: int = 0, *, step_range: Optional[int] = None,
              negative: bool = False) -> Iterator[Tuple[RawHeatMapKey, torch.Tensor]]:
        """``((factor, layer, head), [77, h, w])`` for every key; with ``step_range=i`` the per-key sums over the steps
        of declared range ``i`` (``trace(pipe, step_ranges=[...])``) instead of over every step; with ``negative`` those
        of the unconditional half of the CFG batch (``trace(pipe, negative=True)``)."""
        self.check_heads('all_heat_maps.items')
        for slab in self.read_slabs(step_range, negative):
            for head in range(slab.heads):
                yield (slab.factor, slab.layer_idx, head), slab.key_view(head, prompt, step_range, negative)

    def read_slabs(self, step_range: Optional[int] = None, negative: bool = False) -> List[LayerSlab]:
        """The slabs a read reduces, once every pending accumulate is visible: the live slabs, or with ``step_range``
        those with range slabs, after checking the index and that the range has received a step; with ``negative``
        only those that keep the unconditional half."""
        if step_range is not None:
            self.check_step_range(step_range)
        if negative:
            self.check_negative()
        self._synchronize()
        slabs = self.live_slabs()
        if negative:
            slabs = [s for s in slabs if s.neg is not None]
        if step_range is None:
            return slabs
        if self.range_steps[step_range] == 0:
            raise RuntimeError('No heat maps found for the given parameters.')
        return [s for s in slabs if s.ranges is not None]

    def check_heads(self, what: str):
        """Raises unless the slabs keep one key per head (not a ``trace(pipe, reduce_heads=True)``)."""
        if self.reduce_heads:
            raise RuntimeError(f'{what} reads per-head keys, which a trace(pipe, reduce_heads=True) does not keep: '
                               f'its layers hold the mean over heads only')

    def check_negative(self):
        """Raises unless the slabs keep the unconditional half (``trace(pipe, negative=True)``)."""
        if not self.negative:
            raise RuntimeError('negative heat maps need a trace declared with trace(pipe, negative=True)')

    def check_step_range(self, step_range: int):
        """Raises unless ``step_range`` indexes a range declared with ``trace(pipe, step_ranges=[...])``."""
        if not self.n_ranges:
            raise RuntimeError('step_range needs a trace declared with step_ranges, e.g. trace(pipe, '
                               'step_ranges=[(0, 10)])')
        if not isinstance(step_range, int) or not 0 <= step_range < self.n_ranges:
            raise IndexError(f'step_range {step_range!r} is not one of the {self.n_ranges} declared step ranges')

    def __iter__(self):
        return self.items(0)

    def __len__(self):
        return sum(s.heads for s in self.live_slabs())

    def clear(self):
        """Forget every key (heatmap.py:170-172). Slabs stay allocated and are zeroed in stream order for re-use."""
        live = self.live_slabs()
        if self._zero is not None:
            self._zero(live)
        else:
            for slab in live:
                slab.zero_()
        self.range_steps = [0] * self.n_ranges
        for slab in live:                     # graph-captured layers stay live: replays bypass the Python hook
            slab.touched = slab.captured
        self._order = [i for i in self._order if self.slabs[i].captured]


class WordHeatMap:
    def __init__(self, heatmap: torch.Tensor, word: str = None, word_idx: int = None):
        self.word = word
        self.word_idx = word_idx
        self.heatmap = heatmap

    @property
    def value(self):
        return self.heatmap

    def expand_as(self, image, absolute: bool = False, threshold: Optional[float] = None, plot: bool = False,
                  **plot_kwargs) -> torch.Tensor:
        """Bicubic-upsample to the image size, min-max normalise unless ``absolute``, optionally binarise; returns a
        CPU tensor like heatmap.py:77-93 (a square map keeps its ``size=(image.size[0], image.size[1])`` axis order; a
        non-square ``[h, w]`` map expands to ``[image.height, image.width]``)."""
        _require_cuda(self.heatmap, 'WordHeatMap.expand_as')
        src = self.heatmap.detach().float().contiguous()
        grid = tuple(src.shape[-2:])
        out_h, out_w = _image_size(image, *grid)
        out = torch.empty((out_h, out_w), dtype=torch.float32, device=src.device)
        scratch = torch.empty(_native.EXPAND_SCRATCH_FLOATS, dtype=torch.float32, device=src.device)
        with torch.cuda.device(src.device):
            _native.expand_as(src.data_ptr(), grid, out_h, out_w, absolute, threshold, out.data_ptr(),
                              scratch.data_ptr(), _stream_ptr(src.device))
        im = out.cpu()          # the reference returns a CPU tensor (heatmap.py:93); GlobalHeatMap.expand_words defers this
        if plot:
            self.plot_overlay(image, **plot_kwargs)
        return im

    def plot_overlay(self, image, out_file=None, color_normalize=True, ax=None, **expand_kwargs):
        """Optional visual helper (heatmap.py:20-53, 66-75); needs matplotlib, which the hot path does not."""
        try:
            from matplotlib import pyplot as plt
        except ImportError as e:  # pragma: no cover
            raise RuntimeError('plot_overlay needs matplotlib, which is not part of the heat-map hot path') from e
        import numpy as np
        heat = self.expand_as(image, **expand_kwargs)
        target = plt if ax is None else ax
        if color_normalize:
            target.imshow(heat.numpy(), cmap='jet')
        else:
            heat = heat.clamp(0, 1)
            target.imshow(heat.numpy(), cmap='jet', vmin=0.0, vmax=1.0)
        im = torch.from_numpy(np.array(image)).float() / 255
        target.imshow(torch.cat((im, 1 - heat.unsqueeze(-1)), dim=-1))
        if self.word is not None:
            (plt.title if ax is None else ax.set_title)(self.word)
        if out_file is not None:
            plt.savefig(out_file)

    def compute_ioa(self, other: 'WordHeatMap') -> float:
        """Intersection over own area -- daam/evaluate.py:26-35 (heatmap.py:95-96)."""
        from .evaluate import compute_ioa
        return compute_ioa(self.heatmap, other.heatmap)


class GlobalHeatMap:
    """``[n_prompt_tokens + 2, xh, xw]`` per-token maps plus the word lookup (heatmap.py:114-123); ``xh == xw`` for
    square images."""

    def __init__(self, tokenizer, prompt: str, heat_maps: torch.Tensor):
        self.tokenizer = tokenizer
        self.heat_maps = heat_maps
        self.prompt = prompt
        self.compute_word_heat_map = lru_cache(maxsize=50)(self.compute_word_heat_map)

    def compute_word_heat_map(self, word: str, word_idx: int = None, offset_idx: int = 0) -> WordHeatMap:
        out, word_idx = _word_heat_map(self.tokenizer, self.prompt, self.heat_maps, word, word_idx, offset_idx,
                                       'GlobalHeatMap.compute_word_heat_map')
        return WordHeatMap(out, word, word_idx)

    def expand_words(self, words, image, absolute: bool = False, threshold: Optional[float] = None,
                     word_idx=None, offset_idx: int = 0, to_cpu: bool = True):
        """``[self.compute_word_heat_map(w).expand_as(image, absolute, threshold) for w in words]`` -- the loop every user
        of the reference writes (heatmap.py:121-123 then 77-93) -- as ONE fused launch (gather-mean of the word's rows ->
        bicubic to the image size -> min/max -> normalise / threshold) and one device-to-host copy instead of four
        launches and a blocking copy per word.

        Returns ``(word_heat_maps, expanded)``: a list of :class:`WordHeatMap` (device ``[xh, xw]`` views, same values as
        ``compute_word_heat_map``) and ``expanded`` ``[len(words), out_h, out_w]`` -- the image size as
        :meth:`WordHeatMap.expand_as` orders it -- (CPU by default like
        ``expand_as``; ``to_cpu=False`` keeps it on the device until the caller needs it). ``word_idx`` may be a list
        parallel to ``words``. Raises the reference's ``ValueError`` for a word that is not in the prompt."""
        wl = _WordList(self.tokenizer, self.prompt, self.heat_maps[None], words, word_idx, offset_idx, image, absolute,
                       threshold, to_cpu, 'GlobalHeatMap.expand_words')
        if wl.empty:
            return [], torch.empty((0, wl.out_h, wl.out_w))
        out = torch.empty((len(wl.words), wl.out_h, wl.out_w), dtype=torch.float32, device=wl.dev)
        scratch = wl.scratch(_native.EXPAND_SCRATCH_FLOATS * len(wl.words))
        with torch.cuda.device(wl.dev):      # daam_expand_words takes one map and no map count
            _native.expand_words(wl.maps.data_ptr(), wl.n_rows, wl.grid, wl.rows, wl.out_h, wl.out_w, absolute,
                                 threshold, wl.word_maps.data_ptr(), out.data_ptr(), scratch.data_ptr(),
                                 _stream_ptr(wl.dev))
        _, out = wl.done(out)
        return wl.word_heat_maps(0), out

    def segment(self, words, image, absolute: bool = False, threshold: Optional[float] = None, word_idx=None,
                offset_idx: int = 0, to_cpu: bool = True):
        """A word label per image pixel: which word of ``words`` owns it, or background. With ``m`` the
        ``[len(words), H, W]`` that ``expand_words(words, image, absolute, word_idx=word_idx, offset_idx=offset_idx)``
        returns (no threshold), ``scores = m.max(0).values`` and ``labels = m.argmax(0) + 1`` (the first word on ties),
        set to 0 (background) where ``threshold`` is in effect (Python truthiness, as in ``expand_words``) and
        ``scores > threshold`` fails -- the reference's segmentation rule (``daam/evaluate.py``, tau = 0.4) over a word
        list. Two fused launches; the ``[len(words), H, W]`` stack is never materialised.

        Returns ``(word_heat_maps, labels, scores)``: the list of :class:`WordHeatMap` that ``expand_words`` returns,
        ``labels`` uint8 and ``scores`` fp32, both ``(H, W)`` ordered as ``expand_words`` orders the image size (CPU by
        default, ``to_cpu=False`` keeps them on the device). At most 96 words; repeated words tie and the first wins.
        An empty list gives all-background labels and -inf scores (the max of nothing). Raises the reference's
        ``ValueError`` for a word that is not in the prompt."""
        wl, labels, scores = _segment(self.tokenizer, self.prompt, self.heat_maps[None], words, image, absolute,
                                      threshold, word_idx, offset_idx, to_cpu, 'GlobalHeatMap.segment')
        return wl.word_heat_maps(0), labels[0], scores[0]

    def region_overlap(self, words, image, regions: torch.Tensor, absolute: bool = False,
                       threshold: Optional[float] = None, word_idx=None, offset_idx: int = 0, to_cpu: bool = True):
        """How much of each word's expanded map lies inside each image region: the sums behind the reference's
        ``compute_iou`` / ``compute_ioa`` (``daam/evaluate.py``) for every (word, region) pair at once. With ``m`` the
        ``[len(words), H, W]`` that ``expand_words(words, image, absolute, threshold, word_idx, offset_idx)`` returns
        (0/1 masks when ``threshold`` is in effect) and ``regions`` a device ``bool`` / ``uint8`` ``[R, H, W]`` or
        ``[H, W]`` tensor at that size (nonzero is inside), the :class:`RegionOverlap` holds
        ``intersection[r, w] = (m[w] * (regions[r] != 0)).sum()``, ``word_area[w] = m[w].sum()`` and
        ``region_area[r]``; its ``iou()`` / ``ioa()`` equal ``compute_iou`` / ``compute_ioa`` of every pair, bit for bit,
        when the threshold is in effect. Three fused launches; the ``[len(words), H, W]`` stack is never materialised.

        Returns ``(word_heat_maps, overlap)``: the list of :class:`WordHeatMap` that :meth:`segment` returns and the
        :class:`RegionOverlap` (CPU by default, ``to_cpu=False`` keeps it on the device). A ``[H, W]`` region is one
        region: the region axis stays, of length 1. At most 96 words, 63 regions and 2**24 image pixels. An empty word
        list or region set launches nothing, returns no word heat maps and measures no word (a word axis of length 0).
        Raises the reference's ``ValueError`` for a word that is not in the prompt."""
        wl, overlap = _region_overlap(self.tokenizer, self.prompt, self.heat_maps[None], words, image, regions,
                                      absolute, threshold, word_idx, offset_idx, to_cpu, 'GlobalHeatMap.region_overlap')
        return wl.word_heat_maps(0), overlap.map(0)

    def region_sweep(self, words, image, regions: torch.Tensor, thresholds, absolute: bool = False, word_idx=None,
                     offset_idx: int = 0, to_cpu: bool = True):
        """:meth:`region_overlap` at up to 64 thresholds in one pass: IoU, IoA, precision and recall as functions of the
        binarisation threshold, for every (word, region) pair. With ``m`` the ``[len(words), H, W]`` that
        ``expand_words(words, image, absolute, word_idx=word_idx, offset_idx=offset_idx)`` returns (no threshold) and
        ``R[r] = regions[r] != 0``, the :class:`RegionOverlap` holds the pixel counts ``intersection[k, r, w] = (R[r] &
        (m[w] > thresholds[k])).sum()`` and ``word_area[k, w] = (m[w] > thresholds[k]).sum()``, fp32 ``[T, R, W]`` and
        ``[T, W]``, and ``region_area[r]``; ``iou()``, ``ioa()`` and ``region_mean()`` (recall) are ``[T, R, W]``. For
        every nonzero threshold, slice ``k`` equals ``region_overlap(..., threshold=thresholds[k])`` bit for bit.
        One memset and three fused launches whatever the number of thresholds; the ``[len(words), H, W]`` stack is
        never materialised.

        ``thresholds``: 1 to 64 numbers (a sequence, or a 1-D CPU tensor), rounded to fp32 and then strictly ascending
        and finite, else a ``ValueError`` before anything reaches the device. Every entry is compared literally: unlike
        ``region_overlap``'s ``threshold``, where 0 means "no threshold", a 0 here counts ``m > 0`` and a negative
        value is a threshold too. Returns ``(word_heat_maps, overlap)`` as :meth:`region_overlap` does (CPU by default,
        ``to_cpu=False`` keeps it on the device), with the same limits (96 words, 63 regions, 2**24 image pixels), and
        an empty word list or region set launches nothing and measures no word (``[T, R, 0]``). Raises the reference's
        ``ValueError`` for a word that is not in the prompt."""
        wl, overlap = _region_sweep(self.tokenizer, self.prompt, self.heat_maps[None], words, image, regions,
                                    thresholds, absolute, word_idx, offset_idx, to_cpu, 'GlobalHeatMap.region_sweep')
        return wl.word_heat_maps(0), overlap.map(0)

    def region_ranking(self, words, image, regions: torch.Tensor, absolute: bool = False, word_idx=None,
                       offset_idx: int = 0, to_cpu: bool = True):
        """Threshold-free scores of each word's expanded map against each image region: pixel ROC-AUC and average
        precision, exact, for every (word, region) pair at once. With ``m`` the ``[len(words), H, W]`` that
        ``expand_words(words, image, absolute, word_idx=word_idx, offset_idx=offset_idx)`` returns (no threshold),
        values compared as fp32 numbers, ``P`` the pixels where ``regions[r] != 0`` and ``N`` the others, the
        :class:`RegionRanking` holds ``u2[r, w] = sum_{p in P, q in N} (2 [m_p > m_q] + [m_p == m_q])`` (int64, twice
        the Mann-Whitney U with ties counted half), ``ap[r, w]`` (float64, sklearn's ``average_precision_score`` of
        ``m[w]`` against the region: the area under the exact precision-recall curve, ties taken together) and
        ``region_area[r]``; ``auroc()`` is ``roc_auc_score``. Every plane is sorted on the device; the ``[len(words), H,
        W]`` stack never leaves it, and the results are the same bits on every call.

        Returns ``(word_heat_maps, ranking)``: the list of :class:`WordHeatMap` that :meth:`segment` returns and the
        :class:`RegionRanking` (CPU by default, ``to_cpu=False`` keeps it on the device). A ``[H, W]`` region is one
        region. At most 96 words, 63 regions and 2**24 image pixels. An empty word list or region set launches nothing,
        returns no word heat maps and scores no word (a word axis of length 0). Raises the reference's ``ValueError``
        for a word that is not in the prompt."""
        wl, ranking = _region_ranking(self.tokenizer, self.prompt, self.heat_maps[None], words, image, regions,
                                      absolute, word_idx, offset_idx, to_cpu, 'GlobalHeatMap.region_ranking')
        return wl.word_heat_maps(0), ranking.map(0)

    def region_boundary(self, words, image, regions: torch.Tensor, threshold: float, tolerances=None,
                        absolute: bool = False, word_idx=None, offset_idx: int = 0, to_cpu: bool = True):
        """Where each word's mask boundary lies against each image region's boundary: the boundary F-measure at pixel
        tolerances, the Hausdorff distance and the average symmetric surface distance, exact, for every (word, region)
        pair at once. With ``A`` the mask ``expand_words(words, image, absolute, threshold, word_idx=word_idx,
        offset_idx=offset_idx)`` returns for a word, ``B`` the pixels where ``regions[r] != 0``, ``dM`` the pixels of a
        mask ``M`` with a 4-neighbour outside ``M`` or outside the image, and ``d2`` the squared Euclidean distance
        between pixel centres to the nearest pixel of the other boundary, the :class:`RegionBoundary` holds
        ``word_boundary[w] = |dA|``, ``region_boundary[r] = |dB|``, ``word_hits[k, r, w]`` (the ``dA`` pixels with
        ``d2 <= tolerances[k]**2``), ``region_hits[k, r, w]`` (the ``dB`` pixels likewise), ``max_d2[r, w]`` and
        ``sum_dist[r, w]`` (both directions); ``f_score()``, ``hausdorff()`` and ``assd()`` are the scores. Every
        boundary pixel's nearest boundary pixel of the other set is found on the device; the ``[len(words), H, W]``
        stack never leaves it, and the results are the same bits on every call.

        ``threshold`` is required (the masks are ``expand_words``' thresholded masks) and must be finite.
        ``tolerances``: 1 to 16 pixel distances, finite, ``>= 0`` and strictly ascending after rounding to fp32; the
        default ``None`` is DAVIS's rule, one tolerance ``ceil(0.008 * sqrt(H**2 + W**2))`` (6 px at 512 x 512, 12 px
        at 1024 x 1024). The boundary here is the 4-neighbour boundary; DAVIS's toolkit thins and resizes its
        boundaries, so its F can differ slightly.

        Returns ``(word_heat_maps, boundary)``: the list of :class:`WordHeatMap` that :meth:`segment` returns and the
        :class:`RegionBoundary` (CPU by default, ``to_cpu=False`` keeps it on the device). A ``[H, W]`` region is one
        region. At most 96 words, 63 regions and 2**24 image pixels. An empty word list or region set launches nothing,
        returns no word heat maps and scores no word (a word axis of length 0). Raises the reference's ``ValueError``
        for a word that is not in the prompt."""
        wl, boundary = _region_boundary(self.tokenizer, self.prompt, self.heat_maps[None], words, image, regions,
                                        threshold, tolerances, absolute, word_idx, offset_idx, to_cpu,
                                        'GlobalHeatMap.region_boundary')
        return wl.word_heat_maps(0), boundary.map(0)

    def word_overlap(self, words, image=None, absolute: bool = False, threshold: Optional[float] = None,
                     word_idx=None, offset_idx: int = 0, to_cpu: bool = True):
        """How much each word's expanded map overlaps every other word's: the sums behind ``compute_iou`` /
        ``compute_ioa`` (``daam/evaluate.py``) and ``WordHeatMap.compute_ioa`` for every pair of ``words`` at once. With
        ``m`` the ``[len(words), H, W]`` that ``expand_words(words, image, absolute, threshold, word_idx, offset_idx)``
        returns (0/1 masks when ``threshold`` is in effect), the :class:`WordOverlap` holds ``intersection[a, b] =
        (m[a] * m[b]).sum()`` (symmetric bit for bit) and ``word_area[a] = m[a].sum()``; its ``iou()`` / ``ioa()`` equal
        ``compute_iou`` / ``compute_ioa`` of every pair of masks, bit for bit, when the threshold is in effect.
        ``image=None`` sums over the heat-map grid itself, where ``m`` is the word heat map (normalised unless
        ``absolute``): ``word_overlap(words, absolute=True, threshold=0.15)`` is the DAAM paper's head / dependent
        recipe. Three fused launches; the ``[len(words), H, W]`` stack is never materialised.

        Returns ``(word_heat_maps, overlap)``: the list of :class:`WordHeatMap` that :meth:`segment` returns and the
        :class:`WordOverlap` (CPU by default, ``to_cpu=False`` keeps it on the device). At most 96 words and 2**24
        pixels. An empty word list launches nothing and returns empty axes. Raises the reference's ``ValueError`` for a
        word that is not in the prompt."""
        wl, overlap = _word_overlap(self.tokenizer, self.prompt, self.heat_maps[None], words, image, absolute,
                                    threshold, word_idx, offset_idx, to_cpu, 'GlobalHeatMap.word_overlap')
        return wl.word_heat_maps(0), overlap.map(0)

    def relation_overlap(self, relations, image=None, absolute: bool = False, threshold: Optional[float] = None,
                         offset_idx: int = 0, to_cpu: bool = True) -> 'RelationOverlap':
        """The overlap of head and dependent of every relation of a parse -- what the reference's
        ``dependency_relations()`` pairs up, scored the way the DAAM paper's visuosyntactic analysis scores it, for a
        parse from any parser. ``relations``: ``(head, dep, rel)`` triples whose endpoints are words (``str``, looked up
        like ``compute_word_heat_map(word)``, every occurrence merged) or prompt token indices (``int``, as
        ``word_idx``). An edge with a word that is not in the prompt is skipped, as the reference does. The distinct
        endpoints go through one :meth:`word_overlap` call (at most 96); the returned :class:`RelationOverlap` gathers
        ``iou``, ``iod = ioa()[dep, head]`` and ``ioh = ioa()[head, dep]`` per kept edge. ``relation_overlap(relations,
        absolute=True, threshold=0.15)`` reproduces the paper's per-edge iou / iod / ioh."""
        return _relation_overlap(self.tokenizer, self.prompt, self.heat_maps[None], relations, image, absolute,
                                 threshold, offset_idx, to_cpu, 'GlobalHeatMap.relation_overlap').map(0)

    def word_instances(self, words, image, threshold: float, absolute: bool = False, max_instances: int = 16,
                       word_idx=None, offset_idx: int = 0, to_cpu: bool = True):
        """Where each word is and how many blobs it makes: the 8-connected components of each word's mask. The mask is
        what ``expand_words(words, image, absolute, threshold, word_idx, offset_idx)`` returns, ``pre > threshold`` with
        ``pre`` the expanded map without threshold; its components are those of ``scipy.ndimage.label(mask,
        structure=np.ones((3, 3)))``. The :class:`WordInstances` holds each word's component ``count`` and, for its
        ``max_instances`` largest components (ties to the one whose first pixel comes first in raster order), their
        ``area``, half-open ``box`` ``(y0, x0, y1, x1)``, exact index sums ``sum_yx``, ``peak`` of ``pre`` and the first
        pixel ``peak_yx`` where it is reached. ``largest_box()`` is the box of the weakly supervised localisation
        protocol; ``box_iou(gt_boxes)`` scores it. Fused on the device: the ``[len(words), H, W]`` stack never leaves
        it, and the results are the same bits on every call.

        Returns ``(word_heat_maps, instances)``: the list of :class:`WordHeatMap` that :meth:`segment` returns and the
        :class:`WordInstances` (CPU by default, ``to_cpu=False`` keeps it on the device). ``threshold`` must be truthy
        (a ``ValueError`` otherwise: without a mask there are no components); ``1 <= max_instances <= 64``; at most 96
        words and 2**24 image pixels. An empty word list launches nothing and returns empty axes. Raises the
        reference's ``ValueError`` for a word that is not in the prompt."""
        wl, inst = _word_instances(self.tokenizer, self.prompt, self.heat_maps[None], words, image, threshold, absolute,
                                   max_instances, word_idx, offset_idx, to_cpu, 'GlobalHeatMap.word_instances')
        return wl.word_heat_maps(0), inst.map(0)

    def word_distance(self, words, image, threshold: float, absolute: bool = False, word_idx=None, offset_idx: int = 0,
                      to_cpu: bool = True):
        """How far each pixel lies from each word's mask: the exact signed Euclidean distance transform of the mask
        ``expand_words(words, image, absolute, threshold, word_idx, offset_idx)`` returns, ``M = pre > threshold``
        with ``pre`` the expanded map without threshold. The :class:`WordDistance` holds ``signed_d2`` int32
        ``[len(words), H, W]``: at a pixel outside ``M`` the squared distance between pixel centres to the nearest
        pixel of ``M`` (``>= 1``), at a pixel of ``M`` minus the squared distance to the nearest pixel outside it
        (``<= -1``; the image border is not outside, so a mask touching it is not eaten from it); ``+2**31 - 1`` at
        every pixel of an empty mask and ``-(2**31 - 1)`` of a full one. Its helpers read every edit off it:
        ``mask(r)`` grows the mask by ``r`` pixels (dilation by a disk; ``r < 0`` erodes), ``soft_mask(r,
        feather=f)`` adds a linear edge of ``f`` pixels, ``distance()`` is the signed distance itself. E.g.
        ``word_distance(['dog'], image, 0.4)[1].soft_mask(grow=16, feather=8)[0]`` is an inpainting mask for the dog.
        Fused on the device in O(H W) work per word whatever the distances; the ``[len(words), H, W]`` stack of
        values never leaves it, and the results are the same bits on every call.

        Returns ``(word_heat_maps, distance)``: the list of :class:`WordHeatMap` that :meth:`segment` returns and the
        :class:`WordDistance` (CPU by default, ``to_cpu=False`` keeps it on the device). ``threshold`` must be truthy
        and finite (a ``ValueError`` otherwise); at most 96 words, 2**24 image pixels and 32767 pixels a side. An
        empty word list launches nothing and returns an empty word axis. Raises the reference's ``ValueError`` for a
        word that is not in the prompt."""
        wl, dist = _word_distance(self.tokenizer, self.prompt, self.heat_maps[None], words, image, threshold, absolute,
                                  word_idx, offset_idx, to_cpu, 'GlobalHeatMap.word_distance')
        return wl.word_heat_maps(0), dist.map(0)

    def overlay_words(self, words, image, absolute: bool = False, threshold: Optional[float] = None,
                      color_normalize: bool = True, word_idx=None, offset_idx: int = 0, to_cpu: bool = True):
        """The reference's ``plot_overlay`` (heatmap.py:20-53, 66-75) as pixels, for a word list: each word's expanded
        map coloured with matplotlib's ``jet`` (autoscaled to the map's min / max with ``color_normalize``, else
        clipped to [0, 1]) under the image drawn with alpha ``1 - heat``. With ``m`` the ``[len(words), H, W]`` that
        ``expand_words(words, image, absolute, threshold, word_idx, offset_idx)`` returns, frame ``w`` is, per pixel and
        channel, ``uint8(round((1 - a) * image + a * L[k]))`` with ``a = clamp(m[w], 0, 1)``, ``L`` the 256-entry table
        of :func:`jet_colormap` and ``k`` the colour index of ``m[w]`` (every operation rounded in fp32). Two fused
        launches; the ``[len(words), H, W]`` fp32 stack is never materialised.

        ``image``: a PIL image (converted to RGB), or a numpy / torch ``uint8`` ``[H, W, 3]`` array (a torch one on the
        CPU or on the heat map's device), ``(H, W)`` the size ``expand_words`` gives. Returns ``(word_heat_maps,
        frames)``: the list of :class:`WordHeatMap` that :meth:`segment` returns and ``frames`` uint8 ``[len(words), H,
        W, 3]`` (CPU by default, ``to_cpu=False`` keeps them on the device). At most 96 words; an empty list launches
        nothing. Raises the reference's ``ValueError`` for a word that is not in the prompt."""
        wl, frames = _overlay(self.tokenizer, self.prompt, self.heat_maps[None], words, image, absolute, threshold,
                              color_normalize, word_idx, offset_idx, to_cpu, 'GlobalHeatMap.overlay_words', stack=False)
        return wl.word_heat_maps(0), frames[0]

    def refine_words(self, words, image, radius: int = 8, eps: float = 1e-3, absolute: bool = False,
                     threshold: Optional[float] = None, word_idx=None, offset_idx: int = 0, to_cpu: bool = True):
        """Edge-aware word maps: each word's expanded map run through the guided filter (He, Sun and Tang, "Guided
        Image Filtering", TPAMI 2013, colour-guide form) with the image as guide, so that word boundaries follow the
        image's edges instead of the heat-map grid. With ``m[w]`` what ``expand_words(words, image, absolute,
        word_idx=word_idx, offset_idx=offset_idx)`` returns (no threshold), ``I`` the image's RGB bytes / 255 and
        ``mean`` the box mean over the ``(2 radius + 1)^2`` window clipped to the image (border windows shrink):
        ``mu = mean(I)``, ``Sigma = mean(I I^T) - mu mu^T``, ``a = (Sigma + eps Id)^-1 (mean(I m) - mu mean(m))``,
        ``b = mean(m) - a . mu`` and ``refined[w] = mean(a) . I + mean(b)``. The result is not clamped: it can
        overshoot ``[0, 1]`` slightly. With ``threshold`` in effect (Python truthiness, as in ``expand_words``) it is
        ``(refined > threshold)`` as fp32 1.0 / 0.0. ``eps`` is in the units of ``I^2``: small values keep finer edges.

        ``image``: as :meth:`overlay_words` takes it, a PIL image or a uint8 ``[H, W, 3]`` numpy / torch array at the size
        ``expand_words`` gives. Returns ``(word_heat_maps, refined)``: the list of :class:`WordHeatMap` that
        :meth:`segment` returns and ``refined`` fp32 ``[len(words), H, W]`` (CPU by default, ``to_cpu=False`` keeps it
        on the device). The image statistics come from exact integer window sums; the ``[len(words), H, W]`` stack of
        ``m`` is never written, and the results are the same bits on every call. ``1 <= radius <= 64``, ``eps`` finite
        and > 0 (a ``ValueError`` otherwise); at most 96 words. An empty word list launches nothing. Raises the
        reference's ``ValueError`` for a word that is not in the prompt."""
        wl, refined = _refine(self.tokenizer, self.prompt, self.heat_maps[None], words, image, radius, eps, absolute,
                              threshold, word_idx, offset_idx, to_cpu, 'GlobalHeatMap.refine_words', stack=False)
        return wl.word_heat_maps(0), refined[0]

    def segment_crf(self, words, image, threshold: Optional[float] = None, iterations: int = 5, radius: int = 8,
                    scale: float = 16.0, appearance: float = 10.0, sigma_xy: float = 8.0, sigma_rgb: float = 13.0,
                    smoothness: float = 1.0, sigma_smooth: float = 3.0, absolute: bool = False, word_idx=None,
                    offset_idx: int = 0, probs: bool = False, to_cpu: bool = True):
        """CRF-refined word segmentation: :meth:`segment`'s labels pulled onto the image's edges by mean-field
        inference of a Potts CRF (Kraehenbuehl and Koltun, NeurIPS 2011, in the exact windowed form of Teichmann and
        Cipolla's ConvCRF, BMVC 2019), in which the words compete with one another and with the background.

        With ``m[w]`` what ``expand_words(words, image, absolute, word_idx=word_idx, offset_idx=offset_idx)`` returns
        (no threshold): with ``threshold`` in effect (Python truthiness, as in :meth:`segment`) there are
        ``L = len(words) + 1`` labels, label 0 the background with score ``threshold``; without it ``L = len(words)``
        and no background. Word ``w`` is always label ``w + 1``, with score ``m[w]``. The unary logits are
        ``z = scale * score`` (fp32). The pairwise kernel of pixels ``x`` and ``y`` in the ``(2 radius + 1)^2`` window
        around ``x`` (clipped to the image, not renormalised at the border) is ``A[y - x] exp(-|I_x - I_y|^2 / 2
        sigma_rgb^2) + S[y - x]``, ``I`` the RGB bytes, ``A`` a Gaussian of width ``sigma_xy`` scaled to sum to
        ``appearance`` over the window's offsets and ``S`` one of width ``sigma_smooth`` summing to ``smoothness``
        (computed in float64, rounded once to fp32). Then ``Q = softmax(z)`` and ``iterations`` parallel updates
        ``Q = softmax(z + msg)``, ``msg_l(x) = sum_{y != x} k(x, y) Q_l(y)``.

        Returns ``(word_heat_maps, labels, scores)``, plus ``probs`` when asked: the list of :class:`WordHeatMap` that
        :meth:`segment` returns, ``labels`` uint8 ``(H, W)`` (the argmax of the last logits, the lowest label on
        ties), ``scores`` fp32 ``(H, W)`` (the final ``Q`` of that label) and ``probs`` fp32 ``(L, H, W)`` (the final
        ``Q``), CPU by default, ``to_cpu=False`` keeps them on the device. With ``iterations=0``, or ``appearance =
        smoothness = 0``, and ``scale`` a power of two, ``labels`` equals :meth:`segment`'s bit for bit (the scaling
        is exact and the tie rules match: the background wins at ``max m == threshold``, the first word otherwise).
        Every sum runs in an order fixed by pixel positions, so the results are the same bits on every call.

        ``image``: as :meth:`overlay_words` takes it. ``1 <= radius <= 16``, ``0 <= iterations <= 64``, ``scale``
        and the sigmas (``sigma_rgb`` in byte units) finite and > 0, ``appearance`` and ``smoothness`` finite and
        >= 0, a threshold in effect finite (a ``ValueError`` otherwise); at most 96 words. An empty word list
        launches nothing: every pixel is background with score 1 when the threshold is in effect, label 0 with score
        0 otherwise. Raises the reference's ``ValueError`` for a word that is not in the prompt."""
        wl, labels, scores, *q = _segment_crf(self.tokenizer, self.prompt, self.heat_maps[None], words, image,
                                              threshold, iterations, radius, scale, appearance, sigma_xy, sigma_rgb,
                                              smoothness, sigma_smooth, absolute, word_idx, offset_idx, probs, to_cpu,
                                              'GlobalHeatMap.segment_crf', stack=False)
        return (wl.word_heat_maps(0), labels[0], scores[0]) + ((q[0][0],) if probs else ())

    def segment_superpixels(self, words, image, n_segments: int = 1024, compactness: float = 20.0,
                            iterations: int = 10, threshold: Optional[float] = None, absolute: bool = False,
                            word_idx=None, offset_idx: int = 0, to_cpu: bool = True):
        """Superpixel word segmentation: the words compete per region of the image rather than per pixel, so the
        labels are constant over regions that follow the image's edges instead of the heat-map grid.

        The image is cut into SLIC superpixels (Achanta et al., TPAMI 2012), in the pixel-centric form on the RGB
        bytes with every step defined exactly (``include/daam_b200.h``): a grid of about ``n_segments`` cells, each
        cluster started from its cell's middle pixel, and ``iterations`` passes in which each pixel joins the nearest
        of the 9 clusters around its cell by ``|RGB - centre|^2 + wxy |yx - centre|^2``, ``wxy = compactness^2 *
        cells / (H W)``. ``compactness`` is on the 0-255 RGB scale: larger values give squarer superpixels, smaller
        ones follow colour more closely. The default of 20 is twice skimage's Lab default of 10 because RGB
        differences run larger than Lab's; nobody has measured which value segments DAAM maps best. Superpixels may
        be disconnected (there is no connectivity step).

        With ``m[w]`` what ``expand_words(words, image, absolute, word_idx=word_idx, offset_idx=offset_idx)`` returns
        (no threshold), each superpixel ``s`` gets ``mean[w] = fp32(sum_{p in s} m[w](p) / |s|)`` (the sum in float64
        in a fixed order), ``label = 1 + argmax_w mean[w]`` (the first word on ties), set to 0 (background) where
        ``threshold`` is in effect (Python truthiness, as in :meth:`segment`) and ``max mean > threshold`` fails, and
        ``score = max_w mean[w]``; every pixel takes its superpixel's. With ``n_segments = H * W`` every superpixel
        is one pixel and ``labels`` / ``scores`` equal :meth:`segment`'s bit for bit.

        Returns ``(word_heat_maps, labels, scores, superpixels)``: the list of :class:`WordHeatMap` that
        :meth:`segment` returns, ``labels`` uint8, ``scores`` fp32 and ``superpixels`` int32 (each pixel's cluster
        id, ``cy * nx + cx``; empty clusters leave ids unused), all ``(H, W)``, CPU by default, ``to_cpu=False``
        keeps them on the device. The results are the same bits on every call.

        ``image``: as :meth:`overlay_words` takes it. ``n_segments`` an integer >= 1 whose grid has at most 65536
        cells, ``compactness`` finite and > 0, ``iterations`` an integer in ``[1, 64]``, at most 2**24 pixels (a
        ``ValueError`` otherwise); at most 96 words. An empty word list still makes the partition: every pixel is
        background with score -inf. Raises the reference's ``ValueError`` for a word that is not in the prompt."""
        wl, labels, scores, sp = _segment_superpixels(self.tokenizer, self.prompt, self.heat_maps[None], words, image,
                                                      n_segments, compactness, iterations, threshold, absolute,
                                                      word_idx, offset_idx, to_cpu, 'GlobalHeatMap.segment_superpixels',
                                                      stack=False)
        return wl.word_heat_maps(0), labels[0], scores[0], sp


def _check_rows(rows, n_rows: int):
    """Raises the ``IndexError`` torch's advanced indexing raises on a row out of ``[-n_rows, n_rows)``."""
    for r in rows:
        if not -n_rows <= r < n_rows:
            raise IndexError(f'index {r} is out of bounds for dimension 0 with size {n_rows}')


def _word_heat_map(tokenizer, prompt: str, maps: torch.Tensor, word: str, word_idx, offset_idx: int, what: str):
    """``daam_word_heat_map`` of ``word`` over ``maps`` ``[..., n_rows, xh, xw]``, one launch per ``[n_rows, xh, xw]``
    map: returns ``(out, word_idx)``, ``out`` the device ``[..., xh, xw]`` word heat maps."""
    rows, word_idx = compute_token_merge_indices(tokenizer, prompt, word, word_idx, offset_idx)
    _require_cuda(maps, what)
    *lead, n_rows, h, w = maps.shape           # ``lead``: [] for one map, [n_maps] for a stack
    _check_rows(rows, n_rows)
    maps = maps.detach().float().contiguous()
    out = torch.empty((*lead, h, w), dtype=torch.float32, device=maps.device)
    out_bytes = 4 * h * w                      # one fp32 map of ``out``; ``maps`` holds ``n_rows`` of them per map
    with torch.cuda.device(maps.device):
        stream = _stream_ptr(maps.device)
        for t in range(lead[0] if lead else 1):
            _native.word_heat_map(maps.data_ptr() + t * n_rows * out_bytes, n_rows, (h, w), rows,
                                  out.data_ptr() + t * out_bytes, stream)
    return out, word_idx


class _WordList:
    """One fused word-list call over ``maps`` ``[n_maps, n_rows, xh, xw]``. Its checks run in the order they raise:
    ``compute_token_merge_indices`` of every word (``word_idx`` may be a list parallel to ``words``; the reference's
    ``ValueError`` for a word not in the prompt, then the row range as torch's advanced indexing checks it), then the
    CUDA check. Holds the contiguous fp32 maps, the device word heat maps ``[n_maps, len(words), xh, xw]`` the launch
    writes, and the size ``out_h, out_w`` the maps expand to over ``image`` (the heat-map grid itself ``on_grid``).
    ``empty``: there is no word or no map, and nothing to launch."""

    def __init__(self, tokenizer, prompt: str, maps: torch.Tensor, words, word_idx, offset_idx: int, image,
                 absolute: bool, threshold: Optional[float], to_cpu: bool, what: str, on_grid: bool = False):
        self.words = words = list(words)
        n_maps, n_rows, grid = maps.shape[0], maps.shape[1], tuple(maps.shape[-2:])
        self.n_maps, self.n_rows, self.grid = n_maps, n_rows, grid
        idxs = list(word_idx) if isinstance(word_idx, (list, tuple)) else [word_idx] * len(words)
        self.merged = [compute_token_merge_indices(tokenizer, prompt, w, i, offset_idx) for w, i in zip(words, idxs)]
        self.rows = [rows for rows, _ in self.merged]
        _check_rows([r for rows in self.rows for r in rows], n_rows)
        _require_cuda(maps, what)
        self.dev = dev = maps.device
        self.maps = maps.detach().float().contiguous()
        self.word_maps = torch.empty((n_maps, len(words)) + grid, dtype=torch.float32, device=dev)
        self.out_h, self.out_w = grid if on_grid else _image_size(image, *grid)
        self.absolute, self.threshold, self.to_cpu = absolute, threshold, to_cpu
        self.empty = not words or n_maps == 0

    def scratch(self, n_floats: int) -> torch.Tensor:
        return torch.empty(n_floats, dtype=torch.float32, device=self.dev)

    def launch(self, entry, *args):
        """``entry``, a ``_native`` word-list call over ``n_maps`` maps, on the maps' device and its current stream:
        the arguments every such call starts with, then ``args``."""
        with torch.cuda.device(self.dev):
            entry(self.maps.data_ptr(), self.n_maps, self.n_rows, self.grid, self.rows, self.out_h, self.out_w,
                  self.absolute, self.threshold, *args, _stream_ptr(self.dev))

    def done(self, *results):
        """``(self, *results)``, the results copied to the host when the call asked for it."""
        return (self, *[r.cpu() for r in results]) if self.to_cpu else (self, *results)

    def word_heat_maps(self, i: int) -> List[WordHeatMap]:
        """One :class:`WordHeatMap` per word of map ``i``: its device ``[xh, xw]`` map, the word and its index."""
        maps = self.word_maps[i]
        return [WordHeatMap(maps[j], w, idx) for j, (w, (_, idx)) in enumerate(zip(self.words, self.merged))]


def _segment(tokenizer, prompt: str, maps: torch.Tensor, words, image, absolute, threshold, word_idx, offset_idx: int,
             to_cpu: bool, what: str):
    """``daam_segment_words`` over ``maps`` ``[n_maps, n_rows, xh, xw]``: returns ``(wl, labels, scores)``, the
    :class:`_WordList` and ``labels`` / ``scores`` ``[n_maps, H, W]``."""
    wl = _WordList(tokenizer, prompt, maps, words, word_idx, offset_idx, image, absolute, threshold, to_cpu, what)
    shape = (wl.n_maps, wl.out_h, wl.out_w)
    if wl.empty:
        return wl.done(torch.zeros(shape, dtype=torch.uint8, device=wl.dev),
                       torch.full(shape, float('-inf'), device=wl.dev))
    labels = torch.empty(shape, dtype=torch.uint8, device=wl.dev)
    scores = torch.empty(shape, dtype=torch.float32, device=wl.dev)
    scratch = wl.scratch(_native.segment_scratch_floats(wl.n_maps, len(wl.words)))
    wl.launch(_native.segment_words, wl.word_maps.data_ptr(), labels.data_ptr(), scores.data_ptr(), scratch.data_ptr())
    return wl.done(labels, scores)


@dataclass
class RegionOverlap:
    """Sums of word maps over image regions (:meth:`GlobalHeatMap.region_overlap`): ``intersection`` ``[..., R, W]``
    (``sum_p region[r](p) * m[w](p)``), ``word_area`` ``[..., W]`` (``sum_p m[w](p)``) and ``region_area`` ``[R]``
    (pixels inside each region), fp32. ``...`` is the map axis of a :class:`GlobalHeatMapStack`, absent for one map,
    followed by the threshold axis of :meth:`GlobalHeatMap.region_sweep` (``[..., T, R, W]``, ``[..., T, W]``).
    The scores are the reference's formulas (``daam/evaluate.py``) in the same fp32 operation order."""
    intersection: torch.Tensor
    word_area: torch.Tensor
    region_area: torch.Tensor

    def map(self, i: int) -> 'RegionOverlap':
        """The overlap of map ``i`` of a stack (``region_area`` has no map axis and stays whole)."""
        return RegionOverlap(self.intersection[i], self.word_area[i], self.region_area)

    def cpu(self) -> 'RegionOverlap':
        return RegionOverlap(self.intersection.cpu(), self.word_area.cpu(), self.region_area.cpu())

    def iou(self) -> torch.Tensor:
        """``I / (A_w + A_r - I + 1e-8)``: ``compute_iou(mask, region)`` of every pair."""
        i = self.intersection
        return i / (self.word_area.unsqueeze(-2) + self.region_area.unsqueeze(-1) - i + 1e-8)

    def ioa(self) -> torch.Tensor:
        """``I / (A_w + 1e-8)``: ``compute_ioa(mask, region)`` of every pair, the intersection over the word's area."""
        return self.intersection / (self.word_area.unsqueeze(-2) + 1e-8)

    def region_mean(self) -> torch.Tensor:
        """``I / (A_r + 1e-8)``: without a threshold the mean of the word's expanded map inside the region, with one the
        fraction of the region the word's mask covers."""
        return self.intersection / (self.region_area.unsqueeze(-1) + 1e-8)


def _region_overlap(tokenizer, prompt: str, maps: torch.Tensor, words, image, regions, absolute, threshold, word_idx,
                    offset_idx: int, to_cpu: bool, what: str):
    """``daam_region_overlap`` over ``maps`` ``[n_maps, n_rows, xh, xw]``: returns ``(wl, overlap)``, the
    :class:`_WordList` and the :class:`RegionOverlap` with a leading map axis. Without regions no word is measured: the
    word list then holds no word and no word heat map."""
    wl = _WordList(tokenizer, prompt, maps, words, word_idx, offset_idx, image, absolute, threshold, to_cpu, what)
    n_maps, out_h, out_w, dev = wl.n_maps, wl.out_h, wl.out_w, wl.dev
    region_bytes = _region_bytes(wl, regions, what)
    n_regions, n_words = region_bytes.shape[0], len(wl.words)
    if wl.empty or n_regions == 0:            # no word is measured: the call returns no word heat maps
        return wl.done(_no_region_overlap(wl, (), n_regions))
    inter = torch.empty((n_maps, n_regions, n_words), dtype=torch.float32, device=dev)
    area = torch.empty((n_maps, n_words), dtype=torch.float32, device=dev)
    scratch = wl.scratch(_native.region_scratch_floats(n_maps, n_words, n_regions, out_h, out_w))
    wl.launch(_native.region_overlap, wl.word_maps.data_ptr(), region_bytes.data_ptr(), n_regions, inter.data_ptr(),
              area.data_ptr(), scratch.data_ptr())
    return wl.done(RegionOverlap(inter, area, _region_area(region_bytes)))


def _region_bytes(wl: _WordList, regions, what: str) -> torch.Tensor:
    """``regions`` checked against the word list's output size and device, as uint8 ``[R, H, W]`` on the device: a
    ``[H, W]`` region is one region."""
    if not isinstance(regions, torch.Tensor):
        raise TypeError(f'{what}: regions must be a torch.Tensor, not {type(regions).__name__}')
    if regions.dtype not in (torch.bool, torch.uint8):
        raise TypeError(f'{what}: regions must be bool or uint8, not {regions.dtype}')
    if regions.dim() == 2:
        regions = regions[None]
    out_h, out_w = wl.out_h, wl.out_w
    if regions.dim() != 3 or tuple(regions.shape[1:]) != (out_h, out_w):
        raise ValueError(f'{what}: regions of shape {tuple(regions.shape)} do not match the expanded maps\' '
                         f'(R, {out_h}, {out_w}) (a [{out_h}, {out_w}] region or a stack of them)')
    _require_cuda(regions, what)
    if regions.device != wl.dev:
        raise ValueError(f'{what}: regions are on {regions.device}, the heat maps on {wl.dev}')
    return regions.detach().contiguous().view(torch.uint8)


def _region_area(region_bytes: torch.Tensor) -> torch.Tensor:
    """Exact pixel counts (at most 2**24 pixels): what ``region.float().sum()`` gives in compute_iou."""
    return (region_bytes != 0).sum((-1, -2)).float()


def _no_region_overlap(wl: _WordList, lead: Tuple[int, ...], n_regions: int) -> RegionOverlap:
    """The overlap of a call that measures no word: the word list then holds no word and no word heat map, and the
    sums have a word axis of length 0 after the map axis and ``lead``."""
    n_maps, dev = wl.n_maps, wl.dev
    wl.words, wl.merged = [], []
    wl.word_maps = torch.empty((n_maps, 0) + wl.grid, dtype=torch.float32, device=dev)
    return RegionOverlap(torch.zeros((n_maps, *lead, n_regions, 0), device=dev),
                         torch.zeros((n_maps, *lead, 0), device=dev), torch.zeros((n_regions,), device=dev))


def _sweep_thresholds(thresholds, what: str) -> List[float]:
    """``thresholds`` (a sequence of numbers or a 1-D CPU tensor) rounded to fp32, as the Python floats of those fp32
    values; a ``ValueError`` unless they are 1 to 64 finite, strictly ascending values after the rounding."""
    if isinstance(thresholds, torch.Tensor):
        if thresholds.device.type != 'cpu' or thresholds.dim() != 1 or thresholds.dtype == torch.bool \
                or thresholds.is_complex():
            raise ValueError(f'{what}: thresholds must be a 1-D real CPU tensor, not {thresholds.dim()}-D '
                             f'{thresholds.dtype} on {thresholds.device}')
        taus = thresholds.detach().to(torch.float32)
    else:
        try:
            values = list(thresholds)
        except TypeError:
            raise ValueError(f'{what}: thresholds must be a sequence of numbers, not {thresholds!r}') from None
        if not all(isinstance(x, numbers.Real) and not isinstance(x, bool) for x in values):
            raise ValueError(f'{what}: thresholds must be numbers, not {values!r}')
        taus = torch.tensor([float(x) for x in values], dtype=torch.float64).to(torch.float32)
    n = taus.numel()
    if not 1 <= n <= _native.SWEEP_MAX_THRESHOLDS:
        raise ValueError(f'{what}: {n} thresholds; a sweep takes 1 to {_native.SWEEP_MAX_THRESHOLDS}')
    if not bool(torch.isfinite(taus).all()):
        raise ValueError(f'{what}: thresholds must be finite in fp32, not {taus.tolist()}')
    if not bool((taus[1:] > taus[:-1]).all()):
        raise ValueError(f'{what}: thresholds must be strictly ascending after rounding to fp32, not {taus.tolist()}')
    return taus.tolist()


def _region_sweep(tokenizer, prompt: str, maps: torch.Tensor, words, image, regions, thresholds, absolute, word_idx,
                  offset_idx: int, to_cpu: bool, what: str):
    """``daam_region_sweep`` over ``maps`` ``[n_maps, n_rows, xh, xw]``: returns ``(wl, overlap)``, the
    :class:`_WordList` and the :class:`RegionOverlap` with a leading map axis and a threshold axis before the region
    axis. The thresholds are checked first, then everything ``_region_overlap`` checks, in its order."""
    taus = _sweep_thresholds(thresholds, what)
    wl = _WordList(tokenizer, prompt, maps, words, word_idx, offset_idx, image, absolute, taus, to_cpu, what)
    n_maps, out_h, out_w, dev = wl.n_maps, wl.out_h, wl.out_w, wl.dev
    region_bytes = _region_bytes(wl, regions, what)
    n_regions, n_words, n_thr = region_bytes.shape[0], len(wl.words), len(taus)
    if wl.empty or n_regions == 0:
        return wl.done(_no_region_overlap(wl, (n_thr,), n_regions))
    inter = torch.empty((n_maps, n_thr, n_regions, n_words), dtype=torch.float32, device=dev)
    area = torch.empty((n_maps, n_thr, n_words), dtype=torch.float32, device=dev)
    scratch = wl.scratch(_native.region_sweep_scratch_floats(n_maps, n_words, n_regions, n_thr, out_h, out_w))
    wl.launch(_native.region_sweep, wl.word_maps.data_ptr(), region_bytes.data_ptr(), n_regions, inter.data_ptr(),
              area.data_ptr(), scratch.data_ptr())
    return wl.done(RegionOverlap(inter, area, _region_area(region_bytes)))


# Scratch of one region_ranking call: as many (map, word) planes as fit are sorted per round (about 18 bytes a pixel
# each), so memory does not grow with the number of maps; a plane larger than the budget goes alone.
REGION_RANKING_SCRATCH_BYTES = 256 << 20


@dataclass
class RegionRanking:
    """Threshold-free scores of word maps against image regions (:meth:`GlobalHeatMap.region_ranking`): ``u2`` int64
    ``[..., R, W]`` (twice the Mann-Whitney U of the word's values inside the region against those outside, ties
    counted half), ``ap`` float64 ``[..., R, W]`` (average precision; NaN for an empty region), ``region_area`` int64
    ``[R]`` (pixels inside each region) and ``n_pixels`` (pixels of the image). ``...`` is the map axis of a
    :class:`GlobalHeatMapStack`, absent for one map."""
    u2: torch.Tensor
    ap: torch.Tensor
    region_area: torch.Tensor
    n_pixels: int

    def map(self, i: int) -> 'RegionRanking':
        """The scores of map ``i`` of a stack (``region_area`` has no map axis and stays whole)."""
        return RegionRanking(self.u2[i], self.ap[i], self.region_area, self.n_pixels)

    def cpu(self) -> 'RegionRanking':
        return RegionRanking(self.u2.cpu(), self.ap.cpu(), self.region_area.cpu(), self.n_pixels)

    def auroc(self) -> torch.Tensor:
        """float64 ``[..., R, W]``: ``u2 / (2 n_p n_n)``, the pixel ROC-AUC (``roc_auc_score``) of every pair, with
        ``n_p`` the region's pixels and ``n_n`` the others; NaN when either is 0."""
        n_p = self.region_area.to(device=self.u2.device, dtype=torch.float64).unsqueeze(-1)
        n_n = self.n_pixels - n_p
        denom = 2 * n_p * n_n
        return torch.where(denom > 0, self.u2.double() / denom.clamp(min=1), torch.full_like(denom, float('nan')))


def _region_ranking(tokenizer, prompt: str, maps: torch.Tensor, words, image, regions, absolute, word_idx,
                    offset_idx: int, to_cpu: bool, what: str):
    """``daam_region_ranking`` over ``maps`` ``[n_maps, n_rows, xh, xw]``: returns ``(wl, ranking)``, the
    :class:`_WordList` and the :class:`RegionRanking` with a leading map axis. Checks as ``_region_overlap``, in its
    order. Scratch: :data:`REGION_RANKING_SCRATCH_BYTES`, clipped to the planes the call has, at least one plane."""
    wl = _WordList(tokenizer, prompt, maps, words, word_idx, offset_idx, image, absolute, None, to_cpu, what)
    n_maps, out_h, out_w, dev = wl.n_maps, wl.out_h, wl.out_w, wl.dev
    region_bytes = _region_bytes(wl, regions, what)
    n_regions, n_words = region_bytes.shape[0], len(wl.words)
    if wl.empty or n_regions == 0:            # no word is scored: the call returns no word heat maps
        _no_region_overlap(wl, (), n_regions)
        return wl.done(RegionRanking(torch.zeros((n_maps, n_regions, 0), dtype=torch.int64, device=dev),
                                     torch.zeros((n_maps, n_regions, 0), dtype=torch.float64, device=dev),
                                     torch.zeros((n_regions,), dtype=torch.int64, device=dev), out_h * out_w))
    u2 = torch.empty((n_maps, n_regions, n_words), dtype=torch.int64, device=dev)
    ap = torch.empty((n_maps, n_regions, n_words), dtype=torch.float64, device=dev)
    n_bytes = max(_native.region_ranking_scratch_bytes(1, out_h, out_w),
                  min(REGION_RANKING_SCRATCH_BYTES, _native.region_ranking_scratch_bytes(n_maps * n_words, out_h, out_w)))
    scratch = torch.empty(n_bytes, dtype=torch.uint8, device=dev)
    wl.launch(_native.region_ranking, wl.word_maps.data_ptr(), region_bytes.data_ptr(), n_regions, u2.data_ptr(),
              ap.data_ptr(), scratch.data_ptr(), n_bytes)
    return wl.done(RegionRanking(u2, ap, (region_bytes != 0).sum((-1, -2)), out_h * out_w))


# Scratch of one region_boundary / boundary_scores call: the regions' column distances (about 4 bytes a pixel per
# region) once, then as many planes as fit per round (about 8 bytes a pixel each), so memory does not grow with the
# number of maps. The regions' state alone can exceed the budget -- 63 regions at 1024 x 1024 take about 264 MB -- and
# the call then takes the regions and one plane, whatever the budget.
REGION_BOUNDARY_SCRATCH_BYTES = 256 << 20


@dataclass
class RegionBoundary:
    """Boundary scores of word masks against image regions (:meth:`GlobalHeatMap.region_boundary`,
    :func:`daam_b200.evaluate.boundary_scores`). With ``dA`` a word mask's boundary, ``dB`` a region's and ``d2`` the
    squared distance between pixel centres to the nearest pixel of the other boundary: ``word_boundary`` int32
    ``[..., W]`` (``|dA|``), ``region_boundary`` int32 ``[R]`` (``|dB|``), ``word_hits`` / ``region_hits`` int32 ``[...,
    T, R, W]`` (the ``dA`` / ``dB`` pixels within ``tolerances[k]``), ``max_d2`` int64 ``[..., R, W, 2]`` (the largest
    ``d2`` from ``dA`` and from ``dB``; -1 when either boundary is empty), ``sum_dist`` float64 ``[..., R, W, 2]`` (the
    sums of ``sqrt(d2)``; 0 when either boundary is empty) and ``tolerances`` fp32 ``[T]``. ``...`` is the map axis of a
    :class:`GlobalHeatMapStack`, absent for one map."""
    word_boundary: torch.Tensor
    region_boundary: torch.Tensor
    word_hits: torch.Tensor
    region_hits: torch.Tensor
    max_d2: torch.Tensor
    sum_dist: torch.Tensor
    tolerances: torch.Tensor

    def map(self, i: int) -> 'RegionBoundary':
        """The scores of map ``i`` of a stack (``region_boundary`` and ``tolerances`` have no map axis and stay whole)."""
        return RegionBoundary(self.word_boundary[i], self.region_boundary, self.word_hits[i], self.region_hits[i],
                              self.max_d2[i], self.sum_dist[i], self.tolerances)

    def cpu(self) -> 'RegionBoundary':
        return RegionBoundary(self.word_boundary.cpu(), self.region_boundary.cpu(), self.word_hits.cpu(),
                              self.region_hits.cpu(), self.max_d2.cpu(), self.sum_dist.cpu(), self.tolerances.cpu())

    def _sizes(self):
        """``(|dA|, |dB|)`` as float64, broadcastable to ``[..., R, W]``."""
        dev = self.word_hits.device
        n_a = self.word_boundary.to(device=dev, dtype=torch.float64).unsqueeze(-2)
        n_b = self.region_boundary.to(device=dev, dtype=torch.float64).unsqueeze(-1)
        return n_a, n_b

    def precision(self) -> torch.Tensor:
        """float64 ``[..., T, R, W]``: ``word_hits / |dA|``, the share of the word's boundary within the tolerance of
        the region's; 1 when ``dA`` is empty (DAVIS's ``f_measure``)."""
        n_a, _ = self._sizes()
        n_a = n_a.unsqueeze(-3)
        return torch.where(n_a > 0, self.word_hits.double() / n_a.clamp(min=1), torch.ones_like(n_a))

    def recall(self) -> torch.Tensor:
        """float64 ``[..., T, R, W]``: ``region_hits / |dB|``, the share of the region's boundary within the tolerance
        of the word's; 1 when ``dB`` is empty."""
        _, n_b = self._sizes()
        n_b = n_b.unsqueeze(-3)
        return torch.where(n_b > 0, self.region_hits.double() / n_b.clamp(min=1), torch.ones_like(n_b))

    def f_score(self) -> torch.Tensor:
        """float64 ``[..., T, R, W]``: the boundary F-measure ``2 P R / (P + R)``, 0 when ``P + R = 0``."""
        p, r = self.precision(), self.recall()
        s = p + r
        return torch.where(s > 0, 2 * p * r / torch.where(s > 0, s, torch.ones_like(s)), torch.zeros_like(s))

    def hausdorff(self) -> torch.Tensor:
        """float64 ``[..., R, W]``: the Hausdorff distance between the boundaries, ``sqrt`` of the larger ``max_d2``;
        NaN when either boundary is empty."""
        m = self.max_d2.max(-1).values
        return torch.where(m >= 0, m.clamp(min=0).double().sqrt(), torch.full_like(m, float('nan'), dtype=torch.float64))

    def assd(self) -> torch.Tensor:
        """float64 ``[..., R, W]``: the average symmetric surface distance, both directions' sums of distances over
        ``|dA| + |dB|``; NaN when either boundary is empty."""
        n_a, n_b = self._sizes()
        n_a, n_b = torch.broadcast_tensors(n_a, n_b)
        both = (n_a > 0) & (n_b > 0)
        return torch.where(both, self.sum_dist.sum(-1) / (n_a + n_b).clamp(min=1),
                           torch.full_like(n_a, float('nan')))


def _boundary_tolerances(tolerances, out_h: int, out_w: int, what: str) -> List[float]:
    """``tolerances`` (a sequence of numbers or a 1-D CPU tensor; ``None``: DAVIS's ``ceil(0.008 * diagonal)``) rounded
    to fp32, as the Python floats of those fp32 values; a ``ValueError`` unless they are 1 to 16 finite values ``>= 0``,
    strictly ascending after the rounding."""
    if tolerances is None:
        return [float(math.ceil(0.008 * math.hypot(out_h, out_w)))]
    if isinstance(tolerances, torch.Tensor):
        if tolerances.device.type != 'cpu' or tolerances.dim() != 1 or tolerances.dtype == torch.bool \
                or tolerances.is_complex():
            raise ValueError(f'{what}: tolerances must be a 1-D real CPU tensor, not {tolerances.dim()}-D '
                             f'{tolerances.dtype} on {tolerances.device}')
        tol = tolerances.detach().to(torch.float32)
    else:
        try:
            values = list(tolerances)
        except TypeError:
            raise ValueError(f'{what}: tolerances must be a sequence of numbers, not {tolerances!r}') from None
        if not all(isinstance(x, numbers.Real) and not isinstance(x, bool) for x in values):
            raise ValueError(f'{what}: tolerances must be numbers, not {values!r}')
        tol = torch.tensor([float(x) for x in values], dtype=torch.float64).to(torch.float32)
    n = tol.numel()
    if not 1 <= n <= _native.BOUNDARY_MAX_TOLERANCES:
        raise ValueError(f'{what}: {n} tolerances; a call takes 1 to {_native.BOUNDARY_MAX_TOLERANCES}')
    if not bool((torch.isfinite(tol) & (tol >= 0)).all()):
        raise ValueError(f'{what}: tolerances must be finite and >= 0 in fp32, not {tol.tolist()}')
    if not bool((tol[1:] > tol[:-1]).all()):
        raise ValueError(f'{what}: tolerances must be strictly ascending after rounding to fp32, not {tol.tolist()}')
    return tol.tolist()


def _boundary_outputs(lead: Tuple[int, ...], n_regions: int, n_words: int, n_tol: int, tol: List[float], dev,
                      new=torch.empty) -> RegionBoundary:
    """The buffers of a :class:`RegionBoundary` with leading axes ``lead`` (``new``: ``torch.zeros`` for a call that
    launches nothing)."""
    i32 = dict(dtype=torch.int32, device=dev)
    return RegionBoundary(new((*lead, n_words), **i32), new((n_regions,), **i32),
                          new((*lead, n_tol, n_regions, n_words), **i32), new((*lead, n_tol, n_regions, n_words), **i32),
                          new((*lead, n_regions, n_words, 2), dtype=torch.int64, device=dev),
                          new((*lead, n_regions, n_words, 2), dtype=torch.float64, device=dev),
                          torch.tensor(tol, dtype=torch.float32, device=dev))


def _boundary_scratch(n_regions: int, n_planes: int, out_h: int, out_w: int, dev) -> torch.Tensor:
    """:data:`REGION_BOUNDARY_SCRATCH_BYTES` clipped to the planes the call has, at least the regions and one plane."""
    n_bytes = max(_native.boundary_scratch_bytes(n_regions, 1, out_h, out_w),
                  min(REGION_BOUNDARY_SCRATCH_BYTES, _native.boundary_scratch_bytes(n_regions, n_planes, out_h, out_w)))
    return torch.empty(n_bytes, dtype=torch.uint8, device=dev)


def _boundary_pointers(b: RegionBoundary):
    return (b.word_boundary.data_ptr(), b.region_boundary.data_ptr(), b.word_hits.data_ptr(), b.region_hits.data_ptr(),
            b.max_d2.data_ptr(), b.sum_dist.data_ptr())


def _region_boundary(tokenizer, prompt: str, maps: torch.Tensor, words, image, regions, threshold, tolerances,
                     absolute, word_idx, offset_idx: int, to_cpu: bool, what: str):
    """``daam_region_boundary`` over ``maps`` ``[n_maps, n_rows, xh, xw]``: returns ``(wl, boundary)``, the
    :class:`_WordList` and the :class:`RegionBoundary` with a leading map axis. Checks as ``_region_overlap``, in its
    order, then the threshold (set, truthy and finite) and the tolerances. Scratch: :func:`_boundary_scratch`."""
    wl = _WordList(tokenizer, prompt, maps, words, word_idx, offset_idx, image, absolute, threshold, to_cpu, what)
    n_maps, out_h, out_w, dev = wl.n_maps, wl.out_h, wl.out_w, wl.dev
    region_bytes = _region_bytes(wl, regions, what)
    if not threshold:
        raise ValueError(f'{what}: threshold must be set (truthy), not {threshold!r}: the word masks are the masks '
                         f'expand_words(..., threshold) returns')
    if not math.isfinite(float(threshold)):
        raise ValueError(f'{what}: threshold must be finite, not {threshold!r}')
    tol = _boundary_tolerances(tolerances, out_h, out_w, what)
    n_regions, n_words = region_bytes.shape[0], len(wl.words)
    if wl.empty or n_regions == 0:            # no word is scored: the call returns no word heat maps
        _no_region_overlap(wl, (), n_regions)
        return wl.done(_boundary_outputs((n_maps,), n_regions, 0, len(tol), tol, dev, torch.zeros))
    out = _boundary_outputs((n_maps,), n_regions, n_words, len(tol), tol, dev)
    scratch = _boundary_scratch(n_regions, n_maps * n_words, out_h, out_w, dev)
    wl.launch(_native.region_boundary, tol, wl.word_maps.data_ptr(), region_bytes.data_ptr(), n_regions,
              *_boundary_pointers(out), scratch.data_ptr(), scratch.numel())
    return wl.done(out)


@dataclass
class WordOverlap:
    """Sums of products of word maps (:meth:`GlobalHeatMap.word_overlap`): ``intersection`` ``[..., W, W]``
    (``sum_p m[a](p) * m[b](p)``, symmetric) and ``word_area`` ``[..., W]`` (``sum_p m[a](p)``), fp32. ``...`` is the
    map axis of a :class:`GlobalHeatMapStack`, absent for one map. The scores are the reference's formulas
    (``daam/evaluate.py``) in the same fp32 operation order."""
    intersection: torch.Tensor
    word_area: torch.Tensor

    def map(self, i: int) -> 'WordOverlap':
        """The overlap of map ``i`` of a stack."""
        return WordOverlap(self.intersection[i], self.word_area[i])

    def cpu(self) -> 'WordOverlap':
        return WordOverlap(self.intersection.cpu(), self.word_area.cpu())

    def iou(self) -> torch.Tensor:
        """``[a, b] = I / (A[a] + A[b] - I + 1e-8)``: ``compute_iou(mask_a, mask_b)`` of every pair (and the DAAM
        notebook's ``iou``, exact while ``A[a] + A[b]`` is below 2**24), symmetric."""
        i, a = self.intersection, self.word_area
        return i / (a.unsqueeze(-1) + a.unsqueeze(-2) - i + 1e-8)

    def ioa(self) -> torch.Tensor:
        """``[a, b] = I / (A[a] + 1e-8)``: ``compute_ioa(mask_a, mask_b)``, the share of word ``a`` inside word ``b``
        (0 for an empty word, as the DAAM notebook's ``ioa``)."""
        return self.intersection / (self.word_area.unsqueeze(-1) + 1e-8)


@dataclass
class RelationOverlap:
    """Head / dependent overlap of the relations of a parse (:meth:`GlobalHeatMap.relation_overlap`): the kept
    ``relations`` ``(head, dep, rel)`` and their indices ``kept`` in the input, the distinct endpoints ``words`` (as
    given) and their :class:`WordOverlap`, and per kept edge ``iou``, ``iod`` (the share of the dependent inside the
    head) and ``ioh`` (the share of the head inside the dependent), each ``[..., E]``."""
    relations: List[Tuple]
    kept: List[int]
    words: List[Union[str, int]]
    overlap: 'WordOverlap'
    iou: torch.Tensor
    iod: torch.Tensor
    ioh: torch.Tensor

    def map(self, i: int) -> 'RelationOverlap':
        """The overlap of map ``i`` of a stack."""
        return RelationOverlap(self.relations, self.kept, self.words, self.overlap.map(i), self.iou[i], self.iod[i],
                               self.ioh[i])


def _word_overlap(tokenizer, prompt: str, maps: torch.Tensor, words, image, absolute, threshold, word_idx,
                  offset_idx: int, to_cpu: bool, what: str):
    """``daam_word_overlap`` over ``maps`` ``[n_maps, n_rows, xh, xw]``: returns ``(wl, overlap)``, the
    :class:`_WordList` and the :class:`WordOverlap` with a leading map axis. ``image=None``: the sums run over the
    heat-map grid."""
    wl = _WordList(tokenizer, prompt, maps, words, word_idx, offset_idx, image, absolute, threshold, to_cpu, what,
                   on_grid=image is None)
    n_maps, n, dev = wl.n_maps, len(wl.words), wl.dev
    if wl.empty:
        return wl.done(WordOverlap(torch.zeros((n_maps, n, n), device=dev), torch.zeros((n_maps, n), device=dev)))
    inter = torch.empty((n_maps, n, n), dtype=torch.float32, device=dev)
    area = torch.empty((n_maps, n), dtype=torch.float32, device=dev)
    scratch = wl.scratch(_native.word_overlap_scratch_floats(n_maps, n, wl.out_h, wl.out_w))
    wl.launch(_native.word_overlap, wl.word_maps.data_ptr(), inter.data_ptr(), area.data_ptr(), scratch.data_ptr())
    return wl.done(WordOverlap(inter, area))


def _relation_overlap(tokenizer, prompt: str, maps: torch.Tensor, relations, image, absolute, threshold,
                      offset_idx: int, to_cpu: bool, what: str) -> RelationOverlap:
    """``relation_overlap`` over ``maps`` ``[n_maps, n_rows, xh, xw]``: the distinct endpoints of the edges whose words
    are in the prompt -- one endpoint per row set, so a word given twice, in another case, or as its token index is
    measured once -- then one ``_word_overlap`` call and a gather (on the host when ``to_cpu``); every tensor has a
    leading map axis."""
    kept_edges, kept, words, word_idx, ends = [], [], [], [], []
    slot: Dict[Tuple[int, ...], int] = {}
    for e, edge in enumerate(relations):
        head, dep, _ = edge
        try:
            pair = [compute_token_merge_indices(tokenizer, prompt, x, None, offset_idx)[0]
                    if isinstance(x, str) else [int(x) + 1] for x in (head, dep)]
        except ValueError:          # a word not in the prompt: the reference's ``except ValueError: pass``
            continue
        idx = []
        for x, rows in zip((head, dep), pair):
            key = tuple(rows)
            if key not in slot:
                slot[key] = len(words)
                words.append(x)
                word_idx.append(None if isinstance(x, str) else int(x))
            idx.append(slot[key])
        kept_edges.append(tuple(edge))
        kept.append(e)
        ends.append(idx)
    if len(words) > _native.MAX_SEGMENT_WORDS:
        raise ValueError(f'{what}: {len(words)} distinct endpoints > {_native.MAX_SEGMENT_WORDS}, the word limit of '
                         f'one word_overlap call')
    labels = [x if isinstance(x, str) else str(x) for x in words]
    _, ov = _word_overlap(tokenizer, prompt, maps, labels, image, absolute, threshold, word_idx, offset_idx, to_cpu,
                          what)
    dev = ov.intersection.device
    h = torch.tensor([i for i, _ in ends], dtype=torch.long, device=dev)
    d = torch.tensor([j for _, j in ends], dtype=torch.long, device=dev)
    iou, ioa = ov.iou(), ov.ioa()
    return RelationOverlap(kept_edges, kept, words, ov, iou[..., h, d], ioa[..., d, h], ioa[..., h, d])


# Scratch of one word_instances call: as many (map, word) planes as fit are labelled per round, so memory does not grow
# with the number of maps (a 50-step, 24-word SDXL history would take about 25 GB at once).
WORD_INSTANCES_SCRATCH_BYTES = 256 << 20


@dataclass
class WordInstances:
    """Connected components of word masks (:meth:`GlobalHeatMap.word_instances`), the largest ``K`` per word, sorted by
    area (largest first, ties to the first pixel in raster order): ``count`` int32 ``[..., W]`` (every component, not
    capped at ``K``), ``area`` int32 ``[..., W, K]``, ``box`` int32 ``[..., W, K, 4]`` (``(y0, x0, y1, x1)``, half-open),
    ``sum_yx`` int64 ``[..., W, K, 2]`` (sums of the row and column indices of the pixels), ``peak`` fp32 ``[..., W, K]``
    (the max of the expanded map over the component) and ``peak_yx`` int32 ``[..., W, K, 2]`` (the first pixel where it
    is reached). Slots past ``count`` are 0. ``...`` is the map axis of a :class:`GlobalHeatMapStack`, absent for one
    map. The helpers are plain torch on the fields' device."""
    count: torch.Tensor
    area: torch.Tensor
    box: torch.Tensor
    sum_yx: torch.Tensor
    peak: torch.Tensor
    peak_yx: torch.Tensor

    def map(self, i: int) -> 'WordInstances':
        """The instances of map ``i`` of a stack."""
        return WordInstances(*(getattr(self, f)[i] for f in _INSTANCE_FIELDS))

    def cpu(self) -> 'WordInstances':
        return WordInstances(*(getattr(self, f).cpu() for f in _INSTANCE_FIELDS))

    def centroid(self) -> torch.Tensor:
        """float64 ``[..., W, K, 2]``: ``sum_yx / area``, the mean row and column of each instance; NaN for empty
        slots."""
        area = self.area.double().unsqueeze(-1)
        return torch.where(area > 0, self.sum_yx.double() / area.clamp(min=1), torch.full_like(area, float('nan')))

    def largest_box(self) -> torch.Tensor:
        """int32 ``[..., W, 4]``: the box of each word's largest instance (zeros for a word with none)."""
        return self.box[..., 0, :]

    def box_iou(self, boxes) -> torch.Tensor:
        """float64 ``[..., W, B]``: IoU of each word's largest box against half-open ``(y0, x0, y1, x1)`` boxes ``[B,
        4]`` (e.g. ground-truth boxes), 0 for a word without an instance."""
        lb = self.largest_box().double().unsqueeze(-2)                     # [..., W, 1, 4]
        gt = torch.as_tensor(boxes, dtype=torch.float64, device=lb.device).reshape(-1, 4)
        ih = (torch.minimum(lb[..., 2], gt[:, 2]) - torch.maximum(lb[..., 0], gt[:, 0])).clamp(min=0)
        iw = (torch.minimum(lb[..., 3], gt[:, 3]) - torch.maximum(lb[..., 1], gt[:, 1])).clamp(min=0)
        inter = ih * iw
        a = (lb[..., 2] - lb[..., 0]) * (lb[..., 3] - lb[..., 1])
        b = (gt[:, 2] - gt[:, 0]) * (gt[:, 3] - gt[:, 1])
        union = a + b - inter
        has = (self.area[..., 0] > 0).unsqueeze(-1)
        return torch.where(has & (union > 0), inter / union.clamp(min=1e-300), torch.zeros_like(inter))


_INSTANCE_FIELDS = ('count', 'area', 'box', 'sum_yx', 'peak', 'peak_yx')


def _word_instances(tokenizer, prompt: str, maps: torch.Tensor, words, image, threshold, absolute, max_instances: int,
                    word_idx, offset_idx: int, to_cpu: bool, what: str):
    """``daam_word_instances`` over ``maps`` ``[n_maps, n_rows, xh, xw]``: returns ``(wl, instances)``, the
    :class:`_WordList` and the :class:`WordInstances` with a leading map axis. Scratch:
    :data:`WORD_INSTANCES_SCRATCH_BYTES`, clipped to the planes the call has, at least one plane."""
    words = list(words)
    if not threshold:
        raise ValueError(f'{what}: threshold must be set (truthy), not {threshold!r}: the instances are the connected '
                         f'components of the mask expand_words(..., threshold) returns')
    if isinstance(max_instances, bool) or not isinstance(max_instances, int) \
            or not 1 <= max_instances <= _native.WORD_INSTANCES_MAX:
        raise ValueError(f'{what}: max_instances must be an int in [1, {_native.WORD_INSTANCES_MAX}], not '
                         f'{max_instances!r}')
    if len(words) > _native.MAX_SEGMENT_WORDS:
        raise ValueError(f'{what}: {len(words)} words > {_native.MAX_SEGMENT_WORDS}, the word limit of one call')
    wl = _WordList(tokenizer, prompt, maps, words, word_idx, offset_idx, image, absolute, threshold, to_cpu, what)
    n_maps, dev = wl.n_maps, wl.dev
    n, k = len(words), max_instances
    new = torch.zeros if wl.empty else torch.empty     # the kernels write every slot
    i32 = dict(dtype=torch.int32, device=dev)
    inst = WordInstances(new((n_maps, n), **i32), new((n_maps, n, k), **i32), new((n_maps, n, k, 4), **i32),
                         new((n_maps, n, k, 2), dtype=torch.int64, device=dev),
                         new((n_maps, n, k), dtype=torch.float32, device=dev), new((n_maps, n, k, 2), **i32))
    if not wl.empty:
        plane = _native.word_instances_plane_bytes(wl.out_h, wl.out_w)
        n_bytes = max(plane, min(WORD_INSTANCES_SCRATCH_BYTES, plane * n_maps * n))
        scratch = torch.empty(n_bytes, dtype=torch.uint8, device=dev)
        wl.launch(_native.word_instances, k, wl.word_maps.data_ptr(),
                  *(getattr(inst, f).data_ptr() for f in _INSTANCE_FIELDS), scratch.data_ptr(), n_bytes)
    return wl.done(inst)


# Scratch of one word_distance call: as many (map, word) planes as fit are transformed per round, so memory does not
# grow with the number of maps.
WORD_DISTANCE_SCRATCH_BYTES = 256 << 20


def _real(v, what: str, name: str) -> float:
    """``v`` as a Python float; a ``ValueError`` unless it is a finite real number."""
    if isinstance(v, bool) or not isinstance(v, numbers.Real) or not math.isfinite(float(v)):
        raise ValueError(f'{what}: {name} must be a finite number, not {v!r}')
    return float(v)


@dataclass
class WordDistance:
    """Signed distance maps of masks (:meth:`GlobalHeatMap.word_distance`,
    :func:`daam_b200.evaluate.distance_transform`): ``signed_d2`` int32 ``[..., W, H, W']``, with ``M`` a mask and
    ``d2`` the squared Euclidean distance between pixel centres, ``min d2`` to ``M`` (``>= 1``) at a pixel outside
    ``M`` and ``-min d2`` to the pixels outside ``M`` (``<= -1``, the image border not counted as outside) at a pixel
    of ``M``; every pixel is ``+DISTANCE_NONE`` (``2**31 - 1``) for an empty mask and ``-DISTANCE_NONE`` for a full
    one. ``...`` is the map axis of a :class:`GlobalHeatMapStack`, absent for one map. The helpers are plain torch on
    the field's device; the sentinels count as infinitely far."""
    signed_d2: torch.Tensor

    NONE = _native.DISTANCE_NONE

    def map(self, i: int) -> 'WordDistance':
        """The distances of map ``i`` of a stack."""
        return WordDistance(self.signed_d2[i])

    def cpu(self) -> 'WordDistance':
        return WordDistance(self.signed_d2.cpu())

    def _signed(self) -> torch.Tensor:
        """float64 signed distance ``sign * sqrt(|d2|)``, ``+-inf`` for the sentinels."""
        d2 = self.signed_d2
        s = d2.double().abs().sqrt().copysign(d2.double())
        return torch.where(d2.abs() == self.NONE, d2.double().sign() * math.inf, s)

    def distance(self) -> torch.Tensor:
        """fp32 ``[..., W, H, W']``: the signed Euclidean distance, ``sqrt(d2)`` outside the mask and ``-sqrt(d2)``
        inside, taken in float64 and rounded once; ``+inf`` for an empty mask, ``-inf`` for a full one."""
        return self._signed().float()

    def mask(self, grow: float = 0.0) -> torch.Tensor:
        """bool ``[..., W, H, W']``: the mask grown by ``grow`` pixels. ``grow >= 0``: ``signed_d2 <= grow**2``, the
        binary dilation by the disk ``{dy**2 + dx**2 <= grow**2}`` (``grow = 0`` is the mask itself); ``grow < 0``:
        ``signed_d2 < -grow**2``, the binary erosion by that disk with the image border counted as inside. The
        comparison runs in float64. ``distance_transform(wd.mask(r)).mask(-r)`` is the closing by the disk."""
        g = _real(grow, 'WordDistance.mask', 'grow')
        d = torch.where(self.signed_d2.abs() == self.NONE, self.signed_d2.double().sign() * math.inf,
                        self.signed_d2.double())
        return d <= g * g if g >= 0 else d < -(g * g)

    def soft_mask(self, grow: float = 0.0, *, feather: float) -> torch.Tensor:
        """fp32 ``[..., W, H, W']``: ``clamp((grow + feather - s) / feather, 0, 1)`` with ``s`` the float64 signed
        distance, rounded once: 1 inside the mask grown by ``grow`` pixels, falling linearly to 0 over ``feather``
        pixels beyond it -- an inpainting mask with a soft edge. ``feather`` must be finite and > 0."""
        g = _real(grow, 'WordDistance.soft_mask', 'grow')
        f = _real(feather, 'WordDistance.soft_mask', 'feather')
        if not f > 0:
            raise ValueError(f'WordDistance.soft_mask: feather must be > 0, not {feather!r}')
        return ((g + f - self._signed()) / f).clamp(0, 1).float()


def _distance_size(out_h: int, out_w: int, what: str):
    """A ``ValueError`` unless ``out_h, out_w <= 32767`` and ``out_h * out_w <= 2**24``."""
    if out_h > _native.DISTANCE_MAX_SIDE or out_w > _native.DISTANCE_MAX_SIDE:
        raise ValueError(f'{what}: a {out_h} x {out_w} image has a side > {_native.DISTANCE_MAX_SIDE}')
    if out_h * out_w > 1 << 24:
        raise ValueError(f'{what}: a {out_h} x {out_w} image is more than 2**24 pixels')


def _word_distance(tokenizer, prompt: str, maps: torch.Tensor, words, image, threshold, absolute, word_idx,
                   offset_idx: int, to_cpu: bool, what: str):
    """``daam_word_distance`` over ``maps`` ``[n_maps, n_rows, xh, xw]``: returns ``(wl, distance)``, the
    :class:`_WordList` and the :class:`WordDistance` with a leading map axis. Checks as ``_word_instances``, in its
    order (the threshold set and finite), then the image size. Scratch: :data:`WORD_DISTANCE_SCRATCH_BYTES`, clipped
    to the planes the call has, at least one plane."""
    words = list(words)
    if not threshold:
        raise ValueError(f'{what}: threshold must be set (truthy), not {threshold!r}: the distances are those of the '
                         f'mask expand_words(..., threshold) returns')
    if not math.isfinite(float(threshold)):
        raise ValueError(f'{what}: threshold must be finite, not {threshold!r}')
    if len(words) > _native.MAX_SEGMENT_WORDS:
        raise ValueError(f'{what}: {len(words)} words > {_native.MAX_SEGMENT_WORDS}, the word limit of one call')
    wl = _WordList(tokenizer, prompt, maps, words, word_idx, offset_idx, image, absolute, threshold, to_cpu, what)
    out_h, out_w = wl.out_h, wl.out_w
    _distance_size(out_h, out_w, what)
    shape = (wl.n_maps, len(words), out_h, out_w)
    if wl.empty or out_h * out_w == 0:
        return wl.done(WordDistance(torch.zeros(shape, dtype=torch.int32, device=wl.dev)))
    out = WordDistance(torch.empty(shape, dtype=torch.int32, device=wl.dev))
    plane = _native.distance_plane_bytes(out_h, out_w)
    n_bytes = max(plane, min(WORD_DISTANCE_SCRATCH_BYTES, plane * wl.n_maps * len(words)))
    scratch = torch.empty(n_bytes, dtype=torch.uint8, device=wl.dev)
    wl.launch(_native.word_distance, wl.word_maps.data_ptr(), out.signed_d2.data_ptr(), scratch.data_ptr(), n_bytes)
    return wl.done(out)


def jet_colormap() -> torch.Tensor:
    """The fp32 ``[256, 3]`` table the overlay kernel colours with: ``L[k] = 255 * jet(k / 255)``, matplotlib's ``jet``
    segment data evaluated in float64 and rounded once to fp32 (``L[0] = (0, 0, 127.5)``, ``L[255] = (127.5, 0, 0)``)."""
    return _native.jet_colormap()


def _overlay_image(image, n_maps: int, grid, dev, what: str, stack: bool):
    """``(image, out_h, out_w, per_map)``: ``image`` as a uint8 ``[H, W, 3]`` or, for a stack, ``[n_maps, H, W, 3]``
    tensor (not yet on the device), and the size the maps expand to over it."""
    if isinstance(image, torch.Tensor):
        arr = image
    elif hasattr(image, 'convert') and hasattr(image, 'size'):           # PIL
        import numpy as np
        arr = torch.from_numpy(np.array(image.convert('RGB')))
    elif hasattr(image, '__array_interface__'):                          # numpy
        import numpy as np
        arr = torch.from_numpy(np.ascontiguousarray(image))
    else:
        raise TypeError(f'{what}: image must be a PIL image or a uint8 [H, W, 3] numpy / torch array, not '
                        f'{type(image).__name__}')
    if arr.dtype != torch.uint8:
        raise TypeError(f'{what}: image must be uint8, not {arr.dtype}')
    if arr.device.type != 'cpu' and arr.device != dev:
        raise ValueError(f'{what}: image is on {arr.device}, the heat maps on {dev}')
    per_map = stack and arr.dim() == 4
    if arr.dim() not in ((3, 4) if stack else (3,)) or (per_map and arr.shape[0] != n_maps):
        want = f'[{n_maps}, H, W, 3] or [H, W, 3]' if stack else '[H, W, 3]'
        raise ValueError(f'{what}: an image of shape {tuple(arr.shape)} is not {want}')
    h, w = int(arr.shape[-3]), int(arr.shape[-2])
    out_h, out_w = _image_size(SimpleNamespace(size=(w, h), height=h, width=w), *grid)
    if tuple(arr.shape[-3:]) != (out_h, out_w, 3):
        raise ValueError(f'{what}: an image of shape {tuple(arr.shape)} does not match the expanded maps\' '
                         f'({out_h}, {out_w}, 3)' + (' (a square map keeps the reference\'s (size[0], size[1]) order, '
                                                      'which transposes a non-square image)' if h != w else ''))
    return arr, out_h, out_w, per_map


def _overlay(tokenizer, prompt: str, maps: torch.Tensor, words, image, absolute, threshold, color_normalize, word_idx,
             offset_idx: int, to_cpu: bool, what: str, stack: bool):
    """``daam_overlay_words`` over ``maps`` ``[n_maps, n_rows, xh, xw]``: returns ``(wl, frames)``, the
    :class:`_WordList` and ``frames`` uint8 ``[n_maps, len(words), H, W, 3]``. The image fixes the size the maps
    expand to."""
    wl = _WordList(tokenizer, prompt, maps, words, word_idx, offset_idx, None, absolute, threshold, to_cpu, what,
                   on_grid=True)         # the size is the image's, once _overlay_image has checked it
    n_maps, n_words, dev = wl.n_maps, len(wl.words), wl.dev
    image, wl.out_h, wl.out_w, per_map = _overlay_image(image, n_maps, wl.grid, dev, what, stack)
    shape = (n_maps, n_words, wl.out_h, wl.out_w, 3)
    if wl.empty:
        return wl.done(torch.empty(shape, dtype=torch.uint8, device=dev))
    image = image.to(dev).contiguous()                   # one copy to the device
    # the kernel writes whole 4-byte words: the frames are a view of a buffer rounded up to them
    buf = torch.empty(_native.overlay_frames_bytes(*shape[:4]), dtype=torch.uint8, device=dev)
    frames = buf[:n_maps * n_words * wl.out_h * wl.out_w * 3].view(shape)
    scratch = wl.scratch(_native.segment_scratch_floats(n_maps, n_words))
    wl.launch(_native.overlay_words, color_normalize, wl.word_maps.data_ptr(), image.data_ptr(),
              wl.out_h * wl.out_w * 3 if per_map else 0, buf.data_ptr(), scratch.data_ptr())
    return wl.done(frames)


# Scratch of one refine_words call: the image statistics (36 bytes a pixel, per image) and as many (map, word) planes
# as fit (32 bytes a pixel each) go in a round, so memory does not grow with the number of maps; one image and one
# plane larger than the budget go alone.
REFINE_SCRATCH_BYTES = 256 << 20


def _refine_args(radius, eps, what: str):
    """Raises ``ValueError`` unless ``radius`` is an integer in ``[1, 64]`` and ``eps``, rounded to fp32, is finite
    and > 0."""
    if isinstance(radius, bool) or not isinstance(radius, int) or not 1 <= radius <= _native.REFINE_MAX_RADIUS:
        raise ValueError(f'{what}: radius must be an integer in [1, {_native.REFINE_MAX_RADIUS}], not {radius!r}')
    e32 = ctypes.c_float(float(eps)).value
    if not (math.isfinite(e32) and e32 > 0):
        raise ValueError(f'{what}: eps must be finite and > 0 in fp32, not {eps!r}')


def _refine(tokenizer, prompt: str, maps: torch.Tensor, words, image, radius, eps, absolute, threshold, word_idx,
            offset_idx: int, to_cpu: bool, what: str, stack: bool):
    """``daam_refine_words`` over ``maps`` ``[n_maps, n_rows, xh, xw]``: returns ``(wl, refined)``, the
    :class:`_WordList` and ``refined`` fp32 ``[n_maps, len(words), H, W]``. Checks as :func:`_overlay`, in its order,
    then ``radius`` and ``eps``. Scratch: :data:`REFINE_SCRATCH_BYTES`, clipped to what the call has, at least one
    image and one plane."""
    wl = _WordList(tokenizer, prompt, maps, words, word_idx, offset_idx, None, absolute, threshold, to_cpu, what,
                   on_grid=True)         # the size is the image's, once _overlay_image has checked it
    n_maps, n_words, dev = wl.n_maps, len(wl.words), wl.dev
    image, wl.out_h, wl.out_w, per_map = _overlay_image(image, n_maps, wl.grid, dev, what, stack)
    _refine_args(radius, eps, what)
    refined = torch.empty((n_maps, n_words, wl.out_h, wl.out_w), dtype=torch.float32, device=dev)
    if wl.empty:
        return wl.done(refined)
    image = image.to(dev).contiguous()                   # one copy to the device
    n_bytes = max(_native.refine_scratch_bytes(1, 1, wl.out_h, wl.out_w),
                  min(REFINE_SCRATCH_BYTES, _native.refine_scratch_bytes(n_maps if per_map else 1, n_maps * n_words,
                                                                         wl.out_h, wl.out_w)))
    scratch = torch.empty(n_bytes, dtype=torch.uint8, device=dev)
    wl.launch(_native.refine_words, radius, eps, wl.word_maps.data_ptr(), image.data_ptr(),
              wl.out_h * wl.out_w * 3 if per_map else 0, refined.data_ptr(), scratch.data_ptr(), n_bytes)
    return wl.done(refined)


# Scratch of one segment_crf call: two fp32 Q buffers per map (8 bytes a pixel per label) and the min / max partials;
# as many whole maps as fit go in a round, so memory does not grow with the number of maps; one map larger than the
# budget goes alone.
CRF_SCRATCH_BYTES = 256 << 20


def _crf_args(threshold, iterations, radius, scale, appearance, sigma_xy, sigma_rgb, smoothness, sigma_smooth,
              what: str):
    """Raises ``ValueError`` unless ``radius`` is an integer in ``[1, 16]``, ``iterations`` one in ``[0, 64]``, and,
    rounded to fp32, ``scale`` and the sigmas are finite and > 0, ``appearance`` and ``smoothness`` finite and >= 0,
    and a threshold in effect finite -- daam_segment_crf's checks, in its order."""
    def whole(v, lo, hi, name):
        if isinstance(v, bool) or not isinstance(v, int) or not lo <= v <= hi:
            raise ValueError(f'{what}: {name} must be an integer in [{lo}, {hi}], not {v!r}')

    def f32(v, name):
        try:
            return ctypes.c_float(float(v)).value
        except (TypeError, ValueError):
            raise ValueError(f'{what}: {name} must be a number, not {v!r}') from None

    whole(radius, 1, _native.CRF_MAX_RADIUS, 'radius')
    whole(iterations, 0, _native.CRF_MAX_ITERATIONS, 'iterations')
    for name, v in (('scale', scale), ('sigma_xy', sigma_xy), ('sigma_rgb', sigma_rgb), ('sigma_smooth', sigma_smooth)):
        v32 = f32(v, name)
        if not (math.isfinite(v32) and v32 > 0):
            raise ValueError(f'{what}: {name} must be finite and > 0 in fp32, not {v!r}')
    for name, v in (('appearance', appearance), ('smoothness', smoothness)):
        v32 = f32(v, name)
        if not (math.isfinite(v32) and v32 >= 0):
            raise ValueError(f'{what}: {name} must be finite and >= 0 in fp32, not {v!r}')
    if threshold and not math.isfinite(f32(threshold, 'threshold')):
        raise ValueError(f'{what}: threshold must be finite in fp32, not {threshold!r}')


def _segment_crf(tokenizer, prompt: str, maps: torch.Tensor, words, image, threshold, iterations, radius, scale,
                 appearance, sigma_xy, sigma_rgb, smoothness, sigma_smooth, absolute, word_idx, offset_idx: int,
                 probs: bool, to_cpu: bool, what: str, stack: bool):
    """``daam_segment_crf`` over ``maps`` ``[n_maps, n_rows, xh, xw]``: returns ``(wl, labels, scores)``, plus
    ``probs`` fp32 ``[n_maps, L, H, W]`` when asked; ``labels`` uint8 and ``scores`` fp32 ``[n_maps, H, W]``. Checks as
    :func:`_overlay`, in its order, then the CRF arguments (:func:`_crf_args`). Scratch: :data:`CRF_SCRATCH_BYTES`,
    clipped to what the call has, at least one map."""
    wl = _WordList(tokenizer, prompt, maps, words, word_idx, offset_idx, None, absolute, threshold, to_cpu, what,
                   on_grid=True)         # the size is the image's, once _overlay_image has checked it
    n_maps, n_words, dev = wl.n_maps, len(wl.words), wl.dev
    image, wl.out_h, wl.out_w, per_map = _overlay_image(image, n_maps, wl.grid, dev, what, stack)
    _crf_args(threshold, iterations, radius, scale, appearance, sigma_xy, sigma_rgb, smoothness, sigma_smooth, what)
    n_labels = n_words + (1 if threshold else 0)
    shape = (n_maps, wl.out_h, wl.out_w)
    labels = torch.zeros(shape, dtype=torch.uint8, device=dev)
    scores = torch.empty(shape, dtype=torch.float32, device=dev)
    q = torch.empty((n_maps, n_labels, wl.out_h, wl.out_w), dtype=torch.float32, device=dev) if probs else None
    if wl.empty:                         # only the background, if any: it takes every pixel with Q = 1
        scores.fill_(1.0 if n_labels else 0.0)
        if q is not None:
            q.fill_(1.0)
        return wl.done(labels, scores, *([q] if probs else []))
    image = image.to(dev).contiguous()                   # one copy to the device
    n_bytes = max(_native.crf_scratch_bytes(1, n_labels, wl.out_h, wl.out_w),
                  min(CRF_SCRATCH_BYTES, _native.crf_scratch_bytes(n_maps, n_labels, wl.out_h, wl.out_w)))
    scratch = torch.empty(n_bytes, dtype=torch.uint8, device=dev)
    wl.launch(_native.segment_crf, scale, iterations, radius, appearance, sigma_xy, sigma_rgb, smoothness,
              sigma_smooth, wl.word_maps.data_ptr(), image.data_ptr(), wl.out_h * wl.out_w * 3 if per_map else 0,
              labels.data_ptr(), scores.data_ptr(), q.data_ptr() if probs else 0, scratch.data_ptr(), n_bytes)
    return wl.done(labels, scores, *([q] if probs else []))


# Scratch of one segment_superpixels call: each image's SLIC state (96 bytes a cell) and each map's per-tile sums (8
# bytes per word and cell of a tile's box); as many whole maps as fit go in a round, so memory does not grow with the
# number of maps; one image and one map larger than the budget go alone.
SUPERPIXEL_SCRATCH_BYTES = 256 << 20


def _superpixel_args(out_h: int, out_w: int, n_segments, compactness, iterations, what: str):
    """Raises ``ValueError`` unless the image has at most 2**24 pixels, ``n_segments`` is an integer >= 1,
    ``compactness`` rounded to fp32 is finite and > 0 and ``iterations`` is an integer in ``[1, 64]`` -- the superpixel
    calls' checks, in their order. The cell limit (:func:`_superpixel_grid`) comes next."""
    if out_h * out_w > 1 << 24:
        raise ValueError(f'{what}: a {out_h} x {out_w} image is more than 2**24 pixels')
    if isinstance(n_segments, bool) or not isinstance(n_segments, int) or n_segments < 1:
        raise ValueError(f'{what}: n_segments must be an integer >= 1, not {n_segments!r}')
    try:
        c32 = ctypes.c_float(float(compactness)).value
    except (TypeError, ValueError):
        raise ValueError(f'{what}: compactness must be a number, not {compactness!r}') from None
    if not (math.isfinite(c32) and c32 > 0):
        raise ValueError(f'{what}: compactness must be finite and > 0 in fp32, not {compactness!r}')
    top = _native.SUPERPIXEL_MAX_ITERATIONS
    if isinstance(iterations, bool) or not isinstance(iterations, int) or not 1 <= iterations <= top:
        raise ValueError(f'{what}: iterations must be an integer in [1, {top}], not {iterations!r}')


def _superpixel_grid(out_h: int, out_w: int, n_segments: int, what: str):
    """``(ny, nx)``, the cell grid of an ``out_h x out_w`` image; ``ValueError`` beyond 65536 cells."""
    ny, nx = _native.superpixel_grid(out_h, out_w, n_segments)
    if ny * nx > _native.SUPERPIXEL_MAX_CELLS:
        raise ValueError(f'{what}: {n_segments} segments of a {out_h} x {out_w} image make a {ny} x {nx} grid, more '
                         f'than {_native.SUPERPIXEL_MAX_CELLS} cells')
    return ny, nx


def _image_superpixels(image: torch.Tensor, n_images: int, out_h: int, out_w: int, n_segments, compactness,
                       iterations, ny: int, nx: int) -> torch.Tensor:
    """``daam_image_superpixels`` of ``n_images`` device images back to back: int32 ``[n_images, out_h, out_w]``.
    Scratch: :data:`SUPERPIXEL_SCRATCH_BYTES`, clipped to what the call has, at least one image."""
    dev = image.device
    out = torch.empty((n_images, out_h, out_w), dtype=torch.int32, device=dev)
    one = _native.superpixel_image_bytes(ny, nx)
    n_bytes = max(one, min(SUPERPIXEL_SCRATCH_BYTES // one * one, n_images * one))
    scratch = torch.empty(n_bytes, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _native.image_superpixels(image.data_ptr(), n_images, out_h, out_w, n_segments, compactness, iterations,
                                  out.data_ptr(), scratch.data_ptr(), n_bytes, _stream_ptr(dev))
    return out


def _segment_superpixels(tokenizer, prompt: str, maps: torch.Tensor, words, image, n_segments, compactness,
                         iterations, threshold, absolute, word_idx, offset_idx: int, to_cpu: bool, what: str,
                         stack: bool):
    """``daam_segment_superpixels`` over ``maps`` ``[n_maps, n_rows, xh, xw]``: returns ``(wl, labels, scores,
    superpixels)``, ``labels`` uint8 and ``scores`` fp32 ``[n_maps, H, W]``, ``superpixels`` int32 ``[H, W]`` for one
    image or ``[n_maps, H, W]`` for one per map. Checks as :func:`_overlay`, in its order, then the superpixel
    arguments (:func:`_superpixel_args`, :func:`_superpixel_grid`). An empty word list still makes the partition."""
    wl = _WordList(tokenizer, prompt, maps, words, word_idx, offset_idx, None, absolute, threshold, to_cpu, what,
                   on_grid=True)         # the size is the image's, once _overlay_image has checked it
    n_maps, n_words, dev = wl.n_maps, len(wl.words), wl.dev
    image, wl.out_h, wl.out_w, per_map = _overlay_image(image, n_maps, wl.grid, dev, what, stack)
    h, w = wl.out_h, wl.out_w
    _superpixel_args(h, w, n_segments, compactness, iterations, what)
    ny, nx = _superpixel_grid(h, w, n_segments, what)
    shape = (n_maps, h, w)
    n_images = n_maps if per_map else 1
    if wl.empty:                         # no word: every pixel is background with score -inf, as segment
        sp = torch.empty((n_images, h, w), dtype=torch.int32, device=dev)
        if n_images:
            sp = _image_superpixels(image.to(dev).contiguous(), n_images, h, w, n_segments, compactness, iterations,
                                    ny, nx)
        return wl.done(torch.zeros(shape, dtype=torch.uint8, device=dev),
                       torch.full(shape, float('-inf'), device=dev), sp if per_map else sp[0])
    image = image.to(dev).contiguous()                   # one copy to the device
    labels = torch.empty(shape, dtype=torch.uint8, device=dev)
    scores = torch.empty(shape, dtype=torch.float32, device=dev)
    sp = torch.empty((n_images, h, w), dtype=torch.int32, device=dev)
    n_bytes = max(_native.superpixel_scratch_bytes(1, 1, n_words, ny, nx, h, w),
                  min(SUPERPIXEL_SCRATCH_BYTES,
                      _native.superpixel_scratch_bytes(n_images, n_maps, n_words, ny, nx, h, w)))
    scratch = torch.empty(n_bytes, dtype=torch.uint8, device=dev)
    wl.launch(_native.segment_superpixels, n_segments, compactness, iterations, wl.word_maps.data_ptr(),
              image.data_ptr(), h * w * 3 if per_map else 0, labels.data_ptr(), scores.data_ptr(), sp.data_ptr(),
              scratch.data_ptr(), n_bytes)
    return wl.done(labels, scores, sp if per_map else sp[0])


class GlobalHeatMapStack:
    """Global heat maps of one prompt's text stacked along a first axis: ``heat_maps[t]`` is one
    ``[n_rows, xh, xw]`` map. Base of :class:`TimeHeatMaps` (one map per step), :class:`ImageHeatMaps` (one per
    image), :class:`LayerHeatMaps`, :class:`FactorHeatMaps` and :class:`HeadHeatMaps` (one per layer, resolution or
    head)."""

    def __init__(self, tokenizer, prompt: str, heat_maps: torch.Tensor):
        self.tokenizer = tokenizer
        self.prompt = prompt
        self.heat_maps = heat_maps           # device fp32 [maps, n_rows, xh, xw]

    def __len__(self) -> int:
        return self.heat_maps.shape[0]

    def __getitem__(self, t: int) -> GlobalHeatMap:
        """Map ``t`` as a :class:`GlobalHeatMap` (``compute_word_heat_map``, ``expand_words``)."""
        return GlobalHeatMap(self.tokenizer, self.prompt, self.heat_maps[t])

    def word_heat_maps(self, word: str, word_idx: int = None, offset_idx: int = 0) -> torch.Tensor:
        """``[maps, xh, xw]``: row ``t`` is ``self[t].compute_word_heat_map(word, word_idx, offset_idx).heatmap``."""
        return _word_heat_map(self.tokenizer, self.prompt, self.heat_maps, word, word_idx, offset_idx,
                              f'{type(self).__name__}.word_heat_maps')[0]

    def segment(self, words, image, absolute: bool = False, threshold: Optional[float] = None, word_idx=None,
                offset_idx: int = 0, to_cpu: bool = True):
        """:meth:`GlobalHeatMap.segment` for every map in one call (two launches whatever the map count): returns
        ``(word_maps, labels, scores)`` with ``word_maps`` the device ``[maps, len(words), xh, xw]`` word heat maps and
        ``labels`` / ``scores`` ``[maps, H, W]``; row ``t`` equals ``self[t].segment(...)`` bit for bit (min / max
        normalisation per map and word)."""
        wl, labels, scores = _segment(self.tokenizer, self.prompt, self.heat_maps, words, image, absolute, threshold,
                                      word_idx, offset_idx, to_cpu, f'{type(self).__name__}.segment')
        return wl.word_maps, labels, scores

    def region_overlap(self, words, image, regions: torch.Tensor, absolute: bool = False,
                       threshold: Optional[float] = None, word_idx=None, offset_idx: int = 0, to_cpu: bool = True):
        """:meth:`GlobalHeatMap.region_overlap` for every map in one call (three launches whatever the map count):
        returns ``(word_maps, overlap)`` with ``word_maps`` the device ``[maps, len(words), xh, xw]`` word heat maps and
        ``overlap`` a :class:`RegionOverlap` with a leading map axis (``intersection`` ``[maps, R, W]``, ``word_area``
        ``[maps, W]``); row ``t`` equals ``self[t].region_overlap(...)`` bit for bit (min / max normalisation per map
        and word). E.g. ``overlap.iou()[:, 0, 0]`` is word 0's IoU with region 0 at every step of a history."""
        wl, overlap = _region_overlap(self.tokenizer, self.prompt, self.heat_maps, words, image, regions, absolute,
                                      threshold, word_idx, offset_idx, to_cpu, f'{type(self).__name__}.region_overlap')
        return wl.word_maps, overlap

    def region_sweep(self, words, image, regions: torch.Tensor, thresholds, absolute: bool = False, word_idx=None,
                     offset_idx: int = 0, to_cpu: bool = True):
        """:meth:`GlobalHeatMap.region_sweep` for every map in one call (a memset and three launches whatever the map
        and threshold counts): returns ``(word_maps, overlap)`` with ``word_maps`` the device ``[maps, len(words), xh, xw]`` word heat
        maps and ``overlap`` a :class:`RegionOverlap` with a leading map axis (``intersection`` ``[maps, T, R, W]``,
        ``word_area`` ``[maps, T, W]``); row ``t`` equals ``self[t].region_sweep(...)`` bit for bit (min / max
        normalisation per map and word). E.g. ``overlap.iou()[:, :, 0, 0]`` is word 0's IoU with region 0 at every
        step and threshold."""
        wl, overlap = _region_sweep(self.tokenizer, self.prompt, self.heat_maps, words, image, regions, thresholds,
                                    absolute, word_idx, offset_idx, to_cpu, f'{type(self).__name__}.region_sweep')
        return wl.word_maps, overlap

    def region_ranking(self, words, image, regions: torch.Tensor, absolute: bool = False, word_idx=None,
                       offset_idx: int = 0, to_cpu: bool = True):
        """:meth:`GlobalHeatMap.region_ranking` for every map in one call: returns ``(word_maps, ranking)`` with
        ``word_maps`` the device ``[maps, len(words), xh, xw]`` word heat maps and ``ranking`` a :class:`RegionRanking`
        with a leading map axis (``u2`` and ``ap`` ``[maps, R, W]``); row ``t`` equals ``self[t].region_ranking(...)``
        bit for bit (min / max normalisation per map and word). E.g. ``ranking.auroc()[:, 0, 0]`` is word 0's ROC-AUC
        against region 0 at every step of a history. Scratch stays within a fixed budget whatever the map count: the
        planes are sorted in rounds."""
        wl, ranking = _region_ranking(self.tokenizer, self.prompt, self.heat_maps, words, image, regions, absolute,
                                      word_idx, offset_idx, to_cpu, f'{type(self).__name__}.region_ranking')
        return wl.word_maps, ranking

    def region_boundary(self, words, image, regions: torch.Tensor, threshold: float, tolerances=None,
                        absolute: bool = False, word_idx=None, offset_idx: int = 0, to_cpu: bool = True):
        """:meth:`GlobalHeatMap.region_boundary` for every map in one call: returns ``(word_maps, boundary)`` with
        ``word_maps`` the device ``[maps, len(words), xh, xw]`` word heat maps and ``boundary`` a
        :class:`RegionBoundary` with a leading map axis (``word_hits`` ``[maps, T, R, W]``, ``max_d2`` ``[maps, R, W,
        2]``, ...); row ``t`` equals ``self[t].region_boundary(...)`` bit for bit (min / max normalisation per map and
        word). E.g. ``boundary.f_score()[:, 0, 0, 0]`` is word 0's boundary F against region 0 at every step of a
        history. Scratch stays within a fixed budget whatever the map count: the planes are scored in rounds."""
        wl, boundary = _region_boundary(self.tokenizer, self.prompt, self.heat_maps, words, image, regions, threshold,
                                        tolerances, absolute, word_idx, offset_idx, to_cpu,
                                        f'{type(self).__name__}.region_boundary')
        return wl.word_maps, boundary

    def word_overlap(self, words, image=None, absolute: bool = False, threshold: Optional[float] = None,
                     word_idx=None, offset_idx: int = 0, to_cpu: bool = True):
        """:meth:`GlobalHeatMap.word_overlap` for every map in one call (three launches whatever the map count):
        returns ``(word_maps, overlap)`` with ``word_maps`` the device ``[maps, len(words), xh, xw]`` word heat maps and
        ``overlap`` a :class:`WordOverlap` with a leading map axis (``intersection`` ``[maps, W, W]``, ``word_area``
        ``[maps, W]``); row ``t`` equals ``self[t].word_overlap(...)`` bit for bit (min / max normalisation per map and
        word). E.g. ``overlap.iou()[:, i, j]`` is the IoU of words ``i`` and ``j`` at every step of a history."""
        wl, overlap = _word_overlap(self.tokenizer, self.prompt, self.heat_maps, words, image, absolute, threshold,
                                    word_idx, offset_idx, to_cpu, f'{type(self).__name__}.word_overlap')
        return wl.word_maps, overlap

    def relation_overlap(self, relations, image=None, absolute: bool = False, threshold: Optional[float] = None,
                         offset_idx: int = 0, to_cpu: bool = True) -> 'RelationOverlap':
        """:meth:`GlobalHeatMap.relation_overlap` for every map in one :meth:`word_overlap` call: ``iou``, ``iod`` and
        ``ioh`` are ``[maps, E]``, row ``t`` equal to ``self[t].relation_overlap(...)``'s bit for bit."""
        return _relation_overlap(self.tokenizer, self.prompt, self.heat_maps, relations, image, absolute, threshold,
                                 offset_idx, to_cpu, f'{type(self).__name__}.relation_overlap')

    def word_instances(self, words, image, threshold: float, absolute: bool = False, max_instances: int = 16,
                       word_idx=None, offset_idx: int = 0, to_cpu: bool = True):
        """:meth:`GlobalHeatMap.word_instances` for every map in one call: returns ``(word_maps, instances)`` with
        ``word_maps`` the device ``[maps, len(words), xh, xw]`` word heat maps and ``instances`` a
        :class:`WordInstances` with a leading map axis (``count`` ``[maps, W]``, ``area`` ``[maps, W, K]``, ...); row
        ``t`` equals ``self[t].word_instances(...)`` bit for bit (min / max normalisation per map and word). E.g.
        ``instances.count[:, 0]`` is how many blobs word 0 makes at every step of a history. Scratch stays within a
        fixed budget whatever the map count: the planes are labelled in rounds."""
        wl, inst = _word_instances(self.tokenizer, self.prompt, self.heat_maps, words, image, threshold, absolute,
                                   max_instances, word_idx, offset_idx, to_cpu, f'{type(self).__name__}.word_instances')
        return wl.word_maps, inst

    def word_distance(self, words, image, threshold: float, absolute: bool = False, word_idx=None, offset_idx: int = 0,
                      to_cpu: bool = True):
        """:meth:`GlobalHeatMap.word_distance` for every map in one call: returns ``(word_maps, distance)`` with
        ``word_maps`` the device ``[maps, len(words), xh, xw]`` word heat maps and ``distance`` a :class:`WordDistance`
        with a leading map axis (``signed_d2`` ``[maps, len(words), H, W]``); row ``t`` equals
        ``self[t].word_distance(...)`` bit for bit (min / max normalisation per map and word). E.g.
        ``distance.mask(8)[:, 0]`` is word 0's mask grown by 8 pixels at every step of a history. Scratch stays
        within a fixed budget whatever the map count: the planes are transformed in rounds."""
        wl, dist = _word_distance(self.tokenizer, self.prompt, self.heat_maps, words, image, threshold, absolute,
                                  word_idx, offset_idx, to_cpu, f'{type(self).__name__}.word_distance')
        return wl.word_maps, dist

    def overlay_words(self, words, image, absolute: bool = False, threshold: Optional[float] = None,
                      color_normalize: bool = True, word_idx=None, offset_idx: int = 0, to_cpu: bool = True):
        """:meth:`GlobalHeatMap.overlay_words` for every map in one call (two launches whatever the map count): returns
        ``(word_maps, frames)`` with ``word_maps`` the device ``[maps, len(words), xh, xw]`` word heat maps and
        ``frames`` uint8 ``[maps, len(words), H, W, 3]``; row ``t`` equals ``self[t].overlay_words(...)`` byte for byte
        (colour scale per map and word). ``image`` is one image for every map, or a uint8 ``[maps, H, W, 3]`` array
        with one per map (e.g. the images of ``compute_image_heat_maps()``). ``frames[:, w]`` is word ``w`` forming over
        a history, frame by frame."""
        wl, frames = _overlay(self.tokenizer, self.prompt, self.heat_maps, words, image, absolute, threshold,
                              color_normalize, word_idx, offset_idx, to_cpu, f'{type(self).__name__}.overlay_words',
                              stack=True)
        return wl.word_maps, frames

    def refine_words(self, words, image, radius: int = 8, eps: float = 1e-3, absolute: bool = False,
                     threshold: Optional[float] = None, word_idx=None, offset_idx: int = 0, to_cpu: bool = True):
        """:meth:`GlobalHeatMap.refine_words` for every map in one call: returns ``(word_maps, refined)`` with
        ``word_maps`` the device ``[maps, len(words), xh, xw]`` word heat maps and ``refined`` fp32 ``[maps,
        len(words), H, W]``; row ``t`` equals ``self[t].refine_words(...)`` bit for bit (min / max normalisation per map
        and word). ``image`` is one image for every map (its statistics are computed once), or a uint8 ``[maps, H, W,
        3]`` array with one per map (e.g. the images of ``compute_image_heat_maps()``). Scratch stays within a fixed
        budget whatever the map count: the planes are filtered in rounds."""
        wl, refined = _refine(self.tokenizer, self.prompt, self.heat_maps, words, image, radius, eps, absolute,
                              threshold, word_idx, offset_idx, to_cpu, f'{type(self).__name__}.refine_words',
                              stack=True)
        return wl.word_maps, refined

    def segment_crf(self, words, image, threshold: Optional[float] = None, iterations: int = 5, radius: int = 8,
                    scale: float = 16.0, appearance: float = 10.0, sigma_xy: float = 8.0, sigma_rgb: float = 13.0,
                    smoothness: float = 1.0, sigma_smooth: float = 3.0, absolute: bool = False, word_idx=None,
                    offset_idx: int = 0, probs: bool = False, to_cpu: bool = True):
        """:meth:`GlobalHeatMap.segment_crf` for every map in one call: returns ``(word_maps, labels, scores)``, plus
        ``probs`` when asked, with ``word_maps`` the device ``[maps, len(words), xh, xw]`` word heat maps, ``labels``
        / ``scores`` ``[maps, H, W]`` and ``probs`` ``[maps, L, H, W]``; row ``t`` equals ``self[t].segment_crf(...)``
        bit for bit (min / max normalisation per map and word). ``image`` is one image for every map, or a uint8
        ``[maps, H, W, 3]`` array with one per map (e.g. the images of ``compute_image_heat_maps()``). Scratch stays
        within a fixed budget whatever the map count: the maps go in rounds of whole maps."""
        wl, labels, scores, *q = _segment_crf(self.tokenizer, self.prompt, self.heat_maps, words, image, threshold,
                                              iterations, radius, scale, appearance, sigma_xy, sigma_rgb, smoothness,
                                              sigma_smooth, absolute, word_idx, offset_idx, probs, to_cpu,
                                              f'{type(self).__name__}.segment_crf', stack=True)
        return (wl.word_maps, labels, scores) + tuple(q)

    def segment_superpixels(self, words, image, n_segments: int = 1024, compactness: float = 20.0,
                            iterations: int = 10, threshold: Optional[float] = None, absolute: bool = False,
                            word_idx=None, offset_idx: int = 0, to_cpu: bool = True):
        """:meth:`GlobalHeatMap.segment_superpixels` for every map in one call: returns ``(word_maps, labels, scores,
        superpixels)``, with ``word_maps`` the device ``[maps, len(words), xh, xw]`` word heat maps and ``labels`` /
        ``scores`` ``[maps, H, W]``; row ``t`` equals ``self[t].segment_superpixels(...)`` bit for bit (min / max
        normalisation per map and word). ``image`` is one image for every map, whose partition is made once and
        pooled for every map (``superpixels`` ``[H, W]``), or a uint8 ``[maps, H, W, 3]`` array with one per map
        (e.g. the images of ``compute_image_heat_maps()``; ``superpixels`` ``[maps, H, W]``). Scratch stays within a
        fixed budget whatever the map count: the maps go in rounds of whole maps."""
        wl, labels, scores, sp = _segment_superpixels(self.tokenizer, self.prompt, self.heat_maps, words, image,
                                                      n_segments, compactness, iterations, threshold, absolute,
                                                      word_idx, offset_idx, to_cpu,
                                                      f'{type(self).__name__}.segment_superpixels', stack=True)
        return wl.word_maps, labels, scores, sp


class TimeHeatMaps(GlobalHeatMapStack):
    """One global heat map per traced denoising step (UNet forward) of one prompt: ``heat_maps[t]`` is exactly what
    :meth:`~daam_b200.trace.DiffusionHeatMapHooker.compute_global_heat_map` would return had only step ``t`` been
    traced (per-key bicubic, clamp, mean over keys, ``n_tokens + 2`` rows). ``heat_maps`` is ``[steps, n_rows, xh,
    xw]``; ``word_heat_maps`` and ``segment`` work over every step.

    The steps do not sum to the all-steps map: the clamp comes after the time sum there and per step here."""


class ImageHeatMaps(GlobalHeatMapStack):
    """One global heat map per image of one prompt (``num_images_per_prompt``): ``heat_maps[i]`` is exactly
    :meth:`~daam_b200.trace.DiffusionHeatMapHooker.compute_global_heat_map` with ``image_idx=i``, the DAAM map over
    image ``i``'s keys only. ``heat_maps`` is ``[images, n_rows, xh, xw]``; ``word_heat_maps`` and ``segment`` work over
    every image."""


def _labels(stack: GlobalHeatMapStack, **labels) -> None:
    """Attach one label list per keyword to ``stack``, each with one entry per map."""
    for name, values in labels.items():
        values = list(values)
        if len(values) != len(stack):
            raise ValueError(f'{type(stack).__name__}: {len(values)} {name} for {len(stack)} maps')
        setattr(stack, name, values)


class LayerHeatMaps(GlobalHeatMapStack):
    """One global heat map per traced UNet layer: ``heat_maps[i]`` is exactly
    :meth:`~daam_b200.trace.DiffusionHeatMapHooker.compute_global_heat_map` with ``layer_idx=layers[i]``, the DAAM map
    over that layer's heads only. ``layers[i]``, ``names[i]`` (the module path, ``trace.layer_names``) and
    ``factors[i]`` label map ``i``; ``heat_maps`` is ``[layers, n_rows, xh, xw]``, and the word-list calls work over
    every layer: e.g. ``layers[region_overlap(...)[1].iou()[:, 0, 0].argmax()]`` is the layer that localises word 0
    best."""

    def __init__(self, tokenizer, prompt: str, heat_maps: torch.Tensor, layers, names, factors):
        super().__init__(tokenizer, prompt, heat_maps)
        _labels(self, layers=layers, names=names, factors=factors)


class FactorHeatMaps(GlobalHeatMapStack):
    """One global heat map per traced resolution: ``heat_maps[j]`` is exactly
    :meth:`~daam_b200.trace.DiffusionHeatMapHooker.compute_global_heat_map` with ``factors={factors[j]}``;
    ``factors`` ascends (1 is the finest layer size). ``heat_maps`` is ``[factors, n_rows, xh, xw]``."""

    def __init__(self, tokenizer, prompt: str, heat_maps: torch.Tensor, factors):
        super().__init__(tokenizer, prompt, heat_maps)
        _labels(self, factors=factors)


class HeadHeatMaps(GlobalHeatMapStack):
    """One heat map per key: ``heat_maps[i]`` is the map of
    :meth:`~daam_b200.trace.DiffusionHeatMapHooker.compute_global_heat_map` with ``layer_idx`` and ``head_idx`` of
    ``keys[i] = (factor, layer, head)``, the reference's ``--all-heads`` sweep. ``heat_maps`` is ``[keys, n_rows, xh,
    xw]``."""

    def __init__(self, tokenizer, prompt: str, heat_maps: torch.Tensor, keys):
        super().__init__(tokenizer, prompt, heat_maps)
        _labels(self, keys=keys)
