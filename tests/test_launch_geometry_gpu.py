"""The accumulate launches against float64 at every pack, tile-walk and ring geometry the planner produces.

``daam_accumulate`` / ``_steps`` / ``_range`` sort the layer calls into seven packs (16-bit wgmma, fp32 split form,
SIMT, and 16-bit wgmma / SIMT at 154 and 231 tokens), close a pack at 32 layers or when a layer's accumulator overlaps
one already in it, and launch each pack as one persistent grid. Its CTAs then walk the pack's tiles in one of three
ways: interleaved (single-chunk 16-bit wgmma: tiles b, b + grid, ...), contiguous ranges of ``per`` / ``per + 1``
tiles (split form, SIMT kernels, ``attention_probs``), or contiguous ranges of equal weight (K-chunked wgmma: a CTA
may get no tile at all). Inside a CTA the Q/K ring (2 stages), the accumulator ring (3 slots, ``kC`` per tile at long
contexts), the early-loads L2 prefetch window (6 tiles) and the SIMT ``run`` key restart at fixed tile counts.

:func:`plan` restates the packing and each launch's instance, grid and layer table; :func:`walk` gives every CTA's
tiles in order; :func:`regimes` labels what a case reaches. The case table is built from the SM count and the SIMT
occupancy, each case asserts the regimes it names, and ``tests/test_launch_geometry_host.py`` checks without a GPU
that the cases reach them at several SM counts and occupancies and that the walks cover every tile exactly once.

Every case runs through the C ABI and is checked

* against float64 (``desc_maps64`` within ``accumulate_tolerance`` of each element's own inputs) after two calls;
* bit for bit across launch modes: without PDL, with PDL and with early Q/K loads, and issued pack by pack (one call
  per launch of the plan) -- and a step slab equals one call's accumulator, a range slab the accumulator itself;
* for stray writes: sentinel runs sit around every accumulator and second slab, and the Q/K storage a descriptor does
  not address is NaN;
* for its launches: ``launch_count()`` moves by ``len(plan)`` per call, and one ``torch.profiler`` trace over one call
  of every case lists the instances (template arguments included) and grids the plans name.

The SIMT grid is ``sm_count x`` the occupancy the runtime reports for the pack's shared memory (sized by its largest
head_dim); it is measured here from the traced grid of one large launch per kernel and head_dim, not assumed.

The worst error-to-bound ratio per (instance, dtype) and the measured SIMT grids are printed at the end (``-s``)."""
import bisect
import collections
import dataclasses
import json
import tempfile
from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Tuple

import pytest
import torch

from daam_b200 import _native
from tests.reference64 import (ACC_DIMS, FP32_EPS, accumulate_tolerance, assert_close64, desc_maps64, layer_views64,
                               probs_tolerance)
from tests.util import kernel_events, traced

pytestmark = pytest.mark.gpu
DEV = 'cuda'

TILE = 128                   # kTilePixels
TOKENS = 77
MAX_LAYERS = 32              # kMaxLayersPerLaunch
STAGES = 2                   # kStages: the Q/K ring
ACC_STAGES = 3               # kAccStages: the accumulator ring (16-bit form)
PREFETCH = 6                 # kPrefetchTiles: the early-loads L2 prefetch window
PROBS_PER_SM = 3             # daam_attention_probs: 3 CTAs per SM
CALLS = 2                    # calls per run, back to back

DTYPES = {'fp32': torch.float32, 'fp16': torch.float16, 'bf16': torch.bfloat16}
CODES = {'fp32': _native.DAAM_F32, 'fp16': _native.DAAM_F16, 'bf16': _native.DAAM_BF16}
SLAB_MODE = {'accumulate': 0, 'steps': 1, 'range': 2}
SIMT_KERNEL = {'accumulate': 'accumulate_simt_kernel', 'steps': 'accumulate_simt_step_kernel',
               'range': 'accumulate_simt_range_kernel'}
SIMT_LONG = 'accumulate_simt_long_kernel'
PROBS = 'attention_probs_kernel'
# the pack classes of build_plan, in its order: 77-token 16-bit wgmma, fp32 split form, SIMT; 16-bit wgmma at 154 /
# 231 tokens; SIMT at 154 / 231 tokens
CLASSES = ('mma16', 'split', 'simt', 'mma16-154', 'mma16-231', 'simt-154', 'simt-231')
ENTRY_CLASSES = {'accumulate': CLASSES, 'steps': CLASSES[:3], 'range': CLASSES[:3]}


# ---- the case description ---------------------------------------------------------------------------------------------

@dataclass
class Layer:
    """One layer call: ``[prompts, heads, tokens, hw]`` accumulator, head_dim ``d``."""
    hw: int
    heads: int = 1
    d: int = 64
    dtype: str = 'bf16'
    tokens: int = TOKENS
    prompts: int = 1
    simt: bool = False          # Q / K rows one element off 16-byte alignment: the SIMT kernels on every path
    acc_of: Optional[int] = None    # adds into the accumulator of this earlier layer (same shape)

    @property
    def tiles(self) -> int:
        return -(-self.hw // TILE) * self.heads * self.prompts

    @property
    def chunks(self) -> int:
        return -(-self.d // 64)


@dataclass
class Case:
    entry: str                  # 'accumulate', 'steps', 'range' or 'probs' (daam_attention_probs, one layer)
    flags: int                  # path and update mode; the runs add NO_PDL / PDL / EARLY_LOADS
    layers: List[Layer]
    tags: Tuple[str, ...]       # regimes the case must reach (see regimes())

    def owner(self, i: int) -> int:
        """The layer whose accumulator layer ``i`` adds into."""
        a = self.layers[i].acc_of
        return i if a is None else self.owner(a)


@dataclass
class Launch:
    cls: str                    # pack class (CLASSES), or 'probs'
    instance: str               # kernel name with its template arguments, as the profiler shows it (no spaces)
    G: int                      # the grid before it is capped at the tile count
    grid: int
    walk: str                   # 'interleaved', 'contiguous' or 'weighted'
    layers: List[dict]          # per layer of the launch: index (into the case), tile_begin, tiles, weight, weight_begin
    close: str                  # why the pack closed: 'full', 'overlap' or 'end'
    kC: int = 1                 # 77-token chunks of the context
    chunked: bool = False

    @property
    def total_tiles(self) -> int:
        return sum(e['tiles'] for e in self.layers)

    @property
    def total_weight(self) -> int:
        return sum(e['tiles'] * e['weight'] for e in self.layers)


# ---- the planner, restated ----------------------------------------------------------------------------------------------

def layer_class(layer: Layer, flags: int) -> int:
    """build_plan's pack of a layer: the wgmma kernel takes 16-byte aligned rows with hw % 4 == 0 (fp32 only at 77
    tokens), unless the call forces the SIMT kernel."""
    ctx = layer.tokens // TOKENS
    use_mma = ((flags & 3) != _native.ACC_FORCE_SIMT and layer.hw % 4 == 0 and not layer.simt and
               (ctx == 1 or layer.dtype != 'fp32'))
    if ctx > 1:
        return (1 if use_mma else 3) + ctx
    return (1 if layer.dtype == 'fp32' else 0) if use_mma else 2


def mma_instance(split: bool, chunked: bool, mode: int, kC: int) -> str:
    b = lambda v: 'true' if v else 'false'
    return f'accumulate_mma_kernel<{b(split)},{b(chunked)},{mode},{kC}>'


def simt_instance(cls: str, entry: str) -> str:
    return SIMT_LONG if cls.startswith('simt-') else SIMT_KERNEL[entry]


OccFn = Callable[[str, int], int]     # (SIMT instance, largest head_dim of the pack) -> CTAs per SM


def _launch(case: Case, which: int, members: List[int], close: str, sm_count: int, occ: OccFn) -> Launch:
    cls = CLASSES[which]
    layers = [case.layers[i] for i in members]
    table, tb, wb = [], 0, 0
    for i, L in zip(members, layers):
        weight = L.chunks if cls == 'split' else 1 + 4 * L.chunks
        table.append(dict(index=i, tile_begin=tb, tiles=L.tiles, weight=weight, weight_begin=wb))
        tb += L.tiles
        wb += L.tiles * weight
    chunked = any(L.d > 64 for L in layers)
    kC = layers[0].tokens // TOKENS
    if cls.startswith('mma16') or cls == 'split':
        split = cls == 'split'
        G = sm_count
        inst = mma_instance(split, chunked, SLAB_MODE[case.entry], kC)
        walk = 'weighted' if chunked else ('contiguous' if split else 'interleaved')
    else:
        inst = simt_instance(cls, case.entry)
        G = sm_count * occ(inst, max(L.d for L in layers))
        walk = 'contiguous'
    return Launch(cls, inst, G, min(G, tb), walk, table, close, kC, chunked)


def plan(case: Case, sm_count: int, occ: OccFn) -> List[Launch]:
    """The launches one call of ``case`` makes, in order (build_plan and the prepare_* functions)."""
    if case.entry == 'probs':
        (L,) = case.layers
        G = PROBS_PER_SM * sm_count
        return [Launch('probs', PROBS, G, min(G, L.tiles), 'contiguous',
                       [dict(index=0, tile_begin=0, tiles=L.tiles, weight=1, weight_begin=0)], 'end')]
    packs: List[List[int]] = [[] for _ in CLASSES]
    out: List[Launch] = []

    def close(which: int, why: str):
        if packs[which]:
            out.append(_launch(case, which, packs[which], why, sm_count, occ))
            packs[which] = []

    for i, L in enumerate(case.layers):
        w = layer_class(L, case.flags)
        if any(case.owner(j) == case.owner(i) for j in packs[w]):
            close(w, 'overlap')
        packs[w].append(i)
        if len(packs[w]) == MAX_LAYERS:
            close(w, 'full')
    for w in range(len(CLASSES)):
        close(w, 'end')
    return out


def tile_at_weight(launch: Launch, w: int) -> int:
    """accumulate_mma.cu's tile_at_weight: the first tile whose weight offset is >= w."""
    if w >= launch.total_weight:
        return launch.total_tiles
    e = [x for x in launch.layers if x['weight_begin'] <= w][-1]
    return e['tile_begin'] + -(-(w - e['weight_begin']) // e['weight'])


def cta_tiles(launch: Launch, b: int) -> range:
    """The tiles CTA ``b`` takes, in its order."""
    T, g = launch.total_tiles, launch.grid
    if launch.walk == 'interleaved':
        return range(b, T, g)
    if launch.walk == 'contiguous':
        per, rem = divmod(T, g)
        first = b * per + min(b, rem)
        return range(first, first + per + (1 if b < rem else 0))
    W = launch.total_weight
    return range(tile_at_weight(launch, W * b // g), tile_at_weight(launch, W * (b + 1) // g))


def decode(case: Case, launch: Launch, tile: int) -> Tuple[int, int, int, int]:
    """``(layer, prompt, head, pixel0)`` of a tile of a launch (decode_tile)."""
    starts = [e['tile_begin'] for e in launch.layers]
    e = launch.layers[bisect.bisect_right(starts, tile) - 1]
    L = case.layers[e['index']]
    local = tile - e['tile_begin']
    tph = -(-L.hw // TILE)
    ph = local // tph
    return e['index'], ph // L.heads, ph % L.heads, (local % tph) * TILE


def walk(case: Case, launch: Launch) -> List[List[Tuple[int, int, int, int, int]]]:
    """Per CTA, its tiles in order as ``(tile, layer, prompt, head, pixel0)``."""
    return [[(t,) + decode(case, launch, t) for t in cta_tiles(launch, b)] for b in range(launch.grid)]


# ---- regimes ------------------------------------------------------------------------------------------------------------

def tile_label(T: int, G: int) -> Optional[str]:
    for label, n in (('1', 1), ('G-1', G - 1), ('G', G), ('G+1', G + 1), ('2G+1', 2 * G + 1)):
        if T == n:
            return label
    return None


def regimes(case: Case, launches: List[Launch]) -> set:
    """The regimes one call of ``case`` reaches, as the tags the cases name."""
    tags = set()
    rmw = 'LDST' if case.flags & 0x30 == _native.ACC_RMW_LDST else 'RED'
    tags.add(f'{case.entry} {rmw}')
    if case.flags & 3 == _native.ACC_FORCE_SIMT:
        tags.add('FORCE_SIMT')
    seq = [layer_class(L, case.flags) for L in case.layers]
    if case.entry != 'probs' and len(set(seq)) == len(CLASSES):
        runs = sum(1 for i, w in enumerate(seq) if i == 0 or seq[i - 1] != w)
        if runs > len(CLASSES):
            tags.add('all 7 classes interleaved')
    per_class = collections.Counter(l.cls for l in launches)
    for n, l in enumerate(launches):
        inst, ws = l.instance, walk(case, l)
        counts = [len(w) for w in ws]
        T = l.total_tiles
        label = tile_label(T, l.G)
        if label:
            tags.add(f'{inst}: tiles {label}')
        for c in set(counts):
            if 1 <= c <= 4:
                tags.add(f'{inst}: per CTA {c}')
        if max(counts) >= 8:
            tags.add(f'{inst}: per CTA >= 8')
        if l.walk == 'contiguous':
            tags.add(f'{inst}: rem ' + ('0' if T % l.grid == 0 else '> 0'))
        if l.walk == 'weighted':
            if min(counts) == 0:
                tags.add(f'{inst}: zero-tile CTA')
            starts = {e['weight_begin'] + k * e['weight'] for e in l.layers for k in range(e['tiles'])}
            if any(l.total_weight * b // l.grid not in starts for b in range(1, l.grid)):
                tags.add(f'{inst}: boundary inside a tile')
            for w in ws:
                if {case.layers[t[1]].chunks for t in w} >= {1, 2, 3, 4}:
                    tags.add(f'{inst}: CTA spans 1-4 chunks')
            if sum(case.layers[e['index']].d > 64 for e in l.layers) == 1:
                tags.add(f'{inst}: chunked by one layer')
        if l.cls.startswith('mma16'):
            start = 1 if l.chunked else STAGES
            if max(counts) >= start + PREFETCH:
                tags.add(f'{inst}: prefetch window full')
            if any(start < c < start + PREFETCH for c in counts):
                tags.add(f'{inst}: prefetch window truncated')
            if l.kC > 1 and max(counts) * l.kC > ACC_STAGES:
                tags.add(f'{inst}: accumulator ring wraps')
        for w in ws:
            layers_seen = {t[1] for t in w}
            if len(layers_seen) > 1 and any(case.layers[i].tiles == 1 for i in layers_seen):
                tags.add(f'{inst}: one-tile layer inside a CTA range')
            for a, b in zip(w, w[1:]):
                if a[1] != b[1] and a[2:4] == b[2:4]:
                    tags.add(f'{inst}: same (prompt, head), next layer')
            if l.cls.startswith('mma16'):
                dts = [case.layers[t[1]].dtype for t in w]
                if sum(1 for x, y in zip(dts, dts[1:]) if x != y) >= 2:
                    tags.add('16-bit CTA alternates fp16 / bf16')
        for e in l.layers:
            L = case.layers[e['index']]
            if L.hw % TILE in (4, 64, 124):
                tags.add(f'{inst}: hw mod 128 = {L.hw % TILE}')
            if L.prompts in (2, 3):
                tags.add(f'{inst}: {L.prompts} prompts')
        ds = {case.layers[e['index']].d for e in l.layers}
        if l.cls == 'simt' and {8, 256} <= ds:
            tags.add('SIMT pack with d 256 and d 8')
        if l.close == 'full':
            tags.add(f'{case.entry} {l.cls}: 32 layers')
            rest = [m for m in launches[n + 1:] if m.cls == l.cls]
            if per_class[l.cls] == 2 and len(rest) == 1 and len(rest[0].layers) == 1:
                tags.add(f'{case.entry} {l.cls}: 33 layers')
                first = rest[0].layers[0]['index']
                if any(case.owner(e['index']) == case.owner(first) for e in l.layers):
                    tags.add(f'{l.cls}: overlap at position 32')
        if l.close == 'overlap' and len(l.layers) == MAX_LAYERS - 1:
            tags.add(f'{l.cls}: overlap close at position 31')
    return tags


# ---- the cases ----------------------------------------------------------------------------------------------------------

# head_dims of the single-chunk and the K-chunked packs (1, 2, 3 and 4 chunks of 64). The first is the pack's largest
# (SIMT) or a K-chunked one (wgmma), so that a pack of one layer has the instance and grid of a longer one.
PLAIN_DS = (64, 40, 8)
CHUNKED_DS = (160, 8, 80, 256, 64, 192, 128)
SIMT_CHUNKED_DS = (256, 8, 160, 80)
# the head of every pack: (hw, heads, prompts) -- 3 and 2 prompts, partial last tiles of 64, 124 and 4 pixels, a one-tile
# layer; the rest of the pack's tiles go to one filler layer
HEAD = ((64, 2, 3), (192, 1, 2), (124, 1, 1), (260, 1, 1))


def pack_layers(T: int, ds=PLAIN_DS, dtypes=('bf16', 'fp16'), tokens=TOKENS, simt=False, odd_hw=False) -> List[Layer]:
    """Layers with ``T`` tiles in all: the HEAD layers that fit, then one layer of one head and prompt with the rest.
    ``odd_hw``: every hw one pixel less (not a multiple of 4: the SIMT kernels)."""
    out, rem = [], T
    for hw, heads, prompts in HEAD:
        tiles = -(-hw // TILE) * heads * prompts
        if tiles < rem:
            out.append((hw, heads, prompts))
            rem -= tiles
    if rem:
        out.append((TILE * rem - 64, 1, 1))
    return [Layer(hw - (1 if odd_hw else 0), heads, ds[i % len(ds)], dtypes[i % len(dtypes)], tokens, prompts, simt)
            for i, (hw, heads, prompts) in enumerate(out)]


def class_spec(cls: str, chunked: bool, variant: int) -> dict:
    """pack_layers arguments that put every layer into pack class ``cls`` (under DAAM_ACC_AUTO)."""
    ds = (SIMT_CHUNKED_DS if cls.startswith('simt') else CHUNKED_DS) if chunked else PLAIN_DS
    if cls == 'mma16':
        return dict(ds=ds)
    if cls == 'split':
        return dict(ds=ds, dtypes=('fp32',))
    if cls == 'simt':            # unaligned rows, or pixel counts that are not a multiple of 4
        return dict(ds=ds, dtypes=('fp32', 'bf16', 'fp16'), simt=variant % 2 == 0, odd_hw=variant % 2 == 1)
    ctx = int(cls.split('-')[1])
    if cls.startswith('mma16'):
        return dict(ds=ds, tokens=ctx)
    return dict(ds=ds, dtypes=('fp32',), tokens=ctx)


def class_instance(cls: str, entry: str, chunked: bool) -> str:
    if cls.startswith('simt'):
        return simt_instance(cls, entry)
    kC = int(cls.split('-')[1]) // TOKENS if '-' in cls else 1
    return mma_instance(cls == 'split', chunked, SLAB_MODE[entry], kC)


def class_grid(cls: str, entry: str, chunked: bool, sm: int, occ: OccFn) -> int:
    if not cls.startswith('simt'):
        return sm
    return sm * occ(class_instance(cls, entry, chunked), class_spec(cls, chunked, 0)['ds'][0])


LABELS = {'1': lambda G: 1, 'G-1': lambda G: G - 1, 'G': lambda G: G, 'G+1': lambda G: G + 1,
          '2G+1': lambda G: 2 * G + 1, '3G+1': lambda G: 3 * G + 1, '8G+1': lambda G: 8 * G + 1}


def _grid_case(label: str, entry: str, chunked: bool):
    """Every pack class of ``entry`` at ``label`` tiles (relative to its own grid), one class after the other."""
    variant = list(LABELS).index(label)

    def build(sm: int, occ: OccFn) -> Case:
        layers, tags = [], []
        for cls in ENTRY_CLASSES[entry]:
            G = class_grid(cls, entry, chunked, sm, occ)
            layers += pack_layers(LABELS[label](G), **class_spec(cls, chunked, variant))
            inst = class_instance(cls, entry, chunked)
            if label in ('1', 'G-1', 'G', 'G+1', '2G+1'):
                tags.append(f'{inst}: tiles {label}')
            if not cls.startswith('simt') and not chunked:
                tags += {'G': [f'{inst}: per CTA 1'], '3G+1': [f'{inst}: per CTA 4'],
                         '8G+1': [f'{inst}: per CTA >= 8']}.get(label, [])
        rmw = _native.ACC_RMW_LDST if (variant + chunked) % 2 else _native.ACC_RMW_RED
        return Case(entry, rmw, layers, tuple(tags) + (f'{entry} {"LDST" if rmw == _native.ACC_RMW_LDST else "RED"}',))
    return build


def _probs(label: str, dtype: str):
    def build(sm: int, occ: OccFn) -> Case:
        T = LABELS[label](PROBS_PER_SM * sm)
        prompts = 2 if T % 2 == 0 and T > 2 else 1
        return Case('probs', 0, [Layer(TILE * (T // prompts) - 60, 1, 64, dtype, prompts=prompts)],
                    (f'{PROBS}: tiles {label}',))
    return build


def _mixed_dtypes(sm: int, occ: OccFn) -> Case:
    """Four layers of G tiles, fp16 and bf16 in turn: CTA b takes tile b of each, with the same (prompt, head) and a
    new layer every time (the prefetch window's new_head test)."""
    layers = [Layer(TILE * sm - 4, 1, 64, ('fp16', 'bf16')[i % 2]) for i in range(4)]
    inst = mma_instance(False, False, 0, 1)
    return Case('accumulate', 0, layers, ('16-bit CTA alternates fp16 / bf16', f'{inst}: same (prompt, head), next layer',
                                          f'{inst}: per CTA 4', f'{inst}: hw mod 128 = 124'))


def _chunk_spans(split: bool):
    """A K-chunked pack whose first CTAs each span layers of 1, 2, 3 and 4 chunks, then a filler of 1-chunk tiles."""
    def build(sm: int, occ: OccFn) -> Case:
        dtype = ('fp32',) if split else ('bf16', 'fp16')
        head = [Layer(TILE, 1, d, dtype[i % len(dtype)]) for i, d in enumerate((8, 80, 160, 256) * 4)]
        layers = head + [Layer(TILE * (8 * sm) - 64, 1, 64, dtype[0])]
        inst = mma_instance(split, True, 0, 1)
        return Case('accumulate', _native.ACC_RMW_RED, layers,
                    (f'{inst}: CTA spans 1-4 chunks', f'{inst}: boundary inside a tile', f'{inst}: one-tile layer inside a CTA range'))
    return build


def _one_chunked_layer(entry: str):
    """Single-chunk layers and one of 80 dims: the whole pack takes the weighted walk because of that one layer, and
    at G + 1 tiles some CTAs get none."""
    def build(sm: int, occ: OccFn) -> Case:
        layers = []
        for cls, dt in (('mma16', ('bf16', 'fp16')), ('split', ('fp32',))):
            part = pack_layers(sm + 1, ds=(64,), dtypes=dt)
            part[1].d = 80
            layers += part
        insts = [mma_instance(s, True, SLAB_MODE[entry], 1) for s in (False, True)]
        return Case(entry, _native.ACC_RMW_RED, layers,
                    tuple(f'{i}: chunked by one layer' for i in insts) + tuple(f'{i}: zero-tile CTA' for i in insts))
    return build


def _pack_split(entry: str, n: int):
    """``n`` one-tile layers of every pack class of ``entry``, interleaved in call order."""
    def build(sm: int, occ: OccFn) -> Case:
        classes = ENTRY_CLASSES[entry]
        layers = []
        for i in range(n * len(classes)):
            cls = classes[i % len(classes)]
            spec = class_spec(cls, False, i // len(classes))
            layers += pack_layers(1, **{**spec, 'ds': (PLAIN_DS[i % 3],)})
        tags = tuple(f'{entry} {c}: {k} layers' for c in classes for k in ((32,) if n == 32 else (32, 33)))
        if entry == 'accumulate':
            tags += ('all 7 classes interleaved',)
        return Case(entry, _native.ACC_RMW_LDST if n == 33 else _native.ACC_RMW_RED, layers, tags)
    return build


def _overlap(position: int):
    """Layer ``position`` of the 16-bit and of the SIMT pack adds into layer 0's accumulator: at 31 the pack closes
    early (31 layers), at 32 it has closed full already and the layer starts the next launch either way."""
    def build(sm: int, occ: OccFn) -> Case:
        layers = []
        for cls in ('mma16', 'simt'):
            base = len(layers)
            spec = class_spec(cls, False, 0)
            for i in range(position):
                layers += pack_layers(1 if i else 3, **{**spec, 'ds': (PLAIN_DS[i % 3],)})[-1:]
            layers.append(dataclasses.replace(layers[base], d=40, acc_of=base))
        tag = 'overlap close at position 31' if position == 31 else 'overlap at position 32'
        return Case('accumulate', _native.ACC_RMW_RED, layers, tuple(f'{c}: {tag}' for c in ('mma16', 'simt')))
    return build


def _force_simt(label: str):
    """Aligned 16-bit and fp32 layers under DAAM_ACC_FORCE_SIMT (the vector loads), several prompts and heads."""
    def build(sm: int, occ: OccFn) -> Case:
        G = sm * occ(SIMT_KERNEL['accumulate'], 256)
        layers = pack_layers(LABELS[label](G), ds=(256, 8, 64), dtypes=('bf16', 'fp16', 'fp32'))
        return Case('accumulate', _native.ACC_FORCE_SIMT | _native.ACC_RMW_LDST, layers,
                    ('FORCE_SIMT', 'SIMT pack with d 256 and d 8', f'{SIMT_KERNEL["accumulate"]}: tiles {label}'))
    return build


CASES: Dict[str, Callable[[int, OccFn], Case]] = {
    **{f'grid-{label}-{entry}-{"chunked" if ch else "plain"}': _grid_case(label, entry, ch)
       for label in LABELS for entry in ('accumulate', 'steps', 'range') for ch in (False, True)},
    **{f'probs-{label}': _probs(label, ('bf16', 'fp16', 'fp32')[i % 3])
       for i, label in enumerate(('1', 'G-1', 'G', 'G+1', '2G+1'))},
    'mixed-dtypes': _mixed_dtypes,
    'chunk-spans-16bit': _chunk_spans(False),
    'chunk-spans-split': _chunk_spans(True),
    **{f'one-chunked-layer-{entry}': _one_chunked_layer(entry) for entry in ('accumulate', 'steps', 'range')},
    **{f'pack-{n}-{entry}': _pack_split(entry, n) for n in (32, 33) for entry in ('accumulate', 'steps', 'range')},
    'overlap-31': _overlap(31),
    'overlap-32': _overlap(32),
    'force-simt-G+1': _force_simt('G+1'),
    'force-simt-2G+1': _force_simt('2G+1'),
}
CASE_NAMES = list(CASES)


# ---- running a case -----------------------------------------------------------------------------------------------------

GUARD = 64                   # sentinel floats before and after every accumulator and second slab
SENTINEL = 12345.0
RATIOS: Dict[Tuple[str, str], float] = collections.defaultdict(float)
MEASURED: Dict[Tuple[str, int], int] = {}


def _pool(sizes: List[int], fill: float):
    """One fp32 buffer holding regions of ``sizes`` floats, each 16-byte aligned between sentinel runs; returns the
    buffer, the mask of region elements and the regions."""
    offs, pos = [], GUARD
    for n in sizes:
        offs.append(pos)
        pos = -(-(pos + n + GUARD) // 4) * 4
    buf = torch.full((pos,), SENTINEL, device=DEV)
    inside = torch.zeros(pos, dtype=torch.bool, device=DEV)
    for o, n in zip(offs, sizes):
        inside[o:o + n] = True
    buf[inside] = fill
    return buf, inside, [buf[o:o + n] for o, n in zip(offs, sizes)]


HEAD_PAD = 8                 # NaN elements after every head's d values (rows stay 16-byte multiples)


def _store(x: torch.Tensor, shift: int):
    """``x [P, H, rows, d]`` as the conditional half of a ``[2P, rows, H, d + HEAD_PAD]`` projection in a NaN-filled
    buffer, ``shift`` elements past a 16-byte boundary. NaN lies before the view (the unconditional half), after each
    head's d values, and after the view (TILE more rows: past the last pixel, and past the last token up to the 80
    padded ones), so that a read outside the view makes its result NaN. Returns the buffer, the element offset of x and
    its strides."""
    P, H, rows, d = x.shape
    dp = d + HEAD_PAD
    n = P * rows * H * dp
    store = torch.full((shift + 2 * n + TILE * H * dp,), float('nan'), dtype=x.dtype, device=DEV)
    store[shift + n:shift + 2 * n].view(P, rows, H, dp)[..., :d] = x.permute(0, 2, 1, 3)
    return store, shift + n, (rows * H * dp, H * dp, dp)


class Run:
    """A case's Q / K, descriptors, accumulators and second slabs on the device."""

    def __init__(self, case: Case, seed: int):
        self.case = case
        g = torch.Generator(device=DEV).manual_seed(seed)
        self.q, self.k, self.descs = [], [], []
        for L in case.layers:
            dt = DTYPES[L.dtype]
            q = (torch.randn(L.prompts, L.heads, L.hw, L.d, generator=g, device=DEV) * 1.5).to(dt)
            k = torch.randn(L.prompts, L.heads, L.tokens, L.d, generator=g, device=DEV).to(dt)
            shift = 1 if L.simt else 0
            qs, qo, (qsp, qsr, qsh) = _store(q, shift)
            ks, ko, (ksp, ksr, ksh) = _store(k, shift)
            es = q.element_size()
            self.q.append(qs)
            self.k.append(ks)
            self.descs.append(_native.DaamLayer(
                q=qs.data_ptr() + qo * es, k=ks.data_ptr() + ko * es, acc=None,
                q_stride_prompt=qsp, q_stride_pixel=qsr, q_stride_head=qsh, k_stride_prompt=ksp, k_stride_token=ksr,
                k_stride_head=ksh, n_prompts=L.prompts, heads=L.heads, hw=L.hw, tokens=L.tokens, head_dim=L.d,
                dtype=CODES[L.dtype], scale=float(L.d ** -0.5), reserved=0))
        shape = lambda L: (L.prompts, L.heads, L.tokens, L.hw)
        n = lambda L: L.prompts * L.heads * L.tokens * L.hw
        self.owners = sorted({case.owner(i) for i in range(len(case.layers))})
        if case.entry == 'probs':
            (L,) = case.layers
            self.probs = torch.full((2 * GUARD + n(L),), SENTINEL, dtype=DTYPES[L.dtype], device=DEV)
            return
        self.acc_buf, self.acc_inside, regions = _pool([n(case.layers[o]) for o in self.owners], 0.0)
        self.accs = {o: r.view(shape(case.layers[o])) for o, r in zip(self.owners, regions)}
        for i, d in enumerate(self.descs):
            d.acc = self.accs[case.owner(i)].data_ptr()
        if case.entry != 'accumulate':
            self.slab_fill = -7.0 if case.entry == 'steps' else 0.0      # every element of a step slab is written
            self.slab_buf, self.slab_inside, regions = _pool([n(L) for L in case.layers], self.slab_fill)
            self.slabs = [r.view(shape(L)) for r, L in zip(regions, case.layers)]

    def reset(self):
        self.acc_buf.masked_fill_(self.acc_inside, 0.0)
        if self.case.entry != 'accumulate':
            self.slab_buf.masked_fill_(self.slab_inside, self.slab_fill)

    def call(self, flags: int, subset: Optional[List[int]] = None):
        idx = list(range(len(self.descs))) if subset is None else subset
        descs = [self.descs[i] for i in idx]
        stream = torch.cuda.current_stream().cuda_stream
        if self.case.entry == 'accumulate':
            _native.accumulate(descs, stream, flags)
        elif self.case.entry == 'steps':
            _native.accumulate_steps(descs, [self.slabs[i].data_ptr() for i in idx], stream, flags)
        elif self.case.entry == 'range':
            _native.accumulate_range(descs, [self.slabs[i].data_ptr() for i in idx], stream, flags)
        else:
            _native.attention_probs(self.descs[0], self.probs.data_ptr() + GUARD * self.probs.element_size(), stream)

    def check_guards(self, what: str):
        assert bool((self.acc_buf[~self.acc_inside] == SENTINEL).all()), f'{what}: a write outside the accumulators'
        if self.case.entry != 'accumulate':
            assert bool((self.slab_buf[~self.slab_inside] == SENTINEL).all()), f'{what}: a write outside the slabs'

    def bits(self) -> List[torch.Tensor]:
        out = [self.accs[o].clone().view(torch.int32) for o in self.owners]
        if self.case.entry != 'accumulate':
            out += [s.clone().view(torch.int32) for s in self.slabs]
        return out


def _form(cls: str) -> str:
    return 'wgmma16' if cls.startswith('mma16') else 'split' if cls == 'split' else 'simt'


def _check_float64(run: Run, launches: List[Launch], name: str):
    """Every accumulator against the float64 sum of what its layers add over CALLS calls. An accumulator that m layers
    share takes each layer's own bound for CALLS calls, plus the rounding of the n = m CALLS fp32 adds in their
    interleaved order: the k-th add rounds a partial sum of at most k addends, so all of them err by at most
    ``u n (n + 1) / 2`` times the largest addend, and an addend is at most its probability plus its own bound."""
    case = run.case
    cls_of = {e['index']: (l.cls, l.instance) for l in launches for e in l.layers}
    for o in run.owners:
        members = [i for i in range(len(case.layers)) if case.owner(i) == o]
        ref, tol, largest = None, None, None
        for i in members:
            d = run.descs[i]
            q64, k64 = layer_views64(d, run.q[i], run.k[i])
            r = desc_maps64(d, run.q[i], run.k[i])
            t = accumulate_tolerance(q64, k64, float(d.scale), _form(cls_of[i][0]), CALLS)
            ref, tol = (r * CALLS, t) if ref is None else (ref + r * CALLS, tol + t)
            largest = r + t if largest is None else torch.maximum(largest, r + t)
            del q64, k64
        if len(members) > 1:
            n = CALLS * len(members)
            tol = tol + FP32_EPS * n * (n + 1) / 2 * largest
        L = case.layers[o]
        what = f'{name} layer {o} ({cls_of[o][1]}, {L})'
        worst = assert_close64(run.accs[o], ref, 0.0, tol, what, ACC_DIMS)
        key = (cls_of[o][1], L.dtype)
        RATIOS[key] = max(RATIOS[key], worst)


def _sm_count() -> int:
    return _native.device_info()['sm_count']


def _occupancy_case(inst: str, d: int, sm: int) -> Case:
    """One SIMT layer of 16 sm_count tiles for ``inst`` at head_dim ``d``: its grid is sm_count x the occupancy."""
    entry = {v: k for k, v in SIMT_KERNEL.items()}.get(inst, 'accumulate')
    tokens = 154 if inst == SIMT_LONG else TOKENS
    return Case(entry, 0, [Layer(TILE * 16 * sm - 64, 1, d, 'fp32', tokens, simt=True)], ())


def _trace_main(request: str):
    """Child process of :func:`_traced`: one call of each requested case under a CUDA activity trace; prints the
    traced ``(instance, grid.x)`` list as JSON. ``request``: ``{"occupancy": [[instance, d], ...]}`` or
    ``{"cases": [name, ...], "occ": [[instance, d, CTAs per SM], ...]}``."""
    req = json.loads(request)
    sm = _sm_count()
    if 'occupancy' in req:
        cases = [_occupancy_case(inst, d, sm) for inst, d in req['occupancy']]
    else:
        table = {(inst, d): n for inst, d, n in req['occ']}
        cases = [CASES[name](sm, lambda inst, d: table[inst, d]) for name in req['cases']]
    with tempfile.TemporaryDirectory() as tmp:
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for i, case in enumerate(cases):          # (the set-up kernels between the calls are not listed)
                run = Run(case, seed=i)
                torch.cuda.synchronize()
                run.call(case.flags)
                torch.cuda.synchronize()
                del run
        print(json.dumps(kernel_events(prof, tmp)))


def _traced(request: dict) -> List[Tuple[str, Optional[int]]]:
    """``_trace_main(request)`` in a fresh Python process (``tests.util.traced``)."""
    return traced('tests.test_launch_geometry_gpu', request)


# SIMT occupancy, measured: one launch of 16 sm_count tiles per (instance, largest head_dim), grid read from the trace
_OCC: Dict[Tuple[str, int], int] = {}


def _measure_occupancy(keys):
    sm = _sm_count()
    events = _traced({'occupancy': keys})
    assert [e[0] for e in events] == [inst for inst, _ in keys], events
    for (inst, d), (_, grid) in zip(keys, events):
        assert grid is not None, 'the profiler trace carries no grid for kernel events'
        assert grid % sm == 0 and grid < 16 * sm, (inst, d, grid)
        _OCC[inst, d] = grid // sm
        MEASURED[inst, d] = grid


@pytest.fixture(scope='module')
def occ() -> OccFn:
    """The measured SIMT occupancy of every (instance, head_dim) the cases ask for."""
    wanted = set()

    def record(inst, d):
        wanted.add((inst, d))
        return 1
    for build in CASES.values():
        plan(build(_sm_count(), record), _sm_count(), record)
    _measure_occupancy(sorted(wanted))
    yield lambda inst, d: _OCC[inst, d]
    print('\nmeasured SIMT grids (instance, largest head_dim: grid = SMs x CTAs per SM):')
    for (inst, d), grid in sorted(MEASURED.items()):
        print(f'  {inst:30s} d {d:3d}: {grid} = {_sm_count()} x {grid // _sm_count()}')
    if RATIOS:
        print('worst error / bound (instance, dtype):')
        for key in sorted(RATIOS):
            print(f'  {key[0]:42s} {key[1]:5s} {RATIOS[key]:.3e}')


LAUNCH_MODES = (('NO_PDL', _native.ACC_NO_PDL), ('PDL', 0), ('EARLY_LOADS', _native.ACC_EARLY_LOADS))


@pytest.mark.parametrize('name', CASE_NAMES)
def test_case(occ, name):
    sm = _sm_count()
    case = CASES[name](sm, occ)
    launches = plan(case, sm, occ)
    missing = set(case.tags) - regimes(case, launches)
    assert not missing, f'{name}: the case no longer reaches {sorted(missing)}'
    run = Run(case, seed=CASE_NAMES.index(name))
    torch.cuda.synchronize()                        # Q / K complete before the first launch (EARLY_LOADS)

    if case.entry == 'probs':
        before = _native.launch_count()
        run.call(0)
        torch.cuda.synchronize()
        assert _native.launch_count() - before == 1
        (L,), d = case.layers, run.descs[0]
        g = torch.cat([run.probs[:GUARD], run.probs[-GUARD:]])
        assert bool((g == SENTINEL).all()), f'{name}: probabilities written outside the output'
        got = run.probs[GUARD:-GUARD].view(L.prompts, L.heads, L.hw, TOKENS).transpose(-1, -2)
        q64, k64 = layer_views64(d, run.q[0], run.k[0])
        worst = assert_close64(got, desc_maps64(d, run.q[0], run.k[0]), 0.0,
                               probs_tolerance(q64, k64, float(d.scale), DTYPES[L.dtype]), name, ACC_DIMS)
        RATIOS[PROBS, L.dtype] = max(RATIOS[PROBS, L.dtype], worst)
        return

    if case.entry == 'steps':                        # a step slab holds what one call adds: the accumulator from 0
        run.reset()
        run.call(case.flags | _native.ACC_NO_PDL)
        once = [run.accs[i].clone().view(torch.int32) for i in range(len(case.layers))]
    reference = None
    for mode, extra in LAUNCH_MODES:
        run.reset()
        flags = case.flags | extra
        for _ in range(CALLS):                        # back to back: no synchronisation between the calls
            before = _native.launch_count()
            run.call(flags)
            assert _native.launch_count() - before == len(launches), f'{name} {mode}: launches'
        torch.cuda.synchronize()
        run.check_guards(f'{name} {mode}')
        if case.entry == 'steps':
            for i in range(len(case.layers)):
                assert torch.equal(run.slabs[i].view(torch.int32), once[i]), \
                    f'{name} {mode}: the step slab of layer {i} differs from one call from zero'
        bits = run.bits()
        if reference is None:
            _check_float64(run, launches, name)
            reference = bits
            if case.entry == 'range':
                for i in range(len(case.layers)):
                    assert torch.equal(run.slabs[i].view(torch.int32), run.accs[i].view(torch.int32)), \
                        f'{name}: the range slab of layer {i} differs from its accumulator'
        else:
            for j, (a, b) in enumerate(zip(bits, reference)):
                assert torch.equal(a, b), f'{name}: {mode} differs from NO_PDL in buffer {j}'
    # the same layers, one call per launch of the plan
    run.reset()
    for _ in range(CALLS):
        for l in launches:
            run.call(case.flags, [e['index'] for e in l.layers])
    torch.cuda.synchronize()
    run.check_guards(f'{name} pack by pack')
    for j, (a, b) in enumerate(zip(run.bits(), reference)):
        assert torch.equal(a, b), f'{name}: pack by pack differs from one call in buffer {j}'


def test_every_case_runs_the_launches_its_plan_names(occ):
    """One torch.profiler CUDA trace over one call of every case: the accumulate / attention_probs kernels it lists,
    in order, are the instances and grids plan() names."""
    sm = _sm_count()
    runs = [(name, [(l.instance, l.grid) for l in plan(CASES[name](sm, occ), sm, occ)]) for name in CASE_NAMES]
    got = _traced({'cases': CASE_NAMES, 'occ': [[inst, d, n] for (inst, d), n in sorted(_OCC.items())]})
    want = [x for _, launches in runs for x in launches]
    if got != want:
        pos, lines = 0, []
        for name, launches in runs:
            traced = got[pos:pos + len(launches)]
            if traced != launches:
                lines.append(f'{name}: planned {launches}, traced {traced}')
            pos += len(launches)
        raise AssertionError('launches differ from the plan:\n' + '\n'.join(lines[:20]))
