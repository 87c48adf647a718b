"""daam_accumulate_joint against float64 at every pack, tile-walk, staging and edge geometry it accepts.

The host side sorts a call's layers into three kernel classes, issued in the order fp16
(``accumulate_joint_mma_kernel<false>``), bf16 (``accumulate_joint_mma_kernel<true>``), fp32
(``accumulate_joint_simt_kernel``), each in call order, and closes a class's pack at 64 layers or when a layer's
accumulator shares bytes with one already in it (slabs that only touch do not close it). Each pack is one launch of
``min(tiles, SMs x occupancy)`` CTAs, the occupancy the runtime reports for the shared memory of the pack's largest
head dim; CTA b takes tiles b, b + grid, ..., and ``decode_tile`` moves its layer index forward to each tile.

:func:`plan` restates the packing and each launch's instance and grid, :func:`walk` every CTA's tiles down to
(layer, sample, head, pixel0), :func:`regimes` labels what a case reaches. Every case asserts the regimes it names;
``tests/test_joint_geometry_host.py`` checks without a GPU that they are reached at several SM counts and occupancies
and that the walks take every tile once.

Every case runs through ``ops.make_joint_desc`` and the C ABI, from accumulators of random positive values, and is
checked

* against float64: every element within ``acc0 + ref +- (bound + m 2^-24 |acc0 + ref|)``, ``bound`` the header's
  (``tests.joint64.exp_and_bound``), summed over the m layers that add into the element;
* for stray writes: sentinel runs sit around every accumulator region; Q / K / lse storage the descriptors do not
  address is NaN, so a stray read shows in the values;
* for its launches: ``launch_count()`` moves by the planned launches of every call, and one profiler trace over every
  case lists the instances and grids the plans name, in order;
* bit for bit: one call, one call per planned launch, one call per layer in the documented order, a repeat, and two
  rounds back to back without a synchronisation against the same rounds synchronised.

The occupancy per (instance, largest head dim) is measured from the traced grid of one launch of 16 SMs + 1 tiles.
The measured grids and the worst error-to-bound ratio per instance are printed at the end (``-s``)."""
import collections
import json
import tempfile
from dataclasses import dataclass, replace
from typing import Callable, Dict, List, NamedTuple, Optional, Tuple

import pytest
import torch

from daam_b200 import _native, ops
from tests.joint64 import exp_and_bound
from tests.util import kernel_events, traced

pytestmark = pytest.mark.gpu
DEV = 'cuda'

MMA_PIXELS, SIMT_PIXELS = 64, 128      # kMmaPixels, kSimtPixels: pixels per tile
MAX_LAYERS = 64                        # DAAM_JOINT_MAX_LAYERS
CLASS_ORDER = ('fp16', 'bf16', 'fp32')
INSTANCE = {'fp16': 'accumulate_joint_mma_kernel<false>', 'bf16': 'accumulate_joint_mma_kernel<true>',
            'fp32': 'accumulate_joint_simt_kernel'}
INSTANCES = tuple(INSTANCE.values())
DTYPES = {'fp32': torch.float32, 'fp16': torch.float16, 'bf16': torch.bfloat16}
TAGGED_DS = (8, 24, 136, 248, 16, 64, 128, 256)     # d mod 16 = 8 (a zero-padded k step) and d mod 16 = 0


# ---- the case description ---------------------------------------------------------------------------------------

@dataclass
class Layer:
    """One layer call: ``samples`` kept samples x ``heads`` kept heads, ``tokens`` context rows, ``hw`` pixels."""
    hw: int
    tokens: int = 77
    d: int = 64
    dtype: str = 'bf16'
    samples: int = 1
    heads: int = 1
    keep: str = 'cfg'         # 'cfg': a [uncond x N, cond x N] batch; 'lone': one sample, the upper half of 2 heads
                              # heads (cond_half's head offset); 'whole': every sample and head (whole_batch)
    text_first: bool = False  # [context, image] sequences (FLUX)
    stage: str = 'vec'        # 'vec': 16-byte aligned; 'q+2' / 'k+2': that base 2 bytes off; 'pad4': [B, L, H, d + 4]
    lse: str = 'contig'       # 'contig' [B, H, L]; 'pad32' [B, H, 32 ceil(L / 32)]; 'pixel' [B, L, H]
    at: Optional[Tuple[int, int]] = None    # accumulator at earlier layer j's accumulator + this many floats
    seed: Optional[int] = None              # operands and acc0 from this seed (twins share it), else the index

    @property
    def tile(self) -> int:
        return SIMT_PIXELS if self.dtype == 'fp32' else MMA_PIXELS

    @property
    def tiles(self) -> int:
        return -(-self.hw // self.tile) * self.heads * self.samples

    @property
    def n(self) -> int:
        return self.samples * self.heads * self.tokens * self.hw

    @property
    def total_heads(self) -> int:
        return 2 * self.heads if self.keep == 'lone' else self.heads


@dataclass
class Case:
    layers: List[Layer]
    tags: Tuple[str, ...]
    calls: Optional[List[List[int]]] = None     # layer indices of each call, in order; default one call of all

    def call_list(self) -> List[List[int]]:
        return self.calls if self.calls is not None else [list(range(len(self.layers)))]

    def span(self, i: int) -> Tuple[int, int, int]:
        """``(root layer, first float, end)`` of layer i's accumulator within its root's region."""
        L = self.layers[i]
        root, start = (i, 0) if L.at is None else L.at
        return root, start, start + L.n

    def overlap(self, i: int, j: int) -> bool:
        (ri, si, ei), (rj, sj, ej) = self.span(i), self.span(j)
        return ri == rj and si < ej and sj < ei


@dataclass
class Launch:
    cls: str
    instance: str
    G: int                      # SMs x occupancy of the pack's largest head dim
    grid: int
    dmax: int
    layers: List[dict]          # index (into the case), tile_begin, tiles
    close: str                  # 'full', 'overlap' or 'end'
    closer: Optional[int] = None    # the layer that closed it

    @property
    def total_tiles(self) -> int:
        return sum(e['tiles'] for e in self.layers)


OccFn = Callable[[str, int], int]     # (instance, largest head dim of the pack) -> CTAs per SM


# ---- the host side, restated --------------------------------------------------------------------------------------

def _launch(case: Case, cls: str, members: List[int], close: str, sm: int, occ: OccFn,
            closer: Optional[int] = None) -> Launch:
    table, tb = [], 0
    for i in members:
        table.append(dict(index=i, tile_begin=tb, tiles=case.layers[i].tiles))
        tb += case.layers[i].tiles
    dmax = max(case.layers[i].d for i in members)
    G = sm * occ(INSTANCE[cls], dmax)
    return Launch(cls, INSTANCE[cls], G, min(G, tb), dmax, table, close, closer)


def plan_call(case: Case, idx: List[int], sm: int, occ: OccFn) -> List[Launch]:
    """The launches of one call of the layers ``idx``, in order."""
    out = []
    for cls in CLASS_ORDER:
        pack: List[int] = []
        for i in idx:
            if case.layers[i].dtype != cls:
                continue
            why = 'full' if len(pack) == MAX_LAYERS else 'overlap' if any(case.overlap(i, j) for j in pack) else None
            if why:
                out.append(_launch(case, cls, pack, why, sm, occ, i))
                pack = []
            pack.append(i)
        if pack:
            out.append(_launch(case, cls, pack, 'end', sm, occ))
    return out


def plan(case: Case, sm: int, occ: OccFn) -> List[List[Launch]]:
    """Per call of the case, its launches."""
    return [plan_call(case, idx, sm, occ) for idx in case.call_list()]


def documented_order(case: Case, idx: List[int]) -> List[int]:
    """The order in which a call applies its layers: fp16, bf16, fp32, each in call order."""
    return [i for cls in CLASS_ORDER for i in idx if case.layers[i].dtype == cls]


class Tile(NamedTuple):
    tile: int
    layer: int                  # index into the case
    sample: int
    head: int
    pixel0: int
    passed: int                 # layers decode_tile stepped over entirely to reach this tile


def walk(case: Case, launch: Launch) -> List[List[Tile]]:
    """Per CTA, its tiles in order (the tile loop and decode_tile)."""
    P = launch.layers
    out = []
    for b in range(launch.grid):
        li, tiles = 0, []
        for t in range(b, launch.total_tiles, launch.grid):
            start = li
            while li + 1 < len(P) and t >= P[li + 1]['tile_begin']:
                li += 1
            e = P[li]
            L = case.layers[e['index']]
            local = t - e['tile_begin']
            tph = -(-L.hw // L.tile)
            rest = local // tph
            passed = max(0, li - start - 1) if tiles else li
            tiles.append(Tile(t, e['index'], rest // L.heads, rest % L.heads, (local % tph) * L.tile, passed))
        out.append(tiles)
    return out


# ---- regimes --------------------------------------------------------------------------------------------------------

LABELS = {'1': lambda G: 1, 'G-1': lambda G: G - 1, 'G': lambda G: G, 'G+1': lambda G: G + 1,
          '2G+1': lambda G: 2 * G + 1}


def _layer_tags(inst: str, L: Layer) -> set:
    tags = {f'{inst}: {L.samples} samples', f'{inst}: keep {L.keep}',
            f'{inst}: {"text" if L.text_first else "image"} first'}
    if L.lse != 'pixel' or L.total_heads > 1:            # a pixel stride of 1 is the contiguous layout
        tags.add(f'{inst}: lse {L.lse}')
    if L.d in TAGGED_DS:
        tags.add(f'{inst}: d = {L.d}')
    if L.tokens in (1, 1024):
        tags.add(f'{inst}: tokens = {L.tokens}')
    if L.dtype == 'fp32':
        if L.hw % 128 in (0, 1, 64, 127):
            tags.add(f'{inst}: hw mod 128 = {L.hw % 128}')
        if L.tokens % 32 in (0, 1, 31):
            tags.add(f'{inst}: tokens mod 32 = {L.tokens % 32}')
        if L.tokens % 8:
            tags.add(f'{inst}: tokens mod 8 != 0')
        return tags
    tags.add(f'{inst}: stage {L.stage}')
    if L.hw % 64 in (0, 1, 63):
        tags.add(f'{inst}: hw mod 64 = {L.hw % 64}')
    if L.hw in (1, 2, 17):
        tags.add(f'{inst}: hw = {L.hw}')
    tags.add(f'{inst}: accumulator ' + ('pairs' if L.hw % 2 == 0 else 'scalar'))
    if L.tokens % 64 in (0, 1, 16, 17, 48, 63):
        tags.add(f'{inst}: tokens mod 64 = {L.tokens % 64}')
    return tags


def regimes(case: Case, calls: List[List[Launch]]) -> set:
    """The regimes the calls of ``case`` reach, as the tags the cases name."""
    tags = set()
    same = lambda i, j: case.span(i) == case.span(j)
    for idx, launches in zip(case.call_list(), calls):
        dts = [case.layers[i].dtype for i in idx]
        if set(dts) == set(CLASS_ORDER) and sum(1 for a, b in zip(dts, dts[1:]) if a != b) >= 3:
            tags.add('three classes interleaved')
        for a, b, c in zip(idx, idx[1:], idx[2:]):
            if [case.layers[x].dtype for x in (a, b, c)] == ['fp16', 'bf16', 'fp16'] and same(a, b) and same(b, c):
                tags.add('[fp16, bf16, fp16] into one slab')
        for i in idx:
            for j in idx:
                Li, Lj = case.layers[i], case.layers[j]
                if Li.dtype != Lj.dtype and same(i, j):
                    tags.add('one slab in two classes')
                if (Li.dtype, Lj.dtype) == ('fp16', 'bf16') and case.span(i)[0] != case.span(j)[0]:
                    tags.add('fp16 and bf16 into different slabs')
        sizes = collections.defaultdict(list)
        for l in launches:
            inst = l.instance
            sizes[inst].append((len(l.layers), l.close))
            for label, f in LABELS.items():
                if l.total_tiles == f(l.G):
                    tags.add(f'{inst}: tiles {label}')
            for w in walk(case, l):
                if len({t.layer for t in w}) >= 3:
                    tags.add(f'{inst}: CTA spans >= 3 layers')
                if any(t.passed >= 2 for t in w[1:]):
                    tags.add(f'{inst}: decode passes >= 2 layers')
                for a, b, c in zip(w, w[1:], w[2:]):
                    if case.layers[b.layer].tiles == 1 and a.layer != b.layer != c.layer and \
                            case.layers[a.layer].tiles > 1 and case.layers[c.layer].tiles > 1:
                        tags.add(f'{inst}: one-tile layer between two large layers')
            members = [e['index'] for e in l.layers]
            if {8, 256} <= {case.layers[i].d for i in members}:
                tags.add(f'{inst}: pack with d 8 and d 256')
            for i in members:
                tags |= _layer_tags(inst, case.layers[i])
                for j in members:
                    ri, si, ei = case.span(i)
                    rj, sj, _ = case.span(j)
                    if ri == rj and ei == sj:
                        tags.add(f'{inst}: touching slabs share a launch')
            if l.close == 'overlap':
                if len(members) in (1, 63):
                    tags.add(f'{inst}: overlap close at position {len(members)}')
                _, s, _ = case.span(l.closer)
                for j in members:
                    if case.overlap(l.closer, j):
                        diff = s - case.span(j)[1]
                        if diff > 0 and diff % case.layers[j].hw == 0:
                            tags.add(f'{inst}: partial overlap at a row boundary')
                        if diff == 4:
                            tags.add(f'{inst}: partial overlap 16 bytes in')
        for inst, s in sizes.items():
            if s == [(64, 'end')]:
                tags.add(f'{inst}: 64 layers, one launch')
            if s == [(64, 'full'), (1, 'end')]:
                tags.add(f'{inst}: 65 layers, 64 + 1')
    for inst in INSTANCES:       # calls of one kernel whose largest head dims go 64, 256, 64, every grid G
        seq = [(l[0].dmax, l[0].grid == l[0].G) for l in calls if len(l) == 1 and l[0].instance == inst]
        if any(seq[k:k + 3] == [(64, True), (256, True), (64, True)] for k in range(len(seq))):
            tags.add(f'{inst}: calls at d 64, 256, 64')
    return tags


# ---- the cases --------------------------------------------------------------------------------------------------------

def _filler(cls: str, tiles: int, tokens: int = 17, d: int = 64, **kw) -> Layer:
    """One layer of one sample and head with ``tiles`` tiles, its last tile partial."""
    tile = SIMT_PIXELS if cls == 'fp32' else MMA_PIXELS
    return Layer(tile * tiles - 5, tokens, d, cls, **kw)


def _grid(cls: str, label: str):
    """``label`` tiles relative to the grid of the class's kernel at d = 64. From G + 1 on, CTA 0 takes tile 0 of a
    large layer, then tile G of the last of three one-tile layers (passing the other two), then at 2G + 1 tile 2G of
    a second large layer."""
    def build(sm: int, occ: OccFn) -> Case:
        inst = INSTANCE[cls]
        G = sm * occ(inst, 64)
        T = LABELS[label](G)
        if label == '1':
            layers = [Layer(37 if cls != 'fp32' else 100, 65, 64, cls, keep='whole')]
        elif label in ('G-1', 'G'):
            head = Layer(64 if cls != 'fp32' else 128, 33, 64, cls, samples=2, heads=2)
            layers = [head, _filler(cls, T - head.tiles)]
        else:
            layers = [_filler(cls, G - 2, text_first=True)] + [Layer(40, 33, 64, cls, keep='lone') for _ in range(3)]
            if label == '2G+1':
                layers.append(_filler(cls, G, samples=1, keep='whole'))
        tags = [f'{inst}: tiles {label}']
        if label in ('G+1', '2G+1'):
            tags.append(f'{inst}: decode passes >= 2 layers')
        if label == '2G+1':
            tags += [f'{inst}: CTA spans >= 3 layers', f'{inst}: one-tile layer between two large layers']
        return Case(layers, tuple(tags))
    return build


HW16 = (128, 129, 127, 1, 2, 17)                       # hw mod 64 = 0, 1, 63; hw = 1, 2, 17
HW32 = (256, 257, 192, 255)                            # hw mod 128 = 0, 1, 64, 127
TOKENS16 = (64, 65, 80, 81, 112, 127, 1, 1024)         # tokens mod 64 = 0, 1, 16, 17, 48, 63
TOKENS32 = (32, 33, 63, 1, 1024)                       # tokens mod 32 = 0, 1, 31; 33 and 63 not multiples of 8
STAGES = ('vec', 'q+2', 'k+2', 'pad4')
KEEPS = ('cfg', 'lone', 'whole')
LSES = ('contig', 'pad32', 'pixel')


def _shapes(cls: str):
    """Eight layers in one pack: every head dim, pixel count and context length of the class's lists, 1-3 kept
    samples, each keep mode, image- and text-first, every staging path and lse layout."""
    def build(sm: int, occ: OccFn) -> Case:
        hws, toks = (HW32, TOKENS32) if cls == 'fp32' else (HW16, TOKENS16)
        layers = []
        for i, d in enumerate(TAGGED_DS):
            keep, lse = KEEPS[i % 3], LSES[i % 3]
            layers.append(Layer(hws[i % len(hws)], toks[i % len(toks)], d, cls,
                                samples=1 if keep == 'lone' else 1 + (i // 3) % 3,
                                heads=2 if lse == 'pixel' else 1 + i % 2, keep=keep, text_first=i % 2 == 1,
                                stage=STAGES[i % 4], lse=lse))
        inst = INSTANCE[cls]
        tags = set()
        for L in layers:
            tags |= _layer_tags(inst, L)
        return Case(layers, tuple(sorted(tags)) + (f'{inst}: pack with d 8 and d 256',))
    return build


def _staging(cls: str):
    """Four layers of the same operands and acc0, staged by 16-byte loads and by each scalar path: the same bits."""
    def build(sm: int, occ: OccFn) -> Case:
        layers = [Layer(129, 81, 24, cls, samples=2, heads=2, stage=s, seed=0) for s in STAGES]
        return Case(layers, tuple(f'{INSTANCE[cls]}: stage {s}' for s in STAGES))
    return build


def _pack(n: int):
    """``n`` one-tile layers of every class, the classes interleaved."""
    def build(sm: int, occ: OccFn) -> Case:
        layers = [Layer(30 + r % 7, 17, (8, 64)[r % 2], cls) for r in range(n) for cls in CLASS_ORDER]
        what = '64 layers, one launch' if n == 64 else '65 layers, 64 + 1'
        return Case(layers, tuple(f'{i}: {what}' for i in INSTANCES) + ('three classes interleaved',))
    return build


def _overlap(position: int):
    """Layer ``position`` of each class's pack adds into the accumulator of the class's first layer."""
    def build(sm: int, occ: OccFn) -> Case:
        layers = []
        for cls in CLASS_ORDER:
            base = len(layers)
            layers += [Layer(40, 17, 8, cls) for _ in range(position)]
            layers.append(replace(layers[base], d=24, at=(base, 0)))
            layers.append(Layer(40, 17, 8, cls))
        return Case(layers, tuple(f'{i}: overlap close at position {position}' for i in INSTANCES))
    return build


def _partial_overlaps(sm: int, occ: OccFn) -> Case:
    """Per class: B starts one token row into A (closes A's pack), C and D touch (share a launch), E starts 16 bytes
    into C (closes it)."""
    layers = []
    for cls in CLASS_ORDER:
        a = len(layers)
        A = Layer(64, 5, 64, cls)
        C = Layer(64, 3, 64, cls)
        layers += [A, replace(A, at=(a, 64)), C, replace(C, at=(a + 2, C.n)), replace(C, at=(a + 2, 4))]
    tags = []
    for i in INSTANCES:
        tags += [f'{i}: partial overlap at a row boundary', f'{i}: partial overlap 16 bytes in',
                 f'{i}: touching slabs share a launch']
    return Case(layers, tuple(tags))


def _class_order_one_slab(sm: int, occ: OccFn) -> Case:
    """fp16, bf16, fp16 and fp32 layers into one slab: applied fp16, fp16, bf16, fp32 (four launches)."""
    X = Layer(200, 70, 64, 'fp16', samples=2)
    layers = [X, replace(X, dtype='bf16', d=128, at=(0, 0)), replace(X, d=24, at=(0, 0)),
              replace(X, dtype='fp32', d=40, at=(0, 0))]
    return Case(layers, ('[fp16, bf16, fp16] into one slab', 'one slab in two classes', 'three classes interleaved'))


def _class_split(sm: int, occ: OccFn) -> Case:
    """An fp16 and a bf16 layer into different slabs: two launches."""
    return Case([Layer(200, 70, 64, 'fp16'), Layer(136, 70, 64, 'bf16')], ('fp16 and bf16 into different slabs',))


def _dims_64_256_64(sm: int, occ: OccFn) -> Case:
    """Per kernel, three calls of one layer at d = 64, 256, 64, each with more tiles than either grid: the kernel's
    shared-memory attribute only rises, and the grid still follows each call's own head dim."""
    layers = []
    for cls in CLASS_ORDER:
        inst = INSTANCE[cls]
        T = max(sm * occ(inst, 64), sm * occ(inst, 256)) + 1
        layers += [_filler(cls, T, 1, d) for d in (64, 256, 64)]
    return Case(layers, tuple(f'{i}: calls at d 64, 256, 64' for i in INSTANCES),
                calls=[[i] for i in range(len(layers))])


CASES: Dict[str, Callable[[int, OccFn], Case]] = {
    'dims-64-256-64': _dims_64_256_64,         # first, so that a fresh process raises the attribute here
    **{f'grid-{label}-{cls}': _grid(cls, label) for cls in CLASS_ORDER for label in LABELS},
    **{f'shapes-{cls}': _shapes(cls) for cls in CLASS_ORDER},
    **{f'staging-{cls}': _staging(cls) for cls in ('fp16', 'bf16')},
    'pack-64': _pack(64),
    'pack-65': _pack(65),
    'overlap-1': _overlap(1),
    'overlap-63': _overlap(63),
    'partial-overlaps': _partial_overlaps,
    'class-order-one-slab': _class_order_one_slab,
    'class-split': _class_split,
}
CASE_NAMES = list(CASES)


# ---- running a case ---------------------------------------------------------------------------------------------------

GUARD = 64                   # sentinel floats before and after every accumulator region
SENTINEL = 12345.0
RATIOS: Dict[str, float] = collections.defaultdict(float)
MEASURED: Dict[Tuple[str, int], int] = {}


def _acc0(n: int, seed: int) -> torch.Tensor:
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.rand(n, generator=g, device=DEV) * (3 / 64) + 1 / 64


def _operands(L: Layer, seed: int):
    """The layer's q, k and lse as ``make_joint_desc`` takes them, in NaN-filled storage of its layout (NaN wherever
    the kernel must not read), and the kept operands ``[N, H, hw, d]``, ``[N, H, T, d]``, ``[N, H, hw]``."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    N, H, hw, T, d = L.samples, L.heads, L.hw, L.tokens, L.d
    B, s0, h0 = {'cfg': (2 * N, N, 0), 'lone': (1, 0, H), 'whole': (N, 0, 0)}[L.keep]
    Ht, S, dt = L.total_heads, hw + T, DTYPES[L.dtype]
    img, ctx = (slice(T, S), slice(0, T)) if L.text_first else (slice(0, hw), slice(hw, S))

    def store(shift: int) -> torch.Tensor:
        if L.stage == 'pad4':
            return torch.full((B, S, Ht, d + 4), float('nan'), dtype=dt, device=DEV)[..., :d].permute(0, 2, 1, 3)
        return torch.full((shift + B * Ht * S * d,), float('nan'), dtype=dt, device=DEV)[shift:].view(B, Ht, S, d)

    q, k = store(1 if L.stage == 'q+2' else 0), store(1 if L.stage == 'k+2' else 0)
    qk = (torch.randn(N, H, hw, d, generator=g, device=DEV) * 1.5).to(dt)
    kk = torch.randn(N, H, T, d, generator=g, device=DEV).to(dt)
    q[s0:s0 + N, h0:h0 + H, img] = qk
    k[s0:s0 + N, h0:h0 + H, ctx] = kk
    scale = d ** -0.5
    lk = torch.logsumexp(torch.einsum('nhid,nhjd->nhij', qk.double(), kk.double()) * scale, -1).float()
    if L.lse == 'pixel':
        lse = torch.full((B, S, Ht), float('nan'), device=DEV).permute(0, 2, 1)
    else:
        lse = torch.full((B, Ht, -(-S // 32) * 32 if L.lse == 'pad32' else S), float('nan'), device=DEV)
    lse[s0:s0 + N, h0:h0 + H, img] = lk
    return (q, k, lse, scale), (qk, kk, lk)


class Run:
    """A case's operands, descriptors and accumulator pool on the device."""

    def __init__(self, case: Case, seed: int):
        self.case = case
        n = len(case.layers)
        self.roots = sorted({case.span(i)[0] for i in range(n)})
        size = {r: max(case.span(i)[2] for i in range(n) if case.span(i)[0] == r) for r in self.roots}
        self.off, pos = {}, GUARD
        offs = self.off
        for r in self.roots:
            offs[r] = pos
            pos = -(-(pos + size[r] + GUARD) // 4) * 4
        self.buf = torch.full((pos,), SENTINEL, device=DEV)
        self.inside = torch.zeros(pos, dtype=torch.bool, device=DEV)
        self.region = {}
        for r in self.roots:
            L = case.layers[r]
            self.inside[offs[r]:offs[r] + size[r]] = True
            self.region[r] = self.buf[offs[r]:offs[r] + size[r]]
            self.region[r].copy_(_acc0(size[r], seed * 1000 + 500 + (r if L.seed is None else L.seed)))
        self.init = self.buf.clone()
        self.keep, self.descs = [], []
        for i, L in enumerate(case.layers):
            (q, k, lse, scale), kept = _operands(L, seed * 1000 + (i if L.seed is None else L.seed))
            root, s, e = case.span(i)
            acc = self.region[root][s:e].view(L.samples, L.heads, L.tokens, L.hw)
            self.descs.append(ops.make_joint_desc(q, k, lse, L.hw, acc, L.total_heads, scale,
                                                  text_first=L.text_first, whole_batch=L.keep == 'whole'))
            self.keep.append((q, k, lse, scale, kept))

    def reset(self):
        self.buf.copy_(self.init)

    def call(self, idx: List[int]):
        _native.accumulate_joint([self.descs[i] for i in idx], torch.cuda.current_stream().cuda_stream)

    def check_guards(self, what: str):
        assert bool((self.buf[~self.inside] == SENTINEL).all()), f'{what}: a write outside the accumulators'

    def bits(self) -> torch.Tensor:
        return self.buf.clone().view(torch.int32)

    def check_float64(self, name: str):
        """Every element within acc0 + sum of its layers' float64 values +- (their bounds + m 2^-24 |that sum|)."""
        case = self.case
        for r in self.roots:
            members = [i for i in range(len(case.layers)) if case.span(i)[0] == r]
            expect = self.init[self.off[r]:self.off[r] + self.region[r].numel()].double()
            bound, m = torch.zeros_like(expect), torch.zeros_like(expect)
            for i in members:
                _, s, e = case.span(i)
                qk, kk, lk = self.keep[i][4]
                ref, b = exp_and_bound(qk, kk, lk, self.keep[i][3])
                expect[s:e] += ref.flatten()
                bound[s:e] += b.flatten()
                m[s:e] += 1
            tol = bound + m * 2.0 ** -24 * (expect + bound)
            err = (self.region[r].double() - expect).abs()
            ratio = err / tol
            worst = float(ratio.max())
            insts = {INSTANCE[case.layers[i].dtype] for i in members}
            if not worst <= 1.0:
                j = int(ratio.argmax())
                raise AssertionError(f'{name}: region of layer {r} ({sorted(insts)}): element {j} got '
                                     f'{float(self.region[r][j]):.9e}, want {float(expect[j]):.9e} '
                                     f'+- {float(tol[j]):.3e} ({worst:.2f} x)')
            if len(insts) == 1:
                (inst,) = insts
                RATIOS[inst] = max(RATIOS[inst], worst)


def _sm_count() -> int:
    return _native.device_info()['sm_count']


def _occupancy_case(inst: str, d: int, sm: int) -> Case:
    cls = {v: k for k, v in INSTANCE.items()}[inst]
    return Case([_filler(cls, 16 * sm + 1, 1, d)], ())


def _trace_main(request: str):
    """Child process of :func:`tests.util.traced`: each requested case's calls under a CUDA activity trace; prints the
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
                for idx in case.call_list():
                    run.call(idx)
                torch.cuda.synchronize()
                del run
        print(json.dumps(kernel_events(prof, tmp)))


_OCC: Dict[Tuple[str, int], int] = {}


@pytest.fixture(scope='module')
def occ() -> OccFn:
    """The measured occupancy of every (instance, largest head dim) the cases ask for."""
    sm = _sm_count()
    wanted = set()

    def record(inst, d):
        wanted.add((inst, d))
        return 1
    for build in CASES.values():
        plan(build(sm, record), sm, record)
    keys = sorted(wanted)
    events = traced('tests.test_joint_geometry_gpu', {'occupancy': keys})
    assert [e[0] for e in events] == [inst for inst, _ in keys], events
    for (inst, d), (_, grid) in zip(keys, events):
        assert grid is not None, 'the profiler trace carries no grid for kernel events'
        assert grid % sm == 0 and grid <= 16 * sm, (inst, d, grid)
        _OCC[inst, d] = grid // sm
        MEASURED[inst, d] = grid
    yield lambda inst, d: _OCC[inst, d]
    print('\nmeasured grids (instance, largest head dim: grid = SMs x CTAs per SM):')
    for (inst, d), grid in sorted(MEASURED.items()):
        print(f'  {inst:38s} d {d:3d}: {grid} = {sm} x {grid // sm}')
    if RATIOS:
        print('worst error / bound per instance:')
        for inst in sorted(RATIOS):
            print(f'  {inst:38s} {RATIOS[inst]:.3e}')


@pytest.mark.parametrize('name', CASE_NAMES)
def test_case(occ, name):
    sm = _sm_count()
    case = CASES[name](sm, occ)
    calls = plan(case, sm, occ)
    missing = set(case.tags) - regimes(case, calls)
    assert not missing, f'{name}: the case no longer reaches {sorted(missing)}'
    run = Run(case, seed=CASE_NAMES.index(name))
    torch.cuda.synchronize()

    def rounds(n=1, sync=False):
        for _ in range(n):
            for idx, launches in zip(case.call_list(), calls):
                before = _native.launch_count()
                run.call(idx)
                assert _native.launch_count() - before == len(launches), f'{name}: launches of call {idx}'
            if sync:
                torch.cuda.synchronize()

    run.reset()
    rounds()
    torch.cuda.synchronize()
    run.check_guards(name)
    run.check_float64(name)
    want = run.bits()
    for i, L in enumerate(case.layers):          # twins: the same operands and acc0 give the same bits
        for j in range(i):
            if L.seed is not None and replace(L, stage='vec') == replace(case.layers[j], stage='vec'):
                a, b = (run.region[x].view(torch.int32) for x in (i, j))
                assert torch.equal(a, b), f'{name}: layers {j} ({case.layers[j].stage}) and {i} ({L.stage}) differ'

    def same(what: str):
        torch.cuda.synchronize()
        run.check_guards(f'{name} {what}')
        assert torch.equal(run.bits(), want), f'{name}: {what} differs from one call'

    run.reset()
    rounds()
    same('a repeat')
    run.reset()
    for idx, launches in zip(case.call_list(), calls):
        for l in launches:
            run.call([e['index'] for e in l.layers])
    same('one call per planned launch')
    run.reset()
    for idx in case.call_list():
        for i in documented_order(case, idx):
            run.call([i])
    same('one call per layer in the documented order')
    run.reset()
    rounds(2)
    torch.cuda.synchronize()
    twice = run.bits()
    run.reset()
    rounds(2, sync=True)
    assert torch.equal(run.bits(), twice), f'{name}: back-to-back rounds differ from synchronised ones'


def test_every_case_runs_the_launches_its_plan_names(occ):
    """One torch.profiler CUDA trace over the calls of every case: the joint kernels it lists, in order, are the
    instances and grids plan() names."""
    sm = _sm_count()
    runs = [(name, [(l.instance, l.grid) for c in plan(CASES[name](sm, occ), sm, occ) for l in c])
            for name in CASE_NAMES]
    got = traced('tests.test_joint_geometry_gpu',
                 {'cases': CASE_NAMES, 'occ': [[inst, d, n] for (inst, d), n in sorted(_OCC.items())]})
    want = [x for _, launches in runs for x in launches]
    if got != want:
        pos, lines = 0, []
        for name, launches in runs:
            seen = got[pos:pos + len(launches)]
            if seen != launches:
                lines.append(f'{name}: planned {launches}, traced {seen}')
            pos += len(launches)
        raise AssertionError('launches differ from the plan:\n' + '\n'.join(lines[:20]))


def test_offsets_past_2_31():
    """One bf16 slab of 513 (sample, head) blocks of 1024 x 4096: block 512 starts at element 2^31. The blocks on both
    sides of that boundary against float64, the guards around the slab."""
    if torch.cuda.mem_get_info()[0] < 12 * 2 ** 30:
        pytest.skip('needs 12 GB of free device memory')
    N, T, hw, d = 513, 1024, 4096, 8
    blk = T * hw
    assert (N - 1) * blk == 2 ** 31
    g = torch.Generator(device=DEV).manual_seed(7)
    q = (torch.randn(N, 1, hw + T, d, generator=g, device=DEV) * 1.5).bfloat16()
    k = torch.randn(N, 1, hw + T, d, generator=g, device=DEV).bfloat16()
    scale = d ** -0.5
    lse = torch.empty(N, 1, hw, device=DEV)
    for s in range(0, N, 64):                    # any fp32 lse will do; this one keeps every value <= 1
        lse[s:s + 64] = torch.logsumexp(torch.einsum('nhid,nhjd->nhij', q[s:s + 64, :, :hw].float(),
                                                     k[s:s + 64, :, hw:].float()) * scale, -1)
    buf = torch.full((N * blk + 2 * GUARD,), SENTINEL, device=DEV)
    acc = buf[GUARD:GUARD + N * blk]
    acc.uniform_(1 / 64, 1 / 16, generator=g)
    init = [acc[b * blk:(b + 1) * blk].clone() for b in (N - 2, N - 1)]
    desc = ops.make_joint_desc(q, k, lse, hw, acc.view(N, 1, T, hw), 1, scale, whole_batch=True)
    before = _native.launch_count()
    _native.accumulate_joint([desc], torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert _native.launch_count() - before == 1
    assert bool((buf[:GUARD] == SENTINEL).all()) and bool((buf[-GUARD:] == SENTINEL).all())
    for b, a0 in zip((N - 2, N - 1), init):
        ref, bound = exp_and_bound(q[b:b + 1, :, :hw], k[b:b + 1, :, hw:], lse[b:b + 1], scale)
        expect = a0.double() + ref.flatten()
        tol = bound.flatten() + 2.0 ** -24 * (expect + bound.flatten())
        err = (acc[b * blk:(b + 1) * blk].double() - expect).abs()
        assert bool((err <= tol).all()), f'block {b}: worst {float((err / tol).max()):.2f} x the bound'
    del buf, acc


# ---- make_joint_desc's shape checks ---------------------------------------------------------------------------------

def _desc_args(B=2, H=2, hw=64, T=17, d=64):
    q = torch.zeros(B, H, hw + T, d, dtype=torch.bfloat16, device=DEV)
    k = torch.zeros_like(q)
    lse = torch.zeros(B, H, hw + T, device=DEV)
    acc = torch.zeros(B // 2, H, T, hw, device=DEV)
    return dict(q=q, k=k, lse=lse, n_image=hw, acc=acc, heads=H, scale=0.125)


@pytest.mark.parametrize('change, text', [
    (dict(k=torch.zeros(4, 2, 81, 64, dtype=torch.bfloat16)), 'one batch size'),
    (dict(lse=torch.zeros(4, 2, 81)), 'one batch size'),
    (dict(q=torch.zeros(2, 1, 81, 64, dtype=torch.bfloat16)), 'at least 2 heads'),
    (dict(k=torch.zeros(2, 1, 81, 64, dtype=torch.bfloat16)), 'at least 2 heads'),
    (dict(lse=torch.zeros(2, 1, 81)), 'at least 2 heads'),
    (dict(k=torch.zeros(2, 2, 80, 64, dtype=torch.bfloat16)), 'one sequence length and head dim'),
    (dict(k=torch.zeros(2, 2, 81, 32, dtype=torch.bfloat16)), 'one sequence length and head dim'),
    (dict(n_image=0), 'n_image = 0'),
    (dict(n_image=81), 'n_image = 81'),
    (dict(lse=torch.zeros(2, 2, 63)), 'lse has 63 rows, the kernel reads 64'),
    (dict(lse=torch.zeros(2, 2, 80), text_first=True), 'lse has 80 rows, the kernel reads 81'),
])
def test_make_joint_desc_refuses_operands_the_kernel_would_read_past(change, text):
    args = _desc_args()
    args.update({key: v.to(DEV) if isinstance(v, torch.Tensor) else v for key, v in change.items()})
    before = _native.launch_count()
    with pytest.raises(RuntimeError, match=text):
        ops.make_joint_desc(**args)
    assert _native.launch_count() == before


def test_make_joint_desc_takes_padded_and_text_first_lse():
    args = _desc_args()
    ops.make_joint_desc(**args)
    ops.make_joint_desc(**{**args, 'lse': torch.zeros(2, 2, 96, device=DEV)})       # padded to 32 queries
    ops.make_joint_desc(**{**args, 'lse': torch.zeros(2, 2, 81, device=DEV), 'text_first': True})
