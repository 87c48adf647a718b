"""The banded finalize kernel (``finalize_fast_kernel``, daam_b200/csrc/finalize.cu) against float64 at every band,
chunk and copy geometry it accepts.

Each regime of the kernel has its own index arithmetic: 8- or 4-row bands and a partial last band; the factor-1
(identity) pass with one or several thread groups; the factor-2 / factor-4 chunks (16-, 8- and 4-byte ``cp.async``
units, keys copied by a subset of the threads or by all of them, odd and even chunk counts, a first chunk the previous
class prefetched); a map's classes in any order; the per-map key tables of ``daam_finalize_parts``. :func:`plan`
restates the host's dispatch rule and the kernel's geometry for every map of a call. The cases are built from it, each
asserts the regimes it names (so that a change of the rule cannot send a case to the generic kernel unnoticed), and one
profiler trace confirms which kernel every case ran. Every case is checked

* against float64 (``B_y @ key @ B_x^T``, clamp, mean), with and without ``normalize``;
* against the generic kernel (``DAAM_FINALIZE_GENERIC=1``) within the bound of a reordered fp32 key sum: both kernels
  do the same arithmetic per key and differ only in the order of the key sum;
* for writes outside its maps: the outputs of one call share one buffer with NaN guard runs before, between and after
  the maps, and every key stack has NaN floats before and after it.

The geometries only per-layer and per-factor maps reach (SD-2.1 at 600x800, 800x600 and 512x784; SDXL at 1000x1024 and
1032x1024, where the whole map is generic) are checked layer by layer and factor by factor through the C ABI, and at
600x800 through the tracer's ``compute_layer_heat_maps`` / ``compute_factor_heat_maps``.

Three regimes cannot occur, and ``test_unreachable_regimes`` in ``test_finalize_geometry_host.py`` says why: a key of
exactly 256 copy units, a factor-4 class on one thread group, and an identity pass of more than one pass over the
band."""
import json
from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Tuple

import pytest
import torch

from daam_b200 import _native, trace
from daam_b200.testing.synthetic import SD21_SPEC, SDXL_SPEC, make_pipeline
from tests.reference64 import FP32_EPS, MAP_DIMS, assert_close64, normalized_tolerance, rect_tolerance, up64

pytestmark = pytest.mark.gpu
DEV = 'cuda'

THREADS = 256                # threads of a fast-kernel CTA
STAGE_FLOATS = 4096          # kStageFloats: one chunk buffer
MAX_KEYS = 2048              # kMaxClassKeys: the keys a map may select on the fast kernel
FAST_MAX_W = 256             # the widest map the fast kernel takes
BAND8_MAX_W = 128            # the widest map with 8-row bands


# ---- the case description ---------------------------------------------------------------------------------------------

@dataclass
class Group:
    """One ``daam_key_group``: a ``[blocks, heads, tokens, h, w]`` fp32 key stack."""
    h: int
    w: int
    heads: int
    head_sel: int = -1
    blocks: int = 1           # daam_finalize_maps: the group's blocks (one block per image)
    shift: int = 0            # floats the stack's base sits past a 16-byte boundary

    @property
    def per_block(self) -> int:
        return self.heads if self.head_sel < 0 else 1


@dataclass
class Map:
    """One output map: groups ``[begin, begin + count)`` (``daam_finalize_parts``; every group otherwise) and blocks
    ``[block_begin, block_begin + block_count)`` (``daam_finalize_maps``; block 0 otherwise)."""
    n_rows: int
    begin: int = 0
    count: Optional[int] = None
    block_begin: int = 0
    block_count: int = 1


@dataclass
class Case:
    entry: str                # 'finalize' (one map over every group), 'maps' or 'parts'
    grid: Tuple[int, int]
    groups: List[Group]
    maps: List[Map]
    tags: Tuple[str, ...]     # regimes the case must reach (see regimes())

    def __post_init__(self):
        for m in self.maps:
            if self.entry != 'parts':
                m.begin, m.count = 0, len(self.groups)
            elif m.count is None:
                m.count = len(self.groups) - m.begin

    def tokens(self, i: int) -> int:
        """Rows group ``i`` holds: the most any map that reads it needs (daam_finalize_maps: any map)."""
        reads = [m.n_rows for m in self.maps if self.entry != 'parts' or m.begin <= i < m.begin + m.count]
        return max(reads or [1])


# ---- the dispatch rule and the kernel's geometry, restated --------------------------------------------------------------

def band_rows(oh: int, ow: int, n_rows: int, sm_count: int) -> int:
    """8-row bands unless that leaves fewer than 2 CTAs per SM or the map is wider than 128."""
    return 8 if -(-oh // 8) * n_rows >= 2 * sm_count and ow <= BAND8_MAX_W else 4


def class_geometry(f: int, oh: int, ow: int, br: int, nk: int, prefetched: bool) -> dict:
    """``ChunkGeom`` and ``issue_chunk`` of a factor-2 / factor-4 class of ``nk`` keys at band height ``br``."""
    kh, kw = oh // f, ow // f
    R = br // f
    VR = R + 4
    region, n_src = VR * kw, R * kw
    kg = THREADS // n_src
    kc = STAGE_FLOATS // region
    kc -= kc % kg
    unit = 4 if kw % 4 == 0 else (2 if kw % 2 == 0 else 1)
    key_units = VR * kw // unit
    return dict(f=f, kh=kh, kw=kw, R=R, VR=VR, region=region, n_src=n_src, kg=kg, kc=kc, unit=unit,
                key_units=key_units, keys_par=THREADS // key_units if key_units <= THREADS else 1, nk=nk,
                chunks=-(-nk // kc), prefetched=prefetched)


def identity_pass(rows: int, ow: int) -> dict:
    """``class_pass_identity`` over a band of ``rows`` valid rows."""
    n4 = rows * ow // 4
    return dict(rows=rows, n4=n4, kg=1 if n4 >= THREADS else THREADS // n4, passes=-(-n4 // THREADS))


def plan(case: Case, sm_count: int, generic: bool = False) -> List[dict]:
    """What ``launch_finalize`` does with every map of ``case``: ``kernel`` ('fast' or 'generic') and ``n_keys``; for a
    fast map also ``br``, ``bands``, ``last_rows``, ``classes`` (factors in the order the map's groups first show them)
    and ``geometry`` (per class: :func:`class_geometry`, or for factor 1 ``{'f': 1, 'passes': [identity_pass per
    distinct band height]}``)."""
    oh, ow = case.grid
    fast_grid = (oh != ow or oh % 16 == 0) and ow <= FAST_MAX_W and not generic
    factor = []
    for g in case.groups:
        f = oh // g.h
        ok = (fast_grid and oh % g.h == 0 and ow % g.w == 0 and ow // g.w == f and f in (1, 2, 4)
              and g.shift % 4 == 0 and (g.h * g.w) % 4 == 0)
        factor.append(f if ok else 0)
    plans = []
    for m in case.maps:
        sel = range(m.begin, m.begin + m.count)
        n_keys = sum(case.groups[i].per_block for i in sel) * m.block_count
        p = dict(kernel='generic', n_keys=n_keys, n_rows=m.n_rows,
                 unaligned=any(case.groups[i].shift % 4 for i in sel))
        if all(factor[i] for i in sel) and n_keys <= MAX_KEYS:
            classes, keys = [], {}
            for i in sel:
                if factor[i] not in keys:
                    classes.append(factor[i])
                    keys[factor[i]] = 0
                keys[factor[i]] += case.groups[i].per_block
            br = band_rows(oh, ow, m.n_rows, sm_count)
            bands = -(-oh // br)
            last = oh - (bands - 1) * br
            geometry = []
            for c, f in enumerate(classes):
                if f == 1:
                    heights = ([br] if bands > 1 or last == br else []) + ([last] if last != br else [])
                    geometry.append(dict(f=1, nk=keys[1] * m.block_count, passes=[identity_pass(r, ow) for r in heights]))
                else:       # a class after another one had its chunk 0 prefetched by that one
                    geometry.append(class_geometry(f, oh, ow, br, keys[f] * m.block_count, c > 0))
            p.update(kernel='fast', br=br, bands=bands, last_rows=last, classes=classes, geometry=geometry,
                     band8_possible=-(-oh // 8) * m.n_rows >= 2 * sm_count)
        plans.append(p)
    return plans


def _count_label(nk: int, kc: int) -> List[str]:
    return [label for label, n in (('1', 1), ('kc-1', kc - 1), ('kc', kc), ('kc+1', kc + 1), ('2kc', 2 * kc),
                                   ('2kc+1', 2 * kc + 1)) if nk == n]


def regimes(case: Case, plans: List[dict]) -> set:
    """The regimes a call reaches, as the tags the cases name."""
    oh, ow = case.grid
    tags = {p['kernel'] for p in plans}
    if len(tags) == 2:
        tags.add('fast+generic')
    fast = [p for p in plans if p['kernel'] == 'fast']
    if len({p['br'] for p in fast}) > 1:
        tags.add('mixed bands')
    for m, p in zip(case.maps, plans):
        if p['kernel'] == 'generic':
            if p['n_keys'] > MAX_KEYS:
                tags.add('generic: > 2048 keys')
            if p['unaligned']:
                tags.add('generic: unaligned')
            continue
        br = p['br']
        tags.add(f'band {br}')
        if br == 4 and p['band8_possible']:
            tags.add('band 4 (width > 128)')
        if p['n_keys'] == MAX_KEYS:
            tags.add('2048 keys')
        tags.add('order ' + ','.join(map(str, p['classes'])))
        sel = case.groups[m.begin:m.begin + m.count]
        if any(g.head_sel >= 0 for g in sel):
            tags.add('head_sel')
        if case.entry == 'maps' and m.block_begin > 0 and m.block_count > 1:
            tags.add('maps: block_begin > 0, blocks > 1')
        kinds = [oh // g.h for g in sel]
        runs = [k for i, k in enumerate(kinds) if i == 0 or kinds[i - 1] != k]
        if case.entry == 'parts' and len(runs) > len(set(runs)) and m.begin > 0 and \
                m.begin + m.count < len(case.groups):
            tags.add('parts: range inside an interleaving')
        for c in p['geometry']:
            F = c['f']
            if F == 1:
                for ip in c['passes']:
                    tags.add(f'F1 band {br} rows {ip["rows"]}')
                    tags.add('F1 kg 1' if ip['kg'] == 1 else 'F1 kg > 1')
                    if ip['n4'] == THREADS:
                        tags.add('F1 n4 256')
                    if ip['n4'] < THREADS and THREADS % ip['n4']:
                        tags.add('F1 256 % n4 != 0')
                continue
            state = 'prefetched' if c['prefetched'] else 'own'
            ku = c['key_units']
            tags |= {f'F{F} band {br}', f'F{F} unit {c["unit"]}',
                     f'F{F} key_units ' + ('< 256' if ku < THREADS else '= 256' if ku == THREADS else '> 256'),
                     f'F{F} kg 1' if c['kg'] == 1 else f'F{F} kg > 1',
                     f'F{F} {"odd" if c["chunks"] % 2 else "even"} chunks {state}'}
            if c['kh'] == 1:
                tags.add(f'F{F} kh 1')
            if c['kw'] == 1:
                tags.add(f'F{F} kw 1')
            if oh % br:
                tags.add(f'F{F} partial band {br}')
            tags |= {f'F{F} nk {label} {state}' for label in _count_label(c['nk'], c['kc'])}
    return tags


# ---- the cases ----------------------------------------------------------------------------------------------------------

def rows8(oh: int, sm_count: int) -> int:
    """The fewest rows that give a map of height ``oh`` (at most 128 wide) 8-row bands."""
    return -(-2 * sm_count // -(-oh // 8))


ROWS4 = 2                     # 4-row bands at every height this file uses (ceil(oh / 8) * 2 < 2 * SMs)


def _both(oh, sm, **kw) -> List[Map]:
    """The same range at 8-row and at 4-row bands."""
    return [Map(rows8(oh, sm), **kw), Map(ROWS4, **kw)]


def _identity(r):
    def build(sm):
        oh = 16 + r
        return Case('parts', (oh, 28), [Group(oh, 28, 3)], _both(oh, sm),
                    (f'F1 band 8 rows {r or 8}', f'F1 band 4 rows {r % 4 or 4}', 'F1 kg > 1', 'F1 256 % n4 != 0',
                     'mixed bands'))
    return build


def _three(oh, ow, heads=(2, 3, 2), factors=(1, 2, 4)) -> List[Group]:
    return [Group(oh // f, ow // f, h) for f, h in zip(factors, heads)]


def _geometry(oh, ow, factors, tags, band8=True):
    """Every class alone and all of them together, at both band heights (``band8``) or at 4-row bands."""
    def build(sm):
        groups = _three(oh, ow, factors=factors)
        ranges = [dict(begin=i, count=1) for i in range(len(groups))] + [dict(begin=0, count=len(groups))]
        maps = [m for r in ranges for m in (_both(oh, sm, **r) if band8 else [Map(rows8(oh, sm), **r)])]
        return Case('parts', (oh, ow), groups, maps, tags)
    return build


def _chunks(F):
    """Per band height, class F alone and after another class (which prefetches its chunk 0), with 1, kc - 1, kc,
    kc + 1, 2 kc and 2 kc + 1 keys."""
    oh, ow = 40, 72
    before = 1 if F == 2 else 2           # factor 2 follows an identity pass, factor 4 a factor-2 class pass

    def build(sm):
        groups, maps = [], []
        for n_rows in (rows8(oh, sm), ROWS4):
            kc = class_geometry(F, oh, ow, band_rows(oh, ow, n_rows, sm), 0, False)['kc']
            for n in (1, kc - 1, kc, kc + 1, 2 * kc, 2 * kc + 1):
                groups += [Group(oh // before, ow // before, 2), Group(oh // F, ow // F, n)]
                maps += [Map(n_rows, len(groups) - 1, 1), Map(n_rows, len(groups) - 2, 2)]
        tags = [f'F{F} nk {label} {state}' for label in ('1', 'kc-1', 'kc', 'kc+1', '2kc', '2kc+1')
                for state in ('own', 'prefetched')]
        tags += [f'F{F} {parity} chunks {state}' for parity in ('odd', 'even') for state in ('own', 'prefetched')]
        return Case('parts', (oh, ow), groups, maps, tuple(tags + [f'F{F} band 8', f'F{F} band 4']))
    return build


ORDER = [1, 2, 4, 2, 1, 4, 1, 2, 1, 4, 2, 4, 1]     # the factors of the interleaved group list
ORDER_RANGES = [(0, 3), (2, 3), (3, 3), (5, 3), (10, 2), (8, 2), (6, 5), (3, 7), (1, 11), (0, 13)]
ORDER_TAGS = ('order 1,2,4', 'order 4,2,1', 'order 2,1,4', 'order 4,1,2', 'order 2,4', 'order 1,4')


def _order_groups(blocks=1):
    oh, ow = 44, 80
    return [Group(oh // f, ow // f, 1 + i % 3, head_sel=(i % 3 if i % 4 == 3 else -1), blocks=blocks)
            for i, f in enumerate(ORDER)]


def _orders(sm):
    maps = [m for b, c in ORDER_RANGES for m in _both(44, sm, begin=b, count=c)]
    return Case('parts', (44, 80), _order_groups(), maps,
                ORDER_TAGS + ('head_sel', 'parts: range inside an interleaving', 'F4 partial band 8', 'mixed bands'))


def _orders_finalize(sm):
    return Case('finalize', (44, 80), _order_groups(), [Map(rows8(44, sm))], ('order 1,2,4', 'band 8', 'head_sel'))


def _orders_maps(sm):
    maps = [Map(rows8(44, sm), block_begin=1, block_count=2), Map(ROWS4, block_begin=0, block_count=3),
            Map(5, block_begin=2, block_count=1), Map(ROWS4, block_begin=1, block_count=2)]
    return Case('maps', (44, 80), _order_groups(blocks=3), maps,
                ('order 1,2,4', 'maps: block_begin > 0, blocks > 1', 'head_sel', 'mixed bands'))


def _many_maps(sm):
    """2048 keys (fast) and 2049 (generic) next to maps of both band heights."""
    groups = [Group(8, 16, 1024), Group(8, 16, 1024), Group(8, 16, 1), Group(32, 64, 2), Group(16, 32, 3)]
    maps = [Map(3, 0, 2), Map(3, 0, 3), Map(rows8(32, sm), 3, 2), Map(3, 2, 3), Map(ROWS4, 3, 1)]
    return Case('parts', (32, 64), groups, maps,
                ('2048 keys', 'generic: > 2048 keys', 'mixed bands', 'fast+generic', 'order 4,1,2'))


def _unaligned(sm):
    groups = [Group(40, 72, 2), Group(20, 36, 3, shift=1), Group(10, 18, 2), Group(20, 36, 2)]
    maps = [Map(ROWS4, 0, 1), Map(ROWS4, 1, 1), Map(ROWS4, 0, 3), Map(ROWS4, 2, 2), Map(rows8(40, sm), 3, 1)]
    return Case('parts', (40, 72), groups, maps, ('generic: unaligned', 'fast+generic', 'order 4,2'))


def _width(ow):
    def build(sm):
        groups = _three(40, ow, factors=[f for f in (1, 2, 4) if ow % f == 0])
        maps = [m for r in [dict(begin=0, count=len(groups))] + [dict(begin=i, count=1) for i in range(len(groups))]
                for m in _both(40, sm, **r)]
        return Case('parts', (40, ow), groups, maps, WIDTH_TAGS[ow])
    return build


WIDTH_TAGS = {128: ('band 8', 'F1 n4 256', 'F2 kg 1', 'F2 band 8', 'F4 band 8'),
              129: ('band 4 (width > 128)', 'F1 band 4 rows 4'),
              256: ('band 4 (width > 128)', 'F1 n4 256', 'F2 kg 1', 'F2 unit 4', 'F4 kg > 1'),
              257: ('generic',)}


# the sizes where per-layer or per-factor maps take the fast kernel while the whole map does not
TRACED = [('sd21', (600, 800), ('F1 band 4 rows 3', 'F1 band 8 rows 3', 'fast+generic')),
          ('sd21', (800, 600), ('F1 band 8 rows 4', 'fast+generic')),
          ('sd21', (512, 784), ('F2 unit 1', 'F2 key_units > 256', 'F2 kg 1', 'F2 kg > 1', 'fast+generic')),
          ('sdxl', (1000, 1024), ('F1 band 8 rows 7', 'F1 kg > 1', 'fast+generic')),
          ('sdxl', (1032, 1024), ('F1 band 8 rows 1', 'F1 band 4 rows 1', 'fast+generic'))]
TRACED_ROWS = (12, 77)        # a 10-word prompt and the whole context


def traced_keys(workload: str, image: Tuple[int, int]):
    """``([(h, w, heads)] of every traced layer, grid)`` of ``bench.py``'s SD-2.1 / SDXL workload at ``image``, from
    :class:`~daam_b200.geometry.LatentGeometry` (as ``bench_aspect.py`` derives them)."""
    import bench_aspect
    spec = {'sd21': SD21_SPEC, 'sdxl': SDXL_SPEC}[workload]
    return bench_aspect.layer_keys(workload, spec.sample_size, image)


def _traced(workload, image, tags):
    """Every layer's map, every factor's map (the layers sorted by key size, largest first, as the tracer orders a
    factor read) and the whole map, at 12 and at 77 rows."""
    def build(sm):
        keys, grid = traced_keys(workload, image)
        keys = sorted(keys, key=lambda k: -k[0] * k[1])
        groups = [Group(h, w, heads) for h, w, heads in keys]
        runs, begin = [], 0
        for i in range(1, len(keys) + 1):
            if i == len(keys) or keys[i][:2] != keys[begin][:2]:
                runs.append((begin, i - begin))
                begin = i
        ranges = [(i, 1) for i in range(len(keys))] + runs + [(0, len(keys))]
        maps = [Map(n, b, c) for n in TRACED_ROWS for b, c in ranges]
        return Case('parts', grid, groups, maps, tags)
    return build


CASES: Dict[str, Callable[[int], Case]] = {
    **{f'identity-last-band-{r or 8}-rows': _identity(r) for r in range(8)},
    'identity-n4-256': _geometry(40, 128, (1,), ('F1 n4 256', 'F1 kg 1', 'F1 kg > 1')),
    'f2-odd-kw-32x49': _geometry(64, 98, (1, 2), ('F2 unit 1', 'F2 key_units > 256', 'F2 kg 1', 'F2 kg > 1')),
    'f2-units-264': _geometry(40, 66, (1, 2), ('F2 unit 1', 'F2 key_units > 256', 'F2 key_units < 256')),
    'f2-unit-2-partial-band': _geometry(44, 36, (1, 2), ('F2 unit 2', 'F2 partial band 8', 'F2 band 4')),
    'f2-partial-band-4': _geometry(42, 40, (1, 2), ('F2 partial band 4', 'F2 partial band 8')),
    'f4-odd-kw-units-255': _geometry(48, 204, (1, 2, 4), ('F4 unit 1', 'F4 key_units < 256', 'F2 unit 2',
                                                          'F2 key_units > 256', 'band 4 (width > 128)'), band8=False),
    'f4-odd-kw-units-265': _geometry(48, 212, (1, 2, 4), ('F4 unit 1', 'F4 key_units > 256', 'F2 unit 2'), band8=False),
    'f4-partial-band-8': _geometry(44, 80, (1, 2, 4), ('F4 partial band 8', 'F2 partial band 8', 'F4 unit 4')),
    'kh-1-f2': _geometry(2, 40, (1, 2), ('F2 kh 1', 'F2 partial band 8', 'F2 partial band 4')),
    'kh-1-f4': _geometry(4, 48, (1, 2, 4), ('F4 kh 1', 'F4 partial band 8', 'F2 partial band 8')),
    'kw-1-f2': _geometry(40, 2, (1, 2), ('F2 kw 1', 'F2 unit 1')),
    'kw-1-f4': _geometry(48, 4, (1, 2, 4), ('F4 kw 1', 'F2 unit 2', 'F4 unit 1')),
    'chunks-f2': _chunks(2),
    'chunks-f4': _chunks(4),
    'orders-parts': _orders,
    'orders-finalize': _orders_finalize,
    'orders-maps': _orders_maps,
    'many-maps-2048-keys': _many_maps,
    'unaligned-group': _unaligned,
    **{f'width-{ow}': _width(ow) for ow in (128, 129, 256, 257)},
    **{f'traced-{wl}-{h}x{w}': _traced(wl, (h, w), tags) for wl, (h, w), tags in TRACED},
}
CASE_NAMES = list(CASES)


# ---- running a case -----------------------------------------------------------------------------------------------------

class Buffers:
    """The case's key stacks (seeded randn, negative values too, so the clamp matters), each with NaN floats before
    and after it, and one output buffer holding every map with NaN guard runs before, between and after them (each
    longer than a band, so that a band written past its map's end lands in a guard)."""

    def __init__(self, case: Case, seed: int):
        self.case = case
        oh, ow = case.grid
        g = torch.Generator(device=DEV).manual_seed(seed)
        self.stacks = []
        for i, grp in enumerate(case.groups):
            shape = (grp.blocks, grp.heads, case.tokens(i), grp.h, grp.w)
            n = shape[0] * shape[1] * shape[2] * shape[3] * shape[4]
            lead, tail = 64 + grp.shift, 64 + grp.w          # a row past the stack's end reads NaN
            store = torch.full((lead + n + tail,), float('nan'), device=DEV)
            store[lead:lead + n] = torch.randn(n, generator=g, device=DEV)
            self.stacks.append(store[lead:lead + n].view(shape))
        self.guard = 8 * ow
        sizes = [m.n_rows * oh * ow for m in case.maps]
        self.out = torch.full((self.guard * (len(sizes) + 1) + sum(sizes),), float('nan'), device=DEV)
        self.views, self.written, pos = [], torch.zeros_like(self.out, dtype=torch.bool), self.guard
        for m, size in zip(case.maps, sizes):
            self.views.append(self.out[pos:pos + size].view(m.n_rows, oh, ow))
            self.written[pos:pos + size] = True
            pos += size + self.guard

    def key_groups(self) -> List[_native.DaamKeyGroup]:
        return [_native.DaamKeyGroup(acc=s.data_ptr(), heads=g.heads, h=g.h, w=g.w, tokens=s.shape[2],
                                     head_sel=g.head_sel, n_blocks=g.blocks)
                for g, s in zip(self.case.groups, self.stacks)]

    def run(self, normalize: bool) -> List[torch.Tensor]:
        """One call of the case's entry point into the NaN-filled output buffer."""
        case, stream = self.case, torch.cuda.current_stream().cuda_stream
        self.out.fill_(float('nan'))
        groups = self.key_groups()
        if case.entry == 'finalize':
            (m,), (v,) = case.maps, self.views
            _native.finalize(groups, case.grid, m.n_rows, normalize, v.data_ptr(), stream)
        elif case.entry == 'maps':
            sel = [_native.DaamMapSel(block_begin=m.block_begin, block_count=m.block_count, n_rows=m.n_rows,
                                      out=v.data_ptr()) for m, v in zip(case.maps, self.views)]
            _native.finalize_maps(groups, sel, case.grid, normalize, stream)
        else:
            sel = [_native.DaamMapPart(group_begin=m.begin, group_count=m.count, n_rows=m.n_rows, out=v.data_ptr())
                   for m, v in zip(case.maps, self.views)]
            _native.finalize_parts(groups, sel, case.grid, normalize, stream)
        torch.cuda.synchronize()
        return [v.clone() for v in self.views]

    def check_writes(self, what: str):
        """Every map element written (finite), every guard element still NaN."""
        for i, v in enumerate(self.views):
            assert bool(torch.isfinite(v).all()), f'{what}: map {i} has elements that are not finite'
        stray = ~self.written & ~torch.isnan(self.out)
        assert not bool(stray.any()), f'{what}: {int(stray.sum())} floats written outside the maps'

    def selected(self, m: Map) -> List[torch.Tensor]:
        """The keys map ``m`` reads, per group: ``[keys, n_rows, h, w]``."""
        out = []
        for g, s in zip(self.case.groups[m.begin:m.begin + m.count], self.stacks[m.begin:m.begin + m.count]):
            sel = s[m.block_begin:m.block_begin + m.block_count]
            if g.head_sel >= 0:
                sel = sel[:, g.head_sel:g.head_sel + 1]
            out.append(sel[:, :, :m.n_rows].reshape(-1, m.n_rows, g.h, g.w))
        return out


def reference64(keys: List[torch.Tensor], grid) -> torch.Tensor:
    """The float64 map: every key upsampled, clamped, averaged (in slices of 64 keys)."""
    total, n = None, 0
    for k in keys:
        for part in k.split(64):
            s = up64(part, grid).clamp_(min=0.0).sum(dim=0)
            total = s if total is None else total + s
        n += k.shape[0]
    return total / n


def _norm64(maps: torch.Tensor) -> torch.Tensor:
    return maps / (maps[1:-1].sum(dim=0, keepdim=True) + 1e-6)


TINY = 2.0 ** -149            # the smallest fp32 subnormal: the bound of a 0 against a 0


def reorder_rtol(n_keys: int, n_rows: int, normalize: bool) -> float:
    """Bound of the relative difference of two fp32 sums of the same ``n_keys`` non-negative terms in different orders
    (each within ``(n_keys + 1) u`` of the exact sum), each divided by ``n_keys``; with ``normalize`` also the
    denominators (sums of ``n_rows - 2`` such values) and the division."""
    eps = (n_keys + 1) * FP32_EPS
    return 4 * eps + (2 * n_rows + 4) * FP32_EPS if normalize else 2 * eps + 2 * FP32_EPS


def _sm_count() -> int:
    return _native.device_info()['sm_count']


def _assert_regimes(case: Case, plans: List[dict], what: str):
    missing = set(case.tags) - regimes(case, plans)
    assert not missing, f'{what}: the case no longer reaches {sorted(missing)}'


@pytest.mark.parametrize('name', CASE_NAMES)
def test_case_against_float64_and_the_generic_kernel(monkeypatch, name):
    sm = _sm_count()
    case = CASES[name](sm)
    plans = plan(case, sm)
    _assert_regimes(case, plans, name)
    bufs = Buffers(case, seed=CASE_NAMES.index(name))
    outs = {}
    for normalize in (False, True):
        for generic in (False, True):
            monkeypatch.setenv('DAAM_FINALIZE_GENERIC', '1' if generic else '0')
            outs[normalize, generic] = bufs.run(normalize)
            bufs.check_writes(f'{name} normalize {normalize}' + (' generic' if generic else ''))
    for i, (m, p) in enumerate(zip(case.maps, plans)):
        what = f'{name} map {i} ({p["kernel"]}, groups [{m.begin}, +{m.count}), blocks [{m.block_begin}, ' \
               f'+{m.block_count}), {m.n_rows} rows)'
        keys = bufs.selected(m)
        raw = reference64(keys, case.grid)
        rtol, atol = rect_tolerance(keys, p['n_keys'], case.grid)
        assert_close64(outs[False, False][i], raw, rtol, atol, what, MAP_DIMS)
        assert_close64(outs[True, False][i], _norm64(raw), 0.0, normalized_tolerance(raw, rtol, atol),
                       f'{what} normalized', MAP_DIMS)
        for normalize in (False, True):       # a zero is a sum of zeros in either order: TINY lets 0 match 0
            assert_close64(outs[normalize, False][i], outs[normalize, True][i].double(),
                           reorder_rtol(p['n_keys'], m.n_rows, normalize), TINY,
                           f'{what} normalize {normalize} vs the generic kernel', MAP_DIMS)


def _kernel_kind(name: str) -> Optional[str]:
    if 'finalize_fast_kernel' in name:
        return 'fast'
    if 'finalize_kernel' in name:
        return 'generic'
    return None


def _expected_launches(case: Case, plans: List[dict]) -> List[str]:
    """The finalize kernels one call launches: per call of at most FINALIZE_MAX_MAPS maps, the fast kernel if one of
    its maps is fast, then the generic kernel if one is generic."""
    out = []
    for i in range(0, len(plans), _native.FINALIZE_MAX_MAPS):
        kinds = {p['kernel'] for p in plans[i:i + _native.FINALIZE_MAX_MAPS]}
        out += [k for k in ('fast', 'generic') if k in kinds]
    return out


def test_every_case_runs_the_kernels_its_plan_names(monkeypatch, tmp_path):
    """One torch.profiler CUDA activity trace over one call of every case: the finalize kernels it lists, in order,
    are the ones plan() names."""
    sm = _sm_count()
    monkeypatch.setenv('DAAM_FINALIZE_GENERIC', '0')
    runs = []
    for name in CASE_NAMES:
        case = CASES[name](sm)
        runs.append((name, Buffers(case, seed=0), _expected_launches(case, plan(case, sm))))
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _, bufs, _ in runs:
            bufs.run(normalize=False)
    path = tmp_path / 'finalize.pt.trace.json'
    prof.export_chrome_trace(str(path))
    events = sorted((e['ts'], e['name']) for e in json.loads(path.read_text())['traceEvents']
                    if e.get('cat') == 'kernel' and _kernel_kind(e['name']))
    got = [_kernel_kind(n) for _, n in events]
    want = [k for _, _, kinds in runs for k in kinds]
    if got != want:
        pos, lines = 0, []
        for name, _, kinds in runs:
            lines.append(f'{name}: planned {kinds}, traced {got[pos:pos + len(kinds)]}')
            pos += len(kinds)
        raise AssertionError('kernels differ from the plan:\n' + '\n'.join(lines))


# ---- the tracer at SD-2.1 600x800 ----------------------------------------------------------------------------------------

PROMPT = 'a dog chasing a red ball on the beach'


def test_tracer_layer_and_factor_maps_at_600x800_against_float64():
    """compute_layer_heat_maps / compute_factor_heat_maps of a traced SD-2.1 generation at 600x800 against float64
    maps of the traced slabs themselves. The 75x100 layers' maps take the fast kernel with a partial last band of 3
    rows, the other maps the generic one."""
    pipe = make_pipeline(SD21_SPEC, 'skeleton', dtype=torch.bfloat16, device=DEV, seed=1, init_on_device=True)
    with trace(pipe) as tc:
        pipe(PROMPT, num_inference_steps=2, generator=torch.Generator().manual_seed(7), height=600, width=800)
        grid = tc.geometry.grid
        stacks = {}
        for (factor, layer, head), key in tc.all_heat_maps:
            stacks.setdefault(layer, (factor, {}))[1][head] = key
        stacks = {layer: (f, torch.stack([heads[h] for h in sorted(heads)])) for layer, (f, heads) in stacks.items()}
        for normalize in (False, True):
            layers = tc.compute_layer_heat_maps(normalize=normalize)
            factors = tc.compute_factor_heat_maps(normalize=normalize)
            n_rows = layers.heat_maps.shape[1]
            if not normalize:
                sm = _sm_count()
                case = Case('parts', grid, [Group(*s.shape[-2:], s.shape[0]) for _, s in stacks.values()],
                            [Map(n_rows, i, 1) for i in range(len(stacks))], ())
                tags = regimes(case, plan(case, sm))
                assert {'F1 band 4 rows 3', 'fast', 'generic'} <= tags, sorted(tags)
            reads = [(f'layer {layer}', [stacks[layer][1]]) for layer in layers.layers] + \
                    [(f'factor {f}', [s for g, s in stacks.values() if g == f]) for f in factors.factors]
            got = list(layers.heat_maps) + list(factors.heat_maps)
            assert len(got) == len(reads)
            for (what, keys), out in zip(reads, got):
                keys = [k[:, :n_rows] for k in keys]
                n_keys = sum(k.shape[0] for k in keys)
                raw = reference64(keys, grid)
                rtol, atol = rect_tolerance(keys, n_keys, grid)
                if normalize:
                    assert_close64(out, _norm64(raw), 0.0, normalized_tolerance(raw, rtol, atol), f'{what} normalized',
                                   MAP_DIMS)
                else:
                    assert_close64(out, raw, rtol, atol, what, MAP_DIMS)
