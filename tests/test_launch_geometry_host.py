"""Host checks of the restated accumulate planner and tile walks (``tests/test_launch_geometry_gpu.py``): every case
reaches the regimes it names at several SM counts and SIMT occupancies, the cases together cover every regime of the
packing and the three walks, every walk takes every tile of its launch exactly once, and the plan gives the launch
counts the other accumulate tests assert."""
import random

import pytest

from daam_b200 import _native
from tests.test_launch_geometry_gpu import (CASES, CLASSES, ENTRY_CLASSES, LABELS, PROBS, SIMT_KERNEL, SIMT_LONG, Case,
                                            Launch, Layer, cta_tiles, mma_instance, plan, regimes, walk)

SM_COUNTS = (132, 114, 78)    # H100 SXM, H100 PCIe, a small part
OCCUPANCIES = (1, 2, 3, 4)    # SIMT CTAs per SM


def occ_of(n):
    return lambda inst, d: n


MMA = [mma_instance(s, c, m, 1) for m in (0, 1, 2) for c in (False, True) for s in (False, True)] + \
      [mma_instance(False, c, 0, kC) for kC in (2, 3) for c in (False, True)]
MMA16 = [i for i in MMA if i.startswith('accumulate_mma_kernel<false')]
CHUNKED = [mma_instance(s, True, m, 1) for m in (0, 1, 2) for s in (False, True)] + \
          [mma_instance(False, True, 0, kC) for kC in (2, 3)]
SIMT = list(SIMT_KERNEL.values()) + [SIMT_LONG]
CONTIGUOUS = [i for i in MMA if i.startswith('accumulate_mma_kernel<true,false')] + SIMT + [PROBS]

# every regime the sweep must reach (the issue's list, accumulate_mma.cu, accumulate_simt*.cu, probs.cu, api.cu)
REQUIRED = (
    [f'{i}: tiles {t}' for i in MMA + SIMT + [PROBS] for t in ('1', 'G-1', 'G', 'G+1', '2G+1')] +
    [f'{i}: per CTA {c}' for i in MMA for c in ('1', '2', '3', '4', '>= 8')] +
    [f'{i}: rem {r}' for i in CONTIGUOUS for r in ('0', '> 0')] +
    [f'{i}: {r}' for i in CHUNKED for r in ('zero-tile CTA', 'boundary inside a tile')] +
    [f'{mma_instance(s, True, 0, 1)}: CTA spans 1-4 chunks' for s in (False, True)] +
    [f'{mma_instance(s, True, m, 1)}: chunked by one layer' for s in (False, True) for m in (0, 1, 2)] +
    [f'{i}: prefetch window {w}' for i in MMA16 for w in ('full', 'truncated')] +
    [f'{mma_instance(False, c, 0, kC)}: accumulator ring wraps' for kC in (2, 3) for c in (False, True)] +
    [f'{i}: one-tile layer inside a CTA range' for i in (mma_instance(False, True, 0, 1), mma_instance(True, False, 0, 1),
                                                         SIMT_KERNEL['accumulate'])] +
    [f'{i}: hw mod 128 = {r}' for i in (mma_instance(False, False, 0, 1), mma_instance(True, False, 0, 1),
                                        SIMT_KERNEL['accumulate']) for r in (4, 64, 124)] +
    [f'{i}: {p} prompts' for i in MMA + SIMT for p in (2, 3)] +
    [f'{i}: same (prompt, head), next layer' for i in (mma_instance(False, False, 0, 1), mma_instance(False, True, 0, 1),
                                                       SIMT_KERNEL['accumulate'], SIMT_LONG)] +
    ['16-bit CTA alternates fp16 / bf16'] +
    [f'{e} {c}: {n} layers' for e in ENTRY_CLASSES for c in ENTRY_CLASSES[e] for n in (32, 33)] +
    [f'{c}: {t}' for c in ('mma16', 'simt') for t in ('overlap close at position 31', 'overlap at position 32')] +
    ['all 7 classes interleaved', 'SIMT pack with d 256 and d 8', 'FORCE_SIMT'] +
    [f'{e} {m}' for e in ('accumulate', 'steps', 'range') for m in ('RED', 'LDST')])


@pytest.mark.parametrize('occ', OCCUPANCIES)
@pytest.mark.parametrize('sm', SM_COUNTS)
@pytest.mark.parametrize('name', list(CASES))
def test_every_case_reaches_its_regimes(name, sm, occ):
    case = CASES[name](sm, occ_of(occ))
    missing = set(case.tags) - regimes(case, plan(case, sm, occ_of(occ)))
    assert not missing, f'{name} at {sm} SMs, {occ} SIMT CTAs per SM: {sorted(missing)}'


@pytest.mark.parametrize('occ', OCCUPANCIES)
@pytest.mark.parametrize('sm', SM_COUNTS)
def test_the_cases_cover_every_regime(sm, occ):
    seen = set()
    for build in CASES.values():
        case = build(sm, occ_of(occ))
        seen |= regimes(case, plan(case, sm, occ_of(occ)))
    assert not set(REQUIRED) - seen, sorted(set(REQUIRED) - seen)


def _assert_exact_cover(case: Case, launch: Launch, what: str):
    """Every tile of the launch in exactly one CTA, increasing within each CTA, and decoded to the layer, prompt, head
    and pixel it belongs to."""
    seen = []
    for b, tiles in enumerate(walk(case, launch)):
        ts = [t[0] for t in tiles]
        assert ts == sorted(set(ts)), f'{what}: CTA {b} walks {ts}'
        seen += ts
    assert sorted(seen) == list(range(launch.total_tiles)), f'{what}: tiles missed or repeated'
    expect = []
    for e in launch.layers:
        L = case.layers[e['index']]
        expect += [(e['index'], p, h, px) for p in range(L.prompts) for h in range(L.heads)
                   for px in range(0, L.hw, 128)]
    got = sorted((t for tiles in walk(case, launch) for t in tiles))
    assert [t[1:] for t in got] == expect, f'{what}: tiles decode to the wrong (layer, prompt, head, pixel)'


@pytest.mark.parametrize('sm', SM_COUNTS)
def test_walks_cover_every_tile_once(sm):
    for name, build in CASES.items():
        case = build(sm, occ_of(3))
        for n, launch in enumerate(plan(case, sm, occ_of(3))):
            _assert_exact_cover(case, launch, f'{name} launch {n}')


def test_walks_of_random_packs_at_every_grid():
    """The partition arithmetic itself: random small packs (1-6 layers, head_dims of 1-4 chunks), every grid from 1 to
    the tile count, all three walks."""
    rng = random.Random(5)
    for trial in range(150):
        layers = [Layer(rng.choice((4, 64, 124, 128, 132, 256, 260, 388)), rng.randint(1, 3),
                        rng.choice((8, 64, 80, 160, 256)), 'fp32' if trial % 2 else 'bf16', prompts=rng.randint(1, 3))
                  for _ in range(rng.randint(1, 6))]
        case = Case('accumulate', 0, layers, ())
        (base,) = plan(case, 1 << 20, occ_of(1))
        for walk_kind in ('interleaved', 'contiguous', 'weighted'):
            for grid in range(1, base.total_tiles + 1):
                launch = Launch(base.cls, base.instance, grid, grid, walk_kind, base.layers, 'end')
                _assert_exact_cover(case, launch, f'trial {trial} {walk_kind} grid {grid}')


def test_weighted_ranges_follow_the_weights():
    """A tile is taken by the CTA whose weight range holds the tile's first weight unit, so a heavy tile straddling a
    CTA boundary leaves the next CTA without a tile. Weights 17, then 8 x 5: tile starts 0, 17, 22, ..., 52; CTA
    boundaries 57 b / 9 = 0, 6, 12, 19, 25, 31, 38, 44, 50."""
    layers = [Layer(128, 1, 256), Layer(128 * 8, 1, 8)]
    case = Case('accumulate', 0, layers, ())
    (launch,) = plan(case, 20, occ_of(1))
    assert launch.walk == 'weighted' and launch.total_weight == 57 and launch.grid == 9
    assert [list(cta_tiles(launch, b)) for b in range(9)] == [[0], [], [1], [2], [3], [4, 5], [6], [7], [8]]


def _fp16_layers(n, hw=64, heads=2, d=64, dtype='fp16', **kw):
    return [Layer(hw, heads, d, dtype, **kw) for _ in range(n)]


def test_plan_agrees_with_the_launch_counts_other_tests_assert():
    # test_accumulate_gpu.py::test_many_layers_in_one_call_are_chunked: 45 fp16 layers -> 32 + 13
    launches = plan(Case('accumulate', 0, _fp16_layers(45), ()), 132, occ_of(3))
    assert [len(l.layers) for l in launches] == [32, 13]
    # test_accumulate_range_gpu.py::test_many_layers_of_every_kind_in_one_call: 48 16-bit layers (two packs), 16 fp32
    # split, 16 unaligned SIMT
    kinds = [Layer(256, 4, 64, 'bf16'), Layer(576, 2, 64, 'fp16'), Layer(256, 2, 80, 'fp16'),
             Layer(256, 2, 64, 'fp32'), Layer(256, 2, 64, 'bf16', simt=True)]
    for entry in ('accumulate', 'range'):
        case = Case(entry, _native.ACC_AUTO | _native.ACC_EARLY_LOADS, [kinds[i % 5] for i in range(80)], ())
        launches = plan(case, 132, occ_of(3))
        assert [(l.cls, len(l.layers)) for l in launches] == [('mma16', 32), ('mma16', 16), ('split', 16),
                                                              ('simt', 16)]
        assert launches[0].instance == mma_instance(False, True, 2 if entry == 'range' else 0, 1)
    # test_long_prompt_gpu.py::test_chunked_head_dims_share_a_launch_and_lengths_do_not_mix
    specs = [Layer(1024, 2, 64, 'bf16', 154), Layer(576, 2, 160, 'fp16', 154), Layer(1024, 1, 64, 'fp16', 231),
             Layer(1024, 1, 80, 'bf16', 231), Layer(256, 2, 64, 'bf16'), Layer(256, 1, 40, 'fp32', 231)]
    launches = plan(Case('accumulate', 0, specs, ()), 132, occ_of(3))
    assert [(l.instance, [e['index'] for e in l.layers]) for l in launches] == [
        (mma_instance(False, False, 0, 1), [4]), (mma_instance(False, True, 0, 2), [0, 1]),
        (mma_instance(False, True, 0, 3), [2, 3]), (SIMT_LONG, [5])]
    # DAAM_ACC_FORCE_SIMT: one SIMT pack whatever the dtype
    launches = plan(Case('accumulate', _native.ACC_FORCE_SIMT, _fp16_layers(3) + [Layer(64, 1, 64, 'fp32')], ()),
                    132, occ_of(2))
    assert [(l.instance, l.grid) for l in launches] == [(SIMT_KERNEL['accumulate'], 7)]


def test_overlap_closes():
    """A layer whose accumulator is one already in its pack closes the pack; one that overlaps a layer of a pack that
    has already closed does not close anything."""
    layers = _fp16_layers(3) + [Layer(64, 2, 64, 'fp16', acc_of=1)] + _fp16_layers(2)
    assert [len(l.layers) for l in plan(Case('accumulate', 0, layers, ()), 132, occ_of(1))] == [3, 3]
    layers = _fp16_layers(32) + [Layer(64, 2, 64, 'fp16', acc_of=0)]
    launches = plan(Case('accumulate', 0, layers, ()), 132, occ_of(1))
    assert [(len(l.layers), l.close) for l in launches] == [(32, 'full'), (1, 'end')]
    # different classes never close each other
    layers = _fp16_layers(2) + [Layer(64, 2, 64, 'fp16', simt=True, acc_of=0)]
    assert [(l.cls, len(l.layers)) for l in plan(Case('accumulate', 0, layers, ()), 132, occ_of(1))] == \
        [('mma16', 2), ('simt', 1)]


def test_tile_labels_and_grids():
    """G is the SM count for the wgmma kernel, SM count x occupancy for the SIMT kernels, 3 x SM count for
    attention_probs; the grid is G capped at the tile count."""
    for sm in SM_COUNTS:
        for occ in OCCUPANCIES:
            case = CASES['grid-G+1-accumulate-plain'](sm, occ_of(occ))
            for l in plan(case, sm, occ_of(occ)):
                assert l.G == (sm * occ if l.cls.startswith('simt') else sm) and l.grid == l.G, l.instance
                assert l.total_tiles == l.G + 1
            (p,) = plan(CASES['probs-2G+1'](sm, occ_of(occ)), sm, occ_of(occ))
            assert p.G == 3 * sm and p.total_tiles == 6 * sm + 1
    assert set(CLASSES) == {l.cls for l in plan(CASES['pack-33-accumulate'](132, occ_of(2)), 132, occ_of(2))}
    assert set(LABELS) >= {'1', 'G-1', 'G', 'G+1', '2G+1'}
