"""Host checks of the restated daam_accumulate_joint packing and tile walk (``tests/test_joint_geometry_gpu.py``):
every case reaches the regimes it names at several SM counts and occupancies, the cases together cover every regime,
every walk takes every tile of its launch once, and the plan gives the launch counts the other joint tests assert."""
import random

import pytest

from tests.test_joint_geometry_gpu import (CASES, INSTANCE, INSTANCES, LABELS, STAGES, TAGGED_DS, Case, Launch, Layer,
                                           plan, regimes, walk)

SM_COUNTS = (132, 114, 78)    # H100 SXM, H100 PCIe, a small part
OCCUPANCIES = (1, 2, 3, 4, 5)  # CTAs per SM
MMA = INSTANCES[:2]
SIMT = INSTANCES[2]


def occ_of(n):
    return lambda inst, d: n


REQUIRED = (
    [f'{i}: tiles {t}' for i in INSTANCES for t in LABELS] +
    [f'{i}: {r}' for i in INSTANCES for r in ('CTA spans >= 3 layers', 'decode passes >= 2 layers',
                                              'one-tile layer between two large layers', 'pack with d 8 and d 256',
                                              '64 layers, one launch', '65 layers, 64 + 1',
                                              'overlap close at position 1', 'overlap close at position 63',
                                              'partial overlap at a row boundary', 'partial overlap 16 bytes in',
                                              'touching slabs share a launch', 'calls at d 64, 256, 64',
                                              'keep cfg', 'keep lone', 'keep whole', 'image first', 'text first',
                                              'lse contig', 'lse pad32', 'lse pixel', 'tokens = 1', 'tokens = 1024')] +
    [f'{i}: {n} samples' for i in INSTANCES for n in (1, 2, 3)] +
    [f'{i}: d = {d}' for i in INSTANCES for d in TAGGED_DS] +
    [f'{i}: stage {s}' for i in MMA for s in STAGES] +
    [f'{i}: hw mod 64 = {r}' for i in MMA for r in (0, 1, 63)] +
    [f'{i}: hw = {h}' for i in MMA for h in (1, 2, 17)] +
    [f'{i}: accumulator {a}' for i in MMA for a in ('pairs', 'scalar')] +
    [f'{i}: tokens mod 64 = {r}' for i in MMA for r in (0, 1, 16, 17, 48, 63)] +
    [f'{SIMT}: hw mod 128 = {r}' for r in (0, 1, 64, 127)] +
    [f'{SIMT}: tokens mod 32 = {r}' for r in (0, 1, 31)] + [f'{SIMT}: tokens mod 8 != 0'] +
    ['three classes interleaved', '[fp16, bf16, fp16] into one slab', 'one slab in two classes',
     'fp16 and bf16 into different slabs'])


@pytest.mark.parametrize('occ', OCCUPANCIES)
@pytest.mark.parametrize('sm', SM_COUNTS)
@pytest.mark.parametrize('name', list(CASES))
def test_every_case_reaches_its_regimes(name, sm, occ):
    case = CASES[name](sm, occ_of(occ))
    missing = set(case.tags) - regimes(case, plan(case, sm, occ_of(occ)))
    assert not missing, f'{name} at {sm} SMs, {occ} CTAs per SM: {sorted(missing)}'


@pytest.mark.parametrize('occ', OCCUPANCIES)
@pytest.mark.parametrize('sm', SM_COUNTS)
def test_the_cases_cover_every_regime(sm, occ):
    seen = set()
    for build in CASES.values():
        case = build(sm, occ_of(occ))
        seen |= regimes(case, plan(case, sm, occ_of(occ)))
    assert not set(REQUIRED) - seen, sorted(set(REQUIRED) - seen)


def _assert_exact_cover(case: Case, launch: Launch, what: str):
    """Every tile of the launch in exactly one CTA, increasing within each CTA, and decoded to the layer, sample, head
    and pixel it belongs to."""
    seen = []
    walks = walk(case, launch)
    for b, tiles in enumerate(walks):
        ts = [t.tile for t in tiles]
        assert ts == sorted(set(ts)), f'{what}: CTA {b} walks {ts}'
        seen += ts
    assert sorted(seen) == list(range(launch.total_tiles)), f'{what}: tiles missed or repeated'
    expect = []
    for e in launch.layers:
        L = case.layers[e['index']]
        expect += [(e['index'], p, h, px) for p in range(L.samples) for h in range(L.heads)
                   for px in range(0, L.hw, L.tile)]
    got = sorted((t for tiles in walks for t in tiles))
    assert [tuple(t[1:5]) for t in got] == expect, f'{what}: tiles decode to the wrong (layer, sample, head, pixel)'


@pytest.mark.parametrize('sm', SM_COUNTS)
def test_walks_cover_every_tile_once(sm):
    for name, build in CASES.items():
        case = build(sm, occ_of(3))
        for c, launches in enumerate(plan(case, sm, occ_of(3))):
            for n, launch in enumerate(launches):
                _assert_exact_cover(case, launch, f'{name} call {c} launch {n}')


def test_walks_of_random_packs_at_every_grid():
    """Random small packs (1-6 layers, 1-3 samples and heads, partial last tiles), every grid from 1 to the tile
    count, both tile sizes."""
    rng = random.Random(5)
    for trial in range(150):
        dtype = ('bf16', 'fp32')[trial % 2]
        layers = [Layer(rng.choice((1, 17, 63, 64, 65, 128, 129, 200, 257)), 17, 64, dtype,
                        samples=rng.randint(1, 3), heads=rng.randint(1, 3)) for _ in range(rng.randint(1, 6))]
        case = Case(layers, ())
        ((base,),) = plan(case, 1 << 20, occ_of(1))
        for grid in range(1, base.total_tiles + 1):
            launch = Launch(base.cls, base.instance, grid, grid, base.dmax, base.layers, 'end')
            _assert_exact_cover(case, launch, f'trial {trial} grid {grid}')


def test_plan_agrees_with_the_launch_counts_other_tests_assert():
    # test_joint_gpu.py::test_kernel_production_layer_sizes: 3 bf16 layers, then a fourth into layer 0's slab
    layers = [Layer(4096, 333, 64, 'bf16', heads=24) for _ in range(3)]
    layers.append(Layer(4096, 333, 64, 'bf16', heads=24, at=(0, 0)))
    (launches,) = plan(Case(layers, ()), 132, occ_of(4))
    assert [([e['index'] for e in l.layers], l.close) for l in launches] == [([0, 1, 2], 'overlap'), ([3], 'end')]
    # FLUX.1: 19 double- and 38 single-stream layers of one dtype, each its own slab: one launch
    (launches,) = plan(Case([Layer(4096, 512, 128, 'bf16', heads=24, keep='whole', text_first=True)
                             for _ in range(57)], ()), 132, occ_of(4))
    assert [len(l.layers) for l in launches] == [57]
    # the documented class order: fp16, bf16, fp32, each in call order, whatever the call order
    layers = [Layer(64, 17, 64, dt) for dt in ('fp32', 'bf16', 'fp16', 'bf16', 'fp16')]
    (launches,) = plan(Case(layers, ()), 132, occ_of(4))
    assert [(l.instance, [e['index'] for e in l.layers]) for l in launches] == [
        (INSTANCE['fp16'], [2, 4]), (INSTANCE['bf16'], [1, 3]), (INSTANCE['fp32'], [0])]


def test_packs_close_on_shared_bytes_and_at_64_layers():
    A = Layer(64, 5, 64, 'fp16')
    cases = {
        'touching': ([A, Layer(64, 5, 64, 'fp16', at=(0, A.n))], [[0, 1]]),
        'last float shared': ([A, Layer(64, 5, 64, 'fp16', at=(0, A.n - 4))], [[0], [1]]),
        'other class': ([A, Layer(64, 5, 64, 'bf16', at=(0, 0))], [[0], [1]]),
        '64 + 1': ([Layer(64, 5, 8, 'fp16') for _ in range(65)], [list(range(64)), [64]]),
    }
    for what, (layers, want) in cases.items():
        (launches,) = plan(Case(layers, ()), 132, occ_of(1))
        assert [[e['index'] for e in l.layers] for l in launches] == want, what


def test_tile_labels_and_grids():
    """G is SMs x the occupancy of the pack's largest head dim, the grid G capped at the tile count."""
    for sm in SM_COUNTS:
        for occ in OCCUPANCIES:
            for cls in ('fp16', 'bf16', 'fp32'):
                case = CASES[f'grid-2G+1-{cls}'](sm, occ_of(occ))
                ((l,),) = plan(case, sm, occ_of(occ))
                assert l.G == sm * occ and l.grid == l.G and l.total_tiles == 2 * l.G + 1
