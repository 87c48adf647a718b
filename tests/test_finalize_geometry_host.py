"""Host checks of the restated finalize dispatch rule and geometry (``tests/test_finalize_geometry_gpu.py``): it agrees
with ``bench_aspect.fast_rule`` on whole maps, the case table reaches every regime it names at several SM counts, the
cases together cover every regime of the banded kernel, and the two regimes no geometry reaches stay unreachable."""
import math

import pytest

import bench
import bench_aspect
from tests.test_finalize_geometry_gpu import (BAND8_MAX_W, CASES, FAST_MAX_W, THREADS, TRACED, Case, Group, Map,
                                              class_geometry, identity_pass, plan, regimes, traced_keys)

SM_COUNTS = (132, 114, 78)    # H100 SXM, H100 PCIe, a small part


def _bench_keys(workload, latent):
    """``[(h, w, heads)]`` of a bench workload's layers scaled to the latent ``(H, W)``, as test_finalize_parts_gpu
    builds them."""
    layers = bench.traced_layers(workload)
    side = max(math.isqrt(hw) for hw, _, _ in layers)
    return [(latent[0] * math.isqrt(hw) // side, latent[1] * math.isqrt(hw) // side, heads) for hw, heads, _ in layers]


def _whole_map(keys, grid):
    return Case('finalize', grid, [Group(h, w, heads) for h, w, heads in keys], [Map(12)], ())


@pytest.mark.parametrize('workload', ['sd21', 'sdxl'])
@pytest.mark.parametrize('grid', [(64, 64), (96, 64), (76, 52)], ids=str)
def test_plan_agrees_with_bench_aspect_on_whole_maps(workload, grid):
    keys = _bench_keys(workload, grid)
    for sm in SM_COUNTS:
        assert plan(_whole_map(keys, grid), sm)[0]['kernel'] == bench_aspect.fast_rule(keys, grid)


@pytest.mark.parametrize('workload,image', [(wl, hw) for wl, hw, _ in TRACED], ids=str)
def test_plan_agrees_with_bench_aspect_at_traced_sizes(workload, image):
    """Whole maps and single layers of the sizes where only per-layer maps take the fast kernel."""
    keys, grid = traced_keys(workload, image)
    assert plan(_whole_map(keys, grid), 132)[0]['kernel'] == bench_aspect.fast_rule(keys, grid) == 'generic'
    verdicts = set()
    for k in keys:
        verdict = plan(_whole_map([k], grid), 132)[0]['kernel']
        assert verdict == bench_aspect.fast_rule([k], grid), k
        verdicts.add(verdict)
    assert verdicts == {'fast', 'generic'}


@pytest.mark.parametrize('sm', SM_COUNTS)
@pytest.mark.parametrize('name', list(CASES))
def test_every_case_reaches_its_regimes(name, sm):
    case = CASES[name](sm)
    missing = set(case.tags) - regimes(case, plan(case, sm))
    assert not missing, f'{name} at {sm} SMs: {sorted(missing)}'
    assert len(case.maps) <= 64 or name.startswith('traced-')


# every regime of the banded kernel the sweep must cover (DESIGN.md section 4.3 and finalize.cu)
REQUIRED = (
    [f'F1 band 8 rows {r}' for r in range(1, 9)] + [f'F1 band 4 rows {r}' for r in range(1, 5)] +
    ['F1 kg 1', 'F1 kg > 1', 'F1 n4 256', 'F1 256 % n4 != 0'] +
    [f'F{F} {t}' for F in (2, 4) for t in
     ('unit 4', 'unit 2', 'unit 1', 'key_units < 256', 'key_units > 256', 'kg > 1', 'kh 1', 'kw 1',
      'partial band 8', 'band 4', 'band 8')] + ['F2 kg 1'] +
    [f'F{F} nk {label} {state}' for F in (2, 4) for label in ('1', 'kc-1', 'kc', 'kc+1', '2kc', '2kc+1')
     for state in ('own', 'prefetched')] +
    [f'F{F} {parity} chunks {state}' for F in (2, 4) for parity in ('odd', 'even') for state in ('own', 'prefetched')] +
    ['F2 partial band 4'] +
    [f'order {o}' for o in ('1,2,4', '4,2,1', '2,1,4', '4,1,2', '2,4', '1,4')] +
    ['parts: range inside an interleaving', 'head_sel', 'maps: block_begin > 0, blocks > 1', 'mixed bands',
     '2048 keys', 'generic: > 2048 keys', 'generic: unaligned', 'fast+generic', 'band 4 (width > 128)'])


@pytest.mark.parametrize('sm', SM_COUNTS)
def test_the_cases_cover_every_regime(sm):
    seen = set()
    for build in CASES.values():
        case = build(sm)
        seen |= regimes(case, plan(case, sm))
    assert not set(REQUIRED) - seen, sorted(set(REQUIRED) - seen)
    # the widths at the two limits: 128 / 129 (8-row bands), 256 / 257 (the fast kernel)
    for ow, kernel, br in ((128, 'fast', 8), (129, 'fast', 4), (256, 'fast', 4), (257, 'generic', None)):
        p = plan(CASES[f'width-{ow}'](sm), sm)[0]
        assert p['kernel'] == kernel and p.get('br') == br, (ow, p)


def test_unreachable_regimes():
    """A key of exactly 256 copy units needs VR * kw / unit = 256 with VR = R + 4 in {5, 6, 8}: only VR = 8 (factor 2,
    8-row bands, so kw <= 64) divides 256, and kw = 32 / 64 have 16-byte units (8 / 16 units a row, not 32). A
    factor-4 class has at most 64 source pixels under a band (one row of 64, or two of 32), so its keys are always
    split over 4 or more thread groups. An identity pass covers a band of at most 1024 floats (8 x 128 or 4 x 256), so
    n4 <= 256 and it is always one pass."""
    for F in (2, 4):
        for br in (4, 8):
            for kw in range(1, FAST_MAX_W // F + 1):
                if br == 8 and F * kw > BAND8_MAX_W:
                    continue
                g = class_geometry(F, 16 * F, F * kw, br, 1, False)
                assert g['key_units'] != THREADS and g['n_src'] <= THREADS and g['kc'] >= g['kg'], (F, br, kw, g)
                assert F == 2 or g['kg'] >= 4, (F, br, kw, g)
    for br, max_w in ((8, BAND8_MAX_W), (4, FAST_MAX_W)):
        for ow in range(1, max_w + 1):
            for rows in range(1, br + 1):
                if rows * ow % 4 == 0:
                    assert identity_pass(rows, ow)['passes'] == 1
