"""daam_finalize_parts through the C ABI: map m of one call is bit-identical (torch.equal) to daam_finalize over groups
[group_begin, group_begin + group_count) of the call's list -- single-class maps at every factor, maps mixing classes,
overlapping ranges and the range of every group, head_sel, normalisation, row counts differing per map (and so band
heights), square, rectangular and off-grid maps, a map that must take the generic kernel between maps on the fast one,
a map past 2048 keys, more maps than one call holds; against float64; the launch count; and every refusal."""
import ctypes

import pytest
import torch

import bench
from daam_b200 import _native
from tests.reference64 import assert_close64, finalize_tolerance, global_map64, normalized_tolerance

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def _stacks(layers, seed, tokens=77):
    """One fp32 key stack [heads, tokens, h * w] of seeded randn maps per layer (negative values too, so the clamp
    matters); ``layers[i] = ((h, w), heads)``."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    return [(torch.randn(hd, tokens, h * w, generator=g, device=DEV), h, w) for (h, w), hd in layers]


def _groups(stacks, head_sel=-1):
    return [_native.DaamKeyGroup(acc=t.data_ptr(), heads=t.shape[0], h=h, w=w, tokens=t.shape[1], head_sel=head_sel,
                                 n_blocks=0) for t, h, w in stacks]


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _check_parts(stacks, grid, parts, normalize=False, head_sel=-1, what=''):
    """parts: [(group_begin, group_count, n_rows)]; one daam_finalize_parts call against one daam_finalize per map."""
    groups = _groups(stacks, head_sel)
    outs = [torch.full((n,) + grid, float('nan'), device=DEV) for _, _, n in parts]
    sel = [_native.DaamMapPart(group_begin=b, group_count=c, n_rows=n, out=o.data_ptr())
           for (b, c, n), o in zip(parts, outs)]
    _native.finalize_parts(groups, sel, grid, normalize, _stream())
    for (b, c, n), got in zip(parts, outs):
        ref = torch.empty((n,) + grid, device=DEV)
        _native.finalize(groups[b:b + c], grid, n, normalize, ref.data_ptr(), _stream())
        torch.cuda.synchronize()
        assert torch.isfinite(got).all(), f'{what} part {(b, c, n)}: not written'
        assert torch.equal(got, ref), f'{what} part {(b, c, n)}: differs from daam_finalize on the sub-list'
    return outs


def _layers(workload, latent_hw):
    """The traced layers of a bench workload at latent (H, W): ((h, w), heads) per layer."""
    layers = bench.traced_layers(workload)
    side = max(int(round(hw ** 0.5)) for hw, _, _ in layers)
    lh, lw = latent_hw
    return [((lh * int(round(hw ** 0.5)) // side, lw * int(round(hw ** 0.5)) // side), h) for hw, h, _ in layers]


def _runs(layers):
    """(begin, count) of every maximal run of equally sized layers: single-class maps."""
    runs, begin = [], 0
    for i in range(1, len(layers) + 1):
        if i == len(layers) or layers[i][0] != layers[begin][0]:
            runs.append((begin, i - begin))
            begin = i
    return runs


CASES = [('sd21', (64, 64)), ('sd21', (96, 64)), ('sdxl', (64, 64)), ('sdxl', (76, 52))]


@pytest.mark.parametrize('generic', [False, True])
@pytest.mark.parametrize('normalize', [False, True])
@pytest.mark.parametrize('workload,grid', CASES)
def test_parts_equal_finalize_on_the_sub_list(monkeypatch, workload, grid, normalize, generic):
    """SD-2.1 (15 layers) and SDXL (60) at square and rectangular sizes. One call holds: every layer alone at 3, 12 or
    77 rows (factors 1 / 2 / 4 as each map's only class, 4- and 8-row bands); every run of equally sized layers; ranges
    that mix two and three classes and start at a factor-2 or factor-4 layer; overlapping ranges; the whole list."""
    monkeypatch.setenv('DAAM_FINALIZE_GENERIC', '1' if generic else '0')
    layers = _layers(workload, grid)
    n = len(layers)
    stacks = _stacks(layers, seed=n)
    singles = [(i, 1, (3, 12, 77)[i % 3]) for i in range(n)]
    mixed = [(b, c, 12) for b, c in _runs(layers)] + [(0, n, 77), (0, n, 12), (1, n - 1, 12), (n // 3, n // 3, 77),
                                                      (n // 3 + 1, n // 2, 3), (n - 2, 2, 12), (2, 3, 40)]
    for parts in (singles, mixed):
        _check_parts(stacks, grid, parts, normalize, what=f'{workload} {grid}')
    _check_parts(stacks, grid, singles[:20] + mixed[-6:], normalize, head_sel=3, what=f'{workload} {grid} head_sel 3')


def test_fast_and_generic_agree(monkeypatch):
    """The same call on the banded kernel and, with DAAM_FINALIZE_GENERIC=1, on the gather kernel: the per-key
    arithmetic is the same, the order of the key sum is not."""
    layers = _layers('sd21', (64, 64))
    stacks = _stacks(layers, seed=7)
    parts = [(i, 1, 12) for i in range(len(layers))] + [(0, len(layers), 12)]
    monkeypatch.setenv('DAAM_FINALIZE_GENERIC', '0')
    fast = _check_parts(stacks, (64, 64), parts)
    monkeypatch.setenv('DAAM_FINALIZE_GENERIC', '1')
    generic = _check_parts(stacks, (64, 64), parts)
    for (b, c, _), f, g in zip(parts, fast, generic):
        torch.testing.assert_close(f, g, rtol=1e-5, atol=1e-5, msg=lambda m: f'part {(b, c)}: {m}')


def test_a_generic_map_between_fast_maps():
    """A 60 x 44 map whose factor-4 layer has 15 x 11 = 165 pixels, an odd count the banded kernel does not read: the
    maps that read that group take the generic kernel, their neighbours the fast one, in one call of two launches."""
    layers = [((60, 44), 2), ((30, 22), 3), ((15, 11), 3), ((30, 22), 2), ((60, 44), 1)]
    stacks = _stacks(layers, seed=60)
    before = _native.launch_count()
    _check_parts(stacks, (60, 44), [(0, 2, 12), (2, 1, 12), (3, 2, 12), (0, 5, 12), (1, 2, 9)])
    assert _native.launch_count() - before == 2 + 5        # fast + generic, then the five reference calls


def test_off_grid_parts():
    """SD-2.1 at 600x800: a 75 x 100 map over 75x100 / 38x50 / 19x25 layers. Every map that reads a 38x50 or 19x25
    layer (non-integer factors) takes the generic kernel; the 75x100 layers alone, parts (0, 1) and (4, 1), take the
    fast one with a partial last band of 3 rows (tests/test_finalize_geometry_gpu.py checks such maps against
    float64)."""
    layers = [((75, 100), 5), ((38, 50), 10), ((19, 25), 20), ((38, 50), 10), ((75, 100), 5)]
    stacks = _stacks(layers, seed=600)
    for normalize in (False, True):
        _check_parts(stacks, (75, 100), [(i, 1, 9) for i in range(5)] + [(0, 5, 77), (1, 3, 30)], normalize, what='600x800')


def test_a_map_over_2048_keys():
    """A range of 2100 keys takes the generic kernel, as daam_finalize does for it; the ranges inside it stay fast."""
    layers = [((32, 32), 700), ((16, 16), 700), ((32, 32), 700)]
    stacks = _stacks(layers, seed=2048, tokens=4)
    before = _native.launch_count()
    _check_parts(stacks, (32, 32), [(0, 3, 4), (0, 2, 4), (1, 2, 3), (2, 1, 4)], what='2100 keys')
    assert _native.launch_count() - before == 2 + 4


def test_sd21_against_float64():
    """SD-2.1's 15 layers at 64 x 64, 12 rows: every layer's map, every factor's and the all-layers map of one call
    against the float64 statement of the reduction."""
    layers = _layers('sd21', (64, 64))
    stacks = _stacks(layers, seed=21)
    order = sorted(range(len(layers)), key=lambda i: -layers[i][0][0])       # factor 1, 2, 4: contiguous runs
    stacks = [stacks[i] for i in order]
    layers = [layers[i] for i in order]
    parts = [(i, 1, 12) for i in range(len(layers))] + [(b, c, 12) for b, c in _runs(layers)] + [(0, len(layers), 12)]
    for normalize in (False, True):
        outs = _check_parts(stacks, (64, 64), parts, normalize)
        for (b, c, n), got in zip(parts, outs):
            keys = [t.view(t.shape[0], 77, h, w) for t, h, w in stacks[b:b + c]]
            rtol, atol = finalize_tolerance(keys, sum(k.shape[0] for k in keys), 64)
            raw = global_map64(keys, 64, n)
            if not normalize:
                assert_close64(got, raw, rtol, atol, f'part {(b, c)}')
            else:
                want = global_map64(keys, 64, n, normalize=True)
                assert_close64(got, want, 0.0, normalized_tolerance(raw, rtol, atol), f'part {(b, c)} normalized')


def test_launch_count_and_split():
    """15 maps: one launch, two with normalize. 65 maps: refused by the C entry point, split by the binding."""
    layers = _layers('sd21', (64, 64))
    stacks = _stacks(layers, seed=15)
    groups = _groups(stacks)
    out = torch.empty(15, 12, 64, 64, device=DEV)
    sel = [_native.DaamMapPart(group_begin=i, group_count=1, n_rows=12, out=out[i].data_ptr()) for i in range(15)]
    for normalize, launches in ((False, 1), (True, 2)):
        before = _native.launch_count()
        _native.finalize_parts(groups, sel, (64, 64), normalize, _stream())
        assert _native.launch_count() - before == launches
    outs = torch.empty(65, 5, 64, 64, device=DEV)
    sel = [_native.DaamMapPart(group_begin=i % 11, group_count=1 + i // 15, n_rows=5, out=outs[i].data_ptr())
           for i in range(65)]
    lib = _native.load()
    arr, raw = (_native.DaamKeyGroup * 15)(*groups), (_native.DaamMapPart * 65)(*sel)
    assert lib.daam_finalize_parts(arr, 15, raw, 65, 64, 64, 0, ctypes.c_void_p(_stream())) == _native.E_UNSUPPORTED
    assert b'65 maps > 64' in lib.daam_last_error()
    before = _native.launch_count()
    _native.finalize_parts(groups, sel, (64, 64), False, _stream())       # 64 + 1
    assert _native.launch_count() - before == 2
    ref = torch.empty(5, 64, 64, device=DEV)
    for i in range(65):
        _native.finalize(groups[i % 11:i % 11 + 1 + i // 15], (64, 64), 5, False, ref.data_ptr(), _stream())
        torch.cuda.synchronize()
        assert torch.equal(outs[i], ref), i


def _call(groups, maps, n_groups=None, n_maps=None, h=16, w=16):
    lib = _native.load()
    arr = (_native.DaamKeyGroup * max(len(groups), 1))(*groups)
    sel = (_native.DaamMapPart * max(len(maps), 1))(*maps) if maps is not None else None
    rc = lib.daam_finalize_parts(arr, len(groups) if n_groups is None else n_groups, sel,
                                 (len(maps) if maps else 0) if n_maps is None else n_maps, h, w, 0,
                                 ctypes.c_void_p(_stream()))
    return rc, lib.daam_last_error().decode()


def test_refusals():
    stacks = _stacks([((16, 16), 2), ((8, 8), 2), ((16, 16), 1)], seed=1)
    short = _stacks([((16, 16), 2)], seed=2, tokens=3)
    out = torch.empty(77, 16, 16, device=DEV)
    good_g = _groups(stacks)
    good_m = _native.DaamMapPart(group_begin=0, group_count=3, n_rows=4, out=out.data_ptr())
    assert _call(good_g, [good_m])[0] == 0
    # n_blocks is ignored, as in daam_finalize
    blocks = [_native.DaamKeyGroup(acc=g.acc, heads=g.heads, h=g.h, w=g.w, tokens=g.tokens, head_sel=-1, n_blocks=7)
              for g in good_g]
    assert _call(blocks, [good_m])[0] == 0

    def part(**kw):
        d = dict(group_begin=0, group_count=1, n_rows=4, out=out.data_ptr())
        d.update(kw)
        return _native.DaamMapPart(**d)

    bad_head = _native.DaamKeyGroup(acc=stacks[0][0].data_ptr(), heads=2, h=16, w=16, tokens=77, head_sel=2, n_blocks=0)
    cases = [
        (good_g, None, {'n_maps': 0}, _native.E_INVALID, 'no output map'),
        (good_g, [good_m], {'n_maps': 0}, _native.E_INVALID, 'no output map'),
        (good_g, [part(out=None)], {}, _native.E_INVALID, 'bad map 0'),
        (good_g, [good_m, part(n_rows=0)], {}, _native.E_INVALID, 'bad map 1'),
        (good_g, [part(group_begin=-1)], {}, _native.E_INVALID, 'bad map 0'),
        (good_g, [part(group_count=0)], {}, _native.E_INVALID, 'bad map 0'),
        (good_g, [part(group_begin=2, group_count=2)], {}, _native.E_INVALID, 'groups [2, +2) of 3'),
        (good_g, [part(group_begin=3)], {}, _native.E_INVALID, 'groups [3, +1) of 3'),
        (good_g, [good_m], {'n_groups': 0}, _native.E_INVALID, 'no key selected'),
        (good_g * 54, [good_m], {}, _native.E_UNSUPPORTED, '162 key groups > 160'),
        (good_g + [bad_head], [good_m], {}, _native.E_INVALID, 'bad key group 3'),      # even when no map reads it
        (good_g, [part(n_rows=78)], {}, _native.E_INVALID, 'reads 78 rows but key group 0 holds 77'),
        (good_g + _groups(short), [part(group_begin=1, group_count=3)], {}, _native.E_INVALID,
         'map 0 reads 4 rows but key group 3 holds 3'),
        (good_g, [good_m] * 65, {}, _native.E_UNSUPPORTED, '65 maps > 64'),
        (good_g, [good_m], {'h': 0}, _native.E_INVALID, 'non-positive size'),
    ]
    for groups, maps, kw, code, msg in cases:
        rc, err = _call(groups, maps, **kw)
        assert rc == code and msg in err and err.startswith('daam_finalize_parts'), (kw, msg, rc, err)
    # a short group is fine for the maps that fit it or do not read it
    assert _call(good_g + _groups(short), [part(group_begin=3, n_rows=3), part(group_count=3, n_rows=77)])[0] == 0
    torch.cuda.synchronize()
