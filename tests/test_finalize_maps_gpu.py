"""daam_finalize_maps through the C ABI: map m of one call is bit-identical (torch.equal) to daam_finalize over the
expanded group list `for g: for b in map m's blocks: {acc_g + b * block_stride_g, heads_g, head_sel_g}`, on the fast
and the generic kernel, square, rectangular and off-grid maps, with and without normalisation, maps of different row
counts (and so band heights) and kinds in one call, up to and past the map limit; and every refusal."""
import ctypes

import pytest
import torch

import bench
from daam_b200 import _native

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def _key_stacks(keys_hw, heads, n_blocks, seed):
    """One fp32 stack [n_blocks, heads, 77, h * w] of seeded randn maps per layer (negative values too, so the clamp
    matters); ``keys_hw[i] = (h, w)``."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    return [(torch.randn(n_blocks, hd, 77, h * w, generator=g, device=DEV), h, w) for (h, w), hd in zip(keys_hw, heads)]


def _groups(stacks, head_sel=-1):
    return [_native.DaamKeyGroup(acc=t.data_ptr(), heads=t.shape[1], h=h, w=w, tokens=77, head_sel=head_sel,
                                 n_blocks=t.shape[0]) for t, h, w in stacks]


def _expanded(stacks, blocks, head_sel=-1):
    return [_native.DaamKeyGroup(acc=t[b].data_ptr(), heads=t.shape[1], h=h, w=w, tokens=77, head_sel=head_sel,
                                 n_blocks=0) for t, h, w in stacks for b in blocks]


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _check_maps(stacks, grid, sels, normalize, head_sel=-1, what=''):
    """sels: [(block_begin, block_count, n_rows)]; one daam_finalize_maps call against one daam_finalize per map."""
    outs = [torch.full((n,) + grid, float('nan'), device=DEV) for _, _, n in sels]
    maps = [_native.DaamMapSel(block_begin=b, block_count=c, n_rows=n, out=o.data_ptr())
            for (b, c, n), o in zip(sels, outs)]
    _native.finalize_maps(_groups(stacks, head_sel), maps, grid, normalize, _stream())
    for (b, c, n), got in zip(sels, outs):
        ref = torch.empty((n,) + grid, device=DEV)
        _native.finalize(_expanded(stacks, range(b, b + c), head_sel), grid, n, normalize, ref.data_ptr(), _stream())
        torch.cuda.synchronize()
        assert torch.isfinite(got).all(), f'{what} map {(b, c, n)}: not written'
        assert torch.equal(got, ref), f'{what} map {(b, c, n)}: differs from daam_finalize on the expanded groups'


def _layers(workload, latent_hw):
    """The traced layers of a bench workload at latent (H, W): ((h, w), heads) per layer."""
    layers = bench.traced_layers(workload)
    side = max(int(round(hw ** 0.5)) for hw, _, _ in layers)
    lh, lw = latent_hw
    return [((lh * int(round(hw ** 0.5)) // side, lw * int(round(hw ** 0.5)) // side), h) for hw, h, _ in layers]


# (workload, map grid = the finest layer's size, blocks = images)
CASES = [('sd21', (64, 64), 3), ('sd21', (64, 96), 3), ('sdxl', (64, 64), 2), ('sdxl', (76, 52), 2)]


@pytest.mark.parametrize('generic', [False, True])
@pytest.mark.parametrize('normalize', [False, True])
@pytest.mark.parametrize('workload,grid,blocks', CASES)
def test_maps_equal_finalize_on_expanded_groups(monkeypatch, workload, grid, blocks, normalize, generic):
    """SD-2.1 (175 keys per block) and SDXL (60 layers) at square and rectangular sizes (512x768, 1216x832): every
    block alone and the blend of all blocks, at 12, 40 and 77 rows -- 4- and 8-row bands on an H100 -- in one call.
    SDXL's blend has 2200 keys and so takes the generic kernel next to per-block maps on the fast one."""
    monkeypatch.setenv('DAAM_FINALIZE_GENERIC', '1' if generic else '0')
    layers = _layers(workload, grid)
    stacks = _key_stacks([hw for hw, _ in layers], [h for _, h in layers], blocks, seed=len(layers) + blocks)
    sels = [(b, 1, (12, 77, 40)[b % 3]) for b in range(blocks)] + [(0, blocks, 40), (1, blocks - 1, 12)]
    _check_maps(stacks, grid, sels, normalize, what=f'{workload} {grid}')
    _check_maps(stacks, grid, [(b, 1, 12) for b in range(blocks)] + [(0, blocks, 77)], normalize, head_sel=1,
                what=f'{workload} {grid} head_sel 1')


def test_maps_off_grid_generic():
    """SD-2.1 at 600x800: a 75 x 100 map, layers 75x100 / 38x50 / 19x25 (odd pixel counts, non-integer factors), so
    every map takes the generic kernel."""
    layers = [((75, 100), 5), ((38, 50), 10), ((19, 25), 20), ((38, 50), 10), ((75, 100), 5)]
    stacks = _key_stacks([hw for hw, _ in layers], [h for _, h in layers], 2, seed=600)
    for normalize in (False, True):
        _check_maps(stacks, (75, 100), [(0, 1, 9), (1, 1, 77), (0, 2, 9)], normalize, what='600x800')
        _check_maps(stacks, (75, 100), [(1, 1, 9), (0, 2, 30)], normalize, head_sel=4, what='600x800 head_sel')


def test_map_limit_and_split():
    """64 maps in one call; 65 are refused by the C entry point and split by the binding, with the same bits."""
    stacks = _key_stacks([(16, 16), (8, 8)], [2, 4], 65, seed=64)
    grid = (16, 16)
    outs = torch.empty((65, 5) + grid, device=DEV)
    maps = [_native.DaamMapSel(block_begin=b, block_count=1, n_rows=5, out=outs[b].data_ptr()) for b in range(65)]
    lib = _native.load()
    groups = _groups(stacks)
    arr = (_native.DaamKeyGroup * 2)(*groups)
    sel = (_native.DaamMapSel * 65)(*maps)
    assert _native.FINALIZE_MAX_MAPS == 64
    assert lib.daam_finalize_maps(arr, 2, sel, 65, 16, 16, 0, ctypes.c_void_p(_stream())) == _native.E_UNSUPPORTED
    assert b'65 maps > 64' in lib.daam_last_error()
    assert lib.daam_finalize_maps(arr, 2, sel, 64, 16, 16, 0, ctypes.c_void_p(_stream())) == 0
    torch.cuda.synchronize()
    first = outs.clone()
    _native.finalize_maps(groups, maps, grid, False, _stream())       # 64 + 1
    ref = torch.empty((5,) + grid, device=DEV)
    for b in range(65):
        _native.finalize(_expanded(stacks, [b]), grid, 5, False, ref.data_ptr(), _stream())
        torch.cuda.synchronize()
        assert torch.equal(outs[b], ref), b
        if b < 64:
            assert torch.equal(first[b], ref), b


def _call(groups, maps, n_groups=None, n_maps=None, h=16, w=16):
    lib = _native.load()
    arr = (_native.DaamKeyGroup * max(len(groups), 1))(*groups)
    sel = (_native.DaamMapSel * max(len(maps), 1))(*maps) if maps is not None else None
    rc = lib.daam_finalize_maps(arr, len(groups) if n_groups is None else n_groups, sel,
                                (len(maps) if maps else 0) if n_maps is None else n_maps, h, w, 0,
                                ctypes.c_void_p(_stream()))
    return rc, lib.daam_last_error().decode()


def test_refusals():
    stacks = _key_stacks([(16, 16)], [2], 3, seed=1)
    out = torch.empty(77, 16, 16, device=DEV)
    good_g = _groups(stacks)
    good_m = _native.DaamMapSel(block_begin=0, block_count=3, n_rows=4, out=out.data_ptr())
    assert _call(good_g, [good_m])[0] == 0

    def sel(**kw):
        d = dict(block_begin=0, block_count=1, n_rows=4, out=out.data_ptr())
        d.update(kw)
        return _native.DaamMapSel(**d)

    cases = [
        (good_g, None, {'n_maps': 0}, _native.E_INVALID, 'no output map'),
        (good_g, [good_m], {'n_maps': 0}, _native.E_INVALID, 'no output map'),
        (good_g, [sel(out=None)], {}, _native.E_INVALID, 'bad map 0'),
        (good_g, [good_m, sel(n_rows=0)], {}, _native.E_INVALID, 'bad map 1'),
        (good_g, [sel(block_begin=-1)], {}, _native.E_INVALID, 'bad map 0'),
        (good_g, [sel(block_count=0)], {}, _native.E_INVALID, 'bad map 0'),
        (good_g, [sel(block_begin=2, block_count=2)], {}, _native.E_INVALID, 'reads blocks [2, 4) but key group 0 holds 3'),
        ([_native.DaamKeyGroup(acc=stacks[0][0].data_ptr(), heads=2, h=16, w=16, tokens=77, head_sel=-1, n_blocks=0)],
         [good_m], {}, _native.E_INVALID, 'holds 0'),
        (good_g, [good_m], {'n_groups': 0}, _native.E_INVALID, 'no key selected'),
        (good_g * 161, [good_m], {}, _native.E_UNSUPPORTED, '161 key groups > 160'),
        ([_native.DaamKeyGroup(acc=stacks[0][0].data_ptr(), heads=2, h=16, w=16, tokens=77, head_sel=2, n_blocks=3)],
         [good_m], {}, _native.E_INVALID, 'bad key group 0'),
        (good_g, [sel(n_rows=78)], {}, _native.E_INVALID, 'bad key group 0'),
        (good_g, [good_m] * 65, {}, _native.E_UNSUPPORTED, '65 maps > 64'),
        (good_g, [good_m], {'h': 0}, _native.E_INVALID, 'non-positive size'),
    ]
    for groups, maps, kw, code, msg in cases:
        rc, err = _call(groups, maps, **kw)
        assert rc == code and msg in err and err.startswith('daam_finalize_maps'), (kw, msg, rc, err)
    with pytest.raises(_native.NativeError, match='no output map'):
        _native.finalize_maps(good_g, [], (16, 16), False, _stream())
