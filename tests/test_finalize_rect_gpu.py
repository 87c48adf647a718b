"""The finalize / word-map / expand entry points on rectangular ``(map_h, map_w)`` grids against float64 torch: every
key as ``B_y @ key @ B_x^T`` with ``bicubic64(kh, xh)`` / ``bicubic64(kw, xw)``, then clamp, mean and normalise, within
the finalize tolerances of ``test_production_sizes_gpu.py``. Fast and generic kernels, the grids of SD-2.1 at 512x768 /
768x512 and SDXL at 1216x832 / 1344x768 / 1152x896 (26-wide key rows), a 13-wide key row, an odd grid that falls back,
and the refusals, which name the entry point that was called."""
import pytest
import torch

from daam_b200 import _native
from tests.reference64 import (MAP_DIMS, assert_close64, bicubic64, finalize_tolerance, normalized_tolerance)

pytestmark = pytest.mark.gpu
DEV = 'cuda'

# grid (xh, xw) and the key sizes of its traced levels (factor 1, 2, 4; SDXL has no factor-4 layer); heads per level
GRIDS = {
    'sd21-512x768': ((96, 64), [(96, 64), (48, 32), (24, 16)], [5, 10, 20]),
    'sd21-768x512': ((64, 96), [(64, 96), (32, 48), (16, 24)], [5, 10, 20]),
    'sdxl-1216x832': ((76, 52), [(76, 52), (38, 26)], [10, 20]),
    'sdxl-1344x768': ((84, 48), [(84, 48), (42, 24)], [10, 20]),
    'sdxl-1152x896': ((72, 56), [(72, 56), (36, 28)], [10, 20]),
    'narrow-13': ((64, 52), [(64, 52), (32, 26), (16, 13)], [2, 3, 4]),     # 13-wide factor-4 rows (4-byte units)
    'odd-75x100': ((75, 100), [(75, 100), (38, 50), (19, 25)], [2, 2, 2]),   # non-integer factors: generic only
}


def _stacks(name, seed, layers_per_level=2):
    grid, sizes, heads = GRIDS[name]
    g = torch.Generator(device=DEV).manual_seed(seed)
    stacks = [torch.exp(torch.randn(h, 77, kh, kw, generator=g, device=DEV))
              for (kh, kw), h in zip(sizes, heads) for _ in range(layers_per_level)]
    return grid, stacks


def _groups(stacks, head_sel=None):
    return [_native.DaamKeyGroup(acc=t.data_ptr(), heads=t.shape[0], h=t.shape[2], w=t.shape[3], tokens=t.shape[1],
                                 head_sel=-1 if head_sel is None else head_sel, reserved=0) for t in stacks]


def _up64(keys, grid):
    by = bicubic64(keys.shape[-2], grid[0], keys.device)
    bx = bicubic64(keys.shape[-1], grid[1], keys.device)
    return by @ keys.double() @ bx.T


def _norm64(maps):
    return maps / (maps[..., 1:-1, :, :].sum(dim=-3, keepdim=True) + 1e-6)


def _reference(stacks, grid, n_rows, normalize, head_sel):
    total, n = None, 0
    for t in stacks:
        sel = t[:, :n_rows] if head_sel is None else t[head_sel:head_sel + 1, :n_rows]
        part = _up64(sel, grid).clamp_(min=0.0).sum(dim=0)
        total = part if total is None else total + part
        n += sel.shape[0]
    ref = total / n
    rtol, atol = finalize_tolerance(stacks, n, max(grid))
    if normalize:
        atol = normalized_tolerance(ref, rtol, atol)
        ref, rtol = _norm64(ref), 0.0
    return ref, rtol, atol


def _finalize(monkeypatch, groups, grid, n_rows, normalize, generic, per_key=0):
    monkeypatch.setenv('DAAM_FINALIZE_GENERIC', '1' if generic else '0')
    out = torch.empty(((per_key,) if per_key else ()) + (n_rows,) + grid, device=DEV)
    fn = _native.finalize_per_key if per_key else _native.finalize
    fn(groups, grid, n_rows, normalize, out.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return out


def _bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.parametrize('name', list(GRIDS))
@pytest.mark.parametrize('n_rows', [12, 40, 77])
def test_finalize_rect_against_float64(monkeypatch, name, n_rows):
    grid, stacks = _stacks(name, n_rows)
    options = [{}, {'normalize': True}, {'head_sel': 1}] if n_rows == 40 else [{}]
    for opt in options:
        normalize, head_sel = opt.get('normalize', False), opt.get('head_sel')
        ref, rtol, atol = _reference(stacks, grid, n_rows, normalize, head_sel)
        groups = _groups(stacks, head_sel)
        what = f'{name} n_rows {n_rows} {opt}'
        fast = _finalize(monkeypatch, groups, grid, n_rows, normalize, generic=False)
        again = _finalize(monkeypatch, groups, grid, n_rows, normalize, generic=False)
        generic = _finalize(monkeypatch, groups, grid, n_rows, normalize, generic=True)
        assert torch.equal(_bits(fast), _bits(again)), f'{what}: two runs differ'
        assert_close64(fast, ref, rtol, atol, f'fast {what}', MAP_DIMS)
        assert_close64(generic, ref, rtol, atol, f'generic {what}', MAP_DIMS)


@pytest.mark.parametrize('name', ['sd21-512x768', 'sdxl-1216x832', 'narrow-13', 'odd-75x100'])
@pytest.mark.parametrize('normalize', [False, True])
def test_finalize_per_key_rect(monkeypatch, name, normalize):
    grid, stacks = _stacks(name, 5, layers_per_level=1)
    n_rows = 40
    n_keys = sum(t.shape[0] for t in stacks)
    out = _finalize(monkeypatch, _groups(stacks), grid, n_rows, normalize, generic=False, per_key=n_keys)
    first = 0
    for i, t in enumerate(stacks):
        raw = _up64(t[:, :n_rows], grid).clamp_(min=0.0)
        for h in range(t.shape[0]):
            rtol, atol = finalize_tolerance([t[h:h + 1]], 1, max(grid))
            ref = raw[h]
            if normalize:
                atol = normalized_tolerance(ref, rtol, atol)
                ref, rtol = _norm64(ref), 0.0
            assert_close64(out[first + h], ref, rtol, atol, f'{name} layer {i} head {h}', MAP_DIMS)
        first += t.shape[0]


def _expand64(word_map, out_h, out_w, absolute, threshold):
    im = _up64(word_map[None], (out_h, out_w))[0]
    if not absolute:
        im = (im - im.min()) / (im.max() - im.min() + 1e-8)
    if threshold:
        im = (im > threshold).double()
    return im


@pytest.mark.parametrize('grid,out_hw', [((96, 64), (768, 512)), ((64, 96), (512, 768)), ((76, 52), (1216, 832)),
                                         ((84, 48), (1344, 768)), ((75, 100), (600, 800))])
def test_word_maps_and_expand_words_rect(grid, out_hw):
    g = torch.Generator(device=DEV).manual_seed(3)
    n_rows = 12
    maps = torch.rand((n_rows,) + grid, generator=g, device=DEV)
    words = [[1], [2, 3], [4], [5, 6, 7], [8], [9], [10], [1, 10]]
    stream = torch.cuda.current_stream().cuda_stream
    for rows in words:
        out = torch.empty(grid, device=DEV)
        _native.word_heat_map(maps.data_ptr(), n_rows, grid, rows, out.data_ptr(), stream)
        torch.cuda.synchronize()
        assert_close64(out, maps[rows].double().mean(0), 1e-6, 0.0, f'word map {rows}')
    for absolute, threshold in [(False, None), (True, None), (False, 0.4)]:
        word_maps = torch.empty((len(words),) + grid, device=DEV)
        out = torch.empty((len(words),) + out_hw, device=DEV)
        scratch = torch.empty(_native.EXPAND_SCRATCH_FLOATS * len(words), device=DEV)
        _native.expand_words(maps.data_ptr(), n_rows, grid, words, out_hw[0], out_hw[1], absolute, threshold,
                             word_maps.data_ptr(), out.data_ptr(), scratch.data_ptr(), stream)
        single = torch.empty(out_hw, device=DEV)
        torch.cuda.synchronize()
        for i, rows in enumerate(words):
            wm = maps[rows].double().mean(0)
            assert_close64(word_maps[i], wm, 1e-6, 0.0, f'word map {i}')
            ref = _expand64(word_maps[i].double(), *out_hw, absolute, threshold)
            what = f'expand {grid}->{out_hw} word {i} absolute={absolute} threshold={threshold}'
            if threshold:   # binarised: only pixels within float error of the threshold may flip
                near = (_expand64(word_maps[i].double(), *out_hw, absolute, None) - threshold).abs() < 1e-5
                assert bool(((out[i].double() == ref) | near).all()), what
            else:
                assert_close64(out[i], ref, 1e-5, 1e-6, what)
            _native.expand_as(word_maps[i].data_ptr(), grid, out_hw[0], out_hw[1], absolute, threshold,
                              single.data_ptr(), scratch.data_ptr(), stream)
            torch.cuda.synchronize()
            assert torch.equal(single, out[i]), f'{what}: expand_as differs from expand_words'


def test_refusals_name_the_entry_point_called():
    stream = torch.cuda.current_stream().cuda_stream
    maps = torch.zeros(3, 300, 200, device=DEV)
    out = torch.empty(2, 8, 8, device=DEV)
    scratch = torch.empty(64, device=DEV)
    with pytest.raises(_native.NativeError, match='daam_expand_words: a 300 x 200 map does not fit shared memory'):
        _native.expand_words(maps.data_ptr(), 3, (300, 200), [[1]], 8, 8, False, None, None, out.data_ptr(),
                             scratch.data_ptr(), stream)
    with pytest.raises(_native.NativeError, match='daam_expand_as: a 300 x 200 map does not fit shared memory'):
        _native.expand_as(maps.data_ptr(), (300, 200), 8, 8, False, None, out.data_ptr(), scratch.data_ptr(), stream)
    with pytest.raises(_native.NativeError, match='daam_finalize: null pointer or non-positive size'):
        _native.finalize(_groups([torch.zeros(1, 77, 4, 4, device=DEV)]), (0, 4), 2, False, out.data_ptr(), stream)
