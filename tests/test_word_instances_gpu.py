"""Word instances (GlobalHeatMap.word_instances, GlobalHeatMapStack.word_instances, daam_word_instances) on the GPU.

Every field must equal the exact integer oracle ``tests/components64.py`` run on ``expand_words(..., threshold=None)``
compared against the threshold:

* image sizes: SD-2.1 512^2, SDXL 1024^2 and 1216x832, off-grid 600x800, a square map over a non-square image, and an
  output smaller than the map;
* crafted masks: with ``absolute=True`` and the image the size of the grid the bicubic taps are the identity, so a
  word's row is its mask: spirals and U-shapes across many 32 x 32 labelling tiles, diagonal chains through tile
  corners, components on every tile seam at +-1 pixel, the isolated-pixel lattice, a full plane, an empty mask and
  single corner pixels;
* ranking at K = 1, 16 and 64 with more components than K and area ties;
* stacks from the synthetic pipeline (a time-resolved history and a layer stack), row t equal to ``self[t]``;
* the same bits with scratch for 1, 3 or every plane, and on a repeated call; the C ABI's refusals.
"""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from daam_b200 import _native, trace
from daam_b200.heatmap import GlobalHeatMap
from daam_b200.testing.synthetic import TINY_SPEC, WhitespaceTokenizer, make_pipeline
from tests.components64 import instances64_stack

pytestmark = pytest.mark.gpu
DEV = 'cuda'
TOK = WhitespaceTokenizer()
PROMPT100 = ' '.join(f'w{i}' for i in range(100))
PROMPT = 'a dog chasing a red ball on the beach'
FIELDS = ('count', 'area', 'box', 'sum_yx', 'peak', 'peak_yx')
TILE = 32                                               # the labelling tile of components.cu


def image(h, w):
    return SimpleNamespace(size=(w, h), height=h, width=w)


def rand_maps(grid, seed, n_rows=102, scale=1.0):
    return (torch.rand(n_rows, *grid, generator=torch.Generator().manual_seed(seed)) * scale).to(DEV)


def assert_equal_oracle(inst, pre, threshold, k):
    """Every field of ``inst`` equals the oracle of ``pre`` ``[..., W, H, W]``."""
    ref = instances64_stack(pre.cpu().numpy(), threshold, k)
    for f in FIELDS:
        got = getattr(inst, f).cpu().numpy()
        assert got.shape == ref[f].shape, f
        np.testing.assert_array_equal(got, ref[f].astype(got.dtype), err_msg=f)


def check(ghm, words, img, threshold, absolute=False, k=16):
    """word_instances of one map against the oracle of its expand_words values; returns the instances."""
    _, pre = ghm.expand_words(words, img, absolute=absolute, to_cpu=False)
    _, mask = ghm.expand_words(words, img, absolute=absolute, threshold=threshold, to_cpu=False)
    assert torch.equal(mask, (pre > torch.tensor(threshold, dtype=torch.float32)).float())
    whms, inst = ghm.word_instances(words, img, threshold, absolute=absolute, max_instances=k, to_cpu=False)
    assert [w.word for w in whms] == list(words) and inst.count.is_cuda
    assert inst.count.dtype == torch.int32 and inst.sum_yx.dtype == torch.int64 and inst.peak.dtype == torch.float32
    assert_equal_oracle(inst, pre, threshold, k)
    return inst


# (map grid, image (h, w)): SD-2.1 512^2, SDXL 1024^2, SDXL 1216x832, off-grid 600x800, a square map over a
# non-square image (the reference's (size[0], size[1]) order: 640 x 480), and an output smaller than the map
SIZES = [((64, 64), (512, 512)), ((128, 128), (1024, 1024)), ((76, 52), (1216, 832)), ((75, 100), (600, 800)),
         ((64, 64), (480, 640)), ((96, 96), (40, 56))]


@pytest.mark.parametrize('absolute,threshold,scale', [(False, 0.4, 1.0), (True, 0.3, 0.5)])
@pytest.mark.parametrize('grid,hw', SIZES, ids=[f'{g[0]}x{g[1]}-{h}x{w}' for g, (h, w) in SIZES])
def test_image_sizes(grid, hw, absolute, threshold, scale):
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps(grid, 5 * grid[0] + grid[1], scale=scale))
    inst = check(ghm, ['w1', 'w40 w41', 'w7', 'w1'], image(*hw), threshold, absolute)
    assert torch.equal(inst.area[0], inst.area[3])                     # a repeated word repeats its instances
    assert bool((inst.count > 0).all())


# ---- crafted masks -------------------------------------------------------------------------------------------------
def spiral(h, w):
    m = np.zeros((h, w), bool)
    y0, x0, y1, x1 = 0, 0, h - 1, w - 1
    while y0 <= y1 and x0 <= x1:
        m[y0, x0:x1 + 1] = m[y0:y1 + 1, x1] = m[y1, x0:x1 + 1] = True
        m[y0 + 2:y1 + 1, x0] = True
        y0, x0, y1, x1 = y0 + 2, x0 + 2, y1 - 2, x1 - 2
        if y0 <= y1:
            m[y0 - 1, x0] = False
    return m


def snake(h, w):
    """One path through every other row, turning at alternate ends: a single component across every tile."""
    m = np.zeros((h, w), bool)
    m[::2] = True
    for y in range(1, h - 1, 2):
        m[y, w - 1 if (y // 2) % 2 == 0 else 0] = True
    return m


def u_shapes(h, w):
    """Two arms down from the top that join only along the bottom row, far from where they start, and an inverted U
    whose arms meet only along the top of the last tile row."""
    m = np.zeros((h, w), bool)
    m[:, 3] = m[:, w - 5] = m[h - 1, 3:w - 4] = True
    m[40:h - 8, 20] = m[40:h - 8, w - 30] = m[40, 20:w - 29] = True
    return m


def diagonals(h, w):
    """Chains of single pixels that pass from tile to tile only through tile corners (8-connectivity)."""
    m = np.zeros((h, w), bool)
    n = min(h, w)
    i = np.arange(n)
    m[i, i] = True
    m[i, w - 1 - i] = True
    m[i[::2] // 2 + h // 2 - n // 4, i[::2] // 2] = True
    return m


def seams(h, w):
    """On every seam s of the 32 x 32 tiles: pairs across it (vertical, horizontal, diagonal both ways), pixels one
    off it on both sides (separate components), and pixels just before and after it."""
    m = np.zeros((h, w), bool)
    for s in range(TILE, h, TILE):
        for x in range(2, w - 8, 9):
            m[s - 1, x] = m[s, x] = True                        # vertical pair across a horizontal seam
            m[s - 1, x + 3] = m[s, x + 4] = True                # diagonal pair
            m[s - 1, x + 7] = True                              # one pixel above
    for s in range(TILE, w, TILE):
        for y in range(5, h - 8, 11):
            m[y, s - 1] = m[y, s] = True                        # horizontal pair across a vertical seam
            m[y + 3, s] = m[y + 4, s - 1] = True                # anti-diagonal pair
            m[y + 7, s + 1] = True                              # one pixel past the seam
    return m


def lattice(h, w):
    m = np.zeros((h, w), bool)
    m[::2, ::2] = True
    return m


def corners(h, w):
    m = np.zeros((h, w), bool)
    m[0, 0] = m[0, w - 1] = m[h - 1, 0] = m[h - 1, w - 1] = True
    return m


def checkerboard(h, w):
    return np.indices((h, w)).sum(0) % 2 == 0


MASKS = {'spiral': spiral, 'snake': snake, 'u-shapes': u_shapes, 'diagonals': diagonals, 'seams': seams, 'lattice': lattice,
         'corners': corners, 'checkerboard': checkerboard, 'full': lambda h, w: np.ones((h, w), bool),
         'empty': lambda h, w: np.zeros((h, w), bool)}


def crafted(masks, seed):
    """Global maps whose row of word ``w{i}`` is mask i, with values in (0.5, 1] on the mask (a few repeated, so the
    peak has ties) and [0, 0.5) off it; the other rows are 0."""
    h, w = masks[0].shape
    g = np.random.default_rng(seed)
    maps = np.zeros((102, h, w), np.float32)
    for i, m in enumerate(masks):
        on = 1.0 - np.floor(g.random((h, w)) * 8) / 16                 # 8 levels: ties
        maps[i + 1] = np.where(m, on, g.random((h, w), dtype=np.float32) * 0.5)
    return torch.from_numpy(maps).to(DEV)


# the grid's size limit (200 KB in shared memory): 224 x 224 is 7 x 7 labelling tiles, 160 x 320 is 5 x 10
@pytest.mark.parametrize('hw', [(224, 224), (160, 320), (157, 301)], ids=['224x224', '160x320', '157x301'])
def test_crafted_masks(hw):
    names = list(MASKS)
    masks = [MASKS[n](*hw) for n in names]
    ghm = GlobalHeatMap(TOK, PROMPT100, crafted(masks, hw[0] + hw[1]))
    words = [f'w{i}' for i in range(len(names))]
    _, pre = ghm.expand_words(words, image(*hw), absolute=True, to_cpu=False)
    assert torch.equal(pre, ghm.heat_maps[1:len(names) + 1])           # identity taps: the rows themselves
    inst = check(ghm, words, image(*hw), 0.5, absolute=True, k=64)
    count = dict(zip(names, inst.count.tolist()))
    h, w = hw
    assert count['snake'] == 1 and count['u-shapes'] == 2 and count['checkerboard'] == 1 and count['full'] == 1
    assert count['lattice'] == ((h + 1) // 2) * ((w + 1) // 2) and count['corners'] == 4 and count['empty'] == 0
    full = names.index('full')
    assert inst.area[full, 0] == h * w and inst.box[full, 0].tolist() == [0, 0, h, w]
    e = names.index('empty')
    assert int(inst.area[e].abs().sum() + inst.box[e].abs().sum() + inst.peak[e].abs().sum()) == 0


@pytest.mark.parametrize('k', [1, 16, 64])
def test_ranking_and_ties(k):
    h, w = 192, 256
    g = np.random.default_rng(k)
    blobs = np.zeros((h, w), bool)
    for _ in range(150):                                   # rectangles of a few sizes: many equal areas
        y, x, s = g.integers(0, h - 6), g.integers(0, w - 6), g.integers(1, 4)
        blobs[y:y + s, x:x + s] = True
    masks = [blobs, lattice(h, w), g.random((h, w)) < 0.3]
    ghm = GlobalHeatMap(TOK, PROMPT100, crafted(masks, k))
    inst = check(ghm, ['w0', 'w1', 'w2'], image(h, w), 0.5, absolute=True, k=k)
    assert bool((inst.count > k).all())
    lat = inst.box[1, :, :2].tolist()                      # lattice: every area is 1, so raster order
    assert lat == [[2 * (i // ((w + 1) // 2)), 2 * (i % ((w + 1) // 2))] for i in range(k)]


def test_threshold_is_the_expand_words_mask_with_negative_values():
    # absolute maps with negative values: the peak's orderable bits, and a negative threshold
    maps = (rand_maps((64, 64), 3) - 0.6)
    ghm = GlobalHeatMap(TOK, PROMPT100, maps)
    check(ghm, ['w2', 'w3'], image(512, 512), -0.2, absolute=True)
    check(ghm, ['w2', 'w3'], image(512, 512), 0.1, absolute=True)


# ---- stacks ----------------------------------------------------------------------------------------------------------
def check_stack(stack, words, img, threshold, absolute=False, k=16):
    word_maps, inst = stack.word_instances(words, img, threshold, absolute=absolute, max_instances=k, to_cpu=False)
    assert tuple(inst.area.shape) == (len(stack), len(words), k)
    for t in range(len(stack)):
        whms, row = stack[t].word_instances(words, img, threshold, absolute=absolute, max_instances=k, to_cpu=False)
        for f in FIELDS:
            assert torch.equal(getattr(inst, f)[t], getattr(row, f)), (t, f)
        for i, whm in enumerate(whms):
            assert torch.equal(word_maps[t, i], whm.heatmap)
        _, pre = stack[t].expand_words(words, img, absolute=absolute, to_cpu=False)
        assert_equal_oracle(row, pre, threshold, k)
    return inst


def test_time_resolved_history_and_layer_stack():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=5)
    with trace(pipe, time_resolved=True) as tc:
        pipe(PROMPT, num_inference_steps=4, generator=torch.Generator().manual_seed(3))
        tm = tc.compute_time_heat_maps()
        by_layer = tc.compute_layer_heat_maps()
    assert len(tm) == 4 and len(by_layer) > 1
    check_stack(tm, ['dog', 'red ball', 'beach'], image(512, 512), 0.4)
    check_stack(by_layer, ['dog', 'ball'], image(512, 512), 0.4)
    _, inst = tm.word_instances(['dog'], image(512, 512), 0.4)
    assert not inst.count.is_cuda and tuple(inst.centroid().shape) == (4, 1, 16, 2)


# ---- rounds, repeats and the C ABI -----------------------------------------------------------------------------------
def native_call(maps, grid, rows, out_hw, threshold, k, scratch_planes, absolute=False, scratch_bytes=None):
    n_maps, n_words = maps.shape[0], len(rows)
    plane = _native.word_instances_plane_bytes(*out_hw)
    scratch = torch.empty(scratch_bytes or plane * scratch_planes, dtype=torch.uint8, device=DEV)
    word_maps = torch.empty((n_maps, n_words) + grid, device=DEV)
    i32 = dict(dtype=torch.int32, device=DEV)
    out = [torch.full((n_maps, n_words), -7, **i32), torch.full((n_maps, n_words, k), -7, **i32),
           torch.full((n_maps, n_words, k, 4), -7, **i32), torch.full((n_maps, n_words, k, 2), -7, dtype=torch.int64,
                                                                         device=DEV),
           torch.full((n_maps, n_words, k), -7.0, device=DEV), torch.full((n_maps, n_words, k, 2), -7, **i32)]
    before = _native.launch_count()
    _native.word_instances(maps.data_ptr(), n_maps, maps.shape[1], grid, rows, *out_hw, absolute, threshold, k,
                           word_maps.data_ptr(), *(t.data_ptr() for t in out), scratch.data_ptr(), scratch.numel(),
                           torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return out, word_maps, _native.launch_count() - before


def test_rounds_and_repeats_give_the_same_bits():
    grid, out_hw, k = (64, 64), (384, 320), 16
    maps = torch.stack([rand_maps(grid, 40 + i) for i in range(2)])
    rows = [[1], [5, 6], [9], [13], [20]]                                 # 2 maps x 5 words: 10 planes
    full, word_maps, launches = native_call(maps, grid, rows, out_hw, 0.4, k, 10)
    assert launches == 7
    # 3 planes: words [0, 3) and [3, 5) of each map; 7: one map a round
    for planes, rounds in ((1, 10), (3, 4), (7, 2), (10, 1)):
        out, wm, launches = native_call(maps, grid, rows, out_hw, 0.4, k, planes)
        assert launches == 7 * rounds, planes
        for a, b in zip(out, full):
            assert torch.equal(a, b), planes
        assert torch.equal(wm, word_maps)
    again, _, _ = native_call(maps, grid, rows, out_hw, 0.4, k, 10)
    for a, b in zip(again, full):
        assert torch.equal(a, b)
    for t in range(2):                                                  # and the Python call on each map
        ghm = GlobalHeatMap(TOK, PROMPT100, maps[t])
        # a square map keeps the reference's (size[0], size[1]) order: this image expands to out_hw
        _, pre = ghm.expand_words(['w0', 'w4 w5', 'w8', 'w12', 'w19'], image(out_hw[1], out_hw[0]), to_cpu=False)
        assert tuple(pre.shape[-2:]) == out_hw
        ref = instances64_stack(pre.cpu().numpy(), 0.4, k)
        for f, a in zip(FIELDS, full):
            np.testing.assert_array_equal(a[t].cpu().numpy(), ref[f].astype(a.cpu().numpy().dtype), err_msg=f)


def test_native_refusals():
    maps = rand_maps((16, 16), 1)[None]
    with pytest.raises(_native.NativeError) as e:
        native_call(maps, (16, 16), [[1]], (32, 32), 0.4, 16, 0,          # scratch for less than one plane
                    scratch_bytes=_native.word_instances_plane_bytes(32, 32) - 8)
    assert e.value.code == _native.E_INVALID
    for k, code in ((0, _native.E_INVALID), (65, _native.E_UNSUPPORTED)):
        with pytest.raises(_native.NativeError) as e:
            native_call(maps, (16, 16), [[1]], (32, 32), 0.4, k, 1)
        assert e.value.code == code
    with pytest.raises(_native.NativeError) as e:
        native_call(maps, (16, 16), [[1]] * 97, (32, 32), 0.4, 16, 1)
    assert e.value.code == _native.E_UNSUPPORTED
    with pytest.raises(_native.NativeError) as e:
        native_call(maps, (16, 16), [[1]], (4097, 4097), 0.4, 16, 0, scratch_bytes=256)
    assert e.value.code == _native.E_UNSUPPORTED
