"""Word distance maps (GlobalHeatMap.word_distance / GlobalHeatMapStack.word_distance, daam_word_distance;
evaluate.distance_transform, daam_mask_distance) on the GPU, against the integer reference of tests/distance64.py.

* signed_d2 equals the reference bit for bit over the very masks expand_words(..., threshold, to_cpu=False) returns:
  SD-2.1 512^2 and 768^2, SDXL 1024^2 and 1216x832, off-grid 600x800; 1, 8 and 96 words; empty and full word masks.
* The mask entry at 1x1, 1xW, Hx1, widths off a multiple of 32 and the widest and tallest sides (1 x 32767,
  32767 x 1, 512 x 32767, 32767 x 512); empty, full, single-pixel, corner-pixel, border-touching, thin-line,
  checkerboard and random-blob masks; a corner pixel at 1024^2 (the largest distances of an SDXL image).
* distance_transform of expand_words' masks equals word_distance; stacks equal the per-map calls; several rounds equal
  one; repeated calls give the same bits.
* The C ABI's limit and invalid statuses.
"""
import ctypes
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from daam_b200 import _native, heatmap
from daam_b200.evaluate import distance_transform
from daam_b200.heatmap import GlobalHeatMap, LayerHeatMaps, TimeHeatMaps
from daam_b200.testing.synthetic import WhitespaceTokenizer
from tests.distance64 import NONE, kinds, signed_d2

pytestmark = pytest.mark.gpu
DEV = 'cuda'
TOK = WhitespaceTokenizer()
PROMPT100 = ' '.join(f'w{i}' for i in range(100))


def image(h, w):
    return SimpleNamespace(size=(w, h), height=h, width=w)


def word_list(n):
    words = [f'w{3 * i % 100}' for i in range(n)]
    if n >= 3:
        words[1] = 'w40 w41'
        words[-1] = words[0]
    return words


def rand_maps(grid, seed, n_rows=102, lead=()):
    return torch.rand(*lead, n_rows, *grid, generator=torch.Generator().manual_seed(seed)).to(DEV)


def check_words(ghm, words, img, threshold, **kw):
    """word_distance against the reference of expand_words' thresholded masks; returns (distance, masks)."""
    _, wd = ghm.word_distance(words, img, threshold, to_cpu=False, **kw)
    _, m = ghm.expand_words(words, img, threshold=threshold, to_cpu=False, **kw)
    assert wd.signed_d2.dtype == torch.int32 and wd.signed_d2.is_cuda and wd.signed_d2.shape == m.shape
    np.testing.assert_array_equal(wd.signed_d2.cpu().numpy(), signed_d2(m.cpu().numpy() > 0))
    return wd, m


PAIRS = [((64, 64), (512, 512)), ((96, 96), (768, 768)), ((128, 128), (1024, 1024)), ((76, 52), (1216, 832)),
         ((75, 100), (600, 800))]
PAIR_IDS = [f'{g[0]}x{g[1]}-{h}x{w}' for g, (h, w) in PAIRS]


@pytest.mark.parametrize('n_words', [1, 8])
@pytest.mark.parametrize('grid,hw', PAIRS, ids=PAIR_IDS)
def test_sizes_against_the_reference(grid, hw, n_words):
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps(grid, 1))
    check_words(ghm, word_list(n_words), image(*hw), 0.55)
    check_words(ghm, word_list(n_words), image(*hw), 0.3, absolute=True)


@pytest.mark.parametrize('grid,hw', [PAIRS[0], PAIRS[3]], ids=[PAIR_IDS[0], PAIR_IDS[3]])
def test_96_words(grid, hw):
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps(grid, 2))
    wd, m = check_words(ghm, word_list(96), image(*hw), 0.5)
    assert bool((m > 0).any()) and bool((m == 0).any())


def test_empty_and_full_word_masks():
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((64, 64), 3))
    wd, _ = check_words(ghm, word_list(3), image(512, 512), 2.0)          # a normalised map never passes 2
    assert bool((wd.signed_d2 == NONE).all())
    wd, _ = check_words(ghm, word_list(3), image(512, 512), -1.0)         # every pixel passes -1
    assert bool((wd.signed_d2 == -NONE).all())
    assert bool(torch.isposinf(wd.cpu().distance()).logical_not().all())


# ---- the mask entry --------------------------------------------------------------------------------------------------
SHAPES = [(1, 1), (1, 45), (45, 1), (37, 45), (5, 33), (31, 97), (200, 333), (129, 1000), (1000, 129)]


@pytest.mark.parametrize('hw', SHAPES, ids=[f'{h}x{w}' for h, w in SHAPES])
def test_mask_kinds_and_shapes(hw):
    masks = torch.from_numpy(kinds(sum(hw), *hw))
    for t in (masks.to(DEV), (masks.to(torch.uint8) * 7).to(DEV)):
        wd = distance_transform(t, to_cpu=False)
        assert wd.signed_d2.is_cuda and wd.signed_d2.shape == masks.shape
        np.testing.assert_array_equal(wd.signed_d2.cpu().numpy(), signed_d2(masks.numpy()))


@pytest.mark.parametrize('hw', [(1, 32767), (32767, 1), (3, 20000), (20000, 3)], ids=lambda v: f'{v[0]}x{v[1]}')
def test_widest_and_tallest(hw):
    masks = torch.from_numpy(kinds(7, *hw)).to(DEV)
    got = distance_transform(masks).signed_d2.numpy()
    np.testing.assert_array_equal(got, signed_d2(masks.cpu().numpy()))


@pytest.mark.parametrize('hw', [(1024, 1024), (512, 32767), (32767, 512)], ids=lambda v: f'{v[0]}x{v[1]}')
def test_corner_pixel_has_the_largest_distances(hw):
    h, w = hw
    masks = torch.zeros((2, h, w), dtype=torch.bool, device=DEV)
    masks[0, 0, 0] = True
    masks[1] = True
    masks[1, h - 1, w - 1] = False
    got = distance_transform(masks, to_cpu=False).signed_d2
    yy = torch.arange(h, device=DEV, dtype=torch.int64)[:, None]
    xx = torch.arange(w, device=DEV, dtype=torch.int64)[None, :]
    want = yy * yy + xx * xx
    want[0, 0] = -1
    assert torch.equal(got[0].long(), want)
    assert int(got[0].max()) == (h - 1) ** 2 + (w - 1) ** 2
    want = -((h - 1 - yy) ** 2 + (w - 1 - xx) ** 2)
    want[h - 1, w - 1] = 1
    assert torch.equal(got[1].long(), want)


def test_random_blobs_at_sdxl_size():
    g = torch.Generator().manual_seed(9)
    coarse = torch.rand(4, 1, 32, 32, generator=g)
    blobs = torch.nn.functional.interpolate(coarse, size=(1024, 1024), mode='bilinear')[:, 0] > 0.6
    masks = blobs.to(DEV)
    np.testing.assert_array_equal(distance_transform(masks).signed_d2.numpy(), signed_d2(blobs.numpy()))


# ---- identities --------------------------------------------------------------------------------------------------------
def test_distance_transform_of_expand_words_equals_word_distance():
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((76, 52), 4))
    img, words = image(1216, 832), word_list(8)
    _, wd = ghm.word_distance(words, img, 0.45, to_cpu=False)
    _, m = ghm.expand_words(words, img, threshold=0.45, to_cpu=False)
    assert torch.equal(distance_transform(m > 0, to_cpu=False).signed_d2, wd.signed_d2)
    # the closing composed from the mask entry: the closed mask holds the mask and stays within the dilation
    closed = distance_transform(wd.mask(6), to_cpu=False).mask(-6)
    assert bool((closed >= (m > 0)).all()) and bool((closed <= wd.mask(6)).all())


def test_stacks_equal_per_map_calls():
    maps = rand_maps((64, 64), 5, lead=(4,))
    img, words = image(512, 512), word_list(5)
    for stack in (TimeHeatMaps(TOK, PROMPT100, maps),
                  LayerHeatMaps(TOK, PROMPT100, maps, [0, 1, 2, 3], ['a', 'b', 'c', 'd'], [1, 1, 2, 2])):
        word_maps, wd = stack.word_distance(words, img, 0.5, to_cpu=False)
        assert tuple(wd.signed_d2.shape) == (4, 5, 512, 512) and tuple(word_maps.shape[:2]) == (4, 5)
        for t in range(4):
            whms, one = stack[t].word_distance(words, img, 0.5, to_cpu=False)
            assert torch.equal(one.signed_d2, wd.map(t).signed_d2)
            for i, w in enumerate(whms):
                assert torch.equal(w.heatmap, word_maps[t, i])


def test_rounds_give_the_same_bits(monkeypatch):
    stack = TimeHeatMaps(TOK, PROMPT100, rand_maps((75, 100), 7, lead=(3,)))
    img, words = image(600, 800), word_list(5)
    before = _native.launch_count()
    _, one = stack.word_distance(words, img, 0.5, to_cpu=False)
    assert _native.launch_count() - before == 4                           # every plane in one round
    plane = _native.distance_plane_bytes(600, 800)
    for cap, rounds in ((1, 15), (2, 9), (4, 6), (10, 2)):
        monkeypatch.setattr(heatmap, 'WORD_DISTANCE_SCRATCH_BYTES', cap * plane)
        before = _native.launch_count()
        _, wd = stack.word_distance(words, img, 0.5, to_cpu=False)
        assert _native.launch_count() - before == 4 * rounds
        assert torch.equal(wd.signed_d2, one.signed_d2)


def test_repeated_calls_give_the_same_bits():
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((128, 128), 8))
    img, words = image(1024, 1024), word_list(8)
    _, a = ghm.word_distance(words, img, 0.5, to_cpu=False)
    _, b = ghm.word_distance(words, img, 0.5, to_cpu=False)
    assert torch.equal(a.signed_d2, b.signed_d2)
    _, c = ghm.word_distance(words, img, 0.5)
    assert not c.signed_d2.is_cuda and torch.equal(c.signed_d2, a.signed_d2.cpu())


# ---- limits through the C ABI ------------------------------------------------------------------------------------------
def _word_call(maps, grid, out_hw, n_words=1, threshold=0.5, scratch_bytes=None, scratch_offset=0, out_ptr=None,
               maps_ptr=None, n_maps=1):
    word_maps = torch.empty((1, max(n_words, 1)) + grid, device=DEV)
    out = torch.empty(4, dtype=torch.int32, device=DEV) if out_hw[0] * out_hw[1] > 1 << 24 else \
        torch.empty((max(n_words, 1),) + out_hw, dtype=torch.int32, device=DEV)
    need = _native.distance_plane_bytes(*out_hw)
    scratch = torch.empty((need if need <= 1 << 30 else 8) + 8, dtype=torch.uint8, device=DEV)
    rows = (ctypes.c_int32 * max(n_words, 1))(*([1] * max(n_words, 1)))
    begin = (ctypes.c_int32 * (max(n_words, 1) + 1))(*range(max(n_words, 1) + 1))
    vp = ctypes.c_void_p
    rc = _native.load().daam_word_distance(
        vp(maps.data_ptr() if maps_ptr is None else maps_ptr), n_maps, maps.shape[0], grid[0], grid[1], rows, begin,
        n_words, out_hw[0], out_hw[1], 0, threshold, vp(word_maps.data_ptr()),
        vp(out.data_ptr() if out_ptr is None else out_ptr), vp(scratch.data_ptr() + scratch_offset),
        need if scratch_bytes is None else scratch_bytes, vp(torch.cuda.current_stream().cuda_stream))
    return rc, (_native.load().daam_last_error().decode() if rc else '')


def test_word_entry_statuses():
    grid, out = (16, 16), (72, 40)
    maps = rand_maps(grid, 5)
    assert _word_call(maps, grid, out) == (0, '')
    torch.cuda.synchronize()
    cases = [
        (dict(out_hw=(32768, 8)), _native.E_UNSUPPORTED, 'side > 32767'),
        (dict(out_hw=(8, 32768)), _native.E_UNSUPPORTED, 'side > 32767'),
        (dict(out_hw=(4097, 4097)), _native.E_UNSUPPORTED, 'more than 2^24 pixels'),
        (dict(n_words=97), _native.E_UNSUPPORTED, '97 words > 96'),
        (dict(threshold=float('nan')), _native.E_INVALID, 'threshold nan is not finite'),
        (dict(threshold=float('inf')), _native.E_INVALID, 'is not finite'),
        (dict(scratch_offset=2), _native.E_INVALID, '4-byte aligned'),
        (dict(scratch_bytes=_native.distance_plane_bytes(72, 40) - 1), _native.E_INVALID, 'scratch bytes'),
        (dict(out_ptr=0), _native.E_INVALID, 'null pointer'),
        (dict(maps_ptr=0), _native.E_INVALID, 'null pointer'),
        (dict(n_maps=0), _native.E_INVALID, 'non-positive size'),
        (dict(out_hw=(0, 40)), _native.E_INVALID, 'non-positive size'),
        (dict(n_words=0), _native.E_INVALID, 'empty word list'),
    ]
    for kw, code, msg in cases:
        rc, err = _word_call(maps, grid, kw.pop('out_hw', out), **kw)
        assert rc == code and msg in err and err.startswith('daam_word_distance: '), (kw, rc, err)


def test_mask_entry_statuses():
    masks = torch.zeros(2, 72, 40, dtype=torch.uint8, device=DEV)
    out = torch.empty(2, 72, 40, dtype=torch.int32, device=DEV)
    vp = ctypes.c_void_p

    def call(m_ptr=masks.data_ptr(), n_planes=2, h=72, w=40, o_ptr=out.data_ptr()):
        rc = _native.load().daam_mask_distance(vp(m_ptr), n_planes, h, w, vp(o_ptr),
                                               vp(torch.cuda.current_stream().cuda_stream))
        return rc, (_native.load().daam_last_error().decode() if rc else '')

    assert call() == (0, '')
    torch.cuda.synchronize()
    assert bool((out == NONE).all())
    assert call(w=32768, h=1) == (_native.E_UNSUPPORTED, 'daam_mask_distance: a 1 x 32768 output has a side > 32767')
    assert call(h=32768, w=1)[0] == _native.E_UNSUPPORTED
    assert call(h=4097, w=4097) == (_native.E_UNSUPPORTED,
                                    'daam_mask_distance: a 4097 x 4097 output is more than 2^24 pixels')
    for kw in (dict(m_ptr=0), dict(o_ptr=0), dict(n_planes=0), dict(h=0), dict(w=-1)):
        assert call(**kw) == (_native.E_INVALID, 'daam_mask_distance: null pointer or non-positive size'), kw
