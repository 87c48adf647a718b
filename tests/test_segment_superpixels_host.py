"""Superpixel word segmentation on the host, no GPU: the numpy reference of tests/slic64.py against a brute-force loop
and its grid and cell formulas; the refusals of segment_superpixels and evaluate.superpixels and their order, all
before the native library; the arguments and scratch sizes they hand to the native entries; the empty shapes."""
import contextlib
import os

import numpy as np
import pytest
import torch

from daam_b200 import _native, evaluate, heatmap
from daam_b200.heatmap import GlobalHeatMap, ImageHeatMaps, TimeHeatMaps
from daam_b200.testing.synthetic import WhitespaceTokenizer
from tests.slic64 import cell_begin, cell_of, grid, pooled64, pooled_labels64, slic, slic_brute

TOK = WhitespaceTokenizer()
PROMPT = 'a dog chasing a red ball on the beach'


def noise(h, w, seed, levels=256):
    return np.random.default_rng(seed).integers(0, levels, (h, w, 3), dtype=np.uint8)


# ---- the reference ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('h,w,k,c,t', [(7, 5, 4, 20.0, 3), (9, 11, 6, 5.0, 4), (1, 9, 3, 20.0, 2), (8, 1, 2, 1.0, 3),
                                       (6, 6, 36, 20.0, 2), (10, 7, 1, 20.0, 2), (12, 9, 5, 0.5, 5)])
@pytest.mark.parametrize('levels', [2, 256])
def test_reference_against_brute_force(h, w, k, c, t, levels):
    img = noise(h, w, h * 13 + w + k, levels)
    np.testing.assert_array_equal(slic(img, k, c, t), slic_brute(img, k, c, t))


@pytest.mark.parametrize('h,w', [(1, 1), (1, 37), (29, 1), (7, 5), (48, 40), (512, 512), (1024, 1024), (1216, 832),
                                 (333, 517)])
@pytest.mark.parametrize('k', [1, 4, 100, 1024, 4096, 65536, 10 ** 9])
def test_grid_and_cells(h, w, k):
    ny, nx = grid(h, w, k)
    assert (ny, nx) == _native.superpixel_grid(h, w, k)
    assert 1 <= ny <= h and 1 <= nx <= w
    for n_cells, n in ((ny, h), (nx, w)):
        b = cell_begin(np.arange(n_cells + 1), n_cells, n)
        assert b[0] == 0 and b[-1] == n and bool((np.diff(b) >= 1).all())     # every cell has a pixel row
        y = np.arange(n)
        c = cell_of(y, n_cells, n)
        assert bool((b[c] <= y).all()) and bool((y < b[c + 1]).all())
        # yb(c) <= y  <=>  c n < (y + 1) n_cells, for every c
        cs = np.arange(n_cells + 1)[:, None]
        assert np.array_equal(cell_begin(cs, n_cells, n) <= y[None], cs * n < (y[None] + 1) * n_cells)
    # a 16 x 64 tile's cells, widened by one, fit the box the scratch is sized for
    bh, bw = min(ny, 15 * ny // h + 4), min(nx, 63 * nx // w + 4)
    for y0 in range(0, h, 16):
        assert min(cell_of(min(y0 + 15, h - 1), ny, h) + 1, ny - 1) - max(cell_of(y0, ny, h) - 1, 0) + 1 <= bh
    for x0 in range(0, w, 64):
        assert min(cell_of(min(x0 + 63, w - 1), nx, w) + 1, nx - 1) - max(cell_of(x0, nx, w) - 1, 0) + 1 <= bw
    assert bh * bw == _native.superpixel_box(ny, nx, h, w)


@pytest.mark.parametrize('h,w', [(1, 1), (5, 7), (16, 64), (13, 70)])
def test_one_pixel_cells_are_the_identity(h, w):
    assert grid(h, w, h * w) == (h, w)
    for levels in (1, 256):
        lab = slic(noise(h, w, 3, levels), h * w, 20.0, 3)
        np.testing.assert_array_equal(lab, np.arange(h * w, dtype=np.int32).reshape(h, w))


@pytest.mark.parametrize('h,w,k', [(40, 48, 30), (17, 23, 9), (64, 64, 16)])
def test_a_constant_image_is_geometry_alone(h, w, k):
    parts = [slic(np.full((h, w, 3), col, dtype=np.uint8), k, 20.0, 4) for col in ((0, 0, 0), (200, 17, 90))]
    np.testing.assert_array_equal(parts[0], parts[1])
    ny, nx = grid(h, w, k)
    # every pixel lies next to its own cell: it keeps the nearest seed of the cells around it
    cy = cell_of(np.arange(h), ny, h)[:, None]
    cx = cell_of(np.arange(w), nx, w)[None, :]
    assert bool((np.abs(parts[0] // nx - cy) <= 1).all()) and bool((np.abs(parts[0] % nx - cx) <= 1).all())


def test_colour_splits_flat_blocks():
    img = np.zeros((32, 32, 3), dtype=np.uint8)
    img[:, 16:] = (255, 255, 255)
    lab = slic(img, 4, 1.0, 10)
    assert len(set(lab[:, :16].ravel()) & set(lab[:, 16:].ravel())) == 0


def test_pooled_reference():
    g = np.random.default_rng(1)
    lab = g.integers(0, 5, (6, 7)).astype(np.int32)
    m = g.random((3, 6, 7)).astype(np.float32)
    mean, count = pooled64(m, lab)
    for s in range(5):
        assert count[s] == (lab == s).sum()
        np.testing.assert_allclose(mean[:, s], m[:, lab == s].astype(np.float64).mean(1), rtol=1e-15)
    labels, scores, _ = pooled_labels64(m, lab, threshold=0.5)
    assert labels.shape == (6, 7) and scores.dtype == np.float32
    assert bool(((labels == 0) == (scores <= np.float32(0.5))).all())


# ---- what reaches the native calls ------------------------------------------------------------------------------------
class FakeLib:
    """Stands in for libdaam_b200.so: records the arguments of the superpixel entries."""

    def __init__(self):
        self.calls = []

    def daam_segment_superpixels(self, *args):
        rows, begin, n_words = args[5], args[6], args[7]
        self.calls.append(dict(entry='segment', n_maps=args[1], n_rows=args[2], grid=(args[3], args[4]),
                               rows=[list(rows[begin[w]:begin[w + 1]]) for w in range(n_words)],
                               out=(args[8], args[9]), absolute=args[10], use_threshold=args[11],
                               threshold=args[12], n_segments=args[13], compactness=args[14], iterations=args[15],
                               stride=args[18], scratch_bytes=args[23], n_args=len(args)))
        return 0

    def daam_image_superpixels(self, *args):
        self.calls.append(dict(entry='image', n_images=args[1], out=(args[2], args[3]), n_segments=args[4],
                               compactness=args[5], iterations=args[6], scratch_bytes=args[9], n_args=len(args)))
        return 0


@pytest.fixture
def fake(monkeypatch):
    lib = FakeLib()
    monkeypatch.setattr(_native, 'load', lambda: lib)
    monkeypatch.setattr(heatmap, '_require_cuda', lambda t, what: None)
    monkeypatch.setattr(heatmap, '_stream_ptr', lambda dev: 0)
    monkeypatch.setattr(torch.cuda, 'device', lambda dev: contextlib.nullcontext())
    return lib


def image(h, w, n=None):
    return torch.zeros(((n,) if n else ()) + (h, w, 3), dtype=torch.uint8)


def test_arguments_reach_the_native_call(fake):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16))
    whms, labels, scores, sp = ghm.segment_superpixels(['dog', 'red ball'], image(40, 40))
    call, = fake.calls
    assert call['entry'] == 'segment' and call['n_args'] == 25 and call['n_maps'] == 1 and call['out'] == (40, 40)
    assert call['rows'] == [[2], [5, 6]] and call['absolute'] == 0 and call['use_threshold'] == 0
    assert (call['n_segments'], call['compactness'], call['iterations'], call['stride']) == (1024, 20.0, 10, 0)
    ny, nx = grid(40, 40, 1024)
    assert call['scratch_bytes'] == _native.superpixel_scratch_bytes(1, 1, 2, ny, nx, 40, 40)
    assert tuple(labels.shape) == (40, 40) and labels.dtype == torch.uint8 and scores.dtype == torch.float32
    assert tuple(sp.shape) == (40, 40) and sp.dtype == torch.int32
    assert [w.word for w in whms] == ['dog', 'red ball']
    ghm.segment_superpixels(['beach'], image(24, 24).numpy(), n_segments=7, compactness=3.5, iterations=64,
                            threshold=0.4, absolute=True)
    call = fake.calls[-1]
    assert (call['use_threshold'], call['threshold'], call['n_segments'], call['compactness'], call['iterations'],
            call['absolute']) == (1, 0.4, 7, 3.5, 64, 1)
    ghm.segment_superpixels(['beach'], image(24, 24), threshold=0)                # 0: no threshold, as segment
    assert fake.calls[-1]['use_threshold'] == 0
    rect = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 12, 20))
    _, labels, _, sp = rect.segment_superpixels(['dog'], image(30, 50), n_segments=30 * 50)
    assert fake.calls[-1]['out'] == (30, 50) and tuple(labels.shape) == (30, 50) and tuple(sp.shape) == (30, 50)


def test_stacks_are_one_call_over_every_map(fake, monkeypatch):
    tm = TimeHeatMaps(TOK, PROMPT, torch.zeros(5, 11, 16, 16))
    word_maps, labels, scores, sp = tm.segment_superpixels(['dog', 'beach'], image(32, 32), n_segments=64)
    call, = fake.calls
    assert call['n_maps'] == 5 and call['rows'] == [[2], [9]] and call['stride'] == 0
    assert call['scratch_bytes'] == _native.superpixel_scratch_bytes(1, 5, 2, 8, 8, 32, 32)
    assert tuple(word_maps.shape) == (5, 2, 16, 16) and tuple(labels.shape) == (5, 32, 32)
    assert tuple(scores.shape) == (5, 32, 32) and tuple(sp.shape) == (32, 32)
    # one image per map: its stride, one partition each
    im = ImageHeatMaps(TOK, PROMPT, torch.zeros(3, 11, 16, 16))
    _, _, _, sp = im.segment_superpixels(['dog', 'beach'], image(32, 32, 3), n_segments=64)
    assert fake.calls[-1]['stride'] == 32 * 32 * 3 and fake.calls[-1]['n_maps'] == 3 and tuple(sp.shape) == (3, 32, 32)
    assert fake.calls[-1]['scratch_bytes'] == _native.superpixel_scratch_bytes(3, 3, 2, 8, 8, 32, 32)
    # the scratch budget caps a long stack (rounds of whole maps), and one image and one map is the least a call gets
    monkeypatch.setattr(heatmap, 'SUPERPIXEL_SCRATCH_BYTES', _native.superpixel_scratch_bytes(1, 2, 2, 8, 8, 32, 32))
    tm.segment_superpixels(['dog', 'beach'], image(32, 32), n_segments=64)
    assert fake.calls[-1]['scratch_bytes'] == _native.superpixel_scratch_bytes(1, 2, 2, 8, 8, 32, 32)
    monkeypatch.setattr(heatmap, 'SUPERPIXEL_SCRATCH_BYTES', 1)
    tm.segment_superpixels(['dog', 'beach'], image(32, 32), n_segments=64)
    assert fake.calls[-1]['scratch_bytes'] == _native.superpixel_scratch_bytes(1, 1, 2, 8, 8, 32, 32)


def test_evaluate_reaches_the_image_call(fake):
    sp = evaluate.superpixels(image(32, 48), n_segments=6, compactness=2.0, iterations=3)
    call, = fake.calls
    ny, nx = grid(32, 48, 6)
    assert call == dict(entry='image', n_images=1, out=(32, 48), n_segments=6, compactness=2.0, iterations=3,
                        scratch_bytes=_native.superpixel_image_bytes(ny, nx), n_args=11)
    assert tuple(sp.shape) == (32, 48) and sp.dtype == torch.int32
    sp = evaluate.superpixels(image(32, 48, 4))
    assert fake.calls[-1]['n_images'] == 4 and tuple(sp.shape) == (4, 32, 48)


def test_scratch_size_matches_the_header():
    assert _native.superpixel_image_bytes(32, 32) == 96 * 1024
    assert _native.superpixel_box(32, 32, 512, 512) == 4 * 7
    assert _native.superpixel_map_bytes(8, 32, 32, 512, 512) == 256 * 8 + 8 * 1024 + 8 * 8 * 32 * 8 * 28
    assert _native.superpixel_scratch_bytes(2, 3, 8, 32, 32, 512, 512) == (
        2 * 96 * 1024 + 3 * _native.superpixel_map_bytes(8, 32, 32, 512, 512))
    assert 'daam_segment_superpixels' in _native.EXPORTS and 'daam_image_superpixels' in _native.EXPORTS
    assert _native.SUPERPIXEL_MAX_CELLS == 65536 and _native.SUPERPIXEL_MAX_ITERATIONS == 64
    assert heatmap.SUPERPIXEL_SCRATCH_BYTES == 256 << 20
    header = open(os.path.join(os.path.dirname(_native.__file__), '..', 'include', 'daam_b200.h')).read()
    assert '#define DAAM_SUPERPIXEL_MAX_CELLS 65536' in header
    assert '#define DAAM_SUPERPIXEL_IMAGE_BYTES(ny, nx) (96 * (int64_t)(ny) * (nx))' in header


# ---- refusals, all before the native library ----------------------------------------------------------------------------
@pytest.fixture
def no_native(monkeypatch):
    def load():
        raise AssertionError('the native library was reached')
    monkeypatch.setattr(_native, 'load', load)
    monkeypatch.setattr(heatmap, '_require_cuda', lambda t, what: None)


@pytest.mark.parametrize('kw,text', [
    (dict(n_segments=0), 'n_segments must be an integer >= 1'),
    (dict(n_segments=4.0), 'n_segments must be an integer >= 1'),
    (dict(n_segments=True), 'n_segments must be an integer >= 1'),
    (dict(compactness=0.0), 'compactness must be finite and > 0'),
    (dict(compactness=-1.0), 'compactness must be finite and > 0'),
    (dict(compactness=1e39), 'compactness must be finite and > 0'),
    (dict(compactness=1e-50), 'compactness must be finite and > 0'),
    (dict(compactness=float('nan')), 'compactness must be finite and > 0'),
    (dict(compactness='x'), 'compactness must be a number'),
    (dict(iterations=0), r'iterations must be an integer in \[1, 64\]'),
    (dict(iterations=65), r'iterations must be an integer in \[1, 64\]'),
    (dict(iterations=None), r'iterations must be an integer in \[1, 64\]'),
    (dict(n_segments=600 * 600), '360000 segments of a 300 x 300 image make a 300 x 300 grid, more than 65536 cells'),
])
def test_argument_refusals(no_native, kw, text):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 300, 300))
    with pytest.raises(ValueError, match='GlobalHeatMap.segment_superpixels: ' + text):
        ghm.segment_superpixels(['dog'], image(300, 300), **kw)
    with pytest.raises(ValueError, match='superpixels: ' + text):
        evaluate.superpixels(image(300, 300), **kw)


def test_refusal_order(no_native):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16))
    # the words first, then the row range, then the image, then the pixels, the arguments in the C entry's order, cells
    with pytest.raises(ValueError, match='Search word zebra not found in prompt!'):
        ghm.segment_superpixels(['zebra'], 'not an image', n_segments=0)
    with pytest.raises(IndexError, match='out of bounds'):
        GlobalHeatMap(TOK, PROMPT, torch.zeros(4, 16, 16)).segment_superpixels(['beach'], 'not an image')
    with pytest.raises(TypeError, match='PIL image or a uint8'):
        ghm.segment_superpixels(['dog'], 'not an image', n_segments=0)
    with pytest.raises(TypeError, match='must be uint8'):
        ghm.segment_superpixels(['dog'], torch.zeros(32, 32, 3), iterations=0)
    with pytest.raises(ValueError, match=r'is not \[H, W, 3\]'):
        ghm.segment_superpixels(['dog'], image(32, 32, 2))
    big = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 64, 64))
    with pytest.raises(ValueError, match=r'more than 2\*\*24 pixels'):
        big.segment_superpixels(['dog'], image(4160, 4160), n_segments=0)
    tm = TimeHeatMaps(TOK, PROMPT, torch.zeros(3, 11, 16, 16))
    for kw, first in [(dict(n_segments=0, compactness=0), 'n_segments'), (dict(compactness=0, iterations=0),
                                                                           'compactness'),
                      (dict(iterations=0, n_segments=10 ** 6), 'iterations')]:
        with pytest.raises(ValueError, match=f'TimeHeatMaps.segment_superpixels: {first} '):
            tm.segment_superpixels(['dog'], image(32, 32, 3), **kw)
    with pytest.raises(ValueError, match='n_segments'):
        tm.segment_superpixels([], image(32, 32), n_segments=0)          # an empty list is checked too
    with pytest.raises(TypeError, match='must be a torch.Tensor'):
        evaluate.superpixels(np.zeros((8, 8, 3), dtype=np.uint8))
    with pytest.raises(TypeError, match='must be uint8'):
        evaluate.superpixels(torch.zeros(8, 8, 3), n_segments=0)
    with pytest.raises(ValueError, match=r'must be \[H, W, 3\] or \[N, H, W, 3\]'):
        evaluate.superpixels(image(8, 8)[..., :2], n_segments=0)


def test_cpu_maps_are_refused(monkeypatch):
    monkeypatch.setattr(_native, 'load', lambda: (_ for _ in ()).throw(AssertionError('reached the library')))
    with pytest.raises(RuntimeError, match='GlobalHeatMap.segment_superpixels: .*CUDA tensors only'):
        GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16)).segment_superpixels(['dog'], image(32, 32))
    with pytest.raises(RuntimeError, match='superpixels: .*CUDA tensors only'):
        evaluate.superpixels(image(32, 32))


# ---- empty inputs --------------------------------------------------------------------------------------------------------
def test_empty_inputs(fake):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16))
    # no word: the partition is still made, every pixel is background with score -inf
    whms, labels, scores, sp = ghm.segment_superpixels([], image(32, 32), n_segments=16)
    assert whms == [] and tuple(labels.shape) == (32, 32) and not labels.any()
    assert bool((scores == float('-inf')).all()) and tuple(sp.shape) == (32, 32)
    call, = fake.calls
    assert call['entry'] == 'image' and call['n_images'] == 1 and call['n_segments'] == 16
    word_maps, labels, _, sp = TimeHeatMaps(TOK, PROMPT, torch.zeros(4, 11, 16, 16)).segment_superpixels(
        [], image(32, 32, 4))
    assert tuple(labels.shape) == (4, 32, 32) and tuple(word_maps.shape) == (4, 0, 16, 16)
    assert tuple(sp.shape) == (4, 32, 32) and fake.calls[-1]['n_images'] == 4
    # no map: nothing to label; one shared image still has its partition
    n = len(fake.calls)
    _, labels, _, sp = TimeHeatMaps(TOK, PROMPT, torch.zeros(0, 11, 16, 16)).segment_superpixels(['dog'], image(32, 32))
    assert tuple(labels.shape) == (0, 32, 32) and tuple(sp.shape) == (32, 32) and fake.calls[-1]['entry'] == 'image'
    _, labels, _, sp = TimeHeatMaps(TOK, PROMPT, torch.zeros(0, 11, 16, 16)).segment_superpixels(
        ['dog'], torch.zeros(0, 32, 32, 3, dtype=torch.uint8))
    assert tuple(sp.shape) == (0, 32, 32) and len(fake.calls) == n + 1
    assert tuple(evaluate.superpixels(image(0, 32)).shape) == (0, 32)
    assert tuple(evaluate.superpixels(torch.zeros(0, 32, 32, 3, dtype=torch.uint8)).shape) == (0, 32, 32)
    assert len(fake.calls) == n + 1
