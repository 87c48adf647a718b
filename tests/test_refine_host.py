"""Edge-aware word maps on the host, no GPU: the float64 reference of tests/refine64.py against a brute-force window
loop and the filter's closed-form properties; the refusals of GlobalHeatMap.refine_words and the stacks and their
order, all before the native library; the arguments and scratch sizes they hand to daam_refine_words; the empty
shapes."""
import contextlib
import math

import numpy as np
import pytest
import torch

from daam_b200 import _native, heatmap
from daam_b200.heatmap import GlobalHeatMap, ImageHeatMaps, LayerHeatMaps, TimeHeatMaps
from daam_b200.testing.synthetic import WhitespaceTokenizer
from tests.refine64 import box_sum, refine64, refine_bound, refine_brute, window_count

TOK = WhitespaceTokenizer()
PROMPT = 'a dog chasing a red ball on the beach'


def rand_case(h, w, seed, n=None):
    g = np.random.default_rng(seed)
    return g.random((h, w) if n is None else (n, h, w)), g.integers(0, 256, (h, w, 3), dtype=np.uint8)


# ---- the float64 reference ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('h,w,r', [(7, 9, 1), (6, 5, 2), (5, 8, 20), (9, 4, 3), (1, 6, 2), (6, 1, 1), (1, 1, 5),
                                   (11, 13, 4)])
@pytest.mark.parametrize('eps', [1e-4, 1e-2, 1.0])
def test_reference_against_brute_force(h, w, r, eps):
    # windows clipped on every side, radii larger than the image, 1-pixel rows and columns
    m, img = rand_case(h, w, h * 31 + w * 7 + r)
    np.testing.assert_allclose(refine64(m, img, r, eps), refine_brute(m, img, r, eps), rtol=0, atol=1e-11)


def test_reference_over_a_word_axis():
    m, img = rand_case(12, 10, 3, n=4)
    q = refine64(m, img, 3, 1e-3)
    assert q.shape == (4, 12, 10)
    for k in range(4):
        np.testing.assert_array_equal(refine64(m[k], img, 3, 1e-3), q[k])


def test_window_counts_and_sums():
    n = window_count(5, 7, 2)
    assert n[0, 0] == 9 and n[2, 3] == 25 and n[4, 6] == 9 and n[0, 3] == 15
    f = np.arange(35, dtype=np.int64).reshape(5, 7)
    s = box_sum(f, 2)
    assert s[2, 3] == f[0:5, 1:6].sum() and s[0, 0] == f[:3, :3].sum() and s[4, 6] == f[2:, 4:].sum()
    assert np.array_equal(box_sum(np.ones((5, 7), np.int64), 9), np.full((5, 7), 35))


def test_constant_guide_gives_the_mean_of_the_mean():
    m, _ = rand_case(9, 11, 1)
    img = np.full((9, 11, 3), (40, 200, 7), dtype=np.uint8)
    r = 2
    n = window_count(9, 11, r)
    want = box_sum(box_sum(m, r) / n, r) / n
    np.testing.assert_allclose(refine64(m, img, r, 1e-3), want, rtol=0, atol=1e-13)


def test_constant_map_is_kept():
    _, img = rand_case(10, 8, 2)
    for eps in (1e-4, 1e-2, 1.0):
        np.testing.assert_allclose(refine64(np.full((10, 8), 0.37), img, 3, eps), 0.37, rtol=0, atol=1e-10)


def test_large_eps_tends_to_the_mean_of_the_mean():
    m, img = rand_case(10, 12, 4)
    n = window_count(10, 12, 2)
    want = box_sum(box_sum(m, 2) / n, 2) / n
    errs = [np.abs(refine64(m, img, 2, eps) - want).max() for eps in (1e2, 1e4, 1e6)]
    assert errs[0] > errs[1] > errs[2] and errs[2] < 1e-6
    assert errs[1] / errs[2] == pytest.approx(100, rel=0.05)          # a = O(1 / eps)


def test_an_edge_is_kept():
    # a guide with a vertical colour edge and a map smeared across it: the filter sharpens the step onto the edge
    img = np.zeros((16, 32, 3), dtype=np.uint8)
    img[:, 16:] = (250, 240, 230)
    m = np.clip((np.arange(32) - 10) / 12, 0, 1)[None].repeat(16, 0)
    q = refine64(m, img, 4, 1e-4)
    assert bool((q[:, 13] < m[:, 13]).all()) and bool((q[:, 18] > m[:, 18]).all())
    assert (q[:, 16] - q[:, 15]).min() > 3 * (m[0, 16] - m[0, 15])


def test_bound_grows_with_radius_and_falls_with_eps():
    m, img = rand_case(40, 30, 5, n=2)
    b = {}
    for r, eps in ((1, 1e-2), (8, 1e-2), (8, 1.0), (8, 1e-4)):
        _, parts = refine64(m, img, r, eps, parts=True)
        b[r, eps] = refine_bound(m, parts, r, eps)
        assert b[r, eps].shape == (2, 1, 1) and bool((b[r, eps] > 0).all())
    assert bool((b[1, 1e-2] < b[8, 1e-2]).all()) and bool((b[8, 1.0] < b[8, 1e-2]).all())
    assert bool((b[8, 1e-2] < b[8, 1e-4]).all())


# ---- what reaches the native call -------------------------------------------------------------------------------------
class FakeLib:
    """Stands in for libdaam_b200.so: records the arguments of daam_refine_words."""

    def __init__(self):
        self.calls = []

    def daam_refine_words(self, *args):
        rows, begin, n_words = args[5], args[6], args[7]
        self.calls.append(dict(n_maps=args[1], n_rows=args[2], grid=(args[3], args[4]),
                               rows=[list(rows[begin[w]:begin[w + 1]]) for w in range(n_words)],
                               out=(args[8], args[9]), absolute=args[10], use_threshold=args[11], threshold=args[12],
                               radius=args[13], eps=args[14], stride=args[17], scratch_bytes=args[20],
                               n_args=len(args)))
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
    whms, refined = ghm.refine_words(['dog', 'red ball'], image(40, 40))
    call, = fake.calls
    assert call['n_args'] == 22 and call['n_maps'] == 1 and call['out'] == (40, 40)
    assert call['rows'] == [[2], [5, 6]] and call['absolute'] == 0 and call['use_threshold'] == 0
    assert call['radius'] == 8 and call['eps'] == 1e-3 and call['stride'] == 0
    assert call['scratch_bytes'] == _native.refine_scratch_bytes(1, 2, 40, 40)    # one image, both planes
    assert tuple(refined.shape) == (2, 40, 40) and refined.dtype == torch.float32
    assert [w.word for w in whms] == ['dog', 'red ball']
    ghm.refine_words(['beach'], image(24, 24).numpy(), radius=64, eps=0.5, absolute=True, threshold=0.4)
    call = fake.calls[-1]
    assert (call['radius'], call['eps'], call['absolute'], call['use_threshold'], call['threshold']) == (64, 0.5, 1, 1,
                                                                                                         0.4)
    ghm.refine_words(['beach'], image(24, 24), threshold=0)                       # 0: no threshold, as expand_words
    assert fake.calls[-1]['use_threshold'] == 0
    rect = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 12, 20))
    _, refined = rect.refine_words(['dog'], image(30, 50), radius=1)
    assert fake.calls[-1]['out'] == (30, 50) and tuple(refined.shape) == (1, 30, 50)


def test_stacks_are_one_call_over_every_map(fake, monkeypatch):
    tm = TimeHeatMaps(TOK, PROMPT, torch.zeros(5, 11, 16, 16))
    word_maps, refined = tm.refine_words(['dog', 'beach'], image(32, 32))
    call, = fake.calls
    assert call['n_maps'] == 5 and call['rows'] == [[2], [9]] and call['stride'] == 0
    assert call['scratch_bytes'] == _native.refine_scratch_bytes(1, 10, 32, 32)
    assert tuple(word_maps.shape) == (5, 2, 16, 16) and tuple(refined.shape) == (5, 2, 32, 32)
    # one image per map: its stride, and one set of statistics per map
    im = ImageHeatMaps(TOK, PROMPT, torch.zeros(3, 11, 16, 16))
    im.refine_words(['dog', 'beach'], image(32, 32, 3))
    assert fake.calls[-1]['stride'] == 32 * 32 * 3
    assert fake.calls[-1]['scratch_bytes'] == _native.refine_scratch_bytes(3, 6, 32, 32)
    lm = LayerHeatMaps(TOK, PROMPT, torch.zeros(2, 11, 16, 12), [3, 7], ['a', 'b'], [1, 2])
    _, refined = lm.refine_words(['ball'], image(32, 24))
    assert fake.calls[-1]['n_maps'] == 2 and fake.calls[-1]['grid'] == (16, 12) and tuple(refined.shape) == (2, 1, 32,
                                                                                                            24)
    # the scratch budget caps a long stack (rounds), and one image and one plane are the least a call gets
    monkeypatch.setattr(heatmap, 'REFINE_SCRATCH_BYTES', _native.refine_scratch_bytes(1, 3, 32, 32))
    tm.refine_words(['dog', 'beach'], image(32, 32))
    assert fake.calls[-1]['scratch_bytes'] == _native.refine_scratch_bytes(1, 3, 32, 32)
    monkeypatch.setattr(heatmap, 'REFINE_SCRATCH_BYTES', 1)
    tm.refine_words(['dog', 'beach'], image(32, 32))
    assert fake.calls[-1]['scratch_bytes'] == _native.refine_scratch_bytes(1, 1, 32, 32)


def test_scratch_size_matches_the_header():
    assert _native.refine_guide_bytes(512, 512) == 36 * 512 * 512
    assert _native.refine_plane_bytes(1216, 832) == 32 * 1216 * 832 + 256
    assert _native.refine_scratch_bytes(2, 3, 600, 800) == 2 * 36 * 480000 + 3 * (32 * 480000 + 256)
    assert 'daam_refine_words' in _native.EXPORTS and _native.REFINE_MAX_RADIUS == 64
    assert heatmap.REFINE_SCRATCH_BYTES == 256 << 20


# ---- refusals, all before the native library ----------------------------------------------------------------------------
@pytest.fixture
def no_native(monkeypatch):
    def load():
        raise AssertionError('the native library was reached')
    monkeypatch.setattr(_native, 'load', load)
    monkeypatch.setattr(heatmap, '_require_cuda', lambda t, what: None)


@pytest.mark.parametrize('radius', [0, 65, -1, 8.0, True, '8', None])
def test_radius_refusals(no_native, radius):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16))
    with pytest.raises(ValueError, match=r'GlobalHeatMap.refine_words: radius must be an integer in \[1, 64\]'):
        ghm.refine_words(['dog'], image(32, 32), radius=radius)


@pytest.mark.parametrize('eps', [0.0, -1e-3, float('inf'), float('nan'), 1e-50, 1e39])
def test_eps_refusals(no_native, eps):
    # 1e-50 rounds to 0 in fp32 and 1e39 to inf
    with pytest.raises(ValueError, match='TimeHeatMaps.refine_words: eps must be finite and > 0'):
        TimeHeatMaps(TOK, PROMPT, torch.zeros(2, 11, 16, 16)).refine_words(['dog'], image(32, 32), eps=eps)


def test_refusal_order(no_native):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16))
    # the words first, then the row range, then the image, then radius and eps
    with pytest.raises(ValueError, match='Search word zebra not found in prompt!'):
        ghm.refine_words(['zebra'], 'not an image', radius=0)
    with pytest.raises(IndexError, match='out of bounds'):
        GlobalHeatMap(TOK, PROMPT, torch.zeros(4, 16, 16)).refine_words(['beach'], 'not an image', radius=0)
    with pytest.raises(TypeError, match='PIL image or a uint8'):
        ghm.refine_words(['dog'], 'not an image', radius=0)
    with pytest.raises(TypeError, match='must be uint8'):
        ghm.refine_words(['dog'], torch.zeros(32, 32, 3), eps=0)
    with pytest.raises(ValueError, match=r'does not match .*\(32, 32, 3\)'):
        ghm.refine_words(['dog'], torch.zeros(32, 32, 4, dtype=torch.uint8), radius=0)
    with pytest.raises(ValueError, match='transposes a non-square image'):
        ghm.refine_words(['dog'], image(30, 40), radius=0)
    with pytest.raises(ValueError, match=r'is not \[H, W, 3\]'):
        ghm.refine_words(['dog'], image(32, 32, 2))                   # one map takes one image
    tm = TimeHeatMaps(TOK, PROMPT, torch.zeros(3, 11, 16, 16))
    with pytest.raises(ValueError, match=r'is not \[3, H, W, 3\] or \[H, W, 3\]'):
        tm.refine_words(['dog'], image(32, 32, 2), eps=-1)
    with pytest.raises(ValueError, match='radius'):
        tm.refine_words(['dog'], image(32, 32, 3), radius=0, eps=-1)  # radius before eps
    with pytest.raises(ValueError, match='radius'):
        tm.refine_words([], image(32, 32), radius=0)                  # an empty list is checked too


def test_cpu_maps_are_refused(monkeypatch):
    monkeypatch.setattr(_native, 'load', lambda: (_ for _ in ()).throw(AssertionError('reached the library')))
    with pytest.raises(RuntimeError, match='GlobalHeatMap.refine_words: .*CUDA tensors only'):
        GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16)).refine_words(['dog'], image(32, 32))


# ---- empty inputs --------------------------------------------------------------------------------------------------------
def test_empty_inputs_launch_nothing(fake):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16))
    whms, refined = ghm.refine_words([], image(32, 32))
    assert whms == [] and tuple(refined.shape) == (0, 32, 32) and refined.dtype == torch.float32
    word_maps, refined = TimeHeatMaps(TOK, PROMPT, torch.zeros(4, 11, 16, 16)).refine_words([], image(32, 32, 4))
    assert tuple(refined.shape) == (4, 0, 32, 32) and tuple(word_maps.shape) == (4, 0, 16, 16)
    word_maps, refined = TimeHeatMaps(TOK, PROMPT, torch.zeros(0, 11, 16, 16)).refine_words(['dog'], image(32, 32))
    assert tuple(refined.shape) == (0, 1, 32, 32)
    assert fake.calls == []
    assert not math.isnan(float(heatmap.REFINE_SCRATCH_BYTES))
