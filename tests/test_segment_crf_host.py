"""CRF-refined word segmentation on the host, no GPU: the float64 reference of tests/crf64.py against a brute-force
window loop and its closed-form properties; the refusals of GlobalHeatMap.segment_crf and the stacks and their order,
all before the native library; the arguments and scratch sizes they hand to daam_segment_crf; the empty shapes."""
import contextlib
import math

import numpy as np
import pytest
import torch

from daam_b200 import _native, heatmap
from daam_b200.heatmap import GlobalHeatMap, ImageHeatMaps, LayerHeatMaps, TimeHeatMaps
from daam_b200.testing.synthetic import WhitespaceTokenizer
from tests.crf64 import crf_bound, crf_brute, crf_step64, crf_tables, logits64, softmax64

TOK = WhitespaceTokenizer()
PROMPT = 'a dog chasing a red ball on the beach'
DEFAULTS = dict(appearance=10.0, sigma_xy=8.0, smoothness=1.0, sigma_smooth=3.0, sigma_rgb=13.0)


def rand_case(h, w, n_labels, seed, levels=256):
    g = np.random.default_rng(seed)
    z = 16.0 * g.random((n_labels, h, w))
    q = softmax64(g.normal(size=(n_labels, h, w)))
    return z, q, g.integers(0, levels, (h, w, 3), dtype=np.uint8)


# ---- the float64 reference ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('h,w,r', [(7, 9, 1), (6, 5, 2), (5, 8, 20), (9, 4, 3), (1, 6, 2), (6, 1, 1), (1, 1, 5),
                                   (11, 13, 4)])
@pytest.mark.parametrize('n_labels', [1, 3, 9])
def test_reference_against_brute_force(h, w, r, n_labels):
    # windows clipped on every side, radii larger than the image, 1-pixel rows and columns; few colour levels, so
    # that some pairs are alike and weigh e^0
    z, q, img = rand_case(h, w, n_labels, h * 31 + w * 7 + r, levels=4 if r % 2 else 256)
    tab = crf_tables(r, 10.0, 2.0, 1.0, 1.5, 13.0)
    np.testing.assert_allclose(crf_step64(z, q, img, tab, r), crf_brute(z, q, img, tab, r), rtol=0, atol=1e-13)


def test_reference_over_row_bands():
    z, q, img = rand_case(13, 10, 4, 3)
    tab = crf_tables(3, **DEFAULTS)
    full = crf_step64(z, q, img, tab, 3)
    for rows in ((0, 4), (4, 9), (9, 13), (12, 13)):
        np.testing.assert_allclose(crf_step64(z, q, img, tab, 3, rows=rows), full[:, rows[0]:rows[1]], rtol=0,
                                   atol=1e-15)


def test_tables_are_normalised_gaussians():
    for r in (1, 4, 8, 16):
        t = crf_tables(r, **DEFAULTS)
        assert t['A'].shape == (2 * r + 1,) * 2 and t['A'][r, r] == 0 and t['S'][r, r] == 0
        assert t['A'].sum() == pytest.approx(10.0, rel=1e-14) and t['S'].sum() == pytest.approx(1.0, rel=1e-14)
        assert np.array_equal(t['A'], t['A'].T) and np.array_equal(t['A'], t['A'][::-1])
        assert t['A'][r, r + 1] > t['A'][r + 1, r + 1] and t['A'][r, r + 1] == t['A'][r + 1, r]
    assert crf_tables(2, **DEFAULTS)['coef'] == 1 / (2 * 13.0 ** 2)


def test_logits_put_the_background_first():
    m = np.random.default_rng(0).random((3, 4, 5)).astype(np.float32)
    z = logits64(m, 0.4, 16.0)
    assert z.shape == (4, 4, 5) and np.all(z[0] == 16 * float(np.float32(0.4))) and np.array_equal(z[1:], 16 * m)
    assert np.array_equal(logits64(m, None, 8.0), 8 * m.astype(np.float64))
    assert np.array_equal(logits64(m, 0, 8.0), 8 * m.astype(np.float64))       # 0: no threshold, as segment


def test_zero_weights_give_the_unary_softmax():
    z, q, img = rand_case(9, 11, 5, 1)
    tab = crf_tables(4, 0.0, 8.0, 0.0, 3.0, 13.0)
    np.testing.assert_array_equal(crf_step64(z, q, img, tab, 4), softmax64(z))


def test_single_label_is_certain():
    z, q, img = rand_case(8, 6, 1, 2)
    np.testing.assert_array_equal(crf_step64(z, np.ones_like(q), img, crf_tables(3, **DEFAULTS), 3), 1.0)


def test_constant_image_and_uniform_marginals():
    # every pair alike (e^0) and Q the same everywhere: an interior pixel's message is (appearance + smoothness) Q_l
    r, h, w = 3, 12, 13
    z = np.random.default_rng(4).random((3, h, w))
    qv = np.array([0.2, 0.5, 0.3])
    q = np.broadcast_to(qv[:, None, None], (3, h, w)).copy()
    img = np.full((h, w, 3), (40, 200, 7), dtype=np.uint8)
    _, parts = crf_step64(z, q, img, crf_tables(r, **DEFAULTS), r, parts=True)
    inner = parts['t'][:, r:h - r, r:w - r] - z[:, r:h - r, r:w - r]
    np.testing.assert_allclose(inner, 11.0 * qv[:, None, None] * np.ones_like(inner), rtol=1e-13)
    # at a corner only a quarter of the window is left: the border is not renormalised
    assert (parts['t'][:, 0, 0] - z[:, 0, 0] < 0.5 * 11.0 * qv).all()


def test_an_edge_stops_the_message():
    # two flat colour halves: with sigma_rgb small against the colour step, the appearance term no longer crosses it
    img = np.zeros((10, 16, 3), dtype=np.uint8)
    img[:, 8:] = (250, 240, 230)
    z = np.zeros((2, 10, 16))
    q = np.zeros((2, 10, 16))
    q[0, :, :8], q[1, :, 8:] = 1, 1
    _, parts = crf_step64(z, q, img, crf_tables(4, 10.0, 8.0, 0.0, 3.0, 13.0), 4, parts=True)
    assert parts['t'][1, 5, 7] < 1e-12 and parts['t'][0, 5, 7] > 3.0


def test_bound_grows_with_radius_and_covers_the_unary_softmax():
    z, q, img = rand_case(20, 24, 4, 5)
    b = {}
    for r in (1, 8, 16):
        _, parts = crf_step64(z, q, img, crf_tables(r, **DEFAULTS), r, parts=True)
        b[r], dt = crf_bound(parts, r)
        assert b[r].shape == (4, 20, 24) and dt.shape == (20, 24) and bool((b[r] > 0).all())
    assert bool((b[1] < b[8]).all()) and bool((b[8] < b[16]).all())
    # with zero weights only the softmax's own rounding is left: a few u relative
    _, parts = crf_step64(z, q, img, crf_tables(2, 0.0, 8.0, 0.0, 3.0, 13.0), 2, parts=True)
    bound, _ = crf_bound(parts, 2)
    assert bool((bound < 1e-5 * softmax64(z) + 1e-37).all())


# ---- what reaches the native call -------------------------------------------------------------------------------------
class FakeLib:
    """Stands in for libdaam_b200.so: records the arguments of daam_segment_crf."""

    def __init__(self):
        self.calls = []

    def daam_segment_crf(self, *args):
        rows, begin, n_words = args[5], args[6], args[7]
        self.calls.append(dict(n_maps=args[1], n_rows=args[2], grid=(args[3], args[4]),
                               rows=[list(rows[begin[w]:begin[w + 1]]) for w in range(n_words)],
                               out=(args[8], args[9]), absolute=args[10], use_threshold=args[11], threshold=args[12],
                               scale=args[13], iterations=args[14], radius=args[15], appearance=args[16],
                               sigma_xy=args[17], sigma_rgb=args[18], smoothness=args[19], sigma_smooth=args[20],
                               stride=args[23], probs=args[26], scratch_bytes=args[28], n_args=len(args)))
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
    whms, labels, scores = ghm.segment_crf(['dog', 'red ball'], image(40, 40))
    call, = fake.calls
    assert call['n_args'] == 30 and call['n_maps'] == 1 and call['out'] == (40, 40)
    assert call['rows'] == [[2], [5, 6]] and call['absolute'] == 0 and call['use_threshold'] == 0
    assert (call['iterations'], call['radius'], call['scale'], call['appearance'], call['sigma_xy'], call['sigma_rgb'],
            call['smoothness'], call['sigma_smooth']) == (5, 8, 16.0, 10.0, 8.0, 13.0, 1.0, 3.0)
    assert call['stride'] == 0 and call['probs'] is None
    assert call['scratch_bytes'] == _native.crf_scratch_bytes(1, 2, 40, 40)     # two labels: no background
    assert tuple(labels.shape) == (40, 40) and labels.dtype == torch.uint8 and scores.dtype == torch.float32
    assert [w.word for w in whms] == ['dog', 'red ball']
    out = ghm.segment_crf(['beach'], image(24, 24).numpy(), threshold=0.4, iterations=0, radius=16, scale=8,
                          appearance=0, sigma_xy=2.5, sigma_rgb=40, smoothness=0.5, sigma_smooth=1, absolute=True,
                          probs=True)
    call = fake.calls[-1]
    assert (call['use_threshold'], call['threshold'], call['iterations'], call['radius'], call['scale'],
            call['appearance'], call['sigma_xy'], call['sigma_rgb'], call['smoothness'], call['sigma_smooth'],
            call['absolute']) == (1, 0.4, 0, 16, 8.0, 0.0, 2.5, 40.0, 0.5, 1.0, 1)
    assert call['probs'] is not None and call['scratch_bytes'] == _native.crf_scratch_bytes(1, 2, 24, 24)
    assert len(out) == 4 and tuple(out[3].shape) == (2, 24, 24) and out[3].dtype == torch.float32
    ghm.segment_crf(['beach'], image(24, 24), threshold=0)                        # 0: no threshold, as segment
    assert fake.calls[-1]['use_threshold'] == 0
    rect = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 12, 20))
    _, labels, _ = rect.segment_crf(['dog'], image(30, 50), radius=1)
    assert fake.calls[-1]['out'] == (30, 50) and tuple(labels.shape) == (30, 50)


def test_stacks_are_one_call_over_every_map(fake, monkeypatch):
    tm = TimeHeatMaps(TOK, PROMPT, torch.zeros(5, 11, 16, 16))
    word_maps, labels, scores = tm.segment_crf(['dog', 'beach'], image(32, 32), threshold=0.4)
    call, = fake.calls
    assert call['n_maps'] == 5 and call['rows'] == [[2], [9]] and call['stride'] == 0
    assert call['scratch_bytes'] == _native.crf_scratch_bytes(5, 3, 32, 32)
    assert tuple(word_maps.shape) == (5, 2, 16, 16) and tuple(labels.shape) == (5, 32, 32)
    assert tuple(scores.shape) == (5, 32, 32)
    _, _, _, probs = tm.segment_crf(['dog', 'beach'], image(32, 32), probs=True)
    assert tuple(probs.shape) == (5, 2, 32, 32)
    # one image per map: its stride
    im = ImageHeatMaps(TOK, PROMPT, torch.zeros(3, 11, 16, 16))
    im.segment_crf(['dog', 'beach'], image(32, 32, 3))
    assert fake.calls[-1]['stride'] == 32 * 32 * 3 and fake.calls[-1]['n_maps'] == 3
    lm = LayerHeatMaps(TOK, PROMPT, torch.zeros(2, 11, 16, 12), [3, 7], ['a', 'b'], [1, 2])
    _, labels, _ = lm.segment_crf(['ball'], image(32, 24))
    assert fake.calls[-1]['n_maps'] == 2 and fake.calls[-1]['grid'] == (16, 12) and tuple(labels.shape) == (2, 32, 24)
    # the scratch budget caps a long stack (rounds of whole maps), and one map is the least a call gets
    monkeypatch.setattr(heatmap, 'CRF_SCRATCH_BYTES', _native.crf_scratch_bytes(2, 3, 32, 32))
    tm.segment_crf(['dog', 'beach'], image(32, 32), threshold=0.4)
    assert fake.calls[-1]['scratch_bytes'] == _native.crf_scratch_bytes(2, 3, 32, 32)
    monkeypatch.setattr(heatmap, 'CRF_SCRATCH_BYTES', 1)
    tm.segment_crf(['dog', 'beach'], image(32, 32), threshold=0.4)
    assert fake.calls[-1]['scratch_bytes'] == _native.crf_scratch_bytes(1, 3, 32, 32)


def test_scratch_size_matches_the_header():
    assert _native.crf_map_bytes(9, 512, 512) == 8 * 9 * 512 * 512 + 256 * 9
    assert _native.crf_scratch_bytes(3, 97, 600, 800) == 3 * (8 * 97 * 480000 + 256 * 97)
    assert 'daam_segment_crf' in _native.EXPORTS and _native.CRF_MAX_RADIUS == 16
    assert _native.CRF_MAX_ITERATIONS == 64 and heatmap.CRF_SCRATCH_BYTES == 256 << 20
    import os
    header = open(os.path.join(os.path.dirname(_native.__file__), '..', 'include', 'daam_b200.h')).read()
    assert '#define DAAM_CRF_MAX_RADIUS 16' in header
    assert ('#define DAAM_CRF_MAP_BYTES(n_labels, out_h, out_w) (8 * (int64_t)(n_labels) * (out_h) * (out_w) + '
            '256 * (int64_t)(n_labels))') in header
    assert ('#define DAAM_CRF_SCRATCH_BYTES(n_maps, n_labels, out_h, out_w) ((int64_t)(n_maps) * '
            'DAAM_CRF_MAP_BYTES(n_labels, out_h, out_w))') in header


# ---- refusals, all before the native library ----------------------------------------------------------------------------
@pytest.fixture
def no_native(monkeypatch):
    def load():
        raise AssertionError('the native library was reached')
    monkeypatch.setattr(_native, 'load', load)
    monkeypatch.setattr(heatmap, '_require_cuda', lambda t, what: None)


@pytest.mark.parametrize('kw,text', [
    (dict(radius=0), r'radius must be an integer in \[1, 16\]'),
    (dict(radius=17), r'radius must be an integer in \[1, 16\]'),
    (dict(radius=8.0), r'radius must be an integer in \[1, 16\]'),
    (dict(radius=True), r'radius must be an integer in \[1, 16\]'),
    (dict(iterations=-1), r'iterations must be an integer in \[0, 64\]'),
    (dict(iterations=65), r'iterations must be an integer in \[0, 64\]'),
    (dict(iterations=None), r'iterations must be an integer in \[0, 64\]'),
    (dict(scale=0.0), 'scale must be finite and > 0'),
    (dict(scale=1e39), 'scale must be finite and > 0'),
    (dict(scale='x'), 'scale must be a number'),
    (dict(sigma_xy=-1.0), 'sigma_xy must be finite and > 0'),
    (dict(sigma_rgb=float('nan')), 'sigma_rgb must be finite and > 0'),
    (dict(sigma_smooth=1e-50), 'sigma_smooth must be finite and > 0'),
    (dict(appearance=-0.5), 'appearance must be finite and >= 0'),
    (dict(smoothness=float('inf')), 'smoothness must be finite and >= 0'),
    (dict(threshold=float('inf')), 'threshold must be finite'),
    (dict(threshold=float('nan')), 'threshold must be finite'),
])
def test_argument_refusals(no_native, kw, text):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16))
    with pytest.raises(ValueError, match='GlobalHeatMap.segment_crf: ' + text):
        ghm.segment_crf(['dog'], image(32, 32), **kw)


def test_refusal_order(no_native):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16))
    # the words first, then the row range, then the image, then the CRF arguments in daam_segment_crf's order
    with pytest.raises(ValueError, match='Search word zebra not found in prompt!'):
        ghm.segment_crf(['zebra'], 'not an image', radius=0)
    with pytest.raises(IndexError, match='out of bounds'):
        GlobalHeatMap(TOK, PROMPT, torch.zeros(4, 16, 16)).segment_crf(['beach'], 'not an image', radius=0)
    with pytest.raises(TypeError, match='PIL image or a uint8'):
        ghm.segment_crf(['dog'], 'not an image', radius=0)
    with pytest.raises(TypeError, match='must be uint8'):
        ghm.segment_crf(['dog'], torch.zeros(32, 32, 3), iterations=-1)
    with pytest.raises(ValueError, match='transposes a non-square image'):
        ghm.segment_crf(['dog'], image(30, 40), radius=0)
    with pytest.raises(ValueError, match=r'is not \[H, W, 3\]'):
        ghm.segment_crf(['dog'], image(32, 32, 2))                     # one map takes one image
    tm = TimeHeatMaps(TOK, PROMPT, torch.zeros(3, 11, 16, 16))
    with pytest.raises(ValueError, match=r'is not \[3, H, W, 3\] or \[H, W, 3\]'):
        tm.segment_crf(['dog'], image(32, 32, 2), radius=0)
    for kw, first in [(dict(radius=0, iterations=-1), 'radius'), (dict(iterations=-1, scale=0), 'iterations'),
                      (dict(scale=0, sigma_xy=0), 'scale'), (dict(sigma_xy=0, sigma_rgb=0), 'sigma_xy'),
                      (dict(sigma_rgb=0, sigma_smooth=0), 'sigma_rgb'),
                      (dict(sigma_smooth=0, appearance=-1), 'sigma_smooth'),
                      (dict(appearance=-1, smoothness=-1), 'appearance'),
                      (dict(smoothness=-1, threshold=float('inf')), 'smoothness')]:
        with pytest.raises(ValueError, match=f'TimeHeatMaps.segment_crf: {first} '):
            tm.segment_crf(['dog'], image(32, 32, 3), **kw)
    with pytest.raises(ValueError, match='radius'):
        tm.segment_crf([], image(32, 32), radius=0)                   # an empty list is checked too


def test_cpu_maps_are_refused(monkeypatch):
    monkeypatch.setattr(_native, 'load', lambda: (_ for _ in ()).throw(AssertionError('reached the library')))
    with pytest.raises(RuntimeError, match='GlobalHeatMap.segment_crf: .*CUDA tensors only'):
        GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16)).segment_crf(['dog'], image(32, 32))


# ---- empty inputs --------------------------------------------------------------------------------------------------------
def test_empty_inputs_launch_nothing(fake):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16))
    whms, labels, scores = ghm.segment_crf([], image(32, 32))
    assert whms == [] and tuple(labels.shape) == (32, 32) and not labels.any() and not scores.any()
    whms, labels, scores, probs = ghm.segment_crf([], image(32, 32), threshold=0.4, probs=True)
    assert not labels.any() and bool((scores == 1).all()) and tuple(probs.shape) == (1, 32, 32)
    assert bool((probs == 1).all())
    word_maps, labels, scores, probs = TimeHeatMaps(TOK, PROMPT, torch.zeros(4, 11, 16, 16)).segment_crf(
        [], image(32, 32, 4), probs=True)
    assert tuple(labels.shape) == (4, 32, 32) and tuple(word_maps.shape) == (4, 0, 16, 16)
    assert tuple(probs.shape) == (4, 0, 32, 32)
    _, labels, _ = TimeHeatMaps(TOK, PROMPT, torch.zeros(0, 11, 16, 16)).segment_crf(['dog'], image(32, 32))
    assert tuple(labels.shape) == (0, 32, 32)
    assert fake.calls == []
    assert not math.isnan(float(heatmap.CRF_SCRATCH_BYTES))
