"""Word distance maps on the host, no GPU: the integer reference of tests/distance64.py against brute force and a
separable minimum; WordDistance's mask() against scipy's binary dilation and erosion by disks, the closing composed
from it, and distance() / soft_mask() against numpy float64 formulas bit for bit in fp32; every refusal and its order,
all before the native library; the arguments and scratch GlobalHeatMap.word_distance, the stacks and
evaluate.distance_transform hand to daam_word_distance / daam_mask_distance; and the empty shapes."""
import contextlib
import ctypes
import math

import numpy as np
import pytest
import torch
from scipy import ndimage

from daam_b200 import _native, evaluate, heatmap
from daam_b200.evaluate import distance_transform
from daam_b200.heatmap import GlobalHeatMap, LayerHeatMaps, TimeHeatMaps, WordDistance
from daam_b200.testing.synthetic import WhitespaceTokenizer
from tests.distance64 import NONE, brute_force, kinds, separable, signed_d2, signed_d2_plane

TOK = WhitespaceTokenizer()
PROMPT = 'a dog chasing a red ball on the beach'


class Im:
    def __init__(self, h, w):
        self.size, self.height, self.width = (w, h), h, w


# ---- the reference ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('seed,h,w', [(0, 1, 1), (1, 1, 9), (2, 7, 1), (3, 12, 17), (4, 23, 8), (5, 20, 20)])
def test_reference_against_brute_force(seed, h, w):
    for m in kinds(seed, h, w):
        np.testing.assert_array_equal(signed_d2_plane(m), brute_force(m))


@pytest.mark.parametrize('seed,h,w', [(6, 64, 90), (7, 37, 129), (8, 100, 3)])
def test_reference_against_separable(seed, h, w):
    for m in kinds(seed, h, w):
        np.testing.assert_array_equal(signed_d2_plane(m), separable(m))


def test_reference_definition():
    m = np.zeros((5, 7), bool)
    m[2, 3] = True
    d = signed_d2_plane(m)
    assert d[2, 3] == -1 and d[0, 0] == 4 + 9 and d[4, 6] == 4 + 9 and d.dtype == np.int32
    full = signed_d2_plane(np.ones((3, 4), bool))
    assert (full == -NONE).all() and (signed_d2_plane(np.zeros((3, 4), bool)) == NONE).all()
    # the border is not background: a mask touching it is not eaten from it
    m = np.ones((5, 5), bool)
    m[0, 0] = False
    assert signed_d2_plane(m)[4, 4] == -32 and signed_d2_plane(m)[4, 0] == -16
    assert signed_d2(np.zeros((2, 0, 3, 4))).shape == (2, 0, 3, 4)


# ---- WordDistance's helpers -----------------------------------------------------------------------------------------------
def disk(r):
    k = int(math.floor(abs(r)))
    yy, xx = np.indices((2 * k + 1, 2 * k + 1)) - k
    return (yy * yy + xx * xx).astype(np.float64) <= float(r) * float(r)


RADII = [0, 0.5, 1, 1.4, 1.5, 2, 2.5, 3, 4.2, 7]


@pytest.mark.parametrize('seed,h,w', [(10, 1, 13), (11, 9, 1), (12, 31, 40), (13, 50, 23)])
def test_mask_is_dilation_and_erosion_by_a_disk(seed, h, w):
    masks = kinds(seed, h, w)
    wd = WordDistance(torch.from_numpy(signed_d2(masks)))
    for r in RADII:
        grown, shrunk = wd.mask(r).numpy(), wd.mask(-r).numpy()
        assert grown.dtype == np.bool_ and grown.shape == masks.shape
        for i, m in enumerate(masks):
            np.testing.assert_array_equal(grown[i], ndimage.binary_dilation(m, disk(r)), err_msg=f'{i} +{r}')
            np.testing.assert_array_equal(shrunk[i], ndimage.binary_erosion(m, disk(r), border_value=1),
                                          err_msg=f'{i} -{r}')
    np.testing.assert_array_equal(wd.mask().numpy(), masks)


@pytest.mark.parametrize('r', [1, 1.5, 3, 4.2])
def test_closing_composes(r):
    masks = kinds(14, 40, 56)
    wd = WordDistance(torch.from_numpy(signed_d2(masks)))
    closed = WordDistance(torch.from_numpy(signed_d2(wd.mask(r).numpy()))).mask(-r).numpy()
    for i, m in enumerate(masks):
        want = ndimage.binary_erosion(ndimage.binary_dilation(m, disk(r)), disk(r), border_value=1)
        np.testing.assert_array_equal(closed[i], want, err_msg=str(i))


def _signed64(d2):
    d2 = d2.astype(np.float64)
    s = np.sign(d2) * np.sqrt(np.abs(d2))
    return np.where(np.abs(d2) == NONE, np.sign(d2) * np.inf, s)


@pytest.mark.parametrize('lead', [(), (3,)], ids=['one-map', 'stack'])
def test_distance_and_soft_mask_against_numpy(lead):
    masks = kinds(15, 33, 47)[:7]
    d2 = signed_d2(np.broadcast_to(masks, lead + masks.shape).copy())
    d2[..., 0, 0, 0] = NONE                                               # the sentinels of empty / full masks
    wd = WordDistance(torch.from_numpy(d2))
    s = _signed64(d2)
    dist = wd.distance()
    assert dist.dtype == torch.float32 and tuple(dist.shape) == d2.shape
    np.testing.assert_array_equal(dist.numpy(), s.astype(np.float32))
    assert np.isposinf(dist.numpy()[..., 0, :, :]).all() and np.isneginf(dist.numpy()[..., 1, :, :]).all()
    for grow, feather in [(0, 1), (16, 8), (-2, 3), (2.5, 0.75), (0.1, 1e-3)]:
        soft = wd.soft_mask(grow, feather=feather)
        with np.errstate(invalid='ignore'):
            want = np.clip((grow + feather - s) / feather, 0, 1).astype(np.float32)
        assert soft.dtype == torch.float32
        np.testing.assert_array_equal(soft.numpy(), want, err_msg=f'{grow} {feather}')
        assert bool((soft[wd.mask(grow)] == 1).all())
    assert torch.equal(wd.map(0).signed_d2, wd.signed_d2[0]) if lead else True
    assert wd.cpu().signed_d2 is not None


def test_helper_refusals():
    wd = WordDistance(torch.tensor([[1, -1]], dtype=torch.int32))
    for f in (0, -1, math.inf, math.nan, None, '1'):
        with pytest.raises(ValueError, match='feather'):
            wd.soft_mask(1.0, feather=f)
    for g in (math.inf, -math.inf, math.nan, None, True):
        with pytest.raises(ValueError, match='grow must be a finite number'):
            wd.mask(g)
        with pytest.raises(ValueError, match='grow must be a finite number'):
            wd.soft_mask(g, feather=1.0)
    with pytest.raises(TypeError):
        wd.soft_mask(1.0)                                                 # feather has no default


# ---- refusals -----------------------------------------------------------------------------------------------------------
def no_native():
    raise AssertionError('the native library was reached')


def test_refusals_before_the_native_library(monkeypatch):
    monkeypatch.setattr(_native, 'load', no_native)
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16))
    for t in (None, 0, 0.0, False):
        with pytest.raises(ValueError, match='threshold must be set'):
            ghm.word_distance(['dog'], Im(32, 32), t)
    for t in (math.inf, -math.inf, math.nan):
        with pytest.raises(ValueError, match='threshold must be finite'):
            ghm.word_distance(['zebra'], Im(32, 32), t)                    # before the words
    prompt = ' '.join(f'w{i}' for i in range(100))
    with pytest.raises(ValueError, match='97 words > 96'):
        GlobalHeatMap(TOK, prompt, torch.zeros(102, 16, 16)).word_distance([f'w{i}' for i in range(97)], Im(8, 8), 0.4)
    with pytest.raises(ValueError, match='Search word zebra not found in prompt!'):
        ghm.word_distance(['dog', 'zebra'], Im(32, 32), 0.4)
    with pytest.raises(ValueError, match='Search word zebra not found in prompt!'):
        TimeHeatMaps(TOK, PROMPT, torch.zeros(3, 11, 16, 16)).word_distance(['zebra'], Im(32, 32), 0.4)
    with pytest.raises(RuntimeError, match='GlobalHeatMap.word_distance: .*CUDA tensors only'):
        ghm.word_distance(['dog'], Im(40000, 40000), 0.4)                 # the CUDA check comes before the size
    with pytest.raises(RuntimeError, match='TimeHeatMaps.word_distance: .*CUDA tensors only'):
        TimeHeatMaps(TOK, PROMPT, torch.zeros(3, 11, 16, 16)).word_distance(['dog'], Im(32, 32), 0.4)
    with pytest.raises(TypeError, match='masks must be a torch.Tensor'):
        distance_transform(np.zeros((4, 4), bool))
    with pytest.raises(TypeError, match='masks must be bool or uint8'):
        distance_transform(torch.zeros(4, 4))
    for shape in ((4,), (1, 1, 1, 4, 4)):
        with pytest.raises(ValueError, match=r'masks must be \[H, W\]'):
            distance_transform(torch.zeros(shape, dtype=torch.bool))
    with pytest.raises(RuntimeError, match='distance_transform: .*CUDA tensors only'):
        distance_transform(torch.zeros(1 << 15, 1, dtype=torch.bool))


# ---- what reaches the native calls -----------------------------------------------------------------------------------
class FakeLib:
    """Stands in for libdaam_b200.so: records the arguments of daam_word_distance / daam_mask_distance and writes each
    output plane's index into its first pixel."""

    def __init__(self):
        self.calls = []

    def daam_word_distance(self, *a):
        rows, begin, n_words, n_maps = a[5], a[6], a[7], a[1]
        self.calls.append(dict(entry='word', n_maps=n_maps, n_rows=a[2], grid=(a[3], a[4]), out=(a[8], a[9]),
                               absolute=a[10], threshold=a[11], scratch_bytes=a[15],
                               rows=[list(rows[begin[w]:begin[w + 1]]) for w in range(n_words)]))
        self._mark(a[13].value, n_maps * n_words, a[8] * a[9])
        return 0

    def daam_mask_distance(self, *a):
        self.calls.append(dict(entry='mask', n_planes=a[1], out=(a[2], a[3])))
        self._mark(a[4].value, a[1], a[2] * a[3])
        return 0

    @staticmethod
    def _mark(ptr, planes, n):
        for p in range(planes):
            ctypes.memmove(ptr + 4 * p * n, ctypes.byref(ctypes.c_int32(p)), 4)


@pytest.fixture
def fake(monkeypatch):
    lib = FakeLib()
    monkeypatch.setattr(_native, 'load', lambda: lib)
    monkeypatch.setattr(heatmap, '_require_cuda', lambda t, what: None)
    monkeypatch.setattr(heatmap, '_stream_ptr', lambda dev: 0)
    monkeypatch.setattr(torch.cuda, 'device', lambda dev: contextlib.nullcontext())
    return lib


def test_arguments_and_scratch(fake):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 12, 20))
    whms, wd = ghm.word_distance(['dog', 'red ball'], Im(40, 48), 0.4, absolute=True)
    call, = fake.calls
    plane = _native.distance_plane_bytes(40, 48)
    assert call['n_maps'] == 1 and call['grid'] == (12, 20) and call['out'] == (40, 48) and call['rows'] == [[2], [5, 6]]
    assert call['absolute'] == 1 and call['threshold'] == pytest.approx(0.4) and call['scratch_bytes'] == 2 * plane
    assert [w.word for w in whms] == ['dog', 'red ball'] and isinstance(wd, WordDistance)
    assert tuple(wd.signed_d2.shape) == (2, 40, 48) and wd.signed_d2.dtype == torch.int32 and not wd.signed_d2.is_cuda
    assert wd.signed_d2[:, 0, 0].tolist() == [0, 1]
    GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16)).word_distance(['dog'], Im(30, 44), 0.4)
    assert fake.calls[-1]['out'] == (44, 30) and fake.calls[-1]['absolute'] == 0   # a square map keeps (size[0], size[1])
    # a long stack: scratch stays at the budget
    tm = TimeHeatMaps(TOK, PROMPT, torch.zeros(50, 11, 16, 16))
    _, wd = tm.word_distance(['dog', 'ball', 'beach'], Im(1024, 1024), 0.4)
    assert fake.calls[-1]['scratch_bytes'] == heatmap.WORD_DISTANCE_SCRATCH_BYTES and fake.calls[-1]['n_maps'] == 50
    assert tuple(wd.signed_d2.shape) == (50, 3, 1024, 1024) and wd.signed_d2[7, 2, 0, 0] == 7 * 3 + 2
    lm = LayerHeatMaps(TOK, PROMPT, torch.zeros(2, 11, 16, 16), [0, 1], ['a', 'b'], [1, 1])
    word_maps, wd = lm.word_distance(['dog'], Im(8, 8), 0.4, to_cpu=False)
    assert tuple(word_maps.shape) == (2, 1, 16, 16) and tuple(wd.signed_d2.shape) == (2, 1, 8, 8)
    assert fake.calls[-1]['scratch_bytes'] == 2 * _native.distance_plane_bytes(8, 8)
    # the mask entry: one plane per [H, W] mask, the masks' shape back
    for shape in ((5, 7), (3, 5, 7), (2, 3, 5, 7)):
        out = distance_transform(torch.zeros(shape, dtype=torch.bool))
        assert fake.calls[-1] == dict(entry='mask', n_planes=int(np.prod(shape[:-2])), out=(5, 7))
        assert tuple(out.signed_d2.shape) == shape and out.signed_d2.dtype == torch.int32
        assert out.signed_d2.reshape(-1, 5, 7)[:, 0, 0].tolist() == list(range(int(np.prod(shape[:-2]))))
    distance_transform(torch.zeros(2, 3, dtype=torch.uint8))
    assert fake.calls[-1] == dict(entry='mask', n_planes=1, out=(2, 3))


def test_size_refusals(fake):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 24))
    with pytest.raises(ValueError, match='a 32768 x 8 image has a side > 32767'):
        ghm.word_distance(['dog'], Im(32768, 8), 0.4)
    with pytest.raises(ValueError, match='a 4097 x 4097 image is more than 2\\*\\*24 pixels'):
        ghm.word_distance(['dog'], Im(4097, 4097), 0.4)
    with pytest.raises(ValueError, match='a 1 x 32768 image has a side > 32767'):
        distance_transform(torch.zeros(1, 32768, dtype=torch.bool))
    with pytest.raises(ValueError, match='more than 2\\*\\*24 pixels'):
        distance_transform(torch.zeros(4097, 4097, dtype=torch.bool))
    assert fake.calls == []
    ghm.word_distance(['dog'], Im(32767, 512), 0.4)                       # the largest allowed: 16,776,704 pixels
    assert fake.calls[-1]['out'] == (32767, 512)


def test_plane_bytes_match_the_header():
    # 4 bytes a pixel for the values, 256 for the min / max partials
    assert _native.distance_plane_bytes(512, 512) == 4 * 512 * 512 + 256
    assert _native.distance_plane_bytes(1, 1) == 260
    assert _native.DISTANCE_NONE == NONE == 2 ** 31 - 1 and _native.DISTANCE_MAX_SIDE == 32767
    assert {'daam_word_distance', 'daam_mask_distance'} <= set(_native.EXPORTS)
    assert 'WordDistance' in heatmap.__all__ and 'distance_transform' in evaluate.__all__


def test_empty_inputs_launch_nothing(fake):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16))
    whms, wd = ghm.word_distance([], Im(32, 32), 0.4)
    assert whms == [] and tuple(wd.signed_d2.shape) == (0, 32, 32)
    assert tuple(wd.mask(3).shape) == (0, 32, 32) and tuple(wd.soft_mask(1, feather=2).shape) == (0, 32, 32)
    word_maps, wd = TimeHeatMaps(TOK, PROMPT, torch.zeros(4, 11, 16, 16)).word_distance([], Im(32, 32), 0.4)
    assert tuple(wd.signed_d2.shape) == (4, 0, 32, 32) and tuple(word_maps.shape) == (4, 0, 16, 16)
    _, wd = TimeHeatMaps(TOK, PROMPT, torch.zeros(0, 11, 16, 16)).word_distance(['dog'], Im(32, 32), 0.4)
    assert tuple(wd.signed_d2.shape) == (0, 1, 32, 32)
    for shape in ((0, 5), (3, 0), (0, 4, 4), (2, 0, 4, 4)):
        assert tuple(distance_transform(torch.zeros(shape, dtype=torch.bool)).signed_d2.shape) == shape
    assert fake.calls == []
