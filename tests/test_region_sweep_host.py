"""Threshold sweeps of word-region overlap on the host, no GPU: the threshold checks (type, length, fp32 rounding,
order, finiteness), the word, region and CPU-tensor refusals, all before anything reaches the native library; the
arguments GlobalHeatMap.region_sweep and the stacks hand to daam_region_sweep (fp32 threshold array, T, buffer sizes);
the empty shapes; and RegionOverlap's formulas over a threshold axis against numpy."""
import contextlib
import ctypes

import numpy as np
import pytest
import torch

from daam_b200 import _native, heatmap
from daam_b200.heatmap import GlobalHeatMap, LayerHeatMaps, RegionOverlap, TimeHeatMaps
from daam_b200.testing.synthetic import WhitespaceTokenizer

TOK = WhitespaceTokenizer()
PROMPT = 'a dog chasing a red ball on the beach'
SWEEP = [0.05 * i for i in range(1, 20)]


class Im:
    def __init__(self, h, w):
        self.size, self.height, self.width = (w, h), h, w


# ---- RegionOverlap formulas over a threshold axis -------------------------------------------------------------------
def test_formulas_against_numpy_with_a_threshold_axis():
    g = np.random.default_rng(0)
    inter = g.integers(0, 50, (2, 3, 4, 5)).astype(np.float32)          # [maps 2, T 3, R 4, W 5]
    word_area = inter.max(2) + g.integers(0, 20, (2, 3, 5)).astype(np.float32)
    region_area = np.array([60., 0., 35., 100.], dtype=np.float32)
    ov = RegionOverlap(torch.from_numpy(inter), torch.from_numpy(word_area), torch.from_numpy(region_area))
    eps = np.float32(1e-8)
    iou = inter / (word_area[:, :, None, :] + region_area[None, None, :, None] - inter + eps)
    ioa = inter / (word_area[:, :, None, :] + eps)
    mean = inter / (region_area[None, None, :, None] + eps)
    assert tuple(ov.iou().shape) == (2, 3, 4, 5) and ov.iou().dtype == torch.float32
    np.testing.assert_array_equal(ov.iou().numpy(), iou.astype(np.float32))
    np.testing.assert_array_equal(ov.ioa().numpy(), ioa.astype(np.float32))
    np.testing.assert_array_equal(ov.region_mean().numpy(), mean.astype(np.float32))
    one = ov.map(1)                                                       # one map: [T, R, W]
    assert tuple(one.intersection.shape) == (3, 4, 5) and torch.equal(one.iou(), ov.iou()[1])
    # slice k of a sweep scores like a one-threshold overlap
    k = RegionOverlap(one.intersection[2], one.word_area[2], one.region_area)
    assert torch.equal(k.iou(), one.iou()[2]) and torch.equal(k.ioa(), one.ioa()[2])
    assert torch.equal(k.region_mean(), one.region_mean()[2])


# ---- what reaches the native call ----------------------------------------------------------------------------------
class FakeLib:
    """Stands in for libdaam_b200.so: records the arguments of daam_region_sweep."""

    def __init__(self):
        self.calls = []

    def daam_region_sweep(self, *args):
        rows, begin, n_words = args[5], args[6], args[7]
        taus, n_thr = args[11], args[12]
        assert isinstance(taus, ctypes.Array) and taus._type_ is ctypes.c_float
        self.calls.append(dict(n_maps=args[1], n_rows=args[2], grid=(args[3], args[4]),
                               rows=[list(rows[begin[w]:begin[w + 1]]) for w in range(n_words)],
                               out=(args[8], args[9]), absolute=args[10], thresholds=list(taus[:n_thr]),
                               n_thresholds=n_thr, n_regions=args[15], n_args=len(args)))
        return 0


@pytest.fixture
def fake(monkeypatch):
    lib = FakeLib()
    scratch = []
    monkeypatch.setattr(_native, 'load', lambda: lib)
    monkeypatch.setattr(heatmap, '_require_cuda', lambda t, what: None)
    monkeypatch.setattr(heatmap, '_stream_ptr', lambda dev: 0)
    monkeypatch.setattr(torch.cuda, 'device', lambda dev: contextlib.nullcontext())
    real_scratch = heatmap._WordList.scratch
    monkeypatch.setattr(heatmap._WordList, 'scratch', lambda self, n: scratch.append(n) or real_scratch(self, n))
    lib.scratch = scratch
    return lib


def test_fp32_thresholds_and_sizes_reach_the_native_call(fake):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16))
    regions = torch.zeros(3, 40, 40, dtype=torch.bool)
    whms, ov = ghm.region_sweep(['dog', 'red ball'], Im(40, 40), regions, SWEEP)
    call, = fake.calls
    assert call['n_args'] == 20 and call['n_thresholds'] == 19
    assert call['thresholds'] == [float(np.float32(t)) for t in SWEEP]   # the fp32 values, in order
    assert call['n_maps'] == 1 and call['n_regions'] == 3 and call['out'] == (40, 40) and call['rows'] == [[2], [5, 6]]
    assert call['absolute'] == 0
    assert fake.scratch == [_native.region_sweep_scratch_floats(1, 2, 3, 19, 40, 40)] == [2 * (64 + 4 * 19)]
    assert tuple(ov.intersection.shape) == (19, 3, 2) and tuple(ov.word_area.shape) == (19, 2)
    assert tuple(ov.region_area.shape) == (3,) and ov.intersection.dtype == torch.float32
    assert tuple(ov.iou().shape) == (19, 3, 2)
    assert [w.word for w in whms] == ['dog', 'red ball']


@pytest.mark.parametrize('thresholds', [[0.0], [-1.0, 0.0, 0.5], torch.tensor([0.1, 0.2], dtype=torch.float64),
                                        torch.arange(64) / 64 - 0.5, np.array([0.25, 0.75], dtype=np.float32), (1, 2)])
def test_literal_thresholds_reach_the_native_call(fake, thresholds):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 12, 20))
    _, ov = ghm.region_sweep(['dog'], Im(30, 44), torch.ones(30, 44, dtype=torch.uint8), thresholds, absolute=True)
    call, = fake.calls
    want = torch.as_tensor(np.asarray(thresholds, dtype=np.float64)).float().tolist()
    assert call['thresholds'] == want and call['n_thresholds'] == len(want)   # 0 and negatives are thresholds
    assert call['absolute'] == 1 and call['grid'] == (12, 20) and call['out'] == (30, 44)
    assert tuple(ov.intersection.shape) == (len(want), 1, 1)


def test_stacks_are_one_call_over_every_map(fake):
    tm = TimeHeatMaps(TOK, PROMPT, torch.zeros(5, 11, 16, 16))
    word_maps, ov = tm.region_sweep(['dog', 'beach'], Im(32, 32), torch.zeros(4, 32, 32, dtype=torch.uint8),
                                    [0.2, 0.4, 0.6])
    call, = fake.calls
    assert call['n_maps'] == 5 and call['n_regions'] == 4 and call['rows'] == [[2], [9]]
    assert call['n_thresholds'] == 3
    assert fake.scratch == [_native.region_sweep_scratch_floats(5, 2, 4, 3, 32, 32)]
    assert tuple(word_maps.shape) == (5, 2, 16, 16)
    assert tuple(ov.intersection.shape) == (5, 3, 4, 2) and tuple(ov.word_area.shape) == (5, 3, 2)
    assert tuple(ov.iou().shape) == (5, 3, 4, 2)
    lm = LayerHeatMaps(TOK, PROMPT, torch.zeros(2, 11, 16, 16), [3, 7], ['a', 'b'], [1, 2])
    _, ov = lm.region_sweep(['ball'], Im(32, 32), torch.zeros(32, 32, dtype=torch.bool), [0.5])
    assert fake.calls[-1]['n_maps'] == 2 and tuple(ov.intersection.shape) == (2, 1, 1, 1)


def test_scratch_size_matches_the_header():
    assert _native.region_sweep_scratch_floats(1, 1, 1, 1, 16, 64) == 64 + 2
    assert _native.region_sweep_scratch_floats(3, 8, 4, 64, 1216, 832) == 3 * 8 * (64 + 5 * 64)
    assert _native.region_sweep_scratch_floats(2, 96, 63, 19, 4096, 4096) == 2 * 96 * (64 + 64 * 19)
    assert 'daam_region_sweep' in _native.EXPORTS and _native.SWEEP_MAX_THRESHOLDS == 64


# ---- refusals, all before the native library --------------------------------------------------------------------------
@pytest.fixture
def no_native(monkeypatch):
    def load():
        raise AssertionError('the native library was reached')
    monkeypatch.setattr(_native, 'load', load)


@pytest.mark.parametrize('thresholds,match', [
    ([0.4, 0.2], 'strictly ascending'),
    ([0.1, 0.1], 'strictly ascending'),
    ([0.1, 0.1 + 1e-9], 'strictly ascending'),                   # distinct in float64, one value in fp32
    ([0.5, float('nan')], 'finite'),
    ([float('-inf'), 0.5], 'finite'),
    ([0.5, 1e39], 'finite'),                                     # overflows fp32
    ([], '0 thresholds'),
    ([i / 65 for i in range(65)], '65 thresholds'),
    (torch.zeros(0), '0 thresholds'),
    (torch.tensor(0.4), '1-D'),
    (torch.tensor([[0.1, 0.2]]), '1-D'),
    (torch.tensor([True, False]), '1-D real'),
    (0.4, 'sequence of numbers'),
    (['0.4'], 'numbers'),
    ([True], 'numbers'),
    ([0.2, None], 'numbers'),
])
def test_threshold_refusals(no_native, thresholds, match):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16))
    with pytest.raises(ValueError, match=match):
        ghm.region_sweep(['dog'], Im(32, 32), torch.zeros(1, 32, 32, dtype=torch.bool), thresholds)
    with pytest.raises(ValueError, match=match):
        TimeHeatMaps(TOK, PROMPT, torch.zeros(3, 11, 16, 16)).region_sweep(
            ['dog'], Im(32, 32), torch.zeros(1, 32, 32, dtype=torch.bool), thresholds)


def test_device_thresholds_are_refused(no_native):
    meta = torch.zeros(3, device='meta')                  # stands in for a device tensor: not on the CPU
    with pytest.raises(ValueError, match='CPU tensor'):
        GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16)).region_sweep(
            ['dog'], Im(32, 32), torch.zeros(1, 32, 32, dtype=torch.bool), meta)


def test_region_refusals(fake):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 12, 20))
    img = Im(30, 44)
    with pytest.raises(ValueError, match=r'\(2, 44, 30\).*\(R, 30, 44\)'):
        ghm.region_sweep(['dog'], img, torch.zeros(2, 44, 30, dtype=torch.bool), SWEEP)
    with pytest.raises(ValueError, match=r'\(2, 2, 30, 44\)'):
        ghm.region_sweep(['dog'], img, torch.zeros(2, 2, 30, 44, dtype=torch.bool), SWEEP)
    with pytest.raises(TypeError, match='bool or uint8'):
        ghm.region_sweep(['dog'], img, torch.zeros(1, 30, 44), SWEEP)
    with pytest.raises(TypeError, match='torch.Tensor'):
        ghm.region_sweep(['dog'], img, np.zeros((1, 30, 44), dtype=np.uint8), SWEEP)
    assert fake.calls == []


def test_cpu_tensors_are_refused(monkeypatch, no_native):
    img = Im(32, 32)
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16))
    with pytest.raises(RuntimeError, match='CUDA tensors only'):          # the CPU map
        ghm.region_sweep(['dog'], img, torch.zeros(1, 32, 32, dtype=torch.bool), SWEEP)
    # a device map (stood in for: the 4-d map stack passes the check) with CPU regions: the regions are refused
    real = heatmap._require_cuda
    monkeypatch.setattr(heatmap, '_require_cuda', lambda t, what: None if t.dim() == 4 else real(t, what))
    with pytest.raises(RuntimeError, match='GlobalHeatMap.region_sweep: .*CUDA tensors only'):
        ghm.region_sweep(['dog'], img, torch.zeros(1, 32, 32, dtype=torch.bool), SWEEP)


def test_unknown_words_raise_before_any_cuda_use(no_native):
    img = Im(32, 32)
    regions = torch.zeros(1, 32, 32, dtype=torch.bool)
    with pytest.raises(ValueError, match='Search word zebra not found in prompt!'):
        GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16)).region_sweep(['dog', 'zebra'], img, regions, SWEEP)
    with pytest.raises(ValueError, match='Search word zebra not found in prompt!'):
        TimeHeatMaps(TOK, PROMPT, torch.zeros(3, 11, 16, 16)).region_sweep(['zebra'], img, regions, SWEEP)


# ---- empty inputs ----------------------------------------------------------------------------------------------------
def test_empty_inputs_launch_nothing(fake):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16))
    img = Im(32, 32)
    whms, ov = ghm.region_sweep([], img, torch.zeros(3, 32, 32, dtype=torch.bool), SWEEP)
    assert whms == [] and tuple(ov.intersection.shape) == (19, 3, 0) and tuple(ov.word_area.shape) == (19, 0)
    assert tuple(ov.region_area.shape) == (3,) and tuple(ov.iou().shape) == (19, 3, 0)
    whms, ov = ghm.region_sweep(['dog'], img, torch.zeros(0, 32, 32, dtype=torch.bool), [0.5, 0.6])
    assert whms == [] and tuple(ov.intersection.shape) == (2, 0, 0) and ov.region_area.numel() == 0
    word_maps, ov = TimeHeatMaps(TOK, PROMPT, torch.zeros(4, 11, 16, 16)).region_sweep(
        [], img, torch.zeros(2, 32, 32, dtype=torch.uint8), [0.1, 0.2, 0.3])
    assert tuple(ov.intersection.shape) == (4, 3, 2, 0) and tuple(ov.word_area.shape) == (4, 3, 0)
    assert tuple(word_maps.shape) == (4, 0, 16, 16)
    # the empty shapes are region_overlap's with the threshold axis
    _, one = ghm.region_overlap([], img, torch.zeros(3, 32, 32, dtype=torch.bool))
    assert tuple(one.intersection.shape) == (3, 0) and tuple(one.word_area.shape) == (0,)
    assert fake.calls == [] and fake.scratch == []
