"""Word-region overlap on the host, no GPU: RegionOverlap's formulas against numpy on hand-built sums, the arguments
GlobalHeatMap.region_overlap and TimeHeatMaps.region_overlap hand to daam_region_overlap, the refusals (shapes, dtypes,
CPU tensors, unknown words) before anything reaches the native library, and empty inputs that launch nothing."""
import contextlib

import numpy as np
import pytest
import torch

from daam_b200 import _native, heatmap
from daam_b200.heatmap import GlobalHeatMap, RegionOverlap, TimeHeatMaps
from daam_b200.testing.synthetic import WhitespaceTokenizer

TOK = WhitespaceTokenizer()
PROMPT = 'a dog chasing a red ball on the beach'


class Im:
    def __init__(self, h, w):
        self.size, self.height, self.width = (w, h), h, w


# ---- RegionOverlap formulas ------------------------------------------------------------------------------------------
def _hand_built():
    inter = torch.tensor([[[0., 3., 5.], [2., 0., 5.]], [[1., 1., 0.], [4., 2., 7.]]])      # [maps 2, R 2, W 3]
    word_area = torch.tensor([[4., 3., 9.], [5., 6., 7.]])                                 # [maps, W]
    region_area = torch.tensor([10., 0.])                                                  # [R]; region 1 empty
    return RegionOverlap(inter, word_area, region_area)


def test_formulas_against_numpy():
    ov = _hand_built()
    i, aw, ar = ov.intersection.numpy(), ov.word_area.numpy(), ov.region_area.numpy()
    eps = np.float32(1e-8)
    iou = i / (aw[:, None, :] + ar[None, :, None] - i + eps)
    ioa = i / (aw[:, None, :] + eps)
    mean = i / (ar[None, :, None] + eps)
    assert ov.iou().dtype == torch.float32
    np.testing.assert_array_equal(ov.iou().numpy(), iou.astype(np.float32))
    np.testing.assert_array_equal(ov.ioa().numpy(), ioa.astype(np.float32))
    np.testing.assert_array_equal(ov.region_mean().numpy(), mean.astype(np.float32))
    assert float(ov.iou()[0, 0, 1]) == pytest.approx(3 / (3 + 10 - 3))
    assert float(ov.ioa()[1, 1, 2]) == pytest.approx(1.0)
    # one map: no leading axis
    one = RegionOverlap(ov.intersection[1], ov.word_area[1], ov.region_area)
    assert torch.equal(one.iou(), ov.iou()[1]) and torch.equal(one.ioa(), ov.ioa()[1])


def test_formulas_follow_compute_iou_operation_order():
    # compute_iou: intersection / (a.sum() + b.sum() - intersection + 1e-8) in fp32, with a the word mask, b the region
    a = torch.zeros(64, 64)
    a[:40, :50] = 1
    b = torch.zeros(64, 64)
    b[10:60, 5:64] = 1
    i = (a * b).sum()
    ov = RegionOverlap(i.view(1, 1), a.sum().view(1), b.sum().view(1))
    assert float(ov.iou()[0, 0]) == (i / (a.sum() + b.sum() - i + 1e-8)).item()
    assert float(ov.ioa()[0, 0]) == (i / (a.sum() + 1e-8)).item()
    empty = RegionOverlap(torch.zeros(1, 1), a.sum().view(1), torch.zeros(1))
    assert float(empty.iou()[0, 0]) == 0.0


# ---- what reaches the native call ----------------------------------------------------------------------------------
class FakeLib:
    """Stands in for libdaam_b200.so: records the arguments of daam_region_overlap."""

    def __init__(self):
        self.calls = []

    def daam_region_overlap(self, *args):
        rows, begin, n_words = args[5], args[6], args[7]
        self.calls.append(dict(n_maps=args[1], n_rows=args[2], grid=(args[3], args[4]),
                               rows=[list(rows[begin[w]:begin[w + 1]]) for w in range(n_words)],
                               out=(args[8], args[9]), absolute=args[10], use_threshold=args[11], threshold=args[12],
                               n_regions=args[15]))
        return 0


@pytest.fixture
def fake(monkeypatch):
    lib = FakeLib()
    monkeypatch.setattr(_native, 'load', lambda: lib)
    monkeypatch.setattr(heatmap, '_require_cuda', lambda t, what: None)
    monkeypatch.setattr(heatmap, '_stream_ptr', lambda dev: 0)
    monkeypatch.setattr(torch.cuda, 'device', lambda dev: contextlib.nullcontext())
    return lib


@pytest.mark.parametrize('threshold,use,value', [(None, 0, 0.0), (0, 0, 0.0), (0.4, 1, 0.4), (1, 1, 1.0)])
def test_threshold_truthiness_reaches_the_native_call(fake, threshold, use, value):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16))
    regions = torch.zeros(3, 40, 40, dtype=torch.bool)
    whms, ov = ghm.region_overlap(['dog', 'red ball'], Im(40, 40), regions, threshold=threshold)
    call, = fake.calls
    assert call['use_threshold'] == use and call['threshold'] == pytest.approx(value)
    assert call['n_maps'] == 1 and call['n_regions'] == 3 and call['out'] == (40, 40) and call['rows'] == [[2], [5, 6]]
    assert tuple(ov.intersection.shape) == (3, 2) and tuple(ov.word_area.shape) == (2,)
    assert tuple(ov.region_area.shape) == (3,) and ov.intersection.dtype == torch.float32
    assert [w.word for w in whms] == ['dog', 'red ball']


def test_rectangular_maps_word_idx_and_one_region(fake):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 12, 20))
    img = Im(30, 44)
    region = torch.ones(30, 44, dtype=torch.uint8)
    region[0, 0] = 0
    whms, ov = ghm.region_overlap(['dog', 'x'], img, region, absolute=True, word_idx=[None, 6], offset_idx=0)
    call = fake.calls[-1]
    assert call['grid'] == (12, 20) and call['out'] == (30, 44) and call['absolute'] == 1 and call['rows'] == [[2], [7]]
    assert call['n_regions'] == 1 and tuple(ov.intersection.shape) == (1, 2)
    assert float(ov.region_area[0]) == 30 * 44 - 1
    assert [w.word_idx for w in whms] == [None, 6]


def test_stack_is_one_call_over_every_map(fake):
    tm = TimeHeatMaps(TOK, PROMPT, torch.zeros(5, 11, 16, 16))
    word_maps, ov = tm.region_overlap(['dog', 'beach'], Im(32, 32), torch.zeros(4, 32, 32, dtype=torch.uint8),
                                      threshold=0.4)
    call, = fake.calls
    assert call['n_maps'] == 5 and call['n_regions'] == 4 and call['rows'] == [[2], [9]]
    assert tuple(word_maps.shape) == (5, 2, 16, 16)
    assert tuple(ov.intersection.shape) == (5, 4, 2) and tuple(ov.word_area.shape) == (5, 2)
    assert tuple(ov.iou().shape) == (5, 4, 2)


def test_scratch_size_matches_the_header():
    assert _native.region_scratch_floats(1, 1, 1, 16, 64) == 64 + 2
    assert _native.region_scratch_floats(3, 8, 4, 1216, 832) == 3 * 8 * (64 + 5 * 76 * 13)
    assert _native.region_scratch_floats(1, 2, 3, 17, 65) == 2 * (64 + 4 * 2 * 2)
    assert 'daam_region_overlap' in _native.EXPORTS and _native.MAX_REGIONS == 63


# ---- refusals and empty inputs ---------------------------------------------------------------------------------------
def test_shape_and_dtype_refusals(fake):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 12, 20))
    img = Im(30, 44)
    with pytest.raises(ValueError, match=r'\(2, 44, 30\).*\(R, 30, 44\)'):
        ghm.region_overlap(['dog'], img, torch.zeros(2, 44, 30, dtype=torch.bool))
    with pytest.raises(ValueError, match=r'\(2, 2, 30, 44\)'):
        ghm.region_overlap(['dog'], img, torch.zeros(2, 2, 30, 44, dtype=torch.bool))
    with pytest.raises(TypeError, match='bool or uint8'):
        ghm.region_overlap(['dog'], img, torch.zeros(1, 30, 44))
    with pytest.raises(TypeError, match='torch.Tensor'):
        ghm.region_overlap(['dog'], img, np.zeros((1, 30, 44), dtype=np.uint8))
    assert fake.calls == []


def test_cpu_tensors_are_refused(monkeypatch):
    def no_native():
        raise AssertionError('the native library was reached')
    monkeypatch.setattr(_native, 'load', no_native)
    img = Im(32, 32)
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16))
    with pytest.raises(RuntimeError, match='CUDA tensors only'):          # the CPU map
        ghm.region_overlap(['dog'], img, torch.zeros(1, 32, 32, dtype=torch.bool))
    # a device map (stood in for: the 4-d map stack passes the check) with CPU regions: the regions are refused
    real = heatmap._require_cuda
    monkeypatch.setattr(heatmap, '_require_cuda', lambda t, what: None if t.dim() == 4 else real(t, what))
    with pytest.raises(RuntimeError, match='GlobalHeatMap.region_overlap: .*CUDA tensors only'):
        ghm.region_overlap(['dog'], img, torch.zeros(1, 32, 32, dtype=torch.bool))


def test_unknown_words_raise_before_any_cuda_use(monkeypatch):
    def no_native():
        raise AssertionError('the native library was reached')
    monkeypatch.setattr(_native, 'load', no_native)
    img = Im(32, 32)
    regions = torch.zeros(1, 32, 32, dtype=torch.bool)
    with pytest.raises(ValueError, match='Search word zebra not found in prompt!'):
        GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16)).region_overlap(['dog', 'zebra'], img, regions)
    with pytest.raises(ValueError, match='Search word zebra not found in prompt!'):
        TimeHeatMaps(TOK, PROMPT, torch.zeros(3, 11, 16, 16)).region_overlap(['zebra'], img, regions)


def test_empty_inputs_launch_nothing(fake):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16))
    img = Im(32, 32)
    whms, ov = ghm.region_overlap([], img, torch.zeros(3, 32, 32, dtype=torch.bool))
    assert whms == [] and tuple(ov.intersection.shape) == (3, 0) and tuple(ov.word_area.shape) == (0,)
    assert tuple(ov.iou().shape) == (3, 0)
    whms, ov = ghm.region_overlap(['dog'], img, torch.zeros(0, 32, 32, dtype=torch.bool))
    assert whms == [] and ov.intersection.numel() == 0 and ov.region_area.numel() == 0
    word_maps, ov = TimeHeatMaps(TOK, PROMPT, torch.zeros(4, 11, 16, 16)).region_overlap([], img,
                                                                                        torch.zeros(2, 32, 32,
                                                                                                    dtype=torch.uint8))
    assert tuple(ov.intersection.shape) == (4, 2, 0) and tuple(word_maps.shape) == (4, 0, 16, 16)
    assert fake.calls == []
