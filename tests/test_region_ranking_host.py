"""Region ranking on the host, no GPU: the word, region and CPU-tensor refusals and their order, all before the native
library; the arguments GlobalHeatMap.region_ranking and the stacks hand to daam_region_ranking (sizes, scratch bytes
within the budget); the empty shapes; RegionRanking.auroc() and its NaN rules; and the float64 reference of
tests/ranking64.py against sklearn's roc_auc_score / average_precision_score and scipy's rankdata."""
import contextlib
import math

import numpy as np
import pytest
import torch

from daam_b200 import _native, heatmap
from daam_b200.heatmap import GlobalHeatMap, LayerHeatMaps, RegionRanking, TimeHeatMaps
from daam_b200.testing.synthetic import WhitespaceTokenizer
from tests.ranking64 import ap_bound, ranking64, ranking64_all

TOK = WhitespaceTokenizer()
PROMPT = 'a dog chasing a red ball on the beach'


class Im:
    def __init__(self, h, w):
        self.size, self.height, self.width = (w, h), h, w


# ---- RegionRanking ---------------------------------------------------------------------------------------------------
def test_auroc_and_its_nan_rules():
    n = 100
    area = torch.tensor([0, 30, 100, 1], dtype=torch.int64)               # empty, inside, full, one pixel
    u2 = torch.tensor([[[0, 0], [2100, 4200], [0, 0], [99, 198]],
                       [[0, 0], [0, 4199], [0, 0], [1, 0]]], dtype=torch.int64)   # [maps 2, R 4, W 2]
    rk = RegionRanking(u2, torch.zeros(2, 4, 2, dtype=torch.float64), area, n)
    au = rk.auroc()
    assert au.dtype == torch.float64 and tuple(au.shape) == (2, 4, 2)
    assert bool(torch.isnan(au[:, 0]).all()) and bool(torch.isnan(au[:, 2]).all())
    np.testing.assert_array_equal(au[:, 1].numpy(), np.array([[2100, 4200], [0, 4199]]) / (2 * 30 * 70))
    np.testing.assert_array_equal(au[:, 3].numpy(), np.array([[99, 198], [1, 0]]) / (2 * 1 * 99))
    assert float(au[0, 1, 0]) == 0.5 and float(au[0, 1, 1]) == 1.0 and float(au[1, 1, 0]) == 0.0
    one = rk.map(1)
    assert tuple(one.u2.shape) == (4, 2) and torch.equal(one.region_area, area) and one.n_pixels == n
    assert np.array_equal(one.auroc().numpy(), au[1].numpy(), equal_nan=True)
    c = rk.cpu()
    assert torch.equal(c.u2, u2) and c.n_pixels == n


# ---- the float64 reference --------------------------------------------------------------------------------------------
def _u2_rankdata(v, inside):
    """2 * sum of the mid-ranks of P minus n_p (n_p + 1): twice Mann-Whitney's U of P, from scipy's rankdata."""
    from scipy.stats import rankdata
    r2 = (2 * rankdata(np.asarray(v, dtype=np.float64), method='average')).astype(np.int64)   # integers
    n_p = int(inside.sum())
    return int(r2[inside].sum()) - n_p * (n_p + 1)


def _cases():
    g = np.random.default_rng(0)
    for k, (n, levels, frac) in enumerate([(500, None, 0.3), (4000, None, 0.05), (3000, 4, 0.5), (2000, 2, 0.2),
                                           (1000, 50, 0.9), (800, 1, 0.4), (64, 3, 1 / 64)]):
        v = g.random(n).astype(np.float32) if levels is None else (g.integers(0, levels, n) / 4).astype(np.float32)
        if k == 5:
            v[::2] = -0.0                                                 # -0 and +0 tie
        inside = g.random(n) < frac
        inside[0], inside[1] = True, False                                # both classes present
        yield v, inside


@pytest.mark.parametrize('case', range(7))
def test_reference_against_sklearn(case):
    metrics = pytest.importorskip('sklearn.metrics')
    v, inside = list(_cases())[case]
    u2, ap, groups = ranking64(v, inside)
    n_p, n_n = int(inside.sum()), int((~inside).sum())
    assert u2 == _u2_rankdata(v, inside)
    assert u2 / (2 * n_p * n_n) == pytest.approx(metrics.roc_auc_score(inside, v.astype(np.float64)), rel=1e-15)
    want = metrics.average_precision_score(inside, v.astype(np.float64))
    assert abs(ap - want) <= ap_bound(want, groups) + 1e-15
    assert groups == len(np.unique(v.astype(np.float64)))


def test_reference_edge_rules():
    v = np.array([0.5, 0.25, 0.25, -0.0, 0.0, 1.0], dtype=np.float32)
    u2, ap, groups = ranking64(v, np.zeros(6, dtype=bool))
    assert u2 == 0 and math.isnan(ap) and groups == 4                     # empty region; -0 and +0 one group
    u2, ap, _ = ranking64(v, np.ones(6, dtype=bool))
    assert u2 == 0 and ap == 1.0                                          # full region
    # a constant plane: u2 = n_p n_n, ap = n_p / n
    u2, ap, groups = ranking64(np.full(10, 0.3, dtype=np.float32), np.arange(10) < 3)
    assert (u2, groups) == (21, 1) and ap == pytest.approx(0.3, rel=1e-15)
    # by hand: values 3, 2, 2, 1 with P the 3 and the first 2: the pairs (3, 2) 2, (3, 1) 2, (2, 2) 1, (2, 1) 2
    u2, ap, _ = ranking64(np.array([3, 2, 2, 1], dtype=np.float32), np.array([True, True, False, False]))
    assert u2 == 7 and ap == pytest.approx(0.5 * 1 + 0.5 * (2 / 3), rel=1e-15)


def test_reference_stack_and_complement():
    g = np.random.default_rng(3)
    m = (g.integers(0, 7, (3, 12, 9)) / 7).astype(np.float32)
    regions = (g.random((4, 12, 9)) < 0.4).astype(np.uint8) * 9
    u2, ap, groups = ranking64_all(m, regions)
    u2c, _, _ = ranking64_all(m, (regions == 0).astype(np.uint8))
    n_p = (regions != 0).reshape(4, -1).sum(1)
    np.testing.assert_array_equal(u2 + u2c, (2 * n_p * (108 - n_p))[:, None].repeat(3, 1))
    assert u2.shape == ap.shape == (4, 3) and groups.shape == (3,)
    assert u2[1, 2] == ranking64(m[2], regions[1] != 0)[0]


# ---- what reaches the native call ----------------------------------------------------------------------------------
class FakeLib:
    """Stands in for libdaam_b200.so: records the arguments of daam_region_ranking."""

    def __init__(self):
        self.calls = []

    def daam_region_ranking(self, *args):
        rows, begin, n_words = args[5], args[6], args[7]
        self.calls.append(dict(n_maps=args[1], n_rows=args[2], grid=(args[3], args[4]),
                               rows=[list(rows[begin[w]:begin[w + 1]]) for w in range(n_words)],
                               out=(args[8], args[9]), absolute=args[10], n_regions=args[13],
                               scratch_bytes=args[17], n_args=len(args)))
        return 0


@pytest.fixture
def fake(monkeypatch):
    lib = FakeLib()
    monkeypatch.setattr(_native, 'load', lambda: lib)
    monkeypatch.setattr(heatmap, '_require_cuda', lambda t, what: None)
    monkeypatch.setattr(heatmap, '_stream_ptr', lambda dev: 0)
    monkeypatch.setattr(torch.cuda, 'device', lambda dev: contextlib.nullcontext())
    return lib


def test_sizes_reach_the_native_call(fake):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16))
    regions = torch.zeros(3, 40, 40, dtype=torch.bool)
    regions[1, :10] = True
    whms, rk = ghm.region_ranking(['dog', 'red ball'], Im(40, 40), regions)
    call, = fake.calls
    assert call['n_args'] == 19 and call['n_maps'] == 1 and call['n_regions'] == 3
    assert call['out'] == (40, 40) and call['rows'] == [[2], [5, 6]] and call['absolute'] == 0
    assert call['scratch_bytes'] == _native.region_ranking_scratch_bytes(2, 40, 40)   # both planes in one round
    assert tuple(rk.u2.shape) == (3, 2) and rk.u2.dtype == torch.int64
    assert tuple(rk.ap.shape) == (3, 2) and rk.ap.dtype == torch.float64
    assert rk.region_area.tolist() == [0, 400, 0] and rk.region_area.dtype == torch.int64 and rk.n_pixels == 1600
    assert [w.word for w in whms] == ['dog', 'red ball']
    _, rk = ghm.region_ranking(['dog'], Im(30, 44), torch.ones(44, 30, dtype=torch.uint8), absolute=True)
    assert fake.calls[-1]['absolute'] == 1 and fake.calls[-1]['out'] == (44, 30) and fake.calls[-1]['n_regions'] == 1
    assert tuple(rk.u2.shape) == (1, 1)


def test_stacks_are_one_call_over_every_map(fake, monkeypatch):
    tm = TimeHeatMaps(TOK, PROMPT, torch.zeros(5, 11, 16, 16))
    word_maps, rk = tm.region_ranking(['dog', 'beach'], Im(32, 32), torch.zeros(4, 32, 32, dtype=torch.uint8))
    call, = fake.calls
    assert call['n_maps'] == 5 and call['n_regions'] == 4 and call['rows'] == [[2], [9]]
    assert call['scratch_bytes'] == _native.region_ranking_scratch_bytes(10, 32, 32)
    assert tuple(word_maps.shape) == (5, 2, 16, 16) and tuple(rk.u2.shape) == (5, 4, 2)
    assert tuple(rk.auroc().shape) == (5, 4, 2)
    lm = LayerHeatMaps(TOK, PROMPT, torch.zeros(2, 11, 16, 12), [3, 7], ['a', 'b'], [1, 2])
    _, rk = lm.region_ranking(['ball'], Im(32, 24), torch.zeros(32, 24, dtype=torch.bool))
    assert fake.calls[-1]['n_maps'] == 2 and fake.calls[-1]['grid'] == (16, 12) and tuple(rk.u2.shape) == (2, 1, 1)
    # the scratch budget caps a long stack (rounds), and one plane is the least a call gets
    monkeypatch.setattr(heatmap, 'REGION_RANKING_SCRATCH_BYTES', _native.region_ranking_scratch_bytes(3, 32, 32))
    tm.region_ranking(['dog', 'beach'], Im(32, 32), torch.zeros(4, 32, 32, dtype=torch.uint8))
    assert fake.calls[-1]['scratch_bytes'] == _native.region_ranking_scratch_bytes(3, 32, 32)
    monkeypatch.setattr(heatmap, 'REGION_RANKING_SCRATCH_BYTES', 1)
    tm.region_ranking(['dog', 'beach'], Im(32, 32), torch.zeros(4, 32, 32, dtype=torch.uint8))
    assert fake.calls[-1]['scratch_bytes'] == _native.region_ranking_scratch_bytes(1, 32, 32)


def test_scratch_size_matches_the_header():
    assert _native.region_ranking_plane_bytes(1, 1) == 16 + 1024 + 1540 + 512
    assert _native.region_ranking_plane_bytes(512, 512) == 16 * 512 * 512 + 1024 * 64 + 1540 * 256 + 512
    assert _native.region_ranking_plane_bytes(1216, 832) == 16 * 1011712 + 1024 * 247 + 1540 * 988 + 512
    assert _native.region_ranking_scratch_bytes(3, 600, 800) == 8 * 480000 + 3 * _native.region_ranking_plane_bytes(
        600, 800)
    assert 'daam_region_ranking' in _native.EXPORTS
    assert heatmap.REGION_RANKING_SCRATCH_BYTES == 256 << 20


# ---- refusals, all before the native library --------------------------------------------------------------------------
@pytest.fixture
def no_native(monkeypatch):
    def load():
        raise AssertionError('the native library was reached')
    monkeypatch.setattr(_native, 'load', load)


def test_region_refusals(fake):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 12, 20))
    img = Im(30, 44)
    with pytest.raises(ValueError, match=r'\(2, 44, 30\).*\(R, 30, 44\)'):
        ghm.region_ranking(['dog'], img, torch.zeros(2, 44, 30, dtype=torch.bool))
    with pytest.raises(ValueError, match=r'\(2, 2, 30, 44\)'):
        ghm.region_ranking(['dog'], img, torch.zeros(2, 2, 30, 44, dtype=torch.bool))
    with pytest.raises(TypeError, match='bool or uint8'):
        ghm.region_ranking(['dog'], img, torch.zeros(1, 30, 44))
    with pytest.raises(TypeError, match='torch.Tensor'):
        ghm.region_ranking(['dog'], img, np.zeros((1, 30, 44), dtype=np.uint8))
    # the word is looked up before the regions are checked
    with pytest.raises(ValueError, match='Search word zebra not found in prompt!'):
        ghm.region_ranking(['zebra'], img, np.zeros((1, 30, 44), dtype=np.uint8))
    assert fake.calls == []


def test_cpu_tensors_are_refused(monkeypatch, no_native):
    img = Im(32, 32)
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16))
    with pytest.raises(RuntimeError, match='GlobalHeatMap.region_ranking: .*CUDA tensors only'):   # the CPU map
        ghm.region_ranking(['dog'], img, torch.zeros(1, 32, 32, dtype=torch.bool))
    # a device map (stood in for: the 4-d map stack passes the check) with CPU regions: the regions are refused
    real = heatmap._require_cuda
    monkeypatch.setattr(heatmap, '_require_cuda', lambda t, what: None if t.dim() == 4 else real(t, what))
    with pytest.raises(RuntimeError, match='GlobalHeatMap.region_ranking: .*CUDA tensors only'):
        ghm.region_ranking(['dog'], img, torch.zeros(1, 32, 32, dtype=torch.bool))
    with pytest.raises(RuntimeError, match='TimeHeatMaps.region_ranking: .*CUDA tensors only'):
        TimeHeatMaps(TOK, PROMPT, torch.zeros(3, 11, 16, 16)).region_ranking(
            ['dog'], img, torch.zeros(1, 32, 32, dtype=torch.bool))


def test_unknown_words_raise_before_any_cuda_use(no_native):
    img = Im(32, 32)
    regions = torch.zeros(1, 32, 32, dtype=torch.bool)
    with pytest.raises(ValueError, match='Search word zebra not found in prompt!'):
        GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16)).region_ranking(['dog', 'zebra'], img, regions)
    with pytest.raises(ValueError, match='Search word zebra not found in prompt!'):
        TimeHeatMaps(TOK, PROMPT, torch.zeros(3, 11, 16, 16)).region_ranking(['zebra'], img, regions)
    with pytest.raises(IndexError, match='out of bounds'):
        GlobalHeatMap(TOK, PROMPT, torch.zeros(4, 16, 16)).region_ranking(['beach'], img, regions)


# ---- empty inputs ----------------------------------------------------------------------------------------------------
def test_empty_inputs_launch_nothing(fake):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16))
    img = Im(32, 32)
    whms, rk = ghm.region_ranking([], img, torch.zeros(3, 32, 32, dtype=torch.bool))
    assert whms == [] and tuple(rk.u2.shape) == (3, 0) and tuple(rk.ap.shape) == (3, 0)
    assert rk.u2.dtype == torch.int64 and rk.ap.dtype == torch.float64
    assert tuple(rk.region_area.shape) == (3,) and rk.n_pixels == 1024 and tuple(rk.auroc().shape) == (3, 0)
    whms, rk = ghm.region_ranking(['dog'], img, torch.zeros(0, 32, 32, dtype=torch.bool))
    assert whms == [] and tuple(rk.u2.shape) == (0, 0) and rk.region_area.numel() == 0
    word_maps, rk = TimeHeatMaps(TOK, PROMPT, torch.zeros(4, 11, 16, 16)).region_ranking(
        [], img, torch.zeros(2, 32, 32, dtype=torch.uint8))
    assert tuple(rk.u2.shape) == (4, 2, 0) and tuple(rk.ap.shape) == (4, 2, 0)
    assert tuple(word_maps.shape) == (4, 0, 16, 16)
    assert fake.calls == []
