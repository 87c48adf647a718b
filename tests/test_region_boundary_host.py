"""Boundary scores on the host, no GPU: the float64 reference of tests/boundary64.py against brute-force pairwise
distances; RegionBoundary's score rules (every empty-boundary case, P + R = 0, NaN Hausdorff and ASSD); the default
tolerance; every refusal and its order, all before the native library; the arguments GlobalHeatMap.region_boundary,
the stacks and evaluate.boundary_scores hand to daam_region_boundary / daam_mask_boundary (sizes, tolerances, scratch
bytes within the budget and at least the minimum); and the empty shapes."""
import contextlib
import math

import numpy as np
import pytest
import torch

from daam_b200 import _native, heatmap
from daam_b200.evaluate import boundary_scores
from daam_b200.heatmap import GlobalHeatMap, LayerHeatMaps, RegionBoundary, TimeHeatMaps
from daam_b200.testing.synthetic import WhitespaceTokenizer
from tests.boundary64 import as_stack, boundary, boundary64, brute_force

TOK = WhitespaceTokenizer()
PROMPT = 'a dog chasing a red ball on the beach'


class Im:
    def __init__(self, h, w):
        self.size, self.height, self.width = (w, h), h, w


# ---- the float64 reference --------------------------------------------------------------------------------------------
def _masks(seed, n, h, w):
    g = np.random.default_rng(seed)
    out = []
    for k in range(n):
        kind = k % 7
        if kind == 0:
            m = np.zeros((h, w), bool)                                    # empty
        elif kind == 1:
            m = np.ones((h, w), bool)                                     # full
        elif kind == 2:
            m = np.zeros((h, w), bool)
            m[g.integers(h), g.integers(w)] = True                        # a single pixel
        elif kind == 3:
            m = (np.add.outer(np.arange(h), np.arange(w)) % 2).astype(bool)   # checkerboard
        elif kind == 4:
            m = np.zeros((h, w), bool)                                    # touching the border
            m[:g.integers(1, h + 1), g.integers(w):] = True
        else:
            m = g.random((h, w)) < (0.2 if kind == 5 else 0.7)
        out.append(m)
    return np.stack(out)


@pytest.mark.parametrize('seed,h,w', [(0, 1, 1), (1, 1, 9), (2, 7, 1), (3, 12, 17), (4, 23, 8), (5, 40, 40)])
def test_reference_against_brute_force(seed, h, w):
    planes, regions = _masks(seed, 9, h, w), _masks(seed + 100, 8, h, w)
    tol = [0, 1, 1.5, 2.2, 7, 100]
    a, b = boundary64(planes, regions, tol), brute_force(planes, regions, tol)
    for f in ('word_boundary', 'region_boundary', 'word_hits', 'region_hits', 'max_d2'):
        np.testing.assert_array_equal(a[f], b[f], err_msg=f)
    np.testing.assert_allclose(a['sum_dist'], b['sum_dist'], rtol=1e-15, atol=0)


def test_reference_boundary_definition():
    m = np.zeros((5, 6), bool)
    m[1:4, 1:5] = True
    want = m.copy()
    want[2, 2:4] = False                                                  # the interior has all four neighbours inside
    np.testing.assert_array_equal(boundary(m), want)
    full = np.ones((3, 3), bool)
    full[1, 1] = False                                                    # every pixel but the centre touches the border
    np.testing.assert_array_equal(boundary(np.ones((3, 3), bool)), full)
    # one tolerance of 0 counts the pixels lying on the other boundary; 1.5 reaches the diagonal neighbours
    a = np.zeros((1, 4, 4), bool)
    a[0, 0, 0] = True
    r = np.zeros((1, 4, 4), bool)
    r[0, 1, 1] = True
    out = boundary64(a, r, [0, 1, 1.5])
    assert out['word_hits'][0, :, 0].tolist() == [0, 0, 1] and out['max_d2'][0, 0].tolist() == [2, 2]
    assert out['sum_dist'][0, 0].tolist() == [math.sqrt(2)] * 2


# ---- RegionBoundary ---------------------------------------------------------------------------------------------------
def _rb(word_boundary, region_boundary, word_hits, region_hits, max_d2, sum_dist, tolerances):
    return RegionBoundary(torch.tensor(word_boundary, dtype=torch.int32), torch.tensor(region_boundary, dtype=torch.int32),
                          torch.tensor(word_hits, dtype=torch.int32), torch.tensor(region_hits, dtype=torch.int32),
                          torch.tensor(max_d2, dtype=torch.int64), torch.tensor(sum_dist, dtype=torch.float64),
                          torch.tensor(tolerances, dtype=torch.float32))


def test_score_rules():
    # words: |dA| = 10, 0, 10, 0; regions: |dB| = 20, 0. T = 1, R = 2, W = 4
    b = _rb([10, 0, 10, 0], [20, 0],
            [[[5, 0, 0, 0], [0, 0, 0, 0]]], [[[8, 0, 0, 0], [0, 0, 0, 0]]],
            [[[9, 16], [-1, -1], [25, 4], [-1, -1]], [[-1, -1]] * 4],
            [[[12.0, 30.0], [0, 0], [40.0, 50.0], [0, 0]], [[0, 0]] * 4], [3.0])
    p, r, f = b.precision(), b.recall(), b.f_score()
    assert p.dtype == r.dtype == f.dtype == torch.float64 and tuple(p.shape) == (1, 2, 4)
    # both boundaries nonempty
    assert float(p[0, 0, 0]) == 0.5 and float(r[0, 0, 0]) == 0.4 and float(f[0, 0, 0]) == 2 * 0.5 * 0.4 / 0.9
    # only dA empty: P = 1, R = 0
    assert float(p[0, 0, 1]) == 1 and float(r[0, 0, 1]) == 0 and float(f[0, 0, 1]) == 0
    # only dB empty: P = 0, R = 1
    assert float(p[0, 1, 0]) == 0 and float(r[0, 1, 0]) == 1 and float(f[0, 1, 0]) == 0
    # both empty: P = R = 1
    assert float(p[0, 1, 1]) == 1 and float(r[0, 1, 1]) == 1 and float(f[0, 1, 1]) == 1
    # P + R = 0: F is 0, not NaN
    assert float(p[0, 0, 2]) == 0 and float(r[0, 0, 2]) == 0 and float(f[0, 0, 2]) == 0
    hd, assd = b.hausdorff(), b.assd()
    assert hd.dtype == assd.dtype == torch.float64 and tuple(hd.shape) == (2, 4)
    assert float(hd[0, 0]) == 4.0 and float(hd[0, 2]) == 5.0
    assert float(assd[0, 0]) == 42.0 / 30 and float(assd[0, 2]) == 90.0 / 30
    for i, j in ((0, 1), (0, 3), (1, 0), (1, 1), (1, 2), (1, 3)):
        assert math.isnan(float(hd[i, j])) and math.isnan(float(assd[i, j]))
    # a leading map axis; map(i) and cpu()
    s = RegionBoundary(*(torch.stack([getattr(b, f)] * 3) for f in ('word_boundary',)), b.region_boundary,
                       *(torch.stack([getattr(b, f)] * 3) for f in ('word_hits', 'region_hits', 'max_d2', 'sum_dist')),
                       b.tolerances)
    assert tuple(s.f_score().shape) == (3, 1, 2, 4) and tuple(s.assd().shape) == (3, 2, 4)
    assert torch.equal(s.map(2).f_score(), f) and torch.equal(s.cpu().word_hits, s.word_hits)
    assert np.array_equal(s.map(1).hausdorff().numpy(), hd.numpy(), equal_nan=True)


def test_scores_from_the_reference():
    planes, regions = _masks(7, 7, 20, 30), _masks(8, 7, 20, 30)
    tol = [1, 4]
    ref = as_stack(boundary64(planes, regions, tol), 1, 7)
    b = _rb(*(ref[f][0] if f != 'region_boundary' else ref[f] for f in
              ('word_boundary', 'region_boundary', 'word_hits', 'region_hits', 'max_d2', 'sum_dist')), tol)
    na, nb = ref['word_boundary'][0][None, None, :], ref['region_boundary'][None, :, None]
    with np.errstate(invalid='ignore', divide='ignore'):
        p = np.where(na > 0, ref['word_hits'][0] / na, 1.0)
        r = np.where(nb > 0, ref['region_hits'][0] / nb, 1.0)
    np.testing.assert_array_equal(b.precision().numpy(), p)
    np.testing.assert_array_equal(b.recall().numpy(), r)
    both = (na[0] > 0) & (nb[0] > 0)
    np.testing.assert_array_equal(np.isnan(b.hausdorff().numpy()), ~both)
    np.testing.assert_allclose(b.hausdorff().numpy()[both], np.sqrt(ref['max_d2'][0].max(-1)[both]), rtol=2.3e-16,
                               atol=0)


# ---- what reaches the native call ----------------------------------------------------------------------------------
class FakeLib:
    """Stands in for libdaam_b200.so: records the arguments of daam_region_boundary and daam_mask_boundary."""

    def __init__(self):
        self.calls = []

    def daam_region_boundary(self, *args):
        rows, begin, n_words = args[5], args[6], args[7]
        self.calls.append(dict(n_maps=args[1], n_rows=args[2], grid=(args[3], args[4]),
                               rows=[list(rows[begin[w]:begin[w + 1]]) for w in range(n_words)],
                               out=(args[8], args[9]), absolute=args[10], threshold=args[11],
                               tolerances=list(args[12][:args[13]]), n_regions=args[16], scratch_bytes=args[24],
                               n_args=len(args)))
        return 0

    def daam_mask_boundary(self, *args):
        self.calls.append(dict(n_planes=args[1], out=(args[2], args[3]), n_regions=args[5],
                               tolerances=list(args[6][:args[7]]), scratch_bytes=args[15], n_args=len(args)))
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
    whms, b = ghm.region_boundary(['dog', 'red ball'], Im(40, 40), regions, 0.4, [1, 2.5])
    call, = fake.calls
    assert call['n_args'] == 26 and call['n_maps'] == 1 and call['n_regions'] == 3
    assert call['out'] == (40, 40) and call['rows'] == [[2], [5, 6]] and call['absolute'] == 0
    assert call['threshold'] == pytest.approx(0.4) and call['tolerances'] == [1.0, 2.5]
    assert call['scratch_bytes'] == _native.boundary_scratch_bytes(3, 2, 40, 40)   # both planes in one round
    assert tuple(b.word_boundary.shape) == (2,) and b.word_boundary.dtype == torch.int32
    assert tuple(b.region_boundary.shape) == (3,) and b.region_boundary.dtype == torch.int32
    assert tuple(b.word_hits.shape) == tuple(b.region_hits.shape) == (2, 3, 2) and b.word_hits.dtype == torch.int32
    assert tuple(b.max_d2.shape) == (3, 2, 2) and b.max_d2.dtype == torch.int64
    assert tuple(b.sum_dist.shape) == (3, 2, 2) and b.sum_dist.dtype == torch.float64
    assert b.tolerances.tolist() == [1.0, 2.5] and b.tolerances.dtype == torch.float32
    assert [w.word for w in whms] == ['dog', 'red ball']
    # the default tolerance: DAVIS's ceil(0.008 * diagonal); absolute maps; a [H, W] region
    _, b = ghm.region_boundary(['dog'], Im(30, 44), torch.ones(44, 30, dtype=torch.uint8), 0.5, absolute=True)
    call = fake.calls[-1]
    assert call['absolute'] == 1 and call['out'] == (44, 30) and call['n_regions'] == 1
    assert call['tolerances'] == [1.0] and tuple(b.word_hits.shape) == (1, 1, 1)


@pytest.mark.parametrize('h,w,px', [(512, 512, 6), (768, 768, 9), (1024, 1024, 12), (1216, 832, 12), (600, 800, 8)])
def test_default_tolerance(h, w, px):
    assert heatmap._boundary_tolerances(None, h, w, 'x') == [px] == [math.ceil(0.008 * math.hypot(h, w))]


def test_stacks_are_one_call_over_every_map(fake, monkeypatch):
    tm = TimeHeatMaps(TOK, PROMPT, torch.zeros(5, 11, 16, 16))
    word_maps, b = tm.region_boundary(['dog', 'beach'], Im(32, 32), torch.zeros(4, 32, 32, dtype=torch.uint8), 0.3)
    call, = fake.calls
    assert call['n_maps'] == 5 and call['n_regions'] == 4 and call['rows'] == [[2], [9]]
    assert call['scratch_bytes'] == _native.boundary_scratch_bytes(4, 10, 32, 32)
    assert tuple(word_maps.shape) == (5, 2, 16, 16) and tuple(b.word_hits.shape) == (5, 1, 4, 2)
    assert tuple(b.max_d2.shape) == (5, 4, 2, 2) and tuple(b.f_score().shape) == (5, 1, 4, 2)
    assert tuple(b.map(3).word_hits.shape) == (1, 4, 2)
    lm = LayerHeatMaps(TOK, PROMPT, torch.zeros(2, 11, 16, 12), [3, 7], ['a', 'b'], [1, 2])
    _, b = lm.region_boundary(['ball'], Im(32, 24), torch.zeros(32, 24, dtype=torch.bool), 0.3, [2])
    assert fake.calls[-1]['n_maps'] == 2 and fake.calls[-1]['grid'] == (16, 12)
    assert tuple(b.word_hits.shape) == (2, 1, 1, 1)
    # the scratch budget caps a long stack (rounds), and the regions and one plane are the least a call gets
    monkeypatch.setattr(heatmap, 'REGION_BOUNDARY_SCRATCH_BYTES', _native.boundary_scratch_bytes(4, 3, 32, 32))
    tm.region_boundary(['dog', 'beach'], Im(32, 32), torch.zeros(4, 32, 32, dtype=torch.uint8), 0.3)
    assert fake.calls[-1]['scratch_bytes'] == _native.boundary_scratch_bytes(4, 3, 32, 32)
    monkeypatch.setattr(heatmap, 'REGION_BOUNDARY_SCRATCH_BYTES', 1)
    tm.region_boundary(['dog', 'beach'], Im(32, 32), torch.zeros(4, 32, 32, dtype=torch.uint8), 0.3)
    assert fake.calls[-1]['scratch_bytes'] == _native.boundary_scratch_bytes(4, 1, 32, 32)


def test_boundary_scores_reaches_the_mask_call(fake):
    masks = torch.zeros(3, 5, 24, 20, dtype=torch.bool)
    regions = torch.zeros(2, 24, 20, dtype=torch.uint8)
    b = boundary_scores(masks, regions, [0, 3])
    call, = fake.calls
    assert call['n_args'] == 17 and call['n_planes'] == 15 and call['out'] == (24, 20) and call['n_regions'] == 2
    assert call['tolerances'] == [0.0, 3.0] and call['scratch_bytes'] == _native.boundary_scratch_bytes(2, 15, 24, 20)
    assert tuple(b.word_boundary.shape) == (3, 5) and tuple(b.word_hits.shape) == (3, 2, 2, 5)
    assert tuple(b.max_d2.shape) == (3, 2, 5, 2) and tuple(b.region_boundary.shape) == (2,)
    b = boundary_scores(masks[0].to(torch.uint8), regions[0])
    assert fake.calls[-1]['n_planes'] == 5 and fake.calls[-1]['n_regions'] == 1
    assert fake.calls[-1]['tolerances'] == [1.0]                          # ceil(0.008 * hypot(24, 20))
    assert tuple(b.word_hits.shape) == (1, 1, 5) and tuple(b.sum_dist.shape) == (1, 5, 2)


def test_scratch_size_matches_the_header():
    assert _native.boundary_tile_rows(256) == 16 and _native.boundary_tile_rows(255) == 17
    assert _native.boundary_tile_rows(1) == 4096 and _native.boundary_tile_rows(1000) == 16
    assert _native.boundary_call_bytes(63, 1024, 1024) == 4 * 63 * 1024 * 1024
    assert _native.boundary_call_bytes(2, 3, 3) == 8 * 2 * 5
    assert _native.boundary_plane_bytes(512, 512) == 8 * 512 * 512 + 256 + 10080 * 32
    assert _native.boundary_plane_bytes(601, 801) == 16 * ((601 * 801 + 1) // 2) + 256 + 10080 * 38
    assert _native.boundary_plane_bytes(4096, 1) == 16 * 2048 + 256 + 10080
    assert _native.boundary_scratch_bytes(4, 3, 600, 800) == (_native.boundary_call_bytes(4, 600, 800)
                                                            + 3 * _native.boundary_plane_bytes(600, 800))
    assert _native.boundary_scratch_bytes(63, 1, 1024, 1024) > heatmap.REGION_BOUNDARY_SCRATCH_BYTES == 256 << 20
    assert {'daam_region_boundary', 'daam_mask_boundary'} <= set(_native.EXPORTS)
    assert _native.BOUNDARY_MAX_TOLERANCES == 16


# ---- refusals, all before the native library --------------------------------------------------------------------------
@pytest.fixture
def no_native(monkeypatch):
    def load():
        raise AssertionError('the native library was reached')
    monkeypatch.setattr(_native, 'load', load)


def test_refusals_and_their_order(fake):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 12, 20))
    img = Im(30, 44)
    good = torch.zeros(2, 30, 44, dtype=torch.bool)
    # the word first, then the regions, then the threshold, then the tolerances
    with pytest.raises(ValueError, match='Search word zebra not found in prompt!'):
        ghm.region_boundary(['zebra'], img, np.zeros((1, 30, 44), dtype=np.uint8), None, [-1])
    with pytest.raises(TypeError, match='torch.Tensor'):
        ghm.region_boundary(['dog'], img, np.zeros((1, 30, 44), dtype=np.uint8), None, [-1])
    with pytest.raises(TypeError, match='bool or uint8'):
        ghm.region_boundary(['dog'], img, torch.zeros(1, 30, 44), None, [-1])
    with pytest.raises(ValueError, match=r'\(2, 44, 30\).*\(R, 30, 44\)'):
        ghm.region_boundary(['dog'], img, torch.zeros(2, 44, 30, dtype=torch.bool), None, [-1])
    for thr in (None, 0, 0.0):
        with pytest.raises(ValueError, match='threshold must be set'):
            ghm.region_boundary(['dog'], img, good, thr, [-1])
    for thr in (float('nan'), float('inf')):
        with pytest.raises(ValueError, match='threshold must be finite'):
            ghm.region_boundary(['dog'], img, good, thr, [-1])
    for tol, text in [([], '0 tolerances'), (list(range(17)), '17 tolerances'), ([-1], 'finite and >= 0'),
                      ([float('inf')], 'finite and >= 0'), ([float('nan')], 'finite and >= 0'),
                      ([2, 1], 'strictly ascending'), ([1, 1], 'strictly ascending'),
                      ([1.0, 1.00000001], 'strictly ascending'), (['a'], 'must be numbers'), ([True], 'must be numbers'),
                      (3, 'sequence of numbers'), (torch.zeros(2, 1), '1-D real CPU tensor')]:
        with pytest.raises(ValueError, match=text):
            ghm.region_boundary(['dog'], img, good, 0.5, tol)
    assert fake.calls == []
    # accepted: 0, a CPU tensor, 16 values
    ghm.region_boundary(['dog'], img, good, 0.5, torch.tensor([0.0, 2.0]))
    ghm.region_boundary(['dog'], img, good, 0.5, list(range(16)))
    assert fake.calls[-2]['tolerances'] == [0.0, 2.0] and len(fake.calls[-1]['tolerances']) == 16


def test_boundary_scores_refusals(fake):
    regions = torch.zeros(2, 8, 8, dtype=torch.bool)
    with pytest.raises(TypeError, match='masks must be a torch.Tensor'):
        boundary_scores(np.zeros((1, 8, 8), bool), regions)
    with pytest.raises(TypeError, match='masks must be bool or uint8'):
        boundary_scores(torch.zeros(1, 8, 8), regions)
    with pytest.raises(TypeError, match='regions must be bool or uint8'):
        boundary_scores(torch.zeros(1, 8, 8, dtype=torch.bool), regions.float())
    with pytest.raises(ValueError, match=r'masks must be \[W, H'):
        boundary_scores(torch.zeros(8, 8, dtype=torch.bool), regions)
    with pytest.raises(ValueError, match='do not match'):
        boundary_scores(torch.zeros(1, 8, 9, dtype=torch.bool), regions)
    with pytest.raises(ValueError, match='64 regions > 63'):
        boundary_scores(torch.zeros(1, 8, 8, dtype=torch.bool), torch.zeros(64, 8, 8, dtype=torch.bool))
    with pytest.raises(ValueError, match='strictly ascending'):
        boundary_scores(torch.zeros(1, 8, 8, dtype=torch.bool), regions, [3, 2])
    assert fake.calls == []


def test_cpu_tensors_are_refused(monkeypatch, no_native):
    img = Im(32, 32)
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16))
    with pytest.raises(RuntimeError, match='GlobalHeatMap.region_boundary: .*CUDA tensors only'):
        ghm.region_boundary(['dog'], img, torch.zeros(1, 32, 32, dtype=torch.bool), 0.5)
    with pytest.raises(RuntimeError, match='TimeHeatMaps.region_boundary: .*CUDA tensors only'):
        TimeHeatMaps(TOK, PROMPT, torch.zeros(3, 11, 16, 16)).region_boundary(
            ['dog'], img, torch.zeros(1, 32, 32, dtype=torch.bool), 0.5)
    with pytest.raises(RuntimeError, match='boundary_scores: .*CUDA tensors only'):
        boundary_scores(torch.zeros(1, 32, 32, dtype=torch.bool), torch.zeros(1, 32, 32, dtype=torch.bool))


# ---- empty inputs ----------------------------------------------------------------------------------------------------
def test_empty_inputs_launch_nothing(fake):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16))
    img = Im(32, 32)
    whms, b = ghm.region_boundary([], img, torch.zeros(3, 32, 32, dtype=torch.bool), 0.5, [1, 2])
    assert whms == [] and tuple(b.word_hits.shape) == (2, 3, 0) and tuple(b.max_d2.shape) == (3, 0, 2)
    assert tuple(b.word_boundary.shape) == (0,) and tuple(b.region_boundary.shape) == (3,)
    assert tuple(b.f_score().shape) == (2, 3, 0) and tuple(b.assd().shape) == (3, 0)
    whms, b = ghm.region_boundary(['dog'], img, torch.zeros(0, 32, 32, dtype=torch.bool), 0.5)
    assert whms == [] and tuple(b.word_hits.shape) == (1, 0, 0) and b.region_boundary.numel() == 0
    word_maps, b = TimeHeatMaps(TOK, PROMPT, torch.zeros(4, 11, 16, 16)).region_boundary(
        [], img, torch.zeros(2, 32, 32, dtype=torch.uint8), 0.5)
    assert tuple(b.word_hits.shape) == (4, 1, 2, 0) and tuple(b.sum_dist.shape) == (4, 2, 0, 2)
    assert tuple(word_maps.shape) == (4, 0, 16, 16)
    b = boundary_scores(torch.zeros(2, 0, 32, 32, dtype=torch.bool), torch.zeros(2, 32, 32, dtype=torch.bool))
    assert tuple(b.word_hits.shape) == (2, 1, 2, 0)
    b = boundary_scores(torch.zeros(3, 32, 32, dtype=torch.bool), torch.zeros(0, 32, 32, dtype=torch.bool))
    assert tuple(b.word_hits.shape) == (1, 0, 3) and tuple(b.word_boundary.shape) == (3,)
    assert fake.calls == []
