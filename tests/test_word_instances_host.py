"""Word instances on the host, no GPU: the numpy oracle ``tests/components64.py`` against ``scipy.ndimage.label`` /
``find_objects`` on random, spiral, lattice and checkerboard masks; the refusals before anything reaches the native
library; WordInstances' helpers against numpy; the arguments and scratch that reach daam_word_instances; and the
shapes of empty inputs, which launch nothing."""
import contextlib
import ctypes

import numpy as np
import pytest
import torch

from daam_b200 import _native, heatmap
from daam_b200.heatmap import GlobalHeatMap, TimeHeatMaps, WordInstances
from daam_b200.testing.synthetic import WhitespaceTokenizer
from tests.components64 import components64, instances64, label8

TOK = WhitespaceTokenizer()
PROMPT = 'a dog chasing a red ball on the beach'     # rows: a 1 / 4, dog 2, chasing 3, red 5, ball 6, ..., beach 9


class Im:
    def __init__(self, h, w):
        self.size, self.height, self.width = (w, h), h, w


# ---- the oracle against scipy -----------------------------------------------------------------------------------------
def spiral(n):
    """A square spiral path of width 1 with gaps of 1: one component that winds through the whole plane."""
    m = np.zeros((n, n), bool)
    y, x, dy, dx = 0, 0, 0, 1
    lo_y, lo_x, hi_y, hi_x = 0, 0, n - 1, n - 1
    while lo_y <= hi_y and lo_x <= hi_x:
        m[y, x] = True
        ny, nx = y + dy, x + dx
        if not (lo_y <= ny <= hi_y and lo_x <= nx <= hi_x):
            if (dy, dx) == (0, 1):
                lo_y += 2
            elif (dy, dx) == (1, 0):
                hi_x -= 2
            elif (dy, dx) == (0, -1):
                hi_y -= 2
            else:
                lo_x += 2
            dy, dx = dx, -dy
            ny, nx = y + dy, x + dx
            if not (lo_y - 1 <= ny <= hi_y + 1 and lo_x - 1 <= nx <= hi_x + 1) or lo_y > hi_y or lo_x > hi_x:
                break
        y, x = ny, nx
    return m


def masks():
    g = np.random.default_rng(0)
    lat = np.zeros((301, 257), bool)
    lat[::2, ::2] = True
    return {'random-0.3': g.random((200, 333)) < 0.3, 'random-0.55': g.random((128, 96)) < 0.55,
            'spiral-301': spiral(301), 'spiral-1024': spiral(1024), 'lattice': lat,
            'checkerboard': np.indices((99, 130)).sum(0) % 2 == 0, 'empty': np.zeros((7, 9), bool),
            'full': np.ones((5, 3), bool), 'one-pixel': np.ones((1, 1), bool), 'row': g.random((1, 50)) < 0.5,
            'column': g.random((40, 1)) < 0.5}


@pytest.mark.parametrize('name', list(masks()))
def test_oracle_equals_scipy(name):
    ndi = pytest.importorskip('scipy.ndimage')
    m = masks()[name]
    lab, n = ndi.label(m, structure=np.ones((3, 3)))
    c = components64(m)
    assert len(c['root']) == n
    if name.startswith('spiral'):
        assert n == 1
    # scipy numbers the components in raster order of their first pixel: the oracle's root order
    ours = label8(m).ravel()
    number = np.zeros(m.size, np.int64)
    number[c['root']] = np.arange(1, n + 1)
    np.testing.assert_array_equal(np.where(ours >= 0, number[np.maximum(ours, 0)], 0).reshape(m.shape), lab)
    boxes = np.array([[s[0].start, s[1].start, s[0].stop, s[1].stop] for s in ndi.find_objects(lab)]).reshape(-1, 4)
    np.testing.assert_array_equal(c['box'], boxes)
    np.testing.assert_array_equal(c['area'], np.bincount(lab.ravel(), minlength=n + 1)[1:])
    y, x = np.indices(m.shape)
    idx = np.arange(1, n + 1)
    np.testing.assert_array_equal(c['sum_yx'][:, 0], np.round(ndi.sum_labels(y, lab, idx)).astype(np.int64))
    np.testing.assert_array_equal(c['sum_yx'][:, 1], np.round(ndi.sum_labels(x, lab, idx)).astype(np.int64))


def test_oracle_peak_ranking_and_padding():
    pre = np.array([[0.9, 0.9, 0.0, 0.7, 0.0],
                    [0.0, 0.8, 0.0, 0.0, 0.0],
                    [0.0, 0.0, 0.0, 0.6, 0.6],
                    [0.5, 0.0, 0.0, 0.6, 0.0]], np.float32)
    out = instances64(pre, 0.4, 4)
    # components: {(0,0),(0,1),(1,1)} area 3; {(0,3)} 1; {(2,3),(2,4),(3,3)} 3; {(3,0)} 1 -> area ties in raster order
    assert out['count'] == 4
    np.testing.assert_array_equal(out['area'], [3, 3, 1, 1])
    np.testing.assert_array_equal(out['box'], [[0, 0, 2, 2], [2, 3, 4, 5], [0, 3, 1, 4], [3, 0, 4, 1]])
    np.testing.assert_array_equal(out['peak'], np.float32([0.9, 0.6, 0.7, 0.5]))
    np.testing.assert_array_equal(out['peak_yx'], [[0, 0], [2, 3], [0, 3], [3, 0]])   # the first of each tie
    np.testing.assert_array_equal(out['sum_yx'], [[1, 2], [7, 10], [0, 3], [3, 0]])
    small = instances64(pre, 0.4, 6)
    assert small['area'][4:].sum() == 0 and small['box'][4:].sum() == 0 and small['peak'][4:].sum() == 0
    assert instances64(pre, 0.95, 2)['count'] == 0


# ---- refusals -----------------------------------------------------------------------------------------------------------
def no_native():
    raise AssertionError('the native library was reached')


def test_refusals_before_the_native_library(monkeypatch):
    monkeypatch.setattr(_native, 'load', no_native)
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16))
    for t in (None, 0, 0.0, False):
        with pytest.raises(ValueError, match='threshold must be set'):
            ghm.word_instances(['dog'], Im(32, 32), t)
    for k in (0, 65, -1, 1.5, True):
        with pytest.raises(ValueError, match=r'max_instances must be an int in \[1, 64\]'):
            ghm.word_instances(['dog'], Im(32, 32), 0.4, max_instances=k)
    prompt = ' '.join(f'w{i}' for i in range(100))
    with pytest.raises(ValueError, match='97 words > 96'):
        GlobalHeatMap(TOK, prompt, torch.zeros(102, 16, 16)).word_instances([f'w{i}' for i in range(97)], Im(8, 8), 0.4)
    with pytest.raises(ValueError, match='Search word zebra not found in prompt!'):
        ghm.word_instances(['dog', 'zebra'], Im(32, 32), 0.4)
    with pytest.raises(ValueError, match='Search word zebra not found in prompt!'):
        TimeHeatMaps(TOK, PROMPT, torch.zeros(3, 11, 16, 16)).word_instances(['zebra'], Im(32, 32), 0.4)
    with pytest.raises(RuntimeError, match='GlobalHeatMap.word_instances: .*CUDA tensors only'):
        ghm.word_instances(['dog'], Im(32, 32), 0.4)
    with pytest.raises(RuntimeError, match='TimeHeatMaps.word_instances: .*CUDA tensors only'):
        TimeHeatMaps(TOK, PROMPT, torch.zeros(3, 11, 16, 16)).word_instances(['dog'], Im(32, 32), 0.4)


# ---- helpers ------------------------------------------------------------------------------------------------------------
def sample(lead=()):
    g = torch.Generator().manual_seed(1)
    w, k = 3, 4
    area = torch.randint(1, 50, lead + (w, k), generator=g, dtype=torch.int32)
    area[..., 1, :] = 0                                                   # a word without instances
    area[..., 2, 3] = 0                                                   # a padded slot
    y0 = torch.randint(0, 20, lead + (w, k, 2), generator=g, dtype=torch.int32)
    box = torch.cat([y0, y0 + torch.randint(1, 20, lead + (w, k, 2), generator=g, dtype=torch.int32)], -1)
    box = torch.where(area.unsqueeze(-1) > 0, box, torch.zeros_like(box))
    sums = torch.randint(0, 10 ** 6, lead + (w, k, 2), generator=g) * (area.unsqueeze(-1) > 0)
    count = (area > 0).sum(-1).int()
    return WordInstances(count, area, box, sums, torch.rand(lead + (w, k), generator=g) * (area > 0),
                         torch.zeros(lead + (w, k, 2), dtype=torch.int32))


def np_iou(a, b):
    ih = max(0, min(a[2], b[2]) - max(a[0], b[0]))
    iw = max(0, min(a[3], b[3]) - max(a[1], b[1]))
    inter = ih * iw
    union = (a[2] - a[0]) * (a[3] - a[1]) + (b[2] - b[0]) * (b[3] - b[1]) - inter
    return inter / union if union > 0 else 0.0


@pytest.mark.parametrize('lead', [(), (2,)], ids=['one-map', 'stack'])
def test_helpers_against_numpy(lead):
    inst = sample(lead)
    c = inst.centroid()
    assert c.dtype == torch.float64 and tuple(c.shape) == lead + (3, 4, 2)
    area, sums = inst.area.numpy().astype(np.float64), inst.sum_yx.numpy().astype(np.float64)
    with np.errstate(invalid='ignore', divide='ignore'):
        ref = np.where(area[..., None] > 0, sums / area[..., None], np.nan)
    np.testing.assert_array_equal(c.numpy(), ref)                         # NaN where the slot is empty
    assert bool(torch.isnan(c[..., 1, :, :]).all())
    assert torch.equal(inst.largest_box(), inst.box[..., 0, :])
    gt = np.array([[0, 0, 10, 10], [5, 5, 30, 25], [100, 100, 101, 101]])
    iou = inst.box_iou(torch.tensor(gt))
    assert iou.dtype == torch.float64 and tuple(iou.shape) == lead + (3, 3)
    lb = inst.largest_box().reshape(-1, 3, 4).numpy()
    has = (inst.area[..., 0] > 0).reshape(-1, 3).numpy()
    ref = np.array([[[np_iou(lb[m, w], g) if has[m, w] else 0.0 for g in gt] for w in range(3)]
                    for m in range(lb.shape[0])]).reshape(lead + (3, 3))
    np.testing.assert_allclose(iou.numpy(), ref, rtol=1e-15, atol=0)
    assert bool((iou[..., 1, :] == 0).all())                              # the word without instances
    assert float(inst.box_iou([list(map(int, inst.largest_box().reshape(-1, 4)[0]))]).reshape(-1)[0]) == 1.0


# ---- what reaches the native call -------------------------------------------------------------------------------------
class FakeLib:
    """Stands in for libdaam_b200.so: records the arguments of daam_word_instances and writes count = map + word."""

    def __init__(self):
        self.calls = []

    def daam_word_instances(self, *a):
        rows, begin, n_words, n_maps = a[5], a[6], a[7], a[1]
        self.calls.append(dict(n_maps=n_maps, n_rows=a[2], grid=(a[3], a[4]), out=(a[8], a[9]), absolute=a[10],
                               threshold=a[11], k=a[12], scratch_bytes=a[21],
                               rows=[list(rows[begin[w]:begin[w + 1]]) for w in range(n_words)]))
        count = (torch.arange(n_maps)[:, None] + torch.arange(n_words)[None]).int().contiguous()
        ctypes.memmove(a[14].value, count.data_ptr(), count.numel() * 4)
        return 0


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
    whms, inst = ghm.word_instances(['dog', 'red ball'], Im(40, 48), 0.4, absolute=True, max_instances=5)
    call, = fake.calls
    plane = _native.word_instances_plane_bytes(40, 48)
    assert call['n_maps'] == 1 and call['grid'] == (12, 20) and call['out'] == (40, 48) and call['rows'] == [[2], [5, 6]] and call['k'] == 5
    assert call['absolute'] == 1 and call['threshold'] == pytest.approx(0.4) and call['scratch_bytes'] == 2 * plane
    assert [w.word for w in whms] == ['dog', 'red ball'] and inst.count.tolist() == [0, 1]
    assert tuple(inst.box.shape) == (2, 5, 4) and inst.sum_yx.dtype == torch.int64 and not inst.count.is_cuda
    GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16)).word_instances(['dog'], Im(30, 44), 0.4)
    assert fake.calls[-1]['out'] == (44, 30) and fake.calls[-1]['k'] == 16   # a square map keeps (size[0], size[1])
    # a long stack: scratch stays at the budget
    tm = TimeHeatMaps(TOK, PROMPT, torch.zeros(50, 11, 16, 16))
    _, inst = tm.word_instances(['dog', 'ball', 'beach'], Im(1024, 1024), 0.4)
    assert fake.calls[-1]['scratch_bytes'] == heatmap.WORD_INSTANCES_SCRATCH_BYTES and fake.calls[-1]['n_maps'] == 50
    assert inst.count[7].tolist() == [7, 8, 9] and tuple(inst.peak_yx.shape) == (50, 3, 16, 2)


def test_plane_bytes_match_the_header():
    # 8 bytes a pixel (value and label), 48 per 2 x 2 block (statistics and root list), the root count and min / max
    assert _native.word_instances_plane_bytes(512, 512) == 8 * 512 * 512 + 48 * 256 * 256 + 260
    assert _native.word_instances_plane_bytes(1, 1) == 8 + 48 + 260
    assert _native.word_instances_plane_bytes(601, 799) == 8 * 601 * 799 + 48 * 301 * 400 + 260
    assert 'daam_word_instances' in _native.EXPORTS and _native.WORD_INSTANCES_MAX == 64


def test_empty_inputs_launch_nothing(fake):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16))
    whms, inst = ghm.word_instances([], Im(32, 32), 0.4, max_instances=3)
    assert whms == [] and tuple(inst.count.shape) == (0,) and tuple(inst.area.shape) == (0, 3)
    assert tuple(inst.box.shape) == (0, 3, 4) and tuple(inst.sum_yx.shape) == (0, 3, 2)
    assert tuple(inst.centroid().shape) == (0, 3, 2) and tuple(inst.box_iou([[0, 0, 1, 1]]).shape) == (0, 1)
    word_maps, inst = TimeHeatMaps(TOK, PROMPT, torch.zeros(4, 11, 16, 16)).word_instances([], Im(32, 32), 0.4)
    assert tuple(inst.count.shape) == (4, 0) and tuple(word_maps.shape) == (4, 0, 16, 16)
    _, inst = TimeHeatMaps(TOK, PROMPT, torch.zeros(0, 11, 16, 16)).word_instances(['dog'], Im(32, 32), 0.4)
    assert tuple(inst.count.shape) == (0, 1) and tuple(inst.peak.shape) == (0, 1, 16)
    assert fake.calls == []
