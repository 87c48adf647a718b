"""Threshold sweeps of word-region overlap (GlobalHeatMap.region_sweep / GlobalHeatMapStack.region_sweep,
daam_region_sweep) on the GPU.

* Equality with region_overlap: for every nonzero threshold, slice k of intersection and word_area equals
  region_overlap(threshold=t_k) bit for bit, over SD-2.1, SDXL, 1216x832, off-grid 600x800 and down-sampled outputs,
  absolute and normalised maps, 1 / 8 / 24 / 96 words, 1 / 31 / 32 / 63 regions and T = 1 / 19 / 64.
* Every slice equals int64 counts of the expand_words values without threshold, m > t: 0 and negative thresholds
  (which region_overlap cannot express), and thresholds equal to pixel values (ties count only m > t).
* Counts never increase with the threshold; repeated calls give the same bits; time and layer stacks equal the
  per-map call row by row; the counts agree with the float64 pipeline of tests/words64.py except where
  threshold_unsure cannot decide a pixel.
* Limit statuses through the C ABI.
"""
import ctypes
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from daam_b200 import _native, trace
from daam_b200.heatmap import GlobalHeatMap
from daam_b200.testing.synthetic import TINY_SPEC, WhitespaceTokenizer, make_pipeline
from daam_b200.utils import compute_token_merge_indices
from tests.words64 import bound_for, threshold_unsure

pytestmark = pytest.mark.gpu
DEV = 'cuda'
TOK = WhitespaceTokenizer()
PROMPT100 = ' '.join(f'w{i}' for i in range(100))
PROMPT = 'a dog chasing a red ball on the beach'
SWEEP19 = [round(0.05 * i, 2) for i in range(1, 20)]
SWEEP64 = [-0.1 + 1.2 * i / 63 for i in range(64)]


def image(h, w):
    """A PIL-like image of height ``h`` and width ``w``."""
    return SimpleNamespace(size=(w, h), height=h, width=w)


def out_size(grid, hw):
    """The (H, W) expand_words gives a ``grid`` map over an ``hw`` image."""
    return (hw[1], hw[0]) if grid[0] == grid[1] else hw


def word_list(n):
    """``n`` words of PROMPT100 with a two-token word and a repeated word."""
    words = [f'w{3 * i % 100}' for i in range(n)]
    if n >= 3:
        words[1] = 'w40 w41'
        words[-1] = words[0]
    return words


def rand_maps(grid, seed, n_rows=102, shift=0.0):
    return (torch.rand(n_rows, *grid, generator=torch.Generator().manual_seed(seed)) + shift).to(DEV)


def make_regions(h, w, n, seed):
    """``n`` uint8 regions ``[n, h, w]``: region 0 full, then random rectangles and blobs, some marked with bytes other
    than 1, and an empty one when there are at least three."""
    g = torch.Generator().manual_seed(seed)
    out = torch.zeros((n, h, w), dtype=torch.uint8)
    out[0] = 1
    for r in range(1, n):
        if r == 2:
            continue
        y0, x0 = int(torch.randint(0, h, (1,), generator=g)), int(torch.randint(0, w, (1,), generator=g))
        y1, x1 = int(torch.randint(y0 + 1, h + 1, (1,), generator=g)), int(torch.randint(x0 + 1, w + 1, (1,), generator=g))
        mark = (1, 7, 255)[r % 3]
        if r % 2:
            out[r, y0:y1, x0:x1] = mark
        else:
            out[r] = (torch.rand(h, w, generator=g) < 0.3).to(torch.uint8) * mark
    return out.to(DEV)


def fp32s(xs):
    return [float(np.float32(x)) for x in xs]


def counts_of(m, regions, t):
    """int64 ``(intersection [R, W], word_area [W])`` of ``m > t`` for the stack ``m`` [W, H, W'] in torch."""
    mask = (m > t).flatten(1).double()                       # 0 / 1, exact in float64
    inside = (regions != 0).flatten(1).double()
    return (inside @ mask.T).long(), mask.sum(1).long()


def check_sweep(ghm, words, img, regions, taus, absolute, against_overlap=True):
    """The sweep against int64 counts of expand_words' values for every threshold, and against region_overlap for
    every nonzero one; returns the overlap."""
    _, ov = ghm.region_sweep(words, img, regions, taus, absolute=absolute, to_cpu=False)
    n_thr, n_reg, n_words = len(taus), regions.shape[0], len(words)
    assert tuple(ov.intersection.shape) == (n_thr, n_reg, n_words) and tuple(ov.word_area.shape) == (n_thr, n_words)
    assert ov.intersection.dtype == torch.float32 and ov.intersection.is_cuda
    assert torch.equal(ov.region_area, (regions != 0).sum((-1, -2)).float())
    _, m = ghm.expand_words(words, img, absolute=absolute, to_cpu=False)
    for k, t in enumerate(fp32s(taus)):
        inter, area = counts_of(m, regions, t)
        assert torch.equal(ov.intersection[k].long(), inter), (k, t)
        assert torch.equal(ov.word_area[k].long(), area), (k, t)
        assert bool((ov.intersection[k] == ov.intersection[k].round()).all())
        if t and against_overlap:
            _, one = ghm.region_overlap(words, img, regions, absolute=absolute, threshold=t, to_cpu=False)
            assert torch.equal(ov.intersection[k].view(torch.int32), one.intersection.view(torch.int32)), (k, t)
            assert torch.equal(ov.word_area[k].view(torch.int32), one.word_area.view(torch.int32)), (k, t)
    # counts never increase with the threshold
    assert bool((ov.intersection[1:] <= ov.intersection[:-1]).all())
    assert bool((ov.word_area[1:] <= ov.word_area[:-1]).all())
    assert bool((ov.intersection <= ov.word_area[:, None]).all())
    return ov


# (map grid, image (h, w)): SD-2.1 512^2, SDXL 1024^2, SDXL 1216x832, off-grid 600x800 (tile-edge remainders on both
# axes), and an output smaller than the map
PAIRS = [((64, 64), (512, 512)), ((128, 128), (1024, 1024)), ((76, 52), (1216, 832)), ((75, 100), (600, 800)),
         ((96, 96), (40, 56))]
PAIR_IDS = [f'{g[0]}x{g[1]}-{h}x{w}' for g, (h, w) in PAIRS]


@pytest.mark.parametrize('absolute', [False, True], ids=['normalised', 'absolute'])
@pytest.mark.parametrize('grid,hw', PAIRS, ids=PAIR_IDS)
def test_slices_equal_region_overlap(grid, hw, absolute):
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps(grid, 5 * grid[0] + grid[1]))
    h, w = out_size(grid, hw)
    check_sweep(ghm, word_list(8), image(*hw), make_regions(h, w, 5, h + w), SWEEP19, absolute)


@pytest.mark.parametrize('n_words,n_regions,n_thr', [(1, 1, 1), (8, 31, 19), (24, 32, 64), (96, 63, 64)])
def test_word_region_and_threshold_counts(n_words, n_regions, n_thr):
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((76, 52), n_words + n_regions))
    taus = {1: [0.4], 19: SWEEP19, 64: SWEEP64}[n_thr]
    check_sweep(ghm, word_list(n_words), image(1216, 832), make_regions(1216, 832, n_regions, n_regions), taus, False)


def test_literal_zero_and_negative_thresholds():
    # absolute maps that straddle 0: 0 and negative thresholds are thresholds, m > t, not "no threshold"
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((64, 64), 11, shift=-0.5))
    img, regions, words = image(512, 512), make_regions(512, 512, 4, 3), word_list(6)
    taus = [-0.6, -0.25, -1e-3, 0.0, 1e-3, 0.25]
    ov = check_sweep(ghm, words, img, regions, taus, absolute=True)
    _, m = ghm.expand_words(words, img, absolute=True, to_cpu=False)
    assert 0 < int(ov.word_area[3].sum()) < m.numel()                     # t = 0 counts m > 0 only
    assert int(ov.word_area[0].sum()) != int(ov.word_area[3].sum())
    # normalised maps: the min of every word is exactly 0, so t = 0 leaves it out
    ov = check_sweep(ghm, words, img, regions, [-1.0, 0.0], absolute=False)
    assert bool((ov.word_area[0] == 512 * 512).all()) and bool((ov.word_area[1] < ov.word_area[0]).all())


@pytest.mark.parametrize('absolute', [False, True], ids=['normalised', 'absolute'])
def test_ties_count_only_values_above(absolute):
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((76, 52), 4))
    img, regions, words = image(1216, 832), make_regions(1216, 832, 6, 8), word_list(5)
    _, m = ghm.expand_words(words, img, absolute=absolute, to_cpu=False)
    g = torch.Generator().manual_seed(1)
    picks = m[0].flatten()[torch.randint(0, m[0].numel(), (200,), generator=g).to(DEV)]
    taus = sorted(set(picks.cpu().tolist()))[::4][:30]                   # exact fp32 pixel values of word 0
    ov = check_sweep(ghm, words, img, regions, taus, absolute)
    for k, t in enumerate(taus):
        ties = int((m[0] == t).sum())
        assert ties > 0
        assert int(ov.word_area[k, 0]) == int((m[0] > t).sum()) == int((m[0] >= t).sum()) - ties


def test_repeated_calls_give_the_same_bits():
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((128, 128), 2))
    img, regions, words = image(1024, 1024), make_regions(1024, 1024, 16, 4), word_list(24)
    _, a = ghm.region_sweep(words, img, regions, SWEEP64, to_cpu=False)
    for _ in range(3):
        _, b = ghm.region_sweep(words, img, regions, SWEEP64, to_cpu=False)
        assert torch.equal(a.intersection.view(torch.int32), b.intersection.view(torch.int32))
        assert torch.equal(a.word_area.view(torch.int32), b.word_area.view(torch.int32))
    before = _native.launch_count()
    _, c = ghm.region_sweep(words, img, regions, SWEEP19)                # to the host by default
    assert _native.launch_count() - before == 3
    assert not c.intersection.is_cuda and tuple(c.intersection.shape) == (19, 16, 24)


@pytest.mark.parametrize('absolute', [False, True], ids=['normalised', 'absolute'])
@pytest.mark.parametrize('grid,hw', [((64, 64), (512, 512)), ((75, 100), (600, 800)), ((96, 96), (40, 56))],
                         ids=['64-512', '75x100-600x800', '96-40x56'])
def test_counts_against_float64(grid, hw, absolute):
    maps = rand_maps(grid, 17 + grid[1])
    ghm = GlobalHeatMap(TOK, PROMPT100, maps)
    h, w = out_size(grid, hw)
    words, regions = word_list(6), make_regions(h, w, 5, 7)
    rows = [compute_token_merge_indices(TOK, PROMPT100, word)[0] for word in words]
    exp, bound = bound_for(maps, rows, (h, w), absolute)
    _, ov = ghm.region_sweep(words, image(*hw), regions, SWEEP19, absolute=absolute, to_cpu=False)
    inside = (regions != 0)
    for k, t in enumerate(fp32s(SWEEP19)):
        unsure = threshold_unsure(exp.pre, bound, t)                      # [W, H, W']
        sure_in = (exp.pre > t) & ~unsure
        assert int(unsure.sum()) <= 5e-3 * unsure.numel() + 4 * len(words), (k, t)
        lo_a, n_a = sure_in.flatten(1).sum(1), unsure.flatten(1).sum(1)
        got_a = ov.word_area[k].long()
        assert bool(((lo_a <= got_a) & (got_a <= lo_a + n_a)).all()), (k, t)
        lo_i = (inside[:, None] & sure_in[None]).flatten(2).sum(2)        # [R, W]
        n_i = (inside[:, None] & unsure[None]).flatten(2).sum(2)
        got_i = ov.intersection[k].long()
        assert bool(((lo_i <= got_i) & (got_i <= lo_i + n_i)).all()), (k, t)


# ---- stacks from the tracer ------------------------------------------------------------------------------------------
def check_stack(stack, words, img, regions, taus, **kw):
    before = _native.launch_count()
    word_maps, ov = stack.region_sweep(words, img, regions, taus, to_cpu=False, **kw)
    assert _native.launch_count() - before == 3                    # the whole stack
    n = len(stack)
    assert tuple(ov.intersection.shape) == (n, len(taus), regions.shape[0], len(words))
    assert tuple(ov.word_area.shape) == (n, len(taus), len(words)) and tuple(word_maps.shape[:2]) == (n, len(words))
    for t in range(n):
        whms, one = stack[t].region_sweep(words, img, regions, taus, to_cpu=False, **kw)
        assert torch.equal(one.intersection.view(torch.int32), ov.intersection[t].view(torch.int32)), t
        assert torch.equal(one.word_area.view(torch.int32), ov.word_area[t].view(torch.int32)), t
        for i, w in enumerate(whms):
            assert torch.equal(w.heatmap, word_maps[t, i])
    assert tuple(ov.iou().shape) == (n, len(taus), regions.shape[0], len(words))
    return ov


def test_time_and_layer_stacks():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=5)
    img = image(512, 512)
    regions = make_regions(512, 512, 5, 2)
    words = ['dog', 'red ball', 'beach', 'dog']
    with trace(pipe, time_resolved=True) as tc:
        pipe(PROMPT, num_inference_steps=4, generator=torch.Generator().manual_seed(3))
        tm = tc.compute_time_heat_maps()
        assert len(tm) == 4
        check_stack(tm, words, img, regions, SWEEP19)
        check_stack(tm, words, img, regions, [-0.5, 0.0, 0.5], absolute=True)
        layers = tc.compute_layer_heat_maps()
        assert len(layers) > 1
        check_stack(layers, words, img, regions, SWEEP64)
        # the single-map call of a stack row is the sweep of that map against region_overlap too
        check_sweep(tm[2], words, img, regions, [0.3, 0.6], False)


# ---- limits through the C ABI ------------------------------------------------------------------------------------------
def _abi_call(maps, grid, out_hw, regions_ptr, n_regions, taus, n_thr=None):
    n_thr = len(taus) if n_thr is None else n_thr
    word_maps = torch.empty((1, 1) + grid, device=DEV)
    inter = torch.empty((1, max(n_thr, 1), max(n_regions, 1), 1), device=DEV)
    area = torch.empty((1, max(n_thr, 1), 1), device=DEV)
    scratch = torch.empty(_native.region_sweep_scratch_floats(1, 1, max(n_regions, 1), max(n_thr, 1), *out_hw),
                          device=DEV)
    arr = (ctypes.c_float * max(len(taus), 1))(*taus)
    rows, begin = (ctypes.c_int32 * 1)(1), (ctypes.c_int32 * 2)(0, 1)
    rc = _native.load().daam_region_sweep(ctypes.c_void_p(maps.data_ptr()), 1, maps.shape[0], grid[0], grid[1], rows,
                                          begin, 1, out_hw[0], out_hw[1], 0, arr, n_thr,
                                          ctypes.c_void_p(word_maps.data_ptr()), ctypes.c_void_p(regions_ptr),
                                          n_regions, ctypes.c_void_p(inter.data_ptr()),
                                          ctypes.c_void_p(area.data_ptr()), ctypes.c_void_p(scratch.data_ptr()),
                                          ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    msg = _native.load().daam_last_error().decode() if rc else ''
    return rc, msg, inter, area


def test_limit_statuses():
    grid, out = (16, 16), (72, 40)
    maps = rand_maps(grid, 5)
    regions = make_regions(*out, 64, 3)
    rc, _, inter, area = _abi_call(maps, grid, out, regions.data_ptr(), 63, fp32s(SWEEP64))
    assert rc == 0 and bool((inter[0, 1:] <= inter[0, :-1]).all()) and bool((inter[0] <= area[0, :, None]).all())
    rc, msg, *_ = _abi_call(maps, grid, out, regions.data_ptr(), 1, [i / 65 for i in range(65)])
    assert rc == _native.E_UNSUPPORTED and '65 thresholds > 64' in msg
    rc, msg, *_ = _abi_call(maps, grid, out, regions.data_ptr(), 64, [0.4])
    assert rc == _native.E_UNSUPPORTED and '64 regions > 63' in msg
    rc, msg, *_ = _abi_call(maps, grid, out, regions.data_ptr(), 1, [0.4, 0.2])
    assert rc == _native.E_INVALID and 'strictly ascending' in msg
    rc, msg, *_ = _abi_call(maps, grid, out, regions.data_ptr(), 1, [0.4, 0.4])
    assert rc == _native.E_INVALID and 'strictly ascending' in msg
    for bad in (float('nan'), float('inf'), float('-inf')):
        rc, msg, *_ = _abi_call(maps, grid, out, regions.data_ptr(), 1, [0.1, bad])
        assert rc == _native.E_INVALID and 'not finite' in msg, bad
    rc, _, *_ = _abi_call(maps, grid, out, regions.data_ptr(), 1, [0.4], n_thr=0)
    assert rc == _native.E_INVALID
    rc, _, *_ = _abi_call(maps, grid, out, 0, 1, [0.4])
    assert rc == _native.E_INVALID                                          # null regions
    wide = torch.zeros(4097 * 4096, dtype=torch.uint8, device=DEV)
    rc, msg, *_ = _abi_call(maps, grid, (4096, 4097), wide.data_ptr(), 1, [0.4])
    assert rc == _native.E_UNSUPPORTED and 'more than 2^24 pixels' in msg
    ghm = GlobalHeatMap(TOK, PROMPT100, maps)
    with pytest.raises(_native.NativeError, match='97 words > 96'):
        ghm.region_sweep([f'w{i}' for i in range(97)], image(40, 72), regions[:2], [0.4])


def test_pixel_limit():
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((64, 64), 8, n_rows=12))
    g = torch.Generator().manual_seed(2)
    regions = (torch.rand(4096, 4096, generator=g) < 0.5).to(DEV)
    taus = [0.2, 0.4, 0.8]
    _, ov = ghm.region_sweep(['w3'], image(4096, 4096), regions, taus, to_cpu=False)   # 2^24 pixels
    for k, t in enumerate(taus):
        _, one = ghm.region_overlap(['w3'], image(4096, 4096), regions, threshold=t, to_cpu=False)
        assert torch.equal(ov.intersection[k], one.intersection) and torch.equal(ov.word_area[k], one.word_area)
