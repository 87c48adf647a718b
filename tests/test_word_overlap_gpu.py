"""Word-pair overlap (GlobalHeatMap.word_overlap / relation_overlap, GlobalHeatMapStack.word_overlap /
relation_overlap, daam_word_overlap) on the GPU.

* With a threshold, bit for bit: intersection and word_area equal the torch sums of the expand_words masks, iou() /
  ioa() equal compute_iou / compute_ioa of every pair, and the intersections equal region_overlap's with the masks as
  regions, over square, rectangular, SDXL, off-grid and down-sampled outputs and at image=None on the grid itself, where
  iou() / ioa() also equal the DAAM notebook's iou / ioa of the word heat maps at t = 0.15.
* Without a threshold: within rtol 1e-5 of float64 sums of the same expand_words values, the same bits on every call,
  an exactly symmetric matrix, and at image=None, absolute=True, WordHeatMap.compute_ioa within tolerance.
* Words and limits: 1 to 96 words with a multi-token word, a repeated word and explicit word_idx; one past each limit
  is DAAM_E_UNSUPPORTED through the C ABI; guard floats past every output stay; at most three launches a call; a map
  whose tile windows do not fit in shared memory beside the pair buffers.
* Stacks from the synthetic pipeline: time-resolved, per-image, per-layer and a compact long-prompt map, row t equal to
  the per-map call. Relations: str and int endpoints, skipped words, and the notebook's per-edge loop.
"""
from types import SimpleNamespace

import pytest
import torch

from daam_b200 import _native, trace
from daam_b200.evaluate import compute_ioa, compute_iou
from daam_b200.heatmap import GlobalHeatMap
from daam_b200.testing.synthetic import TINY_SPEC, UNetSpec, WhitespaceTokenizer, make_pipeline
from tests.test_word_geometry_gpu import Case, plan

pytestmark = pytest.mark.gpu
DEV = 'cuda'
TOK = WhitespaceTokenizer()
PROMPT100 = ' '.join(f'w{i}' for i in range(100))
PROMPT = 'a dog chasing a red ball on the beach'
TINY_XL = UNetSpec('tiny-xl', 128, (32, 64, 64), (1, 2, 2), (0, 1, 1), 64, mid_depth=1)


def notebook_iou(a, b, t: float = 0.15) -> float:
    """notebooks/1-visuosyntactic-analyses.ipynb, cell 14."""
    i = ((a > t) & (b > t)).float().sum()
    u = ((a > t) | (b > t)).float().sum()
    if u < 1e-6:
        return 0.0
    else:
        return (i / u).item()


def notebook_ioa(a, b, t: float = 0.15) -> float:
    i = ((a > t) & (b > t)).float().sum()
    a = (a > t).float().sum()
    if a < 1e-6:
        return 0.0
    else:
        return (i / a).item()


def image(h, w):
    """A PIL-like image of height ``h`` and width ``w``."""
    return SimpleNamespace(size=(w, h), height=h, width=w)


def word_list(n):
    """``n`` words of PROMPT100 with a two-token word and a repeated word."""
    words = [f'w{3 * i % 100}' for i in range(n)]
    if n >= 3:
        words[1] = 'w40 w41'
        words[-1] = words[0]
    return words


def rand_maps(grid, seed, n_rows=102, scale=1.0):
    """Uniform rows: normalised maps spread over [0, 1] and absolute ones straddle the thresholds."""
    return (torch.rand(n_rows, *grid, generator=torch.Generator().manual_seed(seed)) * scale).to(DEV)


def pair_sums(m):
    """``(intersection [W, W], word_area [W])`` of the stack ``m`` [W, H, W] in torch."""
    return (m[:, None] * m[None]).sum((-1, -2)), m.sum((-1, -2))


def check_exact(ghm, words, img, absolute, threshold, pairs=True, word_idx=None):
    """word_overlap against the torch sums of the expand_words masks (``img=None``: at the grid, which ``image(*grid)``
    expands to), region_overlap with those masks as regions, and compute_iou / compute_ioa of every pair."""
    eimg = img if img is not None else image(*ghm.heat_maps.shape[-2:])
    _, m = ghm.expand_words(words, eimg, absolute=absolute, threshold=threshold, word_idx=word_idx, to_cpu=False)
    whms, ov = ghm.word_overlap(words, img, absolute=absolute, threshold=threshold, word_idx=word_idx, to_cpu=False)
    n = len(words)
    assert ov.intersection.dtype == torch.float32 and ov.intersection.is_cuda
    assert tuple(ov.intersection.shape) == (n, n) and tuple(ov.word_area.shape) == (n,)
    inter, area = pair_sums(m)
    assert torch.equal(ov.intersection, inter)
    assert torch.equal(ov.word_area, area)
    assert torch.equal(ov.intersection.view(torch.int32), ov.intersection.T.view(torch.int32))
    assert torch.equal(ov.intersection.diagonal(), ov.word_area)
    whms_e, _ = ghm.expand_words(words, image(8, 8), word_idx=word_idx, to_cpu=False)
    for a, b in zip(whms, whms_e):
        assert torch.equal(a.heatmap, b.heatmap) and a.word == b.word
    if n <= _native.MAX_REGIONS:       # an independent kernel path: the masks as the regions of region_overlap
        _, rov = ghm.region_overlap(words, eimg, m.bool(), absolute=absolute, threshold=threshold, word_idx=word_idx,
                                    to_cpu=False)
        assert torch.equal(rov.intersection, ov.intersection)        # [region b, word a]: the matrix is symmetric
    if pairs:
        iou, ioa = ov.iou().cpu(), ov.ioa().cpu()
        for a in range(n):
            for b in range(n):
                assert float(iou[a, b]) == compute_iou(m[a], m[b]), (a, b)
                assert float(ioa[a, b]) == compute_ioa(m[a], m[b]), (a, b)
    return m, ov


# (map grid, image (h, w)): SD-2.1 512^2, 768^2, SDXL 1024^2, SDXL 1216x832, off-grid 600x800 (tile-edge remainders on
# both axes), a smaller output than the map, and a non-square map over a 96x80 image
PAIRS = [((64, 64), (512, 512)), ((96, 96), (768, 768)), ((128, 128), (1024, 1024)), ((76, 52), (1216, 832)),
         ((75, 100), (600, 800)), ((96, 96), (40, 56)), ((96, 64), (96, 80))]
PAIR_IDS = [f'{g[0]}x{g[1]}-{h}x{w}' for g, (h, w) in PAIRS]


@pytest.mark.parametrize('absolute,threshold', [(False, 0.4), (True, 0.4), (True, 0.55)])
@pytest.mark.parametrize('grid,hw', PAIRS, ids=PAIR_IDS)
def test_thresholded_sums_and_scores_are_bit_exact(grid, hw, absolute, threshold):
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps(grid, 7 * grid[0] + grid[1]))
    check_exact(ghm, word_list(5), image(*hw), absolute, threshold)


# the heat-map grid itself: square, rectangular and off the 16 x 64 tile grid on both axes
GRIDS = [(64, 64), (96, 96), (76, 52), (75, 100), (37, 130)]


@pytest.mark.parametrize('grid', GRIDS, ids=[f'{h}x{w}' for h, w in GRIDS])
def test_image_none_is_the_grid_and_the_notebook(grid):
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps(grid, grid[0] + 3 * grid[1], scale=0.4))
    words = word_list(6)
    m, ov = check_exact(ghm, words, None, True, 0.15)
    assert tuple(m.shape[-2:]) == grid
    iou, ioa = ov.iou().cpu(), ov.ioa().cpu()
    maps = [ghm.compute_word_heat_map(w).heatmap for w in words]
    for a in range(len(words)):
        # at equal size the bicubic taps are (0, 1, 0, 0): m is the word heat map itself
        _, raw = ghm.expand_words([words[a]], image(*grid), absolute=True, to_cpu=False)
        assert torch.equal(raw[0], maps[a])
        for b in range(len(words)):
            assert float(iou[a, b]) == notebook_iou(maps[a], maps[b]), (a, b)
            assert float(ioa[a, b]) == notebook_ioa(maps[a], maps[b]), (a, b)


@pytest.mark.parametrize('absolute', [False, True])
@pytest.mark.parametrize('grid,hw', PAIRS + [((64, 64), None), ((75, 100), None)],
                         ids=PAIR_IDS + ['64x64-grid', '75x100-grid'])
def test_unthresholded_sums_against_float64(grid, hw, absolute):
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps(grid, 3 * grid[0] + grid[1]))
    words = word_list(8)
    img = image(*hw) if hw else None
    _, m = ghm.expand_words(words, img or image(*grid), absolute=absolute, to_cpu=False)
    _, ov = ghm.word_overlap(words, img, absolute=absolute, to_cpu=False)
    inter64, area64 = pair_sums(m.double())
    torch.testing.assert_close(ov.intersection.double(), inter64, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(ov.word_area.double(), area64, rtol=1e-5, atol=1e-6)
    assert torch.equal(ov.intersection.view(torch.int32), ov.intersection.T.view(torch.int32))
    _, again = ghm.word_overlap(words, img, absolute=absolute, to_cpu=False)
    assert torch.equal(ov.intersection.view(torch.int32), again.intersection.view(torch.int32))
    assert torch.equal(ov.word_area.view(torch.int32), again.word_area.view(torch.int32))


def test_unthresholded_grid_matches_compute_ioa():
    ghm = GlobalHeatMap(TOK, PROMPT, rand_maps((64, 64), 4, n_rows=11))
    words = ['dog', 'red ball', 'a', 'beach']
    whms, ov = ghm.word_overlap(words, absolute=True)
    ioa = ov.ioa()
    for a in range(len(words)):
        for b in range(len(words)):
            assert float(ioa[a, b]) == pytest.approx(whms[a].compute_ioa(whms[b]), rel=1e-5), (a, b)


def test_threshold_zero_means_no_threshold():
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((64, 64), 2))
    _, a = ghm.word_overlap(['w1', 'w2'], image(512, 512), threshold=0, to_cpu=False)
    _, b = ghm.word_overlap(['w1', 'w2'], image(512, 512), to_cpu=False)
    assert torch.equal(a.intersection, b.intersection) and torch.equal(a.word_area, b.word_area)


@pytest.mark.parametrize('n_words', [1, 2, 8, 24, 96])
@pytest.mark.parametrize('threshold', [0.4, None])
def test_word_counts(n_words, threshold):
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((76, 52), n_words))
    img = image(1216, 832) if n_words <= 24 else image(304, 208)
    words = word_list(n_words)
    if threshold:
        check_exact(ghm, words, img, False, threshold, pairs=n_words <= 8)
    else:
        _, m = ghm.expand_words(words, img, to_cpu=False)
        _, ov = ghm.word_overlap(words, img, to_cpu=False)
        inter64, area64 = pair_sums(m.double())
        torch.testing.assert_close(ov.intersection.double(), inter64, rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(ov.word_area.double(), area64, rtol=1e-5, atol=1e-6)
        assert torch.equal(ov.intersection.view(torch.int32), ov.intersection.T.view(torch.int32))
    if n_words >= 3:                                                  # the repeated word repeats its row
        _, ov = ghm.word_overlap(words, img, threshold=threshold, to_cpu=False)
        assert torch.equal(ov.intersection[0], ov.intersection[-1])


def test_explicit_word_idx():
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((64, 64), 12))
    check_exact(ghm, ['w3', 'x', 'w40 w41'], image(512, 512), False, 0.4, word_idx=[None, 7, None])


def pair_words_per_pass(grid, out, n_words, threshold):
    """The words_per_pass launch_tiles gives word_pair_tile_kernel (words.cu), as ``plan`` of
    tests/test_word_geometry_gpu.py states it: as many of the tile's source windows as fit in 200 KB after the pair
    table, slots and masks / values. 0: no window fits."""
    case = Case('pair', grid, out, n_words=n_words, thresholds=(threshold,))
    return plan(case, _native.device_info()['sm_count'])['by_t'][threshold]['words_per_pass']


# a square map whose tile window is the whole map (224 x 224 floats, 196 KB) over a 16 x 65 output (two tiles: the
# second's window starts at column 220), and a 10 x 5120 map (200 KB) over a 32 x 64 output (two tiles: the second's
# window starts at row 3). Next to the pair buffers of 24 words no window fits, so the kernel interpolates from the
# word maps in global memory.
GLOBAL_READS = [((224, 224), (16, 65)), ((10, 5120), (32, 64))]


@pytest.mark.parametrize('threshold', [0.4, None])
@pytest.mark.parametrize('grid,out', GLOBAL_READS, ids=['224x224-16x65', '10x5120-32x64'])
def test_windows_read_from_the_word_maps(grid, out, threshold):
    words = word_list(24)
    assert pair_words_per_pass(grid, out, len(words), threshold) == 0
    # one word beside a 196 KB window still fits (staged); beside a 200 KB one it does not
    assert pair_words_per_pass(grid, out, 1, threshold) == (1 if grid == (224, 224) else 0)
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps(grid, 9))
    img = image(out[1], out[0]) if grid[0] == grid[1] else image(*out)    # a square map keeps (size[0], size[1])
    if threshold:
        m, _ = check_exact(ghm, words, img, False, threshold, pairs=False)
        check_exact(ghm, words[:1], img, False, threshold)
    else:
        _, m = ghm.expand_words(words, img, to_cpu=False)
        _, ov = ghm.word_overlap(words, img, to_cpu=False)
        inter64, area64 = pair_sums(m.double())
        torch.testing.assert_close(ov.intersection.double(), inter64, rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(ov.word_area.double(), area64, rtol=1e-5, atol=1e-6)
        assert torch.equal(ov.intersection.view(torch.int32), ov.intersection.T.view(torch.int32))
    assert tuple(m.shape[-2:]) == out


# 96 words whose windows take several staging passes: at the 64 x 64 grid (30 words a pass with a threshold, 14
# without) and 96 x 96 down to 40 x 56 (9 and 4); without a threshold each pass is staged again for every chunk
SEVERAL_PASSES = [((64, 64), None), ((96, 96), (40, 56))]


@pytest.mark.parametrize('threshold', [0.4, None])
@pytest.mark.parametrize('grid,out', SEVERAL_PASSES, ids=['64x64-grid', '96x96-40x56'])
def test_windows_in_several_passes(grid, out, threshold):
    words = word_list(96)
    per_pass = pair_words_per_pass(grid, out or grid, len(words), threshold)
    assert 1 < per_pass < len(words) // 2
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps(grid, 11))
    img = None if out is None else image(out[1], out[0])               # a square map keeps (size[0], size[1])
    if threshold:
        m, _ = check_exact(ghm, words, img, False, threshold, pairs=False)
    else:
        _, m = ghm.expand_words(words, img or image(*grid), to_cpu=False)
        _, ov = ghm.word_overlap(words, img, to_cpu=False)
        inter64, area64 = pair_sums(m.double())
        torch.testing.assert_close(ov.intersection.double(), inter64, rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(ov.word_area.double(), area64, rtol=1e-5, atol=1e-6)
        assert torch.equal(ov.intersection.view(torch.int32), ov.intersection.T.view(torch.int32))
    assert tuple(m.shape[-2:]) == (out or grid)


# ---- limits and writes through the C ABI ------------------------------------------------------------------------------
GUARD = 64


def _abi_call(maps, n_maps, n_rows, grid, rows_per_word, out_hw, threshold=0.4):
    """daam_word_overlap with GUARD NaN floats past every output; returns the outputs and the guards."""
    n_words = max(len(rows_per_word), 1)
    word_maps = torch.empty((n_maps, n_words) + grid, device=DEV)
    inter = torch.full((n_maps * n_words * n_words + GUARD,), float('nan'), device=DEV)
    area = torch.full((n_maps * n_words + GUARD,), float('nan'), device=DEV)
    n_scratch = _native.word_overlap_scratch_floats(n_maps, n_words, *out_hw)
    scratch = torch.full((n_scratch + GUARD,), float('nan'), device=DEV)
    _native.word_overlap(maps.data_ptr(), n_maps, n_rows, grid, rows_per_word, out_hw[0], out_hw[1], False, threshold,
                         word_maps.data_ptr(), inter.data_ptr(), area.data_ptr(), scratch.data_ptr(),
                         torch.cuda.current_stream().cuda_stream)
    guards = (inter[-GUARD:], area[-GUARD:], scratch[-GUARD:])
    return (inter[:-GUARD].view(n_maps, n_words, n_words), area[:-GUARD].view(n_maps, n_words), guards)


def _status(fn):
    with pytest.raises(_native.NativeError) as e:
        fn()
    return e.value.code, str(e.value)


def test_word_and_row_limits():
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((16, 16), 5))
    img = image(40, 72)
    check_exact(ghm, [f'w{i}' for i in range(96)], img, False, 0.4, pairs=False)
    code, msg = _status(lambda: ghm.word_overlap([f'w{i}' for i in range(97)], img))
    assert code == _native.E_UNSUPPORTED and '97 words > 96' in msg
    long_words = [' '.join(f'w{(i + j) % 100}' for j in range(4)) for i in range(80)] + ['w1']    # 321 rows
    code, msg = _status(lambda: ghm.word_overlap(long_words, img))
    assert code == _native.E_UNSUPPORTED and 'at most 320 rows' in msg
    maps = ghm.heat_maps
    code, _ = _status(lambda: _abi_call(maps, 1, 102, (16, 16), [], (72, 40)))
    assert code == _native.E_INVALID                                      # no word


@pytest.mark.parametrize('n_maps,n_words,grid,out', [(1, 5, (64, 64), (600, 800)), (3, 96, (16, 16), (40, 72)),
                                                     (7, 24, (76, 52), (1216, 832))])
def test_writes_stay_within_the_outputs(n_maps, n_words, grid, out):
    maps = torch.rand(n_maps, 102, *grid, generator=torch.Generator().manual_seed(n_words)).to(DEV)
    rows = [[1 + (3 * i) % 100] for i in range(n_words)]
    for threshold in (0.4, None):
        before = _native.launch_count()
        inter, area, guards = _abi_call(maps, n_maps, 102, grid, rows, out, threshold)
        assert _native.launch_count() - before <= 3
        torch.cuda.synchronize()
        for g in guards:
            assert bool(torch.isnan(g).all())
        assert bool(torch.isfinite(inter).all()) and bool(torch.isfinite(area).all())


def test_map_limit():
    grid, out = (8, 8), (16, 16)
    maps = torch.rand(65536, 3, *grid, generator=torch.Generator().manual_seed(1)).to(DEV)
    inter, area, _ = _abi_call(maps, 65535, 3, grid, [[1], [2]], out)
    for t in (0, 1234, 65534):
        ghm = GlobalHeatMap(TOK, 'w0 w1', maps[t])
        _, m = ghm.expand_words(['w0', 'w1'], image(*out), threshold=0.4, to_cpu=False)
        want_i, want_a = pair_sums(m)
        assert torch.equal(inter[t], want_i) and torch.equal(area[t], want_a), t
    code, msg = _status(lambda: _abi_call(maps, 65536, 3, grid, [[1]], out))
    assert code == _native.E_UNSUPPORTED and '65536 maps > 65535' in msg


def test_pixel_limit():
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((64, 64), 8, n_rows=12))
    _, ov = ghm.word_overlap(['w3', 'w7'], image(4096, 4096), threshold=0.4, to_cpu=False)   # 2^24 pixels
    _, m = ghm.expand_words(['w3', 'w7'], image(4096, 4096), threshold=0.4, to_cpu=False)
    inter, area = pair_sums(m)
    assert torch.equal(ov.intersection, inter) and torch.equal(ov.word_area, area)
    del m
    code, msg = _status(lambda: _abi_call(ghm.heat_maps, 1, 12, (64, 64), [[1]], (4097, 4096)))
    assert code == _native.E_UNSUPPORTED and 'more than 2^24 pixels' in msg


# ---- stacks from the tracer ------------------------------------------------------------------------------------------
def check_stack(stack, words, img, **kw):
    before = _native.launch_count()
    word_maps, ov = stack.word_overlap(words, img, to_cpu=False, **kw)
    assert _native.launch_count() - before == 3                    # the whole stack
    n = len(stack)
    assert tuple(ov.intersection.shape) == (n, len(words), len(words)) and tuple(ov.word_area.shape) == (n, len(words))
    assert tuple(word_maps.shape[:2]) == (n, len(words))
    for t in range(n):
        whms, one = stack[t].word_overlap(words, img, to_cpu=False, **kw)
        assert torch.equal(one.intersection.view(torch.int32), ov.intersection[t].view(torch.int32)), t
        assert torch.equal(one.word_area.view(torch.int32), ov.word_area[t].view(torch.int32)), t
        for i, w in enumerate(whms):
            assert torch.equal(w.heatmap, word_maps[t, i])
    assert tuple(ov.iou().shape) == (n, len(words), len(words))
    return ov


@pytest.mark.parametrize('spec,hw', [(TINY_SPEC, (512, 512)), (TINY_SPEC, (512, 768)), (TINY_XL, (1216, 832))],
                         ids=['512', '512x768', 'xl-1216x832'])
def test_time_resolved_history(spec, hw):
    pipe = make_pipeline(spec, dtype=torch.float16, device=DEV, seed=5)
    img = image(*hw)
    with trace(pipe, time_resolved=True) as tc:
        pipe(PROMPT, num_inference_steps=4, generator=torch.Generator().manual_seed(3), height=hw[0], width=hw[1])
        tm = tc.compute_time_heat_maps()
        assert len(tm) == 4
        for absolute, threshold in ((False, None), (False, 0.4), (True, 0.15)):
            check_stack(tm, ['dog', 'red ball', 'beach', 'dog'], img, absolute=absolute, threshold=threshold)
        check_stack(tm, ['dog', 'ball', 'beach'], None, absolute=True, threshold=0.15)
        _, ov = tm.word_overlap(['dog', 'ball'], img, threshold=0.4)
        assert not ov.intersection.is_cuda and tuple(ov.iou().shape) == (4, 2, 2)


def test_image_and_layer_maps():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=6)
    with trace(pipe) as tc:
        pipe(PROMPT, num_inference_steps=2, generator=torch.Generator().manual_seed(11), num_images_per_prompt=3)
        per_image = tc.compute_image_heat_maps()
        assert len(per_image) == 3
        check_stack(per_image, ['dog', 'ball', 'beach'], image(512, 512), threshold=0.4)
        check_stack(per_image, ['dog', 'ball'], image(512, 512))
        by_layer = tc.compute_layer_heat_maps()
        assert len(by_layer) > 1
        check_stack(by_layer, ['dog', 'red ball', 'beach'], None, absolute=True, threshold=0.15)
        check_stack(by_layer, ['dog', 'ball'], image(512, 512))


def test_compact_long_prompt_map():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=3)
    words = [f'w{i}' for i in range(150)]
    words[20], words[100] = 'dog', 'lighthouse'                   # 'lighthouse' sits in the second 75-token chunk
    prompt = ' '.join(words)
    g = torch.Generator().manual_seed(5)
    c = pipe.unet.spec.cross_attention_dim
    cond, uncond = torch.randn(1, 154, c, generator=g), torch.randn(1, 154, c, generator=g)
    with trace(pipe, long_prompts=True) as tc:
        pipe(prompt_embeds=cond, negative_prompt_embeds=uncond, num_inference_steps=2,
             generator=torch.Generator().manual_seed(11))
        hm = tc.compute_global_heat_map(prompt=prompt)
        assert hm.heat_maps.shape[0] == 152
        check_exact(hm, ['dog', 'lighthouse', 'w120'], image(512, 512), False, 0.4)
        check_exact(hm, ['dog', 'lighthouse'], None, True, 0.15)


# ---- relations -------------------------------------------------------------------------------------------------------
def notebook_edges(ghm, edges, t=0.15):
    """The notebook's loop (cell 14): word maps by lookup, edges whose words are missing skipped, three scores each."""
    word_maps = {}
    for x in {x for h, d, _ in edges for x in (h, d)}:
        try:
            word_maps[x] = ghm.compute_word_heat_map(x if isinstance(x, str) else str(x),
                                                     word_idx=None if isinstance(x, str) else x).value
        except ValueError:
            pass
    stats = []
    for head, dep, rel in edges:
        if head not in word_maps or dep not in word_maps:
            continue
        a, b = word_maps[head], word_maps[dep]
        stats.append((notebook_iou(a, b, t), notebook_ioa(b, a, t), notebook_ioa(a, b, t)))
    return stats


def test_relations_against_the_notebook():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=7)
    with trace(pipe, time_resolved=True) as tc:
        pipe(PROMPT, num_inference_steps=3, generator=torch.Generator().manual_seed(2))
        ghm = tc.compute_global_heat_map()
        edges = [('chasing', 'dog', 'nsubj'), ('ball', 'red', 'amod'), ('chasing', 'ball', 'obj'),
                 ('ball', 'zebra', 'amod'), ('beach', 'the', 'det'), ('chasing', 'beach', 'obl'),
                 (5, 4, 'amod'), ('ball', 1, 'dep'), ('unicorn', 'a', 'det')]
        rel = ghm.relation_overlap(edges, absolute=True, threshold=0.15)
        assert rel.kept == [0, 1, 2, 4, 5, 6, 7] and rel.relations == [edges[i] for i in rel.kept]
        assert rel.words == ['chasing', 'dog', 'ball', 'red', 'beach', 'the']     # 5 is 'ball', 4 'red', 1 'dog'
        iou, ioa = rel.overlap.iou(), rel.overlap.ioa()
        heads, deps = [0, 2, 0, 4, 0, 2, 2], [1, 3, 2, 5, 4, 3, 1]
        assert torch.equal(rel.iou, iou[heads, deps])
        assert torch.equal(rel.iod, ioa[deps, heads]) and torch.equal(rel.ioh, ioa[heads, deps])
        want = notebook_edges(ghm, edges)
        assert len(want) == len(rel.kept)
        for e, (w_iou, w_iod, w_ioh) in enumerate(want):
            assert (float(rel.iou[e]), float(rel.iod[e]), float(rel.ioh[e])) == (w_iou, w_iod, w_ioh), e
        tm = tc.compute_time_heat_maps()
        per_step = tm.relation_overlap(edges, absolute=True, threshold=0.15)
        assert tuple(per_step.iou.shape) == (3, 7) and per_step.kept == rel.kept
        for t in range(3):
            one = tm[t].relation_overlap(edges, absolute=True, threshold=0.15)
            assert torch.equal(one.iou, per_step.iou[t]) and torch.equal(one.iod, per_step.iod[t])
            assert torch.equal(one.ioh, per_step.ioh[t])
            for e, (w_iou, w_iod, w_ioh) in enumerate(notebook_edges(tm[t], edges)):
                assert (float(one.iou[e]), float(one.iod[e]), float(one.ioh[e])) == (w_iou, w_iod, w_ioh), (t, e)
