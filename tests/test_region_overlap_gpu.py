"""Word-region overlap (GlobalHeatMap.region_overlap / GlobalHeatMapStack.region_overlap, daam_region_overlap) on the
GPU.

* With a threshold, bit for bit: intersection and word_area equal the sums of the expand_words masks over the regions,
  and iou() / ioa() equal daam_b200.evaluate.compute_iou / compute_ioa of every (mask, region) pair, over square,
  rectangular, SDXL, off-grid and down-sampled outputs with tile-edge remainders on both axes.
* Without a threshold: within rtol 1e-5 of float64 sums of the same expand_words values, and the same bits on every call.
* Edge cases: repeated words, empty and full regions, region bytes other than 0 / 1, and the word, region, map and pixel
  limits (one past each is DAAM_E_UNSUPPORTED through the C ABI).
* Stacks: time-resolved, negative and per-image histories from the synthetic pipeline in one call, row t equal to the
  per-map call; a compact long-prompt map with a word in the second chunk.
"""
from types import SimpleNamespace

import pytest
import torch

from daam_b200 import _native, trace
from daam_b200.evaluate import compute_ioa, compute_iou
from daam_b200.heatmap import GlobalHeatMap
from daam_b200.testing.synthetic import TINY_SPEC, UNetSpec, WhitespaceTokenizer, make_pipeline

pytestmark = pytest.mark.gpu
DEV = 'cuda'
TOK = WhitespaceTokenizer()
PROMPT100 = ' '.join(f'w{i}' for i in range(100))
PROMPT = 'a dog chasing a red ball on the beach'
TINY_XL = UNetSpec('tiny-xl', 128, (32, 64, 64), (1, 2, 2), (0, 1, 1), 64, mid_depth=1)


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


def rand_maps(grid, seed, n_rows=102):
    """Uniform rows: normalised maps spread over [0, 1] and absolute ones straddle the thresholds."""
    return torch.rand(n_rows, *grid, generator=torch.Generator().manual_seed(seed)).to(DEV)


def make_regions(h, w, n, seed):
    """``n`` uint8 regions ``[n, h, w]``: region 0 is empty, region 1 full, the others random rectangles and blobs, some
    marked with bytes other than 1."""
    g = torch.Generator().manual_seed(seed)
    out = torch.zeros((n, h, w), dtype=torch.uint8)
    for r in range(n):
        if r == 0:
            continue
        if r == 1:
            out[r] = 1
            continue
        y0, x0 = int(torch.randint(0, h, (1,), generator=g)), int(torch.randint(0, w, (1,), generator=g))
        y1, x1 = int(torch.randint(y0 + 1, h + 1, (1,), generator=g)), int(torch.randint(x0 + 1, w + 1, (1,), generator=g))
        mark = (1, 7, 255)[r % 3]
        if r % 2:
            out[r, y0:y1, x0:x1] = mark
        else:
            out[r] = (torch.rand(h, w, generator=g) < 0.3).to(torch.uint8) * mark
    return out.to(DEV)


def reference_sums(m, regions):
    """``(intersection [R, W], word_area [W])`` of the stack ``m`` [W, H, W] in torch, as the issue states them."""
    inter = (m[:, None] * (regions != 0)[None].float()).sum((-1, -2))
    return inter.T.contiguous(), m.sum((-1, -2))


def check_exact(ghm, words, img, regions, absolute, threshold, pairs=True):
    _, m = ghm.expand_words(words, img, absolute=absolute, threshold=threshold, to_cpu=False)
    whms, ov = ghm.region_overlap(words, img, regions, absolute=absolute, threshold=threshold, to_cpu=False)
    inter, area = reference_sums(m, regions)
    assert ov.intersection.dtype == torch.float32 and ov.intersection.is_cuda
    assert tuple(ov.intersection.shape) == (regions.shape[0], len(words)) and tuple(ov.word_area.shape) == (len(words),)
    assert torch.equal(ov.intersection, inter)
    assert torch.equal(ov.word_area, area)
    assert torch.equal(ov.region_area, (regions != 0).sum((-1, -2)).float())
    whms_e, _ = ghm.expand_words(words, img, absolute=absolute, to_cpu=False)
    for a, b in zip(whms, whms_e):
        assert torch.equal(a.heatmap, b.heatmap) and a.word == b.word
    if pairs:
        iou, ioa = ov.iou().cpu(), ov.ioa().cpu()
        for r in range(regions.shape[0]):
            rf = regions[r].float() if int(regions[r].max()) <= 1 else (regions[r] != 0).float()
            for w in range(len(words)):
                assert float(iou[r, w]) == compute_iou(m[w], rf), (r, w)
                assert float(ioa[r, w]) == compute_ioa(m[w], rf), (r, w)
    return m, ov


# (map grid, image (h, w)): SD-2.1 512^2, 768^2, SDXL 1024^2, SDXL 1216x832, off-grid 600x800 (tile-edge remainders on
# both axes), a smaller output than the map, and a non-square map over a 96x80 image
PAIRS = [((64, 64), (512, 512)), ((96, 96), (768, 768)), ((128, 128), (1024, 1024)), ((76, 52), (1216, 832)),
         ((75, 100), (600, 800)), ((96, 96), (40, 56)), ((96, 64), (96, 80))]
PAIR_IDS = [f'{g[0]}x{g[1]}-{h}x{w}' for g, (h, w) in PAIRS]


@pytest.mark.parametrize('absolute,threshold', [(False, 0.4), (False, 0.7), (True, 0.4), (True, 0.55)])
@pytest.mark.parametrize('grid,hw', PAIRS, ids=PAIR_IDS)
def test_thresholded_sums_and_scores_are_bit_exact(grid, hw, absolute, threshold):
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps(grid, 7 * grid[0] + grid[1]))
    h, w = out_size(grid, hw)
    check_exact(ghm, word_list(5), image(*hw), make_regions(h, w, 5, h + w), absolute, threshold)


@pytest.mark.parametrize('n_words,n_regions', [(8, 4), (24, 16), (3, 31), (2, 32), (4, 63)])
def test_thresholded_word_and_region_counts(n_words, n_regions):
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((76, 52), n_words))
    img = image(1216, 832)
    check_exact(ghm, word_list(n_words), img, make_regions(1216, 832, n_regions, n_regions), False, 0.4,
                pairs=n_words * n_regions <= 64)


@pytest.mark.parametrize('absolute', [False, True])
@pytest.mark.parametrize('grid,hw', PAIRS, ids=PAIR_IDS)
def test_unthresholded_sums_against_float64(grid, hw, absolute):
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps(grid, 3 * grid[0] + grid[1]))
    h, w = out_size(grid, hw)
    regions = make_regions(h, w, 6, h * w)
    words = word_list(8)
    img = image(*hw)
    _, m = ghm.expand_words(words, img, absolute=absolute, to_cpu=False)
    _, ov = ghm.region_overlap(words, img, regions, absolute=absolute, to_cpu=False)
    m64 = m.double()
    inter64 = (m64[:, None] * (regions != 0)[None].double()).sum((-1, -2)).T
    torch.testing.assert_close(ov.intersection.double(), inter64, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(ov.word_area.double(), m64.sum((-1, -2)), rtol=1e-5, atol=1e-6)
    mean64 = inter64 / (regions != 0).sum((-1, -2)).double()[:, None]
    got = ov.region_mean().double()
    keep = (regions != 0).flatten(1).any(1)
    torch.testing.assert_close(got[keep], mean64[keep], rtol=2e-5, atol=1e-6)
    assert bool((got[~keep] == 0).all())
    _, again = ghm.region_overlap(words, img, regions, absolute=absolute, to_cpu=False)
    assert torch.equal(ov.intersection.view(torch.int32), again.intersection.view(torch.int32))
    assert torch.equal(ov.word_area.view(torch.int32), again.word_area.view(torch.int32))


def test_empty_full_and_marked_regions_and_repeated_words():
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((64, 64), 1))
    img = image(512, 512)
    regions = make_regions(512, 512, 4, 9)          # empty, full, a rectangle of 7s, a blob of 1s
    words = ['w3', 'w10', 'w3']
    m, ov = check_exact(ghm, words, img, regions, False, 0.4)
    iou = ov.iou().cpu()
    assert bool((iou[0] == 0).all())                # an empty region: I = 0, so 0 / (A_w + 1e-8)
    assert torch.equal(ov.intersection[1], ov.word_area)                   # a full region holds the whole mask
    assert torch.equal(ov.intersection[:, 0], ov.intersection[:, 2])        # a repeated word repeats its column
    marked = regions.clone()
    marked[marked != 0] = 1
    _, ov1 = ghm.region_overlap(words, img, marked, threshold=0.4, to_cpu=False)
    assert torch.equal(ov1.intersection, ov.intersection)                  # any nonzero byte is inside
    _, ovb = ghm.region_overlap(words, img, regions != 0, threshold=0.4, to_cpu=False)
    assert torch.equal(ovb.intersection, ov.intersection)                  # bool regions
    _, ov2 = ghm.region_overlap(words, img, regions[2], threshold=0.4)     # one [H, W] region: an axis of 1
    assert tuple(ov2.intersection.shape) == (1, 3) and torch.equal(ov2.intersection[0], ov.intersection[2].cpu())
    assert not ov2.intersection.is_cuda and not ov2.region_area.is_cuda


def test_threshold_zero_means_no_threshold():
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((64, 64), 2))
    regions = make_regions(512, 512, 3, 1)
    _, a = ghm.region_overlap(['w1', 'w2'], image(512, 512), regions, threshold=0, to_cpu=False)
    _, b = ghm.region_overlap(['w1', 'w2'], image(512, 512), regions, to_cpu=False)
    assert torch.equal(a.intersection, b.intersection) and torch.equal(a.word_area, b.word_area)


# ---- limits through the C ABI ------------------------------------------------------------------------------------------
def _abi_call(maps, n_maps, n_rows, grid, rows_per_word, out_hw, regions_ptr, n_regions, threshold=0.4):
    n_words = len(rows_per_word)
    word_maps = torch.empty((n_maps, max(n_words, 1)) + grid, device=DEV)
    inter = torch.empty((n_maps, max(n_regions, 1), max(n_words, 1)), device=DEV)
    area = torch.empty((n_maps, max(n_words, 1)), device=DEV)
    scratch = torch.empty(_native.region_scratch_floats(n_maps, max(n_words, 1), max(n_regions, 1), *out_hw),
                          device=DEV)
    _native.region_overlap(maps.data_ptr(), n_maps, n_rows, grid, rows_per_word, out_hw[0], out_hw[1], False,
                           threshold, word_maps.data_ptr(), regions_ptr, n_regions, inter.data_ptr(), area.data_ptr(),
                           scratch.data_ptr(), torch.cuda.current_stream().cuda_stream)
    return inter, area


def _status(fn):
    with pytest.raises(_native.NativeError) as e:
        fn()
    return e.value.code, str(e.value)


def test_word_and_region_limits():
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((16, 16), 5))
    img = image(40, 72)
    regions = make_regions(72, 40, 64, 3)
    check_exact(ghm, [f'w{i}' for i in range(96)], img, regions[:63], False, 0.4, pairs=False)
    code, msg = _status(lambda: ghm.region_overlap([f'w{i}' for i in range(97)], img, regions[:2]))
    assert code == _native.E_UNSUPPORTED and '97 words > 96' in msg
    code, msg = _status(lambda: ghm.region_overlap(['w1'], img, regions))
    assert code == _native.E_UNSUPPORTED and '64 regions > 63' in msg
    long_words = [' '.join(f'w{(i + j) % 100}' for j in range(4)) for i in range(90)]    # 360 rows
    code, msg = _status(lambda: ghm.region_overlap(long_words, img, regions[:2]))
    assert code == _native.E_UNSUPPORTED and 'at most 320 rows' in msg
    maps = ghm.heat_maps
    code, _ = _status(lambda: _abi_call(maps, 1, 102, (16, 16), [[1]], (72, 40), regions.data_ptr(), 0))
    assert code == _native.E_INVALID                                        # no region
    code, _ = _status(lambda: _abi_call(maps, 1, 102, (16, 16), [[1]], (72, 40), 0, 1))
    assert code == _native.E_INVALID                                        # null regions


def test_map_limit():
    grid, out = (8, 8), (16, 16)
    maps = torch.rand(65536, 3, *grid, generator=torch.Generator().manual_seed(1)).to(DEV)
    regions = make_regions(*out, 2, 4)
    inter, area = _abi_call(maps, 65535, 3, grid, [[1], [2]], out, regions.data_ptr(), 2)
    for t in (0, 1234, 65534):
        ghm = GlobalHeatMap(TOK, 'w0', maps[t])
        _, m = ghm.expand_words(['w0', 'w0'], image(*out), threshold=0.4, to_cpu=False)
        want_i, want_a = reference_sums(m, regions)
        # word 1 reads row 2: compare word 0 (row 1) only against the one-word prompt
        assert torch.equal(inter[t, :, 0], want_i[:, 0]) and torch.equal(area[t, 0], want_a[0]), t
    code, msg = _status(lambda: _abi_call(maps, 65536, 3, grid, [[1]], out, regions.data_ptr(), 2))
    assert code == _native.E_UNSUPPORTED and '65536 maps > 65535' in msg


def test_pixel_limit():
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((64, 64), 8, n_rows=12))
    g = torch.Generator().manual_seed(2)
    regions = (torch.rand(4096, 4096, generator=g) < 0.5).to(DEV)
    whms, ov = ghm.region_overlap(['w3'], image(4096, 4096), regions, threshold=0.4, to_cpu=False)   # 2^24 pixels
    _, m = ghm.expand_words(['w3'], image(4096, 4096), threshold=0.4, to_cpu=False)
    inter, area = reference_sums(m, regions[None])
    assert torch.equal(ov.intersection, inter) and torch.equal(ov.word_area, area)
    del m
    maps = ghm.heat_maps
    wide = torch.zeros(4097 * 4096, dtype=torch.uint8, device=DEV)
    code, msg = _status(lambda: _abi_call(maps, 1, 12, (64, 64), [[1]], (4096, 4097), wide.data_ptr(), 1))
    assert code == _native.E_UNSUPPORTED and 'more than 2^24 pixels' in msg


# ---- stacks from the tracer ------------------------------------------------------------------------------------------
def check_stack(stack, words, img, regions, **kw):
    before = _native.launch_count()
    word_maps, ov = stack.region_overlap(words, img, regions, to_cpu=False, **kw)
    assert _native.launch_count() - before == 3                    # the whole stack
    n = len(stack)
    assert tuple(ov.intersection.shape) == (n, regions.shape[0], len(words)) and tuple(ov.word_area.shape) == (n, len(words))
    assert tuple(word_maps.shape[:2]) == (n, len(words))
    for t in range(n):
        whms, one = stack[t].region_overlap(words, img, regions, to_cpu=False, **kw)
        assert torch.equal(one.intersection.view(torch.int32), ov.intersection[t].view(torch.int32)), t
        assert torch.equal(one.word_area.view(torch.int32), ov.word_area[t].view(torch.int32)), t
        for i, w in enumerate(whms):
            assert torch.equal(w.heatmap, word_maps[t, i])
    per_step = ov.iou()
    assert tuple(per_step.shape) == (n, regions.shape[0], len(words))
    return ov


@pytest.mark.parametrize('spec,hw', [(TINY_SPEC, (512, 512)), (TINY_SPEC, (512, 768)), (TINY_XL, (1216, 832))],
                         ids=['512', '512x768', 'xl-1216x832'])
def test_time_resolved_history(spec, hw):
    pipe = make_pipeline(spec, dtype=torch.float16, device=DEV, seed=5)
    img = image(*hw)
    regions = make_regions(*hw, 5, 2)
    with trace(pipe, time_resolved=True, negative=True) as tc:
        pipe(PROMPT, num_inference_steps=4, generator=torch.Generator().manual_seed(3), height=hw[0], width=hw[1],
             negative_prompt='blurry grainy dark photo')
        tm = tc.compute_time_heat_maps()
        assert len(tm) == 4
        for absolute, threshold in ((False, None), (False, 0.4), (True, 0.4)):
            check_stack(tm, ['dog', 'red ball', 'beach', 'dog'], img, regions, absolute=absolute, threshold=threshold)
        neg = tc.compute_time_heat_maps(negative=True)
        check_stack(neg, ['grainy', 'dark', 'photo'], img, regions, threshold=0.4)
        with pytest.raises(ValueError, match='not found'):
            neg.region_overlap(['dog'], img, regions)
        _, ov = tm.region_overlap(['dog'], img, regions, threshold=0.4)
        assert not ov.intersection.is_cuda and tuple(ov.iou().shape) == (4, 5, 1)


def test_image_maps():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=6)
    regions = make_regions(512, 512, 3, 5)
    with trace(pipe) as tc:
        pipe(PROMPT, num_inference_steps=2, generator=torch.Generator().manual_seed(11), num_images_per_prompt=3)
        per_image = tc.compute_image_heat_maps()
        assert len(per_image) == 3
        check_stack(per_image, ['dog', 'ball', 'beach'], image(512, 512), regions, threshold=0.4)
        check_stack(per_image, ['dog', 'ball'], image(512, 512), regions)


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
        regions = make_regions(512, 512, 4, 6)
        check_exact(hm, ['dog', 'lighthouse', 'w120'], image(512, 512), regions, False, 0.4)
        check_exact(hm, ['lighthouse'], image(512, 512), regions, True, 0.3)
