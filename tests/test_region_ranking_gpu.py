"""Region ranking scores (GlobalHeatMap.region_ranking / GlobalHeatMapStack.region_ranking, daam_region_ranking) on
the GPU, against tests/ranking64.py over the very values expand_words(..., to_cpu=False) returns.

* u2 equals the float64 reference's int64 counts exactly; ap is within ap_bound: 2 (G + 3) 2^-53 ap for a plane of G
  tie groups (both sides add G positive terms, each rounded at most three times).
* SD-2.1 512^2, SDXL 1024^2, 1216x832 and off-grid 600x800 outputs, normalised and absolute maps; 1 / 8 / 96 words
  and 1 / 16 / 63 regions.
* Empty regions give NaN ap and AUROC, full regions NaN AUROC and ap 1; a constant word map gives u2 = n_p n_n and
  ap = n_p / (H W); absolute maps with large tied areas (exact zeros, -0 and +0 among them).
* u2(R) + u2(not R) = 2 n_p n_n exactly; time and layer stacks equal the per-map calls bit for bit; a scratch that
  forces several rounds gives the same bits as one round; repeated calls give the same bits.
* The C ABI's limit and invalid statuses.
"""
import ctypes
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from daam_b200 import _native, heatmap, trace
from daam_b200.heatmap import GlobalHeatMap
from daam_b200.testing.synthetic import TINY_SPEC, WhitespaceTokenizer, make_pipeline
from tests.ranking64 import ap_bound, ranking64_all

pytestmark = pytest.mark.gpu
DEV = 'cuda'
TOK = WhitespaceTokenizer()
PROMPT100 = ' '.join(f'w{i}' for i in range(100))
PROMPT = 'a dog chasing a red ball on the beach'


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
    return torch.rand(n_rows, *grid, generator=torch.Generator().manual_seed(seed)).to(DEV)


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


def check_ranking(ghm, words, img, regions, absolute):
    """The ranking against ranking64 of expand_words' values; returns (ranking, u2 reference, groups)."""
    _, rk = ghm.region_ranking(words, img, regions, absolute=absolute, to_cpu=False)
    n_reg, n_words = regions.shape[0], len(words)
    assert tuple(rk.u2.shape) == (n_reg, n_words) and rk.u2.dtype == torch.int64 and rk.u2.is_cuda
    assert tuple(rk.ap.shape) == (n_reg, n_words) and rk.ap.dtype == torch.float64
    area = (regions != 0).sum((-1, -2))
    assert torch.equal(rk.region_area, area) and rk.n_pixels == regions.shape[1] * regions.shape[2]
    _, m = ghm.expand_words(words, img, absolute=absolute, to_cpu=False)
    u2, ap, groups = ranking64_all(m.cpu().numpy(), regions.cpu().numpy())
    np.testing.assert_array_equal(rk.u2.cpu().numpy(), u2)
    got = rk.ap.cpu().numpy()
    nan = np.isnan(ap)
    np.testing.assert_array_equal(np.isnan(got), nan)
    assert bool((nan == (area == 0).cpu().numpy()[:, None]).all())            # NaN exactly for empty regions
    err = np.abs(got - ap)[~nan]
    assert bool((err <= np.broadcast_to(ap_bound(ap, groups[None]), ap.shape)[~nan]).all()), float(err.max())
    # auroc: u2 / (2 n_p n_n), NaN for empty and full regions
    n_p = area.double().cpu().numpy()[:, None]
    n_n = rk.n_pixels - n_p
    with np.errstate(invalid='ignore', divide='ignore'):
        want = np.where(n_p * n_n > 0, u2 / (2 * n_p * n_n), np.nan)
    np.testing.assert_array_equal(rk.auroc().cpu().numpy(), want)
    return rk, u2, groups


# (map grid, image (h, w)): SD-2.1 512^2, SDXL 1024^2, SDXL 1216x832, off-grid 600x800 (tile-edge remainders on both
# axes)
PAIRS = [((64, 64), (512, 512)), ((128, 128), (1024, 1024)), ((76, 52), (1216, 832)), ((75, 100), (600, 800))]
PAIR_IDS = [f'{g[0]}x{g[1]}-{h}x{w}' for g, (h, w) in PAIRS]


@pytest.mark.parametrize('absolute', [False, True], ids=['normalised', 'absolute'])
@pytest.mark.parametrize('grid,hw', PAIRS, ids=PAIR_IDS)
def test_sizes_against_float64(grid, hw, absolute):
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps(grid, 5 * grid[0] + grid[1]))
    h, w = out_size(grid, hw)
    rk, _, _ = check_ranking(ghm, word_list(8), image(*hw), make_regions(h, w, 5, h + w), absolute)
    full = rk.ap[0].cpu()                                                 # region 0 is the whole image
    assert bool((full == 1).all()) and bool(torch.isnan(rk.auroc()[0]).all())
    assert bool(torch.isnan(rk.ap[2]).all()) and bool(torch.isnan(rk.auroc()[2]).all())   # region 2 is empty


@pytest.mark.parametrize('n_words,n_regions,grid,hw', [(1, 1, (64, 64), (512, 512)), (8, 16, (64, 64), (512, 512)),
                                                       (1, 63, (40, 30), (320, 240)), (96, 1, (40, 30), (320, 240)),
                                                       (96, 63, (24, 20), (150, 130))])
def test_word_and_region_counts(n_words, n_regions, grid, hw):
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps(grid, n_words + n_regions))
    h, w = out_size(grid, hw)
    check_ranking(ghm, word_list(n_words), image(*hw), make_regions(h, w, n_regions, n_regions), False)


@pytest.mark.parametrize('absolute', [False, True], ids=['normalised', 'absolute'])
def test_constant_map(absolute):
    # every row 0: v is 0 or -0 at every pixel (the bicubic weights carry their signs), so is m -- one tie group
    ghm = GlobalHeatMap(TOK, PROMPT100, torch.zeros((102, 64, 64), device=DEV))
    regions = make_regions(512, 512, 6, 9)
    rk, _, groups = check_ranking(ghm, word_list(3), image(512, 512), regions, absolute)
    assert bool((torch.as_tensor(groups) == 1).all())
    n_p = (regions != 0).sum((-1, -2))
    n = 512 * 512
    assert torch.equal(rk.u2, (n_p * (n - n_p))[:, None].expand(-1, 3))
    au = rk.auroc()
    inner = (n_p > 0) & (n_p < n)
    assert bool((au[inner] == 0.5).all())
    want = n_p.double() / n
    # one group: ap = (n_p * n_p / n) / n_p, two roundings away from n_p / n
    assert torch.allclose(rk.ap[n_p > 0], want[n_p > 0][:, None].expand(-1, 3), rtol=4.5e-16, atol=0)


def test_absolute_maps_with_large_tied_areas():
    # zero rows over most of the map: the bicubic values there are exact zeros (some -0), a few large tie groups
    maps = rand_maps((64, 64), 3)
    maps[:, :40] = 0.0
    maps[:, :, 50:] = 0.0
    maps[:, 45:48, 10:20] = -0.0
    ghm = GlobalHeatMap(TOK, PROMPT100, maps)
    regions = make_regions(512, 512, 8, 5)
    _, m = ghm.expand_words(word_list(4), image(512, 512), absolute=True, to_cpu=False)
    assert int((m == 0).sum()) > m.numel() // 2
    check_ranking(ghm, word_list(4), image(512, 512), regions, True)
    # thresholded-looking maps, from the normalised values rounded to a few levels: many ties in every region
    check_ranking(GlobalHeatMap(TOK, PROMPT100, (rand_maps((64, 64), 4) * 4).floor() / 4), word_list(4),
                  image(512, 512), regions, True)


def test_complement_invariant():
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((76, 52), 6))
    regions = make_regions(1216, 832, 6, 2)
    both = torch.cat([regions, (regions == 0).to(torch.uint8)])
    _, rk = ghm.region_ranking(word_list(8), image(1216, 832), both, to_cpu=False)
    n_p = (regions != 0).sum((-1, -2))
    total = 2 * n_p * (1216 * 832 - n_p)
    assert torch.equal(rk.u2[:6] + rk.u2[6:], total[:, None].expand(-1, 8))


def test_rounds_give_the_same_bits(monkeypatch):
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((75, 100), 7))
    img, regions, words = image(600, 800), make_regions(600, 800, 7, 1), word_list(5)
    before = _native.launch_count()
    _, one = ghm.region_ranking(words, img, regions, to_cpu=False)
    assert _native.launch_count() - before == 1 + 18                     # every plane in one round
    for planes in (1, 2, 3):
        monkeypatch.setattr(heatmap, 'REGION_RANKING_SCRATCH_BYTES',
                            _native.region_ranking_scratch_bytes(planes, 600, 800))
        before = _native.launch_count()
        _, rk = ghm.region_ranking(words, img, regions, to_cpu=False)
        assert _native.launch_count() - before == 1 + 18 * -(-5 // planes)
        assert torch.equal(rk.u2, one.u2)
        assert torch.equal(rk.ap.view(torch.int64), one.ap.view(torch.int64))


def test_repeated_calls_give_the_same_bits():
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((128, 128), 2))
    img, regions, words = image(1024, 1024), make_regions(1024, 1024, 16, 4), word_list(8)
    _, a = ghm.region_ranking(words, img, regions, to_cpu=False)
    for _ in range(2):
        _, b = ghm.region_ranking(words, img, regions, to_cpu=False)
        assert torch.equal(a.u2, b.u2) and torch.equal(a.ap.view(torch.int64), b.ap.view(torch.int64))
    _, c = ghm.region_ranking(words, img, regions)                        # to the host by default
    assert not c.u2.is_cuda and not c.ap.is_cuda and not c.region_area.is_cuda
    assert torch.equal(c.u2, a.u2.cpu())


# ---- stacks from the tracer ------------------------------------------------------------------------------------------
def check_stack(stack, words, img, regions, **kw):
    word_maps, rk = stack.region_ranking(words, img, regions, to_cpu=False, **kw)
    n = len(stack)
    assert tuple(rk.u2.shape) == (n, regions.shape[0], len(words)) and tuple(rk.ap.shape) == tuple(rk.u2.shape)
    assert tuple(word_maps.shape[:2]) == (n, len(words))
    for t in range(n):
        whms, one = stack[t].region_ranking(words, img, regions, to_cpu=False, **kw)
        assert torch.equal(one.u2, rk.u2[t]), t
        assert torch.equal(one.ap.view(torch.int64), rk.ap[t].view(torch.int64)), t
        for i, w in enumerate(whms):
            assert torch.equal(w.heatmap, word_maps[t, i])
    assert tuple(rk.auroc().shape) == (n, regions.shape[0], len(words))
    return rk


def test_time_and_layer_stacks():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=5)
    img = image(512, 512)
    regions = make_regions(512, 512, 5, 2)
    words = ['dog', 'red ball', 'beach', 'dog']
    with trace(pipe, time_resolved=True) as tc:
        pipe(PROMPT, num_inference_steps=4, generator=torch.Generator().manual_seed(3))
        tm = tc.compute_time_heat_maps()
        assert len(tm) == 4
        check_stack(tm, words, img, regions)
        check_stack(tm, words, img, regions, absolute=True)
        layers = tc.compute_layer_heat_maps()
        assert len(layers) > 1
        check_stack(layers, words, img, regions)
        check_ranking(tm[2], words, img, regions, False)


# ---- limits through the C ABI ------------------------------------------------------------------------------------------
def _abi_call(maps, grid, out_hw, regions_ptr, n_regions, scratch_bytes=None):
    word_maps = torch.empty((1, 1) + grid, device=DEV)
    u2 = torch.empty((1, max(n_regions, 1), 1), dtype=torch.int64, device=DEV)
    ap = torch.empty((1, max(n_regions, 1), 1), dtype=torch.float64, device=DEV)
    need = _native.region_ranking_scratch_bytes(1, *out_hw)
    scratch = torch.empty(need if need <= 1 << 30 else 8, dtype=torch.uint8, device=DEV)
    rows, begin = (ctypes.c_int32 * 1)(1), (ctypes.c_int32 * 2)(0, 1)
    rc = _native.load().daam_region_ranking(ctypes.c_void_p(maps.data_ptr()), 1, maps.shape[0], grid[0], grid[1], rows,
                                            begin, 1, out_hw[0], out_hw[1], 0, ctypes.c_void_p(word_maps.data_ptr()),
                                            ctypes.c_void_p(regions_ptr), n_regions, ctypes.c_void_p(u2.data_ptr()),
                                            ctypes.c_void_p(ap.data_ptr()), ctypes.c_void_p(scratch.data_ptr()),
                                            need if scratch_bytes is None else scratch_bytes,
                                            ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    msg = _native.load().daam_last_error().decode() if rc else ''
    return rc, msg, u2, ap


def test_limit_statuses():
    grid, out = (16, 16), (72, 40)
    maps = rand_maps(grid, 5)
    regions = make_regions(*out, 64, 3)
    rc, _, u2, ap = _abi_call(maps, grid, out, regions.data_ptr(), 63)
    assert rc == 0 and bool((u2 >= 0).all())
    rc, msg, *_ = _abi_call(maps, grid, out, regions.data_ptr(), 64)
    assert rc == _native.E_UNSUPPORTED and '64 regions > 63' in msg
    rc, msg, *_ = _abi_call(maps, grid, out, regions.data_ptr(), 1,
                            scratch_bytes=_native.region_ranking_scratch_bytes(1, *out) - 1)
    assert rc == _native.E_INVALID and 'scratch bytes' in msg
    rc, _, *_ = _abi_call(maps, grid, out, 0, 1)
    assert rc == _native.E_INVALID                                          # null regions
    rc, _, *_ = _abi_call(maps, grid, out, regions.data_ptr(), 0)
    assert rc == _native.E_INVALID                                          # no region
    rc, msg, *_ = _abi_call(maps, grid, (4096, 4097), regions.data_ptr(), 1)
    assert rc == _native.E_UNSUPPORTED and 'more than 2^24 pixels' in msg
    ghm = GlobalHeatMap(TOK, PROMPT100, maps)
    with pytest.raises(_native.NativeError, match='97 words > 96'):
        ghm.region_ranking([f'w{i}' for i in range(97)], image(40, 72), regions[:2])
