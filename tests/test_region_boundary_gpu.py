"""Boundary scores (GlobalHeatMap.region_boundary / GlobalHeatMapStack.region_boundary, daam_region_boundary;
evaluate.boundary_scores, daam_mask_boundary) on the GPU, against tests/boundary64.py over the very masks
expand_words(..., threshold, to_cpu=False) returns.

* word_boundary, region_boundary, both hit arrays and max_d2 equal the float64 reference exactly; sum_dist is within
  n 2^-52 of the exactly rounded sum of n roots.
* SD-2.1 512^2 and 768^2, SDXL 1024^2 and 1216x832, off-grid 600x800; 1 / 8 / 96 words, 1 / 16 / 63 regions, 1 and 16
  tolerances including 0; normalised and absolute maps, word_idx and offset_idx.
* Empty and full masks and regions, single-pixel regions, checkerboards (every pixel a boundary pixel), a region in
  one corner against masks in the opposite corner (the longest scans).
* region_boundary equals boundary_scores of expand_words' masks bit for bit; swapping masks and regions swaps precision
  and recall and keeps Hausdorff and ASSD; time, image and layer stacks equal the per-map calls bit for bit; several
  rounds equal one; repeated calls give the same bits.
* The C ABI's limit and invalid statuses.
"""
import ctypes
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from daam_b200 import _native, heatmap, trace
from daam_b200.evaluate import boundary_scores
from daam_b200.heatmap import GlobalHeatMap, RegionBoundary
from daam_b200.testing.synthetic import TINY_SPEC, WhitespaceTokenizer, make_pipeline
from tests.boundary64 import as_stack, boundary64, sum_bound

pytestmark = pytest.mark.gpu
DEV = 'cuda'
TOK = WhitespaceTokenizer()
PROMPT100 = ' '.join(f'w{i}' for i in range(100))
PROMPT = 'a dog chasing a red ball on the beach'
FIELDS = ('word_boundary', 'region_boundary', 'word_hits', 'region_hits', 'max_d2', 'sum_dist')
TOL16 = [0, 1, 1.5, 2, 3, 4, 5, 6, 8, 10, 12, 16, 24, 32, 64, 1000]


def image(h, w):
    return SimpleNamespace(size=(w, h), height=h, width=w)


def out_size(grid, hw):
    return (hw[1], hw[0]) if grid[0] == grid[1] else hw


def word_list(n):
    words = [f'w{3 * i % 100}' for i in range(n)]
    if n >= 3:
        words[1] = 'w40 w41'
        words[-1] = words[0]
    return words


def rand_maps(grid, seed, n_rows=102):
    return torch.rand(n_rows, *grid, generator=torch.Generator().manual_seed(seed)).to(DEV)


def make_regions(h, w, n, seed):
    """``n`` uint8 regions: region 0 full, region 2 empty (from three on), then rectangles, blobs and single pixels,
    marked with bytes other than 1 too."""
    g = torch.Generator().manual_seed(seed)
    out = torch.zeros((n, h, w), dtype=torch.uint8)
    out[0] = 1
    for r in range(1, n):
        if r == 2:
            continue
        y0, x0 = int(torch.randint(0, h, (1,), generator=g)), int(torch.randint(0, w, (1,), generator=g))
        mark = (1, 7, 255)[r % 3]
        if r % 4 == 3:
            out[r, y0, x0] = mark                                             # a single pixel
            continue
        y1, x1 = int(torch.randint(y0 + 1, h + 1, (1,), generator=g)), int(torch.randint(x0 + 1, w + 1, (1,), generator=g))
        if r % 2:
            out[r, y0:y1, x0:x1] = mark
        else:
            out[r] = (torch.rand(h, w, generator=g) < 0.3).to(torch.uint8) * mark
    return out.to(DEV)


def as_numpy(b: RegionBoundary):
    return {f: getattr(b, f).cpu().numpy() for f in FIELDS}


def assert_matches(got: RegionBoundary, want):
    g = as_numpy(got)
    for f in FIELDS[:-1]:
        np.testing.assert_array_equal(g[f], want[f], err_msg=f)
    err = np.abs(g['sum_dist'] - want['sum_dist'])
    assert bool((err <= sum_bound(want)).all()), float(err.max())


def assert_same_bits(a: RegionBoundary, b: RegionBoundary):
    for f in FIELDS:
        x, y = getattr(a, f), getattr(b, f)
        if x.dtype == torch.float64:
            x, y = x.view(torch.int64), y.view(torch.int64)
        assert torch.equal(x.cpu(), y.cpu()), f


def check_boundary(ghm, words, img, regions, threshold, tolerances=None, **kw):
    """The scores against boundary64 of expand_words' thresholded masks; returns (boundary, masks)."""
    _, b = ghm.region_boundary(words, img, regions, threshold, tolerances, to_cpu=False, **kw)
    n_reg, n_words = regions.shape[0], len(words)
    T = b.tolerances.numel()
    assert tuple(b.word_hits.shape) == (T, n_reg, n_words) and b.word_hits.dtype == torch.int32 and b.word_hits.is_cuda
    assert tuple(b.max_d2.shape) == (n_reg, n_words, 2) and b.max_d2.dtype == torch.int64
    assert tuple(b.sum_dist.shape) == (n_reg, n_words, 2) and b.sum_dist.dtype == torch.float64
    _, m = ghm.expand_words(words, img, threshold=threshold, to_cpu=False, **kw)
    tol = b.tolerances.cpu().numpy()
    want = as_stack(boundary64(m.cpu().numpy() > 0, regions.cpu().numpy(), tol), 1, n_words)
    assert_matches(b, {f: (v[0] if f != 'region_boundary' else v) for f, v in want.items()})
    return b, m


PAIRS = [((64, 64), (512, 512)), ((96, 96), (768, 768)), ((128, 128), (1024, 1024)), ((76, 52), (1216, 832)),
         ((75, 100), (600, 800))]
PAIR_IDS = [f'{g[0]}x{g[1]}-{h}x{w}' for g, (h, w) in PAIRS]


@pytest.mark.parametrize('absolute', [False, True], ids=['normalised', 'absolute'])
@pytest.mark.parametrize('grid,hw', PAIRS, ids=PAIR_IDS)
def test_sizes_against_float64(grid, hw, absolute):
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps(grid, 5 * grid[0] + grid[1]))
    h, w = out_size(grid, hw)
    b, _ = check_boundary(ghm, word_list(8), image(*hw), make_regions(h, w, 5, h + w), 0.6 if not absolute else 0.55)
    assert b.tolerances.tolist() == [float(np.ceil(0.008 * np.hypot(h, w)))]       # DAVIS's default
    assert bool(torch.isnan(b.hausdorff()[2]).all()) and bool(torch.isnan(b.assd()[2]).all())   # region 2 is empty


@pytest.mark.parametrize('n_words,n_regions,n_tol,grid,hw', [(1, 1, 1, (64, 64), (512, 512)),
                                                             (8, 16, 16, (64, 64), (512, 512)),
                                                             (1, 63, 16, (40, 30), (320, 240)),
                                                             (96, 1, 1, (40, 30), (320, 240)),
                                                             (96, 63, 16, (24, 20), (150, 130))])
def test_word_region_and_tolerance_counts(n_words, n_regions, n_tol, grid, hw):
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps(grid, n_words + n_regions))
    h, w = out_size(grid, hw)
    tol = TOL16[:n_tol] if n_tol > 1 else [0]
    check_boundary(ghm, word_list(n_words), image(*hw), make_regions(h, w, n_regions, n_regions), 0.5, tol)


def test_word_idx_and_offset_idx():
    ghm = GlobalHeatMap(TOK, 'a dog and a dog and a cat', rand_maps((64, 64), 11, n_rows=12))
    regions = make_regions(512, 512, 4, 8)
    check_boundary(ghm, ['dog', 'dog', 'cat'], image(512, 512), regions, 0.4, [1, 4], word_idx=[0, 1, None])
    check_boundary(ghm, ['dog', 'cat'], image(512, 512), regions, 0.4, [2], offset_idx=1)


def test_masks_against_float64_hard_cases():
    h, w = 200, 264
    yy, xx = torch.meshgrid(torch.arange(h), torch.arange(w), indexing='ij')
    checker = ((yy + xx) % 2).to(torch.uint8)
    corner = torch.zeros((h, w), dtype=torch.uint8)
    corner[:5, :7] = 1
    far = torch.zeros((h, w), dtype=torch.uint8)
    far[-9:, -4:] = 1
    line = torch.zeros((h, w), dtype=torch.uint8)
    line[:, -1] = 1
    masks = torch.stack([torch.zeros((h, w), dtype=torch.uint8), torch.ones((h, w), dtype=torch.uint8), checker, far,
                         line, 1 - checker]).to(DEV)
    pixel = torch.zeros((h, w), dtype=torch.uint8)
    pixel[h // 2, 0] = 1
    regions = torch.stack([torch.zeros((h, w), dtype=torch.uint8), torch.ones((h, w), dtype=torch.uint8), checker,
                           corner, pixel]).to(DEV)
    tol = [0, 1, 2.5, 300]
    for lead in ((6,), (2, 3)):
        got = boundary_scores(masks.reshape(*lead, h, w), regions, tol)
        m, n_words = (1, 6) if len(lead) == 1 else lead
        want = as_stack(boundary64(masks.cpu().numpy(), regions.cpu().numpy(), tol), m, n_words)
        if len(lead) == 1:
            want = {f: (v[0] if f != 'region_boundary' else v) for f, v in want.items()}
        assert_matches(got, want)
    assert int(got.word_boundary[0, 2]) == h * w // 2 and int(got.region_boundary[2]) == h * w // 2
    # the far corner (map 1, word 0) against the corner region 3: the longest scans; the Hausdorff distance runs from
    # the corner region's pixel (0, 0) to the far mask's nearest boundary pixel (h - 9, w - 4)
    assert float(got.hausdorff()[1, 3, 0]) == np.sqrt(float((h - 9) ** 2 + (w - 4) ** 2))


def test_region_boundary_equals_boundary_scores_of_expand_words():
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((76, 52), 6))
    img, regions, words = image(1216, 832), make_regions(1216, 832, 6, 2), word_list(8)
    _, b = ghm.region_boundary(words, img, regions, 0.5, [1, 3, 12], to_cpu=False)
    _, m = ghm.expand_words(words, img, threshold=0.5, to_cpu=False)
    assert_same_bits(b, boundary_scores(m > 0, regions, [1, 3, 12], to_cpu=False))
    # swapping masks and regions swaps precision and recall, keeps Hausdorff and ASSD
    masks = (m > 0).to(torch.uint8)
    ab = boundary_scores(masks, regions, [1, 3, 12])
    ba = boundary_scores(regions, masks, [1, 3, 12])
    assert torch.equal(ab.precision(), ba.recall().transpose(-1, -2))
    assert torch.equal(ab.recall(), ba.precision().transpose(-1, -2))
    torch.testing.assert_close(ab.hausdorff(), ba.hausdorff().transpose(-1, -2), rtol=0, atol=0, equal_nan=True)
    torch.testing.assert_close(ab.assd(), ba.assd().transpose(-1, -2), rtol=0, atol=0, equal_nan=True)
    assert bool(torch.isnan(ab.hausdorff()[2]).all())                    # region 2 is empty


def test_refine_words_output():
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((64, 64), 12))
    img = torch.randint(0, 256, (512, 512, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(1))
    regions = make_regions(512, 512, 4, 3)
    _, refined = ghm.refine_words(word_list(8), img, threshold=0.4, to_cpu=False)
    b = boundary_scores(refined > 0, regions, to_cpu=False)
    want = as_stack(boundary64(refined.cpu().numpy() > 0, regions.cpu().numpy(), [6]), 1, 8)
    assert_matches(b, {f: (v[0] if f != 'region_boundary' else v) for f, v in want.items()})


def test_rounds_give_the_same_bits(monkeypatch):
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((75, 100), 7))
    img, regions, words = image(600, 800), make_regions(600, 800, 7, 1), word_list(5)
    before = _native.launch_count()
    _, one = ghm.region_boundary(words, img, regions, 0.5, [2, 9], to_cpu=False)
    assert _native.launch_count() - before == 1 + 5                      # every plane in one round
    for planes in (1, 2, 3):
        monkeypatch.setattr(heatmap, 'REGION_BOUNDARY_SCRATCH_BYTES',
                            _native.boundary_scratch_bytes(7, planes, 600, 800))
        before = _native.launch_count()
        _, b = ghm.region_boundary(words, img, regions, 0.5, [2, 9], to_cpu=False)
        assert _native.launch_count() - before == 1 + 5 * -(-5 // planes)
        assert_same_bits(b, one)


def test_repeated_calls_give_the_same_bits():
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((128, 128), 2))
    img, regions, words = image(1024, 1024), make_regions(1024, 1024, 16, 4), word_list(8)
    _, a = ghm.region_boundary(words, img, regions, 0.5, to_cpu=False)
    for _ in range(2):
        _, b = ghm.region_boundary(words, img, regions, 0.5, to_cpu=False)
        assert_same_bits(a, b)
    _, c = ghm.region_boundary(words, img, regions, 0.5)                  # to the host by default
    assert not c.word_hits.is_cuda and not c.sum_dist.is_cuda
    assert_same_bits(a, c)


# ---- stacks from the tracer ------------------------------------------------------------------------------------------
def check_stack(stack, words, img, regions, **kw):
    word_maps, b = stack.region_boundary(words, img, regions, 0.4, [1, 5], to_cpu=False, **kw)
    n = len(stack)
    assert tuple(b.word_hits.shape) == (n, 2, regions.shape[0], len(words))
    assert tuple(word_maps.shape[:2]) == (n, len(words))
    for t in range(n):
        whms, one = stack[t].region_boundary(words, img, regions, 0.4, [1, 5], to_cpu=False, **kw)
        assert_same_bits(one, b.map(t))
        for i, w in enumerate(whms):
            assert torch.equal(w.heatmap, word_maps[t, i])
    assert tuple(b.f_score().shape) == (n, 2, regions.shape[0], len(words))
    return b


def test_time_image_and_layer_stacks():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=5)
    img = image(512, 512)
    regions = make_regions(512, 512, 5, 2)
    words = ['dog', 'red ball', 'beach', 'dog']
    with trace(pipe, time_resolved=True) as tc:
        pipe(PROMPT, num_inference_steps=4, generator=torch.Generator().manual_seed(3))
        tm = tc.compute_time_heat_maps()
        check_stack(tm, words, img, regions)
        check_stack(tm, words, img, regions, absolute=True)
        layers = tc.compute_layer_heat_maps()
        assert len(layers) > 1
        check_stack(layers, words, img, regions)
        check_boundary(tm[2], words, img, regions, 0.4, [1, 5])
    with trace(pipe) as tc:
        pipe(PROMPT, num_inference_steps=2, generator=torch.Generator().manual_seed(11), num_images_per_prompt=3)
        per_image = tc.compute_image_heat_maps()
        assert len(per_image) == 3
        check_stack(per_image, words, img, regions)


# ---- limits through the C ABI ------------------------------------------------------------------------------------------
def _abi_call(maps, grid, out_hw, regions_ptr, n_regions, tolerances=(1.0,), threshold=0.5, scratch_bytes=None,
              scratch_offset=0):
    word_maps = torch.empty((1, 1) + grid, device=DEV)
    R, T = max(n_regions, 1), max(len(tolerances), 1)
    i32 = dict(dtype=torch.int32, device=DEV)
    outs = [torch.empty(1, **i32), torch.empty(R, **i32), torch.empty(T * R, **i32), torch.empty(T * R, **i32),
            torch.empty(2 * R, dtype=torch.int64, device=DEV), torch.empty(2 * R, dtype=torch.float64, device=DEV)]
    need = _native.boundary_scratch_bytes(R, 1, *out_hw)
    scratch = torch.empty((need if need <= 1 << 30 else 8) + 8, dtype=torch.uint8, device=DEV)
    rows, begin = (ctypes.c_int32 * 1)(1), (ctypes.c_int32 * 2)(0, 1)
    tol = (ctypes.c_float * max(len(tolerances), 1))(*tolerances)
    vp = ctypes.c_void_p
    rc = _native.load().daam_region_boundary(vp(maps.data_ptr()), 1, maps.shape[0], grid[0], grid[1], rows, begin, 1,
                                             out_hw[0], out_hw[1], 0, threshold, tol, len(tolerances),
                                             vp(word_maps.data_ptr()), vp(regions_ptr), n_regions,
                                             *(vp(o.data_ptr()) for o in outs), vp(scratch.data_ptr() + scratch_offset),
                                             need if scratch_bytes is None else scratch_bytes,
                                             vp(torch.cuda.current_stream().cuda_stream))
    msg = _native.load().daam_last_error().decode() if rc else ''
    return rc, msg, outs


def test_limit_statuses():
    grid, out = (16, 16), (72, 40)
    maps = rand_maps(grid, 5)
    regions = make_regions(*out, 64, 3)
    rc, _, outs = _abi_call(maps, grid, out, regions.data_ptr(), 63, TOL16)
    assert rc == 0 and bool((outs[2] >= 0).all())
    torch.cuda.synchronize()
    cases = [
        (dict(n_regions=64), _native.E_UNSUPPORTED, '64 regions > 63'),
        (dict(tolerances=list(range(17))), _native.E_UNSUPPORTED, '17 tolerances > 16'),
        (dict(out_hw=(4096, 4097)), _native.E_UNSUPPORTED, 'more than 2^24 pixels'),
        (dict(tolerances=[]), _native.E_INVALID, 'non-positive size'),
        (dict(tolerances=[2, 1]), _native.E_INVALID, 'strictly ascending'),
        (dict(tolerances=[1, 1]), _native.E_INVALID, 'strictly ascending'),
        (dict(tolerances=[-1]), _native.E_INVALID, 'finite and >= 0'),
        (dict(tolerances=[float('inf')]), _native.E_INVALID, 'finite and >= 0'),
        (dict(tolerances=[float('nan')]), _native.E_INVALID, 'finite and >= 0'),
        (dict(threshold=float('nan')), _native.E_INVALID, 'threshold nan is not finite'),
        (dict(threshold=float('inf')), _native.E_INVALID, 'is not finite'),
        (dict(scratch_offset=4), _native.E_INVALID, '8-byte aligned'),
        (dict(scratch_bytes=_native.boundary_scratch_bytes(1, 1, 72, 40) - 1), _native.E_INVALID, 'scratch bytes'),
        (dict(regions_ptr=0), _native.E_INVALID, 'null pointer'),
        (dict(n_regions=0), _native.E_INVALID, 'non-positive size'),
    ]
    for kw, status, text in cases:
        args = dict(out_hw=out, regions_ptr=regions.data_ptr(), n_regions=1)
        args.update(kw)
        rc, msg, _ = _abi_call(maps, grid, args.pop('out_hw'), args.pop('regions_ptr'), args.pop('n_regions'), **args)
        assert rc == status and text in msg, (kw, rc, msg)
    ghm = GlobalHeatMap(TOK, PROMPT100, maps)
    with pytest.raises(_native.NativeError, match='97 words > 96'):
        ghm.region_boundary([f'w{i}' for i in range(97)], image(40, 72), regions[:2], 0.5)
    # the mask entry's statuses
    masks = torch.zeros((2, 72, 40), dtype=torch.uint8, device=DEV)
    i32 = dict(dtype=torch.int32, device=DEV)
    o = [torch.empty(2, **i32), torch.empty(1, **i32), torch.empty(2, **i32), torch.empty(2, **i32),
         torch.empty(4, dtype=torch.int64, device=DEV), torch.empty(4, dtype=torch.float64, device=DEV)]
    need = _native.boundary_scratch_bytes(1, 1, 72, 40)
    scratch = torch.empty(need, dtype=torch.uint8, device=DEV)
    vp = ctypes.c_void_p

    def mask_call(n_planes=2, n_regions=1, tol=(1.0,), n_bytes=need, m_ptr=masks.data_ptr()):
        t = (ctypes.c_float * max(len(tol), 1))(*tol)
        rc = _native.load().daam_mask_boundary(vp(m_ptr), n_planes, 72, 40, vp(regions.data_ptr()), n_regions, t,
                                               len(tol), *(vp(x.data_ptr()) for x in o), vp(scratch.data_ptr()),
                                               n_bytes, vp(torch.cuda.current_stream().cuda_stream))
        return rc, (_native.load().daam_last_error().decode() if rc else '')
    assert mask_call()[0] == 0
    torch.cuda.synchronize()
    assert o[0].tolist() == [0, 0] and int(o[4][0]) == -1
    assert mask_call(n_regions=64) == (_native.E_UNSUPPORTED, 'daam_mask_boundary: 64 regions > 63')
    assert mask_call(tol=[0.0] * 17)[0] == _native.E_UNSUPPORTED
    assert mask_call(tol=[3.0, 2.0])[0] == _native.E_INVALID
    assert mask_call(n_bytes=need - 1)[0] == _native.E_INVALID
    assert mask_call(m_ptr=0)[0] == _native.E_INVALID
    assert mask_call(n_planes=0)[0] == _native.E_INVALID
