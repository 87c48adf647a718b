"""Superpixel word segmentation (GlobalHeatMap.segment_superpixels / GlobalHeatMapStack.segment_superpixels,
evaluate.superpixels, daam_segment_superpixels / daam_image_superpixels) on the GPU.

* The partition equals tests/slic64.py bit for bit: 1x1, 1xW, Hx1, 7x5, 48x40, 512^2, 1024^2 and 1216x832; 1, 4, 100,
  1024, 4096 and H*W segments; 1, 2, 10 and 64 passes; noise, flat blocks, one colour and a checkerboard (ties).
* The pooled scores lie within one fp32 ulp of the float64 means of the values expand_words(..., to_cpu=False)
  returns, and the labels are the float64 argmax wherever the top two means differ by more than that; with one-pixel
  cells labels and scores equal segment's bit for bit. 1, 8 and 96 words, absolute maps, thresholds, SD-2.1, SDXL and
  off-grid sizes.
* The word call's partition is evaluate.superpixels'; stacks equal the per-map calls with one image and with one per
  map; rounds and repeated calls give the same bits.
* The C ABI's statuses.
"""
import ctypes
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from daam_b200 import _native, evaluate, heatmap
from daam_b200.heatmap import GlobalHeatMap, GlobalHeatMapStack
from daam_b200.testing.synthetic import WhitespaceTokenizer
from tests.slic64 import pooled_labels64, slic

pytestmark = pytest.mark.gpu
DEV = 'cuda'
TOK = WhitespaceTokenizer()
PROMPT100 = ' '.join(f'w{i}' for i in range(100))


def size_of(img):
    h, w = int(img.shape[-3]), int(img.shape[-2])
    return SimpleNamespace(size=(w, h), height=h, width=w)


def make_image(h, w, kind, seed=0):
    """uint8 [h, w, 3] on the device: 'noise', 'blocks' (flat random-coloured blocks plus a little noise), 'const' or
    'checker' (two colours alternating per pixel: equal distances to many centres)."""
    g = torch.Generator().manual_seed(seed)
    if kind == 'noise':
        img = torch.randint(0, 256, (h, w, 3), generator=g)
    elif kind == 'blocks':
        by, bx = int(torch.randint(3, 40, (1,), generator=g)), int(torch.randint(3, 40, (1,), generator=g))
        blocks = torch.randint(0, 256, (h // by + 1, w // bx + 1, 3), generator=g)
        img = blocks.repeat_interleave(by, 0).repeat_interleave(bx, 1)[:h, :w]
        img = (img + torch.randint(-6, 7, (h, w, 3), generator=g)).clamp(0, 255)
    elif kind == 'const':
        img = torch.tensor([37, 201, 90]).expand(h, w, 3)
    else:
        yy, xx = torch.meshgrid(torch.arange(h), torch.arange(w), indexing='ij')
        img = (((yy + xx) % 2) * 200 + 20)[..., None].expand(h, w, 3)
    return img.to(torch.uint8).contiguous().to(DEV)


def word_list(n):
    words = [f'w{3 * i % 100}' for i in range(n)]
    if n >= 3:
        words[1] = 'w40 w41'
        words[-1] = words[0]
    return words


def rand_maps(grid, seed, n_maps=None):
    shape = ((n_maps,) if n_maps else ()) + (102,) + tuple(grid)
    return torch.rand(*shape, generator=torch.Generator().manual_seed(seed)).to(DEV)


# ---- the partition ---------------------------------------------------------------------------------------------------------
PARTITIONS = [
    (1, 1, 1, 20.0, 1, 'noise'), (1, 1, 1, 20.0, 64, 'const'),
    (1, 257, 4, 20.0, 10, 'noise'), (1, 257, 257, 20.0, 2, 'checker'), (300, 1, 100, 5.0, 10, 'blocks'),
    (7, 5, 4, 20.0, 2, 'checker'), (7, 5, 35, 20.0, 10, 'noise'), (7, 5, 1, 20.0, 64, 'noise'),
    (48, 40, 100, 20.0, 10, 'blocks'), (48, 40, 1920, 20.0, 2, 'noise'), (48, 40, 4, 1.0, 64, 'checker'),
    (48, 40, 100, 80.0, 64, 'const'),
    (512, 512, 1024, 20.0, 10, 'blocks'), (512, 512, 4096, 20.0, 2, 'noise'), (512, 512, 1, 20.0, 1, 'noise'),
    (512, 512, 100, 20.0, 10, 'const'), (512, 512, 1024, 20.0, 1, 'checker'), (512, 512, 4, 3.0, 10, 'blocks'),
    (256, 256, 65536, 20.0, 2, 'noise'),
    (1024, 1024, 1024, 20.0, 10, 'blocks'), (1024, 1024, 4096, 20.0, 10, 'noise'),
    (1216, 832, 1024, 20.0, 10, 'blocks'), (1216, 832, 4, 20.0, 2, 'checker'),
]


@pytest.mark.parametrize('h,w,k,c,t,kind', PARTITIONS)
def test_partition_is_the_reference(h, w, k, c, t, kind):
    img = make_image(h, w, kind, seed=h + w + k)
    sp = evaluate.superpixels(img, n_segments=k, compactness=c, iterations=t)
    assert sp.dtype == torch.int32 and tuple(sp.shape) == (h, w)
    np.testing.assert_array_equal(sp.numpy(), slic(img.cpu().numpy(), k, c, t))


def test_images_back_to_back():
    imgs = torch.stack([make_image(48, 72, kind, seed=i) for i, kind in enumerate(('noise', 'blocks', 'checker'))])
    sp = evaluate.superpixels(imgs, n_segments=50, iterations=5)
    for i in range(3):
        np.testing.assert_array_equal(sp[i].numpy(), slic(imgs[i].cpu().numpy(), 50, 20.0, 5))


# ---- the pooled labels -----------------------------------------------------------------------------------------------------
def check_pooled(ghm, words, img, k, threshold=None, absolute=False, c=20.0, t=10):
    _, labels, scores, sp = ghm.segment_superpixels(words, img, n_segments=k, compactness=c, iterations=t,
                                                    threshold=threshold, absolute=absolute, to_cpu=False)
    assert torch.equal(sp, evaluate.superpixels(img, n_segments=k, compactness=c, iterations=t, to_cpu=False))
    _, m = ghm.expand_words(words, size_of(img), absolute=absolute, to_cpu=False)
    ref_lab, ref_sc, gap = pooled_labels64(m.cpu().numpy(), sp.cpu().numpy(), threshold)
    sc = scores.cpu().numpy()
    ulp = np.spacing(np.abs(ref_sc))
    assert bool((np.abs(sc.astype(np.float64) - ref_sc) <= ulp).all())
    sure = gap > 2 * ulp
    if threshold:
        sure &= np.abs(ref_sc.astype(np.float64) - np.float32(threshold)) > ulp
    lab = labels.cpu().numpy()
    assert np.array_equal(lab[sure], ref_lab[sure]) and sure.mean() > 0.5
    # a superpixel's pixels share its label and score
    flat = sp.cpu().numpy().ravel()
    first = np.zeros(flat.max() + 1, dtype=np.int64)
    first[flat[::-1]] = np.arange(flat.size)[::-1]
    assert np.array_equal(lab.ravel(), lab.ravel()[first[flat]]) and np.array_equal(sc.ravel(), sc.ravel()[first[flat]])
    return labels, scores, sp


@pytest.mark.parametrize('grid,out,n_words,absolute,threshold,k', [
    ((64, 64), (512, 512), 8, False, None, 1024),
    ((64, 64), (512, 512), 1, False, 0.4, 256),
    ((64, 64), (512, 512), 96, False, 0.4, 1024),
    ((64, 64), (512, 512), 24, True, None, 4096),
    ((128, 128), (1024, 1024), 8, False, 0.4, 4096),
    ((152, 104), (1216, 832), 8, True, None, 1024),
    ((75, 100), (600, 800), 8, False, None, 100),
    ((18, 10), (72, 40), 8, False, 0.4, 1),
    ((18, 10), (72, 40), 3, False, None, 4),
])
def test_pooled_labels_are_the_float64_means(grid, out, n_words, absolute, threshold, k):
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps(grid, n_words + k))
    check_pooled(ghm, word_list(n_words), make_image(*out, 'blocks', seed=k), k, threshold, absolute)


@pytest.mark.parametrize('grid,out,n_words', [((16, 24), (200, 300), 8), ((16, 16), (256, 256), 96),
                                              ((4, 8), (1, 97), 3), ((8, 4), (33, 1), 1)])
@pytest.mark.parametrize('threshold', [None, 0.4])
def test_one_pixel_cells_are_segment(grid, out, n_words, threshold):
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps(grid, n_words))
    img = make_image(*out, 'noise')
    words = word_list(n_words)
    _, labels, scores, sp = ghm.segment_superpixels(words, img, n_segments=out[0] * out[1], threshold=threshold)
    assert torch.equal(sp, torch.arange(out[0] * out[1], dtype=torch.int32).view(out))
    _, seg_labels, seg_scores = ghm.segment(words, size_of(img), threshold=threshold)
    assert torch.equal(labels, seg_labels)
    assert torch.equal(scores.view(torch.int32), seg_scores.view(torch.int32))


# ---- consistency -----------------------------------------------------------------------------------------------------------
def test_stacks_equal_per_map_calls(monkeypatch):
    maps = rand_maps((64, 64), 3, n_maps=4)
    stack = GlobalHeatMapStack(TOK, PROMPT100, maps)
    words = word_list(8)
    img = make_image(512, 512, 'blocks', seed=1)
    imgs = torch.stack([make_image(512, 512, 'blocks', seed=i) for i in range(4)])
    for image, per_map in ((img, False), (imgs, True)):
        word_maps, labels, scores, sp = stack.segment_superpixels(words, image, n_segments=500, threshold=0.3,
                                                                  to_cpu=False)
        assert tuple(sp.shape) == ((4, 512, 512) if per_map else (512, 512))
        for t in range(4):
            wm, lab, sc, spt = GlobalHeatMap(TOK, PROMPT100, maps[t]).segment_superpixels(
                words, image[t] if per_map else image, n_segments=500, threshold=0.3, to_cpu=False)
            assert torch.equal(lab, labels[t]) and torch.equal(sc.view(torch.int32), scores[t].view(torch.int32))
            assert torch.equal(spt, sp[t] if per_map else sp)
            assert torch.equal(torch.stack([w.heatmap for w in wm]), word_maps[t])
        # a budget of one image and one map: four rounds, the same bits
        monkeypatch.setattr(heatmap, 'SUPERPIXEL_SCRATCH_BYTES', 1)
        out = stack.segment_superpixels(words, image, n_segments=500, threshold=0.3, to_cpu=False)
        monkeypatch.undo()
        assert torch.equal(out[1], labels) and torch.equal(out[2].view(torch.int32), scores.view(torch.int32))
        assert torch.equal(out[3], sp)


def test_repeated_calls_give_the_same_bits():
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((128, 128), 9))
    img = make_image(1024, 1024, 'checker')
    first = ghm.segment_superpixels(word_list(24), img, n_segments=4096, to_cpu=False)
    for _ in range(3):
        again = ghm.segment_superpixels(word_list(24), img, n_segments=4096, to_cpu=False)
        assert torch.equal(again[1], first[1]) and torch.equal(again[2].view(torch.int32), first[2].view(torch.int32))
        assert torch.equal(again[3], first[3])


def test_empty_word_list_still_partitions():
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((16, 12), 1))
    img = make_image(64, 48, 'blocks')
    whms, labels, scores, sp = ghm.segment_superpixels([], img, n_segments=30)
    assert whms == [] and not labels.any() and bool((scores == float('-inf')).all())
    np.testing.assert_array_equal(sp.numpy(), slic(img.cpu().numpy(), 30, 20.0, 10))


# ---- the C ABI -------------------------------------------------------------------------------------------------------------
def _abi_call(out_hw=(72, 40), n_words=1, n_segments=50, compactness=20.0, iterations=2, scratch_bytes=None,
              scratch_offset=0, null=None, stride=0):
    """daam_segment_superpixels on one real map (buffers of one map, or of one pixel past the pixel limit: a refused
    call reads none of them); returns (status, message, labels)."""
    grid = (16, 16)
    small = out_hw[0] * out_hw[1] <= 1 << 22
    maps = rand_maps(grid, 5)
    word_maps = torch.empty((1, max(n_words, 1)) + grid, device=DEV)
    shape = out_hw if small else (1, 1)
    image = make_image(*shape, 'blocks')
    labels = torch.full(shape, 255, dtype=torch.uint8, device=DEV)
    scores = torch.full(shape, float('nan'), device=DEV)
    sp = torch.full(shape, -1, dtype=torch.int32, device=DEV)
    if small and n_segments >= 1:
        ny, nx = _native.superpixel_grid(*out_hw, n_segments)
        need = _native.superpixel_scratch_bytes(1, 1, max(n_words, 1), ny, nx, *out_hw)
    else:
        need = 1 << 20
    scratch = torch.empty(min(need, 1 << 30) + 16, dtype=torch.uint8, device=DEV)
    ptrs = {'maps': maps.data_ptr(), 'word_maps': word_maps.data_ptr(), 'image': image.data_ptr(),
            'labels': labels.data_ptr(), 'scores': scores.data_ptr(), 'sp': sp.data_ptr(),
            'scratch': scratch.data_ptr() + scratch_offset}
    if null:
        ptrs[null] = 0
    rows = (ctypes.c_int32 * max(n_words, 1))(*range(1, max(n_words, 1) + 1))
    begin = (ctypes.c_int32 * (max(n_words, 1) + 1))(*range(max(n_words, 1) + 1))
    vp = ctypes.c_void_p
    rc = _native.load().daam_segment_superpixels(
        vp(ptrs['maps']), 1, 102, grid[0], grid[1], rows, begin, n_words, out_hw[0], out_hw[1], 0, 1, 0.4,
        n_segments, compactness, iterations, vp(ptrs['word_maps']), vp(ptrs['image']), stride, vp(ptrs['labels']),
        vp(ptrs['scores']), vp(ptrs['sp']), vp(ptrs['scratch']), need if scratch_bytes is None else scratch_bytes,
        vp(torch.cuda.current_stream().cuda_stream))
    msg = _native.load().daam_last_error().decode() if rc else ''
    return rc, msg, labels


def test_abi_statuses():
    rc, _, labels = _abi_call()
    torch.cuda.synchronize()
    assert rc == 0 and int(labels.max()) <= 1
    for kw in (dict(iterations=64), dict(iterations=1), dict(n_segments=72 * 40), dict(compactness=1e-30)):
        assert _abi_call(**kw)[0] == 0, kw
    for kw, status, text in [
            (dict(null='maps'), _native.E_INVALID, 'null pointer or non-positive size'),
            (dict(null='sp'), _native.E_INVALID, 'null pointer or non-positive size'),
            (dict(null='scratch'), _native.E_INVALID, 'null pointer or non-positive size'),
            (dict(stride=-1), _native.E_INVALID, 'null pointer or non-positive size'),
            (dict(out_hw=(4097, 4096)), _native.E_UNSUPPORTED, 'more than 2^24 pixels'),
            (dict(out_hw=(4097, 4096), n_segments=0), _native.E_UNSUPPORTED, 'more than 2^24 pixels'),
            (dict(n_segments=0), _native.E_INVALID, 'n_segments 0 < 1'),
            (dict(n_segments=0, compactness=0.0), _native.E_INVALID, 'n_segments 0 < 1'),
            (dict(compactness=0.0), _native.E_INVALID, 'compactness 0 is not finite and > 0'),
            (dict(compactness=-2.0), _native.E_INVALID, 'compactness -2 is not finite and > 0'),
            (dict(compactness=float('inf')), _native.E_INVALID, 'compactness inf is not finite and > 0'),
            (dict(compactness=float('nan'), iterations=0), _native.E_INVALID, 'compactness nan'),
            (dict(iterations=0), _native.E_INVALID, 'iterations 0 is not in [1, 64]'),
            (dict(iterations=65), _native.E_INVALID, 'iterations 65 is not in [1, 64]'),
            (dict(out_hw=(300, 300), n_segments=300 * 300), _native.E_UNSUPPORTED, 'grid of cells is more than 65536'),
            (dict(out_hw=(300, 300), n_segments=300 * 300, iterations=0), _native.E_INVALID, 'iterations 0'),
            (dict(scratch_offset=4), _native.E_INVALID, 'scratch must be 8-byte aligned'),
            (dict(scratch_bytes=1024), _native.E_INVALID, 'scratch bytes <'),
            (dict(n_words=0), _native.E_INVALID, 'empty word list'),
            (dict(n_words=97, scratch_bytes=1 << 30), _native.E_UNSUPPORTED, '97 words > 96'),
    ]:
        rc, msg, _ = _abi_call(**kw)
        assert rc == status and text in msg, (kw, rc, msg)
    # the partition alone
    vp = ctypes.c_void_p
    img = make_image(40, 40, 'noise')
    sp = torch.empty((40, 40), dtype=torch.int32, device=DEV)
    scratch = torch.empty(1 << 20, dtype=torch.uint8, device=DEV)
    lib = _native.load()
    stream = vp(torch.cuda.current_stream().cuda_stream)
    for args, status, text in [
            ((40, 40, 16, 20.0, 2, 1 << 20), 0, ''),
            ((40, 40, 0, 20.0, 2, 1 << 20), _native.E_INVALID, 'n_segments 0 < 1'),
            ((40, 40, 16, 0.0, 2, 1 << 20), _native.E_INVALID, 'compactness 0'),
            ((40, 40, 16, 20.0, 65, 1 << 20), _native.E_INVALID, 'iterations 65'),
            ((40, 40, 16, 20.0, 2, 96 * 16 - 1), _native.E_INVALID, 'scratch bytes <'),
            ((4097, 4097, 16, 20.0, 2, 1 << 20), _native.E_UNSUPPORTED, 'more than 2^24 pixels'),
            ((0, 40, 16, 20.0, 2, 1 << 20), _native.E_INVALID, 'null pointer or non-positive size'),
    ]:
        h, w, k, c, t, nb = args
        rc = lib.daam_image_superpixels(vp(img.data_ptr()), 1, h, w, k, c, t, vp(sp.data_ptr()),
                                        vp(scratch.data_ptr()), nb, stream)
        msg = lib.daam_last_error().decode() if rc else ''
        assert rc == status and text in msg, (args, rc, msg)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(sp.cpu().numpy(), slic(img.cpu().numpy(), 16, 20.0, 2))
