"""CRF-refined word segmentation (GlobalHeatMap.segment_crf / GlobalHeatMapStack.segment_crf, daam_segment_crf) on the
GPU, against tests/crf64.py over the very values expand_words(..., to_cpu=False) returns.

* One update at a time: the calls with ``iterations = k`` and ``k + 1`` (``probs=True``) give the device's ``Q_k`` and
  ``Q_{k+1}``; ``crf_step64`` of ``Q_k`` and the exact logits ``z`` (``scale`` a power of two) must lie within
  ``crf_bound`` of ``Q_{k+1}`` everywhere checked, and the labels must be the float64 argmax wherever its top-two
  margin exceeds twice the logit bound. ``Q_0`` is checked against the softmax of ``z`` the same way. At the larger
  sizes the reference covers bands of rows at the top, middle and bottom, borders included.
* SD-2.1 512^2 and 768^2, SDXL 1024^2 and 1216x832, off-grid 600x800; radii 1, 4, 8, 16 and larger than the image; 1,
  8 and 96 words (97 labels take seven label chunks); absolute maps; threshold on and off; word_idx and offset_idx.
* Reduction to segment, bit for bit, at iterations = 0 and at zero weights, ties included.
* Repeated calls and any round split give the same bits; time, image (one image per map) and layer stacks equal the
  per-map calls bit for bit.
* The C ABI's statuses.
* Quality: on flat-coloured shapes with sharp edges, whose word maps are the shapes' masks area-averaged onto the
  64 x 64 grid, the defaults' labels beat segment(threshold=0.4)'s on IoU and boundary F against the true shapes.
"""
import ctypes
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from daam_b200 import _native, heatmap, trace
from daam_b200.evaluate import boundary_scores
from daam_b200.heatmap import GlobalHeatMap, GlobalHeatMapStack
from daam_b200.testing.synthetic import TINY_SPEC, WhitespaceTokenizer, make_pipeline
from tests.crf64 import crf_bound, crf_step64, crf_tables, logits64, softmax64

pytestmark = pytest.mark.gpu
DEV = 'cuda'
TOK = WhitespaceTokenizer()
PROMPT100 = ' '.join(f'w{i}' for i in range(100))
PROMPT = 'a dog chasing a red ball on the beach'
WEIGHTS = dict(appearance=10.0, sigma_xy=8.0, sigma_rgb=13.0, smoothness=1.0, sigma_smooth=3.0)


def size_of(img):
    """A PIL-like size stand-in for expand_words, for an image array [H, W, 3]."""
    h, w = int(img.shape[-3]), int(img.shape[-2])
    return SimpleNamespace(size=(w, h), height=h, width=w)


def make_image(h, w, seed):
    """A uint8 [h, w, 3] device image with edges: flat random-coloured blocks of random sizes plus a little noise."""
    g = torch.Generator().manual_seed(seed)
    by, bx = int(torch.randint(3, 40, (1,), generator=g)), int(torch.randint(3, 40, (1,), generator=g))
    blocks = torch.randint(0, 256, (h // by + 1, w // bx + 1, 3), generator=g).float()
    img = blocks.repeat_interleave(by, 0).repeat_interleave(bx, 1)[:h, :w]
    img = img + torch.randint(-6, 7, (h, w, 3), generator=g)
    return img.clamp(0, 255).to(torch.uint8).to(DEV)


def rand_maps(grid, seed, n_rows=102):
    return torch.rand(n_rows, *grid, generator=torch.Generator().manual_seed(seed)).to(DEV)


def word_list(n):
    """``n`` words of PROMPT100 with a two-token word and a repeated word."""
    words = [f'w{3 * i % 100}' for i in range(n)]
    if n >= 3:
        words[1] = 'w40 w41'
        words[-1] = words[0]
    return words


def bands(h, rows=12):
    """Output rows the float64 reference covers: all of a small image, else top, middle and bottom bands."""
    if h <= 3 * rows:
        return [(0, h)]
    mid = h // 2 - rows // 2
    return [(0, rows), (mid, mid + rows), (h - rows, h)]


def check_updates(ghm, words, img, radius, ks=(0, 2), threshold=None, absolute=False, scale=16.0, weights=WEIGHTS,
                  **kw):
    """Q_0 against softmax(z), and for each k in ks the update Q_k -> Q_{k+1} against crf_step64, within crf_bound;
    labels against the float64 argmax where its margin is safe; scores the Q of the label."""
    crf = dict(threshold=threshold, radius=radius, scale=scale, absolute=absolute, probs=True, to_cpu=False, **weights,
               **kw)
    _, m = ghm.expand_words(words, size_of(img), absolute=absolute, to_cpu=False,
                            **{k: v for k, v in kw.items() if k in ('word_idx', 'offset_idx')})
    z = logits64(m.cpu().numpy(), threshold, scale)
    n_labels, h, _ = z.shape
    off = 0 if threshold else 1
    tab = crf_tables(radius, **weights)
    image = img.cpu().numpy()
    prev = None
    for k in sorted(set(ks) | {0}):
        _, lab0, sc0, q0 = ghm.segment_crf(words, img, iterations=k, **crf)
        assert q0.shape == (n_labels,) + tuple(m.shape[1:]) and lab0.dtype == torch.uint8
        # scores are the Q of the label
        assert torch.equal(sc0, q0.gather(0, (lab0.long() - off)[None])[0])
        if k == 0:                                       # Q_0 = softmax(z): the softmax's own rounding only
            bound, _ = crf_bound(dict(t=z, mass=np.zeros_like(z)), radius)
            assert bool((np.abs(q0.cpu().numpy() - softmax64(z)) <= bound).all())
            assert torch.equal(lab0.cpu(), torch.from_numpy(z.argmax(0) + off).to(torch.uint8))
        if k not in ks:
            continue
        _, lab1, _, q1 = ghm.segment_crf(words, img, iterations=k + 1, **crf)
        q_k, q_next, lab_next = q0.cpu().numpy().astype(np.float64), q1.cpu().numpy(), lab1.cpu().numpy()
        for y0, y1 in bands(h):
            ref, parts = crf_step64(z, q_k, image, tab, radius, rows=(y0, y1), parts=True)
            bound, dt = crf_bound(parts, radius)
            err = np.abs(q_next[:, y0:y1] - ref)
            assert bool((err <= bound).all()), f'k={k} rows {y0}-{y1}: max error {err.max():.3e}, ' \
                                               f'worst ratio {(err / bound).max():.3f}'
            t = np.sort(parts['t'], 0)
            sure = t[-1] - t[-2] > 2 * dt if n_labels > 1 else np.ones(dt.shape, bool)
            want = parts['t'].argmax(0) + off
            assert np.array_equal(lab_next[y0:y1][sure], want[sure]), f'k={k} rows {y0}-{y1}'
        prev = q1
    return prev


# (map grid, output (h, w), radius, words, threshold, absolute): SD-2.1 512^2 and 768^2, SDXL 1024^2, SDXL 1216x832,
# off-grid 600x800
CASES = [((64, 64), (512, 512), 8, 8, 0.4, False), ((96, 96), (768, 768), 4, 1, None, False),
         ((128, 128), (1024, 1024), 16, 8, 0.4, True), ((76, 52), (1216, 832), 1, 8, None, False),
         ((75, 100), (600, 800), 8, 3, 0.4, False)]
CASE_IDS = [f'{g[0]}x{g[1]}-{h}x{w}-r{r}-{n}w' for g, (h, w), r, n, _, _ in CASES]


@pytest.mark.parametrize('case', range(len(CASES)), ids=CASE_IDS)
def test_sizes_against_float64(case):
    grid, hw, radius, n_words, threshold, absolute = CASES[case]
    maps = rand_maps(grid, 5 * grid[0] + grid[1])
    if absolute:
        maps = maps * 0.8                                # word values around the threshold
    ghm = GlobalHeatMap(TOK, PROMPT100, maps)
    check_updates(ghm, word_list(n_words), make_image(*hw, seed=case), radius, threshold=threshold, absolute=absolute)


@pytest.mark.parametrize('grid,hw,radius', [((8, 12), (20, 30), 16), ((5, 7), (9, 33), 16), ((12, 9), (40, 7), 8)],
                         ids=['20x30-r16', '9x33-r16', '40x7-r8'])
@pytest.mark.parametrize('threshold', [None, 0.5])
def test_radius_larger_than_the_image(grid, hw, radius, threshold):
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps(grid, radius))
    check_updates(ghm, word_list(3), make_image(*hw, seed=radius), radius, ks=(0, 1, 4), threshold=threshold)


@pytest.mark.parametrize('n_words', [1, 8, 96])
@pytest.mark.parametrize('threshold', [None, 0.3])
def test_word_counts(n_words, threshold):
    # 1 word without threshold is one label (Q = 1); 96 words with it are 97 labels in seven chunks
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((24, 20), n_words))
    check_updates(ghm, word_list(n_words), make_image(150, 130, n_words), 4, ks=(0, 3), threshold=threshold)


def test_weights_scale_and_word_selection():
    img = make_image(512, 512, 3)
    ghm = GlobalHeatMap(TOK, PROMPT, rand_maps((64, 64), 3, n_rows=11))
    check_updates(ghm, ['a', 'dog', 'a'], img, 8, ks=(1,), threshold=0.4, scale=32.0, word_idx=[None, None, 3])
    ghm100 = GlobalHeatMap(TOK, PROMPT100, rand_maps((64, 64), 4))
    check_updates(ghm100, ['w1', 'w10', 'w20 w21'], img, 4, ks=(1,), scale=0.5, offset_idx=2,
                  weights=dict(appearance=3.0, sigma_xy=2.5, sigma_rgb=40.0, smoothness=0.0, sigma_smooth=1.0))
    whms, lab, sc = ghm100.segment_crf(['w1', 'w10', 'w20 w21'], img.cpu(), radius=4, offset_idx=2)
    assert not lab.is_cuda and not sc.is_cuda and [w.word for w in whms] == ['w1', 'w10', 'w20 w21']
    _, lab_dev, sc_dev = ghm100.segment_crf(['w1', 'w10', 'w20 w21'], img, radius=4, offset_idx=2, to_cpu=False)
    assert torch.equal(lab, lab_dev.cpu()) and torch.equal(sc, sc_dev.cpu())


# ---- reduction to segment -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('threshold', [None, 0.4])
@pytest.mark.parametrize('scale', [16.0, 0.5])
def test_reduces_to_segment(threshold, scale):
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((76, 52), 7))
    img, words = make_image(1216, 832, 7), word_list(8)
    _, want, _ = ghm.segment(words, size_of(img), threshold=threshold, to_cpu=False)
    _, lab, _ = ghm.segment_crf(words, img, threshold=threshold, scale=scale, iterations=0, to_cpu=False)
    assert torch.equal(lab, want)
    _, lab, _ = ghm.segment_crf(words, img, threshold=threshold, scale=scale, iterations=3, appearance=0.0,
                                smoothness=0.0, to_cpu=False)
    assert torch.equal(lab, want)


def test_reduction_keeps_segments_tie_rules():
    # absolute constant maps: every word ties (the first wins), and at max m == threshold the background wins
    maps = torch.full((102, 16, 16), 0.4, device=DEV)
    maps[5] = 0.25
    ghm = GlobalHeatMap(TOK, PROMPT100, maps)
    img, words = make_image(64, 64, 1), ['w4', 'w1', 'w2', 'w1']
    for threshold in (None, 0.4, 0.3):
        _, want, _ = ghm.segment(words, size_of(img), absolute=True, threshold=threshold, to_cpu=False)
        for iterations, weights in ((0, {}), (2, dict(appearance=0.0, smoothness=0.0))):
            _, lab, _ = ghm.segment_crf(words, img, absolute=True, threshold=threshold, iterations=iterations,
                                        to_cpu=False, **weights)
            assert torch.equal(lab, want), (threshold, iterations)
    assert int(want.max()) == 2 and int(want.min()) == 2          # threshold 0.3: the first of the tied words


# ---- determinism, rounds and stacks ---------------------------------------------------------------------------------------
def test_repeated_calls_give_the_same_bits():
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((128, 128), 2))
    img, words = make_image(1024, 1024, 4), word_list(8)
    first = ghm.segment_crf(words, img, threshold=0.4, radius=16, probs=True, to_cpu=False)[1:]
    for _ in range(2):
        again = ghm.segment_crf(words, img, threshold=0.4, radius=16, probs=True, to_cpu=False)[1:]
        for a, b in zip(first, again):
            assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))


def check_stack(stack, words, img, **kw):
    word_maps, labels, scores, probs = stack.segment_crf(words, img, probs=True, to_cpu=False, **kw)
    n = len(stack)
    per_map = isinstance(img, (np.ndarray, torch.Tensor)) and img.ndim == 4
    assert tuple(labels.shape[:1]) == (n,) and tuple(word_maps.shape[:2]) == (n, len(words))
    for t in range(n):
        whms, lab, sc, q = stack[t].segment_crf(words, img[t] if per_map else img, probs=True, to_cpu=False, **kw)
        assert torch.equal(lab, labels[t]) and torch.equal(sc.view(torch.int32), scores[t].view(torch.int32)), t
        assert torch.equal(q.view(torch.int32), probs[t].view(torch.int32)), t
        for i, w in enumerate(whms):
            assert torch.equal(w.heatmap, word_maps[t, i])
    return labels


@pytest.mark.parametrize('maps_per_round', [1, 2])
@pytest.mark.parametrize('per_map', [False, True], ids=['one-image', 'image-per-map'])
def test_rounds_give_the_same_bits(monkeypatch, maps_per_round, per_map):
    maps = torch.stack([rand_maps((30, 50), 40 + t) for t in range(3)])
    stack = GlobalHeatMapStack(TOK, PROMPT100, maps)
    words = word_list(5)
    img = torch.stack([make_image(120, 200, 50 + t) for t in range(3)]) if per_map else make_image(120, 200, 50)
    crf = dict(threshold=0.4, radius=12, iterations=4, probs=True, to_cpu=False)
    before = _native.launch_count()
    one = stack.segment_crf(words, img, **crf)[1:]
    assert _native.launch_count() - before == 2 + 4               # the word maps, Q_0, one launch per update
    monkeypatch.setattr(heatmap, 'CRF_SCRATCH_BYTES', _native.crf_scratch_bytes(maps_per_round, 6, 120, 200))
    before = _native.launch_count()
    got = stack.segment_crf(words, img, **crf)[1:]
    assert _native.launch_count() - before == (2 if maps_per_round == 2 else 3) * 6    # rounds of whole maps
    for a, b in zip(one, got):
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))
    check_stack(stack, words, img, threshold=0.4, radius=12, iterations=4)


def test_time_image_and_layer_stacks():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=5)
    img = make_image(512, 512, 2)
    words = ['dog', 'red ball', 'beach', 'dog']
    with trace(pipe, time_resolved=True) as tc:
        pipe(PROMPT, num_inference_steps=4, generator=torch.Generator().manual_seed(3))
        tm = tc.compute_time_heat_maps()
        assert len(tm) == 4
        check_stack(tm, words, img, threshold=0.4)
        check_stack(tm, words, img, absolute=True, radius=3, iterations=2)
        layers = tc.compute_layer_heat_maps()
        assert len(layers) > 1
        check_stack(layers, words, img, radius=16, threshold=0.4)
        check_updates(tm[2], words, img, 8, ks=(1,), threshold=0.4)
    with trace(pipe) as tc:
        pipe(PROMPT, num_inference_steps=2, generator=torch.Generator().manual_seed(11), num_images_per_prompt=3)
        per_image = tc.compute_image_heat_maps()
        images = torch.stack([make_image(512, 512, 20 + i) for i in range(3)])
        check_stack(per_image, ['dog', 'ball', 'beach'], images, threshold=0.4)
        check_stack(per_image, ['dog', 'ball'], images.cpu().numpy())


# ---- quality: shapes with sharp edges --------------------------------------------------------------------------------------
def shape_scene(h, w, seed):
    """Flat-coloured shapes with sharp edges on a flat background, a little noise: ``(image [h, w, 3] uint8, masks
    [3, h, w] bool)``, a disc, a rectangle and a triangle."""
    g = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    masks = np.stack([(yy - 0.35 * h) ** 2 + (xx - 0.3 * w) ** 2 <= (0.18 * min(h, w)) ** 2,
                      (yy >= 0.55 * h) & (yy < 0.85 * h) & (xx >= 0.45 * w) & (xx < 0.9 * w),
                      (yy >= 0.12 * h) & (yy < 0.45 * h) & (xx >= 0.55 * w) & (yy - 0.12 * h < 0.8 * (xx - 0.55 * w))])
    img = np.zeros((h, w, 3), np.int64) + g.integers(0, 256, 3)
    for m in masks:
        img[m] = g.integers(0, 256, 3)
    img = np.clip(img + g.integers(-4, 5, (h, w, 3)), 0, 255).astype(np.uint8)
    return torch.from_numpy(img).to(DEV), torch.from_numpy(masks).to(DEV)


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_defaults_beat_segment_on_sharp_shapes(seed):
    img, masks = shape_scene(512, 512, seed)
    # each word's heat map is its shape's mask area-averaged onto the 64 x 64 grid: smeared by expansion
    maps = torch.zeros(102, 64, 64, device=DEV)
    maps[1:4] = torch.nn.functional.avg_pool2d(masks.float()[None], 8)[0]
    ghm = GlobalHeatMap(TOK, PROMPT100, maps)
    words = ['w0', 'w1', 'w2']
    _, seg, _ = ghm.segment(words, size_of(img), threshold=0.4, to_cpu=False)
    _, crf, _ = ghm.segment_crf(words, img, threshold=0.4, to_cpu=False)

    def iou(lab):
        pred = torch.stack([lab == w + 1 for w in range(3)])
        return ((pred & masks).flatten(1).sum(1) / (pred | masks).flatten(1).sum(1)).cpu()

    def f_score(lab):
        pred = torch.stack([lab == w + 1 for w in range(3)])
        # tolerance 0: exact boundary pixels (at 2 px the smeared boundary of a large shape already scores 1)
        return boundary_scores(pred, masks, tolerances=[0.0]).f_score()[0].diagonal()

    iou_seg, iou_crf, f_seg, f_crf = iou(seg), iou(crf), f_score(seg), f_score(crf)
    assert bool((iou_crf > iou_seg).all()), (iou_seg, iou_crf)
    assert bool((f_crf > f_seg).all()), (f_seg, f_crf)


# ---- the C ABI -------------------------------------------------------------------------------------------------------------
def _abi_call(grid=(16, 16), out_hw=(72, 40), n_words=1, n_maps=1, radius=4, iterations=2, scale=16.0, appearance=1.0,
              sigma_xy=3.0, sigma_rgb=13.0, smoothness=1.0, sigma_smooth=3.0, use_threshold=1, threshold=0.4,
              scratch_bytes=None, scratch_offset=0, null=None, stride=0):
    """daam_segment_crf on one real map and word (the buffers of one, or of one pixel past the pixel limit: a refused
    call reads none of them); returns (status, message, labels)."""
    small = out_hw[0] * out_hw[1] <= 1 << 22
    maps = rand_maps(grid, 5)
    word_maps = torch.empty((1, max(n_words, 1)) + grid, device=DEV)
    shape = out_hw if small else (1, 1)
    image = torch.zeros(shape + (3,), dtype=torch.uint8, device=DEV)
    labels = torch.full(shape, 255, dtype=torch.uint8, device=DEV)
    scores = torch.full(shape, float('nan'), device=DEV)
    n_labels = n_words + (1 if use_threshold else 0)
    need = _native.crf_scratch_bytes(1, n_labels, *out_hw) if small else 1 << 62
    scratch = torch.empty((need if small else 0) + 16, dtype=torch.uint8, device=DEV)
    ptrs = {'maps': maps.data_ptr(), 'word_maps': word_maps.data_ptr(), 'image': image.data_ptr(),
            'labels': labels.data_ptr(), 'scores': scores.data_ptr(), 'scratch': scratch.data_ptr() + scratch_offset}
    if null:
        ptrs[null] = 0
    rows = (ctypes.c_int32 * n_words)(*range(1, n_words + 1))
    begin = (ctypes.c_int32 * (n_words + 1))(*range(n_words + 1))
    vp = ctypes.c_void_p
    rc = _native.load().daam_segment_crf(vp(ptrs['maps']), n_maps, 102, grid[0], grid[1], rows, begin, n_words,
                                         out_hw[0], out_hw[1], 0, use_threshold, threshold, scale, iterations, radius,
                                         appearance, sigma_xy, sigma_rgb, smoothness, sigma_smooth,
                                         vp(ptrs['word_maps']), vp(ptrs['image']), stride, vp(ptrs['labels']),
                                         vp(ptrs['scores']), None, vp(ptrs['scratch']),
                                         need if scratch_bytes is None else scratch_bytes,
                                         vp(torch.cuda.current_stream().cuda_stream))
    msg = _native.load().daam_last_error().decode() if rc else ''
    return rc, msg, labels


def test_abi_statuses():
    rc, _, labels = _abi_call()
    torch.cuda.synchronize()
    assert rc == 0 and int(labels.max()) <= 1
    for kw in (dict(radius=16, iterations=64), dict(iterations=0), dict(appearance=0.0, smoothness=0.0),
               dict(use_threshold=0, threshold=float('nan'))):
        assert _abi_call(**kw)[0] == 0, kw
    inf, nan = float('inf'), float('nan')
    for kw, status, text in [
            (dict(radius=0), _native.E_INVALID, 'radius 0 is not in [1, 16]'),
            (dict(radius=17), _native.E_INVALID, 'radius 17 is not in [1, 16]'),
            (dict(iterations=-1), _native.E_INVALID, 'iterations -1 is not in [0, 64]'),
            (dict(iterations=65), _native.E_INVALID, 'iterations 65 is not in [0, 64]'),
            (dict(scale=0.0), _native.E_INVALID, 'scale'),
            (dict(scale=inf), _native.E_INVALID, 'scale'),
            (dict(sigma_xy=-1.0), _native.E_INVALID, 'sigma_xy'),
            (dict(sigma_rgb=nan), _native.E_INVALID, 'sigma_rgb'),
            (dict(sigma_smooth=0.0), _native.E_INVALID, 'sigma_smooth'),
            (dict(appearance=-1.0), _native.E_INVALID, 'appearance'),
            (dict(smoothness=inf), _native.E_INVALID, 'smoothness'),
            (dict(threshold=inf), _native.E_INVALID, 'threshold inf is not finite'),
            (dict(scratch_bytes=_native.crf_scratch_bytes(1, 2, 72, 40) - 1), _native.E_INVALID, 'scratch bytes'),
            (dict(scratch_offset=2), _native.E_INVALID, '4-byte aligned'),
            (dict(null='image'), _native.E_INVALID, 'null pointer'),
            (dict(null='labels'), _native.E_INVALID, 'null pointer'),
            (dict(null='scores'), _native.E_INVALID, 'null pointer'),
            (dict(null='scratch'), _native.E_INVALID, 'null pointer'),
            (dict(stride=-1), _native.E_INVALID, 'null pointer'),
            (dict(n_words=97), _native.E_UNSUPPORTED, '97 words > 96'),
            (dict(n_maps=65536), _native.E_UNSUPPORTED, '65536 maps > 65535'),
            (dict(out_hw=(32768, 32769)), _native.E_UNSUPPORTED, 'more than 2^30 pixels'),
            # the checks' order: null pointers, then the CRF arguments, then scratch, then the word list
            (dict(null='image', radius=0), _native.E_INVALID, 'null pointer'),
            (dict(radius=0, iterations=-1), _native.E_INVALID, 'radius'),
            (dict(iterations=-1, scale=0.0), _native.E_INVALID, 'iterations'),
            (dict(sigma_smooth=0.0, appearance=-1.0), _native.E_INVALID, 'sigma_smooth'),
            (dict(smoothness=-1.0, threshold=inf), _native.E_INVALID, 'smoothness'),
            (dict(threshold=inf, scratch_bytes=8), _native.E_INVALID, 'threshold'),
            (dict(scratch_bytes=8, n_words=97), _native.E_INVALID, 'scratch bytes')]:
        rc, msg, _ = _abi_call(**kw)
        assert rc == status and text in msg, (kw, rc, msg)
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((16, 16), 5))
    with pytest.raises(_native.NativeError, match='97 words > 96'):
        ghm.segment_crf([f'w{i}' for i in range(97)], make_image(72, 72, 1))
