"""Edge-aware word maps (GlobalHeatMap.refine_words / GlobalHeatMapStack.refine_words, daam_refine_words) on the GPU,
against tests/refine64.py over the very values expand_words(..., to_cpu=False) returns.

* Every element within refine_bound: the fp32 error of window means over at most 2r + 1 + 2r + 1 terms, propagated
  through c, a = (Sigma + eps Id)^-1 c (scaled by sqrt(3) / eps >= ||(Sigma + eps Id)^-1||_inf), b and q, from the
  plane's max |m|, |a|, |b|, |c| -- see refine64.refine_bound.
* SD-2.1 512^2 and 768^2, SDXL 1024^2, 1216x832 and off-grid 600x800 outputs; radii 1, 8, 32, 64 and larger than the
  image; eps 1e-4, 1e-2 and 1; normalised and absolute maps; 1, 8 and 96 words, word_idx and offset_idx.
* Every launch geometry of refine.cu: a row segment of 256 outputs with its halo clipped on one, both or no sides, a
  last segment 1 column wide, 1-pixel-wide and 1-pixel-tall outputs, column tiles of 64 rows with a last tile 1 row
  tall, and rounds of one plane, of split words and of several maps, with one image or one per map.
* A thresholded call equals refined > t bit for bit; time, image (one image per map) and layer stacks equal the per-map
  calls bit for bit; several rounds equal one round; repeated calls give the same bits.
* The C ABI's statuses.
"""
import ctypes
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from daam_b200 import _native, heatmap, trace
from daam_b200.heatmap import GlobalHeatMap, GlobalHeatMapStack
from daam_b200.testing.synthetic import TINY_SPEC, WhitespaceTokenizer, make_pipeline
from tests.refine64 import refine64, refine_bound

pytestmark = pytest.mark.gpu
DEV = 'cuda'
TOK = WhitespaceTokenizer()
PROMPT100 = ' '.join(f'w{i}' for i in range(100))
PROMPT = 'a dog chasing a red ball on the beach'
EPS = (1e-4, 1e-2, 1.0)


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


def check_refine(ghm, words, img, radius, eps, absolute=False, **kw):
    """refine_words against refine64 of expand_words' values within refine_bound; returns the device result."""
    _, got = ghm.refine_words(words, img, radius=radius, eps=eps, absolute=absolute, to_cpu=False, **kw)
    _, m = ghm.expand_words(words, size_of(img), absolute=absolute, to_cpu=False, **kw)
    assert got.dtype == torch.float32 and got.is_cuda and tuple(got.shape) == tuple(m.shape)
    e32 = float(np.float32(eps))
    m64 = m.cpu().numpy().astype(np.float64)
    q, parts = refine64(m64, img.cpu().numpy(), radius, e32, parts=True)
    bound = refine_bound(m64, parts, radius, e32)
    err = np.abs(got.cpu().numpy() - q)
    assert bool(np.isfinite(got.cpu().numpy()).all())
    assert bool((err <= bound).all()), f'max error {err.max():.3e}, bound {bound.min():.3e}'
    return got


# (map grid, output (h, w)): SD-2.1 512^2 and 768^2, SDXL 1024^2, SDXL 1216x832, off-grid 600x800
PAIRS = [((64, 64), (512, 512)), ((96, 96), (768, 768)), ((128, 128), (1024, 1024)), ((76, 52), (1216, 832)),
         ((75, 100), (600, 800))]
PAIR_IDS = [f'{g[0]}x{g[1]}-{h}x{w}' for g, (h, w) in PAIRS]
RADII = (1, 8, 32, 64)


@pytest.mark.parametrize('radius', RADII)
@pytest.mark.parametrize('pair', range(len(PAIRS)), ids=PAIR_IDS)
def test_sizes_against_float64(pair, radius):
    (grid, hw), k = PAIRS[pair], pair + RADII.index(radius)
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps(grid, 5 * grid[0] + grid[1]))
    check_refine(ghm, word_list(4), make_image(*hw, seed=k), radius, EPS[k % 3], absolute=bool(k % 2))


@pytest.mark.parametrize('eps', EPS)
@pytest.mark.parametrize('grid,hw,radius', [((8, 8), (48, 48), 64), ((5, 7), (30, 50), 40), ((12, 9), (70, 33), 64)],
                         ids=['48x48-r64', '30x50-r40', '70x33-r64'])
def test_radius_larger_than_the_image(grid, hw, radius, eps):
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps(grid, radius))
    for absolute in (False, True):
        check_refine(ghm, word_list(3), make_image(*hw, seed=radius), radius, eps, absolute=absolute)


@pytest.mark.parametrize('n_words', [1, 8, 96])
def test_word_counts(n_words):
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((24, 20), n_words))
    check_refine(ghm, word_list(n_words), make_image(150, 130, n_words), 8, 1e-2)


def test_word_idx_offset_idx_and_cpu_result():
    ghm = GlobalHeatMap(TOK, PROMPT, rand_maps((64, 64), 3, n_rows=11))
    img = make_image(512, 512, 3)
    check_refine(ghm, ['a', 'dog', 'a'], img, 8, 1e-3, word_idx=[None, None, 3])
    ghm100 = GlobalHeatMap(TOK, PROMPT100, rand_maps((64, 64), 4))
    got = check_refine(ghm100, ['w1', 'w10', 'w20 w21'], img, 4, 1e-3, offset_idx=2)
    whms, cpu = ghm100.refine_words(['w1', 'w10', 'w20 w21'], img.cpu(), radius=4, eps=1e-3, offset_idx=2)
    assert not cpu.is_cuda and torch.equal(cpu, got.cpu())
    assert [w.word for w in whms] == ['w1', 'w10', 'w20 w21']


def test_constant_map_and_constant_image():
    img = make_image(256, 256, 1)
    # a constant m (absolute, every row 0.25): c = 0, a = 0, b = 0.25, q = 0.25 up to the window sums' rounding
    ghm = GlobalHeatMap(TOK, PROMPT100, torch.full((102, 32, 32), 0.25, device=DEV))
    q = check_refine(ghm, word_list(2), img, 16, 1e-4, absolute=True)
    assert float((q - 0.25).abs().max()) < 1e-5
    # a constant image: Sigma = 0, a = c / eps, and q = mean(mean(m))
    flat = torch.full((256, 256, 3), 77, dtype=torch.uint8, device=DEV)
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((32, 32), 2))
    check_refine(ghm, word_list(2), flat, 16, 1e-2)


@pytest.mark.parametrize('threshold', [0.3, 0.5])
def test_threshold_is_refined_above_t(threshold):
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((76, 52), 9))
    img = make_image(1216, 832, 9)
    words = word_list(5)
    _, q = ghm.refine_words(words, img, radius=8, eps=1e-3, to_cpu=False)
    _, t = ghm.refine_words(words, img, radius=8, eps=1e-3, threshold=threshold, to_cpu=False)
    assert torch.equal(t, (q > threshold).float())
    _, t0 = ghm.refine_words(words, img, radius=8, eps=1e-3, threshold=0, to_cpu=False)   # 0: no threshold
    assert torch.equal(t0, q)


# ---- launch geometry: row segments of 256 outputs, column tiles of 64 rows, rounds -------------------------------------
@pytest.mark.parametrize('grid,hw,radius', [
    ((9, 7), (65, 257), 1),      # last row segment 1 column wide, last column tile 1 row tall
    ((9, 7), (129, 513), 64),    # 3 segments, the middle one's halo unclipped on both sides
    ((5, 40), (1, 300), 3),      # one output row
    ((40, 5), (300, 1), 3),      # one output column
    ((5, 5), (1, 1), 64),        # one pixel
    ((30, 50), (64, 256), 64),   # one segment and one tile exactly
    ((30, 50), (200, 700), 17),  # halos clipped at the image edges only
], ids=['65x257', '129x513', '1x300', '300x1', '1x1', '64x256', '200x700'])
def test_geometry(grid, hw, radius):
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps(grid, hw[0] + hw[1]))
    for absolute in (False, True):
        check_refine(ghm, word_list(3), make_image(*hw, seed=radius), radius, 1e-2, absolute=absolute)


def check_stack(stack, words, img, **kw):
    word_maps, refined = stack.refine_words(words, img, to_cpu=False, **kw)
    n = len(stack)
    per_map = isinstance(img, (np.ndarray, torch.Tensor)) and img.ndim == 4
    assert tuple(refined.shape[:2]) == (n, len(words)) and tuple(word_maps.shape[:2]) == (n, len(words))
    for t in range(n):
        whms, one = stack[t].refine_words(words, img[t] if per_map else img, to_cpu=False, **kw)
        assert torch.equal(one.view(torch.int32), refined[t].view(torch.int32)), t
        for i, w in enumerate(whms):
            assert torch.equal(w.heatmap, word_maps[t, i])
    return refined


@pytest.mark.parametrize('planes', [1, 2, 3, 7])
@pytest.mark.parametrize('per_map', [False, True], ids=['one-image', 'image-per-map'])
def test_rounds_give_the_same_bits(monkeypatch, planes, per_map):
    maps = torch.stack([rand_maps((30, 50), 40 + t) for t in range(3)])
    stack = GlobalHeatMapStack(TOK, PROMPT100, maps)
    words = word_list(5)
    img = torch.stack([make_image(120, 200, 50 + t) for t in range(3)]) if per_map else make_image(120, 200, 50)
    before = _native.launch_count()
    _, one = stack.refine_words(words, img, radius=12, eps=1e-3, to_cpu=False)
    assert _native.launch_count() - before == 2 + 5            # the statistics, then every plane in one round
    monkeypatch.setattr(heatmap, 'REFINE_SCRATCH_BYTES',
                        _native.refine_scratch_bytes(1, planes, 120, 200) if not per_map else
                        _native.refine_scratch_bytes(max(1, planes // 5), planes, 120, 200))
    _, got = stack.refine_words(words, img, radius=12, eps=1e-3, to_cpu=False)
    assert torch.equal(got.view(torch.int32), one.view(torch.int32))
    # each map's planes, one call per map, are the same bits too
    check_stack(stack, words, img, radius=12, eps=1e-3)


def test_repeated_calls_give_the_same_bits():
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((128, 128), 2))
    img, words = make_image(1024, 1024, 4), word_list(8)
    _, a = ghm.refine_words(words, img, radius=32, eps=1e-3, to_cpu=False)
    for _ in range(2):
        _, b = ghm.refine_words(words, img, radius=32, eps=1e-3, to_cpu=False)
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_time_image_and_layer_stacks():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=5)
    img = make_image(512, 512, 2)
    words = ['dog', 'red ball', 'beach', 'dog']
    with trace(pipe, time_resolved=True) as tc:
        pipe(PROMPT, num_inference_steps=4, generator=torch.Generator().manual_seed(3))
        tm = tc.compute_time_heat_maps()
        assert len(tm) == 4
        check_stack(tm, words, img)
        check_stack(tm, words, img, absolute=True, radius=3, eps=1e-2, threshold=0.4)
        layers = tc.compute_layer_heat_maps()
        assert len(layers) > 1
        check_stack(layers, words, img, radius=16)
        check_refine(tm[2], words, img, 8, 1e-3)
    with trace(pipe) as tc:
        pipe(PROMPT, num_inference_steps=2, generator=torch.Generator().manual_seed(11), num_images_per_prompt=3)
        per_image = tc.compute_image_heat_maps()
        images = torch.stack([make_image(512, 512, 20 + i) for i in range(3)])
        check_stack(per_image, ['dog', 'ball', 'beach'], images, radius=8, eps=1e-3)
        check_stack(per_image, ['dog', 'ball'], images.cpu().numpy())


# ---- the C ABI -------------------------------------------------------------------------------------------------------------
def _abi_call(grid=(16, 16), out_hw=(72, 40), n_words=1, n_maps=1, radius=4, eps=1e-2, scratch_bytes=None,
              scratch_offset=0, null=None, stride=0):
    """daam_refine_words on one real map and word (the buffers of one, or of one pixel past the pixel limit: a refused
    call reads none of them); returns (status, message, out)."""
    small = out_hw[0] * out_hw[1] <= 1 << 22
    maps = rand_maps(grid, 5)
    word_maps = torch.empty((1, max(n_words, 1)) + grid, device=DEV)
    image = torch.zeros((out_hw if small else (1, 1)) + (3,), dtype=torch.uint8, device=DEV)
    out = torch.full((1, 1) + (out_hw if small else (1, 1)), float('nan'), device=DEV)
    need = _native.refine_scratch_bytes(1, 1, *out_hw) if small else 1 << 62
    scratch = torch.empty((need if small else 0) + 16, dtype=torch.uint8, device=DEV)
    ptrs = {'maps': maps.data_ptr(), 'word_maps': word_maps.data_ptr(), 'image': image.data_ptr(),
            'out': out.data_ptr(), 'scratch': scratch.data_ptr() + scratch_offset}
    if null:
        ptrs[null] = 0
    rows = (ctypes.c_int32 * n_words)(*range(1, n_words + 1))
    begin = (ctypes.c_int32 * (n_words + 1))(*range(n_words + 1))
    vp = ctypes.c_void_p
    rc = _native.load().daam_refine_words(vp(ptrs['maps']), n_maps, 102, grid[0], grid[1], rows, begin, n_words,
                                          out_hw[0], out_hw[1], 0, 0, 0.0, radius, eps, vp(ptrs['word_maps']),
                                          vp(ptrs['image']), stride, vp(ptrs['out']), vp(ptrs['scratch']),
                                          need if scratch_bytes is None else scratch_bytes,
                                          vp(torch.cuda.current_stream().cuda_stream))
    msg = _native.load().daam_last_error().decode() if rc else ''
    return rc, msg, out


def test_abi_statuses():
    rc, _, out = _abi_call()
    torch.cuda.synchronize()
    assert rc == 0 and bool(torch.isfinite(out).all())
    rc, _, out = _abi_call(radius=64, eps=1e-4)
    assert rc == 0
    for kw, status, text in [
            (dict(radius=0), _native.E_INVALID, 'radius 0 is not in [1, 64]'),
            (dict(radius=65), _native.E_INVALID, 'radius 65 is not in [1, 64]'),
            (dict(eps=0.0), _native.E_INVALID, 'eps'),
            (dict(eps=-1.0), _native.E_INVALID, 'eps'),
            (dict(eps=float('inf')), _native.E_INVALID, 'eps'),
            (dict(eps=float('nan')), _native.E_INVALID, 'eps'),
            (dict(scratch_bytes=_native.refine_scratch_bytes(1, 1, 72, 40) - 1), _native.E_INVALID, 'scratch bytes'),
            (dict(scratch_offset=2), _native.E_INVALID, '4-byte aligned'),
            (dict(null='image'), _native.E_INVALID, 'null pointer'),
            (dict(null='out'), _native.E_INVALID, 'null pointer'),
            (dict(null='scratch'), _native.E_INVALID, 'null pointer'),
            (dict(stride=-1), _native.E_INVALID, 'null pointer'),
            (dict(n_words=97), _native.E_UNSUPPORTED, '97 words > 96'),
            (dict(n_maps=65536), _native.E_UNSUPPORTED, '65536 maps > 65535'),
            (dict(out_hw=(32768, 32769)), _native.E_UNSUPPORTED, 'more than 2^30 pixels'),
            # the checks' order: null pointers, then radius, then eps, then scratch, then the word list
            (dict(null='image', radius=0), _native.E_INVALID, 'null pointer'),
            (dict(radius=0, eps=0.0), _native.E_INVALID, 'radius'),
            (dict(eps=0.0, scratch_bytes=8), _native.E_INVALID, 'eps'),
            (dict(scratch_bytes=8, n_words=97), _native.E_INVALID, 'scratch bytes')]:
        rc, msg, _ = _abi_call(**kw)
        assert rc == status and text in msg, (kw, rc, msg)
    ghm = GlobalHeatMap(TOK, PROMPT100, rand_maps((16, 16), 5))
    with pytest.raises(_native.NativeError, match='97 words > 96'):
        ghm.refine_words([f'w{i}' for i in range(97)], make_image(72, 72, 1))
