"""Heat-map overlays (GlobalHeatMap.overlay_words / GlobalHeatMapStack.overlay_words, daam_overlay_words) on the GPU.

* Byte equality with the torch composition of expand_words output (tests/overlay_ref.py) over square, rectangular,
  SDXL, off-grid and down-sampled sizes, widths whose rows are not 4-byte aligned, colour normalisation on and off,
  absolute on and off, thresholds None / 0 / 0.4, 1 / 8 / 96 words and random, black and white images.
* The table daam_jet_colormap returns against the float64 restatement, every colour index, constant maps.
* Stacks: a shared image and one image per map, row by row against the single-map call; tracer histories and per-image
  maps; determinism; every limit and one past it through the C ABI.
"""
import numpy as np
import pytest
import torch
from PIL import Image

from daam_b200 import _native, trace
from daam_b200.heatmap import GlobalHeatMap, GlobalHeatMapStack, jet_colormap
from daam_b200.testing.synthetic import TINY_SPEC, WhitespaceTokenizer, make_pipeline
from tests.overlay_ref import color_index, jet_table, overlay_reference
from tests.test_segment_gpu import PAIRS, TINY_XL, synthetic_map, word_list

pytestmark = pytest.mark.gpu
DEV = 'cuda'
TOK = WhitespaceTokenizer()
PROMPT100 = ' '.join(f'w{i}' for i in range(100))
PROMPT = 'a dog chasing a red ball on the beach'
THRESHOLDS = (None, 0, 0.4)
TABLE = jet_table()
# rows of 3 * out_w bytes that are not a multiple of 4: tiles end inside a 4-byte word
ODD = [((64, 64), (97, 97)), ((30, 50), (61, 101)), ((96, 64), (95, 63)), ((64, 64), (1, 1)), ((16, 16), (7, 7))]


def out_size(grid, hw):
    return (hw[1], hw[0]) if grid[0] == grid[1] else hw


def make_image(kind, h, w, seed=0):
    if kind == 'zeros':
        return np.zeros((h, w, 3), dtype=np.uint8)
    if kind == 'white':
        return Image.new('RGB', (w, h), (255, 255, 255))
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (h, w, 3), generator=g, dtype=torch.uint8).to(DEV)


def as_tensor(img):
    if isinstance(img, torch.Tensor):
        return img
    return torch.from_numpy(np.array(img.convert('RGB') if hasattr(img, 'convert') else img))


def check_against_reference(ghm, words, img, idx=None, what=''):
    """overlay_words == overlay_reference(expand_words(...)) for every colour, absolute and threshold form."""
    im = as_tensor(img).to(DEV)
    for absolute in (False, True):
        for t in THRESHOLDS:
            whms_e, m = ghm.expand_words(words, img_size(im), absolute=absolute, threshold=t, word_idx=idx,
                                         to_cpu=False)
            for cn in (True, False):
                whms, frames = ghm.overlay_words(words, img, absolute=absolute, threshold=t, color_normalize=cn,
                                                 word_idx=idx, to_cpu=False)
                assert frames.dtype == torch.uint8 and frames.is_cuda
                assert tuple(frames.shape) == tuple(m.shape) + (3,)
                want = overlay_reference(m, im, cn, TABLE)
                assert torch.equal(frames, want), \
                    f'{what} abs={absolute} t={t} cn={cn}: {int((frames != want).sum())} bytes differ'
                assert [w.word for w in whms] == [w.word for w in whms_e]
                for a, b in zip(whms, whms_e):
                    assert torch.equal(a.heatmap, b.heatmap)


def img_size(im):
    """A PIL-like size stand-in for expand_words, for an image array [H, W, 3]."""
    from types import SimpleNamespace
    h, w = im.shape[0], im.shape[1]
    return SimpleNamespace(size=(w, h), height=h, width=w)


@pytest.mark.parametrize('kind', ['random', 'zeros', 'white'])
@pytest.mark.parametrize('n_words', [1, 8, 96])
@pytest.mark.parametrize('grid,hw', PAIRS + ODD, ids=[f'{g[0]}x{g[1]}-{h}x{w}' for g, (h, w) in PAIRS + ODD])
def test_against_reference(grid, hw, n_words, kind):
    ghm = GlobalHeatMap(TOK, PROMPT100, synthetic_map(grid, n_words + 7 * grid[0] + grid[1]))
    words, idx = word_list(n_words)
    if grid[0] == grid[1] and hw[0] != hw[1]:
        # a square map expands to (image.size[0], image.size[1]): over a non-square image that transposes it
        with pytest.raises(ValueError, match='transposes'):
            ghm.overlay_words(words, make_image(kind, *hw), word_idx=idx)
        return
    img = make_image(kind, *out_size(grid, hw), seed=n_words)
    check_against_reference(ghm, words, img, idx, what=f'{grid} {hw} {n_words} {kind}')


def test_offset_idx_and_cpu_frames():
    ghm = GlobalHeatMap(TOK, PROMPT100, synthetic_map((64, 64), 3))
    img = make_image('random', 512, 512, 4)
    whms, frames = ghm.overlay_words(['w1', 'w10', 'w20 w21'], img.cpu(), offset_idx=2)
    assert not frames.is_cuda
    _, m = ghm.expand_words(['w1', 'w10', 'w20 w21'], img_size(img), offset_idx=2, to_cpu=False)
    assert torch.equal(frames, overlay_reference(m, img, True, TABLE).cpu())


# ---- the table -----------------------------------------------------------------------------------------------------------
def test_table_is_the_float64_restatement():
    got = jet_colormap()
    assert got.dtype == torch.float32 and tuple(got.shape) == (256, 3)
    assert torch.equal(got.view(torch.int32), TABLE.view(torch.int32))


def test_every_colour_index():
    # a linear ramp along x: the expanded, normalised map sweeps [0, 1] in steps far below 1 / 256
    ramp = torch.linspace(0, 1, 64).expand(64, 64)
    maps = torch.rand(4, 64, 64, generator=torch.Generator().manual_seed(0))
    maps[1] = ramp
    ghm = GlobalHeatMap(TOK, 'a b', maps.to(DEV))
    img = make_image('random', 1024, 1024, 1)
    for cn in (True, False):
        _, m = ghm.expand_words(['a'], img_size(img), to_cpu=False)
        assert color_index(m, cn).unique().numel() == 256
        _, frames = ghm.overlay_words(['a'], img, color_normalize=cn, to_cpu=False)
        assert torch.equal(frames, overlay_reference(m, img, cn, TABLE))


def test_constant_maps():
    img = make_image('random', 512, 512, 2)
    # an all-zero map: v = 0 everywhere, so m = 0, hi == lo (c = 0) and alpha 0: the image itself
    ghm = GlobalHeatMap(TOK, 'a b', torch.zeros(4, 64, 64, device=DEV))
    for absolute in (False, True):
        _, frames = ghm.overlay_words(['a'], img, absolute=absolute, to_cpu=False)
        assert torch.equal(frames[0], img)
    # a thresholded map above the threshold everywhere: m = 1, hi == lo, colour 0 at alpha 1
    ghm = GlobalHeatMap(TOK, 'a b', torch.full((4, 64, 64), 0.7, device=DEV))
    _, frames = ghm.overlay_words(['a'], img, absolute=True, threshold=0.4, to_cpu=False)
    _, m = ghm.expand_words(['a'], img_size(img), absolute=True, threshold=0.4, to_cpu=False)
    assert bool((m == 1).all())
    assert torch.equal(frames, overlay_reference(m, img, True, TABLE))
    assert bool((frames[0] == torch.tensor([0, 0, 128], dtype=torch.uint8, device=DEV)).all())


# ---- stacks --------------------------------------------------------------------------------------------------------------
def check_stack(stack, words, img, **kw):
    before = _native.launch_count()
    word_maps, frames = stack.overlay_words(words, img, to_cpu=False, **kw)
    assert _native.launch_count() - before == 2                    # the whole stack
    n = len(stack)
    per_map = isinstance(img, (np.ndarray, torch.Tensor)) and img.ndim == 4
    assert tuple(frames.shape[:2]) == (n, len(words)) and tuple(word_maps.shape[:2]) == (n, len(words))
    for t in range(n):
        whms, one = stack[t].overlay_words(words, img[t] if per_map else img, to_cpu=False, **kw)
        assert torch.equal(one, frames[t]), t
        for i, w in enumerate(whms):
            assert torch.equal(w.heatmap, word_maps[t, i])
    return frames


@pytest.mark.parametrize('grid,hw', [((64, 64), (512, 512)), ((76, 52), (1216, 832)), ((30, 50), (61, 101))],
                         ids=['512', '1216x832', 'odd'])
def test_synthetic_stack(grid, hw):
    maps = torch.stack([synthetic_map(grid, 40 + t) for t in range(5)])
    stack = GlobalHeatMapStack(TOK, PROMPT100, maps)
    words, idx = word_list(8)
    h, w = out_size(grid, hw)
    shared = make_image('random', h, w, 5)
    per_map = torch.randint(0, 256, (5, h, w, 3), generator=torch.Generator().manual_seed(6), dtype=torch.uint8)
    for absolute, threshold, cn in ((False, None, True), (True, 0.4, True), (False, 0.4, False), (True, None, False)):
        check_stack(stack, words, shared, absolute=absolute, threshold=threshold, color_normalize=cn, word_idx=idx)
        check_stack(stack, words, per_map, absolute=absolute, threshold=threshold, color_normalize=cn, word_idx=idx)
        check_stack(stack, words, per_map.numpy(), absolute=absolute, threshold=threshold, color_normalize=cn,
                    word_idx=idx)


def test_determinism():
    maps = torch.stack([synthetic_map((96, 64), 50 + t) for t in range(3)])
    stack = GlobalHeatMapStack(TOK, PROMPT100, maps)
    words, idx = word_list(96)
    img = make_image('random', 95, 63, 7)
    _, a = stack.overlay_words(words, img, word_idx=idx, to_cpu=False)
    for _ in range(3):
        _, b = stack.overlay_words(words, img, word_idx=idx, to_cpu=False)
        assert torch.equal(a, b)


@pytest.mark.parametrize('spec,hw', [(TINY_SPEC, (512, 512)), (TINY_SPEC, (512, 768)), (TINY_XL, (1216, 832))],
                         ids=['512', '512x768', 'xl-1216x832'])
def test_time_resolved_history(spec, hw):
    pipe = make_pipeline(spec, dtype=torch.float16, device=DEV, seed=5)
    img = make_image('random', *hw, seed=8)
    with trace(pipe, time_resolved=True, negative=True) as tc:
        pipe(PROMPT, num_inference_steps=4, generator=torch.Generator().manual_seed(3), height=hw[0], width=hw[1],
             negative_prompt='blurry grainy dark photo')
        tm = tc.compute_time_heat_maps()
        assert len(tm) == 4
        for absolute, threshold in ((False, None), (False, 0.4), (True, 0.4)):
            check_stack(tm, ['dog', 'red ball', 'beach', 'dog'], img, absolute=absolute, threshold=threshold)
        neg = tc.compute_time_heat_maps(negative=True)
        check_stack(neg, ['grainy', 'dark', 'photo'], img, color_normalize=False)
        with pytest.raises(ValueError, match='not found'):
            neg.overlay_words(['dog'], img)
        _, frames = tm.overlay_words(['dog'], img)
        assert not frames.is_cuda and tuple(frames.shape) == (4, 1) + hw + (3,)


def test_image_maps_with_their_images():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=6)
    with trace(pipe) as tc:
        out = pipe(PROMPT, num_inference_steps=2, generator=torch.Generator().manual_seed(11),
                   num_images_per_prompt=3)
        per_image = tc.compute_image_heat_maps()
        assert len(per_image) == 3 and len(out.images) == 3
        # the synthetic pipeline's images are latents: scale three channels of each to a uint8 512 x 512 RGB image
        lat = torch.stack([im.float()[:3] for im in out.images])
        lat = torch.nn.functional.interpolate(lat, size=(512, 512), mode='nearest')
        lo, hi = lat.amin((1, 2, 3), keepdim=True), lat.amax((1, 2, 3), keepdim=True)
        images = ((lat - lo) / (hi - lo) * 255).round().to(torch.uint8).permute(0, 2, 3, 1).contiguous()
        check_stack(per_image, ['dog', 'ball', 'beach'], images, threshold=0.4)
        check_stack(per_image, ['dog', 'ball'], images.cpu().numpy())


# ---- limits through the C ABI ------------------------------------------------------------------------------------------
def _abi_call(maps, n_maps, n_rows, grid, rows_per_word, out_hw, image=None, frames=None, stride=0, null=None):
    n_words = max(len(rows_per_word), 1)
    word_maps = torch.empty((n_maps, n_words) + grid, device=DEV)
    if image is None:
        image = torch.zeros(out_hw + (3,), dtype=torch.uint8, device=DEV)
    if frames is None:
        frames = torch.empty(_native.overlay_frames_bytes(n_maps, n_words, *out_hw), dtype=torch.uint8, device=DEV)
    scratch = torch.empty(_native.segment_scratch_floats(n_maps, n_words), device=DEV)
    ptrs = {'maps': maps.data_ptr(), 'word_maps': word_maps.data_ptr(), 'image': image.data_ptr(),
            'frames': frames.data_ptr(), 'scratch': scratch.data_ptr()}
    if null:
        ptrs[null] = 0
    _native.overlay_words(ptrs['maps'], n_maps, n_rows, grid, rows_per_word, out_hw[0], out_hw[1], False, 0.4, True,
                          ptrs['word_maps'], ptrs['image'], stride, ptrs['frames'], ptrs['scratch'],
                          torch.cuda.current_stream().cuda_stream)
    return frames


def _status(fn):
    with pytest.raises(_native.NativeError) as e:
        fn()
    return e.value.code, str(e.value)


def test_word_and_row_limits():
    ghm = GlobalHeatMap(TOK, PROMPT100, synthetic_map((16, 24), 5))
    img = make_image('random', 40, 72, 9)
    check_against_reference(ghm, [f'w{i}' for i in range(96)], img, what='96 words')
    code, msg = _status(lambda: ghm.overlay_words([f'w{i}' for i in range(97)], img))
    assert code == _native.E_UNSUPPORTED and '97 words > 96' in msg
    long_words = [' '.join(f'w{(i + j) % 100}' for j in range(4)) for i in range(80)]    # 320 rows
    _, frames = ghm.overlay_words(long_words, img, to_cpu=False)
    _, m = ghm.expand_words(long_words, img_size(img), to_cpu=False)
    assert torch.equal(frames, overlay_reference(m, img, True, TABLE))
    long_words = [' '.join(f'w{(i + j) % 100}' for j in range(4)) for i in range(81)]    # 324 rows
    code, msg = _status(lambda: ghm.overlay_words(long_words, img))
    assert code == _native.E_UNSUPPORTED and 'at most 320 rows' in msg


def test_map_size_limit():
    img = make_image('random', 300, 300, 10)
    ok = GlobalHeatMap(TOK, 'a b', torch.rand(4, 320, 160, generator=torch.Generator().manual_seed(1)).to(DEV))
    _, frames = ok.overlay_words(['a', 'b'], img, to_cpu=False)                  # a 200 KB map
    _, m = ok.expand_words(['a', 'b'], img_size(img), to_cpu=False)
    assert torch.equal(frames, overlay_reference(m, img, True, TABLE))
    big = GlobalHeatMap(TOK, 'a b', torch.rand(4, 321, 160).to(DEV))
    code, msg = _status(lambda: big.overlay_words(['a'], img))
    assert code == _native.E_UNSUPPORTED and 'does not fit shared memory' in msg


def test_map_limit():
    grid, out = (8, 8), (16, 16)
    maps = torch.rand(65536, 3, *grid, generator=torch.Generator().manual_seed(1)).to(DEV)
    image = torch.randint(0, 256, (16, 16, 3), generator=torch.Generator().manual_seed(2), dtype=torch.uint8).to(DEV)
    frames = _abi_call(maps, 65535, 3, grid, [[1]], out, image=image)
    frames = frames[:65535 * 16 * 16 * 3].view(65535, 1, 16, 16, 3)
    for t in (0, 1234, 65534):
        ghm = GlobalHeatMap(TOK, 'w0', maps[t])
        _, want = ghm.overlay_words(['w0'], image, threshold=0.4, to_cpu=False)
        assert torch.equal(frames[t, 0], want[0]), t
    code, msg = _status(lambda: _abi_call(maps, 65536, 3, grid, [[1]], out))
    assert code == _native.E_UNSUPPORTED and '65536 maps > 65535' in msg


def test_invalid_arguments():
    maps = synthetic_map((16, 16), 3, n_rows=4)
    for null in ('maps', 'word_maps', 'image', 'frames', 'scratch'):
        code, msg = _status(lambda: _abi_call(maps, 1, 4, (16, 16), [[1]], (8, 8), null=null))
        assert code == _native.E_INVALID and 'null pointer' in msg, null
    code, _ = _status(lambda: _abi_call(maps, 1, 4, (16, 16), [[1]], (8, 8), stride=-1))
    assert code == _native.E_INVALID
    buf = torch.empty(256, dtype=torch.uint8, device=DEV)
    code, msg = _status(lambda: _abi_call(maps, 1, 4, (16, 16), [[1]], (8, 8), frames=buf[1:]))
    assert code == _native.E_INVALID and '4-byte aligned' in msg
    code, msg = _status(lambda: _abi_call(maps, 1, 4, (16, 16), [], (8, 8)))
    assert code == _native.E_INVALID and 'empty word list' in msg
    code, msg = _status(lambda: _abi_call(maps, 1, 4, (16, 16), [[9]], (8, 8)))
    assert code == _native.E_INVALID and 'out of range' in msg


@pytest.mark.parametrize('out_hw', [(1, 1), (3, 5), (61, 101), (97, 97)])
def test_writes_stay_inside_the_buffer(out_hw):
    # frames end inside a 4-byte word: the kernel fills the word's padding and nothing past it
    maps = torch.stack([synthetic_map((30, 50), 60 + t, n_rows=4) for t in range(2)])
    n = _native.overlay_frames_bytes(2, 2, *out_hw)
    buf = torch.full((n + 64,), 0xAB, dtype=torch.uint8, device=DEV)
    image = torch.randint(0, 256, out_hw + (3,), generator=torch.Generator().manual_seed(3), dtype=torch.uint8).to(DEV)
    _abi_call(maps, 2, 4, (30, 50), [[1], [2, 3]], out_hw, image=image, frames=buf)
    assert bool((buf[n:] == 0xAB).all())
    got = buf[:2 * 2 * out_hw[0] * out_hw[1] * 3].view(2, 2, out_hw[0], out_hw[1], 3)
    stack = GlobalHeatMapStack(TOK, 'a b c', maps)
    _, frames = stack.overlay_words(['a', 'b c'], image, threshold=0.4, to_cpu=False)
    assert torch.equal(got, frames)
