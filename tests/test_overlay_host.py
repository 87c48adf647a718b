"""Heat-map overlays without a GPU: the jet table restatement, the image argument and the empty word list."""
import numpy as np
import pytest
import torch
from PIL import Image

from daam_b200 import _native, heatmap
from daam_b200.heatmap import GlobalHeatMap, GlobalHeatMapStack, _overlay_image
from daam_b200.testing.synthetic import WhitespaceTokenizer
from tests.overlay_ref import JET, color_index, jet64, jet_table, overlay_reference

DEV = torch.device('cuda', 0)       # only compared against, never allocated on
TOK = WhitespaceTokenizer()


# ---- the table ---------------------------------------------------------------------------------------------------------
def test_table_endpoints():
    t = jet_table()
    assert t.dtype == torch.float32 and tuple(t.shape) == (256, 3)
    assert t[0].tolist() == [0.0, 0.0, 127.5]
    assert t[255].tolist() == [127.5, 0.0, 0.0]


def test_table_breakpoints_and_range():
    for ch, pts in enumerate(JET):
        for x, y in pts:
            assert jet64(ch, x) == y, (ch, x)          # every segment point is on the curve
        for (x0, y0), (x1, y1) in zip(pts, pts[1:]):
            xm = (x0 + x1) / 2
            assert abs(jet64(ch, xm) - (y0 + y1) / 2) < 1e-15
    t = jet_table()
    assert float(t.min()) == 0.0 and float(t.max()) == 255.0
    # red rises on (0.35, 0.66), green on (0.125, 0.375), blue falls on (0.34, 0.65)
    assert t[89, 0] == 0 and t[90, 0] > 0 and t[168, 0] < 255 and t[169, 0] == 255
    assert t[31, 1] == 0 and t[32, 1] > 0 and t[95, 1] < 255 and t[96, 1] == 255
    assert t[86, 2] == 255 and t[87, 2] < 255 and t[165, 2] > 0 and t[166, 2] == 0
    k = 100
    assert t[k, 0] == np.float32(255.0 * ((k / 255.0 - 0.35) / (0.66 - 0.35)))


def test_reference_composition():
    table = jet_table()
    m = torch.tensor([[[0.0, 0.5], [1.0, 2.0]]])
    assert color_index(m, True).tolist() == [[[0, 64], [128, 255]]]
    assert color_index(m, False).tolist() == [[[0, 128], [255, 255]]]
    assert color_index(torch.full((1, 2, 2), 3.0), True).tolist() == [[[0, 0], [0, 0]]]   # hi == lo
    img = torch.full((2, 2, 3), 100, dtype=torch.uint8)
    out = overlay_reference(m, img, False, table)
    assert out[0, 0, 0].tolist() == [100, 100, 100]                          # alpha 0: the image
    assert out[0, 1, 0].tolist() == [128, 0, 0]                              # alpha 1: jet[255] = 127.5 -> 128
    assert out[0, 1, 1].tolist() == [128, 0, 0]                              # alpha clipped to 1


# ---- the image argument ------------------------------------------------------------------------------------------------
def test_pil_images_are_converted_to_rgb():
    for mode, fill in (('RGB', (10, 20, 30)), ('L', 77), ('RGBA', (1, 2, 3, 4))):
        im = Image.new(mode, (8, 8), fill)
        arr, h, w, per_map = _overlay_image(im, 1, (4, 4), DEV, 'x', stack=False)
        assert arr.dtype == torch.uint8 and tuple(arr.shape) == (8, 8, 3) and (h, w) == (8, 8) and not per_map
        want = np.array(im.convert('RGB'))
        assert np.array_equal(arr.numpy(), want), mode


def test_arrays():
    a = np.random.default_rng(0).integers(0, 256, (6, 10, 3), dtype=np.uint8)
    arr, h, w, _ = _overlay_image(a, 1, (3, 5), DEV, 'x', stack=False)     # non-square map: (height, width)
    assert (h, w) == (6, 10) and torch.equal(arr, torch.from_numpy(a))
    view = torch.from_numpy(np.ascontiguousarray(a.transpose(1, 0, 2))).transpose(0, 1)   # a strided torch view
    arr, h, w, _ = _overlay_image(view, 1, (3, 5), DEV, 'x', stack=False)
    assert (h, w) == (6, 10) and torch.equal(arr, torch.from_numpy(a))
    arr, h, w, _ = _overlay_image(np.asfortranarray(a), 1, (3, 5), DEV, 'x', stack=False)
    assert torch.equal(arr, torch.from_numpy(a))
    sq = np.zeros((8, 8, 3), dtype=np.uint8)
    _, h, w, _ = _overlay_image(sq, 1, (4, 4), DEV, 'x', stack=False)
    assert (h, w) == (8, 8)
    # one image per map, stacks only
    stack = np.zeros((3, 8, 8, 3), dtype=np.uint8)
    arr, h, w, per_map = _overlay_image(stack, 3, (4, 4), DEV, 'x', stack=True)
    assert per_map and (h, w) == (8, 8) and tuple(arr.shape) == (3, 8, 8, 3)
    arr, _, _, per_map = _overlay_image(sq, 3, (4, 4), DEV, 'x', stack=True)
    assert not per_map
    with pytest.raises(ValueError, match='not'):
        _overlay_image(stack, 3, (4, 4), DEV, 'x', stack=False)
    with pytest.raises(ValueError, match='not'):
        _overlay_image(stack, 2, (4, 4), DEV, 'x', stack=True)               # a map count that does not match


def test_wrong_images():
    with pytest.raises(TypeError, match='uint8'):
        _overlay_image(np.zeros((8, 8, 3), dtype=np.float32), 1, (4, 4), DEV, 'x', stack=False)
    with pytest.raises(TypeError, match='uint8'):
        _overlay_image(torch.zeros((8, 8, 3), dtype=torch.int32), 1, (4, 4), DEV, 'x', stack=False)
    with pytest.raises(TypeError, match='PIL'):
        _overlay_image([[0]], 1, (4, 4), DEV, 'x', stack=False)
    for shape in ((8, 8), (8, 8, 4), (8, 8, 1), (1, 8, 8, 3), (9, 8, 3)):
        with pytest.raises(ValueError, match='shape'):
            _overlay_image(np.zeros(shape, dtype=np.uint8), 1, (4, 4), DEV, 'x', stack=False)


def test_square_map_with_a_non_square_image():
    # the reference's size=(image.size[0], image.size[1]) would transpose the image: refused
    with pytest.raises(ValueError, match='transposes'):
        _overlay_image(np.zeros((512, 768, 3), dtype=np.uint8), 1, (64, 64), DEV, 'x', stack=False)
    with pytest.raises(ValueError, match='transposes'):
        _overlay_image(Image.new('RGB', (768, 512)), 1, (64, 64), DEV, 'x', stack=False)
    _, h, w, _ = _overlay_image(Image.new('RGB', (768, 512)), 1, (64, 96), DEV, 'x', stack=False)
    assert (h, w) == (512, 768)


def test_device_mismatch():
    with pytest.raises(ValueError, match='is on meta'):
        _overlay_image(torch.zeros((8, 8, 3), dtype=torch.uint8, device='meta'), 1, (4, 4), DEV, 'x', stack=False)


# ---- the empty word list -----------------------------------------------------------------------------------------------
def test_empty_word_list_launches_nothing(monkeypatch):
    monkeypatch.setattr(heatmap, '_require_cuda', lambda t, what: None)

    def no_launch(*a, **k):
        raise AssertionError('launched')
    monkeypatch.setattr(_native, 'overlay_words', no_launch)
    img = np.zeros((16, 16, 3), dtype=np.uint8)
    whms, frames = GlobalHeatMap(TOK, 'a dog', torch.zeros(4, 8, 8)).overlay_words([], img)
    assert whms == [] and frames.dtype == torch.uint8 and tuple(frames.shape) == (0, 16, 16, 3)
    word_maps, frames = GlobalHeatMapStack(TOK, 'a dog', torch.zeros(5, 4, 8, 8)).overlay_words([], img)
    assert tuple(frames.shape) == (5, 0, 16, 16, 3) and tuple(word_maps.shape) == (5, 0, 8, 8)
    with pytest.raises(ValueError, match='shape'):                          # the image is still checked
        GlobalHeatMap(TOK, 'a dog', torch.zeros(4, 8, 8)).overlay_words([], img[:8])


def test_word_not_in_prompt():
    with pytest.raises(ValueError):
        GlobalHeatMap(TOK, 'a dog', torch.zeros(4, 8, 8)).overlay_words(['cat'], np.zeros((16, 16, 3), np.uint8))


def test_frames_buffer_rounds_up_to_words():
    assert _native.overlay_frames_bytes(1, 1, 1, 1) == 4
    assert _native.overlay_frames_bytes(1, 1, 2, 2) == 12
    assert _native.overlay_frames_bytes(2, 3, 5, 7) == (2 * 3 * 5 * 7 * 3 + 3) // 4 * 4
