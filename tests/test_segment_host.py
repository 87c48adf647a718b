"""Word segmentation on the host, no GPU: the float64 segmentation the GPU tests compare labels with is pinned to the
oracle's port_word_heat_map + port_expand_as followed by an argmax; the arguments GlobalHeatMap.segment and
TimeHeatMaps.segment hand to daam_segment_words (threshold truthiness, absolute, word_idx / offset_idx rows, map
count); unknown words raise ValueError before anything touches CUDA."""
import contextlib

import numpy as np
import pytest
import torch

from daam_b200 import _native, heatmap
from daam_b200.heatmap import GlobalHeatMap, TimeHeatMaps
from daam_b200.testing.synthetic import WhitespaceTokenizer
from oracle import daam_oracle as O
from tests.segment64 import segment64

TOK = WhitespaceTokenizer()
PROMPT = 'a dog chasing a red ball on the beach'


@pytest.mark.parametrize('grid,hw,absolute,threshold', [((16, 16), (40, 40), False, None), ((12, 20), (30, 44), False, 0.4),
                                                        ((16, 16), (12, 12), True, 0.4), ((10, 14), (37, 23), False, 0.4)])
def test_float64_segmentation_matches_the_oracle(grid, hw, absolute, threshold):
    g = torch.Generator().manual_seed(grid[0] + hw[1])
    maps = torch.exp(torch.randn(11, *grid, generator=g))
    if absolute:
        maps = maps / maps.max()
    words = ['dog', 'red ball', 'beach', 'chasing']
    rows_per_word = [heatmap.compute_token_merge_indices(TOK, PROMPT, w)[0] for w in words]
    labels, top, margin, _, _, _ = segment64(maps, rows_per_word, hw, absolute, threshold)
    # the oracle: the reference's compute_word_heat_map + expand_as per word (fp32), then numpy's argmax / threshold
    stack = np.stack([O.port_expand_as(O.port_word_heat_map(maps, TOK, PROMPT, w), hw, absolute).numpy() for w in words])
    assert np.abs(stack.max(0) - top.numpy()).max() < 1e-5
    ref = stack.argmax(0) + 1
    if threshold:
        ref = np.where(stack.max(0) > threshold, ref, 0)
    sure = margin.numpy() > 1e-5                   # decisions further than fp32 noise from a tie or the threshold
    if threshold:
        sure &= np.abs(top.numpy() - threshold) > 1e-5
    assert sure.mean() > 0.99
    assert np.array_equal(labels.numpy()[sure], ref[sure])


class FakeLib:
    """Stands in for libdaam_b200.so: records the arguments of daam_segment_words."""

    def __init__(self):
        self.calls = []

    def daam_segment_words(self, *args):
        rows, begin, n_words = args[5], args[6], args[7]
        self.calls.append(dict(n_maps=args[1], n_rows=args[2], grid=(args[3], args[4]),
                               rows=[list(rows[begin[w]:begin[w + 1]]) for w in range(n_words)],
                               out=(args[8], args[9]), absolute=args[10], use_threshold=args[11], threshold=args[12]))
        return 0


@pytest.fixture
def fake(monkeypatch):
    lib = FakeLib()
    monkeypatch.setattr(_native, 'load', lambda: lib)
    monkeypatch.setattr(heatmap, '_require_cuda', lambda t, what: None)
    monkeypatch.setattr(heatmap, '_stream_ptr', lambda dev: 0)
    monkeypatch.setattr(torch.cuda, 'device', lambda dev: contextlib.nullcontext())
    return lib


@pytest.mark.parametrize('threshold,use,value', [(None, 0, 0.0), (0, 0, 0.0), (0.0, 0, 0.0), (0.4, 1, 0.4), (1, 1, 1.0)])
def test_threshold_truthiness_reaches_the_native_call(fake, threshold, value, use):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16))
    whms, labels, scores = ghm.segment(['dog'], type('Im', (), {'size': (40, 40)})(), threshold=threshold)
    call, = fake.calls
    assert call['use_threshold'] == use and call['threshold'] == pytest.approx(value)
    assert call['absolute'] == 0 and call['out'] == (40, 40) and call['n_maps'] == 1 and call['n_rows'] == 11
    assert labels.dtype == torch.uint8 and scores.dtype == torch.float32 and tuple(labels.shape) == (40, 40)
    assert whms[0].word == 'dog' and tuple(whms[0].heatmap.shape) == (16, 16)


def test_word_idx_offset_idx_and_absolute_reach_the_native_call(fake):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 12, 20))
    img = type('Im', (), {'size': (44, 30), 'height': 30, 'width': 44})()
    whms, _, _ = ghm.segment(['dog', 'red ball', 'x', 'a'], img, absolute=True, word_idx=[None, None, 6, None])
    call = fake.calls[-1]
    assert call['rows'] == [[2], [5, 6], [7], [1, 4]] and call['absolute'] == 1 and call['out'] == (30, 44)
    assert call['grid'] == (12, 20)
    assert [w.word_idx for w in whms] == [None, None, 6, None]
    ghm.segment(['dog', 'ball'], img, offset_idx=1)
    assert fake.calls[-1]['rows'] == [[3], [7]]
    ghm.segment(['dog', 'ball'], img, word_idx=3)                  # one index for every word, as in expand_words
    assert fake.calls[-1]['rows'] == [[4], [4]]


def test_time_heat_maps_segment_is_one_call_over_every_step(fake):
    tm = TimeHeatMaps(TOK, PROMPT, torch.zeros(5, 11, 16, 16))
    word_maps, labels, scores = tm.segment(['dog', 'beach'], type('Im', (), {'size': (32, 32)})(), threshold=0.4)
    call, = fake.calls
    assert call['n_maps'] == 5 and call['rows'] == [[2], [9]] and call['use_threshold'] == 1
    assert tuple(word_maps.shape) == (5, 2, 16, 16) and tuple(labels.shape) == tuple(scores.shape) == (5, 32, 32)


def test_unknown_words_raise_before_any_cuda_use(monkeypatch):
    def no_native():
        raise AssertionError('the native library was reached')
    monkeypatch.setattr(_native, 'load', no_native)
    img = type('Im', (), {'size': (32, 32)})()
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16))         # a CPU map: any CUDA step would raise first
    with pytest.raises(ValueError, match='Search word zebra not found in prompt!'):
        ghm.segment(['dog', 'zebra'], img)
    with pytest.raises(ValueError, match='Search word zebra not found in prompt!'):
        TimeHeatMaps(TOK, PROMPT, torch.zeros(3, 11, 16, 16)).segment(['zebra'], img)
    with pytest.raises(RuntimeError, match='CUDA tensors only'):      # known words: the CPU map is refused
        ghm.segment(['dog'], img)
