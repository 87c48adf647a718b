"""Word-pair overlap on the host, no GPU: WordOverlap's formulas against numpy, compute_iou / compute_ioa and the DAAM
notebook's iou / ioa on hand-built masks; the arguments GlobalHeatMap.word_overlap and TimeHeatMaps.word_overlap hand to
daam_word_overlap (image=None sizing included); the refusals before anything reaches the native library; empty inputs
that launch nothing; and relation_overlap's endpoint deduplication, skipped edges, gather and 96-endpoint limit."""
import contextlib
import ctypes

import numpy as np
import pytest
import torch

from daam_b200 import _native, heatmap
from daam_b200.evaluate import compute_ioa, compute_iou
from daam_b200.heatmap import GlobalHeatMap, RelationOverlap, TimeHeatMaps, WordOverlap
from daam_b200.testing.synthetic import WhitespaceTokenizer

TOK = WhitespaceTokenizer()
PROMPT = 'a dog chasing a red ball on the beach'     # rows: a 1 / 4, dog 2, chasing 3, red 5, ball 6, ..., beach 9


class Im:
    def __init__(self, h, w):
        self.size, self.height, self.width = (w, h), h, w


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


# ---- WordOverlap formulas ----------------------------------------------------------------------------------------------
def masks(n, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    m = (torch.rand(n, h, w, generator=g) < torch.linspace(0.05, 0.6, n)[:, None, None]).float()
    m[-1] = 0                                                         # an empty word
    return m


def overlap_of(m):
    return WordOverlap((m[:, None] * m[None]).sum((-1, -2)), m.sum((-1, -2)))


def test_formulas_against_numpy():
    m = masks(4, 24, 40, 1)
    ov = overlap_of(m)
    i, a = ov.intersection.numpy(), ov.word_area.numpy()
    eps = np.float32(1e-8)
    np.testing.assert_array_equal(ov.iou().numpy(), (i / (a[:, None] + a[None, :] - i + eps)).astype(np.float32))
    np.testing.assert_array_equal(ov.ioa().numpy(), (i / (a[:, None] + eps)).astype(np.float32))
    assert ov.iou().dtype == torch.float32 and torch.equal(ov.iou(), ov.iou().T)
    stack = WordOverlap(torch.stack([ov.intersection, 2 * ov.intersection]), torch.stack([ov.word_area, 2 * ov.word_area]))
    assert torch.equal(stack.iou()[0], ov.iou()) and torch.equal(stack.ioa()[0], ov.ioa())
    assert tuple(stack.iou().shape) == (2, 4, 4)


def test_formulas_equal_compute_iou_ioa_and_the_notebook_bit_for_bit():
    m = masks(5, 32, 48, 2)
    ov = overlap_of(m)
    iou, ioa = ov.iou(), ov.ioa()
    for a in range(5):
        for b in range(5):
            assert float(iou[a, b]) == compute_iou(m[a], m[b]), (a, b)
            assert float(ioa[a, b]) == compute_ioa(m[a], m[b]), (a, b)
            # the notebook binarises raw maps at t: the masks themselves are such maps
            assert float(iou[a, b]) == notebook_iou(m[a], m[b]), (a, b)
            assert float(ioa[a, b]) == notebook_ioa(m[a], m[b]), (a, b)
    assert bool((ioa[4] == 0).all()) and bool((iou[4] == 0).all())      # the empty word: 0, as the notebook's guard


# ---- what reaches the native call ----------------------------------------------------------------------------------
class FakeLib:
    """Stands in for libdaam_b200.so: records the arguments of daam_word_overlap and writes a known symmetric
    intersection (1 + a + b, diagonal 10 + a) and area (the diagonal) into the (host) outputs."""

    def __init__(self):
        self.calls = []

    def daam_word_overlap(self, *args):
        rows, begin, n_words = args[5], args[6], args[7]
        n_maps = args[1]
        self.calls.append(dict(n_maps=n_maps, n_rows=args[2], grid=(args[3], args[4]),
                               rows=[list(rows[begin[w]:begin[w + 1]]) for w in range(n_words)],
                               out=(args[8], args[9]), absolute=args[10], use_threshold=args[11], threshold=args[12]))
        a = torch.arange(n_words, dtype=torch.float32)
        inter = 1 + a[:, None] + a[None]
        inter.diagonal().copy_(10 + a)
        inter = inter.expand(n_maps, n_words, n_words).contiguous() * torch.arange(1, n_maps + 1)[:, None, None]
        area = inter.diagonal(dim1=-2, dim2=-1).contiguous()
        ctypes.memmove(args[14].value, inter.data_ptr(), inter.numel() * 4)
        ctypes.memmove(args[15].value, area.data_ptr(), area.numel() * 4)
        return 0


@pytest.fixture
def fake(monkeypatch):
    lib = FakeLib()
    monkeypatch.setattr(_native, 'load', lambda: lib)
    monkeypatch.setattr(heatmap, '_require_cuda', lambda t, what: None)
    monkeypatch.setattr(heatmap, '_stream_ptr', lambda dev: 0)
    monkeypatch.setattr(torch.cuda, 'device', lambda dev: contextlib.nullcontext())
    return lib


@pytest.mark.parametrize('threshold,use,value', [(None, 0, 0.0), (0, 0, 0.0), (0.15, 1, 0.15), (1, 1, 1.0)])
def test_threshold_truthiness_reaches_the_native_call(fake, threshold, use, value):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16))
    whms, ov = ghm.word_overlap(['dog', 'red ball', 'a'], Im(40, 40), threshold=threshold)
    call, = fake.calls
    assert call['use_threshold'] == use and call['threshold'] == pytest.approx(value)
    assert call['n_maps'] == 1 and call['out'] == (40, 40) and call['rows'] == [[2], [5, 6], [1, 4]]
    assert tuple(ov.intersection.shape) == (3, 3) and tuple(ov.word_area.shape) == (3,)
    assert ov.intersection.dtype == torch.float32 and float(ov.intersection[0, 2]) == 3.0
    assert [w.word for w in whms] == ['dog', 'red ball', 'a']


def test_image_none_sums_over_the_grid(fake):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 12, 20))
    ghm.word_overlap(['dog', 'x'], absolute=True, threshold=0.15, word_idx=[None, 6])
    call = fake.calls[-1]
    assert call['grid'] == (12, 20) and call['out'] == (12, 20) and call['absolute'] == 1 and call['rows'] == [[2], [7]]
    ghm.word_overlap(['dog'], Im(30, 44))                                # a rectangular map over an image
    assert fake.calls[-1]['out'] == (30, 44)
    GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16)).word_overlap(['dog'], Im(30, 44))
    assert fake.calls[-1]['out'] == (44, 30)                             # a square map keeps (size[0], size[1])


def test_stack_is_one_call_over_every_map(fake):
    tm = TimeHeatMaps(TOK, PROMPT, torch.zeros(5, 11, 16, 16))
    word_maps, ov = tm.word_overlap(['dog', 'beach'], Im(32, 32), threshold=0.4)
    call, = fake.calls
    assert call['n_maps'] == 5 and call['rows'] == [[2], [9]] and call['out'] == (32, 32)
    assert tuple(word_maps.shape) == (5, 2, 16, 16)
    assert tuple(ov.intersection.shape) == (5, 2, 2) and tuple(ov.word_area.shape) == (5, 2)
    assert tuple(ov.iou().shape) == (5, 2, 2) and float(ov.intersection[4, 0, 1]) == 5 * 2.0
    _, ov = tm.word_overlap(['dog'])
    assert fake.calls[-1]['out'] == (16, 16)


def test_scratch_size_matches_the_header():
    # per map: 64 min / max floats per word, then W (W + 3) / 2 slots for each of min(tiles, 256) CTAs
    assert _native.word_overlap_scratch_floats(1, 1, 16, 64) == 64 + 2
    assert _native.word_overlap_scratch_floats(1, 8, 512, 512) == 8 * 64 + 44 * 256
    assert _native.word_overlap_scratch_floats(1, 96, 1024, 1024) == 96 * 64 + 4752 * 256
    assert _native.word_overlap_scratch_floats(50, 8, 512, 512) == 50 * (8 * 64 + 44 * 256)
    assert _native.word_overlap_scratch_floats(60, 12, 64, 64) == 60 * (12 * 64 + 90 * 4)
    assert _native.word_overlap_scratch_floats(2, 3, 17, 65) == 2 * (3 * 64 + 9 * 4)
    assert _native.word_overlap_scratch_floats(65535, 2, 8, 8) == 65535 * (128 + 5)
    assert 'daam_word_overlap' in _native.EXPORTS and _native.WORD_OVERLAP_CTAS == 256


# ---- refusals and empty inputs ---------------------------------------------------------------------------------------
def no_native():
    raise AssertionError('the native library was reached')


def test_unknown_words_then_cpu_tensors_are_refused(monkeypatch):
    monkeypatch.setattr(_native, 'load', no_native)
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16))
    # the word lookup first (on a CPU map: the CUDA check comes after it), then the row range, then CUDA
    with pytest.raises(ValueError, match='Search word zebra not found in prompt!'):
        ghm.word_overlap(['dog', 'zebra'])
    with pytest.raises(ValueError, match='Search word zebra not found in prompt!'):
        TimeHeatMaps(TOK, PROMPT, torch.zeros(3, 11, 16, 16)).word_overlap(['zebra'], Im(32, 32))
    with pytest.raises(IndexError, match='out of bounds'):
        ghm.word_overlap(['dog', 'x'], word_idx=[None, 40])
    with pytest.raises(RuntimeError, match='GlobalHeatMap.word_overlap: .*CUDA tensors only'):
        ghm.word_overlap(['dog'])
    with pytest.raises(RuntimeError, match='TimeHeatMaps.relation_overlap: .*CUDA tensors only'):
        TimeHeatMaps(TOK, PROMPT, torch.zeros(3, 11, 16, 16)).relation_overlap([('ball', 'red', 'amod')])


def test_empty_inputs_launch_nothing(fake):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16))
    whms, ov = ghm.word_overlap([])
    assert whms == [] and tuple(ov.intersection.shape) == (0, 0) and tuple(ov.word_area.shape) == (0,)
    assert tuple(ov.iou().shape) == (0, 0) and not ov.intersection.is_cuda
    word_maps, ov = TimeHeatMaps(TOK, PROMPT, torch.zeros(4, 11, 16, 16)).word_overlap([], Im(32, 32))
    assert tuple(ov.intersection.shape) == (4, 0, 0) and tuple(word_maps.shape) == (4, 0, 16, 16)
    word_maps, ov = TimeHeatMaps(TOK, PROMPT, torch.zeros(0, 11, 16, 16)).word_overlap(['dog'])
    assert tuple(ov.intersection.shape) == (0, 1, 1)
    rel = ghm.relation_overlap([])
    assert rel.relations == [] and rel.kept == [] and rel.words == [] and tuple(rel.iou.shape) == (0,)
    rel = TimeHeatMaps(TOK, PROMPT, torch.zeros(3, 11, 16, 16)).relation_overlap([('zebra', 'dog', 'nsubj')])
    assert rel.kept == [] and tuple(rel.iod.shape) == (3, 0) and tuple(rel.overlap.intersection.shape) == (3, 0, 0)
    assert fake.calls == []


# ---- relations -------------------------------------------------------------------------------------------------------
def test_relation_endpoints_are_deduplicated_and_missing_words_skipped(fake):
    ghm = GlobalHeatMap(TOK, PROMPT, torch.zeros(11, 16, 16))
    edges = [('chasing', 'dog', 'nsubj'), ('ball', 'red', 'amod'), ('chasing', 'ball', 'obj'),
             ('zebra', 'dog', 'nsubj'),              # not in the prompt: skipped
             ('Ball', 'the', 'det'),                 # another case of 'ball': the same endpoint
             (6, 9, 'nmod'),                          # token indices: 6 is 'on', 9 is past 'beach' -> row 10
             (1, 'dog', 'self'),                      # token 1 is 'dog': the same rows as 'dog'
             ('chasing', 'unicorn', 'obj')]           # skipped
    rel = ghm.relation_overlap(edges, threshold=0.15, absolute=True)
    assert isinstance(rel, RelationOverlap)
    call, = fake.calls
    assert call['rows'] == [[3], [2], [6], [5], [8], [7], [10]]
    assert call['absolute'] == 1 and call['use_threshold'] == 1 and call['out'] == (16, 16)
    assert rel.words == ['chasing', 'dog', 'ball', 'red', 'the', 6, 9]
    assert rel.kept == [0, 1, 2, 4, 5, 6] and rel.relations == [edges[i] for i in rel.kept]
    heads, deps = [0, 2, 0, 2, 5, 1], [1, 3, 2, 4, 6, 1]
    iou, ioa = rel.overlap.iou(), rel.overlap.ioa()
    assert torch.equal(rel.iou, iou[heads, deps])
    assert torch.equal(rel.iod, ioa[deps, heads]) and torch.equal(rel.ioh, ioa[heads, deps])
    # the fake's matrix: I[a, b] = 1 + a + b off the diagonal, A[a] = 10 + a
    assert float(rel.ioh[0]) == np.float32(2) / (np.float32(10) + np.float32(1e-8))
    assert float(rel.iod[1]) == np.float32(6) / (np.float32(13) + np.float32(1e-8))


def test_relation_stack_gathers_along_the_map_axis(fake):
    tm = TimeHeatMaps(TOK, PROMPT, torch.zeros(3, 11, 16, 16))
    rel = tm.relation_overlap([('ball', 'red', 'amod'), ('chasing', 'dog', 'nsubj')], image=Im(32, 32))
    assert fake.calls[-1]['n_maps'] == 3 and fake.calls[-1]['out'] == (32, 32)
    assert tuple(rel.iou.shape) == (3, 2) and tuple(rel.overlap.intersection.shape) == (3, 4, 4)
    assert torch.equal(rel.ioh, rel.overlap.ioa()[:, [0, 2], [1, 3]])


def test_more_than_96_endpoints_is_a_value_error(monkeypatch):
    monkeypatch.setattr(_native, 'load', no_native)
    prompt = ' '.join(f'w{i}' for i in range(100))
    ghm = GlobalHeatMap(TOK, prompt, torch.zeros(102, 16, 16))
    edges = [(f'w{2 * i}', f'w{2 * i + 1}', 'dep') for i in range(49)]          # 98 endpoints
    with pytest.raises(ValueError, match='98 distinct endpoints > 96'):
        ghm.relation_overlap(edges)
    with pytest.raises(ValueError, match='97 distinct endpoints > 96'):
        ghm.relation_overlap(edges[:48] + [('w0', 'w96', 'dep')])
