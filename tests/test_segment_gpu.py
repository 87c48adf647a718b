"""Word segmentation maps (GlobalHeatMap.segment / TimeHeatMaps.segment, daam_segment_words) on the GPU.

* The contract against expand_words, exactly: scores == m.max(0).values and labels == where(scores > t, argmax + 1, 0)
  with m the expand_words stack, over square, rectangular and off-grid maps, up- and down-sampled images, 1 to 96
  words (multi-token, repeated, explicit word_idx), absolute and every threshold form.
* An independent float64 segmentation (float64 word maps, bicubic64 matrices per axis, float64 normalisation): labels
  agree wherever the float64 decision is further from a tie (or from the threshold) than the fp32 error bound.
* Time-resolved histories in one call (two launches), equal row by row to the per-step call; tracer maps under
  step_range, negative and batch_prompts; ties, determinism and refusals.
"""
import contextlib
from types import SimpleNamespace

import pytest
import torch

from daam_b200 import _native, trace
from daam_b200.heatmap import GlobalHeatMap
from daam_b200.testing.synthetic import TINY_SPEC, UNetSpec, WhitespaceTokenizer, make_pipeline
from tests.segment64 import label_bound, segment64

pytestmark = pytest.mark.gpu
DEV = 'cuda'
TOK = WhitespaceTokenizer()
PROMPT100 = ' '.join(f'w{i}' for i in range(100))
# an SDXL-topology tree (sample_size 128 -> g = 2; no cross-attention at the first level, factors 1 and 2)
TINY_XL = UNetSpec('tiny-xl', 128, (32, 64, 64), (1, 2, 2), (0, 1, 1), 64, mid_depth=1)
PROMPT = 'a dog chasing a red ball on the beach'
THRESHOLDS = (None, 0, 0.4)


def image(h, w):
    """A PIL-like image of height ``h`` and width ``w``."""
    return SimpleNamespace(size=(w, h), height=h, width=w)


# (map grid, image (h, w)): square, rectangular both ways, SDXL 1216x832, off-grid 600x800, a smaller output
PAIRS = [((64, 64), (512, 512)), ((96, 96), (768, 768)), ((64, 96), (512, 768)), ((96, 64), (96, 80)),
         ((76, 52), (1216, 832)), ((75, 100), (600, 800)), ((64, 64), (96, 80))]


def word_list(n):
    """``n`` words of PROMPT100 with a multi-token word, a repeated word and explicit word indices."""
    words = [f'w{3 * i % 100}' for i in range(n)]
    idx = [None] * n
    if n >= 3:
        words[1] = 'w40 w41'                 # two tokens: the mean of two rows
        words[-1] = words[0]                 # repeated: ties with word 0, which wins
    if n >= 8:
        idx[2], idx[5] = 7, 93               # explicit word_idx (the word itself is ignored)
    return words, idx


def synthetic_map(grid, seed, n_rows=102):
    g = torch.Generator().manual_seed(seed)
    return torch.exp(1.5 * torch.randn(n_rows, *grid, generator=g)).to(DEV)


def check_contract(ghm, words, img, absolute=False, word_idx=None, offset_idx=0, what=''):
    """segment == the expand_words composition, bit for bit, for every threshold form."""
    whms_e, m = ghm.expand_words(words, img, absolute=absolute, word_idx=word_idx, offset_idx=offset_idx, to_cpu=False)
    ref_scores = m.max(0).values
    arg = m.argmax(0)                        # torch.argmax: the first maximal index
    for t in THRESHOLDS:
        whms, labels, scores = ghm.segment(words, img, absolute=absolute, threshold=t, word_idx=word_idx,
                                           offset_idx=offset_idx, to_cpu=False)
        assert labels.dtype == torch.uint8 and scores.dtype == torch.float32 and labels.is_cuda
        assert tuple(labels.shape) == tuple(scores.shape) == tuple(m.shape[1:])
        assert torch.equal(scores, ref_scores), f'{what} t={t}: scores'
        want = (arg + 1).to(torch.uint8)
        if t:
            want = torch.where(ref_scores > t, want, torch.zeros_like(want))
        assert torch.equal(labels, want), f'{what} t={t}: labels ({int((labels != want).sum())} differ)'
        assert [w.word for w in whms] == [w.word for w in whms_e]
        assert [w.word_idx for w in whms] == [w.word_idx for w in whms_e]
        for a, b in zip(whms, whms_e):
            assert torch.equal(a.heatmap, b.heatmap), what
    return m


@pytest.mark.parametrize('absolute', [False, True])
@pytest.mark.parametrize('n_words', [1, 3, 8, 24, 96])
@pytest.mark.parametrize('grid,hw', PAIRS, ids=[f'{g[0]}x{g[1]}-{h}x{w}' for g, (h, w) in PAIRS])
def test_contract_against_expand_words(grid, hw, n_words, absolute):
    ghm = GlobalHeatMap(TOK, PROMPT100, synthetic_map(grid, n_words + 7 * grid[0] + grid[1]))
    words, idx = word_list(n_words)
    img = image(*hw)
    m = check_contract(ghm, words, img, absolute, idx, what=f'{grid} {hw} {n_words}')
    # a square map keeps the reference's (image.size[0], image.size[1]) order, a non-square one is (height, width)
    assert tuple(m.shape) == (n_words,) + ((hw[1], hw[0]) if grid[0] == grid[1] else hw)


def test_contract_with_offset_idx():
    ghm = GlobalHeatMap(TOK, PROMPT100, synthetic_map((64, 64), 3))
    check_contract(ghm, ['w1', 'w10', 'w20 w21'], image(512, 512), offset_idx=2, what='offset_idx')


# ---- an independent float64 segmentation ---------------------------------------------------------------------------
F64_CASES = [((64, 64), (512, 512), 8, False, 0.4), ((76, 52), (1216, 832), 24, False, None),
             ((75, 100), (600, 800), 8, True, 0.4), ((64, 96), (512, 768), 3, False, 0.4),
             ((96, 64), (96, 80), 24, False, 0.4), ((96, 96), (768, 768), 96, False, None)]


@pytest.mark.parametrize('grid,hw,n_words,absolute,threshold', F64_CASES, ids=lambda v: str(v))
def test_labels_against_float64(grid, hw, n_words, absolute, threshold):
    # uniform rows in [0, 1): normalised maps spread over [0, 1] and absolute ones straddle the threshold
    maps = torch.rand(102, *grid, generator=torch.Generator().manual_seed(11 + n_words)).to(DEV)
    ghm = GlobalHeatMap(TOK, PROMPT100, maps)
    words = [f'w{3 * i % 100}' for i in range(n_words)]
    rows_per_word = [[int(w[1:]) + 1] for w in words]
    _, labels, scores = ghm.segment(words, image(*hw), absolute=absolute, threshold=threshold, to_cpu=False)
    t32 = float(torch.tensor(threshold, dtype=torch.float32)) if threshold else None   # the kernel's fp32 threshold
    ref, top, margin, wm64, by, bx = segment64(maps, rows_per_word, hw, absolute, t32)
    bound = label_bound(wm64, by, bx, rows_per_word, absolute)
    unsure = margin < 2 * bound
    if threshold:
        unsure |= (top - t32).abs() < bound
    assert bool(((scores.double() - top).abs() <= bound).all())
    excluded = float(unsure.double().mean())
    print(f'{grid} {hw} {n_words} words: bound {float(bound.max()):.2e}, excluded fraction {excluded:.2e}')
    assert excluded < 1e-3
    bad = (labels.long() != ref) & ~unsure
    assert int(bad.sum()) == 0, f'{int(bad.sum())} labels differ from float64 away from ties'


# ---- time-resolved histories ----------------------------------------------------------------------------------------
@contextlib.contextmanager
def _history(spec, hw, steps=4, **kw):
    pipe = make_pipeline(spec, dtype=torch.float16, device=DEV, seed=5)
    with trace(pipe, time_resolved=True, **kw) as tc:
        pipe(PROMPT, num_inference_steps=steps, generator=torch.Generator().manual_seed(3), height=hw[0], width=hw[1],
             negative_prompt='blurry grainy dark photo' if kw.get('negative') else None)
        yield tc


def check_history(tm, words, img, **kw):
    before = _native.launch_count()
    word_maps, labels, scores = tm.segment(words, img, to_cpu=False, **kw)
    assert _native.launch_count() - before <= 2                  # the whole history
    assert labels.shape[0] == scores.shape[0] == word_maps.shape[0] == len(tm)
    for t in range(len(tm)):
        whms, lt, st = tm[t].segment(words, img, to_cpu=False, **kw)
        assert torch.equal(lt, labels[t]) and torch.equal(st.view(torch.int32), scores[t].view(torch.int32)), t
        for i, w in enumerate(whms):
            assert torch.equal(w.heatmap, word_maps[t, i])


HISTORIES = [(TINY_SPEC, (512, 512)), (TINY_SPEC, (512, 768)), (TINY_XL, (1024, 1024)), (TINY_XL, (1216, 832))]


@pytest.mark.parametrize('spec,hw', HISTORIES, ids=[f'{s.name}-{h}x{w}' for s, (h, w) in HISTORIES])
def test_time_series_in_one_call(spec, hw):
    img = image(*hw)
    words = ['dog', 'red ball', 'beach', 'a', 'dog']
    with _history(spec, hw) as tc:
        for normalize in (False, True):
            tm = tc.compute_time_heat_maps(normalize=normalize)
            assert len(tm) == 4
            for absolute, threshold in ((False, None), (False, 0.4), (True, 0.4)):
                check_history(tm, words, img, absolute=absolute, threshold=threshold)
            _, labels, scores = tm.segment(words, img)
            assert not labels.is_cuda and tuple(labels.shape) == (4,) + hw


def test_time_series_negative():
    with _history(TINY_SPEC, (512, 768), negative=True) as tc:
        tm = tc.compute_time_heat_maps(negative=True)
        assert tm.prompt == 'blurry grainy dark photo'
        check_history(tm, ['grainy', 'dark', 'photo'], image(512, 768), threshold=0.4)
        with pytest.raises(ValueError, match='not found'):
            tm.segment(['dog'], image(512, 768))


# ---- maps the tracer hands out ---------------------------------------------------------------------------------------
def test_tracer_maps_step_range_negative_and_batch_prompts():
    img = image(512, 768)
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=6)
    with trace(pipe, step_ranges=[(0, 1), (1, 3)], negative=True) as tc:
        pipe(PROMPT, num_inference_steps=3, generator=torch.Generator().manual_seed(2), height=512, width=768,
             negative_prompt='blurry grainy dark')
        for rng in (0, 1):
            check_contract(tc.compute_global_heat_map(step_range=rng), ['dog', 'ball', 'beach'], img, what=f'range {rng}')
        neg = tc.compute_global_heat_map(negative=True)
        check_contract(neg, ['grainy', 'blurry', 'dark'], img, what='negative')
        check_contract(tc.compute_global_heat_map(negative=True, step_range=1), ['dark', 'blurry'], img,
                       what='negative range')
        with pytest.raises(ValueError, match='not found'):
            neg.segment(['dog'], img)
    prompts = ['a red ball', 'two dogs on the beach', 'a cat']
    with trace(pipe, batch_prompts=True) as tc:
        pipe(prompts, num_inference_steps=2, generator=torch.Generator().manual_seed(1))
        for i, words in enumerate((['red', 'ball'], ['dogs', 'beach', 'two'], ['cat'])):
            check_contract(tc.compute_global_heat_map(prompt_idx=i), words, image(512, 512), what=f'prompt {i}')


# ---- ties, determinism, refusals --------------------------------------------------------------------------------------
def test_identical_rows_take_the_lower_label():
    maps = synthetic_map((64, 64), 1, n_rows=6)
    maps[3] = maps[2]
    ghm = GlobalHeatMap(TOK, 'w0 w1 w2 w3', maps)
    for absolute in (False, True):
        _, labels, _ = ghm.segment(['w1', 'w2'], image(512, 512), absolute=absolute)
        assert bool((labels == 1).all())
        _, labels, _ = ghm.segment(['w2', 'w1', 'w2'], image(96, 80), absolute=absolute)
        assert bool((labels == 1).all())


def test_repeated_calls_give_identical_bytes():
    ghm = GlobalHeatMap(TOK, PROMPT100, synthetic_map((76, 52), 2))
    words, idx = word_list(24)
    a = ghm.segment(words, image(1216, 832), threshold=0.4, word_idx=idx, to_cpu=False)
    b = ghm.segment(words, image(1216, 832), threshold=0.4, word_idx=idx, to_cpu=False)
    assert torch.equal(a[1], b[1]) and torch.equal(a[2].view(torch.int32), b[2].view(torch.int32))


def test_refusals_and_edge_cases():
    ghm = GlobalHeatMap(TOK, PROMPT100, synthetic_map((64, 64), 4))
    img = image(512, 512)
    with pytest.raises(_native.NativeError, match='daam_segment_words: 97 words > 96'):
        ghm.segment([f'w{i}' for i in range(97)], img)
    long_words = [' '.join(f'w{(i + j) % 100}' for j in range(4)) for i in range(90)]    # 360 rows
    with pytest.raises(_native.NativeError, match='daam_segment_words: .*at most 320 rows'):
        ghm.segment(long_words, img)
    before = _native.launch_count()
    with pytest.raises(ValueError, match='Search word zebra not found in prompt!'):
        ghm.segment(['w1', 'zebra'], img)
    whms, labels, scores = ghm.segment([], img)
    assert whms == [] and tuple(labels.shape) == (512, 512) and not labels.is_cuda
    assert bool((labels == 0).all()) and bool(torch.isinf(scores).all())
    assert _native.launch_count() == before                    # nothing launched for either
    assert ghm.expand_words([], img)[0] == []
    whms, labels, scores = ghm.segment(['w5'], img, to_cpu=False)
    assert labels.is_cuda and scores.is_cuda and whms[0].heatmap.is_cuda
    assert bool((labels == 1).all())                            # one word owns every pixel without a threshold
