"""Long-prompt heat maps on the GPU: 154- and 231-token contexts (two or three CLIP chunks of 77 tokens).

* Through the C ABI, ``daam_accumulate`` against a float64 softmax over all ``tokens`` columns, fed the same
  (half-rounded) Q/K, within DESIGN section 3's per-key bounds (x10 for 16-bit inputs): every dtype, the SIMT kernel
  forced against the wgmma result, SD-1.x / 2.x head dims, partial and odd pixel counts, one and two prompts, tile
  counts around the SM count with and without early loads, several calls accumulating; every pixel's rows sum to the
  number of calls; and the refusals.
* Through ``trace(pipe, long_prompts=True)`` on the synthetic pipeline driven by ``prompt_embeds``: raw per-key maps
  against the float64 oracle over the recorded Q/K, compact global, per-head, per-image and negative maps against a
  float64 statement of the finalize over the raw maps' context rows, every launch mode, a CUDA-graph pipeline, word maps
  of words past position 75, and that nothing changes for 77-token contexts.
"""
from types import SimpleNamespace

import pytest
import torch

from daam_b200 import _native, ops, trace
from daam_b200.testing.synthetic import TINY15_SPEC, TINY96_SPEC, TINY_SPEC, make_pipeline
from daam_b200.utils import context_rows
from tests.reference64 import bicubic64, layer_maps64
from tests.util import assert_elementwise

pytestmark = pytest.mark.gpu
DEV = 'cuda'
DTYPES = {'bf16': torch.bfloat16, 'fp16': torch.float16, 'fp32': torch.float32}


@pytest.fixture(autouse=True)
def _exact_fp32():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _qk(n_prompts, hw, heads, d, tokens, dtype, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    q = torch.randn(2 * n_prompts, hw, heads * d, device=DEV, generator=g).to(dtype)
    k = (torch.randn(2 * n_prompts, tokens, heads * d, device=DEV, generator=g) * 1.5).to(dtype)
    return q, k


def _acc(q, k, heads, flags=_native.ACC_AUTO, calls=1):
    n_prompts = q.shape[0] // 2
    acc = ops.new_accumulator(n_prompts, heads, q.shape[1], DEV, k.shape[1])
    d = q.shape[2] // heads
    desc = ops.make_layer_desc(q, k, acc, heads, d ** -0.5)
    torch.cuda.synchronize()
    for _ in range(calls):
        ops.accumulate([desc], DEV, flags=flags)
    torch.cuda.synchronize()
    return acc


def _tol(dtype):
    s = 1.0 if dtype == torch.float32 else 10.0
    return 1e-5 * s, 1e-6 * s


# -- 1. the C ABI ---------------------------------------------------------------------------------------------------
ABI_CASES = [  # (hw, heads, d, n_prompts)
    (4096, 2, 64, 1), (576, 2, 40, 2), (475, 1, 80, 1), (361, 2, 160, 2), (1024, 1, 64, 2),
]


@pytest.mark.parametrize('tokens', [154, 231])
@pytest.mark.parametrize('dtype', list(DTYPES))
@pytest.mark.parametrize('case', ABI_CASES, ids=lambda c: 'hw%d_h%d_d%d_n%d' % c)
def test_accumulate_matches_float64_softmax(tokens, dtype, case):
    hw, heads, d, n = case
    dt = DTYPES[dtype]
    q, k = _qk(n, hw, heads, d, tokens, dt, seed=hw * 7 + d + tokens)
    calls = 2
    got = _acc(q, k, heads, calls=calls)
    ref = layer_maps64(q, k, heads, d ** -0.5) * calls
    rtol, atol = _tol(dt)
    assert_elementwise(got, ref, rtol, atol * calls, f'{dtype} {case} {tokens}')
    sums = got.double().sum(dim=2)                     # every pixel's rows sum to the number of calls
    assert torch.allclose(sums, torch.full_like(sums, float(calls)), rtol=1e-5)
    if dt != torch.float32:                             # the SIMT kernel against the wgmma result
        simt = _acc(q, k, heads, flags=_native.ACC_FORCE_SIMT, calls=calls)
        assert_elementwise(simt, ref, 1e-5, 1e-6 * calls, f'simt {dtype} {case} {tokens}')
        assert_elementwise(got, simt.double(), rtol, atol * calls, f'wgmma vs simt {case}')


@pytest.mark.parametrize('tokens', [154, 231])
@pytest.mark.parametrize('dtype', ['bf16', 'fp16'])
@pytest.mark.parametrize('delta', [-1, 0, 1])
@pytest.mark.parametrize('early', [False, True])
def test_tile_counts_around_the_sm_count(tokens, dtype, delta, early):
    sms = _native.device_info()['sm_count']
    hw, heads, d = 128 * (sms + delta), 1, 64
    q, k = _qk(1, hw, heads, d, tokens, DTYPES[dtype], seed=sms + delta)
    flags = _native.ACC_FORCE_MMA | (_native.ACC_EARLY_LOADS if early else 0)
    got = _acc(q, k, heads, flags=flags, calls=3)
    ref = layer_maps64(q, k, heads, d ** -0.5) * 3
    rtol, atol = _tol(DTYPES[dtype])
    assert_elementwise(got, ref, rtol, 3 * atol, f'{tokens} {dtype} {delta} {early}')


def test_chunked_head_dims_share_a_launch_and_lengths_do_not_mix():
    """Layers of 154 and 231 tokens and of 77, 16-bit and fp32, in one call: each is applied exactly once."""
    specs = [(1024, 2, 64, 154, torch.bfloat16), (576, 2, 160, 154, torch.float16), (1024, 1, 64, 231, torch.float16),
             (1024, 1, 80, 231, torch.bfloat16), (256, 2, 64, 77, torch.bfloat16), (256, 1, 40, 231, torch.float32)]
    descs, accs, refs, keep = [], [], [], []
    for i, (hw, heads, d, tokens, dt) in enumerate(specs):
        q, k = _qk(1, hw, heads, d, tokens, dt, seed=100 + i)
        keep += [q, k]                                 # the descriptors hold raw pointers
        acc = ops.new_accumulator(1, heads, hw, DEV, tokens)
        descs.append(ops.make_layer_desc(q, k, acc, heads, d ** -0.5))
        accs.append(acc)
        refs.append(layer_maps64(q, k, heads, d ** -0.5))
    torch.cuda.synchronize()
    ops.accumulate(descs, DEV)
    torch.cuda.synchronize()
    for spec, acc, ref in zip(specs, accs, refs):
        assert_elementwise(acc, ref, *_tol(spec[4]), str(spec))


def test_refusals():
    q, k = _qk(1, 256, 1, 64, 154, torch.float16, seed=1)
    for tokens in (100, 308):
        kk = torch.randn(2, tokens, 64, device=DEV).half()
        acc = ops.new_accumulator(1, 1, 256, DEV)
        with pytest.raises(_native.NativeError) as e:
            ops.accumulate([ops.make_layer_desc(q, kk, acc, 1, 0.125)], DEV)
        assert e.value.code == _native.E_UNSUPPORTED and '77' in str(e.value)
    acc = ops.new_accumulator(1, 1, 256, DEV, 154)
    desc = ops.make_layer_desc(q, k, acc, 1, 0.125)
    slab = torch.zeros_like(acc)
    for fn in (ops.accumulate_steps, ops.accumulate_range):
        with pytest.raises(_native.NativeError) as e:
            fn([desc], [slab], DEV)
        assert e.value.code == _native.E_UNSUPPORTED
    with pytest.raises(_native.NativeError) as e:
        ops.attention_probs(q, k, 1)
    assert e.value.code == _native.E_UNSUPPORTED
    probs = torch.zeros(2, 256, 154, device=DEV)
    with pytest.raises(_native.NativeError) as e:
        ops.accumulate_probs(probs, torch.zeros(1, 154, 256, device=DEV))
    assert e.value.code == _native.E_UNSUPPORTED


# -- 2. through trace() ---------------------------------------------------------------------------------------------
PROMPT_WORDS = 180                                      # three chunks' worth of whitespace tokens (capped at 150 for 154)


def _prompt(n=PROMPT_WORDS):
    words = [f'w{i}' for i in range(n)]
    for i, w in ((20, 'dog'), (100, 'lighthouse'), (140, 'ball')):
        if i < n:
            words[i] = w
    return ' '.join(words)


class Recorder:
    """Device copies of every (layer, factor, q, k, heads, scale) the hook handed to the kernel."""

    def __init__(self, tc):
        self.calls = []
        inner = tc._enqueue

        def enqueue(layer_idx, factor, q, k, heads, scale):
            self.calls.append((layer_idx, factor, q.detach().clone(), k.detach().clone(), heads, scale))
            return inner(layer_idx, factor, q, k, heads, scale)

        tc._enqueue = enqueue

    def keys(self, negative=False):
        """{(factor, layer, head): float64 [tokens, hw]} summed over the recorded calls (prompt 0)."""
        out = {}
        for layer_idx, factor, q, k, heads, scale in self.calls:
            n = q.shape[0] // 2
            pick = [0, 0] if negative else [n, n]       # the cond (or uncond) sample of prompt 0, as a CFG pair
            maps = layer_maps64(q[pick], k[pick], heads, scale)[0]
            for head in range(heads):
                key = (factor, layer_idx, head)
                out[key] = out.get(key, 0) + maps[head]
        return out


def _global64(stacks, grid, rows, normalize=False):
    """Float64 finalize of key stacks ``[heads, tokens, h, w]`` at context ``rows`` (bicubic, clamp, mean, normalise
    over compact rows 1..n)."""
    xh, xw = grid
    total, n = 0, 0
    for s in stacks:
        by, bx = bicubic64(s.shape[-2], xh, s.device), bicubic64(s.shape[-1], xw, s.device)
        total = total + (by @ s[:, rows].double() @ bx.T).clamp(min=0).sum(0)
        n += s.shape[0]
    out = total / n
    if normalize:
        out = out / (out[1:-1].sum(0, keepdim=True) + 1e-6)
    return out


def _embeds(pipe, tokens, n=1, seed=5):
    g = torch.Generator().manual_seed(seed)
    c = pipe.unet.spec.cross_attention_dim
    return torch.randn(n, tokens, c, generator=g), torch.randn(n, tokens, c, generator=g)


def _generate(pipe, tokens, steps=2, n=1, **kw):
    cond, uncond = _embeds(pipe, tokens, n)
    return pipe(prompt_embeds=cond, negative_prompt_embeds=uncond, num_inference_steps=steps,
                generator=torch.Generator().manual_seed(11), **kw)


def _slab_stacks(tc, negative=False, image=None, heads_per_image=None):
    stacks = []
    for s in tc.all_heat_maps.read_slabs(negative=negative):
        src = s.source(None, negative)[0]
        if image is not None:
            src = src[image * s.heads_per_image:(image + 1) * s.heads_per_image]
        stacks.append((s, src.view(src.shape[0], src.shape[1], s.h, s.w)))
    return stacks


FILTERS = [{}, {'normalize': True}, {'factors': [1, 2]}, {'layer_idx': 9, 'head_idx': 0}, {'head_idx': 1}]


def _selected(stacks, f):
    out = []
    for s, st in stacks:
        if 'factors' in f and s.factor not in f['factors']:
            continue
        if 'layer_idx' in f and s.layer_idx != f['layer_idx']:
            continue
        if 'head_idx' in f:
            if f['head_idx'] >= st.shape[0]:
                continue
            st = st[f['head_idx']:f['head_idx'] + 1]
        out.append(st)
    return out


@pytest.mark.parametrize('tokens', [154, 231])
@pytest.mark.parametrize('dtype', list(DTYPES))
@pytest.mark.parametrize('spec,size', [(TINY_SPEC, None), (TINY15_SPEC, None), (TINY96_SPEC, None),
                                       (TINY_SPEC, (512, 768)), (TINY_SPEC, (600, 800))],
                         ids=['tiny', 'tiny15', 'tiny96', 'tiny_512x768', 'tiny_600x800'])
def test_trace_maps_match_the_oracle(tokens, dtype, spec, size):
    dt = DTYPES[dtype]
    pipe = make_pipeline(spec, dtype=dt, device=DEV, seed=3)
    prompt = _prompt()
    kw = {} if size is None else dict(height=size[0], width=size[1])
    with trace(pipe, long_prompts=True, negative=True) as tc:
        rec = Recorder(tc)
        _generate(pipe, tokens, **kw)
        rtol, atol = _tol(dt)
        raw = dict(tc.all_heat_maps.items())
        ref = rec.keys()
        assert set(raw) == set(ref)
        for key, m in raw.items():
            assert m.shape[0] == tokens
            assert_elementwise(m.reshape(tokens, -1), ref[key], rtol, 2 * atol, f'key {key}')
        n_tok = min(PROMPT_WORDS, 75 * (tokens // 77))
        rows = context_rows(PROMPT_WORDS, tokens)
        stacks = _slab_stacks(tc)
        grid = tc.geometry.grid
        for f in FILTERS:
            ghm = tc.compute_global_heat_map(prompt=prompt, **f)
            assert ghm.heat_maps.shape == (n_tok + 2,) + tuple(grid)
            want = _global64(_selected(stacks, f), grid, rows, f.get('normalize', False))
            assert_elementwise(ghm.heat_maps, want, 1e-4, 1e-5 * want.abs().max().item(), f'global {f}')
        # per-head maps: every key's own compact map
        keys, maps = tc.compute_per_head_heat_maps(prompt=prompt, normalize=True)
        for i in (0, len(keys) - 1):
            s = next(s for s, _ in stacks if s.layer_idx == keys[i][1])
            st = dict((id(a), b) for a, b in stacks)[id(s)][keys[i][2]:keys[i][2] + 1]
            want = _global64([st], grid, rows, True)
            assert_elementwise(maps[i], want, 1e-4, 1e-5 * want.abs().max().item(), f'per-head {keys[i]}')
        # negative half, rows counted from the text given for it
        neg_text = 'blurry low quality'
        ghm = tc.compute_global_heat_map(prompt=neg_text, negative=True)
        want = _global64([st for _, st in _slab_stacks(tc, negative=True)], grid,
                         context_rows(3, tokens))
        assert_elementwise(ghm.heat_maps, want, 1e-4, 1e-5 * want.abs().max().item(), 'negative')
        raw_neg = dict(tc.all_heat_maps.items(negative=True))
        ref_neg = rec.keys(negative=True)
        for key in list(raw_neg)[:3]:
            assert_elementwise(raw_neg[key].reshape(tokens, -1), ref_neg[key], rtol, 2 * atol, f'neg key {key}')


@pytest.mark.parametrize('tokens', [154, 231])
def test_words_past_the_first_chunk_read_their_context_rows(tokens):
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=3)
    prompt = _prompt()
    with trace(pipe, long_prompts=True) as tc:
        _generate(pipe, tokens)
        hm = tc.compute_global_heat_map(prompt=prompt)
        stacks = [st for _, st in _slab_stacks(tc)]
        grid = tc.geometry.grid
        words = ['dog', 'lighthouse'] + (['ball'] if tokens == 231 else [])
        positions = {'dog': 20, 'lighthouse': 100, 'ball': 140}
        for w in words:
            ctx = 77 * (positions[w] // 75) + 1 + positions[w] % 75
            want = _global64(stacks, grid, [ctx])[0]
            got = hm.compute_word_heat_map(w).heatmap
            assert_elementwise(got, want, 1e-4, 1e-5 * want.abs().max().item(), w)
        image = SimpleNamespace(size=(512, 512))         # a PIL-like size: the synthetic images are tensors
        whms, expanded = hm.expand_words(words, image)
        for i, w in enumerate(words):
            assert torch.equal(whms[i].heatmap, hm.compute_word_heat_map(w).heatmap)
            assert torch.allclose(expanded[i], hm.compute_word_heat_map(w).expand_as(image), atol=1e-6)
        _, labels, scores = hm.segment(words, image)
        assert torch.equal(scores, expanded.max(0).values)
        assert torch.equal(labels.long(), expanded.argmax(0) + 1)


@pytest.mark.parametrize('tokens', [154, 231])
def test_image_maps_and_batched_prompts(tokens):
    pipe = make_pipeline(TINY_SPEC, dtype=torch.bfloat16, device=DEV, seed=3)
    with trace(pipe, long_prompts=True) as tc:
        _generate(pipe, tokens, num_images_per_prompt=2)
        prompt = _prompt()
        ims = tc.compute_image_heat_maps(prompt_idx=0, normalize=True, prompt=prompt)
        assert ims.heat_maps.shape[:2] == (2, min(PROMPT_WORDS, 75 * (tokens // 77)) + 2)
        for i in range(2):
            one = tc.compute_global_heat_map(prompt=prompt, image_idx=i, normalize=True).heat_maps
            assert torch.equal(ims.heat_maps[i], one)
    with trace(pipe, long_prompts=True, batch_prompts=True) as tc:
        _generate(pipe, tokens, n=2)
        a, b = _prompt(PROMPT_WORDS), _prompt(60)
        ma = tc.compute_global_heat_map(prompt=a, prompt_idx=0).heat_maps
        mb = tc.compute_global_heat_map(prompt=b, prompt_idx=1).heat_maps
        assert ma.shape[0] == min(PROMPT_WORDS, 75 * (tokens // 77)) + 2 and mb.shape[0] == 62
        for p, text, got in ((0, a, ma), (1, b, mb)):
            stacks = []
            for s in tc.all_heat_maps.read_slabs():
                src = s.acc[p]
                stacks.append(src.view(src.shape[0], src.shape[1], s.h, s.w))
            want = _global64(stacks, tc.geometry.grid, context_rows(len(text.split()), tokens))
            assert_elementwise(got, want, 1e-4, 1e-5 * want.abs().max().item(), f'prompt {p}')


@pytest.mark.parametrize('launch', ['overlap', 'layer'])
def test_launch_modes_are_bit_equal_to_the_step_launch(launch):
    reads = []
    for mode in ('step', launch):
        pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=3)
        with trace(pipe, long_prompts=True, launch=mode) as tc:
            _generate(pipe, 231)
            reads.append([tc.compute_global_heat_map(prompt=_prompt(), **f).heat_maps.clone() for f in FILTERS])
    for x, y in zip(*reads):
        assert torch.equal(x, y)


def test_cuda_graph_pipeline():
    eager = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=3)
    graph = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=3, cuda_graph=True)
    reads = []
    for pipe in (eager, graph):
        with trace(pipe, long_prompts=True) as tc:
            _generate(pipe, 154, steps=4)
            reads.append(tc.compute_global_heat_map(prompt=_prompt()).heat_maps.clone())
    assert torch.allclose(reads[0], reads[1], rtol=1e-5, atol=1e-7)


def test_context_length_changes_between_generations():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=3)
    with trace(pipe, long_prompts=True) as tc:
        for tokens in (154, 231, 154, 77):
            _generate(pipe, tokens, steps=1)
            raw = dict(tc.all_heat_maps.items())
            assert all(m.shape[0] == tokens for m in raw.values())
            for m in raw.values():                     # one call: every pixel's rows sum to 1
                sums = m.double().sum(0)
                assert torch.allclose(sums, torch.ones_like(sums), rtol=1e-5)


@pytest.mark.parametrize('launch', ['step', 'overlap'])
def test_77_token_reads_are_unchanged_by_the_option(launch):
    reads = []
    for long_prompts in (False, True):
        pipe = make_pipeline(TINY_SPEC, dtype=torch.bfloat16, device=DEV, seed=3)
        with trace(pipe, long_prompts=long_prompts, launch=launch, negative=True) as tc:
            pipe('a dog chasing a ball near the lighthouse', num_inference_steps=2,
                 generator=torch.Generator().manual_seed(11), negative_prompt='blurry')
            r = [tc.compute_global_heat_map(**f).heat_maps.clone() for f in FILTERS]
            r.append(tc.compute_per_head_heat_maps(normalize=True)[1].clone())
            r.append(tc.compute_global_heat_map(negative=True).heat_maps.clone())
            r += [m.clone() for _, m in tc.all_heat_maps.items()]
            reads.append(r)
    for x, y in zip(*reads):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))


def test_long_context_without_the_option_finds_no_heat_maps():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=3)
    with trace(pipe) as tc:
        _generate(pipe, 154, steps=1)
        with pytest.raises(RuntimeError, match='No heat maps found'):
            tc.compute_global_heat_map(prompt=_prompt())
