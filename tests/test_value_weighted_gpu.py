"""Value-weighted heat maps on the GPU: every key's map scaled by ``||W_h v||``, the norm of what its token carries
through its head after the output projection.

* ``daam_value_norms`` against float64 for fp32 / fp16 / bf16 values and weights (mixed too), SD-1.x / 2.x head dims,
  every context length, strided cond-half and whole-batch views, within a bound on the squares.
* ``daam_finalize_parts_weighted`` against float64 on the banded kernel and the generic one, at SD-2.1, SDXL,
  non-square and off-grid geometries, several parts per call, every factor class, split key groups and more than 2048
  keys; weights of 1 give the plain bits and weights of 2^k give 2^k times them.
* ``trace(pipe, value_norms=True)`` end to end on the synthetic pipeline against a float64 statement from the recorded
  Q, K, V and output weights, with its filters and modes; the plain reads do not change; stacks and per-head maps agree
  with single reads bit for bit; a context that changes mid-generation makes the weighted reads raise.
* Why it matters: a head whose value for a token is nearly zero stops deciding where the token's map lies.
"""
import ctypes

import pytest
import torch

from daam_b200 import _native, ops, trace
from daam_b200.heatmap import GlobalHeatMap
from daam_b200.testing.synthetic import TINY_SPEC, WhitespaceTokenizer, make_pipeline
from daam_b200.utils import context_rows
from tests.reference64 import assert_close64, normalized_tolerance
from tests.value64 import (trace_weighted_map64, value_norms64, value_norms_bound, weighted_map64,
                           weighted_tolerance)

pytestmark = pytest.mark.gpu
DEV = 'cuda'
PROMPT = 'a dog chasing a red ball on the beach'
DT = {'f32': torch.float32, 'f16': torch.float16, 'bf16': torch.bfloat16}


@pytest.fixture(autouse=True)
def _exact_fp32():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def bits(t):
    return t.contiguous().view(torch.int32)


def stream():
    return torch.cuda.current_stream().cuda_stream


# -- 1. daam_value_norms against float64 ---------------------------------------------------------------------------------
NORM_CASES = [  # v dtype, W dtype, heads, d, tokens, out_dim
    ('f32', 'f32', 5, 64, 77, 320), ('f16', 'f16', 10, 64, 154, 640), ('bf16', 'bf16', 20, 64, 231, 1280),
    ('f16', 'f32', 8, 40, 77, 320), ('bf16', 'f32', 8, 80, 231, 640), ('f32', 'f16', 8, 160, 154, 1280),
    ('f16', 'bf16', 2, 160, 77, 4096), ('bf16', 'f16', 3, 40, 154, 96),
]


def _check_norms(got, value, weight, heads, what):
    ref = value_norms64(value, weight, heads)
    bound = value_norms_bound(value, weight, heads)
    err = (got.double().square() - ref.square()).abs()
    worst = float((err / bound.clamp_min(1e-300)).max())
    assert worst <= 1.0, f'{what}: |n^2 - ref^2| is {worst:.2f} x the bound'


@pytest.mark.parametrize('vd,wd,heads,d,tokens,out_dim', NORM_CASES)
@pytest.mark.parametrize('layout', ['cond_half', 'whole_batch', 'lone_sample', 'fused_kv'])
def test_value_norms_match_float64(vd, wd, heads, d, tokens, out_dim, layout):
    g = torch.Generator(device=DEV).manual_seed(heads * 1000 + d + tokens)
    bsz = 1 if layout == 'lone_sample' else 4
    c = heads * d
    weight = (torch.randn(out_dim, c, device=DEV, generator=g) / c ** 0.5).to(DT[wd])
    if layout == 'fused_kv':                    # value is the second half of a [B, T, 2C] kv buffer: token stride 2C
        kv = torch.randn(bsz, tokens, 2 * c, device=DEV, generator=g).to(DT[vd])
        value = kv[:, :, c:]
    else:
        value = torch.randn(bsz, tokens, c, device=DEV, generator=g).to(DT[vd])
    whole = layout == 'whole_batch'
    got = ops.value_norms(value, weight, heads, whole_batch=whole)
    torch.cuda.synchronize()
    first, n_samples, head0, n_heads = (0, bsz, 0, heads) if whole else ops.cond_half(bsz, heads)
    v = value[first:first + n_samples, :, head0 * d:]
    w = weight[:, head0 * d:]
    assert got.shape == (n_samples, n_heads, tokens)
    _check_norms(got, v, w, n_heads, f'{layout} {vd}/{wd} d {d} T {tokens}')


def test_value_norms_padded_heads_through_the_c_abi():
    """Any head stride: heads padded to 96 channels, W with a padded row stride."""
    heads, d, tokens, out_dim = 4, 64, 77, 320
    g = torch.Generator(device=DEV).manual_seed(5)
    store = torch.randn(2, tokens, heads, 96, device=DEV, generator=g).half()
    wstore = torch.randn(out_dim, heads * d + 16, device=DEV, generator=g)
    out = torch.empty(2, heads, tokens, device=DEV)
    _native.value_norms(store.data_ptr(), _native.DAAM_F16, (store.stride(0), store.stride(1), 96), wstore.data_ptr(),
                        _native.DAAM_F32, wstore.stride(0), 2, heads, tokens, d, out_dim, out.data_ptr(), stream())
    torch.cuda.synchronize()
    _check_norms(out, store[..., :d].reshape(2, tokens, heads * d), wstore[:, :heads * d], heads, 'padded')


def test_value_norms_refusals():
    lib = _native.load()
    v = torch.zeros(2, 77, 64, device=DEV)
    w = torch.zeros(64, 64, device=DEV)
    out = torch.empty(2, 1, 77, device=DEV)

    def call(**kw):
        a = dict(value=v.data_ptr(), vd=0, t=77, d=64, w=w.data_ptr(), wd=0, n=2, heads=1, out_dim=64,
                 out=out.data_ptr())
        a.update(kw)
        return lib.daam_value_norms(a['value'], a['vd'], 77 * 64, 64, 64, a['w'], a['wd'], 64, a['n'], a['heads'],
                                    a['t'], a['d'], a['out_dim'], a['out'], None)

    assert call() == 0
    assert call(t=100) == _native.E_UNSUPPORTED
    assert call(d=264) == _native.E_UNSUPPORTED
    assert call(out_dim=4097) == _native.E_UNSUPPORTED
    assert call(n=65536) == _native.E_UNSUPPORTED
    assert call(value=None) == _native.E_INVALID
    assert call(out=None) == _native.E_INVALID
    assert call(wd=7) == _native.E_INVALID
    assert call(heads=0) == _native.E_INVALID
    torch.cuda.synchronize()


# -- 2. daam_finalize_parts_weighted against float64, and its bit invariants -------------------------------------------
GEOMS = {  # grid, [(h, w, heads)] of the groups
    'sd21': ((64, 64), [(64, 64, 5), (32, 32, 10), (16, 16, 20), (64, 64, 5), (32, 32, 10), (16, 16, 20)]),
    'sdxl': ((128, 128), [(64, 64, 10), (32, 32, 20), (64, 64, 10), (32, 32, 20)]),
    'rect': ((64, 96), [(64, 96, 5), (32, 48, 10), (16, 24, 20)]),
    'offgrid': ((75, 75), [(75, 75, 5), (38, 38, 10), (19, 19, 20)]),
    'many': ((64, 64), [(16, 16, 160)] * 14),       # 2240 keys: past the banded kernel's 2048
}


def _groups(geom, tokens=77, seed=0, head_sel=-1):
    grid, spec = GEOMS[geom]
    g = torch.Generator(device=DEV).manual_seed(seed)
    keys, wts, groups, wptrs = [], [], [], []
    for h, w, heads in spec:
        k = torch.rand(heads, tokens, h * w, device=DEV, generator=g) * 2 - 0.3     # some negative: the clamp acts
        n = torch.rand(heads, tokens, device=DEV, generator=g) * 3
        keys.append(k)
        wts.append(n)
        groups.append(_native.DaamKeyGroup(acc=k.data_ptr(), heads=heads, h=h, w=w, tokens=tokens, head_sel=head_sel,
                                           n_blocks=0))
        wptrs.append(n.data_ptr())
    return grid, keys, wts, groups, wptrs


def _parts(grid, n_rows, spans, n_groups):
    outs = [torch.empty((n_rows,) + grid, device=DEV) for _ in spans]
    parts = [_native.DaamMapPart(group_begin=b, group_count=c, n_rows=n_rows, out=o.data_ptr())
             for (b, c), o in zip(spans, outs)]
    return outs, parts


SPANS = {'sd21': [(0, 6), (0, 3), (1, 1), (2, 4)], 'sdxl': [(0, 4), (1, 2), (3, 1)], 'rect': [(0, 3), (2, 1)],
         'offgrid': [(0, 3), (1, 2)], 'many': [(0, 14), (0, 12), (5, 2)]}


@pytest.mark.parametrize('generic', [False, True], ids=['fast', 'generic'])
@pytest.mark.parametrize('geom', list(GEOMS))
@pytest.mark.parametrize('normalize', [False, True])
def test_weighted_parts_match_float64(geom, generic, normalize, monkeypatch):
    if generic:
        monkeypatch.setenv('DAAM_FINALIZE_GENERIC', '1')
    grid, keys, wts, groups, wptrs = _groups(geom, seed=len(geom))
    n_rows = 12
    outs, parts = _parts(grid, n_rows, SPANS[geom], len(groups))
    _native.finalize_parts(groups, parts, grid, normalize, stream(), wptrs)
    torch.cuda.synchronize()
    for (b, c), out in zip(SPANS[geom], outs):
        k3 = [k.view(k.shape[0], k.shape[1], g.h, g.w) for k, g in zip(keys[b:b + c], groups[b:b + c])]
        ref = weighted_map64(k3, wts[b:b + c], grid, n_rows)
        n_keys = sum(k.shape[0] for k in k3)
        rtol, atol = weighted_tolerance(k3, wts[b:b + c], n_keys, grid)
        if normalize:
            assert_close64(out, ref / (ref[1:-1].sum(0, keepdim=True) + 1e-6), 0.0,
                           normalized_tolerance(ref, rtol, atol), f'{geom} part {b}+{c}')
        else:
            assert_close64(out, ref, rtol, atol, f'{geom} part {b}+{c}', ('row', 'y', 'x'))


@pytest.mark.parametrize('generic', [False, True], ids=['fast', 'generic'])
@pytest.mark.parametrize('geom', list(GEOMS))
@pytest.mark.parametrize('head_sel', [-1, 3])
def test_unit_and_power_of_two_weights_give_the_plain_bits(geom, generic, head_sel, monkeypatch):
    if generic:
        monkeypatch.setenv('DAAM_FINALIZE_GENERIC', '1')
    grid, keys, wts, groups, _ = _groups(geom, seed=7, head_sel=head_sel)
    n_rows = 9
    plain_outs, plain_parts = _parts(grid, n_rows, SPANS[geom], len(groups))
    _native.finalize_parts(groups, plain_parts, grid, False, stream())
    single = torch.empty((n_rows,) + grid, device=DEV)
    _native.finalize(groups, grid, n_rows, False, single.data_ptr(), stream())
    for k in (0, 3, -2):
        ws = [torch.full_like(w, 2.0 ** k) for w in wts]
        outs, parts = _parts(grid, n_rows, SPANS[geom] + [(0, len(groups))], len(groups))
        _native.finalize_parts(groups, parts, grid, False, stream(), [w.data_ptr() for w in ws])
        torch.cuda.synchronize()
        for got, want in zip(outs, plain_outs + [single]):
            assert torch.equal(bits(got), bits(want * 2.0 ** k)), (geom, k)
    ones = [torch.ones_like(w) for w in wts]
    outs, parts = _parts(grid, n_rows, SPANS[geom] + [(0, len(groups))], len(groups))
    _native.finalize_parts(groups, parts, grid, True, stream(), [w.data_ptr() for w in ones])
    _native.finalize_parts(groups, plain_parts, grid, True, stream())
    _native.finalize(groups, grid, n_rows, True, single.data_ptr(), stream())
    torch.cuda.synchronize()
    for got, want in zip(outs, plain_outs + [single]):
        assert torch.equal(bits(got), bits(want)), (geom, 'normalized')


def test_weighted_parts_refusals():
    grid, keys, wts, groups, wptrs = _groups('sd21')
    outs, parts = _parts(grid, 4, [(0, 6)], len(groups))
    lib = _native.load()
    arr = (_native.DaamKeyGroup * len(groups))(*groups)
    sel = (_native.DaamMapPart * 1)(*parts)
    bad = (ctypes.c_void_p * len(groups))(*(wptrs[:-1] + [None]))
    assert lib.daam_finalize_parts_weighted(arr, len(groups), sel, 1, 64, 64, 0, None, None) == _native.E_INVALID
    assert lib.daam_finalize_parts_weighted(arr, len(groups), sel, 1, 64, 64, 0, bad, None) == _native.E_INVALID
    assert 'null weights' in lib.daam_last_error().decode()
    with pytest.raises(ValueError):
        _native.finalize_parts(groups, parts, grid, False, stream(), wptrs[:-1])


# -- 3. the tracer --------------------------------------------------------------------------------------------------------
class Recorder:
    """Device copies of every traced layer call's (layer, q, k, v, W, heads, scale), in call order."""

    def __init__(self, tc):
        self.calls, self._qk = [], None
        enqueue, see = tc._enqueue, tc._see_values

        def _enqueue(layer_idx, factor, q, k, heads, scale):
            self._qk = (layer_idx, q.detach().clone(), k.detach().clone(), heads, scale)
            return enqueue(layer_idx, factor, q, k, heads, scale)

        def _see(layer_idx, ctx, value, weight, heads):
            li, q, k, h, scale = self._qk
            assert li == layer_idx
            self.calls.append((li, q, k, value.detach().clone(), weight.detach().clone(), h, scale))
            return see(layer_idx, ctx, value, weight, heads)

        tc._enqueue, tc._see_values = _enqueue, _see


def _layers(tc, factors=None, layer_idx=None):
    return {s.layer_idx: (s.h, s.w) for s in tc.all_heat_maps.live_slabs()
            if (factors is None or s.factor in factors) and (layer_idx is None or s.layer_idx == layer_idx)}


def _check_traced(tc, rec, got, rows, sample, images=1, image_idx=None, normalize=False, **sel):
    grid = tc.geometry.grid
    ref = trace_weighted_map64(rec.calls, _layers(tc, **sel), rows, grid, sample, len(rows), images, image_idx,
                               normalize)
    # the per-key sums are fp32 sums of a few steps of fp32 probabilities: 1e-5 relative covers them and the finalize
    raw = trace_weighted_map64(rec.calls, _layers(tc, **sel), rows, grid, sample, len(rows), images, image_idx)
    atol = 2e-5 * float(raw.abs().max())
    if normalize:
        assert_close64(got, ref, 0.0, normalized_tolerance(raw, 2e-5, atol), 'normalized')
    else:
        assert_close64(got, ref, 2e-5, atol, 'weighted', ('row', 'y', 'x'))


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
def test_traced_weighted_map_matches_float64(dtype):
    pipe = make_pipeline(TINY_SPEC, dtype=dtype, device=DEV, seed=3)
    with trace(pipe, value_norms=True) as tc:
        rec = Recorder(tc)
        pipe(PROMPT, num_inference_steps=3, generator=torch.Generator().manual_seed(1))
        rows = list(range(len(pipe.tokenizer.tokenize(PROMPT)) + 2))
        b = 1                                                  # the cond half of a [uncond, cond] batch
        for normalize in (False, True):
            got = tc.compute_global_heat_map(value_weighted=True, normalize=normalize).heat_maps
            _check_traced(tc, rec, got, rows, b, normalize=normalize)
        got = tc.compute_global_heat_map(value_weighted=True, factors=[2]).heat_maps
        _check_traced(tc, rec, got, rows, b, factors={2})
        keys, norms = tc.compute_value_norms()
        by_layer = {}
        for li, q, k, v, w, heads, scale in rec.calls:
            by_layer[li] = value_norms64(v[b:b + 1], w, heads)[0][:, :len(rows)]
        ref = torch.stack([by_layer[li][h] for _, li, h in keys])
        assert_close64(norms, ref, 1e-5, 1e-7, 'compute_value_norms')


def test_plain_reads_do_not_change_and_stacks_agree():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=4)
    out = {}
    for on in (False, True):
        with trace(pipe, value_norms=on) as tc:
            pipe(PROMPT, num_inference_steps=2, generator=torch.Generator().manual_seed(2))
            out[on] = [tc.compute_global_heat_map().heat_maps.clone(),
                       tc.compute_global_heat_map(normalize=True).heat_maps.clone(),
                       tc.compute_layer_heat_maps().heat_maps.clone(),
                       tc.compute_factor_heat_maps().heat_maps.clone(),
                       tc.compute_per_head_heat_maps()[1].clone()]
            if on:
                layers = tc.compute_layer_heat_maps(value_weighted=True)
                for i, li in enumerate(layers.layers):
                    one = tc.compute_global_heat_map(layer_idx=li, value_weighted=True).heat_maps
                    assert torch.equal(bits(layers.heat_maps[i]), bits(one)), li
                factors = tc.compute_factor_heat_maps(value_weighted=True, normalize=True)
                for i, f in enumerate(factors.factors):
                    one = tc.compute_global_heat_map(factors=[f], value_weighted=True, normalize=True).heat_maps
                    assert torch.equal(bits(factors.heat_maps[i]), bits(one)), f
                for normalize in (False, True):
                    keys, maps = tc.compute_per_head_heat_maps(value_weighted=True, normalize=normalize)
                    for i, (_, li, h) in enumerate(keys):
                        one = tc.compute_global_heat_map(layer_idx=li, head_idx=h, value_weighted=True,
                                                         normalize=normalize).heat_maps
                        assert torch.equal(bits(maps[i]), bits(one)), (li, h, normalize)
                stack = tc.compute_head_heat_maps(value_weighted=True)
                assert torch.equal(bits(stack.heat_maps), bits(tc.compute_per_head_heat_maps(value_weighted=True)[1]))
    for a, b in zip(out[False], out[True]):
        assert torch.equal(bits(a), bits(b))


def test_traced_modes_match_float64():
    """negative, image_idx, step_range and batch_prompts, each against the float64 statement."""
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float32, device=DEV, seed=5)
    negative = 'blurry dark photo'
    with trace(pipe, value_norms=True, negative=True, batch_prompts=True, step_ranges=[(0, 3)]) as tc:
        rec = Recorder(tc)
        pipe([PROMPT, 'a cat'], num_inference_steps=3, generator=torch.Generator().manual_seed(3),
             negative_prompt=[negative, negative], num_images_per_prompt=2)
        n_rows = lambda text: list(range(len(pipe.tokenizer.tokenize(text)) + 2))
        # batch [uncond p0 i0, p0 i1, p1 i0, p1 i1, cond ...]: prompt p's cond images start at 4 + 2p
        got = tc.compute_global_heat_map(value_weighted=True, prompt_idx=1).heat_maps
        _check_traced(tc, rec, got, n_rows('a cat'), 6, images=2)
        got = tc.compute_global_heat_map(value_weighted=True, image_idx=1).heat_maps
        _check_traced(tc, rec, got, n_rows(PROMPT), 4, images=2, image_idx=1)
        got = tc.compute_global_heat_map(value_weighted=True, negative=True).heat_maps
        _check_traced(tc, rec, got, n_rows(negative), 0, images=2)
        got = tc.compute_global_heat_map(value_weighted=True, step_range=0).heat_maps
        _check_traced(tc, rec, got, n_rows(PROMPT), 4, images=2)      # the range covers every step
        keys, norms = tc.compute_value_norms(negative=True, image_idx=0, prompt_idx=1)
        assert norms.shape == (len(keys), len(n_rows(negative)))


def test_long_context_matches_float64():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=6)
    g = torch.Generator().manual_seed(9)
    embeds = torch.randn(1, 154, 96, generator=g).to(DEV)
    text = ' '.join(f'w{i}' for i in range(100))
    with trace(pipe, value_norms=True, long_prompts=True) as tc:
        rec = Recorder(tc)
        pipe(prompt_embeds=embeds, num_inference_steps=2, generator=torch.Generator().manual_seed(4))
        rows = context_rows(100, 154)
        for normalize in (False, True):
            got = tc.compute_global_heat_map(prompt=text, value_weighted=True, normalize=normalize).heat_maps
            _check_traced(tc, rec, got, rows, 1, normalize=normalize)
        keys, maps = tc.compute_per_head_heat_maps(prompt=text, value_weighted=True)
        _, li, h = keys[0]
        one = tc.compute_global_heat_map(prompt=text, layer_idx=li, head_idx=h, value_weighted=True).heat_maps
        assert torch.equal(bits(maps[0]), bits(one))


def test_a_context_change_makes_the_weighted_read_raise():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float32, device=DEV, seed=7)
    forwards = []

    def swap(_module, args):
        forwards.append(1)
        if len(forwards) == 2:                                 # the second step sees another context
            return (args[0], args[1], args[2] * 1.5) + tuple(args[3:])
        return None

    handle = pipe.unet.register_forward_pre_hook(swap)
    try:
        with trace(pipe, value_norms=True) as tc:
            pipe(PROMPT, num_inference_steps=3, generator=torch.Generator().manual_seed(5))
            plain = tc.compute_global_heat_map()
            assert plain.heat_maps.isfinite().all()
            with pytest.raises(ValueError, match='context changed'):
                tc.compute_global_heat_map(value_weighted=True)
            with pytest.raises(ValueError, match='context changed'):
                tc.compute_per_head_heat_maps(value_weighted=True)
    finally:
        handle.remove()
    # the next generation starts afresh
    with trace(pipe, value_norms=True) as tc:
        pipe(PROMPT, num_inference_steps=2, generator=torch.Generator().manual_seed(5))
        assert tc.compute_global_heat_map(value_weighted=True).heat_maps.isfinite().all()


def test_cuda_graph_capture_is_refused():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=8, cuda_graph=True)
    with trace(pipe, value_norms=True) as tc:
        with pytest.raises(RuntimeError, match='CUDA graph'):
            pipe(PROMPT, num_inference_steps=3, generator=torch.Generator().manual_seed(5))   # step 1 is captured
        tc.synchronize()
    torch.cuda.synchronize()


# -- 4. why the weighting matters ----------------------------------------------------------------------------------------
def test_weighting_moves_the_word_to_the_head_that_carries_it():
    """Head A sends token 1 to the left half with a value norm near zero; head B sends it to the right half with a large
    norm, but more weakly. The plain map prefers the left half, the weighted one the right half."""
    grid, n_rows, h = (64, 64), 3, 64
    acc = torch.zeros(2, 77, h, h, device=DEV)
    acc[0, 1, :, :32] = 0.9                                    # head A: strong, left
    acc[1, 1, :, 32:] = 0.4                                    # head B: weaker, right
    acc[:, 0] = 0.1
    acc[:, 2] = 0.1
    norms = torch.ones(2, 77, device=DEV)
    norms[0, 1], norms[1, 1] = 1e-3, 5.0
    groups = [_native.DaamKeyGroup(acc=acc.data_ptr(), heads=2, h=h, w=h, tokens=77, head_sel=-1, n_blocks=0)]
    out = {w: torch.empty((n_rows,) + grid, device=DEV) for w in (False, True)}
    for weighted, o in out.items():
        part = [_native.DaamMapPart(group_begin=0, group_count=1, n_rows=n_rows, out=o.data_ptr())]
        _native.finalize_parts(groups, part, grid, False, stream(), [norms.data_ptr()] if weighted else None)
    regions = torch.zeros(2, 64, 64, dtype=torch.bool, device=DEV)
    regions[0, :, :32] = True                                  # R1
    regions[1, :, 32:] = True                                  # R2

    class Img:
        size = (64, 64)

    iou = {}
    for weighted, o in out.items():
        hm = GlobalHeatMap(WhitespaceTokenizer(), 'dog', o)
        iou[weighted] = hm.region_overlap(['dog'], Img(), regions, threshold=0.5)[1].iou()     # [region, word]
    assert iou[False][0, 0] > iou[False][1, 0]
    assert iou[True][1, 0] > iou[True][0, 0]
