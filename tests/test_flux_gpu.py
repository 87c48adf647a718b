"""FLUX.1 heat maps on the GPU: the hooked forward of the synthetic FLUX transformer against its reference processor,
every layer's slab against the float64 bound of daam_accumulate_joint on text-first operands (the tiny spec and
FLUX.1-dev-sized layers), the mass invariant, whole-batch semantics, and the reads of trace(pipe) against the float64
restatement in tests/flux64.py and against each other."""
import math

import pytest
import torch
from torch.nn.attention import SDPBackend, sdpa_kernel

from daam_b200 import ops, trace
from daam_b200.testing.synthetic import (TINY_FLUX_SPEC, FluxAttnProcessor, FluxSpec, flux_image_ids,
                                         make_flux_pipeline)
from daam_b200.utils import t5_rows
from tests import flux64

pytestmark = pytest.mark.gpu

DT = {'fp32': torch.float32, 'fp16': torch.float16, 'bf16': torch.bfloat16}
T = TINY_FLUX_SPEC.t5_rows
# 24 heads, as FLUX.1 has, in a one-double one-single tree
HEADS24_SPEC = FluxSpec('tiny-flux-24', 1, 1, heads=24, dim_head=32, axes_dim=(8, 12, 12), in_channels=16,
                        joint_attention_dim=64, pooled_projection_dim=32, t5_rows=24, sample_size=32)


def _check(got, ref, bound, what):
    err = (got.double() - ref).abs()
    bad = err > bound
    assert not bad.any(), f'{what}: {int(bad.sum())} elements off, worst {float((err - bound).max()):.3e}'


def _tol(got, ref, what, rtol=2e-3):
    err = (got.double().cpu() - ref.cpu()).abs()
    lim = rtol * ref.abs().cpu() + 1e-6 * float(ref.abs().max())
    assert (err <= lim).all(), f'{what}: worst {float((err - lim).max()):.3e}'


def _traced(dtype, prompt, steps=2, spec=TINY_FLUX_SPEC, **kw):
    """A traced generation of the synthetic FLUX pipeline; records every layer call's ``(layer, q, k, lse)``."""
    pipe = make_flux_pipeline(spec, dtype=dtype, device='cuda', seed=0)
    trace_kw, rows = kw.pop('trace_kw', {}), kw.pop('max_sequence_length', spec.t5_rows)
    calls = []
    with trace(pipe, **trace_kw) as tc:
        enqueue = tc._enqueue_joint

        def record(layer_idx, q, k, lse, n_image, heads, scale):
            calls.append((layer_idx, q.detach().clone(), k.detach().clone(), lse.detach().clone()))
            return enqueue(layer_idx, q, k, lse, n_image, heads, scale)
        tc._enqueue_joint = record
        out = pipe(prompt, num_inference_steps=steps, max_sequence_length=rows, **kw)
        tc.synchronize()
    return pipe, tc, calls, out


def _transformer_inputs(dtype, bsz, grid=(16, 16), tokens=T, seed=3, spec=TINY_FLUX_SPEC):
    g = torch.Generator(device='cuda').manual_seed(seed)
    hw = grid[0] * grid[1]
    return dict(hidden_states=torch.randn(bsz, hw, spec.in_channels, generator=g, device='cuda').to(dtype),
                encoder_hidden_states=torch.randn(bsz, tokens, spec.joint_attention_dim, generator=g,
                                                  device='cuda').to(dtype),
                pooled_projections=torch.randn(bsz, spec.pooled_projection_dim, generator=g, device='cuda').to(dtype),
                timestep=torch.full((bsz,), 0.5, device='cuda', dtype=dtype),
                img_ids=flux_image_ids(*grid, 'cuda').to(dtype),
                txt_ids=torch.zeros(tokens, 3, device='cuda', dtype=dtype),
                guidance=torch.full((bsz,), 3.5, device='cuda'))


@pytest.mark.parametrize('dtype, backend', [(torch.bfloat16, SDPBackend.FLASH_ATTENTION),
                                            (torch.float16, SDPBackend.FLASH_ATTENTION),
                                            (torch.float32, SDPBackend.EFFICIENT_ATTENTION)])
def test_hooked_forward_is_bit_identical(dtype, backend):
    """The whole transformer (double and single blocks), and one double and one single attention on their own."""
    pipe = make_flux_pipeline(TINY_FLUX_SPEC, dtype=dtype, device='cuda', seed=1)
    kw = _transformer_inputs(dtype, 2)
    tr = pipe.transformer
    g = torch.Generator(device='cuda').manual_seed(4)
    x = torch.randn(2, 256, 64, generator=g, device='cuda').to(dtype)
    c = torch.randn(2, T, 64, generator=g, device='cuda').to(dtype)
    rope = tr.pos_embed(torch.cat([kw['txt_ids'], kw['img_ids']]))
    double, single = tr.transformer_blocks[0].attn, tr.single_transformer_blocks[0].attn
    with torch.no_grad(), sdpa_kernel(backend):
        plain = tr(**kw)[0]
        plain_double = double(x, c, image_rotary_emb=rope)
        plain_single = single(torch.cat([c, x], dim=1), image_rotary_emb=rope)
        with trace(pipe, batch_prompts=True) as tc:
            pipe.check_inputs(['a', 'b'], None, 256, 256)
            hooked = tr(**kw)[0]
            hooked_double = double(x, c, image_rotary_emb=rope)
            hooked_single = single(torch.cat([c, x], dim=1), image_rotary_emb=rope)
            assert isinstance(single.processor, type(tc._attn_hookers[0]))
        assert isinstance(single.processor, FluxAttnProcessor) and isinstance(double.processor, FluxAttnProcessor)
    assert torch.equal(plain, hooked)
    assert torch.equal(plain_double[0], hooked_double[0]) and torch.equal(plain_double[1], hooked_double[1])
    assert torch.equal(plain_single, hooked_single)


@pytest.mark.parametrize('dtype', ['fp32', 'fp16', 'bf16'])
def test_every_layer_slab_against_float64(dtype):
    """One step of the tiny pipeline, two prompts: each layer's slab is the kernel's sum for that call, per element
    within the bound of the header's arithmetic, for every sample and head."""
    pipe, tc, calls, _ = _traced(DT[dtype], ['a cat on a mat', 'a dog'], steps=1, trace_kw=dict(batch_prompts=True))
    assert len(calls) == TINY_FLUX_SPEC.double + TINY_FLUX_SPEC.single
    for layer, q, k, lse in calls:
        ref, bound = flux64.reference_and_bound(q, k, lse, T, 1.0 / math.sqrt(q.shape[-1]))
        slab = tc.all_heat_maps.slabs[layer]
        assert slab.acc.shape == ref.shape and slab.heads == TINY_FLUX_SPEC.heads
        _check(slab.acc, ref, bound, f'{dtype} layer {layer}')


def _text_first_inputs(dtype, bsz, heads, hw, tokens, d, seed, spread=1.0):
    g = torch.Generator(device='cuda').manual_seed(seed)
    L = tokens + hw
    q = (torch.randn(bsz, heads, L, d, generator=g, device='cuda') * spread).to(dtype)
    k = (torch.randn(bsz, heads, L, d, generator=g, device='cuda') * spread).to(dtype)
    scale = 1.0 / math.sqrt(d)
    s = torch.einsum('bhid,bhjd->bhij', q.double(), k.double()) * scale
    return q, k, torch.logsumexp(s, dim=-1).float(), scale


@pytest.mark.parametrize('dtype', ['fp32', 'fp16', 'bf16'])
def test_flux_dev_sized_layers_against_float64(dtype):
    """FLUX.1-dev layer sizes at 1024 px: 4096 image tokens, 512 T5 rows, 128-dim heads; 24 heads of a batch of one,
    and three layers in one launch."""
    hw, tokens, d, heads = 4096, 512, 128, 24
    ins = [_text_first_inputs(DT[dtype], 1, heads if i == 0 else 2, hw, tokens, d, seed=20 + i) for i in range(3)]
    accs = [torch.zeros(1, q.shape[1], tokens, hw, device='cuda') for q, *_ in ins]
    descs = [ops.make_joint_desc(q, k, lse, hw, acc, q.shape[1], s, text_first=True, whole_batch=True)
             for (q, k, lse, s), acc in zip(ins, accs)]
    ops.accumulate_joint(descs, 'cuda')
    for i, ((q, k, lse, s), acc) in enumerate(zip(ins, accs)):
        ref, bound = flux64.reference_and_bound(q, k, lse, tokens, s)
        _check(acc, ref, bound, f'{dtype} layer {i}')


@pytest.mark.parametrize('dtype', ['fp32', 'bf16'])
def test_rows_plus_image_mass_is_the_step_count(dtype):
    heads, hw, tokens, d, steps = 3, 256, 512, 128, 4
    acc = torch.zeros(2, heads, tokens, hw, device='cuda')
    mass = torch.zeros(2, heads, hw, dtype=torch.float64, device='cuda')
    for step in range(steps):
        q, k, lse, scale = _text_first_inputs(DT[dtype], 2, heads, hw, tokens, d, seed=step, spread=1.5)
        ops.accumulate_joint([ops.make_joint_desc(q, k, lse, hw, acc, heads, scale, text_first=True,
                                                  whole_batch=True)], 'cuda')
        mass += flux64.image_mass(q, k, tokens, scale)
    total = acc.double().sum(2) + mass
    assert torch.allclose(total, torch.full_like(total, steps), rtol=0, atol=1e-4), float((total - steps).abs().max())


def test_a_batch_of_one_keeps_all_24_heads():
    pipe, tc, calls, _ = _traced(torch.bfloat16, 'a red fox in the snow', steps=2, spec=HEADS24_SPEC)
    per_layer = flux64.flux_maps(calls, HEADS24_SPEC.t5_rows, (16, 16), 24)
    for layer, slab in tc.all_heat_maps.slabs.items():
        assert slab.heads == 24 and slab.head_offset == 0 and slab.acc.shape[:2] == (1, 24)
        _tol(slab.acc.view(1, 24, -1, 16, 16), per_layer[layer], f'layer {layer}')
    keys, _ = tc.compute_per_head_heat_maps()
    assert len(keys) == 2 * 24


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16, torch.float16])
def test_trace_maps_match_float64(dtype):
    prompt, prompt_2 = 'a cute giraffe eating leaves', 'a Giraffe eating green leaves under a bright sky'
    pipe, tc, calls, _ = _traced(dtype, prompt, prompt_2=prompt_2)
    grid = tc.geometry.grid
    assert grid == (16, 16)
    heads = TINY_FLUX_SPEC.heads
    per_layer = flux64.flux_maps(calls, T, grid, heads)
    n = t5_rows(len(pipe.tokenizer_2.tokenize(prompt_2)), T, clip_tokens=0)
    ghm = tc.compute_global_heat_map()
    assert ghm.prompt == prompt_2 and ghm.heat_maps.shape == (n + 2,) + grid
    assert float(ghm.heat_maps[0].abs().max()) == 0
    _tol(ghm.heat_maps, flux64.global_rows(per_layer, n), 'global')
    assert torch.equal(tc.compute_global_heat_map(encoder='t5').heat_maps, ghm.heat_maps)
    _tol(tc.compute_global_heat_map(normalize=True).heat_maps, flux64.global_rows(per_layer, n, normalize=True),
         'normalized')
    for layer in (0, 3):
        _tol(tc.compute_global_heat_map(layer_idx=layer).heat_maps, flux64.global_rows({layer: per_layer[layer]}, n),
             f'layer {layer}')
    _tol(tc.compute_global_heat_map(head_idx=1).heat_maps,
         flux64.global_rows({l: m[:, 1:2] for l, m in per_layer.items()}, n), 'head 1')
    assert torch.equal(tc.compute_global_heat_map(factors={1}).heat_maps, ghm.heat_maps)
    with pytest.raises(RuntimeError, match='No heat maps found'):
        tc.compute_global_heat_map(factors={2})
    assert ghm.compute_word_heat_map('Giraffe').heatmap.shape == grid
    keys, maps = tc.compute_per_head_heat_maps()
    assert len(keys) == (TINY_FLUX_SPEC.double + TINY_FLUX_SPEC.single) * heads
    for (factor, layer, head), m in zip(keys, maps):
        assert factor == 1
        _tol(m, flux64.global_rows({layer: per_layer[layer][:, head:head + 1]}, n), f'key {layer}/{head}')
    assert torch.equal(tc.compute_head_heat_maps().heat_maps, maps)
    layers = tc.compute_layer_heat_maps()
    assert len(layers.layers) == 5 and layers.names[2] == 'single-attn-0'
    factors = tc.compute_factor_heat_maps()
    assert list(factors.factors) == [1] and torch.equal(factors.heat_maps[0], ghm.heat_maps)
    items = list(tc.all_heat_maps.items())
    assert len(items) == len(keys) and items[0][1].shape == (T,) + grid
    _tol(items[0][1], per_layer[0][0, 0], 'raw key 0')


def test_reads_agree_bit_for_bit_across_launch_modes_prompts_and_images():
    prompts = ['a cat on a mat', 'two birds in flight']
    runs = {launch: _traced(torch.bfloat16, prompts, trace_kw=dict(batch_prompts=True, launch=launch),
                            num_images_per_prompt=2) for launch in ('step', 'layer')}
    pipe, tc, calls, out = runs['step']
    assert len(tc.last_images) == 4
    grid = tc.geometry.grid
    per_layer = flux64.flux_maps(calls, T, grid, TINY_FLUX_SPEC.heads)
    for p, prompt in enumerate(prompts):
        n = t5_rows(len(pipe.tokenizer_2.tokenize(prompt)), T, clip_tokens=0)
        ghm = tc.compute_global_heat_map(prompt_idx=p)
        _tol(ghm.heat_maps, flux64.global_rows(per_layer, n, prompt=p, images=2), f'prompt {p}')
        assert torch.equal(runs['layer'][1].compute_global_heat_map(prompt_idx=p).heat_maps, ghm.heat_maps)
        layers = tc.compute_layer_heat_maps(prompt_idx=p)
        for i, layer in enumerate(layers.layers):
            assert torch.equal(layers.heat_maps[i], tc.compute_global_heat_map(prompt_idx=p, layer_idx=layer).heat_maps)
        images = tc.compute_image_heat_maps(prompt_idx=p)
        assert images.heat_maps.shape == (2, n + 2) + grid
        for i in range(2):
            one = tc.compute_global_heat_map(prompt_idx=p, image_idx=i)
            assert torch.equal(images.heat_maps[i], one.heat_maps)
            ref = flux64.global_rows({l: m[p * 2 + i:p * 2 + i + 1] for l, m in per_layer.items()}, n)
            _tol(one.heat_maps, ref, f'prompt {p} image {i}')
        assert torch.equal(tc.compute_image_heat_maps(prompt_idx=p, normalize=True).heat_maps[1],
                           tc.compute_global_heat_map(prompt_idx=p, image_idx=1, normalize=True).heat_maps)


def test_rectangular_generation():
    pipe, tc, calls, out = _traced(torch.bfloat16, 'a lighthouse on a cliff', height=1216, width=832, steps=1)
    assert tc.geometry.grid == (76, 52)
    per_layer = flux64.flux_maps(calls, T, (76, 52), TINY_FLUX_SPEC.heads)
    n = t5_rows(len(pipe.tokenizer_2.tokenize('a lighthouse on a cliff')), T, clip_tokens=0)
    _tol(tc.compute_global_heat_map().heat_maps, flux64.global_rows(per_layer, n), '1216x832')
    assert next(iter(tc.all_heat_maps.items()))[1].shape == (T, 76, 52)
    assert out.images[0].shape == (3, 152, 104)


class _Image:
    def __init__(self, h, w):
        self.height, self.width, self.size = h, w, (w, h)


def test_words_segmentation_and_experiment_on_the_t5_map(tmp_path):
    pipe, tc, _, out = _traced(torch.bfloat16, 'a dog chasing a red ball', prompt_2='a Dog chasing a crimson ball')
    ghm = tc.compute_global_heat_map()
    words = ['Dog', 'crimson', 'ball']
    maps, expanded = ghm.expand_words(words, _Image(128, 128))
    assert expanded.shape == (len(words), 128, 128) and torch.isfinite(expanded).all()
    assert ghm.segment(words, _Image(128, 128)) is not None
    exp = tc.to_experiment(tmp_path)
    assert exp.prompt == 'a Dog chasing a crimson ball' and torch.equal(exp.global_heat_map, ghm.heat_maps)
    assert tc.last_image is not None and len(tc.last_images) == 1


def test_cuda_graph_capture_of_a_traced_step_raises():
    pipe = make_flux_pipeline(TINY_FLUX_SPEC, dtype=torch.bfloat16, device='cuda')
    kw = _transformer_inputs(torch.bfloat16, 1)
    with trace(pipe) as tc:
        pipe('warm up', num_inference_steps=1, max_sequence_length=T)
        graph = torch.cuda.CUDAGraph()
        with pytest.raises(RuntimeError, match='FLUX joint-attention heat maps cannot be captured into a CUDA graph'):
            with torch.no_grad(), torch.cuda.graph(graph):
                pipe.transformer(**kw)


def test_hooked_attention_against_an_independent_float64_restatement():
    """The hooked double- and single-stream attention against tests/flux64.attention64, which restates FLUX's
    attention from the module weights with text first and RoPE as complex multiplication by the position ids: the
    outputs, and each call's slab against the softmax block of image queries x text keys."""
    pipe = make_flux_pipeline(TINY_FLUX_SPEC, dtype=torch.float32, device='cuda', seed=2)
    tr = pipe.transformer
    kw = _transformer_inputs(torch.float32, 2)
    ids = torch.cat([kw['txt_ids'], kw['img_ids']])
    g = torch.Generator(device='cuda').manual_seed(5)
    x = torch.randn(2, 256, 64, generator=g, device='cuda')
    c = torch.randn(2, T, 64, generator=g, device='cuda')
    joined = torch.cat([c, x], dim=1)
    rope = tr.pos_embed(ids)
    double, single = tr.transformer_blocks[0].attn, tr.single_transformer_blocks[0].attn
    axes = TINY_FLUX_SPEC.axes_dim
    with torch.no_grad(), trace(pipe, batch_prompts=True, launch='layer') as tc:
        pipe.check_inputs(['a', 'b'], None, 256, 256)
        tr(**kw)                                         # (the forward pre-hook records T for the single blocks)
        pipe.check_inputs(['a', 'b'], None, 256, 256)    # a new generation: the slabs start from zero
        (img, ctx) = double(x, c, image_rotary_emb=rope)
        out = single(joined, image_rotary_emb=rope)
        tc.synchronize()
        (img64, ctx64), block_double = flux64.attention64(double, x, c, ids, axes)
        out64, block_single = flux64.attention64(single, joined, None, ids, axes, tokens=T)
        for got, ref, what in ((img, img64, 'double image'), (ctx, ctx64, 'double context'),
                               (out, out64, 'single')):
            assert (got.double() - ref).abs().max() <= 1e-4 * ref.abs().max(), what
        slabs = tc.all_heat_maps.slabs
        _tol(slabs[0].acc, block_double, 'double slab')
        _tol(slabs[TINY_FLUX_SPEC.double].acc, block_single, 'single slab')


def test_a_prompt_that_fills_the_context(tmp_path):
    """A T5 prompt with more pieces than the context has rows: n = T - 1 pieces and the EOS fill every context row,
    and every read returns them after the zero row."""
    prompt_2 = ' '.join(['a red fox'] * 12)                 # 36 pieces for a 24-row context
    pipe, tc, calls, _ = _traced(torch.bfloat16, 'a fox', prompt_2=prompt_2, num_images_per_prompt=2)
    n = t5_rows(len(pipe.tokenizer_2.tokenize(prompt_2)), T, clip_tokens=0)
    assert n == T - 1
    grid = tc.geometry.grid
    per_layer = flux64.flux_maps(calls, T, grid, TINY_FLUX_SPEC.heads)
    ghm = tc.compute_global_heat_map()
    assert ghm.heat_maps.shape == (T + 1,) + grid
    _tol(ghm.heat_maps, flux64.global_rows(per_layer, n, images=2), 'global')
    _tol(tc.compute_global_heat_map(normalize=True).heat_maps,
         flux64.global_rows(per_layer, n, images=2, normalize=True), 'normalized')
    layers = tc.compute_layer_heat_maps()
    for i, layer in enumerate(layers.layers):
        _tol(layers.heat_maps[i], flux64.global_rows({layer: per_layer[layer]}, n, images=2), f'layer {layer}')
    images = tc.compute_image_heat_maps()
    for i in range(2):
        _tol(images.heat_maps[i], flux64.global_rows({l: m[i:i + 1] for l, m in per_layer.items()}, n),
             f'image {i}')
    keys, maps = tc.compute_per_head_heat_maps()
    for (_, layer, head), m in zip(keys, maps):
        ref = flux64.global_rows({layer: per_layer[layer].flatten(0, 1)[None, head:head + 1]}, n)
        _tol(m, ref, f'key {layer}/{head}')
    assert ghm.compute_word_heat_map('fox').heatmap.shape == grid
    assert tc.to_experiment(tmp_path).global_heat_map.shape == (T + 1,) + grid
