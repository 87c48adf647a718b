"""Joint-attention (SD3) heat maps on the GPU: daam_accumulate_joint against float64 at every dtype, context length,
pixel count, head dim, layout and tile edge it takes, the mass invariant, and trace(pipe) of the synthetic SD3
pipeline against the float64 restatement in tests/joint64.py."""
import math

import pytest
import torch
from torch.nn.attention import SDPBackend, sdpa_kernel

from daam_b200 import _native, ops, trace
from daam_b200.testing.synthetic import TINY_SD3_SPEC, JointAttnProcessor, make_sd3_pipeline
from daam_b200.utils import t5_rows
from tests import joint64

pytestmark = pytest.mark.gpu

DT = {'fp32': torch.float32, 'fp16': torch.float16, 'bf16': torch.bfloat16}


def _inputs(dtype, bsz, heads, hw, tokens, d, seed, layout='bhld', spread=1.0):
    """Joint operands ``[B, heads, hw + T, d]`` (or a ``[B, L, heads*d]`` projection viewed that way), and the float64
    lse of the joint softmax rounded to fp32."""
    g = torch.Generator(device='cuda').manual_seed(seed)
    L = hw + tokens
    if layout == 'bhld':
        q = (torch.randn(bsz, heads, L, d, generator=g, device='cuda') * spread).to(dtype)
        k = (torch.randn(bsz, heads, L, d, generator=g, device='cuda') * spread).to(dtype)
    else:
        q = (torch.randn(bsz, L, heads * d, generator=g, device='cuda') * spread).to(dtype)
        k = (torch.randn(bsz, L, heads * d, generator=g, device='cuda') * spread).to(dtype)
        q = q.view(bsz, L, heads, d).transpose(1, 2)
        k = k.view(bsz, L, heads, d).transpose(1, 2)
    scale = 1.0 / math.sqrt(d)
    s = torch.einsum('bhid,bhjd->bhij', q[:, :, :hw].double(), k.double()) * scale
    lse = torch.logsumexp(s, dim=-1).float()
    return q, k, lse, scale


_reference_and_bound = joint64.reference_and_bound


def _check(got, ref, bound, what):
    err = (got.double() - ref).abs()
    bad = err > bound
    assert not bad.any(), f'{what}: {int(bad.sum())} elements off, worst {float((err - bound).max()):.3e}'


@pytest.mark.parametrize('dtype', ['fp32', 'fp16', 'bf16'])
@pytest.mark.parametrize('tokens', [1, 77, 333, 589])
@pytest.mark.parametrize('hw', [1, 17, 1024, 3952, 4096])
@pytest.mark.parametrize('d', [64, 128])
def test_kernel_against_float64(dtype, tokens, hw, d):
    heads = 2
    q, k, lse, scale = _inputs(DT[dtype], 2, heads, hw, tokens, d, seed=hw * 7 + tokens + d)
    acc = torch.zeros(1, heads, tokens, hw, device='cuda')
    ops.accumulate_joint([ops.make_joint_desc(q, k, lse, hw, acc, heads, scale)], 'cuda')
    ref, bound = _reference_and_bound(q, k, lse, hw, scale, slice(1, 2))
    _check(acc, ref, bound, f'{dtype} T={tokens} hw={hw} d={d}')


@pytest.mark.parametrize('dtype', ['fp32', 'bf16', 'fp16'])
@pytest.mark.parametrize('tokens, hw, d', [(16, 64, 8), (17, 65, 24), (63, 63, 40), (64, 128, 256), (65, 129, 136),
                                           (1024, 200, 64), (130, 2, 16)])
def test_kernel_tile_edges(dtype, tokens, hw, d):
    """Token counts around the 16-row warp slices and 64-row passes, pixels around 64- and 128-pixel tiles (odd counts
    take the scalar accumulator path), head dims that are not a multiple of 16 (zero-padded k step) and the largest."""
    heads = 3
    q, k, lse, scale = _inputs(DT[dtype], 2, heads, hw, tokens, d, seed=tokens * 31 + hw)
    acc = torch.zeros(1, heads, tokens, hw, device='cuda')
    ops.accumulate_joint([ops.make_joint_desc(q, k, lse, hw, acc, heads, scale)], 'cuda')
    ref, bound = _reference_and_bound(q, k, lse, hw, scale, slice(1, 2))
    _check(acc, ref, bound, f'{dtype} T={tokens} hw={hw} d={d}')


@pytest.mark.parametrize('dtype', ['fp32', 'bf16'])
def test_kernel_strided_projection_view_and_several_prompts(dtype):
    """``[B, L, heads*d]`` projections viewed as ``[B, heads, L, d]``, 3 prompts x 2 images in the conditional half,
    three steps accumulating."""
    heads, hw, tokens, d, n = 4, 300, 93, 64, 6
    q, k, lse, scale = _inputs(DT[dtype], 2 * n, heads, hw, tokens, d, seed=5, layout='bld')
    acc = torch.zeros(n, heads, tokens, hw, device='cuda')
    desc = ops.make_joint_desc(q, k, lse, hw, acc, heads, scale)
    for _ in range(3):
        ops.accumulate_joint([desc], 'cuda')
    ref, bound = _reference_and_bound(q, k, lse, hw, scale, slice(n, 2 * n))
    _check(acc, 3 * ref, 3 * bound + 3 * ref * 2.0 ** -22, dtype)


def test_kernel_lone_sample_keeps_the_upper_heads():
    heads, hw, tokens, d = 4, 64, 77, 64
    q, k, lse, scale = _inputs(torch.bfloat16, 1, heads, hw, tokens, d, seed=9)
    acc = torch.zeros(1, heads // 2, tokens, hw, device='cuda')
    ops.accumulate_joint([ops.make_joint_desc(q, k, lse, hw, acc, heads, scale)], 'cuda')
    ref, bound = _reference_and_bound(q[:, heads // 2:], k[:, heads // 2:], lse[:, heads // 2:], hw, scale,
                                      slice(0, 1))
    _check(acc, ref, bound, 'B=1')


@pytest.mark.parametrize('name, heads, layers', [('sd3-medium', 24, 3), ('sd3.5-large', 38, 2)])
def test_kernel_production_layer_sizes(name, heads, layers):
    """SD3-medium / SD3.5-large layers at 1024 px (64 x 64 tokens, 333-row context), bf16, several layers per call
    (one launch), two of them into the same slab (separate launches, both added)."""
    hw, tokens, d = 4096, 333, 64
    accs = [torch.zeros(1, heads, tokens, hw, device='cuda') for _ in range(layers)]
    ins = [_inputs(torch.bfloat16, 2, heads, hw, tokens, d, seed=100 + i) for i in range(layers + 1)]
    descs = [ops.make_joint_desc(q, k, lse, hw, acc, heads, s) for (q, k, lse, s), acc in zip(ins, accs)]
    q, k, lse, s = ins[-1]
    descs.append(ops.make_joint_desc(q, k, lse, hw, accs[0], heads, s))
    ops.accumulate_joint(descs, 'cuda')
    for i, acc in enumerate(accs):
        q, k, lse, s = ins[i]
        ref, bound = _reference_and_bound(q, k, lse, hw, s, slice(1, 2))
        if i == 0:
            q, k, lse, s = ins[-1]
            ref2, bound2 = _reference_and_bound(q, k, lse, hw, s, slice(1, 2))
            ref, bound = ref + ref2, bound + bound2 + (ref + ref2) * 2.0 ** -23
        _check(acc, ref, bound, f'{name} layer {i}')


@pytest.mark.parametrize('dtype', ['fp32', 'bf16'])
def test_rows_plus_image_mass_is_the_step_count(dtype):
    heads, hw, tokens, d, steps = 3, 256, 333, 64, 4
    acc = torch.zeros(1, heads, tokens, hw, device='cuda')
    mass = torch.zeros(1, heads, hw, dtype=torch.float64, device='cuda')
    for step in range(steps):
        q, k, lse, scale = _inputs(DT[dtype], 2, heads, hw, tokens, d, seed=step, spread=1.5)
        ops.accumulate_joint([ops.make_joint_desc(q, k, lse, hw, acc, heads, scale)], 'cuda')
        mass += joint64.image_mass(q[1:], k[1:], hw, scale)
    total = acc.double().sum(2) + mass
    assert torch.allclose(total, torch.full_like(total, steps), rtol=0, atol=1e-4), float((total - steps).abs().max())


def test_private_sdpa_ops_are_pinned():
    """The tracer takes the attention's log-sum-exp from two private aten ops: their argument order, that the lse is
    fp32 in natural-log units, and the memory-efficient op's padding of the query axis to a multiple of 32."""
    B, H, L, d = 2, 3, 77 + 50, 64
    g = torch.Generator(device='cuda').manual_seed(0)
    q, k, v = (torch.randn(B, H, L, d, generator=g, device='cuda') for _ in range(3))
    ref = torch.logsumexp(torch.einsum('bhid,bhjd->bhij', q.double(), k.double()) / math.sqrt(d), -1)
    out, lse = torch.ops.aten._scaled_dot_product_flash_attention(q.bfloat16(), k.bfloat16(), v.bfloat16(), 0.0,
                                                                  False, False)[:2]
    assert lse.dtype == torch.float32 and tuple(lse.shape) == (B, H, L) and out.shape == (B, H, L, d)
    assert (lse.double() - ref).abs().max() < 0.1
    out, lse = torch.ops.aten._scaled_dot_product_efficient_attention(q, k, v, None, True, 0.0, False)[:2]
    assert lse.dtype == torch.float32 and tuple(lse.shape) == (B, H, 32 * math.ceil(L / 32))
    assert (lse[..., :L].double() - ref).abs().max() < 1e-4


# ---- trace(pipe) ----------------------------------------------------------------------------------------------
def _traced(dtype, prompt, prompt_3=None, steps=2, **kw):
    pipe = make_sd3_pipeline(TINY_SD3_SPEC, dtype=dtype, device='cuda', seed=0)
    calls = []
    with trace(pipe, **kw.pop('trace_kw', {})) as tc:
        enqueue = tc._enqueue_joint

        def record(layer_idx, q, k, lse, n_image, heads, scale):
            calls.append((layer_idx, q.detach().clone(), k.detach().clone()))
            return enqueue(layer_idx, q, k, lse, n_image, heads, scale)
        tc._enqueue_joint = record
        out = pipe(prompt, prompt_3=prompt_3, num_inference_steps=steps, **kw)
        tc.synchronize()
    return pipe, tc, calls, out


def _tol(got, ref, what, rtol=2e-3):
    err = (got.double().cpu() - ref.cpu()).abs()
    lim = rtol * ref.abs().cpu() + 1e-6 * float(ref.abs().max())
    assert (err <= lim).all(), f'{what}: worst {float((err - lim).max()):.3e}'


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16, torch.float16])
def test_trace_maps_match_float64(dtype):
    """lse from SDPA (not float64) enters the kernel, so the maps agree with the float64 restatement within 2e-3
    relative (+1e-6 of the largest value)."""
    prompt, prompt_3 = 'a cute giraffe eating leaves', 'a Giraffe eating green leaves under a bright sky'
    pipe, tc, calls, _ = _traced(dtype, prompt, prompt_3)
    grid = tc.geometry.grid
    assert grid == (16, 16)
    heads = TINY_SD3_SPEC.heads
    per_layer = joint64.joint_maps(calls, grid[0] * grid[1], grid, heads)
    n = len(prompt.split())
    ghm = tc.compute_global_heat_map()
    _tol(ghm.heat_maps, joint64.global_rows(per_layer, range(n + 2)), 'clip')
    _tol(tc.compute_global_heat_map(normalize=True).heat_maps,
         joint64.global_rows(per_layer, range(n + 2), normalize=True), 'clip normalized')
    pieces = t5_rows(len(pipe.tokenizer_3.tokenize(prompt_3)), 93)
    t5 = tc.compute_global_heat_map(encoder='t5')
    ref = joint64.global_rows(per_layer, range(pieces + 2), first_row=76)
    ref[0] = 0
    _tol(t5.heat_maps, ref, 't5')
    assert t5.compute_word_heat_map('Giraffe').heatmap.shape == grid
    keys, maps = tc.compute_per_head_heat_maps()
    assert len(keys) == TINY_SD3_SPEC.blocks * heads
    for (factor, layer, head), m in zip(keys, maps):
        assert factor == 1
        _tol(m, per_layer[layer][0, head, :n + 2], f'key {layer}/{head}')
    layers = tc.compute_layer_heat_maps(encoder='t5')
    for i, layer in enumerate(layers.layers):
        ref = joint64.global_rows({layer: per_layer[layer]}, range(pieces + 2), first_row=76)
        ref[0] = 0
        _tol(layers.heat_maps[i], ref, f't5 layer {layer}')
    assert torch.equal(tc.compute_head_heat_maps().heat_maps, maps)
    items = list(tc.all_heat_maps.items())
    assert len(items) == len(keys) and items[0][1].shape == (77 + TINY_SD3_SPEC.t5_rows,) + grid


def test_trace_words_and_segmentation_on_both_maps():
    pipe, tc, _, out = _traced(torch.bfloat16, 'a dog chasing a red ball', 'a Dog chasing a crimson ball')
    for ghm, words in ((tc.compute_global_heat_map(), ['dog', 'ball']),
                       (tc.compute_global_heat_map(encoder='t5'), ['Dog', 'crimson', 'ball'])):
        maps, expanded = ghm.expand_words(words, _Image(128, 128))
        assert expanded.shape == (len(words), 128, 128) and torch.isfinite(expanded).all()
        seg = ghm.segment(words, _Image(128, 128))
        assert seg is not None
    assert tc.last_image is not None and len(tc.last_images) == 1


class _Image:
    def __init__(self, h, w):
        self.height, self.width, self.size = h, w, (w, h)


@pytest.mark.parametrize('dtype, backend', [(torch.bfloat16, SDPBackend.FLASH_ATTENTION),
                                            (torch.float16, SDPBackend.FLASH_ATTENTION),
                                            (torch.float32, SDPBackend.EFFICIENT_ATTENTION)])
def test_hooked_forward_is_bit_identical(dtype, backend):
    pipe = make_sd3_pipeline(TINY_SD3_SPEC, dtype=dtype, device='cuda', seed=1)
    g = torch.Generator(device='cuda').manual_seed(3)
    x = torch.randn(4, 4, 32, 32, generator=g, device='cuda').to(dtype)
    ctx = torch.randn(4, 93, 64, generator=g, device='cuda').to(dtype)
    t = torch.full((4,), 500.0, device='cuda')
    with torch.no_grad(), sdpa_kernel(backend):
        plain = pipe.transformer(hidden_states=x, encoder_hidden_states=ctx, timestep=t)[0]
        with trace(pipe, batch_prompts=True) as tc:
            pipe.check_inputs(['a', 'b'], None, None, 256, 256)
            hooked = pipe.transformer(hidden_states=x, encoder_hidden_states=ctx, timestep=t)[0]
            assert isinstance(pipe.transformer.transformer_blocks[0].attn.processor, type(tc._attn_hookers[0]))
        assert isinstance(pipe.transformer.transformer_blocks[0].attn.processor, JointAttnProcessor)
    assert torch.equal(plain, hooked)


@pytest.mark.parametrize('launch', ['step', 'layer'])
def test_batch_prompts_images_and_launch_modes(launch):
    prompts = ['a cat on a mat', 'two birds in flight']
    pipe, tc, calls, _ = _traced(torch.bfloat16, prompts, trace_kw=dict(batch_prompts=True, launch=launch),
                                 num_images_per_prompt=2)
    grid = tc.geometry.grid
    per_layer = joint64.joint_maps(calls, grid[0] * grid[1], grid, TINY_SD3_SPEC.heads)
    for p, prompt in enumerate(prompts):
        n = len(prompt.split())
        _tol(tc.compute_global_heat_map(prompt_idx=p).heat_maps,
             joint64.global_rows(per_layer, range(n + 2), prompt=p, images=2), f'prompt {p}')
        for i in range(2):
            ref = joint64.global_rows({l: m[p * 2 + i:p * 2 + i + 1] for l, m in per_layer.items()}, range(n + 2))
            _tol(tc.compute_global_heat_map(prompt_idx=p, image_idx=i).heat_maps, ref, f'prompt {p} image {i}')
    pieces = t5_rows(len(pipe.tokenizer_3.tokenize(prompts[1])), 93)
    t5ref = joint64.global_rows(per_layer, range(pieces + 2), prompt=1, images=2, first_row=76)
    t5ref[0] = 0
    _tol(tc.compute_global_heat_map(prompt_idx=1, encoder='t5').heat_maps, t5ref, 't5 prompt 1')


def test_rectangular_generation_and_long_t5_context():
    pipe, tc, calls, _ = _traced(torch.bfloat16, 'a lighthouse on a cliff', height=1216, width=832, steps=1,
                                 max_sequence_length=512)
    assert tc.geometry.grid == (76, 52)
    grid = tc.geometry.grid
    per_layer = joint64.joint_maps(calls, 76 * 52, grid, TINY_SD3_SPEC.heads)
    _tol(tc.compute_global_heat_map().heat_maps, joint64.global_rows(per_layer, range(7)), '1216x832')
    assert next(iter(tc.all_heat_maps.items()))[1].shape == (589, 76, 52)


def test_cuda_graph_capture_of_a_traced_step_raises():
    pipe = make_sd3_pipeline(TINY_SD3_SPEC, dtype=torch.bfloat16, device='cuda')
    x = torch.randn(2, 4, 32, 32, device='cuda', dtype=torch.bfloat16)
    ctx = torch.randn(2, 93, 64, device='cuda', dtype=torch.bfloat16)
    t = torch.full((2,), 1.0, device='cuda')
    with trace(pipe) as tc:
        pipe('warm up', num_inference_steps=1)
        graph = torch.cuda.CUDAGraph()
        with pytest.raises(RuntimeError, match='cannot be captured into a CUDA graph'):
            with torch.no_grad(), torch.cuda.graph(graph):
                pipe.transformer(hidden_states=x, encoder_hidden_states=ctx, timestep=t)
