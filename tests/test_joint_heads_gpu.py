"""Head-reduced joint-attention heat maps on the GPU: daam_accumulate_joint_heads against float64 at every dtype,
context length, pixel count, head dim, head count, layout, pack and overlap it takes; its head sum against the
per-head kernel's values, bit for bit; the same bits on every call and launch split; and trace(pipe,
reduce_heads=True) of the synthetic SD3 and FLUX pipelines against the float64 restatements in tests/joint64.py and
tests/flux64.py and against a per-head trace of the same generation."""
import math

import pytest
import torch
from torch.nn.attention import SDPBackend, sdpa_kernel

from daam_b200 import ops, trace
from daam_b200.testing.synthetic import (TINY_FLUX_SPEC, TINY_SD3_SPEC, flux_image_ids, make_flux_pipeline,
                                         make_sd3_pipeline)
from daam_b200.utils import t5_rows
from tests import flux64, joint64

pytestmark = pytest.mark.gpu

DT = {'fp32': torch.float32, 'fp16': torch.float16, 'bf16': torch.bfloat16}
U = 2.0 ** -24          # unit roundoff of fp32


def _inputs(dtype, bsz, heads, hw, tokens, d, seed, layout='bhld', text_first=False):
    """Joint operands ``[B, heads, L, d]`` (or a ``[B, L, heads*d]`` projection viewed that way), image tokens first
    or (``text_first``) last, and the float64 lse of the image queries' joint softmax rounded to fp32, ``[B, heads,
    L]`` (zero on the context rows)."""
    g = torch.Generator(device='cuda').manual_seed(seed)
    L = hw + tokens
    if layout == 'bhld':
        q = torch.randn(bsz, heads, L, d, generator=g, device='cuda').to(dtype)
        k = torch.randn(bsz, heads, L, d, generator=g, device='cuda').to(dtype)
    else:
        q = torch.randn(bsz, L, heads * d, generator=g, device='cuda').to(dtype).view(bsz, L, heads, d).transpose(1, 2)
        k = torch.randn(bsz, L, heads * d, generator=g, device='cuda').to(dtype).view(bsz, L, heads, d).transpose(1, 2)
    scale = 1.0 / math.sqrt(d)
    img = _image_rows(hw, tokens, text_first)
    lse = torch.zeros(bsz, heads, L, device='cuda')
    s = torch.einsum('bhid,bhjd->bhij', q[:, :, img].double(), k.double()) * scale
    lse[:, :, img] = torch.logsumexp(s, dim=-1).float()
    return q, k, lse, scale


def _image_rows(hw, tokens, text_first):
    return slice(tokens, tokens + hw) if text_first else slice(0, hw)


def _per_head_ref(q, k, lse, hw, tokens, scale, keep, text_first=False, heads=slice(None)):
    """float64 exp and bound of every kept (sample, head): ``[N, heads, T, hw]``."""
    img, ctx = _image_rows(hw, tokens, text_first), slice(0, tokens) if text_first else slice(hw, hw + tokens)
    return joint64.exp_and_bound(q[keep, heads, img], k[keep, heads, ctx], lse[keep, heads, img], scale)


def mean_and_bound(ref, bound, acc0=None, bound0=None):
    """The float64 ``acc0 + mean over heads`` of per-head values ``ref`` ``[N, heads, T, hw]`` within ``bound``, and
    its bound: each v_h within its own bound, the fp32 head sum of heads - 1 roundings of partial sums no larger than
    S = sum_h (ref_h + bound_h), the division's rounding, and the accumulate's rounding of acc0 + S / heads."""
    heads = ref.shape[1]
    s = (ref + bound).sum(1)
    mean = ref.sum(1) / heads
    err = (bound.sum(1) + heads * U * s + U * s) / heads * 1.01
    if acc0 is None:
        return mean, err + 1e-37
    return acc0 + mean, bound0 + err + U * (acc0.abs() + bound0 + s / heads) * 1.01 + 1e-37


def _check(got, ref, bound, what):
    err = (got.double() - ref).abs()
    bad = err > bound
    assert not bad.any(), f'{what}: {int(bad.sum())} elements off, worst {float((err - bound).max()):.3e}'


def _head_sum_of_per_head_values(q, k, lse, hw, heads, scale, n_keep, **kw):
    """The header's arithmetic restated on the CPU from the per-head kernel's own values: daam_accumulate_joint into
    zeros gives v_h exactly (0 + v = v), then sum_h in fp32, heads ascending, and an exactly rounded division."""
    tokens = q.shape[2] - hw
    per = torch.zeros(n_keep, heads if kw.get('whole_batch') or q.shape[0] > 1 else heads // 2, tokens, hw,
                      device='cuda')
    ops.accumulate_joint([ops.make_joint_desc(q, k, lse, hw, per, heads, scale, **kw)], 'cuda')
    v = per.cpu()
    s = v[:, 0].clone()
    for h in range(1, v.shape[1]):
        s = s + v[:, h]
    return s / torch.full_like(s, float(v.shape[1]))


def _run_heads(q, k, lse, hw, heads, scale, n_keep, calls=1, **kw):
    tokens = q.shape[2] - hw
    acc = torch.zeros(n_keep, tokens, hw, device='cuda')
    desc = ops.make_joint_desc(q, k, lse, hw, acc, heads, scale, reduce_heads=True, **kw)
    for _ in range(calls):
        ops.accumulate_joint_heads([desc], 'cuda')
    return acc


# ---- the kernel ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dtype', ['fp32', 'fp16', 'bf16'])
@pytest.mark.parametrize('tokens', [1, 77, 333, 589, 1024])
@pytest.mark.parametrize('hw', [1, 17, 3952, 4096])
def test_kernel_against_float64(dtype, tokens, hw):
    """Every context length and pixel count (one pixel, one off every tile edge, off the 64 grid, the 64 x 64 grid),
    2 heads of 64: within the derived bound of float64, and bit for bit the fp32 head sum of the per-head kernel's
    values divided by the head count."""
    heads, d = 2, 64
    q, k, lse, scale = _inputs(DT[dtype], 2, heads, hw, tokens, d, seed=hw * 7 + tokens)
    acc = _run_heads(q, k, lse, hw, heads, scale, 1)
    ref, bound = mean_and_bound(*_per_head_ref(q, k, lse, hw, tokens, scale, slice(1, 2)))
    _check(acc, ref, bound, f'{dtype} T={tokens} hw={hw}')
    assert torch.equal(acc.cpu(), _head_sum_of_per_head_values(q, k, lse, hw, heads, scale, 1))


@pytest.mark.parametrize('dtype', ['fp32', 'fp16', 'bf16'])
@pytest.mark.parametrize('d', [8, 64, 128])
@pytest.mark.parametrize('heads', [1, 2, 24, 38])
def test_kernel_head_dims_and_head_counts(dtype, d, heads):
    """Head dims 8 (not a multiple of 16: a zero-padded k step), 64 and 128; one head (no sum), two, SD3-medium's 24
    and SD3.5-large's 38 (an odd number of staging buffers)."""
    hw, tokens = 300, 77
    q, k, lse, scale = _inputs(DT[dtype], 2, heads, hw, tokens, d, seed=d * 100 + heads)
    acc = _run_heads(q, k, lse, hw, heads, scale, 1)
    ref, bound = mean_and_bound(*_per_head_ref(q, k, lse, hw, tokens, scale, slice(1, 2)))
    _check(acc, ref, bound, f'{dtype} d={d} heads={heads}')
    assert torch.equal(acc.cpu(), _head_sum_of_per_head_values(q, k, lse, hw, heads, scale, 1))


@pytest.mark.parametrize('dtype', ['fp32', 'fp16', 'bf16'])
def test_kernel_strided_views_several_prompts_and_calls(dtype):
    """``[B, L, heads*d]`` projections viewed as ``[B, heads, L, d]``, 3 prompts x 2 images in the conditional half,
    three calls accumulating."""
    heads, hw, tokens, d, n = 4, 300, 93, 64, 6
    q, k, lse, scale = _inputs(DT[dtype], 2 * n, heads, hw, tokens, d, seed=5, layout='bld')
    acc = _run_heads(q, k, lse, hw, heads, scale, n, calls=3)
    one, err = mean_and_bound(*_per_head_ref(q, k, lse, hw, tokens, scale, slice(n, 2 * n)))
    ref, bound = one, err
    for _ in range(2):
        ref, bound = ref + one, bound + err + U * (ref + bound + one + err) * 1.01
    _check(acc, ref, bound, dtype)
    once = _head_sum_of_per_head_values(q, k, lse, hw, heads, scale, n)
    assert torch.equal(acc.cpu(), (once + once) + once)


@pytest.mark.parametrize('dtype', ['fp32', 'fp16', 'bf16'])
def test_kernel_text_first_whole_batch(dtype):
    """FLUX: text-first sequences, every sample of a batch of 2 with all 24 heads of 128, a 512-row context."""
    heads, hw, tokens, d = 24, 1024, 512, 128
    q, k, lse, scale = _inputs(DT[dtype], 2, heads, hw, tokens, d, seed=11, text_first=True)
    kw = dict(text_first=True, whole_batch=True)
    acc = _run_heads(q, k, lse, hw, heads, scale, 2, **kw)
    ref, bound = mean_and_bound(*_per_head_ref(q, k, lse, hw, tokens, scale, slice(0, 2), text_first=True))
    _check(acc, ref, bound, dtype)
    assert torch.equal(acc.cpu(), _head_sum_of_per_head_values(q, k, lse, hw, heads, scale, 2, **kw))


def test_kernel_lone_sample_averages_the_upper_heads():
    heads, hw, tokens, d = 6, 64, 77, 64
    q, k, lse, scale = _inputs(torch.bfloat16, 1, heads, hw, tokens, d, seed=9)
    acc = _run_heads(q, k, lse, hw, heads, scale, 1)
    ref, bound = mean_and_bound(*_per_head_ref(q, k, lse, hw, tokens, scale, slice(0, 1),
                                               heads=slice(heads // 2, heads)))
    _check(acc, ref, bound, 'B=1')
    assert torch.equal(acc.cpu(), _head_sum_of_per_head_values(q, k, lse, hw, heads, scale, 1))


def _pack_layers(n, seed):
    """``n`` small layers of mixed dtypes, head counts and shapes, each into its own head-free slab."""
    layers = []
    for i in range(n):
        dtype = (torch.bfloat16, torch.float16, torch.float32)[i % 3]
        heads, hw, tokens, d = 1 + i % 4, 17 + 13 * (i % 5), 1 + 29 * (i % 4), 8 * (1 + i % 3)
        q, k, lse, scale = _inputs(dtype, 2, heads, hw, tokens, d, seed=seed + i)
        layers.append((q, k, lse, scale, heads, hw, tokens))
    return layers


def _launch(layers, split):
    """Every layer of ``layers`` into a fresh slab, the calls cut into runs of ``split`` layers."""
    accs, descs = [], []
    for q, k, lse, scale, heads, hw, tokens in layers:
        accs.append(torch.zeros(1, tokens, hw, device='cuda'))
        descs.append(ops.make_joint_desc(q, k, lse, hw, accs[-1], heads, scale, reduce_heads=True))
    for i in range(0, len(descs), split):
        ops.accumulate_joint_heads(descs[i:i + split], 'cuda')
    return [a.cpu() for a in accs]


def test_packs_over_64_layers_and_every_launch_split_give_the_same_bits():
    """200 layers of three dtypes: one call (three classes of 66 or 67 layers, each a pack of 64 and the rest), calls
    of 7 and of 1 layer, and the one call again, all bit for bit the same; every layer within its float64 bound."""
    layers = _pack_layers(200, seed=1000)
    whole = _launch(layers, len(layers))
    for split in (len(layers), 7, 1):
        again = _launch(layers, split)
        assert all(torch.equal(a, b) for a, b in zip(whole, again)), split
    for i, ((q, k, lse, scale, heads, hw, tokens), acc) in enumerate(zip(layers, whole)):
        ref, bound = mean_and_bound(*_per_head_ref(q, k, lse, hw, tokens, scale, slice(1, 2)))
        _check(acc.cuda(), ref, bound, f'layer {i}')


@pytest.mark.parametrize('dtype', ['fp32', 'bf16'])
def test_a_layer_that_overlaps_the_launch_starts_the_next_one(dtype):
    """Layers 0 and 3 of one call share a slab, and so do layers 1 and 4: each adds once, in call order, exactly as
    separate calls would."""
    heads, hw, tokens, d = 3, 128, 64, 32
    ins = [_inputs(DT[dtype], 2, heads, hw, tokens, d, seed=40 + i) for i in range(5)]

    def run(split):
        a, b, c = (torch.zeros(1, tokens, hw, device='cuda') for _ in range(3))
        descs = [ops.make_joint_desc(q, k, lse, hw, t, heads, s, reduce_heads=True)
                 for (q, k, lse, s), t in zip(ins, [a, b, c, a, b])]
        for i in range(0, 5, split):
            ops.accumulate_joint_heads(descs[i:i + split], 'cuda')
        return a, b, c
    together, apart = run(5), run(1)
    assert all(torch.equal(x, y) for x, y in zip(together, apart))
    a = together[0]
    r0, b0 = mean_and_bound(*_per_head_ref(*ins[0][:3], hw, tokens, ins[0][3], slice(1, 2)))
    r3, b3 = mean_and_bound(*_per_head_ref(*ins[3][:3], hw, tokens, ins[3][3], slice(1, 2)), r0, b0)
    _check(a, r3, b3, 'shared slab')


# ---- trace(pipe, reduce_heads=True) ---------------------------------------------------------------------------------
def _traced(model, dtype, prompt, steps=2, reduce_heads=True, **kw):
    """A traced generation of the synthetic SD3 or FLUX pipeline; records every layer call's ``(layer, q, k)``."""
    if model == 'sd3':
        pipe = make_sd3_pipeline(TINY_SD3_SPEC, dtype=dtype, device='cuda', seed=0)
    else:
        pipe = make_flux_pipeline(TINY_FLUX_SPEC, dtype=dtype, device='cuda', seed=0)
        kw.setdefault('max_sequence_length', TINY_FLUX_SPEC.t5_rows)
    calls = []
    with trace(pipe, reduce_heads=reduce_heads, **kw.pop('trace_kw', {})) as tc:
        enqueue = tc._enqueue_joint

        def record(layer_idx, q, k, lse, n_image, heads, scale):
            calls.append((layer_idx, q.detach().clone(), k.detach().clone()))
            return enqueue(layer_idx, q, k, lse, n_image, heads, scale)
        tc._enqueue_joint = record
        out = pipe(prompt, num_inference_steps=steps, **kw)
        tc.synchronize()
    return pipe, tc, calls, out


def _per_layer(model, calls, grid, heads, tokens):
    if model == 'sd3':
        return joint64.joint_maps(calls, grid[0] * grid[1], grid, heads)
    return flux64.flux_maps(calls, tokens, grid, heads)


def _rows(model, pipe, per_layer, prompt, tokens, prompt_idx=0, images=1, normalize=False):
    """The float64 map a read returns: SD3 the CLIP rows, FLUX the T5 rows after the zero row."""
    if model == 'sd3':
        return joint64.global_rows(per_layer, range(len(prompt.split()) + 2), prompt=prompt_idx, images=images,
                                   normalize=normalize)
    n = t5_rows(len(pipe.tokenizer_2.tokenize(prompt)), tokens, clip_tokens=0)
    return flux64.global_rows(per_layer, n, prompt=prompt_idx, images=images, normalize=normalize)


def _tol(got, ref, what, rtol=2e-3):
    """The tolerance of the per-head trace tests: the lse enters from SDPA, not float64."""
    err = (got.double().cpu() - ref.cpu()).abs()
    lim = rtol * ref.abs().cpu() + 1e-6 * float(ref.abs().max())
    assert (err <= lim).all(), f'{what}: worst {float((err - lim).max()):.3e}'


def _same_sums(got, ref, n_terms, what):
    """Two fp32 reductions of the same positive values (the kernel's v_h, identical in both traces) in other orders:
    each differs from the exact sum by at most n_terms roundings of a partial sum no larger than the whole."""
    lim = 2 * n_terms * U * ref.double().abs() * 1.01 + 1e-37
    err = (got.double() - ref.double()).abs()
    assert (err <= lim).all(), f'{what}: worst {float((err - lim).max()):.3e}'


def _spec(model):
    return TINY_SD3_SPEC if model == 'sd3' else TINY_FLUX_SPEC


def _tokens(model):
    return 77 + TINY_SD3_SPEC.t5_rows if model == 'sd3' else TINY_FLUX_SPEC.t5_rows


def _n_layers(model):
    return TINY_SD3_SPEC.blocks if model == 'sd3' else TINY_FLUX_SPEC.double + TINY_FLUX_SPEC.single


@pytest.mark.parametrize('model', ['sd3', 'flux'])
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16, torch.float16])
def test_trace_maps_match_float64_and_the_per_head_trace(model, dtype, tmp_path):
    prompt = 'a cute giraffe eating leaves'
    pipe, tc, calls, _ = _traced(model, dtype, prompt)
    _, per_head, _, _ = _traced(model, dtype, prompt, reduce_heads=False)
    grid, heads, tokens = tc.geometry.grid, _spec(model).heads, _tokens(model)
    per_layer = _per_layer(model, calls, grid, heads, tokens)
    steps, layers = 2, _n_layers(model)
    for slab in tc.all_heat_maps.live_slabs():
        assert slab.acc.numel() * 4 == slab.acc.shape[0] * slab.images * tokens * grid[0] * grid[1] * 4
        assert tuple(slab.acc.shape) == (1, 1, tokens, grid[0] * grid[1]) and slab.head_mean == heads
    ghm = tc.compute_global_heat_map()
    _tol(ghm.heat_maps, _rows(model, pipe, per_layer, prompt, tokens), 'global')
    _tol(tc.compute_global_heat_map(normalize=True).heat_maps,
         _rows(model, pipe, per_layer, prompt, tokens, normalize=True), 'normalized')
    n_terms = steps + heads + layers * heads + 4
    _same_sums(ghm.heat_maps, per_head.compute_global_heat_map().heat_maps, n_terms, 'vs the per-head trace')
    for layer in range(layers):
        one = tc.compute_global_heat_map(layer_idx=layer).heat_maps
        _tol(one, _rows(model, pipe, {layer: per_layer[layer]}, prompt, tokens), f'layer {layer}')
        _same_sums(one, per_head.compute_global_heat_map(layer_idx=layer).heat_maps, n_terms, f'layer {layer}')
    stack = tc.compute_layer_heat_maps()
    assert stack.layers == list(range(layers))
    for i, layer in enumerate(stack.layers):
        assert torch.equal(stack.heat_maps[i], tc.compute_global_heat_map(layer_idx=layer).heat_maps)
    factors = tc.compute_factor_heat_maps()
    assert list(factors.factors) == [1]
    assert torch.equal(factors.heat_maps[0], tc.compute_global_heat_map(factors={1}).heat_maps)
    images = tc.compute_image_heat_maps()
    assert torch.equal(images.heat_maps[0], tc.compute_global_heat_map(image_idx=0).heat_maps)
    if model == 'sd3':                                  # the T5 rows of the same slabs
        t5 = tc.compute_global_heat_map(encoder='t5')
        _same_sums(t5.heat_maps, per_head.compute_global_heat_map(encoder='t5').heat_maps, n_terms, 't5')
        assert torch.equal(tc.compute_layer_heat_maps(encoder='t5').heat_maps[1],
                           tc.compute_global_heat_map(encoder='t5', layer_idx=1).heat_maps)
    words = ['giraffe', 'leaves']
    _, expanded = ghm.expand_words(words, _Image(128, 128))
    assert expanded.shape == (2, 128, 128) and torch.isfinite(expanded).all()
    assert ghm.segment(words, _Image(128, 128)) is not None
    assert torch.equal(tc.to_experiment(tmp_path).global_heat_map, ghm.heat_maps)
    with pytest.raises(ValueError, match='head_idx'):
        tc.compute_global_heat_map(head_idx=0)
    with pytest.raises(RuntimeError, match='reduce_heads'):
        tc.compute_per_head_heat_maps()


class _Image:
    def __init__(self, h, w):
        self.height, self.width, self.size = h, w, (w, h)


@pytest.mark.parametrize('model', ['sd3', 'flux'])
@pytest.mark.parametrize('launch', ['step', 'layer'])
def test_batch_prompts_four_images_and_launch_modes(model, launch):
    prompts = ['a cat on a mat', 'two birds in flight']
    pipe, tc, calls, _ = _traced(model, torch.bfloat16, prompts, trace_kw=dict(batch_prompts=True, launch=launch),
                                 num_images_per_prompt=4)
    grid, heads, tokens = tc.geometry.grid, _spec(model).heads, _tokens(model)
    per_layer = _per_layer(model, calls, grid, heads, tokens)
    for slab in tc.all_heat_maps.live_slabs():
        assert slab.acc.numel() * 4 == 8 * tokens * grid[0] * grid[1] * 4 and slab.heads == slab.images == 4
    for p, prompt in enumerate(prompts):
        ghm = tc.compute_global_heat_map(prompt_idx=p)
        _tol(ghm.heat_maps, _rows(model, pipe, per_layer, prompt, tokens, prompt_idx=p, images=4), f'prompt {p}')
        images = tc.compute_image_heat_maps(prompt_idx=p)
        for i in range(4):
            one = tc.compute_global_heat_map(prompt_idx=p, image_idx=i)
            assert torch.equal(images.heat_maps[i], one.heat_maps)
            ref = _rows(model, pipe, {l: m[p * 4 + i:p * 4 + i + 1] for l, m in per_layer.items()}, prompt, tokens)
            _tol(one.heat_maps, ref, f'prompt {p} image {i}')
        layers = tc.compute_layer_heat_maps(prompt_idx=p, image_idx=2)
        assert torch.equal(layers.heat_maps[1],
                           tc.compute_global_heat_map(prompt_idx=p, image_idx=2, layer_idx=1).heat_maps)


@pytest.mark.parametrize('model', ['sd3', 'flux'])
def test_rectangular_generation(model):
    kw = dict(max_sequence_length=512) if model == 'sd3' else {}   # SD3: a 589-row context (77 CLIP + 512 T5)
    prompt = 'a lighthouse on a cliff'
    pipe, tc, calls, _ = _traced(model, torch.bfloat16, prompt, height=1216, width=832, steps=1, **kw)
    assert tc.geometry.grid == (76, 52)
    tokens = 589 if model == 'sd3' else _tokens(model)
    per_layer = _per_layer(model, calls, (76, 52), _spec(model).heads, tokens)
    _tol(tc.compute_global_heat_map().heat_maps, _rows(model, pipe, per_layer, prompt, tokens), '1216x832')
    for slab in tc.all_heat_maps.live_slabs():
        assert slab.acc.numel() * 4 == tokens * 76 * 52 * 4
    if model == 'sd3':
        pieces = t5_rows(len(pipe.tokenizer_3.tokenize(prompt)), tokens)
        ref = joint64.global_rows(per_layer, range(pieces + 2), first_row=76)
        ref[0] = 0
        _tol(tc.compute_global_heat_map(encoder='t5').heat_maps, ref, 't5 589 rows')


@pytest.mark.parametrize('dtype, backend', [(torch.bfloat16, SDPBackend.FLASH_ATTENTION),
                                            (torch.float16, SDPBackend.FLASH_ATTENTION),
                                            (torch.float32, SDPBackend.EFFICIENT_ATTENTION)])
def test_hooked_forward_is_bit_identical(dtype, backend):
    sd3 = make_sd3_pipeline(TINY_SD3_SPEC, dtype=dtype, device='cuda', seed=1)
    g = torch.Generator(device='cuda').manual_seed(3)
    x = torch.randn(4, 4, 32, 32, generator=g, device='cuda').to(dtype)
    ctx = torch.randn(4, 93, 64, generator=g, device='cuda').to(dtype)
    t = torch.full((4,), 500.0, device='cuda')
    with torch.no_grad(), sdpa_kernel(backend):
        plain = sd3.transformer(hidden_states=x, encoder_hidden_states=ctx, timestep=t)[0]
        with trace(sd3, batch_prompts=True, reduce_heads=True):
            sd3.check_inputs(['a', 'b'], None, None, 256, 256)
            hooked = sd3.transformer(hidden_states=x, encoder_hidden_states=ctx, timestep=t)[0]
    assert torch.equal(plain, hooked)
    flux = make_flux_pipeline(TINY_FLUX_SPEC, dtype=dtype, device='cuda', seed=1)
    T = TINY_FLUX_SPEC.t5_rows
    g = torch.Generator(device='cuda').manual_seed(4)
    kw = dict(hidden_states=torch.randn(2, 256, TINY_FLUX_SPEC.in_channels, generator=g, device='cuda').to(dtype),
              encoder_hidden_states=torch.randn(2, T, TINY_FLUX_SPEC.joint_attention_dim, generator=g,
                                                device='cuda').to(dtype),
              pooled_projections=torch.randn(2, TINY_FLUX_SPEC.pooled_projection_dim, generator=g,
                                             device='cuda').to(dtype),
              timestep=torch.full((2,), 0.5, device='cuda', dtype=dtype),
              img_ids=flux_image_ids(16, 16, 'cuda').to(dtype), txt_ids=torch.zeros(T, 3, device='cuda', dtype=dtype),
              guidance=torch.full((2,), 3.5, device='cuda'))
    with torch.no_grad(), sdpa_kernel(backend):
        plain = flux.transformer(**kw)[0]
        with trace(flux, batch_prompts=True, reduce_heads=True) as tc:
            flux.check_inputs(['a', 'b'], None, 256, 256)
            hooked = flux.transformer(**kw)[0]
            tc.synchronize()
            assert all(s.head_mean == TINY_FLUX_SPEC.heads for s in tc.all_heat_maps.live_slabs())
    assert torch.equal(plain, hooked)
