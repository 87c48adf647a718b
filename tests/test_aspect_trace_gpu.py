"""Traced generations at non-square latents against float64: per-key slabs, global maps under every filter, word maps,
expand_words, per-step and step-range maps, batched prompts, save_heads / load_heads, CUDA-graph replay, a tracer that
switches between square and transposed non-square latents, the 1:4 latent the square rule used to scramble, and two
production-size generations (SDXL 1216x832 fp16, SD-2.1 512x768 bf16)."""
from types import SimpleNamespace

import pytest
import torch

from daam_b200 import trace
from daam_b200.geometry import LatentGeometry
from daam_b200.testing.synthetic import SD21_SPEC, SDXL_SPEC, TINY_SPEC, UNetSpec, make_pipeline
from tests.reference64 import MAP_DIMS, assert_close64, bicubic64, layer_maps64

pytestmark = pytest.mark.gpu
DEV = 'cuda'
PROMPT = 'a dog chasing a red ball on the beach'
FILTERS = [{}, {'normalize': True}, {'factors': [1, 2]}, {'layer_idx': 9, 'head_idx': 0}, {'head_idx': 1}]
# an SDXL-topology tree (sample_size 128 -> g = 2; no cross-attention at the first level, factors 1 and 2)
TINY_XL = UNetSpec('tiny-xl', 128, (32, 64, 64), (1, 2, 2), (0, 1, 1), 64, mid_depth=1)
RTOL, ATOL = 1e-3, 1e-4           # the global-map tolerance of the 16-bit traced tests, per step


@pytest.fixture(autouse=True)
def _exact_fp32():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def bits(t):
    return t.contiguous().view(torch.int32)


class Recorder:
    """Device copies of every (layer, factor, q, k) the hooks hand to the kernel, grouped by UNet forward."""

    def __init__(self, tc, unet):
        self.steps = []
        self.tc, inner = tc, tc._enqueue
        self.handle = unet.register_forward_pre_hook(lambda *_: self.steps.append([]))

        def enqueue(layer_idx, factor, q, k, heads, scale):
            self.steps[-1].append((layer_idx, factor, q.detach().clone(), k.detach().clone(), heads, scale))
            return inner(layer_idx, factor, q, k, heads, scale)

        tc._enqueue = enqueue

    def stop(self):
        self.handle.remove()
        del self.tc._enqueue                                     # back to the class's method


def _up64(keys, grid):
    by = bicubic64(keys.shape[-2], grid[0], keys.device)
    bx = bicubic64(keys.shape[-1], grid[1], keys.device)
    return by @ keys.double() @ bx.T


def _keys64(rec, geometry, steps=None, prompt=0):
    """layer -> (factor, [heads, 77, h, w] float64 time sum over ``steps``) from the recorded Q/K."""
    out = {}
    for s in (range(len(rec.steps)) if steps is None else steps):
        for layer_idx, factor, q, k, heads, scale in rec.steps[s]:
            m = layer_maps64(q, k, heads, scale)[prompt]
            h, w, f = geometry.level(m.shape[-1], layer_idx)
            assert f == factor
            m = m.reshape(m.shape[0], m.shape[1], h, w)
            out[layer_idx] = (factor, m if layer_idx not in out else out[layer_idx][1] + m)
    return out


def _global64(keys, grid, n_rows, factors=None, layer_idx=None, head_idx=None, normalize=False):
    total, n = None, 0
    for layer, (factor, m) in keys.items():
        if (factors is not None and factor not in factors) or (layer_idx is not None and layer != layer_idx):
            continue
        sel = m[:, :n_rows] if head_idx is None else m[head_idx:head_idx + 1, :n_rows]
        part = _up64(sel, grid).clamp_(min=0.0).sum(dim=0)
        total = part if total is None else total + part
        n += sel.shape[0]
    out = total / n
    return out / (out[1:-1].sum(dim=0, keepdim=True) + 1e-6) if normalize else out


def _image(h, w):
    return SimpleNamespace(height=h, width=w, size=(w, h))     # the PIL surface expand_as reads


def _run(spec, dtype, height, width, steps=2, seed=3, **kw):
    pipe = make_pipeline(spec, dtype=dtype, device=DEV, seed=seed)
    with trace(pipe, **kw) as tc:
        rec = Recorder(tc, pipe.unet)
        pipe(PROMPT, num_inference_steps=steps, generator=torch.Generator().manual_seed(7), height=height, width=width)
        rec.stop()
        yield pipe, tc, rec


@pytest.mark.parametrize('spec,hw', [(TINY_SPEC, (768, 512)), (TINY_SPEC, (512, 768)), (TINY_XL, (1216, 832))],
                         ids=['tiny-512x768', 'tiny-768x512', 'tinyxl-1216x832'])
@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16, torch.float16])
def test_traced_maps_against_float64(spec, hw, dtype):
    steps = 2
    for pipe, tc, rec in _run(spec, dtype, *hw, steps=steps):
        geo = tc.geometry
        assert geo.grid == ((hw[0] // 8 + geo.g - 1) // geo.g, (hw[1] // 8 + geo.g - 1) // geo.g)
        keys = _keys64(rec, geo)
        for (factor, layer, head), got in tc.all_heat_maps:
            ref_factor, m = keys[layer]
            assert factor == ref_factor and got.shape == m.shape[1:]
            assert_close64(got, m[head], RTOL, ATOL * steps, f'layer {layer} head {head}', ('token', 'y', 'x'))
        n_rows = len(PROMPT.split()) + 2
        for f in FILTERS:
            if 'layer_idx' in f and f['layer_idx'] not in keys:
                continue
            got = tc.compute_global_heat_map(**f)
            assert tuple(got.heat_maps.shape) == (n_rows,) + geo.grid
            ref = _global64(keys, geo.grid, n_rows, **f)
            assert_close64(got.heat_maps, ref, RTOL, ATOL * steps, f'{f}', MAP_DIMS)
        hm = tc.compute_global_heat_map()
        dog = hm.compute_word_heat_map('dog')
        assert tuple(dog.heatmap.shape) == geo.grid
        assert_close64(dog.heatmap, hm.heat_maps[2].double(), 1e-6, 0.0, 'word map')
        image = _image(*hw)
        mask = dog.expand_as(image)
        assert tuple(mask.shape) == hw
        words, masks = hm.expand_words(['dog', 'ball'], image)
        assert tuple(masks.shape) == (2,) + hw
        assert torch.allclose(masks[0], mask, atol=1e-6)
        ref = _up64(hm.heat_maps[2][None].double(), hw)[0]
        ref = (ref - ref.min()) / (ref.max() - ref.min() + 1e-8)
        assert_close64(masks[0], ref.cpu(), 1e-5, 1e-6, 'expand_words')
        per_head_keys, per_head = tc.compute_per_head_heat_maps()
        assert tuple(per_head.shape[-2:]) == geo.grid and len(per_head_keys) == per_head.shape[0]


def test_time_resolved_step_equals_a_one_step_trace():
    hw = (768, 512)
    for _, tc, rec in _run(TINY_SPEC, torch.float32, *hw, steps=3, time_resolved=True):
        tm = tc.compute_time_heat_maps()
        assert tuple(tm.heat_maps.shape[-2:]) == tc.geometry.grid and len(tm) == 3
        assert tuple(tm.word_heat_maps('dog').shape) == (3,) + tc.geometry.grid
        n_rows = tm.heat_maps.shape[1]
        for t in range(3):
            ref = _global64(_keys64(rec, tc.geometry, [t]), tc.geometry.grid, n_rows)
            assert_close64(tm.heat_maps[t], ref, RTOL, ATOL, f'step {t}', MAP_DIMS)
    # step 0 of a time-resolved trace is bit-equal to a one-step trace's global map
    for _, tc, _ in _run(TINY_SPEC, torch.float32, *hw, steps=1):
        one = tc.compute_global_heat_map().heat_maps.clone()
    for _, tc, _ in _run(TINY_SPEC, torch.float32, *hw, steps=2, time_resolved=True):
        assert torch.equal(bits(tc.compute_time_heat_maps().heat_maps[0]), bits(one))


def test_step_ranges_batch_prompts_and_graph_replay():
    hw = (512, 768)
    for _, tc, rec in _run(TINY_XL, torch.float16, 1216, 832, steps=4, step_ranges=[(1, 3)]):
        got = tc.compute_global_heat_map(step_range=0).heat_maps
        ref = _global64(_keys64(rec, tc.geometry, [1, 2]), tc.geometry.grid, got.shape[0])
        assert_close64(got, ref, RTOL, 2 * ATOL, 'step range', MAP_DIMS)
    # batched prompts: prompt i's map equals a single-prompt trace of it
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float32, device=DEV, seed=3)
    prompts = [PROMPT, 'a cat on a sofa']
    with trace(pipe, batch_prompts=True) as tc:
        rec = Recorder(tc, pipe.unet)
        pipe(prompts, num_inference_steps=2, generator=torch.Generator().manual_seed(7), height=hw[0], width=hw[1])
        for i, p in enumerate(prompts):
            got = tc.compute_global_heat_map(prompt_idx=i).heat_maps
            ref = _global64(_keys64(rec, tc.geometry, prompt=i), tc.geometry.grid, len(p.split()) + 2)
            assert_close64(got, ref, RTOL, 2 * ATOL, f'prompt {i}', MAP_DIMS)
    # CUDA-graph replay is bit-equal to eager
    maps = []
    for graph in (False, True):
        pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=4, cuda_graph=graph)
        with trace(pipe) as tc:
            pipe(PROMPT, num_inference_steps=4, generator=torch.Generator().manual_seed(9), height=hw[0], width=hw[1])
            maps.append(tc.compute_global_heat_map().heat_maps.clone())
    assert tuple(maps[0].shape[-2:]) == (64, 96)
    assert torch.equal(bits(maps[0]), bits(maps[1]))


def test_save_heads_and_load_heads(tmp_path):
    hw = (768, 512)
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float32, device=DEV, seed=5)
    with trace(pipe, save_heads=True, data_dir=str(tmp_path)) as tc:
        pipe(PROMPT, num_inference_steps=2, generator=torch.Generator().manual_seed(2), height=hw[0], width=hw[1])
        saved = tc.compute_global_heat_map().heat_maps.clone()
    with trace(pipe, load_heads=True, data_dir=str(tmp_path)) as tc:
        pipe(PROMPT, num_inference_steps=2, generator=torch.Generator().manual_seed(2), height=hw[0], width=hw[1])
        loaded = tc.compute_global_heat_map().heat_maps.clone()
    with trace(pipe) as tc:
        pipe(PROMPT, num_inference_steps=2, generator=torch.Generator().manual_seed(2), height=hw[0], width=hw[1])
        fused = tc.compute_global_heat_map().heat_maps.clone()
    assert tuple(saved.shape[-2:]) == (96, 64)
    assert torch.equal(saved, loaded)
    assert_close64(saved, fused.double(), 1e-4, 1e-6, 'materialised vs fused', MAP_DIMS)


def test_one_tracer_across_square_and_transposed_latents():
    """square -> 512x768 -> 768x512 -> square on one tracer: the square runs are bit-identical to a fresh tracer's, the
    transposed run re-tags every slab (same query counts, transposed keys) and matches float64."""
    def gen(pipe, tc, hw):
        pipe(PROMPT, num_inference_steps=2, generator=torch.Generator().manual_seed(7), height=hw[0], width=hw[1])
        return tc.compute_global_heat_map().heat_maps.clone()

    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=3)
    with trace(pipe) as tc:
        fresh = gen(pipe, tc, (512, 512))
    with trace(pipe) as tc:
        first = gen(pipe, tc, (512, 512))
        tall = gen(pipe, tc, (512, 768))
        rec = Recorder(tc, pipe.unet)
        wide = gen(pipe, tc, (768, 512))
        rec.stop()
        shapes = {layer: key.shape for (_, layer, _), key in tc.all_heat_maps}
        last = gen(pipe, tc, (512, 512))
    assert torch.equal(bits(fresh), bits(first)) and torch.equal(bits(fresh), bits(last))
    assert tuple(tall.shape[-2:]) == (64, 96) and tuple(wide.shape[-2:]) == (96, 64)
    keys = _keys64(rec, LatentGeometry(4096, pipe.unet.config.sample_size, (96, 64)))
    for layer, (_, m) in keys.items():
        assert tuple(shapes[layer]) == tuple(m.shape[1:])
    assert_close64(wide, _global64(keys, (96, 64), wide.shape[0]), RTOL, 2 * ATOL, 'transposed run', MAP_DIMS)


def test_one_to_four_latent_matches_float64():
    """32x128 (256x1024 pixels): every level has a square pixel count, which the square rule reshaped as
    sqrt(n) x sqrt(n) -- scrambled maps. The geometry rule keys them [h, w] and the maps match float64."""
    for _, tc, rec in _run(TINY_SPEC, torch.float32, 256, 1024):
        got = tc.compute_global_heat_map().heat_maps
        assert tuple(got.shape[-2:]) == (32, 128)
        ref = _global64(_keys64(rec, tc.geometry), (32, 128), got.shape[0])
        assert_close64(got, ref, RTOL, 2 * ATOL, '1:4 latent', MAP_DIMS)


@pytest.mark.parametrize('spec,dtype,hw', [(SDXL_SPEC, torch.float16, (1216, 832)),
                                         (SD21_SPEC, torch.bfloat16, (512, 768))],
                         ids=['sdxl-1216x832-fp16', 'sd21-512x768-bf16'])
def test_production_size_against_float64(spec, dtype, hw):
    steps = 2
    pipe = make_pipeline(spec, 'skeleton', dtype=dtype, device=DEV, seed=1, init_on_device=True)
    with trace(pipe) as tc:
        rec = Recorder(tc, pipe.unet)
        pipe(PROMPT, num_inference_steps=steps, generator=torch.Generator().manual_seed(7), height=hw[0], width=hw[1])
        got = tc.compute_global_heat_map().heat_maps
        geo = tc.geometry
        ref = _global64(_keys64(rec, geo), geo.grid, got.shape[0])
    assert tuple(got.shape[-2:]) == geo.grid
    assert_close64(got, ref, RTOL, ATOL * steps, f'{spec.name} {hw}', MAP_DIMS)
