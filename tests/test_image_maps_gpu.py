"""Per-image heat maps through the tracer (num_images_per_prompt > 1): compute_global_heat_map(image_idx=i) against the
oracle fed image i's Q/K and against float64, compute_image_heat_maps()[i] bit-equal to it, the per-image maps
averaging to the blended map, and the combinations with negative, step_range, batch_prompts, a non-square size and
time_resolved."""
from types import SimpleNamespace

import pytest
import torch

from daam_b200 import trace
from daam_b200.testing.synthetic import TINY_SPEC, SyntheticPipeline, make_pipeline
from oracle import daam_oracle as O
from tests.reference64 import assert_close64, finalize_tolerance, global_map64
from tests.util import HookRecorder, rel_err

pytestmark = pytest.mark.gpu
DEV = 'cuda'
PROMPT = 'a dog chasing a red ball on the beach'


@pytest.fixture(autouse=True)
def _exact_fp32():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _image_store(rec, image, images, prompt_idx=0, n_prompts=1):
    """The oracle's heat maps over the keys of one image: the reference run on that image's CFG pair alone."""
    store = O.OracleHeatMaps()
    for layer_idx, factor, q, k, heads, scale in rec.calls:
        n = q.shape[0] // 2
        s = prompt_idx * images + image
        for head, m in enumerate(O.port_layer_step(q[[s, n + s]], k[[s, n + s]], heads, scale)):
            store.update(factor, layer_idx, head, m)
    return store


def _image_stacks(tc, image, prompt_idx=0, **src):
    """Image ``image``'s key stacks [H, 77, h, w] of every live slab (what a daam_key_group of that image points at)."""
    out = []
    for s in tc.all_heat_maps.read_slabs(src.get('step_range'), src.get('negative', False)):
        H = s.heads_per_image
        out.append(s.source(**src)[prompt_idx, image * H:(image + 1) * H].view(H, -1, s.h, s.w))
    return out


@pytest.mark.parametrize('images', [2, 3])
def test_image_maps_against_oracle_and_blend(images):
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float32, device=DEV, seed=3)
    n_tok = len(pipe.tokenizer.tokenize(PROMPT))
    with trace(pipe) as tc:
        rec = HookRecorder(tc)
        pipe(PROMPT, num_inference_steps=2, generator=torch.Generator().manual_seed(11), num_images_per_prompt=images)
        assert {s.images for s in tc.all_heat_maps.live_slabs()} == {images}
        per_image = tc.compute_image_heat_maps()
        assert per_image.heat_maps.shape == (images, n_tok + 2, 64, 64) and len(per_image) == images
        for i in range(images):
            store = _image_store(rec, i, images)
            for kw in [{}, {'normalize': True}, {'factors': [1, 2]}, {'layer_idx': 9, 'head_idx': 0}, {'head_idx': 1}]:
                got = tc.compute_global_heat_map(image_idx=i, **kw).heat_maps
                assert rel_err(got, O.port_global_heat_map(store, 4096, n_tok, **kw)) < 2e-5, (i, kw)
                many = tc.compute_image_heat_maps(**{k: v for k, v in kw.items()})
                assert torch.equal(many.heat_maps[i], got), (i, kw)
            stacks = _image_stacks(tc, i)
            ref = global_map64(stacks, 64, n_tok + 2)
            rtol, atol = finalize_tolerance(stacks, sum(t.shape[0] for t in stacks), 64)
            assert_close64(per_image.heat_maps[i], ref, rtol, atol, f'image {i}')
            assert torch.equal(per_image[i].heat_maps, per_image.heat_maps[i])
        # equal key counts per image: the mean of the per-image maps is the blended map up to rounding
        blended = tc.compute_global_heat_map().heat_maps
        assert rel_err(per_image.heat_maps.mean(0), blended) < 1e-5
        # the reference's meaning of head_idx is unchanged: an index over images x heads
        keys, maps = tc.compute_per_head_heat_maps(image_idx=images - 1)
        assert len(keys) == 25
        _, all_maps = tc.compute_per_head_heat_maps()
        first = start = 0
        for s in tc.all_heat_maps.live_slabs():       # image i's per-head maps are the blended sweep's keys i * H + h
            H = s.heads_per_image
            assert torch.equal(maps[first:first + H], all_maps[start + (images - 1) * H:start + images * H])
            first, start = first + H, start + s.heads
        words = per_image.word_heat_maps('ball')
        for i in range(images):
            assert torch.equal(words[i], per_image[i].compute_word_heat_map('ball').heatmap)
        image = SimpleNamespace(size=(256, 256), height=256, width=256)
        _, labels, scores = per_image.segment(['dog', 'ball', 'beach'], image)
        assert labels.shape == (images, 256, 256)
        for i in range(images):
            _, li, si = per_image[i].segment(['dog', 'ball', 'beach'], image)
            assert torch.equal(labels[i], li) and torch.equal(scores[i], si)
        for bad in (images, -1, 1.0):
            with pytest.raises(IndexError):
                tc.compute_global_heat_map(image_idx=bad)
        with pytest.raises(IndexError):
            tc.compute_per_head_heat_maps(image_idx=images)
        with pytest.raises(IndexError):
            tc.compute_image_heat_maps(prompt_idx=1)


def test_image_maps_negative_ranges_prompts_rectangular():
    """batch_prompts (2 prompts x 2 images), negative=True, a step range and a 512 x 768 image: every (prompt, image)
    map of each half and range against float64 over that image's keys, and compute_image_heat_maps bit-equal."""
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=5)
    prompts = ['a dog on the beach', 'a red ball in a park']
    with trace(pipe, batch_prompts=True, negative=True, step_ranges=[(1, 3)]) as tc:
        pipe(prompts, num_inference_steps=3, generator=torch.Generator().manual_seed(2), num_images_per_prompt=2,
             height=512, width=768, negative_prompt='blurry photo')
        for p in range(2):
            for src in [{}, {'negative': True}, {'step_range': 0}, {'step_range': 0, 'negative': True}]:
                many = tc.compute_image_heat_maps(prompt_idx=p, **src)
                n_rows = many.heat_maps.shape[1]
                for i in range(2):
                    one = tc.compute_global_heat_map(prompt_idx=p, image_idx=i, **src)
                    assert one.heat_maps.shape == (n_rows, 64, 96)
                    assert torch.equal(many.heat_maps[i], one.heat_maps), (p, i, src)
                    assert one.prompt == many.prompt
                    stacks = _image_stacks(tc, i, p, **src)
                    rtol, atol = finalize_tolerance(stacks, sum(t.shape[0] for t in stacks), 96)
                    ref = _rect_global64(stacks, (64, 96), n_rows)
                    assert_close64(one.heat_maps, ref, rtol, atol, f'prompt {p} image {i} {src}')
                blended = tc.compute_global_heat_map(prompt_idx=p, **src).heat_maps
                assert rel_err(many.heat_maps.mean(0), blended) < 1e-5


def _rect_global64(stacks, grid, n_rows):
    """global_map64 for a rectangular grid: per-axis float64 bicubic, clamp, mean over keys."""
    from tests.reference64 import bicubic64
    total, n = 0, 0
    for t in stacks:
        by, bx = bicubic64(t.shape[-2], grid[0], t.device), bicubic64(t.shape[-1], grid[1], t.device)
        total = total + (by @ t[:, :n_rows].double() @ bx.T).clamp_(min=0.0).sum(0)
        n += t.shape[0]
    return total / n


def _unet_inputs(n_images, steps, seed):
    g = torch.Generator().manual_seed(seed)
    spec = TINY_SPEC
    lat = [torch.randn(2 * n_images, spec.in_channels, 64, 64, generator=g).to(DEV) for _ in range(steps)]
    emb = torch.randn(2 * n_images, 77, spec.cross_attention_dim, generator=g).to(DEV)
    return lat, emb


@pytest.mark.parametrize('negative', [False, True])
def test_time_resolved_per_image_rows_equal_one_step_traces(monkeypatch, negative):
    """Per-image history row t equals compute_global_heat_map(image_idx=i) of a trace of step t only, bit for bit, and
    the blended history row equals that trace's blended map; the per-step launch is one finalize call."""
    from daam_b200 import _native
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float32, device=DEV, seed=4)
    images, steps = 3, 3
    lat, emb = _unet_inputs(images, steps, 9)
    t = torch.full((1,), 500.0, device=DEV)
    with torch.no_grad(), trace(pipe, time_resolved=True, negative=negative) as tc:
        tc.last_prompts, tc.last_prompt = ['a cat'], 'a cat'
        tc.last_negative_prompts = [''] if negative else []
        calls = []
        inner = _native.finalize_maps
        monkeypatch.setattr(_native, 'finalize_maps', lambda groups, maps, *a: (calls.append(len(maps)),
                                                                               inner(groups, maps, *a)))
        monkeypatch.setattr(_native, 'finalize', None)     # the step uses no single-map call
        for s in range(steps):
            pipe.unet(lat[s], t, emb)                       # the forward hook issues the step launch and its finalize
        monkeypatch.undo()
        hist = tc.compute_time_heat_maps(negative=negative).heat_maps
        per = [tc.compute_time_heat_maps(image_idx=i, negative=negative).heat_maps for i in range(images)]
        with pytest.raises(IndexError):
            tc.compute_time_heat_maps(image_idx=images)
    assert calls == [(1 + images) * (2 if negative else 1)] * steps   # one call per step: blended + every image
    for s in range(steps):
        with torch.no_grad(), trace(pipe, negative=negative) as one:
            one.last_prompts, one.last_prompt = ['a cat'], 'a cat'
            one.last_negative_prompts = [''] if negative else []
            pipe.unet(lat[s], t, emb)
            assert torch.equal(hist[s], one.compute_global_heat_map(negative=negative).heat_maps), s
            for i in range(images):
                ref = one.compute_global_heat_map(image_idx=i, negative=negative).heat_maps
                assert torch.equal(per[i][s], ref), (s, i)


def test_time_resolved_one_image_is_the_blended_history():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float32, device=DEV, seed=4)
    with trace(pipe, time_resolved=True) as tc:
        pipe(PROMPT, num_inference_steps=2)
        a = tc.compute_time_heat_maps().heat_maps
        b = tc.compute_time_heat_maps(image_idx=0).heat_maps
        assert a.data_ptr() == b.data_ptr() and torch.equal(a, b)
        assert list(tc._history[False]) == [(0, None)]          # no per-image history, no extra work
        with pytest.raises(IndexError):
            tc.compute_time_heat_maps(image_idx=1)


class StableDiffusionXLPipeline(SyntheticPipeline):
    """Named like diffusers' SDXL pipeline, so that the tracer hooks its image post-processing."""


def test_last_images_and_experiment(tmp_path):
    """last_images: every image, prompt-major (the SDXL post-process hook); to_experiment(image_idx=i) records image i."""
    base = make_pipeline(TINY_SPEC, dtype=torch.float32, device=DEV, seed=2)
    pipe = StableDiffusionXLPipeline(base.unet, dtype=torch.float32, device=DEV)
    with trace(pipe, batch_prompts=True) as tc:
        out = pipe(['a dog', 'a cat'], num_inference_steps=1, num_images_per_prompt=2)
        assert len(tc.last_images) == 4
        for a, b in zip(tc.last_images, out.images):
            assert a is b
        assert tc.last_image is out.images[0]
        exp = tc.to_experiment(tmp_path, prompt_idx=1, image_idx=1)
        assert exp.image is out.images[3]
        assert torch.equal(exp.global_heat_map, tc.compute_global_heat_map(prompt_idx=1, image_idx=1).heat_maps)
