"""Layer-, factor- and head-resolved heat maps through the tracer, on the synthetic SD-2.1 and SDXL skeletons:
compute_layer_heat_maps()[i] bit-equal to compute_global_heat_map(layer_idx=...), compute_factor_heat_maps()[j] to
compute_global_heat_map(factors={f}), compute_head_heat_maps() to compute_per_head_heat_maps, under every filter and
trace mode a read takes; the word-list calls over each stack; the launch count; and the error messages."""
from types import SimpleNamespace

import pytest
import torch

from daam_b200 import _native, trace
from daam_b200.heatmap import FactorHeatMaps, HeadHeatMaps, LayerHeatMaps
from daam_b200.testing.synthetic import SD21_SPEC, SDXL_SPEC, TINY_SPEC, make_pipeline

pytestmark = pytest.mark.gpu
DEV = 'cuda'
PROMPT = 'a dog chasing a red ball on the beach'


def _check_stacks(tc, what='', **kw):
    """Both stacks against the single-map reads with the same arguments; returns them."""
    by_layer = tc.compute_layer_heat_maps(**kw)
    assert isinstance(by_layer, LayerHeatMaps) and len(by_layer) == len(by_layer.layers) > 0
    for i, (layer, name, factor) in enumerate(zip(by_layer.layers, by_layer.names, by_layer.factors)):
        one = tc.compute_global_heat_map(layer_idx=layer, **kw)
        assert torch.equal(by_layer.heat_maps[i], one.heat_maps), (what, kw, layer)
        assert one.prompt == by_layer.prompt
        assert name == tc.layer_names[layer] and factor == tc.all_heat_maps.slabs[layer].factor
    by_factor = tc.compute_factor_heat_maps(**kw)
    assert isinstance(by_factor, FactorHeatMaps) and by_factor.factors == sorted(set(by_factor.factors))
    rest = {k: v for k, v in kw.items() if k != 'factors'}
    for j, f in enumerate(by_factor.factors):
        one = tc.compute_global_heat_map(factors={f}, **rest)
        assert torch.equal(by_factor.heat_maps[j], one.heat_maps), (what, kw, f)
    assert set(by_factor.factors) == set(by_layer.factors)
    return by_layer, by_factor


@pytest.mark.parametrize('spec,layers', [(SD21_SPEC, 15), (SDXL_SPEC, None)], ids=['sd21', 'sdxl'])
def test_stacks_equal_the_single_reads(monkeypatch, spec, layers):
    pipe = make_pipeline(spec, dtype=torch.float16, device=DEV, seed=1, init_on_device=True)
    with trace(pipe) as tc:
        pipe(PROMPT, num_inference_steps=2, generator=torch.Generator().manual_seed(3))
        live = tc.all_heat_maps.live_slabs()
        by_layer, by_factor = _check_stacks(tc, spec.name)
        assert by_layer.layers == [s.layer_idx for s in live] and (layers is None or len(by_layer) == layers)
        assert by_layer.heat_maps.shape[1:] == (len(PROMPT.split()) + 2,) + tuple(tc.geometry.grid)
        for kw in [{'normalize': True}, {'factors': {1, 4}}, {'factors': [2]}, {'head_idx': 7},
                   {'head_idx': 2, 'normalize': True}]:
            _check_stacks(tc, spec.name, **kw)
        # head 7 exists in the layers with more than 7 heads only
        assert tc.compute_layer_heat_maps(head_idx=7).layers == [s.layer_idx for s in live if s.heads > 7]
        one_layer = tc.compute_factor_heat_maps(layer_idx=live[0].layer_idx)
        assert one_layer.factors == [live[0].factor]
        assert torch.equal(one_layer.heat_maps[0], tc.compute_global_heat_map(layer_idx=live[0].layer_idx).heat_maps)
        # one finalize launch for every layer, two with the normalisation; no single-map call
        monkeypatch.setattr(_native, 'finalize', None)
        for normalize, launches in ((False, 1), (True, 2)):
            before = _native.launch_count()
            stack = tc.compute_layer_heat_maps(normalize=normalize)
            assert len(stack) <= _native.FINALIZE_MAX_MAPS and _native.launch_count() - before == launches
            before = _native.launch_count()
            tc.compute_factor_heat_maps(normalize=normalize)
            assert _native.launch_count() - before == launches


def test_stacks_in_every_trace_mode():
    """negative, a step range, several images (image_idx), batch_prompts with prompt_idx."""
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=5)
    prompts = ['a dog on the beach', 'a red ball in a park today']
    with trace(pipe, batch_prompts=True, negative=True, step_ranges=[(1, 3)]) as tc:
        pipe(prompts, num_inference_steps=3, generator=torch.Generator().manual_seed(2), num_images_per_prompt=2,
             negative_prompt='blurry photo')
        rows = set()
        for p in range(2):
            for src in [{}, {'negative': True}, {'step_range': 0}, {'step_range': 0, 'negative': True},
                        {'image_idx': 1}, {'image_idx': 0, 'negative': True, 'normalize': True, 'head_idx': 1}]:
                by_layer, _ = _check_stacks(tc, f'prompt {p}', prompt_idx=p, **src)
                rows.add(by_layer.heat_maps.shape[1])
        assert rows == {4, 7, 9}                               # 'blurry photo', and the two prompts
        with pytest.raises(IndexError):
            tc.compute_layer_heat_maps(image_idx=2)
        with pytest.raises(IndexError):
            tc.compute_factor_heat_maps(step_range=1)


@pytest.mark.parametrize('size', [(512, 768), (600, 800)], ids=['512x768', '600x800'])
def test_stacks_at_non_square_and_off_grid_sizes(size):
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float32, device=DEV, seed=3)
    with trace(pipe) as tc:
        pipe(PROMPT, num_inference_steps=2, height=size[0], width=size[1])
        by_layer, _ = _check_stacks(tc, str(size))
        _check_stacks(tc, str(size), normalize=True)
        assert tuple(by_layer.heat_maps.shape[-2:]) == tuple(tc.geometry.grid) == (size[0] // 8, size[1] // 8)


def test_stacks_of_a_long_prompt():
    """A 154-token context whose prompt reaches into the second chunk: the stacks hold the compact rows."""
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=3)
    words = [f'w{i}' for i in range(100)]
    words[20], words[90] = 'dog', 'ball'
    prompt = ' '.join(words)
    g = torch.Generator().manual_seed(5)
    c = pipe.unet.spec.cross_attention_dim
    with trace(pipe, long_prompts=True) as tc:
        pipe(prompt_embeds=torch.randn(1, 154, c, generator=g), negative_prompt_embeds=torch.randn(1, 154, c, generator=g),
             num_inference_steps=2)
        for kw in ({}, {'normalize': True}):
            by_layer, by_factor = _check_stacks(tc, 'long', prompt=prompt, **kw)
            assert by_layer.heat_maps.shape[1] == by_factor.heat_maps.shape[1] == 102
        with pytest.raises(ValueError, match='prompt_embeds'):
            tc.compute_layer_heat_maps()


def test_head_stack_and_word_lists():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float32, device=DEV, seed=3)
    with trace(pipe) as tc:
        pipe(PROMPT, num_inference_steps=2, generator=torch.Generator().manual_seed(11))
        for kw in ({}, {'factors': {1}}, {'normalize': True, 'factors': [2, 4]}):
            keys, maps = tc.compute_per_head_heat_maps(**kw)
            by_head = tc.compute_head_heat_maps(**kw)
            assert isinstance(by_head, HeadHeatMaps) and by_head.keys == keys and torch.equal(by_head.heat_maps, maps)
            assert by_head.prompt == PROMPT
        factor, layer, head = by_head.keys[3]
        torch.testing.assert_close(by_head[3].heat_maps, tc.compute_global_heat_map(
            layer_idx=layer, head_idx=head, normalize=True).heat_maps, rtol=1e-6, atol=1e-9)
        image = SimpleNamespace(size=(256, 256), height=256, width=256)
        regions = torch.zeros(2, 256, 256, dtype=torch.bool, device=DEV)
        regions[0, 40:160, 30:200] = True
        regions[1, :, 128:] = True
        rgb = torch.randint(0, 256, (256, 256, 3), dtype=torch.uint8, generator=torch.Generator().manual_seed(1))
        words = ['dog', 'ball', 'beach']
        stacks = [tc.compute_layer_heat_maps(), tc.compute_factor_heat_maps(), tc.compute_head_heat_maps(factors={4})]
        for stack in stacks:
            _, labels, scores = stack.segment(words, image, threshold=0.4)
            _, ov = stack.region_overlap(words, image, regions, threshold=0.4)
            _, frames = stack.overlay_words(words, rgb)
            assert labels.shape[0] == ov.intersection.shape[0] == frames.shape[0] == len(stack)
            for t in range(len(stack)):
                _, li, si = stack[t].segment(words, image, threshold=0.4)
                assert torch.equal(labels[t], li) and torch.equal(scores[t], si)
                _, oi = stack[t].region_overlap(words, image, regions, threshold=0.4)
                assert torch.equal(ov.intersection[t], oi.intersection) and torch.equal(ov.word_area[t], oi.word_area)
                _, fi = stack[t].overlay_words(words, rgb)
                assert torch.equal(frames[t], fi)
        by_layer = stacks[0]
        _, ov = by_layer.region_overlap(['dog'], image, regions, threshold=0.4)
        assert ov.iou().shape == (len(by_layer), 2, 1)
        assert by_layer.layers[ov.iou()[:, 0, 0].argmax()] in by_layer.layers     # the layer that localises 'dog' best


def test_error_messages():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float32, device=DEV, seed=3)
    with trace(pipe) as tc:
        for read in (tc.compute_layer_heat_maps, tc.compute_factor_heat_maps, tc.compute_head_heat_maps):
            with pytest.raises(RuntimeError, match='No heat maps found. Did you forget'):
                read()
        pipe(PROMPT, num_inference_steps=1)
        with pytest.raises(RuntimeError, match='No heat maps found for the given parameters'):
            tc.compute_layer_heat_maps(head_idx=99)
        with pytest.raises(RuntimeError, match='No heat maps found for the given parameters'):
            tc.compute_factor_heat_maps(layer_idx=99)
        with pytest.raises(RuntimeError, match='No heat maps found. Did you forget'):
            tc.compute_layer_heat_maps(factors={8})
        with pytest.raises(RuntimeError, match='negative=True'):
            tc.compute_layer_heat_maps(negative=True)
        with pytest.raises(RuntimeError, match='step_ranges'):
            tc.compute_factor_heat_maps(step_range=0)
    with trace(pipe, long_prompts=True) as tc:                # layers of two context lengths: one read reduces one
        pipe(PROMPT, num_inference_steps=1)
        live = tc.all_heat_maps.live_slabs()
        s = live[0]
        tc.all_heat_maps.slabs[s.layer_idx] = type(s)(s.layer_idx, s.factor, s.heads, s.h, s.w,
                                                      torch.zeros(1, s.heads, 154, s.h * s.w, device=DEV), touched=True)
        for read in (tc.compute_layer_heat_maps, tc.compute_factor_heat_maps):
            with pytest.raises(RuntimeError, match='contexts of \\[77, 154\\] tokens'):
                read()
