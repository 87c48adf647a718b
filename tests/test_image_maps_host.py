"""Host-side rules of per-image heat maps that need no GPU: the new read arguments are keyword-only and off by default,
the synthetic pipeline repeats embeddings prompt-major and draws one latent per image (and exactly today's draws with
one image), and the safety-checker hook keeps every image in prompt-major order."""
import inspect

import numpy as np
import pytest
import torch

from daam_b200 import _native, trace
from daam_b200.heatmap import GlobalHeatMapStack, ImageHeatMaps, TimeHeatMaps
from daam_b200.testing.synthetic import TINY_SPEC, SyntheticPipeline, make_pipeline


def test_image_idx_is_keyword_only_and_off_by_default():
    for fn in (trace.compute_global_heat_map, trace.compute_per_head_heat_maps, trace.compute_time_heat_maps):
        p = inspect.signature(fn).parameters['image_idx']
        assert p.kind is inspect.Parameter.KEYWORD_ONLY and p.default is None, fn
    params = inspect.signature(trace.compute_image_heat_maps).parameters
    assert list(params)[1:6] == ['prompt_idx', 'factors', 'layer_idx', 'head_idx', 'normalize']
    for name in ('step_range', 'negative'):
        assert params[name].kind is inspect.Parameter.KEYWORD_ONLY
    assert issubclass(TimeHeatMaps, GlobalHeatMapStack) and issubclass(ImageHeatMaps, GlobalHeatMapStack)


def test_map_sel_layout_matches_the_header():
    assert ctypes_size(_native.DaamMapSel) == 24 and _native.DaamMapSel.out.offset == 16
    g = _native.DaamKeyGroup(acc=0, heads=1, h=1, w=1, tokens=77, head_sel=-1, reserved=7)
    assert g.n_blocks == 7 and g.reserved == 7 and ctypes_size(_native.DaamKeyGroup) == 32


def ctypes_size(t):
    import ctypes
    return ctypes.sizeof(t)


def _inputs(pipe, **kw):
    """The UNet inputs of a 1-step generation: (sample, encoder_hidden_states)."""
    seen = []
    h = pipe.unet.register_forward_pre_hook(lambda m, args: seen.append((args[0].clone(), args[2].clone())))
    try:
        out = pipe(['a cat', 'a dog'], num_inference_steps=1, generator=torch.Generator().manual_seed(5), **kw)
    finally:
        h.remove()
    return seen[0], out


def test_synthetic_pipeline_images_per_prompt_draws():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float32, device='cpu', seed=0)
    (lat1, emb1), out1 = _inputs(pipe)
    (lat0, emb0), out0 = _inputs(pipe, num_images_per_prompt=1)
    assert torch.equal(lat0, lat1) and torch.equal(emb0, emb1) and torch.equal(out0.latents, out1.latents)
    (lat3, emb3), out3 = _inputs(pipe, num_images_per_prompt=3)
    assert lat3.shape[0] == emb3.shape[0] == 12 and len(out3.images) == 6
    # embeddings: [uncond x (2 prompts x 3 images), cond x (...)], each prompt repeated in place (prompt-major)
    want = emb1.view(2, 2, *emb1.shape[1:]).repeat_interleave(3, dim=1).reshape(12, *emb1.shape[1:])
    assert torch.equal(emb3, want)
    g = torch.Generator().manual_seed(5)
    pipe.encode(['a cat', 'a dog'], g)                  # the same draws in the same order: embeddings, then latents
    lat = torch.randn(6, TINY_SPEC.in_channels, 64, 64, generator=g)
    assert torch.equal(lat3[:6], lat) and torch.equal(lat3[6:], lat)
    assert not torch.equal(lat[0], lat[1])              # one latent per image


class _WithSafetyChecker(SyntheticPipeline):
    def run_safety_checker(self, image, device=None, dtype=None):
        return image, None

    def numpy_to_pil(self, images):
        return [f'img{i}' for i in range(len(images))]


def test_safety_checker_hook_keeps_every_image_prompt_major():
    base = make_pipeline(TINY_SPEC, dtype=torch.float32, device='cpu', seed=0)
    pipe = _WithSafetyChecker(base.unet, dtype=torch.float32, device='cpu')
    pipe.image_processor = None
    tc = trace(pipe)
    tc.hook()
    try:
        pipe.run_safety_checker(np.zeros((4, 8, 8, 3)))
    finally:
        tc.unhook()
    assert tc.last_images == ['img0', 'img1', 'img2', 'img3']
    assert tc.last_image == 'img3'                      # the reference's rule: the last image
