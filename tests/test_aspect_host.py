"""Non-square images on the host: the geometry rule as a table, its refusals, the square rule left as it was, and the
synthetic UNet calling every attn2 with the query count the rule predicts. No GPU needed."""
import math

import pytest
import torch

from daam_b200.geometry import LatentGeometry
from daam_b200.testing.synthetic import TINY_SPEC, UNetSpec, make_pipeline

# (latent (H, W), sample_size, grid, [(n, (h, w, factor)) per level s = 0, 1, 2, 3]); latent_hw is 4096 throughout
TABLE = [
    ((64, 96), 64, (64, 96), [(6144, (64, 96, 1)), (1536, (32, 48, 2)), (384, (16, 24, 4)), (96, (8, 12, 8))]),
    ((96, 64), 64, (96, 64), [(6144, (96, 64, 1)), (1536, (48, 32, 2)), (384, (24, 16, 4)), (96, (12, 8, 8))]),
    ((152, 104), 128, (76, 52), [(15808, (152, 104, 0)), (3952, (76, 52, 1)), (988, (38, 26, 2)), (247, (19, 13, 4))]),
    ((168, 96), 128, (84, 48), [(16128, (168, 96, 0)), (4032, (84, 48, 1)), (1008, (42, 24, 2)), (252, (21, 12, 4))]),
    ((144, 112), 128, (72, 56), [(16128, (144, 112, 0)), (4032, (72, 56, 1)), (1008, (36, 28, 2)), (252, (18, 14, 4))]),
    ((75, 100), 64, (75, 100), [(7500, (75, 100, 1)), (1900, (38, 50, 2)), (475, (19, 25, 4)), (130, (10, 13, 8))]),
    ((32, 128), 64, (32, 128), [(4096, (32, 128, 1)), (1024, (16, 64, 2)), (256, (8, 32, 4)), (64, (4, 16, 8))]),
]


@pytest.mark.parametrize('shape,sample_size,grid,levels', TABLE, ids=lambda v: str(v))
def test_geometry_rule(shape, sample_size, grid, levels):
    geo = LatentGeometry(4096, sample_size, shape)
    assert not geo.square and geo.grid == grid
    for n, expect in levels:
        assert geo.level(n, 3) == expect
        # the factor-8 level is the one the tracer skips (daam/trace.py:289)
        assert (expect[2] == 8) == (n == levels[3][0] and sample_size == 64)


@pytest.mark.parametrize('latent_hw', [4096, 9216])
def test_square_latents_keep_the_reference_rule(latent_hw):
    x = int(math.sqrt(latent_hw))
    for sample_size in (64, 96, 128):
        for shape in (None, (x, x), (96, 96), (64, 64)):
            geo = LatentGeometry(latent_hw, sample_size, shape)
            assert geo.square and geo.grid == (x, x) and geo.key is None
            for side in (128, 96, 64, 48, 32, 24, 16, 12, 8):
                n = side * side
                assert geo.level(n) == (side, side, int(math.sqrt(latent_hw // n)))
            assert geo.level(6144)[:2] == (None, None)          # not a square count: the tracer raises as before
    # SD-2.1-base at 768 pixels: the reference's factor 0 at the first level
    assert LatentGeometry(4096, 64, (96, 96)).level(9216) == (96, 96, 0)


def test_refusals():
    with pytest.raises(ValueError, match=r'non-square 64x96 latent need unet.config.sample_size / '
                                         r'sqrt\(latent_hw\) = 1 .* or 2 .*32 / 96'):
        LatentGeometry(9216, 32, (64, 96))                   # g = 1/3
    geo = LatentGeometry(4096, 64, (64, 96))
    with pytest.raises(RuntimeError, match=r'layer 5: 1000 query positions match no level of the 64x96 latent'):
        geo.level(1000, 5)


class _Recorder:
    """An attn2 processor that records the query count of every call and does nothing else."""

    def __init__(self, log):
        self.log = log

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None):
        self.log.append(hidden_states.shape[1])
        return hidden_states


TINY_XL = UNetSpec('tiny-xl', 128, (32, 64, 64), (1, 2, 2), (0, 1, 1), 64, mid_depth=1)


@pytest.mark.parametrize('body', ['skeleton', 'full'])
@pytest.mark.parametrize('spec,shape', [(TINY_SPEC, (64, 96)), (TINY_SPEC, (96, 64)), (TINY_SPEC, (75, 100)),
                                        (TINY_SPEC, (32, 128)), (TINY_XL, (152, 104)), (TINY_XL, (168, 96)),
                                        (TINY_XL, (144, 112))], ids=lambda v: str(v) if isinstance(v, tuple) else v.name)
def test_synthetic_unet_calls_attn2_with_the_predicted_counts(spec, shape, body):
    pipe = make_pipeline(spec, body)
    log = []
    for m in pipe.unet.modules():
        if hasattr(m, 'attn2'):
            m.attn2.set_processor(_Recorder(log))
    H, W = shape
    geo = LatentGeometry(4096, spec.sample_size, shape)
    with torch.no_grad():
        pipe.unet(torch.zeros(2, spec.in_channels, H, W), 0, torch.zeros(2, spec.tokens, spec.cross_attention_dim))
    assert log
    for n in log:
        h, w, _ = geo.level(n)                               # raises if a call matches no level
        assert h * w == n


def test_square_synthetic_runs_are_unchanged():
    """Ceil-sized down-sampling and skip-sized up-sampling give the floor / x2 values exactly on even sizes."""
    pipe = make_pipeline(TINY_SPEC, 'full')
    x = torch.randn(2, 4, 64, 64, generator=torch.Generator().manual_seed(0))
    ctx = torch.randn(2, 77, 96, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        a = pipe.unet(x, 10.0, ctx)
        b = pipe.unet(x, 10.0, ctx)
        default = pipe('a cat', num_inference_steps=2, generator=torch.Generator().manual_seed(3))
        explicit = pipe('a cat', num_inference_steps=2, generator=torch.Generator().manual_seed(3), height=512,
                        width=512)
    assert torch.equal(a, b)
    assert torch.equal(default.latents, explicit.latents)


def test_pipeline_height_width_reach_check_inputs_and_the_latent():
    pipe = make_pipeline(TINY_SPEC, 'skeleton')
    seen = []
    inner = pipe.check_inputs
    pipe.check_inputs = lambda prompt, *a, **kw: (seen.append(a), inner(prompt, *a, **kw))[1]
    out = pipe('a cat', num_inference_steps=1, height=768, width=512)
    assert seen == [(768, 512)]
    assert tuple(out.latents.shape[-2:]) == (96, 64)
