"""Image sizes off the 64-pixel grid on the host: the float64 bicubic reference at non-integer ratios (down-sampling
included) against torch's own interpolate, the layer geometry of such sizes as a table and as a sweep over the
synthetic UNets, and the oracle port against the verbatim reference's 600x600 generation. No GPU needed."""
import warnings

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from daam_b200.geometry import LatentGeometry
from daam_b200.testing.synthetic import TINY_SPEC, UNetSpec, make_pipeline
from oracle import daam_oracle as O
from tests.reference64 import bicubic64
from tests.util import golden

warnings.filterwarnings('ignore', category=FutureWarning)

PROMPT = 'a dog chasing a red ball on the beach'
# an SDXL-topology tree (sample_size 128 -> g = 2; no cross-attention at the first level)
TINY_XL = UNetSpec('tiny-xl', 128, (32, 64, 64), (1, 2, 2), (0, 1, 1), 64, mid_depth=1)

RATIOS = [(75, 64), (65, 64), (63, 64), (33, 64), (19, 64), (38, 75), (25, 100), (19, 75)]


def _interpolate_matrix(n_in, n_out):
    """``F.interpolate(mode='bicubic', align_corners=False)`` along one axis as an ``[n_out, n_in]`` matrix: the images
    of the float64 basis vectors (the other axis has size 1 -> 1, which bicubic leaves unchanged)."""
    basis = torch.eye(n_in, dtype=torch.float64).reshape(n_in, 1, n_in, 1)
    out = F.interpolate(basis, size=(n_out, 1), mode='bicubic', align_corners=False)
    return out.reshape(n_in, n_out).T


@pytest.mark.parametrize('n_in,n_out', RATIOS, ids=lambda v: str(v))
def test_bicubic_matrix_matches_interpolate(n_in, n_out):
    want = _interpolate_matrix(n_in, n_out)
    got = torch.from_numpy(O.math_bicubic_matrix(n_in, n_out))
    assert got.shape == (n_out, n_in)
    assert float((got - want).abs().max()) <= 1e-12
    assert torch.equal(bicubic64(n_in, n_out, 'cpu'), got)
    # rows sum to 1: the cubic's weights are a partition of unity, border clamping included
    assert float((got.sum(dim=1) - 1).abs().max()) <= 1e-12


@pytest.mark.parametrize('key,grid', [((19, 25), (75, 100)), ((38, 50), (64, 64)), ((75, 75), (64, 64)),
                                      ((17, 33), (64, 75))], ids=lambda v: str(v))
def test_separable_upsample_matches_interpolate_on_2d_basis(key, grid):
    """``B_y @ key @ B_x^T`` (what the finalize kernels and the float64 reference compute) is 2-D bicubic: the images of
    every 2-D basis image match interpolate's."""
    kh, kw = key
    basis = torch.eye(kh * kw, dtype=torch.float64).reshape(kh * kw, 1, kh, kw)
    want = F.interpolate(basis, size=grid, mode='bicubic', align_corners=False)[:, 0]
    by, bx = bicubic64(kh, grid[0], 'cpu'), bicubic64(kw, grid[1], 'cpu')
    got = by @ basis[:, 0] @ bx.T
    assert float((got - want).abs().max()) <= 1e-12


# (tracer, image (H, W), {attn2 query count: (h, w, factor)} of every level the synthetic UNet calls attn2 at)
TABLE = [
    (TINY_SPEC, (600, 800), {7500: (75, 100, 1), 1900: (38, 50, 2), 475: (19, 25, 4), 130: (10, 13, 8)}),
    (TINY_SPEC, (800, 600), {7500: (100, 75, 1), 1900: (50, 38, 2), 475: (25, 19, 4), 130: (13, 10, 8)}),
    (TINY_SPEC, (576, 712), {6408: (72, 89, 1), 1620: (36, 45, 2), 414: (18, 23, 4), 108: (9, 12, 8)}),
    (TINY_SPEC, (600, 600), {5625: (75, 75, 0), 1444: (38, 38, 1), 361: (19, 19, 3), 100: (10, 10, 6)}),
    (TINY_SPEC, (520, 520), {4225: (65, 65, 0), 1089: (33, 33, 1), 289: (17, 17, 3), 81: (9, 9, 7)}),
    (TINY_SPEC, (576, 576), {5184: (72, 72, 0), 1296: (36, 36, 1), 324: (18, 18, 3), 81: (9, 9, 7)}),
    (TINY_XL, (1000, 1000), {3969: (63, 63, 1), 1024: (32, 32, 2)}),
    (TINY_XL, (1000, 1200), {4725: (63, 75, 1), 1216: (32, 38, 2)}),
]


class _Recorder:
    """An attn2 processor that records the query count of every call and does nothing else."""

    def __init__(self, log):
        self.log = log

    def __call__(self, attn, hidden_states, encoder_hidden_states=None, attention_mask=None):
        self.log.append(hidden_states.shape[1])
        return hidden_states


def _attn2_counts(pipe, spec, latent):
    log = []
    for m in pipe.unet.modules():
        if hasattr(m, 'attn2'):
            m.attn2.set_processor(_Recorder(log))
    with torch.no_grad():
        pipe.unet(torch.zeros(2, spec.in_channels, *latent), 0, torch.zeros(2, spec.tokens, spec.cross_attention_dim))
    assert log
    return set(log)


@pytest.mark.parametrize('spec,image,levels', TABLE, ids=lambda v: str(v) if isinstance(v, tuple) else
                         (v.name if hasattr(v, 'name') else ''))
def test_offgrid_table(spec, image, levels):
    latent = (image[0] // 8, image[1] // 8)
    geo = LatentGeometry(4096, spec.sample_size, latent)
    pipe = make_pipeline(spec, 'skeleton')
    counts = _attn2_counts(pipe, spec, latent)
    assert counts == set(levels), f'{image}: attn2 query counts {sorted(counts)}'
    for n, expect in levels.items():
        assert geo.level(n, 3) == expect
    # at least one traced layer (factor != 8) has a pixel count that is not a multiple of 4
    assert any(n % 4 for n, (_, _, f) in levels.items() if f != 8)


SD_SIDES = [256, 264, 328, 520, 576, 600, 712, 800, 1016]
XL_SIDES = [512, 520, 712, 1000, 1208, 1536]


@pytest.mark.parametrize('spec,sides', [(TINY_SPEC, SD_SIDES), (TINY_XL, XL_SIDES)], ids=['sd', 'sdxl'])
def test_geometry_sweep_resolves_every_attn2_call(spec, sides):
    """Every (H, W) of a grid of multiples of 8 px: each attn2 query count of the synthetic UNet resolves to a level
    whose keys hold exactly that many pixels."""
    pipe = make_pipeline(spec, 'skeleton')
    for H in sides:
        for W in sides:
            latent = (H // 8, W // 8)
            geo = LatentGeometry(4096, spec.sample_size, latent)
            for n in _attn2_counts(pipe, spec, latent):
                h, w, factor = geo.level(n)
                assert h is not None and h * w == n, f'{H}x{W}: {n} -> {(h, w, factor)}'


@pytest.fixture(scope='module')
def one_thread():
    """The fixture was computed on one thread (oracle/make_golden.py): the comparison below is exact."""
    before = torch.get_num_threads()
    torch.set_num_threads(1)
    yield
    torch.set_num_threads(before)


def test_oracle_matches_reference_at_600_square(one_thread):
    """The oracle port, bit for bit, against the verbatim reference's 2-step generation at 600x600 (75^2 latent: keys of
    75^2 / 38^2 / 19^2 at factors 0 / 1 / 3, down-sampled and up-sampled onto 64 x 64)."""
    fx = golden('pipeline_tiny600')
    torch.manual_seed(0)
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float32, seed=int(fx['unet_seed']))
    with O.OracleTrace(pipe) as ot:
        pipe(str(fx['prompt']), num_inference_steps=int(fx['steps']),
             generator=torch.Generator().manual_seed(int(fx['gen_seed'])), height=int(fx['height']),
             width=int(fx['width']))
        keys = {k: v.clone() for k, v in ot.heat_maps}
        assert [list(k) for k in keys] == fx['keys'].tolist()
        assert sorted({k[0] for k in keys}) == [0, 1, 3]
        assert {tuple(v.shape[-2:]) for v in keys.values()} == {(75, 75), (38, 38), (19, 19)}
        np.testing.assert_array_equal(np.array([float(v.double().sum()) for v in keys.values()]), fx['key_sums'])
        np.testing.assert_array_equal(np.array([float(v.abs().max()) for v in keys.values()]), fx['key_absmax'])
        assert list(ot.layer_names) == fx['layer_names'].tolist()
        g = ot.compute_global_heat_map()
        got = {
            'global': g,
            'global_norm': ot.compute_global_heat_map(normalize=True),
            'factors_0': ot.compute_global_heat_map(factors=[0]),
            'factors_3': ot.compute_global_heat_map(factors=[3]),
            'layer9_head0': ot.compute_global_heat_map(layer_idx=9, head_idx=0),
            'word_ball': O.port_word_heat_map(g, pipe.tokenizer, PROMPT, 'ball'),
        }
    for name, v in got.items():
        assert fx[name].shape == tuple(v.shape), name
        np.testing.assert_array_equal(v.numpy(), fx[name], err_msg=name)
    # the float64 restatement agrees with the reference to fp32 rounding at this down-sampling ratio
    ref64 = O.math_global_heat_map([v.numpy() for (f, _, _), v in keys.items() if f in (0, 1)], 64, g.shape[0])
    np.testing.assert_allclose(fx['global'], ref64, rtol=2e-5, atol=2e-6)
