"""Tile coverage of the 16-bit wgmma launch at tile counts around the grid size.

The persistent CTAs walk the launch's tiles in a fixed order (one CTA per SM, grid = min(tiles, SMs)). A tile skipped or
done twice by that walk shows up as a wrong accumulator block, so every element of every layer is checked against the
oracle, with a guard head before and after each slab, at tile counts one below, at and one above the SM count, and at
two full rounds plus one. The launches run back to back, with and without early Q/K loads.
"""
import pytest
import torch

from daam_b200 import _native, ops
from tests.util import assert_elementwise, oracle_layer_maps

pytestmark = pytest.mark.gpu
DEV = 'cuda'


@pytest.mark.parametrize('flags', [_native.ACC_FORCE_MMA, _native.ACC_FORCE_MMA | _native.ACC_EARLY_LOADS],
                         ids=['pdl', 'early-loads'])
@pytest.mark.parametrize('extra', [-1, 0, 1, 'two-rounds-plus-one'])
def test_every_tile_once_around_the_grid_size(extra, flags):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n_tiles = 2 * sms + 1 if extra == 'two-rounds-plus-one' else sms + extra
    # two square maps, n_tiles in all: 18 x 18 (3 tiles per head, the last one partial) and 10 x 10 (1 partial tile)
    h1 = (n_tiles - 1) // 3
    cases = [(324, h1), (100, n_tiles - 3 * h1)]
    g = torch.Generator().manual_seed(n_tiles)
    qs, ks, slabs, descs = [], [], [], []
    for hw, heads in cases:
        q = torch.randn(2, hw, heads * 64, generator=g).bfloat16().to(DEV)
        k = torch.randn(2, 77, heads * 64, generator=g).bfloat16().to(DEV)
        slab = torch.zeros(heads + 2, 77, hw, device=DEV)                # guard heads before and after
        qs.append(q), ks.append(k), slabs.append(slab)
        descs.append(ops.make_layer_desc(q, k, slab[1:-1].unsqueeze(0), heads, 0.125))
    packed = ops.pack(descs)
    for _ in range(3):
        ops.accumulate(packed, DEV, flags=flags)
    torch.cuda.synchronize()
    for (hw, heads), q, k, slab in zip(cases, qs, ks, slabs):
        ref = oracle_layer_maps(q, k, heads, 0.125, steps=3)
        assert_elementwise(slab[1:-1], ref, 1e-4, 3e-5, f'{n_tiles} tiles, hw{hw} H{heads}')
        assert float(slab[0].abs().max()) == 0.0 and float(slab[-1].abs().max()) == 0.0
