"""The 16-bit wgmma form adds into accumulator tiles it has loaded into shared memory and stores them back, instead of
reducing into L2. These tests pin what that must not change: layers of one call that share accumulator elements still
all add (the plan splits them into consecutive launches), the update flags make no difference for 16-bit inputs, and
the result is exactly that of consecutive single-layer calls."""
import pytest
import torch

from daam_b200 import _native, ops

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def _layer(hw, heads, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(2, hw, heads * 64, generator=g).to(dtype).to(DEV)
    k = torch.randn(2, 77, heads * 64, generator=g).to(dtype).to(DEV)
    return q, k


@pytest.mark.parametrize('dtype', [torch.float16, torch.bfloat16])
def test_layers_sharing_an_accumulator_in_one_call_all_add(dtype):
    hw, heads = 576, 3                                          # partial last tile
    layers = [_layer(hw, heads, dtype, s) for s in range(3)]
    one_call = ops.new_accumulator(1, heads, hw, DEV)
    ops.accumulate([ops.make_layer_desc(q, k, one_call, heads, 0.125) for q, k in layers], DEV,
                   flags=_native.ACC_FORCE_MMA)
    separate = ops.new_accumulator(1, heads, hw, DEV)
    for q, k in layers:
        ops.accumulate([ops.make_layer_desc(q, k, separate, heads, 0.125)], DEV, flags=_native.ACC_FORCE_MMA)
    torch.cuda.synchronize()
    assert torch.equal(one_call, separate)
    sums = one_call.double().sum(dim=(2, 3))
    assert torch.allclose(sums, torch.full_like(sums, 3.0 * hw), rtol=1e-5)


def test_partly_overlapping_accumulators_in_one_call():
    """Two layers whose slabs overlap by one head (views into one buffer): the shared head gets both updates."""
    hw, heads = 1024, 2
    buf = torch.zeros(1, heads + 1, 77, hw, device=DEV)
    (q0, k0), (q1, k1) = _layer(hw, heads, torch.bfloat16, 10), _layer(hw, heads, torch.bfloat16, 11)
    ops.accumulate([ops.make_layer_desc(q0, k0, buf[:, :heads], heads, 0.125),
                    ops.make_layer_desc(q1, k1, buf[:, 1:], heads, 0.125)], DEV, flags=_native.ACC_FORCE_MMA)
    a0 = ops.accumulate_layer(q0, k0, heads, 0.125, flags=_native.ACC_FORCE_MMA)
    a1 = ops.accumulate_layer(q1, k1, heads, 0.125, flags=_native.ACC_FORCE_MMA)
    torch.cuda.synchronize()
    assert torch.equal(buf[0, 0], a0[0, 0])
    assert torch.equal(buf[0, 1], a0[0, 1] + a1[0, 0])
    assert torch.equal(buf[0, 2], a1[0, 1])


def test_update_flags_do_not_change_16bit_results():
    shapes = [(256, 4), (1024, 2), (4096, 1), (576, 3)]
    layers = [_layer(hw, heads, torch.bfloat16, 20 + i) for i, (hw, heads) in enumerate(shapes)]
    outs = []
    for mode in (_native.ACC_RMW_AUTO, _native.ACC_RMW_RED, _native.ACC_RMW_LDST):
        accs = [torch.full((1, heads, 77, hw), 0.25, device=DEV) for hw, heads in shapes]
        descs = [ops.make_layer_desc(q, k, a, heads, 0.125) for (q, k), a, (hw, heads) in zip(layers, accs, shapes)]
        for _ in range(2):
            ops.accumulate(descs, DEV, flags=_native.ACC_FORCE_MMA | mode)
        outs.append(accs)
    torch.cuda.synchronize()
    for accs in outs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(outs[0], accs))
