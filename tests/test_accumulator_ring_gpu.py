"""Layers of one call that share accumulator elements: the plan starts a new launch for a layer whose slab overlaps one
already in its pack, on every path (16-bit wgmma, fp32 split form, SIMT) and in every update mode. Without that, tiles
of the two layers run concurrently: the 16-bit form and LDST mode read, add and store them (lost updates), and RED adds
in timing order. These tests pin that every layer adds, that one call equals consecutive single-layer calls bit for bit
within an operand class, that the update flags make no difference for 16-bit inputs, and the values against float64."""
import pytest
import torch

from daam_b200 import _native, ops
from tests.reference64 import ACC_DIMS, assert_close64, layer_maps64
from tests.test_parity_elementwise_gpu import ATOL, RTOL

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


SHARED_PATHS = [('auto', _native.ACC_AUTO), ('simt', _native.ACC_FORCE_SIMT), ('mma', _native.ACC_FORCE_MMA)]
SHARED_MODES = [('red', _native.ACC_RMW_RED), ('ldst', _native.ACC_RMW_LDST)]


@pytest.mark.parametrize('mode,mode_flags', SHARED_MODES)
@pytest.mark.parametrize('path,path_flags', SHARED_PATHS)
@pytest.mark.parametrize('dtype', [torch.float32, torch.float16, torch.bfloat16])
def test_shared_accumulator_is_applied_in_call_order_on_every_path(dtype, path, path_flags, mode, mode_flags):
    """3 layers of (4096, 5, 64) on one accumulator (160 tiles each: their tiles would run at the same time in one
    launch), and two layers overlapping by one head: one call == consecutive single-layer calls, bit for bit."""
    flags = path_flags | mode_flags
    hw, heads = 4096, 5
    layers = [_layer(hw, heads, dtype, 40 + s) for s in range(3)]
    init = torch.rand(1, heads, 77, hw, generator=torch.Generator(DEV).manual_seed(1), device=DEV)
    one_call, separate = init.clone(), init.clone()
    ops.accumulate([ops.make_layer_desc(q, k, one_call, heads, 0.125) for q, k in layers], DEV, flags=flags)
    for q, k in layers:
        ops.accumulate([ops.make_layer_desc(q, k, separate, heads, 0.125)], DEV, flags=flags)
    torch.cuda.synchronize()
    what = f'{dtype} {path} {mode}'
    ref = init.double() + sum(layer_maps64(q, k, heads, 0.125) for q, k in layers)
    assert_close64(one_call, ref, RTOL[dtype], 3 * ATOL[dtype], f'{what}: one call', ACC_DIMS)
    assert torch.equal(one_call, separate), f'{what}: one call differs from consecutive calls'
    # partial overlap: layer 1's head 0 is layer 0's head 4
    buf = torch.zeros(1, 2 * heads - 1, 77, hw, device=DEV)
    (q0, k0), (q1, k1) = layers[0], layers[1]
    ops.accumulate([ops.make_layer_desc(q0, k0, buf[:, :heads], heads, 0.125),
                    ops.make_layer_desc(q1, k1, buf[:, heads - 1:], heads, 0.125)], DEV, flags=flags)
    seq = torch.zeros_like(buf)
    ops.accumulate([ops.make_layer_desc(q0, k0, seq[:, :heads], heads, 0.125)], DEV, flags=flags)
    ops.accumulate([ops.make_layer_desc(q1, k1, seq[:, heads - 1:], heads, 0.125)], DEV, flags=flags)
    torch.cuda.synchronize()
    assert torch.equal(buf, seq), f'{what}: partial overlap differs from consecutive calls'
    m0, m1 = layer_maps64(q0, k0, heads, 0.125), layer_maps64(q1, k1, heads, 0.125)
    ref = torch.cat([m0[:, :heads - 1], m0[:, heads - 1:] + m1[:, :1], m1[:, 1:]], dim=1)
    assert_close64(buf, ref, RTOL[dtype], 2 * ATOL[dtype], f'{what}: partial overlap', ACC_DIMS)


@pytest.mark.parametrize('mode,mode_flags', SHARED_MODES)
def test_shared_accumulator_across_operand_classes(mode, mode_flags):
    """fp32, bf16 and (unaligned, hence SIMT) fp16 layers on one accumulator: three launches, issued class by class, so
    the order of the adds differs from consecutive calls; every layer still adds (within tolerance)."""
    hw, heads = 4096, 5
    qa, ka = _layer(hw, heads, torch.float32, 50)
    qb, kb = _layer(hw, heads, torch.bfloat16, 51)
    g = torch.Generator().manual_seed(52)
    qc = torch.randn(2, hw, heads * 64 + 1, generator=g).half().to(DEV)[..., 1:]     # rows not 16-byte aligned
    kc = torch.randn(2, 77, heads * 64 + 1, generator=g).half().to(DEV)[..., 1:]
    layers = [(qa, ka), (qb, kb), (qc, kc), (qb, kb), (qa, ka)]
    one_call, separate = ops.new_accumulator(1, heads, hw, DEV), ops.new_accumulator(1, heads, hw, DEV)
    ops.accumulate([ops.make_layer_desc(q, k, one_call, heads, 0.125) for q, k in layers], DEV,
                   flags=_native.ACC_AUTO | mode_flags)
    for q, k in layers:
        ops.accumulate([ops.make_layer_desc(q, k, separate, heads, 0.125)], DEV, flags=_native.ACC_AUTO | mode_flags)
    torch.cuda.synchronize()
    ref = sum(layer_maps64(q, k, heads, 0.125) for q, k in layers)
    assert_close64(one_call, ref, RTOL[torch.bfloat16], 5 * ATOL[torch.bfloat16], f'{mode}: one call', ACC_DIMS)
    assert_close64(separate, ref, RTOL[torch.bfloat16], 5 * ATOL[torch.bfloat16], f'{mode}: separate', ACC_DIMS)
