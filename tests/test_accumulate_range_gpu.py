"""daam_accumulate_range: the accumulate kernels also add what they add into a range slab shaped like the accumulator.

What must hold on every path (16-bit wgmma single-chunk and K-chunked, fp32 split form in both update modes, SIMT in
both update modes): the accumulators are bit-identical to daam_accumulate's; a range slab seeded with arbitrary values
ends bit-equal to daam_accumulate run on a copy of that seed (the same arithmetic as the accumulator update, so a range
slab zeroed before a span of steps is the accumulator of a trace of only those steps); nothing around a range slab
changes."""
import zlib

import pytest
import torch

import bench
from daam_b200 import _native, ops
from tests.reference64 import ACC_DIMS, assert_close64, layer_maps64
from tests.test_accumulate_steps_gpu import PATHS, SHAPES, _qk, _scale, bits
from tests.test_parity_elementwise_gpu import ATOL, RTOL

pytestmark = pytest.mark.gpu
DEV = 'cuda'
GUARD = 1024                       # sentinel floats on each side of a range slab (a multiple of 4: keeps 16-byte alignment)
SENTINEL = 12345.0
TRACER_FLAGS = _native.ACC_AUTO | _native.ACC_EARLY_LOADS


class SeededSlab:
    """A range slab holding `seed` with sentinel floats before and after it."""

    def __init__(self, seed: torch.Tensor):
        n = seed.numel()
        self.buf = torch.full((n + 2 * GUARD,), SENTINEL, device=DEV)
        self.slab = self.buf[GUARD:GUARD + n].view(seed.shape)
        self.slab.copy_(seed)

    def check(self, what=''):
        assert (self.buf[:GUARD] == SENTINEL).all() and (self.buf[-GUARD:] == SENTINEL).all(), \
            f'{what}: write outside the range slab'


def _descs(layers, accs):
    return [ops.make_layer_desc(q, k, a, h, _scale(q, h)) for (q, k, h), a in zip(layers, accs)]


def _seed(shape, seed):
    g = torch.Generator(DEV).manual_seed(seed)
    return torch.randn(shape, generator=g, device=DEV) * 3


@pytest.mark.parametrize('path,flags', PATHS)
@pytest.mark.parametrize('hw,heads,d', SHAPES)
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16, torch.float32])
def test_range_slab_adds_like_the_accumulator(dtype, hw, heads, d, path, flags):
    q, k = _qk(hw, heads, d, dtype, hw * 31 + heads * 7 + d)
    layers = [(q, k, heads)]
    shape = (1, heads, 77, hw)
    what = f'{path} hw{hw} H{heads} d{d} {dtype}'
    acc0, seed = torch.rand(shape, generator=torch.Generator(DEV).manual_seed(5), device=DEV), _seed(shape, 6)
    plain, ranged, ref = acc0.clone(), acc0.clone(), seed.clone()
    rs = SeededSlab(seed)
    ops.accumulate(_descs(layers, [plain]), DEV, flags=flags)
    ops.accumulate_range(_descs(layers, [ranged]), [rs.slab], DEV, flags=flags)
    ops.accumulate(_descs(layers, [ref]), DEV, flags=flags)
    torch.cuda.synchronize()
    assert torch.equal(bits(plain), bits(ranged)), f'{what}: accumulator differs from daam_accumulate'
    assert torch.equal(bits(rs.slab), bits(ref)), f'{what}: range slab differs from daam_accumulate on its seed'
    rs.check(what)


def test_many_layers_of_every_kind_in_one_call():
    """80 layers in one call: 48 16-bit ones (two packs, K-chunked among them), 16 fp32 split, 16 unaligned SIMT."""
    kinds = [(256, 4, 64, torch.bfloat16, False), (576, 2, 64, torch.float16, False), (256, 2, 80, torch.float16, False),
             (256, 2, 64, torch.float32, False), (256, 2, 64, torch.bfloat16, True)]
    layers, shapes = [], []
    for i in range(80):
        hw, heads, d, dtype, unaligned = kinds[i % len(kinds)]
        q, k = _qk(hw, heads, d, dtype, 1000 + i, unaligned)
        layers.append((q, k, heads))
        shapes.append((1, heads, 77, hw))
    plain = [torch.full(s, 0.5, device=DEV) for s in shapes]
    ranged = [a.clone() for a in plain]
    seeds = [_seed(s, 100 + i) for i, s in enumerate(shapes)]
    ref = [s.clone() for s in seeds]
    slabs = [SeededSlab(s) for s in seeds]
    ops.accumulate(_descs(layers, plain), DEV, flags=TRACER_FLAGS)
    ops.accumulate_range(_descs(layers, ranged), [r.slab for r in slabs], DEV, flags=TRACER_FLAGS)
    ops.accumulate(_descs(layers, ref), DEV, flags=TRACER_FLAGS)
    torch.cuda.synchronize()
    for i in range(80):
        slabs[i].check(f'layer {i}')
        assert torch.equal(bits(plain[i]), bits(ranged[i])), i
        assert torch.equal(bits(slabs[i].slab), bits(ref[i])), i


def test_invalid_range_slabs_are_rejected():
    hw, heads = 256, 2
    q, k = _qk(hw, heads, 64, torch.bfloat16, 3)
    q2, k2 = _qk(hw, heads, 64, torch.bfloat16, 4)
    buf = torch.zeros(4, heads, 77, hw, device=DEV)
    acc0, acc1, s0, s1 = buf[0:1], buf[1:2], buf[2:3], buf[3:4]
    descs = [ops.make_layer_desc(q, k, acc0, heads, 0.125), ops.make_layer_desc(q2, k2, acc1, heads, 0.125)]
    n = acc0.numel()
    stream = torch.cuda.current_stream().cuda_stream

    def expect(ranges, match):
        with pytest.raises(_native.NativeError, match=match) as e:
            _native.accumulate_range(descs, ranges, stream)
        assert e.value.code == _native.E_INVALID

    expect([s0.data_ptr(), 0], 'null range slab')
    expect([s0.data_ptr() + 4, s1.data_ptr()], 'not 16-byte aligned')
    expect([acc0.data_ptr(), s1.data_ptr()], 'range slab of layer 0 overlaps the accumulator of layer 0')
    expect([acc1.data_ptr(), s1.data_ptr()], 'range slab of layer 0 overlaps the accumulator of layer 1')
    expect([s0.data_ptr(), acc1.data_ptr()], 'range slab of layer 1 overlaps the accumulator of layer 1')
    expect([s0.data_ptr(), s0.data_ptr() + 4 * (n - 4)], 'range slabs of layers 0 and 1 overlap')
    packed = _native.PackedLayers(descs)
    rc = _native.load().daam_accumulate_range(packed.array, None, 2, 0, stream)
    assert rc == _native.E_INVALID and b'range_acc is a null array' in _native.load().daam_last_error()
    # adjacent, non-overlapping slabs are fine, and nothing above launched or wrote anything
    assert (buf == 0).all()
    _native.accumulate_range(descs, [s0.data_ptr(), s1.data_ptr()], stream)
    torch.cuda.synchronize()
    assert torch.equal(bits(s0), bits(acc0)) and torch.equal(bits(s1), bits(acc1))


def test_steps_and_range_calls_do_not_share_a_plan():
    """The same layer array and the same pointer array, alternated: a steps call stores, a range call adds."""
    kinds = [(1024, 4, 64, torch.bfloat16, False), (256, 2, 80, torch.float16, False), (256, 2, 64, torch.float32, False),
             (256, 2, 64, torch.bfloat16, True)]
    layers, accs = [], []
    for i, (hw, heads, d, dtype, unaligned) in enumerate(kinds):
        q, k = _qk(hw, heads, d, dtype, 300 + i, unaligned)
        layers.append((q, k, heads))
        accs.append(torch.zeros(1, heads, 77, hw, device=DEV))
    addend = [a.clone() for a in accs]
    ops.accumulate(_descs(layers, addend), DEV)                       # what one call adds, from zero
    twice = [a.clone() for a in addend]
    ops.accumulate(_descs(layers, twice), DEV)                        # ... and that added once more
    slabs = [torch.full_like(a, 0.25) for a in accs]
    packed = ops.pack(_descs(layers, accs))
    ptrs = _native.StepPointers([s.data_ptr() for s in slabs])
    stream = torch.cuda.current_stream().cuda_stream
    for expected in ('store', 'add', 'store', 'add', 'add'):
        if expected == 'store':
            _native.accumulate_steps(packed, ptrs, stream)
        else:
            _native.accumulate_range(packed, ptrs, stream)
        torch.cuda.synchronize()
        want = addend if expected == 'store' else twice
        for i, (s, w) in enumerate(zip(slabs, want)):
            assert torch.equal(bits(s), bits(w)), f'{expected} layer {i}'
        if expected == 'add':                                      # back to what a store leaves, for the next add
            for s, a in zip(slabs, addend):
                s.copy_(a)


RANGE_CASES = [  # id, workload, dtype, prompts, flags
    ('sd21-bf16', 'sd21', torch.bfloat16, 1, TRACER_FLAGS),
    ('sd21-split-fp32', 'sd21', torch.float32, 1, TRACER_FLAGS),
    ('sd21-split-ldst-fp32', 'sd21', torch.float32, 1, TRACER_FLAGS | _native.ACC_RMW_LDST),
    ('sd21-simt-bf16', 'sd21', torch.bfloat16, 1, _native.ACC_FORCE_SIMT | _native.ACC_EARLY_LOADS),
    ('sd15-fp16', 'sd15', torch.float16, 1, TRACER_FLAGS),
    ('sd15-fp32', 'sd15', torch.float32, 1, TRACER_FLAGS),
    ('sdxl-2prompts-fp16', 'sdxl', torch.float16, 2, TRACER_FLAGS),
]


@pytest.mark.parametrize('case,workload,dtype,prompts,flags', RANGE_CASES, ids=[c[0] for c in RANGE_CASES])
def test_range_slabs_at_production_sizes(case, workload, dtype, prompts, flags):
    """Three launches of distinct Q/K onto seeded accumulators, the first plain and the last two with the range: every
    element of the zeroed range slab matches the float64 sum of those two steps, and the accumulators stay bit-equal
    to daam_accumulate's."""
    steps = 3
    layers = bench.traced_layers(workload)
    g = torch.Generator(device=DEV).manual_seed(zlib.crc32(case.encode()))
    qk = [[(torch.randn(2 * prompts, hw, h * d, generator=g, device=DEV).to(dtype),
            torch.randn(2 * prompts, 77, h * d, generator=g, device=DEV).to(dtype)) for hw, h, d in layers]
          for _ in range(steps)]
    plain = [torch.rand(prompts, h, 77, hw, generator=g, device=DEV) / 77 for hw, h, d in layers]
    ranged = [a.clone() for a in plain]
    slabs = [SeededSlab(torch.zeros_like(a)) for a in plain]

    def descs(s, accs):
        return [ops.make_layer_desc(q, k, a, h, d ** -0.5) for (q, k), a, (hw, h, d) in zip(qk[s], accs, layers)]

    torch.cuda.synchronize()
    for s in range(steps):
        ops.accumulate(descs(s, plain), DEV, flags=flags)
        if s == 0:
            ops.accumulate(descs(s, ranged), DEV, flags=flags)
        else:
            ops.accumulate_range(descs(s, ranged), [r.slab for r in slabs], DEV, flags=flags)
    torch.cuda.synchronize()
    for i, (hw, h, d) in enumerate(layers):
        what = f'{case} layer {i} ({hw}, {h}, {d})'
        slabs[i].check(what)
        assert torch.equal(bits(plain[i]), bits(ranged[i])), f'{what}: accumulator differs from daam_accumulate'
        ref = layer_maps64(*qk[1][i], h, d ** -0.5) + layer_maps64(*qk[2][i], h, d ** -0.5)
        assert_close64(slabs[i].slab, ref, RTOL[dtype], ATOL[dtype] * 2, what, ACC_DIMS)
        del ref
