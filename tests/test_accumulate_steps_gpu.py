"""daam_accumulate_steps: the accumulate kernels also store what they add into a step slab shaped like the accumulator.

What must hold on every path (16-bit wgmma single-chunk and K-chunked, fp32 split form in both update modes, SIMT in
both update modes): the accumulators are bit-identical to daam_accumulate's; starting from acc == 0 the step slab is
bit-equal to the accumulator afterwards; every element of the step slab is written (it starts as NaN) and nothing
around it changes; the step slab matches the oracle with the per-key tolerances of test_accumulate_gpu.py."""
import pytest
import torch

from daam_b200 import _native, ops
from tests.util import oracle_layer_maps, rel_err

pytestmark = pytest.mark.gpu
DEV = 'cuda'
TOL = {torch.float32: 1e-5, torch.float16: 2e-4, torch.bfloat16: 2e-4}
GUARD = 1024                       # sentinel floats on each side of a step slab (a multiple of 4: keeps 16-byte alignment)
SENTINEL = 12345.0

PATHS = [
    ('auto', _native.ACC_AUTO),
    ('auto-early', _native.ACC_AUTO | _native.ACC_EARLY_LOADS),
    ('mma-red', _native.ACC_FORCE_MMA | _native.ACC_RMW_RED),
    ('mma-ldst', _native.ACC_FORCE_MMA | _native.ACC_RMW_LDST),
    ('simt-red', _native.ACC_FORCE_SIMT | _native.ACC_RMW_RED),
    ('simt-ldst', _native.ACC_FORCE_SIMT | _native.ACC_RMW_LDST),
]
SHAPES = [  # hw, heads, head_dim: single-chunk 16-bit, SD-1.x K-chunked head dims, partial tiles
    (4096, 5, 64), (1024, 10, 64), (256, 20, 64), (576, 10, 64), (1024, 8, 80), (256, 8, 160), (4096, 8, 40),
]


def _qk(hw, heads, d, dtype, seed, unaligned=False):
    g = torch.Generator().manual_seed(seed)
    extra = 1 if unaligned else 0      # a one-element offset: rows are no longer 16-byte aligned (SIMT only)
    q = (torch.randn(2, hw, heads * d + extra, generator=g) * 1.5).to(dtype).to(DEV)[..., extra:]
    k = torch.randn(2, 77, heads * d + extra, generator=g).to(dtype).to(DEV)[..., extra:]
    return q, k


class GuardedSlab:
    """A NaN-filled step slab with sentinel floats before and after it."""

    def __init__(self, shape):
        n = 1
        for s in shape:
            n *= s
        self.buf = torch.full((n + 2 * GUARD,), float('nan'), device=DEV)
        self.buf[:GUARD] = SENTINEL
        self.buf[GUARD + n:] = SENTINEL
        self.slab = self.buf[GUARD:GUARD + n].view(shape)

    def check(self, what=''):
        assert not torch.isnan(self.slab).any(), f'{what}: step slab elements left unwritten'
        assert (self.buf[:GUARD] == SENTINEL).all() and (self.buf[-GUARD:] == SENTINEL).all(), \
            f'{what}: write outside the step slab'


def bits(t):
    return t.contiguous().view(torch.int32)


def _run(layers, flags, init):
    """daam_accumulate and daam_accumulate_steps on equal copies of the accumulators; returns both and the slabs."""
    plain = [init(a_shape) for _, _, _, a_shape in layers]
    stepped = [a.clone() for a in plain]
    ops.accumulate([ops.make_layer_desc(q, k, a, h, _scale(q, h)) for (q, k, h, _), a in zip(layers, plain)], DEV,
                   flags=flags)
    guarded = [GuardedSlab(a.shape) for a in stepped]
    ops.accumulate_steps([ops.make_layer_desc(q, k, a, h, _scale(q, h)) for (q, k, h, _), a in zip(layers, stepped)],
                         [g.slab for g in guarded], DEV, flags=flags)
    torch.cuda.synchronize()
    return plain, stepped, guarded


def _scale(q, heads):
    d = q.shape[-1] // heads
    return 0.125 if d == 64 else d ** -0.5


@pytest.mark.parametrize('path,flags', PATHS)
@pytest.mark.parametrize('hw,heads,d', SHAPES)
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float16, torch.float32])
def test_step_slab_next_to_the_accumulate(dtype, hw, heads, d, path, flags):
    q, k = _qk(hw, heads, d, dtype, hw * 31 + heads * 7 + d)
    layer = [(q, k, heads, (1, heads, 77, hw))]
    what = f'{path} hw{hw} H{heads} d{d} {dtype}'
    # from a non-zero accumulator: the accumulate itself is unchanged, bit for bit
    plain, stepped, guarded = _run(layer, flags, lambda s: torch.rand(s, generator=torch.Generator(DEV).manual_seed(5),
                                                                      device=DEV))
    assert torch.equal(bits(plain[0]), bits(stepped[0])), what
    guarded[0].check(what)
    ref = oracle_layer_maps(q, k, heads, _scale(q, heads)).unsqueeze(0)
    err = rel_err(guarded[0].slab, ref)
    assert err <= TOL[dtype], f'{what}: step slab vs oracle {err:.3e}'
    # from zero: the step slab is exactly what landed in the accumulator
    plain, stepped, guarded = _run(layer, flags, lambda s: torch.zeros(s, device=DEV))
    guarded[0].check(what)
    assert torch.equal(bits(plain[0]), bits(stepped[0])), what
    assert torch.equal(bits(guarded[0].slab), bits(stepped[0])), what


@pytest.mark.parametrize('flags', [_native.ACC_AUTO, _native.ACC_RMW_LDST])
@pytest.mark.parametrize('dtype', [torch.bfloat16, torch.float32])
def test_unaligned_view_takes_the_simt_step_kernel(dtype, flags):
    hw, heads, d = 1024, 4, 64
    q, k = _qk(hw, heads, d, dtype, 77, unaligned=True)
    with pytest.raises(_native.NativeError):        # really not a wgmma layer
        ops.accumulate_layer(q, k, heads, flags=_native.ACC_FORCE_MMA)
    layer = [(q, k, heads, (1, heads, 77, hw))]
    plain, stepped, guarded = _run(layer, flags, lambda s: torch.zeros(s, device=DEV))
    guarded[0].check('unaligned')
    assert torch.equal(bits(plain[0]), bits(stepped[0]))
    assert torch.equal(bits(guarded[0].slab), bits(stepped[0]))
    assert rel_err(guarded[0].slab, oracle_layer_maps(q, k, heads, 0.125).unsqueeze(0)) <= TOL[dtype]


def test_many_layers_of_every_kind_in_one_call():
    """80 layers in one call: 48 16-bit ones (two packs, K-chunked among them), 16 fp32 split, 16 unaligned SIMT."""
    kinds = [(256, 4, 64, torch.bfloat16, False), (576, 2, 64, torch.float16, False), (256, 2, 80, torch.float16, False),
             (256, 2, 64, torch.float32, False), (256, 2, 64, torch.bfloat16, True)]
    layers = []
    for i in range(80):
        hw, heads, d, dtype, unaligned = kinds[i % len(kinds)]
        q, k = _qk(hw, heads, d, dtype, 1000 + i, unaligned)
        layers.append((q, k, heads, (1, heads, 77, hw)))
    for init in (lambda s: torch.full(s, 0.5, device=DEV), lambda s: torch.zeros(s, device=DEV)):
        plain, stepped, guarded = _run(layers, _native.ACC_AUTO | _native.ACC_EARLY_LOADS, init)
        for i, (a, b, g) in enumerate(zip(plain, stepped, guarded)):
            g.check(f'layer {i}')
            assert torch.equal(bits(a), bits(b)), i
    for i, (a, g) in enumerate(zip(stepped, guarded)):       # (the last run started from zero)
        assert torch.equal(bits(g.slab), bits(a)), i


def test_batched_prompts_and_repeated_steps():
    """n_prompts > 1, and three consecutive steps: each call's slab holds only that call's addend."""
    hw, heads, d = 1024, 3, 64
    accs = ops.new_accumulator(3, heads, hw, DEV)
    total = ops.new_accumulator(3, heads, hw, DEV)
    step = torch.empty_like(accs)
    for s in range(3):
        g = torch.Generator().manual_seed(50 + s)
        q = torch.randn(6, hw, heads * d, generator=g).bfloat16().to(DEV)
        k = torch.randn(6, 77, heads * d, generator=g).bfloat16().to(DEV)
        ops.accumulate_steps([ops.make_layer_desc(q, k, accs, heads, 0.125)], [step], DEV)
        alone = ops.accumulate_layer(q, k, heads, 0.125)
        ops.accumulate([ops.make_layer_desc(q, k, total, heads, 0.125)], DEV)
        torch.cuda.synchronize()
        assert torch.equal(bits(step), bits(alone)), s
        assert torch.equal(bits(accs), bits(total)), s


def test_invalid_step_slabs_are_rejected():
    hw, heads = 256, 2
    q, k = _qk(hw, heads, 64, torch.bfloat16, 3)
    q2, k2 = _qk(hw, heads, 64, torch.bfloat16, 4)
    buf = torch.zeros(4, heads, 77, hw, device=DEV)
    acc0, acc1, s0, s1 = buf[0:1], buf[1:2], buf[2:3], buf[3:4]
    descs = [ops.make_layer_desc(q, k, acc0, heads, 0.125), ops.make_layer_desc(q2, k2, acc1, heads, 0.125)]
    n = acc0.numel()

    def expect(steps, match):
        with pytest.raises(_native.NativeError, match=match) as e:
            _native.accumulate_steps(descs, steps, torch.cuda.current_stream().cuda_stream)
        assert e.value.code == _native.E_INVALID

    expect([s0.data_ptr(), 0], 'null step slab')
    expect([s0.data_ptr() + 4, s1.data_ptr()], 'not 16-byte aligned')
    expect([acc0.data_ptr(), s1.data_ptr()], 'layer 0 overlaps the accumulator of layer 0')
    expect([acc1.data_ptr(), s1.data_ptr()], 'layer 0 overlaps the accumulator of layer 1')
    expect([s0.data_ptr(), acc1.data_ptr()], 'layer 1 overlaps the accumulator of layer 1')
    expect([s0.data_ptr(), s0.data_ptr() + 4 * (n - 4)], 'step slabs of layers 0 and 1 overlap')
    # adjacent, non-overlapping slabs are fine, and nothing above launched or wrote anything
    assert (buf == 0).all()
    _native.accumulate_steps(descs, [s0.data_ptr(), s1.data_ptr()], torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert torch.equal(bits(s0), bits(acc0)) and torch.equal(bits(s1), bits(acc1))


def test_normalize_maps_matches_finalize_normalize():
    hw, heads = 1024, 2
    q, k = _qk(hw, heads, 64, torch.float16, 9)
    acc = ops.accumulate_layer(q, k, heads, 0.125)
    groups = [_native.DaamKeyGroup(acc=acc[0].data_ptr(), heads=heads, h=32, w=32, tokens=77, head_sel=-1, reserved=0)]
    stream = torch.cuda.current_stream().cuda_stream
    raw = torch.empty(7, 64, 64, device=DEV)
    ref = torch.empty(7, 64, 64, device=DEV)
    _native.finalize(groups, 64, 7, False, raw.data_ptr(), stream)
    _native.finalize(groups, 64, 7, True, ref.data_ptr(), stream)
    both = torch.stack([raw, raw])
    _native.normalize_maps(both.data_ptr(), 2, 7, 64, stream)
    torch.cuda.synchronize()
    assert torch.equal(both[0], ref) and torch.equal(both[1], ref)
