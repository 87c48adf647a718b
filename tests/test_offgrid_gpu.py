"""Image sizes off the 64-pixel grid: layers whose pixel count is not a multiple of 4, against float64.

Diffusers accepts any multiple of 8 px; at most such sizes some traced layer has an odd pixel count (19 x 25 = 475 at
600x800, 19^2 = 361 at 600^2, 63^2 = 3969 for SDXL at 1000^2). Those layers take the SIMT kernel (the wgmma path needs
16-byte accumulator rows), their per-head accumulator bases are not 16-byte aligned, and their keys reach finalize's
generic kernel with sizes that do not divide the grid (75 -> 64 is a bicubic down-sample). Checked here:

* the accumulate kernels element-wise against :func:`layer_maps64` (SURVEY.md section 8c: ``1e-6 * steps + 1e-5 *
  |ref|`` for fp32, x 10 for fp16 / bf16), with guard heads around every slab that must stay bit-exact zeros; the
  step / range slab kernels bit-exact against the accumulator; the materialised-probability kernels;
* finalize / per-key finalize on odd key stacks into 64^2 and 75 x 100 grids against float64;
* traced generations at 600x800, 800x600, 576x712, 600^2, 520^2 and SDXL 1000^2 / 1000x1200 against float64 on the
  identical Q/K, the tracer's options at odd sizes, two production-size models, and the verbatim reference's own
  600^2 generation (tests/golden/pipeline_tiny600.npz)."""
from types import SimpleNamespace

import pytest
import torch

from daam_b200 import _native, ops, trace
from daam_b200.geometry import LatentGeometry
from daam_b200.testing.synthetic import SD21_SPEC, SDXL_SPEC, TINY_SPEC, UNetSpec, make_pipeline
from tests.reference64 import (ACC_DIMS, FP32_EPS, MAP_DIMS, assert_close64, bicubic64, layer_maps64,
                               normalized_tolerance)
from tests.util import golden, rel_err

pytestmark = pytest.mark.gpu
DEV = 'cuda'
PROMPT = 'a dog chasing a red ball on the beach'
TINY_XL = UNetSpec('tiny-xl', 128, (32, 64, 64), (1, 2, 2), (0, 1, 1), 64, mid_depth=1)
DEFAULT_FACTORS = {0, 1, 2, 4, 8, 16, 32, 64}        # compute_global_heat_map's factors=None (daam/trace.py:104)

# element-wise bound of an accumulator after `steps` calls: atol x steps + rtol x |ref|
ACC_RTOL = {torch.float32: 1e-5, torch.float16: 1e-4, torch.bfloat16: 1e-4}
ACC_ATOL = {torch.float32: 1e-6, torch.float16: 1e-5, torch.bfloat16: 1e-5}
# the global-map tolerance of the traced tests, per step
RTOL, ATOL = 1e-3, 1e-4

HWS = [1, 2, 3, 5, 81, 127, 129, 131, 289, 361, 414, 475, 1089, 3969, 4225]
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
SIMT_PATHS = [('auto', _native.ACC_AUTO), ('simt-red', _native.ACC_FORCE_SIMT | _native.ACC_RMW_RED),
              ('simt-ldst', _native.ACC_FORCE_SIMT | _native.ACC_RMW_LDST)]


@pytest.fixture(autouse=True)
def _exact_fp32():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def bits(t):
    return t.contiguous().view(torch.int32)


# ---- accumulate kernels -----------------------------------------------------------------------------------------------

def _qk(bsz, hw, heads, d, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    q = (torch.randn(bsz, hw, heads * d, generator=g) * 1.5).to(dtype).to(DEV)
    k = torch.randn(bsz, 77, heads * d, generator=g).to(dtype).to(DEV)
    return q, k


class GuardedAcc:
    """A zero accumulator ``[n_prompts, heads, 77, hw]`` with at least one head of zeros before and after it. The
    leading guard is rounded up to a multiple of 4 floats: the accumulator itself must start 16-byte aligned, while its
    per-head bases (multiples of 77 * hw floats) are not when hw is odd."""

    def __init__(self, shape):
        self.shape = tuple(shape)
        head = 77 * self.shape[-1]
        self.n = 1
        for s in self.shape:
            self.n *= s
        self.lead = -(-head // 4) * 4
        self.buf = torch.zeros(self.lead + self.n + head, device=DEV)
        self.acc = self.buf[self.lead:self.lead + self.n].view(self.shape)

    def check(self, what):
        before, after = self.buf[:self.lead], self.buf[self.lead + self.n:]
        assert int(bits(before).abs().max()) == 0 and int(bits(after).abs().max()) == 0, \
            f'{what}: a guard head was written'


@pytest.mark.parametrize('dtype', DTYPES, ids=str)
@pytest.mark.parametrize('hw', HWS)
def test_accumulate_odd_hw_against_float64(hw, dtype):
    """1 and 3 prompts (CFG batches) and a lone sample (the upper half of its heads), on every SIMT-capable path; the
    AUTO path routes the layer to the SIMT kernel and gives the same bits as FORCE_SIMT."""
    heads, d, steps = 3, 64, 2
    scale = d ** -0.5
    for bsz in (2, 6, 1):
        q, k = _qk(bsz, hw, heads, d, dtype, seed=hw * 7 + bsz)
        ref = steps * layer_maps64(q, k, heads, scale)
        _, n_prompts, _, n_heads = ops.cond_half(bsz, heads)
        assert tuple(ref.shape) == (n_prompts, n_heads, 77, hw)
        results = {}
        for name, flags in SIMT_PATHS:
            g = GuardedAcc(ref.shape)
            desc = ops.make_layer_desc(q, k, g.acc, heads, scale)
            for _ in range(steps):
                ops.accumulate([desc], DEV, flags=flags)
            torch.cuda.synchronize()
            what = f'hw {hw} {dtype} batch {bsz} {name}'
            assert_close64(g.acc, ref, ACC_RTOL[dtype], ACC_ATOL[dtype] * steps, what, ACC_DIMS)
            g.check(what)
            results[name] = g.acc.clone()
        assert torch.equal(bits(results['auto']), bits(results['simt-red'])), f'hw {hw} batch {bsz}: AUTO != SIMT'


def test_mixed_launch_of_aligned_and_odd_layers():
    """One call with an aligned 16-bit layer (wgmma), an aligned fp32 layer (wgmma split form) and two odd layers (one
    16-bit, one fp32: both SIMT) is exactly three launches; every layer is right, and so is the plan-cache replay."""
    cases = [(1024, 5, torch.bfloat16), (256, 4, torch.float32), (475, 5, torch.float16), (361, 2, torch.float32),
             (3, 3, torch.bfloat16)]
    qs, ks, guards, descs = [], [], [], []
    for i, (hw, heads, dtype) in enumerate(cases):
        q, k = _qk(2, hw, heads, 64, dtype, seed=40 + i)
        g = GuardedAcc((1, heads, 77, hw))
        qs.append(q), ks.append(k), guards.append(g)
        descs.append(ops.make_layer_desc(q, k, g.acc, heads, 0.125))
    packed = ops.pack(descs)
    for rep in (1, 2):
        torch.cuda.synchronize()
        before = _native.launch_count()
        ops.accumulate(packed, DEV)
        torch.cuda.synchronize()
        assert _native.launch_count() - before == 3, f'call {rep}: {_native.launch_count() - before} launches'
        for (hw, heads, dtype), q, k, g in zip(cases, qs, ks, guards):
            what = f'call {rep}: hw {hw} {dtype}'
            ref = rep * layer_maps64(q, k, heads, 0.125)
            assert_close64(g.acc, ref, ACC_RTOL[dtype], ACC_ATOL[dtype] * rep, what, ACC_DIMS)
            g.check(what)


GUARD = 1024                       # sentinel floats on each side of a second slab (a multiple of 4: keeps alignment)
SENTINEL = 12345.0


class GuardedSlab:
    """A second slab filled with `fill`, with sentinel floats before and after it."""

    def __init__(self, shape, fill):
        n = fill.numel()
        self.buf = torch.full((n + 2 * GUARD,), SENTINEL, device=DEV)
        self.buf[GUARD:GUARD + n] = fill.reshape(-1)
        self.slab = self.buf[GUARD:GUARD + n].view(shape)

    def check(self, what):
        assert (self.buf[:GUARD] == SENTINEL).all() and (self.buf[-GUARD:] == SENTINEL).all(), \
            f'{what}: write outside the second slab'


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16], ids=str)
@pytest.mark.parametrize('path,flags', SIMT_PATHS)
def test_step_and_range_slabs_at_odd_hw(path, flags, dtype):
    """daam_accumulate_steps from zero: the step slab equals the accumulator bit for bit (the increment), and the
    accumulator equals daam_accumulate's. daam_accumulate_range on a range slab seeded with X: it ends bit-equal to
    daam_accumulate run on an accumulator holding X."""
    shapes = [(3, 2), (129, 3), (475, 2), (3969, 1)]
    layers = [(*_qk(2, hw, heads, 64, dtype, seed=hw), heads) for hw, heads in shapes]
    shape = lambda q, heads: (1, heads, 77, q.shape[1])
    plain = [torch.zeros(shape(q, h), device=DEV) for q, _, h in layers]
    ops.accumulate([ops.make_layer_desc(q, k, a, h, 0.125) for (q, k, h), a in zip(layers, plain)], DEV, flags=flags)
    stepped = [torch.zeros(shape(q, h), device=DEV) for q, _, h in layers]
    steps = [GuardedSlab(shape(q, h), torch.full(shape(q, h), float('nan'), device=DEV)) for q, _, h in layers]
    ops.accumulate_steps([ops.make_layer_desc(q, k, a, h, 0.125) for (q, k, h), a in zip(layers, stepped)],
                         [s.slab for s in steps], DEV, flags=flags)
    g = torch.Generator(device=DEV).manual_seed(5)
    seeds = [torch.rand(shape(q, h), generator=g, device=DEV) for q, _, h in layers]
    on_x = [x.clone() for x in seeds]
    ops.accumulate([ops.make_layer_desc(q, k, a, h, 0.125) for (q, k, h), a in zip(layers, on_x)], DEV, flags=flags)
    ranged = [torch.zeros(shape(q, h), device=DEV) for q, _, h in layers]
    ranges = [GuardedSlab(shape(q, h), x) for (q, _, h), x in zip(layers, seeds)]
    ops.accumulate_range([ops.make_layer_desc(q, k, a, h, 0.125) for (q, k, h), a in zip(layers, ranged)],
                         [r.slab for r in ranges], DEV, flags=flags)
    torch.cuda.synchronize()
    for i, (q, k, h) in enumerate(layers):
        what = f'{path} {dtype} hw {q.shape[1]}'
        steps[i].check(what)
        ranges[i].check(what)
        assert torch.equal(bits(stepped[i]), bits(plain[i])), f'{what}: accumulator differs from daam_accumulate'
        assert torch.equal(bits(steps[i].slab), bits(stepped[i])), f'{what}: step slab != increment'
        assert torch.equal(bits(ranged[i]), bits(plain[i])), f'{what}: accumulator differs from daam_accumulate'
        assert torch.equal(bits(ranges[i].slab), bits(on_x[i])), f'{what}: range slab != daam_accumulate on X'
        assert_close64(steps[i].slab, layer_maps64(q, k, h, 0.125), ACC_RTOL[dtype], ACC_ATOL[dtype], what, ACC_DIMS)


@pytest.mark.parametrize('dtype', DTYPES, ids=str)
@pytest.mark.parametrize('hw', [3, 127, 475])
def test_force_mma_refuses_odd_hw_and_names_it(hw, dtype):
    q, k = _qk(2, hw, 2, 64, dtype, seed=hw)
    acc = ops.new_accumulator(1, 2, hw, DEV)
    with pytest.raises(_native.NativeError, match=rf'hw = {hw}\b') as e:
        ops.accumulate_layer(q, k, 2, acc=acc, flags=_native.ACC_FORCE_MMA)
    assert e.value.code == _native.E_UNSUPPORTED
    # the same layer through AUTO is accepted (the SIMT kernel)
    ops.accumulate_layer(q, k, 2, acc=acc)
    torch.cuda.synchronize()
    assert_close64(acc, layer_maps64(q, k, 2, 0.125), ACC_RTOL[dtype], ACC_ATOL[dtype], f'hw {hw}', ACC_DIMS)


PROBS_RTOL = {torch.float32: 1e-5, torch.float16: 2 ** -10, torch.bfloat16: 2 ** -7}   # + rounding to the output dtype


@pytest.mark.parametrize('dtype', DTYPES, ids=str)
@pytest.mark.parametrize('hw', [1, 3, 129, 475])
def test_attention_probs_and_accumulate_probs_at_odd_hw(hw, dtype):
    """The save_heads / load_heads kernels with 2 prompts (a CFG batch of 4): every sample's probabilities against a
    float64 softmax, and accumulate_probs adding the conditional half onto a guarded zero accumulator exactly."""
    bsz, heads, d = 4, 3, 64
    q, k = _qk(bsz, hw, heads, d, dtype, seed=hw + 11)
    probs = ops.attention_probs(q, k, heads)
    split = lambda t: t.reshape(bsz, t.shape[1], heads, d).permute(0, 2, 1, 3).reshape(bsz * heads, t.shape[1], d)
    s = torch.bmm(split(q).double(), split(k).double().transpose(1, 2)) * d ** -0.5
    ref = torch.softmax(s, dim=-1)
    torch.cuda.synchronize()
    assert probs.dtype == dtype and tuple(probs.shape) == (bsz * heads, hw, 77)
    assert_close64(probs, ref, PROBS_RTOL[dtype], 1e-6, f'attention_probs hw {hw} {dtype}', ('row', 'pixel', 'token'))
    g = GuardedAcc((2, heads, 77, hw))
    ops.accumulate_probs(probs, g.acc)
    torch.cuda.synchronize()
    g.check(f'accumulate_probs hw {hw}')
    want = probs[bsz * heads // 2:].float().transpose(1, 2).reshape(2, heads, 77, hw)
    assert torch.equal(bits(g.acc), bits(want.contiguous()))


# ---- finalize on odd key stacks ---------------------------------------------------------------------------------------

KEYS = [(75, 75), (38, 38), (19, 19), (65, 65), (63, 63), (19, 25), (38, 50)]


def _groups(stacks, head_sel=None):
    return [_native.DaamKeyGroup(acc=t.data_ptr(), heads=t.shape[0], h=t.shape[2], w=t.shape[3], tokens=t.shape[1],
                                 head_sel=-1 if head_sel is None else head_sel, reserved=0) for t in stacks]


def _up64(keys, grid):
    by = bicubic64(keys.shape[-2], grid[0], keys.device)
    bx = bicubic64(keys.shape[-1], grid[1], keys.device)
    return by @ keys.double() @ bx.T


def _tolerance(stacks, n_keys, grid):
    """``finalize_tolerance`` with the 1-norms of both axes' bicubic matrices (the keys here are not square)."""
    norm = max(float(bicubic64(t.shape[-2], grid[0], 'cpu').abs().sum(dim=1).max()) *
               float(bicubic64(t.shape[-1], grid[1], 'cpu').abs().sum(dim=1).max()) for t in stacks)
    vmax = max(float(t.abs().max()) for t in stacks)
    return max(1e-4, (n_keys + 1) * FP32_EPS), 32 * FP32_EPS * norm * vmax


def _finalize(monkeypatch, groups, grid, n_rows, normalize, generic, per_key=0):
    monkeypatch.setenv('DAAM_FINALIZE_GENERIC', '1' if generic else '0')
    out = torch.empty(((per_key,) if per_key else ()) + (n_rows,) + grid, device=DEV)
    fn = _native.finalize_per_key if per_key else _native.finalize
    fn(groups, grid, n_rows, normalize, out.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return out


def _norm64(maps):
    return maps / (maps[..., 1:-1, :, :].sum(dim=-3, keepdim=True) + 1e-6)


@pytest.mark.parametrize('grid', [(64, 64), (75, 100)], ids=str)
@pytest.mark.parametrize('n_rows', [12, 77])
def test_finalize_odd_keys_against_float64(monkeypatch, grid, n_rows):
    g = torch.Generator(device=DEV).manual_seed(n_rows + grid[1])
    stacks = [torch.exp(torch.randn(2, 77, kh, kw, generator=g, device=DEV)) for kh, kw in KEYS]
    for normalize, head_sel in [(False, None), (True, None), (False, 1), (True, 0)]:
        what = f'{grid} n_rows {n_rows} normalize {normalize} head_sel {head_sel}'
        total, n = None, 0
        for t in stacks:
            sel = t[:, :n_rows] if head_sel is None else t[head_sel:head_sel + 1, :n_rows]
            part = _up64(sel, grid).clamp_(min=0.0).sum(dim=0)
            total = part if total is None else total + part
            n += sel.shape[0]
        ref = total / n
        rtol, atol = _tolerance(stacks, n, grid)
        if normalize:
            atol = normalized_tolerance(ref, rtol, atol)
            ref, rtol = _norm64(ref), 0.0
        groups = _groups(stacks, head_sel)
        out = _finalize(monkeypatch, groups, grid, n_rows, normalize, generic=False)
        generic = _finalize(monkeypatch, groups, grid, n_rows, normalize, generic=True)
        assert torch.equal(bits(out), bits(generic)), f'{what}: odd keys did not take the generic kernel'
        assert_close64(out, ref, rtol, atol, what, MAP_DIMS)
    # per key
    n_keys = sum(t.shape[0] for t in stacks)
    for normalize in (False, True):
        out = _finalize(monkeypatch, _groups(stacks), grid, n_rows, normalize, generic=False, per_key=n_keys)
        generic = _finalize(monkeypatch, _groups(stacks), grid, n_rows, normalize, generic=True, per_key=n_keys)
        assert torch.equal(bits(out), bits(generic)), f'per-key {grid}: odd keys did not take the generic kernel'
        first = 0
        for t in stacks:
            raw = _up64(t[:, :n_rows], grid).clamp_(min=0.0)
            for h in range(t.shape[0]):
                rtol, atol = _tolerance([t[h:h + 1]], 1, grid)
                ref = raw[h]
                if normalize:
                    atol = normalized_tolerance(ref, rtol, atol)
                    ref, rtol = _norm64(ref), 0.0
                what = f'per-key {grid} n_rows {n_rows} key {tuple(t.shape[-2:])} head {h} normalize {normalize}'
                assert_close64(out[first + h], ref, rtol, atol, what, MAP_DIMS)
            first += t.shape[0]


# ---- traced generations ------------------------------------------------------------------------------------------------

FILTERS = [{}, {'normalize': True}, {'factors': [1, 2]}, {'layer_idx': 9, 'head_idx': 0}, {'head_idx': 1}]


class Recorder:
    """Device copies of every (layer, factor, q, k) the hooks hand to the kernel, grouped by UNet forward."""

    def __init__(self, tc, unet):
        self.steps = []
        self.tc, inner = tc, tc._enqueue
        self.handle = unet.register_forward_pre_hook(lambda *_: self.steps.append([]))

        def enqueue(layer_idx, factor, q, k, heads, scale):
            self.steps[-1].append((layer_idx, factor, q.detach().clone(), k.detach().clone(), heads, scale))
            return inner(layer_idx, factor, q, k, heads, scale)

        tc._enqueue = enqueue

    def stop(self):
        self.handle.remove()
        del self.tc._enqueue                                     # back to the class's method


def _keys64(rec, geometry, steps=None, prompt=0):
    """layer -> (factor, [heads, 77, h, w] float64 time sum over ``steps``) from the recorded Q/K."""
    out = {}
    for s in (range(len(rec.steps)) if steps is None else steps):
        for layer_idx, factor, q, k, heads, scale in rec.steps[s]:
            m = layer_maps64(q, k, heads, scale)[prompt]
            h, w, f = geometry.level(m.shape[-1], layer_idx)
            assert f == factor
            m = m.reshape(m.shape[0], m.shape[1], h, w)
            out[layer_idx] = (factor, m if layer_idx not in out else out[layer_idx][1] + m)
    return out


def _global64(keys, grid, n_rows, factors=None, layer_idx=None, head_idx=None, normalize=False):
    factors = DEFAULT_FACTORS if factors is None else set(factors)
    total, n = None, 0
    for layer, (factor, m) in keys.items():
        if factor not in factors or (layer_idx is not None and layer != layer_idx):
            continue
        sel = m[:, :n_rows] if head_idx is None else m[head_idx:head_idx + 1, :n_rows]
        part = _up64(sel, grid).clamp_(min=0.0).sum(dim=0)
        total = part if total is None else total + part
        n += sel.shape[0]
    out = total / n
    return out / (out[1:-1].sum(dim=0, keepdim=True) + 1e-6) if normalize else out


def _expand_tolerance(word_map, out_hw, span):
    """Absolute bound of a min-max normalised fp32 up-sample (``expand_as``) at a non-integer ratio, whose cubic weights
    are rounded to fp32: each value errs by less than ``32 * 2^-24 * N^2 * max |v|`` (``finalize_tolerance``'s stencil
    bound, ``N`` the bicubic matrices' largest row 1-norm), the min and the max by as much again, and ``span`` (the
    exact max - min) divides them; plus the rounding of the subtraction and the division."""
    ny = float(bicubic64(word_map.shape[-2], out_hw[0], 'cpu').abs().sum(dim=1).max())
    nx = float(bicubic64(word_map.shape[-1], out_hw[1], 'cpu').abs().sum(dim=1).max())
    t = 32 * FP32_EPS * ny * nx * float(word_map.abs().max())
    return 2 * t / span + 4 * FP32_EPS


def _image(h, w):
    return SimpleNamespace(height=h, width=w, size=(w, h))     # the PIL surface expand_as reads


def _run(spec, dtype, height, width, steps=2, seed=3, **kw):
    pipe = make_pipeline(spec, dtype=dtype, device=DEV, seed=seed)
    with trace(pipe, **kw) as tc:
        rec = Recorder(tc, pipe.unet)
        pipe(PROMPT, num_inference_steps=steps, generator=torch.Generator().manual_seed(7), height=height, width=width)
        rec.stop()
        yield pipe, tc, rec


SIZES = [(TINY_SPEC, (600, 800)), (TINY_SPEC, (800, 600)), (TINY_SPEC, (576, 712)), (TINY_SPEC, (600, 600)),
         (TINY_SPEC, (520, 520)), (TINY_XL, (1000, 1000)), (TINY_XL, (1000, 1200))]


@pytest.mark.parametrize('spec,hw', SIZES, ids=[f'{s.name}-{h}x{w}' for s, (h, w) in SIZES])
@pytest.mark.parametrize('dtype', DTYPES, ids=str)
def test_traced_offgrid_maps_against_float64(spec, hw, dtype):
    steps = 2
    for pipe, tc, rec in _run(spec, dtype, *hw, steps=steps):
        geo = tc.geometry
        latent = (hw[0] // 8, hw[1] // 8)
        if geo.square:
            assert latent[0] == latent[1] and geo.grid == (64, 64)
        else:
            assert geo.grid == (-(-latent[0] // geo.g), -(-latent[1] // geo.g))
        keys = _keys64(rec, geo)
        assert any((m.shape[-2] * m.shape[-1]) % 4 for _, m in keys.values()), 'no odd layer at this size'
        seen = set()
        for (factor, layer, head), got in tc.all_heat_maps:
            ref_factor, m = keys[layer]
            assert factor == ref_factor and tuple(got.shape) == tuple(m.shape[1:])
            assert_close64(got, m[head], RTOL, ATOL * steps, f'layer {layer} head {head}', ('token', 'y', 'x'))
            seen.add(layer)
        assert seen == set(keys)
        n_rows = len(PROMPT.split()) + 2
        filters = FILTERS + ([{'factors': [0]}, {'factors': [3]}] if geo.square else [])
        for f in filters:
            if 'layer_idx' in f and f['layer_idx'] not in keys:
                continue
            if 'factors' in f and not any(fac in f['factors'] for fac, _ in keys.values()):
                continue
            got = tc.compute_global_heat_map(**f)
            assert tuple(got.heat_maps.shape) == (n_rows,) + geo.grid
            assert_close64(got.heat_maps, _global64(keys, geo.grid, n_rows, **f), RTOL, ATOL * steps, f'{f}', MAP_DIMS)
        hm = tc.compute_global_heat_map()
        dog = hm.compute_word_heat_map('dog')
        assert tuple(dog.heatmap.shape) == geo.grid
        assert_close64(dog.heatmap, hm.heat_maps[2].double(), 1e-6, 0.0, 'word map')
        image = _image(*hw)
        mask = dog.expand_as(image)
        assert tuple(mask.shape) == hw
        words, masks = hm.expand_words(['dog', 'ball'], image)
        assert tuple(masks.shape) == (2,) + hw
        assert torch.allclose(masks[0], mask, atol=1e-6)
        for i, (word, row) in enumerate((('dog', 2), ('ball', 6))):
            ref = _up64(hm.heat_maps[row][None].double(), hw)[0]
            span = float(ref.max() - ref.min())
            ref = (ref - ref.min()) / (span + 1e-8)
            assert_close64(masks[i], ref, 0.0, _expand_tolerance(hm.heat_maps[row], hw, span), f'expand_words {word}')
        per_head_keys, per_head = tc.compute_per_head_heat_maps()
        assert len(per_head_keys) == per_head.shape[0] > 0
        for (factor, layer, head), got in zip(per_head_keys, per_head):
            assert factor in DEFAULT_FACTORS
            ref = _up64(keys[layer][1][head, :n_rows], geo.grid).clamp_(min=0.0)
            assert_close64(got, ref, RTOL, ATOL * steps, f'per-head {(factor, layer, head)}', MAP_DIMS)


def test_time_resolved_and_step_ranges_at_600x800():
    hw = (600, 800)
    for _, tc, rec in _run(TINY_SPEC, torch.float32, *hw, steps=3, time_resolved=True):
        tm = tc.compute_time_heat_maps()
        assert tuple(tm.heat_maps.shape[-2:]) == (75, 100) and len(tm) == 3
        n_rows = tm.heat_maps.shape[1]
        for t in range(3):
            ref = _global64(_keys64(rec, tc.geometry, [t]), tc.geometry.grid, n_rows)
            assert_close64(tm.heat_maps[t], ref, RTOL, ATOL, f'step {t}', MAP_DIMS)
    for _, tc, rec in _run(TINY_SPEC, torch.bfloat16, *hw, steps=4, step_ranges=[(1, 3), (3, 4)]):
        for i, span in enumerate([(1, 2), (3,)]):
            got = tc.compute_global_heat_map(step_range=i).heat_maps
            ref = _global64(_keys64(rec, tc.geometry, span), tc.geometry.grid, got.shape[0])
            assert_close64(got, ref, RTOL, len(span) * ATOL, f'step range {i}', MAP_DIMS)


def test_batch_prompts_at_576x712():
    hw = (576, 712)
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=3)
    prompts = [PROMPT, 'a cat on a sofa', 'two red cars']
    with trace(pipe, batch_prompts=True) as tc:
        rec = Recorder(tc, pipe.unet)
        pipe(prompts, num_inference_steps=2, generator=torch.Generator().manual_seed(7), height=hw[0], width=hw[1])
        rec.stop()
        for i, p in enumerate(prompts):
            got = tc.compute_global_heat_map(prompt_idx=i).heat_maps
            assert tuple(got.shape[-2:]) == (72, 89)
            ref = _global64(_keys64(rec, tc.geometry, prompt=i), tc.geometry.grid, len(p.split()) + 2)
            assert_close64(got, ref, RTOL, 2 * ATOL, f'prompt {i}', MAP_DIMS)


def test_save_heads_and_load_heads_at_600_square(tmp_path):
    hw = (600, 600)
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float32, device=DEV, seed=5)
    gen = lambda: torch.Generator().manual_seed(2)
    with trace(pipe, save_heads=True, data_dir=str(tmp_path)) as tc:
        pipe(PROMPT, num_inference_steps=2, generator=gen(), height=hw[0], width=hw[1])
        saved = tc.compute_global_heat_map().heat_maps.clone()
        saved_keys = {k: v.clone() for k, v in tc.all_heat_maps}
    with trace(pipe, load_heads=True, data_dir=str(tmp_path)) as tc:
        pipe(PROMPT, num_inference_steps=2, generator=gen(), height=hw[0], width=hw[1])
        loaded = tc.compute_global_heat_map().heat_maps.clone()
        loaded_keys = {k: v.clone() for k, v in tc.all_heat_maps}
    with trace(pipe) as tc:
        pipe(PROMPT, num_inference_steps=2, generator=gen(), height=hw[0], width=hw[1])
        fused = tc.compute_global_heat_map().heat_maps.clone()
    assert tuple(saved.shape[-2:]) == (64, 64)
    # save_heads locates the mid block (daam/trace.py:34-35): its 10^2 layer has factor 6 and is traced
    assert {k[0] for k in saved_keys} == {0, 1, 3, 6} and saved_keys.keys() == loaded_keys.keys()
    for k in saved_keys:
        assert torch.equal(bits(saved_keys[k]), bits(loaded_keys[k])), k
    assert torch.equal(bits(saved), bits(loaded))
    assert_close64(saved, fused.double(), 1e-4, 1e-6, 'materialised vs fused', MAP_DIMS)


def test_cuda_graph_replay_at_520_square_is_bit_equal_to_eager():
    hw = (520, 520)
    maps = []
    for graph in (False, True):
        pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=4, cuda_graph=graph)
        with trace(pipe) as tc:
            pipe(PROMPT, num_inference_steps=4, generator=torch.Generator().manual_seed(9), height=hw[0], width=hw[1])
            maps.append((tc.compute_global_heat_map().heat_maps.clone(),
                         {k: v.clone() for k, v in tc.all_heat_maps}))
    assert maps[0][1].keys() == maps[1][1].keys()
    assert {tuple(v.shape[-2:]) for v in maps[0][1].values()} == {(65, 65), (33, 33), (17, 17)}
    for k in maps[0][1]:
        assert torch.equal(bits(maps[0][1][k]), bits(maps[1][1][k])), k
    assert torch.equal(bits(maps[0][0]), bits(maps[1][0]))


def test_mid_block_at_576_square_is_traced_with_factor_7():
    for _, tc, rec in _run(TINY_SPEC, torch.float16, 576, 576, locate_middle_block=True):
        keys = _keys64(rec, tc.geometry)
        assert 15 in keys and keys[15][0] == 7 and tuple(keys[15][1].shape[-2:]) == (9, 9)
        got_keys = {k: v for k, v in tc.all_heat_maps}
        mid = [k for k in got_keys if k[1] == 15]
        assert mid and all(k[0] == 7 for k in mid)
        for (factor, layer, head), got in got_keys.items():
            assert_close64(got, keys[layer][1][head], RTOL, 2 * ATOL, f'layer {layer} head {head}', ('token', 'y', 'x'))
        got = tc.compute_global_heat_map(factors=[7]).heat_maps
        ref = _global64(keys, (64, 64), got.shape[0], factors=[7])
        assert_close64(got, ref, RTOL, 2 * ATOL, 'factor 7', MAP_DIMS)


def test_one_tracer_across_grid_and_offgrid_sizes():
    """512^2 -> 600x800 -> 800x600 -> 600^2 -> 512^2 on one tracer: the 512^2 runs are bit-equal to a fresh tracer's,
    the off-grid runs have their own keys and grids, and the 600^2 run matches float64."""
    def gen(pipe, tc, hw):
        pipe(PROMPT, num_inference_steps=2, generator=torch.Generator().manual_seed(7), height=hw[0], width=hw[1])
        return tc.compute_global_heat_map().heat_maps.clone()

    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=3)
    with trace(pipe) as tc:
        fresh = gen(pipe, tc, (512, 512))
    with trace(pipe) as tc:
        first = gen(pipe, tc, (512, 512))
        wide = gen(pipe, tc, (600, 800))
        tall = gen(pipe, tc, (800, 600))
        shapes_tall = {layer: tuple(key.shape[-2:]) for (_, layer, _), key in tc.all_heat_maps}
        rec = Recorder(tc, pipe.unet)
        square = gen(pipe, tc, (600, 600))
        rec.stop()
        factors_square = {layer: f for (f, layer, _), _ in tc.all_heat_maps}
        last = gen(pipe, tc, (512, 512))
    assert torch.equal(bits(fresh), bits(first)) and torch.equal(bits(fresh), bits(last))
    assert tuple(wide.shape[-2:]) == (75, 100) and tuple(tall.shape[-2:]) == (100, 75)
    assert set(shapes_tall.values()) == {(100, 75), (50, 38), (25, 19)}
    assert set(factors_square.values()) == {0, 1, 3}
    keys = _keys64(rec, LatentGeometry(4096, pipe.unet.config.sample_size, (75, 75)))
    assert_close64(square, _global64(keys, (64, 64), square.shape[0]), RTOL, 2 * ATOL, '600^2 run', MAP_DIMS)


@pytest.mark.parametrize('spec,dtype,hw', [(SD21_SPEC, torch.bfloat16, (600, 800)),
                                         (SDXL_SPEC, torch.float16, (1000, 1000))],
                         ids=['sd21-600x800-bf16', 'sdxl-1000x1000-fp16'])
def test_production_size_offgrid_against_float64(spec, dtype, hw):
    steps = 2
    pipe = make_pipeline(spec, 'skeleton', dtype=dtype, device=DEV, seed=1, init_on_device=True)
    with trace(pipe) as tc:
        rec = Recorder(tc, pipe.unet)
        pipe(PROMPT, num_inference_steps=steps, generator=torch.Generator().manual_seed(7), height=hw[0], width=hw[1])
        rec.stop()
        got = tc.compute_global_heat_map().heat_maps
        geo = tc.geometry
        keys = _keys64(rec, geo)
        assert any((m.shape[-2] * m.shape[-1]) % 4 for _, m in keys.values())
        ref = _global64(keys, geo.grid, got.shape[0])
    assert tuple(got.shape[-2:]) == geo.grid
    assert_close64(got, ref, RTOL, ATOL * steps, f'{spec.name} {hw}', MAP_DIMS)


def test_600_square_against_the_reference_fixture():
    """The verbatim reference's own 600^2 generation (CPU fp32; tests/golden/pipeline_tiny600.npz) vs ours (GPU fp32):
    Q/K differ by GPU-vs-CPU matmul rounding fed back through the UNet steps, hence the pipeline-level 1e-3 of the
    map's max."""
    fx = golden('pipeline_tiny600')
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float32, device=DEV, seed=int(fx['unet_seed']))
    with trace(pipe) as tc:
        pipe(str(fx['prompt']), num_inference_steps=int(fx['steps']),
             generator=torch.Generator().manual_seed(int(fx['gen_seed'])), height=int(fx['height']),
             width=int(fx['width']))
        keys = [k for k, _ in tc.all_heat_maps]
        assert sorted(keys) == sorted(tuple(k) for k in fx['keys'].tolist())
        sums = {k: float(v.double().sum()) for k, v in tc.all_heat_maps}
        for k, s in zip(fx['keys'].tolist(), fx['key_sums']):
            assert abs(sums[tuple(k)] - s) < 1e-4 * s, k
        g = tc.compute_global_heat_map()
        assert g.heat_maps.shape == (11, 64, 64)
        assert rel_err(g.heat_maps, fx['global']) < 1e-3
        assert rel_err(tc.compute_global_heat_map(normalize=True).heat_maps, fx['global_norm']) < 1e-3
        assert rel_err(tc.compute_global_heat_map(factors=[0]).heat_maps, fx['factors_0']) < 1e-3
        assert rel_err(tc.compute_global_heat_map(factors=[3]).heat_maps, fx['factors_3']) < 1e-3
        assert rel_err(tc.compute_global_heat_map(layer_idx=9, head_idx=0).heat_maps, fx['layer9_head0']) < 1e-3
        assert rel_err(g.compute_word_heat_map('ball').heatmap, fx['word_ball']) < 1e-3
