"""The accumulate kernels on every Q / K layout, scale and logit range ``daam_layer`` accepts, against float64.

Every case builds a raw descriptor over one storage buffer (``tests.reference64.build_layout``: the elements the
descriptor does not address are NaN), runs it through the C ABI, and checks each accumulator element against
``desc_maps64`` within ``accumulate_tolerance``, the bound derived from that element's own inputs. The contract:

* DAAM_ACC_AUTO is always within the bound;
* DAAM_ACC_FORCE_MMA is within the bound or, exactly where the stride rule of ``include/daam_b200.h`` excludes the
  layer (a prompt stride <= 0 with several prompts, fp32 at a long context), refused with DAAM_E_UNSUPPORTED naming
  the layer -- never wrong, never DAAM_E_CUDA;
* DAAM_ACC_FORCE_SIMT is within the SIMT bound;
* nothing outside the accumulator and the second slab changes (guard floats on both sides of each);
* a step slab holds what was added; a range slab started at zero equals the accumulator of the same calls bit for
  bit; duplicate K rows give equal maps bit for bit.

The worst error-to-bound ratio per path and dtype is printed at the end of the module (``pytest -s``).
"""
import collections

import pytest
import torch

from daam_b200 import _native, ops
from tests.reference64 import (ACC_DIMS, LAYOUTS, REGIMES, accumulate_tolerance, assert_close64, build_layout,
                               desc_maps64, duplicate_rows, layer_views64, layout_shape, make_regime,
                               mma_accepts_strides, probs_tolerance)

pytestmark = pytest.mark.gpu
DEV = 'cuda'
GUARD = 64                                            # floats before and after every slab (keeps 16-byte alignment)
SENTINEL = 12345.0
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
PATHS = {'auto': _native.ACC_AUTO, 'mma': _native.ACC_FORCE_MMA, 'simt': _native.ACC_FORCE_SIMT}
# (layout, n_prompts): the broadcast layouts at 2 and 3 prompts
LAYOUT_CASES = [(name, n) for name in LAYOUTS
                for n in ((2, 3) if name in ('q_broadcast', 'k_broadcast') else (2,))]
SHAPES = [(576, 40), (4096, 64), (576, 80), (576, 160), (4096, 80), (576, 64), (4096, 160), (4096, 40)]   # (hw, d)
SCALES = ('inv_sqrt_d', 1.0, 0.02, 1.37)
HEAD_DIMS = (40, 64, 80, 160)

RATIOS = collections.defaultdict(float)               # (path, form, dtype) -> worst error / bound


@pytest.fixture(scope='module', autouse=True)
def report_ratios():
    yield
    if RATIOS:
        print('\nworst error / bound (path, form, dtype):')
        for key in sorted(RATIOS, key=str):
            print(f'  {key[0]:5s} {key[1]:8s} {str(key[2]):15s} {RATIOS[key]:.3e}')


def mma_form(dtype, tokens):
    """The wgmma form a layer takes, or None when the wgmma kernel has none (fp32 at a long context)."""
    if dtype == torch.float32:
        return 'split' if tokens == 77 else None
    return 'wgmma16'


def expected_forms(desc, path, dtype, tokens):
    """The forms whose bound applies under ``path``; None: the call must be refused."""
    mma = mma_form(dtype, tokens) if mma_accepts_strides(desc) else None
    if path == 'simt':
        return ['simt']
    if path == 'mma':
        return [mma] if mma else None
    return [mma, 'simt'] if mma else ['simt']


def guarded(n):
    """A fp32 buffer of n zeros between two guard runs of SENTINEL, and the zeros as a view."""
    buf = torch.full((2 * GUARD + n,), SENTINEL, dtype=torch.float32, device=DEV)
    buf[GUARD:GUARD + n] = 0.0
    return buf, buf[GUARD:GUARD + n]


def assert_guards(buf, what):
    g = torch.cat([buf[:GUARD], buf[-GUARD:]])
    assert bool((g == SENTINEL).all()), f'{what}: an element outside the slab changed'


def stream():
    return torch.cuda.current_stream().cuda_stream


def run_case(layout, n_prompts, dtype, path, tokens, regime, scale, hw, d, entry, seed):
    """One descriptor through ``entry`` ('accumulate', 'steps' or 'range') under ``path``; checks the contract and
    returns the accumulator (None when refused) and the descriptor."""
    P, H = layout_shape(layout, n_prompts)
    scale = d ** -0.5 if scale == 'inv_sqrt_d' else scale
    q, k = make_regime(regime, P, H, hw, d, tokens, scale, dtype, seed)
    desc, qs, ks, _, _ = build_layout(layout, q.to(DEV), k.to(DEV), scale)
    shape = (P, H, tokens, hw)
    n = P * H * tokens * hw
    buf, flat = guarded(n)
    acc = flat.view(shape)
    desc.acc = acc.data_ptr()
    second_buf, second = guarded(n) if entry != 'accumulate' else (None, None)
    if entry == 'steps':
        second.fill_(-7.0)                             # every element of a step slab is written
    forms = expected_forms(desc, path, dtype, tokens)
    what = f'{layout}/P{P} {dtype} {path} {entry} T{tokens} {regime} scale {desc.scale:.4g} hw{hw} d{d}'
    calls = 2 if entry == 'range' else 1
    try:
        for _ in range(calls):
            if entry == 'accumulate':
                _native.accumulate([desc], stream(), PATHS[path])
            elif entry == 'steps':
                _native.accumulate_steps([desc], [second.data_ptr()], stream(), PATHS[path])
            else:
                _native.accumulate_range([desc], [second.data_ptr()], stream(), PATHS[path])
        torch.cuda.synchronize()
    except _native.NativeError as e:
        assert forms is None, f'{what}: refused: {e}'
        assert e.code == _native.E_UNSUPPORTED and 'layer 0' in str(e), f'{what}: {e}'
        assert bool((flat == 0).all()), f'{what}: a refused call changed the accumulator'
        assert_guards(buf, what)
        return None, desc
    assert forms is not None, f'{what}: the wgmma path accepted a layer its stride rule excludes'
    assert_guards(buf, f'{what}: accumulator')
    q64, k64 = layer_views64(desc, qs, ks)
    ref = desc_maps64(desc, qs, ks) * calls
    tol = torch.stack([accumulate_tolerance(q64, k64, float(desc.scale), f, calls) for f in forms]).amax(dim=0)
    worst = assert_close64(acc, ref, 0.0, tol, what, dims=ACC_DIMS)
    key = (path, forms[0] if len(forms) == 1 else 'auto', str(dtype).replace('torch.', ''))
    RATIOS[key] = max(RATIOS[key], worst)
    if entry != 'accumulate':
        assert_guards(second_buf, f'{what}: {entry} slab')
        assert torch.equal(second, flat), f'{what}: the {entry} slab differs from the accumulator'
    if regime == 'duplicate_k':
        for rows in duplicate_rows(tokens):
            for r in rows[1:]:
                assert torch.equal(acc[:, :, r], acc[:, :, rows[0]]), f'{what}: tokens {rows[0]} and {r} differ'
    return acc, desc


def _shape(*indices):
    return SHAPES[sum(i * m for i, m in zip(indices, (7, 3, 1, 5))) % len(SHAPES)]


@pytest.mark.parametrize('entry', ['accumulate', 'steps', 'range'])
@pytest.mark.parametrize('path', list(PATHS))
@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('layout,n_prompts', LAYOUT_CASES)
def test_layouts_77_tokens(layout, n_prompts, dtype, path, entry):
    hw, d = _shape(LAYOUT_CASES.index((layout, n_prompts)), DTYPES.index(dtype), list(PATHS).index(path),
                   ['accumulate', 'steps', 'range'].index(entry))
    run_case(layout, n_prompts, dtype, path, 77, 'gaussian', 'inv_sqrt_d', hw, d, entry, seed=hw + d)


@pytest.mark.parametrize('tokens', [154, 231])
@pytest.mark.parametrize('path', list(PATHS))
@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('layout,n_prompts', LAYOUT_CASES)
def test_layouts_long_context(layout, n_prompts, dtype, path, tokens):
    hw, d = _shape(LAYOUT_CASES.index((layout, n_prompts)), DTYPES.index(dtype), list(PATHS).index(path), tokens)
    regime = 'sinks' if (hw + d) % 2 else 'gaussian'
    run_case(layout, n_prompts, dtype, path, tokens, regime, 'inv_sqrt_d', hw, d, 'accumulate', seed=tokens + d)


@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('layout,n_prompts', LAYOUT_CASES)
def test_attention_probs_layouts(layout, n_prompts, dtype):
    """daam_attention_probs reads the same descriptors (every described sample): the SIMT softmax, then one rounding
    to the dtype of q."""
    hw, d = _shape(LAYOUT_CASES.index((layout, n_prompts)), DTYPES.index(dtype))
    P, H = layout_shape(layout, n_prompts)
    scale = d ** -0.5
    q, k = make_regime('gaussian', P, H, hw, d, 77, scale, dtype, seed=d)
    desc, qs, ks, _, _ = build_layout(layout, q.to(DEV), k.to(DEV), scale)
    n = P * H * hw * 77
    es = q.element_size()
    buf = torch.full((2 * GUARD + n,), SENTINEL, dtype=dtype, device=DEV)
    _native.attention_probs(desc, buf.data_ptr() + GUARD * es, stream())
    torch.cuda.synchronize()
    guards = torch.cat([buf[:GUARD], buf[-GUARD:]])
    assert bool((guards == SENTINEL).all()), f'{layout}: probs written outside the output'
    got = buf[GUARD:GUARD + n].view(P, H, hw, 77).transpose(-1, -2)
    q64, k64 = layer_views64(desc, qs, ks)
    tol = probs_tolerance(q64, k64, float(desc.scale), dtype)
    worst = assert_close64(got, desc_maps64(desc, qs, ks), 0.0, tol, f'{layout}/P{P} {dtype} probs', dims=ACC_DIMS)
    key = ('probs', 'simt', str(dtype).replace('torch.', ''))
    RATIOS[key] = max(RATIOS[key], worst)


@pytest.mark.parametrize('path', list(PATHS))
@pytest.mark.parametrize('dtype', DTYPES)
@pytest.mark.parametrize('tokens', [77, 154, 231])
@pytest.mark.parametrize('scale', SCALES)
@pytest.mark.parametrize('regime', REGIMES)
def test_scales_and_regimes(regime, scale, tokens, dtype, path):
    """Every logit regime at every scale, context length, dtype and path; d cycles through SD's head dims so that each
    scale meets d = 64 (where 0.125 = d^-0.5 would hide a scale derived from head_dim). The one-hot sweep runs at
    4096 pixels: 32 tiles, so that every argmax column meets every row of the 128-pixel tile."""
    d = HEAD_DIMS[(REGIMES.index(regime) + SCALES.index(scale) + tokens // 77) % len(HEAD_DIMS)]
    hw = 4096 if regime == 'one_hot' else 576
    run_case('canonical', 2, dtype, path, tokens, regime, scale, hw, d, 'accumulate',
             seed=REGIMES.index(regime) * 100 + tokens + d)


@pytest.mark.parametrize('dtype', DTYPES)
def test_expanded_k_through_make_layer_desc(dtype):
    """``k.expand(2 n, 77, C)`` (one text embedding shared by the batch) as ops.make_layer_desc describes it: prompt
    stride 0 for K with two prompts. AUTO and FORCE_SIMT match float64; FORCE_MMA refuses the layer."""
    heads, d, hw = 2, 64, 1024
    g = torch.Generator().manual_seed(11)
    q = torch.randn(4, hw, heads * d, generator=g).to(dtype).to(DEV)
    k = torch.randn(1, 77, heads * d, generator=g).to(dtype).to(DEV).expand(4, 77, heads * d)
    scale = d ** -0.5
    for path in PATHS:
        acc = ops.new_accumulator(2, heads, hw, DEV)
        desc = ops.make_layer_desc(q, k, acc, heads, scale)
        assert desc.k_stride_prompt == 0 and desc.n_prompts == 2
        if path == 'mma':
            with pytest.raises(_native.NativeError, match='layer 0') as info:
                ops.accumulate([desc], DEV, flags=PATHS[path])
            assert info.value.code == _native.E_UNSUPPORTED
            assert bool((acc == 0).all())
            continue
        ops.accumulate([desc], DEV, flags=PATHS[path])
        torch.cuda.synchronize()
        q64 = q[2:].double().reshape(2, hw, heads, d).permute(0, 2, 1, 3)
        k64 = k[2:].double().reshape(2, 77, heads, d).permute(0, 2, 1, 3)
        forms = ['simt'] if path == 'simt' else ['simt', 'split' if dtype == torch.float32 else 'wgmma16']
        tol = torch.stack([accumulate_tolerance(q64, k64, float(desc.scale), f) for f in forms]).amax(dim=0)
        ref = desc_maps64(desc, q.reshape(-1), k[:1].reshape(-1))
        assert_close64(acc, ref, 0.0, tol, f'expanded k {dtype} {path}', dims=ACC_DIMS)
