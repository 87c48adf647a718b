"""Parity of the fused softmax(QK^T) -> unravel -> accumulate kernel (through the C ABI) with the oracle and with the
golden vectors the verbatim reference produced. Tolerances (stated per SURVEY.md section 8c):

* fp32 inputs, SIMT path: rtol 1e-5 of the map's max, i.e. |err| <= 1e-5 * max|ref| (+1e-7) per element;
* fp16/bf16 inputs: the oracle is fed the same (half-rounded) values in fp32; same bound x 20 (tensor-core
  accumulation order and ex2.approx differ from torch's fp32 softmax).
"""
import pytest
import torch

from daam_b200 import _native, ops
from tests.util import LAYER_FIXTURES, golden, oracle_layer_maps, rel_err

pytestmark = pytest.mark.gpu
DEV = 'cuda'
TOL = {torch.float32: 1e-5, torch.float16: 2e-4, torch.bfloat16: 2e-4}

PATHS = [
    ('simt-ldst', _native.ACC_FORCE_SIMT | _native.ACC_RMW_LDST),
    ('simt-red', _native.ACC_FORCE_SIMT | _native.ACC_RMW_RED),
    ('mma-red', _native.ACC_FORCE_MMA | _native.ACC_RMW_RED),
    ('mma-ldst', _native.ACC_FORCE_MMA | _native.ACC_RMW_LDST),
    ('auto', _native.ACC_AUTO),
]


def skip_unless_mma_applies(path, dtype, head_dim):
    """The wgmma kernel takes every head_dim that is a multiple of 8 up to 192 (16-bit operands directly, fp32 as three
    bf16 terms, 64-wide K chunks); forcing it elsewhere is an error by design."""
    if path.startswith('mma') and (head_dim % 8 != 0 or head_dim > 192):
        pytest.skip('wgmma path: head_dim multiple of 8, <= 192')


def assert_close(got, ref, tol, what=''):
    ref = torch.as_tensor(ref)
    err = rel_err(got, ref)
    assert err <= tol, f'{what}: max|err|/max|ref| = {err:.3e} > {tol:.1e}'


@pytest.mark.parametrize('path,flags', PATHS)
@pytest.mark.parametrize('name', LAYER_FIXTURES)
@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
def test_golden_layers(name, dtype, path, flags):
    """Reference outputs (fixtures) vs the kernel. The fixture inputs are fp16-representable, so the fp16 run reads
    exactly the values the reference saw."""
    fx = golden(name)
    q = torch.from_numpy(fx['q']).to(DEV, dtype)
    k = torch.from_numpy(fx['k']).to(DEV, dtype)
    heads = int(fx['heads'])
    skip_unless_mma_applies(path, dtype, int(fx['head_dim']))
    acc = ops.accumulate_layer(q, k, heads, float(fx['scale']), flags=flags)
    torch.cuda.synchronize()
    ref = torch.from_numpy(fx['maps']).reshape(1, heads, 77, -1)
    assert_close(acc, ref, TOL[dtype], f'{name}/{path}')


SHAPES = [  # hw, heads, head_dim  (SD-2.1 / SDXL layer shapes, SD-1.x head dims, 96-latent partial tiles)
    (4096, 5, 64), (1024, 10, 64), (256, 20, 64), (4096, 10, 64), (1024, 20, 64),
    (1024, 8, 80), (256, 8, 160), (4096, 8, 40), (576, 10, 64), (2304, 5, 64), (144, 20, 64), (16, 2, 64),
]


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize('hw,heads,d', SHAPES)
def test_seeded_shapes_vs_oracle(hw, heads, d, dtype):
    g = torch.Generator().manual_seed(hw * 131 + heads * 7 + d)
    q = (torch.randn(2, hw, heads * d, generator=g) * 1.5).to(dtype).to(DEV)
    k = torch.randn(2, 77, heads * d, generator=g).to(dtype).to(DEV)
    acc = ops.accumulate_layer(q, k, heads)
    torch.cuda.synchronize()
    ref = oracle_layer_maps(q, k, heads, d ** -0.5).unsqueeze(0)
    assert_close(acc, ref, TOL[dtype], f'hw{hw} H{heads} d{d} {dtype}')
    # softmax rows sum to one -> every head sums to hw
    sums = acc.double().sum(dim=(2, 3))
    assert torch.allclose(sums, torch.full_like(sums, float(hw)), rtol=1e-5)
    assert (acc >= 0).all()


@pytest.mark.parametrize('dtype', [torch.float32, torch.bfloat16])
@pytest.mark.parametrize('path,flags', PATHS)
def test_time_accumulation_and_linearity(dtype, path, flags):
    """acc is a running sum over steps (daam/heatmap.py:153-156): 3 different steps, then the same step twice more."""
    hw, heads, d = 1024, 4, 64
    skip_unless_mma_applies(path, dtype, d)
    g = torch.Generator().manual_seed(5)
    acc = ops.new_accumulator(1, heads, hw, DEV)
    ref = torch.zeros(heads, 77, hw)
    for step in range(3):
        q = torch.randn(2, hw, heads * d, generator=g).to(dtype).to(DEV)
        k = torch.randn(2, 77, heads * d, generator=g).to(dtype).to(DEV)
        ops.accumulate_layer(q, k, heads, acc=acc, flags=flags)
        ref += oracle_layer_maps(q, k, heads, d ** -0.5)
    torch.cuda.synchronize()
    assert_close(acc[0], ref, TOL[dtype], path)
    before = acc.clone()
    one = ops.accumulate_layer(q, k, heads, flags=flags)
    ops.accumulate_layer(q, k, heads, acc=acc, flags=flags)
    ops.accumulate_layer(q, k, heads, acc=acc, flags=flags)
    torch.cuda.synchronize()
    assert_close(acc - before, 2 * one, 1e-6, 'linearity')


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
def test_batched_prompts_equal_independent_traces(dtype):
    """[uncond x N, cond x N] in one launch == N single-prompt calls (SURVEY.md section 7: batched = N independent traces)."""
    n, hw, heads, d = 3, 256, 4, 64
    g = torch.Generator().manual_seed(9)
    q = torch.randn(2 * n, hw, heads * d, generator=g).to(dtype).to(DEV)
    k = torch.randn(2 * n, 77, heads * d, generator=g).to(dtype).to(DEV)
    acc = ops.accumulate_layer(q, k, heads)
    assert acc.shape == (n, heads, 77, hw)
    for p in range(n):
        pair_q = torch.stack([q[p], q[n + p]])
        pair_k = torch.stack([k[p], k[n + p]])
        single = ops.accumulate_layer(pair_q, pair_k, heads)
        torch.cuda.synchronize()
        assert torch.equal(single[0], acc[p])
        assert_close(acc[p], oracle_layer_maps(pair_q, pair_k, heads, d ** -0.5), TOL[dtype], f'prompt {p}')


def test_single_sample_keeps_upper_half_of_heads():
    """Without a CFG pair the reference's `map_[map_.size(0)//2:]` keeps heads H/2.. (daam/trace.py:240)."""
    hw, heads, d = 256, 6, 64
    g = torch.Generator().manual_seed(2)
    q = torch.randn(1, hw, heads * d, generator=g).to(DEV)
    k = torch.randn(1, 77, heads * d, generator=g).to(DEV)
    acc = ops.accumulate_layer(q, k, heads)
    torch.cuda.synchronize()
    assert acc.shape == (1, heads // 2, 77, hw)
    ref = oracle_layer_maps(q, k, heads, d ** -0.5)     # the oracle applies the same rule: 3 maps
    assert ref.shape[0] == heads // 2
    assert_close(acc[0], ref, 1e-5)


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
def test_strided_and_unaligned_views(dtype):
    """q/k as slices of wider buffers (row stride != heads*d) and at element offsets that break 16-byte alignment."""
    hw, heads, d = 256, 2, 64
    g = torch.Generator().manual_seed(4)
    wide_q = torch.randn(2, hw, heads * d + 24, generator=g).to(dtype).to(DEV)
    wide_k = torch.randn(2, 77, heads * d + 24, generator=g).to(dtype).to(DEV)
    for off in (0, 8, 3):    # 8 elements keeps fp16 rows 16-byte aligned, 3 does not
        q, k = wide_q[:, :, off:off + heads * d], wide_k[:, :, off:off + heads * d]
        acc = ops.accumulate_layer(q, k, heads)
        torch.cuda.synchronize()
        assert_close(acc[0], oracle_layer_maps(q.contiguous(), k.contiguous(), heads, d ** -0.5), TOL[dtype], f'off {off}')


def test_many_layers_in_one_call_are_chunked():
    """More layer calls than one parameter block holds (32): the library splits them into several launches."""
    hw, heads, d, n_layers = 64, 2, 64, 45
    g = torch.Generator().manual_seed(8)
    qs = [torch.randn(2, hw, heads * d, generator=g).half().to(DEV) for _ in range(n_layers)]
    ks = [torch.randn(2, 77, heads * d, generator=g).half().to(DEV) for _ in range(n_layers)]
    accs = [ops.new_accumulator(1, heads, hw, DEV) for _ in range(n_layers)]
    before = _native.launch_count()
    ops.accumulate([ops.make_layer_desc(q, k, a, heads, d ** -0.5) for q, k, a in zip(qs, ks, accs)], DEV)
    torch.cuda.synchronize()
    assert _native.launch_count() - before == 2
    for i in (0, 31, 32, 44):
        assert_close(accs[i][0], oracle_layer_maps(qs[i], ks[i], heads, d ** -0.5), TOL[torch.float16], f'layer {i}')


def test_mixed_dtypes_and_shapes_in_one_call():
    g = torch.Generator().manual_seed(12)
    cases = [(4096, 5, 64, torch.bfloat16), (256, 20, 64, torch.float16), (1024, 10, 64, torch.float32),
             (1024, 8, 40, torch.float16)]
    qs, ks, accs, descs = [], [], [], []
    for hw, heads, d, dt in cases:
        q = torch.randn(2, hw, heads * d, generator=g).to(dt).to(DEV)
        k = torch.randn(2, 77, heads * d, generator=g).to(dt).to(DEV)
        a = ops.new_accumulator(1, heads, hw, DEV)
        qs.append(q), ks.append(k), accs.append(a)
        descs.append(ops.make_layer_desc(q, k, a, heads, d ** -0.5))
    ops.accumulate(descs, DEV)
    torch.cuda.synchronize()
    for (hw, heads, d, dt), q, k, a in zip(cases, qs, ks, accs):
        assert_close(a[0], oracle_layer_maps(q, k, heads, d ** -0.5), TOL[dt], f'{hw}/{heads}/{d}/{dt}')


def test_extreme_logits_stay_finite():
    """Peaky rows (|logit| ~ 80) must neither overflow nor produce NaN; one-hot rows come out as exactly 0/1 sums."""
    hw, heads, d = 256, 2, 64
    g = torch.Generator().manual_seed(3)
    q = (torch.randn(2, hw, heads * d, generator=g) * 10).half().to(DEV)
    k = (torch.randn(2, 77, heads * d, generator=g) * 8).half().to(DEV)
    acc = ops.accumulate_layer(q, k, heads)
    torch.cuda.synchronize()
    assert torch.isfinite(acc).all()
    assert_close(acc[0], oracle_layer_maps(q, k, heads, d ** -0.5), 1e-3, 'peaky')


def test_invalid_arguments_are_rejected():
    q = torch.randn(2, 64, 128, device=DEV)
    k76 = torch.randn(2, 76, 128, device=DEV)
    acc = ops.new_accumulator(1, 2, 64, DEV)
    with pytest.raises(_native.NativeError) as e:
        ops.accumulate([ops.make_layer_desc(q, k76, acc, 2, 0.125)], DEV)
    assert e.value.code == _native.E_UNSUPPORTED and '77' in str(e.value)
    q12 = torch.randn(2, 64, 24, device=DEV)     # head_dim 12: not a multiple of 8
    k12 = torch.randn(2, 77, 24, device=DEV)
    with pytest.raises(_native.NativeError):
        ops.accumulate([ops.make_layer_desc(q12, k12, acc, 2, 0.3)], DEV)
    with pytest.raises(RuntimeError, match='accumulator must be'):
        ops.make_layer_desc(q, torch.randn(2, 77, 128, device=DEV), ops.new_accumulator(1, 3, 64, DEV), 2, 0.125)
    with pytest.raises(RuntimeError, match='CUDA tensors only'):
        ops.make_layer_desc(q.cpu(), k76.cpu(), acc, 2, 0.125)


def test_forcing_tcgen05_on_unsupported_input_is_an_error():
    wide_q = torch.randn(2, 64, 136, device=DEV)
    wide_k = torch.randn(2, 77, 136, device=DEV)
    q, k = wide_q[:, :, 3:131], wide_k[:, :, 3:131]          # rows not 16-byte aligned: no TMA / vector loads
    with pytest.raises(_native.NativeError) as e:
        ops.accumulate_layer(q, k, 2, flags=_native.ACC_FORCE_MMA)
    assert e.value.code == _native.E_UNSUPPORTED
    acc = ops.accumulate_layer(q, k, 2)                       # AUTO falls back to the SIMT kernel
    torch.cuda.synchronize()
    assert_close(acc[0], oracle_layer_maps(q.contiguous(), k.contiguous(), 2, 0.125), 1e-5)


@pytest.mark.parametrize('mode', [_native.ACC_RMW_RED, _native.ACC_RMW_LDST])
def test_tcgen05_partial_and_tiny_tiles(mode):
    """hw not a multiple of the 128-pixel tile (576 = 4.5 tiles, 144, 16): TMA zero-fills the tail rows and clips the
    reduce; nothing outside the head's [77, hw] slab may be touched (guard rows before/after stay zero)."""
    for hw, heads in [(576, 3), (144, 2), (16, 2), (2304, 2)]:
        g = torch.Generator().manual_seed(hw)
        q = torch.randn(2, hw, heads * 64, generator=g).half().to(DEV)
        k = torch.randn(2, 77, heads * 64, generator=g).half().to(DEV)
        slab = torch.zeros(heads + 2, 77, hw, device=DEV)
        acc = slab[1:-1].unsqueeze(0)
        ops.accumulate([ops.make_layer_desc(q, k, acc, heads, 0.125)], DEV, flags=_native.ACC_FORCE_MMA | mode)
        torch.cuda.synchronize()
        assert_close(acc[0], oracle_layer_maps(q, k, heads, 0.125), TOL[torch.float16], f'hw {hw}')
        assert float(slab[0].abs().max()) == 0.0 and float(slab[-1].abs().max()) == 0.0


def test_full_size_sd21_step_properties():
    """BASELINE configs[1] sizes (all 15 SD-2.1 layers, bf16), checked through size-independent properties:
    per-head sums == steps * hw, non-negativity, and step-linearity."""
    shapes = [(256, 20)] * 3 + [(1024, 10)] * 3 + [(4096, 5)] * 3 + [(4096, 5)] * 2 + [(1024, 10)] * 2 + [(256, 20)] * 2
    g = torch.Generator().manual_seed(21)
    qs = [torch.randn(2, hw, h * 64, generator=g).bfloat16().to(DEV) for hw, h in shapes]
    ks = [torch.randn(2, 77, h * 64, generator=g).bfloat16().to(DEV) for hw, h in shapes]
    accs = [ops.new_accumulator(1, h, hw, DEV) for hw, h in shapes]
    descs = [ops.make_layer_desc(q, k, a, h, 0.125) for q, k, a, (hw, h) in zip(qs, ks, accs, shapes)]
    steps = 4
    for _ in range(steps):
        ops.accumulate(descs, DEV)
    torch.cuda.synchronize()
    for a, (hw, h) in zip(accs, shapes):
        sums = a.double().sum(dim=(2, 3))
        assert torch.allclose(sums, torch.full_like(sums, float(steps * hw)), rtol=2e-5)
        assert (a >= 0).all()
    one = [ops.accumulate_layer(q, k, h) for q, k, (hw, h) in zip(qs, ks, shapes)]
    torch.cuda.synchronize()
    for a, o in zip(accs, one):
        assert_close(a, steps * o, 1e-6, 'steps x single')
    # and one layer of each resolution against the oracle at full size
    for i in (0, 3, 6):
        hw, h = shapes[i]
        assert_close(one[i][0], oracle_layer_maps(qs[i], ks[i], h, 0.125), TOL[torch.bfloat16], f'layer {i}')


@pytest.mark.parametrize('dtype,tol', [(torch.float32, 1e-5), (torch.float16, 1e-3), (torch.bfloat16, 8e-3)])
@pytest.mark.parametrize('hw,heads,d', [(1024, 4, 64), (576, 2, 64), (64, 2, 40), (4096, 1, 64)])
def test_materialised_probs_match_get_attention_scores(hw, heads, d, dtype, tol):
    """daam_attention_probs == diffusers' get_attention_scores (reference call at trace.py:276) for every sample;
    daam_accumulate_probs == _unravel_attn + update on that tensor. Tolerance: one rounding to the output dtype."""
    from daam_b200.testing.synthetic import SyntheticAttention
    g = torch.Generator().manual_seed(hw + d)
    q = torch.randn(2, hw, heads * d, generator=g).to(dtype).to(DEV)
    k = torch.randn(2, 77, heads * d, generator=g).to(dtype).to(DEV)
    probs = ops.attention_probs(q, k, heads)
    torch.cuda.synchronize()
    assert probs.shape == (2 * heads, hw, 77) and probs.dtype == dtype
    attn = SyntheticAttention(heads * d, heads * d, heads, d)
    ref = attn.get_attention_scores(attn.head_to_batch_dim(q.float().cpu()), attn.head_to_batch_dim(k.float().cpu()))
    assert rel_err(probs.float(), ref) < tol
    acc = ops.new_accumulator(1, heads, hw, DEV)
    ops.accumulate_probs(probs, acc)
    ops.accumulate_probs(probs, acc)
    torch.cuda.synchronize()
    from oracle import daam_oracle as O
    want = 2 * O.port_unravel(probs.float().cpu()).reshape(heads, 77, hw)
    assert rel_err(acc[0], want) < 1e-6


def test_fp32_split_path_accuracy_and_properties():
    """fp32 projections on tensor cores (three bf16 terms per value, six products): as accurate as the fp32 SIMT kernel
    (both within 1e-5 of the oracle), including peaky logits, partial tiles and several layers per launch."""
    g = torch.Generator().manual_seed(77)
    for hw, heads, gain in [(4096, 5, 1.0), (1024, 10, 3.0), (576, 3, 1.0), (16, 2, 6.0)]:
        q = (torch.randn(2, hw, heads * 64, generator=g) * gain).to(DEV)
        k = torch.randn(2, 77, heads * 64, generator=g).to(DEV)
        ref = oracle_layer_maps(q, k, heads, 0.125).unsqueeze(0)
        split = ops.accumulate_layer(q, k, heads, flags=_native.ACC_FORCE_MMA)
        simt = ops.accumulate_layer(q, k, heads, flags=_native.ACC_FORCE_SIMT)
        torch.cuda.synchronize()
        e_split, e_simt = rel_err(split, ref), rel_err(simt, ref)
        assert e_split < 1e-5 and e_simt < 1e-5, (hw, heads, e_split, e_simt)
        sums = split.double().sum(dim=(2, 3))
        assert torch.allclose(sums, torch.full_like(sums, float(hw)), rtol=1e-6)


def test_empty_call_and_smallest_maps():
    """Zero layers is a no-op; the smallest map the API admits (2x2 pixels) still goes through both kernels."""
    before = _native.launch_count()
    ops.accumulate([], DEV)
    assert _native.launch_count() == before
    g = torch.Generator().manual_seed(0)
    for dtype, flags in [(torch.float16, _native.ACC_FORCE_MMA), (torch.float32, _native.ACC_FORCE_MMA),
                         (torch.float32, _native.ACC_FORCE_SIMT)]:
        q = torch.randn(2, 4, 64, generator=g).to(dtype).to(DEV)
        k = torch.randn(2, 77, 64, generator=g).to(dtype).to(DEV)
        acc = ops.accumulate_layer(q, k, 1, flags=flags)
        torch.cuda.synchronize()
        assert_close(acc[0], oracle_layer_maps(q, k, 1, 0.125), TOL[dtype], f'{dtype}')


@pytest.mark.parametrize('dtype', [torch.float16, torch.bfloat16, torch.float32])
@pytest.mark.parametrize('hw,heads,d', [(4096, 8, 40), (1024, 8, 80), (256, 8, 160), (64, 4, 128), (1024, 4, 8)])
def test_sd1x_head_dims_on_tensor_cores(hw, heads, d, dtype):
    """SD-1.x head dims (40 / 80 / 160) and other multiples of 8: K-chunked wgmma path == SIMT path == oracle."""
    g = torch.Generator().manual_seed(d * 7 + hw)
    q = torch.randn(2, hw, heads * d, generator=g).to(dtype).to(DEV)
    k = torch.randn(2, 77, heads * d, generator=g).to(dtype).to(DEV)
    mma = ops.accumulate_layer(q, k, heads, flags=_native.ACC_FORCE_MMA)
    simt = ops.accumulate_layer(q, k, heads, flags=_native.ACC_FORCE_SIMT)
    torch.cuda.synchronize()
    ref = oracle_layer_maps(q, k, heads, d ** -0.5).unsqueeze(0)
    assert_close(mma, ref, TOL[dtype], f'mma d{d}')
    assert_close(simt, ref, TOL[dtype], f'simt d{d}')


def test_full_size_sdxl_and_batched_step_properties():
    """BASELINE configs 3-5 sizes: the 60 traced SDXL layers (fp16) with 2 prompts in one call, and SD-2.1 with 8 prompts
    (bf16) -- checked through per-head sums (= steps * hw), non-negativity, and batched == per-prompt launches."""
    import bench
    for workload, dtype, prompts in [('sdxl', torch.float16, 2), ('sd21', torch.bfloat16, 8)]:
        layers = bench.traced_layers(workload)
        g = torch.Generator(device=DEV).manual_seed(5)
        qs = [torch.randn(2 * prompts, hw, h * d, generator=g, device=DEV).to(dtype) for hw, h, d in layers]
        ks = [torch.randn(2 * prompts, 77, h * d, generator=g, device=DEV).to(dtype) for hw, h, d in layers]
        accs = [ops.new_accumulator(prompts, h, hw, DEV) for hw, h, d in layers]
        descs = [ops.make_layer_desc(q, k, a, h, d ** -0.5) for q, k, a, (hw, h, d) in zip(qs, ks, accs, layers)]
        before = _native.launch_count()
        for _ in range(2):
            ops.accumulate(descs, DEV)
        torch.cuda.synchronize()
        assert _native.launch_count() - before == 2 * -(-len(layers) // 32)      # 32 layer descriptors per launch
        for a, (hw, h, d) in zip(accs, layers):
            sums = a.double().sum(dim=(2, 3))
            assert torch.allclose(sums, torch.full_like(sums, 2.0 * hw), rtol=2e-5)
            assert (a >= 0).all()
        for i in (0, len(layers) // 2, len(layers) - 1):       # batched launch == independent single-prompt launches
            hw, h, d = layers[i]
            for p in (0, prompts - 1):
                pair_q, pair_k = torch.stack([qs[i][p], qs[i][prompts + p]]), torch.stack([ks[i][p], ks[i][prompts + p]])
                single = ops.accumulate_layer(pair_q, pair_k, h)
                torch.cuda.synchronize()
                assert_close(accs[i][p], 2 * single[0], 1e-6, f'{workload} layer {i} prompt {p}')
