"""The float64 reference of tests/reference64.py: pinned to the numpy oracle, and shown to tell a wrong result from a
right one where the size-independent properties of the older full-size tests cannot.

Everything here runs on CPU tensors except the one test that checks the CUDA run of the reference against its CPU run.
No kernel is mutated: the wrong results are built from the reference itself.
"""
import numpy as np
import pytest
import torch

from oracle import daam_oracle as O
from tests.reference64 import (ACC_DIMS, MAP_DIMS, assert_close64, finalize_tolerance, global_map64, layer_maps64,
                               per_key_maps64)

PIN = 1e-12


def _qk(b, hw, heads, d, seed, gain=1.5):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(b, hw, heads * d, generator=g) * gain, torch.randn(b, 77, heads * d, generator=g)


def _oracle_layer(q, k, heads, scale):
    """O.math_layer_maps for every kept (prompt, head): [n_prompts, n_heads, 77, hw]."""
    b, hw, c = q.shape
    d = c // heads
    if b % 2 == 0:
        samples, head0 = range(b // 2, b), 0
    else:
        samples, head0 = [0], heads // 2
    out = []
    for s in samples:
        qh = q[s].double().numpy().reshape(hw, heads, d).transpose(1, 0, 2)[head0:]
        kh = k[s].double().numpy().reshape(77, heads, d).transpose(1, 0, 2)[head0:]
        out.append(O.math_layer_maps(qh, kh, scale))
    return torch.from_numpy(np.stack(out))


@pytest.mark.parametrize('b,hw,heads,d', [(2, 256, 3, 64), (4, 64, 2, 40), (6, 144, 5, 80), (1, 64, 5, 64)])
def test_layer_maps64_equals_the_oracle(b, hw, heads, d):
    q, k = _qk(b, hw, heads, d, b * 1000 + hw + d)
    got = layer_maps64(q, k, heads, d ** -0.5)
    want = _oracle_layer(q, k, heads, d ** -0.5)
    assert got.dtype == torch.float64 and got.shape == want.shape
    assert_close64(got, want, PIN, 1e-300, 'layer_maps64', ACC_DIMS)
    # the same slice as the op-for-op port of the reference (fp32 there, so only to its rounding)
    port = O.port_layer_step(q, k, heads, d ** -0.5).reshape(got.shape)
    assert_close64(port, got, 1e-5, 1e-6, 'port_layer_step', ACC_DIMS)


def _stacks(sides, heads, seed, tokens=12):
    g = torch.Generator().manual_seed(seed)
    return [torch.exp(torch.randn(h, tokens, s, s, generator=g, dtype=torch.float64)) for s, h in zip(sides, heads)]


@pytest.mark.parametrize('x,sides', [(64, [64, 32, 16]), (96, [96, 48, 24]), (64, [16])])
@pytest.mark.parametrize('normalize', [False, True])
@pytest.mark.parametrize('head_sel', [None, 1])
def test_global_map64_equals_the_oracle(x, sides, normalize, head_sel):
    stacks = _stacks(sides, [2 + i for i in range(len(sides))], x + len(sides))
    n_rows = 9
    got = global_map64(stacks, x, n_rows, normalize, head_sel)
    keys = [s[h].numpy() for s in stacks for h in (range(s.shape[0]) if head_sel is None else [head_sel])]
    want = torch.from_numpy(O.math_global_heat_map(keys, x, n_rows, normalize))
    # the upsample cancels (negative cubic weights): near-zero elements are pinned relative to the map's scale
    assert_close64(got, want, PIN, PIN * float(want.abs().max()), 'global_map64', MAP_DIMS)


@pytest.mark.parametrize('normalize', [False, True])
def test_per_key_maps64_equals_the_oracle(normalize):
    stack = _stacks([32], [3], 7)[0]
    got = per_key_maps64(stack, 64, 6, normalize)
    for h in range(3):
        want = torch.from_numpy(O.math_global_heat_map([stack[h].numpy()], 64, 6, normalize))
        assert_close64(got[h], want, PIN, PIN * float(want.abs().max()), f'key {h}', MAP_DIMS)


def test_comparator_names_the_worst_element():
    ref = torch.rand(2, 3, 77, 256, dtype=torch.float64) + 0.5
    got = ref.clone()
    got[1, 2, 40, 200] += 1.0
    with pytest.raises(AssertionError, match='layer 4: worst element at prompt 1, head 2, token 40, pixel 200'):
        assert_close64(got, ref, 1e-4, 1e-5, 'layer 4', ACC_DIMS)
    got = ref.clone()
    got[0, 1, 2, 3] = float('nan')
    with pytest.raises(AssertionError, match='prompt 0, head 1, token 2, pixel 3'):
        assert_close64(got, ref, 1e-4, 1e-5, 'nan', ACC_DIMS)
    assert assert_close64(ref.float(), ref, 1e-6, 0.0) <= 1.0


@pytest.mark.gpu
def test_cuda_run_of_the_reference_equals_its_cpu_run():
    q, k = _qk(4, 1024, 5, 64, 3)
    cpu = layer_maps64(q, k, 5, 0.125)
    gpu = layer_maps64(q.cuda(), k.cuda(), 5, 0.125)
    assert_close64(gpu, cpu.cuda(), PIN, 1e-300, 'layer_maps64 cuda vs cpu', ACC_DIMS)
    stacks = _stacks([64, 32, 16], [5, 10, 20], 4, tokens=77)
    cpu = global_map64(stacks, 64, 77, True)
    gpu = global_map64([s.cuda() for s in stacks], 64, 77, True)
    assert_close64(gpu, cpu.cuda(), PIN, PIN * float(cpu.abs().max()), 'global_map64 cuda vs cpu', MAP_DIMS)


# --------------------------------------------------------------------------------------------------------------------
# sensitivity: wrong results the per-head-sum / non-negativity / batched-equals-single properties accept
# --------------------------------------------------------------------------------------------------------------------
RTOL16, ATOL16 = 1e-4, 1e-5          # per-key tolerance of 16-bit inputs (test_parity_elementwise_gpu.py), atol x steps


@pytest.fixture(scope='module')
def two_steps():
    """Two steps of distinct Q/K, 2 prompts x 3 heads x 1024 pixels (8 tiles of 128): the float64 per-step maps, and
    the exact two-step accumulator rounded to fp32 as a kernel would store it."""
    s0 = layer_maps64(*_qk(4, 1024, 3, 64, 10), 3, 0.125)
    s1 = layer_maps64(*_qk(4, 1024, 3, 64, 11), 3, 0.125)
    return s0, s1, (s0 + s1).float()


def _check(acc, ref):
    assert_close64(acc, ref, RTOL16, 2 * ATOL16, 'accumulator', ACC_DIMS)


def _properties_hold(acc, steps, hw):
    sums = acc.double().sum(dim=(2, 3))
    return bool(torch.allclose(sums, torch.full_like(sums, float(steps * hw)), rtol=2e-5)) and bool((acc >= 0).all())


def test_the_exact_accumulator_passes(two_steps):
    s0, s1, acc = two_steps
    _check(acc, s0 + s1)
    assert _properties_hold(acc, 2, 1024)


@pytest.mark.parametrize('case', ['swap_heads', 'swap_tiles', 'swap_prompts'])
def test_permutations_pass_the_properties_and_fail_the_comparator(two_steps, case):
    s0, s1, acc = two_steps
    bad = acc.clone()
    if case == 'swap_heads':
        bad[0, [0, 2]] = bad[0, [2, 0]]
    elif case == 'swap_tiles':                      # two 128-pixel tiles of one head
        bad[1, 1, :, 256:384], bad[1, 1, :, 640:768] = acc[1, 1, :, 640:768], acc[1, 1, :, 256:384]
    else:
        bad[[0, 1]] = bad[[1, 0]]
    assert _properties_hold(bad, 2, 1024)            # why the older full-size checks are not enough
    with pytest.raises(AssertionError, match='worst element'):
        _check(bad, s0 + s1)


def test_a_stale_ring_slot_fails_the_comparator(two_steps):
    """One tile that also received the previous step's values (a ring slot released too early, a skipped load)."""
    s0, s1, acc = two_steps
    bad = acc.clone()
    bad[1, 2, :, 384:512] += s0[1, 2, :, 384:512].float()
    with pytest.raises(AssertionError, match='prompt 1, head 2, token [0-9]+, pixel (38[4-9]|39[0-9]|4[0-9][0-9]|50[0-9]|51[01])'):
        _check(bad, s0 + s1)


def test_one_element_off_by_ten_bounds_fails_the_comparator(two_steps):
    s0, s1, acc = two_steps
    ref = s0 + s1
    bad = acc.clone()
    bad[0, 1, 76, 1023] += 10 * (2 * ATOL16 + RTOL16 * float(ref[0, 1, 76, 1023]))
    with pytest.raises(AssertionError, match='prompt 0, head 1, token 76, pixel 1023'):
        _check(bad, ref)


def test_finalize_chunk_errors_fail_the_comparator():
    """A factor-2 class of 50 keys (several cp.async chunks in the fast kernel): one key left out of a chunk, and a
    chunk counted twice, both still divided by the number of keys."""
    g = torch.Generator().manual_seed(12)
    stacks = [torch.exp(torch.randn(10, 77, 32, 32, generator=g)) for _ in range(5)]
    n_rows, n = 40, 50
    ref = global_map64(stacks, 64, n_rows)
    rtol, atol = finalize_tolerance(stacks, n, 64)
    assert_close64(ref.float(), ref, rtol, atol, 'exact', MAP_DIMS)
    dropped = ref - global_map64([stacks[2][3:4]], 64, n_rows) / n
    with pytest.raises(AssertionError, match='worst element'):
        assert_close64(dropped.float(), ref, rtol, atol, 'key dropped', MAP_DIMS)
    twice = ref + global_map64([stacks[1][4:], stacks[2][:6]], 64, n_rows) * (12 / n)
    with pytest.raises(AssertionError, match='worst element'):
        assert_close64(twice.float(), ref, rtol, atol, 'chunk twice', MAP_DIMS)
