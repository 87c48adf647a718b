"""The float64 reference over raw ``daam_layer`` descriptors and the per-element accumulate bound, without a GPU.

* ``desc_maps64`` rebuilds Q / K from a descriptor's pointers and strides; here it is pinned to the numpy oracle
  (``math_layer_maps``) for every layout ``tests/test_layer_contract_gpu.py`` runs, zero and negative prompt strides
  included.
* ``accumulate_tolerance`` is sound: an fp32 emulation of the kernels' softmax (numpy float32, several summation
  orders) stays inside it in every logit regime. It has teeth: the same emulation with the logits or the probabilities
  rounded to fp16 breaks it.
"""
import numpy as np
import pytest
import torch

from daam_b200 import _native, ops
from oracle import daam_oracle as O
from tests.reference64 import (LAYOUTS, REGIMES, accumulate_tolerance, build_layout, desc_maps64, layer_maps64,
                               layer_views64, layout_shape, make_regime, mma_accepts_strides, one_hot_columns)


@pytest.mark.parametrize('name', LAYOUTS)
@pytest.mark.parametrize('n_prompts', [2, 3])
def test_desc_reference_matches_oracle(name, n_prompts):
    P, H = layout_shape(name, n_prompts)
    hw, d, T = 40, 16, 154
    q, k = make_regime('gaussian', P, H, hw, d, T, 0.25, torch.float32, seed=n_prompts)
    desc, qs, ks, q_eff, k_eff = build_layout(name, q, k, 0.25)
    qv, kv = layer_views64(desc, qs, ks)
    assert torch.equal(qv, q_eff.double()) and torch.equal(kv, k_eff.double())
    got = desc_maps64(desc, qs, ks)
    for p in range(P):
        ref = O.math_layer_maps(q_eff[p].numpy(), k_eff[p].numpy(), 0.25)
        np.testing.assert_allclose(got[p].numpy(), ref, rtol=1e-12, atol=1e-15)
    broadcast = name in ('q_broadcast', 'k_broadcast', 'negative_prompt_stride')
    assert mma_accepts_strides(desc) == (not broadcast), name


def test_desc_reference_matches_layer_maps64():
    """The canonical layout (the conditional half of a CFG batch) and a lone sample of 5 heads (the upper 3 kept), as
    ``ops.make_layer_desc`` describes them, against ``layer_maps64`` of the to_q / to_k tensors."""
    g = torch.Generator().manual_seed(5)
    for bsz, heads in ((4, 2), (1, 5)):
        d, hw = 16, 24
        q = torch.randn(bsz, hw, heads * d, generator=g)
        k = torch.randn(bsz, 77, heads * d, generator=g)
        first, n_prompts, head0, n_heads = ops.cond_half(bsz, heads)
        desc = _native.DaamLayer(
            q=q.data_ptr() + (first * q.stride(0) + head0 * d) * 4, k=k.data_ptr() + (first * k.stride(0) + head0 * d) * 4,
            acc=None, q_stride_prompt=q.stride(0), q_stride_pixel=q.stride(1), q_stride_head=d,
            k_stride_prompt=k.stride(0), k_stride_token=k.stride(1), k_stride_head=d, n_prompts=n_prompts,
            heads=n_heads, hw=hw, tokens=77, head_dim=d, dtype=0, scale=0.25, reserved=0)
        got = desc_maps64(desc, q.reshape(-1), k.reshape(-1))
        torch.testing.assert_close(got, layer_maps64(q, k, heads, 0.25), rtol=1e-12, atol=1e-15)


# ---- fp32 emulation of the kernels' softmax --------------------------------------------------------------------------
F32 = np.float32


def _sum_f32(terms: np.ndarray, order: str) -> np.ndarray:
    """Sum over the last axis with one fp32 rounding per add: left to right, right to left or as a pairwise tree.
    ``terms`` are float64 (exact products); the first level of a tree adds two of them exactly, then rounds."""
    if order == 'reverse':
        terms = terms[..., ::-1]
    if order in ('sequential', 'reverse'):
        acc = np.zeros(terms.shape[:-1], dtype=np.float64)
        for i in range(terms.shape[-1]):
            acc = (acc + terms[..., i]).astype(F32).astype(np.float64)
        return acc
    while terms.shape[-1] > 1:
        if terms.shape[-1] % 2:
            terms = np.concatenate([terms, np.zeros(terms.shape[:-1] + (1,))], axis=-1)
        terms = (terms[..., 0::2] + terms[..., 1::2]).astype(F32).astype(np.float64)
    return terms[..., 0]


def emulate_fp32(q: np.ndarray, k: np.ndarray, scale: float, order: str, round_logits=None,
                 round_probs=None) -> np.ndarray:
    """The kernels' softmax of one head in fp32 arithmetic: ``q [hw, d]``, ``k [T, d]`` (exact fp32 values) ->
    ``[T, hw]``. Dot products with exact products and one rounding per add, ``fma(s, c, -m c)`` with
    ``c = fl(scale * fl(log2 e))``, a correctly rounded exp2, the sum, ``1 / sum`` and the product in fp32.
    ``round_logits`` / ``round_probs``: a numpy dtype to round the logits / the probabilities through."""
    prods = q.astype(np.float64)[:, None, :] * k.astype(np.float64)[None, :, :]      # [hw, T, d], exact
    s = _sum_f32(prods, order)
    if round_logits is not None:
        s = s.astype(round_logits).astype(np.float64)
    c = float(F32(F32(scale) * F32(1.4426950408889634)))
    m = s.max(axis=-1, keepdims=True)
    mc = m * c
    mc = mc.astype(F32).astype(np.float64)
    a = (s * c - mc).astype(F32).astype(np.float64)
    e = np.exp2(a).astype(F32).astype(np.float64)
    e[e < 2.0 ** -126] = 0.0
    total = _sum_f32(e, order)
    inv = (1.0 / total).astype(F32).astype(np.float64)
    p = (e * inv[..., None]).astype(F32).astype(np.float64)
    if round_probs is not None:
        p = p.astype(round_probs).astype(np.float64)
    return p.T


def _worst_ratio(regime: str, T: int, scale: float, order: str, **variant) -> float:
    d, hw = 64, 128
    q, k = make_regime(regime, 1, 1, hw, d, T, scale, torch.float32, seed=T + len(regime))
    scale = float(F32(scale))
    ref = desc_free_maps(q, k, scale)
    tol = accumulate_tolerance(q.double(), k.double(), scale, 'simt')[0, 0].numpy()
    got = emulate_fp32(q[0, 0].numpy(), k[0, 0].numpy(), scale, order, **variant)
    return float((np.abs(got - ref) / tol).max())


def desc_free_maps(q: torch.Tensor, k: torch.Tensor, scale: float) -> np.ndarray:
    """The float64 softmax of head (0, 0) as ``[T, hw]``."""
    return O.math_layer_maps(q[0].numpy(), k[0].numpy(), scale)[0]


@pytest.mark.parametrize('regime', REGIMES)
@pytest.mark.parametrize('T', [77, 231])
@pytest.mark.parametrize('scale', [0.125, 1.0, 0.02, 1.37])
def test_tolerance_holds_for_fp32_emulation(regime, T, scale):
    for order in ('sequential', 'reverse', 'pairwise'):
        worst = _worst_ratio(regime, T, scale, order)
        assert worst <= 1.0, f'{regime} T={T} scale={scale} {order}: error {worst:.2f} x the bound'


@pytest.mark.parametrize('regime', ['gaussian', 'one_hot', 'sinks', 'all_negative'])
def test_tolerance_catches_fp16_logits(regime):
    assert _worst_ratio(regime, 77, 0.125, 'sequential', round_logits=np.float16) > 1.0


@pytest.mark.parametrize('regime', ['gaussian', 'one_hot', 'sinks'])
def test_tolerance_catches_fp16_probabilities(regime):
    """(Not all_negative: 150 nats of offset leave the fp32 logits an error bound above fp16's 2^-11.)"""
    assert _worst_ratio(regime, 77, 0.125, 'sequential', round_probs=np.float16) > 1.0


def test_tolerance_is_tight_enough_to_matter():
    """The fp32 emulation uses a visible share of the bound (the bound is not vacuous)."""
    worst = max(_worst_ratio(r, 77, 0.125, 'sequential') for r in ('gaussian', 'one_hot'))
    assert worst > 1e-2


def test_one_hot_regime_leads_by_40_nats_and_covers_tile_rows():
    for T in (77, 154, 231):
        for dtype in (torch.float32, torch.float16, torch.bfloat16):
            q, k = make_regime('one_hot', 1, 2, 4096, 40, T, 0.02, dtype, seed=T)
            s = (q.double() @ k.double().transpose(-1, -2)) * float(F32(0.02))
            top = s.topk(2, dim=-1).values
            assert float((top[..., 0] - top[..., 1]).min()) >= 40.0
            cols = one_hot_columns(T)
            arg = s.argmax(dim=-1)[0, 0]
            for c in cols:
                rows = {int(i) % 128 for i in torch.nonzero(arg == c).flatten()}
                assert rows == set(range(128)), (T, c)
