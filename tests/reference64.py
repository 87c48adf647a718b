"""Float64 statements of the two hot-path reductions, written in torch so that they run on the GPU next to the kernels,
and an element-wise comparator that stays on the device.

* :func:`layer_maps64` is ``oracle.daam_oracle.math_layer_maps`` (rows a3 + a4) for raw projections, taking the
  conditional half and the head split exactly as ``port_layer_step`` does.
* :func:`global_map64` / :func:`per_key_maps64` are ``math_global_heat_map`` (row a7): every key upsampled as
  ``B_y @ key @ B_x^T`` with the matrices of ``math_bicubic_matrix``, clamped, averaged, optionally normalised.

``tests/test_reference64.py`` pins both to the numpy oracle to 1e-12. They work on one layer / one key stack at a time,
so a production-size workload is never held in float64 as a whole.
"""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import torch

from oracle import daam_oracle as O

ACC_DIMS = ('prompt', 'head', 'token', 'pixel')      # an accumulator [n_prompts, heads, 77, hw]
MAP_DIMS = ('row', 'y', 'x')                         # a global heat map [n_rows, x, x]


def layer_maps64(q: torch.Tensor, k: torch.Tensor, heads: int, scale: float) -> torch.Tensor:
    """softmax_t(scale * q . k) in float64 for ``q [B, hw, heads*d]``, ``k [B, 77, heads*d]`` as ``to_q`` / ``to_k``
    emit them -> ``[n_prompts, n_heads, 77, hw]``, the accumulator layout of the kept slice.

    Kept slice: the second half of the ``B * heads`` axis (daam/trace.py:240, ``port_unravel``): the conditional
    samples with all heads for a CFG batch, the upper half of the heads for a lone sample."""
    b, hw, c = q.shape
    d = c // heads
    first = (b * heads) // 2
    split = lambda t: t.reshape(b, t.shape[1], heads, d).permute(0, 2, 1, 3).reshape(b * heads, t.shape[1], d)
    qh = split(q)[first:].double()
    kh = split(k)[first:].double()
    s = torch.bmm(qh, kh.transpose(1, 2)) * scale                       # [rows, hw, 77]
    s = s - s.amax(dim=-1, keepdim=True)
    e = torch.exp(s)
    p = (e / e.sum(dim=-1, keepdim=True)).transpose(1, 2)               # [rows, 77, hw]
    n_prompts, n_heads = (b // 2, heads) if b % 2 == 0 else (1, b * heads - first)
    return p.reshape(n_prompts, n_heads, k.shape[1], hw).contiguous()


def bicubic64(n_in: int, n_out: int, device) -> torch.Tensor:
    """``math_bicubic_matrix`` as a float64 tensor on ``device``: ``[n_out, n_in]``."""
    return torch.from_numpy(O.math_bicubic_matrix(n_in, n_out)).to(device)


def upsample64(keys: torch.Tensor, x: int) -> torch.Tensor:
    """``[..., h, w]`` -> ``[..., x, x]``: ``B_y @ key @ B_x^T`` in float64."""
    by, bx = bicubic64(keys.shape[-2], x, keys.device), bicubic64(keys.shape[-1], x, keys.device)
    return by @ keys.double() @ bx.T


def _normalize(maps: torch.Tensor) -> torch.Tensor:
    """maps / (sum of rows 1..-2 + 1e-6) per pixel (daam/trace.py:129-130) over the row axis -3."""
    return maps / (maps[..., 1:-1, :, :].sum(dim=-3, keepdim=True) + 1e-6)


def global_map64(keys: Sequence[torch.Tensor], x: int, n_rows: int, normalize: bool = False,
                 head_sel: Optional[int] = None) -> torch.Tensor:
    """``math_global_heat_map`` over key stacks: each element of ``keys`` is ``[heads, tokens, h, w]`` (one layer's
    slab of one prompt, as ``daam_key_group`` points at it); ``head_sel`` keeps one head of every stack. The rows past
    ``n_rows`` are dropped before the upsample (the arithmetic is row-wise). Returns ``[n_rows, x, x]`` float64."""
    total, n = None, 0
    for stack in keys:
        sel = stack[:, :n_rows] if head_sel is None else stack[head_sel:head_sel + 1, :n_rows]
        part = upsample64(sel, x).clamp_(min=0.0).sum(dim=0)
        total = part if total is None else total + part
        n += sel.shape[0]
    if n == 0:
        raise ValueError('no key selected')
    out = total / n
    return _normalize(out) if normalize else out


def per_key_maps64(stack: torch.Tensor, x: int, n_rows: int, normalize: bool = False) -> torch.Tensor:
    """What ``daam_finalize_per_key`` computes for one key stack ``[heads, tokens, h, w]``: every key's own global map
    (bicubic + clamp, optional normalisation) -> ``[heads, n_rows, x, x]`` float64."""
    out = upsample64(stack[:, :n_rows], x).clamp_(min=0.0)
    return _normalize(out) if normalize else out


FP32_EPS = 2.0 ** -24                                # unit roundoff of fp32


def finalize_tolerance(stacks: Sequence[torch.Tensor], n_keys: int, x: int) -> Tuple[float, float]:
    """``(rtol, atol)`` of a fp32 global heat map (``daam_finalize``) against :func:`global_map64`, from an error
    bound rather than from observed errors:

    * rtol: the map is a mean of ``n_keys`` non-negative fp32 terms. Summing them in any order, then dividing, has a
      relative error below ``(n_keys + 1) * 2^-24``: 7e-5 for SDXL's 1200-key class, 1.3e-4 for SDXL with 2 images
      per prompt (2200 keys). The contract's global-map rtol (1e-4, SURVEY.md section 8c) is used where it is larger.
    * atol: each upsampled value is a 16-tap stencil (4 taps per axis) with fp32 weights. Its fp32 evaluation, the
      rounding of the weights and of their products included, errs by less than ``32 * 2^-24`` times
      ``sum |w_y| |w_x| |v|``, which is at most ``N^2 * max |v|``: ``N`` is the largest row 1-norm of the bicubic
      matrices involved (1 for factor 1, 1.28 for factor 2, 1.35 for factor 4 of the A = -0.75 cubic) and ``max |v|``
      the largest key magnitude. The clamp is 1-Lipschitz and the mean of the keys' errors is below their maximum.

    ``stacks``: the key stacks the map reads (only their sides and magnitudes are used)."""
    norm = max(float(bicubic64(s.shape[-1], x, 'cpu').abs().sum(dim=1).max()) for s in stacks)
    vmax = max(float(s.abs().max()) for s in stacks)
    return max(1e-4, (n_keys + 1) * FP32_EPS), 32 * FP32_EPS * norm * norm * vmax


def normalized_tolerance(raw: torch.Tensor, rtol: float, atol: float) -> torch.Tensor:
    """Per-element bound of ``raw / (sum of rows 1..-2 + 1e-6)`` (the ``normalize`` step, computed in fp32 from a fp32
    map within ``atol + rtol * |raw|`` of ``raw``), as an absolute tolerance tensor (use with rtol = 0).
    With ``a`` the element, ``b`` its denominator, ``Ta`` / ``Tb`` their error bounds:
    ``|d(a / b)| <= Ta / b + (a / b) * Tb / b``, plus the rounding of the division. ``Tb`` adds the fp32 summation of
    the ``n_rows - 2`` rows, ``n_rows * 2^-24 * b``."""
    a = raw.double()
    b = a[1:-1].sum(dim=0, keepdim=True) + 1e-6
    ta = atol + rtol * a.abs()
    tb = ta[1:-1].sum(dim=0, keepdim=True) + a.shape[0] * FP32_EPS * b
    return ta / b + (a.abs() / b) * (tb / b + 2 * FP32_EPS)


def _decode(index: int, shape: Tuple[int, ...], dims: Optional[Sequence[str]]) -> str:
    coords = []
    for size in reversed(shape):
        coords.append(index % size)
        index //= size
    coords = coords[::-1]
    if dims is None or len(dims) != len(shape):
        return str(tuple(coords))
    return ', '.join(f'{n} {c}' for n, c in zip(dims, coords))


def assert_close64(got: torch.Tensor, ref: torch.Tensor, rtol: float, atol, what: str = '',
                   dims: Optional[Sequence[str]] = None) -> float:
    """``|got - ref| <= atol + rtol * |ref|`` for every element (the form of ``tests.util.assert_elementwise``), computed
    where the tensors live: only the worst ratio and, on failure, the worst element travel to the host. ``atol`` may be a
    tensor broadcastable to ``ref`` (a per-element bound). ``dims`` names the axes, so that a failure reads e.g.
    ``layer 7: prompt 1, head 3, token 12, pixel 4095``. Returns the worst ratio of error to bound."""
    assert tuple(got.shape) == tuple(ref.shape), f'{what}: shape {tuple(got.shape)} vs {tuple(ref.shape)}'
    ref = ref.to(device=got.device, dtype=torch.float64)
    excess = (got.double() - ref).abs_().div_(ref.abs().mul_(rtol).add_(atol))
    excess = torch.where(torch.isnan(excess), torch.full_like(excess, float('inf')), excess)
    i = int(excess.argmax())
    worst = float(excess.reshape(-1)[i])
    if not worst <= 1.0:
        g, r = float(got.reshape(-1)[i]), float(ref.reshape(-1)[i])
        bound = float(torch.as_tensor(atol, dtype=torch.float64, device=ref.device).expand_as(ref).reshape(-1)[i]) \
            if isinstance(atol, torch.Tensor) else atol
        raise AssertionError(f'{what}: worst element at {_decode(i, tuple(ref.shape), dims)}: got {g:.9e} ref {r:.9e} '
                             f'= {worst:.2f} x (atol {bound:.1e} + rtol {rtol:.1e} * |ref|)')
    return worst
