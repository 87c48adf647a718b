"""Float64 statements of the two hot-path reductions, written in torch so that they run on the GPU next to the kernels,
and an element-wise comparator that stays on the device.

* :func:`layer_maps64` is ``oracle.daam_oracle.math_layer_maps`` (rows a3 + a4) for raw projections, taking the
  conditional half and the head split exactly as ``port_layer_step`` does.
* :func:`global_map64` / :func:`per_key_maps64` are ``math_global_heat_map`` (row a7): every key upsampled as
  ``B_y @ key @ B_x^T`` with the matrices of ``math_bicubic_matrix``, clamped, averaged, optionally normalised.
* :func:`desc_maps64` is the same softmax over a raw ``daam_layer``: the Q / K views are rebuilt from the descriptor's
  pointers and strides (any layout the C ABI accepts), and :func:`accumulate_tolerance` bounds each accumulator
  element a kernel may produce from them. :func:`build_layout` / :func:`make_regime` make the layouts and logit
  regimes ``tests/test_layer_contract_*.py`` run.

``tests/test_reference64.py`` pins both to the numpy oracle to 1e-12. They work on one layer / one key stack at a time,
so a production-size workload is never held in float64 as a whole.
"""
from __future__ import annotations

import math
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


def up64(keys: torch.Tensor, grid: Tuple[int, int]) -> torch.Tensor:
    """``[..., h, w]`` -> ``[..., grid[0], grid[1]]``: ``B_y @ key @ B_x^T`` in float64, each axis with its own
    bicubic matrix (rectangular maps and keys)."""
    by = bicubic64(keys.shape[-2], grid[0], keys.device)
    bx = bicubic64(keys.shape[-1], grid[1], keys.device)
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


def rect_tolerance(stacks: Sequence[torch.Tensor], n_keys: int, grid: Tuple[int, int]) -> Tuple[float, float]:
    """:func:`finalize_tolerance` with the 1-norms of both axes' bicubic matrices (keys and maps that are not square):
    ``stacks`` are ``[..., h, w]`` key stacks, ``grid`` the map's ``(h, w)``."""
    norm = max(float(bicubic64(t.shape[-2], grid[0], 'cpu').abs().sum(dim=1).max()) *
               float(bicubic64(t.shape[-1], grid[1], 'cpu').abs().sum(dim=1).max()) for t in stacks)
    vmax = max(float(t.abs().max()) for t in stacks)
    return max(1e-4, (n_keys + 1) * FP32_EPS), 32 * FP32_EPS * norm * vmax


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


# ---- raw daam_layer descriptors -------------------------------------------------------------------------------------
# ``daam_layer`` takes int64 element strides for the prompt, pixel / token and head axes (the head_dim axis is
# contiguous). The helpers below rebuild what a descriptor describes, bound what a kernel may make of it, and build
# descriptors over one storage buffer in the layouts callers hand the C ABI.

DTYPE_CODES = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}      # enum daam_dtype


def _strided_view(store: torch.Tensor, ptr: int, n_prompts: int, heads: int, rows: int, d: int, s_prompt: int,
                  s_row: int, s_head: int) -> torch.Tensor:
    """``[n_prompts, heads, rows, d]`` float64 of the elements a descriptor addresses from ``ptr`` (a device or host
    address inside the 1-D contiguous ``store``). Each sample is one ``as_strided`` view from the base pointer, so a zero
    prompt stride repeats a sample and a negative one walks the buffer backwards (``as_strided`` itself takes no
    negative stride)."""
    es = store.element_size()
    off, rem = divmod(ptr - store.data_ptr(), es)
    assert rem == 0 and store.dim() == 1 and store.is_contiguous(), 'the pointer is not an element of the storage'
    samples = []
    for p in range(n_prompts):
        base = off + p * s_prompt
        last = base + (heads - 1) * s_head + (rows - 1) * s_row + d - 1
        assert 0 <= base and last < store.numel(), f'sample {p} leaves the storage'
        samples.append(torch.as_strided(store, (heads, rows, d), (s_head, s_row, 1), base))
    return torch.stack(samples).double()


def layer_views64(desc, q_store: torch.Tensor, k_store: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """The Q ``[n_prompts, heads, hw, d]`` and K ``[n_prompts, heads, tokens, d]`` a ``_native.DaamLayer`` describes, in
    float64, read from the 1-D storage tensors its ``q`` / ``k`` pointers point into."""
    q = _strided_view(q_store, desc.q, desc.n_prompts, desc.heads, desc.hw, desc.head_dim, desc.q_stride_prompt,
                      desc.q_stride_pixel, desc.q_stride_head)
    k = _strided_view(k_store, desc.k, desc.n_prompts, desc.heads, desc.tokens, desc.head_dim, desc.k_stride_prompt,
                      desc.k_stride_token, desc.k_stride_head)
    return q, k


def _softmax_maps(q64: torch.Tensor, k64: torch.Tensor, scale: float) -> torch.Tensor:
    """``layer_maps64``'s arithmetic on head-split float64 views: ``[..., hw, d]``, ``[..., T, d]`` -> ``[..., T, hw]``."""
    s = (q64 @ k64.transpose(-1, -2)) * scale
    s = s - s.amax(dim=-1, keepdim=True)
    e = torch.exp(s)
    return (e / e.sum(dim=-1, keepdim=True)).transpose(-1, -2).contiguous()


def desc_maps64(desc, q_store: torch.Tensor, k_store: torch.Tensor) -> torch.Tensor:
    """What one ``daam_accumulate`` of ``desc`` adds to its accumulator, in float64: ``[n_prompts, heads, tokens, hw]``.
    The scale is the descriptor's fp32 value, as the kernels receive it."""
    q, k = layer_views64(desc, q_store, k_store)
    return _softmax_maps(q, k, float(desc.scale))


# Per-element error bound of the accumulate kernels. u = 2^-24 is the unit roundoff of fp32; "logit" is in nats.
FORMS = ('wgmma16', 'split', 'simt')


def _dot_gamma(form: str, d: int) -> float:
    """Bound of |computed - exact| / sum_i |q_i k_i| for one logit's dot product (see accumulate_tolerance)."""
    if form == 'simt':                      # d fma: products exact, d round-to-nearest adds
        return d * FP32_EPS / (1 - d * FP32_EPS)
    if form == 'wgmma16':                   # 16-bit products are exact in fp32; d truncating adds, one bit of slack
        return d * 2.0 ** -22
    if form == 'split':                     # 3d tf32 products (exact) + the dropped terms of x = hi + lo
        return (3 * d * 2.0 ** -22 + 2.0 ** -19) * (1 + 2.0 ** -9)
    raise ValueError(f'unknown form {form!r}')


def accumulate_tolerance(q64: torch.Tensor, k64: torch.Tensor, scale: float, form: str,
                         calls: int = 1) -> torch.Tensor:
    """Absolute bound, per element, of ``calls`` accumulate calls of one layer into a zeroed fp32 accumulator against
    ``calls`` times :func:`desc_maps64`, derived from the kernels' arithmetic rather than from observed errors.
    ``q64 [..., hw, d]``, ``k64 [..., T, d]``: the stored values in float64; ``scale`` the descriptor's fp32 scale;
    ``form``: ``'wgmma16'`` (16-bit wgmma, every context length), ``'split'`` (fp32 wgmma) or ``'simt'`` (SIMT, and the
    two-pass SIMT kernel when T > 77). Returns ``[..., T, hw]`` (the accumulator layout).

    1. Logit error of (pixel, token), ``scale * gamma * sum_i |q_i k_i|``:
       * SIMT: a chain of d fma, ``gamma_d = d u / (1 - d u)``;
       * 16-bit wgmma: the products are exact in fp32 and the order of the d adds is the tensor core's; each add may
         truncate and may lose one more bit to operand alignment, so ``gamma = d 2^-22``;
       * fp32 split form: ``x = hi + lo`` with ``hi = trunc_tf32(x)`` (``|x - hi| < 2^-10 |x|``) and ``lo`` the tf32
         rounding of ``x - hi`` (error ``<= 2^-21 |x|``). The dropped ``q_lo k_lo`` and the two ``lo`` roundings cost
         at most ``2^-19 |q_i k_i|``; the ``3d`` exact tf32 products are added as above, ``3 d 2^-22``; the terms
         sum to at most ``(1 + 2^-9) |q_i k_i|``.
    2. The exponent ``fma(s, c, -m c)`` with ``c = fl(scale * fl(log2 e))``: ``m c`` is rounded once and shared by the
       row, so it cancels; ``c`` (2 roundings) and the fma (1) put ``3 u |l_t - l_max|`` on the logit difference.
       ``4 u`` is used (the kernel's max is of the computed logits). The two-pass SIMT kernel of long contexts adds a
       row offset rounded per chunk (``m_c c``) and rescales its running sum by ``exp2(m c - m_c' c)``: ``3 u max|l|``.
    3. If every logit of a row errs by at most ``E``, every probability of the row by at most ``p (exp(2E) - 1)``.
       ex2.approx (2 ulp: ``4u``) of the numerator and of the sum's terms, the ``T``-term sum (``(T - 1) u``), the
       reciprocal (``2u``) and the product (``u``) add ``(T + 10) u`` relatively (the two-pass kernel: ``5u`` more per
       chunk for its rescale and fma).
    4. Flush-to-zero: an exponential, the probability and the accumulator add may each flush a value below 2^-126:
       ``2^-124`` absolute per call.
    5. ``calls`` fp32 adds of the probability into the accumulator: ``u * calls (calls + 1) / 2`` relatively."""
    p, per_call = _call_tolerance(q64, k64, scale, form)
    adds = FP32_EPS * calls * (calls + 1) / 2
    tol = calls * per_call + adds * calls * (p + per_call)
    return tol.transpose(-1, -2).contiguous()


def _call_tolerance(q64: torch.Tensor, k64: torch.Tensor, scale: float, form: str):
    """Steps 1-4 of :func:`accumulate_tolerance`: ``(p, bound)``, both ``[..., hw, T]``."""
    d, T = q64.shape[-1], k64.shape[-2]
    q64, k64 = q64.double(), k64.double()
    s = (q64 @ k64.transpose(-1, -2)) * scale                            # [..., hw, T]
    smax = s.amax(dim=-1, keepdim=True)
    e = torch.exp(s - smax)
    p = e / e.sum(dim=-1, keepdim=True)
    absdot = (q64.abs() @ k64.abs().transpose(-1, -2)) * scale
    err = _dot_gamma(form, d) * absdot + 4 * FP32_EPS * (s - smax).abs()
    eta = (T + 10) * FP32_EPS
    if form == 'simt' and T > 77:                                        # the two-pass kernel of long contexts
        err = err + 3 * FP32_EPS * s.abs().amax(dim=-1, keepdim=True)
        eta += 5 * FP32_EPS * (T // 77)
    big_e = err.amax(dim=-1, keepdim=True)
    return p, p * (torch.exp(2 * big_e) * (1 + eta) - 1) + 2.0 ** -124


def probs_tolerance(q64: torch.Tensor, k64: torch.Tensor, scale: float, dtype: torch.dtype) -> torch.Tensor:
    """Bound of ``daam_attention_probs`` (the SIMT arithmetic, then one rounding to ``dtype``) against the float64
    softmax, as :func:`accumulate_tolerance` lays it out (``[..., T, hw]``): half an ulp of the dtype relatively, and
    half its smallest subnormal absolutely."""
    p, tol = _call_tolerance(q64, k64, scale, 'simt')
    if dtype != torch.float32:
        mant, tiny = {torch.float16: (11, 2.0 ** -24), torch.bfloat16: (8, 2.0 ** -133)}[dtype]
        tol = tol + (p + tol) * 2.0 ** -mant + tiny / 2
    return tol.transpose(-1, -2).contiguous()


# ---- layouts --------------------------------------------------------------------------------------------------------
# Every layout holds the samples the descriptor reads inside one storage buffer whose other elements are NaN, so a
# kernel that reads outside the described view produces NaN.
LAYOUTS = ('canonical', 'padded_heads', 'head_major', 'fused_qkv', 'sample_padding', 'q_broadcast', 'k_broadcast',
           'negative_prompt_stride', 'lone_sample_5_heads')


def layout_shape(name: str, n_prompts: int = 2, heads: int = 2) -> Tuple[int, int]:
    """``(n_prompts, heads)`` the descriptor of layout ``name`` covers: a lone sample with 5 heads keeps the upper 3
    (``ops.cond_half``)."""
    return (1, 3) if name == 'lone_sample_5_heads' else (n_prompts, heads)


def mma_accepts_strides(desc) -> bool:
    """The stride rule of the wgmma path (include/daam_b200.h, DAAM_ACC_AUTO): positive head and row strides, and
    positive prompt strides when the layer has more than one prompt."""
    return (desc.q_stride_head > 0 and desc.q_stride_pixel > 0 and desc.k_stride_head > 0 and desc.k_stride_token > 0
            and (desc.n_prompts == 1 or (desc.q_stride_prompt > 0 and desc.k_stride_prompt > 0)))


def _place(name: str, x: torch.Tensor, fused: int) -> Tuple[torch.Tensor, int, Tuple[int, int, int], torch.Tensor]:
    """One operand ``x [P, H, rows, d]`` in layout ``name``: ``(store, element offset of sample 0 / head 0,
    (s_prompt, s_row, s_head), effective x)``. ``fused``: the channel multiple of the fused projection buffer (3 for
    ``qkv``, 2 for ``kv``). The effective x is what the descriptor reads (sample 0 repeated for a broadcast)."""
    P, H, rows, d = x.shape
    nan = lambda n: torch.full((n,), float('nan'), dtype=x.dtype, device=x.device)
    cl = x.permute(0, 2, 1, 3)                                           # [P, rows, H, d]: to_q / to_k order
    C = H * d
    if name == 'canonical':                                              # a CFG batch: the conditional half
        store = nan(2 * P * rows * C)
        store[P * rows * C:] = cl.reshape(-1)
        return store, P * rows * C, (rows * C, C, d), x
    if name == 'padded_heads':
        dp = d + 8
        store = nan(P * rows * H * dp)
        store.view(P, rows, H, dp)[..., :d] = cl
        return store, 0, (rows * H * dp, H * dp, dp), x
    if name == 'head_major':                                             # SDPA's [B, H, N, d]
        store = x.contiguous().reshape(-1).clone()
        return store, 0, (H * rows * d, d, rows * d), x
    if name == 'fused':
        store = nan(P * rows * fused * C)
        store.view(P, rows, fused * C)[..., :C] = cl.reshape(P, rows, C)
        return store, 0, (rows * fused * C, fused * C, d), x
    if name == 'sample_padding':
        sp = rows * C + 64
        store = nan(P * sp + 64)
        for p in range(P):
            store[64 + p * sp: 64 + p * sp + rows * C] = cl[p].reshape(-1)
        return store, 64, (sp, C, d), x
    if name == 'broadcast':                                              # x.expand(P, ...): prompt stride 0
        store = cl[0].reshape(-1).clone()
        return store, 0, (0, C, d), x[:1].expand_as(x)
    if name == 'negative':                                               # sample p stored at P - 1 - p
        store = cl.flip(0).reshape(-1).clone()
        return store, (P - 1) * rows * C, (-rows * C, C, d), x
    if name == 'lone':                                                   # a lone sample of 5 heads, the upper 3 kept
        store = nan(rows * 5 * d)
        store.view(rows, 5, d)[:, 5 - H:] = cl[0]
        return store, (5 - H) * d, (rows * 5 * d, 5 * d, d), x
    raise ValueError(name)


def build_layout(name: str, q: torch.Tensor, k: torch.Tensor, scale: float, acc_ptr: Optional[int] = None):
    """A ``_native.DaamLayer`` in layout ``name`` (one of :data:`LAYOUTS`) over fresh storage buffers holding
    ``q [P, H, hw, d]`` and ``k [P, H, T, d]`` (one dtype, one device; ``P, H`` from :func:`layout_shape`).
    Returns ``(desc, q_store, k_store, q_eff, k_eff)``: the 1-D storages and what the descriptor reads."""
    from daam_b200 import _native
    qname, kname = {'canonical': ('canonical', 'canonical'), 'padded_heads': ('padded_heads', 'padded_heads'),
                    'head_major': ('head_major', 'head_major'), 'fused_qkv': ('fused', 'fused'),
                    'sample_padding': ('sample_padding', 'sample_padding'), 'q_broadcast': ('broadcast', 'canonical'),
                    'k_broadcast': ('canonical', 'broadcast'),
                    'negative_prompt_stride': ('negative', 'negative'), 'lone_sample_5_heads': ('lone', 'lone')}[name]
    qs, qo, (qsp, qsr, qsh), q_eff = _place(qname, q, 3)
    ks, ko, (ksp, ksr, ksh), k_eff = _place(kname, k, 2)
    es = q.element_size()
    P, H, hw, d = q.shape
    desc = _native.DaamLayer(
        q=qs.data_ptr() + qo * es, k=ks.data_ptr() + ko * es, acc=acc_ptr,
        q_stride_prompt=qsp, q_stride_pixel=qsr, q_stride_head=qsh,
        k_stride_prompt=ksp, k_stride_token=ksr, k_stride_head=ksh,
        n_prompts=P, heads=H, hw=hw, tokens=k.shape[2], head_dim=d, dtype=DTYPE_CODES[q.dtype], scale=float(scale),
        reserved=0)
    return desc, qs, ks, q_eff, k_eff


# ---- logit regimes --------------------------------------------------------------------------------------------------
REGIMES = ('gaussian', 'uniform', 'one_hot', 'all_negative', 'positive_offset', 'sinks', 'duplicate_k')
KEY_TILE = 128                                       # pixel rows of one accumulate tile


def one_hot_columns(T: int) -> Tuple[int, ...]:
    """The argmax columns the one-hot regime sweeps: the first and last column of every 77-token chunk, the first
    columns of the next one, and the last column of the context."""
    cols = {0, 1, 76, T - 1}
    for c in range(1, T // 77):
        cols |= {77 * c - 1, 77 * c, 77 * c + 1}
    return tuple(sorted(cols))


def duplicate_rows(T: int) -> Sequence[Tuple[int, ...]]:
    """Sets of K rows the duplicate_k regime makes equal: a tail of 24 padding tokens, and for long contexts the rows
    on both sides of every chunk boundary."""
    sets = [tuple(range(T - 25, T))]
    sets += [(77 * c - 1, 77 * c) for c in range(1, T // 77)]
    return sets


def make_regime(regime: str, P: int, H: int, hw: int, d: int, T: int, scale: float, dtype: torch.dtype,
                seed: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """``q [P, H, hw, d]``, ``k [P, H, T, d]`` in ``dtype`` (on the CPU) whose logits ``scale * q . k`` follow
    ``regime``:

    * gaussian: iid N(0, 1) K, N(0, 1.5^2) Q;
    * uniform: Q = 0, every probability is 1/T;
    * one_hot: unit K rows, ``q_i = beta k_t(i)`` with beta chosen so that t(i) leads every other column by at least
      40 nats; t(i) runs through :func:`one_hot_columns` so that each column meets every row of the 128-pixel tile
      once the map has as many tiles as there are columns;
    * all_negative: every logit near -150 nats (noise of 1 nat): a zero padding column in the row max would flush every
      exponential and give NaN;
    * positive_offset: every logit near +200 nats;
    * sinks: tokens 77c .. 77c + 2 lead by 8 nats and carry most of the mass, as BOS does in every CLIP chunk;
    * duplicate_k: gaussian with the K rows of :func:`duplicate_rows` equal."""
    g = torch.Generator().manual_seed(seed)
    randn = lambda *shape: torch.randn(*shape, generator=g, dtype=torch.float64)
    if regime in ('gaussian', 'duplicate_k', 'uniform'):
        q, k = randn(P, H, hw, d) * 1.5, randn(P, H, T, d)
        if regime == 'uniform':
            q.zero_()
        if regime == 'duplicate_k':
            for rows in duplicate_rows(T):
                k[:, :, list(rows)] = k[:, :, rows[0]:rows[0] + 1].clone()
        return q.to(dtype), k.to(dtype)
    if regime == 'one_hot':
        k = randn(P, H, T, d)
        k = (k / k.norm(dim=-1, keepdim=True)).to(dtype).double()
        cols = one_hot_columns(T)
        i = torch.arange(hw)
        t_of = torch.tensor(cols)[(i // KEY_TILE + i % KEY_TILE) % len(cols)]
        gram = k @ k.transpose(-1, -2)
        cross = (gram - torch.diag_embed(torch.full((T,), float('inf'), dtype=torch.float64))).amax(dim=-1)
        lead = (gram.diagonal(dim1=-2, dim2=-1) - cross).amin()          # >= 1 - max cos of two K rows
        beta = 60.0 / (scale * float(lead))
        q = beta * k[:, :, t_of]
        return q.to(dtype), k.to(dtype)
    # offset regimes: dimension 0 carries the offset, the others noise of one nat (std of the noise logit)
    noise = (scale * math.sqrt(d)) ** -0.5
    q, k = randn(P, H, hw, d) * noise, randn(P, H, T, d) * noise
    if regime == 'sinks':
        amp = math.sqrt(8.0 / scale)
        q[..., 0] = amp
        k[..., 0] = 0.0
        for c in range(T // 77):
            k[:, :, 77 * c:77 * c + 3, 0] = amp
    else:
        target = -150.0 if regime == 'all_negative' else 200.0
        amp = math.sqrt(abs(target) / scale)
        q[..., 0] = math.copysign(amp, target)
        k[..., 0] = amp
    return q.to(dtype), k.to(dtype)
