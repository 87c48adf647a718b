"""Tensor-level entry points over the C ABI: build ``daam_layer`` descriptors from torch tensors and launch.

This is the thinnest layer above ``libdaam_b200.so``: no state, no policy. ``trace.py`` uses it from the attention
hook; the parity tests and ``bench.py`` call it directly with Q/K tensors.
"""
from __future__ import annotations

from typing import Optional, Sequence, Tuple

import torch

from . import _native

__all__ = ['cond_half', 'make_layer_desc', 'new_accumulator', 'pack', 'accumulate', 'accumulate_steps',
           'accumulate_range', 'accumulate_layer', 'attention_probs', 'accumulate_probs', 'value_norms',
           'make_joint_desc', 'accumulate_joint', 'accumulate_joint_heads']

_DTYPES = {torch.float32: _native.DAAM_F32, torch.float16: _native.DAAM_F16, torch.bfloat16: _native.DAAM_BF16}


def cond_half(bsz: int, heads: int) -> Tuple[int, int, int, int]:
    """Which slice of the ``batch x heads`` axis the reference keeps (``map_[map_.size(0) // 2:]``, daam/trace.py:240).

    Returns ``(first_sample, n_prompts, first_head, n_heads)``: for a CFG batch ``[uncond x N, cond x N]`` the N
    conditional samples with all heads; for a lone sample (no guidance) the upper half of its heads -- the reference's
    behaviour, kept faithfully. Other odd batch sizes cut through a sample and are rejected.
    """
    if bsz % 2 == 0:
        return bsz // 2, bsz // 2, 0, heads
    if bsz == 1:
        return 0, 1, heads // 2, heads - heads // 2
    raise RuntimeError(f'a batch of {bsz} is neither a CFG pair batch nor a single sample')


def new_accumulator(n_prompts: int, heads: int, hw: int, device, tokens: int = _native.TOKENS) -> torch.Tensor:
    return torch.zeros((n_prompts, heads, tokens, hw), dtype=torch.float32, device=device)


def make_layer_desc(q: torch.Tensor, k: torch.Tensor, acc: torch.Tensor, heads: int, scale: float, *,
                    whole_batch: bool = False) -> _native.DaamLayer:
    """``q [B, hw, heads*d]`` / ``k [B, T, heads*d]`` as ``to_q`` / ``to_k`` emit them (last axis contiguous) and the
    fp32 accumulator ``[n_prompts, n_heads, T, hw]`` of the kept slice -> one ``daam_layer``. ``T`` is the context
    length: 77, or 154 / 231 for a long context (``_native.CONTEXT_TOKENS``). ``whole_batch``: the descriptor covers
    every sample from sample 0 -- both halves of a CFG batch, the unconditional one first -- and ``acc`` is
    ``[B, heads, T, hw]``."""
    if not (q.is_cuda and k.is_cuda and acc.is_cuda):
        raise RuntimeError('daam_b200 computes on CUDA tensors only (there is no CPU fallback)')
    if q.dtype not in _DTYPES or k.dtype != q.dtype:
        raise RuntimeError(f'unsupported projection dtypes {q.dtype}/{k.dtype}')
    if q.stride(-1) != 1 or k.stride(-1) != 1:
        raise RuntimeError('the channel axis of q and k must be contiguous')
    bsz, hw, chan = q.shape
    d = chan // heads
    first, n_prompts, head0, n_heads = (0, bsz, 0, heads) if whole_batch else cond_half(bsz, heads)
    tokens = k.shape[1] if k.shape[1] in _native.CONTEXT_TOKENS else _native.TOKENS
    if tuple(acc.shape) != (n_prompts, n_heads, tokens, hw) or acc.dtype != torch.float32 \
            or not acc.is_contiguous():
        raise RuntimeError(f'accumulator must be contiguous fp32 {(n_prompts, n_heads, tokens, hw)}, '
                           f'got {acc.dtype} {tuple(acc.shape)}')
    es = q.element_size()
    return _native.DaamLayer(
        q=q.data_ptr() + (first * q.stride(0) + head0 * d) * es,
        k=k.data_ptr() + (first * k.stride(0) + head0 * d) * es,
        acc=acc.data_ptr(),
        q_stride_prompt=q.stride(0), q_stride_pixel=q.stride(1), q_stride_head=d,
        k_stride_prompt=k.stride(0), k_stride_token=k.stride(1), k_stride_head=d,
        n_prompts=n_prompts, heads=n_heads, hw=hw, tokens=k.shape[1], head_dim=d,
        dtype=_DTYPES[q.dtype], scale=float(scale), reserved=0)


def pack(descs: Sequence[_native.DaamLayer]) -> _native.PackedLayers:
    """Pre-build the host-side ``daam_layer[]`` once for layer calls that are replayed (bench loops, CUDA graphs)."""
    return _native.PackedLayers(list(descs))


def _run_on(device, stream: Optional[torch.cuda.Stream], launch):
    """``launch(stream_ptr)`` with ``device`` current, on ``stream`` (default: the current stream of ``device``)."""
    dev = device if isinstance(device, torch.device) else torch.device(device)
    index = dev.index if dev.index is not None else torch.cuda.current_device()
    s = torch.cuda.current_stream(index) if stream is None else stream
    if index == torch.cuda.current_device():
        launch(s.cuda_stream)
    else:
        with torch.cuda.device(index):
            launch(s.cuda_stream)


def accumulate(descs, device, stream: Optional[torch.cuda.Stream] = None, flags: int = _native.ACC_AUTO):
    """Enqueue the fused kernel over the given layer calls (sequence of descriptors or :func:`pack` result) on
    ``stream`` (default: the current stream of ``device``)."""
    _run_on(device, stream, lambda s: _native.accumulate(descs, s, flags))


def _accumulate_second(native_fn, word: str, descs, slabs, device, stream, flags: int):
    """``native_fn`` (:func:`_native.accumulate_steps` / :func:`_native.accumulate_range`) over ``descs`` and one second
    slab per descriptor; ``word`` names the slabs in messages."""
    if not isinstance(slabs, _native.StepPointers):
        for t in slabs:
            if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
                raise RuntimeError(f'{word} slabs must be contiguous fp32 CUDA tensors')
        slabs = _native.StepPointers([t.data_ptr() for t in slabs])
    _run_on(device, stream, lambda s: native_fn(descs, slabs, s, flags))


def accumulate_steps(descs, steps, device, stream: Optional[torch.cuda.Stream] = None, flags: int = _native.ACC_AUTO):
    """:func:`accumulate`, and also store what each layer adds into its step slab (``daam_accumulate_steps``).
    ``steps``: one contiguous fp32 tensor per descriptor, shaped like its accumulator, or a prepared
    :class:`_native.StepPointers`."""
    _accumulate_second(_native.accumulate_steps, 'step', descs, steps, device, stream, flags)


def accumulate_range(descs, ranges, device, stream: Optional[torch.cuda.Stream] = None, flags: int = _native.ACC_AUTO):
    """:func:`accumulate`, and also add what each layer adds into its range slab, with the accumulator's arithmetic
    (``daam_accumulate_range``). ``ranges``: one contiguous fp32 tensor per descriptor, shaped like its accumulator, or
    a prepared :class:`_native.StepPointers`."""
    _accumulate_second(_native.accumulate_range, 'range', descs, ranges, device, stream, flags)


def accumulate_layer(q: torch.Tensor, k: torch.Tensor, heads: int, scale: Optional[float] = None,
                     acc: Optional[torch.Tensor] = None, flags: int = _native.ACC_AUTO) -> torch.Tensor:
    """One layer call on the current stream; allocates the accumulator when none is given. Returns it."""
    bsz, hw, chan = q.shape
    _, n_prompts, _, n_heads = cond_half(bsz, heads)
    if acc is None:
        acc = new_accumulator(n_prompts, n_heads, hw, q.device,
                              k.shape[1] if k.shape[1] in _native.CONTEXT_TOKENS else _native.TOKENS)
    if scale is None:
        scale = (chan // heads) ** -0.5
    accumulate([make_layer_desc(q, k, acc, heads, scale)], q.device, flags=flags)
    return acc


def attention_probs(q: torch.Tensor, k: torch.Tensor, heads: int, scale: Optional[float] = None) -> torch.Tensor:
    """Materialised ``softmax(scale * Q K^T)`` for EVERY sample: ``[B*heads, hw, 77]`` in the dtype of ``q`` -- what
    diffusers' ``get_attention_scores`` returns at daam/trace.py:276 (rows ordered ``b*heads + head``). Compatibility
    path for ``save_heads``; the traced hot path never materialises this tensor."""
    if not (q.is_cuda and k.is_cuda):
        raise RuntimeError('daam_b200 computes on CUDA tensors only (there is no CPU fallback)')
    if q.dtype not in _DTYPES or k.dtype != q.dtype:
        raise RuntimeError(f'unsupported projection dtypes {q.dtype}/{k.dtype}')
    if q.stride(-1) != 1 or k.stride(-1) != 1:
        q, k = q.contiguous(), k.contiguous()
    bsz, hw, chan = q.shape
    d = chan // heads
    if scale is None:
        scale = d ** -0.5
    probs = torch.empty((bsz * heads, hw, k.shape[1]), dtype=q.dtype, device=q.device)
    desc = _native.DaamLayer(
        q=q.data_ptr(), k=k.data_ptr(), acc=None,
        q_stride_prompt=q.stride(0), q_stride_pixel=q.stride(1), q_stride_head=d,
        k_stride_prompt=k.stride(0), k_stride_token=k.stride(1), k_stride_head=d,
        n_prompts=bsz, heads=heads, hw=hw, tokens=k.shape[1], head_dim=d,
        dtype=_DTYPES[q.dtype], scale=float(scale), reserved=0)
    with torch.cuda.device(q.device):
        _native.attention_probs(desc, probs.data_ptr(), torch.cuda.current_stream(q.device).cuda_stream)
    return probs


def accumulate_probs(probs: torch.Tensor, acc: torch.Tensor, *, whole_batch: bool = False):
    """``acc[r][t][pixel] += probs[first + r][pixel][t]`` with ``first = rows // 2``: the reference's "second half of
    the batch*heads axis" (daam/trace.py:240) applied to supplied probabilities (``load_heads``, trace.py:281-294).
    ``acc``: fp32 ``[n_prompts, n_heads, 77, hw]`` (its leading two axes flatten to the kept rows). ``whole_batch``:
    ``first = 0``, every row is kept (both halves of a CFG batch)."""
    if not (probs.is_cuda and acc.is_cuda):
        raise RuntimeError('daam_b200 computes on CUDA tensors only (there is no CPU fallback)')
    probs = probs.contiguous()
    rows, hw, tokens = probs.shape
    first = 0 if whole_batch else rows // 2
    kept = rows - first
    if acc.dtype != torch.float32 or not acc.is_contiguous() or acc.numel() != kept * tokens * hw:
        raise RuntimeError(f'accumulator must be contiguous fp32 with {kept} x {tokens} x {hw} elements')
    with torch.cuda.device(probs.device):
        _native.accumulate_probs(probs.data_ptr(), _DTYPES[probs.dtype], first, kept, hw, tokens, acc.data_ptr(),
                                 torch.cuda.current_stream(probs.device).cuda_stream)


def value_norms(value: torch.Tensor, weight: torch.Tensor, heads: int, out: Optional[torch.Tensor] = None, *,
                whole_batch: bool = False) -> torch.Tensor:
    """``||W_h v||`` for every kept (sample, head, context row) (``daam_value_norms``): ``value [B, T, heads*d]`` as
    ``to_v`` emits it (last axis contiguous), ``weight [C_out, heads*d]`` the output projection's. The kept slice is
    :func:`make_layer_desc`'s: the conditional half of a CFG batch (a lone sample: the upper half of its heads), or with
    ``whole_batch`` every sample. Returns (or fills ``out``) fp32 ``[n_samples, n_heads, T]``, contiguous."""
    if not (value.is_cuda and weight.is_cuda):
        raise RuntimeError('daam_b200 computes on CUDA tensors only (there is no CPU fallback)')
    if value.dtype not in _DTYPES or weight.dtype not in _DTYPES:
        raise RuntimeError(f'unsupported value / weight dtypes {value.dtype}/{weight.dtype}')
    if value.stride(-1) != 1:
        value = value.contiguous()
    if weight.stride(-1) != 1:
        weight = weight.contiguous()
    bsz, tokens, chan = value.shape
    d = chan // heads
    if weight.dim() != 2 or weight.shape[1] != chan:
        raise RuntimeError(f'output projection weight {tuple(weight.shape)} does not take {chan} channels')
    first, n_samples, head0, n_heads = (0, bsz, 0, heads) if whole_batch else cond_half(bsz, heads)
    shape = (n_samples, n_heads, tokens)
    if out is None:
        out = torch.empty(shape, dtype=torch.float32, device=value.device)
    elif tuple(out.shape) != shape or out.dtype != torch.float32 or not out.is_contiguous():
        raise RuntimeError(f'value norms must be contiguous fp32 {shape}, got {out.dtype} {tuple(out.shape)}')
    ve, we = value.element_size(), weight.element_size()
    _run_on(value.device, None, lambda s: _native.value_norms(
        value.data_ptr() + (first * value.stride(0) + head0 * d) * ve, _DTYPES[value.dtype],
        (value.stride(0), value.stride(1), d), weight.data_ptr() + head0 * d * we, _DTYPES[weight.dtype],
        weight.stride(0), n_samples, n_heads, tokens, d, weight.shape[0], out.data_ptr(), s))
    return out


def make_joint_desc(q: torch.Tensor, k: torch.Tensor, lse: torch.Tensor, n_image: int, acc: torch.Tensor, heads: int,
                    scale: float, *, text_first: bool = False, whole_batch: bool = False,
                    reduce_heads: bool = False) -> _native.DaamJointLayer:
    """One ``daam_joint_layer`` from a joint attention's operands as SDPA takes them: ``q`` / ``k`` ``[B, heads, L, d]``
    (any strides, ``d`` contiguous; e.g. the concatenation ``[image, context]`` of diffusers' ``JointAttnProcessor2_0``,
    or a ``[B, L, heads*d]`` projection viewed that way), ``lse`` fp32 ``[B, heads, >= n_image]`` (text-first: ``>= L``) the attention's
    log-sum-exp (natural log), ``n_image`` the image tokens ahead of the context in ``L``. The kept samples are
    :func:`cond_half`'s; ``acc`` fp32 ``[n_prompts, n_heads, L - n_image, n_image]`` contiguous.

    ``text_first``: ``L`` is ``[context, image]`` (FLUX): the image queries and their lse start at row
    ``T = L - n_image`` and the context keys at row 0. ``whole_batch``: every sample with every head is kept
    (a batch without a CFG half), and ``acc`` is ``[B, heads, T, n_image]``. ``reduce_heads``: the descriptor of
    :func:`accumulate_joint_heads`, whose ``acc`` has no head axis: ``[n_prompts, T, n_image]`` contiguous fp32."""
    if not (q.is_cuda and k.is_cuda and lse.is_cuda and acc.is_cuda):
        raise RuntimeError('daam_b200 computes on CUDA tensors only (there is no CPU fallback)')
    if q.dtype not in _DTYPES or k.dtype != q.dtype:
        raise RuntimeError(f'unsupported projection dtypes {q.dtype}/{k.dtype}')
    if lse.dtype != torch.float32 or lse.dim() != 3:
        raise RuntimeError(f'lse must be fp32 [B, heads, L], got {lse.dtype} {tuple(lse.shape)}')
    if q.dim() != 4 or k.dim() != 4 or q.stride(-1) != 1 or k.stride(-1) != 1:
        raise RuntimeError('q and k must be [B, heads, L, d] with a contiguous d axis')
    bsz, _, seq, d = q.shape
    if k.shape[0] != bsz or lse.shape[0] != bsz:
        raise RuntimeError(f'q, k and lse must have one batch size, got {bsz}, {k.shape[0]} and {lse.shape[0]}')
    if min(q.shape[1], k.shape[1], lse.shape[1]) < heads:
        raise RuntimeError(f'q, k and lse must have at least {heads} heads, got {q.shape[1]}, {k.shape[1]} and '
                           f'{lse.shape[1]}')
    if k.shape[2] != seq or k.shape[3] != d:
        raise RuntimeError(f'q and k must have one sequence length and head dim, got {tuple(q.shape[2:])} and '
                           f'{tuple(k.shape[2:])}')
    if not 0 < n_image < seq:
        raise RuntimeError(f'n_image = {n_image} must leave image and context tokens in a sequence of {seq}')
    lse_rows = seq if text_first else n_image
    if lse.shape[2] < lse_rows:
        raise RuntimeError(f'lse has {lse.shape[2]} rows, the kernel reads {lse_rows}')
    tokens = seq - n_image
    first, n_prompts, head0, n_heads = (0, bsz, 0, heads) if whole_batch else cond_half(bsz, heads)
    shape = (n_prompts, tokens, n_image) if reduce_heads else (n_prompts, n_heads, tokens, n_image)
    if tuple(acc.shape) != shape or acc.dtype != torch.float32 or not acc.is_contiguous():
        raise RuntimeError(f'accumulator must be contiguous fp32 {shape}, got {acc.dtype} {tuple(acc.shape)}')
    q_row, k_row = (tokens, 0) if text_first else (0, n_image)   # first image query, first context key
    es = q.element_size()
    return _native.DaamJointLayer(
        q=q.data_ptr() + (first * q.stride(0) + head0 * q.stride(1) + q_row * q.stride(2)) * es,
        k=k.data_ptr() + (first * k.stride(0) + head0 * k.stride(1) + k_row * k.stride(2)) * es,
        acc=acc.data_ptr(),
        q_stride_prompt=q.stride(0), q_stride_pixel=q.stride(2), q_stride_head=q.stride(1),
        k_stride_prompt=k.stride(0), k_stride_token=k.stride(2), k_stride_head=k.stride(1),
        n_prompts=n_prompts, heads=n_heads, hw=n_image, tokens=tokens, head_dim=d,
        dtype=_DTYPES[q.dtype], scale=float(scale), reserved=0,
        lse=lse.data_ptr() + (first * lse.stride(0) + head0 * lse.stride(1) + q_row * lse.stride(2)) * 4,
        lse_stride_prompt=lse.stride(0), lse_stride_head=lse.stride(1), lse_stride_pixel=lse.stride(2))


def accumulate_joint(descs, device, stream: Optional[torch.cuda.Stream] = None):
    """Enqueue ``daam_accumulate_joint`` over the given joint layer descriptors on ``stream`` (default: the current
    stream of ``device``)."""
    _run_on(device, stream, lambda s: _native.accumulate_joint(list(descs), s))


def accumulate_joint_heads(descs, device, stream: Optional[torch.cuda.Stream] = None):
    """Enqueue ``daam_accumulate_joint_heads`` over descriptors made with ``make_joint_desc(..., reduce_heads=True)``:
    every sample's head mean of the joint heat map, added into its head-free accumulator."""
    _run_on(device, stream, lambda s: _native.accumulate_joint_heads(list(descs), s))
