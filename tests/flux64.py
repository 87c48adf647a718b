"""float64 restatement of the FLUX.1 heat map: the joint softmax of a ``[text, image]`` sequence, of which the
image-query x text-key block is kept for every sample and head, summed over the traced calls, averaged over the
(sample, head) keys of a prompt; a read's row 0 is zeros and row ``r >= 1`` is context row ``r - 1`` (factor 1: the
bicubic upsample is the identity and every value is already >= 0). Also the per-element bound of the kernel's
arithmetic as ``include/daam_b200.h`` states it."""
import torch

from tests.joint64 import exp_and_bound


def flux_block(q: torch.Tensor, k: torch.Tensor, tokens: int, scale: float) -> torch.Tensor:
    """``q`` / ``k`` ``[B, heads, T + n_image, d]`` (text tokens first): the float64 joint softmax of every image
    query over every key, text-key columns: ``[B, heads, T, n_image]`` (token-major, like a slab)."""
    q, k = q.double(), k.double()
    s = torch.einsum('bhid,bhjd->bhij', q[:, :, tokens:], k) * scale
    return torch.softmax(s, dim=-1)[..., :tokens].transpose(-1, -2).contiguous()


def image_mass(q: torch.Tensor, k: torch.Tensor, tokens: int, scale: float) -> torch.Tensor:
    """``[B, heads, n_image]``: the softmax mass of every image query on the image keys (the part a map drops)."""
    q, k = q.double(), k.double()
    s = torch.einsum('bhid,bhjd->bhij', q[:, :, tokens:], k) * scale
    return torch.softmax(s, dim=-1)[..., tokens:].sum(-1)


def flux_maps(calls, tokens: int, grid, heads: int):
    """The per-layer sums of a traced generation: ``calls`` is a list of ``(layer, q, k, ...)`` over the whole batch.
    Returns ``{layer: [B, heads, T, h, w]}`` in float64."""
    out = {}
    for layer, q, k, *_ in calls:
        block = flux_block(q, k, tokens, q.shape[-1] ** -0.5)
        block = block.view(block.shape[0], heads, tokens, *grid)
        out[layer] = block if layer not in out else out[layer] + block
    return out


def global_rows(per_layer, n: int, prompt: int = 0, images: int = 1, normalize: bool = False):
    """The T5 map of ``prompt`` over ``per_layer`` (``flux_maps``' result): the mean over every layer's keys, rows
    ``[0, n + 2)`` with row 0 zeros and row ``r`` context row ``r - 1``; with ``normalize`` divided by rows
    ``1 .. n`` plus 1e-6 (row 0 zeroed afterwards, as the read does)."""
    keys = [m[prompt * images:(prompt + 1) * images].flatten(0, 1) for m in per_layer.values()]
    mean = torch.cat(keys).mean(0)
    maps = torch.cat([torch.zeros_like(mean[:1]), mean[:n + 1]])
    if normalize:
        maps = maps / (maps[1:-1].sum(0, keepdim=True) + 1e-6)
        maps[0] = 0
    return maps


def reference_and_bound(q, k, lse, tokens: int, scale: float):
    """:func:`tests.joint64.exp_and_bound` of text-first operands ``[B, heads, T + hw, d]`` over every sample:
    ``[B, heads, T, hw]`` and its bound."""
    hw = q.shape[2] - tokens
    return exp_and_bound(q[:, :, tokens:], k[:, :, :tokens], lse[:, :, tokens:tokens + hw], scale)


def rope64(x: torch.Tensor, ids: torch.Tensor, axes_dim, theta: float = 10000.0) -> torch.Tensor:
    """RoPE restated as complex multiplication, independently of the interleaving code under test: the head dim of
    ``x`` ``[B, heads, L, d]`` is ``d / 2`` complex numbers ``x[2j] + i x[2j + 1]``, axis ``a`` of the position ids
    ``[L, 3]`` owns ``axes_dim[a] / 2`` of them, and number ``j`` of axis ``a`` turns by
    ``ids[:, a] * theta ** (-2j / axes_dim[a])`` radians."""
    angles = torch.cat([ids[:, a, None].double() * theta ** (-torch.arange(0, dim, 2, dtype=torch.float64,
                                                                           device=ids.device) / dim)
                        for a, dim in enumerate(axes_dim)], dim=-1)                  # [L, d / 2]
    xc = torch.view_as_complex(x.double().reshape(*x.shape[:-1], -1, 2).contiguous())
    return torch.view_as_real(xc * torch.polar(torch.ones_like(angles), angles)).flatten(-2)


def attention64(attn, hidden, context, ids, axes_dim, tokens: int = 0):
    """A FLUX attention restated in float64 from its module weights: ``hidden`` ``[B, hw, C]`` the image stream,
    ``context`` ``[B, T, C]`` the text stream (a double-stream block), or ``None`` with ``hidden`` the joined
    ``[text, image]`` sequence (a single-stream block, whose first ``tokens`` rows are the text). Text comes first in
    the sequence, RMS norms per head, RoPE by :func:`rope64`. Returns the outputs (image and text for a double block,
    the joined sequence for a single one) and the softmax block of image queries x text keys, ``[B, heads, T, hw]``."""
    def lin(m, t):
        return t.double() @ m.weight.double().T + m.bias.double()

    def rms(m, t):
        return t * torch.rsqrt(t.pow(2).mean(-1, keepdim=True) + m.eps) * m.weight.double()

    heads = attn.heads
    b = hidden.shape[0]
    split = lambda t: t.view(b, -1, heads, t.shape[-1] // heads).transpose(1, 2)
    q, k, v = split(lin(attn.to_q, hidden)), split(lin(attn.to_k, hidden)), split(lin(attn.to_v, hidden))
    q, k = rms(attn.norm_q, q), rms(attn.norm_k, k)
    if context is not None:
        tokens = context.shape[1]
        cq, ck, cv = split(lin(attn.add_q_proj, context)), split(lin(attn.add_k_proj, context)), \
            split(lin(attn.add_v_proj, context))
        q, k, v = (torch.cat([rms(attn.norm_added_q, cq), q], 2), torch.cat([rms(attn.norm_added_k, ck), k], 2),
                   torch.cat([cv, v], 2))
    q, k = rope64(q, ids, axes_dim), rope64(k, ids, axes_dim)
    p = torch.softmax(q @ k.transpose(-1, -2) / q.shape[-1] ** 0.5, dim=-1)
    out = (p @ v).transpose(1, 2).reshape(b, -1, heads * q.shape[-1])
    block = p[:, :, tokens:, :tokens].transpose(-1, -2)
    if context is None:
        return out, block
    return (lin(attn.to_out[0], out[:, tokens:]), lin(attn.to_add_out, out[:, :tokens])), block
