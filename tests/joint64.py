"""float64 restatement of the joint-attention heat map (MM-DiT, Stable Diffusion 3): one softmax over every image and
context key, of which the image-query x context-key block is kept, summed over the traced calls, averaged over the
(sample, head) keys of a prompt; the rows of a read are then taken from that mean (factor 1: the bicubic upsample is
the identity and every value is already >= 0). Also the per-element bound of daam_accumulate_joint's arithmetic as
``include/daam_b200.h`` states it."""
import torch

LOG2E = 1.4426950408889634


def exp_and_bound(q: torch.Tensor, k: torch.Tensor, lse: torch.Tensor, scale: float):
    """``q`` ``[N, heads, hw, d]`` the kept image queries, ``k`` ``[N, heads, T, d]`` the kept context keys, ``lse``
    ``[N, heads, hw]`` fp32: the float64 ``exp(scale32 <q, k> - lse32)``, ``[N, heads, T, hw]``, and the per-element
    bound of the header's arithmetic: the dot product within d 2^-23 sum|q k|, the three fp32 roundings of the
    exponent, and ex2.approx within 2^-22."""
    qd, kd = q.double(), k.double()
    d = q.shape[-1]
    scale32 = float(torch.tensor(scale, dtype=torch.float32))
    dot = torch.einsum('bhid,bhjd->bhji', qd, kd)
    absdot = torch.einsum('bhid,bhjd->bhji', qd.abs(), kd.abs())
    l = lse.double()[:, :, None, :]
    x = dot * scale32 * LOG2E - l * LOG2E
    ref = torch.exp2(x)
    err_x = scale32 * LOG2E * d * 2.0 ** -23 * absdot + (dot.abs() * scale32 * LOG2E + l.abs() * LOG2E
                                                          + x.abs()) * 2.0 ** -23
    bound = ref * (torch.exp2(err_x) - 1) * 1.01 + ref * 2.0 ** -21 + 1e-37
    return ref, bound


def reference_and_bound(q, k, lse, hw: int, scale: float, keep):
    """:func:`exp_and_bound` of image-first operands ``[B, heads, hw + T, d]`` (lse ``[B, heads, >= hw]``) over the
    kept samples ``keep``."""
    return exp_and_bound(q[keep, :, :hw], k[keep, :, hw:], lse[keep, :, :hw], scale)


def joint_block(q: torch.Tensor, k: torch.Tensor, n_image: int, scale: float) -> torch.Tensor:
    """``q`` / ``k`` ``[B, heads, n_image + T, d]`` (image tokens first): the float64 joint softmax of every query over
    every key, image-query rows and context-key columns: ``[B, heads, T, n_image]`` (token-major, like a slab)."""
    q, k = q.double(), k.double()
    s = torch.einsum('bhid,bhjd->bhij', q[:, :, :n_image], k) * scale
    p = torch.softmax(s, dim=-1)
    return p[..., n_image:].transpose(-1, -2).contiguous()


def image_mass(q: torch.Tensor, k: torch.Tensor, n_image: int, scale: float) -> torch.Tensor:
    """``[B, heads, n_image]``: the softmax mass of every image query on the image keys (the part a map drops)."""
    q, k = q.double(), k.double()
    s = torch.einsum('bhid,bhjd->bhij', q[:, :, :n_image], k) * scale
    return torch.softmax(s, dim=-1)[..., :n_image].sum(-1)


def joint_maps(calls, n_image: int, grid, heads: int, prompt: int = 0, n_prompts: int = 1):
    """The per-layer sums of a traced generation: ``calls`` is a list of ``(layer, q, k)`` with the whole CFG batch
    ``[uncond x N, cond x N]``. Returns ``{layer: [N, heads, T, h, w]}`` over the conditional half, in float64."""
    out = {}
    for layer, q, k in calls:
        b = q.shape[0]
        block = joint_block(q[b // 2:], k[b // 2:], n_image, q.shape[-1] ** -0.5)
        block = block.view(block.shape[0], heads, block.shape[2], *grid)
        out[layer] = block if layer not in out else out[layer] + block
    return out


def global_rows(per_layer, rows, prompt: int = 0, images: int = 1, normalize: bool = False, first_row: int = 0):
    """The global map of ``prompt`` over ``per_layer`` (``joint_maps``' result): the mean over every layer's keys of
    context rows ``first_row + r`` for ``r`` in ``rows``; with ``normalize`` divided by rows ``1 .. n - 2`` plus 1e-6."""
    keys = [m[prompt * images:(prompt + 1) * images].flatten(0, 1) for m in per_layer.values()]
    mean = torch.cat(keys).mean(0)
    maps = mean[[first_row + r for r in rows]]
    if normalize:
        maps = maps / (maps[1:-1].sum(0, keepdim=True) + 1e-6)
    return maps
