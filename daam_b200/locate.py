"""Enumeration of a UNet's cross-attention layers in the order that defines ``layer_idx``.

The tracer's layer indices, and therefore every ``(factor, layer, head)`` key, follow the reference's walk
(the reference's ``daam/hook.py:95-127``): the ``up_blocks`` come first, then the ``down_blocks``, then -- only when
asked -- the ``mid_block``; inside a block whose class name contains ``CrossAttn`` every
``attentions[*].transformer_blocks[*].attn2`` is taken in module order. Names restart at 0 in every block
(``up-attn-0`` occurs once per up block), exactly like the reference's.

An MM-DiT transformer (Stable Diffusion 3 / 3.5) has no cross-attention: :class:`JointAttentionLocator` takes the joint
attention ``transformer_blocks[i].attn`` of every block, ``layer_idx = i``, named ``joint-attn-{i}``. The image-only
``attn2`` some SD3.5 blocks add attends to no text and is not located. A FLUX.1 transformer adds
``single_transformer_blocks``, whose attention runs over the already-joined ``[text, image]`` sequence: they follow
the double blocks, ``layer_idx = n_double + j``, named ``single-attn-{j}``.
"""
from __future__ import annotations

from typing import Generic, Iterable, List, Optional, Set, Tuple, TypeVar

import torch.nn as nn

__all__ = ['ModuleLocator', 'UNetCrossAttentionLocator', 'JointAttentionLocator']

ModuleType = TypeVar('ModuleType')


class ModuleLocator(Generic[ModuleType]):
    def locate(self, model: nn.Module) -> List[ModuleType]:
        raise NotImplementedError


def _tagged_blocks(model, with_mid: bool) -> Iterable[Tuple[str, nn.Module]]:
    for block in model.up_blocks:
        yield 'up', block
    for block in model.down_blocks:
        yield 'down', block
    if with_mid:
        yield 'mid', model.mid_block


class UNetCrossAttentionLocator(ModuleLocator):
    """``locate(unet)`` returns the ``attn2`` modules; position in the list == ``layer_idx``; ``layer_names`` is filled
    alongside. ``restrict`` keeps only the given per-block positions (``low_memory`` uses ``{0}``)."""

    def __init__(self, restrict: Optional[Set[int]] = None, locate_middle_block: bool = False):
        self.restrict = restrict
        self.locate_middle_block = locate_middle_block
        self.layer_names: List[str] = []

    def _wanted(self, position: int) -> bool:
        return self.restrict is None or position in self.restrict

    def locate(self, model) -> list:
        found: list = []
        names: List[str] = []
        for tag, block in _tagged_blocks(model, self.locate_middle_block):
            if 'CrossAttn' not in block.__class__.__name__:
                continue
            position = 0
            for transformer in block.attentions:
                for inner in transformer.transformer_blocks:
                    if self._wanted(position):
                        found.append(inner.attn2)
                        names.append(f'{tag}-attn-{position}')
                    position += 1
        self.layer_names[:] = names
        return found


class JointAttentionLocator(ModuleLocator):
    """``locate(transformer)`` returns ``transformer_blocks[*].attn`` in block order, then (FLUX.1) the
    ``single_transformer_blocks[*].attn`` in block order; ``layer_names`` is filled alongside. Double block ``i`` is
    ``layer_idx = i``, named ``joint-attn-{i}``; single block ``j`` is ``layer_idx = n_double + j``, named
    ``single-attn-{j}``."""

    def __init__(self):
        self.layer_names: List[str] = []

    def locate(self, model) -> list:
        found = [block.attn for block in model.transformer_blocks]
        names = [f'joint-attn-{i}' for i in range(len(found))]
        for j, block in enumerate(getattr(model, 'single_transformer_blocks', None) or ()):
            found.append(block.attn)
            names.append(f'single-attn-{j}')
        self.layer_names[:] = names
        return found
