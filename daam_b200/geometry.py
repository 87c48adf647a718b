"""The heat-map geometry of one latent size: the grid the global heat maps live on, and each traced layer's key size
``(h, w)`` and spatial factor. The tracer asks this one object for all of them.

* Square latent (``H == W``, and before the first UNet forward): the reference's rule, bit for bit -- the grid is
  ``sqrt(latent_hw)`` on both axes, a layer of ``n`` query positions has keys ``sqrt(n)`` on both axes and factor
  ``int(sqrt(latent_hw // n))`` (daam/trace.py:32-33, 285-289), including its quirks at square sizes other than the
  model's own (SD-2.1-base at 768 pixels: factor 0).
* Non-square latent: with ``g = unet.config.sample_size / sqrt(latent_hw)`` (1 for SD-1.x / SD-2.x, 2 for SDXL) the grid
  is ``(ceil(H / g), ceil(W / g))``; a layer with ``n`` query positions sits at the level ``s`` where
  ``ceil(H / 2^s) * ceil(W / 2^s) == n`` (diffusers' stride-2 convolutions; the up path resizes to the skip's size), its
  keys are ``[ceil(H / 2^s), ceil(W / 2^s)]`` in row-major pixel order and its factor is ``2^s // g``.
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

__all__ = ['LatentGeometry', 'JointGeometry', 'FluxGeometry']


class LatentGeometry:
    """``latent_hw``: the tracer's ``latent_hw`` (4096 or 9216); ``sample_size``: ``unet.config.sample_size``;
    ``latent_shape``: ``(H, W)`` of the sample the UNet receives, ``None`` while unknown (treated as square)."""

    def __init__(self, latent_hw: int, sample_size: int, latent_shape: Optional[Tuple[int, int]] = None):
        self.latent_hw = latent_hw
        self.latent_shape = None if latent_shape is None else (int(latent_shape[0]), int(latent_shape[1]))
        self.square = self.latent_shape is None or self.latent_shape[0] == self.latent_shape[1]
        if self.square:
            x = int(math.sqrt(latent_hw))
            self.g = None
            self.grid: Tuple[int, int] = (x, x)
        else:
            H, W = self.latent_shape
            g = sample_size / math.sqrt(latent_hw)
            if g not in (1, 2):
                raise ValueError(f'heat maps of a non-square {H}x{W} latent need unet.config.sample_size / '
                                 f'sqrt(latent_hw) = 1 (SD-1.x, SD-2.x) or 2 (SDXL); this UNet has {sample_size} / '
                                 f'{int(math.sqrt(latent_hw))} = {g:g}')
            self.g = int(g)
            self.grid = (-(-H // self.g), -(-W // self.g))

    @property
    def key(self):
        """What the layer rule depends on: equal keys give equal ``(h, w, factor)`` for every ``n``."""
        return None if self.square else self.latent_shape

    def level(self, n: int, layer_idx: int = 0) -> Tuple[Optional[int], Optional[int], int]:
        """``(h, w, factor)`` of a layer with ``n`` query positions. Square rule: ``h = w = None`` when ``n`` is not a
        perfect square (the caller raises if it needs them). Non-square rule: raises ``RuntimeError`` when no level
        matches."""
        if self.square:
            side = int(math.sqrt(n))
            factor = int(math.sqrt(self.latent_hw // n))
            return (side, side, factor) if side * side == n else (None, None, factor)
        H, W = self.latent_shape
        s = 0
        while True:
            h, w = -(-H // (1 << s)), -(-W // (1 << s))
            if h * w == n:
                return h, w, (1 << s) // self.g
            if h * w < n or (h == 1 and w == 1):
                raise RuntimeError(f'layer {layer_idx}: {n} query positions match no level of the {H}x{W} latent '
                                   f'(ceil(H / 2^s) * ceil(W / 2^s) for s = 0, 1, ...)')
            s += 1


class JointGeometry:
    """The heat-map geometry of an MM-DiT (Stable Diffusion 3): the transformer cuts the ``(H, W)`` latent into
    ``patch_size`` x ``patch_size`` patches, one image token each, so the grid is ``(H / p, W / p)`` and every traced
    layer's keys have the grid's size and factor 1. ``latent_shape`` is ``None`` until the first transformer forward."""

    def __init__(self, patch_size: int, latent_shape: Optional[Tuple[int, int]] = None):
        self.patch_size = int(patch_size)
        self.latent_shape = None if latent_shape is None else (int(latent_shape[0]), int(latent_shape[1]))
        self.grid: Tuple[int, int] = (0, 0) if latent_shape is None else \
            (self.latent_shape[0] // self.patch_size, self.latent_shape[1] // self.patch_size)

    def level(self, n: int, layer_idx: int = 0) -> Tuple[int, int, int]:
        """``(h, w, 1)`` for a layer of ``n`` image tokens; raises ``RuntimeError`` when ``n`` is not the grid's size."""
        h, w = self.grid
        if h * w != n:
            raise RuntimeError(f'layer {layer_idx}: {n} image tokens, but the {self.latent_shape} latent in '
                               f'{self.patch_size} x {self.patch_size} patches gives {h} x {w}')
        return h, w, 1


class FluxGeometry:
    """The heat-map geometry of a FLUX.1 transformer: the pipeline packs the ``(height / v, width / v)`` latent
    (``v = vae_scale_factor``) into 2 x 2 patches, one image token each, so the grid is
    ``(height // 2v, width // 2v)`` and every traced layer's keys have the grid's size and factor 1. ``image_size`` is
    the ``(height, width)`` in pixels the pipeline passed to ``check_inputs``, ``None`` until then; the packed latent
    ``[B, hw, 64]`` itself does not say which way round its ``hw`` tokens lie."""

    def __init__(self, vae_scale_factor: int, image_size: Optional[Tuple[int, int]] = None):
        self.vae_scale_factor = int(vae_scale_factor)
        self.image_size = None if image_size is None else (int(image_size[0]), int(image_size[1]))
        cell = 2 * self.vae_scale_factor
        self.grid: Tuple[int, int] = (0, 0) if image_size is None else \
            (self.image_size[0] // cell, self.image_size[1] // cell)

    def level(self, n: int, layer_idx: int = 0) -> Tuple[int, int, int]:
        """``(h, w, 1)`` for a layer of ``n`` image tokens; raises ``RuntimeError`` when ``n`` is not the grid's size."""
        h, w = self.grid
        if h * w != n:
            raise RuntimeError(f'layer {layer_idx}: {n} image tokens, but a {self.image_size} (height, width) image '
                               f'in {2 * self.vae_scale_factor}-pixel patches gives {h} x {w}')
        return h, w, 1
