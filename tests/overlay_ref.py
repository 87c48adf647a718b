"""The heat-map overlay restated: matplotlib's ``jet`` table in float64 and the overlay arithmetic as a torch
composition of ``expand_words`` output. ``GlobalHeatMap.overlay_words`` must equal it byte for byte."""
import numpy as np
import torch

# matplotlib's `jet` segment data (matplotlib/_cm.py): (x, y) points per channel
JET = (
    ((0., 0.), (0.35, 0.), (0.66, 1.), (0.89, 1.), (1., 0.5)),
    ((0., 0.), (0.125, 0.), (0.375, 1.), (0.64, 1.), (0.91, 0.), (1., 0.)),
    ((0., 0.5), (0.11, 1.), (0.34, 1.), (0.65, 0.), (1., 0.)),
)


def jet64(ch: int, x: float) -> float:
    """Channel ``ch`` of ``jet`` at ``x`` in float64: linear between the two segment points around ``x``."""
    pts = JET[ch]
    i = 0
    while i + 2 < len(pts) and x > pts[i + 1][0]:
        i += 1
    (x0, y0), (x1, y1) = pts[i], pts[i + 1]
    t = (x - x0) / (x1 - x0)
    return y0 + (y1 - y0) * t


def jet_table() -> torch.Tensor:
    """``L[k][ch] = fp32(255 * jet_ch(k / 255))``, fp32 ``[256, 3]``."""
    t = np.array([[255.0 * jet64(ch, k / 255.0) for ch in range(3)] for k in range(256)], dtype=np.float64)
    return torch.from_numpy(t.astype(np.float32))


def color_index(m: torch.Tensor, color_normalize: bool) -> torch.Tensor:
    """``k`` per pixel of ``m`` ``[..., H, W]``: matplotlib's N = 256 lookup of the autoscaled or clipped map."""
    if color_normalize:
        lo = m.amin((-2, -1), keepdim=True)
        hi = m.amax((-2, -1), keepdim=True)
        c = torch.where(hi == lo, torch.zeros_like(m), (m - lo) / (hi - lo))
    else:
        c = m.clamp(0, 1)
    return (c * 256.0).to(torch.int64).clamp(max=255)


def overlay_reference(m: torch.Tensor, image: torch.Tensor, color_normalize: bool, table: torch.Tensor) -> torch.Tensor:
    """uint8 ``[..., H, W, 3]`` frames of the fp32 maps ``m`` ``[..., H, W]`` over the uint8 ``image`` ``[H, W, 3]``:
    every operation a separate fp32 rounding, as in the kernel."""
    k = color_index(m, color_normalize)
    a = m.clamp(0, 1).unsqueeze(-1)
    lut = table.to(m.device)[k]
    out = (1 - a) * image.to(m.device).float() + a * lut
    return out.round().clamp(0, 255).to(torch.uint8)
