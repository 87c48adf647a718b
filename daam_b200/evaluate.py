"""Mask overlap measures of the reference's evaluation helpers (``daam/evaluate.py:14-35``).

Only ``compute_iou`` / ``compute_ioa`` are mirrored -- the part of SURVEY.md section 8f rank 4 that touches heat maps.
When the two masks differ in size the reference bicubically resizes the first to the second and binarises it at 1;
that resize runs on the native ``daam_expand_as`` kernel (absolute mode). The COCO evaluators (``UnsupervisedEvaluator``,
``MeanEvaluator``, PNG mask loading) are out of scope.

These functions score one (mask, region) pair per call, each ending in a blocking ``.item()``. To score a word list
against several regions, or every step of a history, use :meth:`GlobalHeatMap.region_overlap
<daam_b200.heatmap.GlobalHeatMap.region_overlap>` / :meth:`GlobalHeatMapStack.region_overlap
<daam_b200.heatmap.GlobalHeatMapStack.region_overlap>`: three fused launches for every (map, region, word), whose
``iou()`` / ``ioa()`` equal ``compute_iou`` / ``compute_ioa`` of each thresholded mask and binary region bit for bit.
To choose the threshold, or to draw IoU, precision and recall against it, use :meth:`GlobalHeatMap.region_sweep
<daam_b200.heatmap.GlobalHeatMap.region_sweep>` / :meth:`GlobalHeatMapStack.region_sweep
<daam_b200.heatmap.GlobalHeatMapStack.region_sweep>`: the same exact counts at up to 64 thresholds in one pass.
For scores that need no threshold at all -- the pixel ROC-AUC and average precision of each word's map against each
region -- use :meth:`GlobalHeatMap.region_ranking <daam_b200.heatmap.GlobalHeatMap.region_ranking>` /
:meth:`GlobalHeatMapStack.region_ranking <daam_b200.heatmap.GlobalHeatMapStack.region_ranking>`: every plane sorted on
the device, exact ``u2`` counts and ``ap`` equal to ``roc_auc_score`` / ``average_precision_score``.
To score every pair of words against each other (``WordHeatMap.compute_ioa``, the DAAM paper's head / dependent
overlap), use :meth:`GlobalHeatMap.word_overlap <daam_b200.heatmap.GlobalHeatMap.word_overlap>` or, for the relations
of a parse, :meth:`GlobalHeatMap.relation_overlap <daam_b200.heatmap.GlobalHeatMap.relation_overlap>`, on one map or a
stack: three fused launches for every pair, with the same bit-for-bit equality for thresholded masks. For the boxes,
counts and centroids of each word's thresholded mask (the localisation protocol: the largest connected component's
box against a ground-truth box), use :meth:`GlobalHeatMap.word_instances <daam_b200.heatmap.GlobalHeatMap.word_instances>`
and ``WordInstances.box_iou``, on one map or a stack. To refine the masks against the image before scoring them
(word boundaries that follow the image's edges rather than the heat-map grid), use :meth:`GlobalHeatMap.refine_words
<daam_b200.heatmap.GlobalHeatMap.refine_words>` / :meth:`GlobalHeatMapStack.refine_words
<daam_b200.heatmap.GlobalHeatMapStack.refine_words>`: the guided filter of each word's map with the image as guide,
fused on the device; score its result with :func:`compute_iou` or torch. To let the words compete for each pixel
with the image's edges as a guide, use :meth:`GlobalHeatMap.segment_crf <daam_b200.heatmap.GlobalHeatMap.segment_crf>`
/ :meth:`GlobalHeatMapStack.segment_crf <daam_b200.heatmap.GlobalHeatMapStack.segment_crf>`: mean-field inference of
a Potts CRF over the word maps, a label per pixel as :meth:`GlobalHeatMap.segment` gives, whose ``labels == w + 1``
masks score with :func:`boundary_scores` like any other.
To measure where each word's boundary lies against each region's -- the boundary F-measure at pixel tolerances, the
Hausdorff distance and the average symmetric surface distance, the scores a smeared or shifted boundary moves and IoU
barely does -- use :meth:`GlobalHeatMap.region_boundary <daam_b200.heatmap.GlobalHeatMap.region_boundary>` /
:meth:`GlobalHeatMapStack.region_boundary <daam_b200.heatmap.GlobalHeatMapStack.region_boundary>` on the thresholded
word masks, or :func:`boundary_scores` on any device masks, such as ``refine_words(...) > t``: every boundary pixel's
nearest boundary pixel of the other set found exactly on the device, in one call for every (mask, region) pair.
To grow, shrink or feather a mask -- a word's mask as an inpainting mask, its confident core, the gaps between its
blobs closed -- use :meth:`GlobalHeatMap.word_distance <daam_b200.heatmap.GlobalHeatMap.word_distance>` on the
thresholded word masks, or :func:`distance_transform` on any device masks: the exact signed distance transform, whose
``mask(r)``, ``soft_mask(r, feather=f)`` and ``distance()`` are the edits.
To let the words compete per region of the image rather than per pixel, use :meth:`GlobalHeatMap.segment_superpixels
<daam_b200.heatmap.GlobalHeatMap.segment_superpixels>` / :meth:`GlobalHeatMapStack.segment_superpixels
<daam_b200.heatmap.GlobalHeatMapStack.segment_superpixels>`: each word's mean over each SLIC superpixel, the labels
constant over each; :func:`superpixels` gives the partition alone.
"""
from __future__ import annotations

import torch

from . import _native

__all__ = ['compute_iou', 'compute_ioa', 'boundary_scores', 'distance_transform', 'superpixels']


def _match_size(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """evaluate.py:15-18 / 27-30: bicubic resize of ``a`` to ``b``'s shape, then ``a < 1 -> 0``, ``a >= 1 -> 1``.
    Like the reference, only ``shape[0]`` decides whether to resize; ``a`` may be rectangular."""
    if a.shape[0] == b.shape[0]:
        return a
    if not a.is_cuda:
        raise RuntimeError('compute_iou/compute_ioa resize on CUDA tensors only (there is no CPU fallback)')
    src = a.detach().float().contiguous()
    out = torch.empty(tuple(b.shape), dtype=torch.float32, device=a.device)
    scratch = torch.empty(2, dtype=torch.float32, device=a.device)
    with torch.cuda.device(a.device):
        _native.expand_as(src.data_ptr(), tuple(src.shape), b.shape[0], b.shape[1], True, None, out.data_ptr(),
                          scratch.data_ptr(), torch.cuda.current_stream(a.device).cuda_stream)
    return (out >= 1).float()


def compute_iou(a: torch.Tensor, b: torch.Tensor) -> float:
    a = _match_size(a, b)
    intersection = (a * b).sum()
    union = a.sum() + b.sum() - intersection
    return (intersection / (union + 1e-8)).item()


def compute_ioa(a: torch.Tensor, b: torch.Tensor) -> float:
    a = _match_size(a, b)
    intersection = (a * b).sum()
    return (intersection / (a.sum() + 1e-8)).item()


def boundary_scores(masks: torch.Tensor, regions: torch.Tensor, tolerances=None, to_cpu: bool = True):
    """Boundary scores of device masks against image regions: :meth:`GlobalHeatMap.region_boundary
    <daam_b200.heatmap.GlobalHeatMap.region_boundary>` with the masks given. ``masks``: bool or uint8 ``[W, H, W']``
    or ``[M, W, H, W']`` on a CUDA device, any nonzero byte inside; the second-to-last mask axis is the word axis, so
    ``refine_words(...) > t`` of a heat map (``[words, H, W]``) or of a stack (``[maps, words, H, W]``) gives the shapes
    ``region_boundary`` gives. ``regions``: bool or uint8 ``[H, W']`` (one region) or ``[R, H, W']`` on the same device.
    ``tolerances`` as for ``region_boundary`` (``None``: ``ceil(0.008 * sqrt(H**2 + W'**2))``). Returns a
    :class:`~daam_b200.heatmap.RegionBoundary` (``word_hits`` ``[..., T, R, W]``, ``max_d2`` ``[..., R, W, 2]``, ...,
    with ``...`` the ``M`` axis of 4-D masks), on the CPU unless ``to_cpu=False``. No mask or no region launches
    nothing and gives empty axes. At most 63 regions and 2**24 pixels."""
    from .heatmap import (RegionBoundary, _boundary_outputs, _boundary_pointers, _boundary_scratch,
                          _boundary_tolerances, _require_cuda, _stream_ptr)
    what = 'boundary_scores'
    for name, t in (('masks', masks), ('regions', regions)):
        if not isinstance(t, torch.Tensor):
            raise TypeError(f'{what}: {name} must be a torch.Tensor, not {type(t).__name__}')
        if t.dtype not in (torch.bool, torch.uint8):
            raise TypeError(f'{what}: {name} must be bool or uint8, not {t.dtype}')
    if masks.dim() not in (3, 4):
        raise ValueError(f'{what}: masks must be [W, H, W\'] or [M, W, H, W\'], not {tuple(masks.shape)}')
    if regions.dim() == 2:
        regions = regions[None]
    out_h, out_w = masks.shape[-2:]
    if regions.dim() != 3 or tuple(regions.shape[1:]) != (out_h, out_w):
        raise ValueError(f'{what}: regions of shape {tuple(regions.shape)} do not match the masks\' (R, {out_h}, '
                         f'{out_w}) (a [{out_h}, {out_w}] region or a stack of them)')
    _require_cuda(masks, what)
    _require_cuda(regions, what)
    if regions.device != masks.device:
        raise ValueError(f'{what}: regions are on {regions.device}, the masks on {masks.device}')
    if out_h * out_w > 1 << 24:
        raise ValueError(f'{what}: a {out_h} x {out_w} mask is more than 2**24 pixels')
    n_regions = regions.shape[0]
    if n_regions > _native.MAX_REGIONS:
        raise ValueError(f'{what}: {n_regions} regions > {_native.MAX_REGIONS}, the region limit of one call')
    tol = _boundary_tolerances(tolerances, out_h, out_w, what)
    lead = tuple(masks.shape[:-3])
    n_words, dev = masks.shape[-3], masks.device
    n_planes = n_words * (lead[0] if lead else 1)
    if n_planes == 0 or n_regions == 0 or out_h * out_w == 0:
        out = _boundary_outputs(lead, n_regions, n_words, len(tol), tol, dev, torch.zeros)
        return out.cpu() if to_cpu else out
    mask_bytes = masks.detach().contiguous().view(torch.uint8)
    region_bytes = regions.detach().contiguous().view(torch.uint8)
    flat = _boundary_outputs((n_planes,), n_regions, 1, len(tol), tol, dev)
    scratch = _boundary_scratch(n_regions, n_planes, out_h, out_w, dev)
    with torch.cuda.device(dev):
        _native.mask_boundary(mask_bytes.data_ptr(), n_planes, out_h, out_w, region_bytes.data_ptr(), n_regions, tol,
                              *_boundary_pointers(flat), scratch.data_ptr(), scratch.numel(), _stream_ptr(dev))
    # the call's planes are (mask, word) in order, the plane axis first: move the word axis last
    m, R, T = n_planes // n_words, n_regions, len(tol)
    shaped = [flat.word_boundary.reshape(m, n_words),
              flat.word_hits.reshape(m, n_words, T, R).permute(0, 2, 3, 1),
              flat.region_hits.reshape(m, n_words, T, R).permute(0, 2, 3, 1),
              flat.max_d2.reshape(m, n_words, R, 2).permute(0, 2, 1, 3),
              flat.sum_dist.reshape(m, n_words, R, 2).permute(0, 2, 1, 3)]
    shaped = [(t if lead else t[0]).contiguous() for t in shaped]
    out = RegionBoundary(shaped[0], flat.region_boundary, *shaped[1:], flat.tolerances)
    return out.cpu() if to_cpu else out


def distance_transform(masks: torch.Tensor, to_cpu: bool = True):
    """The exact signed distance transform of device masks: :meth:`GlobalHeatMap.word_distance
    <daam_b200.heatmap.GlobalHeatMap.word_distance>` with the masks given. ``masks``: bool or uint8 ``[H, W]``,
    ``[N, H, W]`` or ``[M, N, H, W]`` on a CUDA device, any nonzero byte inside, such as ``refine_words(...) > t``,
    ``segment_crf(...)[1] == w + 1`` or a mask this call has grown: ``distance_transform(wd.mask(r)).mask(-r)`` is the
    closing of ``wd``'s masks by the disk of radius ``r``. Returns a :class:`~daam_b200.heatmap.WordDistance` whose
    ``signed_d2`` has the masks' shape, on the CPU unless ``to_cpu=False``. Two launches; no scratch. An empty shape
    launches nothing. At most 2**24 pixels and 32767 pixels a side."""
    from .heatmap import WordDistance, _distance_size, _require_cuda, _stream_ptr
    what = 'distance_transform'
    if not isinstance(masks, torch.Tensor):
        raise TypeError(f'{what}: masks must be a torch.Tensor, not {type(masks).__name__}')
    if masks.dtype not in (torch.bool, torch.uint8):
        raise TypeError(f'{what}: masks must be bool or uint8, not {masks.dtype}')
    if masks.dim() not in (2, 3, 4):
        raise ValueError(f'{what}: masks must be [H, W], [N, H, W] or [M, N, H, W], not {tuple(masks.shape)}')
    _require_cuda(masks, what)
    out_h, out_w = masks.shape[-2:]
    _distance_size(out_h, out_w, what)
    out = WordDistance(torch.empty(masks.shape, dtype=torch.int32, device=masks.device))
    if masks.numel() > 0:
        mask_bytes = masks.detach().contiguous().view(torch.uint8)
        with torch.cuda.device(masks.device):
            _native.mask_distance(mask_bytes.data_ptr(), masks.numel() // (out_h * out_w), out_h, out_w,
                                  out.signed_d2.data_ptr(), _stream_ptr(masks.device))
    return out.cpu() if to_cpu else out


def superpixels(image: torch.Tensor, n_segments: int = 1024, compactness: float = 20.0, iterations: int = 10,
                to_cpu: bool = True):
    """SLIC superpixels of device images: the partition :meth:`GlobalHeatMap.segment_superpixels
    <daam_b200.heatmap.GlobalHeatMap.segment_superpixels>` pools over, with the same arguments and the same bits.
    ``image``: uint8 ``[H, W, 3]`` or ``[N, H, W, 3]`` RGB on a CUDA device. ``compactness`` is on the 0-255 RGB scale
    (the default of 20 is twice skimage's Lab default, because RGB differences run larger than Lab's). Returns int32
    ``[H, W]`` or ``[N, H, W]``, each pixel's cluster id ``cy * nx + cx`` (superpixels may be disconnected and empty
    clusters leave ids unused), on the CPU unless ``to_cpu=False``. ``2 * iterations`` launches. An empty shape
    launches nothing. At most 2**24 pixels and 65536 cells; ``n_segments`` >= 1, ``compactness`` finite and > 0,
    ``iterations`` in ``[1, 64]`` (a ``ValueError`` otherwise)."""
    from .heatmap import _image_superpixels, _require_cuda, _superpixel_args, _superpixel_grid
    what = 'superpixels'
    if not isinstance(image, torch.Tensor):
        raise TypeError(f'{what}: image must be a torch.Tensor, not {type(image).__name__}')
    if image.dtype != torch.uint8:
        raise TypeError(f'{what}: image must be uint8, not {image.dtype}')
    if image.dim() not in (3, 4) or image.shape[-1] != 3:
        raise ValueError(f'{what}: image must be [H, W, 3] or [N, H, W, 3], not {tuple(image.shape)}')
    _require_cuda(image, what)
    out_h, out_w = int(image.shape[-3]), int(image.shape[-2])
    _superpixel_args(out_h, out_w, n_segments, compactness, iterations, what)
    n_images = image.numel() // (3 * out_h * out_w) if out_h * out_w else 0
    if n_images == 0:
        out = torch.empty(image.shape[:-1], dtype=torch.int32, device=image.device)
    else:
        ny, nx = _superpixel_grid(out_h, out_w, n_segments, what)
        out = _image_superpixels(image.detach().contiguous(), n_images, out_h, out_w, n_segments, compactness,
                                 iterations, ny, nx).view(image.shape[:-1])
    return out.cpu() if to_cpu else out
