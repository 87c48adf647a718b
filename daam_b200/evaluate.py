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
fused on the device; score its result with :func:`compute_iou` or torch.
"""
from __future__ import annotations

import torch

from . import _native

__all__ = ['compute_iou', 'compute_ioa']


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
