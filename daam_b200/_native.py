"""ctypes binding of ``libdaam_b200.so`` (C ABI: ``include/daam_b200.h``).

The library is built in-tree by ``__graft_entry__.build()`` (``daam_b200/build.py``). There is no CPU or torch
fallback behind these calls: if the shared object is missing, or a call fails, the caller gets an exception.
ctypes releases the GIL around every foreign call.
"""
from __future__ import annotations

import ctypes
import math
import os
from typing import Optional, Sequence, Tuple

LIB_NAME = 'libdaam_b200.so'
LIB_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), LIB_NAME)

DAAM_F32, DAAM_F16, DAAM_BF16 = 0, 1, 2
ACC_AUTO, ACC_FORCE_SIMT, ACC_FORCE_MMA = 0, 1, 2
ACC_RMW_AUTO, ACC_RMW_LDST, ACC_RMW_RED = 0x00, 0x10, 0x20
ACC_NO_PDL = 0x100
ACC_EARLY_LOADS = 0x200   # see include/daam_b200.h: only valid when q/k were complete before the previous kernel started
ABI_VERSION = 4
E_INVALID, E_UNSUPPORTED, E_CUDA = -1, -2, -3
TOKENS = 77
CONTEXT_TOKENS = (77, 154, 231)   # daam_accumulate: one to three 77-token chunks (DAAM_MAX_TOKENS = 231)
EXPAND_SCRATCH_FLOATS = 64   # DAAM_EXPAND_SCRATCH_FLOATS: per word
MAX_SEGMENT_WORDS = 96       # daam_segment_words: labels 1..96 plus background 0 fit a byte


def segment_scratch_floats(n_maps: int, n_words: int) -> int:
    """``DAAM_SEGMENT_SCRATCH_FLOATS(n_maps, n_words)``."""
    return 64 * n_maps * n_words

MAX_REGIONS = 63             # DAAM_REGION_MAX_REGIONS: regions per daam_region_overlap call


def region_scratch_floats(n_maps: int, n_words: int, n_regions: int, out_h: int, out_w: int) -> int:
    """``DAAM_REGION_SCRATCH_FLOATS(n_maps, n_words, n_regions, out_h, out_w)``."""
    return n_maps * n_words * (64 + (n_regions + 1) * ((out_h + 15) // 16) * ((out_w + 63) // 64))


SWEEP_MAX_THRESHOLDS = 64    # DAAM_REGION_SWEEP_MAX_THRESHOLDS: thresholds per daam_region_sweep call


def region_sweep_scratch_floats(n_maps: int, n_words: int, n_regions: int, n_thresholds: int, out_h: int,
                                out_w: int) -> int:
    """``DAAM_REGION_SWEEP_SCRATCH_FLOATS(n_maps, n_words, n_regions, n_thresholds, out_h, out_w)``: the min / max
    partials and one histogram per (map, word); the output size does not enter."""
    return n_maps * n_words * (64 + (n_regions + 1) * n_thresholds)


WORD_OVERLAP_CTAS = 256      # DAAM_WORD_OVERLAP_CTAS: daam_word_overlap's CTAs per map


def word_overlap_scratch_floats(n_maps: int, n_words: int, out_h: int, out_w: int) -> int:
    """``DAAM_WORD_OVERLAP_SCRATCH_FLOATS(n_maps, n_words, out_h, out_w)``."""
    tiles = ((out_h + 15) // 16) * ((out_w + 63) // 64)
    return n_maps * (n_words * 64 + (n_words * (n_words + 3) // 2) * min(tiles, WORD_OVERLAP_CTAS))


WORD_INSTANCES_MAX = 64      # DAAM_WORD_INSTANCES_MAX: max_instances of daam_word_instances


def word_instances_plane_bytes(out_h: int, out_w: int) -> int:
    """``DAAM_WORD_INSTANCES_PLANE_BYTES(out_h, out_w)``: the scratch bytes daam_word_instances takes per (map, word)
    plane."""
    return 8 * out_h * out_w + 48 * ((out_h + 1) // 2) * ((out_w + 1) // 2) + 260


def region_ranking_plane_bytes(out_h: int, out_w: int) -> int:
    """``DAAM_REGION_RANKING_PLANE_BYTES(out_h, out_w)``: the scratch bytes daam_region_ranking takes per (map, word)
    plane of a round."""
    n = out_h * out_w
    return 16 * n + 1024 * ((n + 4095) // 4096) + 1540 * ((n + 1023) // 1024) + 512


def region_ranking_scratch_bytes(n_planes: int, out_h: int, out_w: int) -> int:
    """``DAAM_REGION_RANKING_SCRATCH_BYTES(n_planes, out_h, out_w)``: the call's region masks and ``n_planes`` planes."""
    return 8 * out_h * out_w + n_planes * region_ranking_plane_bytes(out_h, out_w)


REFINE_MAX_RADIUS = 64       # DAAM_REFINE_MAX_RADIUS: the largest radius of daam_refine_words


def refine_guide_bytes(out_h: int, out_w: int) -> int:
    """``DAAM_REFINE_GUIDE_BYTES(out_h, out_w)``: the scratch bytes daam_refine_words takes per image of a round (its
    mean and the inverse of its regularised covariance, per pixel)."""
    return 36 * out_h * out_w


def refine_plane_bytes(out_h: int, out_w: int) -> int:
    """``DAAM_REFINE_PLANE_BYTES(out_h, out_w)``: the scratch bytes daam_refine_words takes per (map, word) plane of a
    round."""
    return 32 * out_h * out_w + 256


def refine_scratch_bytes(n_images: int, n_planes: int, out_h: int, out_w: int) -> int:
    """``DAAM_REFINE_SCRATCH_BYTES(n_images, n_planes, out_h, out_w)``: ``n_images`` images' statistics and ``n_planes``
    planes; ``(1, 1)`` is the smallest scratch the call takes."""
    return n_images * refine_guide_bytes(out_h, out_w) + n_planes * refine_plane_bytes(out_h, out_w)


CRF_MAX_RADIUS = 16          # DAAM_CRF_MAX_RADIUS: the largest radius of daam_segment_crf
CRF_MAX_ITERATIONS = 64      # the most mean-field updates daam_segment_crf takes


def crf_map_bytes(n_labels: int, out_h: int, out_w: int) -> int:
    """``DAAM_CRF_MAP_BYTES(n_labels, out_h, out_w)``: the scratch bytes daam_segment_crf takes per map of a round (two
    fp32 Q buffers and the min / max partials)."""
    return 8 * n_labels * out_h * out_w + 256 * n_labels


def crf_scratch_bytes(n_maps: int, n_labels: int, out_h: int, out_w: int) -> int:
    """``DAAM_CRF_SCRATCH_BYTES(n_maps, n_labels, out_h, out_w)``: ``n_maps`` maps; ``n_maps = 1`` is the smallest
    scratch the call takes."""
    return n_maps * crf_map_bytes(n_labels, out_h, out_w)


BOUNDARY_MAX_TOLERANCES = 16  # DAAM_BOUNDARY_MAX_TOLERANCES: tolerances of daam_region_boundary / daam_mask_boundary


def boundary_tile_rows(out_w: int) -> int:
    """``DAAM_BOUNDARY_TILE_ROWS(out_w)``: the rows of one query tile of the boundary calls."""
    return 16 if out_w >= 256 else (4096 + out_w - 1) // out_w


def boundary_call_bytes(n_regions: int, out_h: int, out_w: int) -> int:
    """``DAAM_BOUNDARY_CALL_BYTES(n_regions, out_h, out_w)``: the regions' column distances, once per call (about 4
    bytes a pixel per region)."""
    return 8 * n_regions * ((out_h * out_w + 1) // 2)


def boundary_plane_bytes(out_h: int, out_w: int) -> int:
    """``DAAM_BOUNDARY_PLANE_BYTES(out_h, out_w)``: the scratch bytes the boundary calls take per plane of a round."""
    rows = boundary_tile_rows(out_w)
    return 16 * ((out_h * out_w + 1) // 2) + 256 + 10080 * ((out_h + rows - 1) // rows)


def boundary_scratch_bytes(n_regions: int, n_planes: int, out_h: int, out_w: int) -> int:
    """``DAAM_BOUNDARY_SCRATCH_BYTES(n_regions, n_planes, out_h, out_w)``: the regions' state and ``n_planes`` planes;
    ``n_planes = 1`` is the smallest scratch the calls take."""
    return boundary_call_bytes(n_regions, out_h, out_w) + n_planes * boundary_plane_bytes(out_h, out_w)


DISTANCE_NONE = 2 ** 31 - 1   # DAAM_DISTANCE_NONE: every pixel of an empty mask (+), of a full one (-)
DISTANCE_MAX_SIDE = 32767     # DAAM_DISTANCE_MAX_SIDE: the largest out_h and out_w of the distance calls


def distance_plane_bytes(out_h: int, out_w: int) -> int:
    """``DAAM_DISTANCE_PLANE_BYTES(out_h, out_w)``: the scratch bytes daam_word_distance takes per (map, word) plane of a
    round (its values and min / max partials)."""
    return 4 * out_h * out_w + 256


SUPERPIXEL_MAX_CELLS = 65536      # DAAM_SUPERPIXEL_MAX_CELLS: the most cells (ny * nx) of the superpixel grid
SUPERPIXEL_MAX_ITERATIONS = 64    # the most SLIC passes the superpixel calls take


def superpixel_grid(out_h: int, out_w: int, n_segments: int):
    """``(ny, nx)``: the superpixel calls' cell grid, ``S = sqrt(H W / K)`` in float64 and ``clamp(floor(H / S +
    0.5), 1, H)`` rows, columns likewise (include/daam_b200.h)."""
    s = math.sqrt(float(out_h * out_w) / n_segments)
    return (min(max(math.floor(out_h / s + 0.5), 1), out_h), min(max(math.floor(out_w / s + 0.5), 1), out_w))


def superpixel_image_bytes(ny: int, nx: int) -> int:
    """``DAAM_SUPERPIXEL_IMAGE_BYTES(ny, nx)``: one image's SLIC state (two sets of six int64 sums per cell)."""
    return 96 * ny * nx


def superpixel_box(ny: int, nx: int, out_h: int, out_w: int) -> int:
    """``DAAM_SUPERPIXEL_BOX(ny, nx, out_h, out_w)``: the most cells a 16 x 64 pixel tile's pixels can reach."""
    return min(ny, 15 * ny // out_h + 4) * min(nx, 63 * nx // out_w + 4)


def superpixel_map_bytes(n_words: int, ny: int, nx: int, out_h: int, out_w: int) -> int:
    """``DAAM_SUPERPIXEL_MAP_BYTES(n_words, ny, nx, out_h, out_w)``: one map's min / max partials, per-tile sums of
    each word over each cell of the tile's box, and per-superpixel label and score."""
    tiles = ((out_h + 15) // 16) * ((out_w + 63) // 64)
    return 256 * n_words + 8 * ny * nx + 8 * n_words * tiles * superpixel_box(ny, nx, out_h, out_w)


def superpixel_scratch_bytes(n_images: int, n_maps: int, n_words: int, ny: int, nx: int, out_h: int, out_w: int) -> int:
    """``DAAM_SUPERPIXEL_SCRATCH_BYTES(...)``: ``n_images`` images' state and ``n_maps`` maps' buffers; ``(1, 1)`` is
    the smallest scratch daam_segment_superpixels takes."""
    return n_images * superpixel_image_bytes(ny, nx) + n_maps * superpixel_map_bytes(n_words, ny, nx, out_h, out_w)


def overlay_frames_bytes(n_maps: int, n_words: int, out_h: int, out_w: int) -> int:
    """``DAAM_OVERLAY_FRAMES_BYTES(n_maps, n_words, out_h, out_w)``: the frames rounded up to whole 4-byte words."""
    return (n_maps * n_words * out_h * out_w * 3 + 3) // 4 * 4


EXPORTS = ('daam_accumulate', 'daam_accumulate_steps', 'daam_accumulate_range', 'daam_attention_probs', 'daam_accumulate_probs', 'daam_accumulate_joint', 'daam_accumulate_joint_heads', 'daam_finalize',
           'daam_finalize_maps', 'daam_finalize_parts', 'daam_finalize_parts_weighted', 'daam_finalize_per_key', 'daam_value_norms','daam_normalize_maps', 'daam_word_heat_map', 'daam_expand_as', 'daam_expand_words',
           'daam_segment_words', 'daam_region_overlap', 'daam_region_sweep', 'daam_region_ranking', 'daam_region_boundary', 'daam_mask_boundary', 'daam_word_overlap', 'daam_word_instances', 'daam_overlay_words', 'daam_refine_words', 'daam_segment_crf', 'daam_word_distance', 'daam_mask_distance', 'daam_image_superpixels', 'daam_segment_superpixels', 'daam_jet_colormap',
           'daam_side_launcher_create', 'daam_side_launcher_destroy',
           'daam_side_launcher_launch', 'daam_side_launcher_join', 'daam_side_launcher_idle', 'daam_abi_version',
           'daam_last_error', 'daam_device_info', 'daam_launch_count')


class DaamLayer(ctypes.Structure):
    """``struct daam_layer`` (include/daam_b200.h)."""
    _fields_ = [
        ('q', ctypes.c_void_p), ('k', ctypes.c_void_p), ('acc', ctypes.c_void_p),
        ('q_stride_prompt', ctypes.c_int64), ('q_stride_pixel', ctypes.c_int64), ('q_stride_head', ctypes.c_int64),
        ('k_stride_prompt', ctypes.c_int64), ('k_stride_token', ctypes.c_int64), ('k_stride_head', ctypes.c_int64),
        ('n_prompts', ctypes.c_int32), ('heads', ctypes.c_int32), ('hw', ctypes.c_int32), ('tokens', ctypes.c_int32),
        ('head_dim', ctypes.c_int32), ('dtype', ctypes.c_int32), ('scale', ctypes.c_float),
        ('reserved', ctypes.c_int32),
    ]


class DaamJointLayer(ctypes.Structure):
    """``struct daam_joint_layer`` (include/daam_b200.h): ``daam_layer`` plus the joint softmax's log-sum-exp."""
    _fields_ = DaamLayer._fields_ + [
        ('lse', ctypes.c_void_p),
        ('lse_stride_prompt', ctypes.c_int64), ('lse_stride_head', ctypes.c_int64), ('lse_stride_pixel', ctypes.c_int64),
    ]


JOINT_MAX_TOKENS = 1024   # DAAM_JOINT_MAX_TOKENS: context rows of a daam_accumulate_joint layer


class DaamKeyGroup(ctypes.Structure):
    """``struct daam_key_group`` (include/daam_b200.h). ``n_blocks`` is read by ``daam_finalize_maps`` only; its old
    name ``reserved`` still works."""
    _fields_ = [
        ('acc', ctypes.c_void_p), ('heads', ctypes.c_int32), ('h', ctypes.c_int32), ('w', ctypes.c_int32),
        ('tokens', ctypes.c_int32), ('head_sel', ctypes.c_int32), ('n_blocks', ctypes.c_int32),
    ]
    reserved = property(lambda self: self.n_blocks, lambda self, v: setattr(self, 'n_blocks', v))


class DaamMapSel(ctypes.Structure):
    """``struct daam_map_sel`` (include/daam_b200.h): one output map of ``daam_finalize_maps``."""
    _fields_ = [
        ('block_begin', ctypes.c_int32), ('block_count', ctypes.c_int32), ('n_rows', ctypes.c_int32),
        ('reserved', ctypes.c_int32), ('out', ctypes.c_void_p),
    ]


class DaamMapPart(ctypes.Structure):
    """``struct daam_map_part`` (include/daam_b200.h): one output map of ``daam_finalize_parts``."""
    _fields_ = [
        ('group_begin', ctypes.c_int32), ('group_count', ctypes.c_int32), ('n_rows', ctypes.c_int32),
        ('reserved', ctypes.c_int32), ('out', ctypes.c_void_p),
    ]


FINALIZE_MAX_MAPS = 64   # DAAM_FINALIZE_MAX_MAPS: maps per daam_finalize_maps / daam_finalize_parts call


class NativeError(RuntimeError):
    def __init__(self, code: int, message: str):
        super().__init__(f'libdaam_b200: {message} (status {code})')
        self.code = code


_lib: Optional[ctypes.CDLL] = None


def load() -> ctypes.CDLL:
    """dlopen the in-tree library once and declare the prototypes. Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise RuntimeError(
            f'{LIB_PATH} is missing: build it with `python -c "import __graft_entry__ as g; g.build()"` '
            f'(or `python -m daam_b200.build`). daam_b200 has no CPU fallback.')
    lib = ctypes.CDLL(LIB_PATH)
    lib.daam_abi_version.argtypes = []
    lib.daam_abi_version.restype = ctypes.c_int
    if lib.daam_abi_version() != ABI_VERSION:
        raise RuntimeError(f'{LIB_PATH} has ABI version {lib.daam_abi_version()}, this package needs {ABI_VERSION}: '
                           f'rebuild it (`python -m daam_b200.build --force`)')
    i32, u32, i64, vp, f32 = ctypes.c_int32, ctypes.c_uint32, ctypes.c_int64, ctypes.c_void_p, ctypes.c_float
    lib.daam_accumulate.argtypes = [ctypes.POINTER(DaamLayer), i32, u32, vp]
    lib.daam_accumulate.restype = ctypes.c_int
    lib.daam_accumulate_joint.argtypes = [ctypes.POINTER(DaamJointLayer), i32, u32, vp]
    lib.daam_accumulate_joint.restype = ctypes.c_int
    lib.daam_accumulate_joint_heads.argtypes = [ctypes.POINTER(DaamJointLayer), i32, u32, vp]
    lib.daam_accumulate_joint_heads.restype = ctypes.c_int
    lib.daam_accumulate_steps.argtypes = [ctypes.POINTER(DaamLayer), ctypes.POINTER(vp), i32, u32, vp]
    lib.daam_accumulate_steps.restype = ctypes.c_int
    lib.daam_accumulate_range.argtypes = [ctypes.POINTER(DaamLayer), ctypes.POINTER(vp), i32, u32, vp]
    lib.daam_accumulate_range.restype = ctypes.c_int
    lib.daam_normalize_maps.argtypes = [vp, i32, i32, i32, i32, vp]
    lib.daam_normalize_maps.restype = ctypes.c_int
    lib.daam_attention_probs.argtypes = [ctypes.POINTER(DaamLayer), vp, vp]
    lib.daam_attention_probs.restype = ctypes.c_int
    lib.daam_accumulate_probs.argtypes = [vp, i32, i32, i32, i32, i32, vp, vp]
    lib.daam_accumulate_probs.restype = ctypes.c_int
    lib.daam_finalize.argtypes = [ctypes.POINTER(DaamKeyGroup), i32, i32, i32, i32, i32, vp, vp]
    lib.daam_finalize.restype = ctypes.c_int
    lib.daam_finalize_maps.argtypes = [ctypes.POINTER(DaamKeyGroup), i32, ctypes.POINTER(DaamMapSel), i32, i32, i32,
                                       i32, vp]
    lib.daam_finalize_maps.restype = ctypes.c_int
    lib.daam_finalize_parts.argtypes = [ctypes.POINTER(DaamKeyGroup), i32, ctypes.POINTER(DaamMapPart), i32, i32, i32,
                                        i32, vp]
    lib.daam_finalize_parts.restype = ctypes.c_int
    lib.daam_finalize_parts_weighted.argtypes = [ctypes.POINTER(DaamKeyGroup), i32, ctypes.POINTER(DaamMapPart), i32,
                                                 i32, i32, i32, ctypes.POINTER(vp), vp]
    lib.daam_finalize_parts_weighted.restype = ctypes.c_int
    lib.daam_value_norms.argtypes = [vp, i32, i64, i64, i64, vp, i32, i64, i32, i32, i32, i32, i32, vp, vp]
    lib.daam_value_norms.restype = ctypes.c_int
    lib.daam_finalize_per_key.argtypes = [ctypes.POINTER(DaamKeyGroup), i32, i32, i32, i32, i32, vp, vp]
    lib.daam_finalize_per_key.restype = ctypes.c_int
    lib.daam_word_heat_map.argtypes = [vp, i32, i32, i32, ctypes.POINTER(i32), i32, vp, vp]
    lib.daam_word_heat_map.restype = ctypes.c_int
    lib.daam_expand_as.argtypes = [vp, i32, i32, i32, i32, i32, i32, f32, vp, vp, vp]
    lib.daam_expand_as.restype = ctypes.c_int
    lib.daam_expand_words.argtypes = [vp, i32, i32, i32, ctypes.POINTER(i32), ctypes.POINTER(i32), i32, i32, i32, i32,
                                      i32, f32, vp, vp, vp, vp]
    lib.daam_expand_words.restype = ctypes.c_int
    lib.daam_segment_words.argtypes = [vp, i32, i32, i32, i32, ctypes.POINTER(i32), ctypes.POINTER(i32), i32, i32, i32,
                                       i32, i32, f32, vp, vp, vp, vp, vp]
    lib.daam_segment_words.restype = ctypes.c_int
    lib.daam_region_overlap.argtypes = [vp, i32, i32, i32, i32, ctypes.POINTER(i32), ctypes.POINTER(i32), i32, i32, i32,
                                        i32, i32, f32, vp, vp, i32, vp, vp, vp, vp]
    lib.daam_region_overlap.restype = ctypes.c_int
    lib.daam_region_sweep.argtypes = [vp, i32, i32, i32, i32, ctypes.POINTER(i32), ctypes.POINTER(i32), i32, i32, i32,
                                      i32, ctypes.POINTER(f32), i32, vp, vp, i32, vp, vp, vp, vp]
    lib.daam_region_sweep.restype = ctypes.c_int
    lib.daam_region_ranking.argtypes = [vp, i32, i32, i32, i32, ctypes.POINTER(i32), ctypes.POINTER(i32), i32, i32,
                                        i32, i32, vp, vp, i32, vp, vp, vp, i64, vp]
    lib.daam_region_ranking.restype = ctypes.c_int
    lib.daam_word_overlap.argtypes = [vp, i32, i32, i32, i32, ctypes.POINTER(i32), ctypes.POINTER(i32), i32, i32, i32,
                                      i32, i32, f32, vp, vp, vp, vp, vp]
    lib.daam_word_overlap.restype = ctypes.c_int
    lib.daam_word_instances.argtypes = [vp, i32, i32, i32, i32, ctypes.POINTER(i32), ctypes.POINTER(i32), i32, i32,
                                        i32, i32, f32, i32, vp, vp, vp, vp, vp, vp, vp, vp, i64, vp]
    lib.daam_word_instances.restype = ctypes.c_int
    lib.daam_overlay_words.argtypes = [vp, i32, i32, i32, i32, ctypes.POINTER(i32), ctypes.POINTER(i32), i32, i32, i32,
                                       i32, i32, f32, i32, vp, vp, i64, vp, vp, vp]
    lib.daam_overlay_words.restype = ctypes.c_int
    lib.daam_region_boundary.argtypes = [vp, i32, i32, i32, i32, ctypes.POINTER(i32), ctypes.POINTER(i32), i32, i32,
                                         i32, i32, f32, ctypes.POINTER(f32), i32, vp, vp, i32, vp, vp, vp, vp, vp, vp,
                                         vp, i64, vp]
    lib.daam_region_boundary.restype = ctypes.c_int
    lib.daam_mask_boundary.argtypes = [vp, i32, i32, i32, vp, i32, ctypes.POINTER(f32), i32, vp, vp, vp, vp, vp, vp, vp,
                                       i64, vp]
    lib.daam_mask_boundary.restype = ctypes.c_int
    lib.daam_refine_words.argtypes = [vp, i32, i32, i32, i32, ctypes.POINTER(i32), ctypes.POINTER(i32), i32, i32, i32,
                                      i32, i32, f32, i32, f32, vp, vp, i64, vp, vp, i64, vp]
    lib.daam_refine_words.restype = ctypes.c_int
    lib.daam_segment_crf.argtypes = [vp, i32, i32, i32, i32, ctypes.POINTER(i32), ctypes.POINTER(i32), i32, i32, i32,
                                     i32, i32, f32, f32, i32, i32, f32, f32, f32, f32, f32, vp, vp, i64, vp, vp, vp, vp,
                                     i64, vp]
    lib.daam_segment_crf.restype = ctypes.c_int
    lib.daam_word_distance.argtypes = [vp, i32, i32, i32, i32, ctypes.POINTER(i32), ctypes.POINTER(i32), i32, i32, i32,
                                       i32, f32, vp, vp, vp, i64, vp]
    lib.daam_word_distance.restype = ctypes.c_int
    lib.daam_mask_distance.argtypes = [vp, i32, i32, i32, vp, vp]
    lib.daam_mask_distance.restype = ctypes.c_int
    lib.daam_image_superpixels.argtypes = [vp, i32, i32, i32, i32, f32, i32, vp, vp, i64, vp]
    lib.daam_image_superpixels.restype = ctypes.c_int
    lib.daam_segment_superpixels.argtypes = [vp, i32, i32, i32, i32, ctypes.POINTER(i32), ctypes.POINTER(i32), i32, i32,
                                             i32, i32, i32, f32, i32, f32, i32, vp, vp, i64, vp, vp, vp, vp, i64, vp]
    lib.daam_segment_superpixels.restype = ctypes.c_int
    lib.daam_jet_colormap.argtypes = [vp]
    lib.daam_jet_colormap.restype = ctypes.c_int
    lib.daam_side_launcher_create.argtypes = [ctypes.POINTER(vp)]
    lib.daam_side_launcher_create.restype = ctypes.c_int
    lib.daam_side_launcher_destroy.argtypes = [vp]
    lib.daam_side_launcher_destroy.restype = None
    lib.daam_side_launcher_launch.argtypes = [vp, ctypes.POINTER(DaamLayer), i32, u32, vp, vp]
    lib.daam_side_launcher_launch.restype = ctypes.c_int
    lib.daam_side_launcher_join.argtypes = [vp, vp]
    lib.daam_side_launcher_join.restype = ctypes.c_int
    lib.daam_side_launcher_idle.argtypes = [vp]
    lib.daam_side_launcher_idle.restype = ctypes.c_int
    lib.daam_last_error.argtypes = []
    lib.daam_last_error.restype = ctypes.c_char_p
    lib.daam_device_info.argtypes = [ctypes.POINTER(i32)] * 3
    lib.daam_device_info.restype = ctypes.c_int
    lib.daam_launch_count.argtypes = []
    lib.daam_launch_count.restype = i64
    _lib = lib
    return lib


def _check(rc: int):
    if rc != 0:
        raise NativeError(rc, load().daam_last_error().decode('utf-8', 'replace'))


class PackedLayers:
    """A ready-made ``daam_layer[]`` (host array) for call sites that replay the same layer calls."""

    def __init__(self, layers: Sequence[DaamLayer]):
        self.n = len(layers)
        self.array = (DaamLayer * max(self.n, 1))(*layers)


class SideLauncher:
    """``daam_side_launcher``: the event pair behind the tracer's per-step launch on its side stream."""

    def __init__(self):
        self._lib = load()
        handle = ctypes.c_void_p()
        _check(self._lib.daam_side_launcher_create(ctypes.byref(handle)))
        self._h = handle

    def launch(self, packed: 'PackedLayers', flags: int, producer_stream: int, side_stream: int):
        rc = self._lib.daam_side_launcher_launch(self._h, packed.array, packed.n, flags, producer_stream, side_stream)
        if rc != 0:
            _check(rc)

    def join(self, stream: int):
        rc = self._lib.daam_side_launcher_join(self._h, stream)
        if rc != 0:
            _check(rc)

    def idle(self) -> bool:
        rc = self._lib.daam_side_launcher_idle(self._h)
        if rc < 0:
            _check(rc)
        return rc == 1

    def close(self):
        if self._h is not None and self._h.value:
            self._lib.daam_side_launcher_destroy(self._h)
        self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def accumulate(layers, stream: int, flags: int = ACC_AUTO):
    """``layers``: a sequence of :class:`DaamLayer` or a :class:`PackedLayers`."""
    packed = layers if isinstance(layers, PackedLayers) else PackedLayers(layers)
    if packed.n == 0:
        return
    rc = load().daam_accumulate(packed.array, packed.n, flags, stream)
    if rc != 0:
        _check(rc)


def accumulate_joint(layers: Sequence[DaamJointLayer], stream: int):
    """``daam_accumulate_joint`` over a sequence of :class:`DaamJointLayer`: classes fp16, bf16, fp32 in that order,
    each in call order, in one launch per class unless a layer overlaps one already in the launch or the launch holds
    ``DAAM_JOINT_MAX_LAYERS``."""
    if not layers:
        return
    array = (DaamJointLayer * len(layers))(*layers)
    rc = load().daam_accumulate_joint(array, len(layers), 0, stream)
    if rc != 0:
        _check(rc)


def accumulate_joint_heads(layers: Sequence[DaamJointLayer], stream: int):
    """``daam_accumulate_joint_heads``: :func:`accumulate_joint` with every sample's heads summed in the kernel and
    divided by ``heads``, into a head-free accumulator ``[n_prompts][tokens][hw]``; same classes, order and packing."""
    if not layers:
        return
    array = (DaamJointLayer * len(layers))(*layers)
    rc = load().daam_accumulate_joint_heads(array, len(layers), 0, stream)
    if rc != 0:
        _check(rc)


class StepPointers:
    """A ready-made ``float* step_acc[]`` / ``range_acc[]`` (host array of device pointers) for
    :func:`accumulate_steps` and :func:`accumulate_range`."""

    def __init__(self, ptrs: Sequence[int]):
        self.array = (ctypes.c_void_p * max(len(ptrs), 1))(*ptrs)


def _accumulate_second(entry: str, word: str, layers, slabs, stream: int, flags: int):
    """``entry`` (``daam_accumulate_steps`` / ``daam_accumulate_range``) over ``layers`` and one second slab per layer;
    ``word`` names the slabs in messages."""
    packed = layers if isinstance(layers, PackedLayers) else PackedLayers(layers)
    if packed.n == 0:
        return
    arr = slabs if isinstance(slabs, StepPointers) else StepPointers(slabs)
    if len(arr.array) < packed.n:
        raise ValueError(f'{len(arr.array)} {word} slabs for {packed.n} layers')
    rc = getattr(load(), entry)(packed.array, arr.array, packed.n, flags, stream)
    if rc != 0:
        _check(rc)


def accumulate_steps(layers, steps, stream: int, flags: int = ACC_AUTO):
    """``daam_accumulate_steps``: ``layers`` as for :func:`accumulate`; ``steps`` a :class:`StepPointers` or a sequence of
    device pointers, one step slab per layer (the first ``n`` are used)."""
    _accumulate_second('daam_accumulate_steps', 'step', layers, steps, stream, flags)


def accumulate_range(layers, ranges, stream: int, flags: int = ACC_AUTO):
    """``daam_accumulate_range``: ``layers`` as for :func:`accumulate`; ``ranges`` a :class:`StepPointers` or a sequence
    of device pointers, one range slab per layer (the first ``n`` are used)."""
    _accumulate_second('daam_accumulate_range', 'range', layers, ranges, stream, flags)


def map_size(x) -> Tuple[int, int]:
    """A heat-map grid given as its side ``x`` (square) or as ``(h, w)``: returns ``(h, w)``."""
    if isinstance(x, (tuple, list)):      # (torch.Size is a tuple)
        h, w = x
        return int(h), int(w)
    return int(x), int(x)


def normalize_maps(maps_ptr: int, n_maps: int, n_rows: int, x, stream: int):
    """``x``: the map side, or ``(h, w)``."""
    h, w = map_size(x)
    _check(load().daam_normalize_maps(ctypes.c_void_p(maps_ptr), n_maps, n_rows, h, w, ctypes.c_void_p(stream)))


def attention_probs(layer: DaamLayer, probs_ptr: int, stream: int):
    _check(load().daam_attention_probs(ctypes.byref(layer), probs_ptr, stream))


def accumulate_probs(probs_ptr: int, dtype: int, first_row: int, n_rows: int, hw: int, tokens: int, acc_ptr: int,
                     stream: int):
    _check(load().daam_accumulate_probs(probs_ptr, dtype, first_row, n_rows, hw, tokens, acc_ptr, stream))


# The finalize / word-map / expand wrappers take the map grid as its side ``x`` or as ``(h, w)``.
def _finalize(entry: str, groups: Sequence[DaamKeyGroup], x, n_rows: int, normalize: bool, out_ptr: int, stream: int):
    """``entry``: ``daam_finalize`` or ``daam_finalize_per_key`` (same arguments)."""
    h, w = map_size(x)
    n = len(groups)
    arr = (DaamKeyGroup * max(n, 1))(*groups)
    _check(getattr(load(), entry)(arr, n, h, w, n_rows, int(bool(normalize)), ctypes.c_void_p(out_ptr),
                                  ctypes.c_void_p(stream)))


def finalize(groups: Sequence[DaamKeyGroup], x, n_rows: int, normalize: bool, out_ptr: int, stream: int):
    _finalize('daam_finalize', groups, x, n_rows, normalize, out_ptr, stream)


def finalize_maps(groups: Sequence[DaamKeyGroup], maps: Sequence[DaamMapSel], x, normalize: bool, stream: int):
    """``daam_finalize_maps``: ``groups`` with ``n_blocks`` set, one :class:`DaamMapSel` per output map. More than
    :data:`FINALIZE_MAX_MAPS` maps go out in several calls, which changes no map's bits."""
    h, w = map_size(x)
    n = len(groups)
    arr = (DaamKeyGroup * max(n, 1))(*groups)
    lib = load()
    for i in range(0, max(len(maps), 1), FINALIZE_MAX_MAPS):
        part = maps[i:i + FINALIZE_MAX_MAPS]
        sel = (DaamMapSel * max(len(part), 1))(*part)
        _check(lib.daam_finalize_maps(arr, n, sel, len(part), h, w, int(bool(normalize)), ctypes.c_void_p(stream)))


def finalize_parts(groups: Sequence[DaamKeyGroup], parts: Sequence[DaamMapPart], x, normalize: bool, stream: int,
                   weights: Optional[Sequence[int]] = None):
    """``daam_finalize_parts``: one :class:`DaamMapPart` per output map, each a range of ``groups``. More than
    :data:`FINALIZE_MAX_MAPS` maps go out in several calls, which changes no map's bits. A part that is no range of
    ``groups``, or has no rows or output, is a ``ValueError`` before anything is loaded or launched. ``weights``: one
    device pointer per group (``[heads, tokens]`` fp32) -- ``daam_finalize_parts_weighted``; a list of another length
    is a ``ValueError``."""
    h, w = map_size(x)
    n = len(groups)
    if not parts:
        raise ValueError('finalize_parts: no output map')
    for i, part in enumerate(parts):
        if part.group_begin < 0 or part.group_count <= 0 or part.group_begin + part.group_count > n:
            raise ValueError(f'finalize_parts: map {i} reads groups [{part.group_begin}, +{part.group_count}) of {n}')
        if part.n_rows <= 0 or not part.out:
            raise ValueError(f'finalize_parts: map {i} has no rows or no output')
    if weights is not None and len(weights) != n:
        raise ValueError(f'finalize_parts: {len(weights)} weight pointers for {n} key groups')
    arr = (DaamKeyGroup * n)(*groups)
    lib = load()
    wts = None if weights is None else (ctypes.c_void_p * n)(*weights)
    for i in range(0, len(parts), FINALIZE_MAX_MAPS):
        chunk = parts[i:i + FINALIZE_MAX_MAPS]
        sel = (DaamMapPart * len(chunk))(*chunk)
        if wts is None:
            _check(lib.daam_finalize_parts(arr, n, sel, len(chunk), h, w, int(bool(normalize)), ctypes.c_void_p(stream)))
        else:
            _check(lib.daam_finalize_parts_weighted(arr, n, sel, len(chunk), h, w, int(bool(normalize)), wts,
                                                    ctypes.c_void_p(stream)))


def value_norms(value_ptr: int, value_dtype: int, v_strides: Tuple[int, int, int], w_ptr: int, w_dtype: int,
                w_stride_row: int, n_samples: int, heads: int, tokens: int, head_dim: int, out_dim: int, out_ptr: int,
                stream: int):
    """``daam_value_norms``: ``v_strides`` = (sample, token, head) element strides of the value projection."""
    _check(load().daam_value_norms(ctypes.c_void_p(value_ptr), value_dtype, *v_strides, ctypes.c_void_p(w_ptr), w_dtype,
                                   w_stride_row, n_samples, heads, tokens, head_dim, out_dim, ctypes.c_void_p(out_ptr),
                                   ctypes.c_void_p(stream)))


def finalize_per_key(groups: Sequence[DaamKeyGroup], x, n_rows: int, normalize: bool, out_ptr: int, stream: int):
    _finalize('daam_finalize_per_key', groups, x, n_rows, normalize, out_ptr, stream)


def word_heat_map(maps_ptr: int, n_rows: int, x, rows: Sequence[int], out_ptr: int, stream: int):
    h, w = map_size(x)
    arr = (ctypes.c_int32 * max(len(rows), 1))(*rows)
    _check(load().daam_word_heat_map(ctypes.c_void_p(maps_ptr), n_rows, h, w, arr, len(rows), ctypes.c_void_p(out_ptr),
                                     ctypes.c_void_p(stream)))


def expand_as(map_ptr: int, x, out_h: int, out_w: int, absolute: bool, threshold: Optional[float], out_ptr: int,
              scratch_ptr: int, stream: int):
    h, w = map_size(x)
    use_thr = bool(threshold)   # the reference's `if threshold:` (daam/heatmap.py:87)
    _check(load().daam_expand_as(ctypes.c_void_p(map_ptr), h, w, out_h, out_w, int(bool(absolute)), int(use_thr),
                                 float(threshold) if use_thr else 0.0, ctypes.c_void_p(out_ptr),
                                 ctypes.c_void_p(scratch_ptr), ctypes.c_void_p(stream)))


def _word_list(x, rows_per_word: Sequence[Sequence[int]], out_h: int, out_w: int, absolute: bool,
               threshold: Optional[float]):
    """The arguments every word-list entry point takes after its map and row counts: ``h, w, rows, row_begin, n_words,
    out_h, out_w, absolute, use_threshold, threshold``. ``rows_per_word[w]``: the rows word ``w`` averages (already
    offset for SOS); word ``w`` owns ``rows[row_begin[w] .. row_begin[w + 1])``."""
    h, w = map_size(x)
    flat = [r for rows in rows_per_word for r in rows]
    begin = [0]
    for rows in rows_per_word:
        begin.append(begin[-1] + len(rows))
    use_thr = bool(threshold)   # the reference's `if threshold:` (daam/heatmap.py:87)
    return (h, w, (ctypes.c_int32 * max(len(flat), 1))(*flat), (ctypes.c_int32 * len(begin))(*begin), len(rows_per_word),
            out_h, out_w, int(bool(absolute)), int(use_thr), float(threshold) if use_thr else 0.0)


def expand_words(maps_ptr: int, n_rows: int, x, rows_per_word: Sequence[Sequence[int]], out_h: int, out_w: int,
                 absolute: bool, threshold: Optional[float], word_maps_ptr: Optional[int], out_ptr: int, scratch_ptr: int,
                 stream: int):
    """``daam_expand_words``; ``rows_per_word`` as for :func:`_word_list`."""
    _check(load().daam_expand_words(ctypes.c_void_p(maps_ptr), n_rows,
                                    *_word_list(x, rows_per_word, out_h, out_w, absolute, threshold),
                                    ctypes.c_void_p(word_maps_ptr) if word_maps_ptr else None,
                                    ctypes.c_void_p(out_ptr), ctypes.c_void_p(scratch_ptr), ctypes.c_void_p(stream)))


def segment_words(maps_ptr: int, n_maps: int, n_rows: int, x, rows_per_word: Sequence[Sequence[int]], out_h: int,
                  out_w: int, absolute: bool, threshold: Optional[float], word_maps_ptr: int, labels_ptr: int,
                  scores_ptr: int, scratch_ptr: int, stream: int):
    """``daam_segment_words`` over ``n_maps`` maps ``[n_rows, h, w]`` back to back."""
    _check(load().daam_segment_words(ctypes.c_void_p(maps_ptr), n_maps, n_rows,
                                     *_word_list(x, rows_per_word, out_h, out_w, absolute, threshold),
                                     ctypes.c_void_p(word_maps_ptr), ctypes.c_void_p(labels_ptr),
                                     ctypes.c_void_p(scores_ptr), ctypes.c_void_p(scratch_ptr), ctypes.c_void_p(stream)))


def region_overlap(maps_ptr: int, n_maps: int, n_rows: int, x, rows_per_word: Sequence[Sequence[int]], out_h: int,
                   out_w: int, absolute: bool, threshold: Optional[float], word_maps_ptr: int, regions_ptr: int,
                   n_regions: int, intersection_ptr: int, word_area_ptr: int, scratch_ptr: int, stream: int):
    """``daam_region_overlap`` over ``n_maps`` maps ``[n_rows, h, w]`` back to back and ``n_regions`` uint8 regions
    ``[out_h, out_w]``."""
    _check(load().daam_region_overlap(ctypes.c_void_p(maps_ptr), n_maps, n_rows,
                                      *_word_list(x, rows_per_word, out_h, out_w, absolute, threshold),
                                      ctypes.c_void_p(word_maps_ptr), ctypes.c_void_p(regions_ptr), n_regions,
                                      ctypes.c_void_p(intersection_ptr), ctypes.c_void_p(word_area_ptr),
                                      ctypes.c_void_p(scratch_ptr), ctypes.c_void_p(stream)))


def region_sweep(maps_ptr: int, n_maps: int, n_rows: int, x, rows_per_word: Sequence[Sequence[int]], out_h: int,
                 out_w: int, absolute: bool, thresholds: Sequence[float], word_maps_ptr: int, regions_ptr: int,
                 n_regions: int, intersection_ptr: int, word_area_ptr: int, scratch_ptr: int, stream: int):
    """``daam_region_sweep`` over ``n_maps`` maps ``[n_rows, h, w]`` back to back and ``n_regions`` uint8 regions
    ``[out_h, out_w]``, at ``thresholds`` (passed as a host fp32 array): ``intersection`` ``[n_maps, T, n_regions,
    n_words]``, ``word_area`` ``[n_maps, T, n_words]``."""
    taus = (ctypes.c_float * max(len(thresholds), 1))(*thresholds)
    _check(load().daam_region_sweep(ctypes.c_void_p(maps_ptr), n_maps, n_rows,
                                    *_word_list(x, rows_per_word, out_h, out_w, absolute, None)[:-2],
                                    taus, len(thresholds), ctypes.c_void_p(word_maps_ptr), ctypes.c_void_p(regions_ptr),
                                    n_regions, ctypes.c_void_p(intersection_ptr), ctypes.c_void_p(word_area_ptr),
                                    ctypes.c_void_p(scratch_ptr), ctypes.c_void_p(stream)))


def region_ranking(maps_ptr: int, n_maps: int, n_rows: int, x, rows_per_word: Sequence[Sequence[int]], out_h: int,
                   out_w: int, absolute: bool, threshold: Optional[float], word_maps_ptr: int, regions_ptr: int,
                   n_regions: int, u2_ptr: int, ap_ptr: int, scratch_ptr: int, scratch_bytes: int, stream: int):
    """``daam_region_ranking`` over ``n_maps`` maps ``[n_rows, h, w]`` back to back and ``n_regions`` uint8 regions
    ``[out_h, out_w]``: ``u2`` int64 and ``ap`` float64 ``[n_maps, n_regions, n_words]``; ``scratch_bytes`` of scratch,
    at least :func:`region_ranking_scratch_bytes` of one plane. The values are taken without threshold: the call takes
    no ``use_threshold`` (``threshold`` is ignored)."""
    vp = ctypes.c_void_p
    _check(load().daam_region_ranking(vp(maps_ptr), n_maps, n_rows,
                                      *_word_list(x, rows_per_word, out_h, out_w, absolute, None)[:-2],
                                      vp(word_maps_ptr), vp(regions_ptr), n_regions, vp(u2_ptr), vp(ap_ptr),
                                      vp(scratch_ptr), scratch_bytes, vp(stream)))


def word_overlap(maps_ptr: int, n_maps: int, n_rows: int, x, rows_per_word: Sequence[Sequence[int]], out_h: int,
                 out_w: int, absolute: bool, threshold: Optional[float], word_maps_ptr: int, intersection_ptr: int,
                 word_area_ptr: int, scratch_ptr: int, stream: int):
    """``daam_word_overlap`` over ``n_maps`` maps ``[n_rows, h, w]`` back to back: ``intersection`` ``[n_maps, n_words,
    n_words]``, ``word_area`` ``[n_maps, n_words]``."""
    _check(load().daam_word_overlap(ctypes.c_void_p(maps_ptr), n_maps, n_rows,
                                    *_word_list(x, rows_per_word, out_h, out_w, absolute, threshold),
                                    ctypes.c_void_p(word_maps_ptr), ctypes.c_void_p(intersection_ptr),
                                    ctypes.c_void_p(word_area_ptr), ctypes.c_void_p(scratch_ptr), ctypes.c_void_p(stream)))


def word_instances(maps_ptr: int, n_maps: int, n_rows: int, x, rows_per_word: Sequence[Sequence[int]], out_h: int,
                   out_w: int, absolute: bool, threshold: float, max_instances: int, word_maps_ptr: int, count_ptr: int,
                   area_ptr: int, box_ptr: int, sum_yx_ptr: int, peak_ptr: int, peak_yx_ptr: int, scratch_ptr: int,
                   scratch_bytes: int, stream: int):
    """``daam_word_instances`` over ``n_maps`` maps ``[n_rows, h, w]`` back to back: ``count`` int32 ``[n_maps,
    n_words]``, then per kept instance ``area`` int32, ``box`` int32 ``[4]``, ``sum_yx`` int64 ``[2]``, ``peak`` fp32 and
    ``peak_yx`` int32 ``[2]`` (``[n_maps, n_words, max_instances, ...]``); ``scratch_bytes`` of scratch, at least
    :func:`word_instances_plane_bytes`. The threshold is always in effect: the call takes no ``use_threshold``."""
    vp = ctypes.c_void_p
    _check(load().daam_word_instances(vp(maps_ptr), n_maps, n_rows,
                                      *_word_list(x, rows_per_word, out_h, out_w, absolute, threshold)[:-2],
                                      float(threshold), max_instances, vp(word_maps_ptr), vp(count_ptr), vp(area_ptr),
                                      vp(box_ptr), vp(sum_yx_ptr), vp(peak_ptr), vp(peak_yx_ptr), vp(scratch_ptr),
                                      scratch_bytes, vp(stream)))


def overlay_words(maps_ptr: int, n_maps: int, n_rows: int, x, rows_per_word: Sequence[Sequence[int]], out_h: int,
                  out_w: int, absolute: bool, threshold: Optional[float], color_normalize: bool, word_maps_ptr: int,
                  image_ptr: int, image_map_stride: int, frames_ptr: int, scratch_ptr: int, stream: int):
    """``daam_overlay_words`` over ``n_maps`` maps ``[n_rows, h, w]`` back to back; ``image_ptr`` uint8 ``[out_h, out_w,
    3]``, map ``i``'s at ``image_ptr + i * image_map_stride`` bytes (0: one image for all); ``frames_ptr`` a buffer of
    :func:`overlay_frames_bytes` bytes."""
    _check(load().daam_overlay_words(ctypes.c_void_p(maps_ptr), n_maps, n_rows,
                                     *_word_list(x, rows_per_word, out_h, out_w, absolute, threshold),
                                     int(bool(color_normalize)), ctypes.c_void_p(word_maps_ptr),
                                     ctypes.c_void_p(image_ptr), image_map_stride, ctypes.c_void_p(frames_ptr),
                                     ctypes.c_void_p(scratch_ptr), ctypes.c_void_p(stream)))


def region_boundary(maps_ptr: int, n_maps: int, n_rows: int, x, rows_per_word: Sequence[Sequence[int]], out_h: int,
                    out_w: int, absolute: bool, threshold: float, tolerances: Sequence[float], word_maps_ptr: int,
                    regions_ptr: int, n_regions: int, word_boundary_ptr: int, region_boundary_ptr: int,
                    word_hits_ptr: int, region_hits_ptr: int, max_d2_ptr: int, sum_dist_ptr: int, scratch_ptr: int,
                    scratch_bytes: int, stream: int):
    """``daam_region_boundary`` over ``n_maps`` maps ``[n_rows, h, w]`` back to back and ``n_regions`` uint8 regions
    ``[out_h, out_w]``: ``word_boundary`` int32 ``[n_maps, n_words]``, ``region_boundary`` int32 ``[n_regions]``,
    ``word_hits`` / ``region_hits`` int32 ``[n_maps, T, n_regions, n_words]``, ``max_d2`` int64 and ``sum_dist`` float64
    ``[n_maps, n_regions, n_words, 2]``; ``scratch_bytes`` of scratch, at least :func:`boundary_scratch_bytes` of one
    plane. The threshold is always in effect: the call takes no ``use_threshold``."""
    vp = ctypes.c_void_p
    tol = (ctypes.c_float * max(len(tolerances), 1))(*tolerances)
    _check(load().daam_region_boundary(vp(maps_ptr), n_maps, n_rows,
                                       *_word_list(x, rows_per_word, out_h, out_w, absolute, None)[:-2],
                                       float(threshold), tol, len(tolerances), vp(word_maps_ptr), vp(regions_ptr),
                                       n_regions, vp(word_boundary_ptr), vp(region_boundary_ptr), vp(word_hits_ptr),
                                       vp(region_hits_ptr), vp(max_d2_ptr), vp(sum_dist_ptr), vp(scratch_ptr),
                                       scratch_bytes, vp(stream)))


def mask_boundary(masks_ptr: int, n_planes: int, out_h: int, out_w: int, regions_ptr: int, n_regions: int,
                  tolerances: Sequence[float], word_boundary_ptr: int, region_boundary_ptr: int, word_hits_ptr: int,
                  region_hits_ptr: int, max_d2_ptr: int, sum_dist_ptr: int, scratch_ptr: int, scratch_bytes: int,
                  stream: int):
    """``daam_mask_boundary`` over ``n_planes`` uint8 masks ``[out_h, out_w]`` back to back: the outputs of
    :func:`region_boundary` with ``n_maps * n_words`` replaced by ``n_planes``."""
    vp = ctypes.c_void_p
    tol = (ctypes.c_float * max(len(tolerances), 1))(*tolerances)
    _check(load().daam_mask_boundary(vp(masks_ptr), n_planes, out_h, out_w, vp(regions_ptr), n_regions, tol,
                                     len(tolerances), vp(word_boundary_ptr), vp(region_boundary_ptr),
                                     vp(word_hits_ptr), vp(region_hits_ptr), vp(max_d2_ptr), vp(sum_dist_ptr),
                                     vp(scratch_ptr), scratch_bytes, vp(stream)))


def word_distance(maps_ptr: int, n_maps: int, n_rows: int, x, rows_per_word: Sequence[Sequence[int]], out_h: int,
                  out_w: int, absolute: bool, threshold: float, word_maps_ptr: int, signed_d2_ptr: int, scratch_ptr: int,
                  scratch_bytes: int, stream: int):
    """``daam_word_distance`` over ``n_maps`` maps ``[n_rows, h, w]`` back to back: ``signed_d2`` int32 ``[n_maps,
    n_words, out_h, out_w]``; ``scratch_bytes`` of scratch, at least :func:`distance_plane_bytes`. The threshold is
    always in effect: the call takes no ``use_threshold``."""
    vp = ctypes.c_void_p
    _check(load().daam_word_distance(vp(maps_ptr), n_maps, n_rows,
                                     *_word_list(x, rows_per_word, out_h, out_w, absolute, None)[:-2],
                                     float(threshold), vp(word_maps_ptr), vp(signed_d2_ptr), vp(scratch_ptr),
                                     scratch_bytes, vp(stream)))


def mask_distance(masks_ptr: int, n_planes: int, out_h: int, out_w: int, signed_d2_ptr: int, stream: int):
    """``daam_mask_distance`` over ``n_planes`` uint8 masks ``[out_h, out_w]`` back to back: ``signed_d2`` int32
    ``[n_planes, out_h, out_w]``; no scratch."""
    vp = ctypes.c_void_p
    _check(load().daam_mask_distance(vp(masks_ptr), n_planes, out_h, out_w, vp(signed_d2_ptr), vp(stream)))


def refine_words(maps_ptr: int, n_maps: int, n_rows: int, x, rows_per_word: Sequence[Sequence[int]], out_h: int,
                 out_w: int, absolute: bool, threshold: Optional[float], radius: int, eps: float, word_maps_ptr: int,
                 image_ptr: int, image_map_stride: int, out_ptr: int, scratch_ptr: int, scratch_bytes: int, stream: int):
    """``daam_refine_words`` over ``n_maps`` maps ``[n_rows, h, w]`` back to back; ``image_ptr`` uint8 ``[out_h, out_w,
    3]``, map ``i``'s at ``image_ptr + i * image_map_stride`` bytes (0: one image for all); ``out`` fp32 ``[n_maps,
    n_words, out_h, out_w]``; ``scratch_bytes`` of scratch, at least :func:`refine_scratch_bytes` ``(1, 1, ...)``."""
    vp = ctypes.c_void_p
    _check(load().daam_refine_words(vp(maps_ptr), n_maps, n_rows,
                                    *_word_list(x, rows_per_word, out_h, out_w, absolute, threshold), int(radius),
                                    float(eps), vp(word_maps_ptr), vp(image_ptr), image_map_stride, vp(out_ptr),
                                    vp(scratch_ptr), scratch_bytes, vp(stream)))


def segment_crf(maps_ptr: int, n_maps: int, n_rows: int, x, rows_per_word: Sequence[Sequence[int]], out_h: int,
                out_w: int, absolute: bool, threshold: Optional[float], scale: float, iterations: int, radius: int,
                appearance: float, sigma_xy: float, sigma_rgb: float, smoothness: float, sigma_smooth: float,
                word_maps_ptr: int, image_ptr: int, image_map_stride: int, labels_ptr: int, scores_ptr: int,
                probs_ptr: int, scratch_ptr: int, scratch_bytes: int, stream: int):
    """``daam_segment_crf`` over ``n_maps`` maps ``[n_rows, h, w]`` back to back; ``image_ptr`` uint8 ``[out_h, out_w,
    3]``, map ``i``'s at ``image_ptr + i * image_map_stride`` bytes (0: one image for all); ``labels`` uint8 and
    ``scores`` fp32 ``[n_maps, out_h, out_w]``; ``probs_ptr`` fp32 ``[n_maps, L, out_h, out_w]`` or 0;
    ``scratch_bytes`` of scratch, at least :func:`crf_scratch_bytes` ``(1, L, ...)``."""
    vp = ctypes.c_void_p
    _check(load().daam_segment_crf(vp(maps_ptr), n_maps, n_rows,
                                   *_word_list(x, rows_per_word, out_h, out_w, absolute, threshold), float(scale),
                                   int(iterations), int(radius), float(appearance), float(sigma_xy), float(sigma_rgb),
                                   float(smoothness), float(sigma_smooth), vp(word_maps_ptr), vp(image_ptr),
                                   image_map_stride, vp(labels_ptr), vp(scores_ptr), vp(probs_ptr) if probs_ptr else None,
                                   vp(scratch_ptr), scratch_bytes, vp(stream)))


def image_superpixels(image_ptr: int, n_images: int, out_h: int, out_w: int, n_segments: int, compactness: float,
                      iterations: int, superpixels_ptr: int, scratch_ptr: int, scratch_bytes: int, stream: int):
    """``daam_image_superpixels`` over ``n_images`` uint8 images ``[out_h, out_w, 3]`` back to back: ``superpixels``
    int32 ``[n_images, out_h, out_w]``; ``scratch_bytes`` of scratch, at least :func:`superpixel_image_bytes`."""
    vp = ctypes.c_void_p
    _check(load().daam_image_superpixels(vp(image_ptr), n_images, out_h, out_w, int(n_segments), float(compactness),
                                         int(iterations), vp(superpixels_ptr), vp(scratch_ptr), scratch_bytes,
                                         vp(stream)))


def segment_superpixels(maps_ptr: int, n_maps: int, n_rows: int, x, rows_per_word: Sequence[Sequence[int]],
                        out_h: int, out_w: int, absolute: bool, threshold: Optional[float], n_segments: int,
                        compactness: float, iterations: int, word_maps_ptr: int, image_ptr: int,
                        image_map_stride: int, labels_ptr: int, scores_ptr: int, superpixels_ptr: int,
                        scratch_ptr: int, scratch_bytes: int, stream: int):
    """``daam_segment_superpixels`` over ``n_maps`` maps ``[n_rows, h, w]`` back to back; ``image_ptr`` uint8
    ``[out_h, out_w, 3]``, map ``i``'s at ``image_ptr + i * image_map_stride`` bytes (0: one image for all); ``labels``
    uint8 and ``scores`` fp32 ``[n_maps, out_h, out_w]``; ``superpixels`` int32 ``[out_h, out_w]`` (one image) or
    ``[n_maps, out_h, out_w]``; ``scratch_bytes`` of scratch, at least :func:`superpixel_scratch_bytes` ``(1, 1,
    ...)``."""
    vp = ctypes.c_void_p
    _check(load().daam_segment_superpixels(vp(maps_ptr), n_maps, n_rows,
                                           *_word_list(x, rows_per_word, out_h, out_w, absolute, threshold),
                                           int(n_segments), float(compactness), int(iterations), vp(word_maps_ptr),
                                           vp(image_ptr), image_map_stride, vp(labels_ptr), vp(scores_ptr),
                                           vp(superpixels_ptr), vp(scratch_ptr), scratch_bytes, vp(stream)))


def jet_colormap():
    """``daam_jet_colormap``: the fp32 ``[256, 3]`` colour table the overlay kernel reads, as a CPU tensor."""
    import torch
    out = torch.empty((256, 3), dtype=torch.float32)
    _check(load().daam_jet_colormap(ctypes.c_void_p(out.data_ptr())))
    return out


def device_info():
    sm, major, minor = ctypes.c_int32(), ctypes.c_int32(), ctypes.c_int32()
    _check(load().daam_device_info(ctypes.byref(sm), ctypes.byref(major), ctypes.byref(minor)))
    return {'sm_count': sm.value, 'cc': (major.value, minor.value)}


def launch_count() -> int:
    return int(load().daam_launch_count())


def abi_version() -> int:
    return int(load().daam_abi_version())
