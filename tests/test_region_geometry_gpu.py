"""The ranking, boundary and CRF kernels (daam_b200/csrc/ranking.cu, boundary.cu, crf.cu) against float64 at every
sort, segment, scan, tile, label-chunk and round geometry they accept.

``daam_region_ranking`` radix-sorts each plane in 4096-key tiles whose digit counts are scanned 4096 at a time, cuts
the sorted order into 1024-position segments (one warp each, 32 positions a step) and carries the tie group open at a
segment's start across segments. ``daam_region_boundary`` / ``daam_mask_boundary`` walk columns in blocks of 128 and
query rows in tiles of ``DAAM_BOUNDARY_TILE_ROWS`` rows, 8 warps a tile, scanning 32 columns a step. ``daam_segment_crf``
stages a 32 x 8 tile with its halo and the labels in chunks of ``chunk_size(L)``, and ping-pongs Q between two scratch
buffers and ``probs``. All three split their planes (CRF: maps) into rounds that fit the scratch. :func:`plan` restates
these rules; none of them depends on the SM count. :func:`regimes` names what each case reaches, and
``test_region_geometry_host.py`` checks every case's tags and the coverage of ``REQUIRED`` without a GPU.

Every case goes through the C ABI. Where the word map fits the 200 KB word-map limit, the values are planted exactly:
each word is one token of a global map at the output size in absolute mode, where the bicubic taps are (0, 1, 0, 0),
and the case first asserts that ``expand_words`` gives back the planted planes bit for bit. Larger planes (65536
pixels and up, and the 1024 x 1024 CRF) are upsampled random maps. Either way the case is checked against
``tests/ranking64.py``, ``tests/boundary64.py`` or ``tests/crf64.py`` of the values ``expand_words`` returned: integer
outputs exactly, ``ap`` within ``ap_bound``, ``sum_dist`` within ``sum_bound``, one CRF update at a time within
``crf_bound`` and CRF labels wherever the top-two margin is safe. Every output and the scratch have runs of 0xA5 bytes
before and after them, and every output element must be written; the global maps have NaN rows and maps around the
selected ones; a call split into rounds must give the bits of one round.

No value ``expand_words`` produces is -0: a word map is a sum that starts from +0, and so is every bicubic sum, and an
exactly zero fp32 sum that starts from +0 is +0. ``descending_key``'s fold of -0 onto +0 is therefore not reachable
through the C ABI; ``rank-zeros`` asserts that its large groups of exact zeros hold no -0."""
from __future__ import annotations

import zlib
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import numpy as np
import pytest
import torch

from daam_b200 import _native
from tests.boundary64 import as_stack, boundary64, sum_bound
from tests.crf64 import crf_bound, crf_step64, crf_tables, logits64, softmax64
from tests.ranking64 import ap_bound, ranking64_all

pytestmark = pytest.mark.gpu
DEV = 'cuda'

SORT_TILE = 4096             # kSortTile: keys per digit-count tile
SEGMENT = 1024               # kRankSegment: sorted positions per warp of the group kernels
SCAN_STEP = 4096             # digit counts per step of rank_scan_kernel (1024 threads x 4)
CHUNK = 32                   # sorted positions per ballot of load_chunk; columns per step of nearest_d2
QUERY_WARPS = 8              # kQueryWarps
COLUMN_THREADS = 128         # kColumnThreads
BOUNDARY_TILE_BYTES = 10080  # kBoundaryTileBytes
CRF_TILE_H, CRF_TILE_W = 8, 32
CRF_MAX_RADIUS = 16
MAX_ROUND_PLANES = 65535     # planes (CRF: maps) per round, at most
CRF_WEIGHTS = dict(appearance=10.0, sigma_xy=8.0, sigma_rgb=13.0, smoothness=1.0, sigma_smooth=3.0)
CRF_SCALE = 16.0


# ---- the launch rules, restated ----------------------------------------------------------------------------------------

def cdiv(a: int, b: int) -> int:
    return -(-a // b)


def ranking_plane_bytes(h: int, w: int) -> int:
    """ranking_planes_in's buffers for one plane: part_s and part_ap (8 B x 64 per segment), pre, keys and the two
    idx arrays (4 B a pixel each), the digit counts (256 per tile), seg_cnt and seg_pre (4 B x 64 per segment),
    seg_start (4 B per segment), n_pos (64) and the min / max partials (64 floats)."""
    n = h * w
    tiles, segs = cdiv(n, SORT_TILE), cdiv(n, SEGMENT)
    return 2 * 8 * 64 * segs + 4 * 4 * n + 4 * 256 * tiles + 2 * 4 * 64 * segs + 4 * segs + 4 * 64 + 4 * 64


def boundary_tile_rows(w: int) -> int:
    return 16 if w >= 256 else cdiv(4096, w)


def boundary_plane_bytes(h: int, w: int) -> int:
    """boundary_planes_in's per-plane buffers: the tiles' partials, pre and g (4 B a pixel each, rounded up to 8 B a
    pair of pixels so that the next plane's 8-byte arrays stay aligned) and the min / max partials."""
    return BOUNDARY_TILE_BYTES * cdiv(h, boundary_tile_rows(w)) + 16 * cdiv(h * w, 2) + 256


def boundary_call_bytes(n_regions: int, h: int, w: int) -> int:
    return n_regions * 8 * cdiv(h * w, 2)               # the regions' column distances, 8-byte aligned


def chunk_size(n_labels: int) -> int:
    """crf.cu's chunk_size: the fewest chunks of at most 16 labels, each padded to a multiple of 4."""
    chunks = cdiv(n_labels, 16)
    return cdiv(cdiv(n_labels, chunks), 4) * 4


def step_smem(radius: int, kc: int) -> int:
    return 4 * (kc + 1) * (CRF_TILE_H + 2 * radius) * (CRF_TILE_W + 2 * radius)


def crf_map_bytes(n_labels: int, h: int, w: int) -> int:
    return 2 * 4 * n_labels * h * w + 4 * 64 * n_labels   # two Q buffers and 64 min / max floats per label


def plane_rounds(n_maps: int, n_words: int, cap: int) -> List[Tuple[int, int, int, int]]:
    """The rounds ``(map0, nm, w0, nw)`` of daam_region_ranking / daam_region_boundary (and daam_mask_boundary, one word
    per map) for ``cap`` planes of scratch: whole maps while a map's planes fit, else the words of one map in groups."""
    cap = min(cap, MAX_ROUND_PLANES)
    maps_per_round, words_per_round = max(1, cap // n_words), min(cap, n_words)
    return [(m0, min(maps_per_round, n_maps - m0), w0, min(words_per_round, n_words - w0))
            for m0 in range(0, n_maps, maps_per_round) for w0 in range(0, n_words, words_per_round)]


def crf_rounds(n_maps: int, scratch_bytes: int, map_bytes: int) -> List[Tuple[int, int]]:
    per = min(scratch_bytes // map_bytes, MAX_ROUND_PLANES, n_maps)
    return [(m0, min(per, n_maps - m0)) for m0 in range(0, n_maps, per)]


def scan_steps(w: int, x: int, candidates) -> int:
    """The 32-column steps nearest_d2 takes for a query at column ``x`` of a row whose set pixels are ``candidates``,
    ``(dx, d2)`` pairs: it stops once the next step's smallest dx^2 reaches the best d2 found so far."""
    reach, steps, off, best = max(x, w - 1 - x), 0, 0, float('inf')
    while off <= reach:
        steps += 1
        best = min([best] + [d2 for dx, d2 in candidates if off <= dx < off + CHUNK])
        if (off + CHUNK) ** 2 >= best:
            break
        off += CHUNK
    return steps


# ---- the case description ------------------------------------------------------------------------------------------------

@dataclass
class Case:
    entry: str                            # 'ranking', 'boundary' (daam_region_boundary), 'mask' (daam_mask_boundary)
                                          # or 'crf'
    out: Tuple[int, int]                  # (oh, ow)
    pattern: str                          # how the planes and regions are made (make_data)
    n_words: int = 1                      # mask: planes
    n_maps: int = 1
    n_regions: int = 1
    caps: Tuple[int, ...] = (0,)          # one call per entry: planes (CRF: maps) of scratch per round, 0 for all
    tolerances: Tuple[float, ...] = (0.0, 1.0, 3.0)
    grid: Optional[Tuple[int, int]] = None   # word maps' (mh, mw) when not the output size (values not planted)
    use_threshold: bool = False           # CRF
    radius: int = 4                       # CRF
    updates: Tuple[int, ...] = (0, 1, 2)  # CRF: the updates Q_k -> Q_k+1 checked
    image_per_map: bool = False           # CRF
    tags: Tuple[str, ...] = ()

    @property
    def planes(self) -> int:
        return self.n_maps * self.n_words

    @property
    def n_labels(self) -> int:
        return self.n_words + int(self.use_threshold)


def plan(case: Case) -> dict:
    oh, ow = case.out
    n = oh * ow
    p = dict(n=n)
    if case.entry == 'ranking':
        tiles, segs = cdiv(n, SORT_TILE), cdiv(n, SEGMENT)
        p.update(tiles=tiles, segs=segs, scan_steps=cdiv(256 * tiles, SCAN_STEP), last_seg=n - (segs - 1) * SEGMENT,
                 plane_bytes=ranking_plane_bytes(oh, ow), call_bytes=8 * n)
        p['scratch'] = [p['call_bytes'] + (c or case.planes) * p['plane_bytes'] for c in case.caps]
        p['rounds'] = [plane_rounds(case.n_maps, case.n_words, c or case.planes) for c in case.caps]
        p['reduce_blocks'] = [max(cdiv(nm * nw * case.n_regions, 8) for _, nm, _, nw in r) for r in p['rounds']]
    elif case.entry in ('boundary', 'mask'):
        rows = boundary_tile_rows(ow)
        tiles = cdiv(oh, rows)
        last = oh - (tiles - 1) * rows
        p.update(tile_rows=rows, tiles=tiles, last_rows=last,
                 warp_rows=[len(range(v, last, QUERY_WARPS)) for v in range(QUERY_WARPS)],
                 col_blocks=cdiv(ow, COLUMN_THREADS), plane_bytes=boundary_plane_bytes(oh, ow),
                 call_bytes=boundary_call_bytes(case.n_regions, oh, ow))
        p['scratch'] = [p['call_bytes'] + (c or case.planes) * p['plane_bytes'] for c in case.caps]
        n_maps, n_words = (case.n_words, 1) if case.entry == 'mask' else (case.n_maps, case.n_words)
        p['rounds'] = [plane_rounds(n_maps, n_words, c or case.planes) for c in case.caps]
    else:
        L, r = case.n_labels, case.radius
        kc = chunk_size(L)
        chunks = cdiv(L, kc)
        p.update(kc=kc, chunks=chunks, last_chunk=L - (chunks - 1) * kc, smem=step_smem(r, kc),
                 tiles_y=cdiv(oh, CRF_TILE_H), tiles_x=cdiv(ow, CRF_TILE_W), rem_y=oh % CRF_TILE_H,
                 rem_x=ow % CRF_TILE_W, map_bytes=crf_map_bytes(L, oh, ow))
        p['scratch'] = [(c or case.n_maps) * p['map_bytes'] for c in case.caps]
        p['rounds'] = [crf_rounds(case.n_maps, s, p['map_bytes']) for s in p['scratch']]
    return p


# ---- the planted data (numpy, so that the host test sees the same planes) ------------------------------------------------

def from_keys(keys: np.ndarray) -> np.ndarray:
    """The fp32 values whose descending_key is ``keys`` (uint32): the inverse of ``~orderable(f)``."""
    o = ~keys.astype(np.uint32)
    u = np.where(o & np.uint32(0x80000000), o & np.uint32(0x7FFFFFFF), ~o).astype(np.uint32)
    return u.view(np.float32)


KEY_BASES = {0: (0x3A5C7100, 0, 256), 1: (0x9B2E0055, 0, 256), 2: (0x41000077, 0, 256), 3: (0x00123456, 0x48, 0x7F)}


def forced_groups(n: int) -> Tuple[List[Tuple[int, int]], List[int]]:
    """Tie groups ``[a, b)`` of sorted positions planted in a plane of ``n`` pixels, and the extra group starts: single
    pixels at 0 and n - 1, a group straddling a 32-position chunk, one ending at 1024 k - 1 and the next starting at
    1024 k, one starting at a segment's last position and one covering whole segments."""
    spans = [(0, 1), (n - 1, n)]
    if n > 100:
        spans.append((90, 100))
    if n > 4 * SEGMENT:
        spans += [(2 * SEGMENT - 7, 2 * SEGMENT), (2 * SEGMENT, 2 * SEGMENT + 40), (3 * SEGMENT - 1, 3 * SEGMENT + 3)]
    if n > 8 * SEGMENT:
        spans.append((4 * SEGMENT - 100, 7 * SEGMENT + 10))
    if n > 2 * SEGMENT:
        spans.append((n - SEGMENT - 5, n - SEGMENT + 5))
    return spans, []


def planted_order(n: int, rng: np.random.Generator, negative: bool) -> Tuple[np.ndarray, np.ndarray]:
    """``(values, starts)``: the values by sorted position (descending, fp32) and the group start positions: random
    groups of 1 to 6 positions (a few of 50) around the forced ones."""
    start = np.zeros(n + 1, bool)
    sizes = rng.choice([1, 1, 2, 3, 4, 6, 50], size=n)
    pos = np.cumsum(sizes)
    start[pos[pos < n]] = True
    start[0] = True
    spans, _ = forced_groups(n)
    for a, b in spans:
        start[a + 1:b] = False
        start[a] = True
        start[b] = True
    start = start[:n]
    g = np.cumsum(start) - 1                            # group of each position
    n_groups = int(g[-1]) + 1
    top = n_groups // 2 if negative else n_groups
    values = (top - g).astype(np.float32)               # distinct integers: exact in fp32 up to 2^24
    return values, np.flatnonzero(start)


def region_positions(n: int, n_regions: int, rng: np.random.Generator) -> np.ndarray:
    """``[n_regions, n]`` bool by sorted position: Bernoulli fractions that differ per region, with positives at 0,
    n - 1 and both sides of every segment edge; region 2 empty from three regions on and the last full."""
    frac = np.linspace(0.05, 0.6, n_regions)
    inside = rng.random((n_regions, n)) < frac[:, None]
    edges = np.arange(SEGMENT, n, SEGMENT)
    inside[:, 0] = inside[:, n - 1] = True
    inside[:, edges] = inside[:, edges - 1] = True
    if n_regions >= 3:
        inside[2] = False
    if n_regions >= 2:
        inside[-1] = True
    return inside


def blob_masks(k: int, h: int, w: int, rng: np.random.Generator, empty: Tuple[int, ...] = ()) -> np.ndarray:
    """``k`` uint8 masks: unions of rectangles and scattered pixels, some marked with bytes other than 1; the masks in
    ``empty`` are empty."""
    out = np.zeros((k, h, w), np.uint8)
    for i in range(k):
        if i in empty:
            continue
        for _ in range(1 + i % 3):
            y0, x0 = rng.integers(0, h), rng.integers(0, w)
            y1, x1 = rng.integers(y0 + 1, h + 1), rng.integers(x0 + 1, w + 1)
            out[i, y0:y1, x0:x1] = (1, 7, 255)[i % 3]
        out[i][rng.random((h, w)) < 0.02] = 1
    return out


def crf_image(h: int, w: int, rng: np.random.Generator) -> np.ndarray:
    """A uint8 [h, w, 3] image of flat random-coloured blocks plus a little noise."""
    by, bx = int(rng.integers(2, 12)), int(rng.integers(2, 12))
    blocks = rng.integers(0, 256, (cdiv(h, by), cdiv(w, bx), 3))
    img = blocks.repeat(by, 0).repeat(bx, 1)[:h, :w] + rng.integers(-6, 7, (h, w, 3))
    return np.clip(img, 0, 255).astype(np.uint8)


def make_data(case: Case, name: str) -> dict:
    """``planes`` fp32 ``[n_maps, n_words, oh, ow]`` (mask: uint8 ``[n_words, oh, ow]``; with ``case.grid`` the word maps
    themselves), ``regions`` uint8 ``[R, oh, ow]``, CRF ``images`` ``[n_maps or 1, oh, ow, 3]``; ranking planes also give
    ``order`` (pixel of each sorted position) and ``starts`` (group starts) of their first plane."""
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    oh, ow = case.out
    n = oh * ow
    d: dict = {}
    pat = case.pattern
    if case.entry == 'ranking':
        if case.grid:                                    # word maps on a smaller grid
            mh, mw = case.grid
            wm = rng.standard_normal((case.n_maps, case.n_words, mh, mw)).astype(np.float32)
            if pat == 'zeros':                           # bicubic taps of both signs over zeros and -0
                wm[:, 0] = -0.0                          # word 0: every value 0
                wm[:, 1:, :, : mw // 2] = 0.0            # the others: a zero half next to signed values
                wm[:, 1:, : mh // 2, : mw // 2] = -0.0
            d['planes'] = wm
            d['regions'] = blob_masks(case.n_regions, oh, ow, rng)
            return d
        planes = np.zeros((case.n_maps, case.n_words, n), np.float32)
        inside = None
        for m in range(case.n_maps):
            for w in range(case.n_words):
                if pat.startswith('key byte'):
                    k = int(pat[-1])
                    base, lo, hi = KEY_BASES[k]
                    digits = rng.integers(lo, hi, n).astype(np.uint32)
                    keys = np.uint32(base) & ~np.uint32(0xFF << (8 * k)) | (digits << np.uint32(8 * k))
                    planes[m, w] = from_keys(keys)
                    continue
                values, starts = planted_order(n, rng, negative=(m + w) % 2 == 1)
                order = rng.permutation(n)
                planes[m, w, order] = values
                if m == 0 and w == 0:
                    inside = region_positions(n, case.n_regions, rng)
                    d['order'], d['starts'], d['inside'] = order, starts, inside
        if inside is None:
            d['regions'] = blob_masks(case.n_regions, oh, ow, rng, empty=(2,) if case.n_regions > 2 else ())
        else:
            regions = np.zeros((case.n_regions, n), np.uint8)
            regions[:, d['order']] = inside * np.uint8((1, 7, 255)[0])
            d['regions'] = regions.reshape(case.n_regions, oh, ow)
        d['planes'] = planes.reshape(case.n_maps, case.n_words, oh, ow)
        return d
    if case.entry in ('boundary', 'mask'):
        k = case.planes
        if pat == 'blobs':
            masks = blob_masks(k, oh, ow, rng)
            regions = blob_masks(case.n_regions, oh, ow, rng, empty=tuple(range(2, case.n_regions, 7)))
        elif pat == 'dx 32':                             # columns 0 and w - 1: every query's nearest pixel at dx = 32
            masks = np.zeros((k, oh, ow), np.uint8)
            regions = np.zeros((case.n_regions, oh, ow), np.uint8)
            masks[:, :, 0] = 1
            regions[:, :, ow - 1] = 1
        elif pat == 'second step':                       # first step: dx 1, g 40 (1601); second: dx 33, g 0 (1089)
            masks = np.zeros((k, oh, ow), np.uint8)
            regions = np.zeros((case.n_regions, oh, ow), np.uint8)
            masks[:, 40, 0] = 1
            regions[:, 0, 1] = regions[:, 40, 33] = 1
        elif pat == 'ends':                              # one pixel at each end of a line
            masks = np.zeros((k, n), np.uint8)
            regions = np.zeros((case.n_regions, n), np.uint8)
            masks[:, 0] = 1
            regions[:, n - 1] = 1
            masks, regions = masks.reshape(k, oh, ow), regions.reshape(case.n_regions, oh, ow)
        elif pat == 'tolerance equal to a distance':     # d2 = 25 at tolerance 5, and d2 = 0 at tolerance 0
            masks = np.zeros((k, oh, ow), np.uint8)
            regions = np.zeros((case.n_regions, oh, ow), np.uint8)
            masks[:, 10, 10] = 1
            regions[0, 13, 14] = 1
            regions[1, 10, 10] = 1
        else:
            raise ValueError(pat)
        d['regions'] = regions
        if case.entry == 'mask':
            d['planes'] = masks
        else:                                            # 0 / 1 values against the threshold 0.5
            d['planes'] = masks.reshape(case.n_maps, case.n_words, oh, ow).astype(bool).astype(np.float32)
        return d
    d['planes'] = rng.random((case.n_maps, case.n_words) + (case.grid or case.out), dtype=np.float32)
    d['images'] = np.stack([crf_image(oh, ow, rng) for _ in range(case.n_maps if case.image_per_map else 1)])
    return d


# ---- the cases --------------------------------------------------------------------------------------------------------------

def _rank(out, pattern, tags, **kw):
    return Case('ranking', out, pattern, tags=tuple(tags), **kw)


def _line(n: int) -> Tuple[int, int]:
    return (1, n)


CASES: Dict[str, Case] = {
    # sizes at every sort-tile, segment, chunk and scan-step edge
    **{f'rank-n{n}': _rank(_line(n), 'planted', [f'n {n}'], n_regions=3)
       for n in (1, 31, 32, 33, 1023, 1024, 1025, 4095, 4096, 4097)},
    # past the 200 KB word-map limit the values are upsampled random maps, not planted
    'rank-65536': _rank((256, 256), 'random', ['scan steps 1, 16 tiles'], grid=(128, 128), n_regions=5),
    'rank-65537': _rank(_line(65537), 'random', ['scan steps 2', 'last segment 1 position'], grid=(1, 30000),
                        n_regions=5),
    'rank-1024k+1': _rank((1025, 2049), 'random', ['segs 1024 k + 1', 'scan steps 2'], grid=(128, 160), n_regions=2),
    'rank-2^24': _rank((4096, 4096), 'random', ['plane 2^24', 'u2 up to 2^47', 'segment sum over 2^32'],
                       grid=(128, 128), n_regions=3),
    # planted tie groups over 40 segments, the largest plane that fits the word-map limit
    'rank-groups': _rank((160, 256), 'planted', ['group over whole segments', 'group starts at 1024 k',
                                                 'group starts at a segment\'s last position'], n_regions=5),
    # region counts around the second ballot word
    **{f'rank-regions-{r}': _rank((64, 80), 'planted', [f'regions {r}'], n_regions=r) for r in (1, 31, 32, 33, 63)},
    # orders decided by one key byte
    **{f'rank-key-byte-{k}': _rank((64, 80), f'key byte {k}', [f'key byte {k} only'], n_regions=4) for k in range(4)},
    'rank-zeros': _rank((64, 64), 'zeros', ['exact zeros tied', 'negative values'], grid=(16, 16), n_words=2,
                        n_regions=4),
    # rounds: 3 maps x 5 words at 2 and 10 planes of scratch
    'rank-rounds': _rank((40, 52), 'planted', ['round: words split 2 + 2 + 1', 'round: two maps', 'round: map0 > 0',
                                               'round: all planes'], n_maps=3, n_words=5, n_regions=7,
                         caps=(0, 2, 10)),

    # boundary: widths at every column block and warp edge, heights at every tile edge
    **{f'mask-w{w}-h{h}': Case('mask', (h, w), 'blobs', n_words=2, n_regions=3, tags=tuple(t))
       for w, h, t in ((1, 4097, ['w 1, 4096-row tiles', 'last tile 1 row']), (1, 2, ['w 1, 4096-row tiles']),
                       (31, 134, ['last tile 1 row']), (32, 5, ['single tile < 8 rows']), (33, 126, ['last tile 1 row']),
                       (127, 34, ['last tile 1 row']), (128, 33, ['last tile 1 row', 'column blocks 1']),
                       (129, 33, ['last tile 1 row', 'column blocks 2']), (255, 18, ['last tile 1 row']),
                       (256, 17, ['last tile 1 row', 'tile rows 16']), (257, 40, ['tile rows 16']))},
    'mask-dx32': Case('mask', (3, 33), 'dx 32', n_regions=1, tags=('query at x = 0, dx = 32', 'query at x = w - 1, dx = 32')),
    'mask-second-step': Case('mask', (41, 40), 'second step', tags=('nearest in the second step',)),
    'mask-row-131072': Case('mask', (1, 131072), 'ends', tags=('d2 over 2^32 along a row',)),
    'mask-column-131072': Case('mask', (131072, 1), 'ends', tags=('d2 over 2^32 along a column', 'w 1, 4096-row tiles')),
    'mask-row-2^24': Case('mask', (1, 1 << 24), 'ends', tags=('d2 over 2^47 along a row',)),
    'mask-tolerance-exact': Case('mask', (24, 24), 'tolerance equal to a distance', n_regions=2,
                                 tolerances=(0.0, 4.0, 5.0, 6.0), tags=('tolerance^2 = d2', 'tolerance 0')),
    'mask-63-regions-16-tolerances': Case('mask', (64, 64), 'blobs', n_words=2, n_regions=63,
                                          tolerances=tuple(float(t) for t in range(16)),
                                          tags=('regions 63', 'tolerances 16', 'empty regions')),
    'mask-rounds': Case('mask', (48, 40), 'blobs', n_words=7, n_regions=3, caps=(0, 1, 3),
                        tags=('mask round: one plane', 'mask round: 3 planes, 1 left over')),
    'boundary-rounds': Case('boundary', (48, 40), 'blobs', n_maps=3, n_words=5, n_regions=4, caps=(0, 2, 10),
                            tags=('round: words split 2 + 2 + 1', 'round: two maps', 'round: map0 > 0')),

    # CRF: every kC at one chunk, full and partial
    **{f'crf-L{L}': Case('crf', out, 'random', n_words=L - thr, use_threshold=bool(thr), radius=r, tags=tuple(t))
       for L, thr, out, r, t in ((1, 0, (1, 1), 4, ['out 1x1']), (4, 1, (1, 33), 4, ['out 1x33']),
                                 (5, 0, (33, 1), 4, ['out 33x1']), (8, 1, (9, 33), 4, ['out 9x33']),
                                 (9, 0, (17, 65), 4, ['out 17x65']), (12, 1, (9, 33), 16, ['window > tile']),
                                 (13, 0, (17, 65), 16, ['radius 16, kC 16, small']), (16, 1, (9, 33), 2, []),
                                 # several chunks
                                 (17, 1, (17, 65), 4, []), (24, 0, (9, 33), 4, []), (25, 1, (17, 65), 3, []),
                                 (33, 0, (9, 33), 4, []), (49, 1, (17, 65), 2, []), (64, 0, (9, 33), 1, []))},
    'crf-r16-1024': Case('crf', (1024, 1024), 'random', grid=(128, 128), n_words=15, use_threshold=True, radius=16,
                         updates=(0,),
                         tags=('radius 16, kC 16, 1024x1024',)),
    'crf-rounds': Case('crf', (17, 40), 'random', n_maps=3, n_words=13, image_per_map=True, caps=(0, 1, 2),
                       updates=(0, 1), tags=('crf round: 1 map', 'crf round: 2 maps', 'image per map')),
}
CASE_NAMES = list(CASES)

REQUIRED = (
    [f'n {n}' for n in (1, 31, 32, 33, 1023, 1024, 1025, 4095, 4096, 4097)] +
    ['sort tiles 1', 'sort tiles 2', 'scan steps 1, 16 tiles', 'scan steps 2', 'segs 1024 k + 1', 'plane 2^24',
     'last segment 1 position', 'u2 up to 2^47', 'segment sum over 2^32'] +
    [f'regions {r}' for r in (1, 31, 32, 33, 63)] +
    ['group starts at 1024 k', 'group ends at 1024 k - 1', 'group over whole segments',
     'group starts at a segment\'s last position', 'single-pixel group at 0', 'single-pixel group at n - 1',
     'group straddles a 32-position chunk'] +
    [f'key byte {k} only' for k in range(4)] + ['negative values', 'exact zeros tied'] +
    ['round: words split 2 + 2 + 1', 'round: two maps', 'round: map0 > 0', 'round: all planes'] +
    [f'w {w}' for w in (1, 31, 32, 33, 127, 128, 129, 255, 256)] +
    ['w 1, 4096-row tiles', 'last tile 1 row', 'single tile < 8 rows', 'warp without rows', 'column blocks 1',
     'column blocks 2', 'tile rows 16', 'query at x = 0, dx = 32', 'query at x = w - 1, dx = 32',
     'nearest in the second step', 'd2 over 2^32 along a row', 'd2 over 2^32 along a column',
     'tolerance^2 = d2', 'tolerance 0', 'regions 63', 'tolerances 16', 'empty regions',
     'mask round: one plane', 'mask round: 3 planes, 1 left over'] +
    [f'kC {k} one chunk {f}' for k in (4, 8, 12, 16) for f in ('full', 'partial')] +
    ['chunks 2 (12 + 5)', 'chunks 2 (12 + 12)', 'chunks 2 (16 + 9)', 'chunks 3 (12 + 12 + 9)',
     'chunks 4 (16 x 3 + 1)', 'chunks 4 (16 x 4)', 'radius 16, kC 16, 1024x1024', 'radius 16, kC 16, small',
     'smem 174080', 'out 1x1', 'out 1x33', 'out 33x1', 'out 9x33', 'out 17x65', 'tile remainder 1 on y',
     'tile remainder 1 on x', 'window > tile', 'labels 1', 'iterations 1, 2, 3',
     'crf round: 1 map', 'crf round: 2 maps', 'image per map'])


def _ranking_data_regimes(d: dict, n: int) -> set:
    tags = set()
    s = d.get('starts')
    if s is None:
        return tags
    ends = np.append(s[1:], n) - 1                       # last position of each group
    k = s[(s > 0) & (s % SEGMENT == 0)]
    if len(k):
        tags |= {'group starts at 1024 k', 'group ends at 1024 k - 1'}
    if ((s % SEGMENT) == SEGMENT - 1).any():
        tags.add('group starts at a segment\'s last position')
    if len(s) > 1 and s[1] == 1:
        tags.add('single-pixel group at 0')
    if s[-1] == n - 1 and n > 1:
        tags.add('single-pixel group at n - 1')
    if ((s // CHUNK != ends // CHUNK) & (s // SEGMENT == ends // SEGMENT)).any():
        tags.add('group straddles a 32-position chunk')
    # a segment without a group start, after a segment with positives: seg_start -1 with a nonzero run
    segs = cdiv(n, SEGMENT)
    has_start = np.zeros(segs, bool)
    has_start[s // SEGMENT] = True
    if segs > 1 and not has_start[1:].all():
        tags.add('group over whole segments')
    # rank_groups_kernel's per-segment sum of tp_g (FP_< + FP_<=), for each region of the first plane
    g = np.cumsum(np.isin(np.arange(n), s)) - 1
    seg_of_group = ends // SEGMENT
    for inside in d['inside']:
        tp = np.bincount(g, inside, minlength=len(s))
        fp = np.bincount(g, ~inside, minlength=len(s))
        fp_lt = np.cumsum(fp) - fp
        if np.bincount(seg_of_group, tp * (2 * fp_lt + fp)).max() >= 2.0 ** 32:
            tags.add('segment sum over 2^32')
    return tags


def regimes(case: Case, p: dict, d: Optional[dict] = None) -> set:
    """The regimes ``case`` reaches under plan ``p`` (and its data ``d``, for the ranking planes' tie groups)."""
    oh, ow = case.out
    n = oh * ow
    tags = set()
    if case.entry == 'ranking':
        tags.add(f'n {n}')
        tags.add(f'regions {case.n_regions}')
        if p['tiles'] <= 2:
            tags.add(f'sort tiles {p["tiles"]}')
        if p['scan_steps'] == 1 and p['tiles'] == SCAN_STEP // 256:
            tags.add('scan steps 1, 16 tiles')
        if p['scan_steps'] >= 2:
            tags.add('scan steps 2')
        if p['segs'] > 1 and p['last_seg'] == 1:
            tags |= {'last segment 1 position', 'segs 1024 k + 1'}
        if n == 1 << 24:
            tags.add('plane 2^24')
        if n * n // 2 >= 1 << 47:                         # u2 = 2 n_p n_n reaches n^2 / 2
            tags.add('u2 up to 2^47')
        if n >= 1 << 22 and case.n_regions > 1:            # asserted from the data by the GPU test
            tags.add('segment sum over 2^32')
        if case.pattern.startswith('key byte'):
            tags.add(f'key byte {case.pattern[-1]} only')
            if KEY_BASES[int(case.pattern[-1])][0] & 0x80000000:
                tags.add('negative values')
        if case.pattern == 'planted' and case.planes > 1:
            tags.add('negative values')
        if case.pattern == 'zeros':
            tags |= {'exact zeros tied', 'negative values'}
        if d is not None:
            tags |= _ranking_data_regimes(d, n)
    if case.entry in ('boundary', 'mask'):
        tags.add(f'w {ow}')
        if ow == 1 and p['tile_rows'] == 4096:
            tags.add('w 1, 4096-row tiles')
        if p['tiles'] > 1 and p['last_rows'] == 1:
            tags.add('last tile 1 row')
        if p['tiles'] == 1 and p['last_rows'] < QUERY_WARPS:
            tags.add('single tile < 8 rows')
        if 0 in p['warp_rows']:
            tags.add('warp without rows')
        if p['col_blocks'] <= 2:
            tags.add(f'column blocks {p["col_blocks"]}')
        if p['tile_rows'] == 16:
            tags.add('tile rows 16')
        if case.pattern == 'dx 32' and ow == 33 and scan_steps(ow, 0, [(32, 32 * 32)]) == 2:
            tags |= {'query at x = 0, dx = 32', 'query at x = w - 1, dx = 32'}
        if case.pattern == 'second step' and scan_steps(ow, 0, [(1, 1 + 40 * 40), (33, 33 * 33)]) == 2:
            tags.add('nearest in the second step')
        if case.pattern == 'ends' and (n - 1) ** 2 >= 1 << 32:
            tags.add('d2 over 2^32 along a row' if oh == 1 else 'd2 over 2^32 along a column')
            if (n - 1) ** 2 >= 1 << 47:
                tags.add('d2 over 2^47 along a row')
        if case.pattern == 'tolerance equal to a distance' and 5.0 in case.tolerances:
            tags.add('tolerance^2 = d2')
        if 0.0 in case.tolerances:
            tags.add('tolerance 0')
        if case.n_regions == 63:
            tags.add('regions 63')
        if len(case.tolerances) == 16:
            tags.add('tolerances 16')
        if case.pattern == 'blobs' and case.n_regions > 2:
            tags.add('empty regions')
    if case.entry in ('ranking', 'boundary'):
        for rounds in p['rounds']:
            if len(rounds) == 1:
                tags.add('round: all planes')
            if any(m0 > 0 for m0, _, _, _ in rounds):
                tags.add('round: map0 > 0')
            if any(nm == 2 for _, nm, _, _ in rounds):
                tags.add('round: two maps')
            if [nw for m0, _, _, nw in rounds if m0 == 1] == [2, 2, 1]:
                tags.add('round: words split 2 + 2 + 1')
    if case.entry == 'mask':
        for rounds in p['rounds']:
            sizes = [nm for _, nm, _, _ in rounds]
            if len(sizes) > 1 and set(sizes) == {1}:
                tags.add('mask round: one plane')
            if len(sizes) > 1 and sizes[0] == 3 and sizes[-1] == 1:
                tags.add('mask round: 3 planes, 1 left over')
    if case.entry == 'crf':
        L, kc = case.n_labels, p['kc']
        if p['chunks'] == 1:
            tags.add(f'kC {kc} one chunk {"full" if L == kc else "partial"}')
        else:
            sizes = [kc] * (p['chunks'] - 1) + [p['last_chunk']]
            if len(set(sizes)) == 1:
                tags.add(f'chunks {p["chunks"]} ({" + ".join(map(str, sizes))})' if p['chunks'] == 2
                         else f'chunks {p["chunks"]} ({kc} x {p["chunks"]})')
            elif p['chunks'] == 4:
                tags.add(f'chunks 4 ({kc} x 3 + {p["last_chunk"]})')
            else:
                tags.add(f'chunks {p["chunks"]} ({" + ".join(map(str, sizes))})')
        if L == 1:
            tags.add('labels 1')
        if p['smem'] == 174080:
            tags.add('smem 174080')
        if case.radius == 16 and kc == 16:
            tags.add('radius 16, kC 16, 1024x1024' if n >= 1 << 20 else 'radius 16, kC 16, small')
        tags.add(f'out {oh}x{ow}')
        if p['rem_y'] == 1:
            tags.add('tile remainder 1 on y')
        if p['rem_x'] == 1:
            tags.add('tile remainder 1 on x')
        if case.radius > min(CRF_TILE_H, CRF_TILE_W) and n > 1:
            tags.add('window > tile')
        if max(case.updates) >= 2:
            tags.add('iterations 1, 2, 3')
        for rounds in p['rounds']:
            if len(rounds) > 1 and {nm for _, nm in rounds} == {1}:
                tags.add('crf round: 1 map')
            if len(rounds) > 1 and rounds[0][1] == 2:
                tags.add('crf round: 2 maps')
        if case.image_per_map and case.n_maps > 1:
            tags.add('image per map')
    return tags


def case_regimes(name: str) -> set:
    case = CASES[name]
    return regimes(case, plan(case), make_data(case, name) if case.entry == 'ranking' else None)


# ---- buffers with guards ----------------------------------------------------------------------------------------------------

GUARD = 256                  # sentinel bytes before and after every output and the scratch
SENTINEL = 0xA5


class Guarded:
    """``n`` elements of ``dtype`` prefilled with 0xA5 bytes, with ``GUARD`` more such bytes before and after."""

    def __init__(self, n: int, dtype: torch.dtype):
        size = torch.empty((), dtype=dtype).element_size()
        self.buf = torch.full((2 * GUARD + n * size,), SENTINEL, dtype=torch.uint8, device=DEV)
        self.view = self.buf[GUARD:GUARD + n * size].view(dtype)
        self.size, self.n = size, n

    def ptr(self) -> int:
        return self.view.data_ptr()

    def check(self, what: str, written: bool = True):
        assert bool((self.buf[:GUARD] == SENTINEL).all()) and bool((self.buf[GUARD + self.n * self.size:] == SENTINEL).all()), \
            f'{what}: written outside its buffer'
        if written:
            untouched = (self.buf[GUARD:GUARD + self.n * self.size].view(-1, self.size) == SENTINEL).all(1)
            assert not bool(untouched.any()), f'{what}: {int(untouched.sum())} elements not written'


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def global_maps(planes: np.ndarray) -> torch.Tensor:
    """``[n_maps, n_words + 2, h, w]`` device global maps, word ``w`` in row ``w + 1``: rows 0 and ``n_words + 1`` and a
    map before and after the stack are NaN."""
    n_maps, n_words = planes.shape[:2]
    buf = torch.full((n_maps + 2, n_words + 2) + planes.shape[2:], float('nan'), device=DEV)
    buf[1:-1, 1:-1] = torch.from_numpy(planes).to(DEV)
    return buf[1:-1]


def rows_of(n_words: int) -> List[List[int]]:
    return [[w + 1] for w in range(n_words)]


def expanded(case: Case, maps: torch.Tensor, planted: Optional[np.ndarray]) -> np.ndarray:
    """expand_words' absolute values of every map ``[n_maps, n_words, oh, ow]``; with ``planted``, asserted to be the
    planted planes bit for bit."""
    oh, ow = case.out
    grid = tuple(maps.shape[-2:])
    out = torch.empty((case.n_maps, case.n_words, oh, ow), device=DEV)
    wm = torch.empty((case.n_words,) + grid, device=DEV)
    scratch = torch.empty(_native.EXPAND_SCRATCH_FLOATS * case.n_words, device=DEV)
    for m in range(case.n_maps):
        _native.expand_words(maps[m].data_ptr(), maps.shape[1], grid, rows_of(case.n_words), oh, ow, True, None,
                             wm.data_ptr(), out[m].data_ptr(), scratch.data_ptr(), _stream())
    got = out.cpu().numpy()
    if planted is not None:
        assert np.array_equal(got.view(np.int32), planted.view(np.int32)), \
            'expand_words did not give back the planted planes: the taps at the output size are not (0, 1, 0, 0)'
    return got


def _scratch(nbytes: int) -> Guarded:
    return Guarded(cdiv(nbytes, 8), torch.float64)      # 8-byte aligned; its guards must hold, its contents are free


# ---- ranking ------------------------------------------------------------------------------------------------------------

def run_ranking(case: Case, maps: torch.Tensor, regions: torch.Tensor, scratch_bytes: int) -> Tuple[np.ndarray, np.ndarray]:
    oh, ow = case.out
    shape = (case.n_maps, case.n_regions, case.n_words)
    u2, ap = Guarded(int(np.prod(shape)), torch.int64), Guarded(int(np.prod(shape)), torch.float64)
    wm = Guarded(case.planes * int(np.prod(maps.shape[-2:])), torch.float32)
    scratch = _scratch(scratch_bytes)
    _native.region_ranking(maps.data_ptr(), case.n_maps, maps.shape[1], tuple(maps.shape[-2:]), rows_of(case.n_words),
                           oh, ow, True, None, wm.ptr(), regions.data_ptr(), case.n_regions, u2.ptr(), ap.ptr(),
                           scratch.ptr(), scratch_bytes, _stream())
    torch.cuda.synchronize()
    for g, what in ((u2, 'u2'), (ap, 'ap'), (wm, 'word_maps')):
        g.check(f'{what} at {scratch_bytes} scratch bytes')
    scratch.check('scratch', written=False)
    return u2.view.cpu().numpy().reshape(shape), ap.view.cpu().numpy().reshape(shape)


def max_segment_sum(values: np.ndarray, regions: np.ndarray) -> float:
    """The largest per-segment sum of tp_g (FP_< + FP_<=) that rank_groups_kernel accumulates (a group counted in the
    segment of its last position), over the regions of one plane."""
    v = values.reshape(-1).astype(np.float64)
    order = np.argsort(-v, kind='stable')
    sv = v[order]
    start = np.ones(len(sv), bool)
    start[1:] = sv[1:] != sv[:-1]
    g = np.cumsum(start) - 1
    last = np.append(np.flatnonzero(start)[1:], len(sv)) - 1
    best = 0.0
    for inside in regions:
        pos = inside.reshape(-1)[order] != 0
        tp, fp = np.bincount(g, pos), np.bincount(g, ~pos)
        best = max(best, float(np.bincount(last // SEGMENT, tp * (2 * (np.cumsum(fp) - fp) + fp)).max()))
    return best


def check_ranking(name: str, case: Case, d: dict):
    p = plan(case)
    maps = global_maps(d['planes'])
    m = expanded(case, maps, None if case.grid else d['planes'])
    if case.pattern == 'zeros':                        # large tie groups at exactly +0, and never -0 (see the host test)
        zeros = m == 0
        assert zeros.sum() > m.size // 4 and not np.signbit(m[zeros]).any()
    if 'segment sum over 2^32' in case.tags:
        assert max_segment_sum(m[0, 0], d['regions']) >= 2.0 ** 32, \
            f'{name}: no segment sum reaches 2^32'
    regions = torch.from_numpy(d['regions']).to(DEV)
    first = None
    for cap, scratch_bytes in zip(case.caps, p['scratch']):
        u2, ap = run_ranking(case, maps, regions, scratch_bytes)
        if first is not None:
            assert np.array_equal(u2, first[0]) and np.array_equal(ap.view(np.int64), first[1].view(np.int64)), \
                f'{name}: rounds of {cap} planes differ from one round'
            continue
        first = (u2, ap)
        for mi in range(case.n_maps):
            want_u2, want_ap, groups = ranking64_all(m[mi], d['regions'])
            np.testing.assert_array_equal(u2[mi], want_u2, err_msg=f'{name}: u2 of map {mi}')
            nan = np.isnan(want_ap)
            np.testing.assert_array_equal(np.isnan(ap[mi]), nan, err_msg=f'{name}: NaN ap of map {mi}')
            err = np.abs(ap[mi] - want_ap)[~nan]
            bound = np.broadcast_to(ap_bound(want_ap, groups[None]), want_ap.shape)[~nan]
            assert bool((err <= bound).all()), f'{name}: ap of map {mi} off by {err.max():.3e}'
    return p


# ---- boundary ---------------------------------------------------------------------------------------------------------

FIELDS = (('word_boundary', torch.int32), ('region_boundary', torch.int32), ('word_hits', torch.int32),
          ('region_hits', torch.int32), ('max_d2', torch.int64), ('sum_dist', torch.float64))


def run_boundary(case: Case, maps: Optional[torch.Tensor], masks: Optional[torch.Tensor], regions: torch.Tensor,
                 scratch_bytes: int) -> dict:
    """The outputs, plane-major as boundary64 gives them."""
    oh, ow = case.out
    M, W = (case.n_words, 1) if case.entry == 'mask' else (case.n_maps, case.n_words)
    T, R = len(case.tolerances), case.n_regions
    shapes = dict(word_boundary=(M, W), region_boundary=(R,), word_hits=(M, T, R, W), region_hits=(M, T, R, W),
                  max_d2=(M, R, W, 2), sum_dist=(M, R, W, 2))
    out = {f: Guarded(int(np.prod(shapes[f])), dt) for f, dt in FIELDS}
    scratch = _scratch(scratch_bytes)
    ptrs = [out[f].ptr() for f, _ in FIELDS]
    if case.entry == 'mask':
        _native.mask_boundary(masks.data_ptr(), case.n_words, oh, ow, regions.data_ptr(), R, case.tolerances, *ptrs,
                              scratch.ptr(), scratch_bytes, _stream())
    else:
        wm = Guarded(case.planes * oh * ow, torch.float32)
        _native.region_boundary(maps.data_ptr(), case.n_maps, maps.shape[1], (oh, ow), rows_of(case.n_words), oh, ow,
                                True, 0.5, case.tolerances, wm.ptr(), regions.data_ptr(), R, *ptrs, scratch.ptr(),
                                scratch_bytes, _stream())
        torch.cuda.synchronize()
        wm.check('word_maps')
    torch.cuda.synchronize()
    for f, g in out.items():
        g.check(f'{f} at {scratch_bytes} scratch bytes')
    scratch.check('scratch', written=False)
    got = {f: g.view.cpu().numpy().reshape(shapes[f]) for f, g in out.items()}
    return dict(word_boundary=got['word_boundary'].reshape(-1), region_boundary=got['region_boundary'],
                word_hits=got['word_hits'].transpose(0, 3, 1, 2).reshape(M * W, T, R),
                region_hits=got['region_hits'].transpose(0, 3, 1, 2).reshape(M * W, T, R),
                max_d2=got['max_d2'].transpose(0, 2, 1, 3).reshape(M * W, R, 2),
                sum_dist=got['sum_dist'].transpose(0, 2, 1, 3).reshape(M * W, R, 2))


def check_boundary(name: str, case: Case, d: dict):
    p = plan(case)
    regions = torch.from_numpy(d['regions']).to(DEV)
    maps = masks = None
    if case.entry == 'mask':
        masks = torch.from_numpy(d['planes']).to(DEV)
        inside = d['planes'] != 0
    else:
        maps = global_maps(d['planes'])
        inside = expanded(case, maps, d['planes']).reshape(-1, *case.out) > 0.5
    want = boundary64(inside, d['regions'], case.tolerances)
    first = None
    for cap, scratch_bytes in zip(case.caps, p['scratch']):
        got = run_boundary(case, maps, masks, regions, scratch_bytes)
        if first is not None:
            for f, _ in FIELDS:
                a, b = got[f], first[f]
                assert np.array_equal(a.view(np.int64) if a.dtype == np.float64 else a,
                                      b.view(np.int64) if b.dtype == np.float64 else b), \
                    f'{name}: {f} of rounds of {cap} planes differs from one round'
            continue
        first = got
        for f, _ in FIELDS[:-1]:
            np.testing.assert_array_equal(got[f], want[f], err_msg=f'{name}: {f}')
        err = np.abs(got['sum_dist'] - want['sum_dist'])
        bound = sum_bound(as_stack(want, len(inside), 1)).reshape(err.shape)
        assert bool((err <= bound).all()), f'{name}: sum_dist off by {err.max():.3e}'
    return p, want


# ---- CRF ------------------------------------------------------------------------------------------------------------------

def run_crf(case: Case, maps: torch.Tensor, images: torch.Tensor, iterations: int, probs: bool, scratch_bytes: int):
    oh, ow = case.out
    n, L = oh * ow, case.n_labels
    labels, scores = Guarded(case.n_maps * n, torch.uint8), Guarded(case.n_maps * n, torch.float32)
    q = Guarded(case.n_maps * L * n, torch.float32) if probs else None
    wm = Guarded(case.planes * int(np.prod(maps.shape[-2:])), torch.float32)
    scratch = _scratch(scratch_bytes)
    stride = oh * ow * 3 if case.image_per_map else 0
    _native.segment_crf(maps.data_ptr(), case.n_maps, maps.shape[1], tuple(maps.shape[-2:]), rows_of(case.n_words), oh, ow, True,
                        0.5 if case.use_threshold else None, CRF_SCALE, iterations, case.radius, **CRF_WEIGHTS,
                        word_maps_ptr=wm.ptr(), image_ptr=images.data_ptr(), image_map_stride=stride,
                        labels_ptr=labels.ptr(), scores_ptr=scores.ptr(), probs_ptr=q.ptr() if probs else 0,
                        scratch_ptr=scratch.ptr(), scratch_bytes=scratch_bytes, stream=_stream())
    torch.cuda.synchronize()
    for g, what in ((labels, 'labels'), (scores, 'scores'), (wm, 'word_maps')) + (((q, 'probs'),) if probs else ()):
        g.check(f'{what} at {iterations} iterations')
    scratch.check('scratch', written=False)
    out = [labels.view.cpu().numpy().reshape(case.n_maps, oh, ow), scores.view.cpu().numpy().reshape(case.n_maps, oh, ow)]
    return out + ([q.view.cpu().numpy().reshape(case.n_maps, L, oh, ow)] if probs else [])


def crf_bands(h: int, rows: int = 8):
    if h <= 3 * rows:
        return [(0, h)]
    mid = h // 2 - rows // 2
    return [(0, rows), (mid, mid + rows), (h - rows, h)]


def check_crf(name: str, case: Case, d: dict):
    p = plan(case)
    maps = global_maps(d['planes'])
    m = expanded(case, maps, None if case.grid else d['planes'])
    images = torch.from_numpy(d['images']).to(DEV)
    L, off = case.n_labels, 0 if case.use_threshold else 1
    thr = 0.5 if case.use_threshold else None
    tab = crf_tables(case.radius, **CRF_WEIGHTS)
    full = p['scratch'][0]
    runs = {k: run_crf(case, maps, images, k, True, full) for k in sorted(set(case.updates) | {u + 1 for u in case.updates} | {0})}
    for k, (lab, sc, q) in runs.items():
        # without probs the last update lands in q_a or q_b: the same bits
        lab2, sc2 = run_crf(case, maps, images, k, False, full)
        assert np.array_equal(lab, lab2) and np.array_equal(sc.view(np.int32), sc2.view(np.int32)), \
            f'{name}: {k} iterations without probs differ from with probs'
        assert np.array_equal(sc, np.take_along_axis(q, (lab.astype(np.int64) - off)[:, None], 1)[:, 0]), \
            f'{name}: scores are not the Q of the label at {k} iterations'
    for mi in range(case.n_maps):
        z = logits64(m[mi], thr, CRF_SCALE)
        image = d['images'][mi if case.image_per_map else 0]
        bound, _ = crf_bound(dict(t=z, mass=np.zeros_like(z)), case.radius)
        assert bool((np.abs(runs[0][2][mi] - softmax64(z)) <= bound).all()), f'{name}: Q_0 of map {mi}'
        for k in case.updates:
            q_k, q_next, lab_next = runs[k][2][mi].astype(np.float64), runs[k + 1][2][mi], runs[k + 1][0][mi]
            for y0, y1 in crf_bands(case.out[0]):
                ref, parts = crf_step64(z, q_k, image, tab, case.radius, rows=(y0, y1), parts=True)
                bound, dt = crf_bound(parts, case.radius)
                err = np.abs(q_next[:, y0:y1] - ref)
                assert bool((err <= bound).all()), f'{name}: map {mi} update {k} rows {y0}-{y1}: error {err.max():.3e}, ' \
                                                   f'worst ratio {(err / bound).max():.3f}'
                t = np.sort(parts['t'], 0)
                sure = t[-1] - t[-2] > 2 * dt if L > 1 else np.ones(dt.shape, bool)
                want = parts['t'].argmax(0) + off
                assert np.array_equal(lab_next[y0:y1][sure], want[sure]), f'{name}: labels of map {mi} update {k}'
    for cap, scratch_bytes in zip(case.caps[1:], p['scratch'][1:]):
        k = max(case.updates) + 1
        got = run_crf(case, maps, images, k, True, scratch_bytes)
        for a, b, what in zip(got, runs[k], ('labels', 'scores', 'probs')):
            assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), f'{name}: {what} of rounds of {cap} maps'
    return p


# ---- the test ---------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('name', CASE_NAMES)
def test_case_against_float64(name):
    case = CASES[name]
    d = make_data(case, name)
    p = plan(case)
    missing = set(case.tags) - regimes(case, p, d if case.entry == 'ranking' else None)
    assert not missing, f'{name}: the case no longer reaches {sorted(missing)}'
    if case.entry == 'ranking':
        check_ranking(name, case, d)
    elif case.entry in ('boundary', 'mask'):
        _, want = check_boundary(name, case, d)
        if case.pattern == 'tolerance equal to a distance':        # region 0 is hit at 5 and not at 4; region 1 at 0
            assert want['word_hits'][0, :, 0].tolist() == [0, 0, 1, 1] and want['word_hits'][0, 0, 1] == 1
        if case.pattern == 'second step':
            assert want['max_d2'][0, 0, 0] == 33 * 33
        if case.pattern in ('dx 32', 'ends'):
            assert want['max_d2'][0, 0, 0] == (case.out[1] - 1 if case.out[0] == 1 or case.pattern == 'dx 32'
                                               else case.out[0] - 1) ** 2
    else:
        check_crf(name, case, d)
