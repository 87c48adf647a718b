"""The word-list kernels (daam_b200/csrc/words.cu) against float64 at every chunk, pass, window and tile geometry they
accept.

``expand_words_kernel`` splits each word's output pixels into chunks whose min / max meet across a grid barrier;
``segment_minmax_kernel`` does the same for the tile kernels, whose CTAs stage the source windows under a 16 x 64
output tile for a pass of words (one pass when they fit in 48 KB, one word per pass up to 200 KB), interpolate from
tap tables, and (overlay) compute the pixel after a tile row when its last 4-byte word reaches past it. The pair and
sweep kernels keep their own buffers in shared memory and stage windows only in what is left of 200 KB, or none (then
they interpolate from the word maps in global memory); the pair kernel walks tiles ``c, c + 256, ...`` per CTA and,
without a threshold, stages its windows again for every 256-pixel chunk; ``daam_word_instances`` splits its (map, word)
planes into rounds that fit its scratch and labels each round's masks in 32 x 32 tiles (components.cu). :func:`plan`
restates the launch rules for a call; the cases are built from it and each asserts the regimes it names, so that a
change of a rule cannot move a case to another regime unnoticed. Every case goes through the C ABI (a few also
through ``GlobalHeatMap`` / ``GlobalHeatMapStack``) and is checked

* against the float64 pipeline of ``tests/words64.py`` under its error bound ``expand_bound``: expand / expand_as
  element-wise, the word maps, segment labels and scores, region counts (thresholded: between the sure and the
  possible counts) and sums, overlay bytes (inside the range the composition gives over the bounded map); elements
  within the bound of a threshold or a tie are left out, and there must be few of them;
* pair, sweep and instances against ``expand_words`` of the same maps, itself checked against float64 in the case:
  pair and sweep counts equal the int64 counts of its masks bit for bit and lie between the float64 sure and possible
  counts, pair sums without a threshold lie within a bound derived from their summation depth, instances equal
  ``tests/components64.py`` of its values at every round split;
* for stray writes and wrong-row reads: every unselected row of the global maps and a whole map before and after the
  stack are NaN, every output and the scratch have sentinel runs before and after them, and some frames start 4 bytes
  past a 16-byte boundary;
* for its launch count.

``plan`` also places a delta word map's float64 argmax (and argmin) at the first and last pixel of every min / max
chunk of a 1-word call, so that a chunk that skips a pixel at its ends changes lo / hi. Three regimes cannot occur,
and ``test_unreachable_regimes`` in ``test_word_geometry_host.py`` says why: several ``expand_words`` launches on an
H100, an empty expand chunk, and a round of several maps whose words are split."""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import numpy as np
import pytest
import torch

from daam_b200 import _native
from tests.components64 import components64, instances64_stack
from tests.reference64 import bicubic64
from tests.words64 import U, bound_for, fp32, row_mean_bound, threshold_unsure

pytestmark = pytest.mark.gpu
DEV = 'cuda'

THREADS = 256                # threads of every word-list CTA
TILE_H, TILE_W = 16, 64      # kSegTileH x kSegTileW: a tile kernel's output tile
STAGE_FLOATS = 12288         # kSegStageFloats: staged windows per pass when they fit (48 KB)
MAX_CHUNKS = 32              # kWordChunks
MAX_SMEM = 200 * 1024        # kMaxSmem
SM_SMEM = 228 * 1024         # shared memory of an H100 SM; 1 KB of it is reserved per CTA
N_ROWS = 40                  # rows of a synthetic global map: more than any word selects (map_stride > selected rows)
THRESHOLDS = (None, 0, 0.4)


# ---- the case description ---------------------------------------------------------------------------------------------

@dataclass
class Case:
    entry: str                            # 'expand', 'expand_as', 'segment', 'region', 'overlay', 'pair', 'sweep' or
                                          # 'instances'
    grid: Tuple[int, int]                 # the word maps' (mh, mw)
    out: Tuple[int, int]                  # the output's (oh, ow)
    n_words: int = 1
    n_maps: int = 1
    absolute: bool = False
    thresholds: Tuple = (None,)           # sweep: the ascending thresholds of one call; instances: one call each
    color_normalize: bool = True
    n_regions: int = 1
    image_per_map: bool = False
    frames_shift: int = 0                 # bytes the frames start past a 16-byte boundary
    planted: bool = False                 # delta word maps at every chunk end (1 word)
    k: int = 16                           # instances: max_instances
    scratch_planes: Tuple[int, ...] = (0,)   # instances: one call per scratch size, in planes (0: every plane)
    zero_word: bool = False               # the last word's rows are 0: m = 0 at every pixel (absolute)
    pattern: Optional[str] = None         # 'diagonals': crafted 0 / 1 word maps (diagonal_word_maps)
    api: bool = False                     # also through GlobalHeatMap / GlobalHeatMapStack
    tags: Tuple[str, ...] = ()

    def rows_per_word(self) -> List[List[int]]:
        """Word ``i`` selects one row, every third word two; rows 0, 1 and the last rows are never selected."""
        out = []
        for i in range(self.n_words):
            r = 2 + (7 * i) % (N_ROWS - 6)
            out.append([r, r + 1] if i % 3 == 2 else [r])
        return out


# ---- the launch rules, restated -------------------------------------------------------------------------------------------

def taps_floor(dst: np.ndarray, n_in: int, n_out: int) -> np.ndarray:
    """``floor(src)`` of ``make_taps`` in fp32 (the product and the subtraction rounded separately)."""
    scale = np.float32(n_in) / np.float32(n_out)
    src = np.float32(scale * (dst.astype(np.float32) + np.float32(0.5))) - np.float32(0.5)
    return np.floor(src).astype(np.int64)


def expand_per_sm(mh: int, mw: int) -> int:
    """CTAs of ``expand_words_kernel`` an SM holds, as far as shared memory and threads limit them (an upper bound of
    the occupancy query; exact at one CTA per SM)."""
    return max(1, min(2048 // THREADS, SM_SMEM // (mh * mw * 4 + 64 + 1024)))


def tile_windows(case: Case) -> dict:
    """Every tile's ``(th, tw)`` and actual window ``(wh, ww)`` (``block_tile``), per axis."""
    (mh, mw), (oh, ow) = case.grid, case.out
    out = {}
    for axis, (n_in, n_out, t) in (('y', (mh, oh, TILE_H)), ('x', (mw, ow, TILE_W))):
        y0 = np.arange(0, n_out, t)
        th = np.minimum(t, n_out - y0)
        first = np.clip(taps_floor(y0, n_in, n_out) - 1, 0, n_in - 1)
        last = np.clip(taps_floor(y0 + th - 1, n_in, n_out) + 2, 0, n_in - 1)
        unclamped = (taps_floor(y0, n_in, n_out) - 1 < 0) | (taps_floor(y0 + th - 1, n_in, n_out) + 2 > n_in - 1)
        out[axis] = dict(t=th, win=last - first + 1, clamped=bool(unclamped.any()))
    return out


PAIR_CTAS = 256               # kPairCtas: word_pair_tile_kernel's CTAs per map, at most one per tile
PAIR_MASK_STRIDE = 33        # kPairMaskStride
PAIR_CHUNK = 256             # kPairChunk: pixels per step without a threshold
MAX_ROUND_PLANES = 65535     # daam_word_instances: planes per round, at most (grid.y of the components launches)
CC_TILE = 32                 # kCcTile: the labelling tile of components.cu
INSTANCE_LAUNCHES = 7        # per round: segment_minmax_kernel, instance_mask_kernel and the five of components.cu


def pair_smem_bytes(n_words: int, use_threshold: bool) -> int:
    """``pair_smem_floats``: the pair table (two bytes a pair), the slots' partials, and the masks (threshold) or the
    values of a 256-pixel chunk, before word_pair_tile_kernel's windows."""
    pairs = n_words * (n_words + 1) // 2
    return 4 * ((pairs + 1) // 2 + pairs + n_words + n_words * (PAIR_MASK_STRIDE if use_threshold else PAIR_CHUNK))


def sweep_smem_bytes(n_regions: int, n_thresholds: int) -> int:
    """``sweep_smem_floats``: region_sweep_tile_kernel's two histograms of a word, before its windows."""
    return 4 * 2 * (n_regions + 1) * n_thresholds


def words_per_pass(n_words, win, smem_before: Optional[int]):
    """``launch_tiles``: without ``smem_before``, as many windows as fit in 48 KB, at least one; with it, as many as fit
    in 200 KB beside it, possibly none (the kernel then reads the word maps). ``win`` may be an array."""
    if smem_before is None:
        return np.maximum(1, np.minimum(n_words, STAGE_FLOATS // win))
    return np.minimum(n_words, (MAX_SMEM - smem_before) // (4 * win))


def instance_rounds(n_maps: int, n_words: int, cap: int) -> List[Tuple[int, int, int, int]]:
    """``daam_word_instances``'s rounds ``(map0, maps, word0, words)`` for ``cap`` planes of scratch: whole maps while a
    map's planes fit, else the words of one map in groups."""
    maps_per_round, words_per_round = max(1, cap // n_words), min(cap, n_words)
    return [(m0, min(maps_per_round, n_maps - m0), w0, min(words_per_round, n_words - w0))
            for m0 in range(0, n_maps, maps_per_round) for w0 in range(0, n_words, words_per_round)]


def tile_plan(case: Case, n_maps: int, n_words: int, sm_count: int, smem_before: Optional[int] = None) -> dict:
    """``launch_tiles`` for ``n_maps`` maps of ``n_words`` words: ``chunks`` (``ceil(4 sm_count / (n_maps n_words))``,
    at most 32 and one per 256 pixels, 1 without the min / max), the window estimate ``win_h x win_w``,
    ``words_per_pass``, ``passes`` (1 when the windows are not staged) and the dynamic shared memory ``smem``."""
    (mh, mw), (oh, ow) = case.grid, case.out
    n = oh * ow
    minmax = not case.absolute or (case.entry == 'overlay' and case.color_normalize)
    mwords = n_maps * n_words
    chunks = min(MAX_CHUNKS, -(-4 * sm_count // mwords), -(-n // 256))
    if chunks < 1 or not minmax:
        chunks = 1
    win_h = min(mh, math.ceil(TILE_H * mh / oh) + 5)
    win_w = min(mw, math.ceil(TILE_W * mw / ow) + 5)
    wpp = int(words_per_pass(n_words, win_h * win_w, smem_before))
    return dict(minmax=minmax, mwords=mwords, chunks=chunks, per=-(-n // chunks), win_h=win_h, win_w=win_w,
                words_per_pass=wpp, passes=-(-n_words // wpp) if wpp else 1,
                fits=(MAX_SMEM - smem_before) // (4 * win_h * win_w) if smem_before is not None else None,
                smem=(smem_before or 0) + wpp * win_h * win_w * 4)


def plan(case: Case, sm_count: int) -> dict:
    """What the host does with ``case``:

    * expand: ``launches`` (words per launch: ``capacity = per_sm * sm_count``), ``chunks = min(32, capacity //
      n_words, ceil(n / 256))`` and ``chunks_asserted`` (at most 4 words: ``min(32, ceil(n / 256))`` on any device of
      132 or more SMs, whatever the occupancy);
    * tiles: :func:`tile_plan` and the tiles' actual windows; ``launches`` 2 (segment, overlay) or 3 (region);
    * pair: per threshold of the case (``by_t``), :func:`tile_plan` beside ``pair_smem_bytes`` and ``restage`` (no
      threshold, several passes: the windows are staged again for every 256-pixel chunk); ``ctas = min(tiles, 256)``
      per map, CTA ``c`` walking tiles ``c, c + ctas, ...`` (``walk`` of them at most); 3 launches;
    * sweep: :func:`tile_plan` beside ``sweep_smem_bytes``; 3 launches (the memset of the histograms is not one);
    * instances: per scratch size (``splits``), ``cap = min(scratch_bytes // plane_bytes, 65535)``, the rounds and a
      :func:`tile_plan` per round (its own maps and words); 7 launches a round."""
    (mh, mw), (oh, ow) = case.grid, case.out
    n = oh * ow
    p = dict(n=n)
    if case.entry in ('expand', 'expand_as'):
        per_sm = expand_per_sm(mh, mw)
        capacity = per_sm * sm_count
        batch = min(case.n_words, capacity)
        chunks = max(1, min(MAX_CHUNKS, capacity // batch, -(-n // 256)))
        p.update(per_sm=per_sm, capacity=capacity, launches=-(-case.n_words // capacity), chunks=chunks,
                 chunks_asserted=min(MAX_CHUNKS, -(-n // 256)) if case.n_words <= 4 and sm_count >= 132 else None,
                 per=-(-n // chunks))
        return p
    p['tiles'] = tile_windows(case)
    if case.entry == 'pair':
        tiles = len(p['tiles']['y']['t']) * len(p['tiles']['x']['t'])
        ctas = min(tiles, PAIR_CTAS)
        p.update(tile_count=tiles, ctas=ctas, walk=-(-tiles // ctas), launches=3, by_t={})
        for t in case.thresholds:
            q = tile_plan(case, case.n_maps, case.n_words, sm_count, pair_smem_bytes(case.n_words, bool(t)))
            q['restage'] = not t and 0 < q['words_per_pass'] < case.n_words
            p['by_t'][t] = q
        return p
    if case.entry == 'sweep':
        p.update(tile_plan(case, case.n_maps, case.n_words, sm_count,
                           sweep_smem_bytes(case.n_regions, len(case.thresholds))), launches=3)
        return p
    if case.entry == 'instances':
        plane = _native.word_instances_plane_bytes(oh, ow)
        p.update(plane_bytes=plane, splits=[])
        for planes in case.scratch_planes:
            planes = planes or case.n_maps * case.n_words
            cap = min(planes * plane // plane, MAX_ROUND_PLANES)
            rounds = instance_rounds(case.n_maps, case.n_words, cap)
            p['splits'].append(dict(planes=planes, cap=cap, rounds=rounds, launches=INSTANCE_LAUNCHES * len(rounds),
                                    maps_per_round=max(1, cap // case.n_words),
                                    words_per_round=min(cap, case.n_words),
                                    tiles=[tile_plan(case, nm, nw, sm_count) for _, nm, _, nw in rounds]))
        return p
    p.update(tile_plan(case, case.n_maps, case.n_words, sm_count), launches=3 if case.entry == 'region' else 2)
    return p


def _ratio_tags(n_in: int, n_out: int) -> set:
    if n_in == n_out:
        return {'ratio identity'}
    big, small = max(n_in, n_out), min(n_in, n_out)
    dyadic = big % small == 0 and (big // small) & (big // small - 1) == 0
    return {f'{"up" if n_out > n_in else "down"} {"dyadic" if dyadic else "non-dyadic"}', f'ratio {n_in}->{n_out}'}


def overlay_carries(case: Case) -> set:
    """Where the pixel after a tile row lies when that row's last 4-byte word of frames reaches past it: 'tile'
    (the next tile of the row), 'row', 'word', 'map' or 'past the last map'."""
    oh, ow = case.out
    kinds = set()
    x_end = np.minimum(np.arange(0, ow, TILE_W) + TILE_W, ow)
    for mp in range(case.n_maps):
        for w in range(case.n_words):
            for y in range(oh):
                nxt = ((mp * case.n_words + w) * oh + y) * ow + x_end       # the next pixel's index, per tile
                for x, i in zip(x_end, nxt):
                    if (3 * i) % 4 == 0:                                     # case.frames_shift is a multiple of 4
                        continue
                    if x < ow:
                        kinds.add('tile')
                    elif y + 1 < oh:
                        kinds.add('row')
                    elif w + 1 < case.n_words:
                        kinds.add('word')
                    elif mp + 1 < case.n_maps:
                        kinds.add('map')
                    else:
                        kinds.add('past the last map')
    return kinds


def regimes(case: Case, p: dict) -> set:
    """The regimes a call reaches, as the tags the cases name."""
    (mh, mw), (oh, ow) = case.grid, case.out
    tags = _ratio_tags(mh, oh) | _ratio_tags(mw, ow)
    if (oh, ow) == (1, 1):
        tags.add('out 1x1')
    if (mh, mw) == (1, 1):
        tags.add('map 1x1')
    elif mh == 1:
        tags.add('map 1xN')
    elif mw == 1:
        tags.add('map Nx1')
    if (mh, mw) == (2, 3):
        tags.add('map 2x3')
    if mh != mw:
        tags.add('map non-square')
    if mh * mw * 4 == MAX_SMEM:
        tags.add('map 200 KB')
    if case.entry in ('expand', 'expand_as'):
        c, n = p['chunks'], p['n']
        tags.add(f'expand chunks {c}')
        if n == 256 * (c - 1) + 1:
            tags.add('expand chunks c at n = 256 (c - 1) + 1')
        if n == 256 * c:
            tags.add('expand chunks c at n = 256 c')
        if case.n_words == 96:
            tags.add('expand 96 words, one CTA per SM' if p['per_sm'] == 1 else f'expand 96 words on {mh}x{mw}')
        if p['launches'] > 1:
            tags.add('expand several launches')
        if case.planted:
            tags.add('planted expand chunk ends')
        return tags
    if case.entry in ('pair', 'sweep', 'instances'):
        return tags | consumer_regimes(case, p)
    tags.add(f'{case.entry}')
    if case.n_maps > 1:
        tags.add(f'stack {case.entry}')
    c = p['chunks']
    if c == 1:
        tags.add('tile chunks 1 (no min / max)' if not p['minmax'] else
                 'tile chunks 1 (mwords >= 4 SMs)' if p['mwords'] >= 4 * SM_FOR_TAGS[0] else 'tile chunks 1')
    else:
        tags.add('tile chunks 32' if c == MAX_CHUNKS else 'tile chunks in between')
    if case.planted:
        tags.add('planted tile chunk ends')
    tags.add('one pass' if p['passes'] == 1 else 'several passes')
    if p['passes'] > 1 and case.n_words % p['words_per_pass']:
        tags.add('partial last pass')
    if p['words_per_pass'] == 1 and case.n_words == 96:
        tags.add('one word per pass, 96 words')
    if p['win_h'] * p['win_w'] > STAGE_FLOATS:
        tags.add('window > 12288 floats')
    if p['smem'] > 48 * 1024:
        tags.add('dynamic smem > 48 KB')
    ty, tx = p['tiles']['y'], p['tiles']['x']
    if ty['clamped'] or tx['clamped']:
        tags.add('window clamped at a border')
    whole_y, whole_x = bool((ty['win'] == mh).all()), bool((tx['win'] == mw).all())
    if whole_y and whole_x:
        tags.add('window: whole map')
    elif whole_y or whole_x:
        tags.add('window: whole map on one axis')
    for t in set(ty['t'].tolist()) & {16, 15, 1}:
        tags.add(f'th {t}')
    for t in set(tx['t'].tolist()) & {64, 63, 1}:
        tags.add(f'tw {t}')
    if oh < TILE_H and ow < TILE_W:
        tags.add('output smaller than a tile')
    if case.entry == 'region':
        tags.add(f'regions {case.n_regions}')
    if case.entry == 'overlay':
        tags.add(f'3 ow mod 4 = {3 * ow % 4}')
        tags |= {f'carry: {k}' for k in overlay_carries(case)}
        tags.add('image per map' if case.image_per_map else 'one image for all maps')
        if case.frames_shift % 16:
            tags.add('frames 4-byte aligned only')
    return tags


SM_FOR_TAGS = [132]          # the SM count regimes() names 'mwords >= 4 SMs' against (set by the caller)


def diagonal_word_maps(case: Case) -> np.ndarray:
    """``[n_words, mh, mw]`` 0 / 1 maps: even words anti-diagonal lines ``y + x = 0 mod 9`` (each pixel's only
    neighbours on its line are NE and SW, so a line crosses a labelling-tile seam only through a NE pair), odd words
    diagonal lines ``x - y = 0 mod 11`` (NW and SE)."""
    mh, mw = case.grid
    y, x = np.mgrid[:mh, :mw]
    anti, diag = (y + x) % 9 == 0, (x - y) % 11 == 0
    return np.stack([anti if w % 2 == 0 else diag for w in range(case.n_words)]).astype(np.float32)


def _shared_tile_tags(case: Case, q: dict) -> set:
    """The staging and tile-shape tags of one tile launch, as the segment, region and overlay cases name them."""
    ty, tx = tile_windows(case)['y'], tile_windows(case)['x']
    tags = {f'th {t}' for t in set(ty['t'].tolist()) & {16, 15, 1}} | \
        {f'tw {t}' for t in set(tx['t'].tolist()) & {64, 63, 1}}
    if q['words_per_pass']:
        tags.add('one pass' if q['passes'] == 1 else 'several passes')
        if q['passes'] > 1 and case.n_words % q['words_per_pass']:
            tags.add('partial last pass')
    if q['win_h'] * q['win_w'] > STAGE_FLOATS:
        tags.add('window > 12288 floats')
    if q['smem'] > 48 * 1024:
        tags.add('dynamic smem > 48 KB')
    if case.grid[0] * case.grid[1] * 4 == MAX_SMEM:
        tags.add('map 200 KB')
    return tags


def consumer_regimes(case: Case, p: dict) -> set:
    """The regimes of the pair, sweep and instances entries, each tag prefixed with its entry where the other entries
    name the same regime."""
    e, (oh, ow) = case.entry, case.out
    ty, tx = p['tiles']['y']['t'], p['tiles']['x']['t']
    tile_pixels = np.outer(ty, tx).ravel()
    tags = {e}
    if case.n_maps > 1:
        tags.add(f'stack {e}')
    if e == 'pair':
        for t, q in p['by_t'].items():
            tags |= {f'pair {x}' for x in _shared_tile_tags(case, q) - {'several passes'}}
            if q['words_per_pass'] == 0:
                tags.add(f'pair windows not staged, {"threshold" if t else "no threshold"}')
            if q['passes'] > 1:
                tags.add('pair several passes' if t else
                         'pair restaged per chunk' if q['restage'] and tile_pixels.max() > PAIR_CHUNK else
                         'pair several passes, one chunk a tile')
        tags.add('pair ctas = tiles' if p['tile_count'] <= PAIR_CTAS else 'pair several tiles per CTA')
        if p['tile_count'] > PAIR_CTAS and p['tile_count'] % PAIR_CTAS:
            tags.add('pair uneven tiles per CTA')
        if (tile_pixels < PAIR_CHUNK).any():
            tags.add('pair tile of < 256 pixels')
        if (tile_pixels == 1).any():
            tags.add('pair tile 1x1')
        if case.n_words in (1, 96):
            tags.add(f'pair {case.n_words} word{"s" if case.n_words > 1 else ""}')
        return tags
    if e == 'sweep':
        taus = [fp32(t) for t in case.thresholds]
        tags |= {f'sweep {x}' for x in _shared_tile_tags(case, p)}
        if p['words_per_pass'] == 0:
            tags.add('sweep windows not staged')
        elif p['fits'] == 1:
            tags.add('sweep exactly one window fits')
        tags.add(f'sweep thresholds {len(taus)}')
        tags.add(f'sweep regions {case.n_regions}')
        if not case.absolute and max(taus) < 0.99:
            tags.add('sweep bucket T')                    # m of a normalised word reaches 1 - 1e-7 at its max of v
        if case.zero_word and case.absolute:
            if min(taus) >= 0:
                tags.add('sweep bucket 0 only')           # m = 0 everywhere for the zero word
            if 0 in taus:
                tags.add('sweep threshold equal to a pixel value')
        if (tile_pixels % 32).any():
            tags.add('sweep warp partly outside the tile')
        return tags
    for s in p['splits']:
        for (_, _, _, nw), q in zip(s['rounds'], s['tiles']):
            shared = _shared_tile_tags(case, q) - {'partial last pass'}
            if nw == 1:
                shared.discard('one pass')
            tags |= {f'instances {x}' for x in shared}
            if q['words_per_pass'] == 1 and nw > 1:
                tags.add('instances one word per pass')
        if s['cap'] == 1:
            tags.add('round: one plane')
        if s['words_per_round'] < case.n_words and case.n_words % s['words_per_round']:
            tags.add('round: words split, partial last round')
        if s['maps_per_round'] == 1 and s['words_per_round'] == case.n_words and s['cap'] > case.n_words:
            tags.add('round: one map, planes left over')
        if any(nm > 1 for _, nm, _, _ in s['rounds']):
            tags.add('round: several maps')
        if len(s['rounds']) == 1:
            tags.add('round: all planes')
    if (oh, ow) == (1, 1):
        tags.add('cc out 1x1')
    elif oh == 1:
        tags.add('cc out 1xN')
    elif ow == 1:
        tags.add('cc out Nx1')
    if ow > 1 and ow % CC_TILE == 1:
        tags.add('cc last tile 1 column')
    if oh > 1 and oh % CC_TILE == 1:
        tags.add('cc last tile 1 row')
    if oh <= CC_TILE and ow <= CC_TILE:
        tags.add('cc single tile')
    if case.k in (1, 64):
        tags.add(f'instances K {case.k}')
    t = case.thresholds[0]
    if t >= 0 and (((oh, ow) == (1, 1) and not case.absolute) or (case.zero_word and case.absolute)):
        tags.add('count 0')                               # a normalised 1-pixel map is 0; so is the zero word
    if case.pattern == 'diagonals' and case.absolute and case.grid == case.out:     # m is the word map itself
        masks = diagonal_word_maps(case) > t
        if max(len(components64(m)['root']) for m in masks) > case.k:
            tags.add('count > K')
    return tags


# ---- the cases ----------------------------------------------------------------------------------------------------------

def spread(n: int) -> Tuple[float, ...]:
    """``n`` ascending sweep thresholds from -0.05 to 0.85: every pixel of a normalised word passes the first, and
    the pixels near its max pass the last."""
    return tuple(-0.05 + 0.9 * i / max(n - 1, 1) for i in range(n))


def _e(grid, out, tags, **kw):
    return Case('expand', grid, out, thresholds=kw.pop('thresholds', THRESHOLDS), tags=tuple(tags), **kw)


CASES: Dict[str, Case] = {
    # expand: chunk counts, maps and ratios
    'expand-out-1x1': _e((64, 64), (1, 1), ['expand chunks 1', 'out 1x1', 'down dyadic']),
    'expand-map-1x1': _e((1, 1), (5, 7), ['map 1x1', 'expand chunks 1'], absolute=True),
    'expand-n256': _e((64, 64), (16, 16), ['expand chunks 1', 'expand chunks c at n = 256 c']),
    'expand-n257-1xN-out': _e((64, 96), (1, 257), ['expand chunks 2', 'expand chunks c at n = 256 (c - 1) + 1',
                                                  'up non-dyadic', 'map non-square']),
    'expand-n512-map-2x3': _e((2, 3), (16, 32), ['expand chunks 2', 'expand chunks c at n = 256 c', 'map 2x3']),
    'expand-n1537-map-1xN': _e((1, 50), (1, 1537), ['expand chunks 7', 'expand chunks c at n = 256 (c - 1) + 1',
                                                   'map 1xN']),
    'expand-n1792-map-Nx1': _e((50, 1), (1792, 1), ['expand chunks 7', 'expand chunks c at n = 256 c', 'map Nx1']),
    'expand-31-chunks': _e((64, 64), (62, 128), ['expand chunks 31', 'expand chunks c at n = 256 c', 'down non-dyadic',
                                                 'up dyadic'], absolute=True),
    'expand-32-chunks-n7937': _e((64, 80), (1, 7937), ['expand chunks 32', 'expand chunks c at n = 256 (c - 1) + 1']),
    'expand-4-words': _e((75, 100), (600, 800), ['expand chunks 32', 'up dyadic'], n_words=4),
    'expand-ratio-64-96': _e((64, 64), (96, 96), ['ratio 64->96', 'up non-dyadic'], n_words=3),
    'expand-ratio-97-1000': _e((97, 97), (1000, 1000), ['ratio 97->1000', 'expand chunks 32']),
    'expand-ratio-320-300': _e((320, 160), (300, 300), ['ratio 320->300', 'map 200 KB', 'down non-dyadic']),
    'expand-96-words-200KB': _e((320, 160), (40, 80), ['expand 96 words, one CTA per SM'], n_words=96,
                                thresholds=(None,)),
    'expand-96-words-64x64': _e((64, 64), (96, 96), ['expand 96 words on 64x64'], n_words=96, thresholds=(None, 0.4)),
    'expand-as-96-40': Case('expand_as', (96, 96), (40, 40), thresholds=THRESHOLDS, tags=('ratio 96->40',)),
    'expand-as-absolute': Case('expand_as', (52, 76), (832, 1216), absolute=True, thresholds=(None, 0.4),
                               tags=('up dyadic',)),
    'expand-planted': _e((96, 96), (90, 90), ['planted expand chunk ends', 'expand chunks 32'], planted=True,
                         thresholds=(None,)),
    'expand-api': _e((64, 96), (512, 768), ['up dyadic'], n_words=5, api=True),
    # segment
    'segment-planted': Case('segment', (96, 96), (90, 90), planted=True,
                            tags=('planted tile chunk ends', 'tile chunks 32')),
    'segment-stack-mwords': Case('segment', (64, 64), (20, 70), n_words=24, n_maps=22, thresholds=(0.4,),
                                 tags=('tile chunks 1 (mwords >= 4 SMs)', 'stack segment', 'several passes')),
    'segment-one-word-per-pass': Case('segment', (128, 128), (17, 65), n_words=96, thresholds=(None,),
                                      tags=('one word per pass, 96 words', 'window > 12288 floats',
                                            'dynamic smem > 48 KB', 'th 16', 'th 1', 'tw 64', 'tw 1')),
    'segment-small-out': Case('segment', (30, 50), (12, 20), n_words=8, thresholds=(None, 0.4),
                              tags=('output smaller than a tile', 'window: whole map')),
    'segment-abs-chunks-1': Case('segment', (64, 96), (31, 127), n_words=3, absolute=True, thresholds=(None, 0.4),
                                 tags=('tile chunks 1 (no min / max)', 'th 15', 'tw 63')),
    'segment-api-stack': Case('segment', (64, 96), (96, 80), n_words=8, n_maps=3, api=True, thresholds=(0.4,),
                              tags=('stack segment', 'tile chunks in between')),
    # region
    'region-1': Case('region', (64, 64), (40, 130), n_words=3, n_regions=1, thresholds=(None,),
                     tags=('regions 1', 'tw 64')),
    'region-31-stack': Case('region', (64, 96), (33, 65), n_words=4, n_maps=2, n_regions=31, thresholds=(0.4,),
                            tags=('regions 31', 'stack region', 'th 1', 'tw 1')),
    'region-32-abs': Case('region', (75, 100), (47, 63), n_words=5, absolute=True, n_regions=32,
                          thresholds=(None, 0.4), tags=('regions 32', 'tile chunks 1 (no min / max)', 'tw 63')),
    'region-63-two-passes': Case('region', (40, 128), (16, 64), n_words=5, n_regions=63, thresholds=(None, 0),
                                 tags=('regions 63', 'window: whole map', 'several passes', 'partial last pass')),
    'region-200KB-window': Case('region', (320, 160), (16, 16), n_words=2, n_regions=2, thresholds=(None,),
                                tags=('window > 12288 floats', 'dynamic smem > 48 KB', 'map 200 KB')),
    'region-api': Case('region', (64, 64), (100, 100), n_words=3, n_maps=2, n_regions=3, api=True,
                       thresholds=(0.4,), tags=('stack region',)),
    # overlay
    'overlay-mod3': Case('overlay', (64, 64), (31, 129), n_words=3, n_maps=2, frames_shift=4,
                         tags=('3 ow mod 4 = 3', 'carry: tile', 'carry: row', 'carry: word', 'carry: map',
                               'carry: past the last map', 'frames 4-byte aligned only', 'th 15', 'tw 1',
                               'stack overlay', 'one image for all maps')),
    'overlay-mod1-per-map': Case('overlay', (30, 50), (17, 63), n_words=2, n_maps=2, image_per_map=True,
                                 thresholds=(None, 0.4), tags=('3 ow mod 4 = 1', 'image per map', 'th 1', 'tw 63',
                                                               'carry: word', 'carry: map')),
    'overlay-mod2': Case('overlay', (96, 64), (50, 66), n_words=2, frames_shift=4, absolute=True,
                         tags=('3 ow mod 4 = 2', 'carry: tile', 'carry: row')),
    'overlay-mod0-abs-no-cn': Case('overlay', (64, 64), (20, 128), n_words=2, absolute=True, color_normalize=False,
                                   thresholds=(None, 0.4), tags=('3 ow mod 4 = 0', 'tile chunks 1 (no min / max)')),
    'overlay-one-axis-window': Case('overlay', (16, 64), (8, 257), n_words=3, frames_shift=4,
                                    tags=('window: whole map on one axis', 'window clamped at a border',
                                          '3 ow mod 4 = 3')),
    'overlay-200KB': Case('overlay', (320, 160), (16, 16), n_words=2, tags=('window > 12288 floats', 'map 200 KB')),
    'overlay-api-stack': Case('overlay', (64, 96), (40, 70), n_words=2, n_maps=2, image_per_map=True, api=True,
                              tags=('stack overlay', 'image per map')),
    # pair: 257 tiles (CTA 0 walks tiles 0 and 256), 50 of 96 words a pass restaged per chunk without a threshold
    'pair-257-tiles-96-words': Case('pair', (64, 64), (16, 16448), n_words=96, thresholds=(None, 0.4),
                                    tags=('pair several tiles per CTA', 'pair uneven tiles per CTA', 'pair 96 words',
                                          'pair restaged per chunk', 'pair partial last pass', 'pair one pass',
                                          'pair dynamic smem > 48 KB')),
    'pair-two-passes': Case('pair', (64, 64), (64, 64), n_words=40, thresholds=(None, 0.4),
                            tags=('pair several passes', 'pair restaged per chunk', 'pair partial last pass',
                                  'pair ctas = tiles', 'ratio identity')),
    'pair-not-staged': Case('pair', (224, 224), (16, 65), n_words=24, thresholds=(None, 0.4),
                            tags=('pair windows not staged, threshold', 'pair windows not staged, no threshold',
                                  'pair tile of < 256 pixels', 'pair window > 12288 floats', 'pair tw 1')),
    'pair-1-word-1x1-tile': Case('pair', (30, 50), (17, 65), thresholds=(None, 0, 0.4),
                                 tags=('pair 1 word', 'pair tile 1x1', 'pair tile of < 256 pixels', 'pair one pass',
                                       'pair th 16', 'pair th 1', 'pair tw 64', 'pair tw 1')),
    'pair-api-stack': Case('pair', (64, 96), (40, 70), n_words=5, n_maps=3, thresholds=(None, 0.4), api=True,
                           tags=('stack pair',)),
    # sweep: a 224 x 224 map over 16 x 65 has a 196 KB window, which fits exactly beside (R + 1) T = 512 bins
    'sweep-one-window-fits': Case('sweep', (224, 224), (16, 65), n_words=2, n_regions=7, thresholds=spread(64),
                                  tags=('sweep exactly one window fits', 'sweep several passes', 'sweep thresholds 64',
                                        'sweep bucket T', 'sweep warp partly outside the tile',
                                        'sweep dynamic smem > 48 KB', 'sweep window > 12288 floats')),
    'sweep-not-staged-513': Case('sweep', (224, 224), (16, 65), n_words=3, n_regions=8, thresholds=spread(57),
                                 tags=('sweep windows not staged', 'sweep bucket T')),
    'sweep-not-staged-63-regions': Case('sweep', (224, 224), (16, 65), n_words=2, n_regions=63, thresholds=spread(64),
                                        tags=('sweep windows not staged', 'sweep regions 63', 'sweep thresholds 64')),
    'sweep-200KB': Case('sweep', (320, 160), (16, 16), n_words=2, n_regions=1, thresholds=(0.5,),
                        tags=('sweep windows not staged', 'sweep map 200 KB', 'sweep regions 1',
                              'sweep thresholds 1')),
    'sweep-three-passes': Case('sweep', (96, 96), (40, 56), n_words=24, n_regions=63, thresholds=spread(64),
                               tags=('sweep several passes', 'sweep partial last pass', 'sweep regions 63',
                                     'sweep thresholds 64', 'sweep bucket T')),
    'sweep-zero-word-stack': Case('sweep', (64, 96), (33, 70), n_words=4, n_maps=2, absolute=True, zero_word=True,
                                  n_regions=31, thresholds=(0, 0.2, 0.4, 0.6, 0.8), api=True,
                                  tags=('stack sweep', 'sweep bucket 0 only', 'sweep threshold equal to a pixel value',
                                        'sweep regions 31', 'sweep warp partly outside the tile', 'sweep one pass')),
    'sweep-32-regions': Case('sweep', (75, 100), (47, 63), n_words=5, n_regions=32, thresholds=spread(19),
                             tags=('sweep regions 32', 'sweep th 15', 'sweep tw 63')),
    # instances: a 16 128-float window over 17 x 65, one word per pass; scratch for every plane and for one
    'instances-one-word-per-pass': Case('instances', (128, 128), (17, 65), n_words=4, thresholds=(0.4,),
                                        scratch_planes=(0, 1),
                                        tags=('instances one word per pass', 'instances several passes',
                                              'instances window > 12288 floats', 'instances dynamic smem > 48 KB',
                                              'instances th 16', 'instances th 1', 'instances tw 64', 'instances tw 1',
                                              'cc last tile 1 column', 'round: one plane', 'round: all planes')),
    'instances-200KB': Case('instances', (320, 160), (33, 40), n_words=2, k=64, thresholds=(0.4,),
                            tags=('instances map 200 KB', 'instances K 64', 'cc last tile 1 row')),
    'instances-rounds-stack': Case('instances', (64, 96), (40, 70), n_words=5, n_maps=3, k=1, thresholds=(0.4,),
                                   scratch_planes=(3, 7, 10, 0), api=True,
                                   tags=('stack instances', 'instances K 1', 'round: words split, partial last round',
                                         'round: one map, planes left over', 'round: several maps',
                                         'round: all planes')),
    'instances-1xN': Case('instances', (64, 64), (1, 300), n_words=3, thresholds=(0.4,), tags=('cc out 1xN',)),
    'instances-Nx1': Case('instances', (64, 64), (300, 1), n_words=3, thresholds=(0.4,), tags=('cc out Nx1',)),
    'instances-1x1': Case('instances', (30, 50), (1, 1), n_words=2, thresholds=(0.4,),
                          tags=('cc out 1x1', 'cc single tile', 'count 0')),
    'instances-zero-word': Case('instances', (64, 96), (32, 40), n_words=3, absolute=True, zero_word=True,
                                thresholds=(0.3,), tags=('count 0',)),
    'instances-diagonals': Case('instances', (64, 96), (64, 96), n_words=2, absolute=True, k=1, thresholds=(0.5,),
                                pattern='diagonals', scratch_planes=(0, 1),
                                tags=('count > K', 'ratio identity', 'instances K 1', 'round: one plane')),
}
CASE_NAMES = list(CASES)

# the regimes the table must reach at every SM count the host test checks
REQUIRED = (
    ['expand chunks 1', 'expand chunks 2', 'expand chunks 31', 'expand chunks 32',
     'expand chunks c at n = 256 (c - 1) + 1', 'expand chunks c at n = 256 c', 'expand 96 words, one CTA per SM',
     'expand 96 words on 64x64', 'planted expand chunk ends', 'planted tile chunk ends',
     'map 1x1', 'map 1xN', 'map Nx1', 'map 2x3', 'map non-square', 'map 200 KB',
     'up dyadic', 'up non-dyadic', 'down dyadic', 'down non-dyadic', 'ratio 64->96', 'ratio 96->40', 'ratio 320->300',
     'ratio 97->1000', 'out 1x1',
     'tile chunks 1 (mwords >= 4 SMs)', 'tile chunks 1 (no min / max)', 'tile chunks in between', 'tile chunks 32',
     'one pass', 'several passes', 'partial last pass', 'one word per pass, 96 words',
     'window clamped at a border', 'window: whole map on one axis', 'window: whole map', 'window > 12288 floats',
     'dynamic smem > 48 KB', 'th 16', 'th 15', 'th 1', 'tw 64', 'tw 63', 'tw 1', 'output smaller than a tile',
     'regions 1', 'regions 31', 'regions 32', 'regions 63',
     'stack segment', 'stack region', 'stack overlay', 'image per map', 'one image for all maps',
     'frames 4-byte aligned only'] +
    [f'3 ow mod 4 = {r}' for r in range(4)] +
    [f'carry: {k}' for k in ('tile', 'row', 'word', 'map', 'past the last map')] +
    ['pair windows not staged, threshold', 'pair windows not staged, no threshold', 'pair one pass',
     'pair several passes', 'pair restaged per chunk', 'pair partial last pass', 'pair ctas = tiles',
     'pair several tiles per CTA', 'pair uneven tiles per CTA', 'pair tile of < 256 pixels', 'pair tile 1x1',
     'pair 1 word', 'pair 96 words', 'stack pair'] +
    ['sweep windows not staged', 'sweep exactly one window fits', 'sweep several passes', 'sweep partial last pass',
     'sweep thresholds 1', 'sweep thresholds 64', 'sweep bucket T', 'sweep bucket 0 only',
     'sweep threshold equal to a pixel value', 'sweep warp partly outside the tile', 'sweep dynamic smem > 48 KB',
     'stack sweep'] + [f'sweep regions {r}' for r in (1, 31, 32, 63)] +
    [f'instances {t}' for t in ('several passes', 'one word per pass', 'window > 12288 floats', 'map 200 KB',
                                'dynamic smem > 48 KB', 'th 1', 'tw 1')] +
    ['cc out 1xN', 'cc out Nx1', 'cc out 1x1', 'cc last tile 1 column', 'cc last tile 1 row', 'cc single tile',
     'instances K 1', 'instances K 64', 'count > K', 'count 0', 'round: one plane',
     'round: words split, partial last round', 'round: one map, planes left over', 'round: several maps',
     'round: all planes', 'stack instances'])


def case_regimes(case: Case, sm_count: int) -> set:
    SM_FOR_TAGS[0] = sm_count
    return regimes(case, plan(case, sm_count))


def assert_regimes(name: str, sm_count: int):
    case = CASES[name]
    missing = set(case.tags) - case_regimes(case, sm_count)
    assert not missing, f'{name} at {sm_count} SMs: the case no longer reaches {sorted(missing)}'


# ---- buffers with guards --------------------------------------------------------------------------------------------------

GUARD = 256                   # sentinel elements before and after every output
SENTINEL_BYTE = 0xA5


class Guarded:
    """``n`` elements of ``dtype`` with ``GUARD`` sentinels (NaN, or 0xA5 bytes) before and after; ``shift`` more
    elements before (a byte buffer starting ``shift`` bytes past an aligned address)."""

    def __init__(self, n: int, dtype=torch.float32, shift: int = 0):
        self.fill = float('nan') if dtype.is_floating_point else SENTINEL_BYTE
        self.lead = GUARD + shift
        self.buf = torch.full((self.lead + n + GUARD,), self.fill, dtype=dtype, device=DEV)
        self.view = self.buf[self.lead:self.lead + n]
        self.n = n

    def ptr(self) -> int:
        return self.view.data_ptr()

    def reset(self):
        self.buf.fill_(self.fill)

    def check(self, what: str):
        rest = torch.cat([self.buf[:self.lead], self.buf[self.lead + self.n:]])
        ok = torch.isnan(rest).all() if self.buf.dtype.is_floating_point else (rest == SENTINEL_BYTE).all()
        assert bool(ok), f'{what}: written outside its buffer'


def global_maps(case: Case, seed: int, word_maps: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``n_maps`` global maps ``[N_ROWS, mh, mw]`` back to back, with a NaN map before and after them and every row no
    word selects NaN: a kernel that reads a wrong row or map (``map_stride``) produces NaN. The selected rows are
    uniform in [0, 1) (absolute maps straddle 0.4), or the given word maps (one row per word)."""
    mh, mw = case.grid
    buf = torch.full((case.n_maps + 2, N_ROWS, mh, mw), float('nan'), device=DEV)
    maps = buf[1:-1]
    gen = torch.Generator(device=DEV).manual_seed(seed)
    for w, rows in enumerate(case.rows_per_word()):
        for r in rows:
            if word_maps is not None:
                maps[:, r] = word_maps[w]
            else:
                maps[:, r] = torch.rand((case.n_maps, mh, mw), generator=gen, device=DEV)
    if case.zero_word:
        maps[:, case.rows_per_word()[-1]] = 0.0
    return maps


# ---- float64 references ---------------------------------------------------------------------------------------------------

class Ref:
    """The float64 pipeline of one map: ``exp`` (expand64), ``bound`` (expand_bound), ``wm_bound`` (word_mean's)."""

    def __init__(self, maps: torch.Tensor, rows: List[List[int]], out, absolute: bool):
        self.exp, self.bound = bound_for(maps, rows, out, absolute)
        self.wm_bound = row_mean_bound(maps, rows)

    def decided(self, t: Optional[float]):
        """``(m64, unsure)``: the float64 value (thresholded when ``t`` is truthy) and the elements the bound cannot
        decide (``None`` without a threshold)."""
        if not t:
            return self.exp.pre, None
        t32 = fp32(t)
        return (self.exp.pre > t32).double(), threshold_unsure(self.exp.pre, self.bound, t32)


EXCLUDED_MAX = 5e-3           # the largest fraction of elements a check may leave out as undecided


def _few(unsure: torch.Tensor, what: str, n_words: int):
    n = int(unsure.sum())
    assert n <= EXCLUDED_MAX * unsure.numel() + 4 * n_words, f'{what}: {n} of {unsure.numel()} elements within the bound of a ' \
                                                     f'threshold or a tie'


def check_m(got: torch.Tensor, ref: Ref, t, what: str):
    m64, unsure = ref.decided(t)
    if unsure is None:
        excess = (got.double() - m64).abs() - ref.bound
        excess = torch.where(torch.isnan(excess), torch.full_like(excess, float('inf')), excess)
        i = int(excess.argmax())
        assert float(excess.reshape(-1)[i]) <= 0, \
            f'{what}: element {np.unravel_index(i, tuple(got.shape))}: got {float(got.reshape(-1)[i]):.9e} float64 ' \
            f'{float(m64.reshape(-1)[i]):.9e}, bound {float(ref.bound.reshape(-1)[i]):.2e}'
        return
    _few(unsure, what, got.shape[0])
    bad = (got.double() != m64) & ~unsure
    assert not bool(bad.any()), f'{what}: {int(bad.sum())} thresholded elements differ from float64 away from the ' \
                                f'threshold, first at {tuple(bad.nonzero()[0].tolist())}'


def check_word_maps(got: torch.Tensor, ref: Ref, what: str):
    err = (got.double() - ref.exp.word_maps).abs()
    assert bool((err <= ref.wm_bound).all()), f'{what}: word maps beyond (k + 1) u of the float64 row mean'


# ---- running the entries --------------------------------------------------------------------------------------------------

def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _sm_count() -> int:
    return _native.device_info()['sm_count']


def _launches(fn) -> int:
    torch.cuda.synchronize()
    before = _native.launch_count()
    fn()
    torch.cuda.synchronize()
    return _native.launch_count() - before


def run_expand(case: Case, maps: torch.Tensor, refs: List[Ref], p: dict, what: str):
    (mh, mw), (oh, ow) = case.grid, case.out
    rows = case.rows_per_word()
    out = Guarded(case.n_words * oh * ow)
    wmaps = Guarded(case.n_words * mh * mw)
    scratch = torch.empty(_native.EXPAND_SCRATCH_FLOATS * case.n_words, device=DEV)
    for t in case.thresholds:
        out.reset()
        wmaps.reset()
        if case.entry == 'expand_as':
            src = maps[0, rows[0][0]]
            call = lambda: _native.expand_as(src.data_ptr(), case.grid, oh, ow, case.absolute, t, out.ptr(),
                                             scratch.data_ptr(), _stream())
        else:
            call = lambda: _native.expand_words(maps[0].data_ptr(), N_ROWS, case.grid, rows, oh, ow, case.absolute, t,
                                                wmaps.ptr(), out.ptr(), scratch.data_ptr(), _stream())
        n = _launches(call)
        w = f'{what} threshold {t}'
        assert n == p['launches'], f'{w}: {n} launches, the plan says {p["launches"]}'
        out.check(f'{w}: out')
        check_m(out.view.view(case.n_words, oh, ow), refs[0], t, w)
        if case.entry == 'expand':
            wmaps.check(f'{w}: word_maps')
            check_word_maps(wmaps.view.view(case.n_words, mh, mw), refs[0], w)


def _tile_buffers(case: Case):
    (mh, mw), (oh, ow) = case.grid, case.out
    return Guarded(case.n_maps * case.n_words * mh * mw)


def run_segment(case: Case, maps: torch.Tensor, refs: List[Ref], p: dict, what: str):
    (mh, mw), (oh, ow) = case.grid, case.out
    wmaps = _tile_buffers(case)
    labels = Guarded(case.n_maps * oh * ow, torch.uint8)
    scores = Guarded(case.n_maps * oh * ow)
    scratch = torch.empty(_native.segment_scratch_floats(case.n_maps, case.n_words), device=DEV)
    for t in case.thresholds:
        for g in (wmaps, labels, scores):
            g.reset()
        n = _launches(lambda: _native.segment_words(maps.data_ptr(), case.n_maps, N_ROWS, case.grid,
                                                    case.rows_per_word(), oh, ow, case.absolute, t, wmaps.ptr(),
                                                    labels.ptr(), scores.ptr(), scratch.data_ptr(), _stream()))
        w = f'{what} threshold {t}'
        assert n == p['launches'], f'{w}: {n} launches, the plan says {p["launches"]}'
        for g, name in ((wmaps, 'word_maps'), (labels, 'labels'), (scores, 'scores')):
            g.check(f'{w}: {name}')
        check_segment(labels.view.view(case.n_maps, oh, ow), scores.view.view(case.n_maps, oh, ow),
                      wmaps.view.view(case.n_maps, case.n_words, mh, mw), refs, t, w, case.rows_per_word())


def check_segment(labels, scores, wmaps, refs: List[Ref], t, what: str, rows: List[List[int]]):
    """Words that select the same rows have the same bits and tie exactly; the first of them wins. The others are
    decided where the float64 top two differ by more than both bounds."""
    firsts = [i for i, r in enumerate(rows) if rows.index(r) == i]
    for i, ref in enumerate(refs):
        w = f'{what} map {i}'
        check_word_maps(wmaps[i], ref, w)
        pre, b = ref.exp.pre[firsts], ref.bound
        top = pre.topk(min(2, pre.shape[0]), dim=0).values
        bmax = b.amax(0)
        assert bool(((scores[i].double() - top[0]).abs() <= bmax).all()), f'{w}: scores beyond the bound'
        margin = top[0] - top[1] if pre.shape[0] > 1 else torch.full_like(top[0], float('inf'))
        unsure = margin <= 2 * bmax
        want = torch.tensor(firsts, device=pre.device)[pre.argmax(0)] + 1
        if t:
            t32 = fp32(t)
            unsure |= (top[0] - t32).abs() <= bmax
            want = torch.where(top[0] > t32, want, torch.zeros_like(want))
        _few(unsure, w, 1)
        bad = (labels[i].long() != want) & ~unsure
        assert not bool(bad.any()), f'{w}: {int(bad.sum())} labels differ from float64 away from ties'


def make_regions(case: Case, seed: int) -> torch.Tensor:
    """Region 0 the whole image, the others random halves (some as 0 / 2 bytes: nonzero is inside)."""
    oh, ow = case.out
    g = torch.Generator(device=DEV).manual_seed(seed)
    r = torch.randint(0, 2, (case.n_regions, oh, ow), generator=g, device=DEV, dtype=torch.uint8) * 2
    r[0] = 1
    return r


def run_region(case: Case, maps: torch.Tensor, refs: List[Ref], p: dict, what: str, seed: int):
    (mh, mw), (oh, ow) = case.grid, case.out
    regions = make_regions(case, seed)
    wmaps = _tile_buffers(case)
    inter = Guarded(case.n_maps * case.n_regions * case.n_words)
    area = Guarded(case.n_maps * case.n_words)
    scratch = torch.empty(_native.region_scratch_floats(case.n_maps, case.n_words, case.n_regions, oh, ow),
                          device=DEV)
    for t in case.thresholds:
        for g in (wmaps, inter, area):
            g.reset()
        n = _launches(lambda: _native.region_overlap(maps.data_ptr(), case.n_maps, N_ROWS, case.grid,
                                                     case.rows_per_word(), oh, ow, case.absolute, t, wmaps.ptr(),
                                                     regions.data_ptr(), case.n_regions, inter.ptr(), area.ptr(),
                                                     scratch.data_ptr(), _stream()))
        w = f'{what} threshold {t}'
        assert n == p['launches'], f'{w}: {n} launches, the plan says {p["launches"]}'
        for g, name in ((wmaps, 'word_maps'), (inter, 'intersection'), (area, 'word_area')):
            g.check(f'{w}: {name}')
        check_region(inter.view.view(case.n_maps, case.n_regions, case.n_words), area.view.view(case.n_maps,
                     case.n_words), wmaps.view.view(case.n_maps, case.n_words, mh, mw), regions, refs, t, w,
                     tiles=-(-oh // TILE_H) * -(-ow // TILE_W))


def check_region(inter, area, wmaps, regions, refs: List[Ref], t, what: str, tiles: int):
    """Thresholded: every count between the float64 count over the pixels surely inside and that count plus the
    pixels the bound cannot decide. Otherwise: within the summed element bound plus the fp32 summation error: the
    kernels add at most ``4 + 5 + 8`` times inside a tile and ``ceil(tiles / 32) + 5`` times across tiles."""
    masks = torch.cat([torch.ones_like(regions[:1]), regions]) != 0               # slot 0: the word's area
    masks = masks.double().flatten(1)                                           # [slots, pixels]
    depth = 4 + 5 + 8 + -(-tiles // 32) + 5
    for i, ref in enumerate(refs):
        w = f'{what} map {i}'
        check_word_maps(wmaps[i], ref, w)
        got = torch.cat([area[i][None], inter[i]]).double()                      # [slots, words]
        pre, b = ref.exp.pre.flatten(1), ref.bound.flatten(1)                    # [words, pixels]
        if t:
            t32 = fp32(t)
            sure = (pre > t32) & ~threshold_unsure(pre, b, t32)
            unsure = threshold_unsure(pre, b, t32)
            low, extra = masks @ sure.double().T, masks @ unsure.double().T
            bad = (got < low) | (got > low + extra)
            assert not bool(bad.any()), f'{w}: a count outside [sure, sure + undecided]: slot, word ' \
                                        f'{tuple(bad.nonzero()[0].tolist())}'
        else:
            want = masks @ pre.T
            tol = masks @ b.T + depth * U * (masks @ (pre.abs() + b).T)
            bad = (got - want).abs() > tol
            assert not bool(bad.any()), f'{w}: a sum beyond its bound at slot, word {tuple(bad.nonzero()[0].tolist())}'


TABLE = None


def jet() -> torch.Tensor:
    global TABLE
    if TABLE is None:
        TABLE = _native.jet_colormap().double().to(DEV)
    return TABLE


def _range_table(lut: torch.Tensor):
    """``[256, 256, 3]`` min and max of ``lut[k0 .. k1]`` per channel (k0 <= k1)."""
    lo = torch.full((256, 256, 3), float('inf'), dtype=torch.float64, device=lut.device)
    hi = torch.full((256, 256, 3), float('-inf'), dtype=torch.float64, device=lut.device)
    for k0 in range(256):
        lo[k0, k0:] = torch.cummin(lut[k0:], 0).values
        hi[k0, k0:] = torch.cummax(lut[k0:], 0).values
    return lo, hi


RANGES = None


def overlay_range(ref: Ref, t, color_normalize: bool, absolute: bool, image: torch.Tensor):
    """``(low, high)`` bytes ``[words, H, W, 3]``: the range of ``round((1 - a) image + a L[k])`` when m ranges over
    its bound (thresholded: over {0, 1} where undecided), with ``a = clamp(m, 0, 1)``, ``k`` every colour index the
    bounded ``c`` reaches, and the word's lo / hi of m over their bounds. Linear in ``a`` and ``L``: the ends suffice."""
    global RANGES
    if RANGES is None:
        RANGES = _range_table(jet())
    pre, b = ref.exp.pre, ref.bound
    bstar = b.amax((1, 2), keepdim=True)
    lo_pre = torch.zeros_like(ref.exp.lo) if not absolute else ref.exp.lo             # m at the min / max of v
    hi_pre = ((ref.exp.hi - ref.exp.lo) / (ref.exp.hi - ref.exp.lo + 1e-8)) if not absolute else ref.exp.hi
    if t:
        t32 = fp32(t)

        def interval(x, bx):
            one = (x > t32).double()
            unsure = threshold_unsure(x, bx, t32)
            return torch.where(unsure, 0.0, one), torch.where(unsure, 1.0, one)
        m0, m1 = interval(pre, b)
        l0, l1 = interval(lo_pre, bstar)
        h0, h1 = interval(hi_pre, bstar)
    else:
        m0, m1 = pre - b, pre + b
        lz = torch.zeros_like(bstar) if not absolute else bstar
        l0, l1 = lo_pre - lz, lo_pre + lz
        h0, h1 = hi_pre - bstar, hi_pre + bstar
    if color_normalize:
        num0, num1 = m0 - l1, m1 - l0
        den0, den1 = h0 - l1, h1 - l0
        maybe_equal = den0 <= 0                                  # hi == lo possible: c = 0, or anything
        den0 = den0.clamp(min=1e-300)
        c0 = torch.where(num0 >= 0, num0 / den1, num0 / den0)
        c1 = torch.where(num1 >= 0, num1 / den0, num1 / den1)
        c0 = torch.where(maybe_equal, torch.zeros_like(c0), c0)
        c1 = torch.where(maybe_equal, torch.ones_like(c1), c1)
    else:
        c0, c1 = m0.clamp(0, 1), m1.clamp(0, 1)
    slack = 4 * U * torch.maximum(c0.abs(), c1.abs()) + 2.0 ** -60
    k0 = torch.floor(256 * (c0 - slack)).clamp(0, 255).long()
    k1 = torch.floor(256 * (c1 + slack)).clamp(0, 255).long()
    l_lo, l_hi = RANGES[0][k0, k1], RANGES[1][k0, k1]                            # [words, H, W, 3]
    a0, a1 = m0.clamp(0, 1).unsqueeze(-1), m1.clamp(0, 1).unsqueeze(-1)
    img = image.double()
    ends = [(1 - a) * img + a * lut for a in (a0, a1) for lut in (l_lo, l_hi)]
    vmin = torch.stack([e.expand_as(ends[0]) for e in ends]).amin(0)
    vmax = torch.stack([e.expand_as(ends[0]) for e in ends]).amax(0)
    low = torch.ceil(vmin - 0.5 - 1e-3).clamp(0, 255)
    high = torch.floor(vmax + 0.5 + 1e-3).clamp(0, 255)
    return low, high


def make_images(case: Case, seed: int) -> torch.Tensor:
    oh, ow = case.out
    g = torch.Generator(device=DEV).manual_seed(seed)
    n = case.n_maps if case.image_per_map else 1
    return torch.randint(0, 256, (n, oh, ow, 3), generator=g, device=DEV, dtype=torch.uint8)


def run_overlay(case: Case, maps: torch.Tensor, refs: List[Ref], p: dict, what: str, seed: int):
    (mh, mw), (oh, ow) = case.grid, case.out
    images = make_images(case, seed)
    wmaps = _tile_buffers(case)
    n_bytes = case.n_maps * case.n_words * oh * ow * 3
    frames = Guarded(_native.overlay_frames_bytes(case.n_maps, case.n_words, oh, ow), torch.uint8,
                     shift=case.frames_shift)
    assert frames.ptr() % 16 == case.frames_shift
    scratch = torch.empty(_native.segment_scratch_floats(case.n_maps, case.n_words), device=DEV)
    for t in case.thresholds:
        for g in (wmaps, frames):
            g.reset()
        n = _launches(lambda: _native.overlay_words(maps.data_ptr(), case.n_maps, N_ROWS, case.grid,
                                                    case.rows_per_word(), oh, ow, case.absolute, t,
                                                    case.color_normalize, wmaps.ptr(), images.data_ptr(),
                                                    oh * ow * 3 if case.image_per_map else 0, frames.ptr(),
                                                    scratch.data_ptr(), _stream()))
        w = f'{what} threshold {t}'
        assert n == p['launches'], f'{w}: {n} launches, the plan says {p["launches"]}'
        wmaps.check(f'{w}: word_maps')
        frames.check(f'{w}: frames')
        got = frames.view[:n_bytes].view(case.n_maps, case.n_words, oh, ow, 3)
        check_overlay(got, wmaps.view.view(case.n_maps, case.n_words, mh, mw), images, refs, t, case, w)


def check_overlay(frames, wmaps, images, refs: List[Ref], t, case: Case, what: str):
    for i, ref in enumerate(refs):
        w = f'{what} map {i}'
        check_word_maps(wmaps[i], ref, w)
        img = images[i if case.image_per_map else 0]
        low, high = overlay_range(ref, t, case.color_normalize, case.absolute, img)
        got = frames[i].double()
        bad = (got < low) | (got > high)
        if bool(bad.any()):
            j = tuple(bad.nonzero()[0].tolist())
            raise AssertionError(f'{w}: {int(bad.sum())} bytes outside their range, first at word, y, x, ch {j}: '
                                 f'{int(got[j])} not in [{int(low[j])}, {int(high[j])}]')


# ---- pair, sweep and instances: on expand_words' m, checked against float64 in the same case ----------------------------

def expand_each_map(case: Case, maps: torch.Tensor, refs: List[Ref], what: str) -> List[torch.Tensor]:
    """``expand_words`` without threshold of every map, each ``[n_words, oh, ow]`` checked against float64: the values
    the pair, sweep and instance kernels must reproduce bit for bit (every consumer's m is expand_words')."""
    oh, ow = case.out
    scratch = torch.empty(_native.EXPAND_SCRATCH_FLOATS * case.n_words, device=DEV)
    pres = []
    for i in range(case.n_maps):
        out = Guarded(case.n_words * oh * ow)
        _native.expand_words(maps[i].data_ptr(), N_ROWS, case.grid, case.rows_per_word(), oh, ow, case.absolute, None,
                             None, out.ptr(), scratch.data_ptr(), _stream())
        w = f'{what} map {i}: expand_words'
        out.check(w)
        pre = out.view.view(case.n_words, oh, ow)
        check_m(pre, refs[i], None, w)
        pres.append(pre)
    return pres


def decided(pre64: torch.Tensor, b: torch.Tensor, t32: float):
    """``(sure, unsure)`` of ``pre > t32``; a zero bound means the fp32 value is the float64 one, decided even at the
    threshold (the zero word at 0)."""
    unsure = threshold_unsure(pre64, b, t32) & (b > 0)
    return (pre64 > t32) & ~unsure, unsure


def run_pair(case: Case, maps: torch.Tensor, refs: List[Ref], p: dict, what: str) -> dict:
    (mh, mw), (oh, ow) = case.grid, case.out
    n_maps, n_words = case.n_maps, case.n_words
    pres = expand_each_map(case, maps, refs, what)
    wmaps = _tile_buffers(case)
    inter, area = Guarded(n_maps * n_words * n_words), Guarded(n_maps * n_words)
    scratch = Guarded(_native.word_overlap_scratch_floats(n_maps, n_words, oh, ow))
    got = {}
    for t in case.thresholds:
        for g in (wmaps, inter, area, scratch):
            g.reset()
        n = _launches(lambda: _native.word_overlap(maps.data_ptr(), n_maps, N_ROWS, case.grid, case.rows_per_word(),
                                                   oh, ow, case.absolute, t, wmaps.ptr(), inter.ptr(), area.ptr(),
                                                   scratch.ptr(), _stream()))
        w = f'{what} threshold {t}'
        assert n == p['launches'], f'{w}: {n} launches, the plan says {p["launches"]}'
        for g, name in ((wmaps, 'word_maps'), (inter, 'intersection'), (area, 'word_area'), (scratch, 'scratch')):
            g.check(f'{w}: {name}')
        i32 = inter.view.view(n_maps, n_words, n_words).view(torch.int32)
        assert torch.equal(i32, i32.transpose(1, 2)), f'{w}: the intersection matrix is not exactly symmetric'
        check_pair(inter.view.view(n_maps, n_words, n_words), area.view.view(n_maps, n_words),
                   wmaps.view.view(n_maps, n_words, mh, mw), pres, refs, t, p, w)
        got[t] = (inter.view.view(n_maps, n_words, n_words).clone(), area.view.view(n_maps, n_words).clone())
    return got


def check_pair(inter, area, wmaps, pres: List[torch.Tensor], refs: List[Ref], t, p: dict, what: str):
    """Thresholded: the int64 counts of expand_words' masks bit for bit, and between the float64 sure and sure plus
    undecided counts. Otherwise, with ``M`` the float64 m and ``b`` its bound: ``|m_a m_b - M_a M_b| <= |M_a| b_b +
    |M_b| b_a + b_a b_b`` per pixel, and the fp32 sum of the products adds ``gamma_depth sum (|M_a| + b_a) (|M_b| +
    b_b)``, ``depth`` the adds any product passes through: 8 fmas of a lane and a 5-step butterfly per 256-pixel chunk,
    one add per chunk into the CTA's partial (4 chunks a tile, ``walk`` tiles a CTA), then ``ceil(ctas / 32)`` lane
    adds and a 5-step butterfly in word_pair_reduce_kernel; ``gamma_d = d u / (1 - d u) < (d + 1) u``. The areas are
    the same with ``m_b = 1``."""
    depth = 8 + 5 + 4 * p['walk'] + -(-p['ctas'] // 32) + 5
    for i, ref in enumerate(refs):
        w = f'{what} map {i}'
        check_word_maps(wmaps[i], ref, w)
        got_i, got_a = inter[i].double(), area[i].double()
        pre64, b = ref.exp.pre.flatten(1), ref.bound.flatten(1)                  # [words, pixels]
        if t:
            t32 = fp32(t)
            mask = (pres[i].flatten(1) > t32).double()
            assert torch.equal(got_i, mask @ mask.T), f'{w}: intersection differs from the expand_words masks\' counts'
            assert torch.equal(got_a, mask.sum(1)), f'{w}: word_area differs from the expand_words masks\' counts'
            sure, unsure = decided(pre64, b, t32)
            _few(unsure, w, pre64.shape[0])
            s, su = sure.double(), (sure | unsure).double()
            bad = (got_i < s @ s.T) | (got_i > su @ su.T)
            assert not bool(bad.any()), f'{w}: a pair count outside [sure, sure + undecided] at ' \
                                        f'{tuple(bad.nonzero()[0].tolist())}'
            bad = (got_a < s.sum(1)) | (got_a > su.sum(1))
            assert not bool(bad.any()), f'{w}: an area outside [sure, sure + undecided]'
        else:
            a = pre64.abs()
            gamma = (depth + 1) * U
            tol_i = a @ b.T + b @ a.T + b @ b.T + gamma * ((a + b) @ (a + b).T)
            err = (got_i - pre64 @ pre64.T).abs()
            bad = err > tol_i
            assert not bool(bad.any()), f'{w}: a pair sum beyond its bound at {tuple(bad.nonzero()[0].tolist())}: ' \
                                        f'error {float(err[bad][0]):.3e}, bound {float(tol_i[bad][0]):.3e}'
            err = (got_a - pre64.sum(1)).abs()
            assert bool((err <= b.sum(1) + gamma * (a + b).sum(1)).all()), f'{w}: an area beyond its bound'


def run_sweep(case: Case, maps: torch.Tensor, refs: List[Ref], p: dict, what: str, seed: int):
    (mh, mw), (oh, ow) = case.grid, case.out
    n_maps, n_words, n_reg, n_thr = case.n_maps, case.n_words, case.n_regions, len(case.thresholds)
    regions = make_regions(case, seed)
    pres = expand_each_map(case, maps, refs, what)
    wmaps = _tile_buffers(case)
    inter, area = Guarded(n_maps * n_thr * n_reg * n_words), Guarded(n_maps * n_thr * n_words)
    scratch = Guarded(_native.region_sweep_scratch_floats(n_maps, n_words, n_reg, n_thr, oh, ow))
    n = _launches(lambda: _native.region_sweep(maps.data_ptr(), n_maps, N_ROWS, case.grid, case.rows_per_word(), oh,
                                               ow, case.absolute, case.thresholds, wmaps.ptr(), regions.data_ptr(),
                                               n_reg, inter.ptr(), area.ptr(), scratch.ptr(), _stream()))
    assert n == p['launches'], f'{what}: {n} launches, the plan says {p["launches"]}'
    for g, name in ((wmaps, 'word_maps'), (inter, 'intersection'), (area, 'word_area'), (scratch, 'scratch')):
        g.check(f'{what}: {name}')
    got_i, got_a = inter.view.view(n_maps, n_thr, n_reg, n_words), area.view.view(n_maps, n_thr, n_words)
    check_sweep(got_i, got_a, wmaps.view.view(n_maps, n_words, mh, mw), pres, regions, refs, case, what)
    return got_i.clone(), got_a.clone(), regions


def check_sweep(inter, area, wmaps, pres: List[torch.Tensor], regions, refs: List[Ref], case: Case, what: str):
    """Slice k: the int64 counts of expand_words' ``m > fp32(tau_k)`` bit for bit, and between the float64 sure and
    sure plus undecided counts; no count increases with k. The regimes the case names from its data are seen."""
    masks = (torch.cat([torch.ones_like(regions[:1]), regions]) != 0).double().flatten(1)    # slot 0: the area
    for i, ref in enumerate(refs):
        w = f'{what} map {i}'
        check_word_maps(wmaps[i], ref, w)
        got = torch.cat([area[i][:, None], inter[i]], 1).double()                 # [T, slots, words]
        pre64, b = ref.exp.pre.flatten(1), ref.bound.flatten(1)
        for k, tau in enumerate(case.thresholds):
            t32 = fp32(tau)
            want = masks @ (pres[i].flatten(1) > t32).double().T
            bad = got[k] != want
            assert not bool(bad.any()), f'{w} threshold {k} ({t32}): a count differs from expand_words\' at slot, ' \
                                        f'word {tuple(bad.nonzero()[0].tolist())}: {int(got[k][bad][0])} != ' \
                                        f'{int(want[bad][0])}'
            sure, unsure = decided(pre64, b, t32)
            _few(unsure, f'{w} threshold {k}', pre64.shape[0])
            low, extra = masks @ sure.double().T, masks @ unsure.double().T
            assert not bool(((got[k] < low) | (got[k] > low + extra)).any()), \
                f'{w} threshold {k}: a count outside [sure, sure + undecided]'
        assert bool((got[1:] <= got[:-1]).all()), f'{w}: a count increases with the threshold'
        taus = [fp32(t) for t in case.thresholds]
        if not case.absolute:                              # 'sweep bucket T': every word has pixels above every tau
            assert bool((got[-1, 0] > 0).all()), f'{w}: a word with no pixel above the last threshold'
        if case.zero_word:
            assert bool((pres[i][-1] == 0).all())
            if min(taus) >= 0:
                assert bool((got[:, :, -1] == 0).all()), f'{w}: the zero word passes a threshold'


FIELDS = ('count', 'area', 'box', 'sum_yx', 'peak', 'peak_yx')


def run_instances(case: Case, maps: torch.Tensor, refs: List[Ref], p: dict, what: str) -> dict:
    """One call per scratch size of the case, each through a scratch of exactly that many planes: every field equal
    to ``instances64_stack`` of expand_words' values, so the same bits at every round split."""
    (mh, mw), (oh, ow) = case.grid, case.out
    n_maps, n_words, k = case.n_maps, case.n_words, case.k
    t = case.thresholds[0]
    pres = expand_each_map(case, maps, refs, what)
    want = [instances64_stack(pre.cpu().numpy(), t, k) for pre in pres]
    want = {f: np.stack([x[f] for x in want]) for f in FIELDS}
    planes = n_maps * n_words
    shapes = dict(count=(), area=(k,), box=(k, 4), sum_yx=(k, 2), peak=(k,), peak_yx=(k, 2))
    types = dict(count=torch.int32, area=torch.int32, box=torch.int32, sum_yx=torch.int64, peak=torch.float32,
                 peak_yx=torch.int32)
    outs = {f: Guarded(planes * int(np.prod(shapes[f], dtype=np.int64)), types[f]) for f in FIELDS}
    wmaps = _tile_buffers(case)
    got = None
    for s in p['splits']:
        w = f'{what} scratch for {s["planes"]} planes'
        scratch = Guarded(s['planes'] * p['plane_bytes'], torch.uint8)
        for g in (wmaps, *outs.values()):
            g.reset()
        n = _launches(lambda: _native.word_instances(maps.data_ptr(), n_maps, N_ROWS, case.grid, case.rows_per_word(),
                                                     oh, ow, case.absolute, t, k, wmaps.ptr(),
                                                     *(outs[f].ptr() for f in FIELDS), scratch.ptr(), scratch.n,
                                                     _stream()))
        assert n == s['launches'], f'{w}: {n} launches, the plan says {s["launches"]}'
        for g, name in ((wmaps, 'word_maps'), (scratch, 'scratch'), *((outs[f], f) for f in FIELDS)):
            g.check(f'{w}: {name}')
        for i, ref in enumerate(refs):
            check_word_maps(wmaps.view.view(n_maps, n_words, mh, mw)[i], ref, f'{w} map {i}')
        got = {f: outs[f].view.view((n_maps, n_words) + shapes[f]).clone() for f in FIELDS}
        for f in FIELDS:
            np.testing.assert_array_equal(got[f].cpu().numpy(), want[f].astype(got[f].cpu().numpy().dtype),
                                          err_msg=f'{w}: {f}')
    if 'count 0' in case.tags:
        assert bool((got['count'] == 0).any()), f'{what}: no word without an instance'
    if 'count > K' in case.tags:
        assert bool((got['count'] > k).any()), f'{what}: no word with more than K instances'
    return got


# ---- planted extremes -----------------------------------------------------------------------------------------------------

def planted_word_map(pinv_y: torch.Tensor, pinv_x: torch.Tensor, oy: int, ox: int, sign: float) -> torch.Tensor:
    """A word map whose float64 up-sample has its argmax (``sign`` +1) or argmin (-1) at ``(oy, ox)``: columns of the
    pseudo-inverses of the two bicubic matrices, so that a down-sample's ``v`` is the delta at ``(oy, ox)``."""
    return sign * torch.outer(pinv_y[:, oy], pinv_x[:, ox])


def chunk_ends(n: int, chunks: int) -> List[int]:
    per = -(-n // chunks)
    out = []
    for c in range(chunks):
        begin, end = c * per, min(n, c * per + per)
        out += [begin, end - 1]
    return sorted(set(out))


def run_planted(case: Case, p: dict, what: str):
    """For every chunk's first and last pixel and both signs: that pixel is the float64 extreme with a margin of 4
    times the bound over every other pixel, and the kernel's normalised map is within the bound of float64."""
    (mh, mw), (oh, ow) = case.grid, case.out
    pinv_y = torch.linalg.pinv(bicubic64(mh, oh, 'cpu')).to(DEV)
    pinv_x = torch.linalg.pinv(bicubic64(mw, ow, 'cpu')).to(DEV)
    for o in chunk_ends(oh * ow, p['chunks']):
        oy, ox = divmod(o, ow)
        for sign in (1.0, -1.0):
            wm = planted_word_map(pinv_y, pinv_x, oy, ox, sign)
            maps = global_maps(case, 0, wm[None].float())
            ref = Ref(maps[0], case.rows_per_word(), case.out, case.absolute)
            v = ref.exp.v[0].flatten()
            target = sign * v[o]
            others = torch.cat([sign * v[:o], sign * v[o + 1:]])
            assert float(target - others.max()) > 4 * float(ref.bound.max()), \
                f'{what}: no margin for the planted extreme at pixel {o}'
            w = f'{what} planted {"max" if sign > 0 else "min"} at pixel {o}'
            if case.entry == 'expand':
                run_expand(case, maps, [ref], p, w)
            else:
                run_segment(case, maps, [ref], p, w)


# ---- the API route ------------------------------------------------------------------------------------------------------

PROMPT = ' '.join(f'w{i}' for i in range(N_ROWS - 2))          # word i is row i + 1


def api_words(case: Case) -> List[str]:
    return [' '.join(f'w{r - 1}' for r in rows) for rows in case.rows_per_word()]


def run_api(case: Case, maps: torch.Tensor, refs: List[Ref], what: str, seed: int, abi=None):
    """The case through GlobalHeatMap / GlobalHeatMapStack: checked against float64 as the C ABI call is, or (pair,
    sweep, instances) equal bit for bit to ``abi``, what the checked C ABI call returned."""
    from types import SimpleNamespace
    from daam_b200.heatmap import GlobalHeatMap, GlobalHeatMapStack
    from daam_b200.testing.synthetic import WhitespaceTokenizer
    tok = WhitespaceTokenizer()
    (oh, ow), (mh, mw) = case.out, case.grid
    assert mh != mw or oh == ow, 'a square map takes the image size as (size[0], size[1])'
    image = SimpleNamespace(size=(ow, oh), height=oh, width=ow)
    words = api_words(case)
    stack = GlobalHeatMapStack(tok, PROMPT, maps)
    bits = lambda x: x.contiguous().view(torch.int32)
    if case.entry == 'pair':
        for t in case.thresholds:
            _, ov = stack.word_overlap(words, image, case.absolute, t, to_cpu=False)
            assert torch.equal(bits(ov.intersection), bits(abi[t][0])), f'{what} API threshold {t}: intersection'
            assert torch.equal(bits(ov.word_area), bits(abi[t][1])), f'{what} API threshold {t}: word_area'
        return
    if case.entry == 'sweep':
        inter, area, regions = abi
        _, ov = stack.region_sweep(words, image, regions, case.thresholds, case.absolute, to_cpu=False)
        assert torch.equal(bits(ov.intersection), bits(inter)) and torch.equal(bits(ov.word_area), bits(area)), \
            f'{what} API: the sweep differs from the C ABI call'
        return
    if case.entry == 'instances':
        _, inst = stack.word_instances(words, image, case.thresholds[0], case.absolute, case.k, to_cpu=False)
        for f in FIELDS:
            assert torch.equal(getattr(inst, f), abi[f]), f'{what} API: {f} differs from the C ABI call'
        return
    for t in case.thresholds:
        w = f'{what} API threshold {t}'
        if case.entry == 'expand':
            whms, m = GlobalHeatMap(tok, PROMPT, maps[0]).expand_words(words, image, case.absolute, t, to_cpu=False)
            check_m(m, refs[0], t, w)
            check_word_maps(torch.stack([x.heatmap for x in whms]), refs[0], w)
        elif case.entry == 'segment':
            wm, labels, scores = stack.segment(words, image, case.absolute, t, to_cpu=False)
            check_segment(labels, scores, wm, refs, t, w, case.rows_per_word())
        elif case.entry == 'region':
            regions = make_regions(case, seed)
            wm, ov = stack.region_overlap(words, image, regions, case.absolute, t, to_cpu=False)
            check_region(ov.intersection, ov.word_area, wm, regions, refs, t, w,
                         tiles=-(-oh // TILE_H) * -(-ow // TILE_W))
        else:
            images = make_images(case, seed)
            wm, frames = stack.overlay_words(words, images if case.image_per_map else images[0], case.absolute, t,
                                             case.color_normalize, to_cpu=False)
            check_overlay(frames, wm, images, refs, t, case, w)


# ---- the tests ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('name', CASE_NAMES)
def test_case_against_float64(name):
    sm = _sm_count()
    assert_regimes(name, sm)
    case = CASES[name]
    p = plan(case, sm)
    seed = CASE_NAMES.index(name)
    if case.planted:
        run_planted(case, p, name)
        return
    pattern = torch.from_numpy(diagonal_word_maps(case)).to(DEV) if case.pattern == 'diagonals' else None
    maps = global_maps(case, seed, pattern)
    rows = case.rows_per_word()
    refs = [Ref(maps[i], rows, case.out, case.absolute) for i in range(case.n_maps)]
    abi = None
    if case.entry in ('expand', 'expand_as'):
        if p['chunks_asserted'] is not None:
            assert p['chunks'] == p['chunks_asserted']
        run_expand(case, maps, refs, p, name)
    elif case.entry == 'segment':
        run_segment(case, maps, refs, p, name)
    elif case.entry == 'region':
        run_region(case, maps, refs, p, name, seed)
    elif case.entry == 'overlay':
        run_overlay(case, maps, refs, p, name, seed)
    elif case.entry == 'pair':
        abi = run_pair(case, maps, refs, p, name)
    elif case.entry == 'sweep':
        abi = run_sweep(case, maps, refs, p, name, seed)
    else:
        abi = run_instances(case, maps, refs, p, name)
    if case.api:
        run_api(case, maps, refs, name, seed, abi)
