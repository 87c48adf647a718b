"""Host checks of the word-list geometry table (``tests/test_word_geometry_gpu.py``) and of the float64 error bound
(``tests/words64.py``), without a GPU.

* Every case reaches the regimes it names, and the table covers every regime, at 132, 114 and 78 SMs.
* ``expand_bound`` dominates fp32 emulations of ``make_taps`` and ``bicubic_shared`` (with and without fma
  contraction) against ``math_bicubic_matrix``: the coordinate term row by row on a grid of ratios, the whole bound on
  the ratios of the GPU table.
* ``launch_tiles``'s window estimate is never smaller than a tile's actual window.
* Beside the pair and sweep kernels' own shared buffers, the staged windows stay within 200 KB and none is staged
  exactly when none fits, over every word, region and threshold count the C ABI accepts; the word-instance rounds take
  every plane once.
* The regimes that cannot occur, with the reason."""
import numpy as np
import pytest
import torch

from oracle import daam_oracle as O
from tests.test_word_geometry_gpu import (CASE_NAMES, CASES, MAX_CHUNKS, MAX_ROUND_PLANES, MAX_SMEM, REQUIRED, TILE_H,
                                          TILE_W, Case, case_regimes, expand_per_sm, instance_rounds, pair_smem_bytes,
                                          plan, sweep_smem_bytes, words_per_pass)
from tests.words64 import expand64, expand_bound, row_motion, word_maps64

SMS = (132, 114, 78)


@pytest.mark.parametrize('sm', SMS)
@pytest.mark.parametrize('name', CASE_NAMES)
def test_every_case_reaches_its_regimes(name, sm):
    case = CASES[name]
    missing = set(case.tags) - case_regimes(case, sm)
    assert not missing, f'{name} at {sm} SMs: the case no longer reaches {sorted(missing)}'


@pytest.mark.parametrize('sm', SMS)
def test_the_cases_cover_every_regime(sm):
    seen = set()
    for case in CASES.values():
        seen |= case_regimes(case, sm)
    assert not set(REQUIRED) - seen, sorted(set(REQUIRED) - seen)


def test_expand_chunks_of_few_words_do_not_depend_on_the_occupancy():
    """With at most 4 words on 132 SMs, ``capacity // n_words >= 33``: the chunk count is ``min(32, ceil(n / 256))``
    at any occupancy."""
    for n_words in range(1, 5):
        for per_sm in range(1, 9):
            assert per_sm * 132 // n_words >= MAX_CHUNKS
    for name, case in CASES.items():
        if case.entry.startswith('expand') and case.n_words <= 4:
            p = plan(case, 132)
            assert p['chunks'] == p['chunks_asserted'] == min(MAX_CHUNKS, -(-p['n'] // 256)), name


# ---- fp32 emulation of make_taps and bicubic_shared -----------------------------------------------------------------

f32 = np.float32


def _fma(a, b, c):
    """fp32 fma: the product of two fp32 values is exact in float64; the sum rounds to float64 and then to fp32 (the
    rare double rounding is far inside the bound's slack)."""
    d = lambda x: np.asarray(x, dtype=np.float64)
    return (d(a) * d(b) + d(c)).astype(np.float32)


def emulate_taps(n_in: int, n_out: int, fused: bool):
    """``make_taps`` for every ``dst`` in fp32: ``(base [n_out] int, w [4, n_out] fp32)``."""
    a = f32(-0.75)
    d = np.arange(n_out, dtype=np.float32) + f32(0.5)
    scale = f32(n_in) / f32(n_out)
    src = _fma(scale, d, f32(-0.5)) if fused else (scale * d).astype(np.float32) - f32(0.5)
    fl = np.floor(src)
    t = (src - fl).astype(np.float32)

    def near(x):
        if fused:
            return _fma(_fma(a + f32(2), x, -(a + f32(3))) * x, x, f32(1))
        return (((a + f32(2)) * x - (a + f32(3))) * x * x + f32(1)).astype(np.float32)

    def far(x):
        if fused:
            return _fma(_fma(_fma(a, x, -f32(5) * a), x, f32(8) * a), x, -f32(4) * a)
        return (((a * x - f32(5) * a) * x + f32(8) * a) * x - f32(4) * a).astype(np.float32)

    w = np.stack([far(t + f32(1)), near(t), near(f32(1) - t), far(f32(2) - t)])
    return fl.astype(np.int64), w, src


def emulate_expand(word_map: np.ndarray, out_hw, fused: bool) -> np.ndarray:
    """``bicubic_shared`` of an fp32 word map ``[mh, mw]`` at every output pixel, fp32 ``[oh, ow]``."""
    mh, mw = word_map.shape
    by, wy, _ = emulate_taps(mh, out_hw[0], fused)
    bx, wx, _ = emulate_taps(mw, out_hw[1], fused)
    v = np.zeros(out_hw, dtype=np.float32)
    for i in range(4):
        rows = word_map[np.clip(by - 1 + i, 0, mh - 1)]                     # [oh, mw]
        r = np.zeros(out_hw, dtype=np.float32)
        for j in range(4):
            x = rows[:, np.clip(bx - 1 + j, 0, mw - 1)]                      # [oh, ow]
            r = _fma(wx[j][None, :], x, r) if fused else (r + wx[j][None, :] * x).astype(np.float32)
        v = _fma(wy[i][:, None], r, v) if fused else (v + wy[i][:, None] * r).astype(np.float32)
    return v


def emulate_normalize(v: np.ndarray) -> np.ndarray:
    lo, hi = v.min(), v.max()
    return ((v - lo).astype(np.float32) / ((hi - lo).astype(np.float32) + f32(1e-8))).astype(np.float32)


# ratios of the GPU table, and a grid of sides up to 320 against outputs up to 4096
TABLE_RATIOS = sorted({(c.grid[0], c.out[0]) for c in CASES.values()} | {(c.grid[1], c.out[1]) for c in CASES.values()})
GRID_IN = [1, 2, 3, 5, 7, 13, 16, 30, 50, 52, 64, 75, 76, 80, 96, 97, 100, 127, 128, 160, 200, 255, 319, 320]
GRID_OUT = [1, 2, 3, 7, 8, 9, 17, 40, 63, 65, 80, 90, 96, 129, 257, 300, 333, 512, 600, 768, 800, 832, 1000, 1023,
            1216, 1537, 2047, 2999, 4096]


def _row_difference(n_in: int, n_out: int, fused: bool) -> np.ndarray:
    """1-norm of (row of the bicubic matrix at the fp32 coordinate) - (row at the exact one), per ``dst``, over the
    unclamped taps (clamping merges taps, which can only shrink the difference). Weights in float64: this isolates the
    coordinate."""
    base32, _, src32 = emulate_taps(n_in, n_out, fused)
    src32 = src32.astype(np.float64)
    t32 = (src32 - np.floor(src32)).astype(np.float32).astype(np.float64)       # the kernel's t, rounded as it is
    w32 = O._cubic_weights(t32)
    src = (np.arange(n_out, dtype=np.float64) + 0.5) * (n_in / n_out) - 0.5
    base = np.floor(src).astype(np.int64)
    w64 = O._cubic_weights(src - base)
    lo = np.minimum(base, base32)
    dense = np.zeros((n_out, 6))
    rows = np.arange(n_out)
    for j in range(4):
        np.add.at(dense, (rows, base32 - lo + j), w32[j])
        np.add.at(dense, (rows, base - lo + j), -w64[j])
    return np.abs(dense).sum(1)


@pytest.mark.parametrize('fused', [False, True], ids=['separate', 'fma'])
def test_coordinate_term_bounds_the_fp32_taps(fused):
    pairs = {(i, o) for i in GRID_IN for o in GRID_OUT} | set(TABLE_RATIOS)
    worst = 0.0
    for n_in, n_out in sorted(pairs):
        diff = _row_difference(n_in, n_out, fused)
        bound = row_motion(n_in, n_out) + 1e-13              # + float64 rounding of src (up to 320) and the weights
        i = int(np.argmax(diff - bound))
        assert diff[i] <= bound[i], f'{n_in} -> {n_out}: row {i} moves by {diff[i]:.3e} > {bound[i]:.3e}'
        worst = max(worst, float(diff.max()) / 2.0 ** -24)
    assert worst > 100, 'the grid reaches no ratio whose coordinate rounds'


EMULATED = [((64, 64), (96, 96)), ((96, 96), (40, 40)), ((320, 160), (300, 300)), ((97, 97), (1000, 1000)),
            ((64, 80), (1, 7937)), ((2, 3), (16, 32)), ((1, 50), (1, 1537)), ((128, 128), (17, 65)),
            ((30, 50), (17, 63)), ((52, 76), (832, 1216))]


@pytest.mark.parametrize('fused', [False, True], ids=['separate', 'fma'])
@pytest.mark.parametrize('grid,out', EMULATED, ids=[f'{g[0]}x{g[1]}-{o[0]}x{o[1]}' for g, o in EMULATED])
def test_expand_bound_dominates_the_fp32_emulation(grid, out, fused):
    """Absolute and normalised maps of a two-row word (the fp32 row mean too) on signed and non-negative maps."""
    g = torch.Generator().manual_seed(grid[0] * 7 + out[1])
    for maps in (torch.rand(3, *grid, generator=g), torch.randn(3, *grid, generator=g) * 3):
        rows = [[1, 2]]
        x = maps.numpy().astype(np.float32)
        wm32 = ((f32(0) + x[1]) + x[2]).astype(np.float32) / f32(2)
        wm64 = word_maps64(maps, rows)
        v32 = emulate_expand(wm32, out, fused)
        for absolute in (True, False):
            exp = expand64(wm64, out, absolute)
            bound = expand_bound(wm64, out, absolute, [2], word_maps64(maps.abs(), rows), exp)[0].numpy()
            got = v32 if absolute else emulate_normalize(v32)
            err = np.abs(got.astype(np.float64) - exp.pre[0].numpy())
            assert (err <= bound).all(), f'absolute {absolute}: error {err.max():.3e}, bound there ' \
                                         f'{bound.reshape(-1)[np.argmax(err)]:.3e}'


# ---- the window estimate ------------------------------------------------------------------------------------------------

def test_window_estimate_covers_every_tile():
    """``min(n_in, ceil(T n_in / n_out) + 5) >= idx3(last) - idx0(first) + 1`` for every tile of ``T`` outputs (16 rows,
    64 columns; the last tile shorter), sides up to 320 and outputs below 1100, at either fp32 arithmetic.

    Beyond these sizes: the tile's taps span ``floor(src_last) + 2 - (floor(src_first) - 1) + 1`` indices, and
    ``src_last - src_first = (th - 1) n_in / n_out`` up to the fp32 errors (far below 1 at any side that fits the
    200 KB map), so ``floor(src_last) - floor(src_first) <= (T - 1) n_in / n_out + 1``; the window is at most
    ``(T - 1) n_in / n_out + 5 < ceil(T n_in / n_out) + 5``, and clamping only shrinks it. The estimate meets the
    window only where both are clamped to the side."""
    for T in (TILE_H, TILE_W):
        pairs = [(n_out, y0) for n_out in range(1, 1100) for y0 in range(0, n_out, T)]
        n_out = np.array([p[0] for p in pairs])
        y0 = np.array([p[1] for p in pairs])
        last = np.minimum(y0 + T, n_out) - 1
        d0, d1 = y0.astype(np.float32) + f32(0.5), last.astype(np.float32) + f32(0.5)
        for n_in in range(1, 321):
            scale = f32(n_in) / n_out.astype(np.float32)
            est = np.minimum(n_in, np.ceil(T * n_in / n_out).astype(np.int64) + 5)
            for fused in (False, True):
                src = [_fma(scale, d, f32(-0.5)) if fused else (scale * d).astype(np.float32) - f32(0.5)
                       for d in (d0, d1)]
                first = np.clip(np.floor(src[0]).astype(np.int64) - 1, 0, n_in - 1)
                lastc = np.clip(np.floor(src[1]).astype(np.int64) + 2, 0, n_in - 1)
                win = lastc - first + 1
                bad = win > est
                assert not bad.any(), f'T {T}, side {n_in}, output {n_out[bad][0]}, tile at {y0[bad][0]}: window ' \
                                      f'{win[bad][0]} > estimate {est[bad][0]}'


# ---- regimes that cannot occur --------------------------------------------------------------------------------------------

# ---- staging beside the pair and sweep buffers, and the instance rounds -----------------------------------------------

WINDOWS = np.arange(1, MAX_SMEM // 4 + 1)          # every window a map of at most 200 KB can have, in floats


def _check_staging(before: int, n_words, what: str):
    assert before <= MAX_SMEM, f'{what}: {before} bytes before the windows'
    for w in n_words:
        wpp = words_per_pass(w, WINDOWS, before)
        assert (before + wpp * WINDOWS * 4 <= MAX_SMEM).all(), f'{what}, {w} words: more than 200 KB'
        none = wpp == 0
        assert np.array_equal(none, WINDOWS * 4 > MAX_SMEM - before), \
            f'{what}, {w} words: no window staged at window {WINDOWS[none != (WINDOWS * 4 > MAX_SMEM - before)][0]}'
        assert (wpp >= 0).all() and (wpp <= w).all()


def test_pair_staging_stays_within_200KB():
    """For 1 to 96 words, with and without a threshold, and every window: ``pair_smem_bytes + words_per_pass * window
    <= 200 KB``, and no window is staged exactly when one does not fit beside the pair buffers."""
    for n_words in range(1, 97):
        for thr in (False, True):
            _check_staging(pair_smem_bytes(n_words, thr), [n_words], f'pair, threshold {thr}')


def test_sweep_staging_stays_within_200KB():
    """For R <= 63 regions, T <= 64 thresholds and every window, the same of ``sweep_smem_bytes``. The word count only
    caps ``words_per_pass`` from above, so 1, 2, 95 and 96 words stand for every count."""
    for before in sorted({sweep_smem_bytes(r, t) for r in range(1, 64) for t in range(1, 65)}):
        _check_staging(before, (1, 2, 95, 96), f'sweep, {before} bytes of histograms')


def test_the_table_reaches_the_staging_boundaries():
    """The sweep rows of the table sit on both sides of the boundary: a 196 KB window beside 512 bins fits once,
    beside 513 it does not."""
    assert plan(CASES['sweep-one-window-fits'], 132)['fits'] == 1
    assert plan(CASES['sweep-not-staged-513'], 132)['fits'] == 0
    assert sweep_smem_bytes(7, 64) + 224 * 224 * 4 == MAX_SMEM


ROUND_SHAPES = [(1, 1), (1, 5), (3, 5), (7, 2), (4, 96), (2, 33)]


@pytest.mark.parametrize('n_maps,n_words', ROUND_SHAPES, ids=[f'{m}x{w}' for m, w in ROUND_SHAPES])
def test_instance_rounds_split_the_planes(n_maps, n_words):
    """For every scratch size from one plane to all of them and past: each (map, word) plane is in exactly one round,
    no round has more than ``cap`` planes (nor 65535), and a round takes several maps only when every round takes
    whole maps."""
    planes = n_maps * n_words
    for cap in list(range(1, planes + 3)) + [MAX_ROUND_PLANES]:
        rounds = instance_rounds(n_maps, n_words, cap)
        seen = np.zeros((n_maps, n_words), np.int64)
        for m0, nm, w0, nw in rounds:
            assert 1 <= nm * nw <= min(cap, MAX_ROUND_PLANES), (cap, m0, w0)
            seen[m0:m0 + nm, w0:w0 + nw] += 1
        assert (seen == 1).all(), cap
        if any(nm > 1 for _, nm, _, _ in rounds):
            assert all(nw == n_words for _, _, _, nw in rounds), cap


def test_instance_rounds_at_the_plane_limit():
    """65535 maps of 96 words with room for every plane: 65535-plane rounds of 682 whole maps."""
    rounds = instance_rounds(65535, 96, MAX_ROUND_PLANES)
    assert all(nw == 96 and nm * nw <= MAX_ROUND_PLANES for _, nm, _, nw in rounds)
    assert sum(nm for _, nm, _, _ in rounds) == 65535 and rounds[0][1] == 682


def test_unreachable_regimes():
    """* Several ``expand_words`` launches need more words than ``capacity = per_sm * sm_count >= sm_count``; a call
      has at most 96 words, so they need fewer than 96 SMs, and every H100 has 114 or 132.
    * An empty expand chunk (``begin = chunk * per >= n``) needs ``(chunks - 1) * ceil(n / chunks) >= n``, which
      ``chunks <= ceil(n / 256)`` rules out: ``chunks * (chunks - 1) >= n`` would be needed, and ``chunks <= 32``.
    * A round of several word-instance maps whose words are split: ``maps_per_round = max(1, cap // n_words) > 1``
      needs ``cap >= 2 n_words``, and then ``words_per_round = min(cap, n_words)`` is every word."""
    for n_words in range(1, 97):
        for cap in range(1, 3 * n_words):
            if max(1, cap // n_words) > 1:
                assert min(cap, n_words) == n_words
    for sm in (114, 132):
        for n_words in range(1, 97):
            for mh, mw in ((1, 1), (64, 64), (320, 160)):
                case = Case('expand', (mh, mw), (64, 64), n_words=n_words)
                assert plan(case, sm)['launches'] == 1
                assert expand_per_sm(mh, mw) * sm >= n_words
    for n in range(1, 256 * 40):
        for chunks in range(1, min(MAX_CHUNKS, -(-n // 256)) + 1):
            per = -(-n // chunks)
            assert (chunks - 1) * per < n, (n, chunks)
