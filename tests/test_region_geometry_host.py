"""Host checks of the ranking, boundary and CRF geometry table (``tests/test_region_geometry_gpu.py``), without a GPU.

* Every case reaches the regimes it names, and the table covers every regime. None of the launch rules depends on the
  SM count: grids are sized from the plane, the tile and the label count alone, so there is no SM count to vary.
* ``plan``'s scratch arithmetic equals the sizes ``daam_b200._native`` states for the C ABI.
* The round split of daam_region_ranking / daam_region_boundary / daam_mask_boundary takes every (map, word) plane
  exactly once, for every word count from 1 to 96 and every cap from 1 to 200; the CRF's takes every map once.
* The planted data: values whose descending keys differ in one byte only, and tie groups where the table says."""
import numpy as np
import pytest

from daam_b200 import _native
from tests.test_region_geometry_gpu import (CASE_NAMES, CASES, KEY_BASES, REQUIRED, SEGMENT, boundary_call_bytes,
                                            boundary_plane_bytes, boundary_tile_rows, case_regimes, cdiv, chunk_size,
                                            crf_map_bytes, crf_rounds, from_keys, make_data, plan, plane_rounds,
                                            ranking_plane_bytes, scan_steps, step_smem)

REGIMES = {name: case_regimes(name) for name in CASE_NAMES}


@pytest.mark.parametrize('name', CASE_NAMES)
def test_every_case_reaches_its_regimes(name):
    missing = set(CASES[name].tags) - REGIMES[name]
    assert not missing, f'{name}: the case no longer reaches {sorted(missing)}'


def test_the_cases_cover_every_regime():
    seen = set().union(*REGIMES.values())
    assert not set(REQUIRED) - seen, sorted(set(REQUIRED) - seen)


SIZES = [(1, 1), (1, 31), (2, 16), (1, 33), (31, 33), (32, 32), (1, 1025), (64, 64), (64, 65), (256, 256), (1, 65537),
         (600, 800), (1025, 2049), (4096, 4096), (1, 1 << 24), (131072, 1), (4097, 1), (17, 256), (33, 129)]


@pytest.mark.parametrize('h,w', SIZES, ids=[f'{h}x{w}' for h, w in SIZES])
def test_scratch_arithmetic(h, w):
    assert ranking_plane_bytes(h, w) == _native.region_ranking_plane_bytes(h, w)
    for planes in (1, 2, 15):
        assert 8 * h * w + planes * ranking_plane_bytes(h, w) == _native.region_ranking_scratch_bytes(planes, h, w)
    assert boundary_tile_rows(w) == _native.boundary_tile_rows(w)
    assert boundary_plane_bytes(h, w) == _native.boundary_plane_bytes(h, w)
    for r in (1, 3, 63):
        assert boundary_call_bytes(r, h, w) == _native.boundary_call_bytes(r, h, w)
        assert boundary_call_bytes(r, h, w) + 7 * boundary_plane_bytes(h, w) == \
            _native.boundary_scratch_bytes(r, 7, h, w)
    for L in (1, 13, 16, 17, 97):
        assert crf_map_bytes(L, h, w) == _native.crf_map_bytes(L, h, w)
        assert 3 * crf_map_bytes(L, h, w) == _native.crf_scratch_bytes(3, L, h, w)


def test_case_scratch_matches_the_abi():
    for name, case in CASES.items():
        p = plan(case)
        oh, ow = case.out
        for cap, s in zip(case.caps, p['scratch']):
            planes = cap or case.planes
            if case.entry == 'ranking':
                want = _native.region_ranking_scratch_bytes(planes, oh, ow)
            elif case.entry == 'crf':
                want = _native.crf_scratch_bytes(cap or case.n_maps, case.n_labels, oh, ow)
            else:
                want = _native.boundary_scratch_bytes(case.n_regions, planes, oh, ow)
            assert s == want, name


def test_plane_rounds_take_every_plane_once():
    """Every word count 1..96 and cap 1..200 over 1, 3 and 7 maps: each plane in exactly one round, no round above the
    cap, and several maps in a round only when every round takes whole maps."""
    for n_maps in (1, 3, 7):
        for n_words in range(1, 97):
            for cap in range(1, 201):
                seen = np.zeros((n_maps, n_words), np.int64)
                rounds = plane_rounds(n_maps, n_words, cap)
                for m0, nm, w0, nw in rounds:
                    assert 1 <= nm * nw <= cap, (n_maps, n_words, cap)
                    seen[m0:m0 + nm, w0:w0 + nw] += 1
                assert (seen == 1).all(), (n_maps, n_words, cap)
                if any(nm > 1 for _, nm, _, _ in rounds):
                    assert all(nw == n_words for _, _, _, nw in rounds)


def test_plane_rounds_at_the_plane_limit():
    rounds = plane_rounds(65535, 96, 1 << 40)
    assert all(nw == 96 and nm * nw <= 65535 for _, nm, _, nw in rounds) and rounds[0][1] == 682


def test_crf_rounds_take_every_map_once():
    for n_maps in range(1, 12):
        for per in range(1, 14):
            rounds = crf_rounds(n_maps, per * 1000 + 999, 1000)
            assert [m for m0, nm in rounds for m in range(m0, m0 + nm)] == list(range(n_maps))
            assert all(nm <= per for _, nm in rounds)


def test_crf_chunks():
    """chunk_size: one chunk up to 16 labels, whole chunks of at most 16, the last chunk nonempty, and the 174 KB
    launch only at kC 16 and radius 16, within the 227 KB an H100 CTA may take."""
    for L in range(1, 98):
        kc = chunk_size(L)
        chunks = cdiv(L, kc)
        assert kc % 4 == 0 and kc <= 16 and (chunks == 1) == (L <= 16)
        assert chunks == cdiv(L, 16) and L - (chunks - 1) * kc >= 1
    assert step_smem(16, 16) == 174080 <= 227 * 1024
    assert max(step_smem(r, k) for r in range(1, 17) for k in (4, 8, 12, 16) if (r, k) != (16, 16)) < 174080


def test_scan_steps():
    assert scan_steps(33, 0, [(32, 32 * 32)]) == 2 and scan_steps(33, 32, [(32, 32 * 32)]) == 2
    assert scan_steps(40, 0, [(1, 1601), (33, 1089)]) == 2 and scan_steps(40, 0, [(1, 1601)]) == 2
    assert scan_steps(40, 0, [(1, 1)]) == 1 and scan_steps(40, 0, [(5, 2000)]) == 2
    assert scan_steps(1 << 17, 0, [((1 << 17) - 1, ((1 << 17) - 1) ** 2)]) == 1 << 12


@pytest.mark.parametrize('k', range(4))
def test_key_byte_planes_differ_in_one_byte(k):
    """``from_keys`` inverts descending_key (-0 folded, orderable bits, inverted), and the key-byte planes' keys share
    every byte but byte ``k``."""
    base, lo, hi = KEY_BASES[k]
    digits = np.arange(lo, hi, dtype=np.uint32)
    keys = np.uint32(base) & ~np.uint32(0xFF << (8 * k)) | (digits << np.uint32(8 * k))
    f = from_keys(keys)
    assert np.isfinite(f).all() and (np.abs(f[f != 0]) >= np.finfo(np.float32).tiny).all()
    u = f.view(np.uint32)
    back = ~np.where(u & np.uint32(0x80000000), ~u, u | np.uint32(0x80000000)).astype(np.uint32)
    assert np.array_equal(back, keys)
    assert np.array_equal(np.argsort(-f.astype(np.float64), kind='stable'), np.argsort(keys, kind='stable'))


def test_planted_groups():
    d = make_data(CASES['rank-groups'], 'rank-groups')
    s = d['starts']
    assert {0, 1, 90, 100, 2 * SEGMENT, 3 * SEGMENT - 1, 4 * SEGMENT - 100, 7 * SEGMENT + 10, 40959} <= set(s.tolist())
    assert not ((s > 4 * SEGMENT - 100) & (s < 7 * SEGMENT + 10)).any()
    values = d['planes'][0, 0].reshape(-1)
    assert np.array_equal(values[d['order']], np.sort(values)[::-1])
