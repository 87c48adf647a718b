"""Host side of the layer-, factor- and head-resolved heat maps: the stable partition of a read's groups by factor, the
daam_map_part binding against the header, the argument errors of the binding (raised before the library is loaded) and
the labels of the three stacks. No kernel is launched here."""
import ctypes
import os
import subprocess
import tempfile

import pytest
import torch

from daam_b200 import _native
from daam_b200.heatmap import FactorHeatMaps, GlobalHeatMap, GlobalHeatMapStack, HeadHeatMaps, LayerHeatMaps
from daam_b200.testing.synthetic import WhitespaceTokenizer
from daam_b200.trace import _factor_parts

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_factor_partition_is_stable():
    # SD-2.1's traced layers in call order: down 1 1 2 2 4 4, up 4 4 4 2 2 2 1 1 1
    factors = [1, 1, 2, 2, 4, 4, 4, 4, 4, 2, 2, 2, 1, 1, 1]
    order, found, parts = _factor_parts(factors)
    assert found == [1, 2, 4] and parts == [(0, 5), (5, 5), (10, 5)]
    assert order == [0, 1, 12, 13, 14, 2, 3, 9, 10, 11, 4, 5, 6, 7, 8]
    for f, (begin, count) in zip(found, parts):           # each run: the groups a read of that factor alone passes
        assert order[begin:begin + count] == [i for i, g in enumerate(factors) if g == f]
    assert _factor_parts([4]) == ([0], [4], [(0, 1)])
    assert _factor_parts([2, 1, 2, 1]) == ([1, 3, 0, 2], [1, 2], [(0, 2), (2, 2)])
    assert _factor_parts([4, 4, 2]) == ([2, 0, 1], [2, 4], [(0, 1), (1, 2)])
    assert _factor_parts([]) == ([], [], [])


def test_map_part_layout_matches_the_header():
    src = r'''
#include <stdio.h>
#include <stddef.h>
#include "daam_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu\n", sizeof(daam_map_part), offsetof(daam_map_part, group_begin),
         offsetof(daam_map_part, group_count), offsetof(daam_map_part, n_rows), offsetof(daam_map_part, reserved),
         offsetof(daam_map_part, out));
  printf("%zu %d\n", sizeof(daam_map_sel), DAAM_FINALIZE_MAX_MAPS);
  return 0;
}'''
    with tempfile.TemporaryDirectory() as tmp:
        c, exe = os.path.join(tmp, 't.c'), os.path.join(tmp, 't')
        open(c, 'w').write(src)
        subprocess.check_call(['gcc', '-std=c99', '-I', os.path.join(ROOT, 'include'), c, '-o', exe])  # header is plain C
        lines = subprocess.check_output([exe], text=True).split('\n')
    P = _native.DaamMapPart
    assert [int(v) for v in lines[0].split()] == [ctypes.sizeof(P), P.group_begin.offset, P.group_count.offset,
                                                   P.n_rows.offset, P.reserved.offset, P.out.offset]
    assert [int(v) for v in lines[1].split()] == [ctypes.sizeof(_native.DaamMapSel), _native.FINALIZE_MAX_MAPS]
    assert 'daam_finalize_parts' in _native.EXPORTS


def test_argument_errors_come_before_the_library(monkeypatch):
    def no_load():
        raise AssertionError('the library was loaded before the arguments were checked')
    monkeypatch.setattr(_native, 'load', no_load)
    groups = [_native.DaamKeyGroup(acc=16, heads=2, h=4, w=4, tokens=77, head_sel=-1, n_blocks=0)] * 3

    def part(**kw):
        d = dict(group_begin=0, group_count=1, n_rows=4, out=16)
        d.update(kw)
        return _native.DaamMapPart(**d)

    for parts, msg in [([], 'no output map'), ([part(group_begin=-1)], r'map 0 reads groups \[-1, \+1\) of 3'),
                       ([part(), part(group_count=0)], r'map 1 reads groups \[0, \+0\) of 3'),
                       ([part(group_begin=2, group_count=2)], r'map 0 reads groups \[2, \+2\) of 3'),
                       ([part(n_rows=0)], 'map 0 has no rows or no output'),
                       ([part(out=None)], 'map 0 has no rows or no output')]:
        with pytest.raises(ValueError, match=msg):
            _native.finalize_parts(groups, parts, 16, False, 0)
    with pytest.raises(AssertionError, match='was loaded'):      # a good call does reach the library
        _native.finalize_parts(groups, [part(group_count=3)], (16, 16), False, 0)


def test_stack_labels_and_items():
    tok, prompt = WhitespaceTokenizer(), 'a dog and a ball'
    maps = torch.arange(3 * 7 * 4 * 4, dtype=torch.float32).view(3, 7, 4, 4)
    by_layer = LayerHeatMaps(tok, prompt, maps, [0, 1, 5], ['down.a', 'down.b', 'up.c'], [1, 2, 4])
    assert (by_layer.layers, by_layer.names, by_layer.factors) == ([0, 1, 5], ['down.a', 'down.b', 'up.c'], [1, 2, 4])
    by_factor = FactorHeatMaps(tok, prompt, maps, (1, 2, 4))
    assert by_factor.factors == [1, 2, 4]
    by_head = HeadHeatMaps(tok, prompt, maps, [(1, 0, 0), (1, 0, 1), (2, 1, 0)])
    assert by_head.keys == [(1, 0, 0), (1, 0, 1), (2, 1, 0)]
    for stack in (by_layer, by_factor, by_head):
        assert isinstance(stack, GlobalHeatMapStack) and len(stack) == 3
        one = stack[1]
        assert isinstance(one, GlobalHeatMap) and one.prompt == prompt and torch.equal(one.heat_maps, maps[1])
    with pytest.raises(ValueError, match='LayerHeatMaps: 2 names for 3 maps'):
        LayerHeatMaps(tok, prompt, maps, [0, 1, 5], ['a', 'b'], [1, 2, 4])
    with pytest.raises(ValueError, match='FactorHeatMaps: 2 factors for 3 maps'):
        FactorHeatMaps(tok, prompt, maps, [1, 2])
    with pytest.raises(ValueError, match='HeadHeatMaps: 4 keys for 3 maps'):
        HeadHeatMaps(tok, prompt, maps, [(1, 0, 0)] * 4)
