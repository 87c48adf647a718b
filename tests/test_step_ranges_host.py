"""Host-side rules of trace(pipe, step_ranges=[...]) that need no GPU: the option is keyword-only and off by default,
every invalid value or combination is refused at construction, before the native library or the pipeline is touched,
and reads that name a step range fail loudly on a trace without ranges."""
import inspect

import pytest
import torch

from daam_b200 import trace
from daam_b200.heatmap import RawHeatMapCollection
from daam_b200.testing.synthetic import TINY_SPEC, make_pipeline
from daam_b200.trace import _normalize_step_ranges


class Untouchable:
    """A pipeline stand-in that fails on any attribute access: proves the check runs before anything else."""

    def __getattr__(self, name):
        raise AssertionError(f'pipeline.{name} was accessed')


@pytest.fixture
def no_native(monkeypatch):
    from daam_b200 import _native
    monkeypatch.setattr(_native, 'load', lambda: (_ for _ in ()).throw(AssertionError('native library touched')))


@pytest.mark.parametrize('ranges,match', [
    ([], 'at least one range'),
    ([(-1, 3)], '0 <= start < stop'),
    ([(3, 3)], '0 <= start < stop'),
    ([(4, 2)], '0 <= start < stop'),
    ([range(0, 10, 2)], 'step 1'),
    ([range(5, 2)], '0 <= start < stop'),
    ([(0, 5), (4, 8)], 'overlap'),
    ([(4, 8), range(0, 5)], 'overlap'),
    ([(0, 10), (2, 3)], 'overlap'),
    ([(0, 1, 2)], r'\(start, stop\) tuple'),
    ([[0, 1]], r'\(start, stop\) tuple'),
    ([(0.0, 1)], r'\(start, stop\) tuple'),
    ([(True, 2)], r'\(start, stop\) tuple'),
    ((0, 5), 'list of'),
    (range(0, 5), 'list of'),
    (3, 'list of'),
])
def test_invalid_ranges_are_refused_up_front(ranges, match, no_native):
    with pytest.raises(ValueError, match=match):
        trace(Untouchable(), step_ranges=ranges)


@pytest.mark.parametrize('kw,match', [
    ({'launch': 'overlap'}, "launch='step'"),
    ({'launch': 'layer'}, "launch='step'"),
    ({'save_heads': True}, 'save_heads / load_heads'),
    ({'load_heads': True}, 'save_heads / load_heads'),
    ({'time_resolved': True}, 'time_resolved'),
])
def test_unsupported_combinations_are_refused_up_front(kw, match, no_native):
    with pytest.raises(ValueError, match=match):
        trace(Untouchable(), step_ranges=[(0, 2)], **kw)


def test_option_is_keyword_only_and_off_by_default():
    p = inspect.signature(trace.__init__).parameters['step_ranges']
    assert p.kind is inspect.Parameter.KEYWORD_ONLY and p.default is None
    for fn in (trace.compute_global_heat_map, trace.compute_per_head_heat_maps, RawHeatMapCollection.items):
        p = inspect.signature(fn).parameters['step_range']
        assert p.kind is inspect.Parameter.KEYWORD_ONLY and p.default is None, fn


def test_ranges_are_normalised_in_declared_order():
    assert _normalize_step_ranges([(5, 8), range(0, 5), range(10, 11, 1)]) == [(5, 8), (0, 5), (10, 11)]
    assert _normalize_step_ranges(iter([(0, 1)])) == [(0, 1)]


def test_reads_need_the_option():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float32, device='cpu', seed=0)
    tc = trace(pipe)
    assert tc.step_ranges is None and tc.all_heat_maps.n_ranges == 0 and tc._slab_ptrs == []
    for read in (lambda: tc.compute_global_heat_map(step_range=0), lambda: tc.compute_per_head_heat_maps(step_range=0),
                 lambda: list(tc.all_heat_maps.items(step_range=0))):
        with pytest.raises(RuntimeError, match='step_ranges'):
            read()
    tc = trace(pipe, step_ranges=[range(2, 4), (0, 2)])
    assert tc.step_ranges == [(2, 4), (0, 2)] and tc.all_heat_maps.n_ranges == 2 and len(tc._slab_ptrs) == 2
    assert tc.step_range_counts == [0, 0]
    with pytest.raises(IndexError):
        tc.compute_global_heat_map(step_range=2)
    with pytest.raises(RuntimeError, match='No heat maps found for the given parameters'):
        list(tc.all_heat_maps.items(step_range=1))
