"""Host-side rules of trace(pipe, time_resolved=True) that need no GPU: the option combinations it does not support are
refused at construction, before the pipeline or the device is touched, and the per-step accessor fails loudly."""
import inspect

import pytest
import torch

from daam_b200 import GlobalHeatMap, TimeHeatMaps, trace
from daam_b200.testing.synthetic import TINY_SPEC, make_pipeline


class Untouchable:
    """A pipeline stand-in that fails on any attribute access: proves the check runs before anything else."""

    def __getattr__(self, name):
        raise AssertionError(f'pipeline.{name} was accessed')


@pytest.mark.parametrize('kw,match', [
    ({'launch': 'overlap'}, "launch='step'"),
    ({'launch': 'layer'}, "launch='step'"),
    ({'save_heads': True}, 'save_heads / load_heads'),
    ({'load_heads': True}, 'save_heads / load_heads'),
])
def test_unsupported_combinations_are_refused_up_front(kw, match, monkeypatch):
    from daam_b200 import _native
    monkeypatch.setattr(_native, 'load', lambda: (_ for _ in ()).throw(AssertionError('native library touched')))
    with pytest.raises(ValueError, match=match):
        trace(Untouchable(), time_resolved=True, **kw)


def test_option_is_keyword_only_and_off_by_default():
    p = inspect.signature(trace.__init__).parameters['time_resolved']
    assert p.kind is inspect.Parameter.KEYWORD_ONLY and p.default is False


def test_accessor_needs_the_mode_and_a_generation():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float32, device='cpu', seed=0)
    tc = trace(pipe)
    assert tc.all_heat_maps.time_resolved is False and tc._slab_ptrs == []
    with pytest.raises(RuntimeError, match='time_resolved=True'):
        tc.compute_time_heat_maps()
    tc = trace(pipe, time_resolved=True)
    assert tc.all_heat_maps.time_resolved is True and len(tc._slab_ptrs) == 1
    with pytest.raises(RuntimeError, match='No heat maps found'):
        tc.compute_time_heat_maps()


def test_time_heat_maps_container():
    maps = torch.arange(3 * 4 * 2 * 2, dtype=torch.float32).view(3, 4, 2, 2)
    tm = TimeHeatMaps(None, 'a cat', maps)
    assert len(tm) == 3
    step = tm[1]
    assert isinstance(step, GlobalHeatMap) and step.prompt == 'a cat' and torch.equal(step.heat_maps, maps[1])
    assert torch.equal(tm[-1].heat_maps, maps[2])
