"""Head-reduced joint-attention traces without a GPU: the argument checks of daam_accumulate_joint_heads, which run
before any device call, the refusal of reduce_heads=True on UNet pipelines and with every option a joint trace
refuses, the refused per-head reads, and the one-head-count rule of the slabs."""
import pytest
import torch

from daam_b200 import _native, trace
from daam_b200.build import build
from daam_b200.heatmap import RawHeatMapCollection
from daam_b200.testing.synthetic import TINY_FLUX_SPEC, TINY_SD3_SPEC, TINY_SPEC, make_flux_pipeline, \
    make_pipeline, make_sd3_pipeline
from daam_b200.trace import JOINT_REFUSED


@pytest.fixture(scope='module')
def lib():
    build()
    return _native.load()


@pytest.fixture(scope='module')
def sd3(lib):
    return make_sd3_pipeline(TINY_SD3_SPEC)


@pytest.fixture(scope='module')
def flux(lib):
    return make_flux_pipeline(TINY_FLUX_SPEC)


def _layer(**kw):
    base = dict(q=16, k=16, acc=16, q_stride_prompt=0, q_stride_pixel=64, q_stride_head=64, k_stride_prompt=0,
                k_stride_token=64, k_stride_head=64, n_prompts=1, heads=24, hw=64, tokens=333, head_dim=64,
                dtype=_native.DAAM_BF16, scale=0.125, reserved=0, lse=16, lse_stride_prompt=64, lse_stride_head=64,
                lse_stride_pixel=1)
    base.update(kw)
    return _native.DaamJointLayer(**base)


@pytest.mark.parametrize('kw, code, text', [
    (dict(q=None), _native.E_INVALID, 'null pointer'),
    (dict(k=None), _native.E_INVALID, 'null pointer'),
    (dict(acc=None), _native.E_INVALID, 'null pointer'),
    (dict(lse=None), _native.E_INVALID, 'null pointer'),
    (dict(acc=20), _native.E_INVALID, 'not 16-byte aligned'),
    (dict(acc=24), _native.E_INVALID, 'not 16-byte aligned'),
    (dict(tokens=0), _native.E_UNSUPPORTED, 'tokens = 0'),
    (dict(tokens=1025), _native.E_UNSUPPORTED, 'tokens = 1025'),
    (dict(head_dim=12), _native.E_UNSUPPORTED, 'head_dim = 12'),
    (dict(head_dim=264), _native.E_UNSUPPORTED, 'head_dim = 264'),
    (dict(hw=0), _native.E_INVALID, 'non-positive'),
    (dict(heads=0), _native.E_INVALID, 'non-positive'),
    (dict(n_prompts=-1), _native.E_INVALID, 'non-positive'),
    (dict(dtype=7), _native.E_INVALID, 'unknown dtype'),
    (dict(scale=0.0), _native.E_INVALID, 'scale'),
])
def test_accumulate_joint_heads_argument_validation(lib, kw, code, text):
    with pytest.raises(_native.NativeError, match=text) as e:
        _native.accumulate_joint_heads([_layer(), _layer(**kw)], 0)
    assert e.value.code == code
    assert 'daam_accumulate_joint_heads: layer 1' in str(e.value)


def test_accumulate_joint_heads_takes_no_flags(lib):
    array = (_native.DaamJointLayer * 1)(_layer())
    assert lib.daam_accumulate_joint_heads(array, 1, 1, None) == _native.E_INVALID
    assert 'flags = 1' in lib.daam_last_error().decode()
    assert lib.daam_accumulate_joint_heads(None, 1, 0, None) == _native.E_INVALID
    assert lib.daam_accumulate_joint_heads(array, -1, 0, None) == _native.E_INVALID
    assert lib.daam_accumulate_joint_heads(None, 0, 0, None) == 0


def test_the_head_free_slab_size_limit_is_its_own(lib):
    """The size check counts the head-free slab: 2^40 elements with the heads, 2^40 / 64 without."""
    big = dict(n_prompts=1 << 10, tokens=1024, hw=1 << 20, heads=64)
    with pytest.raises(_native.NativeError, match='too large'):
        _native.accumulate_joint([_layer(**big)], 0)
    if not torch.cuda.is_available():
        with pytest.raises(_native.NativeError) as e:
            _native.accumulate_joint_heads([_layer(**big)], 0)
        assert e.value.code == _native.E_CUDA


@pytest.mark.skipif(torch.cuda.is_available(), reason='checks the no-device behaviour')
def test_accumulate_joint_heads_has_no_cpu_fallback(lib):
    with pytest.raises(_native.NativeError) as e:
        _native.accumulate_joint_heads([_layer(tokens=1), _layer(tokens=1024, head_dim=256)], 0)
    assert e.value.code == _native.E_CUDA


def test_a_unet_trace_refuses_reduce_heads(lib):
    with pytest.raises(ValueError, match='reduce_heads=True needs a joint-attention.*upsamples and clamps'):
        trace(make_pipeline(TINY_SPEC), reduce_heads=True)


@pytest.mark.parametrize('name', JOINT_REFUSED)
@pytest.mark.parametrize('model', ['sd3', 'flux'])
def test_reduce_heads_with_a_refused_option_raises(request, model, name):
    pipe = request.getfixturevalue(model)
    value = [(0, 1)] if name == 'step_ranges' else True
    with pytest.raises(ValueError, match=f'{name} is not supported when tracing the joint attention'):
        trace(pipe, reduce_heads=True, **{name: value})


@pytest.mark.parametrize('model', ['sd3', 'flux'])
def test_reduce_heads_refuses_the_overlap_launch(request, model):
    with pytest.raises(ValueError, match="launch='overlap' is not supported"):
        trace(request.getfixturevalue(model), reduce_heads=True, launch='overlap')


@pytest.mark.parametrize('model', ['sd3', 'flux'])
def test_the_option_reaches_the_collection(request, model):
    tc = trace(request.getfixturevalue(model), reduce_heads=True)
    assert tc.reduce_heads and tc.all_heat_maps.reduce_heads
    assert not trace(request.getfixturevalue(model)).all_heat_maps.reduce_heads


@pytest.mark.parametrize('model', ['sd3', 'flux'])
def test_head_idx_and_per_head_reads_are_refused(request, model):
    tc = trace(request.getfixturevalue(model), reduce_heads=True)
    for read in (tc.compute_global_heat_map, tc.compute_layer_heat_maps, tc.compute_factor_heat_maps,
                 tc.compute_image_heat_maps):
        with pytest.raises(ValueError, match='head_idx selects one head.*reduce_heads=True'):
            read(head_idx=0)
    for read in (tc.compute_per_head_heat_maps, tc.compute_head_heat_maps, lambda: list(tc.all_heat_maps.items()),
                 lambda: list(tc.all_heat_maps)):
        with pytest.raises(RuntimeError, match='reduce_heads=True'):
            read()


def test_every_layer_must_average_the_same_number_of_heads():
    coll = RawHeatMapCollection()
    coll.joint = coll.reduce_heads = True
    a = coll.slab_for(0, 1, 2, 3, 4, 5, 'cpu', images=3, tokens=93, head_mean=24)
    assert tuple(a.acc.shape) == (2, 3, 93, 20) and a.heads == 3 and a.heads_per_image == 1 and a.head_mean == 24
    coll.slab_for(1, 1, 2, 3, 4, 5, 'cpu', images=3, tokens=93, head_mean=24)
    coll.slab_for(0, 1, 2, 3, 4, 5, 'cpu', images=3, tokens=93, head_mean=24)   # the same layer again
    with pytest.raises(RuntimeError, match='layer 2: 12 heads, but layer 0 of the same trace has 24'):
        coll.slab_for(2, 1, 2, 3, 4, 5, 'cpu', images=3, tokens=93, head_mean=12)
    coll.clear()                                   # a new generation may use another head count
    assert coll.slab_for(2, 1, 2, 3, 4, 5, 'cpu', images=3, tokens=93, head_mean=12).head_mean == 12
