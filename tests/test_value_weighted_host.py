"""Value-weighted heat maps without a GPU: the option's refusals raise before any native call, and a weighted read of a
trace without value norms raises."""
import pytest
import torch

from daam_b200 import _native, trace
from daam_b200.heatmap import LayerSlab
from daam_b200.testing.synthetic import TINY_SPEC, make_pipeline


@pytest.fixture
def pipe():
    return make_pipeline(TINY_SPEC, dtype=torch.float32, device='cpu', seed=0)


@pytest.fixture
def no_native(monkeypatch):
    """Every foreign call fails the test: what is checked here must raise before the library is used."""
    def refuse(*_a, **_k):
        raise AssertionError('a native call was made')
    monkeypatch.setattr(_native, 'value_norms', refuse)
    monkeypatch.setattr(_native, 'finalize_parts', refuse)
    monkeypatch.setattr(_native, 'finalize_per_key', refuse)
    monkeypatch.setattr(_native, 'finalize', refuse)


@pytest.mark.parametrize('option', ['save_heads', 'load_heads'])
def test_save_and_load_heads_are_refused(pipe, option, monkeypatch, tmp_path):
    monkeypatch.setattr(_native, 'load', lambda: (_ for _ in ()).throw(AssertionError('the library was loaded')))
    with pytest.raises(ValueError, match='value_norms=True does not support save_heads / load_heads'):
        trace(pipe, value_norms=True, data_dir=str(tmp_path), **{option: True})


class _Scaled(torch.nn.Module):
    """An output projection that is not a plain nn.Linear: a LoRA-like wrapper whose weight is not what it applies."""

    def __init__(self, base):
        super().__init__()
        self.base = base
        self.weight = base.weight

    def forward(self, x):
        return 2 * self.base(x)


class _LoraLinear(torch.nn.Linear):
    def forward(self, x):
        return super().forward(x) * 1.5


@pytest.mark.parametrize('kind', ['wrapper', 'subclass', 'hooked'])
def test_an_output_projection_that_is_not_a_plain_linear_is_refused(pipe, no_native, kind):
    for attn in [m for name, m in pipe.unet.named_modules() if name.endswith('attn2')]:
        base = attn.to_out[0]
        if kind == 'wrapper':
            attn.to_out[0] = _Scaled(base)
        elif kind == 'subclass':
            proj = _LoraLinear(base.in_features, base.out_features)
            proj.load_state_dict(base.state_dict())
            attn.to_out[0] = proj
        else:
            base.register_forward_hook(lambda m, i, o: o * 2)
    with trace(pipe, value_norms=True):
        with pytest.raises(RuntimeError, match='plain nn.Linear'):
            pipe('a dog', num_inference_steps=1)


def test_a_diffusers_style_lora_linear_without_lora_is_accepted(pipe):
    from daam_b200.trace import _check_value_norms

    class LoRACompatibleLinear(torch.nn.Linear):      # diffusers' form: a LoRA layer set in place, or None
        def __init__(self, *args):
            super().__init__(*args)
            self.lora_layer = None

        def forward(self, x):
            return super().forward(x)

    attn = next(m for name, m in pipe.unet.named_modules() if name.endswith('attn2'))
    attn.to_out[0] = LoRACompatibleLinear(4, 4)
    _check_value_norms(0, attn)                          # no raise
    attn.to_out[0].lora_layer = torch.nn.Identity()
    with pytest.raises(RuntimeError, match='plain nn.Linear'):
        _check_value_norms(0, attn)


def _fake_slab(tc, norms: bool):
    acc = torch.zeros(1, 2, 77, 16)
    slab = LayerSlab(0, 1, 2, 4, 4, acc, touched=True)
    if norms:
        slab.norms = torch.zeros(1, 2, 77)
        slab.norms_changed = torch.zeros((), dtype=torch.bool)
    tc.all_heat_maps.slabs[0] = slab
    tc.all_heat_maps._order = [0]
    tc.last_prompt = 'a dog'


READS = ['compute_global_heat_map', 'compute_layer_heat_maps', 'compute_factor_heat_maps',
         'compute_per_head_heat_maps', 'compute_head_heat_maps']


@pytest.mark.parametrize('read', READS)
def test_a_weighted_read_needs_the_option(pipe, no_native, read):
    with trace(pipe) as tc:
        _fake_slab(tc, norms=False)
        with pytest.raises(RuntimeError, match=r'trace\(pipe, value_norms=True\)'):
            getattr(tc, read)(value_weighted=True)
        with pytest.raises(RuntimeError, match=r'trace\(pipe, value_norms=True\)'):
            tc.compute_value_norms()


@pytest.mark.parametrize('read', READS)
def test_a_weighted_read_of_changed_norms_names_the_layer(pipe, no_native, read):
    with trace(pipe, value_norms=True) as tc:
        _fake_slab(tc, norms=True)
        tc.all_heat_maps.slabs[0].norms_changed.fill_(True)
        with pytest.raises(ValueError, match='layer 0: the cross-attention context changed'):
            getattr(tc, read)(value_weighted=True)


def test_a_slab_without_norms_in_a_value_norm_trace(pipe, no_native):
    """Slabs made by RawHeatMapCollection.update hold no norms: a weighted read of them raises."""
    with trace(pipe, value_norms=True) as tc:
        _fake_slab(tc, norms=False)
        with pytest.raises(RuntimeError, match=r'trace\(pipe, value_norms=True\)'):
            tc.compute_global_heat_map(value_weighted=True)


def test_value_norms_keys_follow_the_per_head_order(pipe, no_native):
    with trace(pipe, value_norms=True) as tc:
        _fake_slab(tc, norms=True)
        tc.all_heat_maps.slabs[0].norms.copy_(torch.arange(2 * 77, dtype=torch.float32).view(1, 2, 77))
        keys, norms = tc.compute_value_norms()
        assert keys == [(1, 0, 0), (1, 0, 1)]
        n = len(pipe.tokenizer.tokenize('a dog')) + 2
        assert norms.shape == (2, n)
        assert norms[1, 0] == 77 and norms[0, n - 1] == n - 1


def test_finalize_parts_weights_must_match_the_groups():
    g = _native.DaamKeyGroup(acc=16, heads=1, h=4, w=4, tokens=77, head_sel=-1, n_blocks=0)
    part = _native.DaamMapPart(group_begin=0, group_count=1, n_rows=3, out=16)
    with pytest.raises(ValueError, match='1 key groups'):
        _native.finalize_parts([g], [part], 4, False, 0, [16, 32])
