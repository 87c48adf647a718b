"""Host-side rules of trace(pipe, negative=True) that need no GPU: the option and the read switches are keyword-only and
off by default, the negative prompt is bound by name from the pipeline's ``check_inputs`` call whatever its position
(SD and SDXL signatures, positional and keyword), a list of the wrong length is refused, and reads with
``negative=True`` fail loudly on a trace without the mode."""
import inspect

import pytest
import torch

from daam_b200 import trace
from daam_b200.heatmap import RawHeatMapCollection
from daam_b200.testing.synthetic import TINY_SPEC, SyntheticPipeline, make_pipeline


class SDShaped(SyntheticPipeline):
    """diffusers' StableDiffusionPipeline.check_inputs parameter order."""

    def check_inputs(self, prompt, height, width, callback_steps, negative_prompt=None, prompt_embeds=None,
                     negative_prompt_embeds=None, callback_on_step_end_tensor_inputs=None):
        self.seen = (prompt, height, width, callback_steps, negative_prompt)


class SDXLShaped(SyntheticPipeline):
    """diffusers' StableDiffusionXLPipeline.check_inputs parameter order: ``prompt_2`` comes before the size."""

    def check_inputs(self, prompt, prompt_2, height, width, callback_steps, negative_prompt=None,
                     negative_prompt_2=None, prompt_embeds=None, negative_prompt_embeds=None,
                     pooled_prompt_embeds=None, negative_pooled_prompt_embeds=None,
                     callback_on_step_end_tensor_inputs=None):
        self.seen = (prompt, prompt_2, height, width, callback_steps, negative_prompt)


class CatchAll(SyntheticPipeline):
    """A ``check_inputs`` that names nothing but the prompt: a keyword negative prompt lands in ``**kwargs``."""

    def check_inputs(self, prompt, *args, **kwargs):
        self.seen = (prompt, args, kwargs)


def _pipe(cls=SyntheticPipeline):
    base = make_pipeline(TINY_SPEC, dtype=torch.float32, device='cpu', seed=0)
    return cls(base.unet, dtype=torch.float32, device='cpu')


def test_option_is_keyword_only_and_off_by_default():
    p = inspect.signature(trace.__init__).parameters['negative']
    assert p.kind is inspect.Parameter.KEYWORD_ONLY and p.default is False
    for fn in (trace.compute_global_heat_map, trace.compute_per_head_heat_maps, trace.compute_time_heat_maps,
               RawHeatMapCollection.items):
        p = inspect.signature(fn).parameters['negative']
        assert p.kind is inspect.Parameter.KEYWORD_ONLY and p.default is False, fn
    tc = trace(_pipe())
    assert tc.negative is False and tc.all_heat_maps.negative is False


@pytest.mark.parametrize('call,want', [
    (lambda p: p.check_inputs('a cat', 512, 512, None, 'blurry'), ['blurry']),
    (lambda p: p.check_inputs('a cat', 512, 512, None, negative_prompt='blurry'), ['blurry']),
    (lambda p: p.check_inputs('a cat', 512, 512, None), ['']),
    (lambda p: p.check_inputs('a cat', 512, 512, None, None), ['']),
    (lambda p: p.check_inputs('a cat', height=512, width=512, callback_steps=None), ['']),
    (lambda p: p.check_inputs(['a cat', 'a dog'], 512, 512, None, 'blurry'), ['blurry', 'blurry']),
    (lambda p: p.check_inputs(['a cat', 'a dog'], 512, 512, None, ['blurry', 'dark']), ['blurry', 'dark']),
], ids=['positional', 'keyword', 'absent', 'none', 'keywords-only', 'str-for-all', 'one-per-prompt'])
def test_sd_signature_binds_the_negative_prompt(call, want):
    pipe = _pipe(SDShaped)
    with trace(pipe, negative=True, batch_prompts=True) as tc:
        call(pipe)
        assert tc.last_negative_prompts == want
        assert pipe.seen[1:3] == (512, 512)                     # the call reached the pipeline unchanged


@pytest.mark.parametrize('call,want', [
    (lambda p: p.check_inputs('a cat', 'a cat, photo', 1024, 1024, None, 'blurry'), ['blurry']),
    (lambda p: p.check_inputs('a cat', None, 1024, 1024, None, negative_prompt='blurry', negative_prompt_2='x'),
     ['blurry']),
    (lambda p: p.check_inputs('a cat', None, 1024, 1024, None, None, 'only the second encoder'), ['']),
    (lambda p: p.check_inputs('a cat', None, 1024, 1024, None), ['']),
], ids=['positional', 'keyword', 'only-negative-prompt-2', 'absent'])
def test_sdxl_signature_binds_the_negative_prompt(call, want):
    """SDXL's ``prompt_2`` shifts every later parameter by one: the fifth positional argument is callback_steps."""
    pipe = _pipe(SDXLShaped)
    with trace(pipe, negative=True) as tc:
        call(pipe)
        assert tc.last_negative_prompts == want
        assert pipe.seen[0] == 'a cat'


def test_a_keyword_negative_prompt_into_a_catch_all_signature():
    pipe = _pipe(CatchAll)
    with trace(pipe, negative=True) as tc:
        pipe.check_inputs('a cat', 512, 512, negative_prompt='blurry')
        assert tc.last_negative_prompts == ['blurry']
        pipe.check_inputs('a cat', 512, 512, None, 'not bound by any name')
        assert tc.last_negative_prompts == ['']


def test_synthetic_pipeline_names_the_parameter_and_passes_it_in_sd_order():
    pipe = _pipe()
    params = list(inspect.signature(pipe.check_inputs).parameters)
    assert params[:5] == ['prompt', 'height', 'width', 'callback_steps', 'negative_prompt']
    seen = []
    inner = pipe.check_inputs
    pipe.check_inputs = lambda *a, **kw: (seen.append((a, kw)), inner(*a, **kw))[1]
    with pytest.raises(RuntimeError, match='CUDA'):         # the CPU UNet stops at the first traced layer
        with trace(pipe, negative=True):
            pipe('a cat', num_inference_steps=1, negative_prompt='blurry')
    assert seen == [(('a cat', 512, 512, None, 'blurry'), {})]


def test_negative_prompt_changes_no_random_draw():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float32, device='cpu', seed=0)
    a = pipe('a cat', num_inference_steps=2, generator=torch.Generator().manual_seed(3))
    b = pipe('a cat', num_inference_steps=2, generator=torch.Generator().manual_seed(3), negative_prompt='blurry')
    assert torch.equal(a.latents, b.latents)


def test_a_negative_prompt_list_of_the_wrong_length_is_refused():
    pipe = _pipe(SDShaped)
    with trace(pipe, negative=True, batch_prompts=True) as tc:
        pipe.check_inputs(['a cat', 'a dog'], 512, 512, None, ['blurry', 'dark'])
        with pytest.raises(ValueError, match='2 entries for 3 prompts'):
            pipe.check_inputs(['a cat', 'a dog', 'a cow'], 512, 512, None, ['blurry', 'dark'])
        with pytest.raises(ValueError, match='1 entries for 2 prompts'):
            pipe.check_inputs(['a cat', 'a dog'], 512, 512, None, ['blurry'])
        assert tc.last_prompts == ['a cat', 'a dog'] and tc.last_negative_prompts == ['blurry', 'dark']


def test_without_the_mode_nothing_is_bound():
    pipe = _pipe(SDShaped)
    with trace(pipe) as tc:
        pipe.check_inputs('a cat', 512, 512, None, ['one', 'two', 'three'])     # not checked: the mode is off
        assert tc.last_negative_prompts == []


def test_reads_need_the_mode():
    pipe = _pipe()
    tc = trace(pipe)
    for read in (lambda: tc.compute_global_heat_map(negative=True),
                 lambda: tc.compute_per_head_heat_maps(negative=True),
                 lambda: list(tc.all_heat_maps.items(negative=True)),
                 lambda: tc.to_experiment('unused', negative=True)):
        with pytest.raises(RuntimeError, match=r'trace\(pipe, negative=True\)'):
            read()
    tc = trace(pipe, time_resolved=True)
    with pytest.raises(RuntimeError, match=r'trace\(pipe, negative=True\)'):
        tc.compute_time_heat_maps(negative=True)
    tc = trace(pipe, negative=True)
    assert tc.all_heat_maps.negative is True
    with pytest.raises(RuntimeError, match='No heat maps found'):
        tc.compute_global_heat_map(negative=True)
