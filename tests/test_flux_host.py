"""FLUX.1 tracing without a GPU: the locator's order and names, FLUX vs SD3 detection and the hooks, every refusal,
the grid from check_inputs, the T5 row cap, the word lookup through tokenizer_2 / prompt_2 and the encoder default."""
import pytest
import torch

from daam_b200 import _native, trace
from daam_b200.build import build
from daam_b200.geometry import FluxGeometry
from daam_b200.locate import JointAttentionLocator
from daam_b200.testing.synthetic import (FLUX_DEV_SPEC, FLUX_SCHNELL_SPEC, TINY_FLUX_SPEC, TINY_SD3_SPEC,
                                         FluxAttnProcessor, SentencePieceTokenizer, SyntheticFluxTransformer,
                                         make_flux_pipeline, make_sd3_pipeline)
from daam_b200.trace import JOINT_REFUSED, FluxAttentionHooker, JointAttentionHooker
from daam_b200.utils import T5Pieces, compute_token_merge_indices, t5_rows


@pytest.fixture(scope='module')
def lib():
    build()
    return _native.load()


@pytest.fixture(scope='module')
def pipe(lib):
    return make_flux_pipeline(TINY_FLUX_SPEC)


def test_locator_walks_double_then_single_blocks():
    model = SyntheticFluxTransformer(TINY_FLUX_SPEC)
    loc = JointAttentionLocator()
    found = loc.locate(model)
    assert found == [b.attn for b in model.transformer_blocks] + [b.attn for b in model.single_transformer_blocks]
    assert loc.layer_names == ['joint-attn-0', 'joint-attn-1', 'single-attn-0', 'single-attn-1', 'single-attn-2']


def test_flux_dev_and_schnell_have_57_layers_within_one_launch():
    for spec in (FLUX_DEV_SPEC, FLUX_SCHNELL_SPEC):
        assert spec.double + spec.single == 57 <= 64
        assert spec.heads * spec.dim_head == 3072 and sum(spec.axes_dim) == spec.dim_head
    assert (FLUX_DEV_SPEC.t5_rows, FLUX_SCHNELL_SPEC.t5_rows) == (512, 256)


def test_a_flux_pipeline_is_traced_in_flux_mode_and_hooks_are_restored(pipe):
    tc = trace(pipe)
    assert tc.joint and tc.flux and tc.all_heat_maps.joint
    assert all(isinstance(h, FluxAttentionHooker) for h in tc._attn_hookers)
    assert [h.layer_idx for h in tc._attn_hookers] == list(range(5))
    attns = [b.attn for b in pipe.transformer.transformer_blocks] + \
        [b.attn for b in pipe.transformer.single_transformer_blocks]
    originals = [a.processor for a in attns]
    with tc:
        assert all(a.processor is h for a, h in zip(attns, tc._attn_hookers))
        assert tc._pre_hook is not None and tc._forward_hook is not None
    assert [a.processor for a in attns] == originals
    assert all(isinstance(p, FluxAttnProcessor) for p in originals)
    assert tc._pre_hook is None and tc._forward_hook is None


def test_an_sd3_pipeline_stays_in_sd3_mode(lib):
    sd3 = make_sd3_pipeline(TINY_SD3_SPEC)
    tc = trace(sd3)
    assert tc.joint and not tc.flux
    assert all(type(h) is JointAttentionHooker for h in tc._attn_hookers)
    assert tc.layer_names == [f'joint-attn-{i}' for i in range(TINY_SD3_SPEC.blocks)]


@pytest.mark.parametrize('name', JOINT_REFUSED)
def test_flux_trace_refuses_what_it_does_not_implement(pipe, name):
    value = [(0, 1)] if name == 'step_ranges' else True
    with pytest.raises(ValueError, match=f'{name} is not supported when tracing the joint attention of a FLUX'):
        trace(pipe, **{name: value})


def test_flux_trace_refuses_the_overlap_launch(pipe):
    with pytest.raises(ValueError, match="launch='overlap' is not supported when tracing the joint attention of a "
                                         "FLUX"):
        trace(pipe, launch='overlap')
    trace(pipe, launch='layer')
    trace(pipe, launch='step')


@pytest.mark.parametrize('kw', [dict(negative_prompt='blurry'), dict(negative_prompt_2='blurry'),
                                dict(negative_prompt_embeds=torch.zeros(1, 24, 64))])
def test_flux_trace_refuses_negative_prompts_at_check_inputs(pipe, kw):
    with trace(pipe):
        with pytest.raises(ValueError, match=f'{next(iter(kw))} is not supported .* FLUX'):
            pipe.check_inputs('a cat', None, 256, 256, **kw)


def test_flux_trace_refuses_a_true_cfg_generation(pipe):
    with trace(pipe):
        with pytest.raises(ValueError, match='negative_prompt is not supported .* FLUX'):
            pipe('a cat', negative_prompt='a dog', true_cfg_scale=4.0, num_inference_steps=1)


@pytest.mark.parametrize('size, grid', [((1024, 1024), (64, 64)), ((1216, 832), (76, 52)), ((832, 1216), (52, 76)),
                                        ((256, 256), (16, 16)), ((1000, 1000), (62, 62))])
def test_grid_comes_from_check_inputs(pipe, size, grid):
    tc = trace(pipe)
    with tc:
        pipe.check_inputs('a cat', None, *size)
    assert tc.geometry.grid == grid and tc.geometry.image_size == size
    assert tc.geometry.level(grid[0] * grid[1], 3) == grid + (1,)


def test_grid_defaults_to_the_pipeline_size(pipe, monkeypatch):
    class Stop(Exception):
        pass

    def stop(*args):
        raise Stop                                  # the generation ends right after check_inputs
    tc = trace(pipe)
    monkeypatch.setattr(pipe, '_embeds', stop)
    with tc:
        with pytest.raises(Stop):
            pipe('a cat')
    assert tc.geometry.grid == (TINY_FLUX_SPEC.sample_size // 2,) * 2 and tc.geometry.image_size == (256, 256)


def test_a_layer_off_the_grid_names_the_layer():
    geom = FluxGeometry(8, (1216, 832))
    with pytest.raises(RuntimeError, match='layer 40: 4096 image tokens'):
        geom.level(4096, 40)
    with pytest.raises(RuntimeError, match='layer 0'):
        FluxGeometry(8).level(256, 0)


def test_t5_rows_of_a_t5_only_context_are_capped_below_the_context():
    assert t5_rows(10, 512, clip_tokens=0) == 10
    assert t5_rows(511, 512, clip_tokens=0) == 511
    assert t5_rows(600, 512, clip_tokens=0) == 511    # 511 pieces + EOS = 512 context rows
    assert t5_rows(300, 256, clip_tokens=0) == 255
    assert t5_rows(0, 24, clip_tokens=0) == 0


def test_t5_text_is_prompt_2_else_the_prompt(pipe):
    tc = trace(pipe, batch_prompts=True)
    with tc:
        pipe.check_inputs('a cat', 'a Cat on a Mat', 256, 256)
        assert tc.last_prompts_2 == ['a Cat on a Mat']
        pipe.check_inputs(['a cat', 'a dog'], None, 256, 256)
        assert tc.last_prompts_2 == ['a cat', 'a dog']
        pipe.check_inputs(['a cat', 'a dog'], ['Cat', 'Dog'], 256, 256)
        assert tc.last_prompts_2 == ['Cat', 'Dog']
        pipe.check_inputs(None, None, 256, 256, prompt_embeds=torch.zeros(2, 24, 64))
        assert tc.last_prompts_2 == [None, None]


def test_word_lookup_goes_through_tokenizer_2(pipe):
    tc = trace(pipe)
    tok = tc._map_tokenizer('t5', list(range(2 + 6)))
    assert isinstance(tok, T5Pieces) and tok.tokenizer is pipe.tokenizer_2
    # pieces: ▁a ▁Gira ffe ▁on ▁a ▁hill -> rows are piece index + 1, case kept, pieces joined
    assert compute_token_merge_indices(tok, 'a Giraffe on a hill', 'Giraffe')[0] == [2, 3]
    with pytest.raises(ValueError, match='not found'):
        compute_token_merge_indices(tok, 'a Giraffe on a hill', 'giraffe')


def test_encoder_defaults_to_the_traces_own(pipe, lib):
    from daam_b200.testing.synthetic import TINY_SPEC, make_pipeline
    tc = trace(pipe)
    assert tc._encoder(None) == 't5' and tc._encoder('t5') == 't5'
    with pytest.raises(ValueError, match="encoder='clip'.*FLUX"):
        tc._encoder('clip')
    with pytest.raises(ValueError, match="encoder='clip'.*FLUX"):
        tc.compute_global_heat_map(encoder='clip')
    for read in (tc.compute_per_head_heat_maps, tc.compute_head_heat_maps, tc.compute_layer_heat_maps):
        with pytest.raises(ValueError, match="encoder='clip'.*FLUX"):
            read(encoder='clip')
    assert trace(make_sd3_pipeline(TINY_SD3_SPEC))._encoder(None) == 'clip'
    assert trace(make_pipeline(TINY_SPEC))._encoder(None) == 'clip'


def test_flux_hook_refuses_an_attention_mask(pipe):
    tc = trace(pipe)
    with pytest.raises(ValueError, match='attention mask'):
        tc._attn_hookers[0](pipe.transformer.transformer_blocks[0].attn, torch.zeros(1, 4, 64), torch.zeros(1, 3, 64),
                            attention_mask=torch.zeros(1))


def test_a_single_block_outside_a_forward_raises(pipe):
    tc = trace(pipe)
    attn = pipe.transformer.single_transformer_blocks[0].attn
    with pytest.raises(RuntimeError, match='single-stream FLUX block'):
        tc._attn_hookers[2](attn, torch.zeros(1, 8, 64))


def test_sentencepiece_rows_are_the_documented_ones():
    tok = SentencePieceTokenizer()
    assert tok.tokenize('a Giraffe') == ['▁a', '▁Gira', 'ffe']


def test_rope_matches_complex_multiplication():
    """The hook's RoPE and the fixture's position embedding against an independent restatement: each interleaved
    pair of the head dim is one complex number, turned by position x theta^(-2j / axis dim) on its axis."""
    import sys
    from daam_b200.testing.synthetic import FluxPosEmbed, flux_image_ids
    from tests import flux64
    apply = sys.modules['daam_b200.trace']._apply_rotary_emb
    ids = torch.cat([torch.zeros(5, 3), flux_image_ids(3, 4)])
    ids[:5, 0] = torch.arange(5)                  # non-zero ids on every axis
    x = torch.randn(2, 3, ids.shape[0], 128, generator=torch.Generator().manual_seed(0))
    got = apply(x, FluxPosEmbed(10000, (16, 56, 56))(ids))
    assert torch.allclose(got.double(), flux64.rope64(x, ids, (16, 56, 56)), rtol=0, atol=2e-5)


def test_a_flux_read_puts_a_zero_row_ahead_of_the_finalized_rows():
    """A FLUX T5 read finalizes context rows [0, n + 1) and its rows [-1, 0, .., n] put a zero row ahead of them,
    so a context filled with pieces (n = T - 1) needs T finalized rows, not T + 1."""
    from daam_b200.trace import _compact, _finalized_rows
    rows = [-1] + list(range(24))
    assert _finalized_rows(rows) == 24
    maps = torch.rand(3, 24, 2, 5)
    out = _compact(maps, rows, False)
    assert out.shape == (3, 25, 2, 5) and out[:, 0].eq(0).all() and torch.equal(out[:, 1:], maps)


def test_flux_hook_refuses_arguments_it_does_not_compute(pipe):
    tc = trace(pipe)
    attn = pipe.transformer.transformer_blocks[0].attn
    with pytest.raises(ValueError, match='cannot take ip_hidden_states'):
        tc._attn_hookers[0](attn, torch.zeros(1, 4, 64), torch.zeros(1, 3, 64), ip_hidden_states=[torch.zeros(1)])
    with pytest.raises(ValueError, match='cannot take argument 5'):
        tc._attn_hookers[0](attn, torch.zeros(1, 4, 64), torch.zeros(1, 3, 64), None, None, torch.zeros(1))
