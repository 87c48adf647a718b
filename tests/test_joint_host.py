"""Joint-attention (SD3) tracing without a GPU: the locator, the dispatch to joint mode, every refused option, the T5
word lookup and the argument checks of daam_accumulate_joint, which run before any device call."""
import pytest
import torch

from daam_b200 import _native, trace
from daam_b200.build import build
from daam_b200.locate import JointAttentionLocator
from daam_b200.testing.synthetic import (TINY_SD3_SPEC, SentencePieceTokenizer, SyntheticSD3Transformer,
                                         make_sd3_pipeline)
from daam_b200.trace import JOINT_REFUSED, JointAttentionHooker
from daam_b200.utils import T5Pieces, compute_token_merge_indices, t5_rows


@pytest.fixture(scope='module')
def lib():
    build()
    return _native.load()


@pytest.fixture(scope='module')
def pipe(lib):
    return make_sd3_pipeline(TINY_SD3_SPEC)


def test_locator_walks_the_joint_blocks_in_order():
    model = SyntheticSD3Transformer(TINY_SD3_SPEC)
    loc = JointAttentionLocator()
    found = loc.locate(model)
    assert found == [b.attn for b in model.transformer_blocks]
    assert loc.layer_names == [f'joint-attn-{i}' for i in range(TINY_SD3_SPEC.blocks)]


def test_an_sd3_pipeline_is_traced_in_joint_mode(pipe):
    tc = trace(pipe)
    assert tc.joint and tc.all_heat_maps.joint
    assert all(isinstance(h, JointAttentionHooker) for h in tc._attn_hookers)
    assert [h.layer_idx for h in tc._attn_hookers] == list(range(TINY_SD3_SPEC.blocks))
    assert tc.layer_names == [f'joint-attn-{i}' for i in range(TINY_SD3_SPEC.blocks)]
    originals = [b.attn.processor for b in pipe.transformer.transformer_blocks]
    with tc:
        assert all(b.attn.processor is h for b, h in zip(pipe.transformer.transformer_blocks, tc._attn_hookers))
    assert [b.attn.processor for b in pipe.transformer.transformer_blocks] == originals


@pytest.mark.parametrize('name', JOINT_REFUSED)
def test_joint_trace_refuses_what_it_does_not_implement(pipe, name):
    value = [(0, 1)] if name == 'step_ranges' else True
    with pytest.raises(ValueError, match=f'{name} is not supported when tracing the joint attention of an SD3'):
        trace(pipe, **{name: value})


def test_joint_trace_refuses_the_overlap_launch(pipe):
    with pytest.raises(ValueError, match="launch='overlap' is not supported when tracing the joint attention"):
        trace(pipe, launch='overlap')
    trace(pipe, launch='layer')
    trace(pipe, launch='step')


def test_refused_list_is_the_documented_one():
    assert set(JOINT_REFUSED) == {'time_resolved', 'step_ranges', 'negative', 'long_prompts', 'value_norms',
                                  'save_heads', 'load_heads', 'low_memory', 'locate_middle_block'}


def test_joint_hook_refuses_an_attention_mask(pipe):
    tc = trace(pipe)
    hooker = tc._attn_hookers[0]
    with pytest.raises(ValueError, match='attention mask'):
        hooker(pipe.transformer.transformer_blocks[0].attn, torch.zeros(2, 4, 64), torch.zeros(2, 3, 64),
               attention_mask=torch.zeros(1))


def test_a_t5_read_of_a_unet_trace_raises(lib):
    from daam_b200.testing.synthetic import TINY_SPEC, make_pipeline
    tc = trace(make_pipeline(TINY_SPEC))
    with pytest.raises(ValueError, match="encoder='t5'"):
        tc.compute_global_heat_map(encoder='t5')
    with pytest.raises(ValueError, match="encoder must be 'clip' or 't5'"):
        tc.compute_global_heat_map(encoder='clip-g')


def test_t5_merge_indices_keep_case_and_join_pieces():
    tok = T5Pieces(SentencePieceTokenizer(), 100)
    prompt = 'a cute giraffe next to a Giraffe'
    # pieces: ▁a ▁cute ▁gira ffe ▁next ▁to ▁a ▁Gira ffe -> rows are piece index + 1
    assert compute_token_merge_indices(tok, prompt, 'giraffe')[0] == [3, 4]
    assert compute_token_merge_indices(tok, prompt, 'Giraffe')[0] == [8, 9]
    assert compute_token_merge_indices(tok, prompt, 'a')[0] == [1, 7]
    assert compute_token_merge_indices(tok, prompt, 'cute')[0] == [2]
    with pytest.raises(ValueError, match='not found'):
        compute_token_merge_indices(tok, prompt, 'CUTE')


def test_t5_merge_indices_stop_at_the_rows_the_map_has():
    tok = T5Pieces(SentencePieceTokenizer(), 3)      # ▁a ▁cute ▁gira | ffe cut off
    with pytest.raises(ValueError, match='not found'):
        compute_token_merge_indices(tok, 'a cute giraffe', 'giraffe')
    assert compute_token_merge_indices(tok, 'a cute giraffe', 'cute')[0] == [2]


def test_t5_row_count_leaves_room_for_the_eos_row():
    assert t5_rows(10, 333) == 10
    assert t5_rows(300, 333) == 255         # 77 CLIP rows + 255 pieces + EOS = 333
    assert t5_rows(600, 589) == 511
    assert t5_rows(5, 77) == 0


def _layer(**kw):
    base = dict(q=16, k=16, acc=16, q_stride_prompt=0, q_stride_pixel=64, q_stride_head=64, k_stride_prompt=0,
                k_stride_token=64, k_stride_head=64, n_prompts=1, heads=1, hw=64, tokens=333, head_dim=64,
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
    (dict(tokens=0), _native.E_UNSUPPORTED, 'tokens = 0'),
    (dict(tokens=1025), _native.E_UNSUPPORTED, 'tokens = 1025'),
    (dict(head_dim=12), _native.E_UNSUPPORTED, 'head_dim = 12'),
    (dict(head_dim=264), _native.E_UNSUPPORTED, 'head_dim = 264'),
    (dict(hw=0), _native.E_INVALID, 'non-positive'),
    (dict(dtype=7), _native.E_INVALID, 'unknown dtype'),
    (dict(scale=0.0), _native.E_INVALID, 'scale'),
])
def test_accumulate_joint_argument_validation(lib, kw, code, text):
    with pytest.raises(_native.NativeError, match=text) as e:
        _native.accumulate_joint([_layer(), _layer(**kw)], 0)
    assert e.value.code == code
    assert 'layer 1' in str(e.value)


def test_accumulate_joint_takes_no_flags(lib):
    array = (_native.DaamJointLayer * 1)(_layer())
    assert lib.daam_accumulate_joint(array, 1, 1, None) == _native.E_INVALID
    assert lib.daam_accumulate_joint(None, 1, 0, None) == _native.E_INVALID
    assert lib.daam_accumulate_joint(None, 0, 0, None) == 0


@pytest.mark.skipif(torch.cuda.is_available(), reason='checks the no-device behaviour')
def test_accumulate_joint_has_no_cpu_fallback(lib):
    with pytest.raises(_native.NativeError) as e:
        _native.accumulate_joint([_layer(tokens=1), _layer(tokens=1024, head_dim=256)], 0)
    assert e.value.code == _native.E_CUDA
