"""Long-prompt heat maps without a GPU: the context row layout, the option's refusals, generations driven by
``prompt_embeds`` (their prompt count, the missing text, time-resolved traces) and the multi-GPU gather at the compact
row count of a three-chunk context."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from daam_b200 import trace
from daam_b200.distributed import gather_heat_maps, pad_heat_map
from daam_b200.testing.synthetic import TINY_SPEC, WhitespaceTokenizer, make_pipeline
from daam_b200.utils import compute_token_merge_indices, context_rows


def _row(j):
    return 77 * (j // 75) + 1 + j % 75


@pytest.mark.parametrize('tokens', [77, 154, 231])
@pytest.mark.parametrize('n', [0, 1, 74, 75, 76, 150, 151, 225, 226, 400])
def test_context_rows(tokens, n):
    cap = 75 * (tokens // 77)
    m = min(n, cap)
    rows = context_rows(n, tokens)
    assert len(rows) == m + 2
    assert rows[0] == 0
    assert rows[1:-1] == [_row(j) for j in range(m)]
    assert rows[-1] == (_row(m - 1) + 1 if m else 1)
    assert rows == sorted(set(rows)) and rows[-1] < tokens
    if tokens == 77 or m <= 75:                        # a prompt that fits one chunk: the reference's truncation
        assert rows == list(range(m + 2))


def test_context_rows_named_cases():
    assert context_rows(0, 154) == [0, 1]
    assert context_rows(75, 154)[-2:] == [75, 76]        # last token of chunk 0, then that chunk's EOS row
    assert context_rows(76, 154)[-3:] == [75, 78, 79]    # token 75 opens chunk 1 (row 77 is its BOS)
    assert context_rows(150, 154)[-2:] == [152, 153]
    assert context_rows(151, 231)[-3:] == [152, 155, 156]
    assert context_rows(225, 231)[-2:] == [229, 230]
    assert context_rows(300, 154) == context_rows(150, 154)
    with pytest.raises(ValueError):
        context_rows(3, 100)


def test_word_lookup_on_a_compact_map():
    """Compact row r + 1 of prompt token r is context row ``context_rows(n, tokens)[r + 1]``: a word past position 75
    reads the second or third chunk."""
    tok = WhitespaceTokenizer()
    words = [f'w{i}' for i in range(180)]
    words[100], words[170] = 'lighthouse', 'dog'
    prompt = ' '.join(words)
    rows, _ = compute_token_merge_indices(tok, prompt, 'lighthouse')
    assert rows == [101]
    ctx = context_rows(len(tok.tokenize(prompt)), 231)
    assert ctx[rows[0]] == 77 + 1 + 25
    rows, _ = compute_token_merge_indices(tok, prompt, 'dog')
    assert ctx[rows[0]] == 154 + 1 + 20


@pytest.fixture
def pipe():
    return make_pipeline(TINY_SPEC, dtype=torch.float32, device='cpu', seed=0)


@pytest.mark.parametrize('option', [dict(time_resolved=True), dict(step_ranges=[(0, 1)]), dict(save_heads=True),
                                    dict(load_heads=True)])
def test_option_refusals(pipe, option):
    with pytest.raises(ValueError, match='long_prompts=True does not support'):
        trace(pipe, long_prompts=True, **option)


def test_prompt_embeds_count_and_missing_text(pipe):
    embeds = torch.zeros(2, 154, 96)
    with trace(pipe, batch_prompts=True) as tc:
        pipe.check_inputs(None, 512, 512, None, None, prompt_embeds=embeds)
        assert tc.last_prompts == [None, None]
        with pytest.raises(ValueError, match='prompt='):
            tc.compute_global_heat_map()
        with pytest.raises(ValueError, match='prompt='):
            tc.compute_per_head_heat_maps(prompt_idx=1)
    with trace(pipe) as tc:
        pipe.check_inputs(None, 512, 512, None, None, embeds[:1])          # bound by position, too
        assert tc.last_prompts == [None]
        with pytest.raises(ValueError, match='Only single prompt'):
            pipe.check_inputs(None, 512, 512, None, None, prompt_embeds=embeds)


def test_time_resolved_refuses_a_generation_without_text(pipe):
    with trace(pipe, time_resolved=True):
        with pytest.raises(ValueError, match='time_resolved=True needs the prompt text'):
            pipe.check_inputs(None, 512, 512, None, None, prompt_embeds=torch.zeros(1, 77, 96))


def test_unsupported_context_length_raises_at_the_layer(pipe):
    with trace(pipe, long_prompts=True):
        with pytest.raises(ValueError, match='100 tokens'):
            pipe(prompt_embeds=torch.randn(1, 100, 96), num_inference_steps=1)


def test_long_context_is_skipped_without_the_option(pipe):
    with trace(pipe) as tc:
        pipe(prompt_embeds=torch.randn(1, 154, 96), num_inference_steps=1)
        with pytest.raises(RuntimeError, match='No heat maps found'):
            tc.compute_global_heat_map(prompt='a cat')


def test_synthetic_pipeline_takes_embeddings(pipe):
    g = torch.Generator().manual_seed(3)
    cond, uncond = torch.randn(1, 231, 96, generator=g), torch.randn(1, 231, 96, generator=g)
    a = pipe(prompt_embeds=cond, negative_prompt_embeds=uncond, num_inference_steps=2,
             generator=torch.Generator().manual_seed(1))
    b = pipe(prompt_embeds=cond, num_inference_steps=2, generator=torch.Generator().manual_seed(1))
    assert a.latents.shape == b.latents.shape and not torch.equal(a.latents, b.latents)
    with pytest.raises(ValueError, match='Cannot forward both'):
        pipe('a cat', prompt_embeds=cond, num_inference_steps=1)


def _fake_map(i, x=8):
    n_rows = 225 + i % 3                               # compact maps of 223, 224 and 225 prompt tokens
    return torch.full((n_rows, x, x), float(i + 1)) + torch.arange(n_rows).view(-1, 1, 1)


def _worker(rank, world, port, n_total, out_dir):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        mine = [_fake_map(i) for i in range(rank, n_total, world)]
        torch.save(gather_heat_maps(mine, n_total, 8, tokens=75 * 3 + 2), os.path.join(out_dir, f'r{rank}.pt'))
    finally:
        dist.destroy_process_group()


def test_gather_three_chunk_maps_world2(tmp_path):
    """``gather_heat_maps(..., tokens=75 c + 2)``: the compact maps of a three-chunk context, 227 rows at most."""
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        port = s.getsockname()[1]
    mp.spawn(_worker, args=(2, port, 5, str(tmp_path)), nprocs=2, join=True)
    expect = torch.stack([pad_heat_map(_fake_map(i), 227) for i in range(5)])
    for r in range(2):
        got = torch.load(os.path.join(tmp_path, f'r{r}.pt'))
        assert got.shape == (5, 227, 8, 8)
        assert torch.equal(got, expect)
