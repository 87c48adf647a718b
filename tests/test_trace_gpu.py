"""End-to-end parity through the public API: `with trace(pipe) as tc: pipe(...); tc.compute_global_heat_map()` on the
GPU vs the oracle fed the identical Q/K the hooks saw, and (loosely) vs the reference's own run of the same pipeline."""
import pytest
import torch

from daam_b200 import trace
from daam_b200.testing.synthetic import TINY_SPEC, make_pipeline
from oracle import daam_oracle as O
from tests.util import golden, rel_err

pytestmark = pytest.mark.gpu
DEV = 'cuda'
PROMPT = 'a dog chasing a red ball on the beach'


@pytest.fixture(autouse=True)
def _exact_fp32():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


class Recorder:
    """Wraps DiffusionHeatMapHooker._enqueue to keep CPU copies of every (layer, q, k) the hook handed to the kernel."""

    def __init__(self, tc):
        self.calls = []
        inner = tc._enqueue

        def enqueue(layer_idx, factor, q, k, heads, scale):
            self.calls.append((layer_idx, factor, q.detach().float().cpu(), k.detach().float().cpu(), heads, scale))
            return inner(layer_idx, factor, q, k, heads, scale)

        tc._enqueue = enqueue

    def oracle_store(self, prompt_idx=0):
        store = O.OracleHeatMaps()
        for layer_idx, factor, q, k, heads, scale in self.calls:
            n = q.shape[0] // 2
            pair = [prompt_idx, n + prompt_idx]
            maps = O.port_layer_step(q[pair], k[pair], heads, scale)
            for head, m in enumerate(maps):
                store.update(factor, layer_idx, head, m)
        return store


@pytest.mark.parametrize('dtype,tol', [(torch.float32, 2e-5), (torch.bfloat16, 4e-4), (torch.float16, 4e-4)])
@pytest.mark.parametrize('launch', ['step', 'overlap', 'layer'])
def test_pipeline_parity_with_oracle_on_identical_qk(dtype, tol, launch):
    pipe = make_pipeline(TINY_SPEC, dtype=dtype, device=DEV, seed=3)
    with trace(pipe, launch=launch) as tc:
        rec = Recorder(tc)
        pipe(PROMPT, num_inference_steps=3, generator=torch.Generator().manual_seed(11))
        store = rec.oracle_store()
        got = {k: v.clone() for k, v in tc.all_heat_maps}
        assert set(got) == set(k for k, _ in store) and len(got) == 25
        for key, ref in store:
            assert rel_err(got[key], ref) < tol, key
        n_tok = len(pipe.tokenizer.tokenize(PROMPT))
        for kw in [{}, {'normalize': True}, {'factors': [1, 2]}, {'layer_idx': 9, 'head_idx': 0}, {'head_idx': 1}]:
            ref = O.port_global_heat_map(store, 4096, n_tok, **kw)
            out = tc.compute_global_heat_map(**kw).heat_maps
            assert out.shape == ref.shape == (n_tok + 2, 64, 64)
            assert rel_err(out, ref) < tol, kw
        word = tc.compute_global_heat_map().compute_word_heat_map('ball')
        ref_word = O.port_word_heat_map(O.port_global_heat_map(store, 4096, n_tok), pipe.tokenizer, PROMPT, 'ball')
        assert rel_err(word.heatmap, ref_word) < tol
    assert len(rec.calls) == 15 * 3


def test_pipeline_against_reference_fixture():
    """The reference's own run of this pipeline (CPU fp32) vs ours (GPU fp32): Q/K differ by GPU-vs-CPU matmul rounding
    and by SDPA vs explicit softmax in the layer outputs, hence the loose 1e-3."""
    fx = golden('pipeline_tiny')
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float32, device=DEV, seed=int(fx['unet_seed']))
    with trace(pipe) as tc:
        pipe(str(fx['prompt']), num_inference_steps=int(fx['steps']),
             generator=torch.Generator().manual_seed(int(fx['gen_seed'])))
        assert tc.layer_names == fx['layer_names'].tolist()
        keys = sorted(k for k, _ in tc.all_heat_maps)
        assert keys == sorted(tuple(k) for k in fx['keys'].tolist())
        sums = {k: float(v.double().sum()) for k, v in tc.all_heat_maps}
        for k, s in zip(fx['keys'].tolist(), fx['key_sums']):
            assert abs(sums[tuple(k)] - s) < 1e-4 * s
        assert rel_err(tc.compute_global_heat_map().heat_maps, fx['global']) < 1e-3
        assert rel_err(tc.compute_global_heat_map(normalize=True).heat_maps, fx['global_norm']) < 1e-3
        assert rel_err(tc.compute_global_heat_map(factors=[2]).heat_maps, fx['factors_2']) < 1e-3
        assert rel_err(tc.compute_global_heat_map(layer_idx=9, head_idx=0).heat_maps, fx['layer9_head0']) < 1e-3
        assert rel_err(tc.compute_global_heat_map().compute_word_heat_map('ball').heatmap, fx['word_ball']) < 1e-3


def test_state_is_cleared_between_generations_and_trace_is_reusable():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=1)
    with trace(pipe) as tc:
        pipe('a cat', num_inference_steps=2, generator=torch.Generator().manual_seed(1))
        first = tc.compute_global_heat_map().heat_maps.clone()
        pipe('two small dogs', num_inference_steps=1, generator=torch.Generator().manual_seed(2))
        assert tc.last_prompt == 'two small dogs'
        second = tc.compute_global_heat_map().heat_maps.clone()
        assert second.shape[0] == 5 and first.shape[0] == 4
        pipe('a cat', num_inference_steps=2, generator=torch.Generator().manual_seed(1))
        again = tc.compute_global_heat_map().heat_maps
        assert torch.equal(first, again)              # accumulators were zeroed, not carried over
        sums = [float(v.sum()) for _, v in tc.all_heat_maps]
        assert all(abs(s - 2 * v.shape[-1] * v.shape[-2]) < 1e-2 * s for s, (_, v) in zip(sums, tc.all_heat_maps))
    with pytest.raises(RuntimeError, match='Module is not hooked'):
        tc.unhook()
    out = pipe('a cat', num_inference_steps=1)          # un-hooked pipeline still runs (processors restored)
    assert out.latents.shape[0] == 1


def test_hooked_forward_output_matches_unhooked():
    """The processor must not change what the UNet computes (it replaces the reference's explicit softmax with SDPA)."""
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float32, device=DEV, seed=5)
    base = pipe('a cat on a mat', num_inference_steps=2, generator=torch.Generator().manual_seed(3)).latents
    with trace(pipe):
        hooked = pipe('a cat on a mat', num_inference_steps=2, generator=torch.Generator().manual_seed(3)).latents
    assert rel_err(hooked, base) < 1e-5


def test_batch_prompts_mode_equals_independent_traces():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=2)
    prompts = ['a red ball', 'two dogs on the beach', 'a cat']
    with trace(pipe, batch_prompts=True) as tc:
        rec = Recorder(tc)
        pipe(prompts, num_inference_steps=2, generator=torch.Generator().manual_seed(4))
        assert tc.last_prompts == prompts
        for i, p in enumerate(prompts):
            store = rec.oracle_store(i)
            n_tok = len(pipe.tokenizer.tokenize(p))
            ref = O.port_global_heat_map(store, 4096, n_tok)
            out = tc.compute_global_heat_map(prompt_idx=i).heat_maps
            assert out.shape == ref.shape
            assert rel_err(out, ref) < 4e-4, p
            for (key, view), (rkey, rval) in zip(tc.all_heat_maps.items(i), store):
                pass
    with trace(pipe) as tc:
        with pytest.raises(ValueError, match='Only single prompt generation is supported'):
            pipe(prompts, num_inference_steps=1)


def test_low_memory_and_mid_block_options():
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=2)
    with trace(pipe, low_memory=True) as tc:
        pipe('a cat', num_inference_steps=1)
        assert len(tc.layer_names) == 6 and len(list(tc.all_heat_maps)) == sum(h for h in (2, 2, 1, 1, 2, 2))
    with trace(pipe, locate_middle_block=True) as tc:
        pipe('a cat', num_inference_steps=1)
        assert len(tc.layer_names) == 16
        assert 15 not in tc.all_heat_maps.layers()      # the mid layer (factor 8) is located but never traced
        assert tc.all_heat_maps.factors() == {1, 2, 4}
        assert tc._gen_idx == 16


@pytest.mark.parametrize('launch', ['step', 'overlap', 'layer'])
def test_cuda_graph_replay_traces_like_eager(launch):
    """The tracer's kernels become nodes of a captured UNet step: graph replays must accumulate exactly like eager."""
    prompt = 'a dog chasing a red ball'
    eager_pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=4)
    graph_pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=4, cuda_graph=True)
    with trace(eager_pipe, launch=launch) as tc:
        eager_pipe(prompt, num_inference_steps=5, generator=torch.Generator().manual_seed(9))
        ref = tc.compute_global_heat_map().heat_maps.clone()
        ref_keys = {k: v.clone() for k, v in tc.all_heat_maps}
    with trace(graph_pipe, launch=launch) as tc:
        for _ in range(2):    # second generation replays the cached graph from step 0
            graph_pipe(prompt, num_inference_steps=5, generator=torch.Generator().manual_seed(9))
            got = tc.compute_global_heat_map().heat_maps
            assert rel_err(got, ref) < 2e-3          # eager vs graph: cuBLAS may pick other algorithms under capture
            for k, v in tc.all_heat_maps:
                s = float(v.double().sum())
                assert abs(s - 5 * v.shape[-1] * v.shape[-2]) < 1e-3 * s, k     # exactly 5 steps were accumulated
        assert any(st['graph'] is not None for st in graph_pipe._graphs.values())
    base = graph_pipe(prompt, num_inference_steps=3)     # un-hooked: new processors -> new graph, still runs
    assert base.latents.shape[0] == 1


@pytest.mark.parametrize('dtype,tol', [(torch.float32, 2e-5), (torch.float16, 2e-3)])
def test_save_heads_and_load_heads(tmp_path, dtype, tol):
    """Compatibility path (reference trace.py:246-250, 279-302): probabilities are materialised per layer call as
    `{gen_idx}.pt` ([B*H, hw, 77], pipeline dtype); load_heads recomputes maps and layer outputs from those files."""
    steps = 2
    pipe = make_pipeline(TINY_SPEC, dtype=dtype, device=DEV, seed=5)
    with trace(pipe, save_heads=True, data_dir=str(tmp_path)) as tc:
        assert len(tc.layer_names) == 16
        out_save = pipe(PROMPT, num_inference_steps=steps, generator=torch.Generator().manual_seed(2)).latents
        maps_save = tc.compute_global_heat_map().heat_maps.clone()
        keys_save = {k: v.clone() for k, v in tc.all_heat_maps}
    files = sorted(tmp_path.iterdir(), key=lambda p: int(p.stem))
    assert [int(p.stem) for p in files] == list(range(16 * steps))
    # every saved tensor is a row-stochastic [B*H, hw, 77] matrix in the pipeline dtype
    shapes = set()
    for p in files:
        t = torch.load(p)
        assert t.dtype == dtype and t.shape[-1] == 77
        shapes.add(tuple(t.shape))
        assert torch.allclose(t.float().sum(-1), torch.ones_like(t[..., 0]).float(), atol=5e-3)
    assert (2 * 1, 4096, 77) in shapes and (2 * 2, 64, 77) in shapes          # 64x64 head and the mid block (8x8)
    # the maps are exactly the time-sums of the conditional halves of the saved tensors (oracle: unravel + update)
    store = O.OracleHeatMaps()
    per_step = [torch.load(p).float().cpu() for p in files]
    calls = list(range(9, 15)) + [15] + list(range(0, 9))     # execution order: down blocks, mid block, up blocks
    for i, t in enumerate(per_step):
        layer = calls[i % 16]
        factor = int((4096 // t.shape[1]) ** 0.5)
        if factor != 8:
            for head, m in enumerate(O.port_unravel(t)):
                store.update(factor, layer, head, m)
    for key, ref in store:
        assert rel_err(keys_save[key], ref) < 1e-5, key
    # load_heads on a pipeline with other weights reproduces the maps from the files alone
    other = make_pipeline(TINY_SPEC, dtype=dtype, device=DEV, seed=6)
    with trace(other, load_heads=True, data_dir=str(tmp_path)) as tc:
        other(PROMPT, num_inference_steps=steps, generator=torch.Generator().manual_seed(2))
        maps_load = tc.compute_global_heat_map().heat_maps.clone()
    assert torch.equal(maps_load, maps_save)
    # and on the same pipeline it also reproduces the UNet output of the saving run
    with trace(pipe, load_heads=True, data_dir=str(tmp_path)) as tc:
        out_load = pipe(PROMPT, num_inference_steps=steps, generator=torch.Generator().manual_seed(2)).latents
    assert rel_err(out_load, out_save) < 1e-6
    # the materialised path and the fused path see the same attention: their maps agree
    with trace(pipe) as tc:
        pipe(PROMPT, num_inference_steps=steps, generator=torch.Generator().manual_seed(2))
        fused = tc.compute_global_heat_map().heat_maps
    assert rel_err(maps_save, fused) < tol


def test_per_head_heat_maps_equal_the_all_heads_sweep():
    """One launch == the reference's `for head, layer: compute_global_heat_map(layer_idx, head_idx)` loop."""
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=8)
    with trace(pipe) as tc:
        pipe(PROMPT, num_inference_steps=2, generator=torch.Generator().manual_seed(1))
        for normalize in (False, True):
            keys, maps = tc.compute_per_head_heat_maps(normalize=normalize)
            assert len(keys) == 25 and maps.shape == (25, 11, 64, 64)
            for (factor, layer, head), m in zip(keys, maps):
                single = tc.compute_global_heat_map(layer_idx=layer, head_idx=head, normalize=normalize).heat_maps
                assert rel_err(single, m) < 1e-6, (factor, layer, head)
        keys2, _ = tc.compute_per_head_heat_maps(factors=[2])
        assert {k[0] for k in keys2} == {2}


def test_collection_interface_update_and_to_experiment(tmp_path):
    """RawHeatMapCollection keeps the reference's interface (heatmap.py:148-172) on top of the slabs, and to_experiment
    (trace.py:68-81) packages the last generation."""
    from daam_b200 import GenerationExperiment, RawHeatMapCollection
    coll = RawHeatMapCollection()
    a, b = torch.rand(77, 16, 16, device=DEV), torch.rand(77, 16, 16, device=DEV)
    coll.update(4, 2, 0, a)
    coll.update(4, 2, 1, b)
    coll.update(4, 2, 0, b)
    coll.update(1, 5, 0, torch.ones(77, 64, 64, device=DEV))
    got = dict(coll)
    assert set(got) == {(4, 2, 0), (4, 2, 1), (1, 5, 0)}
    assert torch.allclose(got[(4, 2, 0)], a + b) and torch.allclose(got[(4, 2, 1)], b)
    assert coll.factors() == {1, 4} and coll.layers() == {2, 5} and coll.heads() == {0, 1} and len(coll) == 3
    coll.clear()
    assert len(coll) == 0 and list(coll) == []

    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=8)
    with trace(pipe) as tc:
        pipe(PROMPT, num_inference_steps=1, generator=torch.Generator().manual_seed(1))
        exp = tc.to_experiment(str(tmp_path), seed=1, id='gen0', normalize=True)
        ref = tc.compute_global_heat_map(normalize=True).heat_maps
    assert isinstance(exp, GenerationExperiment) and exp.prompt == PROMPT and torch.equal(exp.global_heat_map, ref)
    exp.tokenizer = None          # the synthetic tokenizer is a local class; real ones pickle
    exp.save()
    back = GenerationExperiment.load(tmp_path / 'gen0', map_location='cpu')
    assert torch.equal(back.global_heat_map, ref.cpu()) and back.seed == 1


@pytest.mark.parametrize('dtype,tol', [(torch.float32, 2e-5), (torch.float16, 4e-4)])
def test_sd1x_style_pipeline(dtype, tol):
    """SD-1.x style UNet (head_dim = channels // heads: 40 / 80 / 80): the tracer picks the K-chunked wgmma path; parity
    with the oracle on the identical Q/K the hooks saw."""
    from daam_b200.testing.synthetic import TINY15_SPEC
    pipe = make_pipeline(TINY15_SPEC, dtype=dtype, device=DEV, seed=3)
    with trace(pipe) as tc:
        rec = Recorder(tc)
        pipe(PROMPT, num_inference_steps=2, generator=torch.Generator().manual_seed(11))
        store = rec.oracle_store()
        got = dict(tc.all_heat_maps)
        assert len(got) == 30                     # 15 layers x 2 heads
        for key, ref in store:
            assert rel_err(got[key], ref) < tol, key
        n_tok = len(pipe.tokenizer.tokenize(PROMPT))
        ref = O.port_global_heat_map(store, 4096, n_tok)
        assert rel_err(tc.compute_global_heat_map().heat_maps, ref) < tol
    assert {c[2].shape[-1] // c[4] for c in rec.calls} == {40, 80}


def test_several_images_per_prompt_enumerate_images_x_heads_like_the_reference():
    """num_images_per_prompt > 1: the CFG batch is [uncond x n, cond x n] for ONE prompt and the reference's keys run over
    images x heads (`map_[map_.size(0) // 2:]` keeps n * H rows, trace.py:240, 293-294). Same here: one prompt, n * H keys
    per layer, each equal to the oracle's map for that (image, head)."""
    from tests.util import assert_elementwise
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=6)
    spec = pipe.unet.spec
    g = torch.Generator().manual_seed(3)
    n = 2
    lat = torch.randn(2 * n, spec.in_channels, 64, 64, generator=g).half().to(DEV)
    emb = torch.randn(2 * n, 77, spec.cross_attention_dim, generator=g).half().to(DEV)
    calls = []
    with torch.no_grad(), trace(pipe) as tc:
        inner = tc._enqueue

        def enqueue(layer_idx, factor, q, k, heads, scale):
            calls.append((layer_idx, factor, q.detach().float().cpu(), k.detach().float().cpu(), heads, scale))
            return inner(layer_idx, factor, q, k, heads, scale)

        tc._enqueue = enqueue
        tc.last_prompts, tc.last_prompt = ['a cat'], 'a cat'
        pipe.unet(lat, torch.full((1,), 500.0, device=DEV), emb)
        got = dict(tc.all_heat_maps)
        for layer_idx, factor, q, k, heads, scale in calls:
            ref = O.port_layer_step(q, k, heads, scale)            # [n * H, 77, h, w]: the reference's kept half
            assert ref.shape[0] == n * heads
            for key_head in range(n * heads):
                assert_elementwise(got[(factor, layer_idx, key_head)], ref[key_head], 1e-4, 1e-5, f'{layer_idx}/{key_head}')
        assert len(got) == n * 25
        out = tc.compute_global_heat_map().heat_maps                 # mean over images x heads x layers, one prompt
        assert out.shape == (4, 64, 64)


@pytest.mark.parametrize('launch', ['step', 'overlap', 'layer'])
def test_projections_with_a_strided_channel_axis_are_copied_and_kept_alive(launch):
    """to_q / to_k outputs whose channel axis is not contiguous (stride(-1) != 1) cannot be described to the kernel in
    place: the tracer works on contiguous copies and must keep THOSE alive until the step's launch has run."""
    from tests.util import assert_elementwise
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float16, device=DEV, seed=1)
    g = torch.Generator().manual_seed(7)
    hw, heads, d = 1024, 2, 64
    with trace(pipe, launch=launch) as tc:
        ref = torch.zeros(heads, 77, hw)
        for step in range(3):
            q = torch.randn(2, heads * d, hw, generator=g).half().to(DEV).transpose(1, 2)      # [2, hw, C], stride(-1) = hw
            k = torch.randn(2, heads * d, 77, generator=g).half().to(DEV).transpose(1, 2)
            assert q.stride(-1) != 1
            tc._enqueue(3, 2, q, k, heads, d ** -0.5)
            ref += O.port_layer_step(q.float().cpu(), k.float().cpu(), heads, d ** -0.5).reshape(heads, 77, hw)
            del q, k
            torch.empty(8 << 20, device=DEV).fill_(1.0)          # churn the allocator: freed copies would be overwritten
            tc.flush()
        tc.synchronize()
        torch.cuda.synchronize()
        got = {key: v for key, v in tc.all_heat_maps}
        for head in range(heads):
            assert_elementwise(got[(2, 3, head)], ref[head].reshape(77, 32, 32), 1e-4, 3e-5, f'head {head}')
