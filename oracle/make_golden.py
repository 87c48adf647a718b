"""TEST INFRASTRUCTURE -- writes tests/golden/*.npz from the *verbatim* reference (run in the build container only).

    DAAM_REFERENCE_ROOT=<castorini/daam checkout> python -m oracle.make_golden [vs_reference]

The reference (a Python package) is not part of this repository, so its outputs are: each fixture stores seeded
inputs and what the reference's ``daam`` package itself computed from them on CPU fp32 (one thread).
``tests/test_oracle_golden.py`` and ``tests/test_oracle_vs_reference.py`` pin the oracle to these everywhere; the
``-m gpu`` tests compare the CUDA path with the same files.

Fixtures
  layer_*.npz        q [2, hw, H*d], k [2, 77, H*d] (fp16-representable values stored as fp16) and the maps
                     ``_unravel_attn(get_attention_scores(head_to_batch_dim(q), head_to_batch_dim(k)))`` -> [H,77,h,w]
                     exactly as daam/trace.py:272-276 + 219-244 produce them (rows a3+a4 of SURVEY.md section 8a).
  finalize.npz       hand-filled RawHeatMapCollection (peaky maps so that the clamp fires) and the outputs of
                     ``compute_global_heat_map`` for several filters / normalize (row a7), word maps (a8), expand_as (a10).
  pipeline_tiny.npz  a 2-step generation of the TINY synthetic pipeline under the reference's ``trace``: global heat
                     map, normalised map, filtered maps, per-key sums (rows a1-a9 end to end).
  pipeline_tiny96.npz the same for the 96x96-latent geometry of the 768-pixel models (latent_hw 9216, trace.py:32-33):
                     (96, 96) global maps from keys at 96^2 / 48^2 / 24^2.
  pipeline_tiny600.npz the generation of pipeline_tiny.npz at 600x600 pixels (``python -m oracle.make_golden
                     pipeline_offgrid``): keys at 75^2 / 38^2 / 19^2 (factors 0 / 1 / 3), bicubic down-sampling of the
                     75^2 keys onto the 64 x 64 grid.
  perkey.npz         the reference's --all-heads sweep (daam/run/generate.py:239-255) over finalize.npz's keys:
                     ``compute_global_heat_map(layer_idx=l, head_idx=h)`` for every key, plain and normalised.
  vs_reference.npz   the rest of what tests/test_oracle_vs_reference.py compares with: exact fingerprints of the
                     reference's per-key maps, save_heads files and --all-heads sweep, its error messages and merge
                     indices, the _unravel_attn permutation, and the files of a GenerationExperiment dump it wrote.
"""
from __future__ import annotations

import os
import sys
import warnings
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from daam_b200.testing.synthetic import TINY96_SPEC, TINY_SPEC, SyntheticAttention, WhitespaceTokenizer, make_pipeline  # noqa: E402
from oracle.ref_loader import load_reference  # noqa: E402

OUT = os.path.join(ROOT, 'tests', 'golden')
PROMPT = 'a dog chasing a red ball on the beach'

LAYER_CASES = [
    # name, hw, heads, head_dim, logit gain (bigger = peakier softmax)
    ('layer_hw256_h2_d64', 256, 2, 64, 1.0),
    ('layer_hw1024_h1_d64_peaky', 1024, 1, 64, 4.0),
    ('layer_hw64_h2_d40', 64, 2, 40, 1.0),
    ('layer_hw576_h1_d64', 576, 1, 64, 2.0),     # 24x24: a partial 128-pixel tile (96x96-latent models)
]


def ref_layer_maps(daam, q, k, heads, dim_head):
    attn = SyntheticAttention(heads * dim_head, heads * dim_head, heads, dim_head)
    from daam.trace import UNetCrossAttentionHooker
    hk = UNetCrossAttentionHooker.__new__(UNetCrossAttentionHooker)   # _unravel_attn touches no instance state
    probs = attn.get_attention_scores(attn.head_to_batch_dim(q), attn.head_to_batch_dim(k), None)
    return hk._unravel_attn(probs)


def make_layers(daam):
    for i, (name, hw, heads, d, gain) in enumerate(LAYER_CASES):
        g = torch.Generator().manual_seed(100 + i)
        q = (torch.randn(2, hw, heads * d, generator=g) * gain).half()
        k = torch.randn(2, 77, heads * d, generator=g).half()
        maps = ref_layer_maps(daam, q.float(), k.float(), heads, d)
        np.savez_compressed(os.path.join(OUT, name + '.npz'), q=q.numpy(), k=k.numpy(), maps=maps.numpy(),
                            heads=heads, head_dim=d, scale=d ** -0.5)
        print(name, tuple(maps.shape), float(maps.sum()))


def make_finalize(daam):
    g = torch.Generator().manual_seed(7)
    tokens = 12
    coll = daam.RawHeatMapCollection()
    spec = [(1, 0, 0, 64), (2, 1, 0, 32), (2, 1, 1, 32), (4, 2, 0, 16), (4, 2, 1, 16), (4, 3, 0, 16)]
    keys = {}
    for factor, layer, head, side in spec:
        # two "steps" of peaky non-negative maps: exp of a wide gaussian makes bicubic undershoot below zero
        for _ in range(2):
            m = torch.exp(3.0 * torch.randn(tokens, side, side, generator=g))
            m = m / m.sum(0, keepdim=True)
            coll.update(factor, layer, head, m)
        keys[f'key_{factor}_{layer}_{head}'] = coll.ids_to_heatmaps[(factor, layer, head)].numpy()
    tok = WhitespaceTokenizer()
    prompt = 'one two three four five six seven eight nine'   # 9 words -> 11 rows <= 12 tokens
    fake = SimpleNamespace(all_heat_maps=coll, last_prompt=prompt, latent_hw=4096,
                           pipe=SimpleNamespace(tokenizer=tok))
    cg = daam.trace.compute_global_heat_map
    out = {
        'global': cg(fake).heat_maps,
        'global_norm': cg(fake, normalize=True).heat_maps,
        'factors_2_4': cg(fake, factors=[2, 4]).heat_maps,
        'layer_1': cg(fake, layer_idx=1).heat_maps,
        'head_1': cg(fake, head_idx=1).heat_maps,
        'layer_2_head_0': cg(fake, layer_idx=2, head_idx=0).heat_maps,
    }
    ghm = cg(fake)
    word = ghm.compute_word_heat_map('three')
    out['word_three'] = word.heatmap
    multi = daam.GlobalHeatMap(tok, 'red ball and red car', ghm.heat_maps)
    out['word_red_multi'] = multi.compute_word_heat_map('red').heatmap      # two occurrences -> rows 1 and 4
    img = SimpleNamespace(size=(96, 80))
    out['expand'] = word.expand_as(img)
    out['expand_abs'] = word.expand_as(img, absolute=True)
    out['expand_thr'] = word.expand_as(img, threshold=0.4)
    np.savez_compressed(os.path.join(OUT, 'finalize.npz'), prompt=prompt, tokens=tokens,
                        **keys, **{k: v.numpy() for k, v in out.items()})
    print('finalize', {k: tuple(v.shape) for k, v in out.items()})


def make_pipeline_fixture(daam):
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float32, seed=3)
    with daam.trace(pipe) as tc:
        pipe(PROMPT, num_inference_steps=2, generator=torch.Generator().manual_seed(11))
        keys = [k for k, _ in tc.all_heat_maps]
        sums = np.array([float(v.double().sum()) for _, v in tc.all_heat_maps])
        absmax = np.array([float(v.abs().max()) for _, v in tc.all_heat_maps])
        out = {
            'global': tc.compute_global_heat_map().heat_maps.numpy(),
            'global_norm': tc.compute_global_heat_map(normalize=True).heat_maps.numpy(),
            'factors_2': tc.compute_global_heat_map(factors=[2]).heat_maps.numpy(),
            'layer9_head0': tc.compute_global_heat_map(layer_idx=9, head_idx=0).heat_maps.numpy(),
            'word_ball': tc.compute_global_heat_map().compute_word_heat_map('ball').heatmap.numpy(),
        }
        names = list(tc.layer_names)
    np.savez_compressed(os.path.join(OUT, 'pipeline_tiny.npz'), prompt=PROMPT, steps=2, unet_seed=3, gen_seed=11,
                        keys=np.array(keys), key_sums=sums, key_absmax=absmax, layer_names=np.array(names), **out)
    print('pipeline', len(keys), {k: tuple(v.shape) for k, v in out.items()})


def make_pipeline96_fixture(daam):
    pipe = make_pipeline(TINY96_SPEC, dtype=torch.float32, seed=5)
    with daam.trace(pipe) as tc:
        assert tc.latent_hw == 9216
        pipe(PROMPT, num_inference_steps=2, generator=torch.Generator().manual_seed(13))
        keys = [k for k, _ in tc.all_heat_maps]
        sums = np.array([float(v.double().sum()) for _, v in tc.all_heat_maps])
        out = {
            'global': tc.compute_global_heat_map().heat_maps.numpy(),
            'global_norm': tc.compute_global_heat_map(normalize=True).heat_maps.numpy(),
            'factors_4': tc.compute_global_heat_map(factors=[4]).heat_maps.numpy(),
            'word_ball': tc.compute_global_heat_map().compute_word_heat_map('ball').heatmap.numpy(),
        }
    np.savez_compressed(os.path.join(OUT, 'pipeline_tiny96.npz'), prompt=PROMPT, steps=2, unet_seed=5, gen_seed=13,
                        keys=np.array(keys), key_sums=sums, **out)
    print('pipeline96', len(keys), {k: tuple(v.shape) for k, v in out.items()})


def make_pipeline_offgrid_fixture(daam):
    """The generation of pipeline_tiny.npz at 600x600 pixels: a 75x75 latent off the 64-pixel grid, whose traced layers
    have 75^2 / 38^2 / 19^2 query positions (factors 0 / 1 / 3 under the reference's rule) and odd pixel counts."""
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float32, seed=3)
    with daam.trace(pipe) as tc:
        pipe(PROMPT, num_inference_steps=2, generator=torch.Generator().manual_seed(11), height=600, width=600)
        keys = [k for k, _ in tc.all_heat_maps]
        sums = np.array([float(v.double().sum()) for _, v in tc.all_heat_maps])
        absmax = np.array([float(v.abs().max()) for _, v in tc.all_heat_maps])
        out = {
            'global': tc.compute_global_heat_map().heat_maps.numpy(),
            'global_norm': tc.compute_global_heat_map(normalize=True).heat_maps.numpy(),
            'factors_0': tc.compute_global_heat_map(factors=[0]).heat_maps.numpy(),
            'factors_3': tc.compute_global_heat_map(factors=[3]).heat_maps.numpy(),
            'layer9_head0': tc.compute_global_heat_map(layer_idx=9, head_idx=0).heat_maps.numpy(),
            'word_ball': tc.compute_global_heat_map().compute_word_heat_map('ball').heatmap.numpy(),
        }
        names = list(tc.layer_names)
    np.savez_compressed(os.path.join(OUT, 'pipeline_tiny600.npz'), prompt=PROMPT, steps=2, unet_seed=3, gen_seed=11,
                        height=600, width=600, keys=np.array(keys), key_sums=sums, key_absmax=absmax,
                        layer_names=np.array(names), **out)
    print('pipeline600', len(keys), {k: tuple(v.shape) for k, v in out.items()})


def make_perkey_fixture(daam):
    """Every (layer, head) map of the all-heads sweep, from the keys stored in finalize.npz."""
    fx = np.load(os.path.join(OUT, 'finalize.npz'), allow_pickle=False)
    coll = daam.RawHeatMapCollection()
    order = []
    for name in fx.files:
        if name.startswith('key_'):
            f, l, h = (int(v) for v in name.split('_')[1:])
            coll.update(f, l, h, torch.from_numpy(fx[name]))
            order.append((f, l, h))
    fake = SimpleNamespace(all_heat_maps=coll, last_prompt=str(fx['prompt']), latent_hw=4096,
                           pipe=SimpleNamespace(tokenizer=WhitespaceTokenizer()))
    cg = daam.trace.compute_global_heat_map
    plain = np.stack([cg(fake, layer_idx=l, head_idx=h).heat_maps.numpy() for f, l, h in order])
    norm = np.stack([cg(fake, layer_idx=l, head_idx=h, normalize=True).heat_maps.numpy() for f, l, h in order])
    np.savez_compressed(os.path.join(OUT, 'perkey.npz'), keys=np.array(order), plain=plain, norm=norm)
    print('perkey', plain.shape)


def make_vs_reference_fixture(daam):
    """What tests/test_oracle_vs_reference.py compares the oracle with, beyond pipeline_tiny*.npz: exact fingerprints
    (tests.util.digest) of the reference's per-key maps, save_heads files and per-key sweep, its error messages, token
    merge indices, the _unravel_attn permutation, and the files of a GenerationExperiment dump it wrote."""
    import tempfile
    import PIL.Image
    from tests.util import digest
    out = {}
    torch.manual_seed(0)
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float32, seed=3)
    with daam.trace(pipe) as tc:
        pipe(PROMPT, num_inference_steps=2, generator=torch.Generator().manual_seed(11))
        keys = [(k, v.clone()) for k, v in tc.all_heat_maps]
    out['keys'] = np.array([k for k, _ in keys])
    out['key_digests'] = np.stack([digest(v) for _, v in keys])
    with daam.trace(pipe) as tc:
        pipe(PROMPT, num_inference_steps=2, generator=torch.Generator().manual_seed(11))
        sweep = [(f, l, h) for (f, l, h), _ in keys[::5]]
        out['sweep_keys'] = np.array(sweep)
        out['sweep_digests'] = np.stack([digest(tc.compute_global_heat_map(layer_idx=l, head_idx=h, normalize=True)
                                                .heat_maps) for _, l, h in sweep])
    with daam.trace(pipe) as tc:
        try:
            tc.compute_global_heat_map()
        except RuntimeError as e:
            out['empty_trace_error'] = str(e)
    try:
        daam.compute_token_merge_indices(pipe.tokenizer, PROMPT, 'zebra')
    except ValueError as e:
        out['missing_word_error'] = str(e)
    for word in ['dog', 'red', 'beach']:
        out[f'merge_{word}'] = repr(daam.compute_token_merge_indices(pipe.tokenizer, PROMPT, word))
    out['merge_x_idx3'] = repr(daam.compute_token_merge_indices(pipe.tokenizer, PROMPT, 'x', word_idx=3))
    hooker = daam.trace(pipe).module[0]
    out['unravel_perm'] = hooker._unravel_attn(torch.arange(8 * 64 * 77, dtype=torch.float64)
                                               .reshape(8, 64, 77)).numpy().astype(np.uint16)
    with tempfile.TemporaryDirectory() as tmp:
        pipe = make_pipeline(TINY_SPEC, dtype=torch.float32, seed=5)
        gen = lambda: torch.Generator().manual_seed(2)
        with daam.trace(pipe, save_heads=True, data_dir=tmp) as tc:
            pipe(PROMPT, num_inference_steps=2, generator=gen())
            out['saved_global'] = digest(tc.compute_global_heat_map().heat_maps)
        names = sorted(os.listdir(tmp))
        out['saved_names'] = np.array(names)
        out['saved_digests'] = np.stack([digest(torch.load(os.path.join(tmp, n))) for n in names])
        other = make_pipeline(TINY_SPEC, dtype=torch.float32, seed=6)
        with daam.trace(other, load_heads=True, data_dir=tmp) as tc:
            out['loaded_latents'] = digest(other(PROMPT, num_inference_steps=2, generator=gen()).latents)
            out['loaded_global'] = digest(tc.compute_global_heat_map().heat_maps)
    with tempfile.TemporaryDirectory() as tmp:
        maps = torch.rand(6, 16, 16, generator=torch.Generator().manual_seed(4))
        img = PIL.Image.new('RGB', (16, 16), (10, 20, 30))
        daam.GenerationExperiment(img, maps, 'a red ball', seed=3, id='q1', path=tmp).save(heat_maps=False)
        root = os.path.join(tmp, 'q1')
        files = sorted(os.path.relpath(os.path.join(d, f), root) for d, _, fs in os.walk(root) for f in fs)
        out['experiment_maps'] = maps.numpy()
        out['experiment_files'] = np.array(files)
        for i, f in enumerate(files):
            with open(os.path.join(root, f), 'rb') as fh:
                out[f'experiment_file_{i}'] = np.frombuffer(fh.read(), dtype=np.uint8)
    pipe = make_pipeline(TINY96_SPEC, dtype=torch.float32, seed=5)
    with daam.trace(pipe) as tc:
        pipe(PROMPT, num_inference_steps=2, generator=torch.Generator().manual_seed(13))
        out['keys96'] = np.array([k for k, _ in tc.all_heat_maps])
        out['key96_digests'] = np.stack([digest(v) for _, v in tc.all_heat_maps])
    np.savez_compressed(os.path.join(OUT, 'vs_reference.npz'), **out)
    print('vs_reference', sorted(out))


def main():
    warnings.filterwarnings('ignore', category=FutureWarning)
    os.makedirs(OUT, exist_ok=True)
    os.environ.setdefault('XDG_CACHE_HOME', '/tmp/daam_cache')
    torch.set_num_threads(1)   # fixtures must not depend on the thread count
    daam = load_reference()
    if sys.argv[1:] == ['vs_reference']:
        make_vs_reference_fixture(daam)
        return
    if sys.argv[1:] == ['pipeline_offgrid']:
        make_pipeline_offgrid_fixture(daam)
        return
    make_layers(daam)
    make_finalize(daam)
    make_pipeline_fixture(daam)
    make_pipeline96_fixture(daam)
    make_pipeline_offgrid_fixture(daam)
    make_perkey_fixture(daam)
    make_vs_reference_fixture(daam)


if __name__ == '__main__':
    main()
