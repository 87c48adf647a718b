"""Pins oracle/daam_oracle.py against the verbatim reference's own outputs, stored by oracle/make_golden.py.

pipeline_tiny.npz / pipeline_tiny96.npz hold the reference's heat maps of the two generations below in full;
vs_reference.npz holds exact fingerprints (tests.util.digest: float64 sum + a fixed sample of elements) of the
per-key maps, the save_heads files and the per-key sweep, and the reference's strings, indices and experiment dump.
Every comparison is exact."""
import warnings

import numpy as np
import pytest
import torch

from daam_b200.testing.synthetic import TINY_SPEC, make_pipeline
from oracle import daam_oracle as O
from tests.util import digest, golden

warnings.filterwarnings('ignore', category=FutureWarning)

PROMPT = 'a dog chasing a red ball on the beach'


@pytest.fixture(scope='module', autouse=True)
def one_thread():
    """The fixtures were computed on one thread (oracle/make_golden.py): the UNet's fp32 matmuls sum in a
    thread-count-dependent order, and these comparisons are exact."""
    before = torch.get_num_threads()
    torch.set_num_threads(1)
    yield
    torch.set_num_threads(before)


@pytest.fixture(scope='module')
def ref():
    return golden('vs_reference')


@pytest.fixture(scope='module')
def runs():
    """The reference's 2-step generation (stored) and the same generation under the oracle's trace."""
    torch.manual_seed(0)
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float32, seed=3)
    fx = golden('pipeline_tiny')
    ref_out = {'global': fx['global'], 'norm': fx['global_norm'], 'f2': fx['factors_2'], 'l9h0': fx['layer9_head0'],
               'word': fx['word_ball'], 'names': fx['layer_names'].tolist()}
    with O.OracleTrace(pipe) as ot:
        pipe(PROMPT, num_inference_steps=2, generator=torch.Generator().manual_seed(11))
        ora_keys = {k: v.clone() for k, v in ot.heat_maps}
        g = ot.compute_global_heat_map()
        ora_out = {
            'global': g,
            'norm': ot.compute_global_heat_map(normalize=True),
            'f2': ot.compute_global_heat_map(factors=[2]),
            'l9h0': ot.compute_global_heat_map(layer_idx=9, head_idx=0),
            'word': O.port_word_heat_map(g, pipe.tokenizer, PROMPT, 'ball'),
            'names': list(ot.layer_names),
        }
    return pipe, ref_out, ora_keys, ora_out


def test_layer_order_and_names(ref, runs):
    _, ref_out, ora_keys, ora_out = runs
    assert ref_out['names'] == ora_out['names']
    assert len(ref_out['names']) == 15
    assert ref['keys'].tolist() == [list(k) for k in ora_keys]
    assert sorted({k[0] for k in ora_keys}) == [1, 2, 4]


def test_per_key_accumulators_bit_equal(ref, runs):
    ora_keys = runs[2]
    for k, want in zip(ora_keys, ref['key_digests']):
        np.testing.assert_array_equal(digest(ora_keys[k]), want, err_msg=str(k))


@pytest.mark.parametrize('name', ['global', 'norm', 'f2', 'l9h0', 'word'])
def test_finalize_bit_equal(runs, name):
    _, ref_out, _, ora_out = runs
    assert ref_out[name].shape == tuple(ora_out[name].shape)
    np.testing.assert_array_equal(ora_out[name].numpy(), ref_out[name])


def test_error_messages_match(ref, runs):
    pipe = runs[0]
    with O.OracleTrace(pipe) as ot:
        with pytest.raises(RuntimeError) as e_ora:
            ot.compute_global_heat_map()
    assert str(e_ora.value) == str(ref['empty_trace_error'])
    with pytest.raises(ValueError) as w_ora:
        O.port_token_merge_indices(pipe.tokenizer, PROMPT, 'zebra')
    assert str(w_ora.value) == str(ref['missing_word_error'])


def test_unravel_and_merge_indices_match_reference(ref, runs):
    pipe = runs[0]
    probs = torch.arange(8 * 64 * 77, dtype=torch.float64).reshape(8, 64, 77)     # values = positions
    np.testing.assert_array_equal(O.port_unravel(probs).numpy().astype(np.uint16), ref['unravel_perm'])
    for word in ['dog', 'red', 'beach']:
        assert repr(O.port_token_merge_indices(pipe.tokenizer, PROMPT, word)) == str(ref[f'merge_{word}'])
    assert repr(O.port_token_merge_indices(pipe.tokenizer, PROMPT, 'x', word_idx=3)) == str(ref['merge_x_idx3'])


def test_math_layer_agrees_with_port(runs):
    """The float64 restatement agrees to fp32 rounding with the reference's maps, from the key tensors the previous
    tests pin to the reference's."""
    _, ref_out, ora_keys, _ = runs
    keys = [v.numpy() for v in ora_keys.values()]
    n_rows = ref_out['global'].shape[0]
    g = O.math_global_heat_map(keys, 64, n_rows)
    np.testing.assert_allclose(ref_out['global'], g, rtol=2e-5, atol=2e-6)
    gn = O.math_global_heat_map(keys, 64, n_rows, normalize=True)
    np.testing.assert_allclose(ref_out['norm'], gn, rtol=2e-5, atol=2e-6)


def test_save_and_load_heads_match_reference(ref, tmp_path):
    """save_heads writes the same `{gen_idx}.pt` tensors; load_heads replays them into the same maps (trace.py:246-282)."""
    pipe = make_pipeline(TINY_SPEC, dtype=torch.float32, seed=5)
    d_ora = tmp_path / 'ora'
    gen = lambda: torch.Generator().manual_seed(2)
    d_ora.mkdir()
    with O.OracleTrace(pipe, save_heads=True, data_dir=d_ora) as ot:
        pipe(PROMPT, num_inference_steps=2, generator=gen())
        saved_ora = ot.compute_global_heat_map()
    names = sorted(p.name for p in d_ora.iterdir())
    assert names == ref['saved_names'].tolist() and len(names) == 32
    for nme, want in zip(names, ref['saved_digests']):
        np.testing.assert_array_equal(digest(torch.load(d_ora / nme)), want, err_msg=nme)
    np.testing.assert_array_equal(digest(saved_ora), ref['saved_global'])
    other = make_pipeline(TINY_SPEC, dtype=torch.float32, seed=6)     # different weights: P comes from the files
    with O.OracleTrace(other, load_heads=True, data_dir=d_ora) as ot:
        out_ora = other(PROMPT, num_inference_steps=2, generator=gen()).latents
        loaded_ora = ot.compute_global_heat_map()
    np.testing.assert_array_equal(digest(loaded_ora), ref['loaded_global'])
    np.testing.assert_array_equal(digest(out_ora), ref['loaded_latents'])
    np.testing.assert_array_equal(ref['loaded_global'], ref['saved_global'])   # the maps depend on the files only


def test_reference_experiment_dump_loads_in_daam_b200(ref, tmp_path):
    """generation.pt written by the reference's GenerationExperiment.save (experiment.py:140-167) loads in ours, and back."""
    from daam_b200 import GenerationExperiment
    dump = tmp_path / 'q1'
    for i, name in enumerate(ref['experiment_files'].tolist()):
        (dump / name).parent.mkdir(parents=True, exist_ok=True)
        (dump / name).write_bytes(ref[f'experiment_file_{i}'].tobytes())
    maps = torch.from_numpy(ref['experiment_maps'])
    ours = GenerationExperiment.load(dump)
    assert ours.prompt == 'a red ball' and ours.seed == 3 and torch.equal(ours.global_heat_map, maps)
    assert ours.image.size == (16, 16)
    ours.id = '.'
    ours.save(str(tmp_path / 'again'))
    # same folder layout both ways (the reference's own `load` calls torch.load without weights_only=False and therefore
    # cannot read ANY pickled experiment under torch >= 2.6, its own included, so the reverse direction is checked by name)
    listing = lambda root: sorted(str(p.relative_to(root)) for p in root.rglob('*') if p.is_file())
    assert listing(tmp_path / 'again') == listing(dump)


def test_latent96_geometry_bit_equal(ref):
    """768-pixel models (latent_hw 9216, daam/trace.py:32-33): reference and oracle bit-equal on the 96-latent tree,
    including the full-size 96 x 96 = 9216-position layer."""
    from daam_b200.testing.synthetic import TINY96_SPEC
    pipe = make_pipeline(TINY96_SPEC, dtype=torch.float32, seed=5)
    gen = lambda: torch.Generator().manual_seed(13)
    with O.OracleTrace(pipe) as ot:
        pipe(PROMPT, num_inference_steps=2, generator=gen())
        ora_keys = {k: v.clone() for k, v in ot.heat_maps}
        ora_g = ot.compute_global_heat_map(normalize=True)
    assert ref['keys96'].tolist() == [list(k) for k in ora_keys]
    assert {v.shape[-1] for v in ora_keys.values()} == {96, 48, 24}
    for k, want in zip(ora_keys, ref['key96_digests']):
        np.testing.assert_array_equal(digest(ora_keys[k]), want, err_msg=str(k))
    ref_g = golden('pipeline_tiny96')['global_norm']
    assert ref_g.shape == (11, 96, 96)
    np.testing.assert_array_equal(ora_g.numpy(), ref_g)


def test_per_key_sweep_bit_equal(ref, runs):
    """The --all-heads sweep (daam/run/generate.py:239-255): compute_global_heat_map(layer_idx, head_idx) per key."""
    _, ref_out, ora_keys, _ = runs
    assert ref['sweep_keys'].tolist() == [list(k) for k in list(ora_keys)[::5]]
    for (f, l, h), want in zip(ref['sweep_keys'].tolist(), ref['sweep_digests']):
        got = O.port_global_heat_map(list(ora_keys.items()), 4096, ref_out['global'].shape[0] - 2, layer_idx=l,
                                     head_idx=h, normalize=True)
        np.testing.assert_array_equal(digest(got), want, err_msg=str((f, l, h)))
