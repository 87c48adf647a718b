"""TEST INFRASTRUCTURE -- imports the *verbatim* reference (castorini/daam) from ``$DAAM_REFERENCE_ROOT`` behind stubs.

The reference cannot be imported as-is in the build environment: ``diffusers``, ``matplotlib``, ``spacy`` (and friends) are
not installed and there is no network (SURVEY.md section 8c). None of those packages contributes arithmetic to the hot path
except ``diffusers.models.attention_processor.Attention``, whose 0.21.2 semantics ``daam_b200.testing.synthetic.
SyntheticAttention`` restates. This loader registers empty stand-in modules for the missing imports, points
``diffusers...Attention`` at that restatement, and then imports ``daam`` from the read-only reference tree.

It exists to generate the golden fixtures under ``tests/golden/`` (``oracle/make_golden.py``), which is how the suite
pins ``oracle/daam_oracle.py`` against the reference's own code without needing the reference. Only the golden-vector
generator may use this module; the product (``daam_b200``) never imports anything under ``oracle/``.
"""
from __future__ import annotations

import importlib
import os
import sys
import types

REFERENCE_ROOT = os.environ.get('DAAM_REFERENCE_ROOT', '')   # a castorini/daam v0.2.0 checkout


def reference_available() -> bool:
    return os.path.isfile(os.path.join(REFERENCE_ROOT, 'daam', 'trace.py'))


def _stub(name: str, **attrs) -> types.ModuleType:
    mod = types.ModuleType(name)
    mod.__dict__.update(attrs)
    mod.__path__ = []  # behave like a package so that sub-imports resolve
    sys.modules[name] = mod
    return mod


def _install_stubs():
    from daam_b200.testing.synthetic import SyntheticAttention

    class _Empty:  # the reference only uses these names for annotations and one exact ``type(...) ==`` test
        pass

    if 'diffusers' not in sys.modules:
        names = ['UNet2DConditionModel', 'StableDiffusionPipeline', 'StableDiffusionXLPipeline', 'DiffusionPipeline']
        _stub('diffusers', **{n: type(n, (_Empty,), {}) for n in names})
        _stub('diffusers.models')
        _stub('diffusers.models.attention_processor', Attention=SyntheticAttention)
        _stub('diffusers.image_processor', VaeImageProcessor=type('VaeImageProcessor', (_Empty,), {}))
    for name in ('matplotlib', 'matplotlib.pyplot', 'spacy', 'spacy.tokens', 'gradio', 'inflect', 'nltk', 'ftfy',
                 'skimage', 'numba'):
        if name not in sys.modules:
            try:
                importlib.import_module(name)
            except Exception:
                _stub(name)
    sys.modules['matplotlib'].pyplot = sys.modules['matplotlib.pyplot']
    sys.modules['spacy'].tokens = sys.modules['spacy.tokens']
    if not hasattr(sys.modules['spacy.tokens'], 'Token'):
        sys.modules['spacy.tokens'].Token = type('Token', (), {})


def load_reference():
    """Returns the reference's ``daam`` package (verbatim code, stubbed third-party imports)."""
    if not reference_available():
        raise RuntimeError(f'reference tree not found under {REFERENCE_ROOT!r}: set DAAM_REFERENCE_ROOT to a castorini/daam '
                           f'v0.2.0 checkout')
    repo_root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if repo_root not in sys.path:
        sys.path.insert(0, repo_root)
    _install_stubs()
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    stale = sys.modules.get('daam')
    if stale is not None and not (getattr(stale, '__file__', None) or '').startswith(os.path.abspath(REFERENCE_ROOT)):
        for name in [n for n in sys.modules if n == 'daam' or n.startswith('daam.')]:
            del sys.modules[name]
    import daam  # noqa: E402  (the reference package)
    assert os.path.abspath(daam.__file__).startswith(os.path.abspath(REFERENCE_ROOT)), daam.__file__
    return daam
