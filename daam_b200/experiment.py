"""On-disk record of one generation: image + global heat map + prompt (SURVEY.md section 8f, rank 3).

A reduced mirror of the reference's ``GenerationExperiment`` (``daam/experiment.py:102-344``): the same
fields and the same folder layout -- ``<path>/<id>/<subtype>/generation.pt`` (the pickled dataclass), ``output.png``,
``<path>/<id>/prompt.txt``, ``seed.txt``, ``annotations.json`` (experiment.py:140-175). Compatibility is ONE-WAY: dumps
written by the reference load here (``load`` maps its pickled class path ``daam.experiment.GenerationExperiment`` onto
this class); ``generation.pt`` written here pickles ``daam_b200.experiment.GenerationExperiment`` and is for this
package (the text/PNG side files are identical either way). ``save`` moves the heat map to the CPU so that a dump loads
on a box without a GPU. The COCO label tables, ground-truth / prediction mask handling and matplotlib heat-map rendering of
the reference are out of scope (SURVEY.md section 2 rows 5, 6).
"""
from __future__ import annotations

import json
import pickle
from dataclasses import dataclass
from pathlib import Path
from typing import Any, Dict, Optional, Union

import numpy as np
import torch

__all__ = ['GenerationExperiment']


class _CompatUnpickler(pickle.Unpickler):
    """Resolves the reference's module path to this package when reading its dumps."""

    def find_class(self, module, name):
        if name == 'GenerationExperiment' and module in ('daam.experiment', 'daam_b200.experiment'):
            return GenerationExperiment
        return super().find_class(module, name)


class _CompatPickle:
    """``pickle_module`` for ``torch.load``."""
    __name__ = 'daam_b200_compat_pickle'
    Unpickler = _CompatUnpickler
    load = staticmethod(lambda f, **kw: _CompatUnpickler(f, **kw).load())


@dataclass
class GenerationExperiment:
    """Class to hold experiment parameters. Pickleable (experiment.py:102-117)."""
    image: Any
    global_heat_map: torch.Tensor
    prompt: str

    seed: int = None
    id: str = '.'
    path: Optional[Path] = None

    truth_masks: Optional[Dict[str, torch.Tensor]] = None
    prediction_masks: Optional[Dict[str, torch.Tensor]] = None
    annotations: Optional[Dict[str, Any]] = None
    subtype: Optional[str] = '.'
    tokenizer: Any = None

    def __post_init__(self):
        if isinstance(self.path, str):
            self.path = Path(self.path)
        self.path = None if self.path is None else self.path / self.id

    def nsfw(self) -> bool:
        return np.sum(np.array(self.image)) == 0

    def heat_map(self, tokenizer=None):
        from .heatmap import GlobalHeatMap
        return GlobalHeatMap(self.tokenizer if tokenizer is None else tokenizer, self.prompt, self.global_heat_map)

    def clear_checkpoint(self):
        (self.path / 'generation.pt').unlink(missing_ok=True)

    def save(self, path: str = None, heat_maps: bool = False, tokenizer=None):
        """Writes the folder layout of experiment.py:140-167. ``heat_maps=True`` (per-word PNG overlays) needs
        matplotlib and is not part of the hot path."""
        root = self.path if path is None else Path(path) / self.id
        (root / self.subtype).mkdir(parents=True, exist_ok=True)
        import copy
        on_disk = self
        if torch.is_tensor(self.global_heat_map) and self.global_heat_map.is_cuda:
            on_disk = copy.copy(self)               # (not dataclasses.replace: __post_init__ would re-append the id)
            on_disk.global_heat_map = self.global_heat_map.detach().cpu()
        torch.save(on_disk, root / self.subtype / 'generation.pt')
        if hasattr(self.image, 'save'):                 # a PIL image
            self.image.save(root / self.subtype / 'output.png')
        (root / 'prompt.txt').write_text(self.prompt)
        (root / 'seed.txt').write_text(str(self.seed))
        if heat_maps:
            raise RuntimeError('rendering heat-map PNGs needs matplotlib, which is outside the heat-map hot path')
        self.save_annotations(root)

    def save_annotations(self, path: Path = None):
        path = self.path if path is None else path
        if self.annotations is not None:
            with (path / 'annotations.json').open('w') as f:
                json.dump(self.annotations, f)

    def annotate(self, key: str, value: Any) -> 'GenerationExperiment':
        if self.annotations is None:
            self.annotations = {}
        self.annotations[key] = value
        return self

    @staticmethod
    def read_seed(path: Union[str, Path], prompt_id: str = None) -> int:
        base = Path(path) if prompt_id is None else Path(path) / prompt_id
        return int((base / 'seed.txt').read_text())

    @staticmethod
    def read_prompt(path: Union[str, Path], prompt_id: str = None) -> str:
        return (Path(path) / ('.' if prompt_id is None else prompt_id) / 'prompt.txt').read_text().strip()

    @staticmethod
    def has_experiment(path: Union[str, Path], prompt_id: str) -> bool:
        return (Path(path) / prompt_id / 'generation.pt').exists()

    @staticmethod
    def has_annotations(path: Union[str, Path]) -> bool:
        return Path(path).joinpath('annotations.json').exists()

    @classmethod
    def load(cls, path, subtype: str = '.', map_location=None) -> 'GenerationExperiment':
        """Reads ``<path>/<subtype>/generation.pt`` written by this package or by the reference (experiment.py:303-344,
        without its mask loading)."""
        path = Path(path)
        exp = torch.load(path / subtype / 'generation.pt', map_location=map_location, pickle_module=_CompatPickle,
                         weights_only=False)
        exp.subtype = subtype
        exp.path = path
        ann = path / 'annotations.json'
        exp.annotations = json.load(ann.open()) if ann.exists() else None
        return exp
