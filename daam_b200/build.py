"""Builds ``libdaam_b200.so`` in-tree with nvcc for sm_90a (``python -m daam_b200.build``)."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SOURCES = ['api.cu', 'accumulate_simt.cu', 'accumulate_mma.cu', 'finalize.cu', 'words.cu', 'components.cu', 'ranking.cu', 'boundary.cu', 'distance.cu', 'refine.cu', 'crf.cu', 'superpixels.cu', 'value_norms.cu', 'probs.cu', 'accumulate_joint.cu']
OUT = os.path.join(HERE, 'libdaam_b200.so')
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17', '-Xcompiler', '-fPIC',
              '-I', os.path.join(ROOT, 'include'), '-shared']


def _nvcc() -> str:
    for cand in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', 'nvcc'):
        if cand and (os.path.sep not in cand or os.path.isfile(cand)):
            return cand
    return 'nvcc'


def needs_build() -> bool:
    if not os.path.isfile(OUT):
        return True
    deps = [os.path.join(HERE, 'csrc', f) for f in os.listdir(os.path.join(HERE, 'csrc'))]
    deps.append(os.path.join(ROOT, 'include', 'daam_b200.h'))
    return any(os.path.getmtime(d) > os.path.getmtime(OUT) for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    """``verbose``: compile with ``-Xptxas -v`` and echo the compiler output (registers, shared memory, spills)."""
    if not force and not needs_build():
        return OUT
    cmd = [_nvcc()] + NVCC_FLAGS + (['-Xptxas', '-v'] if verbose else []) + ['-o', OUT] + \
          [os.path.join(HERE, 'csrc', s) for s in SOURCES]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
    if res.returncode != 0:
        raise RuntimeError('nvcc failed building libdaam_b200.so')
    return OUT


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
