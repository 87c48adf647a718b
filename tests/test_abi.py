"""The C-ABI library loads, exports every symbol include/daam_b200.h declares, agrees with the header on struct
layout, and refuses to compute without a CUDA device (no CPU fallback). No kernel is launched here."""
import ctypes
import os
import re
import subprocess
import tempfile

import pytest
import torch

from daam_b200 import _native
from daam_b200.build import build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, 'include', 'daam_b200.h')


@pytest.fixture(scope='module')
def lib():
    build()
    return _native.load()


def declared_functions():
    text = open(HEADER).read()
    text = re.sub(r'/\*.*?\*/', '', text, flags=re.S)
    return sorted(set(re.findall(r'\b(daam_[a-z_0-9]+)\s*\(', text)))


def test_header_and_binding_agree():
    assert declared_functions() == sorted(_native.EXPORTS)


def test_every_declared_symbol_is_exported_at_abi_4(lib):
    for name in declared_functions():
        assert hasattr(lib, name), f'{name} declared in include/daam_b200.h but not exported'
    assert _native.abi_version() == _native.ABI_VERSION == 4
    for name in ('daam_finalize', 'daam_finalize_per_key', 'daam_normalize_maps', 'daam_word_heat_map', 'daam_expand_as',
                 'daam_expand_words'):   # one entry point per operation, no `_rect` twin
        assert not hasattr(lib, name + '_rect'), f'{name}_rect is still exported'


def test_struct_layout_matches_the_header():
    src = r'''
#include <stdio.h>
#include <stddef.h>
#include "daam_b200.h"
int main(void) {
  printf("%zu %zu %zu %zu %zu %zu\n", sizeof(daam_layer), offsetof(daam_layer, acc), offsetof(daam_layer, k_stride_head),
         offsetof(daam_layer, n_prompts), offsetof(daam_layer, dtype), offsetof(daam_layer, scale));
  printf("%zu %zu %zu\n", sizeof(daam_key_group), offsetof(daam_key_group, heads), offsetof(daam_key_group, head_sel));
  printf("%d %d %d %d\n", DAAM_TOKENS, DAAM_F32, DAAM_F16, DAAM_BF16);
  return 0;
}'''
    with tempfile.TemporaryDirectory() as tmp:
        c, exe = os.path.join(tmp, 't.c'), os.path.join(tmp, 't')
        open(c, 'w').write(src)
        subprocess.check_call(['gcc', '-std=c99', '-I', os.path.join(ROOT, 'include'), c, '-o', exe])  # header is plain C
        lines = subprocess.check_output([exe], text=True).split('\n')
    L, K = _native.DaamLayer, _native.DaamKeyGroup
    assert [int(v) for v in lines[0].split()] == [ctypes.sizeof(L), L.acc.offset, L.k_stride_head.offset,
                                                   L.n_prompts.offset, L.dtype.offset, L.scale.offset]
    assert [int(v) for v in lines[1].split()] == [ctypes.sizeof(K), K.heads.offset, K.head_sel.offset]
    assert [int(v) for v in lines[2].split()] == [_native.TOKENS, _native.DAAM_F32, _native.DAAM_F16, _native.DAAM_BF16]


@pytest.mark.skipif(torch.cuda.is_available(), reason='checks the no-device behaviour')
def test_no_cpu_fallback_without_a_device(lib):
    layer = _native.DaamLayer(q=16, k=16, acc=16, q_stride_prompt=0, q_stride_pixel=64, q_stride_head=64,
                              k_stride_prompt=0, k_stride_token=64, k_stride_head=64, n_prompts=1, heads=1, hw=64,
                              tokens=77, head_dim=64, dtype=_native.DAAM_F32, scale=0.125, reserved=0)
    with pytest.raises(_native.NativeError) as e:
        _native.accumulate([layer], 0)
    assert e.value.code == _native.E_CUDA
    with pytest.raises(_native.NativeError):
        _native.device_info()


def test_argument_validation_messages(lib):
    # validation happens after the device probe, so without a GPU only the error channel itself can be checked
    assert isinstance(lib.daam_last_error(), bytes)
    assert _native.launch_count() >= 0


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    monkeypatch.setattr(_native, '_lib', None)
    monkeypatch.setattr(_native, 'LIB_PATH', str(tmp_path / 'nope.so'))
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        _native.load()
