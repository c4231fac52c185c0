"""The C-ABI library loads and exports every symbol include/fastdepth_b200.h declares
(no compute calls: there is no GPU here)."""
import ctypes
import os
import re

import pytest

from conftest import ROOT
from fastdepth_b200 import _lib

HEADER = os.path.join(ROOT, 'include', 'fastdepth_b200.h')


def declared_functions():
    src = open(HEADER).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return sorted(set(re.findall(r'\b(fd_[a-z_0-9]+)\s*\(', src)))


def test_header_and_binding_agree():
    assert declared_functions() == sorted(_lib.SIGNATURES)


def test_library_exports_every_symbol(built_lib):
    lib = ctypes.CDLL(built_lib)
    for name in declared_functions():
        assert hasattr(lib, name), name
    assert _lib.load().fd_abi_version() == 2


def test_no_torch_types_in_signatures():
    src = re.sub(r'/\*.*?\*/', '', open(HEADER).read(), flags=re.S)      # declarations only
    assert 'torch' not in src.lower() and 'at::' not in src and 'std::' not in src
    assert re.findall(r'#include\s*<([^>]+)>', src) == ['stddef.h', 'stdint.h']


def test_fails_loudly_without_gpu(built_lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip('GPU present')
    lib = _lib.load()
    descs = (_lib.StageDesc * 3)()
    handle = ctypes.c_void_p()
    rc = lib.fd_plan_create(descs, 3, 1, 32, 32, _lib.FD_F16, 0, ctypes.byref(handle))
    assert rc == -2 and b'no CPU fallback' in lib.fd_last_error()
    with pytest.raises(RuntimeError):
        _lib.check(rc)


def test_built_for_sm90a_only(built_lib):
    import subprocess
    out = subprocess.run(['cuobjdump', '-lelf', built_lib], capture_output=True, text=True).stdout
    archs = set(re.findall(r'sm_(\d+a?)', out))
    assert archs == {'90a'}, archs
