"""CPU: the C-ABI library builds for sm_90a, loads without a GPU, and exports every symbol include/ptb_b200.h declares."""
import ctypes
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, 'include', 'ptb_b200.h')


def declared_symbols():
    src = open(HEADER).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return sorted(set(re.findall(r'\b(ptb_[a-z0-9_]+)\s*\(', src)))


@pytest.fixture(scope='module')
def lib_path():
    from pointtinybenchmark_b200.csrc import build as b
    return b.build()


def test_header_is_plain_c(tmp_path):
    """the boundary is a C ABI: the header must compile as C (no C++ / torch types)."""
    c = tmp_path / 't.c'
    c.write_text('#include "ptb_b200.h"\nint main(void){ptb_refine_cfg c; c.flags = 0; return c.flags + PTB_ABI_VERSION - 1;}\n')
    r = subprocess.run(['gcc', '-std=c99', '-Wall', '-Werror', '-I', os.path.join(ROOT, 'include'), '-c', str(c), '-o', str(tmp_path / 't.o')],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_library_exports_every_declared_symbol_at_abi_version_2(lib_path):
    syms = declared_symbols()
    assert len(syms) >= 25
    lib = ctypes.CDLL(lib_path)
    missing = [s for s in syms if not hasattr(lib, s)]
    assert not missing, missing
    lib.ptb_abi_version.restype = ctypes.c_int
    assert lib.ptb_abi_version() == 2


def test_ctypes_binding_covers_the_header(lib_path):
    from pointtinybenchmark_b200 import _lib
    _lib.load()
    assert _lib.MISSING == []
    assert sorted(_lib.SIGNATURES) == declared_symbols()


def test_sass_is_sm90a_only(lib_path):
    r = subprocess.run(['cuobjdump', '--list-elf', lib_path], capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip('cuobjdump unavailable')
    archs = set(re.findall(r'sm_\d+a?', r.stdout))
    assert archs == {'sm_90a'}, archs


def test_argument_validation_errors_are_reported_without_a_gpu(lib_path):
    """argument checks run before any CUDA call: a bad call returns non-zero and sets ptb_last_error()."""
    from pointtinybenchmark_b200 import _lib
    lib = _lib.load()
    rc = lib.ptb_linear_rows(None, 4, 30, 30, None, None, 8, None, 8, None)     # Cin % 16 != 0
    assert rc != 0
    assert b'Cin' in lib.ptb_last_error()
    import ctypes
    dummy = ctypes.c_void_p(16)      # never dereferenced: the size check fires first
    rc = lib.ptb_multiclass_nms(dummy, dummy, 1, 5000, 80, 32.0, 32.0, 0.05, 0.5, 100, dummy, dummy, dummy, dummy, dummy, dummy, 0, None)
    assert rc != 0 and b'4096' in lib.ptb_last_error()
