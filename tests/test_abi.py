"""CPU: the C-ABI library builds, loads, and exports every symbol include/pf_b200.h declares (no compute calls)."""
import ctypes
import os
import re

import pytest

from perspectivefields_b200 import _native


@pytest.fixture(scope="module")
def built():
    _native.build()
    return _native.LIB_PATH


def _declared_symbols():
    with open(_native.HEADER) as f:
        src = f.read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(pf_[a-z0-9_]+)\s*\(", src)))


def test_header_declares_the_bound_entry_points():
    assert sorted(_native.EXPORTS) == _declared_symbols()


def test_library_exports_every_declared_symbol(built):
    L = ctypes.CDLL(built)
    for name in _declared_symbols():
        assert hasattr(L, name), name


def test_abi_version_and_error_channel(built):
    L = _native.lib()
    assert L.pf_abi_version() == 3
    assert L.pf_kernel_launch_count() >= 0
    # argument validation happens before any CUDA call
    assert L.pf_create(0, None, None) < 0
    assert b"null" in L.pf_last_error()


def test_sass_is_sm100a_tensor_core_code(built):
    import shutil
    import subprocess

    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    out = subprocess.run(["cuobjdump", "-lelf", built], capture_output=True, text=True).stdout
    assert "sm_90a" in out
