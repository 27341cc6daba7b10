"""CPU-side checks of the C-ABI boundary: the library loads and exports every symbol the header declares."""
import ctypes
import os
import re


def test_library_exports_every_declared_symbol():
    import __graft_entry__ as g
    g.build()
    from hawkeye_b200 import _lib
    protos = _lib.parse_header()
    assert len(protos) >= 20
    lib = ctypes.CDLL(_lib.LIB_PATH)
    missing = [n for n in protos if not hasattr(lib, n)]
    assert not missing, missing
    lib.hk_version.restype = ctypes.c_char_p
    assert b'hawkeye_b200' in lib.hk_version() and b'sm_90a' in lib.hk_version()


def test_no_fallback_when_library_missing(monkeypatch, tmp_path):
    from hawkeye_b200 import _lib
    monkeypatch.setattr(_lib, '_lib', None)
    monkeypatch.setattr(_lib, 'LIB_PATH', str(tmp_path / 'nope.so'))
    import pytest
    with pytest.raises(_lib.HawkeyeLibError):
        _lib.lib()


def test_ops_refuse_cpu_tensors():
    import pytest
    import torch
    from hawkeye_b200 import ops, _lib
    with pytest.raises(_lib.HawkeyeLibError):
        ops.bilinear_pool(torch.rand(1, 128, 4, 4))


def test_product_does_not_import_oracle():
    root = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'hawkeye_b200')
    for dp, _, fs in os.walk(root):
        for f in fs:
            if f.endswith('.py'):
                src = open(os.path.join(dp, f)).read()
                assert not re.search(r'^\s*(from|import)\s+\S*oracle|__import__\([^)]*oracle|import_module\([^)]*oracle', src,
                                     flags=re.M), f
