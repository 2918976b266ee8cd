"""CPU-only: the C-ABI library loads and exports every symbol include/arroy_b200.h declares."""
import os
import re

import arroy_b200

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    with open(os.path.join(ROOT, "include", "arroy_b200.h")) as f:
        src = f.read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(arroy_b200_[a-z0-9_]+)\s*\(", src)) - {"arroy_b200_node_sink", "arroy_b200_cancel_fn"})


def test_library_exports_every_declared_symbol():
    lib = arroy_b200.load()
    names = declared_symbols()
    assert len(names) >= 18
    for name in names:
        assert hasattr(lib, name), name
    bound = {s[0] for s in arroy_b200.SIGNATURES}
    assert set(names) == bound, set(names) ^ bound


def test_version_string():
    assert b"sm_90a" in arroy_b200.load().arroy_b200_version()


def test_create_fails_loudly_without_a_device():
    import ctypes as C
    import torch
    if torch.cuda.is_available():
        return
    lib = arroy_b200.load()
    h = C.c_void_p()
    assert lib.arroy_b200_create(0, C.byref(h)) == arroy_b200._capi.ERR_CUDA
    try:
        arroy_b200.Context(0)
    except arroy_b200.ArroyB200Error as e:
        assert e.code == arroy_b200._capi.ERR_CUDA
    else:
        raise AssertionError("Context() must raise without a CUDA device (no CPU fallback)")
