"""CPU: the C-ABI shared library builds, loads and exports exactly what include/sae_b200.h declares."""
import ctypes
import os
import re

import pytest

from swapping_autoencoder_pytorch_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_functions():
    text = open(os.path.join(ROOT, "include", "sae_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(sae_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build_library()
    lib = ctypes.CDLL(_lib.LIB_PATH)
    declared = _header_functions()
    assert len(declared) >= 15
    for name in declared:
        assert hasattr(lib, name), "header declares %s but the library does not export it" % name
    assert sorted(_lib.SIGNATURES) == declared, "ctypes table and header disagree"


def _header_struct(name):
    """[(field, C type)] of `typedef struct <name> { ... } <name>;` in the header, in declaration order"""
    text = open(os.path.join(ROOT, "include", "sae_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    body = re.search(r"typedef\s+struct\s+%s\s*\{(.*?)\}\s*%s\s*;" % (name, name), text, flags=re.S)
    assert body, name
    fields = []
    for decl in body.group(1).split(";"):
        decl = decl.strip()
        if not decl:
            continue
        m = re.match(r"^((?:const\s+)?[A-Za-z_][A-Za-z0-9_]*\s*\**)\s*(.*)$", decl, flags=re.S)
        ctype = re.sub(r"\s+", " ", m.group(1)).strip()
        for var in m.group(2).split(","):
            var = var.strip()
            stars = var.count("*")
            fields.append((var.lstrip("*").strip(), ctype + "*" * stars))
    return fields


def _ctypes_of(ctype):
    if ctype.endswith("*"):
        return ctypes.c_void_p
    return {"int32_t": ctypes.c_int32, "float": ctypes.c_float}[ctype]


@pytest.mark.parametrize("c_name,py_struct", [("sae_conv_geom", _lib.ConvGeom), ("sae_conv_epilogue", _lib.ConvEpilogue)])
def test_ctypes_structs_match_header(c_name, py_struct):
    """field names, order and C types of the structs the conv entry points read, against their ctypes mirrors: a slip would
    feed the kernels a wrong geometry or wrong epilogue values without any error"""
    declared = [(f, _ctypes_of(t)) for f, t in _header_struct(c_name)]
    assert len(declared) >= 10
    assert [(f, t) for f, t in py_struct._fields_] == declared


def test_abi_version_and_error_reporting():
    lib = _lib.load()
    assert lib.sae_abi_version() == _lib.SAE_ABI_VERSION
    # argument validation happens before any CUDA call, so it can be exercised without a GPU
    rc = lib.sae_upfirdn2d(None, None, None, 1, 4, 4, 4, 3, 3, 1, 1, 1, 1, 0, 0, 0, 0, 0, None)   # major=1, null data
    assert rc == -1 and b"null" in lib.sae_last_error()
    g = _lib.ConvGeom(1, 4, 4, 8, 8, 3, 3, 0, 4, 1, 1, 1)      # P = 0 is invalid
    rc = lib.sae_conv2d_fprop(None, None, None, ctypes.byref(g), None, 0, None)
    assert rc == -1


def test_product_refuses_cpu_tensors():
    import torch
    from swapping_autoencoder_pytorch_b200 import backend
    k = backend.CudaKernels()
    with pytest.raises(_lib.SaeError):
        k.upfirdn2d(torch.zeros(1, 4, 4, 4), torch.ones(3, 3), 1, 1, 1, 1, 1, 1, 1, 1)
