"""The C-ABI library loads on a CPU-only box and exports every symbol declared in include/cape_b200.h."""
import ctypes
import os
import re

from cape_b200 import _lib

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))


def declared_functions():
    src = open(os.path.join(ROOT, "include", "cape_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(cape_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_exported(lib_built):
    names = declared_functions()
    assert len(names) >= 20
    raw = ctypes.CDLL(_lib.LIB_PATH)
    for n in names:
        assert hasattr(raw, n), "declared in the header but not exported: " + n
    assert sorted(_lib.SIGNATURES) == names, "ctypes prototypes and header out of sync"


def test_abi_v4_and_error_string(lib_built):
    assert lib_built.cape_abi_version() == 4
    assert isinstance(lib_built.cape_last_error(), bytes)


def test_set_tuning_rejects_unknown_keys(lib_built):
    """cape_set_tuning takes only the documented knobs and returns the previous value of one it takes."""
    assert lib_built.cape_set_tuning(4, 1) < 0
    prev = lib_built.cape_set_tuning(7, 0)
    try:
        assert prev >= 0
        assert lib_built.cape_set_tuning(7, 0) == 0
    finally:
        lib_built.cape_set_tuning(7, prev)


def test_struct_layout_matches_header():
    """cape_term / cape_conv_args / cape_dw_args field order as declared (ctypes mirrors must not drift)."""
    src = open(os.path.join(ROOT, "include", "cape_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)

    def fields(struct_name):
        body = re.search(r"typedef struct \{([^}]*)\} %s;" % struct_name, src).group(1)
        out = []
        for decl in body.split(";"):
            decl = decl.strip()
            if not decl:
                continue
            for part in decl.split(","):
                out.append(re.sub(r"\[.*\]", "", part.strip().split()[-1].lstrip("*")))
        return out

    assert fields("cape_term") == [f[0] for f in _lib.Term._fields_]
    assert fields("cape_conv_args") == [f[0] for f in _lib.ConvArgs._fields_]
    assert fields("cape_dw_args") == [f[0] for f in _lib.DwArgs._fields_]
    assert fields("cape_gemm_item") == [f[0] for f in _lib.GemmItem._fields_]
    assert fields("cape_wprep") == [f[0] for f in _lib.WPrep._fields_]
    assert fields("cape_apply_term") == [f[0] for f in _lib.ApplyTerm._fields_]
    assert fields("cape_apply_args") == [f[0] for f in _lib.ApplyArgs._fields_]


def test_no_cpu_fallback():
    """Constructing the engine without a GPU must fail loudly, not fall back."""
    import pytest
    import torch
    from cape_b200.engine import Topology
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(_lib.CapeError):
        Topology(0)
