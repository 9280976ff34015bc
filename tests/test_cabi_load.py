"""CPU-side checks of the drop-in boundary: the C-ABI library builds, loads and
exports every symbol include/lb200.h declares (no compute calls without a GPU)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "lb200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(lb_[a-z0-9_]+)\s*\(", src)))


@pytest.fixture(scope="module")
def lib_path():
    from latentblending_b200 import build
    return build.build()


def test_header_symbols_exported(lib_path):
    lib = ctypes.CDLL(lib_path)
    names = _declared()
    assert len(names) >= 8
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/lb200.h but not exported"


def test_ctypes_signatures_cover_header_abi4(lib_path):
    from latentblending_b200 import _cabi
    assert sorted(_cabi.SIGNATURES) == _declared()
    lib = _cabi.load()
    assert lib.lb_abi_version() == 4


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "latentblending_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dp, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", txt, flags=re.M), f
                assert "/root/reference" not in txt, f


def test_cpu_tensors_are_rejected(lib_path):
    import torch
    from latentblending_b200 import utils
    with pytest.raises(RuntimeError):
        utils.interpolate_spherical(torch.zeros(8), torch.ones(8), 0.5)
