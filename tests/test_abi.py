"""CPU tier: the C-ABI library builds for sm_90a, loads without a GPU and exports every symbol that
include/jtb_check.h declares; the ctypes struct images match the header's layout."""
import ctypes
import os
import re

import pytest

from jepsen_tigerbeetle_b200 import abi, history, native

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "jtb_check.h")


def declared_functions():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(jtb_[a-z_]+)\s*\(", src)))


def test_header_and_binding_agree_on_exports():
    assert declared_functions() == sorted(native.EXPORTS)


def test_library_builds_loads_and_exports_every_symbol():
    native.build()
    lib = native.lib()
    for name in declared_functions():
        assert hasattr(lib, name), name
    assert lib.jtb_abi_version() == abi.ABI_VERSION


def test_no_cpu_fallback_without_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    assert native.device_count() <= 0
    with pytest.raises(native.NativeError):
        native.Context(device=0)


def test_struct_sizes_match_the_compiled_library():
    lib = native.lib()
    images = [history.CHistory, history.CModel, abi.COpts, abi.CLinShard, abi.CLinResult, abi.CSetFullShard,
              abi.CSetFullOut, abi.CBankResult, abi.CFinalConfig]
    for which, img in enumerate(images):
        assert lib.jtb_struct_size(which) == ctypes.sizeof(img), img.__name__
    assert lib.jtb_struct_size(99) == -1


def test_product_does_not_import_the_oracle():
    pkg = os.path.join(ROOT, "jepsen_tigerbeetle_b200")
    for dirpath, _dirs, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp", ".h")):
                text = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in text and "from oracle" not in text, f
                assert "oracle/" not in text or f in ("jtb_prep.h",), f
