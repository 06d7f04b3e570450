"""CPU-side checks of the drop-in boundary: the C-ABI library loads and exports every symbol
include/idxtts.h declares; without a GPU it fails loudly instead of falling back."""
import ctypes
import os
import subprocess

import pytest


def test_library_exports_every_declared_symbol(lib_built):
    from indextts_b200 import engine
    lib = engine.load_library()
    syms = engine.declared_symbols()
    assert len(syms) >= 12
    for s in syms:
        assert hasattr(lib, s), s
    assert b"sm_90a" in lib.idx_version()


def test_header_is_plain_c(lib_built, tmp_path):
    """include/idxtts.h must compile as C (no C++/torch types in the boundary)."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "t.c"
    src.write_text('#include "idxtts.h"\nint main(void){ idx_sampling s; (void)s; return 0; }\n')
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(root, "include"),
                           "-c", str(src), "-o", str(tmp_path / "t.o")])


def test_no_gpu_fails_loudly(lib_built):
    """The product path has no CPU fallback: without a device, idx_create reports IDX_ERR_NOGPU."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from indextts_b200.engine import Engine
    with pytest.raises(RuntimeError, match="no CUDA device|no CPU fallback"):
        Engine(0)


def test_product_path_does_not_import_oracle():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    pkg = os.path.join(root, "index-tts_b200")
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dp, f)).read()
                assert "import oracle" not in txt and "from oracle" not in txt, f
