"""The C-ABI shared library loads on a CPU-only box, exports every symbol include/gem_b200.h
declares, and refuses loudly to work without a GPU (no CPU fallback)."""
import ctypes as C
import os
import re

import pytest

import gem_b200
import native
from gem_b200 import _lib, build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    src = open(os.path.join(ROOT, "include", "gem_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(gem_[a-z_0-9]+)\s*\(", src)))


def test_library_is_built_for_sm90a_only():
    lib = build.build()
    assert os.path.exists(lib)
    import subprocess, shutil
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([cuobjdump, "-lelf", lib], capture_output=True, text=True).stdout
    archs = set(re.findall(r"sm_(\d+a?)", out))
    assert archs == {"90a"}, archs


def test_every_declared_symbol_is_exported_and_bound():
    lib = _lib.load()
    names = header_symbols()
    assert len(names) >= 25
    for name in names:
        assert hasattr(lib, name), f"{name} declared in gem_b200.h but not exported"
        assert name in _lib.SYMBOLS, f"{name} has no ctypes prototype"
    assert set(_lib.SYMBOLS) == set(names)
    assert lib.gem_version() == 100


def test_no_cpu_fallback(gpu_available):
    if gpu_available:
        pytest.skip("GPU present")
    with pytest.raises(gem_b200.GemError) as e:
        gem_b200.ElevationMap(64, 0.1)
    assert "GEM_ERR_NO_DEVICE" in str(e.value) and "no CPU fallback" in str(e.value)


def test_create_rejects_bad_arguments():
    lib = _lib.load()
    h = C.c_void_p()
    cfg = _lib.GemConfig()
    cfg.length = 0
    cfg.resolution = 0.1
    assert lib.gem_create(C.byref(cfg), C.byref(h)) == 1
    assert b"length" in lib.gem_last_error(None)
    assert lib.gem_create(None, C.byref(h)) == 1


def test_product_does_not_reference_the_oracle():
    """only tests/, __graft_entry__.smoke() and bench.py's cpu legs may touch oracle/"""
    for dirpath, _, files in os.walk(os.path.join(ROOT, "gem_b200")):
        for fn in files:
            if fn.endswith((".py", ".cu", ".cuh", ".cpp", ".hpp", ".h")):
                txt = open(os.path.join(dirpath, fn), errors="ignore").read()
                if fn == "build.py":
                    txt = txt.split("def build_oracle")[0]
                assert "oracle_lib" not in txt and "gem_oracle" not in txt, os.path.join(dirpath, fn)
    assert "oracle" not in open(os.path.join(ROOT, "include", "gem_b200.h")).read().lower()


def test_ctypes_struct_layouts_match_the_header():
    """the ctypes mirrors in gem_b200/_lib.py must have the sizes and field offsets the C compiler gives the structs of
    include/gem_b200.h (a drift here corrupts every call silently)"""
    native.assert_struct_layouts({"gem_config": _lib.GemConfig, "gem_sensor_model": _lib.GemSensorModel,
                                  "gem_frame": _lib.GemFrame, "gem_stats": _lib.GemStats, "gem_profile": _lib.GemProfile})
