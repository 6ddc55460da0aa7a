"""C++ host side: the header-only facade (include/gem_b200/elevation_map.hpp) and the
source-level shim re-exporting the reference's nine entry points (compat/gpu_process_shim.cpp).
CPU: both compile and link against libgem_b200.so (the shim against the stand-in Eigen header,
the real Eigen is not in this image).  GPU: the program runs and both paths agree."""
import os
import subprocess

import pytest

import native

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def compile_with_shim(out_dir, name, extra_flags=(), shared=False):
    """tests/cxx/<name>.cpp + the shim, linked against libgem_b200.so, built into out_dir (the tree may be read-only):
    a program, or with shared=True the shared library lib<name>.so"""
    srcs = [os.path.join(native.CXX, name + ".cpp"), os.path.join(ROOT, "compat", "gpu_process_shim.cpp")]
    flags = [*extra_flags, *(("-shared", "-fPIC") if shared else ()), "-I", os.path.join(ROOT, "oracle", "mini_eigen")]
    return native.facade_program(f"lib{name}.so" if shared else name, out_dir, flags, sources=srcs)


def test_shim_harness_builds_with_the_nine_entry_points(tmp_path):
    so = compile_with_shim(tmp_path, "shim_harness", shared=True)
    out = subprocess.run(["nm", "-D", "--defined-only", so], capture_output=True, text=True).stdout
    for sym in ("ref_init", "ref_move", "ref_process_points", "ref_fuse", "ref_var_update", "ref_map_feature",
                "ref_raytracing", "ref_optmove", "ref_closeloop"):
        assert f" {sym}" in out, sym


def test_three_thread_program_compiles(tmp_path):
    assert os.path.exists(compile_with_shim(tmp_path, "threads_shim", ["-pthread"]))


@pytest.mark.gpu
def test_node_threading_through_the_shim(tmp_path):
    """the node's three threads (Process_points outside MapMutex_, ElevationMapping.cpp:271-282) through the unmodified
    shim: no failures, sane map"""
    exe = compile_with_shim(tmp_path, "threads_shim", ["-pthread"])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    print(r.stdout, r.stderr[-2000:])
    assert r.returncode == 0 and "failures=0" in r.stdout, r.stdout + r.stderr[-2000:]
    assert "failed" not in r.stderr


def test_facade_and_shim_compile_and_link(tmp_path):
    exe = compile_with_shim(tmp_path, "facade_smoke")
    assert os.path.exists(exe)
    out = subprocess.run(["nm", "-C", "--defined-only", exe], capture_output=True, text=True).stdout
    for sym in ("Init_GPU_elevationmap(int, float, float, float)", "Raytracing(int)", "Map_closeloop(float*, float, int, float)",
                "Mapvar_update(int, float)", "Map_optmove(float*, float, float, int, float*)"):
        assert sym in out, sym


@pytest.mark.gpu
def test_facade_and_shim_run_and_agree(tmp_path):
    exe = compile_with_shim(tmp_path, "facade_smoke")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    print(r.stdout, r.stderr)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "mismatches=0" in r.stdout
