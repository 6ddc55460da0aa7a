"""The tests' native builds in one place: oracle shared libraries, programs against libgem_b200.so and the C compiler's
view of include/gem_b200.h.  Everything goes into one temporary directory per process (the checkout may be read-only),
removed when the process that made it exits.  TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
INCLUDE = os.path.join(ROOT, "include")
CSRC = os.path.join(ROOT, "gem_b200", "csrc")
CXX = os.path.join(HERE, "cxx")

# the C oracles: no contraction and no fast math, so they compute the arithmetic definition the device is compared with
ORACLE_C = ["-O2", "-std=gnu11", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-Wall", "-Wextra"]
# the library's host headers (gem_footprint.h, gem_gridmsg.h, gem_globalmap.h, ...) under g++, contraction off likewise
HOST_CXX = ["-O2", "-std=c++14", "-fPIC", "-ffp-contract=off", "-Wall", "-Wextra", "-I", CSRC]
# the PointCloud2, PCD and ROS framing code: integer and text formatting, no floating-point multiply-add to contract
FORMAT_C = ["-O2", "-std=gnu11", "-fPIC", "-Wall", "-Wextra"]
FORMAT_CXX = ["-O2", "-std=c++14", "-fPIC", "-Wall", "-Wextra", "-I", CSRC]
# programs written against the C++ facade (include/gem_b200/elevation_map.hpp)
FACADE = ["-O2", "-std=c++14", "-Wall"]

_tmp = None


def _dir() -> str:
    global _tmp
    if _tmp is None:
        _tmp = tempfile.mkdtemp(prefix="gem_tests_")
        owner = os.getpid()       # a forked worker inherits the directory but must not remove it under its parent
        atexit.register(lambda: os.getpid() == owner and shutil.rmtree(_tmp, True))
    return _tmp


def shared_library(name, sources, flags, libs=()):
    """lib<name>.so of the sources (g++ for C++ ones, else gcc), built with the flags and loaded"""
    so = os.path.join(_dir(), f"lib{name}.so")
    cc = "g++" if any(s.endswith(".cpp") for s in sources) else "gcc"
    subprocess.run([cc, *flags, "-shared", "-o", so, *sources, *libs], check=True)
    return C.CDLL(so)


def facade_program(name, out_dir=None, extra_flags=(), libs=(), sources=None, flags=FACADE):
    """tests/cxx/<name>.cpp (or the given sources) linked against libgem_b200.so as out_dir/<name> (by default in this
    process's directory); returns the path"""
    from gem_b200 import build
    libdir = os.path.dirname(build.build())
    exe = os.path.join(str(out_dir or _dir()), name)
    srcs = sources or [os.path.join(CXX, name + ".cpp")]
    subprocess.run(["g++", *flags, "-I", INCLUDE, *extra_flags, "-o", exe, *srcs, "-L", libdir, "-lgem_b200", *libs,
                    "-Wl,-rpath," + libdir], check=True)
    return exe


def facade_compiles(name, syntax_only=False):
    """tests/cxx/<name>.cpp compiles without a warning: to an object file, or with syntax_only=True checked only"""
    src = os.path.join(CXX, name + ".cpp")
    if syntax_only:
        cmd = ["g++", "-std=c++14", "-Wall", "-Werror", "-fsyntax-only", "-I", INCLUDE, src]
    else:
        cmd = ["g++", *FACADE, "-Werror", "-I", INCLUDE, "-c", "-o", os.path.join(_dir(), name + ".o"), src]
    subprocess.run(cmd, check=True)


def c_values(exprs, std="c99"):
    """{expression: value} of integer C expressions (sizeof, offsetof, macros) over gem_b200.h, as a C program built
    with -std=<std> (none when std is None) prints them"""
    exprs = list(exprs)
    d = tempfile.mkdtemp(dir=_dir())
    src, exe = os.path.join(d, "values.c"), os.path.join(d, "values")
    with open(src, "w") as f:
        f.write('#include <stdio.h>\n#include <stddef.h>\n#include "gem_b200.h"\nint main(void) {\n')
        f.writelines(f'  printf("%lld\\n", (long long)({e}));\n' for e in exprs)
        f.write("  return 0;\n}\n")
    subprocess.run(["gcc", *([f"-std={std}"] if std else []), "-I", INCLUDE, "-o", exe, src], check=True)
    out = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()
    assert len(out) == len(exprs), out
    return dict(zip(exprs, map(int, out)))


def assert_struct_layouts(structs, consts=None, std="c99"):
    """the size and every field offset of each ctypes mirror {c_name: class} are the C compiler's, and so is the value
    of each {expression: value} in consts"""
    want = dict(consts or {})
    for cname, cls in structs.items():
        want[f"sizeof({cname})"] = C.sizeof(cls)
        for field, *_ in cls._fields_:
            want[f"offsetof({cname}, {field})"] = getattr(cls, field).offset
    assert c_values(want, std) == want
