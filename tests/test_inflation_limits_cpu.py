"""The table bound of gem_costmap_inflate (GEM_INFLATE_MAX_CELLS, DESIGN.md f14) in the ctypes module against the C
compiler's view of the header."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_table_bound_matches_the_header(tmp_path):
    import gem_b200._lib as L
    src = tmp_path / "bound.c"
    src.write_text('#include <stdio.h>\n#include "gem_b200.h"\n'
                   'int main(void) { printf("%d\\n", (int)GEM_INFLATE_MAX_CELLS); return 0; }\n')
    exe = tmp_path / "bound"
    subprocess.run(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], check=True)
    assert int(subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout) == L.INFLATE_MAX_CELLS
