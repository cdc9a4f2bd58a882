"""CPU-side checks of the mesh's C ABI (include/vxb200.h "mesh"): the header's new structs compile as plain C and the ctypes
mirrors in voxels_b200/capi.py have the sizes and field offsets a C compiler gives them."""
import ctypes as C
import os
import shutil
import subprocess

import pytest

from voxels_b200 import capi

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

FIELDS = ["levels", "block_count", "level_blocks", "vertex_span", "index_span", "trans_vertex_span", "trans_index_span",
          "vertex_total", "index_total", "trans_vertex_total", "trans_index_total", "capacity", "stats", "compactions", "growths",
          "generation", "bytes_copied", "apply_ms"]


def test_mesh_mirrors_match_the_header(tmp_path):
    gcc = shutil.which("gcc")
    if not gcc:
        pytest.skip("no gcc")
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "vxb200.h"', 'int main(void)', '{',
             '\tvxb_mesh* m = NULL; vxb_mesh_info i; vxb_draw_lists l; (void)m; (void)i; (void)l;',
             '\tprintf("size %zu\\n", sizeof(vxb_mesh_info));',
             '\tprintf("draw_lists %zu\\n", sizeof(vxb_draw_lists));']
    lines += ['\tprintf("%s %%zu\\n", offsetof(vxb_mesh_info, %s));' % (f, f) for f in FIELDS]
    lines += ['\treturn 0;', '}']
    src = tmp_path / "mesh.c"
    src.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "mesh"
    out = subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(REPO, "include"), str(src), "-o", str(exe)],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    got = dict(line.split() for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got["size"]) == C.sizeof(capi.MeshInfo)
    assert int(got["draw_lists"]) == C.sizeof(capi.DrawLists)
    for f in FIELDS:
        assert int(got[f]) == getattr(capi.MeshInfo, f).offset, f


def test_mesh_is_bound():
    names = ["vxb_mesh_create", "vxb_mesh_destroy", "vxb_mesh_apply", "vxb_mesh_info_get", "vxb_mesh_download", "vxb_mesh_device_arenas",
             "vxb_mesh_select_lod"]
    assert set(names) <= set(capi.EXPORTED_SYMBOLS)
