"""CPU-side checks of the ray queries against the drawn LOD cut (include/vxb200.h "ray queries against the drawn LOD cut"):
the vxb_cut_hit mirror against a C compiler's layout, the bindings, and the numpy oracle (tests/raycast_cut_oracle.py) on
hand-built meshes - the position rule of the vertex shader, transition meshes, the tie rule - and, at lod_factor 1e30, its
equality with the level-0 oracle on the CPU restatement's sphere."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import raycast_cut_oracle as oracle
import raycast_oracle
from voxels_b200 import capi

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32

# A 64^3 grid of three levels.  With the camera at (100, 16, 16) and lod_factor 2 the top node refines (36 voxels from its
# box, lim 128), the level-1 node (1, 0, 0) (x in [32, 64]) refines (36 < 64) and the level-1 node (0, 0, 0) does not (68):
# it is on the cut with block_adj = bit 5 (grid x+, TransitionFaceId order).
N, LEVELS, CAMERA, FACTOR = 64, 3, (100.0, 16.0, 16.0), 2.0
ADJ = 1 << 5
FLAT = dict(pos=[(2, 10, 2), (30, 10, 2), (2, 10, 30)], idx=[0, 1, 2])


def _moved(mask):
    """A horizontal triangle at y = 10 whose secondary positions lie at y = 20, every vertex with `mask`."""
    return dict(pos=[(2, 10, 2), (30, 10, 2), (2, 10, 30)], sec=[(2, 20, 2), (30, 20, 2), (2, 20, 30)], mask=[mask] * 3, idx=[0, 1, 2])


def _down(t_min=0.0, t_max=np.inf):
    return capi.make_rays([(6, 30, 6)], [(0, -1, 0)], t_min, t_max)


def test_cut_hit_mirror_matches_the_header(tmp_path):
    gcc = shutil.which("gcc")
    if not gcc:
        pytest.skip("no gcc")
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "vxb200.h"', 'int main(void)', '{',
             '\tprintf("hit %zu\\n", sizeof(vxb_cut_hit));']
    lines += ['\tprintf("hit.%s %%zu\\n", offsetof(vxb_cut_hit, %s));' % (f, f) for f in capi.CUT_HIT_DTYPE.names]
    lines += ['\treturn 0;', '}']
    src = tmp_path / "cut.c"
    src.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "cut"
    out = subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(REPO, "include"), str(src), "-o", str(exe)],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    got = dict(line.split() for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got["hit"]) == capi.CUT_HIT_DTYPE.itemsize == 56
    for f in capi.CUT_HIT_DTYPE.names:
        assert int(got["hit." + f]) == capi.CUT_HIT_DTYPE.fields[f][1], f
    assert capi.CUT_HIT_DTYPE.descr[:len(capi.RAY_HIT_DTYPE.descr)] == capi.RAY_HIT_DTYPE.descr


def test_raycast_cut_is_bound():
    assert {"vxb_mesh_raycast_cut", "vxb_mesh_raycast_cut_device"} <= set(capi.EXPORTED_SYMBOLS)
    assert all(hasattr(capi.Mesh, a) for a in ("raycast_cut", "raycast_cut_rc", "raycast_cut_device"))


def test_the_hand_built_cut():
    res = oracle.result_from_blocks(N, LEVELS, [(1, (0, 0, 0), FLAT, {})])
    d = oracle.Drawn(res, CAMERA, FACTOR)
    assert d.selected.tolist() == [True] and d.adj.tolist() == [ADJ]


def test_secondary_position_when_the_mask_is_covered():
    covered = oracle.result_from_blocks(N, LEVELS, [(1, (0, 0, 0), _moved(ADJ), {})])
    uncovered = oracle.result_from_blocks(N, LEVELS, [(1, (0, 0, 0), _moved(ADJ | 1), {})])   # face 0 is not in block_adj
    # drawn at y = 20: t = 10 from y = 30; reached with t_max = 15 only when the mask is covered
    h = oracle.raycast_cut(covered, CAMERA, FACTOR, _down(t_max=15.0))
    assert h["slot"][0] == 0 and h["t"][0] == 10.0 and h["position"][0][1] == 20.0
    assert h["level"][0] == 1 and h["face"][0] == oracle.REGULAR and h["block_id"][0] == 1000
    assert oracle.raycast_cut(uncovered, CAMERA, FACTOR, _down(t_max=15.0))["slot"][0] == capi.VXB_RAY_MISS
    # drawn at y = 10: t = 20, past t_min = 15 only when the mask is not covered
    h = oracle.raycast_cut(uncovered, CAMERA, FACTOR, _down(t_min=15.0))
    assert h["slot"][0] == 0 and h["t"][0] == 20.0
    assert oracle.raycast_cut(covered, CAMERA, FACTOR, _down(t_min=15.0))["slot"][0] == capi.VXB_RAY_MISS
    # a zero mask keeps pos
    zero = oracle.result_from_blocks(N, LEVELS, [(1, (0, 0, 0), _moved(0), {})])
    assert oracle.raycast_cut(zero, CAMERA, FACTOR, _down())["t"][0] == 20.0


def test_transition_triangles_of_block_adj_faces_only():
    wall = lambda x: dict(pos=[(x, 2, 2), (x, 30, 2), (x, 2, 30)], idx=[0, 1, 2])   # noqa: E731
    res = oracle.result_from_blocks(N, LEVELS, [(1, (0, 0, 0), FLAT, {0: wall(25.0), 5: wall(31.0)})])
    ray = capi.make_rays([(20, 15, 6)], [(1, 0, 0)])
    h = oracle.raycast_cut(res, CAMERA, FACTOR, ray)
    assert h["slot"][0] == 0 and h["face"][0] == 5 and h["t"][0] == 11.0 and h["triangle"][0] == 0 and h["level"][0] == 1
    # face 0's transition mesh is not drawn; from the other side the face-5 wall is still the first hit
    back = capi.make_rays([(40, 15, 6)], [(-1, 0, 0)])
    assert oracle.raycast_cut(res, CAMERA, FACTOR, back)["t"][0] == 9.0


def test_ties_go_to_slot_then_part_then_triangle():
    two = dict(pos=FLAT["pos"], idx=[0, 1, 2, 0, 1, 2])
    # the same triangle twice in one part: the lower triangle
    res = oracle.result_from_blocks(N, LEVELS, [(1, (0, 0, 0), two, {})])
    h = oracle.raycast_cut(res, CAMERA, FACTOR, _down())
    assert h["triangle"][0] == 0 and h["face"][0] == oracle.REGULAR
    # in the regular mesh and in transition face 5: the regular mesh; in faces 5 only, triangle 1 of face 5 loses to 0
    res = oracle.result_from_blocks(N, LEVELS, [(1, (0, 0, 0), dict(pos=[(0, 0, 0)] * 3, idx=[0, 1, 2]), {5: two})])
    h = oracle.raycast_cut(res, CAMERA, FACTOR, _down())
    assert h["face"][0] == 5 and h["triangle"][0] == 0
    res = oracle.result_from_blocks(N, LEVELS, [(1, (0, 0, 0), FLAT, {5: two})])
    h = oracle.raycast_cut(res, CAMERA, FACTOR, _down())
    assert h["face"][0] == oracle.REGULAR and h["triangle"][0] == 0
    # two cut nodes holding the same triangle (level-1 node (0, 1, 0) is on the cut as well): the lower slot
    res = oracle.result_from_blocks(N, LEVELS, [(1, (0, 1, 0), dict(pos=[(0, 0, 0)] * 3, idx=[0, 1, 2]), {}), (1, (0, 0, 0), FLAT, {}),
                                                 (1, (0, 1, 0), FLAT, {})])
    d = oracle.Drawn(res, CAMERA, FACTOR)
    assert d.selected.tolist() == [True, True, True]
    h = oracle.raycast_cut(res, CAMERA, FACTOR, _down())
    assert h["slot"][0] == 1 and h["block_id"][0] == 1001
    # a level-0 block under the refining node (1, 0, 0) is on the cut too, and a nearer hit there wins
    near = dict(pos=[(2, 12, 2), (30, 12, 2), (2, 12, 30)], idx=[0, 1, 2])
    res = oracle.result_from_blocks(N, LEVELS, [(0, (2, 0, 0), near, {}), (1, (0, 0, 0), FLAT, {})])
    h = oracle.raycast_cut(res, CAMERA, FACTOR, _down())
    assert h["slot"][0] == 0 and h["level"][0] == 0 and h["t"][0] == 18.0


def _restated_sphere_with_levels(restatement):
    """The restatement's level-0 sphere (n = 64), plus level-1 and level-2 records whose triangles cross it."""
    import grids
    dist, mat, blend = grids.sphere(64)
    h = restatement.run(dist, mat, blend)
    try:
        lv = restatement.level(h, 0)
        blocks = []
        for k in range(len(lv.rows)):
            row, verts, idx, _, _ = lv.block(k)
            x, y, z = int(row["min"][0]) // 16, int(row["min"][2]) // 16, int(row["min"][1]) // 16   # grid (x, y, z)
            blocks.append((0, (x, y, z), dict(pos=verts["pos"], nrm=verts["nrm"], idx=idx), {}))
    finally:
        restatement.destroy(h)
    slab = dict(pos=[(0, 32, 0), (64, 32, 0), (0, 32, 64), (64, 32, 64)], sec=[(0, 30, 0), (64, 30, 0), (0, 30, 64), (64, 30, 64)],
                mask=[1] * 4, idx=[0, 1, 2, 1, 3, 2])
    blocks += [(1, (1, 1, 0), slab, {0: slab}), (2, (0, 0, 0), slab, {3: slab})]
    return oracle.result_from_blocks(64, 3, blocks)


def test_factor_1e30_equals_the_level0_oracle(restatement):
    res = _restated_sphere_with_levels(restatement)
    rng = np.random.RandomState(30)
    c = np.full(3, 32.0)
    dirs = rng.normal(size=(256, 3))
    rays = np.concatenate([capi.make_rays(c + dirs / np.linalg.norm(dirs, axis=1, keepdims=True) * 30, -dirs),
                           capi.make_rays(rng.uniform(-8, 72, (128, 3)), rng.normal(size=(128, 3)))])
    d = oracle.Drawn(res, (5.0, 70.0, 9.0), 1e30)
    assert set(np.asarray(d.slot)) == set(np.nonzero(res.records["level"] == 0)[0].tolist()) and set(d.part) == {0}
    got = oracle.raycast_cut(res, (5.0, 70.0, 9.0), 1e30, rays, d)
    want = raycast_oracle.raycast(res, rays)
    assert (got["slot"] != capi.VXB_RAY_MISS).sum() > 200
    a = got.view(np.uint8).reshape(len(got), -1)[:, :48]
    assert np.array_equal(a, want.view(np.uint8).reshape(len(want), -1))
    hit = got["slot"] != capi.VXB_RAY_MISS
    assert (got["level"][hit] == 0).all() and (got["face"][hit] == oracle.REGULAR).all()
    assert (got["level"][~hit] == 0).all() and (got["face"][~hit] == 0).all()
    # at lod_factor 2 from above the level-2 record is drawn and moves the first hits of rays from above
    top = capi.make_rays(rng.uniform(4, 60, (64, 3)) * (1, 0, 1) + (0, 100, 0), np.tile((0.0, -1.0, 0.0), (64, 1)))
    far = oracle.raycast_cut(res, (32.0, 300.0, 32.0), 2.0, top)
    assert (far["level"] == 2).all() and (far["position"][:, 1] == 32.0).all()
