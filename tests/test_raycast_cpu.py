"""CPU-side checks of the ray queries (include/vxb200.h "ray queries"): the ctypes / numpy mirrors of vxb_ray and vxb_ray_hit
against a C compiler's layout, the bindings, and the numpy oracle (tests/raycast_oracle.py) on hand-built meshes and on the
CPU restatement's level-0 mesh of a sphere."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import raycast_oracle as oracle
from voxels_b200 import capi

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32


def test_ray_mirrors_match_the_header(tmp_path):
    gcc = shutil.which("gcc")
    if not gcc:
        pytest.skip("no gcc")
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "vxb200.h"', 'int main(void)', '{',
             '\tprintf("ray %zu\\n", sizeof(vxb_ray));', '\tprintf("hit %zu\\n", sizeof(vxb_ray_hit));',
             '\tprintf("miss %u\\n", (unsigned)VXB_RAY_MISS);']
    lines += ['\tprintf("ray.%s %%zu\\n", offsetof(vxb_ray, %s));' % (f, f) for f in capi.RAY_DTYPE.names]
    lines += ['\tprintf("hit.%s %%zu\\n", offsetof(vxb_ray_hit, %s));' % (f, f) for f in capi.RAY_HIT_DTYPE.names]
    lines += ['\treturn 0;', '}']
    src = tmp_path / "ray.c"
    src.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "ray"
    out = subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(REPO, "include"), str(src), "-o", str(exe)],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    got = dict(line.split() for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got["ray"]) == capi.RAY_DTYPE.itemsize == 32
    assert int(got["hit"]) == capi.RAY_HIT_DTYPE.itemsize == 48
    assert int(got["miss"]) == capi.VXB_RAY_MISS
    for f in capi.RAY_DTYPE.names:
        assert int(got["ray." + f]) == capi.RAY_DTYPE.fields[f][1], f
    for f in capi.RAY_HIT_DTYPE.names:
        assert int(got["hit." + f]) == capi.RAY_HIT_DTYPE.fields[f][1], f


def test_raycast_is_bound():
    assert {"vxb_mesh_raycast", "vxb_mesh_raycast_device"} <= set(capi.EXPORTED_SYMBOLS)
    assert hasattr(capi.Mesh, "raycast") and hasattr(capi.Mesh, "raycast_device")


UP = np.array([0, 1, 0], np.float32)


def _single(pos, ind=(0, 1, 2), block=(0, 0, 0), nrm=None):
    pos = np.asarray(pos, np.float32)
    nrm = np.tile(UP, (len(pos), 1)) if nrm is None else np.asarray(nrm, np.float32)
    return (block, pos, nrm, np.asarray(ind, np.uint32))


def test_oracle_single_triangle():
    res = oracle.result_from_blocks(32, [_single([(1, 2, 1), (9, 2, 1), (1, 2, 9)])])
    rays = capi.make_rays([(3, 10, 3), (3, -5, 3), (8.5, 10, 8.5)], [(0, -1, 0), (0, 2, 0), (0, -1, 0)])
    h = oracle.raycast(res, rays)
    assert h["slot"][0] == 0 and h["t"][0] == F(8) and h["triangle"][0] == 0 and h["block_id"][0] == 1000
    assert np.array_equal(h["position"][0], np.array([3, 2, 3], np.float32))
    assert h["u"][0] == F(0.25) and h["v"][0] == F(0.25)
    assert np.array_equal(h["normal"][0], UP)
    # from below: both faces are hit; t in units of the (length 2) direction
    assert h["slot"][1] == 0 and h["t"][1] == F(3.5)
    # outside the hypotenuse: a miss with t = +inf and zeros everywhere else
    assert h["slot"][2] == capi.VXB_RAY_MISS and np.isinf(h["t"][2])
    miss = h[2:3].copy(); miss["t"] = 0; miss["slot"] = 0
    assert not miss.view(np.uint8).any()


def test_oracle_shared_edge_ties_go_to_lower_slot_then_lower_triangle():
    quad = [(0, 4, 0), (8, 4, 0), (0, 4, 8), (8, 4, 8)]
    # two blocks whose triangles share the edge x + z = 8 (the second block holds the same plane, listed first in its indices)
    b0 = _single(quad[:3], (0, 1, 2), (0, 0, 0))
    b1 = _single(quad, (1, 3, 2, 1, 2, 0), (0, 0, 0))
    res = oracle.result_from_blocks(32, [b0, b1])
    rays = capi.make_rays([(4, 9, 4)], [(0, -1, 0)])
    h = oracle.raycast(res, rays)
    assert h["slot"][0] == 0 and h["triangle"][0] == 0 and h["t"][0] == F(5)
    # the same pair in the other slot order: the triangle of the lower slot (now the quad's) wins, and within it the lower k
    res = oracle.result_from_blocks(32, [b1, b0])
    h = oracle.raycast(res, rays)
    assert h["slot"][0] == 0 and h["triangle"][0] == 0 and h["t"][0] == F(5)


def test_oracle_parallel_ray_misses():
    res = oracle.result_from_blocks(32, [_single([(1, 2, 1), (9, 2, 1), (1, 2, 9)])])
    h = oracle.raycast(res, capi.make_rays([(0, 2, 2), (0, 2.5, 2)], [(1, 0, 0), (1, 0, 0.25)]))
    assert (h["slot"] == capi.VXB_RAY_MISS).all()


def test_oracle_t_min_and_t_max_are_inclusive():
    res = oracle.result_from_blocks(32, [_single([(1, 2, 1), (9, 2, 1), (1, 2, 9)])])
    o, d = [(3, 10, 3)], [(0, -1, 0)]
    for t_min, t_max, hit in [(8, 8, True), (0, 8, True), (8, np.inf, True), (0, np.nextafter(F(8), F(0)), False),
                              (np.nextafter(F(8), F(9)), np.inf, False)]:
        h = oracle.raycast(res, capi.make_rays(o, d, t_min, t_max))
        assert (h["slot"][0] == 0) == hit, (t_min, t_max)
        if hit:
            assert h["t"][0] == F(8)


@pytest.mark.parametrize("scale", [1e-3, 1e3])
def test_oracle_unnormalised_directions(scale):
    res = oracle.result_from_blocks(32, [_single([(1, 2, 1), (9, 2, 1), (1, 2, 9)])])
    d = np.array([0.25, -1.0, 0.5], np.float32) * F(scale)
    h = oracle.raycast(res, capi.make_rays([(2, 10, 2)], [d]))
    assert h["slot"][0] == 0
    assert abs(float(h["t"][0]) * float(np.linalg.norm(d)) - 8 * np.linalg.norm([0.25, 1, 0.5])) < 1e-3
    assert abs(float(h["position"][0][1]) - 2.0) < 1e-4
    # position is o + t * d in float32, exactly
    assert np.array_equal(h["position"][0], np.array([2, 10, 2], np.float32) + h["t"][0] * d)


def test_oracle_invalid_rays_are_misses():
    res = oracle.result_from_blocks(32, [_single([(1, 2, 1), (9, 2, 1), (1, 2, 9)])])
    rays = capi.make_rays([(3, 10, 3)] * 5, [(0, -1, 0), (0, 0, 0), (np.nan, -1, 0), (0, -1, 0), (0, -1, 0)],
                          t_min=[0, 0, 0, np.nan, 5], t_max=[np.inf, np.inf, np.inf, 1, 4])
    h = oracle.raycast(res, rays)
    assert h["slot"][0] == 0 and (h["slot"][1:] == capi.VXB_RAY_MISS).all()


def _restated_level0(restatement, dist, mat, blend):
    """The restatement's level-0 blocks as a capi.Result (slot = the restatement's block order)."""
    h = restatement.run(dist, mat, blend)
    try:
        lv = restatement.level(h, 0)
    finally:
        restatement.destroy(h)
    n = dist.shape[0]
    blocks = []
    for k in range(len(lv.rows)):
        row, verts, idx, _, _ = lv.block(k)
        x, zy = int(row["min"][0]) // 16, (int(row["min"][1]) // 16, int(row["min"][2]) // 16)
        blocks.append(((x, zy[1], zy[0]), verts["pos"], verts["nrm"], idx))
    return oracle.result_from_blocks(n, blocks)


def test_oracle_on_restated_sphere_hits_the_analytic_sphere(restatement):
    import grids
    n = 64
    res = _restated_level0(restatement, *grids.sphere(n))
    c, r = np.full(3, n / 2.0), 0.3 * n
    rng = np.random.RandomState(4)
    dirs = rng.normal(size=(256, 3)); dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    origins = c + dirs * (0.45 * n)
    rays = capi.make_rays(origins, -dirs)
    hits = oracle.raycast(res, rays)
    assert (hits["slot"] != capi.VXB_RAY_MISS).all()
    dist = np.linalg.norm(hits["position"].astype(np.float64) - c, axis=1)
    assert np.abs(dist - r).max() < 1.0, np.abs(dist - r).max()
    # the outward normal of the surface, near the sphere's
    cosine = (hits["normal"].astype(np.float64) * dirs).sum(axis=1)
    assert np.median(np.abs(cosine)) > 0.9
