"""CPU-side checks of the collision queries against the drawn LOD cut (include/vxb200.h "collision queries against the drawn
LOD cut"): the hit mirrors against a C compiler's layout, the bindings, and the numpy oracle (tests/collide_cut_oracle.py) on
hand-built meshes - the position rule of the vertex shader, transition meshes, the tie rule - its equality with the level-0
oracle at lod_factor 1e30, and its geometry against collide_oracle's float64 references."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import collide_cut_oracle as oracle
import collide_oracle
import raycast_cut_oracle
from test_raycast_cut_cpu import ADJ, CAMERA, FACTOR, FLAT, LEVELS, N, _moved, _restated_sphere_with_levels
from voxels_b200 import capi

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32
REGULAR = raycast_cut_oracle.REGULAR


def _down(t_min=0.0, t_max=np.inf):
    return capi.make_rays([(6, 30, 6)], [(0, -1, 0)], t_min, t_max)


def _blocks(*blocks):
    return raycast_cut_oracle.result_from_blocks(N, LEVELS, list(blocks))


def _sweep(res, r, rays=None):
    return oracle.sphere_cast_cut(res, CAMERA, FACTOR, r, _down() if rays is None else rays)


def _point(res, p, md):
    return oracle.closest_points_cut(res, CAMERA, FACTOR, np.array([p], F), md)


def test_hit_mirrors_match_the_header(tmp_path):
    gcc = shutil.which("gcc")
    if not gcc:
        pytest.skip("no gcc")
    structs = {"vxb_sphere_cut_hit": capi.SPHERE_CUT_HIT_DTYPE, "vxb_closest_cut_hit": capi.CLOSEST_CUT_HIT_DTYPE}
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "vxb200.h"', 'int main(void)', '{']
    for s, dt in structs.items():
        lines.append('\tprintf("%s %%zu\\n", sizeof(%s));' % (s, s))
        lines += ['\tprintf("%s.%s %%zu\\n", offsetof(%s, %s));' % (s, f, s, f) for f in dt.names]
    lines += ['\treturn 0;', '}']
    src = tmp_path / "cuthits.c"
    src.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "cuthits"
    out = subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(REPO, "include"), str(src), "-o", str(exe)],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    got = dict(line.split() for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got["vxb_sphere_cut_hit"]) == capi.SPHERE_CUT_HIT_DTYPE.itemsize == 72
    assert int(got["vxb_closest_cut_hit"]) == capi.CLOSEST_CUT_HIT_DTYPE.itemsize == 56
    for s, dt in structs.items():
        for f in dt.names:
            assert int(got[s + "." + f]) == dt.fields[f][1], (s, f)
    assert capi.SPHERE_CUT_HIT_DTYPE.descr[:len(capi.SPHERE_HIT_DTYPE.descr)] == capi.SPHERE_HIT_DTYPE.descr
    assert capi.CLOSEST_CUT_HIT_DTYPE.descr[:len(capi.CLOSEST_HIT_DTYPE.descr)] == capi.CLOSEST_HIT_DTYPE.descr


def test_cut_collision_queries_are_bound():
    names = {"vxb_mesh_sphere_cast_cut", "vxb_mesh_sphere_cast_cut_device", "vxb_mesh_closest_point_cut", "vxb_mesh_closest_point_cut_device"}
    assert names <= set(capi.EXPORTED_SYMBOLS)
    for a in ("sphere_cast_cut", "sphere_cast_cut_rc", "sphere_cast_cut_device", "closest_points_cut", "closest_points_cut_rc",
              "closest_points_cut_device"):
        assert hasattr(capi.Mesh, a), a


def test_secondary_position_when_the_mask_is_covered():
    covered, uncovered = _blocks((1, (0, 0, 0), _moved(ADJ), {})), _blocks((1, (0, 0, 0), _moved(ADJ | 1), {}))
    # drawn at y = 20: the sphere of radius 1 from y = 30 touches at t = 9; drawn at y = 10, at t = 19
    h = _sweep(covered, 1.0)
    assert h["slot"][0] == 0 and h["t"][0] == 9.0 and h["point"][0][1] == 20.0 and h["center"][0][1] == 21.0
    assert h["level"][0] == 1 and h["face"][0] == REGULAR and h["block_id"][0] == 1000 and h["flags"][0] == 0
    assert _sweep(uncovered, 1.0)["t"][0] == 19.0
    zero = _blocks((1, (0, 0, 0), _moved(0), {}))
    assert _sweep(zero, 1.0)["t"][0] == 19.0
    # the point (6, 25, 6) is 5 from the drawn triangle at y = 20 and 15 from the one at y = 10
    h = _point(covered, (6, 25, 6), 10.0)
    assert h["distance"][0] == 5.0 and h["point"][0][1] == 20.0 and h["level"][0] == 1 and h["face"][0] == REGULAR
    assert _point(uncovered, (6, 25, 6), 10.0)["slot"][0] == capi.VXB_RAY_MISS
    assert _point(uncovered, (6, 25, 6), 15.0)["distance"][0] == 15.0
    assert _point(zero, (6, 25, 6), 15.0)["distance"][0] == 15.0


def test_transition_faces_outside_block_adj_are_never_hit():
    wall = lambda x: dict(pos=[(x, 2, 2), (x, 30, 2), (x, 2, 30)], idx=[0, 1, 2])   # noqa: E731
    res = _blocks((1, (0, 0, 0), FLAT, {0: wall(25.0), 5: wall(31.0)}))
    # face 0's wall (x = 25) is not drawn: the sweep passes it and touches face 5's wall (x = 31) at t = 10
    h = _sweep(res, 1.0, capi.make_rays([(20, 15, 6)], [(1, 0, 0)]))
    assert h["slot"][0] == 0 and h["face"][0] == 5 and h["t"][0] == 10.0 and h["triangle"][0] == 0 and h["level"][0] == 1
    # the point (26, 16, 10) is 1 from face 0's wall and 5 from face 5's
    h = _point(res, (26, 16, 10), 6.0)
    assert h["face"][0] == 5 and h["distance"][0] == 5.0
    assert _point(res, (26, 16, 10), 4.0)["slot"][0] == capi.VXB_RAY_MISS


def test_ties_go_to_slot_then_part_then_triangle():
    two = dict(pos=FLAT["pos"], idx=[0, 1, 2, 0, 1, 2])
    dot = dict(pos=[(0, 0, 0)] * 3, idx=[0, 1, 2])
    queries = (lambda res: _sweep(res, 1.0), lambda res: _point(res, (6, 25, 6), 20.0))
    for q in queries:
        # the same triangle twice in one part: the lower triangle
        h = q(_blocks((1, (0, 0, 0), two, {})))
        assert h["triangle"][0] == 0 and h["face"][0] == REGULAR
        # only in face 5 (the regular mesh is a point far away): triangle 0 of face 5
        h = q(_blocks((1, (0, 0, 0), dot, {5: two})))
        assert h["face"][0] == 5 and h["triangle"][0] == 0
        # in the regular mesh and in face 5 at the same t or dd: the regular mesh
        h = q(_blocks((1, (0, 0, 0), FLAT, {5: two})))
        assert h["face"][0] == REGULAR and h["triangle"][0] == 0
        # two cut nodes holding the same triangle: the lower slot
        h = q(_blocks((1, (0, 1, 0), dot, {}), (1, (0, 0, 0), FLAT, {}), (1, (0, 1, 0), FLAT, {})))
        assert h["slot"][0] == 1 and h["block_id"][0] == 1001
    # the tie values themselves
    assert _sweep(_blocks((1, (0, 0, 0), FLAT, {5: two})), 1.0)["t"][0] == 19.0
    assert _point(_blocks((1, (0, 0, 0), FLAT, {5: two})), (6, 25, 6), 20.0)["distance"][0] == 15.0


def _first(h, nbytes):
    return np.ascontiguousarray(h).view(np.uint8).reshape(len(h), -1)[:, :nbytes]


def _sphere_queries(rng):
    c = np.full(3, 32.0)
    dirs = rng.normal(size=(192, 3))
    sweeps = np.concatenate([capi.make_rays(c + dirs / np.linalg.norm(dirs, axis=1, keepdims=True) * 30, -dirs),
                             capi.make_rays(rng.uniform(-8, 72, (96, 3)), rng.normal(size=(96, 3)))])
    pts = np.concatenate([c + dirs[:96] / np.linalg.norm(dirs[:96], axis=1, keepdims=True) * rng.uniform(16, 28, (96, 1)),
                          rng.uniform(-4, 68, (64, 3))]).astype(np.float32)
    return sweeps, pts


def test_factor_1e30_equals_the_level0_oracle(restatement):
    res = _restated_sphere_with_levels(restatement)
    rng = np.random.RandomState(31)
    sweeps, pts = _sphere_queries(rng)
    camera = (5.0, 70.0, 9.0)
    d = raycast_cut_oracle.Drawn(res, camera, 1e30)
    for r in (0.5, 2.0):
        got = oracle.sphere_cast_cut(res, camera, 1e30, r, sweeps, d)
        want = collide_oracle.sphere_cast(res, r, sweeps)
        assert (got["slot"] != capi.VXB_RAY_MISS).sum() > 100
        assert np.array_equal(_first(got, 64), want.view(np.uint8).reshape(len(want), -1))
        hit = got["slot"] != capi.VXB_RAY_MISS
        assert (got["level"] == 0).all() and (got["face"][hit] == REGULAR).all() and (got["face"][~hit] == 0).all()
    for md in (0.0, 2.0, 6.0):
        got = oracle.closest_points_cut(res, camera, 1e30, pts, md, d)
        want = collide_oracle.closest_points(res, pts, md)
        assert np.array_equal(_first(got, 48), want.view(np.uint8).reshape(len(want), -1))
        hit = got["slot"] != capi.VXB_RAY_MISS
        assert (got["level"] == 0).all() and (got["face"][hit] == REGULAR).all() and (got["face"][~hit] == 0).all()
        if md == 6.0:
            assert hit.sum() > 60


def test_geometry_agrees_with_float64(restatement):
    """At lod_factor 2 from above the level-2 slab is drawn (at its secondary height 30 where block_adj covers the mask): every
    sweep contact not started in contact is r from its drawn triangle, no drawn triangle comes closer than r before it, and
    every closest distance is the float64 distance to the drawn set."""
    res = _restated_sphere_with_levels(restatement)
    rng = np.random.RandomState(32)
    sweeps, pts = _sphere_queries(rng)
    camera = (32.0, 300.0, 32.0)
    d = raycast_cut_oracle.Drawn(res, camera, 2.0)
    tris = np.concatenate([p for p in d.tri_pos if len(p)])
    tol = 2e-3
    r = 1.5
    got = oracle.sphere_cast_cut(res, camera, 2.0, r, sweeps, d)
    assert (got["level"][got["slot"] != capi.VXB_RAY_MISS] > 0).any()
    where = {(s, p): b for b, (s, p) in enumerate(zip(d.slot, d.part))}
    for i in rng.choice(len(sweeps), 48, replace=False):
        ray, h = sweeps[i], got[i]
        o, dv = ray["origin"].astype(np.float64), ray["direction"].astype(np.float64)
        if h["slot"] != capi.VXB_RAY_MISS:
            part = 0 if h["face"] == REGULAR else int(h["face"]) + 1
            tri = d.tri_pos[where[(int(h["slot"]), part)]][h["triangle"]]
            dist = collide_oracle.point_triangle_dist64(h["center"], tri[None])[0]
            assert dist <= r + tol if h["flags"] else abs(dist - r) <= tol, (ray, h, dist)
            if h["flags"]:
                continue
        t_hi = float(h["t"]) if h["slot"] != capi.VXB_RAY_MISS else 200.0
        bounds = collide_oracle.segment_bounds64(64, o, dv, float(ray["t_min"]), t_hi, r + 40.0)
        if bounds is None:
            continue
        _, dmin = collide_oracle.sweep_first_contact64(o, dv, bounds[0], bounds[1], r, tris, iters=50)
        assert dmin.min() >= r - tol, (ray, h, dmin.min())
    for md in (2.0, 6.0):
        got = oracle.closest_points_cut(res, camera, 2.0, pts, md, d)
        d64 = np.array([collide_oracle.point_triangle_dist64(p, tris).min() for p in pts])
        hit = got["slot"] != capi.VXB_RAY_MISS
        assert hit.sum() > 10
        assert np.all(np.abs(got["distance"][hit].astype(np.float64) - d64[hit]) <= tol)
        assert np.all(d64[~hit] >= md - tol)
