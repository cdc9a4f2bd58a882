"""CPU-side checks of the collision queries (include/vxb200.h "collision queries"): the numpy mirrors of vxb_sphere_hit and
vxb_closest_hit against a C compiler's layout, the bindings, and the float32 oracle (tests/collide_oracle.py) against its
independent float64 reference on hand-built meshes: every Voronoi region of the closest point, sweeps that first touch the
face, each edge and each vertex, starts in contact, tangent grazes, motion parallel to the plane, zero-area triangles,
signed-zero directions and the tie rules."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import collide_oracle as oracle
import raycast_oracle
from voxels_b200 import capi

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32
TOL = 1e-4    # float32 formulas on coordinates below 32 voxels against float64: a few ulps of 32, with room


def test_collision_mirrors_match_the_header(tmp_path):
    gcc = shutil.which("gcc")
    if not gcc:
        pytest.skip("no gcc")
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "vxb200.h"', 'int main(void)', '{',
             '\tprintf("sphere %zu\\n", sizeof(vxb_sphere_hit));', '\tprintf("closest %zu\\n", sizeof(vxb_closest_hit));',
             '\tprintf("started %u\\n", (unsigned)VXB_SPHERE_STARTED_IN_CONTACT);',
             '\tprintf("rmax %.9g\\n", (double)VXB_SPHERE_RADIUS_MAX);']
    lines += ['\tprintf("sphere.%s %%zu\\n", offsetof(vxb_sphere_hit, %s));' % (f, f) for f in capi.SPHERE_HIT_DTYPE.names]
    lines += ['\tprintf("closest.%s %%zu\\n", offsetof(vxb_closest_hit, %s));' % (f, f) for f in capi.CLOSEST_HIT_DTYPE.names]
    lines += ['\treturn 0;', '}']
    src = tmp_path / "collide.c"
    src.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "collide"
    out = subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(REPO, "include"), str(src), "-o", str(exe)],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    got = dict(line.split() for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got["sphere"]) == capi.SPHERE_HIT_DTYPE.itemsize == 64
    assert int(got["closest"]) == capi.CLOSEST_HIT_DTYPE.itemsize == 48
    assert int(got["started"]) == capi.VXB_SPHERE_STARTED_IN_CONTACT
    assert float(got["rmax"]) == capi.VXB_SPHERE_RADIUS_MAX == 15.0
    for f in capi.SPHERE_HIT_DTYPE.names:
        assert int(got["sphere." + f]) == capi.SPHERE_HIT_DTYPE.fields[f][1], f
    for f in capi.CLOSEST_HIT_DTYPE.names:
        assert int(got["closest." + f]) == capi.CLOSEST_HIT_DTYPE.fields[f][1], f


def test_collision_queries_are_bound():
    names = {"vxb_mesh_sphere_cast", "vxb_mesh_sphere_cast_device", "vxb_mesh_closest_point", "vxb_mesh_closest_point_device"}
    assert names <= set(capi.EXPORTED_SYMBOLS)
    for m in ("sphere_cast", "sphere_cast_device", "sphere_cast_rc", "closest_points", "closest_points_device", "closest_points_rc"):
        assert hasattr(capi.Mesh, m), m


UP = np.array([0, 1, 0], np.float32)
TRI = [(1, 2, 1), (9, 2, 1), (1, 2, 9)]    # a = p0, b = p1, c = p2 in the plane y = 2


def _single(pos, ind=(0, 1, 2), block=(0, 0, 0)):
    pos = np.asarray(pos, np.float32)
    return (block, pos, np.tile(UP, (len(pos), 1)), np.asarray(ind, np.uint32))


def _mesh(*blocks):
    return raycast_oracle.result_from_blocks(32, list(blocks))


def _tris(res):
    lv = raycast_oracle.Level0(res)
    return np.concatenate(lv.tri_pos)


@pytest.mark.parametrize("region,p,want", [
    ("A", (0, 3, 0), (1, 2, 1)), ("B", (10, 3, 0), (9, 2, 1)), ("AB", (5, 3, 0), (5, 2, 1)), ("C", (0, 3, 10), (1, 2, 9)),
    ("AC", (0, 3, 5), (1, 2, 5)), ("BC", (6, 3, 6), (5, 2, 5)), ("face", (3, 5, 3), (3, 2, 3))])
def test_closest_point_regions_agree_with_float64(region, p, want):
    tri = np.asarray([TRI], np.float32)
    q, u, v, reg = oracle.closest_on_triangles(np.asarray(p, np.float32), tri)
    assert oracle.REGIONS[int(reg[0])] == region
    assert np.allclose(q[0], want, atol=TOL)
    # the barycentrics give the point back
    a, b, c = tri[0].astype(np.float64)
    assert np.allclose((1 - u[0] - v[0]) * a + u[0] * b + v[0] * c, q[0], atol=TOL)
    d64 = oracle.point_triangle_dist64(np.asarray(p, np.float64), tri)[0]
    res = _mesh(_single(TRI))
    h = oracle.closest_points(res, [p], 15.0)
    assert h["slot"][0] == 0 and h["block_id"][0] == 1000 and h["triangle"][0] == 0
    assert abs(float(h["distance"][0]) - d64) < TOL
    assert h["distance"][0] == np.sqrt(oracle.dist2(np.asarray(p, np.float32), q[0]))
    assert np.array_equal(h["normal"][0], UP)


def test_closest_point_bound_is_inclusive_and_misses_are_zero():
    res = _mesh(_single(TRI))
    p = [(1, 5, 1)]                                          # exactly 3 from the vertex a
    assert oracle.closest_points(res, p, 3.0)["slot"][0] == 0
    assert oracle.closest_points(res, p, float(np.nextafter(F(3), F(0))))["slot"][0] == capi.VXB_RAY_MISS
    on = oracle.closest_points(res, [(3, 2, 3)], 0.0)        # max_distance 0: a point on the surface
    assert on["slot"][0] == 0 and on["distance"][0] == 0
    miss = oracle.closest_points(res, [(3, 12, 3), (np.nan, 2, 3)], 2.0)
    assert (miss["slot"] == capi.VXB_RAY_MISS).all() and np.isinf(miss["distance"]).all()
    m = miss.copy(); m["distance"] = 0; m["slot"] = 0
    assert not m.view(np.uint8).any()


def _check_sweep(res, o, d, r, t_min=0.0, t_max=np.inf, expect=None):
    """The oracle's sweep against the float64 reference: the same first contact (within TOL along the path), the contact at
    distance r, no triangle closer than r - TOL before it; returns the hit."""
    rays = capi.make_rays([o], [d], t_min, t_max)
    h = oracle.sphere_cast(res, r, rays)[0]
    tris = _tris(res)
    bounds = oracle.segment_bounds64(res.n, o, d, t_min, t_max, r + 1.0)
    assert bounds is not None
    first, _ = oracle.sweep_first_contact64(o, d, bounds[0], bounds[1], r, tris)
    speed = float(np.linalg.norm(np.asarray(d, np.float64)))
    if not np.isfinite(first.min()):
        assert h["slot"] == capi.VXB_RAY_MISS, h
        return h
    assert h["slot"] != capi.VXB_RAY_MISS, (o, d, r, first.min())
    assert abs(float(h["t"]) - first.min()) * speed < TOL * 10, (h["t"], first.min())
    tri = tris[h["triangle"]] if len(res.records) == 1 else None
    if tri is not None and not (h["flags"] & capi.VXB_SPHERE_STARTED_IN_CONTACT):
        assert abs(oracle.point_triangle_dist64(h["center"], tri[None])[0] - r) < TOL
    # the contact point is the closest point of the triangle to the centre, at distance <= r
    assert np.linalg.norm(h["center"].astype(np.float64) - h["point"]) <= r + TOL
    if expect is not None:
        assert np.allclose(h["point"], expect, atol=TOL), (h["point"], expect)
    return h


def test_sweep_face_edges_and_vertices_agree_with_float64():
    res = _mesh(_single(TRI))
    # the face: straight down onto the interior
    h = _check_sweep(res, (3, 10, 3), (0, -1, 0), 1.0, expect=(3, 2, 3))
    assert h["t"] == F(7) and h["flags"] == 0 and np.array_equal(h["center"], np.array([3, 3, 3], np.float32))
    assert np.array_equal(h["normal"], UP)
    # each edge's interior, from outside and above its line
    _check_sweep(res, (5, 3, -5), (0, 0, 1), 1.5, expect=(5, 2, 1))            # ab
    _check_sweep(res, (9, 3, 9), (-1, 0, -1), 1.5, expect=(5, 2, 5))           # bc
    _check_sweep(res, (-5, 3, 5), (1, 0, 0), 1.5, expect=(1, 2, 5))            # ca
    # each vertex, approached from its Voronoi region
    _check_sweep(res, (-5, 2.5, -5), (1, 0, 1), 1.0, expect=(1, 2, 1))         # a
    _check_sweep(res, (15, 2.5, -5), (-1, 0, 1), 1.0, expect=(9, 2, 1))        # b
    _check_sweep(res, (-5, 2.5, 15), (1, 0, -1), 1.0, expect=(1, 2, 9))        # c
    # misses: passing by farther than r, and moving away
    _check_sweep(res, (3, 10, 3), (1, 0, 0), 2.0)
    _check_sweep(res, (3, 4, 3), (0, 1, 0), 1.0)
    # an unnormalised direction: t in units of it
    h = _check_sweep(res, (3, 10, 3), (0, -0.001, 0), 1.0)
    assert abs(float(h["t"]) - 7000) < 1e-2


def test_sweep_started_in_contact():
    res = _mesh(_single(TRI))
    h = _check_sweep(res, (3, 2.5, 3), (0, 1, 0), 1.0)
    assert h["t"] == 0 and h["flags"] == capi.VXB_SPHERE_STARTED_IN_CONTACT
    assert np.array_equal(h["point"], np.array([3, 2, 3], np.float32))
    # t_min moves the start: in contact at t_min = -5 even though the path's t = 0 is above
    h = oracle.sphere_cast(res, 1.0, capi.make_rays([(3, 7.5, 3)], [(0, 1, 0)], -5.0))[0]
    assert h["t"] == F(-5) and h["flags"] == capi.VXB_SPHERE_STARTED_IN_CONTACT


def test_sweep_tangent_graze_and_motion_parallel_to_the_plane():
    res = _mesh(_single(TRI))
    # the path stays at distance exactly r above the plane: first contact where it reaches the edge x = 1
    h = _check_sweep(res, (-5, 3, 3), (1, 0, 0), 1.0)
    assert h["slot"] == 0 and h["t"] == F(6)
    # in the plane's slab (0.5 above it), parallel to it
    h = _check_sweep(res, (-5, 2.5, 3), (1, 0, 0), 1.0)
    assert abs(float(h["t"]) - (6 - np.sqrt(0.75))) < TOL
    # in the plane itself
    _check_sweep(res, (5, 2, -5), (0, 0, 1), 1.0, expect=(5, 2, 1))


def test_zero_area_triangle():
    line = [(1, 2, 1), (5, 2, 1), (9, 2, 1)]
    res = _mesh(_single(line))
    q, u, v, reg = oracle.closest_on_triangles(np.array([5, 4, 1], np.float32), np.asarray([line], np.float32))
    assert np.allclose(q[0], (5, 2, 1), atol=TOL)
    assert abs(float(oracle.closest_points(res, [(5, 4, 1)], 5.0)["distance"][0]) - 2.0) < TOL
    _check_sweep(res, (5, 10, 1), (0, -1, 0), 1.0, expect=(5, 2, 1))
    point = [(4, 2, 4)] * 3
    res = _mesh(_single(point))
    assert oracle.closest_points(res, [(4, 5, 4)], 5.0)["distance"][0] == F(3)
    h = _check_sweep(res, (4, 10, 4), (0, -1, 0), 1.0, expect=(4, 2, 4))
    assert h["t"] == F(7)


def test_signed_zero_direction_components_give_the_same_hit():
    res = _mesh(_single(TRI))
    o = [(3, 10, 3)] * 4
    d = [(0.0, -1, 0.0), (-0.0, -1, 0.0), (0.0, -1, -0.0), (-0.0, -1, -0.0)]
    h = oracle.sphere_cast(res, 1.0, capi.make_rays(o, d))
    assert (h["t"] == F(7)).all()
    assert len(oracle.same(h[1:], np.repeat(h[:1], 3))) == 0


QUAD = [(0, 4, 0), (8, 4, 0), (0, 4, 8), (8, 4, 8)]


def test_shared_edge_ties_go_to_the_lower_slot_then_the_lower_triangle():
    b0 = _single(QUAD[:3], (0, 1, 2))
    b1 = _single(QUAD, (1, 3, 2, 1, 2, 0))        # the same plane; its triangle 0 shares the edge x + z = 8 with b0's
    rays = capi.make_rays([(4, -5, 4)], [(0, 1, 0)])   # up into the shared edge's midpoint: the face test of both at t = 8
    for blocks in ([b0, b1], [b1, b0]):
        res = _mesh(*blocks)
        lv = raycast_oracle.Level0(res)
        ts = [oracle.sweep_triangles((4, -5, 4), (0, 1, 0), 0, np.inf, 1.0, p)[0] for p in lv.tri_pos]
        assert all((t[:1] == F(8)).all() for t in ts)
        h = oracle.sphere_cast(res, 1.0, rays)[0]
        assert h["slot"] == 0 and h["triangle"] == 0 and h["t"] == F(8)
        c = oracle.closest_points(res, [(4, 5, 4)], 2.0)[0]
        assert c["slot"] == 0 and c["triangle"] == 0 and c["distance"] == F(1)


def test_shared_vertex_ties_across_two_slots():
    t0 = _single([(0, 4, 0), (8, 4, 0), (0, 4, 8)])
    t1 = _single([(8, 4, 0), (16, 4, 4), (12, 4, 8)])
    o, d = (8, 4.5, -6), (0, 0, 1)                     # towards the shared vertex (8, 4, 0), from outside both triangles
    for first, second in ((t0, t1), (t1, t0)):
        res = _mesh(first, second)
        lv = raycast_oracle.Level0(res)
        ts = [oracle.sweep_triangles(o, d, 0, np.inf, 1.0, p)[0][0] for p in lv.tri_pos]
        assert ts[0] == ts[1] and np.isfinite(ts[0])
        h = _check_sweep(res, o, d, 1.0, expect=(8, 4, 0))
        assert h["slot"] == 0
        assert np.array_equal(h["point"], np.array([8, 4, 0], np.float32))
        c = oracle.closest_points(res, [(8, 4, -1)], 2.0)[0]
        assert c["slot"] == 0 and c["distance"] == F(1)


def test_oracle_invalid_sweeps_are_misses():
    res = _mesh(_single(TRI))
    rays = capi.make_rays([(3, 10, 3)] * 4, [(0, -1, 0), (0, 0, 0), (np.nan, -1, 0), (0, -1, 0)],
                          t_min=[0, 0, 0, 5], t_max=[np.inf, np.inf, np.inf, 4])
    h = oracle.sphere_cast(res, 1.0, rays)
    assert h["slot"][0] == 0 and (h["slot"][1:] == capi.VXB_RAY_MISS).all() and np.isinf(h["t"][1:]).all()


def test_random_points_and_sweeps_agree_with_float64():
    """Random triangles in one block: the oracle's closest distance equals the float64 minimum, and its first contact the
    float64 one, within TOL."""
    rng = np.random.RandomState(3)
    pos = rng.uniform(0, 16, (24, 3)).astype(np.float32)
    res = _mesh(_single(pos, np.arange(24)))
    tris = _tris(res)
    pts = rng.uniform(-4, 20, (64, 3)).astype(np.float32)
    h = oracle.closest_points(res, pts, 15.0)
    for p, x in zip(pts, h):
        d64 = oracle.point_triangle_dist64(p, tris).min()
        if d64 <= 15.0 - TOL:
            assert abs(float(x["distance"]) - d64) < TOL
    for k in range(32):
        o = rng.uniform(-8, 24, 3)
        d = rng.normal(size=3)
        r = float(rng.choice([0.25, 1.0, 3.0]))
        bounds = oracle.segment_bounds64(res.n, o, d, 0.0, np.inf, r + 1.0)
        if bounds is None:
            continue
        first, dmin = oracle.sweep_first_contact64(o, d, bounds[0], bounds[1], r, tris)
        if np.isfinite(first.min()) and np.sort(dmin)[0] > r - 1e-3:
            continue                                  # a near-tangent graze: the answer hangs on rounding
        _check_sweep(res, o, d, r)
