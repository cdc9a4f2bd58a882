"""CPU-side checks of the capsule queries (include/vxb200.h "capsule queries"): the numpy mirrors of vxb_capsule_sweep,
vxb_segment, vxb_capsule_hit and vxb_segment_hit against a C compiler's layout, the bindings, and the float32 oracle
(tests/capsule_oracle.py) against its independent float64 reference on hand-built meshes: a capsule lying on a face, the
cylinder part touching a triangle vertex and edge, the end caps, a segment parallel to an edge, a segment crossing the
triangle, zero-area triangles, h = 0 (the sphere queries bit for bit), h in the triangle's plane, signed zeros, grazes at
exactly r, and the tie rules across a shared edge and a shared vertex."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import capsule_oracle as oracle
import collide_oracle
import raycast_oracle
from voxels_b200 import capi

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32
TOL = 1e-4
UP = np.array([0, 1, 0], np.float32)
TRI = [(1, 2, 1), (9, 2, 1), (1, 2, 9)]    # in the plane y = 2


def test_capsule_mirrors_match_the_header(tmp_path):
    gcc = shutil.which("gcc")
    if not gcc:
        pytest.skip("no gcc")
    structs = {"vxb_capsule_sweep": capi.CAPSULE_SWEEP_DTYPE, "vxb_segment": capi.SEGMENT_DTYPE,
               "vxb_capsule_hit": capi.CAPSULE_HIT_DTYPE, "vxb_segment_hit": capi.SEGMENT_HIT_DTYPE}
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "vxb200.h"', 'int main(void)', '{']
    for name, dt in structs.items():
        lines.append('\tprintf("%s %%zu\\n", sizeof(%s));' % (name, name))
        lines += ['\tprintf("%s.%s %%zu\\n", offsetof(%s, %s));' % (name, f, name, f) for f in dt.names]
    lines += ['\treturn 0;', '}']
    src = tmp_path / "capsule.c"
    src.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "capsule"
    out = subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(REPO, "include"), str(src), "-o", str(exe)],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    got = dict(line.split() for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert [int(got[n]) for n in structs] == [48, 24, 80, 64]
    for name, dt in structs.items():
        assert int(got[name]) == dt.itemsize
        for f in dt.names:
            assert int(got[name + "." + f]) == dt.fields[f][1], (name, f)


def test_capsule_queries_are_bound():
    names = {"vxb_mesh_capsule_cast", "vxb_mesh_capsule_cast_device", "vxb_mesh_closest_to_segment", "vxb_mesh_closest_to_segment_device"}
    assert names <= set(capi.EXPORTED_SYMBOLS)
    for m in ("capsule_cast", "capsule_cast_device", "capsule_cast_rc", "closest_to_segment", "closest_to_segment_device",
              "closest_to_segment_rc"):
        assert hasattr(capi.Mesh, m), m
    s = capi.make_capsule_sweeps([(1, 2, 3)], [(0, -1, 0)], (0, 3, 0), 0.5, 1.0, 9.0)
    assert s["path"]["origin"][0].tolist() == [1, 2, 3] and s["path"]["t_min"][0] == 1 and s["path"]["t_max"][0] == 9
    assert s["half_axis"][0].tolist() == [0, 3, 0] and s["radius"][0] == F(0.5)


def _single(pos, ind=(0, 1, 2), block=(0, 0, 0)):
    pos = np.asarray(pos, np.float32)
    return (block, pos, np.tile(UP, (len(pos), 1)), np.asarray(ind, np.uint32))


def _mesh(*blocks):
    return raycast_oracle.result_from_blocks(32, list(blocks))


def _tris(res):
    return np.concatenate(raycast_oracle.Level0(res).tri_pos)


def _segment(res, c, h, md=None, want_class=None):
    """The oracle's closest-to-segment against float64 (max_distance at the reach limit by default): distance within TOL,
    point and axis point consistent."""
    cls = []
    md = 15.0 - float(np.max(np.abs(np.asarray(h, np.float32)))) if md is None else md
    x = oracle.closest_to_segment(res, capi.make_segments([c], [h]), md, classes=cls)[0]
    d64 = oracle.segment_triangle_dist64(np.asarray(c, np.float64), h, _tris(res)).min()
    assert x["slot"] != capi.VXB_RAY_MISS, (c, h, d64)
    assert abs(float(x["distance"]) - d64) < TOL, (c, h, x["distance"], d64)
    assert np.linalg.norm(x["axis_point"].astype(np.float64) - x["point"]) <= d64 + TOL
    assert -1 <= x["s"] <= 1
    assert np.allclose(x["axis_point"], np.asarray(c, np.float32) + x["s"] * np.asarray(h, np.float32), atol=TOL)
    if want_class is not None:
        assert cls[0] == want_class, (cls[0], want_class)
    return x


def test_closest_pair_classes_agree_with_float64():
    res = _mesh(_single(TRI))
    x = _segment(res, (3, 6, 3), (0, 2, 0), want_class="endpoint")                  # vertical, above the face
    assert x["distance"] == F(2) and x["s"] == F(-1) and np.array_equal(x["point"], np.array([3, 2, 3], np.float32))
    _segment(res, (3, 6, 3), (0, -2, 0), want_class="endpoint")                      # the other end is the near one
    x = _segment(res, (3, 2, 3), (0, 3, 0), want_class="crossing")                   # through the face
    assert x["distance"] == 0 and np.allclose(x["point"], (3, 2, 3)) and abs(float(x["s"])) < TOL
    _segment(res, (5, 4, -3), (0, 0, 1.5), want_class="endpoint")                    # towards edge ab, short
    x = _segment(res, (5, 3, -1), (6, 0, 0.0), want_class="edge")                   # parallel to edge ab, 1 above it
    assert abs(float(x["distance"]) - np.sqrt(5.0)) < TOL
    x = _segment(res, (-2, 2, 5), (0, 3, 0), want_class="edge")                     # skew to edge ca, beside it
    assert abs(float(x["distance"]) - 3.0) < TOL
    _segment(res, (7, 5, 7), (3, -2, -1), want_class=None)                           # oblique
    x = _segment(res, (3, 5, 3), (4, 0, 0))                                          # in a plane parallel to the face
    assert abs(float(x["distance"]) - 3.0) < TOL
    x = _segment(res, (-3, 2, -3), (1, 0, 1))                                        # in the triangle's plane
    assert abs(float(x["distance"]) - np.sqrt(18.0)) < TOL


def test_zero_half_axis_is_the_closest_point_bit_for_bit():
    rng = np.random.RandomState(11)
    pos = rng.uniform(0, 16, (30, 3)).astype(np.float32)
    res = _mesh(_single(pos, np.arange(30)))
    pts = rng.uniform(-4, 20, (64, 3)).astype(np.float32)
    for md in (0.0, 3.0, 15.0):
        seg = oracle.closest_to_segment(res, capi.make_segments(pts, (0, 0, 0)), md)
        pnt = collide_oracle.closest_points(res, pts, md)
        for f in ("distance", "slot", "block_id", "triangle", "point", "normal", "u", "v"):
            assert np.array_equal(seg[f], pnt[f]), (md, f)
        hit = seg["slot"] != capi.VXB_RAY_MISS
        assert np.array_equal(seg["axis_point"][hit], pts[hit]) and (seg["s"][hit] == -1).all()
    for k in range(24):
        o, d = rng.uniform(-8, 24, 3), rng.normal(size=3)
        r = float(rng.choice([0.25, 1.0, 3.0]))
        cap = oracle.capsule_cast(res, capi.make_capsule_sweeps([o], [d], (0, 0, 0), r))
        sph = collide_oracle.sphere_cast(res, r, capi.make_rays([o], [d]))
        for f in ("t", "slot", "block_id", "triangle", "center", "point", "normal", "u", "v", "flags"):
            assert np.array_equal(cap[f], sph[f]), (k, f)


def _sweep(res, o, d, h, r, t_min=0.0, t_max=np.inf, want_class=None):
    """The oracle's capsule sweep against the float64 first contact, within TOL along the path; returns the hit."""
    cls = []
    x = oracle.capsule_cast(res, capi.make_capsule_sweeps([o], [d], h, r, t_min, t_max), classes=cls)[0]
    tris = _tris(res)
    hm = float(np.max(np.abs(h)))
    bounds = collide_oracle.segment_bounds64(res.n, o, d, t_min, t_max, hm + r + 1.0)
    first, _ = oracle.capsule_first_contact64(o, d, bounds[0], bounds[1], h, r, tris)
    speed = float(np.linalg.norm(np.asarray(d, np.float64)))
    if not np.isfinite(first.min()):
        assert x["slot"] == capi.VXB_RAY_MISS, x
        return x
    assert x["slot"] != capi.VXB_RAY_MISS, (o, d, h, r, first.min())
    assert abs(float(x["t"]) - first.min()) * speed < TOL * 10, (x["t"], first.min())
    gap = oracle.segment_triangle_dist64(x["center"].astype(np.float64), h, tris[x["triangle"]][None])[0]
    if not x["flags"]:
        assert abs(gap - r) < TOL * 10, (gap, r)
    assert np.linalg.norm(x["axis_point"].astype(np.float64) - x["point"]) <= r + TOL
    if want_class is not None:
        assert cls[0] == want_class, (cls[0], want_class)
    return x


def test_sweep_feature_classes_agree_with_float64():
    res = _mesh(_single(TRI))
    # a vertical capsule landing on the face with its lower cap
    x = _sweep(res, (3, 12, 3), (0, -1, 0), (0, 2, 0), 1.0, want_class="cap_face")
    assert x["t"] == F(7) and np.allclose(x["center"], (3, 5, 3)) and x["s"] == F(-1)
    # a horizontal capsule lying down on the face (its cylinder)
    x = _sweep(res, (4, 12, 4), (0, -1, 0), (1.5, 0, 0), 1.0, want_class="cap_face")
    assert x["t"] == F(9)
    # the cylinder part onto a triangle vertex: a long capsule across the vertex a, from above and outside
    _sweep(res, (-0.5, 8, -0.5), (0, -1, 0), (3, 0, -3), 0.5, want_class="lateral_edge")
    # the cylinder part onto a triangle edge (skew): the parallelogram of ab
    _sweep(res, (5, 8, 1), (0, -1, 0), (0, 1, 3), 0.5, want_class="parallelogram")
    # the end cap onto an edge, and onto a vertex
    _sweep(res, (5, 2, -8), (0, 0, 1), (0, 0, 2), 1.0, want_class="cap_edge")
    _sweep(res, (-8, 2.5, -8), (1, 0, 1), (-2, 0, -2), 1.0, want_class="shifted_vertex")
    # a capsule in the triangle's plane, sliding into edge ab side-on
    _sweep(res, (5, 2, -8), (0, 0, 1), (3, 0, 0), 1.0)
    # a graze at exactly r: the path stays 1 above the plane (h in a parallel plane)
    x = _sweep(res, (-8, 3, 3), (1, 0, 0), (0, 0, 1), 1.0)
    assert x["slot"] == 0
    # started in contact
    x = _sweep(res, (3, 4, 3), (0, 1, 0), (0, 2.5, 0), 1.0)
    assert x["flags"] == capi.VXB_SPHERE_STARTED_IN_CONTACT and x["t"] == 0
    # misses
    _sweep(res, (3, 12, 3), (1, 0, 0), (0, 2, 0), 1.0)
    _sweep(res, (3, 12, 3), (0, 1, 0), (0, 2, 0), 1.0)


def test_zero_area_triangles():
    line = [(1, 2, 1), (5, 2, 1), (9, 2, 1)]
    res = _mesh(_single(line))
    _segment(res, (5, 4, 1), (0, 0, 1))
    _segment(res, (5, 4, 3), (2, 0, 0))
    _sweep(res, (5, 10, 1), (0, -1, 0), (0, 0, 2), 1.0)
    _sweep(res, (5, 10, 3), (0, -1, 0), (3, 0, 0), 1.0)
    point = [(4, 2, 4)] * 3
    res = _mesh(_single(point))
    x = _segment(res, (4, 5, 4), (1, 0, 0))
    assert x["distance"] == F(3)
    _sweep(res, (4, 10, 4), (0, -1, 0), (1, 1, 0), 1.0)


def test_signed_zero_components_give_the_same_hit():
    res = _mesh(_single(TRI))
    o = [(3, 12, 3)] * 4
    d = [(0.0, -1, 0.0), (-0.0, -1, 0.0), (0.0, -1, -0.0), (-0.0, -1, -0.0)]
    h = [(0.0, 2, 0.0), (-0.0, 2, 0.0), (0.0, 2, -0.0), (-0.0, 2, -0.0)]
    s = capi.make_capsule_sweeps(o, d, (0, 0, 0), 1.0)
    s["half_axis"] = h
    x = oracle.capsule_cast(res, s)
    assert (x["t"] == F(7)).all()
    for f in ("t", "slot", "triangle", "center", "point", "normal", "u", "v", "s"):
        assert (x[f][1:] == x[f][:1]).all(), f


QUAD = [(0, 4, 0), (8, 4, 0), (0, 4, 8), (8, 4, 8)]


def test_ties_across_a_shared_edge_and_a_shared_vertex():
    b0 = _single(QUAD[:3], (0, 1, 2))
    b1 = _single(QUAD, (1, 3, 2, 1, 2, 0))
    for blocks in ([b0, b1], [b1, b0]):
        res = _mesh(*blocks)
        x = oracle.capsule_cast(res, capi.make_capsule_sweeps([(4, -5, 4)], [(0, 1, 0)], (1, 0, -1), 1.0))[0]
        assert x["slot"] == 0 and x["triangle"] == 0 and x["t"] == F(8)
        c = oracle.closest_to_segment(res, capi.make_segments([(4, 6, 4)], [(0, 1, 0)]), 2.0)[0]
        assert c["slot"] == 0 and c["triangle"] == 0 and c["distance"] == F(1)
    t0 = _single([(0, 4, 0), (8, 4, 0), (0, 4, 8)])
    t1 = _single([(8, 4, 0), (16, 4, 4), (12, 4, 8)])
    for first, second in ((t0, t1), (t1, t0)):
        res = _mesh(first, second)
        x = _sweep(res, (8, 4.5, -8), (0, 0, 1), (0, 0, 1), 1.0)
        assert x["slot"] == 0 and np.array_equal(x["point"], np.array([8, 4, 0], np.float32))
        c = oracle.closest_to_segment(res, capi.make_segments([(8, 4, -2)], [(0, 0, 1)]), 2.0)[0]
        assert c["slot"] == 0 and c["distance"] == F(1)


def test_reach_and_invalid_queries_are_misses():
    res = _mesh(_single(TRI))
    ok = capi.make_capsule_sweeps([(3, 12, 3)] * 6, [(0, -1, 0)] * 6, (0, 2, 0), 1.0)
    ok["half_axis"][1] = (14, 0, 0)                          # at the limit: 14 + 1 = 15
    ok["half_axis"][2] = (14.5, 0, 0)                        # beyond it
    ok["half_axis"][3, 0] = np.nan
    ok["radius"][4] = 0.0
    ok["path"]["direction"][5] = 0.0
    x = oracle.capsule_cast(res, ok)
    assert (x["slot"][:2] != capi.VXB_RAY_MISS).all() and (x["slot"][2:] == capi.VXB_RAY_MISS).all()
    segs = capi.make_segments([(3, 5, 3), (3, 5, 3), (np.inf, 5, 3)], [(0, 12, 0), (0, 12.5, 0), (0, 1, 0)])
    x = oracle.closest_to_segment(res, segs, 3.0)
    assert x["slot"][0] != capi.VXB_RAY_MISS and (x["slot"][1:] == capi.VXB_RAY_MISS).all()
    m = x[1:].copy(); m["distance"] = 0; m["slot"] = 0
    assert not m.view(np.uint8).any()


def test_random_segments_and_sweeps_agree_with_float64():
    rng = np.random.RandomState(5)
    pos = rng.uniform(0, 16, (18, 3)).astype(np.float32)
    res = _mesh(_single(pos, np.arange(18)))
    tris = _tris(res)
    for k in range(24):
        c, h = rng.uniform(-4, 20, 3), rng.normal(size=3) * rng.choice([0.5, 3.0])
        d64 = oracle.segment_triangle_dist64(c, h, tris).min()
        if d64 <= 15.0 - np.abs(h).max() - TOL:
            x = oracle.closest_to_segment(res, capi.make_segments([c], [h]), 15.0 - float(np.abs(h).max()))[0]
            assert abs(float(x["distance"]) - d64) < TOL, (c, h, x["distance"], d64)
    for k in range(6):
        o, d = rng.uniform(-8, 24, 3), rng.normal(size=3)
        h, r = rng.normal(size=3) * 2.0, float(rng.choice([0.5, 2.0]))
        bounds = collide_oracle.segment_bounds64(res.n, o, d, 0.0, np.inf, float(np.abs(h).max()) + r + 1.0)
        if bounds is None:
            continue
        first, dmin = oracle.capsule_first_contact64(o, d, bounds[0], bounds[1], h, r, tris)
        if np.isfinite(first.min()) and np.sort(dmin)[0] > r - 1e-3:
            continue                                  # a near-tangent graze: the answer hangs on rounding
        _sweep(res, o, d, h, r)
