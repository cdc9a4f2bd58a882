"""CPU-side checks of the capsule queries against the drawn LOD cut (include/vxb200.h "capsule queries against the drawn LOD
cut"): the hit mirrors against a C compiler's layout, the bindings, and the numpy oracle (tests/capsule_cut_oracle.py) on
hand-built meshes - the position rule of the vertex shader, transition meshes, the tie rule, the cut reach rule - its equality
with the level-0 capsule oracle at lod_factor 1e30 and with the sphere cut oracle at h = 0, and its geometry against
capsule_oracle's float64 references."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import capsule_cut_oracle as oracle
import capsule_oracle
import collide_cut_oracle
import raycast_cut_oracle
from test_raycast_cut_cpu import ADJ, CAMERA, FACTOR, FLAT, LEVELS, N, _moved, _restated_sphere_with_levels
from voxels_b200 import capi

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32
REGULAR = raycast_cut_oracle.REGULAR
UP2 = (0.0, 2.0, 0.0)


def _blocks(*blocks):
    return raycast_cut_oracle.result_from_blocks(N, LEVELS, list(blocks))


def _sweep(res, h, r, origin=(6, 30, 6), direction=(0, -1, 0), e=0.0):
    return oracle.capsule_cast_cut(res, CAMERA, FACTOR, capi.make_capsule_sweeps([origin], [direction], h, r), e)


def _segment(res, c, h, md, e=0.0):
    return oracle.closest_to_segment_cut(res, CAMERA, FACTOR, capi.make_segments([c], [h]), md, e)


def test_hit_mirrors_match_the_header(tmp_path):
    gcc = shutil.which("gcc")
    if not gcc:
        pytest.skip("no gcc")
    structs = {"vxb_capsule_cut_hit": capi.CAPSULE_CUT_HIT_DTYPE, "vxb_segment_cut_hit": capi.SEGMENT_CUT_HIT_DTYPE}
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "vxb200.h"', 'int main(void)', '{']
    for s, dt in structs.items():
        lines.append('\tprintf("%s %%zu\\n", sizeof(%s));' % (s, s))
        lines += ['\tprintf("%s.%s %%zu\\n", offsetof(%s, %s));' % (s, f, s, f) for f in dt.names]
    lines += ['\treturn 0;', '}']
    src = tmp_path / "capsulecut.c"
    src.write_text("\n".join(lines) + "\n")
    exe = tmp_path / "capsulecut"
    out = subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(REPO, "include"), str(src), "-o", str(exe)],
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    got = dict(line.split() for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines())
    assert int(got["vxb_capsule_cut_hit"]) == capi.CAPSULE_CUT_HIT_DTYPE.itemsize == 88
    assert int(got["vxb_segment_cut_hit"]) == capi.SEGMENT_CUT_HIT_DTYPE.itemsize == 72
    for s, dt in structs.items():
        for f in dt.names:
            assert int(got[s + "." + f]) == dt.fields[f][1], (s, f)
    assert capi.CAPSULE_CUT_HIT_DTYPE.descr[:len(capi.CAPSULE_HIT_DTYPE.descr)] == capi.CAPSULE_HIT_DTYPE.descr
    assert capi.SEGMENT_CUT_HIT_DTYPE.descr[:len(capi.SEGMENT_HIT_DTYPE.descr)] == capi.SEGMENT_HIT_DTYPE.descr


def test_cut_capsule_queries_are_bound():
    names = {"vxb_mesh_capsule_cast_cut", "vxb_mesh_capsule_cast_cut_device", "vxb_mesh_closest_to_segment_cut",
             "vxb_mesh_closest_to_segment_cut_device"}
    assert names <= set(capi.EXPORTED_SYMBOLS)
    for a in ("capsule_cast_cut", "capsule_cast_cut_rc", "capsule_cast_cut_device", "closest_to_segment_cut",
              "closest_to_segment_cut_rc", "closest_to_segment_cut_device"):
        assert hasattr(capi.Mesh, a), a


def test_secondary_position_when_the_mask_is_covered():
    covered, uncovered = _blocks((1, (0, 0, 0), _moved(ADJ), {})), _blocks((1, (0, 0, 0), _moved(ADJ | 1), {}))
    # a vertical capsule (half axis 2, radius 1) from y = 30: its bottom reaches the drawn y = 20 at t = 7, y = 10 at t = 17
    h = _sweep(covered, UP2, 1.0)
    assert h["slot"][0] == 0 and h["t"][0] == 7.0 and h["point"][0][1] == 20.0 and h["center"][0][1] == 23.0
    assert h["axis_point"][0][1] == 21.0 and h["s"][0] == -1.0
    assert h["level"][0] == 1 and h["face"][0] == REGULAR and h["block_id"][0] == 1000 and h["flags"][0] == 0
    assert _sweep(uncovered, UP2, 1.0)["t"][0] == 17.0
    zero = _blocks((1, (0, 0, 0), _moved(0), {}))
    assert _sweep(zero, UP2, 1.0)["t"][0] == 17.0
    # the segment (6, 25 -+ 2, 6) is 3 from the drawn triangle at y = 20 and 13 from the one at y = 10
    h = _segment(covered, (6, 25, 6), UP2, 10.0)
    assert h["distance"][0] == 3.0 and h["point"][0][1] == 20.0 and h["axis_point"][0][1] == 23.0 and h["s"][0] == -1.0
    assert h["level"][0] == 1 and h["face"][0] == REGULAR
    assert _segment(uncovered, (6, 25, 6), UP2, 10.0)["slot"][0] == capi.VXB_RAY_MISS
    assert _segment(uncovered, (6, 25, 6), UP2, 15.0 - 2.0)["distance"][0] == 13.0
    assert _segment(zero, (6, 25, 6), UP2, 13.0)["distance"][0] == 13.0


def test_transition_faces_outside_block_adj_are_never_hit():
    wall = lambda x: dict(pos=[(x, 2, 2), (x, 30, 2), (x, 2, 30)], idx=[0, 1, 2])   # noqa: E731
    res = _blocks((1, (0, 0, 0), FLAT, {0: wall(25.0), 5: wall(31.0)}))
    # face 0's wall (x = 25) is not drawn: the capsule (half axis 1 along x, radius 1) passes it and touches face 5's wall
    # (x = 31) when its centre is at x = 29, t = 9
    h = _sweep(res, (1.0, 0.0, 0.0), 1.0, (20, 15, 6), (1, 0, 0))
    assert h["slot"][0] == 0 and h["face"][0] == 5 and h["t"][0] == 9.0 and h["triangle"][0] == 0 and h["level"][0] == 1
    assert h["axis_point"][0][0] == 30.0 and h["s"][0] == 1.0
    # the segment (26 -+ 1, 16, 10) is 2 from face 0's wall and 4 from face 5's
    h = _segment(res, (26, 16, 10), (1.0, 0.0, 0.0), 6.0)
    assert h["face"][0] == 5 and h["distance"][0] == 4.0
    assert _segment(res, (26, 16, 10), (1.0, 0.0, 0.0), 3.0)["slot"][0] == capi.VXB_RAY_MISS


def test_ties_go_to_slot_then_part_then_triangle():
    two = dict(pos=FLAT["pos"], idx=[0, 1, 2, 0, 1, 2])
    dot = dict(pos=[(0, 0, 0)] * 3, idx=[0, 1, 2])
    queries = (lambda res: _sweep(res, UP2, 1.0), lambda res: _segment(res, (6, 25, 6), UP2, 13.0))
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
    assert _sweep(_blocks((1, (0, 0, 0), FLAT, {5: two})), UP2, 1.0)["t"][0] == 17.0
    assert _segment(_blocks((1, (0, 0, 0), FLAT, {5: two})), (6, 25, 6), UP2, 13.0)["distance"][0] == 13.0


def test_the_cut_reach_rule_is_per_query():
    res = _blocks((1, (0, 0, 0), _moved(ADJ), {}))
    # e + (max |h_i| + r) <= 15 in float32, in that order: with e = 2 a reach of 13 is in, 13.5 is out
    assert oracle.cut_reach_ok(UP2, 11.0, 2.0) and not oracle.cut_reach_ok(UP2, 11.5, 2.0)
    assert not oracle.cut_reach_ok((np.nan, 0, 0), 1.0, 0.0) and not oracle.cut_reach_ok(UP2, 13.5, 0.0)
    # h = 0: the sphere cut's e + R <= 15
    for e in (0.0, 0.3, 4.75):
        limit = collide_cut_oracle.reach_limit(F(e))
        assert oracle.cut_reach_ok((0, 0, 0), limit, e) and not oracle.cut_reach_ok((0, 0, 0), np.nextafter(limit, F(16)), e)
    assert _sweep(res, UP2, 11.0, e=2.0)["slot"][0] == 0
    assert _sweep(res, UP2, 11.5, e=2.0)["slot"][0] == capi.VXB_RAY_MISS
    assert _segment(res, (6, 25, 6), UP2, 11.0, e=2.0)["slot"][0] == 0
    miss = _segment(res, (6, 25, 6), UP2, 11.5, e=2.0)
    assert miss["slot"][0] == capi.VXB_RAY_MISS and miss["distance"][0] == np.inf and miss["level"][0] == 0 and miss["face"][0] == 0


def _first(h, nbytes):
    return np.ascontiguousarray(h).view(np.uint8).reshape(len(h), -1)[:, :nbytes]


def _capsule_queries(rng):
    c = np.full(3, 32.0)
    dirs = rng.normal(size=(160, 3))
    o = np.concatenate([c + dirs / np.linalg.norm(dirs, axis=1, keepdims=True) * 30, rng.uniform(-8, 72, (64, 3))])
    dv = np.concatenate([-dirs, rng.normal(size=(64, 3))])
    h = rng.normal(size=(len(o), 3)) * rng.choice([0.0, 0.5, 3.0], (len(o), 1))
    r = rng.choice([0.5, 2.0], len(o))
    sweeps = capi.make_capsule_sweeps(o, dv, h, r)
    sweeps["half_axis"][-4:] = (12.0, 0.0, 0.0)                 # max |h_i| + r above 15: misses everywhere
    sweeps["radius"][-4:] = 4.0
    centres = np.concatenate([c + dirs[:96] / np.linalg.norm(dirs[:96], axis=1, keepdims=True) * rng.uniform(16, 28, (96, 1)),
                              rng.uniform(-4, 68, (48, 3))])
    segments = capi.make_segments(centres, rng.normal(size=(len(centres), 3)) * rng.choice([0.0, 1.0, 3.0], (len(centres), 1)))
    return sweeps, segments


def test_factor_1e30_equals_the_level0_oracle(restatement):
    res = _restated_sphere_with_levels(restatement)
    rng = np.random.RandomState(41)
    sweeps, segments = _capsule_queries(rng)
    camera = (5.0, 70.0, 9.0)
    d = raycast_cut_oracle.Drawn(res, camera, 1e30)
    got = oracle.capsule_cast_cut(res, camera, 1e30, sweeps, 0.0, d)
    want = capsule_oracle.capsule_cast(res, sweeps)
    hit = got["slot"] != capi.VXB_RAY_MISS
    assert hit.sum() > 80 and not hit[-4:].any()
    assert np.array_equal(_first(got, 80), want.view(np.uint8).reshape(len(want), -1))
    assert (got["level"] == 0).all() and (got["face"][hit] == REGULAR).all() and (got["face"][~hit] == 0).all()
    for md in (0.0, 2.0, 6.0):
        got = oracle.closest_to_segment_cut(res, camera, 1e30, segments, md, 0.0, d)
        want = capsule_oracle.closest_to_segment(res, segments, md)
        assert np.array_equal(_first(got, 64), want.view(np.uint8).reshape(len(want), -1))
        hit = got["slot"] != capi.VXB_RAY_MISS
        assert (got["level"] == 0).all() and (got["face"][hit] == REGULAR).all() and (got["face"][~hit] == 0).all()
        if md == 6.0:
            assert hit.sum() > 60


def test_zero_half_axis_equals_the_sphere_cut_oracle(restatement):
    """h = 0: every field of the sphere cut's hits, with s = -1 and axis_point = center (sweeps) or the query point
    (segments) on a hit; at lod_factor 2 from above, where coarse and transition triangles are drawn."""
    res = _restated_sphere_with_levels(restatement)
    rng = np.random.RandomState(42)
    sweeps, segments = _capsule_queries(rng)
    sweeps, segments = sweeps[:-4], segments.copy()
    sweeps["half_axis"], segments["half_axis"] = 0.0, 0.0
    for camera, factor in (((32.0, 300.0, 32.0), 2.0), ((5.0, 70.0, 9.0), 4.0)):
        d = raycast_cut_oracle.Drawn(res, camera, factor)
        for r in (0.5, 2.0):
            sweeps["radius"] = r
            got = oracle.capsule_cast_cut(res, camera, factor, sweeps, 0.0, d)
            want = collide_cut_oracle.sphere_cast_cut(res, camera, factor, r, sweeps["path"], d)
            hit = got["slot"] != capi.VXB_RAY_MISS
            assert hit.sum() > 80
            for f in want.dtype.names:
                assert np.array_equal(got[f].view(np.uint32), want[f].view(np.uint32)), (camera, r, f)
            assert (got["s"][hit] == -1.0).all() and np.array_equal(got["axis_point"][hit], got["center"][hit])
            assert not got["s"][~hit].any() and not got["axis_point"][~hit].any()
        for md in (2.0, 6.0):
            got = oracle.closest_to_segment_cut(res, camera, factor, segments, md, 0.0, d)
            want = collide_cut_oracle.closest_points_cut(res, camera, factor, segments["center"], md, d)
            hit = got["slot"] != capi.VXB_RAY_MISS
            assert hit.sum() > 5
            for f in want.dtype.names:
                assert np.array_equal(got[f].view(np.uint32), want[f].view(np.uint32)), (camera, md, f)
            assert (got["s"][hit] == -1.0).all() and np.array_equal(got["axis_point"][hit], segments["center"][hit])


def test_geometry_agrees_with_float64(restatement):
    """At lod_factor 2 from above the level-2 slab is drawn: a sweep contact not started in contact is r from its drawn
    triangle, no drawn triangle near the path comes closer than r before it, and every segment distance is the float64
    distance to the drawn set."""
    res = _restated_sphere_with_levels(restatement)
    rng = np.random.RandomState(43)
    sweeps, segments = _capsule_queries(rng)
    camera = (32.0, 300.0, 32.0)
    d = raycast_cut_oracle.Drawn(res, camera, 2.0)
    tol = 2e-3
    got = oracle.capsule_cast_cut(res, camera, 2.0, sweeps, 0.0, d)
    assert (got["level"][got["slot"] != capi.VXB_RAY_MISS] > 0).any()
    where = {(s, p): b for b, (s, p) in enumerate(zip(d.slot, d.part))}
    checked = 0
    for i in rng.choice(len(sweeps) - 4, 24, replace=False):
        sw, x = sweeps[i], got[i]
        h, r = sw["half_axis"].astype(np.float64), float(sw["radius"])
        ray = sw["path"]
        o, dv = ray["origin"].astype(np.float64), ray["direction"].astype(np.float64)
        if x["slot"] != capi.VXB_RAY_MISS:
            part = 0 if x["face"] == REGULAR else int(x["face"]) + 1
            tri = d.tri_pos[where[(int(x["slot"]), part)]][x["triangle"]]
            gap = capsule_oracle.segment_triangle_dist64(x["center"].astype(np.float64), h, tri[None])[0]
            assert gap <= r + tol if x["flags"] else abs(gap - r) <= tol, (sw, x, gap)
            if x["flags"]:
                continue
        t_hi = float(x["t"]) if x["slot"] != capi.VXB_RAY_MISS else 200.0
        near = raycast_cut_oracle._near_parts(d, o.astype(np.float32), dv.astype(np.float32), F(ray["t_min"]), F(t_hi),
                                              float(np.abs(h).max()) + r + 1.0)
        tris = [d.tri_pos[b] for b in near if len(d.tri_pos[b])]
        if not tris:
            continue
        _, dmin = capsule_oracle.capsule_first_contact64(o, dv, float(ray["t_min"]), t_hi, h, r, np.concatenate(tris), iters=40)
        assert dmin.min() >= r - tol, (sw, x, dmin.min())
        checked += 1
    assert checked > 6
    tris = np.concatenate([p for p in d.tri_pos if len(p)])
    for md in (2.0, 6.0):
        got = oracle.closest_to_segment_cut(res, camera, 2.0, segments[:48], md, 0.0, d)
        d64 = np.array([capsule_oracle.segment_triangle_dist64(s["center"], s["half_axis"].astype(np.float64), tris).min()
                        for s in segments[:48]])
        hit = got["slot"] != capi.VXB_RAY_MISS
        ok = np.array([oracle.cut_reach_ok(s["half_axis"], md, 0.0) for s in segments[:48]])
        assert hit.sum() >= 5 and not hit[~ok].any()
        assert np.all(np.abs(got["distance"][hit].astype(np.float64) - d64[hit]) <= tol)
        assert np.all(d64[~hit & ok] >= md - tol)
