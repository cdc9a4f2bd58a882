"""Collision queries against the drawn LOD cut (include/vxb200.h "collision queries against the drawn LOD cut"): every field of
every sphere-sweep and closest-point hit is bit-identical to the numpy oracle (tests/collide_cut_oracle.py) on mesh.download(),
for the sweep and point sets of test_gpu_collide at the cameras and factors of test_gpu_cut and at the reach limit 15 - e,
for queries aimed at drawn transition triangles and at moved regular triangles, across edits, compaction and growth, through
the device variants, with a block whose vertices leave its lattice box, and at 1024^3.  At lod_factor 1e30 the queries equal
vxb_mesh_sphere_cast and vxb_mesh_closest_point; the sweeps contain the cut rays and the closest points find them."""
import ctypes as C

import numpy as np
import pytest

import collide_cut_oracle as oracle
from raycast_cut_oracle import REGULAR, Drawn
from test_gpu_collide import _hit_buffer, _read, _to_device, assert_same, point_sets, sweep_sets
from test_gpu_cut import FACTORS, GRIDS, _applied_mesh, _brush, _cameras
from test_gpu_raycast import _fill, camera_rays, corner_rays, random_rays
from test_gpu_raycast_cut import _aimed_rays, _classes, _move_level1_vertex
from voxels_b200 import capi
from voxels_b200.capi import Op

pytestmark = pytest.mark.gpu

F = np.float32


def _sweeps(res, r, rng, per_set=16):
    _, sets = sweep_sets(res, r, rng, per_set)
    return np.concatenate([s[:per_set] for s in sets.values()])


def _points(res, md, rng, per_set=16):
    return np.concatenate(list(point_sets(res, md, rng, per_set).values())).astype(np.float32)


def _aimed_points(d, rng, per_class=64):
    """Points 1/4 voxel off the centroids of drawn transition triangles and of regular triangles with a vertex at its
    secondary position."""
    targets = []
    for b in range(len(d.slot)):
        if not len(d.tri_pos[b]):
            continue
        pick = np.nonzero(d.moved[b])[0] if d.part[b] == 0 else np.arange(len(d.tri_pos[b]))
        targets += [d.tri_pos[b][k].astype(np.float64).mean(axis=0) for k in pick[:2]]
    if not targets:
        return np.zeros((0, 3), np.float32)
    targets = np.array(targets)[rng.permutation(len(targets))[:2 * per_class]]
    off = rng.normal(size=targets.shape)
    off *= 0.25 / np.linalg.norm(off, axis=1, keepdims=True)
    return (targets + off).astype(np.float32)


def _check_sweeps(mesh, res, camera, factor, r, rays, what, d):
    got = mesh.sphere_cast_cut(camera, factor, r, rays)
    assert_same(got, oracle.sphere_cast_cut(res, camera, factor, r, rays, d), rays, what)
    return got


def _check_points(mesh, res, camera, factor, md, pts, what, d):
    got = mesh.closest_points_cut(camera, factor, pts, md)
    assert_same(got, oracle.closest_points_cut(res, camera, factor, pts, md, d), pts, what)
    return got


def _first(h, nbytes):
    return np.ascontiguousarray(h).view(np.uint8).reshape(len(h), -1)[:, :nbytes]


def _level0_fields(got, want, nbytes, what):
    assert np.array_equal(_first(got, nbytes), want.view(np.uint8).reshape(len(want), -1)), what
    hit = got["slot"] != capi.VXB_RAY_MISS
    assert (got["level"] == 0).all() and (got["face"][hit] == REGULAR).all() and (got["face"][~hit] == 0).all(), what


@pytest.mark.parametrize("name", GRIDS)
def test_sweep_and_point_sets_equal_oracle(gpu_context, name):
    mesh = _applied_mesh(gpu_context, name)
    try:
        res = mesh.download()
        n = res.n
        rng = np.random.RandomState(19)
        limit = oracle.reach_limit(oracle.excursion(res, mesh.bounds()))
        radii, distances = (0.5, 2.0, float(limit)), (0.0, 2.0, float(limit))
        sweeps = {r: _sweeps(res, r, rng, 8) for r in radii}
        points = {md: _points(res, md, rng, 8) for md in distances}
        won_s, won_p = set(), set()
        for factor in FACTORS:
            for c, camera in enumerate(_cameras(n, factor)[:2]):
                d = Drawn(res, camera, factor)
                what = "%s factor %g camera %d" % (name, factor, c)
                for r, rays in (sweeps.items() if c == 0 else ()):
                    got = _check_sweeps(mesh, res, camera, factor, r, rays, "%s r=%g" % (what, r), d)
                    assert (got["slot"] != capi.VXB_RAY_MISS).any()
                    won_s |= _classes(d, got)
                    if factor == 1e30:
                        _level0_fields(got, mesh.sphere_cast(r, rays), 64, "%s r=%g level 0" % (what, r))
                for md, pts in (points.items() if c == 0 else ()):
                    got = _check_points(mesh, res, camera, factor, md, pts, "%s md=%g" % (what, md), d)
                    won_p |= _classes(d, got)
                    if factor == 1e30:
                        _level0_fields(got, mesh.closest_points(pts, md), 48, "%s md=%g level 0" % (what, md))
                aimed = _aimed_rays(d, rng, 24)
                if len(aimed):
                    won_s |= _classes(d, _check_sweeps(mesh, res, camera, factor, 0.5, aimed, what + " aimed sweeps", d))
                near = _aimed_points(d, rng, 24)
                if len(near):
                    won_p |= _classes(d, _check_points(mesh, res, camera, factor, 2.0, near, what + " aimed points", d))
        assert "regular" in won_s and "regular" in won_p, (name, won_s, won_p)
        if name in ("terrain128", "terrain256", "patchwork128"):
            assert {"regular", "secondary", "transition"} <= won_s, (name, won_s)
            assert {"regular", "secondary", "transition"} <= won_p, (name, won_p)
    finally:
        mesh.close()


def test_sweeps_contain_the_cut_rays_and_closest_points_find_them(gpu_context):
    """At a radius of 2^-8 voxel a cut-ray hit implies a cut-sweep contact no later than it (up to 1e-5 |t|), and the closest
    drawn point to a cut-ray hit position, within 1/4 voxel, is within 1e-4 voxel of it for 99 % of the hits and within
    2e-3 voxel for all (a grazing ray's t carries the rounding of a small determinant into its position)."""
    n = 128
    mesh = _applied_mesh(gpu_context, "terrain128")
    rng = np.random.RandomState(3)
    try:
        res = mesh.download()
        rays = np.concatenate([camera_rays(res, 2048, rng), random_rays(n, 1024, rng), corner_rays(n, 512, rng)])
        coarse = 0
        for factor, camera in ((2.0, (0.4 * n, 0.3 * n, 0.45 * n)), (4.0, (0.5 * n, 1.5 * n, 0.55 * n)), (14.6, (0.5 * n, 0.25 * n, 0.75 * n))):
            ray_hits = mesh.raycast_cut(camera, factor, rays)
            sweep_hits = mesh.sphere_cast_cut(camera, factor, 2.0 ** -8, rays)
            hit = ray_hits["slot"] != capi.VXB_RAY_MISS
            assert hit.sum() > 1000
            coarse += int((ray_hits["level"][hit] > 0).sum())
            assert (sweep_hits["slot"][hit] != capi.VXB_RAY_MISS).all()
            t_ray = ray_hits["t"][hit].astype(np.float64)
            assert (sweep_hits["t"][hit] <= t_ray + 1e-5 * np.abs(t_ray)).all()
            near = mesh.closest_points_cut(camera, factor, ray_hits["position"][hit], 0.25)
            assert (near["slot"] != capi.VXB_RAY_MISS).all() and (near["distance"] <= 2e-3).all(), near["distance"].max()
            assert (near["distance"] <= 1e-4).mean() >= 0.99, np.sort(near["distance"])[-20:]
        assert coarse > 0
    finally:
        mesh.close()


def _edit_check(mesh, res, camera, factor, rng, n, what):
    d = Drawn(res, camera, factor)
    limit = float(oracle.reach_limit(oracle.excursion(res, mesh.bounds())))
    sweeps = np.concatenate([random_rays(n, 24, rng), camera_rays(res, 48, rng), corner_rays(n, 16, rng)])
    for r in (2.0, limit):
        _check_sweeps(mesh, res, camera, factor, r, sweeps, "%s r=%g" % (what, r), d)
    pts = np.concatenate([rng.uniform(-4, n + 4, (48, 3)), res.verts["pos"][rng.randint(0, len(res.verts), 48)] + rng.normal(size=(48, 3))])
    for md in (4.0, limit):
        _check_points(mesh, res, camera, factor, md, pts.astype(np.float32), "%s md=%g" % (what, md), d)


def test_after_brush_edits(gpu_context):
    n = 128
    ctx = gpu_context
    mesh = _applied_mesh(ctx, "terrain128")
    rng = np.random.RandomState(22)
    try:
        for edit in range(25):
            x, z = rng.uniform(16, n - 16, 2)
            p = mesh.raycast(capi.make_rays([(x, n + 8.0, z)], [(0, -1, 0)]))
            assert p["slot"][0] != capi.VXB_RAY_MISS
            hit = p["position"][0]
            r = float(rng.choice([4, 6, 8]))
            box = ctx.inject_program(np.array([hit[0], hit[2], hit[1]], F), np.full(3, 2 * r + 4, F), _brush(edit, r), 0 if edit % 2 == 0 else 2)
            ctx.polygonize_region(box[:3], box[3:])
            mesh.apply()
            res = mesh.download()
            camera, factor = _cameras(n, 2.0)[edit % 4], (2.0, 4.0, 14.6)[edit % 3]
            _edit_check(mesh, res, camera, factor, rng, n, "edit %d" % edit)
    finally:
        mesh.close()


def test_after_compaction_and_growth(gpu_context):
    import gridgen
    n = 128
    ctx = gpu_context
    mesh = _applied_mesh(ctx, "patchwork128", (4096, 4096, 1024, 1024))
    ctx.set_launch_limit(2)
    rng = np.random.RandomState(9)
    try:
        for i, (pos, r, ext, add) in enumerate(gridgen.edge_edit_sequence(n, 12)):
            box = ctx.inject_surface(np.array(pos, F), np.full(3, ext, F), capi.Surface.sphere((0, 0, 0), r), 0 if add else 2)
            ctx.polygonize_region(box[:3], box[3:])
            mesh.apply()
            res = mesh.download()
            _edit_check(mesh, res, _cameras(n, 4.0)[i % 4], (2.0, 4.0)[i % 2], rng, n, "edge edit %d" % i)
        info = mesh.info()
        assert info.compactions > 0 and info.growths > 0
    finally:
        ctx.set_launch_limit(0)
        mesh.close()


def test_excursion_is_named_and_bounded(gpu_context):
    n = 128
    ctx = gpu_context
    ctx.set_materials(None, None)
    _fill(ctx, "terrain128")
    ctx.polygonize()
    _move_level1_vertex(ctx, 5.0)
    mesh = ctx.mesh()
    rng = np.random.RandomState(13)
    try:
        mesh.apply()
        res = mesh.download()
        e = oracle.excursion(res, mesh.bounds())
        assert e >= 5.0
        reach = min(10.0, float(oracle.reach_limit(e)))
        sweeps = _sweeps(res, reach, rng, 16)
        pts = _points(res, reach, rng, 16)
        for factor in (2.0, 4.0, 1e30):
            for camera in _cameras(n, factor)[:2]:
                d = Drawn(res, camera, factor)
                aimed = _aimed_rays(d, rng, 16)
                rays = np.concatenate([sweeps, aimed]) if len(aimed) else sweeps
                _check_sweeps(mesh, res, camera, factor, reach, rays, "excursion 5, factor %g sweeps" % factor, d)
                _check_points(mesh, res, camera, factor, reach, pts, "excursion 5, factor %g points" % factor, d)
        camera = (60.0, 90.0, 60.0)
        s_sent = np.frombuffer(bytes(range(256)) * 2, np.uint8)[:4 * 72].copy().view(capi.SPHERE_CUT_HIT_DTYPE)
        c_sent = np.frombuffer(bytes(range(256)) * 2, np.uint8)[:4 * 56].copy().view(capi.CLOSEST_CUT_HIT_DTYPE)
        sh, ch = s_sent.copy(), c_sent.copy()
        assert mesh.sphere_cast_cut_rc(camera, 4.0, 10.5, sweeps[:4], sh) == capi.ERR_STATE and sh.tobytes() == s_sent.tobytes()
        err = ctx.L.vxb_last_error(ctx.h)
        assert b"lattice box by" in err and b"(e)" in err and b"10.5" in err, err
        assert mesh.closest_points_cut_rc(camera, 4.0, 10.5, pts[:4], ch) == capi.ERR_STATE and ch.tobytes() == c_sent.tobytes()
        assert b"lattice box by" in ctx.L.vxb_last_error(ctx.h)
        ctx.polygonize()
        mesh.apply()
        assert mesh.sphere_cast_cut_rc(camera, 4.0, 10.5, sweeps[:4], sh) == 0
        assert mesh.closest_points_cut_rc(camera, 4.0, 10.5, pts[:4], ch) == 0
    finally:
        mesh.close()


def test_device_variants_equal_host_and_see_the_mesh_of_their_queue_position(gpu_context):
    import torch
    n = 128
    ctx = gpu_context
    mesh = _applied_mesh(ctx, "terrain128")
    rng = np.random.RandomState(6)
    camera, factor = (64.0, 150.0, 64.0), 4.0
    try:
        res = mesh.download()
        rays = _sweeps(res, 2.0, rng, 32)
        bad = capi.make_rays([(10, 200, 10)] * 5, [(0, -1, 0), (0, 0, 0), (np.inf, -1, 0), (0, -1, 0), (0, -1, 0)],
                             t_min=[0, 0, 0, np.nan, 5], t_max=[np.inf, np.inf, np.inf, 1, 4])
        bad["origin"][0, 0] = np.nan
        all_rays = np.concatenate([rays, bad])
        rt, ht = _to_device(all_rays), _hit_buffer(len(all_rays), capi.SPHERE_CUT_HIT_DTYPE)
        torch.cuda.synchronize()
        mesh.sphere_cast_cut_device(camera, factor, 2.0, rt.data_ptr(), len(all_rays), ht.data_ptr())
        got = _read(ht, capi.SPHERE_CUT_HIT_DTYPE)
        assert_same(got[:len(rays)], mesh.sphere_cast_cut(camera, factor, 2.0, rays), rays, "sweeps: device vs host")
        miss = np.zeros(len(bad), capi.SPHERE_CUT_HIT_DTYPE); miss["t"] = np.inf; miss["slot"] = capi.VXB_RAY_MISS
        assert_same(got[len(rays):], miss, bad, "invalid sweeps on the device")

        pts = _points(res, 4.0, rng, 32)
        bad_pts = np.array([[np.nan, 1, 1], [1, np.inf, 1], [1, 1, -np.inf]], np.float32)
        all_pts = np.concatenate([pts, bad_pts]).astype(np.float32)
        pt, hp = _to_device(all_pts), _hit_buffer(len(all_pts), capi.CLOSEST_CUT_HIT_DTYPE)
        torch.cuda.synchronize()
        mesh.closest_points_cut_device(camera, factor, 4.0, pt.data_ptr(), len(all_pts), hp.data_ptr())
        got = _read(hp, capi.CLOSEST_CUT_HIT_DTYPE)
        assert_same(got[:len(pts)], mesh.closest_points_cut(camera, factor, pts, 4.0), pts, "points: device vs host")
        miss = np.zeros(len(bad_pts), capi.CLOSEST_CUT_HIT_DTYPE); miss["distance"] = np.inf; miss["slot"] = capi.VXB_RAY_MISS
        assert_same(got[len(pts):], miss, bad_pts, "invalid points on the device")

        # queries queued before an apply see the mesh before it
        before = mesh.download()
        top = mesh.raycast(capi.make_rays([(64, 2 * n, 64)], [(0, -1, 0)]))
        centre = (64.0, 64.0, float(top["position"][0][1]))
        box = ctx.inject_program(centre, (40, 40, 40), [Op.sphere(16)], 2)
        ctx.polygonize_region(box[:3], box[3:])
        o = np.stack([rng.uniform(56, 72, 256), np.full(256, 2.0 * n), rng.uniform(56, 72, 256)], axis=1)
        down = capi.make_rays(o, np.tile([0.0, -1.0, 0.0], (256, 1)))
        crater = np.stack([o[:, 0], np.full(256, float(top["position"][0][1])), o[:, 2]], axis=1).astype(np.float32)
        rt, ht = _to_device(down), _hit_buffer(len(down), capi.SPHERE_CUT_HIT_DTYPE)
        pt, hp = _to_device(crater), _hit_buffer(len(crater), capi.CLOSEST_CUT_HIT_DTYPE)
        torch.cuda.synchronize()
        mesh.sphere_cast_cut_device(camera, factor, 1.0, rt.data_ptr(), len(down), ht.data_ptr())
        mesh.closest_points_cut_device(camera, factor, 8.0, pt.data_ptr(), len(crater), hp.data_ptr())
        mesh.apply()
        old_s, old_p = _read(ht, capi.SPHERE_CUT_HIT_DTYPE), _read(hp, capi.CLOSEST_CUT_HIT_DTYPE)
        assert_same(old_s, oracle.sphere_cast_cut(before, camera, factor, 1.0, down), down, "sweeps queued before the apply")
        assert_same(old_p, oracle.closest_points_cut(before, camera, factor, crater, 8.0), crater, "points queued before the apply")
        after = mesh.download()
        d = Drawn(after, camera, factor)
        new_s = _check_sweeps(mesh, after, camera, factor, 1.0, down, "sweeps after the apply", d)
        new_p = _check_points(mesh, after, camera, factor, 8.0, crater, "points after the apply", d)
        assert not np.array_equal(old_s["t"], new_s["t"]) and not np.array_equal(old_p["distance"], new_p["distance"])
    finally:
        mesh.close()


def test_refusals_leave_hits_untouched(gpu_context):
    assert capi.SPHERE_CUT_HIT_DTYPE.itemsize == 72 and capi.CLOSEST_CUT_HIT_DTYPE.itemsize == 56
    ctx = gpu_context
    L = ctx.L
    n = 64
    ctx.set_materials(None, None)
    ctx.fill(n, capi.Surface.terrain(n))
    ctx.polygonize()
    mesh = ctx.mesh()
    try:
        good = capi.make_rays([(10, 100, 10)] * 4, [(0, -1, 0)] * 4)
        pts = np.full((4, 3), 10.0, np.float32)
        s_sent = np.frombuffer(bytes(range(256)) * 2, np.uint8)[:4 * 72].copy().view(capi.SPHERE_CUT_HIT_DTYPE)
        c_sent = np.frombuffer(bytes(range(256)) * 2, np.uint8)[:4 * 56].copy().view(capi.CLOSEST_CUT_HIT_DTYPE)
        cam = (20.0, 40.0, 20.0)
        cp = capi._ptr(np.array(cam, F))

        def sweep(r=1.0, rays=good, camera=cam, factor=4.0, count=None, fresh=True):
            h = s_sent.copy() if fresh else None
            return mesh.sphere_cast_cut_rc(camera, factor, r, rays, h, count), h

        def point(md=1.0, p=pts, camera=cam, factor=4.0, count=None, fresh=True):
            h = c_sent.copy() if fresh else None
            return mesh.closest_points_cut_rc(camera, factor, md, p, h, count), h

        def refused(rc_h, rc, sentinel):
            assert rc_h[0] == rc and (rc_h[1] is None or rc_h[1].tobytes() == sentinel.tobytes()), rc_h[0]

        refused(sweep(), capi.ERR_STATE, s_sent)                                        # nothing applied yet
        refused(point(), capi.ERR_STATE, c_sent)
        assert L.vxb_mesh_sphere_cast_cut_device(mesh.h, cp, 4.0, 1.0, C.c_void_p(8), 1, C.c_void_p(8)) == capi.ERR_STATE
        assert L.vxb_mesh_closest_point_cut_device(mesh.h, cp, 4.0, 1.0, C.c_void_p(8), 1, C.c_void_p(8)) == capi.ERR_STATE
        mesh.apply()
        assert sweep()[0] == 0 and point()[0] == 0
        for r in (0.0, 15.5, np.nan):
            refused(sweep(r), -2, s_sent)
            assert b"radius" in L.vxb_last_error(ctx.h)
            assert L.vxb_mesh_sphere_cast_cut_device(mesh.h, cp, 4.0, r, C.c_void_p(8), 1, C.c_void_p(8)) == -2, r
        for md in (-1.0, 15.5, np.nan):
            refused(point(md), -2, c_sent)
            assert b"max_distance" in L.vxb_last_error(ctx.h)
            assert L.vxb_mesh_closest_point_cut_device(mesh.h, cp, 4.0, md, C.c_void_p(8), 1, C.c_void_p(8)) == -2, md
        for factor in (1.999, np.nan, np.inf):
            refused(sweep(factor=factor), -2, s_sent)
            assert b"lod_factor" in L.vxb_last_error(ctx.h)
            refused(point(factor=factor), -2, c_sent)
        for bad in ((np.nan, 1, 1), (1, np.inf, 1)):
            refused(sweep(camera=bad), -2, s_sent)
            assert b"lod_camera" in L.vxb_last_error(ctx.h)
            refused(point(camera=bad), -2, c_sent)
        # the cut fault wins over the radius fault
        refused(sweep(r=0.0, factor=1.0), -2, s_sent)
        assert b"lod_factor" in L.vxb_last_error(ctx.h)
        # an invalid sweep or point, named by its index
        r = good.copy(); r["direction"][2, 2] = np.nan
        refused(sweep(rays=r), -2, s_sent)
        assert b"sweep 2" in L.vxb_last_error(ctx.h)
        p = pts.copy(); p[1, 1] = np.inf
        refused(point(p=p), -2, c_sent)
        assert b"point 1" in L.vxb_last_error(ctx.h)
        # NULL pointers with count > 0; count = 0 is a no-op
        refused(sweep(rays=None, count=4), -2, s_sent)
        refused(sweep(camera=None), -2, s_sent)
        assert sweep(fresh=False)[0] == -2
        refused(point(p=None, count=4), -2, c_sent)
        refused(point(camera=None), -2, c_sent)
        assert point(fresh=False)[0] == -2
        assert L.vxb_mesh_sphere_cast_cut_device(mesh.h, cp, 4.0, 1.0, None, 1, C.c_void_p(8)) == -2
        assert L.vxb_mesh_closest_point_cut_device(mesh.h, cp, 4.0, 1.0, C.c_void_p(8), 1, None) == -2
        for rc_h, sentinel in ((sweep(count=0), s_sent), (point(count=0), c_sent)):
            assert rc_h[0] == 0 and rc_h[1].tobytes() == sentinel.tobytes()
        assert sweep(15.0)[0] == 0 and point(0.0)[0] == 0 and point(15.0)[0] == 0
    finally:
        mesh.close()


@pytest.mark.parametrize("max_levels, flags", [(2, 0), (0, capi.FLAG_NO_TRANSITIONS)])
def test_incomplete_mesh_is_refused(gpu_context, max_levels, flags):
    mesh = _applied_mesh(gpu_context, "terrain128", max_levels=max_levels, flags=flags)
    try:
        sh, ch = np.zeros(4, capi.SPHERE_CUT_HIT_DTYPE), np.zeros(4, capi.CLOSEST_CUT_HIT_DTYPE)
        rays = capi.make_rays([(10, 200, 10)] * 4, [(0, -1, 0)] * 4)
        pts = np.full((4, 3), 10.0, np.float32)
        assert mesh.sphere_cast_cut_rc((40.0, 70.0, 50.0), 4.0, 1.0, rays, sh) == capi.ERR_STATE
        assert mesh.closest_points_cut_rc((40.0, 70.0, 50.0), 4.0, 4.0, pts, ch) == capi.ERR_STATE
        assert not sh.view(np.uint8).any() and not ch.view(np.uint8).any()
        assert (mesh.sphere_cast(1.0, rays)["slot"] != capi.VXB_RAY_MISS).all()              # the level-0 sweep as before
    finally:
        mesh.close()


def test_terrain1024_device_host_and_oracle(gpu_context):
    import torch
    n = 1024
    mesh = _applied_mesh(gpu_context, "terrain1024")
    rng = np.random.RandomState(1025)
    camera, factor = (0.5 * n, 0.6 * n, 0.45 * n), 14.6
    try:
        res = mesh.download()
        rays = camera_rays(res, 1 << 16, rng)
        rt, ht = _to_device(rays), _hit_buffer(len(rays), capi.SPHERE_CUT_HIT_DTYPE)
        torch.cuda.synchronize()
        mesh.sphere_cast_cut_device(camera, factor, 2.0, rt.data_ptr(), len(rays), ht.data_ptr())
        got_s = _read(ht, capi.SPHERE_CUT_HIT_DTYPE)
        pts = (res.verts["pos"][rng.randint(0, len(res.verts), 1 << 16)] + rng.normal(size=(1 << 16, 3)) * 1.5).astype(np.float32)
        pt, hp = _to_device(pts), _hit_buffer(len(pts), capi.CLOSEST_CUT_HIT_DTYPE)
        torch.cuda.synchronize()
        mesh.closest_points_cut_device(camera, factor, 4.0, pt.data_ptr(), len(pts), hp.data_ptr())
        got_p = _read(hp, capi.CLOSEST_CUT_HIT_DTYPE)
        del rt, ht, pt, hp
        torch.cuda.empty_cache()
        hit = got_s["slot"] != capi.VXB_RAY_MISS
        assert hit.mean() > 0.9 and (got_s["level"][hit] > 0).any()
        assert (got_p["slot"] != capi.VXB_RAY_MISS).mean() > 0.9
        assert_same(got_s, mesh.sphere_cast_cut(camera, factor, 2.0, rays), rays, "1024^3 sweeps: device vs host")
        assert_same(got_p, mesh.closest_points_cut(camera, factor, pts, 4.0), pts, "1024^3 points: device vs host")
        d = Drawn(res, camera, factor)
        pick = rng.choice(len(rays), 1024, replace=False)
        assert_same(got_s[pick], oracle.sphere_cast_cut(res, camera, factor, 2.0, rays[pick], d), rays[pick], "1024^3 sweeps: oracle")
        assert_same(got_p[pick], oracle.closest_points_cut(res, camera, factor, pts[pick], 4.0, d), pts[pick], "1024^3 points: oracle")
    finally:
        mesh.close()
