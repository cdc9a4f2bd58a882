"""Collision queries against the resident mesh (include/vxb200.h "collision queries"): every field of every sphere-sweep and
closest-point hit is bit-identical to the numpy oracle (tests/collide_oracle.py) on mesh.download(), for sweeps and points
aimed at the walk's hard cases (the grown-box boundaries 16k +- r, block face planes, corners, +-0 direction components,
t bounds at the contact, extreme direction lengths, starts in contact, the inclusive max_distance, points outside the grid
box), across edits, after compactions and growth of the mesh, and through the device variants; a sample of the hits is
checked against the float64 reference."""
import ctypes as C

import numpy as np
import pytest

import collide_oracle as oracle
import raycast_oracle
from test_gpu_raycast import _brush, _fill, camera_rays, corner_rays, face_plane_rays, random_rays, signed_zero_rays
from voxels_b200 import capi
from voxels_b200.capi import Op

pytestmark = pytest.mark.gpu

F = np.float32
TOL64 = 2e-3   # voxels: float32 formulas at coordinates up to 1.25 n (n <= 256) against float64


def axis_sweeps(n, r, rng):
    """Axis-aligned sweeps whose other two coordinates lie on the grown-box planes 16k - r, 16k + r and on 16k itself."""
    ks = sorted({0, 1, n // 32, n // 16 - 1, n // 16} | set(int(v) for v in rng.randint(0, n // 16 + 1, 2)))
    offs = (-r, 0.0, r)
    o, d = [], []
    for a in range(3):
        b, c = [x for x in range(3) if x != a]
        for i in ks:
            for j in ks[::2]:
                for oi in offs:
                    for oj in offs:
                        sign = 1 if (i + j) % 2 else -1
                        p = [0.0, 0.0, 0.0]
                        p[b], p[c] = 16.0 * i + oi, 16.0 * j + oj
                        p[a] = -r - 3.0 if sign > 0 else n + r + 3.0
                        q = [0.0, 0.0, 0.0]; q[a] = float(sign)
                        o.append(p); d.append(q)
    return capi.make_rays(o, d)


def contact_sweeps(lv, r, count, rng):
    """Origins within r / 2 of a vertex of a level-0 triangle (the sweep starts in contact), random directions."""
    tris = np.concatenate(lv.tri_pos)
    v = tris[rng.randint(0, len(tris), size=count), rng.randint(0, 3, size=count)].astype(np.float64)
    off = rng.normal(size=(count, 3)); off *= (0.5 * r / np.linalg.norm(off, axis=1))[:, None]
    return capi.make_rays(v + off, rng.normal(size=(count, 3)))


def bound_sweeps(rays, want):
    """t_max = first contact and one ulp below it; t_min = first contact and one ulp above it."""
    h = (want["slot"] != capi.VXB_RAY_MISS) & (want["flags"] == 0)
    base, t = rays[h], want["t"][h]
    a, b, c, e = base.copy(), base.copy(), base.copy(), base.copy()
    a["t_max"] = np.nextafter(t, F(-np.inf)); b["t_min"] = t; c["t_min"] = np.nextafter(t, F(np.inf)); e["t_max"] = t
    return np.concatenate([a, b, c, e])


def scaled(rays, s):
    r = rays.copy()
    r["direction"] *= F(s)
    return r


def sweep_sets(res, r, rng, per_set=48):
    n = res.n
    lv = raycast_oracle.Level0(res)
    cam = camera_rays(res, per_set, rng)
    cam_want = oracle.sphere_cast(res, r, cam, lv)
    return lv, {
        "camera": cam,
        "random": random_rays(n, per_set, rng),
        "axis": axis_sweeps(n, r, rng)[::3],
        "face_plane": face_plane_rays(n, per_set, rng),
        "corners": corner_rays(n, per_set, rng),
        "signed_zero": signed_zero_rays(n, rng)[::2],
        "t_bounds": bound_sweeps(cam, cam_want)[::2],
        "short": scaled(cam[:16], 1e-3),
        "long": scaled(cam[:16], 1e3),
        "in_contact": contact_sweeps(lv, r, per_set // 2, rng),
    }


def point_sets(res, md, rng, per_set=48):
    n = res.n
    verts = np.concatenate(raycast_oracle.Level0(res).tri_pos).reshape(-1, 3)   # vertices of level-0 triangles
    pick = verts[rng.randint(0, len(verts), size=per_set)]
    snapped = []
    for k in range(1, 4):                            # block faces (one axis), edges (two), corners (three)
        p = pick.copy()
        axes = np.stack([rng.permutation(3)[:k] for _ in range(per_set)])
        for j in range(k):
            p[np.arange(per_set), axes[:, j]] = 16.0 * np.round(p[np.arange(per_set), axes[:, j]] / 16.0)
        snapped.append(p)
    at_md = pick.copy()                              # exactly max_distance from a vertex along an axis
    at_md[np.arange(per_set), rng.randint(0, 3, per_set)] += F(md) * F(rng.choice([-1, 1]))
    edge = verts[(verts < 2).any(axis=1) | (verts > n - 2).any(axis=1)]
    outside = edge[rng.randint(0, max(len(edge), 1), size=per_set)] if len(edge) else pick.copy()
    outside = np.where(outside < 2, outside - F(0.6 * md + 0.25), np.where(outside > n - 2, outside + F(0.6 * md + 0.25), outside))
    return {
        "surface": pick,
        "snapped": np.concatenate(snapped),
        "at_max_distance": at_md,
        "outside_grid": outside.astype(np.float32),
        "random": rng.uniform(-md, n + md, (per_set, 3)).astype(np.float32),
    }


def assert_same(got, want, queries, what):
    bad = oracle.same(got, want)
    if len(bad):
        k = bad[0]
        raise AssertionError("%s: %d of %d queries differ; first: query %s\n  got  %s\n  want %s"
                             % (what, len(bad), len(queries), queries[k], got[k], want[k]))


def _triangle(lv, slot, k):
    b = int(np.nonzero(lv.slots == slot)[0][0])
    return lv.tri_pos[b][k]


def check_sweeps64(res, lv, r, rays, hits, count, rng):
    """A sample of sweep hits against float64: a contact not started in contact is at distance r from its triangle, and no
    triangle comes closer than r - TOL64 to the path before it; a miss never comes closer than r - TOL64."""
    idx = rng.choice(len(rays), min(count, len(rays)), replace=False)
    for i in idx:
        ray, h = rays[i], hits[i]
        if not raycast_oracle.valid_ray(ray):
            continue
        o, d = ray["origin"].astype(np.float64), ray["direction"].astype(np.float64)
        t_hi = float(h["t"]) if h["slot"] != capi.VXB_RAY_MISS else float(ray["t_max"])
        bounds = oracle.segment_bounds64(res.n, o, d, float(ray["t_min"]), t_hi, r + 1.0)
        if h["slot"] != capi.VXB_RAY_MISS:
            dist = oracle.point_triangle_dist64(h["center"], _triangle(lv, h["slot"], h["triangle"])[None])[0]
            if h["flags"]:
                assert dist <= r + TOL64, (ray, h, dist)
                continue
            assert abs(dist - r) <= TOL64, (ray, h, dist)
        if bounds is None:
            continue
        near = raycast_oracle._near_blocks(lv, ray["origin"], ray["direction"], F(bounds[0]), F(bounds[1]), r + 1.0)
        tris = [lv.tri_pos[b] for b in near if len(lv.tri_pos[b])]
        if not tris:
            continue
        _, dmin = oracle.sweep_first_contact64(o, d, bounds[0], bounds[1], r, np.concatenate(tris), iters=60)
        assert dmin.min() >= r - TOL64, (ray, h, dmin.min())


def check_points64(lv, md, points, hits, count, rng):
    idx = rng.choice(len(points), min(count, len(points)), replace=False)
    for i in idx:
        p, h = points[i], hits[i]
        near = oracle._near_point_blocks(lv, p, md + 1.0)
        tris = [lv.tri_pos[b] for b in near if len(lv.tri_pos[b])]
        d64 = oracle.point_triangle_dist64(p, np.concatenate(tris)).min() if tris else np.inf
        if h["slot"] == capi.VXB_RAY_MISS:
            assert d64 >= md - TOL64, (p, d64)
        else:
            assert abs(float(h["distance"]) - d64) <= TOL64, (p, h, d64)


@pytest.mark.parametrize("name", ["terrain128", "terrain256", "sphere64", "hostile64", "patchwork128"])
def test_sweep_and_point_sets_equal_oracle(gpu_context, name):
    ctx = gpu_context
    ctx.set_materials(None, None)
    _fill(ctx, name)
    ctx.polygonize()
    mesh = ctx.mesh()
    try:
        mesh.apply()
        res = mesh.download()
        rng = np.random.RandomState(17)
        contacts = 0
        for r in (0.5, 2.0, 15.0):
            lv, sets = sweep_sets(res, r, rng)
            for set_name, rays in sets.items():
                got = mesh.sphere_cast(r, rays)
                assert_same(got, oracle.sphere_cast(res, r, rays, lv), rays, "%s r=%g %s" % (name, r, set_name))
                contacts += int((got["slot"] != capi.VXB_RAY_MISS).sum())
                if set_name in ("camera", "in_contact", "corners"):
                    check_sweeps64(res, lv, r, rays, got, 6, rng)
            started = mesh.sphere_cast(r, sets["in_contact"])
            assert (started["flags"] == capi.VXB_SPHERE_STARTED_IN_CONTACT).all()
            assert (started["t"] == 0).all()
        assert contacts > 0
        for md in (0.0, 2.0, 15.0):
            for set_name, pts in point_sets(res, md, rng).items():
                got = mesh.closest_points(pts, md)
                assert_same(got, oracle.closest_points(res, pts, md, lv), pts, "%s md=%g %s" % (name, md, set_name))
                if md > 0 and set_name != "surface":
                    check_points64(lv, md, pts, got, 6, rng)
                if set_name == "surface":
                    assert (got["slot"] != capi.VXB_RAY_MISS).all()
                    if md == 0:
                        assert (got["distance"] == 0).all()
        # the bound is inclusive: with max_distance the least float whose square reaches a point's least dd, the point hits;
        # one float below, it misses
        pts = point_sets(res, 4.0, rng, 16)["random"]
        for p in pts:
            tri, _, _ = oracle._gather(lv, oracle._near_point_blocks(lv, p, 16.0))
            if not len(tri):
                continue
            q, _, _, _ = oracle.closest_on_triangles(p, tri)
            dd = oracle.dist2(p, q).min()
            if dd > F(14) * F(14):
                continue
            md = F(np.sqrt(dd))
            while md * md < dd:
                md = np.nextafter(md, F(np.inf))
            while md > 0 and np.nextafter(md, F(0)) * np.nextafter(md, F(0)) >= dd:
                md = np.nextafter(md, F(0))
            at = mesh.closest_points(p[None], float(md))
            assert at["slot"][0] != capi.VXB_RAY_MISS, (p, md, dd)
            assert_same(at, oracle.closest_points(res, p[None], float(md), lv), p[None], "%s at the bound" % name)
            if md > 0:
                below = mesh.closest_points(p[None], float(np.nextafter(md, F(0))))
                assert below["slot"][0] == capi.VXB_RAY_MISS, (p, md, dd)
    finally:
        mesh.close()


def test_sweeps_contain_the_rays(gpu_context):
    """At a radius of 2^-8 voxel, a ray hit implies a sweep contact no later than it (up to 1e-5 |t|)."""
    n = 128
    ctx = gpu_context
    ctx.set_materials(None, None)
    ctx.fill(n, capi.Surface.terrain(n))
    ctx.polygonize()
    mesh = ctx.mesh()
    try:
        mesh.apply()
        res = mesh.download()
        rng = np.random.RandomState(3)
        rays = np.concatenate([camera_rays(res, 2048, rng), random_rays(n, 1024, rng), corner_rays(n, 512, rng)])
        ray_hits = mesh.raycast(rays)
        sweep_hits = mesh.sphere_cast(2.0 ** -8, rays)
        hit = ray_hits["slot"] != capi.VXB_RAY_MISS
        assert hit.sum() > 1000
        assert (sweep_hits["slot"][hit] != capi.VXB_RAY_MISS).all()
        t_ray = ray_hits["t"][hit].astype(np.float64)
        assert (sweep_hits["t"][hit] <= t_ray + 1e-5 * np.abs(t_ray)).all()
    finally:
        mesh.close()


def test_controller_lands_on_the_surface_during_brush_edits(gpu_context):
    """A character controller's round during 25 program-brush edits on terrain128: sweep down onto the surface, then query the
    closest point from the landed centre with max_distance 1.001 r: it is at distance r within 1e-4 r.  Every edit is also
    checked against the oracle."""
    n = 128
    ctx = gpu_context
    ctx.set_materials(None, None)
    ctx.fill(n, capi.Surface.terrain(n))
    ctx.polygonize()
    mesh = ctx.mesh()
    rng = np.random.RandomState(25)
    try:
        mesh.apply()
        for edit in range(25):
            r = float(rng.choice([0.5, 1.5, 3.0]))
            xz = rng.uniform(16, n - 16, (16, 2))
            down = capi.make_rays(np.stack([xz[:, 0], np.full(16, n + 20.0), xz[:, 1]], axis=1), np.tile([0.0, -1.0, 0.0], (16, 1)))
            land = mesh.sphere_cast(r, down)
            assert (land["slot"] != capi.VXB_RAY_MISS).all() and (land["flags"] == 0).all()
            near = mesh.closest_points(land["center"], 1.001 * r)
            assert (near["slot"] != capi.VXB_RAY_MISS).all()
            assert (np.abs(near["distance"].astype(np.float64) - r) <= 1e-4 * r).all(), (r, near["distance"])
            # sculpt at the first landing point, re-polygonize the region, splice it in
            hit = land["point"][0]
            br = float(rng.choice([4, 6, 8]))
            pos, ext = np.array([hit[0], hit[2], hit[1]], np.float32), np.full(3, 2 * br + 4, np.float32)
            box = ctx.inject_program(pos, ext, _brush(edit, br), 0 if edit % 2 == 0 else 2)
            ctx.polygonize_region(box[:3], box[3:])
            mesh.apply()
            res = mesh.download()
            lv = raycast_oracle.Level0(res)
            sweeps = np.concatenate([down, camera_rays(res, 32, rng), corner_rays(n, 16, rng)])
            assert_same(mesh.sphere_cast(r, sweeps), oracle.sphere_cast(res, r, sweeps, lv), sweeps, "edit %d sweeps" % edit)
            pts = np.concatenate([land["center"], land["point"] + F(0.5), rng.uniform(0, n, (16, 3)).astype(np.float32)])
            assert_same(mesh.closest_points(pts, 4.0), oracle.closest_points(res, pts, 4.0, lv), pts, "edit %d points" % edit)
    finally:
        mesh.close()


def test_edge_edits_with_compaction_and_growth_equal_oracle(gpu_context):
    import gridgen
    import grids
    n = 128
    ctx = gpu_context
    ctx.set_materials(None, None)
    ctx.upload_dense(*grids.by_name("patchwork128"))
    ctx.polygonize()
    mesh = ctx.mesh((4096, 4096, 1024, 1024))
    ctx.set_launch_limit(2)
    rng = np.random.RandomState(8)
    try:
        mesh.apply()
        for i, (pos, r, ext, add) in enumerate(gridgen.edge_edit_sequence(n, 12)):
            box = ctx.inject_surface(np.array(pos, np.float32), np.full(3, ext, np.float32), capi.Surface.sphere((0, 0, 0), r), 0 if add else 2)
            ctx.polygonize_region(box[:3], box[3:])
            mesh.apply()
            res = mesh.download()
            lv = raycast_oracle.Level0(res)
            sweeps = np.concatenate([random_rays(n, 32, rng), camera_rays(res, 32, rng), axis_sweeps(n, 2.0, rng)[::17]])
            assert_same(mesh.sphere_cast(2.0, sweeps), oracle.sphere_cast(res, 2.0, sweeps, lv), sweeps, "edge edit %d" % i)
            pts = rng.uniform(-4, n + 4, (64, 3)).astype(np.float32)
            assert_same(mesh.closest_points(pts, 6.0), oracle.closest_points(res, pts, 6.0, lv), pts, "edge edit %d points" % i)
        info = mesh.info()
        assert info.compactions > 0 and info.growths > 0
    finally:
        ctx.set_launch_limit(0)
        mesh.close()


def _to_device(arr):
    import torch
    return torch.from_numpy(arr.view(np.uint8).copy()).to(torch.device("cuda", torch.cuda.current_device()))


def _hit_buffer(count, dtype):
    import torch
    return torch.full((count * dtype.itemsize,), 0x5A, dtype=torch.uint8, device=torch.device("cuda", torch.cuda.current_device()))


def _read(ht, dtype):
    import torch
    torch.cuda.synchronize()
    return ht.cpu().numpy().view(dtype).copy()


def test_device_variants_equal_host_and_see_the_mesh_of_their_queue_position(gpu_context):
    import torch
    n = 128
    ctx = gpu_context
    ctx.set_materials(None, None)
    ctx.fill(n, capi.Surface.terrain(n))
    ctx.polygonize()
    mesh = ctx.mesh()
    rng = np.random.RandomState(5)
    try:
        mesh.apply()
        res = mesh.download()
        _, sets = sweep_sets(res, 2.0, rng, 32)
        rays = np.concatenate(list(sets.values()))
        bad = capi.make_rays([(10, 200, 10)] * 5, [(0, -1, 0), (0, 0, 0), (np.inf, -1, 0), (0, -1, 0), (0, -1, 0)],
                             t_min=[0, 0, 0, np.nan, 5], t_max=[np.inf, np.inf, np.inf, 1, 4])
        bad["origin"][0, 0] = np.nan
        all_rays = np.concatenate([rays, bad])
        rt, ht = _to_device(all_rays), _hit_buffer(len(all_rays), capi.SPHERE_HIT_DTYPE)
        torch.cuda.synchronize()
        mesh.sphere_cast_device(2.0, rt.data_ptr(), len(all_rays), ht.data_ptr())
        got = _read(ht, capi.SPHERE_HIT_DTYPE)
        assert_same(got[:len(rays)], mesh.sphere_cast(2.0, rays), rays, "sweeps: device vs host")
        miss = np.zeros(len(bad), capi.SPHERE_HIT_DTYPE); miss["t"] = np.inf; miss["slot"] = capi.VXB_RAY_MISS
        assert_same(got[len(rays):], miss, bad, "invalid sweeps on the device")

        pts = np.concatenate(list(point_sets(res, 4.0, rng, 32).values()))
        bad_pts = np.array([[np.nan, 1, 1], [1, np.inf, 1], [1, 1, -np.inf]], np.float32)
        all_pts = np.concatenate([pts, bad_pts]).astype(np.float32)
        pt, hp = _to_device(all_pts), _hit_buffer(len(all_pts), capi.CLOSEST_HIT_DTYPE)
        torch.cuda.synchronize()
        mesh.closest_points_device(4.0, pt.data_ptr(), len(all_pts), hp.data_ptr())
        got = _read(hp, capi.CLOSEST_HIT_DTYPE)
        assert_same(got[:len(pts)], mesh.closest_points(pts, 4.0), pts, "points: device vs host")
        miss = np.zeros(len(bad_pts), capi.CLOSEST_HIT_DTYPE); miss["distance"] = np.inf; miss["slot"] = capi.VXB_RAY_MISS
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
        rt, ht = _to_device(down), _hit_buffer(len(down), capi.SPHERE_HIT_DTYPE)
        pt, hp = _to_device(crater), _hit_buffer(len(crater), capi.CLOSEST_HIT_DTYPE)
        torch.cuda.synchronize()
        mesh.sphere_cast_device(1.0, rt.data_ptr(), len(down), ht.data_ptr())
        mesh.closest_points_device(8.0, pt.data_ptr(), len(crater), hp.data_ptr())
        mesh.apply()
        old_s, old_p = _read(ht, capi.SPHERE_HIT_DTYPE), _read(hp, capi.CLOSEST_HIT_DTYPE)
        assert_same(old_s, oracle.sphere_cast(before, 1.0, down), down, "sweeps queued before the apply")
        assert_same(old_p, oracle.closest_points(before, crater, 8.0), crater, "points queued before the apply")
        after = mesh.download()
        new_s, new_p = mesh.sphere_cast(1.0, down), mesh.closest_points(crater, 8.0)
        assert_same(new_s, oracle.sphere_cast(after, 1.0, down), down, "sweeps after the apply")
        assert_same(new_p, oracle.closest_points(after, crater, 8.0), crater, "points after the apply")
        assert not np.array_equal(old_s["t"], new_s["t"]) and not np.array_equal(old_p["distance"], new_p["distance"])
    finally:
        mesh.close()


def test_refusals_leave_hits_untouched(gpu_context):
    ctx = gpu_context
    L = ctx.L
    n = 64
    ctx.fill(n, capi.Surface.terrain(n))
    ctx.polygonize()
    mesh = ctx.mesh()
    try:
        good = capi.make_rays([(10, 100, 10)] * 4, [(0, -1, 0)] * 4)
        pts = np.full((4, 3), 10.0, np.float32)
        s_sent = np.frombuffer(bytes(range(256)), np.uint8)[:4 * 64].copy().view(capi.SPHERE_HIT_DTYPE)
        c_sent = np.frombuffer(bytes(range(256)), np.uint8)[:4 * 48].copy().view(capi.CLOSEST_HIT_DTYPE)

        def sweep(r, rays, count=None, fresh=True):
            h = s_sent.copy() if fresh else None
            return mesh.sphere_cast_rc(r, rays, h, count), h

        def point(md, p, count=None, fresh=True):
            h = c_sent.copy() if fresh else None
            return mesh.closest_points_rc(md, p, h, count), h

        def untouched(h, sentinel):
            return h is None or h.tobytes() == sentinel.tobytes()

        rc, h = sweep(1.0, good)
        assert rc == capi.ERR_STATE and untouched(h, s_sent)                       # nothing applied yet
        rc, h = point(1.0, pts)
        assert rc == capi.ERR_STATE and untouched(h, c_sent)
        assert L.vxb_mesh_sphere_cast_device(mesh.h, 1.0, C.c_void_p(8), 1, C.c_void_p(8)) == capi.ERR_STATE
        assert L.vxb_mesh_closest_point_device(mesh.h, 1.0, C.c_void_p(8), 1, C.c_void_p(8)) == capi.ERR_STATE
        mesh.apply()
        assert sweep(1.0, good)[0] == 0 and point(1.0, pts)[0] == 0
        for r in (0.0, -1.0, 15.0001, np.nan, np.inf):
            rc, h = sweep(r, good)
            assert rc == -2 and untouched(h, s_sent), r
            assert L.vxb_mesh_sphere_cast_device(mesh.h, r, C.c_void_p(8), 1, C.c_void_p(8)) == -2, r
        for md in (-1.0, 15.0001, np.nan, np.inf):
            rc, h = point(md, pts)
            assert rc == -2 and untouched(h, c_sent), md
            assert L.vxb_mesh_closest_point_device(mesh.h, md, C.c_void_p(8), 1, C.c_void_p(8)) == -2, md
        assert sweep(15.0, good)[0] == 0 and point(0.0, pts)[0] == 0 and point(15.0, pts)[0] == 0
        # an invalid sweep or point, named by its index
        for field, axis, value in [("origin", 0, np.inf), ("direction", 2, np.nan)]:
            r = good.copy(); r[field][2, axis] = value
            rc, h = sweep(1.0, r)
            assert rc == -2 and untouched(h, s_sent) and b"sweep 2" in L.vxb_last_error(ctx.h)
        r = good.copy(); r["direction"][3] = 0.0
        rc, h = sweep(1.0, r)
        assert rc == -2 and untouched(h, s_sent) and b"sweep 3" in L.vxb_last_error(ctx.h)
        for value in (np.nan, np.inf, -np.inf):
            p = pts.copy(); p[1, 1] = value
            rc, h = point(1.0, p)
            assert rc == -2 and untouched(h, c_sent) and b"point 1" in L.vxb_last_error(ctx.h)
        # NULL pointers with count > 0; count = 0 is a no-op
        assert sweep(1.0, None, 4)[0] == -2 and sweep(1.0, good, None, False)[0] == -2
        assert point(1.0, None, 4)[0] == -2 and point(1.0, pts, None, False)[0] == -2
        assert L.vxb_mesh_sphere_cast_device(mesh.h, 1.0, None, 1, C.c_void_p(8)) == -2
        assert L.vxb_mesh_closest_point_device(mesh.h, 1.0, C.c_void_p(8), 1, None) == -2
        rc, h = sweep(1.0, good, 0)
        assert rc == 0 and untouched(h, s_sent)
        rc, h = point(1.0, pts, 0)
        assert rc == 0 and untouched(h, c_sent)
        assert L.vxb_mesh_sphere_cast(mesh.h, 1.0, None, 0, None) == 0 and L.vxb_mesh_closest_point(mesh.h, 1.0, None, 0, None) == 0
        assert L.vxb_mesh_sphere_cast_device(mesh.h, 1.0, None, 0, None) == 0
        assert L.vxb_mesh_closest_point_device(mesh.h, 1.0, None, 0, None) == 0
    finally:
        mesh.close()


def test_terrain1024_sweeps_device_host_and_oracle(gpu_context):
    import torch
    n = 1024
    ctx = gpu_context
    ctx.set_materials(None, None)
    ctx.fill(n, capi.Surface.terrain(n))
    ctx.polygonize()
    mesh = ctx.mesh()
    rng = np.random.RandomState(1024)
    try:
        mesh.apply()
        res = mesh.download()
        rays = camera_rays(res, 1 << 20, rng)
        rt, ht = _to_device(rays), _hit_buffer(len(rays), capi.SPHERE_HIT_DTYPE)
        torch.cuda.synchronize()
        mesh.sphere_cast_device(2.0, rt.data_ptr(), len(rays), ht.data_ptr())
        got = _read(ht, capi.SPHERE_HIT_DTYPE)
        del rt, ht
        torch.cuda.empty_cache()
        assert (got["slot"] != capi.VXB_RAY_MISS).mean() > 0.9
        assert_same(got, mesh.sphere_cast(2.0, rays), rays, "1024^3 device vs host")
        pick = rng.choice(len(rays), 4096, replace=False)
        lv = raycast_oracle.Level0(res)
        assert_same(got[pick], oracle.sphere_cast(res, 2.0, rays[pick], lv), rays[pick], "1024^3 oracle")
    finally:
        mesh.close()
