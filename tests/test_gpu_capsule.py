"""Capsule queries against the resident mesh (include/vxb200.h "capsule queries"): every field of every capsule-sweep and
closest-to-segment hit is bit-identical to the numpy oracle (tests/capsule_oracle.py) on mesh.download(), for half axes
along each axis and oblique, extents at the reach limit, paths on the grown-box planes 16k +- (|h_i| + r), in block face
planes and through corners, +-0 components, t bounds at the contact, scaled directions, starts in contact, segments on
block faces, edges and corners and outside the grid; across edits, compactions and growth, and through the device variants.
Also: h = 0 equals the sphere queries, a capsule's contact comes no later than its spheres', a capsule controller lands at
distance r, every refusal, and 2^20 sweeps at 1024^3."""
import ctypes as C

import numpy as np
import pytest

import capsule_oracle as oracle
import raycast_oracle
from test_gpu_collide import _hit_buffer, _read, _to_device, assert_same, contact_sweeps, point_sets
from test_gpu_raycast import _brush, _fill, camera_rays, corner_rays, face_plane_rays, random_rays, signed_zero_rays
from voxels_b200 import capi
from voxels_b200.capi import Op

pytestmark = pytest.mark.gpu

F = np.float32
# (half axis, radius): each axis, oblique, and the two extents at the reach limit
SHAPES = [((2, 0, 0), 0.5), ((0, 2, 0), 2.0), ((0, 0, 2), 0.5), ((1.5, -1, 2), 2.0), ((-0.75, 0.5, 0.25), 0.5), ((0, 4, 0), 0.5), ((14, 0, 0), 1.0),
          ((0, 7, 0), 8.0)]
PER_SET = {"patchwork128": 3}   # its blocks hold the most triangles: the numpy oracle's cost per query is highest there


def capsules(rays, h, r):
    s = np.zeros(len(rays), capi.CAPSULE_SWEEP_DTYPE)
    s["path"], s["half_axis"], s["radius"] = rays, np.asarray(h, np.float32), F(r)
    return s


def axis_paths(n, g, rng):
    """Axis-aligned paths whose other two coordinates lie on the grown-box planes 16k -+ g_i and on 16k itself."""
    ks = sorted({0, 1, n // 32, n // 16 - 1, n // 16} | set(int(v) for v in rng.randint(0, n // 16 + 1, 2)))
    o, d = [], []
    for a in range(3):
        b, c = [x for x in range(3) if x != a]
        for i in ks[::2]:
            for j in ks[1::2]:
                for oi in (-g[b], 0.0, g[b]):
                    for oj in (-g[c], 0.0, g[c]):
                        sign = 1 if (i + j) % 2 else -1
                        p = [0.0, 0.0, 0.0]
                        p[b], p[c] = 16.0 * i + oi, 16.0 * j + oj
                        p[a] = -g[a] - 3.0 if sign > 0 else n + g[a] + 3.0
                        q = [0.0, 0.0, 0.0]; q[a] = float(sign)
                        o.append(p); d.append(q)
    return capi.make_rays(o, d)


def bound_sweeps(sweeps, want):
    h = (want["slot"] != capi.VXB_RAY_MISS) & (want["flags"] == 0)
    base, t = sweeps[h], want["t"][h]
    a, b, c, e = base.copy(), base.copy(), base.copy(), base.copy()
    a["path"]["t_max"] = np.nextafter(t, F(-np.inf)); b["path"]["t_min"] = t
    c["path"]["t_min"] = np.nextafter(t, F(np.inf)); e["path"]["t_max"] = t
    return np.concatenate([a, b, c, e])


def sweep_sets(res, lv, h, r, rng, per_set=8):
    n = res.n
    g = np.abs(np.asarray(h, np.float64)) + r
    cam = capsules(camera_rays(res, per_set, rng), h, r)
    cam_want = oracle.capsule_cast(res, cam, lv)
    scaled_small, scaled_big = cam[:4].copy(), cam[:4].copy()
    scaled_small["path"]["direction"] *= F(1e-3); scaled_big["path"]["direction"] *= F(1e3)
    return {
        "camera": cam,
        "random": capsules(random_rays(n, per_set, rng), h, r),
        "axis": capsules(axis_paths(n, g, rng), h, r)[rng.randint(0, 27)::27],
        "face_plane": capsules(face_plane_rays(n, per_set, rng), h, r),
        "corners": capsules(corner_rays(n, per_set, rng), h, r),
        "signed_zero": capsules(signed_zero_rays(n, rng)[1::7], h, r),
        "t_bounds": bound_sweeps(cam, cam_want)[::2],
        "scaled": np.concatenate([scaled_small, scaled_big]),
        "in_contact": capsules(contact_sweeps(lv, r, per_set // 2, rng), h, r),
    }


def segment_sets(res, h, md, rng, per_set=6):
    pts = point_sets(res, md, rng, per_set)
    verts = np.concatenate(raycast_oracle.Level0(res).tri_pos).reshape(-1, 3)
    crossing = verts[rng.randint(0, len(verts), size=per_set)] + F(0.25) * np.asarray(h, np.float32)
    return {k: capi.make_segments(v, h) for k, v in list(pts.items()) + [("crossing", crossing)]}


def check_sets(mesh, res, name):
    """Every sweep and segment set of every shape on `mesh` against the oracle; returns the feature classes that won."""
    lv = raycast_oracle.Level0(res)
    rng = np.random.RandomState(29)
    contacts = 0
    seen = set()
    for h, r in SHAPES:
        for set_name, sweeps in sweep_sets(res, lv, h, r, rng, PER_SET.get(name, 8)).items():
            got = mesh.capsule_cast(sweeps)
            cls = []
            assert_same(got, oracle.capsule_cast(res, sweeps, lv, classes=cls), sweeps, "%s h=%s r=%g %s" % (name, h, r, set_name))
            seen.update(c for c in cls if c)
            contacts += int((got["slot"] != capi.VXB_RAY_MISS).sum())
            if set_name == "in_contact":
                assert (got["flags"] == capi.VXB_SPHERE_STARTED_IN_CONTACT).all() and (got["t"] == 0).all()
        hm = float(np.max(np.abs(h)))
        for md in (0.0, 15.0 - hm):
            for set_name, segs in segment_sets(res, h, md, rng, PER_SET.get(name, 8) * 3 // 4).items():
                got = mesh.closest_to_segment(segs, md)
                cls = []
                assert_same(got, oracle.closest_to_segment(res, segs, md, lv, classes=cls), segs, "%s h=%s md=%g %s" % (name, h, md, set_name))
                seen.update(c for c in cls if c)
    assert contacts > 0
    return seen


def _sets_on(ctx, name):
    ctx.set_materials(None, None)
    _fill(ctx, name)
    ctx.polygonize()
    mesh = ctx.mesh()
    try:
        mesh.apply()
        return check_sets(mesh, mesh.download(), name)
    finally:
        mesh.close()


@pytest.mark.parametrize("name", ["terrain256", "sphere64", "hostile64", "patchwork128"])
def test_capsule_and_segment_sets_equal_oracle(gpu_context, name):
    _sets_on(gpu_context, name)


def test_terrain128_sets_equal_oracle_and_every_feature_class_wins(gpu_context):
    """The sets on terrain128, and each feature class of the closest pair and of the sweep gives at least one hit there."""
    seen = _sets_on(gpu_context, "terrain128")
    assert seen >= set(oracle.SWEEP_CLASSES) | set(oracle.PAIR_CLASSES), \
        (set(oracle.SWEEP_CLASSES) | set(oracle.PAIR_CLASSES)) - seen


def _terrain_mesh(ctx, n):
    ctx.set_materials(None, None)
    ctx.fill(n, capi.Surface.terrain(n))
    ctx.polygonize()
    mesh = ctx.mesh()
    mesh.apply()
    return mesh


def test_zero_half_axis_equals_the_sphere_queries(gpu_context):
    n = 128
    mesh = _terrain_mesh(gpu_context, n)
    try:
        res = mesh.download()
        rng = np.random.RandomState(4)
        rays = np.concatenate([camera_rays(res, 1024, rng), random_rays(n, 512, rng), corner_rays(n, 256, rng)])
        for r in (0.5, 2.0, 15.0):
            cap, sph = mesh.capsule_cast(capsules(rays, (0, 0, 0), r)), mesh.sphere_cast(r, rays)
            assert (cap["slot"] != capi.VXB_RAY_MISS).sum() > 500
            for f in ("t", "slot", "block_id", "triangle", "center", "point", "normal", "u", "v", "flags"):
                assert np.array_equal(cap[f].view(np.uint32), sph[f].view(np.uint32)), (r, f)
        pts = np.concatenate(list(point_sets(res, 4.0, rng, 256).values()))
        for md in (0.0, 4.0, 15.0):
            seg, pnt = mesh.closest_to_segment(capi.make_segments(pts, (0, 0, 0)), md), mesh.closest_points(pts, md)
            for f in ("distance", "slot", "block_id", "triangle", "point", "normal", "u", "v"):
                assert np.array_equal(seg[f].view(np.uint32), pnt[f].view(np.uint32)), (md, f)
    finally:
        mesh.close()


def test_capsules_contain_their_spheres(gpu_context):
    """Spheres centred at c + x h, x in {-1, 0, 1}, on the same path touch no earlier than the capsule, up to rounding:
    1e-5 |t| plus 1e-4 voxel along the path.  The absolute term is needed near the start of a path.  The capsule's cap test
    works on the shifted vertices a - h and the sphere's face test on the shifted origin o + h; each is rounded to the ulp of
    the coordinates (2^-17 voxel at 64), so the two contact points differ by a few ulps.  On terrain128 a random path whose
    contact lies 0.017 voxel from its start (t = 0.0115, |d| = 1.5) meets the same triangle through the same face test in
    both: the capsule at t = 0.01147071, the top sphere at 0.01146866, and the float64 first contact is 0.01147101.  The
    sphere is the early one, by 3.5e-6 voxel: above 1e-5 |t|, far below a missed triangle."""
    n = 128
    mesh = _terrain_mesh(gpu_context, n)
    try:
        res = mesh.download()
        rng = np.random.RandomState(6)
        rays = np.concatenate([camera_rays(res, 1024, rng), random_rays(n, 512, rng)])
        speed = np.linalg.norm(rays["direction"].astype(np.float64), axis=1)
        for h, r in ((np.array([3.0, 0, 0]), 1.0), (np.array([0, 4.0, 0]), 0.5), (np.array([1.0, 2.0, -2.0]), 2.0)):
            cap = mesh.capsule_cast(capsules(rays, h, r))
            for x in (-1.0, 0.0, 1.0):
                moved = rays.copy()
                moved["origin"] = (rays["origin"] + F(x) * h.astype(np.float32)).astype(np.float32)
                sph = mesh.sphere_cast(r, moved)
                hit = sph["slot"] != capi.VXB_RAY_MISS
                assert hit.sum() > 200
                assert (cap["slot"][hit] != capi.VXB_RAY_MISS).all()
                t = sph["t"].astype(np.float64)
                late = hit & ~(cap["t"] <= t + 1e-5 * np.abs(t) + 1e-4 / speed)
                assert not late.any(), (h, r, x, rays[late], cap[late], sph[late])
    finally:
        mesh.close()


def test_capsule_controller_lands_on_the_surface_during_brush_edits(gpu_context):
    """A capsule controller during 25 brush edits on terrain128: sweep down, then closest_to_segment from the landed pose
    gives distance r within 1e-4 r; every edit is checked against the oracle."""
    n = 128
    ctx = gpu_context
    mesh = _terrain_mesh(ctx, n)
    rng = np.random.RandomState(25)
    try:
        for edit in range(25):
            r = float(rng.choice([0.5, 1.5, 3.0]))
            h = (0.0, float(rng.choice([1.0, 3.0])), 0.0) if edit % 3 else (float(rng.uniform(-2, 2)), 2.0, float(rng.uniform(-2, 2)))
            xz = rng.uniform(16, n - 16, (16, 2))
            down = capi.make_capsule_sweeps(np.stack([xz[:, 0], np.full(16, n + 20.0), xz[:, 1]], axis=1), np.tile([0.0, -1.0, 0.0], (16, 1)), h, r)
            land = mesh.capsule_cast(down)
            assert (land["slot"] != capi.VXB_RAY_MISS).all() and (land["flags"] == 0).all()
            near = mesh.closest_to_segment(capi.make_segments(land["center"], h), 1.001 * r)
            assert (near["slot"] != capi.VXB_RAY_MISS).all()
            assert (np.abs(near["distance"].astype(np.float64) - r) <= 1e-4 * r).all(), (r, h, near["distance"])
            hit = land["point"][0]
            br = float(rng.choice([4, 6, 8]))
            pos, ext = np.array([hit[0], hit[2], hit[1]], np.float32), np.full(3, 2 * br + 4, np.float32)
            box = ctx.inject_program(pos, ext, _brush(edit, br), 0 if edit % 2 == 0 else 2)
            ctx.polygonize_region(box[:3], box[3:])
            mesh.apply()
            res = mesh.download()
            lv = raycast_oracle.Level0(res)
            sweeps = np.concatenate([down, capsules(camera_rays(res, 8, rng), h, r), capsules(corner_rays(n, 4, rng), h, r)])
            assert_same(mesh.capsule_cast(sweeps), oracle.capsule_cast(res, sweeps, lv), sweeps, "edit %d sweeps" % edit)
            segs = capi.make_segments(np.concatenate([land["center"], rng.uniform(0, n, (8, 3)).astype(np.float32)]), h)
            assert_same(mesh.closest_to_segment(segs, 4.0), oracle.closest_to_segment(res, segs, 4.0, lv), segs, "edit %d segments" % edit)
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
            h = (1.0, 2.0, -1.5)
            sweeps = capsules(np.concatenate([random_rays(n, 6, rng), camera_rays(res, 6, rng)]), h, 1.5)
            assert_same(mesh.capsule_cast(sweeps), oracle.capsule_cast(res, sweeps, lv), sweeps, "edge edit %d" % i)
            segs = capi.make_segments(rng.uniform(-4, n + 4, (12, 3)), h)
            assert_same(mesh.closest_to_segment(segs, 6.0), oracle.closest_to_segment(res, segs, 6.0, lv), segs, "edge edit %d segments" % i)
        info = mesh.info()
        assert info.compactions > 0 and info.growths > 0
    finally:
        ctx.set_launch_limit(0)
        mesh.close()


def test_device_variants_equal_host_and_see_the_mesh_of_their_queue_position(gpu_context):
    import torch
    n = 128
    ctx = gpu_context
    mesh = _terrain_mesh(ctx, n)
    rng = np.random.RandomState(5)
    try:
        res = mesh.download()
        lv = raycast_oracle.Level0(res)
        sweeps = np.concatenate(list(sweep_sets(res, lv, (1.0, 2.0, 0.5), 2.0, rng).values()))
        bad = capsules(capi.make_rays([(10, 200, 10)] * 7, [(0, -1, 0)] * 7), (0, 1, 0), 1.0)
        bad["path"]["direction"][0] = 0.0
        bad["path"]["origin"][1, 0] = np.nan
        bad["half_axis"][2, 1] = np.inf
        bad["half_axis"][3, 2] = np.nan
        bad["half_axis"][4] = (14.5, 0, 0)
        bad["radius"][5] = 0.0
        bad["radius"][6] = np.nan
        every = np.concatenate([sweeps, bad])
        st, ht = _to_device(every), _hit_buffer(len(every), capi.CAPSULE_HIT_DTYPE)
        torch.cuda.synchronize()
        mesh.capsule_cast_device(st.data_ptr(), len(every), ht.data_ptr())
        got = _read(ht, capi.CAPSULE_HIT_DTYPE)
        assert_same(got[:len(sweeps)], mesh.capsule_cast(sweeps), sweeps, "capsules: device vs host")
        miss = np.zeros(len(bad), capi.CAPSULE_HIT_DTYPE); miss["t"] = np.inf; miss["slot"] = capi.VXB_RAY_MISS
        assert_same(got[len(sweeps):], miss, bad, "invalid capsules on the device")

        segs = np.concatenate(list(segment_sets(res, (0.5, 1.0, -1.0), 4.0, rng, 12).values()))
        bad_s = capi.make_segments([(np.nan, 1, 1), (1, np.inf, 1), (10, 10, 10), (10, 10, 10)], (0, 1, 0))
        bad_s["half_axis"][2] = (0, 11.5, 0)
        bad_s["half_axis"][3, 0] = np.nan
        every = np.concatenate([segs, bad_s])
        pt, hp = _to_device(every), _hit_buffer(len(every), capi.SEGMENT_HIT_DTYPE)
        torch.cuda.synchronize()
        mesh.closest_to_segment_device(4.0, pt.data_ptr(), len(every), hp.data_ptr())
        got = _read(hp, capi.SEGMENT_HIT_DTYPE)
        assert_same(got[:len(segs)], mesh.closest_to_segment(segs, 4.0), segs, "segments: device vs host")
        miss = np.zeros(len(bad_s), capi.SEGMENT_HIT_DTYPE); miss["distance"] = np.inf; miss["slot"] = capi.VXB_RAY_MISS
        assert_same(got[len(segs):], miss, bad_s, "invalid segments on the device")

        # queries queued before an apply see the mesh before it
        before = mesh.download()
        top = mesh.raycast(capi.make_rays([(64, 2 * n, 64)], [(0, -1, 0)]))
        y = float(top["position"][0][1])
        box = ctx.inject_program((64.0, 64.0, y), (40, 40, 40), [Op.sphere(16)], 2)
        ctx.polygonize_region(box[:3], box[3:])
        o = np.stack([rng.uniform(56, 72, 256), np.full(256, 2.0 * n), rng.uniform(56, 72, 256)], axis=1)
        down = capi.make_capsule_sweeps(o, np.tile([0.0, -1.0, 0.0], (256, 1)), (0, 1.5, 0), 1.0)
        crater = capi.make_segments(np.stack([o[:, 0], np.full(256, y), o[:, 2]], axis=1), (0, 1.5, 0))
        st, ht = _to_device(down), _hit_buffer(len(down), capi.CAPSULE_HIT_DTYPE)
        pt, hp = _to_device(crater), _hit_buffer(len(crater), capi.SEGMENT_HIT_DTYPE)
        torch.cuda.synchronize()
        mesh.capsule_cast_device(st.data_ptr(), len(down), ht.data_ptr())
        mesh.closest_to_segment_device(8.0, pt.data_ptr(), len(crater), hp.data_ptr())
        mesh.apply()
        old_s, old_p = _read(ht, capi.CAPSULE_HIT_DTYPE), _read(hp, capi.SEGMENT_HIT_DTYPE)
        assert_same(old_s, oracle.capsule_cast(before, down), down, "capsules queued before the apply")
        assert_same(old_p, oracle.closest_to_segment(before, crater, 8.0), crater, "segments queued before the apply")
        after = mesh.download()
        new_s, new_p = mesh.capsule_cast(down), mesh.closest_to_segment(crater, 8.0)
        assert_same(new_s, oracle.capsule_cast(after, down), down, "capsules after the apply")
        assert_same(new_p, oracle.closest_to_segment(after, crater, 8.0), crater, "segments after the apply")
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
        good = capi.make_capsule_sweeps([(10, 100, 10)] * 4, [(0, -1, 0)] * 4, (0, 2, 0), 1.0)
        segs = capi.make_segments(np.full((4, 3), 10.0), (0, 2, 0))
        c_sent = np.frombuffer(bytes(range(256)) * 2, np.uint8)[:4 * 80].copy().view(capi.CAPSULE_HIT_DTYPE)
        s_sent = np.frombuffer(bytes(range(256)), np.uint8)[:4 * 64].copy().view(capi.SEGMENT_HIT_DTYPE)

        def sweep(sw, count=None, fresh=True):
            h = c_sent.copy() if fresh else None
            return mesh.capsule_cast_rc(sw, h, count), h

        def segment(md, sg, count=None, fresh=True):
            h = s_sent.copy() if fresh else None
            return mesh.closest_to_segment_rc(md, sg, h, count), h

        def untouched(h, sentinel):
            return h is None or h.tobytes() == sentinel.tobytes()

        rc, h = sweep(good)
        assert rc == capi.ERR_STATE and untouched(h, c_sent)
        rc, h = segment(1.0, segs)
        assert rc == capi.ERR_STATE and untouched(h, s_sent)
        assert L.vxb_mesh_capsule_cast_device(mesh.h, C.c_void_p(8), 1, C.c_void_p(8)) == capi.ERR_STATE
        assert L.vxb_mesh_closest_to_segment_device(mesh.h, 1.0, C.c_void_p(8), 1, C.c_void_p(8)) == capi.ERR_STATE
        mesh.apply()
        assert sweep(good)[0] == 0 and segment(1.0, segs)[0] == 0
        for md in (-1.0, 15.0001, np.nan, np.inf):
            rc, h = segment(md, segs)
            assert rc == -2 and untouched(h, s_sent), md
            assert L.vxb_mesh_closest_to_segment_device(mesh.h, md, C.c_void_p(8), 1, C.c_void_p(8)) == -2, md
        assert segment(13.0, segs)[0] == 0 and segment(13.0001, segs)[0] == -2 and segment(0.0, segs)[0] == 0
        # invalid sweeps, named by their index
        cases = [("path.origin", 0, np.inf), ("path.direction", 2, np.nan), ("half_axis", 1, np.nan), ("half_axis", 0, np.inf)]
        for field, axis, value in cases:
            sw = good.copy()
            if field.startswith("path."):
                sw["path"][field[5:]][2, axis] = value
            else:
                sw[field][2, axis] = value
            rc, h = sweep(sw)
            assert rc == -2 and untouched(h, c_sent) and b"sweep 2" in L.vxb_last_error(ctx.h), field
        for edit in ("zero_direction", "t_order", "radius0", "radius_nan", "reach"):
            sw = good.copy()
            if edit == "zero_direction":
                sw["path"]["direction"][3] = 0.0
            elif edit == "t_order":
                sw["path"]["t_min"][3], sw["path"]["t_max"][3] = 5.0, 4.0
            elif edit == "radius0":
                sw["radius"][3] = 0.0
            elif edit == "radius_nan":
                sw["radius"][3] = np.nan
            else:
                sw["half_axis"][3] = (0, 14.5, 0)
            rc, h = sweep(sw)
            assert rc == -2 and untouched(h, c_sent) and b"sweep 3" in L.vxb_last_error(ctx.h), edit
        at_limit = good.copy(); at_limit["half_axis"][:] = (14, 0, 0)
        assert sweep(at_limit)[0] == 0
        for value in (np.nan, np.inf, -np.inf):
            sg = segs.copy(); sg["center"][1, 1] = value
            rc, h = segment(1.0, sg)
            assert rc == -2 and untouched(h, s_sent) and b"segment 1" in L.vxb_last_error(ctx.h)
            sg = segs.copy(); sg["half_axis"][1, 0] = value
            rc, h = segment(1.0, sg)
            assert rc == -2 and untouched(h, s_sent) and b"segment 1" in L.vxb_last_error(ctx.h)
        # NULL pointers with count > 0; count = 0 is a no-op
        assert sweep(None, 4)[0] == -2 and sweep(good, None, False)[0] == -2
        assert segment(1.0, None, 4)[0] == -2 and segment(1.0, segs, None, False)[0] == -2
        assert L.vxb_mesh_capsule_cast_device(mesh.h, None, 1, C.c_void_p(8)) == -2
        assert L.vxb_mesh_closest_to_segment_device(mesh.h, 1.0, C.c_void_p(8), 1, None) == -2
        rc, h = sweep(good, 0)
        assert rc == 0 and untouched(h, c_sent)
        rc, h = segment(1.0, segs, 0)
        assert rc == 0 and untouched(h, s_sent)
        assert L.vxb_mesh_capsule_cast(mesh.h, None, 0, None) == 0 and L.vxb_mesh_closest_to_segment(mesh.h, 1.0, None, 0, None) == 0
        assert L.vxb_mesh_capsule_cast_device(mesh.h, None, 0, None) == 0
        assert L.vxb_mesh_closest_to_segment_device(mesh.h, 1.0, None, 0, None) == 0
    finally:
        mesh.close()


def test_terrain1024_capsules_device_host_and_oracle(gpu_context):
    import torch
    n = 1024
    mesh = _terrain_mesh(gpu_context, n)
    rng = np.random.RandomState(1024)
    try:
        res = mesh.download()
        sweeps = capsules(camera_rays(res, 1 << 20, rng), (0, 2, 0), 1.0)
        st, ht = _to_device(sweeps), _hit_buffer(len(sweeps), capi.CAPSULE_HIT_DTYPE)
        torch.cuda.synchronize()
        mesh.capsule_cast_device(st.data_ptr(), len(sweeps), ht.data_ptr())
        got = _read(ht, capi.CAPSULE_HIT_DTYPE)
        del st, ht
        torch.cuda.empty_cache()
        assert (got["slot"] != capi.VXB_RAY_MISS).mean() > 0.9
        assert_same(got, mesh.capsule_cast(sweeps), sweeps, "1024^3 device vs host")
        pick = rng.choice(len(sweeps), 512, replace=False)
        lv = raycast_oracle.Level0(res)
        assert_same(got[pick], oracle.capsule_cast(res, sweeps[pick], lv), sweeps[pick], "1024^3 oracle")
    finally:
        mesh.close()
