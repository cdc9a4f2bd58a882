"""Capsule queries against the drawn LOD cut (include/vxb200.h "capsule queries against the drawn LOD cut"): every field of
every capsule-sweep and closest-to-segment hit is bit-identical to the numpy oracle (tests/capsule_cut_oracle.py) on
mesh.download(), for the sweep and segment sets of test_gpu_capsule at the cameras and factors of test_gpu_cut and at the cut
reach limit, for queries aimed at drawn transition triangles and at moved regular triangles, across edits, compaction and
growth, through the device variants, with a block whose vertices leave its lattice box, and at 1024^3.  At lod_factor 1e30
the queries equal vxb_mesh_capsule_cast and vxb_mesh_closest_to_segment; at h = 0 they equal the sphere cut queries; a
capsule touches the drawn cut no later than its spheres."""
import ctypes as C

import numpy as np
import pytest

import capsule_cut_oracle as oracle
import capsule_oracle
import collide_cut_oracle
import raycast_oracle
from raycast_cut_oracle import REGULAR, Drawn
from test_gpu_capsule import SHAPES, capsules, segment_sets, sweep_sets
from test_gpu_collide import _hit_buffer, _read, _to_device, assert_same
from test_gpu_collide_cut import _aimed_points
from test_gpu_cut import FACTORS, GRIDS, _applied_mesh, _brush, _cameras
from test_gpu_raycast import _fill, camera_rays, corner_rays, random_rays
from test_gpu_raycast_cut import _aimed_rays, _classes, _move_level1_vertex
from voxels_b200 import capi
from voxels_b200.capi import Op

pytestmark = pytest.mark.gpu

F = np.float32
# the numpy oracle's cost per query is what bounds these sets: terrain128, where every feature class has to win, gets every
# shape of test_gpu_capsule and more queries per set; the other grids every other shape
PER_SET = {"terrain128": 3}


def _e(mesh, res):
    return collide_cut_oracle.excursion(res, mesh.bounds())


def _limit_shape(e):
    """A vertical half axis of 4 and the radius that puts max |h_i| + r at collide_cut_oracle.reach_limit(e), exactly."""
    limit = collide_cut_oracle.reach_limit(e)
    r = F(limit - F(4))
    assert F(4) + r == limit
    return (0.0, 4.0, 0.0), float(r)


def _check_sweeps(mesh, res, camera, factor, sweeps, e, what, d, classes=None):
    got = mesh.capsule_cast_cut(camera, factor, sweeps)
    assert_same(got, oracle.capsule_cast_cut(res, camera, factor, sweeps, e, d, classes=classes), sweeps, what)
    return got


def _check_segments(mesh, res, camera, factor, md, segs, e, what, d, classes=None):
    got = mesh.closest_to_segment_cut(camera, factor, segs, md)
    assert_same(got, oracle.closest_to_segment_cut(res, camera, factor, segs, md, e, d, classes=classes), segs, what)
    return got


def _first(h, nbytes):
    return np.ascontiguousarray(h).view(np.uint8).reshape(len(h), -1)[:, :nbytes]


def _level0_fields(got, want, nbytes, what):
    assert np.array_equal(_first(got, nbytes), want.view(np.uint8).reshape(len(want), -1)), what
    hit = got["slot"] != capi.VXB_RAY_MISS
    assert (got["level"] == 0).all() and (got["face"][hit] == REGULAR).all() and (got["face"][~hit] == 0).all(), what


def _sweep_batch(res, lv, shapes, rng, per_set):
    return np.concatenate([s for h, r in shapes for s in sweep_sets(res, lv, h, r, rng, per_set).values()])


@pytest.mark.parametrize("name", GRIDS)
def test_sweep_and_segment_sets_equal_oracle(gpu_context, name):
    mesh = _applied_mesh(gpu_context, name)
    try:
        res = mesh.download()
        e = _e(mesh, res)
        lv = raycast_oracle.Level0(res)
        rng = np.random.RandomState(23)
        per_set = PER_SET.get(name, 2)
        lim_h, lim_r = _limit_shape(e)
        some = SHAPES if name == "terrain128" else SHAPES[::2]
        shapes = [(h, r) for h, r in some if oracle.cut_reach_ok(h, r, e)] + [(lim_h, lim_r)]   # the host variant refuses the rest
        sweeps = _sweep_batch(res, lv, shapes, rng, per_set)
        limit = float(collide_cut_oracle.reach_limit(e))
        seg_shapes = {0.0: some[:5:2], 2.0: some[:5], limit: [((0, 0, 0), None)], limit - 4.0: [((0, 4, 0), None)]}
        segments = {md: np.concatenate([s for h, _ in shapes if oracle.cut_reach_ok(h, md, e)
                                        for s in segment_sets(res, h, md, rng, per_set).values()])
                    for md, shapes in seg_shapes.items()}
        won_s, won_p, sweep_cls, pair_cls = set(), set(), set(), set()
        for factor in FACTORS:
            for c, camera in enumerate(_cameras(res.n, factor)[:2]):
                d = Drawn(res, camera, factor)
                what = "%s factor %g camera %d" % (name, factor, c)
                if c == 0 and factor == 1e30:
                    # all of level 0 is drawn: the level-0 queries, which test_gpu_capsule holds to their oracle
                    _level0_fields(mesh.capsule_cast_cut(camera, factor, sweeps), mesh.capsule_cast(sweeps), 80, what + " sweeps level 0")
                    for md, segs in segments.items():
                        _level0_fields(mesh.closest_to_segment_cut(camera, factor, segs, md), mesh.closest_to_segment(segs, md), 64,
                                       "%s md=%g level 0" % (what, md))
                elif c == 0:
                    cls = []
                    got = _check_sweeps(mesh, res, camera, factor, sweeps, e, what + " sweeps", d, cls)
                    assert (got["slot"] != capi.VXB_RAY_MISS).any()
                    won_s |= _classes(d, got)
                    sweep_cls.update(x for x in cls if x)
                    for md, segs in segments.items():
                        cls = []
                        got = _check_segments(mesh, res, camera, factor, md, segs, e, "%s md=%g" % (what, md), d, cls)
                        won_p |= _classes(d, got)
                        pair_cls.update(x for x in cls if x)
                aimed = _aimed_rays(d, rng, 12)
                if len(aimed):
                    aimed_sweeps = np.concatenate([capsules(aimed, (0.5, 0, 0), 0.5), capsules(aimed, (0, 0.25, 0.25), 0.25)])
                    won_s |= _classes(d, _check_sweeps(mesh, res, camera, factor, aimed_sweeps, e, what + " aimed sweeps", d))
                near = _aimed_points(d, rng, 12)
                if len(near):
                    segs = capi.make_segments(near, (0.25, 0, 0))
                    won_p |= _classes(d, _check_segments(mesh, res, camera, factor, 2.0, segs, e, what + " aimed segments", d))
        assert "regular" in won_s and "regular" in won_p, (name, won_s, won_p)
        if name in ("terrain128", "terrain256", "patchwork128"):
            assert {"regular", "secondary", "transition"} <= won_s, (name, won_s)
            assert {"regular", "secondary", "transition"} <= won_p, (name, won_p)
        if name == "terrain128":
            want = set(capsule_oracle.SWEEP_CLASSES) | set(capsule_oracle.PAIR_CLASSES)
            assert want <= sweep_cls | pair_cls, want - (sweep_cls | pair_cls)
    finally:
        mesh.close()


def test_zero_half_axis_equals_the_sphere_cut_queries(gpu_context):
    n = 128
    mesh = _applied_mesh(gpu_context, "terrain128")
    try:
        res = mesh.download()
        rng = np.random.RandomState(4)
        rays = np.concatenate([camera_rays(res, 1024, rng), random_rays(n, 512, rng), corner_rays(n, 256, rng)])
        pts = np.concatenate([rng.uniform(-4, n + 4, (256, 3)), res.verts["pos"][rng.randint(0, len(res.verts), 512)] +
                              rng.normal(size=(512, 3))]).astype(np.float32)
        limit = float(collide_cut_oracle.reach_limit(_e(mesh, res)))
        for factor in (2.0, 4.0, 14.6):
            camera = _cameras(n, factor)[0]
            for r in (0.5, 2.0, limit):
                cap, sph = mesh.capsule_cast_cut(camera, factor, capsules(rays, (0, 0, 0), r)), mesh.sphere_cast_cut(camera, factor, r, rays)
                hit = cap["slot"] != capi.VXB_RAY_MISS
                assert hit.sum() > 500
                for f in sph.dtype.names:
                    assert np.array_equal(cap[f].view(np.uint32), sph[f].view(np.uint32)), (factor, r, f)
                assert (cap["s"][hit] == -1.0).all() and np.array_equal(cap["axis_point"][hit], cap["center"][hit])
            for md in (0.0, 4.0, limit):
                seg, pnt = mesh.closest_to_segment_cut(camera, factor, capi.make_segments(pts, (0, 0, 0)), md), mesh.closest_points_cut(camera, factor, pts, md)
                for f in pnt.dtype.names:
                    assert np.array_equal(seg[f].view(np.uint32), pnt[f].view(np.uint32)), (factor, md, f)
                hit = seg["slot"] != capi.VXB_RAY_MISS
                assert (seg["s"][hit] == -1.0).all() and np.array_equal(seg["axis_point"][hit], pts[hit])
    finally:
        mesh.close()


def test_capsules_contain_their_spheres(gpu_context):
    """Against the drawn cut, spheres centred at c + x h, x in {-1, 0, 1}, on the same path touch no earlier than the capsule,
    within the tolerances of test_gpu_capsule.test_capsules_contain_their_spheres (1e-5 |t| plus 1e-4 voxel along the path)."""
    n = 128
    mesh = _applied_mesh(gpu_context, "terrain128")
    try:
        res = mesh.download()
        rng = np.random.RandomState(6)
        rays = np.concatenate([camera_rays(res, 1024, rng), random_rays(n, 512, rng)])
        speed = np.linalg.norm(rays["direction"].astype(np.float64), axis=1)
        for factor, camera in ((2.0, (0.4 * n, 0.3 * n, 0.45 * n)), (4.0, (0.5 * n, 1.5 * n, 0.55 * n))):
            for h, r in ((np.array([3.0, 0, 0]), 1.0), (np.array([0, 4.0, 0]), 0.5), (np.array([1.0, 2.0, -2.0]), 2.0)):
                cap = mesh.capsule_cast_cut(camera, factor, capsules(rays, h, r))
                assert (cap["level"][cap["slot"] != capi.VXB_RAY_MISS] > 0).any()
                for x in (-1.0, 0.0, 1.0):
                    moved = rays.copy()
                    moved["origin"] = (rays["origin"] + F(x) * h.astype(np.float32)).astype(np.float32)
                    sph = mesh.sphere_cast_cut(camera, factor, r, moved)
                    hit = sph["slot"] != capi.VXB_RAY_MISS
                    assert hit.sum() > 200
                    assert (cap["slot"][hit] != capi.VXB_RAY_MISS).all()
                    t = sph["t"].astype(np.float64)
                    late = hit & ~(cap["t"] <= t + 1e-5 * np.abs(t) + 1e-4 / speed)
                    assert not late.any(), (factor, h, r, x, rays[late], cap[late], sph[late])
    finally:
        mesh.close()


def _edit_check(mesh, res, camera, factor, rng, n, what, at_limit):
    """Sweeps and segments against the oracle after an edit; `at_limit` adds shapes at the cut reach limit (their oracle cost
    is the highest: they reach the most triangles)."""
    d = Drawn(res, camera, factor)
    e = _e(mesh, res)
    rays = np.concatenate([random_rays(n, 8, rng), camera_rays(res, 16, rng), corner_rays(n, 4, rng)])
    sweeps = capsules(rays, (0, 2, 0), 1.0)
    if at_limit:
        lim_h, lim_r = _limit_shape(e)
        sweeps = np.concatenate([sweeps, capsules(rays[::2], lim_h, lim_r)])
    _check_sweeps(mesh, res, camera, factor, sweeps, e, what + " sweeps", d)
    pts = np.concatenate([rng.uniform(-4, n + 4, (12, 3)), res.verts["pos"][rng.randint(0, len(res.verts), 20)] + rng.normal(size=(20, 3))])
    segs = capi.make_segments(pts, rng.normal(size=(len(pts), 3)))
    segs["half_axis"] = np.clip(segs["half_axis"], -3, 3)
    for md in (2.0, float(collide_cut_oracle.reach_limit(e)) - 3.0) if at_limit else (2.0,):
        _check_segments(mesh, res, camera, factor, md, segs, e, "%s md=%g" % (what, md), d)


def test_after_brush_edits(gpu_context):
    n = 128
    ctx = gpu_context
    mesh = _applied_mesh(ctx, "terrain128")
    rng = np.random.RandomState(24)
    try:
        for edit in range(8):
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
            _edit_check(mesh, res, camera, factor, rng, n, "edit %d" % edit, True)
    finally:
        mesh.close()


def test_after_compaction_and_growth(gpu_context):
    import gridgen
    n = 128
    ctx = gpu_context
    mesh = _applied_mesh(ctx, "patchwork128", (4096, 4096, 1024, 1024))
    ctx.set_launch_limit(2)
    rng = np.random.RandomState(10)
    try:
        for i, (pos, r, ext, add) in enumerate(gridgen.edge_edit_sequence(n, 12)):
            box = ctx.inject_surface(np.array(pos, F), np.full(3, ext, F), capi.Surface.sphere((0, 0, 0), r), 0 if add else 2)
            ctx.polygonize_region(box[:3], box[3:])
            mesh.apply()
            res = mesh.download()
            _edit_check(mesh, res, _cameras(n, 4.0)[i % 4], (2.0, 4.0)[i % 2], rng, n, "edge edit %d" % i, i % 4 == 3)
        info = mesh.info()
        assert info.compactions > 0 and info.growths > 0
    finally:
        ctx.set_launch_limit(0)
        mesh.close()


def _sentinel(count, dtype):
    return np.frombuffer(bytes(range(256)) * 4, np.uint8)[:count * dtype.itemsize].copy().view(dtype)


def test_excursion_bounds_each_query(gpu_context):
    """A level-1 vertex 5 voxels outside its block: a reach of 10 equals the oracle; a sweep or segment reaching 10.5 is refused
    by the host variant naming its index, e and R, and is a miss on the device variant while the rest of the batch is
    answered; a max_distance of 10.5 (e + m > 15) refuses the whole segment call on both variants; after the next full apply
    the same queries are accepted.  A vertex 20 voxels outside (e + 1/16 > 15) refuses every call."""
    import torch
    n = 128
    ctx = gpu_context
    ctx.set_materials(None, None)
    _fill(ctx, "terrain128")
    ctx.polygonize()
    _move_level1_vertex(ctx, 5.0)
    mesh = ctx.mesh()
    rng = np.random.RandomState(14)
    try:
        mesh.apply()
        res = mesh.download()
        e = _e(mesh, res)
        assert e >= 5.0
        extra = min(10.0, float(collide_cut_oracle.reach_limit(e))) - 2.0   # max |h_i| + r = max |h_i| + max_distance = 10
        rays = np.concatenate([camera_rays(res, 24, rng), random_rays(n, 12, rng)])
        sweeps = capsules(rays, (0, 2, 0), extra)
        pts = np.concatenate([rng.uniform(-4, n + 4, (16, 3)), res.verts["pos"][rng.randint(0, len(res.verts), 24)] + rng.normal(size=(24, 3))])
        segs = capi.make_segments(pts, (0, 2, 0))
        for factor in (2.0, 4.0, 1e30):
            for camera in _cameras(n, factor)[:1 if factor == 1e30 else 2]:
                d = Drawn(res, camera, factor)
                aimed = _aimed_rays(d, rng, 8)
                batch = np.concatenate([sweeps, capsules(aimed, (0, 2, 0), extra)]) if len(aimed) else sweeps
                _check_sweeps(mesh, res, camera, factor, batch, e, "excursion 5, factor %g sweeps" % factor, d)
                _check_segments(mesh, res, camera, factor, extra, segs, e, "excursion 5, factor %g segments" % factor, d)
        camera, factor = (60.0, 90.0, 60.0), 4.0
        far_s, far_g = sweeps[:6].copy(), segs[:6].copy()
        far_s["radius"][3] = 8.5                                       # R = 10.5
        far_g["half_axis"][4] = (0, 2.5, 0)                            # with max_distance 8: R = 10.5
        s_sent, g_sent = _sentinel(6, capi.CAPSULE_CUT_HIT_DTYPE), _sentinel(6, capi.SEGMENT_CUT_HIT_DTYPE)
        sh, gh = s_sent.copy(), g_sent.copy()
        assert mesh.capsule_cast_cut_rc(camera, factor, far_s, sh) == capi.ERR_STATE and sh.tobytes() == s_sent.tobytes()
        err = ctx.L.vxb_last_error(ctx.h)
        assert b"sweep 3" in err and b"(e)" in err and b"10.5" in err and (b"%g" % float(e)) in err, err
        assert mesh.closest_to_segment_cut_rc(camera, factor, 8.0, far_g, gh) == capi.ERR_STATE and gh.tobytes() == g_sent.tobytes()
        err = ctx.L.vxb_last_error(ctx.h)
        assert b"segment 4" in err and b"(e)" in err and b"10.5" in err, err
        # the device variants: a miss for exactly those queries, the oracle's hits for the rest
        d = Drawn(res, camera, factor)
        st, ht = _to_device(far_s), _hit_buffer(6, capi.CAPSULE_CUT_HIT_DTYPE)
        gt, hg = _to_device(far_g), _hit_buffer(6, capi.SEGMENT_CUT_HIT_DTYPE)
        torch.cuda.synchronize()
        mesh.capsule_cast_cut_device(camera, factor, st.data_ptr(), 6, ht.data_ptr())
        mesh.closest_to_segment_cut_device(camera, factor, 8.0, gt.data_ptr(), 6, hg.data_ptr())
        got_s, got_g = _read(ht, capi.CAPSULE_CUT_HIT_DTYPE), _read(hg, capi.SEGMENT_CUT_HIT_DTYPE)
        want_s = oracle.capsule_cast_cut(res, camera, factor, far_s, e, d)
        want_g = oracle.closest_to_segment_cut(res, camera, factor, far_g, 8.0, e, d)
        assert want_s["slot"][3] == capi.VXB_RAY_MISS and want_g["slot"][4] == capi.VXB_RAY_MISS
        assert (np.delete(want_s["slot"], 3) != capi.VXB_RAY_MISS).any()
        assert_same(got_s, want_s, far_s, "device sweeps out of cut reach")
        assert_same(got_g, want_g, far_g, "device segments out of cut reach")
        # the batch reach: e + max_distance > 15 refuses the whole segment call, host and device, before any query is looked at
        zero_g = far_g.copy()
        zero_g["half_axis"] = 0.0
        gh = g_sent.copy()
        assert mesh.closest_to_segment_cut_rc(camera, factor, 10.5, zero_g, gh) == capi.ERR_STATE and gh.tobytes() == g_sent.tobytes()
        err = ctx.L.vxb_last_error(ctx.h)
        assert b"(e)" in err and b"reaches 10.5 (R)" in err and b"segment" not in err.split(b":")[1], err
        gt, hg = _to_device(zero_g), _to_device(g_sent)
        torch.cuda.synchronize()
        cp = capi._ptr(np.array(camera, F))
        assert ctx.L.vxb_mesh_closest_to_segment_cut_device(mesh.h, cp, factor, 10.5, C.c_void_p(gt.data_ptr()), 6,
                                                            C.c_void_p(hg.data_ptr())) == capi.ERR_STATE
        torch.cuda.synchronize()
        assert _read(hg, capi.SEGMENT_CUT_HIT_DTYPE).tobytes() == g_sent.tobytes()
        ctx.polygonize()
        mesh.apply()
        assert mesh.capsule_cast_cut_rc(camera, factor, far_s, sh) == 0
        assert mesh.closest_to_segment_cut_rc(camera, factor, 8.0, far_g, gh) == 0
        res = mesh.download()
        e = _e(mesh, res)
        assert e + F(10.5) <= F(15)
        assert_same(sh, oracle.capsule_cast_cut(res, camera, factor, far_s, e), far_s, "sweeps after the apply")
        assert_same(gh, oracle.closest_to_segment_cut(res, camera, factor, far_g, 8.0, e), far_g, "segments after the apply")
        # an excursion beyond the walk's reach (e + 1/16 > 15) refuses every capsule cut call, host and device
        ctx.polygonize()
        _move_level1_vertex(ctx, 20.0)
        mesh.apply()
        sh, gh = s_sent.copy(), g_sent.copy()
        assert mesh.capsule_cast_cut_rc(camera, factor, far_s[:1], sh) == capi.ERR_STATE and sh.tobytes() == s_sent.tobytes()
        assert b"the walk reaches 15 - 1/16" in ctx.L.vxb_last_error(ctx.h)
        assert mesh.closest_to_segment_cut_rc(camera, factor, 0.0, far_g[:1], gh) == capi.ERR_STATE and gh.tobytes() == g_sent.tobytes()
        assert b"the walk reaches 15 - 1/16" in ctx.L.vxb_last_error(ctx.h)
        st, ht = _to_device(far_s[:1]), _to_device(s_sent)
        torch.cuda.synchronize()
        cp = capi._ptr(np.array(camera, F))
        assert ctx.L.vxb_mesh_capsule_cast_cut_device(mesh.h, cp, factor, C.c_void_p(st.data_ptr()), 1, C.c_void_p(ht.data_ptr())) == capi.ERR_STATE
        torch.cuda.synchronize()
        assert _read(ht, capi.CAPSULE_CUT_HIT_DTYPE).tobytes() == s_sent.tobytes()
    finally:
        mesh.close()


def test_device_variants_equal_host_and_see_the_mesh_of_their_queue_position(gpu_context):
    import torch
    n = 128
    ctx = gpu_context
    mesh = _applied_mesh(ctx, "terrain128")
    rng = np.random.RandomState(7)
    camera, factor = (64.0, 150.0, 64.0), 4.0
    try:
        res = mesh.download()
        sweeps = capsules(np.concatenate([camera_rays(res, 64, rng), random_rays(n, 32, rng)]), (1.0, 0.5, 0), 1.0)
        bad = capsules(capi.make_rays([(10, 200, 10)] * 7, [(0, -1, 0), (0, 0, 0), (np.inf, -1, 0), (0, -1, 0), (0, -1, 0), (0, -1, 0), (0, -1, 0)],
                                      t_min=[0, 0, 0, np.nan, 5, 0, 0], t_max=[np.inf, np.inf, np.inf, 1, 4, np.inf, np.inf]), (0, 1, 0), 1.0)
        bad["path"]["origin"][0, 0] = np.nan
        bad["radius"][5] = 0.0
        bad["half_axis"][6] = (np.nan, 0, 0)
        all_s = np.concatenate([sweeps, bad])
        st, ht = _to_device(all_s), _hit_buffer(len(all_s), capi.CAPSULE_CUT_HIT_DTYPE)
        torch.cuda.synchronize()
        mesh.capsule_cast_cut_device(camera, factor, st.data_ptr(), len(all_s), ht.data_ptr())
        got = _read(ht, capi.CAPSULE_CUT_HIT_DTYPE)
        assert_same(got[:len(sweeps)], mesh.capsule_cast_cut(camera, factor, sweeps), sweeps, "sweeps: device vs host")
        miss = np.zeros(len(bad), capi.CAPSULE_CUT_HIT_DTYPE); miss["t"] = np.inf; miss["slot"] = capi.VXB_RAY_MISS
        assert_same(got[len(sweeps):], miss, bad, "invalid sweeps on the device")

        pts = np.concatenate([rng.uniform(-4, n + 4, (48, 3)), res.verts["pos"][rng.randint(0, len(res.verts), 48)] + rng.normal(size=(48, 3))])
        segs = capi.make_segments(pts, (0, 1.5, 0.5))
        bad_g = capi.make_segments([[np.nan, 1, 1], [1, np.inf, 1], [1, 1, 1]], (0, 1, 0))
        bad_g["half_axis"][2] = (0, np.inf, 0)
        all_g = np.concatenate([segs, bad_g])
        gt, hg = _to_device(all_g), _hit_buffer(len(all_g), capi.SEGMENT_CUT_HIT_DTYPE)
        torch.cuda.synchronize()
        mesh.closest_to_segment_cut_device(camera, factor, 4.0, gt.data_ptr(), len(all_g), hg.data_ptr())
        got = _read(hg, capi.SEGMENT_CUT_HIT_DTYPE)
        assert_same(got[:len(segs)], mesh.closest_to_segment_cut(camera, factor, segs, 4.0), segs, "segments: device vs host")
        miss = np.zeros(len(bad_g), capi.SEGMENT_CUT_HIT_DTYPE); miss["distance"] = np.inf; miss["slot"] = capi.VXB_RAY_MISS
        assert_same(got[len(segs):], miss, bad_g, "invalid segments on the device")

        # queries queued before an apply see the mesh before it
        before = mesh.download()
        e_before = _e(mesh, before)
        top = mesh.raycast(capi.make_rays([(64, 2 * n, 64)], [(0, -1, 0)]))
        centre = (64.0, 64.0, float(top["position"][0][1]))
        box = ctx.inject_program(centre, (40, 40, 40), [Op.sphere(16)], 2)
        ctx.polygonize_region(box[:3], box[3:])
        o = np.stack([rng.uniform(56, 72, 128), np.full(128, 2.0 * n), rng.uniform(56, 72, 128)], axis=1)
        down = capsules(capi.make_rays(o, np.tile([0.0, -1.0, 0.0], (128, 1))), (0, 2, 0), 1.0)
        crater = capi.make_segments(np.stack([o[:, 0], np.full(128, float(top["position"][0][1])), o[:, 2]], axis=1), (0, 2, 0))
        st, ht = _to_device(down), _hit_buffer(len(down), capi.CAPSULE_CUT_HIT_DTYPE)
        gt, hg = _to_device(crater), _hit_buffer(len(crater), capi.SEGMENT_CUT_HIT_DTYPE)
        torch.cuda.synchronize()
        mesh.capsule_cast_cut_device(camera, factor, st.data_ptr(), len(down), ht.data_ptr())
        mesh.closest_to_segment_cut_device(camera, factor, 8.0, gt.data_ptr(), len(crater), hg.data_ptr())
        mesh.apply()
        old_s, old_g = _read(ht, capi.CAPSULE_CUT_HIT_DTYPE), _read(hg, capi.SEGMENT_CUT_HIT_DTYPE)
        assert_same(old_s, oracle.capsule_cast_cut(before, camera, factor, down, e_before), down, "sweeps queued before the apply")
        assert_same(old_g, oracle.closest_to_segment_cut(before, camera, factor, crater, 8.0, e_before), crater, "segments queued before the apply")
        after = mesh.download()
        e_after, d = _e(mesh, after), Drawn(after, camera, factor)
        new_s = _check_sweeps(mesh, after, camera, factor, down, e_after, "sweeps after the apply", d)
        new_g = _check_segments(mesh, after, camera, factor, 8.0, crater, e_after, "segments after the apply", d)
        assert not np.array_equal(old_s["t"], new_s["t"]) and not np.array_equal(old_g["distance"], new_g["distance"])
    finally:
        mesh.close()


def test_refusals_leave_hits_untouched(gpu_context):
    assert capi.CAPSULE_CUT_HIT_DTYPE.itemsize == 88 and capi.SEGMENT_CUT_HIT_DTYPE.itemsize == 72
    ctx = gpu_context
    L = ctx.L
    n = 64
    ctx.set_materials(None, None)
    ctx.fill(n, capi.Surface.terrain(n))
    ctx.polygonize()
    mesh = ctx.mesh()
    try:
        good = capsules(capi.make_rays([(10, 100, 10)] * 4, [(0, -1, 0)] * 4), (0, 1, 0), 1.0)
        segs = capi.make_segments(np.full((4, 3), 10.0), (0, 1, 0))
        s_sent, g_sent = _sentinel(4, capi.CAPSULE_CUT_HIT_DTYPE), _sentinel(4, capi.SEGMENT_CUT_HIT_DTYPE)
        cam = (20.0, 40.0, 20.0)
        cp = capi._ptr(np.array(cam, F))

        def sweep(s=good, camera=cam, factor=4.0, count=None, fresh=True):
            h = s_sent.copy() if fresh else None
            return mesh.capsule_cast_cut_rc(camera, factor, s, h, count), h

        def segment(md=1.0, g=segs, camera=cam, factor=4.0, count=None, fresh=True):
            h = g_sent.copy() if fresh else None
            return mesh.closest_to_segment_cut_rc(camera, factor, md, g, h, count), h

        def refused(rc_h, rc, sentinel):
            assert rc_h[0] == rc and (rc_h[1] is None or rc_h[1].tobytes() == sentinel.tobytes()), rc_h[0]

        refused(sweep(), capi.ERR_STATE, s_sent)                                        # nothing applied yet
        refused(segment(), capi.ERR_STATE, g_sent)
        assert b"nothing applied" in L.vxb_last_error(ctx.h)
        assert L.vxb_mesh_capsule_cast_cut_device(mesh.h, cp, 4.0, C.c_void_p(8), 1, C.c_void_p(8)) == capi.ERR_STATE
        assert L.vxb_mesh_closest_to_segment_cut_device(mesh.h, cp, 4.0, 1.0, C.c_void_p(8), 1, C.c_void_p(8)) == capi.ERR_STATE
        # count = 0 before the first apply is still a state refusal: the state checks come first
        refused(sweep(count=0), capi.ERR_STATE, s_sent)
        mesh.apply()
        assert sweep()[0] == 0 and segment()[0] == 0
        for md in (-1.0, 15.5, np.nan):
            refused(segment(md), -2, g_sent)
            assert b"max_distance" in L.vxb_last_error(ctx.h)
            assert L.vxb_mesh_closest_to_segment_cut_device(mesh.h, cp, 4.0, md, C.c_void_p(8), 1, C.c_void_p(8)) == -2, md
        for factor in (1.999, np.nan, np.inf):
            refused(sweep(factor=factor), -2, s_sent)
            assert b"lod_factor" in L.vxb_last_error(ctx.h)
            refused(segment(factor=factor), -2, g_sent)
            assert L.vxb_mesh_capsule_cast_cut_device(mesh.h, cp, factor, C.c_void_p(8), 1, C.c_void_p(8)) == -2, factor
        for bad in ((np.nan, 1, 1), (1, np.inf, 1)):
            refused(sweep(camera=bad), -2, s_sent)
            assert b"lod_camera" in L.vxb_last_error(ctx.h)
            refused(segment(camera=bad), -2, g_sent)
        # the cut fault wins over the max_distance fault
        refused(segment(md=-1.0, factor=1.0), -2, g_sent)
        assert b"lod_factor" in L.vxb_last_error(ctx.h)
        # the level-0 per-query rule, named by its index
        for field, value, why in (("radius", 0.0, b"radius"), ("radius", np.nan, b"radius"), ("half_axis", (14.5, 0, 0), b"above 15")):
            s = good.copy(); s[field][2] = value
            refused(sweep(s), -2, s_sent)
            assert b"sweep 2" in L.vxb_last_error(ctx.h) and why in L.vxb_last_error(ctx.h)
        s = good.copy(); s["path"]["direction"][1] = 0.0
        refused(sweep(s), -2, s_sent)
        assert b"sweep 1" in L.vxb_last_error(ctx.h)
        g = segs.copy(); g["center"][3, 0] = np.inf
        refused(segment(g=g), -2, g_sent)
        assert b"segment 3" in L.vxb_last_error(ctx.h)
        g = segs.copy(); g["half_axis"][1] = (0, 14.5, 0)
        refused(segment(g=g), -2, g_sent)
        assert b"segment 1" in L.vxb_last_error(ctx.h)
        # NULL pointers with count > 0; count = 0 is a no-op
        refused(sweep(s=None, count=4), -2, s_sent)
        refused(sweep(camera=None), -2, s_sent)
        assert sweep(fresh=False)[0] == -2
        refused(segment(g=None, count=4), -2, g_sent)
        refused(segment(camera=None), -2, g_sent)
        assert segment(fresh=False)[0] == -2
        assert L.vxb_mesh_capsule_cast_cut_device(mesh.h, cp, 4.0, None, 1, C.c_void_p(8)) == -2
        assert L.vxb_mesh_closest_to_segment_cut_device(mesh.h, cp, 4.0, 1.0, C.c_void_p(8), 1, None) == -2
        for rc_h, sentinel in ((sweep(count=0), s_sent), (segment(count=0), g_sent)):
            assert rc_h[0] == 0 and rc_h[1].tobytes() == sentinel.tobytes()
        assert segment(0.0)[0] == 0 and segment(2.0)[0] == 0
    finally:
        mesh.close()


@pytest.mark.parametrize("max_levels, flags", [(2, 0), (0, capi.FLAG_NO_TRANSITIONS)])
def test_incomplete_mesh_is_refused(gpu_context, max_levels, flags):
    mesh = _applied_mesh(gpu_context, "terrain128", max_levels=max_levels, flags=flags)
    try:
        sh, gh = np.zeros(4, capi.CAPSULE_CUT_HIT_DTYPE), np.zeros(4, capi.SEGMENT_CUT_HIT_DTYPE)
        sweeps = capsules(capi.make_rays([(10, 200, 10)] * 4, [(0, -1, 0)] * 4), (0, 1, 0), 1.0)
        segs = capi.make_segments(np.full((4, 3), 10.0), (0, 1, 0))
        assert mesh.capsule_cast_cut_rc((40.0, 70.0, 50.0), 4.0, sweeps, sh) == capi.ERR_STATE
        assert b"lacks levels" in mesh.ctx.L.vxb_last_error(mesh.ctx.h)
        assert mesh.closest_to_segment_cut_rc((40.0, 70.0, 50.0), 4.0, 4.0, segs, gh) == capi.ERR_STATE
        assert not sh.view(np.uint8).any() and not gh.view(np.uint8).any()
        assert (mesh.capsule_cast(sweeps)["slot"] != capi.VXB_RAY_MISS).all()              # the level-0 sweep as before
    finally:
        mesh.close()


def test_terrain1024_device_host_and_oracle(gpu_context):
    import torch
    n = 1024
    mesh = _applied_mesh(gpu_context, "terrain1024")
    rng = np.random.RandomState(1026)
    camera, factor = (0.5 * n, 0.6 * n, 0.45 * n), 14.6
    try:
        res = mesh.download()
        e = _e(mesh, res)
        rays = camera_rays(res, 1 << 16, rng)
        h = rng.normal(size=(len(rays), 3)).astype(np.float32)
        sweeps = capsules(rays, (0, 0, 0), 1.0)
        sweeps["half_axis"] = h
        st, ht = _to_device(sweeps), _hit_buffer(len(sweeps), capi.CAPSULE_CUT_HIT_DTYPE)
        torch.cuda.synchronize()
        mesh.capsule_cast_cut_device(camera, factor, st.data_ptr(), len(sweeps), ht.data_ptr())
        got_s = _read(ht, capi.CAPSULE_CUT_HIT_DTYPE)
        pts = (res.verts["pos"][rng.randint(0, len(res.verts), 1 << 16)] + rng.normal(size=(1 << 16, 3)) * 1.5).astype(np.float32)
        segs = capi.make_segments(pts, np.clip(rng.normal(size=(1 << 16, 3)), -3, 3))
        gt, hg = _to_device(segs), _hit_buffer(len(segs), capi.SEGMENT_CUT_HIT_DTYPE)
        torch.cuda.synchronize()
        mesh.closest_to_segment_cut_device(camera, factor, 4.0, gt.data_ptr(), len(segs), hg.data_ptr())
        got_g = _read(hg, capi.SEGMENT_CUT_HIT_DTYPE)
        del st, ht, gt, hg
        torch.cuda.empty_cache()
        hit = got_s["slot"] != capi.VXB_RAY_MISS
        assert hit.mean() > 0.9 and (got_s["level"][hit] > 0).any()
        assert (got_g["slot"] != capi.VXB_RAY_MISS).mean() > 0.9
        assert_same(got_s, mesh.capsule_cast_cut(camera, factor, sweeps), sweeps, "1024^3 sweeps: device vs host")
        assert_same(got_g, mesh.closest_to_segment_cut(camera, factor, segs, 4.0), segs, "1024^3 segments: device vs host")
        d = Drawn(res, camera, factor)
        pick = rng.choice(len(rays), 128, replace=False)
        assert_same(got_s[pick], oracle.capsule_cast_cut(res, camera, factor, sweeps[pick], e, d), sweeps[pick], "1024^3 sweeps: oracle")
        assert_same(got_g[pick], oracle.closest_to_segment_cut(res, camera, factor, segs[pick], 4.0, e, d), segs[pick], "1024^3 segments: oracle")
    finally:
        mesh.close()
