"""Ray queries against the drawn LOD cut (include/vxb200.h "ray queries against the drawn LOD cut"): every field of every hit
is bit-identical to the numpy oracle (tests/raycast_cut_oracle.py) on mesh.download(), for the ray sets of
test_gpu_raycast at the cameras and factors of test_gpu_cut, for rays aimed at drawn transition triangles and at moved
regular triangles, across edits, compaction and growth, through the device variant, with a block whose vertices leave its
lattice box, and at 1024^3.  At lod_factor 1e30 the cast equals vxb_mesh_raycast."""
import ctypes as C

import numpy as np
import pytest

import raycast_cut_oracle as oracle
from test_gpu_cut import FACTORS, GRIDS, _applied_mesh, _brush, _cameras
from test_gpu_raycast import _fill, assert_same, camera_rays, corner_rays, face_plane_rays, random_rays, ray_sets
from voxels_b200 import capi

pytestmark = pytest.mark.gpu

F = np.float32


def _aimed_rays(d, rng, per_class=96):
    """Rays towards the centroids of drawn transition triangles and of regular triangles with a vertex at its secondary
    position, from 3 voxels away along a random direction."""
    targets = []
    for b in range(len(d.slot)):
        if not len(d.tri_pos[b]):
            continue
        pick = np.nonzero(d.moved[b])[0] if d.part[b] == 0 else np.arange(len(d.tri_pos[b]))
        targets += [d.tri_pos[b][k].astype(np.float64).mean(axis=0) for k in pick[:2]]
    if not targets:
        return np.zeros(0, capi.RAY_DTYPE)
    targets = np.array(targets)[rng.permutation(len(targets))[:2 * per_class]]
    off = rng.normal(size=targets.shape)
    off *= 3.0 / np.linalg.norm(off, axis=1, keepdims=True)
    return capi.make_rays(targets + off, -off)


def _classes(d, hits):
    """The part classes that won: 'regular', 'secondary' (a regular triangle with a vertex at sec), 'transition'."""
    where = {(s, p): b for b, (s, p) in enumerate(zip(d.slot, d.part))}
    won = set()
    for h in hits[hits["slot"] != capi.VXB_RAY_MISS]:
        if h["face"] != oracle.REGULAR:
            won.add("transition")
        else:
            won.add("secondary" if d.moved[where[(int(h["slot"]), 0)]][h["triangle"]] else "regular")
    return won


def _check(mesh, res, camera, factor, rays, what, drawn=None):
    d = oracle.Drawn(res, camera, factor) if drawn is None else drawn
    got = mesh.raycast_cut(camera, factor, rays)
    assert_same(got, oracle.raycast_cut(res, camera, factor, rays, d), rays, what)
    return got


def _first48(h):
    return np.ascontiguousarray(h).view(np.uint8).reshape(len(h), -1)[:, :48]


def _same_as_level0(mesh, rays, camera, what):
    got = mesh.raycast_cut(camera, 1e30, rays)
    want = mesh.raycast(rays)
    assert np.array_equal(_first48(got), want.view(np.uint8).reshape(len(want), -1)), what
    hit = got["slot"] != capi.VXB_RAY_MISS
    assert (got["level"] == 0).all() and (got["face"][hit] == oracle.REGULAR).all() and (got["face"][~hit] == 0).all(), what


@pytest.mark.parametrize("name", GRIDS)
def test_ray_sets_equal_oracle(gpu_context, name):
    mesh = _applied_mesh(gpu_context, name)
    try:
        res = mesh.download()
        n = res.n
        rng = np.random.RandomState(17)
        _, sets = ray_sets(res, rng, 64)
        sets["axis"] = sets["axis"][::3]
        rays = np.concatenate(list(sets.values()))
        won = set()
        for factor in FACTORS:
            for c, camera in enumerate(_cameras(n, factor)[::2]):
                d = oracle.Drawn(res, camera, factor)
                got = _check(mesh, res, camera, factor, rays, "%s factor %g camera %d" % (name, factor, c), d)
                assert (got["slot"] != capi.VXB_RAY_MISS).any()
                aimed = _aimed_rays(d, rng)
                if len(aimed):
                    won |= _classes(d, _check(mesh, res, camera, factor, aimed, "%s factor %g camera %d aimed" % (name, factor, c), d))
                if factor == 1e30:
                    _same_as_level0(mesh, rays, camera, "%s camera %d" % (name, c))
        assert "regular" in won, (name, won)
        if name in ("terrain128", "terrain256", "patchwork128"):
            assert {"regular", "secondary", "transition"} <= won, (name, won)
    finally:
        mesh.close()


def test_after_brush_edits(gpu_context):
    n = 128
    ctx = gpu_context
    mesh = _applied_mesh(ctx, "terrain128")
    rng = np.random.RandomState(21)
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
            rays = np.concatenate([random_rays(n, 48, rng), camera_rays(res, 96, rng), corner_rays(n, 32, rng), face_plane_rays(n, 32, rng)])
            camera, factor = _cameras(n, 2.0)[edit % 4], (2.0, 4.0, 14.6)[edit % 3]
            _check(mesh, res, camera, factor, rays, "edit %d" % edit)
    finally:
        mesh.close()


def test_after_compaction_and_growth(gpu_context):
    import gridgen
    n = 128
    ctx = gpu_context
    mesh = _applied_mesh(ctx, "patchwork128", (4096, 4096, 1024, 1024))
    ctx.set_launch_limit(2)
    rng = np.random.RandomState(8)
    try:
        for i, (pos, r, ext, add) in enumerate(gridgen.edge_edit_sequence(n, 12)):
            box = ctx.inject_surface(np.array(pos, F), np.full(3, ext, F), capi.Surface.sphere((0, 0, 0), r), 0 if add else 2)
            ctx.polygonize_region(box[:3], box[3:])
            mesh.apply()
            res = mesh.download()
            rays = np.concatenate([random_rays(n, 64, rng), camera_rays(res, 64, rng), corner_rays(n, 32, rng)])
            _check(mesh, res, _cameras(n, 4.0)[i % 4], (2.0, 4.0)[i % 2], rays, "edge edit %d" % i)
        info = mesh.info()
        assert info.compactions > 0 and info.growths > 0
    finally:
        ctx.set_launch_limit(0)
        mesh.close()


def _device_cast(mesh, camera, factor, rays):
    import torch
    dev = torch.device("cuda", torch.cuda.current_device())
    rt = torch.from_numpy(rays.view(np.uint8).copy()).to(dev)
    ht = torch.full((len(rays) * capi.CUT_HIT_DTYPE.itemsize,), 0x5A, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize()
    mesh.raycast_cut_device(camera, factor, rt.data_ptr(), len(rays), ht.data_ptr())
    return rt, ht


def _hits_of(ht):
    import torch
    torch.cuda.synchronize()
    return ht.cpu().numpy().view(capi.CUT_HIT_DTYPE).copy()


def test_device_variant_equals_host_and_sees_the_mesh_of_its_queue_position(gpu_context):
    from voxels_b200.capi import Op
    n = 128
    ctx = gpu_context
    mesh = _applied_mesh(ctx, "terrain128")
    rng = np.random.RandomState(5)
    camera, factor = (64.0, 150.0, 64.0), 4.0
    try:
        res = mesh.download()
        _, sets = ray_sets(res, rng, 96)
        rays = np.concatenate(list(sets.values()))
        bad = capi.make_rays([(10, 200, 10)] * 5, [(0, -1, 0), (0, 0, 0), (np.inf, -1, 0), (0, -1, 0), (0, -1, 0)],
                             t_min=[0, 0, 0, np.nan, 5], t_max=[np.inf, np.inf, np.inf, 1, 4])
        bad["origin"][0, 0] = np.nan
        _, ht = _device_cast(mesh, camera, factor, np.concatenate([rays, bad]))
        got = _hits_of(ht)
        assert_same(got[:len(rays)], mesh.raycast_cut(camera, factor, rays), rays, "device vs host")
        miss = np.zeros(len(bad), capi.CUT_HIT_DTYPE); miss["t"] = np.inf; miss["slot"] = capi.VXB_RAY_MISS
        assert_same(got[len(rays):], miss, bad, "invalid rays on the device")
        # a cast queued before an apply sees the mesh before it
        before = mesh.download()
        top = mesh.raycast(capi.make_rays([(64, 2 * n, 64)], [(0, -1, 0)]))
        centre = (64.0, 64.0, float(top["position"][0][1]))
        box = ctx.inject_program(centre, (40, 40, 40), [Op.sphere(16)], 2)
        ctx.polygonize_region(box[:3], box[3:])
        o = np.stack([rng.uniform(56, 72, 512), np.full(512, 2.0 * n), rng.uniform(56, 72, 512)], axis=1)
        d = np.stack([rng.uniform(-0.05, 0.05, 512), -np.ones(512), rng.uniform(-0.05, 0.05, 512)], axis=1)
        crater = capi.make_rays(o, d)
        _, ht = _device_cast(mesh, camera, factor, crater)
        mesh.apply()
        old = _hits_of(ht)
        assert_same(old, oracle.raycast_cut(before, camera, factor, crater), crater, "queued before the apply")
        after = mesh.download()
        new = _check(mesh, after, camera, factor, crater, "after the apply")
        assert not np.array_equal(old["t"], new["t"])
    finally:
        mesh.close()


class _DeviceBytes:
    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 3}


def _move_level1_vertex(ctx, voxels):
    """Moves pos.x of the first vertex of the first level-1 block of the context's result `voxels` below its lattice box;
    returns that block's grid coordinate."""
    import torch
    res = ctx.download()
    n = res.n
    r = res.records[np.nonzero((res.records["level"] == 1) & (res.records["vertex_count"] > 0))[0][0]]
    nb = (n // 16) >> 1
    gx = int(r["coord_id"]) % nb
    v = np.zeros(1, capi.VERTEX_DTYPE)
    v[0] = res.verts[int(r["vertex_offset"])]
    v["pos"][0, 0] = F(gx * 32 - voxels)
    verts = ctx.device_arenas()[0]
    torch.cuda.synchronize()
    t = torch.as_tensor(_DeviceBytes(verts + int(r["vertex_offset"]) * capi.VERTEX_DTYPE.itemsize, capi.VERTEX_DTYPE.itemsize), device="cuda")
    t.copy_(torch.from_numpy(v.view(np.uint8).copy()))
    torch.cuda.synchronize()
    return r


def test_excursion_is_measured_and_bounded(gpu_context):
    n = 128
    ctx = gpu_context
    ctx.set_materials(None, None)
    _fill(ctx, "terrain128")
    ctx.polygonize()
    _move_level1_vertex(ctx, 5.0)
    mesh = ctx.mesh()
    rng = np.random.RandomState(12)
    try:
        mesh.apply()
        res = mesh.download()
        _, sets = ray_sets(res, rng, 64)
        rays = np.concatenate(list(sets.values()))
        for factor in (2.0, 4.0, 1e30):
            for camera in _cameras(n, factor)[:3]:
                d = oracle.Drawn(res, camera, factor)
                aimed = _aimed_rays(d, rng, 32)
                _check(mesh, res, camera, factor, np.concatenate([rays, aimed]) if len(aimed) else rays, "excursion 5, factor %g" % factor, d)
        ctx.polygonize()
        _move_level1_vertex(ctx, 20.0)
        mesh.apply()
        hits = np.frombuffer(bytes(range(256)) * 2, np.uint8)[:4 * 56].copy().view(capi.CUT_HIT_DTYPE)
        sentinel = hits.copy()
        rc = mesh.raycast_cut_rc((60.0, 90.0, 60.0), 4.0, rays[:4], hits)
        assert rc == capi.ERR_STATE and hits.tobytes() == sentinel.tobytes()
        assert b"lattice box by" in ctx.L.vxb_last_error(ctx.h)
        ctx.polygonize()
        mesh.apply()
        assert mesh.raycast_cut_rc((60.0, 90.0, 60.0), 4.0, rays[:4], hits) == 0
    finally:
        mesh.close()


def test_refusals_leave_hits_untouched(gpu_context):
    ctx = gpu_context
    L = ctx.L
    n = 64
    ctx.set_materials(None, None)
    ctx.fill(n, capi.Surface.terrain(n))
    ctx.polygonize()
    mesh = ctx.mesh()
    try:
        good = capi.make_rays([(10, 100, 10)] * 4, [(0, -1, 0)] * 4)
        sentinel = np.frombuffer(bytes(range(256)) * 2, np.uint8)[:4 * 56].copy().view(capi.CUT_HIT_DTYPE)
        cam = (20.0, 40.0, 20.0)

        def call(rays=good, camera=cam, factor=4.0, count=None, hits="fresh"):
            h = sentinel.copy() if hits == "fresh" else hits
            return mesh.raycast_cut_rc(camera, factor, rays, h, count), h

        def refused(rc_h, rc):
            assert rc_h[0] == rc and rc_h[1].tobytes() == sentinel.tobytes(), rc_h[0]

        refused(call(), capi.ERR_STATE)                                                  # nothing applied yet
        assert L.vxb_mesh_raycast_cut_device(mesh.h, capi._ptr(np.array(cam, F)), 4.0, C.c_void_p(8), 1, C.c_void_p(8)) == capi.ERR_STATE
        mesh.apply()
        for field, axis, value in [("origin", 0, np.inf), ("direction", 2, np.nan)]:
            r = good.copy(); r[field][2, axis] = value
            refused(call(r), -2)
            assert b"ray 2" in L.vxb_last_error(ctx.h)
        for factor in (1.999, -4.0, np.nan, np.inf):
            refused(call(factor=factor), -2)
            assert b"lod_factor" in L.vxb_last_error(ctx.h)
        for bad in ((np.nan, 1, 1), (1, np.inf, 1)):
            refused(call(camera=bad), -2)
            assert b"lod_camera" in L.vxb_last_error(ctx.h)
        refused(call(rays=None, count=4), -2)
        refused(call(camera=None), -2)
        assert call(hits=None)[0] == -2
        assert L.vxb_mesh_raycast_cut_device(mesh.h, capi._ptr(np.array(cam, F)), 4.0, None, 1, C.c_void_p(8)) == -2
        rc, h = call(count=0)
        assert rc == 0 and h.tobytes() == sentinel.tobytes()
        assert call()[0] == 0
    finally:
        mesh.close()


@pytest.mark.parametrize("max_levels, flags", [(2, 0), (0, capi.FLAG_NO_TRANSITIONS)])
def test_incomplete_mesh_is_refused(gpu_context, max_levels, flags):
    mesh = _applied_mesh(gpu_context, "terrain128", max_levels=max_levels, flags=flags)
    try:
        hits = np.zeros(4, capi.CUT_HIT_DTYPE)
        rays = capi.make_rays([(10, 200, 10)] * 4, [(0, -1, 0)] * 4)
        assert mesh.raycast_cut_rc((40.0, 70.0, 50.0), 4.0, rays, hits) == capi.ERR_STATE
        assert not hits.view(np.uint8).any()
        assert (mesh.raycast(rays)["slot"] != capi.VXB_RAY_MISS).all()                   # the level-0 cast as before
    finally:
        mesh.close()


def test_terrain1024_camera_rays_device_host_and_oracle(gpu_context):
    import torch
    n = 1024
    mesh = _applied_mesh(gpu_context, "terrain1024")
    rng = np.random.RandomState(1024)
    camera, factor = (0.5 * n, 0.6 * n, 0.45 * n), 14.6
    try:
        res = mesh.download()
        rays = camera_rays(res, 1 << 20, rng)
        _, ht = _device_cast(mesh, camera, factor, rays)
        got = _hits_of(ht)
        del ht
        torch.cuda.empty_cache()
        assert (got["slot"] != capi.VXB_RAY_MISS).mean() > 0.9
        assert (got["level"][got["slot"] != capi.VXB_RAY_MISS] > 0).any()
        assert_same(got, mesh.raycast_cut(camera, factor, rays), rays, "1024^3 device vs host")
        pick = rng.choice(len(rays), 4096, replace=False)
        assert_same(got[pick], oracle.raycast_cut(res, camera, factor, rays[pick]), rays[pick], "1024^3 oracle")
    finally:
        mesh.close()
