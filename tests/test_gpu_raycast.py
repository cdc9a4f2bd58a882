"""Ray queries against the resident mesh (include/vxb200.h "ray queries"): every field of every hit is bit-identical to the
numpy oracle (tests/raycast_oracle.py) on mesh.download(), for ray sets aimed at the walk's hard cases (block face planes,
block edges and corners, the grid's faces and edges, +-0 direction components, t bounds at the hit, extreme direction
lengths), across edits, after compactions and growth of the mesh, and through the device variant."""
import ctypes as C

import numpy as np
import pytest

import raycast_oracle as oracle
from voxels_b200 import capi
from voxels_b200.capi import Op

pytestmark = pytest.mark.gpu

F = np.float32


def _surface_points(res, count, rng):
    lv = res.level(0)
    return lv.verts["pos"][rng.randint(0, len(lv.verts), size=count)].astype(np.float32)


def camera_rays(res, count, rng):
    """Origins above the grid, towards random level-0 vertices (unnormalised directions)."""
    n = res.n
    o = np.stack([rng.uniform(-n / 4, 5 * n / 4, count), np.full(count, 1.25 * n), rng.uniform(-n / 4, 5 * n / 4, count)], axis=1)
    return capi.make_rays(o, _surface_points(res, count, rng) - o.astype(np.float32))


def random_rays(n, count, rng):
    """Origins in [-n/4, 5n/4]^3 (misses of the grid box, starts inside it), random directions."""
    return capi.make_rays(rng.uniform(-n / 4, 5 * n / 4, (count, 3)), rng.normal(size=(count, 3)))


def axis_rays(n, rng):
    """Axis-aligned rays at integer coordinates: block faces and edges (multiples of 16), the grid's faces and edges (0, n)."""
    coords = sorted({0, 1, 16, 32, n // 2, n - 16, n - 1, n} | set(int(v) for v in rng.randint(0, n + 1, 3)))
    o, d = [], []
    for a in range(3):
        b, c = [x for x in range(3) if x != a]
        for i in coords:
            for j in coords:
                for sign in (1, -1):
                    p = [0.0, 0.0, 0.0]
                    p[b], p[c] = float(i), float(j)
                    p[a] = -3.0 if sign > 0 else n + 3.0
                    q = [0.0, 0.0, 0.0]; q[a] = float(sign)
                    o.append(p); d.append(q)
    return capi.make_rays(o, d)


def face_plane_rays(n, count, rng):
    """Non-axis rays lying in a block face plane (one coordinate a multiple of 16, that direction component 0)."""
    o = rng.uniform(0, n, (count, 3)).astype(np.float32)
    d = rng.normal(size=(count, 3)).astype(np.float32)
    axis = rng.randint(0, 3, count)
    o[np.arange(count), axis] = 16.0 * rng.randint(0, n // 16 + 1, count)
    d[np.arange(count), axis] = 0.0
    return capi.make_rays(o, d)


def corner_rays(n, count, rng):
    """Diagonal rays through block corners (and along block edges' diagonals: one component 0)."""
    corner = 16.0 * rng.randint(0, n // 16 + 1, (count, 3))
    d = rng.choice([-1.0, 1.0], (count, 3))
    d[rng.rand(count) < 0.25, rng.randint(0, 3)] = 0.0
    d[(d == 0).all(axis=1), 0] = 1.0
    s = rng.uniform(1, n / 2, count)[:, None]
    return capi.make_rays(corner - s * d, d)


def signed_zero_rays(n, rng):
    o, d = [], []
    for k in range(64):
        x, z = (float(v) for v in rng.randint(0, n + 1, 2)) if k % 2 else rng.uniform(0, n, 2)
        o.append((x, n + 2.0, z))
        d.append((-0.0 if k & 2 else 0.0, -1.0, -0.0 if k & 4 else 0.0))
    return capi.make_rays(o, d)


def bound_rays(res, rays, want):
    """Both bounds are inclusive: t_max = first hit and nextafter(first hit, -inf); t_min = first hit and nextafter(first hit,
    +inf)."""
    h = want["slot"] != capi.VXB_RAY_MISS
    base, t = rays[h], want["t"][h]
    a, b, c, e = base.copy(), base.copy(), base.copy(), base.copy()
    a["t_max"] = np.nextafter(t, F(-np.inf))
    b["t_min"] = t
    c["t_min"] = np.nextafter(t, F(np.inf))
    e["t_max"] = t
    return np.concatenate([a, b, c, e])


def scaled_rays(rays, scale):
    r = rays.copy()
    r["direction"] *= F(scale)
    return r


def ray_sets(res, rng, per_set=256):
    n = res.n
    cam = camera_rays(res, per_set, rng)
    lv = oracle.Level0(res)
    cam_want = oracle.raycast(res, cam, lv)
    return lv, {
        "random": random_rays(n, per_set, rng),
        "camera": cam,
        "axis": axis_rays(n, rng),
        "face_plane": face_plane_rays(n, per_set, rng),
        "corners": corner_rays(n, per_set, rng),
        "signed_zero": signed_zero_rays(n, rng),
        "t_bounds": bound_rays(res, cam, cam_want),
        "short": scaled_rays(cam[:64], 1e-3),
        "long": scaled_rays(cam[:64], 1e3),
    }


def assert_same(got, want, rays, what):
    bad = oracle.same_hits(got, want)
    if len(bad):
        k = bad[0]
        raise AssertionError("%s: %d of %d rays differ; first: ray %s\n  got  %s\n  want %s"
                             % (what, len(bad), len(rays), rays[k], got[k], want[k]))


def _fill(ctx, name):
    import grids
    if name.startswith("terrain"):
        n = int(name[len("terrain"):])
        ctx.fill(n, capi.Surface.terrain(n))
    else:
        ctx.upload_dense(*grids.by_name(name))


@pytest.mark.parametrize("name", ["terrain128", "terrain256", "sphere64", "hostile64", "patchwork128"])
def test_ray_sets_equal_oracle(gpu_context, name):
    ctx = gpu_context
    ctx.set_materials(None, None)
    _fill(ctx, name)
    ctx.polygonize()
    mesh = ctx.mesh()
    try:
        mesh.apply()
        res = mesh.download()
        rng = np.random.RandomState(11)
        lv, sets = ray_sets(res, rng)
        hits_total = 0
        for set_name, rays in sets.items():
            got = mesh.raycast(rays)
            assert_same(got, oracle.raycast(res, rays, lv), rays, "%s %s" % (name, set_name))
            hits_total += int((got["slot"] != capi.VXB_RAY_MISS).sum())
        assert hits_total > 0
        # the camera rays hit (they aim at surface vertices), the t-bound set has misses and hits
        assert (mesh.raycast(sets["camera"])["slot"] != capi.VXB_RAY_MISS).mean() > 0.9
    finally:
        mesh.close()


def _brush(i, r):
    if i % 3 == 0:
        return [Op.sphere(r)]
    if i % 3 == 1:
        return [Op.box((r, r, r))]
    return [Op.box((0.6 * r, 0.4 * r, r)), Op.sphere(r), Op.smooth_union(1.5)]


def test_terrain_brush_edits_equal_oracle_and_land_in_the_brush_box(gpu_context):
    n = 128
    ctx = gpu_context
    ctx.set_materials(None, None)
    ctx.fill(n, capi.Surface.terrain(n))
    ctx.polygonize()
    mesh = ctx.mesh()
    rng = np.random.RandomState(21)
    try:
        mesh.apply()
        for edit in range(25):
            # a sculpting tool's round: pick the surface under a cursor ray from above, put the brush at the hit, re-polygonize
            x, z = rng.uniform(16, n - 16, 2)
            pick = capi.make_rays([(x, n + 8.0, z)], [(0, -1, 0)])
            p = mesh.raycast(pick)
            assert p["slot"][0] != capi.VXB_RAY_MISS
            hit = p["position"][0]
            r = float(rng.choice([4, 6, 8]))
            pos, ext = np.array([hit[0], hit[2], hit[1]], np.float32), np.full(3, 2 * r + 4, np.float32)   # grid (x, y, z) = output (x, z, y)
            box = ctx.inject_program(pos, ext, _brush(edit, r), 0 if edit % 2 == 0 else 2)
            ctx.polygonize_region(box[:3], box[3:])
            mesh.apply()
            res = mesh.download()
            lv = oracle.Level0(res)
            rays = np.concatenate([pick, random_rays(n, 128, rng), camera_rays(res, 256, rng), corner_rays(n, 64, rng),
                                   face_plane_rays(n, 64, rng)])
            got = mesh.raycast(rays)
            assert_same(got, oracle.raycast(res, rays, lv), rays, "edit %d" % edit)
            # the same cursor ray now lands on the brush: inside the box the edit returned
            lo, hi = box[:3], box[3:]
            assert got["slot"][0] != capi.VXB_RAY_MISS, "edit %d: the pick ray misses after the edit" % edit
            assert (got["position"][0] >= lo).all() and (got["position"][0] <= hi).all(), (edit, got[0], box)
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
            rays = np.concatenate([random_rays(n, 96, rng), camera_rays(res, 96, rng), axis_rays(n, rng)[::7], corner_rays(n, 64, rng)])
            assert_same(mesh.raycast(rays), oracle.raycast(res, rays), rays, "edge edit %d" % i)
        info = mesh.info()
        assert info.compactions > 0 and info.growths > 0
    finally:
        ctx.set_launch_limit(0)
        mesh.close()


def _device_cast(mesh, rays):
    """The device variant on torch CUDA tensors; returns the tensor of hits (bytes) after the context's stream is done."""
    import torch
    dev = torch.device("cuda", torch.cuda.current_device())
    rt = torch.from_numpy(rays.view(np.uint8).copy()).to(dev)
    ht = torch.full((len(rays) * capi.RAY_HIT_DTYPE.itemsize,), 0x5A, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize()
    mesh.raycast_device(rt.data_ptr(), len(rays), ht.data_ptr())
    return rt, ht


def _hits_of(ht):
    import torch
    torch.cuda.synchronize()
    return ht.cpu().numpy().view(capi.RAY_HIT_DTYPE).copy()


def test_device_variant_equals_host_and_sees_the_mesh_of_its_queue_position(gpu_context):
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
        _, sets = ray_sets(res, rng, 128)
        rays = np.concatenate(list(sets.values()))
        # invalid rays: misses on the device (the host variant refuses them)
        bad = capi.make_rays([(10, 200, 10)] * 5, [(0, -1, 0), (0, 0, 0), (np.inf, -1, 0), (0, -1, 0), (0, -1, 0)],
                             t_min=[0, 0, 0, np.nan, 5], t_max=[np.inf, np.inf, np.inf, 1, 4])
        bad["origin"][0, 0] = np.nan
        _, ht = _device_cast(mesh, np.concatenate([rays, bad]))
        got = _hits_of(ht)
        assert_same(got[:len(rays)], mesh.raycast(rays), rays, "device vs host")
        miss = np.zeros(len(bad), capi.RAY_HIT_DTYPE); miss["t"] = np.inf; miss["slot"] = capi.VXB_RAY_MISS
        assert_same(got[len(rays):], miss, bad, "invalid rays on the device")
        # a cast queued before an apply sees the mesh before it
        before = mesh.download()
        top = mesh.raycast(capi.make_rays([(64, 2 * n, 64)], [(0, -1, 0)]))
        assert top["slot"][0] != capi.VXB_RAY_MISS
        centre = (64.0, 64.0, float(top["position"][0][1]))                    # grid (x, y, z) of the surface there
        box = ctx.inject_program(centre, (40, 40, 40), [Op.sphere(16)], 2)
        ctx.polygonize_region(box[:3], box[3:])
        o = np.stack([rng.uniform(56, 72, 512), np.full(512, 2.0 * n), rng.uniform(56, 72, 512)], axis=1)
        d = np.stack([rng.uniform(-0.05, 0.05, 512), -np.ones(512), rng.uniform(-0.05, 0.05, 512)], axis=1)
        cam = capi.make_rays(o, d)                                              # down into the crater
        _, ht = _device_cast(mesh, cam)
        mesh.apply()
        old = _hits_of(ht)
        assert_same(old, oracle.raycast(before, cam), cam, "queued before the apply")
        after = mesh.download()
        new = mesh.raycast(cam)
        assert_same(new, oracle.raycast(after, cam), cam, "after the apply")
        assert not np.array_equal(old["t"], new["t"])
    finally:
        mesh.close()


def test_map_follows_a_grid_of_another_size(gpu_context):
    ctx = gpu_context
    ctx.set_materials(None, None)
    mesh = ctx.mesh()
    rng = np.random.RandomState(9)
    try:
        for n in (64, 128, 64):
            ctx.fill(n, capi.Surface.terrain(n))
            ctx.polygonize()
            mesh.apply()
            res = mesh.download()
            rays = np.concatenate([random_rays(n, 256, rng), camera_rays(res, 256, rng), axis_rays(n, rng)[::5]])
            assert_same(mesh.raycast(rays), oracle.raycast(res, rays), rays, "n = %d" % n)
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
        sentinel = np.frombuffer(bytes(range(256)) * 1, np.uint8)[:4 * 48].copy().view(capi.RAY_HIT_DTYPE)

        def call(rays, count=None, hits="fresh"):
            h = sentinel.copy() if hits == "fresh" else hits
            rc = L.vxb_mesh_raycast(mesh.h, None if rays is None else capi._ptr(rays), len(rays) if count is None else count,
                                    None if h is None else capi._ptr(h))
            return rc, h

        rc, h = call(good)
        assert rc == capi.ERR_STATE and h.tobytes() == sentinel.tobytes()                        # nothing applied yet
        assert L.vxb_mesh_raycast_device(mesh.h, C.c_void_p(8), 1, C.c_void_p(8)) == capi.ERR_STATE
        mesh.apply()
        cases = [("origin", 0, np.inf), ("origin", 0, np.nan), ("direction", 1, np.inf), ("direction", 2, np.nan)]
        for field, axis, value in cases:
            r = good.copy(); r[field][2, axis] = value
            rc, h = call(r)
            assert rc == -2 and h.tobytes() == sentinel.tobytes(), (field, value)
            assert b"ray 2" in L.vxb_last_error(ctx.h)
        for change in ({"direction": (0.0, -0.0, 0.0)}, {"t_min": np.nan}, {"t_min": np.inf}, {"t_min": -np.inf},
                       {"t_max": np.nan}, {"t_min": 5.0, "t_max": 4.0}):
            r = good.copy()
            for k, v in change.items():
                r[k][3] = v
            rc, h = call(r)
            assert rc == -2 and h.tobytes() == sentinel.tobytes(), change
            assert b"ray 3" in L.vxb_last_error(ctx.h), change
        rc, _ = call(None, 4)
        assert rc == -2                                                                          # NULL rays
        rc, _ = call(good, None, None)
        assert rc == -2                                                                          # NULL hits
        assert L.vxb_mesh_raycast_device(mesh.h, None, 1, C.c_void_p(8)) == -2
        rc, h = call(good, 0)
        assert rc == 0 and h.tobytes() == sentinel.tobytes()                                     # count = 0: no-op
        assert L.vxb_mesh_raycast(mesh.h, None, 0, None) == 0 and L.vxb_mesh_raycast_device(mesh.h, None, 0, None) == 0
        # t_max = +inf and t_min = -large are valid
        r = good.copy(); r["t_min"] = -1e30
        assert call(r)[0] == 0
    finally:
        mesh.close()


def test_terrain1024_camera_rays_device_host_and_oracle(gpu_context):
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
        _, ht = _device_cast(mesh, rays)
        got = _hits_of(ht)
        del ht
        torch.cuda.empty_cache()
        assert (got["slot"] != capi.VXB_RAY_MISS).mean() > 0.9
        assert_same(got, mesh.raycast(rays), rays, "1024^3 device vs host")
        pick = rng.choice(len(rays), 4096, replace=False)
        assert_same(got[pick], oracle.raycast(res, rays[pick]), rays[pick], "1024^3 oracle")
    finally:
        mesh.close()
