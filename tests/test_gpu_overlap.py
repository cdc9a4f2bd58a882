"""Box overlap gathers against the resident mesh (include/vxb200.h "box overlap gathers"): every offset and every byte of every
record equals the numpy oracle (tests/overlap_oracle.py) on mesh.download(), for boxes on block boundaries, body-sized boxes
at the surface, boxes crossing or outside the grid, the whole grid, degenerate and random boxes; the capacity rules of both
variants; agreement with the closest-point query and coverage of every triangle by a tiling; edits, compaction and growth;
the device variant's queue position; refusals; and 2^16 boxes at 1024^3."""
import ctypes as C

import numpy as np
import pytest

import overlap_oracle as oracle
import raycast_oracle
from test_gpu_raycast import _brush, _fill
from voxels_b200 import capi

pytestmark = pytest.mark.gpu

F = np.float32


def _vertices(res):
    return np.concatenate(raycast_oracle.Level0(res).tri_pos).reshape(-1, 3)


def body_boxes(centres, rng):
    h = rng.uniform(0.5, 3.0, (len(centres), 3)).astype(np.float32)
    c = np.asarray(centres, np.float32)
    return capi.make_boxes(c - h, c + h)


def box_sets(res, mesh, rng, per_set=48):
    n = res.n
    nb = n // 16
    verts = _vertices(res)
    lo = 16 * rng.randint(-1, nb + 1, (per_set, 3))
    hi = lo + 16 * rng.randint(0, 3, (per_set, 3))
    pts = verts[rng.randint(0, len(verts), per_set)] + rng.normal(scale=2.0, size=(per_set, 3)).astype(np.float32)
    near = mesh.closest_points(pts, 4.0)
    near = near["point"][near["slot"] != capi.VXB_RAY_MISS]
    edge = rng.uniform(-6, 6, (per_set, 3)) + rng.randint(0, 2, (per_set, 3)) * n
    v = verts[rng.randint(0, len(verts), per_set)]
    flat_lo, flat_hi = v - 2, v + 2
    axis = rng.randint(0, 3, per_set)
    flat_lo[np.arange(per_set), axis] = flat_hi[np.arange(per_set), axis] = v[np.arange(per_set), axis]
    c = rng.uniform(-8, n + 8, (per_set, 3))
    h = rng.uniform(0, 12, (per_set, 3)) * (rng.uniform(size=(per_set, 3)) > 0.1)
    return {
        "block_faces": capi.make_boxes(lo, hi),
        "body_at_vertices": body_boxes(verts[rng.randint(0, len(verts), per_set)], rng),
        "body_at_closest": body_boxes(near, rng),
        "grid_faces": capi.make_boxes(edge - 5, edge + 5),
        "outside": capi.make_boxes([(-40, 0, 0), (0, n + 1, 0), (n + 5, n + 5, n + 5), (0, 0, -1e30)],
                                   [(-20, n, n), (n, n + 30, n), (n + 30, n + 40, n + 50), (n, n, -17)]),
        "whole_grid": capi.make_boxes([(-1, -1, -1)], [(n + 1, n + 1, n + 1)]),
        "degenerate": np.concatenate([capi.make_boxes(flat_lo, flat_hi), capi.make_boxes(v[:16], v[:16]),
                                      capi.make_boxes([(-3e38, -3e38, -3e38)], [(3e38, 3e38, 3e38)])]),
        "random": capi.make_boxes(c - h, c + h),
    }


def assert_same(got, want, what):
    d = oracle.same(got, want)
    assert d is None, "%s: %s" % (what, d)


@pytest.mark.parametrize("name", ["terrain128", "terrain256", "sphere64", "hostile64", "patchwork128"])
def test_box_sets_equal_oracle(gpu_context, name):
    ctx = gpu_context
    ctx.set_materials(None, None)
    _fill(ctx, name)
    ctx.polygonize()
    mesh = ctx.mesh()
    try:
        mesh.apply()
        res = mesh.download()
        lv = oracle.Level0Sorted(res)
        rng = np.random.RandomState(31)
        found = 0
        for set_name, boxes in box_sets(res, mesh, rng).items():
            got = mesh.overlap_boxes(boxes)
            assert_same(got, oracle.overlap_boxes(res, boxes, lv), "%s %s" % (name, set_name))
            found += int(got[0][-1])
            if set_name in ("body_at_vertices", "whole_grid"):
                assert (np.diff(got[0]) > 0).all(), set_name
        whole = mesh.overlap_boxes(capi.make_boxes([(-1, -1, -1)], [(res.n + 1,) * 3]))
        assert int(whole[0][-1]) == len(lv.tri) and found > 0
    finally:
        mesh.close()


def _to_device(arr):
    import torch
    return torch.from_numpy(arr.view(np.uint8).copy()).to(torch.device("cuda", torch.cuda.current_device()))


def _buffer(nbytes):
    import torch
    return torch.full((max(nbytes, 1),), 0x5A, dtype=torch.uint8, device=torch.device("cuda", torch.cuda.current_device()))


def _read(t, dtype, count):
    import torch
    torch.cuda.synchronize()
    return t.cpu().numpy()[:count * np.dtype(dtype).itemsize].view(dtype).copy()


def _terrain_mesh(ctx, n):
    ctx.set_materials(None, None)
    ctx.fill(n, capi.Surface.terrain(n))
    ctx.polygonize()
    mesh = ctx.mesh()
    mesh.apply()
    return mesh


def test_capacity_on_both_variants(gpu_context):
    ctx = gpu_context
    mesh = _terrain_mesh(ctx, 128)
    try:
        res = mesh.download()
        rng = np.random.RandomState(2)
        boxes = body_boxes(_vertices(res)[rng.randint(0, 1000, 64)], rng)
        want = oracle.overlap_boxes(res, boxes)
        total = int(want[0][-1])
        assert total > 64
        sentinel = np.frombuffer(bytes(range(256)) * (total * 48 // 256 + 1), np.uint8)[:total * 48].copy().view(capi.OVERLAP_TRIANGLE_DTYPE)
        # host: capacity == total fills; total - 1 is refused with the offsets written and tris untouched; count only
        off, tris = np.zeros(len(boxes) + 1, np.uint64), sentinel.copy()
        assert mesh.overlap_boxes_rc(boxes, off, tris, total) == 0
        assert_same((off, tris), want, "capacity == total")
        off, tris = np.zeros(len(boxes) + 1, np.uint64), sentinel.copy()
        assert mesh.overlap_boxes_rc(boxes, off, tris, total - 1) == capi.ERR_CAPACITY
        assert np.array_equal(off, want[0]) and tris.tobytes() == sentinel.tobytes()
        off = np.zeros(len(boxes) + 1, np.uint64)
        assert mesh.overlap_boxes_rc(boxes, off, None, 0) == 0 and np.array_equal(off, want[0])
        # device: the same three, decided on the device
        bt = _to_device(boxes)
        for cap, fills in ((total, True), (total - 1, False), (0, False)):
            ot, tt = _buffer((len(boxes) + 1) * 8), _to_device(sentinel)
            mesh.overlap_boxes_device(bt.data_ptr(), len(boxes), ot.data_ptr(), tt.data_ptr() if cap else None, cap)
            o, t = _read(ot, np.uint64, len(boxes) + 1), _read(tt, capi.OVERLAP_TRIANGLE_DTYPE, total)
            assert np.array_equal(o, want[0]), cap
            if fills:
                assert_same((o, t), want, "device capacity == total")
            else:
                assert t.tobytes() == sentinel.tobytes(), cap
    finally:
        mesh.close()


def test_closest_points_lie_in_their_box_and_a_tiling_covers_every_triangle(gpu_context):
    ctx = gpu_context
    mesh = _terrain_mesh(ctx, 128)
    try:
        res = mesh.download()
        n = res.n
        rng = np.random.RandomState(4)
        verts = _vertices(res)
        for md in (0.5, 3.0, 15.0):
            p = (verts[rng.randint(0, len(verts), 256)] + rng.normal(scale=md, size=(256, 3))).astype(np.float32)
            hits = mesh.closest_points(p, md)
            hit = hits["slot"] != capi.VXB_RAY_MISS
            assert hit.sum() > 64
            g = F(md) + F(1e-3)
            off, tris = mesh.overlap_boxes(capi.make_boxes(p[hit] - g, p[hit] + g))
            for q, h in enumerate(hits[hit]):
                part = tris[int(off[q]):int(off[q + 1])]
                assert ((part["slot"] == h["slot"]) & (part["triangle"] == h["triangle"])).any(), (p[hit][q], md, h)
        for tile in (16, 24, 40):
            lo = np.stack(np.meshgrid(*[np.arange(0, n, tile)] * 3, indexing="ij"), axis=-1).reshape(-1, 3).astype(np.float32)
            off, tris = mesh.overlap_boxes(capi.make_boxes(lo, lo + tile))
            key = tris["slot"].astype(np.int64) << 32 | tris["triangle"]
            lv = oracle.Level0Sorted(res)
            assert len(np.unique(key)) == len(lv.tri), tile
    finally:
        mesh.close()


def test_brush_edits_equal_oracle(gpu_context):
    n = 128
    ctx = gpu_context
    mesh = _terrain_mesh(ctx, n)
    rng = np.random.RandomState(25)
    try:
        for edit in range(25):
            x, z = rng.uniform(16, n - 16, 2)
            p = mesh.raycast(capi.make_rays([(x, n + 8.0, z)], [(0, -1, 0)]))["position"][0]
            br = float(rng.choice([4, 6, 8]))
            pos, ext = np.array([p[0], p[2], p[1]], np.float32), np.full(3, 2 * br + 4, np.float32)
            box = ctx.inject_program(pos, ext, _brush(edit, br), 0 if edit % 2 == 0 else 2)
            ctx.polygonize_region(box[:3], box[3:])
            mesh.apply()
            res = mesh.download()
            boxes = np.concatenate([body_boxes(np.tile(p, (8, 1)) + rng.normal(scale=br, size=(8, 3)).astype(np.float32), rng),
                                    capi.make_boxes([p - 2 * br], [p + 2 * br]), box_sets(res, mesh, rng, 8)["random"]])
            assert_same(mesh.overlap_boxes(boxes), oracle.overlap_boxes(res, boxes), "edit %d" % edit)
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
            p = np.array([pos[0], pos[2], pos[1]], np.float32)
            boxes = np.concatenate([capi.make_boxes([p - ext], [p + ext]), box_sets(res, mesh, rng, 16)["random"],
                                    box_sets(res, mesh, rng, 8)["block_faces"]])
            assert_same(mesh.overlap_boxes(boxes), oracle.overlap_boxes(res, boxes), "edge edit %d" % i)
        info = mesh.info()
        assert info.compactions > 0 and info.growths > 0
    finally:
        ctx.set_launch_limit(0)
        mesh.close()


def test_device_variant_sees_the_mesh_of_its_queue_position_and_invalid_boxes_are_empty(gpu_context):
    from voxels_b200.capi import Op
    n = 128
    ctx = gpu_context
    mesh = _terrain_mesh(ctx, n)
    rng = np.random.RandomState(5)
    try:
        res = mesh.download()
        boxes = np.concatenate(list(box_sets(res, mesh, rng, 16).values()))
        bad = capi.make_boxes([(np.nan, 0, 0), (0, np.inf, 0), (5, 5, 5), (0, 0, 0)], [(n, n, n), (n, n, n), (4, n, n), (n, n, -np.inf)])
        all_boxes = np.concatenate([boxes[:8], bad, boxes[8:]])
        want = mesh.overlap_boxes(all_boxes[np.r_[0:8, 12:len(all_boxes)]])
        bt, ot = _to_device(all_boxes), _buffer((len(all_boxes) + 1) * 8)
        tt = _buffer(int(want[0][-1]) * 48)
        mesh.overlap_boxes_device(bt.data_ptr(), len(all_boxes), ot.data_ptr(), tt.data_ptr(), int(want[0][-1]))
        o, t = _read(ot, np.uint64, len(all_boxes) + 1), _read(tt, capi.OVERLAP_TRIANGLE_DTYPE, int(want[0][-1]))
        assert (np.diff(o)[8:12] == 0).all()
        assert_same((np.delete(o, np.s_[9:13]), t), want, "device with invalid boxes")
        # a gather queued before an apply sees the mesh before it
        top = mesh.raycast(capi.make_rays([(64, 2 * n, 64)], [(0, -1, 0)]))["position"][0]
        crater = capi.make_boxes([top - 12], [top + 12])
        before = mesh.download()
        box = ctx.inject_program((64.0, 64.0, float(top[1])), (40, 40, 40), [Op.sphere(16)], 2)
        ctx.polygonize_region(box[:3], box[3:])
        old_want = oracle.overlap_boxes(before, crater)
        bt, ot, tt = _to_device(crater), _buffer(16), _buffer(int(old_want[0][-1]) * 48)
        mesh.overlap_boxes_device(bt.data_ptr(), 1, ot.data_ptr(), tt.data_ptr(), int(old_want[0][-1]))
        mesh.apply()
        o, t = _read(ot, np.uint64, 2), _read(tt, capi.OVERLAP_TRIANGLE_DTYPE, int(old_want[0][-1]))
        assert_same((o, t), old_want, "queued before the apply")
        after = mesh.overlap_boxes(crater)
        assert_same(after, oracle.overlap_boxes(mesh.download(), crater), "after the apply")
        assert oracle.same(after, old_want) is not None
    finally:
        mesh.close()


def test_refusals_leave_offsets_and_tris_untouched(gpu_context):
    ctx = gpu_context
    L = ctx.L
    n = 64
    ctx.fill(n, capi.Surface.terrain(n))
    ctx.polygonize()
    mesh = ctx.mesh()
    try:
        good = capi.make_boxes([(0, 0, 0)] * 3, [(n, n, n)] * 3)
        o_sent = np.arange(4, dtype=np.uint64) + 77
        t_sent = np.frombuffer(bytes(range(192)), np.uint8).copy().view(capi.OVERLAP_TRIANGLE_DTYPE)

        def call(boxes, count=None, offsets=True, tris=True, capacity=None):
            o, t = (o_sent.copy() if offsets else None), (t_sent.copy() if tris else None)
            rc = mesh.overlap_boxes_rc(boxes, o, t, capacity, count)
            assert (o is None or o.tobytes() == o_sent.tobytes()) and (t is None or t.tobytes() == t_sent.tobytes()), rc
            return rc

        assert call(good) == capi.ERR_STATE                                           # nothing applied yet
        assert L.vxb_mesh_overlap_box_device(mesh.h, C.c_void_p(8), 1, C.c_void_p(8), None, 0) == capi.ERR_STATE
        mesh.apply()
        for field, axis, value in [("min", 0, np.nan), ("max", 2, np.inf), ("min", 1, -np.inf), ("min", 1, 65.0)]:
            b = good.copy(); b[field][2, axis] = value
            assert call(b) == -2 and b"box 2" in L.vxb_last_error(ctx.h), (field, value)
        assert call(None, 3) == -2 and call(good, offsets=False) == -2 and call(good, tris=False, capacity=5) == -2
        assert L.vxb_mesh_overlap_box_device(mesh.h, None, 1, C.c_void_p(8), None, 0) == -2
        assert L.vxb_mesh_overlap_box_device(mesh.h, C.c_void_p(8), 1, None, None, 0) == -2
        assert L.vxb_mesh_overlap_box_device(mesh.h, C.c_void_p(8), 1, C.c_void_p(8), None, 4) == -2
        assert call(good, 0) == 0                                                    # count = 0 does nothing
        assert L.vxb_mesh_overlap_box(mesh.h, None, 0, None, None, 0) == 0
        assert L.vxb_mesh_overlap_box_device(mesh.h, None, 0, None, None, 0) == 0
    finally:
        mesh.close()


def test_terrain1024_device_host_and_oracle(gpu_context):
    import torch
    n = 1024
    ctx = gpu_context
    mesh = _terrain_mesh(ctx, n)
    rng = np.random.RandomState(1024)
    try:
        res = mesh.download()
        lv = oracle.Level0Sorted(res)
        verts = lv.tri.reshape(-1, 3)
        small = body_boxes(verts[rng.randint(0, len(verts), 1 << 16)], rng)
        lo = np.stack([rng.randint(0, n // 64, 256) * 64, rng.randint(0, n // 64, 256) * 64, rng.randint(0, n // 64, 256) * 64], axis=1)
        surf = verts[rng.randint(0, len(verts), 256)]
        lo[:, 1] = (surf[:, 1] // 64) * 64                                             # tiles at the surface height
        tiles = capi.make_boxes(lo, lo + 64)
        for what, boxes in (("small", small), ("tiles", tiles)):
            want = mesh.overlap_boxes(boxes)
            total = int(want[0][-1])
            bt, ot, tt = _to_device(boxes), _buffer((len(boxes) + 1) * 8), _buffer(total * 48)
            torch.cuda.synchronize()
            mesh.overlap_boxes_device(bt.data_ptr(), len(boxes), ot.data_ptr(), tt.data_ptr(), total)
            got = (_read(ot, np.uint64, len(boxes) + 1), _read(tt, capi.OVERLAP_TRIANGLE_DTYPE, total))
            del bt, ot, tt
            torch.cuda.empty_cache()
            assert_same(got, want, "1024^3 %s: device vs host" % what)
            assert total > len(boxes)
            pick = np.sort(rng.choice(len(boxes), min(len(boxes), 128), replace=False))
            sub = mesh.overlap_boxes(boxes[pick])
            for j, q in enumerate(pick):
                assert np.array_equal(want[1][int(want[0][q]):int(want[0][q + 1])], sub[1][int(sub[0][j]):int(sub[0][j + 1])])
            assert_same(sub, oracle.overlap_boxes(res, boxes[pick], lv), "1024^3 %s: oracle sample" % what)
    finally:
        mesh.close()
