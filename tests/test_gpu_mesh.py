"""The device-resident mesh (include/vxb200.h "mesh"): the whole surface kept in HBM across edits, spliced on the GPU after
every run.  The oracle is the reference's incremental surface: after every edit, EVERY level of the mesh - blocks, their
order, vertices and indices - equals PolygonMap::Levels[l] after Execute(grid, materials, modification), and the mesh's
statistics equal the reference's.  The draw lists built from the mesh follow the renderer contract of test_gpu_draws."""
import numpy as np
import pytest

import compare
import harness
from voxels_b200 import capi
from test_gpu_draws import _finer, _selected

pytestmark = pytest.mark.gpu

FACES = [(0, 0, -1), (0, -1, 0), (-1, 0, 0), (0, 0, 1), (0, 1, 0), (1, 0, 0)]


@pytest.fixture(scope="module")
def program_reference():
    """The reference with the SDF-program calls (tests/program_harness.py); every call of the conftest's reference too."""
    import program_harness
    lib = program_harness.load()
    if lib is None:
        pytest.skip("oracle/_ref/libvxh_programs_ref.so not built (needs the reference checkout)")
    return lib


def _mesh_problems(reference, surf, mesh, what, stats=True):
    got = mesh.download()
    problems = []
    levels = reference.surface_levels(surf)
    assert got.info.levels == levels
    for l in range(levels):
        problems += compare.level_diff(reference.surface_level(surf, l), got.level(l), "%s L%d" % (what, l))
    if stats and not np.array_equal(reference.surface_stats(surf), got.stats):
        problems.append("%s: stats differ: ref %s mesh %s" % (what, reference.surface_stats(surf), got.stats))
    return problems


def _assert_mesh(reference, surf, mesh, what, stats=True):
    problems = _mesh_problems(reference, surf, mesh, what, stats)
    assert not problems, "\n".join(problems[:8])


def _grid(reference, ctx, name, n=128):
    import gridgen
    if name == "terrain128":
        s = capi.Surface.terrain(n)
        g = reference.grid_create_builtin(n, s)
        ctx.fill(n, s)
    else:
        dist, mat, blend = gridgen.patchwork(n)
        g = reference.grid_from_dense(dist, mat, blend)
        ctx.upload_dense(dist, mat, blend)
    return g


def _terrain_edits(reference, g, n, count=25):
    """test_gpu_gridstore._edit_run's terrain generator: sphere adds / subtracts centred near the surface."""
    dist0 = reference.grid_to_dense(g)[0]
    rng = np.random.RandomState(3)
    edits = []
    while len(edits) < count:
        x, y, z = (int(v) for v in rng.randint(16, n - 16, size=3))
        if abs(int(dist0[z, y, x])) >= 4:
            continue
        r = float(rng.choice([4, 6, 8]))
        edits.append((np.array([x, y, z], np.float32), np.full(3, 2 * r + 4, np.float32), capi.Surface.sphere((0, 0, 0), r),
                      0 if len(edits) % 2 == 0 else 2))
    return edits


def _edit_and_apply(reference, ctx, mesh, g, surf, mod, pos, ext, sph, kind):
    box = reference.grid_inject_builtin(g, pos, ext, sph, kind)
    reference.polygonize(g, modification=mod, surface=surf, box=box)
    got_box = ctx.inject_surface(pos, ext, sph, kind)
    assert np.array_equal(box, got_box)
    ctx.polygonize_region(got_box[:3], got_box[3:])
    mesh.apply()


@pytest.mark.parametrize("name", ["terrain128", "patchwork128"])
def test_full_run_apply_equals_download(reference, gpu_context, name):
    ctx = gpu_context
    ctx.set_materials(None, None)
    g = _grid(reference, ctx, name)
    reference.grid_destroy(g)
    ctx.polygonize()
    want = ctx.download()
    mesh = ctx.mesh()
    try:
        info = mesh.apply()
        got = mesh.download()
        assert info.block_count == len(want.records) > 0
        assert np.array_equal(got.records[["level", "coord_id", "id"]], want.records[["level", "coord_id", "id"]])
        for l in range(want.info.levels_total):
            problems = compare.level_diff(want.level(l), got.level(l), "%s L%d" % (name, l))
            assert not problems, "\n".join(problems[:8])
            assert info.level_blocks[l] == int((want.records["level"] == l).sum())
        assert np.array_equal(got.stats, want.stats)
        # the degenerate filter's gaps are squeezed out: the spans are the live data (index ranges padded to 4)
        assert info.vertex_span == info.vertex_total == want.info.vertex_total and info.index_total == want.info.index_total
        assert info.index_span == int(((want.records["index_count"] + 3) // 4 * 4).sum())
        assert info.trans_vertex_total == want.info.trans_vertex_total and info.trans_index_total == want.info.trans_index_total
        assert info.apply_ms > 0 and info.bytes_copied > 0
    finally:
        mesh.close()


def test_full_run_apply_unmapped_materials_have_zero_textures(reference, gpu_context):
    """The marker of an unmapped material (vxb_finish_vertex) becomes the reference's all-zero textures on the device."""
    import grids
    import parity
    dist, mat, blend = grids.SMALL["hostile64"]()
    table = (np.arange(256 * 6) * 7 % 251).astype(np.uint8)
    valid = np.ones(256, np.uint8); valid[1] = 0; valid[2] = 0
    problems, _ = parity.run_both(reference, gpu_context, dist, mat, blend, table=table, valid=valid)
    assert not problems, "\n".join(problems[:8])
    g = reference.grid_from_dense(dist, mat, blend)
    s, _ = reference.polygonize(g, material_table=table, valid_mask=valid)
    mesh = gpu_context.mesh()
    try:
        mesh.apply()
        zero = 0
        got = mesh.download()
        for l in range(reference.surface_levels(s)):
            want = reference.surface_level(s, l)
            problems = compare.level_diff(want, got.level(l), "L%d" % l)
            assert not problems, "\n".join(problems[:8])
            zero += int((got.level(l).verts["tex"] == 0).all(axis=1).sum())
        assert zero > 0, "no vertex of an unmapped material: the case does not exercise the marker"
    finally:
        mesh.close()
        reference.surface_destroy(s); reference.grid_destroy(g)
        gpu_context.set_materials(None, None)


@pytest.mark.parametrize("capacity", [None, (4096, 4096, 1024, 1024)], ids=["sized_by_first_apply", "tiny_capacity"])
def test_terrain_edits_every_level_equals_reference(reference, gpu_context, capacity):
    n = 128
    ctx = gpu_context
    ctx.set_materials(None, None)
    g = _grid(reference, ctx, "terrain128")
    surf, _ = reference.polygonize(g)
    mod = reference.modification_create()
    ctx.polygonize()
    mesh = ctx.mesh(capacity)
    try:
        gen0 = mesh.info().generation
        mesh.apply()
        _assert_mesh(reference, surf, mesh, "full run")
        for i, (pos, ext, sph, kind) in enumerate(_terrain_edits(reference, g, n)):
            _edit_and_apply(reference, ctx, mesh, g, surf, mod, pos, ext, sph, kind)
            _assert_mesh(reference, surf, mesh, "edit %d" % i)
            # the context's result still holds exactly the region's blocks
            assert len(ctx.download().records) == ctx.info().block_count
        info = mesh.info()
        if capacity is not None:
            assert info.compactions > 0 and info.growths > 0 and info.generation != gen0
            assert all(c >= t for c, t in zip(info.capacity, (info.vertex_span, info.index_span, info.trans_vertex_span, info.trans_index_span)))
    finally:
        mesh.close()
        reference.modification_destroy(mod); reference.surface_destroy(surf); reference.grid_destroy(g)


def test_edge_edits_programs_and_host_update_equal_reference(program_reference, gpu_context):
    """patchwork128 with edits at the grid's faces, edges and corners (clipped dirty ranges), the persistent kernels capped
    at 2 CTAs, a few SDF-program brushes and one host-side vxb_grid_update_blocks edit."""
    import gridgen
    from voxels_b200.capi import Op
    reference = program_reference
    n = 128
    ctx = gpu_context
    ctx.set_materials(None, None)
    g = _grid(reference, ctx, "patchwork128")
    surf, _ = reference.polygonize(g)
    mod = reference.modification_create()
    ctx.polygonize()
    mesh = ctx.mesh()
    ctx.set_launch_limit(2)
    try:
        mesh.apply()
        _assert_mesh(reference, surf, mesh, "full run")
        for i, (pos, r, ext, add) in enumerate(gridgen.edge_edit_sequence(n, 18)):
            p, e = np.array(pos, np.float32), np.full(3, ext, np.float32)
            if i % 6 == 3:   # an SDF-program brush at the same place
                ops = [Op.box((0.6 * r, 0.4 * r, 0.5 * r), at=(0.3 * r, 0.0, 0.0)), Op.sphere(0.6 * r, at=(-0.3 * r, 0.0, 0.0)), Op.smooth_union(1.5)]
                box = reference.grid_inject_program(g, p, e, ops, 0 if add else 2)
                reference.polygonize(g, modification=mod, surface=surf, box=box)
                got_box = ctx.inject_program(p, e, ops, 0 if add else 2)
                assert np.array_equal(box, got_box)
                ctx.polygonize_region(got_box[:3], got_box[3:])
                mesh.apply()
            elif i == 10:    # host-side edit: the reference's edited blocks uploaded with vxb_grid_update_blocks
                before = ctx.download_dense()
                box = reference.grid_inject_builtin(g, p, e, capi.Surface.sphere((0, 0, 0), r), 0 if add else 2)
                reference.polygonize(g, modification=mod, surface=surf, box=box)
                after = reference.grid_to_dense(g)
                nb = n // 16
                changed = [(x, y, z) for z in range(nb) for y in range(nb) for x in range(nb)
                           if any(not np.array_equal(a[16 * z:16 * z + 16, 16 * y:16 * y + 16, 16 * x:16 * x + 16],
                                                     b[16 * z:16 * z + 16, 16 * y:16 * y + 16, 16 * x:16 * x + 16]) for a, b in zip(before, after))]
                assert changed

                def blocks(vol):
                    return np.ascontiguousarray(np.stack([vol[16 * z:16 * z + 16, 16 * y:16 * y + 16, 16 * x:16 * x + 16].ravel() for x, y, z in changed]))
                ctx.update_blocks(np.array(changed, np.uint32), blocks(after[0]), blocks(after[1]), blocks(after[2]))
                ctx.polygonize_region(box[:3], box[3:])
                mesh.apply()
            else:
                _edit_and_apply(reference, ctx, mesh, g, surf, mod, p, e, capi.Surface.sphere((0, 0, 0), r), 0 if add else 2)
            _assert_mesh(reference, surf, mesh, "edit %d" % i)
    finally:
        ctx.set_launch_limit(0)
        mesh.close()
        reference.modification_destroy(mod); reference.surface_destroy(surf); reference.grid_destroy(g)


def _coords(level, coord_id, n):
    nb = (n // 16) >> level
    return coord_id % nb, (coord_id // nb) % nb, coord_id // (nb * nb)


def _check_draws(blocks, lists, arenas, camera, base, n, top):
    """`blocks`: {id: (level, coord_id, indices, [trans indices per face], trans index counts)} of the surface; `lists`: the
    mesh's draw lists; `arenas`: the mesh's downloaded index arenas.  The renderer contract of test_gpu_draws, evaluated on
    `blocks`, and the indices behind every command equal the block's."""
    rc, ri, tc, ti = lists
    idx, tidx = arenas
    cam = np.array(camera, np.float64)
    want = {}
    for bid, (level, cid, _, _, _) in blocks.items():
        b = _coords(level, cid, n)
        if not _selected(level, b, cam, base, top):
            continue
        adj = 0
        if level > 0:
            nb = (n // 16) >> level
            for f, d in enumerate(FACES):
                nbr = (b[0] + d[0], b[1] + d[1], b[2] + d[2])
                if min(nbr) >= 0 and max(nbr) < nb and _finer(level, nbr, cam, base, top):
                    adj |= 1 << f
        want[bid] = adj
    assert len(want) > 0
    assert sorted(int(i) for i in ri["block_id"]) == sorted(want)
    assert np.array_equal(rc["first_instance"], np.arange(len(rc)))
    trans = 0
    for cmd, inf in zip(rc, ri):
        bid = int(inf["block_id"])
        level, _, bidx, _, tcounts = blocks[bid]
        assert int(inf["block_adj"]) == want[bid] and int(inf["level"]) == level and int(inf["face"]) == 0xFFFFFFFF
        assert int(cmd["index_count"]) == len(bidx) and int(cmd["instance_count"]) == 1
        assert np.array_equal(idx[int(cmd["first_index"]):int(cmd["first_index"]) + len(bidx)], bidx)
        trans += sum(1 for f in range(6) if (want[bid] >> f) & 1 and tcounts[f])
    assert len(tc) == trans
    for cmd, inf in zip(tc, ti):
        bid, f = int(inf["block_id"]), int(inf["face"])
        _, _, _, btidx, _ = blocks[bid]
        assert (want[bid] >> f) & 1 and int(inf["block_adj"]) == want[bid]
        assert int(cmd["index_count"]) == len(btidx[f])
        assert np.array_equal(tidx[int(cmd["first_index"]):int(cmd["first_index"]) + len(btidx[f])], btidx[f])


def _result_blocks(res):
    out = {}
    for r in res.records:
        t = [res.tidx[o:o + c] for o, c in zip(r["trans_index_offset"], r["trans_index_count"])]
        out[int(r["id"])] = (int(r["level"]), int(r["coord_id"]), res.idx[r["index_offset"]:r["index_offset"] + r["index_count"]], t,
                             [int(c) for c in r["trans_index_count"]])
    return out


CAMERAS = [((40.0, 70.0, 50.0), 48.0), ((128.0, 64.0, 128.0), 20.0), ((-50.0, 300.0, 10.0), 64.0)]


def test_draw_lists_after_full_run_match_context(gpu_context):
    n = 128
    ctx = gpu_context
    ctx.set_materials(None, None)
    ctx.fill(n, capi.Surface.terrain(n))
    info = ctx.polygonize()
    res = ctx.download()
    mesh = ctx.mesh()
    try:
        mesh.apply()
        got = mesh.download()
        for camera, base in CAMERAS:
            want = ctx.select_lod(camera, base)
            lists = mesh.select_lod(camera, base)
            assert len(lists[0]) == len(want[0]) and len(lists[2]) == len(want[2])
            assert sorted(int(i) for i in lists[1]["block_id"]) == sorted(int(i) for i in want[1]["block_id"])
            wadj = {int(i["block_id"]): (int(i["block_adj"]), int(c["index_count"])) for c, i in zip(want[0], want[1])}
            for c, i in zip(lists[0], lists[1]):
                assert wadj[int(i["block_id"])] == (int(i["block_adj"]), int(c["index_count"]))
            wt = sorted((int(i["block_id"]), int(i["face"]), int(c["index_count"])) for c, i in zip(want[2], want[3]))
            assert sorted((int(i["block_id"]), int(i["face"]), int(c["index_count"])) for c, i in zip(lists[2], lists[3])) == wt
            _check_draws(_result_blocks(res), lists, (got.idx, got.tidx), camera, base, n, info.levels_total - 1)
        ptrs = mesh.device_arenas()
        assert all(p for p in ptrs[:3])
    finally:
        mesh.close()


def test_draw_lists_after_edits_follow_the_reference_surface(reference, gpu_context):
    n = 128
    ctx = gpu_context
    ctx.set_materials(None, None)
    g = _grid(reference, ctx, "terrain128")
    surf, _ = reference.polygonize(g)
    mod = reference.modification_create()
    ctx.polygonize()
    mesh = ctx.mesh()
    try:
        mesh.apply()
        for pos, ext, sph, kind in _terrain_edits(reference, g, n, 12):
            _edit_and_apply(reference, ctx, mesh, g, surf, mod, pos, ext, sph, kind)
        _assert_mesh(reference, surf, mesh, "after the edits")
        got = mesh.download()
        # the reference surface's blocks: id -> (level, coord_id, indices, transition indices per face)
        blocks = {}
        for l in range(reference.surface_levels(surf)):
            lv = reference.surface_level(surf, l)
            m = 16 << l; nb = n // m
            for k in range(len(lv.rows)):
                row, _, bidx, _, btidx = lv.block(k)
                x, z, y = (int(v) // m for v in row["min"])           # output axes (x, z, y)
                blocks[int(row["id"])] = (l, (z * nb + y) * nb + x, bidx, btidx, [len(t) for t in btidx])
        for camera, base in CAMERAS:
            _check_draws(blocks, mesh.select_lod(camera, base), (got.idx, got.tidx), camera, base, n, reference.surface_levels(surf) - 1)
    finally:
        mesh.close()
        reference.modification_destroy(mod); reference.surface_destroy(surf); reference.grid_destroy(g)


def _snapshot(mesh):
    r = mesh.download()
    return r.records.copy(), r.verts.copy(), r.idx.copy(), r.tverts.copy(), r.tidx.copy()


def _same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


def test_refused_applies_leave_the_mesh(gpu_context):
    import voxels_b200
    from test_gpu_sharded import configure_virtual_ranks, run_virtual_ranks
    n = 128
    ctx = voxels_b200.Context(0)
    try:
        ctx.fill(n, capi.Surface.terrain(n))
        mesh = ctx.mesh()
        assert mesh.apply_rc() == capi.ERR_STATE                       # no result
        ctx.polygonize()
        mesh.apply()
        snap = _snapshot(mesh)
        assert mesh.apply_rc() == capi.ERR_STATE                       # the same run twice
        assert _same(snap, _snapshot(mesh))
        box = ctx.inject_surface((60, 60, 60), (20, 20, 20), capi.Surface.sphere((0, 0, 0), 8), 0)
        ctx.polygonize_region(box[:3], box[3:])                       # skipped ...
        box = ctx.inject_surface((70, 50, 64), (20, 20, 20), capi.Surface.sphere((0, 0, 0), 8), 2)
        ctx.polygonize_region(box[:3], box[3:])
        assert mesh.apply_rc() == capi.ERR_STATE                       # ... so this region run cannot be spliced
        assert _same(snap, _snapshot(mesh))
        # the context's result still holds only the region's blocks
        region = ctx.region_info()
        part = ctx.download()
        assert len(part.records) == ctx.info().block_count
        assert set(int(i) for i in part.records["id"]) <= set(range(region.id_start[0], region.id_start[0] + sum(region.block_count)))
        ctx.polygonize()                                               # a full run starts the chain again
        mesh.apply()
        # a sharded result (one virtual rank over the same grid)
        d, m, b = ctx.device_pointers()
        other = voxels_b200.Context(0)
        try:
            other.set_device_grid(n, d, m, b)
            other.polygonize()
            om = other.mesh()
            om.apply()
            snap = _snapshot(om)
            bufs = configure_virtual_ranks([other])
            run_virtual_ranks([other], bufs)
            assert om.apply_rc() == capi.ERR_STATE
            assert _same(snap, _snapshot(om))
        finally:
            other.close()
        mesh.close()
    finally:
        ctx.close()
