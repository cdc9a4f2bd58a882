"""The mesh's per-block bounds and the culled select (include/vxb200.h "bounds and the culled select") against the numpy
oracle (tests/cull_oracle.py) on mesh.download(): the boxes after full applies, across edits, compactions and growth; the
per-view draw lists as sets for frusta inside, above and outside the grid, degenerate and touching ones, 1 to 8 views per
call; their relation to the unculled select; conservativeness checked on the vertices themselves; the refusals."""
import ctypes as C

import numpy as np
import pytest

import cull_oracle as oracle
from voxels_b200 import capi
from voxels_b200.capi import Op

pytestmark = pytest.mark.gpu

F = np.float32
GRIDS = ["terrain128", "terrain256", "sphere64", "hostile64", "patchwork128"]


def _fill(ctx, name):
    import grids
    if name.startswith("terrain"):
        n = int(name[len("terrain"):])
        ctx.fill(n, capi.Surface.terrain(n))
    else:
        ctx.upload_dense(*grids.by_name(name))


def _applied_mesh(ctx, name, capacity=None):
    ctx.set_materials(None, None)
    _fill(ctx, name)
    ctx.polygonize()
    mesh = ctx.mesh(capacity)
    mesh.apply()
    return mesh


def _same_boxes(got, want, what):
    assert got.shape == want.shape, what
    bad = np.nonzero(~(got == want).all(axis=1))[0]      # values: -0 == +0
    assert not len(bad), "%s: %d of %d boxes differ; first: block %d got %s want %s" % (what, len(bad), len(want), bad[0], got[bad[0]], want[bad[0]])


def _assert_bounds(mesh, res, what):
    """Every block's box equals the oracle's, through both accessors; the slots of absent blocks hold min > max."""
    want = oracle.block_boxes(res)
    _same_boxes(mesh.bounds(), want, what)
    b = mesh.bounds_device()
    assert b.slots > 0 and b.boxes
    raw = capi._device_to_numpy(b.boxes, b.slots * 8, np.dtype("<f4")).reshape(b.slots, 8)
    slot = np.array(list(b.level_base), np.int64)[res.records["level"]] + res.records["coord_id"]
    assert len(np.unique(slot)) == len(slot)
    _same_boxes(raw[slot][:, [0, 1, 2, 4, 5, 6]], want, what + " (device slots)")
    absent = np.ones(b.slots, bool); absent[slot] = False
    assert (raw[absent][:, 0:3] > raw[absent][:, 4:7]).all(), what + ": the box of an absent block is not min > max"
    return want


@pytest.mark.parametrize("name", GRIDS)
def test_bounds_equal_oracle(gpu_context, name):
    mesh = _applied_mesh(gpu_context, name)
    try:
        res = mesh.download()
        assert len(res.records) > 0 and (res.records["level"] >= 1).any()
        boxes = _assert_bounds(mesh, res, name)
        assert np.isfinite(boxes).all()                      # every block of a run has vertices
        # the boxes are measured, not the lattice's: on a surface they are smaller than the block
        lattice = oracle.lattice_boxes(res.records, res.n)
        assert ((boxes[:, :3] > lattice[:, :3]).any(axis=1) | (boxes[:, 3:] < lattice[:, 3:]).any(axis=1)).any()
    finally:
        mesh.close()


def _brush(i, r):
    if i % 3 == 0:
        return [Op.sphere(r)]
    if i % 3 == 1:
        return [Op.box((r, r, r))]
    return [Op.box((0.6 * r, 0.4 * r, r)), Op.sphere(r), Op.smooth_union(1.5)]


def test_bounds_follow_terrain_brush_edits(gpu_context):
    """test_gpu_raycast's sculpting sequence: 25 program brushes at picked surface points."""
    n = 128
    ctx = gpu_context
    mesh = _applied_mesh(ctx, "terrain128")
    rng = np.random.RandomState(21)
    try:
        erased = 0
        for edit in range(25):
            x, z = rng.uniform(16, n - 16, 2)
            p = mesh.raycast(capi.make_rays([(x, n + 8.0, z)], [(0, -1, 0)]))
            assert p["slot"][0] != capi.VXB_RAY_MISS
            hit = p["position"][0]
            r = float(rng.choice([4, 6, 8]))
            before = len(mesh.download().records)
            box = ctx.inject_program(np.array([hit[0], hit[2], hit[1]], F), np.full(3, 2 * r + 4, F), _brush(edit, r), 0 if edit % 2 == 0 else 2)
            region = ctx.polygonize_region(box[:3], box[3:])
            mesh.apply()
            res = mesh.download()
            erased += before + region.block_count - len(res.records)
            _assert_bounds(mesh, res, "edit %d" % edit)
        assert erased > 0
    finally:
        mesh.close()


def test_bounds_survive_compaction_and_growth(gpu_context):
    """test_gpu_raycast's edge edits on patchwork128 at launch limit 2 and a tiny mesh capacity: the arenas move, the boxes of
    the survivors stay."""
    import gridgen
    n = 128
    ctx = gpu_context
    mesh = _applied_mesh(ctx, "patchwork128", (4096, 4096, 1024, 1024))
    ctx.set_launch_limit(2)
    try:
        _assert_bounds(mesh, mesh.download(), "full run")
        for i, (pos, r, ext, add) in enumerate(gridgen.edge_edit_sequence(n, 12)):
            box = ctx.inject_surface(np.array(pos, F), np.full(3, ext, F), capi.Surface.sphere((0, 0, 0), r), 0 if add else 2)
            ctx.polygonize_region(box[:3], box[3:])
            mesh.apply()
            _assert_bounds(mesh, mesh.download(), "edge edit %d" % i)
        info = mesh.info()
        assert info.compactions > 0 and info.growths > 0
    finally:
        ctx.set_launch_limit(0)
        mesh.close()


def _named_views(n, res, boxes, camera, base):
    """The view volumes of the list tests, and the block the touching planes are built on."""
    selected, _ = oracle.cut(res.records, res.n, res.info.levels, camera, base)
    k = int(np.nonzero(selected)[0][len(np.nonzero(selected)[0]) // 2])     # a block of the cut
    lo, hi = boxes[k, :3], boxes[k, 3:]
    on_max, on_min, past_max = oracle.PASS_ALL.copy(), oracle.PASS_ALL.copy(), oracle.PASS_ALL.copy()
    on_max[0] = [1, 0, 0, -hi[0]]                                            # x >= max x of the block: s == 0, drawn
    on_min[3] = [0, -1, 0, lo[1]]                                            # y <= min y of the block: s == 0, drawn
    past_max[0] = [1, 0, 0, -np.nextafter(hi[0], F(np.inf))]                 # one ulp further: culled
    views = {
        "inside": oracle.perspective((0.4 * n, 0.55 * n, 0.45 * n), (1, -0.2, 0.6), (0, 1, 0), 90, 60, 0.5, 4.0 * n),
        "above": oracle.perspective((0.5 * n, 2.5 * n, 0.5 * n), (0.05, -1, 0.1), (0, 0, 1), 40, 40, 1.0, 4.0 * n),
        "outside": oracle.perspective((-1.5 * n, 0.8 * n, -0.7 * n), (1, -0.1, 0.6), (0, 1, 0), 50, 35, 1.0, 2.2 * n),
        "away": oracle.perspective((-1.5 * n, 0.8 * n, -0.7 * n), (-1, 0, 0), (0, 1, 0), 50, 35, 1.0, 2.2 * n),
        "slab": oracle.box_planes((0.25 * n, -n, 0.3 * n), (0.5 * n, 2 * n, 0.55 * n)),
        "containing": oracle.box_planes((-4.0 * n,) * 3, (5.0 * n,) * 3),
        "nothing": oracle.box_planes((7.0 * n,) * 3, (8.0 * n,) * 3),
        "on_max": on_max, "on_min": on_min, "past_max": past_max,
        "pass_all": oracle.PASS_ALL,
    }
    return views, k


def _sets_equal(got, want, what):
    for kind, g, w in (("regular", got[0], want[0]), ("transition", got[1], want[1])):
        assert g == w, "%s: %s draws differ: %d missing, %d extra; e.g. %s" % (what, kind, len(w - g), len(g - w), sorted(w ^ g)[:2])


CAMERAS = [((40.0, 70.0, 50.0), 48.0), ((128.0, 64.0, 128.0), 20.0), ((-50.0, 300.0, 10.0), 64.0)]


def _check_views(mesh, res, boxes, n, cameras):
    levels = res.info.levels
    ids = res.records["id"]
    outcomes = set()
    for camera, base in cameras:
        scale = n / 128.0
        camera, base = tuple(c * scale for c in camera), base * scale
        views, k = _named_views(n, res, boxes, camera, base)
        unculled_lists = capi.DrawLists()
        unculled = oracle.draw_sets(mesh.select_lod(camera, base, unculled_lists))
        # 1, 3 and 8 views per call, identical views repeated
        calls = [["inside"], ["above", "above", "slab"], ["outside", "containing", "nothing", "on_max", "on_min", "past_max", "pass_all", "inside"],
                 ["away", "pass_all", "away"]]
        for names in calls:
            got = [oracle.draw_sets(l) for l in mesh.select_lod_views(camera, base, np.stack([views[v] for v in names]))]
            want = oracle.expected_draws(res.records, boxes, res.n, levels, camera, base, [views[v] for v in names])
            for v, name in enumerate(names):
                what = "camera %s view %d (%s) of %d" % (camera, v, name, len(names))
                _sets_equal(got[v], want[v], what)
                # the cut is the unculled select's: block_adj and the transition draws of every drawn block are its own
                drawn = {d[0] for d in got[v][0]}
                outcomes.add(len(drawn) > 0)
                assert got[v][0] <= unculled[0], what
                assert got[v][1] == {t for t in unculled[1] if t[0] in drawn}, what
                if name in ("containing", "pass_all"):
                    _sets_equal(got[v], unculled, what + " against the unculled select")
                if name == "nothing":
                    assert not got[v][0] and not got[v][1]
                if name in ("on_max", "on_min"):
                    assert int(ids[k]) in drawn, what + ": a plane on the box's face (s == 0) culls the block"
                if name == "past_max":
                    assert int(ids[k]) not in drawn, what
            for v in range(len(names)):
                for w in range(v):
                    if names[v] == names[w]:
                        assert got[v] == got[w]
        # the unculled select's lists are its own: untouched by the culled calls, and rebuilt the same
        kept = (capi._device_to_numpy(unculled_lists.regular, unculled_lists.regular_count, capi.DRAW_COMMAND_DTYPE),
                capi._device_to_numpy(unculled_lists.regular_info, unculled_lists.regular_count, capi.DRAW_INFO_DTYPE),
                capi._device_to_numpy(unculled_lists.transition, unculled_lists.transition_count, capi.DRAW_COMMAND_DTYPE),
                capi._device_to_numpy(unculled_lists.transition_info, unculled_lists.transition_count, capi.DRAW_INFO_DTYPE))
        assert oracle.draw_sets(kept) == unculled
        assert oracle.draw_sets(mesh.select_lod(camera, base)) == unculled
    assert outcomes == {True, False}


@pytest.mark.parametrize("name", ["terrain128", "hostile64", "patchwork128"])
def test_culled_lists_equal_oracle(gpu_context, name):
    mesh = _applied_mesh(gpu_context, name)
    try:
        res = mesh.download()
        _check_views(mesh, res, oracle.block_boxes(res), res.n, CAMERAS)
    finally:
        mesh.close()


def test_culled_lists_after_edits(gpu_context):
    ctx = gpu_context
    mesh = _applied_mesh(ctx, "terrain128")
    try:
        for i, (x, y, z, r) in enumerate([(40, 60, 50, 8), (64, 64, 64, 6), (90, 70, 30, 8), (20, 60, 100, 4)]):
            box = ctx.inject_surface(np.array([x, y, z], F), np.full(3, 2 * r + 4, F), capi.Surface.sphere((0, 0, 0), r), 0 if i % 2 == 0 else 2)
            ctx.polygonize_region(box[:3], box[3:])
            mesh.apply()
        res = mesh.download()
        _check_views(mesh, res, _assert_bounds(mesh, res, "after the edits"), res.n, CAMERAS[:2])
    finally:
        mesh.close()


@pytest.mark.parametrize("name", ["terrain128", "hostile64"])
def test_random_frusta_keep_every_block_with_a_vertex_inside(gpu_context, name):
    """Conservative, independently of the box formula: a block of the cut with a vertex (either position, regular or
    transition) inside all six planes - float64, by a margin - is drawn."""
    mesh = _applied_mesh(gpu_context, name)
    try:
        res = mesh.download()
        n = res.n
        pts, owner = [], []
        for k, r in enumerate(res.records):
            parts = [res.verts[r["vertex_offset"]:r["vertex_offset"] + r["vertex_count"]]]
            parts += [res.tverts[o:o + c] for o, c in zip(r["trans_vertex_offset"], r["trans_vertex_count"])]
            for p in parts:
                pts += [p["pos"], p["sec"][:, :3]]
                owner += [np.full(2 * len(p), k)]
        pts, owner = np.concatenate(pts).astype(np.float64), np.concatenate(owner)
        rng = np.random.RandomState(77)
        scale = n / 128.0
        camera, base = tuple(c * scale for c in CAMERAS[0][0]), CAMERAS[0][1] * scale
        selected, _ = oracle.cut(res.records, n, res.info.levels, camera, base)
        views = np.stack([oracle.perspective(rng.uniform(-0.5 * n, 1.5 * n, 3), rng.normal(size=3), (0.02, 1, 0.01), rng.uniform(20, 120),
                                             rng.uniform(20, 100), rng.uniform(0.1, 8), rng.uniform(0.3 * n, 3 * n)) for _ in range(24)])
        seen = 0
        for first in range(0, len(views), 8):
            for view, lists in zip(views[first:first + 8], mesh.select_lod_views(camera, base, views[first:first + 8])):
                p = view.astype(np.float64)
                s = pts @ p[:, :3].T + p[:, 3]
                margin = 1e-3 * np.abs(p[:, :3]).sum(axis=1) * n
                must = np.unique(owner[(s >= margin).all(axis=1)])
                must = set(res.records["id"][must[selected[must]]].tolist())
                drawn = set(lists[1]["block_id"].tolist())
                assert must <= drawn, "%d blocks with a vertex inside the frustum are culled" % len(must - drawn)
                seen += len(must)
        assert seen > 0
    finally:
        mesh.close()


def test_refusals_leave_the_previous_lists_and_out(gpu_context):
    ctx = gpu_context
    L = ctx.L
    n = 64
    ctx.set_materials(None, None)
    ctx.fill(n, capi.Surface.terrain(n))
    ctx.polygonize()
    mesh = ctx.mesh()
    try:
        cam = np.array([20, 40, 20], F)
        good = np.stack([oracle.perspective((20, 40, 20), (1, -0.3, 1), (0, 1, 0), 90, 60, 0.5, 200), oracle.PASS_ALL]).astype(F)

        def call(camera=cam, planes=good, count=None, out="fresh"):
            o = (capi.DrawLists * capi.VXB_VIEWS_MAX)()
            C.memset(o, 0xAB, C.sizeof(o))
            sentinel = bytes(o)
            rc = L.vxb_mesh_select_lod_views(mesh.h, None if camera is None else capi._ptr(camera), 32.0,
                                             None if planes is None else capi._ptr(np.ascontiguousarray(planes, F)),
                                             len(planes) if count is None else count, None if out is None else o)
            return rc, bytes(o) == sentinel

        assert call() == (capi.ERR_STATE, True)                                              # nothing applied yet
        assert L.vxb_mesh_bounds_get(mesh.h, C.byref(capi.MeshBounds())) == capi.ERR_STATE
        assert L.vxb_mesh_download_bounds(mesh.h, capi._ptr(np.zeros(6, F))) == capi.ERR_STATE
        mesh.apply()
        lists = (capi.DrawLists * 2)()
        before = [oracle.draw_sets(l) for l in mesh.select_lod_views(cam, 32.0, good, lists)]
        assert before[0][0] and before[0][0] <= before[1][0]

        def previous():
            return [oracle.draw_sets((capi._device_to_numpy(l.regular, l.regular_count, capi.DRAW_COMMAND_DTYPE),
                                      capi._device_to_numpy(l.regular_info, l.regular_count, capi.DRAW_INFO_DTYPE),
                                      capi._device_to_numpy(l.transition, l.transition_count, capi.DRAW_COMMAND_DTYPE),
                                      capi._device_to_numpy(l.transition_info, l.transition_count, capi.DRAW_INFO_DTYPE))) for l in lists]

        assert call(count=0) == (-2, True)
        assert call(planes=np.tile(good[:1], (9, 1, 1))) == (-2, True)                       # view_count 9
        for value in (np.nan, np.inf, -np.inf):
            for component in (0, 3):
                bad = good.copy(); bad[1, 4, component] = value
                assert call(planes=bad) == (-2, True), (value, component)
                assert b"view 1 plane 4" in L.vxb_last_error(ctx.h)
        assert call(camera=None) == (-2, True)
        assert call(planes=None, count=2) == (-2, True)
        assert call(out=None)[0] == -2
        assert L.vxb_mesh_bounds_get(mesh.h, None) == -2 and L.vxb_mesh_download_bounds(mesh.h, None) == -2
        assert previous() == before
        assert call() == (0, False)
    finally:
        mesh.close()


def test_terrain1024_bounds_and_four_views(gpu_context):
    n = 1024
    mesh = _applied_mesh(gpu_context, "terrain1024")
    try:
        res = mesh.download()
        levels = res.info.levels
        got = mesh.bounds()
        assert all((res.records["level"] == l).any() for l in range(levels))
        _same_boxes(got, oracle.block_boxes(res), "1024^3")
        camera, base = (0.5 * n, 0.6 * n, 0.5 * n), 64.0
        views = [oracle.perspective(camera, (1, -0.25, 0.3), (0, 1, 0), 90, 60, 0.5, 2.0 * n),
                 oracle.perspective(camera, (-0.4, -0.1, -1), (0, 1, 0), 90, 60, 0.5, 2.0 * n),
                 oracle.box_planes((0.3 * n, -n, 0.3 * n), (0.7 * n, 2 * n, 0.7 * n)),
                 oracle.perspective((0.5 * n, 3.0 * n, 0.5 * n), (0.01, 1, 0.02), (0, 0, 1), 30, 30, 1.0, 4.0 * n)]   # looks away
        lists = mesh.select_lod_views(camera, base, np.stack(views))
        want = oracle.expected_draws(res.records, got, n, levels, camera, base, views)
        unculled = oracle.draw_sets(mesh.select_lod(camera, base))
        for v in range(4):
            _sets_equal(oracle.draw_sets(lists[v]), want[v], "1024^3 view %d" % v)
            assert want[v][0] <= unculled[0]
        assert [len(w[0]) > 0 for w in want] == [True, True, True, False]
    finally:
        mesh.close()
