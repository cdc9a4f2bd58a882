"""vxb_mesh_select_cut (include/vxb200.h "the LOD cut") against the numpy oracle (tests/cut_oracle.py) on mesh.download():
per-view draw lists as sets on five grids, for cameras inside, above and outside the grid, on node faces and exactly at
lod_factor * s from a box, at factors 2, 4, 14.6 and 1e30, in calls of 1, 3 and 8 views; after brush edits and after edge
edits with compaction and growth; the structure of the drawn cut; the lists of the other selects left alone; the refusals;
and the cut at 1024^3 over a camera orbit."""
import ctypes as C

import numpy as np
import pytest

import cut_oracle as oracle
import cull_oracle
from voxels_b200 import capi
from voxels_b200.capi import Op

pytestmark = pytest.mark.gpu

F = np.float32
GRIDS = ["terrain128", "terrain256", "sphere64", "hostile64", "patchwork128"]
FACTORS = [2.0, 4.0, 14.6, 1e30]


def _fill(ctx, name):
    import grids
    if name.startswith("terrain"):
        n = int(name[len("terrain"):])
        ctx.fill(n, capi.Surface.terrain(n))
    else:
        ctx.upload_dense(*grids.by_name(name))


def _applied_mesh(ctx, name, capacity=None, max_levels=0, flags=0):
    ctx.set_materials(None, None)
    _fill(ctx, name)
    ctx.polygonize(max_levels, flags)
    mesh = ctx.mesh(capacity)
    mesh.apply()
    return mesh


def _cameras(n, factor):
    """Inside, above and outside the grid, on node faces (multiples of 32), and exactly lod_factor * 32 above the level-1
    box [0, 32]^3 (dist2 == lim^2: that node does not refine)."""
    return [(0.4 * n, 0.3 * n, 0.45 * n), (0.5 * n, 1.5 * n, 0.55 * n), (-1.2 * n, 0.7 * n, 1.6 * n), (0.5 * n, 0.25 * n, 0.75 * n),
            (16.0, float(F(32) + F(factor) * F(32)) if factor < 1e3 else 40.0, 16.0)]


def _views(n, res, boxes, camera, factor):
    """The view volumes of test_gpu_cull.py, with the touching planes built on a block of this cut."""
    selected, _ = oracle.cut(res.records, res.n, res.info.levels, camera, factor)
    idx = np.nonzero(selected)[0]
    k = int(idx[len(idx) // 2])
    lo, hi = boxes[k, :3], boxes[k, 3:]
    on_max, on_min, past_max = cull_oracle.PASS_ALL.copy(), cull_oracle.PASS_ALL.copy(), cull_oracle.PASS_ALL.copy()
    on_max[0] = [1, 0, 0, -hi[0]]
    on_min[3] = [0, -1, 0, lo[1]]
    past_max[0] = [1, 0, 0, -np.nextafter(hi[0], F(np.inf))]
    views = {
        "inside": cull_oracle.perspective((0.4 * n, 0.55 * n, 0.45 * n), (1, -0.2, 0.6), (0, 1, 0), 90, 60, 0.5, 4.0 * n),
        "above": cull_oracle.perspective((0.5 * n, 2.5 * n, 0.5 * n), (0.05, -1, 0.1), (0, 0, 1), 40, 40, 1.0, 4.0 * n),
        "outside": cull_oracle.perspective((-1.5 * n, 0.8 * n, -0.7 * n), (1, -0.1, 0.6), (0, 1, 0), 50, 35, 1.0, 2.2 * n),
        "away": cull_oracle.perspective((-1.5 * n, 0.8 * n, -0.7 * n), (-1, 0, 0), (0, 1, 0), 50, 35, 1.0, 2.2 * n),
        "slab": cull_oracle.box_planes((0.25 * n, -n, 0.3 * n), (0.5 * n, 2 * n, 0.55 * n)),
        "containing": cull_oracle.box_planes((-4.0 * n,) * 3, (5.0 * n,) * 3),
        "nothing": cull_oracle.box_planes((7.0 * n,) * 3, (8.0 * n,) * 3),
        "on_max": on_max, "on_min": on_min, "past_max": past_max,
        "pass_all": cull_oracle.PASS_ALL,
    }
    return views, int(res.records["id"][k])


CALLS = [["pass_all"], ["inside", "above", "slab"],
         ["outside", "containing", "nothing", "on_max", "on_min", "past_max", "pass_all", "away"]]


def _sets_equal(got, want, what):
    for kind, g, w in (("regular", got[0], want[0]), ("transition", got[1], want[1])):
        assert g == w, "%s: %s draws differ: %d missing, %d extra; e.g. %s" % (what, kind, len(w - g), len(g - w), sorted(w ^ g)[:2])


def _check_structure(res, camera, factor, drawn):
    """The drawn cut (every view's lists are a subset of the pass-all list): no drawn block has a drawn ancestor, every drawn
    block covers its footprint at its own level in the oracle's level map of the whole octree, and every drawn transition
    face borders a region drawn exactly one level finer."""
    regular, transition = drawn
    n, levels = res.n, res.info.levels
    recs = oracle.full_octree(n, levels)
    selected, _ = oracle.cut(recs, n, levels, camera, factor)
    base = np.cumsum([0] + [((n // 16) >> l) ** 3 for l in range(levels)])
    lmap = oracle.level_map(n, levels, lambda l: selected[base[l]:base[l + 1]])
    by_id = {int(r["id"]): r for r in res.records}
    nodes = set()
    for d in regular:
        r = by_id[d[0]]
        level, nb = int(r["level"]), (n // 16) >> int(r["level"])
        c = int(r["coord_id"])
        nodes.add((level, c % nb, (c // nb) % nb, c // (nb * nb)))
    for level, x, y, z in nodes:
        for up in range(1, levels - level):
            assert (level + up, x >> up, y >> up, z >> up) not in nodes, "a drawn block has a drawn ancestor"
        e = 1 << level
        assert (lmap[x * e:(x + 1) * e, y * e:(y + 1) * e, z * e:(z + 1) * e] == level).all()
    faces = 0
    for t in transition:
        r = by_id[t[0]]
        level, nb, f = int(r["level"]), (n // 16) >> int(r["level"]), t[3]
        c = int(r["coord_id"])
        b = np.array([c % nb, (c // nb) % nb, c // (nb * nb)])
        e = 1 << level
        lo, hi = b * e, (b + 1) * e
        d = oracle.FACES[f]
        axis = int(np.nonzero(d)[0][0])
        lo[axis] = lo[axis] - 1 if d[axis] < 0 else hi[axis]
        hi[axis] = lo[axis] + 1
        slab = lmap[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]]
        assert slab.size and (slab == level - 1).all(), "transition face %d of a level-%d block borders levels %s" % (f, level, np.unique(slab))
        faces += 1
    return faces


def _check_calls(mesh, res, boxes, n, cameras_of, factors=FACTORS, structure=True):
    levels = res.info.levels
    outcomes, faces, levels_seen = set(), 0, set()
    for factor in factors:
        for camera in cameras_of(n, factor):
            views, k_id = _views(n, res, boxes, camera, factor)
            for names in CALLS:
                got = [oracle.draw_sets(l) for l in mesh.select_cut(camera, factor, np.stack([views[v] for v in names]))]
                want = oracle.expected_draws(res.records, boxes, res.n, levels, camera, factor, [views[v] for v in names])
                for v, name in enumerate(names):
                    what = "camera %s factor %g view %d (%s) of %d" % (camera, factor, v, name, len(names))
                    _sets_equal(got[v], want[v], what)
                    drawn = {d[0] for d in got[v][0]}
                    outcomes.add(len(drawn) > 0)
                    if name == "nothing":
                        assert not got[v][0] and not got[v][1]
                    if name in ("on_max", "on_min"):
                        assert k_id in drawn, what
                    if name == "past_max":
                        assert k_id not in drawn, what
                    if name == "pass_all":
                        levels_seen |= {d[1] for d in got[v][0]}
                        if structure:
                            faces += _check_structure(res, camera, factor, got[v])
    assert outcomes == {True, False}
    return faces, levels_seen


@pytest.mark.parametrize("name", GRIDS)
def test_cut_lists_equal_oracle(gpu_context, name):
    mesh = _applied_mesh(gpu_context, name)
    try:
        res = mesh.download()
        faces, levels_seen = _check_calls(mesh, res, cull_oracle.block_boxes(res), res.n, _cameras)
        assert len(levels_seen) >= 2 and faces > 0, (levels_seen, faces)
    finally:
        mesh.close()


def _brush(i, r):
    if i % 3 == 0:
        return [Op.sphere(r)]
    if i % 3 == 1:
        return [Op.box((r, r, r))]
    return [Op.box((0.6 * r, 0.4 * r, r)), Op.sphere(r), Op.smooth_union(1.5)]


def _few_cameras(n, factor):
    return _cameras(n, factor)[::2]


def test_cut_after_brush_edits(gpu_context):
    """test_gpu_cull's sculpting sequence: 25 program brushes at picked surface points."""
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
            if edit % 8 == 7 or edit == 24:
                res = mesh.download()
                _check_calls(mesh, res, cull_oracle.block_boxes(res), n, _few_cameras, factors=[2.0, 14.6], structure=edit == 24)
    finally:
        mesh.close()


def test_cut_after_compaction_and_growth(gpu_context):
    import gridgen
    n = 128
    ctx = gpu_context
    mesh = _applied_mesh(ctx, "patchwork128", (4096, 4096, 1024, 1024))
    ctx.set_launch_limit(2)
    try:
        for i, (pos, r, ext, add) in enumerate(gridgen.edge_edit_sequence(n, 12)):
            box = ctx.inject_surface(np.array(pos, F), np.full(3, ext, F), capi.Surface.sphere((0, 0, 0), r), 0 if add else 2)
            ctx.polygonize_region(box[:3], box[3:])
            mesh.apply()
            if i % 4 == 3:
                res = mesh.download()
                _check_calls(mesh, res, cull_oracle.block_boxes(res), n, _few_cameras, factors=[2.0, 4.0], structure=False)
        info = mesh.info()
        assert info.compactions > 0 and info.growths > 0
    finally:
        ctx.set_launch_limit(0)
        mesh.close()


def _lists_bytes(l):
    return b"".join(a.tobytes() for a in (
        capi._device_to_numpy(l.regular, l.regular_count, capi.DRAW_COMMAND_DTYPE),
        capi._device_to_numpy(l.regular_info, l.regular_count, capi.DRAW_INFO_DTYPE),
        capi._device_to_numpy(l.transition, l.transition_count, capi.DRAW_COMMAND_DTYPE),
        capi._device_to_numpy(l.transition_info, l.transition_count, capi.DRAW_INFO_DTYPE),
        capi._device_to_numpy(l.counts, 2, np.dtype("<u4"))))


def test_other_selects_lists_undisturbed(gpu_context):
    n = 128
    mesh = _applied_mesh(gpu_context, "terrain128")
    try:
        res = mesh.download()
        camera = (0.4 * n, 0.5 * n, 0.45 * n)
        views, _ = _views(n, res, cull_oracle.block_boxes(res), camera, 2.0)
        three = np.stack([views["inside"], views["pass_all"], views["slab"]])
        lod = capi.DrawLists()
        mesh.select_lod(camera, 20.0, lod)
        culled = (capi.DrawLists * 3)()
        mesh.select_lod_views(camera, 20.0, three, culled)
        before = [_lists_bytes(lod)] + [_lists_bytes(l) for l in culled]
        cut = (capi.DrawLists * 8)()
        for factor in (2.0, 1e30):                 # 1e30: every level-0 block, more entries than either other list
            mesh.select_cut(camera, factor, np.stack([views[v] for v in CALLS[2]]), cut)
            assert [_lists_bytes(lod)] + [_lists_bytes(l) for l in culled] == before
        assert cut[6].regular_count > lod.regular_count
        # and the other way round: the cut's lists stay as they are across the other two selects
        kept = [_lists_bytes(l) for l in cut]
        mesh.select_lod(camera, 64.0)
        mesh.select_lod_views(camera, 64.0, three)
        assert [_lists_bytes(l) for l in cut] == kept
    finally:
        mesh.close()


def _refusal(mesh, camera=(20.0, 40.0, 20.0), factor=4.0, planes=None, count=None, out=True):
    """vxb_mesh_select_cut's return code, and whether `out` (8 entries of 0xAB) is untouched."""
    planes = np.stack([cull_oracle.perspective((20, 40, 20), (1, -0.3, 1), (0, 1, 0), 90, 60, 0.5, 200), cull_oracle.PASS_ALL]) if planes is None else planes
    o = (capi.DrawLists * capi.VXB_VIEWS_MAX)()
    C.memset(o, 0xAB, C.sizeof(o))
    sentinel = bytes(o)
    rc = mesh.select_cut_rc(None if camera is None else np.array(camera, F), factor, None if planes is None or planes is False else planes,
                            o if out else None, count)
    return rc, bytes(o) == sentinel


def test_refusals_leave_the_previous_lists_and_out(gpu_context):
    ctx = gpu_context
    L = ctx.L
    n = 64
    ctx.set_materials(None, None)
    ctx.fill(n, capi.Surface.terrain(n))
    ctx.polygonize()
    mesh = ctx.mesh()
    try:
        good = np.stack([cull_oracle.perspective((20, 40, 20), (1, -0.3, 1), (0, 1, 0), 90, 60, 0.5, 200), cull_oracle.PASS_ALL]).astype(F)
        assert _refusal(mesh) == (capi.ERR_STATE, True)                                   # nothing applied yet
        mesh.apply()
        lists = (capi.DrawLists * 2)()
        mesh.select_cut((20.0, 40.0, 20.0), 4.0, good, lists)
        before = [_lists_bytes(l) for l in lists]
        assert lists[1].regular_count > lists[0].regular_count > 0
        for factor in (1.99, np.nextafter(F(2), F(0)), 0.0, -4.0, np.nan, np.inf, -np.inf):
            assert _refusal(mesh, factor=factor) == (-2, True), factor
            assert b"lod_factor" in L.vxb_last_error(ctx.h)
        for bad in ((np.nan, 0, 0), (0, np.inf, 0), (0, 0, -np.inf)):
            assert _refusal(mesh, camera=bad) == (-2, True), bad
        assert _refusal(mesh, count=0) == (-2, True)
        assert _refusal(mesh, planes=np.tile(good[:1], (9, 1, 1))) == (-2, True)          # view_count 9
        for value in (np.nan, np.inf, -np.inf):
            bad = good.copy(); bad[1, 4, 3] = value
            assert _refusal(mesh, planes=bad) == (-2, True)
            assert b"view 1 plane 4" in L.vxb_last_error(ctx.h)
        assert _refusal(mesh, camera=None) == (-2, True)
        assert _refusal(mesh, planes=False, count=2) == (-2, True)
        assert _refusal(mesh, out=False)[0] == -2
        assert _refusal(mesh, factor=2.0) == (0, False)                                    # the least factor is accepted
        mesh.select_cut((20.0, 40.0, 20.0), 4.0, good, lists)
        assert [_lists_bytes(l) for l in lists] == before
        # a region run without transition meshes after a complete full run: refused until the next complete full apply
        box = ctx.inject_surface(np.array([32, 30, 32], F), np.full(3, 12, F), capi.Surface.sphere((0, 0, 0), 4), 0)
        ctx.polygonize_region(box[:3], box[3:], capi.FLAG_NO_TRANSITIONS)
        mesh.apply()
        assert _refusal(mesh) == (capi.ERR_STATE, True)
        assert b"transition" in L.vxb_last_error(ctx.h)
        assert [_lists_bytes(l) for l in lists] == before
        box = ctx.inject_surface(np.array([20, 30, 40], F), np.full(3, 12, F), capi.Surface.sphere((0, 0, 0), 4), 2)
        ctx.polygonize_region(box[:3], box[3:])
        mesh.apply()
        assert _refusal(mesh) == (capi.ERR_STATE, True)                                   # a complete region run does not lift it
        ctx.polygonize()
        mesh.apply()
        assert _refusal(mesh)[0] == 0
    finally:
        mesh.close()


@pytest.mark.parametrize("max_levels, flags", [(2, 0), (0, capi.FLAG_NO_TRANSITIONS)])
def test_incomplete_full_runs_are_refused(gpu_context, max_levels, flags):
    mesh = _applied_mesh(gpu_context, "terrain128", max_levels=max_levels, flags=flags)
    try:
        assert mesh.info().levels == 4
        assert _refusal(mesh) == (capi.ERR_STATE, True)
        # the other selects and the apply behave as before
        mesh.select_lod((40.0, 70.0, 50.0), 48.0)
        mesh.select_lod_views((40.0, 70.0, 50.0), 48.0, cull_oracle.PASS_ALL[None])
    finally:
        mesh.close()


def _orbit(mesh, n, k, positions=64):
    a = 2 * np.pi * k / positions
    x, z = 0.5 * n + 0.25 * n * np.cos(a), 0.5 * n + 0.25 * n * np.sin(a)
    hit = mesh.raycast(capi.make_rays([(x, n + 8.0, z)], [(0, -1, 0)]))
    eye = (x, (hit["position"][0][1] if hit["slot"][0] != capi.VXB_RAY_MISS else 0.5 * n) + 2.0, z)
    return eye, cull_oracle.perspective(eye, (-np.sin(a), 0, np.cos(a)), (0, 1, 0), 90, 60, 0.5, 2.0 * n)


def test_terrain1024_orbit(gpu_context):
    """The orbit of tools/bench_cull.py.  At lod_factor 14.6 the cut is levels 0 and 1 for every camera: a level-2 node
    (s = 64) refines within 14.6 * 64 = 934 voxels of its box, and from the orbit (radius 256 around the centre, near the
    surface) every level-2 box of the 1024^3 grid is closer than that.  At lod_factor 4 (level l refines within 64 * 2^l)
    the cut holds at least four levels.  Culling by the frustum removes draws for most cameras."""
    n = 1024
    mesh = _applied_mesh(gpu_context, "terrain1024")
    try:
        res = mesh.download()
        boxes = cull_oracle.block_boxes(res)
        for factor, want_levels in ((14.6, 2), (4.0, 4)):
            smaller = 0
            for k in range(64):
                eye, view = _orbit(mesh, n, k)
                culled, unculled = (oracle.draw_sets(l) for l in mesh.select_cut(eye, factor, np.stack([view, cull_oracle.PASS_ALL])))
                got_levels = sorted({d[1] for d in unculled[0]})
                assert got_levels == list(range(len(got_levels))) and len(got_levels) >= want_levels, (factor, k, got_levels)
                assert unculled[1], "no transition draws"
                assert culled[0] <= unculled[0] and culled[1] <= unculled[1]
                smaller += len(culled[0]) < len(unculled[0])
                if k % 8 == 0:
                    want = oracle.expected_draws(res.records, boxes, n, res.info.levels, eye, factor, [view, cull_oracle.PASS_ALL])
                    _sets_equal(culled, want[0], "1024^3 factor %g camera %d culled" % (factor, k))
                    _sets_equal(unculled, want[1], "1024^3 factor %g camera %d unculled" % (factor, k))
            assert smaller > 32, (factor, smaller)
    finally:
        mesh.close()
