"""The block kernels' per-block capacities and the output and mesh arenas at their exact capacities, against the reference.

  a. thresholds256 (tests/gridgen.py, pinned by tests/test_thresholds_cpu.py) puts level-0, level-1 and level-2 blocks at
     exactly CAP - 1, CAP and CAP + 1 non-trivial cells and level-0 blocks at VL - 1, VL and VL + 1 new vertices
     (VxbBlockCaps, voxels_b200/csrc/vxb_emit.cuh): every level and the statistics equal the reference's, with the
     persistent kernels capped at a few CTAs (full and handed-off blocks in one CTA's item sequence) and with tiny output
     arenas (the retry while big blocks are in flight).
  b. Flip pairs in region runs: a block moves between the in-CTA path and vxb_big_block_kernel from one run to the next,
     with the consistency and material pages carried over; the reference is an incremental run over the edited grid.
  c. Output arenas at span - 1, span and span + 1 (one arena at a time, then all together): the run that fits exactly is
     accepted as is, the one that misses by one element retries; both give the unconstrained run's output.  The
     cell-record arena has no setter and no reported total, so it is not covered here.
  d. Mesh arenas at exact fit: a model of vxb_mesh_apply's rule (append at the tail, compact, grow) predicts every
     apply's compactions, growths, capacities and spans; the mesh equals the reference's incremental surface and a batch
     of rays equals the numpy oracle on the mesh's own arenas, which the query kernels read up to their last element.
The file takes about 70 seconds on one H100 80GB (700 W)."""
import functools

import numpy as np
import pytest

import compare
import golden_hash
import gridgen
import grids
import harness
import raycast_oracle
from parity import run_both
from test_gpu_mesh import _assert_mesh, _grid, _terrain_edits
from test_gpu_gridstore import _tail
from test_gpu_raycast import assert_same, axis_rays, camera_rays, random_rays
from test_thresholds_cpu import flip_box

pytestmark = pytest.mark.gpu

LIMITS = (0, 1, 2, 3, 7)


@functools.lru_cache(maxsize=1)
def _thresholds():
    return gridgen.thresholds256()


def _context(limit=0, capacity=None):
    import voxels_b200
    ctx = voxels_b200.Context(0)
    ctx.set_launch_limit(limit)
    if capacity:
        ctx.set_capacity(*capacity)
    return ctx


# ---- a. full runs ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("limit", LIMITS)
def test_thresholds256_every_level(reference, limit):
    ctx = _context(limit)
    try:
        problems, _ = run_both(reference, ctx, *_thresholds())
        assert not problems, ("launch limit %d:\n" % limit) + "\n".join(problems[:10])
    finally:
        ctx.close()


def test_thresholds256_tiny_arenas_retry(reference):
    ctx = _context(2, (1024, 1024, 64, 64))
    try:
        problems, _ = run_both(reference, ctx, *_thresholds())
        assert not problems, "\n".join(problems[:10])
    finally:
        ctx.close()


# ---- b. flip pairs in region runs ------------------------------------------------------------------------------------------

def _level0_blocks(name):
    """The level-0 blocks (x, y, z) under a flip block."""
    level, (bx, by, bz), _, _ = gridgen.TH_BLOCKS[name]
    r = 1 << level
    return [(bx * r + x, by * r + y, bz * r + z) for z in range(r) for y in range(r) for x in range(r)]


def _blocks_of(vol, coords):
    return np.ascontiguousarray(np.stack([vol[16 * z:16 * z + 16, 16 * y:16 * y + 16, 16 * x:16 * x + 16].ravel() for x, y, z in coords]))


def _assert_region_result(reference, surf, ctx, what):
    """The context's result after a region run: the re-created blocks, the tail of every reference level (:443-450, :1293)."""
    part = ctx.download()
    for l in range(ctx.region_info().levels):
        want = reference.surface_level(surf, l)
        got = part.level(l)
        k = len(got.rows)
        tail = harness.LevelDump(want.rows[len(want.rows) - k:], *_tail(want, k))
        problems = compare.level_diff(tail, got, "%s L%d" % (what, l))
        assert not problems, "\n".join(problems[:5])


@pytest.mark.parametrize("limit", (0, 2))
def test_flips_in_region_runs(reference, limit):
    """Every flip pair A -> B -> A, one block per region run: vxb_grid_update_blocks with the block's new bytes,
    vxb_polygonize_region over its box, vxb_mesh_apply.  The reference runs incrementally over the edited grid."""
    dist, mat, blend = _thresholds()
    ctx = _context(limit)
    g = reference.grid_from_dense(dist, mat, blend)
    surf, _ = reference.polygonize(g)
    live = [g]
    mod = reference.modification_create()
    mesh = None
    try:
        ctx.set_materials(None, None)
        ctx.upload_dense(dist, mat, blend)
        ctx.polygonize()
        mesh = ctx.mesh()
        mesh.apply()
        _assert_mesh(reference, surf, mesh, "full run")
        cur = dist
        for name in gridgen.TH_FLIPS:
            coords = _level0_blocks(name)
            box = flip_box(name)
            for to_b in (True, False):
                cur = gridgen.th_restamp(cur, name, to_b)
                live.append(reference.grid_from_dense(cur, mat, blend))
                reference.polygonize(live[-1], modification=mod, surface=surf, box=box)
                ctx.update_blocks(np.array(coords, np.uint32), _blocks_of(cur, coords))
                ctx.polygonize_region(box[:3], box[3:])
                what = "%s -> %s" % (name, "B" if to_b else "A")
                _assert_region_result(reference, surf, ctx, what)
                mesh.apply()
                _assert_mesh(reference, surf, mesh, what)
        assert np.array_equal(cur, dist)
    finally:
        if mesh is not None:
            mesh.close()
        ctx.close()
        reference.modification_destroy(mod); reference.surface_destroy(surf)
        for x in live:
            reference.grid_destroy(x)


# ---- c. output arenas at exact fit -----------------------------------------------------------------------------------------

def _spans(info):
    return (info.vertex_span, info.index_span, info.trans_vertex_span, info.trans_index_span)


def _totals(info):
    return (info.vertex_total, info.index_total, info.trans_vertex_total, info.trans_index_total, info.block_count)


def _digest(ctx, info):
    res = ctx.download()
    return [golden_hash.level_digests(res.level(l)) for l in range(info.levels_total)], [int(v) for v in res.stats]


@pytest.mark.parametrize("name", ["hostile64", "patchwork128", "thresholds256"])
def test_output_arenas_at_exact_fit(reference, name):
    dist, mat, blend = _thresholds() if name == "thresholds256" else grids.by_name(name)
    for limit in (0, 2):
        ctx = _context(limit)
        try:
            if limit == 0:   # the unconstrained run, once against the reference
                problems, _ = run_both(reference, ctx, dist, mat, blend)
                assert not problems, "\n".join(problems[:10])
            else:
                ctx.set_materials(None, None)
                ctx.upload_dense(dist, mat, blend)
            info = ctx.polygonize()
            spans, totals, want = _spans(info), _totals(info), _digest(ctx, info)
            # thresholds256 has no transition cells (its content lies inside the blocks): those arenas stay empty
            used = [a for a in range(4) if spans[a] > 1]
            assert used[:2] == [0, 1] and (name == "thresholds256" or len(used) == 4), spans
            large = [2 * s + 4096 for s in spans]
            for arenas in [[a] for a in used] + [used]:
                for delta in (-1, 0, 1):
                    cap = list(large)
                    for a in arenas:
                        cap[a] = spans[a] + delta
                    ctx.set_capacity(*cap)
                    got = ctx.polygonize()
                    what = "%s limit %d capacity %s (spans %s)" % (name, limit, cap, spans)
                    assert _spans(got) == spans and _totals(got) == totals, what
                    assert _digest(ctx, got) == want, what
        finally:
            ctx.close()   # the capacities were the context's: nothing to restore on another one


# ---- d. mesh arenas at exact fit -------------------------------------------------------------------------------------------

def _elems(recs):
    """The arena elements of directory records: vertices, indices and transition indices padded to 4 per range."""
    if len(recs) == 0:
        return np.zeros(4, np.int64)
    pad = lambda c: (c.astype(np.int64) + 3) // 4 * 4
    return np.array([recs["vertex_count"].astype(np.int64).sum(), pad(recs["index_count"]).sum(),
                     recs["trans_vertex_count"].astype(np.int64).sum(), pad(recs["trans_index_count"]).sum()], np.int64)


def _dirty(recs, region, n):
    """Records whose block lies in the region run's dirty range of its level (vxb_mesh_dirty)."""
    out = np.zeros(len(recs), bool)
    for k, r in enumerate(recs):
        l = int(r["level"]); m = 16 << l; nb = (n // 16) >> l
        cid = int(r["coord_id"])
        b = (cid % nb, (cid // nb) % nb, cid // (nb * nb))
        lo, hi = region.min_dirty[l], region.max_dirty[l]      # output axes (x, z, y)
        lo3, hi3 = (lo[0] / m, lo[2] / m, lo[1] / m), (hi[0] / m, hi[2] / m, hi[1] / m)
        out[k] = all(lo3[a] <= b[a] < hi3[a] for a in range(3))
    return out


def _grown(live):
    return (max(live + live // 2, 1024) + 3) & ~3


class MeshModel:
    """vxb_mesh_apply's documented rule: compact iff, for any arena, tail + fresh > capacity or tail - survivors > live;
    grow iff live > capacity, to max(1.5 live, 1024) rounded up to 4.  A full apply replaces the content (no compaction)."""

    def __init__(self, capacity):
        self.cap = [(c + 3) & ~3 for c in capacity]     # vxb_mesh_create rounds every capacity up to 4
        self.span = [0, 0, 0, 0]
        self.compactions = self.growths = 0

    def apply(self, mesh_recs, run_recs, region, n):
        surv = _elems(mesh_recs[~_dirty(mesh_recs, region, n)]) if region is not None else np.zeros(4, np.int64)
        fresh = _elems(run_recs)
        live = surv + fresh
        tail = self.span if region is not None else [0, 0, 0, 0]
        new_cap = [_grown(int(live[a])) if live[a] > self.cap[a] else self.cap[a] for a in range(4)]
        grow = new_cap != self.cap
        compact = region is not None and any(tail[a] + fresh[a] > self.cap[a] or tail[a] - surv[a] > live[a] for a in range(4))
        had = any(self.cap)
        self.span = [int(live[a]) if (compact or region is None) else int(tail[a] + fresh[a]) for a in range(4)]
        self.cap = new_cap
        self.compactions += int(compact)
        self.growths += int(grow and had)
        return compact, grow

    def check(self, info, what):
        got = (list(info.capacity), [info.vertex_span, info.index_span, info.trans_vertex_span, info.trans_index_span],
               info.compactions, info.growths)
        assert got == (self.cap, self.span, self.compactions, self.growths), "%s: mesh %s, model %s" % (
            what, got, (self.cap, self.span, self.compactions, self.growths))


def _rays(res, rng):
    n = res.n
    return np.concatenate([random_rays(n, 96, rng), camera_rays(res, 96, rng), axis_rays(n, rng)[::5]])


def _assert_rays(mesh, rng, what):
    res = mesh.download()
    rays = _rays(res, rng)
    assert_same(mesh.raycast(rays), raycast_oracle.raycast(res, rays), rays, what)


def _run_state(ctx, region):
    """(run directory, dirty range or None) of the context's last run."""
    return ctx.download().records, (ctx.region_info() if region else None)


# an additive edit of _terrain_edits after which every arena's span is a multiple of 4: the mesh keeps its capacities in
# granules of 4 elements (vxb_mesh_create and grownCapacity round up to 4), so only such a span can end exactly at one
EDGE_EDIT = 10


def _ceil4(v):
    return (v + 3) & ~3


def test_mesh_arenas_at_exact_fit(reference, gpu_context):
    """One mesh per case on one context, every mesh applies every run: the full run, then EDGE_EDIT with capacity[a] in
    {S1, S1 - 4, ceil4(L1), ceil4(L1) - 4} (S1 = the spans after the region apply without compaction, L1 = the live data
    after it; the other arenas large) and all arenas at S1; then the other edits through the S1 and the ceil4(L1) - 4
    meshes of the vertex and the index arena."""
    n = 128
    ctx = gpu_context
    ctx.set_materials(None, None)
    g = _grid(reference, ctx, "terrain128")
    surf, _ = reference.polygonize(g)
    mod = reference.modification_create()
    edits = _terrain_edits(reference, g, n)
    assert edits[EDGE_EDIT][3] == 0   # an edit that adds
    meshes = []
    try:
        # the probe: large arenas, so that the region run is appended at the tail
        ctx.polygonize()
        probe = ctx.mesh((1 << 22, 1 << 22, 1 << 20, 1 << 20))
        meshes.append(probe)
        probe.apply()
        s0 = _spans(probe.info())
        pos, ext, sph, kind = edits[EDGE_EDIT]
        box = reference.grid_inject_builtin(g, pos, ext, sph, kind)
        got_box = ctx.inject_surface(pos, ext, sph, kind)
        assert np.array_equal(box, got_box)
        ctx.polygonize_region(box[:3], box[3:])
        probe.apply()
        pi = probe.info()
        assert pi.compactions == 0 and pi.growths == 0
        s1 = _spans(pi)
        l1 = tuple(int(v) for v in _elems(probe.download().records))
        assert all(a <= b for a, b in zip(l1, s1)) and all(a <= b for a, b in zip(s0, s1)), (s0, s1, l1)
        assert all(v % 4 == 0 for v in s1) and all(a <= _ceil4(b) - 4 for a, b in zip(s0, l1)), (s0, s1, l1)
        probe.close(); meshes.remove(probe)

        # one mesh per case; every mesh takes the full run and then the region run of EDGE_EDIT
        large = [4 * s + 4096 for s in s1]
        cases = []
        for a in range(4):
            for label, v in (("S1", s1[a]), ("S1-4", s1[a] - 4), ("ceil4(L1)", _ceil4(l1[a])), ("ceil4(L1)-4", _ceil4(l1[a]) - 4)):
                cap = list(large); cap[a] = v
                cases.append(("arena %d at %s" % (a, label), cap))
        cases.append(("all arenas at S1", list(s1)))
        reference.surface_destroy(surf); reference.grid_destroy(g)
        g = _grid(reference, ctx, "terrain128")   # the grid again, before edit 0
        surf, _ = reference.polygonize(g)
        ctx.polygonize()
        run = _run_state(ctx, False)
        models = []
        for what, cap in cases:
            mesh = ctx.mesh(cap)
            meshes.append(mesh)
            model = MeshModel(cap)
            model.apply(None, run[0], None, n)
            mesh.apply()
            model.check(mesh.info(), what + ", full run")
            models.append(model)
        _assert_mesh(reference, surf, meshes[0], "full run")
        rng = np.random.RandomState(5)

        def region_step(i, sel):
            pos, ext, sph, kind = edits[i]
            box = reference.grid_inject_builtin(g, pos, ext, sph, kind)
            reference.polygonize(g, modification=mod, surface=surf, box=box)
            got_box = ctx.inject_surface(pos, ext, sph, kind)
            assert np.array_equal(box, got_box)
            ctx.polygonize_region(got_box[:3], got_box[3:])
            recs, region = _run_state(ctx, True)
            for k in sel:
                (what, _), mesh, model = cases[k], meshes[k], models[k]
                before = mesh.download().records
                outcome = model.apply(before, recs, region, n)
                mesh.apply()
                model.check(mesh.info(), "%s, edit %d" % (what, i))
                _assert_mesh(reference, surf, mesh, "%s, edit %d" % (what, i))
                _assert_rays(mesh, rng, "%s, edit %d" % (what, i))
                yield k, outcome, mesh.info()

        outcomes = {k: (o, info) for k, o, info in region_step(EDGE_EDIT, range(len(cases)))}
        # the cases reach the edges they were built for: the tail ends exactly at the capacity / one granule past it
        # (compaction); the live data fills the compacted arena / one granule too many (growth)
        for a in range(4):
            (c, gr), i = outcomes[4 * a]
            assert not c and not gr and _spans(i)[a] == i.capacity[a] == s1[a], "arena %d at S1" % a
            (c, gr), i = outcomes[4 * a + 1]
            assert c and not gr and _spans(i)[a] == l1[a] and i.capacity[a] == s1[a] - 4, "arena %d at S1 - 4" % a
            (c, gr), i = outcomes[4 * a + 2]
            assert c and not gr and _spans(i)[a] == l1[a] and i.capacity[a] == _ceil4(l1[a]), "arena %d at ceil4(L1)" % a
            (c, gr), i = outcomes[4 * a + 3]
            assert c and gr and i.capacity[a] == _grown(l1[a]), "arena %d at ceil4(L1) - 4" % a
        (c, gr), i = outcomes[len(cases) - 1]
        assert not c and not gr and _spans(i) == tuple(i.capacity) == s1
        # the other edits through the S1 and ceil4(L1) - 4 meshes of the vertex and the index arena
        keep = [0, 3, 4, 7]
        for k in range(len(cases)):
            if k not in keep:
                meshes[k].close()
        for i in [k for k in range(len(edits)) if k != EDGE_EDIT]:
            for _ in region_step(i, keep):
                pass
    finally:
        for m in meshes:
            m.close()
        reference.modification_destroy(mod); reference.surface_destroy(surf); reference.grid_destroy(g)
