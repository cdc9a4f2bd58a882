"""The ladder grid of the block kernels' per-block capacities (gridgen.thresholds256), pinned with the reference alone.

VxbBlockCaps (voxels_b200/csrc/vxb_emit.cuh) gives vxb_block_kernel<0|1|2> room for CAP = 1024 non-trivial cells and, at
level 0, VL = 2048 new vertices per block; a block past either goes to vxb_big_block_kernel.  The route a block takes is a
function of those two counts, so pinning the counts here pins the routes the GPU tests (tests/test_gpu_thresholds.py) reach:
  - every ladder block has its declared cell count at its level, counted from the dense array, and (level 0) its declared
    vertex count in the reference's output; every rung of every ladder is present;
  - nothing is skipped at level 0 and the reference gives the same output at 1 and 4 threads (every level is defined);
  - variant B of a flip pair changes the counts of its own block only (and of the finer blocks under it);
  - the incremental oracle: a reference run over an edited grid built from the dense arrays (a grid swap) gives the
    surface of an in-place edit, which is how the GPU flip tests get a reference for arbitrary block contents."""
import functools

import numpy as np
import pytest

import compare
import gridgen
import grids
import harness

CAP_CELLS, CAP_VERTS = 1024, 2048
LADDERS = {
    (0, "cells"): (255, 256, 257, 511, 512, 513, 1023, 1024, 1025, 4096),
    (0, "verts"): (1023, 1024, 1025, 2047, 2048, 2049),
    (1, "cells"): (511, 512, 513, 1023, 1024, 1025),
    (2, "cells"): (511, 512, 513, 1023, 1024, 1025),
}


@functools.lru_cache(maxsize=2)
def _grid(variant=None):
    return gridgen.thresholds256(variant)


def _cells(dist, level, block):
    return int(gridgen.nontrivial_cells_per_block(dist, level)[block[2], block[1], block[0]])


def _level0_vertices(reference, dist, mat, blend, threads=4):
    """{(bx, by, bz): new vertices} of level 0 in the reference's output."""
    g = reference.grid_from_dense(dist, mat, blend)
    s, _ = reference.polygonize(g, threads=threads)
    rows = reference.surface_level(s, 0).rows
    reference.surface_destroy(s); reference.grid_destroy(g)
    mn = rows["min"].astype(np.int64) // 16          # output axes (x, z, y)
    return {(int(x), int(y), int(z)): int(v) for (x, z, y), v in zip(mn, rows["nv"])}


def _variants(name):
    _, _, a, b = gridgen.TH_BLOCKS[name]
    return [(None, a)] + ([(name, b)] if b is not None else [])


def test_every_rung_is_present():
    seen = {key: set() for key in LADDERS}
    for name, (level, block, a, b) in gridgen.TH_BLOCKS.items():
        for _, cells, verts in [a] + ([b] if b else []):
            if (level, "cells") in seen:
                seen[(level, "cells")].add(cells)
            if verts is not None and cells <= CAP_CELLS:
                seen[(0, "verts")].add(verts)
    for key, rungs in LADDERS.items():
        assert set(rungs) <= seen[key], "%s: rungs missing: %s" % (key, sorted(set(rungs) - seen[key]))
    both = {(a[1], a[2]) for _, _, a, _ in gridgen.TH_BLOCKS.values()} | \
           {(b[1], b[2]) for _, _, _, b in gridgen.TH_BLOCKS.values() if b}
    for combined in ((1024, 2048), (1024, 2049), (1025, 2048)):
        assert combined in both, combined
    assert len(gridgen.TH_FLIPS) >= 5 and {gridgen.TH_BLOCKS[f][0] for f in gridgen.TH_FLIPS} == {0, 1, 2}


@pytest.mark.parametrize("variant", (None,) + gridgen.TH_FLIPS)
def test_declared_cell_counts(variant):
    """Non-trivial cells of every ladder block at its level, in the grid of every flip variant."""
    dist, _, _ = _grid(variant)
    per_level = {l: gridgen.nontrivial_cells_per_block(dist, l) for l in (0, 1, 2)}
    for name, (level, (bx, by, bz), a, b) in gridgen.TH_BLOCKS.items():
        want = (b if name == variant else a)[1]
        assert int(per_level[level][bz, by, bx]) == want, (name, variant)


def test_declared_vertex_counts_no_skip_and_threads(reference):
    """Level-0 vertices of every ladder block in the reference's output; the cell-only rungs stay within VL; no level-0
    block with non-trivial cells is skipped; the same digests at 1 and 4 threads."""
    import golden_hash
    from test_routes_cpu import skipped_blocks
    dist, mat, blend = _grid()
    nv = _level0_vertices(reference, dist, mat, blend)
    for name, (level, block, (_, cells, verts), _) in gridgen.TH_BLOCKS.items():
        if level != 0:
            continue
        if verts is not None:
            assert nv[block] == verts, (name, nv[block])
        elif cells <= CAP_CELLS:
            assert nv[block] <= CAP_VERTS, (name, nv[block])
    nb = dist.shape[0] // 16
    g = reference.grid_from_dense(dist, mat, blend)
    try:
        empty = reference.grid_empty_flags(g).reshape(nb, nb, nb).astype(bool)
        skipped = skipped_blocks(empty) & (gridgen.nontrivial_cells_per_block(dist, 0) > 0)
        assert not skipped.any(), skipped.sum()
        digests = []
        for threads in (1, 4):
            s, _ = reference.polygonize(g, threads=threads)
            digests.append([golden_hash.level_digests(reference.surface_level(s, l)) for l in range(reference.surface_levels(s))])
            reference.surface_destroy(s)
        assert digests[0] == digests[1]
    finally:
        reference.grid_destroy(g)


def _footprint(level, block, at_level):
    """The [bz, by, bx] slices of the level-`at_level` blocks under (at_level <= level) a level-`level` block."""
    r = 1 << (level - at_level)
    return tuple(slice(b * r, b * r + r) for b in reversed(block))


@pytest.mark.parametrize("name", gridgen.TH_FLIPS)
def test_flip_changes_only_its_block(reference, name):
    """Variant B differs from A only inside local 1..15 of the flip block: at its level only that block's counts change,
    at the finer levels only the blocks under it, at the coarser ones nothing."""
    level, block, a, b = gridgen.TH_BLOCKS[name]
    da, ma, ba = _grid()
    db, mb, bb = _grid(name)
    assert np.array_equal(ma, mb) and np.array_equal(ba, bb)
    m = 16 << level
    inner = np.zeros(da.shape, bool)
    inner[tuple(slice(v * m + 1, v * m + m) for v in reversed(block))] = True
    assert not (da != db)[~inner].any(), "%s: variant B differs outside local 1..15 of its block" % name
    assert np.array_equal(gridgen.th_restamp(da, name, True), db) and np.array_equal(gridgen.th_restamp(db, name, False), da)
    for l in range(4):
        ca, cb = gridgen.nontrivial_cells_per_block(da, l), gridgen.nontrivial_cells_per_block(db, l)
        allowed = np.zeros(ca.shape, bool)
        if l <= level:
            allowed[_footprint(level, block, l)] = True
        assert not (ca != cb)[~allowed].any(), "%s: cells of other level-%d blocks changed" % (name, l)
        if l == level:
            assert int(cb[block[2], block[1], block[0]]) == b[1] and int(ca[block[2], block[1], block[0]]) == a[1]
    nva, nvb = _level0_vertices(reference, da, ma, ba), _level0_vertices(reference, db, mb, bb)
    under = _footprint(level, block, 0)
    for k in set(nva) | set(nvb):
        if not all(s.start <= c < s.stop for s, c in zip(under, reversed(k))):
            assert nva.get(k) == nvb.get(k), "%s: vertices of level-0 block %s changed" % (name, k)
    if level == 0:
        assert nvb[block] == b[2] if b[2] is not None else nvb[block] <= CAP_VERTS


# ---- the incremental oracle: a grid swap gives the surface of an in-place edit -------------------------------------------

def _levels(reference, s):
    return [reference.surface_level(s, l) for l in range(reference.surface_levels(s))]


def _by_coordinate(level):
    """A LevelDump with its blocks sorted by their minimal corner and the ids cleared (a full run numbers blocks by
    coordinate, an incremental run gives the re-created blocks new ids)."""
    order = np.lexsort(level.rows["min"].T[::-1])
    parts = [level.block(int(i)) for i in order]
    rows = level.rows[order].copy()
    rows["id"] = 0

    def cat(arrs, like):
        arrs = [a for a in arrs if len(a)]
        return np.concatenate(arrs) if arrs else like[:0]
    return harness.LevelDump(rows, cat([p[1] for p in parts], level.verts), cat([p[2] for p in parts], level.idx),
                             cat([t for p in parts for t in p[3]], level.tverts), cat([t for p in parts for t in p[4]], level.tidx))


def test_grid_swap_equals_in_place_edit(reference):
    """patchwork64 with one sphere edit: the edit in place (InjectSurface + incremental Execute) and an incremental Execute
    over a new grid built from the edited dense arrays, with the same box, give the same surface, every level and the
    statistics."""
    from voxels_b200 import capi
    dist, mat, blend = grids.by_name("patchwork64")
    g1 = reference.grid_from_dense(dist, mat, blend)
    g2 = reference.grid_from_dense(dist, mat, blend)
    s1, _ = reference.polygonize(g1)
    s2, _ = reference.polygonize(g2)
    mod1, mod2 = reference.modification_create(), reference.modification_create()
    g3 = None
    try:
        box = reference.grid_inject_builtin(g1, np.array([30, 22, 37], np.float32), np.full(3, 20, np.float32),
                                            capi.Surface.sphere((0, 0, 0), 8.0), 0)
        reference.polygonize(g1, modification=mod1, surface=s1, box=box)
        edited = reference.grid_to_dense(g1)
        assert not np.array_equal(edited[0], dist)
        g3 = reference.grid_from_dense(*edited)
        reference.polygonize(g3, modification=mod2, surface=s2, box=box)
        a, b = _levels(reference, s1), _levels(reference, s2)
        assert len(a) == len(b)
        for l, (x, y) in enumerate(zip(a, b)):
            problems = compare.level_diff(x, y, "L%d" % l)
            assert not problems, "\n".join(problems[:8])
        assert np.array_equal(reference.surface_stats(s1), reference.surface_stats(s2))
    finally:
        for g in (g1, g2, g3):
            if g:
                reference.grid_destroy(g)
        reference.surface_destroy(s1); reference.surface_destroy(s2)
        reference.modification_destroy(mod1); reference.modification_destroy(mod2)


def flip_box(name):
    """The box of a flip block, in output axes (x, z, y) as the reference's edits report it: the block's extent."""
    level, (bx, by, bz), _, _ = gridgen.TH_BLOCKS[name]
    m = 16 << level
    lo = np.array([bx * m, bz * m, by * m], np.float32)
    return np.concatenate([lo, lo + m])


@pytest.mark.parametrize("name", ["L0_cells1024_verts2048", "L2_cells1024"])
def test_grid_swap_flip_equals_full_run(reference, name):
    """A thresholds256 flip A -> B by grid swap: every block of the incremental surface equals the full run of B's block
    at the same coordinate (ids aside: the re-created blocks get new ones)."""
    a, b = _grid(), _grid(name)
    ga, gb = reference.grid_from_dense(*a), reference.grid_from_dense(*b)
    sa, _ = reference.polygonize(ga)
    sb, _ = reference.polygonize(gb)
    mod = reference.modification_create()
    try:
        reference.polygonize(gb, modification=mod, surface=sa, box=flip_box(name))
        assert len(reference.modification_blocks(mod)) > 0
        x, y = _levels(reference, sa), _levels(reference, sb)
        assert len(x) == len(y)
        for l, (u, v) in enumerate(zip(x, y)):
            problems = compare.level_diff(_by_coordinate(u), _by_coordinate(v), "%s L%d" % (name, l))
            assert not problems, "\n".join(problems[:8])
    finally:
        reference.modification_destroy(mod)
        reference.surface_destroy(sa); reference.surface_destroy(sb)
        reference.grid_destroy(ga); reference.grid_destroy(gb)
