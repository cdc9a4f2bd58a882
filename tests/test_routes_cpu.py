"""The patchwork grids (tests/gridgen.py) reach every hand-off route and every grid edge of the kernels: counted from
the dense arrays and the reference's own output, so a change of the generator that loses a route fails here instead of
silently thinning the GPU tests (tests/test_gpu_paths.py) that rely on it.

Routes (DESIGN.md section 2):
  - a level-0 block with more than 1024 non-trivial cells -> vxb_big_block_kernel
  - a level-0 block with at most 1024 non-trivial cells but more than 2048 vertices -> vxb_big_block_kernel (!inCta)
  - a level-1 / level-2 block with more than 1024 non-trivial cells -> vxb_big_block_kernel
  - emitted blocks on every face, edge and corner of the grid, at level 0 and at the coarsest level of 2^3 blocks or more
and, in the grid built for it (gridgen.skip_quirk), the level-0 skip of a block whose 27-neighbourhood is BF_Empty although
the surface runs along its faces (TransVoxelImpl.cpp:520).  The patchwork grids must never reach that skip: the
reference's coarse cells over a skipped block read an uninitialised material, so their output is not defined.

Here a route only has to be reached; the exact edges of the capacities (1023 / 1024 / 1025 cells at levels 0-2, 2047 /
2048 / 2049 level-0 vertices, both at once, and the flips between them) live in the threshold grid, gridgen.thresholds256,
whose counts tests/test_thresholds_cpu.py pins.

The grid store's thresholds are pinned the same way: the rle_edges grids reach BF_Empty through the walk of
vxb_block_info_kernel with both outcomes, the 2048 / 2049-run codec boundary in all three channels, and (only
rle_edges_skipped) the skip; hostile64_full_range spans the whole int8 range."""
import itertools

import numpy as np
import pytest

import gridgen
import grids

CAP_CELLS, CAP_VERTS = 1024, 2048


def _positions(nb):
    """The face / edge / corner classes a block grid of nb blocks per axis has: per axis low, high or (nb >= 3) between."""
    axis = ["lo", "hi"] + (["mid"] if nb >= 3 else [])
    return {c for c in itertools.product(axis, repeat=3) if c != ("mid",) * 3}


def _position(b, nb):
    return tuple("lo" if v == 0 else ("hi" if v == nb - 1 else "mid") for v in b)


def _block_coords(rows, level):
    """(bx, by, bz) of every row of a level dump: the corners are in output axes (x, z, y)."""
    m = 16 << level
    mn = rows["min"].astype(np.int64) // m
    return mn[:, 0], mn[:, 2], mn[:, 1]


def routes(reference, dist, mat, blend):
    n = dist.shape[0]
    g = reference.grid_from_dense(dist, mat, blend)
    empty = reference.grid_empty_flags(g).reshape((n >> 4,) * 3).astype(bool)
    s, _ = reference.polygonize(g)
    levels = [reference.surface_level(s, l) for l in range(reference.surface_levels(s))]
    reference.surface_destroy(s); reference.grid_destroy(g)
    out = {}
    nt0 = gridgen.nontrivial_cells_per_block(dist, 0)
    out["L0 skipped with non-trivial cells"] = int((skipped_blocks(empty) & (nt0 > 0)).sum())
    out["L0 > 1024 cells"] = int((nt0 > CAP_CELLS).sum())
    bx, by, bz = _block_coords(levels[0].rows, 0)
    heavy = (levels[0].rows["nv"] > CAP_VERTS) & (nt0[bz, by, bx] <= CAP_CELLS)
    out["L0 <= 1024 cells, > 2048 vertices"] = int(heavy.sum())
    for l in (1, 2):
        out["L%d > 1024 cells" % l] = int((gridgen.nontrivial_cells_per_block(dist, l) > CAP_CELLS).sum())
    coarse = max(l for l in range(len(levels)) if (n >> (4 + l)) >= 2 and len(levels[l].rows))
    for l in (0, coarse):
        nb = n >> (4 + l)
        bx, by, bz = _block_coords(levels[l].rows, l)
        seen = {_position(b, nb) for b in zip(bx, by, bz)}
        out["L%d face/edge/corner classes missing" % l] = sorted(_positions(nb) - seen)
    return out


def skipped_blocks(empty):
    """AreBlockAndNeighborsEmpty (TransVoxelImpl.cpp:1511-1527) of every level-0 block: its clamped 27-neighbourhood
    is BF_Empty.  empty = [bz, by, bx] flags."""
    nb = empty.shape[0]
    pad = np.pad(empty, 1, mode="edge")
    out = np.ones_like(empty)
    for dz, dy, dx in itertools.product(range(3), repeat=3):
        out &= pad[dz:dz + nb, dy:dy + nb, dx:dx + nb]
    return out


def test_skip_quirk_grid_reaches_the_skip(reference):
    dist, mat, blend = gridgen.skip_quirk()
    g = reference.grid_from_dense(dist, mat, blend)
    empty = reference.grid_empty_flags(g).reshape(4, 4, 4).astype(bool)
    reference.grid_destroy(g)
    skipped = skipped_blocks(empty) & (gridgen.nontrivial_cells_per_block(dist, 0) > 0)
    assert skipped.sum() >= 8 and not skipped.all(), skipped.sum()


@pytest.mark.parametrize("name", ["patchwork64", "patchwork128", "patchwork256"])
def test_patchwork_reaches_every_route(reference, name):
    dist, mat, blend = grids.by_name(name)
    got = routes(reference, dist, mat, blend)
    print("\n%s: %s" % (name, got))
    for what, v in got.items():
        if what.endswith("missing"):
            assert not v, "%s: %s: %s" % (name, what, v)
        elif what.startswith("L0 skipped"):
            assert v == 0, "%s: %d level-0 blocks are skipped although they have non-trivial cells" % (name, v)
        else:
            assert v > 0, "%s reaches no block of the route '%s'" % (name, what)


def test_patchwork_is_deterministic_and_bounded():
    a = gridgen.patchwork(128)
    b = gridgen.patchwork(128)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    kinds = gridgen.patchwork_kinds(1024)
    assert 1000 < int((kinds != gridgen.UNI_POS).sum()) < 20000   # a bounded amount of work at 1024^3
    for k in range(len(gridgen.KIND_NAMES)):
        assert (gridgen.patchwork_kinds(128) == k).any(), "patchwork128 has no %s block" % gridgen.KIND_NAMES[k]


# ---- the grid store's thresholds (gridgen.rle_edges_*, hostile64_full_range; tests/test_gpu_gridstore_edges.py) ------

RLE_EDGES = ("rle_edges_kept", "rle_edges_skipped")
BF_EMPTY = 1


def _blocks(a):
    """Every 16^3 block of a as a row of 4096 bytes in CompressBlock's order, block order z, y, x."""
    nb = a.shape[0] // 16
    return a.reshape(nb, 16, nb, 16, nb, 16).transpose(0, 2, 4, 1, 3, 5).reshape(-1, 4096)


def _pack_table(blob, nb):
    """(sizes [blocks, 3], flags [blocks]) of a PackForSave blob."""
    sizes = blob[16:16 + nb ** 3 * 12].view(np.uint32).reshape(-1, 3).astype(np.int64)
    offsets = 16 + nb ** 3 * 12 + np.concatenate([[0], np.cumsum(4 + sizes.sum(axis=1))[:-1]])
    flags = np.array([int(blob[o:o + 4].view(np.uint32)[0]) for o in offsets])
    return sizes, flags


def _reference_state(reference, dist, mat, blend):
    g = reference.grid_from_dense(dist, mat, blend)
    try:
        return reference.grid_empty_flags(g), reference.grid_pack(g)
    finally:
        reference.grid_destroy(g)


@pytest.mark.parametrize("name", RLE_EDGES)
def test_rle_edges_empty_flags(reference, restatement, name):
    """Every threshold block has the BF_Empty flag it was built for in the reference, and the restatement agrees."""
    dist, mat, blend = grids.by_name(name)
    nb = dist.shape[0] // 16
    empty, _ = _reference_state(reference, dist, mat, blend)
    want = name == "rle_edges_skipped"
    for kind, s, (bx, by, bz) in gridgen.rle_edges_thresholds(name):
        assert bool(empty[(bz * nb + by) * nb + bx]) == want, "%s %+d at block %s" % (kind, s, (bx, by, bz))
    h = restatement.run(dist, mat, blend)
    try:
        assert np.array_equal(restatement.empty_flags(h, dist.shape[0]), empty)
    finally:
        restatement.destroy(h)


def test_rle_edges_reach_the_walk_both_ways(reference):
    """A numpy model of the scan's in-row count: one-signed blocks with a count in [1777, 2047] are walked, with both
    outcomes; one-signed blocks with 2048 are decided non-empty without a walk; 1776 is not walked.  The model's run count
    (runs of one value cut every 255 bytes) decides BF_Empty exactly as the reference does."""
    seen = set()
    for name in RLE_EDGES:
        dist, mat, blend = grids.by_name(name)
        empty, _ = _reference_state(reference, dist, mat, blend)
        for b, flat in enumerate(_blocks(dist)):
            one_signed = (flat > 0).all() or (flat < 0).all()
            changes, runs = gridgen.inrow_changes(flat), gridgen.runs_of(flat)
            assert bool(empty[b]) == (one_signed and runs <= 2048), "%s block %d: %d runs" % (name, b, runs)
            if not one_signed:
                continue
            if 1777 <= changes < 2048:
                seen.add(("walked", bool(empty[b]), runs))
            elif changes >= 2048:
                seen.add(("non-empty without a walk", bool(empty[b]), None))
            seen.add(("in-row", changes))
    for want in [("walked", True, 2047), ("walked", True, 2048), ("walked", False, 2049),
                 ("non-empty without a walk", False, None), ("in-row", 1776), ("in-row", 1777), ("in-row", 2047), ("in-row", 2048)]:
        assert want in seen, want


def test_rle_edges_pack_table(reference):
    """PackForSave's size table holds channels of exactly 4096 run-length coded bytes (raw flag clear, 2048 runs) next to
    raw ones, in all three channels; the model's run count gives every size."""
    coded4096, raw = set(), set()
    for name in RLE_EDGES:
        arrays = grids.by_name(name)
        nb = arrays[0].shape[0] // 16
        _, blob = _reference_state(reference, *arrays)
        sizes, flags = _pack_table(blob, nb)
        for ch, a in enumerate(arrays):
            runs = np.array([gridgen.runs_of(flat) for flat in _blocks(a)])
            is_raw = (flags >> (1 + ch)) & 1 == 1
            assert np.array_equal(is_raw, runs > 2048), (name, ch)
            assert np.array_equal(sizes[:, ch], np.where(is_raw, 4096, 2 * runs)), (name, ch)
            if ((sizes[:, ch] == 4096) & ~is_raw).any():
                coded4096.add(ch)
            if is_raw.any():
                raw.add(ch)
    assert coded4096 == raw == {0, 1, 2}, (coded4096, raw)


@pytest.mark.parametrize("name", RLE_EDGES + ("hostile64_full_range",))
def test_rle_edges_skip_and_full_range(reference, name):
    """rle_edges_skipped skips level-0 blocks with non-trivial cells; rle_edges_kept and hostile64_full_range skip none
    (their coarse levels are defined in the reference: it gives the same output at 1 and 4 threads)."""
    import golden_hash
    dist, mat, blend = grids.by_name(name)
    nb = dist.shape[0] // 16
    empty, _ = _reference_state(reference, dist, mat, blend)
    skipped = skipped_blocks(empty.reshape(nb, nb, nb).astype(bool)) & (gridgen.nontrivial_cells_per_block(dist, 0) > 0)
    if name == "rle_edges_skipped":
        assert skipped.sum() >= 8, skipped.sum()
        return
    assert not skipped.any(), skipped.sum()
    g = reference.grid_from_dense(dist, mat, blend)
    digests = []
    for threads in (1, 4):
        s, _ = reference.polygonize(g, threads=threads)
        digests.append([golden_hash.level_digests(reference.surface_level(s, l)) for l in range(reference.surface_levels(s))])
        reference.surface_destroy(s)
    reference.grid_destroy(g)
    assert digests[0] == digests[1]


def test_full_range_grid_spans_int8():
    dist, _, _ = grids.by_name("hostile64_full_range")
    d = dist.astype(np.int64)
    assert d.min() == -128 and d.max() == 127 and (d == 0).any()
    assert len(np.unique(d)) == 256
    for axis in range(3):   # (-128, 127) and (127, -128) on cell edges along every axis
        a, b = np.moveaxis(d, axis, 0)[:-1], np.moveaxis(d, axis, 0)[1:]
        assert ((a == -128) & (b == 127)).any() and ((a == 127) & (b == -128)).any(), axis
