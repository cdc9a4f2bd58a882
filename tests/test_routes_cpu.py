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
reference's coarse cells over a skipped block read an uninitialised material, so their output is not defined."""
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
