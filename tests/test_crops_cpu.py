"""The crop rule of tests/crops.py, pinned with the reference alone: every block a crop determines matches the full run of
the big grid, on terrain and on the hostile grids (big blocks, the BF_Empty neighbour skip, vertex-heavy blocks), and two
negative controls show that the comparison is live and that the rule's margin is needed."""
import functools

import numpy as np
import pytest

import crops
import gridgen

# (size of the big grid, crop size, crop origins (x, y, z), levels the crops must reach): near and far corner, interior,
# crops with one or two faces on the grid's edge.  The terrain and hostile surfaces lie across the middle of z, so their
# crops stay in that band.  A level-2 block (64^3) needs a 64-voxel margin or the grid's edge on both sides of each axis:
# the 256^3 terrain crops have room for it, the 128^3 crops only at the grid's corners, where only patchwork has content.
CASES = {
    "terrain512": (512, 256, [(0, 0, 128), (256, 256, 128), (128, 128, 128), (0, 128, 128), (128, 256, 128),
                              (256, 0, 0), (0, 256, 256)], 3),
    "patchwork256": (256, 128, [(0, 0, 0), (128, 128, 128), (64, 64, 64), (0, 64, 64), (64, 128, 64), (64, 64, 0)], 3),
    "hostile256": (256, 128, [(0, 0, 64), (128, 128, 64), (64, 64, 64), (0, 64, 64), (64, 128, 64), (128, 0, 64)], 2),
}


def _grid(name):
    if name == "terrain512":
        from voxels_b200 import synth
        return tuple(t.numpy() for t in synth.terrain(512))
    return {"patchwork256": gridgen.patchwork, "hostile256": gridgen.hostile}[name](256)


@functools.lru_cache(maxsize=None)
def _runs(reference, name):
    """The grid, the reference's full run of it and its runs of every crop of CASES."""
    n, w, origins, reached = CASES[name]
    dist, mat, blend = _grid(name)
    g = reference.grid_from_dense(dist, mat, blend)
    big = crops.reference_levels(reference, g, n)
    reference.grid_destroy(g)
    parts = {}
    for x, y, z in origins:
        cut = [np.ascontiguousarray(a[z:z + w, y:y + w, x:x + w]) for a in (dist, mat, blend)]
        g = reference.grid_from_dense(*cut)
        parts[(x, y, z)] = crops.reference_levels(reference, g, w)
        reference.grid_destroy(g)
    return big, parts


@pytest.mark.parametrize("name", sorted(CASES))
def test_crop_blocks_match_the_full_run(reference, name):
    n, w, origins, reached = CASES[name]
    big, parts = _runs(reference, name)
    totals = {}
    for origin, lv in parts.items():
        counts, problems = crops.compare_crop(lambda l: lv[l], lambda l: big[l], origin, w, len(lv))
        print("%s crop %s: blocks compared per level %s" % (name, origin, counts))
        assert not problems, "\n".join(problems[:10])
        assert counts[0] > 0, "crop %s selects no level-0 block" % (origin,)
        for l, k in counts.items():
            totals[l] = totals.get(l, 0) + k
    assert all(totals[l] > 0 for l in range(reached)), totals


@pytest.mark.parametrize("name", sorted(CASES))
def test_crop_shifted_by_one_block_fails(reference, name):
    """The crop's output laid over the big run one level-0 block off its origin must not match."""
    n, w, origins, reached = CASES[name]
    big, parts = _runs(reference, name)
    for (x, y, z), lv in parts.items():
        shifted = (x + 16 if x + w + 16 <= n else x - 16, y, z)
        _, problems = crops.compare_crop(lambda l: lv[l], lambda l: big[l], shifted, w, len(lv))
        assert problems, "crop %s compared at %s found no mismatch" % ((x, y, z), shifted)


@pytest.mark.parametrize("name", sorted(CASES))
def test_crop_blocks_without_the_margin_mismatch(reference, name):
    """Blocks on a crop face inside the grid see the crop's edge as the grid's: selecting them too finds mismatches."""
    n, w, origins, reached = CASES[name]
    big, parts = _runs(reference, name)
    inner = [o for o in parts if any(0 < c and c + w < n for c in o)]
    assert inner
    for origin in inner:
        lv = parts[origin]
        _, problems = crops.compare_crop(lambda l: lv[l], lambda l: big[l], origin, w, len(lv), margin=False)
        assert problems, "crop %s: every block matched without the margin" % (origin,)
