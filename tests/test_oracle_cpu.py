"""CPU tests of the test infrastructure itself (no GPU): the CPU restatement (oracle/restate) is pinned
  (a) against the unmodified reference compiled under oracle/_ref, when that build is present, and
  (b) against the committed digests of the reference's output (tests/golden/reference_hashes.json)."""
import json
import os

import numpy as np
import pytest

import compare
import golden_hash
import grids

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_hashes.json")


def golden():
    with open(GOLDEN) as f:
        return json.load(f)["grids"]


@pytest.mark.parametrize("name", sorted(grids.SMALL))
def test_restatement_matches_reference(reference, restatement, name):
    dist, mat, blend = grids.SMALL[name]()
    g = reference.grid_from_dense(dist, mat, blend)
    s, _ = reference.polygonize(g, threads=4)
    h = restatement.run(dist, mat, blend)
    assert np.array_equal(reference.grid_empty_flags(g), restatement.empty_flags(h, dist.shape[0])), "BF_Empty rule"
    assert np.array_equal(reference.surface_stats(s), restatement.stats(h))
    for l in range(reference.surface_levels(s)):
        a, b = reference.surface_level(s, l), restatement.level(h, l)
        assert not compare.level_diff(a, b, "L%d" % l)
        assert compare.normals_max_ulp(a, b) == 0
    reference.surface_destroy(s); reference.grid_destroy(g); restatement.destroy(h)


@pytest.mark.parametrize("name", sorted(grids.SMALL) + ["hostile128"])
def test_restatement_matches_golden_digests(restatement, name):
    dist, mat, blend = (grids.SMALL.get(name) or grids.MEDIUM[name])()
    want = golden()[name]
    assert golden_hash.input_digest(dist, mat, blend) == want["input_sha256"], "test grid generator changed: regenerate the golden file"
    h = restatement.run(dist, mat, blend)
    assert [int(v) for v in restatement.stats(h)] == want["stats"]
    assert restatement.levels(h) == len(want["levels"])
    for l, w in enumerate(want["levels"]):
        got = golden_hash.level_digests(restatement.level(h, l))
        assert got["counts"] == w["counts"], "level %d counts" % l
        assert got["exact"] == w["exact"], "level %d bit-exact fields" % l
        assert got["normals"] == w["normals"], "level %d normals (0 ULP expected on x86-64 without FMA)" % l
    restatement.destroy(h)


def test_reference_determinism_across_threads(reference):
    """The reference is bit-deterministic across OpenMP thread counts (SURVEY.md section 4.3)."""
    dist, mat, blend = grids.SMALL["hostile64"]()
    g = reference.grid_from_dense(dist, mat, blend)
    dumps = []
    for threads in (1, 4):
        s, _ = reference.polygonize(g, threads=threads)
        dumps.append([golden_hash.level_digests(reference.surface_level(s, l)) for l in range(reference.surface_levels(s))])
        reference.surface_destroy(s)
    reference.grid_destroy(g)
    assert dumps[0] == dumps[1]


def test_reference_config1_anchors(reference):
    """BASELINE config 1 (64^3 sphere) through Grid::Create + Polygonizer::Execute: the survey's expected counts."""
    g = reference.grid_sphere(64, (32, 32, 32), 19.2)
    s, _ = reference.polygonize(g, threads=2)
    st = reference.surface_stats(s)
    assert reference.surface_levels(s) == 3 and st[0] == 73 and st[2] == 9096
    l0 = reference.surface_level(s, 0)
    assert len(l0.verts) == 8832 and len(l0.idx) == 41496
    assert int((l0.verts["tex"][:, 0] != 0).sum()) == 0  # Reserved byte is value-initialised to 0
    reference.surface_destroy(s); reference.grid_destroy(g)


def test_terrain_generator_is_deterministic_and_parity_on_it(reference, restatement):
    from voxels_b200 import synth
    d1, m1, b1 = (t.numpy() for t in synth.terrain(64))
    d2, m2, b2 = (t.numpy() for t in synth.terrain(64))
    assert np.array_equal(d1, d2) and np.array_equal(m1, m2) and np.array_equal(b1, b2)
    assert d1.min() == -4 and d1.max() == 4 and set(np.unique(m1)) <= {0, 1, 2, 3}
    g = reference.grid_from_dense(d1, m1, b1)
    s, _ = reference.polygonize(g, threads=4)
    h = restatement.run(d1, m1, b1)
    for l in range(reference.surface_levels(s)):
        assert not compare.level_diff(reference.surface_level(s, l), restatement.level(h, l), "L%d" % l)
    reference.surface_destroy(s); reference.grid_destroy(g); restatement.destroy(h)


def test_skip_quirk_level0_and_statistics(reference, restatement):
    """Level-0 blocks skipped with their BF_Empty neighbourhood although the surface runs along their faces (:520).  The
    coarse cells over them read an uninitialised Cell::Material in the reference (:1052-1086; the texture bytes of their
    vertices change with the thread count), which this project defines as {EMPTY, 0}; level 0 and the statistics are
    defined and must match."""
    import gridgen
    dist, mat, blend = gridgen.skip_quirk()
    g = reference.grid_from_dense(dist, mat, blend)
    s, _ = reference.polygonize(g, threads=4)
    h = restatement.run(dist, mat, blend)
    assert np.array_equal(reference.grid_empty_flags(g), restatement.empty_flags(h, dist.shape[0]))
    assert np.array_equal(reference.surface_stats(s), restatement.stats(h))
    assert reference.surface_levels(s) == restatement.levels(h)
    assert not compare.level_diff(reference.surface_level(s, 0), restatement.level(h, 0), "L0")
    assert len(reference.surface_level(s, 1).rows) > 0      # the coarse levels do have a surface over the skipped blocks
    reference.surface_destroy(s); reference.grid_destroy(g); restatement.destroy(h)
