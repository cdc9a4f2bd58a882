"""The persistent-loop, coarse-lattice and grid-edge paths of the kernels on hostile content, against the reference.

The work-list kernels launch an occupancy-sized grid, so on a small grid every CTA takes at most one work item and the
code that runs only from a CTA's second item on (the two-ahead cursor, the re-issued level-0 tile, the mbarrier phase
flip, the double-buffer swap of the levels >= 1, the per-CTA accumulators, the item loops of the big-block and
transition kernels) never sees hostile content.  vxb_set_launch_limit caps those grids at a few CTAs, so each one
walks many items of mixed kinds.  patchwork512 / patchwork1024 reach the coarse lattice of mode 1 (level 2 of a
1024^3 grid) with big blocks on it."""
import pytest

import gridgen
import grids
from parity import run_both, run_skipping_grid

pytestmark = pytest.mark.gpu

HOSTILE = sorted(name for name in list(grids.SMALL) + list(grids.MEDIUM)
                 if name.startswith(("hostile", "noise", "patchwork")))
LIMITS = (1, 2, 3, 7)


def _context(limit, capacity=None):
    import voxels_b200
    ctx = voxels_b200.Context(0)
    ctx.set_launch_limit(limit)
    if capacity:
        ctx.set_capacity(*capacity)
    return ctx


@pytest.mark.parametrize("name", HOSTILE)
def test_few_ctas_all_levels(reference, name):
    dist, mat, blend = grids.by_name(name)
    for limit in LIMITS:
        ctx = _context(limit)
        try:
            problems, res = run_both(reference, ctx, dist, mat, blend)
            assert not problems, ("launch limit %d:\n" % limit) + "\n".join(problems[:10])
        finally:
            ctx.close()


@pytest.mark.parametrize("name", HOSTILE)
def test_few_ctas_level0_regular_cells(reference, name):
    import voxels_b200
    dist, mat, blend = grids.by_name(name)
    ctx = _context(2)
    try:
        problems, res = run_both(reference, ctx, dist, mat, blend, max_levels=1, flags=voxels_b200.FLAG_NO_TRANSITIONS)
        assert not problems, "\n".join(problems[:10])
    finally:
        ctx.close()


@pytest.mark.parametrize("name", ["hostile64", "patchwork64", "patchwork128", "noise64"])
def test_few_ctas_tiny_arenas_retry(reference, name):
    """The arenas overflow while the CTAs still hold later items: the run must notice, grow and still match."""
    dist, mat, blend = grids.by_name(name)
    ctx = _context(2, (1024, 1024, 64, 64))
    try:
        problems, res = run_both(reference, ctx, dist, mat, blend)
        assert not problems, "\n".join(problems[:10])
    finally:
        ctx.close()


def test_launch_limit_changes_no_output(gpu_context):
    """The same context with and without a limit (the captured run is rebuilt for each) gives the same bytes."""
    import golden_hash
    dist, mat, blend = grids.by_name("patchwork64")
    gpu_context.set_materials(None, None)
    gpu_context.upload_dense(dist, mat, blend)
    digests = []
    for limit in (0, 1, 0):
        gpu_context.set_launch_limit(limit)
        info = gpu_context.polygonize()
        res = gpu_context.download()
        digests.append(([golden_hash.level_digests(res.level(l)) for l in range(info.levels_total)], [int(v) for v in res.stats]))
    gpu_context.set_launch_limit(0)
    assert digests[0] == digests[1] == digests[2]


@pytest.mark.parametrize("limit", (0, 1, 2, 7))
def test_skip_quirk_against_reference_and_restatement(reference, restatement, limit):
    """Level-0 blocks skipped with their BF_Empty neighbourhood although the surface runs along their faces (:520): level 0
    and the statistics against the reference; every level against the CPU restatement, because the reference's coarse
    cells over the skipped blocks read an uninitialised material (:1052-1086) that both define as {EMPTY, 0}."""
    dist, mat, blend = gridgen.skip_quirk()
    ctx = _context(limit)
    try:
        problems = run_skipping_grid(reference, restatement, ctx, dist, mat, blend)
        assert not problems, "\n".join(problems[:10])
    finally:
        ctx.close()


def test_patchwork512_all_levels(reference, gpu_context):
    dist, mat, blend = grids.by_name("patchwork512")
    problems, res = run_both(reference, gpu_context, dist, mat, blend)
    assert not problems, "\n".join(problems[:10])


def test_patchwork1024_mode1_coarse_lattice(reference, gpu_context):
    """1024^3: level 2 has 4096 blocks, so it runs in vxb_block_kernel<1> on the coarse lattice; the aligned 64^3 noise
    region makes one of those blocks a big block."""
    dist, mat, blend = grids.by_name("patchwork1024")
    assert (gridgen.nontrivial_cells_per_block(dist, 2) > 1024).any(), "no level-2 big block: the generator drifted"
    problems, res = run_both(reference, gpu_context, dist, mat, blend, max_levels=4)
    assert not problems, "levels 0-3:\n" + "\n".join(problems[:10])
    assert res.info.levels_computed == 4 and res.info.trans_vertex_total > 0
    problems, res = run_both(reference, gpu_context, dist, mat, blend)
    assert not problems, "all levels:\n" + "\n".join(problems[:10])
