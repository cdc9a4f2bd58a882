"""The block walk of levels 0 and 1 (vxb_select_kernel) against counts taken on the host.

Level 0 takes a non-skipped block exactly when one of its cells is non-trivial: its own sign flags and the low-face
summaries of its +1 neighbours (planes, lines, corner; vxb_scan_kernel) cover the 17^3 samples its cells read.  So every
work item of vxb_block_kernel<0> emits a block (items == emitted), on hostile grids, at any launch limit, in incremental
runs after edits at the grid's edges and on every rank of a sharded run.  On the benchmark's terrain the count equals a
numpy count of the blocks with a non-trivial cell outside the 27-neighbour BF_Empty skip rule.  Level 1 keeps a superset
test: it takes at least every block with a sign mix or a child page."""
import numpy as np
import pytest

import gridgen
import grids

pytestmark = pytest.mark.gpu

PATH_GRIDS = sorted(name for name in list(grids.SMALL) + list(grids.MEDIUM)
                    if name.startswith(("hostile", "noise", "patchwork"))) + sorted(grids.RLE_EDGES)
LIMITS = (0, 2, 7)


def _level0_exact(ctx, what):
    items, emitted = ctx.run_work_items(0)
    assert items == emitted, "%s: level 0 took %d blocks, %d had a non-trivial cell" % (what, items, emitted)
    return items


def _skip_rule(dist):
    """[bz, by, bx] True where AreBlockAndNeighborsEmpty skips the level-0 block: all 27 (clamped) neighbours are BF_Empty
    = run-length coded (<= 2048 runs) with every voxel of one strict sign."""
    n = dist.shape[0]
    nb = n // 16
    blocks = dist.reshape(nb, 16, nb, 16, nb, 16).transpose(0, 2, 4, 1, 3, 5).reshape(nb, nb, nb, 4096)
    neg, pos, zero = (blocks < 0).any(-1), (blocks > 0).any(-1), (blocks == 0).any(-1)
    empty = (neg != pos) & ~zero
    changes = (blocks[..., 1:] != blocks[..., :-1]).sum(-1)
    for b in np.argwhere(empty & (changes + 17 >= 2049)):   # runs <= changes + 1 + 16 cuts at 255 bytes
        empty[tuple(b)] = gridgen.runs_of(blocks[tuple(b)]) <= 2048
    e = np.pad(empty, 1, mode="edge")
    skip = np.ones_like(empty)
    for dz in range(3):
        for dy in range(3):
            for dx in range(3):
                skip &= e[dz:dz + nb, dy:dy + nb, dx:dx + nb]
    return skip


def _assert_processed_cells(info, skip):
    """The 27-neighbour rule is untouched: the processed cells of the statistics (trivial + non-trivial) are 4096 per
    non-skipped level-0 block plus 4096 per block of every computed level above (modulo 2^32)."""
    nb = skip.shape[0]
    want = int((~skip).sum()) * 4096 + sum((nb >> l) ** 3 for l in range(1, info.levels_computed)) * 4096
    assert (int(info.stats[1]) + int(info.stats[2])) % (1 << 32) == want % (1 << 32)


@pytest.mark.parametrize("name", PATH_GRIDS + ["skip_quirk"])
def test_level0_items_are_emitted_blocks(name):
    import voxels_b200
    dist, mat, blend = gridgen.skip_quirk() if name == "skip_quirk" else grids.by_name(name)
    skip = _skip_rule(dist)
    ctx = voxels_b200.Context(0)
    try:
        ctx.set_materials(None, None)
        ctx.upload_dense(dist, mat, blend)
        counts = set()
        for limit in LIMITS:
            ctx.set_launch_limit(limit)
            info = ctx.polygonize()
            _assert_processed_cells(info, skip)
            counts.add(_level0_exact(ctx, "%s, launch limit %d" % (name, limit)))
        assert len(counts) == 1, counts
    finally:
        ctx.close()


def test_level0_items_after_edge_edits():
    """Incremental runs over dirty ranges clipped at the grid's faces, edges and corners (device-side sphere edits)."""
    import voxels_b200
    from voxels_b200 import capi
    n = 128
    dist, mat, blend = grids.by_name("patchwork128")
    ctx = voxels_b200.Context(0)
    try:
        ctx.set_materials(None, None)
        ctx.upload_dense(dist, mat, blend)
        ctx.set_launch_limit(2)
        ctx.polygonize()
        _level0_exact(ctx, "full run")
        for i, (pos, r, ext, add) in enumerate(gridgen.edge_edit_sequence(n, 18)):
            box = ctx.inject_surface(np.array(pos, np.float32), np.full(3, ext, np.float32), capi.Surface.sphere((0, 0, 0), r), 0 if add else 2)
            ctx.polygonize_region(box[:3], box[3:])
            _level0_exact(ctx, "edit %d" % i)
    finally:
        ctx.close()


@pytest.mark.parametrize("world", (2, 4))
def test_level0_items_on_virtual_ranks(gpu_context, world):
    import voxels_b200
    from test_gpu_sharded import configure_virtual_ranks, run_virtual_ranks
    dist, mat, blend = grids.by_name("patchwork128")
    gpu_context.set_materials(None, None)
    gpu_context.upload_dense(dist, mat, blend)
    gpu_context.polygonize()
    single = _level0_exact(gpu_context, "single run")
    d, m, b = gpu_context.device_pointers()
    contexts = [voxels_b200.Context(0) for _ in range(world)]
    try:
        for c in contexts:
            c.set_device_grid(128, d, m, b)
        run_virtual_ranks(contexts, configure_virtual_ranks(contexts))
        per_rank = [_level0_exact(c, "rank %d of %d" % (r, world)) for r, c in enumerate(contexts)]
        assert sum(per_rank) == single, (per_rank, single)
    finally:
        for c in contexts:
            c.close()


@pytest.mark.parametrize("n", (256, 512))
def test_terrain_counts(gpu_context, n):
    import torch
    from voxels_b200 import synth
    dist_t, mat_t, blend_t = synth.terrain(n, torch.device("cuda", 0))
    torch.cuda.synchronize()
    gpu_context.set_materials(None, None)
    gpu_context.set_device_grid(n, dist_t.data_ptr(), mat_t.data_ptr(), blend_t.data_ptr(), keep=(dist_t, mat_t, blend_t))
    info = gpu_context.polygonize()
    dist = dist_t.cpu().numpy()

    skip = _skip_rule(dist)
    _assert_processed_cells(info, skip)
    nt0 = gridgen.nontrivial_cells_per_block(dist, 0)
    emit0 = (nt0 > 0) & ~skip
    items0 = _level0_exact(gpu_context, "terrain %d" % n)
    assert items0 == int(emit0.sum())

    nt1 = gridgen.nontrivial_cells_per_block(dist, 1)
    h = emit0.shape[0] // 2
    child = emit0.reshape(h, 2, h, 2, h, 2).any(axis=(1, 3, 5))
    items1, emitted1 = gpu_context.run_work_items(1)
    assert emitted1 == int((nt1 > 0).sum())
    assert items1 >= int(((nt1 > 0) | child).sum()), (items1, int(((nt1 > 0) | child).sum()))
