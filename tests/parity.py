"""The GPU-vs-reference comparison shared by the GPU parity tests."""
import numpy as np

import compare


def run_both(reference, ctx, dist, mat, blend, table=None, valid=None, max_levels=0, flags=0):
    g = reference.grid_from_dense(dist, mat, blend)
    s, _ = reference.polygonize(g, material_table=table, valid_mask=valid)
    ctx.set_materials(table, valid)
    ctx.upload_dense(dist, mat, blend)
    info = ctx.polygonize(max_levels, flags)
    res = ctx.download()
    problems = []
    levels = reference.surface_levels(s)
    assert info.levels_total == levels
    ncmp = levels if max_levels == 0 else min(levels, max_levels)
    for l in range(ncmp):
        problems += compare.level_diff(reference.surface_level(s, l), res.level(l), "L%d" % l)
    if max_levels == 0:
        rs = reference.surface_stats(s)
        if not np.array_equal(rs, res.stats):
            problems.append("stats differ: ref %s gpu %s" % (rs, res.stats))
    reference.surface_destroy(s)
    reference.grid_destroy(g)
    return problems, res


def run_skipping_grid(reference, restatement, ctx, dist, mat, blend):
    """A grid whose level-0 skip (TransVoxelImpl.cpp:520) drops blocks with a surface on their faces: level 0 and the
    statistics against the reference, every level against the CPU restatement, because the reference's coarse cells over
    the skipped blocks read an uninitialised material (:1052-1086) that both define as {EMPTY, 0}."""
    problems, _ = run_both(reference, ctx, dist, mat, blend, max_levels=1)
    if problems:
        return problems
    ctx.polygonize()
    res = ctx.download()
    h = restatement.run(dist, mat, blend)
    try:
        for l in range(restatement.levels(h)):
            problems += compare.level_diff(restatement.level(h, l), res.level(l), "L%d" % l)
        if not np.array_equal(restatement.stats(h), res.stats):
            problems.append("stats differ: restatement %s gpu %s" % (restatement.stats(h), res.stats))
    finally:
        restatement.destroy(h)
    return problems
