"""Numpy oracle of vxb_mesh_select_cut (include/vxb200.h "the LOD cut"): the box rule over arrays, in float32 and in the
header's order (numpy does not fuse), and the draw sets it implies.  The culling and the draw sets are tests/cull_oracle.py's.

  refines         refine(l, b) for an array of grid block coordinates of one level
  cut             (on the cut, block_adj) per record of a directory
  expected_draws  per view the set of regular and of transition draws (cull_oracle.draws_of over box_passes)
  full_octree     records of every (level, coord) slot of an n^3 grid, for statements about the whole octree
  level_map       the level of the cut node above every level-0 block of the grid (-1 where none is: a gap)
"""
import numpy as np

from cull_oracle import FACES, box_passes, draw_sets, draws_of  # noqa: F401  (draw_sets is re-exported for the tests)

F = np.float32


def refines(level, b, camera, lod_factor):
    """refine(level, b) for b: (count, 3) grid block coordinates (x, y, z) of one level."""
    b = np.asarray(b, np.int64).reshape(-1, 3)
    if level == 0:
        return np.zeros(len(b), bool)
    cam = np.asarray(camera, F)
    s = F(16 << level)
    lo = b[:, [0, 2, 1]].astype(F) * s                          # output axes (x, z, y); exact
    hi = lo + s
    with np.errstate(over="ignore", invalid="ignore"):
        e = np.maximum(np.maximum(lo - cam, cam - hi), F(0))
        dist2 = (e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1]) + e[:, 2] * e[:, 2]
        lim = F(lod_factor) * s
        return dist2 < lim * lim


def _coords(records, n, level, at):
    nb = (n // 16) >> level
    cid = records["coord_id"][at].astype(np.int64)
    return np.stack([cid % nb, (cid // nb) % nb, cid // (nb * nb)], axis=1), nb


def cut(records, n, levels, camera, lod_factor):
    """(on the cut, block_adj) per record: vxb_mesh_select_cut's rule; block_adj is 0 off the cut."""
    top = levels - 1
    selected = np.zeros(len(records), bool)
    adj = np.zeros(len(records), np.uint32)
    for level in range(levels):
        at = np.nonzero(records["level"] == level)[0]
        if not len(at):
            continue
        b, nb = _coords(records, n, level, at)
        sel = ~refines(level, b, camera, lod_factor)
        if level < top:
            sel &= refines(level + 1, b >> 1, camera, lod_factor)
        a = np.zeros(len(at), np.uint32)
        if level > 0:
            for f, d in enumerate(FACES):
                nbr = b + d
                inside = ((nbr >= 0) & (nbr < nb)).all(axis=1)
                a |= (inside & refines(level, nbr, camera, lod_factor)).astype(np.uint32) << np.uint32(f)
        selected[at] = sel
        adj[at] = np.where(sel, a, 0)
    return selected, adj


def expected_draws(records, boxes, n, levels, camera, lod_factor, views):
    """Per view the (regular, transition) sets: the cut of (camera, lod_factor), culled by box_passes."""
    selected, adj = cut(records, n, levels, camera, lod_factor)
    return [draws_of(records, selected & box_passes(boxes, v), adj) for v in np.asarray(views, F).reshape(-1, 6, 4)]


def full_octree(n, levels):
    """Records (level, coord_id) of every slot of an n^3 grid of `levels` levels, level by level."""
    from voxels_b200 import capi
    parts = []
    for level in range(levels):
        nb = (n // 16) >> level
        part = np.zeros(nb ** 3, capi.RECORD_DTYPE)
        part["level"], part["coord_id"] = level, np.arange(nb ** 3)
        parts.append(part)
    return np.concatenate(parts)


def level_map(n, levels, selected_at):
    """(nb0, nb0, nb0) int array indexed [x, y, z] (grid block coordinates of level 0): the level of the cut node above each
    level-0 block, -1 where no node is and -2 where two are.  selected_at(level) -> bool array over that level's coord_ids."""
    nb0 = n // 16
    out = np.full((nb0, nb0, nb0), -1, np.int64)
    for level in range(levels):
        nb = nb0 >> level
        sel = np.asarray(selected_at(level), bool).reshape(nb, nb, nb).transpose(2, 1, 0)     # coord_id = x + nb (y + nb z)
        cover = np.repeat(np.repeat(np.repeat(sel, 1 << level, 0), 1 << level, 1), 1 << level, 2)
        out = np.where(cover, np.where(out == -1, level, -2), out)
    return out
