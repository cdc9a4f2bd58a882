"""Crops as an oracle for grids too large to run through the reference whole.

A block's output depends only on the voxels of its box grown by one block of its own level on every side; where that
grown box reaches past the grid, what lies beyond is the grid's edge.  So a cube crop [origin, origin + w)^3 of an n^3
grid, run through the unmodified reference, gives the exact output of every block of the crop whose grown box lies inside
the crop, or, on a side where it leaves the grid, whose crop side is that same grid edge.  Such a block's counts, indices,
texture bytes, flag bits and transition meshes are the big grid's; its positions and the xyz of its secondary positions
are the big grid's minus the origin, in output axes (x, z, y).  Positions are dyadic with few fraction bits, so adding
the origin in float64 is exact."""
import numpy as np

from compare import NORMAL_TOL


def _exclusive(counts):
    c = np.asarray(counts, np.int64).ravel()
    return np.concatenate([[0], np.cumsum(c)[:-1]]) if len(c) else c


def _gather(offsets, counts):
    """The element indices of the ranges [offsets[i], offsets[i] + counts[i]) concatenated in order."""
    o = np.asarray(offsets, np.int64).ravel(); c = np.asarray(counts, np.int64).ravel()
    total = int(c.sum())
    return np.repeat(o - _exclusive(c), c) + np.arange(total, dtype=np.int64)


def level_base(n, level):
    """Block ids of a full run start at the number of blocks of all lower levels (GenerateBlockListForLevel)."""
    return sum(((n // 16) >> l) ** 3 for l in range(level))


class Blocks:
    """One level of a run: per block its coordinate id ((z * nb + y) * nb + x, ascending), id, and the counts and offsets
    of its regular and transition (6 faces) vertices and indices into the level's arrays."""

    def __init__(self, n, level, coord, ids, counts, offsets, verts, idx, tverts, tidx):
        self.n, self.level, self.coord, self.ids = n, level, np.asarray(coord, np.int64), np.asarray(ids, np.int64)
        self.counts, self.offsets = counts, offsets   # dicts: "v", "i" -> [blocks]; "tv", "ti" -> [blocks, 6]
        self.verts, self.idx, self.tverts, self.tidx = verts, idx, tverts, tidx
        assert np.all(np.diff(self.coord) > 0), "blocks are not in (z, y, x) order"

    @classmethod
    def from_dump(cls, dump, n, level):
        """A harness.LevelDump of the reference (rows in block order, arrays concatenated block by block, face by face)."""
        r = dump.rows
        m = 16 << level
        nb = n // m
        b = (r["min"] / m).astype(np.int64)           # output axes (x, z, y)
        coord = (b[:, 1] * nb + b[:, 2]) * nb + b[:, 0]
        counts = {"v": r["nv"].astype(np.int64), "i": r["ni"].astype(np.int64), "tv": r["tnv"].astype(np.int64),
                  "ti": r["tni"].astype(np.int64)}
        offsets = {k: _exclusive(c).reshape(c.shape) for k, c in counts.items()}
        return cls(n, level, coord, r["id"], counts, offsets, dump.verts, dump.idx, dump.tverts, dump.tidx)

    @classmethod
    def from_result(cls, res, level):
        """A voxels_b200 Result (directory records with offsets into the downloaded arenas)."""
        rec = res.records[res.records["level"] == level]
        counts = {"v": rec["vertex_count"].astype(np.int64), "i": rec["index_count"].astype(np.int64),
                  "tv": rec["trans_vertex_count"].astype(np.int64), "ti": rec["trans_index_count"].astype(np.int64)}
        offsets = {"v": rec["vertex_offset"].astype(np.int64), "i": rec["index_offset"].astype(np.int64),
                   "tv": rec["trans_vertex_offset"].astype(np.int64), "ti": rec["trans_index_offset"].astype(np.int64)}
        return cls(res.n, level, rec["coord_id"], rec["id"], counts, offsets, res.verts, res.idx, res.tverts, res.tidx)

    def subset(self, keep):
        """The blocks where `keep` is true (the level's arrays are shared)."""
        return Blocks(self.n, self.level, self.coord[keep], self.ids[keep], {k: c[keep] for k, c in self.counts.items()},
                      {k: o[keep] for k, o in self.offsets.items()}, self.verts, self.idx, self.tverts, self.tidx)

    def find(self, coord):
        """Index of each coordinate id, -1 where this level has no such block."""
        coord = np.asarray(coord, np.int64)
        if not len(self.coord):
            return np.full(len(coord), -1, np.int64)
        at = np.minimum(np.searchsorted(self.coord, coord), len(self.coord) - 1)
        return np.where(self.coord[at] == coord, at, -1)


def selected(origin, w, n, level, margin=True):
    """Crop-local block coordinates (bx, by, bz) of the level-`level` blocks of the crop whose output it determines.
    margin=False selects every block of the crop instead (the rule without its margin, for negative controls)."""
    m = 16 << level
    if w < m or any(int(o) % m for o in origin):
        return tuple(np.zeros(0, np.int64) for _ in range(3))
    c = np.arange(0, w, m, dtype=np.int64)
    ok = []
    for o in origin:
        g = int(o) + c
        ok.append(np.ones(len(c), bool) if not margin else
                  ((g == 0) | (g - m >= int(o))) & ((g + m == n) | (g + 2 * m <= int(o) + w)))
    bz, by, bx = np.meshgrid(c[ok[2]] // m, c[ok[1]] // m, c[ok[0]] // m, indexing="ij")
    return bx.ravel(), by.ravel(), bz.ravel()


def _verts_diff(a, b, shift, what):
    """Vertices of the crop (a) against the big grid's (b): positions and secondary xyz as a + shift == b in float64."""
    msgs = []
    for field, cols in (("pos", 3), ("sec", 3)):
        ne = (a[field][:, :cols].astype(np.float64) + shift) != b[field][:, :cols].astype(np.float64)
        if ne.any():
            k = int(np.nonzero(ne.any(axis=1))[0][0])
            msgs.append((k, "%s: %s differs at %d vertices, first %s + %s vs %s" % (
                what, field, int(ne.any(axis=1).sum()), a[field][k], shift, b[field][k])))
    ne = a["sec"][:, 3].view(np.uint32) != b["sec"][:, 3].view(np.uint32)
    if ne.any():
        k = int(np.nonzero(ne)[0][0])
        msgs.append((k, "%s: sec.w flag bits differ at %d vertices, first %s vs %s" % (what, int(ne.sum()), a["sec"][k], b["sec"][k])))
    ne = (a["tex"] != b["tex"]).any(axis=1)
    if ne.any():
        k = int(np.nonzero(ne)[0][0])
        msgs.append((k, "%s: texture bytes differ at %d vertices, first %s vs %s" % (what, int(ne.sum()), a["tex"][k], b["tex"][k])))
    dn = np.abs(a["nrm"].astype(np.float64) - b["nrm"].astype(np.float64)).max(axis=1) if len(a) else np.zeros(0)
    if (dn > NORMAL_TOL).any():
        k = int(np.nonzero(dn > NORMAL_TOL)[0][0])
        msgs.append((k, "%s: normals differ (max %g) at %d vertices, first %s vs %s" % (
            what, dn.max(), int((dn > NORMAL_TOL).sum()), a["nrm"][k], b["nrm"][k])))
    return msgs


def compare_level(crop, big, origin, w, margin=True, big_ids=True):
    """Every selected block of one level: the crop's run (`crop`, Blocks of the w^3 crop) against the big run (`big`,
    Blocks of the same level).  A block present on one side only is a mismatch.  big_ids=False leaves the big run's ids
    unchecked (an incremental run numbers its re-created blocks on from the previous run).  Returns (blocks compared,
    problems)."""
    level, n = big.level, big.n
    m = 16 << level
    bx, by, bz = selected(origin, w, n, level, margin)
    wb, nb = w // m, n // m
    ox, oy, oz = (int(o) // m for o in origin)
    c_coord = (bz * wb + by) * wb + bx
    b_coord = ((bz + oz) * nb + (by + oy)) * nb + (bx + ox)
    ci, bi = crop.find(c_coord), big.find(b_coord)
    what = "L%d origin %s" % (level, tuple(int(o) for o in origin))
    problems = []
    one = (ci < 0) != (bi < 0)
    if one.any():
        k = int(np.nonzero(one)[0][0])
        problems.append("%s: %d blocks on one side only, first crop-local block (x, y, z) %s: %s" % (
            what, int(one.sum()), (int(bx[k]), int(by[k]), int(bz[k])), "crop only" if ci[k] >= 0 else "big run only"))
    both = (ci >= 0) & (bi >= 0)
    ci, bi, c_coord, b_coord = ci[both], bi[both], c_coord[both], b_coord[both]
    if not np.array_equal(crop.ids[ci], level_base(w, level) + c_coord):
        problems.append("%s: crop block ids are not base + coordinate" % what)
    if big_ids and not np.array_equal(big.ids[bi], level_base(n, level) + b_coord):
        problems.append("%s: big-run block ids are not base + coordinate" % what)
    same = np.ones(len(ci), bool)
    for k in ("v", "i", "tv", "ti"):
        ne = crop.counts[k][ci] != big.counts[k][bi]
        ne = ne if ne.ndim == 1 else ne.any(axis=1)
        if ne.any():
            j = int(np.nonzero(ne)[0][0])
            problems.append("%s: %s counts differ in %d blocks, first big coordinate id %d: %s vs %s" % (
                what, k, int(ne.sum()), b_coord[j], crop.counts[k][ci[j]], big.counts[k][bi[j]]))
        same &= ~ne
    ci, bi, b_coord = ci[same], bi[same], b_coord[same]
    shift = np.array([int(origin[0]), int(origin[2]), int(origin[1])], np.float64)   # output axes (x, z, y)
    for kind, vk, ik, va, vb, ia, ib in (("regular", "v", "i", crop.verts, big.verts, crop.idx, big.idx),
                                        ("transition", "tv", "ti", crop.tverts, big.tverts, crop.tidx, big.tidx)):
        cnt_v = crop.counts[vk][ci]
        ga = _gather(crop.offsets[vk][ci], cnt_v); gb = _gather(big.offsets[vk][bi], big.counts[vk][bi])
        per_block_v = cnt_v if cnt_v.ndim == 1 else cnt_v.sum(axis=1)
        for k, msg in _verts_diff(va[ga], vb[gb], shift, "%s %s" % (what, kind)):
            blk = int(np.searchsorted(np.cumsum(per_block_v), k, side="right"))
            problems.append("%s (big coordinate id %d)" % (msg, b_coord[blk]))
        cnt_i = crop.counts[ik][ci]
        xa = ia[_gather(crop.offsets[ik][ci], cnt_i)]; xb = ib[_gather(big.offsets[ik][bi], big.counts[ik][bi])]
        if not np.array_equal(xa, xb):
            k = int(np.nonzero(xa != xb)[0][0])
            blk = int(np.searchsorted(np.cumsum(cnt_i if cnt_i.ndim == 1 else cnt_i.sum(axis=1)), k, side="right"))
            problems.append("%s %s: indices differ at %d positions, first in big coordinate id %d" % (
                what, kind, int((xa != xb).sum()), b_coord[blk]))
    return int(both.sum()), problems


def compare_crop(crop_level, big_level, origin, w, levels, margin=True):
    """compare_level for levels 0 .. levels - 1; crop_level(l) / big_level(l) give the Blocks of level l.
    Returns ({level: blocks compared}, problems)."""
    counts, problems = {}, []
    for l in range(levels):
        if (16 << l) > w:
            break
        k, p = compare_level(crop_level(l), big_level(l), origin, w, margin)
        counts[l] = k
        problems += p
    return counts, problems


def reference_levels(reference, grid, w):
    """The reference's full run of a w^3 crop grid as Blocks per level (the grid handle stays the caller's)."""
    s, _ = reference.polygonize(grid)
    try:
        return [Blocks.from_dump(reference.surface_level(s, l), w, l) for l in range(reference.surface_levels(s))]
    finally:
        reference.surface_destroy(s)
