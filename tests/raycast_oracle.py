"""numpy oracle of vxb_mesh_raycast (include/vxb200.h "ray queries"): the float32 Moeller-Trumbore test in the header's order
(explicit np.float32 throughout, so nothing is promoted to float64), the global minimum by the tie rule (least t, then lower
slot, then lower triangle) over every level-0 triangle of a downloaded mesh (capi.Result).

A float64 slab test per block, with the block's box grown by one voxel, skips blocks the segment does not come near: a
triangle lies in the closed box of its block, and an accepted hit lies within rounding of its triangle, so the skipped
blocks hold no hit."""
import numpy as np

from voxels_b200 import capi

F = np.float32


class Level0:
    """The level-0 triangles of a mesh, grouped by directory slot: positions, normals and boxes (OUTPUT, Y-up coordinates)."""

    def __init__(self, res):
        n = res.n
        nb = n // 16
        recs = res.records
        self.slots = np.nonzero(recs["level"] == 0)[0].astype(np.int64)
        rec0 = recs[self.slots]
        cid = rec0["coord_id"].astype(np.int64)
        bx, by, bz = cid % nb, (cid // nb) % nb, cid // (nb * nb)
        self.lo = np.stack([bx, bz, by], axis=1).astype(np.float64) * 16.0   # output axes (x, z, y) of the grid block
        self.hi = self.lo + 16.0
        self.ids = rec0["id"].astype(np.uint32)
        self.tri_pos, self.tri_nrm = [], []
        pos = res.verts["pos"].astype(np.float32)
        nrm = res.verts["nrm"].astype(np.float32)
        for r in rec0:
            ic, io, vo = int(r["index_count"]), int(r["index_offset"]), int(r["vertex_offset"])
            tri = res.idx[io:io + ic].astype(np.int64).reshape(-1, 3) + vo
            self.tri_pos.append(pos[tri])     # [T, 3 vertices, 3]
            self.tri_nrm.append(nrm[tri])


def valid_ray(ray):
    o, d = ray["origin"], ray["direction"]
    return bool(np.all(np.isfinite(o)) and np.all(np.isfinite(d)) and np.any(d != 0) and np.isfinite(ray["t_min"])
                and not np.isnan(ray["t_max"]) and ray["t_min"] <= ray["t_max"])


def _near_blocks(lv, o, d, t_min, t_max, grow=1.0):
    """Indices (into lv.slots) of the blocks whose box grown by `grow` meets the segment, float64."""
    o64, d64 = o.astype(np.float64), d.astype(np.float64)
    te = np.full(len(lv.slots), float(t_min)); tx = np.full(len(lv.slots), float(t_max))
    for a in range(3):
        lo, hi = lv.lo[:, a] - grow, lv.hi[:, a] + grow
        if d64[a] == 0.0:
            outside = (o64[a] < lo) | (o64[a] > hi)
            te[outside] = np.inf
            continue
        ta, tb = (lo - o64[a]) / d64[a], (hi - o64[a]) / d64[a]
        te = np.maximum(te, np.minimum(ta, tb)); tx = np.minimum(tx, np.maximum(ta, tb))
    return np.nonzero(te <= tx)[0]


def moller_trumbore(o, d, t_min, t_max, p):
    """The header's test on triangles p [T, 3, 3] (float32): (hit mask, t, u, v)."""
    dx, dy, dz = F(d[0]), F(d[1]), F(d[2])
    p0x, p0y, p0z = p[:, 0, 0], p[:, 0, 1], p[:, 0, 2]
    e1x, e1y, e1z = p[:, 1, 0] - p0x, p[:, 1, 1] - p0y, p[:, 1, 2] - p0z
    e2x, e2y, e2z = p[:, 2, 0] - p0x, p[:, 2, 1] - p0y, p[:, 2, 2] - p0z
    sx, sy, sz = F(o[0]) - p0x, F(o[1]) - p0y, F(o[2]) - p0z
    pvx = dy * e2z - dz * e2y; pvy = dz * e2x - dx * e2z; pvz = dx * e2y - dy * e2x
    det = (e1x * pvx + e1y * pvy) + e1z * pvz
    inv = F(1) / det
    u = ((sx * pvx + sy * pvy) + sz * pvz) * inv
    qvx = sy * e1z - sz * e1y; qvy = sz * e1x - sx * e1z; qvz = sx * e1y - sy * e1x
    v = ((dx * qvx + dy * qvy) + dz * qvz) * inv
    t = ((e2x * qvx + e2y * qvy) + e2z * qvz) * inv
    hit = (det != 0) & (u >= 0) & (u <= 1) & (v >= 0) & (u + v <= 1) & (t >= F(t_min)) & (t <= F(t_max))
    return hit, t, u, v


def raycast(res, rays, level0=None, counts=None):
    """RAY_HIT_DTYPE hits of `rays` (RAY_DTYPE) against the level-0 triangles of `res`.  Invalid rays are misses (the device
    variant's rule).  `counts`, when a list, receives (blocks tested, triangles tested) per ray."""
    lv = Level0(res) if level0 is None else level0
    hits = np.zeros(len(rays), capi.RAY_HIT_DTYPE)
    hits["t"] = np.inf
    hits["slot"] = capi.VXB_RAY_MISS
    with np.errstate(all="ignore"):
        for r, ray in enumerate(rays):
            if not valid_ray(ray):
                if counts is not None:
                    counts.append((0, 0))
                continue
            o, d = ray["origin"].astype(np.float32), ray["direction"].astype(np.float32)
            t_min, t_max = F(ray["t_min"]), F(ray["t_max"])
            near = _near_blocks(lv, o, d, t_min, t_max)
            best = None
            tested = 0
            for b in near:
                p = lv.tri_pos[b]
                tested += len(p)
                if not len(p):
                    continue
                hit, t, u, v = moller_trumbore(o, d, t_min, t_max, p)
                ks = np.nonzero(hit)[0]
                if not len(ks):
                    continue
                k = ks[np.lexsort((ks, t[ks]))[0]]           # least t, then lower triangle
                cand = (t[k], int(lv.slots[b]), int(k), u[k], v[k], b)
                if best is None or (cand[0], cand[1], cand[2]) < (best[0], best[1], best[2]):
                    best = cand
            if counts is not None:
                counts.append((len(near), tested))
            if best is None:
                continue
            t, slot, k, u, v, b = best
            h = hits[r]
            h["t"], h["u"], h["v"], h["slot"], h["block_id"], h["triangle"] = t, u, v, slot, lv.ids[b], k
            h["position"] = o + t * d
            n0, n1, n2 = lv.tri_nrm[b][k]
            w = (F(1) - u) - v
            nv = (w * n0 + u * n1) + v * n2
            length = np.sqrt((nv[0] * nv[0] + nv[1] * nv[1]) + nv[2] * nv[2])
            h["normal"] = nv / length if length > 0 else np.zeros(3, np.float32)
    return hits


def result_from_blocks(n, blocks):
    """A capi.Result holding only level-0 blocks, for hand-built meshes: blocks = [(grid block coordinate (x, y, z), positions
    [V, 3], normals [V, 3], indices [I])] in directory order (slot = list position)."""
    nb = n // 16
    records = np.zeros(len(blocks), capi.RECORD_DTYPE)
    verts, idx = [], []
    vo = io = 0
    for s, ((x, y, z), pos, nrm, ind) in enumerate(blocks):
        rec = records[s]
        rec["level"], rec["coord_id"], rec["id"] = 0, (z * nb + y) * nb + x, 1000 + s
        rec["vertex_count"], rec["index_count"], rec["vertex_offset"], rec["index_offset"] = len(pos), len(ind), vo, io
        v = np.zeros(len(pos), capi.VERTEX_DTYPE)
        v["pos"], v["nrm"] = pos, nrm
        verts.append(v); idx.append(np.asarray(ind, np.uint32))
        vo += len(pos); io += len(ind)
    res = capi.Result.__new__(capi.Result)
    res.n, res.info, res.records = n, None, records
    res.verts = np.concatenate(verts) if verts else np.zeros(0, capi.VERTEX_DTYPE)
    res.idx = np.concatenate(idx) if idx else np.zeros(0, np.uint32)
    res.tverts, res.tidx = np.zeros(0, capi.VERTEX_DTYPE), np.zeros(0, np.uint32)
    return res


def same_hits(got, want):
    """Every field of every hit bit-identical: the indices of the rays that differ."""
    a, b = got.view(np.uint32).reshape(len(got), -1), want.view(np.uint32).reshape(len(want), -1)
    return np.nonzero((a != b).any(axis=1))[0]
