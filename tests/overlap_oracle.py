"""numpy oracle of vxb_mesh_overlap_box (include/vxb200.h "box overlap gathers"): the float32 separating-axis test in the
header's order (explicit np.float32 throughout, so nothing is promoted to float64), over every level-0 triangle of a
downloaded mesh (capi.Result), in the header's result order (ascending coord_id of the block, then ascending triangle).

A block whose closed lattice box misses the query box is skipped: an accepted triangle passes the exact box-axis test, so its
vertices, which lie in their block's lattice box, put that box in contact with the query box.  The skip is exact (float64
holds the multiples of 16 and every float32 box exactly).

clip64 is an independent float64 reference with no formula in common with the test: the triangle is clipped by the six
planes of the closed box (Sutherland-Hodgman) and overlaps iff something is left."""
import numpy as np

from voxels_b200 import capi
import raycast_oracle

F = np.float32


class Level0Sorted:
    """The level-0 triangles of a mesh flattened in the result order: tri [T, 3, 3] positions, slot, block id and index k per
    triangle, and per block (in coord_id order) its lattice box and its range of triangles."""

    def __init__(self, res):
        lv = raycast_oracle.Level0(res)
        nb = res.n // 16
        cid = res.records["coord_id"][lv.slots].astype(np.int64)
        order = np.argsort(cid, kind="stable")
        self.lo, self.hi = lv.lo[order], lv.hi[order]
        counts = np.array([len(lv.tri_pos[b]) for b in order], np.int64)
        self.start = np.concatenate([[0], np.cumsum(counts)])
        tris = [lv.tri_pos[b] for b in order]
        self.tri = np.concatenate(tris).astype(np.float32) if tris and counts.sum() else np.zeros((0, 3, 3), np.float32)
        self.slot = np.repeat(lv.slots[order].astype(np.uint32), counts)
        self.block_id = np.repeat(lv.ids[order], counts)
        self.k = np.concatenate([np.arange(c, dtype=np.uint32) for c in counts]) if len(counts) else np.zeros(0, np.uint32)
        self.nb = nb


def valid_box(box):
    lo, hi = np.asarray(box["min"]), np.asarray(box["max"])
    return bool(np.all(np.isfinite(lo)) and np.all(np.isfinite(hi)) and np.all(lo <= hi))


def _separates(ax, ay, az, v, hx, hy, hz):
    """Axis (ax, ay, az) [T] against vertices v [T, 3, 3] (box frame): separated mask."""
    s = [(ax * v[:, k, 0] + ay * v[:, k, 1]) + az * v[:, k, 2] for k in range(3)]
    r = (hx * np.abs(ax) + hy * np.abs(ay)) + hz * np.abs(az)
    return ((s[0] > r) & (s[1] > r) & (s[2] > r)) | ((s[0] < -r) & (s[1] < -r) & (s[2] < -r))


def sat(box, p, counts=None):
    """The header's test of triangles p [T, 3, 3] (float32) against one box: overlap mask.  `counts`, a dict, receives how
    many triangles each stage excluded ("box", "normal", "edge")."""
    p = np.asarray(p, np.float32)
    lo, hi = np.asarray(box["min"], np.float32), np.asarray(box["max"], np.float32)
    keep = np.ones(len(p), bool)
    for i in range(3):                                            # 1: box axes, exact
        keep &= (p[:, :, i].min(axis=1) <= hi[i]) & (p[:, :, i].max(axis=1) >= lo[i])
    if counts is not None:
        counts["box"] = counts.get("box", 0) + int((~keep).sum())
    idx = np.nonzero(keep)[0]
    if not len(idx):
        return keep
    q = p[idx]
    with np.errstate(all="ignore"):
        c = (lo + hi) * F(0.5)                                    # 2: box frame
        h = hi * F(0.5) - lo * F(0.5)
        v = q - c
        e = [v[:, 1] - v[:, 0], v[:, 2] - v[:, 1], v[:, 0] - v[:, 2]]
        hx, hy, hz = h[0], h[1], h[2]
        n = (e[0][:, 1] * e[1][:, 2] - e[0][:, 2] * e[1][:, 1], e[0][:, 2] * e[1][:, 0] - e[0][:, 0] * e[1][:, 2],
             e[0][:, 0] * e[1][:, 1] - e[0][:, 1] * e[1][:, 0])
        sep = _separates(n[0], n[1], n[2], v, hx, hy, hz)        # 3: the normal, then u_i x e_j
        by_normal = sep.copy()
        zero = np.zeros(len(q), np.float32)
        for i in range(3):
            for j in range(3):
                ex, ey, ez = e[j][:, 0], e[j][:, 1], e[j][:, 2]
                a = [(zero, -ez, ey), (ez, zero, -ex), (-ey, ex, zero)][i]
                sep |= _separates(a[0], a[1], a[2], v, hx, hy, hz)
    if counts is not None:
        counts["normal"] = counts.get("normal", 0) + int(by_normal.sum())
        counts["edge"] = counts.get("edge", 0) + int((sep & ~by_normal).sum())
    keep[idx[sep]] = False
    return keep


def overlap_boxes(res, boxes, level0=None, counts=None):
    """(offsets [count + 1] uint64, OVERLAP_TRIANGLE_DTYPE array) of `boxes` (BOX_DTYPE) against the level-0 triangles of `res`.
    Invalid boxes have 0 triangles (the device variant's rule).  `counts`, when a list, receives (blocks tested, triangles
    tested) per box: the blocks whose lattice box meets the box, and their triangles."""
    lv = Level0Sorted(res) if level0 is None else level0
    per_box, offsets = [], np.zeros(len(boxes) + 1, np.uint64)
    for q, box in enumerate(boxes):
        take = np.zeros(0, np.int64)
        blocks = 0
        if valid_box(box):
            lo, hi = box["min"].astype(np.float64), box["max"].astype(np.float64)
            near = np.nonzero(np.all((lv.lo <= hi) & (lv.hi >= lo), axis=1))[0]
            blocks = len(near)
            if len(near):
                cand = np.concatenate([np.arange(lv.start[b], lv.start[b + 1]) for b in near])
                take = cand[sat(box, lv.tri[cand])] if len(cand) else cand
                if counts is not None:
                    counts.append((blocks, len(cand)))
            elif counts is not None:
                counts.append((0, 0))
        elif counts is not None:
            counts.append((0, 0))
        per_box.append(take)
        offsets[q + 1] = offsets[q] + len(take)
    idx = np.concatenate(per_box) if per_box else np.zeros(0, np.int64)
    tris = np.zeros(len(idx), capi.OVERLAP_TRIANGLE_DTYPE)
    tris["p"], tris["slot"], tris["block_id"], tris["triangle"] = lv.tri[idx], lv.slot[idx], lv.block_id[idx], lv.k[idx]
    return offsets, tris


def _clip(poly, axis, bound, keep_ge):
    out = []
    m = len(poly)
    for a in range(m):
        p, q = poly[a], poly[(a + 1) % m]
        pin = p[axis] >= bound if keep_ge else p[axis] <= bound
        qin = q[axis] >= bound if keep_ge else q[axis] <= bound
        if pin:
            out.append(p)
        if pin != qin:
            t = (bound - p[axis]) / (q[axis] - p[axis])
            x = p + t * (q - p)
            x[axis] = bound
            out.append(x)
    return out


def clip64(lo, hi, tri):
    """float64 Sutherland-Hodgman: does the triangle tri [3, 3] keep any point inside the closed box [lo, hi]?"""
    poly = [np.asarray(v, np.float64) for v in tri]
    for axis in range(3):
        poly = _clip(poly, axis, float(lo[axis]), True)
        if not poly:
            return False
        poly = _clip(poly, axis, float(hi[axis]), False)
        if not poly:
            return False
    return True


def same(got, want):
    """(offsets, tris) pairs bit-identical: a description of the first difference, or None."""
    (go, gt), (wo, wt) = got, want
    if not np.array_equal(go, wo):
        q = int(np.nonzero(go != wo)[0][0])
        return "offsets differ first at %d: got %d, want %d" % (q, int(go[q]), int(wo[q]))
    if len(gt) != len(wt):
        return "%d records, want %d" % (len(gt), len(wt))
    a, b = gt.view(np.uint32).reshape(len(gt), 12), wt.view(np.uint32).reshape(len(wt), 12)
    bad = np.nonzero((a != b).any(axis=1))[0]
    if len(bad):
        k = int(bad[0])
        return "%d of %d records differ; first %d: got %s, want %s" % (len(bad), len(gt), k, gt[k], wt[k])
    return None
