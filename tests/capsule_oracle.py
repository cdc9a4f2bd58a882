"""numpy oracle of vxb_mesh_capsule_cast and vxb_mesh_closest_to_segment (include/vxb200.h "capsule queries"): the header's
float32 formulas in its order (explicit np.float32 throughout), the global minimum by the tie rule over every level-0
triangle of a downloaded mesh (capi.Result).  It reuses tests/collide_oracle.py's closest point, edge and vertex tests,
_gather and _least, and has no per-triangle reject: bit-equality with the kernels shows that their reject changes nothing.

For tests it also reports which feature class gave each result (PAIR_CLASSES for the closest pair, SWEEP_CLASSES for the
sweep), and it has an independent float64 reference: the segment-triangle distance as the minimum over x in [-1, 1] of
collide_oracle.point_triangle_dist64(c + x h) (convex in x, golden-section search), and the first contact from the convexity
of that distance along the path."""
import numpy as np

import collide_oracle as co
from raycast_oracle import Level0, _near_blocks, valid_ray
from voxels_b200 import capi

F = np.float32
INF = F(np.inf)
EPS = F(0.0625)
_dot, _cross = co._dot, co._cross

PAIR_CLASSES = ("endpoint", "edge", "crossing")
SWEEP_CLASSES = ("started", "cap_face", "parallelogram", "cap_edge", "lateral_edge", "shifted_vertex")


def _clamp01(x):
    return np.where(x < 0, F(0), np.where(x > 1, F(1), x)).astype(np.float32)


def _segment_edge(p0, D, A, q0, q1):
    """Candidate 3 for the edges q0 -> q1 [T, 3]: (dd [T], edge point [T, 3], t [T], w [T]); dd = +inf when A == 0."""
    E, R = q1 - q0, p0 - q0
    e, f = _dot(E, E), _dot(E, R)
    Db = np.broadcast_to(D, E.shape)
    c, b = _dot(Db, R), _dot(Db, E)
    den = A * e - b * b
    w_gen = np.where(den != 0, _clamp01((b * f - c * e) / den), F(0))
    t_gen = (b * w_gen + f) / e
    w_neg, w_pos = _clamp01(-c / A), _clamp01((b - c) / A)
    t = np.where(e == 0, F(0), np.where(t_gen < 0, F(0), np.where(t_gen > 1, F(1), t_gen))).astype(np.float32)
    w = np.where(e == 0, w_neg, np.where(t_gen < 0, w_neg, np.where(t_gen > 1, w_pos, w_gen))).astype(np.float32)
    y = q0 + t[:, None] * E
    dd = co.dist2(p0 + w[:, None] * D, y)
    if A == 0:
        dd = np.full(len(E), INF)
    return dd, y, t, w


@np.errstate(all="ignore")
def segment_triangles(ctr, h, tri):
    """The header's closest pair of the segment ctr -+ h and each triangle of tri [T, 3, 3] (float32):
    (dd [T], point [T, 3], u [T], v [T], w [T], class [T] as PAIR_CLASSES indices)."""
    ctr, h = np.asarray(ctr, np.float32), np.asarray(h, np.float32)
    p0, p1, D = ctr - h, ctr + h, h + h
    a, b, c = tri[:, 0], tri[:, 1], tri[:, 2]
    q, u, v, _ = co.closest_on_triangles(p0, tri)
    best = co.dist2(p0, q)
    w = np.zeros(len(tri), np.float32)
    cls = np.zeros(len(tri), np.int8)
    q1, u1, v1, _ = co.closest_on_triangles(p1, tri)
    d1 = co.dist2(p1, q1)
    take = d1 < best
    best, q, u, v, w = np.where(take, d1, best), np.where(take[:, None], q1, q), np.where(take, u1, u), np.where(take, v1, v), np.where(take, F(1), w)
    A = (D[0] * D[0] + D[1] * D[1]) + D[2] * D[2]
    one = F(1)
    for q0, q1e, uv in ((a, b, lambda t: (t, np.zeros_like(t))), (b, c, lambda t: (one - t, t)), (c, a, lambda t: (np.zeros_like(t), one - t))):
        de, y, t, we = _segment_edge(p0, D, A, q0, q1e)
        take = de < best
        ue, ve = uv(t)
        best, q, u, v, w = np.where(take, de, best), np.where(take[:, None], y, q), np.where(take, ue, u), np.where(take, ve, v), np.where(take, we, w)
        cls = np.where(take, 1, cls)
    e1, e2, s = b - a, c - a, p0 - a
    Db = np.broadcast_to(D, e2.shape)
    pv = _cross(Db, e2)
    det = _dot(e1, pv)
    inv = F(1) / det
    fu = _dot(s, pv) * inv
    qv = _cross(s, e1)
    fv = _dot(Db, qv) * inv
    fw = _dot(e2, qv) * inv
    take = (det != 0) & (fu >= 0) & (fu <= 1) & (fv >= 0) & (fu + fv <= 1) & (fw >= 0) & (fw <= 1) & (F(0) < best)
    pt = (a + e1 * fu[:, None]) + e2 * fv[:, None]
    best, q, u, v, w = np.where(take, F(0), best), np.where(take[:, None], pt, q), np.where(take, fu, u), np.where(take, fv, v), np.where(take, fw, w)
    cls = np.where(take, 2, cls)
    return best.astype(np.float32), q.astype(np.float32), u.astype(np.float32), v.astype(np.float32), w.astype(np.float32), cls


def _face_t(o, d, c0, r, t_min, t_max, a, b, c, quad):
    """The sphere sweep's face test on the vertices a, b, c [T, 3]; quad: the parallelogram a, b, b + c - a."""
    e1, e2 = b - a, c - a
    n = _cross(e1, e2)
    length = np.sqrt(_dot(n, n))
    side = _dot(c0 - a, n)
    k = np.where(side >= 0, r, -r)
    s = (o - k[:, None] * (n / length[:, None])) - a
    Db = np.broadcast_to(d, e2.shape)
    pv = _cross(Db, e2)
    det = _dot(e1, pv)
    inv = F(1) / det
    fu = _dot(s, pv) * inv
    qv = _cross(s, e1)
    fv = _dot(Db, qv) * inv
    ft = _dot(e2, qv) * inv
    inside = (fv <= 1) if quad else (fu + fv <= 1)
    ok = np.where(side >= 0, det > 0, det < 0) & (fu >= 0) & (fu <= 1) & (fv >= 0) & inside & (ft >= t_min) & (ft <= t_max)
    return np.where(ok, ft, INF)


@np.errstate(all="ignore")
def capsule_sweep_triangles(o, d, t_min, t_max, h, r, tri):
    """The header's per-triangle capsule sweep on tri [T, 3, 3] (float32): (contact t [T], +inf where none; started [T];
    class [T] as SWEEP_CLASSES indices, the first test in the header's order that gives the t)."""
    o, d, h = np.asarray(o, np.float32), np.asarray(d, np.float32), np.asarray(h, np.float32)
    t_min, t_max, r = F(t_min), F(t_max), F(r)
    rr = r * r
    dd = (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]
    c0 = o + t_min * d
    started = segment_triangles(c0, h, tri)[0] <= rr
    a, b, c = tri[:, 0], tri[:, 1], tri[:, 2]
    am, bm, cm, ap, bp, cp = a - h, b - h, c - h, a + h, b + h, c + h
    tests = [(_face_t(o, d, c0, r, t_min, t_max, am, bm, cm, False), 1), (_face_t(o, d, c0, r, t_min, t_max, ap, bp, cp, False), 1),
             (_face_t(o, d, c0, r, t_min, t_max, am, bm, ap, True), 2), (_face_t(o, d, c0, r, t_min, t_max, bm, cm, bp, True), 2),
             (_face_t(o, d, c0, r, t_min, t_max, cm, am, cp, True), 2)]
    tests += [(co._edge_t(o, d, q0, q1, rr, t_min, t_max), 3) for q0, q1 in ((am, bm), (bm, cm), (cm, am), (ap, bp), (bp, cp), (cp, ap))]
    tests += [(co._edge_t(o, d, q0, q1, rr, t_min, t_max), 4) for q0, q1 in ((am, ap), (bm, bp), (cm, cp))]
    tests += [(co._vertex_t(o, d, q, rr, dd, t_min, t_max), 5) for q in (am, bm, cm, ap, bp, cp)]
    t = np.full(len(tri), INF)
    cls = np.zeros(len(tri), np.int8)
    for tt, k in tests:
        take = tt < t
        t, cls = np.where(take, tt, t), np.where(take, k, cls)
    return np.where(started, t_min, t), started, np.where(started, 0, cls)


def reach_ok(h, extra):
    """The reach rule in float32: a finite half axis and max_i |h_i| + extra <= 15."""
    h = np.asarray(h, np.float32)
    return bool(np.all(np.isfinite(h)) and F(np.max(np.abs(h))) + F(extra) <= F(capi.VXB_SPHERE_RADIUS_MAX))


def _reject_passes(o, d, t_min, t_max, h, r, tri):
    """How many triangles pass the sweep kernel's per-triangle reject (the slab test on the box grown by |h_i| + r + eps)."""
    g = (np.abs(h) + F(r)) + EPS
    lo, hi = tri.min(axis=1) - g, tri.max(axis=1) + g
    te, tx = np.full(len(tri), F(t_min)), np.full(len(tri), F(t_max))
    for a in range(3):
        if d[a] == 0:
            out = ~((o[a] >= lo[:, a]) & (o[a] <= hi[:, a]))
            te[out], tx[out] = INF, -INF
            continue
        x, y = (lo[:, a] - o[a]) / d[a], (hi[:, a] - o[a]) / d[a]
        if d[a] < 0:
            x, y = y, x
        te, tx = np.maximum(te, x), np.minimum(tx, y)
    return int((te <= tx).sum())


def _pair_fields(h, ctr, tri1):
    _, q, u, v, w, _ = segment_triangles(ctr, h, tri1)
    s = (w[0] + w[0]) - F(1)
    return q[0], ctr + s * h, u[0], v[0], s


def capsule_cast(res, sweeps, level0=None, counts=None, classes=None):
    """CAPSULE_HIT_DTYPE hits of the CAPSULE_SWEEP_DTYPE `sweeps` against the level-0 triangles of `res`.  Invalid sweeps are
    misses (the device variant's rule).  `counts`, when a list, receives (blocks, triangles, triangles passing the kernel's
    reject) per sweep; `classes`, when a list, the SWEEP_CLASSES name of each hit (None for a miss)."""
    lv = Level0(res) if level0 is None else level0
    hits = np.zeros(len(sweeps), capi.CAPSULE_HIT_DTYPE)
    hits["t"] = np.inf
    hits["slot"] = capi.VXB_RAY_MISS
    with np.errstate(all="ignore"):
        for i, sw in enumerate(sweeps):
            ray, h, r = sw["path"], sw["half_axis"].astype(np.float32), F(sw["radius"])
            if not valid_ray(ray) or not r > 0 or not reach_ok(h, r):
                if counts is not None:
                    counts.append((0, 0, 0))
                if classes is not None:
                    classes.append(None)
                continue
            o, d = ray["origin"].astype(np.float32), ray["direction"].astype(np.float32)
            t_min, t_max = F(ray["t_min"]), F(ray["t_max"])
            near = _near_blocks(lv, o, d, t_min, t_max, float(np.max(np.abs(h))) + float(r) + 1.0)
            tri, blk, kk = co._gather(lv, near)
            if counts is not None:
                counts.append((len(near), len(tri), _reject_passes(o, d, t_min, t_max, h, r, tri) if len(tri) else 0))
            j = None
            if len(tri):
                ts, st, cl = capsule_sweep_triangles(o, d, t_min, t_max, h, r, tri)
                j = co._least(ts, lv, blk, kk, ts < INF)
            if classes is not None:
                classes.append(None if j is None else SWEEP_CLASSES[int(cl[j])])
            if j is None:
                continue
            t, b, k = ts[j], int(blk[j]), int(kk[j])
            x = hits[i]
            center = o + t * d
            x["point"], x["axis_point"], x["u"], x["v"], x["s"] = _pair_fields(h, center, lv.tri_pos[b][k:k + 1])
            x["t"], x["slot"], x["block_id"], x["triangle"], x["center"] = t, int(lv.slots[b]), lv.ids[b], k, center
            x["normal"] = co.blend_normal(lv.tri_nrm[b][k], x["u"], x["v"])
            x["flags"] = capi.VXB_SPHERE_STARTED_IN_CONTACT if st[j] else 0
    return hits


def _near_segment_blocks(lv, c, reach):
    """Blocks whose box is within `reach` of c along every axis (float64)."""
    c = np.asarray(c, np.float64)
    g = np.maximum(np.maximum(lv.lo - c, c - lv.hi), 0.0)
    return np.nonzero((g <= reach).all(axis=1))[0]


def closest_to_segment(res, segments, max_distance, level0=None, counts=None, classes=None):
    """SEGMENT_HIT_DTYPE hits of the SEGMENT_DTYPE `segments` within `max_distance`.  Invalid segments are misses (the device
    variant's rule); `counts` receives (blocks, triangles) per segment, `classes` the PAIR_CLASSES name of each hit."""
    lv = Level0(res) if level0 is None else level0
    md = F(max_distance)
    md2 = md * md
    hits = np.zeros(len(segments), capi.SEGMENT_HIT_DTYPE)
    hits["distance"] = np.inf
    hits["slot"] = capi.VXB_RAY_MISS
    with np.errstate(all="ignore"):
        for i, sg in enumerate(segments):
            c, h = sg["center"].astype(np.float32), sg["half_axis"].astype(np.float32)
            if not np.all(np.isfinite(c)) or not reach_ok(h, md):
                if counts is not None:
                    counts.append((0, 0))
                if classes is not None:
                    classes.append(None)
                continue
            near = _near_segment_blocks(lv, c, float(np.max(np.abs(h))) + float(md) + 1.0)
            tri, blk, kk = co._gather(lv, near)
            if counts is not None:
                counts.append((len(near), len(tri)))
            j = None
            if len(tri):
                dds, _, _, _, _, cl = segment_triangles(c, h, tri)
                j = co._least(dds, lv, blk, kk, dds <= md2)
            if classes is not None:
                classes.append(None if j is None else PAIR_CLASSES[int(cl[j])])
            if j is None:
                continue
            b, k = int(blk[j]), int(kk[j])
            x = hits[i]
            x["point"], x["axis_point"], x["u"], x["v"], x["s"] = _pair_fields(h, c, lv.tri_pos[b][k:k + 1])
            x["distance"], x["slot"], x["block_id"], x["triangle"] = np.sqrt(dds[j]), int(lv.slots[b]), lv.ids[b], k
            x["normal"] = co.blend_normal(lv.tri_nrm[b][k], x["u"], x["v"])
    return hits


same = co.same


# ---- the independent float64 reference ----------------------------------------------------------------------------------

_G = (np.sqrt(5.0) - 1) / 2


def segment_triangle_dist64(ctr, h, tri, iters=60):
    """Distances [T] from the segment ctr -+ h (ctr [3] or [T, 3]) to the triangles tri [T, 3, 3], float64: the minimum over
    x in [-1, 1] of the point distance at ctr + x h, by golden-section search (the distance is convex in x)."""
    tri = np.asarray(tri, np.float64)
    T = len(tri)
    ctr = np.broadcast_to(np.asarray(ctr, np.float64), (T, 3))
    h = np.asarray(h, np.float64)
    f = lambda x: co.point_triangle_dist64(ctr + x[:, None] * h, tri)  # noqa: E731
    lo, hi = np.full(T, -1.0), np.full(T, 1.0)
    for _ in range(iters):
        x1, x2 = hi - _G * (hi - lo), lo + _G * (hi - lo)
        left = f(x1) <= f(x2)
        hi, lo = np.where(left, x2, hi), np.where(left, lo, x1)
    return np.minimum(f(0.5 * (lo + hi)), np.minimum(f(np.full(T, -1.0)), f(np.full(T, 1.0))))


def capsule_first_contact64(o, d, t_lo, t_hi, h, r, tri, iters=60, slack=1e-9):
    """Per triangle, the first t in [t_lo, t_hi] (finite) with segment distance <= r + slack (+inf when none), and the least
    distance over the interval: golden-section search for the minimum along the path, then bisection left of it."""
    r = r + slack
    o, d = np.asarray(o, np.float64), np.asarray(d, np.float64)
    T = len(tri)
    f = lambda t: segment_triangle_dist64(o + t[:, None] * d, h, tri, iters=50)  # noqa: E731
    lo, hi = np.full(T, float(t_lo)), np.full(T, float(t_hi))
    for _ in range(iters):
        x1, x2 = hi - _G * (hi - lo), lo + _G * (hi - lo)
        left = f(x1) <= f(x2)
        hi, lo = np.where(left, x2, hi), np.where(left, lo, x1)
    tm = 0.5 * (lo + hi)
    f_lo = f(np.full(T, float(t_lo)))
    dmin = np.minimum(f(tm), np.minimum(f_lo, f(np.full(T, float(t_hi)))))
    tm = np.where(f_lo <= dmin, float(t_lo), tm)
    first = np.full(T, np.inf)
    start = f_lo <= r
    first[start] = float(t_lo)
    lo, hi = np.full(T, float(t_lo)), tm.copy()
    for _ in range(iters):
        mid = 0.5 * (lo + hi)
        inside = f(mid) <= r
        hi, lo = np.where(inside, mid, hi), np.where(inside, lo, mid)
    return np.where((dmin <= r) & ~start, hi, first), dmin
