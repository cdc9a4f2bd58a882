"""numpy oracle of vxb_mesh_sphere_cast and vxb_mesh_closest_point (include/vxb200.h "collision queries"): the header's float32
formulas in its order (explicit np.float32 throughout, so nothing is promoted to float64), the global minimum by the tie rule
(least t or distance, then lower slot, then lower triangle) over every level-0 triangle of a downloaded mesh (capi.Result).

Blocks the query cannot reach are skipped by a float64 box test with the box grown by the reach plus one voxel; every
other block is tested in full.

Also an independent float64 reference that shares none of the oracle's formulas: the distance from a point to a triangle by
projection onto the plane and onto the three edges, and the sweep's first contact per triangle by the convexity of
dist(c(t), triangle) in t (the minimum by golden-section search, then bisection of the branch left of it)."""
import numpy as np

from raycast_oracle import Level0, _near_blocks, valid_ray
from voxels_b200 import capi

F = np.float32
INF = F(np.inf)


def _dot(x, y):
    return (x[..., 0] * y[..., 0] + x[..., 1] * y[..., 1]) + x[..., 2] * y[..., 2]


def _cross(x, y):
    return np.stack([x[..., 1] * y[..., 2] - x[..., 2] * y[..., 1], x[..., 2] * y[..., 0] - x[..., 0] * y[..., 2],
                     x[..., 0] * y[..., 1] - x[..., 1] * y[..., 0]], axis=-1)


# region numbers of closest_on_triangles, in the header's test order
REGIONS = ("A", "B", "AB", "C", "AC", "BC", "face")


@np.errstate(all="ignore")
def closest_on_triangles(p, tri):
    """Ericson's ClosestPtPointTriangle as the header states it, for the point p [3] (or [T, 3]) and triangles tri [T, 3, 3]
    (float32): (point [T, 3], u [T], v [T], region [T])."""
    p = np.asarray(p, np.float32)
    a, b, c = tri[:, 0], tri[:, 1], tri[:, 2]
    ab, ac, ap = b - a, c - a, p - a
    d1, d2 = _dot(ab, ap), _dot(ac, ap)
    bp = p - b
    d3, d4 = _dot(ab, bp), _dot(ac, bp)
    vc = d1 * d4 - d3 * d2
    cp = p - c
    d5, d6 = _dot(ab, cp), _dot(ac, cp)
    vb = d5 * d2 - d1 * d6
    va = d3 * d6 - d5 * d4
    e43, e56 = d4 - d3, d5 - d6
    region = np.select([(d1 <= 0) & (d2 <= 0), (d3 >= 0) & (d4 <= d3), (vc <= 0) & (d1 >= 0) & (d3 <= 0), (d6 >= 0) & (d5 <= d6),
                        (vb <= 0) & (d2 >= 0) & (d6 <= 0), (va <= 0) & (e43 >= 0) & (e56 >= 0)], [0, 1, 2, 3, 4, 5], 6)
    w_ab = d1 / (d1 - d3)
    w_ac = d2 / (d2 - d6)
    w_bc = e43 / (e43 + e56)
    den = F(1) / ((va + vb) + vc)
    fv, fw = vb * den, vc * den
    q = np.empty_like(a)
    u = np.zeros(len(a), np.float32)
    v = np.zeros(len(a), np.float32)
    sel = [region == i for i in range(7)]
    q[sel[0]] = a[sel[0]]
    q[sel[1]] = b[sel[1]]; u[sel[1]] = F(1)
    q[sel[2]] = (a + w_ab[:, None] * ab)[sel[2]]; u[sel[2]] = w_ab[sel[2]]
    q[sel[3]] = c[sel[3]]; v[sel[3]] = F(1)
    q[sel[4]] = (a + w_ac[:, None] * ac)[sel[4]]; v[sel[4]] = w_ac[sel[4]]
    q[sel[5]] = (b + w_bc[:, None] * (c - b))[sel[5]]; u[sel[5]] = (F(1) - w_bc)[sel[5]]; v[sel[5]] = w_bc[sel[5]]
    q[sel[6]] = ((a + ab * fv[:, None]) + ac * fw[:, None])[sel[6]]; u[sel[6]] = fv[sel[6]]; v[sel[6]] = fw[sel[6]]
    return q, u, v, region


def dist2(p, q):
    d = np.asarray(p, np.float32) - q
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def _edge_t(o, d, q0, q1, rr, t_min, t_max):
    e, w = q1 - q0, o - q0
    ee = _dot(e, e)
    de, we = _cross(np.broadcast_to(d, e.shape), e), _cross(w, e)
    A, B, g = _dot(de, de), _dot(de, we), _dot(np.broadcast_to(d, we.shape), we)
    disc = ee * (rr * A - g * g)
    t = (-B - np.sqrt(disc)) / A
    s = ((w[:, 0] + t * d[0]) * e[:, 0] + (w[:, 1] + t * d[1]) * e[:, 1]) + (w[:, 2] + t * d[2]) * e[:, 2]
    ok = (A > 0) & (disc >= 0) & (s >= 0) & (s <= ee) & (t >= t_min) & (t <= t_max)
    return np.where(ok, t, INF)


def _vertex_t(o, d, q, rr, dd, t_min, t_max):
    w = o - q
    B = (w[:, 0] * d[0] + w[:, 1] * d[1]) + w[:, 2] * d[2]
    x = _cross(w, np.broadcast_to(d, w.shape))
    disc = rr * dd - _dot(x, x)
    t = (-B - np.sqrt(disc)) / dd
    ok = (dd > 0) & (disc >= 0) & (t >= t_min) & (t <= t_max)
    return np.where(ok, t, INF)


@np.errstate(all="ignore")
def sweep_triangles(o, d, t_min, t_max, r, tri):
    """The header's per-triangle sweep on tri [T, 3, 3] (float32): (contact t [T], +inf where none; started [T])."""
    o, d = np.asarray(o, np.float32), np.asarray(d, np.float32)
    t_min, t_max, r = F(t_min), F(t_max), F(r)
    rr = r * r
    dd = (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]
    c0 = o + t_min * d
    q, _, _, _ = closest_on_triangles(c0, tri)
    started = dist2(c0, q) <= rr
    a, b, c = tri[:, 0], tri[:, 1], tri[:, 2]
    e1, e2 = b - a, c - a
    n = _cross(e1, e2)
    length = np.sqrt(_dot(n, n))
    side = _dot(c0 - a, n)
    k = np.where(side >= 0, r, -r)
    s = (o - k[:, None] * (n / length[:, None])) - a
    pv = _cross(np.broadcast_to(d, e2.shape), e2)
    det = _dot(e1, pv)
    inv = F(1) / det
    fu = _dot(s, pv) * inv
    qv = _cross(s, e1)
    fv = _dot(np.broadcast_to(d, qv.shape), qv) * inv
    ft = _dot(e2, qv) * inv
    face = np.where(side >= 0, det > 0, det < 0) & (fu >= 0) & (fu <= 1) & (fv >= 0) & (fu + fv <= 1) & (ft >= t_min) & (ft <= t_max)
    t = np.where(face, ft, INF)
    for q0, q1 in ((a, b), (b, c), (c, a)):
        t = np.minimum(t, _edge_t(o, d, q0, q1, rr, t_min, t_max))
    for q0 in (a, b, c):
        t = np.minimum(t, _vertex_t(o, d, q0, rr, dd, t_min, t_max))
    return np.where(started, t_min, t), started


def blend_normal(nrm, u, v):
    """The ray hit's normal: nrm [3 vertices, 3] blended at (u, v), normalised, float32."""
    n0, n1, n2 = nrm
    w = (F(1) - u) - v
    nv = (w * n0 + u * n1) + v * n2
    length = np.sqrt((nv[0] * nv[0] + nv[1] * nv[1]) + nv[2] * nv[2])
    return nv / length if length > 0 else np.zeros(3, np.float32)


def _gather(lv, near):
    """The triangles of the blocks `near` (indices into lv.slots) as one array: (positions [T, 3, 3], block index [T],
    triangle number within its block [T])."""
    if not hasattr(lv, "flat"):
        counts = np.array([len(p) for p in lv.tri_pos], np.int64)
        lv.flat = (np.concatenate(lv.tri_pos) if len(lv.tri_pos) else np.zeros((0, 3, 3), np.float32),
                   np.concatenate([[0], np.cumsum(counts)]), counts)
    pos, start, counts = lv.flat
    c = counts[near]
    blk = np.repeat(near, c)
    k = np.arange(c.sum()) - np.repeat(np.cumsum(c) - c, c)
    return pos[start[blk] + k], blk, k


def _least(key, lv, blk, k, ok):
    """The index (into the gathered triangles) of the least (key, slot, triangle) among `ok`, or None."""
    ks = np.nonzero(ok)[0]
    if not len(ks):
        return None
    return ks[np.lexsort((k[ks], lv.slots[blk[ks]], key[ks]))[0]]


def sphere_cast(res, radius, rays, level0=None, counts=None):
    """SPHERE_HIT_DTYPE hits of sweeps of a sphere of `radius` along `rays` (RAY_DTYPE) against the level-0 triangles of
    `res`.  Invalid rays are misses (the device variant's rule).  `counts`, when a list, receives (blocks tested, triangles
    tested) per sweep."""
    lv = Level0(res) if level0 is None else level0
    r = F(radius)
    hits = np.zeros(len(rays), capi.SPHERE_HIT_DTYPE)
    hits["t"] = np.inf
    hits["slot"] = capi.VXB_RAY_MISS
    with np.errstate(all="ignore"):
        for i, ray in enumerate(rays):
            if not valid_ray(ray):
                if counts is not None:
                    counts.append((0, 0))
                continue
            o, d = ray["origin"].astype(np.float32), ray["direction"].astype(np.float32)
            t_min, t_max = F(ray["t_min"]), F(ray["t_max"])
            near = _near_blocks(lv, o, d, t_min, t_max, float(r) + 1.0)
            tri, blk, kk = _gather(lv, near)
            if counts is not None:
                counts.append((len(near), len(tri)))
            if not len(tri):
                continue
            ts, st = sweep_triangles(o, d, t_min, t_max, r, tri)
            j = _least(ts, lv, blk, kk, ts < INF)
            if j is None:
                continue
            t, b, k, started = ts[j], int(blk[j]), int(kk[j]), bool(st[j])
            slot = int(lv.slots[b])
            h = hits[i]
            center = o + t * d
            q, u, v, _ = closest_on_triangles(center, lv.tri_pos[b][k:k + 1])
            h["t"], h["slot"], h["block_id"], h["triangle"] = t, slot, lv.ids[b], k
            h["center"], h["point"], h["u"], h["v"] = center, q[0], u[0], v[0]
            h["normal"] = blend_normal(lv.tri_nrm[b][k], u[0], v[0])
            h["flags"] = capi.VXB_SPHERE_STARTED_IN_CONTACT if started else 0
    return hits


def _near_point_blocks(lv, p, reach):
    p = np.asarray(p, np.float64)
    g = np.maximum(np.maximum(lv.lo - p, p - lv.hi), 0.0)
    return np.nonzero(np.sqrt((g * g).sum(axis=1)) <= reach)[0]


def closest_points(res, points, max_distance, level0=None, counts=None):
    """CLOSEST_HIT_DTYPE hits of the [count, 3] `points` within `max_distance` of the level-0 triangles of `res`.  Points
    with a non-finite coordinate are misses (the device variant's rule)."""
    lv = Level0(res) if level0 is None else level0
    pts = np.asarray(points, np.float32).reshape(-1, 3)
    md = F(max_distance)
    md2 = md * md
    hits = np.zeros(len(pts), capi.CLOSEST_HIT_DTYPE)
    hits["distance"] = np.inf
    hits["slot"] = capi.VXB_RAY_MISS
    with np.errstate(all="ignore"):
        for i, p in enumerate(pts):
            if not np.all(np.isfinite(p)):
                if counts is not None:
                    counts.append((0, 0))
                continue
            near = _near_point_blocks(lv, p, float(md) + 1.0)
            tri, blk, kk = _gather(lv, near)
            if counts is not None:
                counts.append((len(near), len(tri)))
            if not len(tri):
                continue
            qs, us, vs, _ = closest_on_triangles(p, tri)
            d2s = dist2(p, qs)
            j = _least(d2s, lv, blk, kk, d2s <= md2)
            if j is None:
                continue
            d2, b, k, q, u, v = d2s[j], int(blk[j]), int(kk[j]), qs[j], us[j], vs[j]
            slot = int(lv.slots[b])
            h = hits[i]
            h["distance"], h["slot"], h["block_id"], h["triangle"] = np.sqrt(d2), slot, lv.ids[b], k
            h["point"], h["u"], h["v"] = q, u, v
            h["normal"] = blend_normal(lv.tri_nrm[b][k], u, v)
    return hits


def same(got, want):
    """Every field of every hit bit-identical: the indices of the queries that differ."""
    a, b = got.view(np.uint32).reshape(len(got), -1), want.view(np.uint32).reshape(len(want), -1)
    return np.nonzero((a != b).any(axis=1))[0]


# ---- the independent float64 reference ----------------------------------------------------------------------------------

def _seg_dist64(p, a, b):
    """Distances [T] from points p [T, 3] to segments a -> b [T, 3] (float64)."""
    e = b - a
    ee = (e * e).sum(axis=1)
    s = np.where(ee > 0, ((p - a) * e).sum(axis=1) / np.where(ee > 0, ee, 1.0), 0.0)
    s = np.clip(s, 0.0, 1.0)
    return np.linalg.norm(p - (a + s[:, None] * e), axis=1)


def point_triangle_dist64(p, tri):
    """Distances [T] from p ([3] or [T, 3]) to the triangles tri [T, 3, 3], float64: the plane's foot when it lies inside
    the triangle (same-side tests against the three edges), otherwise the nearest of the three edges."""
    tri = np.asarray(tri, np.float64)
    p = np.broadcast_to(np.asarray(p, np.float64), (len(tri), 3))
    a, b, c = tri[:, 0], tri[:, 1], tri[:, 2]
    n = np.cross(b - a, c - a)
    nn = np.linalg.norm(n, axis=1)
    edge = np.minimum(np.minimum(_seg_dist64(p, a, b), _seg_dist64(p, b, c)), _seg_dist64(p, c, a))
    ok = nn > 1e-12 * np.maximum(1.0, np.linalg.norm(b - a, axis=1) * np.linalg.norm(c - a, axis=1))
    unit = n / np.where(ok, nn, 1.0)[:, None]
    h = ((p - a) * unit).sum(axis=1)
    foot = p - h[:, None] * unit
    inside = ok.copy()
    for x, y in ((a, b), (b, c), (c, a)):
        inside &= (np.cross(y - x, foot - x) * unit).sum(axis=1) >= 0
    return np.where(inside, np.abs(h), edge)


def sweep_first_contact64(o, d, t_lo, t_hi, r, tri, iters=80, slack=1e-9):
    """Per triangle of tri [T, 3, 3], the first t in [t_lo, t_hi] (finite) with dist(o + t d, triangle) <= r + slack, +inf
    when the path never comes that close; and the least distance over the interval.  float64, by convexity in t (the slack
    keeps a tangent graze at exactly r, whose float64 minimum can round a hair above r, a contact)."""
    r = r + slack
    o, d = np.asarray(o, np.float64), np.asarray(d, np.float64)
    T = len(tri)
    f = lambda t: point_triangle_dist64(o + t[:, None] * d, tri)  # noqa: E731
    lo, hi = np.full(T, float(t_lo)), np.full(T, float(t_hi))
    g = (np.sqrt(5.0) - 1) / 2
    for _ in range(iters):                                   # golden-section search for the minimum
        x1, x2 = hi - g * (hi - lo), lo + g * (hi - lo)
        left = f(x1) <= f(x2)
        hi = np.where(left, x2, hi)
        lo = np.where(left, lo, x1)
    tm = 0.5 * (lo + hi)
    dmin = np.minimum(f(tm), np.minimum(f(np.full(T, float(t_lo))), f(np.full(T, float(t_hi)))))
    tm = np.where(f(np.full(T, float(t_lo))) <= dmin, float(t_lo), tm)
    first = np.full(T, np.inf)
    touch = dmin <= r
    start = f(np.full(T, float(t_lo))) <= r
    first[start] = float(t_lo)
    lo, hi = np.full(T, float(t_lo)), tm.copy()
    for _ in range(iters):                                   # bisection of the decreasing branch
        mid = 0.5 * (lo + hi)
        inside = f(mid) <= r
        hi = np.where(inside, mid, hi)
        lo = np.where(inside, lo, mid)
    first = np.where(touch & ~start, hi, first)
    return first, dmin


def segment_bounds64(n, o, d, t_min, t_max, reach):
    """The finite parameter range of the segment inside the grid box grown by `reach` (None when it misses the box)."""
    o, d = np.asarray(o, np.float64), np.asarray(d, np.float64)
    lo, hi = float(t_min), float(t_max)
    for a in range(3):
        if d[a] == 0:
            if o[a] < -reach or o[a] > n + reach:
                return None
            continue
        ta, tb = (-reach - o[a]) / d[a], (n + reach - o[a]) / d[a]
        lo, hi = max(lo, min(ta, tb)), min(hi, max(ta, tb))
    return (lo, hi) if lo <= hi else None
