"""numpy oracle of vxb_mesh_sphere_cast_cut and vxb_mesh_closest_point_cut (include/vxb200.h "collision queries against the
drawn LOD cut"): the drawn parts of raycast_cut_oracle.Drawn (the cut of tests/cut_oracle.py, each vertex at the position
the renderer selects), collide_oracle's float32 sweep and closest-point formulas on those positions, and the cut's tie rule
(least t or dd, then lower slot, then lower part - regular, face 0 ... face 5 - then lower triangle).

A float64 test on each part's own box of selected positions, grown by the reach (r or max_distance) plus one voxel, skips
parts the query cannot reach.  It shares nothing with the kernels' walk or with the excursion."""
import numpy as np

from collide_oracle import INF, _near_point_blocks, blend_normal, closest_on_triangles, dist2, sweep_triangles
from raycast_cut_oracle import REGULAR, Drawn, _near_parts
from raycast_oracle import valid_ray
from voxels_b200 import capi

F = np.float32


def _gather(d, near):
    """The triangles of the parts `near` (indices into d.slot) as one array: (positions [T, 3, 3], part index [T], triangle
    number within its part [T])."""
    if not hasattr(d, "flat"):
        counts = np.array([len(p) for p in d.tri_pos], np.int64)
        d.flat = (np.concatenate(d.tri_pos) if len(d.tri_pos) else np.zeros((0, 3, 3), np.float32),
                  np.concatenate([[0], np.cumsum(counts)]), counts, np.array(d.slot, np.int64), np.array(d.part, np.int64))
    pos, start, counts, _, _ = d.flat
    c = counts[near]
    blk = np.repeat(near, c)
    k = np.arange(c.sum()) - np.repeat(np.cumsum(c) - c, c)
    return pos[start[blk] + k], blk, k


def _least(key, d, blk, k, ok):
    """The index (into the gathered triangles) of the least (key, slot, part, triangle) among `ok`, or None."""
    ks = np.nonzero(ok)[0]
    if not len(ks):
        return None
    slots, parts = d.flat[3], d.flat[4]
    return ks[np.lexsort((k[ks], parts[blk[ks]], slots[blk[ks]], key[ks]))[0]]


# The NaN that CUDA's float arithmetic produces (sign clear, all fraction bits set); numpy on the host produces another bit
# pattern.  A degenerate drawn triangle (a transition triangle whose selected positions coincide) can win a sweep and give
# NaN contact fields; the oracle writes them with the device's bits so that whole hits still compare bit for bit.
CUDA_NAN = np.uint32(0x7FFFFFFF).view(np.float32)


def _canonical_nan(h, fields):
    for f in fields:
        h[f] = np.where(np.isnan(h[f]), CUDA_NAN, h[f])


def _where(h, d, b, k):
    slot, part = d.slot[b], d.part[b]
    h["slot"], h["block_id"], h["triangle"] = slot, d.ids[slot], k
    h["level"] = d.levels[slot]
    h["face"] = REGULAR if part == 0 else part - 1


def sphere_cast_cut(res, camera, lod_factor, radius, rays, drawn=None, counts=None):
    """SPHERE_CUT_HIT_DTYPE hits of sweeps of a sphere of `radius` along `rays` (RAY_DTYPE) against the drawn cut of
    (camera, lod_factor).  Invalid rays are misses (the device variant's rule).  `counts`, when a list, receives (parts
    tested, triangles tested) per sweep."""
    d = Drawn(res, camera, lod_factor) if drawn is None else drawn
    r = F(radius)
    hits = np.zeros(len(rays), capi.SPHERE_CUT_HIT_DTYPE)
    hits["t"] = np.inf
    hits["slot"] = capi.VXB_RAY_MISS
    with np.errstate(all="ignore"):
        for i, ray in enumerate(rays):
            if not valid_ray(ray):
                if counts is not None:
                    counts.append((0, 0))
                continue
            o, dv = ray["origin"].astype(np.float32), ray["direction"].astype(np.float32)
            t_min, t_max = F(ray["t_min"]), F(ray["t_max"])
            near = _near_parts(d, o, dv, t_min, t_max, float(r) + 1.0)
            tri, blk, kk = _gather(d, near)
            if counts is not None:
                counts.append((len(near), len(tri)))
            if not len(tri):
                continue
            ts, st = sweep_triangles(o, dv, t_min, t_max, r, tri)
            j = _least(ts, d, blk, kk, ts < INF)
            if j is None:
                continue
            t, b, k = ts[j], int(blk[j]), int(kk[j])
            h = hits[i]
            center = o + t * dv
            q, u, v, _ = closest_on_triangles(center, tri[j:j + 1])
            _where(h, d, b, k)
            h["t"], h["center"], h["point"], h["u"], h["v"] = t, center, q[0], u[0], v[0]
            h["normal"] = blend_normal(d.tri_nrm[b][k], u[0], v[0])
            h["flags"] = capi.VXB_SPHERE_STARTED_IN_CONTACT if st[j] else 0
            _canonical_nan(h, ("t", "center", "point", "normal", "u", "v"))
    return hits


def closest_points_cut(res, camera, lod_factor, points, max_distance, drawn=None, counts=None):
    """CLOSEST_CUT_HIT_DTYPE hits of the [count, 3] `points` within `max_distance` of the drawn cut of (camera, lod_factor).
    Points with a non-finite coordinate are misses (the device variant's rule).  `counts` as for sphere_cast_cut."""
    d = Drawn(res, camera, lod_factor) if drawn is None else drawn
    pts = np.asarray(points, np.float32).reshape(-1, 3)
    md = F(max_distance)
    md2 = md * md
    hits = np.zeros(len(pts), capi.CLOSEST_CUT_HIT_DTYPE)
    hits["distance"] = np.inf
    hits["slot"] = capi.VXB_RAY_MISS
    with np.errstate(all="ignore"):
        for i, p in enumerate(pts):
            if not np.all(np.isfinite(p)):
                if counts is not None:
                    counts.append((0, 0))
                continue
            near = _near_point_blocks(d, p, float(md) + 1.0)
            tri, blk, kk = _gather(d, near)
            if counts is not None:
                counts.append((len(near), len(tri)))
            if not len(tri):
                continue
            qs, us, vs, _ = closest_on_triangles(p, tri)
            d2s = dist2(p, qs)
            j = _least(d2s, d, blk, kk, d2s <= md2)
            if j is None:
                continue
            b, k = int(blk[j]), int(kk[j])
            h = hits[i]
            _where(h, d, b, k)
            h["distance"], h["point"], h["u"], h["v"] = np.sqrt(d2s[j]), qs[j], us[j], vs[j]
            h["normal"] = blend_normal(d.tri_nrm[b][k], us[j], vs[j])
            _canonical_nan(h, ("distance", "point", "normal", "u", "v"))
    return hits


def _round_up(x):
    """float64 values [...] rounded up to float32."""
    f = x.astype(np.float32)
    return np.where(f.astype(np.float64) < x, np.nextafter(f, F(np.inf)), f)


def excursion(res, bounds):
    """The excursion e as the mesh measures it: per block the largest distance by which its measured box ([block_count, 6]
    {min xyz, max xyz} in directory order, Mesh.bounds()) leaves its lattice box along an axis, each difference rounded up to
    float32; the largest over the blocks, at least 0."""
    if not len(res.records):
        return F(0)
    level = res.records["level"].astype(np.int64)
    cid = res.records["coord_id"].astype(np.int64)
    nb, s = (res.n // 16) >> level, (16 << level).astype(np.float64)
    lo = np.stack([cid % nb, cid // (nb * nb), (cid // nb) % nb], axis=1) * s[:, None]   # output axes (x, z, y); exact
    box = np.asarray(bounds, np.float32).astype(np.float64)
    e = np.maximum(_round_up(lo - box[:, :3]), _round_up(box[:, 3:] - (lo + s[:, None])))
    return F(max(0.0, float(e.max())))


def reach_limit(e):
    """The largest float32 R <= 15 with e + R <= 15 in float32: the farthest reach the cut queries accept."""
    R = F(15) - F(e)
    while F(e) + R > F(15):
        R = np.nextafter(R, F(0))
    return R
