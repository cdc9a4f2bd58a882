"""numpy oracle of vxb_mesh_capsule_cast_cut and vxb_mesh_closest_to_segment_cut (include/vxb200.h "capsule queries against
the drawn LOD cut"): the drawn parts of raycast_cut_oracle.Drawn (the cut of tests/cut_oracle.py, each vertex at the position
the renderer selects), capsule_oracle's float32 capsule sweep, closest pair and pair fields on those positions, and the cut's
tie rule (least t or dd, then lower slot, then lower part - regular, face 0 ... face 5 - then lower triangle) through
collide_cut_oracle's gather and least.

A float64 test on each part's own box of selected positions, grown by max_i |h_i| + r (or max_distance) plus one voxel,
skips parts the query cannot reach.  It shares nothing with the kernels' walk.  The cut reach rule needs the mesh's
excursion e (collide_cut_oracle.excursion); a query out of reach is a miss, the device variants' rule."""
import numpy as np

import capsule_oracle as co
from collide_cut_oracle import _canonical_nan, _gather, _least, _where
from collide_oracle import blend_normal
from raycast_cut_oracle import Drawn, _near_parts
from raycast_oracle import valid_ray
from voxels_b200 import capi

F = np.float32
INF = F(np.inf)


def reach(h, extra):
    """A query's reach R = max_i |h_i| + extra in float32."""
    return F(np.max(np.abs(np.asarray(h, np.float32)))) + F(extra)


def cut_reach_ok(h, extra, e):
    """The cut reach rule in float32 and in the header's order: capsule_oracle.reach_ok, then e + (max_i |h_i| + extra) <= 15."""
    return co.reach_ok(h, extra) and F(e) + reach(h, extra) <= F(capi.VXB_SPHERE_RADIUS_MAX)


def capsule_cast_cut(res, camera, lod_factor, sweeps, e, drawn=None, counts=None, classes=None):
    """CAPSULE_CUT_HIT_DTYPE hits of the CAPSULE_SWEEP_DTYPE `sweeps` against the drawn cut of (camera, lod_factor) of a mesh
    with excursion e.  Invalid sweeps and sweeps out of cut reach are misses.  `counts`, when a list, receives (parts,
    triangles, triangles passing the kernel's reject) per sweep; `classes`, when a list, the SWEEP_CLASSES name of each hit
    (None for a miss)."""
    d = Drawn(res, camera, lod_factor) if drawn is None else drawn
    hits = np.zeros(len(sweeps), capi.CAPSULE_CUT_HIT_DTYPE)
    hits["t"] = np.inf
    hits["slot"] = capi.VXB_RAY_MISS
    with np.errstate(all="ignore"):
        for i, sw in enumerate(sweeps):
            ray, h, r = sw["path"], sw["half_axis"].astype(np.float32), F(sw["radius"])
            if not valid_ray(ray) or not r > 0 or not cut_reach_ok(h, r, e):
                if counts is not None:
                    counts.append((0, 0, 0))
                if classes is not None:
                    classes.append(None)
                continue
            o, dv = ray["origin"].astype(np.float32), ray["direction"].astype(np.float32)
            t_min, t_max = F(ray["t_min"]), F(ray["t_max"])
            near = _near_parts(d, o, dv, t_min, t_max, float(np.max(np.abs(h))) + float(r) + 1.0)
            tri, blk, kk = _gather(d, near)
            if counts is not None:
                counts.append((len(near), len(tri), co._reject_passes(o, dv, t_min, t_max, h, r, tri) if len(tri) else 0))
            j = None
            if len(tri):
                ts, st, cl = co.capsule_sweep_triangles(o, dv, t_min, t_max, h, r, tri)
                j = _least(ts, d, blk, kk, ts < INF)
            if classes is not None:
                classes.append(None if j is None else co.SWEEP_CLASSES[int(cl[j])])
            if j is None:
                continue
            t, b, k = ts[j], int(blk[j]), int(kk[j])
            x = hits[i]
            center = o + t * dv
            _where(x, d, b, k)
            x["point"], x["axis_point"], x["u"], x["v"], x["s"] = co._pair_fields(h, center, tri[j:j + 1])
            x["t"], x["center"] = t, center
            x["normal"] = blend_normal(d.tri_nrm[b][k], x["u"], x["v"])
            x["flags"] = capi.VXB_SPHERE_STARTED_IN_CONTACT if st[j] else 0
            _canonical_nan(x, ("t", "center", "point", "axis_point", "normal", "u", "v", "s"))
    return hits


def closest_to_segment_cut(res, camera, lod_factor, segments, max_distance, e, drawn=None, counts=None, classes=None):
    """SEGMENT_CUT_HIT_DTYPE hits of the SEGMENT_DTYPE `segments` within `max_distance` of the drawn cut of (camera,
    lod_factor) of a mesh with excursion e.  Invalid segments and segments out of cut reach are misses; `counts` receives
    (parts, triangles) per segment, `classes` the PAIR_CLASSES name of each hit."""
    d = Drawn(res, camera, lod_factor) if drawn is None else drawn
    md = F(max_distance)
    md2 = md * md
    hits = np.zeros(len(segments), capi.SEGMENT_CUT_HIT_DTYPE)
    hits["distance"] = np.inf
    hits["slot"] = capi.VXB_RAY_MISS
    with np.errstate(all="ignore"):
        for i, sg in enumerate(segments):
            c, h = sg["center"].astype(np.float32), sg["half_axis"].astype(np.float32)
            if not np.all(np.isfinite(c)) or not cut_reach_ok(h, md, e):
                if counts is not None:
                    counts.append((0, 0))
                if classes is not None:
                    classes.append(None)
                continue
            near = co._near_segment_blocks(d, c, float(np.max(np.abs(h))) + float(md) + 1.0)
            tri, blk, kk = _gather(d, near)
            if counts is not None:
                counts.append((len(near), len(tri)))
            j = None
            if len(tri):
                dds, _, _, _, _, cl = co.segment_triangles(c, h, tri)
                j = _least(dds, d, blk, kk, dds <= md2)
            if classes is not None:
                classes.append(None if j is None else co.PAIR_CLASSES[int(cl[j])])
            if j is None:
                continue
            b, k = int(blk[j]), int(kk[j])
            x = hits[i]
            _where(x, d, b, k)
            x["point"], x["axis_point"], x["u"], x["v"], x["s"] = co._pair_fields(h, c, tri[j:j + 1])
            x["distance"] = np.sqrt(dds[j])
            x["normal"] = blend_normal(d.tri_nrm[b][k], x["u"], x["v"])
            _canonical_nan(x, ("distance", "point", "axis_point", "normal", "u", "v", "s"))
    return hits
