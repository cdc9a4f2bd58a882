"""numpy oracle of vxb_mesh_raycast_cut (include/vxb200.h "ray queries against the drawn LOD cut"): the cut of
tests/cut_oracle.py, the drawn triangles of every (slot, part) with each vertex at the position the renderer selects (sec
when its mask, the bits of sec[3], is non-zero and covered by block_adj), raycast_oracle's float32 Moeller-Trumbore test and
the tie rule (least t, then lower slot, then lower part - regular, face 0 ... face 5 - then lower triangle).

A float64 slab test per part, on the part's own box of selected positions grown by one voxel, skips parts the segment does
not come near: an accepted hit lies within rounding of its triangle.  It uses neither the kernel's walk nor its excursion."""
import types

import numpy as np

import cut_oracle
from raycast_oracle import F, moller_trumbore, valid_ray
from voxels_b200 import capi

REGULAR = 0xFFFFFFFF


class Drawn:
    """The drawn set of the cut of (camera, lod_factor) over a downloaded mesh `res`: per part (slot, part index 0 regular /
    1 + f transition face f) the selected triangle positions [T, 3, 3], normals [T, 3, 3], whether a vertex of the triangle
    took its secondary position [T] and a float64 box."""

    def __init__(self, res, camera, lod_factor):
        recs = res.records
        self.selected, self.adj = cut_oracle.cut(recs, res.n, int(res.info.levels), camera, lod_factor)
        self.slot, self.part, self.tri_pos, self.tri_nrm, self.moved, lo, hi = [], [], [], [], [], [], []
        for s in np.nonzero(self.selected)[0]:
            r, a = recs[s], np.uint32(self.adj[s])
            pieces = [(0, res.verts, res.idx, int(r["vertex_offset"]), int(r["index_offset"]), int(r["index_count"]))]
            for f in range(6):
                if (int(a) >> f) & 1:
                    pieces.append((1 + f, res.tverts, res.tidx, int(r["trans_vertex_offset"][f]), int(r["trans_index_offset"][f]),
                                   int(r["trans_index_count"][f])))
            for p, verts, idx, vo, io, ic in pieces:
                tri = idx[io:io + ic].astype(np.int64).reshape(-1, 3) + vo
                v = verts[tri]                                                    # [T, 3] vertices
                mask = np.ascontiguousarray(v["sec"][..., 3]).view(np.uint32)
                use = (mask != 0) & ((mask & a) == mask)
                pos = np.where(use[..., None], v["sec"][..., :3], v["pos"]).astype(np.float32)
                self.slot.append(int(s)); self.part.append(p); self.moved.append(use.any(axis=1))
                self.tri_pos.append(pos); self.tri_nrm.append(v["nrm"].astype(np.float32))
                flat = pos.reshape(-1, 3).astype(np.float64)
                lo.append(flat.min(axis=0) if len(flat) else np.full(3, np.inf))
                hi.append(flat.max(axis=0) if len(flat) else np.full(3, -np.inf))
        self.lo = np.array(lo, np.float64).reshape(-1, 3)
        self.hi = np.array(hi, np.float64).reshape(-1, 3)
        self.ids = recs["id"].astype(np.uint32)
        self.levels = recs["level"].astype(np.uint32)


def _near_parts(d, o, dv, t_min, t_max, grow=1.0):
    o64, d64 = o.astype(np.float64), dv.astype(np.float64)
    te = np.full(len(d.lo), float(t_min)); tx = np.full(len(d.lo), float(t_max))
    for a in range(3):
        lo, hi = d.lo[:, a] - grow, d.hi[:, a] + grow
        if d64[a] == 0.0:
            te[(o64[a] < lo) | (o64[a] > hi)] = np.inf
            continue
        ta, tb = (lo - o64[a]) / d64[a], (hi - o64[a]) / d64[a]
        te = np.maximum(te, np.minimum(ta, tb)); tx = np.minimum(tx, np.maximum(ta, tb))
    return np.nonzero(te <= tx)[0]


def raycast_cut(res, camera, lod_factor, rays, drawn=None, counts=None):
    """CUT_HIT_DTYPE hits of `rays` against the drawn cut.  Invalid rays are misses (the device variant's rule).  `counts`,
    when a list, receives (blocks tested, triangles tested) per ray."""
    d = Drawn(res, camera, lod_factor) if drawn is None else drawn
    hits = np.zeros(len(rays), capi.CUT_HIT_DTYPE)
    hits["t"] = np.inf
    hits["slot"] = capi.VXB_RAY_MISS
    with np.errstate(all="ignore"):
        for r, ray in enumerate(rays):
            if not valid_ray(ray):
                if counts is not None:
                    counts.append((0, 0))
                continue
            o, dv = ray["origin"].astype(np.float32), ray["direction"].astype(np.float32)
            t_min, t_max = F(ray["t_min"]), F(ray["t_max"])
            near = _near_parts(d, o, dv, t_min, t_max)
            best = None
            tested = 0
            for b in near:
                p = d.tri_pos[b]
                tested += len(p)
                if not len(p):
                    continue
                hit, t, u, v = moller_trumbore(o, dv, t_min, t_max, p)
                ks = np.nonzero(hit)[0]
                if not len(ks):
                    continue
                k = ks[np.lexsort((ks, t[ks]))[0]]
                cand = (t[k], d.slot[b], d.part[b], int(k), u[k], v[k], b)
                if best is None or cand[:4] < best[:4]:
                    best = cand
            if counts is not None:
                counts.append((len({d.slot[b] for b in near}), tested))
            if best is None:
                continue
            t, slot, part, k, u, v, b = best
            h = hits[r]
            h["t"], h["u"], h["v"], h["slot"], h["block_id"], h["triangle"] = t, u, v, slot, d.ids[slot], k
            h["position"] = o + t * dv
            n0, n1, n2 = d.tri_nrm[b][k]
            w = (F(1) - u) - v
            nv = (w * n0 + u * n1) + v * n2
            length = np.sqrt((nv[0] * nv[0] + nv[1] * nv[1]) + nv[2] * nv[2])
            h["normal"] = nv / length if length > 0 else np.zeros(3, np.float32)
            h["level"] = d.levels[slot]
            h["face"] = REGULAR if part == 0 else part - 1
    return hits


def _vertices(pos, sec=None, mask=None, nrm=None):
    v = np.zeros(len(pos), capi.VERTEX_DTYPE)
    v["pos"] = pos
    v["nrm"] = (0.0, 1.0, 0.0) if nrm is None else nrm
    if sec is not None:
        v["sec"][:, :3] = sec
        v["sec"][:, 3] = np.asarray(mask, np.uint32).view(np.float32)
    return v


def result_from_blocks(n, levels, blocks):
    """A capi.Result for hand-built meshes: blocks = [(level, grid block coordinate (x, y, z), regular, {face: transition})] in
    directory order, each mesh a dict(pos=[V, 3], idx=[I], and optionally sec=[V, 3], mask=[V], nrm=[V, 3])."""
    records = np.zeros(len(blocks), capi.RECORD_DTYPE)
    verts, idx, tverts, tidx = [], [], [], []
    vo = io = tvo = tio = 0
    for s, (level, (x, y, z), reg, trans) in enumerate(blocks):
        nb = (n // 16) >> level
        rec = records[s]
        rec["level"], rec["coord_id"], rec["id"] = level, (z * nb + y) * nb + x, 1000 + s
        v = _vertices(reg["pos"], reg.get("sec"), reg.get("mask"), reg.get("nrm"))
        rec["vertex_count"], rec["index_count"], rec["vertex_offset"], rec["index_offset"] = len(v), len(reg["idx"]), vo, io
        verts.append(v); idx.append(np.asarray(reg["idx"], np.uint32))
        vo += len(v); io += len(reg["idx"])
        for f, t in trans.items():
            tv = _vertices(t["pos"], t.get("sec"), t.get("mask"), t.get("nrm"))
            rec["trans_vertex_count"][f], rec["trans_index_count"][f] = len(tv), len(t["idx"])
            rec["trans_vertex_offset"][f], rec["trans_index_offset"][f] = tvo, tio
            tverts.append(tv); tidx.append(np.asarray(t["idx"], np.uint32))
            tvo += len(tv); tio += len(t["idx"])
    res = capi.Result.__new__(capi.Result)
    res.n, res.info, res.records = n, types.SimpleNamespace(levels=levels), records
    cat = lambda parts, dt: np.concatenate(parts) if parts else np.zeros(0, dt)  # noqa: E731
    res.verts, res.idx = cat(verts, capi.VERTEX_DTYPE), cat(idx, np.uint32)
    res.tverts, res.tidx = cat(tverts, capi.VERTEX_DTYPE), cat(tidx, np.uint32)
    return res
