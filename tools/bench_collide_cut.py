#!/usr/bin/env python
"""Collision queries against the drawn LOD cut (vxb_mesh_sphere_cast_cut* / vxb_mesh_closest_point_cut*) on an n^3 seeded
terrain after one full run and apply, with the level-0 queries on the same sweeps and points in the same process.  Reports,
with the card's name and power limit read in the same run:

  sweep_ms / point_ms   the host variants, one query per call at lod_factor 14.6, median and p99 over --calls calls
  sweeps / points       the device variants, --count camera sweeps at r = --radius and --count points near the surface at
                        max_distance = --max-distance, at lod_factor 4, 14.6 and 1e30, and vxb_mesh_sphere_cast_device /
                        vxb_mesh_closest_point_device on the same queries; CUDA events
  rebuild               the first cut query after an apply (the all-level map, the excursion and its read-back) against a
                        later one, host clock around a one-sweep host-variant call, median over --edits full runs and applies
  --verify              4096 queries of each kind at each factor against the numpy oracle (tests/collide_cut_oracle.py), with
                        the oracle's mean parts and triangles tested per query

    python tools/bench_collide_cut.py [--size 1024] [--count 1048576] [--calls 1000] [--radius 2] [--max-distance 4] [--verify]
"""
import argparse
import json
import os
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (REPO, os.path.join(REPO, "tools"), os.path.join(REPO, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402

from bench_collide import surface_points  # noqa: E402
from bench_raycast import camera_rays  # noqa: E402
from bench_resident import card  # noqa: E402

FACTORS = (4.0, 14.6, 1e30)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--count", type=int, default=1 << 20)
    ap.add_argument("--calls", type=int, default=1000)
    ap.add_argument("--radius", type=float, default=2.0)
    ap.add_argument("--max-distance", type=float, default=4.0)
    ap.add_argument("--edits", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--verify", action="store_true")
    args = ap.parse_args()

    import torch
    import voxels_b200
    from voxels_b200 import capi
    if not torch.cuda.is_available():
        raise SystemExit("bench_collide_cut: needs a CUDA device")
    name, power = card()
    n, r, md = args.size, args.radius, args.max_distance
    rng = np.random.RandomState(2027)
    ctx = voxels_b200.Context(0)
    ctx.fill(n, capi.Surface.terrain(n))
    ctx.polygonize()
    mesh = ctx.mesh()
    mesh.apply()
    res = mesh.download()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.ExternalStream(ctx.stream(), device=dev)
    camera = (0.5 * n, 0.75 * n, 0.5 * n)   # the LOD camera: above the middle of the terrain
    out = {"card": name, "power_limit": power, "size": n, "radius": r, "max_distance": md, "blocks": int(mesh.info().block_count),
           "lod_camera": camera}

    # (a) one query per call through the host variants
    sweeps = camera_rays(res, args.calls, rng)
    points = surface_points(res, args.calls, rng, md / 2)
    mesh.sphere_cast_cut(camera, 14.6, r, sweeps[:16]); mesh.closest_points_cut(camera, 14.6, points[:16], md)
    for key, call in (("sweep_ms", lambda k: mesh.sphere_cast_cut(camera, 14.6, r, sweeps[k:k + 1])),
                      ("point_ms", lambda k: mesh.closest_points_cut(camera, 14.6, points[k:k + 1], md))):
        lat = []
        for k in range(args.calls):
            t0 = time.perf_counter()
            call(k)
            lat.append(time.perf_counter() - t0)
        lat = np.array(lat) * 1e3
        out[key] = {"median": round(float(np.median(lat)), 4), "p99": round(float(np.percentile(lat, 99)), 4)}

    # (b) the device variants, cut and level 0 on the same queries
    def device_rate(queries, launch, hit_dtype):
        qt = torch.from_numpy(queries.view(np.uint8).copy()).to(dev)
        ht = torch.empty(len(queries) * hit_dtype.itemsize, dtype=torch.uint8, device=dev)
        torch.cuda.synchronize()
        launch(qt.data_ptr(), len(queries), ht.data_ptr())                   # warm-up
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record(stream)
        for _ in range(args.iters):
            launch(qt.data_ptr(), len(queries), ht.data_ptr())
        ev[1].record(stream)
        torch.cuda.synchronize()
        ms = ev[0].elapsed_time(ev[1]) / args.iters
        hits = ht.cpu().numpy().view(hit_dtype)
        got = {"ms": round(ms, 4), "per_s": round(len(queries) / (ms * 1e-3), 0),
               "hit_fraction": round(float((hits["slot"] != capi.VXB_RAY_MISS).mean()), 4)}
        if "level" in hit_dtype.names:
            got["hit_levels"] = {int(lv): int(c) for lv, c in zip(*np.unique(hits["level"][hits["slot"] != capi.VXB_RAY_MISS], return_counts=True))}
        return got

    rays = camera_rays(res, args.count, rng)
    pts = surface_points(res, args.count, rng, md / 2)
    out["sweeps"] = {"count": len(rays), "level0": device_rate(rays, lambda q, c, h: mesh.sphere_cast_device(r, q, c, h), capi.SPHERE_HIT_DTYPE)}
    out["points"] = {"count": len(pts), "level0": device_rate(pts, lambda q, c, h: mesh.closest_points_device(md, q, c, h), capi.CLOSEST_HIT_DTYPE)}
    for f in FACTORS:
        out["sweeps"]["cut %g" % f] = device_rate(rays, lambda q, c, h: mesh.sphere_cast_cut_device(camera, f, r, q, c, h),
                                                  capi.SPHERE_CUT_HIT_DTYPE)
        out["points"]["cut %g" % f] = device_rate(pts, lambda q, c, h: mesh.closest_points_cut_device(camera, f, md, q, c, h),
                                                  capi.CLOSEST_CUT_HIT_DTYPE)

    # (c) the rebuild: the first cut query after an apply against the next one
    first, later = [], []
    for _ in range(args.edits):
        ctx.polygonize()
        mesh.apply()
        t0 = time.perf_counter()
        mesh.sphere_cast_cut(camera, 14.6, r, sweeps[:1])
        t1 = time.perf_counter()
        mesh.sphere_cast_cut(camera, 14.6, r, sweeps[:1])
        t2 = time.perf_counter()
        first.append((t1 - t0) * 1e3); later.append((t2 - t1) * 1e3)
    out["rebuild_ms"] = {"first_query_median": round(float(np.median(first)), 4), "query_median": round(float(np.median(later)), 4),
                         "rebuild_median": round(float(np.median(np.array(first) - np.array(later))), 4)}

    if args.verify:
        import collide_cut_oracle as oracle
        import collide_oracle
        import raycast_cut_oracle
        res = mesh.download()
        q = rays[rng.choice(len(rays), 4096, replace=False)]
        p = pts[rng.choice(len(pts), 4096, replace=False)]
        ver = {}
        for f in FACTORS:
            d = raycast_cut_oracle.Drawn(res, camera, f)
            cs, cp = [], []
            want_s = oracle.sphere_cast_cut(res, camera, f, r, q, d, cs)
            want_p = oracle.closest_points_cut(res, camera, f, p, md, d, cp)
            cs, cp = np.array(cs, np.float64), np.array(cp, np.float64)
            ver["%g" % f] = {
                "sweeps": {"queries": len(q), "differ": int(len(collide_oracle.same(mesh.sphere_cast_cut(camera, f, r, q), want_s))),
                           "oracle_parts_per_query": round(float(cs[:, 0].mean()), 2), "oracle_triangles_per_query": round(float(cs[:, 1].mean()), 1)},
                "points": {"queries": len(p), "differ": int(len(collide_oracle.same(mesh.closest_points_cut(camera, f, p, md), want_p))),
                           "oracle_parts_per_query": round(float(cp[:, 0].mean()), 2), "oracle_triangles_per_query": round(float(cp[:, 1].mean()), 1)}}
        out["verify"] = ver
    mesh.close()
    ctx.close()
    print(json.dumps(out))
    if args.verify and any(v[k]["differ"] for v in out["verify"].values() for k in ("sweeps", "points")):
        sys.exit(1)


if __name__ == "__main__":
    main()
