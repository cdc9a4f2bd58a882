#!/usr/bin/env python
"""Capsule queries against the drawn LOD cut (vxb_mesh_capsule_cast_cut* / vxb_mesh_closest_to_segment_cut*) on an n^3 seeded
terrain after one full run and apply, with the level-0 capsule queries on the same sweeps and segments in the same process.
Reports, with the card's name and power limit read in the same run:

  capsule_ms / segment_ms   the host variants, one query per call at lod_factor 14.6, median and p99 over --calls calls
  capsules / segments       the device variants, --count camera sweeps of a capsule (half axis --half-axis, radius --radius)
                            and --count segments near the surface at max_distance = --max-distance, at lod_factor 4, 14.6
                            and 1e30, and vxb_mesh_capsule_cast_device / vxb_mesh_closest_to_segment_device on the same
                            queries; CUDA events
  rebuild_ms                the first cut query after an apply (the all-level map, the excursion and its read-back) against
                            a later one, host clock around a one-sweep host-variant call, median over --edits full runs and
                            applies
  --verify                  --verify-count queries of each kind at each factor against the numpy oracle
                            (tests/capsule_cut_oracle.py), with the oracle's mean parts and triangles tested per query

The LOD camera is bench_collide_cut.py's.

    python tools/bench_capsule_cut.py [--size 1024] [--count 1048576] [--calls 300] [--radius 0.5] [--half-axis 0 1.5 0]
                                      [--max-distance 2] [--verify]
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
    ap.add_argument("--calls", type=int, default=300)
    ap.add_argument("--radius", type=float, default=0.5)
    ap.add_argument("--half-axis", type=float, nargs=3, default=(0.0, 1.5, 0.0))
    ap.add_argument("--max-distance", type=float, default=2.0)
    ap.add_argument("--edits", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--verify", action="store_true")
    ap.add_argument("--verify-count", type=int, default=1024)
    args = ap.parse_args()

    import torch
    import voxels_b200
    from voxels_b200 import capi
    if not torch.cuda.is_available():
        raise SystemExit("bench_capsule_cut: needs a CUDA device")
    name, power = card()
    n, r, md, h = args.size, args.radius, args.max_distance, np.asarray(args.half_axis, np.float32)
    rng = np.random.RandomState(2028)
    ctx = voxels_b200.Context(0)
    ctx.fill(n, capi.Surface.terrain(n))
    ctx.polygonize()
    mesh = ctx.mesh()
    mesh.apply()
    res = mesh.download()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.ExternalStream(ctx.stream(), device=dev)
    camera = (0.5 * n, 0.75 * n, 0.5 * n)   # the LOD camera of bench_collide_cut.py: above the middle of the terrain
    out = {"card": name, "power_limit": power, "size": n, "radius": r, "half_axis": [float(x) for x in h], "max_distance": md,
           "blocks": int(mesh.info().block_count), "lod_camera": camera}

    def capsules(rays):
        s = np.zeros(len(rays), capi.CAPSULE_SWEEP_DTYPE)
        s["path"], s["half_axis"], s["radius"] = rays, h, np.float32(r)
        return s

    def segments(points):
        return capi.make_segments(points, h)

    # (a) one query per call through the host variants
    sweeps = capsules(camera_rays(res, args.calls, rng))
    segs = segments(surface_points(res, args.calls, rng, md / 2))
    mesh.capsule_cast_cut(camera, 14.6, sweeps[:16]); mesh.closest_to_segment_cut(camera, 14.6, segs[:16], md)
    for key, call in (("capsule_ms", lambda k: mesh.capsule_cast_cut(camera, 14.6, sweeps[k:k + 1])),
                      ("segment_ms", lambda k: mesh.closest_to_segment_cut(camera, 14.6, segs[k:k + 1], md))):
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

    caps = capsules(camera_rays(res, args.count, rng))
    segq = segments(surface_points(res, args.count, rng, md / 2))
    out["capsules"] = {"count": len(caps), "level0": device_rate(caps, lambda q, c, x: mesh.capsule_cast_device(q, c, x), capi.CAPSULE_HIT_DTYPE)}
    out["segments"] = {"count": len(segq), "level0": device_rate(segq, lambda q, c, x: mesh.closest_to_segment_device(md, q, c, x),
                                                                 capi.SEGMENT_HIT_DTYPE)}
    for f in FACTORS:
        out["capsules"]["cut %g" % f] = device_rate(caps, lambda q, c, x: mesh.capsule_cast_cut_device(camera, f, q, c, x),
                                                    capi.CAPSULE_CUT_HIT_DTYPE)
        out["segments"]["cut %g" % f] = device_rate(segq, lambda q, c, x: mesh.closest_to_segment_cut_device(camera, f, md, q, c, x),
                                                    capi.SEGMENT_CUT_HIT_DTYPE)

    # (c) the rebuild: the first cut query after an apply against the next one
    first, later = [], []
    for _ in range(args.edits):
        ctx.polygonize()
        mesh.apply()
        t0 = time.perf_counter()
        mesh.capsule_cast_cut(camera, 14.6, sweeps[:1])
        t1 = time.perf_counter()
        mesh.capsule_cast_cut(camera, 14.6, sweeps[:1])
        t2 = time.perf_counter()
        first.append((t1 - t0) * 1e3); later.append((t2 - t1) * 1e3)
    out["rebuild_ms"] = {"first_query_median": round(float(np.median(first)), 4), "query_median": round(float(np.median(later)), 4),
                         "rebuild_median": round(float(np.median(np.array(first) - np.array(later))), 4)}

    if args.verify:
        import capsule_cut_oracle as oracle
        import collide_cut_oracle
        import collide_oracle
        import raycast_cut_oracle
        res = mesh.download()
        e = collide_cut_oracle.excursion(res, mesh.bounds())
        q = caps[rng.choice(len(caps), args.verify_count, replace=False)]
        p = segq[rng.choice(len(segq), args.verify_count, replace=False)]
        ver = {"excursion": float(e)}
        for f in FACTORS:
            d = raycast_cut_oracle.Drawn(res, camera, f)
            cs, cp = [], []
            want_s = oracle.capsule_cast_cut(res, camera, f, q, e, d, cs)
            want_p = oracle.closest_to_segment_cut(res, camera, f, p, md, e, d, cp)
            cs, cp = np.array(cs, np.float64), np.array(cp, np.float64)
            ver["%g" % f] = {
                "capsules": {"queries": len(q), "differ": int(len(collide_oracle.same(mesh.capsule_cast_cut(camera, f, q), want_s))),
                             "oracle_parts_per_query": round(float(cs[:, 0].mean()), 2),
                             "oracle_triangles_per_query": round(float(cs[:, 1].mean()), 1),
                             "triangles_passing_reject_per_query": round(float(cs[:, 2].mean()), 1)},
                "segments": {"queries": len(p), "differ": int(len(collide_oracle.same(mesh.closest_to_segment_cut(camera, f, p, md), want_p))),
                             "oracle_parts_per_query": round(float(cp[:, 0].mean()), 2),
                             "oracle_triangles_per_query": round(float(cp[:, 1].mean()), 1)}}
        out["verify"] = ver
    mesh.close()
    ctx.close()
    print(json.dumps(out))
    if args.verify and any(v[k]["differ"] for fk, v in out["verify"].items() if fk != "excursion" for k in ("capsules", "segments")):
        sys.exit(1)


if __name__ == "__main__":
    main()
