#!/usr/bin/env python
"""Capsule queries against the resident mesh (vxb_mesh_capsule_cast* / vxb_mesh_closest_to_segment*) on an n^3 seeded terrain
after one full run and apply.  Reports, with the card's name and power limit read in the same run:

  capsule_ms / segment_ms   the host variants, one query per call, median and p99 over --calls calls, host clock
  capsules                  the device variant, --count camera sweeps of a capsule (half axis --half-axis, radius --radius),
                            CUDA events
  spheres                   the sphere sweep at the same radius on the same paths, for comparison, CUDA events
  segments                  the device variant, --count segments near the surface at max_distance = --max-distance
  --verify                  --verify-count queries of each kind against the numpy oracle (tests/capsule_oracle.py), with the
                            oracle's mean blocks, triangles and triangles passing the kernel's per-triangle reject per query

    python tools/bench_capsule.py [--size 1024] [--count 1048576] [--calls 1000] [--radius 0.5] [--half-axis 0 1.5 0]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--count", type=int, default=1 << 20)
    ap.add_argument("--calls", type=int, default=1000)
    ap.add_argument("--radius", type=float, default=0.5)
    ap.add_argument("--half-axis", type=float, nargs=3, default=(0.0, 1.5, 0.0))
    ap.add_argument("--max-distance", type=float, default=2.0)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--verify", action="store_true")
    ap.add_argument("--verify-count", type=int, default=1024)
    args = ap.parse_args()

    import torch
    import voxels_b200
    from voxels_b200 import capi
    if not torch.cuda.is_available():
        raise SystemExit("bench_capsule: needs a CUDA device")
    name, power = card()
    n, r, md, h = args.size, args.radius, args.max_distance, np.asarray(args.half_axis, np.float32)
    rng = np.random.RandomState(2026)
    ctx = voxels_b200.Context(0)
    ctx.fill(n, capi.Surface.terrain(n))
    ctx.polygonize()
    mesh = ctx.mesh()
    mesh.apply()
    res = mesh.download()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.ExternalStream(ctx.stream(), device=dev)
    out = {"card": name, "power_limit": power, "size": n, "radius": r, "half_axis": [float(x) for x in h], "max_distance": md,
           "level0_blocks": int(mesh.info().level_blocks[0])}

    def capsules(rays):
        s = np.zeros(len(rays), capi.CAPSULE_SWEEP_DTYPE)
        s["path"], s["half_axis"], s["radius"] = rays, h, np.float32(r)
        return s

    def segments(points):
        return capi.make_segments(points, h)

    # one query per call through the host variants
    sweeps = capsules(camera_rays(res, args.calls, rng))
    segs = segments(surface_points(res, args.calls, rng, md / 2))
    mesh.capsule_cast(sweeps[:16]); mesh.closest_to_segment(segs[:16], md)
    for key, call in (("capsule_ms", lambda k: mesh.capsule_cast(sweeps[k:k + 1])),
                      ("segment_ms", lambda k: mesh.closest_to_segment(segs[k:k + 1], md))):
        lat = []
        for k in range(args.calls):
            t0 = time.perf_counter()
            call(k)
            lat.append(time.perf_counter() - t0)
        lat = np.array(lat) * 1e3
        out[key] = {"median": round(float(np.median(lat)), 4), "p99": round(float(np.percentile(lat, 99)), 4)}

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
        return {"count": len(queries), "ms": round(ms, 4), "per_s": round(len(queries) / (ms * 1e-3), 0),
                "hit_fraction": round(float((hits["slot"] != capi.VXB_RAY_MISS).mean()), 4)}

    rays = camera_rays(res, args.count, rng)
    out["capsules"] = device_rate(capsules(rays), lambda q, c, x: mesh.capsule_cast_device(q, c, x), capi.CAPSULE_HIT_DTYPE)
    out["spheres"] = device_rate(rays, lambda q, c, x: mesh.sphere_cast_device(r, q, c, x), capi.SPHERE_HIT_DTYPE)
    out["segments"] = device_rate(segments(surface_points(res, args.count, rng, md / 2)),
                                  lambda q, c, x: mesh.closest_to_segment_device(md, q, c, x), capi.SEGMENT_HIT_DTYPE)

    if args.verify:
        import capsule_oracle as oracle
        import raycast_oracle
        lv = raycast_oracle.Level0(res)
        ver = {}
        q = capsules(camera_rays(res, args.verify_count, rng))
        counts = []
        want = oracle.capsule_cast(res, q, lv, counts)
        c = np.array(counts, np.float64)
        ver["capsules"] = {"queries": len(q), "differ": int(len(oracle.same(mesh.capsule_cast(q), want))),
                           "oracle_blocks_per_query": round(float(c[:, 0].mean()), 2),
                           "oracle_triangles_per_query": round(float(c[:, 1].mean()), 1),
                           "triangles_passing_reject_per_query": round(float(c[:, 2].mean()), 1)}
        p = segments(surface_points(res, args.verify_count, rng, md / 2))
        counts = []
        want = oracle.closest_to_segment(res, p, md, lv, counts)
        c = np.array(counts, np.float64)
        ver["segments"] = {"queries": len(p), "differ": int(len(oracle.same(mesh.closest_to_segment(p, md), want))),
                           "oracle_blocks_per_query": round(float(c[:, 0].mean()), 2),
                           "oracle_triangles_per_query": round(float(c[:, 1].mean()), 1)}
        out["verify"] = ver
    mesh.close()
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
