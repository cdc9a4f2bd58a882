#!/usr/bin/env python
"""Collision queries against the resident mesh (vxb_mesh_sphere_cast* / vxb_mesh_closest_point*) on an n^3 seeded terrain
after one full run and apply.  Reports, with the card's name and power limit read in the same run:

  sweep_ms / point_ms   the host variants, one query per call, median and p99 over --calls calls, host clock
  sweeps                the device variant, --count camera sweeps at r = --radius, CUDA events
  points                the device variant, --count points near the surface at max_distance = --max-distance, CUDA events
  --verify              4096 queries of each kind against the numpy oracle (tests/collide_oracle.py), with the oracle's
                        mean blocks and triangles tested per query

    python tools/bench_collide.py [--size 1024] [--count 1048576] [--calls 1000] [--radius 2] [--max-distance 4] [--verify]
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

from bench_raycast import camera_rays  # noqa: E402
from bench_resident import card  # noqa: E402


def surface_points(res, count, rng, spread):
    lv = res.level(0)
    v = lv.verts["pos"][rng.randint(0, len(lv.verts), size=count)].astype(np.float32)
    return v + rng.uniform(-spread, spread, (count, 3)).astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--count", type=int, default=1 << 20)
    ap.add_argument("--calls", type=int, default=1000)
    ap.add_argument("--radius", type=float, default=2.0)
    ap.add_argument("--max-distance", type=float, default=4.0)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--verify", action="store_true")
    args = ap.parse_args()

    import torch
    import voxels_b200
    from voxels_b200 import capi
    if not torch.cuda.is_available():
        raise SystemExit("bench_collide: needs a CUDA device")
    name, power = card()
    n, r, md = args.size, args.radius, args.max_distance
    rng = np.random.RandomState(2026)
    ctx = voxels_b200.Context(0)
    ctx.fill(n, capi.Surface.terrain(n))
    ctx.polygonize()
    mesh = ctx.mesh()
    mesh.apply()
    res = mesh.download()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.ExternalStream(ctx.stream(), device=dev)
    out = {"card": name, "power_limit": power, "size": n, "radius": r, "max_distance": md,
           "level0_blocks": int(mesh.info().level_blocks[0])}

    # one query per call through the host variants
    sweeps = camera_rays(res, args.calls, rng)
    points = surface_points(res, args.calls, rng, md / 2)
    mesh.sphere_cast(r, sweeps[:16]); mesh.closest_points(points[:16], md)
    for key, call in (("sweep_ms", lambda k: mesh.sphere_cast(r, sweeps[k:k + 1])),
                      ("point_ms", lambda k: mesh.closest_points(points[k:k + 1], md))):
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

    out["sweeps"] = device_rate(camera_rays(res, args.count, rng), lambda q, c, h: mesh.sphere_cast_device(r, q, c, h),
                                capi.SPHERE_HIT_DTYPE)
    out["points"] = device_rate(surface_points(res, args.count, rng, md / 2),
                                lambda q, c, h: mesh.closest_points_device(md, q, c, h), capi.CLOSEST_HIT_DTYPE)

    if args.verify:
        import collide_oracle as oracle
        import raycast_oracle
        lv = raycast_oracle.Level0(res)
        ver = {}
        q = camera_rays(res, 4096, rng)
        counts = []
        want = oracle.sphere_cast(res, r, q, lv, counts)
        c = np.array(counts, np.float64)
        ver["sweeps"] = {"queries": len(q), "differ": int(len(oracle.same(mesh.sphere_cast(r, q), want))),
                         "oracle_blocks_per_query": round(float(c[:, 0].mean()), 2), "oracle_triangles_per_query": round(float(c[:, 1].mean()), 1)}
        p = surface_points(res, 4096, rng, md / 2)
        counts = []
        want = oracle.closest_points(res, p, md, lv, counts)
        c = np.array(counts, np.float64)
        ver["points"] = {"queries": len(p), "differ": int(len(oracle.same(mesh.closest_points(p, md), want))),
                         "oracle_blocks_per_query": round(float(c[:, 0].mean()), 2), "oracle_triangles_per_query": round(float(c[:, 1].mean()), 1)}
        out["verify"] = ver
    mesh.close()
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
