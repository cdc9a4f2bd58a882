#!/usr/bin/env python
"""Ray queries against the drawn LOD cut (vxb_mesh_raycast_cut / _device) on an n^3 seeded terrain after one full run and
apply, with vxb_mesh_raycast on the same rays in the same process.  Reports, with the card's name and power limit read in
the same run:

  pick        the host variant, one ray per call (cursor pick) at lod_factor 14.6, median and p99 over --picks calls
  camera      the device variant, --rays camera rays (origins above the terrain towards random surface points) at lod_factor
              4, 14.6 and 1e30, and vxb_mesh_raycast_device on the same rays; CUDA events
  rebuild     the first cut cast after an apply (the all-level map, the excursion and its read-back) against a later one,
              host clock around a one-ray host-variant cast, median over --edits full runs and applies
  --verify    4096 of the camera rays at each factor against the numpy oracle (tests/raycast_cut_oracle.py), with the oracle's
              mean blocks and triangles tested per ray

    python tools/bench_raycast_cut.py [--size 1024] [--rays 1048576] [--picks 1000] [--edits 5] [--verify]
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

FACTORS = (4.0, 14.6, 1e30)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--rays", type=int, default=1 << 20)
    ap.add_argument("--picks", type=int, default=1000)
    ap.add_argument("--edits", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--verify", action="store_true")
    args = ap.parse_args()

    import torch
    import voxels_b200
    from voxels_b200 import capi
    if not torch.cuda.is_available():
        raise SystemExit("bench_raycast_cut: needs a CUDA device")
    name, power = card()
    n = args.size
    rng = np.random.RandomState(2025)
    ctx = voxels_b200.Context(0)
    ctx.fill(n, capi.Surface.terrain(n))
    ctx.polygonize()
    mesh = ctx.mesh()
    mesh.apply()
    res = mesh.download()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.ExternalStream(ctx.stream(), device=dev)
    camera = (0.5 * n, 0.75 * n, 0.5 * n)   # the LOD camera: above the middle of the terrain
    out = {"card": name, "power_limit": power, "size": n, "blocks": int(mesh.info().block_count), "lod_camera": camera}

    # (a) picks: one ray per call through the host variant
    cam = camera_rays(res, args.picks, rng)
    mesh.raycast_cut(camera, 14.6, cam[:16])
    lat = []
    for k in range(args.picks):
        t0 = time.perf_counter()
        mesh.raycast_cut(camera, 14.6, cam[k:k + 1])
        lat.append(time.perf_counter() - t0)
    lat = np.array(lat) * 1e3
    out["pick_ms"] = {"median": round(float(np.median(lat)), 4), "p99": round(float(np.percentile(lat, 99)), 4)}

    # (b) 2^20 camera rays through the device variants
    rays = camera_rays(res, args.rays, rng)
    rt = torch.from_numpy(rays.view(np.uint8).copy()).to(dev)
    ht = torch.empty(len(rays) * capi.CUT_HIT_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize()

    def timed(cast):
        cast()                                                                    # warm-up
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record(stream)
        for _ in range(args.iters):
            cast()
        ev[1].record(stream)
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]) / args.iters

    def rate(ms, hits):
        return {"ms": round(ms, 4), "rays_per_s": round(len(rays) / (ms * 1e-3), 0),
                "hit_fraction": round(float((hits["slot"] != capi.VXB_RAY_MISS).mean()), 4)}

    ms = timed(lambda: mesh.raycast_device(rt.data_ptr(), len(rays), ht.data_ptr()))
    out["level0"] = rate(ms, ht[:len(rays) * capi.RAY_HIT_DTYPE.itemsize].cpu().numpy().view(capi.RAY_HIT_DTYPE))
    cut = {}
    for f in FACTORS:
        ms = timed(lambda: mesh.raycast_cut_device(camera, f, rt.data_ptr(), len(rays), ht.data_ptr()))
        hits = ht.cpu().numpy().view(capi.CUT_HIT_DTYPE)
        r = rate(ms, hits)
        r["hit_levels"] = {int(lv): int(c) for lv, c in zip(*np.unique(hits["level"][hits["slot"] != capi.VXB_RAY_MISS], return_counts=True))}
        cut["%g" % f] = r
    out["cut"] = cut
    del ht

    # (c) the rebuild: the first cut cast after an apply against the next one
    first, later = [], []
    for _ in range(args.edits):
        ctx.polygonize()
        mesh.apply()
        t0 = time.perf_counter()
        mesh.raycast_cut(camera, 14.6, cam[:1])
        t1 = time.perf_counter()
        mesh.raycast_cut(camera, 14.6, cam[:1])
        t2 = time.perf_counter()
        first.append((t1 - t0) * 1e3); later.append((t2 - t1) * 1e3)
    out["rebuild_ms"] = {"first_cast_median": round(float(np.median(first)), 4), "cast_median": round(float(np.median(later)), 4),
                         "rebuild_median": round(float(np.median(np.array(first) - np.array(later))), 4)}

    if args.verify:
        import raycast_cut_oracle as oracle
        import raycast_oracle
        res = mesh.download()
        pick = rays[rng.choice(len(rays), 4096, replace=False)]
        ver = {}
        for f in FACTORS:
            counts = []
            want = oracle.raycast_cut(res, camera, f, pick, counts=counts)
            got = mesh.raycast_cut(camera, f, pick)
            c = np.array(counts, np.float64)
            ver["%g" % f] = {"rays": len(pick), "differ": int(len(raycast_oracle.same_hits(got, want))),
                             "oracle_blocks_per_ray": round(float(c[:, 0].mean()), 2),
                             "oracle_triangles_per_ray": round(float(c[:, 1].mean()), 1)}
        out["verify"] = ver
    mesh.close()
    ctx.close()
    print(json.dumps(out))
    if args.verify and any(v["differ"] for v in out["verify"].values()):
        sys.exit(1)


if __name__ == "__main__":
    main()
