#!/usr/bin/env python
"""Ray queries against the resident mesh (vxb_mesh_raycast / vxb_mesh_raycast_device) on an n^3 seeded terrain after one full
run and apply.  Reports, with the card's name and power limit read in the same run:

  pick        the host variant, one ray per call (cursor pick), median and p99 over --picks calls, host clock
  camera      the device variant, --rays camera rays (origins above the terrain towards random surface points), CUDA events
  grazing     the device variant, --rays near-horizontal rays through the terrain (long block walks), CUDA events
  map         the rebuild of the level-0 block map after a region apply: a one-ray cast right after the apply against one
              without the rebuild, CUDA events, median over --edits brush edits
  --verify    4096 random rays of each set against the numpy oracle (tests/raycast_oracle.py), with the oracle's mean blocks
              and triangles tested per ray

    python tools/bench_raycast.py [--size 1024] [--rays 1048576] [--picks 1000] [--edits 20] [--verify]
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

from bench_resident import card  # noqa: E402


def camera_rays(res, count, rng):
    n = res.n
    from voxels_b200 import capi
    lv = res.level(0)
    target = lv.verts["pos"][rng.randint(0, len(lv.verts), size=count)].astype(np.float32)
    o = np.stack([rng.uniform(0, n, count), np.full(count, 1.25 * n), rng.uniform(0, n, count)], axis=1).astype(np.float32)
    return capi.make_rays(o, target - o)


def grazing_rays(n, count, rng):
    from voxels_b200 import capi
    a = rng.uniform(0, 2 * np.pi, count)
    o = np.stack([rng.uniform(0, n, count), rng.uniform(0.45 * n, 0.75 * n, count), rng.uniform(0, n, count)], axis=1)
    d = np.stack([np.cos(a), rng.uniform(-0.03, 0.01, count), np.sin(a)], axis=1)
    return capi.make_rays(o, d)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--rays", type=int, default=1 << 20)
    ap.add_argument("--picks", type=int, default=1000)
    ap.add_argument("--edits", type=int, default=20)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--verify", action="store_true")
    args = ap.parse_args()

    import torch
    import voxels_b200
    from voxels_b200 import capi
    from voxels_b200.capi import Op
    if not torch.cuda.is_available():
        raise SystemExit("bench_raycast: needs a CUDA device")
    name, power = card()
    n = args.size
    rng = np.random.RandomState(2024)
    ctx = voxels_b200.Context(0)
    ctx.fill(n, capi.Surface.terrain(n))
    ctx.polygonize()
    mesh = ctx.mesh()
    mesh.apply()
    res = mesh.download()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.ExternalStream(ctx.stream(), device=dev)
    out = {"card": name, "power_limit": power, "size": n, "level0_blocks": int(mesh.info().level_blocks[0])}

    # (a) picks: one ray per call through the host variant
    cam = camera_rays(res, args.picks, rng)
    mesh.raycast(cam[:16])
    lat = []
    for k in range(args.picks):
        t0 = time.perf_counter()
        mesh.raycast(cam[k:k + 1])
        lat.append(time.perf_counter() - t0)
    lat = np.array(lat) * 1e3
    out["pick_ms"] = {"median": round(float(np.median(lat)), 4), "p99": round(float(np.percentile(lat, 99)), 4)}

    def device_rate(rays):
        rt = torch.from_numpy(rays.view(np.uint8).copy()).to(dev)
        ht = torch.empty(len(rays) * capi.RAY_HIT_DTYPE.itemsize, dtype=torch.uint8, device=dev)
        torch.cuda.synchronize()
        mesh.raycast_device(rt.data_ptr(), len(rays), ht.data_ptr())        # warm-up (and the map)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record(stream)
        for _ in range(args.iters):
            mesh.raycast_device(rt.data_ptr(), len(rays), ht.data_ptr())
        ev[1].record(stream)
        torch.cuda.synchronize()
        ms = ev[0].elapsed_time(ev[1]) / args.iters
        hits = ht.cpu().numpy().view(capi.RAY_HIT_DTYPE)
        return {"ms": round(ms, 4), "rays_per_s": round(len(rays) / (ms * 1e-3), 0),
                "hit_fraction": round(float((hits["slot"] != capi.VXB_RAY_MISS).mean()), 4)}

    sets = {"camera": camera_rays(res, args.rays, rng), "grazing": grazing_rays(n, args.rays, rng)}
    for k, rays in sets.items():
        out[k] = device_rate(rays)

    # (c) the map rebuild after a region apply
    one = torch.from_numpy(sets["camera"][:1].view(np.uint8).copy()).to(dev)
    oh = torch.empty(capi.RAY_HIT_DTYPE.itemsize, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize()

    def one_cast_ms():
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record(stream)
        mesh.raycast_device(one.data_ptr(), 1, oh.data_ptr())
        ev[1].record(stream)
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1])

    dist0 = ctx.download_dense()[0]
    rebuild, plain = [], []
    while len(rebuild) < args.edits:
        x, y, z = (int(v) for v in rng.randint(16, n - 16, size=3))
        if abs(int(dist0[z, y, x])) >= 4:
            continue
        box = ctx.inject_program(np.array([x, y, z], np.float32), np.full(3, 20.0, np.float32), [Op.sphere(8.0)], len(rebuild) % 2 * 2)
        ctx.polygonize_region(box[:3], box[3:])
        mesh.apply()
        rebuild.append(one_cast_ms())
        plain.append(one_cast_ms())
    out["map_rebuild_ms"] = {"cast_after_apply_median": round(float(np.median(rebuild)), 4),
                             "cast_median": round(float(np.median(plain)), 4),
                             "rebuild_median": round(float(np.median(np.array(rebuild) - np.array(plain))), 4)}

    if args.verify:
        import raycast_oracle as oracle
        res = mesh.download()
        lv = oracle.Level0(res)
        ver = {}
        for k, rays in (("camera", camera_rays(res, 4096, rng)), ("grazing", grazing_rays(n, 4096, rng))):
            counts = []
            want = oracle.raycast(res, rays, lv, counts)
            got = mesh.raycast(rays)
            c = np.array(counts, np.float64)
            ver[k] = {"rays": len(rays), "differ": int(len(oracle.same_hits(got, want))),
                      "oracle_blocks_per_ray": round(float(c[:, 0].mean()), 2), "oracle_triangles_per_ray": round(float(c[:, 1].mean()), 1)}
        out["verify"] = ver
    mesh.close()
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
