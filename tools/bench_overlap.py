#!/usr/bin/env python
"""Box overlap gathers (vxb_mesh_overlap_box / _device) on an n^3 seeded terrain after one full run and apply.  Reports, with
the card's name and power limit read in the same run:

  host        one 4^3 body box centred on a surface vertex per call (a physics mid-phase query), median and p99 over --calls
              calls, host clock
  body        --boxes such boxes through the device variant: count only (tris NULL), and count plus fill; CUDA events;
              triangles written per second
  tiles       4096 navmesh-tile boxes of 64^3 around the surface, count plus fill
  whole       the single box covering the whole grid (one warp walks every block), count plus fill
  --verify    256 body boxes and 16 tiles against the numpy oracle (tests/overlap_oracle.py), with the oracle's mean blocks and
              triangles tested per box

    python tools/bench_overlap.py [--size 1024] [--boxes 1048576] [--calls 1000] [--verify]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--boxes", type=int, default=1 << 20)
    ap.add_argument("--calls", type=int, default=1000)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--verify", action="store_true")
    args = ap.parse_args()

    import torch
    import voxels_b200
    from voxels_b200 import capi
    if not torch.cuda.is_available():
        raise SystemExit("bench_overlap: needs a CUDA device")
    name, power = card()
    n = args.size
    rng = np.random.RandomState(2026)
    ctx = voxels_b200.Context(0)
    ctx.fill(n, capi.Surface.terrain(n))
    ctx.polygonize()
    mesh = ctx.mesh()
    mesh.apply()
    res = mesh.download()
    lvl0 = res.records[res.records["level"] == 0]
    pos = res.verts["pos"].astype(np.float32)
    verts = np.concatenate([pos[int(r["vertex_offset"]):int(r["vertex_offset"]) + int(r["vertex_count"])] for r in lvl0])
    tris0 = int((lvl0["index_count"] // 3).sum())
    dev = torch.device("cuda", 0)
    stream = torch.cuda.ExternalStream(ctx.stream(), device=dev)
    out = {"card": name, "power_limit": power, "size": n, "level0_blocks": int(len(lvl0)), "level0_triangles": tris0}

    def body(count):
        c = verts[rng.randint(0, len(verts), count)]
        return capi.make_boxes(c - 2.0, c + 2.0)

    # (a) one body box per call through the host variant
    one = body(args.calls)
    mesh.overlap_boxes(one[:16])
    lat = []
    for k in range(args.calls):
        t0 = time.perf_counter()
        mesh.overlap_boxes(one[k:k + 1])
        lat.append(time.perf_counter() - t0)
    lat = np.array(lat) * 1e3
    out["host_ms"] = {"median": round(float(np.median(lat)), 4), "p99": round(float(np.percentile(lat, 99)), 4)}

    def timed(call):
        call()                                                                    # warm-up
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record(stream)
        for _ in range(args.iters):
            call()
        ev[1].record(stream)
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1]) / args.iters

    def device_case(boxes, count_only):
        off = np.zeros(len(boxes) + 1, np.uint64)
        ctx._check(mesh.overlap_boxes_rc(boxes, off), "vxb_mesh_overlap_box")
        total = int(off[-1])
        bt = torch.from_numpy(boxes.view(np.uint8).copy()).to(dev)
        ot = torch.empty((len(boxes) + 1) * 8, dtype=torch.uint8, device=dev)
        tt = torch.empty(max(total, 1) * 48, dtype=torch.uint8, device=dev)
        r = {"boxes": len(boxes), "triangles": total, "triangles_per_box": round(total / len(boxes), 2)}
        torch.cuda.synchronize()
        if count_only:
            ms = timed(lambda: mesh.overlap_boxes_device(bt.data_ptr(), len(boxes), ot.data_ptr(), None, 0))
            r["count_ms"] = round(ms, 4)
            r["boxes_per_s"] = round(len(boxes) / (ms * 1e-3), 0)
        ms = timed(lambda: mesh.overlap_boxes_device(bt.data_ptr(), len(boxes), ot.data_ptr(), tt.data_ptr(), total))
        got = ot.cpu().numpy().view(np.uint64)
        assert np.array_equal(got, off), "device offsets differ from the host variant's"
        r["fill_ms"] = round(ms, 4)
        r["triangles_per_s"] = round(total / (ms * 1e-3), 0)
        del bt, ot, tt
        torch.cuda.empty_cache()
        return r

    # (b) 2^20 body boxes; (c) navmesh tiles around the surface; (d) the whole grid
    bodies = body(args.boxes)
    out["body"] = device_case(bodies, True)
    surf = verts[rng.randint(0, len(verts), 4096)]
    lo = (np.floor(surf / 64.0) * 64.0).astype(np.float32)
    tiles = capi.make_boxes(lo, lo + 64)
    out["tiles"] = device_case(tiles, True)
    whole = capi.make_boxes([(-1, -1, -1)], [(n + 1, n + 1, n + 1)])
    out["whole_grid"] = device_case(whole, False)

    if args.verify:
        import overlap_oracle as oracle
        lv = oracle.Level0Sorted(res)
        ver = {}
        for what, boxes in (("body", bodies[rng.choice(len(bodies), 256, replace=False)]),
                            ("tiles", tiles[rng.choice(len(tiles), 16, replace=False)])):
            counts = []
            want = oracle.overlap_boxes(res, boxes, lv, counts=counts)
            got = mesh.overlap_boxes(boxes)
            c = np.array(counts, np.float64)
            ver[what] = {"boxes": len(boxes), "differ": oracle.same(got, want) is not None,
                         "oracle_blocks_per_box": round(float(c[:, 0].mean()), 2),
                         "oracle_triangles_per_box": round(float(c[:, 1].mean()), 1),
                         "triangles_per_box": round(float(got[0][-1]) / len(boxes), 2)}
        out["verify"] = ver
    mesh.close()
    ctx.close()
    print(json.dumps(out))
    if args.verify and any(v["differ"] for v in out["verify"].values()):
        sys.exit(1)


if __name__ == "__main__":
    main()
