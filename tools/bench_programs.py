#!/usr/bin/env python
"""SDF programs on the device grid store (include/vxb200.h vxb_grid_fill_program / vxb_grid_inject_program): one JSON line.

  sphere     fill of a one-op SPHERE program at n^3 next to vxb_grid_fill of the same built-in sphere (host clock, median)
  scene      fill of the 32-primitive scene (tests/programs.py: boxes, capsules, tori, smooth unions, a subtracted terrain
             cave) at n^3: fraction of blocks the interval pass writes as constants, pass A / pass B device time (CUDA events),
             and the 3 n^3 bytes written over the time of both passes against the H100's 3.35 TB/s
  edits      K box and capsule brush edits on a terrain grid (vxb_grid_inject_program) each followed by vxb_polygonize_region
             and the download of the re-created blocks; timed per edit as tools/bench_edits.py times its "device" column

    python tools/bench_programs.py [--size 1024] [--edit-size 512] [--edits 1000] [--repeat 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))

import numpy as np  # noqa: E402

HBM_TBPS = 3.35


def card():
    """(name, power limit in W) of GPU 0, read in this run."""
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, watts = [s.strip() for s in out.split(",")[:2]]
        return name, float(watts)
    except Exception:
        import torch
        return torch.cuda.get_device_name(0), None


def median_ms(fn, repeat):
    fn()  # warm-up (allocations, module load)
    times = []
    for _ in range(repeat):
        t0 = time.perf_counter()
        fn()
        times.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--edit-size", type=int, default=512)
    ap.add_argument("--edits", type=int, default=1000)
    ap.add_argument("--repeat", type=int, default=5)
    args = ap.parse_args()
    import torch
    import programs
    import voxels_b200
    from voxels_b200 import capi
    from voxels_b200.capi import Op
    name, watts = card()
    n = args.size
    ctx = voxels_b200.Context(0)
    out = {"metric": "SDF program fill / edits on the device grid store", "gpu": name, "power_limit_w": watts, "size": n}

    c = (n / 2, n / 2, n / 2)
    sphere_ms = median_ms(lambda: ctx.fill(n, capi.Surface.sphere(c, 0.3 * n, 1, 0)), args.repeat)
    program_ms = median_ms(lambda: ctx.fill_program(n, [Op.sphere(0.3 * n, at=c, material=1)]), args.repeat)
    st = ctx.program_stats()
    out["sphere"] = {"builtin_fill_ms": round(sphere_ms, 3), "program_fill_ms": round(program_ms, 3),
                     "culled_fraction": round(st.culled / st.blocks, 4), "pass_a_ms": round(st.pass_a_ms, 3), "pass_b_ms": round(st.pass_b_ms, 3)}

    ops, start, step = programs.scene(n)
    scene_ms = median_ms(lambda: ctx.fill_program(n, ops, start, step), args.repeat)
    passes = []
    for _ in range(args.repeat):
        ctx.fill_program(n, ops, start, step)
        s = ctx.program_stats()
        passes.append((s.pass_a_ms, s.pass_b_ms, s.culled, s.blocks))
    a_ms, b_ms = float(np.median([p[0] for p in passes])), float(np.median([p[1] for p in passes]))
    dev_ms = a_ms + b_ms
    out["scene"] = {"primitives": 32, "ops": len(ops), "fill_ms_host": round(scene_ms, 3), "culled_fraction": round(passes[0][2] / passes[0][3], 4),
                    "pass_a_ms": round(a_ms, 3), "pass_b_ms": round(b_ms, 3),
                    "write_tbps": round(3 * n ** 3 / (dev_ms * 1e-3) / 1e12, 3), "write_bound_ms": round(3 * n ** 3 / (HBM_TBPS * 1e12) * 1e3, 3)}
    out["scene"]["fraction_of_write_bound"] = round(out["scene"]["write_bound_ms"] / dev_ms, 3)
    ctx.close()

    # brush edits on a terrain grid, each followed by the incremental re-polygonization and its download
    m = args.edit_size
    ectx = voxels_b200.Context(0)
    ectx.fill(m, capi.Surface.terrain(m))
    ectx.polygonize()
    dist = ectx.download_dense()[0]
    rng = np.random.RandomState(42)
    edits = []
    while len(edits) < args.edits:
        x, y, z = (int(v) for v in rng.randint(32, m - 32, size=3))
        if abs(int(dist[z, y, x])) >= 4:
            continue
        r = float(rng.choice([4, 6, 8, 10]))
        rotation = programs.rot(int(rng.randint(3)), float(rng.uniform(0, 90)))
        brush = [Op.box((r, 0.7 * r, 0.5 * r), rotation=rotation)] if len(edits) % 2 == 0 else [Op.capsule(0.5 * r, r, rotation=rotation)]
        edits.append((np.array([x, y, z], np.float32), np.full(3, 2 * r + 4, np.float32), brush, 0 if (len(edits) // 2) % 2 == 0 else 2))
    pin = {"verts": torch.empty(64 << 20, dtype=torch.uint8).pin_memory(), "idx": torch.empty(32 << 20, dtype=torch.uint8).pin_memory(),
           "tverts": torch.empty(32 << 20, dtype=torch.uint8).pin_memory(), "tidx": torch.empty(16 << 20, dtype=torch.uint8).pin_memory()}
    into = {k: v.data_ptr() for k, v in pin.items()}
    acc = {"inject": 0.0, "polygonize": 0.0, "download": 0.0}
    blocks = 0
    for pos, ext, brush, kind in edits:
        t0 = time.perf_counter()
        box = ectx.inject_program(pos, ext, brush, kind)
        t1 = time.perf_counter()
        ectx.polygonize_region(box[:3], box[3:])
        t2 = time.perf_counter()
        part = ectx.download(into=into)
        t3 = time.perf_counter()
        acc["inject"] += t1 - t0; acc["polygonize"] += t2 - t1; acc["download"] += t3 - t2
        blocks += len(part.records)
    total = sum(acc.values())
    out["edits"] = {"grid": m, "count": len(edits), "edits_per_s": round(len(edits) / total, 1), "ms_per_edit": round(1e3 * total / len(edits), 3),
                    "blocks_recreated_per_edit": round(blocks / len(edits), 2),
                    "host_ms": {k: round(1e3 * v / len(edits), 3) for k, v in acc.items()},
                    "what": "vxb_grid_inject_program (box / capsule brush) + vxb_polygonize_region + vxb_result_download, host clock per edit"}
    ectx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
