#!/usr/bin/env python
"""The mesh's bounds and the culled select (include/vxb200.h "bounds and the culled select") on an n^3 seeded terrain.

Three measurements, one JSON line:
  apply    what the bounds add to vxb_mesh_apply: the device time (vxb_mesh_info.apply_ms) of a full apply and of the
           per-edit apply of tools/bench_resident.py's edit loop, --runs processes of this build alternated with as many of
           another build (--against DIR: a directory that holds that build's voxels_b200 package with its library)
  select   the latency of vxb_mesh_select_lod and of vxb_mesh_select_lod_views with 1, 4 and 8 views: host clock around the
           call (it ends in a device synchronise), median and p99 over --calls calls
  orbit    what culling buys: 64 camera positions on a circle, the eye 2 voxels above the surface, looking along the circle
           through a 90 x 60 degree frustum; regular and transition draws and indexed triangles of the culled lists against
           the unculled cut.  --verify checks every view of the orbit against tests/cull_oracle.py, and reports how many
           blocks' boxes exceed their lattice box and what culling by the lattice boxes would have kept.

    python tools/bench_cull.py [--size 1024] [--edits 200] [--runs 3] [--against DIR] [--calls 1000] [--verify]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def apply_child(args):
    """One process of the apply comparison, on the package found first on sys.path; prints one JSON line."""
    import numpy as np
    import voxels_b200
    from voxels_b200 import capi
    from bench_edits import edit_sequence
    n = args.size
    ctx = voxels_b200.Context(0)
    ctx.fill(n, capi.Surface.terrain(n))
    dist = np.empty((n, n, n), np.int8)
    ctx._check(ctx.L.vxb_grid_download_dense(ctx.h, capi._ptr(dist), None, None), "vxb_grid_download_dense")
    edits = edit_sequence(n, args.edits, dist)
    del dist
    mesh = ctx.mesh()
    full = []
    for _ in range(6):                       # the first run and apply load the kernels' modules
        ctx.polygonize()
        full.append(mesh.apply().apply_ms)
    info = mesh.info()
    device, host = [], []
    for pos, radius, extent, kind in edits:
        box = ctx.inject_surface(np.array(pos, np.float32), np.full(3, extent, np.float32), capi.Surface.sphere((0, 0, 0), radius), kind)
        ctx.polygonize_region(box[:3], box[3:])
        t0 = time.perf_counter()
        mi = mesh.apply()
        host.append(1e3 * (time.perf_counter() - t0))
        device.append(mi.apply_ms)
    print(json.dumps({"library": os.path.relpath(capi.library_path(), REPO), "blocks": info.block_count, "full_bytes_copied": info.bytes_copied,
                      "full_apply_ms": [round(x, 4) for x in full[1:]], "full_apply_ms_median": round(float(np.median(full[1:])), 4),
                      "edit_apply_device_ms_median": round(float(np.median(device)), 4), "edit_apply_device_ms_mean": round(float(np.mean(device)), 4),
                      "edit_apply_host_ms_median": round(float(np.median(host)), 4)}))
    mesh.close()
    ctx.close()


def compare_applies(args):
    roots = [("this", REPO)] + ([("other", os.path.abspath(args.against))] if args.against else [])
    out = {name: [] for name, _ in roots}
    for _ in range(args.runs):
        for name, root in roots:           # alternated: both builds see the same drift of the machine
            env = dict(os.environ, PYTHONPATH=os.pathsep.join([root, os.path.join(REPO, "tools")]))
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--apply-child", "--size", str(args.size), "--edits", str(args.edits)],
                               env=env, capture_output=True, text=True, cwd=os.path.join(REPO, "tools"))
            if r.returncode != 0:
                raise RuntimeError("apply run of %s failed:\n%s" % (root, r.stderr[-2000:]))
            out[name].append(json.loads(r.stdout.strip().splitlines()[-1]))
    return out


def stats_ms(xs):
    import numpy as np
    a = np.array(xs) * 1e3
    return {"median": round(float(np.median(a)), 4), "p99": round(float(np.percentile(a, 99)), 4)}


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
    return [s.strip() for s in out.splitlines()[0].split(",")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--edits", type=int, default=200, help="edits of each apply run")
    ap.add_argument("--runs", type=int, default=3, help="apply runs per build")
    ap.add_argument("--against", help="directory holding another build's voxels_b200 package, for the apply comparison")
    ap.add_argument("--calls", type=int, default=1000)
    ap.add_argument("--verify", action="store_true", help="check every view of the orbit against tests/cull_oracle.py")
    ap.add_argument("--apply-child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.apply_child:
        return apply_child(args)
    for p in (REPO, os.path.join(REPO, "tests"), os.path.join(REPO, "tools")):
        if p not in sys.path:
            sys.path.insert(0, p)
    import numpy as np
    import voxels_b200
    from voxels_b200 import capi
    import cull_oracle as oracle
    n = args.size
    name, power = card()
    out = {"metric": "bounds and culled select on the resident mesh", "card": name, "power_limit": power,
           "config": {"workload": "%d^3 seeded terrain (vxb_grid_fill), one full run and apply" % n, "base_distance": 64.0}}
    out["apply"] = compare_applies(args)

    ctx = voxels_b200.Context(0)
    ctx.fill(n, capi.Surface.terrain(n))
    ctx.polygonize()
    mesh = ctx.mesh()
    mi = mesh.apply()
    out["config"]["blocks"] = mi.block_count
    base = 64.0

    # ---- select latency ----
    cam = np.array([0.5 * n, 0.6 * n, 0.5 * n], np.float32)
    view = oracle.perspective(cam, (1, -0.2, 0.4), (0, 1, 0), 90, 60, 0.5, 2.0 * n)
    lists = (capi.DrawLists * capi.VXB_VIEWS_MAX)()
    sel = {}

    def timed(call):
        for _ in range(20):
            call()
        ts = []
        for _ in range(args.calls):
            t0 = time.perf_counter()
            call()
            ts.append(time.perf_counter() - t0)
        return stats_ms(ts)

    sel["select_lod"] = timed(lambda: ctx._check(ctx.L.vxb_mesh_select_lod(mesh.h, capi._ptr(cam), base, C.byref(lists[0])), "vxb_mesh_select_lod"))
    for count in (1, 4, 8):
        views = capi.make_views(np.stack([view] * count))
        sel["select_lod_views_%d" % count] = timed(
            lambda: ctx._check(ctx.L.vxb_mesh_select_lod_views(mesh.h, capi._ptr(cam), base, views, count, lists), "vxb_mesh_select_lod_views"))
    out["select_ms"] = dict(sel, calls=args.calls)

    # ---- the orbit ----
    res = boxes = lattice = None
    lattice_regular = 0
    if args.verify:
        res = mesh.download()
        boxes = oracle.block_boxes(res)
        lattice = oracle.lattice_boxes(res.records, n)
        out["blocks_outside_their_lattice_box"] = int(((boxes[:, :3] < lattice[:, :3]).any(axis=1) | (boxes[:, 3:] > lattice[:, 3:]).any(axis=1)).sum())
    tot = {k: 0 for k in ("regular", "transition", "triangles", "culled_regular", "culled_transition", "culled_triangles")}
    mismatches = 0
    positions = 64
    for k in range(positions):
        a = 2 * np.pi * k / positions
        x, z = 0.5 * n + 0.25 * n * np.cos(a), 0.5 * n + 0.25 * n * np.sin(a)
        hit = mesh.raycast(capi.make_rays([(x, n + 8.0, z)], [(0, -1, 0)]))
        eye = (x, (hit["position"][0][1] if hit["slot"][0] != capi.VXB_RAY_MISS else 0.5 * n) + 2.0, z)
        v = oracle.perspective(eye, (-np.sin(a), 0, np.cos(a)), (0, 1, 0), 90, 60, 0.5, 2.0 * n)
        rc, _, tc, _ = mesh.select_lod(eye, base)
        got = mesh.select_lod_views(eye, base, v[None])[0]
        tot["regular"] += len(rc); tot["transition"] += len(tc)
        tot["triangles"] += (int(rc["index_count"].sum()) + int(tc["index_count"].sum())) // 3
        tot["culled_regular"] += len(got[0]); tot["culled_transition"] += len(got[2])
        tot["culled_triangles"] += (int(got[0]["index_count"].sum()) + int(got[2]["index_count"].sum())) // 3
        if args.verify:
            want = oracle.expected_draws(res.records, boxes, n, res.info.levels, eye, base, [v])[0]
            mismatches += 0 if oracle.draw_sets(got) == want else 1
            lattice_regular += len(oracle.expected_draws(res.records, lattice, n, res.info.levels, eye, base, [v])[0][0])
    out["orbit"] = dict(tot, positions=positions, frustum="90 x 60 degrees, near 0.5, far %d" % (2 * n),
                        draws_kept=round((tot["culled_regular"] + tot["culled_transition"]) / max(tot["regular"] + tot["transition"], 1), 4),
                        triangles_kept=round(tot["culled_triangles"] / max(tot["triangles"], 1), 4))
    if args.verify:
        out["verify_mismatches"] = mismatches
        out["orbit"]["regular_kept_by_lattice_boxes"] = lattice_regular   # what the block lattice boxes would have drawn
    mesh.close()
    ctx.close()
    print(json.dumps(out))
    if args.verify and mismatches:
        sys.exit(1)


if __name__ == "__main__":
    main()
