#!/usr/bin/env python
"""The resident mesh (include/vxb200.h "mesh") against today's download path, in one process on one context.

Workload: an n^3 seeded terrain filled on the device (vxb_grid_fill), one full run, mesh.apply() (device time and bytes
copied), then K seeded sphere add / subtract edits from tools/bench_edits.py's generator.  Edits alternate between
    resident   vxb_grid_inject_surface -> vxb_polygonize_region -> vxb_mesh_apply -> vxb_mesh_select_lod   (nothing leaves HBM)
    download   vxb_grid_inject_surface -> vxb_polygonize_region -> vxb_result_download of the re-created blocks (pinned buffers)
timed per edit with the host clock, stage by stage (every stage ends in a device synchronise).  The download edits are
applied to the mesh too, untimed, so that it sees every run.  --verify keeps a host splice of every edit's re-created blocks
(erase the blocks in the dirty range, append the new ones: the drop-in's PolygonSurface) and compares it with the mesh.

    python tools/bench_resident.py [--size 1024] [--edits 1000] [--verify]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))

import numpy as np  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        name, power = (s.strip() for s in out.splitlines()[0].split(","))
        return name, power
    except Exception:
        return None, None


def stats_ms(xs):
    a = np.array(xs) * 1e3
    return {"mean": round(float(a.mean()), 4), "median": round(float(np.median(a)), 4), "p99": round(float(np.percentile(a, 99)), 4)} if len(a) else None


class HostSplice:
    """Per level the blocks in surface order: (id, coord_id, vertices, indices, trans vertices, trans indices)."""

    def __init__(self, levels):
        self.levels = [[] for _ in range(levels)]

    def take(self, res, region=None, n=0):
        for l in range(len(self.levels)):
            recs = res.records[res.records["level"] == l]
            if region is None:
                self.levels[l] = []
            else:
                m = 16 << l; nb = n // m
                lo, hi = np.array(region.min_dirty[l]), np.array(region.max_dirty[l])
                cid = np.array([b[1] for b in self.levels[l]], np.int64)
                mn = np.stack([cid % nb, cid // (nb * nb), (cid // nb) % nb], axis=1).astype(np.float64) * m   # output axes (x, z, y)
                erase = np.all((mn >= lo) & (mn < hi), axis=1) if len(cid) else np.zeros(0, bool)
                self.levels[l] = [b for b, e in zip(self.levels[l], erase) if not e]
            for r in recs:
                tv = [res.tverts[o:o + c].copy() for o, c in zip(r["trans_vertex_offset"], r["trans_vertex_count"])]
                ti = [res.tidx[o:o + c].copy() for o, c in zip(r["trans_index_offset"], r["trans_index_count"])]
                self.levels[l].append((int(r["id"]), int(r["coord_id"]), res.verts[r["vertex_offset"]:r["vertex_offset"] + r["vertex_count"]].copy(),
                                       res.idx[r["index_offset"]:r["index_offset"] + r["index_count"]].copy(), tv, ti))

    def mismatches(self, mesh_res):
        bad = 0
        for l, blocks in enumerate(self.levels):
            recs = mesh_res.records[mesh_res.records["level"] == l]
            if len(recs) != len(blocks):
                bad += 1
                continue
            for r, (bid, cid, v, i, tv, ti) in zip(recs, blocks):
                ok = int(r["id"]) == bid and int(r["coord_id"]) == cid
                ok = ok and mesh_res.verts[r["vertex_offset"]:r["vertex_offset"] + r["vertex_count"]].tobytes() == v.tobytes()
                ok = ok and np.array_equal(mesh_res.idx[r["index_offset"]:r["index_offset"] + r["index_count"]], i)
                for f in range(6):
                    ok = ok and mesh_res.tverts[r["trans_vertex_offset"][f]:r["trans_vertex_offset"][f] + r["trans_vertex_count"][f]].tobytes() == tv[f].tobytes()
                    ok = ok and np.array_equal(mesh_res.tidx[r["trans_index_offset"][f]:r["trans_index_offset"][f] + r["trans_index_count"][f]], ti[f])
                bad += 0 if ok else 1
        return bad


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--edits", type=int, default=1000)
    ap.add_argument("--verify", action="store_true", help="compare the mesh with a host splice of every edit's blocks at the end")
    args = ap.parse_args()
    import torch
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
    camera, base = (n * 0.5, n * 0.6, n * 0.5), 64.0

    # the first full run and apply load the kernels' modules: the second ones are timed
    mesh = ctx.mesh()
    ctx.polygonize()
    mesh.apply()
    t0 = time.perf_counter()
    info = ctx.polygonize()
    full_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    mi = mesh.apply()
    full_apply = {"device_ms": round(mi.apply_ms, 4), "host_ms": round(1e3 * (time.perf_counter() - t0), 4), "bytes_copied": mi.bytes_copied,
                  "blocks": mi.block_count, "gb_per_s": round(mi.bytes_copied / (mi.apply_ms * 1e-3) / 1e9, 1)}
    splice = None
    if args.verify:
        splice = HostSplice(info.levels_total)
        splice.take(ctx.download())

    pin = {"verts": torch.empty(64 << 20, dtype=torch.uint8).pin_memory(), "idx": torch.empty(32 << 20, dtype=torch.uint8).pin_memory(),
           "tverts": torch.empty(32 << 20, dtype=torch.uint8).pin_memory(), "tidx": torch.empty(16 << 20, dtype=torch.uint8).pin_memory()}
    into = {k: v.data_ptr() for k, v in pin.items()}
    lists = capi.DrawLists()
    cam = np.ascontiguousarray(camera, np.float32)
    res = {"total": [], "inject": [], "region": [], "apply": [], "select": [], "apply_device": [], "bytes": []}
    dl = {"total": [], "inject": [], "region": [], "download": []}
    blocks = 0
    for k, (pos, radius, extent, kind) in enumerate(edits):
        sphere = capi.Surface.sphere((0, 0, 0), radius)
        p32, e32 = np.array(pos, np.float32), np.full(3, extent, np.float32)
        t0 = time.perf_counter()
        box = ctx.inject_surface(p32, e32, sphere, kind)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        ri = ctx.polygonize_region(box[:3], box[3:])
        t2 = time.perf_counter()
        blocks += ri.block_count
        if k % 2 == 0:
            mi = mesh.apply()
            t3 = time.perf_counter()
            ctx._check(ctx.L.vxb_mesh_select_lod(mesh.h, capi._ptr(cam), base, C.byref(lists)), "vxb_mesh_select_lod")
            t4 = time.perf_counter()
            for key, v in (("total", t4 - t0), ("inject", t1 - t0), ("region", t2 - t1), ("apply", t3 - t2), ("select", t4 - t3)):
                res[key].append(v)
            res["apply_device"].append(mi.apply_ms * 1e-3); res["bytes"].append(mi.bytes_copied)
        else:
            ctx.download(into=into)
            t3 = time.perf_counter()
            for key, v in (("total", t3 - t0), ("inject", t1 - t0), ("region", t2 - t1), ("download", t3 - t2)):
                dl[key].append(v)
            mesh.apply()   # untimed: the mesh takes every run
        if splice is not None:
            splice.take(ctx.download(), ctx.region_info(), n)
    mi = mesh.info()
    out = {"metric": "ms per edit, resident mesh vs download of the re-created blocks (host clock, device-synchronised stages)",
           "config": {"workload": "%d^3 seeded terrain (vxb_grid_fill), %d sphere add/subtract edits (tools/bench_edits.py generator), "
                                  "edits alternating between the two paths" % (n, len(edits)), "camera": camera, "base_distance": base},
           "card": card()[0], "power_limit": card()[1],
           "full_run": {"polygonize_s": round(full_s, 4), "blocks": info.block_count, "mesh_apply": full_apply},
           "resident": {k: stats_ms(v) for k, v in res.items() if k != "bytes"},
           "resident_bytes_copied_per_edit": int(np.mean(res["bytes"])) if res["bytes"] else 0,
           "download": {k: stats_ms(v) for k, v in dl.items()},
           "blocks_recreated_per_edit": blocks / max(len(edits), 1),
           "mesh": {"blocks": mi.block_count, "compactions": mi.compactions, "growths": mi.growths, "generation": mi.generation,
                    "bytes": int(mi.vertex_span * 48 + mi.index_span * 4 + mi.trans_vertex_span * 48 + mi.trans_index_span * 4),
                    "live_bytes": int(mi.vertex_total * 48 + mi.index_total * 4 + mi.trans_vertex_total * 48 + mi.trans_index_total * 4),
                    "capacity_bytes": int(mi.capacity[0] * 48 + mi.capacity[1] * 4 + mi.capacity[2] * 48 + mi.capacity[3] * 4)}}
    if splice is not None:
        out["verify_mismatches"] = splice.mismatches(mesh.download())
    mesh.close()
    ctx.close()
    print(json.dumps(out))
    if splice is not None and out["verify_mismatches"]:
        sys.exit(1)


if __name__ == "__main__":
    main()
