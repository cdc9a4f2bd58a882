#!/usr/bin/env python
"""The LOD cut (include/vxb200.h "the LOD cut", vxb_mesh_select_cut) on an n^3 seeded terrain after one full run and apply.

One JSON line:
  select   latency of vxb_mesh_select_cut with 1, 4 and 8 views at lod_factor 2, 4 and 14.6: host clock around the call (it
           ends in a device synchronise), median and p99 over --calls calls
  orbit    tools/bench_cull.py's 64 camera positions (a circle, the eye 2 voxels above the surface, looking along the circle
           through a 90 x 60 degree frustum), per factor: regular draws per level and triangles per view, culled by that
           frustum and unculled (one pass-everything view), averaged over the orbit.  --verify checks every view against
           tests/cut_oracle.py
  cracks   the drawn triangles of the unculled cut at orbit camera 0, welded by exact float3 position, each vertex at the
           position the renderer contract selects (Rendering.md:48-54: the secondary position when its mask is non-zero
           and covered by the draw's block_adj); an edge used by exactly one triangle and not lying in a face of the grid
           box is a crack edge.  The same count for the all-level-0 draw (lod_factor 1e30) is the baseline.

    python tools/bench_cut.py [--size 1024] [--calls 1000] [--verify]
"""
import argparse
import json
import os
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FACTORS = (2.0, 4.0, 14.6)


def stats_ms(xs):
    import numpy as np
    a = np.array(xs) * 1e3
    return {"median": round(float(np.median(a)), 4), "p99": round(float(np.percentile(a, 99)), 4)}


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
    return [s.strip() for s in out.splitlines()[0].split(",")]


def crack_edges(res, lists, n):
    """(crack edges, welded triangles, degenerate triangles) of the draws in `lists` (the four arrays of one view)."""
    import numpy as np
    rc, ri, tc, ti = lists
    by_id = {int(i): k for k, i in enumerate(res.records["id"])}
    pos, tris = [], []
    base = 0
    for cmds, infos, verts, idx, trans in ((rc, ri, res.verts, res.idx, False), (tc, ti, res.tverts, res.tidx, True)):
        for c, inf in zip(cmds, infos):
            r = res.records[by_id[int(inf["block_id"])]]
            if trans:
                f = int(inf["face"])
                v = verts[r["trans_vertex_offset"][f]:r["trans_vertex_offset"][f] + r["trans_vertex_count"][f]]
            else:
                v = verts[r["vertex_offset"]:r["vertex_offset"] + r["vertex_count"]]
            mask = v["sec"][:, 3].view(np.uint32)
            adj = np.uint32(inf["block_adj"])
            use_sec = (mask != 0) & ((mask & adj) == mask)
            pos.append(np.where(use_sec[:, None], v["sec"][:, :3], v["pos"]))
            tris.append(idx[c["first_index"]:c["first_index"] + c["index_count"]].astype(np.int64).reshape(-1, 3) + base)
            base += len(v)
    if not tris:
        return 0, 0, 0
    pos = np.concatenate(pos).astype(np.float32)
    tris = np.concatenate(tris)
    _, weld = np.unique(np.ascontiguousarray(pos).view(np.dtype((np.void, 12))).ravel(), return_inverse=True)
    t = weld.ravel()[tris]
    degenerate = (t[:, 0] == t[:, 1]) | (t[:, 1] == t[:, 2]) | (t[:, 0] == t[:, 2])
    t = t[~degenerate]
    e = np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]])
    e.sort(axis=1)
    edges, count = np.unique(e, axis=0, return_counts=True)
    lone = edges[count == 1]
    # edges lying in a face of the grid box: both ends on the same boundary plane
    upos = np.zeros((weld.max() + 1, 3), np.float32)
    upos[weld.ravel()] = pos
    a, b = upos[lone[:, 0]], upos[lone[:, 1]]
    on_box = (((a == 0) & (b == 0)) | ((a == n) & (b == n))).any(axis=1)
    return int((~on_box).sum()), int(len(t)), int(degenerate.sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--calls", type=int, default=1000)
    ap.add_argument("--verify", action="store_true", help="check every view of the orbit against tests/cut_oracle.py")
    args = ap.parse_args()
    for p in (REPO, os.path.join(REPO, "tests")):
        if p not in sys.path:
            sys.path.insert(0, p)
    import numpy as np
    import voxels_b200
    from voxels_b200 import capi
    import cull_oracle
    import cut_oracle as oracle
    n = args.size
    name, power = card()
    out = {"metric": "LOD cut on the resident mesh (vxb_mesh_select_cut)", "card": name, "power_limit": power,
           "config": {"workload": "%d^3 seeded terrain (vxb_grid_fill), one full run and apply" % n}}
    ctx = voxels_b200.Context(0)
    ctx.fill(n, capi.Surface.terrain(n))
    ctx.polygonize()
    mesh = ctx.mesh()
    mi = mesh.apply()
    out["config"]["blocks"] = mi.block_count
    out["config"]["levels"] = mi.levels

    # ---- select latency ----
    cam = np.array([0.5 * n, 0.6 * n, 0.5 * n], np.float32)
    view = cull_oracle.perspective(cam, (1, -0.2, 0.4), (0, 1, 0), 90, 60, 0.5, 2.0 * n)
    lists = (capi.DrawLists * capi.VXB_VIEWS_MAX)()
    sel = {}
    for factor in FACTORS:
        for count in (1, 4, 8):
            views = capi.make_views(np.stack([view] * count))
            call = lambda: ctx._check(ctx.L.vxb_mesh_select_cut(mesh.h, capi._ptr(cam), factor, views, count, lists), "vxb_mesh_select_cut")
            for _ in range(20):
                call()
            ts = []
            for _ in range(args.calls):
                t0 = time.perf_counter()
                call()
                ts.append(time.perf_counter() - t0)
            sel["factor_%g_views_%d" % (factor, count)] = stats_ms(ts)
    out["select_ms"] = dict(sel, calls=args.calls)

    # ---- the orbit ----
    res = mesh.download() if args.verify else None
    boxes = cull_oracle.block_boxes(res) if args.verify else None
    mismatches = 0
    positions = 64
    orbit = {}
    eyes = []
    for k in range(positions):
        a = 2 * np.pi * k / positions
        x, z = 0.5 * n + 0.25 * n * np.cos(a), 0.5 * n + 0.25 * n * np.sin(a)
        hit = mesh.raycast(capi.make_rays([(x, n + 8.0, z)], [(0, -1, 0)]))
        eye = (x, (hit["position"][0][1] if hit["slot"][0] != capi.VXB_RAY_MISS else 0.5 * n) + 2.0, z)
        eyes.append((eye, cull_oracle.perspective(eye, (-np.sin(a), 0, np.cos(a)), (0, 1, 0), 90, 60, 0.5, 2.0 * n)))
    for factor in FACTORS:
        per_level = {"culled": np.zeros(mi.levels, np.int64), "unculled": np.zeros(mi.levels, np.int64)}
        tri = {"culled": 0, "unculled": 0}
        trans = {"culled": 0, "unculled": 0}
        smaller = 0
        for eye, v in eyes:
            got = mesh.select_cut(eye, factor, np.stack([v, cull_oracle.PASS_ALL]))
            for kind, g in zip(("culled", "unculled"), got):
                per_level[kind] += np.bincount(g[1]["level"].astype(np.int64), minlength=mi.levels)[:mi.levels]
                tri[kind] += (int(g[0]["index_count"].sum()) + int(g[2]["index_count"].sum())) // 3
                trans[kind] += len(g[2])
            smaller += len(got[0][0]) < len(got[1][0])
            if args.verify:
                want = oracle.expected_draws(res.records, boxes, n, res.info.levels, eye, factor, [v, cull_oracle.PASS_ALL])
                mismatches += sum(oracle.draw_sets(g) != w for g, w in zip(got, want))
        orbit["factor_%g" % factor] = {
            kind: {"regular_per_level": [round(float(x) / positions, 1) for x in per_level[kind]],
                   "transition_draws": round(trans[kind] / positions, 1), "triangles": round(tri[kind] / positions)}
            for kind in ("culled", "unculled")}
        orbit["factor_%g" % factor]["cameras_with_fewer_culled_draws"] = smaller
    out["orbit"] = dict(orbit, positions=positions, frustum="90 x 60 degrees, near 0.5, far %d" % (2 * n), per="view, averaged over the orbit")
    if args.verify:
        out["verify_views"] = positions * len(FACTORS) * 2
        out["verify_mismatches"] = int(mismatches)

    # ---- cracks ----
    res = res if res is not None else mesh.download()
    eye = eyes[0][0]
    cracks = {}
    for label, factor in (("cut_14.6", 14.6), ("cut_4", 4.0), ("cut_2", 2.0), ("all_level0", 1e30)):
        edges, tris, degenerate = crack_edges(res, mesh.select_cut(eye, factor, cull_oracle.PASS_ALL[None])[0], n)
        cracks[label] = {"crack_edges": edges, "triangles": tris, "degenerate_skipped": degenerate}
    out["cracks"] = dict(cracks, camera=[round(float(c), 2) for c in eye])
    mesh.close()
    ctx.close()
    print(json.dumps(out))
    if args.verify and mismatches:
        sys.exit(1)


if __name__ == "__main__":
    main()
