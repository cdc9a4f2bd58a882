#!/usr/bin/env python
"""Summarises an `ncu --set full` report of one bench.py step: per launch a table row (markdown) and per kernel kind the
DRAM traffic (json, read by bench.py for `roofline.traffic`).

    ncu -i X.ncu-rep --page raw --csv > raw.csv ;  python tools/ncu_kernels.py raw.csv out_prefix "capture description" [first N launches]
"""
import csv
import json
import sys

KINDS = [("vxb_scan", "scan"), ("vxb_block_info", "select"), ("vxb_pyramid", "select"), ("vxb_select", "select"), ("vxb_plan", "select"),
         ("vxb_block_kernel<0", "block_level0"), ("vxb_block_kernel<1", "block_levels1plus"), ("vxb_block_kernel<2", "block_levels1plus"),
         ("vxb_classify", "classify"), ("vxb_big_block", "block_levels1plus"), ("vxb_mark_split", "select"), ("vxb_vertex", "vertex"),
         ("vxb_triangle", "triangle"), ("vxb_transition", "transition"), ("vxb_finish", "finish"), ("vxb_publish", "exchange")]
COLS = {"us": "gpu__time_duration.sum", "rd": "dram__bytes_read.sum", "wr": "dram__bytes_write.sum", "regs": "launch__registers_per_thread",
        "warps": "sm__warps_active.avg.pct_of_peak_sustained_active", "inst": "smsp__inst_executed.sum", "grid": "launch__grid_size",
        "ipc": "sm__inst_executed.avg.per_cycle_elapsed"}


def scale(value, unit, want):
    f = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "ns": 1e-3, "us": 1.0, "ms": 1e3, "usecond": 1.0, "nsecond": 1e-3, "msecond": 1e3}
    v = float(value.replace(",", "")) if value else 0.0
    return v * f.get(unit, 1.0)


def kernel_source_digest():
    import hashlib, os
    h = hashlib.sha256()
    d = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "voxels_b200", "csrc")
    for name in sorted(os.listdir(d)):
        if name.endswith((".cu", ".cuh", ".h")):
            h.update(open(os.path.join(d, name), "rb").read())
    return h.hexdigest()[:16]


def main(path, prefix, description, limit=None):
    rows = list(csv.reader(open(path)))
    if limit:
        rows = rows[:2 + limit]
    hdr, units = rows[0], rows[1]
    idx = {k: hdr.index(v) for k, v in COLS.items()}
    name_i = hdr.index("Kernel Name")
    per_kind, lines = {}, ["| # | kernel | grid | us | DRAM read MB | DRAM write MB | regs | warps active % | IPC | warp-instr (M) |", "|---|---|---|---|---|---|---|---|---|---|"]
    for n, r in enumerate(rows[2:]):
        name = r[name_i].split("(")[0]
        if name.startswith("void "):
            name = name[5:]
        name = name.replace(", ", ",")
        us = scale(r[idx["us"]], units[idx["us"]], "us")
        rd = scale(r[idx["rd"]], units[idx["rd"]], "byte")
        wr = scale(r[idx["wr"]], units[idx["wr"]], "byte")
        lines.append("| %d | %s | %s | %.1f | %.1f | %.1f | %s | %.1f | %.2f | %.1f |" % (n, name, r[idx["grid"]], us, rd / 1e6, wr / 1e6, r[idx["regs"]],
                                                                                 float(r[idx["warps"]] or 0), float(r[idx["ipc"]] or 0), float(r[idx["inst"]].replace(",", "") or 0) / 1e6))
        kind = next((k for p, k in KINDS if name.startswith(p)), None)
        if kind:
            e = per_kind.setdefault(kind, {"us": 0.0, "dram_read": 0.0, "dram_write": 0.0, "launches": 0})
            e["us"] += us; e["dram_read"] += rd; e["dram_write"] += wr; e["launches"] += 1
    open(prefix + "_kernels.md", "w").write("\n".join(lines) + "\n")
    step = {k: sum(e[k] for e in per_kind.values()) for k in ("us", "dram_read", "dram_write", "launches")}
    json.dump({"capture": description, "kernel_source_digest": kernel_source_digest(), "step": step, "per_kind": per_kind}, open(prefix + "_traffic.json", "w"), indent=1)
    total = sum(e["us"] for e in per_kind.values())
    print("serialised sum %.1f us; shares: %s" % (total, ", ".join("%s %.1f%%" % (k, 100 * e["us"] / total) for k, e in per_kind.items())))


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2], sys.argv[3] if len(sys.argv) > 3 else "", int(sys.argv[4]) if len(sys.argv) > 4 else None)
