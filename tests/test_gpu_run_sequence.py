"""The launch sequence of a run: how many kernels each kind of run launches, that every launch path (a captured graph,
its replay, plain launches on one stream with per-kernel timing, plain launches with VXB200_NO_GRAPH) computes the same
result, and that a context gives back all device memory when it is destroyed.

The launch counts are what bench.py reports as `launches_per_step` and as the per-kind `launches` of its roofline
table.  They were recorded from the launch sequence as it stood before its host code was restructured; a change to
them is a change to the sequence and has to be deliberate."""
import os

import numpy as np
import pytest

import compare
import grids

pytestmark = pytest.mark.gpu

KINDS = 10


def _terrain(n):
    import torch
    from voxels_b200 import synth
    grid = synth.terrain(n, torch.device("cuda", 0))
    torch.cuda.synchronize()
    return grid


def _context(grid=None, limit=0):
    import voxels_b200
    ctx = voxels_b200.Context(0)
    ctx.set_materials(None, None)
    ctx.set_launch_limit(limit)
    if grid is not None:
        d, m, b = grid
        ctx.set_device_grid(d.shape[0], d.data_ptr(), m.data_ptr(), b.data_ptr(), keep=grid)
    return ctx


def _kinds(ctx):
    return [ctx.kernel_ms(k)[1] for k in range(KINDS)]


def _full_run_counts(ctx, run):
    """(total, per-kind) launches of a captured run, its replay and a VXB_FLAG_KERNEL_TIMES run of `run(flags)`."""
    import voxels_b200
    out = {}
    for name, flags in (("captured", 0), ("replayed", 0), ("timed", voxels_b200.FLAG_KERNEL_TIMES)):
        run(flags)
        out[name] = [ctx.info().kernel_launches, _kinds(ctx)]
    return out


def _virtual_rank_counts(contexts):
    """Phases 0, 1 and 2 of two virtual ranks: per rank, the total after phase 2 and the per-kind launches summed over
    the three phases."""
    import torch
    from test_gpu_sharded import _view, configure_virtual_ranks
    bufs = configure_virtual_ranks(contexts)
    kinds = [[0] * KINDS for _ in contexts]

    def phase(p):
        for r, c in enumerate(contexts):
            assert c.polygonize_sharded(p) == 0
            kinds[r] = [a + b for a, b in zip(kinds[r], _kinds(c))]
        torch.cuda.synchronize()

    phase(0)
    chunk = bufs[0].chunk_bytes
    views = [_view(b.block_info, b.block_info_bytes) for b in bufs]
    for src in range(len(contexts)):
        for dst in range(len(contexts)):
            if src != dst:
                views[dst][src * chunk:(src + 1) * chunk].copy_(views[src][src * chunk:(src + 1) * chunk])
    torch.cuda.synchronize()
    phase(1)
    phase(2)
    return {"rank%d" % r: [c.info().kernel_launches, kinds[r]] for r, c in enumerate(contexts)}


def measure(case):
    """The launch counts of one kind of run, by name (see EXPECTED)."""
    import voxels_b200
    sizes = {"full64": 64, "full256": 256, "full1024": 1024}
    grid = _terrain(sizes.get(case, 256))
    if case == "ranks2":
        contexts = [_context(grid) for _ in range(2)]
        try:
            return _virtual_rank_counts(contexts)
        finally:
            for c in contexts:
                c.close()
    ctx = _context(grid, limit=2 if case == "limit2" else 0)
    try:
        if case in sizes or case == "limit2":
            return _full_run_counts(ctx, lambda flags: ctx.polygonize(0, flags))
        if case == "levels2":
            return _full_run_counts(ctx, lambda flags: ctx.polygonize(2, flags))
        if case == "no_transitions":
            return _full_run_counts(ctx, lambda flags: ctx.polygonize(0, flags | voxels_b200.FLAG_NO_TRANSITIONS))
        if case == "phase3":
            ctx.shard_configure(0, 1)
            return _full_run_counts(ctx, lambda flags: ctx.polygonize_sharded(3, flags))
        if case == "region":
            ctx.polygonize()
            out = {}
            for name, flags in (("plain", 0), ("timed", voxels_b200.FLAG_KERNEL_TIMES)):
                ctx.polygonize_region((100, 90, 80), (140, 130, 120), flags)
                out[name] = [ctx.info().kernel_launches, _kinds(ctx)]
            return out
        raise KeyError(case)
    finally:
        ctx.close()


# case -> run -> [kernel_launches, launches of kinds 0..9]
EXPECTED = {
    "full64": {"captured": [16, [1, 5, 3, 1, 1, 1, 2, 1, 0, 0]], "timed": [16, [1, 5, 3, 1, 1, 1, 2, 1, 0, 0]]},
    "full256": {"captured": [17, [1, 6, 3, 1, 1, 1, 2, 1, 0, 0]], "timed": [17, [1, 6, 3, 1, 1, 1, 2, 1, 0, 0]]},
    "full1024": {"captured": [19, [1, 7, 4, 1, 1, 1, 2, 1, 0, 0]], "timed": [19, [1, 7, 4, 1, 1, 1, 2, 1, 0, 0]]},
    "levels2": {"captured": [15, [1, 5, 2, 1, 1, 1, 2, 1, 0, 0]], "timed": [15, [1, 5, 2, 1, 1, 1, 2, 1, 0, 0]]},
    "no_transitions": {"captured": [15, [1, 6, 3, 1, 1, 1, 0, 1, 0, 0]], "timed": [15, [1, 6, 3, 1, 1, 1, 0, 1, 0, 0]]},
    "region": {"plain": [17, [1, 6, 3, 1, 1, 1, 2, 1, 0, 0]], "timed": [17, [1, 6, 3, 1, 1, 1, 2, 1, 0, 0]]},
    "limit2": {"captured": [17, [1, 6, 3, 1, 1, 1, 2, 1, 0, 0]], "timed": [17, [1, 6, 3, 1, 1, 1, 2, 1, 0, 0]]},
    "ranks2": {"rank0": [19, [1, 7, 3, 1, 1, 1, 2, 1, 0, 1]], "rank1": [19, [1, 7, 3, 1, 1, 1, 2, 1, 0, 1]]},
    "phase3": {"captured": [18, [1, 7, 3, 1, 1, 1, 2, 1, 0, 0]], "timed": [18, [1, 7, 3, 1, 1, 1, 2, 1, 0, 0]]},
}


@pytest.mark.parametrize("case", ["full64", "full256", "full1024", "levels2", "no_transitions", "region", "limit2",
                                  "ranks2", "phase3"])
def test_launch_counts(case):
    got = measure(case)
    replayed = got.pop("replayed", None)
    assert got == EXPECTED[case]
    if replayed is not None:
        # a replay reports the launches of the run it replays, per kind too
        assert replayed == got["captured"]


def _snapshot(ctx):
    """The result of the context's last run: its info (without the device time) and the digests of every level's blocks,
    vertices and indices in block order (where a block's data sits in the arenas depends on the order the CTAs ran)."""
    import golden_hash
    info = ctx.info()
    fields = {}
    for name, _ in info._fields_:
        if name != "device_ms":
            v = getattr(info, name)
            fields[name] = list(v) if hasattr(v, "__len__") else v
    res = ctx.download()
    return fields, [golden_hash.level_digests(res.level(l)) for l in range(info.levels_total)]


@pytest.mark.parametrize("name,limit", [("hostile128", 0), ("patchwork256", 2), ("terrain512", 0)])
def test_launch_paths_same_result(name, limit):
    import torch
    import voxels_b200
    if name == "terrain512":
        grid = _terrain(512)
    else:
        grid = tuple(torch.from_numpy(a).cuda() for a in grids.by_name(name))
        torch.cuda.synchronize()
    ctx = _context(grid, limit)
    os.environ["VXB200_NO_GRAPH"] = "1"
    try:
        plain = _context(grid, limit)
    finally:
        del os.environ["VXB200_NO_GRAPH"]
    try:
        ctx.polygonize()
        captured = _snapshot(ctx)
        ctx.polygonize()
        replayed = _snapshot(ctx)
        ctx.polygonize(0, voxels_b200.FLAG_KERNEL_TIMES)
        timed = _snapshot(ctx)
        plain.polygonize()
        ungraphed = _snapshot(plain)
        assert replayed == captured
        assert timed == captured
        assert ungraphed == captured
    finally:
        ctx.close()
        plain.close()


def test_phase3_at_world1_equals_polygonize():
    grid = _terrain(256)
    single, sharded = _context(grid), _context(grid)
    try:
        info = single.polygonize()
        want = single.download()
        sharded.shard_configure(0, 1)
        assert sharded.polygonize_sharded(3) == 0
        got = sharded.download()
        problems = []
        for l in range(info.levels_total):
            problems += compare.level_diff(want.level(l), got.level(l), "L%d" % l)
        if not np.array_equal(want.stats, got.stats):
            problems.append("stats differ: %s vs %s" % (want.stats, got.stats))
        assert not problems, "\n".join(problems[:10])
    finally:
        single.close()
        sharded.close()


def test_destroy_frees_device_memory():
    """create -> fill -> polygonize -> mesh apply -> region edit -> destroy, ten times: after the first round, which
    may leave lazily created driver state behind, free device memory returns to the same value every round.  Within one
    2 MiB allocation granule: this catches a large buffer left behind, or a small one left behind every round, not a
    single small one."""
    import torch
    import voxels_b200
    from voxels_b200 import capi
    granule = 2 << 20
    free = []
    for _ in range(10):
        ctx = voxels_b200.Context(0)
        ctx.fill(128, capi.Surface.terrain(128))
        ctx.polygonize()
        mesh = ctx.mesh()
        mesh.apply()
        box = ctx.inject_surface((60, 60, 60), (20, 20, 20), capi.Surface.sphere((0, 0, 0), 8), 0)
        ctx.polygonize_region(box[:3], box[3:])
        mesh.apply()
        ctx.close()
        torch.cuda.synchronize()
        free.append(torch.cuda.mem_get_info()[0])
    assert max(free[1:]) - min(free[1:]) <= granule, free
