"""SDF programs on the device (vxb_grid_fill_program / vxb_grid_inject_program) against the UNMODIFIED reference grid store
fed the same program through its VoxelSurface callback (tests/harness/vxh_programs.cpp: ProgramSurface), byte for byte:
  fill_program      == Grid::Create(n, n, n, start, step, &program)       at 64^3 / 128^3, and the host generator at 512^3
  one-op programs   == vxb_grid_fill of the built-in surface
  inject_program    == Grid::InjectSurface(..., &program) + the returned box, then vxb_polygonize_region == incremental Execute
  malformed programs are refused and leave the grid as it was; cube pieces of two virtual ranks merge into the whole fill."""
import numpy as np
import pytest

import programs
from test_gpu_gridstore import _device_edits, assert_dense_equal
from test_programs_cpu import MALFORMED, malformed
from voxels_b200 import capi
from voxels_b200.capi import Op

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def reference():
    """The unmodified reference with the SDF-program calls (oracle/_ref/libvxh_programs_ref.so, built by oracle/programs.mk
    from tests/harness/vxh_capi.cpp + vxh_programs.cpp): every call of the conftest's reference plus the program ones."""
    import program_harness
    lib = program_harness.load()
    if lib is None:
        pytest.skip("oracle/_ref/libvxh_programs_ref.so not built (needs the reference checkout: make -C oracle -f programs.mk programs)")
    return lib


def _equal(want, got, what):
    for a, b, ch in zip(want, got, ("distance", "material", "blend")):
        if not np.array_equal(a, b):
            bad = np.argwhere(a != b)
            raise AssertionError("%s %s differs at %d voxels, first (z,y,x)=%s: want %d, device %d"
                                 % (what, ch, len(bad), bad[0], a[tuple(bad[0])], b[tuple(bad[0])]))


@pytest.mark.parametrize("name", sorted(programs.SMALL))
@pytest.mark.parametrize("n", [64, 128])
def test_fill_program_equals_reference_constructor(reference, gpu_context, name, n):
    ops, start, step = programs.SMALL[name](n)
    g = reference.grid_create_program(n, ops, start, step)
    gpu_context.fill_program(n, ops, start, step)
    assert_dense_equal(reference, g, gpu_context, "fill_program %s" % name)
    reference.grid_destroy(g)


@pytest.mark.parametrize("name", ["scene", "margin", "margin_past"])
def test_fill_program_512_equals_host_generator(reference, gpu_context, name):
    """The cull path at scale: bytes, not counts; and the device's cull count equals the host's decision."""
    n = 512
    ops, start, step = programs.scene(n) if name == "scene" else programs.SMALL[name](n)
    gpu_context.fill_program(n, ops, start, step)
    _equal(reference.program_dense(n, ops, start, step), gpu_context.download_dense(), name)
    flags, _ = reference.program_cull_flags(n, ops, start, step)
    st = gpu_context.program_stats()
    assert st.blocks == (n // 16) ** 3 and st.culled == int(flags.sum())
    if name == "scene":
        assert st.culled > st.blocks // 2


@pytest.mark.parametrize("surface,op", [
    (capi.Surface.sphere((30.5, 20.25, 33.0), 17.5, 3, 40), Op.sphere(17.5, at=(30.5, 20.25, 33.0), material=3, blend=40)),
    (capi.Surface.plane((0.37, 0.61, 0.7), 40.25, 1, 200), Op.plane((0.37, 0.61, 0.7), 40.25, material=1, blend=200)),
    (capi.Surface.terrain(128, origin=(100, 7), seed=99), Op.terrain(128, origin=(100, 7), seed=99)),
])
def test_one_op_program_equals_builtin_fill(gpu_context, surface, op):
    n = 128
    gpu_context.fill(n, surface)
    want = gpu_context.download_dense()
    gpu_context.fill_program(n, [op])
    _equal(want, gpu_context.download_dense(), "one-op %d" % op.code)


def _brushes(n, count, seed):
    rng = np.random.RandomState(seed)
    out = []
    for i in range(count):
        r = float(rng.choice([3, 4, 6]))
        kind = i % 4
        rotation = programs.rot(int(rng.randint(3)), float(rng.uniform(0, 90)))
        if kind == 0:
            ops = [Op.box((r, 0.7 * r, 0.5 * r), rotation=rotation)]
        elif kind == 1:
            ops = [Op.capsule(0.5 * r, r, rotation=rotation)]
        elif kind == 2:
            ops = [Op.torus(r, 0.4 * r, rotation=rotation)]
        else:
            ops = [Op.sphere(0.7 * r, at=(-0.5 * r, 0.0, 0.0)), Op.box((0.5 * r, 0.5 * r, 0.5 * r), at=(0.5 * r, 0.25, 0.0)),
                   Op.smooth_union(1.5)]
        if i % 5 == 4:   # fractional centre and odd extents
            pos = rng.uniform(8, n - 8, size=3).round(2)
            ext = np.array([2 * r + 3, 2 * r + 5, 2 * r + 1], np.float32)
        else:
            pos = rng.randint(4, n - 4, size=3).astype(np.float32)
            ext = np.full(3, 2 * r + 4, np.float32)
        if i % 7 == 6:   # hanging over the grid edge
            pos[rng.randint(3)] = rng.choice([1.0, n - 2.0])
        out.append((pos.astype(np.float32), ext, ops, i % 3))
    return out


def test_inject_program_equals_reference(reference, gpu_context):
    n = 64
    s = capi.Surface.terrain(n)
    g = reference.grid_create_builtin(n, s)
    gpu_context.fill(n, s)
    for i, (pos, ext, ops, kind) in enumerate(_brushes(n, 40, 5)):
        want_box = reference.grid_inject_program(g, pos, ext, ops, kind)
        got_box = gpu_context.inject_program(pos, ext, ops, kind)
        assert np.array_equal(want_box, got_box), "edit %d: returned box %s vs %s" % (i, want_box, got_box)
        assert_dense_equal(reference, g, gpu_context, "edit %d (pos %s ext %s type %d)" % (i, pos, ext, kind))
    reference.grid_destroy(g)


class _ProgramBrush:
    """Adapts a program to the (reference, device) inject calls _device_edits makes with a built-in surface."""

    def __init__(self, ops):
        self.ops = ops


def test_program_edits_then_incremental_polygonize_match_reference(reference, gpu_context, monkeypatch):
    """Program brushes on a program-filled grid, each followed by vxb_polygonize_region, against InjectSurface +
    the reference's incremental Execute (as test_device_edits_then_incremental_polygonize_match_reference)."""
    n = 128
    ctx = gpu_context
    ctx.set_materials(None, None)
    ops, start, step = programs.terrain_cave(n)
    g = reference.grid_create_program(n, ops, start, step)
    ctx.fill_program(n, ops, start, step)
    surf, _ = reference.polygonize(g)
    mod = reference.modification_create()
    ctx.polygonize()
    dist0 = reference.grid_to_dense(g)[0]
    rng = np.random.RandomState(3)
    edits = []
    brushes = _brushes(n, 60, 9)
    while len(edits) < 20:
        x, y, z = (int(v) for v in rng.randint(16, n - 16, size=3))
        if abs(int(dist0[z, y, x])) >= 4:
            continue
        _, ext, bops, _ = brushes[len(edits)]
        edits.append((np.array([x, y, z], np.float32), ext, _ProgramBrush(bops), len(edits) % 3))
    monkeypatch.setattr(reference, "grid_inject_builtin", lambda grid, p, e, b, k: reference.grid_inject_program(grid, p, e, b.ops, k), raising=False)
    monkeypatch.setattr(ctx, "inject_surface", lambda p, e, b, k: ctx.inject_program(p, e, b.ops, k), raising=False)
    _device_edits(reference, ctx, g, surf, mod, edits)


@pytest.mark.parametrize("case", MALFORMED)
def test_malformed_program_is_refused_and_leaves_the_grid(gpu_context, case):
    n = 64
    gpu_context.fill_program(n, programs.union_box_sphere(n)[0])
    before = gpu_context.download_dense()
    ops = malformed(case)
    for call in (lambda: gpu_context.fill_program(n, ops), lambda: gpu_context.inject_program((32, 32, 32), (12, 12, 12), ops, 0)):
        with pytest.raises(capi.VxbError) as e:
            call()
        assert "(-2)" in str(e.value) and " op " in str(e.value), str(e.value)
    _equal(before, gpu_context.download_dense(), "after refusing " + case)


def test_cube_pieces_of_two_ranks_merge_into_the_fill(gpu_context):
    """Cube mode, virtual ranks (world 2): each rank's fill_program writes the pieces it backs; together they are the fill."""
    import os
    import torch
    import voxels_b200
    from voxels_b200.dist import owned_pieces
    n, world, group = 256, 2, 32
    ops, start, step = programs.terrain_cave(n)
    gpu_context.fill_program(n, ops, start, step)
    want = gpu_context.download_dense()
    contexts = [voxels_b200.Context(0) for _ in range(world)]
    try:
        for r, c in enumerate(contexts):
            c.cube_create(n, r, world, group)
        channels = contexts[0].cube_info()[1]
        for r, c in enumerate(contexts):
            for p, _, _ in owned_pieces(n, r, world, group):
                for ch in range(channels):
                    fd = c.cube_export(ch, p)
                    for q, peer in enumerate(contexts):
                        if q != r:
                            peer.cube_import(ch, p, fd)
                    os.close(fd)
        for c in contexts:
            c.fill_program(n, ops, start, step)
        torch.cuda.synchronize()
        for r, c in enumerate(contexts):
            for p, z0, z1 in owned_pieces(n, r, world, group):
                pd, pm, pbl, size = contexts[1 - r].cube_piece(p)   # read through the peer's mapping
                for ptr, vol in ((pd, want[0]), (pm, want[1]), (pbl, want[2])):
                    got = torch.as_tensor(capi.DevicePointer(ptr, size), device="cuda:0").cpu().numpy()
                    assert np.array_equal(got, vol[z0:z1].reshape(-1).view(np.uint8)), "piece %d of rank %d" % (p, r)
    finally:
        for c in contexts:
            c.close()
