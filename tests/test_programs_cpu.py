"""SDF programs (include/vxb200.h vxb_op, voxels_b200/csrc/vxb_program.h) on the host, without a GPU:
  * the host generator (the evaluator the fill kernels share) equals the UNMODIFIED reference's Grid::Create fed the same
    program through its VoxelSurface callback, byte for byte;
  * the fill's per-block cull decision (the same source as the device's pass A) only ever writes blocks that are constant,
    culls most of the 32-primitive scene, and keeps the margin cases and TERRAIN-selected blocks for the per-voxel pass;
  * the validator rejects malformed programs at the right op;
  * libvxb200.so exports the new entry points."""
import ctypes as C

import numpy as np
import pytest

import programs
from voxels_b200 import capi
from voxels_b200.capi import Op


@pytest.fixture(scope="module")
def reference():
    """The unmodified reference with the SDF-program calls (oracle/_ref/libvxh_programs_ref.so, built by oracle/programs.mk
    from tests/harness/vxh_capi.cpp + vxh_programs.cpp): every call of the conftest's reference plus the program ones."""
    import program_harness
    lib = program_harness.load()
    if lib is None:
        pytest.skip("oracle/_ref/libvxh_programs_ref.so not built (needs the reference checkout: make -C oracle -f programs.mk programs)")
    return lib


@pytest.mark.parametrize("name", sorted(programs.SMALL))
@pytest.mark.parametrize("n", [32, 64])
def test_program_dense_equals_reference_constructor(reference, name, n):
    ops, start, step = programs.SMALL[name](n)
    g = reference.grid_create_program(n, ops, start, step)
    want = reference.grid_to_dense(g)
    reference.grid_destroy(g)
    got = reference.program_dense(n, ops, start, step)
    for a, b, ch in zip(want, got, ("distance", "material", "blend")):
        if not np.array_equal(a, b):
            bad = np.argwhere(a != b)
            raise AssertionError("%s %s: %d voxels differ, first (z,y,x)=%s" % (name, ch, len(bad), bad[0]))


def test_programs_cover_every_op_code():
    codes = {o.code for f in programs.SMALL.values() for o in f(64)[0]}
    assert codes == {capi.OP_SPHERE, capi.OP_BOX, capi.OP_CYLINDER, capi.OP_CAPSULE, capi.OP_TORUS, capi.OP_PLANE, capi.OP_TERRAIN,
                     capi.OP_UNION, capi.OP_INTERSECT, capi.OP_SUBTRACT, capi.OP_SMOOTH_UNION, capi.OP_OFFSET, capi.OP_SHELL}


def test_program_materials_follow_the_selected_value(reference):
    """SUBTRACT / SMOOTH_UNION / ties: the material of the side that won, the left one on a tie."""
    n = 64
    d, m, b = reference.program_dense(n, programs.subtract_materials(n)[0])
    assert {7, 8} <= set(np.unique(m[np.abs(d) < 4]).tolist())
    d, m, b = reference.program_dense(n, programs.smooth_union_materials(n)[0])
    assert {9, 10} <= set(np.unique(m).tolist())
    d, m, b = reference.program_dense(n, programs.ties(n)[0])
    assert np.all(m[:, :, n // 2] != 12), "the mid plane ties between the spheres go to the left one"
    assert 14 not in set(np.unique(m).tolist()), "an op intersected with an identical copy keeps the left material"


def _check_culled_blocks_are_constant(reference, n, ops, start, step):
    flags, values = reference.program_cull_flags(n, ops, start, step)
    dist, mat, blend = reference.program_dense(n, ops, start, step)
    nb = n // 16
    for b in np.nonzero(flags)[0]:
        bx, by, bz = b % nb, (b // nb) % nb, b // (nb * nb)
        sl = np.s_[bz * 16:bz * 16 + 16, by * 16:by * 16 + 16, bx * 16:bx * 16 + 16]
        assert np.all(dist[sl] == values[b, 0]) and abs(values[b, 0]) == 4, "block %d is not constant distance" % b
        assert np.all(mat[sl] == values[b, 1]) and np.all(blend[sl] == values[b, 2]), "block %d is not constant material" % b
    return flags


@pytest.mark.parametrize("name", sorted(programs.SMALL))
def test_cull_writes_only_constant_blocks(reference, name):
    ops, start, step = programs.SMALL[name](128)
    _check_culled_blocks_are_constant(reference, 128, ops, start, step)


def test_scene_culls_a_majority_of_blocks(reference):
    ops, start, step = programs.scene(1024)
    flags, _ = reference.program_cull_flags(1024, ops, start, step)
    assert flags.mean() > 0.5, "culled %.3f of the blocks" % flags.mean()
    # and at a size where the whole volume can be checked: every culled block is constant
    ops, start, step = programs.scene(256)
    _check_culled_blocks_are_constant(reference, 256, ops, start, step)


@pytest.mark.parametrize("past", [False, True])
def test_margin_blocks_are_not_culled(reference, past):
    n, nb = 128, 8
    ops, start, step = programs.margin(n, past)
    flags = _check_culled_blocks_are_constant(reference, n, ops, start, step).reshape(nb, nb, nb)   # [bz, by, bx]
    dist = reference.program_dense(n, ops, start, step)[0]
    # z = 16 quantises to 3 (exact 3) / to 4 (just past 3, within rounding of 3): the whole layer bz = 1 stays listed
    assert np.all(dist[16] == (4 if past else 3))
    assert not flags[1].any()
    # the spheres tie on x = 40 (block column bx = 2) around z = 90 (bz = 5): listed, while blocks above the spheres at
    # the grid's sides, clearly nearer one of them, are culled
    assert not flags[4:7, 1:4, 2].any()
    assert flags[7, 2, 0] and flags[7, 2, 7]
    # the two parallel planes of `past` tie within rounding: nothing is culled where they select the result (bz < 3)
    if past:
        assert not flags[:3].any()


def test_terrain_selected_blocks_are_not_culled(reference):
    n = 128
    flags, _ = reference.program_cull_flags(n, [Op.terrain(n, seed=5)])
    assert not flags.any()
    # a low terrain (period 16: its height stays within 8 +- 23) and a sphere above it
    ops = [Op.terrain(16, seed=5), Op.sphere(10.0, at=(64.0, 64.0, 110.0), material=9), Op.union()]
    flags, values = reference.program_cull_flags(n, ops)
    assert flags.any() and np.all(values[flags == 1, 1] == 9), "only blocks won by the sphere may be culled"


@pytest.mark.parametrize("case,index", [
    ("empty", 0), ("unknown", 1), ("underflow", 1), ("two_left", 2), ("nan", 0), ("inf_xform", 1), ("k_zero", 2),
    ("negative_radius", 0), ("negative_extent", 0), ("too_many_ops", 64), ("too_many_terrain", 2), ("too_deep", 8),
    ("negative_shell", 1), ("material_256", 0),
])
def test_validator_names_the_op(reference, case, index):
    ops = malformed(case)
    assert reference.program_validate(ops) == index


def malformed(case):
    """Malformed programs (shared with the GPU test): each returns the op list the library must refuse."""
    s = Op.sphere(4.0, at=(8.0, 8.0, 8.0))
    if case == "empty":
        return (Op * 0)()
    if case == "unknown":
        o = Op.union(); o.code = 20
        return [s, o]
    if case == "underflow":
        return [s, Op.union()]
    if case == "two_left":
        return [s, Op.sphere(2.0)]
    if case == "nan":
        o = Op.sphere(4.0); o.p[0] = float("nan")
        return [o]
    if case == "inf_xform":
        o = Op.box((1.0, 1.0, 1.0)); o.xform[10] = float("inf")
        return [s, o, Op.union()]
    if case == "k_zero":
        return [s, Op.sphere(2.0), Op.smooth_union(0.0)]
    if case == "negative_radius":
        return [Op.sphere(-1.0)]
    if case == "negative_extent":
        return [Op.box((1.0, -2.0, 1.0))]
    if case == "too_many_ops":
        return [s] + [Op.offset(0.0)] * 64
    if case == "too_many_terrain":
        return [Op.terrain(32), Op.terrain(32), Op.terrain(32), Op.union(), Op.union()]
    if case == "too_deep":
        return [s] * 9 + [Op.union()] * 8
    if case == "negative_shell":
        return [s, Op.shell(-1.0)]
    if case == "material_256":
        return [Op.sphere(4.0, material=256)]
    raise KeyError(case)


MALFORMED = ["empty", "unknown", "underflow", "two_left", "nan", "inf_xform", "k_zero", "negative_radius", "negative_extent",
             "too_many_ops", "too_many_terrain", "too_deep", "negative_shell", "material_256"]


def test_op_layout_matches_header():
    assert C.sizeof(Op) == 96 and C.sizeof(capi.ProgramStats) == 24


def test_library_exports_the_program_entry_points():
    lib = C.CDLL(capi.library_path())
    for name in ("vxb_grid_fill_program", "vxb_grid_inject_program", "vxb_grid_program_stats"):
        assert hasattr(lib, name), name


def test_op_constructors_store_the_inverse_placement():
    o = Op.sphere(3.0, at=(1.5, -2.0, 4.25))
    assert list(o.xform) == [1, 0, 0, 0, 1, 0, 0, 0, 1, -1.5, 2.0, -4.25]
    r = programs.rot(2, 90)
    o = Op.box((1, 2, 3), at=(0.0, 0.0, 0.0), rotation=r)
    m = np.array(list(o.xform[:9]), np.float64).reshape(3, 3)
    assert np.allclose(m @ r, np.eye(3), atol=1e-6)
