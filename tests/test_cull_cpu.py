"""The culling oracle (tests/cull_oracle.py) against a float64 geometric statement: a plane culls a box iff all eight corners
are outside it.  Hand-built boxes and planes with small dyadic coordinates, so that float32 and float64 agree exactly."""
import ctypes as C
import itertools

import numpy as np

import cull_oracle as oracle
from voxels_b200 import capi

F = np.float32


def corners(box):
    return np.array([[box[3 * i + 0], box[3 * j + 1], box[3 * k + 2]] for i, j, k in itertools.product((0, 1), repeat=3)], np.float64)


def passes_geometric(box, planes):
    """float64: the box passes a plane unless all eight corners are strictly outside."""
    c = corners(np.asarray(box, np.float64))
    p = np.asarray(planes, np.float64)
    return all(((c @ pl[:3]) + pl[3] >= 0).any() for pl in p)


def view_of(*planes):
    v = oracle.PASS_ALL.copy()
    for k, p in enumerate(planes):
        v[k] = p
    return v


BOX = np.array([2, 4, 6, 10, 8, 7], F)


def check(box, view, want=None):
    got = bool(oracle.box_passes(np.asarray(box, F)[None], view)[0])
    assert got == passes_geometric(box, view)
    if want is not None:
        assert got == want
    return got


def test_planes_through_corner_edge_and_face_pass():
    # s == 0 passes: the plane touches the box at its p-vertex
    check(BOX, view_of(oracle.plane((1, 1, 1), (2, 4, 6))), True)              # box on the inside, touching at the min corner
    check(BOX, view_of(oracle.plane((-1, -1, -1), (2, 4, 6))), True)           # box outside but for that corner
    check(BOX, view_of(oracle.plane((-1, -1, -1), (1.75, 4, 6))), False)       # a quarter further: culled
    check(BOX, view_of(oracle.plane((1, 1, 0), (10, 8, 0))), True)             # through the edge x = 10, y = 8
    check(BOX, view_of(oracle.plane((1, 1, 0), (10.25, 8, 0))), False)
    check(BOX, view_of(oracle.plane((0, 1, 0), (0, 8, 0))), True)              # on the face y = 8, looking away from the box
    check(BOX, view_of(oracle.plane((0, 1, 0), (0, 8.5, 0))), False)
    check(BOX, view_of(oracle.plane((0, -1, 0), (0, 4, 0))), True)             # on the face y = 4
    check(BOX, view_of(oracle.plane((0, -1, 0), (0, 3.5, 0))), False)


def test_zero_and_negative_zero_normal_components():
    # a zero component of either sign picks max; the product is 0 either way
    for z in (0.0, -0.0):
        p = np.array([z, 1.0, z, -8.0], F)
        check(BOX, view_of(p), True)
        p = np.array([z, 1.0, z, -8.25], F)
        check(BOX, view_of(p), False)
        p = np.array([-1.0, z, z, 2.0], F)
        check(BOX, view_of(p), True)
        p = np.array([-1.0, z, z, 1.75], F)
        check(BOX, view_of(p), False)


def test_pass_everything_plane_and_partial_views():
    assert oracle.box_passes(BOX[None], oracle.PASS_ALL)[0]
    assert oracle.box_passes(BOX[None], np.tile(np.array([0, 0, 0, 0], F), (6, 1)))[0]           # d = 0 passes too
    assert not oracle.box_passes(BOX[None], view_of(np.array([0, 0, 0, -1], F)))[0]              # d < 0 passes nothing
    # one culling plane among pass-everything planes decides, in whichever position
    cull = oracle.plane((1, 0, 0), (10.5, 0, 0))
    for k in range(6):
        v = oracle.PASS_ALL.copy(); v[k] = cull
        assert not oracle.box_passes(BOX[None], v)[0]


def test_point_box():
    pt = np.array([3, 3, 3, 3, 3, 3], F)
    check(pt, view_of(oracle.plane((1, 2, -1), (3, 3, 3))), True)              # the plane through the point
    check(pt, view_of(oracle.plane((1, 2, -1), (3.5, 3, 3))), False)
    check(pt, view_of(oracle.plane((1, 2, -1), (2.5, 3, 3))), True)
    check(pt, oracle.box_planes((3, 3, 3), (3, 3, 3)), True)                   # an orthographic volume that is the point


def test_empty_box_passes_no_plane_with_a_normal():
    assert not oracle.box_passes(oracle.EMPTY_BOX[None], view_of(oracle.plane((0, 1, 0), (0, -1000, 0))))[0]


def test_random_dyadic_boxes_and_planes_equal_the_corner_statement():
    rng = np.random.RandomState(5)
    seen = set()
    for _ in range(4000):
        lo = rng.randint(-32, 32, 3) / 4.0
        hi = lo + rng.randint(0, 24, 3) / 4.0
        box = np.concatenate([lo, hi]).astype(F)
        planes = np.concatenate([rng.randint(-4, 5, (6, 3)) / 2.0, rng.randint(-64, 65, (6, 1)) / 4.0], axis=1).astype(F)
        planes[rng.randint(0, 6)] = oracle.PASS_ALL[0]
        seen.add(check(box, planes))
    assert seen == {True, False}


def test_frustum_builders_face_inwards():
    v = oracle.perspective((0, 0, 0), (0, 0, 1), (0, 1, 0), 90, 60, 1, 100)
    inside = np.array([0, 0, 50, 0, 0, 50], F)
    behind = np.array([0, 0, -50, 0, 0, -50], F)
    beside = np.array([80, 0, 50, 80, 0, 50], F)
    assert oracle.box_passes(np.stack([inside, behind, beside]), v).tolist() == [True, False, False]
    b = oracle.box_planes((0, 0, 0), (16, 16, 16))
    assert oracle.box_passes(np.array([[16, 16, 16, 20, 20, 20], [16.5, 0, 0, 20, 4, 4]], F), b).tolist() == [True, False]


def test_block_boxes_of_a_hand_built_mesh():
    res = capi.Result.__new__(capi.Result)
    res.n = 64
    res.records = np.zeros(3, capi.RECORD_DTYPE)
    res.verts = np.zeros(5, capi.VERTEX_DTYPE)
    res.tverts = np.zeros(2, capi.VERTEX_DTYPE)
    res.verts["pos"] = [(1, 2, 3), (4, 0, 3), (9, 9, 9), (0, 0, 0), (5, 5, 5)]
    res.verts["sec"] = [(1, 2, 3, 77), (4, 0, -1, 99), (9, 9, 9, 0), (0, 0, 0, 0), (5, 6, 5, 1000)]
    res.tverts["pos"] = [(20, 1, 1), (1, 1, 1)]
    res.tverts["sec"] = [(20, 1, 1, 0), (1, -7, 1, 0)]
    r = res.records
    r[0]["vertex_offset"], r[0]["vertex_count"] = 0, 2
    r[0]["trans_vertex_offset"][4], r[0]["trans_vertex_count"][4] = 0, 1           # one transition vertex on face 4
    r[1]["vertex_offset"], r[1]["vertex_count"] = 4, 1
    r[1]["trans_vertex_offset"][0], r[1]["trans_vertex_count"][0] = 1, 1
    got = oracle.block_boxes(res)
    assert got[0].tolist() == [1, 0, -1, 20, 2, 3]                                 # sec[3] (77, 99) is not part of it
    assert got[1].tolist() == [1, -7, 1, 5, 6, 5]
    assert np.array_equal(got[2], oracle.EMPTY_BOX)                                # a block without vertices
    assert np.array_equal(oracle.block_boxes(res, np.array([1])), got[1:2])
    r["level"] = [0, 1, 1]; r["coord_id"] = [5, 1, 7]
    assert oracle.lattice_boxes(r, 64).tolist() == [[16, 0, 16, 32, 16, 32], [32, 0, 0, 64, 32, 32], [32, 32, 32, 64, 64, 64]]


def test_cut_restates_the_draw_tests_cut():
    """The array / float32 cut equals the scalar statement of test_gpu_draws on every (level, coord) slot of a 128^3 grid."""
    from test_gpu_draws import _finer, _selected
    n, levels = 128, 4
    recs = []
    for level in range(levels):
        nb = (n // 16) >> level
        part = np.zeros(nb ** 3, capi.RECORD_DTYPE)
        part["level"], part["coord_id"] = level, np.arange(nb ** 3)
        recs.append(part)
    recs = np.concatenate(recs)
    for camera, base in [((40.0, 70.0, 50.0), 48.0), ((128.0, 64.0, 128.0), 20.0), ((-50.0, 300.0, 10.0), 64.0)]:
        selected, adj = oracle.cut(recs, n, levels, camera, base)
        cam = np.array(camera, np.float64)
        for k, r in enumerate(recs):
            level = int(r["level"]); nb = (n // 16) >> level; c = int(r["coord_id"])
            b = (c % nb, (c // nb) % nb, c // (nb * nb))
            want = _selected(level, b, cam, base, levels - 1)
            assert bool(selected[k]) == want
            if want and level > 0:
                a = 0
                for f, d in enumerate(oracle.FACES):
                    nbr = tuple(int(v) for v in np.array(b) + d)
                    if min(nbr) >= 0 and max(nbr) < nb and _finer(level, nbr, cam, base, levels - 1):
                        a |= 1 << f
                assert int(adj[k]) == a
        assert selected.any()


def test_struct_mirrors_of_view_and_bounds():
    assert C.sizeof(capi.View) == 6 * 4 * 4 and C.sizeof(capi.MeshBounds) == 8 + 12 * 4 + 4 + 4
    assert C.sizeof(capi.View) * capi.VXB_VIEWS_MAX == 768
    v = capi.make_views(np.arange(48, dtype=np.float32).reshape(2, 6, 4))
    assert len(v) == 2 and v[1].planes[5][3] == 47.0 and v[0].planes[1][0] == 4.0
