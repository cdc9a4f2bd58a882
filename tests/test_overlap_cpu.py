"""The box overlap oracle (tests/overlap_oracle.py) on hand-built meshes, without a GPU: the header's test at its boundaries
(touching faces, edges and corners, one ulp away, the normal and edge axes alone, degenerate triangles and boxes, +-0), the
result order, the struct mirrors against a C build of include/vxb200.h, and agreement with the float64 clipping reference."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import overlap_oracle as oracle
from raycast_oracle import result_from_blocks
from voxels_b200 import capi

F = np.float32
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def box(lo, hi):
    return capi.make_boxes([lo], [hi])[0]


def tri(*v):
    return np.array(v, np.float32).reshape(1, 3, 3)


def overlaps(b, t):
    return bool(oracle.sat(b, t)[0])


def separating_axes(b, t):
    """Which of the 13 axes separate (0-2 box axes, 3 the normal, 4-12 u_i x e_j): evaluated one by one, float32."""
    p = np.asarray(t, np.float32)[0]
    lo, hi = b["min"].astype(np.float32), b["max"].astype(np.float32)
    out = [i for i in range(3) if not (p[:, i].min() <= hi[i] and p[:, i].max() >= lo[i])]
    c, h = (lo + hi) * F(0.5), hi * F(0.5) - lo * F(0.5)
    v = (p - c)[None]
    e = [v[0, 1] - v[0, 0], v[0, 2] - v[0, 1], v[0, 0] - v[0, 2]]
    n = np.array([e[0][1] * e[1][2] - e[0][2] * e[1][1], e[0][2] * e[1][0] - e[0][0] * e[1][2], e[0][0] * e[1][1] - e[0][1] * e[1][0]], np.float32)
    axes = [n] + [np.array(a, np.float32) for i in range(3) for ej in e
                  for a in [[(0, -ej[2], ej[1]), (ej[2], 0, -ej[0]), (-ej[1], ej[0], 0)][i]]]
    for k, a in enumerate(axes):
        if oracle._separates(a[0:1], a[1:2], a[2:3], v, h[0], h[1], h[2])[0]:
            out.append(3 + k)
    return out


def agrees64(b, t):
    return oracle.clip64(b["min"], b["max"], t[0]) == overlaps(b, t)


def up(x):
    return F(np.nextafter(F(x), F(np.inf)))


def down(x):
    return F(np.nextafter(F(x), F(-np.inf)))


B = box((4, 4, 4), (8, 8, 8))


@pytest.mark.parametrize("name,t,away", [
    # a vertex on the face x = 8; away: that vertex one ulp beyond it
    ("face", tri((8, 5, 6), (12, 5, 6), (12, 7, 7)), tri((up(8), 5, 6), (12, 5, 6), (12, 7, 7))),
    # a vertex on the edge x = y = 8
    ("edge", tri((8, 8, 6), (12, 9, 6), (12, 12, 7)), tri((up(8), 8, 6), (12, 9, 6), (12, 12, 7))),
    # a vertex on the corner (8, 8, 8)
    ("corner", tri((8, 8, 8), (12, 9, 9), (10, 12, 11)), tri((8, 8, up(8)), (12, 9, 9), (10, 12, 11))),
    # a triangle edge crossing the box edge x = y = 8 at z = 6 (no vertex on the box): the axis u_z x e decides
    ("edge_by_edge", tri((7, 9, 6), (9, 7, 6), (9, 9, 6)), tri((up(7), up(9), 6), (up(9), up(7), 6), (9, 9, 6))),
    # a face of the triangle touching the box corner (4, 4, 4) (plane x + y + z = 12): the normal decides
    ("corner_by_face", tri((0, 6, 6), (6, 0, 6), (6, 6, 0)), tri((0, down(6), 6), (down(6), 0, 6), (6, 6, -0.5))),
])
def test_touching_is_included_and_one_ulp_away_is_not(name, t, away):
    assert overlaps(B, t), name
    assert oracle.clip64(B["min"], B["max"], t[0]), name
    assert not overlaps(B, away), name
    assert agrees64(B, away), name


def test_excluded_by_one_edge_axis_only():
    b = box((2, 2, 8), (4, 4, 10))
    t = tri((3.75, 4.75, 9), (4.75, 3.75, 9), (10, 10, 0))    # the edge on x + y = 8.5; the plane crosses the box
    assert separating_axes(b, t) == [3 + 1 + 2 * 3 + 0]          # u_z x e0 only
    assert not overlaps(b, t) and agrees64(b, t)
    counts = {}
    oracle.sat(b, t, counts)
    assert counts == {"box": 0, "normal": 0, "edge": 1}


def test_excluded_by_the_normal_axis_only():
    t = tri((13, 6, 6), (6, 13, 6), (6, 6, 13))                  # the plane x + y + z = 25 passes the corner (8, 8, 8) by 1
    assert separating_axes(B, t) == [3]
    assert not overlaps(B, t) and agrees64(B, t)
    counts = {}
    oracle.sat(B, t, counts)
    assert counts == {"box": 0, "normal": 1, "edge": 0}


def test_large_triangle_through_the_box_with_every_vertex_outside():
    b = box((6, 6, 6), (10, 10, 10))
    t = tri((0, 0, 8), (16, 0, 8), (0, 16, 8))
    assert all(not np.all((v >= 6) & (v <= 10)) for v in t[0])
    assert overlaps(b, t) and agrees64(b, t)
    t2 = tri((0, 0, 0), (16, 0, 8), (0, 16, 8))                 # oblique, z = (x + y) / 2: through (7, 7, 7)
    assert overlaps(b, t2) and agrees64(b, t2)


def test_collinear_and_zero_area_triangles():
    b = box((6, 6, 6), (10, 10, 10))
    assert overlaps(b, tri((0, 8, 8), (8, 8, 8), (16, 8, 8)))           # a segment through the box
    miss = tri((2, 10, 8), (6, 14, 8), (10, 18, 8))                      # y = x + 8: its box touches the box at y = 10, x in [6, 10]
    assert not overlaps(b, miss) and agrees64(b, miss)
    assert 0 not in separating_axes(b, miss) and 1 not in separating_axes(b, miss)
    assert overlaps(b, tri((7, 7, 7), (7, 7, 7), (7, 7, 7)))           # a point inside
    assert overlaps(b, tri((10, 10, 10), (10, 10, 10), (10, 10, 10)))  # a point on the corner
    assert not overlaps(b, tri((up(10), 10, 10), (up(10), 10, 10), (up(10), 10, 10)))
    assert overlaps(b, tri((0, 0, 0), (16, 16, 16), (16, 16, 16)))     # two equal vertices: the diagonal
    shifted = tri((0, 0, 5), (16, 16, 21), (16, 16, 21))                # the diagonal 5 voxels up in z: its box meets the box
    assert not overlaps(b, shifted) and agrees64(b, shifted)


def test_signed_zeros():
    t = tri((0.0, 0.0, 0.0), (4, 0, 0), (0, 4, 0))
    for lo, hi in [((-0.0, -0.0, -0.0), (1, 1, 1)), ((-1, -1, -1), (-0.0, -0.0, -0.0)), ((-1, -1, -1), (0.0, 0.0, 0.0))]:
        assert overlaps(box(lo, hi), t), (lo, hi)
    neg = tri((-0.0, -0.0, -0.0), (-4, -0.0, 0), (-0.0, -4, -0.0))
    assert overlaps(box((0, 0, 0), (1, 1, 1)), neg)
    assert not overlaps(box((up(0), 0, 0), (1, 1, 1)), neg)


def test_degenerate_boxes():
    t = tri((0, 0, 8), (16, 0, 8), (0, 16, 8))
    assert overlaps(box((4, 4, 8), (4, 4, 8)), t)                        # a point inside the triangle
    assert overlaps(box((0, 0, 8), (0, 0, 8)), t)                        # its vertex
    assert overlaps(box((8, 8, 8), (8, 8, 8)), t)                        # on its edge x + y = 16
    assert not overlaps(box((8, up(8), 8), (8, up(8), 8)), t)
    assert not overlaps(box((4, 4, 8.5), (4, 4, 8.5)), t)
    assert overlaps(box((2, 2, 8), (3, 3, 8)), t)                        # flat along z, in the plane
    assert overlaps(box((2, 2, 0), (3, 3, 16)), t)                       # a column through it
    assert not overlaps(box((12, 12, 0), (13, 13, 16)), t)               # a column beside it (box axes pass, an edge axis separates)
    assert not overlaps(box((2, 2, up(8)), (3, 3, 9)), t)
    t3 = tri((0, 0, 0), (16, 0, 16), (0, 16, 16))
    assert overlaps(box((4, 4, 8), (4, 4, 8)), t3)                       # a point on an oblique triangle (z = x + y)


def _flat_block(x0, z0, y_out, k):
    """k triangles in the plane y = y_out over the output xz cell [x0, x0 + 16] x [z0, z0 + 16]."""
    pos, ind = [], []
    for i in range(k):
        a = x0 + 1 + 2 * i
        pos += [(a, y_out, z0 + 1), (a + 1, y_out, z0 + 1), (a, y_out, z0 + 2)]
        ind += [3 * i, 3 * i + 1, 3 * i + 2]
    return np.array(pos, np.float32), np.zeros((len(pos), 3), np.float32), ind


def test_order_is_coord_id_then_triangle_on_a_mesh_whose_slots_are_out_of_order():
    n = 64
    blocks = []
    # grid coordinates (x, y, z) -> output (x, z, y); listed so that slot order is neither coord_id order nor its reverse
    for gx, gy, gz in [(1, 0, 0), (0, 1, 0), (0, 0, 0), (1, 1, 0), (0, 0, 1)]:
        pos, nrm, ind = _flat_block(16 * gx, 16 * gy, 16 * gz + 8, 3)
        blocks.append(((gx, gy, gz), pos, nrm, ind))
    res = result_from_blocks(n, blocks)
    offsets, tris = oracle.overlap_boxes(res, capi.make_boxes([(0, 0, 0), (0, 8, 0), (16, 0, 16)], [(32, 32, 32), (32, 8, 32), (32, 32, 32)]))
    cid = res.records["coord_id"][tris["slot"]]
    assert list(offsets) == [0, 15, 27, 30]
    for q in range(3):
        part = slice(int(offsets[q]), int(offsets[q + 1]))
        keys = list(zip(cid[part], tris["triangle"][part]))
        assert keys == sorted(keys)
    assert list(tris["slot"][:15]) == [2, 2, 2, 0, 0, 0, 1, 1, 1, 3, 3, 3, 4, 4, 4]
    assert (tris["block_id"] == 1000 + tris["slot"]).all()
    first = res.records[2]
    want = res.verts["pos"][first["vertex_offset"] + res.idx[first["index_offset"]:first["index_offset"] + 3]]
    assert np.array_equal(tris["p"][0], want)
    # an invalid box has no triangles, and does not move the others
    bad = capi.make_boxes([(0, 0, 0), (np.nan, 0, 0), (5, 0, 0)], [(32, 32, 32), (1, 1, 1), (4, 1, 1)])
    o2, t2 = oracle.overlap_boxes(res, bad)
    assert list(o2) == [0, 15, 15, 15] and oracle.same((o2[:2], t2), (offsets[:2], tris[:15])) is None


def test_oracle_agrees_with_float64_clipping_on_random_pairs():
    rng = np.random.RandomState(4242)
    count, excluded, overlapping = 20000, 0, 0
    for _ in range(count):
        c = rng.uniform(-8, 8, 3)
        h = rng.uniform(0.05, 4, 3) * (rng.uniform(size=3) > 0.05)     # some flat boxes
        b = box((c - h).astype(np.float32), (c + h).astype(np.float32))
        t = (c + rng.normal(scale=rng.choice([0.5, 3, 8]), size=(3, 3))).astype(np.float32)[None]
        if rng.uniform() < 0.05:
            t[0, 2] = t[0, 1]                                           # zero area
        lo, hi = b["min"].astype(np.float64), b["max"].astype(np.float64)
        inward = np.where(hi - lo > 2e-4, 1e-4, 0.0)                   # a flat axis is not shrunk
        grown, shrunk = oracle.clip64(lo - 1e-4, hi + 1e-4, t[0]), oracle.clip64(lo + inward, hi - inward, t[0])
        inside = oracle.clip64(lo, hi, t[0])
        if grown != inside or shrunk != inside:
            excluded += 1                                               # within 1e-4 voxel of touching
            continue
        assert overlaps(b, t) == inside, (b, t)
        overlapping += inside
    print("random pairs: %d, excluded within 1e-4: %d, overlapping: %d" % (count, excluded, overlapping))
    assert excluded < count // 20 and count // 4 < overlapping < count * 3 // 4


def test_struct_mirrors_match_a_c_build(tmp_path):
    gcc = shutil.which("gcc")
    if not gcc:
        pytest.skip("no gcc")
    src = tmp_path / "t.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "vxb200.h"\nint main(void) { printf("%u %u %u %u %u %u\\n", '
                   '(unsigned)sizeof(vxb_box), (unsigned)offsetof(vxb_box, max), (unsigned)sizeof(vxb_overlap_triangle), '
                   '(unsigned)offsetof(vxb_overlap_triangle, slot), (unsigned)offsetof(vxb_overlap_triangle, block_id), '
                   '(unsigned)offsetof(vxb_overlap_triangle, triangle)); return 0; }\n')
    exe = tmp_path / "t"
    subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(REPO, "include"), "-o", str(exe), str(src)],
                   check=True, capture_output=True)
    got = [int(x) for x in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split()]
    d, b = capi.OVERLAP_TRIANGLE_DTYPE, capi.BOX_DTYPE
    assert got == [b.itemsize, b.fields["max"][1], d.itemsize, d.fields["slot"][1], d.fields["block_id"][1], d.fields["triangle"][1]]
