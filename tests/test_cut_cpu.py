"""The LOD cut's rule (include/vxb200.h "the LOD cut") as restated by tests/cut_oracle.py, on whole octrees of 64^3 to 1024^3
grids: refinement is monotone, the cut tiles the grid, touching cut nodes (face, edge or corner) differ by at most one
level, and block_adj names exactly the faces across which the grid is drawn one level finer - for seeded cameras and
factors in [2, 64] and for the float edge cases.  A negative control shows that the balance check fails on the centre
distance rule of vxb_mesh_select_lod without its top-level stop.  The capi mirror of the header's constant."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import cut_oracle as oracle
from voxels_b200 import capi

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = np.float32
# the 13 directions of one half of the 26-neighbourhood of a level-0 block
HALF26 = [d for d in np.ndindex(3, 3, 3) if (np.array(d) - 1).tolist() > [0, 0, 0]]


def levels_for(n):
    return int(np.log2(n // 16)) + 1


def coords(n, level):
    nb = (n // 16) >> level
    cid = np.arange(nb ** 3)
    return np.stack([cid % nb, (cid // nb) % nb, cid // (nb * nb)], axis=1)


def shifted(a, d):
    """Pairs (a[q], a[q + d]) over every q with both inside, for a direction d in {-1, 0, 1}^3."""
    src = tuple(slice(max(0, -k), a.shape[i] - max(0, k)) for i, k in enumerate(d))
    dst = tuple(slice(max(0, k), a.shape[i] - max(0, -k)) for i, k in enumerate(d))
    return a[src], a[dst]


def max_touching_difference(lmap):
    """The largest level difference between two touching cut nodes: two nodes touch iff a level-0 block of one is in the
    26-neighbourhood of a level-0 block of the other."""
    worst = 0
    for d in HALF26:
        a, b = shifted(lmap, np.array(d) - 1)
        worst = max(worst, int(np.abs(a - b).max()) if a.size else 0)
    return worst


def check_cut(n, camera, factor):
    """Every statement about the cut of (camera, factor) on the whole n^3 octree; returns the level map."""
    levels = levels_for(n)
    top = levels - 1
    ref = {l: oracle.refines(l, coords(n, l), camera, factor) for l in range(levels)}
    # monotone: refine(child) => refine(parent)
    for l in range(1, top):
        child = ref[l]
        b = coords(n, l) >> 1
        nbp = (n // 16) >> (l + 1)
        parent = ref[l + 1][b[:, 0] + nbp * (b[:, 1] + nbp * b[:, 2])]
        assert not (child & ~parent).any(), "refine is not monotone at level %d" % l
    # the O(1) test is the descent: no refine at the node, every ancestor refines
    recs = oracle.full_octree(n, levels)
    selected, adj = oracle.cut(recs, n, levels, camera, factor)
    base = np.cumsum([0] + [((n // 16) >> l) ** 3 for l in range(levels)])
    for l in range(levels):
        b = coords(n, l)
        want = ~ref[l]
        for k in range(l + 1, levels):
            nbk = (n // 16) >> k
            a = b >> (k - l)
            want &= ref[k][a[:, 0] + nbk * (a[:, 1] + nbk * a[:, 2])]
        assert np.array_equal(selected[base[l]:base[l + 1]], want), "level %d" % l
    lmap = oracle.level_map(n, levels, lambda l: selected[base[l]:base[l + 1]])
    assert (lmap >= 0).all(), "the cut does not tile the grid: %d gaps, %d overlaps" % ((lmap == -1).sum(), (lmap == -2).sum())
    assert max_touching_difference(lmap) <= 1
    # block_adj, per level-0 block on face f of its cut node: bit f <=> the block across the face is one level finer
    nb0 = n // 16
    amap = np.zeros_like(lmap)
    for l in range(levels):
        nb = nb0 >> l
        a = adj[base[l]:base[l + 1]].astype(np.int64).reshape(nb, nb, nb).transpose(2, 1, 0)
        s = selected[base[l]:base[l + 1]].reshape(nb, nb, nb).transpose(2, 1, 0)
        rep = lambda x: np.repeat(np.repeat(np.repeat(x, 1 << l, 0), 1 << l, 1), 1 << l, 2)
        amap = np.where(rep(s), rep(a), amap)
    q = np.stack(np.meshgrid(np.arange(nb0), np.arange(nb0), np.arange(nb0), indexing="ij"), axis=-1)
    size = np.left_shift(1, lmap)
    for f, d in enumerate(oracle.FACES):
        axis = int(np.nonzero(d)[0][0])
        on_face = (q[..., axis] % size == 0) if d[axis] < 0 else (q[..., axis] % size == size - 1)
        across = q[..., axis] + d[axis]
        inside = (across >= 0) & (across < nb0)
        bit = (amap >> f) & 1
        assert not (on_face & ~inside & (bit == 1)).any(), "block_adj names a face on the grid box"
        nbr = np.roll(lmap, -int(d[axis]), axis=axis)
        m = on_face & inside
        assert np.array_equal(bit[m] == 1, nbr[m] == lmap[m] - 1), "face %d" % f
    return lmap


def test_seeded_cameras_and_factors():
    rng = np.random.RandomState(31)
    seen = set()
    for n, count in ((64, 1200), (128, 800), (256, 300), (512, 80), (1024, 24)):
        for _ in range(count):
            camera = rng.uniform(-0.5 * n, 1.5 * n, 3).astype(F)
            if rng.rand() < 0.3:                                     # on block faces, edges and corners of some level
                camera = (np.round(camera / 32) * 32).astype(F)
            factor = F(np.exp(rng.uniform(np.log(2), np.log(64))))
            lmap = check_cut(n, camera, factor)
            seen.add((n, int(lmap.max()) - int(lmap.min())))
    assert {d for n, d in seen if n >= 256} >= {0, 1, 2}


def test_float_edge_cases():
    n = 256
    levels = levels_for(n)
    for factor in (2.0, 4.0, 14.6):
        for camera in [(0.0, 0.0, 0.0), (128.0, 64.0, 32.0), (256.0, 256.0, 256.0), (100.3, 17.0, 250.5),   # faces, inside
                       (1e6, -3e5, 7e5), (-1e7, 1e7, -1e7), (1e30, 0.0, 0.0)]:                                 # far outside
            check_cut(n, np.array(camera, F), factor)
    # every node refines but level 0: the cut is the whole level 0 (lim * lim overflows to +inf)
    recs = oracle.full_octree(n, levels)
    selected, adj = oracle.cut(recs, n, levels, (128, 300, 128), 1e30)
    assert np.array_equal(selected, recs["level"] == 0) and not adj.any()
    # a camera far outside the grid: the top node alone
    selected, _ = oracle.cut(recs, n, levels, (1e6, 1e6, 1e6), 64.0)
    assert np.array_equal(selected, recs["level"] == levels - 1)


def test_camera_exactly_at_the_limit_does_not_refine():
    """dist2 == lim^2 does not refine; one ulp closer does.  Node (level 2, b = (1, 0, 2)): s = 64, box x [64, 128], y (= b.z)
    [128, 192], z (= b.y) [0, 64]."""
    b = np.array([[1, 0, 2]])
    for factor in (2.0, 3.0, 4.0):
        lim = factor * 64
        for axis, edge, sign in ((0, 128.0, 1), (0, 64.0, -1), (1, 192.0, 1), (2, 0.0, -1)):
            cam = np.array([96.0, 160.0, 32.0], F)
            cam[axis] = edge + sign * lim
            assert not oracle.refines(2, b, cam, factor)[0]
            assert oracle.refines(2, b, cam, np.nextafter(F(factor), F(np.inf)))[0]        # one ulp more lod_factor
            if sign > 0:                        # one ulp closer: c - hi is exact there (Sterbenz), lo - c of a negative c is not
                cam[axis] = np.nextafter(F(cam[axis]), F(edge))
                assert oracle.refines(2, b, cam, factor)[0]
    # diagonal, the rule alone (the call refuses factors below 2): level 1, b = (0, 0, 0), box [0, 32]^3; e = (24, 32, 0),
    # dist2 = 1600 = (1.25 * 32)^2
    cam = np.array([32.0 + 24.0, 32.0 + 32.0, 16.0], F)
    assert not oracle.refines(1, np.array([[0, 0, 0]]), cam, 40.0 / 32.0)[0]
    assert oracle.refines(1, np.array([[0, 0, 0]]), cam, np.nextafter(F(40.0 / 32.0), F(2)))[0]
    # inside the box: e = 0 refines at any factor, on any face too
    for cam in ([96.0, 160.0, 32.0], [64.0, 128.0, 0.0], [128.0, 192.0, 64.0]):
        assert oracle.refines(2, b, np.array(cam, F), 2.0)[0]


def old_rule_cut_levels(n, camera, base):
    """The level map of vxb_mesh_select_lod's centre-distance rule with the top-level stop removed."""
    levels = levels_for(n)
    cam = np.asarray(camera, F)

    def refine(l, b):
        if l == 0:
            return np.zeros(len(b), bool)
        c = (b.astype(F) + F(0.5)) * F(16 << l)
        dx, dy, dz = c[:, 0] - cam[0], c[:, 2] - cam[1], c[:, 1] - cam[2]
        lim = F(base) * F(1 << l)
        return (dx * dx + dy * dy) + dz * dz < lim * lim

    def selected(l):
        b = coords(n, l)
        sel = ~refine(l, b)
        for k in range(l + 1, levels):
            sel &= refine(k, b >> (k - l))
        return sel
    return oracle.level_map(n, levels, selected)


def test_balance_check_fails_on_the_centre_rule():
    rng = np.random.RandomState(8)
    worst = 0
    for _ in range(20):
        lmap = old_rule_cut_levels(512, rng.uniform(0, 512, 3), 8.0)
        assert (lmap >= 0).all()
        worst = max(worst, max_touching_difference(lmap))
    assert worst >= 2


def test_lod_factor_constant_matches_the_header(tmp_path):
    gcc = shutil.which("gcc")
    if not gcc:
        pytest.skip("no gcc")
    src = tmp_path / "cut.c"
    src.write_text('#include <stdio.h>\n#include "vxb200.h"\nint main(void)\n{\n\tint (*call)(vxb_mesh*, const float*, float, const vxb_view*, '
                   'uint32_t, vxb_draw_lists*) = vxb_mesh_select_cut;\n\t(void)call;\n\tprintf("%.9g\\n", (double)VXB_LOD_FACTOR_MIN);\n'
                   '\treturn 0;\n}\n')
    exe = tmp_path / "cut"
    out = subprocess.run([gcc, "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(REPO, "include"), str(src), "-o", str(exe),
                          "-Wl,--unresolved-symbols=ignore-all"], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    got = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()
    assert float(got[0]) == capi.VXB_LOD_FACTOR_MIN == 2.0
    assert "vxb_mesh_select_cut" in capi.EXPORTED_SYMBOLS
