"""SDF programs (include/vxb200.h vxb_op) shared by the CPU and GPU tests of the program fill / edits, and the 32-primitive
scene tools/bench_programs.py measures.  Every function returns (ops, start, step) for an n^3 grid."""
import numpy as np

from voxels_b200.capi import Op


def rot(axis, degrees):
    """3x3 rotation about a coordinate axis (0 = x, 1 = y, 2 = z)."""
    c, s = np.cos(np.radians(degrees)), np.sin(np.radians(degrees))
    i, j = [(1, 2), (2, 0), (0, 1)][axis]
    m = np.eye(3)
    m[i, i], m[i, j], m[j, i], m[j, j] = c, -s, s, c
    return m


def union_box_sphere(n):
    h = n / 2
    return [Op.sphere(0.3 * n, at=(h, h, h), material=1, blend=10),
            Op.box((0.2 * n, 0.1 * n, 0.15 * n), at=(h + 3.5, h - 2.25, h + 0.5), rotation=rot(2, 30), material=2, blend=20),
            Op.union()], (0.0, 0.0, 0.0), 1.0


def intersect_cylinder_capsule(n):
    h = n / 2
    scaled = rot(0, 35) @ np.diag([1.0, 1.5, 0.75])          # a sheared, non-metric local frame
    return [Op.cylinder(0.3 * n, 0.35 * n, at=(h, h, h), rotation=rot(1, 20), material=3, blend=30),
            Op.capsule(0.2 * n, 0.25 * n, at=(h + 1.25, h, h - 0.5), rotation=scaled, material=4, blend=40),
            Op.intersect()], (0.0, 0.0, 0.0), 1.0


def torus_shell_offset_plane(n):
    h = n / 2
    return [Op.torus(0.25 * n, 0.08 * n, at=(h, h + 0.5, h), rotation=rot(0, 60), material=5, blend=50),
            Op.shell(1.5), Op.offset(-0.75),
            Op.plane((0.0, 0.0, 1.0), 0.2 * n, material=6, blend=60),
            Op.union()], (0.0, 0.0, 0.0), 1.0


def subtract_materials(n):
    """SUBTRACT takes the material of whichever side won: the box outside the hole, the sphere's on the hole's wall."""
    h = n / 2
    return [Op.box((0.3 * n, 0.3 * n, 0.3 * n), at=(h, h, h), material=7, blend=70),
            Op.sphere(0.25 * n, at=(h + 0.2 * n, h, h + 0.1 * n), material=8, blend=80),
            Op.subtract()], (0.0, 0.0, 0.0), 1.0


def smooth_union_materials(n):
    h = n / 2
    return [Op.sphere(0.2 * n, at=(h - 0.15 * n, h, h), material=9, blend=90),
            Op.capsule(0.12 * n, 0.2 * n, at=(h + 0.15 * n, h, h), rotation=rot(1, 80), material=10, blend=100),
            Op.smooth_union(0.1 * n)], (0.0, 0.0, 0.0), 1.0


def ties(n):
    """Equidistant operands: mirror-image spheres (exact ties on the mid plane) and an op unioned with an identical copy."""
    h = n / 2
    return [Op.sphere(0.2 * n, at=(h - 0.25 * n, h, h), material=11, blend=1),
            Op.sphere(0.2 * n, at=(h + 0.25 * n, h, h), material=12, blend=2),
            Op.union(),
            Op.box((0.1 * n, 0.1 * n, 0.1 * n), at=(h, h, 0.25 * n), material=13, blend=3),
            Op.box((0.1 * n, 0.1 * n, 0.1 * n), at=(h, h, 0.25 * n), material=14, blend=4),
            Op.intersect(),
            Op.union()], (0.0, 0.0, 0.0), 1.0


def terrain_cave(n):
    """A terrain with a cave: SUBTRACT of (a sphere INTERSECT a second terrain), plus a smooth-unioned rock."""
    h = n / 2
    return [Op.terrain(n, seed=7),
            Op.sphere(0.2 * n, at=(h, h, 0.5 * n), material=2, blend=5),
            Op.terrain(n / 2, origin=(3.0, 5.0), seed=11, at=(0.0, 0.0, 0.25 * n)),
            Op.intersect(),
            Op.subtract(),
            Op.box((0.1 * n, 0.08 * n, 0.06 * n), at=(0.3 * n, 0.6 * n, 0.6 * n), rotation=rot(2, 15) @ rot(0, 25), material=4, blend=9),
            Op.smooth_union(3.0)], (0.0, 0.0, 0.0), 1.0


def fractional_start(n):
    """Non-integer start and step: the grid samples world space at start + i * step."""
    return [Op.sphere(6.5, at=(3.0, 4.0, 5.0), material=1, blend=2),
            Op.torus(5.0, 1.75, at=(4.5, 3.25, 6.0), rotation=rot(1, 45), material=3, blend=4),
            Op.smooth_union(1.5),
            Op.box((1.5, 2.0, 2.5), at=(2.0, 2.0, 2.0), material=5, blend=6),
            Op.subtract(),
            Op.offset(0.25)], (-2.0, 1.5, 0.25), 0.375


def margin(n, past=False):
    """Samples at a quantised distance of exactly 3 and equidistant operands of different materials (laid out for n = 128).
    The plane d = z - 13 puts the exact 3 at z = 16, in the block layer bz = 1; the mirror-image spheres tie on the plane
    x = 40 (block column bx = 2) around z = 90, where they are nearer than the plane.  past=True: the plane is intersected
    with a copy shifted by one float ulp, whose value at z = 16 is just past 3 and which ties with it within rounding."""
    ops = [Op.plane((0.0, 0.0, 1.0), 13.0, material=1, blend=1)]
    if past:
        ops += [Op.plane((0.0, 0.0, 1.0), float(np.nextafter(np.float32(13.0), np.float32(0.0))), material=2, blend=2),
                Op.intersect()]
    return ops + [Op.sphere(6.0, at=(20.0, 40.0, 90.0), material=3, blend=3),
                  Op.sphere(6.0, at=(60.0, 40.0, 90.0), material=4, blend=4),
                  Op.union(),
                  Op.union()], (0.0, 0.0, 0.0), 1.0


def margin_past(n):
    return margin(n, past=True)


def every_op(n):
    """One program with every op code."""
    h = n / 2
    return [Op.sphere(0.2 * n, at=(h, h, h), material=1),
            Op.box((0.1 * n, 0.2 * n, 0.1 * n), at=(h + 4, h, h), rotation=rot(0, 10), material=2),
            Op.union(),
            Op.cylinder(0.08 * n, 0.3 * n, at=(h, h - 3, h), rotation=rot(1, 90), material=3),
            Op.subtract(),
            Op.capsule(0.06 * n, 0.2 * n, at=(h - 5, h + 5, h), material=4),
            Op.smooth_union(2.5),
            Op.torus(0.3 * n, 0.05 * n, at=(h, h, h + 2.5), material=5),
            Op.shell(1.0),
            Op.union(),
            Op.plane((0.1, 0.2, 0.97), 0.3 * n, material=6),
            Op.offset(1.5),
            Op.intersect(),
            Op.terrain(n, seed=3),
            Op.union()], (0.0, 0.0, 0.0), 1.0


SMALL = {f.__name__: f for f in (union_box_sphere, intersect_cylinder_capsule, torus_shell_offset_plane, subtract_materials,
                                 smooth_union_materials, ties, terrain_cave, fractional_start, margin, margin_past, every_op)}


def scene(n=1024):
    """The 32-primitive scene: a ground slab, 29 boxes / capsules / tori (smooth-unioned every third), and a cave - a
    sphere intersected with a terrain - subtracted from it all.  Sizes scale with n; positions are seeded."""
    rng = np.random.RandomState(2024)
    ops = [Op.box((0.5 * n, 0.5 * n, 0.1 * n), at=(0.5 * n, 0.5 * n, 0.1 * n), material=1, blend=0)]
    for i in range(29):
        at = rng.uniform(0.15 * n, 0.85 * n, size=3)
        at[2] = rng.uniform(0.2 * n, 0.6 * n)
        r = rot(int(rng.randint(3)), float(rng.uniform(0, 90))) @ rot(int(rng.randint(3)), float(rng.uniform(0, 90)))
        s = float(rng.uniform(0.02, 0.06)) * n
        mat, bl = 2 + i % 5, int(rng.randint(256))
        kind = i % 3
        if kind == 0:
            ops.append(Op.box((s, 0.7 * s, 0.5 * s), at=at, rotation=r, material=mat, blend=bl))
        elif kind == 1:
            ops.append(Op.capsule(0.4 * s, s, at=at, rotation=r, material=mat, blend=bl))
        else:
            ops.append(Op.torus(s, 0.3 * s, at=at, rotation=r, material=mat, blend=bl))
        ops.append(Op.smooth_union(0.01 * n) if i % 3 == 2 else Op.union())
    ops += [Op.sphere(0.12 * n, at=(0.5 * n, 0.45 * n, 0.18 * n), material=7, blend=0),
            Op.terrain(n / 8, seed=5, at=(0.0, 0.0, 0.12 * n)),
            Op.intersect(),
            Op.subtract()]
    assert len(ops) == 63 and sum(o.code < 16 for o in ops) == 32
    return ops, (0.0, 0.0, 0.0), 1.0
