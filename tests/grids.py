"""Named seeded test grids shared by the CPU and GPU parity tests: name -> (dist, mat, blend) int8/uint8 [z,y,x]."""
import numpy as np

import gridgen


def _quantise(d):
    q = np.sign(d) * np.ceil(np.abs(d))  # reference `round` (VoxelGrid.cpp:37-40) + clamp +-4 (:42-50)
    return np.clip(q, -4, 4).astype(np.int8)


def sphere(n):
    d = _quantise(gridgen.sphere_floats(n))
    z = np.zeros((n, n, n), np.uint8)
    return d, z, z.copy()


def two_material_plane(n):
    z, y, x = np.meshgrid(np.arange(n), np.arange(n), np.arange(n), indexing="ij")
    d = _quantise(0.37 * (x - n / 2.0) + 0.61 * (y - n / 2.0) + 0.7 * (z - n / 2.0) + 0.25)
    mat = np.where(x + y > n, 1, 2).astype(np.uint8)
    blend = ((x * 3 + y * 5 + z * 7) % 256).astype(np.uint8)
    return np.ascontiguousarray(d), np.ascontiguousarray(mat), np.ascontiguousarray(blend)


SMALL = {
    "sphere64": lambda: sphere(64),
    "plane32": lambda: two_material_plane(32),
    "hostile64": lambda: gridgen.hostile(64),
    "hostile64_big_values": lambda: gridgen.hostile(64, seed=5, vmax=8, materials=5),
    "noise32": lambda: gridgen.noise_full(32),
    "noise16": lambda: gridgen.noise_full(16, seed=2),
    "positive_noise32": lambda: gridgen.noise_full(32, seed=4, lo=1, hi=4),
    "patchwork64": lambda: gridgen.patchwork(64),
    "hostile64_full_range": lambda: gridgen.hostile_full_range(64),
}
MEDIUM = {
    "hostile128": lambda: gridgen.hostile(128, seed=11),
    "sphere128": lambda: sphere(128),
    "noise64": lambda: gridgen.noise_full(64, seed=9, lo=-3, hi=2),
    "patchwork128": lambda: gridgen.patchwork(128),
}


def _terrain(n):
    from voxels_b200 import synth
    return tuple(t.numpy() for t in synth.terrain(n))


# the benchmark's terrain at a size the golden digests can cover (generated on the host: the same bytes everywhere)
LARGE = {
    "terrain256": lambda: _terrain(256),
    "patchwork256": lambda: gridgen.patchwork(256),
}

# only against the live reference (tests/test_gpu_paths.py): too large for the CPU tests
HUGE = {
    "patchwork512": lambda: gridgen.patchwork(512),
    "patchwork1024": lambda: gridgen.patchwork(1024),
}


# the grid store's thresholds (tests/test_gpu_gridstore_edges.py): not in the tables above, whose every level is compared
# with the reference, because the reference's coarse levels of rle_edges_skipped are undefined (see gridgen.skip_quirk)
RLE_EDGES = {
    "rle_edges_kept": gridgen.rle_edges_kept,
    "rle_edges_skipped": gridgen.rle_edges_skipped,
}


# the block kernels' per-block capacities (tests/test_thresholds_cpu.py, tests/test_gpu_thresholds.py): not in the tables
# above, so that their golden digests stay as they are
THRESHOLDS = {
    "thresholds256": gridgen.thresholds256,
}


def by_name(name):
    for table in (SMALL, MEDIUM, LARGE, HUGE, RLE_EDGES, THRESHOLDS):
        if name in table:
            return table[name]()
    raise KeyError(name)
