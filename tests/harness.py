"""ctypes driver for tests/harness/vxh_capi.cpp (test infrastructure).

The same flat C ABI is compiled over (a) the unmodified reference -> oracle/_ref/libvxh_ref.so
and (b) this repo's drop-in Polygonizer backend -> build/libvxh_b200.so, so a parity test is
"run both libraries on the same grid, compare `LevelDump`s".
"""
import ctypes as C
import os

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = os.path.join(REPO, "oracle", "_ref", "libvxh_ref.so")
B200_LIB = os.path.join(REPO, "build", "libvxh_b200.so")

VERTEX_DTYPE = np.dtype([("pos", "<f4", 3), ("sec", "<f4", 4), ("nrm", "<f4", 3), ("tex", "u1", 8)])
ROW_DTYPE = np.dtype([("id", "<u4"), ("min", "<f4", 3), ("max", "<f4", 3), ("nv", "<u4"), ("ni", "<u4"),
                      ("tnv", "<u4", 6), ("tni", "<u4", 6)])
assert VERTEX_DTYPE.itemsize == 48 and ROW_DTYPE.itemsize == 84

IT_ADD, IT_SUBTRACT_ADD_INNER, IT_SUBTRACT = 0, 1, 2


class LevelDump:
    """One LOD level flattened: block rows + concatenated vertex / index arrays."""

    def __init__(self, rows, verts, idx, tverts, tidx):
        self.rows, self.verts, self.idx, self.tverts, self.tidx = rows, verts, idx, tverts, tidx

    def block(self, i):
        """Slices of block i: (row, verts, idx, [tverts per face], [tidx per face])."""
        r = self.rows
        v0 = int(r["nv"][:i].sum()); i0 = int(r["ni"][:i].sum())
        tv0 = int(r["tnv"][:i].sum()); ti0 = int(r["tni"][:i].sum())
        tvs, tis = [], []
        for f in range(6):
            tvs.append(self.tverts[tv0:tv0 + int(r["tnv"][i][f])]); tv0 += int(r["tnv"][i][f])
            tis.append(self.tidx[ti0:ti0 + int(r["tni"][i][f])]); ti0 += int(r["tni"][i][f])
        return r[i], self.verts[v0:v0 + int(r["nv"][i])], self.idx[i0:i0 + int(r["ni"][i])], tvs, tis


class VoxelsLib:
    def __init__(self, path):
        if not os.path.exists(path):
            raise FileNotFoundError(path)
        self.path = path
        L = self.L = C.CDLL(path)
        vp, u, f, d = C.c_void_p, C.c_uint, C.c_float, C.c_double
        sig = {
            "vxh_init": (C.c_int, []),
            "vxh_error_logs": (u, []),
            "vxh_set_threads": (None, [C.c_int]),
            "vxh_max_threads": (C.c_int, []),
            "vxh_grid_create_from_floats": (vp, [u, vp, vp, vp]),
            "vxh_grid_create_sphere": (vp, [u, f, f, f, f, C.c_ubyte, C.c_ubyte]),
            "vxh_grid_from_dense": (vp, [u, vp, vp, vp]),
            "vxh_grid_size": (u, [vp]),
            "vxh_grid_to_dense": (None, [vp, vp, vp, vp]),
            "vxh_grid_empty_flags": (C.c_int, [vp, vp]),
            "vxh_grid_inject_sphere": (None, [vp, f, f, f, f, f, C.c_int, vp]),
            "vxh_grid_create_builtin": (vp, [u, vp, f, f, f, f]),
            "vxh_builtin_dense": (None, [u, vp, vp, vp, vp]),
            "vxh_grid_inject_builtin": (None, [vp, vp, vp, vp, C.c_int, vp]),
            "vxh_grid_inject_material": (None, [vp, vp, vp, u, C.c_int, vp]),
            "vxh_grid_pack_size": (u, [vp, C.POINTER(vp)]),
            "vxh_pack_data": (vp, [vp]),
            "vxh_pack_destroy": (None, [vp]),
            "vxh_grid_load": (vp, [vp, u]),
            "vxh_grid_destroy": (None, [vp]),
            "vxh_modification_create": (vp, []),
            "vxh_modification_destroy": (None, [vp]),
            "vxh_modification_blocks": (u, [vp, vp, u]),
            "vxh_polygonize": (vp, [vp, vp, vp, vp, vp, vp, C.POINTER(d)]),
            "vxh_surface_destroy": (None, [vp]),
            "vxh_surface_levels": (u, [vp]),
            "vxh_surface_blocks": (u, [vp, u]),
            "vxh_surface_extents": (None, [vp, vp]),
            "vxh_surface_cache_bytes": (u, [vp]),
            "vxh_surface_polygon_bytes": (u, [vp]),
            "vxh_surface_stats": (None, [vp, vp]),
            "vxh_surface_level_totals": (None, [vp, u, vp]),
            "vxh_surface_level_dump": (None, [vp, u, vp, vp, vp, vp, vp]),
        }
        for name, (res, args) in sig.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = res, args
        err = L.vxh_init()
        if err != 0:
            raise RuntimeError("InitializeVoxels failed: %d" % err)

    # ---- grids ----
    @staticmethod
    def _ptr(a):
        return None if a is None else a.ctypes.data_as(C.c_void_p)

    def grid_from_dense(self, dist, mat=None, blend=None):
        n = dist.shape[0]
        assert dist.shape == (n, n, n) and dist.dtype == np.int8 and dist.flags.c_contiguous
        for a in (mat, blend):
            assert a is None or (a.shape == (n, n, n) and a.dtype == np.uint8 and a.flags.c_contiguous)
        return self.L.vxh_grid_from_dense(n, self._ptr(dist), self._ptr(mat), self._ptr(blend))

    def grid_from_floats(self, dist, mat=None, blend=None):
        n = dist.shape[0]
        assert dist.shape == (n, n, n) and dist.dtype == np.float32 and dist.flags.c_contiguous
        return self.L.vxh_grid_create_from_floats(n, self._ptr(dist), self._ptr(mat), self._ptr(blend))

    def grid_sphere(self, n, center, radius, material=0, blend=0):
        return self.L.vxh_grid_create_sphere(n, center[0], center[1], center[2], radius, material, blend)

    def grid_to_dense(self, grid):
        """(dist, mat, blend) arrays indexed [z, y, x]."""
        n = self.L.vxh_grid_size(grid)
        dist = np.empty((n, n, n), np.int8); mat = np.empty((n, n, n), np.uint8); blend = np.empty((n, n, n), np.uint8)
        self.L.vxh_grid_to_dense(grid, self._ptr(dist), self._ptr(mat), self._ptr(blend))
        return dist, mat, blend

    def grid_empty_flags(self, grid):
        nb = self.L.vxh_grid_size(grid) // 16
        flags = np.zeros(nb ** 3, np.uint8)
        ok = self.L.vxh_grid_empty_flags(grid, self._ptr(flags))
        return flags if ok else None

    def grid_inject_sphere(self, grid, pos, radius, extent, inject_type):
        box = np.zeros(6, np.float32)
        self.L.vxh_grid_inject_sphere(grid, pos[0], pos[1], pos[2], radius, extent, inject_type, self._ptr(box))
        return box

    # ---- built-in procedural surfaces (voxels_b200/csrc/vxb_surfaces.h evaluated on the host, fed to the reference) ----
    def grid_create_builtin(self, n, surface, start=(0.0, 0.0, 0.0), step=1.0):
        """Grid::Create(n, n, n, start, step, &surface) with a capi.Surface."""
        return self.L.vxh_grid_create_builtin(n, C.cast(C.byref(surface), C.c_void_p), start[0], start[1], start[2], step)

    def builtin_dense(self, n, surface):
        """(dist, mat, blend) [z, y, x]: the surface quantised the reference's way, on all host threads."""
        dist = np.empty((n, n, n), np.int8); mat = np.empty((n, n, n), np.uint8); blend = np.empty((n, n, n), np.uint8)
        self.L.vxh_builtin_dense(n, C.cast(C.byref(surface), C.c_void_p), self._ptr(dist), self._ptr(mat), self._ptr(blend))
        return dist, mat, blend

    def grid_inject_builtin(self, grid, pos, ext, surface, inject_type):
        box = np.zeros(6, np.float32)
        p = np.ascontiguousarray(pos, np.float32); e = np.ascontiguousarray(ext, np.float32)
        self.L.vxh_grid_inject_builtin(grid, self._ptr(p), self._ptr(e), C.cast(C.byref(surface), C.c_void_p), inject_type, self._ptr(box))
        return box

    def grid_inject_material(self, grid, pos, ext, material, add_subtract_blend):
        box = np.zeros(6, np.float32)
        p = np.ascontiguousarray(pos, np.float32); e = np.ascontiguousarray(ext, np.float32)
        self.L.vxh_grid_inject_material(grid, self._ptr(p), self._ptr(e), material, 1 if add_subtract_blend else 0, self._ptr(box))
        return box

    def grid_pack(self, grid):
        pack = C.c_void_p()
        size = self.L.vxh_grid_pack_size(grid, C.byref(pack))
        data = C.string_at(self.L.vxh_pack_data(pack), size)
        self.L.vxh_pack_destroy(pack)
        return np.frombuffer(data, np.uint8).copy()

    def grid_load(self, blob):
        """Grid::Load of a PackForSave-format blob (numpy uint8); None when the reference refuses it."""
        blob = np.ascontiguousarray(blob, np.uint8)
        g = self.L.vxh_grid_load(self._ptr(blob), blob.size)
        return g or None

    def grid_destroy(self, grid):
        self.L.vxh_grid_destroy(grid)

    # ---- polygonization ----
    def polygonize(self, grid, material_table=None, valid_mask=None, modification=None, surface=None, box=None,
                   threads=0):
        if threads:
            self.L.vxh_set_threads(threads)
        seconds = C.c_double(0)
        box_arr = None if box is None else np.ascontiguousarray(box, np.float32)
        s = self.L.vxh_polygonize(grid, self._ptr(material_table), self._ptr(valid_mask), modification, surface,
                                  self._ptr(box_arr), C.byref(seconds))
        return s, seconds.value

    def modification_create(self):
        return self.L.vxh_modification_create()

    def modification_blocks(self, mod):
        n = self.L.vxh_modification_blocks(mod, None, 0)
        out = np.zeros(n, np.uint32)
        if n:
            self.L.vxh_modification_blocks(mod, self._ptr(out), n)
        return out

    def modification_destroy(self, mod):
        self.L.vxh_modification_destroy(mod)

    def surface_levels(self, s):
        return self.L.vxh_surface_levels(s)

    def surface_extents(self, s):
        e = np.zeros(3, np.float32)
        self.L.vxh_surface_extents(s, self._ptr(e))
        return e

    def surface_stats(self, s):
        st = np.zeros(20, np.uint32)
        self.L.vxh_surface_stats(s, self._ptr(st))
        return st

    def surface_level(self, s, level):
        nb = self.L.vxh_surface_blocks(s, level)
        totals = np.zeros(4, np.uint64)
        self.L.vxh_surface_level_totals(s, level, self._ptr(totals))
        rows = np.zeros(nb, ROW_DTYPE)
        verts = np.zeros(int(totals[0]), VERTEX_DTYPE); idx = np.zeros(int(totals[1]), np.uint32)
        tverts = np.zeros(int(totals[2]), VERTEX_DTYPE); tidx = np.zeros(int(totals[3]), np.uint32)
        self.L.vxh_surface_level_dump(s, level, self._ptr(rows), self._ptr(verts), self._ptr(idx), self._ptr(tverts),
                                      self._ptr(tidx))
        return LevelDump(rows, verts, idx, tverts, tidx)

    def surface_destroy(self, s):
        self.L.vxh_surface_destroy(s)


_libs = {}


def load(path):
    if path not in _libs:
        _libs[path] = VoxelsLib(path)
    return _libs[path]


def reference():
    return load(REF_LIB)
