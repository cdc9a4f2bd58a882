"""ctypes driver for the SDF-program harness (tests/harness/vxh_programs.cpp, test infrastructure).

oracle/_ref/libvxh_programs_ref.so (oracle/programs.mk) is vxh_capi.cpp + vxh_programs.cpp over the UNMODIFIED reference, so
`ProgramLib` is a harness.VoxelsLib - every grid / polygonization call of the parity tests - plus the program calls:
Grid::Create / Grid::InjectSurface with a ProgramSurface serving voxels_b200/csrc/vxb_program.h, the multi-threaded host
generator of a program fill and the fill's per-block cull decision computed on the host.
"""
import ctypes as C
import os

import numpy as np

import harness

PROGRAMS_LIB = os.path.join(harness.REPO, "oracle", "_ref", "libvxh_programs_ref.so")


class ProgramLib(harness.VoxelsLib):
    def __init__(self, path):
        super().__init__(path)
        vp, u, f = C.c_void_p, C.c_uint, C.c_float
        sig = {
            "vxh_program_validate": (C.c_int, [vp, u]),
            "vxh_grid_create_program": (vp, [u, vp, u, f, f, f, f]),
            "vxh_grid_inject_program": (None, [vp, vp, vp, vp, u, C.c_int, vp]),
            "vxh_program_dense": (None, [u, vp, u, vp, f, vp, vp, vp]),
            "vxh_program_cull_flags": (u, [u, vp, u, vp, f, vp, vp]),
        }
        for name, (res, args) in sig.items():
            fn = getattr(self.L, name)
            fn.restype, fn.argtypes = res, args

    @staticmethod
    def _program(ops):
        from voxels_b200 import capi
        arr = capi.program_array(ops)
        return C.cast(arr, C.c_void_p), len(arr), arr

    def program_validate(self, ops):
        """-1 for a well-formed program, else the index of the op the library names."""
        p, count, _keep = self._program(ops)
        return self.L.vxh_program_validate(p, count)

    def grid_create_program(self, n, ops, start=(0.0, 0.0, 0.0), step=1.0):
        """Grid::Create(n, n, n, start, step, &ProgramSurface)."""
        p, count, _keep = self._program(ops)
        return self.L.vxh_grid_create_program(n, p, count, start[0], start[1], start[2], step)

    def grid_inject_program(self, grid, pos, ext, ops, inject_type):
        """Grid::InjectSurface(pos, ext, &ProgramSurface, type); returns the box the reference returns."""
        box = np.zeros(6, np.float32)
        pa = np.ascontiguousarray(pos, np.float32); e = np.ascontiguousarray(ext, np.float32)
        p, count, _keep = self._program(ops)
        self.L.vxh_grid_inject_program(grid, self._ptr(pa), self._ptr(e), p, count, inject_type, self._ptr(box))
        return box

    def program_dense(self, n, ops, start=(0.0, 0.0, 0.0), step=1.0):
        """(dist, mat, blend) [z, y, x]: what a fill with the program writes, on all host threads."""
        dist = np.empty((n, n, n), np.int8); mat = np.empty((n, n, n), np.uint8); blend = np.empty((n, n, n), np.uint8)
        st = np.ascontiguousarray(start, np.float32)
        p, count, _keep = self._program(ops)
        self.L.vxh_program_dense(n, p, count, self._ptr(st), step, self._ptr(dist), self._ptr(mat), self._ptr(blend))
        return dist, mat, blend

    def program_cull_flags(self, n, ops, start=(0.0, 0.0, 0.0), step=1.0):
        """The fill's per-block cull decision on the host: (flags [nb^3] 1 = constant block, values [nb^3, 4] = its
        {distance, material, blend, 0}), VoxelGrid block order."""
        nb = n // 16
        flags = np.zeros(nb ** 3, np.uint8); values = np.zeros((nb ** 3, 4), np.int32)
        st = np.ascontiguousarray(start, np.float32)
        p, count, _keep = self._program(ops)
        self.L.vxh_program_cull_flags(n, p, count, self._ptr(st), step, self._ptr(flags), self._ptr(values))
        return flags, values


_lib = None


def load():
    """The program harness, or None when it has not been built (it needs the reference checkout: oracle/programs.mk)."""
    global _lib
    if _lib is None and os.path.exists(PROGRAMS_LIB):
        _lib = ProgramLib(PROGRAMS_LIB)
    return _lib
