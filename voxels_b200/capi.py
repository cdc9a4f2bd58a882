"""ctypes binding of include/vxb200.h (libvxb200.so).  Mirrors the C ABI one to one."""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
FLAG_NO_TRANSITIONS = 1
FLAG_KERNEL_TIMES = 2

VERTEX_DTYPE = np.dtype([("pos", "<f4", 3), ("sec", "<f4", 4), ("nrm", "<f4", 3), ("tex", "u1", 8)])
RECORD_DTYPE = np.dtype([("level", "<u4"), ("coord_id", "<u4"), ("id", "<u4"), ("vertex_count", "<u4"),
                         ("index_count", "<u4"), ("vertex_offset", "<u4"), ("index_offset", "<u4"),
                         ("trans_vertex_count", "<u4", 6), ("trans_index_count", "<u4", 6),
                         ("trans_vertex_offset", "<u4", 6), ("trans_index_offset", "<u4", 6), ("reserved", "<u4")])
assert VERTEX_DTYPE.itemsize == 48 and RECORD_DTYPE.itemsize == 128

# what tests/harness.py calls a block row (the reference-facing view of a block)
ROW_DTYPE = np.dtype([("id", "<u4"), ("min", "<f4", 3), ("max", "<f4", 3), ("nv", "<u4"), ("ni", "<u4"),
                      ("tnv", "<u4", 6), ("tni", "<u4", 6)])


class ResultInfo(C.Structure):
    _fields_ = [("levels_total", C.c_uint32), ("levels_computed", C.c_uint32), ("block_count", C.c_uint32),
                ("pad", C.c_uint32), ("vertex_span", C.c_uint64), ("index_span", C.c_uint64),
                ("trans_vertex_span", C.c_uint64), ("trans_index_span", C.c_uint64), ("vertex_total", C.c_uint64),
                ("index_total", C.c_uint64), ("trans_vertex_total", C.c_uint64), ("trans_index_total", C.c_uint64),
                ("stats", C.c_uint32 * 20), ("used_materials", C.c_uint32 * 8), ("device_ms", C.c_float),
                ("kernel_launches", C.c_uint32)]


class RegionInfo(C.Structure):
    _fields_ = [("levels", C.c_uint32), ("pad", C.c_uint32), ("min_dirty", (C.c_float * 3) * 12), ("max_dirty", (C.c_float * 3) * 12),
                ("id_start", C.c_uint32 * 12), ("block_count", C.c_uint32 * 12)]


class ShardBuffers(C.Structure):
    _fields_ = [("block_info", C.c_void_p), ("block_info_bytes", C.c_uint64), ("chunk_bytes", C.c_uint64), ("pages", C.c_void_p),
                ("pages_bytes", C.c_uint64), ("valid", C.c_void_p), ("valid_bytes", C.c_uint64), ("super_level", C.c_uint32),
                ("pad", C.c_uint32)]


class Surface(C.Structure):
    """vxb_surface (include/vxb200.h): a built-in procedural surface."""
    _fields_ = [("kind", C.c_uint32), ("material", C.c_uint32), ("blend", C.c_uint32), ("seed", C.c_uint32), ("p", C.c_float * 8)]

    @staticmethod
    def sphere(center, radius, material=0, blend=0):
        s = Surface(); s.kind = 0; s.material = material; s.blend = blend
        s.p[0], s.p[1], s.p[2], s.p[3] = center[0], center[1], center[2], radius
        return s

    @staticmethod
    def plane(normal, d0, material=0, blend=0):
        s = Surface(); s.kind = 1; s.material = material; s.blend = blend
        s.p[0], s.p[1], s.p[2], s.p[3] = normal[0], normal[1], normal[2], d0
        return s

    @staticmethod
    def terrain(period, origin=(0.0, 0.0), seed=1234):
        s = Surface(); s.kind = 2; s.seed = seed
        s.p[0], s.p[1], s.p[2] = float(period), float(origin[0]), float(origin[1])
        return s


OP_SPHERE, OP_BOX, OP_CYLINDER, OP_CAPSULE, OP_TORUS, OP_PLANE, OP_TERRAIN = range(7)
OP_UNION, OP_INTERSECT, OP_SUBTRACT, OP_SMOOTH_UNION = range(16, 20)
OP_OFFSET, OP_SHELL = 32, 33
PROGRAM_MAX_OPS, PROGRAM_MAX_DEPTH, PROGRAM_MAX_TERRAIN = 64, 8, 2


class Op(C.Structure):
    """vxb_op (include/vxb200.h): one instruction of an SDF program.  Primitives take their placement as `at` (the local
    origin in grid coordinates) and `rotation` (3x3, local -> grid axes; any invertible matrix, so scales and shears too):
    the stored transform is local = inverse(rotation) (p - at).  `xform` (12 floats, rows {m0, m1, m2, t}) overrides both."""
    _fields_ = [("code", C.c_uint32), ("material", C.c_uint32), ("blend", C.c_uint32), ("seed", C.c_uint32),
                ("xform", C.c_float * 12), ("p", C.c_float * 8)]

    @staticmethod
    def _make(code, params=(), at=None, rotation=None, xform=None, material=0, blend=0, seed=0):
        o = Op()
        o.code, o.material, o.blend, o.seed = code, material, blend, seed
        for k, v in enumerate(params):
            o.p[k] = v
        if code < 16:
            if xform is None:
                m = np.eye(3) if rotation is None else np.linalg.inv(np.asarray(rotation, np.float64))
                c = np.zeros(3) if at is None else np.asarray(at, np.float64)
                xform = np.concatenate([m.ravel(), -(m @ c)])
            for k, v in enumerate(np.asarray(xform, np.float32).ravel()):
                o.xform[k] = float(v)
        return o

    @staticmethod
    def sphere(radius, at=None, rotation=None, material=0, blend=0, xform=None):
        return Op._make(OP_SPHERE, (radius,), at, rotation, xform, material, blend)

    @staticmethod
    def box(half, at=None, rotation=None, material=0, blend=0, xform=None):
        return Op._make(OP_BOX, tuple(half), at, rotation, xform, material, blend)

    @staticmethod
    def cylinder(radius, half_height, at=None, rotation=None, material=0, blend=0, xform=None):
        return Op._make(OP_CYLINDER, (radius, half_height), at, rotation, xform, material, blend)

    @staticmethod
    def capsule(radius, half_length, at=None, rotation=None, material=0, blend=0, xform=None):
        return Op._make(OP_CAPSULE, (radius, half_length), at, rotation, xform, material, blend)

    @staticmethod
    def torus(ring, tube, at=None, rotation=None, material=0, blend=0, xform=None):
        return Op._make(OP_TORUS, (ring, tube), at, rotation, xform, material, blend)

    @staticmethod
    def plane(normal, d0, at=None, rotation=None, material=0, blend=0, xform=None):
        return Op._make(OP_PLANE, (normal[0], normal[1], normal[2], d0), at, rotation, xform, material, blend)

    @staticmethod
    def terrain(period, origin=(0.0, 0.0), seed=1234, at=None, rotation=None, xform=None):
        return Op._make(OP_TERRAIN, (float(period), float(origin[0]), float(origin[1])), at, rotation, xform, seed=seed)

    @staticmethod
    def union():
        return Op._make(OP_UNION)

    @staticmethod
    def intersect():
        return Op._make(OP_INTERSECT)

    @staticmethod
    def subtract():
        return Op._make(OP_SUBTRACT)

    @staticmethod
    def smooth_union(k):
        return Op._make(OP_SMOOTH_UNION, (k,))

    @staticmethod
    def offset(r):
        return Op._make(OP_OFFSET, (r,))

    @staticmethod
    def shell(thickness):
        return Op._make(OP_SHELL, (thickness,))


def program_array(ops):
    """A list of Op as the contiguous vxb_op array the C ABI takes (also accepts such an array)."""
    if isinstance(ops, C.Array):
        return ops
    return (Op * len(ops))(*ops)


class ProgramStats(C.Structure):
    _fields_ = [("blocks", C.c_uint64), ("culled", C.c_uint64), ("pass_a_ms", C.c_float), ("pass_b_ms", C.c_float)]


class DrawLists(C.Structure):
    _fields_ = [("regular_count", C.c_uint32), ("transition_count", C.c_uint32), ("counts", C.c_void_p), ("regular", C.c_void_p),
                ("regular_info", C.c_void_p), ("transition", C.c_void_p), ("transition_info", C.c_void_p)]


DRAW_COMMAND_DTYPE = np.dtype([("index_count", "<u4"), ("instance_count", "<u4"), ("first_index", "<u4"), ("base_vertex", "<i4"), ("first_instance", "<u4")])
DRAW_INFO_DTYPE = np.dtype([("block_id", "<u4"), ("level", "<u4"), ("block_adj", "<u4"), ("face", "<u4")])

# vxb_ray / vxb_ray_hit (include/vxb200.h "ray queries")
VXB_RAY_MISS = 0xFFFFFFFF
RAY_DTYPE = np.dtype([("origin", "<f4", 3), ("t_min", "<f4"), ("direction", "<f4", 3), ("t_max", "<f4")])
RAY_HIT_DTYPE = np.dtype([("t", "<f4"), ("u", "<f4"), ("v", "<f4"), ("slot", "<u4"), ("block_id", "<u4"), ("triangle", "<u4"),
                          ("position", "<f4", 3), ("normal", "<f4", 3)])
assert RAY_DTYPE.itemsize == 32 and RAY_HIT_DTYPE.itemsize == 48
# vxb_cut_hit (include/vxb200.h "ray queries against the drawn LOD cut"): vxb_ray_hit's 48 bytes, then level and face
CUT_HIT_DTYPE = np.dtype(RAY_HIT_DTYPE.descr + [("level", "<u4"), ("face", "<u4")])
CUT_FACE_REGULAR = 0xFFFFFFFF
assert CUT_HIT_DTYPE.itemsize == 56


def make_rays(origins, directions, t_min=0.0, t_max=np.inf):
    """A RAY_DTYPE array from [count, 3] origins and directions (OUTPUT, Y-up coordinates); t_min / t_max: scalars or [count]."""
    o = np.asarray(origins, np.float32).reshape(-1, 3)
    d = np.asarray(directions, np.float32).reshape(-1, 3)
    rays = np.zeros(len(o), RAY_DTYPE)
    rays["origin"], rays["direction"] = o, d
    rays["t_min"], rays["t_max"] = np.float32(t_min) if np.isscalar(t_min) else np.asarray(t_min, np.float32), \
        np.float32(t_max) if np.isscalar(t_max) else np.asarray(t_max, np.float32)
    return rays


# vxb_sphere_hit / vxb_closest_hit (include/vxb200.h "collision queries")
VXB_SPHERE_RADIUS_MAX = 15.0
VXB_SPHERE_STARTED_IN_CONTACT = 1
SPHERE_HIT_DTYPE = np.dtype([("t", "<f4"), ("slot", "<u4"), ("block_id", "<u4"), ("triangle", "<u4"), ("center", "<f4", 3),
                             ("point", "<f4", 3), ("normal", "<f4", 3), ("u", "<f4"), ("v", "<f4"), ("flags", "<u4")])
CLOSEST_HIT_DTYPE = np.dtype([("distance", "<f4"), ("slot", "<u4"), ("block_id", "<u4"), ("triangle", "<u4"), ("point", "<f4", 3),
                              ("normal", "<f4", 3), ("u", "<f4"), ("v", "<f4")])
assert SPHERE_HIT_DTYPE.itemsize == 64 and CLOSEST_HIT_DTYPE.itemsize == 48
# vxb_sphere_cut_hit / vxb_closest_cut_hit (include/vxb200.h "collision queries against the drawn LOD cut"): the level-0 hits,
# then level and face
SPHERE_CUT_HIT_DTYPE = np.dtype(SPHERE_HIT_DTYPE.descr + [("level", "<u4"), ("face", "<u4")])
CLOSEST_CUT_HIT_DTYPE = np.dtype(CLOSEST_HIT_DTYPE.descr + [("level", "<u4"), ("face", "<u4")])
assert SPHERE_CUT_HIT_DTYPE.itemsize == 72 and CLOSEST_CUT_HIT_DTYPE.itemsize == 56

# vxb_capsule_sweep / vxb_segment / vxb_capsule_hit / vxb_segment_hit (include/vxb200.h "capsule queries")
CAPSULE_SWEEP_DTYPE = np.dtype([("path", RAY_DTYPE), ("half_axis", "<f4", 3), ("radius", "<f4")])
SEGMENT_DTYPE = np.dtype([("center", "<f4", 3), ("half_axis", "<f4", 3)])
CAPSULE_HIT_DTYPE = np.dtype([("t", "<f4"), ("slot", "<u4"), ("block_id", "<u4"), ("triangle", "<u4"), ("center", "<f4", 3),
                              ("point", "<f4", 3), ("axis_point", "<f4", 3), ("normal", "<f4", 3), ("u", "<f4"), ("v", "<f4"),
                              ("s", "<f4"), ("flags", "<u4")])
SEGMENT_HIT_DTYPE = np.dtype([("distance", "<f4"), ("slot", "<u4"), ("block_id", "<u4"), ("triangle", "<u4"), ("point", "<f4", 3),
                              ("axis_point", "<f4", 3), ("normal", "<f4", 3), ("u", "<f4"), ("v", "<f4"), ("s", "<f4")])
assert CAPSULE_SWEEP_DTYPE.itemsize == 48 and SEGMENT_DTYPE.itemsize == 24
assert CAPSULE_HIT_DTYPE.itemsize == 80 and SEGMENT_HIT_DTYPE.itemsize == 64
# vxb_capsule_cut_hit / vxb_segment_cut_hit (include/vxb200.h "capsule queries against the drawn LOD cut"): the level-0 hits,
# then level and face
CAPSULE_CUT_HIT_DTYPE = np.dtype(CAPSULE_HIT_DTYPE.descr + [("level", "<u4"), ("face", "<u4")])
SEGMENT_CUT_HIT_DTYPE = np.dtype(SEGMENT_HIT_DTYPE.descr + [("level", "<u4"), ("face", "<u4")])
assert CAPSULE_CUT_HIT_DTYPE.itemsize == 88 and SEGMENT_CUT_HIT_DTYPE.itemsize == 72

# vxb_box / vxb_overlap_triangle (include/vxb200.h "box overlap gathers")
BOX_DTYPE = np.dtype([("min", "<f4", 3), ("max", "<f4", 3)])
OVERLAP_TRIANGLE_DTYPE = np.dtype([("p", "<f4", (3, 3)), ("slot", "<u4"), ("block_id", "<u4"), ("triangle", "<u4")])
assert BOX_DTYPE.itemsize == 24 and OVERLAP_TRIANGLE_DTYPE.itemsize == 48


def make_boxes(mins, maxs):
    """A BOX_DTYPE array from [count, 3] minima and maxima (OUTPUT, Y-up coordinates)."""
    lo = np.asarray(mins, np.float32).reshape(-1, 3)
    boxes = np.zeros(len(lo), BOX_DTYPE)
    boxes["min"], boxes["max"] = lo, np.asarray(maxs, np.float32).reshape(-1, 3)
    return boxes


def make_capsule_sweeps(origins, directions, half_axes, radius, t_min=0.0, t_max=np.inf):
    """A CAPSULE_SWEEP_DTYPE array: the centre paths as make_rays, `half_axes` [count, 3] or [3], `radius` a scalar or [count]."""
    rays = make_rays(origins, directions, t_min, t_max)
    sweeps = np.zeros(len(rays), CAPSULE_SWEEP_DTYPE)
    sweeps["path"] = rays
    sweeps["half_axis"] = np.broadcast_to(np.asarray(half_axes, np.float32), (len(rays), 3))
    sweeps["radius"] = np.float32(radius) if np.isscalar(radius) else np.asarray(radius, np.float32)
    return sweeps


def make_segments(centers, half_axes):
    """A SEGMENT_DTYPE array from [count, 3] centres and [count, 3] (or [3]) half axes."""
    c = np.asarray(centers, np.float32).reshape(-1, 3)
    segs = np.zeros(len(c), SEGMENT_DTYPE)
    segs["center"] = c
    segs["half_axis"] = np.broadcast_to(np.asarray(half_axes, np.float32), (len(c), 3))
    return segs


class MeshInfo(C.Structure):
    """vxb_mesh_info (include/vxb200.h)."""
    _fields_ = [("levels", C.c_uint32), ("block_count", C.c_uint32), ("level_blocks", C.c_uint32 * 12), ("vertex_span", C.c_uint64),
                ("index_span", C.c_uint64), ("trans_vertex_span", C.c_uint64), ("trans_index_span", C.c_uint64),
                ("vertex_total", C.c_uint64), ("index_total", C.c_uint64), ("trans_vertex_total", C.c_uint64),
                ("trans_index_total", C.c_uint64), ("capacity", C.c_uint64 * 4), ("stats", C.c_uint32 * 20),
                ("compactions", C.c_uint32), ("growths", C.c_uint32), ("generation", C.c_uint64), ("bytes_copied", C.c_uint64),
                ("apply_ms", C.c_float), ("pad", C.c_uint32)]


VXB_VIEWS_MAX = 8
VXB_LOD_FACTOR_MIN = 2.0


class View(C.Structure):
    """vxb_view (include/vxb200.h "culled select"): six planes {nx, ny, nz, d} in OUTPUT coordinates, pointing into the view."""
    _fields_ = [("planes", (C.c_float * 4) * 6)]


class MeshBounds(C.Structure):
    """vxb_mesh_bounds (include/vxb200.h "bounds")."""
    _fields_ = [("boxes", C.c_void_p), ("level_base", C.c_uint32 * 12), ("slots", C.c_uint32), ("pad", C.c_uint32)]


def make_views(planes):
    """A View array from [views, 6, 4] plane coefficients."""
    p = np.ascontiguousarray(planes, np.float32).reshape(-1, 6, 4)
    views = (View * len(p))()
    C.memmove(views, p.ctypes.data, p.nbytes)
    return views


class NcclId(C.Structure):
    _fields_ = [("internal", C.c_char * 128)]


ERR_STATE = -3
ERR_CAPACITY = -4

# vxb_pack_producer (include/vxb200.h): void (*)(void* user, uint32_t layer0, uint32_t layer1)
PackProducer = C.CFUNCTYPE(None, C.c_void_p, C.c_uint32, C.c_uint32)


class DevicePointer:
    """A raw device range as a CUDA-array-interface object: torch.as_tensor(DevicePointer(p, nbytes), device=...) is a
    zero-copy uint8 view (how dist.py hands the exchange buffers of a sharded run to torch.distributed)."""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (int(nbytes),), "typestr": "|u1", "data": (int(ptr), False), "version": 3,
                                         "strides": None}


class VxbError(RuntimeError):
    pass


def library_path():
    return os.path.join(_HERE, "lib", "libvxb200.so")


_lib = None


def load_library():
    """Loads libvxb200.so; raises (never falls back) when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    path = library_path()
    if not os.path.exists(path):
        raise VxbError("%s is missing - run `python -c 'import __graft_entry__ as g; g.build()'` (needs nvcc); "
                       "there is no CPU fallback" % path)
    L = C.CDLL(path)
    vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
    sig = {
        "vxb_create": (C.c_int, [C.c_int, C.POINTER(vp)]),
        "vxb_destroy": (None, [vp]),
        "vxb_last_error": (C.c_char_p, [vp]),
        "vxb_stream": (vp, [vp]),
        "vxb_exchange_stream": (vp, [vp]),
        "vxb_grid_upload_dense": (C.c_int, [vp, u32, vp, vp, vp]),
        "vxb_grid_upload_blocks": (C.c_int, [vp, u32, vp, vp, vp]),
        "vxb_grid_set_device": (C.c_int, [vp, u32, vp, vp, vp]),
        "vxb_grid_upload_packed": (C.c_int, [vp, vp, C.c_size_t]),
        "vxb_grid_upload_packed_streamed": (C.c_int, [vp, vp, C.c_size_t, PackProducer, vp]),
        "vxb_result_download_begin": (C.c_int, [vp, vp, vp, vp, vp, vp]),
        "vxb_result_download_end": (C.c_int, [vp]),
        "vxb_pack_dense_bound": (C.c_size_t, [u32]),
        "vxb_pack_dense": (C.c_int, [u32, vp, vp, vp, vp, C.c_size_t, C.POINTER(C.c_size_t)]),
        "vxb_grid_device_pointers": (C.c_int, [vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)]),
        "vxb_set_materials": (C.c_int, [vp, vp, vp]),
        "vxb_grid_fill": (C.c_int, [vp, u32, C.POINTER(Surface), vp, C.c_float]),
        "vxb_grid_inject_surface": (C.c_int, [vp, vp, vp, C.POINTER(Surface), C.c_int, vp, vp]),
        "vxb_grid_inject_material": (C.c_int, [vp, vp, vp, u32, C.c_int, vp, vp]),
        "vxb_grid_pack": (C.c_int, [vp, vp, C.c_size_t, C.POINTER(C.c_size_t)]),
        "vxb_grid_download_dense": (C.c_int, [vp, vp, vp, vp]),
        "vxb_grid_fill_program": (C.c_int, [vp, u32, vp, u32, vp, C.c_float]),
        "vxb_grid_inject_program": (C.c_int, [vp, vp, vp, vp, u32, C.c_int, vp, vp]),
        "vxb_grid_program_stats": (C.c_int, [vp, C.POINTER(ProgramStats)]),
        "vxb_result_device_arenas": (C.c_int, [vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)]),
        "vxb_result_select_lod": (C.c_int, [vp, vp, C.c_float, C.POINTER(DrawLists)]),
        "vxb_result_download_draws": (C.c_int, [vp, vp, vp, vp, vp]),
        "vxb_polygonize": (C.c_int, [vp, u32, u32]),
        "vxb_result_info_get": (C.c_int, [vp, C.POINTER(ResultInfo)]),
        "vxb_grid_update_blocks": (C.c_int, [vp, u32, vp, vp, vp, vp]),
        "vxb_polygonize_region": (C.c_int, [vp, vp, vp, u32]),
        "vxb_region_info_get": (C.c_int, [vp, C.POINTER(RegionInfo)]),
        "vxb_polygonize_sharded": (C.c_int, [vp, u32, u32]),
        "vxb_shard_configure": (C.c_int, [vp, u32, u32, u32]),
        "vxb_shard_buffers_get": (C.c_int, [vp, C.POINTER(ShardBuffers)]),
        "vxb_shard_set_peer": (C.c_int, [vp, u32, vp, vp]),
        "vxb_shard_export": (C.c_int, [vp, C.POINTER(C.c_int)]),
        "vxb_shard_import": (C.c_int, [vp, u32, C.c_int]),
        "vxb_shard_nccl_unique_id": (C.c_int, [C.POINTER(NcclId)]),
        "vxb_shard_nccl_init": (C.c_int, [vp, C.POINTER(NcclId), u32, u32]),
        "vxb_cube_create": (C.c_int, [vp, u32, u32, u32, u32]),
        "vxb_cube_info": (C.c_int, [vp, C.POINTER(u32), C.POINTER(u32), C.POINTER(u64 * 4)]),
        "vxb_cube_export": (C.c_int, [vp, u32, u32, C.POINTER(C.c_int)]),
        "vxb_cube_import": (C.c_int, [vp, u32, u32, C.c_int]),
        "vxb_cube_piece": (C.c_int, [vp, u32, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(u64)]),
        "vxb_result_download": (C.c_int, [vp, vp, vp, vp, vp, vp]),
        "vxb_set_capacity": (C.c_int, [vp, u64, u64, u64, u64]),
        "vxb_set_launch_limit": (C.c_int, [vp, u32]),
        "vxb_run_work_items": (C.c_int, [vp, u32, C.POINTER(u32), C.POINTER(u32)]),
        "vxb_kernel_ms": (C.c_int, [vp, C.c_int, C.POINTER(C.c_float), C.POINTER(u32)]),
        "vxb_result_unmapped_materials": (u64, [vp, vp, u64]),
        "vxb_mesh_create": (C.c_int, [vp, vp, C.POINTER(vp)]),
        "vxb_mesh_destroy": (None, [vp]),
        "vxb_mesh_apply": (C.c_int, [vp]),
        "vxb_mesh_info_get": (C.c_int, [vp, C.POINTER(MeshInfo)]),
        "vxb_mesh_download": (C.c_int, [vp, vp, vp, vp, vp, vp]),
        "vxb_mesh_device_arenas": (C.c_int, [vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp)]),
        "vxb_mesh_select_lod": (C.c_int, [vp, vp, C.c_float, C.POINTER(DrawLists)]),
        "vxb_mesh_bounds_get": (C.c_int, [vp, C.POINTER(MeshBounds)]),
        "vxb_mesh_download_bounds": (C.c_int, [vp, vp]),
        "vxb_mesh_select_lod_views": (C.c_int, [vp, vp, C.c_float, vp, u32, vp]),
        "vxb_mesh_select_cut": (C.c_int, [vp, vp, C.c_float, vp, u32, vp]),
        "vxb_mesh_raycast": (C.c_int, [vp, vp, u32, vp]),
        "vxb_mesh_raycast_device": (C.c_int, [vp, vp, u32, vp]),
        "vxb_mesh_raycast_cut": (C.c_int, [vp, vp, C.c_float, vp, u32, vp]),
        "vxb_mesh_raycast_cut_device": (C.c_int, [vp, vp, C.c_float, vp, u32, vp]),
        "vxb_mesh_sphere_cast": (C.c_int, [vp, C.c_float, vp, u32, vp]),
        "vxb_mesh_sphere_cast_device": (C.c_int, [vp, C.c_float, vp, u32, vp]),
        "vxb_mesh_closest_point": (C.c_int, [vp, C.c_float, vp, u32, vp]),
        "vxb_mesh_closest_point_device": (C.c_int, [vp, C.c_float, vp, u32, vp]),
        "vxb_mesh_sphere_cast_cut": (C.c_int, [vp, vp, C.c_float, C.c_float, vp, u32, vp]),
        "vxb_mesh_sphere_cast_cut_device": (C.c_int, [vp, vp, C.c_float, C.c_float, vp, u32, vp]),
        "vxb_mesh_closest_point_cut": (C.c_int, [vp, vp, C.c_float, C.c_float, vp, u32, vp]),
        "vxb_mesh_closest_point_cut_device": (C.c_int, [vp, vp, C.c_float, C.c_float, vp, u32, vp]),
        "vxb_mesh_capsule_cast": (C.c_int, [vp, vp, u32, vp]),
        "vxb_mesh_capsule_cast_device": (C.c_int, [vp, vp, u32, vp]),
        "vxb_mesh_closest_to_segment": (C.c_int, [vp, C.c_float, vp, u32, vp]),
        "vxb_mesh_closest_to_segment_device": (C.c_int, [vp, C.c_float, vp, u32, vp]),
        "vxb_mesh_capsule_cast_cut": (C.c_int, [vp, vp, C.c_float, vp, u32, vp]),
        "vxb_mesh_capsule_cast_cut_device": (C.c_int, [vp, vp, C.c_float, vp, u32, vp]),
        "vxb_mesh_closest_to_segment_cut": (C.c_int, [vp, vp, C.c_float, C.c_float, vp, u32, vp]),
        "vxb_mesh_closest_to_segment_cut_device": (C.c_int, [vp, vp, C.c_float, C.c_float, vp, u32, vp]),
        "vxb_mesh_overlap_box": (C.c_int, [vp, vp, u32, vp, vp, u64]),
        "vxb_mesh_overlap_box_device": (C.c_int, [vp, vp, u32, vp, vp, u64]),
        "vxb_host_alloc": (vp, [C.c_size_t]),
        "vxb_host_free": (None, [vp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)  # AttributeError = a symbol include/vxb200.h declares is not exported
        fn.restype, fn.argtypes = res, args
    _lib = L
    return L


EXPORTED_SYMBOLS = ["vxb_create", "vxb_destroy", "vxb_last_error", "vxb_stream", "vxb_exchange_stream", "vxb_grid_upload_dense",
                    "vxb_grid_upload_blocks", "vxb_grid_upload_packed", "vxb_pack_dense_bound", "vxb_pack_dense", "vxb_grid_set_device", "vxb_grid_device_pointers", "vxb_set_materials",
                    "vxb_polygonize", "vxb_polygonize_region", "vxb_region_info_get", "vxb_grid_update_blocks", "vxb_result_info_get", "vxb_result_download", "vxb_set_capacity", "vxb_set_launch_limit", "vxb_run_work_items", "vxb_kernel_ms",
                    "vxb_result_unmapped_materials", "vxb_host_alloc", "vxb_host_free", "vxb_polygonize_sharded", "vxb_shard_configure",
                    "vxb_shard_buffers_get", "vxb_shard_set_peer", "vxb_shard_export", "vxb_shard_import", "vxb_shard_nccl_unique_id",
                    "vxb_shard_nccl_init", "vxb_grid_fill", "vxb_grid_inject_surface", "vxb_grid_inject_material", "vxb_grid_pack",
                    "vxb_grid_download_dense", "vxb_result_device_arenas", "vxb_result_select_lod", "vxb_result_download_draws", "vxb_cube_create", "vxb_cube_info", "vxb_cube_export", "vxb_cube_import", "vxb_cube_piece",
                    "vxb_grid_upload_packed_streamed", "vxb_result_download_begin", "vxb_result_download_end",
                    "vxb_grid_fill_program", "vxb_grid_inject_program", "vxb_grid_program_stats",
                    "vxb_mesh_create", "vxb_mesh_destroy", "vxb_mesh_apply", "vxb_mesh_info_get", "vxb_mesh_download",
                    "vxb_mesh_device_arenas", "vxb_mesh_select_lod", "vxb_mesh_bounds_get", "vxb_mesh_download_bounds",
                    "vxb_mesh_select_lod_views", "vxb_mesh_select_cut", "vxb_mesh_raycast", "vxb_mesh_raycast_device",
                    "vxb_mesh_raycast_cut", "vxb_mesh_raycast_cut_device",
                    "vxb_mesh_sphere_cast", "vxb_mesh_sphere_cast_device", "vxb_mesh_closest_point", "vxb_mesh_closest_point_device",
                    "vxb_mesh_sphere_cast_cut", "vxb_mesh_sphere_cast_cut_device", "vxb_mesh_closest_point_cut",
                    "vxb_mesh_closest_point_cut_device",
                    "vxb_mesh_capsule_cast", "vxb_mesh_capsule_cast_device", "vxb_mesh_closest_to_segment",
                    "vxb_mesh_closest_to_segment_device", "vxb_mesh_capsule_cast_cut", "vxb_mesh_capsule_cast_cut_device",
                    "vxb_mesh_closest_to_segment_cut", "vxb_mesh_closest_to_segment_cut_device", "vxb_mesh_overlap_box",
                    "vxb_mesh_overlap_box_device"]


def nccl_unique_id():
    """128 bytes from ncclGetUniqueId (through libvxb200.so's dlopen of libnccl.so.2)."""
    L = load_library()
    nid = NcclId()
    rc = L.vxb_shard_nccl_unique_id(C.byref(nid))
    if rc != 0:
        raise VxbError("vxb_shard_nccl_unique_id failed (%d): %s" % (rc, L.vxb_last_error(None).decode()))
    return bytes(C.string_at(C.byref(nid), 128))


def _ptr(a):
    if a is None:
        return None
    if isinstance(a, int):
        return C.c_void_p(a)
    return a.ctypes.data_as(C.c_void_p)


def _dev(p):  # a device address (e.g. a torch tensor's data_ptr()), or None for a NULL pointer
    return None if p is None else C.c_void_p(p)


def _batch(a, dtype):  # a host batch as a contiguous `dtype` array, or None for a NULL pointer
    return None if a is None else np.ascontiguousarray(a, dtype)


def pack_dense(dist, mat, blend, out=None):
    """Host helper: the reference's PackForSave bytes for dense [z,y,x] volumes (numpy uint8 array).  No GPU needed."""
    L = load_library()
    n = dist.shape[0]
    bound = L.vxb_pack_dense_bound(n)
    buf = np.empty(bound, np.uint8) if out is None else out
    written = C.c_size_t(0)
    rc = L.vxb_pack_dense(n, _ptr(dist), _ptr(mat), _ptr(blend), _ptr(buf), buf.size, C.byref(written))
    if rc != 0:
        raise VxbError("vxb_pack_dense failed (%d)" % rc)
    return buf[:written.value]


class LevelView:
    """One LOD level in the layout tests/harness.LevelDump uses (rows + concatenated arrays, block order)."""

    def __init__(self, rows, verts, idx, tverts, tidx):
        self.rows, self.verts, self.idx, self.tverts, self.tidx = rows, verts, idx, tverts, tidx


class Result:
    def __init__(self, n, info, records, verts, idx, tverts, tidx):
        self.n, self.info, self.records = n, info, records
        self.verts, self.idx, self.tverts, self.tidx = verts, idx, tverts, tidx
        self.stats = np.array(list(info.stats), np.uint32)

    def level(self, level):
        recs = self.records[self.records["level"] == level]
        m = 16 << level
        nb = self.n // m
        rows = np.zeros(len(recs), ROW_DTYPE)
        cid = recs["coord_id"].astype(np.int64)
        bx, by, bz = cid % nb, (cid // nb) % nb, cid // (nb * nb)
        rows["id"] = recs["id"]
        rows["min"] = np.stack([bx, bz, by], axis=1).astype(np.float32) * m  # y/z swapped on output
        rows["max"] = rows["min"] + np.float32(m)
        rows["nv"], rows["ni"] = recs["vertex_count"], recs["index_count"]
        rows["tnv"], rows["tni"] = recs["trans_vertex_count"], recs["trans_index_count"]

        def gather(arr, offs, counts):
            parts = [arr[o:o + c] for o, c in zip(offs, counts) if c]
            return np.concatenate(parts) if parts else arr[:0]

        verts = gather(self.verts, recs["vertex_offset"], recs["vertex_count"])
        idx = gather(self.idx, recs["index_offset"], recs["index_count"])
        tverts = gather(self.tverts, recs["trans_vertex_offset"].ravel(), recs["trans_vertex_count"].ravel())
        tidx = gather(self.tidx, recs["trans_index_offset"].ravel(), recs["trans_index_count"].ravel())
        return LevelView(rows, verts, idx, tverts, tidx)


def merge_results(results):
    """The per-rank results of a sharded run as ONE result: arenas concatenated in rank order, directory offsets
    rebased and sorted by (level, coord_id) - the reference's block order - statistics summed.  Block ids need no
    fixing: they are a function of (level, coordinate) in a full run (TransVoxelImpl.cpp:395-401)."""
    recs, bases = [], [0, 0, 0, 0]
    for r in results:
        rr = r.records.copy()
        rr["vertex_offset"] += np.uint32(bases[0]); rr["index_offset"] += np.uint32(bases[1])
        rr["trans_vertex_offset"] += np.uint32(bases[2]); rr["trans_index_offset"] += np.uint32(bases[3])
        recs.append(rr)
        bases = [bases[0] + len(r.verts), bases[1] + len(r.idx), bases[2] + len(r.tverts), bases[3] + len(r.tidx)]
    records = np.concatenate(recs)
    records = records[np.lexsort((records["coord_id"], records["level"]))]
    merged = Result.__new__(Result)
    merged.n, merged.info, merged.records = results[0].n, None, records
    merged.verts = np.concatenate([r.verts for r in results]); merged.idx = np.concatenate([r.idx for r in results])
    merged.tverts = np.concatenate([r.tverts for r in results]); merged.tidx = np.concatenate([r.tidx for r in results])
    merged.stats = np.sum([r.stats.astype(np.uint64) for r in results], axis=0).astype(np.uint32)
    return merged


def _device_to_numpy(ptr, count, dtype):
    """`count` elements of `dtype` at a device address, copied to a numpy array (through torch)."""
    import torch
    out = np.zeros(count, dtype)
    if count:
        t = torch.as_tensor(DevicePointer(ptr, count * dtype.itemsize), device=torch.device("cuda", torch.cuda.current_device()))
        out.view(np.uint8)[:] = t.cpu().numpy()
    return out


class Mesh:
    """vxb_mesh: the polygonized surface kept in HBM across edits (include/vxb200.h "mesh").  apply() after every run of the
    context (full or region) splices the run into the mesh on the GPU in the reference's block order."""

    def __init__(self, ctx, capacity=None):
        self.ctx, self.L = ctx, ctx.L
        h = C.c_void_p()
        cap = None if capacity is None else (C.c_uint64 * 4)(*capacity)
        ctx._check(self.L.vxb_mesh_create(ctx.h, cap, C.byref(h)), "vxb_mesh_create")
        self.h = h
        ctx._meshes.append(self)

    def close(self):
        if getattr(self, "h", None) and self.ctx.h:
            self.L.vxb_mesh_destroy(self.h)
            self.ctx._meshes.remove(self)
        self.h = None

    def apply_rc(self):
        """vxb_mesh_apply's return code (0, or ERR_STATE when the apply is refused)."""
        return self.L.vxb_mesh_apply(self.h)

    def apply(self):
        self.ctx._check(self.apply_rc(), "vxb_mesh_apply")
        return self.info()

    def info(self):
        i = MeshInfo()
        self.ctx._check(self.L.vxb_mesh_info_get(self.h, C.byref(i)), "vxb_mesh_info_get")
        return i

    def download(self):
        """The directory in mesh order and the used prefix of each arena, as a Result (Result.level(l) = surface order)."""
        info = self.info()
        records = np.zeros(info.block_count, RECORD_DTYPE)
        verts = np.zeros(info.vertex_span, VERTEX_DTYPE); idx = np.zeros(info.index_span, np.uint32)
        tverts = np.zeros(info.trans_vertex_span, VERTEX_DTYPE); tidx = np.zeros(info.trans_index_span, np.uint32)
        self.ctx._check(self.L.vxb_mesh_download(self.h, _ptr(records), _ptr(verts), _ptr(idx), _ptr(tverts), _ptr(tidx)), "vxb_mesh_download")
        return Result(self.ctx.n, info, records, verts, idx, tverts, tidx)

    def device_arenas(self):
        """(records, vertices, indices, trans vertices, trans indices) device addresses."""
        p = [C.c_void_p() for _ in range(5)]
        self.ctx._check(self.L.vxb_mesh_device_arenas(self.h, *[C.byref(x) for x in p]), "vxb_mesh_device_arenas")
        return tuple(x.value for x in p)

    def select_lod(self, camera, base_distance, lists_out=None):
        """(regular commands, regular infos, transition commands, transition infos) copied to numpy; the device-resident
        vxb_draw_lists go to `lists_out` (a DrawLists) when given."""
        cam = np.ascontiguousarray(camera, np.float32)
        lists = DrawLists() if lists_out is None else lists_out
        self.ctx._check(self.L.vxb_mesh_select_lod(self.h, _ptr(cam), base_distance, C.byref(lists)), "vxb_mesh_select_lod")
        return (_device_to_numpy(lists.regular, lists.regular_count, DRAW_COMMAND_DTYPE),
                _device_to_numpy(lists.regular_info, lists.regular_count, DRAW_INFO_DTYPE),
                _device_to_numpy(lists.transition, lists.transition_count, DRAW_COMMAND_DTYPE),
                _device_to_numpy(lists.transition_info, lists.transition_count, DRAW_INFO_DTYPE))

    def bounds(self):
        """The blocks' boxes as a (block_count, 6) float32 array {min xyz, max xyz} in directory order (vxb_mesh_download_bounds)."""
        out = np.zeros((self.info().block_count, 6), np.float32)
        self.ctx._check(self.L.vxb_mesh_download_bounds(self.h, _ptr(out)), "vxb_mesh_download_bounds")
        return out

    def bounds_device(self):
        """vxb_mesh_bounds_get: a MeshBounds (device address of the boxes, the slot of every level, the slot count)."""
        b = MeshBounds()
        self.ctx._check(self.L.vxb_mesh_bounds_get(self.h, C.byref(b)), "vxb_mesh_bounds_get")
        return b

    def select_lod_views(self, lod_camera, base_distance, views, lists_out=None):
        """vxb_mesh_select_lod_views: the cut of (lod_camera, base_distance) culled against each of `views` ([views, 6, 4]
        plane coefficients or a View array).  Returns, per view, the four arrays select_lod returns; the device-resident
        vxb_draw_lists go to `lists_out` (a DrawLists array of len(views)) when given."""
        cam = np.ascontiguousarray(lod_camera, np.float32)
        views = views if isinstance(views, C.Array) else make_views(views)
        lists = (DrawLists * len(views))() if lists_out is None else lists_out
        self.ctx._check(self.L.vxb_mesh_select_lod_views(self.h, _ptr(cam), base_distance, views, len(views), lists), "vxb_mesh_select_lod_views")
        return [(_device_to_numpy(l.regular, l.regular_count, DRAW_COMMAND_DTYPE),
                 _device_to_numpy(l.regular_info, l.regular_count, DRAW_INFO_DTYPE),
                 _device_to_numpy(l.transition, l.transition_count, DRAW_COMMAND_DTYPE),
                 _device_to_numpy(l.transition_info, l.transition_count, DRAW_INFO_DTYPE)) for l in lists]

    def select_cut_rc(self, lod_camera, lod_factor, views, lists_out=None, count=None):
        """vxb_mesh_select_cut's return code: `lod_camera` and `views` ([views, 6, 4] plane coefficients or a View array) may be
        None for NULL pointers, `lists_out` (a DrawLists array) None for a NULL out; `count` defaults to len(views)."""
        cam = _batch(lod_camera, np.float32)
        if views is not None and not isinstance(views, C.Array):
            views = make_views(views)
        n = (0 if views is None else len(views)) if count is None else count
        return self.L.vxb_mesh_select_cut(self.h, _ptr(cam), lod_factor, views, n, lists_out)

    def select_cut(self, lod_camera, lod_factor, views, lists_out=None):
        """vxb_mesh_select_cut: the balanced LOD cut of (lod_camera, lod_factor) culled against each of `views` ([views, 6, 4]
        plane coefficients or a View array).  Returns, per view, the four arrays select_lod returns; the device-resident
        vxb_draw_lists go to `lists_out` (a DrawLists array of len(views)) when given."""
        views = views if isinstance(views, C.Array) else make_views(views)
        lists = (DrawLists * len(views))() if lists_out is None else lists_out
        self.ctx._check(self.select_cut_rc(lod_camera, lod_factor, views, lists), "vxb_mesh_select_cut")
        return [(_device_to_numpy(l.regular, l.regular_count, DRAW_COMMAND_DTYPE),
                 _device_to_numpy(l.regular_info, l.regular_count, DRAW_INFO_DTYPE),
                 _device_to_numpy(l.transition, l.transition_count, DRAW_COMMAND_DTYPE),
                 _device_to_numpy(l.transition_info, l.transition_count, DRAW_INFO_DTYPE)) for l in lists[:len(views)]]

    def raycast_rc(self, rays, hits=None):
        """vxb_mesh_raycast's return code for a RAY_DTYPE array; the hits go to `hits` (a RAY_HIT_DTYPE array, or None for a
        NULL pointer)."""
        rays = _batch(rays, RAY_DTYPE)
        return self.L.vxb_mesh_raycast(self.h, _ptr(rays), 0 if rays is None else len(rays), _ptr(hits))

    def raycast(self, origins, directions=None, t_min=0.0, t_max=np.inf):
        """Casts rays against the mesh's level-0 triangles (vxb_mesh_raycast): `origins` / `directions` are [count, 3] in OUTPUT
        (Y-up) coordinates, or `origins` is a RAY_DTYPE array and `directions` None.  Returns a RAY_HIT_DTYPE array."""
        rays = np.ascontiguousarray(origins if directions is None else make_rays(origins, directions, t_min, t_max), RAY_DTYPE)
        hits = np.zeros(len(rays), RAY_HIT_DTYPE)
        self.ctx._check(self.raycast_rc(rays, hits), "vxb_mesh_raycast")
        return hits

    def raycast_device(self, rays_ptr, count, hits_ptr):
        """vxb_mesh_raycast_device: `count` vxb_ray at the device address `rays_ptr`, hits to `hits_ptr` (e.g. torch tensors'
        data_ptr()); enqueued on the context's stream, returns without waiting."""
        self.ctx._check(self.L.vxb_mesh_raycast_device(self.h, _dev(rays_ptr), count, _dev(hits_ptr)), "vxb_mesh_raycast_device")

    def raycast_cut_rc(self, lod_camera, lod_factor, rays, hits=None, count=None):
        """vxb_mesh_raycast_cut's return code: `lod_camera` and `rays` (a RAY_DTYPE array) may be None for NULL pointers, `hits`
        (a CUT_HIT_DTYPE array) None for a NULL pointer; `count` defaults to len(rays)."""
        rays = _batch(rays, RAY_DTYPE)
        n = (0 if rays is None else len(rays)) if count is None else count
        return self.L.vxb_mesh_raycast_cut(self.h, _ptr(_batch(lod_camera, np.float32)), lod_factor, _ptr(rays), n, _ptr(hits))

    def raycast_cut(self, lod_camera, lod_factor, origins, directions=None, t_min=0.0, t_max=np.inf):
        """Casts rays against the triangles vxb_mesh_select_cut's cut of (lod_camera, lod_factor) draws (vxb_mesh_raycast_cut):
        `origins` / `directions` as for raycast.  Returns a CUT_HIT_DTYPE array."""
        rays = np.ascontiguousarray(origins if directions is None else make_rays(origins, directions, t_min, t_max), RAY_DTYPE)
        hits = np.zeros(len(rays), CUT_HIT_DTYPE)
        self.ctx._check(self.raycast_cut_rc(lod_camera, lod_factor, rays, hits), "vxb_mesh_raycast_cut")
        return hits

    def raycast_cut_device(self, lod_camera, lod_factor, rays_ptr, count, hits_ptr):
        """vxb_mesh_raycast_cut_device: `count` vxb_ray at the device address `rays_ptr`, hits to `hits_ptr`; enqueued on the
        context's stream (the first cast after an apply waits for it once)."""
        self.ctx._check(self.L.vxb_mesh_raycast_cut_device(self.h, _ptr(_batch(lod_camera, np.float32)), lod_factor, _dev(rays_ptr),
                                                           count, _dev(hits_ptr)), "vxb_mesh_raycast_cut_device")

    def sphere_cast_rc(self, radius, rays, hits=None, count=None):
        """vxb_mesh_sphere_cast's return code for a RAY_DTYPE array (or None for a NULL pointer); the hits go to `hits` (a
        SPHERE_HIT_DTYPE array, or None for a NULL pointer); `count` defaults to len(rays)."""
        rays = _batch(rays, RAY_DTYPE)
        n = (0 if rays is None else len(rays)) if count is None else count
        return self.L.vxb_mesh_sphere_cast(self.h, radius, _ptr(rays), n, _ptr(hits))

    def sphere_cast(self, radius, origins, directions=None, t_min=0.0, t_max=np.inf):
        """Sweeps a sphere of `radius` voxels along each segment against the mesh's level-0 triangles (vxb_mesh_sphere_cast):
        `origins` / `directions` are [count, 3] in OUTPUT (Y-up) coordinates, or `origins` is a RAY_DTYPE array and
        `directions` None.  Returns a SPHERE_HIT_DTYPE array."""
        rays = np.ascontiguousarray(origins if directions is None else make_rays(origins, directions, t_min, t_max), RAY_DTYPE)
        hits = np.zeros(len(rays), SPHERE_HIT_DTYPE)
        self.ctx._check(self.sphere_cast_rc(radius, rays, hits), "vxb_mesh_sphere_cast")
        return hits

    def sphere_cast_device(self, radius, rays_ptr, count, hits_ptr):
        """vxb_mesh_sphere_cast_device: `count` vxb_ray at the device address `rays_ptr`, hits to `hits_ptr`; enqueued on the
        context's stream, returns without waiting."""
        self.ctx._check(self.L.vxb_mesh_sphere_cast_device(self.h, radius, _dev(rays_ptr), count, _dev(hits_ptr)),
                        "vxb_mesh_sphere_cast_device")

    def closest_points_rc(self, max_distance, points, hits=None, count=None):
        """vxb_mesh_closest_point's return code for [count, 3] float32 points (or None for a NULL pointer); the hits go to
        `hits` (a CLOSEST_HIT_DTYPE array, or None for a NULL pointer); `count` defaults to len(points)."""
        pts = _batch(points, np.float32)
        pts = None if pts is None else pts.reshape(-1, 3)
        n = (0 if pts is None else len(pts)) if count is None else count
        return self.L.vxb_mesh_closest_point(self.h, max_distance, _ptr(pts), n, _ptr(hits))

    def closest_points(self, points, max_distance):
        """The nearest level-0 surface point within `max_distance` voxels of each of the [count, 3] `points` (OUTPUT, Y-up
        coordinates), vxb_mesh_closest_point.  Returns a CLOSEST_HIT_DTYPE array."""
        pts = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
        hits = np.zeros(len(pts), CLOSEST_HIT_DTYPE)
        self.ctx._check(self.closest_points_rc(max_distance, pts, hits), "vxb_mesh_closest_point")
        return hits

    def closest_points_device(self, max_distance, points_ptr, count, hits_ptr):
        """vxb_mesh_closest_point_device: `count` points (3 floats each) at the device address `points_ptr`, hits to
        `hits_ptr`; enqueued on the context's stream, returns without waiting."""
        self.ctx._check(self.L.vxb_mesh_closest_point_device(self.h, max_distance, _dev(points_ptr), count, _dev(hits_ptr)),
                        "vxb_mesh_closest_point_device")

    def sphere_cast_cut_rc(self, lod_camera, lod_factor, radius, rays, hits=None, count=None):
        """vxb_mesh_sphere_cast_cut's return code: `lod_camera` and `rays` (a RAY_DTYPE array) may be None for NULL pointers,
        `hits` (a SPHERE_CUT_HIT_DTYPE array) None for a NULL pointer; `count` defaults to len(rays)."""
        rays = _batch(rays, RAY_DTYPE)
        n = (0 if rays is None else len(rays)) if count is None else count
        return self.L.vxb_mesh_sphere_cast_cut(self.h, _ptr(_batch(lod_camera, np.float32)), lod_factor, radius, _ptr(rays), n, _ptr(hits))

    def sphere_cast_cut(self, lod_camera, lod_factor, radius, origins, directions=None, t_min=0.0, t_max=np.inf):
        """Sweeps a sphere of `radius` voxels along each segment against the triangles vxb_mesh_select_cut's cut of (lod_camera,
        lod_factor) draws (vxb_mesh_sphere_cast_cut): `origins` / `directions` as for sphere_cast.  Returns a
        SPHERE_CUT_HIT_DTYPE array."""
        rays = np.ascontiguousarray(origins if directions is None else make_rays(origins, directions, t_min, t_max), RAY_DTYPE)
        hits = np.zeros(len(rays), SPHERE_CUT_HIT_DTYPE)
        self.ctx._check(self.sphere_cast_cut_rc(lod_camera, lod_factor, radius, rays, hits), "vxb_mesh_sphere_cast_cut")
        return hits

    def sphere_cast_cut_device(self, lod_camera, lod_factor, radius, rays_ptr, count, hits_ptr):
        """vxb_mesh_sphere_cast_cut_device: `count` vxb_ray at the device address `rays_ptr`, hits to `hits_ptr`; enqueued on
        the context's stream (the first cut query after an apply waits for it once)."""
        self.ctx._check(self.L.vxb_mesh_sphere_cast_cut_device(self.h, _ptr(_batch(lod_camera, np.float32)), lod_factor, radius,
                                                               _dev(rays_ptr), count, _dev(hits_ptr)), "vxb_mesh_sphere_cast_cut_device")

    def closest_points_cut_rc(self, lod_camera, lod_factor, max_distance, points, hits=None, count=None):
        """vxb_mesh_closest_point_cut's return code: `lod_camera` and `points` ([count, 3] float32) may be None for NULL
        pointers, `hits` (a CLOSEST_CUT_HIT_DTYPE array) None for a NULL pointer; `count` defaults to len(points)."""
        pts = _batch(points, np.float32)
        pts = None if pts is None else pts.reshape(-1, 3)
        n = (0 if pts is None else len(pts)) if count is None else count
        return self.L.vxb_mesh_closest_point_cut(self.h, _ptr(_batch(lod_camera, np.float32)), lod_factor, max_distance, _ptr(pts), n,
                                                 _ptr(hits))

    def closest_points_cut(self, lod_camera, lod_factor, points, max_distance):
        """The nearest drawn surface point of the cut of (lod_camera, lod_factor) within `max_distance` voxels of each of the
        [count, 3] `points` (OUTPUT, Y-up coordinates), vxb_mesh_closest_point_cut.  Returns a CLOSEST_CUT_HIT_DTYPE array."""
        pts = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
        hits = np.zeros(len(pts), CLOSEST_CUT_HIT_DTYPE)
        self.ctx._check(self.closest_points_cut_rc(lod_camera, lod_factor, max_distance, pts, hits), "vxb_mesh_closest_point_cut")
        return hits

    def closest_points_cut_device(self, lod_camera, lod_factor, max_distance, points_ptr, count, hits_ptr):
        """vxb_mesh_closest_point_cut_device: `count` points (3 floats each) at the device address `points_ptr`, hits to
        `hits_ptr`; enqueued on the context's stream (the first cut query after an apply waits for it once)."""
        self.ctx._check(self.L.vxb_mesh_closest_point_cut_device(self.h, _ptr(_batch(lod_camera, np.float32)), lod_factor,
                                                                 max_distance, _dev(points_ptr), count, _dev(hits_ptr)),
                        "vxb_mesh_closest_point_cut_device")

    def capsule_cast_rc(self, sweeps, hits=None, count=None):
        """vxb_mesh_capsule_cast's return code for a CAPSULE_SWEEP_DTYPE array (or None for a NULL pointer); the hits go to
        `hits` (a CAPSULE_HIT_DTYPE array, or None for a NULL pointer); `count` defaults to len(sweeps)."""
        sweeps = _batch(sweeps, CAPSULE_SWEEP_DTYPE)
        n = (0 if sweeps is None else len(sweeps)) if count is None else count
        return self.L.vxb_mesh_capsule_cast(self.h, _ptr(sweeps), n, _ptr(hits))

    def capsule_cast(self, sweeps):
        """Sweeps capsules against the mesh's level-0 triangles (vxb_mesh_capsule_cast): `sweeps` is a CAPSULE_SWEEP_DTYPE
        array (make_capsule_sweeps), OUTPUT (Y-up) coordinates.  Returns a CAPSULE_HIT_DTYPE array."""
        sweeps = np.ascontiguousarray(sweeps, CAPSULE_SWEEP_DTYPE)
        hits = np.zeros(len(sweeps), CAPSULE_HIT_DTYPE)
        self.ctx._check(self.capsule_cast_rc(sweeps, hits), "vxb_mesh_capsule_cast")
        return hits

    def capsule_cast_device(self, sweeps_ptr, count, hits_ptr):
        """vxb_mesh_capsule_cast_device: `count` vxb_capsule_sweep at the device address `sweeps_ptr`, hits to `hits_ptr`;
        enqueued on the context's stream, returns without waiting."""
        self.ctx._check(self.L.vxb_mesh_capsule_cast_device(self.h, _dev(sweeps_ptr), count, _dev(hits_ptr)),
                        "vxb_mesh_capsule_cast_device")

    def closest_to_segment_rc(self, max_distance, segments, hits=None, count=None):
        """vxb_mesh_closest_to_segment's return code for a SEGMENT_DTYPE array (or None for a NULL pointer); the hits go to
        `hits` (a SEGMENT_HIT_DTYPE array, or None for a NULL pointer); `count` defaults to len(segments)."""
        segments = _batch(segments, SEGMENT_DTYPE)
        n = (0 if segments is None else len(segments)) if count is None else count
        return self.L.vxb_mesh_closest_to_segment(self.h, max_distance, _ptr(segments), n, _ptr(hits))

    def closest_to_segment(self, segments, max_distance):
        """The nearest level-0 surface point within `max_distance` voxels of each segment (a SEGMENT_DTYPE array, make_segments;
        OUTPUT, Y-up coordinates), vxb_mesh_closest_to_segment.  Returns a SEGMENT_HIT_DTYPE array."""
        segments = np.ascontiguousarray(segments, SEGMENT_DTYPE)
        hits = np.zeros(len(segments), SEGMENT_HIT_DTYPE)
        self.ctx._check(self.closest_to_segment_rc(max_distance, segments, hits), "vxb_mesh_closest_to_segment")
        return hits

    def closest_to_segment_device(self, max_distance, segments_ptr, count, hits_ptr):
        """vxb_mesh_closest_to_segment_device: `count` vxb_segment at the device address `segments_ptr`, hits to `hits_ptr`;
        enqueued on the context's stream, returns without waiting."""
        self.ctx._check(self.L.vxb_mesh_closest_to_segment_device(self.h, max_distance, _dev(segments_ptr), count, _dev(hits_ptr)),
                        "vxb_mesh_closest_to_segment_device")

    def capsule_cast_cut_rc(self, lod_camera, lod_factor, sweeps, hits=None, count=None):
        """vxb_mesh_capsule_cast_cut's return code: `lod_camera` and `sweeps` (a CAPSULE_SWEEP_DTYPE array) may be None for NULL
        pointers, `hits` (a CAPSULE_CUT_HIT_DTYPE array) None for a NULL pointer; `count` defaults to len(sweeps)."""
        sweeps = _batch(sweeps, CAPSULE_SWEEP_DTYPE)
        n = (0 if sweeps is None else len(sweeps)) if count is None else count
        return self.L.vxb_mesh_capsule_cast_cut(self.h, _ptr(_batch(lod_camera, np.float32)), lod_factor, _ptr(sweeps), n, _ptr(hits))

    def capsule_cast_cut(self, lod_camera, lod_factor, sweeps):
        """Sweeps capsules (a CAPSULE_SWEEP_DTYPE array, make_capsule_sweeps) against the triangles vxb_mesh_select_cut's cut of
        (lod_camera, lod_factor) draws (vxb_mesh_capsule_cast_cut).  Returns a CAPSULE_CUT_HIT_DTYPE array."""
        sweeps = np.ascontiguousarray(sweeps, CAPSULE_SWEEP_DTYPE)
        hits = np.zeros(len(sweeps), CAPSULE_CUT_HIT_DTYPE)
        self.ctx._check(self.capsule_cast_cut_rc(lod_camera, lod_factor, sweeps, hits), "vxb_mesh_capsule_cast_cut")
        return hits

    def capsule_cast_cut_device(self, lod_camera, lod_factor, sweeps_ptr, count, hits_ptr):
        """vxb_mesh_capsule_cast_cut_device: `count` vxb_capsule_sweep at the device address `sweeps_ptr`, hits to `hits_ptr`;
        enqueued on the context's stream (the first cut query after an apply waits for it once).  A sweep out of reach is a
        miss."""
        self.ctx._check(self.L.vxb_mesh_capsule_cast_cut_device(self.h, _ptr(_batch(lod_camera, np.float32)), lod_factor,
                                                                _dev(sweeps_ptr), count, _dev(hits_ptr)), "vxb_mesh_capsule_cast_cut_device")

    def closest_to_segment_cut_rc(self, lod_camera, lod_factor, max_distance, segments, hits=None, count=None):
        """vxb_mesh_closest_to_segment_cut's return code: `lod_camera` and `segments` (a SEGMENT_DTYPE array) may be None for
        NULL pointers, `hits` (a SEGMENT_CUT_HIT_DTYPE array) None for a NULL pointer; `count` defaults to len(segments)."""
        segments = _batch(segments, SEGMENT_DTYPE)
        n = (0 if segments is None else len(segments)) if count is None else count
        return self.L.vxb_mesh_closest_to_segment_cut(self.h, _ptr(_batch(lod_camera, np.float32)), lod_factor, max_distance,
                                                      _ptr(segments), n, _ptr(hits))

    def closest_to_segment_cut(self, lod_camera, lod_factor, segments, max_distance):
        """The nearest drawn surface point of the cut of (lod_camera, lod_factor) within `max_distance` voxels of each segment
        (a SEGMENT_DTYPE array, make_segments), vxb_mesh_closest_to_segment_cut.  Returns a SEGMENT_CUT_HIT_DTYPE array."""
        segments = np.ascontiguousarray(segments, SEGMENT_DTYPE)
        hits = np.zeros(len(segments), SEGMENT_CUT_HIT_DTYPE)
        self.ctx._check(self.closest_to_segment_cut_rc(lod_camera, lod_factor, max_distance, segments, hits),
                        "vxb_mesh_closest_to_segment_cut")
        return hits

    def closest_to_segment_cut_device(self, lod_camera, lod_factor, max_distance, segments_ptr, count, hits_ptr):
        """vxb_mesh_closest_to_segment_cut_device: `count` vxb_segment at the device address `segments_ptr`, hits to
        `hits_ptr`; enqueued on the context's stream (the first cut query after an apply waits for it once).  A segment out of
        reach is a miss."""
        self.ctx._check(self.L.vxb_mesh_closest_to_segment_cut_device(self.h, _ptr(_batch(lod_camera, np.float32)), lod_factor,
                                                                      max_distance, _dev(segments_ptr), count, _dev(hits_ptr)),
                        "vxb_mesh_closest_to_segment_cut_device")

    def overlap_boxes_rc(self, boxes, offsets, tris=None, capacity=None, count=None):
        """vxb_mesh_overlap_box's return code for a BOX_DTYPE array (or None for a NULL pointer): offsets to `offsets` (a uint64
        array of count + 1, or None), triangles to `tris` (an OVERLAP_TRIANGLE_DTYPE array, or None for a NULL pointer);
        `capacity` defaults to len(tris) (0 without), `count` to len(boxes)."""
        boxes = _batch(boxes, BOX_DTYPE)
        n = (0 if boxes is None else len(boxes)) if count is None else count
        cap = (0 if tris is None else len(tris)) if capacity is None else capacity
        return self.L.vxb_mesh_overlap_box(self.h, _ptr(boxes), n, _ptr(offsets), _ptr(tris), cap)

    def overlap_boxes(self, boxes):
        """The level-0 triangles overlapping each box of a BOX_DTYPE array (make_boxes; OUTPUT, Y-up coordinates),
        vxb_mesh_overlap_box: a count-only call, then the fill.  Returns (offsets [count + 1] uint64, OVERLAP_TRIANGLE_DTYPE
        array): box q's triangles are tris[offsets[q]:offsets[q + 1]]."""
        boxes = np.ascontiguousarray(boxes, BOX_DTYPE)
        offsets = np.zeros(len(boxes) + 1, np.uint64)
        self.ctx._check(self.overlap_boxes_rc(boxes, offsets), "vxb_mesh_overlap_box")
        tris = np.zeros(int(offsets[-1]), OVERLAP_TRIANGLE_DTYPE)
        self.ctx._check(self.overlap_boxes_rc(boxes, offsets, tris), "vxb_mesh_overlap_box")
        return offsets, tris

    def overlap_boxes_device(self, boxes_ptr, count, offsets_ptr, tris_ptr, capacity):
        """vxb_mesh_overlap_box_device: `count` vxb_box at the device address `boxes_ptr`, count + 1 uint64 offsets to
        `offsets_ptr`, at most `capacity` triangles to `tris_ptr` (None: count only); enqueued on the context's stream, returns
        without waiting."""
        self.ctx._check(self.L.vxb_mesh_overlap_box_device(self.h, _dev(boxes_ptr), count, _dev(offsets_ptr), _dev(tris_ptr), capacity),
                        "vxb_mesh_overlap_box_device")


class Context:
    """vxb_context wrapper.  Raises VxbError on any failure (no CUDA device included)."""

    def __init__(self, device=0):
        self.L = load_library()
        h = C.c_void_p()
        rc = self.L.vxb_create(device, C.byref(h))
        if rc != 0:
            raise VxbError("vxb_create failed (%d): %s" % (rc, self.L.vxb_last_error(None).decode()))
        self.h = h
        self.n = 0
        self._keep = None
        self._meshes = []

    def close(self):
        if getattr(self, "h", None):
            for m in self._meshes:   # vxb_destroy releases them
                m.h = None
            self._meshes = []
            self.L.vxb_destroy(self.h)
            self.h = None

    def mesh(self, capacity=None):
        """A device-resident mesh of this context (capacity: {vertices, indices, trans vertices, trans indices} or None)."""
        return Mesh(self, capacity)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc, what):
        if rc != 0:
            raise VxbError("%s failed (%d): %s" % (what, rc, self.L.vxb_last_error(self.h).decode()))

    def upload_dense(self, dist, mat=None, blend=None):
        """dist/mat/blend: host arrays (numpy or anything with .ctypes / an int address) indexed [z, y, x]."""
        n = dist.shape[0]
        self._check(self.L.vxb_grid_upload_dense(self.h, n, _ptr(dist), _ptr(mat), _ptr(blend)), "vxb_grid_upload_dense")
        self.n = n

    def upload_dense_ptr(self, n, dist_ptr, mat_ptr, blend_ptr):
        self._check(self.L.vxb_grid_upload_dense(self.h, n, C.c_void_p(dist_ptr), C.c_void_p(mat_ptr), C.c_void_p(blend_ptr)),
                    "vxb_grid_upload_dense")
        self.n = n

    def upload_blocks(self, n, dist_blocks, mat_blocks=None, blend_blocks=None):
        self._check(self.L.vxb_grid_upload_blocks(self.h, n, _ptr(dist_blocks), _ptr(mat_blocks), _ptr(blend_blocks)),
                    "vxb_grid_upload_blocks")
        self.n = n

    def upload_packed(self, blob, size=None):
        """blob: the bytes of Grid::PackForSave (numpy uint8 array, bytes, or an int address with `size`)."""
        if isinstance(blob, int):
            ptr, nbytes = C.c_void_p(blob), size
        elif isinstance(blob, (bytes, bytearray)):
            arr = np.frombuffer(blob, np.uint8); ptr, nbytes = _ptr(arr), arr.size
            self._blob_keep = arr
        else:
            ptr, nbytes = _ptr(blob), blob.size
        self._check(self.L.vxb_grid_upload_packed(self.h, ptr, nbytes), "vxb_grid_upload_packed")
        self.n = int(np.frombuffer(C.string_at(ptr, 8), np.uint32)[1])

    def upload_packed_streamed(self, blob, produce):
        """vxb_grid_upload_packed_streamed: `blob` (numpy uint8) holds the header and the complete size table; produce(layer0,
        layer1) is called on this thread before the data of those block layers is copied and must have written it."""
        cb = PackProducer(lambda user, l0, l1: produce(int(l0), int(l1)))
        self._check(self.L.vxb_grid_upload_packed_streamed(self.h, _ptr(blob), blob.size, cb, None), "vxb_grid_upload_packed_streamed")
        self.n = int(blob[:8].view(np.uint32)[1])

    # ---- device-resident grid store (fill / edit / pack) ----
    def fill(self, n, surface, start=(0.0, 0.0, 0.0), step=1.0):
        """Grid::Create(n, n, n, start, step, &surface) on the device (a capi.Surface); with a cube: this rank's pieces."""
        st = np.ascontiguousarray(start, np.float32)
        self._check(self.L.vxb_grid_fill(self.h, n, C.byref(surface), _ptr(st), step), "vxb_grid_fill")
        self.n = n

    def inject_surface(self, position, extents, surface, inject_type):
        """VoxelGrid::InjectSurface on the device grid; returns the modified box (6 floats, Y-up) the reference returns."""
        p = np.ascontiguousarray(position, np.float32); e = np.ascontiguousarray(extents, np.float32)
        lo = np.zeros(3, np.float32); hi = np.zeros(3, np.float32)
        self._check(self.L.vxb_grid_inject_surface(self.h, _ptr(p), _ptr(e), C.byref(surface), inject_type, _ptr(lo), _ptr(hi)), "vxb_grid_inject_surface")
        return np.concatenate([lo, hi])

    def inject_material(self, position, extents, material, add_subtract_blend):
        p = np.ascontiguousarray(position, np.float32); e = np.ascontiguousarray(extents, np.float32)
        lo = np.zeros(3, np.float32); hi = np.zeros(3, np.float32)
        self._check(self.L.vxb_grid_inject_material(self.h, _ptr(p), _ptr(e), material, 1 if add_subtract_blend else 0, _ptr(lo), _ptr(hi)), "vxb_grid_inject_material")
        return np.concatenate([lo, hi])

    def fill_program(self, n, ops, start=(0.0, 0.0, 0.0), step=1.0):
        """Grid::Create(n, n, n, start, step, &surface) with an SDF program (a list of Op); with a cube: this rank's pieces."""
        arr = program_array(ops)
        st = np.ascontiguousarray(start, np.float32)
        self._check(self.L.vxb_grid_fill_program(self.h, n, C.cast(arr, C.c_void_p), len(arr), _ptr(st), step), "vxb_grid_fill_program")
        self.n = n

    def inject_program(self, position, extents, ops, inject_type):
        """VoxelGrid::InjectSurface with an SDF program sampled relative to `position`; returns the modified box (Y-up)."""
        arr = program_array(ops)
        p = np.ascontiguousarray(position, np.float32); e = np.ascontiguousarray(extents, np.float32)
        lo = np.zeros(3, np.float32); hi = np.zeros(3, np.float32)
        self._check(self.L.vxb_grid_inject_program(self.h, _ptr(p), _ptr(e), C.cast(arr, C.c_void_p), len(arr), inject_type, _ptr(lo), _ptr(hi)),
                    "vxb_grid_inject_program")
        return np.concatenate([lo, hi])

    def program_stats(self):
        """The last fill_program: blocks covered, blocks written by the cull pass, pass A / pass B device milliseconds."""
        s = ProgramStats()
        self._check(self.L.vxb_grid_program_stats(self.h, C.byref(s)), "vxb_grid_program_stats")
        return s

    def pack(self):
        """Grid::PackForSave of the device grid (GPU run-length coding): numpy uint8 blob."""
        buf = np.empty(self.L.vxb_pack_dense_bound(self.n), np.uint8)
        written = C.c_size_t(0)
        self._check(self.L.vxb_grid_pack(self.h, _ptr(buf), buf.size, C.byref(written)), "vxb_grid_pack")
        return buf[:written.value].copy()

    def download_dense(self):
        n = self.n
        dist = np.empty((n, n, n), np.int8); mat = np.empty((n, n, n), np.uint8); blend = np.empty((n, n, n), np.uint8)
        self._check(self.L.vxb_grid_download_dense(self.h, _ptr(dist), _ptr(mat), _ptr(blend)), "vxb_grid_download_dense")
        return dist, mat, blend

    # ---- consumer side: LOD cut + indirect draw lists on the device ----
    def select_lod(self, camera, base_distance):
        """(regular commands, regular infos, transition commands, transition infos) as numpy record arrays (copied back for
        inspection; a renderer consumes the device-resident lists of vxb_draw_lists directly)."""
        cam = np.ascontiguousarray(camera, np.float32)
        lists = DrawLists()
        self._check(self.L.vxb_result_select_lod(self.h, _ptr(cam), base_distance, C.byref(lists)), "vxb_result_select_lod")
        rc = np.zeros(lists.regular_count, DRAW_COMMAND_DTYPE); ri = np.zeros(lists.regular_count, DRAW_INFO_DTYPE)
        tc = np.zeros(lists.transition_count, DRAW_COMMAND_DTYPE); ti = np.zeros(lists.transition_count, DRAW_INFO_DTYPE)
        self._check(self.L.vxb_result_download_draws(self.h, _ptr(rc), _ptr(ri), _ptr(tc), _ptr(ti)), "vxb_result_download_draws")
        return rc, ri, tc, ti

    def device_arenas(self):
        v, i, tv, ti = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_void_p()
        self._check(self.L.vxb_result_device_arenas(self.h, C.byref(v), C.byref(i), C.byref(tv), C.byref(ti)), "vxb_result_device_arenas")
        return v.value, i.value, tv.value, ti.value

    def set_device_grid(self, n, d_dist, d_mat, d_blend, keep=None):
        """Device pointers (ints) of dense volumes that stay resident (e.g. torch tensors' data_ptr())."""
        self._check(self.L.vxb_grid_set_device(self.h, n, C.c_void_p(d_dist), C.c_void_p(d_mat), C.c_void_p(d_blend)),
                    "vxb_grid_set_device")
        self.n = n
        self._keep = keep

    def set_materials(self, table=None, valid=None):
        self._check(self.L.vxb_set_materials(self.h, _ptr(table), _ptr(valid)), "vxb_set_materials")

    def set_capacity(self, vertices=0, indices=0, trans_vertices=0, trans_indices=0):
        self._check(self.L.vxb_set_capacity(self.h, vertices, indices, trans_vertices, trans_indices), "vxb_set_capacity")

    def set_launch_limit(self, ctas=0):
        """Test hook: at most `ctas` CTAs for the persistent kernels (0 = the default, occupancy-sized grids)."""
        self._check(self.L.vxb_set_launch_limit(self.h, ctas), "vxb_set_launch_limit")

    def run_work_items(self, level):
        """Test hook: (work items selected, blocks emitted) at `level` in the last completed run."""
        items, emitted = C.c_uint32(0), C.c_uint32(0)
        self._check(self.L.vxb_run_work_items(self.h, level, C.byref(items), C.byref(emitted)), "vxb_run_work_items")
        return items.value, emitted.value

    def polygonize(self, max_levels=0, flags=0):
        self._check(self.L.vxb_polygonize(self.h, max_levels, flags), "vxb_polygonize")
        return self.info()

    def update_blocks(self, coords, dist_blocks, mat_blocks=None, blend_blocks=None):
        """coords: uint32 [count, 3] block coordinates (x, y, z); *_blocks: uint8/int8 [count, 4096]."""
        coords = np.ascontiguousarray(coords, np.uint32)
        self._check(self.L.vxb_grid_update_blocks(self.h, len(coords), _ptr(coords), _ptr(dist_blocks), _ptr(mat_blocks), _ptr(blend_blocks)),
                    "vxb_grid_update_blocks")

    def polygonize_region(self, min_corner, max_corner, flags=0):
        lo = np.ascontiguousarray(min_corner, np.float32); hi = np.ascontiguousarray(max_corner, np.float32)
        self._check(self.L.vxb_polygonize_region(self.h, _ptr(lo), _ptr(hi), flags), "vxb_polygonize_region")
        return self.info()

    # ---- sharded runs (include/vxb200.h: vxb_polygonize_sharded, vxb_shard_*, vxb_cube_*) ----
    def shard_configure(self, rank, world, group_planes=0):
        self._check(self.L.vxb_shard_configure(self.h, rank, world, group_planes), "vxb_shard_configure")

    def shard_buffers(self):
        x = ShardBuffers()
        self._check(self.L.vxb_shard_buffers_get(self.h, C.byref(x)), "vxb_shard_buffers_get")
        return x

    def shard_set_peer(self, peer, pages, valid):
        self._check(self.L.vxb_shard_set_peer(self.h, peer, C.c_void_p(pages), C.c_void_p(valid)), "vxb_shard_set_peer")

    def shard_export(self):
        fd = C.c_int(-1)
        self._check(self.L.vxb_shard_export(self.h, C.byref(fd)), "vxb_shard_export")
        return fd.value

    def shard_import(self, peer, fd):
        self._check(self.L.vxb_shard_import(self.h, peer, fd), "vxb_shard_import")

    def shard_nccl_init(self, id_bytes, rank, world):
        nid = NcclId()
        C.memmove(C.byref(nid), bytes(id_bytes), 128)
        self._check(self.L.vxb_shard_nccl_init(self.h, C.byref(nid), rank, world), "vxb_shard_nccl_init")

    def polygonize_sharded(self, phase, flags=0):
        """phase 0 / 1 / 2: the pieces around the two exchanges; 3: the whole step (NCCL inside).  Returns 0, or
        ERR_CAPACITY from phase 2 / 3 (arenas grown: every rank repeats the run)."""
        rc = self.L.vxb_polygonize_sharded(self.h, phase, flags)
        if rc == ERR_CAPACITY and phase >= 2:
            return rc
        self._check(rc, "vxb_polygonize_sharded")
        return 0

    def cube_create(self, n, rank, world, group_planes=0):
        self._check(self.L.vxb_cube_create(self.h, n, rank, world, group_planes), "vxb_cube_create")
        self.n = n

    def cube_info(self):
        """(pieces, channels, bytes per piece of each channel)."""
        pieces, channels, sizes = C.c_uint32(0), C.c_uint32(0), (C.c_uint64 * 4)()
        self._check(self.L.vxb_cube_info(self.h, C.byref(pieces), C.byref(channels), C.byref(sizes)), "vxb_cube_info")
        return pieces.value, channels.value, list(sizes)

    def cube_export(self, channel, piece):
        fd = C.c_int(-1)
        self._check(self.L.vxb_cube_export(self.h, channel, piece, C.byref(fd)), "vxb_cube_export")
        return fd.value

    def cube_import(self, channel, piece, fd):
        self._check(self.L.vxb_cube_import(self.h, channel, piece, fd), "vxb_cube_import")

    def cube_piece(self, piece):
        """(dist, mat, blend) device addresses of a piece and its size in bytes per channel."""
        d, m, b, size = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_uint64(0)
        self._check(self.L.vxb_cube_piece(self.h, piece, C.byref(d), C.byref(m), C.byref(b), C.byref(size)), "vxb_cube_piece")
        return d.value, m.value, b.value, size.value

    def device_pointers(self):
        d, m, b = C.c_void_p(), C.c_void_p(), C.c_void_p()
        self._check(self.L.vxb_grid_device_pointers(self.h, C.byref(d), C.byref(m), C.byref(b)), "vxb_grid_device_pointers")
        return d.value, m.value, b.value

    def stream(self):
        return self.L.vxb_stream(self.h)

    def exchange_stream(self):
        return self.L.vxb_exchange_stream(self.h)

    def region_info(self):
        ri = RegionInfo()
        self._check(self.L.vxb_region_info_get(self.h, C.byref(ri)), "vxb_region_info_get")
        return ri

    def info(self):
        info = ResultInfo()
        self._check(self.L.vxb_result_info_get(self.h, C.byref(info)), "vxb_result_info_get")
        return info

    def kernel_ms(self, which):
        ms, launches = C.c_float(0), C.c_uint32(0)
        self._check(self.L.vxb_kernel_ms(self.h, which, C.byref(ms), C.byref(launches)), "vxb_kernel_ms")
        return ms.value, launches.value

    def unmapped_materials(self):
        n = self.L.vxb_result_unmapped_materials(self.h, None, 0)
        out = np.zeros(n, np.uint8)
        if n:
            self.L.vxb_result_unmapped_materials(self.h, _ptr(out), n)
        return out

    def download_begin(self):
        """vxb_result_download_begin into fresh numpy arrays: returns a Result whose records are valid at once and whose
        arenas are valid after download_end()."""
        info = self.info()
        records = np.zeros(info.block_count, RECORD_DTYPE)
        verts = np.zeros(info.vertex_span, VERTEX_DTYPE); idx = np.zeros(info.index_span, np.uint32)
        tverts = np.zeros(info.trans_vertex_span, VERTEX_DTYPE); tidx = np.zeros(info.trans_index_span, np.uint32)
        self._check(self.L.vxb_result_download_begin(self.h, _ptr(records), _ptr(verts), _ptr(idx), _ptr(tverts), _ptr(tidx)),
                    "vxb_result_download_begin")
        return Result(self.n, info, records, verts, idx, tverts, tidx)

    def download_end(self):
        self._check(self.L.vxb_result_download_end(self.h), "vxb_result_download_end")

    def download(self, into=None):
        """Device -> host copy of the directory and the arenas.  `into` may supply preallocated (pinned) buffers:
        dict with keys records/verts/idx/tverts/tidx holding int addresses."""
        info = self.info()
        records = np.zeros(info.block_count, RECORD_DTYPE)
        if into is None:
            verts = np.zeros(info.vertex_span, VERTEX_DTYPE); idx = np.zeros(info.index_span, np.uint32)
            tverts = np.zeros(info.trans_vertex_span, VERTEX_DTYPE); tidx = np.zeros(info.trans_index_span, np.uint32)
            self._check(self.L.vxb_result_download(self.h, _ptr(records), _ptr(verts), _ptr(idx), _ptr(tverts), _ptr(tidx)),
                        "vxb_result_download")
            return Result(self.n, info, records, verts, idx, tverts, tidx)
        self._check(self.L.vxb_result_download(self.h, _ptr(records), C.c_void_p(into["verts"]), C.c_void_p(into["idx"]),
                                               C.c_void_p(into["tverts"]), C.c_void_p(into["tidx"])), "vxb_result_download")
        return Result(self.n, info, records, None, None, None, None)
