/* vxb200.h - C ABI of the H100-native Transvoxel polygonizer backend (libvxb200.so).
 *
 * This is the thin extern "C" layer between host code and the sm_90a CUDA kernels: plain pointers
 * and sizes only, no C++/torch types.  It replaces the reference's hot path
 *     Voxels::Polygonizer::Execute            /root/reference/src/TransVoxelImpl.cpp:74-79, :2153-2169
 *     TransVoxelRun::Execute (level loop)     /root/reference/src/TransVoxelImpl.cpp:468-538
 * and consumes exactly what that path reads from the grid store
 *     VoxelGrid::GetBlockData / GetMaterialBlockData / IsBlockEmpty   src/VoxelGrid.h:49-55
 *     (public form: Grid::GetBlockDistanceData / GetBlockMaterialData  include/Grid.h:127-139)
 * The C++ drop-in (voxels_b200/csrc/polygonizer_host.cpp: Voxels::Polygonizer, Modification,
 * PolygonSurface, BlockPolygons with the reference's vtable order) is built on top of these calls;
 * INTEGRATION.md shows the binding a maintainer of the reference would add.
 *
 * Conventions: grid coordinates are Z-up, x fastest; output vertices are Y-up exactly as the
 * reference emits them (TransVoxelImpl.cpp:1289-1291, :1336-1360).  All functions return 0 on
 * success or a negative vxb_status; vxb_last_error() gives the text.  No function falls back to
 * the CPU: without a CUDA device every call fails with VXB_ERR_CUDA.
 */
#ifndef VXB200_H
#define VXB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct vxb_context vxb_context;

typedef enum vxb_status
{
	VXB_OK = 0,
	VXB_ERR_CUDA = -1,        /* CUDA runtime/driver error (text in vxb_last_error) */
	VXB_ERR_ARGUMENT = -2,    /* bad size (cube, power of two, >= 16), null pointer, ... */
	VXB_ERR_STATE = -3,       /* call order (no grid uploaded, no result yet, ...) */
	VXB_ERR_CAPACITY = -4     /* output arenas too small even after growing */
} vxb_status;

/* Flags of vxb_polygonize */
enum
{
	VXB_FLAG_NO_TRANSITIONS = 1,  /* do not emit transition meshes (BASELINE config 2); the reference always emits them */
	VXB_FLAG_KERNEL_TIMES = 2     /* bracket every kernel with CUDA events (vxb_kernel_ms); adds a little stream overhead */
};

/* One emitted block (a block that produced >= 1 regular vertex; reference: PushBlocksToResult
 * TransVoxelImpl.cpp:1266-1428).  Offsets index the arrays vxb_result_download fills. */
typedef struct vxb_block_record
{
	uint32_t level;
	uint32_t coord_id;            /* z*nb*nb + y*nb + x at that level (:399) */
	uint32_t id;                  /* Block id as the reference assigns it (:395-401) */
	uint32_t vertex_count;
	uint32_t index_count;         /* after the degenerate-triangle filter (:1300-1321) */
	uint32_t vertex_offset;       /* in vertices */
	uint32_t index_offset;        /* in indices */
	uint32_t trans_vertex_count[6];   /* face order = BlockPolygons::TransitionFaceId (include/Polygonizer.h:58-68) */
	uint32_t trans_index_count[6];
	uint32_t trans_vertex_offset[6];
	uint32_t trans_index_offset[6];
	uint32_t reserved;
} vxb_block_record;               /* 32 x 4 bytes */

typedef struct vxb_result_info
{
	uint32_t levels_total;        /* log2(n/16)+1 (:490) */
	uint32_t levels_computed;
	uint32_t block_count;         /* number of vxb_block_record */
	uint32_t pad;
	uint64_t vertex_span;         /* elements to allocate for each download array (spans include   */
	uint64_t index_span;          /* the gaps left by removed degenerate triangles)                 */
	uint64_t trans_vertex_span;
	uint64_t trans_index_span;
	uint64_t vertex_total;        /* exact totals over all records */
	uint64_t index_total;
	uint64_t trans_vertex_total;
	uint64_t trans_index_total;
	/* PolygonizationStatistics (include/Polygonizer.h:110-132): BlocksCalculated, TrivialCells,
	 * NonTrivialCells, DegenerateTrianglesRemoved, PerCaseCellsCount[16] */
	uint32_t stats[20];
	uint32_t used_materials[8];   /* bit per material id that occurs in an emitted vertex */
	float device_ms;              /* device time of the last vxb_polygonize (CUDA events) */
	uint32_t kernel_launches;     /* kernels launched by the last vxb_polygonize */
} vxb_result_info;

/* ---- context ------------------------------------------------------------------------------- */
int vxb_create(int device, vxb_context** out);
void vxb_destroy(vxb_context* ctx);
const char* vxb_last_error(const vxb_context* ctx);   /* ctx may be NULL: error of a failed vxb_create */
/* cudaStream_t the context launches on (as void*), for callers that time with their own events */
void* vxb_stream(vxb_context* ctx);
/* the context's second cudaStream_t (transition cells run on it next to the flat vertex / triangle kernels) */
void* vxb_exchange_stream(vxb_context* ctx);

/* ---- grid (input provider side: VoxelGrid accessors, src/VoxelGrid.h:49-55) ------------------ */
/* n^3 dense volumes in HOST memory, index (z*n + y)*n + x.  mat/blend may be NULL (zeros). */
int vxb_grid_upload_dense(vxb_context* ctx, uint32_t n, const int8_t* dist, const uint8_t* mat, const uint8_t* blend);
/* HOST memory, 16^3 blocks exactly as Grid::GetBlockDistanceData/GetBlockMaterialData return them,
 * concatenated in VoxelGrid block order (id = x + y*nb + z*nb*nb, VoxelGrid.h:139-144; 4096 B each). */
int vxb_grid_upload_blocks(vxb_context* ctx, uint32_t n, const int8_t* dist_blocks, const uint8_t* mat_blocks, const uint8_t* blend_blocks);
/* The grid in the reference's own serialised form, i.e. exactly the bytes Grid::PackForSave() returns
 * (VoxelGrid::PackForSave src/VoxelGrid.cpp:269-315: {version=1, w, d, h}, 3 x uint32 sizes per block, then per block
 * {flags, RLE distance, RLE material, RLE blend}; RLE = (length, value) byte pairs, VoxelGrid::CompressBlock :610-672).
 * HOST memory.  The blob is copied to the device as is (typically 10-30x smaller than the dense volumes) and the
 * run-length decoding (VoxelGrid::DecompressBlock :674-694) happens on the GPU. */
int vxb_grid_upload_packed(vxb_context* ctx, const void* blob, size_t size);
/* The same upload fed slab by slab, for a caller that is still gathering the grid store's blocks into `blob` (the drop-in's
 * Execute: VoxelGrid's per-block vectors -> one pinned blob).  At the call the 16-byte header and the COMPLETE size table
 * must be in place; the block data is produced on demand: before the library copies the data of the block layers
 * [layer0, layer1) (blocks layer0*nb*nb .. layer1*nb*nb-1 in VoxelGrid order) it calls produce(user, layer0, layer1) on the
 * calling thread, which must have written those blocks' {flags, distance, material, blend} bytes on return.  The copy and the
 * GPU decode of one slab run while the producer fills the next.  Layers are asked for in ascending order, each exactly once
 * (a context with a cube: only the layers of the pieces this rank backs).  produce = NULL: vxb_grid_upload_packed. */
typedef void (*vxb_pack_producer)(void* user, uint32_t layer0, uint32_t layer1);
int vxb_grid_upload_packed_streamed(vxb_context* ctx, const void* blob, size_t size, vxb_pack_producer produce, void* user);
/* Host-side helper (no GPU involved): writes the PackForSave form of dense n^3 volumes into `out` (capacity bytes).
 * Byte-identical to what the reference produces for the same voxels.  vxb_pack_dense_bound = worst-case size. */
size_t vxb_pack_dense_bound(uint32_t n);
int vxb_pack_dense(uint32_t n, const int8_t* dist, const uint8_t* mat, const uint8_t* blend, void* out, size_t capacity, size_t* written);

/* Dense volumes already resident in DEVICE memory (not copied; must stay valid; 16-byte aligned). */
int vxb_grid_set_device(vxb_context* ctx, uint32_t n, const int8_t* d_dist, const uint8_t* d_mat, const uint8_t* d_blend);
/* Device pointers of the context-owned dense volumes (after an upload), for tools/benchmarks. */
int vxb_grid_device_pointers(vxb_context* ctx, const int8_t** d_dist, const uint8_t** d_mat, const uint8_t** d_blend);

/* ---- device-resident grid store (the steps before the polygonizer; reference src/VoxelGrid.cpp) ------------------
 * A built-in procedural surface: the device-side analogue of a client's Voxels::VoxelSurface (include/VoxelSurface.h:35-40;
 * a client callback cannot run on the GPU, these can).  voxels_b200/csrc/vxb_surfaces.h evaluates them with bit-identical
 * floats on the device and on the host (the test harness serves the same functions to the unmodified reference grid store).
 *   SPHERE   p = {cx, cy, cz, r}: d = |x - c| - r             material / blend: constants
 *   PLANE    p = {nx, ny, nz, d0}: d = n . x - d0              material / blend: constants
 *   TERRAIN  p = {N, ox, oy}: the seeded Perlin terrain of BASELINE configs[1..4] (SURVEY.md 8d): heightfield 0.5 N +
 *            0.18 N fbm2 + 6 perlin3 detail, 3 material bands + ore pockets, smooth blends; N = horizontal period (the grid
 *            edge), (ox, oy) = window origin; seed = permutation table
 * Distances are clamped to +-100 before quantisation (keeps the reference's char conversion defined, VoxelGrid.cpp:37-40). */
enum { VXB_SURFACE_SPHERE = 0, VXB_SURFACE_PLANE = 1, VXB_SURFACE_TERRAIN = 2 };
typedef struct vxb_surface
{
	uint32_t kind;
	uint32_t material, blend;     /* SPHERE / PLANE */
	uint32_t seed;                /* TERRAIN */
	float p[8];
} vxb_surface;
/* Grid::Create(n, n, n, start_x, start_y, start_z, step, &surface) (VoxelGrid.cpp:79-132) into context-owned dense volumes -
 * or, when the context has a cube (sharded runs), into the pieces this rank backs: sample, round away from zero, clamp to +-4. */
int vxb_grid_fill(vxb_context* ctx, uint32_t n, const vxb_surface* surface, const float start[3], float step);
/* VoxelGrid::InjectSurface (VoxelGrid.cpp:388-488) on the device copy: position / extents in grid (Z-up) coordinates, type =
 * InjectionType (0 IT_Add, 1 IT_SubtractAddInner, 2 IT_Subtract; include/Grid.h).  The surface is sampled relative to
 * `position` exactly as the reference samples the client's surface (:419-428).  out_min / out_max = the modified box the
 * reference returns (Y-up "DX style", :479-487) = what Modification::MinCornerModified / MaxCornerModified take.
 * Needs a context-owned grid (upload or fill). */
int vxb_grid_inject_surface(vxb_context* ctx, const float position[3], const float extents[3], const vxb_surface* surface, int type,
	float out_min[3], float out_max[3]);
/* VoxelGrid::InjectMaterial (VoxelGrid.cpp:490-584). */
int vxb_grid_inject_material(vxb_context* ctx, const float position[3], const float extents[3], uint32_t material, int add_subtract_blend,
	float out_min[3], float out_max[3]);
/* Grid::PackForSave of the device grid (VoxelGrid::CompressBlock :610-672 + PackForSave :269-315): every block run-length coded on
 * the GPU (raw fallback when RLE is ineffective, BF_Empty flag), then the blob copied to HOST memory `out` (capacity bytes,
 * vxb_pack_dense_bound is enough).  Byte-identical to what the reference produces for the same voxels. */
int vxb_grid_pack(vxb_context* ctx, void* out, size_t capacity, size_t* written);
/* The dense volumes back to HOST memory (n^3 bytes each; any pointer may be NULL). */
int vxb_grid_download_dense(vxb_context* ctx, int8_t* dist, uint8_t* mat, uint8_t* blend);

/* ---- client-composed surfaces: SDF programs ---------------------------------------------------------------------------
 * A client's own VoxelSurface as data: a stack program of SDF primitives and CSG operators, evaluated on the device by the
 * fill and edit kernels and on the host by voxels_b200/csrc/vxb_program.h (the same source, bit-identical floats).  Ops run
 * in order on a value stack; every value carries the material / blend of the primitive it came from.
 *
 * Primitives (push one value).  The sample point p (grid, Z-up coordinates) is first mapped to local coordinates
 * q = M p + t, xform = rows {m0, m1, m2, t}, each component ((m_i.x * p.x + m_i.y * p.y) + m_i.z * p.z) + t_i:
 *   SPHERE    p[0] = r:               |q| - r = sqrt((qx*qx + qy*qy) + qz*qz) - r
 *   BOX       p[0..2] = half extents: e = |q| - h per axis; sqrt((mx*mx + my*my) + mz*mz) + min(max(ex, max(ey, ez)), 0)
 *                                     with m = max(e, 0) (the exact box distance)
 *   CYLINDER  p[0] = r, p[1] = half height, axis = local z: a = sqrt(qx*qx + qy*qy) - r, b = |qz| - h;
 *                                     min(max(a, b), 0) + sqrt(max(a, 0)^2 + max(b, 0)^2)
 *   CAPSULE   p[0] = r, p[1] = half length of the segment along local z: c = qz - clamp(qz, -h, h);
 *                                     sqrt((qx*qx + qy*qy) + c*c) - r
 *   TORUS     p[0] = R (ring), p[1] = r (tube), ring in the local xy plane: a = sqrt(qx*qx + qy*qy) - R; sqrt(a*a + qz*qz) - r
 *   PLANE     p[0..2] = n, p[3] = d0:  ((nx*qx + ny*qy) + nz*qz) - d0
 *   TERRAIN   p[0] = N, p[1..2] = (ox, oy), seed: VXB_SURFACE_TERRAIN evaluated at q (its own material and blend)
 * SPHERE, PLANE and TERRAIN are vxb_surface's formulas: a one-op program with M = identity and t = -centre (t = 0 for PLANE
 * and TERRAIN) gives the bytes vxb_grid_fill gives.  Every primitive value is clamped to +-100, as the final value is.
 * Operators (a = the value below the top, b = the top):
 *   UNION         min(a, b)                              material of the smaller value
 *   INTERSECT     max(a, b)                              material of the larger value
 *   SUBTRACT      max(a, -b)                             material of the side that won
 *   SMOOTH_UNION  p[0] = k > 0: h = max(k - |a - b|, 0) / k; min(a, b) - ((h*h) * k) * 0.25   material of the smaller value
 *   OFFSET        p[0] = r: d - r                        material kept
 *   SHELL         p[0] = thickness: |d| - thickness      material kept
 * Ties go to the left operand (a).  Floats: +, -, *, /, sqrt, floor and compare-selects only, in the order written.
 * Limits: at most VXB_PROGRAM_MAX_OPS ops, a stack depth of VXB_PROGRAM_MAX_DEPTH, at most VXB_PROGRAM_MAX_TERRAIN TERRAIN
 * ops.  A malformed program (NULL / empty, unknown code, stack underflow or overflow, not exactly one value at the end, a
 * non-finite float in any op, k <= 0, a negative radius / extent / thickness, N <= 0, material or blend > 255, too many
 * ops or TERRAIN ops) returns VXB_ERR_ARGUMENT naming the op index in vxb_last_error and leaves the grid untouched. */
enum
{
	VXB_OP_SPHERE = 0, VXB_OP_BOX, VXB_OP_CYLINDER, VXB_OP_CAPSULE, VXB_OP_TORUS, VXB_OP_PLANE, VXB_OP_TERRAIN,  /* push one value */
	VXB_OP_UNION = 16, VXB_OP_INTERSECT, VXB_OP_SUBTRACT, VXB_OP_SMOOTH_UNION,                               /* pop two, push one */
	VXB_OP_OFFSET = 32, VXB_OP_SHELL                                                                        /* pop one, push one */
};
enum { VXB_PROGRAM_MAX_OPS = 64, VXB_PROGRAM_MAX_DEPTH = 8, VXB_PROGRAM_MAX_TERRAIN = 2 };
typedef struct vxb_op
{
	uint32_t code, material, blend, seed;  /* material / blend: primitives; seed: TERRAIN */
	float xform[12];                       /* primitives: local = M p + t, rows {m0, m1, m2, t} */
	float p[8];                            /* shape parameters; SMOOTH_UNION p[0] = k; OFFSET p[0] = r; SHELL p[0] = thickness */
} vxb_op;                                  /* 96 bytes */
/* vxb_grid_fill with a program: the same sample coordinates, quantisation (round away from zero, clamp +-4), cube pieces
 * and bookkeeping.  Two passes: a per-block interval pass writes the 16^3 blocks it proves constant (every sample +4 or
 * every sample -4, one primitive selected throughout, not TERRAIN) and lists the others; the listed blocks are then
 * evaluated per voxel. */
int vxb_grid_fill_program(vxb_context* ctx, uint32_t n, const vxb_op* ops, uint32_t count, const float start[3], float step);
/* vxb_grid_inject_surface with a program: the same sample coordinates, combine rules for `type` and returned box. */
int vxb_grid_inject_program(vxb_context* ctx, const float position[3], const float extents[3], const vxb_op* ops, uint32_t count,
	int type, float out_min[3], float out_max[3]);
/* What the last vxb_grid_fill_program of this context did (this rank's pieces with a cube): blocks it covered, blocks the
 * interval pass wrote, and the device time of the two passes (CUDA events). */
typedef struct vxb_program_stats
{
	uint64_t blocks, culled;
	float pass_a_ms, pass_b_ms;
} vxb_program_stats;
int vxb_grid_program_stats(vxb_context* ctx, vxb_program_stats* out);

/* MaterialMap::GetMaterial pre-tabulated (include/MaterialMap.h:19-30): table = 256 x
 * {DiffuseIds0[3], DiffuseIds1[3]}, valid = 256 bytes (0 = GetMaterial returned nullptr).
 * NULL table = identity map, NULL valid = all valid. */
int vxb_set_materials(vxb_context* ctx, const uint8_t* table, const uint8_t* valid);

/* ---- polygonization -------------------------------------------------------------------------- */
/* Full run over LOD levels [0, max_levels) (0 = all, as the reference).  Results stay in device
 * arenas until the next call.  Blocks until the device work is done. */
int vxb_polygonize(vxb_context* ctx, uint32_t max_levels, uint32_t flags);
int vxb_result_info_get(vxb_context* ctx, vxb_result_info* out);

/* ---- incremental re-polygonization (Execute with a Modification, TransVoxelImpl.cpp:362-364, :429-465) ---- */
/* Replaces `count` 16^3 blocks of the context-owned grid (after an edit such as Grid::InjectSurface).
 * block_coords = count x {x, y, z} block coordinates; dist/mat/blend = count x 4096 bytes each in the same order
 * (Grid::GetBlockDistanceData / GetBlockMaterialData layout); mat and blend may be NULL (unchanged). HOST memory. */
int vxb_grid_update_blocks(vxb_context* ctx, uint32_t count, const uint32_t* block_coords, const int8_t* dist, const uint8_t* mat, const uint8_t* blend);

/* Per level: the dirty box of the last vxb_polygonize_region and the ids it handed out.  A caller that keeps a
 * surface erases its blocks whose minimal corner lies in [min_dirty, max_dirty) (:443-450) and appends the new ones;
 * ids id_start .. id_start+block_count-1 are Modification::GetModifiedBlocks (:463). Corners are OUTPUT (Y-up) coordinates. */
typedef struct vxb_region_info
{
	uint32_t levels;
	uint32_t pad;
	float min_dirty[12][3];
	float max_dirty[12][3];
	uint32_t id_start[12];
	uint32_t block_count[12];
} vxb_region_info;

/* Re-polygonizes the blocks of every level around the box [min_corner, max_corner] (Modification::MinCornerModified /
 * MaxCornerModified, OUTPUT coordinates: the box Grid::InjectSurface returns).  Needs a preceding full vxb_polygonize of
 * the same context: its consistency / material caches are updated in place exactly like the reference's PolygonMap
 * caches (bits are only ever set, votes only overwrite), block ids continue the context's running counter.  The
 * result (vxb_result_info / vxb_result_download) holds ONLY the re-created blocks; a vxb_mesh keeps the whole surface. */
int vxb_polygonize_region(vxb_context* ctx, const float min_corner[3], const float max_corner[3], uint32_t flags);
int vxb_region_info_get(vxb_context* ctx, vxb_region_info* out);

/* ---- Sharded runs: ONE grid polygonized by `world` ranks, one GPU each (SURVEY.md section 8e; BASELINE configs[3]) ----
 * The reference balances its OpenMP block loop by blocks (TransVoxelImpl.cpp:500-503); so does this: WORK is dealt by
 * blocks, independently of where the DATA lives.
 *
 * Data.  The cube (vxb_cube_*): each volume is ONE contiguous n^3 virtual range on every rank; the z-axis is cut into
 * pieces of `group_planes` planes, piece p backed by the HBM of rank p % world (cyclic, so that a terrain's surface - a
 * few z-layers - is spread over all ranks' memories) and mapped into every peer over NVLink.  Kernels and TMA tensor maps
 * address the cube exactly like a single-GPU grid.  A fourth channel holds the even-lattice copy the level-1 tiles read.
 *
 * Work.  Every rank streams its OWN pieces once (vxb_scan_kernel: flags per 16^3 block); ONE ncclAllGather makes the
 * 4-byte-per-block info complete everywhere (exchange 0).  From it every rank derives the same work split: the
 * "super-blocks" (blocks of the last level with more than 4096 blocks) in coordinate order, cut where the running count of
 * surface-crossing level-0 blocks passes total * r / world.  A rank polygonizes every level up to the super-block
 * level inside its super-blocks - the material votes of a cell only read its own children (:763-837), so this chain is
 * rank-local - and stores the pages of its super-blocks into every peer's page buffer (peer stores, exchange 1, ordered by a
 * second tiny all-gather).  The few coarse levels above are classified by every rank (identical votes), and block b of
 * level l is emitted by rank (b + l) % world.  Block ids are the reference's full-run ids (:395-401), so the directories
 * of the ranks concatenate and sort into exactly the single-GPU directory; statistics are the sum over the ranks.
 *
 *   vxb_cube_create(ctx, n, rank, world, group_planes)      reserve the ranges, back + map the local pieces (0 = n / world)
 *   vxb_cube_export / vxb_cube_import                        one POSIX file descriptor per (channel, piece), sent to the peers
 *   vxb_shard_configure(ctx, rank, world, group_planes)     work-split state + the page buffer (needs a grid: the cube, or for
 *                                                            virtual ranks of one process a shared vxb_grid_set_device)
 *   vxb_shard_export / vxb_shard_import                      the page buffer, likewise (or vxb_shard_set_peer with raw pointers)
 *   vxb_shard_nccl_unique_id / vxb_shard_nccl_init           the communicator of the two all-gathers (libnccl.so.2 via dlopen; the
 *                                                            id travels by the caller's own means, e.g. torch.distributed)
 *   vxb_polygonize_sharded(ctx, 3, flags)                    the whole step, one stream-ordered sequence (replayed as a CUDA graph)
 *   vxb_polygonize_sharded(ctx, 0 | 1 | 2, flags)            the three pieces around the two exchanges, for callers that do
 *                                                            the exchanges themselves (tests: device copies between virtual ranks):
 *                                                            after 0 gather block_info (rank r's chunk = bytes [r, r+1) * chunk_bytes),
 *                                                            after 1 synchronise all ranks; 2 blocks and delivers the result.
 * VXB_ERR_CAPACITY means the arenas were grown: every rank repeats the run. */
typedef struct vxb_nccl_id { char internal[128]; } vxb_nccl_id;   /* = ncclUniqueId */
typedef struct vxb_shard_buffers
{
	void* block_info;             /* device: one 32-bit word per level-0 block, rank-major (the layout of the all-gather) */
	uint64_t block_info_bytes;
	uint64_t chunk_bytes;         /* block_info_bytes / world */
	void* pages;                  /* device: {material id, blend} of every cell of every super-block, block-major (z,y,x) */
	uint64_t pages_bytes;
	void* valid;                  /* device: one byte per super-block */
	uint64_t valid_bytes;
	uint32_t super_level;
	uint32_t pad;
} vxb_shard_buffers;
int vxb_shard_configure(vxb_context* ctx, uint32_t rank, uint32_t world, uint32_t group_planes);
int vxb_shard_buffers_get(vxb_context* ctx, vxb_shard_buffers* out);
int vxb_shard_set_peer(vxb_context* ctx, uint32_t peer, void* pages, void* valid);
int vxb_shard_export(vxb_context* ctx, int* fd);
int vxb_shard_import(vxb_context* ctx, uint32_t peer, int fd);
int vxb_shard_nccl_unique_id(vxb_nccl_id* id);
int vxb_shard_nccl_init(vxb_context* ctx, const vxb_nccl_id* id, uint32_t rank, uint32_t world);
int vxb_polygonize_sharded(vxb_context* ctx, uint32_t phase, uint32_t flags);

/* The cube: see above.  Every piece (group_planes * n^2 bytes; the lattice channel an eighth of that) must be a multiple of
 * the allocation granularity (2 MiB); when only the lattice pieces are not, the cube has three channels and level 1 gathers
 * its tiles.  vxb_cube_info: number of pieces, channels and bytes per piece of each channel (uint64_t[4]).
 * vxb_cube_piece: device pointers of piece `piece` (any rank's: the whole cube is addressable) and its size in bytes. */
int vxb_cube_create(vxb_context* ctx, uint32_t n, uint32_t rank, uint32_t world, uint32_t group_planes);
int vxb_cube_info(vxb_context* ctx, uint32_t* pieces, uint32_t* channels, uint64_t* piece_bytes);
int vxb_cube_export(vxb_context* ctx, uint32_t channel, uint32_t piece, int* fd);
int vxb_cube_import(vxb_context* ctx, uint32_t channel, uint32_t piece, int fd);
int vxb_cube_piece(vxb_context* ctx, uint32_t piece, int8_t** dist, uint8_t** mat, uint8_t** blend, uint64_t* bytes_per_channel);
/* Copies the directory (sorted by level, then coord_id = the reference's block order) and the
 * arenas to HOST memory sized from vxb_result_info spans.  Vertices are 48-byte
 * Voxels::PolygonVertex (include/Polygonizer.h:14-48).  Any pointer may be NULL to skip it. */
int vxb_result_download(vxb_context* ctx, vxb_block_record* records, void* vertices, uint32_t* indices,
	void* trans_vertices, uint32_t* trans_indices);
/* The same download in two steps: _begin queues the copies of the arenas and returns as soon as the directory has arrived
 * and been sorted (`records` is filled), so that the caller can build its per-block views (pointers into the arenas:
 * PushBlocksToResult, src/TransVoxelImpl.cpp:1274-1293) while the arenas are still in flight; _end waits for them (and
 * restores the all-zero textures of unmapped materials).  The arenas must not be read, and no run started, in between. */
int vxb_result_download_begin(vxb_context* ctx, vxb_block_record* records, void* vertices, uint32_t* indices,
                              void* trans_vertices, uint32_t* trans_indices);
int vxb_result_download_end(vxb_context* ctx);

/* ---- consumer side: the result as indirect draws, without leaving HBM (doc_source/Rendering.md:18-58) ------------------
 * The arenas are merged vertex / index buffers: a block is drawn with {index_count, first_index, base_vertex} (indices are
 * block-local).  vxb_result_device_arenas hands the device pointers to the renderer (CUDA-graphics interop / external
 * memory).  vxb_result_select_lod runs, per frame, the cut through the LOD octree on the GPU: node of level l around the
 * camera is refined while the camera is closer than base_distance * 2^l to its centre; for every drawn block of level > 0
 * `block_adj` has bit f set when the neighbour across face f (BlockPolygons::TransitionFaceId order) is drawn finer - then
 * the block's transition mesh f is drawn too and the vertex shader selects the secondary position of the vertices whose
 * mask (SecondaryPosition.w) is covered by block_adj (Rendering.md:44-52).  Both lists are VkDrawIndexedIndirectCommand /
 * D3D12_DRAW_INDEXED_ARGUMENTS arrays with first_instance = the draw's index into the info array. */
typedef struct vxb_draw_command { uint32_t index_count, instance_count, first_index; int32_t base_vertex; uint32_t first_instance; } vxb_draw_command;
typedef struct vxb_draw_info { uint32_t block_id, level, block_adj, face; /* face = 0xFFFFFFFF: the regular mesh */ } vxb_draw_info;
typedef struct vxb_draw_lists
{
	uint32_t regular_count, transition_count;   /* also resident on the device: counts[0], counts[1] (for *IndirectCount draws) */
	const uint32_t* counts;                     /* device */
	const vxb_draw_command* regular; const vxb_draw_info* regular_info;          /* device, regular_count entries */
	const vxb_draw_command* transition; const vxb_draw_info* transition_info;    /* device, transition_count entries */
} vxb_draw_lists;
int vxb_result_device_arenas(vxb_context* ctx, const void** vertices, const uint32_t** indices, const void** trans_vertices, const uint32_t** trans_indices);
int vxb_result_select_lod(vxb_context* ctx, const float camera[3], float base_distance, vxb_draw_lists* out);
/* the two lists copied to HOST memory (tests, debugging); capacities in entries, any pointer may be NULL */
int vxb_result_download_draws(vxb_context* ctx, vxb_draw_command* regular, vxb_draw_info* regular_info, vxb_draw_command* transition, vxb_draw_info* transition_info);

/* ---- the mesh: the polygonized surface kept resident in HBM across edits -------------------------------------------------
 * The context's result holds what the LAST run made: after vxb_polygonize_region only the re-created blocks.  A mesh keeps
 * the whole surface: vxb_mesh_apply takes the context's last run into it on the GPU, in the reference's block order
 * (PolygonMap::Levels[l].Blocks after Execute, TransVoxelImpl.cpp:395-401, :443-450, :1293):
 *   after vxb_polygonize          the content is replaced by the run's blocks, per level in coord_id order
 *   after vxb_polygonize_region   per level, the blocks whose block coordinates lie in the run's dirty range (the box of
 *                                 vxb_region_info.min_dirty / max_dirty) are erased, the survivors keep their order and
 *                                 the re-created blocks follow them in coord_id order
 * The mesh copies (it never aliases the context's arenas; vxb_result_* behave as without it).  Vertices are the bytes of
 * vxb_result_download: unmapped materials have all-zero textures.  Block ids are the context's.  An apply is refused with
 * VXB_ERR_STATE, leaving the mesh untouched, when the context has no result, when the result is a sharded run's, when that
 * run was already applied, and for a region run when the mesh missed one of the context's runs since its last full run.
 * Every block's index ranges start at a multiple of 4 indices (16-byte aligned); the arenas also hold the ranges of erased
 * blocks until the next compaction (when the tail would overflow, or when the garbage exceeds the live data, the live
 * blocks are copied into a second arena set, grown to 1.5 x the live data when needed).  Pointers from
 * vxb_mesh_device_arenas and vxb_mesh_select_lod stay valid until an apply changes `generation`.  vxb_destroy releases the
 * context's meshes. */
typedef struct vxb_mesh vxb_mesh;
/* capacity: initial arena capacities in elements {vertices, indices, trans vertices, trans indices}; NULL = sized by the
 * first apply */
int vxb_mesh_create(vxb_context* ctx, const uint64_t capacity[4], vxb_mesh** out);
void vxb_mesh_destroy(vxb_mesh* mesh);
int vxb_mesh_apply(vxb_mesh* mesh);
typedef struct vxb_mesh_info
{
	uint32_t levels;              /* LOD levels of the grid the mesh was built from */
	uint32_t block_count;
	uint32_t level_blocks[12];    /* blocks per level */
	uint64_t vertex_span;         /* download sizes: the used prefix of each arena (elements) */
	uint64_t index_span;
	uint64_t trans_vertex_span;
	uint64_t trans_index_span;
	uint64_t vertex_total;        /* live elements over all blocks */
	uint64_t index_total;
	uint64_t trans_vertex_total;
	uint64_t trans_index_total;
	uint64_t capacity[4];         /* arena capacities in elements */
	uint32_t stats[20];           /* vxb_result_info.stats of the last applied run (PolygonMap::Stats after it) */
	uint32_t compactions;         /* applies that copied the live blocks into the second arena set */
	uint32_t growths;             /* applies that enlarged the arenas */
	uint64_t generation;          /* changes whenever the directory or an arena moves (growth, compaction) */
	uint64_t bytes_copied;        /* device bytes the last apply wrote into the mesh (arenas and directory) */
	float apply_ms;               /* device time of the last apply (CUDA events) */
	uint32_t pad;
} vxb_mesh_info;
int vxb_mesh_info_get(vxb_mesh* mesh, vxb_mesh_info* out);
/* The directory in mesh order (level ascending, then surface order) and the used prefix of each arena (spans of
 * vxb_mesh_info) to HOST memory; any pointer may be NULL. */
int vxb_mesh_download(vxb_mesh* mesh, vxb_block_record* records, void* vertices, uint32_t* indices, void* trans_vertices, uint32_t* trans_indices);
int vxb_mesh_device_arenas(vxb_mesh* mesh, const vxb_block_record** records, const void** vertices, const uint32_t** indices,
	const void** trans_vertices, const uint32_t** trans_indices);
/* vxb_result_select_lod over the mesh's blocks; the lists are the mesh's own (the context's stay as they are) */
int vxb_mesh_select_lod(vxb_mesh* mesh, const float camera[3], float base_distance, vxb_draw_lists* out);

/* ---- bounds and the culled select: the cut drawn only where a view sees it ---------------------------------------------
 * bounds        For every block the mesh keeps one axis-aligned box in OUTPUT (Y-up) coordinates: the component-wise min and
 *               max of pos[0..2] and sec[0..2] (the primary and the secondary position; sec[3] is the flag word) over the
 *               block's regular vertices and the transition vertices of all six faces.  It covers both positions because
 *               the vertex shader may pick either (Rendering.md:44-52), and the transition vertices so that one box serves
 *               the block's regular draw and its transition draws.  It is measured from the vertices, not taken from the
 *               block lattice: it is usually much smaller than the block (a surface fills a part of it), and it does not
 *               rest on the vertices staying inside the block at levels >= 1, where t is recomputed after the LOD descent
 *               (TransVoxelImpl.cpp:1671-1699).  Min and max are exact: the box is a pure function of the block's vertices
 *               (compare values: -0 and +0 are equal).
 *               vxb_mesh_apply computes the boxes of the blocks it takes in; a surviving block keeps its box across edits,
 *               compactions and growth; an erased block's box becomes min = +inf, max = -inf.  A renderer may read the boxes
 *               for its own passes (occlusion tests, cascade fitting): vxb_mesh_bounds_get; the pointer stays valid until an
 *               apply changes the grid size.  VXB_ERR_STATE before the first apply.
 * culled select vxb_mesh_select_lod_views builds, in one pass over the directory, one pair of draw lists per view.  The CUT is
 *               vxb_mesh_select_lod's for (lod_camera, base_distance) in every view - which blocks are drawn, block_adj,
 *               which transition meshes - so that a shadow cascade and the colour pass draw the same geometry; only the
 *               frustum differs.  A block of the cut is in view v's lists iff its box passes every plane k of the view, in
 *               float32 without fused multiply-add, in exactly this order:
 *                   c_i = n_i >= 0 ? max_i : min_i         (i = x, y, z; -0 >= 0)
 *                   s   = ((nx*cx + ny*cy) + nz*cz) + d     pass iff s >= 0
 *               Its transition draws follow it (same box).  block_adj is the cut's and does not depend on visibility: a
 *               culled neighbour is still "drawn finer".  Per view the lists are a pure function of (mesh, lod_camera,
 *               base_distance, view) as a set of (command, info) pairs; their order is unspecified; first_instance is the
 *               draw's index into its own view's info array.  The lists are the mesh's own (vxb_mesh_select_lod's and the
 *               context's stay as they are) and stay valid until the next vxb_mesh_select_lod_views or until an apply
 *               changes `generation`.  The call blocks, like vxb_mesh_select_lod.
 * Refusals (previous lists and `out` untouched): VXB_ERR_STATE before the first apply; VXB_ERR_ARGUMENT for a NULL pointer,
 * for view_count = 0 or > VXB_VIEWS_MAX, and for a non-finite plane component (vxb_last_error names the view and the plane).
 * There is no matrix input: the planes of a view-projection matrix are ten lines on the client and depend on its clip
 * conventions. */
typedef struct vxb_mesh_bounds
{
	const float* boxes;        /* DEVICE: 8 floats per (level, coord) slot: min xyz, 0, max xyz, 0; min > max for absent blocks */
	uint32_t level_base[12];   /* slot of a block = level_base[level] + coord_id */
	uint32_t slots;
	uint32_t pad;
} vxb_mesh_bounds;
int vxb_mesh_bounds_get(vxb_mesh* mesh, vxb_mesh_bounds* out);
/* tests / debugging: HOST, block_count x 6 floats {min xyz, max xyz} in directory order */
int vxb_mesh_download_bounds(vxb_mesh* mesh, float* bounds);
#define VXB_VIEWS_MAX 8
/* Six planes, each {nx, ny, nz, d} in OUTPUT coordinates, pointing INTO the view volume: a point p is inside plane k
 * iff ((nx*px + ny*py) + nz*pz) + d >= 0.  A plane {0,0,0,d>=0} passes everything (a view with fewer than six planes). */
typedef struct vxb_view { float planes[6][4]; } vxb_view;
int vxb_mesh_select_lod_views(vxb_mesh* mesh, const float lod_camera[3], float base_distance,
                              const vxb_view* views, uint32_t view_count, vxb_draw_lists* out /* view_count entries */);

/* ---- the LOD cut: a descending, balanced cut of the mesh's octree, culled against up to eight views ----------------------
 * vxb_mesh_select_cut draws the mesh at every level of detail: fine blocks near lod_camera, coarser ones farther away,
 * never two touching blocks more than one level apart, so the transition meshes close every seam (Rendering.md:23,35-38).
 * The rule.  A node (level l, grid block coordinates b) has the lattice box, in OUTPUT (Y-up) axes:
 *     s = 16 * 2^l,   lo = (bx, bz, by) * s,   hi = lo + s
 * and, in float32 without fused multiply-add, in exactly this order (c = lod_camera):
 *     e_i    = max(max(lo_i - c_i, c_i - hi_i), 0)          i = x, y, z
 *     dist2  = ((ex*ex + ey*ey) + ez*ez)
 *     lim    = lod_factor * s
 *     refine(l, b) = l > 0 && dist2 < lim*lim
 *     on the cut   = !refine(l, b) && (l == top || refine(l + 1, b >> 1))
 *     block_adj bit f (TransitionFaceId order, as above) = the same-level neighbour across face f is inside the grid and
 *                  refine(l, neighbour)
 * In words: a node is refined while the camera is closer than lod_factor times its edge length to its box (0 inside it).
 * Monotone, also in float32.  A child's box lies inside its parent's box, so every lo_i - c_i and c_i - hi_i of the child is
 * at most the parent's; rounding is monotone, so every e_i, each product and each sum can only grow from the parent to the
 * child.  The child's lim is exactly half the parent's (s is a power of two), so its lim*lim is at most the parent's.  Hence
 * refine(child) implies refine(parent), and by induction every ancestor's.  That is why "on the cut" is the O(1) test
 * above: a node whose parent refines has every ancestor refining, with no loop over the ancestors; and the cut tiles the
 * grid, every level-0 block lying under exactly one node of the cut.
 * Balanced for lod_factor >= sqrt(3).  Let N (level l, edge s_l) be on the cut and touch (share a face, an edge or a
 * corner with) a cut node of level <= l - 2.  That node's ancestor P of level l - 1 refines (a node of the cut has every
 * ancestor refining) and touches N (it contains the touching node, and it is not inside N, whose descendants do not refine).  The distance from the camera
 * to a box grows by at most the diameter of the boxes it is measured across, so with k = lod_factor
 *     dist(N) <= dist(P) + diam(P) < k*s_l/2 + sqrt(3)*s_l/2 = (k + sqrt(3))*s_l/2 <= k*s_l    for k >= sqrt(3),
 * which contradicts N not refining.  So every pair of touching cut nodes differs by at
 * most one level, and the finer neighbours a drawn block's block_adj names are exactly one level finer - the case the
 * transition meshes are made for.  The call refuses lod_factor < VXB_LOD_FACTOR_MIN (a margin over sqrt(3) against the
 * rounding of the float formula), NaN and infinity.
 * Choosing lod_factor.  A cell of a level-l block spans 2^l voxels and the block's edge is 16 cells, so where the block stops
 * refining (distance lod_factor * s) a cell covers about H / (32 * tan(theta / 2) * lod_factor) pixels of a viewport H
 * pixels high with a vertical field of view theta.  For at most p pixels per cell: lod_factor = H / (32 * tan(theta / 2) * p);
 * e.g. 1080 px, 60 degrees, 4 px per cell: 14.6.
 * Views.  The culling is vxb_mesh_select_lod_views', unchanged: a block of the cut is in view v's lists iff its box passes
 * every plane of the view (the p-vertex test above); its transition draws follow it; block_adj is the cut's and does not
 * depend on visibility; the order within a list is unspecified; first_instance is the draw's index into its own view's
 * info array.  For an unculled cut pass one view of pass-everything planes.
 * Buffers.  The lists are the call's own device buffers (per view block_count regular and 6 x block_count transition
 * entries); they stay valid until the next vxb_mesh_select_cut or until an apply changes `generation`, and the call leaves
 * the lists of vxb_mesh_select_lod and vxb_mesh_select_lod_views as they are.  The call blocks (one read of the counts).
 * Refusals (previous lists and `out` untouched): VXB_ERR_STATE before the first apply, and when the mesh does not hold
 * every level with its transition meshes - some run applied since the last full apply had max_levels below the grid's
 * levels or VXB_FLAG_NO_TRANSITIONS (the next complete full run and apply lift it); VXB_ERR_ARGUMENT for a NULL pointer,
 * view_count = 0 or > VXB_VIEWS_MAX, a non-finite plane component (vxb_last_error names the view and the plane), a
 * non-finite lod_camera component, and a bad lod_factor. */
#define VXB_LOD_FACTOR_MIN 2.0f
int vxb_mesh_select_cut(vxb_mesh* mesh, const float lod_camera[3], float lod_factor,
                        const vxb_view* views, uint32_t view_count, vxb_draw_lists* out /* view_count entries */);

/* ---- ray queries against the mesh: picking, line of sight, projectile hits, without leaving HBM ------------------------
 * Rays are cast against the LEVEL-0 regular triangles of the mesh (the full-detail surface, the one edits change); levels >= 1
 * and transition meshes are not part of the query.
 *   The hit     over every level-0 triangle that passes the test below, the one with the least t; ties go to the lower slot,
 *               then to the lower triangle.  A pure function of the mesh (content and order) and the ray: it does not depend
 *               on the launch configuration, on the variant or on the other rays of the batch.  Both faces are hit (no
 *               back-face culling).  A miss: slot = VXB_RAY_MISS, t = +inf, every other field zero.
 *   The test    Moeller-Trumbore in float32, in exactly this order (no fused multiply-add, IEEE division and square root):
 *                 p0, p1, p2 = pos of vertices index[3k], index[3k+1], index[3k+2] (+ vertex_offset)
 *                 e1 = p1 - p0; e2 = p2 - p0; s = o - p0                                   (per component)
 *                 pv = d x e2: pvx = dy*e2z - dz*e2y; pvy = dz*e2x - dx*e2z; pvz = dx*e2y - dy*e2x
 *                 det = (e1x*pvx + e1y*pvy) + e1z*pvz; inv = 1 / det
 *                 u = ((sx*pvx + sy*pvy) + sz*pvz) * inv
 *                 qv = s x e1 (same pattern): qvx = sy*e1z - sz*e1y; qvy = sz*e1x - sx*e1z; qvz = sx*e1y - sy*e1x
 *                 v = ((dx*qvx + dy*qvy) + dz*qvz) * inv
 *                 t = ((e2x*qvx + e2y*qvy) + e2z*qvz) * inv
 *                 hit iff det != 0 && u >= 0 && u <= 1 && v >= 0 && u + v <= 1 && t >= t_min && t <= t_max
 *               (positive comparisons: a NaN - a tiny det makes inv infinite and u NaN - fails the test).
 *   position    o_i + t * d_i
 *   normal      w = (1 - u) - v; n_i = (w*n0_i + u*n1_i) + v*n2_i; len = sqrt((nx*nx + ny*ny) + nz*nz); n_i / len if len > 0,
 *               else (0, 0, 0)
 * A level-0 triangle lies in the closed box of its block.  The walk tests the triangles of every block whose box, grown by
 * 1/16 voxel, meets the segment; an accepted hit lies within rounding of its triangle (far less than 1/16 voxel unless det
 * is close to zero), so this is every triangle that can pass the test.
 * Refusals: VXB_ERR_STATE before the first vxb_mesh_apply; VXB_ERR_ARGUMENT for a NULL pointer with count > 0; count = 0 does
 * nothing.  The HOST variant also refuses with VXB_ERR_ARGUMENT, naming the ray index in vxb_last_error and writing nothing to
 * `hits`, a ray with a non-finite origin or direction, a zero direction, a NaN or non-finite t_min, a NaN t_max or
 * t_min > t_max.  The DEVICE variant cannot read the rays before it runs: there such a ray is a miss.
 * The first cast after an apply (or after the mesh changed grid size) also rebuilds a per-mesh map from level-0 block
 * coordinates to slots ((n/16)^3 x 4 bytes: 1 MB at 1024^3), stream-ordered before the cast. */
/* One ray in OUTPUT (Y-up) coordinates, the space of the vertices and of vxb_mesh_select_lod's camera.  The direction
 * need not be unit length; t is in units of it.  The ray is the segment origin + t * direction, t in [t_min, t_max]
 * (both inclusive; t_max may be +inf). */
typedef struct vxb_ray { float origin[3]; float t_min; float direction[3]; float t_max; } vxb_ray;          /* 32 bytes */
#define VXB_RAY_MISS 0xFFFFFFFFu   /* a macro, not an enum: ISO C limits enumerators to the range of int */
typedef struct vxb_ray_hit
{
	float t, u, v;          /* ray parameter; barycentrics of the triangle's 2nd and 3rd vertex */
	uint32_t slot;          /* mesh directory slot of the block (vxb_mesh_device_arenas / vxb_mesh_download order); VXB_RAY_MISS */
	uint32_t block_id;      /* vxb_block_record.id of that block */
	uint32_t triangle;      /* k: the triangle is indices [index_offset + 3k, index_offset + 3k + 3) of the block */
	float position[3];      /* origin + t * direction */
	float normal[3];        /* the vertex normals blended at (u, v), normalised; (0,0,0) when the blend is zero */
} vxb_ray_hit;                                                                                               /* 48 bytes */
/* HOST memory; blocks until the hits are written. */
int vxb_mesh_raycast(vxb_mesh* mesh, const vxb_ray* rays, uint32_t count, vxb_ray_hit* hits);
/* DEVICE memory; enqueued on vxb_stream(ctx) after everything queued there (an apply included), returns without waiting.
 * The mesh's state at the call is what the cast sees: a later apply is queued after it. */
int vxb_mesh_raycast_device(vxb_mesh* mesh, const vxb_ray* rays, uint32_t count, vxb_ray_hit* hits);

/* ---- ray queries against the drawn LOD cut: picking what the renderer shows --------------------------------------------
 * vxb_mesh_raycast answers about the level-0 surface; where the renderer draws coarser blocks (vxb_mesh_select_cut) the
 * drawn surface differs from it by up to a cell of the drawn level (2^l voxels).  vxb_mesh_raycast_cut casts against the
 * triangles the renderer draws for the cut of (lod_camera, lod_factor), so that a cursor or a marker lands on what is seen.
 *   The drawn set   The cut is exactly vxb_mesh_select_cut's for (lod_camera, lod_factor): the same refine, the same "on the
 *                   cut" test and the same block_adj; view culling plays no part.  For every block of the cut, the drawn
 *                   set is its regular triangles and, for every face f with bit f of block_adj set, the triangles of its
 *                   transition mesh f.  Every vertex (regular or transition) takes the position the vertex shader selects
 *                   (Rendering.md:48-54): with mask = the bits of sec[3], sec[0..2] when mask != 0 and (mask & block_adj) ==
 *                   mask, otherwise pos.
 *   The hit         The test, position, normal and miss value are vxb_mesh_raycast's, on the selected positions (the normal
 *                   blends the vertices' nrm, which both positions share).  Least t wins; ties go to the lower slot, then to
 *                   the lower part (the regular mesh before transition face 0, ..., face 5), then to the lower triangle.  A
 *                   pure function of the mesh (content and order), of (lod_camera, lod_factor) and of the ray: not of the
 *                   launch, the variant or the rest of the batch.  A miss: slot = VXB_RAY_MISS, t = +inf, every other field
 *                   (level and face too) zero.
 *   At lod_factor = 1e30, lim*lim overflows to +inf, so every node above level 0 refines: the cut is all of level 0 with
 *                   block_adj = 0 and no transition draws.  There the first 48 bytes of every hit equal vxb_mesh_raycast's,
 *                   with level = 0 and face = 0xFFFFFFFF on a hit.
 *   The walk        At levels >= 1 a drawn vertex is not proven to stay inside its block's lattice box (t is recomputed after
 *                   the LOD descent), so the cast rests on the mesh's bounds (the measured boxes above) and on the excursion
 *                   e: the largest distance by which any block's measured box leaves its lattice box.  The first cut cast
 *                   after an apply (or after the mesh changed grid size) rebuilds a map from every (level, coord) slot of the
 *                   bounds to the directory (bounds.slots x 4 bytes: 1.2 MB at 1024^3) and measures e, and WAITS for the
 *                   stream once to read e back.  Later casts until the next apply do not wait (the device variant).
 * Refusals (`hits` untouched): VXB_ERR_STATE before the first apply, when the mesh does not hold every level with its
 * transition meshes (as vxb_mesh_select_cut), and when e + 1/16 exceeds 15 voxels, the reach of the walk (vxb_last_error
 * names e); VXB_ERR_ARGUMENT for a NULL pointer with count > 0, a lod_factor below VXB_LOD_FACTOR_MIN or not finite, and a
 * non-finite lod_camera component.  count = 0 does nothing.  The HOST variant also refuses an invalid ray as
 * vxb_mesh_raycast does, naming its index; on the DEVICE variant such a ray is a miss. */
typedef struct vxb_cut_hit
{
	float t, u, v;          /* as vxb_ray_hit */
	uint32_t slot;          /* mesh directory slot of the drawn block; VXB_RAY_MISS */
	uint32_t block_id;      /* vxb_block_record.id of that block */
	uint32_t triangle;      /* k: indices [part offset + 3k, +3) of the part `face` names (index_offset or trans_index_offset[face]) */
	float position[3];      /* origin + t * direction */
	float normal[3];        /* as vxb_ray_hit */
	uint32_t level;         /* the hit block's level */
	uint32_t face;          /* 0xFFFFFFFF: the regular mesh; f: the transition mesh of face f (TransitionFaceId order) */
} vxb_cut_hit;                                                                      /* 56 bytes; the first 48 are vxb_ray_hit's */
/* HOST memory; blocks until the hits are written. */
int vxb_mesh_raycast_cut(vxb_mesh* mesh, const float lod_camera[3], float lod_factor,
                         const vxb_ray* rays, uint32_t count, vxb_cut_hit* hits);
/* DEVICE memory; enqueued on vxb_stream(ctx) like vxb_mesh_raycast_device (the first cast after an apply waits, see above). */
int vxb_mesh_raycast_cut_device(vxb_mesh* mesh, const float lod_camera[3], float lod_factor,
                                const vxb_ray* rays, uint32_t count, vxb_cut_hit* hits);

/* ---- collision queries against the mesh: sphere sweeps and closest points, for character controllers and cameras -------
 * Like the ray queries: the LEVEL-0 regular triangles only, both faces, OUTPUT (Y-up) coordinates, a pure function of the
 * mesh (content and order) and of the query (not of the launch, the variant or the rest of the batch), float32 with no fused
 * multiply-add, IEEE division and square root, in exactly the order written here.  x.y = (xx*yx + xy*yy) + xz*yz with the
 * left operand as written; a x b = (ay*bz - az*by, az*bx - ax*bz, ax*by - ay*bx).
 *   Closest point of triangle (a, b, c) (p0, p1, p2 as for the rays) to a point p: Ericson's ClosestPtPointTriangle, the
 *   regions tested in this order, the first that holds gives point, u (weight of b) and v (weight of c):
 *     ab = b - a; ac = c - a; ap = p - a; d1 = ab.ap; d2 = ac.ap
 *     A    d1 <= 0 && d2 <= 0                                  point = a, u = 0, v = 0
 *          bp = p - b; d3 = ab.bp; d4 = ac.bp
 *     B    d3 >= 0 && d4 <= d3                                 point = b, u = 1, v = 0
 *          vc = d1*d4 - d3*d2
 *     AB   vc <= 0 && d1 >= 0 && d3 <= 0                       w = d1 / (d1 - d3); point_i = a_i + w*ab_i, u = w, v = 0
 *          cp = p - c; d5 = ab.cp; d6 = ac.cp
 *     C    d6 >= 0 && d5 <= d6                                 point = c, u = 0, v = 1
 *          vb = d5*d2 - d1*d6
 *     AC   vb <= 0 && d2 >= 0 && d6 <= 0                       w = d2 / (d2 - d6); point_i = a_i + w*ac_i, u = 0, v = w
 *          va = d3*d6 - d5*d4
 *     BC   va <= 0 && (d4 - d3) >= 0 && (d5 - d6) >= 0         w = (d4 - d3) / ((d4 - d3) + (d5 - d6));
 *                                                              point_i = b_i + w*(c_i - b_i), u = 1 - w, v = w
 *     face otherwise                                           den = 1 / ((va + vb) + vc); u = vb*den; v = vc*den;
 *                                                              point_i = (a_i + ab_i*u) + ac_i*v
 *   and dd = (qx*qx + qy*qy) + qz*qz with q = p - point.
 *   Normal: the ray hit's blended normal at (u, v).
 *
 *   vxb_mesh_closest_point: for a query point p and max_distance m, every level-0 triangle with dd <= m*m (inclusive, m*m
 *     in float) is a candidate; the result is the one with the least dd, then the lower slot, then the lower triangle, with
 *     distance = sqrt(dd).  A miss: slot = VXB_RAY_MISS, distance = +inf, every other field zero.  This is the query for
 *     resolving penetration (the depth is r - distance for a sphere of radius r at p).
 *
 *   vxb_mesh_sphere_cast: a sphere of radius r whose centre moves along c(t) = o_i + t*d_i, t in [t_min, t_max] (a vxb_ray,
 *     the same validity rules).  With c0_i = o_i + t_min*d_i, rr = r*r and dd_d = (dx*dx + dy*dy) + dz*dz, each triangle's
 *     contact t is:
 *       started in contact   the closest point of the triangle to c0 has dd <= rr: t = t_min, and the hit's flags have
 *                            VXB_SPHERE_STARTED_IN_CONTACT.
 *       otherwise            the least of these, each +inf when it fails:
 *         face     e1 = b - a; e2 = c - a; n = e1 x e2; len = sqrt((nx*nx + ny*ny) + nz*nz); side = (c0 - a).n;
 *                  k = side >= 0 ? r : -r; o'_i = o_i - k*(n_i / len); Moeller-Trumbore of the ray (o', d) exactly as for the
 *                  ray queries, giving det, u, v, t, accepted iff (side >= 0 ? det > 0 : det < 0) && u >= 0 && u <= 1 &&
 *                  v >= 0 && u + v <= 1 && t >= t_min && t <= t_max (the plane offset by r toward the side the sphere
 *                  starts on, approached; a zero-area triangle makes len 0 and fails)
 *         edges    ab, bc, ca in turn, for the edge q0 -> q1: e = q1 - q0; w = o - q0; ee = e.e; de = d x e; we = w x e;
 *                  A = de.de; B = de.we; g = d.we; disc = ee * (rr*A - g*g); t = (-B - sqrt(disc)) / A;
 *                  s = ((wx + t*dx)*ex + (wy + t*dy)*ey) + (wz + t*dz)*ez;
 *                  accepted iff A > 0 && disc >= 0 && s >= 0 && s <= ee && t >= t_min && t <= t_max
 *         vertices a, b, c in turn, for the vertex q: w = o - q; B = w.d; x = w x d; disc = rr*dd_d - x.x;
 *                  t = (-B - sqrt(disc)) / dd_d; accepted iff dd_d > 0 && disc >= 0 && t >= t_min && t <= t_max
 *                            (both discriminants are the Lagrange-identity forms, which keep their precision for
 *                            origins far from the triangle).
 *     A triangle with a finite contact t is a candidate; the hit is the one with the least t, then the lower slot, then the
 *     lower triangle.  Sweeps that start in contact with several triangles therefore report the lowest slot, not the deepest
 *     penetration: use vxb_mesh_closest_point for that.  center_i = o_i + t*d_i; point, u and v are the closest point of
 *     the triangle to center (the contact point; center - point is the contact normal); normal as for the closest point.
 *     A miss: slot = VXB_RAY_MISS, t = +inf, every other field zero.
 *
 * The walk of the sweeps is the ray cast's block walk with the block boxes grown by r + 1/16 voxel instead of 1/16: a
 * contact puts the centre within r of its triangle's block.  VXB_SPHERE_RADIUS_MAX caps r and max_distance at 15 voxels so
 * that every block within reach of a point stays within one block of that point's block (27 neighbours, as for the rays).
 * Refusals: as for the ray queries (VXB_ERR_STATE before the first vxb_mesh_apply; VXB_ERR_ARGUMENT for a NULL pointer with
 * count > 0; count = 0 does nothing; the same map rebuild), and VXB_ERR_ARGUMENT on both variants for a radius outside
 * 0 < r <= 15 or a max_distance outside 0 <= m <= 15 (NaN and infinities included).  The HOST variants refuse an invalid
 * sweep (the ray rules) or a point with a non-finite coordinate, naming its index in vxb_last_error; the DEVICE variants
 * return a miss for it.  A refused call writes nothing to `hits`. */
#define VXB_SPHERE_RADIUS_MAX 15.0f          /* sweeps and closest-point queries reach at most this far (voxels) */
#define VXB_SPHERE_STARTED_IN_CONTACT 1u     /* vxb_sphere_hit.flags */
typedef struct vxb_sphere_hit
{
	float t;                /* centre = origin + t * direction at the first contact */
	uint32_t slot;          /* as vxb_ray_hit; VXB_RAY_MISS */
	uint32_t block_id;
	uint32_t triangle;
	float center[3];        /* origin + t * direction */
	float point[3];         /* the contact point: the closest point of the triangle to `center` */
	float normal[3];        /* the vertex normals blended at (u, v), the ray hit's formula */
	float u, v;             /* barycentrics of `point` (2nd and 3rd vertex) */
	uint32_t flags;         /* VXB_SPHERE_STARTED_IN_CONTACT */
} vxb_sphere_hit;                                                                                            /* 64 bytes */
typedef struct vxb_closest_hit
{
	float distance;         /* |query - point|; +inf on a miss */
	uint32_t slot;          /* as vxb_ray_hit; VXB_RAY_MISS */
	uint32_t block_id;
	uint32_t triangle;
	float point[3];         /* the closest point of the level-0 surface within max_distance */
	float normal[3];        /* the vertex normals blended at (u, v), the ray hit's formula */
	float u, v;             /* barycentrics of `point` (2nd and 3rd vertex) */
} vxb_closest_hit;                                                                                           /* 48 bytes */
/* HOST memory; block until the hits are written.  `points` is count x 3 floats. */
int vxb_mesh_sphere_cast(vxb_mesh* mesh, float radius, const vxb_ray* rays, uint32_t count, vxb_sphere_hit* hits);
int vxb_mesh_closest_point(vxb_mesh* mesh, float max_distance, const float* points, uint32_t count, vxb_closest_hit* hits);
/* DEVICE memory; enqueued on vxb_stream(ctx) like vxb_mesh_raycast_device: they see the mesh as of their place in the queue. */
int vxb_mesh_sphere_cast_device(vxb_mesh* mesh, float radius, const vxb_ray* rays, uint32_t count, vxb_sphere_hit* hits);
int vxb_mesh_closest_point_device(vxb_mesh* mesh, float max_distance, const float* points, uint32_t count, vxb_closest_hit* hits);

/* ---- capsule queries against the mesh: capsule sweeps and closest points to segments, for capsule character controllers ---
 * A capsule is the segment [c - h, c + h] (c = centre, h = half axis: any direction, zero allowed) with a radius r.  Like the
 * collision queries above: LEVEL-0 regular triangles only, both faces, OUTPUT (Y-up) coordinates, a pure function of the mesh
 * and the query, float32 with no fused multiply-add in exactly the order written here, the same dot and cross products, and
 * the same tie rule (least t or dd, then the lower slot, then the lower triangle).
 *   Closest pair of the segment (c, h) and triangle (a, b, c_) - one routine for both queries and the sweep's start test.
 *     p0_i = c_i - h_i; p1_i = c_i + h_i; D_i = h_i + h_i.  Candidates, in this order, each a triangle point `point` with
 *     barycentrics (u, v), a segment parameter w in [0, 1] and a dd:
 *       1  p0: the closest point of the triangle to p0 (the collision queries' routine), dd = |p0 - point|^2, w = 0
 *       2  p1: the same for p1, w = 1
 *       3  the edges ab, bc, ca in turn (Ericson's ClosestPtSegmentSegment, exact zero tests for his epsilons), for the edge
 *          q0 -> q1: E = q1 - q0; R = p0 - q0; A = D.D; e = E.E; f = E.R.  A == 0: no candidate (1 gives the distance).
 *          Otherwise c = D.R and, if e == 0: t = 0, w = clamp(-c / A); else b = D.E; den = A*e - b*b;
 *          w = den != 0 ? clamp((b*f - c*e) / den) : 0; t = (b*w + f) / e; t < 0: t = 0, w = clamp(-c / A);
 *          else t > 1: t = 1, w = clamp((b - c) / A).  clamp(x) = x < 0 ? 0 : (x > 1 ? 1 : x).
 *          X_i = p0_i + w*D_i; point_i = q0_i + t*E_i; dd = |X - point|^2; (u, v) = (t, 0) on ab, (1 - t, t) on bc, (0, 1 - t)
 *          on ca.
 *       4  the segment crossing the triangle: Moeller-Trumbore of the ray queries from p0 along D (s = p0 - a, e1 = b - a,
 *          e2 = c_ - a), giving det, u, v and w, accepted iff det != 0 && u >= 0 && u <= 1 && v >= 0 && u + v <= 1 && w >= 0
 *          && w <= 1; dd = 0, point_i = (a_i + e1_i*u) + e2_i*v.
 *     The result is the candidate with the least dd, the first in this order on a tie; s = (w + w) - 1 and
 *     axis_point_i = c_i + s*h_i.  With h = 0 only candidates 1 and 2 exist and agree, so the result is the collision
 *     queries' closest point bit for bit (s = -1).
 *
 *   vxb_mesh_closest_to_segment: every triangle whose dd is at most max_distance*max_distance (in float) is a candidate; the
 *     result is the least dd by the tie rule, distance = sqrt(dd).  The penetration depth of a capsule is r - distance.
 *
 *   vxb_mesh_capsule_cast: the capsule's centre moves along the path (a vxb_ray, the same rules), its half axis and radius fixed.
 *     It touches triangle T when the sphere of radius r at the centre touches P = T + [-h, h] (Minkowski sum).  With
 *     c0_i = o_i + t_min*d_i:
 *       started in contact   the closest pair at c0 has dd <= r*r: t = t_min, flags = VXB_SPHERE_STARTED_IN_CONTACT.
 *       otherwise            the least t of these tests, each the sphere sweep's formula (and +inf when it fails):
 *         faces     the caps (a - h, b - h, c_ - h) and (a + h, b + h, c_ + h), then the parallelograms of ab, bc, ca:
 *                   for the edge q0 -> q1 the sphere's face test on the vertices (q0 - h, q1 - h, q0 + h), with u <= 1 and
 *                   v <= 1 in place of u + v <= 1 (the parallelogram q0 - h, q1 - h, q1 + h, q0 + h).
 *         edges     the cap edges ab, bc, ca of the cap -h, the same of the cap +h, then the lateral edges a - h -> a + h,
 *                   b - h -> b + h, c_ - h -> c_ + h.
 *         vertices  a - h, b - h, c_ - h, a + h, b + h, c_ + h.
 *       (shifted points per component: q_i - h_i, q_i + h_i).  Every feature lies in P, so no test fires before the first
 *       contact; the faces cover P, so the first contact is on one of them or on their edges and vertices.  With h = 0 the
 *       t is the sphere sweep's bit for bit: the parallelograms and lateral edges fail through det = 0 and A = 0.
 *     The hit: t, center_i = o_i + t*d_i, and point, axis_point, u, v and s of the closest pair at that centre; normal as for
 *     the closest point.  Ties of several triangles as for the sphere sweep.
 * A miss: slot = VXB_RAY_MISS, t (distance) = +inf, every other field zero.
 * Reach: a sweep is valid when r > 0 and max_i |h_i| + r <= VXB_SPHERE_RADIUS_MAX, a segment when max_i |h_i| +
 * max_distance <= VXB_SPHERE_RADIUS_MAX (both sums in float); a contact puts the centre within |h_i| + r of its triangle
 * along axis i, so every block within reach stays one of the 27 neighbours of the centre's block.  The sweep walk grows the
 * block boxes by max_i |h_i| + r + 1/16.
 * Refusals: VXB_ERR_STATE before the first vxb_mesh_apply; VXB_ERR_ARGUMENT for a NULL pointer with count > 0 (count = 0
 * does nothing) and, on both variants, for a max_distance outside 0 <= m <= 15.  The HOST variants refuse a query with an
 * invalid path (the ray rules), a non-finite half axis or radius, a shape out of reach, or a non-finite centre, naming its
 * index in vxb_last_error and writing nothing to `hits`; the DEVICE variants return a miss for it. */
typedef struct vxb_capsule_sweep
{
	vxb_ray path;           /* the centre's path */
	float half_axis[3];     /* h: the segment is centre -+ h */
	float radius;           /* r > 0 */
} vxb_capsule_sweep;                                                                                         /* 48 bytes */
typedef struct vxb_segment { float center[3]; float half_axis[3]; } vxb_segment;                           /* 24 bytes */
typedef struct vxb_capsule_hit
{
	float t;                /* centre = origin + t * direction at the first contact */
	uint32_t slot;          /* as vxb_ray_hit; VXB_RAY_MISS */
	uint32_t block_id;
	uint32_t triangle;
	float center[3];        /* path.origin + t * path.direction */
	float point[3];         /* the contact point on the triangle */
	float axis_point[3];    /* the point of the capsule's segment paired with it: center + s * half_axis */
	float normal[3];        /* the vertex normals blended at (u, v), the ray hit's formula */
	float u, v, s;          /* barycentrics of `point`; s in [-1, 1] */
	uint32_t flags;         /* VXB_SPHERE_STARTED_IN_CONTACT */
} vxb_capsule_hit;                                                                                           /* 80 bytes */
typedef struct vxb_segment_hit
{
	float distance;         /* sqrt(dd) of the closest pair; +inf on a miss */
	uint32_t slot;          /* as vxb_ray_hit; VXB_RAY_MISS */
	uint32_t block_id;
	uint32_t triangle;
	float point[3];         /* the closest point of the level-0 surface within max_distance of the segment */
	float axis_point[3];    /* the segment's point paired with it: center + s * half_axis */
	float normal[3];        /* the vertex normals blended at (u, v), the ray hit's formula */
	float u, v, s;          /* barycentrics of `point`; s in [-1, 1] */
} vxb_segment_hit;                                                                                           /* 64 bytes */
/* HOST memory; block until the hits are written. */
int vxb_mesh_capsule_cast(vxb_mesh* mesh, const vxb_capsule_sweep* sweeps, uint32_t count, vxb_capsule_hit* hits);
int vxb_mesh_closest_to_segment(vxb_mesh* mesh, float max_distance, const vxb_segment* segments, uint32_t count, vxb_segment_hit* hits);
/* DEVICE memory; enqueued on vxb_stream(ctx) like vxb_mesh_raycast_device: they see the mesh as of their place in the queue. */
int vxb_mesh_capsule_cast_device(vxb_mesh* mesh, const vxb_capsule_sweep* sweeps, uint32_t count, vxb_capsule_hit* hits);
int vxb_mesh_closest_to_segment_device(vxb_mesh* mesh, float max_distance, const vxb_segment* segments, uint32_t count, vxb_segment_hit* hits);

/* ---- collision queries against the drawn LOD cut: sphere sweeps and closest points on what the renderer shows -------------
 * The collision queries above answer about the level-0 surface; where the renderer draws coarser blocks the drawn surface
 * differs from it by up to a cell of the drawn level.  vxb_mesh_sphere_cast_cut and vxb_mesh_closest_point_cut answer about
 * the triangles the renderer draws for the cut of (lod_camera, lod_factor), so that a camera boom stops at the hill the
 * player sees and a marker snapped to the surface sits on the drawn triangles.
 *   The drawn set   vxb_mesh_raycast_cut's: the cut of (lod_camera, lod_factor) as vxb_mesh_select_cut makes it (view culling
 *                   plays no part), each cut block's regular triangles and the transition meshes its block_adj names, every
 *                   vertex at the position the vertex shader selects (sec when its mask is non-zero and covered by
 *                   block_adj, pos otherwise).
 *   The tests       vxb_mesh_sphere_cast's sweep (start in contact, the offset face, the three edge cylinders, the three
 *                   vertex spheres) and vxb_mesh_closest_point's closest point (Ericson's routine, dd <= m*m inclusive),
 *                   unchanged, on the selected positions.  center, point, u, v and the blended normal are computed as there,
 *                   on the drawn triangle's nrm (both positions share it).
 *   The hit         Least t (sweeps) or dd (points); ties go to the lower slot, then to the lower part (the regular mesh
 *                   before transition face 0, ..., face 5), then to the lower triangle: vxb_mesh_raycast_cut's rule.  A pure
 *                   function of the mesh (content and order), of (lod_camera, lod_factor) and of the query: not of the
 *                   launch, the variant or the rest of the batch.  A miss is the level-0 query's miss with level and face 0.
 *   At lod_factor = 1e30 the cut is all of level 0 with block_adj = 0, so the first 64 bytes (sweeps) or 48 bytes (points) of
 *                   every hit equal vxb_mesh_sphere_cast's or vxb_mesh_closest_point's, with level = 0 and face = 0xFFFFFFFF
 *                   on a hit.
 *   The reach       The walk rests on the measured boxes and the excursion e as vxb_mesh_raycast_cut's does, with every box
 *                   grown by the query's reach R (the radius r for sweeps, max_distance m for points): a block within reach
 *                   of a query point then stays within e + R + 1/16 < 16 voxels of it, one of the 27 neighbours of its block.
 *                   The first cut query after an apply (of any of the three kinds) rebuilds the all-level map, measures e
 *                   and waits for the stream once.
 * Refusals (`hits` untouched), arguments first: VXB_ERR_ARGUMENT for a NULL pointer with count > 0, a bad lod_factor or
 * lod_camera (as vxb_mesh_raycast_cut), a radius outside 0 < r <= 15 or a max_distance outside 0 <= m <= 15 (as the
 * collision queries); VXB_ERR_STATE before the first apply and for a mesh without every level and transition mesh (as
 * vxb_mesh_select_cut); then, after the map, VXB_ERR_STATE when e + 1/16 > 15 (as vxb_mesh_raycast_cut) or when e + R > 15
 * in float (vxb_last_error names e and R).  count = 0 does nothing.  The HOST variants also refuse an invalid sweep (the ray
 * rules) or a point with a non-finite coordinate, naming its index; on the DEVICE variants such a query is a miss. */
typedef struct vxb_sphere_cut_hit
{
	float t;                /* as vxb_sphere_hit: the first 64 bytes are its fields */
	uint32_t slot;          /* mesh directory slot of the drawn block; VXB_RAY_MISS */
	uint32_t block_id;
	uint32_t triangle;      /* k: indices [part offset + 3k, +3) of the part `face` names (as vxb_cut_hit) */
	float center[3];
	float point[3];         /* the closest point of the drawn triangle to `center` */
	float normal[3];
	float u, v;
	uint32_t flags;         /* VXB_SPHERE_STARTED_IN_CONTACT */
	uint32_t level;         /* the hit block's level */
	uint32_t face;          /* 0xFFFFFFFF: the regular mesh; f: the transition mesh of face f (TransitionFaceId order) */
} vxb_sphere_cut_hit;                                                       /* 72 bytes; the first 64 are vxb_sphere_hit's */
typedef struct vxb_closest_cut_hit
{
	float distance;         /* as vxb_closest_hit: the first 48 bytes are its fields */
	uint32_t slot;
	uint32_t block_id;
	uint32_t triangle;
	float point[3];         /* the closest point of the drawn surface within max_distance */
	float normal[3];
	float u, v;
	uint32_t level, face;   /* as vxb_sphere_cut_hit */
} vxb_closest_cut_hit;                                                     /* 56 bytes; the first 48 are vxb_closest_hit's */
/* HOST memory; block until the hits are written.  `points` is count x 3 floats. */
int vxb_mesh_sphere_cast_cut(vxb_mesh* mesh, const float lod_camera[3], float lod_factor, float radius,
                             const vxb_ray* rays, uint32_t count, vxb_sphere_cut_hit* hits);
int vxb_mesh_closest_point_cut(vxb_mesh* mesh, const float lod_camera[3], float lod_factor, float max_distance,
                               const float* points, uint32_t count, vxb_closest_cut_hit* hits);
/* DEVICE memory; enqueued on vxb_stream(ctx) like vxb_mesh_raycast_cut_device (the first cut query after an apply waits). */
int vxb_mesh_sphere_cast_cut_device(vxb_mesh* mesh, const float lod_camera[3], float lod_factor, float radius,
                                    const vxb_ray* rays, uint32_t count, vxb_sphere_cut_hit* hits);
int vxb_mesh_closest_point_cut_device(vxb_mesh* mesh, const float lod_camera[3], float lod_factor, float max_distance,
                                      const float* points, uint32_t count, vxb_closest_cut_hit* hits);

/* ---- capsule queries against the drawn LOD cut: capsule sweeps and closest points to segments on what the renderer shows --
 * The capsule queries above answer about the level-0 surface; a capsule character standing on a drawn level-l block would
 * float above the triangles on screen or sink into them by up to 2^l voxels, and its penetration depth r - distance would
 * be measured against a surface nobody sees.  vxb_mesh_capsule_cast_cut and vxb_mesh_closest_to_segment_cut answer about the
 * triangles the renderer draws for the cut of (lod_camera, lod_factor).
 *   The drawn set   vxb_mesh_raycast_cut's (see "collision queries against the drawn LOD cut").
 *   The tests       vxb_mesh_capsule_cast's sweep (the closest pair at c0; the caps, the parallelograms, the cap and lateral
 *                   edges, the shifted vertices) and vxb_mesh_closest_to_segment's closest pair, unchanged, on the selected
 *                   positions.  center, point, axis_point, u, v, s and the blended normal are computed as there, on the
 *                   drawn triangle's nrm.
 *   The hit         Least t (sweeps) or dd (segments); ties go to the lower slot, then to the lower part (the regular mesh
 *                   before transition face 0, ..., face 5), then to the lower triangle: vxb_mesh_raycast_cut's rule.  level
 *                   and face as in vxb_sphere_cut_hit.  A miss is the level-0 query's miss with level and face 0.
 *   At lod_factor = 1e30 the first 80 bytes (sweeps) or 64 bytes (segments) of every hit equal vxb_mesh_capsule_cast's or
 *                   vxb_mesh_closest_to_segment's, with level = 0 and face = 0xFFFFFFFF on a hit.
 *   The reach       A query's reach R is max_i |h_i| + r for a sweep and max_i |h_i| + max_distance for a segment.  Unlike
 *                   the sphere cut's radius, R travels with each query, so the cut reach rule is per query: a query is in
 *                   reach when it passes the level-0 capsule queries' rule and, in float and in this order,
 *                   e + (max_i |h_i| + r) <= 15 (sweeps) or e + (max_i |h_i| + max_distance) <= 15 (segments), e the mesh's
 *                   excursion.  With h = 0 this is the sphere cut's e + R <= 15.  A contact or closest pair then puts the
 *                   centre within e + R + 1/16 < 16 voxels of the drawn block's lattice box, one of the 27 neighbours of
 *                   its block.  The first cut query after an apply (of any kind) rebuilds the all-level map, measures e and
 *                   waits for the stream once.
 * Refusals (`hits` untouched), in this order: VXB_ERR_ARGUMENT for a NULL pointer with count > 0, a bad lod_factor or
 * lod_camera (as vxb_mesh_raycast_cut), and a max_distance outside 0 <= m <= 15; VXB_ERR_STATE before the first apply and
 * for a mesh without every level and transition mesh (as vxb_mesh_select_cut); count = 0 does nothing; the HOST variants'
 * per-query rule of vxb_mesh_capsule_cast and vxb_mesh_closest_to_segment (VXB_ERR_ARGUMENT, naming the index); after the
 * map, VXB_ERR_STATE when e + 1/16 > 15 and, for segments, when e + max_distance > 15; then, HOST variants only,
 * VXB_ERR_STATE for the first query out of cut reach (vxb_last_error names its index, e and its R).
 * The DEVICE variants answer an invalid query and a query out of cut reach with a miss and the rest of the batch as usual.
 * This differs from vxb_mesh_sphere_cast_cut_device, whose one radius serves the whole batch, so that there the whole call
 * is refused. */
typedef struct vxb_capsule_cut_hit
{
	float t;                /* as vxb_capsule_hit: the first 80 bytes are its fields */
	uint32_t slot;          /* mesh directory slot of the drawn block; VXB_RAY_MISS */
	uint32_t block_id;
	uint32_t triangle;      /* k: indices [part offset + 3k, +3) of the part `face` names (as vxb_cut_hit) */
	float center[3];
	float point[3];         /* the contact point on the drawn triangle */
	float axis_point[3];    /* center + s * half_axis */
	float normal[3];
	float u, v, s;
	uint32_t flags;         /* VXB_SPHERE_STARTED_IN_CONTACT */
	uint32_t level;         /* the hit block's level */
	uint32_t face;          /* 0xFFFFFFFF: the regular mesh; f: the transition mesh of face f (TransitionFaceId order) */
} vxb_capsule_cut_hit;                                                     /* 88 bytes; the first 80 are vxb_capsule_hit's */
typedef struct vxb_segment_cut_hit
{
	float distance;         /* as vxb_segment_hit: the first 64 bytes are its fields */
	uint32_t slot;
	uint32_t block_id;
	uint32_t triangle;
	float point[3];         /* the closest point of the drawn surface within max_distance of the segment */
	float axis_point[3];
	float normal[3];
	float u, v, s;
	uint32_t level, face;   /* as vxb_capsule_cut_hit */
} vxb_segment_cut_hit;                                                     /* 72 bytes; the first 64 are vxb_segment_hit's */
/* HOST memory; block until the hits are written. */
int vxb_mesh_capsule_cast_cut(vxb_mesh* mesh, const float lod_camera[3], float lod_factor,
                              const vxb_capsule_sweep* sweeps, uint32_t count, vxb_capsule_cut_hit* hits);
int vxb_mesh_closest_to_segment_cut(vxb_mesh* mesh, const float lod_camera[3], float lod_factor, float max_distance,
                                    const vxb_segment* segments, uint32_t count, vxb_segment_cut_hit* hits);
/* DEVICE memory; enqueued on vxb_stream(ctx) like vxb_mesh_raycast_cut_device (the first cut query after an apply waits). */
int vxb_mesh_capsule_cast_cut_device(vxb_mesh* mesh, const float lod_camera[3], float lod_factor,
                                     const vxb_capsule_sweep* sweeps, uint32_t count, vxb_capsule_cut_hit* hits);
int vxb_mesh_closest_to_segment_cut_device(vxb_mesh* mesh, const float lod_camera[3], float lod_factor, float max_distance,
                                           const vxb_segment* segments, uint32_t count, vxb_segment_cut_hit* hits);

/* ---- box overlap gathers: the level-0 triangles in axis-aligned boxes, for a client's physics mid-phase and navmesh tiles --
 * Every other query returns one answer per query; vxb_mesh_overlap_box returns, per box, every triangle that overlaps it, so
 * that a physics engine runs its own narrowphase for its own shapes (processAllTriangles-style callbacks), a navmesh builder
 * rebuilds the tiles around an edit, and a decal clips what it covers.
 *   Scope       The LEVEL-0 regular triangles only, both faces, OUTPUT (Y-up) coordinates.  The query box is closed.
 *   The test    A separating-axis test in float32 with no fused multiply-add, in exactly this order, with p0, p1, p2 the pos
 *               of vertices index[3k], index[3k+1], index[3k+2] (+ vertex_offset):
 *     1  box axes, exact (no arithmetic): for each i, min(p0_i, p1_i, p2_i) <= max_i && max(p0_i, p1_i, p2_i) >= min_i,
 *        else no overlap.
 *     2  box frame: c_i = (min_i + max_i) * 0.5; h_i = max_i*0.5 - min_i*0.5 (finite for every finite box, unlike
 *        (max_i - min_i) * 0.5); v_k = p_k - c per component; e0 = v1 - v0, e1 = v2 - v1, e2 = v0 - v2.
 *     3  the axes, in this order: the normal n = e0 x e1 (the collision queries' cross product), then u_i x e_j for i = x, y, z
 *        (outer) and j = 0, 1, 2 (inner), written with their literal zero:
 *            u_x x e = (0, -e_z, e_y);   u_y x e = (e_z, 0, -e_x);   u_z x e = (-e_y, e_x, 0).
 *        For an axis a: s_k = (a_x*v_k.x + a_y*v_k.y) + a_z*v_k.z for k = 0, 1, 2 (all three vertices on every axis: in float
 *        the two vertices of an edge do not project equally, so Akenine-Moller's two-vertex shortcut is not taken);
 *        r = (h_x*|a_x| + h_y*|a_y|) + h_z*|a_z|; the axis separates iff (s0 > r && s1 > r && s2 > r) || (s0 < -r && s1 < -r
 *        && s2 < -r), i.e. min(s) > r || max(s) < -r with positive comparisons (a NaN s never separates).
 *     4  the triangle overlaps iff no axis separates.  A zero axis (a degenerate edge, a collinear triangle) never separates.
 *   A kernel may drop the products with a literal zero component: h and v are finite, so such a product is +-0, and
 *   x + (+-0) == x.  At most the sign of a zero s or r changes, which no comparison above sees.
 *   The result  offsets has count + 1 entries: the exclusive prefix sum of the boxes' triangle counts, offsets[count] = the
 *               total; tris[offsets[q] .. offsets[q+1]) are the triangles of box q, in ascending coord_id of their block (grid
 *               order), then ascending triangle index.  A pure function of the mesh (content and order) and the box: not of the
 *               launch, the variant or the other boxes of the batch.
 *   Capacity    tris == NULL (with capacity == 0) counts only and returns VXB_OK.  The HOST variant returns VXB_ERR_CAPACITY
 *               when offsets[count] > capacity; it still writes `offsets` (size tris from offsets[count] and repeat) and
 *               leaves `tris` untouched.  The DEVICE variant always writes `offsets` and writes `tris` only when offsets[count]
 *               <= capacity, decided on the device, with no host synchronisation: compare the two when reading them.
 *   The walk    An accepted triangle's vertices lie in its block's closed lattice box and in its measured box (the bounds
 *               above), and they meet the query box (test 1).  So the candidates are the blocks whose closed lattice box
 *               meets the query box, clipped to the grid, and a candidate whose measured box misses the query box is skipped.
 *               Both tests are exact: the gather needs no epsilon.  There is no limit on box size; a box partly or wholly
 *               outside the grid is legal.  One box is walked by one warp, so a single very large box takes as long as its
 *               blocks and triangles take one warp.  The level-0 map is the ray queries'.
 * Refusals (`offsets` and `tris` untouched): VXB_ERR_STATE before the first vxb_mesh_apply; VXB_ERR_ARGUMENT for a NULL boxes
 * or offsets, or a NULL tris with capacity > 0, when count > 0; count = 0 does nothing.  The HOST variant refuses a box with
 * a non-finite component or min_i > max_i (NaN included), naming its index in vxb_last_error; on the DEVICE variant such a
 * box has 0 triangles. */
typedef struct vxb_box { float min[3]; float max[3]; } vxb_box;                          /* 24 bytes, OUTPUT (Y-up) coordinates */
typedef struct vxb_overlap_triangle
{
	float p[3][3];          /* pos of the triangle's three vertices, index order */
	uint32_t slot;          /* mesh directory slot, as vxb_ray_hit */
	uint32_t block_id;      /* vxb_block_record.id */
	uint32_t triangle;      /* k: indices [index_offset + 3k, +3) of the block */
} vxb_overlap_triangle;                                                                  /* 48 bytes */
/* HOST memory; blocks.  offsets: count + 1 entries. */
int vxb_mesh_overlap_box(vxb_mesh* mesh, const vxb_box* boxes, uint32_t count,
                         uint64_t* offsets, vxb_overlap_triangle* tris, uint64_t capacity);
/* DEVICE memory; enqueued on vxb_stream(ctx) like the other _device queries (it sees the mesh as of its place in the queue),
 * returns without waiting. */
int vxb_mesh_overlap_box_device(vxb_mesh* mesh, const vxb_box* boxes, uint32_t count,
                                uint64_t* offsets, vxb_overlap_triangle* tris, uint64_t capacity);

/* GetMaterial(id) == nullptr handling (TransVoxelImpl.cpp:1364-1368: textures stay zero, one LS_Error log per
 * vertex): after vxb_result_download the material ids of those vertices, in the reference's logging order
 * (level, block, regular vertices, then transition faces), can be read here.  Returns the count; copies at
 * most `capacity` ids. */
uint64_t vxb_result_unmapped_materials(vxb_context* ctx, uint8_t* ids, uint64_t capacity);

/* Page-locked host memory for the upload/download buffers (plain cudaHostAlloc/cudaFreeHost). */
void* vxb_host_alloc(size_t bytes);
void vxb_host_free(void* p);

/* Initial arena capacities in elements (0 = keep default).  Arenas grow and the run repeats
 * automatically on overflow; this only avoids the retry. */
int vxb_set_capacity(vxb_context* ctx, uint64_t vertices, uint64_t indices, uint64_t trans_vertices, uint64_t trans_indices);

/* Test hook: caps the grid of the persistent kernels (vxb_block_kernel<0|1|2>, vxb_big_block_kernel,
 * vxb_transition_kernel and the flat vertex / triangle kernels) at `ctas` CTAs; 0 = the occupancy-sized grid (the
 * default).  The cap only ever lowers a grid, so every CTA of a launch stays resident, as the coarse levels' waits
 * for their children need.  With a few CTAs each one walks many work items, so small grids exercise the code that
 * runs only from a CTA's second item on.  The output does not depend on it. */
int vxb_set_launch_limit(vxb_context* ctx, uint32_t ctas);

/* Test hook: the block walk of the last completed run at `level`: *items = the blocks it selected as work items of the
 * per-block kernel, *emitted = the blocks that kernel found a non-trivial cell in (and emitted).  Levels from the first
 * coarse level on are walked inside the coarse kernel, which selects no list: *items is 0 there.  Sharded runs: this
 * rank's counts.  Either pointer may be NULL. */
int vxb_run_work_items(vxb_context* ctx, uint32_t level, uint32_t* items, uint32_t* emitted);

/* Per-kernel device time of the last vxb_polygonize run with VXB_FLAG_KERNEL_TIMES, for bench.py's roofline line:
 * which = 0: vxb_scan_kernel (streams the level-0 distance volume once), 1: block info, sign-mix pyramid + selection kernels,
 * 2: vxb_block_kernel<1>/<2> (levels >= 1: classification, votes, decisions) + vxb_big_block_kernel, 3: vxb_block_kernel<0>
 * (level 0: classification, decisions, vertices and triangles in one pass), 4: vxb_vertex_kernel (levels >= 1),
 * 5: vxb_triangle_kernel (levels >= 1), 6: vxb_transition_kernel + vertices, 7: vxb_finish_kernel; sharded runs (phase 3) also
 * 8: exchange 0 (lattice publication + ncclAllGather of the block info), 9: exchange 1 (page publication + the ordering all-gather).
 * Milliseconds, summed per kind. */
int vxb_kernel_ms(vxb_context* ctx, int which, float* ms, uint32_t* launches);

#ifdef __cplusplus
}
#endif
#endif /* VXB200_H */
