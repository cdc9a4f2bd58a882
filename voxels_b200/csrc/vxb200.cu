// libvxb200.so - host side of the C ABI declared in include/vxb200.h: context, device memory,
// kernel launches (CUDA stream + events), result directory.  No CPU fallback: every entry point
// needs a CUDA device.  Kernels live in vxb_kernels.cuh.
#include <cuda_runtime.h>
#include <cuda.h> // CUtensorMap types only; cuTensorMapEncodeTiled is resolved through the runtime (no libcuda link)

#include <dlfcn.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "../../include/vxb200.h"

// the Transvoxel tables twice: __constant__ (generic kernel, uniform-ish reads) and plain global memory
// (vxbG*: divergent per-thread lookups go through L1 instead of serialising in the constant cache)
#define VXB_TABLE_QUAL __constant__
#include "vxb_tables_data.h"
#undef VXB_TABLE_QUAL
#undef VXB_TABLE_NAME
#define VXB_TABLE_QUAL __device__
#define VXB_TABLE_NAME(x) vxbG##x
#include "vxb_tables_data.h"
#include "vxb_cell.h"
#include "vxb_kernels.cuh"
#include "vxb_emit.cuh"
#include "vxb_grid.cuh"
#include "vxb_draw.cuh"
#include "vxb_mesh.cuh"
#include "vxb_ray.cuh"
#include "vxb_collide.cuh"
#include "vxb_cutray.cuh"
#include "vxb_query.cuh"
#include "vxb_overlap.cuh"

static_assert(sizeof(VxbVertex) == 48, "PolygonVertex layout");
static_assert(sizeof(vxb_block_record) == 128, "record layout");
static_assert(sizeof(vxb_ray) == 32 && sizeof(vxb_ray_hit) == 48, "ray layouts");
static_assert(sizeof(vxb_sphere_hit) == 64 && sizeof(vxb_closest_hit) == 48, "collision layouts");
static_assert(sizeof(vxb_capsule_sweep) == 48 && sizeof(vxb_segment) == 24 && sizeof(vxb_capsule_hit) == 80 && sizeof(vxb_segment_hit) == 64,
	"capsule layouts");
static_assert(sizeof(vxb_view) == 96 && sizeof(vxb_mesh_bounds) == 64 && VXB_MAX_LEVELS == 12, "view and bounds layouts");
static_assert(sizeof(vxb_cut_hit) == 56 && offsetof(vxb_cut_hit, level) == 48, "vxb_cut_hit layout");
static_assert(sizeof(vxb_sphere_cut_hit) == 72 && offsetof(vxb_sphere_cut_hit, level) == 64 && sizeof(vxb_closest_cut_hit) == 56 &&
	offsetof(vxb_closest_cut_hit, level) == 48, "cut collision layouts");
static_assert(sizeof(vxb_capsule_cut_hit) == 88 && offsetof(vxb_capsule_cut_hit, level) == 80 && sizeof(vxb_segment_cut_hit) == 72 &&
	offsetof(vxb_segment_cut_hit, level) == 64, "cut capsule layouts");
static_assert(sizeof(vxb_box) == 24 && sizeof(vxb_overlap_triangle) == 48, "overlap layouts");

namespace
{
std::string g_createError;

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
	const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// device buffers free themselves; release() is for code that frees one early on purpose.  Not copyable (the move
// assignment deletes the copies); movable, so that a struct of buffers can be reset to a fresh one (releaseShard).
template <typename T>
struct DevBuf
{
	T* p = nullptr;
	size_t count = 0;
	DevBuf& operator=(DevBuf&& o) noexcept { release(); std::swap(p, o.p); std::swap(count, o.count); return *this; }
	~DevBuf() { release(); }
	cudaError_t ensure(size_t want)
	{
		if (want <= count) return cudaSuccess;
		if (p) cudaFree(p);
		p = nullptr; count = 0;
		const cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&p), want * sizeof(T));
		if (e == cudaSuccess) count = want;
		return e;
	}
	void release() { if (p) cudaFree(p); p = nullptr; count = 0; }
};
}

struct vxb_context
{
	int device = 0;
	int smCount = 0;
	cudaStream_t stream = nullptr, stream2 = nullptr;
	cudaEvent_t evBegin = nullptr, evEnd = nullptr, evDir = nullptr;
	cudaEvent_t evFork = nullptr, evJoin = nullptr;               // the transition cells on stream2
	cudaEvent_t evLatticeFork = nullptr, evLatticeJoin = nullptr; // the coarse levels' lattices on stream2
	std::vector<cudaEvent_t> evChunks; // packed upload: one per z-chunk
	std::vector<cudaEvent_t> kevents; // per-kernel timing (pairs)
	std::string error;
	EncodeTiledFn encodeTiled = nullptr;

	uint32_t n = 0;
	int levels = 0;
	bool haveGrid = false, ownsGrid = false;
	const int8_t* dDist = nullptr; const uint8_t* dMat = nullptr; const uint8_t* dBlend = nullptr;
	DevBuf<uint8_t> volDist, volMat, volBlend, staging;
	DevBuf<unsigned long long> packOffsets;
	DevBuf<float> fillColumns;
	DevBuf<unsigned int> progList, progCount;       // vxb_grid_fill_program: blocks left to the per-voxel pass + their count
	cudaEvent_t progEv[3] = { nullptr, nullptr, nullptr };
	vxb_program_stats progStats = { 0, 0, 0.f, 0.f };
	DevBuf<vxb_draw_command> drawCmd, drawTCmd;
	DevBuf<vxb_draw_info> drawInfo, drawTInfo;
	DevBuf<unsigned int> drawCounts;
	vxb_draw_lists drawLists;
	VxbDev lastDev; // kernel-side view of the last run (records, arenas), for the consumer-side kernels
	DevBuf<unsigned int> packSizes, packFlags, packError;
	struct PinnedBuf // page-locked host scratch (grows, never shrinks, frees itself)
	{
		void* p = nullptr; size_t bytes = 0;
		PinnedBuf& operator=(PinnedBuf&&) = delete; // and with it the copies
		~PinnedBuf() { if (p) cudaFreeHost(p); }
		bool ensure(size_t want)
		{
			if (want <= bytes) return true;
			if (p) cudaFreeHost(p);
			p = nullptr; bytes = 0;
			if (cudaHostAlloc(&p, want, cudaHostAllocDefault) != cudaSuccess) { p = nullptr; return false; }
			bytes = want; return true;
		}
	} hostOffsets, hostRecords;
	DevBuf<unsigned int> scanFlags;
	DevBuf<unsigned int> blockInfo;
	DevBuf<unsigned int> consPages;
	DevBuf<unsigned char> validFlags; // consValid + cacheValid[l] packed
	DevBuf<unsigned short> cachePages;
	DevBuf<unsigned int> worklist, emitList, bigList, transList, ntScratch, cellBlock, vlist;
	DevBuf<VxbCellRec> cellRecs;
	DevBuf<uint2> tvlist;
	DevBuf<VxbBlockRec> blockRecs;
	DevBuf<VxbVertex> verts, tverts;
	DevBuf<unsigned int> idx, tidx;
	DevBuf<vxb_block_record> records;
	DevBuf<VxbCounters> counters;
	DevBuf<VxbMaterialLut> lut;
	uint64_t capV = 0, capI = 0, capTV = 0, capTI = 0;
	CUtensorMap tmap, tmap1, tmapDist19;
	DevBuf<uint8_t> lattice1;
	uint8_t* latticePtr = nullptr;  // lattice1.p, or the cube's fourth channel
	bool haveLattice1 = false, latticeOff = false;
	int gridBlock[3] = { 0, 0, 0 }, gridBigBlock = 0, gridTransition = 0;
	uint32_t launchLimit = 0;      // vxb_set_launch_limit: cap on the persistent kernels' grids (0 = none)
	uint32_t runWork[VXB_MAX_LEVELS] = { 0 }, runEmit[VXB_MAX_LEVELS] = { 0 }; // vxb_run_work_items: the last run's counters
	unsigned persistentGrid(int grid) const { return launchLimit ? std::min<unsigned>((unsigned)grid, launchLimit) : (unsigned)grid; }
	DevBuf<unsigned char> mixInfo, coarseDone;
	DevBuf<unsigned short> mixCount;
	// lattices of the coarse levels (VxbDev::coarseLattice): own buffer, or - sharded runs - an area of the buffer the peers map
	DevBuf<unsigned char> coarseLatticeBuf;
	DevBuf<CUtensorMap> coarseMaps;
	unsigned char* coarseLatticeBase = nullptr;
	size_t coarseLatticeOff[VXB_MAX_LEVELS] = { 0 }, coarseLatticeBytes = 0;
	int coarseLo = 2;
	uint64_t capC = 0;
	bool haveFullRun = false;      // device caches (consistency / material pages) describe the current grid
	uint32_t nextId = 0;           // PolygonMap::GetNextBlockId (TransVoxelImpl.cpp:149-152)
	vxb_region_info region;
	DevBuf<unsigned int> updCoords;
	bool directoryFetched = false;
	bool downloadOpen = false;            // between vxb_result_download_begin and _end
	void* downloadVerts = nullptr;
	void* downloadTransVerts = nullptr;
	// sharded runs (vxb_shard_*)
	struct Shard
	{
		bool on = false;
		uint32_t rank = 0, world = 1, groupLayers = 0; // groups of groupLayers level-0 block layers, dealt cyclically
		int sbLevel = 0;                               // super-block level = coarseLo - 1
		DevBuf<unsigned char> sbMine;
		DevBuf<unsigned int> sbWeight;
		// level-sbLevel pages + valid flags in ONE buffer the peers can map: VMM allocation (real ranks) or cudaMalloc (virtual ranks)
		unsigned char* pagesBuf = nullptr; size_t pagesBytes = 0, validBytes = 0, latticeBytes = 0, bufBytes = 0;
		// the layout of that buffer, this rank's (base = pagesBuf) or a peer's (base = its pages):
		// pages | valid flags | coarse lattices | barrier area (8 peer slots, the epoch at +64, the CTA arrival counter at +128)
		static const size_t barrierBytes = 256;
		size_t barrierOffset() const { return pagesBytes + validBytes + latticeBytes; }
		unsigned short* pages(void* base) const { return static_cast<unsigned short*>(base); }
		unsigned char* valid(void* base) const { return static_cast<unsigned char*>(base) + pagesBytes; }
		unsigned char* lattices(void* base) const { return valid(base) + validBytes; }
		unsigned char* barrier(void* base) const { return static_cast<unsigned char*>(base) + barrierOffset(); }
		unsigned long long* slots(void* base) const { return reinterpret_cast<unsigned long long*>(barrier(base)); }
		unsigned long long* epoch() const { return reinterpret_cast<unsigned long long*>(barrier(pagesBuf) + 64); }
		unsigned int* arrived() const { return reinterpret_cast<unsigned int*>(barrier(pagesBuf) + 128); }
		bool pagesVmm = false;
		CUdeviceptr pagesVa = 0; CUmemGenericAllocationHandle pagesHandle = 0;
		unsigned short* peerPages[8] = { nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr };
		unsigned char* peerValid[8] = { nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr };
		bool peerSet[8] = { false, false, false, false, false, false, false, false };
		std::vector<std::pair<CUdeviceptr, size_t> > peerMapped;
		std::vector<CUmemGenericAllocationHandle> peerHandles;
		void* comm = nullptr;                          // ncclComm_t
		uint32_t phaseLaunches = 0;
	} shard;
	// the launch sequence of a full run as a CUDA graph, re-instantiated when any kernel argument changes
	cudaGraphExec_t graphExec = nullptr;
	std::vector<unsigned char> graphKey;
	uint32_t graphLaunches = 0, graphKindLaunches[10] = { 0, 0, 0, 0, 0, 0, 0, 0, 0, 0 }; // what a replay reports
	bool graphDisabled = false;
	// the cube of a sharded run (vxb_cube_*): one virtual range per volume, this rank's slab local, peers' slabs imported
	struct Cube
	{
		bool active = false, lattice = false;
		uint32_t rank = 0, world = 1, n = 0;
		uint32_t groupPlanes = 0, pieces = 0;          // piece p = planes [p * groupPlanes, (p + 1) * groupPlanes), owner p % world
		CUdeviceptr va[4] = { 0, 0, 0, 0 };            // distance, material, blend, even lattice ((n/2)^3)
		size_t vaBytes[4] = { 0, 0, 0, 0 };
		std::vector<CUmemGenericAllocationHandle> local[4]; // this rank's pieces, in order of local index (piece = rank + k * world)
		std::vector<CUmemGenericAllocationHandle> imported;
		std::vector<std::pair<CUdeviceptr, size_t> > mapped; // every mapped piece
		size_t pieceBytes(int channel) const { return channel < 3 ? (size_t)groupPlanes * n * n : (size_t)(groupPlanes / 2) * (n / 2) * (n / 2); }
	} cube;

	bool haveResult = false;
	uint64_t runSerial = 0;                 // counts the runs (vxb_polygonize*), so that a mesh can tell whether it missed one
	bool resultSharded = false, resultRegion = false;
	bool resultComplete = false;            // the last run made every level and the transition meshes (vxb_mesh_select_cut)
	std::vector<vxb_mesh*> meshes;          // released by vxb_destroy
	vxb_result_info info;
	std::vector<vxb_block_record> sortedRecords;
	uint8_t lutValid[256];
	std::vector<uint8_t> unmapped; // material ids of vertices whose material had no mapping, in logging order
	float kindMs[10] = { 0, 0, 0, 0, 0, 0, 0, 0, 0, 0 };        // 8, 9: the two exchanges of a sharded run
	uint32_t kindLaunches[10] = { 0, 0, 0, 0, 0, 0, 0, 0, 0, 0 };
};

namespace
{
int fail(vxb_context* ctx, int code, const char* what, cudaError_t e = cudaSuccess)
{
	char buf[512];
	if (e != cudaSuccess) snprintf(buf, sizeof(buf), "%s: %s", what, cudaGetErrorString(e));
	else snprintf(buf, sizeof(buf), "%s", what);
	if (ctx) ctx->error = buf; else g_createError = buf;
	return code;
}

#define VXB_CUDA(ctx, call) do { const cudaError_t e_ = (call); if (e_ != cudaSuccess) return fail(ctx, VXB_ERR_CUDA, #call, e_); } while (0)

bool validSize(uint32_t n) { return n >= 16 && n <= 4096 && (n & (n - 1)) == 0; }

int levelsFor(uint32_t n) { int l = 1; for (uint32_t v = n >> 4; v >>= 1;) ++l; return l; }


int ensureGridStorage(vxb_context* ctx, uint32_t n)
{
	const size_t vol = (size_t)n * n * n;
	VXB_CUDA(ctx, ctx->volDist.ensure(vol));
	VXB_CUDA(ctx, ctx->volMat.ensure(vol));
	VXB_CUDA(ctx, ctx->volBlend.ensure(vol));
	ctx->dDist = reinterpret_cast<const int8_t*>(ctx->volDist.p);
	ctx->dMat = ctx->volMat.p; ctx->dBlend = ctx->volBlend.p;
	ctx->n = n; ctx->levels = levelsFor(n);
	// haveGrid becomes true only when an upload has completed (a failed upload leaves no half-filled grid behind)
	ctx->ownsGrid = true; ctx->haveGrid = false; ctx->haveResult = false; ctx->haveFullRun = false;
	return VXB_OK;
}


int encodeTileMap(vxb_context* ctx, CUtensorMap* map, const void* base, uint32_t n, uint32_t rows = 17, uint32_t pitch = VXB_TILE_PITCH)
{
	const cuuint64_t dims[3] = { n, n, n };
	const cuuint64_t strides[2] = { n, (cuuint64_t)n * n };
	const cuuint32_t box[3] = { pitch, rows, rows };
	const cuuint32_t estr[3] = { 1, 1, 1 };
	const CUresult r = ctx->encodeTiled(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<void*>(base), dims, strides, box, estr,
		CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
	if (r != CUDA_SUCCESS)
	{
		char buf[128]; snprintf(buf, sizeof(buf), "cuTensorMapEncodeTiled failed: CUresult %d", (int)r);
		return fail(ctx, VXB_ERR_CUDA, buf);
	}
	return VXB_OK;
}

size_t blocksAtLevel(uint32_t n, int level) { const size_t nb = (n / 16) >> level; return nb * nb * nb; }

// coarse levels: from the first level with <= 512 blocks (but not below 2) everything runs in one launch
int coarseLoFor(uint32_t n, int levels)
{
	int lo = 2;
	while (lo < levels && blocksAtLevel(n, lo) > 512) ++lo;
	return lo;
}

// level l owns entries [blockBase[l], +blocks[l]) of every per-block array of a run (VxbDev::workBase = idBase, written
// into `dev`) and of a mesh (VxbMeshRange::levelBase); its valid flags, material pages and sign-mix bytes (levels >= 1)
// start at validOff / pageOff / mixOff; the coarse levels' blocks (>= coarseLo) are numbered from coarseBase[l]
struct LevelLayout
{
	size_t blocks[VXB_MAX_LEVELS], blockBase[VXB_MAX_LEVELS], validOff[VXB_MAX_LEVELS], pageOff[VXB_MAX_LEVELS];
	size_t mixOff[VXB_MAX_LEVELS], coarseBase[VXB_MAX_LEVELS];
	size_t totalBlocks = 0, validBytes = 0, pageEntries = 0, mixBytes = 0, coarseBlocks = 0;
};

LevelLayout levelLayout(uint32_t n, int levels, int coarseLo, VxbDev* dev = nullptr)
{
	LevelLayout L;
	for (int l = 0; l < levels; ++l)
	{
		const size_t b = blocksAtLevel(n, l);
		L.blocks[l] = b;
		L.blockBase[l] = L.totalBlocks; L.totalBlocks += b;
		L.validOff[l] = L.validBytes; L.validBytes += (b + 15) & ~(size_t)15;
		L.pageOff[l] = L.pageEntries; if (l >= 1) L.pageEntries += b * 4096;
		L.mixOff[l] = L.mixBytes; if (l >= 1) L.mixBytes += (b + 15) & ~(size_t)15;
		L.coarseBase[l] = L.coarseBlocks; if (l >= coarseLo) L.coarseBlocks += b;
		if (dev) { dev->workBase[l] = dev->idBase[l] = (unsigned)L.blockBase[l]; dev->coarseBase[l] = (unsigned)L.coarseBase[l]; }
	}
	return L;
}

#define VXB_LATTICE_LO 2 // levels >= 2 have their own sample lattice (VxbDev::coarseLattice)

// byte layout of the coarse levels' lattices in one buffer: level l at offsets[l], (h + 1)^2 rows of h + 16 bytes
size_t coarseLatticeLayout(uint32_t n, int levels, size_t offsets[VXB_MAX_LEVELS])
{
	size_t total = 0;
	for (int l = 0; l < VXB_MAX_LEVELS; ++l) offsets[l] = 0;
	for (int l = VXB_LATTICE_LO; l < levels; ++l)
	{
		const size_t h = n >> l;
		offsets[l] = total;
		total += ((h + 16) * (h + 1) * (h + 1) + 127) & ~(size_t)127;
	}
	return total;
}

// (re)builds the coarse levels' lattice area and tensor maps: base = where the lattices live
int buildCoarseLattices(vxb_context* ctx, unsigned char* sharedBase)
{
	const uint32_t n = ctx->n;
	ctx->coarseLo = coarseLoFor(n, ctx->levels);
	ctx->coarseLatticeBytes = coarseLatticeLayout(n, ctx->levels, ctx->coarseLatticeOff);
	if (sharedBase) ctx->coarseLatticeBase = sharedBase;
	else
	{
		VXB_CUDA(ctx, ctx->coarseLatticeBuf.ensure(ctx->coarseLatticeBytes ? ctx->coarseLatticeBytes : 128));
		ctx->coarseLatticeBase = ctx->coarseLatticeBuf.p;
	}
	VXB_CUDA(ctx, ctx->coarseMaps.ensure(VXB_MAX_LEVELS));
	CUtensorMap maps[VXB_MAX_LEVELS];
	memset(maps, 0, sizeof(maps));
	for (int l = VXB_LATTICE_LO; l < ctx->levels; ++l)
	{
		const cuuint64_t h = n >> l;
		const cuuint64_t dims[3] = { h + 1, h + 1, h + 1 };
		const cuuint64_t strides[2] = { h + 16, (h + 16) * (h + 1) };
		const cuuint32_t box[3] = { VXB_TILE_PITCH, 17, 17 };
		const cuuint32_t estr[3] = { 1, 1, 1 };
		const CUresult r = ctx->encodeTiled(&maps[l], CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, ctx->coarseLatticeBase + ctx->coarseLatticeOff[l], dims, strides, box, estr,
			CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
		if (r != CUDA_SUCCESS)
		{
			char buf[128]; snprintf(buf, sizeof(buf), "cuTensorMapEncodeTiled (coarse level %d) failed: CUresult %d", l, (int)r);
			return fail(ctx, VXB_ERR_CUDA, buf);
		}
	}
	VXB_CUDA(ctx, cudaMemcpy(ctx->coarseMaps.p, maps, sizeof(maps), cudaMemcpyHostToDevice));
	return VXB_OK;
}

int buildTensorMap(vxb_context* ctx)
{
	int r = encodeTileMap(ctx, &ctx->tmap, ctx->dDist, ctx->n);
	if (r == VXB_OK) r = encodeTileMap(ctx, &ctx->tmapDist19, ctx->dDist, ctx->n, 19, VXB_DTILE_PITCH);
	if (r != VXB_OK) return r;
	// even-lattice copy for level 1 (written by vxb_scan_kernel each run); needs at least one 16-sample row.  In a sharded
	// run every rank writes the part of its own layers, so the copy must be shared like the volumes (the cube's fourth
	// channel); without that level 1 gathers its tiles from the distance volume.
	const bool cubeLattice = ctx->cube.active && ctx->cube.lattice;
	ctx->haveLattice1 = ctx->n >= 64 && !ctx->latticeOff && (!ctx->cube.active || cubeLattice);
	ctx->latticePtr = nullptr;
	if (ctx->haveLattice1)
	{
		const size_t h = ctx->n / 2;
		if (cubeLattice) ctx->latticePtr = reinterpret_cast<uint8_t*>(ctx->cube.va[3]);
		else { VXB_CUDA(ctx, ctx->lattice1.ensure(h * h * h)); ctx->latticePtr = ctx->lattice1.p; }
		r = encodeTileMap(ctx, &ctx->tmap1, ctx->latticePtr, (uint32_t)h);
	}
	else ctx->tmap1 = ctx->tmap;
	if (r == VXB_OK) r = buildCoarseLattices(ctx, ctx->shard.on ? ctx->shard.lattices(ctx->shard.pagesBuf) : nullptr);
	return r;
}

int finishUpload(vxb_context* ctx)
{
	const int r = buildTensorMap(ctx);
	if (r == VXB_OK) ctx->haveGrid = true;
	return r;
}

// dirty box of an incremental run, per level (GenerateBlockListForLevel :429-465): the run keeps the caches of the last
// full run and continues its block ids
struct Region
{
	int rangeMin[VXB_MAX_LEVELS][3], rangeMax[VXB_MAX_LEVELS][3]; // grid (x, y, z) block coordinates, [min, max)
	unsigned idStart[VXB_MAX_LEVELS];
	size_t count[VXB_MAX_LEVELS];
};

// Launches the kernels of one run and counts them: each launch toward the run's total and toward its kind (vxb_kernel_ms:
// 0 scan, 1 block walk, 2 levels >= 1 and big blocks, 3 level 0, 4 vertices, 5 triangles, 6 transition cells, 7 finish,
// 8 and 9 the two exchanges of a sharded run).  With VXB_FLAG_KERNEL_TIMES, when every launch is on the context's stream,
// each launch of a kind sits between a pair of events.
struct Launcher
{
	static const int kNoKind = -1; // vxb_mark_split_kernel: counted in the total only, and not timed

	vxb_context* ctx;
	bool timed;
	uint32_t total = 0;            // the per-kind counts are ctx->kindLaunches
	std::vector<int> bracketKinds; // kind of each event pair in ctx->kevents

	Launcher(vxb_context* c, bool t) : ctx(c), timed(t) { reset(); }
	void reset() { total = 0; memset(ctx->kindLaunches, 0, sizeof(ctx->kindLaunches)); }
	template <typename... P, typename... A>
	void operator()(int kind, cudaStream_t s, void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, const A&... args)
	{
		++total;
		bracket(kind, [&] { kernel<<<grid, block, smem, s>>>(args...); });
	}
	// a launch of `kind` outside the total: the all-gather of exchange 0, which is not a kernel, is timed and counted as kind 8
	template <typename F> void bracket(int kind, F launch)
	{
		if (kind != kNoKind) ++ctx->kindLaunches[kind];
		if (!timed || kind == kNoKind) { launch(); return; }
		const size_t used = 2 * bracketKinds.size();
		while (ctx->kevents.size() < used + 2) { cudaEvent_t e; cudaEventCreate(&e); ctx->kevents.push_back(e); }
		cudaEventRecord(ctx->kevents[used], ctx->stream);
		launch();
		cudaEventRecord(ctx->kevents[used + 1], ctx->stream);
		bracketKinds.push_back(kind);
	}
	void collectTimes() const
	{
		for (int k = 0; k < 10; ++k) ctx->kindMs[k] = 0.f;
		for (size_t i = 0; i < bracketKinds.size(); ++i)
		{
			float ms = 0.f; cudaEventElapsedTime(&ms, ctx->kevents[2 * i], ctx->kevents[2 * i + 1]);
			ctx->kindMs[bracketKinds[i]] += ms;
		}
	}
};
}

// ---- the cube of a sharded run: virtual memory management through driver entry points (no libcuda link) ----
namespace
{
struct VmmApi
{
	decltype(&cuMemAddressReserve) addressReserve = nullptr;
	decltype(&cuMemAddressFree) addressFree = nullptr;
	decltype(&cuMemCreate) create = nullptr;
	decltype(&cuMemRelease) release = nullptr;
	decltype(&cuMemMap) map = nullptr;
	decltype(&cuMemUnmap) unmap = nullptr;
	decltype(&cuMemSetAccess) setAccess = nullptr;
	decltype(&cuMemExportToShareableHandle) exportHandle = nullptr;
	decltype(&cuMemImportFromShareableHandle) importHandle = nullptr;
	decltype(&cuMemGetAllocationGranularity) granularity = nullptr;
	bool ok = false;
};

const VmmApi& vmmApi()
{
	static VmmApi api;
	static bool tried = false;
	if (tried) return api;
	tried = true;
	struct Entry { const char* name; void** slot; };
	const Entry entries[] = {
		{ "cuMemAddressReserve", (void**)&api.addressReserve }, { "cuMemAddressFree", (void**)&api.addressFree },
		{ "cuMemCreate", (void**)&api.create }, { "cuMemRelease", (void**)&api.release },
		{ "cuMemMap", (void**)&api.map }, { "cuMemUnmap", (void**)&api.unmap }, { "cuMemSetAccess", (void**)&api.setAccess },
		{ "cuMemExportToShareableHandle", (void**)&api.exportHandle }, { "cuMemImportFromShareableHandle", (void**)&api.importHandle },
		{ "cuMemGetAllocationGranularity", (void**)&api.granularity },
	};
	bool all = true;
	for (const Entry& e : entries)
	{
		cudaDriverEntryPointQueryResult q;
		if (cudaGetDriverEntryPoint(e.name, e.slot, cudaEnableDefault, &q) != cudaSuccess || !*e.slot) all = false;
	}
	api.ok = all;
	return api;
}

int failCu(vxb_context* ctx, const char* what, CUresult r)
{
	char buf[160]; snprintf(buf, sizeof(buf), "%s failed: CUresult %d", what, (int)r);
	return fail(ctx, VXB_ERR_CUDA, buf);
}
#define VXB_CU(ctx, call) do { const CUresult r_ = (call); if (r_ != CUDA_SUCCESS) return failCu(ctx, #call, r_); } while (0)

void releaseCube(vxb_context* ctx)
{
	vxb_context::Cube& c = ctx->cube;
	if (!c.active) return;
	const VmmApi& api = vmmApi();
	for (const auto& m : c.mapped) api.unmap(m.first, m.second);
	for (CUmemGenericAllocationHandle h : c.imported) api.release(h);
	for (int k = 0; k < 4; ++k)
	{
		for (CUmemGenericAllocationHandle h : c.local[k]) api.release(h);
		if (c.va[k]) api.addressFree(c.va[k], c.vaBytes[k]);
	}
	c = vxb_context::Cube();
}

void releaseShard(vxb_context* ctx)
{
	vxb_context::Shard& sh = ctx->shard;
	const VmmApi& api = vmmApi();
	for (const auto& m : sh.peerMapped) { api.unmap(m.first, m.second); api.addressFree(m.first, m.second); }
	for (CUmemGenericAllocationHandle h : sh.peerHandles) api.release(h);
	if (sh.pagesVmm)
	{
		if (sh.pagesVa) { api.unmap(sh.pagesVa, sh.bufBytes); api.addressFree(sh.pagesVa, sh.bufBytes); }
		if (sh.pagesHandle) api.release(sh.pagesHandle);
	}
	else if (sh.pagesBuf) cudaFree(sh.pagesBuf);
	sh.sbMine.release(); sh.sbWeight.release();
	void* comm = sh.comm;
	sh = vxb_context::Shard();
	sh.comm = comm; // the communicator outlives a re-configuration (vxb_destroy ends it)
}

CUmemAllocationProp slabProp(int device)
{
	CUmemAllocationProp prop;
	memset(&prop, 0, sizeof(prop));
	prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
	prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
	prop.location.id = device;
	prop.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
	return prop;
}

int mapRange(vxb_context* ctx, CUdeviceptr at, size_t bytes, CUmemGenericAllocationHandle handle, std::vector<std::pair<CUdeviceptr, size_t> >& mapped)
{
	const VmmApi& api = vmmApi();
	VXB_CU(ctx, api.map(at, bytes, 0, handle, 0));
	mapped.push_back(std::make_pair(at, bytes));
	CUmemAccessDesc access;
	memset(&access, 0, sizeof(access));
	access.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
	access.location.id = ctx->device;
	access.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
	VXB_CU(ctx, api.setAccess(at, bytes, &access, 1));
	return VXB_OK;
}

// ---- NCCL through dlopen (the library torch.distributed already loaded, or the system one): the data path of a
// sharded run calls ncclAllGather itself so that a whole step is ONE stream-ordered sequence (and one CUDA graph) ----
struct NcclApi
{
	int (*getUniqueId)(void*) = nullptr;
	int (*commInitRank)(void**, int, vxb_nccl_id, int) = nullptr;
	int (*allGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
	int (*commDestroy)(void*) = nullptr;
	const char* (*getErrorString)(int) = nullptr;
	bool ok = false;
};

const NcclApi& ncclApi()
{
	static NcclApi api;
	static bool tried = false;
	if (tried) return api;
	tried = true;
	void* lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
	if (!lib) lib = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
	if (!lib) return api;
	api.getUniqueId = (int (*)(void*))dlsym(lib, "ncclGetUniqueId");
	api.commInitRank = (int (*)(void**, int, vxb_nccl_id, int))dlsym(lib, "ncclCommInitRank");
	api.allGather = (int (*)(const void*, void*, size_t, int, void*, cudaStream_t))dlsym(lib, "ncclAllGather");
	api.commDestroy = (int (*)(void*))dlsym(lib, "ncclCommDestroy");
	api.getErrorString = (const char* (*)(int))dlsym(lib, "ncclGetErrorString");
	api.ok = api.getUniqueId && api.commInitRank && api.allGather && api.commDestroy;
	return api;
}

int failNccl(vxb_context* ctx, const char* what, int r)
{
	char buf[200];
	const NcclApi& api = ncclApi();
	snprintf(buf, sizeof(buf), "%s failed: ncclResult %d (%s)", what, r, api.getErrorString ? api.getErrorString(r) : "?");
	return fail(ctx, VXB_ERR_CUDA, buf);
}
}

extern "C"
{

// The cube of a sharded run: pieces of `group_planes` planes, piece p owned by rank p % world.
int vxb_cube_create(vxb_context* ctx, uint32_t n, uint32_t rank, uint32_t world, uint32_t groupPlanes)
{
	if (!ctx) return VXB_ERR_ARGUMENT;
	if (!validSize(n)) return fail(ctx, VXB_ERR_ARGUMENT, "vxb_cube_create: n must be a power of two in [16, 4096]");
	if (world == 0 || world > 8 || rank >= world) return fail(ctx, VXB_ERR_ARGUMENT, "vxb_cube_create: world in [1, 8], rank < world");
	if (groupPlanes == 0) groupPlanes = n / world;
	if (groupPlanes % 32 != 0 || n % groupPlanes != 0 || (n / groupPlanes) % world != 0)
		return fail(ctx, VXB_ERR_ARGUMENT, "vxb_cube_create: group_planes must be a multiple of 32 planes that divides n into a multiple of `world` pieces");
	const VmmApi& api = vmmApi();
	if (!api.ok) return fail(ctx, VXB_ERR_CUDA, "vxb_cube_create: the driver does not export the virtual memory management entry points");
	cudaSetDevice(ctx->device);
	cudaFree(nullptr); // make sure the primary context exists and is current for the driver calls
	releaseCube(ctx);
	vxb_context::Cube& c = ctx->cube;
	c.rank = rank; c.world = world; c.n = n;
	c.groupPlanes = groupPlanes; c.pieces = n / groupPlanes;
	const CUmemAllocationProp prop = slabProp(ctx->device);
	size_t gran = 0;
	VXB_CU(ctx, api.granularity(&gran, &prop, CU_MEM_ALLOC_GRANULARITY_MINIMUM));
	if (!gran || c.pieceBytes(0) % gran != 0)
	{
		char buf[200]; snprintf(buf, sizeof(buf), "vxb_cube_create: a piece (%zu bytes) is not a multiple of the allocation granularity (%zu bytes)", c.pieceBytes(0), gran);
		c = vxb_context::Cube();
		return fail(ctx, VXB_ERR_ARGUMENT, buf);
	}
	c.lattice = n >= 64 && c.pieceBytes(3) % gran == 0; // else level-1 tiles are gathered from the distance volume
	c.active = true;
	const int channels = c.lattice ? 4 : 3;
	for (int k = 0; k < channels; ++k)
	{
		c.vaBytes[k] = c.pieceBytes(k) * c.pieces;
		VXB_CU(ctx, api.addressReserve(&c.va[k], c.vaBytes[k], 0, 0, 0));
		for (uint32_t p = rank; p < c.pieces; p += world)
		{
			CUmemGenericAllocationHandle h = 0;
			VXB_CU(ctx, api.create(&h, c.pieceBytes(k), &prop, 0));
			c.local[k].push_back(h);
			const int r = mapRange(ctx, c.va[k] + (CUdeviceptr)(c.pieceBytes(k) * p), c.pieceBytes(k), h, c.mapped);
			if (r != VXB_OK) return r;
		}
	}
	ctx->dDist = reinterpret_cast<const int8_t*>(c.va[0]);
	ctx->dMat = reinterpret_cast<const uint8_t*>(c.va[1]);
	ctx->dBlend = reinterpret_cast<const uint8_t*>(c.va[2]);
	ctx->n = n; ctx->levels = levelsFor(n);
	ctx->ownsGrid = false; ctx->haveGrid = true; ctx->haveResult = false; ctx->haveFullRun = false;
	return buildTensorMap(ctx);
}

int vxb_cube_info(vxb_context* ctx, uint32_t* pieces, uint32_t* channels, uint64_t* pieceBytes)
{
	if (!ctx) return VXB_ERR_ARGUMENT;
	const vxb_context::Cube& c = ctx->cube;
	if (!c.active) return fail(ctx, VXB_ERR_STATE, "vxb_cube_info: no cube");
	if (pieces) *pieces = c.pieces;
	if (channels) *channels = c.lattice ? 4u : 3u;
	if (pieceBytes) for (int k = 0; k < 4; ++k) pieceBytes[k] = (k < 3 || c.lattice) ? c.pieceBytes(k) : 0;
	return VXB_OK;
}

int vxb_cube_export(vxb_context* ctx, uint32_t channel, uint32_t piece, int* fd)
{
	if (!ctx || !fd) return VXB_ERR_ARGUMENT;
	const vxb_context::Cube& c = ctx->cube;
	if (!c.active || channel >= (c.lattice ? 4u : 3u) || piece >= c.pieces || piece % c.world != c.rank)
		return fail(ctx, VXB_ERR_ARGUMENT, "vxb_cube_export: no cube, bad channel, or a piece this rank does not own");
	cudaSetDevice(ctx->device);
	int out = -1;
	VXB_CU(ctx, vmmApi().exportHandle(&out, c.local[channel][piece / c.world], CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0));
	*fd = out;
	return VXB_OK;
}

int vxb_cube_import(vxb_context* ctx, uint32_t channel, uint32_t piece, int fd)
{
	if (!ctx) return VXB_ERR_ARGUMENT;
	vxb_context::Cube& c = ctx->cube;
	if (!c.active || channel >= (c.lattice ? 4u : 3u) || piece >= c.pieces || piece % c.world == c.rank || fd < 0)
		return fail(ctx, VXB_ERR_ARGUMENT, "vxb_cube_import: no cube, or bad channel / piece / descriptor");
	cudaSetDevice(ctx->device);
	CUmemGenericAllocationHandle h = 0;
	VXB_CU(ctx, vmmApi().importHandle(&h, (void*)(uintptr_t)fd, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR));
	c.imported.push_back(h);
	return mapRange(ctx, c.va[channel] + (CUdeviceptr)(c.pieceBytes(channel) * piece), c.pieceBytes(channel), h, c.mapped);
}

int vxb_cube_piece(vxb_context* ctx, uint32_t piece, int8_t** dist, uint8_t** mat, uint8_t** blend, uint64_t* bytes)
{
	if (!ctx) return VXB_ERR_ARGUMENT;
	const vxb_context::Cube& c = ctx->cube;
	if (!c.active || piece >= c.pieces) return fail(ctx, VXB_ERR_STATE, "vxb_cube_piece: no cube, or bad piece");
	const size_t off = c.pieceBytes(0) * piece;
	if (dist) *dist = reinterpret_cast<int8_t*>(c.va[0] + off);
	if (mat) *mat = reinterpret_cast<uint8_t*>(c.va[1] + off);
	if (blend) *blend = reinterpret_cast<uint8_t*>(c.va[2] + off);
	if (bytes) *bytes = c.pieceBytes(0);
	return VXB_OK;
}

int vxb_create(int device, vxb_context** out)
{
	if (!out) return fail(nullptr, VXB_ERR_ARGUMENT, "vxb_create: out is null");
	*out = nullptr;
	int count = 0;
	cudaError_t e = cudaGetDeviceCount(&count);
	if (e != cudaSuccess || count == 0) return fail(nullptr, VXB_ERR_CUDA, "vxb_create: no CUDA device (this library has no CPU fallback)", e);
	if (device < 0 || device >= count) return fail(nullptr, VXB_ERR_ARGUMENT, "vxb_create: bad device index");
	e = cudaSetDevice(device);
	if (e != cudaSuccess) return fail(nullptr, VXB_ERR_CUDA, "cudaSetDevice", e);
	cudaDeviceProp prop;
	e = cudaGetDeviceProperties(&prop, device);
	if (e != cudaSuccess) return fail(nullptr, VXB_ERR_CUDA, "cudaGetDeviceProperties", e);
	if (prop.major != 9 || prop.minor != 0) return fail(nullptr, VXB_ERR_CUDA, "vxb_create: the kernels are built for sm_90a (Hopper) only");

	vxb_context* ctx = new vxb_context;
	ctx->device = device; ctx->smCount = prop.multiProcessorCount;
	memset(&ctx->info, 0, sizeof(ctx->info));
	memset(&ctx->drawLists, 0, sizeof(ctx->drawLists));
	memset(&ctx->lastDev, 0, sizeof(ctx->lastDev));
	if ((e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking)) != cudaSuccess ||
		(e = cudaStreamCreateWithFlags(&ctx->stream2, cudaStreamNonBlocking)) != cudaSuccess ||
		(e = cudaEventCreate(&ctx->evBegin)) != cudaSuccess || (e = cudaEventCreate(&ctx->evEnd)) != cudaSuccess)
	{ fail(nullptr, VXB_ERR_CUDA, "stream/event creation", e); vxb_destroy(ctx); return VXB_ERR_CUDA; }
	for (cudaEvent_t* ev : { &ctx->evDir, &ctx->evFork, &ctx->evJoin, &ctx->evLatticeFork, &ctx->evLatticeJoin })
		if ((e = cudaEventCreateWithFlags(ev, cudaEventDisableTiming)) != cudaSuccess) { fail(nullptr, VXB_ERR_CUDA, "stream/event creation", e); vxb_destroy(ctx); return VXB_ERR_CUDA; }

	void* fn = nullptr;
	cudaDriverEntryPointQueryResult qres;
	e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
	if (e != cudaSuccess || !fn) { fail(nullptr, VXB_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available", e); vxb_destroy(ctx); return VXB_ERR_CUDA; }
	ctx->encodeTiled = reinterpret_cast<EncodeTiledFn>(fn);

	ctx->graphDisabled = getenv("VXB200_NO_GRAPH") != nullptr; // plain launches (debugging, A/B timing)
	struct KernelSetup { const void* fn; size_t smem; int* grid; const char* name; int threads; };
	const KernelSetup setups[5] = {
		{ (const void*)vxb_block_kernel<0>, sizeof(VxbBlockSmem<0>), &ctx->gridBlock[0], "vxb_block_kernel<0>", VXB_THREADS },
		{ (const void*)vxb_block_kernel<1>, sizeof(VxbBlockSmem<1>), &ctx->gridBlock[1], "vxb_block_kernel<1>", VXB_THREADS },
		{ (const void*)vxb_block_kernel<2>, sizeof(VxbBlockSmem<2>), &ctx->gridBlock[2], "vxb_block_kernel<2>", VXB_THREADS },
		{ (const void*)vxb_big_block_kernel, sizeof(VxbBigBlockSmem), &ctx->gridBigBlock, "vxb_big_block_kernel", VXB_THREADS },
		{ (const void*)vxb_transition_kernel, 0, &ctx->gridTransition, "vxb_transition_kernel", VXB_TR_THREADS },
	};
	for (const KernelSetup& k : setups)
	{
		int occ = 0;
		e = cudaFuncSetAttribute(k.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k.smem);
		if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k.fn, k.threads, k.smem);
		if (e != cudaSuccess || occ < 1) { fail(nullptr, VXB_ERR_CUDA, k.name, e); vxb_destroy(ctx); return VXB_ERR_CUDA; }
		*k.grid = occ * ctx->smCount;
	}

	if (ctx->counters.ensure(1) != cudaSuccess || ctx->lut.ensure(1) != cudaSuccess) { fail(nullptr, VXB_ERR_CUDA, "cudaMalloc"); vxb_destroy(ctx); return VXB_ERR_CUDA; }
	*out = ctx;
	const int r = vxb_set_materials(ctx, nullptr, nullptr);
	if (r != VXB_OK) { g_createError = ctx->error; vxb_destroy(ctx); *out = nullptr; return r; }
	return VXB_OK;
}

void vxb_destroy(vxb_context* ctx)
{
	if (!ctx) return;
	cudaSetDevice(ctx->device);
	for (vxb_mesh* m : std::vector<vxb_mesh*>(ctx->meshes)) vxb_mesh_destroy(m);
	if (ctx->stream) cudaStreamSynchronize(ctx->stream);
	if (ctx->stream2) cudaStreamSynchronize(ctx->stream2);
	if (ctx->graphExec) cudaGraphExecDestroy(ctx->graphExec);
	releaseShard(ctx);
	if (ctx->shard.comm && ncclApi().ok) { ncclApi().commDestroy(ctx->shard.comm); ctx->shard.comm = nullptr; }
	releaseCube(ctx);
	for (cudaEvent_t e : ctx->progEv) if (e) cudaEventDestroy(e);
	for (cudaEvent_t e : ctx->kevents) cudaEventDestroy(e);
	for (cudaEvent_t e : { ctx->evBegin, ctx->evEnd, ctx->evDir, ctx->evFork, ctx->evJoin, ctx->evLatticeFork, ctx->evLatticeJoin })
		if (e) cudaEventDestroy(e);
	for (cudaEvent_t e : ctx->evChunks) if (e) cudaEventDestroy(e);
	if (ctx->stream2) cudaStreamDestroy(ctx->stream2);
	if (ctx->stream) cudaStreamDestroy(ctx->stream);
	delete ctx; // the buffers free themselves
}

const char* vxb_last_error(const vxb_context* ctx) { return ctx ? ctx->error.c_str() : g_createError.c_str(); }

void* vxb_stream(vxb_context* ctx) { return ctx ? (void*)ctx->stream : nullptr; }

void* vxb_exchange_stream(vxb_context* ctx) { return ctx ? (void*)ctx->stream2 : nullptr; }

int vxb_grid_upload_dense(vxb_context* ctx, uint32_t n, const int8_t* dist, const uint8_t* mat, const uint8_t* blend)
{
	if (!ctx) return VXB_ERR_ARGUMENT;
	if (!validSize(n) || !dist) return fail(ctx, VXB_ERR_ARGUMENT, "vxb_grid_upload_dense: n must be a power of two in [16, 4096] and dist non-null");
	cudaSetDevice(ctx->device);
	int r = ensureGridStorage(ctx, n);
	if (r != VXB_OK) return r;
	const size_t vol = (size_t)n * n * n;
	VXB_CUDA(ctx, cudaMemcpyAsync(ctx->volDist.p, dist, vol, cudaMemcpyHostToDevice, ctx->stream));
	if (mat) VXB_CUDA(ctx, cudaMemcpyAsync(ctx->volMat.p, mat, vol, cudaMemcpyHostToDevice, ctx->stream));
	else VXB_CUDA(ctx, cudaMemsetAsync(ctx->volMat.p, 0, vol, ctx->stream));
	if (blend) VXB_CUDA(ctx, cudaMemcpyAsync(ctx->volBlend.p, blend, vol, cudaMemcpyHostToDevice, ctx->stream));
	else VXB_CUDA(ctx, cudaMemsetAsync(ctx->volBlend.p, 0, vol, ctx->stream));
	VXB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return finishUpload(ctx);
}

int vxb_grid_upload_blocks(vxb_context* ctx, uint32_t n, const int8_t* distBlocks, const uint8_t* matBlocks, const uint8_t* blendBlocks)
{
	if (!ctx) return VXB_ERR_ARGUMENT;
	if (!validSize(n) || !distBlocks) return fail(ctx, VXB_ERR_ARGUMENT, "vxb_grid_upload_blocks: bad size or null dist");
	cudaSetDevice(ctx->device);
	int r = ensureGridStorage(ctx, n);
	if (r != VXB_OK) return r;
	const size_t vol = (size_t)n * n * n;
	VXB_CUDA(ctx, ctx->staging.ensure(vol));
	const unsigned blocks = (unsigned)(vol / 4096);
	const void* src[3] = { distBlocks, matBlocks, blendBlocks };
	uint8_t* dst[3] = { ctx->volDist.p, ctx->volMat.p, ctx->volBlend.p };
	for (int c = 0; c < 3; ++c)
	{
		if (!src[c]) { VXB_CUDA(ctx, cudaMemsetAsync(dst[c], 0, vol, ctx->stream)); continue; }
		VXB_CUDA(ctx, cudaMemcpyAsync(ctx->staging.p, src[c], vol, cudaMemcpyHostToDevice, ctx->stream));
		vxb_unpack_blocks_kernel<<<blocks, VXB_THREADS, 0, ctx->stream>>>(reinterpret_cast<const uint4*>(ctx->staging.p), dst[c], (int)n);
		VXB_CUDA(ctx, cudaGetLastError());
	}
	VXB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return finishUpload(ctx);
}

int vxb_grid_upload_packed(vxb_context* ctx, const void* blob, size_t size)
{
	return vxb_grid_upload_packed_streamed(ctx, blob, size, nullptr, nullptr);
}

int vxb_grid_upload_packed_streamed(vxb_context* ctx, const void* blob, size_t size, vxb_pack_producer produce, void* user)
{
	if (!ctx) return VXB_ERR_ARGUMENT;
	if (!blob || size < 16) return fail(ctx, VXB_ERR_ARGUMENT, "vxb_grid_upload_packed: null or truncated blob");
	const unsigned char* bytes = static_cast<const unsigned char*>(blob);
	uint32_t header[4];
	memcpy(header, bytes, 16);
	if (header[0] != 1) return fail(ctx, VXB_ERR_ARGUMENT, "vxb_grid_upload_packed: unsupported file version (VoxelGrid.cpp:227-231)");
	const uint32_t n = header[1];
	if (!validSize(n) || header[2] != n || header[3] != n) return fail(ctx, VXB_ERR_ARGUMENT, "vxb_grid_upload_packed: the grid must be a cube with a power-of-two edge");
	const size_t nb = n / 16, blocks = nb * nb * nb;
	const size_t tableBytes = blocks * 12;
	if (size < 16 + tableBytes) return fail(ctx, VXB_ERR_ARGUMENT, "vxb_grid_upload_packed: truncated size table");
	cudaSetDevice(ctx->device);
	// a context with a cube (sharded runs) receives only the pieces this rank backs: the same blob on every rank, each
	// copies and decodes the byte ranges of its own block layers
	const bool pieces = ctx->cube.active;
	if (pieces && ctx->cube.n != n) return fail(ctx, VXB_ERR_ARGUMENT, "vxb_grid_upload_packed: the blob's grid size differs from the cube's");
	int r = pieces ? VXB_OK : ensureGridStorage(ctx, n);
	if (r != VXB_OK) return r;
	VXB_CUDA(ctx, ctx->staging.ensure(size + 16));
	VXB_CUDA(ctx, ctx->packOffsets.ensure(blocks));
	const bool trace = getenv("VXB200_TRACE") != nullptr;
	auto now = [] { return std::chrono::steady_clock::now(); };
	auto msSince = [&](std::chrono::steady_clock::time_point t) { return std::chrono::duration<double, std::milli>(now() - t).count(); };
	const auto t0 = now();
	// Pipeline: header + size table first; while that moves, the per-block byte offsets (prefix sum of the size table) are
	// computed on the host; then the block data in z-chunks on the copy stream, each chunk decoded on the second stream
	// as soon as it has landed, so that only the last chunk's decode is exposed.
	const size_t head = 16 + tableBytes;
	if (!ctx->hostOffsets.ensure(blocks * sizeof(unsigned long long))) return fail(ctx, VXB_ERR_CUDA, "vxb_grid_upload_packed: pinned scratch allocation failed");
	unsigned long long* const hostOffsets = static_cast<unsigned long long*>(ctx->hostOffsets.p);
	VXB_CUDA(ctx, cudaMemcpyAsync(ctx->staging.p, blob, head, cudaMemcpyHostToDevice, ctx->stream));
	bool corrupt = false, truncated = false;
	unsigned long long off = head;
	{
		// per-block byte offsets = prefix sum of the size table (sequential, 12 bytes per block).  The blocks' flag words lie
		// scattered through the blob (one cache miss each on the host), so they are checked where they are read anyway:
		// on the device, by vxb_unpack_rle_kernel (packError)
		const unsigned char* table = bytes + 16;
		for (size_t b = 0; b < blocks; ++b)
		{
			uint32_t sz[3];
			memcpy(sz, table + b * 12, 12);
			if (sz[0] > 4096 || sz[1] > 4096 || sz[2] > 4096) { corrupt = true; break; }
			hostOffsets[b] = off;
			off += 4ull + sz[0] + sz[1] + sz[2];
		}
		if (!corrupt && off > size) truncated = true;
	}
	const double msTable = msSince(t0);
	if (corrupt || truncated || off > size)
	{
		cudaStreamSynchronize(ctx->stream);
		ctx->haveGrid = false;
		return fail(ctx, VXB_ERR_ARGUMENT, corrupt ? "vxb_grid_upload_packed: corrupt size table or block flags" : "vxb_grid_upload_packed: truncated block data");
	}
	VXB_CUDA(ctx, cudaMemcpyAsync(ctx->packOffsets.p, hostOffsets, blocks * sizeof(unsigned long long), cudaMemcpyHostToDevice, ctx->stream));
	VXB_CUDA(ctx, ctx->packError.ensure(1));
	VXB_CUDA(ctx, cudaMemsetAsync(ctx->packError.p, 0, sizeof(unsigned int), ctx->stream));
	std::vector<std::pair<size_t, size_t> > ranges; // block layers [first, second)
	if (pieces)
	{
		const size_t g = ctx->cube.groupPlanes / 16;
		for (size_t p = ctx->cube.rank; p < ctx->cube.pieces; p += ctx->cube.world) ranges.push_back(std::make_pair(p * g, (p + 1) * g));
	}
	else
	{
		const int chunks = nb >= 32 && produce ? 8 : (nb >= 16 ? 4 : 1); // a producer overlaps with the copies: finer slabs
		for (int c = 0; c < chunks; ++c) ranges.push_back(std::make_pair(nb * c / chunks, nb * (c + 1) / chunks));
	}
	while (ctx->evChunks.size() < ranges.size())
	{
		cudaEvent_t ev = nullptr;
		VXB_CUDA(ctx, cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
		ctx->evChunks.push_back(ev);
	}
	unsigned char* const outDist = pieces ? reinterpret_cast<unsigned char*>(ctx->cube.va[0]) : ctx->volDist.p;
	unsigned char* const outMat = pieces ? reinterpret_cast<unsigned char*>(ctx->cube.va[1]) : ctx->volMat.p;
	unsigned char* const outBlend = pieces ? reinterpret_cast<unsigned char*>(ctx->cube.va[2]) : ctx->volBlend.p;
	const size_t groupsPerLayer = ((nb + 7) / 8) * nb;
	for (size_t c = 0; c < ranges.size(); ++c)
	{
		const size_t layer0 = ranges[c].first, layer1 = ranges[c].second;
		const unsigned long long byte0 = hostOffsets[layer0 * nb * nb], byte1 = (layer1 == nb) ? off : hostOffsets[layer1 * nb * nb];
		if (produce) produce(user, (uint32_t)layer0, (uint32_t)layer1); // the caller fills this slab while the previous one moves
		VXB_CUDA(ctx, cudaMemcpyAsync(ctx->staging.p + byte0, bytes + byte0, (size_t)(byte1 - byte0), cudaMemcpyHostToDevice, ctx->stream));
		VXB_CUDA(ctx, cudaEventRecord(ctx->evChunks[c], ctx->stream));
		VXB_CUDA(ctx, cudaStreamWaitEvent(ctx->stream2, ctx->evChunks[c], 0));
		vxb_unpack_rle_kernel<<<(unsigned)(groupsPerLayer * (layer1 - layer0)), VXB_THREADS, 0, ctx->stream2>>>(ctx->staging.p, ctx->packOffsets.p,
			reinterpret_cast<const unsigned int*>(ctx->staging.p + 16), outDist, outMat, outBlend, (int)n, (int)layer0, ctx->packError.p);
	}
	VXB_CUDA(ctx, cudaGetLastError());
	VXB_CUDA(ctx, cudaEventRecord(ctx->evJoin, ctx->stream2));
	VXB_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ctx->evJoin, 0));
	unsigned int packError = 0;
	VXB_CUDA(ctx, cudaMemcpyAsync(&packError, ctx->packError.p, sizeof(packError), cudaMemcpyDeviceToHost, ctx->stream));
	VXB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	if (packError)
	{
		ctx->haveGrid = false;
		return fail(ctx, VXB_ERR_ARGUMENT, "vxb_grid_upload_packed: malformed block data (a raw channel must hold 4096 bytes, a run-length coded one whole (length, value) pairs whose lengths add up to 4096)");
	}
	const double msKernel = msSince(t0);
	if (pieces) { ctx->haveResult = false; ctx->haveFullRun = false; r = VXB_OK; }
	else r = finishUpload(ctx);
	if (trace) fprintf(stderr, "[vxb200] upload_packed: offsets ready at %.3f ms, copy + decode done at %.3f ms, maps at %.3f ms\n", msTable, msKernel, msSince(t0));
	return r;
}

size_t vxb_pack_dense_bound(uint32_t n)
{
	const size_t nb = n / 16, blocks = nb * nb * nb;
	return 16 + blocks * 12 + blocks * (4 + 3 * 4096);
}

namespace
{
// VoxelGrid::CompressBlock (VoxelGrid.cpp:610-672): returns the stored size; raw 4096 bytes when RLE would be larger
unsigned compressChannel(const unsigned char* data, unsigned char* out, bool signedValues, bool* uncompressed, bool* isEmpty)
{
	unsigned counter = 0, size = 1;
	const int initial = signedValues ? (int)(signed char)data[0] : (int)data[0];
	unsigned char last = data[0];
	bool empty = true, effective = true;
	unsigned ctrPos = 0;
	for (unsigned i = 0; i < 4096; ++i)
	{
		const unsigned char cur = data[i];
		if (last == cur && counter < 0xFF) { ++counter; continue; }
		out[ctrPos] = (unsigned char)counter;
		out[size++] = last;
		ctrPos = size++;
		counter = 1;
		last = cur;
		const int lv = signedValues ? (int)(signed char)last : (int)last;
		if (initial * lv <= 0) empty = false;
		if (size > 4096) { effective = false; break; }
	}
	if (effective)
	{
		out[ctrPos] = (unsigned char)counter;
		out[size++] = last;
		*uncompressed = false;
		if (isEmpty) *isEmpty = empty;
		return size;
	}
	memcpy(out, data, 4096);
	*uncompressed = true;
	if (isEmpty) *isEmpty = false;
	return 4096;
}
}

int vxb_pack_dense(uint32_t n, const int8_t* dist, const uint8_t* mat, const uint8_t* blend, void* out, size_t capacity, size_t* written)
{
	if (!validSize(n) || !dist || !mat || !blend || !out) return VXB_ERR_ARGUMENT;
	const size_t nb = n / 16, blocks = nb * nb * nb;
	if (capacity < 16 + blocks * 12) return VXB_ERR_CAPACITY;
	unsigned char* bytes = static_cast<unsigned char*>(out);
	const uint32_t header[4] = { 1u, n, n, n };
	memcpy(bytes, header, 16);
	// pass 1 (parallel): compress every block into a private slot of a scratch area; pass 2: concatenate
	std::vector<unsigned char> scratch(blocks * (4 + 3 * 4096));
	std::vector<uint32_t> sizes(blocks * 3);
	const uint8_t* chans[3] = { reinterpret_cast<const uint8_t*>(dist), mat, blend };
	#pragma omp parallel for schedule(static)
	for (long b = 0; b < (long)blocks; ++b)
	{
		const size_t bx = b % nb, by = (b / nb) % nb, bz = b / (nb * nb);
		unsigned char raw[4096];
		unsigned char* slot = scratch.data() + (size_t)b * (4 + 3 * 4096);
		uint32_t flags = 0;
		unsigned pos = 4;
		for (int ch = 0; ch < 3; ++ch)
		{
			for (int z = 0; z < 16; ++z) for (int y = 0; y < 16; ++y)
				memcpy(raw + z * 256 + y * 16, chans[ch] + ((bz * 16 + z) * n + by * 16 + y) * n + bx * 16, 16);
			bool uncompressed = false, isEmpty = false;
			const unsigned sz = compressChannel(raw, slot + pos, ch == 0, &uncompressed, ch == 0 ? &isEmpty : nullptr);
			if (uncompressed) flags |= 2u << ch;         // BF_DistanceUncompressed / Material / Blend (VoxelGrid.h:70-79)
			if (ch == 0 && isEmpty) flags |= 1u;         // BF_Empty
			sizes[b * 3 + ch] = sz;
			pos += sz;
		}
		memcpy(slot, &flags, 4);
	}
	memcpy(bytes + 16, sizes.data(), blocks * 12);
	size_t off = 16 + blocks * 12;
	for (size_t b = 0; b < blocks; ++b)
	{
		const size_t len = 4ull + sizes[b * 3] + sizes[b * 3 + 1] + sizes[b * 3 + 2];
		if (off + len > capacity) return VXB_ERR_CAPACITY;
		memcpy(bytes + off, scratch.data() + b * (4 + 3 * 4096), len);
		off += len;
	}
	if (written) *written = off;
	return VXB_OK;
}

int vxb_grid_fill(vxb_context* ctx, uint32_t n, const vxb_surface* surface, const float start[3], float step)
{
	if (!ctx) return VXB_ERR_ARGUMENT;
	if (!validSize(n) || !surface || surface->kind > VXB_SURFACE_TERRAIN) return fail(ctx, VXB_ERR_ARGUMENT, "vxb_grid_fill: bad size or surface");
	cudaSetDevice(ctx->device);
	const bool pieces = ctx->cube.active;
	if (pieces && ctx->cube.n != n) return fail(ctx, VXB_ERR_ARGUMENT, "vxb_grid_fill: n differs from the cube's");
	int r = pieces ? VXB_OK : ensureGridStorage(ctx, n);
	if (r != VXB_OK) return r;
	VxbFillArgs* args = new VxbFillArgs;
	memset(args, 0, sizeof(*args));
	args->surface = *surface;
	vxs_permutation(surface->seed, args->perm);
	for (int k = 0; k < 3; ++k) args->start[k] = start ? start[k] : 0.f;
	args->step = step;
	args->n = (int)n;
	signed char* dDist = const_cast<signed char*>(reinterpret_cast<const signed char*>(pieces ? ctx->dDist : reinterpret_cast<const int8_t*>(ctx->volDist.p)));
	unsigned char* dMat = pieces ? const_cast<unsigned char*>(ctx->dMat) : ctx->volMat.p;
	unsigned char* dBlend = pieces ? const_cast<unsigned char*>(ctx->dBlend) : ctx->volBlend.p;
	if (surface->kind == VXB_SURFACE_TERRAIN)
	{
		if (ctx->fillColumns.ensure((size_t)n * n * 4) != cudaSuccess) { delete args; return fail(ctx, VXB_ERR_CUDA, "vxb_grid_fill: column buffer allocation failed"); }
		args->columns = ctx->fillColumns.p;
		vxb_fill_columns_kernel<<<(unsigned)(((size_t)n * n + 255) / 256), 256, 0, ctx->stream>>>(*args);
	}
	std::vector<std::pair<int, int> > ranges;
	if (pieces) for (uint32_t p = ctx->cube.rank; p < ctx->cube.pieces; p += ctx->cube.world) ranges.push_back(std::make_pair((int)(p * ctx->cube.groupPlanes), (int)((p + 1) * ctx->cube.groupPlanes)));
	else ranges.push_back(std::make_pair(0, (int)n));
	for (const auto& rg : ranges)
	{
		args->z0 = rg.first; args->z1 = rg.second;
		vxb_fill_kernel<<<(unsigned)ctx->smCount * 16, 256, 0, ctx->stream>>>(*args, dDist, dMat, dBlend);
	}
	const cudaError_t e = cudaGetLastError();
	const cudaError_t e2 = cudaStreamSynchronize(ctx->stream);
	delete args;
	if (e != cudaSuccess || e2 != cudaSuccess) return fail(ctx, VXB_ERR_CUDA, "vxb_grid_fill", e != cudaSuccess ? e : e2);
	if (pieces) { ctx->haveResult = false; ctx->haveFullRun = false; return VXB_OK; }
	return finishUpload(ctx);
}

namespace
{
// touched block range + the box the reference returns (VoxelGrid.cpp:479-487 / :577-584: "DX-style" Y-up)
int prepareEdit(vxb_context* ctx, const char* who, const float position[3], const float extents[3], VxbEditArgs& a, float outMin[3], float outMax[3])
{
	if (!ctx->haveGrid || !ctx->ownsGrid) return fail(ctx, VXB_ERR_STATE, who);
	const float n = (float)ctx->n;
	memset(&a, 0, sizeof(a));
	a.n = (int)ctx->n;
	const int nb = (int)(ctx->n / 16);
	bool any = true;
	for (int k = 0; k < 3; ++k)
	{
		a.position[k] = position[k]; a.extents[k] = extents[k];
		const float lo = position[k] - extents[k] / 2.f, hi = lo + extents[k];
		// blocks whose section is non-empty: the ones the half-open range [lo, hi) clipped to the grid reaches
		const float clo = lo < 0.f ? 0.f : lo, chi = hi > n ? n : hi;
		if (!(chi > clo)) any = false;
		int b0 = (int)floorf(clo / 16.f), b1 = (int)ceilf(chi / 16.f);
		if (b0 < 0) b0 = 0;
		if (b1 > nb) b1 = nb;
		a.b0[k] = b0; a.bn[k] = b1 > b0 ? b1 - b0 : 0;
		if (a.bn[k] == 0) any = false;
	}
	const float icp[3] = { position[0] - extents[0] / 2.f, position[1] - extents[1] / 2.f, position[2] - extents[2] / 2.f };
	const float gs[3] = { std::max(0.f, icp[0]), std::max(0.f, icp[2]), std::max(0.f, icp[1]) };
	if (outMin) { outMin[0] = gs[0]; outMin[1] = gs[1]; outMin[2] = gs[2]; }
	if (outMax) { outMax[0] = std::min(n, gs[0] + extents[0]); outMax[1] = std::min(n, gs[1] + extents[2]); outMax[2] = std::min(n, gs[2] + extents[1]); }
	return any ? VXB_OK : 1; // 1 = nothing to touch
}
}

int vxb_grid_inject_surface(vxb_context* ctx, const float position[3], const float extents[3], const vxb_surface* surface, int type, float outMin[3], float outMax[3])
{
	if (!ctx || !position || !extents || !surface) return VXB_ERR_ARGUMENT;
	if (type < 0 || type > 2 || surface->kind > VXB_SURFACE_TERRAIN) return fail(ctx, VXB_ERR_ARGUMENT, "vxb_grid_inject_surface: bad injection type or surface");
	cudaSetDevice(ctx->device);
	VxbEditArgs a;
	const int r = prepareEdit(ctx, "vxb_grid_inject_surface: needs a context-owned grid (upload or fill)", position, extents, a, outMin, outMax);
	if (r < 0) return r;
	if (r == 1) return VXB_OK;
	a.surface = *surface; a.type = type;
	if (surface->kind == VXB_SURFACE_TERRAIN) vxs_permutation(surface->seed, a.perm);
	vxb_inject_surface_kernel<<<(unsigned)(a.bn[0] * a.bn[1] * a.bn[2]), 256, 0, ctx->stream>>>(a, reinterpret_cast<signed char*>(ctx->volDist.p));
	VXB_CUDA(ctx, cudaGetLastError());
	ctx->haveResult = false;
	return VXB_OK;
}

int vxb_grid_inject_material(vxb_context* ctx, const float position[3], const float extents[3], uint32_t material, int addSubtractBlend, float outMin[3], float outMax[3])
{
	if (!ctx || !position || !extents) return VXB_ERR_ARGUMENT;
	if (material > 255) return fail(ctx, VXB_ERR_ARGUMENT, "vxb_grid_inject_material: material id > 255");
	cudaSetDevice(ctx->device);
	VxbEditArgs a;
	const int r = prepareEdit(ctx, "vxb_grid_inject_material: needs a context-owned grid (upload or fill)", position, extents, a, outMin, outMax);
	if (r < 0) return r;
	if (r == 1) return VXB_OK;
	a.material = (int)material; a.addBlend = addSubtractBlend ? 1 : 0;
	vxb_inject_material_kernel<<<(unsigned)(a.bn[0] * a.bn[1] * a.bn[2]), 256, 0, ctx->stream>>>(a, ctx->volMat.p, ctx->volBlend.p);
	VXB_CUDA(ctx, cudaGetLastError());
	ctx->haveResult = false;
	return VXB_OK;
}

namespace
{
// validates the program (vxp_validate) and copies it into its kernel-parameter form, with the permutation tables of its
// TERRAIN ops; nothing on the device is touched before this has passed
int loadProgram(vxb_context* ctx, const char* who, const vxb_op* ops, uint32_t count, VxbProgram& p)
{
	const char* why = "";
	const int bad = vxp_validate(ops, count, &why);
	if (bad >= 0)
	{
		char buf[256];
		snprintf(buf, sizeof(buf), "%s: op %d: %s", who, bad, why);
		return fail(ctx, VXB_ERR_ARGUMENT, buf);
	}
	memset(&p, 0, sizeof(p));
	memcpy(p.ops, ops, count * sizeof(vxb_op));
	p.count = (int)count;
	int t = 0;
	for (uint32_t i = 0; i < count; ++i)
		if (ops[i].code == VXB_OP_TERRAIN) vxs_permutation(ops[i].seed, p.perm[t++]);
	return VXB_OK;
}
}

int vxb_grid_fill_program(vxb_context* ctx, uint32_t n, const vxb_op* ops, uint32_t count, const float start[3], float step)
{
	if (!ctx) return VXB_ERR_ARGUMENT;
	if (!validSize(n)) return fail(ctx, VXB_ERR_ARGUMENT, "vxb_grid_fill_program: bad size");
	std::unique_ptr<VxbProgramFillArgs> args(new VxbProgramFillArgs);
	int r = loadProgram(ctx, "vxb_grid_fill_program", ops, count, args->prog);
	if (r != VXB_OK) return r;
	cudaSetDevice(ctx->device);
	const bool pieces = ctx->cube.active;
	if (pieces && ctx->cube.n != n) return fail(ctx, VXB_ERR_ARGUMENT, "vxb_grid_fill_program: n differs from the cube's");
	r = pieces ? VXB_OK : ensureGridStorage(ctx, n);
	if (r != VXB_OK) return r;
	const size_t nb = n / 16;
	VXB_CUDA(ctx, ctx->progList.ensure(nb * nb * nb));
	VXB_CUDA(ctx, ctx->progCount.ensure(1));
	for (cudaEvent_t& e : ctx->progEv) if (!e) VXB_CUDA(ctx, cudaEventCreate(&e));
	for (int k = 0; k < 3; ++k) args->start[k] = start ? start[k] : 0.f;
	args->step = step;
	args->n = (int)n;
	signed char* dDist = const_cast<signed char*>(reinterpret_cast<const signed char*>(pieces ? ctx->dDist : reinterpret_cast<const int8_t*>(ctx->volDist.p)));
	unsigned char* dMat = pieces ? const_cast<unsigned char*>(ctx->dMat) : ctx->volMat.p;
	unsigned char* dBlend = pieces ? const_cast<unsigned char*>(ctx->dBlend) : ctx->volBlend.p;
	// block ranges: the whole grid, or the z-pieces this rank backs (multiples of 32 planes, so whole block layers)
	std::vector<std::pair<unsigned, unsigned> > ranges;
	if (pieces) for (uint32_t p = ctx->cube.rank; p < ctx->cube.pieces; p += ctx->cube.world)
		ranges.push_back(std::make_pair((unsigned)(p * ctx->cube.groupPlanes / 16 * nb * nb), (unsigned)((p + 1) * ctx->cube.groupPlanes / 16 * nb * nb)));
	else ranges.push_back(std::make_pair(0u, (unsigned)(nb * nb * nb)));
	uint64_t blocks = 0;
	VXB_CUDA(ctx, cudaMemsetAsync(ctx->progCount.p, 0, sizeof(unsigned), ctx->stream));
	cudaEventRecord(ctx->progEv[0], ctx->stream);
	for (const auto& rg : ranges)
	{
		args->b0 = rg.first; args->b1 = rg.second;
		blocks += rg.second - rg.first;
		vxb_program_cull_kernel<<<(rg.second - rg.first + 255) / 256, 256, 0, ctx->stream>>>(*args, dDist, dMat, dBlend, ctx->progList.p, ctx->progCount.p);
	}
	cudaEventRecord(ctx->progEv[1], ctx->stream);
	vxb_program_fill_kernel<<<(unsigned)ctx->smCount * 8, 256, 0, ctx->stream>>>(*args, ctx->progList.p, ctx->progCount.p, dDist, dMat, dBlend);
	cudaEventRecord(ctx->progEv[2], ctx->stream);
	const cudaError_t e = cudaGetLastError();
	const cudaError_t e2 = cudaStreamSynchronize(ctx->stream);
	if (e != cudaSuccess || e2 != cudaSuccess) return fail(ctx, VXB_ERR_CUDA, "vxb_grid_fill_program", e != cudaSuccess ? e : e2);
	unsigned listed = 0;
	VXB_CUDA(ctx, cudaMemcpy(&listed, ctx->progCount.p, sizeof(unsigned), cudaMemcpyDeviceToHost));
	ctx->progStats.blocks = blocks;
	ctx->progStats.culled = blocks - listed;
	cudaEventElapsedTime(&ctx->progStats.pass_a_ms, ctx->progEv[0], ctx->progEv[1]);
	cudaEventElapsedTime(&ctx->progStats.pass_b_ms, ctx->progEv[1], ctx->progEv[2]);
	if (pieces) { ctx->haveResult = false; ctx->haveFullRun = false; return VXB_OK; }
	return finishUpload(ctx);
}

int vxb_grid_inject_program(vxb_context* ctx, const float position[3], const float extents[3], const vxb_op* ops, uint32_t count,
	int type, float outMin[3], float outMax[3])
{
	if (!ctx || !position || !extents) return VXB_ERR_ARGUMENT;
	if (type < 0 || type > 2) return fail(ctx, VXB_ERR_ARGUMENT, "vxb_grid_inject_program: bad injection type");
	std::unique_ptr<VxbProgramEditArgs> a(new VxbProgramEditArgs);
	const int lr = loadProgram(ctx, "vxb_grid_inject_program", ops, count, a->prog);
	if (lr != VXB_OK) return lr;
	cudaSetDevice(ctx->device);
	VxbEditArgs e;
	const int r = prepareEdit(ctx, "vxb_grid_inject_program: needs a context-owned grid (upload or fill)", position, extents, e, outMin, outMax);
	if (r < 0) return r;
	if (r == 1) return VXB_OK;
	for (int k = 0; k < 3; ++k) { a->position[k] = e.position[k]; a->extents[k] = e.extents[k]; a->b0[k] = e.b0[k]; a->bn[k] = e.bn[k]; }
	a->type = type; a->n = e.n;
	vxb_inject_program_kernel<<<(unsigned)(e.bn[0] * e.bn[1] * e.bn[2]), 256, 0, ctx->stream>>>(*a, reinterpret_cast<signed char*>(ctx->volDist.p));
	VXB_CUDA(ctx, cudaGetLastError());
	ctx->haveResult = false;
	return VXB_OK;
}

int vxb_grid_program_stats(vxb_context* ctx, vxb_program_stats* out)
{
	if (!ctx || !out) return VXB_ERR_ARGUMENT;
	*out = ctx->progStats;
	return VXB_OK;
}

int vxb_grid_pack(vxb_context* ctx, void* out, size_t capacity, size_t* written)
{
	if (!ctx || !out) return VXB_ERR_ARGUMENT;
	if (!ctx->haveGrid) return fail(ctx, VXB_ERR_STATE, "vxb_grid_pack: no grid");
	cudaSetDevice(ctx->device);
	const uint32_t n = ctx->n;
	const size_t nb = n / 16, blocks = nb * nb * nb;
	const size_t head = 16 + blocks * 12;
	if (capacity < head) return fail(ctx, VXB_ERR_CAPACITY, "vxb_grid_pack: capacity below the header + size table");
	VXB_CUDA(ctx, ctx->packSizes.ensure(blocks * 3));
	VXB_CUDA(ctx, ctx->packFlags.ensure(blocks));
	VXB_CUDA(ctx, ctx->packOffsets.ensure(blocks + 1));
	const unsigned char* d = reinterpret_cast<const unsigned char*>(ctx->dDist);
	vxb_pack_sizes_kernel<<<(unsigned)blocks, VXB_THREADS, 0, ctx->stream>>>(d, ctx->dMat, ctx->dBlend, (int)n, ctx->packSizes.p, ctx->packFlags.p);
	vxb_pack_offsets_kernel<<<1, 1024, 0, ctx->stream>>>(ctx->packSizes.p, ctx->packOffsets.p, blocks, (unsigned long long)head);
	unsigned long long total = 0;
	VXB_CUDA(ctx, cudaMemcpyAsync(&total, ctx->packOffsets.p + blocks, sizeof(total), cudaMemcpyDeviceToHost, ctx->stream));
	VXB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	if (total > capacity) return fail(ctx, VXB_ERR_CAPACITY, "vxb_grid_pack: capacity too small (vxb_pack_dense_bound is always enough)");
	VXB_CUDA(ctx, ctx->staging.ensure((size_t)total + 16));
	vxb_pack_write_kernel<<<(unsigned)blocks, VXB_THREADS, 0, ctx->stream>>>(d, ctx->dMat, ctx->dBlend, (int)n, ctx->packFlags.p, ctx->packOffsets.p, ctx->staging.p);
	VXB_CUDA(ctx, cudaGetLastError());
	unsigned char* bytes = static_cast<unsigned char*>(out);
	const uint32_t header[4] = { 1u, n, n, n };
	memcpy(bytes, header, 16);
	VXB_CUDA(ctx, cudaMemcpyAsync(bytes + 16, ctx->packSizes.p, blocks * 12, cudaMemcpyDeviceToHost, ctx->stream));
	VXB_CUDA(ctx, cudaMemcpyAsync(bytes + head, ctx->staging.p + head, (size_t)total - head, cudaMemcpyDeviceToHost, ctx->stream));
	VXB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	if (written) *written = (size_t)total;
	return VXB_OK;
}

int vxb_grid_download_dense(vxb_context* ctx, int8_t* dist, uint8_t* mat, uint8_t* blend)
{
	if (!ctx) return VXB_ERR_ARGUMENT;
	if (!ctx->haveGrid) return fail(ctx, VXB_ERR_STATE, "vxb_grid_download_dense: no grid");
	cudaSetDevice(ctx->device);
	const size_t vol = (size_t)ctx->n * ctx->n * ctx->n;
	if (dist) VXB_CUDA(ctx, cudaMemcpyAsync(dist, ctx->dDist, vol, cudaMemcpyDeviceToHost, ctx->stream));
	if (mat) VXB_CUDA(ctx, cudaMemcpyAsync(mat, ctx->dMat, vol, cudaMemcpyDeviceToHost, ctx->stream));
	if (blend) VXB_CUDA(ctx, cudaMemcpyAsync(blend, ctx->dBlend, vol, cudaMemcpyDeviceToHost, ctx->stream));
	VXB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return VXB_OK;
}

int vxb_grid_set_device(vxb_context* ctx, uint32_t n, const int8_t* dDist, const uint8_t* dMat, const uint8_t* dBlend)
{
	if (!ctx) return VXB_ERR_ARGUMENT;
	if (!validSize(n) || !dDist || !dMat || !dBlend) return fail(ctx, VXB_ERR_ARGUMENT, "vxb_grid_set_device: bad size or null pointer");
	if ((reinterpret_cast<uintptr_t>(dDist) & 15) != 0) return fail(ctx, VXB_ERR_ARGUMENT, "vxb_grid_set_device: dist must be 16-byte aligned");
	cudaSetDevice(ctx->device);
	ctx->dDist = dDist; ctx->dMat = dMat; ctx->dBlend = dBlend;
	ctx->n = n; ctx->levels = levelsFor(n);
	ctx->ownsGrid = false; ctx->haveGrid = true; ctx->haveResult = false; ctx->haveFullRun = false;
	return buildTensorMap(ctx);
}

int vxb_grid_device_pointers(vxb_context* ctx, const int8_t** dDist, const uint8_t** dMat, const uint8_t** dBlend)
{
	if (!ctx || !ctx->haveGrid) return fail(ctx, VXB_ERR_STATE, "no grid");
	if (dDist) *dDist = ctx->dDist;
	if (dMat) *dMat = ctx->dMat;
	if (dBlend) *dBlend = ctx->dBlend;
	return VXB_OK;
}

int vxb_set_materials(vxb_context* ctx, const uint8_t* table, const uint8_t* valid)
{
	if (!ctx) return VXB_ERR_ARGUMENT;
	cudaSetDevice(ctx->device);
	VxbMaterialLut lut;
	for (unsigned i = 0; i < 256; ++i)
	{
		unsigned d0[3], d1[3];
		for (int k = 0; k < 3; ++k) { d0[k] = table ? table[i * 6 + k] : i; d1[k] = table ? table[i * 6 + 3 + k] : i; }
		// byte order of PolygonVertex::Textures: Reserved, Blend, Uxz, Txz | Uny, Upy, Tny, Tpy  (TransVoxelImpl.cpp:1253-1261)
		lut.tex0[i] = (d1[1] << 16) | (d0[1] << 24);
		lut.tex1[i] = d1[2] | (d1[0] << 8) | (d0[2] << 16) | (d0[0] << 24);
		lut.valid[i] = valid ? (valid[i] != 0) : 1;
	}
	VXB_CUDA(ctx, cudaMemcpy(ctx->lut.p, &lut, sizeof(lut), cudaMemcpyHostToDevice));
	memcpy(ctx->lutValid, lut.valid, 256);
	return VXB_OK;
}

int vxb_set_capacity(vxb_context* ctx, uint64_t v, uint64_t i, uint64_t tv, uint64_t ti)
{
	if (!ctx) return VXB_ERR_ARGUMENT;
	if (v) ctx->capV = v;
	if (i) ctx->capI = i;
	if (tv) ctx->capTV = tv;
	if (ti) ctx->capTI = ti;
	return VXB_OK;
}

int vxb_set_launch_limit(vxb_context* ctx, uint32_t ctas)
{
	if (!ctx) return VXB_ERR_ARGUMENT;
	ctx->launchLimit = ctas; // part of the graph key: the next run re-captures
	return VXB_OK;
}

int vxb_run_work_items(vxb_context* ctx, uint32_t level, uint32_t* items, uint32_t* emitted)
{
	if (!ctx || level >= VXB_MAX_LEVELS) return VXB_ERR_ARGUMENT;
	if (!ctx->haveResult) return fail(ctx, VXB_ERR_STATE, "vxb_run_work_items: no run has completed");
	if (items) *items = ctx->runWork[level];
	if (emitted) *emitted = ctx->runEmit[level];
	return VXB_OK;
}

} // extern "C"

namespace
{
// what a run is: a whole run on one context, or - vxb_polygonize_sharded's phase - a piece of a sharded run around the
// two exchanges, or a whole sharded step with the exchanges inside
enum RunPhase
{
	kRunSingle = -1,
	kShardScan = 0,   // scan + block info (no sync)
	kShardLevels = 1, // plan + the levels below the coarse ones + page publication (no sync)
	kShardTail = 2,   // coarse levels, emission, directory (syncs, result)
	kShardWhole = 3,  // everything, the two exchanges by ncclAllGather on the context's stream (needs vxb_shard_nccl_init)
};

// one run of a context and its parts; a full run is all of them in order, a whole sharded step has an exchange after the
// scan and after the levels
struct Run
{
	vxb_context* ctx;
	vxb_context::Shard& sh;
	cudaStream_t st;
	const Region* region; // an incremental run's dirty box per level; null for a full run
	RunPhase phase;
	uint32_t flags;
	bool sharded;
	bool kernelTimes = false, latticeForked = false; // latticeForked: the coarse lattices are being built on stream2
	int computed = 0;
	LevelLayout L;
	VxbDev dev;
	VxbCoarseLattices scanLat;
	VxbPeers peers;
	VxbPeerLattices peerLat;
	size_t blocksAt(int l) const { return region ? region->count[l] : L.blocks[l]; }
	void joinLattice() { if (latticeForked) { cudaStreamWaitEvent(st, ctx->evLatticeJoin, 0); latticeForked = false; } }

	// checks, the per-level layout, the per-run buffers, the kernels' view of the run (VxbDev) and of the peers
	int prepare(uint32_t maxLevels)
	{
		if (!ctx->haveGrid) return fail(ctx, VXB_ERR_STATE, "vxb_polygonize: no grid uploaded");
		if (ctx->downloadOpen) return fail(ctx, VXB_ERR_STATE, "vxb_polygonize: a result download is open (vxb_result_download_end first)");
		cudaSetDevice(ctx->device);
		ctx->haveResult = false;
		++ctx->runSerial;
		const uint32_t n = ctx->n;
		const int levels = ctx->levels, coarseLo = ctx->coarseLo;
		const size_t blocks0 = blocksAtLevel(n, 0);
		computed = (maxLevels == 0 || (int)maxLevels > levels) ? levels : (int)maxLevels;
		kernelTimes = (flags & VXB_FLAG_KERNEL_TIMES) != 0 && (!sharded || phase == kShardWhole);

		VXB_CUDA(ctx, ctx->scanFlags.ensure(blocks0));
		VXB_CUDA(ctx, ctx->blockInfo.ensure(blocks0));
		VXB_CUDA(ctx, ctx->consPages.ensure(blocks0 * 128));
		memset(&dev, 0, sizeof(dev));
		L = levelLayout(n, levels, coarseLo, &dev);
		VXB_CUDA(ctx, ctx->validFlags.ensure(L.validBytes));
		VXB_CUDA(ctx, ctx->cachePages.ensure(L.pageEntries ? L.pageEntries : 1));
		VXB_CUDA(ctx, ctx->mixInfo.ensure(L.mixBytes ? L.mixBytes : 16));
		VXB_CUDA(ctx, ctx->mixCount.ensure(L.mixBytes ? L.mixBytes : 16));
		VXB_CUDA(ctx, ctx->coarseDone.ensure(L.coarseBlocks ? L.coarseBlocks : 16));
		VXB_CUDA(ctx, ctx->worklist.ensure(L.totalBlocks));
		VXB_CUDA(ctx, ctx->records.ensure(L.totalBlocks));
		VXB_CUDA(ctx, ctx->emitList.ensure(L.totalBlocks));
		VXB_CUDA(ctx, ctx->bigList.ensure(L.totalBlocks));
		VXB_CUDA(ctx, ctx->transList.ensure(L.totalBlocks));
		VXB_CUDA(ctx, ctx->blockRecs.ensure(L.totalBlocks));
		VXB_CUDA(ctx, ctx->ntScratch.ensure(L.totalBlocks * 256));

		const uint64_t vol = sharded ? (uint64_t)n * n * n / sh.world * 2 : (uint64_t)n * n * n;
		if (!ctx->capV) ctx->capV = std::max<uint64_t>(1u << 20, vol / 24);
		if (!ctx->capI) ctx->capI = ctx->capV * 6;
		if (!ctx->capTV) ctx->capTV = std::max<uint64_t>(1u << 18, ctx->capV / 8);
		if (!ctx->capTI) ctx->capTI = ctx->capTV * 6;
		if (!ctx->capC) ctx->capC = ctx->capV + ctx->capV / 4;

		dev.grid.dist = ctx->dDist; dev.grid.mat = ctx->dMat; dev.grid.blend = ctx->dBlend; dev.grid.n = (int)n;
		dev.n = (int)n; dev.levels = levels; dev.lastLevel = levels - 1; dev.computed = computed;
		dev.scanFlags = ctx->scanFlags.p; dev.blockInfo = ctx->blockInfo.p;
		dev.consPages = ctx->consPages.p;
		dev.consValid = ctx->validFlags.p + L.validOff[0];
		for (int l = 1; l < levels; ++l)
		{
			dev.cachePages[l] = ctx->cachePages.p + L.pageOff[l]; dev.cacheValid[l] = ctx->validFlags.p + L.validOff[l];
			dev.mixInfo[l] = ctx->mixInfo.p + L.mixOff[l];
			dev.mixCount[l] = ctx->mixCount.p + L.mixOff[l];
		}
		dev.coarseLo = coarseLo; dev.coarseDone = ctx->coarseDone.p;
		memset(&scanLat, 0, sizeof(scanLat));
		scanLat.lo = VXB_LATTICE_LO; scanLat.levels = levels;
		for (int l = VXB_LATTICE_LO; l < levels; ++l) { dev.coarseLattice[l] = ctx->coarseLatticeBase + ctx->coarseLatticeOff[l]; scanLat.p[l] = dev.coarseLattice[l]; }
		dev.coarseMaps = ctx->coarseMaps.p;
		dev.latticeLo = VXB_LATTICE_LO;
		dev.worklist = ctx->worklist.p;
		dev.records = ctx->records.p; dev.rcap = (unsigned)L.totalBlocks;
		dev.counters = ctx->counters.p; dev.lut = ctx->lut.p;
		dev.transitions = (flags & VXB_FLAG_NO_TRANSITIONS) ? 0 : 1;
		dev.emitList = ctx->emitList.p; dev.bigList = ctx->bigList.p; dev.transList = ctx->transList.p; dev.ntScratch = ctx->ntScratch.p;
		dev.blockRecs = ctx->blockRecs.p;
		dev.lattice1 = ctx->haveLattice1 ? ctx->latticePtr : nullptr;
		dev.incremental = dev.ranged = region ? 1 : 0;
		if (region)
			for (int l = 0; l < levels; ++l)
			{
				for (int a = 0; a < 3; ++a) { dev.rangeMin[l][a] = region->rangeMin[l][a]; dev.rangeMax[l][a] = region->rangeMax[l][a]; }
				dev.idStart[l] = region->idStart[l];
			}
		memset(&peers, 0, sizeof(peers));
		memset(&peerLat, 0, sizeof(peerLat));
		if (!sharded) return VXB_OK;
		if (!sh.on) return fail(ctx, VXB_ERR_STATE, "vxb_polygonize_sharded: call vxb_shard_configure first");
		if (sh.sbLevel != coarseLo - 1 || coarseLo >= levels) return fail(ctx, VXB_ERR_STATE, "vxb_polygonize_sharded: the grid changed since vxb_shard_configure");
		dev.shardWorld = (int)sh.world; dev.shardRank = (int)sh.rank; dev.shardLayers = (int)sh.groupLayers;
		dev.sbLevel = sh.sbLevel; dev.sbMine = sh.sbMine.p; dev.sbWeight = sh.sbWeight.p;
		// the pages of the super-block level live in the buffer the peers write into
		dev.cachePages[sh.sbLevel] = sh.pages(sh.pagesBuf);
		dev.cacheValid[sh.sbLevel] = sh.valid(sh.pagesBuf);
		for (uint32_t p = 0; p < sh.world; ++p)
		{
			if (p == sh.rank) continue;
			if (!sh.peerSet[p]) return fail(ctx, VXB_ERR_STATE, "vxb_polygonize_sharded: a peer's page buffer is not set (vxb_shard_set_peer / vxb_shard_import)");
			peers.pages[peers.count] = sh.peerPages[p]; peers.valid[peers.count] = sh.peerValid[p];
			peers.peerSlots[peers.count] = sh.slots(sh.peerPages[p]);
			peerLat.base[peers.count] = sh.lattices(sh.peerPages[p]);
			++peers.count;
		}
		peerLat.count = peers.count;
		peers.mySlots = sh.slots(sh.pagesBuf);
		peers.epoch = sh.epoch();
		peers.arrived = sh.arrived();
		peers.rank = (int)sh.rank;
		if (phase == kShardWhole && sh.world > 1 && (!sh.comm || !ncclApi().ok)) return fail(ctx, VXB_ERR_STATE, "vxb_polygonize_sharded: phase 3 needs vxb_shard_nccl_init");
		return VXB_OK;
	}

	// the scan, the coarse levels' lattices and the block info
	int enqueueScan(Launcher& launch)
	{
		const size_t nb0 = ctx->n / 16;
		const int scanWorld = sharded ? (int)sh.world : 1, scanRank = sharded ? (int)sh.rank : 0, scanGroup = sharded ? (int)sh.groupLayers : (int)nb0;
		VXB_CUDA(ctx, cudaMemsetAsync(ctx->counters.p, 0, sizeof(VxbCounters), st));
		if (!region) VXB_CUDA(ctx, cudaMemsetAsync(ctx->validFlags.p, 0, L.validBytes, st)); // incremental runs keep the caches (:362-364)
		if (sharded) VXB_CUDA(ctx, cudaMemsetAsync(sh.valid(sh.pagesBuf), 0, sh.validBytes, st));
		if (L.coarseBlocks) VXB_CUDA(ctx, cudaMemsetAsync(ctx->coarseDone.p, 0, L.coarseBlocks, st));
		// incremental runs: only the block layers of the level-0 dirty box changed since the last run
		const int zBase = region ? std::max(0, region->rangeMin[0][2]) : 0;
		const size_t myLayers = region ? (size_t)std::max(0, std::min((int)nb0, region->rangeMax[0][2]) - zBase) : nb0 / scanWorld;
		if (!myLayers) return VXB_OK;
		const int perCta = nb0 >= 32 ? 32 : 8;
		const dim3 grid((unsigned)((nb0 + perCta - 1) / perCta), (unsigned)nb0, (unsigned)myLayers);
		unsigned char* lattice1 = ctx->haveLattice1 ? ctx->latticePtr : nullptr;
		launch(0, st, perCta == 32 ? vxb_scan_kernel<32> : vxb_scan_kernel<8>, grid, VXB_THREADS, 0,
			ctx->dDist, (int)ctx->n, ctx->scanFlags.p, lattice1, scanGroup, scanWorld, scanRank, zBase);
		if (VXB_LATTICE_LO < computed)
		{
			// the sample lattices of levels >= 2: needed only by vxb_block_kernel<2>, so a single-GPU run computes them on the
			// second stream next to the block walk and the level-0 kernel; a sharded rank does the rows of its own planes here
			const bool cubeRows = sharded && ctx->cube.active; // the volumes are split over the ranks: own rows here, then published
			const cudaStream_t ls = (cubeRows || kernelTimes || phase == kShardScan) ? st : ctx->stream2;
			if (ls != st) { VXB_CUDA(ctx, cudaEventRecord(ctx->evLatticeFork, st)); VXB_CUDA(ctx, cudaStreamWaitEvent(ls, ctx->evLatticeFork, 0)); }
			launch(1, ls, vxb_coarse_lattice_kernel, (unsigned)ctx->smCount * 4, 256, 0, reinterpret_cast<const signed char*>(ctx->dDist), (int)ctx->n, scanLat,
				cubeRows ? (int)sh.groupLayers * 16 : 1, cubeRows ? (int)sh.world : 0, cubeRows ? (int)sh.rank : 0);
			if (ls != st) { VXB_CUDA(ctx, cudaEventRecord(ctx->evLatticeJoin, ls)); latticeForked = true; }
		}
		// the lattice planes of my layers -> every peer (ordered before the peers' coarse levels by the exchanges)
		if (sharded && ctx->cube.active && peerLat.count && VXB_LATTICE_LO < ctx->levels)
			launch(8, st, vxb_publish_lattice_kernel, (unsigned)ctx->smCount, VXB_THREADS, 0, dev, peerLat, ctx->coarseLatticeBase);
		const size_t mine = myLayers * nb0 * nb0;
		const unsigned g2 = (unsigned)std::min<size_t>((mine + 255) / 256, (size_t)ctx->smCount * 8);
		launch(1, st, vxb_block_info_kernel, g2, 256, 0, ctx->dDist, (int)ctx->n, ctx->scanFlags.p, ctx->blockInfo.p, mine, scanGroup, scanWorld, scanRank, zBase);
		return VXB_OK;
	}

	// the sign-mix pyramid, level 0 and the levels below the coarse ones; a sharded run plans its share first and publishes
	// its pages to the peers last
	int enqueueLevels(Launcher& launch)
	{
		const int levels = ctx->levels;
		auto selectLevel = [&](int l) {
			const size_t b = blocksAt(l);
			launch(1, st, vxb_select_kernel, (unsigned)std::min<size_t>((b + 255) / 256, (size_t)ctx->smCount * 8), 256, 0, dev, l);
			return b;
		};
		if (levels > 1)
		{
			// sign-mix pyramid: the block walk of levels >= 2 and (sharded runs) the weights of the super-blocks
			size_t threadsA = 0;
			for (int l = 1; l < levels && l <= 2; ++l) threadsA += L.blocks[l];
			launch(1, st, vxb_pyramid_kernel, (unsigned)((threadsA + 255) / 256), 256, 0, dev);
			if (levels > 3) launch(1, st, vxb_pyramid_top_kernel, 1, 1024, 0, dev);
		}
		if (sharded) launch(1, st, vxb_plan_kernel, 1, 1024, 0, dev);
		if (selectLevel(0))
			launch(3, st, vxb_block_kernel<0>, ctx->persistentGrid(ctx->gridBlock[0]), VXB_THREADS, sizeof(VxbBlockSmem<0>), ctx->tmapDist19, ctx->tmapDist19, dev, 0);
		launch(Launcher::kNoKind, st, vxb_mark_split_kernel, 1, 1, 0, dev); // level 0 is complete: the flat kernels work behind the split
		for (int l = 1; l < ctx->coarseLo && l < computed; ++l)
		{
			if (!selectLevel(l)) continue;
			if (l >= VXB_LATTICE_LO) joinLattice();
			launch(2, st, vxb_block_kernel<1>, ctx->persistentGrid(ctx->gridBlock[1]), VXB_THREADS, sizeof(VxbBlockSmem<1>), ctx->tmap, ctx->tmap1, dev, l);
		}
		if (sharded && peers.count) launch(9, st, vxb_publish_kernel, (unsigned)ctx->smCount * 4, VXB_THREADS, 0, dev, peers);
		VXB_CUDA(ctx, cudaGetLastError());
		return VXB_OK;
	}

	// the coarse levels, the big blocks, vertices, triangles and transition cells, and the directory
	int enqueueTail(Launcher& launch)
	{
		const unsigned flatGrid = ctx->persistentGrid(ctx->smCount * 8);
		if (computed > ctx->coarseLo)
		{
			joinLattice(); // the lattices are complete
			launch(2, st, vxb_block_kernel<2>, ctx->persistentGrid(ctx->gridBlock[2]), VXB_THREADS, sizeof(VxbBlockSmem<2>), ctx->tmap, ctx->tmap1, dev, ctx->coarseLo);
		}
		// blocks too large for the shared-memory path of vxb_block_kernel (> 1024 non-trivial cells / > 2048 level-0 vertices)
		launch(2, st, vxb_big_block_kernel, ctx->persistentGrid(ctx->gridBigBlock), VXB_THREADS, sizeof(VxbBigBlockSmem), ctx->tmap, ctx->tmap1, dev);
		// vertices + triangles of everything but the level-0 blocks done inside vxb_block_kernel<0>, next to the transition
		// cells (which need the block records and the material pages only)
		const bool transitions = dev.transitions && computed > 1;
		const bool fork = transitions && !kernelTimes;
		if (fork) { VXB_CUDA(ctx, cudaEventRecord(ctx->evFork, st)); VXB_CUDA(ctx, cudaStreamWaitEvent(ctx->stream2, ctx->evFork, 0)); }
		launch(4, st, vxb_vertex_kernel, flatGrid, VXB_THREADS, 0, dev);
		launch(5, st, vxb_triangle_kernel, flatGrid, VXB_THREADS, 0, dev);
		if (transitions)
		{
			const cudaStream_t ts = fork ? ctx->stream2 : st;
			launch(6, ts, vxb_transition_kernel, ctx->persistentGrid(ctx->gridTransition), VXB_TR_THREADS, 0, dev);
			launch(6, ts, vxb_transition_vertex_kernel, flatGrid, VXB_THREADS, 0, dev);
			if (fork) { VXB_CUDA(ctx, cudaEventRecord(ctx->evJoin, ctx->stream2)); VXB_CUDA(ctx, cudaStreamWaitEvent(st, ctx->evJoin, 0)); }
		}
		joinLattice();
		launch(7, st, vxb_finish_kernel, (unsigned)ctx->smCount * 2, VXB_THREADS, 0, dev);
		VXB_CUDA(ctx, cudaGetLastError());
		return VXB_OK;
	}

	// a whole sharded step exchanges after the scan and after the levels (one rank has nothing to exchange)
	int enqueueAll(Launcher& launch)
	{
		const bool exchanges = phase == kShardWhole && sh.world > 1;
		int rc = enqueueScan(launch);
		if (rc == VXB_OK && exchanges)
		{
			// exchange 0: all-gather of the block info; every rank's layers are one contiguous chunk (rank-major layout)
			const size_t chunk = blocksAtLevel(ctx->n, 0) / sh.world;
			launch.bracket(8, [&] { rc = ncclApi().allGather(ctx->blockInfo.p + chunk * sh.rank, ctx->blockInfo.p, chunk * sizeof(unsigned int), /*ncclUint8*/ 1, sh.comm, st); });
			if (rc != 0) return failNccl(ctx, "ncclAllGather (block info)", rc);
		}
		if (rc == VXB_OK) rc = enqueueLevels(launch);
		// exchange 1: the pages were written straight into the peers' buffers by vxb_publish_kernel, whose last CTA announced
		// this step's epoch to every peer; waiting for the peers' epochs orders every rank's coarse levels after every rank's
		// publication (a device-side barrier over the mapped buffers: ~5 us instead of a ~40 us one-word all-gather)
		if (rc == VXB_OK && exchanges) launch(9, st, vxb_peer_wait_kernel, 1, 32, 0, peers, (int)sh.world);
		if (rc == VXB_OK) rc = enqueueTail(launch);
		return rc;
	}

	// every kernel argument of the run, its flags and the launch limit: a re-upload into other buffers, grown arenas or
	// other flags make a new key
	std::vector<unsigned char> graphKey() const
	{
		std::vector<unsigned char> key(sizeof(VxbDev) + sizeof(VxbPeers) + sizeof(VxbPeerLattices) + 3 * sizeof(CUtensorMap) + 64, 0);
		unsigned char* k = key.data();
		memcpy(k, &dev, sizeof(VxbDev)); k += sizeof(VxbDev);
		memcpy(k, &peers, sizeof(VxbPeers)); k += sizeof(VxbPeers);
		memcpy(k, &peerLat, sizeof(VxbPeerLattices)); k += sizeof(VxbPeerLattices);
		const CUtensorMap* maps[3] = { &ctx->tmap, &ctx->tmap1, &ctx->tmapDist19 };
		for (const CUtensorMap* mp : maps) { memcpy(k, mp, sizeof(CUtensorMap)); k += sizeof(CUtensorMap); }
		const void* ptrs[4] = { ctx->dDist, ctx->scanFlags.p, ctx->blockInfo.p, ctx->haveLattice1 ? ctx->latticePtr : nullptr };
		memcpy(k, ptrs, sizeof(ptrs)); k += sizeof(ptrs);
		const int scalars[7] = { computed, (int)L.validBytes, (int)(ctx->n / 16), (int)ctx->n, (int)phase, (int)flags, (int)ctx->launchLimit };
		memcpy(k, scalars, sizeof(scalars));
		return key;
	}

	// vxb_result_info, the statistics, and what later runs need to know about this one
	void finish(const VxbCounters& hc)
	{
		// the directory stays on the device (it is part of the result resident in HBM); vxb_result_download fetches and
		// sorts it into the reference's block order on demand
		ctx->lastDev = dev; ctx->directoryFetched = false; ctx->sortedRecords.clear();

		vxb_result_info& info = ctx->info;
		info.levels_total = (uint32_t)ctx->levels; info.levels_computed = (uint32_t)computed;
		info.block_count = hc.records; info.pad = 0;
		info.vertex_span = hc.vertices; info.index_span = hc.indices;
		info.trans_vertex_span = hc.transVertices; info.trans_index_span = hc.transIndices;
		info.vertex_total = hc.vertices; info.index_total = (uint64_t)hc.indices - 3ull * hc.degenerate;
		info.trans_vertex_total = hc.transVertices; info.trans_index_total = hc.transIndices;
		// statistics (TransVoxelImpl.cpp:528-531): BlocksCalculated counts every block of every computed level;
		// TrivialCells only those of processed (not skipped) blocks.  The statistics of a sharded run are the SUM over the
		// ranks (modulo 2^32): rank 0 carries the terms that do not depend on the work split.
		uint64_t blocksCalculated = 0, processedCells = (uint64_t)hc.nonSkippedLevel0 * 4096ull;
		if (!sharded || sh.rank == 0)
			for (int l = 0; l < computed; ++l)
			{
				blocksCalculated += blocksAt(l);
				if (l) processedCells += blocksAt(l) * 4096ull;
			}
		info.stats[0] = (uint32_t)blocksCalculated;
		info.stats[1] = (uint32_t)(processedCells - hc.nonTrivial);
		info.stats[2] = hc.nonTrivial;
		info.stats[3] = hc.degenerate;
		for (int i = 0; i < 16; ++i) info.stats[4 + i] = hc.perCase[i];
		for (int i = 0; i < 8; ++i) info.used_materials[i] = hc.usedMaterials[i];
		memcpy(ctx->runWork, hc.workCount, sizeof(ctx->runWork));
		memcpy(ctx->runEmit, hc.emitCount, sizeof(ctx->runEmit));
		ctx->haveResult = true;
		ctx->resultSharded = sharded; ctx->resultRegion = region != nullptr;
		ctx->resultComplete = computed == ctx->levels && dev.transitions;
		if (!region && !sharded) { ctx->haveFullRun = (computed == ctx->levels); ctx->nextId = (uint32_t)L.totalBlocks; }
		else if (sharded) ctx->haveFullRun = false;
	}
};

// A run has no host decision inside its sequence, so it is captured once into a CUDA graph and replayed while its key
// stays the same; a replay reports the launch counts of the captured run.  A failed capture turns graphs off for good:
// then nothing is enqueued, the counts are reset for the plain launches that follow, and *replayed stays false.
template <typename Enqueue>
int launchGraph(vxb_context* ctx, const std::vector<unsigned char>& key, Enqueue enqueue, Launcher& launch, bool* replayed)
{
	if (!ctx->graphExec || key != ctx->graphKey)
	{
		if (ctx->graphExec) { cudaGraphExecDestroy(ctx->graphExec); ctx->graphExec = nullptr; }
		cudaGraph_t graph = nullptr;
		cudaError_t ce = cudaStreamBeginCapture(ctx->stream, cudaStreamCaptureModeThreadLocal);
		if (ce == cudaSuccess)
		{
			const int rc = enqueue(launch);
			ce = cudaStreamEndCapture(ctx->stream, &graph);
			if (rc != VXB_OK && ce == cudaSuccess) ce = cudaErrorUnknown;
		}
		if (ce == cudaSuccess) ce = cudaGraphInstantiate(&ctx->graphExec, graph, 0);
		if (graph) cudaGraphDestroy(graph);
		if (ce != cudaSuccess) { ctx->graphExec = nullptr; ctx->graphDisabled = true; cudaGetLastError(); }
		else { ctx->graphKey = key; ctx->graphLaunches = launch.total; memcpy(ctx->graphKindLaunches, ctx->kindLaunches, sizeof(ctx->kindLaunches)); }
	}
	if (!ctx->graphExec) { launch.reset(); return VXB_OK; }
	VXB_CUDA(ctx, cudaGraphLaunch(ctx->graphExec, ctx->stream));
	launch.total = ctx->graphLaunches;
	memcpy(ctx->kindLaunches, ctx->graphKindLaunches, sizeof(ctx->kindLaunches));
	*replayed = true;
	return VXB_OK;
}

int runPolygonize(vxb_context* ctx, uint32_t maxLevels, uint32_t flags, const Region* region, RunPhase phase = kRunSingle)
{
	if (!ctx) return VXB_ERR_ARGUMENT;
	Run r{ ctx, ctx->shard, ctx->stream, region, phase, flags, phase != kRunSingle };
	int rc = r.prepare(maxLevels);
	if (rc != VXB_OK) return rc;
	const cudaStream_t st = ctx->stream;
	VxbCounters hc;
	for (int attempt = 0; attempt < 6; ++attempt)
	{
		const uint64_t lim = 0xFFFFFFF0ull;
		ctx->capV = std::min(ctx->capV, lim); ctx->capI = std::min(ctx->capI, lim);
		ctx->capTV = std::min(ctx->capTV, lim); ctx->capTI = std::min(ctx->capTI, lim);
		ctx->capV = std::min<uint64_t>(ctx->capV, 0x0FFFFFF0ull); ctx->capC = std::min<uint64_t>(ctx->capC, 0x0FFFFFF0ull); // 28-bit cell index in the vertex list
		VXB_CUDA(ctx, ctx->verts.ensure(ctx->capV));
		VXB_CUDA(ctx, ctx->idx.ensure(ctx->capI));
		VXB_CUDA(ctx, ctx->tverts.ensure(ctx->capTV));
		VXB_CUDA(ctx, ctx->tidx.ensure(ctx->capTI));
		VXB_CUDA(ctx, ctx->vlist.ensure(ctx->capV));
		VXB_CUDA(ctx, ctx->tvlist.ensure(ctx->capTV));
		VXB_CUDA(ctx, ctx->cellRecs.ensure(ctx->capC));
		VXB_CUDA(ctx, ctx->cellBlock.ensure(ctx->capC));
		VxbDev& dev = r.dev;
		dev.verts = ctx->verts.p; dev.idx = ctx->idx.p; dev.tverts = ctx->tverts.p; dev.tidx = ctx->tidx.p;
		dev.vcap = (unsigned)ctx->capV; dev.icap = (unsigned)ctx->capI; dev.tvcap = (unsigned)ctx->capTV; dev.ticap = (unsigned)ctx->capTI;
		dev.vlist = ctx->vlist.p; dev.cellRecs = ctx->cellRecs.p; dev.cellBlock = ctx->cellBlock.p; dev.ccap = (unsigned)ctx->capC; dev.tvlist = ctx->tvlist.p;

		Launcher launch(ctx, r.kernelTimes);
		r.latticeForked = false;
		// phases 0 and 1 of a sharded run end at an exchange the caller makes: no sync, no result
		if (phase == kShardScan || phase == kShardLevels)
		{
			if (phase == kShardScan) VXB_CUDA(ctx, cudaEventRecord(ctx->evBegin, st));
			rc = phase == kShardScan ? r.enqueueScan(launch) : r.enqueueLevels(launch);
			if (phase == kShardScan) VXB_CUDA(ctx, cudaGetLastError());
			ctx->shard.phaseLaunches = (phase == kShardScan ? 0 : ctx->shard.phaseLaunches) + launch.total;
			return rc;
		}
		if (phase != kShardTail) VXB_CUDA(ctx, cudaEventRecord(ctx->evBegin, st));
		bool replayed = false;
		if (phase != kShardTail && !region && !r.kernelTimes && !ctx->graphDisabled)
			if ((rc = launchGraph(ctx, r.graphKey(), [&](Launcher& l) { return r.enqueueAll(l); }, launch, &replayed)) != VXB_OK) return rc;
		if (!replayed && (rc = phase == kShardTail ? r.enqueueTail(launch) : r.enqueueAll(launch)) != VXB_OK) return rc;
		if (phase == kShardTail) launch.total += ctx->shard.phaseLaunches;
		VXB_CUDA(ctx, cudaGetLastError());
		VXB_CUDA(ctx, cudaEventRecord(ctx->evEnd, st));
		VXB_CUDA(ctx, cudaMemcpyAsync(&hc, ctx->counters.p, sizeof(hc), cudaMemcpyDeviceToHost, st));
		VXB_CUDA(ctx, cudaStreamSynchronize(st));
		float ms = 0.f;
		VXB_CUDA(ctx, cudaEventElapsedTime(&ms, ctx->evBegin, ctx->evEnd));
		launch.collectTimes();
		ctx->info.device_ms = ms;
		ctx->info.kernel_launches = launch.total;

		const bool overflow = hc.vertices > ctx->capV || hc.indices > ctx->capI || hc.transVertices > ctx->capTV || hc.transIndices > ctx->capTI || hc.cells > ctx->capC;
		if (!overflow) break;
		if (attempt == 5) return fail(ctx, VXB_ERR_CAPACITY, "vxb_polygonize: output arenas overflowed after growing");
		if (hc.vertices > ctx->capV) ctx->capV = (uint64_t)hc.vertices + hc.vertices / 8 + 1024;
		if (hc.indices > ctx->capI) ctx->capI = (uint64_t)hc.indices + hc.indices / 8 + 1024;
		if (hc.transVertices > ctx->capTV) ctx->capTV = (uint64_t)hc.transVertices + hc.transVertices / 8 + 1024;
		if (hc.transIndices > ctx->capTI) ctx->capTI = (uint64_t)hc.transIndices + hc.transIndices / 8 + 1024;
		if (hc.cells > ctx->capC) ctx->capC = (uint64_t)hc.cells + hc.cells / 8 + 1024;
		// a sharded run is collective: the caller repeats it on every rank
		if (r.sharded) return fail(ctx, VXB_ERR_CAPACITY, "vxb_polygonize_sharded: output arenas overflowed; capacities were grown, repeat the run on every rank");
	}
	r.finish(hc);
	return VXB_OK;
}
}

extern "C"
{

int vxb_polygonize(vxb_context* ctx, uint32_t maxLevels, uint32_t flags)
{
	return runPolygonize(ctx, maxLevels, flags, nullptr);
}

int vxb_polygonize_region(vxb_context* ctx, const float minCorner[3], const float maxCorner[3], uint32_t flags)
{
	if (!ctx || !minCorner || !maxCorner) return VXB_ERR_ARGUMENT;
	if (!ctx->haveGrid || !ctx->haveFullRun) return fail(ctx, VXB_ERR_STATE, "vxb_polygonize_region: needs a full vxb_polygonize of this grid first (the caches of that run are updated in place)");
	// GenerateBlockListForLevel, modification branch (TransVoxelImpl.cpp:429-465); corners are in OUTPUT (Y-up) coordinates
	Region region;
	vxb_region_info& ri = ctx->region;
	memset(&ri, 0, sizeof(ri));
	ri.levels = (uint32_t)ctx->levels;
	const float extent = (float)ctx->n;
	uint32_t id = ctx->nextId;
	for (int l = 0; l < ctx->levels; ++l)
	{
		const float blockMult = (float)((1 << l) * 16);
		float minBlock[3], maxBlock[3];
		for (int c = 0; c < 3; ++c)
		{
			float lo = floorf(minCorner[c] / blockMult - 1.0f) * blockMult, hi = floorf(maxCorner[c] / blockMult + 2.0f) * blockMult;
			lo = lo < 0.f ? 0.f : (lo > extent ? extent : lo);
			hi = hi < 0.f ? 0.f : (hi > extent ? extent : hi);
			ri.min_dirty[l][c] = lo; ri.max_dirty[l][c] = hi;
			minBlock[c] = lo / blockMult; maxBlock[c] = hi / blockMult;
		}
		// back to grid (Z-up) axes: x <- x, y <- output z, z <- output y  (:455-458)
		const unsigned lo3[3] = { (unsigned)minBlock[0], (unsigned)minBlock[2], (unsigned)minBlock[1] };
		const unsigned hi3[3] = { (unsigned)maxBlock[0], (unsigned)maxBlock[2], (unsigned)maxBlock[1] };
		size_t count = 1;
		for (int a = 0; a < 3; ++a)
		{
			region.rangeMin[l][a] = (int)lo3[a]; region.rangeMax[l][a] = (int)hi3[a];
			count *= hi3[a] > lo3[a] ? hi3[a] - lo3[a] : 0;
		}
		region.idStart[l] = id; region.count[l] = count;
		ri.id_start[l] = id; ri.block_count[l] = (uint32_t)count;
		id += (uint32_t)count;
	}
	const int r = runPolygonize(ctx, 0, flags, &region);
	if (r == VXB_OK) ctx->nextId = id;
	return r;
}

// ---- sharded runs (SURVEY.md section 8e): one grid, `world` ranks, one GPU each ----

int vxb_shard_configure(vxb_context* ctx, uint32_t rank, uint32_t world, uint32_t groupPlanes)
{
	if (!ctx) return VXB_ERR_ARGUMENT;
	if (!ctx->haveGrid) return fail(ctx, VXB_ERR_STATE, "vxb_shard_configure: no grid (vxb_cube_create or vxb_grid_set_device first)");
	const uint32_t n = ctx->n;
	if (world == 0 || world > 8 || rank >= world) return fail(ctx, VXB_ERR_ARGUMENT, "vxb_shard_configure: world in [1, 8], rank < world");
	if (groupPlanes == 0) groupPlanes = n / world;
	if (groupPlanes % 32 != 0 || n % groupPlanes != 0 || (n / groupPlanes) % world != 0)
		return fail(ctx, VXB_ERR_ARGUMENT, "vxb_shard_configure: group_planes must be a multiple of 32 planes that divides n into a multiple of `world` pieces");
	if (ctx->cube.active && (ctx->cube.groupPlanes != groupPlanes || ctx->cube.world != world || ctx->cube.rank != rank))
		return fail(ctx, VXB_ERR_ARGUMENT, "vxb_shard_configure: rank / world / group_planes differ from the cube's");
	const int coarseLo = coarseLoFor(n, ctx->levels);
	if (coarseLo >= ctx->levels) return fail(ctx, VXB_ERR_ARGUMENT, "vxb_shard_configure: the grid is too small to shard (n >= 64)");
	cudaSetDevice(ctx->device);
	releaseShard(ctx);
	vxb_context::Shard& sh = ctx->shard;
	sh.rank = rank; sh.world = world; sh.groupLayers = groupPlanes / 16; sh.sbLevel = coarseLo - 1;
	const size_t sb = blocksAtLevel(n, sh.sbLevel);
	VXB_CUDA(ctx, sh.sbMine.ensure(sb));
	VXB_CUDA(ctx, sh.sbWeight.ensure(sb));
	sh.pagesBytes = sb * 4096 * sizeof(unsigned short);
	sh.validBytes = (sb + 255) & ~(size_t)255;
	size_t offs[VXB_MAX_LEVELS];
	sh.latticeBytes = (coarseLatticeLayout(n, ctx->levels, offs) + 255) & ~(size_t)255;
	sh.bufBytes = sh.barrierOffset() + sh.barrierBytes;
	const VmmApi& api = vmmApi();
	if (api.ok)
	{
		// exportable (the peers map it and store their pages into it)
		const CUmemAllocationProp prop = slabProp(ctx->device);
		size_t gran = 0;
		VXB_CU(ctx, api.granularity(&gran, &prop, CU_MEM_ALLOC_GRANULARITY_MINIMUM));
		sh.bufBytes = (sh.bufBytes + gran - 1) / gran * gran;
		VXB_CU(ctx, api.addressReserve(&sh.pagesVa, sh.bufBytes, 0, 0, 0));
		VXB_CU(ctx, api.create(&sh.pagesHandle, sh.bufBytes, &prop, 0));
		std::vector<std::pair<CUdeviceptr, size_t> > scratch;
		const int r = mapRange(ctx, sh.pagesVa, sh.bufBytes, sh.pagesHandle, scratch);
		if (r != VXB_OK) return r;
		sh.pagesVmm = true;
		sh.pagesBuf = reinterpret_cast<unsigned char*>(sh.pagesVa);
	}
	else
	{
		VXB_CUDA(ctx, cudaMalloc(reinterpret_cast<void**>(&sh.pagesBuf), sh.bufBytes));
	}
	VXB_CUDA(ctx, cudaMemset(sh.barrier(sh.pagesBuf), 0, sh.barrierBytes));
	sh.on = true;
	// virtual ranks over one shared upload: no shared even-lattice copy => level 1 gathers its tiles.  The coarse levels'
	// lattices move into the buffer the peers map (buildTensorMap -> buildCoarseLattices).
	if (!ctx->cube.active) ctx->latticeOff = true;
	{
		const int r = buildTensorMap(ctx);
		if (r != VXB_OK) return r;
	}
	if (ctx->graphExec) { cudaGraphExecDestroy(ctx->graphExec); ctx->graphExec = nullptr; }
	ctx->graphKey.clear();
	return VXB_OK;
}

int vxb_shard_buffers_get(vxb_context* ctx, vxb_shard_buffers* out)
{
	if (!ctx || !out) return VXB_ERR_ARGUMENT;
	const vxb_context::Shard& sh = ctx->shard;
	if (!sh.on) return fail(ctx, VXB_ERR_STATE, "vxb_shard_buffers_get: call vxb_shard_configure first");
	const size_t nb0 = ctx->n / 16, blocks0 = nb0 * nb0 * nb0;
	cudaSetDevice(ctx->device);
	VXB_CUDA(ctx, ctx->blockInfo.ensure(blocks0));
	memset(out, 0, sizeof(*out));
	out->block_info = ctx->blockInfo.p;
	out->block_info_bytes = blocks0 * sizeof(unsigned int);
	out->chunk_bytes = blocks0 / sh.world * sizeof(unsigned int);
	out->pages = sh.pagesBuf;
	out->pages_bytes = sh.pagesBytes;
	out->valid = sh.valid(sh.pagesBuf);
	out->valid_bytes = sh.validBytes;
	out->super_level = (uint32_t)sh.sbLevel;
	return VXB_OK;
}

int vxb_shard_set_peer(vxb_context* ctx, uint32_t peer, void* pages, void* valid)
{
	if (!ctx) return VXB_ERR_ARGUMENT;
	vxb_context::Shard& sh = ctx->shard;
	if (!sh.on || peer >= sh.world || peer == sh.rank || !pages || !valid) return fail(ctx, VXB_ERR_ARGUMENT, "vxb_shard_set_peer: not configured, or bad peer / pointer");
	sh.peerPages[peer] = static_cast<unsigned short*>(pages);
	sh.peerValid[peer] = static_cast<unsigned char*>(valid);
	sh.peerSet[peer] = true;
	return VXB_OK;
}

int vxb_shard_export(vxb_context* ctx, int* fd)
{
	if (!ctx || !fd) return VXB_ERR_ARGUMENT;
	const vxb_context::Shard& sh = ctx->shard;
	if (!sh.on || !sh.pagesVmm) return fail(ctx, VXB_ERR_STATE, "vxb_shard_export: needs vxb_shard_configure (and a driver with the virtual memory management API)");
	cudaSetDevice(ctx->device);
	int out = -1;
	VXB_CU(ctx, vmmApi().exportHandle(&out, sh.pagesHandle, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0));
	*fd = out;
	return VXB_OK;
}

int vxb_shard_import(vxb_context* ctx, uint32_t peer, int fd)
{
	if (!ctx) return VXB_ERR_ARGUMENT;
	vxb_context::Shard& sh = ctx->shard;
	if (!sh.on || !sh.pagesVmm || peer >= sh.world || peer == sh.rank || fd < 0) return fail(ctx, VXB_ERR_ARGUMENT, "vxb_shard_import: not configured, or bad peer / descriptor");
	cudaSetDevice(ctx->device);
	const VmmApi& api = vmmApi();
	CUmemGenericAllocationHandle h = 0;
	VXB_CU(ctx, api.importHandle(&h, (void*)(uintptr_t)fd, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR));
	sh.peerHandles.push_back(h);
	CUdeviceptr va = 0;
	VXB_CU(ctx, api.addressReserve(&va, sh.bufBytes, 0, 0, 0));
	const int r = mapRange(ctx, va, sh.bufBytes, h, sh.peerMapped);
	if (r != VXB_OK) return r;
	return vxb_shard_set_peer(ctx, peer, reinterpret_cast<void*>(va), sh.valid(reinterpret_cast<void*>(va)));
}

int vxb_shard_nccl_unique_id(vxb_nccl_id* id)
{
	if (!id) return VXB_ERR_ARGUMENT;
	const NcclApi& api = ncclApi();
	if (!api.ok) return fail(nullptr, VXB_ERR_CUDA, "vxb_shard_nccl_unique_id: libnccl.so.2 could not be loaded");
	const int r = api.getUniqueId(id);
	return r == 0 ? VXB_OK : failNccl(nullptr, "ncclGetUniqueId", r);
}

int vxb_shard_nccl_init(vxb_context* ctx, const vxb_nccl_id* id, uint32_t rank, uint32_t world)
{
	if (!ctx || !id) return VXB_ERR_ARGUMENT;
	const NcclApi& api = ncclApi();
	if (!api.ok) return fail(ctx, VXB_ERR_CUDA, "vxb_shard_nccl_init: libnccl.so.2 could not be loaded");
	cudaSetDevice(ctx->device);
	if (ctx->shard.comm) { api.commDestroy(ctx->shard.comm); ctx->shard.comm = nullptr; }
	const int r = api.commInitRank(&ctx->shard.comm, (int)world, *id, (int)rank);
	return r == 0 ? VXB_OK : failNccl(ctx, "ncclCommInitRank", r);
}

int vxb_polygonize_sharded(vxb_context* ctx, uint32_t phase, uint32_t flags)
{
	if (!ctx) return VXB_ERR_ARGUMENT;
	if (phase > 3) return fail(ctx, VXB_ERR_ARGUMENT, "vxb_polygonize_sharded: phase is 0, 1, 2 (the pieces around the two exchanges) or 3 (everything, NCCL inside)");
	return runPolygonize(ctx, 0, flags, nullptr, (RunPhase)phase);
}

int vxb_region_info_get(vxb_context* ctx, vxb_region_info* out)
{
	if (!ctx || !out) return VXB_ERR_ARGUMENT;
	*out = ctx->region;
	return VXB_OK;
}

int vxb_grid_update_blocks(vxb_context* ctx, uint32_t count, const uint32_t* blockCoords, const int8_t* dist, const uint8_t* mat, const uint8_t* blend)
{
	if (!ctx) return VXB_ERR_ARGUMENT;
	if (!ctx->haveGrid || !ctx->ownsGrid) return fail(ctx, VXB_ERR_STATE, "vxb_grid_update_blocks: needs a grid uploaded into context-owned storage");
	if (!count) return VXB_OK;
	if (!blockCoords || !dist) return fail(ctx, VXB_ERR_ARGUMENT, "vxb_grid_update_blocks: null pointer");
	cudaSetDevice(ctx->device);
	const size_t bytes = (size_t)count * 4096;
	VXB_CUDA(ctx, ctx->staging.ensure(bytes));
	VXB_CUDA(ctx, ctx->updCoords.ensure((size_t)count * 3));
	const uint32_t nb = ctx->n / 16;
	for (uint32_t i = 0; i < count * 3; ++i) if (blockCoords[i] >= nb) return fail(ctx, VXB_ERR_ARGUMENT, "vxb_grid_update_blocks: block coordinate out of range");
	VXB_CUDA(ctx, cudaMemcpyAsync(ctx->updCoords.p, blockCoords, (size_t)count * 12, cudaMemcpyHostToDevice, ctx->stream));
	const void* src[3] = { dist, mat, blend };
	uint8_t* dst[3] = { ctx->volDist.p, ctx->volMat.p, ctx->volBlend.p };
	for (int c = 0; c < 3; ++c)
	{
		if (!src[c]) continue; // channel unchanged
		VXB_CUDA(ctx, cudaMemcpyAsync(ctx->staging.p, src[c], bytes, cudaMemcpyHostToDevice, ctx->stream));
		vxb_unpack_block_list_kernel<<<count, VXB_THREADS, 0, ctx->stream>>>(reinterpret_cast<const uint4*>(ctx->staging.p), ctx->updCoords.p, dst[c], (int)ctx->n);
		VXB_CUDA(ctx, cudaGetLastError());
		VXB_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); // staging is reused by the next channel
	}
	ctx->haveResult = false;
	return VXB_OK;
}

int vxb_result_info_get(vxb_context* ctx, vxb_result_info* out)
{
	if (!ctx || !out) return VXB_ERR_ARGUMENT;
	if (!ctx->haveResult) return fail(ctx, VXB_ERR_STATE, "no result: call vxb_polygonize first");
	*out = ctx->info;
	return VXB_OK;
}

int vxb_result_download(vxb_context* ctx, vxb_block_record* records, void* vertices, uint32_t* indices, void* transVertices, uint32_t* transIndices)
{
	const int r = vxb_result_download_begin(ctx, records, vertices, indices, transVertices, transIndices);
	return r != VXB_OK ? r : vxb_result_download_end(ctx);
}

int vxb_result_download_begin(vxb_context* ctx, vxb_block_record* records, void* vertices, uint32_t* indices, void* transVertices, uint32_t* transIndices)
{
	if (!ctx) return VXB_ERR_ARGUMENT;
	if (!ctx->haveResult) return fail(ctx, VXB_ERR_STATE, "no result: call vxb_polygonize first");
	if (ctx->downloadOpen) return fail(ctx, VXB_ERR_STATE, "vxb_result_download_begin: the previous download was not ended");
	cudaSetDevice(ctx->device);
	const vxb_result_info& info = ctx->info;
	// directory first (small, into page-locked scratch), the arenas queued right behind it; the directory is sorted into the
	// reference's block order (level, then z,y,x = coord id; :395-401, :1278) on the host while the arenas are in flight
	const bool fetch = !ctx->directoryFetched;
	if (fetch && info.block_count)
	{
		if (!ctx->hostRecords.ensure(sizeof(vxb_block_record) * info.block_count)) return fail(ctx, VXB_ERR_CUDA, "vxb_result_download: pinned scratch allocation failed");
		VXB_CUDA(ctx, cudaMemcpyAsync(ctx->hostRecords.p, ctx->records.p, sizeof(vxb_block_record) * info.block_count, cudaMemcpyDeviceToHost, ctx->stream));
		VXB_CUDA(ctx, cudaEventRecord(ctx->evDir, ctx->stream));
	}
	if (vertices && info.vertex_span) VXB_CUDA(ctx, cudaMemcpyAsync(vertices, ctx->verts.p, info.vertex_span * sizeof(VxbVertex), cudaMemcpyDeviceToHost, ctx->stream));
	if (indices && info.index_span) VXB_CUDA(ctx, cudaMemcpyAsync(indices, ctx->idx.p, info.index_span * 4, cudaMemcpyDeviceToHost, ctx->stream));
	if (transVertices && info.trans_vertex_span) VXB_CUDA(ctx, cudaMemcpyAsync(transVertices, ctx->tverts.p, info.trans_vertex_span * sizeof(VxbVertex), cudaMemcpyDeviceToHost, ctx->stream));
	if (transIndices && info.trans_index_span) VXB_CUDA(ctx, cudaMemcpyAsync(transIndices, ctx->tidx.p, info.trans_index_span * 4, cudaMemcpyDeviceToHost, ctx->stream));
	if (fetch)
	{
		ctx->sortedRecords.resize(info.block_count);
		if (info.block_count)
		{
			VXB_CUDA(ctx, cudaEventSynchronize(ctx->evDir));
			memcpy(ctx->sortedRecords.data(), ctx->hostRecords.p, sizeof(vxb_block_record) * info.block_count);
		}
		std::sort(ctx->sortedRecords.begin(), ctx->sortedRecords.end(), [](const vxb_block_record& a, const vxb_block_record& b) {
			return a.level != b.level ? a.level < b.level : a.coord_id < b.coord_id; });
		ctx->directoryFetched = true;
	}
	if (records && info.block_count) memcpy(records, ctx->sortedRecords.data(), sizeof(vxb_block_record) * info.block_count);
	ctx->downloadOpen = true;
	ctx->downloadVerts = vertices;
	ctx->downloadTransVerts = transVertices;
	return VXB_OK;
}

int vxb_result_download_end(vxb_context* ctx)
{
	if (!ctx) return VXB_ERR_ARGUMENT;
	if (!ctx->downloadOpen) return fail(ctx, VXB_ERR_STATE, "vxb_result_download_end without vxb_result_download_begin");
	ctx->downloadOpen = false;
	cudaSetDevice(ctx->device);
	const vxb_result_info& info = ctx->info;
	void* const vertices = ctx->downloadVerts;
	void* const transVertices = ctx->downloadTransVerts;
	VXB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));

	// vertices of unmapped materials carry a marker (vxb_finish_vertex); restore the reference's all-zero textures
	ctx->unmapped.clear();
	bool anyUnmapped = false;
	for (unsigned i = 0; i < 256; ++i) if (!ctx->lutValid[i] && ((info.used_materials[i >> 5] >> (i & 31)) & 1u)) anyUnmapped = true;
	if (anyUnmapped)
	{
		auto fix = [&](void* base, uint64_t off, uint32_t count) {
			if (!base) return;
			VxbVertex* v = static_cast<VxbVertex*>(base) + off;
			for (uint32_t i = 0; i < count; ++i)
				if ((v[i].tex[0] & 0xFFu) == 0xFFu) { ctx->unmapped.push_back((uint8_t)(v[i].tex[0] >> 8)); v[i].tex[0] = 0; v[i].tex[1] = 0; }
		};
		for (const vxb_block_record& r : ctx->sortedRecords)
		{
			fix(vertices, r.vertex_offset, r.vertex_count);
			for (int f = 0; f < 6; ++f) fix(transVertices, r.trans_vertex_offset[f], r.trans_vertex_count[f]);
		}
	}
	return VXB_OK;
}

int vxb_result_device_arenas(vxb_context* ctx, const void** vertices, const uint32_t** indices, const void** transVertices, const uint32_t** transIndices)
{
	if (!ctx) return VXB_ERR_ARGUMENT;
	if (!ctx->haveResult) return fail(ctx, VXB_ERR_STATE, "no result: call vxb_polygonize first");
	if (vertices) *vertices = ctx->verts.p;
	if (indices) *indices = ctx->idx.p;
	if (transVertices) *transVertices = ctx->tverts.p;
	if (transIndices) *transIndices = ctx->tidx.p;
	return VXB_OK;
}

} // extern "C"

namespace
{
// vxb_lod_select_kernel over `blocks` records of d.records into the given lists (sized to `cap` blocks)
int selectLod(vxb_context* ctx, const VxbDev& d, uint32_t blocks, size_t cap, const float camera[3], float baseDistance,
	DevBuf<vxb_draw_command>& cmd, DevBuf<vxb_draw_info>& info, DevBuf<vxb_draw_command>& tcmd, DevBuf<vxb_draw_info>& tinfo,
	DevBuf<unsigned int>& counts, vxb_draw_lists& l)
{
	VXB_CUDA(ctx, cmd.ensure(cap)); VXB_CUDA(ctx, info.ensure(cap));
	VXB_CUDA(ctx, tcmd.ensure(cap * 6)); VXB_CUDA(ctx, tinfo.ensure(cap * 6));
	VXB_CUDA(ctx, counts.ensure(2));
	VXB_CUDA(ctx, cudaMemsetAsync(counts.p, 0, 8, ctx->stream));
	VxbLodArgs a;
	for (int k = 0; k < 3; ++k) a.camera[k] = camera[k];
	a.lod = baseDistance;
	a.counts = counts.p;
	a.regular = cmd.p; a.regularInfo = info.p; a.transition = tcmd.p; a.transitionInfo = tinfo.p;
	a.capacity = (unsigned)(cap * 6);
	if (blocks) vxb_lod_select_kernel<<<(blocks + 255) / 256, 256, 0, ctx->stream>>>(d, a, blocks);
	unsigned n[2] = { 0, 0 };
	VXB_CUDA(ctx, cudaMemcpyAsync(n, counts.p, 8, cudaMemcpyDeviceToHost, ctx->stream));
	VXB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	VXB_CUDA(ctx, cudaGetLastError());
	l.regular_count = n[0]; l.transition_count = n[1];
	l.counts = counts.p;
	l.regular = cmd.p; l.regular_info = info.p; l.transition = tcmd.p; l.transition_info = tinfo.p;
	return VXB_OK;
}
}

extern "C"
{

int vxb_result_select_lod(vxb_context* ctx, const float camera[3], float baseDistance, vxb_draw_lists* out)
{
	if (!ctx || !camera) return VXB_ERR_ARGUMENT;
	if (!ctx->haveResult) return fail(ctx, VXB_ERR_STATE, "no result: call vxb_polygonize first");
	cudaSetDevice(ctx->device);
	const uint32_t blocks = ctx->info.block_count;
	const int r = selectLod(ctx, ctx->lastDev, blocks, blocks ? blocks : 1, camera, baseDistance, ctx->drawCmd, ctx->drawInfo, ctx->drawTCmd,
		ctx->drawTInfo, ctx->drawCounts, ctx->drawLists);
	if (r != VXB_OK) return r;
	if (out) *out = ctx->drawLists;
	return VXB_OK;
}

int vxb_result_download_draws(vxb_context* ctx, vxb_draw_command* regular, vxb_draw_info* regularInfo, vxb_draw_command* transition, vxb_draw_info* transitionInfo)
{
	if (!ctx) return VXB_ERR_ARGUMENT;
	cudaSetDevice(ctx->device);
	const vxb_draw_lists& l = ctx->drawLists;
	if (regular && l.regular_count) VXB_CUDA(ctx, cudaMemcpy(regular, l.regular, sizeof(vxb_draw_command) * l.regular_count, cudaMemcpyDeviceToHost));
	if (regularInfo && l.regular_count) VXB_CUDA(ctx, cudaMemcpy(regularInfo, l.regular_info, sizeof(vxb_draw_info) * l.regular_count, cudaMemcpyDeviceToHost));
	if (transition && l.transition_count) VXB_CUDA(ctx, cudaMemcpy(transition, l.transition, sizeof(vxb_draw_command) * l.transition_count, cudaMemcpyDeviceToHost));
	if (transitionInfo && l.transition_count) VXB_CUDA(ctx, cudaMemcpy(transitionInfo, l.transition_info, sizeof(vxb_draw_info) * l.transition_count, cudaMemcpyDeviceToHost));
	return VXB_OK;
}

uint64_t vxb_result_unmapped_materials(vxb_context* ctx, uint8_t* ids, uint64_t capacity)
{
	if (!ctx) return 0;
	const uint64_t n = ctx->unmapped.size();
	if (ids) memcpy(ids, ctx->unmapped.data(), (size_t)std::min<uint64_t>(n, capacity));
	return n;
}

void* vxb_host_alloc(size_t bytes)
{
	void* p = nullptr;
	if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) return nullptr;
	return p;
}

void vxb_host_free(void* p) { if (p) cudaFreeHost(p); }

int vxb_kernel_ms(vxb_context* ctx, int which, float* ms, uint32_t* launches)
{
	if (!ctx || which < 0 || which > 9) return VXB_ERR_ARGUMENT;
	if (ms) *ms = ctx->kindMs[which];
	if (launches) *launches = ctx->kindLaunches[which];
	return VXB_OK;
}

} // extern "C"

// ---- the mesh (include/vxb200.h "mesh"; kernels: vxb_mesh.cuh) ----
struct vxb_mesh
{
	vxb_context* ctx = nullptr;
	struct Arenas
	{
		DevBuf<VxbVertex> v, tv;
		DevBuf<unsigned int> i, ti;
		VxbMeshArenas view() const { VxbMeshArenas a; a.v = v.p; a.i = i.p; a.tv = tv.p; a.ti = ti.p; return a; }
		cudaError_t ensure(const uint64_t cap[4])
		{
			cudaError_t e = v.ensure(cap[0]);
			if (e == cudaSuccess) e = i.ensure(cap[1]);
			if (e == cudaSuccess) e = tv.ensure(cap[2]);
			if (e == cudaSuccess) e = ti.ensure(cap[3]);
			return e;
		}
		void release() { v.release(); i.release(); tv.release(); ti.release(); }
	} set[2];                                   // set[active] holds the mesh; the other one is the target of a compaction
	int active = 0;
	uint64_t cap[4] = { 0, 0, 0, 0 }, span[4] = { 0, 0, 0, 0 }, total[4] = { 0, 0, 0, 0 };
	DevBuf<vxb_block_record> dir, scratch;      // the directory, and the merged one an apply writes before it replaces it
	size_t dirCap = 0;                          // every (level, coord) slot of the grid: a mesh holds each block at most once
	DevBuf<unsigned int> keys, vals, keysOut, valsOut, jobSrc, jobDst;
	DevBuf<VxbMeshScan> items, prefix;
	DevBuf<unsigned char> cubTemp;
	DevBuf<VxbMeshCounts> counts;
	DevBuf<vxb_draw_command> drawCmd, drawTCmd;
	DevBuf<vxb_draw_info> drawInfo, drawTInfo;
	DevBuf<unsigned int> drawCounts;
	vxb_draw_lists drawLists;
	// bounds: two float4 {min, max} per (level, coord) slot, written by the apply; `bounds` describes them as of the last apply
	DevBuf<float4> boxes;
	vxb_mesh_bounds bounds;
	DevBuf<float> boundsOut;                    // vxb_mesh_download_bounds' device staging
	// the per-view lists of vxb_mesh_select_lod_views and of vxb_mesh_select_cut, each call its own: view v owns entries
	// [v * stride, +stride) (transition: 6 x) and counts[2v], counts[2v + 1]
	struct ViewLists
	{
		DevBuf<vxb_draw_command> cmd, tcmd;
		DevBuf<vxb_draw_info> info, tinfo;
		DevBuf<unsigned int> counts;
	} viewLists, cutLists;
	cudaEvent_t ev[2] = { nullptr, nullptr };
	bool content = false;                       // a run has been applied
	bool complete = false;                      // every run applied since the last full apply made all levels and transitions
	uint64_t serial = 0;                        // vxb_context::runSerial of that run
	uint32_t n = 0;
	vxb_mesh_info info;
	// A map built lazily for one applied run (`serial`) on one grid (`n`); every apply has a new serial.
	struct LazyMap
	{
		DevBuf<unsigned int> buf;
		bool built = false;
		uint64_t serial = 0;
		uint32_t n = 0;
	};
	// ray casts and the other level-0 queries (vxb_ray.cuh): the level-0 coord_id -> slot map
	LazyMap rayMap;
	// cut ray casts (vxb_cutray.cuh): the all-level map (bounds slot -> directory slot) and the excursion measured with it;
	// separate from rayMap, so the level-0 queries never see them
	LazyMap cutMap;
	DevBuf<unsigned int> cutExcursion;
	float excursion = 0.f;
	// the host variants' device staging of queries and hits, shared by every query and grown as needed
	DevBuf<unsigned char> stageIn, stageOut;
	// box overlap gathers (vxb_overlap.cuh): the per-box counts and the scan's storage, the host variant's offsets
	DevBuf<uint64_t> overlapCounts, overlapOffsets;
	DevBuf<unsigned char> overlapTemp;
};

namespace
{
void deleteMesh(vxb_mesh* m)
{
	for (cudaEvent_t e : m->ev) if (e) cudaEventDestroy(e);
	delete m; // the buffers free themselves
}

uint64_t grownCapacity(uint64_t live) { return (std::max<uint64_t>(live + live / 2, 1024) + 3) & ~(uint64_t)3; }

// Whether `map` was built for another applied run or grid.  If so, it is readied on ctx->stream for its rebuild: grown to
// `entries` (a query still queued may read the old map, so the stream drains first) and filled with VXB_RAY_MISS.
int staleMap(vxb_mesh* m, vxb_mesh::LazyMap& map, size_t entries, bool& stale)
{
	vxb_context* ctx = m->ctx;
	stale = !map.built || map.serial != m->serial || map.n != m->n;
	if (!stale) return VXB_OK;
	if (entries > map.buf.count)
	{
		VXB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
		VXB_CUDA(ctx, map.buf.ensure(entries));
	}
	VXB_CUDA(ctx, cudaMemsetAsync(map.buf.p, 0xFF, entries * sizeof(unsigned int), ctx->stream));
	return VXB_OK;
}

void markBuilt(const vxb_mesh* m, vxb_mesh::LazyMap& map) { map.built = true; map.serial = m->serial; map.n = m->n; }

// The level-0 map for the applied run, queued on ctx->stream, and the kernels' view of the mesh.
int ensureMap(vxb_mesh* m, VxbRayMesh& rm)
{
	const uint32_t nb = m->n / 16;
	bool stale;
	const int e = staleMap(m, m->rayMap, (size_t)nb * nb * nb, stale);
	if (e != VXB_OK) return e;
	if (stale)
	{
		const unsigned level0 = m->info.level_blocks[0];
		if (level0) vxb_ray_map_kernel<<<(level0 + 255) / 256, 256, 0, m->ctx->stream>>>(m->dir.p, level0, m->rayMap.buf.p);
		VXB_CUDA(m->ctx, cudaGetLastError());
		markBuilt(m, m->rayMap);
	}
	rm.dir = m->dir.p; rm.map = m->rayMap.buf.p; rm.verts = m->set[m->active].v.p; rm.idx = m->set[m->active].i.p; rm.nb = (int)nb;
	return VXB_OK;
}

// The all-level map and the excursion for the applied run, queued on ctx->stream; the excursion is read back, so a rebuild
// waits for the stream once.  Then the refusals of an excursion beyond the walk's reach, alone and with the query's reach
// `reach` (the sweep radius or max_distance; 0 for rays), and the kernel's view of the mesh.
int ensureCutMap(vxb_mesh* m, const char* what, float reach, VxbCutRayMesh& c)
{
	vxb_context* ctx = m->ctx;
	cudaStream_t st = ctx->stream;
	const uint32_t nb = m->n / 16;
	VxbCutMapArgs a;
	for (int l = 0; l < VXB_MAX_LEVELS; ++l) a.levelBase[l] = m->bounds.level_base[l];
	a.nb = (int)nb;
	bool stale;
	const int e = staleMap(m, m->cutMap, m->bounds.slots, stale);
	if (e != VXB_OK) return e;
	if (stale)
	{
		VXB_CUDA(ctx, m->cutExcursion.ensure(1));
		VXB_CUDA(ctx, cudaMemsetAsync(m->cutExcursion.p, 0, sizeof(unsigned int), st));
		const unsigned blocks = m->info.block_count;
		if (blocks) vxb_cutray_map_kernel<<<(blocks + 255) / 256, 256, 0, st>>>(m->dir.p, blocks, a, m->boxes.p, m->cutMap.buf.p, m->cutExcursion.p);
		VXB_CUDA(ctx, cudaGetLastError());
		unsigned bits = 0;
		VXB_CUDA(ctx, cudaMemcpyAsync(&bits, m->cutExcursion.p, sizeof(bits), cudaMemcpyDeviceToHost, st));
		VXB_CUDA(ctx, cudaStreamSynchronize(st));
		memcpy(&m->excursion, &bits, sizeof(bits));
		markBuilt(m, m->cutMap);
	}
	if (!(m->excursion + VXB_RAY_EPS <= 15.f))
	{
		char buf[192];
		snprintf(buf, sizeof(buf), "%s: a block's vertices leave its lattice box by %g voxels; the walk reaches 15 - 1/16", what, (double)m->excursion);
		return fail(ctx, VXB_ERR_STATE, buf);
	}
	if (!(m->excursion + reach <= 15.f))
	{
		char buf[224];
		snprintf(buf, sizeof(buf), "%s: a block's vertices leave its lattice box by %g voxels (e) and the query reaches %g (R); "
			"e + R must be at most 15", what, (double)m->excursion, (double)reach);
		return fail(ctx, VXB_ERR_STATE, buf);
	}
	c.m.dir = m->dir.p; c.m.map = m->cutMap.buf.p; c.m.verts = m->set[m->active].v.p; c.m.idx = m->set[m->active].i.p; c.m.nb = (int)nb;
	c.tverts = m->set[m->active].tv.p; c.tidx = m->set[m->active].ti.p;
	c.boxes = m->boxes.p;
	c.slots = a;
	c.top = (int)m->info.levels - 1;
	c.grow = std::nextafter(m->excursion + VXB_RAY_EPS, INFINITY);
	c.excursion = m->excursion;
	memset(&c.cut, 0, sizeof(c.cut));
	return VXB_OK;
}

// CTAs of a persistent one-warp-per-query launch
unsigned queryCtas(const vxb_context* ctx, uint32_t count, unsigned threads)
{
	const unsigned warpsPerCta = threads / 32;
	return std::min<unsigned>((count + warpsPerCta - 1) / warpsPerCta, (unsigned)std::max(ctx->smCount, 1) * 8);
}

// A level-0 query's launch on ctx->stream: `kernel(rm, args...)`, one warp per query over the level-0 map (ensureMap).
template <class Kernel, class... Args>
int launchLevel0(vxb_mesh* m, Kernel kernel, unsigned threads, uint32_t count, Args... args)
{
	VxbRayMesh rm;
	const int e = ensureMap(m, rm);
	if (e != VXB_OK) return e;
	kernel<<<queryCtas(m->ctx, count, threads), threads, 0, m->ctx->stream>>>(rm, args...);
	VXB_CUDA(m->ctx, cudaGetLastError());
	return VXB_OK;
}

// A cut query's launch on ctx->stream: `kernel(c, args...)`, one warp per query over the all-level map (ensureCutMap, with
// the batch's reach) and the cut of (camera, lodFactor).  `inReach(e)` runs between the map and the launch: the host capsule
// variants' per-query reach check against the excursion e (anyReach for every other query).
template <class InReach, class Kernel, class... Args>
int launchCut(vxb_mesh* m, const char* what, const float camera[3], float lodFactor, float reach, InReach&& inReach, Kernel kernel,
	unsigned threads, uint32_t count, Args... args)
{
	VxbCutRayMesh c;
	int e = ensureCutMap(m, what, reach, c);
	if (e == VXB_OK) e = inReach(c.excursion);
	if (e != VXB_OK) return e;
	for (int k = 0; k < 3; ++k) c.cut.camera[k] = camera[k];
	c.cut.lod = lodFactor;
	kernel<<<queryCtas(m->ctx, count, threads), threads, 0, m->ctx->stream>>>(c, args...);
	VXB_CUDA(m->ctx, cudaGetLastError());
	return VXB_OK;
}

int anyReach(float) { return VXB_OK; }

int enqueueRaycastCut(vxb_mesh* m, const char* what, const float camera[3], float lodFactor, const vxb_ray* rays, uint32_t count, vxb_cut_hit* hits)
{
	return launchCut(m, what, camera, lodFactor, 0.f, anyReach, vxb_raycast_cut_kernel, VXB_RAY_THREADS, count, rays, count, hits);
}

int enqueueSphereCastCut(vxb_mesh* m, const char* what, const float camera[3], float lodFactor, float radius, const vxb_ray* rays,
	uint32_t count, vxb_sphere_cut_hit* hits)
{
	return launchCut(m, what, camera, lodFactor, radius, anyReach, vxb_sphere_cast_cut_kernel, VXB_COLLIDE_THREADS, count, radius, rays, count, hits);
}

int enqueueClosestPointCut(vxb_mesh* m, const char* what, const float camera[3], float lodFactor, float maxDistance, const float* points,
	uint32_t count, vxb_closest_cut_hit* hits)
{
	return launchCut(m, what, camera, lodFactor, maxDistance, anyReach, vxb_closest_point_cut_kernel, VXB_COLLIDE_THREADS, count, maxDistance,
		points, count, hits);
}

// The host capsule cut queries' per-query reach (vxb_capsule_cut_reach) against the excursion e: the first of the `count`
// queries out of reach is refused with VXB_ERR_STATE, naming its index, e and its reach R.  shape(i, h, extra) gives query
// i's half axis and its radius or max_distance.  NULL `noun`: the device variants, whose kernels answer such a query with a
// miss.
template <class Shape>
int capsuleCutReach(vxb_mesh* m, const char* what, const char* noun, uint32_t count, float e, Shape&& shape)
{
	if (!noun) return VXB_OK;
	for (uint32_t i = 0; i < count; ++i)
	{
		float3 h;
		float extra;
		shape(i, h, extra);
		if (vxb_capsule_cut_reach(h, extra, e)) continue;
		char buf[256];
		snprintf(buf, sizeof(buf), "%s: %s %u: a block's vertices leave its lattice box by %g voxels (e) and the %s reaches %g (R); "
			"e + R must be at most 15", what, noun, i, (double)e, noun, (double)(std::max(std::max(std::fabs(h.x), std::fabs(h.y)), std::fabs(h.z)) + extra));
		return fail(m->ctx, VXB_ERR_STATE, buf);
	}
	return VXB_OK;
}

// `checked`: the host copy of the queries for the host variant's reach check, NULL for the device variant
int enqueueCapsuleCastCut(vxb_mesh* m, const char* what, const float camera[3], float lodFactor, const vxb_capsule_sweep* checked,
	const vxb_capsule_sweep* sweeps, uint32_t count, vxb_capsule_cut_hit* hits)
{
	const auto inReach = [&](float e) {
		return capsuleCutReach(m, what, checked ? "sweep" : nullptr, count, e, [&](uint32_t i, float3& h, float& extra) {
			h = make_float3(checked[i].half_axis[0], checked[i].half_axis[1], checked[i].half_axis[2]);
			extra = checked[i].radius;
		});
	};
	return launchCut(m, what, camera, lodFactor, 0.f, inReach, vxb_capsule_cast_cut_kernel, VXB_COLLIDE_THREADS, count, sweeps, count, hits);
}

int enqueueClosestToSegmentCut(vxb_mesh* m, const char* what, const float camera[3], float lodFactor, float maxDistance,
	const vxb_segment* checked, const vxb_segment* segments, uint32_t count, vxb_segment_cut_hit* hits)
{
	const auto inReach = [&](float e) {
		return capsuleCutReach(m, what, checked ? "segment" : nullptr, count, e, [&](uint32_t i, float3& h, float& extra) {
			h = make_float3(checked[i].half_axis[0], checked[i].half_axis[1], checked[i].half_axis[2]);
			extra = maxDistance;
		});
	};
	return launchCut(m, what, camera, lodFactor, maxDistance, inReach, vxb_closest_segment_cut_kernel, VXB_COLLIDE_THREADS, count,
		maxDistance, segments, count, hits);
}

// the gather kernels' view of the mesh: the level-0 map (ensureMap) and the level-0 bounds
int overlapView(vxb_mesh* m, VxbOverlapMesh& om)
{
	const int e = ensureMap(m, om.m);
	om.boxes = m->boxes.p;
	om.base0 = m->bounds.level_base[0];
	return e;
}

// The gather's pipeline on ctx->stream: the count kernel, the exclusive scan of the counts into `offsets` (count + 1
// entries), and, when tris is given, the write kernel (which compares offsets[count] with capacity on the device).  Scratch
// that grows waits for the stream first: a gather still queued may use it.
int enqueueOverlap(vxb_mesh* m, const vxb_box* boxes, uint32_t count, uint64_t* offsets, vxb_overlap_triangle* tris, uint64_t capacity)
{
	vxb_context* ctx = m->ctx;
	cudaStream_t st = ctx->stream;
	VxbOverlapMesh om;
	const int e = overlapView(m, om);
	if (e != VXB_OK) return e;
	const uint64_t entries = (uint64_t)count + 1;
	size_t tempBytes = 0;
	VXB_CUDA(ctx, cub::DeviceScan::ExclusiveSum(nullptr, tempBytes, m->overlapCounts.p, offsets, entries, st));
	if (entries > m->overlapCounts.count || tempBytes > m->overlapTemp.count)
	{
		VXB_CUDA(ctx, cudaStreamSynchronize(st));
		VXB_CUDA(ctx, m->overlapCounts.ensure(entries)); VXB_CUDA(ctx, m->overlapTemp.ensure(std::max<size_t>(tempBytes, 1)));
	}
	const unsigned ctas = queryCtas(ctx, count, VXB_OVERLAP_THREADS);
	vxb_overlap_kernel<false><<<ctas, VXB_OVERLAP_THREADS, 0, st>>>(om, boxes, count, m->overlapCounts.p, nullptr, 0);
	VXB_CUDA(ctx, cudaGetLastError());
	VXB_CUDA(ctx, cub::DeviceScan::ExclusiveSum(m->overlapTemp.p, tempBytes, m->overlapCounts.p, offsets, entries, st));
	if (tris)
	{
		vxb_overlap_kernel<true><<<ctas, VXB_OVERLAP_THREADS, 0, st>>>(om, boxes, count, offsets, tris, capacity);
		VXB_CUDA(ctx, cudaGetLastError());
	}
	return VXB_OK;
}

// A host variant's round trip on ctx->stream: `inBytes` of queries to the staging, the enqueued query, `count` hits back;
// blocks.
template <class In, class Out, class Enqueue>
int hostQuery(vxb_mesh* m, const In* queries, size_t inBytes, uint32_t count, Out* hits, Enqueue&& enqueue)
{
	vxb_context* ctx = m->ctx;
	cudaStream_t st = ctx->stream;
	const size_t outBytes = sizeof(Out) * count;
	if (inBytes > m->stageIn.count || outBytes > m->stageOut.count)
	{
		VXB_CUDA(ctx, cudaStreamSynchronize(st)); // nothing queued may still use the staging being replaced
		VXB_CUDA(ctx, m->stageIn.ensure(inBytes)); VXB_CUDA(ctx, m->stageOut.ensure(outBytes));
	}
	VXB_CUDA(ctx, cudaMemcpyAsync(m->stageIn.p, queries, inBytes, cudaMemcpyHostToDevice, st));
	const int r = enqueue((const In*)m->stageIn.p, (Out*)m->stageOut.p);
	if (r != VXB_OK) return r;
	VXB_CUDA(ctx, cudaMemcpyAsync(hits, m->stageOut.p, outBytes, cudaMemcpyDeviceToHost, st));
	VXB_CUDA(ctx, cudaStreamSynchronize(st));
	return VXB_OK;
}

// the batch arguments of the queries (include/vxb200.h): why one is refused, or NULL.  NaN fails.
const char* radiusFault(float r) { return r > 0.f && r <= VXB_SPHERE_RADIUS_MAX ? nullptr : "radius must be in (0, 15]"; }
const char* maxDistanceFault(float d) { return d >= 0.f && d <= VXB_SPHERE_RADIUS_MAX ? nullptr : "max_distance must be in [0, 15]"; }
const char* cutFault(const float camera[3], float lodFactor)
{
	if (!std::isfinite(lodFactor) || !(lodFactor >= VXB_LOD_FACTOR_MIN)) return "lod_factor must be finite and >= 2";
	if (camera && (!std::isfinite(camera[0]) || !std::isfinite(camera[1]) || !std::isfinite(camera[2]))) return "non-finite lod_camera component";
	return nullptr;
}
// the first of two batch-argument faults, or NULL
const char* firstFault(const char* a, const char* b) { return a ? a : b; }

// the host variants' point rule (include/vxb200.h): why point i is refused, or NULL
const char* pointFault(const float* points, uint32_t i)
{
	const float* p = points + 3 * (size_t)i;
	return std::isfinite(p[0]) && std::isfinite(p[1]) && std::isfinite(p[2]) ? nullptr : "non-finite coordinate";
}

// the host variants' ray rule (include/vxb200.h): why the ray is refused, or NULL
const char* rayFault(const vxb_ray& x)
{
	bool finite = true;
	for (int a = 0; a < 3; ++a) finite = finite && std::isfinite(x.origin[a]) && std::isfinite(x.direction[a]);
	if (!finite) return "non-finite origin or direction";
	if (x.direction[0] == 0.f && x.direction[1] == 0.f && x.direction[2] == 0.f) return "zero direction";
	if (!std::isfinite(x.t_min)) return "t_min is NaN or infinite";
	if (std::isnan(x.t_max)) return "t_max is NaN";
	if (x.t_min > x.t_max) return "t_min > t_max";
	return nullptr;
}

// A host variant's per-query rule: fault(i) is why query i is refused, or NULL; `noun` names the query in the refusal.  A
// device variant has none (noun NULL): its queries are in device memory, and the kernels answer an invalid one with a miss.
template <class Fault> struct Rule { const char* noun; Fault fault; };
template <class Fault> Rule<Fault> rule(const char* noun, Fault fault) { return { noun, fault }; }
const Rule<const char* (*)(uint32_t)> deviceRule = { nullptr, nullptr };

// What a query entry checks before its rule (include/vxb200.h)
struct Entry
{
	const char* name;      // the entry point, which starts every message
	bool null;             // a pointer the call needs when count > 0 is NULL, of ...
	const char* pointers;  // ... these, as the message names them
	const char* batch;     // why a batch argument is refused, or NULL
	bool levels = false;   // the query reads every level and transition mesh: the mesh must be complete
};

// Every query entry's path, its checks in one order: a NULL pointer (only when count > 0), the batch arguments, nothing
// applied, an incomplete mesh, count == 0 (VXB_OK), the host variant's per-query rule; then `run`, the staging round trip or
// the direct enqueue, on the context's device.  Every argument check comes before every state check.
template <class Fault, class Run>
int meshQuery(vxb_mesh* m, const Entry& q, uint32_t count, const Rule<Fault>& rule, Run&& run)
{
	if (!m) return VXB_ERR_ARGUMENT;
	vxb_context* ctx = m->ctx;
	char buf[256];
	if (count && q.null) { snprintf(buf, sizeof(buf), "%s: NULL %s", q.name, q.pointers); return fail(ctx, VXB_ERR_ARGUMENT, buf); }
	if (q.batch) { snprintf(buf, sizeof(buf), "%s: %s", q.name, q.batch); return fail(ctx, VXB_ERR_ARGUMENT, buf); }
	if (!m->content) { snprintf(buf, sizeof(buf), "%s: nothing applied yet", q.name); return fail(ctx, VXB_ERR_STATE, buf); }
	if (q.levels && !m->complete)
	{
		snprintf(buf, sizeof(buf), "%s: the mesh lacks levels or transition meshes (a run since the last full apply had max_levels "
			"below the grid's levels or VXB_FLAG_NO_TRANSITIONS)", q.name);
		return fail(ctx, VXB_ERR_STATE, buf);
	}
	if (!count) return VXB_OK;
	if (rule.noun)
		for (uint32_t i = 0; i < count; ++i)
			if (const char* why = rule.fault(i))
			{
				snprintf(buf, sizeof(buf), "%s: %s %u: %s", q.name, rule.noun, i, why);
				return fail(ctx, VXB_ERR_ARGUMENT, buf);
			}
	cudaSetDevice(ctx->device);
	return run();
}

// The culled selects' shared body, after the caller's NULL, view-count and state checks: the plane check (a refusal names the
// view and the plane and leaves `lists` and `out` untouched), one pass of vxb_lod_select_views_kernel<Cut> into `lists`, one
// read of the counts.  lod: the Cut's parameter (VxbLodArgs::lod).
template <class Cut>
int selectViews(vxb_mesh* m, const char* what, const float camera[3], float lod, const vxb_view* views, uint32_t viewCount,
	vxb_mesh::ViewLists& lists, vxb_draw_lists* out)
{
	vxb_context* ctx = m->ctx;
	VxbViews vs;
	memset(&vs, 0, sizeof(vs));
	for (uint32_t v = 0; v < viewCount; ++v)
	{
		for (int k = 0; k < 6; ++k)
			for (int c = 0; c < 4; ++c)
				if (!std::isfinite(views[v].planes[k][c]))
				{
					char buf[160]; snprintf(buf, sizeof(buf), "%s: view %u plane %d: non-finite component", what, v, k);
					return fail(ctx, VXB_ERR_ARGUMENT, buf);
				}
		vs.view[v] = views[v];
	}
	cudaSetDevice(ctx->device);
	cudaStream_t st = ctx->stream;
	const uint32_t blocks = m->info.block_count;
	const size_t stride = blocks ? blocks : 1;
	VXB_CUDA(ctx, lists.cmd.ensure(stride * viewCount)); VXB_CUDA(ctx, lists.info.ensure(stride * viewCount));
	VXB_CUDA(ctx, lists.tcmd.ensure(stride * viewCount * 6)); VXB_CUDA(ctx, lists.tinfo.ensure(stride * viewCount * 6));
	VXB_CUDA(ctx, lists.counts.ensure(2 * VXB_VIEWS_MAX));
	VXB_CUDA(ctx, cudaMemsetAsync(lists.counts.p, 0, sizeof(unsigned int) * 2 * VXB_VIEWS_MAX, st));
	VxbDev d;
	memset(&d, 0, sizeof(d));
	d.n = (int)m->n; d.levels = (int)m->info.levels; d.lastLevel = d.levels - 1;
	d.records = m->dir.p;
	for (int l = 0; l < VXB_MAX_LEVELS; ++l) d.idBase[l] = m->bounds.level_base[l];
	VxbLodArgs a;
	for (int k = 0; k < 3; ++k) a.camera[k] = camera[k];
	a.lod = lod;
	a.counts = lists.counts.p;
	a.regular = lists.cmd.p; a.regularInfo = lists.info.p; a.transition = lists.tcmd.p; a.transitionInfo = lists.tinfo.p;
	a.capacity = (unsigned)(stride * 6);
	if (blocks) vxb_lod_select_views_kernel<Cut><<<(blocks + 255) / 256, 256, 0, st>>>(d, a, blocks, vs, viewCount, m->boxes.p, (unsigned)stride);
	unsigned n[2 * VXB_VIEWS_MAX];
	VXB_CUDA(ctx, cudaMemcpyAsync(n, lists.counts.p, sizeof(n), cudaMemcpyDeviceToHost, st));
	VXB_CUDA(ctx, cudaStreamSynchronize(st));
	VXB_CUDA(ctx, cudaGetLastError());
	for (uint32_t v = 0; v < viewCount; ++v)
	{
		vxb_draw_lists& l = out[v];
		l.regular_count = n[2 * v]; l.transition_count = n[2 * v + 1];
		l.counts = lists.counts.p + 2 * v;
		l.regular = lists.cmd.p + stride * v; l.regular_info = lists.info.p + stride * v;
		l.transition = lists.tcmd.p + stride * v * 6; l.transition_info = lists.tinfo.p + stride * v * 6;
	}
	return VXB_OK;
}
}

extern "C"
{

int vxb_mesh_create(vxb_context* ctx, const uint64_t capacity[4], vxb_mesh** out)
{
	if (!ctx || !out) return VXB_ERR_ARGUMENT;
	*out = nullptr;
	cudaSetDevice(ctx->device);
	vxb_mesh* m = new vxb_mesh;
	m->ctx = ctx;
	memset(&m->info, 0, sizeof(m->info));
	memset(&m->drawLists, 0, sizeof(m->drawLists));
	memset(&m->bounds, 0, sizeof(m->bounds));
	cudaError_t e = cudaEventCreate(&m->ev[0]);
	if (e == cudaSuccess) e = cudaEventCreate(&m->ev[1]);
	if (e == cudaSuccess && capacity)
	{
		for (int a = 0; a < 4; ++a) m->cap[a] = (capacity[a] + 3) & ~(uint64_t)3;
		e = m->set[0].ensure(m->cap);
	}
	if (e != cudaSuccess) { deleteMesh(m); return fail(ctx, VXB_ERR_CUDA, "vxb_mesh_create", e); }
	ctx->meshes.push_back(m);
	*out = m;
	return VXB_OK;
}

void vxb_mesh_destroy(vxb_mesh* m)
{
	if (!m) return;
	vxb_context* ctx = m->ctx;
	cudaSetDevice(ctx->device);
	cudaStreamSynchronize(ctx->stream);
	ctx->meshes.erase(std::remove(ctx->meshes.begin(), ctx->meshes.end(), m), ctx->meshes.end());
	deleteMesh(m);
}

int vxb_mesh_apply(vxb_mesh* m)
{
	if (!m) return VXB_ERR_ARGUMENT;
	vxb_context* ctx = m->ctx;
	if (!ctx->haveResult) return fail(ctx, VXB_ERR_STATE, "vxb_mesh_apply: no result: call vxb_polygonize first");
	if (ctx->resultSharded) return fail(ctx, VXB_ERR_STATE, "vxb_mesh_apply: the result is a sharded run's (a mesh takes single-context runs)");
	if (m->content && m->serial == ctx->runSerial) return fail(ctx, VXB_ERR_STATE, "vxb_mesh_apply: this run was already applied");
	const bool region = ctx->resultRegion;
	if (region && !(m->content && m->serial + 1 == ctx->runSerial))
		return fail(ctx, VXB_ERR_STATE, "vxb_mesh_apply: the mesh missed a run of the context since its last full run (apply every run, or start again from a full run)");
	cudaSetDevice(ctx->device);
	cudaStream_t st = ctx->stream;
	const uint32_t n = ctx->n;
	const int levels = ctx->levels;

	// ---- buffers: every (level, coord) slot of the grid; a new grid size moves the directory ----
	VxbMeshRange g;
	memset(&g, 0, sizeof(g));
	g.erase = region ? 1 : 0;
	const LevelLayout L = levelLayout(n, levels, ctx->coarseLo);
	const size_t slots = L.totalBlocks;
	for (int l = 0; l < levels; ++l)
	{
		g.levelBase[l] = (unsigned)L.blockBase[l];
		g.nb[l] = (int)((n >> 4) >> l);
		if (region)
		{
			// the dirty box in OUTPUT axes (x, z, y) and block units; its corners are multiples of the block size
			const float m3 = (float)((1 << l) * 16);
			const float* lo = ctx->region.min_dirty[l]; const float* hi = ctx->region.max_dirty[l];
			g.lo[l][0] = (int)(lo[0] / m3); g.lo[l][1] = (int)(lo[2] / m3); g.lo[l][2] = (int)(lo[1] / m3);
			g.hi[l][0] = (int)(hi[0] / m3); g.hi[l][1] = (int)(hi[2] / m3); g.hi[l][2] = (int)(hi[1] / m3);
		}
	}
	if (slots > m->dirCap)
	{
		VXB_CUDA(ctx, m->dir.ensure(slots)); VXB_CUDA(ctx, m->scratch.ensure(slots));
		VXB_CUDA(ctx, m->drawCmd.ensure(slots)); VXB_CUDA(ctx, m->drawInfo.ensure(slots));
		VXB_CUDA(ctx, m->drawTCmd.ensure(slots * 6)); VXB_CUDA(ctx, m->drawTInfo.ensure(slots * 6));
		VXB_CUDA(ctx, m->drawCounts.ensure(2));
		VXB_CUDA(ctx, m->boxes.ensure(slots * 2));
		m->dirCap = slots;
		++m->info.generation;
	}
	VXB_CUDA(ctx, m->keys.ensure(slots)); VXB_CUDA(ctx, m->vals.ensure(slots));
	VXB_CUDA(ctx, m->keysOut.ensure(slots)); VXB_CUDA(ctx, m->valsOut.ensure(slots));
	VXB_CUDA(ctx, m->jobSrc.ensure(slots * 2)); VXB_CUDA(ctx, m->jobDst.ensure(slots * 2));
	VXB_CUDA(ctx, m->items.ensure(slots * 2)); VXB_CUDA(ctx, m->prefix.ensure(slots * 2));
	VXB_CUDA(ctx, m->counts.ensure(1));

	const unsigned meshCount = region ? m->info.block_count : 0, runCount = ctx->info.block_count, all = meshCount + runCount;
	int sortBits = 1;
	while (sortBits < 32 && ((size_t)1 << sortBits) < slots) ++sortBits;
	size_t sortBytes = 0, scanBytes = 0;
	VXB_CUDA(ctx, cub::DeviceRadixSort::SortPairs(nullptr, sortBytes, m->keys.p, m->keysOut.p, m->vals.p, m->valsOut.p, (int)runCount, 0, sortBits, st));
	VXB_CUDA(ctx, cub::DeviceScan::ExclusiveScan(nullptr, scanBytes, m->items.p, m->prefix.p, VxbMeshScanSum(), VxbMeshScan{ 0, 0, 0, 0, 0 }, (int)all, st));
	size_t tempBytes = std::max<size_t>(std::max(sortBytes, scanBytes), 1);
	VXB_CUDA(ctx, m->cubTemp.ensure(tempBytes));
	tempBytes = m->cubTemp.count;

	// ---- count, sort the run's records by (level, coord_id), read the totals ----
	VXB_CUDA(ctx, cudaEventRecord(m->ev[0], st));
	VXB_CUDA(ctx, cudaMemsetAsync(m->counts.p, 0, sizeof(VxbMeshCounts), st));
	if (all)
		vxb_mesh_count_kernel<<<(all + 255) / 256, 256, 0, st>>>(m->dir.p, meshCount, ctx->records.p, runCount, g, m->items.p, m->keys.p, m->vals.p, m->counts.p);
	if (runCount)
	{
		VXB_CUDA(ctx, cub::DeviceRadixSort::SortPairs(m->cubTemp.p, tempBytes, m->keys.p, m->keysOut.p, m->vals.p, m->valsOut.p, (int)runCount, 0, sortBits, st));
		vxb_mesh_gather_kernel<<<(runCount + 255) / 256, 256, 0, st>>>(ctx->records.p, m->valsOut.p, runCount, m->items.p + meshCount);
	}
	VXB_CUDA(ctx, cudaGetLastError());
	VxbMeshCounts c;
	VXB_CUDA(ctx, cudaMemcpyAsync(&c, m->counts.p, sizeof(c), cudaMemcpyDeviceToHost, st));
	VXB_CUDA(ctx, cudaStreamSynchronize(st));

	// ---- where the blocks go: the tail of the active set, or a compaction into the other one ----
	uint64_t live[4], newCap[4], tail[4];
	bool compact = false, grow = false;
	for (int a = 0; a < 4; ++a)
	{
		live[a] = c.survivorElems[a] + c.freshElems[a];
		tail[a] = region ? m->span[a] : 0;
		newCap[a] = live[a] > m->cap[a] ? grownCapacity(live[a]) : m->cap[a];
		grow = grow || newCap[a] != m->cap[a];
		if (region && (tail[a] + c.freshElems[a] > m->cap[a] || tail[a] - c.survivorElems[a] > live[a])) compact = true;
	}
	if (tail[0] > 0xFFFFFFFFull || tail[1] > 0xFFFFFFFFull || tail[2] > 0xFFFFFFFFull || tail[3] > 0xFFFFFFFFull ||
		newCap[0] > 0xFFFFFFFFull || newCap[1] > 0xFFFFFFFFull || newCap[2] > 0xFFFFFFFFull || newCap[3] > 0xFFFFFFFFull)
		return fail(ctx, VXB_ERR_CAPACITY, "vxb_mesh_apply: the mesh outgrows 32-bit arena offsets");
	const bool hadArenas = m->cap[0] || m->cap[1] || m->cap[2] || m->cap[3];
	int target = m->active;
	if (compact)
	{
		target = 1 - m->active;
		VXB_CUDA(ctx, m->set[target].ensure(newCap));
	}
	else if (grow)
	{
		// a full apply replaces the content: the active set is simply reallocated
		m->set[m->active].release();
		VXB_CUDA(ctx, m->set[m->active].ensure(newCap));
	}
	for (int a = 0; a < 4; ++a) { if (compact || !region) tail[a] = 0; }

	bool anyUnmapped = false;
	for (unsigned i = 0; i < 256; ++i) if (!ctx->lutValid[i] && ((ctx->info.used_materials[i >> 5] >> (i & 31)) & 1u)) anyUnmapped = true;

	// the boxes of the blocks that leave: all of them, or the ones in the dirty range (the copy writes the new blocks')
	if (!region) vxb_mesh_bounds_reset_kernel<<<(unsigned)((slots + 255) / 256), 256, 0, st>>>(m->boxes.p, (unsigned)slots);
	else if (meshCount) vxb_mesh_bounds_erase_kernel<<<(meshCount + 255) / 256, 256, 0, st>>>(m->dir.p, meshCount, g, m->boxes.p);
	if (all)
	{
		VXB_CUDA(ctx, cub::DeviceScan::ExclusiveScan(m->cubTemp.p, tempBytes, m->items.p, m->prefix.p, VxbMeshScanSum(), VxbMeshScan{ 0, 0, 0, 0, 0 }, (int)all, st));
		const uint4 t4 = make_uint4((unsigned)tail[0], (unsigned)tail[1], (unsigned)tail[2], (unsigned)tail[3]);
		vxb_mesh_place_kernel<<<(all + 255) / 256, 256, 0, st>>>(m->dir.p, meshCount, ctx->records.p, m->valsOut.p, runCount, g, m->prefix.p,
			m->counts.p, t4, compact ? 1 : 0, m->scratch.p, m->jobSrc.p, m->jobDst.p);
	}
	unsigned survivors = 0, fresh = 0;
	for (int l = 0; l < VXB_MAX_LEVELS; ++l) { survivors += c.survivors[l]; fresh += c.fresh[l]; }
	const unsigned jobs = compact ? survivors + fresh : fresh;
	VxbMeshArenas runSrc;
	runSrc.v = ctx->verts.p; runSrc.i = ctx->idx.p; runSrc.tv = ctx->tverts.p; runSrc.ti = ctx->tidx.p;
	if (jobs)
		vxb_mesh_copy_kernel<<<jobs, 128, 0, st>>>(m->jobSrc.p, m->jobDst.p, m->dir.p, ctx->records.p, m->scratch.p, m->set[m->active].view(),
			runSrc, m->set[target].view(), anyUnmapped ? 1 : 0, m->keys.p, m->boxes.p);
	VXB_CUDA(ctx, cudaGetLastError());
	const unsigned merged = survivors + fresh;
	if (merged) VXB_CUDA(ctx, cudaMemcpyAsync(m->dir.p, m->scratch.p, sizeof(vxb_block_record) * merged, cudaMemcpyDeviceToDevice, st));
	VXB_CUDA(ctx, cudaEventRecord(m->ev[1], st));
	VXB_CUDA(ctx, cudaStreamSynchronize(st));

	// ---- the new state ----
	if (compact && grow) m->set[m->active].release(); // too small to take the next compaction
	if (compact || grow) ++m->info.generation;
	if (compact) ++m->info.compactions;
	if (grow && hadArenas) ++m->info.growths;
	m->active = target;
	const uint64_t elemBytes[4] = { sizeof(VxbVertex), 4, sizeof(VxbVertex), 4 };
	uint64_t copied = (uint64_t)merged * sizeof(vxb_block_record);
	for (int a = 0; a < 4; ++a)
	{
		const uint64_t moved = c.freshElems[a] + (compact ? c.survivorElems[a] : 0);
		copied += moved * elemBytes[a];
		m->cap[a] = newCap[a];
		m->span[a] = (compact || !region) ? live[a] : tail[a] + c.freshElems[a];
		m->total[a] = c.survivorRaw[a] + c.freshRaw[a];
	}
	vxb_mesh_info& i = m->info;
	i.levels = (uint32_t)levels;
	i.block_count = merged;
	for (int l = 0; l < 12; ++l) i.level_blocks[l] = c.survivors[l] + c.fresh[l];
	i.vertex_span = m->span[0]; i.index_span = m->span[1]; i.trans_vertex_span = m->span[2]; i.trans_index_span = m->span[3];
	i.vertex_total = m->total[0]; i.index_total = m->total[1]; i.trans_vertex_total = m->total[2]; i.trans_index_total = m->total[3];
	for (int a = 0; a < 4; ++a) i.capacity[a] = m->cap[a];
	memcpy(i.stats, ctx->info.stats, sizeof(i.stats));
	i.bytes_copied = copied;
	VXB_CUDA(ctx, cudaEventElapsedTime(&i.apply_ms, m->ev[0], m->ev[1]));
	m->bounds.boxes = reinterpret_cast<const float*>(m->boxes.p);
	for (int l = 0; l < VXB_MAX_LEVELS; ++l) m->bounds.level_base[l] = g.levelBase[l];
	m->bounds.slots = (uint32_t)slots;
	m->complete = ctx->resultComplete && (!region || m->complete);
	m->content = true;
	m->serial = ctx->runSerial;
	m->n = n;
	return VXB_OK;
}

int vxb_mesh_info_get(vxb_mesh* m, vxb_mesh_info* out)
{
	if (!m || !out) return VXB_ERR_ARGUMENT;
	*out = m->info;
	return VXB_OK;
}

int vxb_mesh_download(vxb_mesh* m, vxb_block_record* records, void* vertices, uint32_t* indices, void* transVertices, uint32_t* transIndices)
{
	if (!m) return VXB_ERR_ARGUMENT;
	vxb_context* ctx = m->ctx;
	cudaSetDevice(ctx->device);
	const vxb_mesh::Arenas& a = m->set[m->active];
	cudaStream_t st = ctx->stream;
	if (records && m->info.block_count) VXB_CUDA(ctx, cudaMemcpyAsync(records, m->dir.p, sizeof(vxb_block_record) * m->info.block_count, cudaMemcpyDeviceToHost, st));
	if (vertices && m->span[0]) VXB_CUDA(ctx, cudaMemcpyAsync(vertices, a.v.p, m->span[0] * sizeof(VxbVertex), cudaMemcpyDeviceToHost, st));
	if (indices && m->span[1]) VXB_CUDA(ctx, cudaMemcpyAsync(indices, a.i.p, m->span[1] * 4, cudaMemcpyDeviceToHost, st));
	if (transVertices && m->span[2]) VXB_CUDA(ctx, cudaMemcpyAsync(transVertices, a.tv.p, m->span[2] * sizeof(VxbVertex), cudaMemcpyDeviceToHost, st));
	if (transIndices && m->span[3]) VXB_CUDA(ctx, cudaMemcpyAsync(transIndices, a.ti.p, m->span[3] * 4, cudaMemcpyDeviceToHost, st));
	VXB_CUDA(ctx, cudaStreamSynchronize(st));
	return VXB_OK;
}

int vxb_mesh_device_arenas(vxb_mesh* m, const vxb_block_record** records, const void** vertices, const uint32_t** indices,
	const void** transVertices, const uint32_t** transIndices)
{
	if (!m) return VXB_ERR_ARGUMENT;
	const vxb_mesh::Arenas& a = m->set[m->active];
	if (records) *records = m->dir.p;
	if (vertices) *vertices = a.v.p;
	if (indices) *indices = a.i.p;
	if (transVertices) *transVertices = a.tv.p;
	if (transIndices) *transIndices = a.ti.p;
	return VXB_OK;
}

int vxb_mesh_select_lod(vxb_mesh* m, const float camera[3], float baseDistance, vxb_draw_lists* out)
{
	if (!m || !camera) return VXB_ERR_ARGUMENT;
	vxb_context* ctx = m->ctx;
	if (!m->content) return fail(ctx, VXB_ERR_STATE, "vxb_mesh_select_lod: nothing applied yet");
	cudaSetDevice(ctx->device);
	VxbDev d;
	memset(&d, 0, sizeof(d));
	d.n = (int)m->n; d.levels = (int)m->info.levels; d.lastLevel = d.levels - 1;
	d.records = m->dir.p;
	const int r = selectLod(ctx, d, m->info.block_count, m->dirCap, camera, baseDistance, m->drawCmd, m->drawInfo, m->drawTCmd, m->drawTInfo,
		m->drawCounts, m->drawLists);
	if (r != VXB_OK) return r;
	if (out) *out = m->drawLists;
	return VXB_OK;
}

int vxb_mesh_bounds_get(vxb_mesh* m, vxb_mesh_bounds* out)
{
	if (!m || !out) return VXB_ERR_ARGUMENT;
	if (!m->content) return fail(m->ctx, VXB_ERR_STATE, "vxb_mesh_bounds_get: nothing applied yet");
	*out = m->bounds;
	return VXB_OK;
}

int vxb_mesh_download_bounds(vxb_mesh* m, float* bounds)
{
	if (!m || !bounds) return VXB_ERR_ARGUMENT;
	vxb_context* ctx = m->ctx;
	if (!m->content) return fail(ctx, VXB_ERR_STATE, "vxb_mesh_download_bounds: nothing applied yet");
	cudaSetDevice(ctx->device);
	const unsigned blocks = m->info.block_count;
	if (!blocks) return VXB_OK;
	VXB_CUDA(ctx, m->boundsOut.ensure((size_t)blocks * 6));
	vxb_mesh_bounds_gather_kernel<<<(blocks + 255) / 256, 256, 0, ctx->stream>>>(m->dir.p, blocks, m->bounds, m->boundsOut.p);
	VXB_CUDA(ctx, cudaGetLastError());
	VXB_CUDA(ctx, cudaMemcpyAsync(bounds, m->boundsOut.p, sizeof(float) * 6 * blocks, cudaMemcpyDeviceToHost, ctx->stream));
	VXB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return VXB_OK;
}

int vxb_mesh_select_lod_views(vxb_mesh* m, const float camera[3], float baseDistance, const vxb_view* views, uint32_t viewCount,
	vxb_draw_lists* out)
{
	if (!m) return VXB_ERR_ARGUMENT;
	vxb_context* ctx = m->ctx;
	if (!camera || !views || !out) return fail(ctx, VXB_ERR_ARGUMENT, "vxb_mesh_select_lod_views: NULL lod_camera, views or out");
	if (viewCount == 0 || viewCount > VXB_VIEWS_MAX) return fail(ctx, VXB_ERR_ARGUMENT, "vxb_mesh_select_lod_views: view_count must be in [1, 8]");
	if (!m->content) return fail(ctx, VXB_ERR_STATE, "vxb_mesh_select_lod_views: nothing applied yet");
	return selectViews<VxbCentreCut>(m, "vxb_mesh_select_lod_views", camera, baseDistance, views, viewCount, m->viewLists, out);
}

int vxb_mesh_select_cut(vxb_mesh* m, const float camera[3], float lodFactor, const vxb_view* views, uint32_t viewCount, vxb_draw_lists* out)
{
	if (!m) return VXB_ERR_ARGUMENT;
	vxb_context* ctx = m->ctx;
	if (!camera || !views || !out) return fail(ctx, VXB_ERR_ARGUMENT, "vxb_mesh_select_cut: NULL lod_camera, views or out");
	if (viewCount == 0 || viewCount > VXB_VIEWS_MAX) return fail(ctx, VXB_ERR_ARGUMENT, "vxb_mesh_select_cut: view_count must be in [1, 8]");
	if (!std::isfinite(lodFactor) || !(lodFactor >= VXB_LOD_FACTOR_MIN))
		return fail(ctx, VXB_ERR_ARGUMENT, "vxb_mesh_select_cut: lod_factor must be finite and >= 2");
	if (!std::isfinite(camera[0]) || !std::isfinite(camera[1]) || !std::isfinite(camera[2]))
		return fail(ctx, VXB_ERR_ARGUMENT, "vxb_mesh_select_cut: non-finite lod_camera component");
	if (!m->content) return fail(ctx, VXB_ERR_STATE, "vxb_mesh_select_cut: nothing applied yet");
	if (!m->complete)
		return fail(ctx, VXB_ERR_STATE, "vxb_mesh_select_cut: the mesh lacks levels or transition meshes (a run since the last full "
			"apply had max_levels below the grid's levels or VXB_FLAG_NO_TRANSITIONS)");
	return selectViews<VxbBoxCut>(m, "vxb_mesh_select_cut", camera, lodFactor, views, viewCount, m->cutLists, out);
}

int vxb_mesh_raycast(vxb_mesh* m, const vxb_ray* rays, uint32_t count, vxb_ray_hit* hits)
{
	return meshQuery(m, { "vxb_mesh_raycast", !rays || !hits, "rays or hits", nullptr }, count,
		rule("ray", [=](uint32_t i) { return rayFault(rays[i]); }), [&] {
			return hostQuery(m, rays, sizeof(vxb_ray) * count, count, hits, [&](const vxb_ray* in, vxb_ray_hit* out) {
				return launchLevel0(m, vxb_raycast_kernel, VXB_RAY_THREADS, count, in, count, out); }); });
}

int vxb_mesh_raycast_device(vxb_mesh* m, const vxb_ray* rays, uint32_t count, vxb_ray_hit* hits)
{
	return meshQuery(m, { "vxb_mesh_raycast_device", !rays || !hits, "rays or hits", nullptr }, count, deviceRule,
		[&] { return launchLevel0(m, vxb_raycast_kernel, VXB_RAY_THREADS, count, rays, count, hits); });
}

int vxb_mesh_raycast_cut(vxb_mesh* m, const float camera[3], float lodFactor, const vxb_ray* rays, uint32_t count, vxb_cut_hit* hits)
{
	const char* what = "vxb_mesh_raycast_cut";
	return meshQuery(m, { what, !camera || !rays || !hits, "lod_camera, rays or hits", cutFault(camera, lodFactor), true }, count,
		rule("ray", [=](uint32_t i) { return rayFault(rays[i]); }), [&] {
			return hostQuery(m, rays, sizeof(vxb_ray) * count, count, hits, [&](const vxb_ray* in, vxb_cut_hit* out) {
				return enqueueRaycastCut(m, what, camera, lodFactor, in, count, out); }); });
}

int vxb_mesh_raycast_cut_device(vxb_mesh* m, const float camera[3], float lodFactor, const vxb_ray* rays, uint32_t count, vxb_cut_hit* hits)
{
	const char* what = "vxb_mesh_raycast_cut_device";
	return meshQuery(m, { what, !camera || !rays || !hits, "lod_camera, rays or hits", cutFault(camera, lodFactor), true }, count,
		deviceRule, [&] { return enqueueRaycastCut(m, what, camera, lodFactor, rays, count, hits); });
}

int vxb_mesh_sphere_cast(vxb_mesh* m, float radius, const vxb_ray* rays, uint32_t count, vxb_sphere_hit* hits)
{
	return meshQuery(m, { "vxb_mesh_sphere_cast", !rays || !hits, "rays or hits", radiusFault(radius) }, count,
		rule("sweep", [=](uint32_t i) { return rayFault(rays[i]); }), [&] {
			return hostQuery(m, rays, sizeof(vxb_ray) * count, count, hits, [&](const vxb_ray* in, vxb_sphere_hit* out) {
				return launchLevel0(m, vxb_sphere_cast_kernel, VXB_COLLIDE_THREADS, count, radius, in, count, out); }); });
}

int vxb_mesh_sphere_cast_device(vxb_mesh* m, float radius, const vxb_ray* rays, uint32_t count, vxb_sphere_hit* hits)
{
	return meshQuery(m, { "vxb_mesh_sphere_cast_device", !rays || !hits, "rays or hits", radiusFault(radius) }, count, deviceRule,
		[&] { return launchLevel0(m, vxb_sphere_cast_kernel, VXB_COLLIDE_THREADS, count, radius, rays, count, hits); });
}

int vxb_mesh_closest_point(vxb_mesh* m, float maxDistance, const float* points, uint32_t count, vxb_closest_hit* hits)
{
	return meshQuery(m, { "vxb_mesh_closest_point", !points || !hits, "points or hits", maxDistanceFault(maxDistance) }, count,
		rule("point", [=](uint32_t i) { return pointFault(points, i); }), [&] {
			return hostQuery(m, points, 3 * sizeof(float) * count, count, hits, [&](const float* in, vxb_closest_hit* out) {
				return launchLevel0(m, vxb_closest_point_kernel, VXB_COLLIDE_THREADS, count, maxDistance, in, count, out); }); });
}

int vxb_mesh_closest_point_device(vxb_mesh* m, float maxDistance, const float* points, uint32_t count, vxb_closest_hit* hits)
{
	return meshQuery(m, { "vxb_mesh_closest_point_device", !points || !hits, "points or hits", maxDistanceFault(maxDistance) }, count,
		deviceRule, [&] { return launchLevel0(m, vxb_closest_point_kernel, VXB_COLLIDE_THREADS, count, maxDistance, points, count, hits); });
}

int vxb_mesh_sphere_cast_cut(vxb_mesh* m, const float camera[3], float lodFactor, float radius, const vxb_ray* rays, uint32_t count,
	vxb_sphere_cut_hit* hits)
{
	const char* what = "vxb_mesh_sphere_cast_cut";
	return meshQuery(m, { what, !camera || !rays || !hits, "lod_camera, rays or hits", firstFault(cutFault(camera, lodFactor), radiusFault(radius)),
		true }, count, rule("sweep", [=](uint32_t i) { return rayFault(rays[i]); }), [&] {
			return hostQuery(m, rays, sizeof(vxb_ray) * count, count, hits, [&](const vxb_ray* in, vxb_sphere_cut_hit* out) {
				return enqueueSphereCastCut(m, what, camera, lodFactor, radius, in, count, out); }); });
}

int vxb_mesh_sphere_cast_cut_device(vxb_mesh* m, const float camera[3], float lodFactor, float radius, const vxb_ray* rays, uint32_t count,
	vxb_sphere_cut_hit* hits)
{
	const char* what = "vxb_mesh_sphere_cast_cut_device";
	return meshQuery(m, { what, !camera || !rays || !hits, "lod_camera, rays or hits", firstFault(cutFault(camera, lodFactor), radiusFault(radius)),
		true }, count, deviceRule, [&] { return enqueueSphereCastCut(m, what, camera, lodFactor, radius, rays, count, hits); });
}

int vxb_mesh_closest_point_cut(vxb_mesh* m, const float camera[3], float lodFactor, float maxDistance, const float* points, uint32_t count,
	vxb_closest_cut_hit* hits)
{
	const char* what = "vxb_mesh_closest_point_cut";
	return meshQuery(m, { what, !camera || !points || !hits, "lod_camera, points or hits",
		firstFault(cutFault(camera, lodFactor), maxDistanceFault(maxDistance)), true }, count,
		rule("point", [=](uint32_t i) { return pointFault(points, i); }), [&] {
			return hostQuery(m, points, 3 * sizeof(float) * count, count, hits, [&](const float* in, vxb_closest_cut_hit* out) {
				return enqueueClosestPointCut(m, what, camera, lodFactor, maxDistance, in, count, out); }); });
}

int vxb_mesh_closest_point_cut_device(vxb_mesh* m, const float camera[3], float lodFactor, float maxDistance, const float* points,
	uint32_t count, vxb_closest_cut_hit* hits)
{
	const char* what = "vxb_mesh_closest_point_cut_device";
	return meshQuery(m, { what, !camera || !points || !hits, "lod_camera, points or hits",
		firstFault(cutFault(camera, lodFactor), maxDistanceFault(maxDistance)), true }, count, deviceRule,
		[&] { return enqueueClosestPointCut(m, what, camera, lodFactor, maxDistance, points, count, hits); });
}

// the host variants' capsule rules (include/vxb200.h "capsule queries"): why the query is refused, or NULL
const char* sweepFault(const vxb_capsule_sweep& s)
{
	if (const char* why = rayFault(s.path)) return why;
	if (!(s.radius > 0.f)) return "radius must be > 0";
	if (!vxb_capsule_reach(make_float3(s.half_axis[0], s.half_axis[1], s.half_axis[2]), s.radius))
		return "non-finite half axis or radius, or max |half_axis| + radius above 15";
	return nullptr;
}
const char* segmentFault(const vxb_segment& s, float maxDistance)
{
	const float* c = s.center;
	const float* h = s.half_axis;
	if (!std::isfinite(c[0]) || !std::isfinite(c[1]) || !std::isfinite(c[2])) return "non-finite centre";
	if (!vxb_capsule_reach(make_float3(h[0], h[1], h[2]), maxDistance)) return "non-finite half axis, or max |half_axis| + max_distance above 15";
	return nullptr;
}

int vxb_mesh_capsule_cast(vxb_mesh* m, const vxb_capsule_sweep* sweeps, uint32_t count, vxb_capsule_hit* hits)
{
	return meshQuery(m, { "vxb_mesh_capsule_cast", !sweeps || !hits, "sweeps or hits", nullptr }, count,
		rule("sweep", [=](uint32_t i) { return sweepFault(sweeps[i]); }), [&] {
		return hostQuery(m, sweeps, sizeof(vxb_capsule_sweep) * count, count, hits, [&](const vxb_capsule_sweep* in, vxb_capsule_hit* out) {
			return launchLevel0(m, vxb_capsule_cast_kernel, VXB_COLLIDE_THREADS, count, in, count, out); }); });
}

int vxb_mesh_capsule_cast_device(vxb_mesh* m, const vxb_capsule_sweep* sweeps, uint32_t count, vxb_capsule_hit* hits)
{
	return meshQuery(m, { "vxb_mesh_capsule_cast_device", !sweeps || !hits, "sweeps or hits", nullptr }, count, deviceRule,
		[&] { return launchLevel0(m, vxb_capsule_cast_kernel, VXB_COLLIDE_THREADS, count, sweeps, count, hits); });
}

int vxb_mesh_closest_to_segment(vxb_mesh* m, float maxDistance, const vxb_segment* segments, uint32_t count, vxb_segment_hit* hits)
{
	return meshQuery(m, { "vxb_mesh_closest_to_segment", !segments || !hits, "segments or hits", maxDistanceFault(maxDistance) }, count,
		rule("segment", [=](uint32_t i) { return segmentFault(segments[i], maxDistance); }), [&] {
			return hostQuery(m, segments, sizeof(vxb_segment) * count, count, hits, [&](const vxb_segment* in, vxb_segment_hit* out) {
				return launchLevel0(m, vxb_closest_segment_kernel, VXB_COLLIDE_THREADS, count, maxDistance, in, count, out); }); });
}

int vxb_mesh_closest_to_segment_device(vxb_mesh* m, float maxDistance, const vxb_segment* segments, uint32_t count, vxb_segment_hit* hits)
{
	return meshQuery(m, { "vxb_mesh_closest_to_segment_device", !segments || !hits, "segments or hits", maxDistanceFault(maxDistance) },
		count, deviceRule,
		[&] { return launchLevel0(m, vxb_closest_segment_kernel, VXB_COLLIDE_THREADS, count, maxDistance, segments, count, hits); });
}

int vxb_mesh_capsule_cast_cut(vxb_mesh* m, const float camera[3], float lodFactor, const vxb_capsule_sweep* sweeps, uint32_t count,
	vxb_capsule_cut_hit* hits)
{
	const char* what = "vxb_mesh_capsule_cast_cut";
	return meshQuery(m, { what, !camera || !sweeps || !hits, "lod_camera, sweeps or hits", cutFault(camera, lodFactor), true }, count,
		rule("sweep", [=](uint32_t i) { return sweepFault(sweeps[i]); }), [&] {
			return hostQuery(m, sweeps, sizeof(vxb_capsule_sweep) * count, count, hits, [&](const vxb_capsule_sweep* in, vxb_capsule_cut_hit* out) {
				return enqueueCapsuleCastCut(m, what, camera, lodFactor, sweeps, in, count, out); }); });
}

int vxb_mesh_capsule_cast_cut_device(vxb_mesh* m, const float camera[3], float lodFactor, const vxb_capsule_sweep* sweeps, uint32_t count,
	vxb_capsule_cut_hit* hits)
{
	const char* what = "vxb_mesh_capsule_cast_cut_device";
	return meshQuery(m, { what, !camera || !sweeps || !hits, "lod_camera, sweeps or hits", cutFault(camera, lodFactor), true }, count,
		deviceRule, [&] { return enqueueCapsuleCastCut(m, what, camera, lodFactor, nullptr, sweeps, count, hits); });
}

int vxb_mesh_closest_to_segment_cut(vxb_mesh* m, const float camera[3], float lodFactor, float maxDistance, const vxb_segment* segments,
	uint32_t count, vxb_segment_cut_hit* hits)
{
	const char* what = "vxb_mesh_closest_to_segment_cut";
	return meshQuery(m, { what, !camera || !segments || !hits, "lod_camera, segments or hits",
		firstFault(cutFault(camera, lodFactor), maxDistanceFault(maxDistance)), true }, count,
		rule("segment", [=](uint32_t i) { return segmentFault(segments[i], maxDistance); }), [&] {
			return hostQuery(m, segments, sizeof(vxb_segment) * count, count, hits, [&](const vxb_segment* in, vxb_segment_cut_hit* out) {
				return enqueueClosestToSegmentCut(m, what, camera, lodFactor, maxDistance, segments, in, count, out); }); });
}

int vxb_mesh_closest_to_segment_cut_device(vxb_mesh* m, const float camera[3], float lodFactor, float maxDistance,
	const vxb_segment* segments, uint32_t count, vxb_segment_cut_hit* hits)
{
	const char* what = "vxb_mesh_closest_to_segment_cut_device";
	return meshQuery(m, { what, !camera || !segments || !hits, "lod_camera, segments or hits",
		firstFault(cutFault(camera, lodFactor), maxDistanceFault(maxDistance)), true }, count, deviceRule,
		[&] { return enqueueClosestToSegmentCut(m, what, camera, lodFactor, maxDistance, nullptr, segments, count, hits); });
}

// The host gather: count and scan, then the total decides the fill: the triangles are only written when they fit.
int vxb_mesh_overlap_box(vxb_mesh* m, const vxb_box* boxes, uint32_t count, uint64_t* offsets, vxb_overlap_triangle* tris, uint64_t capacity)
{
	const char* what = "vxb_mesh_overlap_box";
	return meshQuery(m, { what, !boxes || !offsets || (!tris && capacity), "boxes, offsets or tris", nullptr }, count,
		rule("box", [=](uint32_t i) { return vxb_box_valid(boxes[i]) ? nullptr : "non-finite component or min > max"; }), [&]() -> int {
		vxb_context* ctx = m->ctx;
		cudaStream_t st = ctx->stream;
		const uint64_t entries = (uint64_t)count + 1;
		if (sizeof(vxb_box) * count > m->stageIn.count || entries > m->overlapOffsets.count)
		{
			VXB_CUDA(ctx, cudaStreamSynchronize(st)); // nothing queued may still use the staging being replaced
			VXB_CUDA(ctx, m->stageIn.ensure(sizeof(vxb_box) * count)); VXB_CUDA(ctx, m->overlapOffsets.ensure(entries));
		}
		const vxb_box* in = (const vxb_box*)m->stageIn.p;
		VXB_CUDA(ctx, cudaMemcpyAsync(m->stageIn.p, boxes, sizeof(vxb_box) * count, cudaMemcpyHostToDevice, st));
		int r = enqueueOverlap(m, in, count, m->overlapOffsets.p, nullptr, 0);
		if (r != VXB_OK) return r;
		uint64_t total = 0;
		VXB_CUDA(ctx, cudaMemcpyAsync(&total, m->overlapOffsets.p + count, sizeof(total), cudaMemcpyDeviceToHost, st));
		VXB_CUDA(ctx, cudaStreamSynchronize(st));
		if (tris && total <= capacity && total)
		{
			const size_t bytes = sizeof(vxb_overlap_triangle) * total;
			if (bytes > m->stageOut.count) VXB_CUDA(ctx, m->stageOut.ensure(bytes)); // the stream is idle here
			VxbOverlapMesh om;
			r = overlapView(m, om);   // the map is built: this queues nothing
			if (r != VXB_OK) return r;
			vxb_overlap_kernel<true><<<queryCtas(ctx, count, VXB_OVERLAP_THREADS), VXB_OVERLAP_THREADS, 0, st>>>(om, in, count,
				m->overlapOffsets.p, (vxb_overlap_triangle*)m->stageOut.p, total);
			VXB_CUDA(ctx, cudaGetLastError());
			VXB_CUDA(ctx, cudaMemcpyAsync(tris, m->stageOut.p, bytes, cudaMemcpyDeviceToHost, st));
		}
		VXB_CUDA(ctx, cudaMemcpyAsync(offsets, m->overlapOffsets.p, sizeof(uint64_t) * entries, cudaMemcpyDeviceToHost, st));
		VXB_CUDA(ctx, cudaStreamSynchronize(st));
		if (tris && total > capacity)
		{
			char buf[192];
			snprintf(buf, sizeof(buf), "%s: %llu triangles exceed the capacity of %llu; offsets are written", what,
				(unsigned long long)total, (unsigned long long)capacity);
			return fail(ctx, VXB_ERR_CAPACITY, buf);
		}
		return VXB_OK;
	});
}

int vxb_mesh_overlap_box_device(vxb_mesh* m, const vxb_box* boxes, uint32_t count, uint64_t* offsets, vxb_overlap_triangle* tris, uint64_t capacity)
{
	return meshQuery(m, { "vxb_mesh_overlap_box_device", !boxes || !offsets || (!tris && capacity), "boxes, offsets or tris", nullptr },
		count, deviceRule, [&] { return enqueueOverlap(m, boxes, count, offsets, tris, capacity); });
}

} // extern "C"
