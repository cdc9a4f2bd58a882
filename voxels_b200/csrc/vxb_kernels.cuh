// sm_90a (H100) kernels of the Transvoxel polygonizer.  Included by vxb200.cu only.
//
// Pipeline per vxb_polygonize call (reference: TransVoxelRun::Execute, TransVoxelImpl.cpp:468-538):
//   vxb_scan_kernel          streams the level-0 distance volume ONCE (coalesced 16-byte loads) and
//                            reduces, per 16^3 block, sign/zero/lattice flags, the signs of its low faces + a
//                            run-count bound (VoxelGrid::CompressBlock's BF_Empty rule, VoxelGrid.cpp:610-672).
//   vxb_block_info_kernel    turns the raw flags into BF_Empty / sign-mix / low-face bits (exact slow path when
//                            the run-count bound is inconclusive).
//   vxb_select_kernel        per LOD level, the block walk (GenerateBlockListForLevel :385-466 + AreBlockAndNeighborsEmpty
//                            :1511-1527): appends the blocks that can produce output or side effects.
//   then the per-block and flat kernels of vxb_emit.cuh (PolygonizeBlock :1529-1750, GenerateTransitionCells :1754-2131,
//   PushBlocksToResult :1266-1428).  Launch order and costs: DESIGN.md §4.
#pragma once

#define VXB_MAX_LEVELS 12
#define VXB_THREADS 256
#define VXB_TILE_PITCH 32
#define VXB_TILE_BYTES (17 * 17 * VXB_TILE_PITCH)

// blockInfo bits (one word per level-0 block)
#define VXB_BI_NEG 1u
#define VXB_BI_NONNEG 2u
#define VXB_BI_EMPTY 4u
#define VXB_BI_NEG_E 8u      // level-1 lattice (even coordinates)
#define VXB_BI_NONNEG_E 16u
// low-face summaries: a (has a negative sample, has a non-negative one) bit pair at these shifts for the samples of the block
// with local coordinate 0 on the named axes - the planes x = 0, y = 0, z = 0 and the lines x = y = 0, x = z = 0, y = z = 0 -
// and the sign of the corner sample (0, 0, 0).  They are what the cells of the -x / -y / -z neighbours (and of the edge and
// corner neighbours) sample of this block.
#define VXB_BI_LOW_X 8
#define VXB_BI_LOW_Y 10
#define VXB_BI_LOW_Z 12
#define VXB_BI_LOW_XY 14
#define VXB_BI_LOW_XZ 16
#define VXB_BI_LOW_YZ 18
#define VXB_BI_CORNER_NEG (1u << 20)
// the same summaries in vxb_scan_kernel's flag word (its bits 8-19 hold the in-row change count): the six pairs at bits
// 20-31 (blockInfo's bits 8-19 shifted up by 12), the corner at bit 5
#define VXB_SF_LOW_SHIFT 12
#define VXB_SF_CORNER_NEG 32u

// (neg, nonneg) of the samples of a block with local coordinate 0 on the axes set in `axes` (bit 0 = x, 1 = y, 2 = z; not 0)
__device__ __forceinline__ unsigned vxb_bi_low(unsigned bi, int axes)
{
	if (axes == 7) return (bi & VXB_BI_CORNER_NEG) ? VXB_BI_NEG : VXB_BI_NONNEG;
	const int shift = axes == 1 ? VXB_BI_LOW_X : axes == 2 ? VXB_BI_LOW_Y : axes == 4 ? VXB_BI_LOW_Z
		: axes == 3 ? VXB_BI_LOW_XY : axes == 5 ? VXB_BI_LOW_XZ : VXB_BI_LOW_YZ;
	return (bi >> shift) & 3u;
}

struct VxbCounters
{
	unsigned int vertices, indices, transVertices, transIndices; // arena cursors (may exceed capacity = overflow)
	unsigned int records;
	unsigned int nonSkippedLevel0;
	unsigned int nonTrivial;
	unsigned int degenerate;
	unsigned int perCase[16];
	unsigned int usedMaterials[8];
	unsigned int workCount[VXB_MAX_LEVELS];
	unsigned int workCursor[VXB_MAX_LEVELS];
	unsigned int emitCount[VXB_MAX_LEVELS]; // emitted blocks (blocks with non-trivial cells), per level (vxb_block_kernel)
	unsigned int bigCount, bigCursor;       // bigList: blocks for vxb_big_block_kernel
	unsigned int cells;                     // cursor of the cell-record arena
	unsigned int splitVertices, splitCells; // cursors after level 0: the flat kernels work behind them
	unsigned int transBlocks, transCursor;  // emitted mid-level blocks (vxb_transition_kernel work list)
	unsigned int finishCursor;
	unsigned int coarseCursor;              // item cursor of the single launch that handles the coarse levels
};

// One non-trivial cell of an emitted block (written by vxb_block_kernel<1|2> and vxb_big_block_kernel, read by the flat kernels)
struct VxbCellRec
{
	unsigned int a; // cell id (0..4095) | case code << 12 | zero mask << 20 | reuse mask << 28
	unsigned int b; // material id | blend << 8 | owned-slot nibbles << 16
	unsigned int c; // new-vertex mask | v0-quirk mask << 12
	unsigned int d; // vertex base | triangle base << 16 (block local, serial cell order)
};

// One emitted block (slot = directory slot)
struct VxbBlockRec
{
	unsigned int packed;   // level << 28 | coordId
	unsigned int emitIdx;  // index into emitList / ntScratch
	unsigned int voff, ioff, cellBase, ntc, nverts, ntris, removed;
	unsigned int tvoff[6], tioff[6], tvcount[6], ticount[6];
	unsigned int pad[3];
};

struct VxbDev
{
	VxbGrid grid;
	int n, levels, lastLevel;
	unsigned int* scanFlags;
	unsigned int* blockInfo;                    // [nb0^3] VXB_BI_* (rank-major in sharded runs)
	unsigned int* consPages;                    // [nb0^3][128]
	unsigned char* consValid;                   // [nb0^3]
	unsigned short* cachePages[VXB_MAX_LEVELS]; // level l >= 1: [nb_l^3][4096] {id, blend}
	unsigned char* cacheValid[VXB_MAX_LEVELS];
	unsigned int* worklist;
	unsigned int workBase[VXB_MAX_LEVELS];
	unsigned int idBase[VXB_MAX_LEVELS];
	// incremental runs (GenerateBlockListForLevel, modification branch :429-465): per level a box of blocks and the
	// id of its first block; ids follow the z,y,x loop order of :456-464
	int incremental;
	int ranged; // block selection uses rangeMin/rangeMax (incremental runs and the slab of a sharded run)
	int rangeMin[VXB_MAX_LEVELS][3], rangeMax[VXB_MAX_LEVELS][3];
	unsigned int idStart[VXB_MAX_LEVELS];
	VxbVertex* verts; unsigned int* idx; VxbVertex* tverts; unsigned int* tidx;
	vxb_block_record* records;
	unsigned int vcap, icap, tvcap, ticap, rcap;
	VxbCounters* counters;
	const VxbMaterialLut* lut;
	int transitions;
	unsigned int* emitList;   // [workBase[l] + i] = level<<28 | coordId
	unsigned int* ntScratch;  // per emit-list entry: 128 words of non-trivial bits + 128 words of their exclusive prefix
	unsigned int* bigList;    // emit-list indices
	unsigned int* transList;  // block slots of emitted mid-level blocks
	VxbCellRec* cellRecs; unsigned int* cellBlock; unsigned int ccap;
	unsigned int* vlist;      // vertex (arena index) -> cell record index << 4 | table vertex
	uint2* tvlist;            // transition vertex (arena index) -> {block slot, face << 12 | cell << 4 | table vertex}
	VxbBlockRec* blockRecs;
	const unsigned char* lattice1; // (n/2)^3 even-lattice copy of the distance volume (level-1 samples), or null
	int computed;                  // levels [0, computed) are polygonized
	// sign-mix pyramid (vxb_pyramid_kernel): per block of level l >= 1, bit 0 = some covered level-0 block holds a negative
	// sample, bit 1 = a non-negative one.  Lets the block walk of levels >= 2 skip blocks that cannot have a non-trivial cell.
	unsigned char* mixInfo[VXB_MAX_LEVELS];
	unsigned short* mixCount[VXB_MAX_LEVELS];  // level-0 blocks with both signs under the block (saturating; exact up to level 5)
	// coarse levels (one launch, vxb_block_kernel<2>): levels [coarseLo, computed); a block waits for the done flags of its children
	int coarseLo;
	// their sample lattices: level l holds the samples at multiples of 2^l plus, per axis, one extra entry for the clamped
	// far-edge coordinate n (= the sample at n - 1, :1037-1047): (h + 1)^3 entries, h = n >> l, rows of h + 16 bytes.  Written by
	// vxb_coarse_lattice_kernel; a 17^3 tile of any coarse block is ONE TMA box of its level's map.
	unsigned char* coarseLattice[VXB_MAX_LEVELS];
	const CUtensorMap* coarseMaps;             // [VXB_MAX_LEVELS], device memory
	int latticeLo;                             // levels >= latticeLo have such a lattice (2; levels <= 1 read the volume / the even lattice)
	unsigned char* coarseDone;                 // [coarseBase[l] + coordId], zeroed per run
	unsigned int coarseBase[VXB_MAX_LEVELS];
	// sharded runs (vxb_shard_*): the z-axis is cut into groups of shardLayers level-0 block layers, dealt cyclically to
	// shardWorld ranks; blockInfo is stored rank-major (every rank's layers contiguous: the layout of the all-gather)
	int shardWorld, shardRank, shardLayers;
	// work ownership of a sharded run: blocks of levels <= sbLevel belong to the rank that owns their level-sbLevel ancestor
	// ("super-block"; sbMine[coordId at sbLevel] != 0 = mine, written by vxb_plan_kernel from the weights the pyramid kernel
	// counts); the coarse levels above are classified by every rank and emitted by rank (coordId + level) % world
	int sbLevel;
	unsigned char* sbMine;
	unsigned int* sbWeight;
};

__device__ __forceinline__ bool vxb_block_is_mine(const VxbDev& d, int level, int bx, int by, int bz)
{
	if (!d.shardWorld) return true;
	const int sh = d.sbLevel - level, nbs = (d.n >> 4) >> d.sbLevel;
	return d.sbMine[((size_t)(bz >> sh) * nbs + (by >> sh)) * nbs + (bx >> sh)] != 0;
}

__device__ __forceinline__ bool vxb_coarse_emit_is_mine(const VxbDev& d, int level, unsigned coordId)
{
	return !d.shardWorld || (int)((coordId + (unsigned)level) % (unsigned)d.shardWorld) == d.shardRank;
}

// layer z of the level-0 block grid -> its slot in blockInfo (identity unless the run is sharded)
__device__ __forceinline__ int vxb_layer_slot(const VxbDev& d, int z)
{
	if (!d.shardWorld) return z;
	const int g = z / d.shardLayers, owner = g % d.shardWorld, perRank = (d.n >> 4) / d.shardWorld;
	return owner * perRank + (g / d.shardWorld) * d.shardLayers + z % d.shardLayers;
}

__device__ __forceinline__ const unsigned int* vxb_binfo_row(const VxbDev& d, int y, int z)
{
	const int nb0 = d.n >> 4;
	return d.blockInfo + ((size_t)vxb_layer_slot(d, z) * nb0 + y) * nb0;
}

// ------------------------------------------------------------------------------------------------
// small PTX wrappers (mbarrier + TMA), sm_90a
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned vxb_smem_addr(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void vxb_mbar_init(unsigned long long* bar, unsigned count)
{
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(vxb_smem_addr(bar)), "r"(count));
	asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

__device__ __forceinline__ void vxb_mbar_expect_tx(unsigned long long* bar, unsigned bytes)
{
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(vxb_smem_addr(bar)), "r"(bytes) : "memory");
}

__device__ __forceinline__ void vxb_mbar_wait(unsigned long long* bar, unsigned parity)
{
	const unsigned addr = vxb_smem_addr(bar);
	unsigned done, spins = 0;
	do
	{
		asm volatile(
			"{\n"
			".reg .pred p;\n"
			"mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
			"selp.u32 %0, 1, 0, p;\n"
			"}\n" : "=r"(done) : "r"(addr), "r"(parity) : "memory");
		if (!done && ++spins > (1u << 26)) __trap(); // a TMA that never lands must fail the launch, not hang the GPU
	} while (!done);
}

// 3-D tiled TMA load global -> shared, completion on an mbarrier (SASS: UTMALDG)
__device__ __forceinline__ void vxb_tma_load_3d(void* dst, const CUtensorMap* map, int x, int y, int z, unsigned long long* bar)
{
	asm volatile(
		"cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
		::"r"(vxb_smem_addr(dst)), "l"(map), "r"(x), "r"(y), "r"(z), "r"(vxb_smem_addr(bar)) : "memory");
}

__device__ __forceinline__ void vxb_fence_proxy_async()
{
	asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// exclusive scan over the threads of the CTA (<= 256); every thread gets the grand total too
__device__ __forceinline__ unsigned vxb_block_scan(unsigned v, unsigned* warpSums /*[8]*/, unsigned& total)
{
	const int nwarps = (int)(blockDim.x >> 5);
	const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	unsigned inc = v;
#pragma unroll
	for (int o = 1; o < 32; o <<= 1)
	{
		const unsigned t = __shfl_up_sync(0xFFFFFFFFu, inc, o);
		if (lane >= (unsigned)o) inc += t;
	}
	__syncthreads(); // previous users of warpSums are done
	if (lane == 31) warpSums[warp] = inc;
	__syncthreads();
	unsigned base = 0, tot = 0;
#pragma unroll
	for (int w = 0; w < VXB_THREADS / 32; ++w)
	{
		if (w >= nwarps) break;
		const unsigned s = warpSums[w];
		if ((unsigned)w < warp) base += s;
		tot += s;
	}
	total = tot;
	return base + inc - v;
}

// ------------------------------------------------------------------------------------------------
// K1: scan - one pass over the level-0 distance volume
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned vxb_zero_bytes(unsigned w) // 0x80 in every byte of w that is zero (exact)
{
	return ~(((w & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | w) & 0x80808080u;
}

// J = x-adjacent blocks per CTA = lanes per row: a load instruction of a warp covers (32 / (32/J))... J * 16 contiguous
// bytes.  J = 32 (grids of >= 32 blocks per row): every warp-wide load is 512 contiguous bytes, which keeps DRAM pages open
// longer than the 128-byte pieces of J = 8 (small grids).
// the coarse levels' lattices (VxbDev::coarseLattice), as a scan-kernel argument
struct VxbCoarseLattices
{
	unsigned char* p[VXB_MAX_LEVELS];
	int lo, levels; // levels [lo, levels) have a lattice (lo >= 2)
};

// The coarse levels' lattices from the distance volume: one warp per lattice row (level, lz, ly) reads the source row
// (y = min(ly 2^l, n-1), z likewise) once, coalesced, and keeps every 2^l-th sample plus the clamped far-edge entry.
// Off the critical path of a single-GPU run (second stream, needed only by vxb_block_kernel<2>); sharded runs: every rank
// does the rows of its own planes (zOwnerWorld > 0) before publishing them.
__global__ void __launch_bounds__(256) vxb_coarse_lattice_kernel(const signed char* __restrict__ dist, int n, const __grid_constant__ VxbCoarseLattices lat,
	int planesPerPiece, int zOwnerWorld, int zOwnerRank)
{
	const int lane = threadIdx.x & 31;
	const unsigned warpsPerGrid = gridDim.x * (blockDim.x >> 5);
	unsigned w = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
	for (int l = lat.lo; l < lat.levels; ++l)
	{
		const int h = n >> l, pitch = h + 16, m = 1 << l;
		const unsigned rows = (unsigned)(h + 1) * (h + 1);
		for (; w < rows; w += warpsPerGrid)
		{
			const int lz = (int)(w / (h + 1)), ly = (int)(w % (h + 1));
			const int z = min(lz << l, n - 1), y = min(ly << l, n - 1);
			if (zOwnerWorld && (z / planesPerPiece) % zOwnerWorld != zOwnerRank) continue;
			const signed char* src = dist + ((size_t)z * n + y) * n;
			unsigned char* out = lat.p[l] + ((size_t)lz * (h + 1) + ly) * pitch;
			for (int lx = lane; lx <= h; lx += 32) out[lx] = (unsigned char)src[min(lx * m, n - 1)];
		}
		w -= rows; // continue with the next level's rows
	}
}

template <int J>
__global__ void __launch_bounds__(VXB_THREADS, (J == 32 ? 3 : 4)) vxb_scan_kernel(const signed char* __restrict__ dist, int n, unsigned int* __restrict__ scanFlags,
	unsigned char* __restrict__ lattice1 /* (n/2)^3: the samples at even coordinates = the level-1 lattice, or null */,
	int groupLayers, int world, int rank /* sharded runs: blockIdx.z counts this rank's layers (groups of groupLayers block layers,
	                                        dealt cyclically to the ranks); unsharded: world = 1 */,
	int zBase /* first block layer (incremental runs rescan only the layers of the level-0 dirty box) */)
{
	constexpr int RG = VXB_THREADS / J; // row groups: thread (j, rg) reads rows rg, rg + RG, ... of block j
	__shared__ unsigned sFlags[J];
	__shared__ unsigned sChanges[J];
	const int nb = n >> 4;
	const int bx0 = blockIdx.x * J, by = blockIdx.y;
	const int bz = zBase + ((int)(blockIdx.z / groupLayers) * world + rank) * groupLayers + (int)(blockIdx.z % groupLayers);
	const int tid = threadIdx.x;
	const int j = tid % J, rg = tid / J;
	if (tid < J) { sFlags[tid] = 0; sChanges[tid] = 0; }
	__syncthreads();

	unsigned neg = 0, pos = 0, zero = 0, negE = 0, nonnegE = 0, changes = 0;
	unsigned low = 0; // the low-face summaries, at their bits of the flag word (VXB_SF_*)
	if (bx0 + j < nb)
	{
		const uint4* src = reinterpret_cast<const uint4*>(dist + (((size_t)bz * 16) * n + (size_t)by * 16) * n + (size_t)(bx0 + j) * 16);
		const size_t ys = (size_t)n >> 4, zs = ys * n; // strides of y and z in 16-byte units
		// row q * RG + rg of the block: RG = 32: (y, z) = (rg & 15, 2q + (rg >> 4));  RG = 8: (y, z) = ((q & 1) * 8 + rg, q >> 1)
		const int y0 = (RG == 32) ? (rg & 15) : rg, z0 = (RG == 32) ? (rg >> 4) : 0;
		const uint4* p = src + (size_t)z0 * zs + (size_t)y0 * ys;
#pragma unroll 1
		for (int batch = 0; batch < J / 8; ++batch, p += (RG == 32 ? 16 : 4) * zs)
		{
			uint4 rows[8];
#pragma unroll
			for (int i = 0; i < 8; ++i)
				rows[i] = __ldg(p + ((RG == 32) ? (size_t)(2 * i) * zs : (size_t)(i >> 1) * zs + (size_t)((i & 1) * 8) * ys));
#pragma unroll
			for (int i = 0; i < 8; ++i)
			{
				const int y = (RG == 32) ? y0 : ((i & 1) * 8 + y0), z = (RG == 32) ? (z0 + 2 * i + batch * 16) : ((i >> 1) + batch * 4);
				const unsigned w[4] = { rows[i].x, rows[i].y, rows[i].z, rows[i].w };
				const bool even = !((y | z) & 1);
				// a row of 16 equal bytes (the common case away from the surface) has no value change inside it
				const unsigned splat = (w[0] & 0xFFu) * 0x01010101u;
				const bool flat = (w[0] == splat) & (w[1] == splat) & (w[2] == splat) & (w[3] == splat);
				if (even && lattice1)
				{
					// by-product: the even-x bytes of the even rows, so that level 1 can stage its tiles with TMA too
					const int h = n >> 1;
					uint2 e;
					e.x = __byte_perm(w[0], w[1], 0x6420);
					e.y = __byte_perm(w[2], w[3], 0x6420);
					*reinterpret_cast<uint2*>(lattice1 + (((size_t)(bz * 8 + (z >> 1))) * h + (by * 8 + (y >> 1))) * h + (size_t)(bx0 + j) * 8) = e;
				}
#pragma unroll
				for (int q = 0; q < 4; ++q)
				{
					const unsigned zb = vxb_zero_bytes(w[q]);
					neg |= w[q] & 0x80808080u;
					zero |= zb;
					pos |= ~w[q] & 0x80808080u & ~zb;
					if (even) { negE |= w[q] & 0x00800080u; nonnegE |= ~w[q] & 0x00800080u; }
				}
				{
					// low faces (zero counts as non-negative, as in the case code): byte 0 of every row is on the plane x = 0,
					// the rows with y = 0 / z = 0 are on those planes
					const unsigned s0 = (w[0] & 0x80u) ? VXB_BI_NEG : VXB_BI_NONNEG;
					const unsigned sr = (((w[0] | w[1] | w[2] | w[3]) & 0x80808080u) ? VXB_BI_NEG : 0u)
						| (((w[0] & w[1] & w[2] & w[3] & 0x80808080u) != 0x80808080u) ? VXB_BI_NONNEG : 0u);
					low |= s0 << (VXB_BI_LOW_X + VXB_SF_LOW_SHIFT);
					if (y == 0) low |= (sr << (VXB_BI_LOW_Y + VXB_SF_LOW_SHIFT)) | (s0 << (VXB_BI_LOW_XY + VXB_SF_LOW_SHIFT));
					if (z == 0) low |= (sr << (VXB_BI_LOW_Z + VXB_SF_LOW_SHIFT)) | (s0 << (VXB_BI_LOW_XZ + VXB_SF_LOW_SHIFT));
					if ((y | z) == 0) low |= (sr << (VXB_BI_LOW_YZ + VXB_SF_LOW_SHIFT)) | ((w[0] & 0x80u) ? VXB_SF_CORNER_NEG : 0u);
				}
				if (!flat)
				{
#pragma unroll
					for (int q = 0; q < 4; ++q)
					{
						// adjacent-byte changes inside the 16-byte row: compare byte k with byte k+1
						const unsigned nxt = (q < 3) ? w[q + 1] : (w[3] >> 24);
						const unsigned shifted = (w[q] >> 8) | (nxt << 24);
						const unsigned x = w[q] ^ shifted;
						unsigned diff = ((x & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | x; // bit 7 of each byte set iff byte != 0
						diff &= (q < 3) ? 0x80808080u : 0x00808080u;               // byte 15 has no right neighbour in the row
						changes += __popc(diff);
					}
				}
			}
		}
	}
	// bits 0-4: flags, 5 and 20-31: low faces; bits 8-19 take the in-row change count (<= 256 rows x 15 = 3840) below
	unsigned f = (neg ? 1u : 0u) | (pos ? 2u : 0u) | (zero ? 4u : 0u) | (negE ? 8u : 0u) | (nonnegE ? 16u : 0u) | low;
#pragma unroll
	for (int o = J; o < 32; o <<= 1) { f |= __shfl_xor_sync(0xFFFFFFFFu, f, o); changes += __shfl_xor_sync(0xFFFFFFFFu, changes, o); } // lanes of the same block
	if ((tid & 31) < J) { atomicOr(&sFlags[j], f); atomicAdd(&sChanges[j], changes); }
	__syncthreads();
	if (tid < J && bx0 + tid < nb)
		scanFlags[((size_t)bz * nb + by) * nb + bx0 + tid] = sFlags[tid] | (sChanges[tid] << 8);
}

// K1b: raw flags -> blockInfo.  One thread per level-0 block.
__global__ void vxb_block_info_kernel(const signed char* __restrict__ dist, int n, const unsigned int* __restrict__ scanFlags, unsigned int* __restrict__ blockInfo,
	size_t total /* blocks of this rank: whole layers, z-major */, int groupLayers, int world, int rank, int zBase /* as vxb_scan_kernel */)
{
	const int nb = n >> 4;
	const size_t layerBlocks = (size_t)nb * nb;
	for (size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x; q < total; q += (size_t)gridDim.x * blockDim.x)
	{
		// q = rank-local index (layer-major); b = the block's coordinate id; the result goes to the rank-major slot
		const int lz = (int)(q / layerBlocks);
		const int tz = zBase + ((lz / groupLayers) * world + rank) * groupLayers + lz % groupLayers;
		const size_t b = (size_t)tz * layerBlocks + q % layerBlocks;
		const unsigned f = scanFlags[b];
		const bool neg = f & 1, pos = f & 2, zero = f & 4;
		const unsigned changes = (f >> 8) & 0xFFFu; // value changes inside 16-byte rows (lower bound of run ends)
		bool empty = (neg != pos) && !zero; // every sample non-zero with one strict sign
		if (empty)
		{
			// CompressBlock stores the block raw (and never flags it empty) once 2048 run ends were seen.
			// runs <= changes + 255 (row seams) + 16 (255-length splits) + 1
			if (changes >= 2048u) empty = false;
			else if (changes + 272u >= 2049u)
			{
				// inconclusive: walk the block exactly (rare: strictly one-signed AND very noisy)
				const int bx = (int)(b % nb), by = (int)((b / nb) % nb), bz = (int)(b / ((size_t)nb * nb));
				unsigned counter = 0, runEnds = 0;
				int last = 0;
				for (int i = 0; i < 4096 && empty; ++i)
				{
					const int x = i & 15, y = (i >> 4) & 15, z = i >> 8;
					const int cur = dist[(((size_t)bz * 16 + z) * n + (size_t)by * 16 + y) * n + (size_t)bx * 16 + x];
					if (i == 0) last = cur;
					if (last == cur && counter < 0xFF) { ++counter; continue; }
					++runEnds; counter = 1; last = cur;
					if (1 + 2 * runEnds > 4096) empty = false;
				}
			}
		}
		blockInfo[world == 1 ? b : (size_t)rank * total + q] = (neg ? VXB_BI_NEG : 0u) | ((pos || zero) ? VXB_BI_NONNEG : 0u) | (empty ? VXB_BI_EMPTY : 0u)
			| ((f & 8) ? VXB_BI_NEG_E : 0u) | ((f & 16) ? VXB_BI_NONNEG_E : 0u)
			| ((f >> VXB_SF_LOW_SHIFT) & (0xFFFu << VXB_BI_LOW_X)) | ((f & VXB_SF_CORNER_NEG) ? VXB_BI_CORNER_NEG : 0u);
	}
}

// K1c: sign-mix pyramid over the level-0 blockInfo: mixInfo[l][b] = OR of (NEG, NONNEG) over the (2^l)^3 level-0 blocks that
// block b of level l covers; mixCount[l][b] = how many of them hold both signs (the weight of a super-block in sharded runs).
// vxb_pyramid_kernel: levels 1 and 2 straight from blockInfo, one thread per block (8 / 64 word reads).
// vxb_pyramid_top_kernel: levels >= 3 from their eight children, level by level, in ONE CTA (<= 4681 blocks in total).
__global__ void __launch_bounds__(256) vxb_pyramid_kernel(const VxbDev d)
{
	const int nb0 = d.n >> 4;
	unsigned q = blockIdx.x * 256u + threadIdx.x;
	int level = 0;
	for (int l = 1; l <= 2 && l < d.levels; ++l)
	{
		const unsigned cnt = (unsigned)(nb0 >> l) * (nb0 >> l) * (nb0 >> l);
		if (q < cnt) { level = l; break; }
		q -= cnt;
	}
	if (!level) return;
	const int nb = nb0 >> level, span = 1 << level;
	const int bx = q % nb, by = (q / nb) % nb, bz = q / (nb * nb);
	unsigned u = 0, mixed = 0;
	for (int z = 0; z < span; ++z) for (int y = 0; y < span; ++y)
	{
		const unsigned int* row = vxb_binfo_row(d, by * span + y, bz * span + z) + bx * span;
		for (int x = 0; x < span; ++x) { u |= row[x]; mixed += (row[x] & 3u) == 3u; }
	}
	d.mixInfo[level][q] = (unsigned char)(u & 3u);
	d.mixCount[level][q] = (unsigned short)mixed;
	if (d.sbWeight && level == d.sbLevel) d.sbWeight[q] = mixed;
}

__global__ void __launch_bounds__(1024) vxb_pyramid_top_kernel(const VxbDev d)
{
	const int nb0 = d.n >> 4;
	for (int level = 3; level < d.levels; ++level)
	{
		const int nb = nb0 >> level, cnb = nb * 2;
		const unsigned cnt = (unsigned)nb * nb * nb;
		for (unsigned q = threadIdx.x; q < cnt; q += 1024u)
		{
			const int bx = q % nb, by = (q / nb) % nb, bz = q / (nb * nb);
			unsigned u = 0, mixed = 0;
			for (int c = 0; c < 8; ++c)
			{
				const size_t cb = ((size_t)(bz * 2 + (c >> 2)) * cnb + (by * 2 + ((c >> 1) & 1))) * cnb + (bx * 2 + (c & 1));
				u |= d.mixInfo[level - 1][cb];
				mixed += d.mixCount[level - 1][cb];
			}
			d.mixInfo[level][q] = (unsigned char)(u & 3u);
			d.mixCount[level][q] = (unsigned short)min(mixed, 65535u);
			if (d.sbWeight && level == d.sbLevel) d.sbWeight[q] = mixed;
		}
		__syncthreads(); // the next level reads what this one wrote (same CTA: visible after the barrier)
	}
}

// Upload helper: 16^3 blocks (VoxelGrid block order) -> dense volume.  One CTA per block, 256 threads x 16 bytes.
__global__ void __launch_bounds__(VXB_THREADS) vxb_unpack_blocks_kernel(const uint4* __restrict__ blocks, unsigned char* __restrict__ dense, int n)
{
	const int nb = n >> 4;
	const size_t b = blockIdx.x;
	const int bx = (int)(b % nb), by = (int)((b / nb) % nb), bz = (int)(b / ((size_t)nb * nb));
	const int row = threadIdx.x, y = row & 15, z = row >> 4;
	const uint4 v = blocks[b * 256 + row];
	*reinterpret_cast<uint4*>(dense + (((size_t)bz * 16 + z) * n + (size_t)by * 16 + y) * n + (size_t)bx * 16) = v;
}

// Incremental grid update: a list of 16^3 blocks -> their places in the dense volume
__global__ void __launch_bounds__(VXB_THREADS) vxb_unpack_block_list_kernel(const uint4* __restrict__ blocks, const unsigned int* __restrict__ coords,
	unsigned char* __restrict__ dense, int n)
{
	const size_t b = blockIdx.x;
	const int bx = (int)coords[b * 3], by = (int)coords[b * 3 + 1], bz = (int)coords[b * 3 + 2];
	const int row = threadIdx.x, y = row & 15, z = row >> 4;
	*reinterpret_cast<uint4*>(dense + (((size_t)bz * 16 + z) * n + (size_t)by * 16 + y) * n + (size_t)bx * 16) = blocks[b * 256 + row];
}

// Upload helper: run-length decoding of the packed 16^3 blocks (VoxelGrid::DecompressBlock, VoxelGrid.cpp:674-694; block
// layout of PackForSave :304-312).  One CTA per 8 x-adjacent blocks: most channels of most blocks are a single value (17
// runs of <= 255), those are written as full 128-byte lines (8 lanes x 16 bytes, the layout of vxb_scan_kernel's reads);
// the others are decoded by the whole CTA, thread t producing row t by a binary search of the run covering its first byte.
__device__ __forceinline__ void vxb_decode_channel(const unsigned char* src, unsigned size, bool raw, unsigned char* out, int n, int bx, int by, int bz,
	unsigned short* start, unsigned char* value, unsigned* warpSums, unsigned int* error)
{
	const int tid = threadIdx.x, y = tid & 15, z = tid >> 4;
	uint4 row;
	unsigned char* rb = reinterpret_cast<unsigned char*>(&row);
	if (raw) // BF_*Uncompressed (VoxelGrid.h:70-79): 4096 raw bytes
	{
		for (int i = 0; i < 16; ++i) rb[i] = src[tid * 16 + i];
	}
	else
	{
		const unsigned runs = min(size >> 1, 2048u);
		const unsigned per = (runs + VXB_THREADS - 1) / VXB_THREADS;
		const unsigned r0 = min(tid * per, runs), r1 = min(r0 + per, runs);
		unsigned sum = 0;
		for (unsigned r = r0; r < r1; ++r) sum += src[2 * r];
		unsigned total;
		unsigned base = vxb_block_scan(sum, warpSums, total);
		for (unsigned r = r0; r < r1; ++r) { start[r] = (unsigned short)min(base, 4096u); value[r] = src[2 * r + 1]; base += src[2 * r]; }
		if (tid == 0) { start[runs] = 4096; if (total != 4096u) *error = 1u; } // the runs of a block cover exactly its 4096 voxels (:674-694)
		__syncthreads();
		const unsigned p0 = tid * 16;
		unsigned lo = 0, hi = runs; // last run with start <= p0
		while (hi - lo > 1) { const unsigned mid = (lo + hi) >> 1; if (start[mid] <= p0) lo = mid; else hi = mid; }
		unsigned r = lo;
		for (int i = 0; i < 16; ++i)
		{
			while (r + 1 < runs && start[r + 1] <= p0 + i) ++r;
			rb[i] = value[r];
		}
		__syncthreads();
	}
	*reinterpret_cast<uint4*>(out + (((size_t)bz * 16 + z) * n + (size_t)by * 16 + y) * n + (size_t)bx * 16) = row;
}

__global__ void __launch_bounds__(VXB_THREADS) vxb_unpack_rle_kernel(const unsigned char* __restrict__ blob, const unsigned long long* __restrict__ blockOffsets,
	const unsigned int* __restrict__ sizes, unsigned char* __restrict__ dist, unsigned char* __restrict__ mat, unsigned char* __restrict__ blend, int n,
	int zLayer0 /* first block layer of this launch: the blob is decoded in z-chunks while the rest is still being copied */,
	unsigned int* __restrict__ error /* set when a block's flags word contradicts its sizes; such a channel is zero-filled */)
{
	__shared__ unsigned short start[2049];
	__shared__ unsigned char value[2048];
	__shared__ unsigned warpSums[8];
	__shared__ unsigned long long sOff[8][3];  // byte offset of the channel's data in the blob
	__shared__ unsigned sSize[8][3];
	__shared__ int sKind[8][3];                // >= 0: every run has this value; -1: run-length coded; -2: raw
	const int nb = n >> 4;
	const int groups = (nb + 7) >> 3;          // CTAs per row of blocks
	const int bx0 = (int)(blockIdx.x % groups) * 8, by = (int)((blockIdx.x / groups) % nb), bz = (int)(blockIdx.x / ((size_t)groups * nb)) + zLayer0;
	const int tid = threadIdx.x;
	if (tid < 24)
	{
		const int j = tid / 3, ch = tid % 3;
		int kind = -1;
		if (bx0 + j < nb)
		{
			const size_t b = ((size_t)bz * nb + by) * nb + bx0 + j;
			const unsigned char* src = blob + blockOffsets[b];
			const unsigned flags = src[0] | (src[1] << 8) | (src[2] << 16) | ((unsigned)src[3] << 24);
			unsigned long long off = blockOffsets[b] + 4;
			for (int c = 0; c < ch; ++c) off += sizes[b * 3 + c];
			const unsigned size = sizes[b * 3 + ch];
			sOff[j][ch] = off; sSize[j][ch] = size;
			if ((flags >> (1 + ch)) & 1u)
			{
				if (size == 4096u) kind = -2;
				else { kind = 0; *error = 1u; } // a raw channel holds exactly 4096 bytes: never read past what the table says
			}
			else if (size == 0u || (size & 1u)) { kind = 0; *error = 1u; } // whole (length, value) pairs
			else
			{
				const unsigned char* p = blob + off;
				const unsigned runs = size >> 1;
				bool same = runs >= 1 && runs <= 64;
				unsigned covered = same ? p[0] : 0u;
				for (unsigned r = 1; r < runs && same; ++r) { same = p[2 * r + 1] == p[1]; covered += p[2 * r]; }
				if (same) { kind = p[1]; if (covered != 4096u) *error = 1u; }
			}
		}
		sKind[j][ch] = kind;
	}
	__syncthreads();
	unsigned char* const outs[3] = { dist, mat, blend };
	{
		// single-valued channels: lane group j writes block j's 16 bytes of each row => full 128-byte lines
		const int j = tid & 7, rg = tid >> 3;
		if (bx0 + j < nb)
#pragma unroll
			for (int ch = 0; ch < 3; ++ch)
			{
				const int kind = sKind[j][ch];
				if (kind < 0) continue;
				const unsigned v4 = (unsigned)kind * 0x01010101u;
				const uint4 row = make_uint4(v4, v4, v4, v4);
#pragma unroll
				for (int i = 0; i < 8; ++i)
				{
					const int r = i * 32 + rg, y = r & 15, z = r >> 4;
					*reinterpret_cast<uint4*>(outs[ch] + (((size_t)bz * 16 + z) * n + (size_t)by * 16 + y) * n + (size_t)(bx0 + j) * 16) = row;
				}
			}
	}
	for (int e = 0; e < 24; ++e) // block-uniform loop over the channels that need real decoding
	{
		const int j = e / 3, ch = e % 3;
		if (bx0 + j >= nb || sKind[j][ch] >= 0) continue;
		vxb_decode_channel(blob + sOff[j][ch], sSize[j][ch], sKind[j][ch] == -2, outs[ch], n, bx0 + j, by, bz, start, value, warpSums, error);
	}
}

// ------------------------------------------------------------------------------------------------
// K2: block selection for one level
// ------------------------------------------------------------------------------------------------
// Levels >= 2: can block (bx, by, bz) have a non-trivial cell or a vote to cast?  Its cells sample the closed box
// [origin, origin + 16 m], i.e. the level-(l-1) blocks 2b .. 2b+2 per axis (superset: the whole +2 block instead of its first
// plane); without a sign mix there no cell is non-trivial, and without a child page no vote can succeed (:763-837), so the
// block leaves no trace in the result, the caches or the statistics (BlocksCalculated / TrivialCells count every block).
__device__ __forceinline__ bool vxb_coarse_block_needed(const VxbDev& d, int level, int bx, int by, int bz)
{
	const int cnb = (d.n >> 4) >> (level - 1);
	const unsigned char* mix = d.mixInfo[level - 1];
	const unsigned char* valid = d.cacheValid[level - 1];
	unsigned u = 0, anyChild = 0;
	for (int z = 0; z < 3; ++z) for (int y = 0; y < 3; ++y) for (int x = 0; x < 3; ++x)
	{
		const int cx = min(2 * bx + x, cnb - 1), cy = min(2 * by + y, cnb - 1), cz = min(2 * bz + z, cnb - 1);
		const size_t cb = ((size_t)cz * cnb + cy) * cnb + cx;
		u |= mix[cb];
		if (x < 2 && y < 2 && z < 2) anyChild |= __ldcg(valid + cb);
	}
	return u == 3u || anyChild != 0u;
}

__global__ void vxb_select_kernel(VxbDev d, int level)
{
	const int m = 1 << level, nb = d.n / 16 / m, nb0 = d.n / 16;
	// full run: every block of the level; incremental run: the dirty box of the level; sharded run: the rank's slab
	const int x0 = d.ranged ? d.rangeMin[level][0] : 0, y0 = d.ranged ? d.rangeMin[level][1] : 0, z0 = d.ranged ? d.rangeMin[level][2] : 0;
	const int nx = d.ranged ? d.rangeMax[level][0] - x0 : nb, ny = d.ranged ? d.rangeMax[level][1] - y0 : nb, nz = d.ranged ? d.rangeMax[level][2] - z0 : nb;
	const unsigned total = (nx > 0 && ny > 0 && nz > 0) ? (unsigned)nx * ny * nz : 0u;
	for (unsigned base = blockIdx.x * blockDim.x; base < total; base += gridDim.x * blockDim.x)
	{
		const unsigned q = base + threadIdx.x;
		unsigned b = 0;
		bool take = false, counted = false;
		if (q < total)
		{
			const int bx = x0 + (int)(q % nx), by = y0 + (int)((q / nx) % ny), bz = z0 + (int)(q / ((unsigned)nx * ny));
			b = ((unsigned)bz * nb + by) * nb + bx;
			if (!vxb_block_is_mine(d, level, bx, by, bz)) { /* another rank's block */ }
			else if (level == 0)
			{
				// AreBlockAndNeighborsEmpty :1511-1527
				bool skip = true;
				for (int z = -1; z < 2 && skip; ++z) for (int y = -1; y < 2 && skip; ++y) for (int x = -1; x < 2; ++x)
				{
					const int cx = min(max(bx + x, 0), nb - 1), cy = min(max(by + y, 0), nb - 1), cz = min(max(bz + z, 0), nb - 1);
					if (!(vxb_binfo_row(d, cy, cz)[cx] & VXB_BI_EMPTY)) { skip = false; break; }
				}
				if (!skip)
				{
					counted = true;
					// Exact test: the cells of this block sample the 17^3 points [0, 16]^3 - the block itself, the low plane of
					// its +x / +y / +z neighbours, the low line of its three edge neighbours and the low corner of the +xyz one
					// (a neighbour beyond the far grid edge adds nothing: its samples clamp onto points already counted).  Those points form
					// a connected lattice whose every edge is an edge of one of the block's cells, so when they hold both signs
					// some edge joins a negative sample to a non-negative one and its cell is non-trivial; without both signs
					// no cell is.  A block that fails the test has no non-trivial cell and vxb_block_kernel<0> would write
					// nothing for it: no page, no statistics, no histogram.
					const bool hx = bx + 1 < nb, hy = by + 1 < nb, hz = bz + 1 < nb;
					const unsigned* r00 = vxb_binfo_row(d, by, bz);
					unsigned u = r00[bx] & 3u;
					if (hx) u |= vxb_bi_low(r00[bx + 1], 1);
					if (hy)
					{
						const unsigned* r10 = vxb_binfo_row(d, by + 1, bz);
						u |= vxb_bi_low(r10[bx], 2);
						if (hx) u |= vxb_bi_low(r10[bx + 1], 3);
					}
					if (hz)
					{
						const unsigned* r01 = vxb_binfo_row(d, by, bz + 1);
						u |= vxb_bi_low(r01[bx], 4);
						if (hx) u |= vxb_bi_low(r01[bx + 1], 5);
						if (hy)
						{
							const unsigned* r11 = vxb_binfo_row(d, by + 1, bz + 1);
							u |= vxb_bi_low(r11[bx], 6);
							if (hx) u |= vxb_bi_low(r11[bx + 1], 7);
						}
					}
					take = u == (VXB_BI_NEG | VXB_BI_NONNEG);
				}
			}
			else if (level == 1)
			{
				// sign mix (superset) of the block's samples: the even lattice of the eight covered level-0 blocks, and of
				// the +2 level-0 neighbours the samples at their local coordinate 0 on the +2 axes - the low plane, line or
				// corner summary, which covers all of them.  Blocks on the far grid edge sample the clamped coordinate n-1,
				// which is off the lattice: there every block of the neighbourhood adds its whole sign flags.
				unsigned u = 0; bool anyChild = false;
				const bool edge = (bx == nb - 1) || (by == nb - 1) || (bz == nb - 1);
#pragma unroll
				for (int z = 0; z < 3; ++z)
#pragma unroll
					for (int y = 0; y < 3; ++y)
#pragma unroll
						for (int x = 0; x < 3; ++x)
						{
							const int cx = min(2 * bx + x, nb0 - 1), cy = min(2 * by + y, nb0 - 1), cz = min(2 * bz + z, nb0 - 1);
							const size_t cb = ((size_t)cz * nb0 + cy) * nb0 + cx;
							const unsigned bi = vxb_binfo_row(d, cy, cz)[cx];
							const int far = (x == 2 ? 1 : 0) | (y == 2 ? 2 : 0) | (z == 2 ? 4 : 0);
							u |= far ? vxb_bi_low(bi, far) : (bi >> 3) & 3u;
							if (edge) u |= bi & 3u;
							if (!far && d.consValid[cb]) anyChild = true;
						}
				take = (u == 3u) || anyChild;
			}
			else take = vxb_coarse_block_needed(d, level, bx, by, bz);
		}
		const unsigned ballot = __ballot_sync(0xFFFFFFFFu, take);
		const unsigned cballot = __ballot_sync(0xFFFFFFFFu, counted);
		const unsigned lane = threadIdx.x & 31;
		unsigned off = 0;
		if (lane == 0)
		{
			if (ballot) off = atomicAdd(&d.counters->workCount[level], __popc(ballot));
			if (cballot) atomicAdd(&d.counters->nonSkippedLevel0, __popc(cballot));
		}
		off = __shfl_sync(0xFFFFFFFFu, off, 0);
		if (take) d.worklist[d.workBase[level] + off + __popc(ballot & ((1u << lane) - 1u))] = b;
	}
}

// Sharded runs: which super-blocks are mine.  Every rank runs this on the same (all-gathered) blockInfo, so all ranks
// agree: super-blocks in coordinate order, cut where the running weight (level-0 blocks with a sign mix) crosses
// total * r / world.  One CTA of 1024 threads; <= 32768 super-blocks.
__global__ void __launch_bounds__(1024) vxb_plan_kernel(const VxbDev d)
{
	__shared__ unsigned long long sums[32];
	__shared__ unsigned long long sTotal;
	const int nbs = (d.n >> 4) >> d.sbLevel;
	const unsigned count = (unsigned)nbs * nbs * nbs;   // a power of 8: a multiple of 4
	const unsigned per = ((count + 1023u) / 1024u + 3u) & ~3u;
	const unsigned i0 = min(threadIdx.x * per, count), i1 = min(i0 + per, count);
	// the chunk's weights in registers (independent 16-byte loads), used twice
	uint4 w[8];
	unsigned long long mine = 0;
#pragma unroll
	for (int q = 0; q < 8; ++q)
	{
		const unsigned i = i0 + 4u * q;
		w[q] = (i < i1 && (unsigned)q * 4u < per) ? *reinterpret_cast<const uint4*>(d.sbWeight + i) : make_uint4(0, 0, 0, 0);
	}
#pragma unroll
	for (int q = 0; q < 8; ++q)
	{
		const unsigned i = i0 + 4u * q;
		if (i < i1) mine += ((unsigned long long)w[q].x + w[q].y + w[q].z + w[q].w) * 1024ull + 4ull; // + 1 each: a super-block without a mixed block still costs a look
	}
	unsigned long long inc = mine;
	const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	for (int o = 1; o < 32; o <<= 1) { const unsigned long long t = __shfl_up_sync(0xFFFFFFFFu, inc, o); if (lane >= (unsigned)o) inc += t; }
	if (lane == 31) sums[warp] = inc;
	__syncthreads();
	if (threadIdx.x == 0)
	{
		unsigned long long acc = 0;
		for (int k = 0; k < 32; ++k) { const unsigned long long v = sums[k]; sums[k] = acc; acc += v; }
		sTotal = acc;
	}
	__syncthreads();
	unsigned long long run = sums[warp] + inc - mine; // exclusive prefix of this thread's chunk
	const unsigned long long total = sTotal;
	// owner = floor(run * world / total) = the number of r in [1, world) with run >= ceil(r * total / world): my range is
	// [lo, hi) without a division per super-block
	const unsigned long long W = (unsigned long long)d.shardWorld, r = (unsigned long long)d.shardRank;
	const unsigned long long lo = (r * total + W - 1) / W, hi = (r + 1 == W) ? ~0ull : ((r + 1) * total + W - 1) / W;
#pragma unroll
	for (int q = 0; q < 8; ++q)
	{
		const unsigned i = i0 + 4u * q;
		if (i >= i1) continue;
		const unsigned ws[4] = { w[q].x, w[q].y, w[q].z, w[q].w };
		unsigned packed = 0;
#pragma unroll
		for (int k = 0; k < 4; ++k)
		{
			if (run >= lo && run < hi) packed |= 1u << (8 * k);
			run += (unsigned long long)ws[k] * 1024ull + 1ull;
		}
		*reinterpret_cast<unsigned*>(d.sbMine + i) = packed;
	}
}

// Sharded runs: the material pages of level sbLevel that this rank produced go to every peer (plain 16-byte stores
// through the peers' mapped buffers: NVLink), so that every rank can classify the coarse levels above.
struct VxbPeers
{
	unsigned short* pages[8];
	unsigned char* valid[8];
	int count;
	// the barrier that orders every rank's coarse levels after every rank's page stores: a slot per source rank in each
	// rank's (peer-mapped) buffer; the LAST CTA of the publishing kernel - it has seen every other CTA's fenced stores -
	// writes this step's epoch into slot [myRank] of every peer, vxb_peer_wait_kernel waits for the peers' epochs
	unsigned long long* peerSlots[8];  // peers' slot arrays (remote)
	unsigned long long* mySlots;       // [8] local: written by the peers
	unsigned long long* epoch;         // local step counter
	unsigned int* arrived;             // local CTA counter of the publishing kernel
	int rank;
};

// Sharded runs: the planes of the coarse levels' lattices this rank wrote while scanning its pieces go to every peer
// (the lattices live in the buffer the peers map; byte offsets are the same on every rank).
struct VxbPeerLattices
{
	unsigned char* base[8];    // the peers' lattice areas
	int count;
};

__global__ void __launch_bounds__(VXB_THREADS) vxb_publish_lattice_kernel(const VxbDev d, const VxbPeerLattices peers, unsigned char* myBase)
{
	const int planesPerPiece = d.shardLayers * 16;
	for (int l = d.coarseLo; l < d.levels; ++l)
	{
		const int h = d.n >> l, pitch = h + 16;
		const size_t planeBytes = (size_t)pitch * (h + 1);
		for (int lz = blockIdx.x; lz <= h; lz += gridDim.x)
		{
			const int z = min(lz << l, d.n - 1);
			if ((z / planesPerPiece) % d.shardWorld != d.shardRank) continue;
			const uint4* src = reinterpret_cast<const uint4*>(d.coarseLattice[l] + planeBytes * lz);
			const size_t off = (size_t)(d.coarseLattice[l] - myBase) + planeBytes * lz;
			for (size_t i = threadIdx.x; i < planeBytes / 16; i += VXB_THREADS)
			{
				const uint4 v = src[i];
				for (int p = 0; p < peers.count; ++p) reinterpret_cast<uint4*>(peers.base[p] + off)[i] = v;
			}
		}
	}
}

__global__ void __launch_bounds__(VXB_THREADS) vxb_publish_kernel(const VxbDev d, const VxbPeers peers)
{
	__shared__ unsigned sLast;
	const int nbs = (d.n >> 4) >> d.sbLevel;
	const unsigned count = (unsigned)nbs * nbs * nbs;
	for (unsigned b = blockIdx.x; b < count; b += gridDim.x)
	{
		if (!d.sbMine[b] || !d.cacheValid[d.sbLevel][b]) continue;
		const uint4* src = reinterpret_cast<const uint4*>(d.cachePages[d.sbLevel] + (size_t)b * 4096);
		const uint4 v0 = src[threadIdx.x], v1 = src[threadIdx.x + VXB_THREADS];
		for (int p = 0; p < peers.count; ++p)
		{
			uint4* dst = reinterpret_cast<uint4*>(peers.pages[p] + (size_t)b * 4096);
			dst[threadIdx.x] = v0; dst[threadIdx.x + VXB_THREADS] = v1;
			if (threadIdx.x == 0) peers.valid[p][b] = 1;
		}
	}
	// signal: every thread's stores are fenced system-wide before its CTA counts itself in; the last CTA to arrive has
	// therefore observed all of them and announces this step's epoch to the peers
	__threadfence_system();
	__syncthreads();
	if (threadIdx.x == 0) sLast = (atomicAdd(peers.arrived, 1u) == gridDim.x - 1) ? 1u : 0u;
	__syncthreads();
	if (sLast && threadIdx.x < (unsigned)peers.count)
	{
		__threadfence_system();
		const unsigned long long e = *peers.epoch + 1ull;
		*(volatile unsigned long long*)(peers.peerSlots[threadIdx.x] + peers.rank) = e;
	}
	if (sLast)
	{
		__syncthreads();
		if (threadIdx.x == 0) { *peers.epoch += 1ull; *peers.arrived = 0u; __threadfence(); }
	}
}

// waits until every peer has announced the current epoch (vxb_publish_kernel): one lane per peer slot
__global__ void vxb_peer_wait_kernel(const VxbPeers peers, const int world)
{
	const int p = threadIdx.x;
	if (p >= world || p == peers.rank) return;
	const unsigned long long e = *(volatile unsigned long long*)peers.epoch; // already advanced by this rank's publishing kernel
	const volatile unsigned long long* slot = peers.mySlots + p;
	unsigned spins = 0;
	while (*slot < e) { __nanosleep(100); if (++spins > (1u << 26)) __trap(); } // a peer that never arrives must fail the step, not hang it
	__threadfence_system();
}

// ------------------------------------------------------------------------------------------------
// K3: polygonize
// ------------------------------------------------------------------------------------------------
// 17^3 sample tile of block (bx,by,bz) at `level` -> smem: level 0 by one 3-D TMA load (issued early by thread 0, so
// it can be in flight while the CTA still works on the previous block), coarser levels by a clamped strided gather.
// level 0 reads the distance volume itself, level 1 (away from the far grid edge, where the reference clamps to the odd
// coordinate n-1) reads the even-lattice copy written by vxb_scan_kernel; both through the same 32x17x17 TMA box
__device__ __forceinline__ bool vxb_tile_uses_tma(const VxbDev& d, int level, int bx, int by, int bz)
{
	if (level == 0) return true;
	if (level >= d.latticeLo) return true; // the level's own lattice (far-edge entries included)
	if (level != 1 || !d.lattice1) return false;
	const int nb = d.n / 32;
	return bx != nb - 1 && by != nb - 1 && bz != nb - 1;
}

__device__ __forceinline__ void vxb_tile_issue(signed char* tile, unsigned long long* mbar, const CUtensorMap* tmap0, const CUtensorMap* tmap1,
	const VxbDev& d, int level, int bx, int by, int bz)
{
	if (threadIdx.x == 0 && vxb_tile_uses_tma(d, level, bx, by, bz))
	{
		vxb_fence_proxy_async();
		vxb_mbar_expect_tx(mbar, VXB_TILE_BYTES);
		vxb_tma_load_3d(tile, level == 0 ? tmap0 : (level >= d.latticeLo ? d.coarseMaps + level : tmap1), bx * 16, by * 16, bz * 16, mbar);
	}
}

__device__ __forceinline__ void vxb_tile_complete(signed char* tile, unsigned long long* mbar, unsigned& phase,
	const VxbDev& d, int level, int bx, int by, int bz)
{
	const int tid = threadIdx.x;
	const int n = d.n, m = 1 << level, nb = n / 16 / m;
	if (vxb_tile_uses_tma(d, level, bx, by, bz))
	{
		vxb_mbar_wait(mbar, phase);
		phase ^= 1;
		if (level >= d.latticeLo) return; // lattice tiles need no fix-up
		// level 0, far grid edge: the +1 plane is outside the volume (TMA zero-fills); the reference clamps (:1037-1047)
		if (bx == nb - 1) { __syncthreads(); for (int i = tid; i < 17 * 17; i += (int)blockDim.x) tile[i * VXB_TILE_PITCH + 16] = tile[i * VXB_TILE_PITCH + 15]; }
		if (by == nb - 1) { __syncthreads(); for (int i = tid; i < 17 * 17; i += (int)blockDim.x) { const int z = i / 17, x = i % 17; tile[(z * 17 + 16) * VXB_TILE_PITCH + x] = tile[(z * 17 + 15) * VXB_TILE_PITCH + x]; } }
		if (bz == nb - 1) { __syncthreads(); for (int i = tid; i < 17 * 17; i += (int)blockDim.x) { const int y = i / 17, x = i % 17; tile[(16 * 17 + y) * VXB_TILE_PITCH + x] = tile[(15 * 17 + y) * VXB_TILE_PITCH + x]; } }
	}
	else
	{
		const int lim = n - 1;
		const signed char* dist = d.grid.dist;
		for (int i = tid; i < 17 * 17 * 17; i += (int)blockDim.x)
		{
			const int x = i % 17, y = (i / 17) % 17, z = i / 289;
			const int gx = min((bx * 16 + x) * m, lim), gy = min((by * 16 + y) * m, lim), gz = min((bz * 16 + z) * m, lim);
			tile[(z * 17 + y) * VXB_TILE_PITCH + x] = dist[((size_t)gz * n + gy) * n + gx];
		}
	}
}

struct VxbVoteSource // what a vote at `level` reads: the child level's validity flags + pages (+ level-0 materials)
{
	const unsigned char* valid;  // consValid (level 1) / cacheValid[level - 1]
	const void* pages;           // consPages (level 1) / cachePages[level - 1]
	const unsigned char* mat;
	const unsigned char* blend;
	int n, level;
};

__device__ __forceinline__ VxbVoteSource vxb_vote_source(const VxbDev& d, int level)
{
	VxbVoteSource v;
	v.valid = (level == 1) ? d.consValid : d.cacheValid[level - 1];
	v.pages = (level == 1) ? (const void*)d.consPages : (const void*)d.cachePages[level - 1];
	v.mat = d.grid.mat; v.blend = d.grid.blend; v.n = d.n; v.level = level;
	return v;
}

// Could the vote of this cell succeed?  The first tests of vxb_vote_cell as independent loads (no early exit, no call), so
// that a caller can have the loads of several cells in flight at once.  Pages of blocks that were never written are
// readable (the page space is reserved for every block) and are masked by the valid flag.
__device__ __forceinline__ bool vxb_vote_candidate(const VxbVoteSource& d, const int bx0, const int by0, const int bz0)
{
	const int sh = d.level - 1, cnb = (d.n / 16) >> sh;
	const int cx = bx0 >> sh, cy = by0 >> sh, cz = bz0 >> sh;
	const size_t bid = ((size_t)(cz >> 4) * cnb + (cy >> 4)) * cnb + (cx >> 4);
	const int lx = cx & 15, ly = cy & 15, lz = cz & 15;
	const unsigned valid = __ldcg(d.valid + bid); // L2: a flag byte shares its line with blocks other CTAs of this launch finish (coarse levels)
	if (d.level == 1)
	{
		const unsigned short* rows = reinterpret_cast<const unsigned short*>(static_cast<const unsigned int*>(d.pages) + bid * 128);
		const unsigned r = (unsigned)rows[lz * 16 + ly] | rows[lz * 16 + ly + 1] | rows[(lz + 1) * 16 + ly] | rows[(lz + 1) * 16 + ly + 1];
		return valid != 0u && ((r >> lx) & 3u) != 0u;
	}
	const unsigned int* page = reinterpret_cast<const unsigned int*>(static_cast<const unsigned short*>(d.pages) + bid * 4096);
	const int o = (lz * 256 + ly * 16 + lx) >> 1;
	const unsigned all = page[o] & page[o + 8] & page[o + 128] & page[o + 136];
	return valid != 0u && (all & 0x00FF00FFu) != 0x00FF00FFu;
}

// returns id | blend << 8, or -1 when no child carries a material (results in a register: reference outputs would go
// through local memory).  Inlined: as a call, the callee-saved registers of vxb_block_kernel<1> went to the stack around
// every vote.
__device__ __forceinline__ int vxb_vote_cell(const VxbVoteSource d, const int bx0, const int by0, const int bz0)
{
	const int level = d.level;
	const int base[3] = { bx0, by0, bz0 };
	const int cm = (1 << level) >> 1, cnb = d.n / 16 / cm;
	const int cx = base[0] / cm, cy = base[1] / cm, cz = base[2] / cm;            // child-level cell coordinates (even)
	const size_t bid = ((size_t)(cz >> 4) * cnb + (cy >> 4)) * cnb + (cx >> 4);
	const int lx = cx & 15, ly = cy & 15, lz = cz & 15;
	unsigned cid[8], cbl[8]; // children, x fastest (:773-775); fully unrolled below so they live in registers
	if (level == 1)
	{
		if (!__ldcg(d.valid + bid)) return -1;
		const unsigned short* rows = reinterpret_cast<const unsigned short*>(static_cast<const unsigned int*>(d.pages) + bid * 128); // 16 bits per (z,y) row
		const unsigned r00 = (rows[lz * 16 + ly] >> lx) & 3u, r01 = (rows[lz * 16 + ly + 1] >> lx) & 3u;
		const unsigned r10 = (rows[(lz + 1) * 16 + ly] >> lx) & 3u, r11 = (rows[(lz + 1) * 16 + ly + 1] >> lx) & 3u;
		const unsigned bits = r00 | (r01 << 2) | (r10 << 4) | (r11 << 6); // child q = x + 2y + 4z
		if (!bits) return -1;
#pragma unroll
		for (int q = 0; q < 8; ++q)
		{
			cid[q] = VXB_EMPTY_MATERIAL; cbl[q] = 0;
			if ((bits >> q) & 1u)
			{
				const size_t gi = ((size_t)(base[2] + (q >> 2)) * d.n + (base[1] + ((q >> 1) & 1))) * d.n + (base[0] + (q & 1));
				cid[q] = d.mat[gi]; cbl[q] = d.blend[gi];
			}
		}
	}
	else
	{
		if (!__ldcg(d.valid + bid)) return -1;
		const unsigned int* page = reinterpret_cast<const unsigned int*>(static_cast<const unsigned short*>(d.pages) + bid * 4096); // 2 cells per word
		const int o = (lz * 256 + ly * 16 + lx) >> 1;
		const unsigned e0 = page[o], e1 = page[o + 8], e2 = page[o + 128], e3 = page[o + 136];
		if ((e0 & e1 & e2 & e3 & 0x00FF00FFu) == 0x00FF00FFu) return -1; // all eight children EMPTY_MATERIAL
		cid[0] = e0 & 0xFF; cbl[0] = (e0 >> 8) & 0xFF; cid[1] = (e0 >> 16) & 0xFF; cbl[1] = e0 >> 24;
		cid[2] = e1 & 0xFF; cbl[2] = (e1 >> 8) & 0xFF; cid[3] = (e1 >> 16) & 0xFF; cbl[3] = e1 >> 24;
		cid[4] = e2 & 0xFF; cbl[4] = (e2 >> 8) & 0xFF; cid[5] = (e2 >> 16) & 0xFF; cbl[5] = e2 >> 24;
		cid[6] = e3 & 0xFF; cbl[6] = (e3 >> 8) & 0xFF; cid[7] = (e3 >> 16) & 0xFF; cbl[7] = e3 >> 24;
	}
	// majority vote (:812-834) without the candidate arrays: candidate = first occurrence of an id, in order of first
	// appearance; a later candidate wins only with a strictly larger count (std::max_element keeps the first maximum)
	int bestCount = 0; unsigned bestId = 0, bestBlend = 0;
#pragma unroll
	for (int q = 0; q < 8; ++q)
	{
		bool first = cid[q] != VXB_EMPTY_MATERIAL;
#pragma unroll
		for (int p = 0; p < q; ++p) first = first && (cid[p] != cid[q]);
		int cnt = 0; unsigned bsum = 0;
#pragma unroll
		for (int p = q; p < 8; ++p) if (cid[p] == cid[q]) { ++cnt; bsum += cbl[p]; }
		if (first && cnt > bestCount) { bestCount = cnt; bestId = cid[q]; bestBlend = bsum; }
	}
	if (!bestCount) return -1;
	return (int)(bestId | (((bestBlend / (unsigned)bestCount) & 0xFFu) << 8));
}

// Block id as the reference assigns it: full run = running counter over levels in z,y,x order (:395-401);
// incremental run = continuation of that counter over the level's dirty box (:456-464)
__device__ __forceinline__ unsigned vxb_block_id(const VxbDev& d, int level, unsigned coordId)
{
	if (!d.incremental) return d.idBase[level] + coordId;
	const int nb = d.n / 16 >> level;
	const int bx = coordId % nb, by = (coordId / nb) % nb, bz = coordId / (nb * nb);
	const int nx = d.rangeMax[level][0] - d.rangeMin[level][0], ny = d.rangeMax[level][1] - d.rangeMin[level][1];
	return d.idStart[level] + (unsigned)(((bz - d.rangeMin[level][2]) * ny + (by - d.rangeMin[level][1])) * nx + (bx - d.rangeMin[level][0]));
}

__device__ __forceinline__ void vxb_store_vertex(VxbVertex* dst, const VxbVertex& v)
{
	const uint4* src = reinterpret_cast<const uint4*>(&v);
	uint4* out = reinterpret_cast<uint4*>(dst);
	out[0] = src[0]; out[1] = src[1]; out[2] = src[2];
}

