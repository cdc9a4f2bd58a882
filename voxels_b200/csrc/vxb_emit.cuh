// Per-block and flat kernels of the polygonizer (included by vxb200.cu after vxb_kernels.cuh).
//
//   vxb_block_kernel<0|1|2> one pass per block: tile -> non-trivial cells, consistency page or material votes, statistics,
//                           then the decide passes (vxb_decide_cells) and the arena reservation.  Level 0 makes the block's
//                           vertices and triangles itself; levels >= 1 write cell records + the vertex work list.
//   vxb_big_block_kernel    the decide passes of the blocks too large for the shared-memory path of vxb_block_kernel.
//   vxb_vertex_kernel, vxb_triangle_kernel   flat, one thread per new vertex / per cell of the blocks with cell records.
//   vxb_transition_kernel   per face of an emitted mid-level block: the transition cells (:1754-2131).
//   vxb_finish_kernel       per emitted block: order-preserving compaction where triangles were removed + directory.
//
// Launch order, occupancy and costs: DESIGN.md §4.  Bit-exactness notes are in vxb_kernels.cuh / vxb_cell.h.
#pragma once
#ifndef VXB_OCC
#define VXB_OCC 4 // resident CTAs per SM the per-block kernels are compiled for (register cap 65536 / (256 * VXB_OCC))
#endif
#ifndef VXB_FLAT_OCC
#define VXB_FLAT_OCC 4 // same for the flat per-vertex kernels
#endif

// Non-trivial bits of all 4096 cells from the tile, 16 cells per thread-step instead of one:
// a cell is non-trivial iff its 8 corner signs are neither all 0 nor all 1 (Cell::CalcCaseCode :741-750, :1560).
// `tile` points at sample (0,0,0) of the block; rows are PITCH bytes apart, z-slices ROWS rows.
template <int PITCH, int ROWS>
__device__ __forceinline__ void vxb_classify_bits(const signed char* tile, unsigned int* rowSign, unsigned int* nt32)
{
	const int tid = threadIdx.x, nthreads = (int)blockDim.x;
	for (int r = tid; r < 17 * 17; r += nthreads)
	{
		const unsigned int* w = reinterpret_cast<const unsigned int*>(tile + ((r / 17) * ROWS + (r % 17)) * PITCH);
		unsigned m = 0;
#pragma unroll
		for (int q = 0; q < 4; ++q) m |= ((((w[q] >> 7) & 0x01010101u) * 0x01020408u) >> 24 & 0xFu) << (4 * q);
		m |= ((w[4] >> 7) & 1u) << 16;
		rowSign[r] = m;
	}
	__syncthreads();
	for (int t = tid; t < 256; t += nthreads)
	{
		const int z = t >> 4, y = t & 15;
		const unsigned a = rowSign[z * 17 + y], b = rowSign[z * 17 + y + 1], c = rowSign[(z + 1) * 17 + y], e = rowSign[(z + 1) * 17 + y + 1];
		const unsigned any = a | b | c | e, all = a & b & c & e;
		reinterpret_cast<unsigned short*>(nt32)[t] = (unsigned short)((any | (any >> 1)) & ~(all & (all >> 1)) & 0xFFFFu);
	}
}

template <int PITCH, int ROWS>
__device__ __forceinline__ void vxb_tile_samples(const signed char* tile, int c, signed char v[8])
{
	const int lx = c & 15, ly = (c >> 4) & 15, lz = c >> 8;
	const signed char* p = tile + (lz * ROWS + ly) * PITCH + lx;
	v[0] = p[0]; v[1] = p[1]; v[2] = p[PITCH]; v[3] = p[PITCH + 1];
	p += ROWS * PITCH;
	v[4] = p[0]; v[5] = p[1]; v[6] = p[PITCH]; v[7] = p[PITCH + 1];
}

__device__ __forceinline__ void vxb_init_cache_page(const VxbDev& d, int level, unsigned coordId)
{
	unsigned int* page = reinterpret_cast<unsigned int*>(d.cachePages[level] + (size_t)coordId * 4096);
	for (int i = threadIdx.x; i < 2048; i += (int)blockDim.x) page[i] = 0x00FF00FFu; // {EMPTY_MATERIAL, 0} x 2  (:424)
}

__device__ __forceinline__ unsigned vxb_rank_of(const unsigned int* nt32, const unsigned int* wpre, int c)
{
	return wpre[c >> 5] + __popc(nt32[c >> 5] & ((1u << (c & 31)) - 1u));
}

// Level-0 halo tile (vxb_block_kernel<0>): the block's distance neighbourhood, coordinates [origin - 1, origin + 17] per
// axis, as 19 x 19 rows of 48 bytes (the TMA box starts on a 16-byte boundary one 16-byte group before the block).
#define VXB_DTILE_PITCH 48
#define VXB_DTILE_BYTES (19 * 19 * VXB_DTILE_PITCH)
// Capacities of the shared-memory path of vxb_block_kernel<0|1|2>: non-trivial cells of a block (larger blocks go to
// vxb_big_block_kernel) and new vertices of a level-0 block generated inside the CTA (more => the flat kernels).
template <int MODE> struct VxbBlockCaps { static constexpr int CAP = 1024, VL = (MODE == 0 ? 2048 : 8), NBUF = (MODE == 0 ? 1 : 2); }; // level 0: one tile buffer => 4 CTAs per SM

// ------------------------------------------------------------------------------------------------
// vxb_block_kernel<0|1|2>: everything that needs the block as a unit, in ONE pass over its sample tile
//   tile -> case codes -> non-trivial bits; consistency page (level 0) or majority votes of the non-trivial cells and of
//   every transition-face cell into the level's material page (CalculateMaterialForCellCache :753-838, called from :1568
//   and :1859) - the only cross-level dependency; statistics; then, for blocks with non-trivial cells: ordered compaction,
//   materials, owned reuse slots, new-vs-reuse decisions, block scans -> vertex / triangle bases, arena reservation.
//   Three kernels, one body each (<0> level 0, <1> one level below the coarse ones, <2> all coarse levels), over the
//   shared phases below.
// ------------------------------------------------------------------------------------------------
template <int MODE>
struct __align__(128) VxbBlockSmem
{
	typedef VxbBlockCaps<MODE> Caps;
	signed char tiles[Caps::NBUF][MODE == 0 ? (VXB_DTILE_BYTES + 80) : (VXB_TILE_BYTES + 96)]; // NBUF = 2: the next block's tile lands while this one is worked on
	unsigned int rowSign[17 * 17 + 3]; // bit x = sample (x, y, z) of the tile is negative
	unsigned int nt32[128];
	unsigned int wpre[132];
	unsigned char tabClass[256];
	unsigned char tabCell[256];
	unsigned short tabVert[3072];
	unsigned int warpSums[8];
	unsigned int hist[16];
	unsigned int used[8];
	unsigned long long mbar[2];
	unsigned int item, ahead, hasChild, pageReady, emitIdx, voff, ioff, cellBase, slot, take, removed;
	unsigned int levelEnd[VXB_MAX_LEVELS + 1];
	unsigned int recA[Caps::CAP];     // matId | matBlend<<8 | slotK<<16
	unsigned int recB[Caps::CAP];     // newMask | quirkMask<<12 | reuse mask << 24
	unsigned short list[Caps::CAP];   // compact index -> cell id
	unsigned short cz[Caps::CAP];     // case code | zero mask << 8
	unsigned short vbase[Caps::CAP];  // exclusive scan of new-vertex counts
	unsigned short tbase[Caps::CAP];  // exclusive scan of triangle counts
	unsigned short vl[Caps::VL];      // MODE 0: block-local vertex -> compact cell index << 4 | table vertex
};

// true when an arena overflowed: the host grows the arenas and repeats the run, the later kernels do nothing
__device__ __forceinline__ bool vxb_overflowed(const VxbDev& d)
{
	const VxbCounters* c = d.counters;
	return c->vertices > d.vcap || c->indices > d.icap || c->cells > d.ccap || c->records > d.rcap;
}

// ---- the steps both per-block kernels (vxb_block_kernel, vxb_big_block_kernel) take over a block's non-trivial cells;
// their shared memory has the arrays nt32, wpre, list, cz, recA, recB, vbase, tbase, the three tables and warpSums ----

// ordered compact list of the non-trivial cells: thread = cell row (z, y), 16 bits each (VXB_THREADS = 256 rows)
__device__ __forceinline__ void vxb_compact_cells(const unsigned int* nt32, const unsigned int* wpre, unsigned short* list)
{
	const int r = threadIdx.x;
	unsigned bits = reinterpret_cast<const unsigned short*>(nt32)[r];
	unsigned pos = wpre[r >> 1] + ((r & 1) ? __popc(nt32[r >> 1] & 0xFFFFu) : 0u);
	while (bits) { const int x = __ffs(bits) - 1; bits &= bits - 1; list[pos++] = (unsigned short)(r * 16 + x); }
}

// The decide passes over the ntc cells of the compact list: pass A, pass B and the block scans; nverts / ntris = the block's
// totals.  HIST: pass A takes the level-0 case histogram (PerCaseCellsCount :1574) into s.hist.  Ends without a barrier.
template <int PITCH, int ROWS, bool HIST, class Smem>
__device__ __forceinline__ void vxb_decide_cells(Smem& s, const signed char* tile, const VxbDev& d, int level, unsigned coordId,
	int bx, int by, int bz, unsigned ntc, unsigned& nverts, unsigned& ntris)
{
	const int tid = threadIdx.x;
	const VxbGrid g = d.grid;
	// ---- pass A: material, case code, zero mask, owned slots ----
	for (unsigned i = tid; i < ntc; i += VXB_THREADS)
	{
		const int c = s.list[i];
		signed char v[8];
		vxb_tile_samples<PITCH, ROWS>(tile, c, v);
		const unsigned code = vxb_case_code(v);
		const unsigned zm = vxb_zero_mask(v);
		unsigned matId, matBlend;
		if (level == 0)
		{
			if constexpr (HIST) atomicAdd(&s.hist[s.tabClass[code]], 1u);
			const size_t gi = ((size_t)((bz * 16 + (c >> 8))) * d.n + (by * 16 + ((c >> 4) & 15))) * d.n + (bx * 16 + (c & 15));
			matId = g.mat[gi]; matBlend = g.blend[gi];
		}
		else
		{
			const unsigned e = d.cachePages[level][(size_t)coordId * 4096 + c]; // the vote of vxb_block_kernel
			matId = e & 0xFF; matBlend = e >> 8;
		}
		unsigned slotK = 0xFFFFu;
		const int nv = s.tabCell[s.tabClass[code] * 16] >> 4;
		for (int k = 0; k < nv; ++k)
		{
			const VxbVertexDesc vd = vxb_regular_vertex_desc_lite(s.tabVert[code * 12 + k], zm);
			const int sl = vxb_regular_owned_slot(vd);
			if (sl >= 0) slotK = (slotK & ~(0xFu << (4 * sl))) | ((unsigned)k << (4 * sl));
		}
		s.cz[i] = (unsigned short)(code | (zm << 8));
		s.recA[i] = matId | (matBlend << 8) | (slotK << 16);
	}
	__syncthreads();

	// ---- pass B: new-vs-reuse decisions ----
	for (unsigned i = tid; i < ntc; i += VXB_THREADS)
	{
		const int c = s.list[i];
		const unsigned code = s.cz[i] & 0xFF, zm = s.cz[i] >> 8;
		const unsigned geo = s.tabCell[s.tabClass[code] * 16];
		const unsigned rowStart = vxb_rank_of(s.nt32, s.wpre, c & ~15), sliceStart = s.wpre[(c >> 8) * 8];
		const int mask = (i > rowStart ? 1 : 0) | (rowStart > sliceStart ? 2 : 0) | (sliceStart > 0 ? 4 : 0);
		const unsigned myMat = s.recA[i] & 0xFF;
		unsigned newMask = 0, quirkMask = 0;
		for (int k = 0; k < (int)(geo >> 4); ++k)
		{
			// new-vs-reuse decision (:1610-1644) from the owner cell's record
			const VxbVertexDesc vd = vxb_regular_vertex_desc_lite(s.tabVert[code * 12 + k], zm);
			bool isNew = true;
			if (!vd.atC7 && (vd.dir & mask) == vd.dir) // dir == 8 never passes: mask < 8
			{
				const int oc = c - (vd.dir & 1) - ((vd.dir >> 1) & 1) * 16 - ((vd.dir >> 2) & 1) * 256;
				int ok = VXB_NO_SLOT; unsigned oa = 0;
				if ((s.nt32[oc >> 5] >> (oc & 31)) & 1u)
				{
					oa = s.recA[vxb_rank_of(s.nt32, s.wpre, oc)];
					ok = (oa >> (16 + 4 * vd.slot)) & 0xF;
				}
				if (ok != VXB_NO_SLOT) { if ((oa & 0xFF) == myMat) isNew = false; } // else: material split, new at its natural place
				else if (vd.endpoint) quirkMask |= 1u << k;                            // :1633-1640 creates the vertex at v0
			}
			if (isNew) newMask |= 1u << k;
		}
		s.recB[i] = newMask | (quirkMask << 12) | ((unsigned)mask << 24);
		s.vbase[i] = (unsigned short)__popc(newMask);
		s.tbase[i] = (unsigned short)(geo & 0xF);
	}
	__syncthreads();

	// ---- exclusive scans in serial cell order (contiguous chunk per thread) ----
	const unsigned per = (ntc + VXB_THREADS - 1) / VXB_THREADS;
	const unsigned i0 = min(tid * per, ntc), i1 = min(i0 + per, ntc);
	unsigned sv = 0, st = 0;
	for (unsigned i = i0; i < i1; ++i) { sv += s.vbase[i]; st += s.tbase[i]; }
	unsigned total;
	const unsigned base = vxb_block_scan(sv | (st << 16), s.warpSums, total);
	nverts = total & 0xFFFF; ntris = total >> 16;
	unsigned bv = base & 0xFFFF, bt = base >> 16;
	for (unsigned i = i0; i < i1; ++i)
	{
		const unsigned cv = s.vbase[i], ct = s.tbase[i];
		s.vbase[i] = (unsigned short)bv; s.tbase[i] = (unsigned short)bt;
		bv += cv; bt += ct;
	}
}

// the block's non-trivial bits and their prefix, read back by vxb_big_block_kernel and vxb_triangle_kernel
__device__ __forceinline__ void vxb_save_nt(const VxbDev& d, unsigned emitIdx, const unsigned int* nt32, const unsigned int* wpre)
{
	const int tid = threadIdx.x;
	if (tid < 128) { d.ntScratch[(size_t)emitIdx * 256 + tid] = nt32[tid]; d.ntScratch[(size_t)emitIdx * 256 + 128 + tid] = wpre[tid]; }
}

// one 16-byte record per cell + the vertex work list entries of its new vertices, for the flat kernels
template <class Smem>
__device__ __forceinline__ void vxb_write_cell_records(const Smem& s, const VxbDev& d, unsigned ntc, unsigned voff, unsigned cellBase, unsigned slot)
{
	for (unsigned i = threadIdx.x; i < ntc; i += VXB_THREADS)
	{
		const unsigned rb = s.recB[i];
		VxbCellRec cr;
		cr.a = (unsigned)s.list[i] | ((unsigned)s.cz[i] << 12) | ((rb >> 24) << 28);
		cr.b = s.recA[i];
		cr.c = rb & 0x00FFFFFFu;
		cr.d = (unsigned)s.vbase[i] | ((unsigned)s.tbase[i] << 16);
		*reinterpret_cast<uint4*>(&d.cellRecs[cellBase + i]) = *reinterpret_cast<const uint4*>(&cr);
		d.cellBlock[cellBase + i] = slot;
		unsigned nm = rb & 0xFFFu, j = voff + s.vbase[i];
		while (nm) { const int k = __ffs(nm) - 1; nm &= nm - 1; d.vlist[j++] = ((cellBase + i) << 4) | (unsigned)k; }
	}
}

// the block's record in directory slot `slot` (one thread); a mid-level block also joins the transition work list
__device__ __forceinline__ void vxb_write_block_rec(const VxbDev& d, unsigned slot, int level, unsigned coordId, unsigned emitIdx,
	unsigned voff, unsigned ioff, unsigned cellBase, unsigned ntc, unsigned nverts, unsigned ntris, unsigned removed)
{
	VxbBlockRec br;
	br.packed = ((unsigned)level << 28) | coordId; br.emitIdx = emitIdx; br.voff = voff; br.ioff = ioff; br.cellBase = cellBase;
	br.ntc = ntc; br.nverts = nverts; br.ntris = ntris; br.removed = removed;
	for (int f = 0; f < 6; ++f) { br.tvoff[f] = 0; br.tioff[f] = 0; br.tvcount[f] = 0; br.ticount[f] = 0; }
	br.pad[0] = br.pad[1] = br.pad[2] = 0;
	d.blockRecs[slot] = br;
	if (level > 0 && level != d.lastLevel && d.transitions) d.transList[atomicAdd(&d.counters->transBlocks, 1u)] = slot;
}

// ---- the phases of vxb_block_kernel<0|1|2> that more than one of them runs ----

template <class Smem>
__device__ __forceinline__ void vxb_block_prologue(Smem& s)
{
	const int tid = threadIdx.x;
	if (tid == 0) { vxb_mbar_init(&s.mbar[0], 1); vxb_mbar_init(&s.mbar[1], 1); }
	if (tid < 16) s.hist[tid] = 0;
	if (tid < 8) s.used[tid] = 0;
	for (int i = tid; i < 256; i += VXB_THREADS) { s.tabClass[i] = vxbGRegularCellClass[i]; s.tabCell[i] = vxbGRegularCellData[i]; }
	for (int i = tid; i < 3072; i += VXB_THREADS) s.tabVert[i] = vxbGRegularVertexData[i];
}

// the CTA's statistics, once per CTA
template <class Smem>
__device__ __forceinline__ void vxb_block_epilogue(const Smem& s, const VxbDev& d, unsigned statNonTrivial)
{
	const int tid = threadIdx.x;
	__syncthreads();
	if (tid < 16 && s.hist[tid]) atomicAdd(&d.counters->perCase[tid], s.hist[tid]);
	if (tid < 8 && s.used[tid]) atomicOr(&d.counters->usedMaterials[tid], s.used[tid]);
	if (tid == 0 && statNonTrivial) atomicAdd(&d.counters->nonTrivial, statNonTrivial);
}

// block coordinates of entry `item` of a level's work list (coordIds, x fastest; blocks per axis: a power of two)
__device__ __forceinline__ void vxb_work_block(const VxbDev& d, const unsigned* worklist, unsigned item, int level, int& bx, int& by, int& bz)
{
	const int nbl = (d.n >> 4) >> level, sh = __ffs(nbl) - 1;
	const unsigned c = worklist[item];
	bx = c & (nbl - 1); by = (c >> sh) & (nbl - 1); bz = c >> (2 * sh);
}

// thread 0 takes the next item from the cursor into s.item and clears the per-item flags; the caller's barrier publishes them
template <class Smem>
__device__ __forceinline__ void vxb_take_item(Smem& s, unsigned* cursor)
{
	if (threadIdx.x == 0) { s.item = atomicAdd(cursor, 1u); s.hasChild = 0; s.pageReady = 0; s.take = 1; s.removed = 0; }
}

// tile -> non-trivial bits (s.nt32) and their exclusive prefix per word (s.wpre); returns the block's non-trivial cells
template <int PITCH, int ROWS, class Smem>
__device__ __forceinline__ unsigned vxb_count_cells(Smem& s, const signed char* tile)
{
	const int tid = threadIdx.x;
	vxb_classify_bits<PITCH, ROWS>(tile, s.rowSign, s.nt32);
	__syncthreads();
	unsigned ntc;
	const unsigned cnt = (tid < 128) ? __popc(s.nt32[tid]) : 0u; // one word per thread
	const unsigned ex = vxb_block_scan(cnt, s.warpSums, ntc);
	if (tid < 128) s.wpre[tid] = ex;
	__syncthreads();
	return ntc;
}

// A block with ntc > 0 non-trivial cells: the level's page (level 0: consistency bits; above: the material page), the
// compact list (inCap), the emission index (emitMine; thread 0 counts the cells in statNonTrivial), the statistics
// (PerCaseCellsCount :1574) and, above level 0, the material of every non-trivial cell (:1568): majority vote of its 8
// children, stored in the level's page.  An in-capacity level-0 block takes its histogram in pass A instead.
template <int PITCH, int ROWS, class Smem>
__device__ __forceinline__ void vxb_block_cells(Smem& s, const signed char* tile, const VxbDev& d, int level, unsigned coordId,
	int bx, int by, int bz, unsigned ntc, bool inCap, bool emitMine, unsigned& statNonTrivial)
{
	const int tid = threadIdx.x, m = 1 << level;
	if (level == 0)
	{
		if (tid < 128)
		{
			unsigned* page = d.consPages + (size_t)coordId * 128;
			// bits are only ever set (:757); a full run has cleared consValid, and this block is the only one that sets its flag
			page[tid] = (d.incremental && d.consValid[coordId]) ? (page[tid] | s.nt32[tid]) : s.nt32[tid];
		}
	}
	else if (!d.cacheValid[level][coordId]) vxb_init_cache_page(d, level, coordId);
	if (inCap) vxb_compact_cells(s.nt32, s.wpre, s.list);
	__syncthreads();
	if (tid == 0)
	{
		if (level == 0) d.consValid[coordId] = 1; else d.cacheValid[level][coordId] = 1;
		s.pageReady = 1;
		if (emitMine)
		{
			const unsigned idx = d.workBase[level] + atomicAdd(&d.counters->emitCount[level], 1u);
			d.emitList[idx] = ((unsigned)level << 28) | coordId;
			s.emitIdx = idx;
			statNonTrivial += ntc;
		}
	}
	auto cellWork = [&](int c) {
		signed char v[8];
		vxb_tile_samples<PITCH, ROWS>(tile, c, v);
		if (emitMine) atomicAdd(&s.hist[s.tabClass[vxb_case_code(v)]], 1u);
		if (level > 0)
		{
			const VxbVoteSource voteSrc = vxb_vote_source(d, level);
			const int vote = vxb_vote_cell(voteSrc, (bx * 16 + (c & 15)) * m, (by * 16 + ((c >> 4) & 15)) * m, (bz * 16 + (c >> 8)) * m);
			if (vote >= 0) d.cachePages[level][(size_t)coordId * 4096 + c] = (unsigned short)vote;
		}
	};
	if (inCap) { if (level > 0) for (unsigned i = tid; i < ntc; i += VXB_THREADS) cellWork(s.list[i]); }
	else
	{
		for (int r = tid; r < 256; r += VXB_THREADS)
		{
			unsigned bits = reinterpret_cast<const unsigned short*>(s.nt32)[r];
			while (bits) { const int x = __ffs(bits) - 1; bits &= bits - 1; cellWork(r * 16 + x); }
		}
	}
	__syncthreads();
	if (!inCap && emitMine) vxb_save_nt(d, s.emitIdx, s.nt32, s.wpre);
}

// A mid-level block (levels >= 1 below the last): every cell of every transition face votes too, trivial ones included
// (:1859) - observable at the next level.  Ends without a barrier.
template <class Smem>
__device__ __forceinline__ void vxb_face_votes(Smem& s, const VxbDev& d, int level, int nb, unsigned coordId, int bx, int by, int bz)
{
	const int tid = threadIdx.x, m = 1 << level;
	const VxbVoteSource voteSrc = vxb_vote_source(d, level);
	if (tid < 8)
	{
		const int cnb = nb * 2;
		const size_t cb = ((size_t)(bz * 2 + (tid >> 2)) * cnb + (by * 2 + ((tid >> 1) & 1))) * cnb + (bx * 2 + (tid & 1));
		const bool valid = (level == 1) ? __ldcg(d.consValid + cb) : __ldcg(d.cacheValid[level - 1] + cb);
		if (valid) atomicOr(&s.hasChild, 1u);
	}
	__syncthreads();
	if (!s.hasChild) return;
	// an all-{EMPTY,0} page is indistinguishable from no page, so it can be created before the votes
	if (!s.pageReady)
	{
		if (!d.cacheValid[level][coordId]) vxb_init_cache_page(d, level, coordId);
		__syncthreads();
		if (tid == 0) { d.cacheValid[level][coordId] = 1; s.pageReady = 1; }
	}
	for (int fc = tid; fc < 256; fc += VXB_THREADS)
	{
		const int row = fc >> 4, col = fc & 15;
		// most face cells have no child with a material: test all six faces first (independent loads, all in flight
		// together), then run the vote only where it can succeed
		unsigned candidates = 0;
#pragma unroll
		for (int face = 0; face < 6; ++face)
		{
			int axis, ua, va;
			vxb_face_axes(face, axis, ua, va);
			const int bc = (axis == 0) ? bx : (axis == 1 ? by : bz);
			const bool outside = face < 3 ? (bc == 0) : (bc == nb - 1); // neighbour block outside the grid (:1829-1835)
			const int edge = (face >= 3) ? 15 : 0;
			const int lx = axis == 0 ? edge : col, ly = axis == 1 ? edge : (axis == 2 ? row : col), lz = axis == 2 ? edge : row;
			if (vxb_vote_candidate(voteSrc, (bx * 16 + lx) * m, (by * 16 + ly) * m, (bz * 16 + lz) * m) && !outside) candidates |= 1u << face;
		}
		while (candidates)
		{
			const int face = __ffs(candidates) - 1;
			candidates &= candidates - 1;
			int axis, ua, va;
			vxb_face_axes(face, axis, ua, va);
			// local[axis] = edge, local[ua] = col, local[va] = row, written with selects (an indexed array would be local memory)
			const int edge = (face >= 3) ? 15 : 0;
			const int local[3] = { axis == 0 ? edge : col, axis == 1 ? edge : (axis == 2 ? row : col), axis == 2 ? edge : row };
			const int vote = vxb_vote_cell(voteSrc, (bx * 16 + local[0]) * m, (by * 16 + local[1]) * m, (bz * 16 + local[2]) * m);
			if (vote >= 0) d.cachePages[level][(size_t)coordId * 4096 + local[2] * 256 + local[1] * 16 + local[0]] = (unsigned short)vote;
		}
	}
}

// The block's ranges of the arenas and its directory slot: four independent atomics from four warps, one round trip instead
// of four in a row.  `cells`: the block writes cell records (else cellBase = 0).  A block that does not fit writes nothing;
// the run is repeated with larger arenas.  (The caller tests the fit: returned from here, the test compiles worse.)
template <class Smem>
__device__ __forceinline__ void vxb_reserve(Smem& s, const VxbDev& d, unsigned ntc, unsigned nverts, unsigned ntris, bool cells,
	unsigned& voff, unsigned& ioff, unsigned& cellBase, unsigned& slot)
{
	const int tid = threadIdx.x;
	if (tid == 0) s.voff = atomicAdd(&d.counters->vertices, nverts);
	if (tid == 32) s.ioff = atomicAdd(&d.counters->indices, ntris * 3);
	if (tid == 64 && cells) s.cellBase = atomicAdd(&d.counters->cells, ntc);
	if (tid == 96) s.slot = atomicAdd(&d.counters->records, 1u);
	__syncthreads();
	voff = s.voff; ioff = s.ioff; cellBase = cells ? s.cellBase : 0u; slot = s.slot;
}

// levels >= 1: the decide passes over the compact list -> cell records + vertex work list for the flat kernels, the block's
// non-trivial bits for vxb_triangle_kernel, and its directory record
template <class Smem>
__device__ __forceinline__ void vxb_emit_cell_records(Smem& s, const signed char* tile, const VxbDev& d, int level, unsigned coordId,
	int bx, int by, int bz, unsigned ntc)
{
	unsigned nverts, ntris, voff, ioff, cellBase, slot;
	vxb_decide_cells<VXB_TILE_PITCH, 17, true>(s, tile, d, level, coordId, bx, by, bz, ntc, nverts, ntris);
	vxb_reserve(s, d, ntc, nverts, ntris, true, voff, ioff, cellBase, slot);
	const bool fits = (unsigned long long)voff + nverts <= d.vcap && (unsigned long long)ioff + ntris * 3ull <= d.icap
		&& (unsigned long long)cellBase + ntc <= d.ccap && slot < d.rcap;
	if (fits)
	{
		vxb_write_cell_records(s, d, ntc, voff, cellBase, slot);
		vxb_save_nt(d, s.emitIdx, s.nt32, s.wpre);
	}
	if (fits && threadIdx.x == 0) vxb_write_block_rec(d, slot, level, coordId, s.emitIdx, voff, ioff, cellBase, ntc, nverts, ntris, 0u);
}

template <int MODE>
__global__ void vxb_block_kernel(const __grid_constant__ CUtensorMap tmapA, const __grid_constant__ CUtensorMap tmapB, const VxbDev d, const int levelArg);

// Level 0 from its work list: the halo tile by one TMA load (tmapA: the 48 x 19 x 19 box of the distance volume) into one
// tile buffer; the new vertices and the triangles are produced right here from shared memory (no per-cell records in
// global memory).  Blocks over the capacities go to vxb_big_block_kernel + the flat kernels.
template <>
__global__ void __launch_bounds__(VXB_THREADS, VXB_OCC) vxb_block_kernel<0>(const __grid_constant__ CUtensorMap tmapA, const __grid_constant__ CUtensorMap, const VxbDev d, const int)
{
	extern __shared__ __align__(128) unsigned char smemRaw[];
	VxbBlockSmem<0>& s = *reinterpret_cast<VxbBlockSmem<0>*>(smemRaw);
	const int tid = threadIdx.x;
	const VxbGrid g = d.grid;
	const int nb = d.n / 16;
	unsigned phase = 0, statNonTrivial = 0;
	vxb_block_prologue(s);
	const unsigned workCount = d.counters->workCount[0];
	const unsigned* const worklist = d.worklist + d.workBase[0];
	unsigned* const cursor = &d.counters->workCursor[0];
	// thread 0 requests the halo tile of item `it`.  The tile starts one sample before the block (x: 16 samples, a 16-byte
	// aligned start); on the low grid edge the box starts at a negative coordinate and TMA zero-fills what lies outside.
	auto issue = [&](unsigned it) {
		if (tid != 0) return;
		int x, y, z;
		vxb_work_block(d, worklist, it, 0, x, y, z);
		vxb_fence_proxy_async();
		vxb_mbar_expect_tx(&s.mbar[0], VXB_DTILE_BYTES);
		vxb_tma_load_3d(s.tiles[0], &tmapA, x * 16 - 16, y * 16 - 1, z * 16 - 1, &s.mbar[0]);
	};

	// items are taken two ahead: the cursor's round trip for the item after next overlaps a whole block
	if (tid == 0) { s.item = atomicAdd(cursor, 1u); s.ahead = atomicAdd(cursor, 1u); }
	__syncthreads();
	unsigned item = s.item, aheadItem = s.ahead;
	if (item < workCount) issue(item);

	while (item < workCount)
	{
		const unsigned nextItem = aheadItem;
		unsigned ahead = 0; // thread 0: the item after next, published in s.ahead at the end of this block
		if (tid == 0) { ahead = atomicAdd(cursor, 1u); s.removed = 0; }
		bool nextIssued = false; // one tile buffer: the next tile is requested as soon as this one is not read any more
		int bx, by, bz;
		vxb_work_block(d, worklist, item, 0, bx, by, bz);
		const unsigned coordId = ((unsigned)bz * nb + by) * nb + bx;
		signed char* const tileRaw = s.tiles[0];
		const int hsx = bx * 16 - 16, hsy = by * 16 - 1, hsz = bz * 16 - 1; // first coordinate held by the halo tile

		vxb_mbar_wait(&s.mbar[0], phase);
		phase ^= 1u;
		// grid edges: TMA zero-fills outside the volume, the reference clamps the coordinate to [0, n-1] (:1037-1047, :1198).
		// One axis after the other, so that edge and corner entries copy values already fixed on the earlier axes.
		const int lastX = d.n - 1 - hsx, lastY = d.n - 1 - hsy, lastZ = d.n - 1 - hsz; // tile index of coordinate n-1
		if (bx == 0 || bx == nb - 1)
		{
			__syncthreads();
			for (int i = tid; i < 19 * 19; i += VXB_THREADS)
			{
				signed char* r = tileRaw + i * VXB_DTILE_PITCH;
				if (bx == 0) r[15] = r[16];
				if (bx == nb - 1) { r[lastX + 1] = r[lastX]; r[lastX + 2] = r[lastX]; }
			}
		}
		if (by == 0 || by == nb - 1)
		{
			__syncthreads();
			for (int i = tid; i < 19 * VXB_DTILE_PITCH; i += VXB_THREADS)
			{
				const int z = i / VXB_DTILE_PITCH, x = i % VXB_DTILE_PITCH;
				signed char* p = tileRaw + z * 19 * VXB_DTILE_PITCH + x;
				if (by == 0) p[0] = p[VXB_DTILE_PITCH];
				if (by == nb - 1) for (int q = lastY + 1; q < 19; ++q) p[q * VXB_DTILE_PITCH] = p[lastY * VXB_DTILE_PITCH];
			}
		}
		if (bz == 0 || bz == nb - 1)
		{
			__syncthreads();
			for (int i = tid; i < 19 * VXB_DTILE_PITCH; i += VXB_THREADS)
			{
				const int y = i / VXB_DTILE_PITCH, x = i % VXB_DTILE_PITCH;
				signed char* p = tileRaw + y * VXB_DTILE_PITCH + x;
				if (bz == 0) p[0] = p[19 * VXB_DTILE_PITCH];
				if (bz == nb - 1) for (int q = lastZ + 1; q < 19; ++q) p[q * 19 * VXB_DTILE_PITCH] = p[lastZ * 19 * VXB_DTILE_PITCH];
			}
		}
		const signed char* const tile = tileRaw + (19 + 1) * VXB_DTILE_PITCH + 16; // sample (0, 0, 0) of the block
		__syncthreads();

		const unsigned ntc = vxb_count_cells<VXB_DTILE_PITCH, 19>(s, tile);
		const bool inCap = ntc <= (unsigned)VxbBlockCaps<0>::CAP;
		if (ntc > 0) vxb_block_cells<VXB_DTILE_PITCH, 19>(s, tile, d, 0, coordId, bx, by, bz, ntc, inCap, true, statNonTrivial);
		if (ntc > 0 && !inCap) { if (tid == 0) d.bigList[atomicAdd(&d.counters->bigCount, 1u)] = s.emitIdx; }
		else if (ntc > 0)
		{
			unsigned nverts, ntris, voff, ioff, cellBase, slot;
			vxb_decide_cells<VXB_DTILE_PITCH, 19, true>(s, tile, d, 0, coordId, bx, by, bz, ntc, nverts, ntris);
			if (nverts > (unsigned)VxbBlockCaps<0>::VL)
			{
				// too many vertices for the in-CTA path: hand the block to vxb_big_block_kernel + the flat kernels
				__syncthreads();
				vxb_save_nt(d, s.emitIdx, s.nt32, s.wpre);
				if (tid == 0) d.bigList[atomicAdd(&d.counters->bigCount, 1u)] = s.emitIdx;
			}
			else
			{
				vxb_reserve(s, d, ntc, nverts, ntris, false, voff, ioff, cellBase, slot);
				const bool fits = (unsigned long long)voff + nverts <= d.vcap && (unsigned long long)ioff + ntris * 3ull <= d.icap
					&& (unsigned long long)cellBase + ntc <= d.ccap && slot < d.rcap;
				if (fits)
				{
					// ---- the block's new vertices, one thread each (:1576-1726), from the halo tile ----
					for (unsigned i = tid; i < ntc; i += VXB_THREADS)
					{
						unsigned nm = s.recB[i] & 0xFFFu, j = s.vbase[i];
						while (nm) { const int k = __ffs(nm) - 1; nm &= nm - 1; s.vl[j++] = (unsigned short)((i << 4) | (unsigned)k); }
					}
					__syncthreads();
					VxbTileView tv;
					tv.dist = tileRaw; tv.ox = bx * 16; tv.oy = by * 16; tv.oz = bz * 16; tv.sx = hsx; tv.sy = hsy; tv.sz = hsz;
					tv.mat = g.mat; tv.blend = g.blend; tv.n = d.n; // the two material / blend taps of a vertex stay global loads
					for (unsigned j = tid; j < nverts; j += VXB_THREADS)
					{
						const unsigned e = s.vl[j];
						const unsigned i = e >> 4; const int k = e & 15;
						const int c = s.list[i];
						const unsigned code = s.cz[i] & 0xFF, zm = s.cz[i] >> 8;
						const int local[3] = { c & 15, (c >> 4) & 15, c >> 8 };
						const int base[3] = { bx * 16 + local[0], by * 16 + local[1], bz * 16 + local[2] };
						const unsigned ra = s.recA[i];
						const unsigned matId = ra & 0xFF, matBlend = (ra >> 8) & 0xFF;
						VxbVertexDesc vd = vxb_regular_vertex_desc_lite(s.tabVert[code * 12 + k], zm);
						VxbRawVertex rv;
						if (vd.endpoint)
						{
							const bool quirk = (s.recB[i] >> (12 + k)) & 1u;
							vxb_corner_vertex(tv, 0, base, local, quirk ? vd.v0 : ((vd.t == 0) ? vd.v1 : vd.v0), matId, matBlend, rv);
						}
						else
						{
							const int a = vxb_dist(tv, base[0] + (vd.v0 & 1), base[1] + ((vd.v0 >> 1) & 1), base[2] + (vd.v0 >> 2));
							const int b = vxb_dist(tv, base[0] + (vd.v1 & 1), base[1] + ((vd.v1 >> 1) & 1), base[2] + (vd.v1 >> 2));
							vd.t = vxb_fixed_t(a, b); // :1591
							vxb_edge_vertex(tv, 0, base, local, vd, matId, matBlend, rv);
						}
						vxb_regular_secondary(0, rv);
						VxbVertex ov;
						vxb_finish_vertex(rv, *d.lut, ov);
						vxb_store_vertex(d.verts + voff + j, ov);
						atomicOr(&s.used[matId >> 5], 1u << (matId & 31));
					}
					__syncthreads(); // the positions are read back by the degenerate test below
					if (nextItem < workCount) { issue(nextItem); nextIssued = true; } // the tile is not read any more
					// ---- triangles, one thread per non-trivial cell (:1714-1726 + the degenerate filter of :1300-1321) ----
					// (the step of vxb_triangle_kernel with the owner records in shared memory; one function shared by the two
					// gives vxb_triangle_kernel a 40th register)
					unsigned removed = 0;
					for (unsigned i = tid; i < ntc; i += VXB_THREADS)
					{
						const int c = s.list[i];
						const unsigned code = s.cz[i] & 0xFF, zm = s.cz[i] >> 8;
						const unsigned char* cd = &s.tabCell[s.tabClass[code] * 16];
						const unsigned geo = cd[0];
						const unsigned newMask = s.recB[i] & 0xFFFu;
						unsigned w[6] = { 0u, 0u, 0u, 0u, 0u, 0u }; // block-local vertex ids as 16-bit halves (an indexed array would be local memory)
						unsigned nextNew = s.vbase[i];
						const int nv = (int)(geo >> 4);
#pragma unroll
						for (int k = 0; k < 12; ++k)
						{
							if (k < nv)
							{
								unsigned vid;
								if ((newMask >> k) & 1u) vid = nextNew++;
								else
								{
									const VxbVertexDesc vd = vxb_regular_vertex_desc_lite(s.tabVert[code * 12 + k], zm);
									const int oc = c - (vd.dir & 1) - ((vd.dir >> 1) & 1) * 16 - ((vd.dir >> 2) & 1) * 256; // reused => the owner exists
									const unsigned oi = vxb_rank_of(s.nt32, s.wpre, oc);
									const unsigned ok = (s.recA[oi] >> (16 + 4 * vd.slot)) & 0xF;
									vid = (unsigned)s.vbase[oi] + __popc(s.recB[oi] & 0xFFFu & ((1u << ok) - 1u));
								}
								w[k >> 1] |= vid << ((k & 1) * 16);
							}
						}
						auto vidOf = [&](unsigned k) -> unsigned {
							const unsigned q = k >> 1;
							const unsigned pair = q == 0 ? w[0] : q == 1 ? w[1] : q == 2 ? w[2] : q == 3 ? w[3] : q == 4 ? w[4] : w[5];
							return (k & 1u) ? (pair >> 16) : (pair & 0xFFFFu);
						};
						unsigned* out = d.idx + ioff + (unsigned)s.tbase[i] * 3;
						// a level-0 cell without a zero sample cannot produce a degenerate triangle (see vxb_triangle_kernel)
						const bool cannotDegenerate = zm == 0u;
						for (unsigned tr = 0; tr < (geo & 0xF); ++tr, out += 3)
						{
							const unsigned a = vidOf(cd[1 + tr * 3]), b = vidOf(cd[2 + tr * 3]), cc = vidOf(cd[3 + tr * 3]);
							bool kept = true;
							if (!cannotDegenerate)
							{
								const float* fa = d.verts[voff + a].pos; const float* fb = d.verts[voff + b].pos; const float* fc = d.verts[voff + cc].pos;
								const float pa[3] = { fa[0] * 256.f, fa[2] * 256.f, fa[1] * 256.f };
								const float pb[3] = { fb[0] * 256.f, fb[2] * 256.f, fb[1] * 256.f };
								const float pc[3] = { fc[0] * 256.f, fc[2] * 256.f, fc[1] * 256.f };
								kept = vxb_triangle_kept(pa, pb, pc);
							}
							if (kept) { out[0] = a; out[1] = b; out[2] = cc; }
							else { out[0] = 0xFFFFFFFFu; out[1] = 0xFFFFFFFFu; out[2] = 0xFFFFFFFFu; ++removed; }
						}
					}
					if (removed) atomicAdd(&s.removed, removed);
					__syncthreads();
					if (tid == 0) vxb_write_block_rec(d, slot, 0, coordId, s.emitIdx, voff, ioff, cellBase, ntc, nverts, ntris, s.removed);
				}
			}
		}
		if (tid == 0) s.ahead = ahead;
		__syncthreads();
		if (!nextIssued && nextItem < workCount) issue(nextItem);
		item = nextItem;
		aheadItem = s.ahead;
	}
	vxb_block_epilogue(s, d, statNonTrivial);
}

// One level below the coarse ones (levelArg) from its work list.  17^3 tile (vxb_tile_issue: TMA on the even lattice of
// level 1 / the level's lattice, strided gather else), double buffered: the next block's tile lands while this one is
// worked on.  Writes 16-byte cell records + the vertex work list for the flat per-vertex / per-cell kernels.
template <>
__global__ void __launch_bounds__(VXB_THREADS, VXB_OCC) vxb_block_kernel<1>(const __grid_constant__ CUtensorMap tmapA, const __grid_constant__ CUtensorMap tmapB, const VxbDev d, const int levelArg)
{
	extern __shared__ __align__(128) unsigned char smemRaw[];
	VxbBlockSmem<1>& s = *reinterpret_cast<VxbBlockSmem<1>*>(smemRaw);
	const int tid = threadIdx.x;
	const int level = levelArg;
	unsigned phaseBits = 0, statNonTrivial = 0; // mbarrier phase of each tile buffer, bit = buffer
	vxb_block_prologue(s);
	const unsigned workCount = d.counters->workCount[level];
	const unsigned* const worklist = d.worklist + d.workBase[level];
	unsigned* const cursor = &d.counters->workCursor[level];
	auto issue = [&](int buf, unsigned it) { int x, y, z; vxb_work_block(d, worklist, it, level, x, y, z); vxb_tile_issue(s.tiles[buf], &s.mbar[buf], &tmapA, &tmapB, d, level, x, y, z); };

	if (tid == 0) s.item = atomicAdd(cursor, 1u);
	__syncthreads();
	unsigned item = s.item;
	int buf = 0;
	if (item < workCount) issue(0, item);
	__syncthreads();
	while (item < workCount)
	{
		vxb_take_item(s, cursor);
		__syncthreads();
		const unsigned nextItem = s.item;
		if (nextItem < workCount) issue(buf ^ 1, nextItem);
		int bx, by, bz;
		vxb_work_block(d, worklist, item, level, bx, by, bz);
		const int nb = d.n / 16 / (1 << level);
		const unsigned coordId = ((unsigned)bz * nb + by) * nb + bx;
		const bool midLevel = level > 0 && level != d.lastLevel;
		const signed char* const tile = s.tiles[buf];
		unsigned ph = (phaseBits >> buf) & 1u;
		vxb_tile_complete(s.tiles[buf], &s.mbar[buf], ph, d, level, bx, by, bz);
		phaseBits = (phaseBits & ~(1u << buf)) | (ph << buf);
		__syncthreads();

		const unsigned ntc = vxb_count_cells<VXB_TILE_PITCH, 17>(s, tile);
		const bool inCap = ntc <= (unsigned)VxbBlockCaps<1>::CAP;
		if (ntc > 0) vxb_block_cells<VXB_TILE_PITCH, 17>(s, tile, d, level, coordId, bx, by, bz, ntc, inCap, true, statNonTrivial);
		if (midLevel) vxb_face_votes(s, d, level, nb, coordId, bx, by, bz);
		__syncthreads(); // the votes of this block are visible to the CTA (pass A reads the page back)
		if (ntc > 0 && !inCap) { if (tid == 0) d.bigList[atomicAdd(&d.counters->bigCount, 1u)] = s.emitIdx; }
		else if (ntc > 0) vxb_emit_cell_records(s, tile, d, level, coordId, bx, by, bz, ntc);
		__syncthreads();
		item = nextItem;
		buf ^= 1;
	}
	vxb_block_epilogue(s, d, statNonTrivial);
}

// All coarse levels [coarseLo, computed) in ONE launch: items = the blocks in level order from one cursor.  A block waits
// for its children, applies the block-walk test itself, then works like <1>; it is released to its parent right after its
// votes.
template <>
__global__ void __launch_bounds__(VXB_THREADS, VXB_OCC) vxb_block_kernel<2>(const __grid_constant__ CUtensorMap, const __grid_constant__ CUtensorMap, const VxbDev d, const int)
{
	extern __shared__ __align__(128) unsigned char smemRaw[];
	VxbBlockSmem<2>& s = *reinterpret_cast<VxbBlockSmem<2>*>(smemRaw);
	const int tid = threadIdx.x;
	unsigned phase = 0, statNonTrivial = 0;
	vxb_block_prologue(s);
	if (tid == 0)
	{
		unsigned acc = 0;
		for (int l = d.coarseLo; l < d.computed; ++l)
		{
			const int nbl = (d.n >> 4) >> l;
			const int nx = d.ranged ? d.rangeMax[l][0] - d.rangeMin[l][0] : nbl, ny = d.ranged ? d.rangeMax[l][1] - d.rangeMin[l][1] : nbl, nz = d.ranged ? d.rangeMax[l][2] - d.rangeMin[l][2] : nbl;
			acc += (nx > 0 && ny > 0 && nz > 0) ? (unsigned)nx * ny * nz : 0u;
			s.levelEnd[l - d.coarseLo] = acc; // end of the items of level l
		}
	}
	__syncthreads();
	const unsigned workCount = (d.computed > d.coarseLo) ? s.levelEnd[d.computed - d.coarseLo - 1] : 0u;
	unsigned* const cursor = &d.counters->coarseCursor;

	if (tid == 0) s.item = atomicAdd(cursor, 1u);
	__syncthreads();
	unsigned item = s.item;
	__syncthreads();
	while (item < workCount)
	{
		vxb_take_item(s, cursor);
		__syncthreads();
		const unsigned nextItem = s.item;
		int q = 0;
		while (item >= s.levelEnd[q]) ++q;
		const int level = d.coarseLo + q, nbl = (d.n >> 4) >> level;
		const unsigned r = item - (q ? s.levelEnd[q - 1] : 0u);
		const int x0 = d.ranged ? d.rangeMin[level][0] : 0, y0 = d.ranged ? d.rangeMin[level][1] : 0, z0 = d.ranged ? d.rangeMin[level][2] : 0;
		const int nx = d.ranged ? d.rangeMax[level][0] - x0 : nbl, ny = d.ranged ? d.rangeMax[level][1] - y0 : nbl;
		const int bx = x0 + (int)(r % nx), by = y0 + (int)((r / nx) % ny), bz = z0 + (int)(r / ((unsigned)nx * ny));
		const int nb = d.n / 16 / (1 << level);
		const unsigned coordId = ((unsigned)bz * nb + by) * nb + bx;
		const bool midLevel = level > 0 && level != d.lastLevel;

		// warp 0: wait for the children of this run (blocks of the previous coarse level inside the run's range), one lane
		// each, then the block walk test (vxb_coarse_block_needed) with one lane per child-level neighbour.  The children
		// were taken earlier from the same cursor, so they are running or done: no deadlock.
		if (tid < 32)
		{
			const int cnb = nb * 2, cl = level - 1;
			if (level > d.coarseLo && tid < 8)
			{
				const int cx = bx * 2 + (tid & 1), cy = by * 2 + ((tid >> 1) & 1), cz = bz * 2 + (tid >> 2);
				const bool inRun = !(d.ranged && (cx < d.rangeMin[cl][0] || cx >= d.rangeMax[cl][0] || cy < d.rangeMin[cl][1] || cy >= d.rangeMax[cl][1] || cz < d.rangeMin[cl][2] || cz >= d.rangeMax[cl][2]));
				if (inRun)
				{
					const volatile unsigned char* flag = d.coarseDone + d.coarseBase[cl] + ((size_t)cz * cnb + cy) * cnb + cx;
					unsigned spins = 0;
					while (!*flag) { __nanosleep(32); if (++spins > (1u << 24)) __trap(); }
				}
				__threadfence();
			}
			__syncwarp();
			unsigned u = 0, anyChild = 0;
			if (tid < 27)
			{
				const int x = tid % 3, y = (tid / 3) % 3, z = tid / 9;
				const int cx = min(2 * bx + x, cnb - 1), cy = min(2 * by + y, cnb - 1), cz = min(2 * bz + z, cnb - 1);
				const size_t cb = ((size_t)cz * cnb + cy) * cnb + cx;
				u = d.mixInfo[cl][cb];
				if (x < 2 && y < 2 && z < 2) anyChild = __ldcg(d.cacheValid[cl] + cb);
			}
			u = __reduce_or_sync(0xFFFFFFFFu, u);
			anyChild = __reduce_or_sync(0xFFFFFFFFu, anyChild);
			if (tid == 0)
			{
				s.take = (u == 3u || anyChild != 0u) ? 1u : 0u;
				if (s.take)
				{
					// the block's 17^3 samples: one TMA box of the level's lattice (far-edge entries included, no fix-up)
					vxb_fence_proxy_async();
					vxb_mbar_expect_tx(&s.mbar[0], VXB_TILE_BYTES);
					vxb_tma_load_3d(s.tiles[0], d.coarseMaps + level, bx * 16, by * 16, bz * 16, &s.mbar[0]);
				}
			}
		}
		__syncthreads();
		if (!s.take)
		{
			if (tid == 0) { __threadfence(); *(volatile unsigned char*)(d.coarseDone + d.coarseBase[level] + coordId) = 1; }
			__syncthreads();
			item = nextItem;
			continue;
		}
		const signed char* const tile = s.tiles[0];
		vxb_mbar_wait(&s.mbar[0], phase);
		phase ^= 1u;
		__syncthreads();

		const unsigned ntc = vxb_count_cells<VXB_TILE_PITCH, 17>(s, tile);
		const bool inCap = ntc <= (unsigned)VxbBlockCaps<2>::CAP;
		// sharded runs: every rank classifies the coarse levels (the votes feed the next level), one of them emits the block
		const bool emitMine = vxb_coarse_emit_is_mine(d, level, coordId);
		if (ntc > 0) vxb_block_cells<VXB_TILE_PITCH, 17>(s, tile, d, level, coordId, bx, by, bz, ntc, inCap, emitMine, statNonTrivial);
		if (midLevel) vxb_face_votes(s, d, level, nb, coordId, bx, by, bz);
		__syncthreads(); // the votes of this block are visible to the CTA (pass A reads the page back)
		// the parent only needs this block's page, so it is released before the block's own emission work
		if (tid == 0) { __threadfence(); *(volatile unsigned char*)(d.coarseDone + d.coarseBase[level] + coordId) = 1; }
		if (ntc > 0 && !inCap) { if (tid == 0 && emitMine) d.bigList[atomicAdd(&d.counters->bigCount, 1u)] = s.emitIdx; }
		else if (ntc > 0 && emitMine) vxb_emit_cell_records(s, tile, d, level, coordId, bx, by, bz, ntc);
		__syncthreads();
		item = nextItem;
	}
	vxb_block_epilogue(s, d, statNonTrivial);
}

// ------------------------------------------------------------------------------------------------
// vxb_big_block_kernel: the blocks vxb_block_kernel hands over in bigList (more than 1024 non-trivial cells, or a level-0
// block with more than 2048 new vertices).  Reloads the block's tile and its non-trivial bits, runs the decide passes over
// up to 4096 cells (every possible block) and writes cell records + the vertex work list for the flat kernels.
// ------------------------------------------------------------------------------------------------
struct __align__(128) VxbBigBlockSmem
{
	signed char tile[VXB_TILE_BYTES + 96];
	unsigned int nt32[128];
	unsigned int wpre[132];
	unsigned char tabClass[256];
	unsigned char tabCell[256];
	unsigned short tabVert[3072];
	unsigned int warpSums[8];
	unsigned long long mbar;
	unsigned int item, voff, ioff, cellBase, slot;
	unsigned int recA[4096];     // matId | matBlend<<8 | slotK<<16
	unsigned int recB[4096];     // newMask | quirkMask<<12 | reuse mask << 24
	unsigned short list[4096];   // compact index -> cell id
	unsigned short cz[4096];     // case code | zero mask << 8
	unsigned short vbase[4096];  // exclusive scan of new-vertex counts
	unsigned short tbase[4096];  // exclusive scan of triangle counts
};

__global__ void __launch_bounds__(VXB_THREADS, 2) vxb_big_block_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ CUtensorMap tmap1, const VxbDev d)
{
	extern __shared__ __align__(128) unsigned char smemRaw[];
	VxbBigBlockSmem& s = *reinterpret_cast<VxbBigBlockSmem*>(smemRaw);
	const int tid = threadIdx.x;
	unsigned phase = 0;

	if (tid == 0) vxb_mbar_init(&s.mbar, 1);
	for (int i = tid; i < 256; i += VXB_THREADS) { s.tabClass[i] = vxbGRegularCellClass[i]; s.tabCell[i] = vxbGRegularCellData[i]; }
	for (int i = tid; i < 3072; i += VXB_THREADS) s.tabVert[i] = vxbGRegularVertexData[i];
	__syncthreads();
	const unsigned workCount = d.counters->bigCount;

	for (;;)
	{
		if (tid == 0) s.item = atomicAdd(&d.counters->bigCursor, 1u);
		__syncthreads();
		const unsigned item = s.item;
		if (item >= workCount) break;
		const unsigned emitIdx = d.bigList[item];
		const unsigned packed = d.emitList[emitIdx];
		const int level = (int)(packed >> 28);
		const unsigned coordId = packed & 0x0FFFFFFFu;
		const int m = 1 << level, nb = d.n / 16 / m;
		const int bx = coordId % nb, by = (coordId / nb) % nb, bz = coordId / (nb * nb);

		if (tid < 128) { s.nt32[tid] = d.ntScratch[(size_t)emitIdx * 256 + tid]; s.wpre[tid] = d.ntScratch[(size_t)emitIdx * 256 + 128 + tid]; }
		__syncthreads();
		const unsigned ntc = s.wpre[127] + __popc(s.nt32[127]);
		vxb_tile_issue(s.tile, &s.mbar, &tmap, &tmap1, d, level, bx, by, bz);
		vxb_tile_complete(s.tile, &s.mbar, phase, d, level, bx, by, bz);
		vxb_compact_cells(s.nt32, s.wpre, s.list);
		__syncthreads();
		unsigned nverts, ntris;
		vxb_decide_cells<VXB_TILE_PITCH, 17, false>(s, s.tile, d, level, coordId, bx, by, bz, ntc, nverts, ntris);
		if (tid == 0)
		{
			s.voff = atomicAdd(&d.counters->vertices, nverts);
			s.ioff = atomicAdd(&d.counters->indices, ntris * 3);
			s.cellBase = atomicAdd(&d.counters->cells, ntc);
			s.slot = atomicAdd(&d.counters->records, 1u);
		}
		__syncthreads();
		const unsigned voff = s.voff, ioff = s.ioff, cellBase = s.cellBase, slot = s.slot;
		const bool fits = (unsigned long long)voff + nverts <= d.vcap && (unsigned long long)ioff + ntris * 3ull <= d.icap
			&& (unsigned long long)cellBase + ntc <= d.ccap && slot < d.rcap;
		if (fits)
		{
			vxb_write_cell_records(s, d, ntc, voff, cellBase, slot);
			if (tid == 0) vxb_write_block_rec(d, slot, level, coordId, emitIdx, voff, ioff, cellBase, ntc, nverts, ntris, 0u);
		}
		__syncthreads();
	}
}

// ------------------------------------------------------------------------------------------------
// flat kernels over the blocks with cell records (levels >= 1 and the level-0 blocks of vxb_big_block_kernel): their
// vertices and cells lie behind the split vxb_mark_split_kernel takes once vxb_block_kernel<0> is done
// ------------------------------------------------------------------------------------------------
__global__ void vxb_mark_split_kernel(const VxbDev d)
{
	d.counters->splitVertices = d.counters->vertices;
	d.counters->splitCells = d.counters->cells;
}

__global__ void __launch_bounds__(VXB_THREADS, VXB_FLAT_OCC) vxb_vertex_kernel(const VxbDev d)
{
	__shared__ unsigned sUsed[8];
	if (threadIdx.x < 8) sUsed[threadIdx.x] = 0;
	__syncthreads();
	if (!vxb_overflowed(d))
	{
		const VxbGrid g = d.grid;
		const unsigned total = d.counters->vertices;
		for (unsigned j = d.counters->splitVertices + blockIdx.x * blockDim.x + threadIdx.x; j < total; j += gridDim.x * blockDim.x)
		{
			const unsigned e = d.vlist[j];
			const unsigned ci = e >> 4; const int k = e & 15;
			const uint4 crv = *reinterpret_cast<const uint4*>(&d.cellRecs[ci]);
			const unsigned packed = d.blockRecs[d.cellBlock[ci]].packed;
			const int level = (int)(packed >> 28);
			const unsigned coordId = packed & 0x0FFFFFFFu;
			const int m = 1 << level, nb = d.n / 16 / m;
			const int c = crv.x & 0xFFF;
			const unsigned code = (crv.x >> 12) & 0xFF, zm = (crv.x >> 20) & 0xFF;
			const int local[3] = { c & 15, (c >> 4) & 15, c >> 8 };
			const int base[3] = { (int)((coordId % nb) * 16 + local[0]) * m, (int)(((coordId / nb) % nb) * 16 + local[1]) * m, (int)((coordId / (nb * nb)) * 16 + local[2]) * m };
			const unsigned matId = crv.y & 0xFF, matBlend = (crv.y >> 8) & 0xFF;
			VxbVertexDesc vd = vxb_regular_vertex_desc_lite(vxbGRegularVertexData[code * 12 + k], zm);
			VxbRawVertex rv;
			if (vd.endpoint)
			{
				const bool quirk = (crv.z >> (12 + k)) & 1u;
				vxb_corner_vertex(g, level, base, local, quirk ? vd.v0 : ((vd.t == 0) ? vd.v1 : vd.v0), matId, matBlend, rv);
			}
			else
			{
				if (level == 0)
				{
					const int a = vxb_dist(g, base[0] + (vd.v0 & 1), base[1] + ((vd.v0 >> 1) & 1), base[2] + (vd.v0 >> 2));
					const int b = vxb_dist(g, base[0] + (vd.v1 & 1), base[1] + ((vd.v1 >> 1) & 1), base[2] + (vd.v1 >> 2));
					vd.t = vxb_fixed_t(a, b); // :1591 (coarser levels recompute t after the LOD descent)
				}
				vxb_edge_vertex(g, level, base, local, vd, matId, matBlend, rv);
			}
			vxb_regular_secondary(level, rv);
			VxbVertex ov;
			vxb_finish_vertex(rv, *d.lut, ov);
			vxb_store_vertex(d.verts + j, ov);
			atomicOr(&sUsed[matId >> 5], 1u << (matId & 31));
		}
	}
	__syncthreads();
	if (threadIdx.x < 8 && sUsed[threadIdx.x]) atomicOr(&d.counters->usedMaterials[threadIdx.x], sUsed[threadIdx.x]);
}

__global__ void __launch_bounds__(VXB_THREADS) vxb_triangle_kernel(const VxbDev d)
{
	if (vxb_overflowed(d)) return;
	const unsigned total = d.counters->cells;
	for (unsigned ci = d.counters->splitCells + blockIdx.x * blockDim.x + threadIdx.x; ci < total; ci += gridDim.x * blockDim.x)
	{
		const uint4 crv = *reinterpret_cast<const uint4*>(&d.cellRecs[ci]);
		const unsigned slot = d.cellBlock[ci];
		const VxbBlockRec* br = &d.blockRecs[slot];
		const unsigned voff = br->voff, ioff = br->ioff, cellBase = br->cellBase;
		const unsigned int* nt32 = d.ntScratch + (size_t)br->emitIdx * 256;
		const unsigned int* wpre = nt32 + 128;
		const int c = crv.x & 0xFFF;
		const unsigned code = (crv.x >> 12) & 0xFF, zm = (crv.x >> 20) & 0xFF;
		const unsigned cls = vxbGRegularCellClass[code];
		const unsigned char* cd = &vxbGRegularCellData[cls * 16];
		const unsigned geo = cd[0];
		const unsigned newMask = crv.z & 0xFFF;
		// block-local vertex ids (< 49152) as 16-bit halves of six registers: a table-indexed array would live in local memory
		unsigned w[6] = { 0u, 0u, 0u, 0u, 0u, 0u };
		unsigned nextNew = crv.w & 0xFFFF;
		const int nv = (int)(geo >> 4);
#pragma unroll
		for (int k = 0; k < 12; ++k)
		{
			if (k < nv) // (no break: the loop must unroll completely for w[] to stay in registers)
			{
				unsigned vid;
				if ((newMask >> k) & 1u) vid = nextNew++;
				else
				{
					const VxbVertexDesc vd = vxb_regular_vertex_desc_lite(vxbGRegularVertexData[code * 12 + k], zm);
					const int oc = c - (vd.dir & 1) - ((vd.dir >> 1) & 1) * 16 - ((vd.dir >> 2) & 1) * 256; // reused => the owner exists
					const unsigned oi = vxb_rank_of(nt32, wpre, oc);
					const uint4 orec = *reinterpret_cast<const uint4*>(&d.cellRecs[cellBase + oi]);
					const unsigned ok = (orec.y >> (16 + 4 * vd.slot)) & 0xF;
					vid = (orec.w & 0xFFFF) + __popc(orec.z & 0xFFFu & ((1u << ok) - 1u));
				}
				w[k >> 1] |= vid << ((k & 1) * 16);
			}
		}
		auto vidOf = [&](unsigned k) -> unsigned {
			const unsigned i = k >> 1;
			const unsigned pair = i == 0 ? w[0] : i == 1 ? w[1] : i == 2 ? w[2] : i == 3 ? w[3] : i == 4 ? w[4] : w[5];
			return (k & 1u) ? (pair >> 16) : (pair & 0xFFFFu);
		};
		unsigned* out = d.idx + ioff + (crv.w >> 16) * 3;
		unsigned removed = 0;
		// A level-0 cell without a zero sample has every table vertex strictly inside a distinct cell edge (t in 1..255):
		// no two coincide and no three are collinear, and with |coordinates differences| <= 256 the reference's float cross
		// product is exact, so its degenerate test (:1309-1311) cannot fire - the positions need not be read back.
		const bool cannotDegenerate = (br->packed >> 28) == 0u && zm == 0u;
		for (unsigned tr = 0; tr < (geo & 0xF); ++tr, out += 3)
		{
			const unsigned a = vidOf(cd[1 + tr * 3]), b = vidOf(cd[2 + tr * 3]), cc = vidOf(cd[3 + tr * 3]);
			bool kept = true;
			if (!cannotDegenerate)
			{
				const float* fa = d.verts[voff + a].pos; const float* fb = d.verts[voff + b].pos; const float* fc = d.verts[voff + cc].pos;
				// back to grid axes, x256 (exact: positions are multiples of 1/256)
				const float pa[3] = { fa[0] * 256.f, fa[2] * 256.f, fa[1] * 256.f };
				const float pb[3] = { fb[0] * 256.f, fb[2] * 256.f, fb[1] * 256.f };
				const float pc[3] = { fc[0] * 256.f, fc[2] * 256.f, fc[1] * 256.f };
				kept = vxb_triangle_kept(pa, pb, pc);
			}
			if (kept) { out[0] = a; out[1] = b; out[2] = cc; }
			else { out[0] = 0xFFFFFFFFu; out[1] = 0xFFFFFFFFu; out[2] = 0xFFFFFFFFu; ++removed; }
		}
		if (removed) atomicAdd(&d.blockRecs[slot].removed, removed);
	}
}

// per emitted block: compaction of the triangle list where degenerate triangles were removed + the directory record
__global__ void __launch_bounds__(VXB_THREADS) vxb_finish_kernel(const VxbDev d)
{
	__shared__ unsigned sWarp[8];
	__shared__ unsigned sItem;
	if (vxb_overflowed(d)) return;
	const int tid = threadIdx.x;
	const unsigned count = d.counters->records;
	unsigned statRemoved = 0;
	for (;;)
	{
		if (tid == 0) sItem = atomicAdd(&d.counters->finishCursor, VXB_THREADS);
		__syncthreads();
		const unsigned first = sItem;
		if (first >= count) break;
		// fast path: one thread per block writes the record when nothing was removed
		const unsigned slot = first + tid;
		unsigned removed = 0;
		if (slot < count) removed = d.blockRecs[slot].removed;
		const unsigned anyRemoved = __syncthreads_or(removed != 0);
		if (anyRemoved)
		{
			for (unsigned q = 0; q < VXB_THREADS && first + q < count; ++q) // block-uniform loop
			{
				const VxbBlockRec* br = &d.blockRecs[first + q];
				if (!br->removed) continue;
				const unsigned ntris = br->ntris, ioff = br->ioff;
				unsigned written = 0;
				for (unsigned t0 = 0; t0 < ntris; t0 += VXB_THREADS)
				{
					const unsigned t = t0 + tid;
					unsigned a = 0xFFFFFFFFu, b = 0, cc = 0;
					if (t < ntris) { const unsigned* in = d.idx + ioff + t * 3; a = in[0]; b = in[1]; cc = in[2]; }
					const bool keep = (t < ntris) && a != 0xFFFFFFFFu;
					unsigned chunkTotal;
					const unsigned pos = vxb_block_scan(keep ? 1u : 0u, sWarp, chunkTotal);
					if (keep) { unsigned* out = d.idx + ioff + (written + pos) * 3; out[0] = a; out[1] = b; out[2] = cc; }
					written += chunkTotal;
					__syncthreads();
				}
			}
		}
		if (slot < count)
		{
			const VxbBlockRec br = d.blockRecs[slot];
			vxb_block_record r;
			const int level = (int)(br.packed >> 28);
			const unsigned coordId = br.packed & 0x0FFFFFFFu;
			r.level = level; r.coord_id = coordId; r.id = vxb_block_id(d, level, coordId);
			r.vertex_count = br.nverts; r.index_count = (br.ntris - br.removed) * 3;
			r.vertex_offset = br.voff; r.index_offset = br.ioff;
			for (int f = 0; f < 6; ++f)
			{
				// internal face order (z-,y-,x-,z+,y+,x+) is already the output enum order (YNeg,ZNeg,XNeg,YPos,ZPos,XPos)
				r.trans_vertex_count[f] = br.tvcount[f]; r.trans_index_count[f] = br.ticount[f];
				r.trans_vertex_offset[f] = br.tvcount[f] ? br.tvoff[f] : 0u; r.trans_index_offset[f] = br.ticount[f] ? br.tioff[f] : 0u;
			}
			r.reserved = 0;
			d.records[slot] = r;
			statRemoved += br.removed;
		}
		__syncthreads();
	}
	if (statRemoved) atomicAdd(&d.counters->degenerate, statRemoved);
}

// ------------------------------------------------------------------------------------------------
// transition cells (:1754-2131).  Work item = ONE FACE of one emitted mid-level block (the reference numbers the vertices
// of every face from zero - TransitionVertices[face], :1293 - so the six faces of a block are independent): a 64-thread
// CTA stages the face's 33 x 33 half-stride lattice, takes the 256 case codes, compacts the non-trivial cells and runs
// the slot / reuse / scan / emit passes over them.  cell = row * 16 + col.
// ------------------------------------------------------------------------------------------------
#define VXB_TR_THREADS 64
struct __align__(16) VxbTransSmem
{
	// per NON-TRIVIAL transition cell of the face, in the reference's serial order (row, col) = compact index
	unsigned long long slots[256]; // 10 owned-slot nibbles
	unsigned short cell[256];      // row * 16 + col
	unsigned short newMask[256];
	unsigned short vbase[256];     // new-vertex count, then its exclusive scan
	unsigned short tbase[256];     // triangle count, then its exclusive scan
	unsigned char mat[256];
	unsigned short code[256];      // per CELL (not compact): 9-bit transition case code, 0 = trivial
	signed char face[1092];        // the 33 x 33 half-stride sample lattice of the face plane (clamped reads)
	unsigned int nt[8];            // non-trivial bits, cell order
	unsigned int pre[9];           // exclusive prefix of popc(nt): compact index base of each word
	unsigned int warpSums[8];
	unsigned int tvoff, tioff, tvcount, ticount;
	unsigned int item;
};

// the 13 samples of transition cell (row, col) from the staged lattice (:1867-1911)
__device__ __forceinline__ void vxb_face_cell_samples(const signed char* lattice, int row, int col, signed char v[13])
{
	const signed char* p = lattice + (2 * row) * 33 + 2 * col;
	v[0] = p[0]; v[1] = p[1]; v[2] = p[2];
	v[3] = p[33]; v[4] = p[34]; v[5] = p[35];
	v[6] = p[66]; v[7] = p[67]; v[8] = p[68];
	v[9] = v[0]; v[10] = v[2]; v[11] = v[6]; v[12] = v[8];
}

// sample i (0..12) of a transition cell straight from the staged lattice (p = the cell's first sample): no per-thread
// sample array, whose table-driven indexing would live in local memory
__device__ __forceinline__ int vxb_lattice_sample(const signed char* p, int i)
{
	const int off = (i < 9) ? (i / 3) * 33 + (i % 3) : ((i - 9) & 1) * 2 + ((i - 9) >> 1) * 66;
	return p[off];
}

__device__ __forceinline__ VxbTransVertexDesc vxb_lattice_vertex_desc(unsigned vd, const signed char* p)
{
	return vxb_transition_vertex_desc_ab(vd, vxb_lattice_sample(p, (vd >> 4) & 0xF), vxb_lattice_sample(p, vd & 0xF), vxbGTransitionCornerData);
}

__global__ void __launch_bounds__(VXB_TR_THREADS, 16) vxb_transition_kernel(const VxbDev d)
{
	__shared__ VxbTransSmem s;
	if (vxb_overflowed(d)) return;
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const VxbGrid g = d.grid;
	const unsigned workCount = d.counters->transBlocks * 6u;
	for (;;)
	{
		if (tid == 0) s.item = atomicAdd(&d.counters->transCursor, 1u);
		__syncthreads();
		const unsigned item = s.item;
		if (item >= workCount) break;
		const unsigned slot = d.transList[item / 6u];
		const int face = (int)(item % 6u);
		const unsigned packed = d.blockRecs[slot].packed;
		const int level = (int)(packed >> 28);
		const unsigned coordId = packed & 0x0FFFFFFFu;
		const int m = 1 << level, nb = d.n / 16 / m;
		const int bx = coordId % nb, by = (coordId / nb) % nb, bz = coordId / (nb * nb);
		int axis, ua, va;
		vxb_face_axes(face, axis, ua, va);
		const int bc = (axis == 0) ? bx : (axis == 1 ? by : bz);
		if (face < 3 ? (bc == 0) : (bc == nb - 1)) // no neighbour block inside the grid (:1829-1835): the face stays empty (the record was zeroed by vxb_block_kernel)
		{
			__syncthreads();
			continue;
		}

		// T0: stage the half-stride lattice of the face plane (clamped reads)
		{
			const int h = m >> 1, lim = d.n - 1;
			const int origin[3] = { bx * 16 * m, by * 16 * m, bz * 16 * m };
			const int f3 = face >= 3 ? face - 3 : face;
			const int off = (face >= 3) ? 16 * m : 0;
			if (level == 1 && f3 != 2)
			{
				// level 1: the lattice is the level-0 volume itself, so a row of a face normal to z or y is 33 CONTIGUOUS bytes
				// starting on a 32-byte boundary: two 16-byte loads + one byte instead of 33 sector-sized byte loads
				for (int q = tid; q < 33 * 3; q += VXB_TR_THREADS)
				{
					const int j = q / 3, part = q - j * 3;
					const int py = origin[1] + (f3 == 1 ? off : j), pz = origin[2] + (f3 == 0 ? off : j);
					const signed char* row = g.dist + ((size_t)min(pz, lim) * d.n + min(py, lim)) * d.n + origin[0];
					signed char* dst = &s.face[j * 33];
					if (part < 2)
					{
						const uint4 v = *reinterpret_cast<const uint4*>(row + part * 16);
						const unsigned w[4] = { v.x, v.y, v.z, v.w };
#pragma unroll
						for (int k = 0; k < 16; ++k) dst[part * 16 + k] = (signed char)(w[k >> 2] >> ((k & 3) * 8));
					}
					else dst[32] = row[min(32, lim - origin[0])];
				}
			}
			else
			{
				// vxb_face_axes: f3 = 0: axis z, (u, v) = (x, y); 1: axis y, (x, z); 2: axis x, (y, z); six independent loads in flight
				for (int idx0 = tid; idx0 < 1089; idx0 += 6 * VXB_TR_THREADS)
				{
					signed char v[6];
#pragma unroll
					for (int u = 0; u < 6; ++u)
					{
						const int r = min(idx0 + u * VXB_TR_THREADS, 1088);
						const int j = r / 33, i = r - j * 33;
						const int cu = i * h, cv = j * h;
						const int px = origin[0] + (f3 == 2 ? off : cu);
						const int py = origin[1] + (f3 == 1 ? off : (f3 == 0 ? cv : cu));
						const int pz = origin[2] + (f3 == 0 ? off : cv);
						v[u] = g.dist[((size_t)min(pz, lim) * d.n + min(py, lim)) * d.n + min(px, lim)];
					}
#pragma unroll
					for (int u = 0; u < 6; ++u)
					{
						const int r = idx0 + u * VXB_TR_THREADS;
						if (r < 1089) s.face[r] = v[u];
					}
				}
			}
		}
		__syncthreads();
		// T1: case code of every cell (cell order = the reference's row-major order)
		for (int c0 = tid; c0 < 256; c0 += VXB_TR_THREADS)
		{
			signed char v[13];
			vxb_face_cell_samples(s.face, c0 >> 4, c0 & 15, v);
			unsigned code = vxb_transition_case_code(v);
			if (code == 511u) code = 0;
			const unsigned bal = __ballot_sync(0xFFFFFFFFu, code != 0u);
			if (lane == 0) s.nt[c0 >> 5] = bal;
			s.code[c0] = (unsigned short)code;
		}
		__syncthreads();
		unsigned ntc;
		{
			const unsigned cnt = (tid < 8) ? __popc(s.nt[tid]) : 0u;
			const unsigned ex = vxb_block_scan(cnt, s.warpSums, ntc);
			if (tid < 8) s.pre[tid] = ex;
			if (tid == 0) s.pre[8] = ntc;
		}
		__syncthreads();
		if (tid == 0) { s.tvcount = 0; s.ticount = 0; s.tvoff = 0; s.tioff = 0; }
		if (ntc > 0) // block-uniform
		{
			// ordered compact list of the non-trivial cells
			for (int ci = tid; ci < 256; ci += VXB_TR_THREADS)
				if (s.code[ci]) s.cell[s.pre[ci >> 5] + __popc(s.nt[ci >> 5] & ((1u << (ci & 31)) - 1u))] = (unsigned short)ci;
			__syncthreads();
			// T2: owned slots + material, one thread per non-trivial cell
			for (unsigned i = tid; i < ntc; i += VXB_TR_THREADS)
			{
				const int ci = s.cell[i], row = ci >> 4, col = ci & 15;
				const unsigned code = s.code[ci];
				int local[3];
				local[axis] = (face >= 3) ? 15 : 0; local[ua] = col; local[va] = row;
				const signed char* lat = s.face + (2 * row) * 33 + 2 * col;
				unsigned long long slots = ~0ull;
				const int nv = vxbGTransitionCellData[(vxbGTransitionCellClass[code] & 0x7F) * 40] >> 4;
				for (int k = 0; k < nv; ++k)
				{
					const VxbTransVertexDesc td = vxb_lattice_vertex_desc(vxbGTransitionVertexData[code * 12 + k], lat);
					if (td.dir == 8) slots = (slots & ~(0xFull << (4 * td.slot))) | ((unsigned long long)k << (4 * td.slot)); // stored only when no reuse was attempted (:2097)
				}
				s.slots[i] = slots;
				s.mat[i] = (unsigned char)(d.cachePages[level][(size_t)coordId * 4096 + local[2] * 256 + local[1] * 16 + local[0]] & 0xFF);
			}
			__syncthreads();
			// T3: new-vs-reuse decisions (owner = previous row / previous column of the same face, :1958-1978)
			for (unsigned i = tid; i < ntc; i += VXB_TR_THREADS)
			{
				const int ci = s.cell[i], row = ci >> 4, col = ci & 15;
				const unsigned code = s.code[ci];
				const signed char* lat = s.face + (2 * row) * 33 + 2 * col;
				const unsigned geo = vxbGTransitionCellData[(vxbGTransitionCellClass[code] & 0x7F) * 40];
				const unsigned rowBits = (s.nt[ci >> 5] >> (ci & 16)) & 0xFFFFu;
				const int mask = ((row > 0) ? 2 : 0) | ((rowBits & ((1u << col) - 1u)) ? 1 : 0);
				const unsigned myMat = s.mat[i];
				unsigned newMask = 0;
				for (int k = 0; k < (int)(geo >> 4); ++k)
				{
					const VxbTransVertexDesc td = vxb_lattice_vertex_desc(vxbGTransitionVertexData[code * 12 + k], lat);
					bool isNew = true;
					if ((td.dir & mask) == td.dir)
					{
						const int oc = ci - ((td.dir >> 1) & 1) * 16 - (td.dir & 1);
						if ((s.nt[oc >> 5] >> (oc & 31)) & 1u)
						{
							const unsigned oi = s.pre[oc >> 5] + __popc(s.nt[oc >> 5] & ((1u << (oc & 31)) - 1u));
							const int ok = (int)((s.slots[oi] >> (4 * td.slot)) & 0xF);
							if (ok != VXB_NO_SLOT && s.mat[oi] == myMat) isNew = false;
						}
					}
					if (isNew) newMask |= 1u << k;
				}
				s.newMask[i] = (unsigned short)newMask;
				s.vbase[i] = (unsigned short)__popc(newMask);
				s.tbase[i] = (unsigned short)(geo & 0xF);
			}
			__syncthreads();
			// exclusive scan over the face's non-trivial cells (serial order)
			unsigned faceVerts, faceTris;
			{
				const unsigned per = (ntc + VXB_TR_THREADS - 1) / VXB_TR_THREADS;
				const unsigned i0 = min(tid * per, ntc), i1 = min(i0 + per, ntc);
				unsigned sv = 0, st = 0;
				for (unsigned i = i0; i < i1; ++i) { sv += s.vbase[i]; st += s.tbase[i]; }
				unsigned total;
				const unsigned base = vxb_block_scan(sv | (st << 16), s.warpSums, total);
				unsigned bv = base & 0xFFFF, bt = base >> 16;
				for (unsigned i = i0; i < i1; ++i)
				{
					const unsigned cv = s.vbase[i], ct = s.tbase[i];
					s.vbase[i] = (unsigned short)bv; s.tbase[i] = (unsigned short)bt;
					bv += cv; bt += ct;
				}
				faceVerts = total & 0xFFFF; faceTris = total >> 16;
			}
			if (tid == 0)
			{
				s.tvcount = faceVerts; s.ticount = faceTris * 3;
				s.tvoff = faceVerts ? atomicAdd(&d.counters->transVertices, faceVerts) : 0u;
			}
			if (tid == 32) s.tioff = faceTris ? atomicAdd(&d.counters->transIndices, faceTris * 3) : 0u;
			__syncthreads();
			// T4: indices + the vertex work list
			const unsigned tvoff = s.tvoff, tioff = s.tioff;
			const bool fits = (unsigned long long)tvoff + faceVerts <= d.tvcap && (unsigned long long)tioff + faceTris * 3ull <= d.ticap;
			for (unsigned i = tid; fits && i < ntc; i += VXB_TR_THREADS)
			{
				const int ci = s.cell[i], row = ci >> 4, col = ci & 15;
				const unsigned code = s.code[ci];
				const signed char* lat = s.face + (2 * row) * 33 + 2 * col;
				const unsigned cls = vxbGTransitionCellClass[code];
				const unsigned char* cd = &vxbGTransitionCellData[(cls & 0x7F) * 40];
				const int nv = cd[0] >> 4, ntri = cd[0] & 0xF;
				const unsigned newMask = s.newMask[i];
				unsigned vids[12];
				unsigned nextNew = s.vbase[i];
				for (int k = 0; k < nv; ++k)
				{
					if ((newMask >> k) & 1u)
					{
						// the vertex itself is computed by vxb_transition_vertex_kernel, one thread per entry
						d.tvlist[tvoff + nextNew] = make_uint2(slot, (code << 16) | ((unsigned)face << 12) | ((unsigned)ci << 4) | (unsigned)k);
						vids[k] = nextNew++;
					}
					else
					{
						const VxbTransVertexDesc td = vxb_lattice_vertex_desc(vxbGTransitionVertexData[code * 12 + k], lat);
						const int oc = ci - ((td.dir >> 1) & 1) * 16 - (td.dir & 1);
						const unsigned oi = s.pre[oc >> 5] + __popc(s.nt[oc >> 5] & ((1u << (oc & 31)) - 1u));
						const unsigned ok = (unsigned)((s.slots[oi] >> (4 * td.slot)) & 0xF);
						vids[k] = (unsigned)s.vbase[oi] + __popc((unsigned)s.newMask[oi] & ((1u << ok) - 1u));
					}
				}
				const bool flip = (((cls >> 7) & 1u) ^ (unsigned)(face & 1)) != 0;
				unsigned* out = d.tidx + tioff + (unsigned)s.tbase[i] * 3;
				for (int tr = 0; tr < ntri; ++tr)
				{
					const unsigned a = vids[cd[1 + tr * 3]], b = vids[cd[2 + tr * 3]], cc = vids[cd[3 + tr * 3]];
					out[tr * 3] = a; out[tr * 3 + 1] = flip ? cc : b; out[tr * 3 + 2] = flip ? b : cc;
				}
			}
		}
		__syncthreads();
		if (tid == 0)
		{
			VxbBlockRec* br = &d.blockRecs[slot];
			br->tvoff[face] = s.tvoff; br->tioff[face] = s.tioff; br->tvcount[face] = s.tvcount; br->ticount[face] = s.ticount;
		}
		__syncthreads();
	}
}

// flat: one thread per new transition vertex (:1980-2092)
__global__ void __launch_bounds__(VXB_THREADS, VXB_FLAT_OCC) vxb_transition_vertex_kernel(const VxbDev d)
{
	__shared__ unsigned sUsed[8];
	if (threadIdx.x < 8) sUsed[threadIdx.x] = 0;
	__syncthreads();
	if (!vxb_overflowed(d) && d.counters->transVertices <= d.tvcap && d.counters->transIndices <= d.ticap)
	{
		const VxbGrid g = d.grid;
		const unsigned total = d.counters->transVertices;
		for (unsigned j = blockIdx.x * blockDim.x + threadIdx.x; j < total; j += gridDim.x * blockDim.x)
		{
			const uint2 e = d.tvlist[j];
			const unsigned packed = d.blockRecs[e.x].packed;
			const int level = (int)(packed >> 28);
			const unsigned coordId = packed & 0x0FFFFFFFu;
			const int m = 1 << level, nb = d.n / 16 / m;
			const int bx = coordId % nb, by = (coordId / nb) % nb, bz = coordId / (nb * nb);
			const int face = (int)((e.y >> 12) & 7), cell = (int)((e.y >> 4) & 0xFF), k = (int)(e.y & 15);
			const unsigned code = e.y >> 16; // the cell's 9-bit case code, known to vxb_transition_kernel
			const int row = cell >> 4, col = cell & 15;
			int axis, ua, va;
			vxb_face_axes(face, axis, ua, va);
			int local[3];
			local[axis] = (face >= 3) ? 15 : 0; local[ua] = col; local[va] = row;
			const int base[3] = { (bx * 16 + local[0]) * m, (by * 16 + local[1]) * m, (bz * 16 + local[2]) * m };
			// only the two samples at the ends of the vertex's edge are needed
			const unsigned vd = vxbGTransitionVertexData[code * 12 + k];
			int pa[3], pb[3];
			vxb_transition_sample_pos(face, level, base, (vd >> 4) & 0xF, pa);
			vxb_transition_sample_pos(face, level, base, vd & 0xF, pb);
			const VxbTransVertexDesc td = vxb_transition_vertex_desc_ab(vd, vxb_dist(g, pa[0], pa[1], pa[2]), vxb_dist(g, pb[0], pb[1], pb[2]), vxbGTransitionCornerData);
			const unsigned ent = d.cachePages[level][(size_t)coordId * 4096 + local[2] * 256 + local[1] * 16 + local[0]];
			const unsigned matId = ent & 0xFF, matBlend = ent >> 8;
			VxbRawVertex rv;
			vxb_transition_vertex(g, face, level, base, local, td, matId, matBlend, rv);
			VxbVertex ov;
			vxb_finish_vertex(rv, *d.lut, ov);
			vxb_store_vertex(d.tverts + j, ov);
			atomicOr(&sUsed[matId >> 5], 1u << (matId & 31));
		}
	}
	__syncthreads();
	if (threadIdx.x < 8 && sUsed[threadIdx.x]) atomicOr(&d.counters->usedMaterials[threadIdx.x], sUsed[threadIdx.x]);
}
