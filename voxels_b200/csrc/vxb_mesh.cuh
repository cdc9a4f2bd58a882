// The device-resident mesh (include/vxb200.h "mesh"): a copy of the polygonized surface that outlives the context's
// result and is spliced on the GPU after every run, in the order the reference's PolygonMap keeps its blocks:
//   full run     the level lists are replaced by the run's blocks in (level, coord_id) order        (:395-401)
//   region run   per level, the blocks whose coordinates lie in the run's dirty range are erased      (:443-450)
//                and the re-created blocks are appended after the survivors in coord_id order        (:456-464, :1293)
// An apply is: count (survivors, new blocks, arena elements) -> radix sort of the new records by (level, coord_id) ->
// one exclusive scan over [mesh records | sorted new records] -> place (merged directory, destination offsets, copy
// jobs) -> copy (one CTA per block).  The directory is rewritten densely; the arenas keep the survivors in place and
// take the new blocks at their tail, or - when the tail would overflow or the garbage exceeds the live data - are
// compacted into the second arena set.
// Beside the directory the mesh keeps one box per (level, coord) slot - the sort key's slot space, so a survivor's box
// never moves: the exact bounds of the block's vertices (include/vxb200.h "bounds"), reduced by the copy of a new block.
#pragma once

#include <cub/cub.cuh>

// what an apply needs to know before it can place anything (the one device-to-host read of an apply)
struct VxbMeshCounts
{
	unsigned int survivors[VXB_MAX_LEVELS];   // mesh records kept, per level
	unsigned int fresh[VXB_MAX_LEVELS];       // records of the run, per level
	unsigned long long survivorElems[4];      // arena elements of the kept records: vertices, indices, trans v, trans i
	unsigned long long freshElems[4];         // (index ranges padded to a multiple of 4: every range starts 16-byte aligned)
	unsigned long long survivorRaw[4];        // the same without the padding (live totals)
	unsigned long long freshRaw[4];
};

// the scanned quantity of a record: one directory entry and its padded arena ranges
struct VxbMeshScan
{
	unsigned int n, v, i, tv, ti;
};

struct VxbMeshScanSum
{
	__device__ __forceinline__ VxbMeshScan operator()(const VxbMeshScan& a, const VxbMeshScan& b) const
	{
		VxbMeshScan s;
		s.n = a.n + b.n; s.v = a.v + b.v; s.i = a.i + b.i; s.tv = a.tv + b.tv; s.ti = a.ti + b.ti;
		return s;
	}
};

// the slot space of the sort key and, for a region apply, the dirty range of every level in grid (x, y, z) block units
struct VxbMeshRange
{
	int erase;                                     // 0: full apply (nothing survives)
	unsigned int levelBase[VXB_MAX_LEVELS];        // first (level, coord) slot of each level
	int lo[VXB_MAX_LEVELS][3], hi[VXB_MAX_LEVELS][3];
	int nb[VXB_MAX_LEVELS];
};

struct VxbMeshArenas
{
	VxbVertex* v; unsigned int* i; VxbVertex* tv; unsigned int* ti;
};

VXB_FN unsigned vxb_pad4(unsigned c) { return (c + 3u) & ~3u; }

VXB_FN VxbMeshScan vxb_mesh_item(const vxb_block_record& r)
{
	VxbMeshScan s;
	s.n = 1; s.v = r.vertex_count; s.i = vxb_pad4(r.index_count); s.tv = 0; s.ti = 0;
	for (int f = 0; f < 6; ++f) { s.tv += r.trans_vertex_count[f]; s.ti += vxb_pad4(r.trans_index_count[f]); }
	return s;
}

// the block's minimal corner lies in [min_dirty, max_dirty) of its level (:443-450), in block units
VXB_FN bool vxb_mesh_dirty(const VxbMeshRange& g, const vxb_block_record& r)
{
	const int l = (int)r.level, nb = g.nb[l];
	const int b[3] = { (int)(r.coord_id % nb), (int)((r.coord_id / nb) % nb), (int)(r.coord_id / (nb * nb)) };
	bool in = true;
	for (int a = 0; a < 3; ++a) in = in && b[a] >= g.lo[l][a] && b[a] < g.hi[l][a];
	return in;
}

// threads [0, meshCount): mesh records (survive or not); [meshCount, meshCount + runCount): the run's records (sort keys)
__global__ void __launch_bounds__(256) vxb_mesh_count_kernel(const vxb_block_record* __restrict__ mesh, unsigned meshCount,
	const vxb_block_record* __restrict__ run, unsigned runCount, const VxbMeshRange g, VxbMeshScan* __restrict__ items,
	unsigned* __restrict__ keys, unsigned* __restrict__ vals, VxbMeshCounts* __restrict__ counts)
{
	__shared__ unsigned sLevel[2][VXB_MAX_LEVELS];
	__shared__ unsigned long long sElems[2][6]; // [survivor | fresh][v, i, tv, ti padded; i, ti raw]
	if (threadIdx.x < 2 * VXB_MAX_LEVELS) (&sLevel[0][0])[threadIdx.x] = 0;
	if (threadIdx.x < 12) (&sElems[0][0])[threadIdx.x] = 0;
	__syncthreads();
	const unsigned t = blockIdx.x * blockDim.x + threadIdx.x;
	unsigned e[6] = { 0, 0, 0, 0, 0, 0 };
	bool fresh = false;
	if (t < meshCount + runCount)
	{
		fresh = t >= meshCount;
		const vxb_block_record r = fresh ? run[t - meshCount] : mesh[t];
		VxbMeshScan s = vxb_mesh_item(r);
		bool counted = true;
		if (fresh) { keys[t - meshCount] = g.levelBase[r.level] + r.coord_id; vals[t - meshCount] = t - meshCount; }
		else
		{
			counted = !vxb_mesh_dirty(g, r);
			if (!counted) { s.n = 0; s.v = 0; s.i = 0; s.tv = 0; s.ti = 0; }
			items[t] = s;
		}
		if (counted)
		{
			atomicAdd(&sLevel[fresh ? 1 : 0][r.level], 1u);
			e[0] = s.v; e[1] = s.i; e[2] = s.tv; e[3] = s.ti; e[4] = r.index_count;
			for (int f = 0; f < 6; ++f) e[5] += r.trans_index_count[f];
		}
	}
	// per warp and kind (a warp can straddle the boundary between mesh and run records), then one shared add per lane 0
	for (int k = 0; k < 2; ++k)
		for (int a = 0; a < 6; ++a)
		{
			const unsigned sum = __reduce_add_sync(0xFFFFFFFFu, (fresh == (k == 1)) ? e[a] : 0u);
			if ((threadIdx.x & 31) == 0 && sum) atomicAdd(&sElems[k][a], (unsigned long long)sum);
		}
	__syncthreads();
	if (threadIdx.x < VXB_MAX_LEVELS)
	{
		if (sLevel[0][threadIdx.x]) atomicAdd(&counts->survivors[threadIdx.x], sLevel[0][threadIdx.x]);
		if (sLevel[1][threadIdx.x]) atomicAdd(&counts->fresh[threadIdx.x], sLevel[1][threadIdx.x]);
	}
	else if (threadIdx.x >= 32 && threadIdx.x < 48)
	{
		// vertex ranges are not padded: their raw totals are the padded ones
		const unsigned k = (threadIdx.x - 32) >> 3, raw = ((threadIdx.x - 32) >> 2) & 1, a = threadIdx.x & 3;
		const unsigned long long v = sElems[k][raw && (a & 1) ? 4 + (a >> 1) : a];
		unsigned long long* dst = k ? (raw ? counts->freshRaw : counts->freshElems) : (raw ? counts->survivorRaw : counts->survivorElems);
		if (v) atomicAdd(&dst[a], v);
	}
}

// the scan items of the run's records in sorted order, behind the mesh's
__global__ void __launch_bounds__(256) vxb_mesh_gather_kernel(const vxb_block_record* __restrict__ run, const unsigned* __restrict__ sorted,
	unsigned runCount, VxbMeshScan* __restrict__ items)
{
	const unsigned j = blockIdx.x * blockDim.x + threadIdx.x;
	if (j < runCount) items[j] = vxb_mesh_item(run[sorted[j]]);
}

VXB_FN void vxb_mesh_set_offsets(vxb_block_record& r, unsigned v, unsigned i, unsigned tv, unsigned ti)
{
	r.vertex_offset = v; r.index_offset = i;
	for (int f = 0; f < 6; ++f)
	{
		r.trans_vertex_offset[f] = tv; tv += r.trans_vertex_count[f];
		r.trans_index_offset[f] = ti; ti += vxb_pad4(r.trans_index_count[f]);
	}
}

// the merged directory: per level the survivors in mesh order, then the new blocks in (level, coord_id) order.
// compact = 0: survivors keep their ranges, new blocks go to tail[]; compact = 1: everything is laid out from 0
// (survivors first) in the other arena set.  A block to copy gets job `jobSrc` = its source (mesh slot, or run slot |
// 0x80000000) and `jobDst` = its slot in the merged directory.
__global__ void __launch_bounds__(256) vxb_mesh_place_kernel(const vxb_block_record* __restrict__ mesh, unsigned meshCount,
	const vxb_block_record* __restrict__ run, const unsigned* __restrict__ sorted, unsigned runCount, const VxbMeshRange g,
	const VxbMeshScan* __restrict__ prefix, const VxbMeshCounts* __restrict__ counts, const uint4 tail, int compact,
	vxb_block_record* __restrict__ out, unsigned* __restrict__ jobSrc, unsigned* __restrict__ jobDst)
{
	const unsigned t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= meshCount + runCount) return;
	const bool fresh = t >= meshCount;
	vxb_block_record r = fresh ? run[sorted[t - meshCount]] : mesh[t];
	if (!fresh && vxb_mesh_dirty(g, r)) return;
	const int level = (int)r.level;
	unsigned survivorsUpTo = 0, survivors = 0, freshBelow = 0;
	for (int l = 0; l < VXB_MAX_LEVELS; ++l)
	{
		survivors += counts->survivors[l];
		if (l <= level) survivorsUpTo += counts->survivors[l];
		if (l < level) freshBelow += counts->fresh[l];
	}
	const VxbMeshScan p = prefix[t];
	unsigned pos, job;
	if (!fresh)
	{
		pos = p.n + freshBelow;
		job = p.n;
		if (compact) vxb_mesh_set_offsets(r, p.v, p.i, p.tv, p.ti);
	}
	else
	{
		pos = survivorsUpTo + (p.n - survivors);
		job = compact ? p.n : p.n - survivors;
		if (compact) vxb_mesh_set_offsets(r, p.v, p.i, p.tv, p.ti);
		else
		{
			const VxbMeshScan b = prefix[meshCount]; // the survivors' totals
			vxb_mesh_set_offsets(r, tail.x + (p.v - b.v), tail.y + (p.i - b.i), tail.z + (p.tv - b.tv), tail.w + (p.ti - b.ti));
		}
	}
	out[pos] = r;
	if (fresh || compact) { jobSrc[job] = fresh ? (sorted[t - meshCount] | 0x80000000u) : t; jobDst[job] = pos; }
}

// vertices as 16-byte words (3 per 48-byte vertex); the third word of a vertex is {nrm.y, nrm.z, tex[0], tex[1]}: the
// unmapped-material marker of vxb_finish_vertex (tex[0] low byte 0xFF) becomes the reference's all-zero textures.
// bound: the thread's running min / max of pos[0..2] and sec[0..2] take in the words that pass through it: the first
// word of a vertex is {pos.x, pos.y, pos.z, sec.x}, the second starts with {sec.y, sec.z}
__device__ __forceinline__ void vxb_mesh_copy_vertices(const VxbVertex* src, VxbVertex* dst, unsigned count, int fixMarkers, bool bound,
	float (&lo)[3], float (&hi)[3])
{
	const uint4* s = reinterpret_cast<const uint4*>(src);
	uint4* d = reinterpret_cast<uint4*>(dst);
	for (unsigned k = threadIdx.x; k < 3 * count; k += blockDim.x)
	{
		uint4 w = __ldg(s + k);
		const unsigned part = k % 3;
		if (fixMarkers && part == 2 && (w.z & 0xFFu) == 0xFFu) { w.z = 0; w.w = 0; }
		d[k] = w;
		if (bound && part == 0)
		{
			const float x = __uint_as_float(w.x), y = __uint_as_float(w.y), z = __uint_as_float(w.z), sx = __uint_as_float(w.w);
			lo[0] = fminf(lo[0], fminf(x, sx)); hi[0] = fmaxf(hi[0], fmaxf(x, sx));
			lo[1] = fminf(lo[1], y); hi[1] = fmaxf(hi[1], y);
			lo[2] = fminf(lo[2], z); hi[2] = fmaxf(hi[2], z);
		}
		else if (bound && part == 1)
		{
			const float sy = __uint_as_float(w.x), sz = __uint_as_float(w.y);
			lo[1] = fminf(lo[1], sy); hi[1] = fmaxf(hi[1], sy);
			lo[2] = fminf(lo[2], sz); hi[2] = fmaxf(hi[2], sz);
		}
	}
}

__device__ __forceinline__ unsigned vxb_mesh_pick(const uint4& lo, const uint4& hi, unsigned i)
{
	const unsigned a = (i & 1) ? ((i & 2) ? lo.w : lo.y) : ((i & 2) ? lo.z : lo.x);
	const unsigned b = (i & 1) ? ((i & 2) ? hi.w : hi.y) : ((i & 2) ? hi.z : hi.x);
	return (i & 4) ? b : a;
}

// indices start at any word in the source and at a 16-byte boundary in the destination: every destination word
// k*4 .. k*4+3 is assembled from the (at most two) aligned source words that hold it; the padding words become 0
__device__ __forceinline__ void vxb_mesh_copy_indices(const unsigned* src, unsigned* dst, unsigned count)
{
	const unsigned r = (unsigned)(reinterpret_cast<uintptr_t>(src) >> 2) & 3u;
	const uint4* s = reinterpret_cast<const uint4*>(src - r);
	uint4* d = reinterpret_cast<uint4*>(dst);
	const unsigned vecs = (count + 3) >> 2;
	for (unsigned k = threadIdx.x; k < vecs; k += blockDim.x)
	{
		const uint4 lo = __ldg(s + k);
		const uint4 hi = (r && 4 * k + 4 - r < count) ? __ldg(s + k + 1) : lo;
		uint4 w;
		w.x = 4 * k + 0 < count ? vxb_mesh_pick(lo, hi, r + 0) : 0u;
		w.y = 4 * k + 1 < count ? vxb_mesh_pick(lo, hi, r + 1) : 0u;
		w.z = 4 * k + 2 < count ? vxb_mesh_pick(lo, hi, r + 2) : 0u;
		w.w = 4 * k + 3 < count ? vxb_mesh_pick(lo, hi, r + 3) : 0u;
		d[k] = w;
	}
}

// the box of a slot without a block: min > max
__device__ __forceinline__ void vxb_mesh_box_clear(float4* __restrict__ boxes, unsigned slot)
{
	const float inf = __int_as_float(0x7F800000);
	boxes[2 * (size_t)slot] = make_float4(inf, inf, inf, 0.f);
	boxes[2 * (size_t)slot + 1] = make_float4(-inf, -inf, -inf, 0.f);
}

// a full apply: every slot starts without a block
__global__ void __launch_bounds__(256) vxb_mesh_bounds_reset_kernel(float4* __restrict__ boxes, unsigned slots)
{
	const unsigned t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t < slots) vxb_mesh_box_clear(boxes, t);
}

// a region apply: the slots of the erased blocks
__global__ void __launch_bounds__(256) vxb_mesh_bounds_erase_kernel(const vxb_block_record* __restrict__ mesh, unsigned meshCount,
	const VxbMeshRange g, float4* __restrict__ boxes)
{
	const unsigned t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= meshCount) return;
	const vxb_block_record r = mesh[t];
	if (vxb_mesh_dirty(g, r)) vxb_mesh_box_clear(boxes, g.levelBase[r.level] + r.coord_id);
}

// the boxes in directory order, 6 floats per block (vxb_mesh_download_bounds)
__global__ void __launch_bounds__(256) vxb_mesh_bounds_gather_kernel(const vxb_block_record* __restrict__ mesh, unsigned meshCount,
	const __grid_constant__ vxb_mesh_bounds b, float* __restrict__ out)
{
	const unsigned t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= meshCount) return;
	const float* box = b.boxes + 8 * (size_t)(b.level_base[mesh[t].level] + mesh[t].coord_id);
	float* o = out + 6 * (size_t)t;
	o[0] = box[0]; o[1] = box[1]; o[2] = box[2]; o[3] = box[4]; o[4] = box[5]; o[5] = box[6];
}

// one CTA per job: the block's regular and transition vertices and indices from its source arenas (the mesh's other
// set for survivors of a compaction, the context's result for new blocks) to the ranges `out` gives it.  A new block's
// box is reduced from the vertices on their way through the registers and stored at its (level, coord) slot: keys[run
// slot], as the count kernel wrote it (the sort leaves its input as it was).  A survivor keeps the box it has.
__global__ void __launch_bounds__(128) vxb_mesh_copy_kernel(const unsigned* __restrict__ jobSrc, const unsigned* __restrict__ jobDst,
	const vxb_block_record* __restrict__ mesh, const vxb_block_record* __restrict__ run, const vxb_block_record* __restrict__ out,
	const VxbMeshArenas meshSrc, const VxbMeshArenas runSrc, const VxbMeshArenas dst, int fixMarkers,
	const unsigned* __restrict__ keys, float4* __restrict__ boxes)
{
	__shared__ float sBox[4][6];
	const unsigned src = jobSrc[blockIdx.x];
	const bool fresh = (src & 0x80000000u) != 0;
	const vxb_block_record& s = fresh ? run[src & 0x7FFFFFFFu] : mesh[src];
	const vxb_block_record& o = out[jobDst[blockIdx.x]];
	// pointers picked one by one: a reference to either parameter struct would put both on the stack
	const VxbVertex* v = fresh ? runSrc.v : meshSrc.v;
	const unsigned* i = fresh ? runSrc.i : meshSrc.i;
	const VxbVertex* tv = fresh ? runSrc.tv : meshSrc.tv;
	const unsigned* ti = fresh ? runSrc.ti : meshSrc.ti;
	const float inf = __int_as_float(0x7F800000);
	float lo[3] = { inf, inf, inf }, hi[3] = { -inf, -inf, -inf };
	vxb_mesh_copy_vertices(v + s.vertex_offset, dst.v + o.vertex_offset, s.vertex_count, fixMarkers, fresh, lo, hi);
	vxb_mesh_copy_indices(i + s.index_offset, dst.i + o.index_offset, s.index_count);
	for (int f = 0; f < 6; ++f)
	{
		vxb_mesh_copy_vertices(tv + s.trans_vertex_offset[f], dst.tv + o.trans_vertex_offset[f], s.trans_vertex_count[f], fixMarkers, fresh, lo, hi);
		vxb_mesh_copy_indices(ti + s.trans_index_offset[f], dst.ti + o.trans_index_offset[f], s.trans_index_count[f]);
	}
	if (!fresh) return; // the whole CTA
	// min and max are exact: the box does not depend on the order of this reduction
	for (int a = 0; a < 3; ++a)
		for (int sh = 16; sh; sh >>= 1)
		{
			lo[a] = fminf(lo[a], __shfl_xor_sync(0xFFFFFFFFu, lo[a], sh));
			hi[a] = fmaxf(hi[a], __shfl_xor_sync(0xFFFFFFFFu, hi[a], sh));
		}
	if ((threadIdx.x & 31) == 0)
		for (int a = 0; a < 3; ++a) { sBox[threadIdx.x >> 5][a] = lo[a]; sBox[threadIdx.x >> 5][3 + a] = hi[a]; }
	__syncthreads();
	if (threadIdx.x < 2)
	{
		// thread 0: min, thread 1: max, over the four warps
		const int b = 3 * threadIdx.x;
		float c[3];
		for (int a = 0; a < 3; ++a)
		{
			c[a] = sBox[0][b + a];
			for (int w = 1; w < 4; ++w) c[a] = threadIdx.x ? fmaxf(c[a], sBox[w][b + a]) : fminf(c[a], sBox[w][b + a]);
		}
		boxes[2 * (size_t)keys[src & 0x7FFFFFFFu] + threadIdx.x] = make_float4(c[0], c[1], c[2], 0.f);
	}
}
