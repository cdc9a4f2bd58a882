// Consumer-side packaging (SURVEY.md section 8 f4): the result stays in HBM and is handed to a renderer as indirect draws.
// The arenas already are merged vertex / index buffers (every block a contiguous range, indices block-local), so a
// draw of a block is {index_count, first_index, base_vertex}.  What the renderer contract of the reference adds
// (doc_source/Rendering.md:18-58) is per frame: WHICH blocks to draw (a cut through the LOD octree: finer near the
// camera), for each drawn block of level > 0 which of its six faces border a finer-level neighbour - there the block's
// transition mesh is drawn and the vertex shader swaps in the secondary position of the vertices whose mask
// (SecondaryPosition.w) is covered by that face set (`blockAdj`, Rendering.md:44-52).
#pragma once

struct VxbLodArgs
{
	float camera[3];      // output (Y-up) coordinates, like the vertices
	float lod;            // the cut's parameter: base_distance (VxbCentreCut) or lod_factor (VxbBoxCut)
	unsigned int* counts; // [0] regular draws, [1] transition draws
	vxb_draw_command* regular; vxb_draw_info* regularInfo;
	vxb_draw_command* transition; vxb_draw_info* transitionInfo;
	unsigned int capacity; // entries of each list
};

// does the octree node (level, grid block coordinates) stop the descent?  (the top level always does)
__device__ __forceinline__ bool vxb_lod_stops(const VxbDev& d, const VxbLodArgs& a, int level, int bx, int by, int bz)
{
	if (level == d.lastLevel) return true;
	const float m = (float)(16 << level);
	// node centre in output axes: (x, z, y) (:1289-1291)
	const float cx = ((float)bx + 0.5f) * m, cy = ((float)bz + 0.5f) * m, cz = ((float)by + 0.5f) * m;
	const float dx = cx - a.camera[0], dy = cy - a.camera[1], dz = cz - a.camera[2];
	const float dist2 = (dx * dx + dy * dy) + dz * dz;
	const float lim = a.lod * (float)(1 << level);
	return dist2 >= lim * lim;
}

// is the node part of the cut: it stops and every ancestor descends
__device__ __forceinline__ bool vxb_lod_selected(const VxbDev& d, const VxbLodArgs& a, int level, int bx, int by, int bz)
{
	if (level > 0 && !vxb_lod_stops(d, a, level, bx, by, bz)) return false; // level 0 cannot descend further
	for (int l = level + 1; l <= d.lastLevel; ++l)
		if (vxb_lod_stops(d, a, l, bx >> (l - level), by >> (l - level), bz >> (l - level))) return false;
	return true;
}

// is the region of node (level, b) drawn with FINER blocks: the node descends and so does every ancestor
__device__ __forceinline__ bool vxb_lod_finer(const VxbDev& d, const VxbLodArgs& a, int level, int bx, int by, int bz)
{
	for (int l = level; l <= d.lastLevel; ++l)
		if (vxb_lod_stops(d, a, l, bx >> (l - level), by >> (l - level), bz >> (l - level))) return false;
	return level > 0;
}

// which faces of the block border a region drawn finer (bit f in the output enum order = internal order z-, y-, x-, z+, y+, x+
// of vxb_finish_kernel); level 0 has none
__device__ __forceinline__ unsigned vxb_lod_block_adj(const VxbDev& d, const VxbLodArgs& a, int level, int nb, int bx, int by, int bz)
{
	unsigned adj = 0;
	if (level > 0)
	{
		const int dxyz[6][3] = { { 0, 0, -1 }, { 0, -1, 0 }, { -1, 0, 0 }, { 0, 0, 1 }, { 0, 1, 0 }, { 1, 0, 0 } };
		for (int f = 0; f < 6; ++f)
		{
			const int nx = bx + dxyz[f][0], ny = by + dxyz[f][1], nz = bz + dxyz[f][2];
			if (nx < 0 || ny < 0 || nz < 0 || nx >= nb || ny >= nb || nz >= nb) continue;
			if (vxb_lod_finer(d, a, level, nx, ny, nz)) adj |= 1u << f;
		}
	}
	return adj;
}

// the block's regular draw and the transition draws `adj` asks for, appended to a's lists
__device__ __forceinline__ void vxb_lod_emit(const VxbLodArgs& a, const vxb_block_record& r, unsigned adj)
{
	const unsigned k = atomicAdd(&a.counts[0], 1u);
	if (k < a.capacity)
	{
		vxb_draw_command c;
		c.index_count = r.index_count; c.instance_count = 1; c.first_index = r.index_offset; c.base_vertex = (int)r.vertex_offset; c.first_instance = k;
		a.regular[k] = c;
		vxb_draw_info inf;
		inf.block_id = r.id; inf.level = r.level; inf.block_adj = adj; inf.face = 0xFFFFFFFFu;
		a.regularInfo[k] = inf;
	}
	for (int f = 0; f < 6; ++f)
	{
		if (!((adj >> f) & 1u) || !r.trans_index_count[f]) continue;
		const unsigned t = atomicAdd(&a.counts[1], 1u);
		if (t >= a.capacity) continue;
		vxb_draw_command c;
		c.index_count = r.trans_index_count[f]; c.instance_count = 1; c.first_index = r.trans_index_offset[f]; c.base_vertex = (int)r.trans_vertex_offset[f]; c.first_instance = t;
		a.transition[t] = c;
		vxb_draw_info inf;
		inf.block_id = r.id; inf.level = r.level; inf.block_adj = adj; inf.face = (unsigned)f;
		a.transitionInfo[t] = inf;
	}
}

// one thread per emitted block (directory slot)
__global__ void __launch_bounds__(256) vxb_lod_select_kernel(const VxbDev d, const VxbLodArgs a, const unsigned int blockCount)
{
	const unsigned slot = blockIdx.x * blockDim.x + threadIdx.x;
	if (slot >= blockCount) return;
	const vxb_block_record r = d.records[slot];
	const int level = (int)r.level, nb = (d.n >> 4) >> level;
	const int bx = r.coord_id % nb, by = (r.coord_id / nb) % nb, bz = r.coord_id / (nb * nb);
	if (!vxb_lod_selected(d, a, level, bx, by, bz)) return;
	vxb_lod_emit(a, r, vxb_lod_block_adj(d, a, level, nb, bx, by, bz));
}

// The same cut, culled against view frusta (include/vxb200.h "culled select").  Only the frustum differs between the views: the
// cut and block_adj are the LOD camera's in every one of them (a cut per view would draw different geometry in a shadow and
// a colour pass).  boxes: the mesh's per-block bounds, slot d.idBase[level] + coord_id, {min xyz, 0}, {max xyz, 0}.
struct VxbViews
{
	vxb_view view[VXB_VIEWS_MAX];
};

// does the box pass every plane of the view: the p-vertex test, float32 without fused multiply-add in the header's order
__device__ __forceinline__ bool vxb_view_sees(const vxb_view& v, const float4& lo, const float4& hi)
{
	bool in = true;
	for (int k = 0; k < 6; ++k)
	{
		const float nx = v.planes[k][0], ny = v.planes[k][1], nz = v.planes[k][2];
		const float cx = nx >= 0.f ? hi.x : lo.x, cy = ny >= 0.f ? hi.y : lo.y, cz = nz >= 0.f ? hi.z : lo.z;
		const float s = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(nx, cx), __fmul_rn(ny, cy)), __fmul_rn(nz, cz)), v.planes[k][3]);
		in = in && s >= 0.f;
	}
	return in;
}

// The two cut rules the views kernel is instantiated with: whether a block is on the cut, and its block_adj.
// VxbCentreCut: vxb_mesh_select_lod's (centre distance against a.lod = base_distance * 2^l, the top level always stops).
struct VxbCentreCut
{
	static __device__ __forceinline__ bool on_cut(const VxbDev& d, const VxbLodArgs& a, int level, int, int bx, int by, int bz)
	{
		return vxb_lod_selected(d, a, level, bx, by, bz);
	}
	static __device__ __forceinline__ unsigned block_adj(const VxbDev& d, const VxbLodArgs& a, int level, int nb, int bx, int by, int bz)
	{
		return vxb_lod_block_adj(d, a, level, nb, bx, by, bz);
	}
};

// VxbBoxCut: vxb_mesh_select_cut's (include/vxb200.h "the LOD cut"): a node is refined while the camera is closer than
// a.lod = lod_factor times its edge to its lattice box.  Refinement is monotone up the octree and the cut is balanced (the
// header's two arguments), so the cut test and block_adj are O(1): no walk over the ancestors.
struct VxbBoxCut
{
	// refine(l, b): float32 without fused multiply-add, in the header's order
	static __device__ __forceinline__ bool refines(const VxbLodArgs& a, int level, int bx, int by, int bz)
	{
		if (level == 0) return false;
		const float s = (float)(16 << level);
		// the lattice box in output axes (x, z, y); lo and hi are exact (integers below 2^24)
		const float lo[3] = { (float)bx * s, (float)bz * s, (float)by * s };
		float e[3];
		for (int i = 0; i < 3; ++i) e[i] = fmaxf(fmaxf(__fsub_rn(lo[i], a.camera[i]), __fsub_rn(a.camera[i], __fadd_rn(lo[i], s))), 0.f);
		const float dist2 = __fadd_rn(__fadd_rn(__fmul_rn(e[0], e[0]), __fmul_rn(e[1], e[1])), __fmul_rn(e[2], e[2]));
		const float lim = __fmul_rn(a.lod, s);
		return dist2 < __fmul_rn(lim, lim);
	}
	static __device__ __forceinline__ bool on_cut(const VxbDev& d, const VxbLodArgs& a, int level, int, int bx, int by, int bz)
	{
		return !refines(a, level, bx, by, bz) && (level == d.lastLevel || refines(a, level + 1, bx >> 1, by >> 1, bz >> 1));
	}
	// bit f (vxb_lod_block_adj's face order): the same-level neighbour across face f is inside the grid and refines
	static __device__ __forceinline__ unsigned block_adj(const VxbDev&, const VxbLodArgs& a, int level, int nb, int bx, int by, int bz)
	{
		unsigned adj = 0;
		if (level > 0)
		{
			const int dxyz[6][3] = { { 0, 0, -1 }, { 0, -1, 0 }, { -1, 0, 0 }, { 0, 0, 1 }, { 0, 1, 0 }, { 1, 0, 0 } };
			for (int f = 0; f < 6; ++f)
			{
				const int nx = bx + dxyz[f][0], ny = by + dxyz[f][1], nz = bz + dxyz[f][2];
				if (nx < 0 || ny < 0 || nz < 0 || nx >= nb || ny >= nb || nz >= nb) continue;
				if (refines(a, level, nx, ny, nz)) adj |= 1u << f;
			}
		}
		return adj;
	}
};

// one thread per directory slot; the Cut rule decides the cut and block_adj, view v appends to counts[2v], counts[2v + 1]
// and to its `stride` (regular) / 6 * stride (transition) entries of a's lists
template <class Cut>
__global__ void __launch_bounds__(256) vxb_lod_select_views_kernel(const VxbDev d, const VxbLodArgs a, const unsigned int blockCount,
	const __grid_constant__ VxbViews views, const unsigned int viewCount, const float4* __restrict__ boxes, const unsigned int stride)
{
	const unsigned slot = blockIdx.x * blockDim.x + threadIdx.x;
	if (slot >= blockCount) return;
	const vxb_block_record r = d.records[slot];
	const int level = (int)r.level, nb = (d.n >> 4) >> level;
	const int bx = r.coord_id % nb, by = (r.coord_id / nb) % nb, bz = r.coord_id / (nb * nb);
	if (!Cut::on_cut(d, a, level, nb, bx, by, bz)) return;
	const unsigned adj = Cut::block_adj(d, a, level, nb, bx, by, bz);
	const float4 lo = boxes[2 * (size_t)(d.idBase[level] + r.coord_id)], hi = boxes[2 * (size_t)(d.idBase[level] + r.coord_id) + 1];
	for (unsigned v = 0; v < viewCount; ++v)
	{
		if (!vxb_view_sees(views.view[v], lo, hi)) continue;
		VxbLodArgs av = a;
		av.counts += 2 * v;
		av.regular += (size_t)v * stride; av.regularInfo += (size_t)v * stride;
		av.transition += (size_t)v * stride * 6; av.transitionInfo += (size_t)v * stride * 6;
		vxb_lod_emit(av, r, adj);
	}
}
