// Ray casts against the drawn LOD cut of the resident mesh (include/vxb200.h "vxb_mesh_raycast_cut").
//
// The drawn set of vxb_mesh_select_cut's cut (VxbBoxCut, view culling aside): every cut node's regular triangles and the
// transition meshes its block_adj names, each vertex at the position the vertex shader selects (sec when its mask is
// non-zero and covered by block_adj, pos otherwise).  At levels >= 1 nothing proves that a drawn vertex stays inside its
// node's lattice box (vxb_lod_descent recomputes t from two samples that need not change sign), so the walk does not rest
// on the lattice box.  It rests on the mesh's measured boxes (the bounds: min / max of pos and sec over the regular and the
// transition vertices) and on the EXCURSION e, the largest distance by which any live block's measured box leaves its
// lattice box along an axis, measured once per apply (vxb_cutray_map_kernel, rounded up).  The walk is vxb_ray_walk_by over
// the level-0 block lattice, the grid box clipped grown by g = e + VXB_RAY_EPS (rounded up); the host refuses the cast
// when e + VXB_RAY_EPS > 15.
//
//   tested set   every cut node with a directory entry whose measured box grown by VXB_RAY_EPS (rounded outwards) meets the
//                clipped segment.  Every drawn vertex of the node is inside its measured box, so every drawn triangle is, and
//                an accepted hit lies within rounding of its triangle (as for the level-0 walk), so inside the grown box: no
//                accepted hit is lost.  The clip box holds every such box: a measured box lies within e of its lattice box,
//                which lies in the grid.
//   anchoring    a tested node is handled at the DDA cell whose interval [t0, t1) holds its grown-box entry te (the last cell's
//                interval is closed); the intervals partition the clipped segment, so te picks exactly one cell.  The ray
//                point at te lies in the node's grown measured box (up to rounding), hence within e + VXB_RAY_EPS <= 15 (+
//                rounding) < 16 of the node's lattice box along every axis, and inside the anchor cell (up to rounding; cell
//                indices clamped into the grid along an axis where the point lies outside it).  The lattice box is a run of
//                whole level-0 blocks along each axis, so along each axis a block of the node is at most one block away from
//                the anchor cell: one of the anchor cell's 27 neighbours lies inside the node.  The cut tiles the grid, so
//                that neighbour's covering cut node IS this node: lane k finds the covering node of neighbour k (refine from
//                the top down: by monotonicity the first node that does not refine is on the cut), looks its directory slot
//                up in the all-level map and tests the node's grown box.  Several lanes can reach one node in one cell; the
//                walk hands it on once (__match_any_sync, lowest lane).  So every tested node is handled exactly once.
//   stop         unchanged: te is two correctly rounded operations from a plane, the plane holds the grown box, and a hit
//                inside that box has t >= the true te.  A node not handled yet has te >= t1 of the current cell.
#pragma once

// The all-level map (bounds slot level_base[l] + coord_id -> directory slot, VXB_RAY_MISS where no block is, after a memset
// to 0xFF) and the excursion: per block max(0, lo_i - min_i, max_i - hi_i) over the three axes of its lattice box
// [lo, hi] and its measured box [min, max], rounded up; the largest one as float bits (non-negative floats order as their
// bits) in *excursion, which starts at 0.
struct VxbCutMapArgs
{
	unsigned levelBase[VXB_MAX_LEVELS];
	int nb;                    // level-0 blocks per axis
};

__global__ void __launch_bounds__(256) vxb_cutray_map_kernel(const vxb_block_record* __restrict__ dir, unsigned count, const VxbCutMapArgs a,
	const float4* __restrict__ boxes, unsigned* __restrict__ map, unsigned* __restrict__ excursion)
{
	const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
	float e = 0.f;
	if (i < count)
	{
		const unsigned level = __ldg(&dir[i].level), cid = __ldg(&dir[i].coord_id);
		const unsigned key = a.levelBase[level] + cid;
		map[key] = i;
		const int nb = a.nb >> level;
		const float s = (float)(16 << level);
		// the lattice box in output axes (x, z, y); exact
		const float lo[3] = { (float)(int)(cid % nb) * s, (float)(int)(cid / (nb * nb)) * s, (float)(int)((cid / nb) % nb) * s };
		const float4 mn = boxes[2 * (size_t)key], mx = boxes[2 * (size_t)key + 1];
		const float bmin[3] = { mn.x, mn.y, mn.z }, bmax[3] = { mx.x, mx.y, mx.z };
		for (int k = 0; k < 3; ++k) e = fmaxf(e, fmaxf(__fsub_ru(lo[k], bmin[k]), __fsub_ru(bmax[k], lo[k] + s)));
	}
	for (int o = 16; o > 0; o >>= 1) e = fmaxf(e, __shfl_xor_sync(0xFFFFFFFFu, e, o));
	if ((threadIdx.x & 31) == 0 && e > 0.f) atomicMax(excursion, __float_as_uint(e));
}

struct VxbCutRayMesh
{
	VxbRayMesh m;              // map: the all-level map; verts / idx: the regular arenas
	const VxbVertex* tverts;   // the transition arenas
	const unsigned* tidx;
	const float4* boxes;       // the measured boxes, 2 per bounds slot
	VxbCutMapArgs slots;       // level_base and nb
	int top;                   // the top level
	float grow;                // e + VXB_RAY_EPS, rounded up: the clip box's growth
	VxbLodArgs cut;            // camera and lod (lod_factor); the list pointers are unused
};

// the position of vertex vo + i the renderer draws under block_adj `adj`: sec when its mask is non-zero and covered by adj
VXB_FN float3 vxb_cut_vertex(const VxbVertex* verts, unsigned vo, unsigned i, unsigned adj)
{
	const VxbVertex* x = verts + vo + i;
	const unsigned mask = __float_as_uint(__ldg(&x->sec[3]));
	const float* p = (mask != 0u && (mask & adj) == mask) ? x->sec : x->pos;
	return make_float3(__ldg(p), __ldg(p + 1), __ldg(p + 2));
}

// One warp per ray, persistent over the batch.  Rays and hits in OUTPUT (Y-up) coordinates.  A lane's candidate key is
// part << 24 | triangle (part 0: the regular mesh, 1 + f: transition face f; a block holds fewer than 2^24 triangles), so
// vxb_ray_before and vxb_ray_winner order (t, slot, part, triangle) by the tie rule.
__global__ void __launch_bounds__(VXB_RAY_THREADS) vxb_raycast_cut_kernel(const VxbCutRayMesh c, const vxb_ray* __restrict__ rays, unsigned count,
	vxb_cut_hit* __restrict__ hits)
{
	const unsigned lane = threadIdx.x & 31;
	const unsigned warps = gridDim.x * (VXB_RAY_THREADS / 32);
	const VxbRayMesh& m = c.m;
	for (unsigned r = blockIdx.x * (VXB_RAY_THREADS / 32) + (threadIdx.x >> 5); r < count; r += warps)
	{
		const vxb_ray ray = rays[r];
		const float px = ray.origin[0], py = ray.origin[1], pz = ray.origin[2];
		const float dx = ray.direction[0], dy = ray.direction[1], dz = ray.direction[2];
		const float tMin = ray.t_min, tMax = ray.t_max;
		float bt = CUDART_INF_F, bu = 0.f, bv = 0.f;   // this lane's best hit
		unsigned bs = VXB_RAY_MISS, bk = VXB_RAY_MISS;
		// the triangles [0, tris) of one part of slot s, strided over the lanes
		auto part = [&](unsigned s, unsigned key, const VxbVertex* verts, const unsigned* idx, unsigned vo, unsigned io, unsigned tris, unsigned adj) {
			for (unsigned k = lane; k < tris; k += 32)
			{
				const unsigned* ip = idx + io + 3 * k;
				const float3 p0 = vxb_cut_vertex(verts, vo, __ldg(ip), adj);
				const float3 p1 = vxb_cut_vertex(verts, vo, __ldg(ip + 1), adj);
				const float3 p2 = vxb_cut_vertex(verts, vo, __ldg(ip + 2), adj);
				float t, u, v;
				if (vxb_ray_mt(px, py, pz, dx, dy, dz, tMin, tMax, p0, p1, p2, t, u, v) && vxb_ray_before(t, s, key | k, bt, bs, bk))
				{
					bt = t; bs = s; bk = key | k; bu = u; bv = v;
				}
			}
		};
		vxb_ray_walk_by<true>(m.nb, ray, c.grow, bt,
			[&](int bx, int by, int bz, float T0, float T1, float t0, float t1, bool last, unsigned& slot) {
				// the cut node over level-0 block (bx, by, bz): grid (x, y, z) = output (x, z, y)
				const int gx = bx, gy = bz, gz = by;
				int level = 0;
				for (int l = c.top; l > 0; --l)
					if (!VxbBoxCut::refines(c.cut, l, gx >> l, gy >> l, gz >> l)) { level = l; break; }
				const unsigned nbl = (unsigned)(m.nb >> level);
				const unsigned key = c.slots.levelBase[level] + ((unsigned)(gz >> level) * nbl + (unsigned)(gy >> level)) * nbl + (unsigned)(gx >> level);
				const unsigned s = __ldg(&m.map[key]);
				if (s == VXB_RAY_MISS) return false;
				const float4 lo = __ldg(&c.boxes[2 * (size_t)key]), hi = __ldg(&c.boxes[2 * (size_t)key + 1]);
				float te = T0, tx = T1;
				vxb_ray_slab(px, dx, __fsub_rd(lo.x, VXB_RAY_EPS), __fadd_ru(hi.x, VXB_RAY_EPS), te, tx);
				vxb_ray_slab(py, dy, __fsub_rd(lo.y, VXB_RAY_EPS), __fadd_ru(hi.y, VXB_RAY_EPS), te, tx);
				vxb_ray_slab(pz, dz, __fsub_rd(lo.z, VXB_RAY_EPS), __fadd_ru(hi.z, VXB_RAY_EPS), te, tx);
				if (!(te <= tx && te >= t0 && (te < t1 || last))) return false;
				slot = s;
				return true;
			},
			[&](const unsigned s) {
				const vxb_block_record* rec = m.dir + s;
				const int level = (int)__ldg(&rec->level);
				const unsigned cid = __ldg(&rec->coord_id);
				const int nbl = m.nb >> level;
				const unsigned adj = VxbBoxCut::block_adj(VxbDev(), c.cut, level, nbl, (int)(cid % nbl), (int)((cid / nbl) % nbl), (int)(cid / (nbl * nbl)));
				part(s, 0u, m.verts, m.idx, __ldg(&rec->vertex_offset), __ldg(&rec->index_offset), __ldg(&rec->index_count) / 3, adj);
				for (int f = 0; f < 6; ++f)
					if ((adj >> f) & 1u)
						part(s, (unsigned)(1 + f) << 24, c.tverts, c.tidx, __ldg(&rec->trans_vertex_offset[f]), __ldg(&rec->trans_index_offset[f]),
							__ldg(&rec->trans_index_count[f]) / 3, adj);
			});
		// ---- the winner by the tie rule; its lane writes the hit ----
		if (lane == vxb_ray_winner(bt, bs, bk))
		{
			vxb_cut_hit h;
			h.u = 0.f; h.v = 0.f; h.slot = VXB_RAY_MISS; h.block_id = 0; h.triangle = 0;
			h.t = CUDART_INF_F;
			h.position[0] = h.position[1] = h.position[2] = 0.f;
			h.normal[0] = h.normal[1] = h.normal[2] = 0.f;
			h.level = 0; h.face = 0;
			if (bs != VXB_RAY_MISS)
			{
				const vxb_block_record* rec = m.dir + bs;
				const unsigned p = bk >> 24, k = bk & 0xFFFFFFu;
				h.t = bt; h.u = bu; h.v = bv; h.slot = bs; h.block_id = __ldg(&rec->id); h.triangle = k;
				h.position[0] = px + bt * dx; h.position[1] = py + bt * dy; h.position[2] = pz + bt * dz;
				h.level = __ldg(&rec->level); h.face = p ? p - 1 : 0xFFFFFFFFu;
				if (p) vxb_blend_normal(c.tverts, __ldg(&rec->trans_vertex_offset[p - 1]), c.tidx + __ldg(&rec->trans_index_offset[p - 1]) + 3 * k, bu, bv, h.normal);
				else vxb_blend_normal(m.verts, __ldg(&rec->vertex_offset), m.idx + __ldg(&rec->index_offset) + 3 * k, bu, bv, h.normal);
			}
			hits[r] = h;
		}
	}
}
