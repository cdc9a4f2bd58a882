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
//
// Sphere sweeps against the cut (vxb_sphere_cast_cut_kernel) run the same walk with the clip box grown by e + r + VXB_RAY_EPS
// and every node's measured box by r + VXB_RAY_EPS (both rounded up); the host refuses e + r > 15:
//   tested set   a contact the sweep's tests accept puts the centre within r (+ rounding) of its drawn triangle, hence of the
//                node's measured box, hence inside that box grown by r + eps; a sweep that starts in contact has c(t_min)
//                there too, so the node's te is the clipped start.  The clip box holds every such box.
//   anchoring    the centre at te lies in the node's grown box (up to rounding), hence within e + r + eps <= 15 + 1/16 < 16
//                (+ rounding) of the node's lattice box along every axis.  The argument above then holds word for word: one
//                of the anchor cell's 27 neighbours lies inside the node, and its covering cut node is this node.
//   stop         unchanged: the grown box holds every contact's centre, and te is still two rounded operations from a plane.
// Closest points against the cut need no walk; their proof is with vxb_closest_point_cut_kernel.
//
// Capsules against the cut (vxb_capsule_cast_cut_kernel, vxb_closest_segment_cut_kernel).  The reach R' is r for sweeps and
// max_distance m for segments, and the shape's reach max_i |h_i| + R' travels with each query while e is the mesh's, so the
// rule is per query (vxb_capsule_cut_reach): e + (max_i |h_i| + R') <= 15 in float; a query that fails it is a miss.
//   sweeps       the walk above with the clip box grown by e + max_i |h_i| + r + VXB_RAY_EPS and every node's measured box by
//                max_i |h_i| + r + VXB_RAY_EPS (both rounded up).  A contact puts the centre within |h_i| + r (+ rounding) of
//                its drawn triangle along axis i (the capsule point paired with the contact is within r of it and within
//                |h_i| of the centre), hence inside the node's grown box; a sweep that starts in contact has c(t_min) there.
//                The centre at te then lies within e + max_i |h_i| + r + eps <= 15 + 1/16 < 16 (+ rounding) of the node's
//                lattice box along every axis, and the 27-neighbour argument of the ray cast holds word for word.  The
//                per-triangle reject in front of the capsule's tests is the level-0 kernel's (vxb_path_meets_box on the box
//                grown by |h_i| + r + eps); it never changes a result.
//   segments     as the closest points, with the per-axis gap: a closest pair within m puts the centre within |h_i| + m (+
//                rounding) of its drawn triangle along axis i, so of the node's measured box, and the node is kept when its
//                box lies within |h_i| + m + eps of the centre along every axis.  Its lattice box then lies within e +
//                max_i |h_i| + m + eps <= 15 + 1/16 < 16 of the centre along every axis: one of the 27 neighbours of the
//                centre's clamped block lies in it, and its covering cut node is it.
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
	float excursion;           // e itself, for the capsule queries' per-query reach (vxb_capsule_cut_reach); it fills the
	                           // padding before `cut`, so the layout the other cut kernels read is unchanged
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

// The cut node covering level-0 block (gx, gy, gz) (GRID axes): refined from the top down (by monotonicity the first node
// that does not refine is on the cut).  Its bounds slot goes to `key`; returns its directory slot from the all-level map
// (VXB_RAY_MISS where no block is).
VXB_FN unsigned vxb_cut_node(const VxbCutRayMesh& c, int gx, int gy, int gz, unsigned& key)
{
	int level = 0;
	for (int l = c.top; l > 0; --l)
		if (!VxbBoxCut::refines(c.cut, l, gx >> l, gy >> l, gz >> l)) { level = l; break; }
	const unsigned nbl = (unsigned)(c.m.nb >> level);
	key = c.slots.levelBase[level] + ((unsigned)(gz >> level) * nbl + (unsigned)(gy >> level)) * nbl + (unsigned)(gx >> level);
	return __ldg(&c.m.map[key]);
}

// The walk's candidate step for the cut (vxb_ray_walk_by's `cand`): the covering cut node of level-0 block (bx, by, bz)
// (OUTPUT axes), when it has a directory slot and its measured box grown by g (rounded outwards) has its entry te in the
// cell [t0, t1) (closed when `last`).  g = VXB_RAY_EPS for rays, r + VXB_RAY_EPS (rounded up) for sweeps.
VXB_FN bool vxb_cut_candidate(const VxbCutRayMesh& c, const vxb_ray& ray, float g, int bx, int by, int bz, float T0, float T1,
	float t0, float t1, bool last, unsigned& slot)
{
	unsigned key;
	const unsigned s = vxb_cut_node(c, bx, bz, by, key);   // grid (x, y, z) = output (x, z, y)
	if (s == VXB_RAY_MISS) return false;
	const float4 lo = __ldg(&c.boxes[2 * (size_t)key]), hi = __ldg(&c.boxes[2 * (size_t)key + 1]);
	float te = T0, tx = T1;
	vxb_ray_slab(ray.origin[0], ray.direction[0], __fsub_rd(lo.x, g), __fadd_ru(hi.x, g), te, tx);
	vxb_ray_slab(ray.origin[1], ray.direction[1], __fsub_rd(lo.y, g), __fadd_ru(hi.y, g), te, tx);
	vxb_ray_slab(ray.origin[2], ray.direction[2], __fsub_rd(lo.z, g), __fadd_ru(hi.z, g), te, tx);
	if (!(te <= tx && te >= t0 && (te < t1 || last))) return false;
	slot = s;
	return true;
}

// the block_adj the cut gives the cut node at directory record rec
VXB_FN unsigned vxb_cut_adj(const VxbCutRayMesh& c, const vxb_block_record* rec)
{
	const int level = (int)__ldg(&rec->level);
	const unsigned cid = __ldg(&rec->coord_id);
	const int nbl = c.m.nb >> level;
	return VxbBoxCut::block_adj(VxbDev(), c.cut, level, nbl, (int)(cid % nbl), (int)((cid / nbl) % nbl), (int)(cid / (nbl * nbl)));
}

// f(key, p0, p1, p2) for each drawn triangle of cut node s, strided over the lanes: its regular triangles, then the
// transition meshes of the faces its block_adj names, each vertex at the position vxb_cut_vertex selects.  key = part << 24 |
// triangle (part 0: the regular mesh, 1 + f: transition face f; a block holds fewer than 2^24 triangles), so that
// vxb_ray_before and vxb_ray_winner order (t, slot, part, triangle) by the tie rule.
template <class F>
VXB_FN void vxb_cut_triangles(const VxbCutRayMesh& c, const unsigned s, F&& f)
{
	const unsigned lane = threadIdx.x & 31;
	const vxb_block_record* rec = c.m.dir + s;
	const unsigned adj = vxb_cut_adj(c, rec);
	const auto part = [&](unsigned key, const VxbVertex* verts, const unsigned* idx, unsigned vo, unsigned io, unsigned tris) {
		for (unsigned k = lane; k < tris; k += 32)
		{
			const unsigned* ip = idx + io + 3 * k;
			const float3 p0 = vxb_cut_vertex(verts, vo, __ldg(ip), adj);
			const float3 p1 = vxb_cut_vertex(verts, vo, __ldg(ip + 1), adj);
			const float3 p2 = vxb_cut_vertex(verts, vo, __ldg(ip + 2), adj);
			f(key | k, p0, p1, p2);
		}
	};
	part(0u, c.m.verts, c.m.idx, __ldg(&rec->vertex_offset), __ldg(&rec->index_offset), __ldg(&rec->index_count) / 3);
	for (int x = 0; x < 6; ++x)
		if ((adj >> x) & 1u)
			part((unsigned)(1 + x) << 24, c.tverts, c.tidx, __ldg(&rec->trans_vertex_offset[x]), __ldg(&rec->trans_index_offset[x]),
				__ldg(&rec->trans_index_count[x]) / 3);
}

// One warp per ray, persistent over the batch.  Rays and hits in OUTPUT (Y-up) coordinates.
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
		vxb_ray_walk_by<true>(m.nb, ray, c.grow, bt,
			[&](int bx, int by, int bz, float T0, float T1, float t0, float t1, bool last, unsigned& slot) {
				return vxb_cut_candidate(c, ray, VXB_RAY_EPS, bx, by, bz, T0, T1, t0, t1, last, slot);
			},
			[&](const unsigned s) {
				vxb_cut_triangles(c, s, [&](unsigned key, const float3& p0, const float3& p1, const float3& p2) {
					float t, u, v;
					if (vxb_ray_mt(px, py, pz, dx, dy, dz, tMin, tMax, p0, p1, p2, t, u, v) && vxb_ray_before(t, s, key, bt, bs, bk))
					{
						bt = t; bs = s; bk = key; bu = u; bv = v;
					}
				});
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

// The winning triangle of a sweep or point hit: triangle key (part << 24 | k) of cut node rec, its part's vertices `verts`
// from vertex offset vo and its indices at ip (for vxb_blend_normal and vxb_cut_vertex).  Returns the hit's face field.
VXB_FN unsigned vxb_cut_hit_part(const VxbCutRayMesh& c, const vxb_block_record* rec, unsigned key, const VxbVertex*& verts,
	unsigned& vo, const unsigned*& ip)
{
	const unsigned p = key >> 24, k = key & 0xFFFFFFu;
	if (p)
	{
		verts = c.tverts; vo = __ldg(&rec->trans_vertex_offset[p - 1]); ip = c.tidx + __ldg(&rec->trans_index_offset[p - 1]) + 3 * k;
		return p - 1;
	}
	verts = c.m.verts; vo = __ldg(&rec->vertex_offset); ip = c.m.idx + __ldg(&rec->index_offset) + 3 * k;
	return 0xFFFFFFFFu;
}

// One warp per sweep, persistent over the batch: the cut walk with the clip box grown by e + r + VXB_RAY_EPS and every node's
// measured box by r + VXB_RAY_EPS (both rounded up; "sphere sweeps" at the top), the sphere sweep's tests (vxb_sweep_triangle)
// on the drawn triangles.  Sweeps and hits in OUTPUT (Y-up) coordinates.  (A minimum of one CTA per SM in the launch bounds:
// without it ptxas holds this kernel to 64 registers and spills.)
__global__ void __launch_bounds__(VXB_COLLIDE_THREADS, 1) vxb_sphere_cast_cut_kernel(const VxbCutRayMesh c, const float r,
	const vxb_ray* __restrict__ rays, unsigned count, vxb_sphere_cut_hit* __restrict__ hits)
{
	const unsigned lane = threadIdx.x & 31;
	const unsigned warps = gridDim.x * (VXB_COLLIDE_THREADS / 32);
	const float rr = r * r;
	const float g = __fadd_ru(r, VXB_RAY_EPS), clip = __fadd_ru(c.grow, r);
	for (unsigned q = blockIdx.x * (VXB_COLLIDE_THREADS / 32) + (threadIdx.x >> 5); q < count; q += warps)
	{
		const vxb_ray ray = rays[q];
		const float3 o = make_float3(ray.origin[0], ray.origin[1], ray.origin[2]);
		const float3 d = make_float3(ray.direction[0], ray.direction[1], ray.direction[2]);
		const float tMin = ray.t_min, tMax = ray.t_max;
		const float3 c0 = make_float3(o.x + tMin * d.x, o.y + tMin * d.y, o.z + tMin * d.z);
		const float dd = (d.x * d.x + d.y * d.y) + d.z * d.z;
		float bt = CUDART_INF_F;   // this lane's first contact
		unsigned bs = VXB_RAY_MISS, bk = VXB_RAY_MISS;
		bool bStarted = false;
		vxb_ray_walk_by<true>(c.m.nb, ray, clip, bt,
			[&](int bx, int by, int bz, float T0, float T1, float t0, float t1, bool last, unsigned& slot) {
				return vxb_cut_candidate(c, ray, g, bx, by, bz, T0, T1, t0, t1, last, slot);
			},
			[&](const unsigned s) {
				vxb_cut_triangles(c, s, [&](unsigned key, const float3& p0, const float3& p1, const float3& p2) {
					bool started;
					const float t = vxb_sweep_triangle(o, d, c0, r, rr, dd, tMin, tMax, p0, p1, p2, started);
					if (t < CUDART_INF_F && vxb_ray_before(t, s, key, bt, bs, bk)) { bt = t; bs = s; bk = key; bStarted = started; }
				});
			});
		if (lane == vxb_ray_winner(bt, bs, bk))
		{
			vxb_sphere_cut_hit h;
			h.t = CUDART_INF_F; h.slot = VXB_RAY_MISS; h.block_id = 0; h.triangle = 0;
			h.center[0] = h.center[1] = h.center[2] = 0.f;
			h.point[0] = h.point[1] = h.point[2] = 0.f;
			h.normal[0] = h.normal[1] = h.normal[2] = 0.f;
			h.u = 0.f; h.v = 0.f; h.flags = 0; h.level = 0; h.face = 0;
			if (bs != VXB_RAY_MISS)
			{
				const vxb_block_record* rec = c.m.dir + bs;
				const VxbVertex* verts;
				unsigned vo;
				const unsigned* ip;
				h.face = vxb_cut_hit_part(c, rec, bk, verts, vo, ip);
				const unsigned adj = vxb_cut_adj(c, rec);
				const float3 p0 = vxb_cut_vertex(verts, vo, __ldg(ip), adj);
				const float3 p1 = vxb_cut_vertex(verts, vo, __ldg(ip + 1), adj);
				const float3 p2 = vxb_cut_vertex(verts, vo, __ldg(ip + 2), adj);
				const float3 ct = make_float3(o.x + bt * d.x, o.y + bt * d.y, o.z + bt * d.z);
				float3 x;
				vxb_closest_on_triangle(ct, p0, p1, p2, x, h.u, h.v);
				h.t = bt; h.slot = bs; h.block_id = __ldg(&rec->id); h.triangle = bk & 0xFFFFFFu;
				h.center[0] = ct.x; h.center[1] = ct.y; h.center[2] = ct.z;
				h.point[0] = x.x; h.point[1] = x.y; h.point[2] = x.z;
				vxb_blend_normal(verts, vo, ip, h.u, h.v, h.normal);
				h.flags = bStarted ? VXB_SPHERE_STARTED_IN_CONTACT : 0u;
				h.level = __ldg(&rec->level);
			}
			hits[q] = h;
		}
	}
}

// One warp per query point, persistent over the batch.  Lane k < 27 takes neighbour k of the point's block clamped into the
// grid (vxb_point_candidate's arithmetic), finds that block's covering cut node and keeps it when the node's measured box is
// within max_distance + VXB_RAY_EPS of the point.  Lanes that reach the same node hand it on once (the lowest lane); the warp
// then tests each node's drawn triangles strided over the lanes.  Points and hits in OUTPUT (Y-up) coordinates.
//   every contributing node is a candidate   a drawn triangle within max_distance m of p (the test accepts it) is within m
//                   (+ rounding) of a point of the node's measured box, which holds every drawn vertex; the float box distance
//                   is within a few ulps of the true one, so the node is kept.  Its lattice box then lies within e + m + eps <=
//                   15 + 1/16 < 16 of p along every axis (the host refuses e + m > 15).  Along an axis where p lies inside the
//                   grid, the lattice box (a run of whole level-0 blocks) holds a block whose index is that of p's block +-1;
//                   where p lies outside, it holds the first or last block of the axis, the clamped index.  So one of the 27
//                   neighbours lies inside the node, and since the cut tiles the grid, that neighbour's covering node is it.
//   handled once    __match_any_sync over the lanes' slots, the lowest lane of each group hands the node on.
__global__ void __launch_bounds__(VXB_COLLIDE_THREADS) vxb_closest_point_cut_kernel(const VxbCutRayMesh c, const float maxDistance,
	const float* __restrict__ points, unsigned count, vxb_closest_cut_hit* __restrict__ hits)
{
	const unsigned lane = threadIdx.x & 31;
	const unsigned warps = gridDim.x * (VXB_COLLIDE_THREADS / 32);
	const float md2 = maxDistance * maxDistance, reach = maxDistance + VXB_RAY_EPS;
	const int nb = c.m.nb;
	for (unsigned q = blockIdx.x * (VXB_COLLIDE_THREADS / 32) + (threadIdx.x >> 5); q < count; q += warps)
	{
		const float3 p = make_float3(points[3 * q], points[3 * q + 1], points[3 * q + 2]);
		float bd = CUDART_INF_F, bu = 0.f, bv = 0.f;   // this lane's nearest triangle
		float3 bp = make_float3(0.f, 0.f, 0.f);
		unsigned bs = VXB_RAY_MISS, bk = VXB_RAY_MISS;
		unsigned slot = VXB_RAY_MISS;
		if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z) && lane < 27)
		{
			const float top = (float)(nb - 1);
			const int bx = (int)fminf(fmaxf(floorf(p.x * 0.0625f), 0.f), top) + (int)(lane % 3) - 1;
			const int by = (int)fminf(fmaxf(floorf(p.y * 0.0625f), 0.f), top) + (int)((lane / 3) % 3) - 1;
			const int bz = (int)fminf(fmaxf(floorf(p.z * 0.0625f), 0.f), top) + (int)(lane / 9) - 1;
			if (bx >= 0 && by >= 0 && bz >= 0 && bx < nb && by < nb && bz < nb)
			{
				unsigned key;
				const unsigned s = vxb_cut_node(c, bx, bz, by, key);   // grid (x, y, z) = output (x, z, y)
				if (s != VXB_RAY_MISS)
				{
					const float4 lo = __ldg(&c.boxes[2 * (size_t)key]), hi = __ldg(&c.boxes[2 * (size_t)key + 1]);
					const float gx = fmaxf(fmaxf(lo.x - p.x, p.x - hi.x), 0.f);
					const float gy = fmaxf(fmaxf(lo.y - p.y, p.y - hi.y), 0.f);
					const float gz = fmaxf(fmaxf(lo.z - p.z, p.z - hi.z), 0.f);
					if (VXB_SQRT((gx * gx + gy * gy) + gz * gz) <= reach) slot = s;
				}
			}
		}
		const unsigned peers = __match_any_sync(0xFFFFFFFFu, slot);   // every lane takes part
		vxb_warp_each(slot != VXB_RAY_MISS && (peers & ((1u << lane) - 1u)) == 0, slot, [&](const unsigned s) {
			vxb_cut_triangles(c, s, [&](unsigned key, const float3& p0, const float3& p1, const float3& p2) {
				float3 x;
				float u, v;
				vxb_closest_on_triangle(p, p0, p1, p2, x, u, v);
				const float d2 = vxb_dist2(p, x);
				if (d2 <= md2 && vxb_ray_before(d2, s, key, bd, bs, bk)) { bd = d2; bs = s; bk = key; bu = u; bv = v; bp = x; }
			});
		});
		if (lane == vxb_ray_winner(bd, bs, bk))
		{
			vxb_closest_cut_hit h;
			h.distance = CUDART_INF_F; h.slot = VXB_RAY_MISS; h.block_id = 0; h.triangle = 0;
			h.point[0] = h.point[1] = h.point[2] = 0.f;
			h.normal[0] = h.normal[1] = h.normal[2] = 0.f;
			h.u = 0.f; h.v = 0.f; h.level = 0; h.face = 0;
			if (bs != VXB_RAY_MISS)
			{
				const vxb_block_record* rec = c.m.dir + bs;
				const VxbVertex* verts;
				unsigned vo;
				const unsigned* ip;
				h.face = vxb_cut_hit_part(c, rec, bk, verts, vo, ip);
				h.distance = VXB_SQRT(bd); h.slot = bs; h.block_id = __ldg(&rec->id); h.triangle = bk & 0xFFFFFFu;
				h.point[0] = bp.x; h.point[1] = bp.y; h.point[2] = bp.z;
				h.u = bu; h.v = bv;
				vxb_blend_normal(verts, vo, ip, bu, bv, h.normal);
				h.level = __ldg(&rec->level);
			}
			hits[q] = h;
		}
	}
}

// The cut reach of a capsule query (include/vxb200.h "capsule queries against the drawn LOD cut"), in float for the host
// check and the kernels alike: the level-0 rule vxb_capsule_reach, then e + (max_i |h_i| + extra) <= 15; extra is the radius
// of a sweep or the max_distance of a segment, e the mesh's excursion.
VXB_HD bool vxb_capsule_cut_reach(const float3 h, float extra, float e)
{
	const float hm = fmaxf(fmaxf(fabsf(h.x), fabsf(h.y)), fabsf(h.z));
	return vxb_capsule_reach(h, extra) && e + (hm + extra) <= VXB_SPHERE_RADIUS_MAX;
}

// One warp per capsule sweep, persistent over the batch: the cut walk with the clip box grown by e + max_i |h_i| + r +
// VXB_RAY_EPS and every node's measured box by max_i |h_i| + r + VXB_RAY_EPS (both rounded up; "capsules" at the top), then
// on the drawn triangles the level-0 kernel's per-triangle reject and the capsule's tests (vxb_capsule_triangle).  A sweep
// out of cut reach is a miss.  Sweeps and hits in OUTPUT (Y-up) coordinates.  (Two CTAs per SM in the launch bounds: ptxas
// then fits the kernel in 127 registers without a stack frame or spills, the occupancy of vxb_capsule_cast_kernel; with one
// CTA per SM it takes 136 registers and runs slower, DESIGN.md section 6.)
__global__ void __launch_bounds__(VXB_COLLIDE_THREADS, 2) vxb_capsule_cast_cut_kernel(const VxbCutRayMesh c,
	const vxb_capsule_sweep* __restrict__ sweeps, unsigned count, vxb_capsule_cut_hit* __restrict__ hits)
{
	const unsigned lane = threadIdx.x & 31;
	const unsigned warps = gridDim.x * (VXB_COLLIDE_THREADS / 32);
	for (unsigned q = blockIdx.x * (VXB_COLLIDE_THREADS / 32) + (threadIdx.x >> 5); q < count; q += warps)
	{
		const vxb_capsule_sweep cs = sweeps[q];
		const vxb_ray& ray = cs.path;
		const float3 o = make_float3(ray.origin[0], ray.origin[1], ray.origin[2]);
		const float3 d = make_float3(ray.direction[0], ray.direction[1], ray.direction[2]);
		const float3 h = make_float3(cs.half_axis[0], cs.half_axis[1], cs.half_axis[2]);
		const float r = cs.radius, rr = r * r;
		const float tMin = ray.t_min, tMax = ray.t_max;
		const float3 c0 = make_float3(o.x + tMin * d.x, o.y + tMin * d.y, o.z + tMin * d.z);
		const float dd = (d.x * d.x + d.y * d.y) + d.z * d.z;
		const float3 g = make_float3(fabsf(h.x) + r + VXB_RAY_EPS, fabsf(h.y) + r + VXB_RAY_EPS, fabsf(h.z) + r + VXB_RAY_EPS);
		const float R = __fadd_ru(fmaxf(fmaxf(fabsf(h.x), fabsf(h.y)), fabsf(h.z)), r);
		const float gn = __fadd_ru(R, VXB_RAY_EPS), clip = __fadd_ru(c.grow, R);
		float bt = CUDART_INF_F;   // this lane's first contact
		unsigned bs = VXB_RAY_MISS, bk = VXB_RAY_MISS;
		bool bStarted = false;
		if (r > 0.f && vxb_capsule_cut_reach(h, r, c.excursion))   // the same for the whole warp
			vxb_ray_walk_by<true>(c.m.nb, ray, clip, bt,
				[&](int bx, int by, int bz, float T0, float T1, float t0, float t1, bool last, unsigned& slot) {
					return vxb_cut_candidate(c, ray, gn, bx, by, bz, T0, T1, t0, t1, last, slot);
				},
				[&](const unsigned s) {
					vxb_cut_triangles(c, s, [&](unsigned key, const float3& p0, const float3& p1, const float3& p2) {
						if (!vxb_path_meets_box(ray, g, p0, p1, p2)) return;
						bool started;
						const float t = vxb_capsule_triangle(o, d, c0, h, r, rr, dd, tMin, tMax, p0, p1, p2, started);
						if (t < CUDART_INF_F && vxb_ray_before(t, s, key, bt, bs, bk)) { bt = t; bs = s; bk = key; bStarted = started; }
					});
				});
		if (lane == vxb_ray_winner(bt, bs, bk))
		{
			vxb_capsule_cut_hit x;
			x.t = CUDART_INF_F; x.slot = VXB_RAY_MISS; x.block_id = 0; x.triangle = 0;
			x.center[0] = x.center[1] = x.center[2] = 0.f;
			x.point[0] = x.point[1] = x.point[2] = 0.f;
			x.axis_point[0] = x.axis_point[1] = x.axis_point[2] = 0.f;
			x.normal[0] = x.normal[1] = x.normal[2] = 0.f;
			x.u = 0.f; x.v = 0.f; x.s = 0.f; x.flags = 0; x.level = 0; x.face = 0;
			if (bs != VXB_RAY_MISS)
			{
				const vxb_block_record* rec = c.m.dir + bs;
				const VxbVertex* verts;
				unsigned vo;
				const unsigned* ip;
				x.face = vxb_cut_hit_part(c, rec, bk, verts, vo, ip);
				const unsigned adj = vxb_cut_adj(c, rec);
				const float3 p0 = vxb_cut_vertex(verts, vo, __ldg(ip), adj);
				const float3 p1 = vxb_cut_vertex(verts, vo, __ldg(ip + 1), adj);
				const float3 p2 = vxb_cut_vertex(verts, vo, __ldg(ip + 2), adj);
				const float3 ct = make_float3(o.x + bt * d.x, o.y + bt * d.y, o.z + bt * d.z);
				float3 pq, px;
				vxb_pair_fields(ct, h, p0, p1, p2, pq, px, x.u, x.v, x.s);
				x.point[0] = pq.x; x.point[1] = pq.y; x.point[2] = pq.z;
				x.axis_point[0] = px.x; x.axis_point[1] = px.y; x.axis_point[2] = px.z;
				x.t = bt; x.slot = bs; x.block_id = __ldg(&rec->id); x.triangle = bk & 0xFFFFFFu;
				x.center[0] = ct.x; x.center[1] = ct.y; x.center[2] = ct.z;
				vxb_blend_normal(verts, vo, ip, x.u, x.v, x.normal);
				x.flags = bStarted ? VXB_SPHERE_STARTED_IN_CONTACT : 0u;
				x.level = __ldg(&rec->level);
			}
			hits[q] = x;
		}
	}
}

// One warp per segment, persistent over the batch.  Lane k < 27 takes neighbour k of the centre's block clamped into the
// grid (vxb_point_candidate's arithmetic), finds that block's covering cut node and keeps it when the node's measured box
// lies within |h_i| + max_distance + VXB_RAY_EPS of the centre along every axis (the proof under "capsules" at the top).
// Lanes that reach the same node hand it on once (the lowest lane); the warp then runs the level-0 kernel's per-axis reject
// and the closest pair (vxb_segment_triangle) on each node's drawn triangles, strided over the lanes.  A segment out of cut
// reach is a miss.  OUTPUT (Y-up) coordinates.  (A minimum of one CTA per SM in the launch bounds, as
// vxb_closest_segment_kernel.)
__global__ void __launch_bounds__(VXB_COLLIDE_THREADS, 1) vxb_closest_segment_cut_kernel(const VxbCutRayMesh c, const float maxDistance,
	const vxb_segment* __restrict__ segments, unsigned count, vxb_segment_cut_hit* __restrict__ hits)
{
	const unsigned lane = threadIdx.x & 31;
	const unsigned warps = gridDim.x * (VXB_COLLIDE_THREADS / 32);
	const float md2 = maxDistance * maxDistance;
	const int nb = c.m.nb;
	for (unsigned q = blockIdx.x * (VXB_COLLIDE_THREADS / 32) + (threadIdx.x >> 5); q < count; q += warps)
	{
		const vxb_segment sg = segments[q];
		const float3 p = make_float3(sg.center[0], sg.center[1], sg.center[2]);
		const float3 h = make_float3(sg.half_axis[0], sg.half_axis[1], sg.half_axis[2]);
		const float3 g = make_float3(fabsf(h.x) + maxDistance + VXB_RAY_EPS, fabsf(h.y) + maxDistance + VXB_RAY_EPS,
			fabsf(h.z) + maxDistance + VXB_RAY_EPS);
		float bd = CUDART_INF_F;   // this lane's nearest triangle
		unsigned bs = VXB_RAY_MISS, bk = VXB_RAY_MISS;
		unsigned slot = VXB_RAY_MISS;
		if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z) && vxb_capsule_cut_reach(h, maxDistance, c.excursion) && lane < 27)
		{
			const float top = (float)(nb - 1);
			const int bx = (int)fminf(fmaxf(floorf(p.x * 0.0625f), 0.f), top) + (int)(lane % 3) - 1;
			const int by = (int)fminf(fmaxf(floorf(p.y * 0.0625f), 0.f), top) + (int)((lane / 3) % 3) - 1;
			const int bz = (int)fminf(fmaxf(floorf(p.z * 0.0625f), 0.f), top) + (int)(lane / 9) - 1;
			if (bx >= 0 && by >= 0 && bz >= 0 && bx < nb && by < nb && bz < nb)
			{
				unsigned key;
				const unsigned s = vxb_cut_node(c, bx, bz, by, key);   // grid (x, y, z) = output (x, z, y)
				if (s != VXB_RAY_MISS)
				{
					const float4 lo = __ldg(&c.boxes[2 * (size_t)key]), hi = __ldg(&c.boxes[2 * (size_t)key + 1]);
					if (!(lo.x - p.x > g.x || p.x - hi.x > g.x) && !(lo.y - p.y > g.y || p.y - hi.y > g.y) &&
						!(lo.z - p.z > g.z || p.z - hi.z > g.z)) slot = s;
				}
			}
		}
		const unsigned peers = __match_any_sync(0xFFFFFFFFu, slot);   // every lane takes part
		vxb_warp_each(slot != VXB_RAY_MISS && (peers & ((1u << lane) - 1u)) == 0, slot, [&](const unsigned s) {
			vxb_cut_triangles(c, s, [&](unsigned key, const float3& p0, const float3& p1, const float3& p2) {
				if (fminf(fminf(p0.x, p1.x), p2.x) - p.x > g.x || p.x - fmaxf(fmaxf(p0.x, p1.x), p2.x) > g.x ||
					fminf(fminf(p0.y, p1.y), p2.y) - p.y > g.y || p.y - fmaxf(fmaxf(p0.y, p1.y), p2.y) > g.y ||
					fminf(fminf(p0.z, p1.z), p2.z) - p.z > g.z || p.z - fmaxf(fmaxf(p0.z, p1.z), p2.z) > g.z) return;
				float3 x;
				float u, v, w;
				const float d2 = vxb_segment_triangle(p, h, p0, p1, p2, x, u, v, w);
				if (d2 <= md2 && vxb_ray_before(d2, s, key, bd, bs, bk)) { bd = d2; bs = s; bk = key; }
			});
		});
		if (lane == vxb_ray_winner(bd, bs, bk))
		{
			vxb_segment_cut_hit x;
			x.distance = CUDART_INF_F; x.slot = VXB_RAY_MISS; x.block_id = 0; x.triangle = 0;
			x.point[0] = x.point[1] = x.point[2] = 0.f;
			x.axis_point[0] = x.axis_point[1] = x.axis_point[2] = 0.f;
			x.normal[0] = x.normal[1] = x.normal[2] = 0.f;
			x.u = 0.f; x.v = 0.f; x.s = 0.f; x.level = 0; x.face = 0;
			if (bs != VXB_RAY_MISS)
			{
				const vxb_block_record* rec = c.m.dir + bs;
				const VxbVertex* verts;
				unsigned vo;
				const unsigned* ip;
				x.face = vxb_cut_hit_part(c, rec, bk, verts, vo, ip);
				const unsigned adj = vxb_cut_adj(c, rec);
				const float3 p0 = vxb_cut_vertex(verts, vo, __ldg(ip), adj);
				const float3 p1 = vxb_cut_vertex(verts, vo, __ldg(ip + 1), adj);
				const float3 p2 = vxb_cut_vertex(verts, vo, __ldg(ip + 2), adj);
				float3 pq, px;
				vxb_pair_fields(p, h, p0, p1, p2, pq, px, x.u, x.v, x.s);
				x.point[0] = pq.x; x.point[1] = pq.y; x.point[2] = pq.z;
				x.axis_point[0] = px.x; x.axis_point[1] = px.y; x.axis_point[2] = px.z;
				x.distance = VXB_SQRT(bd); x.slot = bs; x.block_id = __ldg(&rec->id); x.triangle = bk & 0xFFFFFFu;
				vxb_blend_normal(verts, vo, ip, x.u, x.v, x.normal);
				x.level = __ldg(&rec->level);
			}
			hits[q] = x;
		}
	}
}
