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
// Closest points against the cut need no walk; their proof is with VxbCutSurface::point.
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

// The winning triangle of a hit: triangle key (part << 24 | k) of cut node rec, its part's vertices `verts` from vertex offset vo
// and its indices at ip (for vxb_blend_normal and vxb_cut_vertex).
VXB_FN void vxb_cut_hit_part(const VxbCutRayMesh& c, const vxb_block_record* rec, unsigned key, const VxbVertex*& verts, unsigned& vo,
	const unsigned*& ip)
{
	const unsigned p = key >> 24, k = key & 0xFFFFFFu;
	if (p) { verts = c.tverts; vo = __ldg(&rec->trans_vertex_offset[p - 1]); ip = c.tidx + __ldg(&rec->trans_index_offset[p - 1]) + 3 * k; }
	else { verts = c.m.verts; vo = __ldg(&rec->vertex_offset); ip = c.m.idx + __ldg(&rec->index_offset) + 3 * k; }
}

// The cut reach of a capsule query (include/vxb200.h "capsule queries against the drawn LOD cut"), in float for the host
// check and the kernels alike: the level-0 rule vxb_capsule_reach, then e + (max_i |h_i| + extra) <= 15; extra is the radius
// of a sweep or the max_distance of a segment, e the mesh's excursion.
VXB_HD bool vxb_capsule_cut_reach(const float3 h, float extra, float e)
{
	const float hm = fmaxf(fmaxf(fabsf(h.x), fabsf(h.y)), fabsf(h.z));
	return vxb_capsule_reach(h, extra) && e + (hm + extra) <= VXB_SPHERE_RADIUS_MAX;
}

// ---- the drawn cut as a surface ------------------------------------------------------------------------------------------
//
// The drawn triangles of the cut for the query bodies (vxb_query.cuh), as VxbLevel0Surface is for level 0.  Keys are
// part << 24 | triangle (vxb_cut_triangles); the hit's tail is the winning node's level and the face of its part.
struct VxbCutSurface
{
	const VxbCutRayMesh& c;

	// The cut walk of a shape whose reach splits as hm = max_i |h_i| and r (both 0 for rays, hm = -0 for spheres): with R = hm + r
	// rounded up, the clip box grown by e + R + VXB_RAY_EPS and every node's measured box by R + VXB_RAY_EPS (both rounded up;
	// the proofs at the top).  For rays R = 0, and for spheres R = r, so their growths are c.grow and VXB_RAY_EPS, r + eps.
	template <class Block>
	VXB_FN void walk(const vxb_ray& ray, float hm, float r, const float& best, Block&& block) const
	{
		const float R = __fadd_ru(hm, r);
		const float g = __fadd_ru(R, VXB_RAY_EPS);
		vxb_ray_walk_by<true>(c.m.nb, ray, __fadd_ru(c.grow, R), best,
			[&](int bx, int by, int bz, float T0, float T1, float t0, float t1, bool last, unsigned& slot) {
				return vxb_cut_candidate(c, ray, g, bx, by, bz, T0, T1, t0, t1, last, slot);
			},
			block);
	}

	// The point candidate: lane k < 27 takes neighbour k of the point's block clamped into the grid (vxb_point_candidate),
	// finds that block's covering cut node and keeps it when `near(lo, hi)` accepts the node's measured box.  Lanes that reach
	// the same node hand it on once (the lowest lane).  For a closest-point query within max_distance m:
	//   every contributing node is a candidate   a drawn triangle within max_distance m of p (the test accepts it) is within m
	//                   (+ rounding) of a point of the node's measured box, which holds every drawn vertex; the float box distance
	//                   is within a few ulps of the true one, so the node is kept.  Its lattice box then lies within e + m + eps <=
	//                   15 + 1/16 < 16 of p along every axis (the host refuses e + m > 15).  Along an axis where p lies inside the
	//                   grid, the lattice box (a run of whole level-0 blocks) holds a block whose index is that of p's block +-1;
	//                   where p lies outside, it holds the first or last block of the axis, the clamped index.  So one of the 27
	//                   neighbours lies inside the node, and since the cut tiles the grid, that neighbour's covering node is it.
	//   handled once    __match_any_sync over the lanes' slots, the lowest lane of each group hands the node on.
	template <class Near>
	VXB_FN bool point(const float3 p, bool ok, Near&& near, unsigned& slot) const
	{
		vxb_point_candidate(c.m.nb, p, ok, [&](int bx, int by, int bz, unsigned& s) {
			unsigned key;
			const unsigned n = vxb_cut_node(c, bx, bz, by, key);   // grid (x, y, z) = output (x, z, y)
			if (n == VXB_RAY_MISS) return false;
			const float4 lo = __ldg(&c.boxes[2 * (size_t)key]), hi = __ldg(&c.boxes[2 * (size_t)key + 1]);
			if (!near(make_float3(lo.x, lo.y, lo.z), make_float3(hi.x, hi.y, hi.z))) return false;
			s = n;
			return true;
		}, slot);
		const unsigned lane = threadIdx.x & 31;
		const unsigned peers = __match_any_sync(0xFFFFFFFFu, slot);   // every lane takes part (lanes without a node hold VXB_RAY_MISS)
		return slot != VXB_RAY_MISS && (peers & ((1u << lane) - 1u)) == 0;
	}

	template <class F>
	VXB_FN void triangles(unsigned s, F&& f) const { vxb_cut_triangles(c, s, f); }

	VXB_FN const vxb_block_record* record(unsigned s) const { return c.m.dir + s; }

	// the positions of the winning triangle key (part << 24 | k) of the cut node at directory record rec as the renderer draws
	// them, and its blended normal at (u, v)
	VXB_FN void corners(const vxb_block_record* rec, unsigned key, float3& p0, float3& p1, float3& p2) const
	{
		const VxbVertex* verts;
		unsigned vo;
		const unsigned* ip;
		vxb_cut_hit_part(c, rec, key, verts, vo, ip);
		const unsigned adj = vxb_cut_adj(c, rec);
		p0 = vxb_cut_vertex(verts, vo, __ldg(ip), adj);
		p1 = vxb_cut_vertex(verts, vo, __ldg(ip + 1), adj);
		p2 = vxb_cut_vertex(verts, vo, __ldg(ip + 2), adj);
	}
	VXB_FN void normal(const vxb_block_record* rec, unsigned key, float u, float v, float* out) const
	{
		const VxbVertex* verts;
		unsigned vo;
		const unsigned* ip;
		vxb_cut_hit_part(c, rec, key, verts, vo, ip);
		vxb_blend_normal(verts, vo, ip, u, v, out);
	}

	VXB_FN unsigned triangle(unsigned key) const { return key & 0xFFFFFFu; }

	VXB_FN bool reach(const float3 h, float extra) const { return vxb_capsule_cut_reach(h, extra, c.excursion); }

	// level and face (0xFFFFFFFF for the regular part) of a hit, 0 and 0 for a miss
	template <class Hit>
	VXB_FN void tail(Hit& h, unsigned s, unsigned key) const
	{
		h.level = 0; h.face = 0;
		if (s != VXB_RAY_MISS)
		{
			const unsigned p = key >> 24;
			h.level = __ldg(&c.m.dir[s].level); h.face = p ? p - 1 : 0xFFFFFFFFu;
		}
	}
};
