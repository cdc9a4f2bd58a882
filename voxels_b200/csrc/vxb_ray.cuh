// Ray casts against the level-0 triangles of the resident mesh (include/vxb200.h "vxb_mesh_raycast").
//
// Level-0 vertices lie on the cell edges of their own block (t in [0, 256], exact dyadic positions), so every level-0
// triangle lies in the closed box of its block.  A ray therefore only needs the triangles of the blocks whose box it meets.
// The walk visits those blocks with a 3-D DDA (Amanatides-Woo) over the level-0 block lattice, made conservative:
//
//   tested set   every block whose closed box grown by VXB_RAY_EPS meets the clipped segment (te <= tx below).  A triangle
//                the test accepts has its hit point within rounding (about 1e-3 voxel at n = 4096 for a well-conditioned
//                test) of the triangle, hence inside the grown box of its block; so no accepted hit is lost to the walk.
//   anchoring    a tested block is handled at the DDA cell whose parameter interval [t0, t1) holds the block's grown-box
//                entry te (the last cell's interval is closed).  The intervals of the visited cells partition the clipped
//                segment exactly (each t1 is the next cell's t0, the same float), so every tested block is handled exactly
//                once.  The ray point at te is within VXB_RAY_EPS (+ rounding) of the block and inside the anchor cell (up to
//                rounding), so the block is one of the anchor cell's 27 neighbours: lane k of the warp evaluates neighbour k.
//                This covers rays in a block face plane (two columns), along a block edge (four) and through corners (eight).
//   stop         after cell c, every block not handled yet has te >= t1(c).  te = (plane - o) / d is two correctly rounded
//                operations, so the true entry is at least t1 - 2^-22 |t1|, and a hit in that block (inside its grown box) has
//                t >= that.  With the margin 2^-20 |t1|, t1 > best + margin proves t > best for every remaining hit: no hit
//                can tie or beat the best one, and the walk ends.
//
// Sphere sweeps (vxb_sphere_cast_body) run the same walk with the boxes grown by g = r + VXB_RAY_EPS instead of VXB_RAY_EPS:
//   tested set   a contact the sweep's tests accept puts the centre within r (+ rounding) of its triangle, hence of the
//                triangle's block, hence inside that block's box grown by r + eps.  A sweep that starts in contact has
//                c(t_min) there too, so the block's te is the clipped start.  The planes 16 b -+ g are now rounded (g is any
//                float), but a rounded plane moves by 2^-24 |16 b| at most, far inside the eps slack, so the box the walk uses
//                still holds every such centre; the proof above needs nothing else of the planes.
//   anchoring    the centre at te is within g (+ rounding) of the block and inside the anchor cell (up to rounding) along
//                every axis where it lies inside the grid.  Where it lies outside the grid (the clip box is grown by g too),
//                the cell index is clamped to 0 or nb - 1, and only that block is within g of the centre along that axis.
//                With r <= VXB_SPHERE_RADIUS_MAX = 15, g + rounding < 16 = one block: the block is still one of the anchor
//                cell's 27 neighbours.  A larger radius would need a wider neighbourhood, which is why the radius is capped.
//   stop         unchanged: te is still two correctly rounded operations from the (rounded) plane, and a contact inside the
//                grown box has t >= the true te.
//
// Capsule sweeps (half axis h, radius r; vxb_capsule_cast_body) run it with g = max_i |h_i| + r + VXB_RAY_EPS:
//   tested set   a contact pairs a point c + x h of the capsule's segment (|x| <= 1) with a triangle point within r of it, so
//                the centre c is within |x h_i| + r <= |h_i| + r <= g - eps (+ rounding) of the triangle along every axis
//                i, hence inside its block's box grown by g.  A sweep that starts in contact has c(t_min) there too.
//   anchoring    as for spheres with g in place of r + eps: the reach rule max_i |h_i| + r <= 15 keeps g + rounding < 16.
//   stop         unchanged.
#pragma once

#include <math_constants.h>

#define VXB_RAY_EPS 0.0625f        // growth of a block's box in voxels (1/16: a multiple of 2^-4, so 16 b +- eps is exact)
#define VXB_RAY_MARGIN_EXP (-20)   // stop margin: 2^-20 |t1| (te is within 2^-22 |te| of its true value, see above)
#define VXB_RAY_THREADS 256

// the dense level-0 map: coord_id -> mesh directory slot (VXB_RAY_MISS where no block is), after a memset to 0xFF
__global__ void __launch_bounds__(256) vxb_ray_map_kernel(const vxb_block_record* __restrict__ dir, unsigned count, unsigned* __restrict__ map)
{
	const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < count) map[__ldg(&dir[i].coord_id)] = i;
}

struct VxbRayMesh
{
	const vxb_block_record* dir;   // mesh directory (level 0 first)
	const unsigned* map;           // nb^3 slots, grid (Z-up) coord_id order
	const VxbVertex* verts;
	const unsigned* idx;
	int nb;                        // level-0 blocks per axis
};

// entry / exit parameters of the slab [lo, hi] along one axis; d == 0 (either sign): all t, or none when o is outside
VXB_FN void vxb_ray_slab(float o, float d, float lo, float hi, float& tin, float& tout)
{
	if (d == 0.f)
	{
		if (!(o >= lo && o <= hi)) { tin = CUDART_INF_F; tout = -CUDART_INF_F; }
		return;
	}
	float a = VXB_DIV(lo - o, d), b = VXB_DIV(hi - o, d);
	if (d < 0.f) { const float s = a; a = b; b = s; }
	tin = fmaxf(tin, a); tout = fminf(tout, b);
}

// the box of block index b along one axis, grown by g
VXB_FN float vxb_ray_lo(int b, float g) { return (float)(16 * b) - g; }
VXB_FN float vxb_ray_hi(int b, float g) { return (float)(16 * b + 16) + g; }

// the next cell boundary crossed along one axis (ungrown planes); +inf when the step would leave the grid
VXB_FN float vxb_ray_next(int c, float o, float d, int nb)
{
	if (d > 0.f && c + 1 < nb) return VXB_DIV((float)(16 * (c + 1)) - o, d);
	if (d < 0.f && c > 0) return VXB_DIV((float)(16 * c) - o, d);
	return CUDART_INF_F;
}

VXB_FN bool vxb_ray_valid(const vxb_ray& r)
{
	const bool finite = isfinite(r.origin[0]) && isfinite(r.origin[1]) && isfinite(r.origin[2]) && isfinite(r.direction[0]) &&
		isfinite(r.direction[1]) && isfinite(r.direction[2]) && isfinite(r.t_min) && !isnan(r.t_max);
	const bool nonzero = r.direction[0] != 0.f || r.direction[1] != 0.f || r.direction[2] != 0.f;
	return finite && nonzero && r.t_min <= r.t_max;
}

// (t, slot, triangle) ordered by the tie rule: least t, then lower slot, then lower triangle
VXB_FN bool vxb_ray_before(float t, unsigned s, unsigned k, float t2, unsigned s2, unsigned k2)
{
	return t < t2 || (t == t2 && (s < s2 || (s == s2 && k < k2)));
}


// the positions of triangle k of the block at (vertex offset vo, index offset io)
VXB_FN void vxb_ray_triangle(const VxbRayMesh& m, unsigned vo, unsigned io, unsigned k, float3& a, float3& b, float3& c)
{
	const unsigned* ip = m.idx + io + 3 * k;
	const float* pa = m.verts[vo + __ldg(ip)].pos;
	const float* pb = m.verts[vo + __ldg(ip + 1)].pos;
	const float* pc = m.verts[vo + __ldg(ip + 2)].pos;
	a = make_float3(__ldg(pa), __ldg(pa + 1), __ldg(pa + 2));
	b = make_float3(__ldg(pb), __ldg(pb + 1), __ldg(pb + 2));
	c = make_float3(__ldg(pc), __ldg(pc + 1), __ldg(pc + 2));
}

// Moeller-Trumbore exactly as include/vxb200.h states it (-fmad=false: no contraction): does the segment (p, d, [tMin, tMax])
// hit the triangle (p0, p1, p2), with its (t, u, v)
VXB_FN bool vxb_ray_mt(float px, float py, float pz, float dx, float dy, float dz, float tMin, float tMax, const float3& p0,
	const float3& p1, const float3& p2, float& t, float& u, float& v)
{
	const float e1x = p1.x - p0.x, e1y = p1.y - p0.y, e1z = p1.z - p0.z;
	const float e2x = p2.x - p0.x, e2y = p2.y - p0.y, e2z = p2.z - p0.z;
	const float sx = px - p0.x, sy = py - p0.y, sz = pz - p0.z;
	const float pvx = dy * e2z - dz * e2y, pvy = dz * e2x - dx * e2z, pvz = dx * e2y - dy * e2x;
	const float det = (e1x * pvx + e1y * pvy) + e1z * pvz;
	const float inv = VXB_DIV(1.f, det);
	u = ((sx * pvx + sy * pvy) + sz * pvz) * inv;
	const float qvx = sy * e1z - sz * e1y, qvy = sz * e1x - sx * e1z, qvz = sx * e1y - sy * e1x;
	v = ((dx * qvx + dy * qvy) + dz * qvz) * inv;
	t = ((e2x * qvx + e2y * qvy) + e2z * qvz) * inv;
	// positive comparisons only: a NaN fails
	return det != 0.f && u >= 0.f && u <= 1.f && v >= 0.f && u + v <= 1.f && t >= tMin && t <= tMax;
}

// The vertex normals of the triangle at indices ip (+ vertex offset vo into verts) blended at (u, v) and normalised, the hit
// normal of include/vxb200.h: w = (1 - u) - v; n_i = (w*n0_i + u*n1_i) + v*n2_i; n_i / sqrt((nx*nx + ny*ny) + nz*nz), or
// (0, 0, 0) when that is 0.
VXB_FN void vxb_blend_normal(const VxbVertex* verts, unsigned vo, const unsigned* ip, float u, float v, float* out)
{
	const float* n0 = verts[vo + __ldg(ip)].nrm;
	const float* n1 = verts[vo + __ldg(ip + 1)].nrm;
	const float* n2 = verts[vo + __ldg(ip + 2)].nrm;
	const float w = (1.f - u) - v;
	const float nxv = (w * __ldg(n0) + u * __ldg(n1)) + v * __ldg(n2);
	const float nyv = (w * __ldg(n0 + 1) + u * __ldg(n1 + 1)) + v * __ldg(n2 + 1);
	const float nzv = (w * __ldg(n0 + 2) + u * __ldg(n1 + 2)) + v * __ldg(n2 + 2);
	const float len = VXB_SQRT((nxv * nxv + nyv * nyv) + nzv * nzv);
	out[0] = out[1] = out[2] = 0.f;
	if (len > 0.f) { out[0] = VXB_DIV(nxv, len); out[1] = VXB_DIV(nyv, len); out[2] = VXB_DIV(nzv, len); }
}

// The lane holding the warp's least (t, slot, triangle) by the tie rule (every lane takes part; each candidate is held by
// one lane, and a warp of misses - slot = triangle = VXB_RAY_MISS everywhere - yields lane 0).
VXB_FN unsigned vxb_ray_winner(float t, unsigned s, unsigned k)
{
	float wt = t; unsigned ws = s, wk = k;
	for (int o = 16; o > 0; o >>= 1)
	{
		const float t2 = __shfl_xor_sync(0xFFFFFFFFu, wt, o);
		const unsigned s2 = __shfl_xor_sync(0xFFFFFFFFu, ws, o), k2 = __shfl_xor_sync(0xFFFFFFFFu, wk, o);
		if (vxb_ray_before(t2, s2, k2, wt, ws, wk)) { wt = t2; ws = s2; wk = k2; }
	}
	return __ffs(__ballot_sync(0xFFFFFFFFu, s == ws && k == wk)) - 1;
}

// The slot hand-off: `block(slot)` is called by the whole warp (every lane takes part) once for each lane that has `take`,
// with that lane's slot, in lane order.  Returns whether any lane had one.
template <class Block>
VXB_FN bool vxb_warp_each(bool take, unsigned slot, Block&& block)
{
	unsigned todo = __ballot_sync(0xFFFFFFFFu, take);
	const bool any = todo != 0;
	while (todo)
	{
		const unsigned src = __ffs(todo) - 1;
		todo &= todo - 1;
		block(__shfl_sync(0xFFFFFFFFu, slot, src));
	}
	return any;
}

// f(k, a, b, c) for each triangle k of level-0 slot s with its positions, strided over the lanes (k = lane, lane + 32, ...)
template <class F>
VXB_FN void vxb_slot_triangles(const VxbRayMesh& m, unsigned s, F&& f)
{
	const vxb_block_record* rec = m.dir + s;
	const unsigned tris = __ldg(&rec->index_count) / 3, vo = __ldg(&rec->vertex_offset), io = __ldg(&rec->index_offset);
	for (unsigned k = threadIdx.x & 31; k < tris; k += 32)
	{
		float3 a, b, c;
		vxb_ray_triangle(m, vo, io, k, a, b, c);
		f(k, a, b, c);
	}
}

// The conservative block walk of the proof at the top, for one segment per warp (every lane calls it with the same ray),
// with the candidate step as a parameter: lane k < 27 calls `cand(bx, by, bz, T0, T1, t0, t1, last, slot)` for neighbour k
// of the cell [t0, t1) when that block lies in the grid; it returns whether there is a directory slot to test there, and
// writes it to `slot`.
// The grid box is clipped grown by `grow`.  With Dedup, lanes that return the same slot hand it on once (the lowest lane).
// `block(s)` is called by the whole warp once per slot handed on, in walk order; it tests the slot's triangles (strided
// over the lanes) and lowers this lane's best parameter `best`, which the stop rule reads.  Rays and blocks in OUTPUT
// (Y-up) coordinates; block coordinates of the map are grid (Z-up): output (x, y, z) = grid (x, z, y).
template <bool Dedup, class Cand, class Block>
VXB_FN void vxb_ray_walk_by(const int nb, const vxb_ray& ray, const float grow, const float& best, Cand&& cand, Block&& block)
{
	const unsigned lane = threadIdx.x & 31;
	const float n = (float)(16 * nb);
	// this lane's neighbour offset (lanes 27..31 have none)
	const int ox = (int)(lane % 3) - 1, oy = (int)((lane / 3) % 3) - 1, oz = (int)(lane / 9) - 1;
	const float px = ray.origin[0], py = ray.origin[1], pz = ray.origin[2];
	const float dx = ray.direction[0], dy = ray.direction[1], dz = ray.direction[2];
	// ---- clip to the grown grid box [-g, n + g]^3 (the union of the grown block boxes, computed with the same planes) ----
	float T0 = ray.t_min, T1 = ray.t_max;
	if (!vxb_ray_valid(ray)) return;
	vxb_ray_slab(px, dx, -grow, n + grow, T0, T1);
	vxb_ray_slab(py, dy, -grow, n + grow, T0, T1);
	vxb_ray_slab(pz, dz, -grow, n + grow, T0, T1);
	if (!(T0 <= T1)) return;
	// the first cell: the block of the clipped entry point, clamped into the grid
	int cx = min(max((int)floorf((px + T0 * dx) * 0.0625f), 0), nb - 1);
	int cy = min(max((int)floorf((py + T0 * dy) * 0.0625f), 0), nb - 1);
	int cz = min(max((int)floorf((pz + T0 * dz) * 0.0625f), 0), nb - 1);
	float nx = vxb_ray_next(cx, px, dx, nb), ny = vxb_ray_next(cy, py, dy, nb), nz = vxb_ray_next(cz, pz, dz, nb);
	float t0 = T0;
	for (;;)
	{
		const float tn = fminf(nx, fminf(ny, nz));
		const bool last = !(tn < T1);
		const float t1 = last ? T1 : fmaxf(tn, t0);
		// ---- the neighbours anchored in [t0, t1) ----
		const int bx = cx + ox, by = cy + oy, bz = cz + oz;
		bool take = false;
		unsigned slot = VXB_RAY_MISS;
		if (lane < 27 && bx >= 0 && by >= 0 && bz >= 0 && bx < nb && by < nb && bz < nb) take = cand(bx, by, bz, T0, T1, t0, t1, last, slot);
		if constexpr (Dedup)
		{
			const unsigned peers = __match_any_sync(0xFFFFFFFFu, slot);   // every lane takes part (lanes without a slot hold VXB_RAY_MISS)
			take = take && (peers & ((1u << lane) - 1u)) == 0;
		}
		const bool tested = vxb_warp_each(take, slot, block);
		if (last) break;
		if (tested)
		{
			float w = best;
			for (int o = 16; o > 0; o >>= 1) w = fminf(w, __shfl_xor_sync(0xFFFFFFFFu, w, o));
			if (t1 > w + ldexpf(fabsf(t1), VXB_RAY_MARGIN_EXP)) break;
		}
		// ---- step across the nearest boundary (ties: x, then y, then z; the others follow with empty intervals) ----
		if (nx == tn) { cx += dx > 0.f ? 1 : -1; nx = vxb_ray_next(cx, px, dx, nb); }
		else if (ny == tn) { cy += dy > 0.f ? 1 : -1; ny = vxb_ray_next(cy, py, dy, nb); }
		else { cz += dz > 0.f ? 1 : -1; nz = vxb_ray_next(cz, pz, dz, nb); }
		t0 = t1;
	}
}

// The level-0 walk: the tested set is every level-0 block whose lattice box grown by `grow` (VXB_RAY_EPS for rays,
// r + VXB_RAY_EPS for sweeps) meets the clipped segment and has a map entry; each one is anchored once, so no merging.
template <class Block>
VXB_FN void vxb_ray_walk(const VxbRayMesh& m, const vxb_ray& ray, const float grow, const float& best, Block&& block)
{
	const float px = ray.origin[0], py = ray.origin[1], pz = ray.origin[2];
	const float dx = ray.direction[0], dy = ray.direction[1], dz = ray.direction[2];
	const int nb = m.nb;
	vxb_ray_walk_by<false>(nb, ray, grow, best,
		[&](int bx, int by, int bz, float T0, float T1, float t0, float t1, bool last, unsigned& slot) {
			float te = T0, tx = T1;
			vxb_ray_slab(px, dx, vxb_ray_lo(bx, grow), vxb_ray_hi(bx, grow), te, tx);
			vxb_ray_slab(py, dy, vxb_ray_lo(by, grow), vxb_ray_hi(by, grow), te, tx);
			vxb_ray_slab(pz, dz, vxb_ray_lo(bz, grow), vxb_ray_hi(bz, grow), te, tx);
			if (te <= tx && te >= t0 && (te < t1 || last))
			{
				slot = __ldg(&m.map[((unsigned)by * nb + (unsigned)bz) * nb + (unsigned)bx]);   // output y = grid z
				return slot != VXB_RAY_MISS;
			}
			return false;
		},
		block);
}
