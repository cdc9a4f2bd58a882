// Sphere sweeps and closest-point queries against the level-0 triangles of the resident mesh (include/vxb200.h "collision
// queries").  Both use the level-0 block map of the ray casts (vxb_ray.cuh) and its rules.
//
//   sweeps          vxb_ray_walk with the block boxes grown by r + VXB_RAY_EPS; the proof of the walk, extended to that
//                   growth, is at the top of vxb_ray.cuh.
//   closest points  no walk: a triangle within max_distance of the query lies in a block whose box is within max_distance
//                   of the query (a level-0 triangle lies in the closed box of its block), and the float test below skips
//                   a block only when its box is farther than max_distance + VXB_RAY_EPS (the float box distance is within
//                   a few ulps of the true one; an accepted triangle is within max_distance plus rounding).  Such a block
//                   lies within max_distance + eps <= 15 + 1/16 < 16 of the query along every axis.  Along an axis where the
//                   query lies inside the grid, its index is that of the query's block +-1.  Along an axis where the query
//                   lies outside (below 0 or above n), only the first or last block of the axis is that close, and that is
//                   the clamped index.  So the 27 neighbours of the clamped block hold every block that can contribute, for
//                   queries inside and outside the grid box alike.
#pragma once

#define VXB_COLLIDE_THREADS VXB_RAY_THREADS

// Ericson's ClosestPtPointTriangle (Real-Time Collision Detection 5.1.5) in the order include/vxb200.h states: the point
// q of triangle (a, b, c) closest to p, and its barycentrics u (of b) and v (of c).
VXB_FN void vxb_closest_on_triangle(const float3 p, const float3 a, const float3 b, const float3 c, float3& q, float& u, float& v)
{
	const float abx = b.x - a.x, aby = b.y - a.y, abz = b.z - a.z;
	const float acx = c.x - a.x, acy = c.y - a.y, acz = c.z - a.z;
	const float apx = p.x - a.x, apy = p.y - a.y, apz = p.z - a.z;
	const float d1 = (abx * apx + aby * apy) + abz * apz;
	const float d2 = (acx * apx + acy * apy) + acz * apz;
	if (d1 <= 0.f && d2 <= 0.f) { q = a; u = 0.f; v = 0.f; return; }                                          // A
	const float bpx = p.x - b.x, bpy = p.y - b.y, bpz = p.z - b.z;
	const float d3 = (abx * bpx + aby * bpy) + abz * bpz;
	const float d4 = (acx * bpx + acy * bpy) + acz * bpz;
	if (d3 >= 0.f && d4 <= d3) { q = b; u = 1.f; v = 0.f; return; }                                           // B
	const float vc = d1 * d4 - d3 * d2;
	if (vc <= 0.f && d1 >= 0.f && d3 <= 0.f)                                                                   // AB
	{
		const float w = VXB_DIV(d1, d1 - d3);
		q = make_float3(a.x + w * abx, a.y + w * aby, a.z + w * abz); u = w; v = 0.f; return;
	}
	const float cpx = p.x - c.x, cpy = p.y - c.y, cpz = p.z - c.z;
	const float d5 = (abx * cpx + aby * cpy) + abz * cpz;
	const float d6 = (acx * cpx + acy * cpy) + acz * cpz;
	if (d6 >= 0.f && d5 <= d6) { q = c; u = 0.f; v = 1.f; return; }                                           // C
	const float vb = d5 * d2 - d1 * d6;
	if (vb <= 0.f && d2 >= 0.f && d6 <= 0.f)                                                                   // AC
	{
		const float w = VXB_DIV(d2, d2 - d6);
		q = make_float3(a.x + w * acx, a.y + w * acy, a.z + w * acz); u = 0.f; v = w; return;
	}
	const float va = d3 * d6 - d5 * d4;
	const float e43 = d4 - d3, e56 = d5 - d6;
	if (va <= 0.f && e43 >= 0.f && e56 >= 0.f)                                                                 // BC
	{
		const float w = VXB_DIV(e43, e43 + e56);
		q = make_float3(b.x + w * (c.x - b.x), b.y + w * (c.y - b.y), b.z + w * (c.z - b.z)); u = 1.f - w; v = w; return;
	}
	const float den = VXB_DIV(1.f, (va + vb) + vc);                                                            // face
	const float fv = vb * den, fw = vc * den;
	q = make_float3((a.x + abx * fv) + acx * fw, (a.y + aby * fv) + acy * fw, (a.z + abz * fv) + acz * fw); u = fv; v = fw;
}

// |p - q|^2 as the header states it: d = p - q; (dx*dx + dy*dy) + dz*dz
VXB_FN float vxb_dist2(const float3 p, const float3 q)
{
	const float dx = p.x - q.x, dy = p.y - q.y, dz = p.z - q.z;
	return (dx * dx + dy * dy) + dz * dz;
}

// The sweep's edge test against the segment q0 -> q1: the smaller root of the ray against the cylinder of radius r around
// the edge's line, kept when the centre there projects onto the segment (+inf otherwise).
VXB_FN float vxb_sweep_edge(const float3 o, const float3 d, const float3 q0, const float3 q1, float rr, float tMin, float tMax)
{
	const float ex = q1.x - q0.x, ey = q1.y - q0.y, ez = q1.z - q0.z;
	const float wx = o.x - q0.x, wy = o.y - q0.y, wz = o.z - q0.z;
	const float ee = (ex * ex + ey * ey) + ez * ez;
	const float dex = d.y * ez - d.z * ey, dey = d.z * ex - d.x * ez, dez = d.x * ey - d.y * ex;
	const float wex = wy * ez - wz * ey, wey = wz * ex - wx * ez, wez = wx * ey - wy * ex;
	const float A = (dex * dex + dey * dey) + dez * dez;
	const float B = (dex * wex + dey * wey) + dez * wez;
	const float g = (d.x * wex + d.y * wey) + d.z * wez;
	const float disc = ee * (rr * A - g * g);
	const float t = VXB_DIV(-B - VXB_SQRT(disc), A);
	const float s = ((wx + t * d.x) * ex + (wy + t * d.y) * ey) + (wz + t * d.z) * ez;
	return A > 0.f && disc >= 0.f && s >= 0.f && s <= ee && t >= tMin && t <= tMax ? t : CUDART_INF_F;
}

// The sweep's vertex test: the smaller root of |o + t d - q|^2 = r^2 (+inf when it is not in [t_min, t_max]); dd = d.d
VXB_FN float vxb_sweep_vertex(const float3 o, const float3 d, const float3 q, float rr, float dd, float tMin, float tMax)
{
	const float wx = o.x - q.x, wy = o.y - q.y, wz = o.z - q.z;
	const float B = (wx * d.x + wy * d.y) + wz * d.z;
	const float xx = wy * d.z - wz * d.y, xy = wz * d.x - wx * d.z, xz = wx * d.y - wy * d.x;
	const float disc = rr * dd - ((xx * xx + xy * xy) + xz * xz);
	const float t = VXB_DIV(-B - VXB_SQRT(disc), dd);
	return dd > 0.f && disc >= 0.f && t >= tMin && t <= tMax ? t : CUDART_INF_F;
}

// The first contact of the sphere (radius r, centre o + t d, t in [t_min, t_max]) with triangle (a, b, c), include/vxb200.h
// "sphere sweep": +inf when there is none; `started` when the sphere touches the triangle at t_min already.  c0 = o + t_min d.
VXB_FN float vxb_sweep_triangle(const float3 o, const float3 d, const float3 c0, float r, float rr, float dd, float tMin, float tMax,
	const float3 a, const float3 b, const float3 c, bool& started)
{
	started = false;
	{
		float3 q; float u, v;
		vxb_closest_on_triangle(c0, a, b, c, q, u, v);
		if (vxb_dist2(c0, q) <= rr) { started = true; return tMin; }
	}
	// the face: the plane offset by r toward the side of c0, as a Moeller-Trumbore cast of the ray moved by -r along that side
	const float e1x = b.x - a.x, e1y = b.y - a.y, e1z = b.z - a.z;
	const float e2x = c.x - a.x, e2y = c.y - a.y, e2z = c.z - a.z;
	const float nx = e1y * e2z - e1z * e2y, ny = e1z * e2x - e1x * e2z, nz = e1x * e2y - e1y * e2x;
	const float len = VXB_SQRT((nx * nx + ny * ny) + nz * nz);
	const float side = ((c0.x - a.x) * nx + (c0.y - a.y) * ny) + (c0.z - a.z) * nz;
	const float k = side >= 0.f ? r : -r;
	const float sx = (o.x - k * VXB_DIV(nx, len)) - a.x, sy = (o.y - k * VXB_DIV(ny, len)) - a.y, sz = (o.z - k * VXB_DIV(nz, len)) - a.z;
	const float pvx = d.y * e2z - d.z * e2y, pvy = d.z * e2x - d.x * e2z, pvz = d.x * e2y - d.y * e2x;
	const float det = (e1x * pvx + e1y * pvy) + e1z * pvz;
	const float inv = VXB_DIV(1.f, det);
	const float fu = ((sx * pvx + sy * pvy) + sz * pvz) * inv;
	const float qvx = sy * e1z - sz * e1y, qvy = sz * e1x - sx * e1z, qvz = sx * e1y - sy * e1x;
	const float fv = ((d.x * qvx + d.y * qvy) + d.z * qvz) * inv;
	const float ft = ((e2x * qvx + e2y * qvy) + e2z * qvz) * inv;
	float t = (side >= 0.f ? det > 0.f : det < 0.f) && fu >= 0.f && fu <= 1.f && fv >= 0.f && fu + fv <= 1.f && ft >= tMin &&
		ft <= tMax ? ft : CUDART_INF_F;
	// the edges ab, bc, ca, then the vertices a, b, c
	t = fminf(t, vxb_sweep_edge(o, d, a, b, rr, tMin, tMax));
	t = fminf(t, vxb_sweep_edge(o, d, b, c, rr, tMin, tMax));
	t = fminf(t, vxb_sweep_edge(o, d, c, a, rr, tMin, tMax));
	t = fminf(t, vxb_sweep_vertex(o, d, a, rr, dd, tMin, tMax));
	t = fminf(t, vxb_sweep_vertex(o, d, b, rr, dd, tMin, tMax));
	t = fminf(t, vxb_sweep_vertex(o, d, c, rr, dd, tMin, tMax));
	return t;
}

// One warp per sweep, persistent over the batch: the block walk of the ray casts with boxes grown by r + eps.  Sweeps and hits
// in OUTPUT (Y-up) coordinates.
__global__ void __launch_bounds__(VXB_COLLIDE_THREADS) vxb_sphere_cast_kernel(const VxbRayMesh m, const float r, const vxb_ray* __restrict__ rays,
	unsigned count, vxb_sphere_hit* __restrict__ hits)
{
	const unsigned lane = threadIdx.x & 31;
	const unsigned warps = gridDim.x * (VXB_COLLIDE_THREADS / 32);
	const float rr = r * r;
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
		vxb_ray_walk(m, ray, r + VXB_RAY_EPS, bt, [&](const unsigned s) {
			const vxb_block_record* rec = m.dir + s;
			const unsigned tris = __ldg(&rec->index_count) / 3, vo = __ldg(&rec->vertex_offset), io = __ldg(&rec->index_offset);
			for (unsigned k = lane; k < tris; k += 32)
			{
				float3 a, b, c;
				vxb_ray_triangle(m, vo, io, k, a, b, c);
				bool started;
				const float t = vxb_sweep_triangle(o, d, c0, r, rr, dd, tMin, tMax, a, b, c, started);
				if (t < CUDART_INF_F && vxb_ray_before(t, s, k, bt, bs, bk)) { bt = t; bs = s; bk = k; bStarted = started; }
			}
		});
		if (lane == vxb_ray_winner(bt, bs, bk))
		{
			vxb_sphere_hit h;
			h.t = CUDART_INF_F; h.slot = VXB_RAY_MISS; h.block_id = 0; h.triangle = 0;
			h.center[0] = h.center[1] = h.center[2] = 0.f;
			h.point[0] = h.point[1] = h.point[2] = 0.f;
			h.normal[0] = h.normal[1] = h.normal[2] = 0.f;
			h.u = 0.f; h.v = 0.f; h.flags = 0;
			if (bs != VXB_RAY_MISS)
			{
				const vxb_block_record* rec = m.dir + bs;
				float3 a, b, c, p;
				vxb_ray_triangle(m, __ldg(&rec->vertex_offset), __ldg(&rec->index_offset), bk, a, b, c);
				const float3 ct = make_float3(o.x + bt * d.x, o.y + bt * d.y, o.z + bt * d.z);
				vxb_closest_on_triangle(ct, a, b, c, p, h.u, h.v);
				h.t = bt; h.slot = bs; h.block_id = __ldg(&rec->id); h.triangle = bk;
				h.center[0] = ct.x; h.center[1] = ct.y; h.center[2] = ct.z;
				h.point[0] = p.x; h.point[1] = p.y; h.point[2] = p.z;
				vxb_ray_blend_normal(m, bs, bk, h.u, h.v, h.normal);
				h.flags = bStarted ? VXB_SPHERE_STARTED_IN_CONTACT : 0u;
			}
			hits[q] = h;
		}
	}
}

// One warp per query point, persistent over the batch: lane k < 27 takes neighbour k of the query's block (clamped into the
// grid), the warp then tests the candidate blocks' triangles strided over the lanes.  Points and hits in OUTPUT (Y-up)
// coordinates.
__global__ void __launch_bounds__(VXB_COLLIDE_THREADS) vxb_closest_point_kernel(const VxbRayMesh m, const float maxDistance,
	const float* __restrict__ points, unsigned count, vxb_closest_hit* __restrict__ hits)
{
	const unsigned lane = threadIdx.x & 31;
	const unsigned warps = gridDim.x * (VXB_COLLIDE_THREADS / 32);
	const int nb = m.nb;
	const float md2 = maxDistance * maxDistance, reach = maxDistance + VXB_RAY_EPS;
	const int ox = (int)(lane % 3) - 1, oy = (int)((lane / 3) % 3) - 1, oz = (int)(lane / 9) - 1;
	for (unsigned q = blockIdx.x * (VXB_COLLIDE_THREADS / 32) + (threadIdx.x >> 5); q < count; q += warps)
	{
		const float3 p = make_float3(points[3 * q], points[3 * q + 1], points[3 * q + 2]);
		float bd = CUDART_INF_F, bu = 0.f, bv = 0.f;   // this lane's nearest triangle
		float3 bp = make_float3(0.f, 0.f, 0.f);
		unsigned bs = VXB_RAY_MISS, bk = VXB_RAY_MISS;
		bool cand = false;
		unsigned slot = VXB_RAY_MISS;
		if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z) && lane < 27)
		{
			const float top = (float)(nb - 1);
			const int bx = (int)fminf(fmaxf(floorf(p.x * 0.0625f), 0.f), top) + ox;
			const int by = (int)fminf(fmaxf(floorf(p.y * 0.0625f), 0.f), top) + oy;
			const int bz = (int)fminf(fmaxf(floorf(p.z * 0.0625f), 0.f), top) + oz;
			if (bx >= 0 && by >= 0 && bz >= 0 && bx < nb && by < nb && bz < nb)
			{
				const float gx = fmaxf(fmaxf((float)(16 * bx) - p.x, p.x - (float)(16 * bx + 16)), 0.f);
				const float gy = fmaxf(fmaxf((float)(16 * by) - p.y, p.y - (float)(16 * by + 16)), 0.f);
				const float gz = fmaxf(fmaxf((float)(16 * bz) - p.z, p.z - (float)(16 * bz + 16)), 0.f);
				if (VXB_SQRT((gx * gx + gy * gy) + gz * gz) <= reach)
				{
					slot = __ldg(&m.map[((unsigned)by * nb + (unsigned)bz) * nb + (unsigned)bx]);   // output y = grid z
					cand = slot != VXB_RAY_MISS;
				}
			}
		}
		unsigned todo = __ballot_sync(0xFFFFFFFFu, cand);
		while (todo)
		{
			const unsigned src = __ffs(todo) - 1;
			todo &= todo - 1;
			const unsigned s = __shfl_sync(0xFFFFFFFFu, slot, src);
			const vxb_block_record* rec = m.dir + s;
			const unsigned tris = __ldg(&rec->index_count) / 3, vo = __ldg(&rec->vertex_offset), io = __ldg(&rec->index_offset);
			for (unsigned k = lane; k < tris; k += 32)
			{
				float3 a, b, c, x;
				float u, v;
				vxb_ray_triangle(m, vo, io, k, a, b, c);
				vxb_closest_on_triangle(p, a, b, c, x, u, v);
				const float d2 = vxb_dist2(p, x);
				if (d2 <= md2 && vxb_ray_before(d2, s, k, bd, bs, bk)) { bd = d2; bs = s; bk = k; bu = u; bv = v; bp = x; }
			}
		}
		if (lane == vxb_ray_winner(bd, bs, bk))
		{
			vxb_closest_hit h;
			h.distance = CUDART_INF_F; h.slot = VXB_RAY_MISS; h.block_id = 0; h.triangle = 0;
			h.point[0] = h.point[1] = h.point[2] = 0.f;
			h.normal[0] = h.normal[1] = h.normal[2] = 0.f;
			h.u = 0.f; h.v = 0.f;
			if (bs != VXB_RAY_MISS)
			{
				h.distance = VXB_SQRT(bd); h.slot = bs; h.block_id = __ldg(&m.dir[bs].id); h.triangle = bk;
				h.point[0] = bp.x; h.point[1] = bp.y; h.point[2] = bp.z;
				h.u = bu; h.v = bv;
				vxb_ray_blend_normal(m, bs, bk, bu, bv, h.normal);
			}
			hits[q] = h;
		}
	}
}
