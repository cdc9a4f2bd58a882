// The resident-mesh queries: one body per query shape, over a surface (VxbLevel0Surface: the level-0 triangles, vxb_collide.cuh;
// VxbCutSurface: the drawn LOD cut, vxb_cutray.cuh), and the ten named kernels that run them.
//
// Every body runs one warp per query, persistent over the batch.  The surface hands candidate blocks to the warp (the walk
// for swept shapes, the 27-neighbour step for point shapes; the proofs are at the top of vxb_ray.cuh, vxb_collide.cuh and
// vxb_cutray.cuh); the warp tests each block's triangles strided over the lanes, each lane keeping its best by the tie rule
// (vxb_ray_before on (t or squared distance, slot, key)); the winner's lane (vxb_ray_winner) writes the hit, a miss when no
// lane has one.  A level-0 hit struct and its cut twin share every field name but the cut's `level` and `face`, which the
// surface writes (`tail`).  Queries and hits in OUTPUT (Y-up) coordinates.
#pragma once

template <class Surface, class Hit>
VXB_FN void vxb_raycast_body(const Surface& surf, const vxb_ray* __restrict__ rays, unsigned count, Hit* __restrict__ hits)
{
	const unsigned lane = threadIdx.x & 31;
	const unsigned warps = gridDim.x * (VXB_RAY_THREADS / 32);
	for (unsigned r = blockIdx.x * (VXB_RAY_THREADS / 32) + (threadIdx.x >> 5); r < count; r += warps)
	{
		const vxb_ray ray = rays[r];
		const float px = ray.origin[0], py = ray.origin[1], pz = ray.origin[2];
		const float dx = ray.direction[0], dy = ray.direction[1], dz = ray.direction[2];
		const float tMin = ray.t_min, tMax = ray.t_max;
		float bt = CUDART_INF_F, bu = 0.f, bv = 0.f;   // this lane's best hit
		unsigned bs = VXB_RAY_MISS, bk = VXB_RAY_MISS;
		surf.walk(ray, 0.f, 0.f, bt, [&](const unsigned s) {
			surf.triangles(s, [&](unsigned k, const float3& p0, const float3& p1, const float3& p2) {
				float t, u, v;
				if (vxb_ray_mt(px, py, pz, dx, dy, dz, tMin, tMax, p0, p1, p2, t, u, v) && vxb_ray_before(t, s, k, bt, bs, bk))
				{
					bt = t; bs = s; bk = k; bu = u; bv = v;
				}
			});
		});
		// ---- the winner by the tie rule; its lane writes the hit ----
		if (lane == vxb_ray_winner(bt, bs, bk))
		{
			Hit h;
			h.u = 0.f; h.v = 0.f; h.slot = VXB_RAY_MISS; h.block_id = 0; h.triangle = 0;
			h.t = CUDART_INF_F;
			h.position[0] = h.position[1] = h.position[2] = 0.f;
			h.normal[0] = h.normal[1] = h.normal[2] = 0.f;
			if (bs != VXB_RAY_MISS)
			{
				const vxb_block_record* rec = surf.record(bs);
				h.t = bt; h.u = bu; h.v = bv; h.slot = bs; h.block_id = __ldg(&rec->id); h.triangle = surf.triangle(bk);
				h.position[0] = px + bt * dx; h.position[1] = py + bt * dy; h.position[2] = pz + bt * dz;
				surf.normal(rec, bk, bu, bv, h.normal);
			}
			surf.tail(h, bs, bk);
			hits[r] = h;
		}
	}
}

// The sphere sweep (radius r): the walk grown by the radius, vxb_sweep_triangle on each triangle.
template <class Surface, class Hit>
VXB_FN void vxb_sphere_cast_body(const Surface& surf, const float r, const vxb_ray* __restrict__ rays, unsigned count,
	Hit* __restrict__ hits)
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
		surf.walk(ray, -0.f, r, bt, [&](const unsigned s) {   // hm = -0: -0 + r is r exactly, and the compiler drops the add
			surf.triangles(s, [&](unsigned k, const float3& a, const float3& b, const float3& c) {
				bool started;
				const float t = vxb_sweep_triangle(o, d, c0, r, rr, dd, tMin, tMax, a, b, c, started);
				if (t < CUDART_INF_F && vxb_ray_before(t, s, k, bt, bs, bk)) { bt = t; bs = s; bk = k; bStarted = started; }
			});
		});
		if (lane == vxb_ray_winner(bt, bs, bk))
		{
			Hit h;
			h.t = CUDART_INF_F; h.slot = VXB_RAY_MISS; h.block_id = 0; h.triangle = 0;
			h.center[0] = h.center[1] = h.center[2] = 0.f;
			h.point[0] = h.point[1] = h.point[2] = 0.f;
			h.normal[0] = h.normal[1] = h.normal[2] = 0.f;
			h.u = 0.f; h.v = 0.f; h.flags = 0;
			if (bs != VXB_RAY_MISS)
			{
				const vxb_block_record* rec = surf.record(bs);
				float3 a, b, c, p;
				surf.corners(rec, bk, a, b, c);
				const float3 ct = make_float3(o.x + bt * d.x, o.y + bt * d.y, o.z + bt * d.z);
				vxb_closest_on_triangle(ct, a, b, c, p, h.u, h.v);
				h.t = bt; h.slot = bs; h.block_id = __ldg(&rec->id); h.triangle = surf.triangle(bk);
				h.center[0] = ct.x; h.center[1] = ct.y; h.center[2] = ct.z;
				h.point[0] = p.x; h.point[1] = p.y; h.point[2] = p.z;
				surf.normal(rec, bk, h.u, h.v, h.normal);
				h.flags = bStarted ? VXB_SPHERE_STARTED_IN_CONTACT : 0u;
			}
			surf.tail(h, bs, bk);
			hits[q] = h;
		}
	}
}

// The closest point within max_distance: the point candidates whose box is within max_distance + VXB_RAY_EPS of the point,
// vxb_closest_on_triangle on each triangle.
template <class Surface, class Hit>
VXB_FN void vxb_closest_point_body(const Surface& surf, const float maxDistance, const float* __restrict__ points, unsigned count,
	Hit* __restrict__ hits)
{
	const unsigned lane = threadIdx.x & 31;
	const unsigned warps = gridDim.x * (VXB_COLLIDE_THREADS / 32);
	const float md2 = maxDistance * maxDistance, reach = maxDistance + VXB_RAY_EPS;
	for (unsigned q = blockIdx.x * (VXB_COLLIDE_THREADS / 32) + (threadIdx.x >> 5); q < count; q += warps)
	{
		const float3 p = make_float3(points[3 * q], points[3 * q + 1], points[3 * q + 2]);
		float bd = CUDART_INF_F, bu = 0.f, bv = 0.f;   // this lane's nearest triangle
		float3 bp = make_float3(0.f, 0.f, 0.f);
		unsigned bs = VXB_RAY_MISS, bk = VXB_RAY_MISS;
		unsigned slot;
		const bool cand = surf.point(p, isfinite(p.x) && isfinite(p.y) && isfinite(p.z), [&](const float3 lo, const float3 hi) {
			const float gx = fmaxf(fmaxf(lo.x - p.x, p.x - hi.x), 0.f);
			const float gy = fmaxf(fmaxf(lo.y - p.y, p.y - hi.y), 0.f);
			const float gz = fmaxf(fmaxf(lo.z - p.z, p.z - hi.z), 0.f);
			return VXB_SQRT((gx * gx + gy * gy) + gz * gz) <= reach;
		}, slot);
		vxb_warp_each(cand, slot, [&](const unsigned s) {
			surf.triangles(s, [&](unsigned k, const float3& a, const float3& b, const float3& c) {
				float3 x;
				float u, v;
				vxb_closest_on_triangle(p, a, b, c, x, u, v);
				const float d2 = vxb_dist2(p, x);
				if (d2 <= md2 && vxb_ray_before(d2, s, k, bd, bs, bk)) { bd = d2; bs = s; bk = k; bu = u; bv = v; bp = x; }
			});
		});
		if (lane == vxb_ray_winner(bd, bs, bk))
		{
			Hit h;
			h.distance = CUDART_INF_F; h.slot = VXB_RAY_MISS; h.block_id = 0; h.triangle = 0;
			h.point[0] = h.point[1] = h.point[2] = 0.f;
			h.normal[0] = h.normal[1] = h.normal[2] = 0.f;
			h.u = 0.f; h.v = 0.f;
			if (bs != VXB_RAY_MISS)
			{
				const vxb_block_record* rec = surf.record(bs);
				h.distance = VXB_SQRT(bd); h.slot = bs; h.block_id = __ldg(&rec->id); h.triangle = surf.triangle(bk);
				h.point[0] = bp.x; h.point[1] = bp.y; h.point[2] = bp.z;
				h.u = bu; h.v = bv;
				surf.normal(rec, bk, bu, bv, h.normal);
			}
			surf.tail(h, bs, bk);
			hits[q] = h;
		}
	}
}

// The capsule sweep (half axis h, radius r): the walk grown by the reach max_i |h_i| + r, then per triangle the reject
// vxb_path_meets_box on its box grown by |h_i| + r + eps and vxb_capsule_triangle.  A sweep out of the surface's reach is a
// miss.
template <class Surface, class Hit>
VXB_FN void vxb_capsule_cast_body(const Surface& surf, const vxb_capsule_sweep* __restrict__ sweeps, unsigned count,
	Hit* __restrict__ hits)
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
		float bt = CUDART_INF_F;   // this lane's first contact
		unsigned bs = VXB_RAY_MISS, bk = VXB_RAY_MISS;
		bool bStarted = false;
		if (r > 0.f && surf.reach(h, r))   // the same for the whole warp
			surf.walk(ray, fmaxf(fmaxf(fabsf(h.x), fabsf(h.y)), fabsf(h.z)), r, bt, [&](const unsigned s) {
				surf.triangles(s, [&](unsigned k, const float3& a, const float3& b, const float3& c) {
					if (!vxb_path_meets_box(ray, g, a, b, c)) return;
					bool started;
					const float t = vxb_capsule_triangle(o, d, c0, h, r, rr, dd, tMin, tMax, a, b, c, started);
					if (t < CUDART_INF_F && vxb_ray_before(t, s, k, bt, bs, bk)) { bt = t; bs = s; bk = k; bStarted = started; }
				});
			});
		if (lane == vxb_ray_winner(bt, bs, bk))
		{
			Hit x;
			x.t = CUDART_INF_F; x.slot = VXB_RAY_MISS; x.block_id = 0; x.triangle = 0;
			x.center[0] = x.center[1] = x.center[2] = 0.f;
			x.point[0] = x.point[1] = x.point[2] = 0.f;
			x.axis_point[0] = x.axis_point[1] = x.axis_point[2] = 0.f;
			x.normal[0] = x.normal[1] = x.normal[2] = 0.f;
			x.u = 0.f; x.v = 0.f; x.s = 0.f; x.flags = 0;
			if (bs != VXB_RAY_MISS)
			{
				const vxb_block_record* rec = surf.record(bs);
				float3 a, b, c;
				surf.corners(rec, bk, a, b, c);
				const float3 ct = make_float3(o.x + bt * d.x, o.y + bt * d.y, o.z + bt * d.z);
				float3 pq, px;
				vxb_pair_fields(ct, h, a, b, c, pq, px, x.u, x.v, x.s);
				x.point[0] = pq.x; x.point[1] = pq.y; x.point[2] = pq.z;
				x.axis_point[0] = px.x; x.axis_point[1] = px.y; x.axis_point[2] = px.z;
				x.t = bt; x.slot = bs; x.block_id = __ldg(&rec->id); x.triangle = surf.triangle(bk);
				x.center[0] = ct.x; x.center[1] = ct.y; x.center[2] = ct.z;
				surf.normal(rec, bk, x.u, x.v, x.normal);
				x.flags = bStarted ? VXB_SPHERE_STARTED_IN_CONTACT : 0u;
			}
			surf.tail(x, bs, bk);
			hits[q] = x;
		}
	}
}

// The closest pair to a segment (centre p, half axis h) within max_distance: the point candidates whose box lies within
// |h_i| + max_distance + VXB_RAY_EPS of the centre along every axis, the same per-axis reject per triangle, then
// vxb_segment_triangle.  A segment out of the surface's reach is a miss.
template <class Surface, class Hit>
VXB_FN void vxb_closest_segment_body(const Surface& surf, const float maxDistance, const vxb_segment* __restrict__ segments,
	unsigned count, Hit* __restrict__ hits)
{
	const unsigned lane = threadIdx.x & 31;
	const unsigned warps = gridDim.x * (VXB_COLLIDE_THREADS / 32);
	const float md2 = maxDistance * maxDistance;
	for (unsigned q = blockIdx.x * (VXB_COLLIDE_THREADS / 32) + (threadIdx.x >> 5); q < count; q += warps)
	{
		const vxb_segment sg = segments[q];
		const float3 p = make_float3(sg.center[0], sg.center[1], sg.center[2]);
		const float3 h = make_float3(sg.half_axis[0], sg.half_axis[1], sg.half_axis[2]);
		const float3 g = make_float3(fabsf(h.x) + maxDistance + VXB_RAY_EPS, fabsf(h.y) + maxDistance + VXB_RAY_EPS,
			fabsf(h.z) + maxDistance + VXB_RAY_EPS);
		float bd = CUDART_INF_F;   // this lane's nearest triangle
		unsigned bs = VXB_RAY_MISS, bk = VXB_RAY_MISS;
		unsigned slot;
		const bool ok = isfinite(p.x) && isfinite(p.y) && isfinite(p.z) && surf.reach(h, maxDistance);
		const bool cand = surf.point(p, ok, [&](const float3 lo, const float3 hi) {
			return !(lo.x - p.x > g.x || p.x - hi.x > g.x) && !(lo.y - p.y > g.y || p.y - hi.y > g.y) &&
				!(lo.z - p.z > g.z || p.z - hi.z > g.z);
		}, slot);
		vxb_warp_each(cand, slot, [&](const unsigned s) {
			surf.triangles(s, [&](unsigned k, const float3& a, const float3& b, const float3& c) {
				if (fminf(fminf(a.x, b.x), c.x) - p.x > g.x || p.x - fmaxf(fmaxf(a.x, b.x), c.x) > g.x ||
					fminf(fminf(a.y, b.y), c.y) - p.y > g.y || p.y - fmaxf(fmaxf(a.y, b.y), c.y) > g.y ||
					fminf(fminf(a.z, b.z), c.z) - p.z > g.z || p.z - fmaxf(fmaxf(a.z, b.z), c.z) > g.z) return;
				float3 x;
				float u, v, w;
				const float d2 = vxb_segment_triangle(p, h, a, b, c, x, u, v, w);
				if (d2 <= md2 && vxb_ray_before(d2, s, k, bd, bs, bk)) { bd = d2; bs = s; bk = k; }
			});
		});
		if (lane == vxb_ray_winner(bd, bs, bk))
		{
			Hit x;
			x.distance = CUDART_INF_F; x.slot = VXB_RAY_MISS; x.block_id = 0; x.triangle = 0;
			x.point[0] = x.point[1] = x.point[2] = 0.f;
			x.axis_point[0] = x.axis_point[1] = x.axis_point[2] = 0.f;
			x.normal[0] = x.normal[1] = x.normal[2] = 0.f;
			x.u = 0.f; x.v = 0.f; x.s = 0.f;
			if (bs != VXB_RAY_MISS)
			{
				const vxb_block_record* rec = surf.record(bs);
				float3 a, b, c;
				surf.corners(rec, bk, a, b, c);
				float3 pq, px;
				vxb_pair_fields(p, h, a, b, c, pq, px, x.u, x.v, x.s);
				x.point[0] = pq.x; x.point[1] = pq.y; x.point[2] = pq.z;
				x.axis_point[0] = px.x; x.axis_point[1] = px.y; x.axis_point[2] = px.z;
				x.distance = VXB_SQRT(bd); x.slot = bs; x.block_id = __ldg(&rec->id); x.triangle = surf.triangle(bk);
				surf.normal(rec, bk, x.u, x.v, x.normal);
			}
			surf.tail(x, bs, bk);
			hits[q] = x;
		}
	}
}

// ---- the ten kernels ---------------------------------------------------------------------------------------------------
// Named per shape and surface, each with its own measured launch bounds (DESIGN.md section 6).

__global__ void __launch_bounds__(VXB_RAY_THREADS) vxb_raycast_kernel(const VxbRayMesh m, const vxb_ray* __restrict__ rays, unsigned count,
	vxb_ray_hit* __restrict__ hits)
{
	vxb_raycast_body(VxbLevel0Surface{ m }, rays, count, hits);
}

__global__ void __launch_bounds__(VXB_RAY_THREADS) vxb_raycast_cut_kernel(const VxbCutRayMesh c, const vxb_ray* __restrict__ rays, unsigned count,
	vxb_cut_hit* __restrict__ hits)
{
	vxb_raycast_body(VxbCutSurface{ c }, rays, count, hits);
}

__global__ void __launch_bounds__(VXB_COLLIDE_THREADS) vxb_sphere_cast_kernel(const VxbRayMesh m, const float r, const vxb_ray* __restrict__ rays,
	unsigned count, vxb_sphere_hit* __restrict__ hits)
{
	vxb_sphere_cast_body(VxbLevel0Surface{ m }, r, rays, count, hits);
}

// (A minimum of one CTA per SM in the launch bounds: without it ptxas holds this kernel to 64 registers and spills.)
__global__ void __launch_bounds__(VXB_COLLIDE_THREADS, 1) vxb_sphere_cast_cut_kernel(const VxbCutRayMesh c, const float r,
	const vxb_ray* __restrict__ rays, unsigned count, vxb_sphere_cut_hit* __restrict__ hits)
{
	vxb_sphere_cast_body(VxbCutSurface{ c }, r, rays, count, hits);
}

__global__ void __launch_bounds__(VXB_COLLIDE_THREADS) vxb_closest_point_kernel(const VxbRayMesh m, const float maxDistance,
	const float* __restrict__ points, unsigned count, vxb_closest_hit* __restrict__ hits)
{
	vxb_closest_point_body(VxbLevel0Surface{ m }, maxDistance, points, count, hits);
}

__global__ void __launch_bounds__(VXB_COLLIDE_THREADS) vxb_closest_point_cut_kernel(const VxbCutRayMesh c, const float maxDistance,
	const float* __restrict__ points, unsigned count, vxb_closest_cut_hit* __restrict__ hits)
{
	vxb_closest_point_body(VxbCutSurface{ c }, maxDistance, points, count, hits);
}

__global__ void __launch_bounds__(VXB_COLLIDE_THREADS) vxb_capsule_cast_kernel(const VxbRayMesh m, const vxb_capsule_sweep* __restrict__ sweeps,
	unsigned count, vxb_capsule_hit* __restrict__ hits)
{
	vxb_capsule_cast_body(VxbLevel0Surface{ m }, sweeps, count, hits);
}

// (Two CTAs per SM in the launch bounds: ptxas then fits the kernel in 127 registers without a stack frame or spills, the
// occupancy of vxb_capsule_cast_kernel; with one CTA per SM it takes 136 registers and runs slower, DESIGN.md section 6.)
__global__ void __launch_bounds__(VXB_COLLIDE_THREADS, 2) vxb_capsule_cast_cut_kernel(const VxbCutRayMesh c,
	const vxb_capsule_sweep* __restrict__ sweeps, unsigned count, vxb_capsule_cut_hit* __restrict__ hits)
{
	vxb_capsule_cast_body(VxbCutSurface{ c }, sweeps, count, hits);
}

// (A minimum of one CTA per SM in the launch bounds: without it ptxas holds this kernel to 64 registers and spills.)
__global__ void __launch_bounds__(VXB_COLLIDE_THREADS, 1) vxb_closest_segment_kernel(const VxbRayMesh m, const float maxDistance,
	const vxb_segment* __restrict__ segments, unsigned count, vxb_segment_hit* __restrict__ hits)
{
	vxb_closest_segment_body(VxbLevel0Surface{ m }, maxDistance, segments, count, hits);
}

// (A minimum of one CTA per SM in the launch bounds, as vxb_closest_segment_kernel.)
__global__ void __launch_bounds__(VXB_COLLIDE_THREADS, 1) vxb_closest_segment_cut_kernel(const VxbCutRayMesh c, const float maxDistance,
	const vxb_segment* __restrict__ segments, unsigned count, vxb_segment_cut_hit* __restrict__ hits)
{
	vxb_closest_segment_body(VxbCutSurface{ c }, maxDistance, segments, count, hits);
}
