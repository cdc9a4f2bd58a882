// Sphere sweeps and closest-point queries against the level-0 triangles of the resident mesh (include/vxb200.h "collision
// queries").  Both use the level-0 block map of the ray casts (vxb_ray.cuh) and its rules.
//
//   sweeps          vxb_ray_walk with the block boxes grown by r + VXB_RAY_EPS; the proof of the walk, extended to that
//                   growth, is at the top of vxb_ray.cuh.
//   closest points  no walk: the 27 neighbours of the query's clamped block (vxb_point_candidate, with the proof).
//   capsules        the same two routes with the reach |h_i| + r (sweeps: the walk grown by max_i |h_i| + r + eps) or
//                   |h_i| + max_distance (segments: the per-axis box gap instead of the distance); see "capsules" below.
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

// The sweep's face test: the plane of (a, b, c) offset by r toward the side of c0, as a Moeller-Trumbore cast of the ray
// moved by -r along that side (+inf when it fails).  Quad: the parallelogram a, b, b + c - a (v <= 1 in place of u + v <= 1).
template <bool Quad>
VXB_FN float vxb_sweep_face(const float3 o, const float3 d, const float3 c0, float r, float tMin, float tMax, const float3 a,
	const float3 b, const float3 c)
{
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
	return (side >= 0.f ? det > 0.f : det < 0.f) && fu >= 0.f && fu <= 1.f && fv >= 0.f && (Quad ? fv <= 1.f : fu + fv <= 1.f) &&
		ft >= tMin && ft <= tMax ? ft : CUDART_INF_F;
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
	float t = vxb_sweep_face<false>(o, d, c0, r, tMin, tMax, a, b, c);
	// the edges ab, bc, ca, then the vertices a, b, c
	t = fminf(t, vxb_sweep_edge(o, d, a, b, rr, tMin, tMax));
	t = fminf(t, vxb_sweep_edge(o, d, b, c, rr, tMin, tMax));
	t = fminf(t, vxb_sweep_edge(o, d, c, a, rr, tMin, tMax));
	t = fminf(t, vxb_sweep_vertex(o, d, a, rr, dd, tMin, tMax));
	t = fminf(t, vxb_sweep_vertex(o, d, b, rr, dd, tMin, tMax));
	t = fminf(t, vxb_sweep_vertex(o, d, c, rr, dd, tMin, tMax));
	return t;
}

// The point neighbourhood of the closest-point and closest-to-segment queries: this lane's candidate slot, neighbour k = lane
// (< 27) of the block of p clamped into the grid, when `ok` (the same for the whole warp) holds, the block lies in the grid
// and `at(bx, by, bz, slot)` yields a slot there (the surface's step: its box accepted by the shape's `near`, then its slot;
// VxbLevel0Surface::point, VxbCutSurface::point).
//   closest points  a triangle within max_distance of the query lies in a block whose box is within max_distance of the
//                   query (a level-0 triangle lies in the closed box of its block), and `near` rejects a block only when its
//                   box is farther than max_distance + VXB_RAY_EPS (the float box distance is within a few ulps of the true
//                   one; an accepted triangle is within max_distance plus rounding).  Such a block lies within max_distance +
//                   eps <= 15 + 1/16 < 16 of the query along every axis.  Along an axis where the query lies inside the grid,
//                   its index is that of the query's block +-1.  Along an axis where the query lies outside (below 0 or above
//                   n), only the first or last block of the axis is that close, and that is the clamped index.  So the 27
//                   neighbours of the clamped block hold every block that can contribute, for queries inside and outside the
//                   grid box alike.
//   segments        the same with the per-axis gap: `near` rejects a block only when its box is farther than |h_i| +
//                   max_distance + eps from the centre along some axis, and the reach rule keeps that below 16.
template <class At>
VXB_FN bool vxb_point_candidate(const int nb, const float3 p, bool ok, At&& at, unsigned& slot)
{
	const unsigned lane = threadIdx.x & 31;
	bool cand = false;
	slot = VXB_RAY_MISS;
	if (ok && lane < 27)
	{
		const float top = (float)(nb - 1);
		const int bx = (int)fminf(fmaxf(floorf(p.x * 0.0625f), 0.f), top) + (int)(lane % 3) - 1;
		const int by = (int)fminf(fmaxf(floorf(p.y * 0.0625f), 0.f), top) + (int)((lane / 3) % 3) - 1;
		const int bz = (int)fminf(fmaxf(floorf(p.z * 0.0625f), 0.f), top) + (int)(lane / 9) - 1;
		if (bx >= 0 && by >= 0 && bz >= 0 && bx < nb && by < nb && bz < nb) cand = at(bx, by, bz, slot);
	}
	return cand;
}

// ---- capsules (include/vxb200.h "capsule queries") ---------------------------------------------------------------------
//
// A capsule (segment c -+ h, radius r) touches triangle T exactly when the sphere of radius r at c touches the convex set
// P = T + [-h, h].  The sweep runs the sphere's tests on P's features:
//   no early contact   every face, edge and vertex tested lies in P, and each accepted test puts the centre within r (up to
//                      rounding) of a point of its feature, so no test fires before the first contact with P.
//   the faces cover P  take z = y + x h in P (y in T, |x| <= 1) and the parameters {s : z + s h in T} = [s0, s1], which hold
//                      -x.  If -1 or 1 is in it, z lies in the cap T + h or T - h; otherwise [s0, s1] lies inside (-1, 1),
//                      z + s0 h is on an edge of T and z lies in that edge's parallelogram.  This holds for any h, also
//                      one in T's plane, where P is flat.
//   first contact      at the first contact t*, the point z of P nearest the centre lies on a face F of that cover.  If the
//                      centre - z is normal to F, it is r from F's plane on the side the centre is on; that signed distance
//                      is affine in t and has not yet risen to r at t* from above, so c0 is on the same side: F's offset-
//                      plane test (side from c0) accepts t*.  Otherwise z is on F's boundary, an edge of T +- h or a lateral
//                      edge, and the cylinder test of that edge (or, at an end of it, the sphere test of the vertex) accepts
//                      t*.  A path parallel to F at distance r first touches F's boundary, so it is the same case.
// With h = 0 the caps are T, the parallelograms and the lateral edges have zero extent and fail (det = 0, A = 0), and the cap
// edges and shifted vertices are the sphere's: the contact t is the sphere sweep's.
//
// The per-triangle reject.  A contact puts the centre within |h_i| + r of its triangle along axis i (the capsule point paired
// with the contact is within r, and it is within |h_i| of the centre), so inside the triangle's box grown by g_i = |h_i| + r +
// VXB_RAY_EPS.  The reject runs the walk's slab test on that box: a triangle whose grown box the path misses has no contact,
// by the walk's argument at the top of vxb_ray.cuh (rounded planes and slab parameters stay far inside the eps slack).  The
// closest-to-segment query rejects a triangle (and skips a block) whose box is farther than |h_i| + max_distance + eps from
// the centre along some axis, for the same reason.  The reject never changes a result; it only avoids the full tests.

VXB_FN float vxb_clamp01(float x) { return x < 0.f ? 0.f : (x > 1.f ? 1.f : x); }

// Candidate 3 of the closest pair for the edge q0 -> q1 (Ericson's ClosestPtSegmentSegment, exact zero tests): dd (+inf when
// the segment has zero length), the edge point y at parameter t, and the segment parameter w.  p0, D: the segment p0 + w D;
// A = D.D.
VXB_FN float vxb_segment_edge(const float3 p0, const float3 D, float A, const float3 q0, const float3 q1, float3& y, float& t, float& w)
{
	t = 0.f; w = 0.f; y = q0;
	if (A == 0.f) return CUDART_INF_F;
	const float ex = q1.x - q0.x, ey = q1.y - q0.y, ez = q1.z - q0.z;
	const float rx = p0.x - q0.x, ry = p0.y - q0.y, rz = p0.z - q0.z;
	const float e = (ex * ex + ey * ey) + ez * ez;
	const float f = (ex * rx + ey * ry) + ez * rz;
	const float c = (D.x * rx + D.y * ry) + D.z * rz;
	if (e == 0.f) w = vxb_clamp01(VXB_DIV(-c, A));
	else
	{
		const float b = (D.x * ex + D.y * ey) + D.z * ez;
		const float den = A * e - b * b;
		w = den != 0.f ? vxb_clamp01(VXB_DIV(b * f - c * e, den)) : 0.f;
		t = VXB_DIV(b * w + f, e);
		if (t < 0.f) { t = 0.f; w = vxb_clamp01(VXB_DIV(-c, A)); }
		else if (t > 1.f) { t = 1.f; w = vxb_clamp01(VXB_DIV(b - c, A)); }
	}
	y = make_float3(q0.x + t * ex, q0.y + t * ey, q0.z + t * ez);
	return vxb_dist2(make_float3(p0.x + w * D.x, p0.y + w * D.y, p0.z + w * D.z), y);
}

// The closest pair of the segment ctr -+ h and triangle (a, b, c) in the order include/vxb200.h states: dd, the triangle point
// q with barycentrics (u, v), and the segment parameter w in [0, 1] (s = 2w - 1).
VXB_FN float vxb_segment_triangle(const float3 ctr, const float3 h, const float3 a, const float3 b, const float3 c, float3& q, float& u,
	float& v, float& w)
{
	const float3 p0 = make_float3(ctr.x - h.x, ctr.y - h.y, ctr.z - h.z);
	const float3 D = make_float3(h.x + h.x, h.y + h.y, h.z + h.z);
	vxb_closest_on_triangle(p0, a, b, c, q, u, v);
	float best = vxb_dist2(p0, q);
	w = 0.f;
	{
		const float3 p1 = make_float3(ctr.x + h.x, ctr.y + h.y, ctr.z + h.z);
		float3 q1; float u1, v1;
		vxb_closest_on_triangle(p1, a, b, c, q1, u1, v1);
		const float d1 = vxb_dist2(p1, q1);
		if (d1 < best) { best = d1; q = q1; u = u1; v = v1; w = 1.f; }
	}
	const float A = (D.x * D.x + D.y * D.y) + D.z * D.z;
	float3 y; float t, we;
	float de = vxb_segment_edge(p0, D, A, a, b, y, t, we);
	if (de < best) { best = de; q = y; u = t; v = 0.f; w = we; }
	de = vxb_segment_edge(p0, D, A, b, c, y, t, we);
	if (de < best) { best = de; q = y; u = 1.f - t; v = t; w = we; }
	de = vxb_segment_edge(p0, D, A, c, a, y, t, we);
	if (de < best) { best = de; q = y; u = 0.f; v = 1.f - t; w = we; }
	// the segment crossing the triangle: Moeller-Trumbore from p0 along D
	const float e1x = b.x - a.x, e1y = b.y - a.y, e1z = b.z - a.z;
	const float e2x = c.x - a.x, e2y = c.y - a.y, e2z = c.z - a.z;
	const float sx = p0.x - a.x, sy = p0.y - a.y, sz = p0.z - a.z;
	const float pvx = D.y * e2z - D.z * e2y, pvy = D.z * e2x - D.x * e2z, pvz = D.x * e2y - D.y * e2x;
	const float det = (e1x * pvx + e1y * pvy) + e1z * pvz;
	const float inv = VXB_DIV(1.f, det);
	const float fu = ((sx * pvx + sy * pvy) + sz * pvz) * inv;
	const float qvx = sy * e1z - sz * e1y, qvy = sz * e1x - sx * e1z, qvz = sx * e1y - sy * e1x;
	const float fv = ((D.x * qvx + D.y * qvy) + D.z * qvz) * inv;
	const float fw = ((e2x * qvx + e2y * qvy) + e2z * qvz) * inv;
	if (det != 0.f && fu >= 0.f && fu <= 1.f && fv >= 0.f && fu + fv <= 1.f && fw >= 0.f && fw <= 1.f && 0.f < best)
	{
		best = 0.f; u = fu; v = fv; w = fw;
		q = make_float3((a.x + e1x * fu) + e2x * fv, (a.y + e1y * fu) + e2y * fv, (a.z + e1z * fu) + e2z * fv);
	}
	return best;
}

// The first contact of the capsule (half axis h, radius r, centre o + t d, t in [t_min, t_max]) with triangle (a, b, c),
// include/vxb200.h "capsule sweep": +inf when there is none; `started` when it touches the triangle at t_min already.
VXB_FN float vxb_capsule_triangle(const float3 o, const float3 d, const float3 c0, const float3 h, float r, float rr, float dd, float tMin,
	float tMax, const float3 a, const float3 b, const float3 c, bool& started)
{
	started = false;
	{
		float3 q; float u, v, w;
		if (vxb_segment_triangle(c0, h, a, b, c, q, u, v, w) <= rr) { started = true; return tMin; }
	}
	const float3 am = make_float3(a.x - h.x, a.y - h.y, a.z - h.z), ap = make_float3(a.x + h.x, a.y + h.y, a.z + h.z);
	const float3 bm = make_float3(b.x - h.x, b.y - h.y, b.z - h.z), bp = make_float3(b.x + h.x, b.y + h.y, b.z + h.z);
	const float3 cm = make_float3(c.x - h.x, c.y - h.y, c.z - h.z), cp = make_float3(c.x + h.x, c.y + h.y, c.z + h.z);
	// the faces: the caps, then the parallelograms of ab, bc, ca
	float t = vxb_sweep_face<false>(o, d, c0, r, tMin, tMax, am, bm, cm);
	t = fminf(t, vxb_sweep_face<false>(o, d, c0, r, tMin, tMax, ap, bp, cp));
	t = fminf(t, vxb_sweep_face<true>(o, d, c0, r, tMin, tMax, am, bm, ap));
	t = fminf(t, vxb_sweep_face<true>(o, d, c0, r, tMin, tMax, bm, cm, bp));
	t = fminf(t, vxb_sweep_face<true>(o, d, c0, r, tMin, tMax, cm, am, cp));
	// the edges of the cap -h, of the cap +h, then the lateral edges
	t = fminf(t, vxb_sweep_edge(o, d, am, bm, rr, tMin, tMax));
	t = fminf(t, vxb_sweep_edge(o, d, bm, cm, rr, tMin, tMax));
	t = fminf(t, vxb_sweep_edge(o, d, cm, am, rr, tMin, tMax));
	t = fminf(t, vxb_sweep_edge(o, d, ap, bp, rr, tMin, tMax));
	t = fminf(t, vxb_sweep_edge(o, d, bp, cp, rr, tMin, tMax));
	t = fminf(t, vxb_sweep_edge(o, d, cp, ap, rr, tMin, tMax));
	t = fminf(t, vxb_sweep_edge(o, d, am, ap, rr, tMin, tMax));
	t = fminf(t, vxb_sweep_edge(o, d, bm, bp, rr, tMin, tMax));
	t = fminf(t, vxb_sweep_edge(o, d, cm, cp, rr, tMin, tMax));
	// the shifted vertices
	t = fminf(t, vxb_sweep_vertex(o, d, am, rr, dd, tMin, tMax));
	t = fminf(t, vxb_sweep_vertex(o, d, bm, rr, dd, tMin, tMax));
	t = fminf(t, vxb_sweep_vertex(o, d, cm, rr, dd, tMin, tMax));
	t = fminf(t, vxb_sweep_vertex(o, d, ap, rr, dd, tMin, tMax));
	t = fminf(t, vxb_sweep_vertex(o, d, bp, rr, dd, tMin, tMax));
	t = fminf(t, vxb_sweep_vertex(o, d, cp, rr, dd, tMin, tMax));
	return t;
}

// the reach of a capsule shape (include/vxb200.h), in float for the host pre-check and the kernels alike: a finite half axis
// and max_i |h_i| + extra <= VXB_SPHERE_RADIUS_MAX
VXB_HD bool vxb_capsule_reach(const float3 h, float extra)
{
	const float hm = fmaxf(fmaxf(fabsf(h.x), fabsf(h.y)), fabsf(h.z));
	return isfinite(h.x) && isfinite(h.y) && isfinite(h.z) && hm + extra <= VXB_SPHERE_RADIUS_MAX;
}

// The per-triangle reject of the sweep: whether the path meets the box of (a, b, c) grown by g along each axis.
VXB_FN bool vxb_path_meets_box(const vxb_ray& ray, const float3 g, const float3 a, const float3 b, const float3 c)
{
	float te = ray.t_min, tx = ray.t_max;
	vxb_ray_slab(ray.origin[0], ray.direction[0], fminf(fminf(a.x, b.x), c.x) - g.x, fmaxf(fmaxf(a.x, b.x), c.x) + g.x, te, tx);
	vxb_ray_slab(ray.origin[1], ray.direction[1], fminf(fminf(a.y, b.y), c.y) - g.y, fmaxf(fmaxf(a.y, b.y), c.y) + g.y, te, tx);
	vxb_ray_slab(ray.origin[2], ray.direction[2], fminf(fminf(a.z, b.z), c.z) - g.z, fmaxf(fmaxf(a.z, b.z), c.z) + g.z, te, tx);
	return te <= tx;
}

// the hit fields of the closest pair at `ctr`: point q, axis point x = ctr + s h, u, v and s = 2w - 1
VXB_FN void vxb_pair_fields(const float3 ctr, const float3 h, const float3 a, const float3 b, const float3 c, float3& q, float3& x,
	float& u, float& v, float& s)
{
	float w;
	vxb_segment_triangle(ctr, h, a, b, c, q, u, v, w);
	s = (w + w) - 1.f;
	x = make_float3(ctr.x + s * h.x, ctr.y + s * h.y, ctr.z + s * h.z);
}

// ---- the level-0 surface -----------------------------------------------------------------------------------------------
//
// The level-0 triangles as the query bodies (vxb_query.cuh) see them; VxbCutSurface (vxb_cutray.cuh) is the drawn cut's.
// A surface supplies the candidate blocks (the walk of a swept shape, the 27-neighbour step of a point shape), a block's
// triangles, the winning triangle, the capsule reach rule and the tail of the hit.  Keys are triangle indices.
struct VxbLevel0Surface
{
	const VxbRayMesh& m;

	// The walk of a shape whose reach splits as hm = max_i |h_i| and r (both 0 for rays, hm = -0 for spheres): the level-0
	// boxes grown by (hm + r) + VXB_RAY_EPS, which is max_i (|h_i| + r + eps) in float (rounding is monotone).
	template <class Block>
	VXB_FN void walk(const vxb_ray& ray, float hm, float r, const float& best, Block&& block) const
	{
		vxb_ray_walk(m, ray, (hm + r) + VXB_RAY_EPS, best, block);
	}

	// the point candidate: the block's lattice box [16 b, 16 b + 16] accepted by `near(lo, hi)`, then its map slot
	template <class Near>
	VXB_FN bool point(const float3 p, bool ok, Near&& near, unsigned& slot) const
	{
		const int nb = m.nb;
		return vxb_point_candidate(nb, p, ok, [&](int bx, int by, int bz, unsigned& s) {
			const float3 lo = make_float3((float)(16 * bx), (float)(16 * by), (float)(16 * bz));
			const float3 hi = make_float3((float)(16 * bx + 16), (float)(16 * by + 16), (float)(16 * bz + 16));
			if (!near(lo, hi)) return false;
			s = __ldg(&m.map[((unsigned)by * nb + (unsigned)bz) * nb + (unsigned)bx]);   // output y = grid z
			return s != VXB_RAY_MISS;
		}, slot);
	}

	template <class F>
	VXB_FN void triangles(unsigned s, F&& f) const { vxb_slot_triangles(m, s, f); }

	VXB_FN const vxb_block_record* record(unsigned s) const { return m.dir + s; }

	// the positions of the winning triangle k of the block at directory record rec, and its blended normal at (u, v)
	VXB_FN void corners(const vxb_block_record* rec, unsigned k, float3& p0, float3& p1, float3& p2) const
	{
		vxb_ray_triangle(m, __ldg(&rec->vertex_offset), __ldg(&rec->index_offset), k, p0, p1, p2);
	}
	VXB_FN void normal(const vxb_block_record* rec, unsigned k, float u, float v, float* out) const
	{
		vxb_blend_normal(m.verts, __ldg(&rec->vertex_offset), m.idx + __ldg(&rec->index_offset) + 3 * k, u, v, out);
	}

	VXB_FN unsigned triangle(unsigned k) const { return k; }

	VXB_FN bool reach(const float3 h, float extra) const { return vxb_capsule_reach(h, extra); }

	template <class Hit>
	VXB_FN void tail(Hit&, unsigned, unsigned) const {}
};
