// SDF programs (include/vxb200.h vxb_op): a client-composed surface, the device-side analogue of a client's
// Voxels::VoxelSurface (reference include/VoxelSurface.h:35-40) that is data instead of a callback.  Written once and compiled
//   * by nvcc as __device__ code for the fill / edit kernels (vxb_grid.cuh), and
//   * by g++ as plain inline C++ for the VoxelSurface adapter of the test harness (tests/harness/vxh_capi.cpp), which feeds
//     the UNMODIFIED reference grid store,
// under the discipline of vxb_surfaces.h: +, -, *, /, sqrt, floor, fabs and compare-selects in a fixed order, no FMA
// contraction, so that both sides evaluate bit-identical floats.  SPHERE, PLANE and TERRAIN are vxs_surface_value itself.
//
// Two evaluators of the same op sequence:
//   vxp_eval        float, one sample: the value the grid store quantises + the material / blend of the selected primitive
//   vxp_eval_box    double interval arithmetic over a box of samples with a bound on the float rounding error: the per-block
//                   cull decision of the fill (vxp_block_cull), identical on the device and on the host
// Both keep the value stack in an array indexed only by constants (the top is element 0, push / pop shift the array), so the
// device code holds it in registers.
#pragma once
#include <stdint.h>

#include "vxb_surfaces.h"

#if defined(__CUDACC__)
#define VXP_FABS(x) fabsf(x)
#define VXP_DSQRT(x) sqrt(x)
#else
#define VXP_FABS(x) std::fabs(x)
#define VXP_DSQRT(x) std::sqrt(x)
#endif

// ---- validation (host) -----------------------------------------------------------------------------------------------
inline bool vxp_finite(float v) { return v == v && v - v == 0.f; }

// -1 when the program is well formed; else the index of the offending op (count: the state at the end) and the reason
inline int vxp_validate(const vxb_op* ops, uint32_t count, const char** why)
{
	*why = "";
	if (!ops || count == 0) { *why = "empty program"; return 0; }
	if (count > VXB_PROGRAM_MAX_OPS) { *why = "more than VXB_PROGRAM_MAX_OPS ops"; return VXB_PROGRAM_MAX_OPS; }
	int depth = 0, terrain = 0;
	for (uint32_t i = 0; i < count; ++i)
	{
		const vxb_op& o = ops[i];
		for (int k = 0; k < 12; ++k) if (!vxp_finite(o.xform[k])) { *why = "non-finite xform"; return (int)i; }
		for (int k = 0; k < 8; ++k) if (!vxp_finite(o.p[k])) { *why = "non-finite parameter"; return (int)i; }
		const float* p = o.p;
		switch (o.code)
		{
		case VXB_OP_SPHERE: if (p[0] < 0.f) { *why = "negative radius"; return (int)i; } break;
		case VXB_OP_BOX: if (p[0] < 0.f || p[1] < 0.f || p[2] < 0.f) { *why = "negative half extent"; return (int)i; } break;
		case VXB_OP_CYLINDER:
		case VXB_OP_CAPSULE:
		case VXB_OP_TORUS: if (p[0] < 0.f || p[1] < 0.f) { *why = "negative radius or length"; return (int)i; } break;
		case VXB_OP_PLANE: break;
		case VXB_OP_TERRAIN:
			if (!(p[0] > 0.f)) { *why = "terrain period N <= 0"; return (int)i; }
			if (++terrain > VXB_PROGRAM_MAX_TERRAIN) { *why = "more than VXB_PROGRAM_MAX_TERRAIN TERRAIN ops"; return (int)i; }
			break;
		case VXB_OP_UNION: case VXB_OP_INTERSECT: case VXB_OP_SUBTRACT: break;
		case VXB_OP_SMOOTH_UNION: if (!(p[0] > 0.f)) { *why = "smooth union k <= 0"; return (int)i; } break;
		case VXB_OP_OFFSET: break;
		case VXB_OP_SHELL: if (p[0] < 0.f) { *why = "negative shell thickness"; return (int)i; } break;
		default: *why = "unknown op code"; return (int)i;
		}
		if (o.code < 16)
		{
			if (o.material > 255 || o.blend > 255) { *why = "material or blend > 255"; return (int)i; }
			if (++depth > VXB_PROGRAM_MAX_DEPTH) { *why = "stack deeper than VXB_PROGRAM_MAX_DEPTH"; return (int)i; }
		}
		else if (o.code < 32) { if (depth < 2) { *why = "stack underflow"; return (int)i; } --depth; }
		else if (depth < 1) { *why = "stack underflow"; return (int)i; }
	}
	if (depth != 1) { *why = "the program does not leave exactly one value"; return (int)count; }
	return -1;
}

// ---- float evaluation (the values the grid store quantises) ---------------------------------------------------------
VXS_FN float vxp_min(float a, float b) { return b < a ? b : a; }   // ties: the left operand
VXS_FN float vxp_max(float a, float b) { return b > a ? b : a; }

// sample coordinate i of an axis of a fill (= vxb_fill_coord: the block's start, then k steps inside the block)
VXS_FN float vxp_fill_coord(float start, float step, int i) { return (start + (float)(i & ~15) * step) + (float)(i & 15) * step; }

// primitive op `o` at grid point (x, y, z): clamped distance, material | blend << 8
VXS_FN float vxp_primitive(const vxb_op& o, const unsigned char* perm, float x, float y, float z, unsigned& mb)
{
	const float* m = o.xform;
	const float qx = ((m[0] * x + m[1] * y) + m[2] * z) + m[9];
	const float qy = ((m[3] * x + m[4] * y) + m[5] * z) + m[10];
	const float qz = ((m[6] * x + m[7] * y) + m[8] * z) + m[11];
	const float* p = o.p;
	mb = o.material | (o.blend << 8);
	float d;
	switch (o.code)
	{
	case VXB_OP_SPHERE:
	case VXB_OP_PLANE:
	case VXB_OP_TERRAIN:
	{
		// vxs_surface_value: sphere centred at the local origin, the plane and the terrain as they are (already clamped)
		vxb_surface s;
		s.kind = o.code == VXB_OP_SPHERE ? VXB_SURFACE_SPHERE : (o.code == VXB_OP_PLANE ? VXB_SURFACE_PLANE : VXB_SURFACE_TERRAIN);
		s.material = o.material; s.blend = o.blend; s.seed = o.seed;
		for (int k = 0; k < 8; ++k) s.p[k] = 0.f;
		if (o.code == VXB_OP_SPHERE) s.p[3] = p[0];
		else { s.p[0] = p[0]; s.p[1] = p[1]; s.p[2] = p[2]; s.p[3] = p[3]; }
		unsigned sm, sb;
		const float v = vxs_surface_value(s, perm, qx, qy, qz, sm, sb);
		mb = sm | (sb << 8);
		return v;
	}
	case VXB_OP_BOX:
	{
		const float ex = VXP_FABS(qx) - p[0], ey = VXP_FABS(qy) - p[1], ez = VXP_FABS(qz) - p[2];
		const float mx = vxp_max(ex, 0.f), my = vxp_max(ey, 0.f), mz = vxp_max(ez, 0.f);
		d = VXS_SQRT((mx * mx + my * my) + mz * mz) + vxp_min(vxp_max(ex, vxp_max(ey, ez)), 0.f);
		break;
	}
	case VXB_OP_CYLINDER:
	{
		const float a = VXS_SQRT(qx * qx + qy * qy) - p[0], b = VXP_FABS(qz) - p[1];
		const float ma = vxp_max(a, 0.f), mb2 = vxp_max(b, 0.f);
		d = vxp_min(vxp_max(a, b), 0.f) + VXS_SQRT(ma * ma + mb2 * mb2);
		break;
	}
	case VXB_OP_CAPSULE:
	{
		const float c = qz - vxs_clampf(qz, -p[1], p[1]);
		d = VXS_SQRT((qx * qx + qy * qy) + c * c) - p[0];
		break;
	}
	default: // VXB_OP_TORUS
	{
		const float a = VXS_SQRT(qx * qx + qy * qy) - p[0];
		d = VXS_SQRT(a * a + qz * qz) - p[1];
		break;
	}
	}
	return vxs_clampf(d, -100.f, 100.f);
}

// The program at one grid point: final distance (clamped to +-100) and the material / blend of the value that was selected.
// perms = VXB_PROGRAM_MAX_TERRAIN tables of 512 bytes, one per TERRAIN op in program order.
VXS_FN float vxp_eval(const vxb_op* ops, int count, const unsigned char* perms, float x, float y, float z, unsigned& mat, unsigned& blend)
{
	float s[VXB_PROGRAM_MAX_DEPTH];
	unsigned w[VXB_PROGRAM_MAX_DEPTH];
#pragma unroll
	for (int k = 0; k < VXB_PROGRAM_MAX_DEPTH; ++k) { s[k] = 0.f; w[k] = 0u; }
	int terrain = 0;
	for (int i = 0; i < count; ++i)
	{
		const vxb_op& o = ops[i];
		const unsigned c = o.code;
		if (c < 16u)
		{
			unsigned mb;
			const float v = vxp_primitive(o, perms + 512 * terrain, x, y, z, mb);
			if (c == VXB_OP_TERRAIN) ++terrain;
#pragma unroll
			for (int k = VXB_PROGRAM_MAX_DEPTH - 1; k > 0; --k) { s[k] = s[k - 1]; w[k] = w[k - 1]; }
			s[0] = v; w[0] = mb;
		}
		else if (c < 32u)
		{
			const float a = s[1], b = s[0];
			float v;
			bool right; // the result takes the material of b
			if (c == VXB_OP_UNION) { right = b < a; v = right ? b : a; }
			else if (c == VXB_OP_INTERSECT) { right = b > a; v = right ? b : a; }
			else if (c == VXB_OP_SUBTRACT) { const float nb = -b; right = nb > a; v = right ? nb : a; }
			else
			{
				// polynomial smooth minimum
				const float k = o.p[0];
				const float h = VXS_DIV(vxp_max(k - VXP_FABS(a - b), 0.f), k);
				right = b < a;
				v = (right ? b : a) - ((h * h) * k) * 0.25f;
			}
			const unsigned mb = right ? w[0] : w[1];
			s[0] = v; w[0] = mb;
#pragma unroll
			for (int k = 1; k < VXB_PROGRAM_MAX_DEPTH - 1; ++k) { s[k] = s[k + 1]; w[k] = w[k + 1]; }
		}
		else if (c == VXB_OP_OFFSET) s[0] = s[0] - o.p[0];
		else s[0] = VXP_FABS(s[0]) - o.p[0]; // VXB_OP_SHELL
	}
	mat = w[0] & 0xFFu;
	blend = w[0] >> 8;
	return vxs_clampf(s[0], -100.f, 100.f);
}

// ---- interval evaluation (the per-block cull of the fill) ------------------------------------------------------------
// A value of the interval pass: every exact (real-number) value of the expression over the box lies in [lo, hi], and the
// float the per-voxel pass computes for any sample of the box differs from that sample's exact value by at most e.
//
// The margin mu of a decision is this e, derived op by op from the magnitudes the interval already has.  With
// u = 2^-24 (float round-to-nearest) every float op returns fl(r) = r (1 + d), |d| <= u, so for operands carrying errors
// Ea, Eb and magnitudes Ma = max(|lo|, |hi|):
//   a +- b       Ea + Eb + u (M(result) + Ea + Eb)
//   a * b        Ma Eb + Mb Ea + Ea Eb + u (Ma + Ea)(Mb + Eb)        (b an exact constant: Eb = 0)
//   a / k        (Ea + u (Ma + Ea)) / |k|                             (k an exact constant)
//   sqrt(a)      min(sqrt(Ea), Ea / sqrt(lo)) + u sqrt(hi + Ea)      (|sqrt x - sqrt y| <= |x - y| / sqrt y, <= sqrt |x - y|)
//   |a|, -a, min, max, clamp    max(Ea, Eb): 1-Lipschitz and exact in float
// The sample coordinates are the exact floats of the per-voxel pass (e = 0).  The endpoints themselves are computed in
// double (relative error 2^-53 per op); VXP_U adds 2^-40 to u, which covers that with a wide margin.
struct VxpIv
{
	double lo, hi, e;
};
#define VXP_U (5.9604644775390625e-08 + 9.094947017729282e-13) // 2^-24 + 2^-40

VXS_FN double vxp_dmax(double a, double b) { return b > a ? b : a; }
VXS_FN double vxp_dmin(double a, double b) { return b < a ? b : a; }
VXS_FN double vxp_mag(const VxpIv& a) { return vxp_dmax(a.lo < 0. ? -a.lo : a.lo, a.hi < 0. ? -a.hi : a.hi); }
VXS_FN VxpIv vxp_iv(double lo, double hi, double e) { VxpIv r; r.lo = lo; r.hi = hi; r.e = e; return r; }
VXS_FN VxpIv vxp_const(float c) { return vxp_iv(c, c, 0.); }
VXS_FN VxpIv vxp_add(const VxpIv& a, const VxpIv& b)
{
	VxpIv r = vxp_iv(a.lo + b.lo, a.hi + b.hi, 0.);
	r.e = (a.e + b.e) + VXP_U * ((vxp_mag(r) + a.e) + b.e);
	return r;
}
VXS_FN VxpIv vxp_sub(const VxpIv& a, const VxpIv& b)
{
	VxpIv r = vxp_iv(a.lo - b.hi, a.hi - b.lo, 0.);
	r.e = (a.e + b.e) + VXP_U * ((vxp_mag(r) + a.e) + b.e);
	return r;
}
VXS_FN VxpIv vxp_mul(const VxpIv& a, const VxpIv& b)
{
	const double p0 = a.lo * b.lo, p1 = a.lo * b.hi, p2 = a.hi * b.lo, p3 = a.hi * b.hi;
	const double ma = vxp_mag(a), mb = vxp_mag(b);
	return vxp_iv(vxp_dmin(vxp_dmin(p0, p1), vxp_dmin(p2, p3)), vxp_dmax(vxp_dmax(p0, p1), vxp_dmax(p2, p3)),
		((ma * b.e + mb * a.e) + a.e * b.e) + VXP_U * ((ma + a.e) * (mb + b.e)));
}
VXS_FN VxpIv vxp_sqr(const VxpIv& a) // a * a (the same float op; the interval knows it is a square)
{
	const double l2 = a.lo * a.lo, h2 = a.hi * a.hi, ma = vxp_mag(a);
	const double lo = a.lo >= 0. ? l2 : (a.hi <= 0. ? h2 : 0.);
	return vxp_iv(lo, vxp_dmax(l2, h2), (2. * ma * a.e + a.e * a.e) + VXP_U * ((ma + a.e) * (ma + a.e)));
}
VXS_FN VxpIv vxp_div(const VxpIv& a, float k) // k > 0, exact
{
	return vxp_iv(a.lo / k, a.hi / k, (a.e + VXP_U * (vxp_mag(a) + a.e)) / k);
}
VXS_FN VxpIv vxp_sqrt(const VxpIv& a)
{
	const double lo = a.lo > 0. ? a.lo : 0., hi = a.hi > 0. ? a.hi : 0.;
	const double slo = VXP_DSQRT(lo);
	double prop = VXP_DSQRT(a.e);
	if (slo > 0.) prop = vxp_dmin(prop, a.e / slo);
	return vxp_iv(slo, VXP_DSQRT(hi), prop + VXP_U * VXP_DSQRT(hi + a.e));
}
VXS_FN VxpIv vxp_abs(const VxpIv& a)
{
	if (a.lo >= 0.) return a;
	if (a.hi <= 0.) return vxp_iv(-a.hi, -a.lo, a.e);
	return vxp_iv(0., vxp_dmax(-a.lo, a.hi), a.e);
}
VXS_FN VxpIv vxp_neg(const VxpIv& a) { return vxp_iv(-a.hi, -a.lo, a.e); }
VXS_FN VxpIv vxp_imin(const VxpIv& a, const VxpIv& b) { return vxp_iv(vxp_dmin(a.lo, b.lo), vxp_dmin(a.hi, b.hi), vxp_dmax(a.e, b.e)); }
VXS_FN VxpIv vxp_imax(const VxpIv& a, const VxpIv& b) { return vxp_iv(vxp_dmax(a.lo, b.lo), vxp_dmax(a.hi, b.hi), vxp_dmax(a.e, b.e)); }
VXS_FN VxpIv vxp_clamp(const VxpIv& a, double lo, double hi)
{
	return vxp_iv(vxp_dmin(vxp_dmax(a.lo, lo), hi), vxp_dmin(vxp_dmax(a.hi, lo), hi), a.e);
}
// clamp to +-100 (the primitives and the final value).  Where every float is past a bound the result is that bound
// exactly, in float and in exact arithmetic alike (e = 0): far from every primitive all of them clamp to 100 and tie.
VXS_FN VxpIv vxp_clamp100(const VxpIv& a)
{
	if (a.lo - a.e >= 100.) return vxp_iv(100., 100., 0.);
	if (a.hi + a.e <= -100.) return vxp_iv(-100., -100., 0.);
	return vxp_clamp(a, -100., 100.);
}
// every float of `a` is below every float of `b` (strictly / or equal): a compare-select decides the same way at every
// sample.  Ties go to the left operand, so `left <= right` everywhere decides a min for the left one.
VXS_FN bool vxp_below(const VxpIv& a, const VxpIv& b) { return a.hi + a.e < b.lo - b.e; }
VXS_FN bool vxp_below_eq(const VxpIv& a, const VxpIv& b) { return a.hi + a.e <= b.lo - b.e; }

// ((m0 x + m1 y) + m2 z) + t over the box, in the float op order of vxp_primitive
VXS_FN VxpIv vxp_row(const float* m, float t, const VxpIv& x, const VxpIv& y, const VxpIv& z)
{
	return vxp_add(vxp_add(vxp_add(vxp_mul(vxp_const(m[0]), x), vxp_mul(vxp_const(m[1]), y)), vxp_mul(vxp_const(m[2]), z)), vxp_const(t));
}

// primitive op `o` over the box; its material is constant unless it is TERRAIN
VXS_FN VxpIv vxp_primitive_box(const vxb_op& o, const VxpIv& x, const VxpIv& y, const VxpIv& z)
{
	const float* m = o.xform;
	const VxpIv qx = vxp_row(m, m[9], x, y, z), qy = vxp_row(m + 3, m[10], x, y, z), qz = vxp_row(m + 6, m[11], x, y, z);
	const float* p = o.p;
	const VxpIv zero = vxp_const(0.f);
	VxpIv d;
	switch (o.code)
	{
	case VXB_OP_SPHERE:
		d = vxp_sub(vxp_sqrt(vxp_add(vxp_add(vxp_sqr(qx), vxp_sqr(qy)), vxp_sqr(qz))), vxp_const(p[0]));
		break;
	case VXB_OP_PLANE:
		d = vxp_sub(vxp_add(vxp_add(vxp_mul(vxp_const(p[0]), qx), vxp_mul(vxp_const(p[1]), qy)), vxp_mul(vxp_const(p[2]), qz)), vxp_const(p[3]));
		break;
	case VXB_OP_TERRAIN:
	{
		// d = (z - height) + 6 noise3, height = 0.5 N + 0.18 N fbm2.  |noise3| <= 2 (every corner's gradient dot product is
		// +-u +- v with |u|, |v| <= 1, the trilinear weights sum to 1), so |fbm2| <= 2 (1 + 1/2 + 1/4 + 1/8 + 1/16); 2.01
		// instead of 2 absorbs the float rounding of the noise (relative 1e-6).  Error of the two outer float ops:
		// 4u (|z| + 1.2 N + 13).
		const double N = p[0], nb = 2.01, hdev = 0.18 * N * (1.9375 * nb);
		const double h0 = 0.5 * N - hdev, h1 = 0.5 * N + hdev;
		d = vxp_iv(qz.lo - h1 - 6. * nb, qz.hi - h0 + 6. * nb, qz.e + 4. * VXP_U * (vxp_mag(qz) + 1.2 * N + 13.));
		break;
	}
	case VXB_OP_BOX:
	{
		const VxpIv ex = vxp_sub(vxp_abs(qx), vxp_const(p[0])), ey = vxp_sub(vxp_abs(qy), vxp_const(p[1])), ez = vxp_sub(vxp_abs(qz), vxp_const(p[2]));
		const VxpIv mx = vxp_imax(ex, zero), my = vxp_imax(ey, zero), mz = vxp_imax(ez, zero);
		d = vxp_add(vxp_sqrt(vxp_add(vxp_add(vxp_sqr(mx), vxp_sqr(my)), vxp_sqr(mz))), vxp_imin(vxp_imax(ex, vxp_imax(ey, ez)), zero));
		break;
	}
	case VXB_OP_CYLINDER:
	{
		const VxpIv a = vxp_sub(vxp_sqrt(vxp_add(vxp_sqr(qx), vxp_sqr(qy))), vxp_const(p[0])), b = vxp_sub(vxp_abs(qz), vxp_const(p[1]));
		d = vxp_add(vxp_imin(vxp_imax(a, b), zero), vxp_sqrt(vxp_add(vxp_sqr(vxp_imax(a, zero)), vxp_sqr(vxp_imax(b, zero)))));
		break;
	}
	case VXB_OP_CAPSULE:
	{
		const VxpIv c = vxp_sub(qz, vxp_clamp(qz, -p[1], p[1]));
		d = vxp_sub(vxp_sqrt(vxp_add(vxp_add(vxp_sqr(qx), vxp_sqr(qy)), vxp_sqr(c))), vxp_const(p[0]));
		break;
	}
	default: // VXB_OP_TORUS
	{
		const VxpIv a = vxp_sub(vxp_sqrt(vxp_add(vxp_sqr(qx), vxp_sqr(qy))), vxp_const(p[0]));
		d = vxp_sub(vxp_sqrt(vxp_add(vxp_sqr(a), vxp_sqr(qz))), vxp_const(p[1]));
		break;
	}
	}
	return vxp_clamp100(d);
}

// The program over the box [x] x [y] x [z].  sel = the primitive whose material every sample ends with, or -1 when a
// compare-select on the chain that reaches the result is not decided the same way over the whole box (or the selected
// primitive is TERRAIN, whose material varies).
VXS_FN VxpIv vxp_eval_box(const vxb_op* ops, int count, const VxpIv& x, const VxpIv& y, const VxpIv& z, int& sel)
{
	VxpIv s[VXB_PROGRAM_MAX_DEPTH];
	int w[VXB_PROGRAM_MAX_DEPTH];
#pragma unroll
	for (int k = 0; k < VXB_PROGRAM_MAX_DEPTH; ++k) { s[k] = vxp_const(0.f); w[k] = -1; }
	for (int i = 0; i < count; ++i)
	{
		const vxb_op& o = ops[i];
		const unsigned c = o.code;
		if (c < 16u)
		{
			const VxpIv v = vxp_primitive_box(o, x, y, z);
#pragma unroll
			for (int k = VXB_PROGRAM_MAX_DEPTH - 1; k > 0; --k) { s[k] = s[k - 1]; w[k] = w[k - 1]; }
			s[0] = v; w[0] = c == VXB_OP_TERRAIN ? -1 : i;
		}
		else if (c < 32u)
		{
			const VxpIv a = s[1], b = s[0];
			VxpIv v;
			int ws;
			if (c == VXB_OP_INTERSECT || c == VXB_OP_SUBTRACT)
			{
				const VxpIv bb = c == VXB_OP_SUBTRACT ? vxp_neg(b) : b;   // max(a, bb): bb wins when bb > a
				v = vxp_imax(a, bb);
				ws = vxp_below(a, bb) ? w[0] : (vxp_below_eq(bb, a) ? w[1] : -1);
			}
			else
			{
				const VxpIv mn = vxp_imin(a, b);                          // min(a, b): b wins when b < a
				ws = vxp_below(b, a) ? w[0] : (vxp_below_eq(a, b) ? w[1] : -1);
				if (c == VXB_OP_UNION) v = mn;
				else
				{
					const float k = o.p[0];
					const VxpIv h = vxp_div(vxp_imax(vxp_sub(vxp_const(k), vxp_abs(vxp_sub(a, b))), vxp_const(0.f)), k);
					v = vxp_sub(mn, vxp_mul(vxp_mul(vxp_sqr(h), vxp_const(k)), vxp_const(0.25f)));
				}
			}
			s[0] = v; w[0] = ws;
#pragma unroll
			for (int k = 1; k < VXB_PROGRAM_MAX_DEPTH - 1; ++k) { s[k] = s[k + 1]; w[k] = w[k + 1]; }
		}
		else if (c == VXB_OP_OFFSET) s[0] = vxp_sub(s[0], vxp_const(o.p[0]));
		else s[0] = vxp_sub(vxp_abs(s[0]), vxp_const(o.p[0]));
	}
	sel = w[0];
	return vxp_clamp100(s[0]);
}

// Cull decision of fill block (bx, by, bz): 1 when every sample of the block quantises to the same +-4 with the material and
// blend of one primitive (returned in dist / mat / blend), 0 when the block needs the per-voxel pass.  A float value v
// quantises to +4 exactly when v > 3 (round away from zero, clamp +-4), so the bound is 3 plus the error e.
VXS_FN int vxp_block_cull(const vxb_op* ops, int count, const float start[3], float step, int bx, int by, int bz, int& dist, unsigned& mat, unsigned& blend)
{
	VxpIv box[3];
	const int b[3] = { bx, by, bz };
	for (int k = 0; k < 3; ++k)
	{
		const double c0 = vxp_fill_coord(start[k], step, b[k] * 16), c1 = vxp_fill_coord(start[k], step, b[k] * 16 + 15);
		box[k] = vxp_iv(vxp_dmin(c0, c1), vxp_dmax(c0, c1), 0.);   // the samples of a block are monotonic in k
	}
	int sel;
	const VxpIv v = vxp_eval_box(ops, count, box[0], box[1], box[2], sel);
	if (sel < 0) return 0;
	if (v.lo - v.e > 3.) dist = 4;
	else if (v.hi + v.e < -3.) dist = -4;
	else return 0;
	mat = ops[sel].material;
	blend = ops[sel].blend;
	return 1;
}
