// Per-cell / per-vertex arithmetic of the Transvoxel polygonizer, written once and compiled
//   * by nvcc as __device__ code for the sm_90a kernels (vxb_kernels.cuh), and
//   * by g++ as plain inline C++ for the CPU restatement under oracle/ (test infrastructure).
//
// Everything here restates what the reference computes per cell; the cross-cell structure
// (ordering, reuse, compaction) lives in the kernels.  Citations are reference file:line,
// all in /root/reference/src/TransVoxelImpl.cpp unless noted.
//
// Floating point: expressions keep the reference's operation order and must be compiled without
// FMA contraction (-fmad=false for nvcc; g++ without -mfma), so results are IEEE-identical.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define VXB_FN __device__ __forceinline__
#define VXB_FN_BIG __device__ __forceinline__ // the per-vertex helpers: inlined, a call would pass the vertex through local memory
#define VXB_HD __host__ __device__ __forceinline__ // a query rule the host pre-check and the kernels both evaluate
#define VXB_SQRT(x) __fsqrt_rn(x)
#define VXB_DIV(a, b) __fdiv_rn((a), (b))
#else
#include <cmath>
#define VXB_FN inline
#define VXB_FN_BIG inline
#define VXB_HD inline
#define VXB_SQRT(x) std::sqrt(x)
#define VXB_DIV(a, b) ((a) / (b))
#endif

#define VXB_BLOCK 16
#define VXB_EMPTY_MATERIAL 255 // VoxelGrid.h:15
#define VXB_NO_SLOT 0xF

// Internal face bits, grid (Z-up) axes: Cell::FaceId (:548-558)
enum { VXB_ZPOS = 0, VXB_YPOS = 1, VXB_XPOS = 2, VXB_ZNEG = 3, VXB_YNEG = 4, VXB_XNEG = 5 };

// Dense level-0 volumes, x fastest: index = (z*n + y)*n + x.
struct VxbGrid
{
	const signed char* dist;
	const unsigned char* mat;
	const unsigned char* blend;
	int n;
};

// Output vertex, byte-identical to Voxels::PolygonVertex (include/Polygonizer.h:14-48).
struct VxbVertex
{
	float pos[3];
	float sec[4];
	float nrm[3];
	uint32_t tex[2]; // bytes: Reserved, Blend, Uxz, Txz | Uny, Upy, Tny, Tpy
};

// Material id -> packed texture words (FillTextureIdsForVertex :1248-1264); blend is OR-ed into tex0 bits 8..15.
struct VxbMaterialLut
{
	uint32_t tex0[256];
	uint32_t tex1[256];
	uint8_t valid[256];
};

VXB_FN int vxb_clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

VXB_FN size_t vxb_index(const VxbGrid& g, int x, int y, int z)
{
	const int m = g.n - 1;
	x = vxb_clampi(x, 0, m); y = vxb_clampi(y, 0, m); z = vxb_clampi(z, 0, m);
	return ((size_t)z * g.n + y) * g.n + x;
}

// GridBlocksCache::GetGridValue(coord) :1140-1151 - coordinates are clamped to the grid.
VXB_FN int vxb_dist(const VxbGrid& g, int x, int y, int z) { return g.dist[vxb_index(g, x, y, z)]; }

// Level-0 block neighbourhood staged in shared memory (device only): distance samples for coordinates
// [origin-1, origin+17] per axis (19^3).  Clamping at the grid edges is baked in when the tile is filled.
struct VxbTileView
{
	const signed char* dist;     // 19 x 19 rows of 48 bytes, first sample = (sx, sy, sz)
	const unsigned char* mat;    // the global material / blend volumes (two taps per vertex: not worth a tile)
	const unsigned char* blend;
	int ox, oy, oz;              // block origin (grid coordinates of its first voxel)
	int sx, sy, sz;              // first coordinate held by the distance tile: (origin.x - 16, origin.y - 1, origin.z - 1)
	                             // - TMA needs a 16-byte aligned innermost start -, also on the low grid edge
	int n;                       // grid edge
};

// every tap of a level-0 vertex lies in [origin - 1, origin + 17]: the tile holds it, clamped values included
VXB_FN int vxb_dist(const VxbTileView& g, int x, int y, int z)
{
	return g.dist[((z - g.sz) * 19 + (y - g.sy)) * 48 + (x - g.sx)];
}
VXB_FN size_t vxb_tile_mat_index(const VxbTileView& g, int x, int y, int z)
{
	const int m = g.n - 1; // the two material taps of a vertex (cell corners) are clamped like every grid read (:1242-1244)
	return ((size_t)(z > m ? m : z) * g.n + (y > m ? m : y)) * g.n + (x > m ? m : x);
}
VXB_FN unsigned vxb_mat(const VxbTileView& g, int x, int y, int z) { return g.mat[vxb_tile_mat_index(g, x, y, z)]; }
VXB_FN unsigned vxb_blend(const VxbTileView& g, int x, int y, int z) { return g.blend[vxb_tile_mat_index(g, x, y, z)]; }
VXB_FN unsigned vxb_mat(const VxbGrid& g, int x, int y, int z) { return g.mat[vxb_index(g, x, y, z)]; }
VXB_FN unsigned vxb_blend(const VxbGrid& g, int x, int y, int z) { return g.blend[vxb_index(g, x, y, z)]; }

// Case code: bit i = sign bit of corner i (Cell::CalcCaseCode :741-750)
VXB_FN unsigned vxb_case_code(const signed char v[8])
{
	unsigned code = 0;
#pragma unroll
	for (int i = 0; i < 8; ++i) code |= (v[i] < 0 ? 1u : 0u) << i;
	return code;
}

// normalizeFixZero :93-103 (glm::length = sqrt((x*x + y*y) + z*z), component-wise true division)
VXB_FN void vxb_normalize_fix_zero(float& x, float& y, float& z)
{
	const float len = VXB_SQRT((x * x + y * y) + z * z);
	if (len <= 1.1920928955078125e-07f) { x = 0.f; y = 0.f; z = 0.f; return; }
	x = VXB_DIV(x, len); y = VXB_DIV(y, len); z = VXB_DIV(z, len);
}

// CalcNormal :1239-1246 - central differences on the level-0 grid, taps clamped (the point itself
// may lie at coordinate n); the result is already in output (Y-up) axes: (d/dx, d/dz, d/dy).
VXB_FN_BIG void vxb_normal(const VxbGrid& g, int x, int y, int z, float n[3])
{
	const int m = g.n - 1;
	const size_t nn = (size_t)g.n;
	const size_t x0 = (size_t)vxb_clampi(x - 1, 0, m), x1 = (size_t)vxb_clampi(x, 0, m), x2 = (size_t)vxb_clampi(x + 1, 0, m);
	const size_t y0 = (size_t)vxb_clampi(y - 1, 0, m) * nn, y1 = (size_t)vxb_clampi(y, 0, m) * nn, y2 = (size_t)vxb_clampi(y + 1, 0, m) * nn;
	const size_t z0 = (size_t)vxb_clampi(z - 1, 0, m) * nn * nn, z1 = (size_t)vxb_clampi(z, 0, m) * nn * nn, z2 = (size_t)vxb_clampi(z + 1, 0, m) * nn * nn;
	const signed char* d = g.dist;
	const int ax = d[z1 + y1 + x2], bx = d[z1 + y1 + x0];
	const int az = d[z2 + y1 + x1], bz = d[z0 + y1 + x1];
	const int ay = d[z1 + y2 + x1], by = d[z1 + y0 + x1];
	n[0] = (float)(ax - bx) * 0.5f;
	n[1] = (float)(az - bz) * 0.5f;
	n[2] = (float)(ay - by) * 0.5f;
	vxb_normalize_fix_zero(n[0], n[1], n[2]);
}

VXB_FN void vxb_normal(const VxbTileView& g, int x, int y, int z, float n[3])
{
	n[0] = (float)(vxb_dist(g, x + 1, y, z) - vxb_dist(g, x - 1, y, z)) * 0.5f;
	n[1] = (float)(vxb_dist(g, x, y, z + 1) - vxb_dist(g, x, y, z - 1)) * 0.5f;
	n[2] = (float)(vxb_dist(g, x, y + 1, z) - vxb_dist(g, x, y - 1, z)) * 0.5f;
	vxb_normalize_fix_zero(n[0], n[1], n[2]);
}

// (b * 256) / (b - a), C integer division (:1591, :1674, :1942, :2025), for int8 samples with b != a.
// Device: one IEEE float division.  Exact: |b*256| <= 2^15 and |b-a| <= 255, so a non-integer quotient is at
// least 1/255 away from the next integer while the float result is within 2^-10 of it - truncation cannot flip.
VXB_FN int vxb_fixed_t(int a, int b)
{
#if defined(__CUDA_ARCH__)
	return __float2int_rz(__fdiv_rn((float)(b * 256), (float)(b - a)));
#else
	return (b * 256) / (b - a);
#endif
}

// FindBestVertexInLODChain :1484-1509 followed by the t recomputation :1671-1678 / :2022-2029.
template <class G>
VXB_FN_BIG int vxb_lod_descent(const G& g, int steps, int p0[3], int p1[3])
{
	for (int s = 0; s < steps; ++s)
	{
		const int mx = p0[0] + (p1[0] - p0[0]) / 2, my = p0[1] + (p1[1] - p0[1]) / 2, mz = p0[2] + (p1[2] - p0[2]) / 2;
		const int mid = vxb_dist(g, mx, my, mz);
		const int v0 = vxb_dist(g, p0[0], p0[1], p0[2]);
		if (v0 * mid <= 0) { p1[0] = mx; p1[1] = my; p1[2] = mz; }
		else { p0[0] = mx; p0[1] = my; p0[2] = mz; }
	}
	const int a = vxb_dist(g, p0[0], p0[1], p0[2]);
	const int b = vxb_dist(g, p1[0], p1[1], p1[2]);
	return (a != b) ? vxb_fixed_t(a, b) : 0;
}

// out-of-range float -> unsigned char the way x86 does it (cvttss2si, low byte) :1699, :2085
VXB_FN unsigned vxb_blend_u8(float f) { return (unsigned)((int)f) & 0xFFu; }

// Cell::CornerOnBlockBoundary :593-618 (0 on level 0 and for interior cells)
VXB_FN int vxb_corner_flags(int level, int lx, int ly, int lz, int corner)
{
	if (level == 0) return 0;
	int r = 0;
	if (lx == 0 && !(corner & 1)) r |= 1 << VXB_XNEG;
	if (lx == VXB_BLOCK - 1 && (corner & 1)) r |= 1 << VXB_XPOS;
	if (ly == 0 && !(corner & 2)) r |= 1 << VXB_YNEG;
	if (ly == VXB_BLOCK - 1 && (corner & 2)) r |= 1 << VXB_YPOS;
	if (lz == 0 && !(corner & 4)) r |= 1 << VXB_ZNEG;
	if (lz == VXB_BLOCK - 1 && (corner & 4)) r |= 1 << VXB_ZPOS;
	return r;
}

// Flags swap applied on output (:1350-1356): internal FaceId bits -> BlockPolygons::TransitionFaceId bits.
VXB_FN uint32_t vxb_swap3(uint32_t f) { return f ? ((f >> 3) | ((f & 7u) << 3)) : 0u; }

// AccumulateVertexTransitionDelta :1473-1482 in units of 1/4 cell: sum of inward unit vectors of the flagged faces.
VXB_FN void vxb_inward_sum(int flags, int d[3])
{
	d[0] = ((flags >> VXB_XNEG) & 1) - ((flags >> VXB_XPOS) & 1);
	d[1] = ((flags >> VXB_YNEG) & 1) - ((flags >> VXB_YPOS) & 1);
	d[2] = ((flags >> VXB_ZNEG) & 1) - ((flags >> VXB_ZPOS) & 1);
}

// ------------------------------------------------------------------------------------------------
// Regular cells (PolygonizeBlock :1529-1750)
// ------------------------------------------------------------------------------------------------

struct VxbVertexDesc
{
	int v0, v1;    // edge endpoints (corner ids), v0 < v1
	int t;         // 8.8 fixed-point interpolation parameter from the cell's own samples (:1591)
	int dir;       // reuse direction after the endpoint override (:1594-1608)
	int slot;      // reuse slot after the endpoint override
	bool endpoint; // (t & 0xFF) == 0
	bool atC7;     // endpoint at corner 7: never reused, owns slot 0 (:1597, :1653)
};

// zero mask of a cell: bit i = (sample i == 0).  A table vertex lies on an edge endpoint iff one of the edge's two
// samples is 0: t = 256*b/(b-a) with exactly one of a,b negative is 0 iff b == 0 and 256 iff a == 0 (|b| <= |b-a| < 256),
// so the endpoint logic of :1594-1608 needs no division.
VXB_FN unsigned vxb_zero_mask(const signed char v[8])
{
	unsigned z = 0;
#pragma unroll
	for (int i = 0; i < 8; ++i) z |= (v[i] == 0 ? 1u : 0u) << i;
	return z;
}

// descriptor without the interpolation parameter (d.t is only valid as 0 / 256 for endpoints, -1 otherwise)
VXB_FN VxbVertexDesc vxb_regular_vertex_desc_lite(unsigned vd, unsigned zeroMask)
{
	VxbVertexDesc d;
	d.v0 = (vd >> 4) & 0xF;
	d.v1 = vd & 0xF;
	d.dir = (vd >> 12) & 0xF;
	d.slot = (vd >> 8) & 0xF;
	const bool z0 = (zeroMask >> d.v0) & 1u, z1 = (zeroMask >> d.v1) & 1u;
	d.endpoint = z0 || z1;
	d.atC7 = false;
	d.t = -1;
	if (d.endpoint)
	{
		d.t = z1 ? 0 : 256;
		d.atC7 = (z1 && d.v1 == 7);
		if (!d.atC7) d.dir = (z1 ? d.v1 : d.v0) ^ 7;
		d.slot = 0;
	}
	return d;
}

VXB_FN VxbVertexDesc vxb_regular_vertex_desc(unsigned vd, const signed char v[8])
{
	VxbVertexDesc d = vxb_regular_vertex_desc_lite(vd, vxb_zero_mask(v));
	if (!d.endpoint) d.t = vxb_fixed_t(v[d.v0], v[d.v1]); // :1591
	return d;
}

// Which slot (if any) a table vertex claims in its own cell (:1653-1654, :1709-1712); -1 = none.
VXB_FN int vxb_regular_owned_slot(const VxbVertexDesc& d)
{
	if (d.endpoint) return d.atC7 ? 0 : -1;
	return (d.dir == 8) ? d.slot : -1;
}

// Pre-output vertex: x256 fixed-point position in grid axes + attributes.
struct VxbRawVertex
{
	float p[3];     // grid axes, x256
	float s[3];     // secondary position, grid axes, x256
	float n[3];     // normal, already in output axes
	int flags;      // internal face bits
	unsigned matId, blend;
};

// Vertex at a cell corner (GenerateVertexFromPoint :1450-1467).
template <class G>
VXB_FN_BIG void vxb_corner_vertex(const G& g, int level, const int base[3], const int local[3], int corner,
	unsigned cellMatId, unsigned cellMatBlend, VxbRawVertex& out)
{
	const int m = 1 << level;
	const int px = base[0] + ((corner & 1) ? m : 0), py = base[1] + ((corner & 2) ? m : 0), pz = base[2] + ((corner & 4) ? m : 0);
	const unsigned myId = vxb_mat(g, px, py, pz), myBlend = vxb_blend(g, px, py, pz); // both taps in flight while the normal is computed
	vxb_normal(g, px, py, pz, out.n);
	out.matId = cellMatId;
	out.blend = (myId != cellMatId) ? cellMatBlend : myBlend;
	out.p[0] = (float)px * 256.f; out.p[1] = (float)py * 256.f; out.p[2] = (float)pz * 256.f;
	out.flags = vxb_corner_flags(level, local[0], local[1], local[2], corner);
}

// Vertex in the interior of an edge (:1659-1704).
template <class G>
VXB_FN_BIG void vxb_edge_vertex(const G& g, int level, const int base[3], const int local[3], const VxbVertexDesc& d,
	unsigned cellMatId, unsigned cellMatBlend, VxbRawVertex& out)
{
	const int m = 1 << level;
	int p0[3] = { base[0] + ((d.v0 & 1) ? m : 0), base[1] + ((d.v0 & 2) ? m : 0), base[2] + ((d.v0 & 4) ? m : 0) };
	int p1[3] = { base[0] + ((d.v1 & 1) ? m : 0), base[1] + ((d.v1 & 2) ? m : 0), base[2] + ((d.v1 & 4) ? m : 0) };
	int t = d.t;
	if (level > 0) t = vxb_lod_descent(g, level, p0, p1);
	const int u = 256 - t;
	const float ft = (float)t, fu = (float)u;

	// the four material / blend taps are issued before the normals so that their latency overlaps the arithmetic
	const unsigned m0 = vxb_mat(g, p0[0], p0[1], p0[2]), m1 = vxb_mat(g, p1[0], p1[1], p1[2]);
	const unsigned b0 = vxb_blend(g, p0[0], p0[1], p0[2]), b1 = vxb_blend(g, p1[0], p1[1], p1[2]);
	float n0[3], n1[3];
	vxb_normal(g, p0[0], p0[1], p0[2], n0);
	vxb_normal(g, p1[0], p1[1], p1[2], n1);

	out.p[0] = ft * (float)p0[0] + fu * (float)p1[0];
	out.p[1] = ft * (float)p0[1] + fu * (float)p1[1];
	out.p[2] = ft * (float)p0[2] + fu * (float)p1[2];
	out.flags = vxb_corner_flags(level, local[0], local[1], local[2], d.v0) & vxb_corner_flags(level, local[0], local[1], local[2], d.v1);

	out.matId = cellMatId;
	if (m0 == m1 && m0 == cellMatId)
		out.blend = vxb_blend_u8((ft * (float)(int)b0 + fu * (float)(int)b1) / 256.f);
	else
		out.blend = cellMatBlend;

	const float w0 = ft / 256.f, w1 = fu / 256.f;
	out.n[0] = n0[0] * w0 + n1[0] * w1;
	out.n[1] = n0[1] * w0 + n1[1] * w1;
	out.n[2] = n0[2] * w0 + n1[2] * w1;
	vxb_normalize_fix_zero(out.n[0], out.n[1], out.n[2]);
}

// Secondary position of a regular-cell vertex (:1728-1738): primary + 0.25 cell per flagged face, inwards.
VXB_FN void vxb_regular_secondary(int level, VxbRawVertex& v)
{
	int d[3];
	vxb_inward_sum(v.flags, d);
	const float q = 64.f * (float)(1 << level); // 0.25 * m * 256
	v.s[0] = v.p[0] + (float)d[0] * q;
	v.s[1] = v.p[1] + (float)d[1] * q;
	v.s[2] = v.p[2] + (float)d[2] * q;
}

// PushBlocksToResult vertex conversion (:1330-1369, :1391-1423): /256, y<->z swap, flag swizzle, textures.
VXB_FN_BIG void vxb_finish_vertex(const VxbRawVertex& r, const VxbMaterialLut& lut, VxbVertex& o)
{
	const float k = 1.f / 256.f;
	o.pos[0] = r.p[0] * k; o.pos[1] = r.p[2] * k; o.pos[2] = r.p[1] * k;
	o.sec[0] = r.s[0] * k; o.sec[1] = r.s[2] * k; o.sec[2] = r.s[1] * k;
	const uint32_t f = vxb_swap3((uint32_t)r.flags);
#if defined(__CUDA_ARCH__)
	o.sec[3] = __uint_as_float(f);
#else
	union { uint32_t u; float f; } cv; cv.u = f; o.sec[3] = cv.f;
#endif
	o.nrm[0] = r.n[0]; o.nrm[1] = r.n[1]; o.nrm[2] = r.n[2];
	if (lut.valid[r.matId]) { o.tex[0] = lut.tex0[r.matId] | (r.blend << 8); o.tex[1] = lut.tex1[r.matId]; }
	else { o.tex[0] = 0xFFu | (r.matId << 8); o.tex[1] = 0; } // GetMaterial returned null (:1364-1368): marker {Reserved=0xFF, Blend=id};
	                                                          // the host clears it to all-zero textures and logs (vxb_result_download)
}

// Degenerate-triangle test on the x256 positions (:1300-1321): keep iff |cross|^2 >= FLT_EPSILON.
VXB_FN bool vxb_triangle_kept(const float a[3], const float b[3], const float c[3])
{
	const float ax = b[0] - a[0], ay = b[1] - a[1], az = b[2] - a[2];
	const float bx = c[0] - a[0], by = c[1] - a[1], bz = c[2] - a[2];
	const float cx = ay * bz - by * az;
	const float cy = az * bx - bz * ax;
	const float cz = ax * by - bx * ay;
	return ((cx * cx + cy * cy) + cz * cz) >= 1.1920928955078125e-07f;
}

// ------------------------------------------------------------------------------------------------
// Majority vote of the 8 children (CalculateMaterialForCellCache :753-838)
// ------------------------------------------------------------------------------------------------

struct VxbVote
{
	unsigned char ids[8];
	int counts[8];
	unsigned blends[8];
	unsigned n;
};

VXB_FN void vxb_vote_init(VxbVote& v) { v.n = 0; }

// children must be fed x-fastest, then y, then z (:773-775); EMPTY children are ignored (:821)
VXB_FN void vxb_vote_add(VxbVote& v, unsigned id, unsigned blend)
{
	for (unsigned i = 0; i < v.n; ++i)
		if (v.ids[i] == id) { ++v.counts[i]; v.blends[i] += blend; return; }
	if (id != VXB_EMPTY_MATERIAL) { v.ids[v.n] = (unsigned char)id; v.counts[v.n] = 1; v.blends[v.n] = blend; ++v.n; }
}

// first maximum wins (std::max_element :830); false when no child carried a material
VXB_FN bool vxb_vote_result(const VxbVote& v, unsigned& id, unsigned& blend)
{
	if (!v.n) return false;
	unsigned best = 0;
	for (unsigned i = 1; i < v.n; ++i) if (v.counts[i] > v.counts[best]) best = i;
	id = v.ids[best];
	blend = (v.blends[best] / (unsigned)v.counts[best]) & 0xFFu;
	return true;
}

// ------------------------------------------------------------------------------------------------
// Transition cells (GenerateTransitionCells :1754-2131).  face = 0..5: z=0, y=0, x=0, z=15, y=15, x=15.
// ------------------------------------------------------------------------------------------------

// axis normal to the face, and the in-plane (column, row) axes (:1764-1772)
VXB_FN void vxb_face_axes(int face, int& axis, int& ua, int& va)
{
	const int f = face % 3;
	axis = (f == 0) ? 2 : (f == 1 ? 1 : 0);
	ua = (f == 2) ? 1 : 0;
	va = (f == 0) ? 1 : 2;
}

// internal FaceId of the low-resolution cell's face (:1795-1803)
VXB_FN int vxb_face_internal(int face)
{
	return (face == 0) ? VXB_ZNEG : (face == 1) ? VXB_YNEG : (face == 2) ? VXB_XNEG : (face == 3) ? VXB_ZPOS : (face == 4) ? VXB_YPOS : VXB_XPOS;
}

// corner id of the low-res cell for transition samples 9..12 (Cell::GetCornerIdsForFace :570-581)
VXB_FN int vxb_face_low_corner(int face, int k)
{
	int axis, ua, va;
	vxb_face_axes(face, axis, ua, va);
	return ((face >= 3) ? (1 << axis) : 0) | ((k & 1) ? (1 << ua) : 0) | ((k & 2) ? (1 << va) : 0);
}

// position of transition sample i (0..12) of the cell with base cellBase (grid coords, unclamped)
VXB_FN void vxb_transition_sample_pos(int face, int level, const int cellBase[3], int i, int p[3])
{
	int axis, ua, va;
	vxb_face_axes(face, axis, ua, va);
	const int m = 1 << level, h = m >> 1;
	int c, r;
	if (i < 9) { c = (i % 3) * h; r = (i / 3) * h; }
	else { c = ((i - 9) & 1) * m; r = ((i - 9) >> 1) * m; }
	p[0] = cellBase[0]; p[1] = cellBase[1]; p[2] = cellBase[2];
	p[axis] += (face >= 3) ? m : 0;
	p[ua] += c;
	p[va] += r;
}

// the 13 samples of a transition cell (:1867-1911): 0..8 on the half-stride lattice of the face plane, 9..12 = 0,2,6,8
VXB_FN_BIG void vxb_transition_samples(const VxbGrid& g, int face, int level, const int cellBase[3], signed char v[13])
{
	for (int i = 0; i < 9; ++i)
	{
		int p[3];
		vxb_transition_sample_pos(face, level, cellBase, i, p);
		v[i] = (signed char)vxb_dist(g, p[0], p[1], p[2]);
	}
	v[9] = v[0]; v[10] = v[2]; v[11] = v[6]; v[12] = v[8];
}

VXB_FN unsigned vxb_transition_case_code(const signed char v[9])
{
	unsigned code = 0;
	code |= (v[0] < 0) ? 0x01u : 0; code |= (v[1] < 0) ? 0x02u : 0; code |= (v[2] < 0) ? 0x04u : 0;
	code |= (v[3] < 0) ? 0x80u : 0; code |= (v[4] < 0) ? 0x100u : 0; code |= (v[5] < 0) ? 0x08u : 0;
	code |= (v[6] < 0) ? 0x40u : 0; code |= (v[7] < 0) ? 0x20u : 0; code |= (v[8] < 0) ? 0x10u : 0;
	return code; // weights :1819
}

struct VxbTransVertexDesc
{
	int v0, v1;
	int t;
	int dir, slot; // after the corner override (:1951-1956)
	bool endpoint;
};

// a, b = the samples at the vertex's edge endpoints v0 = (vd >> 4) & 15, v1 = vd & 15
VXB_FN VxbTransVertexDesc vxb_transition_vertex_desc_ab(unsigned vd, int a, int b, const unsigned char* cornerData)
{
	VxbTransVertexDesc d;
	d.v0 = (vd >> 4) & 0xF;
	d.v1 = vd & 0xF;
	d.dir = (vd >> 12) & 0xF;
	d.slot = (vd >> 8) & 0xF;
	d.endpoint = (a == 0) || (b == 0); // t in {0, 256}, see vxb_zero_mask
	if (d.endpoint)
	{
		d.t = (b == 0) ? 0 : 256;
		const int corner = (b == 0) ? d.v1 : d.v0;
		d.dir = cornerData[corner] >> 4;
		d.slot = cornerData[corner] & 0xF;
	}
	else d.t = vxb_fixed_t(a, b); // :1942
	return d;
}

VXB_FN VxbTransVertexDesc vxb_transition_vertex_desc(unsigned vd, const signed char v[13], const unsigned char* cornerData)
{
	return vxb_transition_vertex_desc_ab(vd, v[(vd >> 4) & 0xF], v[vd & 0xF], cornerData);
}

// New transition vertex (:1980-2092).  local = low-res cell's local coords, base = its base.
VXB_FN_BIG void vxb_transition_vertex(const VxbGrid& g, int face, int level, const int base[3], const int local[3],
	const VxbTransVertexDesc& d, unsigned cellMatId, unsigned cellMatBlend, VxbRawVertex& out)
{
	const int m = 1 << level;
	int p0[3], p1[3];
	vxb_transition_sample_pos(face, level, base, d.v0, p0);
	vxb_transition_sample_pos(face, level, base, d.v1, p1);
	const bool low0 = d.v0 >= 9, low1 = d.v1 >= 9;

	int t = d.t, u = 0, adj = 0;
	float n0[3] = { 0.f, 0.f, 0.f }, n1[3] = { 0.f, 0.f, 0.f };
	if (d.endpoint)
	{
		if (t == 0)
		{
			u = 256;
			vxb_normal(g, p1[0], p1[1], p1[2], n1);
			if (low1) adj = vxb_corner_flags(level, local[0], local[1], local[2], vxb_face_low_corner(face, d.v1 - 9));
		}
		else
		{
			u = 0; t = 256;
			vxb_normal(g, p0[0], p0[1], p0[2], n0);
			if (low0) adj = vxb_corner_flags(level, local[0], local[1], local[2], vxb_face_low_corner(face, d.v0 - 9));
		}
	}
	else
	{
		const int lod = low0 ? level : level - 1;
		if (lod > 0) t = vxb_lod_descent(g, lod, p0, p1);
		u = 256 - t;
		vxb_normal(g, p0[0], p0[1], p0[2], n0);
		vxb_normal(g, p1[0], p1[1], p1[2], n1);
		if (low0 && low1)
			adj = vxb_corner_flags(level, local[0], local[1], local[2], vxb_face_low_corner(face, d.v0 - 9))
				& vxb_corner_flags(level, local[0], local[1], local[2], vxb_face_low_corner(face, d.v1 - 9));
	}
	const size_t i0 = vxb_index(g, p0[0], p0[1], p0[2]), i1 = vxb_index(g, p1[0], p1[1], p1[2]);
	const unsigned m0 = g.mat[i0], m1 = g.mat[i1];

	float P0[3] = { (float)p0[0], (float)p0[1], (float)p0[2] }, P1[3] = { (float)p1[0], (float)p1[1], (float)p1[2] };
	float S0[3] = { P0[0], P0[1], P0[2] }, S1[3] = { P1[0], P1[1], P1[2] };
	if (low0 || low1)
	{
		int dsum[3];
		vxb_inward_sum(adj, dsum);
		const float q = 0.25f * (float)m;
		const float delta[3] = { (float)dsum[0] * q, (float)dsum[1] * q, (float)dsum[2] * q };
		const int fi = vxb_face_internal(face);
		const bool simple = adj == (1 << fi);
		int mv[3];
		vxb_inward_sum(1 << fi, mv);
		const float move[3] = { (float)mv[0] * q, (float)mv[1] * q, (float)mv[2] * q };
		if (low0)
		{
			S0[0] += delta[0]; S0[1] += delta[1]; S0[2] += delta[2];
			if (simple) { P0[0] += move[0]; P0[1] += move[1]; P0[2] += move[2]; }
		}
		if (low1)
		{
			S1[0] += delta[0]; S1[1] += delta[1]; S1[2] += delta[2];
			if (simple) { P1[0] += move[0]; P1[1] += move[1]; P1[2] += move[2]; }
		}
	}
	const float ft = (float)t, fu = (float)u;
	out.p[0] = ft * P0[0] + fu * P1[0]; out.p[1] = ft * P0[1] + fu * P1[1]; out.p[2] = ft * P0[2] + fu * P1[2];
	out.s[0] = ft * S0[0] + fu * S1[0]; out.s[1] = ft * S0[1] + fu * S1[1]; out.s[2] = ft * S0[2] + fu * S1[2];
	out.flags = adj;

	const float w0 = ft / 256.f, w1 = fu / 256.f;
	out.n[0] = n0[0] * w0 + n1[0] * w1;
	out.n[1] = n0[1] * w0 + n1[1] * w1;
	out.n[2] = n0[2] * w0 + n1[2] * w1;
	vxb_normalize_fix_zero(out.n[0], out.n[1], out.n[2]);

	out.matId = cellMatId;
	if (m0 == m1 && m0 == cellMatId)
		out.blend = vxb_blend_u8((ft * (float)(int)g.blend[i0] + fu * (float)(int)g.blend[i1]) / 256.f);
	else
		out.blend = cellMatBlend;
}
