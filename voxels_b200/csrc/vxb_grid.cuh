// Device-resident grid store (SURVEY.md section 8 f1-f3): the steps either side of the polygonizer, on the dense HBM volumes.
//   vxb_fill_columns_kernel / vxb_fill_kernel     Grid::Create(w, d, h, sx, sy, sz, step, &surface)   src/VoxelGrid.cpp:79-132
//   vxb_inject_surface_kernel                     VoxelGrid::InjectSurface                              :388-488
//   vxb_inject_material_kernel                    VoxelGrid::InjectMaterial                             :490-584
//   vxb_pack_sizes_kernel / vxb_pack_write_kernel VoxelGrid::CompressBlock + PackForSave                :610-672, :269-315
// The surfaces are the built-in ones of vxb_surfaces.h (a client callback cannot run on the device); their floats are
// bit-identical to the CPU adapter's, so the bytes equal what the reference grid store produces for the same surface.
//   vxb_program_cull_kernel + vxb_program_fill_kernel   Grid::Create with an SDF program (vxb_program.h): block cull, per voxel
//   vxb_inject_program_kernel                     VoxelGrid::InjectSurface with an SDF program
#pragma once
#include "vxb_surfaces.h"
#include "vxb_program.h"

struct VxbFillArgs
{
	vxb_surface surface;
	unsigned char perm[512];
	float start[3], step;
	int n, z0, z1;          // planes [z0, z1) of the n^3 grid are written
	float* columns;          // terrain: per (x, y) column {height, h1, h2, unused}
};

// coordinate of sample i of an axis the way the reference's constructor and a client surface produce it: the block's start
// (start + blockIndex * 16 * step, VoxelGrid.cpp:100-105) plus k steps inside the block (VoxelSurface::GetSurface)
__device__ __forceinline__ float vxb_fill_coord(float start, float step, int i)
{
	return (start + (float)(i & ~15) * step) + (float)(i & 15) * step;
}

// terrain only: the three per-column heights (the same expressions as vxs_surface_value; evaluated once per column
// instead of once per voxel - identical floats either way)
__global__ void __launch_bounds__(256) vxb_fill_columns_kernel(const __grid_constant__ VxbFillArgs a)
{
	const int n = a.n;
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n * n) return;
	const int x = i % n, y = i / n;
	const float fx = vxb_fill_coord(a.start[0], a.step, x), fy = vxb_fill_coord(a.start[1], a.step, y);
	const float N = a.surface.p[0];
	const float gx = fx + a.surface.p[1], gy = fy + a.surface.p[2];
	const float height = 0.5f * N + (0.18f * N) * vxs_fbm2(a.perm, VXS_DIV(gx, N) * 4.f, VXS_DIV(gy, N) * 4.f);
	const float h1 = 0.45f * N + (0.03f * N) * vxs_noise2(a.perm, VXS_DIV(gx, 37.f), VXS_DIV(gy, 37.f));
	const float h2 = 0.60f * N + (0.03f * N) * vxs_noise2(a.perm, VXS_DIV(gx, 53.f) + 7.7f, VXS_DIV(gy, 53.f) + 3.3f);
	reinterpret_cast<float4*>(a.columns)[i] = make_float4(height, h1, h2, 0.f);
}

// one thread per 4 x-adjacent voxels: surface value -> round away from zero -> clamp +-4 (VoxelGrid.cpp:37-50, :126)
__global__ void __launch_bounds__(256) vxb_fill_kernel(const __grid_constant__ VxbFillArgs a, signed char* __restrict__ dist, unsigned char* __restrict__ mat, unsigned char* __restrict__ blend)
{
	const int n = a.n, q = n >> 2;
	const size_t total = (size_t)(a.z1 - a.z0) * n * q;
	for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x)
	{
		const int x4 = (int)(i % q) * 4, y = (int)((i / q) % n), z = a.z0 + (int)(i / ((size_t)q * n));
		const float fy = vxb_fill_coord(a.start[1], a.step, y), fz = vxb_fill_coord(a.start[2], a.step, z);
		unsigned pd = 0, pm = 0, pb = 0;
#pragma unroll
		for (int k = 0; k < 4; ++k)
		{
			const int x = x4 + k;
			const float fx = vxb_fill_coord(a.start[0], a.step, x);
			unsigned m, bl;
			float d;
			if (a.surface.kind == VXB_SURFACE_TERRAIN)
			{
				const float4 col = reinterpret_cast<const float4*>(a.columns)[(size_t)y * n + x];
				const float gx = fx + a.surface.p[1], gy = fy + a.surface.p[2];
				d = (fz - col.x) + 6.f * vxs_noise3(a.perm, VXS_DIV(gx, 24.f), VXS_DIV(gy, 24.f), VXS_DIV(fz, 24.f));
				m = fz < col.y ? 0u : (fz < col.z ? 1u : 2u);
				if (vxs_noise3(a.perm, VXS_DIV(gx, 48.f) + 11.1f, VXS_DIV(gy, 48.f) + 5.5f, VXS_DIV(fz, 48.f) + 2.2f) > 0.35f) m = 3u;
				float span = col.z - col.y;
				if (span < 1.f) span = 1.f;
				const float t = vxs_clampf(VXS_DIV(fz - col.y, span), 0.f, 1.f);
				bl = (unsigned)(int)(255.f * (t * t * (3.f - 2.f * t)));
				d = vxs_clampf(d, -100.f, 100.f);
			}
			else d = vxs_surface_value(a.surface, a.perm, fx, fy, fz, m, bl);
			int v = vxs_round_away(d);
			v = v > 4 ? 4 : (v < -4 ? -4 : v); // toGridDistValue
			pd |= ((unsigned)v & 0xFFu) << (8 * k);
			pm |= (m & 0xFFu) << (8 * k);
			pb |= (bl & 0xFFu) << (8 * k);
		}
		const size_t o = ((size_t)z * n + y) * n + x4;
		*reinterpret_cast<unsigned*>(dist + o) = pd;
		*reinterpret_cast<unsigned*>(mat + o) = pm;
		*reinterpret_cast<unsigned*>(blend + o) = pb;
	}
}

// ---- edits -------------------------------------------------------------------------------------
struct VxbEditArgs
{
	vxb_surface surface;
	unsigned char perm[512];
	float position[3], extents[3];
	int type;                // InjectionType: 0 add, 1 subtract-add-inner, 2 subtract (include/Grid.h)
	int material, addBlend;  // InjectMaterial
	int n;
	int b0[3], bn[3];        // first touched block and number of touched blocks per axis
};

// the section of block (base = its first voxel) an edit at position/extents touches, per axis: CalculateTouchedBlockSection
// (:365-386), then the float loop `for (v = start; v < end; ++v)` (:432-434) = count iterations from start
__device__ __forceinline__ void vxb_edit_section(float position, float extent, float base, float& start, int& count)
{
	const float lo = base, hi = base + 16.f;
	const float icp = position - extent / 2.f;
	const float s = fminf(fmaxf(icp, lo), hi) - lo;
	const float e = fminf(fmaxf(icp + extent, lo), hi) - lo;
	start = s;
	int c = 0;
	for (float v = s; v < e; v += 1.f) ++c;
	count = c;
}

// one CTA per touched block
__global__ void __launch_bounds__(256) vxb_inject_surface_kernel(const __grid_constant__ VxbEditArgs a, signed char* __restrict__ dist)
{
	const int bx = a.b0[0] + (int)(blockIdx.x % a.bn[0]), by = a.b0[1] + (int)((blockIdx.x / a.bn[0]) % a.bn[1]), bz = a.b0[2] + (int)(blockIdx.x / (a.bn[0] * a.bn[1]));
	const float base[3] = { (float)(bx * 16), (float)(by * 16), (float)(bz * 16) };
	float start[3]; int cnt[3];
	for (int k = 0; k < 3; ++k) vxb_edit_section(a.position[k], a.extents[k], base[k], start[k], cnt[k]);
	const int total = cnt[0] * cnt[1] * cnt[2];
	// the surface is sampled from surfaceCoordStart = blockBase + blockStart - position in steps of 1 (:419-428)
	const float s0[3] = { base[0] + start[0] - a.position[0], base[1] + start[1] - a.position[1], base[2] + start[2] - a.position[2] };
	for (int i = threadIdx.x; i < total; i += blockDim.x)
	{
		const int kx = i % cnt[0], ky = (i / cnt[0]) % cnt[1], kz = i / (cnt[0] * cnt[1]);
		const unsigned vx = (unsigned)(start[0] + (float)kx), vy = (unsigned)(start[1] + (float)ky), vz = (unsigned)(start[2] + (float)kz);
		unsigned m, bl;
		const float sv = vxs_surface_value(a.surface, a.perm, s0[0] + (float)kx, s0[1] + (float)ky, s0[2] + (float)kz, m, bl);
		const size_t o = ((size_t)(bz * 16 + vz) * a.n + (by * 16 + vy)) * a.n + (bx * 16 + vx);
		const float value = (float)dist[o];
		float f;
		if (a.type == 0) f = fminf(value, sv);            // IT_Add            :443
		else if (a.type == 1) f = fmaxf(value, sv);       // IT_SubtractAddInner :446
		else f = fmaxf(-sv, value);                       // IT_Subtract       :449
		dist[o] = (signed char)vxs_round_away(f);         // no +-4 clamp here (:441-452)
	}
}

__global__ void __launch_bounds__(256) vxb_inject_material_kernel(const __grid_constant__ VxbEditArgs a, unsigned char* __restrict__ mat, unsigned char* __restrict__ blend)
{
	const int bx = a.b0[0] + (int)(blockIdx.x % a.bn[0]), by = a.b0[1] + (int)((blockIdx.x / a.bn[0]) % a.bn[1]), bz = a.b0[2] + (int)(blockIdx.x / (a.bn[0] * a.bn[1]));
	const float base[3] = { (float)(bx * 16), (float)(by * 16), (float)(bz * 16) };
	float start[3]; int cnt[3];
	for (int k = 0; k < 3; ++k) vxb_edit_section(a.position[k], a.extents[k], base[k], start[k], cnt[k]);
	const int total = cnt[0] * cnt[1] * cnt[2];
	const float coeff = (a.extents[0] / 2.0f) * 0.75f; // extDivCoeff.x (:500-501)
	for (int i = threadIdx.x; i < total; i += blockDim.x)
	{
		const int kx = i % cnt[0], ky = (i / cnt[0]) % cnt[1], kz = i / (cnt[0] * cnt[1]);
		const float x = start[0] + (float)kx, y = start[1] + (float)ky, z = start[2] + (float)kz;
		const float dx = (x + base[0]) - a.position[0], dy = (y + base[1]) - a.position[1], dz = (z + base[2]) - a.position[2];
		const float d = VXS_DIV(VXS_SQRT((dx * dx + dy * dy) + dz * dz), coeff);       // glm::length / extDivCoeff.x (:535)
		const float w = fminf(1.f, fmaxf(0.f, 1.f - d)) * 255.f;
		const int outputBlend = (int)(unsigned char)(int)w;                            // (unsigned char)(float) (:537)
		const size_t o = ((size_t)(bz * 16 + (unsigned)z) * a.n + (by * 16 + (unsigned)y)) * a.n + (bx * 16 + (unsigned)x);
		const int cm = mat[o], cb = blend[o];
		if (cm == a.material)
		{
			const int v = (a.addBlend ? 1 : -1) * outputBlend + cb;                    // :543
			blend[o] = (unsigned char)(v < 0 ? 0 : (v > 255 ? 255 : v));
		}
		else { mat[o] = (unsigned char)a.material; blend[o] = (unsigned char)outputBlend; }
	}
}

// ---- SDF programs (vxb_program.h): Grid::Create / InjectSurface with a client-composed surface ----------------------
// The program travels by value as a __grid_constant__ kernel parameter (64 ops = 6 KB): no device buffer and no
// __constant__ symbol shared between the contexts of one process.
struct VxbProgram
{
	vxb_op ops[VXB_PROGRAM_MAX_OPS];
	unsigned char perm[VXB_PROGRAM_MAX_TERRAIN][512]; // one table per TERRAIN op, in program order
	int count;
};

struct VxbProgramFillArgs
{
	VxbProgram prog;
	float start[3], step;
	int n;
	unsigned b0, b1;         // pass A: block ids [b0, b1) (VoxelGrid order, id = x + y nb + z nb^2)
};

__device__ __forceinline__ void vxb_program_perm_to_smem(const VxbProgram& p, unsigned char* sPerm)
{
	for (int i = threadIdx.x; i < VXB_PROGRAM_MAX_TERRAIN * 512; i += blockDim.x) sPerm[i] = p.perm[i >> 9][i & 511];
	__syncthreads();
}

// Pass A: one thread per 16^3 block decides (vxp_block_cull, double interval arithmetic) whether every sample quantises to
// the same +-4 with one primitive's material; the CTA then writes its constant blocks row by row (thread i: row i / cnt of
// block i % cnt, so that neighbouring threads store neighbouring 16-byte segments of a grid row) and appends the others
// to `list` for pass B.
__global__ void __launch_bounds__(256) vxb_program_cull_kernel(const __grid_constant__ VxbProgramFillArgs a, signed char* __restrict__ dist,
	unsigned char* __restrict__ mat, unsigned char* __restrict__ blend, unsigned* __restrict__ list, unsigned* __restrict__ listCount)
{
	__shared__ unsigned sConst[256]; // bit 31: constant block; bits 0-7 distance byte, 8-15 material, 16-23 blend
	const unsigned nb = (unsigned)a.n >> 4;
	const unsigned first = a.b0 + blockIdx.x * 256u;
	const unsigned cnt = min(256u, a.b1 - first);
	const unsigned t = threadIdx.x;
	unsigned word = 0;
	bool listed = false;
	if (t < cnt)
	{
		const unsigned b = first + t;
		int d;
		unsigned m, bl;
		if (vxp_block_cull(a.prog.ops, a.prog.count, a.start, a.step, (int)(b % nb), (int)((b / nb) % nb), (int)(b / (nb * nb)), d, m, bl))
			word = 0x80000000u | ((unsigned)d & 0xFFu) | (m << 8) | (bl << 16);
		else listed = true;
	}
	sConst[t] = word;
	const unsigned lane = t & 31u, mask = __ballot_sync(0xFFFFFFFFu, listed);
	unsigned base = 0;
	if (lane == 0 && mask) base = atomicAdd(listCount, (unsigned)__popc(mask));
	base = __shfl_sync(0xFFFFFFFFu, base, 0);
	if (listed) list[base + __popc(mask & ((1u << lane) - 1u))] = first + t;
	__syncthreads();
	const size_t n = (size_t)a.n;
	for (unsigned i = t; i < 256u * cnt; i += 256u)
	{
		const unsigned j = i % cnt, r = i / cnt;
		const unsigned wv = sConst[j];
		if (!(wv >> 31)) continue;
		const unsigned b = first + j;
		const size_t bx = b % nb, by = (b / nb) % nb, bz = b / (nb * nb);
		const size_t o = ((bz * 16 + (r >> 4)) * n + by * 16 + (r & 15)) * n + bx * 16;
		const unsigned dd = (wv & 0xFFu) * 0x01010101u, mm = ((wv >> 8) & 0xFFu) * 0x01010101u, bb = ((wv >> 16) & 0xFFu) * 0x01010101u;
		*reinterpret_cast<uint4*>(dist + o) = make_uint4(dd, dd, dd, dd);
		*reinterpret_cast<uint4*>(mat + o) = make_uint4(mm, mm, mm, mm);
		*reinterpret_cast<uint4*>(blend + o) = make_uint4(bb, bb, bb, bb);
	}
}

// Pass B: one CTA per listed block (grid-stride over the list), thread = one 16-voxel row: every thread runs the same op
// sequence (uniform branches); the row's bytes are collected in 16-byte shift registers and stored once per channel.
__global__ void __launch_bounds__(256) vxb_program_fill_kernel(const __grid_constant__ VxbProgramFillArgs a, const unsigned* __restrict__ list,
	const unsigned* __restrict__ listCount, signed char* __restrict__ dist, unsigned char* __restrict__ mat, unsigned char* __restrict__ blend)
{
	__shared__ unsigned char sPerm[VXB_PROGRAM_MAX_TERRAIN * 512];
	vxb_program_perm_to_smem(a.prog, sPerm);
	const unsigned total = *listCount;
	const unsigned nb = (unsigned)a.n >> 4;
	const int y = (int)(threadIdx.x & 15), z = (int)(threadIdx.x >> 4);
	for (unsigned it = blockIdx.x; it < total; it += gridDim.x)
	{
		const unsigned b = list[it];
		const int bx = (int)(b % nb), by = (int)((b / nb) % nb), bz = (int)(b / (nb * nb));
		const float fy = vxb_fill_coord(a.start[1], a.step, by * 16 + y), fz = vxb_fill_coord(a.start[2], a.step, bz * 16 + z);
		uint4 rd = make_uint4(0, 0, 0, 0), rm = rd, rb = rd;
		for (int k = 0; k < 16; ++k)
		{
			const float fx = vxb_fill_coord(a.start[0], a.step, bx * 16 + k);
			unsigned m, bl;
			const float d = vxp_eval(a.prog.ops, a.prog.count, sPerm, fx, fy, fz, m, bl);
			int v = vxs_round_away(d);
			v = v > 4 ? 4 : (v < -4 ? -4 : v); // toGridDistValue
			// 16-byte shift registers: after 16 steps byte k holds voxel k
			rd = make_uint4((rd.x >> 8) | (rd.y << 24), (rd.y >> 8) | (rd.z << 24), (rd.z >> 8) | (rd.w << 24), (rd.w >> 8) | (((unsigned)v & 0xFFu) << 24));
			rm = make_uint4((rm.x >> 8) | (rm.y << 24), (rm.y >> 8) | (rm.z << 24), (rm.z >> 8) | (rm.w << 24), (rm.w >> 8) | ((m & 0xFFu) << 24));
			rb = make_uint4((rb.x >> 8) | (rb.y << 24), (rb.y >> 8) | (rb.z << 24), (rb.z >> 8) | (rb.w << 24), (rb.w >> 8) | ((bl & 0xFFu) << 24));
		}
		const size_t o = (((size_t)bz * 16 + z) * a.n + (size_t)by * 16 + y) * a.n + (size_t)bx * 16;
		*reinterpret_cast<uint4*>(dist + o) = rd;
		*reinterpret_cast<uint4*>(mat + o) = rm;
		*reinterpret_cast<uint4*>(blend + o) = rb;
	}
}

struct VxbProgramEditArgs
{
	VxbProgram prog;
	float position[3], extents[3];
	int type, n;
	int b0[3], bn[3];        // first touched block and number of touched blocks per axis (prepareEdit)
};

// vxb_inject_surface_kernel with a program: one CTA per touched block, no cull pass (edit boxes are small)
__global__ void __launch_bounds__(256) vxb_inject_program_kernel(const __grid_constant__ VxbProgramEditArgs a, signed char* __restrict__ dist)
{
	__shared__ unsigned char sPerm[VXB_PROGRAM_MAX_TERRAIN * 512];
	vxb_program_perm_to_smem(a.prog, sPerm);
	const int bx = a.b0[0] + (int)(blockIdx.x % a.bn[0]), by = a.b0[1] + (int)((blockIdx.x / a.bn[0]) % a.bn[1]), bz = a.b0[2] + (int)(blockIdx.x / (a.bn[0] * a.bn[1]));
	const float base[3] = { (float)(bx * 16), (float)(by * 16), (float)(bz * 16) };
	float start[3]; int cnt[3];
	for (int k = 0; k < 3; ++k) vxb_edit_section(a.position[k], a.extents[k], base[k], start[k], cnt[k]);
	const int total = cnt[0] * cnt[1] * cnt[2];
	const float s0[3] = { base[0] + start[0] - a.position[0], base[1] + start[1] - a.position[1], base[2] + start[2] - a.position[2] };
	for (int i = threadIdx.x; i < total; i += blockDim.x)
	{
		const int kx = i % cnt[0], ky = (i / cnt[0]) % cnt[1], kz = i / (cnt[0] * cnt[1]);
		const unsigned vx = (unsigned)(start[0] + (float)kx), vy = (unsigned)(start[1] + (float)ky), vz = (unsigned)(start[2] + (float)kz);
		unsigned m, bl;
		const float sv = vxp_eval(a.prog.ops, a.prog.count, sPerm, s0[0] + (float)kx, s0[1] + (float)ky, s0[2] + (float)kz, m, bl);
		const size_t o = ((size_t)(bz * 16 + vz) * a.n + (by * 16 + vy)) * a.n + (bx * 16 + vx);
		const float value = (float)dist[o];
		float f;
		if (a.type == 0) f = fminf(value, sv);            // IT_Add            :443
		else if (a.type == 1) f = fmaxf(value, sv);       // IT_SubtractAddInner :446
		else f = fmaxf(-sv, value);                       // IT_Subtract       :449
		dist[o] = (signed char)vxs_round_away(f);         // no +-4 clamp here (:441-452)
	}
}

// ---- run-length coding of the 16^3 blocks (VoxelGrid::CompressBlock :610-672) ----------------------------------
// One CTA per block, thread t owns the 16 bytes of row t (block order: x fastest, then y, then z).  A pair boundary is a
// value change, or every 255th byte of a run (the counter is a byte).  The channel is stored raw when more than 2048
// pairs would be needed (:650-655).  Returns (to every thread) the stored size; pairs (start index per pair) are left in
// `starts` when the channel is run-length coded.
__device__ __forceinline__ unsigned vxb_rle_channel(const unsigned char* __restrict__ vol, int n, int bx, int by, int bz,
	unsigned char rowBytes[16], unsigned short* starts /*[2049] smem*/, int* sLast /*[256] smem*/, unsigned* warpSums /*[8] smem*/, unsigned char* sPrev /*[256] smem*/, bool& raw)
{
	const int t = threadIdx.x, y = t & 15, z = t >> 4;
	const uint4 row = *reinterpret_cast<const uint4*>(vol + (((size_t)bz * 16 + z) * n + (size_t)by * 16 + y) * n + (size_t)bx * 16);
	*reinterpret_cast<uint4*>(rowBytes) = row;
	sPrev[t] = rowBytes[15];
	__syncthreads();
	{
		// most channels of most blocks hold one value: 4096 = 16 runs of 255 + one of 16, no scans needed
		const unsigned splat = (unsigned)sPrev[0] * 0x01010101u;
		const int uniform = __syncthreads_and(row.x == splat && row.y == splat && row.z == splat && row.w == splat);
		if (uniform)
		{
			if (t <= 17) starts[t] = (unsigned short)(t < 17 ? t * 255 : 4096);
			raw = false;
			__syncthreads();
			return 34u;
		}
	}
	const int prev = t ? sPrev[t - 1] : -1;
	// last value change at or before each of my bytes: first within the row, then the incoming one from earlier rows
	unsigned changeMask = 0;
	for (int k = 0; k < 16; ++k) if ((k ? rowBytes[k - 1] : prev) != rowBytes[k]) changeMask |= 1u << k;
	sLast[t] = changeMask ? t * 16 + (31 - __clz(changeMask)) : -1;
	__syncthreads();
	// inclusive max-scan over the rows (Hillis-Steele on 256 entries)
	for (int o = 1; o < 256; o <<= 1)
	{
		const int v = (t >= o) ? sLast[t - o] : -1;
		__syncthreads();
		if (v > sLast[t]) sLast[t] = v;
		__syncthreads();
	}
	int runStart = t ? sLast[t - 1] : 0; // start of the run my first byte continues (byte 0 of the block always starts one)
	unsigned boundary = 0;
	for (int k = 0; k < 16; ++k)
	{
		const int i = t * 16 + k;
		if ((changeMask >> k) & 1u) runStart = i;
		if (i == runStart || (i - runStart) % 255 == 0) boundary |= 1u << k;
	}
	unsigned total;
	const unsigned base = vxb_block_scan(__popc(boundary), warpSums, total);
	raw = total >= 2049u;
	if (!raw)
	{
		unsigned j = base;
		for (int k = 0; k < 16; ++k) if ((boundary >> k) & 1u) starts[j++] = (unsigned short)(t * 16 + k);
		if (t == 0) starts[total] = 4096;
	}
	__syncthreads();
	return raw ? 4096u : 2u * total;
}

// pass 1: stored sizes of the three channels + the flags word of every block (BF_Empty from the distance channel:
// no value change crosses or touches zero relative to the first value, :622-667)
__global__ void __launch_bounds__(VXB_THREADS) vxb_pack_sizes_kernel(const unsigned char* __restrict__ dist, const unsigned char* __restrict__ mat, const unsigned char* __restrict__ blend, int n,
	unsigned int* __restrict__ sizes /*[blocks][3]*/, unsigned int* __restrict__ flags /*[blocks]*/)
{
	__shared__ unsigned short starts[2049];
	__shared__ int sLast[256];
	__shared__ unsigned warpSums[8];
	__shared__ unsigned char sPrev[256];
	__shared__ int sInitial;
	const int nb = n >> 4;
	const size_t b = blockIdx.x;
	const int bx = (int)(b % nb), by = (int)((b / nb) % nb), bz = (int)(b / ((size_t)nb * nb));
	const unsigned char* chans[3] = { dist, mat, blend };
	unsigned f = 0;
	for (int ch = 0; ch < 3; ++ch)
	{
		unsigned char rowBytes[16];
		bool raw;
		const unsigned size = vxb_rle_channel(chans[ch], n, bx, by, bz, rowBytes, starts, sLast, warpSums, sPrev, raw);
		if (raw) f |= 2u << ch; // BF_DistanceUncompressed / Material / Blend (VoxelGrid.h:70-79)
		if (ch == 0)
		{
			// isEmpty (:622-667): no run value v (the 255-byte splits re-check the value of a long run, so every byte counts,
			// the first included) with initial * v <= 0, i.e. no zero and one strict sign; a raw block is never flagged
			if (threadIdx.x == 0) sInitial = (signed char)rowBytes[0];
			__syncthreads();
			const int initial = sInitial;
			int bad = 0;
			for (int k = 0; k < 16; ++k) if (initial * (int)(signed char)rowBytes[k] <= 0) bad = 1;
			const int anyBad = __syncthreads_or(bad);
			if (!raw && !anyBad) f |= 1u; // BF_Empty
		}
		if (threadIdx.x == 0) sizes[b * 3 + ch] = size;
		__syncthreads();
	}
	if (threadIdx.x == 0) flags[b] = f;
}

// exclusive prefix sum of the per-block byte counts (4 + three sizes): one CTA, every thread a contiguous chunk
__global__ void __launch_bounds__(1024) vxb_pack_offsets_kernel(const unsigned int* __restrict__ sizes, unsigned long long* __restrict__ offsets /*[blocks + 1]*/, size_t blocks, unsigned long long head)
{
	__shared__ unsigned long long sums[32];
	const size_t per = (blocks + 1023) / 1024;
	const size_t i0 = min((size_t)threadIdx.x * per, blocks), i1 = min(i0 + per, blocks);
	unsigned long long mine = 0;
	for (size_t i = i0; i < i1; ++i) mine += 4ull + sizes[i * 3] + sizes[i * 3 + 1] + sizes[i * 3 + 2];
	unsigned long long inc = mine;
	const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	for (int o = 1; o < 32; o <<= 1) { const unsigned long long v = __shfl_up_sync(0xFFFFFFFFu, inc, o); if (lane >= (unsigned)o) inc += v; }
	if (lane == 31) sums[warp] = inc;
	__syncthreads();
	if (threadIdx.x == 0) { unsigned long long acc = 0; for (int w = 0; w < 32; ++w) { const unsigned long long v = sums[w]; sums[w] = acc; acc += v; } }
	__syncthreads();
	unsigned long long run = head + sums[warp] + inc - mine;
	for (size_t i = i0; i < i1; ++i) { offsets[i] = run; run += 4ull + sizes[i * 3] + sizes[i * 3 + 1] + sizes[i * 3 + 2]; }
	if (threadIdx.x == 1023) offsets[blocks] = run;
}

// pass 2: the block data at its offset: {flags, distance, material, blend} (PackForSave :304-312)
__global__ void __launch_bounds__(VXB_THREADS) vxb_pack_write_kernel(const unsigned char* __restrict__ dist, const unsigned char* __restrict__ mat, const unsigned char* __restrict__ blend, int n,
	const unsigned int* __restrict__ flags, const unsigned long long* __restrict__ offsets, unsigned char* __restrict__ out)
{
	__shared__ unsigned short starts[2049];
	__shared__ int sLast[256];
	__shared__ unsigned warpSums[8];
	__shared__ unsigned char sPrev[256];
	__shared__ unsigned char sBytes[4096];
	const int nb = n >> 4;
	const size_t b = blockIdx.x;
	const int bx = (int)(b % nb), by = (int)((b / nb) % nb), bz = (int)(b / ((size_t)nb * nb));
	const unsigned char* chans[3] = { dist, mat, blend };
	unsigned char* dst = out + offsets[b];
	if (threadIdx.x < 4) dst[threadIdx.x] = (unsigned char)(flags[b] >> (8 * threadIdx.x));
	dst += 4;
	for (int ch = 0; ch < 3; ++ch)
	{
		unsigned char rowBytes[16];
		bool raw;
		const unsigned size = vxb_rle_channel(chans[ch], n, bx, by, bz, rowBytes, starts, sLast, warpSums, sPrev, raw);
		if (raw) { for (int k = 0; k < 16; ++k) dst[threadIdx.x * 16 + k] = rowBytes[k]; }
		else
		{
			for (int k = 0; k < 16; ++k) sBytes[threadIdx.x * 16 + k] = rowBytes[k];
			__syncthreads();
			for (unsigned j = threadIdx.x; j < size / 2; j += VXB_THREADS)
			{
				const unsigned s0 = starts[j];
				dst[2 * j] = (unsigned char)(starts[j + 1] - s0);
				dst[2 * j + 1] = sBytes[s0];
			}
		}
		dst += size;
		__syncthreads();
	}
}
