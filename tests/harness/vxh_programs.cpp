// Test harness for SDF programs (include/vxb200.h vxb_op): the client-composed surfaces of the device grid store served to the
// reference's PUBLIC C++ API (include/Voxels.h) through its VoxelSurface callback.
//
// Linked together with vxh_capi.cpp and the UNMODIFIED reference into oracle/_ref/libvxh_programs_ref.so (oracle/programs.mk),
// so one library holds the reference's grids and the whole vxh_* ABI of tests/harness.py plus the calls below:
//   vxh_grid_create_program / vxh_grid_inject_program   Grid::Create / Grid::InjectSurface with a ProgramSurface
//   vxh_program_dense                                   the same voxels on every host thread (full-size inputs)
//   vxh_program_cull_flags                              the fill's per-block cull decision, computed on the host
//   vxh_program_validate                                the library's program validation
// voxels_b200/csrc/vxb_program.h is compiled here as plain host C++: the floats are the device kernels' floats.
//
// Nothing here is shipped; it is test infrastructure.
#include <cstddef>
#include <cstdlib>
#include <Voxels.h>

#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>

#include "../../voxels_b200/csrc/vxb_program.h"

using namespace Voxels;

namespace
{
// an SDF program as a client VoxelSurface: values x-fastest, then y, then z (VoxelGrid.cpp:116-126), sample k of an axis at
// start + k * step (the grid hands out whole blocks / whole sections: VoxelGrid.cpp:100-113, :419-428)
struct ProgramSurface : public VoxelSurface
{
	std::vector<vxb_op> Ops;
	unsigned char Perm[VXB_PROGRAM_MAX_TERRAIN][512];
	ProgramSurface(const vxb_op* ops, unsigned count) : Ops(ops, ops + count)
	{
		memset(Perm, 0, sizeof(Perm));
		int t = 0;
		for (unsigned i = 0; i < count && t < VXB_PROGRAM_MAX_TERRAIN; ++i)
			if (ops[i].code == VXB_OP_TERRAIN) vxs_permutation(ops[i].seed, Perm[t++]);
	}
	float Eval(float x, float y, float z, unsigned& m, unsigned& b) const
	{
		return vxp_eval(Ops.data(), int(Ops.size()), &Perm[0][0], x, y, z, m, b);
	}

	virtual void GetSurface(float xStart, float xEnd, float xStep,
		float yStart, float yEnd, float yStep,
		float zStart, float zEnd, float zStep,
		float* output, unsigned char* materialid, unsigned char* blend) override
	{
		size_t id = 0;
		int nx = 0, ny = 0, nz = 0;
		for (float x = xStart; x < xEnd; x += xStep) ++nx;
		for (float y = yStart; y < yEnd; y += yStep) ++ny;
		for (float z = zStart; z < zEnd; z += zStep) ++nz;
		for (int kz = 0; kz < nz; ++kz)
		for (int ky = 0; ky < ny; ++ky)
		for (int kx = 0; kx < nx; ++kx)
		{
			unsigned m, b;
			output[id] = Eval(xStart + float(kx) * xStep, yStart + float(ky) * yStep, zStart + float(kz) * zStep, m, b);
			if (materialid) materialid[id] = (unsigned char)m;
			if (blend) blend[id] = (unsigned char)b;
			++id;
		}
	}
};
}

extern "C"
{

// -1 when the program is well formed, else the index of the offending op (the library's vxp_validate)
int vxh_program_validate(const vxb_op* ops, unsigned count)
{
	const char* why;
	return vxp_validate(ops, count, &why);
}

// Grid::Create(n, n, n, sx, sy, sz, step, &program)
void* vxh_grid_create_program(unsigned n, const vxb_op* ops, unsigned count, float sx, float sy, float sz, float step)
{
	ProgramSurface s(ops, count);
	return Grid::Create(n, n, n, sx, sy, sz, step, &s);
}

// Grid::InjectSurface(pos, ext, &program, type); out6 = the returned box
void vxh_grid_inject_program(void* gridPtr, const float* pos, const float* ext, const vxb_op* ops, unsigned count, int type, float* out6)
{
	Grid* grid = static_cast<Grid*>(gridPtr);
	ProgramSurface s(ops, count);
	const float3pair box = grid->InjectSurface(float3(pos[0], pos[1], pos[2]), float3(ext[0], ext[1], ext[2]), &s, InjectionType(type));
	out6[0] = box.first.x; out6[1] = box.first.y; out6[2] = box.first.z;
	out6[3] = box.second.x; out6[4] = box.second.y; out6[5] = box.second.z;
}

// The fill's voxels as dense arrays, on every host thread (full-size inputs; the reference's constructor is serial): the fill's
// sample coordinates (start + block start + k steps), the program, round away from zero, clamp to +-4.
void vxh_program_dense(unsigned n, const vxb_op* ops, unsigned count, const float* start, float step,
	signed char* dist, unsigned char* mat, unsigned char* blend)
{
	const ProgramSurface s(ops, count);
	#pragma omp parallel for schedule(static)
	for (long zy = 0; zy < long(n) * n; ++zy)
	{
		const int z = int(zy / n), y = int(zy % n);
		const float fy = vxp_fill_coord(start[1], step, y), fz = vxp_fill_coord(start[2], step, z);
		for (unsigned x = 0; x < n; ++x)
		{
			unsigned m, b;
			const float d = s.Eval(vxp_fill_coord(start[0], step, int(x)), fy, fz, m, b);
			int v = vxs_round_away(d);
			v = v > 4 ? 4 : (v < -4 ? -4 : v);
			const size_t g = (size_t(z) * n + y) * n + x;
			dist[g] = (signed char)v; mat[g] = (unsigned char)m; blend[g] = (unsigned char)b;
		}
	}
}

// The fill's per-block cull decision (vxp_block_cull) on the host: per block (VoxelGrid order) 0 = evaluated per voxel,
// 1 = written as a constant block; value4 (may be NULL) = {distance, material, blend, 0} of the constant blocks.
// Returns the number of constant blocks.
unsigned vxh_program_cull_flags(unsigned n, const vxb_op* ops, unsigned count, const float* start, float step,
	unsigned char* flags, int* value4)
{
	const int nb = int(n / 16);
	unsigned culled = 0;
	#pragma omp parallel for schedule(dynamic, 64) reduction(+ : culled)
	for (long b = 0; b < long(nb) * nb * nb; ++b)
	{
		int d = 0;
		unsigned m = 0, bl = 0;
		const int c = vxp_block_cull(ops, int(count), start, step, int(b % nb), int((b / nb) % nb), int(b / (long(nb) * nb)), d, m, bl);
		flags[b] = (unsigned char)c;
		if (value4) { value4[b * 4] = c ? d : 0; value4[b * 4 + 1] = c ? int(m) : 0; value4[b * 4 + 2] = c ? int(bl) : 0; value4[b * 4 + 3] = 0; }
		culled += unsigned(c);
	}
	return culled;
}

} // extern "C"
