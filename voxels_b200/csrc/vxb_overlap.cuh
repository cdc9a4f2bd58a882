// Box overlap gathers against the level-0 triangles of the resident mesh (include/vxb200.h "vxb_mesh_overlap_box").
//
// The walk is exact: it needs no epsilon, unlike the ray walks (vxb_ray.cuh).  A triangle the test accepts passes the box
// axes, test 1, which has no arithmetic: along every axis i, min(p0_i, p1_i, p2_i) <= max_i and max(p0_i, p1_i, p2_i) >= min_i.
//   lattice box    Level-0 vertices lie on the cell edges of their own block, so each of them lies in the closed lattice box
//                  [16 b_i, 16 b_i + 16] of its block.  With test 1, 16 b_i <= min(p_i) <= max_i and 16 b_i + 16 >= max(p_i)
//                  >= min_i: the block's closed lattice box meets the closed query box.  The candidate blocks are the
//                  b_i with ceil(min_i / 16) - 1 <= b_i <= floor(max_i / 16), clipped to the grid.  The division by 16 is
//                  exact, except where it underflows into the subnormals; there it rounds toward zero, which can only widen
//                  the range by one block.
//   measured box   The mesh bounds hold, per block, the exact min and max of its vertices' pos (among other points).  With
//                  test 1 again, box.min_i <= min(p_i) <= max_i and box.max_i >= max(p_i) >= min_i: the measured box meets the
//                  query box too.  A candidate whose measured box misses it holds no accepted triangle and is skipped.  An
//                  absent or erased block has min = +inf, max = -inf and is skipped by the same comparisons.
// So every block holding an accepted triangle is visited, and nothing is rounded on the way.
//
// Order.  The candidates are visited in coord_id order (output y = grid z outermost, then output z, then x) and the triangles
// of a block in index order, 32 at a time, one per lane; a triangle's place among its box's results is the number of accepted
// triangles before it in that order.  The count kernel sums the ballots; the write kernel walks the same candidates and writes
// at base + popc(ballot & lanemask_lt).  Neither depends on the launch.
#pragma once

#define VXB_OVERLAP_THREADS 256

struct VxbOverlapMesh
{
	VxbRayMesh m;           // directory, level-0 map, arenas
	const float4* boxes;    // the mesh bounds: {min, max} per (level, coord) slot, OUTPUT coordinates
	unsigned base0;         // vxb_mesh_bounds.level_base[0]
};

// the box rule (include/vxb200.h), which the host variant checks and the kernels answer with 0 triangles: finite components
// and min_i <= max_i (NaN fails)
VXB_HD bool vxb_box_valid(const vxb_box& b)
{
	bool ok = true;
	for (int i = 0; i < 3; ++i) ok = ok && isfinite(b.min[i]) && isfinite(b.max[i]) && b.min[i] <= b.max[i];
	return ok;
}

// Does the axis a separate the triangle v0, v1, v2 (box frame) from the box of half extents h?  All three vertices are
// projected; positive comparisons, so a NaN projection never separates.
VXB_FN bool vxb_overlap_separates(float ax, float ay, float az, const float3& v0, const float3& v1, const float3& v2,
	float hx, float hy, float hz)
{
	const float s0 = (ax * v0.x + ay * v0.y) + az * v0.z;
	const float s1 = (ax * v1.x + ay * v1.y) + az * v1.z;
	const float s2 = (ax * v2.x + ay * v2.y) + az * v2.z;
	const float r = (hx * fabsf(ax) + hy * fabsf(ay)) + hz * fabsf(az);
	return (s0 > r && s1 > r && s2 > r) || (s0 < -r && s1 < -r && s2 < -r);
}

// The separating-axis test of include/vxb200.h, in its order (-fmad=false: no contraction).  The products with a literal
// zero axis component are kept, so every s and r has the bits of the stated formula.
VXB_FN bool vxb_overlap_triangle_box(const vxb_box& b, const float3& p0, const float3& p1, const float3& p2)
{
	// 1: the box axes, exact
	if (!(fminf(p0.x, fminf(p1.x, p2.x)) <= b.max[0] && fmaxf(p0.x, fmaxf(p1.x, p2.x)) >= b.min[0])) return false;
	if (!(fminf(p0.y, fminf(p1.y, p2.y)) <= b.max[1] && fmaxf(p0.y, fmaxf(p1.y, p2.y)) >= b.min[1])) return false;
	if (!(fminf(p0.z, fminf(p1.z, p2.z)) <= b.max[2] && fmaxf(p0.z, fmaxf(p1.z, p2.z)) >= b.min[2])) return false;
	// 2: the box frame
	const float cx = (b.min[0] + b.max[0]) * 0.5f, cy = (b.min[1] + b.max[1]) * 0.5f, cz = (b.min[2] + b.max[2]) * 0.5f;
	const float hx = b.max[0] * 0.5f - b.min[0] * 0.5f, hy = b.max[1] * 0.5f - b.min[1] * 0.5f, hz = b.max[2] * 0.5f - b.min[2] * 0.5f;
	const float3 v0 = make_float3(p0.x - cx, p0.y - cy, p0.z - cz);
	const float3 v1 = make_float3(p1.x - cx, p1.y - cy, p1.z - cz);
	const float3 v2 = make_float3(p2.x - cx, p2.y - cy, p2.z - cz);
	const float3 e[3] = { make_float3(v1.x - v0.x, v1.y - v0.y, v1.z - v0.z), make_float3(v2.x - v1.x, v2.y - v1.y, v2.z - v1.z),
		make_float3(v0.x - v2.x, v0.y - v2.y, v0.z - v2.z) };
	// 3: the normal e0 x e1, then u_i x e_j (i = x, y, z outer; j = 0, 1, 2 inner)
	const float nx = e[0].y * e[1].z - e[0].z * e[1].y, ny = e[0].z * e[1].x - e[0].x * e[1].z, nz = e[0].x * e[1].y - e[0].y * e[1].x;
	if (vxb_overlap_separates(nx, ny, nz, v0, v1, v2, hx, hy, hz)) return false;
#pragma unroll
	for (int j = 0; j < 3; ++j)
		if (vxb_overlap_separates(0.f, -e[j].z, e[j].y, v0, v1, v2, hx, hy, hz)) return false;
#pragma unroll
	for (int j = 0; j < 3; ++j)
		if (vxb_overlap_separates(e[j].z, 0.f, -e[j].x, v0, v1, v2, hx, hy, hz)) return false;
#pragma unroll
	for (int j = 0; j < 3; ++j)
		if (vxb_overlap_separates(-e[j].y, e[j].x, 0.f, v0, v1, v2, hx, hy, hz)) return false;
	return true;
}

// The candidate blocks of the proof at the top, for one box per warp (every lane calls it with the same box): 32 candidates
// at a time, one per lane, are tested against their measured boxes; `block(s)` is called by the whole warp for each slot that
// passes, in coord_id order.
template <class Block>
VXB_FN void vxb_overlap_walk(const VxbOverlapMesh& om, const vxb_box& b, Block&& block)
{
	if (!vxb_box_valid(b)) return;
	const unsigned lane = threadIdx.x & 31;
	const int nb = om.m.nb;
	int lo[3], hi[3];
	for (int i = 0; i < 3; ++i)
	{
		const float l = fmaxf(ceilf(b.min[i] * 0.0625f) - 1.f, 0.f), h = fminf(floorf(b.max[i] * 0.0625f), (float)(nb - 1));
		if (!(l <= h)) return;
		lo[i] = (int)l; hi[i] = (int)h;
	}
	const unsigned ex = (unsigned)(hi[0] - lo[0] + 1), ez = (unsigned)(hi[2] - lo[2] + 1);
	const unsigned total = ex * ez * (unsigned)(hi[1] - lo[1] + 1);
	for (unsigned j0 = 0; j0 < total; j0 += 32)
	{
		const unsigned j = j0 + lane;
		unsigned slot = VXB_RAY_MISS;
		if (j < total)
		{
			const unsigned q = j / ex;
			const unsigned bx = lo[0] + j % ex, bz = lo[2] + q % ez, by = lo[1] + q / ez;
			const unsigned cid = (by * nb + bz) * nb + bx;   // output y = grid z
			const float4 mn = __ldg(&om.boxes[2 * (om.base0 + cid)]), mx = __ldg(&om.boxes[2 * (om.base0 + cid) + 1]);
			if (mn.x <= b.max[0] && mx.x >= b.min[0] && mn.y <= b.max[1] && mx.y >= b.min[1] && mn.z <= b.max[2] && mx.z >= b.min[2])
				slot = __ldg(&om.m.map[cid]);
		}
		vxb_warp_each(slot != VXB_RAY_MISS, slot, block);
	}
}

// One warp per box, persistent over the batch.  Write = false: the count kernel, counts[q] = the box's triangles and
// counts[count] = 0 (the exclusive scan of counts is the offsets).  Write = true: the write kernel, which reads those
// offsets and writes the triangles when offsets[count] <= capacity (decided here, with no host read).
template <bool Write>
__global__ void __launch_bounds__(VXB_OVERLAP_THREADS) vxb_overlap_kernel(const VxbOverlapMesh om, const vxb_box* __restrict__ boxes,
	unsigned count, uint64_t* __restrict__ counts, vxb_overlap_triangle* __restrict__ tris, uint64_t capacity)
{
	if constexpr (Write)
	{
		if (counts[count] > capacity) return;
	}
	else
	{
		if (blockIdx.x == 0 && threadIdx.x == 0) counts[count] = 0;
	}
	const unsigned lane = threadIdx.x & 31;
	const unsigned warps = gridDim.x * (VXB_OVERLAP_THREADS / 32);
	for (unsigned q = blockIdx.x * (VXB_OVERLAP_THREADS / 32) + (threadIdx.x >> 5); q < count; q += warps)
	{
		const vxb_box b = boxes[q];
		uint64_t at = Write ? counts[q] : 0;   // the write kernel: the next record; the count kernel: triangles so far
		vxb_overlap_walk(om, b, [&](const unsigned s) {
			const vxb_block_record* rec = om.m.dir + s;
			const unsigned n = __ldg(&rec->index_count) / 3, vo = __ldg(&rec->vertex_offset), io = __ldg(&rec->index_offset);
			const unsigned id = Write ? __ldg(&rec->id) : 0;
			for (unsigned k0 = 0; k0 < n; k0 += 32)
			{
				const unsigned k = k0 + lane;
				float3 p0, p1, p2;
				bool hit = false;
				if (k < n)
				{
					vxb_ray_triangle(om.m, vo, io, k, p0, p1, p2);
					hit = vxb_overlap_triangle_box(b, p0, p1, p2);
				}
				const unsigned ballot = __ballot_sync(0xFFFFFFFFu, hit);
				if constexpr (Write)
				{
					if (hit)
					{
						vxb_overlap_triangle t;
						t.p[0][0] = p0.x; t.p[0][1] = p0.y; t.p[0][2] = p0.z;
						t.p[1][0] = p1.x; t.p[1][1] = p1.y; t.p[1][2] = p1.z;
						t.p[2][0] = p2.x; t.p[2][1] = p2.y; t.p[2][2] = p2.z;
						t.slot = s; t.block_id = id; t.triangle = k;
						tris[at + __popc(ballot & ((1u << lane) - 1u))] = t;
					}
				}
				at += __popc(ballot);
			}
		});
		if constexpr (!Write)
		{
			if (lane == 0) counts[q] = at;
		}
	}
}
