// remove.cuh -- taking particles out of a set-up simulator at a sub-step boundary (cb200_sim_remove_particles / _rows,
// include/claymore_b200.h, DESIGN.md section 2.10).
//   * select and compact: sdf.cuh's count / write pair over one model's gathered rows (checkpoint layout), with an item kind per way
//     of choosing the rows; an item is kept (survives) unless it is selected, and a kept row is copied whole, in row order;
//   * the velocity-kept rule of the commit: grid[0]'s mass is rasterised from the survivors, and every node then takes the velocity
//     p / m it had before the call.
#pragma once
#include "checkpoint.cuh"
#include "collider.cuh"
#include "sdf.cuh"

namespace cb200 {

// the survivors' rows, C channels each, from the gathered rows `in`
struct RemoveRows {
	const float* in;
	float* out;
	int C;
	using Row = long long;  // the source row
	__device__ __forceinline__ void emit(long long r, const Row& i) const {
		for(int c = 0; c < C; ++c) out[r * C + c] = __ldg(in + i * C + c);
	}
};

// by region: a row is removed when its position, mapped into object k's material space with k's frame at time t as the boundary chain
// maps a node (collider_material_point), lies in any of the n objects of b.objects (object_query); with `outside`, when it lies in none
struct RemoveRegions : RemoveRows {
	Boundaries b;  // objects only
	float t;
	int outside;
	__device__ __forceinline__ void prepare() const { boundary_frames_cta<false, true>(b, t); }
	// LEVELSETS: level-set objects answered from the views levelset_views_cta copied
	template<bool LEVELSETS = false>
	__device__ __forceinline__ bool select(long long i, Row& row) const {
		const BoundaryFrames& s = boundary_frames();
		const float p[3] = {__ldg(in + i * C), __ldg(in + i * C + 1), __ldg(in + i * C + 2)};
		bool hit = false;
		for(int k = 0; k < b.objects.n; ++k) {
			float xm[3], x[3], n[3];
			collider_material_point(s.o[k], s.f[k], p, xm, x);
			if constexpr(LEVELSETS) hit |= object_query_levelsets(s.o[k], x, n);
			else hit |= object_query(s.o[k], x, n);
		}
		row = i;
		return hit == (outside != 0);
	}
	__device__ __forceinline__ bool eval(long long i, Row& row) const { return select(i, row); }
};
// the same with level-set objects among the regions, their lattices in ls (DESIGN.md section 2.11)
struct RemoveRegionsLevelsets : RemoveRegions {
	LevelSets ls;
	__device__ __forceinline__ void prepare() const {
		levelset_views_cta(ls);  // published by the frame builder's barrier
		RemoveRegions::prepare();
	}
	__device__ __forceinline__ bool eval(long long i, Row& row) const { return select<true>(i, row); }
};
static_assert(sizeof(RemoveRegionsLevelsets) + sizeof(SdfScan) <= 4096, "the level-set sink selection's parameters must fit the 4 KiB kernel-parameter limit");

// by mask: a row is removed when its byte is non-zero
struct RemoveMask : RemoveRows {
	const unsigned char* mask;
	__device__ __forceinline__ bool eval(long long i, Row& row) const {
		row = i;
		return __ldg(mask + i) == 0;
	}
};

// The velocity-kept rule, in scatter_grid_kernel's form: a warp per saved block (its key, its 1 KiB), a table query, absent keys
// skipped.  A node of the rebuilt grid[0] holds the survivors' mass m'; it takes the momentum m' (p / m) from the saved node (m, p),
// 0 where m = 0.  Each lane takes two nodes of every channel (float2, cell_pair_vel_sq's split).
__global__ void __launch_bounds__(256) keep_velocity_kernel(Cfg cfg, int count, const int* keys, const float* blocks, const int* table, int nbc, float* grid) {
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	for(int h = blockIdx.x * 8 + warp; h < count; h += gridDim.x * 8) {
		const int bno = table_query(cfg, table, keys[3 * h], keys[3 * h + 1], keys[3 * h + 2]);
		if(bno < 0 || bno >= nbc) continue;
		const float2* s = reinterpret_cast<const float2*>(blocks + (size_t) h * kGridBlockFloats);
		float2* d = reinterpret_cast<float2*>(grid + (size_t) bno * kGridBlockFloats);
		const float2 m = s[lane], mn = d[lane];
#pragma unroll
		for(int c = 1; c < 4; ++c) {
			const float2 p = s[32 * c + lane];
			d[32 * c + lane] = make_float2(m.x != 0.f ? mn.x * (p.x / m.x) : 0.f, m.y != 0.f ? mn.y * (p.y / m.y) : 0.f);
		}
	}
}

}  // namespace cb200
