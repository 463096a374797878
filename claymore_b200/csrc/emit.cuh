// emit.cuh -- adding particles to a set-up simulator at a sub-step boundary (cb200_sim_add_particles*, include/claymore_b200.h).
//   * the checks of the candidates and the empty-cell filter, read against the current partition's cell offsets;
//   * the union's block counts and per-cell counts, built on a scratch table so that nothing live is touched before the commit;
//   * the state rows of the new particles, in the checkpoint's layout, so the commit is initial_setup over saved rows.
// One-time work per call, thread per candidate.
#pragma once
#include "checkpoint.cuh"
#include "init.cuh"

namespace cb200 {

enum : int { kEmitBadPosition = 1, kEmitCellOverflow = 2 };

// The current partition's occupancy: at a sub-step boundary with roll R the particle blocks are part[R]'s first pbc keys, and their
// cell-major buckets (sizes and per-cell offsets) are the Rn buffers the last rebuild wrote.
struct EmitCells {
	Cfg cfg;
	const int* table;   // part[R].index_table
	const int* pbc;     // &StepState::pbc
	int n_models;
	const unsigned short* offs[kMaxModels];  // celloffs[Rn]: [blocks][64]
	const int* sizes[kMaxModels];            // pb[Rn].particle_bucket_sizes
};

// particles of every model in bucket cell (cx, cy, cz) (cell index - 2, as build_particle_cell_buckets buckets them).  A model's cell
// offsets of a block are valid only where its bucket is not empty: rebuild_kernel writes no offsets for a model with no particle in
// a block, so that row still holds what an earlier partition left at the same block number.
__device__ __forceinline__ int emit_occupancy(const EmitCells& c, int cx, int cy, int cz) {
	const int b = table_query(c.cfg, c.table, cx >> 2, cy >> 2, cz >> 2);
	if(b < 0 || b >= *c.pbc) return 0;
	const int cell = (cx & 3) * 16 + (cy & 3) * 4 + (cz & 3);
	int n = 0;
	for(int m = 0; m < c.n_models; ++m) {
		const int size = c.sizes[m][b];
		if(size == 0) continue;
		const unsigned short* o = c.offs[m] + (size_t) b * kBlockVol;
		n += (cell < kBlockVol - 1 ? (int) o[cell + 1] : size) - (int) o[cell];
	}
	return n;
}

// A candidate is bad when a coordinate is not finite or its bucket block (cell index - 2, floor) lies outside the domain; the range is
// checked on the rounded float before cell_index converts it.  keep[p]: 0 for a bad candidate and, with `empty`, for one whose
// cell holds a particle.
__global__ void emit_filter_kernel(EmitCells c, int n, const float* pos, int empty, int* keep, int* bad) {
	const float top = (float) (4 * c.cfg.gsize + 2);
	for(int p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) {
		bool ok = true;
#pragma unroll
		for(int d = 0; d < 3; ++d) {
			const float x = pos[3 * p + d];
			const float r = roundf(x * c.cfg.dx_inv);
			ok &= isfinite(x) && r >= 2.f && r < top;
		}
		if(!ok) {
			keep[p] = 0;
			atomicOr(bad, kEmitBadPosition);
			continue;
		}
		keep[p] = !(empty && emit_occupancy(c, cell_index(c.cfg, pos[3 * p]) - 2, cell_index(c.cfg, pos[3 * p + 1]) - 2, cell_index(c.cfg, pos[3 * p + 2]) - 2) > 0);
	}
}

// the kept candidates in their order: offs is the exclusive scan of keep
__global__ void emit_compact_kernel(int n, const float* pos, const int* keep, const int* offs, float* out) {
	for(int p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x)
		if(keep[p])
			for(int d = 0; d < 3; ++d) out[3 * offs[p] + d] = pos[3 * p + d];
}

// the current particle blocks into the scratch table, so that they come first, as in the rebuilt partition
__global__ void emit_insert_keys_kernel(Cfg cfg, int count, const int* keys, int* table, int* out_keys, int* out_count, int capacity) {
	for(int b = blockIdx.x * blockDim.x + threadIdx.x; b < count; b += gridDim.x * blockDim.x) partition_insert(cfg, table, out_keys, out_count, capacity, nullptr, keys[3 * b], keys[3 * b + 1], keys[3 * b + 2]);
}

// new particles per cell of the union's particle blocks (scratch numbering, [blocks][64])
__global__ void emit_count_kernel(Cfg cfg, int n, const float* pos, const int* table, int* cells) {
	for(int p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) {
		const int cx = cell_index(cfg, pos[3 * p]) - 2, cy = cell_index(cfg, pos[3 * p + 1]) - 2, cz = cell_index(cfg, pos[3 * p + 2]) - 2;
		const int b = table_query(cfg, table, cx >> 2, cy >> 2, cz >> 2);
		atomicAdd(cells + (size_t) b * kBlockVol + (cx & 3) * 16 + (cy & 3) * 4 + (cz & 3), 1);
	}
}

// a cell of a candidate that would hold more than max_ppc particles, existing and new
__global__ void emit_overflow_kernel(EmitCells c, int n, const float* pos, const int* table, const int* cells, int* bad) {
	for(int p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) {
		const int cx = cell_index(c.cfg, pos[3 * p]) - 2, cy = cell_index(c.cfg, pos[3 * p + 1]) - 2, cz = cell_index(c.cfg, pos[3 * p + 2]) - 2;
		const int b = table_query(c.cfg, table, cx >> 2, cy >> 2, cz >> 2);
		const int added = cells[(size_t) b * kBlockVol + (cx & 3) * 16 + (cy & 3) * 4 + (cz & 3)];
		if(emit_occupancy(c, cx, cy, cz) + added > c.cfg.max_ppc) atomicOr(bad, kEmitCellOverflow);
	}
}

// the state rows of new particles (checkpoint channels): their start state
__global__ void emit_rows_kernel(int material, int n, const float* pos, float* rows) {
	const int C = ck_channels(material);
	for(int p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) start_state(material, pos + 3 * p, rows + (size_t) p * C, 1);
}

}  // namespace cb200
