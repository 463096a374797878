// grid.cuh -- sparse-grid block kernels: velocity update + max query (+ fused clears), carry copy.
#pragma once
#include "collider.cuh"
#include "common.cuh"
#include "mgsp.cuh"

namespace cb200 {

constexpr int kGridThreads = 256;  // 8 warps, one grid block per warp per iteration

struct GridUpdateArgs {
	Cfg cfg;
	StepState* state;  // nullable: device-resident counts / dt
	int nbc, ebc;      // immediates when state == nullptr
	float dt;
	float* grid;             // mass/momentum in, velocity out (channels 1-3), nbc blocks
	const int* keys;
	float* max_vel;          // device float holding max |v|^2 (non-negative)
	float* clear_grid;       // nullable: next grid, nbc blocks zeroed        (clear_grid, mgmpm_kernels.cuh:106-115)
	int n_clear;             // number of cell-count arrays to zero over ebc blocks (cudaMemsetAsync at gmpm_simulator.cuh:389)
	int* clear_counts[kMaxModels];
	float time;              // boundary kernels, state == nullptr: time the boundaries are placed at (the driver reads StepState::sim_time)
};

// CTAs per SM a boundary instance is compiled for: the level-set-only one fits the driver's 4 at 256 threads (64 registers); the ones
// with objects take 2, without which ptxas picks 64 registers and spills
template<bool COLLIDE, bool OBJECTS>
constexpr int kBoundaryMinCtas = OBJECTS ? 2 : 4;

// ---- the boundary impulse report (DESIGN.md section 2.13) ----------------------------------------------------------------------
// Body 0 is the level-set collider, body 1 + i object i of the list.  Per body the grid update adds J = sum m (v_in - v_out) and
// L = sum (p - b(t)) x m (v_in - v_out) over the nodes with mass, v_in the velocity the body receives in the chain and v_out the one it
// leaves, p = n dx and b(t) = trans + trans_vel t the pivot its omega turns about; (Jx, Jy, Jz, Lx, Ly, Lz) per body.
constexpr int kForceBodies = 1 + CB200_MAX_COLLISION_OBJECTS;
constexpr int kForceComps = 6;
// A kernel parameter of its own beside Boundaries, so that GridUpdateArgs and the instances without the report keep their block.
struct ForceArgs {
	double* impulses;          // [kForceBodies][6], added into (one atomicAdd per CTA and non-zero component)
	const int* overlap_marks;  // nullable (MGSP): bit p of block b set when peer p also resolves b; b counts on the lowest rank holding it
	unsigned lower_ranks;      // (1u << rank) - 1
};
// the CTA's per-warp sums: each warp's lane 0 adds to its own slot, the CTA adds the 8 slots at its end
__device__ __forceinline__ double (*force_slots())[kForceBodies * kForceComps] {
	__shared__ double s[kGridThreads / 32][kForceBodies * kForceComps];
	return s;
}
__device__ __forceinline__ void force_slots_clear() {
	double* s = &force_slots()[0][0];
	for(int i = threadIdx.x; i < (kGridThreads / 32) * kForceBodies * kForceComps; i += kGridThreads) s[i] = 0.0;
}
// body k's impulse on the two cells a lane holds (velocities in i*, out o*; hx / hy: which have mass) added to the warp's slot k; the
// offset p - b is collider_material_point's xm.  A warp in which no lane changed a velocity skips the reduction (a lane's two
// contributions may cancel in J and not in L, so the test is on the velocities, not on the sums).
__device__ __forceinline__ void warp_body_impulse(double* slot, int lane, float dx, int nx, int ny, int nz, float2 m, bool hx, bool hy, const ColliderFrame& f, float2 i0, float2 i1, float2 i2,
                                                  float2 o0, float2 o1, float2 o2) {
	float r[kForceComps] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
	auto cell = [&](float mc, int z, float d0, float d1, float d2) {
		const float j[3] = {mc * d0, mc * d1, mc * d2};
		const float xm[3] = {(float) nx * dx - f.b[0], (float) ny * dx - f.b[1], (float) z * dx - f.b[2]};
		r[0] += j[0];
		r[1] += j[1];
		r[2] += j[2];
		r[3] += xm[1] * j[2] - xm[2] * j[1];
		r[4] += xm[2] * j[0] - xm[0] * j[2];
		r[5] += xm[0] * j[1] - xm[1] * j[0];
	};
	const bool cx = hx && (i0.x != o0.x || i1.x != o1.x || i2.x != o2.x), cy = hy && (i0.y != o0.y || i1.y != o1.y || i2.y != o2.y);
	if(!__any_sync(0xffffffffu, cx || cy)) return;
	if(cx) cell(m.x, nz, i0.x - o0.x, i1.x - o1.x, i2.x - o2.x);
	if(cy) cell(m.y, nz + 1, i0.y - o0.y, i1.y - o1.y, i2.y - o2.y);
#pragma unroll
	for(int c = 0; c < kForceComps; ++c) {
#pragma unroll
		for(int off = 16; off > 0; off >>= 1) r[c] += __shfl_xor_sync(0xffffffffu, r[c], off);
	}
	if(lane == 0) {
#pragma unroll
		for(int c = 0; c < kForceComps; ++c) slot[c] += (double) r[c];
	}
}

// update_grid_velocity_query_max (mgmpm_kernels.cuh:325-420): one warp per grid block, two cells per lane as
// one 8-byte access per channel; warp max by redux, one atomicMax per CTA on the float's bit pattern.
// Quirks kept: wall blocks zero the masked component BEFORE gravity is added to y (Appendix B #1);
// NaN -> +inf (B #3).
// COLLIDE / OBJECTS: the MGSP form with a Boundary (mgmpm_kernels.cuh:323-399): after gravity, cells with mass resolve against the
// boundary chain of `bd` (collider.cuh: the SignedDistanceGrid, then the analytic objects of DESIGN.md section 2.9); the max is |v|^2
// where that kernel reports 2|v|^2 (Appendix B #11).
// FORCES: the chain runs one body at a time over both cells of a lane (boundaries_resolve_pair) and each body's impulse is added to
// fa->impulses (section 2.13); the velocities are those of the instance without it.
// TRACKS (OBJECTS): the objects with a track in tr move on it (section 2.14), the pivot of their impulse report is c(t).
template<bool COLLIDE, bool OBJECTS, bool LEVELSETS = false, bool FORCES = false, bool TRACKS = false>
__device__ __forceinline__ void grid_update_body(const GridUpdateArgs& a, const Boundaries* bd, const ForceArgs* fa = nullptr, const Tracks* tr = nullptr) {
	static_assert(!FORCES || COLLIDE || OBJECTS, "the report needs a body");
	__shared__ unsigned s_max[kGridThreads / 32];
	if constexpr(FORCES) force_slots_clear();  // published by the frame builder's barrier
	const BoundaryFrames* fr = nullptr;
	if constexpr(TRACKS) fr = &boundary_frames_tracks_cta<COLLIDE>(*bd, *tr, a.state ? (float) a.state->sim_time : a.time);
	else if constexpr(COLLIDE || OBJECTS) fr = &boundary_frames_cta<COLLIDE, OBJECTS>(*bd, a.state ? (float) a.state->sim_time : a.time);
	const Cfg& cfg = a.cfg;
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const int nbc = a.state ? a.state->nbc : a.nbc;
	const int ebc = a.state ? a.state->ebc : a.ebc;
	const float dt = a.state ? a.state->dt : a.dt;
	const int total = max(nbc, (a.n_clear > 0) ? ebc : 0);
	const int g = cfg.gsize, bc = cfg.boundary;
	const float gdt = cfg.gravity * dt;
	unsigned vmax = 0u;
	for(int b = blockIdx.x * (kGridThreads / 32) + warp; b < total; b += gridDim.x * (kGridThreads / 32)) {
		if(b < nbc) {
			const int kx = a.keys[3 * b], ky = a.keys[3 * b + 1], kz = a.keys[3 * b + 2];
			const bool wx = (kx < bc) | (kx >= g - bc), wy = (ky < bc) | (ky >= g - bc), wz = (kz < bc) | (kz >= g - bc);
			float2* blk = reinterpret_cast<float2*>(a.grid + (size_t) b * kGridBlockFloats);
			const float2 m = blk[lane];
			float2 v0 = blk[32 + lane], v1 = blk[64 + lane], v2 = blk[96 + lane];
			float sq0 = 0.f, sq1 = 0.f;
			const bool hx = node_has_mass(m.x), hy = node_has_mass(m.y);
			if constexpr(FORCES) {
				if(hx) {
					const float mi = 1.f / m.x;
					v0.x = wx ? 0.f : v0.x * mi;
					v1.x = (wy ? 0.f : v1.x * mi) + gdt;
					v2.x = wz ? 0.f : v2.x * mi;
				}
				if(hy) {
					const float mi = 1.f / m.y;
					v0.y = wx ? 0.f : v0.y * mi;
					v1.y = (wy ? 0.f : v1.y * mi) + gdt;
					v2.y = wz ? 0.f : v2.y * mi;
				}
				const int nx = 4 * kx + (lane >> 3), ny = 4 * ky + ((lane >> 1) & 3), nz = 4 * kz + 2 * (lane & 1);
				const bool counted = !fa->overlap_marks || (fa->overlap_marks[b] & fa->lower_ranks) == 0u;  // warp-uniform
				double* slots = force_slots()[warp];
				if constexpr(TRACKS) {
					auto stage = [&](int k, const ColliderFrame& f, float2 i0, float2 i1, float2 i2) {
						if(counted) warp_body_impulse(slots + k * kForceComps, lane, cfg.dx, nx, ny, nz, m, hx, hy, f, i0, i1, i2, v0, v1, v2);
					};
					boundaries_resolve_pair<COLLIDE, OBJECTS, LEVELSETS, decltype(stage)&, true>(*bd, *fr, cfg, nx, ny, nz, hx, hy, v0, v1, v2, stage, tr);
				} else {
					boundaries_resolve_pair<COLLIDE, OBJECTS, LEVELSETS>(*bd, *fr, cfg, nx, ny, nz, hx, hy, v0, v1, v2, [&](int k, const ColliderFrame& f, float2 i0, float2 i1, float2 i2) {
						if(counted) warp_body_impulse(slots + k * kForceComps, lane, cfg.dx, nx, ny, nz, m, hx, hy, f, i0, i1, i2, v0, v1, v2);
					});
				}
				if(hx) sq0 = v0.x * v0.x + v1.x * v1.x + v2.x * v2.x;
				if(hy) sq1 = v0.y * v0.y + v1.y * v1.y + v2.y * v2.y;
			} else {
				if(hx) {
					const float mi = 1.f / m.x;
					v0.x = wx ? 0.f : v0.x * mi;
					v1.x = (wy ? 0.f : v1.x * mi) + gdt;
					v2.x = wz ? 0.f : v2.x * mi;
					if constexpr(COLLIDE || OBJECTS) boundaries_resolve<COLLIDE, OBJECTS, LEVELSETS, TRACKS>(*bd, *fr, cfg, 4 * kx + (lane >> 3), 4 * ky + ((lane >> 1) & 3), 4 * kz + 2 * (lane & 1), v0.x, v1.x, v2.x, tr);
					sq0 = v0.x * v0.x + v1.x * v1.x + v2.x * v2.x;
				}
				if(hy) {
					const float mi = 1.f / m.y;
					v0.y = wx ? 0.f : v0.y * mi;
					v1.y = (wy ? 0.f : v1.y * mi) + gdt;
					v2.y = wz ? 0.f : v2.y * mi;
					if constexpr(COLLIDE || OBJECTS) boundaries_resolve<COLLIDE, OBJECTS, LEVELSETS, TRACKS>(*bd, *fr, cfg, 4 * kx + (lane >> 3), 4 * ky + ((lane >> 1) & 3), 4 * kz + 2 * (lane & 1) + 1, v0.y, v1.y, v2.y, tr);
					sq1 = v0.y * v0.y + v1.y * v1.y + v2.y * v2.y;
				}
			}
			if(hx || hy) {
				blk[32 + lane] = v0;
				blk[64 + lane] = v1;
				blk[96 + lane] = v2;
			}
			if(isnan(sq0)) sq0 = INFINITY;
			if(isnan(sq1)) sq1 = INFINITY;
			vmax = max(vmax, __float_as_uint(fmaxf(sq0, sq1)));
			if(a.clear_grid) {
				float4* c = reinterpret_cast<float4*>(a.clear_grid + (size_t) b * kGridBlockFloats);
				c[lane] = make_float4(0.f, 0.f, 0.f, 0.f);
				c[32 + lane] = make_float4(0.f, 0.f, 0.f, 0.f);
			}
		}
		if(b < ebc) {
			for(int m = 0; m < a.n_clear; ++m) reinterpret_cast<int2*>(a.clear_counts[m] + (size_t) b * kBlockVol)[lane] = make_int2(0, 0);
		}
	}
	vmax = __reduce_max_sync(0xffffffffu, vmax);
	if(lane == 0) s_max[warp] = vmax;
	__syncthreads();
	if(threadIdx.x == 0) {
		unsigned m = s_max[0];
#pragma unroll
		for(int i = 1; i < kGridThreads / 32; ++i) m = max(m, s_max[i]);
		if(m) atomicMax(reinterpret_cast<unsigned*>(a.max_vel), m);
	}
	if constexpr(FORCES) {  // behind the max's barrier: every warp's slots are complete
		for(int i = threadIdx.x; i < kForceBodies * kForceComps; i += kGridThreads) {
			double sum = 0.0;
#pragma unroll
			for(int w = 0; w < kGridThreads / 32; ++w) sum += force_slots()[w][i];
			if(sum != 0.0) atomicAdd(fa->impulses + i, sum);
		}
	}
}
__global__ void __launch_bounds__(kGridThreads) grid_update_kernel(const GridUpdateArgs a) { grid_update_body<false, false>(a, nullptr); }
// the same with the boundaries of bd (COLLIDE: bd.has_collider; OBJECTS: bd.objects.n >= 1)
template<bool COLLIDE, bool OBJECTS>
__global__ void __launch_bounds__(kGridThreads, (kBoundaryMinCtas<COLLIDE, OBJECTS>)) grid_update_boundary_kernel(const GridUpdateArgs a, const __grid_constant__ Boundaries bd) {
	grid_update_body<COLLIDE, OBJECTS>(a, &bd);
}
static_assert(sizeof(GridUpdateArgs) + sizeof(Boundaries) <= 4096, "the boundary grid update's parameters must fit the 4 KiB kernel-parameter limit");
// the same with level-set objects among bd's objects, their lattices in ls (DESIGN.md section 2.11); COLLIDE: bd.has_collider
template<bool COLLIDE>
__global__ void __launch_bounds__(kGridThreads, (kBoundaryMinCtas<COLLIDE, true>)) grid_update_levelset_kernel(const GridUpdateArgs a, const __grid_constant__ Boundaries bd, const __grid_constant__ LevelSets ls) {
	levelset_views_cta(ls);  // published by the frame builder's barrier
	grid_update_body<COLLIDE, true, true>(a, &bd);
}
static_assert(sizeof(GridUpdateArgs) + sizeof(Boundaries) + sizeof(LevelSets) <= 4096, "the level-set grid update's parameters must fit the 4 KiB kernel-parameter limit");
// the two with the impulse report of fa (section 2.13)
template<bool COLLIDE, bool OBJECTS>
__global__ void __launch_bounds__(kGridThreads, (kBoundaryMinCtas<COLLIDE, OBJECTS>)) grid_update_boundary_forces_kernel(const GridUpdateArgs a, const __grid_constant__ Boundaries bd, const __grid_constant__ ForceArgs fa) {
	grid_update_body<COLLIDE, OBJECTS, false, true>(a, &bd, &fa);
}
static_assert(sizeof(GridUpdateArgs) + sizeof(Boundaries) + sizeof(ForceArgs) <= 4096, "the reporting boundary grid update's parameters must fit the 4 KiB kernel-parameter limit");
template<bool COLLIDE>
__global__ void __launch_bounds__(kGridThreads, (kBoundaryMinCtas<COLLIDE, true>)) grid_update_levelset_forces_kernel(const GridUpdateArgs a, const __grid_constant__ Boundaries bd, const __grid_constant__ LevelSets ls,
                                                                                                                     const __grid_constant__ ForceArgs fa) {
	levelset_views_cta(ls);
	grid_update_body<COLLIDE, true, true, true>(a, &bd, &fa);
}
static_assert(sizeof(GridUpdateArgs) + sizeof(Boundaries) + sizeof(LevelSets) + sizeof(ForceArgs) <= 4096, "the reporting level-set grid update's parameters must fit the 4 KiB kernel-parameter limit");
// the same with the objects' tracks tr (section 2.14), with or without level-set objects (ls) and the report (fa); COLLIDE: bd.has_collider
template<bool COLLIDE, bool LEVELSETS, bool FORCES>
__global__ void __launch_bounds__(kGridThreads, (kBoundaryMinCtas<COLLIDE, true>)) grid_update_tracks_kernel(const GridUpdateArgs a, const __grid_constant__ Boundaries bd, const __grid_constant__ LevelSets ls,
                                                                                                            const __grid_constant__ ForceArgs fa, const __grid_constant__ Tracks tr) {
	if constexpr(LEVELSETS) levelset_views_cta(ls);  // published by the frame builder's barrier
	grid_update_body<COLLIDE, true, LEVELSETS, FORCES, true>(a, &bd, &fa, &tr);
}
static_assert(sizeof(GridUpdateArgs) + sizeof(Boundaries) + sizeof(LevelSets) + sizeof(ForceArgs) + sizeof(Tracks) <= 4096, "the tracked grid update's parameters must fit the 4 KiB kernel-parameter limit");

// clear_grid (mgmpm_kernels.cuh:106-115)
__global__ void clear_grid_kernel(int block_count, float* grid) {
	const size_t n4 = (size_t) block_count * (kGridBlockFloats / 4);
	float4* g = reinterpret_cast<float4*>(grid);
	for(size_t i = blockIdx.x * (size_t) blockDim.x + threadIdx.x; i < n4; i += (size_t) gridDim.x * blockDim.x) g[i] = make_float4(0.f, 0.f, 0.f, 0.f);
}

// Carry of the next-grid into the new numbering.  The reference clears grid[0] and scatters marked blocks
// through the new table (clear_grid + copy_selected_grid_blocks, mgmpm_kernels.cuh:1002-1020,
// gmpm_simulator.cuh:536-541).  Here every block of the NEW numbering pulls its source through the OLD table:
// one pass, each destination written exactly once (zero when it had no predecessor), no marks needed because
// copying an all-zero block equals clearing it.
struct CarryArgs {
	Cfg cfg;
	const int* new_count;   // device: number of blocks to produce (new neighbour count)
	const int* new_keys;
	const int* old_table;
	const StepState* state; // old nbc = state->nbc
	const float* old_grid;
	float* new_grid;
	float* next_max_vel;    // nullable (MGSP): max |v|^2 the NEXT grid update will find on this rank, so that the all-reduce
	                        // of it can ride on the end-of-step key exchange instead of being a sync point of its own
	// MGSP: reset the tagging state of the new partition on the way (reset_overlap_marks, hash_table.cuh:64-66);
	// the launch sits behind mgsp_done_wait_kernel: the old next-grid is complete only when every peer's halo reductions have landed
	int mgsp;
	MgspView view;
	int* overlap_marks;
};
// COLLIDE / OBJECTS (MGSP): the predictor applies the boundaries of bd at the time the next grid update sees
template<bool COLLIDE, bool OBJECTS, bool LEVELSETS = false, bool TRACKS = false>
__device__ __forceinline__ void carry_grid_body(const CarryArgs& a, const Boundaries* bd, const Tracks* tr = nullptr) {
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const int n = *a.new_count;
	const int old_nbc = a.state->nbc;
	const int g = a.cfg.gsize, bc = a.cfg.boundary;
	if(a.mgsp && blockIdx.x == 0 && (int) threadIdx.x < a.view.world) a.view.overlap_count[threadIdx.x] = 0;
	float gdt = 0.f;
	if(a.next_max_vel) gdt = a.cfg.gravity * device_compute_dt(a.cfg, a.state->max_vel_sq, a.state->step_time, a.state->frame_time, a.state->dt_default);
	const BoundaryFrames* fr = nullptr;
	if constexpr(TRACKS) fr = &boundary_frames_tracks_cta<COLLIDE>(*bd, *tr, (float) (a.state->sim_time + (double) a.state->dt));
	else if constexpr(COLLIDE || OBJECTS) fr = &boundary_frames_cta<COLLIDE, OBJECTS>(*bd, (float) (a.state->sim_time + (double) a.state->dt));  // the clock rolls by this sub-step's dt
	unsigned vmax = 0u;
	for(int j = blockIdx.x * 8 + warp; j < n; j += gridDim.x * 8) {
		const int kx = a.new_keys[3 * j], ky = a.new_keys[3 * j + 1], kz = a.new_keys[3 * j + 2];
		const int src = table_query(a.cfg, a.old_table, kx, ky, kz);
		if(a.mgsp) {
			if(lane == 0) a.overlap_marks[j] = 0;
			if(lane < a.view.world) a.view.peer_bno[(size_t) lane * a.view.L.max_blocks + j] = -1;
		}
		float4* d = reinterpret_cast<float4*>(a.new_grid + (size_t) j * kGridBlockFloats);
		if(src >= 0 && src < old_nbc) {
			const float4* s = reinterpret_cast<const float4*>(a.old_grid + (size_t) src * kGridBlockFloats);
			d[lane] = s[lane];
			d[32 + lane] = s[32 + lane];
			if(a.next_max_vel) {
				const float2* s2 = reinterpret_cast<const float2*>(s);
				const bool wx = (kx < bc) | (kx >= g - bc), wy = (ky < bc) | (ky >= g - bc), wz = (kz < bc) | (kz >= g - bc);
				if constexpr(COLLIDE || OBJECTS) vmax = max(vmax, __float_as_uint(cell_pair_vel_sq_boundaries<COLLIDE, OBJECTS, LEVELSETS, TRACKS>(a.cfg, *bd, *fr, s2, lane, kx, ky, kz, wx, wy, wz, gdt, tr)));
				else vmax = max(vmax, __float_as_uint(cell_pair_vel_sq(s2[lane], s2[32 + lane], s2[64 + lane], s2[96 + lane], wx, wy, wz, gdt)));
			}
		} else {
			d[lane] = make_float4(0.f, 0.f, 0.f, 0.f);
			d[32 + lane] = make_float4(0.f, 0.f, 0.f, 0.f);
		}
	}
	if(a.next_max_vel) {
		vmax = __reduce_max_sync(0xffffffffu, vmax);
		if(lane == 0 && vmax) atomicMax(reinterpret_cast<unsigned*>(a.next_max_vel), vmax);
	}
}
__global__ void __launch_bounds__(256) carry_grid_kernel(const CarryArgs a) { carry_grid_body<false, false>(a, nullptr); }
template<bool COLLIDE, bool OBJECTS>
__global__ void __launch_bounds__(256, (kBoundaryMinCtas<COLLIDE, OBJECTS>)) carry_grid_boundary_kernel(const CarryArgs a, const __grid_constant__ Boundaries bd) {
	carry_grid_body<COLLIDE, OBJECTS>(a, &bd);
}
static_assert(sizeof(CarryArgs) + sizeof(Boundaries) <= 4096, "the boundary carry's parameters must fit the 4 KiB kernel-parameter limit");
template<bool COLLIDE>
__global__ void __launch_bounds__(256, (kBoundaryMinCtas<COLLIDE, true>)) carry_grid_levelset_kernel(const CarryArgs a, const __grid_constant__ Boundaries bd, const __grid_constant__ LevelSets ls) {
	levelset_views_cta(ls);
	carry_grid_body<COLLIDE, true, true>(a, &bd);
}
static_assert(sizeof(CarryArgs) + sizeof(Boundaries) + sizeof(LevelSets) <= 4096, "the level-set carry's parameters must fit the 4 KiB kernel-parameter limit");
template<bool COLLIDE, bool LEVELSETS>
__global__ void __launch_bounds__(256, (kBoundaryMinCtas<COLLIDE, true>)) carry_grid_tracks_kernel(const CarryArgs a, const __grid_constant__ Boundaries bd, const __grid_constant__ LevelSets ls, const __grid_constant__ Tracks tr) {
	if constexpr(LEVELSETS) levelset_views_cta(ls);
	carry_grid_body<COLLIDE, true, LEVELSETS, true>(a, &bd, &tr);
}
static_assert(sizeof(CarryArgs) + sizeof(Boundaries) + sizeof(LevelSets) + sizeof(Tracks) <= 4096, "the tracked carry's parameters must fit the 4 KiB kernel-parameter limit");

// max |v|^2 the grid update will find, without touching the grid (MGSP start-up)
template<bool COLLIDE, bool OBJECTS, bool LEVELSETS = false, bool TRACKS = false>
__device__ __forceinline__ void grid_max_body(const Cfg& cfg, const StepState* state, const float* grid, const int* keys, float* max_vel, const Boundaries* bd, const Tracks* tr = nullptr) {
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const int g = cfg.gsize, bc = cfg.boundary;
	const float gdt = cfg.gravity * state->dt;
	const BoundaryFrames* fr = nullptr;
	if constexpr(TRACKS) fr = &boundary_frames_tracks_cta<COLLIDE>(*bd, *tr, (float) state->sim_time);
	else if constexpr(COLLIDE || OBJECTS) fr = &boundary_frames_cta<COLLIDE, OBJECTS>(*bd, (float) state->sim_time);
	unsigned vmax = 0u;
	for(int b = blockIdx.x * 8 + warp; b < state->nbc; b += gridDim.x * 8) {
		const int kx = keys[3 * b], ky = keys[3 * b + 1], kz = keys[3 * b + 2];
		const bool wx = (kx < bc) | (kx >= g - bc), wy = (ky < bc) | (ky >= g - bc), wz = (kz < bc) | (kz >= g - bc);
		const float2* s2 = reinterpret_cast<const float2*>(grid + (size_t) b * kGridBlockFloats);
		if constexpr(COLLIDE || OBJECTS) vmax = max(vmax, __float_as_uint(cell_pair_vel_sq_boundaries<COLLIDE, OBJECTS, LEVELSETS, TRACKS>(cfg, *bd, *fr, s2, lane, kx, ky, kz, wx, wy, wz, gdt, tr)));
		else vmax = max(vmax, __float_as_uint(cell_pair_vel_sq(s2[lane], s2[32 + lane], s2[64 + lane], s2[96 + lane], wx, wy, wz, gdt)));
	}
	vmax = __reduce_max_sync(0xffffffffu, vmax);
	if(lane == 0 && vmax) atomicMax(reinterpret_cast<unsigned*>(max_vel), vmax);
}
__global__ void __launch_bounds__(256) grid_max_kernel(Cfg cfg, const StepState* state, const float* grid, const int* keys, float* max_vel) {
	grid_max_body<false, false>(cfg, state, grid, keys, max_vel, nullptr);
}
template<bool COLLIDE, bool OBJECTS>
__global__ void __launch_bounds__(256, (kBoundaryMinCtas<COLLIDE, OBJECTS>)) grid_max_boundary_kernel(Cfg cfg, const StepState* state, const float* grid, const int* keys, float* max_vel, const __grid_constant__ Boundaries bd) {
	grid_max_body<COLLIDE, OBJECTS>(cfg, state, grid, keys, max_vel, &bd);
}
template<bool COLLIDE>
__global__ void __launch_bounds__(256, (kBoundaryMinCtas<COLLIDE, true>)) grid_max_levelset_kernel(Cfg cfg, const StepState* state, const float* grid, const int* keys, float* max_vel, const __grid_constant__ Boundaries bd, const __grid_constant__ LevelSets ls) {
	levelset_views_cta(ls);
	grid_max_body<COLLIDE, true, true>(cfg, state, grid, keys, max_vel, &bd);
}
template<bool COLLIDE, bool LEVELSETS>
__global__ void __launch_bounds__(256, (kBoundaryMinCtas<COLLIDE, true>)) grid_max_tracks_kernel(Cfg cfg, const StepState* state, const float* grid, const int* keys, float* max_vel, const __grid_constant__ Boundaries bd,
                                                                                                const __grid_constant__ LevelSets ls, const __grid_constant__ Tracks tr) {
	if constexpr(LEVELSETS) levelset_views_cta(ls);
	grid_max_body<COLLIDE, true, LEVELSETS, true>(cfg, state, grid, keys, max_vel, &bd, &tr);
}

// ---- launching the three boundary passes ---------------------------------------------------------------------------------------
inline bool has_levelset_objects(const Boundaries& bd) {
	for(int i = 0; i < bd.objects.n; ++i)
		if(bd.objects.o[i].shape == CB200_SHAPE_LEVELSET) return true;
	return false;
}
// Calls f(COLLIDE, OBJECTS, LEVELSETS), three std::bool_constant, with the instance flags that apply bd: the level set when
// bd.has_collider, the objects when the list is non-empty, the level-set instances (OBJECTS too) only when an object is a level set;
// none is the plain kernel.  Each pass keeps all four instances without level sets, because the level-set-only one fits 4 CTAs per SM
// and the level set + objects one does not.
template<class F>
void with_boundaries(const Boundaries& bd, F&& f) {
	using T = std::true_type;
	using N = std::false_type;
	if(has_levelset_objects(bd)) {
		if(bd.has_collider) f(T(), T(), T());
		else f(N(), T(), T());
	} else if(bd.has_collider && bd.objects.n > 0) f(T(), T(), N());
	else if(bd.has_collider) f(T(), N(), N());
	else if(bd.objects.n > 0) f(N(), T(), N());
	else f(N(), N(), N());
}
// f(COLLIDE, LEVELSETS), two std::bool_constant, for the tracked instances that apply bd (section 2.14)
template<class F>
void with_tracks(const Boundaries& bd, F&& f) {
	using T = std::true_type;
	using N = std::false_type;
	if(has_levelset_objects(bd)) {
		if(bd.has_collider) f(T(), T());
		else f(N(), T());
	} else if(bd.has_collider) f(T(), N());
	else f(N(), N());
}
// f(COLLIDE, OBJECTS) for each boundary instance without level sets
template<class F>
void for_each_boundary_instance(F&& f) {
	f(std::true_type(), std::false_type());
	f(std::false_type(), std::true_type());
	f(std::true_type(), std::true_type());
}
// ls: the lattices bd's level-set objects index (read only when one is); fa (nullable): report the impulses there (no body: nothing)
// tr (nullable): the objects' tracks; the tracked instances run only when one of bd's objects has a track
inline void launch_grid_update(const GridUpdateArgs& a, const Boundaries& bd, const LevelSets& ls, int ctas, cudaStream_t st, const ForceArgs* fa = nullptr, const Tracks* tr = nullptr) {
	if(tracks_any(tr)) {
		const ForceArgs none {};
		with_tracks(bd, [&](auto C, auto L) {
			if(fa) grid_update_tracks_kernel<C, L, true><<<ctas, kGridThreads, 0, st>>>(a, bd, ls, *fa, *tr);
			else grid_update_tracks_kernel<C, L, false><<<ctas, kGridThreads, 0, st>>>(a, bd, ls, none, *tr);
		});
		return;
	}
	with_boundaries(bd, [&](auto C, auto O, auto L) {
		if constexpr(L) {
			if(fa) grid_update_levelset_forces_kernel<C><<<ctas, kGridThreads, 0, st>>>(a, bd, ls, *fa);
			else grid_update_levelset_kernel<C><<<ctas, kGridThreads, 0, st>>>(a, bd, ls);
		} else if constexpr(C || O) {
			if(fa) grid_update_boundary_forces_kernel<C, O><<<ctas, kGridThreads, 0, st>>>(a, bd, *fa);
			else grid_update_boundary_kernel<C, O><<<ctas, kGridThreads, 0, st>>>(a, bd);
		} else {
			grid_update_kernel<<<ctas, kGridThreads, 0, st>>>(a);
		}
	});
}
inline void launch_carry_grid(const CarryArgs& a, const Boundaries& bd, const LevelSets& ls, int ctas, cudaStream_t st, const Tracks* tr = nullptr) {
	if(tracks_any(tr)) {
		with_tracks(bd, [&](auto C, auto L) { carry_grid_tracks_kernel<C, L><<<ctas, 256, 0, st>>>(a, bd, ls, *tr); });
		return;
	}
	with_boundaries(bd, [&](auto C, auto O, auto L) {
		if constexpr(L) carry_grid_levelset_kernel<C><<<ctas, 256, 0, st>>>(a, bd, ls);
		else if constexpr(C || O) carry_grid_boundary_kernel<C, O><<<ctas, 256, 0, st>>>(a, bd);
		else carry_grid_kernel<<<ctas, 256, 0, st>>>(a);
	});
}
inline void launch_grid_max(const Cfg& cfg, const StepState* state, const float* grid, const int* keys, float* max_vel, const Boundaries& bd, const LevelSets& ls, int ctas, cudaStream_t st,
                            const Tracks* tr = nullptr) {
	if(tracks_any(tr)) {
		with_tracks(bd, [&](auto C, auto L) { grid_max_tracks_kernel<C, L><<<ctas, 256, 0, st>>>(cfg, state, grid, keys, max_vel, bd, ls, *tr); });
		return;
	}
	with_boundaries(bd, [&](auto C, auto O, auto L) {
		if constexpr(L) grid_max_levelset_kernel<C><<<ctas, 256, 0, st>>>(cfg, state, grid, keys, max_vel, bd, ls);
		else if constexpr(C || O) grid_max_boundary_kernel<C, O><<<ctas, 256, 0, st>>>(cfg, state, grid, keys, max_vel, bd);
		else grid_max_kernel<<<ctas, 256, 0, st>>>(cfg, state, grid, keys, max_vel);
	});
}

// copy_selected_grid_blocks (mgmpm_kernels.cuh:1002-1020), drop-in form: scatter marked blocks
__global__ void copy_selected_grid_blocks_kernel(Cfg cfg, int prev_block_count, const int* prev_blockids, const int* table, const int* marks, const float* prev_grid, float* grid) {
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	for(int b = blockIdx.x * 8 + warp; b < prev_block_count; b += gridDim.x * 8) {
		if(!marks[b]) continue;
		const int bno = table_query(cfg, table, prev_blockids[3 * b], prev_blockids[3 * b + 1], prev_blockids[3 * b + 2]);
		if(bno < 0) continue;
		const float4* s = reinterpret_cast<const float4*>(prev_grid + (size_t) b * kGridBlockFloats);
		float4* d = reinterpret_cast<float4*>(grid + (size_t) bno * kGridBlockFloats);
		d[lane] = s[lane];
		d[32 + lane] = s[32 + lane];
	}
}

// mark_active_grid_blocks (mgmpm_kernels.cuh:939-952): warp per block, ballot over the mass channel
__global__ void mark_active_grid_blocks_kernel(int block_count, const float* grid, int* marks) {
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	for(int b = blockIdx.x * 8 + warp; b < block_count; b += gridDim.x * 8) {
		const float2 m = reinterpret_cast<const float2*>(grid + (size_t) b * kGridBlockFloats)[lane];
		const unsigned any = __ballot_sync(0xffffffffu, m.x != 0.f || m.y != 0.f);
		if(lane == 0 && any) marks[b] = 1;
	}
}

}  // namespace cb200
