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
	ColliderView col;        // COLLIDE only
	float time;              // COLLIDE, state == nullptr: time the collider is placed at (the driver reads StepState::sim_time)
};

// update_grid_velocity_query_max (mgmpm_kernels.cuh:325-420): one warp per grid block, two cells per lane as
// one 8-byte access per channel; warp max by redux, one atomicMax per CTA on the float's bit pattern.
// Quirks kept: wall blocks zero the masked component BEFORE gravity is added to y (Appendix B #1);
// NaN -> +inf (B #3).
// COLLIDE: the MGSP form with a SignedDistanceGrid (mgmpm_kernels.cuh:323-399): after gravity, cells with mass resolve against
// the collider (collider.cuh); the max is |v|^2 where that kernel reports 2|v|^2 (Appendix B #11).
// OBJECTS: then the analytic objects of `objs` in list order (collider.cuh, DESIGN.md section 2.9), placed at the collider's time.
template<bool COLLIDE, bool OBJECTS>
__device__ __forceinline__ void grid_update_body(const GridUpdateArgs& a, const ObjectList* objs) {
	__shared__ unsigned s_max[kGridThreads / 32];
	const ColliderFrame* fr = nullptr;
	const ObjectFrames* of = nullptr;
	if constexpr(OBJECTS) of = &object_frames_cta<COLLIDE>(a.col, *objs, a.state ? (float) a.state->sim_time : a.time);
	else if constexpr(COLLIDE) fr = &collider_frame_cta(a.col, a.state ? (float) a.state->sim_time : a.time);
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
			if(hx) {
				const float mi = 1.f / m.x;
				v0.x = wx ? 0.f : v0.x * mi;
				v1.x = (wy ? 0.f : v1.x * mi) + gdt;
				v2.x = wz ? 0.f : v2.x * mi;
				if constexpr(OBJECTS) objects_resolve<COLLIDE>(a.col, *of, objs->n, cfg, 4 * kx + (lane >> 3), 4 * ky + ((lane >> 1) & 3), 4 * kz + 2 * (lane & 1), v0.x, v1.x, v2.x);
				else if constexpr(COLLIDE) collider_resolve(a.col, *fr, cfg, 4 * kx + (lane >> 3), 4 * ky + ((lane >> 1) & 3), 4 * kz + 2 * (lane & 1), v0.x, v1.x, v2.x);
				sq0 = v0.x * v0.x + v1.x * v1.x + v2.x * v2.x;
			}
			if(hy) {
				const float mi = 1.f / m.y;
				v0.y = wx ? 0.f : v0.y * mi;
				v1.y = (wy ? 0.f : v1.y * mi) + gdt;
				v2.y = wz ? 0.f : v2.y * mi;
				if constexpr(OBJECTS) objects_resolve<COLLIDE>(a.col, *of, objs->n, cfg, 4 * kx + (lane >> 3), 4 * ky + ((lane >> 1) & 3), 4 * kz + 2 * (lane & 1) + 1, v0.y, v1.y, v2.y);
				else if constexpr(COLLIDE) collider_resolve(a.col, *fr, cfg, 4 * kx + (lane >> 3), 4 * ky + ((lane >> 1) & 3), 4 * kz + 2 * (lane & 1) + 1, v0.y, v1.y, v2.y);
				sq1 = v0.y * v0.y + v1.y * v1.y + v2.y * v2.y;
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
}
template<bool COLLIDE>
__global__ void __launch_bounds__(kGridThreads) grid_update_kernel(const GridUpdateArgs a) { grid_update_body<COLLIDE, false>(a, nullptr); }
// the same with analytic objects (objs.n >= 1): the list is a parameter of its own, so the kernels above keep their parameter block
template<bool COLLIDE>
__global__ void __launch_bounds__(kGridThreads, 2) grid_update_objects_kernel(const GridUpdateArgs a, const __grid_constant__ ObjectList objs) { grid_update_body<COLLIDE, true>(a, &objs); }
static_assert(sizeof(GridUpdateArgs) + sizeof(ObjectList) <= 4096, "the objects grid update's parameters must fit the 4 KiB kernel-parameter limit");

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
	ColliderView col;  // COLLIDE: the predictor applies the collider at the time the next grid update sees
};
template<bool COLLIDE, bool OBJECTS>
__device__ __forceinline__ void carry_grid_body(const CarryArgs& a, const ObjectList* objs) {
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const int n = *a.new_count;
	const int old_nbc = a.state->nbc;
	const int g = a.cfg.gsize, bc = a.cfg.boundary;
	if(a.mgsp && blockIdx.x == 0 && (int) threadIdx.x < a.view.world) a.view.overlap_count[threadIdx.x] = 0;
	float gdt = 0.f;
	if(a.next_max_vel) gdt = a.cfg.gravity * device_compute_dt(a.cfg, a.state->max_vel_sq, a.state->step_time, a.state->frame_time, a.state->dt_default);
	const ColliderFrame* fr = nullptr;
	const ObjectFrames* of = nullptr;
	if constexpr(OBJECTS) of = &object_frames_cta<COLLIDE>(a.col, *objs, (float) (a.state->sim_time + (double) a.state->dt));
	else if constexpr(COLLIDE) fr = &collider_frame_cta(a.col, (float) (a.state->sim_time + (double) a.state->dt));  // the clock rolls by this sub-step's dt
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
				if constexpr(OBJECTS) vmax = max(vmax, __float_as_uint(cell_pair_vel_sq_objects<COLLIDE>(a.cfg, a.col, *of, objs->n, s2, lane, kx, ky, kz, wx, wy, wz, gdt)));
				else if constexpr(COLLIDE) vmax = max(vmax, __float_as_uint(cell_pair_vel_sq_collide(a.cfg, a.col, *fr, s2, lane, kx, ky, kz, wx, wy, wz, gdt)));
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
template<bool COLLIDE>
__global__ void __launch_bounds__(256) carry_grid_kernel(const CarryArgs a) { carry_grid_body<COLLIDE, false>(a, nullptr); }
// OBJECTS: the predictor applies the objects too (MGSP; objs.n >= 1)
template<bool COLLIDE>
__global__ void __launch_bounds__(256, 2) carry_grid_objects_kernel(const CarryArgs a, const __grid_constant__ ObjectList objs) { carry_grid_body<COLLIDE, true>(a, &objs); }
static_assert(sizeof(CarryArgs) + sizeof(ObjectList) <= 4096, "the objects carry's parameters must fit the 4 KiB kernel-parameter limit");

// max |v|^2 the grid update will find, without touching the grid (MGSP start-up)
template<bool COLLIDE>
__global__ void __launch_bounds__(256) grid_max_kernel(Cfg cfg, const StepState* state, const float* grid, const int* keys, float* max_vel, const ColliderView col) {
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const int g = cfg.gsize, bc = cfg.boundary;
	const float gdt = cfg.gravity * state->dt;
	const ColliderFrame* fr = nullptr;
	if constexpr(COLLIDE) fr = &collider_frame_cta(col, (float) state->sim_time);
	unsigned vmax = 0u;
	for(int b = blockIdx.x * 8 + warp; b < state->nbc; b += gridDim.x * 8) {
		const int kx = keys[3 * b], ky = keys[3 * b + 1], kz = keys[3 * b + 2];
		const bool wx = (kx < bc) | (kx >= g - bc), wy = (ky < bc) | (ky >= g - bc), wz = (kz < bc) | (kz >= g - bc);
		const float2* s2 = reinterpret_cast<const float2*>(grid + (size_t) b * kGridBlockFloats);
		if constexpr(COLLIDE) vmax = max(vmax, __float_as_uint(cell_pair_vel_sq_collide(cfg, col, *fr, s2, lane, kx, ky, kz, wx, wy, wz, gdt)));
		else vmax = max(vmax, __float_as_uint(cell_pair_vel_sq(s2[lane], s2[32 + lane], s2[64 + lane], s2[96 + lane], wx, wy, wz, gdt)));
	}
	vmax = __reduce_max_sync(0xffffffffu, vmax);
	if(lane == 0 && vmax) atomicMax(reinterpret_cast<unsigned*>(max_vel), vmax);
}
// the same with the analytic objects after the collider (objs.n >= 1)
template<bool COLLIDE>
__global__ void __launch_bounds__(256, 2) grid_max_objects_kernel(Cfg cfg, const StepState* state, const float* grid, const int* keys, float* max_vel, const ColliderView col, const __grid_constant__ ObjectList objs) {
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const int g = cfg.gsize, bc = cfg.boundary;
	const float gdt = cfg.gravity * state->dt;
	const ObjectFrames& of = object_frames_cta<COLLIDE>(col, objs, (float) state->sim_time);
	unsigned vmax = 0u;
	for(int b = blockIdx.x * 8 + warp; b < state->nbc; b += gridDim.x * 8) {
		const int kx = keys[3 * b], ky = keys[3 * b + 1], kz = keys[3 * b + 2];
		const bool wx = (kx < bc) | (kx >= g - bc), wy = (ky < bc) | (ky >= g - bc), wz = (kz < bc) | (kz >= g - bc);
		const float2* s2 = reinterpret_cast<const float2*>(grid + (size_t) b * kGridBlockFloats);
		vmax = max(vmax, __float_as_uint(cell_pair_vel_sq_objects<COLLIDE>(cfg, col, of, objs.n, s2, lane, kx, ky, kz, wx, wy, wz, gdt)));
	}
	vmax = __reduce_max_sync(0xffffffffu, vmax);
	if(lane == 0 && vmax) atomicMax(reinterpret_cast<unsigned*>(max_vel), vmax);
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
