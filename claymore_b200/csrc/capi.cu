// capi.cu -- kernel-level C ABI: one entry point per reference kernel on the hot path (see include/claymore_b200.h).
#include <cstdio>

#include "g2p2g.cuh"
#include "grid.cuh"
#include "init.cuh"
#include "partition.cuh"

using namespace cb200;

namespace cb200 {
// per-DEVICE caches: one process may drive several GPUs (MGSP worker threads, mgsp_benchmark.cuh:322-323)
constexpr int kMaxDevices = 64;
static int g_num_sms[kMaxDevices] = {};
static inline int current_device() {
	int dev = 0;
	cudaGetDevice(&dev);
	return (dev >= 0 && dev < kMaxDevices) ? dev : 0;
}
int num_sms() {
	const int dev = current_device();
	if(!g_num_sms[dev]) {
		int n = 0;
		cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
		g_num_sms[dev] = n > 0 ? n : 132;
	}
	return g_num_sms[dev];
}
static inline int grid_for(long long work_items, int per_block, int max_blocks_per_sm = 8) {
	long long b = (work_items + per_block - 1) / per_block;
	const long long cap = (long long) num_sms() * max_blocks_per_sm;
	if(b > cap) b = cap;
	if(b < 1) b = 1;
	return (int) b;
}

template<int MAT>
static int g2p2g_blocks_per_sm() {
	static int cache[kMaxDevices] = {};  // the shared-memory opt-in is per device (function attributes are per context)
	int& v = cache[current_device()];
	if(!v) {
		cudaFuncSetAttribute(g2p2g_kernel<MAT, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) sizeof(G2P2GSmem));
		cudaFuncSetAttribute(g2p2g_kernel<MAT, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) sizeof(G2P2GSmem));
		int u = 0;
		if(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&v, g2p2g_kernel<MAT, false>, kG2P2GThreads, sizeof(G2P2GSmem)) != cudaSuccess || v <= 0) v = 3;
		if(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&u, g2p2g_kernel<MAT, true>, kG2P2GThreads, sizeof(G2P2GSmem)) == cudaSuccess && u > 0 && u < v) v = u;
	}
	return v;
}
template<int MAT>
static void g2p2g_launch_one(const G2P2GArgs& a, bool sorted, int grid, cudaStream_t s) {
	if(sorted) g2p2g_kernel<MAT, true><<<grid, kG2P2GThreads, sizeof(G2P2GSmem), s>>>(a);
	else g2p2g_kernel<MAT, false><<<grid, kG2P2GThreads, sizeof(G2P2GSmem), s>>>(a);
}

// resolves occupancy / shared-memory attributes of every material up front (see preload_kernels in engine.cu)
void g2p2g_prepare_all() {
	g2p2g_blocks_per_sm<CB200_J_FLUID>();
	g2p2g_blocks_per_sm<CB200_FIXED_COROTATED>();
	g2p2g_blocks_per_sm<CB200_SAND>();
	g2p2g_blocks_per_sm<CB200_NACC>();
}

// launches the material-specialised kernel on a persistent grid (a multiple of the SM count)
cudaError_t launch_g2p2g(int material, const G2P2GArgs& a, int block_hint, cudaStream_t s) {
	int per_sm = 0;
	switch(material) {
		case CB200_J_FLUID: per_sm = g2p2g_blocks_per_sm<CB200_J_FLUID>(); break;
		case CB200_FIXED_COROTATED: per_sm = g2p2g_blocks_per_sm<CB200_FIXED_COROTATED>(); break;
		case CB200_SAND: per_sm = g2p2g_blocks_per_sm<CB200_SAND>(); break;
		case CB200_NACC: per_sm = g2p2g_blocks_per_sm<CB200_NACC>(); break;
		default: return cudaErrorInvalidValue;
	}
	int grid = num_sms() * per_sm;
	if(block_hint >= 0 && block_hint < grid) grid = block_hint;
	if(grid < 1) return cudaSuccess;
	bool sorted = a.n_models > 0;  // the cell-offset form needs the offsets of every model of the launch
	for(int m = 0; m < a.n_models; ++m) sorted &= a.m[m].next_offs != nullptr;
	switch(material) {
		case CB200_J_FLUID: g2p2g_launch_one<CB200_J_FLUID>(a, sorted, grid, s); break;
		case CB200_FIXED_COROTATED: g2p2g_launch_one<CB200_FIXED_COROTATED>(a, sorted, grid, s); break;
		case CB200_SAND: g2p2g_launch_one<CB200_SAND>(a, sorted, grid, s); break;
		case CB200_NACC: g2p2g_launch_one<CB200_NACC>(a, sorted, grid, s); break;
	}
	return cudaGetLastError();
}
}  // namespace cb200

#define CB_CFG(cfgptr)                                      \
	if(!(cfgptr) || !cfg_valid(*(cfgptr))) return (int) cudaErrorInvalidValue; \
	const Cfg cfg = make_cfg(*(cfgptr))

extern "C" {

const char* cb200_version(void) { return "claymore_b200 0.1 (sm_90a)"; }
const char* cb200_error_string(int err) { return err == CB200_ERROR_OUTPUT_IO ? "frame output: a file could not be opened or written" : cudaGetErrorString((cudaError_t) err); }

int cb200_g2p2g(const cb200_config* c, float dt, float new_dt, int pbc, cb200_particle_buffer cur, cb200_particle_buffer next, cb200_partition prev_partition, cb200_partition partition, const float* grid, float* next_grid, void* stream) {
	CB_CFG(c);
	if(cur.material != next.material) return (int) cudaErrorInvalidValue;
	G2P2GArgs a {};
	a.cfg = cfg;
	a.state = nullptr;
	a.dt = dt;
	a.new_dt = new_dt;
	a.block_count = pbc;
	a.n_models = 1;
	a.m[0].cur = view(cur);
	a.m[0].next = view(next);
	a.m[0].mat = mat_of(cur);
	a.m[0].next_offs = nullptr;  // the caller's bucket may be in any order (the reference's is atomics-dependent)
	a.prev_table = prev_partition.index_table;
	a.table = partition.index_table;
	a.keys = partition.active_keys;
	a.grid = grid;
	a.next_grid = next_grid;
	a.error = nullptr;
	a.work_counter = nullptr;
	return (int) launch_g2p2g(cur.material, a, pbc, (cudaStream_t) stream);
}

int cb200_update_grid_velocity_query_max(const cb200_config* c, int block_count, float* grid, cb200_partition partition, float dt, float* max_vel, void* stream) {
	CB_CFG(c);
	if(block_count <= 0) return 0;
	GridUpdateArgs a {};
	a.cfg = cfg;
	a.state = nullptr;
	a.nbc = block_count;
	a.ebc = 0;
	a.dt = dt;
	a.grid = grid;
	a.keys = partition.active_keys;
	a.max_vel = max_vel;
	a.clear_grid = nullptr;
	a.n_clear = 0;
	grid_update_kernel<false><<<grid_for(block_count, kGridThreads / 32), kGridThreads, 0, (cudaStream_t) stream>>>(a);
	return (int) cudaGetLastError();
}

int cb200_update_grid_velocity_query_max_collider(const cb200_config* c, int block_count, float* grid, cb200_partition partition, float dt, const cb200_collider* collider, float time, float* max_vel, void* stream) {
	CB_CFG(c);
	if(!collider_valid(collider) || !collider->sdf) return (int) cudaErrorInvalidValue;
	if(block_count <= 0) return 0;
	GridUpdateArgs a {};
	a.cfg = cfg;
	a.state = nullptr;
	a.nbc = block_count;
	a.ebc = 0;
	a.dt = dt;
	a.grid = grid;
	a.keys = partition.active_keys;
	a.max_vel = max_vel;
	a.clear_grid = nullptr;
	a.n_clear = 0;
	a.col = *collider;
	a.time = time;
	grid_update_kernel<true><<<grid_for(block_count, kGridThreads / 32), kGridThreads, 0, (cudaStream_t) stream>>>(a);
	return (int) cudaGetLastError();
}

int cb200_clear_grid(int block_count, float* grid, void* stream) {
	if(block_count <= 0) return 0;
	clear_grid_kernel<<<grid_for((long long) block_count * 64, 256), 256, 0, (cudaStream_t) stream>>>(block_count, grid);
	return (int) cudaGetLastError();
}

int cb200_cell_bucket_to_block(const cb200_config* c, int block_count, const int* cell_particle_counts, const int* cellbuckets, int* particle_bucket_sizes, int* buckets, void* stream) {
	CB_CFG(c);
	if(block_count <= 0) return 0;
	cell_bucket_to_block_kernel<<<grid_for(block_count, 1, 16), kBucketThreads, 0, (cudaStream_t) stream>>>(cfg, block_count, cell_particle_counts, cellbuckets, particle_bucket_sizes, buckets);
	return (int) cudaGetLastError();
}

int cb200_mark_active_grid_blocks(int block_count, const float* grid, int* marks, void* stream) {
	if(block_count <= 0) return 0;
	mark_active_grid_blocks_kernel<<<grid_for(block_count, 8), 256, 0, (cudaStream_t) stream>>>(block_count, grid, marks);
	return (int) cudaGetLastError();
}
int cb200_mark_active_particle_blocks(int block_count, const int* sizes, int* marks, void* stream) {
	if(block_count <= 0) return 0;
	mark_active_particle_blocks_kernel<<<grid_for(block_count, 256), 256, 0, (cudaStream_t) stream>>>(block_count, sizes, marks);
	return (int) cudaGetLastError();
}

int cb200_exclusive_scan(int count, const int* in, int* out, void* stream) {
	if(count <= 0) return 0;
	ScanArgs a {};
	a.count = count_imm(count);
	a.count_plus = 0;
	a.in = in;
	a.out = out;
	scan_kernel<<<1, 1024, 0, (cudaStream_t) stream>>>(a);
	return (int) cudaGetLastError();
}
int cb200_exclusive_scan_inverse(int count, const int* map, int* map_inv, void* stream) {
	if(count <= 0) return 0;
	scan_inverse_kernel<<<grid_for(count, 256), 256, 0, (cudaStream_t) stream>>>(count, map, map_inv);
	return (int) cudaGetLastError();
}

int cb200_update_partition(const cb200_config* c, int block_count, const int* source_nos, cb200_partition partition, cb200_partition next_partition, void* stream) {
	CB_CFG(c);
	if(block_count <= 0) return 0;
	update_partition_kernel<<<grid_for(block_count, 128), 128, 0, (cudaStream_t) stream>>>(cfg, block_count, source_nos, partition.active_keys, next_partition.active_keys, next_partition.index_table);
	return (int) cudaGetLastError();
}
int cb200_update_buckets(const cb200_config* c, int block_count, const int* source_nos, cb200_particle_buffer pb, cb200_particle_buffer next_pb, void* stream) {
	CB_CFG(c);
	if(block_count <= 0) return 0;
	update_buckets_kernel<<<grid_for(block_count, 1, 16), 128, 0, (cudaStream_t) stream>>>(cfg, block_count, source_nos, pb.particle_bucket_sizes, pb.blockbuckets, next_pb.particle_bucket_sizes, next_pb.blockbuckets);
	return (int) cudaGetLastError();
}
int cb200_compute_bin_capacity(int block_count, const int* sizes, int* bin_sizes, void* stream) {
	if(block_count <= 0) return 0;
	compute_bin_capacity_kernel<<<grid_for(block_count, 256), 256, 0, (cudaStream_t) stream>>>(block_count, sizes, bin_sizes);
	return (int) cudaGetLastError();
}

static int register_blocks(const cb200_config* c, int block_count, cb200_partition p, int lo, int span, void* stream) {
	CB_CFG(c);
	if(block_count <= 0) return 0;
	RegisterArgs a {};
	a.cfg = cfg;
	a.block_count = count_imm(block_count);
	a.table = p.index_table;
	a.keys = p.active_keys;
	a.count = p.count;
	a.capacity = 0x7fffffff;
	a.error = nullptr;
	a.lo = lo;
	a.span = span;
	register_blocks_kernel<<<grid_for((long long) block_count * span * span * span, 128), 128, 0, (cudaStream_t) stream>>>(a);
	return (int) cudaGetLastError();
}
int cb200_register_neighbor_blocks(const cb200_config* c, int block_count, cb200_partition p, void* stream) { return register_blocks(c, block_count, p, 0, 2, stream); }
int cb200_register_exterior_blocks(const cb200_config* c, int block_count, cb200_partition p, void* stream) { return register_blocks(c, block_count, p, -1, 3, stream); }

int cb200_copy_selected_grid_blocks(const cb200_config* c, int prev_block_count, const int* prev_blockids, cb200_partition partition, const int* marks, const float* prev_grid, float* grid, void* stream) {
	CB_CFG(c);
	if(prev_block_count <= 0) return 0;
	copy_selected_grid_blocks_kernel<<<grid_for(prev_block_count, 8), 256, 0, (cudaStream_t) stream>>>(cfg, prev_block_count, prev_blockids, partition.index_table, marks, prev_grid, grid);
	return (int) cudaGetLastError();
}

int cb200_reset_table(const cb200_config* c, cb200_partition partition, void* stream) {
	CB_CFG(c);
	const size_t n = (size_t) cfg.gsize * cfg.gsize * cfg.gsize;
	return (int) cudaMemsetAsync(partition.index_table, 0xff, n * sizeof(int), (cudaStream_t) stream);
}

int cb200_activate_blocks(const cb200_config* c, int n, const float* positions, cb200_partition p, void* stream) {
	CB_CFG(c);
	if(n <= 0) return 0;
	activate_blocks_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t) stream>>>(cfg, n, positions, p.index_table, p.active_keys, p.count, 0x7fffffff, nullptr);
	return (int) cudaGetLastError();
}
int cb200_build_particle_cell_buckets(const cb200_config* c, int n, const float* positions, cb200_particle_buffer pb, cb200_partition p, void* stream) {
	CB_CFG(c);
	if(n <= 0) return 0;
	build_particle_cell_buckets_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t) stream>>>(cfg, n, positions, view(pb), p.index_table, nullptr);
	return (int) cudaGetLastError();
}
int cb200_array_to_buffer(const cb200_config* c, int block_count, const float* positions, cb200_particle_buffer pb, void* stream) {
	CB_CFG(c);
	if(block_count <= 0) return 0;
	array_to_buffer_kernel<<<grid_for(block_count, 1, 16), 128, 0, (cudaStream_t) stream>>>(cfg, pb.material, block_count, positions, view(pb));
	return (int) cudaGetLastError();
}
int cb200_rasterize(const cb200_config* c, int n, const float* positions, float* grid, cb200_partition p, float mass, const float* v0, void* stream) {
	CB_CFG(c);
	if(n <= 0) return 0;
	rasterize_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t) stream>>>(cfg, n, positions, grid, p.index_table, mass, v0[0], v0[1], v0[2], nullptr);
	return (int) cudaGetLastError();
}
int cb200_init_adv_bucket(const cb200_config* c, int block_count, const int* sizes, int* buckets, void* stream) {
	CB_CFG(c);
	if(block_count <= 0) return 0;
	init_adv_bucket_kernel<<<grid_for(block_count, 1, 16), 128, 0, (cudaStream_t) stream>>>(cfg, block_count, sizes, buckets);
	return (int) cudaGetLastError();
}
int cb200_retrieve_particle_buffer(const cb200_config* c, int block_count, cb200_partition partition, cb200_partition prev_partition, cb200_particle_buffer pb, cb200_particle_buffer next_pb, float* out_positions, int* parcount, void* stream) {
	CB_CFG(c);
	if(block_count <= 0) return 0;
	retrieve_kernel<<<grid_for(block_count, 1, 16), 128, 0, (cudaStream_t) stream>>>(cfg, pb.material, count_imm(block_count), partition.active_keys, prev_partition.index_table, view(pb), view(next_pb), out_positions, 3, parcount);
	return (int) cudaGetLastError();
}

int cb200_mark_overlapping_blocks(const cb200_config* c, int block_count, int otherdid, const int* incoming, cb200_partition p, int* count, int* out_blockids, void* stream) {
	CB_CFG(c);
	if(block_count <= 0) return 0;
	mark_overlapping_blocks_kernel<<<grid_for(block_count, 128), 128, 0, (cudaStream_t) stream>>>(cfg, count_imm(block_count), otherdid, incoming, p.index_table, p.overlap_marks, count, out_blockids);
	return (int) cudaGetLastError();
}
int cb200_collect_blockids_for_halo_reduction(const cb200_config* c, int particle_block_count, cb200_partition p, void* stream) {
	CB_CFG(c);
	if(particle_block_count <= 0) return 0;
	collect_halo_blockids_kernel<<<grid_for(particle_block_count, 128), 128, 0, (cudaStream_t) stream>>>(cfg, count_imm(particle_block_count), p.index_table, p.active_keys, p.overlap_marks, p.halo_marks, p.halo_count, p.halo_blocks);
	return (int) cudaGetLastError();
}
int cb200_collect_grid_blocks(const cb200_config* c, int count, const int* blockids, const float* grid, cb200_partition p, float* halo_grid, void* stream) {
	CB_CFG(c);
	if(count <= 0) return 0;
	collect_grid_blocks_kernel<<<grid_for(count, 8), 256, 0, (cudaStream_t) stream>>>(cfg, count_imm(count), blockids, grid, p.index_table, halo_grid);
	return (int) cudaGetLastError();
}
int cb200_reduce_grid_blocks(const cb200_config* c, int count, const int* blockids, float* grid, cb200_partition p, const float* halo_grid, void* stream) {
	CB_CFG(c);
	if(count <= 0) return 0;
	reduce_grid_blocks_kernel<<<grid_for(count, 8), 256, 0, (cudaStream_t) stream>>>(cfg, count_imm(count), blockids, grid, p.index_table, halo_grid);
	return (int) cudaGetLastError();
}

}  // extern "C"

// ---- test-only hooks: the device math of g2p2g on caller-supplied vectors (tests/test_gpu_scale.py) ----------------------------
namespace cb200 {
__global__ void test_svd_kernel(int n, const float* F, float* U, float* S, float* V) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if(i >= n) return;
	float f[9], u[9], s[3], v[9];
	for(int k = 0; k < 9; ++k) f[k] = F[9 * i + k];
	svd3(f, u, s, v);
	for(int k = 0; k < 9; ++k) {
		U[9 * i + k] = u[k];
		V[9 * i + k] = v[k];
	}
	for(int k = 0; k < 3; ++k) S[3 * i + k] = s[k];
}
// mode 0: the path g2p2g takes (FIXED_COROTATED: Newton polar with SVD fall-back); mode 1: FIXED_COROTATED through the SVD
__global__ void test_stress_kernel(int material, int mode, Mat m, int n, const float* F_in, const float* log_jp_in, float* F_out, float* PF_out, float* log_jp_out) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if(i >= n) return;
	float f[9], pf[9];
	for(int k = 0; k < 9; ++k) f[k] = F_in[9 * i + k];
	float lj = log_jp_in ? log_jp_in[i] : 0.f;
	if(material == CB200_FIXED_COROTATED) {
		if(mode == 0) stress_fixed_corotated_polar(m, f, pf);
		else stress_fixed_corotated(m, f, pf);
	} else if(material == CB200_SAND) {
		stress_sand(m, f, pf, lj);
	} else {
		stress_nacc(m, f, pf, lj);
	}
	for(int k = 0; k < 9; ++k) {
		F_out[9 * i + k] = f[k];
		PF_out[9 * i + k] = pf[k];
	}
	if(log_jp_out) log_jp_out[i] = lj;
}
}  // namespace cb200

extern "C" {
int cb200_test_svd3(int n, const float* F, float* U, float* S, float* V, void* stream) {
	if(n <= 0) return 0;
	test_svd_kernel<<<(n + 127) / 128, 128, 0, (cudaStream_t) stream>>>(n, F, U, S, V);
	return (int) cudaGetLastError();
}
int cb200_test_stress(int material, int mode, cb200_particle_buffer params, int n, const float* F_in, const float* log_jp_in, float* F_out, float* PF_out, float* log_jp_out, void* stream) {
	if(n <= 0) return 0;
	if(material < CB200_FIXED_COROTATED || material > CB200_NACC) return (int) cudaErrorInvalidValue;
	test_stress_kernel<<<(n + 127) / 128, 128, 0, (cudaStream_t) stream>>>(material, mode, mat_of(params), n, F_in, log_jp_in, F_out, PF_out, log_jp_out);
	return (int) cudaGetLastError();
}
// ParticleBuffer<M> defaults (particle_buffer.cuh:141-264) as the step driver sets them (engine.cu)
void cb200_default_material(const cb200_config* cfg, int material, cb200_particle_buffer* out);
}
