// engine.cu -- the step driver: H100-native counterpart of GmpmSimulator (reference
// Projects/GMPM/gmpm_simulator.cuh:23-786) and of one MgspBenchmark device worker
// (Projects/MGSP/mgsp_benchmark.cuh:156-776).
//
// What differs from the reference driver, by design:
//   * block counts, bin counts, dt, max velocity and the frame clock live in a device-resident StepState; the
//     reference copies seven counters to the host and synchronises after each (gmpm_simulator.cuh:344,462,502,
//     517,541,564 + syncStream), here a sub-step is a fixed sequence of launches with no host round trip;
//   * that sequence is captured once per roll parity into a CUDA graph and replayed;
//   * every kernel runs on a persistent grid sized from the SM count and loops over device-read counts;
//   * clears, marks, bucket compaction and the grid carry are fused as described in partition.cuh / grid.cuh.
//   * per-frame .bgeo output: the body of each file is gathered on the device, a writer thread the simulator owns writes the files
//     while the next sub-steps run (the reference's IO thread, Library/MnSystem/IO/IO.h).
// The JSON scene loader lives in the Python host layer (claymore_b200/scene.py).
#include <fcntl.h>
#include <unistd.h>

#include <cerrno>
#include <condition_variable>
#include <cstdio>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "checkpoint.cuh"
#include "g2p2g.cuh"
#include "grid.cuh"
#include "init.cuh"
#include "mgsp.cuh"
#include "output.cuh"
#include "partition.cuh"

namespace cb200 {
int num_sms();
cudaError_t launch_g2p2g(int material, const G2P2GArgs& a, int block_hint, cudaStream_t s);
void g2p2g_prepare_all();
}  // namespace cb200
using namespace cb200;

#define CK(expr)                        \
	do {                                \
		const int _e = (int) (expr);    \
		if(_e != 0) return _e;          \
	} while(0)

namespace {
// Device-memory pool.  The reference frees and re-allocates its containers through raw cudaMalloc/cudaFree
// (GmpmSimulator::DeviceAllocator, gmpm_simulator.cuh:40-51); multi-GB cudaFree/cudaMalloc pairs cost tens to hundreds
// of milliseconds, so released blocks are kept (per device, exact size) and handed out again.  cb200_trim_pool() returns
// everything to the driver.  Buffers exposed through CUDA IPC are pooled as well: a re-used buffer has the same IPC handle, and
// the importing side keeps every mapping it has opened (IpcCache below), so a second simulator of a process costs neither a
// cudaMalloc nor a cudaIpcOpenMemHandle (they were ~0.4 s of the 8-rank end-to-end time in round 1).
class DevicePool {
public:
	cudaError_t alloc(void** p, size_t bytes) {
		int dev = 0;
		cudaGetDevice(&dev);
		{
			std::lock_guard<std::mutex> g(mu_);
			auto it = free_.find({dev, bytes});
			if(it != free_.end()) {
				*p = it->second;
				free_.erase(it);
				live_[*p] = {dev, bytes};
				return cudaSuccess;
			}
		}
		cudaError_t e = cudaMalloc(p, bytes);
		if(e == cudaErrorMemoryAllocation) {
			cudaGetLastError();
			trim();
			e = cudaMalloc(p, bytes);
		}
		if(e == cudaSuccess) {
			std::lock_guard<std::mutex> g(mu_);
			live_[*p] = {dev, bytes};
		}
		return e;
	}
	void release(void* p) {
		if(!p) return;
		std::lock_guard<std::mutex> g(mu_);
		auto it = live_.find(p);
		if(it == live_.end()) {
			cudaFree(p);
			return;
		}
		free_.emplace(it->second, p);
		live_.erase(it);
	}
	void trim() {
		std::lock_guard<std::mutex> g(mu_);
		for(auto& kv : free_) cudaFree(kv.second);
		free_.clear();
	}

private:
	std::mutex mu_;
	std::map<void*, std::pair<int, size_t>> live_;
	std::multimap<std::pair<int, size_t>, void*> free_;
};
DevicePool g_pool;

// mappings of peer buffers opened through CUDA IPC, kept for the life of the process (a handle can be opened once per process)
class IpcCache {
public:
	cudaError_t open(void** p, const cudaIpcMemHandle_t& h) {
		std::lock_guard<std::mutex> g(mu_);
		const std::string key(reinterpret_cast<const char*>(&h), sizeof(h));
		auto it = map_.find(key);
		if(it != map_.end()) {
			*p = it->second;
			return cudaSuccess;
		}
		const cudaError_t e = cudaIpcOpenMemHandle(p, h, cudaIpcMemLazyEnablePeerAccess);
		if(e == cudaSuccess) map_[key] = *p;
		return e;
	}

private:
	std::mutex mu_;
	std::map<std::string, void*> map_;
};
IpcCache g_ipc;

// pinned StepState mirrors are recycled: cudaMallocHost / cudaFreeHost are page-locking system calls (milliseconds), paid per
// simulator otherwise
class PinnedStates {
public:
	cudaError_t get(StepState** p) {
		{
			std::lock_guard<std::mutex> g(mu_);
			if(!free_.empty()) {
				*p = free_.back();
				free_.pop_back();
				return cudaSuccess;
			}
		}
		return cudaMallocHost(p, sizeof(StepState));
	}
	void put(StepState* p) {
		if(!p) return;
		std::lock_guard<std::mutex> g(mu_);
		free_.push_back(p);
	}

private:
	std::mutex mu_;
	std::vector<StepState*> free_;
};
PinnedStates g_pinned;
template<typename T>
cudaError_t pool_alloc(T** p, size_t bytes) { return g_pool.alloc(reinterpret_cast<void**>(p), bytes); }

struct Model {
	int material = 0;
	cb200_particle_buffer pb[2];
	long long bin_capacity = 0;
	float* d_pos = nullptr;
	int n = 0;
	float v0[3] = {0, 0, 0};
	int* bin_sizes = nullptr;
	unsigned short* celloffs[2] = {nullptr, nullptr};  // per buffer: start of every cell inside the (cell-major) block bucket, [blocks][64]
	// output staging (retrieve): device buffer + pinned host mirror, grown on demand, reused across frames
	float* d_out = nullptr;
	float* h_out = nullptr;
	size_t out_floats = 0;
};

void default_material(const cb200_config& cfg, int material, cb200_particle_buffer& pb) {
	// defaults of ParticleBuffer<M>, reference Projects/GMPM/particle_buffer.cuh:141-264
	const float cells = (float) (1u << cfg.domain_bits);
	const float E = 5e3f, nu = 0.4f;
	pb.material = material;
	pb.rho = 1e3f;
	pb.mass = 1e3f / cells / cells / cells / 8.f;
	pb.volume = ((material == CB200_FIXED_COROTATED || material == CB200_SAND) ? 10.f : 1.f) / cells / cells / cells / 8.f;
	pb.bulk = 4e4f;
	pb.gamma = 7.15f;
	pb.viscosity = 0.01f;
	pb.lambda = E * nu / ((1 + nu) * (1 - 2 * nu));
	pb.mu = E / (2 * (1 + nu));
	pb.cohesion = 0.f;
	pb.beta = material == CB200_NACC ? 0.5f : 1.f;
	pb.yield_surface = 0.816496580927726f * 2.f * 0.5f / (3.f - 0.5f);
	pb.volume_correction = 1;
	pb.bm = 2.f / 3.f * (E / (2 * (1 + nu))) + (E * nu / ((1 + nu) * (1 - 2 * nu)));
	pb.xi = 0.8f;
	pb.msqr = 3.423772074299613f;
	pb.hardening_on = 1;
}
}  // namespace

struct cb200_sim {
	cb200_sim_desc desc;
	Cfg cfg;
	cudaStream_t stream = nullptr;
	StepState* d_state = nullptr;
	StepState* h_state = nullptr;  // pinned
	cb200_partition part[2];
	float* grid[2] = {nullptr, nullptr};
	int* tile_sums = nullptr;     // [tiles + 1][kScanComps] of summary_kernel / rebuild_kernel
	int* block_totals = nullptr;  // [kMaxModels][max_blocks] particles per old block
	int* d_scratch = nullptr;  // [0] new_pbc, [1] new_nbc snapshot, [2] parcount
	std::vector<Model> models;
	int rollid = 0;
	long long launches = 0;
	long long launches_per_step = 0;
	cudaGraphExec_t graph[2] = {nullptr, nullptr};
	bool setup_done = false;
	size_t table_entries = 0;
	// MGSP
	int* peer_overlap_keys = nullptr;   // blockids of my blocks overlapping each peer: [world][max_blocks*3]
	int* peer_overlap_count = nullptr;  // [world]
	InboxLayout inbox_layout {};
	unsigned char* inbox_local = nullptr;
	unsigned char* inbox_peer[kMaxRanks] = {};
	bool peers_ready = false;
	int* peer_bno = nullptr;                 // [world][max_blocks]
	float* grid1_peer[kMaxRanks] = {};       // every rank's next grid mapped here (fused remote halo reduction)
	int* mgsp_done = nullptr;    // [4] last-CTA counters
	int* mgsp_epochs = nullptr;  // [3]
	// per-kernel timing (cudaEvent pairs around the g2p2g launches; stream mode only)
	bool profiling = false;
	std::vector<std::pair<cudaEvent_t, cudaEvent_t>> prof_events;
	size_t prof_used = 0;
	// phase marks (profiling mode only): one event after every phase of a sub-step
	std::vector<cudaEvent_t> phase_events;
	std::vector<int> phase_ids;
	size_t phase_used = 0;
	bool capturing = false;
	bool owns_stream = false;
	int frame_roll = 0;  // mirror of StepState::frame_roll
	// capacity polling (auto_grow): an asynchronous copy of the step state, looked at when it has arrived
	StepState* h_poll = nullptr;  // pinned
	cudaEvent_t poll_event = nullptr;
	bool poll_pending = false;
	int steps_since_poll = 15;  // the first sub-step polls
	int grow_events = 0;
	// signed-distance collider (cb200_sim_set_collider): parameters, and the device field this simulator owns
	bool has_collider = false;
	ColliderView collider {};
	float* sdf = nullptr;
	long long frames_done = 0;  // frames finished by cb200_sim_advance_frame (restored from a checkpoint)
	// checkpoint (cb200_sim_checkpoint_begin / _end): device staging blob, per-model scans of the bucket sizes, pinned copy of the
	// blob written on a stream of its own; allocated on first use, grown with the block capacity
	unsigned char* ck_dev = nullptr;
	size_t ck_dev_bytes = 0;
	int* ck_base = nullptr;  // [kMaxModels][max_blocks + 1]
	size_t ck_base_bytes = 0;
	unsigned char* ck_host = nullptr;  // pinned
	size_t ck_host_bytes = 0;
	cudaStream_t ck_stream = nullptr;
	cudaEvent_t ck_gathered = nullptr, ck_copied = nullptr;
	bool ck_pending = false;  // a copy was queued and end has not collected it
	bool ck_ready = false;    // ck_host holds a complete blob of ck_bytes
	size_t ck_bytes = 0;
	// cb200_sim_restore_models: the checkpoint's header and its state staged on the device, consumed by initial_setup
	bool restore_pending = false;
	cb200_checkpoint_info restore_info {};
	float* restore_state[kMaxModels] = {};
	unsigned char* restore_grid = nullptr;  // grid blocks, then keys
	// frame output (cb200_sim_frame_output): device staging of the records, its pinned copy (written on a stream of its own), and the
	// writer thread with its one job; allocated / started on first use.  `out_busy`: a frame is queued or being written
	unsigned char* out_dev = nullptr;
	size_t out_dev_bytes = 0;
	unsigned char* out_host = nullptr;  // pinned
	size_t out_host_bytes = 0;
	cudaStream_t out_stream = nullptr;
	cudaEvent_t out_copied = nullptr;
	std::thread out_thread;
	std::mutex out_mu;
	std::condition_variable out_cv;
	bool out_busy = false, out_quit = false;
	struct OutputFile {
		std::string path;
		std::vector<unsigned char> header;
		const unsigned char* body;
		size_t body_bytes;
	};
	std::vector<OutputFile> out_files;
	int out_errno = 0;  // first failure of a queued frame, until cb200_sim_frame_output_wait collects it
};

namespace {
int alloc_partition(cb200_sim* s, cb200_partition& p) {
	const size_t mb = (size_t) s->desc.max_blocks;
	CK(pool_alloc(&p.count, sizeof(int)));
	CK(pool_alloc(&p.index_table, s->table_entries * sizeof(int)));
	CK(pool_alloc(&p.active_keys, (mb + 1) * 3 * sizeof(int)));
	CK(pool_alloc(&p.halo_count, sizeof(int)));
	CK(pool_alloc(&p.halo_marks, mb + 1));
	CK(pool_alloc(&p.overlap_marks, (mb + 1) * sizeof(int)));
	p.halo_blocks = nullptr;
	CK(cudaMemsetAsync(p.count, 0, sizeof(int), s->stream));
	CK(cudaMemsetAsync(p.index_table, 0xff, s->table_entries * sizeof(int), s->stream));
	CK(cudaMemsetAsync(p.active_keys, 0, (mb + 1) * 3 * sizeof(int), s->stream));
	CK(cudaMemsetAsync(p.halo_count, 0, sizeof(int), s->stream));
	CK(cudaMemsetAsync(p.halo_marks, 0, mb + 1, s->stream));
	CK(cudaMemsetAsync(p.overlap_marks, 0, (mb + 1) * sizeof(int), s->stream));
	return 0;
}
void free_partition(cb200_partition& p) {
	g_pool.release(p.count);
	g_pool.release(p.index_table);
	g_pool.release(p.active_keys);
	g_pool.release(p.halo_count);
	g_pool.release(p.halo_marks);
	g_pool.release(p.overlap_marks);
}
inline int grid_blocks(int per_sm) { return num_sms() * per_sm; }

int pull_state(cb200_sim* s) {
	CK(cudaMemcpyAsync(s->h_state, s->d_state, sizeof(StepState), cudaMemcpyDeviceToHost, s->stream));
	CK(cudaStreamSynchronize(s->stream));
	return 0;
}
int push_state(cb200_sim* s) {
	CK(cudaMemcpyAsync(s->d_state, s->h_state, sizeof(StepState), cudaMemcpyHostToDevice, s->stream));
	return 0;
}

// one launch per material: all models of that material share the staged neighbourhood of a block
G2P2GArgs make_g2p2g_args(cb200_sim* s, int material, int R) {
	const int Rn = R ^ 1;
	G2P2GArgs a {};
	a.cfg = s->cfg;
	a.state = s->d_state;
	a.n_models = 0;
	for(const Model& m : s->models) {
		if(m.material != material) continue;
		G2P2GModel& gm = a.m[a.n_models++];
		gm.cur = view(m.pb[R]);
		gm.next = view(m.pb[Rn]);
		gm.mat = mat_of(m.pb[R]);
		gm.next_offs = m.celloffs[Rn];  // the buckets of the driver are cell-major: phase 2 takes its particle ranges from these offsets
	}
	a.prev_table = s->part[Rn].index_table;
	a.table = s->part[R].index_table;
	a.keys = s->part[R].active_keys;
	a.grid = s->grid[0];
	a.next_grid = s->grid[1];
	a.error = &s->d_state->error;
	// one queue per launch: each material's launch of a sub-step pulls from its own counter
	a.work_counter = &s->d_state->work_counter_mat[material];
	if(s->desc.mgsp_world > 1) {
		a.overlap_marks = s->part[R].overlap_marks;
		a.peer_bno = s->peer_bno;
		a.peer_stride = s->desc.max_blocks;
		for(int r = 0; r < s->desc.mgsp_world; ++r) a.peer_grid[r] = s->grid1_peer[r];
	}
	return a;
}

// ---- phase A: grid update (+ fused clears) -------------------------------------------------------
int enqueue_grid_update(cb200_sim* s, int R) {
	const int Rn = R ^ 1;
	GridUpdateArgs gu {};
	gu.cfg = s->cfg;
	gu.state = s->d_state;
	gu.grid = s->grid[0];
	gu.keys = s->part[R].active_keys;
	gu.max_vel = &s->d_state->max_vel_sq;
	gu.clear_grid = s->grid[1];
	if(s->desc.mgsp_world > 1) {
		// the global max |v|^2 was agreed on at the end of the previous sub-step (it rides on the key exchange) and the next grid
		// was cleared there as well, before the peers were told they may reduce into it
		gu.max_vel = reinterpret_cast<float*>(s->d_scratch + 5);
		gu.clear_grid = nullptr;
	}
	gu.n_clear = (int) s->models.size();
	for(size_t m = 0; m < s->models.size(); ++m) gu.clear_counts[m] = s->models[m].pb[Rn].cell_particle_counts;
	if(s->has_collider) {  // placed at StepState::sim_time, the start of this sub-step
		gu.col = s->collider;
		grid_update_kernel<true><<<grid_blocks(4), kGridThreads, 0, s->stream>>>(gu);
	} else {
		grid_update_kernel<false><<<grid_blocks(4), kGridThreads, 0, s->stream>>>(gu);
	}
	++s->launches;
	return (int) cudaGetLastError();
}
// ---- phase B: g2p2g --------------------------------------------------------------------------------
int enqueue_g2p2g(cb200_sim* s, int R) {
	cudaStream_t st = s->stream;
	for(int material = 0; material < 4; ++material) {
		const G2P2GArgs a = make_g2p2g_args(s, material, R);
		if(a.n_models == 0) continue;
		const bool timed = s->profiling && !s->capturing;
		if(timed) {
			if(s->prof_used == s->prof_events.size()) {
				cudaEvent_t e0, e1;
				CK(cudaEventCreate(&e0));
				CK(cudaEventCreate(&e1));
				s->prof_events.emplace_back(e0, e1);
			}
			CK(cudaEventRecord(s->prof_events[s->prof_used].first, st));
		}
		CK(launch_g2p2g(material, a, -1, st));
		if(timed) CK(cudaEventRecord(s->prof_events[s->prof_used++].second, st));
		++s->launches;
	}
	return 0;
}
// ---- phase C: partition / bucket rebuild -------------------------------------------------------------
int enqueue_rebuild(cb200_sim* s, int R) {
	const int Rn = R ^ 1;
	const int nm = (int) s->models.size();
	cudaStream_t st = s->stream;
	const int tiles = (s->desc.max_blocks + kRebuildTile - 1) / kRebuildTile;
	{
		SummaryArgs a {};
		a.cfg = s->cfg;
		a.state = s->d_state;
		a.n_models = nm;
		for(int m = 0; m < nm; ++m) {
			a.cell_counts[m] = s->models[m].pb[Rn].cell_particle_counts;
			a.bin_offsets[m] = s->models[m].pb[R].bin_offsets;
		}
		a.block_totals = s->block_totals;
		a.tile_sums = s->tile_sums;
		a.max_blocks = s->desc.max_blocks;
		a.stale_table = s->part[Rn].index_table;
		a.stale_keys = s->part[Rn].active_keys;
		a.stale_count = s->part[Rn].count;
		a.new_pbc = s->d_scratch + 0;
		summary_kernel<<<tiles, kSummaryThreads, 0, st>>>(a);
		++s->launches;
	}
	{
		RebuildArgs a {};
		a.cfg = s->cfg;
		a.state = s->d_state;
		a.n_models = nm;
		a.old_keys = s->part[R].active_keys;
		a.new_keys = s->part[Rn].active_keys;
		a.new_table = s->part[Rn].index_table;
		a.block_totals = s->block_totals;
		a.tile_sums = s->tile_sums;
		a.max_blocks = s->desc.max_blocks;
		for(int m = 0; m < nm; ++m) {
			a.cell_counts[m] = s->models[m].pb[Rn].cell_particle_counts;
			a.cellbuckets[m] = s->models[m].pb[Rn].cellbuckets;
			a.dst_sizes[m] = s->models[m].pb[R].particle_bucket_sizes;
			a.dst_buckets[m] = s->models[m].pb[R].blockbuckets;
			a.bin_offsets[m] = s->models[m].pb[R].bin_offsets;
			a.dst_offs[m] = s->models[m].celloffs[R];
		}
		rebuild_kernel<<<tiles, kRebuildThreads, 0, st>>>(a);
		++s->launches;
	}
	{
		RegisterArgs a {};
		a.cfg = s->cfg;
		a.block_count = count_dev(s->d_scratch + 0);
		a.table = s->part[Rn].index_table;
		a.keys = s->part[Rn].active_keys;
		a.count = s->part[Rn].count;
		a.capacity = s->desc.max_blocks;
		a.error = &s->d_state->error;
		a.lo = 0;
		a.span = 2;
		a.done_counter = &s->d_state->done_counter;  // the last CTA snapshots the neighbour count
		a.snapshot_out = s->d_scratch + 1;
		register_blocks_kernel<<<grid_blocks(4), 128, 0, st>>>(a);
		++s->launches;
	}
	return (int) cudaGetLastError();
}
int mark_phase(cb200_sim* s, int id);
MgspView mgsp_view(cb200_sim* s);

// End of a sub-step.  Single GPU: carry the grid, register exterior blocks (its last CTA rolls the state); the neighbour count
// was snapshotted by the last CTA of the neighbour registration.
// MGSP: the same, interleaved with the end-of-step exchange so that its wait sits behind local work:
//   reset tags -> carry (+ this rank's max |v|^2 of the new grid) -> clear the next grid -> PUBLISH keys + max
//   -> register exterior blocks -> WAIT for the peers' messages, tag overlaps, global max -> roll the state.
// A peer may reduce into this rank's next grid as soon as it has seen this rank's message: the clear comes before the publish.
int enqueue_carry_and_exterior(cb200_sim* s, int R) {
	const int Rn = R ^ 1;
	cudaStream_t st = s->stream;
	const bool mgsp = s->desc.mgsp_world > 1;
	float* local_max = reinterpret_cast<float*>(s->d_scratch + 3);
	float* global_max = reinterpret_cast<float*>(s->d_scratch + 4);
	{
		CarryArgs a {};
		if(mgsp) {  // behind the wait for the peers' "reductions landed" flags; resets the tagging state of the new partition on the way
			mgsp_done_wait_kernel<<<1, 32, 0, st>>>(mgsp_view(s));
			++s->launches;
			a.mgsp = 1;
			a.view = mgsp_view(s);
			a.overlap_marks = s->part[Rn].overlap_marks;
		}
		a.cfg = s->cfg;
		a.new_count = s->d_scratch + 1;
		a.new_keys = s->part[Rn].active_keys;
		a.old_table = s->part[R].index_table;
		a.state = s->d_state;
		a.old_grid = s->grid[1];
		a.new_grid = s->grid[0];
		a.next_max_vel = mgsp ? local_max : nullptr;
		if(mgsp && s->has_collider) {  // the predicted max must be the one the next grid update finds
			a.col = s->collider;
			carry_grid_kernel<true><<<grid_blocks(4), 256, 0, st>>>(a);
		} else {
			carry_grid_kernel<false><<<grid_blocks(4), 256, 0, st>>>(a);
		}
		++s->launches;
	}
	if(mgsp) {
		mgsp_clear_publish_kernel<<<grid_blocks(2), 256, 0, st>>>(mgsp_view(s), s->part[Rn].active_keys, s->d_scratch + 1, local_max, s->grid[1]);
		++s->launches;
	}
	FinalizeArgs fin {};
	fin.cfg = s->cfg;
	fin.state = s->d_state;
	fin.new_pbc = s->d_scratch + 0;
	fin.new_nbc = s->d_scratch + 1;
	fin.new_count = s->part[Rn].count;
	fin.max_blocks = s->desc.max_blocks;
	fin.n_models = (int) s->models.size();
	for(size_t m = 0; m < s->models.size(); ++m) fin.bin_capacity[m] = s->models[m].bin_capacity;
	fin.next_max_vel = mgsp ? global_max : nullptr;
	{
		RegisterArgs a {};
		a.cfg = s->cfg;
		a.block_count = count_dev(s->d_scratch + 0);
		a.table = s->part[Rn].index_table;
		a.keys = s->part[Rn].active_keys;
		a.count = s->part[Rn].count;
		a.capacity = s->desc.max_blocks;
		a.error = &s->d_state->error;
		a.lo = -1;
		a.span = 3;
		if(!mgsp) {  // the last CTA rolls the step state (MGSP: the tagging kernels come first)
			a.done_counter = &s->d_state->done_counter;
			a.do_finalize = 1;
			a.fin = fin;
		}
		register_blocks_kernel<<<grid_blocks(4), 128, 0, st>>>(a);
		++s->launches;
	}
	mark_phase(s, 9);
	if(mgsp) {
		mgsp_tag_kernel<<<grid_blocks(1), 256, 0, st>>>(s->cfg, mgsp_view(s), s->part[Rn].index_table, s->part[Rn].overlap_marks, s->d_scratch + 1, local_max, global_max, 1, fin);
		++s->launches;
		mark_phase(s, 8);
	}
	return (int) cudaGetLastError();
}

// ---- MGSP exchange phases ----------------------------------------------------------------------------------
MgspView mgsp_view(cb200_sim* s) {
	MgspView v {};
	v.L = s->inbox_layout;
	v.rank = s->desc.mgsp_rank;
	v.world = s->desc.mgsp_world;
	for(int r = 0; r < v.world; ++r) v.inbox[r] = s->inbox_peer[r];
	v.overlap_keys = s->peer_overlap_keys;
	v.overlap_count = s->peer_overlap_count;
	v.peer_bno = s->peer_bno;
	v.done = s->mgsp_done;
	v.epochs = s->mgsp_epochs;
	return v;
}

// profiling aid: records an event after a phase (ids: 0 start, 1 grid update, 5 g2p2g, 6 MGSP done publish, 7 rebuild,
// 9 carry + exterior registration (single GPU: + state roll), 8 MGSP halo tagging + state roll; ids 2-4 are not recorded)
int mark_phase(cb200_sim* s, int id) {
	if(!s->profiling || s->capturing) return 0;
	if(s->phase_used == s->phase_events.size()) {
		cudaEvent_t e;
		CK(cudaEventCreate(&e));
		s->phase_events.push_back(e);
		s->phase_ids.push_back(0);
	}
	s->phase_ids[s->phase_used] = id;
	CK(cudaEventRecord(s->phase_events[s->phase_used++], s->stream));
	return 0;
}

int enqueue_substep(cb200_sim* s, int R) {
	int e;
	mark_phase(s, 0);
	if((e = enqueue_grid_update(s, R))) return e;
	mark_phase(s, 1);
	// MGSP: no halo / interior split, one g2p2g launch per material as on one GPU: the arena flush of a block reduces into this rank's next grid and, for grid blocks
	// shared with a peer, straight into that peer's next grid over NVLink (no pack, no send, no unpack kernels; the reference:
	// halo g2p2g, barrier, collect_grid_blocks + cudaMemcpyPeerAsync, non-halo g2p2g, barrier, reduce_grid_blocks; :421-467,
	// 723-776).  The key exchange at the end of the previous sub-step doubles as "every rank has cleared its next grid"; the
	// done flag below as "every remote reduction has landed".
	if((e = enqueue_g2p2g(s, R))) return e;
	mark_phase(s, 5);
	if(s->desc.mgsp_world > 1) {
		mgsp_done_publish_kernel<<<1, 32, 0, s->stream>>>(mgsp_view(s));  // the wait sits at the head of the grid carry
		++s->launches;
		mark_phase(s, 6);
	}
	if((e = enqueue_rebuild(s, R))) return e;
	mark_phase(s, 7);
	return enqueue_carry_and_exterior(s, R);  // MGSP: includes the key / max-velocity exchange and the halo tagging (:530)
}
}  // namespace

namespace {
// CUDA loads kernels lazily on first launch and that load can synchronise the context.  A rank whose stream holds a
// kernel spinning on a peer's flag must therefore never be the one that still has to load a kernel: load all up front.
template<typename K>
void preload(K k) {
	cudaFuncAttributes a;
	(void) cudaFuncGetAttributes(&a, k);
}
void preload_kernels() {
	static bool done[64] = {};  // per device: modules are loaded per context
	int dev = 0;
	cudaGetDevice(&dev);
	if(dev < 0 || dev >= 64) dev = 0;
	if(done[dev]) return;
	done[dev] = true;
	preload(g2p2g_kernel<CB200_J_FLUID, false>);
	preload(g2p2g_kernel<CB200_FIXED_COROTATED, false>);
	preload(g2p2g_kernel<CB200_SAND, false>);
	preload(g2p2g_kernel<CB200_NACC, false>);
	preload(g2p2g_kernel<CB200_J_FLUID, true>);
	preload(g2p2g_kernel<CB200_FIXED_COROTATED, true>);
	preload(g2p2g_kernel<CB200_SAND, true>);
	preload(g2p2g_kernel<CB200_NACC, true>);
	preload(grid_update_kernel<false>);
	preload(grid_update_kernel<true>);
	preload(clear_grid_kernel);
	preload(carry_grid_kernel<false>);
	preload(carry_grid_kernel<true>);
	preload(scan_kernel);
	preload(summary_kernel);
	preload(rebuild_kernel);
	preload(register_blocks_kernel);
	preload(cell_bucket_to_block_kernel);
	preload(compute_bin_capacity_kernel);
	preload(activate_blocks_kernel<true>);
	preload(build_particle_cell_buckets_kernel<true>);
	preload(array_to_buffer_kernel);
	preload(rasterize_kernel);
	preload(rasterize_blocks_kernel);
	preload(init_adv_bucket_kernel);
	preload(retrieve_kernel);
	preload(collect_halo_blockids_kernel);
	preload(mgsp_allreduce_maxvel_kernel);
	preload(mgsp_pack_send_kernel);
	preload(mgsp_wait_reduce_kernel);
	preload(mgsp_tag_reset_kernel);
	preload(mgsp_tag_kernel);
	preload(mgsp_done_publish_kernel);
	preload(mgsp_done_wait_kernel);
	preload(mgsp_clear_publish_kernel);
	preload(grid_max_kernel<false>);
	preload(grid_max_kernel<true>);
	preload(snapshot_kernel);
	preload(state_positions_kernel);
	preload(state_to_bins_kernel);
	preload(scatter_grid_kernel);
	preload(output_kernel);
	g2p2g_prepare_all();
}
int ensure_graph(cb200_sim* s, int R) {
	if(s->graph[R]) return 0;
	const long long before = s->launches;
	cudaGraph_t g = nullptr;
	CK(cudaStreamBeginCapture(s->stream, cudaStreamCaptureModeThreadLocal));
	s->capturing = true;
	const int e = enqueue_substep(s, R);
	s->capturing = false;
	const cudaError_t ce = cudaStreamEndCapture(s->stream, &g);
	if(e) return e;
	CK(ce);
	CK(cudaGraphInstantiate(&s->graph[R], g, 0));
	cudaGraphDestroy(g);
	s->launches_per_step = s->launches - before;
	s->launches = before;
	return 0;
}
}  // namespace

namespace {
// Grows one block-indexed device array: allocate the larger one, copy the live prefix, initialise the tail the way
// cb200_sim_create / cb200_sim_init_model initialised it, release the old one.  One array at a time, so the peak is the
// footprint plus the largest array.
template<typename T>
int grow_array(cb200_sim* s, T*& p, size_t old_elems, size_t new_elems, int fill_byte) {
	T* q = nullptr;
	CK(pool_alloc(&q, new_elems * sizeof(T)));
	int e = 0;
	if(p && old_elems) e = (int) cudaMemcpyAsync(q, p, old_elems * sizeof(T), cudaMemcpyDeviceToDevice, s->stream);
	if(!e && new_elems > old_elems) e = (int) cudaMemsetAsync(q + old_elems, fill_byte, (new_elems - old_elems) * sizeof(T), s->stream);
	if(!e) e = (int) cudaStreamSynchronize(s->stream);
	if(e) {
		g_pool.release(q);
		return e;
	}
	g_pool.release(p);
	p = q;
	return 0;
}

// ---- frame output: the writer thread ------------------------------------------------------------------------------------------
// One file: header, body, trailer.  Returns 0 or the errno of the failing open / write / close; a partially written file is removed.
int write_bgeo(const cb200_sim::OutputFile& f) {
	const int fd = open(f.path.c_str(), O_WRONLY | O_CREAT | O_TRUNC | O_CLOEXEC, 0644);
	if(fd < 0) return errno;
	auto put = [fd](const unsigned char* p, size_t n) {
		while(n > 0) {
			const ssize_t w = write(fd, p, std::min<size_t>(n, (size_t) 1 << 30));
			if(w < 0) {
				if(errno == EINTR) continue;
				return errno;
			}
			p += w;
			n -= (size_t) w;
		}
		return 0;
	};
	int e = put(f.header.data(), f.header.size());
	if(!e) e = put(f.body, f.body_bytes);
	if(!e) e = put(kBgeoTrailer, sizeof(kBgeoTrailer));
	if(close(fd) != 0 && !e) e = errno;
	if(e) unlink(f.path.c_str());
	return e;
}
// Waits for the queued frame's copy, writes its files, records the first failure.  Ends when destroy asks it to and nothing is queued.
void output_writer(cb200_sim* s) {
	std::unique_lock<std::mutex> lk(s->out_mu);
	for(;;) {
		s->out_cv.wait(lk, [s] { return s->out_busy || s->out_quit; });
		if(!s->out_busy) return;
		std::vector<cb200_sim::OutputFile> files;
		files.swap(s->out_files);
		lk.unlock();
		const bool copied = cudaEventSynchronize(s->out_copied) == cudaSuccess;  // (failed: nothing of this frame is written)
		int e = copied ? 0 : EIO;
		for(size_t i = 0; copied && i < files.size(); ++i) {
			const int fe = write_bgeo(files[i]);
			if(fe && !e) e = fe;
		}
		lk.lock();
		if(e && !s->out_errno) s->out_errno = e;
		s->out_busy = false;
		s->out_cv.notify_all();
	}
}
// blocks until no frame is queued or being written
void output_idle(cb200_sim* s) {
	std::unique_lock<std::mutex> lk(s->out_mu);
	s->out_cv.wait(lk, [s] { return !s->out_busy; });
}
}  // namespace

extern "C" {

void cb200_default_material(const cb200_config* cfg, int material, cb200_particle_buffer* out) {
	if(!cfg || !out) return;
	memset(out, 0, sizeof(*out));
	default_material(*cfg, material, *out);
}

// In-place growth of the block capacity between sub-steps: what GmpmSimulator::check_capacity + the resize calls of main_loop do
// (gmpm_simulator.cuh:283-300, 371-376, 404-411, 528-548), except that every live array keeps its contents (the reference
// resizes the *next* buffers, whose contents are dead at that point of its loop; here the call may come at any sub-step
// boundary).  The sub-step graphs are re-captured on the next step.
// A failure part-way (out of memory) leaves a valid simulator at the old capacity: arrays already moved are merely larger.
int cb200_sim_reserve(cb200_sim* s, int new_max_blocks) {
	if(!s || new_max_blocks <= 0) return (int) cudaErrorInvalidValue;
	if(new_max_blocks <= s->desc.max_blocks) return 0;
	if(s->desc.mgsp_world > 1) return (int) cudaErrorNotSupported;  // the next grid / inbox are mapped into the peers (CUDA IPC)
	CK(cudaStreamSynchronize(s->stream));
	if(s->ck_pending) CK(cudaEventSynchronize(s->ck_copied));  // the next begin re-sizes the staging blob
	output_idle(s);
	const size_t ob = (size_t) s->desc.max_blocks, nb = (size_t) new_max_blocks;
	for(int i = 0; i < 2; ++i) {
		if(s->graph[i]) {
			cudaGraphExecDestroy(s->graph[i]);
			s->graph[i] = nullptr;
		}
		cb200_partition& p = s->part[i];
		CK(grow_array(s, p.active_keys, (ob + 1) * 3, (nb + 1) * 3, 0));
		CK(grow_array(s, p.halo_marks, ob + 1, nb + 1, 0));
		CK(grow_array(s, p.overlap_marks, ob + 1, nb + 1, 0));
		CK(grow_array(s, s->grid[i], (ob + 1) * kGridBlockFloats, (nb + 1) * kGridBlockFloats, 0));
	}
	{  // scratch of the rebuild: produced and consumed inside a sub-step, nothing to keep
		g_pool.release(s->tile_sums);
		g_pool.release(s->block_totals);
		s->tile_sums = nullptr;
		s->block_totals = nullptr;
		const size_t tiles = (nb + kRebuildTile - 1) / kRebuildTile + 1;
		CK(pool_alloc(&s->tile_sums, tiles * kScanComps * sizeof(int)));
		CK(pool_alloc(&s->block_totals, (size_t) kMaxModels * nb * sizeof(int)));
	}
	const size_t ppb = (size_t) s->cfg.ppb;
	for(Model& m : s->models) {
		const size_t binf = m.material == CB200_J_FLUID ? 128 : 512;
		const long long new_bins = (long long) m.n / kBinCap + (long long) nb;
		for(int i = 0; i < 2; ++i) {
			cb200_particle_buffer& pb = m.pb[i];
			CK(grow_array(s, pb.bins, (size_t) m.bin_capacity * binf, (size_t) new_bins * binf, 0));
			CK(grow_array(s, pb.cell_particle_counts, (ob + 1) * kBlockVol, (nb + 1) * kBlockVol, 0));
			CK(grow_array(s, pb.particle_bucket_sizes, ob + 2, nb + 2, 0));
			CK(grow_array(s, pb.cellbuckets, (ob + 1) * ppb, (nb + 1) * ppb, 0));
			CK(grow_array(s, pb.blockbuckets, (ob + 1) * ppb, (nb + 1) * ppb, 0));
			CK(grow_array(s, pb.bin_offsets, ob + 2, nb + 2, 0));
		}
		CK(grow_array(s, m.bin_sizes, ob + 2, nb + 2, 0));
		for(int i = 0; i < 2; ++i) CK(grow_array(s, m.celloffs[i], (ob + 1) * kBlockVol, (nb + 1) * kBlockVol, 0));
		m.bin_capacity = new_bins;
	}
	s->desc.max_blocks = new_max_blocks;
	++s->grow_events;
	return 0;
}

// check_capacity (gmpm_simulator.cuh:283-300): when the exterior block count exceeds 3/4 of the capacity, the capacity becomes
// 3/2 of it.  Bins need no rule of their own: their capacity is n/32 + max_blocks, an upper bound of the demand.
// *grown (nullable) receives the new capacity, or 0 when nothing changed.  Synchronises.
int cb200_sim_check_capacity(cb200_sim* s, int* grown) {
	if(grown) *grown = 0;
	if(!s || !s->setup_done) return (int) cudaErrorInvalidValue;
	CK(pull_state(s));
	const long long cap = s->desc.max_blocks;
	if((long long) s->h_state->ebc * 4 > cap * 3) {
		const long long want = cap * 3 / 2 + 1;
		CK(cb200_sim_reserve(s, (int) want));
		if(grown) *grown = (int) want;
	}
	return 0;
}
int cb200_sim_capacity(cb200_sim* s, int* max_blocks, int* grow_events) {
	if(!s) return (int) cudaErrorInvalidValue;
	if(max_blocks) *max_blocks = s->desc.max_blocks;
	if(grow_events) *grow_events = s->grow_events;
	return 0;
}

static int sim_create_impl(cb200_sim* s, const cb200_sim_desc* desc, void* stream);

int cb200_sim_create(const cb200_sim_desc* desc, void* stream, cb200_sim** out) {
	if(!desc || !out || !cfg_valid(desc->cfg) || desc->max_blocks <= 0) return (int) cudaErrorInvalidValue;
	preload_kernels();
	cb200_sim* s = new cb200_sim();
	const int e = sim_create_impl(s, desc, stream);
	if(e) {  // give back whatever was allocated before the failing call (every pointer of the struct starts out null)
		cb200_sim_destroy(s);
		return e;
	}
	*out = s;
	return 0;
}

static int sim_create_impl(cb200_sim* s, const cb200_sim_desc* desc, void* stream) {
	s->desc = *desc;
	if(s->desc.mgsp_world < 1) s->desc.mgsp_world = 1;
	s->cfg = make_cfg(desc->cfg);
	s->stream = (cudaStream_t) stream;
	if(!s->stream) {  // the legacy default stream cannot be captured into a graph: own a stream instead
		CK(cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking));
		s->owns_stream = true;
	}
	s->table_entries = (size_t) s->cfg.gsize * s->cfg.gsize * s->cfg.gsize;
	const size_t mb = (size_t) desc->max_blocks;
	CK(pool_alloc(&s->d_state, sizeof(StepState)));
	CK(cudaMemsetAsync(s->d_state, 0, sizeof(StepState), s->stream));
	CK(g_pinned.get(&s->h_state));
	memset(s->h_state, 0, sizeof(StepState));
	for(int i = 0; i < 2; ++i) {
		int e = alloc_partition(s, s->part[i]);
		if(e) return e;
		CK(pool_alloc(&s->grid[i], (mb + 1) * kGridBlockFloats * sizeof(float)));
		CK(cudaMemsetAsync(s->grid[i], 0, (mb + 1) * kGridBlockFloats * sizeof(float), s->stream));
	}
	{
		const size_t tiles = (mb + kRebuildTile - 1) / kRebuildTile + 1;
		CK(pool_alloc(&s->tile_sums, tiles * kScanComps * sizeof(int)));
		CK(pool_alloc(&s->block_totals, (size_t) kMaxModels * mb * sizeof(int)));
	}
	CK(pool_alloc(&s->d_scratch, 16 * sizeof(int)));
	CK(cudaMemsetAsync(s->d_scratch, 0, 16 * sizeof(int), s->stream));
	if(s->desc.mgsp_world > 1) {
		if(s->desc.mgsp_world > kMaxRanks || s->desc.mgsp_rank < 0 || s->desc.mgsp_rank >= s->desc.mgsp_world) return (int) cudaErrorInvalidValue;
		if(s->desc.mgsp_halo_cap <= 0) s->desc.mgsp_halo_cap = desc->max_blocks / 2;
		CK(pool_alloc(&s->peer_overlap_keys, (size_t) s->desc.mgsp_world * mb * 3 * sizeof(int)));
		CK(pool_alloc(&s->peer_overlap_count, (size_t) s->desc.mgsp_world * sizeof(int)));
		CK(cudaMemsetAsync(s->peer_overlap_count, 0, (size_t) s->desc.mgsp_world * sizeof(int), s->stream));
		s->inbox_layout = make_inbox_layout(s->desc.mgsp_world, s->desc.mgsp_halo_cap, desc->max_blocks);
		CK(pool_alloc(&s->inbox_local, inbox_bytes(s->inbox_layout)));
		CK(cudaMemsetAsync(s->inbox_local, 0, inbox_bytes(s->inbox_layout), s->stream));
		s->inbox_peer[s->desc.mgsp_rank] = s->inbox_local;
		s->grid1_peer[s->desc.mgsp_rank] = s->grid[1];
		CK(pool_alloc(&s->peer_bno, (size_t) s->desc.mgsp_world * mb * sizeof(int)));
		CK(cudaMemsetAsync(s->peer_bno, 0xff, (size_t) s->desc.mgsp_world * mb * sizeof(int), s->stream));
		CK(pool_alloc(&s->mgsp_done, 16 * sizeof(int)));
		CK(cudaMemsetAsync(s->mgsp_done, 0, 16 * sizeof(int), s->stream));
		s->mgsp_epochs = s->mgsp_done + 4;
		CK(cudaStreamSynchronize(s->stream));
	}
	return 0;
}

int cb200_sim_destroy(cb200_sim* s) {
	if(!s) return 0;
	cudaStreamSynchronize(s->stream);
	if(s->out_thread.joinable()) {  // the queued frame is written, then the writer ends: no thread outlives the simulator
		{
			std::lock_guard<std::mutex> g(s->out_mu);
			s->out_quit = true;
		}
		s->out_cv.notify_all();
		s->out_thread.join();
	}
	g_pool.release(s->out_dev);
	if(s->out_host) cudaFreeHost(s->out_host);
	if(s->out_copied) cudaEventDestroy(s->out_copied);
	if(s->out_stream) cudaStreamDestroy(s->out_stream);
	if(s->ck_stream) cudaStreamSynchronize(s->ck_stream);  // a checkpoint copy may still read the staging blob
	g_pool.release(s->ck_dev);
	g_pool.release(s->ck_base);
	for(float* p : s->restore_state) g_pool.release(p);
	g_pool.release(s->restore_grid);
	if(s->ck_host) cudaFreeHost(s->ck_host);
	if(s->ck_gathered) cudaEventDestroy(s->ck_gathered);
	if(s->ck_copied) cudaEventDestroy(s->ck_copied);
	if(s->ck_stream) cudaStreamDestroy(s->ck_stream);
	for(auto& ev : s->prof_events) {
		cudaEventDestroy(ev.first);
		cudaEventDestroy(ev.second);
	}
	for(int i = 0; i < 2; ++i) {
		if(s->graph[i]) cudaGraphExecDestroy(s->graph[i]);
		free_partition(s->part[i]);
		g_pool.release(s->grid[i]);
	}
	for(Model& m : s->models) {
		for(int i = 0; i < 2; ++i) {
			g_pool.release(m.pb[i].bins);
			g_pool.release(m.pb[i].cell_particle_counts);
			g_pool.release(m.pb[i].particle_bucket_sizes);
			g_pool.release(m.pb[i].cellbuckets);
			g_pool.release(m.pb[i].blockbuckets);
			g_pool.release(m.pb[i].bin_offsets);
		}
		g_pool.release(m.d_pos);
		g_pool.release(m.bin_sizes);
		g_pool.release(m.celloffs[0]);
		g_pool.release(m.celloffs[1]);
		g_pool.release(m.d_out);
		cudaFreeHost(m.h_out);
	}
	g_pool.release(s->tile_sums);
	g_pool.release(s->block_totals);
	g_pool.release(s->d_scratch);
	g_pool.release(s->d_state);
	g_pool.release(s->peer_overlap_keys);
	g_pool.release(s->peer_overlap_count);
	// peer mappings stay open (IpcCache): the exporting rank pools the buffer, the next simulator maps the same handle
	g_pool.release(s->peer_bno);
	g_pool.release(s->inbox_local);
	g_pool.release(s->mgsp_done);
	g_pool.release(s->sdf);
	g_pinned.put(s->h_state);
	g_pinned.put(s->h_poll);
	if(s->poll_event) cudaEventDestroy(s->poll_event);
	if(s->owns_stream) cudaStreamDestroy(s->stream);
	delete s;
	return 0;
}

// the containers of one model of m.material and m.n particles (init_model and restore; the caller fills d_pos)
static int alloc_model(cb200_sim* s, Model& m) {
	const int material = m.material, n = m.n;
	const size_t mb = (size_t) s->desc.max_blocks;
	const size_t binf = material == CB200_J_FLUID ? 128 : 512;
	// capacity rule of init_model (gmpm_simulator.cuh:173): n/32 bins + one partial bin per block
	m.bin_capacity = (long long) n / kBinCap + (long long) mb;
	for(int i = 0; i < 2; ++i) {
		cb200_particle_buffer& pb = m.pb[i];
		memset(&pb, 0, sizeof(pb));
		default_material(s->desc.cfg, material, pb);
		CK(pool_alloc(&pb.bins, (size_t) m.bin_capacity * binf * sizeof(float)));
		CK(pool_alloc(&pb.cell_particle_counts, (mb + 1) * kBlockVol * sizeof(int)));
		CK(pool_alloc(&pb.particle_bucket_sizes, (mb + 2) * sizeof(int)));
		CK(pool_alloc(&pb.cellbuckets, (mb + 1) * (size_t) s->cfg.ppb * sizeof(int)));
		CK(pool_alloc(&pb.blockbuckets, (mb + 1) * (size_t) s->cfg.ppb * sizeof(int)));
		CK(pool_alloc(&pb.bin_offsets, (mb + 2) * sizeof(int)));
		CK(cudaMemsetAsync(pb.cell_particle_counts, 0, (mb + 1) * kBlockVol * sizeof(int), s->stream));
		CK(cudaMemsetAsync(pb.particle_bucket_sizes, 0, (mb + 2) * sizeof(int), s->stream));
		CK(cudaMemsetAsync(pb.bin_offsets, 0, (mb + 2) * sizeof(int), s->stream));
	}
	CK(pool_alloc(&m.bin_sizes, (mb + 2) * sizeof(int)));
	CK(cudaMemsetAsync(m.bin_sizes, 0, (mb + 2) * sizeof(int), s->stream));
	for(int i = 0; i < 2; ++i) {
		CK(pool_alloc(&m.celloffs[i], (mb + 1) * kBlockVol * sizeof(unsigned short)));
		CK(cudaMemsetAsync(m.celloffs[i], 0, (mb + 1) * kBlockVol * sizeof(unsigned short), s->stream));
	}
	CK(pool_alloc(&m.d_pos, (size_t) n * 3 * sizeof(float)));
	return 0;
}

int cb200_sim_init_model(cb200_sim* s, int material, const float* positions_host, int n, const float* v0, int* model_id) {
	if(!s || s->setup_done || material < 0 || material > 3 || n <= 0 || (int) s->models.size() >= kMaxModels) return (int) cudaErrorInvalidValue;
	Model m;
	m.material = material;
	m.n = n;
	for(int d = 0; d < 3; ++d) m.v0[d] = v0 ? v0[d] : 0.f;
	CK(alloc_model(s, m));
	CK(cudaMemcpyAsync(m.d_pos, positions_host, (size_t) n * 3 * sizeof(float), cudaMemcpyHostToDevice, s->stream));
	CK(cudaStreamSynchronize(s->stream));
	if(model_id) *model_id = (int) s->models.size();
	s->models.push_back(m);
	return 0;
}

static int set_elastic(cb200_sim* s, int model, int material, float rho, float vol, float ym, float pr) {
	if(!s || model < 0 || model >= (int) s->models.size() || s->models[model].material != material) return (int) cudaErrorInvalidValue;
	for(int i = 0; i < 2; ++i) {
		cb200_particle_buffer& pb = s->models[model].pb[i];
		pb.rho = rho;
		pb.volume = vol;
		pb.mass = vol * rho;
		pb.lambda = ym * pr / ((1 + pr) * (1 - 2 * pr));
		pb.mu = ym / (2 * (1 + pr));
	}
	return 0;
}
// ParticleBuffer<FIXED_COROTATED>::update_parameters  particle_buffer.cuh:178-184
int cb200_sim_update_fr_parameters(cb200_sim* s, int model, float rho, float vol, float ym, float pr) { return set_elastic(s, model, CB200_FIXED_COROTATED, rho, vol, ym, pr); }
int cb200_sim_update_sand_parameters(cb200_sim* s, int model, float rho, float vol, float ym, float pr) { return set_elastic(s, model, CB200_SAND, rho, vol, ym, pr); }
// ParticleBuffer<J_FLUID>::update_parameters  particle_buffer.cuh:152-159
int cb200_sim_update_j_fluid_parameters(cb200_sim* s, int model, float rho, float vol, float bulk, float gamma, float visc) {
	if(!s || model < 0 || model >= (int) s->models.size() || s->models[model].material != CB200_J_FLUID) return (int) cudaErrorInvalidValue;
	for(int i = 0; i < 2; ++i) {
		cb200_particle_buffer& pb = s->models[model].pb[i];
		pb.rho = rho;
		pb.volume = vol;
		pb.mass = vol * rho;
		pb.bulk = bulk;
		pb.gamma = gamma;
		pb.viscosity = visc;
	}
	return 0;
}
// ParticleBuffer<NACC>::update_parameters  particle_buffer.cuh:250-259
int cb200_sim_update_nacc_parameters(cb200_sim* s, int model, float rho, float vol, float ym, float pr, float beta, float xi) {
	int e = set_elastic(s, model, CB200_NACC, rho, vol, ym, pr);
	if(e) return e;
	for(int i = 0; i < 2; ++i) {
		cb200_particle_buffer& pb = s->models[model].pb[i];
		pb.bm = 2.f / 3.f * (ym / (2 * (1 + pr))) + (ym * pr / ((1 + pr) * (1 - 2 * pr)));
		pb.beta = beta;
		pb.xi = xi;
	}
	return 0;
}

// What cb200_sim_restore puts in place of the rasterised start: the saved state, already on the device.
struct RestoreSrc {
	const cb200_checkpoint_info* info;
	const float* state[kMaxModels];  // [count][channels] per model
	const int* keys;                 // [nbc][3]
	const float* grid;               // [nbc][256]
};

// initial_setup  gmpm_simulator.cuh:637-781 (counts are read back here: one-time cost).  With `rs` (restore) it differs in three
// places: the bins get the saved channels, grid[0] gets the saved blocks (no MGSP halo reduction: they hold the full sums), and the
// step state gets the saved clock.
static int setup_impl(cb200_sim* s, const RestoreSrc* rs) {
	if(!s || s->setup_done || s->models.empty()) return (int) cudaErrorInvalidValue;
	cudaStream_t st = s->stream;
	const Cfg& cfg = s->cfg;
	const int R = s->rollid, Rn = R ^ 1;
	const int cap = s->desc.max_blocks;
	int* err = &s->d_state->error;
	int pbc = 0, nbc = 0, ebc = 0;
	auto blocks_for = [](long long n, int per) { return (int) std::max<long long>(1, std::min<long long>((n + per - 1) / per, (long long) num_sms() * 16)); };

	for(Model& m : s->models) {
		activate_blocks_kernel<true><<<blocks_for(m.n, 256), 256, 0, st>>>(cfg, m.n, m.d_pos, s->part[Rn].index_table, s->part[Rn].active_keys, s->part[Rn].count, cap, err);
		++s->launches;
	}
	CK(cudaMemcpyAsync(&pbc, s->part[Rn].count, sizeof(int), cudaMemcpyDeviceToHost, st));
	CK(cudaStreamSynchronize(st));
	if(pbc > cap) return (int) cudaErrorMemoryAllocation;
	for(Model& m : s->models) {
		build_particle_cell_buckets_kernel<true><<<blocks_for(m.n, 256), 256, 0, st>>>(cfg, m.n, m.d_pos, view(m.pb[R]), s->part[Rn].index_table, err);
		cell_bucket_to_block_kernel<<<blocks_for(pbc, 1), kBucketThreads, 0, st>>>(cfg, pbc, m.pb[R].cell_particle_counts, m.pb[R].cellbuckets, m.pb[R].particle_bucket_sizes, m.pb[R].blockbuckets, m.celloffs[Rn]);
		compute_bin_capacity_kernel<<<blocks_for(pbc + 1, 256), 256, 0, st>>>(pbc + 1, m.pb[R].particle_bucket_sizes, m.bin_sizes);
		ScanArgs a {};
		a.count = count_imm(pbc + 1);
		a.in = m.bin_sizes;
		a.out = m.pb[R].bin_offsets;
		scan_kernel<<<1, 1024, 0, st>>>(a);
		if(rs) state_to_bins_kernel<<<blocks_for(pbc, 1), 128, 0, st>>>(cfg, m.material, pbc, rs->state[&m - s->models.data()], view(m.pb[R]));
		else array_to_buffer_kernel<<<blocks_for(pbc, 1), 128, 0, st>>>(cfg, m.material, pbc, m.d_pos, view(m.pb[R]));
		s->launches += 5;
	}
	{
		RegisterArgs a {};
		a.cfg = cfg;
		a.block_count = count_imm(pbc);
		a.table = s->part[Rn].index_table;
		a.keys = s->part[Rn].active_keys;
		a.count = s->part[Rn].count;
		a.capacity = cap;
		a.error = err;
		a.lo = 0;
		a.span = 2;
		register_blocks_kernel<<<blocks_for((long long) pbc * 8, 128), 128, 0, st>>>(a);
		CK(cudaMemcpyAsync(&nbc, s->part[Rn].count, sizeof(int), cudaMemcpyDeviceToHost, st));
		CK(cudaStreamSynchronize(st));
		if(s->desc.mgsp_world > 1) {  // halo_tagging of the initial partition (mgsp_benchmark.cuh:633), with the kernels of the sub-step
			if(!s->peers_ready) return (int) cudaErrorNotReady;
			const MgspView v = mgsp_view(s);
			float* local_max = reinterpret_cast<float*>(s->d_scratch + 3);
			CK(cudaMemcpyAsync(s->d_scratch + 1, &nbc, sizeof(int), cudaMemcpyHostToDevice, st));  // key count of the exchange
			CK(cudaMemsetAsync(s->d_scratch + 3, 0, 2 * sizeof(int), st));
			mgsp_tag_reset_kernel<<<grid_blocks(1), 256, 0, st>>>(v, s->part[Rn].overlap_marks, s->d_scratch + 1);
			// the next grid is still all zero from cb200_sim_create: the clear changes nothing, and the flag still goes out behind it
			mgsp_clear_publish_kernel<<<grid_blocks(2), 256, 0, st>>>(v, s->part[Rn].active_keys, s->d_scratch + 1, local_max, s->grid[1]);
			mgsp_tag_kernel<<<grid_blocks(1), 256, 0, st>>>(cfg, v, s->part[Rn].index_table, s->part[Rn].overlap_marks, s->d_scratch + 1, local_max, reinterpret_cast<float*>(s->d_scratch + 4), 0, FinalizeArgs {});
			s->launches += 3;
		}
		a.lo = -1;
		a.span = 3;
		register_blocks_kernel<<<blocks_for((long long) pbc * 27, 128), 128, 0, st>>>(a);
		CK(cudaMemcpyAsync(&ebc, s->part[Rn].count, sizeof(int), cudaMemcpyDeviceToHost, st));
		CK(cudaStreamSynchronize(st));
		s->launches += 2;
	}
	if(nbc > cap || ebc > cap) return (int) cudaErrorMemoryAllocation;
	// background copies (gmpm_simulator.cuh:745-756); the device count is copied too so that the stale-key
	// un-insert of the first rebuild knows how many entries the table holds
	CK(cudaMemcpyAsync(s->part[R].index_table, s->part[Rn].index_table, s->table_entries * sizeof(int), cudaMemcpyDeviceToDevice, st));
	CK(cudaMemcpyAsync(s->part[R].active_keys, s->part[Rn].active_keys, (size_t) ebc * 3 * sizeof(int), cudaMemcpyDeviceToDevice, st));
	CK(cudaMemcpyAsync(s->part[R].count, s->part[Rn].count, sizeof(int), cudaMemcpyDeviceToDevice, st));
	if(s->desc.mgsp_world > 1)  // "need to copy halo tag info as well" (mgsp_benchmark.cuh:639-640)
		CK(cudaMemcpyAsync(s->part[R].overlap_marks, s->part[Rn].overlap_marks, (size_t) nbc * sizeof(int), cudaMemcpyDeviceToDevice, st));
	for(Model& m : s->models) {
		CK(cudaMemcpyAsync(m.pb[Rn].bin_offsets, m.pb[R].bin_offsets, (size_t) (pbc + 1) * sizeof(int), cudaMemcpyDeviceToDevice, st));
		CK(cudaMemcpyAsync(m.pb[Rn].particle_bucket_sizes, m.pb[R].particle_bucket_sizes, (size_t) pbc * sizeof(int), cudaMemcpyDeviceToDevice, st));
	}
	clear_grid_kernel<<<blocks_for((long long) nbc * 64, 256), 256, 0, st>>>(nbc, s->grid[0]);
	++s->launches;
	int* missing = s->d_scratch + 6;
	if(rs) {  // the saved blocks by key; a key the rebuilt partition has no neighbour block for is counted, not written
		const int saved = rs->info->neighbor_block_count;
		CK(cudaMemsetAsync(missing, 0, sizeof(int), st));
		scatter_grid_kernel<<<blocks_for(saved, 8), 256, 0, st>>>(cfg, saved, rs->keys, rs->grid, s->part[R].index_table, nbc, s->grid[0], missing);
		++s->launches;
	}
	for(Model& m : s->models) {
		if(!rs) {
			rasterize_blocks_kernel<<<blocks_for(pbc, 1), 256, 0, st>>>(cfg, m.material, pbc, s->part[R].active_keys, s->part[R].index_table, view(m.pb[R]), s->grid[0], m.pb[R].mass, m.v0[0], m.v0[1], m.v0[2], err);
			++s->launches;
		}
		init_adv_bucket_kernel<<<blocks_for(pbc, 1), 128, 0, st>>>(cfg, pbc, m.pb[Rn].particle_bucket_sizes, m.pb[Rn].blockbuckets);
		++s->launches;
	}
	CK(cudaGetLastError());
	if(rs) {  // a blob that passed inspect but does not rebuild the saved partition (hand-edited): nothing to step
		int miss = 0;
		CK(cudaMemcpyAsync(&miss, missing, sizeof(int), cudaMemcpyDeviceToHost, st));
		CK(cudaStreamSynchronize(st));
		const cb200_checkpoint_info& I = *rs->info;
		if(miss || pbc != I.particle_block_count || nbc != I.neighbor_block_count || ebc != I.exterior_block_count) return (int) cudaErrorIllegalState;
	}
	if(s->desc.mgsp_world > 1 && !rs) {  // the rasterised halo blocks are partial sums: reduce them (mgsp_benchmark.cuh:653-654, 723-776)
		mgsp_pack_send_kernel<<<grid_blocks(2), 256, 0, st>>>(cfg, mgsp_view(s), s->grid[0], s->part[R].index_table);
		mgsp_wait_reduce_kernel<<<grid_blocks(2), 256, 0, st>>>(cfg, mgsp_view(s), s->grid[0], s->part[R].index_table, err);
		s->launches += 2;
		CK(cudaGetLastError());
	}
	// device-resident step state; initial dt as in main_loop's preamble (gmpm_simulator.cuh:305-315)
	CK(pull_state(s));
	StepState& h = *s->h_state;
	h.pbc = pbc;
	h.nbc = nbc;
	h.ebc = ebc;
	h.prev_nbc = nbc;
	h.prev_ebc = ebc;
	h.dt_default = s->desc.dt_default;
	h.frame_time = s->desc.fps > 0 ? 1.f / (float) s->desc.fps : 0.f;
	h.step_time = 0.f;
	h.sim_time = 0.0;
	if(rs) {
		const cb200_checkpoint_info& I = *rs->info;
		h.frame_time = I.frame_time;
		h.step_time = I.step_time;
		h.sim_time = I.sim_time;
		h.dt = I.dt;
		h.next_dt = I.next_dt;
		h.steps = I.steps;
		h.error |= I.error;
		h.max_vel_sq = 0.f;
		s->frames_done = I.frames;
		CK(push_state(s));
	}
	float mv = 0.f;
	for(const Model& m : s->models) mv = fmaxf(mv, sqrtf(m.v0[0] * m.v0[0] + m.v0[1] * m.v0[1] + m.v0[2] * m.v0[2]));
	if(s->desc.mgsp_world > 1 && !rs) {  // every rank must start from the same dt: max over the ranks' initial speeds
		h.max_vel_sq = mv * mv;
		CK(push_state(s));
		mgsp_allreduce_maxvel_kernel<<<1, 32, 0, st>>>(mgsp_view(s), &s->d_state->max_vel_sq);
		++s->launches;
		CK(pull_state(s));
		mv = sqrtf(s->h_state->max_vel_sq);
	}
	if(!rs) {
		float dt = h.dt_default;
		if(mv > 0.f) dt = fminf(dt, cfg.dx * cfg.cfl / mv);
		if(h.frame_time > 0.f) dt = fminf(dt, h.frame_time);
		h.dt = dt;
		h.next_dt = dt;
		h.max_vel_sq = 0.f;
		CK(push_state(s));
	}
	if(s->desc.mgsp_world > 1) {
		// global max |v|^2 of the start grid (later sub-steps get it from the end-of-step exchange of the previous one)
		if(s->has_collider) grid_max_kernel<true><<<grid_blocks(2), 256, 0, st>>>(cfg, s->d_state, s->grid[0], s->part[R].active_keys, &s->d_state->max_vel_sq, s->collider);
		else grid_max_kernel<false><<<grid_blocks(2), 256, 0, st>>>(cfg, s->d_state, s->grid[0], s->part[R].active_keys, &s->d_state->max_vel_sq, ColliderView {});
		mgsp_allreduce_maxvel_kernel<<<1, 32, 0, st>>>(mgsp_view(s), &s->d_state->max_vel_sq);
		s->launches += 2;
	}
	CK(cudaStreamSynchronize(st));
	if(s->desc.use_graph) {  // instantiate both roll parities now: never later, while a peer may be waiting on this rank
		CK(ensure_graph(s, 0));
		CK(ensure_graph(s, 1));
	}
	s->setup_done = true;
	return 0;
}
int cb200_sim_initial_setup(cb200_sim* s) {
	if(!s || !s->restore_pending) return setup_impl(s, nullptr);
	RestoreSrc rs {};
	rs.info = &s->restore_info;
	for(int m = 0; m < kMaxModels; ++m) rs.state[m] = s->restore_state[m];
	rs.grid = reinterpret_cast<const float*>(s->restore_grid);
	rs.keys = reinterpret_cast<const int*>(s->restore_grid + s->restore_info.grid_bytes);
	int e = setup_impl(s, &rs);
	if(!e) e = (int) cudaStreamSynchronize(s->stream);
	if(!e) {  // the staged state is in the bins and the grid now
		for(float*& p : s->restore_state) {
			g_pool.release(p);
			p = nullptr;
		}
		g_pool.release(s->restore_grid);
		s->restore_grid = nullptr;
		s->restore_pending = false;
	}
	return e;
}

static int set_frame_roll(cb200_sim* s, int on) {
	if(s->frame_roll == on) return 0;
	static const int kVals[2] = {0, 1};
	s->frame_roll = on;
	return (int) cudaMemcpyAsync(&s->d_state->frame_roll, &kVals[on], sizeof(int), cudaMemcpyHostToDevice, s->stream);
}
static int step_impl(cb200_sim* s, int n);

// With fps > 0 the frame clock restarts on the device whenever a frame is complete (the reference's outer frame loop), so
// stepping past a frame boundary never leaves dt at 0.
int cb200_sim_step(cb200_sim* s, int n) {
	if(!s || !s->setup_done) return (int) cudaErrorInvalidValue;
	CK(set_frame_roll(s, s->desc.fps > 0 ? 1 : 0));
	return step_impl(s, n);
}
// auto_grow: every 16 sub-steps an asynchronous copy of the step state is queued; once it has arrived (no host wait) the
// reference's 3/4 rule is applied to it.  The capacity check therefore lags the simulation by at most 32 sub-steps, against
// a head-room of 25 % of the capacity.
static int poll_capacity(cb200_sim* s) {
	if(s->poll_pending && cudaEventQuery(s->poll_event) == cudaSuccess) {
		s->poll_pending = false;
		if((long long) s->h_poll->ebc * 4 > (long long) s->desc.max_blocks * 3 && s->desc.mgsp_world <= 1) CK(cb200_sim_reserve(s, (int) ((long long) s->desc.max_blocks * 3 / 2 + 1)));
	}
	if(!s->poll_pending && ++s->steps_since_poll >= 16) {
		s->steps_since_poll = 0;
		if(!s->h_poll) {
			CK(g_pinned.get(&s->h_poll));
			CK(cudaEventCreateWithFlags(&s->poll_event, cudaEventDisableTiming));
		}
		CK(cudaMemcpyAsync(s->h_poll, s->d_state, sizeof(StepState), cudaMemcpyDeviceToHost, s->stream));
		CK(cudaEventRecord(s->poll_event, s->stream));
		s->poll_pending = true;
	}
	return 0;
}
static int step_impl(cb200_sim* s, int n) {
	for(int i = 0; i < n; ++i) {
		if(s->desc.auto_grow) CK(poll_capacity(s));
		const int R = s->rollid;
		if(s->desc.use_graph && !s->profiling) {
			CK(ensure_graph(s, R));
			CK(cudaGraphLaunch(s->graph[R], s->stream));
			s->launches += s->launches_per_step;
		} else {
			const int e = enqueue_substep(s, R);
			if(e) return e;
		}
		s->rollid ^= 1;
	}
	return 0;
}

// main_loop's inner for-loop (gmpm_simulator.cuh:324): sub-steps until step_time reaches the frame time.
// dt never exceeds dt_default, so ceil(remaining / dt_default) sub-steps can be queued before the host
// looks at the device clock again.
int cb200_sim_advance_frame(cb200_sim* s, int* steps_taken) {
	if(!s || !s->setup_done || s->desc.fps <= 0) return (int) cudaErrorInvalidValue;
	int taken = 0;
	CK(set_frame_roll(s, 0));  // this loop owns the frame clock
	CK(pull_state(s));
	// the reference restarts current_step_time at 0 for every frame
	s->h_state->step_time = 0.f;
	CK(cudaMemcpyAsync(&s->d_state->step_time, &s->h_state->step_time, sizeof(float), cudaMemcpyHostToDevice, s->stream));
	const float frame = s->h_state->frame_time;
	for(;;) {
		CK(pull_state(s));
		if(s->h_state->error) break;
		const float left = frame - s->h_state->step_time;
		if(!(left > 0.f)) break;
		// dt never exceeds dt_default and the device clamps it to the time left, so floor(left / dt_default) sub-steps can
		// be queued without looking at the device clock in between (one host sync per batch, none per sub-step)
		int batch = (int) floorf(left / s->h_state->dt_default);
		if(batch < 1) batch = 1;
		if(batch > 4096) batch = 4096;
		const int e = step_impl(s, batch);
		if(e) return e;
		taken += batch;
	}
	++s->frames_done;
	if(steps_taken) *steps_taken = taken;
	return 0;
}

int cb200_sim_sync(cb200_sim* s) {
	if(!s) return (int) cudaErrorInvalidValue;
	return (int) cudaStreamSynchronize(s->stream);
}

int cb200_sim_stats_get(cb200_sim* s, cb200_sim_stats* out) {
	if(!s || !out) return (int) cudaErrorInvalidValue;
	CK(pull_state(s));
	const StepState& h = *s->h_state;
	out->particle_block_count = h.pbc;
	out->neighbor_block_count = h.nbc;
	out->exterior_block_count = h.ebc;
	for(int m = 0; m < 8; ++m) out->bin_count[m] = h.bin_count[m];
	out->dt = h.dt;
	out->next_dt = h.next_dt;
	out->max_vel = sqrtf(h.max_vel_sq);
	out->step_time = h.step_time;
	out->error = h.error;
	out->steps = h.steps;
	return 0;
}

// output_model (gmpm_simulator.cuh:594-634): particles -> flat array -> host.  The staging buffers persist (the reference borrows
// and re-allocates per frame) and the device->host copy lands in pinned memory; `host` == nullptr returns the pinned mirror itself.
static int retrieve_impl(cb200_sim* s, int model, float* host, int nch, int* n_out, const float** pinned_out) {
	if(!s || !s->setup_done || model < 0 || model >= (int) s->models.size()) return (int) cudaErrorInvalidValue;
	Model& m = s->models[model];
	const int R = s->rollid, Rn = R ^ 1;
	const size_t need = (size_t) m.n * nch;
	if(m.out_floats < need) {
		g_pool.release(m.d_out);
		cudaFreeHost(m.h_out);
		m.d_out = nullptr;
		m.h_out = nullptr;
		CK(pool_alloc(&m.d_out, need * sizeof(float)));
		m.out_floats = need;
	}
	if(!host && !m.h_out) CK(cudaMallocHost(&m.h_out, m.out_floats * sizeof(float)));
	float* dst = host ? host : m.h_out;  // caller memory (fast when it is pinned) or the simulator's pinned mirror
	CK(cudaMemsetAsync(s->d_scratch + 2, 0, sizeof(int), s->stream));
	retrieve_kernel<<<num_sms() * 8, 128, 0, s->stream>>>(s->cfg, m.material, count_dev(&s->d_state->pbc), s->part[R].active_keys, s->part[Rn].index_table, view(m.pb[R]), view(m.pb[Rn]), m.d_out, nch, s->d_scratch + 2);
	++s->launches;
	// the count is only known on the device: copy the full staging buffer behind the kernel, read the count with it
	CK(cudaMemcpyAsync(dst, m.d_out, need * sizeof(float), cudaMemcpyDeviceToHost, s->stream));
	int n = 0;
	CK(cudaMemcpyAsync(&n, s->d_scratch + 2, sizeof(int), cudaMemcpyDeviceToHost, s->stream));
	CK(cudaStreamSynchronize(s->stream));
	if(n > m.n) n = m.n;
	if(pinned_out) *pinned_out = m.h_out;
	if(n_out) *n_out = n;
	return 0;
}
int cb200_sim_retrieve(cb200_sim* s, int model, float* positions_host, int* n_out) { return retrieve_impl(s, model, positions_host, 3, n_out, nullptr); }
// zero-copy variant: *positions_pinned points at the simulator's pinned staging buffer (valid until the next retrieve of that model)
int cb200_sim_retrieve_pinned(cb200_sim* s, int model, const float** positions_pinned, int* n_out) { return retrieve_impl(s, model, nullptr, 3, n_out, positions_pinned); }
int cb200_sim_particle_state(cb200_sim* s, int model, float* state_host, int* n_out) {
	if(!s || model < 0 || model >= (int) s->models.size()) return (int) cudaErrorInvalidValue;
	const int mat = s->models[model].material;
	return retrieve_impl(s, model, state_host, mat == CB200_J_FLUID ? 4 : (mat == CB200_FIXED_COROTATED ? 12 : 13), n_out, nullptr);
}

int cb200_sim_active_keys(cb200_sim* s, int* keys_host, int capacity_blocks, int* n_out) {
	if(!s || !s->setup_done) return (int) cudaErrorInvalidValue;
	CK(pull_state(s));
	const int n = std::min(s->h_state->ebc, capacity_blocks);
	CK(cudaMemcpy(keys_host, s->part[s->rollid].active_keys, (size_t) n * 3 * sizeof(int), cudaMemcpyDeviceToHost));
	if(n_out) *n_out = n;
	return 0;
}
int cb200_sim_grid(cb200_sim* s, float* grid_host, int capacity_blocks, int* n_out) {
	if(!s || !s->setup_done) return (int) cudaErrorInvalidValue;
	CK(pull_state(s));
	const int n = std::min(s->h_state->nbc, capacity_blocks);
	CK(cudaMemcpy(grid_host, s->grid[0], (size_t) n * kGridBlockFloats * sizeof(float), cudaMemcpyDeviceToHost));
	if(n_out) *n_out = n;
	return 0;
}
long long cb200_sim_launch_count(cb200_sim* s) { return s ? s->launches : 0; }

// The sub-step graphs hold the grid-update and carry launches of the collider state they were captured with: drop them and,
// once set up, instantiate both roll parities again right away (never later, while an MGSP peer may be waiting on this rank).
static int recapture(cb200_sim* s) {
	for(int i = 0; i < 2; ++i) {
		if(s->graph[i]) cudaGraphExecDestroy(s->graph[i]);
		s->graph[i] = nullptr;
	}
	if(s->setup_done && s->desc.use_graph) {
		CK(ensure_graph(s, 0));
		CK(ensure_graph(s, 1));
	}
	return 0;
}
// init_boundary (mgsp_benchmark.cuh:257-266) + fill_signed_distance_field (boundary_condition.cuh:253-295): the four dense
// row-major node arrays are re-laid out into 1 KiB blocks on the host and uploaded into a pooled device field.
int cb200_sim_set_collider(cb200_sim* s, const cb200_collider* params, const float* sdf_host) {
	if(!s || !collider_valid(params) || (!sdf_host && !s->sdf)) return (int) cudaErrorInvalidValue;
	CK(cudaStreamSynchronize(s->stream));
	if(sdf_host) {
		const int G = s->cfg.gsize, N = 4 * G;
		const size_t blocks = (size_t) G * G * G, nodes = (size_t) N * N * N;
		if(!s->sdf) CK(pool_alloc(&s->sdf, blocks * kGridBlockFloats * sizeof(float)));
		std::vector<float> f(blocks * kGridBlockFloats);
		for(int ch = 0; ch < 4; ++ch)
			for(int i = 0; i < N; ++i)
				for(int j = 0; j < N; ++j)
					for(int k = 0; k < N; ++k)
						f[(((size_t) (i >> 2) * G + (j >> 2)) * G + (k >> 2)) * kGridBlockFloats + ch * 64 + (i & 3) * 16 + (j & 3) * 4 + (k & 3)] = sdf_host[ch * nodes + ((size_t) i * N + j) * N + k];
		CK(cudaMemcpyAsync(s->sdf, f.data(), f.size() * sizeof(float), cudaMemcpyHostToDevice, s->stream));
		CK(cudaStreamSynchronize(s->stream));
	}
	s->collider = *params;
	s->collider.sdf = s->sdf;
	s->has_collider = true;
	return recapture(s);
}
int cb200_sim_clear_collider(cb200_sim* s) {
	if(!s) return (int) cudaErrorInvalidValue;
	CK(cudaStreamSynchronize(s->stream));
	s->has_collider = false;
	s->collider = ColliderView {};
	g_pool.release(s->sdf);
	s->sdf = nullptr;
	return recapture(s);
}
int cb200_sim_time(cb200_sim* s, double* time) {
	if(!s || !time) return (int) cudaErrorInvalidValue;
	CK(pull_state(s));
	*time = s->h_state->sim_time;
	return 0;
}
// ---- checkpoint / restore (format and kernels: checkpoint.cuh) ---------------------------------------------------------------
int cb200_checkpoint_inspect(const void* blob, size_t bytes, cb200_checkpoint_info* info) { return ck_parse(blob, bytes, info); }

}  // extern "C"
namespace {
size_t ck_capacity(const cb200_sim* s) {
	int mats[kMaxModels];
	long long counts[kMaxModels];
	for(size_t m = 0; m < s->models.size(); ++m) {
		mats[m] = s->models[m].material;
		counts[m] = s->models[m].n;
	}
	return (size_t) ck_layout((int) s->models.size(), mats, counts, s->desc.max_blocks).total;
}
// grows a checkpoint buffer to `need` bytes (contents are not kept)
template<typename T>
int ck_grow(T*& p, size_t& have, size_t need) {
	if(have >= need) return 0;
	g_pool.release(p);
	p = nullptr;
	have = 0;
	CK(pool_alloc(&p, need));
	have = need;
	return 0;
}
}  // namespace
extern "C" {

// The row each particle block starts at in the checkpoint's order, per model: an exclusive scan of the bucket sizes of the current
// partition into ck_base (entry pbc: the model's count), enqueued on the sim stream.  Shared by the checkpoint and the frame output,
// which both wait for their gather before returning.
static int enqueue_bucket_scans(cb200_sim* s) {
	CK(ck_grow(s->ck_base, s->ck_base_bytes, (size_t) kMaxModels * (s->desc.max_blocks + 1) * sizeof(int)));
	const int Rn = s->rollid ^ 1;
	for(size_t m = 0; m < s->models.size(); ++m) {
		ScanArgs sc {};
		sc.count = count_dev(&s->d_state->pbc);
		sc.count_plus = 1;
		sc.in = s->models[m].pb[Rn].particle_bucket_sizes;
		sc.out = s->ck_base + m * (s->desc.max_blocks + 1);
		scan_kernel<<<1, 1024, 0, s->stream>>>(sc);
		++s->launches;
	}
	return 0;
}

int cb200_sim_checkpoint_begin(cb200_sim* s, size_t* bytes) {
	if(!s || !s->setup_done) return (int) cudaErrorInvalidValue;
	if(s->ck_pending) CK(cudaEventSynchronize(s->ck_copied));  // the pinned blob and the staging blob are re-used
	s->ck_pending = s->ck_ready = false;
	if(!s->ck_stream) {
		CK(cudaStreamCreateWithFlags(&s->ck_stream, cudaStreamNonBlocking));
		CK(cudaEventCreateWithFlags(&s->ck_gathered, cudaEventDisableTiming));
		CK(cudaEventCreateWithFlags(&s->ck_copied, cudaEventDisableTiming));
	}
	const size_t cap = ck_capacity(s);
	CK(ck_grow(s->ck_dev, s->ck_dev_bytes, cap));
	if(s->ck_host_bytes < cap) {
		if(s->ck_host) cudaFreeHost(s->ck_host);
		s->ck_host = nullptr;
		s->ck_host_bytes = 0;
		CK(cudaMallocHost(&s->ck_host, cap));
		s->ck_host_bytes = cap;
	}
	const int R = s->rollid, Rn = R ^ 1;
	const int nm = (int) s->models.size();
	cudaStream_t st = s->stream;
	CK(enqueue_bucket_scans(s));
	SnapshotArgs a {};
	a.cfg = s->cfg;
	a.state = s->d_state;
	a.n_models = nm;
	for(int m = 0; m < nm; ++m) {
		const Model& md = s->models[m];
		a.material[m] = md.material;
		a.cur[m] = view(md.pb[R]);
		a.next[m] = view(md.pb[Rn]);
		a.base[m] = s->ck_base + (size_t) m * (s->desc.max_blocks + 1);
	}
	a.keys = s->part[R].active_keys;
	a.prev_table = s->part[Rn].index_table;
	a.grid = s->grid[0];
	a.out = s->ck_dev;
	snapshot_kernel<<<num_sms() * 8, kSnapThreads, 0, st>>>(a);
	++s->launches;
	CK(cudaGetLastError());
	CK(cudaEventRecord(s->ck_gathered, st));
	// the counts the layout follows from: the step state (pbc, nbc, clock), then each model's total, entry pbc of its scan
	CK(pull_state(s));
	const StepState& h = *s->h_state;
	int totals[kMaxModels] = {};
	for(int m = 0; m < nm; ++m) CK(cudaMemcpyAsync(&totals[m], s->ck_base + (size_t) m * (s->desc.max_blocks + 1) + h.pbc, sizeof(int), cudaMemcpyDeviceToHost, st));
	CK(cudaStreamSynchronize(st));
	cb200_checkpoint_info I;
	memset(&I, 0, sizeof(I));
	int mats[kMaxModels];
	long long counts[kMaxModels];
	for(int m = 0; m < nm; ++m) {
		mats[m] = s->models[m].material;
		counts[m] = totals[m];
	}
	const CkLayout L = ck_layout(nm, mats, counts, h.nbc);
	I.version = CB200_CHECKPOINT_VERSION;
	I.n_models = nm;
	I.bytes = L.total;
	I.cfg = s->desc.cfg;
	I.dt_default = s->desc.dt_default;
	I.fps = s->desc.fps;
	I.mgsp_rank = s->desc.mgsp_world > 1 ? s->desc.mgsp_rank : 0;
	I.mgsp_world = s->desc.mgsp_world;
	I.error = h.error;
	I.dt = h.dt;
	I.next_dt = h.next_dt;
	I.step_time = h.step_time;
	I.frame_time = h.frame_time;
	I.sim_time = h.sim_time;
	I.steps = h.steps;
	I.frames = s->frames_done;
	I.particle_block_count = h.pbc;
	I.neighbor_block_count = h.nbc;
	I.exterior_block_count = h.ebc;
	I.max_blocks = s->desc.max_blocks;
	I.keys_offset = L.keys_off;
	I.keys_bytes = L.keys_bytes;
	I.grid_offset = L.grid_off;
	I.grid_bytes = L.grid_bytes;
	for(int m = 0; m < nm; ++m) {
		cb200_checkpoint_model& md = I.models[m];
		md.material = mats[m];
		md.channels = ck_channels(mats[m]);
		md.count = counts[m];
		md.offset = L.model_off[m];
		md.bytes = L.model_bytes[m];
		md.params = s->models[m].pb[0];
		md.params.bins = nullptr;
		md.params.cell_particle_counts = md.params.particle_bucket_sizes = md.params.cellbuckets = md.params.blockbuckets = md.params.bin_offsets = nullptr;
	}
	ck_write_header(s->ck_host, I);
	// the data sections: behind the snapshot, on the copy stream, so that sub-steps enqueued from here on run alongside
	CK(cudaStreamWaitEvent(s->ck_stream, s->ck_gathered, 0));
	CK(cudaMemcpyAsync(s->ck_host + kCkHeader, s->ck_dev + kCkHeader, L.total - kCkHeader, cudaMemcpyDeviceToHost, s->ck_stream));
	CK(cudaEventRecord(s->ck_copied, s->ck_stream));
	s->ck_bytes = L.total;
	s->ck_pending = true;
	if(bytes) *bytes = L.total;
	return 0;
}

int cb200_sim_checkpoint_end(cb200_sim* s, const void** blob, size_t* bytes) {
	if(!s || (!s->ck_pending && !s->ck_ready)) return (int) cudaErrorInvalidValue;
	if(s->ck_pending) {
		CK(cudaEventSynchronize(s->ck_copied));
		s->ck_pending = false;
		s->ck_ready = true;
	}
	if(blob) *blob = s->ck_host;
	if(bytes) *bytes = s->ck_bytes;
	return 0;
}

int cb200_sim_restore_models(cb200_sim* s, const void* blob, size_t bytes) {
	cb200_checkpoint_info I;
	if(!s || s->setup_done || s->restore_pending || !s->models.empty() || ck_parse(blob, bytes, &I) != 0) return (int) cudaErrorInvalidValue;
	output_idle(s);
	const cb200_config& c = s->desc.cfg;
	if(c.domain_bits != I.cfg.domain_bits || c.max_ppc != I.cfg.max_ppc || c.boundary != I.cfg.boundary || memcmp(&c.gravity, &I.cfg.gravity, sizeof(float)) != 0 ||
	   memcmp(&c.cfl, &I.cfg.cfl, sizeof(float)) != 0 || memcmp(&s->desc.dt_default, &I.dt_default, sizeof(float)) != 0 || s->desc.fps != I.fps ||
	   s->desc.mgsp_world != I.mgsp_world || (s->desc.mgsp_world > 1 ? s->desc.mgsp_rank : 0) != I.mgsp_rank)
		return (int) cudaErrorInvalidValue;
	if(s->desc.max_blocks < I.exterior_block_count) return (int) cudaErrorMemoryAllocation;
	const unsigned char* src = static_cast<const unsigned char*>(blob);
	cudaStream_t st = s->stream;
	s->restore_info = I;
	s->restore_pending = true;
	for(int m = 0; m < I.n_models; ++m) {
		const cb200_checkpoint_model& md = I.models[m];
		Model model;
		model.material = md.material;
		model.n = (int) md.count;
		CK(alloc_model(s, model));
		for(int i = 0; i < 2; ++i) {  // the saved parameters, the containers of this simulator
			cb200_particle_buffer& pb = model.pb[i];
			cb200_particle_buffer p = md.params;
			p.bins = pb.bins;
			p.cell_particle_counts = pb.cell_particle_counts;
			p.particle_bucket_sizes = pb.particle_bucket_sizes;
			p.cellbuckets = pb.cellbuckets;
			p.blockbuckets = pb.blockbuckets;
			p.bin_offsets = pb.bin_offsets;
			pb = p;
		}
		s->models.push_back(model);
		CK(pool_alloc(&s->restore_state[m], md.bytes));
		CK(cudaMemcpyAsync(s->restore_state[m], src + md.offset, md.bytes, cudaMemcpyHostToDevice, st));
		state_positions_kernel<<<num_sms() * 4, 256, 0, st>>>(md.count, md.channels, s->restore_state[m], s->models.back().d_pos);
		++s->launches;
	}
	CK(pool_alloc(&s->restore_grid, (size_t) I.grid_bytes + (size_t) I.keys_bytes));
	CK(cudaMemcpyAsync(s->restore_grid, src + I.grid_offset, I.grid_bytes, cudaMemcpyHostToDevice, st));
	CK(cudaMemcpyAsync(s->restore_grid + I.grid_bytes, src + I.keys_offset, I.keys_bytes, cudaMemcpyHostToDevice, st));
	CK(cudaGetLastError());
	return (int) cudaStreamSynchronize(st);
}

int cb200_sim_restore(cb200_sim* s, const void* blob, size_t bytes) {
	CK(cb200_sim_restore_models(s, blob, bytes));
	return cb200_sim_initial_setup(s);
}

// ---- per-frame .bgeo output (format and kernel: output.cuh) ---------------------------------------------------------------------
int cb200_bgeo_header(long long points, unsigned attributes, void* out, size_t capacity, size_t* bytes) {
	const std::vector<unsigned char> h = bgeo_header(points, attributes);
	if(h.empty() || !out || capacity < h.size()) return (int) cudaErrorInvalidValue;
	memcpy(out, h.data(), h.size());
	if(bytes) *bytes = h.size();
	return 0;
}
int cb200_bgeo_trailer(void* out, size_t capacity, size_t* bytes) {
	if(!out || capacity < sizeof(kBgeoTrailer)) return (int) cudaErrorInvalidValue;
	memcpy(out, kBgeoTrailer, sizeof(kBgeoTrailer));
	if(bytes) *bytes = sizeof(kBgeoTrailer);
	return 0;
}

// One frame in flight: the next call waits for the writer (back-pressure) before its gather re-uses the staging and pinned buffers.
// A disk slower than the frames therefore slows the run down to the disk's pace instead of queueing frames in host memory without
// bound.
int cb200_sim_frame_output(cb200_sim* s, const char* const* paths, unsigned attributes) {
	if(!s || !s->setup_done || !paths || (attributes & ~kOutAttrs)) return (int) cudaErrorInvalidValue;
	const int nm = (int) s->models.size();
	for(int m = 0; m < nm; ++m)
		if(!paths[m]) return (int) cudaErrorInvalidValue;
	output_idle(s);
	{
		std::lock_guard<std::mutex> g(s->out_mu);
		if(s->out_errno) return CB200_ERROR_OUTPUT_IO;  // an earlier frame failed: report it before writing more
	}
	if(!s->out_stream) {
		CK(cudaStreamCreateWithFlags(&s->out_stream, cudaStreamNonBlocking));
		CK(cudaEventCreateWithFlags(&s->out_copied, cudaEventDisableTiming));
	}
	const int W = out_words(attributes);
	OutputArgs a {};
	size_t need = 0;
	for(int m = 0; m < nm; ++m) {  // a section per model, sized for all its particles
		a.off[m] = need;
		a.cap[m] = s->models[m].n;
		need += (size_t) s->models[m].n * W * sizeof(float);
	}
	CK(ck_grow(s->out_dev, s->out_dev_bytes, need));
	if(s->out_host_bytes < need) {
		if(s->out_host) cudaFreeHost(s->out_host);
		s->out_host = nullptr;
		s->out_host_bytes = 0;
		CK(cudaMallocHost(&s->out_host, need));
		s->out_host_bytes = need;
	}
	const int R = s->rollid, Rn = R ^ 1;
	CK(enqueue_bucket_scans(s));
	a.cfg = s->cfg;
	a.state = s->d_state;
	a.n_models = nm;
	a.attrs = attributes;
	for(int m = 0; m < nm; ++m) {
		const Model& md = s->models[m];
		a.material[m] = md.material;
		a.cur[m] = view(md.pb[R]);
		a.next[m] = view(md.pb[Rn]);
		a.base[m] = s->ck_base + (size_t) m * (s->desc.max_blocks + 1);
	}
	a.keys = s->part[R].active_keys;
	a.table = s->part[R].index_table;
	a.prev_table = s->part[Rn].index_table;
	a.grid = s->grid[0];
	a.out = s->out_dev;
	output_kernel<<<num_sms() * 8, kOutThreads, 0, s->stream>>>(a);
	++s->launches;
	CK(cudaGetLastError());
	// the counts the headers need (each model's total, entry pbc of its scan): this is the only wait, and it ends with the gather
	CK(pull_state(s));
	int totals[kMaxModels] = {};
	for(int m = 0; m < nm; ++m) CK(cudaMemcpyAsync(&totals[m], a.base[m] + s->h_state->pbc, sizeof(int), cudaMemcpyDeviceToHost, s->stream));
	CK(cudaStreamSynchronize(s->stream));
	std::vector<cb200_sim::OutputFile> files((size_t) nm);
	for(int m = 0; m < nm; ++m) {
		if(totals[m] < 0 || totals[m] > s->models[m].n) return (int) cudaErrorIllegalState;
		files[m].path = paths[m];
		files[m].header = bgeo_header(totals[m], attributes);
		files[m].body = s->out_host + a.off[m];
		files[m].body_bytes = (size_t) totals[m] * W * sizeof(float);
		// the gather has finished (the host waited for it above): the copy needs no event to order it behind the kernel
		if(files[m].body_bytes) CK(cudaMemcpyAsync(s->out_host + a.off[m], s->out_dev + a.off[m], files[m].body_bytes, cudaMemcpyDeviceToHost, s->out_stream));
	}
	CK(cudaEventRecord(s->out_copied, s->out_stream));
	if(!s->out_thread.joinable()) s->out_thread = std::thread(output_writer, s);
	{
		std::lock_guard<std::mutex> g(s->out_mu);
		s->out_files.swap(files);
		s->out_busy = true;
	}
	s->out_cv.notify_all();
	return 0;
}

int cb200_sim_frame_output_wait(cb200_sim* s, int* os_errno) {
	if(os_errno) *os_errno = 0;
	if(!s) return (int) cudaErrorInvalidValue;
	output_idle(s);
	std::lock_guard<std::mutex> g(s->out_mu);
	if(!s->out_errno) return 0;
	if(os_errno) *os_errno = s->out_errno;
	s->out_errno = 0;
	return CB200_ERROR_OUTPUT_IO;
}

int cb200_trim_pool(void) {
	g_pool.trim();
	return 0;
}

// ---- MGSP peer wiring ------------------------------------------------------------------------------------------
int cb200_sim_mgsp_inbox(cb200_sim* s, void** inbox, void** next_grid, size_t* inbox_bytes_out) {
	if(!s || s->desc.mgsp_world <= 1) return (int) cudaErrorInvalidValue;
	if(inbox) *inbox = s->inbox_local;
	if(next_grid) *next_grid = s->grid[1];
	if(inbox_bytes_out) *inbox_bytes_out = inbox_bytes(s->inbox_layout);
	return 0;
}
// CB200_MGSP_HANDLE_BYTES (160) bytes: cudaIpcMemHandle_t of the inbox, then of the next-grid buffer (target of the peers' fused halo
// reductions), then the parameters every rank must agree on -- the inbox layout is computed from them on BOTH sides of a
// transfer: {max_blocks, halo_cap, world, domain_bits, max_ppc}
static void mgsp_layout_words(const cb200_sim* s, int* w) {
	w[0] = s->desc.max_blocks;
	w[1] = s->desc.mgsp_halo_cap;
	w[2] = s->desc.mgsp_world;
	w[3] = s->desc.cfg.domain_bits;
	w[4] = s->desc.cfg.max_ppc;
	w[5] = w[6] = w[7] = 0;
}
int cb200_sim_mgsp_ipc_handle(cb200_sim* s, void* handle) {
	if(!s || s->desc.mgsp_world <= 1 || !handle) return (int) cudaErrorInvalidValue;
	static_assert(sizeof(cudaIpcMemHandle_t) == 64 && CB200_MGSP_HANDLE_BYTES == 160, "IPC handle blob layout");
	cudaIpcMemHandle_t h;
	CK(cudaIpcGetMemHandle(&h, s->inbox_local));
	memcpy(handle, &h, 64);
	CK(cudaIpcGetMemHandle(&h, s->grid[1]));
	memcpy((unsigned char*) handle + 64, &h, 64);
	int w[8];
	mgsp_layout_words(s, w);
	memcpy((unsigned char*) handle + 128, w, 32);
	return 0;
}
int cb200_sim_mgsp_open_peers(cb200_sim* s, const void* handles) {
	if(!s || s->desc.mgsp_world <= 1 || !handles) return (int) cudaErrorInvalidValue;
	int mine[8];
	mgsp_layout_words(s, mine);
	for(int r = 0; r < s->desc.mgsp_world; ++r) {  // a rank with another block capacity would lay out its messages differently
		int theirs[8];
		memcpy(theirs, (const unsigned char*) handles + CB200_MGSP_HANDLE_BYTES * r + 128, 32);
		if(memcmp(mine, theirs, 32) != 0) return (int) cudaErrorInvalidValue;
	}
	for(int r = 0; r < s->desc.mgsp_world; ++r) {
		if(r == s->desc.mgsp_rank) continue;
		cudaIpcMemHandle_t h;
		void* p = nullptr;
		memcpy(&h, (const unsigned char*) handles + CB200_MGSP_HANDLE_BYTES * r, 64);
		CK(g_ipc.open(&p, h));
		s->inbox_peer[r] = (unsigned char*) p;
		memcpy(&h, (const unsigned char*) handles + CB200_MGSP_HANDLE_BYTES * r + 64, 64);
		CK(g_ipc.open(&p, h));
		s->grid1_peer[r] = (float*) p;
	}
	s->peers_ready = true;
	return 0;
}
int cb200_sim_mgsp_set_peers(cb200_sim* s, void* const* inbox_ptrs, void* const* next_grid_ptrs) {
	if(!s || s->desc.mgsp_world <= 1 || !inbox_ptrs || !next_grid_ptrs) return (int) cudaErrorInvalidValue;
	for(int r = 0; r < s->desc.mgsp_world; ++r)
		if(r != s->desc.mgsp_rank) {
			s->inbox_peer[r] = (unsigned char*) inbox_ptrs[r];
			s->grid1_peer[r] = (float*) next_grid_ptrs[r];
		}
	s->peers_ready = true;
	return 0;
}
int cb200_sim_mgsp_halo_counts(cb200_sim* s, int* shared, int* halo_particle_blocks) {
	if(!s || s->desc.mgsp_world <= 1) return (int) cudaErrorInvalidValue;
	if(s->setup_done) {  // the halo particle blocks are statistics only in the fused path: counted on demand, not per sub-step
		const int P = s->rollid;
		CK(cudaMemsetAsync(s->part[P].halo_count, 0, sizeof(int), s->stream));
		collect_halo_blockids_kernel<<<grid_blocks(2), 128, 0, s->stream>>>(s->cfg, count_dev(&s->d_state->pbc), s->part[P].index_table, s->part[P].active_keys, s->part[P].overlap_marks, s->part[P].halo_marks, s->part[P].halo_count, nullptr);
		++s->launches;
	}
	CK(cudaStreamSynchronize(s->stream));
	if(shared) CK(cudaMemcpy(shared, s->peer_overlap_count, s->desc.mgsp_world * sizeof(int), cudaMemcpyDeviceToHost));
	if(halo_particle_blocks) CK(cudaMemcpy(halo_particle_blocks, s->part[s->rollid].halo_count, sizeof(int), cudaMemcpyDeviceToHost));
	return 0;
}

// per-kernel timing for the roofline: CUDA-event pairs around every g2p2g launch (sub-steps are issued as plain
// stream launches while profiling is on, so the events bracket exactly one kernel each)
int cb200_sim_profile(cb200_sim* s, int enable) {
	if(!s) return (int) cudaErrorInvalidValue;
	CK(cudaStreamSynchronize(s->stream));
	s->profiling = enable != 0;
	s->prof_used = 0;
	s->phase_used = 0;
	return 0;
}
// summed milliseconds per phase id (see mark_phase) since profiling was enabled; out_ms[10]
int cb200_sim_profile_phases(cb200_sim* s, double* out_ms) {
	if(!s || !out_ms) return (int) cudaErrorInvalidValue;
	CK(cudaStreamSynchronize(s->stream));
	for(int i = 0; i < 10; ++i) out_ms[i] = 0.0;
	for(size_t i = 1; i < s->phase_used; ++i) {
		if(s->phase_ids[i] == 0) continue;  // start of a sub-step: the gap before it belongs to nobody
		float ms = 0.f;
		CK(cudaEventElapsedTime(&ms, s->phase_events[i - 1], s->phase_events[i]));
		out_ms[s->phase_ids[i]] += ms;
	}
	return 0;
}
int cb200_sim_profile_read(cb200_sim* s, double* g2p2g_ms_total, int* launches) {
	if(!s) return (int) cudaErrorInvalidValue;
	CK(cudaStreamSynchronize(s->stream));
	double total = 0.0;
	for(size_t i = 0; i < s->prof_used; ++i) {
		float ms = 0.f;
		CK(cudaEventElapsedTime(&ms, s->prof_events[i].first, s->prof_events[i].second));
		total += ms;
	}
	if(g2p2g_ms_total) *g2p2g_ms_total = total;
	if(launches) *launches = (int) s->prof_used;
	s->prof_used = 0;
	return 0;
}

}  // extern "C"
