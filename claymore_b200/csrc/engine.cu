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
#include <cmath>
#include <condition_variable>
#include <cstdio>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "checkpoint.cuh"
#include "emit.cuh"
#include "g2p2g.cuh"
#include "grid.cuh"
#include "init.cuh"
#include "levelset.cuh"
#include "mesh.cuh"
#include "mgsp.cuh"
#include "output.cuh"
#include "partition.cuh"
#include "remove.cuh"
#include "sdf.cuh"

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

// Where a read-out lands before the host has it: a device buffer from the pool and its pinned host mirror, grown on demand (contents
// are not kept) and reused; with open_stream(), a stream of its own for the device->host copy and the event that marks the copy done.
// `pending`: a copy was queued on that stream and nobody has waited for it yet.
struct Staging {
	unsigned char* dev = nullptr;
	unsigned char* host = nullptr;  // pinned
	size_t dev_bytes = 0, host_bytes = 0;
	cudaStream_t stream = nullptr;
	cudaEvent_t copied = nullptr;
	bool pending = false;

	// at least `bytes` on the device and, with `mirror`, in the pinned mirror (a copy into caller memory needs none)
	int grow(size_t bytes, bool mirror) {
		if(dev_bytes < bytes) {
			g_pool.release(dev);
			dev = nullptr;
			dev_bytes = 0;
			CK(pool_alloc(&dev, bytes));
			dev_bytes = bytes;
		}
		if(mirror && host_bytes < bytes) {
			if(host) cudaFreeHost(host);
			host = nullptr;
			host_bytes = 0;
			CK(cudaMallocHost(&host, bytes));
			host_bytes = bytes;
		}
		return 0;
	}
	int open_stream() {
		if(stream) return 0;
		CK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
		return (int) cudaEventCreateWithFlags(&copied, cudaEventDisableTiming);
	}
	int wait() {
		if(!pending) return 0;
		CK(cudaEventSynchronize(copied));
		pending = false;
		return 0;
	}
	// after every copy on the stream has finished
	void release() {
		if(stream) cudaStreamSynchronize(stream);
		g_pool.release(dev);
		if(host) cudaFreeHost(host);
		if(copied) cudaEventDestroy(copied);
		if(stream) cudaStreamDestroy(stream);
		*this = Staging {};
	}
};

struct Model {
	int material = 0;
	cb200_particle_buffer pb[2];
	long long bin_capacity = 0;
	float* d_pos = nullptr;
	int n = 0;
	float v0[3] = {0, 0, 0};
	int* bin_sizes = nullptr;
	unsigned short* celloffs[2] = {nullptr, nullptr};  // per buffer: start of every cell inside the (cell-major) block bucket, [blocks][64]
	Staging out;  // retrieve and particle_state
};
// capacity rule of init_model (gmpm_simulator.cuh:173): n/32 bins + one partial bin per block
inline long long bin_rows(long long n, long long max_blocks) { return n / kBinCap + max_blocks; }

// counters and maxima the driver's kernels hand to each other within a sub-step (or a set-up, a retrieve)
struct DeviceScratch {
	int new_pbc;         // particle blocks of the rebuilt partition (summary_kernel)
	int new_nbc;         // neighbour blocks, snapshotted by the last CTA of their registration; MGSP: the exchange's key count
	float local_max;     // MGSP: this rank's max |v|^2 of the new grid
	float global_max;    // MGSP: the max over the ranks
	float mgsp_grid_max; // MGSP: the grid update's max |v|^2, never read (the exchange agreed on the max already)
	int missing;         // saved grid blocks scatter_grid_kernel found no block for
	int model_count[kMaxModels];  // each model's particle count, from its last bucket scan (enqueue_bucket_scan)
};
// MGSP: the last-CTA counters and the exchange epochs (MgspView::done / ::epochs)
struct MgspCounters {
	int done[4];
	int epochs[3];
};

// the simulation clock: what a checkpoint saves of StepState (+ the frames cb200_sim_advance_frame finished) and a start sets
struct Clock {
	float dt, next_dt, step_time, frame_time;
	double sim_time;
	long long steps, frames;
	int error;
};
Clock clock_of(const StepState& h, long long frames) { return Clock {h.dt, h.next_dt, h.step_time, h.frame_time, h.sim_time, h.steps, frames, h.error}; }
void set_clock(StepState& h, long long& frames, const Clock& c) {
	h.dt = c.dt;
	h.next_dt = c.next_dt;
	h.step_time = c.step_time;
	h.frame_time = c.frame_time;
	h.sim_time = c.sim_time;
	h.steps = c.steps;
	h.error |= c.error;
	frames = c.frames;
}
// min(dt, dx·cfl/mv), dt for mv = 0: initial_setup's dt rule (gmpm_simulator.cuh:305-315) for the start and for an emission, whose dt
// is held to a set-up's bitwise
float cfl_dt(const Cfg& cfg, float dt, float mv) { return mv > 0.f ? fminf(dt, cfg.dx * cfg.cfl / mv) : dt; }

struct BlockCounts {
	int pbc, nbc, ebc;
};
// What a start (initial_setup) is made of.  Each part may be absent, and then set-up makes it itself.
struct StartSrc {
	const float* rows[kMaxModels] = {};  // per model, [n][channels] state rows; absent: the start state at d_pos
	const float* grid = nullptr;         // [grid_count][256] saved grid blocks with their keys [grid_count][3]; absent: rasterise the bins
	const int* keys = nullptr;
	int grid_count = 0;                  // a checkpoint's nbc; an emission's old nbc, a subset of the rebuilt partition's
	const Clock* clock = nullptr;        // absent: the fresh clock of desc and the models' v0
	const BlockCounts* expect = nullptr; // the block counts the rebuild must reproduce; absent: no check
	const float* vel = nullptr;          // [vel_count][256] saved grid blocks with their keys [vel_count][3] whose node velocities p / m
	const int* vel_keys = nullptr;       // the rasterised mass takes (a removal); absent: the models' v0.  Not with `grid`.
	int vel_count = 0;
};

// cb200_sim_restore_models: the checkpoint's state, clock and block counts, staged on the device until initial_setup consumes them
struct RestoreStaging {
	bool pending = false;
	Clock clock {};
	BlockCounts counts {};
	float* rows[kMaxModels] = {};
	unsigned char* grid = nullptr;  // grid blocks, then keys
	size_t grid_bytes = 0;

	StartSrc start() const {
		StartSrc s;
		if(!pending) return s;
		for(int m = 0; m < kMaxModels; ++m) s.rows[m] = rows[m];
		s.grid = reinterpret_cast<const float*>(grid);
		s.keys = reinterpret_cast<const int*>(grid + grid_bytes);
		s.grid_count = counts.nbc;
		s.clock = &clock;
		s.expect = &counts;
		return s;
	}
	// after every read of the staged buffers has finished
	void release() {
		for(float* p : rows) g_pool.release(p);
		g_pool.release(grid);
		*this = RestoreStaging {};
	}
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
	DeviceScratch* scr = nullptr;
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
	MgspCounters* mgsp_sync = nullptr;
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
	// the signed-distance collider (cb200_sim_set_collider), whose device field this simulator owns (sdf), and the analytic collision
	// objects (cb200_sim_set_collision_objects) resolved after it in list order
	Boundaries boundaries {};
	float* sdf = nullptr;
	// the lattices of the level-set collision objects (cb200_sim_add_collision_levelset), owned by this simulator, in registry order
	LevelSets levelsets {};
	long long frames_done = 0;  // frames finished by cb200_sim_advance_frame (restored from a checkpoint)
	// the boundary impulse report (cb200_sim_set_force_report): its sums, [kForceBodies][kForceComps] doubles, then the simulated time of
	// its last reset (force_reset)
	bool force_report = false;
	double* forces = nullptr;
	// the objects' motion tracks (cb200_sim_set_object_track): each tracked object's prepared keys, and their concatenation in object
	// order on the device (track_table, CB200_MAX_TRACK_KEYS records) that `tracks` indexes
	std::vector<cb200_track_record> track_keys[CB200_MAX_COLLISION_OBJECTS];
	int track_flags[CB200_MAX_COLLISION_OBJECTS] = {};
	cb200_track_record* track_table = nullptr;
	Tracks tracks {};
	// the rows each particle block starts at in every read-out, per model: the scans of the bucket sizes, [kMaxModels][max_blocks + 1]
	int* ck_base = nullptr;
	// checkpoint (cb200_sim_checkpoint_begin / _end): the blob, copied to the host on the staging's own stream
	Staging ck;
	size_t ck_bytes = 0;  // bytes of the blob the last begin queued (0: none)
	RestoreStaging restore;
	// frame output (cb200_sim_frame_output): the records, copied to the host on the staging's own stream, and the writer thread with
	// its one job, which waits for that copy; started on first use.  `out_busy`: a frame is queued or being written
	Staging out;
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
// ---- the device arrays of each owner (a model, a partition, the simulator), listed once -------------------------------------------
// An entry is the pointer an array lives in, its bytes at the capacity the list was made for, and the byte every element starts as.
// Allocation, growth, the emission's reset and release all walk these lists.  A list holds pointers into its owner: it is made from
// the owner at the call and used there, never kept.
constexpr int kNoFill = -1;  // the contents are left as allocated: every element is written before it is read
struct DevArray {
	void** p;
	size_t bytes;
	int fill;
};
using DevArrays = std::vector<DevArray>;
template<typename T>
DevArray dev_array(T*& p, size_t count, int fill) { return {reinterpret_cast<void**>(&p), count * sizeof(T), fill}; }

// one roll's particle buffer at block capacity mb, with `rows` bins
void buffer_arrays(DevArrays& a, const cb200_sim* s, const Model& m, cb200_particle_buffer& pb, size_t mb, long long rows) {
	const size_t ppb = (size_t) s->cfg.ppb;
	a.push_back(dev_array(pb.bins, (size_t) rows * bin_floats(m.material), kNoFill));
	a.push_back(dev_array(pb.cell_particle_counts, (mb + 1) * kBlockVol, 0));
	a.push_back(dev_array(pb.particle_bucket_sizes, mb + 2, 0));
	a.push_back(dev_array(pb.cellbuckets, (mb + 1) * ppb, kNoFill));
	a.push_back(dev_array(pb.blockbuckets, (mb + 1) * ppb, kNoFill));
	a.push_back(dev_array(pb.bin_offsets, mb + 2, 0));
}
// a model: both rolls' buffers, the bin sizes, both rolls' cell offsets and the m.n start positions (the caller fills those)
DevArrays model_arrays(const cb200_sim* s, Model& m, size_t mb, long long rows) {
	DevArrays a;
	for(cb200_particle_buffer& pb : m.pb) buffer_arrays(a, s, m, pb, mb, rows);
	a.push_back(dev_array(m.bin_sizes, mb + 2, 0));
	for(unsigned short*& offs : m.celloffs) a.push_back(dev_array(offs, (mb + 1) * kBlockVol, 0));
	a.push_back(dev_array(m.d_pos, (size_t) m.n * 3, kNoFill));
	return a;
}
// a partition, empty (halo_blocks stays null: the fused MGSP path collects no halo block list)
DevArrays partition_arrays(const cb200_sim* s, cb200_partition& p, size_t mb) {
	return {dev_array(p.count, 1, 0),
	        dev_array(p.index_table, s->table_entries, 0xff),
	        dev_array(p.active_keys, (mb + 1) * 3, 0),
	        dev_array(p.halo_count, 1, 0),
	        dev_array(p.halo_marks, mb + 1, 0),
	        dev_array(p.overlap_marks, mb + 1, 0)};
}
// the simulator's own: step state, scratch, both grids, the rebuild's scratch (produced and consumed inside a sub-step) and the
// read-outs' scans (produced and consumed inside a read-out)
DevArrays sim_arrays(cb200_sim* s, size_t mb) {
	const size_t tiles = (mb + kRebuildTile - 1) / kRebuildTile + 1;
	return {dev_array(s->d_state, 1, 0),
	        dev_array(s->scr, 1, 0),
	        dev_array(s->grid[0], (mb + 1) * kGridBlockFloats, 0),
	        dev_array(s->grid[1], (mb + 1) * kGridBlockFloats, 0),
	        dev_array(s->tile_sums, tiles * kScanComps, kNoFill),
	        dev_array(s->block_totals, (size_t) kMaxModels * mb, kNoFill),
	        dev_array(s->ck_base, (size_t) kMaxModels * (mb + 1), kNoFill),
	        dev_array(s->forces, (size_t) kForceBodies * kForceComps + 1, 0),
	        dev_array(s->track_table, (size_t) CB200_MAX_TRACK_KEYS, kNoFill)};
}

int fill_arrays(cb200_sim* s, const DevArrays& a) {
	for(const DevArray& d : a)
		if(d.fill != kNoFill) CK(cudaMemsetAsync(*d.p, d.fill, d.bytes, s->stream));
	return 0;
}
int alloc_arrays(cb200_sim* s, const DevArrays& a) {
	for(const DevArray& d : a) CK(g_pool.alloc(d.p, d.bytes));
	return fill_arrays(s, a);
}
void free_arrays(const DevArrays& a) {
	for(const DevArray& d : a) g_pool.release(*d.p);
}
// Grows the arrays of `from` to their sizes in `to`, the same list at a larger capacity: allocate the larger array, copy the live
// prefix, fill the tail by the array's rule, release the old one.  One array at a time, so the peak is the footprint plus the
// largest array; a failure leaves every array valid, those already moved merely larger.
int grow_arrays(cb200_sim* s, const DevArrays& from, const DevArrays& to) {
	for(size_t i = 0; i < to.size(); ++i) {
		const DevArray& d = to[i];
		const size_t old_bytes = from[i].bytes;
		if(d.bytes <= old_bytes) continue;
		void* q = nullptr;
		CK(g_pool.alloc(&q, d.bytes));
		int e = (int) cudaMemcpyAsync(q, *d.p, old_bytes, cudaMemcpyDeviceToDevice, s->stream);
		if(!e && d.fill != kNoFill) e = (int) cudaMemsetAsync((unsigned char*) q + old_bytes, d.fill, d.bytes - old_bytes, s->stream);
		if(!e) e = (int) cudaStreamSynchronize(s->stream);
		if(e) {
			g_pool.release(q);
			return e;
		}
		g_pool.release(*d.p);
		*d.p = q;
	}
	return 0;
}

// the material parameters of `from` (every field from rho on), the containers of `to`
void copy_params(cb200_particle_buffer& to, const cb200_particle_buffer& from) {
	memcpy(&to.rho, &from.rho, sizeof(to) - offsetof(cb200_particle_buffer, rho));
}
void drop_graphs(cb200_sim* s) {
	for(cudaGraphExec_t& g : s->graph) {
		if(g) cudaGraphExecDestroy(g);
		g = nullptr;
	}
}

// A new model of `material`, n particles and the default parameters (init_model, init_model_sdf, restore): its containers, then
// fill(m) enqueues the n start positions into m.d_pos on the sim stream.  Appended once they are there; a failure releases it.
template<class Fill>
int add_model(cb200_sim* s, int material, int n, const float* v0, int* model_id, Fill&& fill) {
	if(material < 0 || material > 3 || n <= 0 || (int) s->models.size() >= kMaxModels) return (int) cudaErrorInvalidValue;
	Model m;
	m.material = material;
	m.n = n;
	for(int d = 0; d < 3; ++d) m.v0[d] = v0 ? v0[d] : 0.f;
	const long long mb = s->desc.max_blocks;
	m.bin_capacity = bin_rows(n, mb);
	for(cb200_particle_buffer& pb : m.pb) {
		memset(&pb, 0, sizeof(pb));
		default_material(s->desc.cfg, material, pb);
	}
	const DevArrays a = model_arrays(s, m, (size_t) mb, m.bin_capacity);
	int e = alloc_arrays(s, a);
	if(!e) e = fill(m);
	if(!e) e = (int) cudaStreamSynchronize(s->stream);
	if(e) {
		cudaStreamSynchronize(s->stream);
		free_arrays(a);
		return e;
	}
	if(model_id) *model_id = (int) s->models.size();
	s->models.push_back(m);
	return 0;
}

inline int grid_blocks(int per_sm) { return num_sms() * per_sm; }
// A registration thread walks its (block, offset) pairs one after the other, each a key read and then a table CAS that waits for L2:
// the launch is bound by how many threads walk at once, so it fills every thread slot of the SMs (16 x 128; the kernel takes 32 registers)
constexpr int kRegisterCtasPerSm = 16;

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

// zeroes the report's sums and starts its span at StepState::sim_time, stream-ordered
int force_reset(cb200_sim* s) {
	constexpr size_t n = (size_t) kForceBodies * kForceComps;
	CK(cudaMemsetAsync(s->forces, 0, n * sizeof(double), s->stream));
	CK(cudaMemcpyAsync(s->forces + n, &s->d_state->sim_time, sizeof(double), cudaMemcpyDeviceToDevice, s->stream));
	return 0;
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
		gu.max_vel = &s->scr->mgsp_grid_max;
		gu.clear_grid = nullptr;
	}
	gu.n_clear = (int) s->models.size();
	for(size_t m = 0; m < s->models.size(); ++m) gu.clear_counts[m] = s->models[m].pb[Rn].cell_particle_counts;
	// MGSP: a block every rank holding it resolves counts on the lowest of them (the marks the previous sub-step's tagging left)
	const ForceArgs fa {s->forces, s->desc.mgsp_world > 1 ? s->part[R].overlap_marks : nullptr, (1u << s->desc.mgsp_rank) - 1u};
	launch_grid_update(gu, s->boundaries, s->levelsets, grid_blocks(4), s->stream, s->force_report ? &fa : nullptr, &s->tracks);  // placed at StepState::sim_time, the start of this sub-step
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
		a.new_pbc = &s->scr->new_pbc;
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
		rebuild_kernel<<<tiles * kRebuildSplit, kRebuildThreads, 0, st>>>(a);
		++s->launches;
	}
	{
		RegisterArgs a {};
		a.cfg = s->cfg;
		a.block_count = count_dev(&s->scr->new_pbc);
		a.table = s->part[Rn].index_table;
		a.keys = s->part[Rn].active_keys;
		a.count = s->part[Rn].count;
		a.capacity = s->desc.max_blocks;
		a.error = &s->d_state->error;
		a.lo = 0;
		a.span = 2;
		a.done_counter = &s->d_state->done_counter;  // the last CTA snapshots the neighbour count
		a.snapshot_out = &s->scr->new_nbc;
		register_blocks_kernel<<<grid_blocks(kRegisterCtasPerSm), 128, 0, st>>>(a);
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
	DeviceScratch* scr = s->scr;
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
		a.new_count = &scr->new_nbc;
		a.new_keys = s->part[Rn].active_keys;
		a.old_table = s->part[R].index_table;
		a.state = s->d_state;
		a.old_grid = s->grid[1];
		a.new_grid = s->grid[0];
		a.next_max_vel = mgsp ? &scr->local_max : nullptr;
		// MGSP: the boundaries, so that the predicted max is the one the next grid update finds; a single domain predicts nothing
		launch_carry_grid(a, mgsp ? s->boundaries : Boundaries {}, s->levelsets, grid_blocks(4), st, mgsp ? &s->tracks : nullptr);
		++s->launches;
	}
	if(mgsp) {
		mgsp_clear_publish_kernel<<<grid_blocks(2), 256, 0, st>>>(mgsp_view(s), s->part[Rn].active_keys, &scr->new_nbc, &scr->local_max, s->grid[1]);
		++s->launches;
	}
	FinalizeArgs fin {};
	fin.cfg = s->cfg;
	fin.state = s->d_state;
	fin.new_pbc = &scr->new_pbc;
	fin.new_nbc = &scr->new_nbc;
	fin.new_count = s->part[Rn].count;
	fin.max_blocks = s->desc.max_blocks;
	fin.n_models = (int) s->models.size();
	for(size_t m = 0; m < s->models.size(); ++m) fin.bin_capacity[m] = s->models[m].bin_capacity;
	fin.next_max_vel = mgsp ? &scr->global_max : nullptr;
	{
		RegisterArgs a {};
		a.cfg = s->cfg;
		a.block_count = count_dev(&scr->new_pbc);
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
		register_blocks_kernel<<<grid_blocks(kRegisterCtasPerSm), 128, 0, st>>>(a);
		++s->launches;
	}
	mark_phase(s, 9);
	if(mgsp) {
		mgsp_tag_kernel<<<grid_blocks(1), 256, 0, st>>>(s->cfg, mgsp_view(s), s->part[Rn].index_table, s->part[Rn].overlap_marks, &scr->new_nbc, &scr->local_max, &scr->global_max, 1, fin);
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
	v.done = s->mgsp_sync->done;
	v.epochs = s->mgsp_sync->epochs;
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
	preload(grid_update_kernel);
	preload(clear_grid_kernel);
	preload(carry_grid_kernel);
	preload(grid_max_kernel);
	for_each_boundary_instance([](auto C, auto O) {
		preload(grid_update_boundary_kernel<C, O>);
		preload(carry_grid_boundary_kernel<C, O>);
		preload(grid_max_boundary_kernel<C, O>);
	});
	for_each_boundary_instance([](auto C, auto O) {
		if constexpr(O) {
			preload(grid_update_levelset_kernel<C>);
			preload(carry_grid_levelset_kernel<C>);
			preload(grid_max_levelset_kernel<C>);
		}
	});
	preload(scan_kernel);
	preload(summary_kernel);
	preload(rebuild_kernel);
	preload(register_blocks_kernel);
	preload(warp_flatten_kernel);
	preload(compute_bin_capacity_kernel);
	preload(activate_blocks_kernel<true>);
	preload(build_particle_cell_buckets_kernel<true>);
	preload(array_to_buffer_kernel);
	preload(rasterize_kernel);
	preload(rasterize_blocks_kernel);
	preload(init_adv_bucket_kernel);
	preload(collect_halo_blockids_kernel);
	preload(mgsp_allreduce_maxvel_kernel);
	preload(mgsp_pack_send_kernel);
	preload(mgsp_wait_reduce_kernel);
	preload(mgsp_tag_reset_kernel);
	preload(mgsp_tag_kernel);
	preload(mgsp_done_publish_kernel);
	preload(mgsp_done_wait_kernel);
	preload(mgsp_clear_publish_kernel);
	preload(snapshot_kernel);
	preload(state_positions_kernel);
	preload(scatter_grid_kernel);
	preload(output_kernel);
	preload(state_rows_kernel<true>);
	preload(state_rows_kernel<false>);
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
		const bool copied = cudaEventSynchronize(s->out.copied) == cudaSuccess;  // (failed: nothing of this frame is written)
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
	CK(s->ck.wait());  // the next begin re-sizes the staging blob
	output_idle(s);
	const size_t ob = (size_t) s->desc.max_blocks, nb = (size_t) new_max_blocks;
	drop_graphs(s);
	for(cb200_partition& p : s->part) CK(grow_arrays(s, partition_arrays(s, p, ob), partition_arrays(s, p, nb)));
	CK(grow_arrays(s, sim_arrays(s, ob), sim_arrays(s, nb)));
	for(Model& m : s->models) {
		const long long rows = std::max(m.bin_capacity, bin_rows(m.n, (long long) nb));
		CK(grow_arrays(s, model_arrays(s, m, ob, m.bin_capacity), model_arrays(s, m, nb, rows)));
		m.bin_capacity = rows;
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
	CK(g_pinned.get(&s->h_state));
	memset(s->h_state, 0, sizeof(StepState));
	CK(alloc_arrays(s, sim_arrays(s, mb)));
	for(cb200_partition& p : s->part) CK(alloc_arrays(s, partition_arrays(s, p, mb)));
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
		CK(pool_alloc(&s->mgsp_sync, sizeof(MgspCounters)));
		CK(cudaMemsetAsync(s->mgsp_sync, 0, sizeof(MgspCounters), s->stream));
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
	s->out.release();
	s->ck.release();  // (a checkpoint copy may still read the staging blob: release waits for it)
	s->restore.release();
	for(auto& ev : s->prof_events) {
		cudaEventDestroy(ev.first);
		cudaEventDestroy(ev.second);
	}
	drop_graphs(s);
	const size_t mb = (size_t) s->desc.max_blocks;
	for(cb200_partition& p : s->part) free_arrays(partition_arrays(s, p, mb));
	for(Model& m : s->models) {
		free_arrays(model_arrays(s, m, mb, m.bin_capacity));
		m.out.release();
	}
	free_arrays(sim_arrays(s, mb));
	g_pool.release(s->peer_overlap_keys);
	g_pool.release(s->peer_overlap_count);
	// peer mappings stay open (IpcCache): the exporting rank pools the buffer, the next simulator maps the same handle
	g_pool.release(s->peer_bno);
	g_pool.release(s->inbox_local);
	g_pool.release(s->mgsp_sync);
	g_pool.release(s->sdf);
	for(int i = 0; i < s->levelsets.count; ++i) g_pool.release(const_cast<float*>(s->levelsets.v[i].lattice));
	g_pinned.put(s->h_state);
	g_pinned.put(s->h_poll);
	if(s->poll_event) cudaEventDestroy(s->poll_event);
	if(s->owns_stream) cudaStreamDestroy(s->stream);
	delete s;
	return 0;
}

int cb200_sim_init_model(cb200_sim* s, int material, const float* positions_host, int n, const float* v0, int* model_id) {
	if(!s || s->setup_done) return (int) cudaErrorInvalidValue;
	return add_model(s, material, n, v0, model_id, [&](Model& m) {
		return (int) cudaMemcpyAsync(m.d_pos, positions_host, (size_t) n * 3 * sizeof(float), cudaMemcpyHostToDevice, s->stream);
	});
}

static int recapture(cb200_sim* s);
// make_g2p2g_args passes each model's parameters by value, so the sub-step graphs hold the ones they were captured with: a setter
// called between sub-steps re-captures them (after the sub-steps issued before it), and the change applies from the next sub-step
// in graph and stream mode alike.  The clock and the force report are kept.
static int params_changed(cb200_sim* s) {
	CK(cudaStreamSynchronize(s->stream));
	return recapture(s);
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
int cb200_sim_update_fr_parameters(cb200_sim* s, int model, float rho, float vol, float ym, float pr) {
	CK(set_elastic(s, model, CB200_FIXED_COROTATED, rho, vol, ym, pr));
	return params_changed(s);
}
int cb200_sim_update_sand_parameters(cb200_sim* s, int model, float rho, float vol, float ym, float pr) {
	CK(set_elastic(s, model, CB200_SAND, rho, vol, ym, pr));
	return params_changed(s);
}
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
	return params_changed(s);
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
	return params_changed(s);
}

// register_blocks_kernel over the (lo, span) ring of the first pbc blocks of partition p; returns p's new block count in *out
// (synchronises).  initial_setup's neighbour (0, 2) and exterior (-1, 3) registrations.
static int register_ring(cb200_sim* s, Part p, int capacity, int* error, int pbc, int lo, int span, int* out) {
	RegisterArgs a {};
	a.cfg = s->cfg;
	a.block_count = count_imm(pbc);
	a.table = p.table;
	a.keys = p.keys;
	a.count = p.count;
	a.capacity = capacity;
	a.error = error;
	a.lo = lo;
	a.span = span;
	register_blocks_kernel<<<grid_for((long long) pbc * span * span * span, 128, 16), 128, 0, s->stream>>>(a);
	++s->launches;
	CK(cudaMemcpyAsync(out, p.count, sizeof(int), cudaMemcpyDeviceToHost, s->stream));
	return (int) cudaStreamSynchronize(s->stream);
}

// initial_setup  gmpm_simulator.cuh:637-781 (counts are read back here: one-time cost), from the parts `src` has and the models'
// positions: the bins get the start state or the saved rows, grid[0] the rasterised particles or the saved blocks (no MGSP halo
// reduction: they hold the full sums) or, with src.vel, the rasterised mass at the saved velocities, the step state the fresh clock or
// the saved one.
constexpr float kZeroVel[3] = {0.f, 0.f, 0.f};
static int setup_impl(cb200_sim* s, const StartSrc& src) {
	if(!s || s->setup_done || s->models.empty()) return (int) cudaErrorInvalidValue;
	cudaStream_t st = s->stream;
	const Cfg& cfg = s->cfg;
	const int R = s->rollid, Rn = R ^ 1;
	const int cap = s->desc.max_blocks;
	const bool mgsp = s->desc.mgsp_world > 1;
	int* err = &s->d_state->error;
	int pbc = 0, nbc = 0, ebc = 0;
	cb200_partition& P = s->part[Rn];  // the partition set-up builds

	// it builds into P and roll R's buckets: both start empty (stream-ordered only: MGSP ranks set up concurrently)
	CK(fill_arrays(s, partition_arrays(s, P, (size_t) cap)));
	for(Model& m : s->models) {
		DevArrays a;
		buffer_arrays(a, s, m, m.pb[R], (size_t) cap, m.bin_capacity);
		CK(fill_arrays(s, a));
	}
	for(Model& m : s->models) {
		activate_blocks_kernel<true><<<grid_for(m.n, 256, 16), 256, 0, st>>>(cfg, m.n, m.d_pos, P.index_table, P.active_keys, P.count, cap, err);
		++s->launches;
	}
	CK(cudaMemcpyAsync(&pbc, P.count, sizeof(int), cudaMemcpyDeviceToHost, st));
	CK(cudaStreamSynchronize(st));
	if(pbc > cap) return (int) cudaErrorMemoryAllocation;
	for(Model& m : s->models) {
		build_particle_cell_buckets_kernel<true><<<grid_for(m.n, 256, 16), 256, 0, st>>>(cfg, m.n, m.d_pos, view(m.pb[R]), P.index_table, err);
		// the sub-step's flatten, in place: the driver's cell buckets have one (slot-grouped) layout whoever wrote them
		warp_flatten_kernel<<<grid_for(pbc, 8, 8), 256, 0, st>>>(cfg, pbc, m.pb[R].cell_particle_counts, m.pb[R].cellbuckets, m.pb[R].particle_bucket_sizes, m.pb[R].blockbuckets, m.celloffs[Rn]);
		compute_bin_capacity_kernel<<<grid_for(pbc + 1, 256, 16), 256, 0, st>>>(pbc + 1, m.pb[R].particle_bucket_sizes, m.bin_sizes);
		ScanArgs a {};
		a.count = count_imm(pbc + 1);
		a.in = m.bin_sizes;
		a.out = m.pb[R].bin_offsets;
		scan_kernel<<<1, 1024, 0, st>>>(a);
		array_to_buffer_kernel<<<grid_for(pbc, 1, 16), 128, 0, st>>>(cfg, m.material, pbc, m.d_pos, src.rows[&m - s->models.data()], view(m.pb[R]));
		s->launches += 5;
	}
	CK(register_ring(s, view(P), cap, err, pbc, 0, 2, &nbc));
	if(mgsp) {  // halo_tagging of the initial partition (mgsp_benchmark.cuh:633), with the kernels of the sub-step
		if(!s->peers_ready) return (int) cudaErrorNotReady;
		const MgspView v = mgsp_view(s);
		DeviceScratch* scr = s->scr;
		CK(cudaMemcpyAsync(&scr->new_nbc, &nbc, sizeof(int), cudaMemcpyHostToDevice, st));  // key count of the exchange
		CK(cudaMemsetAsync(&scr->local_max, 0, sizeof(float), st));
		CK(cudaMemsetAsync(&scr->global_max, 0, sizeof(float), st));
		mgsp_tag_reset_kernel<<<grid_blocks(1), 256, 0, st>>>(v, P.overlap_marks, &scr->new_nbc);
		// the next grid is still all zero from cb200_sim_create: the clear changes nothing, and the flag still goes out behind it
		mgsp_clear_publish_kernel<<<grid_blocks(2), 256, 0, st>>>(v, P.active_keys, &scr->new_nbc, &scr->local_max, s->grid[1]);
		mgsp_tag_kernel<<<grid_blocks(1), 256, 0, st>>>(cfg, v, P.index_table, P.overlap_marks, &scr->new_nbc, &scr->local_max, &scr->global_max, 0, FinalizeArgs {});
		s->launches += 3;
	}
	CK(register_ring(s, view(P), cap, err, pbc, -1, 3, &ebc));
	if(nbc > cap || ebc > cap) return (int) cudaErrorMemoryAllocation;
	// a blob that passed inspect but does not rebuild the saved partition (hand-edited): nothing to step
	if(src.expect && (pbc != src.expect->pbc || nbc != src.expect->nbc || ebc != src.expect->ebc)) return (int) cudaErrorIllegalState;
	// background copies (gmpm_simulator.cuh:745-756); the device count is copied too so that the stale-key
	// un-insert of the first rebuild knows how many entries the table holds
	CK(cudaMemcpyAsync(s->part[R].index_table, s->part[Rn].index_table, s->table_entries * sizeof(int), cudaMemcpyDeviceToDevice, st));
	CK(cudaMemcpyAsync(s->part[R].active_keys, s->part[Rn].active_keys, (size_t) ebc * 3 * sizeof(int), cudaMemcpyDeviceToDevice, st));
	CK(cudaMemcpyAsync(s->part[R].count, s->part[Rn].count, sizeof(int), cudaMemcpyDeviceToDevice, st));
	if(mgsp)  // "need to copy halo tag info as well" (mgsp_benchmark.cuh:639-640)
		CK(cudaMemcpyAsync(s->part[R].overlap_marks, s->part[Rn].overlap_marks, (size_t) nbc * sizeof(int), cudaMemcpyDeviceToDevice, st));
	for(Model& m : s->models) {
		CK(cudaMemcpyAsync(m.pb[Rn].bin_offsets, m.pb[R].bin_offsets, (size_t) (pbc + 1) * sizeof(int), cudaMemcpyDeviceToDevice, st));
		CK(cudaMemcpyAsync(m.pb[Rn].particle_bucket_sizes, m.pb[R].particle_bucket_sizes, (size_t) pbc * sizeof(int), cudaMemcpyDeviceToDevice, st));
	}
	clear_grid_kernel<<<grid_for((long long) nbc * 64, 256, 16), 256, 0, st>>>(nbc, s->grid[0]);
	++s->launches;
	if(src.grid) {  // the saved blocks by key; a key the rebuilt partition has no neighbour block for is counted, not written
		int* missing = &s->scr->missing;
		CK(cudaMemsetAsync(missing, 0, sizeof(int), st));
		scatter_grid_kernel<<<grid_for(src.grid_count, 8, 16), 256, 0, st>>>(cfg, src.grid_count, src.keys, src.grid, s->part[R].index_table, nbc, s->grid[0], missing);
		++s->launches;
		int miss = 0;
		CK(cudaMemcpyAsync(&miss, missing, sizeof(int), cudaMemcpyDeviceToHost, st));
		CK(cudaStreamSynchronize(st));
		if(miss) return (int) cudaErrorIllegalState;
	}
	for(Model& m : s->models) {
		if(!src.grid) {
			const float* v0 = src.vel ? kZeroVel : m.v0;
			rasterize_blocks_kernel<<<grid_for(pbc, 1, 16), 256, 0, st>>>(cfg, m.material, pbc, s->part[R].active_keys, s->part[R].index_table, view(m.pb[R]), s->grid[0], m.pb[R].mass, v0[0], v0[1], v0[2], err);
			++s->launches;
		}
		init_adv_bucket_kernel<<<grid_for(pbc, 1, 16), 128, 0, st>>>(cfg, pbc, m.pb[Rn].particle_bucket_sizes, m.pb[Rn].blockbuckets);
		++s->launches;
	}
	if(src.vel) {
		keep_velocity_kernel<<<grid_for(src.vel_count, 8, 16), 256, 0, st>>>(cfg, src.vel_count, src.vel_keys, src.vel, s->part[R].index_table, nbc, s->grid[0]);
		++s->launches;
	}
	CK(cudaGetLastError());
	if(mgsp && !src.grid) {  // the rasterised halo blocks are partial sums: reduce them (mgsp_benchmark.cuh:653-654, 723-776)
		mgsp_pack_send_kernel<<<grid_blocks(2), 256, 0, st>>>(cfg, mgsp_view(s), s->grid[0], s->part[R].index_table);
		mgsp_wait_reduce_kernel<<<grid_blocks(2), 256, 0, st>>>(cfg, mgsp_view(s), s->grid[0], s->part[R].index_table, err);
		s->launches += 2;
		CK(cudaGetLastError());
	}
	// device-resident step state
	CK(pull_state(s));
	StepState& h = *s->h_state;
	h.pbc = pbc;
	h.nbc = nbc;
	h.ebc = ebc;
	h.prev_nbc = nbc;
	h.prev_ebc = ebc;
	h.dt_default = s->desc.dt_default;
	Clock c {};
	if(src.clock) {
		c = *src.clock;
	} else {  // main_loop's preamble (gmpm_simulator.cuh:305-315)
		c.frame_time = s->desc.fps > 0 ? 1.f / (float) s->desc.fps : 0.f;
		float mv = 0.f;
		for(const Model& m : s->models) mv = fmaxf(mv, sqrtf(m.v0[0] * m.v0[0] + m.v0[1] * m.v0[1] + m.v0[2] * m.v0[2]));
		if(mgsp) {  // every rank must start from the same dt: max over the ranks' initial speeds
			h.max_vel_sq = mv * mv;
			CK(push_state(s));
			mgsp_allreduce_maxvel_kernel<<<1, 32, 0, st>>>(mgsp_view(s), &s->d_state->max_vel_sq);
			++s->launches;
			CK(pull_state(s));
			mv = sqrtf(h.max_vel_sq);
		}
		c.dt = cfl_dt(cfg, h.dt_default, mv);
		if(c.frame_time > 0.f) c.dt = fminf(c.dt, c.frame_time);
		c.next_dt = c.dt;
	}
	set_clock(h, s->frames_done, c);
	h.max_vel_sq = 0.f;
	CK(push_state(s));
	if(mgsp) {
		// global max |v|^2 of the start grid (later sub-steps get it from the end-of-step exchange of the previous one)
		launch_grid_max(cfg, s->d_state, s->grid[0], s->part[R].active_keys, &s->d_state->max_vel_sq, s->boundaries, s->levelsets, grid_blocks(2), st, &s->tracks);
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
	if(!s) return (int) cudaErrorInvalidValue;
	CK(setup_impl(s, s->restore.start()));
	s->restore.release();  // (setup_impl has synchronised: a staged state is in the bins and the grid now)
	return force_reset(s);  // a restore starts the report's span at the restored clock; adding or removing particles keeps the sums
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

// The sub-step graphs hold the grid-update and carry launches of the collider and object state they were captured with, and the
// g2p2g launches of the material parameters: drop them and,
// once set up, instantiate both roll parities again right away (never later, while an MGSP peer may be waiting on this rank).
static int recapture(cb200_sim* s) {
	drop_graphs(s);
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
	s->boundaries.col = *params;
	s->boundaries.col.sdf = s->sdf;
	s->boundaries.has_collider = true;
	CK(force_reset(s));
	return recapture(s);
}
int cb200_sim_clear_collider(cb200_sim* s) {
	if(!s) return (int) cudaErrorInvalidValue;
	CK(cudaStreamSynchronize(s->stream));
	s->boundaries.has_collider = false;
	s->boundaries.col = ColliderView {};
	g_pool.release(s->sdf);
	s->sdf = nullptr;
	CK(force_reset(s));
	return recapture(s);
}
int cb200_sim_set_collision_objects(cb200_sim* s, const cb200_collision_object* objs, int n) {
	ObjectList l;
	if(!s || !objects_prepare(objs, n, l, s->levelsets.count)) return (int) cudaErrorInvalidValue;
	CK(cudaStreamSynchronize(s->stream));
	s->boundaries.objects = l;
	for(int i = 0; i < CB200_MAX_COLLISION_OBJECTS; ++i) s->track_keys[i].clear();  // a new list: every track is cleared
	s->tracks = Tracks {};
	CK(force_reset(s));
	return recapture(s);
}
// ---- motion tracks (DESIGN.md section 2.14) -----------------------------------------------------------------------------------
int cb200_sim_set_object_track(cb200_sim* s, int object, const cb200_track_key* keys, int n, int flags) {
	if(!s || object < 0 || object >= s->boundaries.objects.n || n < 0 || n > CB200_MAX_TRACK_KEYS) return (int) cudaErrorInvalidValue;
	std::vector<cb200_track_record> rec((size_t) n);
	if(n > 0 && (!track_object_ok(s->boundaries.objects.o[object]) || !track_prepare(keys, n, flags, rec.data()))) return (int) cudaErrorInvalidValue;
	size_t total = rec.size();
	for(int i = 0; i < s->boundaries.objects.n; ++i)
		if(i != object) total += s->track_keys[i].size();
	if(total > CB200_MAX_TRACK_KEYS) return (int) cudaErrorInvalidValue;
	// the table in object order, and the spans into it
	std::vector<cb200_track_record> table;
	table.reserve(total);
	Tracks tr {};
	tr.rec = reinterpret_cast<const float4*>(s->track_table);
	for(int i = 0; i < s->boundaries.objects.n; ++i) {
		const std::vector<cb200_track_record>& k = i == object ? rec : s->track_keys[i];
		tr.off[i] = (int) table.size();
		tr.n[i] = (int) k.size();
		tr.flags[i] = i == object ? flags : s->track_flags[i];
		table.insert(table.end(), k.begin(), k.end());
	}
	CK(cudaStreamSynchronize(s->stream));
	if(!table.empty()) {
		CK(cudaMemcpyAsync(s->track_table, table.data(), table.size() * sizeof(cb200_track_record), cudaMemcpyHostToDevice, s->stream));
		CK(cudaStreamSynchronize(s->stream));
	}
	s->track_keys[object] = std::move(rec);
	s->track_flags[object] = flags;
	s->tracks = tr;
	CK(force_reset(s));
	return recapture(s);
}
// phi is uploaded into scratch, the lattice built from it on the device; the registry takes the lattice only once it is complete
int cb200_sim_add_collision_levelset(cb200_sim* s, const cb200_sdf_header* header, const float* phi_host, int* id) {
	if(!s || !levelset_dims_valid(header) || !std::isfinite(header->h) || !(header->h > 0.f) || !phi_host || s->levelsets.count >= CB200_MAX_COLLISION_LEVELSETS)
		return (int) cudaErrorInvalidValue;
	CK(cudaStreamSynchronize(s->stream));
	const size_t nodes = (size_t) header->ni * header->nj * header->nk;
	float* phi = nullptr;
	float* lattice = nullptr;
	cudaError_t e = pool_alloc(&phi, nodes * sizeof(float));
	if(e == cudaSuccess) e = pool_alloc(&lattice, nodes * 4 * sizeof(float));
	if(e == cudaSuccess) e = cudaMemcpyAsync(phi, phi_host, nodes * sizeof(float), cudaMemcpyHostToDevice, s->stream);
	if(e == cudaSuccess) e = launch_levelset_prepare(*header, phi, lattice, s->stream);
	if(e == cudaSuccess) e = cudaStreamSynchronize(s->stream);
	g_pool.release(phi);
	if(e != cudaSuccess) {
		g_pool.release(lattice);
		return (int) e;
	}
	s->launches += 1;
	const int k = s->levelsets.count++;
	s->levelsets.v[k] = cb200_levelset {lattice, header->ni, header->nj, header->nk};
	if(id) *id = k;
	return recapture(s);
}
int cb200_sim_clear_collision_levelsets(cb200_sim* s) {
	if(!s || has_levelset_objects(s->boundaries)) return (int) cudaErrorInvalidValue;
	CK(cudaStreamSynchronize(s->stream));
	for(int i = 0; i < s->levelsets.count; ++i) g_pool.release(const_cast<float*>(s->levelsets.v[i].lattice));
	s->levelsets = LevelSets {};
	return recapture(s);
}
int cb200_sim_time(cb200_sim* s, double* time) {
	if(!s || !time) return (int) cudaErrorInvalidValue;
	CK(pull_state(s));
	*time = s->h_state->sim_time;
	return 0;
}
// ---- the boundary impulse report (DESIGN.md section 2.13) ---------------------------------------------------------------------
int cb200_sim_set_force_report(cb200_sim* s, int enable) {
	if(!s) return (int) cudaErrorInvalidValue;
	CK(cudaStreamSynchronize(s->stream));
	s->force_report = enable != 0;
	CK(force_reset(s));
	return recapture(s);
}
int cb200_sim_collision_forces(cb200_sim* s, double* out, int capacity, int* n_bodies, double* elapsed) {
	const int rows = s ? 1 + s->boundaries.objects.n : 0;
	if(!s || !s->force_report || !out || !n_bodies || !elapsed || capacity < rows) return (int) cudaErrorInvalidValue;
	constexpr size_t n = (size_t) kForceBodies * kForceComps;
	double h[n + 1];
	CK(cudaMemcpyAsync(h, s->forces, sizeof(h), cudaMemcpyDeviceToHost, s->stream));
	CK(pull_state(s));  // synchronises
	memcpy(out, h, (size_t) rows * kForceComps * sizeof(double));
	*n_bodies = rows;
	*elapsed = s->h_state->sim_time - h[n];
	return force_reset(s);
}

// ---- checkpoint / restore (format and kernels: checkpoint.cuh) ---------------------------------------------------------------
int cb200_checkpoint_inspect(const void* blob, size_t bytes, cb200_checkpoint_info* info) { return ck_parse(blob, bytes, info); }

}  // extern "C"
namespace {
// the checkpoint layout of the simulator's models with counts[m] particles each and nbc grid blocks
CkLayout models_layout(const cb200_sim* s, const long long* counts, long long nbc) {
	int mats[kMaxModels];
	for(size_t m = 0; m < s->models.size(); ++m) mats[m] = s->models[m].material;
	return ck_layout((int) s->models.size(), mats, counts, nbc);
}
size_t ck_capacity(const cb200_sim* s) {
	long long counts[kMaxModels];
	for(size_t m = 0; m < s->models.size(); ++m) counts[m] = s->models[m].n;
	return (size_t) models_layout(s, counts, s->desc.max_blocks).total;
}
// model m's row of ck_base: the exclusive scan of its bucket sizes, entry pbc its particle count
int* ck_row(const cb200_sim* s, int m) { return s->ck_base + (size_t) m * (s->desc.max_blocks + 1); }

// The row each particle block of model m starts at in every read-out: an exclusive scan of the bucket sizes of the current
// partition into ck_row (entry pbc and model_count[m]: the model's count), enqueued on the sim stream
int enqueue_bucket_scan(cb200_sim* s, int m) {
	ScanArgs sc {};
	sc.count = count_dev(&s->d_state->pbc);
	sc.count_plus = 1;
	sc.in = s->models[m].pb[s->rollid ^ 1].particle_bucket_sizes;
	sc.out = ck_row(s, m);
	sc.total_out = &s->scr->model_count[m];
	scan_kernel<<<1, 1024, 0, s->stream>>>(sc);
	++s->launches;
	return (int) cudaGetLastError();
}
// the current state's particles as the gathers read them, every model's rows placed by its bucket scan
GatherSrc gather_src(const cb200_sim* s) {
	const int R = s->rollid, Rn = R ^ 1;
	GatherSrc g {};
	g.n_models = (int) s->models.size();
	for(int m = 0; m < g.n_models; ++m) {
		const Model& md = s->models[m];
		g.material[m] = md.material;
		g.cur[m] = view(md.pb[R]);
		g.next[m] = view(md.pb[Rn]);
		g.base[m] = ck_row(s, m);
		g.cap[m] = md.n;
	}
	g.keys = s->part[R].active_keys;
	g.prev_table = s->part[Rn].index_table;
	return g;
}

// every model's particle count from the bucket scans queued before (synchronises)
int read_totals(cb200_sim* s, long long* counts) {
	const int nm = (int) s->models.size();
	int totals[kMaxModels] = {};
	CK(cudaMemcpyAsync(totals, s->scr->model_count, nm * sizeof(int), cudaMemcpyDeviceToHost, s->stream));
	CK(cudaStreamSynchronize(s->stream));
	for(int m = 0; m < nm; ++m) {
		if(totals[m] < 0 || totals[m] > s->models[m].n) return (int) cudaErrorIllegalState;
		counts[m] = totals[m];
	}
	return 0;
}

// A read-out of every model (the checkpoint's and the emission's snapshot_kernel, the frame's output_kernel): the bucket scans and the
// gather `kernel` over `a` (its cfg, state and src filled in here) on the sim stream, then the step state and every model's count.
// The host has waited for the gather when this returns, so a copy of its staging queued on another stream needs no event behind it.
template<class Args>
int read_out(cb200_sim* s, void (*kernel)(Args), Args a, long long* counts) {
	for(int m = 0; m < (int) s->models.size(); ++m) CK(enqueue_bucket_scan(s, m));
	a.cfg = s->cfg;
	a.state = s->d_state;
	a.src = gather_src(s);
	kernel<<<num_sms() * 8, kGatherThreads, 0, s->stream>>>(a);
	++s->launches;
	CK(cudaGetLastError());
	CK(pull_state(s));
	return read_totals(s, counts);
}

// output_model (gmpm_simulator.cuh:594-634): one model's rows -> host, in the order of the checkpoint's section of that model.  The
// staging persists (the reference borrows and re-allocates per frame) and the device->host copy lands in pinned memory; `host` ==
// nullptr returns the pinned mirror itself.
int retrieve_impl(cb200_sim* s, int model, float* host, bool positions, int* n_out, const float** pinned_out) {
	if(!s || !s->setup_done || model < 0 || model >= (int) s->models.size()) return (int) cudaErrorInvalidValue;
	Model& m = s->models[model];
	const size_t bytes = (size_t) m.n * (positions ? 3 : ck_channels(m.material)) * sizeof(float);
	CK(m.out.grow(bytes, !host));
	CK(enqueue_bucket_scan(s, model));
	float* out = reinterpret_cast<float*>(m.out.dev);
	if(positions)
		state_rows_kernel<true><<<num_sms() * 8, kGatherThreads, 0, s->stream>>>(s->cfg, s->d_state, gather_src(s), model, out);
	else
		state_rows_kernel<false><<<num_sms() * 8, kGatherThreads, 0, s->stream>>>(s->cfg, s->d_state, gather_src(s), model, out);
	++s->launches;
	CK(cudaGetLastError());
	// the count is only known on the device: copy the full staging buffer behind the kernel, read the count with it
	CK(cudaMemcpyAsync(host ? (void*) host : m.out.host, m.out.dev, bytes, cudaMemcpyDeviceToHost, s->stream));
	int n = 0;
	CK(cudaMemcpyAsync(&n, &s->scr->model_count[model], sizeof(int), cudaMemcpyDeviceToHost, s->stream));
	CK(cudaStreamSynchronize(s->stream));
	if(n > m.n) n = m.n;
	if(pinned_out) *pinned_out = reinterpret_cast<const float*>(m.out.host);
	if(n_out) *n_out = n;
	return 0;
}
}  // namespace
extern "C" {

int cb200_sim_retrieve(cb200_sim* s, int model, float* positions_host, int* n_out) { return retrieve_impl(s, model, positions_host, true, n_out, nullptr); }
// zero-copy variant: *positions_pinned points at the simulator's pinned staging buffer (valid until the next retrieve of that model)
int cb200_sim_retrieve_pinned(cb200_sim* s, int model, const float** positions_pinned, int* n_out) { return retrieve_impl(s, model, nullptr, true, n_out, positions_pinned); }
int cb200_sim_particle_state(cb200_sim* s, int model, float* state_host, int* n_out) { return retrieve_impl(s, model, state_host, false, n_out, nullptr); }

int cb200_sim_checkpoint_begin(cb200_sim* s, size_t* bytes) {
	if(!s || !s->setup_done) return (int) cudaErrorInvalidValue;
	for(const Model& m : s->models)
		if(m.n == 0) return (int) cudaErrorNotSupported;  // format version 1 holds no empty model
	CK(s->ck.wait());  // the pinned blob and the staging blob are re-used
	s->ck_bytes = 0;
	CK(s->ck.open_stream());
	CK(s->ck.grow(ck_capacity(s), true));
	// the counts the layout follows from: the step state (pbc, nbc, clock), then each model's total
	SnapshotArgs a {};
	a.grid = s->grid[0];
	a.out = s->ck.dev;
	long long counts[kMaxModels];
	CK(read_out(s, snapshot_kernel, a, counts));
	const int nm = (int) s->models.size();
	const StepState& h = *s->h_state;
	const CkLayout L = models_layout(s, counts, h.nbc);
	cb200_checkpoint_info I;
	memset(&I, 0, sizeof(I));
	I.version = CB200_CHECKPOINT_VERSION;
	I.n_models = nm;
	I.bytes = L.total;
	I.cfg = s->desc.cfg;
	I.dt_default = s->desc.dt_default;
	I.fps = s->desc.fps;
	I.mgsp_rank = s->desc.mgsp_world > 1 ? s->desc.mgsp_rank : 0;
	I.mgsp_world = s->desc.mgsp_world;
	const Clock c = clock_of(h, s->frames_done);
	I.error = c.error;
	I.dt = c.dt;
	I.next_dt = c.next_dt;
	I.step_time = c.step_time;
	I.frame_time = c.frame_time;
	I.sim_time = c.sim_time;
	I.steps = c.steps;
	I.frames = c.frames;
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
		md.material = s->models[m].material;
		md.channels = ck_channels(md.material);
		md.count = counts[m];
		md.offset = L.model_off[m];
		md.bytes = L.model_bytes[m];
		md.params = s->models[m].pb[0];  // (ck_write_header writes the parameters only)
	}
	ck_write_header(s->ck.host, I);
	// the data sections: on the copy stream (the snapshot has finished), so that sub-steps enqueued from here on run alongside
	CK(cudaMemcpyAsync(s->ck.host + kCkHeader, s->ck.dev + kCkHeader, L.total - kCkHeader, cudaMemcpyDeviceToHost, s->ck.stream));
	CK(cudaEventRecord(s->ck.copied, s->ck.stream));
	s->ck.pending = true;
	s->ck_bytes = L.total;
	if(bytes) *bytes = L.total;
	return 0;
}

int cb200_sim_checkpoint_end(cb200_sim* s, const void** blob, size_t* bytes) {
	if(!s || !s->ck_bytes) return (int) cudaErrorInvalidValue;
	CK(s->ck.wait());
	if(blob) *blob = s->ck.host;
	if(bytes) *bytes = s->ck_bytes;
	return 0;
}

int cb200_sim_restore_models(cb200_sim* s, const void* blob, size_t bytes) {
	cb200_checkpoint_info I;
	if(!s || s->setup_done || s->restore.pending || !s->models.empty() || ck_parse(blob, bytes, &I) != 0) return (int) cudaErrorInvalidValue;
	output_idle(s);
	const cb200_config& c = s->desc.cfg;
	if(c.domain_bits != I.cfg.domain_bits || c.max_ppc != I.cfg.max_ppc || c.boundary != I.cfg.boundary || memcmp(&c.gravity, &I.cfg.gravity, sizeof(float)) != 0 ||
	   memcmp(&c.cfl, &I.cfg.cfl, sizeof(float)) != 0 || memcmp(&s->desc.dt_default, &I.dt_default, sizeof(float)) != 0 || s->desc.fps != I.fps ||
	   s->desc.mgsp_world != I.mgsp_world || (s->desc.mgsp_world > 1 ? s->desc.mgsp_rank : 0) != I.mgsp_rank)
		return (int) cudaErrorInvalidValue;
	if(s->desc.max_blocks < I.exterior_block_count) return (int) cudaErrorMemoryAllocation;
	const unsigned char* src = static_cast<const unsigned char*>(blob);
	cudaStream_t st = s->stream;
	RestoreStaging& rs = s->restore;
	rs.pending = true;
	rs.clock = Clock {I.dt, I.next_dt, I.step_time, I.frame_time, I.sim_time, I.steps, I.frames, I.error};
	rs.counts = BlockCounts {I.particle_block_count, I.neighbor_block_count, I.exterior_block_count};
	for(int m = 0; m < I.n_models; ++m) {
		const cb200_checkpoint_model& md = I.models[m];
		CK(add_model(s, md.material, (int) md.count, nullptr, nullptr, [&](Model& model) {
			for(cb200_particle_buffer& pb : model.pb) copy_params(pb, md.params);
			CK(pool_alloc(&rs.rows[m], md.bytes));
			CK(cudaMemcpyAsync(rs.rows[m], src + md.offset, md.bytes, cudaMemcpyHostToDevice, st));
			state_positions_kernel<<<num_sms() * 4, 256, 0, st>>>(md.count, md.channels, rs.rows[m], model.d_pos);
			++s->launches;
			return (int) cudaGetLastError();
		}));
	}
	rs.grid_bytes = I.grid_bytes;
	CK(pool_alloc(&rs.grid, (size_t) I.grid_bytes + (size_t) I.keys_bytes));
	CK(cudaMemcpyAsync(rs.grid, src + I.grid_offset, I.grid_bytes, cudaMemcpyHostToDevice, st));
	CK(cudaMemcpyAsync(rs.grid + I.grid_bytes, src + I.keys_offset, I.keys_bytes, cudaMemcpyHostToDevice, st));
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
	CK(s->out.open_stream());
	const int W = out_words(attributes);
	OutputArgs a {};
	size_t need = 0;
	for(int m = 0; m < nm; ++m) {  // a section per model, sized for all its particles
		a.off[m] = need;
		need += (size_t) s->models[m].n * W * sizeof(float);
	}
	CK(s->out.grow(need, true));
	a.attrs = attributes;
	a.table = s->part[s->rollid].index_table;
	a.grid = s->grid[0];
	a.out = s->out.dev;
	// the counts the headers need (each model's total): this is the only wait, and it ends with the gather
	long long totals[kMaxModels];
	CK(read_out(s, output_kernel, a, totals));
	std::vector<cb200_sim::OutputFile> files((size_t) nm);
	for(int m = 0; m < nm; ++m) {
		files[m].path = paths[m];
		files[m].header = bgeo_header(totals[m], attributes);
		files[m].body = s->out.host + a.off[m];
		files[m].body_bytes = (size_t) totals[m] * W * sizeof(float);
		if(files[m].body_bytes) CK(cudaMemcpyAsync(s->out.host + a.off[m], s->out.dev + a.off[m], files[m].body_bytes, cudaMemcpyDeviceToHost, s->out.stream));
	}
	CK(cudaEventRecord(s->out.copied, s->out.stream));
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

// ---- particle models from level sets (format, plan and kernels: sdf.cuh) -------------------------------------------------------------
}  // extern "C"
namespace {
// One sampling run: phi on the device, the valid-cell list (random mode) and the tile offsets of the last count, all from the pool.
// count() runs the passes up to the particle count; write() fills `out` (device) in candidate / lattice-point order.
struct SdfRun {
	SdfPlan P {};
	cudaStream_t st = nullptr;
	float* phi = nullptr;
	int* list = nullptr;
	long long* tile_off = nullptr;
	unsigned* done = nullptr;
	SdfScan scan {};
	int tiles = 0;
	long long count = 0;
	SdfRandom rnd {};
	SdfLattice lat {};
	~SdfRun() {
		g_pool.release(phi);
		g_pool.release(list);
		g_pool.release(tile_off);
		g_pool.release(done);
	}
	// the count kernel over n_items: scan / tiles describe the launch, *total the kept items
	template<class G>
	int count_pass(const G& g, long long n_items, long long* total) {
		*total = 0;
		if(n_items <= 0) return 0;
		g_pool.release(tile_off);
		tile_off = nullptr;
		// at most 64 Ki tiles, so the last CTA's scan stays short
		const long long per_round = kSdfThreads, min_rounds = (n_items + 65536LL * per_round - 1) / (65536LL * per_round);
		scan.n_items = n_items;
		scan.rounds = (int) std::max<long long>(8, min_rounds);
		tiles = (int) ((n_items + per_round * scan.rounds - 1) / (per_round * scan.rounds));
		CK(pool_alloc(&tile_off, (size_t) (tiles + 1) * sizeof(long long)));
		scan.tile_off = tile_off;
		scan.done = done;
		CK(cudaMemsetAsync(done, 0, sizeof(unsigned), st));
		sdf_count_kernel<G><<<tiles, kSdfThreads, 0, st>>>(g, scan);
		CK(cudaGetLastError());
		CK(cudaMemcpyAsync(total, tile_off + tiles, sizeof(long long), cudaMemcpyDeviceToHost, st));
		return (int) cudaStreamSynchronize(st);
	}
	template<class G>
	int write_pass(const G& g) {
		if(!tiles) return 0;
		sdf_write_kernel<G><<<tiles, kSdfThreads, 0, st>>>(g, scan);
		return (int) cudaGetLastError();
	}
	int run_count(const cb200_config& cfg, const cb200_sdf_header& hdr, const float* phi_host, const cb200_sdf_sampling& smp) {
		if(!phi_host) return (int) cudaErrorInvalidValue;
		CK(sdf_plan(cfg, hdr, smp, P));
		const size_t nodes = (size_t) hdr.ni * hdr.nj * hdr.nk;
		CK(pool_alloc(&phi, nodes * sizeof(float)));
		CK(pool_alloc(&done, sizeof(unsigned)));
		CK(cudaMemcpyAsync(phi, phi_host, nodes * sizeof(float), cudaMemcpyHostToDevice, st));
		const SdfField f {phi, hdr.ni, hdr.nj};
		if(P.mode == CB200_SDF_LATTICE) {
			lat.f = f;
			lat.nk = hdr.nk;
			lat.k = P.k;
			for(int d = 0; d < 3; ++d) {
				lat.lo[d] = P.lo[d];
				lat.ext[d] = P.ext[d];
				lat.off[d] = P.offset[d];
			}
			lat.dx = P.dx;
			lat.c = P.c;
			return count_pass(lat, P.lattice_items, &count);
		}
		SdfClassify cls {f, nullptr};
		long long n_valid = 0;
		CK(count_pass(cls, (long long) (hdr.ni - 1) * (hdr.nj - 1) * (hdr.nk - 1), &n_valid));
		if(!n_valid) return 0;
		CK(pool_alloc(&list, (size_t) n_valid * sizeof(int)));
		cls.list = list;
		CK(write_pass(cls));
		const double cand = std::floor((double) n_valid * P.spc);
		if(!(cand < 0x1p62)) return (int) cudaErrorInvalidValue;
		rnd.f = f;
		rnd.list = list;
		rnd.n_valid = n_valid;
		rnd.spc = P.spc;
		rnd.c = P.c;
		for(int d = 0; d < 3; ++d) rnd.off[d] = P.offset[d];
		rnd.key = make_uint2((unsigned) smp.seed, (unsigned) (smp.seed >> 32));
		return count_pass(rnd, (long long) cand, &count);
	}
	int run_write(float* out) {
		if(P.mode == CB200_SDF_LATTICE) {
			lat.out = out;
			return write_pass(lat);
		}
		rnd.out = out;
		return write_pass(rnd);
	}
};
}  // namespace
extern "C" {

int cb200_sdf_parse(const char* text, size_t bytes, cb200_sdf_header* header, float* phi, size_t capacity) {
	return sdf_parse(text, bytes, header, phi, capacity);
}

int cb200_sample_sdf(const cb200_config* cfg, const cb200_sdf_header* header, const float* phi_host, const cb200_sdf_sampling* sampling,
                     float* pos_host, long long capacity, long long* n_out, void* stream) {
	if(!cfg || !cfg_valid(*cfg) || !header || !sampling || !n_out) return (int) cudaErrorInvalidValue;
	SdfRun r;
	r.st = (cudaStream_t) stream;
	CK(r.run_count(*cfg, *header, phi_host, *sampling));
	*n_out = r.count;
	if(!pos_host || !r.count) return 0;
	if(capacity < r.count) return (int) cudaErrorInvalidValue;
	float* staging = nullptr;
	CK(pool_alloc(&staging, (size_t) r.count * 3 * sizeof(float)));
	int e = r.run_write(staging);
	if(!e) e = (int) cudaMemcpyAsync(pos_host, staging, (size_t) r.count * 3 * sizeof(float), cudaMemcpyDeviceToHost, r.st);
	if(!e) e = (int) cudaStreamSynchronize(r.st);
	g_pool.release(staging);
	return e;
}

int cb200_sim_init_model_sdf(cb200_sim* s, int material, const cb200_sdf_header* header, const float* phi_host, const cb200_sdf_sampling* sampling,
                             const float* v0, int* model_id, int* n_out) {
	if(!s || s->setup_done || material < 0 || material > 3 || (int) s->models.size() >= kMaxModels || !header || !sampling) return (int) cudaErrorInvalidValue;
	SdfRun r;
	r.st = s->stream;
	CK(r.run_count(s->desc.cfg, *header, phi_host, *sampling));
	if(r.count <= 0 || r.count >= (1LL << 31)) return (int) cudaErrorInvalidValue;
	CK(add_model(s, material, (int) r.count, v0, model_id, [&](Model& m) { return r.run_write(m.d_pos); }));
	if(n_out) *n_out = (int) r.count;
	return 0;
}

// ---- level sets from triangle meshes (kernels: mesh.cuh) --------------------------------------------------------------------------
}  // extern "C"
namespace {
// every device buffer of one build, from the pool and back to it
struct MeshRun {
	float* x = nullptr;
	int* tri = nullptr;
	MeshTri* boxes = nullptr;
	longlong2* counts = nullptr;  // per triangle (band nodes, crossing columns)
	longlong2* offs = nullptr;    // [nt + 1] their exclusive prefix
	longlong2* tile = nullptr;
	unsigned* done = nullptr;
	unsigned long long* packed = nullptr;  // per node: phi bits << 32 | closest triangle
	int* cross = nullptr;                  // per node: crossings in (i - 1, i], then phi
	~MeshRun() {
		for(void* p : {(void*) x, (void*) tri, (void*) boxes, (void*) counts, (void*) offs, (void*) tile, (void*) done, (void*) packed, (void*) cross}) g_pool.release(p);
	}
};

// one CTA per SM: a plane holds at most a few nodes per thread, and the grid barrier, paid 16 (ni + nj + nk) times, costs more
// the more CTAs it joins
int mesh_sweep_grid() { return num_sms(); }
}  // namespace
extern "C" {

int cb200_obj_parse(const char* text, size_t bytes, cb200_mesh_header* header, float* vertices, int* triangles, size_t v_capacity, size_t t_capacity) {
	return obj_parse(text, bytes, header, vertices, triangles, v_capacity, t_capacity);
}

int cb200_mesh_levelset(const float* vertices, int nv, const int* triangles, int nt, const cb200_mesh_levelset_params* params, cb200_sdf_header* out,
                        float* phi, size_t capacity, void* stream) {
	if(!params || !out) return (int) cudaErrorInvalidValue;
	cb200_sdf_header hdr {};
	CK(mesh_header(vertices, nv, triangles, nt, *params, hdr));
	const long long nodes = (long long) hdr.ni * hdr.nj * hdr.nk;
	if(phi && capacity < (size_t) nodes) return (int) cudaErrorInvalidValue;
	*out = hdr;
	if(!phi) return 0;
	const cudaStream_t st = (cudaStream_t) stream;
	MeshRun r;
	const int tiles = (nt + kMeshThreads * kMeshScanPer - 1) / (kMeshThreads * kMeshScanPer);
	CK(pool_alloc(&r.x, (size_t) nv * 3 * sizeof(float)));
	CK(pool_alloc(&r.tri, (size_t) nt * 3 * sizeof(int)));
	CK(pool_alloc(&r.boxes, (size_t) nt * sizeof(MeshTri)));
	CK(pool_alloc(&r.counts, (size_t) nt * sizeof(longlong2)));
	CK(pool_alloc(&r.offs, (size_t) (nt + 1) * sizeof(longlong2)));
	CK(pool_alloc(&r.tile, (size_t) tiles * sizeof(longlong2)));
	CK(pool_alloc(&r.done, sizeof(unsigned)));
	CK(pool_alloc(&r.packed, (size_t) nodes * sizeof(unsigned long long)));
	CK(pool_alloc(&r.cross, (size_t) nodes * sizeof(int)));
	CK(cudaMemcpyAsync(r.x, vertices, (size_t) nv * 3 * sizeof(float), cudaMemcpyHostToDevice, st));
	CK(cudaMemcpyAsync(r.tri, triangles, (size_t) nt * 3 * sizeof(int), cudaMemcpyHostToDevice, st));
	CK(cudaMemsetAsync(r.done, 0, sizeof(unsigned), st));
	MeshGeom g {r.x, r.tri, nt, hdr.min[0], hdr.min[1], hdr.min[2], hdr.h, hdr.ni, hdr.nj, hdr.nk};
	// phi.assign((ni+nj+nk)*dx): int times float
	const float init = (float) (hdr.ni + hdr.nj + hdr.nk) * hdr.h;
	mesh_init_kernel<<<grid_for(nodes, kMeshThreads), kMeshThreads, 0, st>>>(nodes, mesh_pack(init, -1), r.packed, r.cross);
	mesh_setup_kernel<<<(nt + kMeshThreads - 1) / kMeshThreads, kMeshThreads, 0, st>>>(g, params->exact_band, r.boxes, r.counts);
	const MeshScan sc {r.counts, r.offs, r.tile, r.done, nt};
	mesh_scan_tiles_kernel<<<tiles, kMeshThreads, 0, st>>>(sc);
	mesh_scan_write_kernel<<<tiles, kMeshThreads, 0, st>>>(sc);
	CK(cudaGetLastError());
	longlong2 total {};
	CK(cudaMemcpyAsync(&total, r.offs + nt, sizeof(longlong2), cudaMemcpyDeviceToHost, st));
	CK(cudaStreamSynchronize(st));
	mesh_band_kernel<<<grid_for(total.x, kMeshThreads), kMeshThreads, 0, st>>>(g, r.boxes, r.offs, init, r.packed);
	if(total.y) mesh_cross_kernel<<<grid_for(total.y, kMeshThreads), kMeshThreads, 0, st>>>(g, r.boxes, r.offs, r.cross);
	CK(cudaGetLastError());
	void* args[] = {(void*) &g, (void*) &r.packed};
	CK(cudaLaunchCooperativeKernel((const void*) mesh_sweep_kernel, mesh_sweep_grid(), kMeshThreads, args, 0, st));
	mesh_sign_kernel<<<grid_for((long long) hdr.nj * hdr.nk * 32, kMeshThreads), kMeshThreads, 0, st>>>(g, r.packed, r.cross);
	CK(cudaGetLastError());
	CK(cudaMemcpyAsync(phi, r.cross, (size_t) nodes * sizeof(float), cudaMemcpyDeviceToHost, st));
	return (int) cudaStreamSynchronize(st);
}

// ---- adding particles at a sub-step boundary (kernels: emit.cuh) ----------------------------------------------------------------------
}  // extern "C"
namespace {
// every buffer one call allocates; what the commit swaps out of the model (its old bins and positions) lands here and goes back too
struct EmitBuffers {
	float* cand = nullptr;  // [n][3] candidates
	int* keep = nullptr;    // [n]
	int* offs = nullptr;    // [n + 1] exclusive scan of keep
	float* kept = nullptr;  // [k][3] kept candidates, in candidate order
	int* word = nullptr;    // [0] scratch partition count, [1] kEmit* bits
	int* table = nullptr;   // scratch partition of the union: table, keys
	int* keys = nullptr;
	int* cells = nullptr;   // [union pbc][64] new particles per cell
	unsigned char* blob = nullptr;  // the gathered state, checkpoint layout
	float* rows = nullptr;  // the model's rows with the new ones appended
	float* bins[2] = {nullptr, nullptr};
	float* pos = nullptr;
	~EmitBuffers() {
		for(void* p : {(void*) cand, (void*) keep, (void*) offs, (void*) kept, (void*) word, (void*) table, (void*) keys, (void*) cells, (void*) blob, (void*) rows,
		               (void*) bins[0], (void*) bins[1], (void*) pos})
			g_pool.release(p);
	}
};

// The live state of every model, gathered (checkpoint layout) into a blob from the pool that the caller releases: each model's count
// and the layout of the sections, for the grid of nbc blocks.  Reads the live state only.
int gather_live(cb200_sim* s, long long nbc, unsigned char** blob, long long* counts, CkLayout* L) {
	CK(pool_alloc(blob, ck_capacity(s)));
	SnapshotArgs sa {};
	sa.grid = s->grid[0];
	sa.out = *blob;
	CK(read_out(s, snapshot_kernel, sa, counts));
	*L = models_layout(s, counts, nbc);
	return 0;
}

// The commit of an emission or a removal: model m becomes the n[m] state rows rows[m] (device), its positions follow from them (into
// its d_pos, which holds n[m] positions), and initial_setup runs over src with those rows, re-capturing the sub-step graphs.  The old
// graphs are dropped first: from here on a failure leaves a simulator that cannot step.
int commit_rows(cb200_sim* s, const long long* n, const float* const* rows, StartSrc& src) {
	drop_graphs(s);
	for(int m = 0; m < (int) s->models.size(); ++m) {
		Model& mm = s->models[m];
		mm.n = (int) n[m];
		src.rows[m] = rows[m];
		state_positions_kernel<<<num_sms() * 4, 256, 0, s->stream>>>(mm.n, ck_channels(mm.material), src.rows[m], mm.d_pos);
		++s->launches;
	}
	s->setup_done = false;
	return setup_impl(s, src);
}

int emit_precheck(cb200_sim* s, int model, unsigned flags, const float* v0) {
	if(!s) return (int) cudaErrorInvalidValue;
	if(s->desc.mgsp_world > 1) return (int) cudaErrorNotSupported;  // a rank's rebuild would have to be agreed with its peers
	if(!s->setup_done || model < 0 || model >= (int) s->models.size() || (flags & ~CB200_EMIT_EMPTY_CELLS)) return (int) cudaErrorInvalidValue;
	if(v0 && !(std::isfinite(v0[0]) && std::isfinite(v0[1]) && std::isfinite(v0[2]))) return (int) cudaErrorInvalidValue;  // NaN momentum, or dt = 0
	return 0;
}

// The shared path of both entries, with the n candidates in eb.cand.  Everything up to the commit reads the live state and writes
// scratch only, so a rejection leaves the simulator as it was.
int emit_impl(cb200_sim* s, int model, EmitBuffers& eb, int n, const float* v0, unsigned flags, int* n_added) {
	cudaStream_t st = s->stream;
	const Cfg& cfg = s->cfg;
	const int nm = (int) s->models.size();
	const float v[3] = {v0 ? v0[0] : 0.f, v0 ? v0[1] : 0.f, v0 ? v0[2] : 0.f};
	// (1) finite, inside the domain, the empty-cell filter: against the current partition's buckets
	CK(pool_alloc(&eb.keep, (size_t) n * sizeof(int)));
	CK(pool_alloc(&eb.offs, ((size_t) n + 1) * sizeof(int)));
	CK(pool_alloc(&eb.word, 4 * sizeof(int)));
	CK(cudaMemsetAsync(eb.word, 0, 4 * sizeof(int), st));
	EmitCells occ {};
	{
		const int R = s->rollid, Rn = R ^ 1;
		occ.cfg = cfg;
		occ.table = s->part[R].index_table;
		occ.pbc = &s->d_state->pbc;
		occ.n_models = nm;
		for(int m = 0; m < nm; ++m) {
			occ.offs[m] = s->models[m].celloffs[Rn];
			occ.sizes[m] = s->models[m].pb[Rn].particle_bucket_sizes;
		}
	}
	emit_filter_kernel<<<grid_for(n, 256, 16), 256, 0, st>>>(occ, n, eb.cand, (flags & CB200_EMIT_EMPTY_CELLS) ? 1 : 0, eb.keep, eb.word + 1);
	ScanArgs sc {};
	sc.count = count_imm(n);
	sc.count_plus = 1;
	sc.in = eb.keep;
	sc.out = eb.offs;
	scan_kernel<<<1, 1024, 0, st>>>(sc);
	s->launches += 2;
	CK(cudaGetLastError());
	int k = 0, bad = 0;
	CK(cudaMemcpyAsync(&k, eb.offs + n, sizeof(int), cudaMemcpyDeviceToHost, st));
	CK(cudaMemcpyAsync(&bad, eb.word + 1, sizeof(int), cudaMemcpyDeviceToHost, st));
	CK(cudaStreamSynchronize(st));
	if(bad) return (int) cudaErrorInvalidValue;
	if(k == 0) return 0;
	CK(pool_alloc(&eb.kept, (size_t) k * 3 * sizeof(float)));
	emit_compact_kernel<<<grid_for(n, 256, 16), 256, 0, st>>>(n, eb.cand, eb.keep, eb.offs, eb.kept);
	++s->launches;
	// (2) the union's partition on a scratch table: the current particle blocks first, then the candidates' blocks, then the neighbour
	// and exterior registrations of initial_setup.  Its capacity holds every block they can register, so the counts are exact.
	CK(pull_state(s));
	const StepState h0 = *s->h_state;
	const int cap_s = (int) std::min<long long>((long long) s->table_entries, 27LL * ((long long) h0.pbc + k));
	CK(pool_alloc(&eb.table, s->table_entries * sizeof(int)));
	CK(pool_alloc(&eb.keys, ((size_t) cap_s + 1) * 3 * sizeof(int)));
	CK(cudaMemsetAsync(eb.table, 0xff, s->table_entries * sizeof(int), st));
	emit_insert_keys_kernel<<<grid_for(h0.pbc, 256, 16), 256, 0, st>>>(cfg, h0.pbc, s->part[s->rollid].active_keys, eb.table, eb.keys, eb.word, cap_s);
	activate_blocks_kernel<true><<<grid_for(k, 256, 16), 256, 0, st>>>(cfg, k, eb.kept, eb.table, eb.keys, eb.word, cap_s, nullptr);
	s->launches += 2;
	BlockCounts u {};  // the union's
	CK(cudaMemcpyAsync(&u.pbc, eb.word, sizeof(int), cudaMemcpyDeviceToHost, st));
	CK(cudaStreamSynchronize(st));
	const Part scratch {eb.word, eb.table, eb.keys};
	CK(register_ring(s, scratch, cap_s, nullptr, u.pbc, 0, 2, &u.nbc));
	CK(register_ring(s, scratch, cap_s, nullptr, u.pbc, -1, 3, &u.ebc));
	// (3) no cell above max_ppc, existing and new particles together
	CK(pool_alloc(&eb.cells, (size_t) u.pbc * kBlockVol * sizeof(int)));
	CK(cudaMemsetAsync(eb.cells, 0, (size_t) u.pbc * kBlockVol * sizeof(int), st));
	emit_count_kernel<<<grid_for(k, 256, 16), 256, 0, st>>>(cfg, k, eb.kept, eb.table, eb.cells);
	emit_overflow_kernel<<<grid_for(k, 256, 16), 256, 0, st>>>(occ, k, eb.kept, eb.table, eb.cells, eb.word + 1);
	s->launches += 2;
	CK(cudaGetLastError());
	CK(cudaMemcpyAsync(&bad, eb.word + 1, sizeof(int), cudaMemcpyDeviceToHost, st));
	CK(cudaStreamSynchronize(st));
	if(bad) return (int) cudaErrorInvalidValue;
	if((long long) s->models[model].n + k > 0x7fffffffLL) return (int) cudaErrorInvalidValue;  // n bounds the model's live count
	// (4) capacity: the union's exterior blocks must fit (auto_grow: grow to 4/3 of them, after everything else that can fail)
	int new_mb = s->desc.max_blocks;
	if(u.ebc > new_mb) {
		if(!s->desc.auto_grow) return (int) cudaErrorMemoryAllocation;
		new_mb = (int) (((long long) u.ebc * 4 + 2) / 3);
	}
	// (5) gather the current state (checkpoint layout) and allocate what the commit swaps in: nothing live is written yet
	long long counts[kMaxModels];
	CkLayout L;
	CK(gather_live(s, h0.nbc, &eb.blob, counts, &L));
	Model& md = s->models[model];
	const int C = ck_channels(md.material);
	const long long n_union = counts[model] + k;
	const long long new_bins = bin_rows(n_union, new_mb);
	CK(pool_alloc(&eb.rows, (size_t) n_union * C * sizeof(float)));
	CK(pool_alloc(&eb.pos, (size_t) n_union * 3 * sizeof(float)));
	if(new_bins > md.bin_capacity)
		for(float*& bins : eb.bins) CK(pool_alloc(&bins, (size_t) new_bins * bin_floats(md.material) * sizeof(float)));
	if(L.model_bytes[model]) CK(cudaMemcpyAsync(eb.rows, eb.blob + L.model_off[model], L.model_bytes[model], cudaMemcpyDeviceToDevice, st));
	emit_rows_kernel<<<grid_for(k, 256, 16), 256, 0, st>>>(md.material, k, eb.kept, eb.rows + (size_t) counts[model] * C);
	++s->launches;
	CK(cudaGetLastError());
	CK(cudaStreamSynchronize(st));
	// the last step that can reject: cb200_sim_reserve (an out-of-memory failure there leaves a valid simulator, part-grown)
	if(new_mb > s->desc.max_blocks) CK(cb200_sim_reserve(s, new_mb));
	// (6) commit: initial_setup over the union's saved rows and grid[0], then the new particles' mass and momentum added to grid[0]
	if(eb.bins[0] && new_bins > md.bin_capacity) {  // (reserve may have grown the bins past the new count's rule already)
		for(int i = 0; i < 2; ++i) std::swap(md.pb[i].bins, eb.bins[i]);
		md.bin_capacity = new_bins;
	}
	std::swap(md.d_pos, eb.pos);
	long long n_rows[kMaxModels];
	const float* rows[kMaxModels];
	for(int m = 0; m < nm; ++m) {
		n_rows[m] = m == model ? n_union : counts[m];
		rows[m] = m == model ? eb.rows : reinterpret_cast<const float*>(eb.blob + L.model_off[m]);
	}
	StartSrc src;
	src.keys = reinterpret_cast<const int*>(eb.blob + L.keys_off);
	src.grid = reinterpret_cast<const float*>(eb.blob + L.grid_off);
	src.grid_count = h0.nbc;
	src.expect = &u;
	// the clock stays; dt and next_dt follow initial_setup's rule for v0
	Clock clock = clock_of(h0, s->frames_done);
	clock.dt = clock.next_dt = cfl_dt(cfg, h0.dt, sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]));
	src.clock = &clock;
	CK(commit_rows(s, n_rows, rows, src));
	// every stencil node of a new particle inside the domain lies in a neighbour block of its particle block; nodes past the top face
	// are dropped, as rasterize_blocks_kernel drops them
	rasterize_kernel<<<grid_for(k, 256, 16), 256, 0, st>>>(cfg, k, eb.kept, s->grid[0], s->part[s->rollid].index_table, md.pb[0].mass, v[0], v[1], v[2], nullptr);
	++s->launches;
	CK(cudaGetLastError());
	CK(cudaStreamSynchronize(st));
	if(n_added) *n_added = k;
	return 0;
}
}  // namespace
extern "C" {

int cb200_sim_add_particles(cb200_sim* s, int model, const float* positions_host, int n, const float* v0, unsigned flags, int* n_added) {
	if(n_added) *n_added = 0;
	CK(emit_precheck(s, model, flags, v0));
	if(n < 0 || (n > 0 && !positions_host)) return (int) cudaErrorInvalidValue;
	if(n == 0) return 0;
	CK(cudaStreamSynchronize(s->stream));
	EmitBuffers eb;
	CK(pool_alloc(&eb.cand, (size_t) n * 3 * sizeof(float)));
	CK(cudaMemcpyAsync(eb.cand, positions_host, (size_t) n * 3 * sizeof(float), cudaMemcpyHostToDevice, s->stream));
	return emit_impl(s, model, eb, n, v0, flags, n_added);
}

int cb200_sim_add_particles_sdf(cb200_sim* s, int model, const cb200_sdf_header* header, const float* phi_host, const cb200_sdf_sampling* sampling,
                                const float* v0, unsigned flags, int* n_added) {
	if(n_added) *n_added = 0;
	CK(emit_precheck(s, model, flags, v0));
	if(!header || !sampling) return (int) cudaErrorInvalidValue;
	CK(cudaStreamSynchronize(s->stream));
	SdfRun r;
	r.st = s->stream;
	CK(r.run_count(s->desc.cfg, *header, phi_host, *sampling));
	if(r.count >= (1LL << 31)) return (int) cudaErrorInvalidValue;
	if(r.count == 0) return 0;
	EmitBuffers eb;
	CK(pool_alloc(&eb.cand, (size_t) r.count * 3 * sizeof(float)));
	CK(r.run_write(eb.cand));
	return emit_impl(s, model, eb, (int) r.count, v0, flags, n_added);
}

// ---- removing particles at a sub-step boundary (kernels: remove.cuh) ------------------------------------------------------------------
}  // extern "C"
namespace {
// every buffer one call allocates, and the selection runs (their tile offsets)
struct RemoveBuffers {
	unsigned char* blob = nullptr;  // the gathered state, checkpoint layout
	unsigned char* mask = nullptr;  // cb200_sim_remove_rows: the host mask
	float* rows[kMaxModels] = {};   // per model with removals, the survivors' rows
	SdfRun runs[kMaxModels];
	~RemoveBuffers() {
		g_pool.release(blob);
		g_pool.release(mask);
		for(float* p : rows) g_pool.release(p);
	}
};

int remove_precheck(cb200_sim* s, long long* removed) {
	if(removed)
		for(int m = 0; m < kMaxModels; ++m) removed[m] = 0;
	if(!s) return (int) cudaErrorInvalidValue;
	if(s->desc.mgsp_world > 1) return (int) cudaErrorNotSupported;  // a rank's rebuild would have to be agreed with its peers
	return s->setup_done ? 0 : (int) cudaErrorInvalidValue;
}

// The shared path of both entries: the models of `mask` lose the rows `sel` (a RemoveRegions or RemoveMask with everything but the
// rows set) does not keep.  The gather, the selection and the compaction read the live state and write scratch only, so a rejection,
// or a call that removes nothing, leaves the simulator as it was.  mask_host / mask_n: RemoveMask's host bytes (one model).
template<class Sel>
int remove_impl(cb200_sim* s, unsigned mask, Sel sel, const unsigned char* mask_host, long long mask_n, long long* removed) {
	cudaStream_t st = s->stream;
	const int nm = (int) s->models.size();
	CK(cudaStreamSynchronize(st));
	CK(pull_state(s));
	const StepState h0 = *s->h_state;
	RemoveBuffers rb;
	long long counts[kMaxModels];
	CkLayout L;
	CK(gather_live(s, h0.nbc, &rb.blob, counts, &L));
	if constexpr(std::is_same<Sel, RemoveMask>::value) {
		if(mask_n != counts[__builtin_ctz(mask)]) return (int) cudaErrorInvalidValue;
		if(mask_n) {
			CK(pool_alloc(&rb.mask, (size_t) mask_n));
			CK(cudaMemcpyAsync(rb.mask, mask_host, (size_t) mask_n, cudaMemcpyHostToDevice, st));
		}
		sel.mask = rb.mask;
	}
	// (1) per selected model, the survivors' count
	long long n_rows[kMaxModels], live = 0, gone = 0;
	for(int m = 0; m < nm; ++m) {
		n_rows[m] = counts[m];
		if(mask >> m & 1) {
			rb.runs[m].st = st;
			CK(pool_alloc(&rb.runs[m].done, sizeof(unsigned)));
			sel.in = reinterpret_cast<const float*>(rb.blob + L.model_off[m]);
			sel.C = ck_channels(s->models[m].material);
			CK(rb.runs[m].count_pass(sel, counts[m], &n_rows[m]));
			gone += counts[m] - n_rows[m];
		}
		live += n_rows[m];
	}
	if(gone == 0) return 0;
	if(live == 0) return (int) cudaErrorInvalidValue;  // a sub-step over no particle block is not a state the driver runs
	// (2) the survivors' rows, in row order
	const float* rows[kMaxModels];
	for(int m = 0; m < nm; ++m) {
		rows[m] = reinterpret_cast<const float*>(rb.blob + L.model_off[m]);
		if(!(mask >> m & 1) || n_rows[m] == counts[m]) continue;
		sel.in = rows[m];
		sel.C = ck_channels(s->models[m].material);
		CK(pool_alloc(&rb.rows[m], (size_t) std::max(1LL, n_rows[m]) * sel.C * sizeof(float)));
		sel.out = rb.rows[m];
		CK(rb.runs[m].write_pass(sel));
		s->launches += 2;
		rows[m] = rb.rows[m];
	}
	// (3) commit: initial_setup over the survivors, grid[0] the survivors' mass at the velocities of the saved grid; the clock is kept
	StartSrc src;
	src.vel = reinterpret_cast<const float*>(rb.blob + L.grid_off);
	src.vel_keys = reinterpret_cast<const int*>(rb.blob + L.keys_off);
	src.vel_count = h0.nbc;
	const Clock clock = clock_of(h0, s->frames_done);
	src.clock = &clock;
	CK(commit_rows(s, n_rows, rows, src));
	if(removed)
		for(int m = 0; m < nm; ++m) removed[m] = counts[m] - n_rows[m];
	return 0;
}
}  // namespace
extern "C" {

int cb200_sim_remove_particles(cb200_sim* s, unsigned model_mask, const cb200_collision_object* regions, int n, unsigned flags, long long* removed) {
	CK(remove_precheck(s, removed));
	RemoveRegions sel {};
	const int nm = (int) s->models.size();
	if(!model_mask || (model_mask >> nm) || (flags & ~CB200_REMOVE_OUTSIDE) || !objects_prepare(regions, n, sel.b.objects, s->levelsets.count)) return (int) cudaErrorInvalidValue;
	if(n == 0) return 0;
	CK(cudaStreamSynchronize(s->stream));
	CK(pull_state(s));
	sel.t = (float) s->h_state->sim_time;
	sel.outside = (flags & CB200_REMOVE_OUTSIDE) ? 1 : 0;
	if(has_levelset_objects(sel.b)) {
		RemoveRegionsLevelsets lsel {};
		static_cast<RemoveRegions&>(lsel) = sel;
		lsel.ls = s->levelsets;
		return remove_impl(s, model_mask, lsel, nullptr, 0, removed);
	}
	return remove_impl(s, model_mask, sel, nullptr, 0, removed);
}

int cb200_sim_remove_rows(cb200_sim* s, int model, const unsigned char* remove_host, long long n, long long* removed) {
	CK(remove_precheck(s, removed));
	if(model < 0 || model >= (int) s->models.size() || n < 0 || (n > 0 && !remove_host)) return (int) cudaErrorInvalidValue;
	RemoveMask sel {};
	static const unsigned char kNone = 0;
	return remove_impl(s, 1u << model, sel, n ? remove_host : &kNone, n, removed);
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
