// mgsp.cuh -- multi-GPU static particle partition (MGSP) exchange kernels.
//
// Protocol of the reference (Projects/MGSP/mgsp_benchmark.cuh:421-467, 661-776; halo_kernels.cuh:22-97):
// every GPU owns a fixed particle set and its own sparse partition; grid blocks that are active on two GPUs are
// "halo" blocks whose P2G sums must be added on both owners.  Per sub-step: tag overlapping blocks from the peers'
// key lists, run g2p2g on halo particle blocks first, pack + send their next-grid blocks, run the remaining blocks
// while the transfer is in flight, add what arrived.  The reference does this with one host thread per GPU,
// cudaMemcpyPeerAsync, events and six host barriers per sub-step.
//
// This library's form (one process per GPU): every rank exposes an INBOX and its next grid through CUDA IPC.  A sub-step has no
// halo / interior split: its one g2p2g launch bulk-reduces every shared grid block straight into the peer's next grid over
// NVLink (g2p2g.cuh), and the done publish / wait pair below is the barrier behind those reductions.  At the end of the
// sub-step every rank stores its block keys and its max |v|^2 into the peers' inboxes and tags the blocks it shares with each
// peer from theirs (mgsp_clear_publish_kernel, mgsp_tag_kernel).  Whole grid blocks travel through the inbox only once, at
// setup: the halo sums of the rasterised start grid (mgsp_pack_send_kernel, mgsp_wait_reduce_kernel).
// Producers store straight into the consumer's inbox or grid over NVLink (no staging buffer, no copy engine, no host-known
// sizes), then publish an epoch flag with a system-scope release; consumers spin on their local flag with a system-scope
// acquire.  Nothing on this path returns to the host, so the whole sub-step stays a fixed kernel sequence.
// Inbox segments are double-buffered by epoch parity: a rank can be at most one exchange ahead of a peer (it needs
// the peer's flag of the previous exchange to get there).
#pragma once
#include "common.cuh"
#include "partition.cuh"

namespace cb200 {

constexpr int kMaxRanks = 8;

struct InboxHeader {   // 64 bytes, one per (parity, source rank)
	int halo_count;
	int key_count;
	float max_vel_sq;
	int flag_mv;
	int flag_halo;
	int flag_keys;
	int pad[10];
};

struct InboxLayout {
	size_t seg_bytes;      // one segment
	size_t off_halo_keys;  // int[halo_cap*3]
	size_t off_halo_blocks;// float[halo_cap*256]
	size_t off_keys;       // int[max_blocks*3]
	int halo_cap, max_blocks, world;
};

inline InboxLayout make_inbox_layout(int world, int halo_cap, int max_blocks) {
	InboxLayout L;
	auto align = [](size_t x) { return (x + 255) & ~size_t(255); };
	L.world = world;
	L.halo_cap = halo_cap;
	L.max_blocks = max_blocks;
	L.off_halo_keys = align(sizeof(InboxHeader));
	L.off_halo_blocks = align(L.off_halo_keys + (size_t) halo_cap * 3 * sizeof(int));
	L.off_keys = align(L.off_halo_blocks + (size_t) halo_cap * kGridBlockFloats * sizeof(float));
	L.seg_bytes = align(L.off_keys + (size_t) (max_blocks + 1) * 3 * sizeof(int));
	return L;
}
inline size_t inbox_bytes(const InboxLayout& L) { return 2 * (size_t) L.world * L.seg_bytes; }

struct MgspView {
	InboxLayout L;
	int rank, world;
	unsigned char* inbox[kMaxRanks];  // inbox of every rank mapped into this process (inbox[rank] is local)
	int* overlap_keys;                // [world][max_blocks*3]: my blocks that peer p also has
	int* overlap_count;               // [world]
	int* peer_bno;                    // [world][max_blocks]: block number of my block b in peer p's partition (-1: not shared)
	int* done;                        // [4] last-CTA counters
	int* epochs;                      // device: [0] max-vel, [1] halo, [2] keys
};

__device__ __forceinline__ unsigned char* seg_of(const MgspView& v, int owner, int parity, int src) { return v.inbox[owner] + ((size_t) parity * v.world + src) * v.L.seg_bytes; }
__device__ __forceinline__ void st_release_sys(int* p, int val) { asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(p), "r"(val) : "memory"); }
__device__ __forceinline__ int ld_acquire_sys(const int* p) {
	int v;
	asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
	return v;
}
__device__ __forceinline__ void wait_flag(const int* flag, int epoch) {
	while(ld_acquire_sys(flag) < epoch) __nanosleep(200);
}

// ---- max |v|^2 all-reduce (replaces the host max over devices, mgsp_benchmark.cuh:410-416) ------------------------
// one CTA: publish my value to every inbox, then wait for everybody's and take the max
__global__ void mgsp_allreduce_maxvel_kernel(MgspView v, float* max_vel_sq) {
	const int epoch = v.epochs[0] + 1, par = epoch & 1;
	const int t = threadIdx.x;
	if(t < v.world) {
		InboxHeader* h = reinterpret_cast<InboxHeader*>(seg_of(v, t, par, v.rank));
		h->max_vel_sq = *max_vel_sq;
		__threadfence_system();
		st_release_sys(&h->flag_mv, epoch);
	}
	__syncthreads();
	__shared__ float s_m[kMaxRanks];
	if(t < v.world) {
		InboxHeader* h = reinterpret_cast<InboxHeader*>(seg_of(v, v.rank, par, t));
		wait_flag(&h->flag_mv, epoch);
		s_m[t] = *reinterpret_cast<volatile float*>(&h->max_vel_sq);
	}
	__syncthreads();
	if(t == 0) {
		float m = 0.f;
		for(int r = 0; r < v.world; ++r) m = fmaxf(m, s_m[r]);
		*max_vel_sq = m;
		v.epochs[0] = epoch;
	}
}

// ---- "my remote reductions have landed" barrier: replaces pack / send / reduce in the fused path ---------------------------
// It follows g2p2g on the same stream (whose bulk reductions into the peers' grids are complete at the kernel boundary): an epoch
// flag goes to every peer with a system-scope release, and everybody's is awaited.  The step driver uses it as two halves:
// the flag is published right behind g2p2g, the wait sits in front of the first kernel that reads the reduced grid (the grid carry),
// behind the partition rebuild -- a rank that finishes its g2p2g late costs its peers nothing as long as it is less late than their
// rebuild takes.  epochs[1] is advanced by the tag kernel (mgsp_wait_reduce_kernel at setup).
__global__ void mgsp_done_publish_kernel(MgspView v) {
	const int epoch = v.epochs[1] + 1, par = epoch & 1;
	const int t = threadIdx.x;
	if(t < v.world && t != v.rank) {
		InboxHeader* h = reinterpret_cast<InboxHeader*>(seg_of(v, t, par, v.rank));
		__threadfence_system();
		st_release_sys(&h->flag_halo, epoch);
	}
}
// one warp: a wide kernel spinning on the flags would hold the SMs of ranks that share a GPU (tests) hostage
__global__ void mgsp_done_wait_kernel(MgspView v) {
	const int epoch = v.epochs[1] + 1, par = epoch & 1;
	const int t = threadIdx.x;
	if(t < v.world && t != v.rank) wait_flag(&reinterpret_cast<InboxHeader*>(seg_of(v, v.rank, par, t))->flag_halo, epoch);
}

// ---- halo pack + send (collect_grid_blocks + HaloGridBlocks::send, halo_kernels.cuh:65-80, halo_buffer.cuh:54-59) ---
// warp per block: reads my next-grid block, stores it (and its key) into the peer's inbox over NVLink
__global__ void __launch_bounds__(256) mgsp_pack_send_kernel(Cfg cfg, MgspView v, const float* grid, const int* table) {
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const int epoch = v.epochs[1] + 1, par = epoch & 1;
	for(int p = 0; p < v.world; ++p) {
		if(p == v.rank) continue;
		const int n = min(v.overlap_count[p], v.L.halo_cap);
		unsigned char* seg = seg_of(v, p, par, v.rank);
		int* rkeys = reinterpret_cast<int*>(seg + v.L.off_halo_keys);
		float* rblocks = reinterpret_cast<float*>(seg + v.L.off_halo_blocks);
		const int* mykeys = v.overlap_keys + (size_t) p * v.L.max_blocks * 3;
		for(int h = blockIdx.x * 8 + warp; h < n; h += gridDim.x * 8) {
			const int x = mykeys[3 * h], y = mykeys[3 * h + 1], z = mykeys[3 * h + 2];
			const int bno = table_query(cfg, table, x, y, z);
			float4* d = reinterpret_cast<float4*>(rblocks + (size_t) h * kGridBlockFloats);
			if(bno >= 0) {
				const float4* s = reinterpret_cast<const float4*>(grid + (size_t) bno * kGridBlockFloats);
				d[lane] = s[lane];
				d[32 + lane] = s[32 + lane];
			} else {
				d[lane] = make_float4(0.f, 0.f, 0.f, 0.f);
				d[32 + lane] = make_float4(0.f, 0.f, 0.f, 0.f);
			}
			if(lane < 3) rkeys[3 * h + lane] = mykeys[3 * h + lane];
		}
	}
	// last CTA publishes the counts and the epoch flags
	__threadfence_system();
	__syncthreads();
	__shared__ int s_last;
	if(threadIdx.x == 0) s_last = atomicAdd(&v.done[0], 1) == (int) gridDim.x - 1;
	__syncthreads();
	if(s_last) {
		__threadfence_system();
		if((int) threadIdx.x < v.world && (int) threadIdx.x != v.rank) {
			const int p = threadIdx.x;
			InboxHeader* h = reinterpret_cast<InboxHeader*>(seg_of(v, p, par, v.rank));
			h->halo_count = min(v.overlap_count[p], v.L.halo_cap);
			__threadfence_system();
			st_release_sys(&h->flag_halo, epoch);
		}
		if(threadIdx.x == 0) v.done[0] = 0;
	}
}

// ---- wait + reduce (reduce_grid_blocks, halo_kernels.cuh:83-97) -------------------------------------------------------
// A block can be shared with several peers, so two messages may hit the same cell: native global float reductions.
__global__ void __launch_bounds__(256) mgsp_wait_reduce_kernel(Cfg cfg, MgspView v, float* grid, const int* table, int* error) {
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const int epoch = v.epochs[1] + 1, par = epoch & 1;
	for(int p = 0; p < v.world; ++p) {
		if(p == v.rank) continue;
		unsigned char* seg = seg_of(v, v.rank, par, p);
		InboxHeader* hd = reinterpret_cast<InboxHeader*>(seg);
		if(threadIdx.x == 0) wait_flag(&hd->flag_halo, epoch);
		__syncthreads();
		const int n = *reinterpret_cast<volatile int*>(&hd->halo_count);
		const int* rkeys = reinterpret_cast<const int*>(seg + v.L.off_halo_keys);
		const float* rblocks = reinterpret_cast<const float*>(seg + v.L.off_halo_blocks);
		for(int h = blockIdx.x * 8 + warp; h < n; h += gridDim.x * 8) {
			const int bno = table_query(cfg, table, rkeys[3 * h], rkeys[3 * h + 1], rkeys[3 * h + 2]);
			if(bno < 0) continue;
			const float4* s = reinterpret_cast<const float4*>(rblocks + (size_t) h * kGridBlockFloats);
			float* d = grid + (size_t) bno * kGridBlockFloats;
#pragma unroll
			for(int r = 0; r < 2; ++r) {
				const float4 y = s[32 * r + lane];
				float* q = d + (32 * r + lane) * 4;
				atomicAdd(q, y.x);
				atomicAdd(q + 1, y.y);
				atomicAdd(q + 2, y.z);
				atomicAdd(q + 3, y.w);
			}
		}
	}
	__syncthreads();
	__shared__ int s_last;
	if(threadIdx.x == 0) s_last = atomicAdd(&v.done[1], 1) == (int) gridDim.x - 1;
	__syncthreads();
	if(s_last && threadIdx.x == 0) {
		v.done[1] = 0;
		v.epochs[1] = epoch;
		for(int p = 0; p < v.world; ++p)
			if(p != v.rank && v.overlap_count[p] > v.L.halo_cap && error) atomicOr(error, kErrBlockCapacity);
	}
}

// ---- key all-gather for halo tagging (halo_tagging, mgsp_benchmark.cuh:661-720) -----------------------------------
// Clears this rank's next grid (new numbering) and publishes the keys in ONE launch.  The flag goes out only after every CTA has
// finished both loops, so a peer that sees it may reduce into the cleared grid.
// The message also carries this rank's max |v|^2 of the grid the NEXT sub-step starts from (computed by the carry kernel), so
// that the tag kernel, which waits for every peer's message anyway, yields the global maximum: one sync point per sub-step less.
__global__ void __launch_bounds__(256) mgsp_clear_publish_kernel(MgspView v, const int* keys, const int* key_count, const float* local_max_vel, float* clear_grid) {
	const int epoch = v.epochs[2] + 1, par = epoch & 1;
	const int nk = min(*key_count, v.L.max_blocks);
	{
		const size_t n4 = (size_t) nk * (kGridBlockFloats / 4);
		float4* g = reinterpret_cast<float4*>(clear_grid);
		for(size_t i = blockIdx.x * (size_t) blockDim.x + threadIdx.x; i < n4; i += (size_t) gridDim.x * blockDim.x) g[i] = make_float4(0.f, 0.f, 0.f, 0.f);
	}
	const int n3 = nk * 3;
	for(int p = 0; p < v.world; ++p) {
		if(p == v.rank) continue;
		int* rk = reinterpret_cast<int*>(seg_of(v, p, par, v.rank) + v.L.off_keys);
		for(int i = blockIdx.x * blockDim.x + threadIdx.x; i < n3; i += gridDim.x * blockDim.x) rk[i] = keys[i];
	}
	__threadfence_system();
	__syncthreads();
	__shared__ int s_last;
	if(threadIdx.x == 0) s_last = atomicAdd(&v.done[2], 1) == (int) gridDim.x - 1;
	__syncthreads();
	if(s_last) {
		__threadfence_system();
		if((int) threadIdx.x < v.world && (int) threadIdx.x != v.rank) {
			InboxHeader* h = reinterpret_cast<InboxHeader*>(seg_of(v, threadIdx.x, par, v.rank));
			h->key_count = nk;
			h->max_vel_sq = *local_max_vel;
			__threadfence_system();
			st_release_sys(&h->flag_keys, epoch);
		}
		if(threadIdx.x == 0) v.done[2] = 0;
	}
}

// reset of the tagging state at setup (reset_overlap_marks, hash_table.cuh:64-66); the step driver resets it in the grid carry
__global__ void mgsp_tag_reset_kernel(MgspView v, int* overlap_marks, const int* key_count) {
	const int n = *key_count;
	for(int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		overlap_marks[i] = 0;
		for(int p = 0; p < v.world; ++p) v.peer_bno[(size_t) p * v.L.max_blocks + i] = -1;
	}
	if(blockIdx.x == 0 && (int) threadIdx.x < v.world) v.overlap_count[threadIdx.x] = 0;
}

// mark_overlapping_blocks for every peer (halo_kernels.cuh:22-35), keys read from my inbox; the last CTA publishes the global
// max |v|^2 of the peers' messages.
// key_limit: only blocks numbered below it (particle + neighbour blocks) can overlap; exterior blocks registered meanwhile are ignored
// do_finalize (end of a sub-step): the last CTA also advances the halo epoch of this sub-step, rolls the device-resident step state
// (finalize_step) and resets this rank's local maximum for the next carry.  Setup runs without it: there mgsp_wait_reduce_kernel
// advances the halo epoch.
__global__ void __launch_bounds__(256) mgsp_tag_kernel(Cfg cfg, MgspView v, const int* table, int* overlap_marks, const int* key_limit, float* local_max_vel, float* global_max_vel, int do_finalize, FinalizeArgs fin) {
	const int limit = *key_limit;
	float gmax = *local_max_vel;
	const int epoch = v.epochs[2] + 1, par = epoch & 1;
	for(int p = 0; p < v.world; ++p) {
		if(p == v.rank) continue;
		unsigned char* seg = seg_of(v, v.rank, par, p);
		InboxHeader* hd = reinterpret_cast<InboxHeader*>(seg);
		if(threadIdx.x == 0) wait_flag(&hd->flag_keys, epoch);
		__syncthreads();
		const int n = *reinterpret_cast<volatile int*>(&hd->key_count);
		gmax = fmaxf(gmax, *reinterpret_cast<volatile float*>(&hd->max_vel_sq));
		const int* rk = reinterpret_cast<const int*>(seg + v.L.off_keys);
		int* outk = v.overlap_keys + (size_t) p * v.L.max_blocks * 3;
		for(int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
			const int x = rk[3 * i], y = rk[3 * i + 1], z = rk[3 * i + 2];
			const int bno = table_query(cfg, table, x, y, z);
			if(bno >= 0 && bno < limit) {
				atomicOr(overlap_marks + bno, 1 << p);
				v.peer_bno[(size_t) p * v.L.max_blocks + bno] = i;  // the peer's keys arrive in its block order
				const int h = atomicAdd(&v.overlap_count[p], 1);
				if(h < v.L.max_blocks) {
					outk[3 * h] = x;
					outk[3 * h + 1] = y;
					outk[3 * h + 2] = z;
				}
			}
		}
	}
	__syncthreads();
	__shared__ int s_last;
	if(threadIdx.x == 0) {
		__threadfence();
		s_last = atomicAdd(&v.done[3], 1) == (int) gridDim.x - 1;
	}
	__syncthreads();
	if(s_last && threadIdx.x == 0) {
		__threadfence();
		v.done[3] = 0;
		v.epochs[2] = epoch;
		*global_max_vel = gmax;  // every CTA saw every header; the last one publishes
		if(do_finalize) {
			v.epochs[1] = v.epochs[1] + 1;  // the halo ("my reductions have landed") epoch of this sub-step: published behind g2p2g, awaited by the carry
			finalize_step(fin);             // reads *global_max_vel through fin.next_max_vel
			*local_max_vel = 0.f;           // for the next sub-step's carry
		}
	}
}

}  // namespace cb200
