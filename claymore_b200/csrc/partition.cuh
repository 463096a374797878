// partition.cuh -- sparse-grid partition / bucket rebuild kernels.
#pragma once
#include "common.cuh"

namespace cb200 {

// Partition::insert (hash_table.cuh:117-127): CAS the table entry, then claim the next block number.
// Out-of-domain keys are skipped (the reference indexes out of bounds); overflow sets an error bit.
__device__ __forceinline__ int partition_insert(const Cfg& cfg, int* table, int* keys, int* count, int capacity, int* error, int x, int y, int z) {
	if(!in_domain(cfg, x, y, z)) return -1;
	int* slot = table + table_offset(cfg, x, y, z);
	if(atomicCAS(slot, -1, 0) == -1) {
		const int idx = atomicAdd(count, 1);
		if(idx >= capacity) {
			if(error) atomicOr(error, kErrBlockCapacity);
			*slot = -1;
			return -1;
		}
		*slot = idx;
		keys[3 * idx] = x;
		keys[3 * idx + 1] = y;
		keys[3 * idx + 2] = z;
		return idx;
	}
	return -1;
}

// ------------------------------------------------------------------------------------------------
// exclusive scan of `count` ints (+ total at out[count]) by ONE CTA of 1024 threads.
// Replaces thrust::exclusive_scan (gmpm_simulator.cuh:257-260); the count may be device-resident.
// ------------------------------------------------------------------------------------------------
struct ScanArgs {
	Count count;
	int count_plus;      // scan count + count_plus elements (reference scans ext+1 / pbc+1)
	const int* in;
	int* out;
	int* total_out;      // nullable: receives the sum of the first `count` elements
	int* total_out2;     // nullable: second destination (e.g. Partition::count)
	int limit;           // if > 0: total above this sets *error |= error_bit and total is clamped to 0
	int* error;
	int error_bit;
};
constexpr int kScanPer = 8;  // elements per thread per pass (8192 per CTA pass)
__device__ __forceinline__ void scan_body(const ScanArgs& a) {
	__shared__ int s_warp[32];
	__shared__ int s_carry;
	const int n = a.count.get();
	const int n_out = n + a.count_plus;
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	if(tid == 0) s_carry = 0;
	__syncthreads();
	for(int base = 0; base < n_out; base += 1024 * kScanPer) {
		const int i0 = base + tid * kScanPer;
		int v[kScanPer];
		int tsum = 0;
#pragma unroll
		for(int k = 0; k < kScanPer; ++k) {
			v[k] = (i0 + k < n) ? a.in[i0 + k] : 0;
			tsum += v[k];
		}
		int inc = tsum;
#pragma unroll
		for(int o = 1; o < 32; o <<= 1) {
			const int t = __shfl_up_sync(0xffffffffu, inc, o);
			if(lane >= o) inc += t;
		}
		if(lane == 31) s_warp[warp] = inc;
		__syncthreads();
		if(warp == 0) {
			int w = s_warp[lane];
#pragma unroll
			for(int o = 1; o < 32; o <<= 1) {
				const int t = __shfl_up_sync(0xffffffffu, w, o);
				if(lane >= o) w += t;
			}
			s_warp[lane] = w;
		}
		__syncthreads();
		const int carry = s_carry;
		int ex = carry + (warp ? s_warp[warp - 1] : 0) + inc - tsum;
#pragma unroll
		for(int k = 0; k < kScanPer; ++k) {
			if(i0 + k < n_out) a.out[i0 + k] = ex;
			ex += v[k];
		}
		__syncthreads();
		if(tid == 1023) s_carry = carry + s_warp[31];
		__syncthreads();
	}
	if(tid == 0) {
		int total = s_carry;
		if(a.limit > 0 && total > a.limit) {
			if(a.error) atomicOr(a.error, a.error_bit);
			total = 0;
		}
		if(a.total_out) *a.total_out = total;
		if(a.total_out2) *a.total_out2 = total;
	}
}
__global__ void __launch_bounds__(1024) scan_kernel(const ScanArgs a) { scan_body(a); }
// exclusive_scan_inverse (Library/MnBase/Algorithm/MappingKernels.cuh:44-55)
__global__ void scan_inverse_kernel(int num, const int* map, int* map_inv) {
	for(int i = blockIdx.x * blockDim.x + threadIdx.x; i < num; i += gridDim.x * blockDim.x) {
		const int m = map[i];
		if(m != map[i + 1]) map_inv[m] = i;
	}
}

// ------------------------------------------------------------------------------------------------
// cell buckets -> block bucket (cell_bucket_to_block, mgmpm_kernels.cuh:70-84).
// This library's form: the 64 cell counts are prefix-summed by one warp, then all tags are copied with coalesced
// writes (each thread finds its cell by a 6-step search of the 65-entry prefix in shared memory), instead of
// 128 rounds of warp-aggregated atomics each ending in a block barrier.  Bucket order is CELL-MAJOR: lanes of
// a warp in g2p2g then share stencil nodes and read near-contiguous source slots.
// dst_block lets the caller write straight into the compacted numbering (fuses update_buckets, :979-1000).
// ------------------------------------------------------------------------------------------------
constexpr int kBucketThreads = 128;
__device__ __forceinline__ int flatten_block(const Cfg& cfg, const int* __restrict__ cell_counts_blk, const int* __restrict__ cellbuckets_blk, int* __restrict__ dst, int* s_prefix, unsigned short* __restrict__ offs = nullptr) {
	const int tid = threadIdx.x, lane = tid & 31;
	if(tid < 32) {
		const int2 c = reinterpret_cast<const int2*>(cell_counts_blk)[lane];
		const int pair = c.x + c.y;
		int inc = pair;
#pragma unroll
		for(int o = 1; o < 32; o <<= 1) {
			const int t = __shfl_up_sync(0xffffffffu, inc, o);
			if(lane >= o) inc += t;
		}
		s_prefix[2 * lane] = inc - pair;
		s_prefix[2 * lane + 1] = inc - pair + c.x;
		if(lane == 31) s_prefix[64] = inc;
	}
	__syncthreads();
	const int total = s_prefix[64];
	if(offs && tid < 64) offs[tid] = (unsigned short) s_prefix[tid];  // where the cells start inside the cell-major bucket (read by g2p2g's phase 2)
	for(int i = tid; i < total; i += kBucketThreads) {
		int c = 0;
#pragma unroll
		for(int s = 32; s > 0; s >>= 1)
			if(s_prefix[c + s] <= i) c += s;
		dst[i] = cellbuckets_blk[(c << cfg.ppc_shift) + (i - s_prefix[c])];
	}
	__syncthreads();
	return total;
}

__global__ void __launch_bounds__(kBucketThreads) cell_bucket_to_block_kernel(Cfg cfg, int block_count, const int* cell_particle_counts, const int* cellbuckets, int* particle_bucket_sizes, int* buckets, unsigned short* cell_offsets = nullptr) {
	__shared__ int s_prefix[65];
	for(int b = blockIdx.x; b < block_count; b += gridDim.x) {
		const int total = flatten_block(cfg, cell_particle_counts + (size_t) b * kBlockVol, cellbuckets + ((size_t) b << cfg.ppb_shift), buckets + ((size_t) b << cfg.ppb_shift), s_prefix, cell_offsets ? cell_offsets + (size_t) b * kBlockVol : nullptr);
		if(threadIdx.x == 0) particle_bucket_sizes[b] += total;
	}
}

// ------------------------------------------------------------------------------------------------
// step-driver fused kernels.  The reference's rebuild is: mark_active_particle_blocks, thrust::exclusive_scan of the
// marks (gmpm_simulator.cuh:257-260), update_partition (mgmpm_kernels.cuh:966-977), cell_bucket_to_block + update_buckets,
// compute_bin_capacity and a second thrust scan.  Here: two launches over tiles of 64 old blocks, no single-CTA scan:
//   summary_kernel   per tile: particle totals of its blocks, the tile's aggregates (marked blocks, bins per model);
//                    the LAST CTA to finish scans the few thousand tile aggregates and writes the totals;
//   rebuild_kernel   per tile: scan inside the tile + the tile prefix = new block number / bin offset of every marked
//                    block; keys, table, buckets are written straight in the new numbering.
// ------------------------------------------------------------------------------------------------
constexpr int kRebuildTile = 64;        // old blocks per CTA
constexpr int kSummaryThreads = 256;    // 8 warps x 8 blocks (eight independent row loads in flight per warp)
constexpr int kRebuildThreads = 1024;   // 32 warps x 2 blocks: a marked block costs a dozen dependent gather rounds
constexpr int kScanComps = kMaxModels + 1;  // component 0: marked blocks, 1 + m: bins of model m

struct SummaryArgs {
	Cfg cfg;
	StepState* state;
	int n_models;
	const int* cell_counts[kMaxModels];  // next buffers' cell_particle_counts (old numbering)
	int* block_totals;                   // [n_models][max_blocks]: particles per old block
	int* tile_sums;                      // [tiles][kScanComps]: aggregate, then (last CTA) exclusive prefix
	int max_blocks;
	// the partition that is about to be rebuilt: un-insert its keys (replaces cudaMemsetAsync(0xff, 4*G^3),
	// hash_table.cuh:110-112, by touching only the entries that were set) -- in this launch, because every stale
	// entry must be gone before rebuild_kernel writes the first new one
	int* stale_table;
	const int* stale_keys;
	int* stale_count;                    // Partition::count: stale count in, number of new particle blocks out
	int* new_pbc;
	int* bin_offsets[kMaxModels];        // cur buffers: [new_pbc] = total bins
};
__global__ void __launch_bounds__(kSummaryThreads) summary_kernel(const SummaryArgs a) {
	constexpr int PER_WARP = kRebuildTile / (kSummaryThreads / 32);
	__shared__ int s_tot[kMaxModels][kRebuildTile];
	__shared__ int s_last;
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const int nm = a.n_models, nc = nm + 1;
	const int ebc = a.state->ebc;
	const int n_tiles = (ebc + kRebuildTile - 1) / kRebuildTile;
	const int stale = min(*(volatile int*) a.stale_count, a.max_blocks);
	for(int i = blockIdx.x * blockDim.x + tid; i < stale; i += gridDim.x * blockDim.x) {
		const int x = a.stale_keys[3 * i], y = a.stale_keys[3 * i + 1], z = a.stale_keys[3 * i + 2];
		if(in_domain(a.cfg, x, y, z)) a.stale_table[table_offset(a.cfg, x, y, z)] = -1;
	}
	const int tile = blockIdx.x, b0 = tile * kRebuildTile;
	if(tile < n_tiles) {
		// warp w sums the cell counts of its blocks (one coalesced 256-byte row per block and model)
#pragma unroll
		for(int j = 0; j < PER_WARP; ++j) {
			const int t = warp * PER_WARP + j, b = b0 + t;
			for(int m = 0; m < nm; ++m) {
				int tot = 0;
				if(b < ebc) {
					const int2 c = reinterpret_cast<const int2*>(a.cell_counts[m] + (size_t) b * kBlockVol)[lane];
					tot = __reduce_add_sync(0xffffffffu, c.x + c.y);
				}
				if(lane == 0) {
					s_tot[m][t] = tot;
					if(b < ebc) a.block_totals[(size_t) m * a.max_blocks + b] = tot;
				}
			}
		}
		__syncthreads();
		if(warp == 0) {
			for(int c = 0; c < nc; ++c) {
				int v = 0;
#pragma unroll
				for(int h = 0; h < kRebuildTile / 32; ++h) {
					const int t = h * 32 + lane;
					if(c == 0) {
						int any = 0;
						for(int m = 0; m < nm; ++m) any |= s_tot[m][t];
						v += any > 0;
					} else {
						v += (s_tot[c - 1][t] + kBinCap - 1) / kBinCap;
					}
				}
				v = __reduce_add_sync(0xffffffffu, v);
				if(lane == 0) a.tile_sums[(size_t) tile * kScanComps + c] = v;
			}
		}
	}
	// ---- the last CTA to finish turns the tile aggregates into exclusive prefixes and publishes the totals
	__syncthreads();
	if(tid == 0) {
		__threadfence();
		s_last = atomicAdd(&a.state->done_counter, 1) == (int) gridDim.x - 1;
	}
	__syncthreads();
	if(!s_last) return;
	__threadfence();
	if(tid == 0) a.state->done_counter = 0;
	// CTA-wide scan per component: thread i owns the tiles [i K, (i + 1) K)
	{
		__shared__ int s_wsum[kSummaryThreads / 32];
		const int K = (n_tiles + kSummaryThreads - 1) / kSummaryThreads;
		for(int c = 0; c < nc; ++c) {
			volatile int* col = a.tile_sums + c;
			int sum = 0;
			for(int k = 0; k < K; ++k) {
				const int t = tid * K + k;
				if(t < n_tiles) sum += col[(size_t) t * kScanComps];
			}
			int inc = sum;
#pragma unroll
			for(int o = 1; o < 32; o <<= 1) {
				const int u = __shfl_up_sync(0xffffffffu, inc, o);
				if(lane >= o) inc += u;
			}
			if(lane == 31) s_wsum[warp] = inc;
			__syncthreads();
			int base = 0, total = 0;
#pragma unroll
			for(int w = 0; w < kSummaryThreads / 32; ++w) {
				const int v = s_wsum[w];
				if(w < warp) base += v;
				total += v;
			}
			int run = base + inc - sum;  // exclusive prefix of this thread's first tile
			for(int k = 0; k < K; ++k) {
				const int t = tid * K + k;
				if(t < n_tiles) {
					const int v = col[(size_t) t * kScanComps];
					col[(size_t) t * kScanComps] = run;
					run += v;
				}
			}
			if(tid == 0) col[(size_t) n_tiles * kScanComps] = total;  // grand total behind the last tile
			__syncthreads();
		}
	}
	__syncthreads();
	if(tid == 0) {
		volatile int* tot = a.tile_sums + (size_t) n_tiles * kScanComps;
		const int n_new = tot[0];
		*a.new_pbc = n_new;
		*a.stale_count = n_new;
		if(n_new > a.max_blocks) atomicOr(&a.state->error, kErrBlockCapacity);
		for(int m = 0; m < nm; ++m) {
			a.bin_offsets[m][n_new] = tot[1 + m];
			a.state->bin_count[m] = tot[1 + m];
		}
	}
}

// one WARP per old block: the 64 cell counts are prefix-summed with shuffles, a tag finds its cell by a 6-step binary
// search over the lane-distributed prefix (shuffles, no shared memory, no block barrier), so the eight warps of a CTA
// stream independent blocks and hide each other's latency.
__device__ __forceinline__ int warp_flatten_block(const Cfg& cfg, const int* __restrict__ cell_counts_blk, const int* __restrict__ cellbuckets_blk, int* __restrict__ dst, unsigned short* __restrict__ offs) {
	const int lane = threadIdx.x & 31;
	const int2 c = reinterpret_cast<const int2*>(cell_counts_blk)[lane];
	const int pair = c.x + c.y;
	int inc = pair;
#pragma unroll
	for(int o = 1; o < 32; o <<= 1) {
		const int t = __shfl_up_sync(0xffffffffu, inc, o);
		if(lane >= o) inc += t;
	}
	const int p_even = inc - pair;       // exclusive prefix of cell 2*lane
	const int p_odd = p_even + c.x;      // exclusive prefix of cell 2*lane + 1
	const int total = __shfl_sync(0xffffffffu, inc, 31);
	if(offs) reinterpret_cast<ushort2*>(offs)[lane] = make_ushort2((unsigned short) p_even, (unsigned short) p_odd);  // cell starts inside the bucket
#pragma unroll 2
	for(int i0 = 0; i0 < total; i0 += 32) {
		const int i = i0 + lane;
		// largest lane L with p_even(L) <= i
		int L = 0;
#pragma unroll
		for(int s = 16; s > 0; s >>= 1) {
			const int probe = __shfl_sync(0xffffffffu, p_even, (L + s) & 31);
			if(probe <= i) L += s;
		}
		const int pe = __shfl_sync(0xffffffffu, p_even, L);
		const int po = __shfl_sync(0xffffffffu, p_odd, L);
		const bool odd = po <= i;
		const int cell = 2 * L + (odd ? 1 : 0);
		const int off = i - (odd ? po : pe);
		if(i < total) dst[i] = cellbuckets_blk[(cell << cfg.ppc_shift) + off];
	}
	return total;
}

struct RebuildArgs {
	Cfg cfg;
	const StepState* state;
	int n_models;
	const int* old_keys;
	int* new_keys;
	int* new_table;
	const int* block_totals;             // from summary_kernel
	const int* tile_sums;                // exclusive tile prefixes
	int max_blocks;
	const int* cell_counts[kMaxModels];  // next buffers (old numbering)
	const int* cellbuckets[kMaxModels];
	int* dst_sizes[kMaxModels];          // cur buffers (new numbering)
	int* dst_buckets[kMaxModels];
	int* bin_offsets[kMaxModels];        // cur buffers: exclusive scan of the bin demand
	unsigned short* dst_offs[kMaxModels];  // cur buffers (new numbering): start of every cell inside the cell-major block bucket
};
__global__ void __launch_bounds__(kRebuildThreads, 2) rebuild_kernel(const RebuildArgs a) {  // 2 CTAs/SM: the gather rounds of a marked block are latency bound
	constexpr int PER_WARP = kRebuildTile / (kRebuildThreads / 32);
	static_assert(kRebuildTile == 64, "the tile scan below is written for two warps");
	__shared__ int s_tot[kMaxModels][kRebuildTile];
	__shared__ int s_pre[kScanComps][kRebuildTile];  // exclusive prefix inside a 32-block half
	__shared__ int s_half[kScanComps];               // aggregate of the first half
	const Cfg& cfg = a.cfg;
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const int nm = a.n_models, nc = nm + 1;
	const int ebc = a.state->ebc;
	const int tile = blockIdx.x, b0 = tile * kRebuildTile;
	if(b0 >= ebc) return;
	if(tid < kRebuildTile) {  // thread t = block b0 + t
		const int b = b0 + tid;
		int any = 0;
		for(int m = 0; m < nm; ++m) {
			const int tot = b < ebc ? a.block_totals[(size_t) m * a.max_blocks + b] : 0;
			s_tot[m][tid] = tot;
			any |= tot;
		}
		for(int c = 0; c < nc; ++c) {
			const int v = c == 0 ? (any > 0) : (s_tot[c - 1][tid] + kBinCap - 1) / kBinCap;
			int inc = v;
#pragma unroll
			for(int o = 1; o < 32; o <<= 1) {
				const int u = __shfl_up_sync(0xffffffffu, inc, o);
				if(lane >= o) inc += u;
			}
			s_pre[c][tid] = inc - v;
			if(tid == 31) s_half[c] = inc;
		}
	}
	__syncthreads();
	// ---- compaction: warp per marked old block
	for(int j = 0; j < PER_WARP; ++j) {
		const int t = warp * PER_WARP + j, b = b0 + t;
		if(b >= ebc) break;
		int any = 0;
		for(int m = 0; m < nm; ++m) any |= s_tot[m][t];
		if(!any) continue;
		const int* tp = a.tile_sums + (size_t) tile * kScanComps;
		const int nb = tp[0] + s_pre[0][t] + (t >= 32 ? s_half[0] : 0);
		if(lane == 0) {
			const int x = a.old_keys[3 * b], y = a.old_keys[3 * b + 1], z = a.old_keys[3 * b + 2];
			a.new_keys[3 * nb] = x;
			a.new_keys[3 * nb + 1] = y;
			a.new_keys[3 * nb + 2] = z;
			a.new_table[table_offset(cfg, x, y, z)] = nb;
		}
		for(int m = 0; m < nm; ++m) {
			if(s_tot[m][t] == 0) {  // nothing to flatten
				if(lane == 0) {
					a.dst_sizes[m][nb] = 0;
					a.bin_offsets[m][nb] = tp[1 + m] + s_pre[1 + m][t] + (t >= 32 ? s_half[1 + m] : 0);
				}
				continue;
			}
			const int total = warp_flatten_block(cfg, a.cell_counts[m] + (size_t) b * kBlockVol, a.cellbuckets[m] + ((size_t) b << cfg.ppb_shift), a.dst_buckets[m] + ((size_t) nb << cfg.ppb_shift),
			                                     a.dst_offs[m] ? a.dst_offs[m] + (size_t) nb * kBlockVol : nullptr);
			if(lane == 0) {
				a.dst_sizes[m][nb] = total;
				a.bin_offsets[m][nb] = tp[1 + m] + s_pre[1 + m][t] + (t >= 32 ? s_half[1 + m] : 0);
			}
		}
	}
}

// (3) end of sub-step: roll the device-resident counters and clock (gmpm_simulator.cuh:578-579 and the
//     D2H counter copies at :462,:502,:517,:564)
struct FinalizeArgs {
	Cfg cfg;
	StepState* state;
	const int* new_pbc;
	const int* new_nbc;   // value of Partition::count after neighbour registration (snapshot)
	const int* new_count; // Partition::count after exterior registration
	int max_blocks;
	int n_models;
	long long bin_capacity[kMaxModels];
	const float* next_max_vel;  // nullable (MGSP): global max |v|^2 of the grid the next sub-step starts from
};
__device__ __forceinline__ void finalize_step(const FinalizeArgs& a) {
	StepState* s = a.state;
	const float next_dt = [&] {
		float dt = s->dt_default;
		const float mv = sqrtf(s->max_vel_sq);
		if(mv > 0.f) dt = fminf(dt, a.cfg.dx * a.cfg.cfl / mv);
		if(s->frame_time > 0.f) dt = fminf(dt, s->frame_time - s->step_time);
		return dt;
	}();
	s->next_dt = next_dt;
	s->prev_nbc = s->nbc;
	s->prev_ebc = s->ebc;
	s->pbc = min(*a.new_pbc, a.max_blocks);
	s->nbc = min(*a.new_nbc, a.max_blocks);
	s->ebc = min(*(volatile const int*) a.new_count, a.max_blocks);
	for(int m = 0; m < a.n_models; ++m)
		if(s->bin_count[m] > a.bin_capacity[m]) s->error |= kErrBinCapacity;
	s->sim_time += (double) s->dt;  // the dt this sub-step ran with
	s->dt = next_dt;
	// the reference's loop increment runs after `dt = next_dt` (gmpm_simulator.cuh:324,579): the clock advances by the NEW dt
	s->step_time += next_dt;
	if(s->frame_roll && s->frame_time > 0.f && s->step_time >= s->frame_time) s->step_time = 0.f;
	s->max_vel_sq = a.next_max_vel ? *a.next_max_vel : 0.f;
	for(int m = 0; m < 4; ++m) s->work_counter_mat[m] = 0;
	s->steps += 1;
}
// (4) neighbour / exterior registration (register_neighbor_blocks :117-133, register_exterior_blocks :135-151):
//     one thread per (particle block, offset) so the CAS traffic is spread over the whole grid.
struct RegisterArgs {
	Cfg cfg;
	Count block_count;  // particle blocks of the partition
	int* table;
	int* keys;
	int* count;
	int capacity;
	int* error;
	int lo, span;       // offsets per axis in [lo, lo+span): (0,2) neighbours, (-1,3) exterior
	// what the LAST CTA to finish does, in place of one-thread kernels of their own:
	int* done_counter;  // nullable: zero before the launch, zero again after it
	int* snapshot_out;  // nullable: receives *count once every insertion of this launch is done
	int do_finalize;    // roll the step state (fin)
	FinalizeArgs fin;
};
__global__ void register_blocks_kernel(const RegisterArgs a) {
	const int n = a.block_count.get();
	const int per = a.span * a.span * a.span;
	const long long total = (long long) n * per;
	for(long long t = blockIdx.x * (long long) blockDim.x + threadIdx.x; t < total; t += (long long) gridDim.x * blockDim.x) {
		const int b = (int) (t / per), o = (int) (t % per);
		const int i = o / (a.span * a.span) + a.lo, j = (o / a.span) % a.span + a.lo, k = o % a.span + a.lo;
		partition_insert(a.cfg, a.table, a.keys, a.count, a.capacity, a.error, a.keys[3 * b] + i, a.keys[3 * b + 1] + j, a.keys[3 * b + 2] + k);
	}
	if(a.done_counter) {
		__syncthreads();
		if(threadIdx.x == 0) {
			__threadfence();
			if(atomicAdd(a.done_counter, 1) == (int) gridDim.x - 1) {
				__threadfence();
				*a.done_counter = 0;
				// partition_insert keeps counting past the capacity (the overflow is flagged in `error`): every consumer of the
				// count -- the snapshot, the step state, the next registration -- must see the clamped value, or the grid carry,
				// the clears and the next grid update would index keys / grids past their max_blocks + 1 allocations
				int c = *(volatile int*) a.count;
				if(c > a.capacity) {
					c = a.capacity;
					*a.count = c;
				}
				if(a.snapshot_out) *a.snapshot_out = c;
				if(a.do_finalize) finalize_step(a.fin);
			}
		}
	}
}


// ------------------------------------------------------------------------------------------------
// drop-in forms of the remaining reference kernels (one thread per element)
// ------------------------------------------------------------------------------------------------
__global__ void mark_active_particle_blocks_kernel(int block_count, const int* sizes, int* marks) {
	for(int b = blockIdx.x * blockDim.x + threadIdx.x; b < block_count; b += gridDim.x * blockDim.x)
		if(sizes[b] > 0) marks[b] = 1;
}
__global__ void compute_bin_capacity_kernel(int block_count, const int* sizes, int* bin_sizes) {
	for(int b = blockIdx.x * blockDim.x + threadIdx.x; b < block_count; b += gridDim.x * blockDim.x) bin_sizes[b] = (sizes[b] + kBinCap - 1) / kBinCap;
}
__global__ void update_partition_kernel(Cfg cfg, int block_count, const int* source_nos, const int* keys, int* next_keys, int* next_table) {
	for(int b = blockIdx.x * blockDim.x + threadIdx.x; b < block_count; b += gridDim.x * blockDim.x) {
		const int s = source_nos[b];
		const int x = keys[3 * s], y = keys[3 * s + 1], z = keys[3 * s + 2];
		next_keys[3 * b] = x;
		next_keys[3 * b + 1] = y;
		next_keys[3 * b + 2] = z;
		if(in_domain(cfg, x, y, z)) next_table[table_offset(cfg, x, y, z)] = b;
	}
}
__global__ void update_buckets_kernel(Cfg cfg, int block_count, const int* source_nos, const int* sizes, const int* buckets, int* next_sizes, int* next_buckets) {
	for(int b = blockIdx.x; b < block_count; b += gridDim.x) {
		const int s = source_nos[b];
		const int n = sizes[s];
		if(threadIdx.x == 0) next_sizes[b] = n;
		for(int i = threadIdx.x; i < n; i += blockDim.x) next_buckets[((size_t) b << cfg.ppb_shift) + i] = buckets[((size_t) s << cfg.ppb_shift) + i];
	}
}

}  // namespace cb200
