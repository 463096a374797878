// g2p2g.cuh -- the fused grid-to-particle / constitutive update / particle-to-grid kernel for sm_90a.
//
// Replaces g2p2g<Partition<1>, GridBuffer, M> (reference Projects/GMPM/mgmpm_kernels.cuh:665-937, with
// fetch_particle_buffer_data :428-462, calculate_contribution_and_store_particle_data :470-663 and
// ParticleBufferImpl::add_advection particle_buffer.cuh:100-135).  Same inputs, same outputs, same containers;
// different machine mapping:
//   * one CTA of 192 threads pulls particle blocks from a device-side queue (persistent grid, 4 CTAs per SM) instead
//     of one 128-thread CUDA block per particle block;
//   * the 2x2x2 neighbourhood of grid blocks is staged with eight 768-byte TMA bulk copies (the three velocity
//     channels of a grid block are contiguous) signalled on an mbarrier, then transposed in shared memory to one
//     float4 per node so that G2P issues 27 LDS.128 instead of 81 LDS.32 (reference: 1536 scalar global loads each
//     preceded by a table query, :700-726);
//   * the particle gathers are a software pipeline of 4-byte cp.async copies (no registers held, no reliance on the
//     ~20 KB of L1 left beside 208 KB of shared memory): tags land in the unused w words of the velocity arena, a
//     particle's position / F / J / logJp in its own staged-record slot, which is written only at the end of its
//     iteration; positions run one particle ahead, F is in flight during G2P;
//   * P2G does NOT scatter per particle.  Shared-memory float atomicAdd is a compare-and-swap loop on this
//     hardware (LDS, FADD, ATOMS.CAST.SPIN, BRA) and 108 of them per particle were 63 % of all instructions in the
//     first version of this kernel (profiles/r01_v0_*).  Instead:
//       phase 1  particle-parallel: gather, G2P, advection, F update, stress, bin store, re-bucketing; the P2G
//                inputs of each particle (local position, q = m v - C x_p, D = C dx: 15 floats) are staged in
//                shared memory (XOR-swizzled slots) and counting-sorted by cell with native integer shared atomics;
//       phase 2  cell-parallel: thread (cell, x-slice) walks the particles of its cell and accumulates its 9 nodes x
//                4 channels in registers: 108 adds per CELL, not per particle; registers -> arena by plain
//                read-add-write in two rounds of plane-disjoint (half-)warps, no atomics.  A particle that changed cell
//                but stayed in the particle block has the stencil of the cell it moved to and is accumulated there
//                (any order: counting-sorted by that cell; SORTED fixed-corotated: an arrival list of up to 8 per cell);
//       phase 3  the rest of the particles that changed cell in this step (leaving the particle block, or beyond a cell's
//                arrival list) are scattered node-parallel (atomics);
//   * the arena has the grid-block layout, so the write-back is eight 1-KiB cp.reduce.async.bulk f32-add operations
//     executed by the TMA unit, not 2048 SM-issued global atomics (:910-936); in MGSP mode a second bulk reduction
//     per shared grid block goes straight into the peer GPU's grid over NVLink;
//   * the 27 neighbour block numbers and source bin offsets are resolved once per block into shared memory instead
//     of two dependent global loads per particle (:761-767, particle_buffer.cuh:101-102).
// The kernel makes no assumption on the order of a block bucket (the reference's order is atomics-dependent);
// cell-major buckets (partition.cuh) merely make the gathers of phase 1 nearly contiguous and the records bank-regular.
#pragma once
#include "math3.cuh"

namespace cb200 {

// Launch shape.  Measured on one H100 80GB HBM3 SXM (400 W limit) on the 40 M-particle two-sphere scene, g2p2g ms per sub-step:
// 192 threads x 4 CTAs/SM (80 registers, no spills) 4.0-4.1; 192 x 3 (96 registers) 4.4; 256 x 3 (80) 4.25; 256 x 4 (64, spills) 4.85.
// The kernel is latency bound: with the spills gone, warps in flight win.
#ifndef CB200_G2P2G_THREADS
#define CB200_G2P2G_THREADS 192
#endif
#ifndef CB200_G2P2G_MIN_CTAS
#define CB200_G2P2G_MIN_CTAS 4
#endif
constexpr int kG2P2GThreads = CB200_G2P2G_THREADS;  // >= 192 = 64 cells x 3 stencil slices in phase 2
static_assert(kG2P2GThreads >= 192 && kG2P2GThreads % 32 == 0, "phase 2 maps one thread to (cell, slice)");
constexpr int kChunk = 512;         // particles staged per pass (64 cells x 8 ppc)

struct G2P2GModel {
	PBuf cur, next;
	Mat mat;
	// nullable: start of every cell inside next.blockbuckets (cell-major buckets of the step driver, [blocks][64]).  With it the staged
	// chunk is already grouped by home cell: phase 2 takes its particle ranges from these offsets and the counting sort is skipped.
	const unsigned short* next_offs;
};
struct G2P2GArgs {
	Cfg cfg;
	const StepState* state;  // nullable: when set, dt/new_dt/block count come from the device
	float dt, new_dt;
	int block_count;
	int n_models;             // models of the SAME material handled by one launch: the neighbourhood of a block is staged
	G2P2GModel m[kMaxModels]; // and written back once for all of them (the reference launches g2p2g once per model, :386-396)
	const int* prev_table;
	const int* table;
	const int* keys;
	const float* grid;
	float* next_grid;
	int* error;  // nullable
	int* work_counter;  // nullable: dynamic block queue (device int, zero before the launch); static striding otherwise
	// MGSP fused halo reduction: a grid block that is also active on peer p (bit p of overlap_marks) receives this CTA's
	// partial sums on BOTH owners: the arena flush issues a second bulk add-reduction straight into the peer's next grid
	// (CUDA-IPC mapped, NVLink) at the block number the peer gave that key (peer_bno).  nullptr = single-GPU.
	const int* overlap_marks;
	const int* peer_bno;     // [world][peer_stride]
	int peer_stride;
	float* peer_grid[8];
};

// accumulation arena: [block 2x2x2][channel 4][cell 4x4x4] floats == eight grid blocks back to back
__device__ __forceinline__ int acc_off_x(int X) { return ((X >> 2) << 2) * 256 + ((X & 3) << 4); }
__device__ __forceinline__ int acc_off_y(int Y) { return ((Y >> 2) << 1) * 256 + ((Y & 3) << 2); }
__device__ __forceinline__ int acc_off_z(int Z) { return (Z >> 2) * 256 + (Z & 3); }

// What a particle block's processing starts from.  Resolved one block ahead (the CTA knows its next ticket during the whole
// current block), in shared memory only, by cp.async copies issued where the current block waits anyway: so a block starts
// with its TMA copy and its first positions in flight right away instead of after five dependent round trips.
struct G2P2GHeader {
	int blk;                // the particle block this header describes (-1: none)
	int key[3];
	int size[kMaxModels];   // bucket size of every model
	int nbr[27];            // neighbour block numbers (next partition)
	int prevno[27];         // the same neighbours' block numbers in the previous partition
	int srcbin[27];         // their first bins in the source buffer of the block's first non-empty model (then of the model processed)
};

struct G2P2GSmem {
	float4 vel4[512];                // node-major velocity arena (v_y, v_z, v_x, gather tag in flight), index (X*8+Y)*8+Z
	float acc[8 * 256];              // accumulation arena (grid-block layout)
	float4 rec[4][kChunk];           // staged P2G records, SoA over the 4 quads; 6 KiB of quad 1 double as the TMA landing
	                                 // zone (8 blocks x 3 channels x 64 cells) while a block's neighbourhood is staged
	unsigned short idx[kChunk];      // (swizzled) record slots sorted by cell
	unsigned short movers[kChunk];   // staged slots of particles that changed cell
	unsigned short offs[66];         // SORTED: cell starts of the current model's bucket, [64] = bucket size
	int cnt[64];
	G2P2GHeader hdr[2];              // the current block's header and the next one's, being resolved
	int nmovers;
	int cur_blk, next_blk, hsel;     // hsel: hdr[hsel] is the current block's
	unsigned valid;                  // bit b: grid block b of the 2x2x2 neighbourhood exists
	unsigned long long bar;
#ifdef CB200_G2P2G_PHASE_CLOCKS
	long long clk_t0, clk_mark;      // thread 0's clock at kernel entry and at the last phase boundary
	unsigned long long clk[8];       // this CTA's sums, added to g2p2g_phase_clocks when it exits
#endif
};

// Per-phase cycle counters (off by default; `make EXTRA=-DCB200_G2P2G_PHASE_CLOCKS`, read by tools/g2p2g_phase_clocks.py).
// Thread 0 of every CTA reads clock64() at the phase boundaries below and adds the intervals up; the sums of all CTAs are
// added into this array when they exit.  Without the switch the macros expand to nothing and the kernel is unchanged.
enum G2P2GClock {
	kClkPrologue = 0,  // block top (from the previous block's B6) to S2: a header not resolved ahead, neighbourhood, first positions; empty blocks
	kClkPhase1,        // S2 (or a chunk's own prologue) to B1
	kClkPhase2,        // B1 to the second arena-round barrier
	kClkPhase3,        // node-parallel movers
	kClkFlush,         // end of the last chunk's phase 3 to B6
	kClkChunkPrologue, // every chunk after a block's first (later chunks, later models): barriers, source bins, tags, first positions
	kClkLateFirst,     // count: blocks whose first non-empty model is not model 0
	kClkTotal,         // whole CTA, kernel entry to exit
	kClkCount
};
#ifdef CB200_G2P2G_PHASE_CLOCKS
static_assert(kClkCount <= 8, "G2P2GSmem::clk");
__device__ unsigned long long g2p2g_phase_clocks[kClkCount];
#define CB200_CLK_START()                                                                      \
	do {                                                                                       \
		if(threadIdx.x == 0) {                                                                 \
			for(int k_ = 0; k_ < kClkCount; ++k_) sm.clk[k_] = 0;                              \
			sm.clk_t0 = sm.clk_mark = clock64();                                               \
		}                                                                                      \
	} while(0)
#define CB200_CLK_MARK(k)                                                                      \
	do {                                                                                       \
		if(threadIdx.x == 0) {                                                                 \
			const long long now_ = clock64();                                                  \
			sm.clk[(k)] += (unsigned long long) (now_ - sm.clk_mark);                          \
			sm.clk_mark = now_;                                                                \
		}                                                                                      \
	} while(0)
#define CB200_CLK_COUNT(k)                                                                     \
	do {                                                                                       \
		if(threadIdx.x == 0) sm.clk[(k)] += 1;                                                 \
	} while(0)
#define CB200_CLK_END()                                                                        \
	do {                                                                                       \
		if(threadIdx.x == 0) {                                                                 \
			sm.clk[kClkTotal] = (unsigned long long) (clock64() - sm.clk_t0);                  \
			for(int k_ = 0; k_ < kClkCount; ++k_) atomicAdd(&g2p2g_phase_clocks[k_], sm.clk[k_]); \
		}                                                                                      \
	} while(0)
#else
#define CB200_CLK_START() do {} while(0)
#define CB200_CLK_MARK(k) do {} while(0)
#define CB200_CLK_COUNT(k) do {} while(0)
#define CB200_CLK_END() do {} while(0)
#endif

// four CTAs per SM: 228 KB of shared memory per SM, 1 KB of it reserved per CTA
static_assert(CB200_G2P2G_MIN_CTAS * (sizeof(G2P2GSmem) + 1024) <= 228 * 1024, "G2P2GSmem no longer fits the CTAs per SM of the launch bounds");

// Staged records are XOR-swizzled: cell-major buckets put the p-th particles of consecutive cells 8 slots = 128 B apart,
// i.e. in the same four banks; unswizzled, phase 2 spent 3-5 wavefronts per 16-byte read (profiles/r01_final_*).
__device__ __forceinline__ int rec_slot(int slot) { return slot ^ ((slot >> 3) & 7); }
// threadIdx.x through a volatile read the compiler cannot move: values derived from it are computed where they are used
// instead of being hoisted out of the block loop (where, at 80 registers, they end up on the stack)
__device__ __forceinline__ int opaque_tid() {
	int t;
	asm volatile("mov.u32 %0, %%tid.x;" : "=r"(t));
	return t;
}
constexpr int kRecMover = 1 << 30;
constexpr int kRecDrop = 1 << 29;
// SORTED fixed-corotated: per-cell capacity of the arrival lists of in-block movers (sm.cnt / sm.idx, unused by the sorted path otherwise)
constexpr int kArrivals = 8;
static_assert(64 * kArrivals <= kChunk, "arrival lists live in sm.idx");
// the stencil base (0..5 per axis, arena node coordinates) packed in a record code: in this particle block when it is 1..4 on every
// axis, and then the particle is accumulated by the phase-2 thread of cell code_cell
__device__ __forceinline__ bool code_in_block(int code) {
	return ((code & 7) - 1u < 4u) & (((code >> 3) & 7) - 1u < 4u) & (((code >> 6) & 7) - 1u < 4u);
}
__device__ __forceinline__ int code_cell(int code) { return (((code & 7) - 1) << 4) | ((((code >> 3) & 7) - 1) << 2) | (((code >> 6) & 7) - 1); }

// quadratic B-spline weight of stencil node i as a polynomial in d = local position / dx in [0.5, 1.5)
__device__ __forceinline__ void bspline_poly(int i, float& a, float& b, float& c) {
	a = i == 0 ? 1.125f : (i == 1 ? -0.25f : 0.125f);
	b = i == 0 ? -1.5f : (i == 1 ? 2.f : -0.5f);
	c = i == 1 ? -1.f : 0.5f;
}

// SORTED: every model's bucket is cell-major and comes with its cell offsets (the step driver); otherwise any bucket order is
// accepted (kernel-level ABI: the reference's order is atomics-dependent) and the staged particles are counting-sorted by cell.
template<int MAT, bool SORTED>
__global__ void __launch_bounds__(kG2P2GThreads, CB200_G2P2G_MIN_CTAS) g2p2g_kernel(const G2P2GArgs a) {
	constexpr int BINF = (MAT == CB200_J_FLUID) ? 128 : 512;
	constexpr int T = kG2P2GThreads;
	constexpr int ITERS = (kChunk + T - 1) / T;
	// SORTED: in-block movers go to per-cell arrival lists that phase 2 walks.  Only the fixed-corotated build has them: in the
	// others (whose kernels are larger or whose phase 1 is shorter) the extra code cost 2-5 % on sand and fluid scenes that have no
	// movers (H100, DESIGN section 2.1), so their movers all take phase 3 as before.
	constexpr bool ARRIVALS = SORTED && MAT == CB200_FIXED_COROTATED;
	// Block headers resolved one block ahead (G2P2GHeader) in the fixed-corotated and fluid builds.  The sand build was 4-5 % slower
	// with them on the sand column (H100, DESIGN section 4), so it and the NACC build (the same SVD-heavy phase 1, not measured)
	// resolve each block's header at its top, one load after another, as before.
	constexpr bool AHEAD = MAT == CB200_FIXED_COROTATED || MAT == CB200_J_FLUID;

	extern __shared__ __align__(128) unsigned char smem_raw[];
	G2P2GSmem& sm = *reinterpret_cast<G2P2GSmem*>(smem_raw);
	uint64_t* bar = reinterpret_cast<uint64_t*>(&sm.bar);
	float* const velsoa = reinterpret_cast<float*>(&sm.rec[1][0]);  // landing zone of the TMA copies: consumed (transposed into vel4)
	                                                                // before anything is staged in quads 1-3 of the records

	const Cfg& cfg = a.cfg;
	float dt = a.dt, new_dt = a.new_dt;
	int nblocks = a.block_count;
	if(a.state) {
		dt = a.state->dt;
		new_dt = device_compute_dt(cfg, a.state->max_vel_sq, a.state->step_time, a.state->frame_time, a.state->dt_default);
		nblocks = a.state->pbc;
	}
	if(threadIdx.x == 0) {
		mbar_init(bar, 1);
		mbar_fence_init();
		sm.nmovers = 0;
	}
	if(threadIdx.x < 64) sm.cnt[threadIdx.x] = 0;
	CB200_CLK_START();
	__syncthreads();
	unsigned phase = 0;
	const float dx = cfg.dx, dx_inv = cfg.dx_inv, d_inv = cfg.d_inv;
	const int ppb_mask = cfg.ppb - 1;

	// block queue: CTAs pull particle blocks from a device counter, so a launch that shares the SMs with another launch or
	// starts late still balances.  The queue runs two blocks ahead: thread 0 keeps the newest ticket in a register, so the
	// atomic's round trip hides behind a whole block, and the queue shift rides on the flush barrier of the block before.
	// Barriers per (single-chunk) block: S2, B1, B2 (any-order form only), two for the arena rounds, B6; without AHEAD also S1.
	int q_pending = 0;
	if(threadIdx.x == 0) {
		if(a.work_counter) {
			sm.cur_blk = atomicAdd(a.work_counter, 1);
			sm.next_blk = atomicAdd(a.work_counter, 1);
		} else {
			sm.cur_blk = (int) blockIdx.x;
			sm.next_blk = (int) (blockIdx.x + gridDim.x);
		}
		sm.hdr[0].blk = sm.hdr[1].blk = -1;
		sm.hsel = 0;
	}
	__syncthreads();

	// ---- the block header (G2P2GHeader), in stages.  Every thread that issues one of these copies waits for it with a
	// cp_async_wait<0> before any counted wait of phase 1 (they ride in the positions' group, or are followed by the wait<0>
	// before B6), and each is published by a barrier or read only by the thread that copied it.
	// sizes and key of block b (warp 1)
	auto hdr_sizes_key = [&](G2P2GHeader& h, int b) {
		const int t = opaque_tid() - 32;
		if(t >= 0 && t < a.n_models) cp_async4(&h.size[t], a.m[t].next.particle_bucket_sizes + b);
		else if(t >= kMaxModels && t < kMaxModels + 3) cp_async4(&h.key[t - kMaxModels], a.keys + 3 * b + (t - kMaxModels));
	};
	// neighbour block numbers in both partitions, from the landed key (thread 32 + d: neighbour d)
	auto hdr_tables = [&](G2P2GHeader& h) {
		const int d = opaque_tid() - 32;
		if(d >= 0 && d < 27) {
			const int x = h.key[0] + d / 9 - 1, y = h.key[1] + (d / 3) % 3 - 1, z = h.key[2] + d % 3 - 1;
			if(in_domain(cfg, x, y, z)) {
				const int o = table_offset(cfg, x, y, z);
				cp_async4(&h.nbr[d], a.table + o);
				cp_async4(&h.prevno[d], a.prev_table + o);
			} else {
				h.nbr[d] = h.prevno[d] = -1;
			}
		}
	};
	// first model from `from` on with particles in the block (n_models: none)
	auto hdr_first = [&](const G2P2GHeader& h, int from) {
		int f = from;
		while(f < a.n_models && h.size[f] == 0) ++f;
		return f;
	};
	// source bins of model f, by the thread that copied prevno[d] (it waits for its own copies: no barrier)
	auto hdr_srcbin = [&](G2P2GHeader& h, int f) {
		const int d = opaque_tid() - 32;
		if(d >= 0 && d < 27) {
			cp_async_wait<0>();
			const int pno = h.prevno[d];
			if(pno >= 0) cp_async4(&h.srcbin[d], a.m[f].cur.bin_offsets + pno);
			else h.srcbin[d] = -1;
		}
	};
	// gather tags of the first chunk of model f, into the unused w components of the velocity arena (512 words for 512 staged
	// particles); thread t fetches the tags it will consume itself
	auto hdr_tags = [&](const G2P2GHeader& h, int b, int f) {
		const int t = opaque_tid();
		const int size0 = min(h.size[f], kChunk);
		const int* bucket0 = a.m[f].next.blockbuckets + ((size_t) b << cfg.ppb_shift);
#pragma unroll
		for(int it = 0; it < ITERS; ++it)
			if(it * T + t < size0) cp_async4(&sm.vel4[it * T + t].w, bucket0 + it * T + t);
	};

	for(;;) {
		const int tid = opaque_tid();  // (not loop-invariant to the compiler: see opaque_tid)
		const int qi = sm.cur_blk, qn = sm.next_blk;  // published by the last barrier every thread passed
		if(qi >= nblocks) break;
		if(tid == 0) q_pending = a.work_counter ? atomicAdd(a.work_counter, 1) : qn + (int) gridDim.x;
		const int blk = qi;
		G2P2GHeader& H = sm.hdr[AHEAD ? sm.hsel : 0];
		int kx = 0, ky = 0, kz = 0;  // without AHEAD: the key, in registers
		int first;  // first model with particles in the block (n_models: none)
		if constexpr(AHEAD) {
			if(H.blk != qi) {
				// not resolved ahead (the CTA's first block, or the one after an empty block): the stages one after another
				hdr_sizes_key(H, qi);
				cp_async_commit();
				cp_async_wait<0>();
				__syncthreads();  // R1: sizes, key
				hdr_tables(H);
				const int f = hdr_first(H, 0);
				if(f < a.n_models) hdr_tags(H, qi, f);
				cp_async_commit();
				if(f < a.n_models) hdr_srcbin(H, f);
				cp_async_commit();
				cp_async_wait<0>();
				__syncthreads();  // R2: tables, source bins, tags
			}
			first = hdr_first(H, 0);
		} else {
			first = 0;
			while(first < a.n_models && a.m[first].next.particle_bucket_sizes[blk] == 0) ++first;
		}
		if(first == a.n_models) {
			__syncthreads();
			if(tid == 0) {
				sm.cur_blk = qn;
				sm.next_blk = q_pending;
				if(AHEAD) sm.hsel ^= 1;
			}
			__syncthreads();
			CB200_CLK_MARK(kClkPrologue);
			continue;
		}
		if constexpr(!AHEAD) {
			kx = a.keys[3 * blk], ky = a.keys[3 * blk + 1], kz = a.keys[3 * blk + 2];
			// gather tags of the first chunk, copied while the neighbourhood is staged (thread t fetches the tags it consumes itself)
			const int size0 = min(a.m[first].next.particle_bucket_sizes[blk], kChunk);
			const int* bucket0 = a.m[first].next.blockbuckets + ((size_t) blk << cfg.ppb_shift);
#pragma unroll
			for(int it = 0; it < ITERS; ++it)
				if(it * T + tid < size0) cp_async4(&sm.vel4[it * T + tid].w, bucket0 + it * T + tid);
			cp_async_commit();
		}

		// ---- stage the neighbourhood, request the first positions --------------------------------------------
		// (the landing zone aliases the records of the previous block: its last readers are behind that block's B6)
		if(tid < 32) {
			const int lb = tid & 7;
			const int bno = AHEAD ? H.nbr[(((lb >> 2) & 1) + 1) * 9 + (((lb >> 1) & 1) + 1) * 3 + (lb & 1) + 1]
			                      : table_query(cfg, a.table, kx + ((lb >> 2) & 1), ky + ((lb >> 1) & 1), kz + (lb & 1));
			const unsigned valid = __ballot_sync(0xffffffffu, tid < 8 && bno >= 0);
			if(tid == 0) {
				sm.valid = valid;  // released by the arrive, acquired by every thread's wait
				mbar_arrive_expect_tx(bar, __popc(valid) * 768);
			}
			__syncwarp();
			if(tid < 8 && bno >= 0) tma_load_1d(velsoa + lb * 192, a.grid + (size_t) bno * kGridBlockFloats + 64, 768, bar);
		} else if(!AHEAD && tid < 32 + 27) {
			const int d = tid - 32;
			const int ox = d / 9 - 1, oy = (d / 3) % 3 - 1, oz = d % 3 - 1;
			H.nbr[d] = table_query(cfg, a.table, kx + ox, ky + oy, kz + oz);
			const int pno = table_query(cfg, a.prev_table, kx + ox, ky + oy, kz + oz);
			H.prevno[d] = pno;
			H.srcbin[d] = pno >= 0 ? a.m[first].cur.bin_offsets[pno] : -1;  // further models resolve theirs below
		}
		bool acc_dirty = true;  // the arena still feeds the previous block's bulk reductions: it is drained and zeroed just
		                        // before this block's first accumulation, i.e. behind its whole phase 1
		// source row of the particle staged in `slot` (its gather tag sits in vel4[slot].w) and the copy of its position
		auto src_of = [&](const float* bins, int slot) {
			const int tag = __float_as_int(sm.vel4[slot].w);
			const int sp = tag & ppb_mask;
			return bins + ((size_t) H.srcbin[tag >> cfg.ppb_shift] + (sp >> 5)) * BINF + (sp & 31);
		};
		auto fetch_pos = [&](const float* bins, int slot) {
			const float* sb = src_of(bins, slot);
			float* dst = &sm.rec[0][rec_slot(slot)].x;
			cp_async4(dst, sb);
			cp_async4(dst + 1, sb + 32);
			cp_async4(dst + 2, sb + 64);
		};
		if constexpr(AHEAD) {
			// the next block's sizes and key ride in the first positions' group (waited for in phase 1 or before B1)
			if(qn < nblocks) hdr_sizes_key(sm.hdr[sm.hsel ^ 1], qn);
			if(tid < min(H.size[first], kChunk)) fetch_pos(a.m[first].cur.bins, tid);
			cp_async_commit();
		} else {
			const int size0 = min(a.m[first].next.particle_bucket_sizes[blk], kChunk);
			__syncthreads();  // S1: srcbin
			cp_async_wait<0>();  // this thread's tags
			if(tid < size0) fetch_pos(a.m[first].cur.bins, tid);
			cp_async_commit();
		}
		mbar_wait(bar, phase);
		phase ^= 1;
		// SoA landing zone -> one float4 per node (zero where the grid block does not exist)
		{
			const unsigned valid = sm.valid;
			for(int n = tid; n < 512; n += T) {
				const int X = n >> 6, Y = (n >> 3) & 7, Z = n & 7;
				const int bi = ((X >> 2) << 2) | ((Y >> 2) << 1) | (Z >> 2);
				const int o = bi * 192 + (((X & 3) << 4) | ((Y & 3) << 2) | (Z & 3));
				const bool ok = (valid >> bi) & 1u;  // w holds a gather tag: write x, y, z only
				// node layout (v_y, v_z, v_x, -): G2P's packed arithmetic pairs the components (1, 2)
				*reinterpret_cast<float2*>(&sm.vel4[n].x) = ok ? make_float2(velsoa[o + 64], velsoa[o + 128]) : make_float2(0.f, 0.f);
				sm.vel4[n].z = ok ? velsoa[o] : 0.f;
			}
		}
		__syncthreads();  // S2: vel4
		CB200_CLK_MARK(kClkPrologue);
		if(first != 0) CB200_CLK_COUNT(kClkLateFirst);

		bool first_chunk = true;
		for(int mi = first; mi < a.n_models; ++mi) {
		const G2P2GModel& M = a.m[mi];
		const int bucket_size = AHEAD ? H.size[mi] : M.next.particle_bucket_sizes[blk];
		if(bucket_size == 0) continue;
		const float mass = M.mat.mass;
		const int dst_bin0 = M.next.bin_offsets[blk];
		const int* __restrict__ bucket = M.next.blockbuckets + ((size_t) blk << cfg.ppb_shift);

		for(int c0 = 0; c0 < bucket_size; c0 += kChunk) {
			const int nchunk = min(kChunk, bucket_size - c0);
			if constexpr(SORTED) {  // previous readers of sm.offs are behind a barrier (B6 / the arena rounds); B1 publishes the new values
				if(c0 == 0 && tid <= 64) sm.offs[tid] = tid < 64 ? M.next_offs[(size_t) blk * kBlockVol + tid] : (unsigned short) bucket_size;
			}
			// Software pipeline of the gathers (no registers held, no reliance on the few KB of L1 left beside 208 KB of shared
			// memory): tags sit in vel4[].w; the position of particle `slot` is copied into rec[0][slot] and its F / J / logJp into
			// rec[1..3][slot] -- the particle's own record slot, which is written only at the end of its iteration.  Positions
			// run one iteration ahead, F is in flight during G2P.  The first chunk of the first non-empty model came with the
			// header: its tags and source bins were resolved ahead and its positions requested at the top of the block.
			if(!first_chunk) {
				// every chunk after the first of a block waits for the previous one's phase 3; a further model resolves its bins
				__syncthreads();
				if(tid == 0) sm.nmovers = 0;
				if(c0 == 0 && tid < 27) {
					const int pno = H.prevno[tid];
					H.srcbin[tid] = pno >= 0 ? M.cur.bin_offsets[pno] : -1;
				}
				__syncthreads();
#pragma unroll
				for(int it = 0; it < ITERS; ++it)
					if(it * T + tid < nchunk) cp_async4(&sm.vel4[it * T + tid].w, bucket + c0 + it * T + tid);
				cp_async_commit();
				cp_async_wait<0>();
				if(tid < nchunk) fetch_pos(M.cur.bins, tid);
				cp_async_commit();
				CB200_CLK_MARK(kClkChunkPrologue);
			}
			first_chunk = false;
			// the block's last chunk resolves the next block's header (stages after B1, in the arena rounds, before B6)
			auto resolves_next = [&]() { return AHEAD && qn < nblocks && c0 + kChunk >= bucket_size && hdr_first(H, mi + 1) == a.n_models; };
			int cr0 = -1, cr1 = -1, cr2 = -1;  // (home cell << 16) | rank of the up-to-three particles of this thread
			static_assert(ITERS <= 3, "cellrank registers");

			// ================= phase 1: particle-parallel ==============================================
#pragma unroll 1
			for(int it = 0; it < ITERS; ++it) {
				const int slot = it * T + tid;
				if(slot >= nchunk) continue;
				const int pidib = c0 + slot;
				const int rs = rec_slot(slot);
				const float* __restrict__ sbin = src_of(M.cur.bins, slot);
				{  // group A: the channels needed after G2P
					float* dst = &sm.rec[1][rs].x;
					if constexpr(MAT == CB200_J_FLUID) {
						cp_async4(dst, sbin + 96);
					} else {
#pragma unroll
						for(int d = 0; d < 4; ++d) cp_async4(dst + d, sbin + (3 + d) * 32);
						dst = &sm.rec[2][rs].x;
#pragma unroll
						for(int d = 0; d < 4; ++d) cp_async4(dst + d, sbin + (7 + d) * 32);
						dst = &sm.rec[3][rs].x;
						cp_async4(dst, sbin + 11 * 32);
						if constexpr(MAT != CB200_FIXED_COROTATED) cp_async4(dst + 1, sbin + 12 * 32);
					}
					cp_async_commit();
				}
				cp_async_wait<1>();  // everything but group A: this particle's position has landed
				float pos[3];
				{
					const float4 p4 = sm.rec[0][rs];
					pos[0] = p4.x;
					pos[1] = p4.y;
					pos[2] = p4.z;
				}
				if(slot + T < nchunk) fetch_pos(M.cur.bins, slot + T);  // group B: next particle's position, a whole iteration ahead
				cp_async_commit();
				int base[3], ab[3];
				float lp[3], w[3][3];
#pragma unroll
				for(int d = 0; d < 3; ++d) {
					base[d] = cell_index(cfg, pos[d]) - 1;
					lp[d] = pos[d] - base[d] * dx;
					if(d > 0) bspline_weights(lp[d] * dx_inv, w[d][0], w[d][1], w[d][2]);
					ab[d] = ((base[d] - 1) & 3) + 1;
				}
				// G2P: velocity and APIC matrix (A as in the reference: sum W v (x_i - x_p)^T, column-major A[c + 3d]),
				// sum-factorised over the separable weights: a node's (v_y, v_z) is the register pair its LDS.128 delivered and is
				// carried as one f2, the weights enter as scalars.
				// A, F and the stress stay in the packed 3x3 form (rows 1-2 of a column = one pair) up to the staged record.
				float velx;
				f2 velyz;
				M3p A;
				{
					float wyx[3];
					f2 wzp[3];  // (w_z[k], w_z[k] * (z_k - z_p))
#pragma unroll
					for(int i = 0; i < 3; ++i) {
						wyx[i] = w[1][i] * (i * dx - lp[1]);
						wzp[i] = mk2(w[2][i], w[2][i] * (i * dx - lp[2]));
					}
					const f2 z2 = mk2(0.f, 0.f);
					f2 vyz = z2, A12 = z2, A45 = z2, A78 = z2, vxA6 = z2;
					float A0 = 0.f, A3 = 0.f;
					const float4* vp = &sm.vel4[(ab[0] * 8 + ab[1]) * 8 + ab[2]];
					// The x planes are a real loop: unrolled (even behind a compiler fence) the scheduler hoists all 27 LDS.128 of the stencil
					// and spills.  The plane's weight rotates through three registers instead of being selected by the loop index.
					float wx, wx_n, wx_nn;
					bspline_weights(lp[0] * dx_inv, wx, wx_n, wx_nn);
					float xi = -lp[0];
#pragma unroll 1
					for(int i = 0; i < 3; ++i, vp += 64) {
						const float wxx = wx * xi;
						f2 Ryz = z2, Yyz = z2, Zyz = z2, RxZx = z2;
						float Yx = 0.f;
#pragma unroll
						for(int j = 0; j < 3; ++j) {
							const float4 v0 = vp[j * 8], v1 = vp[j * 8 + 1], v2 = vp[j * 8 + 2];
							f2 Pyz = mul2(mk2(v0.x, v0.y), wzp[0].x), Qyz = mul2(mk2(v0.x, v0.y), wzp[0].y), PxQx = mul2(wzp[0], v0.z);
							Pyz = fma2(mk2(v1.x, v1.y), wzp[1].x, Pyz);
							Qyz = fma2(mk2(v1.x, v1.y), wzp[1].y, Qyz);
							PxQx = fma2(wzp[1], v1.z, PxQx);
							Pyz = fma2(mk2(v2.x, v2.y), wzp[2].x, Pyz);
							Qyz = fma2(mk2(v2.x, v2.y), wzp[2].y, Qyz);
							PxQx = fma2(wzp[2], v2.z, PxQx);
							Ryz = fma2(Pyz, w[1][j], Ryz);
							Yyz = fma2(Pyz, wyx[j], Yyz);
							Zyz = fma2(Qyz, w[1][j], Zyz);
							RxZx = fma2(PxQx, w[1][j], RxZx);
							Yx = fmaf(wyx[j], PxQx.x, Yx);
						}
						vyz = fma2(Ryz, wx, vyz);
						A12 = fma2(Ryz, wxx, A12);
						A45 = fma2(Yyz, wx, A45);
						A78 = fma2(Zyz, wx, A78);
						vxA6 = fma2(RxZx, wx, vxA6);
						A0 = fmaf(wxx, RxZx.x, A0);
						A3 = fmaf(wx, Yx, A3);
						wx = wx_n;
						wx_n = wx_nn;
						xi += dx;
					}
					velx = vxA6.x;
					velyz = vyz;
					A.s[0] = A0, A.s[1] = A3, A.s[2] = vxA6.y;
					A.p[0] = A12, A.p[1] = A45, A.p[2] = A78;
				}
				pos[0] = fmaf(velx, dt, pos[0]);
				pos[1] = fmaf(velyz.x, dt, pos[1]);
				pos[2] = fmaf(velyz.y, dt, pos[2]);

				// ---- re-bucket (add_advection), part 1: claim a slot in the new cell NOW so that the round trip of the
				// global atomic overlaps the deformation-gradient / stress arithmetic below; the tag is stored after it
				int nb[3], cell[3];
				int rb_slot = -1, rb_tag = 0;
				size_t rb_cell = 0;
				{
					int rel[3];
					bool far = false;
#pragma unroll
					for(int d = 0; d < 3; ++d) {
						nb[d] = cell_index(cfg, pos[d]) - 1;
						cell[d] = nb[d] - 1;
					}
					rel[0] = (cell[0] >> 2) - (AHEAD ? H.key[0] : kx);
					rel[1] = (cell[1] >> 2) - (AHEAD ? H.key[1] : ky);
					rel[2] = (cell[2] >> 2) - (AHEAD ? H.key[2] : kz);
#pragma unroll
					for(int d = 0; d < 3; ++d) far |= (rel[d] < -1) | (rel[d] > 1);
					const int bno = far ? -1 : H.nbr[(rel[0] + 1) * 9 + (rel[1] + 1) * 3 + rel[2] + 1];
					if(bno >= 0) {
						const int dirtag = (1 - rel[0]) * 9 + (1 - rel[1]) * 3 + (1 - rel[2]);
						const int cellno = ((cell[0] & 3) << 4) | ((cell[1] & 3) << 2) | (cell[2] & 3);
						rb_cell = (size_t) bno * kBlockVol + cellno;
						rb_tag = (dirtag << cfg.ppb_shift) | pidib;
						rb_slot = atomicAdd(M.next.cell_particle_counts + rb_cell, 1);
					} else if(a.error) {
						atomicOr(a.error, kErrLostParticle);
					}
				}

				M3p S;  // stress contribution P F^T vol (fluid: the Cauchy-like term of :474-516)
				float* __restrict__ dbin = M.next.bins + ((size_t) dst_bin0 + (pidib >> 5)) * BINF + (pidib & 31);
				if constexpr(MAT == CB200_J_FLUID) {
					cp_async_wait<1>();  // group A has landed (group B may still be in flight)
					float J = sm.rec[1][rs].x;
					J += (A.s[0] + A.p[1].x + A.p[2].y) * dt * d_inv * J;
					if(J < 0.1f) J = 0.1f;
					const float voln = J * M.mat.volume;
					const float pressure = M.mat.bulk * (powf(J, -M.mat.gamma) - 1.f);
					const float vs = d_inv * M.mat.viscosity;
					const float s01 = (A.p[0].x + A.s[1]) * vs * voln, s02 = (A.p[0].y + A.s[2]) * vs * voln, s12 = (A.p[1].y + A.p[2].x) * vs * voln;
					S.s[0] = ((A.s[0] + A.s[0]) * vs - pressure) * voln;
					S.p[0] = mk2(s01, s02);
					S.s[1] = s01;
					S.p[1] = mk2(((A.p[1].x + A.p[1].x) * vs - pressure) * voln, s12);
					S.s[2] = s02;
					S.p[2] = mk2(s12, ((A.p[2].y + A.p[2].y) * vs - pressure) * voln);
					dbin[0] = pos[0];
					dbin[32] = pos[1];
					dbin[64] = pos[2];
					dbin[96] = J;
				} else {
					cp_async_wait<1>();  // group A has landed (group B may still be in flight)
					const float4 fa = sm.rec[1][rs], fb = sm.rec[2][rs], fc = sm.rec[3][rs];
					const float Fo[9] = {fa.x, fa.y, fa.z, fa.w, fb.x, fb.y, fb.z, fb.w, fc.x};
					// F <- (I + A dt D_inv) F
					const float sc = dt * d_inv;
					M3p G, F;
					G.s[0] = fmaf(A.s[0], sc, 1.f), G.s[1] = A.s[1] * sc, G.s[2] = A.s[2] * sc;
					G.p[0] = mul2(A.p[0], sc);
					G.p[1] = fma2(A.p[1], sc, mk2(1.f, 0.f));
					G.p[2] = fma2(A.p[2], sc, mk2(0.f, 1.f));
#pragma unroll
					for(int c = 0; c < 3; ++c) {
						F.p[c] = fma2(G.p[2], Fo[3 * c + 2], fma2(G.p[1], Fo[3 * c + 1], mul2(G.p[0], Fo[3 * c])));
						F.s[c] = fmaf(G.s[2], Fo[3 * c + 2], fmaf(G.s[1], Fo[3 * c + 1], G.s[0] * Fo[3 * c]));
					}
					dbin[0] = pos[0];
					dbin[32] = pos[1];
					dbin[64] = pos[2];
					if constexpr(MAT == CB200_FIXED_COROTATED) {
#pragma unroll
						for(int c = 0; c < 3; ++c) {
							dbin[(3 + 3 * c) * 32] = F.s[c];
							dbin[(4 + 3 * c) * 32] = F.p[c].x;
							dbin[(5 + 3 * c) * 32] = F.p[c].y;
						}
						if(!stress_fixed_corotated_polar_packed(M.mat, F, S)) {
							float Fa[9], PFa[9];
							m3p_to_array(F, Fa);
							stress_fixed_corotated(M.mat, Fa, PFa);
							S = m3p_from_array(PFa);
						}
					} else {
						float log_jp = fc.y;
						float Fa[9], PFa[9];
						m3p_to_array(F, Fa);
						if constexpr(MAT == CB200_SAND) stress_sand(M.mat, Fa, PFa, log_jp);
						else stress_nacc(M.mat, Fa, PFa, log_jp);
#pragma unroll
						for(int d = 0; d < 9; ++d) dbin[(3 + d) * 32] = Fa[d];
						dbin[12 * 32] = log_jp;
						S = m3p_from_array(PFa);
					}
				}
				// D = (A m - stress new_dt) D_inv dx   (the affine momentum matrix in units of the cell size, column-major c + 3d)
				M3p D;
				{
					const float ka = mass * d_inv * dx, ks = -new_dt * d_inv * dx;
#pragma unroll
					for(int c = 0; c < 3; ++c) {
						D.s[c] = fmaf(A.s[c], ka, S.s[c] * ks);
						D.p[c] = fma2(A.p[c], ka, mul2(S.p[c], ks));
					}
				}

				// ---- re-bucket, part 2: store the advection tag into the claimed slot --------------------
#pragma unroll
				for(int d = 0; d < 3; ++d) lp[d] = (pos[d] - nb[d] * dx) * dx_inv;
				if(rb_slot >= 0) {
					if(rb_slot >= cfg.max_ppc) {
						atomicSub(M.next.cell_particle_counts + rb_cell, 1);
						if(a.error) atomicOr(a.error, kErrCellOverflow);
					} else {
						// SORTED (the step driver): its own slot-grouped layout, which its flatten reads (grouped_cell_slot).  Otherwise the
						// reference's rows of the kernel-level ABI: block * ppb + cell * max_ppc + slot == (block*64 + cell) * max_ppc + slot
						if constexpr(SORTED) M.next.cellbuckets[grouped_cell_slot(cfg, rb_cell >> 6, (int) rb_cell & 63, rb_slot)] = rb_tag;
						else M.next.cellbuckets[(rb_cell << cfg.ppc_shift) + rb_slot] = rb_tag;
					}
				}

				// ---- stage the P2G record ----------------------------------------------------------
				int nab[3];
				bool oob = false, moved = false;
#pragma unroll
				for(int d = 0; d < 3; ++d) {
					nab[d] = ab[d] + (nb[d] - base[d]);
					oob |= (nab[d] < 0) | (nab[d] > 5);
					moved |= nb[d] != base[d];
				}
				int code = (nab[0] & 7) | ((nab[1] & 7) << 3) | ((nab[2] & 7) << 6);
				if(oob) {  // moved more than one cell: the reference drops the contribution (mgmpm_kernels.cuh:881-885)
					code = kRecDrop;
					if(a.error) atomicOr(a.error, kErrLostParticle);
				} else if(moved && (SORTED || !code_in_block(code))) {
					code |= kRecMover;  // SORTED: the home-range walk of phase 2 skips every mover
					if constexpr(!ARRIVALS) sm.movers[atomicAdd(&sm.nmovers, 1)] = (unsigned short) slot;
				}
				// momentum of node (i, j, k) of the particle's stencil: q + i D[:,0] + j D[:,1] + k D[:,2], with q = m v - D x_p
				const float q0 = fmaf(mass, velx, -fmaf(D.s[2], lp[2], fmaf(D.s[1], lp[1], D.s[0] * lp[0])));
				const f2 q12 = fma2(D.p[2], -lp[2], fma2(D.p[1], -lp[1], fma2(D.p[0], -lp[0], mul2(velyz, mass))));
				// record layout chosen for phase 2's packed arithmetic: (y, z) and the (component 1, component 2) terms are aligned pairs
				sm.rec[0][rs] = make_float4(lp[1], lp[2], lp[0], __int_as_float(code));
				sm.rec[1][rs] = make_float4(q12.x, q12.y, D.p[0].x, D.p[0].y);
				sm.rec[2][rs] = make_float4(D.p[1].x, D.p[1].y, D.p[2].x, D.p[2].y);
				sm.rec[3][rs] = make_float4(q0, D.s[0], D.s[1], D.s[2]);
				// A particle is accumulated by the phase-2 thread of the cell its stencil starts from (code_cell): its home cell, or for
				// a mover the new cell when that lies in this particle block (lp is relative to the new base).  Movers that leave the
				// block are scattered by phase 3.
				if constexpr(ARRIVALS) {
					// the home ranges come from the cell-major bucket, so a cell's arrivals get a list of their own (sm.idx, unused
					// otherwise); the ones beyond its kArrivals entries go to phase 3
					if(code & kRecMover) {
						const int dc = code_cell(code);
						const int k = code_in_block(code) ? atomicAdd(&sm.cnt[dc], 1) : kArrivals;
						if(k < kArrivals) sm.idx[dc * kArrivals + k] = (unsigned short) rec_slot(slot);
						else sm.movers[atomicAdd(&sm.nmovers, 1)] = (unsigned short) slot;
					}
				} else if constexpr(!SORTED) {
					// counting sort by accumulation cell: an in-block mover is an ordinary phase-2 particle of its new cell
					int cr = -1;
					if(!(code & (kRecMover | kRecDrop))) cr = (code_cell(code) << 16) | atomicAdd(&sm.cnt[code_cell(code)], 1);
					if(it == 0) cr0 = cr;
					else if(it == 1) cr1 = cr;
					else cr2 = cr;
				}
			}
			cp_async_wait<0>();
			if(acc_dirty) {
				// The arena still feeds the previous block's bulk reductions.  The LAST warp drains and zeroes it: with 512 particles
				// on 192 threads that warp has no particle in the third pass, so the drain rides in its idle time instead of sitting
				// between two barriers of the whole CTA (its threads issued the reductions, see the flush below).
				if(tid >= T - 32) {
					if(tid < T - 24) tma_wait_read<0>();  // the TMA unit has read the arena
					__syncwarp();
					float4* acc4 = reinterpret_cast<float4*>(sm.acc);
#pragma unroll 4
					for(int i = tid - (T - 32); i < 8 * 256 / 4; i += 32) acc4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
				}
				acc_dirty = false;
			}
			__syncthreads();  // B1: records, cell counts and the mover list of this chunk are complete; the arena is zero
			CB200_CLK_MARK(kClkPhase1);
			if(resolves_next()) {
				// the next block's tables from its landed key, and the tags of its first chunk: phases 2 and 3 do not read vel4, and a
				// later chunk or model of this block would still read its own tags there
				G2P2GHeader& Nx = sm.hdr[sm.hsel ^ 1];
				hdr_tables(Nx);
				const int nf = hdr_first(Nx, 0);
				if(nf < a.n_models) hdr_tags(Nx, qn, nf);
				cp_async_commit();
				if(tid == 0) Nx.blk = qn;  // read at the top of the next block, behind B6 and every thread's wait<0> before it
			}
			// ================= phase 2: cell-parallel accumulation =====================================
			// thread = (home cell hc, x-slice sl of its 3x3x3 stencil); a half-warp holds the 16 cells of one x-plane.
			// The thread's cell, weight polynomial and nine arena offsets are derived from a fresh read of the thread index (see
			// opaque_tid), so they are computed here instead of being kept in registers or on the stack since earlier.
			const int ptid = opaque_tid();
			const int lane = ptid & 31;
			const int wrp = ptid >> 5;
			const bool p2 = ptid < 192;
			// warp: (cx, sl) of lanes 0-15 / lanes 16-31 -> node plane X = cx + sl + 1
			//   w0: (1,0) (0,1) -> 2 2    w1: (2,0) (1,1) -> 3 3    w2: (3,0) (2,1) -> 4 4    w3: (3,1) (2,2) -> 5 5
			//   w4: (0,0) (3,2) -> 1 6    w5: (0,2) (1,2) -> 3 4
			const int hi = lane >> 4;
			const int sl = wrp < 3 ? hi : (wrp == 3 ? 1 + hi : (wrp == 4 ? 2 * hi : 2));
			// (a function of the thread index: re-derived from a fresh read after the home-range loop, so it is not held across it)
			auto cell_of = [](int t) {
				const int w = t >> 5, h = (t >> 4) & 1;
				const int cx = w < 3 ? w + 1 - h : (w == 3 ? 3 - h : (w == 4 ? 3 * h : h));
				return ((cx & 3) << 4) | (t & 15);
			};
			int hc = cell_of(ptid);
			int n, st;
			if constexpr(SORTED) {
				// the bucket is cell-major, so the staged slots of this chunk are already grouped by home cell: cell hc owns the
				// slots [offs[hc], offs[hc + 1]) - c0, clipped to the chunk.  No counting sort, no second barrier.
				const int lo = min(max((int) sm.offs[hc] - c0, 0), nchunk), hiE = min(max((int) sm.offs[hc + 1] - c0, 0), nchunk);
				st = lo;
				n = p2 ? hiE - lo : 0;
			} else {
				// exclusive scan of the 64 cell counts, redundantly in every warp (lane l holds cells 2l and 2l+1): no barrier,
				// no shared prefix array
				const int c0v = sm.cnt[2 * lane], c1v = sm.cnt[2 * lane + 1];
				int excl = c0v + c1v;
#pragma unroll
				for(int o = 1; o < 32; o <<= 1) {
					const int t = __shfl_up_sync(0xffffffffu, excl, o);
					if(lane >= o) excl += t;
				}
				excl -= c0v + c1v;
				auto cell_start = [&](int h) {  // every lane of the warp must call it
					const int e = __shfl_sync(0xffffffffu, excl, h >> 1), c = __shfl_sync(0xffffffffu, c0v, h >> 1);
					return e + ((h & 1) ? c : 0);
				};
				{
					const int s0 = cell_start(max(cr0, 0) >> 16), s1 = cell_start(max(cr1, 0) >> 16), s2 = cell_start(max(cr2, 0) >> 16);
					// (the swizzled record slot is stored: phase 2 reads it three times per particle, once per x-slice)
					if(cr0 >= 0) sm.idx[s0 + (cr0 & 0xffff)] = (unsigned short) rec_slot(tid);
					if(cr1 >= 0) sm.idx[s1 + (cr1 & 0xffff)] = (unsigned short) rec_slot(T + tid);
					if(cr2 >= 0) sm.idx[s2 + (cr2 & 0xffff)] = (unsigned short) rec_slot(2 * T + tid);
				}
				n = p2 ? sm.cnt[hc] : 0;
				st = cell_start(hc);
				__syncthreads();  // B2: idx complete, every warp has read the cell counts
				if(tid < 64) sm.cnt[tid] = 0;  // for the next chunk / block (ordered by the barriers below)
			}
			{
				float pa, pb, pc;
				bspline_poly(sl, pa, pb, pc);
				const float fi = (float) sl;
				// accumulators of the 9 nodes (j, k) of this x-slice: sum of W (times the particle mass at the write-back) and the
				// three momentum channels
				float acc[9][4];
#pragma unroll
				for(int n9 = 0; n9 < 9; ++n9) acc[n9][0] = acc[n9][1] = acc[n9][2] = acc[n9][3] = 0.f;
				auto accumulate = [&](int slot, const float4 r0) {  // r0 = rec[0][slot] = (y, z, x, code)
					const float4 r1 = sm.rec[1][slot], r2 = sm.rec[2][slot], r3 = sm.rec[3][slot];
					// B-spline weights as polynomials in the local position: two FMA each, with immediates for y and z
					const float wx = fmaf(fmaf(pc, r0.z, pb), r0.z, pa);
					float wy[3], wz[3];
#pragma unroll
					for(int i = 0; i < 3; ++i) {
						float qa, qb, qc;
						bspline_poly(i, qa, qb, qc);
						wy[i] = fmaf(fmaf(qc, r0.x, qb), r0.x, qa);
						wz[i] = fmaf(fmaf(qc, r0.y, qb), r0.y, qa);
					}
					// momentum at node (sl, j, k) of the stencil: q + sl D[:,0] + j D[:,1] + k D[:,2], walked by additions
					float bx = fmaf(fi, r3.y, r3.x), by = fmaf(fi, r1.z, r1.x), bz = fmaf(fi, r1.w, r1.y);
#pragma unroll
					for(int j = 0; j < 3; ++j) {
						const float wxy = wx * wy[j];
						float px = bx, py = by, pz = bz;
#pragma unroll
						for(int k = 0; k < 3; ++k) {
							const float W = wxy * wz[k];
							float* an = acc[j * 3 + k];
							an[0] += W;
							an[1] = fmaf(px, W, an[1]);
							an[2] = fmaf(py, W, an[2]);
							an[3] = fmaf(pz, W, an[3]);
							if(k < 2) {
								px += r3.w;
								py += r2.z;
								pz += r2.w;
							}
						}
						if(j < 2) {
							bx += r3.z;
							by += r2.x;
							bz += r2.y;
						}
					}
				};
				for(int p = 0; p < n; ++p) {  // (requesting the next particle's index / first quad one iteration ahead measured 0.8 % slower)
					const int slot = SORTED ? rec_slot(st + p) : (int) sm.idx[st + p];
					const float4 r0 = sm.rec[0][slot];  // (y, z, x, code)
					if(__float_as_int(r0.w) & (kRecMover | kRecDrop)) continue;  // phase 3, or (SORTED) another cell's arrival
					accumulate(slot, r0);
				}
				if constexpr(ARRIVALS) {
					hc = cell_of(opaque_tid());
					// then the movers that arrived in this cell.  A warp none of whose cells has one skips the pass, so a sub-step
					// without movers runs the home-range loop alone.
					const int na = p2 ? min(sm.cnt[hc], kArrivals) : 0;
					if(__any_sync(0xffffffffu, na > 0)) {
						for(int p = 0; p < na; ++p) {
							const int slot = sm.idx[hc * kArrivals + p];
							accumulate(slot, sm.rec[0][slot]);
						}
						n += na;  // (the write-back below skips threads of cells without particles)
					}
				}
				// Registers -> arena by plain read-add-write, no atomics (a shared float atomicAdd is a compare-and-swap loop: 36 per
				// thread were 60 % of the kernel's shared-memory wavefronts).  All lanes of a warp execute the same stencil offset
				// (j, k) on different cells, i.e. on different nodes, and a thread only writes the node plane X of its slice, so
				// warps (half-warps) that own different planes never meet; the rest is ordered by rounds.
				// Round 0: w0-w3 (both halves hold the same plane: exchange by shuffle, lanes 0-15 add channels 0-1, lanes 16-31
				// channels 2-3) and w4 (planes 1 and 6, all four channels per lane); round 1: w5 (planes 3 and 4).  The rounds are
				// straight-line code: in a loop the accumulators of every warp stay live across its back-edge and spill.
				const int X = (hc >> 4) + 1 + sl, Y = ((hc >> 2) & 3) + 1, Z = (hc & 3) + 1;
				const int ox = acc_off_x(X);
				// (the __syncwarp orders a lane's write of one node before another lane's read of it at the next stencil offset)
				auto add_quad = [&]() {  // all four channels of this thread's nodes
#pragma unroll
					for(int j = 0; j < 3; ++j)
#pragma unroll
						for(int k = 0; k < 3; ++k) {
							if(n > 0) {
								const int o = ox + acc_off_y(Y + j) + acc_off_z(Z + k);
								const float m0 = sm.acc[o], m1 = sm.acc[o + 64], m2 = sm.acc[o + 128], m3 = sm.acc[o + 192];
								sm.acc[o] = fmaf(mass, acc[j * 3 + k][0], m0);
								sm.acc[o + 64] = m1 + acc[j * 3 + k][1];
								sm.acc[o + 128] = m2 + acc[j * 3 + k][2];
								sm.acc[o + 192] = m3 + acc[j * 3 + k][3];
							}
							__syncwarp();
						}
				};
				if(wrp < 4) {
#pragma unroll
					for(int j = 0; j < 3; ++j)
#pragma unroll
						for(int k = 0; k < 3; ++k) {
							// partner = same (cy, cz), the other (cx, sl) of this plane: same node
							const float v0 = mass * acc[j * 3 + k][0], v1 = acc[j * 3 + k][1], v2 = acc[j * 3 + k][2], v3 = acc[j * 3 + k][3];
							const float ra = __shfl_xor_sync(0xffffffffu, hi ? v0 : v2, 16), rb = __shfl_xor_sync(0xffffffffu, hi ? v1 : v3, 16);
							const int oc = ox + acc_off_y(Y + j) + acc_off_z(Z + k) + (hi ? 128 : 0);
							const float m0 = sm.acc[oc], m1 = sm.acc[oc + 64];
							sm.acc[oc] = m0 + ((hi ? v2 : v0) + ra);
							sm.acc[oc + 64] = m1 + ((hi ? v3 : v1) + rb);
							__syncwarp();
						}
				} else if(wrp == 4) {
					add_quad();
				}
				__syncthreads();
				if(wrp == 5) add_quad();
				else if(wrp == 1 && resolves_next()) {  // the next block's source bins, from its landed previous-partition numbers
					G2P2GHeader& Nx = sm.hdr[sm.hsel ^ 1];
					const int nf = hdr_first(Nx, 0);
					if(nf < a.n_models) hdr_srcbin(Nx, nf);
					cp_async_commit();
				}
				__syncthreads();
				CB200_CLK_MARK(kClkPhase2);
				// arrival counts for the next chunk / block (ordered before its phase 1 by the barrier that starts it)
				if(ARRIVALS && tid < 64) sm.cnt[tid] = 0;
			}
			// ================= phase 3: particles that changed cell, node-parallel ====================
			{
				const int total = sm.nmovers * 27;
				for(int wk = tid; wk < total; wk += T) {
					const int m = wk / 27, nn = wk - 27 * m;
					const int i = nn / 9, j = (nn / 3) % 3, k = nn % 3;
					const int slot = rec_slot(sm.movers[m]);
					const float4 r0 = sm.rec[0][slot], r1 = sm.rec[1][slot], r2 = sm.rec[2][slot], r3 = sm.rec[3][slot];
					const int code = __float_as_int(r0.w);
					float pa, pb, pc;
					bspline_poly(i, pa, pb, pc);
					const float wx = pa + r0.z * (pb + pc * r0.z);
					bspline_poly(j, pa, pb, pc);
					const float wy = pa + r0.x * (pb + pc * r0.x);
					bspline_poly(k, pa, pb, pc);
					const float wz = pa + r0.y * (pb + pc * r0.y);
					const float W = wx * wy * wz;
					const float fi = (float) i, fj = (float) j, fk = (float) k;
					const int o = acc_off_x((code & 7) + i) + acc_off_y(((code >> 3) & 7) + j) + acc_off_z(((code >> 6) & 7) + k);
					atomicAdd(&sm.acc[o], mass * W);
					atomicAdd(&sm.acc[o + 64], W * (r3.x + fi * r3.y + fj * r3.z + fk * r3.w));
					atomicAdd(&sm.acc[o + 128], W * (r1.x + fi * r1.z + fj * r2.x + fk * r2.z));
					atomicAdd(&sm.acc[o + 192], W * (r1.y + fi * r1.w + fj * r2.y + fk * r2.w));
				}
				CB200_CLK_MARK(kClkPhase3);
			}
		}
		}  // models

		// ---- arena -> next grid: eight 1-KiB bulk add-reductions ----------------------------------
		const int ft = tid - (T - 32);  // the flush is issued by the first eight lanes of the LAST warp (they also drain it, see above)
		const int flush_bno = (ft >= 0 && ft < 8) ? H.nbr[(((ft >> 2) & 1) + 1) * 9 + (((ft >> 1) & 1) + 1) * 3 + (ft & 1) + 1] : -1;
		fence_proxy_async();
		if constexpr(AHEAD) cp_async_wait<0>();  // the next block's header copies this thread issued
		if(tid == 0) {  // queue shift: every thread read cur/next/hsel at the top of this block, barriers ago
			sm.cur_blk = qn;
			sm.next_blk = q_pending;
			if(AHEAD) sm.hsel ^= 1;
		}
		__syncthreads();  // B6: arena, records and neighbour tables of this block are no longer written or read by the SM
		CB200_CLK_MARK(kClkFlush);
		if(tid == 0) sm.nmovers = 0;
		if(ft >= 0 && ft < 8) {
			const int bno = flush_bno;
			if(bno >= 0) {
				tma_reduce_add_f32(a.next_grid + (size_t) bno * kGridBlockFloats, sm.acc + ft * 256, 1024);
				if(a.overlap_marks) {
					unsigned mask = (unsigned) a.overlap_marks[bno];
					while(mask) {
						const int p = __ffs(mask) - 1;
						mask &= mask - 1;
						const int rb = a.peer_bno[(size_t) p * a.peer_stride + bno];
						if(rb >= 0) tma_reduce_add_f32(a.peer_grid[p] + (size_t) rb * kGridBlockFloats, sm.acc + ft * 256, 1024);
						else if(a.error) atomicOr(a.error, kErrHaloMap);  // tagged as shared but the peer's block number is unknown: never silently drop a halo sum
					}
				}
			}
			tma_commit();  // not waited for here: see acc_dirty
		}
	}
	if((int) threadIdx.x >= kG2P2GThreads - 32 && (int) threadIdx.x < kG2P2GThreads - 24) tma_wait_all<0>();
	CB200_CLK_END();
}

}  // namespace cb200
