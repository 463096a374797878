// init.cuh -- one-time setup kernels (initial partition, bins, rasterisation) and particle retrieval.
// They run once per model / once per output frame and are not on the timed path; they keep the
// reference's structure (thread per particle) with bounds checks added.
#pragma once
#include "math3.cuh"
#include "partition.cuh"

namespace cb200 {

// Particle block of a bucket cell (cell index - 2).  The reference divides with C's truncation, so a particle less than 1.5 dx
// from a low face (cell - 2 < 0) lands in block 0 although g2p2g's stencil offset and re-bucketing use floor semantics
// (DESIGN.md section 3, quirk #8).  The step driver uses the floor (FLOOR = true): the block is negative, the particle is flagged
// lost at set-up and never bucketed.  The kernel-level drop-in entries keep the reference's truncation.
template<bool FLOOR> __device__ __forceinline__ int bucket_block(int c) { return FLOOR ? c >> 2 : c / 4; }

// activate_blocks (mgmpm_kernels.cuh:21-34)
template<bool FLOOR>
__global__ void activate_blocks_kernel(Cfg cfg, int n, const float* pos, int* table, int* keys, int* count, int capacity, int* error) {
	for(int p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) {
		const int x = bucket_block<FLOOR>(cell_index(cfg, pos[3 * p]) - 2), y = bucket_block<FLOOR>(cell_index(cfg, pos[3 * p + 1]) - 2), z = bucket_block<FLOOR>(cell_index(cfg, pos[3 * p + 2]) - 2);
		partition_insert(cfg, table, keys, count, capacity, error, x, y, z);
	}
}

// build_particle_cell_buckets (mgmpm_kernels.cuh:36-68).  FLOOR = true is the step driver's: it writes the driver's slot-grouped cell
// buckets (grouped_cell_slot), which its warp flatten reads; the kernel-level drop-in writes the reference's cell-major rows.
template<bool FLOOR>
__global__ void build_particle_cell_buckets_kernel(Cfg cfg, int n, const float* pos, PBuf pb, const int* table, int* error) {
	for(int p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) {
		const int cx = cell_index(cfg, pos[3 * p]) - 2, cy = cell_index(cfg, pos[3 * p + 1]) - 2, cz = cell_index(cfg, pos[3 * p + 2]) - 2;
		const int bno = table_query(cfg, table, bucket_block<FLOOR>(cx), bucket_block<FLOOR>(cy), bucket_block<FLOOR>(cz));
		if(bno < 0) {
			if(error) atomicOr(error, kErrLostParticle);
			continue;
		}
		const int cellno = (cx & 3) * 16 + (cy & 3) * 4 + (cz & 3);
		int* cnt = pb.cell_particle_counts + (size_t) bno * kBlockVol + cellno;
		const int slot = atomicAdd(cnt, 1);
		if(slot >= cfg.max_ppc) {
			atomicSub(cnt, 1);
			if(error) atomicOr(error, kErrCellOverflow);
			continue;
		}
		if(FLOOR) pb.cellbuckets[grouped_cell_slot(cfg, bno, cellno, slot)] = p;
		else pb.cellbuckets[((size_t) bno << cfg.ppb_shift) + (cellno << cfg.ppc_shift) + slot] = p;
	}
}

// array_to_buffer (mgmpm_kernels.cuh:221-323): every bucketed particle's row into its bin slot.  The row of particle p is its start
// state at pos[p] or, with `rows` (a restore, an emission), the saved row rows[p] of ck_channels(material) channels.
__global__ void array_to_buffer_kernel(Cfg cfg, int material, int block_count, const float* pos, const float* rows, PBuf pb) {
	const int binf = bin_floats(material), C = ck_channels(material);
	for(int b = blockIdx.x; b < block_count; b += gridDim.x) {
		const int n = pb.particle_bucket_sizes[b];
		const int* bucket = pb.blockbuckets + ((size_t) b << cfg.ppb_shift);
		for(int i = threadIdx.x; i < n; i += blockDim.x) {
			const int pid = bucket[i];
			float* bin = bin_slot(pb.bins, pb.bin_offsets[b], i, binf);
			if(!rows) {
				start_state(material, pos + 3 * pid, bin, kBinCap);
				continue;
			}
			const float* row = rows + (size_t) pid * C;
			for(int c = 0; c < C; ++c) bin[c * kBinCap] = row[c];
		}
	}
}

// rasterize (mgmpm_kernels.cuh:153-219): initial mass / momentum; one-time, global float atomics are fine here
__global__ void rasterize_kernel(Cfg cfg, int n, const float* pos, float* grid, const int* table, float mass, float v0x, float v0y, float v0z, int* error) {
	for(int p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) {
		int base[3];
		float w[3][3];
#pragma unroll
		for(int d = 0; d < 3; ++d) {
			base[d] = cell_index(cfg, pos[3 * p + d]) - 1;
			const float lp = pos[3 * p + d] - base[d] * cfg.dx;
			bspline_weights(lp * cfg.dx_inv, w[d][0], w[d][1], w[d][2]);
		}
#pragma unroll
		for(int i = 0; i < 3; ++i)
#pragma unroll
			for(int j = 0; j < 3; ++j)
#pragma unroll
				for(int k = 0; k < 3; ++k) {
					const int gx = base[0] + i, gy = base[1] + j, gz = base[2] + k;
					const int bno = table_query(cfg, table, gx >> 2, gy >> 2, gz >> 2);
					if(bno < 0) {
						if(error) atomicOr(error, kErrLostParticle);
						continue;
					}
					const float wm = mass * (w[0][i] * w[1][j] * w[2][k]);
					float* blk = grid + (size_t) bno * kGridBlockFloats + ((gx & 3) * 16 + (gy & 3) * 4 + (gz & 3));
					atomicAdd(blk, wm);
					atomicAdd(blk + 64, wm * v0x);
					atomicAdd(blk + 128, wm * v0y);
					atomicAdd(blk + 192, wm * v0z);
				}
	}
}

// Block-parallel form of rasterize for the step driver: the particles are already bucketed per block and sit in the bins, so a
// CTA accumulates the MASS of one particle block's particles in a shared-memory arena (2x2x2 grid blocks, as g2p2g) and flushes
// it once: 4 global atomics per touched node instead of 108 per particle (the momentum of a model is v0 x its mass field, since
// every particle of a model starts with the same velocity, :212-215).
__global__ void __launch_bounds__(256) rasterize_blocks_kernel(Cfg cfg, int material, int block_count, const int* keys, const int* table, PBuf pb, float* grid, float mass, float v0x, float v0y, float v0z, int* error) {
	__shared__ float arena[8 * 64];
	__shared__ int s_bno[8];
	const int binf = bin_floats(material);
	for(int b = blockIdx.x; b < block_count; b += gridDim.x) {
		const int n = pb.particle_bucket_sizes[b];
		if(n == 0) continue;
		const int kx = keys[3 * b], ky = keys[3 * b + 1], kz = keys[3 * b + 2];
		for(int i = threadIdx.x; i < 512; i += blockDim.x) arena[i] = 0.f;
		if(threadIdx.x < 8) s_bno[threadIdx.x] = table_query(cfg, table, kx + ((threadIdx.x >> 2) & 1), ky + ((threadIdx.x >> 1) & 1), kz + (threadIdx.x & 1));
		__syncthreads();
		const int first = pb.bin_offsets[b];
		// the bucket is cell-major: neighbouring lanes would hold particles of one cell and fight over the same 27 nodes (a shared float
		// atomicAdd is a compare-and-swap loop).  A lane takes every (n/32)-th particle instead, so a warp's lanes sit in different cells.
		const int per_lane = (n + 31) >> 5;
		for(int t = threadIdx.x; t < per_lane * 32; t += blockDim.x) {
			const int i = (t & 31) * per_lane + (t >> 5);
			if(i >= n) continue;
			const float* bin = bin_slot(pb.bins, first, i, binf);
			int ab[3];
			float w[3][3];
#pragma unroll
			for(int d = 0; d < 3; ++d) {
				const float x = bin[32 * d];
				const int base = cell_index(cfg, x) - 1;
				bspline_weights((x - base * cfg.dx) * cfg.dx_inv, w[d][0], w[d][1], w[d][2]);
				ab[d] = base - 4 * (d == 0 ? kx : (d == 1 ? ky : kz));  // 1..4: node index inside the 8^3 arena
			}
			if(((unsigned) (ab[0] - 1) > 3u) | ((unsigned) (ab[1] - 1) > 3u) | ((unsigned) (ab[2] - 1) > 3u)) {  // not a particle of this block
				if(error) atomicOr(error, kErrLostParticle);
				continue;
			}
#pragma unroll
			for(int i3 = 0; i3 < 3; ++i3)
#pragma unroll
				for(int j = 0; j < 3; ++j)
#pragma unroll
					for(int k = 0; k < 3; ++k) {
						const int X = ab[0] + i3, Y = ab[1] + j, Z = ab[2] + k;
						const int bi = ((X >> 2) << 2) | ((Y >> 2) << 1) | (Z >> 2);
						atomicAdd(&arena[bi * 64 + (((X & 3) << 4) | ((Y & 3) << 2) | (Z & 3))], mass * (w[0][i3] * w[1][j] * w[2][k]));
					}
		}
		__syncthreads();
		for(int i = threadIdx.x; i < 512; i += blockDim.x) {
			const float m = arena[i];
			if(m == 0.f) continue;
			const int lb = i >> 6, bno = s_bno[lb];
			if(bno < 0) {
				// a node beyond the top face (the stencil of a particle at cell index 4G - 1 or 4G) does not exist: its share is
				// dropped, as g2p2g's flush drops it every sub-step.  A missing block inside the domain is a lost particle.
				if(error && in_domain(cfg, kx + ((lb >> 2) & 1), ky + ((lb >> 1) & 1), kz + (lb & 1))) atomicOr(error, kErrLostParticle);
				continue;
			}
			float* cell = grid + (size_t) bno * kGridBlockFloats + (i & 63);
			atomicAdd(cell, m);
			atomicAdd(cell + 64, m * v0x);
			atomicAdd(cell + 128, m * v0y);
			atomicAdd(cell + 192, m * v0z);
		}
		__syncthreads();
	}
}

// init_adv_bucket (mgmpm_kernels.cuh:96-104): identity tags (dir 13 == no block change)
__global__ void init_adv_bucket_kernel(Cfg cfg, int block_count, const int* sizes, int* buckets) {
	for(int b = blockIdx.x; b < block_count; b += gridDim.x)
		for(int i = threadIdx.x; i < sizes[b]; i += blockDim.x) buckets[((size_t) b << cfg.ppb_shift) + i] = (13 << cfg.ppb_shift) | i;
}

// retrieve_particle_buffer (mgmpm_kernels.cuh:1087-1122); nch > 3 also exports the remaining channels
// (F / J / logJp) -- the reference exports positions only, so a run can be checkpointed here.
__global__ void retrieve_kernel(Cfg cfg, int material, Count block_count, const int* keys, const int* prev_table, PBuf pb, PBuf next_pb, float* out, int nch, int* parcount) {
	const int binf = bin_floats(material);
	const int n = block_count.get();
	__shared__ int s_base;
	for(int b = blockIdx.x; b < n; b += gridDim.x) {
		const int cnt = next_pb.particle_bucket_sizes[b];
		__syncthreads();
		if(threadIdx.x == 0) s_base = atomicAdd(parcount, cnt);
		__syncthreads();
		const int base = s_base;
		const int kx = keys[3 * b], ky = keys[3 * b + 1], kz = keys[3 * b + 2];
		for(int i = threadIdx.x; i < cnt; i += blockDim.x) {
			const int advect = next_pb.blockbuckets[((size_t) b << cfg.ppb_shift) + i];
			const int dir = advect >> cfg.ppb_shift, sp = advect & (cfg.ppb - 1);
			const int sno = table_query(cfg, prev_table, kx + dir / 9 - 1, ky + (dir / 3) % 3 - 1, kz + dir % 3 - 1);
			if(sno < 0) continue;
			const float* bin = bin_slot(pb.bins, pb.bin_offsets[sno], sp, binf);
			for(int c = 0; c < nch; ++c) out[(size_t) (base + i) * nch + c] = bin[c * 32];
		}
	}
}

// ------------------------------------------------------------------------------------------------
// MGSP halo protocol (Projects/MGSP/halo_kernels.cuh:22-97)
// ------------------------------------------------------------------------------------------------
// mark_overlapping_blocks :22-35 -- which of MY blocks are also active on peer `otherdid`
__global__ void mark_overlapping_blocks_kernel(Cfg cfg, Count block_count, int otherdid, const int* incoming, const int* table, int* overlap_marks, int* count, int* out_blockids) {
	const int n = block_count.get();
	for(int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const int x = incoming[3 * i], y = incoming[3 * i + 1], z = incoming[3 * i + 2];
		const int bno = table_query(cfg, table, x, y, z);
		if(bno >= 0) {
			atomicOr(overlap_marks + bno, 1 << otherdid);
			const int h = atomicAdd(count, 1);
			out_blockids[3 * h] = x;
			out_blockids[3 * h + 1] = y;
			out_blockids[3 * h + 2] = z;
		}
	}
}
// collect_blockids_for_halo_reduction :38-62 -- particle blocks whose 2x2x2 footprint touches an overlapping block
__global__ void collect_halo_blockids_kernel(Cfg cfg, Count particle_block_count, const int* table, const int* keys, const int* overlap_marks, char* halo_marks, int* halo_count, int* halo_blocks) {
	const int n = particle_block_count.get();
	for(int b = blockIdx.x * blockDim.x + threadIdx.x; b < n; b += gridDim.x * blockDim.x) {
		const int x = keys[3 * b], y = keys[3 * b + 1], z = keys[3 * b + 2];
		bool hit = false;
		for(int o = 0; o < 8 && !hit; ++o) {
			const int nno = table_query(cfg, table, x + (o >> 2), y + ((o >> 1) & 1), z + (o & 1));
			hit = nno >= 0 && overlap_marks[nno] != 0;
		}
		halo_marks[b] = hit ? 1 : 0;
		if(hit) {
			const int h = atomicAdd(halo_count, 1);
			if(halo_blocks) {
				halo_blocks[3 * h] = x;
				halo_blocks[3 * h + 1] = y;
				halo_blocks[3 * h + 2] = z;
			}
		}
	}
}
// collect_grid_blocks :65-80 -- pack; reduce_grid_blocks :83-97 -- unpack + add (each destination cell is owned
// by exactly one thread per message, messages are applied one after another on the stream: plain adds, no atomics)
__global__ void collect_grid_blocks_kernel(Cfg cfg, Count count, const int* blockids, const float* grid, const int* table, float* halo_grid) {
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const int n = count.get();
	for(int h = blockIdx.x * 8 + warp; h < n; h += gridDim.x * 8) {
		const int bno = table_query(cfg, table, blockids[3 * h], blockids[3 * h + 1], blockids[3 * h + 2]);
		float4* d = reinterpret_cast<float4*>(halo_grid + (size_t) h * kGridBlockFloats);
		if(bno >= 0) {
			const float4* s = reinterpret_cast<const float4*>(grid + (size_t) bno * kGridBlockFloats);
			d[lane] = s[lane];
			d[32 + lane] = s[32 + lane];
		} else {
			d[lane] = make_float4(0.f, 0.f, 0.f, 0.f);
			d[32 + lane] = make_float4(0.f, 0.f, 0.f, 0.f);
		}
	}
}
__global__ void reduce_grid_blocks_kernel(Cfg cfg, Count count, const int* blockids, float* grid, const int* table, const float* halo_grid) {
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const int n = count.get();
	for(int h = blockIdx.x * 8 + warp; h < n; h += gridDim.x * 8) {
		const int bno = table_query(cfg, table, blockids[3 * h], blockids[3 * h + 1], blockids[3 * h + 2]);
		if(bno < 0) continue;
		const float4* s = reinterpret_cast<const float4*>(halo_grid + (size_t) h * kGridBlockFloats);
		float4* d = reinterpret_cast<float4*>(grid + (size_t) bno * kGridBlockFloats);
#pragma unroll
		for(int r = 0; r < 2; ++r) {
			float4 x = d[32 * r + lane];
			const float4 y = s[32 * r + lane];
			x.x += y.x;
			x.y += y.y;
			x.z += y.z;
			x.w += y.w;
			d[32 * r + lane] = x;
		}
	}
}

}  // namespace cb200
