// checkpoint.cuh -- portable checkpoint of a running simulation (layout: include/claymore_b200.h, "Checkpoint / restore").
//   * the one parser of the blob format (host only: cb200_checkpoint_inspect and cb200_sim_restore share it) and its writer;
//   * the row gather every particle read-out shares, and its state rows (retrieve, particle_state);
//   * the snapshot gather: every model's particles and the keyed grid blocks of grid[0] packed into a device staging blob in
//     partition order, in one launch behind a scan of the per-block particle counts;
//   * the restore kernels: the positions of a saved state and a keyed scatter of the saved grid blocks (array_to_buffer_kernel,
//     init.cuh, puts the saved rows into the bins).
#pragma once
#include <algorithm>
#include <cstring>
#include <type_traits>
#include <vector>

#include "common.cuh"

namespace cb200 {

constexpr size_t kCkHeader = CB200_CHECKPOINT_HEADER_BYTES;
constexpr size_t kCkTocEntry = 96;
constexpr size_t kCkAlign = 256;
constexpr char kCkMagic[8] = {'C', 'B', '2', '0', '0', 'C', 'K', 'P'};
static_assert(256 + kMaxModels * kCkTocEntry <= kCkHeader, "checkpoint table of contents must fit the header");

__host__ __device__ inline unsigned long long ck_align(unsigned long long x) { return (x + kCkAlign - 1) & ~(unsigned long long) (kCkAlign - 1); }

// Section offsets of the blob the snapshot writes, from the particle counts and nbc: the host writer of the header evaluates it
// on the counts the gather kernel left on the device, and the kernel walks the same sections in its prologue.
struct CkLayout {
	unsigned long long model_off[kMaxModels], model_bytes[kMaxModels];
	unsigned long long keys_off, keys_bytes, grid_off, grid_bytes, total;
};
__host__ __device__ inline CkLayout ck_layout(int n_models, const int* materials, const long long* counts, long long nbc) {
	CkLayout L {};
	unsigned long long o = kCkHeader;
	for(int m = 0; m < n_models; ++m) {
		L.model_off[m] = o;
		L.model_bytes[m] = (unsigned long long) counts[m] * ck_channels(materials[m]) * sizeof(float);
		o = ck_align(o + L.model_bytes[m]);
	}
	L.keys_off = o;
	L.keys_bytes = (unsigned long long) nbc * 3 * sizeof(int);
	L.grid_off = ck_align(o + L.keys_bytes);
	L.grid_bytes = (unsigned long long) nbc * kGridBlockFloats * sizeof(float);
	L.total = L.grid_off + L.grid_bytes;
	return L;
}

// ---- host: the format ---------------------------------------------------------------------------------------------
// The format is little-endian and so is every host this library builds for (x86-64, aarch64): fields are copied as they lie.
template<typename T>
inline T ck_get(const unsigned char* p, size_t off) {
	T v;
	memcpy(&v, p + off, sizeof(T));
	return v;
}
template<typename T>
inline void ck_put(unsigned char* p, size_t off, T v) { memcpy(p + off, &v, sizeof(T)); }

// the sixteen 4-byte material parameters of a table-of-contents entry, in cb200_particle_buffer order
inline void ck_put_params(unsigned char* e, const cb200_particle_buffer& b) {
	const float f[11] = {b.rho, b.volume, b.mass, b.bulk, b.gamma, b.viscosity, b.lambda, b.mu, b.cohesion, b.beta, b.yield_surface};
	memcpy(e, f, sizeof(f));
	ck_put<int>(e, 44, b.volume_correction);
	ck_put<float>(e, 48, b.bm);
	ck_put<float>(e, 52, b.xi);
	ck_put<float>(e, 56, b.msqr);
	ck_put<int>(e, 60, b.hardening_on);
}
inline void ck_get_params(const unsigned char* e, int material, cb200_particle_buffer& b) {
	memset(&b, 0, sizeof(b));
	b.material = material;
	float f[11];
	memcpy(f, e, sizeof(f));
	b.rho = f[0], b.volume = f[1], b.mass = f[2], b.bulk = f[3], b.gamma = f[4], b.viscosity = f[5];
	b.lambda = f[6], b.mu = f[7], b.cohesion = f[8], b.beta = f[9], b.yield_surface = f[10];
	b.volume_correction = ck_get<int>(e, 44);
	b.bm = ck_get<float>(e, 48);
	b.xi = ck_get<float>(e, 52);
	b.msqr = ck_get<float>(e, 56);
	b.hardening_on = ck_get<int>(e, 60);
}

// Header of a blob described by `info` (sections, counts and clock filled in by the caller).
inline void ck_write_header(unsigned char* h, const cb200_checkpoint_info& info) {
	memset(h, 0, kCkHeader);
	memcpy(h, kCkMagic, 8);
	ck_put<unsigned>(h, 8, info.version);
	ck_put<unsigned>(h, 12, (unsigned) info.n_models);
	ck_put<unsigned long long>(h, 16, info.bytes);
	ck_put<int>(h, 24, info.cfg.domain_bits);
	ck_put<int>(h, 28, info.cfg.max_ppc);
	ck_put<int>(h, 32, info.cfg.boundary);
	ck_put<float>(h, 36, info.cfg.gravity);
	ck_put<float>(h, 40, info.cfg.cfl);
	ck_put<float>(h, 44, info.dt_default);
	ck_put<int>(h, 48, info.fps);
	ck_put<int>(h, 52, info.mgsp_rank);
	ck_put<int>(h, 56, info.mgsp_world);
	ck_put<int>(h, 60, info.error);
	ck_put<float>(h, 64, info.dt);
	ck_put<float>(h, 68, info.next_dt);
	ck_put<float>(h, 72, info.step_time);
	ck_put<float>(h, 76, info.frame_time);
	ck_put<double>(h, 80, info.sim_time);
	ck_put<long long>(h, 88, info.steps);
	ck_put<long long>(h, 96, info.frames);
	ck_put<int>(h, 104, info.particle_block_count);
	ck_put<int>(h, 108, info.neighbor_block_count);
	ck_put<int>(h, 112, info.exterior_block_count);
	ck_put<int>(h, 116, info.max_blocks);
	ck_put<unsigned long long>(h, 120, info.keys_offset);
	ck_put<unsigned long long>(h, 128, info.keys_bytes);
	ck_put<unsigned long long>(h, 136, info.grid_offset);
	ck_put<unsigned long long>(h, 144, info.grid_bytes);
	for(int m = 0; m < info.n_models; ++m) {
		unsigned char* e = h + 256 + kCkTocEntry * m;
		const cb200_checkpoint_model& md = info.models[m];
		ck_put<int>(e, 0, md.material);
		ck_put<int>(e, 4, md.channels);
		ck_put<long long>(e, 8, md.count);
		ck_put<unsigned long long>(e, 16, md.offset);
		ck_put<unsigned long long>(e, 24, md.bytes);
		ck_put_params(e + 32, md.params);
	}
}

// The parser: every check of cb200_checkpoint_inspect, before anything reads a data section other than the keys.
inline int ck_parse(const void* blob, size_t bytes, cb200_checkpoint_info* out) {
	const int bad = (int) cudaErrorInvalidValue;
	if(!blob || !out || bytes < kCkHeader) return bad;
	const unsigned char* h = static_cast<const unsigned char*>(blob);
	if(memcmp(h, kCkMagic, 8) != 0) return bad;
	cb200_checkpoint_info I;
	memset(&I, 0, sizeof(I));
	I.version = ck_get<unsigned>(h, 8);
	if(I.version != CB200_CHECKPOINT_VERSION) return bad;
	const unsigned nm = ck_get<unsigned>(h, 12);
	if(nm < 1 || nm > (unsigned) kMaxModels) return bad;
	I.n_models = (int) nm;
	I.bytes = ck_get<unsigned long long>(h, 16);
	if(I.bytes != (unsigned long long) bytes) return bad;  // truncated, or trailing bytes
	I.cfg.domain_bits = ck_get<int>(h, 24);
	I.cfg.max_ppc = ck_get<int>(h, 28);
	I.cfg.boundary = ck_get<int>(h, 32);
	I.cfg.gravity = ck_get<float>(h, 36);
	I.cfg.cfl = ck_get<float>(h, 40);
	if(!cfg_valid(I.cfg)) return bad;
	I.dt_default = ck_get<float>(h, 44);
	I.fps = ck_get<int>(h, 48);
	I.mgsp_rank = ck_get<int>(h, 52);
	I.mgsp_world = ck_get<int>(h, 56);
	if(I.mgsp_world < 1 || I.mgsp_rank < 0 || I.mgsp_rank >= I.mgsp_world) return bad;
	I.error = ck_get<int>(h, 60);
	I.dt = ck_get<float>(h, 64);
	I.next_dt = ck_get<float>(h, 68);
	I.step_time = ck_get<float>(h, 72);
	I.frame_time = ck_get<float>(h, 76);
	I.sim_time = ck_get<double>(h, 80);
	I.steps = ck_get<long long>(h, 88);
	I.frames = ck_get<long long>(h, 96);
	I.particle_block_count = ck_get<int>(h, 104);
	I.neighbor_block_count = ck_get<int>(h, 108);
	I.exterior_block_count = ck_get<int>(h, 112);
	I.max_blocks = ck_get<int>(h, 116);
	const int pbc = I.particle_block_count, nbc = I.neighbor_block_count, ebc = I.exterior_block_count;
	if(pbc < 1 || nbc < pbc || ebc < nbc) return bad;
	I.keys_offset = ck_get<unsigned long long>(h, 120);
	I.keys_bytes = ck_get<unsigned long long>(h, 128);
	I.grid_offset = ck_get<unsigned long long>(h, 136);
	I.grid_bytes = ck_get<unsigned long long>(h, 144);
	if(I.keys_bytes != (unsigned long long) nbc * 12 || I.grid_bytes != (unsigned long long) nbc * kGridBlockFloats * sizeof(float)) return bad;
	std::vector<std::pair<unsigned long long, unsigned long long>> sec;  // [begin, end) of every data section
	for(int m = 0; m < I.n_models; ++m) {
		const unsigned char* e = h + 256 + kCkTocEntry * m;
		cb200_checkpoint_model& md = I.models[m];
		md.material = ck_get<int>(e, 0);
		if(md.material < 0 || md.material > 3) return bad;
		md.channels = ck_get<int>(e, 4);
		md.count = ck_get<long long>(e, 8);
		md.offset = ck_get<unsigned long long>(e, 16);
		md.bytes = ck_get<unsigned long long>(e, 24);
		if(md.channels != ck_channels(md.material) || md.count <= 0 || md.count > 0x7fffffffLL) return bad;
		if(md.bytes != (unsigned long long) md.count * md.channels * sizeof(float)) return bad;
		ck_get_params(e + 32, md.material, md.params);
		sec.emplace_back(md.offset, md.bytes);
	}
	sec.emplace_back(I.keys_offset, I.keys_bytes);
	sec.emplace_back(I.grid_offset, I.grid_bytes);
	for(auto& s : sec) {  // (offset, size) -> [begin, end), with the size checked against the room left so nothing wraps
		if(s.first < kCkHeader || s.first > I.bytes || s.second > I.bytes - s.first) return bad;
		s.second += s.first;
	}
	std::sort(sec.begin(), sec.end());
	for(size_t i = 1; i < sec.size(); ++i)
		if(sec[i].first < sec[i - 1].second) return bad;
	// every key inside the domain, no key twice
	const int G = 1 << (I.cfg.domain_bits - 2);
	std::vector<long long> hk((size_t) nbc);
	for(int b = 0; b < nbc; ++b) {
		int k[3];
		memcpy(k, h + I.keys_offset + (size_t) b * 12, 12);
		for(int d = 0; d < 3; ++d)
			if(k[d] < 0 || k[d] >= G) return bad;
		hk[b] = ((long long) k[0] * G + k[1]) * G + k[2];
	}
	std::sort(hk.begin(), hk.end());
	if(std::adjacent_find(hk.begin(), hk.end()) != hk.end()) return bad;
	*out = I;
	return 0;
}

// ---- device: the row gather ---------------------------------------------------------------------------------------------------
// Every read-out of particles (snapshot, frame output, retrieve / particle_state) walks the current partition's buckets with one
// routine, so all of them emit rows in one order: particle blocks in partition order, then bucket order inside a block.
constexpr int kGatherThreads = 256;

// where the particles of every model are read from
struct GatherSrc {
	int n_models;
	int material[kMaxModels];
	PBuf cur[kMaxModels];          // the bins the particles live in
	PBuf next[kMaxModels];         // the buckets of the current partition: advection tags into `cur`
	const int* base[kMaxModels];   // [pbc + 1]: exclusive scan of next.particle_bucket_sizes (entry pbc: the model's count)
	int cap[kMaxModels];           // rows the model's section of the destination holds (its particle count)
	const int* keys;               // current partition
	const int* prev_table;         // the partition the tags point into
};

// f(std::integral_constant<int, C>) with the material's channel count C as a compile-time value
template<class F>
__device__ __forceinline__ void with_channels(int material, F&& f) {
	switch(material) {
	case CB200_J_FLUID: f(std::integral_constant<int, 4>()); break;
	case CB200_FIXED_COROTATED: f(std::integral_constant<int, 12>()); break;
	default: f(std::integral_constant<int, 13>()); break;
	}
}

// A state row: the first W of the C channels of a particle (the snapshot and particle_state: W = C, retrieve: W = 3)
template<int C_, int W>
struct StateRow {
	static constexpr int C = C_;
	__device__ __forceinline__ int words() const { return W; }
	__device__ __forceinline__ void operator()(float* rec, const float* __restrict__ src) const {
#pragma unroll
		for(int c = 0; c < W; ++c) rec[c] = src ? __ldg(src + c * 32) : 0.f;
	}
};

// One particle block b of model m: each warp takes 32 rows, resolves each tag to its slot in the bins (one row per lane, the source
// reads coalesced along the bin lanes), has `row` fill the lane's row of a shared tile, and writes the tile's 32 rows of
// row.words() words to `out` as one contiguous run, rows below the model's cap only.  `row` gets src == nullptr for a tag without a
// source block: the partition lost that particle (error bit set by the sub-step) and its row is zeros.
template<class Row, class T>
__device__ __forceinline__ void gather_block(const Cfg& cfg, const GatherSrc& g, int m, int b, int kx, int ky, int kz, T* out, T* tile, const Row& row) {
	const int W = row.words(), S = W | 1;  // odd row stride: the lanes' row writes fall on distinct banks
	constexpr int binf = Row::C == 4 ? 128 : 512;
	const PBuf cur = g.cur[m], nx = g.next[m];
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const int cnt = nx.particle_bucket_sizes[b];
	const long long row0 = g.base[m][b];
	for(int c0 = warp * 32; c0 < cnt; c0 += kGatherThreads) {
		const int i = c0 + lane;
		if(i < cnt) {
			const int tag = __ldg(nx.blockbuckets + ((size_t) b << cfg.ppb_shift) + i);
			const int dir = tag >> cfg.ppb_shift, sp = tag & (cfg.ppb - 1);
			const int sno = table_query(cfg, g.prev_table, kx + dir / 9 - 1, ky + (dir / 3) % 3 - 1, kz + dir % 3 - 1);
			row(tile + lane * S, sno >= 0 ? bin_slot(cur.bins, __ldg(cur.bin_offsets + sno), sp, binf) : nullptr);
		}
		__syncwarp();
		const int rows = min(min(32, cnt - c0), g.cap[m] - (int) (row0 + c0));
		T* dst = out + (size_t) (row0 + c0) * W;
		for(int j = lane; j < rows * W; j += 32) dst[j] = tile[(j / W) * S + j % W];
		__syncwarp();
	}
}

// One model's state rows, the first 3 channels of each (positions) or all of them, for retrieve and particle_state
template<bool kPositions>
__global__ void __launch_bounds__(kGatherThreads) state_rows_kernel(const Cfg cfg, const StepState* state, const GatherSrc g, int m, float* out) {
	__shared__ float s_tile[kGatherThreads / 32][32 * (kPositions ? 3 : 13)];
	const int pbc = state->pbc;
	float* tile = s_tile[threadIdx.x >> 5];
	for(int u = blockIdx.x; u < pbc; u += gridDim.x) {
		const int kx = g.keys[3 * u], ky = g.keys[3 * u + 1], kz = g.keys[3 * u + 2];
		with_channels(g.material[m], [&](auto c) {
			constexpr int C = decltype(c)::value;
			gather_block(cfg, g, m, u, kx, ky, kz, out, tile, StateRow<C, kPositions ? 3 : C>());
		});
	}
}

// ---- device: snapshot -------------------------------------------------------------------------------------------------
struct SnapshotArgs {
	Cfg cfg;
	const StepState* state;
	GatherSrc src;
	const float* grid;             // grid[0]
	unsigned char* out;            // staging blob (the header is written by the host)
};

// One launch: units [0, pbc) are particle blocks (all models of the block), units [pbc, pbc + ceil(nbc / 8)) eight grid blocks each
// (a warp per block: its key and its 1 KiB as float4).
__global__ void __launch_bounds__(kGatherThreads) snapshot_kernel(const SnapshotArgs a) {
	__shared__ float s_tile[kGatherThreads / 32][32 * 13];
	__shared__ unsigned long long s_off[kMaxModels + 2];
	const GatherSrc& g = a.src;
	const int pbc = a.state->pbc, nbc = a.state->nbc;
	if(threadIdx.x == 0) {  // ck_layout's walk, one section at a time (no local arrays)
		unsigned long long o = kCkHeader;
		for(int m = 0; m < g.n_models; ++m) {
			s_off[m] = o;
			o = ck_align(o + (unsigned long long) g.base[m][pbc] * ck_channels(g.material[m]) * sizeof(float));
		}
		s_off[kMaxModels] = o;
		s_off[kMaxModels + 1] = ck_align(o + (unsigned long long) nbc * 3 * sizeof(int));
	}
	__syncthreads();
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	float* tile = s_tile[warp];
	const int units = pbc + (nbc + 7) / 8;
	for(int u = blockIdx.x; u < units; u += gridDim.x) {
		if(u < pbc) {
			const int kx = g.keys[3 * u], ky = g.keys[3 * u + 1], kz = g.keys[3 * u + 2];
			for(int m = 0; m < g.n_models; ++m) {
				float* out = reinterpret_cast<float*>(a.out + s_off[m]);
				with_channels(g.material[m], [&](auto c) {
					constexpr int C = decltype(c)::value;
					gather_block(a.cfg, g, m, u, kx, ky, kz, out, tile, StateRow<C, C>());
				});
			}
		} else {
			const int b = (u - pbc) * 8 + warp;
			if(b < nbc) {
				int* keys = reinterpret_cast<int*>(a.out + s_off[kMaxModels]);
				if(lane < 3) keys[3 * b + lane] = g.keys[3 * b + lane];
				const float4* s = reinterpret_cast<const float4*>(a.grid + (size_t) b * kGridBlockFloats);
				float4* d = reinterpret_cast<float4*>(a.out + s_off[kMaxModels + 1]) + (size_t) b * (kGridBlockFloats / 4);
				d[lane] = s[lane];
				d[32 + lane] = s[32 + lane];
			}
		}
	}
}

// ---- device: restore -----------------------------------------------------------------------------------------------------
// the positions of a saved state, as the AoS array the set-up kernels read
__global__ void state_positions_kernel(long long n, int channels, const float* state, float* pos) {
	for(long long p = blockIdx.x * (long long) blockDim.x + threadIdx.x; p < n; p += (long long) gridDim.x * blockDim.x)
		for(int d = 0; d < 3; ++d) pos[3 * p + d] = state[p * channels + d];
}

// keyed grid scatter: warp per saved block, table query, float4 copy.  A saved key without a block among the first `nbc` of the
// rebuilt partition is counted in *missing and skipped.
__global__ void scatter_grid_kernel(Cfg cfg, int count, const int* keys, const float* blocks, const int* table, int nbc, float* grid, int* missing) {
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	for(int h = blockIdx.x * 8 + warp; h < count; h += gridDim.x * 8) {
		const int bno = table_query(cfg, table, keys[3 * h], keys[3 * h + 1], keys[3 * h + 2]);
		if(bno < 0 || bno >= nbc) {
			if(lane == 0) atomicAdd(missing, 1);
			continue;
		}
		const float4* s = reinterpret_cast<const float4*>(blocks + (size_t) h * kGridBlockFloats);
		float4* d = reinterpret_cast<float4*>(grid + (size_t) bno * kGridBlockFloats);
		d[lane] = s[lane];
		d[32 + lane] = s[32 + lane];
	}
}

}  // namespace cb200
