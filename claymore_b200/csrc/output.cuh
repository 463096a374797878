// output.cuh -- per-frame particle output as point-only BGEO V5 files (the reference's output_model + write_partio,
// gmpm_simulator.cuh:594-634, ParticleIO.hpp:14-28, written by partio's writeBGEO).
//   * the device gather: every model's points packed as big-endian BGEO point records into a staging buffer, one launch behind
//     the checkpoint's scan of the per-block particle counts, rows in the checkpoint's order (partition order, then bucket order);
//   * the host side of the format: the header with the attribute definitions, and the trailer.  The body is produced on the GPU.
//
// A record is  x y z 1.0 [v_x v_y v_z] [J], every word big-endian:
//   * v: MLS-MPM keeps no particle velocity.  At a sub-step boundary the motion lives in grid[0], the carried P2G mass and
//     momentum of the current partition, so v is the G2P of that grid's node velocities at the particle's stored position,
//     v_p = sum_i w_ip (mv_i / m_i) (0 where m_i = 0), with g2p2g's base cell and quadratic B-spline weights.  Right after
//     initial_setup with a uniform initial velocity v0 this is v0 (the rasterised momentum is m v0 at every node).
//     MGSP: grid[0]'s blocks hold the full sums on every rank that has them, and a particle's stencil lies in the 2x2x2 blocks of
//     its particle block, which are the blocks its next G2P reads; so the read sees the same node velocities as that G2P.
//   * J: the fluid's channel 3; det F for FIXED_COROTATED, SAND and NACC.
#pragma once
#include <cstring>
#include <vector>

#include "math3.cuh"

namespace cb200 {

constexpr unsigned kOutAttrs = CB200_OUTPUT_V | CB200_OUTPUT_J;
__host__ __device__ inline int out_words(unsigned attrs) { return 4 + ((attrs & CB200_OUTPUT_V) ? 3 : 0) + ((attrs & CB200_OUTPUT_J) ? 1 : 0); }

// ---- host: the format ------------------------------------------------------------------------------------------------------
// Header of a point-only BGEO V5 file as partio's writeBGEO lays it out: magic "Bgeo", 'V', then nine big-endian int32 (version 5,
// points, primitives, point groups, primitive groups, point attributes, vertex attributes, primitive attributes, detail
// attributes), then per point attribute other than the position: int16 name length, the name, uint16 size, int32 type (0 float,
// 5 vector) and `size` int32 zero defaults.  Empty when the point count does not fit the 32-bit field.
inline std::vector<unsigned char> bgeo_header(long long points, unsigned attrs) {
	std::vector<unsigned char> h;
	if(points < 0 || points > 0x7fffffffLL || (attrs & ~kOutAttrs)) return h;
	auto be = [&h](unsigned v, int bytes) {
		for(int i = bytes - 1; i >= 0; --i) h.push_back((unsigned char) (v >> (8 * i)));
	};
	const char head[5] = {'B', 'g', 'e', 'o', 'V'};
	h.insert(h.end(), head, head + 5);
	const unsigned nattr = ((attrs & CB200_OUTPUT_V) ? 1 : 0) + ((attrs & CB200_OUTPUT_J) ? 1 : 0);
	const unsigned fields[9] = {5u, (unsigned) points, 0u, 0u, 0u, nattr, 0u, 0u, 0u};
	for(unsigned f : fields) be(f, 4);
	auto attribute = [&](const char* name, unsigned size, unsigned type) {
		const unsigned len = (unsigned) strlen(name);
		be(len, 2);
		h.insert(h.end(), name, name + len);
		be(size, 2);
		be(type, 4);
		for(unsigned i = 0; i < size; ++i) be(0u, 4);
	};
	if(attrs & CB200_OUTPUT_V) attribute("v", 3, 5);
	if(attrs & CB200_OUTPUT_J) attribute("J", 1, 0);
	return h;
}
// what follows the body: no detail attributes (nothing), then the two bytes partio's writer ends every file with
constexpr unsigned char kBgeoTrailer[2] = {0x00, 0xff};

// ---- device: the gather ------------------------------------------------------------------------------------------------------
constexpr int kOutThreads = 256;
struct OutputArgs {
	Cfg cfg;
	const StepState* state;
	int n_models;
	unsigned attrs;
	int material[kMaxModels];
	PBuf cur[kMaxModels];          // the bins the particles live in
	PBuf next[kMaxModels];         // the buckets of the current partition: advection tags into `cur`
	const int* base[kMaxModels];   // [pbc + 1]: exclusive scan of next.particle_bucket_sizes (the checkpoint's scan)
	long long cap[kMaxModels];     // rows the model's staging section holds (its particle count)
	unsigned long long off[kMaxModels];  // byte offset of the model's section in `out`
	const int* keys;               // current partition
	const int* table;              // current partition: grid[0]'s block numbers
	const int* prev_table;         // the partition the tags point into
	const float* grid;             // grid[0]: mass and momentum
	unsigned char* out;
};

__device__ __forceinline__ unsigned be32(float f) { return __byte_perm(__float_as_uint(f), 0, 0x0123); }

// One particle block of one model, snapshot_block's pattern: each warp takes 32 rows, gathers them through the tags (one row per
// lane), builds the records in a shared tile and writes the tile's 32 * W words as one contiguous run.
template<int C>
__device__ __forceinline__ void output_block(const OutputArgs& a, int m, int b, int kx, int ky, int kz, const float4* __restrict__ vel, unsigned* tile) {
	const Cfg& cfg = a.cfg;
	const PBuf cur = a.cur[m], nx = a.next[m];
	const bool want_v = a.attrs & CB200_OUTPUT_V, want_j = a.attrs & CB200_OUTPUT_J;
	const int W = out_words(a.attrs), S = W | 1;  // odd row stride: the lanes' row writes fall on distinct banks
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	const int cnt = nx.particle_bucket_sizes[b];
	const long long row0 = a.base[m][b];
	const int binf = C == 4 ? 128 : 512;
	unsigned* out = reinterpret_cast<unsigned*>(a.out + a.off[m]);
	for(int c0 = warp * 32; c0 < cnt; c0 += kOutThreads) {
		const int i = c0 + lane;
		if(i < cnt) {
			float p[3] = {0.f, 0.f, 0.f}, v[3] = {0.f, 0.f, 0.f}, J = 0.f;
			const int tag = __ldg(nx.blockbuckets + ((size_t) b << cfg.ppb_shift) + i);
			const int dir = tag >> cfg.ppb_shift, sp = tag & (cfg.ppb - 1);
			const int sno = table_query(cfg, a.prev_table, kx + dir / 9 - 1, ky + (dir / 3) % 3 - 1, kz + dir % 3 - 1);
			if(sno >= 0) {  // (a tag without a source block: the partition lost this particle; the record is zero, as in the checkpoint)
				const float* src = cur.bins + ((size_t) __ldg(cur.bin_offsets + sno) + (sp >> 5)) * binf + (sp & 31);
#pragma unroll
				for(int d = 0; d < 3; ++d) p[d] = __ldg(src + d * 32);
				if(want_j) {
					if constexpr(C == 4) {
						J = __ldg(src + 96);
					} else {
						float F[9];
#pragma unroll
						for(int c = 0; c < 9; ++c) F[c] = __ldg(src + (3 + c) * 32);
						J = F[0] * (F[4] * F[8] - F[7] * F[5]) - F[3] * (F[1] * F[8] - F[7] * F[2]) + F[6] * (F[1] * F[5] - F[4] * F[2]);
					}
				}
				if(want_v) {  // g2p2g's G2P: base cell, local position, weights, node (ab + i) of the 8^3 arena
					int ab[3];
					float w[3][3];
#pragma unroll
					for(int d = 0; d < 3; ++d) {
						const int base = cell_index(cfg, p[d]) - 1;
						const float lp = p[d] - base * cfg.dx;
						bspline_weights(lp * cfg.dx_inv, w[d][0], w[d][1], w[d][2]);
						ab[d] = ((base - 1) & 3) + 1;
					}
#pragma unroll
					for(int x = 0; x < 3; ++x)
#pragma unroll
						for(int y = 0; y < 3; ++y)
#pragma unroll
							for(int z = 0; z < 3; ++z) {
								const float wt = w[0][x] * w[1][y] * w[2][z];
								const float4 n = vel[((ab[0] + x) * 8 + ab[1] + y) * 8 + ab[2] + z];
								v[0] = fmaf(wt, n.x, v[0]);
								v[1] = fmaf(wt, n.y, v[1]);
								v[2] = fmaf(wt, n.z, v[2]);
							}
				}
			}
			unsigned* rec = tile + lane * S;
			rec[0] = be32(p[0]);
			rec[1] = be32(p[1]);
			rec[2] = be32(p[2]);
			rec[3] = be32(1.f);
			int k = 4;
			if(want_v) {
				rec[4] = be32(v[0]);
				rec[5] = be32(v[1]);
				rec[6] = be32(v[2]);
				k = 7;
			}
			if(want_j) rec[k] = be32(J);
		}
		__syncwarp();
		const long long rows = min((long long) min(32, cnt - c0), a.cap[m] - (row0 + c0));
		unsigned* dst = out + (size_t) (row0 + c0) * W;
		for(int j = lane; j < rows * W; j += 32) dst[j] = tile[(j / W) * S + j % W];
		__syncwarp();
	}
}

// One launch: a CTA per particle block (persistent).  With v requested, the block's 2x2x2 grid blocks of grid[0] are staged through
// the current table and turned into node velocities in shared memory once (zero where a block is missing or a node has no mass).
__global__ void __launch_bounds__(kOutThreads) output_kernel(const OutputArgs a) {
	__shared__ float4 s_vel[512];  // node (X * 8 + Y) * 8 + Z of the arena, as in g2p2g
	__shared__ unsigned s_tile[kOutThreads / 32][32 * 9];
	__shared__ int s_bno[8];
	const int pbc = a.state->pbc;
	const bool want_v = a.attrs & CB200_OUTPUT_V;
	unsigned* tile = s_tile[threadIdx.x >> 5];
	for(int u = blockIdx.x; u < pbc; u += gridDim.x) {
		const int kx = a.keys[3 * u], ky = a.keys[3 * u + 1], kz = a.keys[3 * u + 2];
		if(want_v) {
			__syncthreads();  // the previous block's readers of s_vel are done
			if(threadIdx.x < 8) s_bno[threadIdx.x] = table_query(a.cfg, a.table, kx + ((threadIdx.x >> 2) & 1), ky + ((threadIdx.x >> 1) & 1), kz + (threadIdx.x & 1));
			__syncthreads();
			for(int n = threadIdx.x; n < 512; n += kOutThreads) {
				const int X = n >> 6, Y = (n >> 3) & 7, Z = n & 7;
				const int bno = s_bno[((X >> 2) << 2) | ((Y >> 2) << 1) | (Z >> 2)];
				float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
				if(bno >= 0) {
					const float* g = a.grid + (size_t) bno * kGridBlockFloats + (((X & 3) << 4) | ((Y & 3) << 2) | (Z & 3));
					const float mass = __ldg(g);
					if(mass > 0.f) v = make_float4(__ldg(g + 64) / mass, __ldg(g + 128) / mass, __ldg(g + 192) / mass, 0.f);
				}
				s_vel[n] = v;
			}
			__syncthreads();
		}
		for(int m = 0; m < a.n_models; ++m) {
			switch(a.material[m]) {
			case CB200_J_FLUID: output_block<4>(a, m, u, kx, ky, kz, s_vel, tile); break;
			case CB200_FIXED_COROTATED: output_block<12>(a, m, u, kx, ky, kz, s_vel, tile); break;
			default: output_block<13>(a, m, u, kx, ky, kz, s_vel, tile); break;
			}
		}
	}
}

}  // namespace cb200
