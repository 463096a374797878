// sdf.cuh -- particle models sampled from an SDFGen `.sdf` level set (the reference's read_sdf + SampleGenerator,
// Library/MnSystem/IO/ParticleIO.hpp:65-97, PoissonDisk/SampleGenerator.h:68-93,149-177), with the quirks S1-S4 of DESIGN §2.7 fixed.
//   * the host side of the format: the parser (strtof, so values are bitwise those of LoadSDF's `>>`) and the sampling plan
//     (uniform fit of the node box into the domain, candidates per valid cell, lattice range);
//   * the device side: one count / write kernel pair over "items", instantiated three times:
//       classify  items = level-set cells, kept when a corner is negative, written as the ascending valid-cell list;
//       random    items = candidates j (Philox4x32-10 at counter j), kept when the trilinear phi is negative;
//       lattice   items = k^3 points per simulation cell of the range that covers the node box, kept inside the box where phi < 0.
//     count: per tile a kept count, the last CTA turns the counts into exclusive tile offsets (summary_kernel's pattern);
//     write: a second launch re-evaluates each item and writes it at its tile offset + warp-ballot rank, so rows are in item order.
//     (remove.cuh instantiates the pair twice more, over a model's rows, to keep the survivors of a removal in row order.)
// phi is read through the read-only path; the dragons' 14.6 MB stay in L2 between the passes.
// Every floating-point step of phi and of the positions is an explicitly rounded double operation, so the rows are bitwise those of
// the float64 restatement (tests/sdf_ref.py).
#pragma once
#include <algorithm>
#include <cerrno>
#include <cmath>
#include <cstdlib>
#include <string>
#include <type_traits>
#include <utility>

#include "common.cuh"

namespace cb200 {

// ---- host: the format -------------------------------------------------------------------------------------------------------------
// `ni nj nk`, `min_x min_y min_z`, `h`, then ni nj nk values with i fastest (SampleGenerator.h:68-93).  0 or cudaErrorInvalidValue.
inline int sdf_parse(const char* text, size_t bytes, cb200_sdf_header* hdr, float* phi, size_t capacity) {
	if(!text || !hdr) return (int) cudaErrorInvalidValue;
	const std::string s(text, bytes);  // strtol / strtof need a terminated string
	const char* p = s.c_str();
	const char* const end = p + s.size();
	long dims[3];
	for(int d = 0; d < 3; ++d) {
		char* e = nullptr;
		errno = 0;
		dims[d] = strtol(p, &e, 10);
		if(e == p || errno || dims[d] < 2 || dims[d] > 0x7fffffffL) return (int) cudaErrorInvalidValue;
		p = e;
	}
	const long long total = (long long) dims[0] * dims[1] * dims[2];
	if(total >= (1LL << 31)) return (int) cudaErrorInvalidValue;
	float head[4];  // min_x min_y min_z h
	for(int d = 0; d < 4; ++d) {
		char* e = nullptr;
		head[d] = strtof(p, &e);
		if(e == p || !std::isfinite(head[d])) return (int) cudaErrorInvalidValue;
		p = e;
	}
	if(!(head[3] > 0.f)) return (int) cudaErrorInvalidValue;
	if(phi && capacity < (size_t) total) return (int) cudaErrorInvalidValue;
	for(long long i = 0; i < total; ++i) {
		char* e = nullptr;
		const float v = strtof(p, &e);
		if(e == p || !std::isfinite(v)) return (int) cudaErrorInvalidValue;  // too few values, a token that is no number, inf / nan
		if(phi) phi[i] = v;
		p = e;
	}
	while(p < end && (*p == ' ' || *p == '\t' || *p == '\n' || *p == '\r' || *p == '\v' || *p == '\f')) ++p;
	if(p != end) return (int) cudaErrorInvalidValue;  // too many values (or trailing text)
	hdr->ni = (int) dims[0];
	hdr->nj = (int) dims[1];
	hdr->nk = (int) dims[2];
	for(int d = 0; d < 3; ++d) hdr->min[d] = head[d];
	hdr->h = head[3];
	return 0;
}

// ---- host: the plan ---------------------------------------------------------------------------------------------------------------
struct SdfPlan {
	int n[3];            // nodes per axis
	double offset[3];    // world position of node 0
	double c;            // world size of one level-set cell: node q maps to offset + q c
	int mode, k;         // lattice: k points per axis and simulation cell
	double spc;          // random: candidates per valid level-set cell, ppc (c / dx)^3
	double dx;
	int lo[3], ext[3];   // lattice: simulation cells [lo, lo + ext) per axis
	long long lattice_items;
};

// 0 or cudaErrorInvalidValue (bad header, mode, ppc, span, or a node box outside [0, 1]^3)
inline int sdf_plan(const cb200_config& cfg, const cb200_sdf_header& hdr, const cb200_sdf_sampling& smp, SdfPlan& P) {
	const int n[3] = {hdr.ni, hdr.nj, hdr.nk};
	for(int d = 0; d < 3; ++d)
		if(n[d] < 2) return (int) cudaErrorInvalidValue;
	if((long long) n[0] * n[1] * n[2] >= (1LL << 31) || !std::isfinite(hdr.h) || !(hdr.h > 0.f)) return (int) cudaErrorInvalidValue;
	if(smp.mode != CB200_SDF_RANDOM && smp.mode != CB200_SDF_LATTICE) return (int) cudaErrorInvalidValue;
	if(smp.ppc <= 0) return (int) cudaErrorInvalidValue;
	P.k = 0;
	if(smp.mode == CB200_SDF_LATTICE) {
		for(int k = 1; k <= 4; ++k)
			if(k * k * k == smp.ppc) P.k = k;
		if(!P.k) return (int) cudaErrorInvalidValue;
	}
	const double h = (double) hdr.h;
	double s = INFINITY;
	for(int d = 0; d < 3; ++d) {
		if(!std::isfinite(smp.span[d]) || !(smp.span[d] > 0.0) || !std::isfinite(smp.offset[d])) return (int) cudaErrorInvalidValue;
		const double sd = smp.span[d] / ((double) (n[d] - 1) * h);
		if(sd < s) s = sd;
	}
	P.c = s * h;
	P.dx = 1.0 / (double) (1 << cfg.domain_bits);
	const int cells = 1 << cfg.domain_bits;
	P.lattice_items = 1;
	for(int d = 0; d < 3; ++d) {
		P.n[d] = n[d];
		P.offset[d] = smp.offset[d];
		const double hi = smp.offset[d] + (double) (n[d] - 1) * P.c;
		if(!(smp.offset[d] >= 0.0) || !(hi <= 1.0)) return (int) cudaErrorInvalidValue;
		// every lattice point of a cell lies within half a cell of it, so one cell of margin covers the box
		P.lo[d] = std::max(0, (int) std::floor(smp.offset[d] / P.dx) - 1);
		const int top = std::min(cells, (int) std::ceil(hi / P.dx) + 2);
		P.ext[d] = top - P.lo[d];
		P.lattice_items *= P.ext[d];
	}
	const double r = P.c / P.dx;
	P.spc = (double) smp.ppc * (r * r * r);
	P.mode = smp.mode;
	P.lattice_items *= (long long) P.k * P.k * P.k;
	return 0;
}

// ---- device -----------------------------------------------------------------------------------------------------------------------
constexpr int kSdfThreads = 256;

// Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC 2011)
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
	for(int r = 0; r < 10; ++r) {
		if(r) {
			k.x += 0x9E3779B9u;
			k.y += 0xBB67AE85u;
		}
		const unsigned hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
		const unsigned hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
		c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
	}
	return c;
}

struct SdfField {
	const float* phi;
	int ni, nj;
	__device__ __forceinline__ double at(int i, int j, int k) const { return (double) __ldg(phi + i + (size_t) ni * (j + (size_t) nj * k)); }
	// fetchGridTrilinear (SampleGenerator.h:30-53) in double: its floor / ceil corners and its interpolation order, no contraction
	__device__ __forceinline__ double trilinear(double x, double y, double z) const {
		const double fx = floor(x), fy = floor(y), fz = floor(z);
		const double dx = __dsub_rn(x, fx), dy = __dsub_rn(y, fy), dz = __dsub_rn(z, fz);
		const int x0 = (int) fx, y0 = (int) fy, z0 = (int) fz, x1 = (int) ceil(x), y1 = (int) ceil(y), z1 = (int) ceil(z);
		const double c000 = at(x0, y0, z0), c001 = at(x0, y0, z1), c010 = at(x0, y1, z0), c011 = at(x0, y1, z1);
		const double c100 = at(x1, y0, z0), c101 = at(x1, y0, z1), c110 = at(x1, y1, z0), c111 = at(x1, y1, z1);
		auto lerp = [](double a, double b, double t) { return __dadd_rn(__dmul_rn(a, __dsub_rn(1.0, t)), __dmul_rn(b, t)); };
		const double c00 = lerp(c000, c100, dx), c01 = lerp(c001, c101, dx), c10 = lerp(c010, c110, dx), c11 = lerp(c011, c111, dx);
		const double c0 = lerp(c00, c10, dy), c1 = lerp(c01, c11, dy);
		return lerp(c0, c1, dz);
	}
};

// classify: cell id = i + (ni - 1) (j + (nj - 1) k) is valid when one of its eight nodes is negative (SampleGenerator.h:152-159)
struct SdfClassify {
	SdfField f;
	int* list;  // write: the valid cell ids, ascending
	using Row = int;
	__device__ __forceinline__ bool eval(long long id, Row& row) const {
		const int ci = f.ni - 1, cj = f.nj - 1;
		const int i = (int) (id % ci), j = (int) ((id / ci) % cj), k = (int) (id / ((long long) ci * cj));
		bool neg = false;
#pragma unroll
		for(int c = 0; c < 8; ++c) neg |= f.at(i + (c >> 2), j + ((c >> 1) & 1), k + (c & 1)) < 0.0;
		row = (int) id;
		return neg;
	}
	__device__ __forceinline__ void emit(long long r, const Row& row) const { list[r] = row; }
};

// random: candidate j of valid cell v for floor(v spc) <= j < floor((v + 1) spc); q = cell + u, u from Philox at counter j
struct SdfRandom {
	SdfField f;
	const int* list;
	long long n_valid;
	double spc, c, off[3];
	uint2 key;
	float* out;
	struct Row {
		float x[3];
	};
	__device__ __forceinline__ bool eval(long long j, Row& row) const {
		const double g = floor((double) j / spc);  // a guess, corrected by the two loops
		long long v = g < (double) n_valid ? (long long) g : n_valid - 1;
		while(v > 0 && floor(__dmul_rn((double) v, spc)) > (double) j) --v;
		while(v + 1 < n_valid && floor(__dmul_rn((double) (v + 1), spc)) <= (double) j) ++v;
		const int id = __ldg(list + v), ci = f.ni - 1, cj = f.nj - 1;
		const int cell[3] = {id % ci, (id / ci) % cj, id / (ci * cj)};
		const uint4 r = philox4x32_10(make_uint4((unsigned) j, (unsigned) ((unsigned long long) j >> 32), 0u, 0u), key);
		const unsigned w[3] = {r.x, r.y, r.z};
		double q[3];
#pragma unroll
		for(int d = 0; d < 3; ++d) {
			q[d] = __dadd_rn((double) cell[d], (double) (w[d] >> 8) * 0x1p-24);
			row.x[d] = __double2float_rn(__dadd_rn(off[d], __dmul_rn(q[d], c)));
		}
		return f.trilinear(q[0], q[1], q[2]) < 0.0;
	}
	__device__ __forceinline__ void emit(long long r, const Row& row) const {
#pragma unroll
		for(int d = 0; d < 3; ++d) out[3 * r + d] = row.x[d];
	}
};

// lattice: item p = (cell of the range, row-major with x slowest) k^3 + m (x slowest); x = (cell + (m - (k - 1) / 2) / k) dx,
// kept when q = (x_f32 - offset) / c lies in [0, n - 1] on every axis and phi(q) < 0
struct SdfLattice {
	SdfField f;
	int nk, k, lo[3], ext[3];
	double dx, c, off[3];
	float* out;
	struct Row {
		float x[3];
	};
	__device__ __forceinline__ bool eval(long long p, Row& row) const {
		float* x = row.x;
		const int k3 = k * k * k;
		const long long cellid = p / k3;
		const int m = (int) (p - cellid * k3);
		const int mm[3] = {m / (k * k), (m / k) % k, m % k};
		const long long yz = (long long) ext[1] * ext[2];
		const int cell[3] = {lo[0] + (int) (cellid / yz), lo[1] + (int) ((cellid / ext[2]) % ext[1]), lo[2] + (int) (cellid % ext[2])};
		const int n[3] = {f.ni, f.nj, nk};
		double q[3];
		bool in = true;
#pragma unroll
		for(int d = 0; d < 3; ++d) {
			const double a = __ddiv_rn(__dsub_rn((double) mm[d], (double) (k - 1) * 0.5), (double) k);
			x[d] = __double2float_rn(__dmul_rn(__dadd_rn((double) cell[d], a), dx));
			q[d] = __ddiv_rn(__dsub_rn((double) x[d], off[d]), c);
			in &= q[d] >= 0.0 && q[d] <= (double) (n[d] - 1);
		}
		return in && f.trilinear(q[0], q[1], q[2]) < 0.0;
	}
	__device__ __forceinline__ void emit(long long r, const Row& row) const {
#pragma unroll
		for(int d = 0; d < 3; ++d) out[3 * r + d] = row.x[d];
	}
};

// A kind may build per-CTA state (shared memory) before its first eval: prepare(), run by every thread once, barrier included.  The
// kinds without one compile to the kernels they had before it existed.
template<class G, class = void>
struct has_prepare : std::false_type {};
template<class G>
struct has_prepare<G, std::void_t<decltype(std::declval<const G&>().prepare())>> : std::true_type {};

// items [tile T, tile (T + 1)) with T = kSdfThreads * rounds; in round r thread t takes item tile_base + r kSdfThreads + t
struct SdfScan {
	long long n_items;
	int rounds;
	long long* tile_off;  // [tiles + 1]: kept count, then (last CTA) exclusive prefix; [tiles] = total
	unsigned* done;       // last-CTA counter, zero at launch
};

template<class G>
__global__ void __launch_bounds__(kSdfThreads) sdf_count_kernel(const G g, const SdfScan a) {
	__shared__ int s_warp[kSdfThreads / 32];
	__shared__ bool s_last;
	if constexpr(has_prepare<G>::value) g.prepare();
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const long long base = (long long) blockIdx.x * kSdfThreads * a.rounds;
	int cnt = 0;
	for(int r = 0; r < a.rounds; ++r) {
		const long long i = base + (long long) r * kSdfThreads + tid;
		typename G::Row row;
		cnt += (i < a.n_items && g.eval(i, row)) ? 1 : 0;
	}
	cnt = __reduce_add_sync(0xffffffffu, cnt);
	if(lane == 0) s_warp[warp] = cnt;
	__syncthreads();
	if(tid == 0) {
		int t = 0;
		for(int w = 0; w < kSdfThreads / 32; ++w) t += s_warp[w];
		a.tile_off[blockIdx.x] = t;
		__threadfence();
		s_last = atomicAdd(a.done, 1u) == gridDim.x - 1;
	}
	__syncthreads();
	if(!s_last) return;
	__threadfence();
	// the last CTA: exclusive scan of the tile counts, thread i owns the tiles [i K, (i + 1) K)
	const int tiles = (int) gridDim.x, K = (tiles + kSdfThreads - 1) / kSdfThreads;
	volatile long long* col = a.tile_off;
	long long sum = 0;
	for(int k = 0; k < K; ++k) {
		const int t = tid * K + k;
		if(t < tiles) sum += col[t];
	}
	long long inc = sum;
#pragma unroll
	for(int o = 1; o < 32; o <<= 1) {
		const long long u = __shfl_up_sync(0xffffffffu, inc, o);
		if(lane >= o) inc += u;
	}
	__shared__ long long s_wsum[kSdfThreads / 32];
	if(lane == 31) s_wsum[warp] = inc;
	__syncthreads();
	long long run = inc - sum, total = 0;
	for(int w = 0; w < kSdfThreads / 32; ++w) {
		if(w < warp) run += s_wsum[w];
		total += s_wsum[w];
	}
	for(int k = 0; k < K; ++k) {
		const int t = tid * K + k;
		if(t < tiles) {
			const long long v = col[t];
			col[t] = run;
			run += v;
		}
	}
	if(tid == 0) {
		col[tiles] = total;
		*a.done = 0u;
	}
}

template<class G>
__global__ void __launch_bounds__(kSdfThreads) sdf_write_kernel(const G g, const SdfScan a) {
	__shared__ int s_warp[2][kSdfThreads / 32];
	if constexpr(has_prepare<G>::value) g.prepare();
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const long long base = (long long) blockIdx.x * kSdfThreads * a.rounds;
	long long run = a.tile_off[blockIdx.x];
	for(int r = 0; r < a.rounds; ++r) {
		const long long i = base + (long long) r * kSdfThreads + tid;
		typename G::Row row;
		const bool kept = i < a.n_items && g.eval(i, row);
		const unsigned bal = __ballot_sync(0xffffffffu, kept);
		if(lane == 0) s_warp[r & 1][warp] = __popc(bal);
		__syncthreads();
		long long pos = run;
		int tot = 0;
#pragma unroll
		for(int w = 0; w < kSdfThreads / 32; ++w) {
			const int v = s_warp[r & 1][w];
			if(w < warp) pos += v;
			tot += v;
		}
		if(kept) g.emit(pos + __popc(bal & ((1u << lane) - 1u)), row);
		run += tot;
		// s_warp is double-buffered: round r + 2 writes this half only after every thread has passed round r + 1's barrier
	}
}

}  // namespace cb200
