// mesh.cuh -- level sets from triangle meshes: SDFGen's make_level_set3 (Externals/SDFGen/makelevelset3.cpp:118-183) on the device,
// bit for bit, and a Wavefront OBJ parser with the quirks M1-M8 of DESIGN §2.12 fixed.
//   * host: obj_parse (two calls, like sdf_parse) and mesh_header (SDFGen's main, main.cpp:63-118, in float arithmetic);
//   * device, in stream order:
//       setup     one thread per triangle: its band box and its crossing columns, and both item counts (64-bit);
//       scan      exclusive prefix of the (band, crossing) counts over the triangles (tile sums, the last CTA scans them, then a
//                 second launch writes every prefix), so no thread owns a whole triangle: one large triangle spreads over the grid;
//       band      one item per (triangle, band node): point_triangle_distance, kept by a 64-bit atomicMin on (bits of d) << 32 | t,
//                 which orders as SDFGen's strict `<` over triangles in order (smallest d, then lowest t);
//       crossing  one item per (triangle, (j, k) column): point_in_triangle_2d with SOS orientation in double, then fi, ceil and the
//                 enlarged first interval; the counts are integer atomics, so their order does not matter;
//       sweep     one cooperative persistent kernel: 2 x 8 directions in SDFGen's order; within a direction node (i, j, k) reads only
//                 its 7 upstream neighbours (direction-adjusted index sums 1-3 lower) and writes only itself, so the diagonal planes
//                 i' + j' + k' = s in increasing s, with a grid barrier between planes, give the sequential Gauss-Seidel result;
//       sign      one warp per (j, k) row: the prefix parity of the counts along i negates phi; phi overwrites the counts.
// Every floating-point operation is an explicitly rounded intrinsic: the library builds with nvcc's default -fmad=true, and one
// contracted multiply-add would break bit identity with SDFGen's float / double arithmetic.
#pragma once
#include <cerrno>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include <cooperative_groups.h>

#include "common.cuh"

namespace cb200 {

// ---- host: OBJ -------------------------------------------------------------------------------------------------------------------
// `v x y z [w ...]` and `f a b c [d ...]` with a = index, index/uv, index//n or index/uv/n; negative indices count back from the
// last vertex read; polygons become the fan (v0, v_i, v_{i+1}).  Every other line is ignored.  0 or cudaErrorInvalidValue.
inline int obj_parse(const char* text, size_t bytes, cb200_mesh_header* hdr, float* vertices, int* triangles, size_t v_capacity, size_t t_capacity) {
	if(!hdr || (!text && bytes)) return (int) cudaErrorInvalidValue;
	const std::string s(text ? text : "", bytes);
	std::vector<float> v;
	std::vector<long long> f;  // 0-based vertex indices, three per triangle, checked against the final count below
	const char* p = s.c_str();
	const char* const end = p + s.size();
	auto space = [](char c) { return c == ' ' || c == '\t' || c == '\r' || c == '\v' || c == '\f'; };
	while(p < end) {
		const char* eol = p;
		while(eol < end && *eol != '\n') ++eol;
		std::string line(p, eol);
		p = eol < end ? eol + 1 : end;
		std::vector<std::string> tok;
		for(size_t a = 0; a < line.size();) {
			while(a < line.size() && space(line[a])) ++a;
			size_t b = a;
			while(b < line.size() && !space(line[b])) ++b;
			if(b > a) tok.emplace_back(line, a, b - a);
			a = b;
		}
		if(tok.empty()) continue;
		if(tok[0] == "v") {
			if(tok.size() < 4) return (int) cudaErrorInvalidValue;
			for(int d = 1; d <= 3; ++d) {
				char* e = nullptr;
				const float x = strtof(tok[d].c_str(), &e);
				if(e == tok[d].c_str() || *e || !std::isfinite(x)) return (int) cudaErrorInvalidValue;
				v.push_back(x);
			}
			if(v.size() / 3 > 0x7fffffffULL) return (int) cudaErrorInvalidValue;
		} else if(tok[0] == "f") {
			if(tok.size() < 4) return (int) cudaErrorInvalidValue;
			std::vector<long long> poly;
			for(size_t a = 1; a < tok.size(); ++a) {
				char* e = nullptr;
				errno = 0;
				const long long r = strtoll(tok[a].c_str(), &e, 10);
				if(e == tok[a].c_str() || errno || (*e && *e != '/') || r == 0) return (int) cudaErrorInvalidValue;
				const long long idx = r > 0 ? r - 1 : (long long) (v.size() / 3) + r;
				if(idx < 0) return (int) cudaErrorInvalidValue;
				poly.push_back(idx);
			}
			for(size_t a = 1; a + 1 < poly.size(); ++a) {
				f.push_back(poly[0]);
				f.push_back(poly[a]);
				f.push_back(poly[a + 1]);
			}
			if(f.size() / 3 > 0x7fffffffULL) return (int) cudaErrorInvalidValue;
		}
	}
	const long long nv = (long long) v.size() / 3, nt = (long long) f.size() / 3;
	for(long long i : f)
		if(i >= nv) return (int) cudaErrorInvalidValue;
	if(vertices && v_capacity < (size_t) nv) return (int) cudaErrorInvalidValue;
	if(triangles && t_capacity < (size_t) nt) return (int) cudaErrorInvalidValue;
	hdr->nv = (int) nv;
	hdr->nt = (int) nt;
	for(int d = 0; d < 3; ++d) {
		hdr->min[d] = nv ? INFINITY : 0.f;
		hdr->max[d] = nv ? -INFINITY : 0.f;
	}
	for(long long i = 0; i < nv; ++i)
		for(int d = 0; d < 3; ++d) {
			hdr->min[d] = std::min(hdr->min[d], v[3 * i + d]);
			hdr->max[d] = std::max(hdr->max[d], v[3 * i + d]);
		}
	if(vertices) std::memcpy(vertices, v.data(), v.size() * sizeof(float));
	if(triangles)
		for(size_t i = 0; i < f.size(); ++i) triangles[i] = (int) f[i];
	return 0;
}

// ---- host: the lattice -----------------------------------------------------------------------------------------------------------
// SDFGen's main in float: min = box min - padding h, max = box max + padding h, n = (unsigned) ((max - min) / h), padding < 1 -> 1.
// cudaErrorInvalidValue for a bad h or band, no triangles, an index out of range, a non-finite vertex, n_d < 2 or ni nj nk >= 2^31.
inline int mesh_header(const float* x, int nv, const int* tri, int nt, const cb200_mesh_levelset_params& prm, cb200_sdf_header& out) {
	const float h = prm.h;
	if(!x || !tri || nv <= 0 || nt <= 0 || !std::isfinite(h) || !(h > 0.f) || prm.exact_band < 0 || prm.exact_band > 8) return (int) cudaErrorInvalidValue;
	for(long long i = 0; i < 3LL * nt; ++i)
		if(tri[i] < 0 || tri[i] >= nv) return (int) cudaErrorInvalidValue;
	float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
	for(long long i = 0; i < nv; ++i)
		for(int d = 0; d < 3; ++d) {
			const float v = x[3 * i + d];
			if(!std::isfinite(v)) return (int) cudaErrorInvalidValue;
			lo[d] = std::min(lo[d], v);
			hi[d] = std::max(hi[d], v);
		}
	const int padding = prm.padding < 1 ? 1 : prm.padding;
	volatile float pad = (float) padding * h;  // volatile: each step rounded to float, as SDFGen's Vec3f arithmetic
	long long total = 1;
	int n[3];
	for(int d = 0; d < 3; ++d) {
		volatile float mn = lo[d] - pad, mx = hi[d] + pad;
		volatile float span = mx - mn;
		volatile float q = span / h;
		if(!std::isfinite(mn) || !(q < 2147483648.f)) return (int) cudaErrorInvalidValue;
		n[d] = (int) (unsigned) q;
		if(n[d] < 2) return (int) cudaErrorInvalidValue;
		total *= n[d];
		out.min[d] = mn;
	}
	if(total >= (1LL << 31)) return (int) cudaErrorInvalidValue;
	out.ni = n[0];
	out.nj = n[1];
	out.nk = n[2];
	out.h = h;
	return 0;
}

// ---- device: SDFGen's geometry, explicitly rounded --------------------------------------------------------------------------------
constexpr int kMeshThreads = 256;

struct MV {
	float x, y, z;
};
__device__ __forceinline__ MV mv_sub(MV a, MV b) { return {__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y), __fsub_rn(a.z, b.z)}; }
__device__ __forceinline__ float mv_dot(MV a, MV b) { return __fadd_rn(__fadd_rn(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)), __fmul_rn(a.z, b.z)); }
__device__ __forceinline__ float mv_dist(MV a, MV b) {
	const MV d = mv_sub(a, b);
	return __fsqrt_rn(mv_dot(d, d));
}
__device__ __forceinline__ float sdf_min(float a, float b) { return b < a ? b : a; }  // std::min

// point_segment_distance (makelevelset3.cpp:4-17): m2 and the division in double
__device__ __forceinline__ float point_segment_distance(MV x0, MV x1, MV x2) {
	const MV dx = mv_sub(x2, x1);
	const double m2 = (double) mv_dot(dx, dx);
	float s12 = __double2float_rn(__ddiv_rn((double) mv_dot(mv_sub(x2, x0), dx), m2));
	if(s12 < 0.f) s12 = 0.f;
	else if(s12 > 1.f) s12 = 1.f;
	const float t = __fsub_rn(1.f, s12);
	const MV c = {__fadd_rn(__fmul_rn(s12, x1.x), __fmul_rn(t, x2.x)), __fadd_rn(__fmul_rn(s12, x1.y), __fmul_rn(t, x2.y)),
	              __fadd_rn(__fmul_rn(s12, x1.z), __fmul_rn(t, x2.z))};
	return mv_dist(x0, c);
}

// point_triangle_distance (makelevelset3.cpp:20-41)
__device__ __forceinline__ float point_triangle_distance(MV x0, MV x1, MV x2, MV x3) {
	const MV x13 = mv_sub(x1, x3), x23 = mv_sub(x2, x3), x03 = mv_sub(x0, x3);
	const float m13 = mv_dot(x13, x13), m23 = mv_dot(x23, x23), d = mv_dot(x13, x23);
	float det = __fsub_rn(__fmul_rn(m13, m23), __fmul_rn(d, d));
	if(det < 1e-30f) det = 1e-30f;  // std::max(det, 1e-30f)
	const float invdet = __fdiv_rn(1.f, det);
	const float a = mv_dot(x13, x03), b = mv_dot(x23, x03);
	const float w23 = __fmul_rn(invdet, __fsub_rn(__fmul_rn(m23, a), __fmul_rn(d, b)));
	const float w31 = __fmul_rn(invdet, __fsub_rn(__fmul_rn(m13, b), __fmul_rn(d, a)));
	const float w12 = __fsub_rn(__fsub_rn(1.f, w23), w31);
	if(w23 >= 0.f && w31 >= 0.f && w12 >= 0.f) {
		const MV c = {__fadd_rn(__fadd_rn(__fmul_rn(w23, x1.x), __fmul_rn(w31, x2.x)), __fmul_rn(w12, x3.x)),
		              __fadd_rn(__fadd_rn(__fmul_rn(w23, x1.y), __fmul_rn(w31, x2.y)), __fmul_rn(w12, x3.y)),
		              __fadd_rn(__fadd_rn(__fmul_rn(w23, x1.z), __fmul_rn(w31, x2.z)), __fmul_rn(w12, x3.z))};
		return mv_dist(x0, c);
	}
	if(w23 > 0.f) return sdf_min(point_segment_distance(x0, x1, x2), point_segment_distance(x0, x1, x3));
	if(w31 > 0.f) return sdf_min(point_segment_distance(x0, x1, x2), point_segment_distance(x0, x2, x3));
	return sdf_min(point_segment_distance(x0, x1, x3), point_segment_distance(x0, x2, x3));
}

// orientation (makelevelset3.cpp:84-94): twice the signed area, with SOS for exact zeros
__device__ __forceinline__ int sos_orientation(double x1, double y1, double x2, double y2, double& area) {
	area = __dsub_rn(__dmul_rn(y1, x2), __dmul_rn(x1, y2));
	if(area > 0.0) return 1;
	if(area < 0.0) return -1;
	if(y2 > y1) return 1;
	if(y2 < y1) return -1;
	if(x1 > x2) return 1;
	if(x1 < x2) return -1;
	return 0;
}

// point_in_triangle_2d (makelevelset3.cpp:98-116)
__device__ __forceinline__ bool point_in_triangle_2d(double x0, double y0, double x1, double y1, double x2, double y2, double x3, double y3, double& a,
                                                     double& b, double& c) {
	x1 = __dsub_rn(x1, x0);
	x2 = __dsub_rn(x2, x0);
	x3 = __dsub_rn(x3, x0);
	y1 = __dsub_rn(y1, y0);
	y2 = __dsub_rn(y2, y0);
	y3 = __dsub_rn(y3, y0);
	const int sa = sos_orientation(x2, y2, x3, y3, a);
	if(sa == 0) return false;
	if(sos_orientation(x3, y3, x1, y1, b) != sa) return false;
	if(sos_orientation(x1, y1, x2, y2, c) != sa) return false;
	const double sum = __dadd_rn(__dadd_rn(a, b), c);
	a = __ddiv_rn(a, sum);
	b = __ddiv_rn(b, sum);
	c = __ddiv_rn(c, sum);
	return true;
}

struct MeshGeom {
	const float* x;    // [nv][3]
	const int* tri;    // [nt][3]
	int nt;
	float ox, oy, oz, h;
	int ni, nj, nk;
	__device__ __forceinline__ MV vtx(int v) const { return {__ldg(x + 3 * v), __ldg(x + 3 * v + 1), __ldg(x + 3 * v + 2)}; }
	// Vec3f gx(i*dx+origin[0], ...)
	__device__ __forceinline__ MV node(int i, int j, int k) const {
		return {__fadd_rn(__fmul_rn((float) i, h), ox), __fadd_rn(__fmul_rn((float) j, h), oy), __fadd_rn(__fmul_rn((float) k, h), oz)};
	}
	__device__ __forceinline__ float distance(MV g, int t) const {
		return point_triangle_distance(g, vtx(__ldg(tri + 3 * t)), vtx(__ldg(tri + 3 * t + 1)), vtx(__ldg(tri + 3 * t + 2)));
	}
	// ((double) x - origin) / dx of triangle t's three vertices, per axis: f[axis][vertex]
	__device__ __forceinline__ void grid_coords(int t, double f[3][3]) const {
		const double o[3] = {(double) ox, (double) oy, (double) oz};
		for(int c = 0; c < 3; ++c) {
			const int v = __ldg(tri + 3 * t + c);
			for(int d = 0; d < 3; ++d) f[d][c] = __ddiv_rn(__dsub_rn((double) __ldg(x + 3 * v + d), o[d]), (double) h);
		}
	}
	__device__ __forceinline__ size_t at(int i, int j, int k) const { return (size_t) i + (size_t) ni * ((size_t) j + (size_t) nj * k); }
};

// util.h's min(a1, a2, a3) = std::min(a1, std::min(a2, a3)), likewise max
__device__ __forceinline__ double min3(double a, double b, double c) {
	const double m = c < b ? c : b;
	return m < a ? m : a;
}
__device__ __forceinline__ double max3(double a, double b, double c) {
	const double m = b < c ? c : b;
	return a < m ? m : a;
}

// a triangle's two boxes: band [b0, b0 + be) (i fastest), crossing columns [c0, c0 + ce) in (j, k)
struct MeshTri {
	int b0[3], be[3];
	int c0[2], ce[2];
};

__device__ __forceinline__ int clampi(int a, int lo, int hi) { return a < lo ? lo : (a > hi ? hi : a); }

__global__ void __launch_bounds__(kMeshThreads) mesh_setup_kernel(const MeshGeom g, int exact_band, MeshTri* __restrict__ boxes, longlong2* __restrict__ counts) {
	const int t = blockIdx.x * blockDim.x + threadIdx.x;
	if(t >= g.nt) return;
	double f[3][3];
	g.grid_coords(t, f);
	const int n[3] = {g.ni, g.nj, g.nk};
	MeshTri m;
	long long band = 1;
	for(int d = 0; d < 3; ++d) {
		const int lo = clampi((int) min3(f[d][0], f[d][1], f[d][2]) - exact_band, 0, n[d] - 1);
		const int hi = clampi((int) max3(f[d][0], f[d][1], f[d][2]) + exact_band + 1, 0, n[d] - 1);
		m.b0[d] = lo;
		m.be[d] = hi - lo + 1;
		band *= m.be[d];
	}
	long long cols = 1;
	for(int d = 1; d < 3; ++d) {
		const int lo = clampi((int) ceil(min3(f[d][0], f[d][1], f[d][2])), 0, n[d] - 1);
		const int hi = clampi((int) floor(max3(f[d][0], f[d][1], f[d][2])), 0, n[d] - 1);
		m.c0[d - 1] = lo;
		m.ce[d - 1] = hi >= lo ? hi - lo + 1 : 0;
		cols *= m.ce[d - 1];
	}
	boxes[t] = m;
	counts[t] = make_longlong2(band, cols);
}

// exclusive scan of counts[0, n) into offs[0, n] (offs[n] = the totals): tiles of kMeshThreads * kMeshScanPer items
constexpr int kMeshScanPer = 8;
struct MeshScan {
	const longlong2* in;
	longlong2* offs;
	longlong2* tile;  // [tiles]: sums, then (last CTA) exclusive prefixes
	unsigned* done;
	int n;
};

__device__ __forceinline__ longlong2 ll2_add(longlong2 a, longlong2 b) { return make_longlong2(a.x + b.x, a.y + b.y); }

// the block's exclusive prefix of v (and the block total)
__device__ __forceinline__ longlong2 mesh_block_scan(longlong2 v, longlong2& total) {
	__shared__ longlong2 s_w[kMeshThreads / 32];
	const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
	longlong2 inc = v;
#pragma unroll
	for(int o = 1; o < 32; o <<= 1) {
		const long long ux = __shfl_up_sync(0xffffffffu, inc.x, o), uy = __shfl_up_sync(0xffffffffu, inc.y, o);
		if(lane >= o) inc = ll2_add(inc, make_longlong2(ux, uy));
	}
	if(lane == 31) s_w[warp] = inc;
	__syncthreads();
	longlong2 run = make_longlong2(inc.x - v.x, inc.y - v.y);
	total = make_longlong2(0, 0);
	for(int w = 0; w < kMeshThreads / 32; ++w) {
		if(w < warp) run = ll2_add(run, s_w[w]);
		total = ll2_add(total, s_w[w]);
	}
	__syncthreads();
	return run;
}

__global__ void __launch_bounds__(kMeshThreads) mesh_scan_tiles_kernel(const MeshScan a) {
	__shared__ bool s_last;
	const int base = blockIdx.x * kMeshThreads * kMeshScanPer + threadIdx.x * kMeshScanPer;
	longlong2 sum = make_longlong2(0, 0);
	for(int r = 0; r < kMeshScanPer; ++r)
		if(base + r < a.n) sum = ll2_add(sum, a.in[base + r]);
	longlong2 total;
	mesh_block_scan(sum, total);
	if(threadIdx.x == 0) {
		a.tile[blockIdx.x] = total;
		__threadfence();
		s_last = atomicAdd(a.done, 1u) == gridDim.x - 1;
	}
	__syncthreads();
	if(!s_last) return;
	__threadfence();
	// the last CTA: exclusive prefix of the tile sums, thread i owning tiles [i K, (i + 1) K)
	const int tiles = (int) gridDim.x, K = (tiles + kMeshThreads - 1) / kMeshThreads;
	volatile long long* col = reinterpret_cast<volatile long long*>(a.tile);
	longlong2 own = make_longlong2(0, 0);
	for(int k = 0; k < K; ++k) {
		const int t = threadIdx.x * K + k;
		if(t < tiles) own = ll2_add(own, make_longlong2(col[2 * t], col[2 * t + 1]));
	}
	longlong2 run = mesh_block_scan(own, total);
	for(int k = 0; k < K; ++k) {
		const int t = threadIdx.x * K + k;
		if(t < tiles) {
			const longlong2 v = make_longlong2(col[2 * t], col[2 * t + 1]);
			col[2 * t] = run.x;
			col[2 * t + 1] = run.y;
			run = ll2_add(run, v);
		}
	}
	if(threadIdx.x == 0) {
		a.offs[a.n] = total;
		*a.done = 0u;
	}
}

__global__ void __launch_bounds__(kMeshThreads) mesh_scan_write_kernel(const MeshScan a) {
	const int base = blockIdx.x * kMeshThreads * kMeshScanPer + threadIdx.x * kMeshScanPer;
	longlong2 sum = make_longlong2(0, 0);
	for(int r = 0; r < kMeshScanPer; ++r)
		if(base + r < a.n) sum = ll2_add(sum, a.in[base + r]);
	longlong2 total;
	longlong2 run = ll2_add(mesh_block_scan(sum, total), a.tile[blockIdx.x]);
	for(int r = 0; r < kMeshScanPer; ++r)
		if(base + r < a.n) {
			a.offs[base + r] = run;
			run = ll2_add(run, a.in[base + r]);
		}
}

// the triangle of item `it`: the last t with offs[t] <= it (component X: band, Y: crossings)
template<bool BAND>
__device__ __forceinline__ int mesh_item_owner(const longlong2* offs, int nt, long long it) {
	int lo = 0, hi = nt - 1;
	while(lo < hi) {
		const int mid = (lo + hi + 1) >> 1;
		const longlong2 o = __ldg(offs + mid);
		if((BAND ? o.x : o.y) <= it) lo = mid;
		else hi = mid - 1;
	}
	return lo;
}

// packed node: (float bits of phi) << 32 | closest triangle (0xffffffff: none)
__host__ __device__ __forceinline__ unsigned long long mesh_pack(float d, int t) {
#ifdef __CUDA_ARCH__
	const unsigned bits = __float_as_uint(d);
#else
	unsigned bits;
	std::memcpy(&bits, &d, sizeof(bits));
#endif
	return ((unsigned long long) bits << 32) | (unsigned) t;
}

__global__ void __launch_bounds__(kMeshThreads) mesh_init_kernel(long long n, unsigned long long init, unsigned long long* __restrict__ packed, int* __restrict__ counts) {
	for(long long i = blockIdx.x * (long long) blockDim.x + threadIdx.x; i < n; i += (long long) gridDim.x * blockDim.x) {
		packed[i] = init;
		counts[i] = 0;
	}
}

__global__ void __launch_bounds__(kMeshThreads) mesh_band_kernel(const MeshGeom g, const MeshTri* __restrict__ boxes, const longlong2* __restrict__ offs, float init,
                                                                 unsigned long long* __restrict__ packed) {
	const long long total = __ldg(offs + g.nt).x;
	for(long long it = blockIdx.x * (long long) blockDim.x + threadIdx.x; it < total; it += (long long) gridDim.x * blockDim.x) {
		const int t = mesh_item_owner<true>(offs, g.nt, it);
		const MeshTri m = boxes[t];
		const long long l = it - __ldg(offs + t).x;
		const int i = m.b0[0] + (int) (l % m.be[0]);
		const long long r = l / m.be[0];
		const int j = m.b0[1] + (int) (r % m.be[1]), k = m.b0[2] + (int) (r / m.be[1]);
		const float d = g.distance(g.node(i, j, k), t);
		if(d < init) atomicMin(packed + g.at(i, j, k), mesh_pack(d, t));
	}
}

__global__ void __launch_bounds__(kMeshThreads) mesh_cross_kernel(const MeshGeom g, const MeshTri* __restrict__ boxes, const longlong2* __restrict__ offs, int* __restrict__ counts) {
	const long long total = __ldg(offs + g.nt).y;
	for(long long it = blockIdx.x * (long long) blockDim.x + threadIdx.x; it < total; it += (long long) gridDim.x * blockDim.x) {
		const int t = mesh_item_owner<false>(offs, g.nt, it);
		const MeshTri m = boxes[t];
		const long long l = it - __ldg(offs + t).y;
		const int j = m.c0[0] + (int) (l % m.ce[0]), k = m.c0[1] + (int) (l / m.ce[0]);
		double f[3][3], a, b, c;
		g.grid_coords(t, f);
		if(point_in_triangle_2d((double) j, (double) k, f[1][0], f[2][0], f[1][1], f[2][1], f[1][2], f[2][2], a, b, c)) {
			const double fi = __dadd_rn(__dadd_rn(__dmul_rn(a, f[0][0]), __dmul_rn(b, f[0][1])), __dmul_rn(c, f[0][2]));
			const int ii = (int) ceil(fi);  // the crossing lies in (ii - 1, ii]
			if(ii < 0) atomicAdd(counts + g.at(0, j, k), 1);  // the first interval takes everything on its -i side
			else if(ii < g.ni) atomicAdd(counts + g.at(ii, j, k), 1);
		}
	}
}

// the sweep directions of makelevelset3.cpp:163-172, in order
__constant__ signed char kMeshSweepDir[8][3] = {{1, 1, 1}, {-1, -1, -1}, {1, 1, -1}, {-1, -1, 1}, {1, -1, 1}, {-1, 1, -1}, {1, -1, -1}, {-1, 1, 1}};

// node (i, j, k) of one sweep direction: check_neighbour (makelevelset3.cpp:43-55) for its 7 upstream neighbours in SDFGen's order.
// The packed values are read with __ldcg: other CTAs wrote them in earlier planes of this launch.
__device__ __forceinline__ void mesh_sweep_node(const MeshGeom& g, unsigned long long* packed, int i, int j, int k, int di, int dj, int dk) {
	const size_t self = g.at(i, j, k);
	const unsigned long long own = __ldcg(packed + self);
	float phi = __uint_as_float((unsigned) (own >> 32));
	int best = (int) (unsigned) own;
	const MV gx = g.node(i, j, k);
	const int nb[7][3] = {{i - di, j, k}, {i, j - dj, k}, {i - di, j - dj, k}, {i, j, k - dk}, {i - di, j, k - dk}, {i, j - dj, k - dk}, {i - di, j - dj, k - dk}};
#pragma unroll
	for(int c = 0; c < 7; ++c) {
		const int t = (int) (unsigned) __ldcg(packed + g.at(nb[c][0], nb[c][1], nb[c][2]));
		if(t >= 0) {
			const float d = g.distance(gx, t);
			if(d < phi) {
				phi = d;
				best = t;
			}
		}
	}
	if(best != (int) (unsigned) own || __float_as_uint(phi) != (unsigned) (own >> 32)) packed[self] = mesh_pack(phi, best);
}

// All 16 sweeps in one cooperative launch.  Direction-adjusted indices a = i or ni - 1 - i (likewise b, c) run over [1, n - 1], as
// sweep()'s loop bounds do; plane s holds a + b + c = s, s = 3 .. (ni - 1) + (nj - 1) + (nk - 1).  Each CTA strides over the (b, c)
// rectangle of the plane and skips the a outside [1, ni - 1].
__global__ void __launch_bounds__(kMeshThreads) mesh_sweep_kernel(const MeshGeom g, unsigned long long* packed) {
	namespace cg = cooperative_groups;
	cg::grid_group grid = cg::this_grid();
	const int A = g.ni - 1, B = g.nj - 1, Cn = g.nk - 1;
	const long long stride = (long long) gridDim.x * blockDim.x, tid = blockIdx.x * (long long) blockDim.x + threadIdx.x;
	for(int pass = 0; pass < 2; ++pass)
		for(int dir = 0; dir < 8; ++dir) {
			const int di = kMeshSweepDir[dir][0], dj = kMeshSweepDir[dir][1], dk = kMeshSweepDir[dir][2];
			for(int s = 3; s <= A + B + Cn; ++s) {
				const int c_lo = max(1, s - A - B), c_hi = min(Cn, s - 2);
				const int b_lo = max(1, s - A - c_hi), b_hi = min(B, s - 1 - c_lo);
				const int bw = b_hi - b_lo + 1;
				const long long rect = (long long) bw * (c_hi - c_lo + 1);
				for(long long q = tid; q < rect; q += stride) {
					const int b = b_lo + (int) (q % bw), c = c_lo + (int) (q / bw), a = s - b - c;
					if(a < 1 || a > A) continue;
					mesh_sweep_node(g, packed, di > 0 ? a : A - a, dj > 0 ? b : B - b, dk > 0 ? c : Cn - c, di, dj, dk);
				}
				grid.sync();
			}
		}
}

// sign (makelevelset3.cpp:174-182): one warp per (j, k) row; phi (negated where the prefix parity is odd) replaces the counts
__global__ void __launch_bounds__(kMeshThreads) mesh_sign_kernel(const MeshGeom g, const unsigned long long* __restrict__ packed, int* counts) {
	const long long rows = (long long) g.nj * g.nk, warps = (long long) gridDim.x * (blockDim.x / 32);
	const int lane = threadIdx.x & 31;
	for(long long r = (blockIdx.x * (long long) blockDim.x + threadIdx.x) / 32; r < rows; r += warps) {
		const size_t base = (size_t) r * g.ni;
		unsigned parity = 0;
		for(int i0 = 0; i0 < g.ni; i0 += 32) {
			const int i = i0 + lane;
			const bool odd = i < g.ni && (counts[base + i] & 1);
			const unsigned bal = __ballot_sync(0xffffffffu, odd);
			const unsigned mine = parity ^ (__popc(bal & (0xffffffffu >> (31 - lane))) & 1);
			if(i < g.ni) {
				const unsigned bits = (unsigned) (__ldg(packed + base + i) >> 32);
				counts[base + i] = (int) (mine ? bits ^ 0x80000000u : bits);
			}
			parity ^= __popc(bal) & 1;
		}
	}
}

}  // namespace cb200
