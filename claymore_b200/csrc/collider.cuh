// collider.cuh -- signed-distance collision object applied to grid nodes (SignedDistanceGrid, Projects/MGSP/boundary_condition.cuh:25-250).
//
// The level set is dense over the whole domain in the reference's layout (signed_distance_field_, boundary_condition.cuh:15-16):
// one 1 KiB block per grid block, blocks row-major (x*G*G + y*G + z), inside a block 4 channels SoA (distance, gradient x, y, z)
// of 64 cells (cell = x*16 + y*4 + z).  Every caller (the grid update and the two next-max predictors of grid.cuh) applies the
// same boundary chain (boundaries_resolve), so the max the MGSP ranks agree on is the max the next grid update finds.
#pragma once
#include "common.cuh"

namespace cb200 {

using ColliderView = cb200_collider;  // POD: device field pointer + the SignedDistanceGrid members (boundary_condition.cuh:28-35)

// parameters the resolve can work with: a BoundaryT value and a scale it may divide by
inline bool collider_valid(const cb200_collider* c) { return c && c->type >= CB200_STICKY && c->type <= CB200_SEPARATE && c->scale != 0.f; }

// the time-dependent part of detect_and_resolve_collision (:160-179), evaluated once per CTA
struct ColliderFrame {
	float rot[9];   // current_rot_mat = rot_mat * Rx(omega_x t) * Ry(omega_y t) * Rz(omega_z t), vec3x3 storage
	float b[3];     // trans + trans_vel * t
	float s_inv;    // 1 / (1 + dsdt * t)
};

// rot_angle_to_matrix (:67-90) in vec3x3 storage (element (i, j) at 3 * i + j)
__device__ __forceinline__ void collider_axis_rot(float a, int dim, float* r) {
	const float c = cosf(a), s = sinf(a);
#pragma unroll
	for(int i = 0; i < 9; ++i) r[i] = 0.f;
	if(dim == 0) {
		r[0] = 1.f;
		r[4] = r[8] = c;
		r[7] = s;
		r[5] = -s;
	} else if(dim == 1) {
		r[4] = 1.f;
		r[0] = r[8] = c;
		r[2] = s;
		r[6] = -s;
	} else {
		r[8] = 1.f;
		r[0] = r[4] = c;
		r[3] = s;
		r[1] = -s;
	}
}
// matrix_matrix_multiplication_3d (Library/MnBase/Math/Matrix/MatrixUtils.h:147-157)
__device__ __forceinline__ void collider_mat_mul(const float* a, const float* b, float* c) {
#pragma unroll
	for(int j = 0; j < 3; ++j)
#pragma unroll
		for(int i = 0; i < 3; ++i) c[3 * j + i] = a[i] * b[3 * j] + a[3 + i] * b[3 * j + 1] + a[6 + i] * b[3 * j + 2];
}

// P: any struct with the cb200_collider motion fields (cb200_collider, cb200_collision_object)
template<class P>
__device__ __forceinline__ void collider_make_frame(const P& c, float t, ColliderFrame& f) {
	float cur[9], r[9], prev[9];
#pragma unroll
	for(int i = 0; i < 9; ++i) cur[i] = c.rot_mat[i];
#pragma unroll
	for(int d = 0; d < 3; ++d) {
		collider_axis_rot(c.omega[d] * t, d, r);
#pragma unroll
		for(int i = 0; i < 9; ++i) prev[i] = cur[i];
		collider_mat_mul(prev, r, cur);
	}
#pragma unroll
	for(int i = 0; i < 9; ++i) f.rot[i] = cur[i];
#pragma unroll
	for(int d = 0; d < 3; ++d) f.b[d] = c.trans[d] + c.trans_vel[d] * t;
	f.s_inv = 1.f / (1.f + c.dsdt * t);
}

// get_signed_distance_and_normal + query_sdf (:98-143) at the material-space point x.  The wall band reports no hit (kept); the
// normal is normalised only when it is non-zero (the reference divides 0 by 0); the +1 node must lie in the domain (the reference
// always has a wall band there).  Reads go through the read-only path at addresses computed from the node's block key.
__device__ __forceinline__ bool collider_query(const ColliderView& c, const Cfg& cfg, const float* x, float* n) {
	const float lo = (float) cfg.boundary * cfg.dx * 4.f, hi = (float) (cfg.gsize - cfg.boundary) * 4.f * cfg.dx;
	if(x[0] < lo || x[0] >= hi || x[1] < lo || x[1] >= hi || x[2] < lo || x[2] >= hi) return false;
	int gc[3];
	float w1[3][2];
	const int top = cfg.gsize * 4;
#pragma unroll
	for(int d = 0; d < 3; ++d) {
		gc[d] = (int) (x[d] / cfg.dx);  // a true division, as the reference
		if(gc[d] + 1 >= top) return false;
		const float dl = x[d] - (float) gc[d] * cfg.dx;
		w1[d][0] = 1.f - dl / cfg.dx;
		w1[d][1] = dl / cfg.dx;
	}
	float sd = 0.f;
	n[0] = n[1] = n[2] = 0.f;
#pragma unroll
	for(int i = 0; i < 2; ++i)
#pragma unroll
		for(int j = 0; j < 2; ++j)
#pragma unroll
			for(int k = 0; k < 2; ++k) {
				const int px = gc[0] + i, py = gc[1] + j, pz = gc[2] + k;
				const float w = w1[0][i] * w1[1][j] * w1[2][k];
				const float* blk = c.sdf + (size_t) table_offset(cfg, px >> 2, py >> 2, pz >> 2) * kGridBlockFloats + ((px & 3) * 16 + (py & 3) * 4 + (pz & 3));
				sd += w * __ldg(blk);
				n[0] += w * __ldg(blk + 64);
				n[1] += w * __ldg(blk + 128);
				n[2] += w * __ldg(blk + 192);
			}
	const float nn = n[0] * n[0] + n[1] * n[1] + n[2] * n[2];
	if(nn > 0.f) {
		const float len = sqrtf(nn);
		n[0] /= len;
		n[1] /= len;
		n[2] /= len;
	}
	return sd <= 0.f;
}

// the point p's image in the material space of an object placed by f (P: its parameters): x = R^T ((p - b) s_inv) scale + trans;
// xm = p - b, the offset the object velocity is taken at
template<class P>
__device__ __forceinline__ void collider_material_point(const P& c, const ColliderFrame& f, const float* p, float* xm, float* x) {
#pragma unroll
	for(int d = 0; d < 3; ++d) xm[d] = p[d] - f.b[d];
	const float x0[3] = {xm[0] * f.s_inv, xm[1] * f.s_inv, xm[2] * f.s_inv};
	const float* R = f.rot;
#pragma unroll
	for(int d = 0; d < 3; ++d) x[d] = (R[3 * d] * x0[0] + R[3 * d + 1] * x0[1] + R[3 * d + 2] * x0[2]) * c.scale + c.trans[d];  // mat_t_mul_vec_3d
}

// detect_and_resolve_collision (:159-249) of the velocity v at grid node (nx, ny, nz) against the object with parameters c (P: a
// struct with the collider's motion, type and friction fields) placed by f.  query(x, n) tests the material-space point x and
// writes the material-space normal n (0 where it has none): collider_query for the level set, object_query for an analytic shape.
// The object velocity takes a true omega x r where the reference's vec3_cross_vec3 (:92-95) adds all products;
// get_material_velocity keeps MnBase's vec_cross_mul_vec_3d as it is (MatrixUtils.h:54-58).
template<class P, class Q>
__device__ __forceinline__ void collider_resolve(const P& c, const ColliderFrame& f, float dx, int nx, int ny, int nz, float& vx, float& vy, float& vz, Q&& query) {
	const float p[3] = {(float) nx * dx, (float) ny * dx, (float) nz * dx};
	float xm[3], x[3];
	collider_material_point(c, f, p, xm, x);
	const float* R = f.rot;
	float on[3];
	if(!query(x, on)) return;
	const float* w = c.omega;
	float vo[3] = {w[1] * xm[2] - w[2] * xm[1], w[2] * xm[0] - w[0] * xm[2], w[0] * xm[1] - w[1] * xm[0]};
	const float ds = c.dsdt / c.scale;
#pragma unroll
	for(int d = 0; d < 3; ++d) vo[d] += xm[d] * ds;
	{
		const float r[3] = {x[0] - c.trans[0], x[1] - c.trans[1], x[2] - c.trans[2]};
		const float mv[3] = {w[1] * r[2] + w[2] * r[1] + c.trans_vel[0], w[2] * r[0] + w[0] * r[2] + c.trans_vel[1], w[0] * r[1] + w[1] * r[0] + c.trans_vel[2]};
#pragma unroll
		for(int d = 0; d < 3; ++d) vo[d] += (R[d] * mv[0] + R[3 + d] * mv[1] + R[6 + d] * mv[2]) * c.scale + c.trans_vel[d];  // matrix_vector_multiplication_3d
	}
	float v[3] = {vx - vo[0], vy - vo[1], vz - vo[2]};
	if(c.type == CB200_STICKY) {
		v[0] = v[1] = v[2] = 0.f;
	} else {
		if(c.type == CB200_SEPARATE && on[0] == 0.f && on[1] == 0.f && on[2] == 0.f) {
			vx = vy = vz = 0.f;  // :222-225 returns before the object velocity is added back
			return;
		}
		float n[3];
#pragma unroll
		for(int d = 0; d < 3; ++d) n[d] = R[d] * on[0] + R[3 + d] * on[1] + R[6 + d] * on[2];
		const float vn = n[0] * v[0] + n[1] * v[1] + n[2] * v[2];
		const bool slip = c.type == CB200_SLIP;
		if(slip || vn < 0.f) {
#pragma unroll
			for(int d = 0; d < 3; ++d) v[d] -= n[d] * vn;
			if((slip ? c.friction > 0.f : c.friction != 0.f) && vn < 0.f) {
				const float len = sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
				if(-vn * c.friction < len) {
					const float fr = vn * c.friction;
#pragma unroll
					for(int d = 0; d < 3; ++d) v[d] += v[d] / len * fr;
				} else {
					v[0] = v[1] = v[2] = 0.f;
				}
			}
		}
	}
	vx = v[0] + vo[0];
	vy = v[1] + vo[1];
	vz = v[2] + vo[2];
}

// ---- analytic collision objects (DESIGN.md section 2.9) ----------------------------------------------------------------------
struct ObjectList {
	int n;
	cb200_collision_object o[CB200_MAX_COLLISION_OBJECTS];
};

inline bool finite_all(const float* v, int n) {
	for(int i = 0; i < n; ++i)
		if(!std::isfinite(v[i])) return false;
	return true;
}
// checks every entry of objs[0, n) and copies them into out, the plane normals made unit length in double; false (out
// unchanged) on an unknown shape or type, scale 0, a non-finite value, a zero plane normal, lo > hi, a radius or half height
// <= 0, or n outside [0, CB200_MAX_COLLISION_OBJECTS].  CB200_SHAPE_LEVELSET is known only with levelsets > 0 registered lattices:
// its spacing b[0] must be > 0 and its index b[1] an exact integer in [0, levelsets)
inline bool objects_prepare(const cb200_collision_object* objs, int n, ObjectList& out, int levelsets = 0) {
	if(n < 0 || n > CB200_MAX_COLLISION_OBJECTS || (n > 0 && !objs)) return false;
	ObjectList l {};
	l.n = n;
	const int last_shape = levelsets > 0 ? (int) CB200_SHAPE_LEVELSET : (int) CB200_SHAPE_CYLINDER;
	for(int i = 0; i < n; ++i) {
		cb200_collision_object o = objs[i];
		if(o.shape < CB200_SHAPE_PLANE || o.shape > last_shape || o.type < CB200_STICKY || o.type > CB200_SEPARATE || o.scale == 0.f) return false;
		if(!finite_all(&o.friction, 1) || !finite_all(o.a, 3) || !finite_all(o.b, 3) || !finite_all(o.rot_mat, 9) || !finite_all(o.trans, 3) ||
		   !finite_all(o.trans_vel, 3) || !finite_all(o.omega, 3) || !finite_all(&o.dsdt, 1) || !finite_all(&o.scale, 1))
			return false;
		if(o.shape == CB200_SHAPE_PLANE) {
			const double len = std::sqrt((double) o.b[0] * o.b[0] + (double) o.b[1] * o.b[1] + (double) o.b[2] * o.b[2]);
			if(!(len > 0.0)) return false;
			for(int d = 0; d < 3; ++d) o.b[d] = (float) (o.b[d] / len);
		} else if(o.shape == CB200_SHAPE_BOX) {
			if(o.a[0] > o.b[0] || o.a[1] > o.b[1] || o.a[2] > o.b[2]) return false;
		} else if(o.shape == CB200_SHAPE_LEVELSET) {
			if(!(o.b[0] > 0.f) || !(o.b[1] >= 0.f) || o.b[1] >= (float) levelsets || o.b[1] != std::floor(o.b[1])) return false;
		} else if(!(o.b[0] > 0.f) || (o.shape == CB200_SHAPE_CYLINDER && !(o.b[1] > 0.f))) {
			return false;
		}
		l.o[i] = o;
	}
	out = l;
	return true;
}

// hit test (phi <= 0) and material-space normal of one shape at the material-space point x; the distance is not needed
__device__ __forceinline__ bool object_query(const cb200_collision_object& o, const float* x, float* n) {
	const float *a = o.a, *b = o.b;
	n[0] = n[1] = n[2] = 0.f;
	if(o.shape == CB200_SHAPE_PLANE) {  // a: point, b: unit normal
		if((x[0] - a[0]) * b[0] + (x[1] - a[1]) * b[1] + (x[2] - a[2]) * b[2] > 0.f) return false;
		n[0] = b[0];
		n[1] = b[1];
		n[2] = b[2];
		return true;
	}
	if(o.shape == CB200_SHAPE_BOX) {  // a: lo, b: hi
		if(!(a[0] <= x[0] && x[0] <= b[0] && a[1] <= x[1] && x[1] <= b[1] && a[2] <= x[2] && x[2] <= b[2])) return false;
		int axis = 0;
		float best = -INFINITY, sgn = 1.f;
#pragma unroll
		for(int d = 0; d < 3; ++d) {
			const float ql = a[d] - x[d], qh = x[d] - b[d];
			const float q = fmaxf(ql, qh);
			if(q > best) {  // the lowest axis wins a tie
				best = q;
				axis = d;
				sgn = ql > qh ? -1.f : 1.f;  // the low face when strictly nearer: +1 at the exact centre
			}
		}
		n[0] = axis == 0 ? sgn : 0.f;  // no dynamic index: n stays in registers
		n[1] = axis == 1 ? sgn : 0.f;
		n[2] = axis == 2 ? sgn : 0.f;
		return true;
	}
	const float d0 = x[0] - a[0], d1 = x[1] - a[1], d2 = x[2] - a[2];
	const float r = b[0];
	if(o.shape == CB200_SHAPE_SPHERE) {  // a: centre, b[0]: radius
		const float dd = d0 * d0 + d1 * d1 + d2 * d2;
		if(dd > r * r) return false;
		if(dd > 0.f) {
			const float len = sqrtf(dd);
			n[0] = d0 / len;
			n[1] = d1 / len;
			n[2] = d2 / len;
		}
		return true;
	}
	// CYLINDER: a: centre, b[0]: radius, b[1]: half height, axis along material-space y, capped
	const float rho2 = d0 * d0 + d2 * d2, h = b[1];
	if(rho2 > r * r || fabsf(d1) > h) return false;
	const float rho = sqrtf(rho2);
	if(h - fabsf(d1) < r - rho) {
		n[1] = d1 < 0.f ? -1.f : 1.f;
	} else if(rho > 0.f) {
		n[0] = d0 / rho;
		n[2] = d2 / rho;
	}
	return true;
}

// ---- level-set collision objects (DESIGN.md section 2.11) ---------------------------------------------------------------------
using LevelSetView = cb200_levelset;  // POD: device lattice (float4 per node: phi, g_i, g_j, g_k; i fastest) + its node counts
// The registered lattices a kernel may query: a kernel parameter of its own beside Boundaries, so that Boundaries and every instance
// without level sets keep their parameter block.
struct LevelSets {
	int count;
	LevelSetView v[CB200_MAX_COLLISION_LEVELSETS];
};
// the CTA's copy of the views, indexed by an object's b[1]
__device__ __forceinline__ LevelSetView* levelset_views() {
	__shared__ LevelSetView s[CB200_MAX_COLLISION_LEVELSETS];
	return s;
}
// thread k copies view k (static indices: the views may sit in a by-value kernel parameter); the caller's next barrier publishes them
__device__ __forceinline__ void levelset_views_cta(const LevelSets& ls) {
#pragma unroll
	for(int k = 0; k < CB200_MAX_COLLISION_LEVELSETS; ++k)
		if((int) threadIdx.x == k && k < ls.count) levelset_views()[k] = ls.v[k];
}

// hit test (phi <= 0) and material-space normal of the level-set object o (a: node 0, b[0]: spacing c) on its lattice l at the
// material-space point x: trilinear in the corner order of collider_query, no hit outside the node box
__device__ __forceinline__ bool levelset_query(const LevelSetView& l, const cb200_collision_object& o, const float* x, float* n) {
	const int dims[3] = {l.ni, l.nj, l.nk};
	int i0[3];
	float w1[3][2];
	n[0] = n[1] = n[2] = 0.f;
#pragma unroll
	for(int d = 0; d < 3; ++d) {
		const float q = (x[d] - o.a[d]) / o.b[0];  // a true division, as collider_query divides by dx
		if(!(q >= 0.f && q <= (float) (dims[d] - 1))) return false;
		i0[d] = min((int) floorf(q), dims[d] - 2);
		const float t = q - (float) i0[d];
		w1[d][0] = 1.f - t;
		w1[d][1] = t;
	}
	const float4* node = reinterpret_cast<const float4*>(l.lattice) + ((size_t) i0[2] * l.nj + i0[1]) * l.ni + i0[0];
	const size_t sj = (size_t) l.ni, sk = (size_t) l.ni * l.nj;
	float sd = 0.f;
#pragma unroll
	for(int i = 0; i < 2; ++i)
#pragma unroll
		for(int j = 0; j < 2; ++j)
#pragma unroll
			for(int k = 0; k < 2; ++k) {
				const float w = w1[0][i] * w1[1][j] * w1[2][k];
				const float4 p = __ldg(node + i + j * sj + k * sk);
				sd += w * p.x;
				n[0] += w * p.y;
				n[1] += w * p.z;
				n[2] += w * p.w;
			}
	const float nn = n[0] * n[0] + n[1] * n[1] + n[2] * n[2];
	if(nn > 0.f) {
		const float len = sqrtf(nn);
		n[0] /= len;
		n[1] /= len;
		n[2] /= len;
	}
	return sd <= 0.f;
}
// object_query with CB200_SHAPE_LEVELSET answered by the lattice levelset_views_cta copied for index b[1]
__device__ __forceinline__ bool object_query_levelsets(const cb200_collision_object& o, const float* x, float* n) {
	if(o.shape == CB200_SHAPE_LEVELSET) return levelset_query(levelset_views()[(int) o.b[1]], o, x, n);
	return object_query(o, x, n);
}

// ---- the boundary chain -------------------------------------------------------------------------------------------------------
// The solid boundaries of a simulator, applied in this order: the level-set collider (has_collider), then the analytic objects in
// list order, each resolving the velocity the previous one left.  Passed by value as a kernel parameter of its own beside the argument
// struct, so the plain kernels keep their parameter block; which of the two parts a kernel compiles in is its COLLIDE / OBJECTS flags.
struct Boundaries {
	bool has_collider;
	ColliderView col;
	ObjectList objects;  // n = 0: none
};

// the per-CTA state of the chain: the level-set collider's frame (COLLIDE), and each object's parameters and frame (OBJECTS)
struct BoundaryFrames {
	ColliderFrame col;
	ColliderFrame f[CB200_MAX_COLLISION_OBJECTS];
	cb200_collision_object o[CB200_MAX_COLLISION_OBJECTS];
};
__device__ __forceinline__ BoundaryFrames& boundary_frames() {
	__shared__ BoundaryFrames s;
	return s;
}
// thread 0 builds the collider's frame at time t and thread i object i's, from thread 32 on with the collider (another warp, so that
// the two run side by side); one barrier
template<bool COLLIDE, bool OBJECTS>
__device__ __forceinline__ const BoundaryFrames& boundary_frames_cta(const Boundaries& b, float t) {
	BoundaryFrames& s = boundary_frames();
	if constexpr(COLLIDE) {
		if(threadIdx.x == 0) collider_make_frame(b.col, t, s.col);
	}
	if constexpr(OBJECTS) {
		const int i = (int) threadIdx.x - (COLLIDE ? 32 : 0);
		if(i >= 0 && i < b.objects.n) {
			s.o[i] = b.objects.o[i];
			collider_make_frame(s.o[i], t, s.f[i]);
		}
	}
	__syncthreads();
	return s;
}
// the chain at grid node (nx, ny, nz), its frames s built by boundary_frames_cta; LEVELSETS (implies OBJECTS): level-set objects are
// answered from the views levelset_views_cta copied
template<bool COLLIDE, bool OBJECTS, bool LEVELSETS = false>
__device__ __forceinline__ void boundaries_resolve(const Boundaries& b, const BoundaryFrames& s, const Cfg& cfg, int nx, int ny, int nz, float& vx, float& vy, float& vz) {
	static_assert(OBJECTS || !LEVELSETS, "level-set objects are objects");
	if constexpr(COLLIDE) collider_resolve(b.col, s.col, cfg.dx, nx, ny, nz, vx, vy, vz, [&](const float* x, float* n) { return collider_query(b.col, cfg, x, n); });
	if constexpr(OBJECTS) {
		for(int i = 0; i < b.objects.n; ++i) {
			const cb200_collision_object& o = s.o[i];
			collider_resolve(o, s.f[i], cfg.dx, nx, ny, nz, vx, vy, vz, [&](const float* x, float* n) {
				if constexpr(LEVELSETS) return object_query_levelsets(o, x, n);
				else return object_query(o, x, n);
			});
		}
	}
}

// The chain over the two cells a lane holds, (nx, ny, nz) and (nx, ny, nz + 1) (hx / hy: which have mass), one body at a time: each
// body resolves both cells through the same collider_resolve as boundaries_resolve, then stage(k, f, in0, in1, in2) sees body k
// (0: the level-set collider, 1 + i: object i), its frame f and the velocities it received (channels 0-2, .x / .y the two cells);
// v0-v2 hold the velocities it left.  Each cell goes through the same calls in the same order as with boundaries_resolve.
template<bool COLLIDE, bool OBJECTS, bool LEVELSETS, class Stage>
__device__ __forceinline__ void boundaries_resolve_pair(const Boundaries& b, const BoundaryFrames& s, const Cfg& cfg, int nx, int ny, int nz, bool hx, bool hy, float2& v0, float2& v1,
                                                        float2& v2, Stage&& stage) {
	static_assert(OBJECTS || !LEVELSETS, "level-set objects are objects");
	if constexpr(COLLIDE) {
		const float2 i0 = v0, i1 = v1, i2 = v2;
		auto q = [&](const float* x, float* n) { return collider_query(b.col, cfg, x, n); };
		if(hx) collider_resolve(b.col, s.col, cfg.dx, nx, ny, nz, v0.x, v1.x, v2.x, q);
		if(hy) collider_resolve(b.col, s.col, cfg.dx, nx, ny, nz + 1, v0.y, v1.y, v2.y, q);
		stage(0, s.col, i0, i1, i2);
	}
	if constexpr(OBJECTS) {
		for(int i = 0; i < b.objects.n; ++i) {
			const cb200_collision_object& o = s.o[i];
			const float2 i0 = v0, i1 = v1, i2 = v2;
			auto q = [&](const float* x, float* n) {
				if constexpr(LEVELSETS) return object_query_levelsets(o, x, n);
				else return object_query(o, x, n);
			};
			if(hx) collider_resolve(o, s.f[i], cfg.dx, nx, ny, nz, v0.x, v1.x, v2.x, q);
			if(hy) collider_resolve(o, s.f[i], cfg.dx, nx, ny, nz + 1, v0.y, v1.y, v2.y, q);
			stage(1 + i, s.f[i], i0, i1, i2);
		}
	}
}

// grid-update velocity of one cell (wall mask, gravity on y, the chain) and its |v|^2, NaN -> +inf; no mass -> 0
template<bool COLLIDE, bool OBJECTS, bool LEVELSETS = false>
__device__ __forceinline__ float cell_vel_sq_boundaries(float m, float p0, float p1, float p2, bool wx, bool wy, bool wz, float gdt, const Boundaries& bd, const BoundaryFrames& s, const Cfg& cfg, int nx, int ny, int nz) {
	if(!node_has_mass(m)) return 0.f;
	const float mi = 1.f / m;
	float a = wx ? 0.f : p0 * mi, b = (wy ? 0.f : p1 * mi) + gdt, d = wz ? 0.f : p2 * mi;
	boundaries_resolve<COLLIDE, OBJECTS, LEVELSETS>(bd, s, cfg, nx, ny, nz, a, b, d);
	const float sq = a * a + b * b + d * d;
	return isnan(sq) ? INFINITY : sq;
}
// cell_pair_vel_sq (common.cuh) with the chain: the two cells lane holds of block (kx, ky, kz), whose grid block is s2 (float2 view)
template<bool COLLIDE, bool OBJECTS, bool LEVELSETS = false>
__device__ __forceinline__ float cell_pair_vel_sq_boundaries(const Cfg& cfg, const Boundaries& bd, const BoundaryFrames& s, const float2* s2, int lane, int kx, int ky, int kz, bool wx, bool wy, bool wz, float gdt) {
	const float2 m = s2[lane], p0 = s2[32 + lane], p1 = s2[64 + lane], p2 = s2[96 + lane];
	const int nx = 4 * kx + (lane >> 3), ny = 4 * ky + ((lane >> 1) & 3), nz = 4 * kz + 2 * (lane & 1);
	return fmaxf(cell_vel_sq_boundaries<COLLIDE, OBJECTS, LEVELSETS>(m.x, p0.x, p1.x, p2.x, wx, wy, wz, gdt, bd, s, cfg, nx, ny, nz),
	             cell_vel_sq_boundaries<COLLIDE, OBJECTS, LEVELSETS>(m.y, p0.y, p1.y, p2.y, wx, wy, wz, gdt, bd, s, cfg, nx, ny, nz + 1));
}

}  // namespace cb200
