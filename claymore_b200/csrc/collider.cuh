// collider.cuh -- signed-distance collision object applied to grid nodes (SignedDistanceGrid, Projects/MGSP/boundary_condition.cuh:25-250).
//
// The level set is dense over the whole domain in the reference's layout (signed_distance_field_, boundary_condition.cuh:15-16):
// one 1 KiB block per grid block, blocks row-major (x*G*G + y*G + z), inside a block 4 channels SoA (distance, gradient x, y, z)
// of 64 cells (cell = x*16 + y*4 + z).  Every caller (the grid update and the two next-max predictors of grid.cuh) applies the
// same boundary chain (boundaries_resolve), so the max the MGSP ranks agree on is the max the next grid update finds.
#pragma once
#include <algorithm>
#include <cmath>
#include <vector>

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

// ---- motion tracks (DESIGN.md section 2.14) -----------------------------------------------------------------------------------
// The tracks of a kernel's objects: a kernel parameter of its own, so that every instance without tracks keeps its parameter block.
// Object i moves on rec[off[i], off[i] + n[i]) (cb200_track_record, four float4 each) when n[i] > 0.
struct Tracks {
	const float4* rec;
	int off[CB200_MAX_COLLISION_OBJECTS];
	int n[CB200_MAX_COLLISION_OBJECTS];
	int flags[CB200_MAX_COLLISION_OBJECTS];
};
inline bool tracks_any(const Tracks* t) {
	if(!t) return false;
	for(int i = 0; i < CB200_MAX_COLLISION_OBJECTS; ++i)
		if(t->n[i] > 0) return true;
	return false;
}
// a tracked object's kinematic velocity at the frame's time: the pivot's c'(t) and the world angular velocity omega(t)
struct TrackKin {
	float v[3], w[3];
};
__device__ __forceinline__ TrackKin* track_kins() {
	__shared__ TrackKin s[CB200_MAX_COLLISION_OBJECTS];
	return s;
}
// the rotation matrix of the quaternion q = (w, x, y, z), row-major (element (i, k) at 3 i + k)
__device__ __forceinline__ void track_quat_mat(const float* q, float* Q) {
	const float w = q[0], x = q[1], y = q[2], z = q[3];
	Q[0] = 1.f - 2.f * (y * y + z * z);
	Q[1] = 2.f * (x * y - w * z);
	Q[2] = 2.f * (x * z + w * y);
	Q[3] = 2.f * (x * y + w * z);
	Q[4] = 1.f - 2.f * (x * x + z * z);
	Q[5] = 2.f * (y * z - w * x);
	Q[6] = 2.f * (x * z - w * y);
	Q[7] = 2.f * (y * z + w * x);
	Q[8] = 1.f - 2.f * (x * x + y * y);
}
// The pose of the object o on its n records rec (flags: CB200_TRACK_*) at time t, as the frame f and the kinematic velocity k.  The
// periodic wrap, the segment search and u are float: t' = t_0 + fmodf(t - t_0, t_last - t_0) for t >= t_last, then the segment s with
// t_s <= t' < t_{s+1} by bisection; before t_0 and from t_last on the key's pose at rest.  f.rot holds R(t) = Q(t) R0 as collider_make_frame
// holds its rotation (element (i, j) of the world-from-material matrix at 3 j + i), f.b = c(t), f.s_inv = 1.
template<class P>
__device__ __forceinline__ void track_make_frame(const P& o, const float4* rec, int n, int flags, float t, ColliderFrame& f, TrackKin& k) {
	const float t0 = __ldg(&rec[0].x), tn = __ldg(&rec[4 * (n - 1)].x);
	if((flags & CB200_TRACK_PERIODIC) && n > 1 && t >= tn) t = t0 + fmodf(t - t0, tn - t0);
	float c[3], q[4], v[3] = {0.f, 0.f, 0.f}, w[3] = {0.f, 0.f, 0.f};
	if(n > 1 && t >= t0 && t < tn) {
		int lo = 0, hi = n - 1;
		while(hi - lo > 1) {
			const int mid = (lo + hi) >> 1;
			if(t >= __ldg(&rec[4 * mid].x)) lo = mid;
			else hi = mid;
		}
		const float4 a0 = __ldg(rec + 4 * lo), a1 = __ldg(rec + 4 * lo + 1), a2 = __ldg(rec + 4 * lo + 2), a3 = __ldg(rec + 4 * lo + 3);
		const float4 b0 = __ldg(rec + 4 * lo + 4), b2 = __ldg(rec + 4 * lo + 6);
		const float h = b0.x - a0.x, u = (t - a0.x) / h;
		const float ck[3] = {a0.y, a0.z, a0.w}, c1[3] = {b0.y, b0.z, b0.w}, mk[3] = {a2.x, a2.y, a2.z}, m1[3] = {b2.x, b2.y, b2.z};
		if(flags & CB200_TRACK_SMOOTH) {
			const float u2 = u * u, u3 = u2 * u;
			const float h00 = 2.f * u3 - 3.f * u2 + 1.f, h10 = u3 - 2.f * u2 + u, h01 = 3.f * u2 - 2.f * u3, h11 = u3 - u2;
			const float d00 = 6.f * u2 - 6.f * u, d10 = 3.f * u2 - 4.f * u + 1.f, d11 = 3.f * u2 - 2.f * u;
#pragma unroll
			for(int d = 0; d < 3; ++d) {
				c[d] = h00 * ck[d] + h10 * h * mk[d] + h01 * c1[d] + h11 * h * m1[d];
				v[d] = d00 * (ck[d] - c1[d]) / h + d10 * mk[d] + d11 * m1[d];
			}
		} else {
#pragma unroll
			for(int d = 0; d < 3; ++d) {
				c[d] = ck[d] + u * (c1[d] - ck[d]);
				v[d] = (c1[d] - ck[d]) / h;
			}
		}
		// q = q_k (x) exp(u r / 2), r = theta_k a_k; omega = R(q_k) r / h
		const float qk[4] = {a1.x, a1.y, a1.z, a1.w}, r[3] = {a2.w, a3.x, a3.y};
		const float th = sqrtf(r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
		float e[4] = {1.f, 0.f, 0.f, 0.f};
		if(th > 0.f) {
			const float hlf = 0.5f * u * th, sn = sinf(hlf) / th;
			e[0] = cosf(hlf);
			e[1] = r[0] * sn;
			e[2] = r[1] * sn;
			e[3] = r[2] * sn;
		}
		q[0] = qk[0] * e[0] - qk[1] * e[1] - qk[2] * e[2] - qk[3] * e[3];
		q[1] = qk[0] * e[1] + qk[1] * e[0] + qk[2] * e[3] - qk[3] * e[2];
		q[2] = qk[0] * e[2] - qk[1] * e[3] + qk[2] * e[0] + qk[3] * e[1];
		q[3] = qk[0] * e[3] + qk[1] * e[2] - qk[2] * e[1] + qk[3] * e[0];
		float Qk[9];
		track_quat_mat(qk, Qk);
#pragma unroll
		for(int d = 0; d < 3; ++d) w[d] = (Qk[3 * d] * r[0] + Qk[3 * d + 1] * r[1] + Qk[3 * d + 2] * r[2]) / h;
	} else {
		const int kk = (n > 1 && t >= tn) ? n - 1 : 0;
		const float4 a0 = __ldg(rec + 4 * kk), a1 = __ldg(rec + 4 * kk + 1);
		c[0] = a0.y;
		c[1] = a0.z;
		c[2] = a0.w;
		q[0] = a1.x;
		q[1] = a1.y;
		q[2] = a1.z;
		q[3] = a1.w;
	}
	float Q[9];
	track_quat_mat(q, Q);
#pragma unroll
	for(int j = 0; j < 3; ++j)
#pragma unroll
		for(int i = 0; i < 3; ++i) f.rot[3 * j + i] = Q[3 * i] * o.rot_mat[3 * j] + Q[3 * i + 1] * o.rot_mat[3 * j + 1] + Q[3 * i + 2] * o.rot_mat[3 * j + 2];
#pragma unroll
	for(int d = 0; d < 3; ++d) {
		f.b[d] = c[d];
		k.v[d] = v[d];
		k.w[d] = w[d];
	}
	f.s_inv = 1.f;
}
// collider_resolve for a tracked object: the same material point (s_inv = 1), query and response, with the rigid object velocity
// vo = c'(t) + omega(t) x (p - c(t)) of its kinematic velocity k.  The response is a copy of collider_resolve's, statement for
// statement: sharing one body changes the instruction schedule the untracked instances compile to.
template<class P, class Q>
__device__ __forceinline__ void track_resolve(const P& c, const ColliderFrame& f, const TrackKin& k, float dx, int nx, int ny, int nz, float& vx, float& vy, float& vz, Q&& query) {
	const float p[3] = {(float) nx * dx, (float) ny * dx, (float) nz * dx};
	float xm[3], x[3];
	collider_material_point(c, f, p, xm, x);
	const float* R = f.rot;
	float on[3];
	if(!query(x, on)) return;
	const float* w = k.w;
	const float vo[3] = {k.v[0] + (w[1] * xm[2] - w[2] * xm[1]), k.v[1] + (w[2] * xm[0] - w[0] * xm[2]), k.v[2] + (w[0] * xm[1] - w[1] * xm[0])};
	float v[3] = {vx - vo[0], vy - vo[1], vz - vo[2]};
	if(c.type == CB200_STICKY) {
		v[0] = v[1] = v[2] = 0.f;
	} else {
		if(c.type == CB200_SEPARATE && on[0] == 0.f && on[1] == 0.f && on[2] == 0.f) {
			vx = vy = vz = 0.f;
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

// ---- motion tracks: the host side (DESIGN.md section 2.14) --------------------------------------------------------------------
// cb200_track_prepare: validates keys[0, n) with flags and writes their records to out (untouched on a rejection), in double
inline bool track_prepare(const cb200_track_key* keys, int n, int flags, cb200_track_record* out) {
	if(!keys || !out || n < 1 || n > CB200_MAX_TRACK_KEYS || (flags & ~(CB200_TRACK_SMOOTH | CB200_TRACK_PERIODIC))) return false;
	const bool periodic = (flags & CB200_TRACK_PERIODIC) != 0;
	if(periodic && n < 2) return false;
	std::vector<double> q((size_t) n * 4);
	for(int k = 0; k < n; ++k) {
		const cb200_track_key& key = keys[k];
		if(!finite_all(&key.t, 1) || !finite_all(key.pos, 3) || !finite_all(key.rot, 4)) return false;
		if(k > 0 && !(key.t > keys[k - 1].t)) return false;
		double* qk = &q[4 * (size_t) k];
		double nn = 0.0;
		for(int c = 0; c < 4; ++c) nn += (double) key.rot[c] * key.rot[c];
		if(!(nn > 0.0)) return false;
		const double len = std::sqrt(nn);
		for(int c = 0; c < 4; ++c) qk[c] = key.rot[c] / len;
	}
	if(periodic) {
		const cb200_track_key &a = keys[0], &b = keys[n - 1];
		if(a.pos[0] != b.pos[0] || a.pos[1] != b.pos[1] || a.pos[2] != b.pos[2]) return false;
		bool same = true, flip = true;
		for(int c = 0; c < 4; ++c) {
			same &= (float) q[c] == (float) q[4 * (size_t) (n - 1) + c];
			flip &= (float) q[c] == (float) -q[4 * (size_t) (n - 1) + c];
		}
		if(!same && !flip) return false;
	}
	for(int k = 1; k < n; ++k) {  // one hemisphere: each quaternion on the side of the one before it
		const double *p0 = &q[4 * (size_t) (k - 1)];
		double* p1 = &q[4 * (size_t) k];
		const double d = p0[0] * p1[0] + p0[1] * p1[1] + p0[2] * p1[2] + p0[3] * p1[3];
		if(d == 0.0) return false;  // 180 degrees apart: the arc is ambiguous
		if(d < 0.0)
			for(int c = 0; c < 4; ++c) p1[c] = -p1[c];
	}
	std::vector<cb200_track_record> rec((size_t) n);
	for(int k = 0; k < n; ++k) {
		cb200_track_record& r = rec[k];
		r = cb200_track_record {};
		r.t = keys[k].t;
		for(int d = 0; d < 3; ++d) r.pos[d] = keys[k].pos[d];
		for(int c = 0; c < 4; ++c) r.rot[c] = (float) q[4 * (size_t) k + c];
		if((flags & CB200_TRACK_SMOOTH) && n > 1) {  // m_k = (c_{k+1} - c_{k-1}) / (t_{k+1} - t_{k-1}); one-sided ends, or wrapped around
			int lo = k - 1, hi = k + 1;
			double span = 0.0;
			if(periodic && (k == 0 || k == n - 1)) {
				lo = n - 2;
				hi = 1;
				span = ((double) keys[1].t - keys[0].t) + ((double) keys[n - 1].t - keys[n - 2].t);
			} else {
				lo = std::max(lo, 0);
				hi = std::min(hi, n - 1);
				span = (double) keys[hi].t - keys[lo].t;
			}
			for(int d = 0; d < 3; ++d) r.tangent[d] = (float) (((double) keys[hi].pos[d] - keys[lo].pos[d]) / span);
		}
		if(k + 1 < n) {  // r = conj(q_k) (x) q_{k+1} = exp(theta a / 2)
			const double *a = &q[4 * (size_t) k], *b = &q[4 * (size_t) (k + 1)];
			const double w = a[0] * b[0] + a[1] * b[1] + a[2] * b[2] + a[3] * b[3];
			const double v[3] = {a[0] * b[1] - a[1] * b[0] - a[2] * b[3] + a[3] * b[2], a[0] * b[2] + a[1] * b[3] - a[2] * b[0] - a[3] * b[1],
			                     a[0] * b[3] - a[1] * b[2] + a[2] * b[1] - a[3] * b[0]};
			const double sn = std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
			if(sn > 0.0) {
				const double th = 2.0 * std::atan2(sn, w);
				for(int d = 0; d < 3; ++d) r.rotvec[d] = (float) (v[d] / sn * th);
			}
		}
	}
	std::copy(rec.begin(), rec.end(), out);
	return true;
}
// whether object o may move on a track: the reference motion model's velocities all 0
inline bool track_object_ok(const cb200_collision_object& o) {
	for(int d = 0; d < 3; ++d)
		if(o.trans_vel[d] != 0.f || o.omega[d] != 0.f) return false;
	return o.dsdt == 0.f;
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
// boundary_frames_cta with the objects' tracks tr (section 2.14): thread i builds object i's frame from its track when it has one
// (and its kinematic velocity in track_kins), else as boundary_frames_cta does; one barrier
template<bool COLLIDE>
__device__ __forceinline__ const BoundaryFrames& boundary_frames_tracks_cta(const Boundaries& b, const Tracks& tr, float t) {
	BoundaryFrames& s = boundary_frames();
	if constexpr(COLLIDE) {
		if(threadIdx.x == 0) collider_make_frame(b.col, t, s.col);
	}
	const int i = (int) threadIdx.x - (COLLIDE ? 32 : 0);
	if(i >= 0 && i < b.objects.n) {
		s.o[i] = b.objects.o[i];
		if(tr.n[i] > 0) track_make_frame(s.o[i], tr.rec + 4 * tr.off[i], tr.n[i], tr.flags[i], t, s.f[i], track_kins()[i]);
		else collider_make_frame(s.o[i], t, s.f[i]);
	}
	__syncthreads();
	return s;
}
// one object of the chain: object i (parameters o, frame f) with its query; TRACKS: a tracked object (tr->n[i] > 0) takes its
// kinematic velocity from track_kins
template<bool LEVELSETS, bool TRACKS>
__device__ __forceinline__ void object_resolve_one(const Tracks* tr, int i, const cb200_collision_object& o, const ColliderFrame& f, float dx, int nx, int ny, int nz, float& vx, float& vy, float& vz) {
	auto q = [&](const float* x, float* n) {
		if constexpr(LEVELSETS) return object_query_levelsets(o, x, n);
		else return object_query(o, x, n);
	};
	if constexpr(TRACKS) {
		if(tr->n[i] > 0) {
			track_resolve(o, f, track_kins()[i], dx, nx, ny, nz, vx, vy, vz, q);
			return;
		}
	}
	collider_resolve(o, f, dx, nx, ny, nz, vx, vy, vz, q);
}
// the chain at grid node (nx, ny, nz), its frames s built by boundary_frames_cta; LEVELSETS (implies OBJECTS): level-set objects are
// answered from the views levelset_views_cta copied; TRACKS (implies OBJECTS): frames from boundary_frames_tracks_cta, tracks tr
template<bool COLLIDE, bool OBJECTS, bool LEVELSETS = false, bool TRACKS = false>
__device__ __forceinline__ void boundaries_resolve(const Boundaries& b, const BoundaryFrames& s, const Cfg& cfg, int nx, int ny, int nz, float& vx, float& vy, float& vz, const Tracks* tr = nullptr) {
	static_assert(OBJECTS || !LEVELSETS, "level-set objects are objects");
	static_assert(OBJECTS || !TRACKS, "tracks move objects");
	if constexpr(COLLIDE) collider_resolve(b.col, s.col, cfg.dx, nx, ny, nz, vx, vy, vz, [&](const float* x, float* n) { return collider_query(b.col, cfg, x, n); });
	if constexpr(OBJECTS && TRACKS) {
		for(int i = 0; i < b.objects.n; ++i) object_resolve_one<LEVELSETS, true>(tr, i, s.o[i], s.f[i], cfg.dx, nx, ny, nz, vx, vy, vz);
	} else if constexpr(OBJECTS) {
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
template<bool COLLIDE, bool OBJECTS, bool LEVELSETS, class Stage, bool TRACKS = false>
__device__ __forceinline__ void boundaries_resolve_pair(const Boundaries& b, const BoundaryFrames& s, const Cfg& cfg, int nx, int ny, int nz, bool hx, bool hy, float2& v0, float2& v1,
                                                        float2& v2, Stage&& stage, const Tracks* tr = nullptr) {
	static_assert(OBJECTS || !LEVELSETS, "level-set objects are objects");
	if constexpr(OBJECTS && TRACKS) {
		if constexpr(COLLIDE) {
			const float2 i0 = v0, i1 = v1, i2 = v2;
			auto q = [&](const float* x, float* n) { return collider_query(b.col, cfg, x, n); };
			if(hx) collider_resolve(b.col, s.col, cfg.dx, nx, ny, nz, v0.x, v1.x, v2.x, q);
			if(hy) collider_resolve(b.col, s.col, cfg.dx, nx, ny, nz + 1, v0.y, v1.y, v2.y, q);
			stage(0, s.col, i0, i1, i2);
		}
		for(int i = 0; i < b.objects.n; ++i) {
			const float2 i0 = v0, i1 = v1, i2 = v2;
			if(hx) object_resolve_one<LEVELSETS, true>(tr, i, s.o[i], s.f[i], cfg.dx, nx, ny, nz, v0.x, v1.x, v2.x);
			if(hy) object_resolve_one<LEVELSETS, true>(tr, i, s.o[i], s.f[i], cfg.dx, nx, ny, nz + 1, v0.y, v1.y, v2.y);
			stage(1 + i, s.f[i], i0, i1, i2);
		}
		return;
	}
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
template<bool COLLIDE, bool OBJECTS, bool LEVELSETS = false, bool TRACKS = false>
__device__ __forceinline__ float cell_vel_sq_boundaries(float m, float p0, float p1, float p2, bool wx, bool wy, bool wz, float gdt, const Boundaries& bd, const BoundaryFrames& s, const Cfg& cfg, int nx, int ny, int nz,
                                                        const Tracks* tr = nullptr) {
	if(!node_has_mass(m)) return 0.f;
	const float mi = 1.f / m;
	float a = wx ? 0.f : p0 * mi, b = (wy ? 0.f : p1 * mi) + gdt, d = wz ? 0.f : p2 * mi;
	boundaries_resolve<COLLIDE, OBJECTS, LEVELSETS, TRACKS>(bd, s, cfg, nx, ny, nz, a, b, d, tr);
	const float sq = a * a + b * b + d * d;
	return isnan(sq) ? INFINITY : sq;
}
// cell_pair_vel_sq (common.cuh) with the chain: the two cells lane holds of block (kx, ky, kz), whose grid block is s2 (float2 view)
template<bool COLLIDE, bool OBJECTS, bool LEVELSETS = false, bool TRACKS = false>
__device__ __forceinline__ float cell_pair_vel_sq_boundaries(const Cfg& cfg, const Boundaries& bd, const BoundaryFrames& s, const float2* s2, int lane, int kx, int ky, int kz, bool wx, bool wy, bool wz, float gdt,
                                                             const Tracks* tr = nullptr) {
	const float2 m = s2[lane], p0 = s2[32 + lane], p1 = s2[64 + lane], p2 = s2[96 + lane];
	const int nx = 4 * kx + (lane >> 3), ny = 4 * ky + ((lane >> 1) & 3), nz = 4 * kz + 2 * (lane & 1);
	return fmaxf(cell_vel_sq_boundaries<COLLIDE, OBJECTS, LEVELSETS, TRACKS>(m.x, p0.x, p1.x, p2.x, wx, wy, wz, gdt, bd, s, cfg, nx, ny, nz, tr),
	             cell_vel_sq_boundaries<COLLIDE, OBJECTS, LEVELSETS, TRACKS>(m.y, p0.y, p1.y, p2.y, wx, wy, wz, gdt, bd, s, cfg, nx, ny, nz + 1, tr));
}

}  // namespace cb200
