// collider.cuh -- signed-distance collision object applied to grid nodes (SignedDistanceGrid, Projects/MGSP/boundary_condition.cuh:25-250).
//
// The level set is dense over the whole domain in the reference's layout (signed_distance_field_, boundary_condition.cuh:15-16):
// one 1 KiB block per grid block, blocks row-major (x*G*G + y*G + z), inside a block 4 channels SoA (distance, gradient x, y, z)
// of 64 cells (cell = x*16 + y*4 + z).  Every caller (the grid update and the two next-max predictors of grid.cuh) shares
// collider_resolve, so the max the MGSP ranks agree on is the max the next grid update finds.
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

__device__ __forceinline__ void collider_make_frame(const ColliderView& c, float t, ColliderFrame& f) {
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

// one thread builds the frame, the CTA reads it from shared memory
__device__ __forceinline__ const ColliderFrame& collider_frame_cta(const ColliderView& c, float t) {
	__shared__ ColliderFrame s_frame;
	if(threadIdx.x == 0) collider_make_frame(c, t, s_frame);
	__syncthreads();
	return s_frame;
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

// detect_and_resolve_collision (:159-249) of the velocity v at grid node (nx, ny, nz).  The object velocity takes a true
// omega x r where the reference's vec3_cross_vec3 (:92-95) adds all products; get_material_velocity keeps MnBase's
// vec_cross_mul_vec_3d as it is (MatrixUtils.h:54-58).
__device__ __forceinline__ void collider_resolve(const ColliderView& c, const ColliderFrame& f, const Cfg& cfg, int nx, int ny, int nz, float& vx, float& vy, float& vz) {
	const float xm[3] = {(float) nx * cfg.dx - f.b[0], (float) ny * cfg.dx - f.b[1], (float) nz * cfg.dx - f.b[2]};
	const float x0[3] = {xm[0] * f.s_inv, xm[1] * f.s_inv, xm[2] * f.s_inv};
	const float* R = f.rot;
	float x[3];
#pragma unroll
	for(int d = 0; d < 3; ++d) x[d] = (R[3 * d] * x0[0] + R[3 * d + 1] * x0[1] + R[3 * d + 2] * x0[2]) * c.scale + c.trans[d];  // mat_t_mul_vec_3d
	float on[3];
	if(!collider_query(c, cfg, x, on)) return;
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

// grid-update velocity of one cell (wall mask, gravity on y, collider) and its |v|^2, NaN -> +inf; no mass -> 0
__device__ __forceinline__ float cell_vel_sq_collide(float m, float p0, float p1, float p2, bool wx, bool wy, bool wz, float gdt, const ColliderView& c, const ColliderFrame& f, const Cfg& cfg, int nx, int ny, int nz) {
	if(!(m > 0.f)) return 0.f;
	const float mi = 1.f / m;
	float a = wx ? 0.f : p0 * mi, b = (wy ? 0.f : p1 * mi) + gdt, d = wz ? 0.f : p2 * mi;
	collider_resolve(c, f, cfg, nx, ny, nz, a, b, d);
	const float sq = a * a + b * b + d * d;
	return isnan(sq) ? INFINITY : sq;
}
// cell_pair_vel_sq (common.cuh) with the collider: the two cells lane holds of block (kx, ky, kz), whose grid block is s2 (float2 view)
__device__ __forceinline__ float cell_pair_vel_sq_collide(const Cfg& cfg, const ColliderView& c, const ColliderFrame& f, const float2* s2, int lane, int kx, int ky, int kz, bool wx, bool wy, bool wz, float gdt) {
	const float2 m = s2[lane], p0 = s2[32 + lane], p1 = s2[64 + lane], p2 = s2[96 + lane];
	const int nx = 4 * kx + (lane >> 3), ny = 4 * ky + ((lane >> 1) & 3), nz = 4 * kz + 2 * (lane & 1);
	return fmaxf(cell_vel_sq_collide(m.x, p0.x, p1.x, p2.x, wx, wy, wz, gdt, c, f, cfg, nx, ny, nz), cell_vel_sq_collide(m.y, p0.y, p1.y, p2.y, wx, wy, wz, gdt, c, f, cfg, nx, ny, nz + 1));
}

}  // namespace cb200
