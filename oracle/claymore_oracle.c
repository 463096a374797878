/*
 * claymore_oracle.c -- CPU restatement of the claymore GMPM hot path.
 * TEST INFRASTRUCTURE ONLY (see claymore_oracle.h).  Plain C99 + OpenMP, FP32 arithmetic,
 * compiled with -ffp-contract=off so that products and sums round separately like the
 * reference's __fadd_rn/__fsub_rn-pinned SVD (Library/MnBase/Math/Matrix/svd.cuh:124-158).
 *
 * All "ref:" citations are relative to /root/reference.
 */
#include "claymore_oracle.h"

#include <float.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

/* ------------------------------------------------------------------------------------------ */
/* config helpers (ref: Projects/GMPM/settings.h:56-79)                                        */
/* ------------------------------------------------------------------------------------------ */
static int g_threads = 1;
void orc_set_num_threads(int n) { g_threads = n > 0 ? n : 1; }
int orc_get_num_threads(void) { return g_threads; }

#define BLOCK_VOL 64
#define BIN_CAP 32

static inline float cfg_dxinv(const orc_config* c) { return (float) (1 << c->domain_bits); }
static inline float cfg_dx(const orc_config* c) { return 1.f / cfg_dxinv(c); }
static inline float cfg_dinv(const orc_config* c) { return 4.f * cfg_dxinv(c) * cfg_dxinv(c); }
static inline int cfg_gsize(const orc_config* c) { return 1 << (c->domain_bits - 2); }
static inline int cfg_ppb(const orc_config* c) { return c->max_ppc * BLOCK_VOL; }
static inline int bin_floats(int material) { return material == ORC_J_FLUID ? 128 : 512; }

/* row-major table offset, ref: Library/MnBase/Math/Vec.h:51-63 */
static inline long tbl(const orc_config* c, int x, int y, int z) {
	const long g = cfg_gsize(c);
	return ((long) x * g + y) * g + z;
}
static inline int in_domain(const orc_config* c, int x, int y, int z) {
	const int g = cfg_gsize(c);
	return x >= 0 && y >= 0 && z >= 0 && x < g && y < g && z < g;
}
/* Partition::query, ref: Projects/GMPM/hash_table.cuh:129-131 (out-of-domain keys -> -1 instead of UB) */
static inline int part_query(const orc_config* c, const orc_partition* p, int x, int y, int z) {
	if(!in_domain(c, x, y, z)) return -1;
	return p->index_table[tbl(c, x, y, z)];
}
/* Partition::insert, ref: Projects/GMPM/hash_table.cuh:117-127 (sequential form of CAS + atomicAdd) */
static inline int part_insert(const orc_config* c, orc_partition* p, int x, int y, int z) {
	if(!in_domain(c, x, y, z)) return -1;
	int* slot = &p->index_table[tbl(c, x, y, z)];
	if(*slot == -1) {
		const int idx = (*p->count)++;
		*slot = idx;
		p->active_keys[3 * idx + 0] = x;
		p->active_keys[3 * idx + 1] = y;
		p->active_keys[3 * idx + 2] = z;
		return idx;
	}
	return -1;
}
/* get_block_id, ref: Projects/GMPM/utility_funcs.hpp:21-23 */
static inline int cell_of(const orc_config* c, float p) { return (int) lroundf(p * cfg_dxinv(c)); }

/* bspline_weight, ref: Projects/GMPM/utility_funcs.hpp:10-19 */
void orc_bspline_weight(const orc_config* cfg, float p, float* w) {
	float d = p * cfg_dxinv(cfg);
	w[0] = 0.5f * (1.5f - d) * (1.5f - d);
	d -= 1.0f;
	w[1] = 0.75f - d * d;
	d = 0.5f + d;
	w[2] = 0.5f * d * d;
}

/* ------------------------------------------------------------------------------------------ */
/* 3x3 SVD: restatement of the McAdams et al. minimal-branching algorithm as carried by        */
/* ref: Library/MnBase/Math/Matrix/svd.cuh:28-1124.  Matrices are row/col indexed m[r][c].     */
/* ------------------------------------------------------------------------------------------ */
#define SVD_FOUR_GAMMA_SQ 5.8284273147583007813f
#define SVD_SIN_PI_8 0.38268342614173889160f /* bits 1053028117, svd.cuh:11 */
#define SVD_COS_PI_8 0.92387956380844116211f /* bits 1064076127 (one ulp above the nearest float), svd.cuh:12 */
#define SVD_TINY 1.e-20f
#define SVD_SMALL 1.e-12f
#define SVD_SWEEPS 4

/* __frsqrt_rn stand-in: correctly rounded 1/sqrt via double */
static inline float rsqrt_rn(float x) { return (float) (1.0 / sqrt((double) x)); }
/* one Newton step on rsqrt as at svd.cuh:486-491 */
static inline float rsqrt_refined(float x) {
	float r = rsqrt_rn(x);
	float h = r * 0.5f;
	float t = r * h;
	t = r * t;
	t = x * t;
	r = r + h;
	r = r - t;
	return r;
}

/* One Jacobi conjugation on the symmetric matrix entries (a=S_pp, b=S_qp, c=S_qq, d=S_rp, e=S_rq, f=S_rr)
 * accumulating into quaternion q=(s; x,y,z) permuted so that "z" is the rotation axis.
 * ref: svd.cuh:165-262 (first instance), :268-365, :371-470 (cyclic permutations). */
static void jacobi_conjugate(float* a, float* b, float* c, float* d, float* e, float* f, float* qs, float* qx, float* qy, float* qz) {
	float sh = *b * 0.5f;
	float t5 = *a - *c;
	float ch;
	if(sh * sh >= SVD_TINY) {
		ch = t5;
	} else {
		sh = 0.f;
		ch = 1.f;
	}
	float t1 = sh * sh;
	float t2 = ch * ch;
	float t3 = t1 + t2;
	float t4 = rsqrt_rn(t3);
	sh = t4 * sh;
	ch = t4 * ch;
	t1 = SVD_FOUR_GAMMA_SQ * t1;
	if(t2 <= t1) {
		sh = SVD_SIN_PI_8;
		ch = SVD_COS_PI_8;
	}
	t1 = sh * sh;
	t2 = ch * ch;
	const float cc = t2 - t1;
	float ss = ch * sh;
	ss = ss + ss;

	/* Givens conjugation */
	t3 = t1 + t2;
	*f = *f * t3;
	*d = *d * t3;
	*e = *e * t3;
	*f = *f * t3;

	t1 = ss * *d;
	t2 = ss * *e;
	*d = cc * *d;
	*e = cc * *e;
	*d = t2 + *d;
	*e = *e - t1;

	t2 = ss * ss;
	t1 = *c * t2;
	t3 = *a * t2;
	t4 = cc * cc;
	*a = *a * t4;
	*c = *c * t4;
	*a = *a + t1;
	*c = *c + t3;
	t4 = t4 - t2;
	t2 = *b + *b;
	*b = *b * t4;
	t4 = cc * ss;
	t2 = t2 * t4;
	t5 = t5 * t4;
	*a = *a + t2;
	*b = *b - t5;
	*c = *c - t2;

	/* cumulative rotation */
	t1 = sh * *qx;
	t2 = sh * *qy;
	t3 = sh * *qz;
	sh = sh * *qs;
	*qs = ch * *qs;
	*qx = ch * *qx;
	*qy = ch * *qy;
	*qz = ch * *qz;
	*qz = *qz + sh;
	*qs = *qs - t3;
	*qx = *qx + t2;
	*qy = *qy - t1;
}

/* conditional column swap with sign fix, ref: svd.cuh:611-770 */
static void cond_swap_cols(float B[3][3], float V[3][3], float* n, int p, int q, int neg) {
	if(n[p] < n[q]) {
		for(int r = 0; r < 3; ++r) {
			float t = B[r][p];
			B[r][p] = B[r][q];
			B[r][q] = t;
			t = V[r][p];
			V[r][p] = V[r][q];
			V[r][q] = t;
		}
		float t = n[p];
		n[p] = n[q];
		n[q] = t;
		for(int r = 0; r < 3; ++r) {
			B[r][neg] = B[r][neg] * -1.f;
			V[r][neg] = V[r][neg] * -1.f;
		}
	}
}

/* Givens rotation zeroing B[q][p] against pivot B[p][p]; rows p,q of B and columns p,q of U are rotated.
 * ref: svd.cuh:786-905 (first), :907-1005 (second), :1007-1105 (third). */
static void qr_givens(float B[3][3], float U[3][3], int p, int q) {
	const float pivot = B[p][p];
	const float below = B[q][p];
	float sh = (below * below >= SVD_SMALL) ? below : 0.f;
	float ch = 0.f - pivot;
	ch = fmaxf(ch, pivot);
	ch = fmaxf(ch, SVD_SMALL);
	const int pivot_nonneg = pivot >= 0.f;

	float t1 = ch * ch;
	float t2 = sh * sh;
	t2 = t1 + t2;
	t1 = rsqrt_refined(t2);
	t1 = t1 * t2; /* sqrt(ch^2+sh^2) */
	ch = ch + t1;
	if(!pivot_nonneg) {
		const float t = ch;
		ch = sh;
		sh = t;
	}
	t1 = ch * ch;
	t2 = sh * sh;
	t2 = t1 + t2;
	t1 = rsqrt_refined(t2);
	ch = ch * t1;
	sh = sh * t1;
	float c = ch * ch;
	float s = sh * sh;
	c = c - s;
	s = sh * ch;
	s = s + s;

	for(int col = 0; col < 3; ++col) {
		const float a1 = s * B[p][col];
		const float a2 = s * B[q][col];
		B[p][col] = c * B[p][col];
		B[q][col] = c * B[q][col];
		B[p][col] = B[p][col] + a2;
		B[q][col] = B[q][col] - a1;
	}
	for(int row = 0; row < 3; ++row) {
		const float a1 = s * U[row][p];
		const float a2 = s * U[row][q];
		U[row][p] = c * U[row][p];
		U[row][q] = c * U[row][q];
		U[row][p] = U[row][p] + a2;
		U[row][q] = U[row][q] - a1;
	}
}

/* F, U, V column-major (m[r + 3c]) exactly as compute_stress passes them (constitutive_models.cuh:43) */
void orc_svd3(const float* Fcm, float* Ucm, float* S, float* Vcm) {
	float A[3][3];
	for(int r = 0; r < 3; ++r)
		for(int c = 0; c < 3; ++c) A[r][c] = Fcm[r + 3 * c];

	/* normal equations A^T A, lower triangle; ref: svd.cuh:120-158 */
	float s11 = A[0][0] * A[0][0];
	s11 = A[1][0] * A[1][0] + s11;
	s11 = A[2][0] * A[2][0] + s11;
	float s21 = A[0][1] * A[0][0];
	s21 = A[1][1] * A[1][0] + s21;
	s21 = A[2][1] * A[2][0] + s21;
	float s31 = A[0][2] * A[0][0];
	s31 = A[1][2] * A[1][0] + s31;
	s31 = A[2][2] * A[2][0] + s31;
	float s22 = A[0][1] * A[0][1];
	s22 = A[1][1] * A[1][1] + s22;
	s22 = A[2][1] * A[2][1] + s22;
	float s32 = A[0][2] * A[0][1];
	s32 = A[1][2] * A[1][1] + s32;
	s32 = A[2][2] * A[2][1] + s32;
	float s33 = A[0][2] * A[0][2];
	s33 = A[1][2] * A[1][2] + s33;
	s33 = A[2][2] * A[2][2] + s33;

	float qs = 1.f, qx = 0.f, qy = 0.f, qz = 0.f;
	for(int sweep = 0; sweep < SVD_SWEEPS; ++sweep) {
		jacobi_conjugate(&s11, &s21, &s22, &s31, &s32, &s33, &qs, &qx, &qy, &qz);
		jacobi_conjugate(&s22, &s32, &s33, &s21, &s31, &s11, &qs, &qy, &qz, &qx);
		jacobi_conjugate(&s33, &s31, &s11, &s32, &s21, &s22, &qs, &qz, &qx, &qy);
	}

	/* normalise quaternion, ref: svd.cuh:476-498 */
	float n2 = qs * qs;
	n2 = qx * qx + n2;
	n2 = qy * qy + n2;
	n2 = qz * qz + n2;
	const float rn = rsqrt_refined(n2);
	qs *= rn;
	qx *= rn;
	qy *= rn;
	qz *= rn;

	/* quaternion -> V, ref: svd.cuh:504-531 */
	float V[3][3];
	{
		float t1 = qx * qx, t2 = qy * qy, t3 = qz * qz;
		float v11 = qs * qs;
		float v22 = v11 - t1;
		float v33 = v22 - t2;
		v33 = v33 + t3;
		v22 = v22 + t2;
		v22 = v22 - t3;
		v11 = v11 + t1;
		v11 = v11 - t2;
		v11 = v11 - t3;
		t1 = qx + qx;
		t2 = qy + qy;
		t3 = qz + qz;
		float v32 = qs * t1;
		float v13 = qs * t2;
		float v21 = qs * t3;
		t1 = qy * t1;
		t2 = qz * t2;
		t3 = qx * t3;
		const float v12 = t1 - v21;
		const float v23 = t2 - v32;
		const float v31 = t3 - v13;
		v21 = t1 + v21;
		v32 = t2 + v32;
		v13 = t3 + v13;
		V[0][0] = v11; V[0][1] = v12; V[0][2] = v13;
		V[1][0] = v21; V[1][1] = v22; V[1][2] = v23;
		V[2][0] = v31; V[2][1] = v32; V[2][2] = v33;
	}

	/* B = A V, ref: svd.cuh:537-589 */
	float B[3][3];
	for(int r = 0; r < 3; ++r)
		for(int c = 0; c < 3; ++c) {
			float acc = V[0][c] * A[r][0];
			acc = acc + V[1][c] * A[r][1];
			acc = acc + V[2][c] * A[r][2];
			B[r][c] = acc;
		}

	/* sort columns by squared norm, ref: svd.cuh:595-770 */
	float n[3];
	for(int c = 0; c < 3; ++c) {
		float acc = B[0][c] * B[0][c];
		acc = acc + B[1][c] * B[1][c];
		acc = acc + B[2][c] * B[2][c];
		n[c] = acc;
	}
	cond_swap_cols(B, V, n, 0, 1, 1);
	cond_swap_cols(B, V, n, 0, 2, 0);
	cond_swap_cols(B, V, n, 1, 2, 2);

	/* QR by Givens, ref: svd.cuh:776-1105 */
	float U[3][3] = {{1.f, 0.f, 0.f}, {0.f, 1.f, 0.f}, {0.f, 0.f, 1.f}};
	qr_givens(B, U, 0, 1);
	qr_givens(B, U, 0, 2);
	qr_givens(B, U, 1, 2);

	for(int r = 0; r < 3; ++r)
		for(int c = 0; c < 3; ++c) {
			Ucm[r + 3 * c] = U[r][c];
			Vcm[r + 3 * c] = V[r][c];
		}
	S[0] = B[0][0];
	S[1] = B[1][1];
	S[2] = B[2][2];
}

/* ------------------------------------------------------------------------------------------ */
/* column-major 3x3 helpers, ref: Library/MnBase/Math/Matrix/MatrixUtils.h                     */
/* ------------------------------------------------------------------------------------------ */
/* matmul_mat_diag_mat_t_3d, MatrixUtils.h:29-41 */
static void mat_diag_mat_t(float* out, const float* m1, const float* dg, const float* m2) {
	for(int c = 0; c < 3; ++c)
		for(int r = 0; r < 3; ++r) out[r + 3 * c] = m1[r] * dg[0] * m2[c] + m1[r + 3] * dg[1] * m2[c + 3] + m1[r + 6] * dg[2] * m2[c + 6];
}
/* matrix_matrix_multiplication_3d, MatrixUtils.h:147-157 */
static void mat_mul(const float* a, const float* b, float* c) {
	for(int col = 0; col < 3; ++col)
		for(int r = 0; r < 3; ++r) c[r + 3 * col] = a[r] * b[3 * col] + a[r + 3] * b[3 * col + 1] + a[r + 6] * b[3 * col + 2];
}
/* P * F^T * volume as written out at constitutive_models.cuh:63-71 */
static void p_ft_vol(const float* P, const float* F, float volume, float* PF) {
	for(int c = 0; c < 3; ++c)
		for(int r = 0; r < 3; ++r) PF[r + 3 * c] = (P[r] * F[c] + P[r + 3] * F[c + 3] + P[r + 6] * F[c + 6]) * volume;
}

/* ------------------------------------------------------------------------------------------ */
/* constitutive models                                                                         */
/* ------------------------------------------------------------------------------------------ */
/* ref: Projects/GMPM/constitutive_models.cuh:36-73 */
static void stress_fixed_corotated(float volume, float mu, float lambda, const float* F, float* PF) {
	float U[9], S[3], V[9];
	orc_svd3(F, U, S, V);
	const float J = S[0] * S[1] * S[2];
	const float scaled_mu = 2.0f * mu;
	const float scaled_lambda = lambda * (J - 1.0f);
	float Ph[3];
	Ph[0] = scaled_mu * (S[0] - 1.f) + scaled_lambda * (S[1] * S[2]);
	Ph[1] = scaled_mu * (S[1] - 1.f) + scaled_lambda * (S[0] * S[2]);
	Ph[2] = scaled_mu * (S[2] - 1.f) + scaled_lambda * (S[0] * S[1]);
	float P[9];
	for(int c = 0; c < 3; ++c)
		for(int r = 0; r < 3; ++r) P[r + 3 * c] = Ph[0] * U[r] * V[c] + Ph[1] * U[r + 3] * V[c + 3] + Ph[2] * U[r + 6] * V[c + 6];
	p_ft_vol(P, F, volume, PF);
}

/* ref: Projects/GMPM/constitutive_models.cuh:239-335 */
static void stress_sand(const orc_particle_buffer* pb, float* F, float* PF, float* log_jp_io) {
	const float mu = pb->mu, lambda = pb->lambda, volume = pb->volume;
	float U[9], S[3], V[9];
	orc_svd3(F, U, S, V);
	const float scaled_mu = 2.0f * mu;
	float eps[3], newS[3] = {0.f, 0.f, 0.f}, newF[9];
	float log_jp = *log_jp_io;
	for(int i = 0; i < 3; ++i) {
		float a = S[i] > 0 ? S[i] : -S[i];
		a = a > 1e-4f ? a : 1e-4f;
		eps[i] = logf(a) - pb->cohesion;
	}
	const float sum_eps = eps[0] + eps[1] + eps[2];
	const float trace_eps = sum_eps + log_jp;
	float eh[3];
	for(int i = 0; i < 3; ++i) eh[i] = eps[i] - (trace_eps / 3.0f);
	const float eh_norm = sqrtf(eh[0] * eh[0] + eh[1] * eh[1] + eh[2] * eh[2]);

	if(trace_eps >= 0.0f) { /* case II: cone tip */
		newS[0] = newS[1] = newS[2] = expf(pb->cohesion);
		mat_diag_mat_t(newF, U, newS, V);
		memcpy(F, newF, sizeof(newF));
		if(pb->volume_correction) log_jp = pb->beta * sum_eps + log_jp;
	} else if(mu != 0) {
		log_jp = 0;
		const float delta_gamma = eh_norm + (3.0f * lambda + scaled_mu) / scaled_mu * trace_eps * pb->yield_surface;
		float H[3];
		if(delta_gamma <= 0) { /* case I */
			for(int i = 0; i < 3; ++i) H[i] = eps[i] + pb->cohesion;
		} else { /* case III */
			for(int i = 0; i < 3; ++i) H[i] = eps[i] - (delta_gamma / eh_norm) * eh[i] + pb->cohesion;
		}
		for(int i = 0; i < 3; ++i) newS[i] = expf(H[i]);
		mat_diag_mat_t(newF, U, newS, V);
		memcpy(F, newF, sizeof(newF));
	}
	const float ls[3] = {logf(newS[0]), logf(newS[1]), logf(newS[2])};
	const float tr = ls[0] + ls[1] + ls[2];
	float Ph[3];
	for(int i = 0; i < 3; ++i) Ph[i] = (scaled_mu * ls[i] + lambda * tr) / newS[i];
	float P[9];
	mat_diag_mat_t(P, U, Ph, V);
	p_ft_vol(P, F, volume, PF);
	*log_jp_io = log_jp;
}

/* ref: Projects/GMPM/constitutive_models.cuh:78-234 (USE_JOSH_FRACTURE_PAPER == 1) */
static void stress_nacc(const orc_particle_buffer* pb, float* F, float* PF, float* log_jp_io) {
	const float mu = pb->mu, volume = pb->volume, bm = pb->bm, beta = pb->beta, msqr = pb->msqr;
	float log_jp = *log_jp_io;
	float U[9], S[3], V[9];
	orc_svd3(F, U, S, V);
	const float p0 = bm * (0.00001f + sinhf(pb->xi * (-log_jp > 0 ? -log_jp : 0)));
	const float p_min = -beta * p0;
	const float Je_trial = S[0] * S[1] * S[2];
	const float Bh[3] = {S[0] * S[0], S[1] * S[1], S[2] * S[2]};
	const float trB3 = (Bh[0] + Bh[1] + Bh[2]) / 3.f;
	const float Jm = mu * powf(Je_trial, -2.f / 3.f);
	const float sh[3] = {Jm * (Bh[0] - trB3), Jm * (Bh[1] - trB3), Jm * (Bh[2] - trB3)};
	const float psi_kappa = bm * 0.5f * (Je_trial - 1.f / Je_trial);
	const float p_trial = -psi_kappa * Je_trial;
	const float ys_coeff = 3.f / 2.f * (1 + 2.f * beta);
	const float y_p_half = msqr * (p_trial - p_min) * (p_trial - p0);
	const float s_sq = sh[0] * sh[0] + sh[1] * sh[1] + sh[2] * sh[2];
	const float y = ys_coeff * s_sq + y_p_half;
	float newF[9];

	if(p_trial > p0) {
		const float Je_new = sqrtf(-2.f * p0 / bm + 1.f);
		S[0] = S[1] = S[2] = powf(Je_new, 1.f / 3.f);
		mat_diag_mat_t(newF, U, S, V);
		memcpy(F, newF, sizeof(newF));
		if(pb->hardening_on) log_jp += logf(Je_trial / Je_new);
	} else if(p_trial < p_min) {
		const float Je_new = sqrtf(-2.f * p_min / bm + 1.f);
		S[0] = S[1] = S[2] = powf(Je_new, 1.f / 3.f);
		mat_diag_mat_t(newF, U, S, V);
		memcpy(F, newF, sizeof(newF));
		if(pb->hardening_on) log_jp += logf(Je_trial / Je_new);
	} else if(y >= 1e-4) {
		const float Bs = powf(Je_trial, 2.f / 3.f) / mu * sqrtf(-y_p_half / ys_coeff) / sqrtf(s_sq);
		for(int i = 0; i < 3; ++i) S[i] = sqrtf(sh[i] * Bs + trB3);
		mat_diag_mat_t(newF, U, S, V);
		memcpy(F, newF, sizeof(newF));
		if(pb->hardening_on && p0 > 1e-4 && p_trial < p0 - 1e-4 && p_trial > 1e-4 + p_min) {
			const float p_center = (1.0f - beta) * p0 / 2;
			const float q_trial = sqrtf(3.f / 2.f * s_sq);
			float dir[2] = {p_center - p_trial, -q_trial};
			const float dn = sqrtf(dir[0] * dir[0] + dir[1] * dir[1]);
			dir[0] /= dn;
			dir[1] /= dn;
			const float C = msqr * (p_center - p_min) * (p_center - p0);
			const float B = msqr * dir[0] * (2 * p_center - p0 - p_min);
			const float A = msqr * dir[0] * dir[0] + (1 + 2 * beta) * dir[1] * dir[1];
			const float l1 = (-B + sqrtf(B * B - 4 * A * C)) / (2 * A);
			const float l2 = (-B - sqrtf(B * B - 4 * A * C)) / (2 * A);
			const float p1 = p_center + l1 * dir[0];
			const float p2 = p_center + l2 * dir[0];
			const float p_fake = (p_trial - p_center) * (p1 - p_center) > 0 ? p1 : p2;
			const float tJ = (-2 * p_fake / bm + 1);
			const float Je_fake = sqrtf(tJ > 0 ? tJ : -tJ);
			if(Je_fake > 1e-4) log_jp += logf(Je_trial / Je_fake);
		}
	}
	const float J = S[0] * S[1] * S[2];
	/* b = F F^T (MatrixUtils.h:257-269), deviator (MatrixUtils.h:272-286) */
	float b[9], bd[9];
	for(int c = 0; c < 3; ++c)
		for(int r = 0; r < 3; ++r) b[r + 3 * c] = F[r] * F[c] + F[r + 3] * F[c + 3] + F[r + 6] * F[c + 6];
	memcpy(bd, b, sizeof(b));
	bd[0] = b[0] * (float) (2.0 / 3.0) - (b[4] + b[8]) / 3.0f;
	bd[4] = b[4] * (float) (2.0 / 3.0) - (b[0] + b[8]) / 3.0f;
	bd[8] = b[8] * (float) (2.0 / 3.0) - (b[0] + b[4]) / 3.0f;
	const float dev_c = mu * powf(J, -2.f / 3.f);
	const float i_c = bm * .5f * ((J * J - 1.f) * 0.5f - logf(J));
	for(int i = 0; i < 9; ++i) PF[i] = (dev_c * bd[i] + ((i % 4 == 0) ? i_c : 0.f)) * volume;
	*log_jp_io = log_jp;
}

void orc_compute_stress(int material, const orc_particle_buffer* pb, float* F, float* PF, float* log_jp) {
	switch(material) {
		case ORC_FIXED_COROTATED: stress_fixed_corotated(pb->volume, pb->mu, pb->lambda, F, PF); break;
		case ORC_SAND: stress_sand(pb, F, PF, log_jp); break;
		case ORC_NACC: stress_nacc(pb, F, PF, log_jp); break;
		default: memset(PF, 0, 9 * sizeof(float)); break;
	}
}

/* ------------------------------------------------------------------------------------------ */
/* init-only kernels                                                                           */
/* ------------------------------------------------------------------------------------------ */
/* ref: Projects/GMPM/mgmpm_kernels.cuh:21-34 */
void orc_activate_blocks(const orc_config* cfg, int n, const float* pos, orc_partition part) {
	for(int p = 0; p < n; ++p) {
		int b[3];
		for(int d = 0; d < 3; ++d) b[d] = (cell_of(cfg, pos[3 * p + d]) - 2) / 4;
		part_insert(cfg, &part, b[0], b[1], b[2]);
	}
}

/* ref: Projects/GMPM/mgmpm_kernels.cuh:36-68 */
void orc_build_particle_cell_buckets(const orc_config* cfg, int n, const float* pos, orc_particle_buffer pb, orc_partition part) {
	for(int p = 0; p < n; ++p) {
		int c[3];
		for(int d = 0; d < 3; ++d) c[d] = cell_of(cfg, pos[3 * p + d]) - 2;
		const int blockno = part_query(cfg, &part, c[0] / 4, c[1] / 4, c[2] / 4);
		const int cellno = (c[0] & 3) * 16 + (c[1] & 3) * 4 + (c[2] & 3);
		int* cnt = &pb.cell_particle_counts[(long) blockno * BLOCK_VOL + cellno];
		const int slot = (*cnt)++;
		if(slot >= cfg->max_ppc) {
			(*cnt)--;
			continue;
		}
		pb.cellbuckets[(long) blockno * cfg_ppb(cfg) + cellno * cfg->max_ppc + slot] = p;
	}
}

/* ref: Projects/GMPM/mgmpm_kernels.cuh:70-84 -- pass i takes slot i of every cell that has one; cells ascend
 * (warp-aggregated increment hands out ranks in lane order; the two warps of the CUDA block race, the
 * restatement takes warp 0 then warp 1). */
void orc_cell_bucket_to_block(const orc_config* cfg, int block_count, const int* cell_particle_counts, const int* cellbuckets, int* particle_bucket_sizes, int* buckets) {
	const int ppb = cfg_ppb(cfg);
#pragma omp parallel for num_threads(g_threads) schedule(static)
	for(int b = 0; b < block_count; ++b) {
		int size = particle_bucket_sizes[b];
		for(int i = 0; i < cfg->max_ppc; ++i)
			for(int c = 0; c < BLOCK_VOL; ++c)
				if(i < cell_particle_counts[(long) b * BLOCK_VOL + c]) buckets[(long) b * ppb + size++] = cellbuckets[(long) b * ppb + c * cfg->max_ppc + i];
		particle_bucket_sizes[b] = size;
	}
}

/* ref: Projects/GMPM/mgmpm_kernels.cuh:86-94 */
void orc_compute_bin_capacity(int block_count, const int* particle_bucket_sizes, int* bin_sizes) {
	for(int b = 0; b < block_count; ++b) bin_sizes[b] = (particle_bucket_sizes[b] + BIN_CAP - 1) / BIN_CAP;
}

/* thrust::exclusive_scan, ref: Projects/GMPM/gmpm_simulator.cuh:257-260 */
void orc_exclusive_scan(int count, const int* in, int* out) {
	int acc = 0;
	for(int i = 0; i < count; ++i) {
		const int v = in[i];
		out[i] = acc;
		acc += v;
	}
}

/* ref: Library/MnBase/Algorithm/MappingKernels.cuh:44-55 */
void orc_exclusive_scan_inverse(int num, const int* map, int* map_inv) {
	for(int i = 0; i < num; ++i)
		if(map[i] != map[i + 1]) map_inv[map[i]] = i;
}

/* ref: Projects/GMPM/mgmpm_kernels.cuh:221-323 (one overload per material) */
void orc_array_to_buffer(const orc_config* cfg, int block_count, const float* pos, orc_particle_buffer pb) {
	const int bf = bin_floats(pb.material);
	for(int b = 0; b < block_count; ++b) {
		const int n = pb.particle_bucket_sizes[b];
		const int* bucket = pb.blockbuckets + (long) b * cfg_ppb(cfg);
		for(int i = 0; i < n; ++i) {
			const int pid = bucket[i];
			float* bin = pb.bins + (long) (pb.bin_offsets[b] + i / BIN_CAP) * bf;
			const int l = i % BIN_CAP;
			bin[0 * 32 + l] = pos[3 * pid + 0];
			bin[1 * 32 + l] = pos[3 * pid + 1];
			bin[2 * 32 + l] = pos[3 * pid + 2];
			if(pb.material == ORC_J_FLUID) {
				bin[3 * 32 + l] = 1.0f;
			} else {
				for(int d = 0; d < 9; ++d) bin[(3 + d) * 32 + l] = (d % 4 == 0) ? 1.f : 0.f;
				if(pb.material == ORC_SAND) bin[12 * 32 + l] = 0.0f;   /* LOG_JP_0, particle_buffer.cuh:207 */
				if(pb.material == ORC_NACC) bin[12 * 32 + l] = -0.01f; /* LOG_JP_0, particle_buffer.cuh:241 */
			}
		}
	}
}

/* ref: Projects/GMPM/mgmpm_kernels.cuh:153-219 */
void orc_rasterize(const orc_config* cfg, int n, const float* pos, float* grid, orc_partition part, float mass, const float* v0) {
	const float dx = cfg_dx(cfg);
	for(int p = 0; p < n; ++p) {
		int base[3];
		float lp[3], w[3][3];
		for(int d = 0; d < 3; ++d) {
			base[d] = cell_of(cfg, pos[3 * p + d]) - 1;
			lp[d] = pos[3 * p + d] - base[d] * dx;
			orc_bspline_weight(cfg, lp[d], w[d]);
		}
		for(int i = 0; i < 3; ++i)
			for(int j = 0; j < 3; ++j)
				for(int k = 0; k < 3; ++k) {
					const int g[3] = {base[0] + i, base[1] + j, base[2] + k};
					const float W = w[0][i] * w[1][j] * w[2][k];
					const float wm = mass * W;
					const int blockno = part_query(cfg, &part, g[0] >> 2, g[1] >> 2, g[2] >> 2);
					if(blockno < 0) continue; /* node beyond the top face: no block (the reference indexes out of bounds) */
					float* blk = grid + (long) blockno * 256;
					const int c = (g[0] & 3) * 16 + (g[1] & 3) * 4 + (g[2] & 3);
					blk[c] += wm;
					blk[64 + c] += wm * v0[0];
					blk[128 + c] += wm * v0[1];
					blk[192 + c] += wm * v0[2];
				}
	}
}

/* ref: Projects/GMPM/mgmpm_kernels.cuh:96-104 */
void orc_init_adv_bucket(const orc_config* cfg, int block_count, const int* particle_bucket_sizes, int* buckets) {
	for(int b = 0; b < block_count; ++b)
		for(int i = 0; i < particle_bucket_sizes[b]; ++i) buckets[(long) b * cfg_ppb(cfg) + i] = (13 * cfg_ppb(cfg)) | i;
}

/* ------------------------------------------------------------------------------------------ */
/* per-step kernels                                                                            */
/* ------------------------------------------------------------------------------------------ */
/* ref: Projects/GMPM/mgmpm_kernels.cuh:106-115 */
void orc_clear_grid(int block_count, float* grid) { memset(grid, 0, (size_t) block_count * 1024); }

/* ref: Projects/GMPM/hash_table.cuh:110-112 */
void orc_reset_table(const orc_config* cfg, orc_partition part) {
	const long g = cfg_gsize(cfg);
	memset(part.index_table, 0xff, sizeof(int) * g * g * g);
}

/* ref: Projects/GMPM/mgmpm_kernels.cuh:117-133 */
void orc_register_neighbor_blocks(const orc_config* cfg, int block_count, orc_partition part) {
	for(int b = 0; b < block_count; ++b) {
		const int* k = part.active_keys + 3 * b;
		const int kx = k[0], ky = k[1], kz = k[2];
		for(int i = 0; i < 2; ++i)
			for(int j = 0; j < 2; ++j)
				for(int l = 0; l < 2; ++l) part_insert(cfg, &part, kx + i, ky + j, kz + l);
	}
}

/* ref: Projects/GMPM/mgmpm_kernels.cuh:135-151 */
void orc_register_exterior_blocks(const orc_config* cfg, int block_count, orc_partition part) {
	for(int b = 0; b < block_count; ++b) {
		const int* k = part.active_keys + 3 * b;
		const int kx = k[0], ky = k[1], kz = k[2];
		for(int i = -1; i < 2; ++i)
			for(int j = -1; j < 2; ++j)
				for(int l = -1; l < 2; ++l) part_insert(cfg, &part, kx + i, ky + j, kz + l);
	}
}

/* A node holds mass only when its mass is a normal float: the reference is built with --use_fast_math, which
 * flushes subnormal results to zero.  A subnormal mass (a stencil's far corner, weights of order 2^-39 per axis, of a
 * particle one ulp from a cell's half below x = 0.5) would make 1 / m inf and the node's velocity 0 * inf = NaN. */
static inline int node_has_mass(float m) { return m >= FLT_MIN; }

/* ref: Projects/GMPM/mgmpm_kernels.cuh:325-420.  Quirk kept: wall-zeroed y velocity still receives
 * gravity (SURVEY.md Appendix B #1); NaN -> +inf (B #3).  The one body of every grid update: `resolve` (NULL: none) is the
 * boundaries' hook, run on each node with mass after gravity and before |v|^2 (the collider oracle's, collider_oracle.c). */
typedef void (*orc_node_resolve)(const void* ctx, const int* node, float* v);
static void boundaries_update(const orc_config* cfg, int block_count, float* grid, orc_partition part, float dt, orc_node_resolve resolve, const void* ctx,
                              float* max_vel) {
	const int g = cfg_gsize(cfg), bc = cfg->boundary;
	float mx = *max_vel;
#pragma omp parallel for num_threads(g_threads) schedule(static) reduction(max : mx)
	for(int b = 0; b < block_count; ++b) {
		const int* k = part.active_keys + 3 * b;
		const int ob = ((k[0] < bc || k[0] >= g - bc) << 2) | ((k[1] < bc || k[1] >= g - bc) << 1) | (k[2] < bc || k[2] >= g - bc);
		float* blk = grid + (long) b * 256;
		for(int c = 0; c < BLOCK_VOL; ++c) {
			const float mass = blk[c];
			float vsq = 0.f;
			if(node_has_mass(mass)) {
				const float mi = 1.f / mass;
				float v[3];
				v[0] = (ob & 4) ? 0.f : blk[64 + c] * mi;
				v[1] = (ob & 2) ? 0.f : blk[128 + c] * mi;
				v[1] += cfg->gravity * dt;
				v[2] = (ob & 1) ? 0.f : blk[192 + c] * mi;
				if(resolve) {
					const int node[3] = {4 * k[0] + ((c & 0x30) >> 4), 4 * k[1] + ((c & 0xc) >> 2), 4 * k[2] + (c & 0x3)};
					resolve(ctx, node, v);
				}
				blk[64 + c] = v[0];
				blk[128 + c] = v[1];
				blk[192 + c] = v[2];
				vsq += v[0] * v[0];
				vsq += v[1] * v[1];
				vsq += v[2] * v[2];
			}
			if(isnan(vsq)) vsq = INFINITY;
			if(vsq > mx) mx = vsq;
		}
	}
	*max_vel = mx;
}

void orc_update_grid_velocity_query_max(const orc_config* cfg, int block_count, float* grid, orc_partition part, float dt, float* max_vel) {
	boundaries_update(cfg, block_count, grid, part, dt, NULL, NULL, max_vel);
}

static inline void dir_components(int dir, int* d) {
	d[2] = (dir % 3) - 1;
	d[1] = ((dir / 3) % 3) - 1;
	d[0] = ((dir / 9) % 3) - 1;
}

/* arena index (x,y,z in [0,8)) -> flat, ref: mgmpm_kernels.cuh:676-684 */
#define AR(x, y, z) (((x) * 8 + (y)) * 8 + (z))

/* ref: Projects/GMPM/mgmpm_kernels.cuh:665-937 with fetch (:428-462), calculate_contribution_and_store
 * (:470-663) and ParticleBufferImpl::add_advection (particle_buffer.cuh:100-135). */
void orc_g2p2g(const orc_config* cfg, float dt, float new_dt, int block_count, orc_particle_buffer cur, orc_particle_buffer next, orc_partition prev_part, orc_partition part, const float* grid, float* next_grid) {
	const float dx = cfg_dx(cfg), dinv = cfg_dinv(cfg);
	const int ppb = cfg_ppb(cfg);
	const int bf = bin_floats(cur.material);
	const int mat = cur.material;
#pragma omp parallel for num_threads(g_threads) schedule(dynamic, 4)
	for(int src_blockno = 0; src_blockno < block_count; ++src_blockno) {
		const int* bk = part.active_keys + 3 * src_blockno;
		const int bucket_size = next.particle_bucket_sizes[src_blockno];
		if(bucket_size == 0) continue;
		float g2p[3][512];
		float p2g[4][512];
		memset(p2g, 0, sizeof(p2g));
		for(int lb = 0; lb < 8; ++lb) {
			const int bno = part_query(cfg, &part, bk[0] + ((lb & 4) ? 1 : 0), bk[1] + ((lb & 2) ? 1 : 0), bk[2] + ((lb & 1) ? 1 : 0));
			const float* blk = grid + (long) bno * 256;
			for(int c = 0; c < 64; ++c) {
				const int x = (c >> 4) + ((lb & 4) ? 4 : 0), y = ((c >> 2) & 3) + ((lb & 2) ? 4 : 0), z = (c & 3) + ((lb & 1) ? 4 : 0);
				for(int ch = 0; ch < 3; ++ch) g2p[ch][AR(x, y, z)] = bno >= 0 ? blk[64 * (ch + 1) + c] : 0.f;
			}
		}
		for(int pidib = 0; pidib < bucket_size; ++pidib) {
			const int advect = next.blockbuckets[(long) src_blockno * ppb + pidib];
			int off[3];
			dir_components(advect / ppb, off);
			const int source_pidib = advect & (ppb - 1);
			const int src_no = part_query(cfg, &prev_part, bk[0] + off[0], bk[1] + off[1], bk[2] + off[2]);
			const long src_bin = (long) cur.bin_offsets[src_no] + source_pidib / BIN_CAP;
			const float* sbin = cur.bins + src_bin * bf;
			const int sl = source_pidib % BIN_CAP;
			float pos[3] = {sbin[sl], sbin[32 + sl], sbin[64 + sl]};
			float J = (mat == ORC_J_FLUID) ? sbin[96 + sl] : 0.f;

			int base[3], abase[3];
			float lp[3], w[3][3];
			for(int d = 0; d < 3; ++d) {
				base[d] = cell_of(cfg, pos[d]) - 1;
				lp[d] = pos[d] - base[d] * dx;
				orc_bspline_weight(cfg, lp[d], w[d]);
				abase[d] = ((base[d] - 1) & 3) + 1;
			}
			float vel[3] = {0.f, 0.f, 0.f}, A[9] = {0.f};
			for(int i = 0; i < 3; ++i)
				for(int j = 0; j < 3; ++j)
					for(int k = 0; k < 3; ++k) {
						const float xixp[3] = {i * dx - lp[0], j * dx - lp[1], k * dx - lp[2]};
						const float W = w[0][i] * w[1][j] * w[2][k];
						const int a = AR(abase[0] + i, abase[1] + j, abase[2] + k);
						const float vi[3] = {g2p[0][a], g2p[1][a], g2p[2][a]};
						for(int c = 0; c < 3; ++c) vel[c] += W * vi[c];
						for(int d = 0; d < 3; ++d)
							for(int c = 0; c < 3; ++c) A[c + 3 * d] += W * vi[c] * xixp[d];
					}
			for(int d = 0; d < 3; ++d) pos[d] += vel[d] * dt;

			float contrib[9];
			float* dbin = next.bins + ((long) next.bin_offsets[src_blockno] + pidib / BIN_CAP) * bf;
			const int dl = pidib % BIN_CAP;
			if(mat == ORC_J_FLUID) { /* mgmpm_kernels.cuh:474-516 */
				J += (A[0] + A[4] + A[8]) * dt * dinv * J;
				if(J < 0.1) J = 0.1;
				const float voln = J * cur.volume;
				const float pressure = cur.bulk * (powf(J, -cur.gamma) - 1.f);
				contrib[0] = ((A[0] + A[0]) * dinv * cur.viscosity - pressure) * voln;
				contrib[1] = (A[1] + A[3]) * dinv * cur.viscosity * voln;
				contrib[2] = (A[2] + A[6]) * dinv * cur.viscosity * voln;
				contrib[3] = (A[3] + A[1]) * dinv * cur.viscosity * voln;
				contrib[4] = ((A[4] + A[4]) * dinv * cur.viscosity - pressure) * voln;
				contrib[5] = (A[5] + A[7]) * dinv * cur.viscosity * voln;
				contrib[6] = (A[6] + A[2]) * dinv * cur.viscosity * voln;
				contrib[7] = (A[7] + A[5]) * dinv * cur.viscosity * voln;
				contrib[8] = ((A[8] + A[8]) * dinv * cur.viscosity - pressure) * voln;
				dbin[dl] = pos[0];
				dbin[32 + dl] = pos[1];
				dbin[64 + dl] = pos[2];
				dbin[96 + dl] = J;
			} else { /* mgmpm_kernels.cuh:518-663 */
				float dws[9], Fold[9], F[9];
				for(int d = 0; d < 9; ++d) dws[d] = A[d] * dt * dinv + ((d & 3) != 0 ? 0.f : 1.f);
				for(int d = 0; d < 9; ++d) Fold[d] = sbin[(3 + d) * 32 + sl];
				float log_jp = (mat == ORC_SAND || mat == ORC_NACC) ? sbin[12 * 32 + sl] : 0.f;
				mat_mul(dws, Fold, F);
				if(mat == ORC_FIXED_COROTATED) {
					/* trial F is stored before the stress (SURVEY.md Appendix B #7) */
					for(int d = 0; d < 9; ++d) dbin[(3 + d) * 32 + dl] = F[d];
					orc_compute_stress(mat, &cur, F, contrib, &log_jp);
				} else {
					orc_compute_stress(mat, &cur, F, contrib, &log_jp);
					for(int d = 0; d < 9; ++d) dbin[(3 + d) * 32 + dl] = F[d];
					dbin[12 * 32 + dl] = log_jp;
				}
				dbin[dl] = pos[0];
				dbin[32 + dl] = pos[1];
				dbin[64 + dl] = pos[2];
			}
			for(int d = 0; d < 9; ++d) contrib[d] = (A[d] * cur.mass - contrib[d] * new_dt) * dinv;

			int nbase[3];
			for(int d = 0; d < 3; ++d) {
				nbase[d] = cell_of(cfg, pos[d]) - 1;
				lp[d] = pos[d] - nbase[d] * dx;
			}
			{ /* add_advection, particle_buffer.cuh:100-135 */
				int dv[3], cell[3];
				for(int d = 0; d < 3; ++d) {
					dv[d] = (base[d] - 1) / 4 - (nbase[d] - 1) / 4;
					cell[d] = nbase[d] - 1;
				}
				const int dirtag = (dv[0] + 1) * 9 + (dv[1] + 1) * 3 + dv[2] + 1;
				const int bno = part_query(cfg, &part, cell[0] / 4, cell[1] / 4, cell[2] / 4);
				if(bno != -1) {
					const int cellno = ((cell[0] & 3) << 4) | ((cell[1] & 3) << 2) | (cell[2] & 3);
					int* cnt = &next.cell_particle_counts[(long) bno * BLOCK_VOL + cellno];
					int slot;
#pragma omp atomic capture
					slot = (*cnt)++;
					if(slot >= cfg->max_ppc) {
#pragma omp atomic
						(*cnt)--;
					} else {
						next.cellbuckets[(long) bno * ppb + cellno * cfg->max_ppc + slot] = (dirtag * ppb) | pidib;
					}
				}
			}
			int oob = 0;
			for(int d = 0; d < 3; ++d) {
				orc_bspline_weight(cfg, lp[d], w[d]);
				abase[d] = (((base[d] - 1) & 3) + 1) + (nbase[d] - base[d]);
				if(abase[d] < 0 || abase[d] + 2 >= 8) oob = 1;
			}
			if(oob) continue; /* SURVEY.md Appendix B #4: contribution dropped */
			for(int i = 0; i < 3; ++i)
				for(int j = 0; j < 3; ++j)
					for(int k = 0; k < 3; ++k) {
						const float xp[3] = {i * dx - lp[0], j * dx - lp[1], k * dx - lp[2]};
						const float W = w[0][i] * w[1][j] * w[2][k];
						const float wm = cur.mass * W;
						const int a = AR(abase[0] + i, abase[1] + j, abase[2] + k);
						p2g[0][a] += wm;
						p2g[1][a] += wm * vel[0] + (contrib[0] * xp[0] + contrib[3] * xp[1] + contrib[6] * xp[2]) * W;
						p2g[2][a] += wm * vel[1] + (contrib[1] * xp[0] + contrib[4] * xp[1] + contrib[7] * xp[2]) * W;
						p2g[3][a] += wm * vel[2] + (contrib[2] * xp[0] + contrib[5] * xp[1] + contrib[8] * xp[2]) * W;
					}
		}
		/* arena -> next grid, ref: mgmpm_kernels.cuh:910-936 */
		for(int lb = 0; lb < 8; ++lb) {
			const int bno = part_query(cfg, &part, bk[0] + ((lb & 4) ? 1 : 0), bk[1] + ((lb & 2) ? 1 : 0), bk[2] + ((lb & 1) ? 1 : 0));
			if(bno < 0) continue;
			float* blk = next_grid + (long) bno * 256;
			for(int ch = 0; ch < 4; ++ch)
				for(int c = 0; c < 64; ++c) {
					const int x = (c >> 4) + ((lb & 4) ? 4 : 0), y = ((c >> 2) & 3) + ((lb & 2) ? 4 : 0), z = (c & 3) + ((lb & 1) ? 4 : 0);
					const float v = p2g[ch][AR(x, y, z)];
#pragma omp atomic
					blk[64 * ch + c] += v;
				}
		}
	}
}

/* ref: Projects/GMPM/mgmpm_kernels.cuh:939-952 */
void orc_mark_active_grid_blocks(int block_count, const float* grid, int* marks) {
	for(int b = 0; b < block_count; ++b)
		for(int c = 0; c < BLOCK_VOL; ++c)
			if(grid[(long) b * 256 + c] != 0.0f) {
				marks[b] = 1;
				break;
			}
}

/* ref: Projects/GMPM/mgmpm_kernels.cuh:954-964 */
void orc_mark_active_particle_blocks(int block_count, const int* particle_bucket_sizes, int* marks) {
	for(int b = 0; b < block_count; ++b)
		if(particle_bucket_sizes[b] > 0) marks[b] = 1;
}

/* ref: Projects/GMPM/mgmpm_kernels.cuh:966-977 */
void orc_update_partition(const orc_config* cfg, int block_count, const int* source_nos, orc_partition part, orc_partition next_part) {
	for(int b = 0; b < block_count; ++b) {
		const int* k = part.active_keys + 3 * source_nos[b];
		next_part.active_keys[3 * b + 0] = k[0];
		next_part.active_keys[3 * b + 1] = k[1];
		next_part.active_keys[3 * b + 2] = k[2];
		next_part.index_table[tbl(cfg, k[0], k[1], k[2])] = b;
	}
}

/* ref: Projects/GMPM/mgmpm_kernels.cuh:979-1000 */
void orc_update_buckets(const orc_config* cfg, int block_count, const int* source_nos, orc_particle_buffer pb, orc_particle_buffer next_pb) {
	const int ppb = cfg_ppb(cfg);
	for(int b = 0; b < block_count; ++b) {
		const int s = source_nos[b];
		const int n = pb.particle_bucket_sizes[s];
		next_pb.particle_bucket_sizes[b] = n;
		memcpy(next_pb.blockbuckets + (long) b * ppb, pb.blockbuckets + (long) s * ppb, sizeof(int) * n);
	}
}

/* ref: Projects/GMPM/mgmpm_kernels.cuh:1002-1020 */
void orc_copy_selected_grid_blocks(const orc_config* cfg, int prev_block_count, const int* prev_blockids, orc_partition part, const int* marks, const float* prev_grid, float* grid) {
	for(int b = 0; b < prev_block_count; ++b) {
		if(!marks[b]) continue;
		const int* k = prev_blockids + 3 * b;
		const int bno = part_query(cfg, &part, k[0], k[1], k[2]);
		if(bno == -1) continue;
		memcpy(grid + (long) bno * 256, prev_grid + (long) b * 256, 1024);
	}
}

/* ref: Projects/GMPM/mgmpm_kernels.cuh:1087-1122 */
int orc_retrieve_particle_buffer(const orc_config* cfg, int block_count, orc_partition part, orc_partition prev_part, orc_particle_buffer pb, orc_particle_buffer next_pb, float* out_pos) {
	const int ppb = cfg_ppb(cfg), bf = bin_floats(pb.material);
	int n = 0;
	for(int b = 0; b < block_count; ++b) {
		const int cnt = next_pb.particle_bucket_sizes[b];
		const int* k = part.active_keys + 3 * b;
		for(int i = 0; i < cnt; ++i) {
			const int advect = next_pb.blockbuckets[(long) b * ppb + i];
			int off[3];
			dir_components(advect / ppb, off);
			const int sp = advect % ppb;
			const int sno = part_query(cfg, &prev_part, k[0] + off[0], k[1] + off[1], k[2] + off[2]);
			const float* bin = pb.bins + ((long) pb.bin_offsets[sno] + sp / BIN_CAP) * bf;
			out_pos[3 * n + 0] = bin[sp % BIN_CAP];
			out_pos[3 * n + 1] = bin[32 + sp % BIN_CAP];
			out_pos[3 * n + 2] = bin[64 + sp % BIN_CAP];
			++n;
		}
	}
	return n;
}

/* ------------------------------------------------------------------------------------------ */
/* MGSP halo protocol, ref: Projects/MGSP/halo_kernels.cuh                                     */
/* ------------------------------------------------------------------------------------------ */
/* :22-35 */
void orc_mark_overlapping_blocks(const orc_config* cfg, int block_count, int otherdid, const int* incoming, orc_partition part, int* count, int* out_blockids) {
	for(int i = 0; i < block_count; ++i) {
		const int* k = incoming + 3 * i;
		const int bno = part_query(cfg, &part, k[0], k[1], k[2]);
		if(bno >= 0) {
			part.overlap_marks[bno] |= 1 << otherdid;
			const int h = (*count)++;
			out_blockids[3 * h + 0] = k[0];
			out_blockids[3 * h + 1] = k[1];
			out_blockids[3 * h + 2] = k[2];
		}
	}
}
/* :38-62 */
void orc_collect_blockids_for_halo_reduction(const orc_config* cfg, int particle_block_count, orc_partition part) {
	for(int b = 0; b < particle_block_count; ++b) {
		const int* k = part.active_keys + 3 * b;
		part.halo_marks[b] = 0;
		int hit = 0;
		for(int i = 0; i < 2 && !hit; ++i)
			for(int j = 0; j < 2 && !hit; ++j)
				for(int l = 0; l < 2 && !hit; ++l) {
					const int nno = part_query(cfg, &part, k[0] + i, k[1] + j, k[2] + l);
					if(nno >= 0 && part.overlap_marks[nno]) hit = 1;
				}
		if(hit) {
			part.halo_marks[b] = 1;
			const int h = (*part.halo_count)++;
			part.halo_blocks[3 * h + 0] = k[0];
			part.halo_blocks[3 * h + 1] = k[1];
			part.halo_blocks[3 * h + 2] = k[2];
		}
	}
}
/* :65-80 */
void orc_collect_grid_blocks(const orc_config* cfg, int count, const int* blockids, const float* grid, orc_partition part, float* halo_grid) {
	for(int h = 0; h < count; ++h) {
		const int* k = blockids + 3 * h;
		const int bno = part_query(cfg, &part, k[0], k[1], k[2]);
		memcpy(halo_grid + (long) h * 256, grid + (long) bno * 256, 1024);
	}
}
/* :83-97 */
void orc_reduce_grid_blocks(const orc_config* cfg, int count, const int* blockids, float* grid, orc_partition part, const float* halo_grid) {
	for(int h = 0; h < count; ++h) {
		const int* k = blockids + 3 * h;
		const int bno = part_query(cfg, &part, k[0], k[1], k[2]);
		for(int i = 0; i < 256; ++i) grid[(long) bno * 256 + i] += halo_grid[(long) h * 256 + i];
	}
}

/* ------------------------------------------------------------------------------------------ */
/* GmpmSimulator restated (host driver), ref: Projects/GMPM/gmpm_simulator.cuh                 */
/* ------------------------------------------------------------------------------------------ */
#define ORC_MAX_MODELS 8
struct orc_sim {
	orc_config cfg;
	int max_blocks;
	float dt_default, dt, next_dt, max_vel;
	int rollid;
	int nmodels;
	orc_particle_buffer bins[2][ORC_MAX_MODELS];
	long bin_capacity[ORC_MAX_MODELS];
	float* init_pos[ORC_MAX_MODELS];
	int count[ORC_MAX_MODELS];
	float v0[ORC_MAX_MODELS][3];
	orc_partition parts[2];
	float* grids[2];
	int pbc, nbc, ebc;
	int *marks, *destinations, *sources, *bin_sizes;
};

static void default_buffer(const orc_config* cfg, int material, orc_particle_buffer* pb) {
	/* ref: Projects/GMPM/particle_buffer.cuh:141-264 defaults */
	memset(pb, 0, sizeof(*pb));
	const float cells = (float) (1u << cfg->domain_bits);
	const float E = 5e3f, nu = 0.4f;
	pb->material = material;
	pb->rho = 1e3f;
	pb->mass = (1e3f / cells / cells / cells / 8.0f);
	pb->volume = ((material == ORC_FIXED_COROTATED || material == ORC_SAND) ? 10.f : 1.f) / cells / cells / cells / 8.0f;
	pb->bulk = 4e4f;
	pb->gamma = 7.15f;
	pb->viscosity = 0.01f;
	pb->lambda = E * nu / ((1 + nu) * (1 - 2 * nu));
	pb->mu = E / (2 * (1 + nu));
	pb->cohesion = 0.f;
	pb->beta = (material == ORC_NACC) ? 0.5f : 1.0f;
	pb->yield_surface = 0.816496580927726f * 2.f * 0.5f / (3.f - 0.5f);
	pb->volume_correction = 1;
	pb->bm = 2.f / 3.f * (E / (2 * (1 + nu))) + (E * nu / ((1 + nu) * (1 - 2 * nu)));
	pb->xi = 0.8f;
	pb->msqr = 3.423772074299613f;
	pb->hardening_on = 1;
}

static void alloc_partition(const orc_config* cfg, orc_partition* p, int max_blocks) {
	const long g = cfg_gsize(cfg);
	p->count = (int*) calloc(1, sizeof(int));
	p->index_table = (int*) malloc(sizeof(int) * g * g * g);
	memset(p->index_table, 0xff, sizeof(int) * g * g * g);
	p->active_keys = (int*) calloc((size_t) max_blocks * 3, sizeof(int));
	p->halo_count = (int*) calloc(1, sizeof(int));
	p->halo_marks = (char*) calloc(max_blocks, 1);
	p->overlap_marks = (int*) calloc(max_blocks, sizeof(int));
	p->halo_blocks = (int*) calloc((size_t) max_blocks * 3, sizeof(int));
}
static void free_partition(orc_partition* p) {
	free(p->count);
	free(p->index_table);
	free(p->active_keys);
	free(p->halo_count);
	free(p->halo_marks);
	free(p->overlap_marks);
	free(p->halo_blocks);
}

orc_sim* orc_sim_create(const orc_config* cfg, float dt_default, int max_blocks) {
	orc_sim* s = (orc_sim*) calloc(1, sizeof(orc_sim));
	s->cfg = *cfg;
	s->max_blocks = max_blocks;
	s->dt_default = dt_default;
	for(int i = 0; i < 2; ++i) {
		alloc_partition(cfg, &s->parts[i], max_blocks);
		s->grids[i] = (float*) calloc((size_t) max_blocks * 256, sizeof(float));
	}
	s->marks = (int*) calloc(max_blocks + 1, sizeof(int));
	s->destinations = (int*) calloc(max_blocks + 2, sizeof(int));
	s->sources = (int*) calloc(max_blocks + 2, sizeof(int));
	s->bin_sizes = (int*) calloc(max_blocks + 2, sizeof(int));
	return s;
}

void orc_sim_destroy(orc_sim* s) {
	if(!s) return;
	for(int i = 0; i < 2; ++i) {
		free_partition(&s->parts[i]);
		free(s->grids[i]);
		for(int m = 0; m < s->nmodels; ++m) {
			orc_particle_buffer* pb = &s->bins[i][m];
			free(pb->bins);
			free(pb->cell_particle_counts);
			free(pb->particle_bucket_sizes);
			free(pb->cellbuckets);
			free(pb->blockbuckets);
			free(pb->bin_offsets);
		}
	}
	for(int m = 0; m < s->nmodels; ++m) free(s->init_pos[m]);
	free(s->marks);
	free(s->destinations);
	free(s->sources);
	free(s->bin_sizes);
	free(s);
}

/* ref: gmpm_simulator.cuh:168-209 (init_model) + particle_buffer.cuh:71-86 (reserve_buckets) */
int orc_sim_init_model(orc_sim* s, int material, const float* pos, int n, const float* v0) {
	const int m = s->nmodels++;
	const int ppb = cfg_ppb(&s->cfg);
	s->bin_capacity[m] = n / BIN_CAP + s->max_blocks;
	for(int i = 0; i < 2; ++i) {
		orc_particle_buffer* pb = &s->bins[i][m];
		default_buffer(&s->cfg, material, pb);
		pb->bins = (float*) calloc((size_t) s->bin_capacity[m] * bin_floats(material), sizeof(float));
		pb->cell_particle_counts = (int*) calloc((size_t) s->max_blocks * BLOCK_VOL, sizeof(int));
		pb->particle_bucket_sizes = (int*) calloc(s->max_blocks + 1, sizeof(int));
		pb->cellbuckets = (int*) calloc((size_t) s->max_blocks * ppb, sizeof(int));
		pb->blockbuckets = (int*) calloc((size_t) s->max_blocks * ppb, sizeof(int));
		pb->bin_offsets = (int*) calloc(s->max_blocks + 1, sizeof(int));
	}
	s->init_pos[m] = (float*) malloc(sizeof(float) * 3 * n);
	memcpy(s->init_pos[m], pos, sizeof(float) * 3 * n);
	s->count[m] = n;
	for(int d = 0; d < 3; ++d) s->v0[m][d] = v0[d];
	return m;
}

/* ref: particle_buffer.cuh:152-159, 178-184, 250-259 (update_parameters) via gmpm_simulator.cuh:211-254 */
void orc_sim_update_fr_parameters(orc_sim* s, int model, float rho, float vol, float ym, float pr) {
	for(int i = 0; i < 2; ++i) {
		orc_particle_buffer* pb = &s->bins[i][model];
		pb->rho = rho;
		pb->volume = vol;
		pb->mass = vol * rho;
		pb->lambda = ym * pr / ((1 + pr) * (1 - 2 * pr));
		pb->mu = ym / (2 * (1 + pr));
	}
}
void orc_sim_update_sand_parameters(orc_sim* s, int model, float rho, float vol, float ym, float pr) { orc_sim_update_fr_parameters(s, model, rho, vol, ym, pr); }
void orc_sim_update_j_fluid_parameters(orc_sim* s, int model, float rho, float vol, float bulk, float gamma, float visc) {
	for(int i = 0; i < 2; ++i) {
		orc_particle_buffer* pb = &s->bins[i][model];
		pb->rho = rho;
		pb->volume = vol;
		pb->mass = vol * rho;
		pb->bulk = bulk;
		pb->gamma = gamma;
		pb->viscosity = visc;
	}
}
void orc_sim_update_nacc_parameters(orc_sim* s, int model, float rho, float vol, float ym, float pr, float beta, float xi) {
	for(int i = 0; i < 2; ++i) {
		orc_particle_buffer* pb = &s->bins[i][model];
		pb->rho = rho;
		pb->volume = vol;
		pb->mass = vol * rho;
		pb->lambda = ym * pr / ((1 + pr) * (1 - 2 * pr));
		pb->mu = ym / (2 * (1 + pr));
		pb->bm = 2.f / 3.f * (ym / (2 * (1 + pr))) + (ym * pr / ((1 + pr) * (1 - 2 * pr)));
		pb->beta = beta;
		pb->xi = xi;
	}
}

/* compute_dt, ref: Projects/GMPM/utility_funcs.hpp:36-49 */
static float compute_dt(const orc_config* cfg, float max_vel, float time_left, float dt_default) {
	float dt = dt_default;
	if(max_vel > 0.0f) {
		const float ndt = cfg_dx(cfg) * cfg->cfl / max_vel;
		dt = ndt < dt ? ndt : dt;
	}
	dt = dt < time_left ? dt : time_left;
	return dt;
}

static void check_blocks(const orc_sim* s, int n, const char* what) {
	if(n > s->max_blocks) {
		fprintf(stderr, "oracle: too many %s blocks: %d > %d\n", what, n, s->max_blocks);
		abort();
	}
}

/* ref: gmpm_simulator.cuh:637-781 */
void orc_sim_initial_setup(orc_sim* s) {
	const orc_config* cfg = &s->cfg;
	const int R = s->rollid, Rn = R ^ 1;
	{ /* main_loop preamble :305-315 */
		float mv = 0.f;
		for(int m = 0; m < s->nmodels; ++m) {
			const float* v = s->v0[m];
			const float nrm = sqrtf(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
			if(nrm > mv) mv = nrm;
		}
		s->dt = compute_dt(cfg, mv, 1e30f, s->dt_default);
	}
	for(int m = 0; m < s->nmodels; ++m) orc_activate_blocks(cfg, s->count[m], s->init_pos[m], s->parts[Rn]);
	s->pbc = *s->parts[Rn].count;
	check_blocks(s, s->pbc, "particle");
	for(int m = 0; m < s->nmodels; ++m) orc_build_particle_cell_buckets(cfg, s->count[m], s->init_pos[m], s->bins[R][m], s->parts[Rn]);
	for(int m = 0; m < s->nmodels; ++m) {
		orc_particle_buffer pb = s->bins[R][m];
		memset(pb.particle_bucket_sizes, 0, sizeof(int) * (s->pbc + 1));
		orc_cell_bucket_to_block(cfg, s->pbc, pb.cell_particle_counts, pb.cellbuckets, pb.particle_bucket_sizes, pb.blockbuckets);
		orc_compute_bin_capacity(s->pbc + 1, pb.particle_bucket_sizes, s->bin_sizes);
		orc_exclusive_scan(s->pbc + 1, s->bin_sizes, pb.bin_offsets);
		orc_array_to_buffer(cfg, s->pbc, s->init_pos[m], pb);
	}
	orc_register_neighbor_blocks(cfg, s->pbc, s->parts[Rn]);
	s->nbc = *s->parts[Rn].count;
	check_blocks(s, s->nbc, "neighbour");
	orc_register_exterior_blocks(cfg, s->pbc, s->parts[Rn]);
	s->ebc = *s->parts[Rn].count;
	check_blocks(s, s->ebc, "exterior");

	/* :745-756 copy partition + bucket metadata to the background copies */
	{
		const long g = cfg_gsize(cfg);
		memcpy(s->parts[R].index_table, s->parts[Rn].index_table, sizeof(int) * g * g * g);
		memcpy(s->parts[R].active_keys, s->parts[Rn].active_keys, sizeof(int) * 3 * s->ebc);
		for(int m = 0; m < s->nmodels; ++m) {
			memcpy(s->bins[Rn][m].bin_offsets, s->bins[R][m].bin_offsets, sizeof(int) * (s->pbc + 1));
			memcpy(s->bins[Rn][m].particle_bucket_sizes, s->bins[R][m].particle_bucket_sizes, sizeof(int) * s->pbc);
		}
	}
	orc_clear_grid(s->nbc, s->grids[0]);
	for(int m = 0; m < s->nmodels; ++m) {
		orc_rasterize(cfg, s->count[m], s->init_pos[m], s->grids[0], s->parts[R], s->bins[R][m].mass, s->v0[m]);
		orc_init_adv_bucket(cfg, s->pbc, s->bins[Rn][m].particle_bucket_sizes, s->bins[Rn][m].blockbuckets);
	}
}

/* ref: gmpm_simulator.cuh:337-579: one sub-step after its grid update (:337-362), which left the max |v|^2 max_vel_sq.  The
 * collider oracle's sub-step (orc_csim_step) runs it after its own grid update. */
static void sim_step_after_grid_update(orc_sim* s, float max_vel_sq, float time_left) {
	const orc_config* cfg = &s->cfg;
	const int R = s->rollid, Rn = R ^ 1;
	s->max_vel = sqrtf(max_vel_sq);
	s->next_dt = compute_dt(cfg, s->max_vel, time_left, s->dt_default);
	/* :383-398 */
	orc_clear_grid(s->nbc, s->grids[1]);
	for(int m = 0; m < s->nmodels; ++m) {
		memset(s->bins[Rn][m].cell_particle_counts, 0, sizeof(int) * (size_t) s->ebc * BLOCK_VOL);
		orc_g2p2g(cfg, s->dt, s->next_dt, s->pbc, s->bins[R][m], s->bins[Rn][m], s->parts[Rn], s->parts[R], s->grids[0], s->grids[1]);
	}
	/* :424-431 */
	for(int m = 0; m < s->nmodels; ++m) {
		orc_particle_buffer pb = s->bins[Rn][m];
		memset(pb.particle_bucket_sizes, 0, sizeof(int) * (s->ebc + 1));
		orc_cell_bucket_to_block(cfg, s->ebc, pb.cell_particle_counts, pb.cellbuckets, pb.particle_bucket_sizes, pb.blockbuckets);
	}
	/* :438-470 */
	memset(s->marks, 0, sizeof(int) * s->nbc);
	orc_mark_active_grid_blocks(s->nbc, s->grids[1], s->marks);
	memset(s->sources, 0, sizeof(int) * (s->ebc + 1));
	for(int m = 0; m < s->nmodels; ++m) orc_mark_active_particle_blocks(s->ebc + 1, s->bins[Rn][m].particle_bucket_sizes, s->sources);
	orc_exclusive_scan(s->ebc + 1, s->sources, s->destinations);
	const int new_pbc = s->destinations[s->ebc];
	*s->parts[Rn].count = new_pbc;
	orc_exclusive_scan_inverse(s->ebc, s->destinations, s->sources);
	orc_reset_table(cfg, s->parts[Rn]);
	check_blocks(s, new_pbc, "particle");
	/* :480-505 */
	orc_update_partition(cfg, new_pbc, s->sources, s->parts[R], s->parts[Rn]);
	for(int m = 0; m < s->nmodels; ++m) {
		orc_update_buckets(cfg, new_pbc, s->sources, s->bins[Rn][m], s->bins[R][m]);
		/* the reference reads particle_bucket_sizes[pbc] (one past the compacted range, a stale value)
		 * for the (pbc+1)-th bin size; only bin_offsets[0..pbc] are consumed, so the restatement zeroes it */
		s->bins[R][m].particle_bucket_sizes[new_pbc] = 0;
		orc_compute_bin_capacity(new_pbc + 1, s->bins[R][m].particle_bucket_sizes, s->bin_sizes);
		orc_exclusive_scan(new_pbc + 1, s->bin_sizes, s->bins[R][m].bin_offsets);
		if(s->bins[R][m].bin_offsets[new_pbc] > s->bin_capacity[m]) {
			fprintf(stderr, "oracle: bin capacity exceeded\n");
			abort();
		}
	}
	/* :513-524 */
	orc_register_neighbor_blocks(cfg, new_pbc, s->parts[Rn]);
	const int prev_nbc = s->nbc;
	const int new_nbc = *s->parts[Rn].count;
	check_blocks(s, new_nbc, "neighbour");
	/* :536-541 (the reference clears ext blocks of the previous numbering; the new exterior count
	 * is not known yet.  Clearing max(ebc, new_nbc) keeps every block later read well defined.) */
	orc_clear_grid(s->ebc > new_nbc ? s->ebc : new_nbc, s->grids[0]);
	orc_copy_selected_grid_blocks(cfg, prev_nbc, s->parts[R].active_keys, s->parts[Rn], s->marks, s->grids[1], s->grids[0]);
	/* :560-570 */
	orc_register_exterior_blocks(cfg, new_pbc, s->parts[Rn]);
	const int new_ebc = *s->parts[Rn].count;
	check_blocks(s, new_ebc, "exterior");
	s->pbc = new_pbc;
	s->nbc = new_nbc;
	s->ebc = new_ebc;
	/* :578-579 */
	s->rollid = Rn;
	s->dt = s->next_dt;
}

/* ref: gmpm_simulator.cuh:324-580 (one pass of the inner loop) */
void orc_sim_step(orc_sim* s, float time_left) {
	float mv = 0.f; /* :337-362 */
	orc_update_grid_velocity_query_max(&s->cfg, s->nbc, s->grids[0], s->parts[s->rollid], s->dt, &mv);
	sim_step_after_grid_update(s, mv, time_left);
}

int orc_sim_counts(orc_sim* s, int* pbc, int* nbc, int* ebc) {
	*pbc = s->pbc;
	*nbc = s->nbc;
	*ebc = s->ebc;
	return s->nmodels;
}
float orc_sim_dt(orc_sim* s) { return s->dt; }
float orc_sim_max_vel(orc_sim* s) { return s->max_vel; }

/* ref: gmpm_simulator.cuh:594-634 (output_model) */
int orc_sim_retrieve(orc_sim* s, int model, float* out_pos) {
	const int R = s->rollid;
	return orc_retrieve_particle_buffer(&s->cfg, s->pbc, s->parts[R], s->parts[R ^ 1], s->bins[R][model], s->bins[R ^ 1][model], out_pos);
}

const int* orc_sim_active_keys(orc_sim* s) { return s->parts[s->rollid].active_keys; }
const float* orc_sim_grid(orc_sim* s) { return s->grids[0]; }

/* full particle state (all channels) in retrieve order -- same traversal as retrieve_particle_buffer */
int orc_sim_particle_state(orc_sim* s, int model, float* out) {
	const orc_config* cfg = &s->cfg;
	const int R = s->rollid;
	orc_particle_buffer pb = s->bins[R][model], nx = s->bins[R ^ 1][model];
	const int ppb = cfg_ppb(cfg), bf = bin_floats(pb.material);
	const int nch = pb.material == ORC_J_FLUID ? 4 : (pb.material == ORC_FIXED_COROTATED ? 12 : 13);
	int n = 0;
	for(int b = 0; b < s->pbc; ++b) {
		const int cnt = nx.particle_bucket_sizes[b];
		const int* k = s->parts[R].active_keys + 3 * b;
		for(int i = 0; i < cnt; ++i) {
			const int advect = nx.blockbuckets[(long) b * ppb + i];
			int off[3];
			dir_components(advect / ppb, off);
			const int sp = advect % ppb;
			const int sno = part_query(cfg, &s->parts[R ^ 1], k[0] + off[0], k[1] + off[1], k[2] + off[2]);
			const float* bin = pb.bins + ((long) pb.bin_offsets[sno] + sp / BIN_CAP) * bf;
			for(int c = 0; c < nch; ++c) out[(long) n * nch + c] = bin[c * 32 + sp % BIN_CAP];
			++n;
		}
	}
	return n;
}

/* raw container access for kernel-level differential tests: which = 0 -> buffers indexed [rollid], 1 -> [rollid^1] */
void orc_sim_get_buffer(orc_sim* s, int model, int which, orc_particle_buffer* out) { *out = s->bins[s->rollid ^ (which & 1)][model]; }
void orc_sim_get_partition(orc_sim* s, int which, orc_partition* out) { *out = s->parts[s->rollid ^ (which & 1)]; }
float* orc_sim_get_grid(orc_sim* s, int which) { return s->grids[which & 1]; }
long orc_sim_bin_capacity(orc_sim* s, int model) { return s->bin_capacity[model]; }
