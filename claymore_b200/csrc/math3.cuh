// math3.cuh -- register-resident 3x3 math for the G2P2G kernel: B-spline weights, symmetric Jacobi
// eigen-solver / SVD, constitutive models.  Column-major 3x3 (m[r + 3c]) like the reference's
// MatrixUtils.h.  Everything is FP32 and stays in registers (no tensor cores: 3x3 contractions).
//
// Behavioural contracts (results must agree with the reference to FP32 tolerance, not bitwise):
//   svd3            <-> math::svd            Library/MnBase/Math/Matrix/svd.cuh:28-1124
//   stress_*        <-> compute_stress<M>    Projects/GMPM/constitutive_models.cuh:36-73,78-234,239-335
//   bspline_weights <-> bspline_weight       Projects/GMPM/utility_funcs.hpp:10-19
#pragma once
#include "common.cuh"

namespace cb200 {

// ------------------------------------------------------------------------------------------------
// FP32 pairs.  The separable-weight arithmetic of G2P / P2G and the packed 3x3 form carry aligned pairs of values; sm_90a
// has no packed FP32 FMA, so each pair operation is two scalar FFMA / FMUL / FADD, and the compiler is free to contract a
// multiply and a following add into one FFMA like any other scalar code.
// ------------------------------------------------------------------------------------------------
using f2 = float2;
__device__ __forceinline__ f2 mk2(float a, float b) { return make_float2(a, b); }
__device__ __forceinline__ f2 dup2(float a) { return make_float2(a, a); }
__device__ __forceinline__ f2 fma2(f2 a, f2 b, f2 c) { return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)); }
__device__ __forceinline__ f2 fma2(f2 a, float s, f2 c) { return make_float2(fmaf(a.x, s, c.x), fmaf(a.y, s, c.y)); }
__device__ __forceinline__ f2 mul2(f2 a, f2 b) { return make_float2(a.x * b.x, a.y * b.y); }
__device__ __forceinline__ f2 mul2(f2 a, float s) { return make_float2(a.x * s, a.y * s); }
__device__ __forceinline__ f2 add2(f2 a, f2 b) { return make_float2(a.x + b.x, a.y + b.y); }

// quadratic B-spline weights of the 3 nodes covering local position p in [0.5dx, 1.5dx)
__device__ __forceinline__ void bspline_weights(float p_times_dxinv, float& w0, float& w1, float& w2) {
	float d = p_times_dxinv;
	w0 = 0.5f * (1.5f - d) * (1.5f - d);
	d -= 1.0f;
	w1 = 0.75f - d * d;
	d = 0.5f + d;
	w2 = 0.5f * d * d;
}

// ------------------------------------------------------------------------------------------------
// 3x3 SVD  A = U diag(S) V^T with U, V rotations, |S0| >= |S1| >= |S2| (S2 may be negative).
// Jacobi eigen-iteration on A^T A with the gamma-tested approximate Givens quaternion, followed by a
// Givens QR of A V (the minimal-branching scheme of McAdams et al. 2011, which the reference carries).
// ------------------------------------------------------------------------------------------------
struct Sym3 {
	float s11, s21, s22, s31, s32, s33;
};
struct Quat {
	float s, x, y, z;
};

// one cyclic Jacobi rotation annihilating `b` (the (q,p) entry); (a,c) diagonal pair, (d,e) the third
// row entries, f the third diagonal; (qx,qy,qz) permuted so that qz is the rotation axis
__device__ __forceinline__ void jacobi_rotate(float& a, float& b, float& c, float& d, float& e, float& f, float& qs, float& qx, float& qy, float& qz) {
	constexpr float kFourGammaSq = 5.8284273147583007813f;
	constexpr float kSinPi8 = 0.3826834261417388916f;
	constexpr float kCosPi8 = 0.92387956380844116211f;
	float sh = 0.5f * b;
	float diff = a - c;
	const bool tiny = sh * sh < 1.e-20f;
	float ch = tiny ? 1.f : diff;
	sh = tiny ? 0.f : sh;
	const float sh2 = sh * sh, ch2 = ch * ch;
	const float r = rsqrtf(sh2 + ch2);
	const bool big = ch2 <= kFourGammaSq * sh2;
	sh = big ? kSinPi8 : r * sh;
	ch = big ? kCosPi8 : r * ch;
	const float s2 = sh * sh, c2 = ch * ch;
	const float cc = c2 - s2;
	const float ss = 2.f * ch * sh;
	const float nrm = s2 + c2;  // == 1 up to rounding; kept so the scale of S stays consistent

	// conjugate the symmetric matrix
	f *= nrm * nrm;
	d *= nrm;
	e *= nrm;
	const float d0 = d, e0 = e;
	d = cc * d0 + ss * e0;
	e = cc * e0 - ss * d0;
	const float ss2 = ss * ss, cc2 = cc * cc, cs = cc * ss;
	const float a0 = a, b0 = b, c0 = c;
	a = a0 * cc2 + c0 * ss2 + 2.f * b0 * cs;
	c = c0 * cc2 + a0 * ss2 - 2.f * b0 * cs;
	b = b0 * (cc2 - ss2) - diff * cs;

	// accumulate the rotation
	const float x0 = qx, y0 = qy, z0 = qz, w0 = qs;
	qs = ch * w0 - sh * z0;
	qx = ch * x0 + sh * y0;
	qy = ch * y0 - sh * x0;
	qz = ch * z0 + sh * w0;
}

// Jacobi sweeps on a symmetric matrix; returns the accumulated rotation as a normalised quaternion
template<int SWEEPS>
__device__ __forceinline__ Quat jacobi_eigen_quat(Sym3 m) {
	Quat q {1.f, 0.f, 0.f, 0.f};
#pragma unroll 1
	for(int it = 0; it < SWEEPS; ++it) {
		// converged: the off-diagonal is below FP32 resolution of the diagonal (further rotations would be identities).
		// Nearly undeformed particles (sand at rest, elastic bodies in free flight) leave after zero or one sweep.
		const float off = m.s21 * m.s21 + m.s31 * m.s31 + m.s32 * m.s32;
		const float dia = m.s11 * m.s11 + m.s22 * m.s22 + m.s33 * m.s33;
		if(off <= 1e-14f * dia) break;
		jacobi_rotate(m.s11, m.s21, m.s22, m.s31, m.s32, m.s33, q.s, q.x, q.y, q.z);
		jacobi_rotate(m.s22, m.s32, m.s33, m.s21, m.s31, m.s11, q.s, q.y, q.z, q.x);
		jacobi_rotate(m.s33, m.s31, m.s11, m.s32, m.s21, m.s22, q.s, q.z, q.x, q.y);
	}
	const float n = rsqrtf(q.s * q.s + q.x * q.x + q.y * q.y + q.z * q.z);
	q.s *= n;
	q.x *= n;
	q.y *= n;
	q.z *= n;
	return q;
}

// quaternion -> rotation matrix (column-major)
__device__ __forceinline__ void quat_to_mat(const Quat& q, float* V) {
	const float xx = q.x * q.x, yy = q.y * q.y, zz = q.z * q.z, ww = q.s * q.s;
	const float xy = q.x * q.y, yz = q.y * q.z, zx = q.z * q.x;
	const float wx = q.s * q.x, wy = q.s * q.y, wz = q.s * q.z;
	V[0] = ww + xx - yy - zz;
	V[4] = ww - xx + yy - zz;
	V[8] = ww - xx - yy + zz;
	V[1] = 2.f * (xy + wz);  // v21
	V[3] = 2.f * (xy - wz);  // v12
	V[5] = 2.f * (yz + wx);  // v32
	V[7] = 2.f * (yz - wx);  // v23
	V[6] = 2.f * (zx + wy);  // v13
	V[2] = 2.f * (zx - wy);  // v31
}

// swap columns p,q of B and V when |B_p| < |B_q|, flipping the sign of column `neg` to stay a rotation
__device__ __forceinline__ void sort_cols(float* B, float* V, float& np, float& nq, int p, int q, int neg) {
	const bool sw = np < nq;
#pragma unroll
	for(int r = 0; r < 3; ++r) {
		const float bp = B[r + 3 * p], bq = B[r + 3 * q];
		B[r + 3 * p] = sw ? bq : bp;
		B[r + 3 * q] = sw ? bp : bq;
		const float vp = V[r + 3 * p], vq = V[r + 3 * q];
		V[r + 3 * p] = sw ? vq : vp;
		V[r + 3 * q] = sw ? vp : vq;
	}
	const float t = np;
	np = sw ? nq : np;
	nq = sw ? t : nq;
	const float sg = sw ? -1.f : 1.f;
#pragma unroll
	for(int r = 0; r < 3; ++r) {
		B[r + 3 * neg] *= sg;
		V[r + 3 * neg] *= sg;
	}
}

// Givens rotation of rows p,q of B zeroing B[q,p]; columns p,q of U follow
__device__ __forceinline__ void qr_rotate(float* B, float* U, int p, int q) {
	const float pivot = B[p + 3 * p];
	const float below = B[q + 3 * p];
	float sh = (below * below >= 1.e-12f) ? below : 0.f;
	float ch = fmaxf(fabsf(pivot), 1.e-12f);
	const float rho = sqrtf(ch * ch + sh * sh);
	ch += rho;
	if(pivot < 0.f) {
		const float t = ch;
		ch = sh;
		sh = t;
	}
	const float r = rsqrtf(ch * ch + sh * sh);
	ch *= r;
	sh *= r;
	const float c = ch * ch - sh * sh;
	const float s = 2.f * sh * ch;
#pragma unroll
	for(int col = 0; col < 3; ++col) {
		const float x = B[p + 3 * col], y = B[q + 3 * col];
		B[p + 3 * col] = c * x + s * y;
		B[q + 3 * col] = c * y - s * x;
	}
#pragma unroll
	for(int row = 0; row < 3; ++row) {
		const float x = U[row + 3 * p], y = U[row + 3 * q];
		U[row + 3 * p] = c * x + s * y;
		U[row + 3 * q] = c * y - s * x;
	}
}

__device__ __forceinline__ void svd3(const float* A, float* U, float* S, float* V) {
	Sym3 m;
	m.s11 = A[0] * A[0] + A[1] * A[1] + A[2] * A[2];
	m.s21 = A[3] * A[0] + A[4] * A[1] + A[5] * A[2];
	m.s31 = A[6] * A[0] + A[7] * A[1] + A[8] * A[2];
	m.s22 = A[3] * A[3] + A[4] * A[4] + A[5] * A[5];
	m.s32 = A[6] * A[3] + A[7] * A[4] + A[8] * A[5];
	m.s33 = A[6] * A[6] + A[7] * A[7] + A[8] * A[8];
	const Quat q = jacobi_eigen_quat<4>(m);
	quat_to_mat(q, V);
	float B[9];
#pragma unroll
	for(int c = 0; c < 3; ++c)
#pragma unroll
		for(int r = 0; r < 3; ++r) B[r + 3 * c] = A[r] * V[3 * c] + A[r + 3] * V[3 * c + 1] + A[r + 6] * V[3 * c + 2];
	float n0 = B[0] * B[0] + B[1] * B[1] + B[2] * B[2];
	float n1 = B[3] * B[3] + B[4] * B[4] + B[5] * B[5];
	float n2 = B[6] * B[6] + B[7] * B[7] + B[8] * B[8];
	sort_cols(B, V, n0, n1, 0, 1, 1);
	sort_cols(B, V, n0, n2, 0, 2, 0);
	sort_cols(B, V, n1, n2, 1, 2, 2);
#pragma unroll
	for(int i = 0; i < 9; ++i) U[i] = (i % 4 == 0) ? 1.f : 0.f;
	qr_rotate(B, U, 0, 1);
	qr_rotate(B, U, 0, 2);
	qr_rotate(B, U, 1, 2);
	S[0] = B[0];
	S[1] = B[4];
	S[2] = B[8];
}

// out = M1 diag(d) M2^T
__device__ __forceinline__ void mat_diag_mat_t(float* out, const float* m1, const float* d, const float* m2) {
#pragma unroll
	for(int c = 0; c < 3; ++c)
#pragma unroll
		for(int r = 0; r < 3; ++r) out[r + 3 * c] = m1[r] * d[0] * m2[c] + m1[r + 3] * d[1] * m2[c + 3] + m1[r + 6] * d[2] * m2[c + 6];
}
// out = P F^T * vol
__device__ __forceinline__ void p_ft_vol(float* out, const float* P, const float* F, float vol) {
#pragma unroll
	for(int c = 0; c < 3; ++c)
#pragma unroll
		for(int r = 0; r < 3; ++r) out[r + 3 * c] = (P[r] * F[c] + P[r + 3] * F[c + 3] + P[r + 6] * F[c + 6]) * vol;
}

// FIXED_COROTATED: P_hat_i = 2 mu (s_i - 1) + lambda (J - 1) prod_{j != i} s_j ; PF = U P_hat V^T F^T vol
__device__ __forceinline__ void stress_fixed_corotated(const Mat& m, const float* F, float* PF) {
	float U[9], S[3], V[9];
	svd3(F, U, S, V);
	const float J = S[0] * S[1] * S[2];
	const float mu2 = 2.f * m.mu;
	const float lam = m.lambda * (J - 1.f);
	float Ph[3];
	Ph[0] = mu2 * (S[0] - 1.f) + lam * (S[1] * S[2]);
	Ph[1] = mu2 * (S[1] - 1.f) + lam * (S[0] * S[2]);
	Ph[2] = mu2 * (S[2] - 1.f) + lam * (S[0] * S[1]);
	float P[9];
	mat_diag_mat_t(P, U, Ph, V);
	p_ft_vol(PF, P, F, m.volume);
}

// FIXED_COROTATED without the SVD.  With the polar decomposition F = R S:
//   P F^T = 2 mu (F - R) F^T + lambda (J - 1) J I          (identical to U P_hat V^T F^T of the reference)
// R is obtained by Newton's iteration R <- (R + R^-T) / 2 (quadratically convergent; 3-4 iterations for the stretches
// an elastic body sees), which costs ~1/4 of the Jacobi SVD + QR.  Inverted or nearly singular F (det <= 1e-6), where the
// reference's SVD convention (proper rotations, negative last singular value) matters, takes the SVD path.
__device__ __forceinline__ void stress_fixed_corotated_polar(const Mat& m, const float* F, float* PF) {
	float R[9];
#pragma unroll
	for(int i = 0; i < 9; ++i) R[i] = F[i];
	float J = 1.f;
	bool ok = false;  // set when the iteration has converged; anything else (inverted, nearly singular, slow) takes the SVD path
#pragma unroll 1
	for(int it = 0; it < 12; ++it) {
		float C[9];  // cofactor matrix (column-major): R^-T = C / det
		C[0] = R[4] * R[8] - R[7] * R[5];
		C[1] = R[6] * R[5] - R[3] * R[8];
		C[2] = R[3] * R[7] - R[6] * R[4];
		C[3] = R[7] * R[2] - R[1] * R[8];
		C[4] = R[0] * R[8] - R[6] * R[2];
		C[5] = R[6] * R[1] - R[0] * R[7];
		C[6] = R[1] * R[5] - R[4] * R[2];
		C[7] = R[3] * R[2] - R[0] * R[5];
		C[8] = R[0] * R[4] - R[3] * R[1];
		const float det = R[0] * C[0] + R[3] * C[3] + R[6] * C[6];
		if(it == 0) {
			J = det;
			if(det <= 1e-6f) break;
		}
		const float h = __fdividef(0.5f, det);
		float d2 = 0.f;
#pragma unroll
		for(int i = 0; i < 9; ++i) {
			const float r = fmaf(h, C[i], 0.5f * R[i]);
			const float d = r - R[i];
			d2 = fmaf(d, d, d2);
			R[i] = r;
		}
		if(d2 < 2e-8f) {  // quadratic contraction: the step after this one would be below FP32 rounding
			ok = true;
			break;
		}
	}
	if(!ok) {
		stress_fixed_corotated(m, F, PF);
		return;
	}
	float D[9];
#pragma unroll
	for(int i = 0; i < 9; ++i) D[i] = F[i] - R[i];
	const float mu2v = 2.f * m.mu * m.volume;
	const float iso = m.lambda * (J - 1.f) * J * m.volume;
#pragma unroll
	for(int c = 0; c < 3; ++c)
#pragma unroll
		for(int r = 0; r < 3; ++r) PF[r + 3 * c] = mu2v * (D[r] * F[c] + D[r + 3] * F[c + 3] + D[r + 6] * F[c + 6]) + ((r == c) ? iso : 0.f);
}

// ------------------------------------------------------------------------------------------------
// 3x3 matrix in packed form (column-major m[r + 3c]): per column the rows (1, 2) as an aligned pair, row 0 as a scalar.
// g2p2g keeps the APIC matrix, F and the stress in this form from the G2P accumulators to the staged P2G record.
// ------------------------------------------------------------------------------------------------
struct M3p {
	float s[3];  // m[0 + 3c]
	f2 p[3];     // (m[1 + 3c], m[2 + 3c])
	__device__ __forceinline__ float at(int r, int c) const { return r == 0 ? s[c] : (r == 1 ? p[c].x : p[c].y); }
};
__device__ __forceinline__ void m3p_to_array(const M3p& m, float* a) {
#pragma unroll
	for(int c = 0; c < 3; ++c) a[3 * c] = m.s[c], a[3 * c + 1] = m.p[c].x, a[3 * c + 2] = m.p[c].y;
}
__device__ __forceinline__ M3p m3p_from_array(const float* a) {
	M3p m;
#pragma unroll
	for(int c = 0; c < 3; ++c) m.s[c] = a[3 * c], m.p[c] = mk2(a[3 * c + 1], a[3 * c + 2]);
	return m;
}
// C = A B^T scaled: C[r + 3c] = k * sum_j A[r + 3j] B[c + 3j]
__device__ __forceinline__ M3p m3p_mul_abt(const M3p& A, const M3p& B, float k) {
	M3p C;
#pragma unroll
	for(int c = 0; c < 3; ++c) {
		const float b0 = B.at(c, 0) * k, b1 = B.at(c, 1) * k, b2 = B.at(c, 2) * k;
		C.p[c] = fma2(A.p[2], b2, fma2(A.p[1], b1, mul2(A.p[0], b0)));
		C.s[c] = fmaf(A.s[2], b2, fmaf(A.s[1], b1, A.s[0] * b0));
	}
	return C;
}

// FIXED_COROTATED without the SVD, packed form of stress_fixed_corotated_polar (same function of F).  Returns false when the
// Newton iteration did not converge (inverted / nearly singular F): the caller takes the SVD path.
// Convergence: Newton's polar iteration contracts quadratically, |R_{k+1} - R| ~ |R_{k+1} - R_k|^2 / 2, so a last step of
// squared Frobenius length < 2e-8 leaves R_{k+1} exact to FP32 rounding (the previous threshold 1e-13 always spent one more
// iteration to observe that).
__device__ __forceinline__ bool stress_fixed_corotated_polar_packed(const Mat& m, const M3p& F, M3p& PF) {
	M3p R = F;
	float J = 1.f;
	bool ok = false;
#pragma unroll 1
	for(int it = 0; it < 12; ++it) {
		const float r0 = R.s[0], r1 = R.p[0].x, r2 = R.p[0].y, r3 = R.s[1], r4 = R.p[1].x, r5 = R.p[1].y, r6 = R.s[2], r7 = R.p[2].x, r8 = R.p[2].y;
		// cofactor matrix (column-major): R^-T = C / det
		const float c0 = r4 * r8 - r7 * r5, c1 = r6 * r5 - r3 * r8, c2 = r3 * r7 - r6 * r4;
		const float c3 = r7 * r2 - r1 * r8, c4 = r0 * r8 - r6 * r2, c5 = r6 * r1 - r0 * r7;
		const float c6 = r1 * r5 - r4 * r2, c7 = r3 * r2 - r0 * r5, c8 = r0 * r4 - r3 * r1;
		const float det = r0 * c0 + r3 * c3 + r6 * c6;
		if(it == 0) {
			J = det;
			if(det <= 1e-6f) break;
		}
		const float h = __fdividef(0.5f, det);
		M3p N;
		N.s[0] = fmaf(h, c0, 0.5f * r0);
		N.s[1] = fmaf(h, c3, 0.5f * r3);
		N.s[2] = fmaf(h, c6, 0.5f * r6);
		N.p[0] = fma2(mk2(c1, c2), h, mul2(R.p[0], 0.5f));
		N.p[1] = fma2(mk2(c4, c5), h, mul2(R.p[1], 0.5f));
		N.p[2] = fma2(mk2(c7, c8), h, mul2(R.p[2], 0.5f));
		f2 d2p = mk2(0.f, 0.f);
		float d2 = 0.f;
#pragma unroll
		for(int c = 0; c < 3; ++c) {
			const f2 d = fma2(R.p[c], -1.f, N.p[c]);
			d2p = fma2(d, d, d2p);
			const float e = N.s[c] - R.s[c];
			d2 = fmaf(e, e, d2);
		}
		R = N;
		if(d2 + d2p.x + d2p.y < 2e-8f) {
			ok = true;
			break;
		}
	}
	if(!ok) return false;
	// P F^T vol = 2 mu vol (F - R) F^T + lambda (J - 1) J vol I
	M3p D;
#pragma unroll
	for(int c = 0; c < 3; ++c) {
		D.s[c] = F.s[c] - R.s[c];
		D.p[c] = fma2(R.p[c], -1.f, F.p[c]);
	}
	PF = m3p_mul_abt(D, F, 2.f * m.mu * m.volume);
	const float iso = m.lambda * (J - 1.f) * J * m.volume;
	PF.s[0] += iso;
	PF.p[1].x += iso;
	PF.p[2].y += iso;
	return true;
}

// SAND: Drucker-Prager return mapping on the Hencky strain, StVK-Hencky elasticity; F and log_jp are updated
__device__ __forceinline__ void stress_sand(const Mat& m, float* F, float* PF, float& log_jp) {
	float U[9], S[3], V[9];
	svd3(F, U, S, V);
	const float mu2 = 2.f * m.mu;
	float eps[3], newS[3] = {0.f, 0.f, 0.f};
#pragma unroll
	for(int i = 0; i < 3; ++i) eps[i] = logf(fmaxf(fabsf(S[i]), 1e-4f)) - m.cohesion;
	const float sum_eps = eps[0] + eps[1] + eps[2];
	const float trace_eps = sum_eps + log_jp;
	float eh[3];
#pragma unroll
	for(int i = 0; i < 3; ++i) eh[i] = eps[i] - (trace_eps / 3.0f);
	const float eh_norm = sqrtf(eh[0] * eh[0] + eh[1] * eh[1] + eh[2] * eh[2]);
	bool changed = false;
	if(trace_eps >= 0.f) {
		newS[0] = newS[1] = newS[2] = expf(m.cohesion);
		changed = true;
		if(m.volume_correction) log_jp = m.beta * sum_eps + log_jp;
	} else if(m.mu != 0.f) {
		log_jp = 0.f;
		const float delta_gamma = eh_norm + (3.f * m.lambda + mu2) / mu2 * trace_eps * m.yield_surface;
		float H[3];
		if(delta_gamma <= 0.f) {
#pragma unroll
			for(int i = 0; i < 3; ++i) H[i] = eps[i] + m.cohesion;
		} else {
#pragma unroll
			for(int i = 0; i < 3; ++i) H[i] = eps[i] - (delta_gamma / eh_norm) * eh[i] + m.cohesion;
		}
#pragma unroll
		for(int i = 0; i < 3; ++i) newS[i] = expf(H[i]);
		changed = true;
	}
	if(changed) mat_diag_mat_t(F, U, newS, V);
	const float l0 = logf(newS[0]), l1 = logf(newS[1]), l2 = logf(newS[2]);
	const float tr = l0 + l1 + l2;
	float Ph[3];
	Ph[0] = (mu2 * l0 + m.lambda * tr) / newS[0];
	Ph[1] = (mu2 * l1 + m.lambda * tr) / newS[1];
	Ph[2] = (mu2 * l2 + m.lambda * tr) / newS[2];
	float P[9];
	mat_diag_mat_t(P, U, Ph, V);
	p_ft_vol(PF, P, F, m.volume);
}

// NACC: non-associated Cam-Clay with hardening in log_jp
__device__ __forceinline__ void stress_nacc(const Mat& m, float* F, float* PF, float& log_jp) {
	float U[9], S[3], V[9];
	svd3(F, U, S, V);
	const float bm = m.bm, beta = m.beta, msqr = m.msqr, mu = m.mu;
	const float p0 = bm * (0.00001f + sinhf(m.xi * fmaxf(-log_jp, 0.f)));
	const float p_min = -beta * p0;
	const float Je_trial = S[0] * S[1] * S[2];
	const float B0 = S[0] * S[0], B1 = S[1] * S[1], B2 = S[2] * S[2];
	const float trB3 = (B0 + B1 + B2) / 3.f;
	const float Jm = mu * powf(Je_trial, -2.f / 3.f);
	const float sh0 = Jm * (B0 - trB3), sh1 = Jm * (B1 - trB3), sh2 = Jm * (B2 - trB3);
	const float psi_kappa = bm * 0.5f * (Je_trial - 1.f / Je_trial);
	const float p_trial = -psi_kappa * Je_trial;
	const float ys_coeff = 3.f / 2.f * (1.f + 2.f * beta);
	const float y_p_half = msqr * (p_trial - p_min) * (p_trial - p0);
	const float s_sq = sh0 * sh0 + sh1 * sh1 + sh2 * sh2;
	const float y = ys_coeff * s_sq + y_p_half;
	bool changed = false;
	if(p_trial > p0) {
		const float Je_new = sqrtf(-2.f * p0 / bm + 1.f);
		S[0] = S[1] = S[2] = powf(Je_new, 1.f / 3.f);
		changed = true;
		if(m.hardening_on) log_jp += logf(Je_trial / Je_new);
	} else if(p_trial < p_min) {
		const float Je_new = sqrtf(-2.f * p_min / bm + 1.f);
		S[0] = S[1] = S[2] = powf(Je_new, 1.f / 3.f);
		changed = true;
		if(m.hardening_on) log_jp += logf(Je_trial / Je_new);
	} else if(y >= 1e-4f) {
		const float Bs = powf(Je_trial, 2.f / 3.f) / mu * sqrtf(-y_p_half / ys_coeff) / sqrtf(s_sq);
		S[0] = sqrtf(sh0 * Bs + trB3);
		S[1] = sqrtf(sh1 * Bs + trB3);
		S[2] = sqrtf(sh2 * Bs + trB3);
		changed = true;
		if(m.hardening_on && p0 > 1e-4f && p_trial < p0 - 1e-4f && p_trial > 1e-4f + p_min) {
			const float p_center = (1.f - beta) * p0 / 2.f;
			const float q_trial = sqrtf(3.f / 2.f * s_sq);
			float d0 = p_center - p_trial, d1 = -q_trial;
			const float dn = sqrtf(d0 * d0 + d1 * d1);
			d0 /= dn;
			d1 /= dn;
			const float C = msqr * (p_center - p_min) * (p_center - p0);
			const float B = msqr * d0 * (2.f * p_center - p0 - p_min);
			const float A = msqr * d0 * d0 + (1.f + 2.f * beta) * d1 * d1;
			const float disc = sqrtf(B * B - 4.f * A * C);
			const float l1 = (-B + disc) / (2.f * A);
			const float l2 = (-B - disc) / (2.f * A);
			const float p1 = p_center + l1 * d0;
			const float p2 = p_center + l2 * d0;
			const float p_fake = (p_trial - p_center) * (p1 - p_center) > 0.f ? p1 : p2;
			const float tJ = -2.f * p_fake / bm + 1.f;
			const float Je_fake = sqrtf(fabsf(tJ));
			if(Je_fake > 1e-4f) log_jp += logf(Je_trial / Je_fake);
		}
	}
	if(changed) mat_diag_mat_t(F, U, S, V);
	const float J = S[0] * S[1] * S[2];
	float b[9];
#pragma unroll
	for(int c = 0; c < 3; ++c)
#pragma unroll
		for(int r = 0; r < 3; ++r) b[r + 3 * c] = F[r] * F[c] + F[r + 3] * F[c + 3] + F[r + 6] * F[c + 6];
	const float b0 = b[0], b4 = b[4], b8 = b[8];
	b[0] = b0 * (2.f / 3.f) - (b4 + b8) / 3.f;
	b[4] = b4 * (2.f / 3.f) - (b0 + b8) / 3.f;
	b[8] = b8 * (2.f / 3.f) - (b0 + b4) / 3.f;
	const float dev_c = mu * powf(J, -2.f / 3.f);
	const float i_c = bm * .5f * ((J * J - 1.f) * 0.5f - logf(J));
#pragma unroll
	for(int i = 0; i < 9; ++i) PF[i] = (dev_c * b[i] + ((i % 4 == 0) ? i_c : 0.f)) * m.volume;
}

}  // namespace cb200
