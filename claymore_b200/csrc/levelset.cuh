// levelset.cuh -- the device lattice of a level-set collision object (CB200_SHAPE_LEVELSET, DESIGN.md section 2.11): one float4 per
// node of an SDFGen level set, (phi, g_i, g_j, g_k), built on the device from phi after one upload.
#pragma once
#include "common.cuh"

namespace cb200 {

// a header the lattice can be built for: every dimension >= 2 (each axis has a difference) and fewer than 2^31 nodes
inline bool levelset_dims_valid(const cb200_sdf_header* h) {
	return h && h->ni >= 2 && h->nj >= 2 && h->nk >= 2 && (long long) h->ni * h->nj * h->nk < (1LL << 31);
}

// g along one axis at node index c of n, neighbours at +-stride: 0.5f * (phi[+1] - phi[-1]) in float32, one-sided on the faces
__device__ __forceinline__ float levelset_diff(const float* phi, long long idx, int c, int n, long long stride) {
	if(c == 0) return __ldg(phi + idx + stride) - __ldg(phi + idx);
	if(c == n - 1) return __ldg(phi + idx) - __ldg(phi + idx - stride);
	return 0.5f * (__ldg(phi + idx + stride) - __ldg(phi + idx - stride));
}
// one thread per node, i fastest
__global__ void __launch_bounds__(256) levelset_prepare_kernel(int ni, int nj, int nk, const float* phi, float4* lattice) {
	const long long n = (long long) ni * nj * nk, sk = (long long) ni * nj;
	for(long long idx = blockIdx.x * (long long) blockDim.x + threadIdx.x; idx < n; idx += (long long) gridDim.x * blockDim.x) {
		const int i = (int) (idx % ni), j = (int) (idx / ni % nj), k = (int) (idx / sk);
		lattice[idx] = make_float4(__ldg(phi + idx), levelset_diff(phi, idx, i, ni, 1), levelset_diff(phi, idx, j, nj, ni), levelset_diff(phi, idx, k, nk, sk));
	}
}
inline cudaError_t launch_levelset_prepare(const cb200_sdf_header& h, const float* phi, float* lattice, cudaStream_t st) {
	const long long n = (long long) h.ni * h.nj * h.nk;
	const long long ctas = std::min((n + 255) / 256, 1LL << 20);
	levelset_prepare_kernel<<<(int) ctas, 256, 0, st>>>(h.ni, h.nj, h.nk, phi, reinterpret_cast<float4*>(lattice));
	return cudaGetLastError();
}

}  // namespace cb200
