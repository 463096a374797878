// Host shim over the REFERENCE's own level-set sampler: SampleGenerator::LoadSDF and GenerateUniformSamples
// (Library/MnSystem/IO/PoissonDisk/SampleGenerator.h:68-93,149-177, compiled where it lies by build_ref_sdf.sh).  TEST INFRASTRUCTURE
// ONLY: it pins the library's .sdf parser and the float64 restatement of the sampler (tests/sdf_ref.py) against the code that
// sampled the reference's models.
#include <PoissonDisk/SampleGenerator.h>

#include <cstdlib>
#include <vector>

namespace {
struct Probe : SampleGenerator {
	float at(int i, int j, int k) { return fetchGrid(i, j, k); }
};
}  // namespace

extern "C" {

// LoadSDF: dims[3], mins[3], *h; phi (nullable) receives the ni nj nk values with i fastest when capacity allows
int ref_sdf_load(const char* path, int* dims, float* mins, float* h, float* phi, long long capacity) {
	Probe g;
	g.LoadSDF(path, *h, mins[0], mins[1], mins[2], dims[0], dims[1], dims[2]);
	const long long n = (long long) dims[0] * dims[1] * dims[2];
	if(phi && capacity >= n)
		for(int k = 0; k < dims[2]; ++k)
			for(int j = 0; j < dims[1]; ++j)
				for(int i = 0; i < dims[0]; ++i) phi[i + (long long) dims[0] * (j + (long long) dims[1] * k)] = g.at(i, j, k);
	return 0;
}

// srand(seed), then GenerateUniformSamples(samples_per_cell): returns its sampleNum; out (nullable) receives the index-space samples
// when capacity (in samples) allows.  The level set must have a negative node: the reference's loop has no way out otherwise.
long long ref_sdf_uniform(const char* path, unsigned seed, float samples_per_cell, float* out, long long capacity) {
	Probe g;
	float h, mx, my, mz;
	int ni, nj, nk;
	g.LoadSDF(path, h, mx, my, mz, ni, nj, nk);
	srand(seed);
	std::vector<float> s;
	const int num = g.GenerateUniformSamples(samples_per_cell, s);
	if(out && capacity >= (long long) s.size() / 3)
		for(size_t i = 0; i < s.size(); ++i) out[i] = s[i];
	return num;
}

}  // extern "C"
