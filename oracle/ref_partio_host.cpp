// Host shim over the REFERENCE's own particle IO: mn::write_partio (Library/MnSystem/IO/ParticleIO.hpp:14-28) and partio
// (Externals/partio, compiled where it lies by build_ref_partio.sh).  TEST INFRASTRUCTURE ONLY: it pins the library's .bgeo
// writer and claymore_b200.bgeo against the code that wrote the reference's frame files.
#include <MnSystem/IO/ParticleIO.hpp>

#include <Partio.h>

#include <array>
#include <cstring>
#include <vector>

extern "C" {

// positions only, through the reference's own write_partio (the call output_model hands to its IO thread)
int ref_write_partio(const char* path, const float* pos, long long n) {
	std::vector<std::array<float, 3>> data((size_t) n);
	for(long long i = 0; i < n; ++i)
		for(int d = 0; d < 3; ++d) data[i][d] = pos[3 * i + d];
	mn::write_partio<float, 3>(path, data);
	return 0;
}

// positions plus the optional attributes, with write_partio's calls: Partio::addAttribute("v", VECTOR, 3) / ("J", FLOAT, 1)
int ref_write_partio_attributes(const char* path, const float* pos, const float* v, const float* J, long long n) {
	Partio::ParticlesDataMutable* parts = Partio::create();
	Partio::ParticleAttribute pa = parts->addAttribute("position", Partio::VECTOR, 3);
	Partio::ParticleAttribute va, ja;
	if(v) va = parts->addAttribute("v", Partio::VECTOR, 3);
	if(J) ja = parts->addAttribute("J", Partio::FLOAT, 1);
	parts->addParticles((int) n);
	for(int i = 0; i < (int) n; ++i) {
		memcpy(parts->dataWrite<float>(pa, i), pos + 3 * i, 12);
		if(v) memcpy(parts->dataWrite<float>(va, i), v + 3 * i, 12);
		if(J) memcpy(parts->dataWrite<float>(ja, i), J + i, 4);
	}
	Partio::write(path, *parts);
	parts->release();
	return 0;
}

// Partio::read of a file: *n gets the point count and *attrs bit 0 / 1 whether it has "v" / "J"; arrays (nullable) are filled when
// given.  -1 when partio cannot read the file.
int ref_read_partio(const char* path, long long* n, int* attrs, float* pos, float* v, float* J) {
	Partio::ParticlesDataMutable* parts = Partio::read(path, false);
	if(!parts) return -1;
	Partio::ParticleAttribute pa, va, ja;
	const bool hp = parts->attributeInfo("position", pa), hv = parts->attributeInfo("v", va), hj = parts->attributeInfo("J", ja);
	*n = parts->numParticles();
	*attrs = (hv ? 1 : 0) | (hj ? 2 : 0);
	for(int i = 0; i < parts->numParticles(); ++i) {
		if(pos && hp) memcpy(pos + 3 * i, parts->data<float>(pa, i), 12);
		if(v && hv) memcpy(v + 3 * i, parts->data<float>(va, i), 12);
		if(J && hj) memcpy(J + i, parts->data<float>(ja, i), 4);
	}
	parts->release();
	return 0;
}

}  // extern "C"
