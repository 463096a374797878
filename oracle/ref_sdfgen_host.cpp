// Host shim over SDFGen (Externals/SDFGen: makelevelset3.cpp and main.cpp, compiled where they lie by build_ref_sdfgen.sh with
// -O2 -ffp-contract=off and no -march, so the host does no fused multiply-add either).  TEST INFRASTRUCTURE ONLY: it pins the
// library's mesh level sets (claymore_b200/csrc/mesh.cuh) against the tool that made the reference's .sdf files.
#include "makelevelset3.h"

#include <vector>

int sdfgen_main(int argc, char* argv[]);  // main.cpp, renamed by -Dmain=sdfgen_main

extern "C" {

// make_level_set3 on x[3 nv] / tri[3 nt] (0-based); phi receives ni nj nk values, i fastest
int ref_sdfgen_make_level_set3(const float* x, int nv, const int* tri, int nt, const float* origin, float dx, int ni, int nj, int nk, int exact_band,
                               float* phi) {
	std::vector<Vec3f> v(nv);
	for(int i = 0; i < nv; ++i) v[i] = Vec3f(x[3 * i], x[3 * i + 1], x[3 * i + 2]);
	std::vector<Vec3ui> t(nt);
	for(int i = 0; i < nt; ++i) t[i] = Vec3ui(tri[3 * i], tri[3 * i + 1], tri[3 * i + 2]);
	Array3f out;
	make_level_set3(t, v, Vec3f(origin[0], origin[1], origin[2]), dx, ni, nj, nk, out, exact_band);
	for(size_t i = 0; i < out.a.size(); ++i) phi[i] = out.a[i];
	return 0;
}

// SDFGen's whole main: `SDFGen <obj_path> <dx> <padding>` writes <obj_path without .obj>.sdf.  main exits the process on a bad
// file, so the caller passes only files it has checked.
int ref_sdfgen_main(const char* obj_path, const char* dx, const char* padding) {
	char prog[] = "SDFGen";
	char* argv[] = {prog, const_cast<char*>(obj_path), const_cast<char*>(dx), const_cast<char*>(padding), nullptr};
	return sdfgen_main(4, argv);
}

}  // extern "C"
