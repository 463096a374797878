#!/usr/bin/env bash
# Builds oracle/_ref/libclaymore_ref_partio.so: the REFERENCE's own partio (Externals/partio core + io, system zlib) compiled for the
# host where it lies, with ref_partio_host.cpp (the reference's mn::write_partio and Partio::read behind a C ABI).
# TEST INFRASTRUCTURE ONLY: it pins the library's .bgeo output byte for byte.  The CUDA qualifiers of the reference's Vec.h are
# defined away (host-only use) and AssetDirPath, which only its unused .sdf sampler reads, is given an empty value.
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
R="${CLAYMORE_REFERENCE:-/root/reference}"
OUT="$HERE/_ref"
mkdir -p "$OUT"
[ -d "$R" ] || { echo "reference checkout not found at $R; keeping prebuilt $OUT"; exit 0; }
CXX=/usr/bin/g++; [ -x "$CXX" ] || CXX=g++
SO="$OUT/libclaymore_ref_partio.so"
if [ ! -f "$SO" ] || [ "$HERE/ref_partio_host.cpp" -nt "$SO" ] || [ "$HERE/build_ref_partio.sh" -nt "$SO" ]; then
  P="$R/Externals/partio"
  $CXX -std=c++17 -O2 -fPIC -shared -w -D__host__= -D__device__= -D__forceinline__=inline '-DAssetDirPath=""' \
      -I"$P" -I"$R/Library" -I"$R/Externals/function_ref" -I"$R/Externals/optional" -I"$R/Externals/variant" \
      -o "$SO" "$HERE/ref_partio_host.cpp" "$P"/core/*.cpp "$P"/io/*.cpp -lz
fi
echo "oracle/_ref/libclaymore_ref_partio.so up to date"
