#!/usr/bin/env bash
# Builds oracle/_ref/libclaymore_ref_sdfgen.so: the REFERENCE's vendored SDFGen (Externals/SDFGen/makelevelset3.cpp and main.cpp)
# compiled for the host where it lies, with ref_sdfgen_host.cpp behind a C ABI.  main.cpp is renamed (-Dmain=sdfgen_main) and gets
# an empty config.h of its own, so HAVE_VTK stays undefined and it writes the text .sdf.  -ffp-contract=off and no -march: the
# host computes SDFGen's float / double expressions without fused multiply-add.
# TEST INFRASTRUCTURE ONLY: tests/golden/make_ref_sdfgen_golden.py records its level sets as fixtures.
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
R="${CLAYMORE_REFERENCE:-/root/reference}"
OUT="$HERE/_ref"
mkdir -p "$OUT"
[ -d "$R" ] || { echo "reference checkout not found at $R; keeping prebuilt $OUT"; exit 0; }
CXX=/usr/bin/g++; [ -x "$CXX" ] || CXX=g++
S="$R/Externals/SDFGen"
SO="$OUT/libclaymore_ref_sdfgen.so"
INC="$OUT/sdfgen_include"
if [ ! -f "$SO" ] || [ "$HERE/ref_sdfgen_host.cpp" -nt "$SO" ] || [ "$HERE/build_ref_sdfgen.sh" -nt "$SO" ]; then
  mkdir -p "$INC"
  : > "$INC/config.h"
  FLAGS=(-std=c++17 -O2 -ffp-contract=off -fPIC -w -I"$INC" -I"$S")
  $CXX "${FLAGS[@]}" -c -o "$OUT/sdfgen_makelevelset3.o" "$S/makelevelset3.cpp"
  $CXX "${FLAGS[@]}" -Dmain=sdfgen_main -c -o "$OUT/sdfgen_main.o" "$S/main.cpp"
  $CXX "${FLAGS[@]}" -shared -o "$SO" "$HERE/ref_sdfgen_host.cpp" "$OUT/sdfgen_makelevelset3.o" "$OUT/sdfgen_main.o"
fi
echo "oracle/_ref/libclaymore_ref_sdfgen.so up to date"
