#!/usr/bin/env bash
# Builds oracle/_ref/libclaymore_ref_sdf.so: the REFERENCE's own level-set sampler (Library/MnSystem/IO/PoissonDisk/SampleGenerator.h
# with its cyPoint.h / cySampleElim.h) compiled for the host where it lies, with ref_sdf_host.cpp behind a C ABI.
# TEST INFRASTRUCTURE ONLY: tests/golden/make_ref_sdf_golden.py records its parses and samples as fixtures.
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
R="${CLAYMORE_REFERENCE:-/root/reference}"
OUT="$HERE/_ref"
mkdir -p "$OUT"
[ -d "$R" ] || { echo "reference checkout not found at $R; keeping prebuilt $OUT"; exit 0; }
CXX=/usr/bin/g++; [ -x "$CXX" ] || CXX=g++
SO="$OUT/libclaymore_ref_sdf.so"
if [ ! -f "$SO" ] || [ "$HERE/ref_sdf_host.cpp" -nt "$SO" ] || [ "$HERE/build_ref_sdf.sh" -nt "$SO" ]; then
  $CXX -std=c++17 -O2 -fPIC -shared -w -I"$R/Library/MnSystem/IO" -o "$SO" "$HERE/ref_sdf_host.cpp"
fi
echo "oracle/_ref/libclaymore_ref_sdf.so up to date"
