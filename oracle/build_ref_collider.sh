#!/usr/bin/env bash
# Builds oracle/_ref/libclaymore_ref_collider.so: the REFERENCE's own signed-distance collider (SignedDistanceGrid,
# Projects/MGSP/boundary_condition.cuh) compiled for the host where it lies, at DOMAIN_BITS 5.  TEST INFRASTRUCTURE ONLY.
# Generated into a scratch directory under _ref and deleted after the build: an MGSP settings header with the constant rewritten
# by sed (named to ref_collider_host.cpp in CB200_MGSP_SETTINGS), and a {fmt} stub whose print is a no-op.
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
R="${CLAYMORE_REFERENCE:-/root/reference}"
OUT="$HERE/_ref"
mkdir -p "$OUT"
[ -d "$R" ] || { echo "reference checkout not found at $R; keeping prebuilt $OUT"; exit 0; }
CXX=/usr/bin/g++; [ -x "$CXX" ] || CXX=g++
CSO="$OUT/libclaymore_ref_collider.so"
if [ ! -f "$CSO" ] || [ "$HERE/ref_collider_host.cpp" -nt "$CSO" ] || [ "$HERE/build_ref_collider.sh" -nt "$CSO" ]; then
  GEN="$OUT/gen_collider"
  mkdir -p "$GEN/fmt"
  printf '#pragma once\nnamespace fmt {\ntemplate<typename... A>\ninline void print(A&&...) {}\n}  // namespace fmt\n' > "$GEN/fmt/core.h"
  printf '#pragma once\n#include "core.h"\n' > "$GEN/fmt/color.h"
  sed -e "s/\\(DOMAIN_BITS[[:space:]]*=[[:space:]]*\\)8;/\\15;/" "$R/Projects/MGSP/settings.h" > "$GEN/mgsp_settings.h"
  grep -q "DOMAIN_BITS[[:space:]]*=[[:space:]]*5;" "$GEN/mgsp_settings.h"
  $CXX -std=c++17 -O2 -fPIC -shared -ffp-contract=off -DGRID_BUFFER_CUH "-DCB200_MGSP_SETTINGS=\"$GEN/mgsp_settings.h\"" -I"$GEN" \
      -I$R/Library -I$R/Projects/MGSP -I$R/Externals/function_ref -I$R/Externals/optional -I$R/Externals/variant \
      -o "$CSO" "$HERE/ref_collider_host.cpp"
  rm -rf "$GEN"
fi
echo "oracle/_ref/libclaymore_ref_collider.so up to date"
