#!/bin/bash
# TEST INFRASTRUCTURE ONLY — builds oracle/_ref/libactivation_ref.so: oracle/ref_activation.cpp, which drives the REFERENCE's CoarseDistanceMap
# and mirrors activatePointsMT's selection loop, linked with the reference objects ref_build.sh compiles from /root/reference (read-only;
# nothing is copied into the repo) and ref_harness.o (the link-time leftovers of the translation units that are not compiled).  A library of
# its own (loaded RTLD_LOCAL), so that the reference's process-global settings do not alias libdso_ref.so's.  Flags of the reference's
# CMakeLists.txt:L44-57 (-O3, no -march) and the stand-in headers of oracle/shim/.  Output goes to oracle/_ref/ only (git-ignored).
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
REF=${REF_ROOT:-/root/reference}
if [ ! -d "$REF/src/dso" ]; then echo "ref_build_activation: $REF/src/dso not present: keeping the prebuilt oracle/_ref, if any"; exit 0; fi
OUT="$HERE/_ref"
if [ ! -f "$OUT/libdso_ref.so" ]; then bash "$HERE/ref_build.sh"; fi
CXX=${CXX:-g++}
FLAGS="-std=c++17 -O3 -fPIC -w -I$HERE/shim -I$REF/src/dso -I$REF/src"
mkdir -p "$OUT/obj"
$CXX $FLAGS -c "$HERE/ref_activation.cpp" -o "$OUT/obj/ref_activation.o"
O="$OUT/obj"
$CXX -shared -pthread -o "$OUT/libactivation_ref.so" "$O/ref_activation.o" "$O/ref_harness.o" "$O/AccumulatedTopHessian.o" "$O/AccumulatedSCHessian.o" \
     "$O/EnergyFunctional.o" "$O/EnergyFunctionalStructs.o" "$O/HessianBlocks.o" "$O/Residuals.o" "$O/ImmaturePoint.o" "$O/CoarseTracker.o" \
     "$O/CoarseInitializer.o" "$O/PixelSelector2.o" "$O/settings.o" "$O/globalCalib.o" "$O/TimeMeasurement.o" -l:libstdc++.so.6
echo "ref_build_activation: $OUT/libactivation_ref.so"
