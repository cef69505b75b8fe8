#!/bin/bash
# TEST INFRASTRUCTURE ONLY — builds oracle/_ref/libdso_ref.so from the REFERENCE's own sources where they lie under
# /root/reference (read-only; nothing is copied into the repo) plus oracle/ref_harness.cpp.  The reference's build system is
# not run: a plain g++ loop over the hot-path translation units, with the flags of its CMakeLists.txt:L44-57 (-O3, no
# -march).  Eigen / Sophus-on-Eigen / Boost.Thread are absent from this image: oracle/shim/ provides stand-ins (first on the
# include path), and shadows the two reference headers that pull in GTSAM / yaml-cpp (FullSystem/FullSystem.h,
# IMU/IMUIntegration.hpp).  Output goes to oracle/_ref/ only (git-ignored).
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
REF=${REF_ROOT:-/root/reference}
if [ ! -d "$REF/src/dso" ]; then echo "ref_build: $REF/src/dso not present: keeping the prebuilt oracle/_ref, if any"; exit 0; fi
OUT="$HERE/_ref"
CXX=${CXX:-g++}
FLAGS="-std=c++17 -O3 -fPIC -w -I$HERE/shim -I$REF/src/dso -I$REF/src"
LIBNAME=libdso_ref.so
OBJDIR=obj
if [ "$1" = "tree" ]; then  # sensitivity build: halves-splitting inner products in the stand-in Eigen (see oracle/shim/Eigen/Core)
  FLAGS="$FLAGS -DEIGSHIM_TREE_REDUX"; LIBNAME=libdso_ref_tree.so; OBJDIR=obj_tree
fi
DROPIN=0
if [ "$1" = "dropin" ]; then  # drop-in proof (VERDICT r1 #8): same reference objects + oracle/dropin_stubs.cpp FIRST on the link line; its definitions of
  # CoarseTracker::calcRes/calcGSSSE and EnergyFunctional::accumulateAF_MT/accumulateSCF_MT/resubstituteF_MT replace the reference's
  # (-Wl,--allow-multiple-definition keeps the first; -fPIC calls between members go through the PLT, so callers inside the reference's own
  # objects — solveSystemF, trackNewestCoarse — reach the stubs), which forward to ../dm-vio_b200/libdmvio_b200.so through include/dmvio_b200.h
  DROPIN=1; LIBNAME=libdso_ref_dropin.so
fi
mkdir -p "$OUT/$OBJDIR"
SRCS="dso/OptimizationBackend/AccumulatedTopHessian.cpp dso/OptimizationBackend/AccumulatedSCHessian.cpp dso/OptimizationBackend/EnergyFunctional.cpp
dso/OptimizationBackend/EnergyFunctionalStructs.cpp dso/FullSystem/HessianBlocks.cpp dso/FullSystem/Residuals.cpp dso/FullSystem/ImmaturePoint.cpp
dso/FullSystem/CoarseTracker.cpp dso/FullSystem/CoarseInitializer.cpp dso/FullSystem/PixelSelector2.cpp dso/util/settings.cpp dso/util/globalCalib.cpp util/TimeMeasurement.cpp"
OBJS=""
for s in $SRCS; do
  o="$OUT/$OBJDIR/$(basename "$s" .cpp).o"
  if [ ! -f "$o" ] || [ "$REF/src/$s" -nt "$o" ] || [ "$HERE/shim/Eigen/Core" -nt "$o" ] || [ "$HERE/shim/sophus/se3.hpp" -nt "$o" ]; then
    $CXX $FLAGS -c "$REF/src/$s" -o "$o" &
  fi
  OBJS="$OBJS $o"
done
wait
if [ $DROPIN = 1 ]; then
  LIBDIR="$(cd "$HERE/../dm-vio_b200" && pwd)"
  if [ ! -f "$LIBDIR/libdmvio_b200.so" ]; then echo "ref_build dropin: build dm-vio_b200/libdmvio_b200.so first"; exit 1; fi
  $CXX $FLAGS -DDMV_DROPIN -c "$HERE/ref_harness.cpp" -o "$OUT/$OBJDIR/ref_harness_dropin.o"
  $CXX $FLAGS -c "$HERE/dropin_stubs.cpp" -o "$OUT/$OBJDIR/dropin_stubs.o"
  $CXX -shared -pthread -Wl,--allow-multiple-definition -o "$OUT/$LIBNAME" "$OUT/$OBJDIR/dropin_stubs.o" $OBJS "$OUT/$OBJDIR/ref_harness_dropin.o" \
       -L"$LIBDIR" -ldmvio_b200 -Wl,-rpath,'$ORIGIN/../../dm-vio_b200'
  echo "ref_build: $OUT/$LIBNAME"
  exit 0
fi
$CXX $FLAGS -c "$HERE/ref_harness.cpp" -o "$OUT/$OBJDIR/ref_harness.o"
$CXX -shared -pthread -o "$OUT/$LIBNAME" $OBJS "$OUT/$OBJDIR/ref_harness.o"
echo "ref_build: $OUT/$LIBNAME"
