#!/bin/bash
# TEST INFRASTRUCTURE ONLY — builds oracle/_ref/ from the REFERENCE's own sources where they lie under /root/reference (read-only;
# nothing is copied into the repo) plus the C harnesses oracle/ref_*.cpp.  The reference's build system is not run: a plain g++ loop
# over the hot-path translation units, with the flags of its CMakeLists.txt:L44-57 (-O3, no -march).  Eigen / Sophus-on-Eigen /
# Boost.Thread are absent from this image: oracle/shim/ provides stand-ins (first on the include path), and shadows the two reference
# headers that pull in GTSAM / yaml-cpp (FullSystem/FullSystem.h, IMU/IMUIntegration.hpp).  Output goes to oracle/_ref/ only (git-ignored).
#
#   ref_build.sh          libdso_ref.so (ref_harness.cpp), libselect_ref.so (ref_select.cpp: PixelSelector, makeImages, ImmaturePoint),
#                         libactivation_ref.so (ref_activation.cpp: CoarseDistanceMap) and libundistort_ref.so (ref_undistort.cpp:
#                         Undistort.cpp and settings.cpp alone).  Separate libraries, loaded RTLD_LOCAL, so that the reference's
#                         process-global settings do not alias between them.
#   ref_build.sh tree     libdso_ref_tree.so: the same sources with halves-splitting inner products in the stand-in Eigen
#                         (see oracle/shim/Eigen/Core; tools/eigen_order_sensitivity.py)
#   ref_build.sh dropin   libdso_ref_dropin.so: the drop-in proof (tests/test_dropin.py), see below
#
# An object is rebuilt when it is missing or older than its source or any stand-in header.
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
REF=${REF_ROOT:-/root/reference}
case "$1" in ""|tree|dropin) ;; *) echo "usage: ref_build.sh [tree|dropin]"; exit 2 ;; esac
if [ ! -d "$REF/src/dso" ]; then echo "ref_build: $REF/src/dso not present: keeping the prebuilt oracle/_ref, if any"; exit 0; fi
OUT="$HERE/_ref"
CXX=${CXX:-g++}
FLAGS="-std=c++17 -O3 -fPIC -w -I$HERE/shim -I$REF/src/dso -I$REF/src"
O="$OUT/obj"
if [ "$1" = "tree" ]; then FLAGS="$FLAGS -DEIGSHIM_TREE_REDUX"; O="$OUT/obj_tree"; fi
mkdir -p "$O"

PIDS=""
compile() {  # source -> $O/<name>.o in the background, if stale
  local o="$O/$(basename "$1" .cpp).o"
  if [ ! -f "$o" ] || [ "$1" -nt "$o" ] || [ -n "$(find "$HERE/shim" -newer "$o" -print -quit)" ]; then
    $CXX $FLAGS -c "$1" -o "$o" &
    PIDS="$PIDS $!"
  fi
}
finish() {  # waits for every compile, failing if one failed
  for p in $PIDS; do wait "$p"; done
  PIDS=""
}

SRCS="dso/OptimizationBackend/AccumulatedTopHessian.cpp dso/OptimizationBackend/AccumulatedSCHessian.cpp dso/OptimizationBackend/EnergyFunctional.cpp
dso/OptimizationBackend/EnergyFunctionalStructs.cpp dso/FullSystem/HessianBlocks.cpp dso/FullSystem/Residuals.cpp dso/FullSystem/ImmaturePoint.cpp
dso/FullSystem/CoarseTracker.cpp dso/FullSystem/CoarseInitializer.cpp dso/FullSystem/PixelSelector2.cpp dso/util/settings.cpp dso/util/globalCalib.cpp util/TimeMeasurement.cpp"
OBJS=""
for s in $SRCS; do
  compile "$REF/src/$s"
  OBJS="$OBJS $O/$(basename "$s" .cpp).o"
done

case "$1" in
"")
  for h in ref_harness ref_select ref_activation ref_undistort; do compile "$HERE/$h.cpp"; done
  compile "$REF/src/dso/util/Undistort.cpp"
  finish
  $CXX -shared -pthread -o "$OUT/libdso_ref.so" $OBJS "$O/ref_harness.o"
  # ref_harness.o holds the link-time leftovers of the translation units that are not compiled
  for x in select activation; do
    $CXX -shared -pthread -o "$OUT/lib${x}_ref.so" "$O/ref_$x.o" "$O/ref_harness.o" $OBJS -l:libstdc++.so.6
  done
  $CXX -shared -o "$OUT/libundistort_ref.so" "$O/Undistort.o" "$O/settings.o" "$O/ref_undistort.o" -l:libstdc++.so.6
  echo "ref_build: $OUT/libdso_ref.so libselect_ref.so libactivation_ref.so libundistort_ref.so"
  ;;
tree)
  compile "$HERE/ref_harness.cpp"
  finish
  $CXX -shared -pthread -o "$OUT/libdso_ref_tree.so" $OBJS "$O/ref_harness.o"
  echo "ref_build: $OUT/libdso_ref_tree.so"
  ;;
dropin)
  # the same reference objects + oracle/dropin_stubs.cpp FIRST on the link line; its definitions of CoarseTracker::calcRes/calcGSSSE and
  # EnergyFunctional::accumulateAF_MT/accumulateSCF_MT/resubstituteF_MT replace the reference's (-Wl,--allow-multiple-definition keeps the
  # first; -fPIC calls between members go through the PLT, so callers inside the reference's own objects — solveSystemF, trackNewestCoarse —
  # reach the stubs), which forward to ../dm-vio_b200/libdmvio_b200.so through include/dmvio_b200.h
  finish
  LIBDIR="$(cd "$HERE/../dm-vio_b200" && pwd)"
  if [ ! -f "$LIBDIR/libdmvio_b200.so" ]; then echo "ref_build dropin: build dm-vio_b200/libdmvio_b200.so first"; exit 1; fi
  $CXX $FLAGS -DDMV_DROPIN -c "$HERE/ref_harness.cpp" -o "$O/ref_harness_dropin.o"
  $CXX $FLAGS -c "$HERE/dropin_stubs.cpp" -o "$O/dropin_stubs.o"
  $CXX -shared -pthread -Wl,--allow-multiple-definition -o "$OUT/libdso_ref_dropin.so" "$O/dropin_stubs.o" $OBJS "$O/ref_harness_dropin.o" \
       -L"$LIBDIR" -ldmvio_b200 -Wl,-rpath,'$ORIGIN/../../dm-vio_b200'
  echo "ref_build: $OUT/libdso_ref_dropin.so"
  ;;
esac
