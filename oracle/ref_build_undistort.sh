#!/bin/bash
# TEST INFRASTRUCTURE ONLY — builds oracle/_ref/libundistort_ref.so from the REFERENCE's own util/Undistort.cpp and util/settings.cpp
# where they lie under /root/reference (read-only; nothing is copied into the repo) plus oracle/ref_undistort.cpp, with the flags of
# its CMakeLists.txt:L44-57 (-O3, no -march) and the stand-in headers of oracle/shim/ (see ref_build.sh).  A library of its own (loaded RTLD_LOCAL), so
# that the reference's process-global settings do not alias libdso_ref.so's.  Output goes to oracle/_ref/ only (git-ignored).
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
REF=${REF_ROOT:-/root/reference}
if [ ! -d "$REF/src/dso" ]; then echo "ref_build_undistort: $REF/src/dso not present: keeping the prebuilt oracle/_ref, if any"; exit 0; fi
OUT="$HERE/_ref"
CXX=${CXX:-g++}
FLAGS="-std=c++17 -O3 -fPIC -w -I$HERE/shim -I$REF/src/dso -I$REF/src"
mkdir -p "$OUT/obj_undistort"
O="$OUT/obj_undistort"
$CXX $FLAGS -c "$REF/src/dso/util/Undistort.cpp" -o "$O/Undistort.o" &
$CXX $FLAGS -c "$REF/src/dso/util/settings.cpp" -o "$O/settings.o" &
$CXX $FLAGS -c "$HERE/ref_undistort.cpp" -o "$O/ref_undistort.o" &
wait
$CXX -shared -o "$OUT/libundistort_ref.so" "$O/Undistort.o" "$O/settings.o" "$O/ref_undistort.o" -l:libstdc++.so.6
echo "ref_build_undistort: $OUT/libundistort_ref.so"
