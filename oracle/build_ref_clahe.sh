#!/usr/bin/env bash
# oracle/build_ref_clahe.sh -- build oracle/_ref/libalva_ref_clahe.so (oracle/ref_clahe.cpp) beside libalva_ref.so.
# TEST INFRASTRUCTURE: git-ignored like libalva_ref.so, loaded only by the CLAHE tests and tools/make_golden_clahe.py.
# Needs the OpenCV / Ceres configuration oracle/build_ref.sh leaves in $ALVA_REF_PREFIX (default /tmp/probe) and the reference
# tree for its headers; optional like that build -- without it the tests read tests/golden/clahe.npz.
set -euo pipefail
HERE="$(cd "$(dirname "$0")" && pwd)"
REF=${ALVA_REFERENCE:-/root/reference}
P=${ALVA_REF_PREFIX:-/tmp/probe}
OUT="$HERE/_ref"
[ -d "$REF/src/slam/src" ] || { echo "reference tree not found at $REF" >&2; exit 3; }
[ -f "$P/ocv_install/lib/libopencv_imgproc.a" ] || { echo "no OpenCV build under $P: run oracle/build_ref.sh first" >&2; exit 3; }
mkdir -p "$OUT"
INC="-I$REF/src/slam/src -I$REF/src/libs/opencv/modules/highgui/include -I$REF/src/libs/opencv/modules/imgcodecs/include -I$REF/src/libs/opencv/modules/videoio/include -I$REF/src/libs/opengv/include -I$P/ocv_install/include/opencv4 -I$REF/src/libs/eigen -I$REF/src/libs/Sophus \
 -I$P/ceres_install/include -I$P/ceres_install/include/ceres/internal/miniglog"
g++ -std=c++20 -O2 -w -fPIC -shared -o "$OUT/libalva_ref_clahe.so" "$HERE/ref_clahe.cpp" $INC \
  -Wl,--start-group "$P"/ocv_install/lib/libopencv_imgproc.a "$P"/ocv_install/lib/libopencv_core.a \
  "$P"/ocv_install/lib/opencv4/3rdparty/libzlib.a -Wl,--end-group \
  -lpthread -ldl -static-libstdc++ -static-libgcc -Wl,--exclude-libs,ALL
echo "built $OUT/libalva_ref_clahe.so"
