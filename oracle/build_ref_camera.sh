#!/usr/bin/env bash
# oracle/build_ref_camera.sh -- build oracle/_ref/libalva_ref_camera.so (oracle/ref_camera.cpp + the reference's own
# camera_calibration.cpp, compiled where it lies) beside libalva_ref.so.
# TEST INFRASTRUCTURE: git-ignored like libalva_ref.so, loaded only by the lens-distortion tests and
# tools/make_golden_distortion.py.  Needs the OpenCV configuration oracle/build_ref.sh leaves in $ALVA_REF_PREFIX (default
# /tmp/probe) and the reference tree; optional like that build -- without it the tests read tests/golden/camera.npz.
set -euo pipefail
HERE="$(cd "$(dirname "$0")" && pwd)"
REF=${ALVA_REFERENCE:-/root/reference}
P=${ALVA_REF_PREFIX:-/tmp/probe}
OUT="$HERE/_ref"
[ -d "$REF/src/slam/src" ] || { echo "reference tree not found at $REF" >&2; exit 3; }
[ -f "$P/ocv_install/lib/libopencv_calib3d.a" ] || { echo "no OpenCV build under $P: run oracle/build_ref.sh first" >&2; exit 3; }
mkdir -p "$OUT"
INC="-I$REF/src/slam/src -I$P/ocv_install/include/opencv4 -I$REF/src/libs/eigen -I$REF/src/libs/Sophus"
g++ -std=c++17 -O2 -w -fPIC -shared -o "$OUT/libalva_ref_camera.so" "$HERE/ref_camera.cpp" "$REF/src/slam/src/camera_calibration.cpp" $INC \
  -Wl,--start-group "$P"/ocv_install/lib/libopencv_calib3d.a "$P"/ocv_install/lib/libopencv_features2d.a \
  "$P"/ocv_install/lib/libopencv_flann.a "$P"/ocv_install/lib/libopencv_imgproc.a "$P"/ocv_install/lib/libopencv_core.a \
  "$P"/ocv_install/lib/opencv4/3rdparty/libzlib.a -Wl,--end-group \
  -lpthread -ldl -static-libstdc++ -static-libgcc -Wl,--exclude-libs,ALL
echo "built $OUT/libalva_ref_camera.so"
