#!/usr/bin/env bash
# oracle/build_ref_distortion_full.sh -- build oracle/_ref/libalva_ref_distortion_full.so (oracle/ref_distortion_full.cpp over the
# reference's vendored OpenCV 4.5.5 calib3d: cv::undistortPoints / cv::projectPoints with the whole distortion vector) beside
# libalva_ref.so.
# TEST INFRASTRUCTURE: git-ignored like libalva_ref.so, loaded only by the full-vector lens tests and
# tools/make_golden_distortion_full.py.  Needs the OpenCV build oracle/build_ref.sh leaves in $ALVA_REF_PREFIX (default
# /tmp/probe); optional like that build -- without it the tests read tests/golden/camera_full.npz.
set -euo pipefail
HERE="$(cd "$(dirname "$0")" && pwd)"
P=${ALVA_REF_PREFIX:-/tmp/probe}
OUT="$HERE/_ref"
[ -f "$P/ocv_install/lib/libopencv_calib3d.a" ] || { echo "no OpenCV build under $P: run oracle/build_ref.sh first" >&2; exit 3; }
mkdir -p "$OUT"
g++ -std=c++17 -O2 -w -fPIC -shared -o "$OUT/libalva_ref_distortion_full.so" "$HERE/ref_distortion_full.cpp" -I"$P/ocv_install/include/opencv4" \
  -Wl,--start-group "$P"/ocv_install/lib/libopencv_calib3d.a "$P"/ocv_install/lib/libopencv_features2d.a \
  "$P"/ocv_install/lib/libopencv_flann.a "$P"/ocv_install/lib/libopencv_imgproc.a "$P"/ocv_install/lib/libopencv_core.a \
  "$P"/ocv_install/lib/opencv4/3rdparty/libzlib.a -Wl,--end-group \
  -lpthread -ldl -static-libstdc++ -static-libgcc -Wl,--exclude-libs,ALL
echo "built $OUT/libalva_ref_distortion_full.so"
