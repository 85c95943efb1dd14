#!/usr/bin/env bash
# oracle/build_ref_preset.sh -- build oracle/_ref/libalva_ref_preset.so (oracle/ref_preset.cpp) beside libalva_ref.so.
# TEST INFRASTRUCTURE: git-ignored like libalva_ref.so, loaded only by the preset tests and tools/make_golden_presets.py.
# It links against libalva_ref.so (the State / Frame constructors and System::reset it calls are that library's), so it needs
# that library, the configuration oracle/build_ref.sh leaves in $ALVA_REF_PREFIX (default /tmp/probe) and the reference tree
# for its headers; optional like that build -- without it the tests read the tests/golden/*preset* files.
set -euo pipefail
HERE="$(cd "$(dirname "$0")" && pwd)"
REF=${ALVA_REFERENCE:-/root/reference}
P=${ALVA_REF_PREFIX:-/tmp/probe}
OUT="$HERE/_ref"
[ -d "$REF/src/slam/src" ] || { echo "reference tree not found at $REF" >&2; exit 3; }
[ -f "$OUT/libalva_ref.so" ] || { echo "no $OUT/libalva_ref.so: run oracle/build_ref.sh first" >&2; exit 3; }
[ -d "$P/ocv_install/include/opencv4" ] || { echo "no OpenCV build under $P: run oracle/build_ref.sh first" >&2; exit 3; }
INC="-I$REF/src/slam/src -I$REF/src/libs/opencv/modules/highgui/include -I$REF/src/libs/opencv/modules/imgcodecs/include -I$REF/src/libs/opencv/modules/videoio/include -I$REF/src/libs/opengv/include -I$P/ocv_install/include/opencv4 -I$REF/src/libs/eigen -I$REF/src/libs/Sophus \
 -I$P/ceres_install/include -I$P/ceres_install/include/ceres/internal/miniglog"
# OpenCV's core is linked statically as in build_ref_clahe.sh: libalva_ref.so keeps its copy private (--exclude-libs), and the
# inline cv::Mat members of the Frame assignment refer to it
g++ -std=c++20 -O2 -w -fPIC -shared -o "$OUT/libalva_ref_preset.so" "$HERE/ref_preset.cpp" $INC \
  -L"$OUT" -l:libalva_ref.so -Wl,-rpath,'$ORIGIN' \
  -Wl,--start-group "$P"/ocv_install/lib/libopencv_core.a "$P"/ocv_install/lib/opencv4/3rdparty/libzlib.a -Wl,--end-group \
  -lpthread -ldl -static-libstdc++ -static-libgcc -Wl,--exclude-libs,ALL -Wl,--no-undefined
echo "built $OUT/libalva_ref_preset.so"
