#!/usr/bin/env python3
"""Dump the full-vector lens golden vectors (committed) from OpenCV's own cv::undistortPoints / cv::projectPoints
(oracle/_ref/libalva_ref_distortion_full.so, oracle/build_ref_distortion_full.sh, over the reference's vendored OpenCV 4.5.5).

tests/golden/camera_full.npz: for every lens of tests/camera_full_util.CASES (k3 at 5 coefficients, a rational wide-angle at 8,
a thin prism at 12, a tilted sensor at 14, and a lens that folds back inside the image, so that icdist < 0 fires):
  {name}/K, {name}/D               the camera matrix and the coefficients
  {name}/px, {name}/X              SHA-256 digests (tests/ref_golden.digest) of the seeded inputs
  {name}/unpx, {name}/uv           digests of OpenCV's float results (NaNs canonicalised)
  {name}/unpx_diff, /uv_diff       the flat indices where camera_model.h's float bits differ from OpenCV's, with OpenCV's float
  {name}/*_ref32, /*_ref64         there and the double it was rounded from (the rounding-boundary exemption)
  {name}/n_fold                    pixels whose iteration meets icdist < 0 (the pinhole fallback)
Run from the repository root after oracle/build_ref.sh and oracle/build_ref_distortion_full.sh."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from camera_full_util import CASES, case_K, case_pixels, case_points, host_lib, n_fold, ref_lib, rounding_exempt, run_points, run_ref  # noqa: E402
from camera_util import cdigest  # noqa: E402
from ref_golden import digest  # noqa: E402


def main():
    R = ref_lib()
    if R is None:
        sys.exit("oracle/_ref/libalva_ref_distortion_full.so is not built: run oracle/build_ref.sh and oracle/build_ref_distortion_full.sh")
    H = host_lib()
    d = {}
    for k, (name, w, h, _) in enumerate(CASES):
        K, D = case_K(k)
        px, X = case_pixels(k), case_points(k)
        ru, ru64 = run_ref(R.ref_full_undistort_points, px, K, D)
        rp, rp64 = run_ref(R.ref_full_project_points, X, K, D)
        hu, hp = run_points(H.cpu_full_undistort_points, px, K, D), run_points(H.cpu_full_project_points, X, K, D)
        d[f"{name}/K"], d[f"{name}/D"] = K, D
        d[f"{name}/px"], d[f"{name}/X"] = digest(px), digest(X)
        d[f"{name}/unpx"], d[f"{name}/uv"] = cdigest(ru), cdigest(rp)
        for key, mine, r32, r64 in (("unpx", hu, ru, ru64), ("uv", hp, rp, rp64)):
            idx, _ = rounding_exempt(mine, r32, r64)
            d[f"{name}/{key}_diff"] = idx.astype(np.int64)
            d[f"{name}/{key}_ref32"] = r32.ravel()[idx]
            d[f"{name}/{key}_ref64"] = r64.ravel()[idx]
        d[f"{name}/n_fold"] = np.int64(n_fold(px, K, D))
        print(f"{name}: {len(px)} pixels ({int(d[name + '/n_fold'])} fold back), {len(X)} points, "
              f"{len(d[name + '/unpx_diff'])} + {len(d[name + '/uv_diff'])} float results differ from the header")
    out = os.path.join(ROOT, "tests", "golden", "camera_full.npz")
    np.savez_compressed(out, **d)
    print("wrote", out)


if __name__ == "__main__":
    main()
