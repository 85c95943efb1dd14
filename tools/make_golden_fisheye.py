#!/usr/bin/env python3
"""Dump the fisheye golden vectors (committed) from OpenCV's own cv::fisheye (oracle/_ref/libalva_ref_fisheye.so,
oracle/build_ref_fisheye.sh, over the reference's vendored OpenCV 4.5.5).

tests/golden/fisheye.npz: for every case of tests/fisheye_util.CASES (a mild wide-angle lens at 640x480, a ~180 degree lens at
1280x720, and a lens whose Newton iteration fails or flips over much of the image, so that the (-1e6, -1e6) branch fires):
  {name}/K, {name}/D               the camera matrix and the coefficients
  {name}/px, {name}/X              SHA-256 digests (tests/ref_golden.digest) of the seeded inputs: ~8e4 pixels inside, at the
                                   corners of and up to 100 px outside the image, and the principal point; ~2.4e4 camera points
                                   up to 86 degrees off the axis, behind the camera (z < 0), on its plane (z = 0) and on the axis
  {name}/unpx, {name}/uv           digests of cv::fisheye::undistortPoints / projectPoints' float results (NaNs canonicalised)
  {name}/unpx_diff, /uv_diff       the flat indices where camera_model.h's float bits differ from OpenCV's (the rounding-boundary
  {name}/unpx_ref32, /unpx_ref64   exemption of tests/test_oracle_fisheye.py), with OpenCV's float there and the double it was
  {name}/uv_ref32, /uv_ref64       rounded from -- so that the test can check the exemption without the library
  {name}/n_fail                    pixels OpenCV returns as (-1e6, -1e6)
Run from the repository root after oracle/build_ref.sh and oracle/build_ref_fisheye.sh."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from camera_util import cdigest  # noqa: E402
from fisheye_util import CASES, case_K, case_pixels, case_points, cpu_system_lib, ref_lib, rounding_exempt, run_points, run_ref  # noqa: E402
from ref_golden import digest  # noqa: E402


def main():
    R = ref_lib()
    if R is None:
        sys.exit("oracle/_ref/libalva_ref_fisheye.so is not built: run oracle/build_ref.sh and oracle/build_ref_fisheye.sh")
    S = cpu_system_lib()
    d = {}
    for k, (name, w, h, _, _) in enumerate(CASES):
        K, D = case_K(k)
        px, X = case_pixels(k), case_points(k)
        ru, ru64 = run_ref(R.ref_fisheye_undistort_points, px, K, D)
        rp, rp64 = run_ref(R.ref_fisheye_project_points, X, K, D)
        hu, hp = run_points(S.cpu_fish_undistort_points, px, K, D), run_points(S.cpu_fish_project_points, X, K, D)
        d[f"{name}/K"], d[f"{name}/D"] = K, D
        d[f"{name}/px"], d[f"{name}/X"] = digest(px), digest(X)
        d[f"{name}/unpx"], d[f"{name}/uv"] = cdigest(ru), cdigest(rp)
        for key, mine, r32, r64 in (("unpx", hu, ru, ru64), ("uv", hp, rp, rp64)):
            idx, _ = rounding_exempt(mine, r32, r64)
            d[f"{name}/{key}_diff"] = idx.astype(np.int64)
            d[f"{name}/{key}_ref32"] = r32.ravel()[idx]
            d[f"{name}/{key}_ref64"] = r64.ravel()[idx]
        d[f"{name}/n_fail"] = np.int64(((ru[:, 0] == -1e6) & (ru[:, 1] == -1e6)).sum())
        print(f"{name}: {len(px)} pixels ({int(d[name + '/n_fail'])} fail), {len(X)} points, "
              f"{len(d[name + '/unpx_diff'])} + {len(d[name + '/uv_diff'])} float results differ from the header")
    out = os.path.join(ROOT, "tests", "golden", "fisheye.npz")
    np.savez_compressed(out, **d)
    print("wrote", out)


if __name__ == "__main__":
    main()
