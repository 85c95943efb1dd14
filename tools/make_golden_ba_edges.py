"""Write tests/golden/ba_edges.npz: what ceres::Solve with the reference's cost functor (oracle/_ref/libalva_ref.so, built by
oracle/build_ref.sh) computes for the widest local-BA problem of tests/test_oracle_ba_edges.py -- 21 free poses (a 126-wide
reduced camera system) among 140 keyframes, tracks of 20 observations -- through ref_ba_solve and ref_ba_local.  The
problem itself is regenerated from its seed by tests/ba_util.py; the file keeps a digest of it so that a change of the
generator is caught instead of compared against outputs of another problem.

    python tools/make_golden_ba_edges.py        (needs oracle/_ref/libalva_ref.so)"""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import ba_util as B  # noqa: E402


def main():
    so = os.path.join(ROOT, "oracle", "_ref", "libalva_ref.so")
    if not os.path.exists(so):
        sys.exit(f"{so} is not built: run oracle/build_ref.sh first")
    R = C.CDLL(so)
    R.ref_config(0, 1)
    pb = B.wide_problem()
    out = B.ceres_outputs(R, pb)
    out["problem_digest"] = B.problem_digest(pb)
    path = os.path.join(ROOT, "tests", "golden", "ba_edges.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {B.nfree(pb)} free poses, {len(pb['poses'])} keyframes, {len(pb['obs_lm'])} observations; "
          f"solve summary {out['solve_summary'][:5]}, local summary {out['local_summary']}")


if __name__ == "__main__":
    main()
