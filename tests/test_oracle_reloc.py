"""CPU: the relocalisation oracle (oracle/reloc_oracle.c) -- the grouped Hamming 2-NN against a numpy brute force, the match
rules, and P3P-RANSAC against P3P-LMedS on correspondences with a majority of outliers."""
import numpy as np
import pytest

from alvaar_b200 import synth
from reloc_util import P, knn2_grouped_numpy, knn2_grouped_oracle, random_table, reloc_oracle_lib


@pytest.fixture(scope="module")
def L():
    return reloc_oracle_lib()


CASES = ["random", "groups_of_1", "groups_of_30", "one_group", "empty_table", "ties", "empty_groups"]


@pytest.mark.parametrize("case", CASES)
def test_knn2_grouped_oracle_equals_brute_force(L, case):
    rng = np.random.default_rng(11 + CASES.index(case))
    if case == "random":
        q, ds, d = random_table(rng, 120, 12, 200)
    elif case == "groups_of_1":
        q, ds, d = random_table(rng, 150, 1, 100)
    elif case == "groups_of_30":
        q, ds, d = random_table(rng, 40, 30, 100, min_rows=30)
    elif case == "one_group":
        q, ds, d = random_table(rng, 1, 7, 50)
    elif case == "empty_table":
        q, ds, d = rng.integers(0, 256, (20, 32), dtype=np.uint8), np.zeros(1, np.int32), np.zeros((0, 32), np.uint8)
    elif case == "ties":
        # every group holds copies of a few descriptors: equal distances across groups everywhere
        base = rng.integers(0, 256, (3, 32), dtype=np.uint8)
        d = base[rng.integers(0, 3, 90)]
        ds = np.arange(0, 91, 3, dtype=np.int32)
        q = base[rng.integers(0, 3, 40)] ^ np.packbits(rng.random((40, 256)) < 0.02, axis=1)
    else:   # groups without rows between the others (never candidates)
        rows = rng.integers(0, 4, 80)
        ds = np.concatenate([[0], np.cumsum(rows)]).astype(np.int32)
        d = rng.integers(0, 256, (int(ds[-1]), 32), dtype=np.uint8)
        q = d[rng.integers(0, len(d), 30)] ^ np.packbits(rng.random((30, 256)) < 0.05, axis=1)
    got = knn2_grouped_oracle(L, q, ds, d)
    want = knn2_grouped_numpy(q, ds, d)
    assert (got == want).all()
    if case == "empty_table":
        assert (got == -1).all()
    if case == "one_group":
        assert (got[:, 0] == 0).all() and (got[:, 2] == -1).all() and (got[:, 3] == -1).all()
    if case == "ties":
        assert ((got[:, 1] == got[:, 3]) & (got[:, 0] < got[:, 2])).any()   # ties did occur and went to the lower group


def test_reloc_select_rules(L):
    """gate <= 51, 5 d0 < 4 d1, one query per group (smallest distance, then lowest query index), ascending query order"""
    knn = np.array([[0, 10, 1, 40],    # kept for group 0?  10 < 0.8 * 40: passes; but query 3 is closer to group 0
                    [1, 52, 2, 90],    # gate
                    [2, 40, 3, 50],    # 5 * 40 = 200 == 4 * 50: fails the strict ratio test
                    [0, 5, 4, 60],     # group 0's best
                    [5, 30, -1, -1],   # a single candidate passes the ratio test
                    [6, 20, 7, 30],    # 100 < 120: passes
                    [6, 20, 8, 40],    # same group and distance as query 5: the lower index (5) wins
                    [-1, -1, -1, -1]], np.int32)
    mq = np.zeros(8, np.int32); mg = np.zeros(8, np.int32)
    n = L.orc_reloc_select(P(knn), len(knn), 9, 51, P(mq), P(mg))
    assert mq[:n].tolist() == [3, 4, 5] and mg[:n].tolist() == [0, 5, 6]


def _solve(fn, pr, n, fx, max_iter):
    T = np.zeros(12); out = np.zeros(n, np.uint8); info = np.zeros(4)
    ok = fn(P(pr["bv"]), P(pr["X"]), n, max_iter, 3.0, fx, fx, 12345, P(T), P(out), P(info))
    return ok, T, out, info


def _T12(pose):
    R = synth.quat_to_R(pose[3:])
    return np.concatenate([R, pose[:3, None]], 1).reshape(-1)


# The share of gross outliers (25-px errors) at which LMedS was seen to break down on this problem.  With noise-free inliers
# it still found the pose at 60, 65, 70 and 75 % (seed 3); at 80 % (seed 4) its pose is 7e-2 off while RANSAC's is exact.
OUTLIER_SHARE, SEED = 0.8, 4


def test_ransac_recovers_where_lmeds_breaks_down(L):
    n, w, h = 300, 1280, 720
    pr = synth.make_pose_problem(n=n, seed=SEED, w=w, h=h, noise_px=0.0, outlier_frac=OUTLIER_SHARE)
    fx = float(pr["K"][0])
    want = _T12(pr["pose_true"])
    ok_l, T_l, _, _ = _solve(L.lmeds, pr, n, fx, 100)
    assert not ok_l or np.abs(T_l - want).max() > 1e-2, "LMedS survived this outlier share: raise OUTLIER_SHARE"
    ok_r, T_r, out_r, info = _solve(L.orc_p3p_ransac, pr, n, fx, 512)
    assert ok_r == 1 and info[1] >= 0
    assert np.abs(T_r - want).max() < 1e-6
    # the inlier set is exactly what the true pose classifies as inliers at the same threshold
    focal = np.float32((np.float32(fx) + np.float32(fx)) / 2)
    thr = 1.0 - np.cos(np.arctan(np.float32(3.0) / focal, dtype=np.float32), dtype=np.float32)
    R = synth.quat_to_R(pr["pose_true"][3:])
    q = (pr["X"] - pr["pose_true"][:3]) @ R
    dist = 1.0 - (q / np.linalg.norm(q, axis=1, keepdims=True) * pr["bv"]).sum(1)
    assert ((dist <= float(thr)) == (out_r == 0)).all()
    assert (out_r == 0).sum() >= (~pr["outlier_true"]).sum()
