"""GPU test (H100), deliberately the LAST gpu test file in collection order: the experimental front-end instantiation
(alva_set_option("frontend_antipodal", 1)) against the default kernel.  Kept apart so that nothing else shares a process state
with an experimental kernel before it has been seen on a GPU."""
import numpy as np
import pytest
import torch

from alvaar_b200 import synth

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def test_frontend_antipodal_variant_matches_default(gpu_ctx):
    """The experimental pre-test variant (alva_set_option("frontend_antipodal", 1); fast_swar.h -- 8 of the 16 ring flag words
    assembled from their antipodal partners) must return exactly the default kernel's corners (which the tests above pin to the
    reference).  Its logic is checked on the CPU by host emulation (tests/test_fast_swar_host.py); it has not been validated on a
    GPU yet, so a mismatch is reported as XFAIL instead of failing the suite -- the default path does not depend on it."""
    n, w, h = 4, 1280, 720
    frames, _ = synth.make_frames(n, w, h)
    d_in = dev(frames)
    cap = 32768
    res = []
    try:
        for opt, thr in ((0, 20), (1, 20), (0, 150), (1, 150), (0, 7), (1, 7)):
            gpu_ctx.L.alva_set_option(b"frontend_antipodal", opt)
            keys = torch.zeros((n, cap), dtype=torch.int32, device=DEV)
            counts = torch.zeros(n, dtype=torch.int32, device=DEV)
            l0 = torch.zeros((n, h, w), dtype=torch.uint8, device=DEV)
            l1 = torch.zeros((n, h // 2, w // 2), dtype=torch.uint8, device=DEV)
            gpu_ctx.frontend(d_in, w, h, n, l0, l1, None, None, thr, keys, counts, cap, True)
            torch.cuda.synchronize()
            res.append((keys.cpu().numpy(), counts.cpu().numpy(), l0.cpu().numpy(), l1.cpu().numpy()))
    finally:
        gpu_ctx.L.alva_set_option(b"frontend_antipodal", 0)
    for a, b in ((res[0], res[1]), (res[2], res[3]), (res[4], res[5])):
        same = (a[1] == b[1]).all() and all((a[0][f, :a[1][f]] == b[0][f, :b[1][f]]).all() for f in range(n)) and (a[2] == b[2]).all() and (a[3] == b[3]).all()
        if not same:
            pytest.xfail("experimental antipodal pre-test differs from the default kernel on this GPU")
    assert res[0][1].min() > 5000


@pytest.mark.parametrize("w,h,n,thr", [(1280, 720, 3, 20), (1920, 1080, 2, 20), (640, 480, 2, 7), (1280, 720, 1, 150), (128, 64, 2, 20),
                                       (256, 200, 2, 30)])
def test_frontend_variant2_matches_round1_kernel(gpu_ctx, w, h, n, thr):
    """frontend_tile_kernel_v2 (the default since round 2: lean gray phase, 4-wide pyramid, antipodal pre-test, transposed
    compaction, corner queue) against the round-1 kernel (alva_set_option("frontend_variant", 0)), which the parity tests of
    round 1 pinned to the reference: identical gray, L1 and corner lists; also in gray-input mode (alva_k_fast9)."""
    frames, _ = synth.make_frames(n, w, h)
    d_in = dev(frames)
    cap = max(32768, w * h // 16)
    res = []
    try:
        for var in (0, 2):
            assert gpu_ctx.L.alva_set_option(b"frontend_variant", var) == 0
            keys = torch.zeros((n, cap), dtype=torch.int32, device=DEV)
            counts = torch.zeros(n, dtype=torch.int32, device=DEV)
            l0 = torch.zeros((n, h, w), dtype=torch.uint8, device=DEV)
            l1 = torch.zeros((n, (h + 1) // 2, (w + 1) // 2), dtype=torch.uint8, device=DEV)
            gpu_ctx.frontend(d_in, w, h, n, l0, l1, None, None, thr, keys, counts, cap, True)
            k2 = torch.zeros((n, cap), dtype=torch.int32, device=DEV)
            c2 = torch.zeros(n, dtype=torch.int32, device=DEV)
            gpu_ctx.fast9(l0, w, h, n, thr, k2, c2, cap, True)
            torch.cuda.synchronize()
            res.append((keys.cpu().numpy(), counts.cpu().numpy(), l0.cpu().numpy(), l1.cpu().numpy(), k2.cpu().numpy(), c2.cpu().numpy()))
    finally:
        gpu_ctx.L.alva_set_option(b"frontend_variant", 2)
    a, b = res
    assert (a[2] == b[2]).all() and (a[3] == b[3]).all()
    assert (a[1] == b[1]).all() and (a[5] == b[5]).all() and (a[1] == a[5]).all()
    for f in range(n):
        assert (a[0][f, :a[1][f]] == b[0][f, :b[1][f]]).all()
        assert (a[4][f, :a[5][f]] == b[4][f, :b[5][f]]).all()
        assert (a[0][f, :a[1][f]] == a[4][f, :a[5][f]]).all()
    if thr <= 30 and w >= 256:
        assert a[1].min() > 100
