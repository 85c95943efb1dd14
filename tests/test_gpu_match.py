"""GPU parity tests (H100): Mapper::matchToMap on flat device arenas through the C ABI vs the CPU oracle and the golden vectors
dumped from the reference's own Mapper.  Exact: identical keypoint -> map point maps."""
import numpy as np
import pytest
import torch

from conftest import golden
from alvaar_b200 import synth
from match_util import oracle_match

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def gpu_match(ctx, p, order, nkp3d):
    idx = {int(i): k for k, i in enumerate(p["mp_id"])}
    kp_mp = np.array([idx.get(int(i), -1) for i in p["kp_id"]], np.int32)
    local_mp = np.array([idx.get(int(i), -1) for i in order], np.int32)
    n_kp = len(kp_mp)
    out = torch.full((n_kp,), -7, dtype=torch.int32, device=DEV)
    dist = torch.zeros(n_kp, dtype=torch.float32, device=DEV)
    cnt = torch.zeros(1, dtype=torch.int32, device=DEV)
    ctx.match_to_map(p["w"], p["h"], 40, [float(v) for v in p["K"]], dev(p["cur_T"]), dev(kp_mp), dev(p["kp_px"]), nkp3d, dev(p["kf_T"]),
                     dev(p["mp_wpt"]), dev(p["mp_is3d"]), dev(p["obs_start"]), dev(p["obs_kf"]), dev(p["obs_px"]), dev(p["desc_start"]),
                     dev(p["desc"]), dev(local_mp), out, dist, cnt)
    torch.cuda.synchronize()
    o = out.cpu().numpy()
    assert int(cnt.item()) == int((o >= 0).sum())
    return {int(p["kp_id"][k]): int(p["mp_id"][o[k]]) for k in range(n_kp) if o[k] >= 0}, dist.cpu().numpy()


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
@pytest.mark.parametrize("nkp3d", [100, 10])
def test_match_golden(gpu_ctx, seed, nkp3d):
    g = golden("match")
    p = synth.make_match_problem(seed, n_frame_kp=150 + 20 * seed, n_local=350 + 50 * seed)
    m, _ = gpu_match(gpu_ctx, p, g[f"s{seed}_{nkp3d}_order"], nkp3d)
    assert sorted(m) == g[f"s{seed}_{nkp3d}_kp"].tolist()
    assert [m[k] for k in sorted(m)] == g[f"s{seed}_{nkp3d}_mp"].tolist()


@pytest.mark.parametrize("seed,nkp,nloc,w,h", [(21, 500, 3000, 1280, 720), (22, 576, 5760, 1280, 720), (23, 1296, 6000, 1920, 1080), (24, 40, 60, 640, 480)])
def test_match_vs_oracle_full_size(gpu_ctx, oracle, seed, nkp, nloc, w, h):
    """C2 / C3-sized maps: frameMaxNumKeypoints keypoints (576 @720p, 1296 @1080p), local map up to 10x that (mapper.cpp:296),
    30 keyframes."""
    p = synth.make_match_problem(seed, w=w, h=h, n_kf=30 if nkp > 100 else 4, n_frame_kp=nkp, n_local=nloc, dup_frac=0.3)
    rng = np.random.default_rng(seed)
    order = p["local_ids"][rng.permutation(len(p["local_ids"]))]
    for nk in (200, 7):
        want = oracle_match(oracle, p, order, nk)
        got, dist = gpu_match(gpu_ctx, p, order, nk)
        assert got == want and len(want) > min(20, nkp // 8)
        assert dist.max() <= 51.0


def test_match_rejects_too_many_keyframes(gpu_ctx):
    import alvaar_b200
    p = synth.make_match_problem(1, n_kf=70)
    with pytest.raises(alvaar_b200.AlvaError):
        gpu_match(gpu_ctx, p, p["local_ids"], 100)
