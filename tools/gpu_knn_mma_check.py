"""GPU check of the tensor-core Hamming matcher (hamming_mma.cu): raw accumulators of the first tile (dot products for
operand kinds 0 and 1, distances for kind 2) and the final 2-NN lists against numpy, for one shared-memory layout mode
(argv[1]) and operand kind (argv[3]), then timing against the LOP3/POPC kernel on the bench's shape.  Run one mode per
process (a bad descriptor traps the context):  python tools/gpu_knn_mma_check.py 0 time 2"""
import ctypes as C
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import alvaar_b200

mode = int(sys.argv[1]) if len(sys.argv) > 1 else 0
do_time = len(sys.argv) > 2 and sys.argv[2] == "time"
kind = int(sys.argv[3]) if len(sys.argv) > 3 else 1
dev = "cuda:0"
ctx = alvaar_b200.Context(0, torch.cuda.current_stream().cuda_stream)
L = ctx.L
vp, i32 = C.c_void_p, C.c_int
L.alva_debug_knn2_mma.argtypes = [vp, vp, i32, vp, i32, vp, vp]
assert L.alva_set_option(b"knn_mma_mode", mode) == 0
assert L.alva_set_option(b"knn_mma_kind", kind) == 0
P = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731

POP = np.array([bin(i).count("1") for i in range(256)], np.int32)


def ham(q, t):
    return POP[q[:, None, :] ^ t[None, :, :]].sum(-1)


def ref_knn2(q, t):
    d = ham(q, t).astype(np.int64)
    key = d * (1 << 22) + np.arange(t.shape[0])[None, :]
    o = np.argsort(key, axis=1, kind="stable")[:, :2]
    out = np.full((q.shape[0], 4), -1, np.int32)
    out[:, 0] = o[:, 0]
    out[:, 1] = np.take_along_axis(d, o[:, :1], 1)[:, 0]
    if t.shape[0] > 1:
        out[:, 2] = o[:, 1]
        out[:, 3] = np.take_along_axis(d, o[:, 1:2], 1)[:, 0]
    return out


rng = np.random.default_rng(5)
ok_all = True
for (nq, nt) in [(128, 128), (300, 1000), (1000, 2500), (257, 129)]:
    q = rng.integers(0, 256, (nq, 32), dtype=np.uint8)
    t = rng.integers(0, 256, (nt, 32), dtype=np.uint8)
    t[nt // 2] = t[3]                      # duplicate train rows: the tie rule
    q[::5] = t[rng.integers(0, nt, len(q[::5]))]
    dq, dt = torch.from_numpy(q).to(dev), torch.from_numpy(t).to(dev)
    out = torch.full((nq, 4), -7, dtype=torch.int32, device=dev)
    dbg = torch.full((128, 128), -99999, dtype=torch.int32, device=dev)
    rc = L.alva_debug_knn2_mma(ctx.h, P(dq), nq, P(dt), nt, P(out), P(dbg))
    torch.cuda.synchronize()
    if rc != 0:
        print("mode", mode, "rc", rc, L.alva_last_error().decode())
        sys.exit(2)
    g = dbg.cpu().numpy()
    m, n = min(nq, 128), min(nt, 128)
    want = ham(q[:m], t[:n]) if kind == 2 else 256 - 2 * ham(q[:m], t[:n])
    tile_ok = np.array_equal(g[:m, :n], want)
    got = out.cpu().numpy()
    ref = ref_knn2(q, t)
    res_ok = np.array_equal(got, ref)
    print(f"kind {kind} mode {mode} nq {nq} nt {nt}: first tile {'OK' if tile_ok else 'MISMATCH'}  2-NN {'OK' if res_ok else 'MISMATCH'}")
    if not tile_ok:
        bad = np.argwhere(g[:m, :n] != want)
        print("  mismatching cells:", len(bad), "of", m * n, " first:", bad[:5].tolist())
        print("  got[0,:8] ", g[0, :8].tolist(), "\n  want[0,:8]", want[0, :8].tolist())
        print("  got[:8,0] ", g[:8, 0].tolist(), "\n  want[:8,0]", want[:8, 0].tolist())
        # does the produced tile equal the expected one under a row / column permutation?
        rows_match = [int(np.where((want == g[i, :n]).all(1))[0][0]) if (want == g[i, :n]).all(1).any() else -1 for i in range(min(m, 16))]
        print("  got row i == want row:", rows_match)
        print("  value range got", int(g[:m, :n].min()), int(g[:m, :n].max()), "parity-odd cells", int((g[:m, :n] & 1).sum()))
    if not res_ok:
        bad = np.argwhere((got != ref).any(1))[:, 0]
        print("  rows differing:", len(bad), "first", bad[:5].tolist(), got[bad[:3]].tolist(), ref[bad[:3]].tolist())
    ok_all &= tile_ok and res_ok

if ok_all and do_time:
    nb, qcap, live, nt = 64, 1536, 1137, 10000
    q = rng.integers(0, 256, (nb * qcap, 32), dtype=np.uint8)
    t = rng.integers(0, 256, (nt, 32), dtype=np.uint8)
    q[::3] = t[rng.integers(0, nt, len(q[::3]))] ^ (rng.random((len(q[::3]), 32)) < 0.05).astype(np.uint8)
    dq, dt = torch.from_numpy(q).to(dev), torch.from_numpy(t).to(dev)
    counts = torch.from_numpy(rng.integers(live - 100, live + 100, nb).astype(np.int32)).to(dev)
    outs = {}
    for opt in (0, 2):
        assert L.alva_set_option(b"knn_mma", opt) == 0
        out = torch.zeros((nb * qcap, 4), dtype=torch.int32, device=dev)
        for _ in range(3):
            ctx.hamming_knn2_batch(dq, counts, nb, qcap, dt, nt, out)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(10):
            ctx.hamming_knn2_batch(dq, counts, nb, qcap, dt, nt, out)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 10
        nd = float(counts.sum().item()) * nt
        print(f"knn2_batch 64 x ~{live} x {nt}, knn_mma={opt}: {ms * 1000:.1f} us -> {nd / ms / 1e9:.2f} T dist/s")
        outs[opt] = out.cpu().numpy()
    same = np.array_equal(outs[0], outs[2])
    print("tensor-core result == LOP3 result on the bench shape:", same)
    ok_all &= same
    L.alva_set_option(b"knn_mma", 1)
print("RESULT kind", kind, "mode", mode, "PASS" if ok_all else "FAIL")
sys.exit(0 if ok_all else 1)
