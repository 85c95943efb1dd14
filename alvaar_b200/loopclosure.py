"""ctypes binding of the cross-stream loop-closure detector (alva_lc_*, csrc/loopclosure.cu) plus the NCCL exchange of the
keyframe blocks (torch.distributed all-gather on the caller's current stream).  Wire format of a block: include/alva_b200.h."""
import ctypes as C

import numpy as np

from .lib import AlvaError, lib

MAGIC, VERSION, HEADER_BYTES, PAIR_CAP = 0x464B4C41, 1, 64, 512


class LcConfig(C.Structure):
    _fields_ = [("n_max", C.c_int32), ("kf_per_step", C.c_int32), ("world", C.c_int32), ("rank", C.c_int32), ("min_matches", C.c_int32),
                ("max_dist", C.c_int32), ("ratio_num", C.c_int32), ("ratio_den", C.c_int32), ("min_consecutive", C.c_int32),
                ("min_inliers", C.c_int32), ("err_px", C.c_float), ("fx_hint", C.c_float), ("fy_hint", C.c_float)]


class LcEvent(C.Structure):
    _fields_ = [("local_kf", C.c_int32), ("remote_rank", C.c_int32), ("remote_kf", C.c_int32), ("n_matches", C.c_int32),
                ("n_inliers", C.c_int32), ("consecutive", C.c_int32), ("Rt", C.c_double * 12)]


def block_bytes(n_max):
    return HEADER_BYTES + 40 * n_max


class LoopClosure:
    """One detector per rank.  `ctx`: the alvaar_b200.Context whose stream the exchange and the matching run on (a side stream, so
    that the collective never sits on the per-frame path)."""

    def __init__(self, ctx, n_max, kf_per_step, world, rank, K4, **kw):
        self.L = lib()
        L = self.L
        L.alva_lc_create.restype = C.c_void_p
        L.alva_lc_create.argtypes = [C.c_void_p, C.c_void_p]
        L.alva_lc_destroy.argtypes = [C.c_void_p]
        L.alva_lc_block_bytes.restype = C.c_size_t
        L.alva_lc_pack.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        L.alva_lc_detect.argtypes = [C.c_void_p, C.c_void_p]
        L.alva_lc_poll.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
        L.alva_lc_last_scores.argtypes = [C.c_void_p, C.c_void_p]
        cfg = LcConfig(n_max=n_max, kf_per_step=kf_per_step, world=world, rank=rank, fx_hint=float(K4[0]), fy_hint=float(K4[1]), **kw)
        self.ctx, self.n_max, self.K, self.world, self.rank = ctx, n_max, kf_per_step, world, rank
        self.K4 = np.asarray(K4, np.float32).copy()
        self.block_bytes = block_bytes(n_max)
        assert int(L.alva_lc_block_bytes(n_max)) == self.block_bytes
        h = L.alva_lc_create(ctx.h, C.byref(cfg))
        if not h:
            raise AlvaError(L.alva_last_error().decode())
        self.h = C.c_void_p(h)
        self.seq = 0

    def close(self):
        if getattr(self, "h", None):
            self.L.alva_lc_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _chk(self, rc):
        if rc < 0:
            raise AlvaError(f"rc={rc}: {self.L.alva_last_error().decode()}")
        return rc

    def pack(self, desc, pts, counts, kf_frames, send, on=None):
        """desc [nframes, cap, 32] u8, pts [nframes, cap, 2] f32, counts [nframes] i32, kf_frames [K] i32 (device tensors) ->
        send (device u8 tensor of K * block_bytes).  on: the alvaar_b200.Context whose stream runs the pack (default: the detector's)"""
        p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
        self.L.alva_lc_pack_on.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
        self._chk(self.L.alva_lc_pack_on(self.h, on.h if on is not None else None, p(desc), p(pts), p(counts), int(desc.shape[1]), p(kf_frames),
                                         self.seq, self.K4.ctypes.data_as(C.c_void_p), p(send)))
        self.seq += self.K

    def detect(self, gathered):
        self.L.alva_lc_inflight.argtypes = [C.c_void_p]
        if self.L.alva_lc_inflight(self.h) >= 3:          # at most 4 steps in flight: drain before enqueueing more
            self.backlog = getattr(self, "backlog", []) + self.poll(wait=True)
        self._chk(self.L.alva_lc_detect(self.h, C.c_void_p(gathered.data_ptr())))

    def exchange_and_detect(self, send, gathered):
        """all-gather of the step's blocks over the process group (NCCL over NVLink on a GPU job), then detection on them"""
        import torch.distributed as dist
        dist.all_gather_into_tensor(gathered, send)
        self.detect(gathered)

    def poll(self, wait=False, cap=64):
        ev = (LcEvent * cap)()
        n = self._chk(self.L.alva_lc_poll(self.h, ev, cap, 1 if wait else 0))
        pre, self.backlog = getattr(self, "backlog", []), []
        return pre + [dict(local_kf=e.local_kf, remote_rank=e.remote_rank, remote_kf=e.remote_kf, n_matches=e.n_matches, n_inliers=e.n_inliers,
                     consecutive=e.consecutive, Rt=np.array(list(e.Rt)).reshape(3, 4)) for e in ev[:n]]

    def last_scores(self):
        """[K, world, 4]: putative matches, verdict (0 too few matches / check failed, 1 geometric check passed, 2 enough matches but not
        the step's newest keyframe: not checked), inliers, remote keyframe sequence number"""
        out = np.zeros((self.K, self.world, 4))
        self._chk(self.L.alva_lc_last_scores(self.h, out.ctypes.data_as(C.c_void_p)))
        return out

    def last_matches(self):
        """internal state of the last step (tests / diagnostics): nn [K, world, n_max, 4] = (idx0, dist0, idx1, dist1) of the 2-NN, -1
        where there is none, defined below the local live count; npair [K, world] = correspondences of the geometric check;
        bv_local, bv_remote [K, world, PAIR_CAP, 3] = bearing vectors of the putative matches in local-index order"""
        nn = np.zeros((self.K, self.world, self.n_max, 4), np.int32)
        npair = np.zeros((self.K, self.world), np.int32)
        bvl = np.zeros((self.K, self.world, PAIR_CAP, 3))
        bvr = np.zeros((self.K, self.world, PAIR_CAP, 3))
        self.L.alva_lc_last_matches.argtypes = [C.c_void_p] * 5
        self._chk(self.L.alva_lc_last_matches(self.h, *(a.ctypes.data_as(C.c_void_p) for a in (nn, npair, bvl, bvr))))
        return nn, npair, bvl, bvr
