"""ctypes binding of the alva_pipeline object (include/alva_b200.h): the whole per-frame hot path on batches."""
import ctypes as C

import numpy as np

from .lib import AlvaError, lib


class _Config(C.Structure):
    _fields_ = [("w", C.c_int), ("h", C.c_int), ("batch", C.c_int), ("fast_thr", C.c_int), ("nfeatures", C.c_int),
                ("orb_flags", C.c_int), ("map_size", C.c_int), ("kf_interval", C.c_int), ("ba_nkf", C.c_int),
                ("ba_nlm", C.c_int), ("ba_nobs", C.c_int), ("ba_max_iter", C.c_int), ("ba_huber", C.c_double),
                ("derivatives", C.c_int), ("reserved", C.c_int)]


BUF = dict(l0=0, l1=1, l2=2, l3=3, blur=4, keys=5, counts=6, sel=7, selcounts=8, pts=9, angles=10, desc=11, kept=12,
           matches=13, ba_poses=14, ba_invd=15, ba_summary=16, d0=17, d1=18, d2=19, d3=20)


class Pipeline:
    def __init__(self, ctx, w, h, batch, fast_thr=20, nfeatures=1000, orb_flags=2, map_size=0, kf_interval=0, ba_nkf=0,
                 ba_nlm=0, ba_nobs=0, ba_max_iter=5, ba_huber=0.0, derivatives=False):
        self.ctx, self.L = ctx, lib()
        L = self.L
        L.alva_pipeline_create.restype = C.c_void_p
        L.alva_pipeline_create.argtypes = [C.c_void_p, C.POINTER(_Config)]
        L.alva_pipeline_destroy.argtypes = [C.c_void_p]
        L.alva_pipeline_set_map.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        L.alva_pipeline_set_ba.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 9
        L.alva_pipeline_step_dev.argtypes = [C.c_void_p, C.c_void_p]
        L.alva_pipeline_step_host.argtypes = [C.c_void_p] * 6
        L.alva_pipeline_submit_host.argtypes = [C.c_void_p] * 6
        L.alva_pipeline_wait.argtypes = [C.c_void_p]
        L.alva_pipeline_profile.argtypes = [C.c_void_p, C.c_int]
        L.alva_pipeline_frontend_ms.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        L.alva_pipeline_info.argtypes = [C.c_void_p, C.c_void_p]
        L.alva_pipeline_buffer.restype = C.c_void_p
        L.alva_pipeline_buffer.argtypes = [C.c_void_p, C.c_int]
        self.cfg = _Config(w, h, batch, fast_thr, nfeatures, orb_flags, map_size, kf_interval, ba_nkf, ba_nlm, ba_nobs,
                           ba_max_iter, ba_huber, 1 if derivatives else 0, 0)
        h_ = L.alva_pipeline_create(ctx.h, C.byref(self.cfg))
        if not h_:
            raise AlvaError(L.alva_last_error().decode())
        self.h = C.c_void_p(h_)
        info = (C.c_int32 * 4)()
        L.alva_pipeline_info(self.h, info)
        self.fcap, self.kcap, self.nprob, self.map_size = list(info)
        self._keep = []

    def _chk(self, rc):
        if rc < 0:
            raise AlvaError(f"rc={rc}: {self.L.alva_last_error().decode()}")
        return rc

    def close(self):
        if getattr(self, "h", None):
            self.L.alva_pipeline_destroy(self.h)
            self.h = None

    def set_map(self, desc):
        d = np.ascontiguousarray(desc, np.uint8)
        self._chk(self.L.alva_pipeline_set_map(self.h, d.ctypes.data_as(C.c_void_p), len(d)))

    def set_ba(self, slot, pb):
        arrs = [np.ascontiguousarray(pb[k]) for k in ("calib", "poses", "pose_const", "invd", "anch_kf", "anch_uv", "obs_kf",
                                                      "obs_lm", "obs_uv")]
        self._chk(self.L.alva_pipeline_set_ba(self.h, slot, *[a.ctypes.data_as(C.c_void_p) for a in arrs]))

    def step_dev(self, rgba_dev):
        self._chk(self.L.alva_pipeline_step_dev(self.h, C.c_void_p(rgba_dev.data_ptr())))

    def step_host(self, rgba_host, nfeat=None, matches=None, ba_poses=None, ba_summary=None):
        p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None  # noqa: E731
        self._chk(self.L.alva_pipeline_step_host(self.h, p(rgba_host), p(nfeat), p(matches), p(ba_poses), p(ba_summary)))

    def submit_host(self, rgba_host, nfeat=None, matches=None, ba_poses=None, ba_summary=None):
        """asynchronous step_host: returns at once; at most two outstanding; pair every submit with a wait()"""
        p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None  # noqa: E731
        self._keep.append((rgba_host, nfeat, matches, ba_poses, ba_summary))
        self._keep = self._keep[-4:]
        self._chk(self.L.alva_pipeline_submit_host(self.h, p(rgba_host), p(nfeat), p(matches), p(ba_poses), p(ba_summary)))

    def wait(self):
        self._chk(self.L.alva_pipeline_wait(self.h))

    def profile(self, on):
        self._chk(self.L.alva_pipeline_profile(self.h, 1 if on else 0))

    def drain(self):
        """join every BA chain still in flight ("pipeline_ba_lag" = 1 leaves the last step's) into the context stream"""
        self._chk(self.L.alva_pipeline_drain(self.h))

    def graph_stats(self):
        """(CUDA graphs captured so far, re-captures after a workspace or option change included; graph launches so far;
        capture failed -> direct launches)"""
        out = (C.c_int32 * 3)()
        self.L.alva_pipeline_graph_stats.argtypes = [C.c_void_p, C.c_void_p]
        self._chk(self.L.alva_pipeline_graph_stats(self.h, out))
        return int(out[0]), int(out[1]), bool(out[2])

    def frontend_ms(self, n):
        n = min(n, 64)
        out = (C.c_float * n)()
        m = self._chk(self.L.alva_pipeline_frontend_ms(self.h, out, n))
        return [out[i] for i in range(m)]

    def buffer(self, name, shape, dtype):
        """torch view (no copy) of an internal device buffer -- tests only."""
        import torch
        ptr = self.L.alva_pipeline_buffer(self.h, BUF[name])
        n = int(np.prod(shape))
        itemsize = torch.empty(0, dtype=dtype).element_size()

        class _Holder:
            pass
        hold = _Holder()
        hold.__cuda_array_interface__ = {"shape": (n * itemsize,), "typestr": "|u1", "data": (ptr, False), "version": 2}
        t = torch.as_tensor(hold, device=f"cuda:{self.ctx.device}")
        return t.view(dtype).reshape(shape)
