"""The reference's outputs that the *_live_reference / *_vs_reference tests compare with.

With oracle/_ref/libalva_ref.so built in the tree they are computed live; without it they are read from
tests/golden/ref_live.npz, which holds what the reference computed for exactly the same seeded inputs.
ALVA_RECORD_REF=1 (with the reference built) rewrites the stored entries.  Outputs too large to store are kept as
SHA-256 digests of their bytes (`digest`), and the tests compare digests: still bit for bit."""
import ctypes as C
import hashlib
import os

import numpy as np

STORE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_live.npz")
_cache = {}


def digest(a):
    a = np.ascontiguousarray(a)
    h = hashlib.sha256(f"{a.dtype.str}{a.shape}".encode())
    h.update(a.tobytes())
    return np.frombuffer(h.digest(), np.uint8).copy()


def _stored():
    if "all" not in _cache:
        _cache["all"] = dict(np.load(STORE)) if os.path.exists(STORE) else {}
    return _cache["all"]


def ref_outputs(ref, key, compute):
    """compute(ref) -> {name: array} from the live reference, or the stored arrays of `key` when it is not built here."""
    if ref is not None:
        out = {k: np.asarray(v) for k, v in compute(ref).items()}
        if os.environ.get("ALVA_RECORD_REF") == "1":
            allv = _stored()
            for k in [k for k in allv if k.startswith(key + "/")]:
                del allv[k]
            allv.update({f"{key}/{k}": v for k, v in out.items()})
            np.savez_compressed(STORE, **allv)
        return out
    out = {k[len(key) + 1:]: v for k, v in _stored().items() if k.startswith(key + "/")}
    assert out, f"no stored reference outputs for {key}: build oracle/_ref and record them (ALVA_RECORD_REF=1)"
    return out


class EssentialHook:
    """The reference's compute5ptEssentialMatrix (ref_essential_5pt) as the initialisation hook of the CPU state machine
    (cpu_system_set_essential_hook): live when the reference is built, else replaying what it returned, call by call, for the
    same inputs (the inputs' digest is stored and checked).  `ptr` is the function pointer to hand over; call `finish()` after
    the run."""
    PROTO = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_int, C.c_float, C.c_float,
                        C.c_void_p, C.c_void_p)

    def __init__(self, ref, key):
        self.ref, self.key, self.calls, self.errors = ref, key, [], []
        if ref is not None:
            ref.ref_essential_5pt.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_int, C.c_float, C.c_float,
                                              C.c_void_p, C.c_void_p]
        else:
            self.stored = ref_outputs(None, key, None)
        self.cb = self.PROTO(self._call)
        self.ptr = C.cast(self.cb, C.c_void_p)

    def _call(self, b1, b2, n, max_iter, err, opt, fx, fy, Rt, outl):
        try:
            i = len(self.calls)
            ins = digest(np.concatenate([np.ctypeslib.as_array((C.c_double * (3 * n)).from_address(b1)),
                                         np.ctypeslib.as_array((C.c_double * (3 * n)).from_address(b2)),
                                         np.array([max_iter, err, opt, fx, fy], np.float64)]))
            if self.ref is not None:
                ok = self.ref.ref_essential_5pt(b1, b2, n, max_iter, err, opt, fx, fy, Rt, outl)
                self.calls.append({"in": ins, "ok": np.int32(ok), "Rt": np.ctypeslib.as_array((C.c_double * 12).from_address(Rt)).copy(),
                                   "outl": np.ctypeslib.as_array((C.c_uint8 * n).from_address(outl)).copy()})
                return ok
            s = {k: self.stored[f"c{i}_{k}"] for k in ("in", "ok", "Rt", "outl")}
            self.calls.append(s)
            if not (s["in"] == ins).all() or len(s["outl"]) != n:
                self.errors.append(f"call {i}: inputs differ from the recorded ones")
            C.memmove(Rt, np.ascontiguousarray(s["Rt"]).ctypes.data, 96)
            C.memmove(outl, np.ascontiguousarray(s["outl"]).ctypes.data, n)
            return int(s["ok"])
        except Exception as e:   # an exception cannot cross the C frame: report it from finish()
            self.errors.append(repr(e))
            return 0

    def finish(self):
        assert not self.errors, self.errors
        if self.ref is not None:
            ref_outputs(self.ref, self.key, lambda R: dict({"ncalls": len(self.calls)},
                                                           **{f"c{i}_{k}": v for i, c in enumerate(self.calls) for k, v in c.items()}))
        else:
            assert len(self.calls) == int(self.stored["ncalls"]), (len(self.calls), int(self.stored["ncalls"]))
