import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with -m gpu on a machine that has one)")


def P(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="session")
def oracle():
    """The plain-C CPU oracle (oracle/alva_oracle.c), built on demand.  Test infrastructure only."""
    so = os.path.join(ROOT, "oracle", "_build", "libalva_oracle.so")
    srcs = [os.path.join(ROOT, "oracle", f) for f in ("alva_oracle.c", "ba_oracle.c", "klt_oracle.c", "pose_oracle.c", "detect_oracle.c", "match_oracle.c", "init_oracle.c")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle")], stdout=subprocess.DEVNULL)
    L = C.CDLL(so)
    L.orc_fast_atan2.restype = C.c_float
    L.orc_fast_atan2.argtypes = [C.c_float, C.c_float]
    return L


@pytest.fixture(scope="session")
def ref():
    """The reference itself (oracle/_ref/libalva_ref.so), if it was built in this tree; else None."""
    so = os.path.join(ROOT, "oracle", "_ref", "libalva_ref.so")
    if not os.path.exists(so):
        return None
    L = C.CDLL(so)
    L.ref_config(0, 1)
    return L


def golden(name):
    return np.load(os.path.join(GOLDEN, name + ".npz"))


@pytest.fixture(scope="session")
def gpu_ctx():
    import torch
    if not torch.cuda.is_available():   # a plain `pytest tests` on a machine without a GPU: skip, do not error
        pytest.skip("gpu tests need a CUDA device")
    import alvaar_b200
    ctx = alvaar_b200.Context(0, torch.cuda.current_stream().cuda_stream)
    yield ctx
    ctx.close()
