"""alvaar_b200 -- H100-native per-frame visual-SLAM hot path behind AlvaAR's System API.

The product is the CUDA shared library ``libalva_b200.so`` (C ABI in ``include/alva_b200.h``); this
package is the thin ctypes binding the tests and ``bench.py`` use.  There is NO CPU fallback: importing
works anywhere (so the symbol table can be checked), but creating a context without an H100 (sm_90) raises.
"""
from .lib import (AlvaError, Context, lib, lib_path, key_x, key_y, key_score, unpack_keys,
                  ORB_FMA, ORB_IC_ANGLE, ORB_HARRIS)
from .system import System

__all__ = ["AlvaError", "Context", "lib", "lib_path", "key_x", "key_y", "key_score", "unpack_keys",
           "ORB_FMA", "ORB_IC_ANGLE", "ORB_HARRIS", "System"]
