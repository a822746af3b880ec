"""ctypes binding of tests/optimize_oracle.c (the rounds of tbvh_optimize restated on the host), compiled on first use into a temporary
directory: the repository tree is not written."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import portpy

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRCS = [os.path.join(_HERE, "optimize_oracle.c"), os.path.join(os.path.dirname(_HERE), "oracle", "tbvh_oracle.h")]
_lib = None


def lib():
    global _lib
    if _lib is None:
        portpy.build_lib()   # orc_sah_cost comes from the oracle library
        odir = os.path.dirname(portpy.PORT_SO)
        # the library's directory is in the key: the object's runpath names it, so another checkout's copy would load that checkout's library
        key = hashlib.sha256(odir.encode() + b"".join(open(s, "rb").read() for s in _SRCS)).hexdigest()[:16]
        so = os.path.join(tempfile.gettempdir(), f"tbvh_optimize_oracle_{os.getuid()}_{key}.so")
        if not os.path.isfile(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.check_call(["gcc", "-std=c11", "-O2", "-mavx2", "-mfma", "-ffp-contract=off", "-fPIC", "-shared", "-Wall", _SRCS[0], "-o", tmp,
                                   "-L" + odir, "-l:" + os.path.basename(portpy.PORT_SO), "-Wl,-rpath," + odir, "-lm"])
            os.replace(tmp, so)
        L = C.CDLL(so)
        vp, u32, f32 = C.c_void_p, C.c_uint32, C.c_float
        L.orc_optimize.restype, L.orc_optimize.argtypes = u32, [vp, u32, vp, u32, f32, f32, u32, vp, vp, vp, vp]
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def optimize(nodes, prim_idx, max_rounds, c_trav=1.0, c_int=1.0):
    """orc_optimize -> (nodes NODE32 of the result, accepted rounds, final SAHCost, SAHCost after each accepted round)."""
    src = np.ascontiguousarray(nodes).view(portpy.NODE32).reshape(-1)
    idx = np.ascontiguousarray(prim_idx, np.uint32)
    out = np.zeros(src.shape[0], portpy.NODE32)
    per = np.zeros(max(int(max_rounds), 1), np.float32)
    rounds, sah = C.c_uint32(), C.c_float()
    used = lib().orc_optimize(_ptr(src), src.shape[0], _ptr(idx), idx.shape[0], c_trav, c_int, int(max_rounds), _ptr(out),
                              C.byref(rounds), C.byref(sah), _ptr(per))
    return out[:used].copy(), int(rounds.value), np.float32(sah.value), per[: rounds.value].copy()
