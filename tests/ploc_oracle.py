"""ctypes binding of tests/ploc_oracle.c (TBVH_BUILD_PLOC restated on the host), compiled on first use into a temporary directory: the
repository tree is not written."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import portpy

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRCS = [os.path.join(_HERE, "ploc_oracle.c"), os.path.join(os.path.dirname(_HERE), "oracle", "tbvh_oracle.h")]
_lib = None


def lib():
    global _lib
    if _lib is None:
        portpy.build_lib()   # orc_refit and orc_sah_cost come from the oracle library
        odir = os.path.dirname(portpy.PORT_SO)
        # the library's directory is in the key: the object's runpath names it, so another checkout's copy would load that checkout's library
        key = hashlib.sha256(odir.encode() + b"".join(open(s, "rb").read() for s in _SRCS)).hexdigest()[:16]
        so = os.path.join(tempfile.gettempdir(), f"tbvh_ploc_oracle_{os.getuid()}_{key}.so")
        if not os.path.isfile(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.check_call(["gcc", "-std=c11", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-Wall", _SRCS[0], "-o", tmp,
                                   "-L" + odir, "-l:" + os.path.basename(portpy.PORT_SO), "-Wl,-rpath," + odir, "-lm"])
            os.replace(tmp, so)
        L = C.CDLL(so)
        vp, u32, f32 = C.c_void_p, C.c_uint32, C.c_float
        L.orc_build_ploc.restype, L.orc_build_ploc.argtypes = u32, [vp, u32, f32, f32, vp, vp, vp, vp]
        _lib = L
    return _lib


def build(verts, c_trav=1.0, c_int=1.0):
    """orc_build_ploc over verts ((3 n, 4) float32) -> (nodes NODE32, primIdx, clustering iterations, SAHCost)."""
    v = np.ascontiguousarray(verts, np.float32).reshape(-1, 4)
    n = v.shape[0] // 3
    nodes = np.zeros(2 * n + 2, portpy.NODE32)
    idx = np.zeros(n, np.uint32)
    iters, sah = C.c_uint32(), C.c_float()
    used = lib().orc_build_ploc(v.ctypes.data_as(C.c_void_p), n, c_trav, c_int, nodes.ctypes.data_as(C.c_void_p), idx.ctypes.data_as(C.c_void_p),
                                C.byref(iters), C.byref(sah))
    return nodes[:used].copy(), idx, int(iters.value), np.float32(sah.value)
