"""ctypes binding of tests/cwbvh_refit_oracle.c (the CWBVH of a refitted tree over the collapse of the built one), compiled on first use into a
temporary directory: the repository tree is not written."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import portpy

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRCS = [os.path.join(_HERE, "cwbvh_refit_oracle.c"), os.path.join(os.path.dirname(_HERE), "oracle", "tbvh_oracle_cwbvh.c"),
         os.path.join(os.path.dirname(_HERE), "oracle", "tbvh_oracle.h")]
_lib = None


def lib():
    global _lib
    if _lib is None:
        portpy.build_lib()   # orc_tlas_walk1, which the included file calls, comes from the oracle library
        odir = os.path.dirname(portpy.PORT_SO)
        # the library's directory is in the key: the object's runpath names it, so another checkout's copy would load that checkout's library
        key = hashlib.sha256(odir.encode() + b"".join(open(s, "rb").read() for s in _SRCS)).hexdigest()[:16]
        so = os.path.join(tempfile.gettempdir(), f"tbvh_cwbvh_refit_oracle_{os.getuid()}_{key}.so")
        if not os.path.isfile(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.check_call(["gcc", "-std=c11", "-O3", "-mavx2", "-mfma", "-ffp-contract=off", "-fPIC", "-shared", _SRCS[0], "-o", tmp,
                                   "-L" + odir, "-l:" + os.path.basename(portpy.PORT_SO), "-Wl,-rpath," + odir, "-lm"])
            os.replace(tmp, so)
        L = C.CDLL(so)
        vp, u32 = C.c_void_p, C.c_uint32
        L.orc_cwbvh_refit_from_bvh.restype, L.orc_cwbvh_refit_from_bvh.argtypes = u32, [vp, vp, u32, vp, u32, vp, u32, vp, vp]
        _lib = L
    return _lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


class RefitCWBVH(portpy.PortCWBVH):
    """orc_cwbvh_refit_from_bvh: the CWBVH that keeps the 8-wide collapse of built_nodes and takes its boxes from refit_nodes (the same tree
    refitted to `verts`) - what tbvh_refit_layouts computes; .intersect is the reference's CPU walk (orc_cwbvh_intersect)."""

    def __init__(self, built_nodes, refit_nodes, prim_idx, verts, idx_count=None):
        built = np.ascontiguousarray(built_nodes).view(portpy.NODE32).reshape(-1)
        refit = np.ascontiguousarray(refit_nodes).view(portpy.NODE32).reshape(-1)
        assert built.shape == refit.shape
        prim_idx = np.ascontiguousarray(prim_idx, np.uint32)
        self.verts = np.ascontiguousarray(verts, np.float32).reshape(-1, 4)
        n = self.verts.shape[0] // 3
        ic = int(idx_count) if idx_count is not None else prim_idx.shape[0]
        pidx = np.zeros(ic, np.uint32)
        pidx[: prim_idx.shape[0]] = prim_idx
        data = np.zeros((n * 5, 4), np.float32)
        self.tris = np.zeros((ic * 3, 4), np.float32)
        blocks = lib().orc_cwbvh_refit_from_bvh(_ptr(built), _ptr(refit), built.shape[0], _ptr(pidx), ic, _ptr(self.verts), n, _ptr(data), _ptr(self.tris))
        self.nodes = data[:blocks].copy()
