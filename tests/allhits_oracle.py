"""ctypes binding of tests/allhits_oracle.c (tbvh_intersect_all restated on the host), compiled on first use into a temporary directory:
the repository tree is not written."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import portpy

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "allhits_oracle.c")
_lib = None
NO_PRIM = 0xFFFFFFFF


def lib():
    global _lib
    if _lib is None:
        key = hashlib.sha256(open(_SRC, "rb").read()).hexdigest()[:16]
        so = os.path.join(tempfile.gettempdir(), f"tbvh_allhits_oracle_{os.getuid()}_{key}.so")
        if not os.path.isfile(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.check_call(["gcc", "-std=c11", "-O2", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-Wall",
                                   _SRC, "-o", tmp, "-lm"])
            os.replace(tmp, so)
        L = C.CDLL(so)
        vp, u32, u64, i32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int
        L.orc_ah_brute.restype, L.orc_ah_brute.argtypes = None, [vp, u32, vp, vp, vp, u32, u64, u32, vp, vp, vp]
        L.orc_ah_walk.restype, L.orc_ah_walk.argtypes = None, [vp, u32, vp, vp, vp, u32, u64, u32, vp, vp, i32]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _args(nodes, prim_idx, verts, rays):
    nodes = np.ascontiguousarray(nodes, portpy.NODE32)
    idx = np.ascontiguousarray(prim_idx, np.uint32)
    v = np.ascontiguousarray(verts, np.float32).reshape(-1, 4)
    r = np.ascontiguousarray(rays).reshape(-1)
    assert r.dtype.itemsize % 16 == 0 and r.dtype.itemsize >= 64, "ray records of a multiple of 16 bytes, at least 64"
    return nodes, idx, v, r, r.dtype.itemsize, r.shape[0]


def brute(nodes, prim_idx, verts, rays, k):
    """the definition over every reached reference -> (hits (n, k, 4) float32 with prim bits in column 3, counts uint32 (n,), keys (n, k))"""
    nodes, idx, v, r, stride, n = _args(nodes, prim_idx, verts, rays)
    hits = np.zeros((n, k, 4), np.float32)
    counts = np.zeros(n, np.uint32)
    keys = np.zeros((n, k), np.float32)
    lib().orc_ah_brute(_p(nodes), nodes.shape[0], _p(idx), _p(v), _p(r), stride, n, k, _p(hits), _p(counts), _p(keys))
    return hits, counts, keys


def walk(nodes, prim_idx, verts, rays, k, reverse=False):
    """the pruned walk of the same rules (host threads) -> (hits, counts) as brute; reverse visits the other child first"""
    nodes, idx, v, r, stride, n = _args(nodes, prim_idx, verts, rays)
    hits = np.zeros((n, k, 4), np.float32)
    counts = np.zeros(n, np.uint32)
    lib().orc_ah_walk(_p(nodes), nodes.shape[0], _p(idx), _p(v), _p(r), stride, n, k, _p(hits), _p(counts), int(reverse))
    return hits, counts


def prims(hits):
    return np.ascontiguousarray(hits).view(np.uint32)[..., 3]
