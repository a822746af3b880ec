"""ctypes binding of tests/allhits_tlas_oracle.c (tbvh_intersect_all_tlas restated on the host, over tests/allhits_oracle.c, which it
includes), compiled on first use into a temporary directory: the repository tree is not written."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import portpy

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRCS = [os.path.join(_HERE, f) for f in ("allhits_tlas_oracle.c", "allhits_oracle.c")]
_lib = None
NO_PRIM = 0xFFFFFFFF


def lib():
    global _lib
    if _lib is None:
        key = hashlib.sha256(b"".join(open(s, "rb").read() for s in _SRCS)).hexdigest()[:16]
        so = os.path.join(tempfile.gettempdir(), f"tbvh_allhits_tlas_oracle_{os.getuid()}_{key}.so")
        if not os.path.isfile(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.check_call(["gcc", "-std=c11", "-O2", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-Wall",
                                   _SRCS[0], "-o", tmp, "-lm"])
            os.replace(tmp, so)
        L = C.CDLL(so)
        vp, u32, u64, i32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int
        L.orc_ah_tlas_brute.restype, L.orc_ah_tlas_brute.argtypes = None, [vp, u32, vp, vp, vp, u32, vp, u32, u64, u32, vp, vp, vp, vp]
        L.orc_ah_tlas_walk.restype, L.orc_ah_tlas_walk.argtypes = None, [vp, u32, vp, vp, vp, u32, vp, u32, u64, u32, vp, vp, vp, i32]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class _Blas(C.Structure):
    _fields_ = [("nodes", C.c_void_p), ("used_nodes", C.c_uint32), ("prim_idx", C.c_void_p), ("verts", C.c_void_p)]


def _args(tnodes, tidx, instances, blasses, rays):
    """blasses: (nodes, prim_idx, verts) per BLAS; instances: the 192-byte BLASInstance records, already updated"""
    tnodes = np.ascontiguousarray(tnodes).view(portpy.NODE32).reshape(-1)
    tidx = np.ascontiguousarray(tidx, np.uint32)
    inst = np.ascontiguousarray(instances)
    assert inst.dtype.itemsize == 192
    keep = [(np.ascontiguousarray(nd).view(portpy.NODE32).reshape(-1), np.ascontiguousarray(ix, np.uint32),
             np.ascontiguousarray(v, np.float32).reshape(-1, 4)) for nd, ix, v in blasses]
    table = (_Blas * len(keep))(*[_Blas(nd.ctypes.data, nd.shape[0], ix.ctypes.data, v.ctypes.data) for nd, ix, v in keep])
    r = np.ascontiguousarray(rays).reshape(-1)
    assert r.dtype.itemsize % 16 == 0 and r.dtype.itemsize >= 64, "ray records of a multiple of 16 bytes, at least 64"
    return tnodes, tidx, inst, keep, table, r, r.dtype.itemsize, r.shape[0]


def brute(tnodes, tidx, instances, blasses, rays, k):
    """the two-level definition over every reached reference -> (hits (n, k, 4) float32 with prim bits in column 3, insts uint32 (n, k),
    counts uint32 (n,), keys (n, k))"""
    tnodes, tidx, inst, keep, table, r, stride, n = _args(tnodes, tidx, instances, blasses, rays)
    hits = np.zeros((n, k, 4), np.float32)
    insts = np.zeros((n, k), np.uint32)
    counts = np.zeros(n, np.uint32)
    keys = np.zeros((n, k), np.float32)
    lib().orc_ah_tlas_brute(_p(tnodes), tnodes.shape[0], _p(tidx), _p(inst), C.cast(table, C.c_void_p), len(keep), _p(r), stride, n, k,
                            _p(hits), _p(insts), _p(counts), _p(keys))
    return hits, insts, counts, keys


def walk(tnodes, tidx, instances, blasses, rays, k, reverse=False):
    """the pruned two-level walk (host threads) -> (hits, insts, counts) as brute; reverse visits the other child first and a leaf's
    instances from the last"""
    tnodes, tidx, inst, keep, table, r, stride, n = _args(tnodes, tidx, instances, blasses, rays)
    hits = np.zeros((n, k, 4), np.float32)
    insts = np.zeros((n, k), np.uint32)
    counts = np.zeros(n, np.uint32)
    lib().orc_ah_tlas_walk(_p(tnodes), tnodes.shape[0], _p(tidx), _p(inst), C.cast(table, C.c_void_p), len(keep), _p(r), stride, n, k,
                           _p(hits), _p(insts), _p(counts), int(reverse))
    return hits, insts, counts
