"""ctypes binding of tests/wn_oracle.c (tbvh_winding_number_prepare / tbvh_winding_number restated on the host), compiled on first use
into a temporary directory: the repository tree is not written."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import portpy
from tests import sdf_oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "wn_oracle.c")
_lib = None
NONE = 0xFFFFFFFF
DAG, RANGE = 1, 2


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha256(open(_SRC, "rb").read())
        so = os.path.join(tempfile.gettempdir(), f"tbvh_wn_oracle_{os.getuid()}_{h.hexdigest()[:16]}.so")
        if not os.path.isfile(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.check_call(["gcc", "-std=c11", "-O2", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-Wall",
                                   _SRC, "-o", tmp, "-lm"])
            os.replace(tmp, so)
        L = C.CDLL(so)
        vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
        L.orc_wn_prepare.restype, L.orc_wn_prepare.argtypes = u32, [vp, u32, vp, u32, vp, u32, u32, vp, vp]
        L.orc_wn_query.restype, L.orc_wn_query.argtypes = None, [vp, u32, vp, vp, vp, vp, u64, C.c_float, vp]
        L.orc_wn_atan2v.restype, L.orc_wn_atan2v.argtypes = None, [vp, vp, u64, vp]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _f4(a):
    return np.ascontiguousarray(a, np.float32).reshape(-1, 4)


def atan2(y, x):
    """the fixed atan2 of both sides, elementwise over float32 arrays"""
    y, x = np.ascontiguousarray(y, np.float32).reshape(-1), np.ascontiguousarray(x, np.float32).reshape(-1)
    out = np.zeros(y.shape[0], np.float32)
    lib().orc_wn_atan2v(_p(y), _p(x), y.shape[0], _p(out))
    return out


def depth(nodes):
    """levels below the root of the slots reached from node 0 (node 1 never), stopping at 255 steps: the reach steps of the prepare"""
    nodes = np.ascontiguousarray(nodes, portpy.NODE32)
    frontier, d = np.zeros(1, np.int64), 0
    while d < 256:
        inner = frontier[nodes["triCount"][frontier] == 0]
        first = nodes["leftFirst"][inner].astype(np.int64)
        first = first[first + 1 < max(nodes.shape[0], 2)]
        nxt = np.stack([first, first + 1], 1).reshape(-1)
        nxt = nxt[nxt != 1]
        if nxt.size == 0:
            break
        frontier, d = nxt, d + 1
    return d


class Table:
    """the prepared table of a Wald-layout tree: records (slots + 1, 16) float32, the root's last; own[idx_count]; flag"""

    def __init__(self, nodes, prim_idx, verts):
        self.nodes = np.ascontiguousarray(nodes, portpy.NODE32)
        self.idx = np.ascontiguousarray(prim_idx, np.uint32)
        self.verts = _f4(verts)
        used = self.nodes.shape[0]
        S = max(used, 2)
        self.records = np.zeros((S + 1, 16), np.float32)
        self.own = np.zeros(max(self.idx.shape[0], 1), np.uint32)
        self.flag = lib().orc_wn_prepare(_p(self.nodes), used, _p(self.idx), self.idx.shape[0], _p(self.verts), self.verts.shape[0] // 3,
                                         depth(self.nodes), _p(self.records), _p(self.own))

    def query(self, queries, beta):
        q = _f4(queries)
        out = np.zeros(q.shape[0], np.float32)
        lib().orc_wn_query(_p(self.nodes), self.nodes.shape[0], _p(self.own), _p(self.verts), _p(self.records), _p(q), q.shape[0],
                           float(beta), _p(out))
        return out


def winding(nodes, prim_idx, verts, queries, beta):
    """prepare + query; raises on a refused tree"""
    t = Table(nodes, prim_idx, verts)
    assert t.flag == 0, f"the prepare refuses this tree (flag {t.flag})"
    return t.query(queries, beta)


def brute(verts, queries):
    """the exact sum over every triangle in prim order: a one-leaf tree at beta = inf"""
    nodes, idx = sdf_oracle.one_leaf(verts)
    return winding(nodes, idx, verts, queries, np.inf)
