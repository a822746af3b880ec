"""ctypes binding of tests/closest_oracle.c (tbvh_closest_point / tbvh_sphere_overlap restated on the host), compiled on first use into a
temporary directory: the repository tree is not written."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import portpy

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "closest_oracle.c")
_lib = None
NO_PRIM = 0xFFFFFFFF


def lib():
    global _lib
    if _lib is None:
        key = hashlib.sha256(open(_SRC, "rb").read()).hexdigest()[:16]
        so = os.path.join(tempfile.gettempdir(), f"tbvh_closest_oracle_{os.getuid()}_{key}.so")
        if not os.path.isfile(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.check_call(["gcc", "-std=c11", "-O2", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-Wall",
                                   _SRC, "-o", tmp, "-lm"])
            os.replace(tmp, so)
        L = C.CDLL(so)
        vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
        for name in ("orc_cp_brute", "orc_cp_walk"):
            getattr(L, name).restype, getattr(L, name).argtypes = None, [vp, u32, vp, vp, vp, u64, vp, vp]
        L.orc_cp_node_bounds.restype, L.orc_cp_node_bounds.argtypes = None, [vp, u32, vp, vp]
        L.orc_cp_triangles.restype, L.orc_cp_triangles.argtypes = None, [vp, vp, u64, vp]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _f4(a, cols=4):
    return np.ascontiguousarray(a, np.float32).reshape(-1, cols)


def triangles(points, v0, e1, e2):
    """orc_cp_triangle per row: points, v0, e1, e2 (n, 3 or 4) -> (d2_raw, u, v) float32 arrays"""
    n = np.asarray(points).shape[0]
    pts = np.zeros((n, 4), np.float32)
    pts[:, :3] = np.asarray(points, np.float32)[:, :3]
    recs = np.zeros((n, 12), np.float32)
    for k, a in enumerate((v0, e1, e2)):
        recs[:, 4 * k: 4 * k + 3] = np.asarray(a, np.float32)[:, :3]
    out = np.zeros((n, 4), np.float32)
    lib().orc_cp_triangles(_p(pts), _p(recs), n, _p(out))
    return out[:, 0], out[:, 1], out[:, 2]


def _run(fn, nodes, prim_idx, verts, queries, any_):
    nodes = np.ascontiguousarray(nodes, portpy.NODE32)
    idx = np.ascontiguousarray(prim_idx, np.uint32)
    v, q = _f4(verts), _f4(queries)
    n = q.shape[0]
    if any_:
        bits = np.zeros((n + 31) // 32, np.uint32)
        getattr(lib(), fn)(_p(nodes), nodes.shape[0], _p(idx), _p(v), _p(q), n, None, _p(bits))
        return bits
    res = np.zeros((n, 4), np.float32)
    getattr(lib(), fn)(_p(nodes), nodes.shape[0], _p(idx), _p(v), _p(q), n, _p(res), None)
    return res


def brute(nodes, prim_idx, verts, queries, any_=False):
    """every reference of the tree: closest -> (n, 4) float32 records {d, u, v, prim bits}; any_ -> uint32 overlap words"""
    return _run("orc_cp_brute", nodes, prim_idx, verts, queries, any_)


def walk(nodes, prim_idx, verts, queries, any_=False):
    """the pruned walk of the same rules (host threads), same outputs as brute"""
    return _run("orc_cp_walk", nodes, prim_idx, verts, queries, any_)


def node_bounds(nodes, point):
    """path bound P of every node for one point (-1 for slots the root does not reach)"""
    nodes = np.ascontiguousarray(nodes, portpy.NODE32)
    p = np.zeros(4, np.float32)
    p[:3] = point[:3]
    out = np.zeros(nodes.shape[0], np.float32)
    lib().orc_cp_node_bounds(_p(nodes), nodes.shape[0], _p(p), _p(out))
    return out


def record_prims(res):
    return np.ascontiguousarray(res).view(np.uint32)[:, 3]
