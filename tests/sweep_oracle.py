"""ctypes binding of tests/sweep_oracle.c (tbvh_sphere_cast / tbvh_sphere_cast_occluded restated on the host over closest_oracle.c),
compiled on first use into a temporary directory: the repository tree is not written."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import portpy

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "sweep_oracle.c")
_DEP = os.path.join(_HERE, "closest_oracle.c")
_lib = None
NO_PRIM = 0xFFFFFFFF


def lib():
    global _lib
    if _lib is None:
        key = hashlib.sha256(open(_SRC, "rb").read() + open(_DEP, "rb").read()).hexdigest()[:16]
        so = os.path.join(tempfile.gettempdir(), f"tbvh_sweep_oracle_{os.getuid()}_{key}.so")
        if not os.path.isfile(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.check_call(["gcc", "-std=c11", "-O2", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-Wall",
                                   _SRC, "-o", tmp, "-lm"])
            os.replace(tmp, so)
        L = C.CDLL(so)
        vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
        for name in ("orc_sc_brute", "orc_sc_walk"):
            getattr(L, name).restype, getattr(L, name).argtypes = None, [vp, u32, vp, vp, vp, u64, vp, vp]
        L.orc_sc_node_bounds.restype, L.orc_sc_node_bounds.argtypes = None, [vp, u32, vp, vp]
        L.orc_sc_triangles.restype, L.orc_sc_triangles.argtypes = None, [vp, vp, u64, vp]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def queries(c, d, r, tmax):
    """(n, 8) float32 records { cx, cy, cz, r, dx, dy, dz, tmax } from centres and directions (n, 3) and radii / tmax (scalars or (n,))"""
    c = np.asarray(c, np.float32)
    q = np.empty((c.shape[0], 8), np.float32)
    q[:, :3] = c[:, :3]
    q[:, 3] = np.asarray(r, np.float32)
    q[:, 4:7] = np.asarray(d, np.float32)[:, :3]
    q[:, 7] = np.asarray(tmax, np.float32)
    return q


def triangles(q, v0, e1, e2):
    """orc_sc_triangle per row: q (n, 8), v0, e1, e2 (n, 3 or 4) -> (contact bool, t, u, v) float32 arrays"""
    q = np.ascontiguousarray(q, np.float32).reshape(-1, 8)
    n = q.shape[0]
    recs = np.zeros((n, 12), np.float32)
    for k, a in enumerate((v0, e1, e2)):
        recs[:, 4 * k: 4 * k + 3] = np.asarray(a, np.float32)[:, :3]
    out = np.zeros((n, 4), np.float32)
    lib().orc_sc_triangles(_p(q), _p(recs), n, _p(out))
    return out[:, 3] > 0, out[:, 0], out[:, 1], out[:, 2]


def _run(fn, nodes, prim_idx, verts, q, any_):
    nodes = np.ascontiguousarray(nodes, portpy.NODE32)
    idx = np.ascontiguousarray(prim_idx, np.uint32)
    v = np.ascontiguousarray(verts, np.float32).reshape(-1, 4)
    q = np.ascontiguousarray(q, np.float32).reshape(-1, 8)
    n = q.shape[0]
    if any_:
        bits = np.zeros((n + 31) // 32, np.uint32)
        getattr(lib(), fn)(_p(nodes), nodes.shape[0], _p(idx), _p(v), _p(q), n, None, _p(bits))
        return bits
    res = np.zeros((n, 4), np.float32)
    getattr(lib(), fn)(_p(nodes), nodes.shape[0], _p(idx), _p(v), _p(q), n, _p(res), None)
    return res


def brute(nodes, prim_idx, verts, q, any_=False):
    """every reached reference of the tree: (n, 4) float32 records {t, u, v, prim bits}; any_ -> uint32 blocked words"""
    return _run("orc_sc_brute", nodes, prim_idx, verts, q, any_)


def walk(nodes, prim_idx, verts, q, any_=False):
    """the pruned walk of the same rules (host threads), same outputs as brute"""
    return _run("orc_sc_walk", nodes, prim_idx, verts, q, any_)


def node_bounds(nodes, q):
    """path bound P of every node for one query (8 floats; -1 for slots the root does not reach)"""
    nodes = np.ascontiguousarray(nodes, portpy.NODE32)
    q = np.ascontiguousarray(q, np.float32).reshape(8)
    out = np.zeros(nodes.shape[0], np.float32)
    lib().orc_sc_node_bounds(_p(nodes), nodes.shape[0], _p(q), _p(out))
    return out


def record_prims(res):
    return np.ascontiguousarray(res).view(np.uint32)[:, 3]
