"""ctypes binding of tests/sdf_oracle.c (tbvh_signed_distance_prepare / tbvh_signed_distance restated on the host), compiled on first use
into a temporary directory: the repository tree is not written."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import portpy

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "sdf_oracle.c")
_lib = None
NO_PRIM = 0xFFFFFFFF
FACE, V0, V1, V2, AB, AC, BC = range(7)


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha256()
        for f in (_SRC, os.path.join(_HERE, "closest_oracle.c")):
            h.update(open(f, "rb").read())
        so = os.path.join(tempfile.gettempdir(), f"tbvh_sdf_oracle_{os.getuid()}_{h.hexdigest()[:16]}.so")
        if not os.path.isfile(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.check_call(["gcc", "-std=c11", "-O2", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-Wall",
                                   "-I" + _HERE, _SRC, "-o", tmp, "-lm"])
            os.replace(tmp, so)
        L = C.CDLL(so)
        vp, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
        L.orc_sd_prepare.restype, L.orc_sd_prepare.argtypes = None, [vp, u32, vp]
        L.orc_sd_brute.restype, L.orc_sd_brute.argtypes = None, [vp, u32, vp, vp, vp, vp, u64, vp, C.c_int]
        L.orc_sd_triangles.restype, L.orc_sd_triangles.argtypes = None, [vp, vp, u64, vp]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _f4(a):
    return np.ascontiguousarray(a, np.float32).reshape(-1, 4)


def triangles(points, v0, e1, e2):
    """orc_sd_triangle per row -> (d2_raw, u, v, feature)"""
    n = np.asarray(points).shape[0]
    pts = np.zeros((n, 4), np.float32)
    pts[:, :3] = np.asarray(points, np.float32)[:, :3]
    recs = np.zeros((n, 12), np.float32)
    for k, a in enumerate((v0, e1, e2)):
        recs[:, 4 * k: 4 * k + 3] = np.asarray(a, np.float32)[:, :3]
    out = np.zeros((n, 4), np.float32)
    lib().orc_sd_triangles(_p(pts), _p(recs), n, _p(out))
    return out[:, 0], out[:, 1], out[:, 2], out[:, 3].view(np.uint32)


def prepare(verts):
    """the pseudonormal table of a soup of float4 vertices (3 per triangle) -> (prims, 7, 4) float32: face, v0, v1, v2, AB, AC, BC"""
    v = _f4(verts)
    prims = v.shape[0] // 3
    table = np.zeros((prims, 7, 4), np.float32)
    lib().orc_sd_prepare(_p(v), prims, _p(table))
    return table


def brute(nodes, prim_idx, verts, queries, table=None, walk=False):
    """the signed record {sd, u, v, prim bits} of every query over every reference of the tree (walk: through the pruned walk, which
    gives the same records, for large meshes)"""
    if table is None:
        table = prepare(verts)
    nodes = np.ascontiguousarray(nodes, portpy.NODE32)
    idx = np.ascontiguousarray(prim_idx, np.uint32)
    v, q = _f4(verts), _f4(queries)
    res = np.zeros((q.shape[0], 4), np.float32)
    lib().orc_sd_brute(_p(nodes), nodes.shape[0], _p(idx), _p(v), _p(np.ascontiguousarray(table, np.float32)), _p(q), q.shape[0], _p(res), int(walk))
    return res


def one_leaf(verts):
    """a tree of one leaf over every triangle (node 0 the root, node 1 unused): brute over it is a brute force over the mesh"""
    tri = _f4(verts)[:, :3]
    n = tri.shape[0] // 3
    nodes = np.zeros(2, portpy.NODE32)
    nodes[0] = (tri.min(0), 0, tri.max(0), n)
    return nodes, np.arange(n, dtype=np.uint32)


def signed(verts, queries, table=None):
    """brute over a one-leaf tree of the mesh"""
    nodes, idx = one_leaf(verts)
    return brute(nodes, idx, verts, queries, table)
