"""ctypes binding of tests/meshdist_oracle.c (tbvh_mesh_distance / tbvh_mesh_distance_pairs restated on the host), compiled on first use
into a temporary directory: the repository tree is not written.  Also an independent fp64 triangle-triangle distance (fp64_tt)."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import portpy
from tests.tritri_oracle import to_pairs

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "meshdist_oracle.c")
_DEPS = [_SRC, os.path.join(_HERE, "closest_oracle.c"), os.path.join(_HERE, "tritri_oracle.c")]
_lib = None
NO_PRIM = 0xFFFFFFFF


def lib():
    global _lib
    if _lib is None:
        key = hashlib.sha256(b"".join(open(p, "rb").read() for p in _DEPS)).hexdigest()[:16]
        so = os.path.join(tempfile.gettempdir(), f"tbvh_meshdist_oracle_{os.getuid()}_{key}.so")
        if not os.path.isfile(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.check_call(["gcc", "-std=c11", "-O2", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-Wall",
                                   "-Wno-unused-function", _SRC, "-o", tmp, "-lm"])
            os.replace(tmp, so)
        L = C.CDLL(so)
        vp, u64, i32, u32, f32 = C.c_void_p, C.c_uint64, C.c_int, C.c_uint32, C.c_float
        L.orc_tt_dist2_pairs.restype, L.orc_tt_dist2_pairs.argtypes = None, [vp, vp, u64, vp]
        L.orc_md_tree.restype, L.orc_md_tree.argtypes = None, [vp, u32, vp, vp, vp, u64, f32, i32, i32, vp, vp, vp, vp]
        _lib = L
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _f4(v):
    return np.ascontiguousarray(v, np.float32).reshape(-1, 4)


def dist2(a, b):
    """tt_dist2 of row k of a against row k of b; a, b: (n, 3, 3) or (n, 9) corners -> float32 (n,), NaN for a non-finite pair"""
    a = np.ascontiguousarray(a, np.float32).reshape(-1, 9)
    b = np.ascontiguousarray(b, np.float32).reshape(-1, 9)
    out = np.zeros(a.shape[0], np.float32)
    lib().orc_tt_dist2_pairs(_p(a), _p(b), a.shape[0], _p(out))
    return out


def _args(nodes, prim_idx, vb, va, self):
    self = va is None if self is None else self
    nodes = np.ascontiguousarray(nodes, portpy.NODE32)
    idx = np.ascontiguousarray(prim_idx, np.uint32)
    vb = _f4(vb)
    va = vb if va is None else _f4(va)
    return (nodes, idx, vb, va), (_p(nodes), nodes.shape[0], _p(idx), _p(vb), _p(va), va.shape[0] // 3), self


def nearest(nodes, prim_idx, vb, va=None, r_max=np.inf, brute=False, self=None):
    """the nearest record { d, j } of every triangle of va (None: the self query of vb) over B's tree -> (d float32, j uint32)"""
    keep, a, self = _args(nodes, prim_idx, vb, va, self)
    rec = np.zeros((a[-1], 2), np.float32)
    lib().orc_md_tree(*a, float(r_max), int(self), int(brute), _p(rec), None, None, None)
    return rec[:, 0].copy(), rec[:, 1].view(np.uint32).copy()


def pairs(nodes, prim_idx, vb, va=None, r=0.0, brute=False, self=None):
    """every (i, j) with some reference of j reached at value <= r^2 -> (sorted unique pairs, raw keys, counts); the pruned walk's raw
    keys and counts are the device's exactly"""
    keep, a, self = _args(nodes, prim_idx, vb, va, self)
    na = a[-1]
    counts = np.zeros(na, np.uint32)
    lib().orc_md_tree(*a, float(r), int(self), int(brute), None, _p(counts), None, None)
    offsets = np.zeros(na + 1, np.uint64)
    np.cumsum(counts, out=offsets[1:])
    keys = np.zeros(int(offsets[-1]), np.uint64)
    if keys.shape[0]:
        lib().orc_md_tree(*a, float(r), int(self), int(brute), None, _p(counts), _p(offsets), _p(keys))
    return to_pairs(keys), keys, counts


# ---- an independent fp64 reference ------------------------------------------------------------------------------------------------

def _seg_seg(p1, q1, p2, q2):
    """Ericson's clamped ClosestPtSegmentSegment (RTCD 5.1.9) in fp64, vectorised, zero-length segments included: squared distances"""
    d1, d2, r = q1 - p1, q2 - p2, p1 - p2
    a, e, f = (d1 * d1).sum(1), (d2 * d2).sum(1), (d2 * r).sum(1)
    c, b = (d1 * r).sum(1), (d1 * d2).sum(1)
    sa, se = np.where(a > 0, a, 1), np.where(e > 0, e, 1)
    den = a * e - b * b
    s = np.where(den > 0, np.clip((b * f - c * e) / np.where(den > 0, den, 1), 0, 1), 0.0)
    t = (b * s + f) / se
    s = np.where(t < 0, np.clip(-c / sa, 0, 1), np.where(t > 1, np.clip((b - c) / sa, 0, 1), s))
    t = np.clip(t, 0, 1)
    # one or both segments a point
    s = np.where(e > 0, s, np.clip(-c / sa, 0, 1))
    t = np.where(e > 0, t, 0.0)
    s = np.where(a > 0, s, 0.0)
    t = np.where(a > 0, t, np.clip(f / se, 0, 1))
    w = p1 + s[:, None] * d1 - (p2 + t[:, None] * d2)
    return (w * w).sum(1)


def fp64_tt(T, U):
    """the distance between triangles T and U ((n, 3, 3)) in fp64: the least of the six vertex-triangle distances and the nine clamped
    segment-segment distances; 0 where the triangles meet (by tritri_oracle.exact_tt in the caller) is not decided here"""
    from tests.test_closest_point import fp64_closest
    T, U = np.asarray(T, np.float64), np.asarray(U, np.float64)
    best = np.full(T.shape[0], np.inf)
    for c in range(3):
        best = np.minimum(best, fp64_closest(U[:, c], T[:, 0], T[:, 1], T[:, 2]) ** 2)
        best = np.minimum(best, fp64_closest(T[:, c], U[:, 0], U[:, 1], U[:, 2]) ** 2)
    for k in range(3):
        for m in range(3):
            best = np.minimum(best, _seg_seg(T[:, k], T[:, (k + 1) % 3], U[:, m], U[:, (m + 1) % 3]))
    return np.sqrt(best)
