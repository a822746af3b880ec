"""ctypes binding of tests/toi_oracle.c (tbvh_mesh_toi / tbvh_mesh_toi_pairs restated on the host), compiled on first use into a
temporary directory: the repository tree is not written.  Also an independent fp64 conservative advancement (toi64)."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import portpy
from tests import meshdist_oracle as md
from tests.tritri_oracle import to_pairs

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "toi_oracle.c")
_DEPS = [_SRC] + md._DEPS
_lib = None
NO_PRIM = 0xFFFFFFFF


def lib():
    global _lib
    if _lib is None:
        key = hashlib.sha256(b"".join(open(p, "rb").read() for p in _DEPS)).hexdigest()[:16]
        so = os.path.join(tempfile.gettempdir(), f"tbvh_toi_oracle_{os.getuid()}_{key}.so")
        if not os.path.isfile(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.check_call(["gcc", "-std=c11", "-O2", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-Wall",
                                   "-Wno-unused-function", _SRC, "-o", tmp, "-lm"])
            os.replace(tmp, so)
        L = C.CDLL(so)
        vp, u64, i32, u32, f32 = C.c_void_p, C.c_uint64, C.c_int, C.c_uint32, C.c_float
        L.orc_toi_pairs.restype, L.orc_toi_pairs.argtypes = None, [vp, vp, vp, vp, u64, f32, f32, u32, vp]
        L.orc_toi_tree.restype, L.orc_toi_tree.argtypes = None, [vp, u32, vp, vp, vp, vp, vp, u64, f32, f32, u32, i32, i32, vp, vp, vp, vp]
        _lib = L
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _f4(v):
    v = np.asarray(v, np.float32)
    if v.ndim == 2 and v.shape[1] == 3:
        v = np.concatenate([v, np.zeros((v.shape[0], 1), np.float32)], 1)
    return np.ascontiguousarray(v, np.float32).reshape(-1, 4)


def pair(t0, t1, u0, u1, eta, xi, max_iters=64):
    """conservative advancement of row k of each ((n, 3, 3) or (n, 9) corners) -> (contact bool, t, d float32, iters uint32); t = d = inf
    without contact, NaN for a non-finite pair"""
    a = [np.ascontiguousarray(x, np.float32).reshape(-1, 9) for x in (t0, t1, u0, u1)]
    out = np.zeros((a[0].shape[0], 4), np.float32)
    lib().orc_toi_pairs(*[_p(x) for x in a], a[0].shape[0], float(eta), float(xi), int(max_iters), _p(out))
    return out[:, 3] > 0, out[:, 0].copy(), out[:, 1].copy(), out[:, 2].astype(np.uint32)


def _args(nodes, prim_idx, vb0, vb1, va0, va1, self):
    self = va0 is None if self is None else self
    nodes = np.ascontiguousarray(nodes, portpy.NODE32)
    idx = np.ascontiguousarray(prim_idx, np.uint32)
    vb0, vb1 = _f4(vb0), _f4(vb1)
    va0, va1 = (vb0, vb1) if va0 is None else (_f4(va0), _f4(va1))
    return (nodes, idx, vb0, vb1, va0, va1), (_p(nodes), nodes.shape[0], _p(idx), _p(vb0), _p(vb1), _p(va0), _p(va1), va0.shape[0] // 3), self


def nearest(nodes, prim_idx, vb0, vb1, va0=None, va1=None, eta=0.0, xi=1e-3, max_iters=64, brute=False, self=None):
    """the record { t, d, j, iters } of every triangle of A (va0 None: the self query of B) -> (t, d float32, j, iters uint32)"""
    keep, a, self = _args(nodes, prim_idx, vb0, vb1, va0, va1, self)
    rec = np.zeros((a[-1], 4), np.float32)
    lib().orc_toi_tree(*a, float(eta), float(xi), int(max_iters), int(self), int(brute), _p(rec), None, None, None)
    return rec[:, 0].copy(), rec[:, 1].copy(), rec[:, 2].view(np.uint32).copy(), rec[:, 3].view(np.uint32).copy()


def pairs(nodes, prim_idx, vb0, vb1, va0=None, va1=None, eta=0.0, xi=1e-3, max_iters=64, brute=False, self=None):
    """every reached (i, j) in contact within the step -> (sorted unique pairs (m, 2) uint32, their times float32)"""
    keep, a, self = _args(nodes, prim_idx, vb0, vb1, va0, va1, self)
    na = a[-1]
    counts = np.zeros(na, np.uint32)
    lib().orc_toi_tree(*a, float(eta), float(xi), int(max_iters), int(self), int(brute), None, _p(counts), None, None)
    offsets = np.zeros(na + 1, np.uint64)
    np.cumsum(counts, out=offsets[1:])
    keys = np.zeros(int(offsets[-1]), np.uint64)
    if keys.shape[0]:
        lib().orc_toi_tree(*a, float(eta), float(xi), int(max_iters), int(self), int(brute), None, _p(counts), _p(offsets), _p(keys))
    p = to_pairs(keys)
    A0, A1, B0, B1 = (x.reshape(-1, 3, 4)[:, :, :3] for x in (keep[4], keep[5], keep[2], keep[3]))
    t = pair(A0[p[:, 0]], A1[p[:, 0]], B0[p[:, 1]], B1[p[:, 1]], eta, xi, max_iters)[1] if p.shape[0] else np.zeros(0, np.float32)
    return p, t


# ---- an independent fp64 reference ------------------------------------------------------------------------------------------------

def toi64(t0, t1, u0, u1, e, iters=20000, tol=1e-13):
    """the first time in [0, 1] the fp64 distance (meshdist_oracle.fp64_tt) of the linearly moving pairs ((n, 3, 3) each) reaches e, by
    conservative advancement in fp64 with the exact speed bound, stopped within tol * (1 + |x|) of e; inf when it does not happen"""
    t0, t1, u0, u1 = (np.asarray(x, np.float64).reshape(-1, 3, 3) for x in (t0, t1, u0, u1))
    dT, dU = t1 - t0, u1 - u0
    L = np.sqrt(((dT[:, :, None, :] - dU[:, None, :, :]) ** 2).sum(-1)).max((1, 2))
    mag = 1.0 + np.abs(np.concatenate([t0, t1, u0, u1], 1)).max((1, 2))
    t = np.zeros(t0.shape[0])
    live = np.ones(t0.shape[0], bool)
    for _ in range(iters):
        if not live.any():
            break
        k = np.nonzero(live)[0]
        s = t[k][:, None, None]
        d = md.fp64_tt(t0[k] + s * dT[k], u0[k] + s * dU[k])
        done = d - e <= tol * mag[k]
        step = np.where(L[k] > 0, (d - e) / np.where(L[k] > 0, L[k], 1), np.inf)
        nt = np.where(done, t[k], t[k] + step)
        t[k] = nt
        live[k] = ~done & (nt <= 1)
    t[t > 1] = np.inf
    return t
