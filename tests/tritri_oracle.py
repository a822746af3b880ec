"""ctypes binding of tests/tritri_oracle.c (tbvh_mesh_overlap_pairs / tbvh_mesh_overlap_bits restated on the host), compiled on first use
into a temporary directory: the repository tree is not written.  Also two exact references in Python numbers (ints or Fractions): the
same predicates evaluated exactly (exact_tt), and an independent separating-axis test (sat_tt)."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import portpy

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "tritri_oracle.c")
_lib = None


def lib():
    global _lib
    if _lib is None:
        key = hashlib.sha256(open(_SRC, "rb").read()).hexdigest()[:16]
        so = os.path.join(tempfile.gettempdir(), f"tbvh_tritri_oracle_{os.getuid()}_{key}.so")
        if not os.path.isfile(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.check_call(["gcc", "-std=c11", "-O2", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-fPIC", "-shared", "-Wall",
                                   _SRC, "-o", tmp, "-lm"])
            os.replace(tmp, so)
        L = C.CDLL(so)
        vp, u64, i32, u32 = C.c_void_p, C.c_uint64, C.c_int, C.c_uint32
        L.orc_tt_pairs.restype, L.orc_tt_pairs.argtypes = None, [vp, vp, u64, i32, vp]
        L.orc_overlap_all.restype, L.orc_overlap_all.argtypes = None, [vp, u64, vp, u64, i32, vp, vp, vp, vp]
        L.orc_overlap_tree.restype, L.orc_overlap_tree.argtypes = None, [vp, u32, vp, vp, vp, u64, i32, i32, vp, vp, vp, vp]
        _lib = L
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _f4(v):
    return np.ascontiguousarray(v, np.float32).reshape(-1, 4)


def tt(a, b, self=False):
    """the pair test (or the self rules) of row k of a against row k of b; a, b: (n, 3, 3) or (n, 9) corners -> bool (n,)"""
    a = np.ascontiguousarray(a, np.float32).reshape(-1, 9)
    b = np.ascontiguousarray(b, np.float32).reshape(-1, 9)
    out = np.zeros(a.shape[0], np.uint8)
    lib().orc_tt_pairs(_p(a), _p(b), a.shape[0], int(self), _p(out))
    return out.astype(bool)


def _collect(run, na):
    """two passes of an oracle form: per-triangle counts, then the raw keys at their offsets -> (raw keys, counts)"""
    counts = np.zeros(na, np.uint32)
    run(counts, None, None)
    offsets = np.zeros(na + 1, np.uint64)
    np.cumsum(counts, out=offsets[1:])
    keys = np.zeros(int(offsets[-1]), np.uint64)
    if keys.shape[0]:
        run(counts, offsets, keys)
    return keys, counts


def to_pairs(keys):
    """raw keys -> the sorted, unique (m, 2) uint32 pairs (i, j)"""
    k = np.unique(np.asarray(keys, np.uint64))
    return np.stack([(k >> np.uint64(32)).astype(np.uint32), (k & np.uint64(0xFFFFFFFF)).astype(np.uint32)], 1).reshape(-1, 2)


def all_pairs(va, vb=None, self=None):
    """every (A triangle, B triangle) pair; vb None: the self query over va -> (pairs, bit words)"""
    self = vb is None if self is None else self
    va = _f4(va)
    vb = va if vb is None else _f4(vb)
    na, nb = va.shape[0] // 3, vb.shape[0] // 3
    keys, _ = _collect(lambda c, o, k: lib().orc_overlap_all(_p(va), na, _p(vb), nb, int(self), _p(c), _p(o), _p(k), None), na)
    bits = np.zeros(max((na + 31) // 32, 1), np.uint32)
    lib().orc_overlap_all(_p(va), na, _p(vb), nb, int(self), None, None, None, _p(bits))
    return to_pairs(keys), bits


def tree(nodes, prim_idx, vb, va=None, brute=False, self=None):
    """over the tree (nodes, prim_idx) of B's vertices vb; va None: the self query (self=True with va: the self query of va, the first
    triangles of vb, against all of vb) -> (pairs, bit words, raw keys, counts).  brute: the
    definition (reached slots marked, no pruning), whose raw keys and counts are in slot order; else the kernel's pruned walk, whose raw
    keys and counts are the device's exactly."""
    self = va is None if self is None else self
    nodes = np.ascontiguousarray(nodes, portpy.NODE32)
    idx = np.ascontiguousarray(prim_idx, np.uint32)
    vb = _f4(vb)
    va = vb if va is None else _f4(va)
    na = va.shape[0] // 3
    args = (_p(nodes), nodes.shape[0], _p(idx), _p(vb), _p(va), na, int(self), int(brute))
    keys, counts = _collect(lambda c, o, k: lib().orc_overlap_tree(*args, _p(c), _p(o), _p(k), None), na)
    bits = np.zeros(max((na + 31) // 32, 1), np.uint32)
    lib().orc_overlap_tree(*args, None, None, None, _p(bits))
    return to_pairs(keys), bits, keys, counts


def member_bits(pairs, n, self):
    """bit words of 'triangle i is a member of some pair' (self: either member)"""
    m = np.zeros(n, bool)
    m[pairs[:, 0]] = True
    if self:
        m[pairs[:, 1]] = True
    words = np.zeros(max((n + 31) // 32, 1), np.uint32)
    packed = np.packbits(np.r_[m, np.zeros(words.shape[0] * 32 - n, bool)], bitorder="little")
    words[:] = packed.view(np.uint32)
    return words


# ---- exact references ------------------------------------------------------------------------------------------------------------

def _sub(a, b):
    return (a[0] - b[0], a[1] - b[1], a[2] - b[2])


def _cross(a, b):
    return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])


def _dot(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


class _Track:
    """the least |value| of the 3D predicates (degree 3) and the 2D ones (degree 2) an exact run evaluated"""
    def __init__(self):
        self.m3, self.m2 = None, None

    def v3(self, x):
        self.m3 = abs(x) if self.m3 is None else min(self.m3, abs(x))
        return x

    def v2(self, x):
        self.m2 = abs(x) if self.m2 is None else min(self.m2, abs(x))
        return x


def _key(f):
    u = int(np.float32(f).view(np.uint32))
    return (~u) & 0xFFFFFFFF if u & 0x80000000 else u | 0x80000000


def exact_tt(a, b, self=False, num=int, track=None):
    """orc_tt's rules in exact arithmetic: a, b are three corners of float32 values; num converts a coordinate (int for lattice inputs,
    fractions.Fraction for any float); the canonical order and the shared corners are decided on the float32 values as the engine does"""
    a = np.asarray(a, np.float32).reshape(3, 3)
    b = np.asarray(b, np.float32).reshape(3, 3)
    if not (np.isfinite(a).all() and np.isfinite(b).all()):
        return False
    if (a.max(0) < b.min(0)).any() or (b.max(0) < a.min(0)).any():
        return False
    tr = track or _Track()
    swap = False
    for x, y in zip(a.reshape(-1), b.reshape(-1)):
        if _key(x) != _key(y):
            swap = _key(y) < _key(x)
            break
    rt, ru = (b, a) if swap else (a, b)
    T = [tuple(num(float(c)) for c in r) for r in rt]
    U = [tuple(num(float(c)) for c in r) for r in ru]
    nT, nU = _cross(_sub(T[1], T[0]), _sub(T[2], T[0])), _cross(_sub(U[1], U[0]), _sub(U[2], U[0]))
    if nT == (0, 0, 0) or nU == (0, 0, 0):
        return False

    def side(x, o, n):
        return tr.v3(_dot(_sub(x, o), n))

    def o3(p, q, r, s):
        return side(s, p, _cross(_sub(q, p), _sub(r, p)))

    def axes(n):
        ax, ay, az = (abs(c) for c in n)
        if ax > az and ax >= ay:
            return 1, 2
        if ay > az and ay >= ax:
            return 2, 0
        return 0, 1

    def o2(p, q, r, i, j):
        return tr.v2((q[i] - p[i]) * (r[j] - p[j]) - (q[j] - p[j]) * (r[i] - p[i]))

    def same3(x, y, z):
        return (x > 0 and y > 0 and z > 0) or (x < 0 and y < 0 and z < 0)

    def sep2(p, q, r, ys, i, j):
        s = o2(p, q, r, i, j)
        return s != 0 and all((o2(p, q, y, i, j) < 0) if s > 0 else (o2(p, q, y, i, j) > 0) for y in ys)

    def seg_tri(p, q, sp, sq, X, n):
        if (sp > 0 and sq > 0) or (sp < 0 and sq < 0):
            return False
        if sp == 0 and sq == 0:
            i, j = axes(n)
            if any(sep2(X[e], X[(e + 1) % 3], X[(e + 2) % 3], (p, q), i, j) for e in range(3)):
                return False
            return not same3(*(o2(p, q, X[k], i, j) for k in range(3)))
        if sp == 0 or sq == 0:
            i, j = axes(n)
            x = p if sp == 0 else q
            return not any(sep2(X[e], X[(e + 1) % 3], X[(e + 2) % 3], (x,), i, j) for e in range(3))
        o = [o3(p, q, X[0], X[1]), o3(p, q, X[1], X[2]), o3(p, q, X[2], X[0])]
        return all(v >= 0 for v in o) or all(v <= 0 for v in o)

    dU = [side(U[c], T[0], nT) for c in range(3)]
    dT = [side(T[c], U[0], nU) for c in range(3)]
    if self:
        match = [[bool((rt[x] == ru[y]).all()) for y in range(3)] for x in range(3)]
        tm = [any(match[x]) for x in range(3)]
        um = [any(match[x][y] for x in range(3)) for y in range(3)]
        shared = sum(tm)
        if shared == 3:
            return True
        if shared == 1:
            ta = tm.index(True)
            ub = match[ta].index(True)
            return (seg_tri(T[(ta + 1) % 3], T[(ta + 2) % 3], dT[(ta + 1) % 3], dT[(ta + 2) % 3], U, nU)
                    or seg_tri(U[(ub + 1) % 3], U[(ub + 2) % 3], dU[(ub + 1) % 3], dU[(ub + 2) % 3], T, nT))
        if shared == 2:
            if any(dU) or any(dT):
                return False
            t3, u3 = tm.index(False), um.index(False)
            i, j = axes(nT)
            s1 = o2(T[(t3 + 1) % 3], T[(t3 + 2) % 3], T[t3], i, j)
            s2 = o2(T[(t3 + 1) % 3], T[(t3 + 2) % 3], U[u3], i, j)
            return (s1 > 0 and s2 > 0) or (s1 < 0 and s2 < 0)
    if same3(*dU) or same3(*dT):
        return False
    if not any(dU):
        i, j = axes(nT)
        return not any(sep2(T[e], T[(e + 1) % 3], T[(e + 2) % 3], U, i, j) or sep2(U[e], U[(e + 1) % 3], U[(e + 2) % 3], T, i, j)
                       for e in range(3))
    return any(seg_tri(T[e], T[(e + 1) % 3], dT[e], dT[(e + 1) % 3], U, nU) or seg_tri(U[e], U[(e + 1) % 3], dU[e], dU[(e + 1) % 3], T, nT)
               for e in range(3))


def sat_tt(a, b):
    """closed triangles meet: an independent exact test by separating axes (the two normals, the nine edge-edge cross products and the
    six in-plane edge normals), for non-degenerate triangles with int or Fraction coordinates"""
    T = [tuple(r) for r in a]
    U = [tuple(r) for r in b]
    eT = [_sub(T[(k + 1) % 3], T[k]) for k in range(3)]
    eU = [_sub(U[(k + 1) % 3], U[k]) for k in range(3)]
    nT, nU = _cross(eT[0], eT[1]), _cross(eU[0], eU[1])
    axes = [nT, nU] + [_cross(x, y) for x in eT for y in eU] + [_cross(nT, x) for x in eT] + [_cross(nU, y) for y in eU]
    for ax in axes:
        if ax == (0, 0, 0):
            continue
        pa = [_dot(p, ax) for p in T]
        pb = [_dot(p, ax) for p in U]
        if max(pa) < min(pb) or max(pb) < min(pa):
            return False
    return True
