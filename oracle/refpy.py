"""ctypes binding of oracle/_ref/libtinybvh_ref.so (the unmodified reference behind oracle/ref_wrap.cpp).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
--impl reference arms.  The product package (tinybvh_b200/) never imports this module.
"""
from __future__ import annotations

import ctypes as C
import os
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
REF_SO = os.path.join(_HERE, "_ref", "libtinybvh_ref.so")
_lib = None

NODE32 = np.dtype([("aabbMin", "3f4"), ("leftFirst", "u4"), ("aabbMax", "3f4"), ("triCount", "u4")])
NODE64 = np.dtype([("lmin", "3f4"), ("left", "u4"), ("lmax", "3f4"), ("right", "u4"),
                   ("rmin", "3f4"), ("triCount", "u4"), ("rmax", "3f4"), ("firstTri", "u4")])


def available() -> bool:
    return os.path.isfile(REF_SO)


def lib():
    global _lib
    if _lib is None:
        if not available():
            raise FileNotFoundError(f"{REF_SO} missing: run `make -C oracle ref` where /root/reference exists")
        L = C.CDLL(REF_SO)
        vp, u32, u64, i32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int
        sig = {
            "ref_hardware_threads": (i32, []),
            "ref_bvh_build": (vp, [vp, u32, i32, i32]),
            "ref_bvh_build_costs": (vp, [vp, u32, i32, i32, C.c_float, C.c_float]),
            "ref_bvh_build_indexed": (vp, [vp, u32, vp, u32, i32, i32]),
            "ref_bvh_destroy": (None, [vp]),
            "ref_bvh_used_nodes": (u32, [vp]), "ref_bvh_idx_count": (u32, [vp]), "ref_bvh_tri_count": (u32, [vp]),
            "ref_bvh_nodes": (vp, [vp]), "ref_bvh_prim_idx": (vp, [vp]),
            "ref_bvh_sah_cost": (C.c_float, [vp]),
            "ref_bvh_compact": (None, [vp]), "ref_bvh_refit": (None, [vp]), "ref_bvh_split_leafs": (None, [vp, u32]),
            "ref_bvh_from_arrays": (vp, [vp, u32, vp, u32, vp, u32]),
            "ref_bvh_optimize": (vp, [vp, u32, u32, i32, i32]),
            "ref_bvh_intersect": (None, [vp, vp, u64, i32]),
            "ref_bvh_intersect_cost": (u64, [vp, vp, u64, i32]),
            "ref_bvh_occluded": (None, [vp, vp, u64, vp, i32]),
            "ref_clip_frag": (i32, [vp, vp, vp, vp, vp, vp, u32]),
            "ref_split_frag": (None, [vp, vp, vp, vp, vp, u32, C.c_float, vp, vp]),
            "ref_instance_update": (None, [vp, vp, vp]),
            "ref_tlas_build": (vp, [vp, u32, vp, u32]), "ref_tlas_destroy": (None, [vp]), "ref_tlas_bvh": (vp, [vp]),
            "ref_sizeof_blas_instance": (i32, []), "ref_inst_idx_bits": (i32, []), "ref_offsetof_hit_inst": (i32, []),
            "ref_bvhgpu_from_bvh": (vp, [vp, i32]), "ref_bvhgpu_destroy": (None, [vp]),
            "ref_bvhgpu_used_nodes": (u32, [vp]), "ref_bvhgpu_nodes": (vp, [vp]),
            "ref_bvhgpu_intersect": (None, [vp, vp, u64, i32]),
            "ref_cwbvh_build": (vp, [vp, u32, i32, i32]), "ref_cwbvh_destroy": (None, [vp]),
            "ref_cwbvh_used_blocks": (u32, [vp]), "ref_cwbvh_idx_count": (u32, [vp]), "ref_cwbvh_tri_count": (u32, [vp]),
            "ref_cwbvh_nodes": (vp, [vp]), "ref_cwbvh_tris": (vp, [vp]), "ref_cwbvh_source_bvh": (vp, [vp]),
            "ref_cwbvh_intersect": (None, [vp, vp, u64, i32]),
            "ref_bvh8cpu_build": (vp, [vp, u32, i32]), "ref_bvh8cpu_destroy": (None, [vp]),
            "ref_bvh8cpu_intersect": (None, [vp, vp, u64, i32]),
            "ref_bvh8cpu_occluded": (None, [vp, vp, u64, vp, i32]),
        }
        for name, (res, args) in sig.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = res, args
        _lib = L
    return _lib


FRAGMENT = np.dtype([("bmin", "3f4"), ("primIdx", "u4"), ("bmax", "3f4"), ("clipped", "u4")])  # BVHBase::Fragment :792


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


def _view(addr, dtype, count):
    """COPY of `count` records at `addr` (a copy, so the array outlives the reference object that owns the memory)."""
    buf = (C.c_char * (np.dtype(dtype).itemsize * count)).from_address(addr)
    return np.frombuffer(buf, dtype=dtype, count=count).copy()


class _Traceable:
    _intersect = _occluded = None

    def intersect(self, rays: np.ndarray, threads: int = 0) -> np.ndarray:
        assert rays.dtype.itemsize == 128 and rays.flags.c_contiguous
        getattr(lib(), self._intersect)(self.h, _ptr(rays), rays.shape[0], threads)
        return rays

    def occluded(self, rays: np.ndarray, threads: int = 0) -> np.ndarray:
        assert rays.dtype.itemsize == 128 and rays.flags.c_contiguous
        bits = np.zeros((rays.shape[0] + 31) // 32, np.uint32)
        getattr(lib(), self._occluded)(self.h, _ptr(rays), rays.shape[0], _ptr(bits), threads)
        return bits


class RefBVH(_Traceable):
    """BVH::Build / BuildAVX / BuildHQ + BVH::Intersect / IsOccluded - THE parity oracle (mode 0)."""
    _intersect, _occluded = "ref_bvh_intersect", "ref_bvh_occluded"

    def intersect_cost(self, rays: np.ndarray, threads: int = 0) -> int:
        """trace and return the sum of BVH::Intersect's return values (traversal cost, tiny_bvh.h:3303)"""
        assert rays.dtype.itemsize == 128 and rays.flags.c_contiguous
        return int(lib().ref_bvh_intersect_cost(self.h, _ptr(rays), rays.shape[0], threads))

    def __init__(self, verts: np.ndarray = None, mode: int = 0, threaded: bool = False, _handle=None, _owner=None, indices=None, costs=None):
        self._owner = _owner
        if _handle is not None:
            self.h, self._own = _handle, False
            return
        self.verts = np.array(verts, np.float32, copy=True).reshape(-1, 4)   # own copy: refit() overwrites it in place
        if costs is not None:   # (c_trav, c_int)
            self.h = lib().ref_bvh_build_costs(_ptr(self.verts), self.verts.shape[0] // 3, mode, int(threaded), float(costs[0]), float(costs[1]))
        elif indices is None:
            self.h = lib().ref_bvh_build(_ptr(self.verts), self.verts.shape[0] // 3, mode, int(threaded))
        else:  # the ( vertices, indices, primCount ) overloads; the object keeps both arrays alive (the reference keeps pointers)
            self.indices = np.ascontiguousarray(indices, np.uint32).reshape(-1)
            self.h = lib().ref_bvh_build_indexed(_ptr(self.verts), self.verts.shape[0], _ptr(self.indices), self.indices.shape[0] // 3, mode, int(threaded))
        self._own = True

    @classmethod
    def from_arrays(cls, nodes, prim_idx, verts):
        self = cls.__new__(cls)
        self._owner = None
        self.verts = np.ascontiguousarray(verts, np.float32).reshape(-1, 4)
        nodes = np.ascontiguousarray(nodes)
        prim_idx = np.ascontiguousarray(prim_idx, np.uint32)
        self.h = lib().ref_bvh_from_arrays(_ptr(nodes), nodes.shape[0], _ptr(prim_idx), prim_idx.shape[0],
                                           _ptr(self.verts), self.verts.shape[0] // 3)
        self._own = True
        return self

    @classmethod
    def optimized(cls, verts, iterations: int = 25, extreme: bool = False, stochastic: bool = False):
        """BVH::Build followed by the reference's BVH::Optimize( iterations, extreme, stochastic ) (ref_bvh_optimize)."""
        self = cls.__new__(cls)
        self._owner = None
        self.verts = np.array(verts, np.float32, copy=True).reshape(-1, 4)
        self.h = lib().ref_bvh_optimize(_ptr(self.verts), self.verts.shape[0] // 3, int(iterations), int(extreme), int(stochastic))
        self._own = True
        return self

    def __del__(self):
        if getattr(self, "_own", False) and self.h:
            lib().ref_bvh_destroy(self.h)
            self.h = None

    used_nodes = property(lambda s: lib().ref_bvh_used_nodes(s.h))
    idx_count = property(lambda s: lib().ref_bvh_idx_count(s.h))
    tri_count = property(lambda s: lib().ref_bvh_tri_count(s.h))
    nodes = property(lambda s: _view(lib().ref_bvh_nodes(s.h), NODE32, s.used_nodes))
    prim_idx = property(lambda s: _view(lib().ref_bvh_prim_idx(s.h), np.uint32, s.idx_count))

    def clip_frag(self, frag, bmin, bmax, min_dim, axis):
        """BVH::ClipFrag (:8614) on one FRAGMENT record -> (has_verts, new fragment)."""
        out = np.zeros(1, FRAGMENT)
        a = [np.ascontiguousarray(x, np.float32) for x in (bmin, bmax, min_dim)]
        ok = lib().ref_clip_frag(self.h, _ptr(frag), _ptr(out), _ptr(a[0]), _ptr(a[1]), _ptr(a[2]), int(axis))
        return bool(ok), out

    def split_frag(self, frag, min_dim, axis, pos):
        """BVH::SplitFrag (:8731) -> (left_ok, right_ok, left, right)."""
        l, r = np.zeros(1, FRAGMENT), np.zeros(1, FRAGMENT)
        lo, ro = C.c_int(), C.c_int()
        md = np.ascontiguousarray(min_dim, np.float32)
        lib().ref_split_frag(self.h, _ptr(frag), _ptr(l), _ptr(r), _ptr(md), int(axis), float(pos), C.byref(lo), C.byref(ro))
        return bool(lo.value), bool(ro.value), l, r

    def sah_cost(self):
        return float(lib().ref_bvh_sah_cost(self.h))

    def refit(self, new_verts):
        """BVH::Refit (:3055): the reference reads the vertex array it was built from - overwrite it in place, then refit."""
        self.verts[...] = np.asarray(new_verts, np.float32).reshape(self.verts.shape)
        lib().ref_bvh_refit(self.h)

    def compact(self):
        lib().ref_bvh_compact(self.h)

    def split_leafs(self, n):
        lib().ref_bvh_split_leafs(self.h, n)


# BLASInstance :1443 - 192 bytes: row-major 4x4 transform / inverse, world box, BLAS number, ray mask
BLAS_INSTANCE = np.dtype([("transform", "16f4"), ("invTransform", "16f4"), ("aabbMin", "3f4"), ("blasIdx", "u4"),
                          ("aabbMax", "3f4"), ("mask", "u4"), ("dummy", "8u4")])


def make_instances(transforms, blas_idx, masks=None):
    """BLASInstance records with transform / blasIdx / mask set and the rest at the class defaults (identity inverse, empty box)."""
    t = np.asarray(transforms, np.float32).reshape(-1, 16)
    inst = np.zeros(t.shape[0], BLAS_INSTANCE)
    inst["transform"] = t
    inst["invTransform"] = np.eye(4, dtype=np.float32).reshape(-1)
    inst["aabbMin"], inst["aabbMax"] = 1e30, -1e30
    inst["blasIdx"] = np.asarray(blas_idx, np.uint32)
    inst["mask"] = 0xFFFF if masks is None else np.asarray(masks, np.uint32)
    return inst


class RefTLAS(_Traceable):
    """BVH::Build( BLASInstance*, n, BVHBase**, m ) + IntersectTLAS / IsOccludedTLAS through BVH::Intersect / IsOccluded.
    `instances` (BLAS_INSTANCE array) is updated in place by BLASInstance::Update, exactly as the reference does."""
    _intersect, _occluded = "ref_bvh_intersect", "ref_bvh_occluded"

    def __init__(self, instances: np.ndarray, blasses):
        assert instances.dtype == BLAS_INSTANCE and instances.flags.c_contiguous
        self.instances, self.blasses = instances, list(blasses)
        hs = (C.c_void_p * len(self.blasses))(*[b.h for b in self.blasses])
        self.t = lib().ref_tlas_build(_ptr(instances), instances.shape[0], hs, len(self.blasses))
        self.h = lib().ref_tlas_bvh(self.t)

    def __del__(self):
        if getattr(self, "t", None):
            lib().ref_tlas_destroy(self.t)
            self.t = None

    def bvh(self) -> RefBVH:
        return RefBVH(_handle=self.h, _owner=self)


class RefBVHGPU(_Traceable):
    _intersect = "ref_bvhgpu_intersect"

    def __init__(self, bvh: RefBVH, compact: bool = True):
        self.src = bvh
        self.h = lib().ref_bvhgpu_from_bvh(bvh.h, int(compact))

    def __del__(self):
        if self.h:
            lib().ref_bvhgpu_destroy(self.h)
            self.h = None

    used_nodes = property(lambda s: lib().ref_bvhgpu_used_nodes(s.h))
    nodes = property(lambda s: _view(lib().ref_bvhgpu_nodes(s.h), NODE64, s.used_nodes))


class RefCWBVH(_Traceable):
    """mode 0 Build, 1 BuildHQ, 2 = the Build conversion chain over the scalar BVH::Build tree."""
    _intersect = "ref_cwbvh_intersect"

    def __init__(self, verts: np.ndarray, mode: int = 2, threaded: bool = False):
        self.verts = np.ascontiguousarray(verts, np.float32).reshape(-1, 4)
        self.h = lib().ref_cwbvh_build(_ptr(self.verts), self.verts.shape[0] // 3, mode, int(threaded))

    def __del__(self):
        if self.h:
            lib().ref_cwbvh_destroy(self.h)
            self.h = None

    used_blocks = property(lambda s: lib().ref_cwbvh_used_blocks(s.h))
    idx_count = property(lambda s: lib().ref_cwbvh_idx_count(s.h))
    nodes = property(lambda s: _view(lib().ref_cwbvh_nodes(s.h), np.float32, s.used_blocks * 4).reshape(-1, 4))
    tris = property(lambda s: _view(lib().ref_cwbvh_tris(s.h), np.float32, s.idx_count * 12).reshape(-1, 4))

    def source_bvh(self) -> RefBVH:
        return RefBVH(_handle=lib().ref_cwbvh_source_bvh(self.h), _owner=self)


class RefBVH8CPU(_Traceable):
    """BVH8_CPU (AVX2) - the CPU performance baseline; NOT a parity oracle (SURVEY 8c)."""
    _intersect, _occluded = "ref_bvh8cpu_intersect", "ref_bvh8cpu_occluded"

    def __init__(self, verts: np.ndarray, hq: bool = False):
        self.verts = np.ascontiguousarray(verts, np.float32).reshape(-1, 4)
        self.h = lib().ref_bvh8cpu_build(_ptr(self.verts), self.verts.shape[0] // 3, int(hq))

    def __del__(self):
        if self.h:
            lib().ref_bvh8cpu_destroy(self.h)
            self.h = None


def hardware_threads() -> int:
    return lib().ref_hardware_threads()
