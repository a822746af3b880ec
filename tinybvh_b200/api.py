"""Python mirror of the reference's operator interface for the hot path, over the C-ABI.

Names, argument meaning and error behaviour follow tiny_bvh.h: `BVH.Build(verts, primCount)` (:2124),
`BVH.Intersect` (:3222) / `IsOccluded` (:3382) - here over whole `Ray` batches (the reference has per-ray calls only;
its GPU "batch" is a kernel launch, tiny_bvh_speedtest.cpp:1092-1241) -, `BVH_GPU.ConvertFrom` (:4612),
`BVH8_CWBVH.ConvertFrom` (:5884).  Rays are numpy arrays of the 128-byte host record (rays.RAY_DTYPE) or torch CUDA
tensors of 64-/128-byte records.  Errors raise TbvhError (the reference prints and exit(1)s, :1617-1620).
"""
from __future__ import annotations

import ctypes as C
import numpy as np

from . import _lib
from ._lib import LAYOUT_BVH, LAYOUT_BVH_GPU, LAYOUT_CWBVH, HOST, DEVICE, BUILD_PLOC, TbvhError, check

NODE32 = np.dtype([("aabbMin", "3f4"), ("leftFirst", "u4"), ("aabbMax", "3f4"), ("triCount", "u4")])
NODE64 = np.dtype([("lmin", "3f4"), ("left", "u4"), ("lmax", "3f4"), ("right", "u4"),
                   ("rmin", "3f4"), ("triCount", "u4"), ("rmax", "3f4"), ("firstTri", "u4")])

_contexts = {}


def context(device: int = 0):
    """One engine context per CUDA device (lazily created)."""
    if device not in _contexts:
        h = C.c_void_p()
        check(_lib.lib().tbvh_ctx_create(device, C.byref(h)))
        _contexts[device] = h
    return _contexts[device]


def set_option(key: str, value: int, device: int = 0) -> None:
    """Tuning knob of the engine context (tbvh_set_option).  Keys:
      traversal     trace_variant (BVH2 walk kernel: 0 generic, 3 octant switch, 4 persistent warps),
                    inst_idx_bits (the host program's INST_IDX_BITS: 32, or 4..31 top bits of hit.prim)
      Build         small_t (subtrees of at most this many primitives go to the warp kernel, 8..256),
                    small_mode (warp kernel: bit 0 fragments staged in shared memory, bit 1 aggregated bin updates),
                    build_mode (0 one persistent launch for the large phase, 1 one launch per stage and level),
                    build_ctas (CTAs per SM of the persistent large phase, 0 = default, capped at the occupancy and 16)
      BuildHQ       hq_small (nodes of at most this many fragments go to the warp-per-subtree kernel, clamped to 8..256),
                    hq_cluster (largest thread-block cluster a node of the level phase may get, clamped to 1..16)
      host rays     d2h_mode (0..3), h2d_split (1..4), host_path (0, 1, 2), scatter_threads (1..64), chunk_rays (>= 4096)
    An unknown key raises TbvhError."""
    check(_lib.lib().tbvh_set_option(context(device), key.encode(), int(value)))


def device_count() -> int:
    return _lib.lib().tbvh_device_count()


def launch_count() -> int:
    return int(_lib.lib().tbvh_launch_count())


def _np_ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


def _is_torch(x) -> bool:
    return type(x).__module__.startswith("torch")


def _stream_arg(stream, device):
    """cudaStream_t of a `stream` argument: a torch.cuda.Stream, a raw handle, or None for torch's current stream on `device`."""
    import torch
    if stream is None:
        return torch.cuda.current_stream(device).cuda_stream
    return getattr(stream, "cuda_stream", stream)


def _verts_arg(verts):
    """-> (pointer, stride, vertex count, space, keepalive)"""
    if _is_torch(verts):
        import torch
        assert verts.is_cuda and verts.is_contiguous() and verts.dtype.is_floating_point and verts.element_size() == 4
        v = verts.reshape(-1, 4)
        # device-space inputs are read on the engine's own stream (include/tinybvh_b200.h "device-space inputs"): whatever torch
        # has queued to produce them must have finished
        torch.cuda.current_stream(verts.device).synchronize()
        return C.c_void_p(v.data_ptr()), 16, v.shape[0], DEVICE, v
    v = np.ascontiguousarray(verts, np.float32).reshape(-1, 4)
    return _np_ptr(v), 16, v.shape[0], HOST, v


def _query_radius(points, r):
    """(n, 4) rows are {x, y, z, r} records whose fourth column is the radius; (n, 3) points take the radius from r (a scalar or one per
    point).  Giving both, or neither, is an error."""
    assert points.ndim == 2 and points.shape[1] in (3, 4), "points must be (n, 3) or (n, 4)"
    if points.shape[1] == 4 and r is not None:
        raise TbvhError("(n, 4) queries carry their radius in the fourth column: pass no radius argument")
    if points.shape[1] == 3 and r is None:
        raise TbvhError("(n, 3) points need a radius argument (np.inf: unbounded)")


def _np_queries(points, r):
    """-> contiguous float32 {x, y, z, r} rows (_query_radius's rules)"""
    p = np.asarray(points, np.float32)
    _query_radius(p, r)
    if p.shape[1] == 4:
        return np.ascontiguousarray(p)
    q = np.empty((p.shape[0], 4), np.float32)
    q[:, :3] = p
    q[:, 3] = np.asarray(r, np.float32)
    return q


def _torch_queries(points, r):
    """_np_queries for a CUDA tensor, made on torch's current stream"""
    import torch
    assert points.is_cuda, "points must be a CUDA tensor"
    _query_radius(points, r)
    if points.shape[1] == 4:
        return points.to(torch.float32).contiguous()
    q = torch.empty((points.shape[0], 4), dtype=torch.float32, device=points.device)
    q[:, :3] = points
    q[:, 3] = torch.as_tensor(r, dtype=torch.float32, device=points.device)
    return q


class _Base:
    layout = LAYOUT_BVH
    build_flavour = _lib.BUILD_AVX   # derived layouts build through BuildDefault; set to _lib.BUILD_REFERENCE for BVH::Build's tree

    def __init__(self, device: int = 0):
        self.device = device
        self.ctx = context(device)
        self.h = C.c_void_p()
        check(_lib.lib().tbvh_bvh_create(self.ctx, C.byref(self.h)))
        self.c_trav, self.c_int = 1.0, 1.0  # BVHBase::c_trav / c_int (:819-820)
        self.vert_count = 0                 # vertices of the last build when it was indexed (refit_batch_indexed), else 0

    def _build(self, vertices, primCount, flavour, indices=None):
        """tbvh_build_flavour, or tbvh_build_indexed for the (vertices, indices, primCount) overloads (tiny_bvh.h:889-900)."""
        p, stride, nv, space, keep = _verts_arg(vertices)
        self.vert_count = 0
        if indices is None:
            check(_lib.lib().tbvh_build_flavour(self.h, p, stride, primCount or nv // 3, space, self.c_trav, self.c_int, flavour))
            return
        if _is_torch(indices):
            assert space == DEVICE and indices.is_cuda and indices.is_contiguous() and indices.element_size() == 4
            ip, ni = C.c_void_p(indices.data_ptr()), indices.numel()
        else:
            assert space == HOST, "device vertices need device indices"
            indices = np.ascontiguousarray(indices, np.uint32).reshape(-1)
            ip, ni = _np_ptr(indices), indices.shape[0]
        check(_lib.lib().tbvh_build_indexed(self.h, p, stride, nv, ip, primCount or ni // 3, space, self.c_trav, self.c_int, flavour))
        self.vert_count = nv

    def __del__(self):
        try:
            if getattr(self, "h", None) and self.h.value:
                _lib.lib().tbvh_bvh_destroy(self.h)
                self.h = None
        except Exception:
            pass

    # -- info (the reference's public members usedNodes / idxCount / triCount / aabbMin / aabbMax)
    def info(self) -> _lib.Info:
        i = _lib.Info()
        check(_lib.lib().tbvh_bvh_info(self.h, C.byref(i)))
        return i

    usedNodes = property(lambda s: s.info().used_nodes)
    idxCount = property(lambda s: s.info().idx_count)
    triCount = property(lambda s: s.info().prim_count)

    # -- traversal over batches
    def Intersect(self, rays, hits=None, stream=None):
        """Closest hit for every ray, in place (t,u,v,prim at bytes 48..63).  numpy -> host path (copies inside);
        torch CUDA tensor -> device path, asynchronous on `stream` (a torch.cuda.Stream or a raw cudaStream_t; default: torch's
        current stream)."""
        L = _lib.lib()
        if _is_torch(rays):
            assert rays.is_cuda and rays.is_contiguous()
            stride = rays.stride(0) * rays.element_size() if rays.dim() > 1 else None
            assert stride in (64, 128), "ray tensor must be [n, 64|128 bytes]"
            st = _stream_arg(stream, rays.device)
            hp = C.c_void_p(hits.data_ptr()) if hits is not None else None
            check(L.tbvh_intersect_device(self.h, self.layout, C.c_void_p(rays.data_ptr()), stride, hp, rays.shape[0], C.c_void_p(st)))
            return rays if hits is None else hits
        assert rays.dtype.itemsize in (64, 128) and rays.flags.c_contiguous
        check(L.tbvh_intersect(self.h, self.layout, _np_ptr(rays), rays.dtype.itemsize, rays.shape[0]))
        return rays

    def IntersectPacked(self, rays, hits=None):
        """Host path with packed results: rays untouched, hits -> HIT_DTYPE array (tbvh_intersect_packed)."""
        from .rays import HIT_DTYPE
        assert not _is_torch(rays) and rays.dtype.itemsize in (64, 128) and rays.flags.c_contiguous
        if hits is None:
            hits = np.zeros(rays.shape[0], HIT_DTYPE)
        check(_lib.lib().tbvh_intersect_packed(self.h, self.layout, _np_ptr(rays), rays.dtype.itemsize, rays.shape[0], _np_ptr(hits)))
        return hits

    def IsOccluded(self, rays, bits=None, stream=None):
        """Any hit within [0, ray.hit.t] per ray -> uint32 bit mask, bit (i&31) of word i>>5."""
        L = _lib.lib()
        if _is_torch(rays):
            import torch
            assert rays.is_cuda and rays.is_contiguous()
            stride = rays.stride(0) * rays.element_size()
            n = rays.shape[0]
            if bits is None:
                bits = torch.empty((n + 31) // 32, dtype=torch.int32, device=rays.device)
            st = _stream_arg(stream, rays.device)
            check(L.tbvh_occluded_device(self.h, self.layout, C.c_void_p(rays.data_ptr()), stride, C.c_void_p(bits.data_ptr()), n, C.c_void_p(st)))
            return bits
        assert rays.dtype.itemsize in (64, 128) and rays.flags.c_contiguous
        n = rays.shape[0]
        if bits is None:
            bits = np.zeros((n + 31) // 32, np.uint32)
        check(L.tbvh_occluded(self.h, self.layout, _np_ptr(rays), rays.dtype.itemsize, n, _np_ptr(bits)))
        return bits

    # -- proximity queries over the BVH-layout tree (tbvh_closest_point / tbvh_sphere_overlap, DESIGN.md §4.9)
    def closest_point(self, points, r_max=None, stream=None):
        """Nearest triangle within r_max of every point -> (d, u, v, prim): the closest point is v0 + u (v1 - v0) + v (v2 - v0) of
        triangle prim; prim 0xffffffff and d = r_max where nothing lies within r_max.  points: (n, 3) with r_max a scalar or one per
        point (np.inf: unbounded), or (n, 4) {x, y, z, r_max} records, the C-ABI's own, with r_max left out (TbvhError otherwise).  numpy -> host path, numpy arrays (prim uint32); torch CUDA tensor -> device path, everything queued
        on `stream` (default: torch's current stream), tensors (prim as int32 bits).  No autograd."""
        L = _lib.lib()
        if _is_torch(points):
            import torch
            st = _stream_arg(stream, points.device)
            with torch.cuda.stream(torch.cuda.ExternalStream(st, device=points.device)):
                q = _torch_queries(points, r_max)
                rec = torch.empty((q.shape[0], 4), dtype=torch.float32, device=q.device)
                check(L.tbvh_closest_point(self.h, C.c_void_p(q.data_ptr()), C.c_void_p(rec.data_ptr()), q.shape[0], DEVICE, C.c_void_p(st)))
            return rec[:, 0], rec[:, 1], rec[:, 2], rec[:, 3].view(torch.int32)
        q = _np_queries(points, r_max)
        rec = np.empty((q.shape[0], 4), np.float32)
        check(L.tbvh_closest_point(self.h, _np_ptr(q), _np_ptr(rec), q.shape[0], HOST, None))
        return rec[:, 0].copy(), rec[:, 1].copy(), rec[:, 2].copy(), rec[:, 3].view(np.uint32).copy()

    def sphere_overlap(self, centers, radii=None, stream=None):
        """The batched BVH::IntersectSphere under the engine's definition: True where some triangle lies within the radius of the centre.
        centers: (n, 3) with radii a scalar or one per centre, or (n, 4) {x, y, z, r} records with radii left out, as closest_point.  numpy -> bool array; torch CUDA tensor -> bool tensor queued on `stream`."""
        L = _lib.lib()
        if _is_torch(centers):
            import torch
            st = _stream_arg(stream, centers.device)
            with torch.cuda.stream(torch.cuda.ExternalStream(st, device=centers.device)):
                q = _torch_queries(centers, radii)
                n = q.shape[0]
                words = torch.empty(max((n + 31) // 32, 1), dtype=torch.int32, device=q.device)
                check(L.tbvh_sphere_overlap(self.h, C.c_void_p(q.data_ptr()), C.c_void_p(words.data_ptr()), n, DEVICE, C.c_void_p(st)))
                shifts = torch.arange(32, dtype=torch.int32, device=q.device)
                return ((words[:, None] >> shifts) & 1).reshape(-1)[:n].bool()
        q = _np_queries(centers, radii)
        n = q.shape[0]
        words = np.zeros(max((n + 31) // 32, 1), np.uint32)
        check(L.tbvh_sphere_overlap(self.h, _np_ptr(q), _np_ptr(words), n, HOST, None))
        return np.unpackbits(words.view(np.uint8), bitorder="little")[:n].astype(bool)

    # -- signed distances (tbvh_signed_distance_prepare / tbvh_signed_distance, DESIGN.md §4.10)
    def prepare_signed_distance(self):
        """Build the pseudonormal table the signed-distance query reads (on the device; returns when done).  Any later build, upload
        of a tree, optimize or refit makes it stale: call this again before the next signed_distance.  Conversions keep it."""
        check(_lib.lib().tbvh_signed_distance_prepare(self.h))
        return self

    def signed_distance(self, points, r_max=None, stream=None):
        """closest_point with the distance signed: negative inside a closed, consistently oriented mesh (outward normals by the
        right-hand rule on v0, v1, v2) -> (sd, u, v, prim).  Where nothing lies within r_max, sd = r_max and prim 0xffffffff (no sign is
        known).  points and r_max follow closest_point's rules; numpy -> host path, torch CUDA tensor -> queued on `stream`."""
        L = _lib.lib()
        if _is_torch(points):
            import torch
            st = _stream_arg(stream, points.device)
            with torch.cuda.stream(torch.cuda.ExternalStream(st, device=points.device)):
                q = _torch_queries(points, r_max)
                rec = torch.empty((q.shape[0], 4), dtype=torch.float32, device=q.device)
                check(L.tbvh_signed_distance(self.h, C.c_void_p(q.data_ptr()), C.c_void_p(rec.data_ptr()), q.shape[0], DEVICE, C.c_void_p(st)))
            return rec[:, 0], rec[:, 1], rec[:, 2], rec[:, 3].view(torch.int32)
        q = _np_queries(points, r_max)
        rec = np.empty((q.shape[0], 4), np.float32)
        check(L.tbvh_signed_distance(self.h, _np_ptr(q), _np_ptr(rec), q.shape[0], HOST, None))
        return rec[:, 0].copy(), rec[:, 1].copy(), rec[:, 2].copy(), rec[:, 3].view(np.uint32).copy()

    # -- generalized winding numbers (tbvh_winding_number_prepare / tbvh_winding_number, DESIGN.md §4.11)
    def prepare_winding_number(self):
        """Build the table of subtree moments the winding-number query reads (on the device; returns when done).  Any later build,
        upload of a tree, optimize or refit makes it stale: call this again before the next winding_number.  Conversions keep it."""
        check(_lib.lib().tbvh_winding_number_prepare(self.h))
        return self

    def winding_number(self, points, beta=2.0, stream=None):
        """The generalized winding number of every point -> w: 1 inside and 0 outside a closed mesh with outward normals (right-hand
        rule on v0, v1, v2), 2 where two such solids overlap, smooth across holes; NaN for a NaN coordinate.  Subtrees farther than
        beta times their radius take a second-order expansion (beta > 1; 2 as Barill et al. recommend; np.inf: the exact sum).
        points: (n, 3), or (n, 4) with the fourth column ignored.  numpy -> host path, float32 array; torch CUDA tensor -> float32
        tensor queued on `stream` (default: torch's current stream).
        An inside/outside sign that works on open meshes: d from closest_point, negative where winding_number(...) > 0.5."""
        L = _lib.lib()
        assert points.ndim == 2 and points.shape[1] in (3, 4), "points must be (n, 3) or (n, 4)"
        if _is_torch(points):
            import torch
            assert points.is_cuda, "points must be a CUDA tensor"
            st = _stream_arg(stream, points.device)
            with torch.cuda.stream(torch.cuda.ExternalStream(st, device=points.device)):
                q = torch.zeros((points.shape[0], 4), dtype=torch.float32, device=points.device)
                q[:, :3] = points[:, :3]
                w = torch.empty(q.shape[0], dtype=torch.float32, device=q.device)
                check(L.tbvh_winding_number(self.h, C.c_void_p(q.data_ptr()), C.c_void_p(w.data_ptr()), q.shape[0], float(beta), DEVICE, C.c_void_p(st)))
            return w
        p = np.asarray(points, np.float32)
        q = np.zeros((p.shape[0], 4), np.float32)
        q[:, :3] = p[:, :3]
        w = np.empty(q.shape[0], np.float32)
        check(L.tbvh_winding_number(self.h, _np_ptr(q), _np_ptr(w), q.shape[0], float(beta), HOST, None))
        return w

    # -- intersecting triangle pairs (tbvh_mesh_overlap_pairs / tbvh_mesh_overlap_bits, DESIGN.md §4.12)
    def overlap_pairs(self, other=None, stream=None):
        """The pairs (i, j) of a triangle i of self and a triangle j of other that intersect (closed triangles: touching counts), sorted
        by (i, j) -> (m, 2).  other=None: the self-intersections of this mesh, pairs i < j, where neighbours that only share corners or an
        edge are not reported (DESIGN.md §4.12).  Both handles' vertices are in one space.  stream=None -> uint32 numpy array;
        a torch.cuda.Stream (or raw cudaStream_t) -> int32 CUDA tensor holding the bits of the uint32 values, the work ordered after
        that stream's.  The call returns when done; it starts with a capacity guess and repeats once with the returned count."""
        L = _lib.lib()
        o = self if other is None else other
        n = self.triCount
        count = C.c_uint64()
        if stream is None:
            out = np.zeros((max(n, 1), 2), np.uint32)
            check(L.tbvh_mesh_overlap_pairs(self.h, o.h, _np_ptr(out), out.shape[0], C.byref(count), HOST, None))
            if count.value > out.shape[0]:
                out = np.zeros((count.value, 2), np.uint32)
                check(L.tbvh_mesh_overlap_pairs(self.h, o.h, _np_ptr(out), out.shape[0], C.byref(count), HOST, None))
            return out[: count.value].copy()
        import torch
        st = getattr(stream, "cuda_stream", stream)
        dev = torch.device("cuda", self.device)
        out = torch.empty((max(n, 1), 2), dtype=torch.int32, device=dev)
        check(L.tbvh_mesh_overlap_pairs(self.h, o.h, C.c_void_p(out.data_ptr()), out.shape[0], C.byref(count), DEVICE, C.c_void_p(st)))
        if count.value > out.shape[0]:
            out = torch.empty((count.value, 2), dtype=torch.int32, device=dev)
            check(L.tbvh_mesh_overlap_pairs(self.h, o.h, C.c_void_p(out.data_ptr()), out.shape[0], C.byref(count), DEVICE, C.c_void_p(st)))
        return out[: count.value]

    def overlapping(self, other=None, stream=None):
        """Per triangle of self: True where it intersects some triangle of other (other=None: some other triangle of this mesh, under
        overlap_pairs' rules for neighbours).  stream=None -> numpy bool array; a torch.cuda.Stream (or raw cudaStream_t) -> bool CUDA
        tensor queued on that stream."""
        L = _lib.lib()
        o = self if other is None else other
        n = self.triCount
        if stream is None:
            words = np.zeros(max((n + 31) // 32, 1), np.uint32)
            check(L.tbvh_mesh_overlap_bits(self.h, o.h, _np_ptr(words), HOST, None))
            return np.unpackbits(words.view(np.uint8), bitorder="little")[:n].astype(bool)
        import torch
        st = getattr(stream, "cuda_stream", stream)
        dev = torch.device("cuda", self.device)
        with torch.cuda.stream(torch.cuda.ExternalStream(st, device=dev)):
            words = torch.empty(max((n + 31) // 32, 1), dtype=torch.int32, device=dev)
            check(L.tbvh_mesh_overlap_bits(self.h, o.h, C.c_void_p(words.data_ptr()), DEVICE, C.c_void_p(st)))
            shifts = torch.arange(32, dtype=torch.int32, device=dev)
            return ((words[:, None] >> shifts) & 1).reshape(-1)[:n].bool()

    # -- distances between meshes (tbvh_mesh_distance / tbvh_mesh_distance_pairs, DESIGN.md §4.13)
    def nearest_triangles(self, other=None, r_max=np.inf, stream=None):
        """The nearest triangle of other within r_max of every triangle of self -> (d, j): j 0xffffffff and d = r_max where there is none
        (or the triangle has a non-finite coordinate).  other=None: the nearest triangle of this mesh that shares no corner with it (thin
        walls, near-touching sheets).  Both handles' vertices are in one space; the separation of the meshes is d.min().
        stream=None -> numpy arrays (d float32, j uint32); a torch.cuda.Stream (or raw cudaStream_t) -> CUDA tensors (j as int32 bits)
        queued on that stream."""
        L = _lib.lib()
        o = self if other is None else other
        n = self.triCount
        if stream is None:
            rec = np.zeros((n, 2), np.float32)
            check(L.tbvh_mesh_distance(self.h, o.h, float(r_max), _np_ptr(rec), HOST, None))
            return rec[:, 0].copy(), rec[:, 1].view(np.uint32).copy()
        import torch
        st = getattr(stream, "cuda_stream", stream)
        dev = torch.device("cuda", self.device)
        with torch.cuda.stream(torch.cuda.ExternalStream(st, device=dev)):
            rec = torch.empty((max(n, 1), 2), dtype=torch.float32, device=dev)
            check(L.tbvh_mesh_distance(self.h, o.h, float(r_max), C.c_void_p(rec.data_ptr()), DEVICE, C.c_void_p(st)))
        return rec[:n, 0], rec[:n, 1].view(torch.int32)

    def distance_pairs(self, other=None, r=None, stream=None):
        """The pairs (i, j) of a triangle i of self and a triangle j of other within distance r of each other (r = 0: touching and
        crossing pairs), sorted by (i, j) -> (m, 2).  other=None: pairs i < j of this mesh that share no corner.  stream and the
        capacity retry as overlap_pairs."""
        if r is None:
            raise TbvhError("distance_pairs needs a distance r")
        L = _lib.lib()
        o = self if other is None else other
        n = self.triCount
        count = C.c_uint64()
        if stream is None:
            out = np.zeros((max(n, 1), 2), np.uint32)
            check(L.tbvh_mesh_distance_pairs(self.h, o.h, float(r), _np_ptr(out), out.shape[0], C.byref(count), HOST, None))
            if count.value > out.shape[0]:
                out = np.zeros((count.value, 2), np.uint32)
                check(L.tbvh_mesh_distance_pairs(self.h, o.h, float(r), _np_ptr(out), out.shape[0], C.byref(count), HOST, None))
            return out[: count.value].copy()
        import torch
        st = getattr(stream, "cuda_stream", stream)
        dev = torch.device("cuda", self.device)
        out = torch.empty((max(n, 1), 2), dtype=torch.int32, device=dev)
        check(L.tbvh_mesh_distance_pairs(self.h, o.h, float(r), C.c_void_p(out.data_ptr()), out.shape[0], C.byref(count), DEVICE, C.c_void_p(st)))
        if count.value > out.shape[0]:
            out = torch.empty((count.value, 2), dtype=torch.int32, device=dev)
            check(L.tbvh_mesh_distance_pairs(self.h, o.h, float(r), C.c_void_p(out.data_ptr()), out.shape[0], C.byref(count), DEVICE, C.c_void_p(st)))
        return out[: count.value]

    def device_view(self, layout: int = None) -> _lib.DeviceView:
        """tbvh_device_view: the view a kernel of the caller's passes to the device functions of include/tinybvh_b200_device.cuh, for
        `layout` (default: the layout Intersect walks).  Host work only; valid until the handle's arrays change (include/tinybvh_b200.h)."""
        v = _lib.DeviceView()
        check(_lib.lib().tbvh_device_view(self.h, self.layout if layout is None else layout, C.byref(v)))
        return v

    def set_stats(self, enable: bool):
        check(_lib.lib().tbvh_set_stats(self.h, int(enable)))

    def get_stats(self):
        """(node visits, triangle tests, CWBVH child-pair steps) of the last traversal call with statistics enabled"""
        out = (C.c_uint64 * 4)()
        check(_lib.lib().tbvh_get_stats_ex(self.h, C.byref(out)))
        return out[0], out[1], out[2]


class BVH(_Base):
    """tinybvh::BVH (tiny_bvh.h:846-985): Wald 32-byte nodes; binned-SAH Build on the GPU."""
    layout = LAYOUT_BVH

    def Build(self, vertices, primCount: int = 0, indices=None):
        """BVH::Build( vertices, primCount ) :2124 / ( vertices, indices, primCount ) :2139."""
        self._build(vertices, primCount, _lib.BUILD_REFERENCE, indices)
        return self

    def BuildAVX(self, vertices, primCount: int = 0, indices=None):
        """BVH::BuildAVX (tiny_bvh.h:6400) - the flavour BuildDefault uses on x86."""
        self._build(vertices, primCount, _lib.BUILD_AVX, indices)
        return self

    def BuildHQ(self, vertices, primCount: int = 0, indices=None):
        """BVH::BuildHQ (tiny_bvh.h:2623): SBVH with spatial splits; idxCount becomes primCount + primCount/2."""
        self._build(vertices, primCount, _lib.BUILD_HQ, indices)
        return self

    def BuildPLOC(self, vertices, primCount: int = 0, indices=None):
        """Not in the reference: the bottom-up PLOC build (TBVH_BUILD_PLOC, DESIGN.md §4.8), a refittable tree for per-frame rebuilds."""
        self._build(vertices, primCount, _lib.BUILD_PLOC, indices)
        return self

    def SAHCost(self) -> float:
        """BVH::SAHCost( 0 ) (tiny_bvh.h:1889): host recursion over the downloaded nodes, the reference's value bit for bit."""
        out = C.c_float()
        check(_lib.lib().tbvh_sah_cost(self.h, self.c_trav, self.c_int, C.byref(out)))
        return float(out.value)

    def optimize(self, max_rounds: int, c_trav: float = 1.0, c_int: float = 1.0):
        """tbvh_optimize: rounds of parallel subtree reinsertion on the device that lower the tree's SAH cost; not the reference's
        BVH::Optimize (tiny_bvh.h:3043), which reinserts one subtree at a time.  -> (rounds kept, final SAHCost)."""
        return _optimize(self, max_rounds, c_trav, c_int)

    def Refit(self, vertices):
        """BVH::Refit (tiny_bvh.h:3055): same triangles, new positions.  The reference re-reads the caller's vertex array through
        the pointer it kept; the engine holds its own copy, so the array is passed again."""
        p, stride, nv, space, keep = _verts_arg(vertices)
        check(_lib.lib().tbvh_refit(self.h, p, stride, nv // 3, space))
        return self

    def upload(self, nodes, primIdx, vertices):
        """Consume a tree built elsewhere in the reference's BVH layout (bvhNode / primIdx / verts, :952-964)."""
        p, stride, nv, space, keep = _verts_arg(vertices)
        nodes = np.ascontiguousarray(nodes)
        primIdx = np.ascontiguousarray(primIdx, np.uint32)
        assert nodes.dtype.itemsize == 32
        self.vert_count = 0
        check(_lib.lib().tbvh_upload_bvh(self.h, _np_ptr(nodes), nodes.shape[0], _np_ptr(primIdx), primIdx.shape[0], p, stride, nv // 3, space))
        return self

    def download(self):
        """-> (bvhNode[usedNodes] as NODE32, primIdx[idxCount]) in the reference layout."""
        i = self.info()
        nodes = np.zeros(i.used_nodes, NODE32)
        idx = np.zeros(i.idx_count, np.uint32)
        check(_lib.lib().tbvh_download_bvh(self.h, _np_ptr(nodes), _np_ptr(idx), HOST))
        return nodes, idx


BLAS_INSTANCE = np.dtype([("transform", "16f4"), ("invTransform", "16f4"), ("aabbMin", "3f4"), ("blasIdx", "u4"),
                          ("aabbMax", "3f4"), ("mask", "u4"), ("dummy", "8u4")])   # tinybvh::BLASInstance, tiny_bvh.h:1443 (192 bytes)


class TLAS(BVH):
    """A tinybvh::BVH built with Build( BLASInstance*, instCount, BVHBase**, blasCount ) (tiny_bvh.h:2221): Intersect / IsOccluded on
    it are IntersectTLAS / IsOccludedTLAS.  `instances`: BLAS_INSTANCE records already Update()d by the caller (inverse transform
    and world box, as BLASInstance::Update :8386 computes them); `blasses`: BVH objects of this module, kept alive by this one."""

    def Build(self, instances, blasses, update: bool = True, blas_layout: int = LAYOUT_BVH):
        """update=True: BLASInstance::Update (:8386) is applied to every record first - in place, as the reference's Build does when it
        is handed the BLAS list (:2245-2250); update=False: the records already carry inverse transform and world box.
        blas_layout=LAYOUT_CWBVH: Intersect / IsOccluded walk every BLAS in its BVH8_CWBVH layout (the arrangement of the reference's GPU
        path, traverse_tlas.cl); the BLASses must hold that layout when the TLAS is built (BVH8_CWBVH objects, or tbvh_convert)."""
        inst = instances
        self.layout = blas_layout
        assert inst.dtype.itemsize == 192 and inst.flags.c_contiguous
        self.blasses = list(blasses)
        if update:
            if int(inst["blasIdx"].max()) >= len(self.blasses):
                raise TbvhError("TLAS: an instance names a BLAS past the list")
            for i in range(inst.shape[0]):
                check(_lib.lib().tbvh_instance_update(C.c_void_p(inst[i:i + 1].ctypes.data), self.blasses[int(inst["blasIdx"][i])].h))
        hs = (C.c_void_p * len(self.blasses))(*[b.h for b in self.blasses])
        self.vert_count = 0
        check(_lib.lib().tbvh_build_tlas(self.h, _np_ptr(inst), 192, inst.shape[0], hs, len(self.blasses), self.c_trav, self.c_int))
        return self

    def Rebuild(self, instances, blasses=None, blas_layout: int = None):
        """The per-frame call of an animated scene (tbvh_build_tlas_update): BLASInstance::Update of every record on the device and the
        TLAS over the new boxes, in one call.  The records end up as Build( .., update=True ) leaves them, and so does the TLAS.
        instances: a NumPy array of BLAS_INSTANCE records, or of bytes with shape [n, >= 160] (rows a multiple of 4 bytes apart),
        updated in place through one copy each way; or a CUDA torch tensor of bytes, shape [n, >= 160] with rows a multiple of 16
        bytes apart at a 16-byte-aligned address, updated in place on the device - transforms written by a torch kernel never
        visit the host.
        blasses / blas_layout: as for Build; by default those of the last Build or Rebuild.  On the handle of a TLAS of the same
        instance and BLAS counts the device tables are reused."""
        if blasses is not None:
            self.blasses = list(blasses)
        if blas_layout is not None:
            self.layout = blas_layout
        if not getattr(self, "blasses", None):
            raise TbvhError("TLAS.Rebuild: no BLAS list (pass blasses, or Build first)")
        if _is_torch(instances):
            import torch
            assert instances.is_cuda and instances.dim() == 2 and instances.element_size() == 1 and instances.stride(1) == 1 and instances.shape[1] >= 160
            torch.cuda.current_stream(instances.device).synchronize()   # device-space input: read on the engine's own stream
            p, stride, n, space = C.c_void_p(instances.data_ptr()), instances.stride(0), instances.shape[0], DEVICE
        else:
            assert instances.flags.writeable and (instances.ndim == 1 and instances.dtype.itemsize >= 160 or
                                                  instances.ndim == 2 and instances.dtype.itemsize == 1 and instances.strides[1] == 1 and instances.shape[1] >= 160)
            p, stride, n, space = _np_ptr(instances), instances.strides[0], instances.shape[0], HOST
        hs = (C.c_void_p * len(self.blasses))(*[b.h for b in self.blasses])
        self.vert_count = 0
        check(_lib.lib().tbvh_build_tlas_update(self.h, p, stride, n, space, hs, len(self.blasses), self.c_trav, self.c_int))
        return self


def _optimize(obj, max_rounds, c_trav, c_int, layout=LAYOUT_BVH):
    rounds, sah = C.c_uint32(), C.c_float()
    check(_lib.lib().tbvh_optimize(obj.h, max_rounds, c_trav, c_int, C.byref(rounds), C.byref(sah)))
    if rounds.value and layout != LAYOUT_BVH:
        check(_lib.lib().tbvh_convert(obj.h, layout))   # the optimised BVH2 converted again, as Build converts the built one
    return int(rounds.value), float(sah.value)


def _refit_layouts(obj, vertices):
    p, stride, nv, space, keep = _verts_arg(vertices)
    check(_lib.lib().tbvh_refit_layouts(obj.h, p, stride, nv // 3, space))
    return obj


class BVH_GPU(_Base):
    """tinybvh::BVH_GPU (tiny_bvh.h:1092-1127): Aila-Laine 64-byte nodes."""
    layout = LAYOUT_BVH_GPU

    def Build(self, vertices, primCount: int = 0, indices=None):
        # BVH_GPU::Build -> bvh.BuildDefault (tiny_bvh.h:4580-4590) = BuildAVX on x86, then ConvertFrom
        self._build(vertices, primCount, self.build_flavour, indices)
        check(_lib.lib().tbvh_convert(self.h, LAYOUT_BVH_GPU))
        return self

    def BuildHQ(self, vertices, primCount: int = 0, indices=None):
        """BVH_GPU::BuildHQ (tiny_bvh.h:4588): bvh.BuildHQ, then ConvertFrom."""
        self._build(vertices, primCount, _lib.BUILD_HQ, indices)
        check(_lib.lib().tbvh_convert(self.h, LAYOUT_BVH_GPU))
        return self

    def optimize(self, max_rounds: int, c_trav: float = 1.0, c_int: float = 1.0):
        """BVH.optimize of the underlying tree, then ConvertFrom again on the device.  -> (rounds kept, final SAHCost)."""
        return _optimize(self, max_rounds, c_trav, c_int, LAYOUT_BVH_GPU)

    def Refit(self, vertices):
        """BVH::Refit of the underlying tree, then ConvertFrom again on the device (tbvh_refit_layouts): same triangles, new
        positions, numpy or torch CUDA vertices as BVH.Refit."""
        return _refit_layouts(self, vertices)

    def upload(self, nodes, primIdx, vertices):
        p, stride, nv, space, keep = _verts_arg(vertices)
        nodes = np.ascontiguousarray(nodes)
        primIdx = np.ascontiguousarray(primIdx, np.uint32)
        assert nodes.dtype.itemsize == 64
        self.vert_count = 0
        check(_lib.lib().tbvh_upload_bvh_gpu(self.h, _np_ptr(nodes), nodes.shape[0], _np_ptr(primIdx), primIdx.shape[0], p, stride, nv // 3, space))
        return self

    def download(self):
        i = self.info()
        nodes = np.zeros(i.used_nodes_gpu, NODE64)
        check(_lib.lib().tbvh_download_bvh_gpu(self.h, _np_ptr(nodes), HOST))
        return nodes


class BVH8_CWBVH(_Base):
    """tinybvh::BVH8_CWBVH (tiny_bvh.h:1334-1362): 80-byte compressed wide nodes + 48-byte triangles."""
    layout = LAYOUT_CWBVH

    def Build(self, vertices, primCount: int = 0, indices=None):
        # BVH8_CWBVH::Build -> bvh8.bvh.BuildDefault (tiny_bvh.h:5830) = BuildAVX on x86, then the conversion chain
        self._build(vertices, primCount, self.build_flavour, indices)
        check(_lib.lib().tbvh_convert(self.h, LAYOUT_CWBVH))
        return self

    def BuildHQ(self, vertices, primCount: int = 0, indices=None):
        """BVH8_CWBVH::BuildHQ (tiny_bvh.h:5859): bvh.BuildHQ, SplitLeafs(3), 8-wide collapse, CWBVH encode."""
        self._build(vertices, primCount, _lib.BUILD_HQ, indices)
        check(_lib.lib().tbvh_convert(self.h, LAYOUT_CWBVH))
        return self

    def optimize(self, max_rounds: int, c_trav: float = 1.0, c_int: float = 1.0):
        """BVH.optimize of the underlying tree, then the CWBVH conversion chain again.  -> (rounds kept, final SAHCost)."""
        return _optimize(self, max_rounds, c_trav, c_int, LAYOUT_CWBVH)

    def Refit(self, vertices):
        """Refit without a new collapse (tbvh_refit_layouts): BVH::Refit of the underlying tree, then BVH8_CWBVH::ConvertFrom of the
        8-wide collapse kept from the last conversion with the refitted boxes - same wide-node count, in place.  The reference has no
        BVH8_CWBVH::Refit; it refits the BVH2 and converts again (Build once more for that)."""
        return _refit_layouts(self, vertices)

    def upload(self, bvh8Data, bvh8Tris):
        """bvh8Data: float32 [usedBlocks,4]; bvh8Tris: float32 [3*triCount,4] (public members :1356-1357)."""
        d = np.ascontiguousarray(bvh8Data, np.float32).reshape(-1, 4)
        t = np.ascontiguousarray(bvh8Tris, np.float32).reshape(-1, 4)
        check(_lib.lib().tbvh_upload_cwbvh(self.h, _np_ptr(d), d.shape[0], _np_ptr(t), t.shape[0] // 3, HOST))
        return self

    def download(self):
        i = self.info()
        d = np.zeros((i.used_blocks, 4), np.float32)
        t = np.zeros((i.cwbvh_tri_count * 3, 4), np.float32)
        check(_lib.lib().tbvh_download_cwbvh(self.h, _np_ptr(d), _np_ptr(t), HOST))
        return d, t


def build_batch(bvhs, meshes, flavour: int = _lib.BUILD_REFERENCE, indices=None):
    """tbvh_build_batch: one binned-SAH tree per mesh, all built in one call.  bvhs[i] ends up as bvhs[i].Build(meshes[i]) (flavour
    BUILD_REFERENCE) or .BuildAVX (BUILD_AVX) would leave it; flavour BUILD_HQ builds one SBVH per mesh (tbvh_build_batch_hq), as
    .BuildHQ would, and BUILD_PLOC one PLOC tree per mesh, as .BuildPLOC would.  `meshes`: numpy vertex arrays, or torch CUDA tensors - one space per
    call; `indices`: None, or one entry per mesh (None for a flat mesh, else its vertex indices in the same space).  BVH_GPU and
    BVH8_CWBVH objects are converted afterwards, as their Build does (the BVH8_CWBVH objects in one convert_batch).  A refused batch
    raises TbvhError and leaves every object as it was."""
    bvhs, meshes = list(bvhs), list(meshes)
    if len(bvhs) != len(meshes):
        raise TbvhError("build_batch: one object per mesh")
    indices = [None] * len(meshes) if indices is None else list(indices)
    if len(indices) != len(meshes):
        raise TbvhError("build_batch: one index entry per mesh")
    if len({_is_torch(m) for m in meshes}) > 1:
        raise TbvhError("build_batch: host and device meshes in one call")
    recs = (_lib.Mesh * max(len(meshes), 1))()
    keep, space = [], HOST
    for r, m, ix in zip(recs, meshes, indices):
        p, stride, nv, space, k = _verts_arg(m)
        keep.append(k)
        r.verts, r.stride = p.value, stride
        if ix is None:
            r.vert_count, r.indices, r.prim_count = 0, None, nv // 3
            continue
        if _is_torch(ix):
            assert space == DEVICE and ix.is_cuda and ix.is_contiguous() and ix.element_size() == 4
            r.indices, n = ix.data_ptr(), ix.numel()
        else:
            assert space == HOST, "device vertices need device indices"
            ix = np.ascontiguousarray(ix, np.uint32).reshape(-1)
            r.indices, n = ix.ctypes.data, ix.shape[0]
        keep.append(ix)
        r.vert_count, r.prim_count = nv, n // 3
    hs = (C.c_void_p * max(len(bvhs), 1))(*[b.h for b in bvhs]) if bvhs else None
    c0 = bvhs[0] if bvhs else None
    c_trav, c_int = (c0.c_trav, c0.c_int) if c0 else (1.0, 1.0)
    if flavour == _lib.BUILD_HQ:
        check(_lib.lib().tbvh_build_batch_hq(hs, recs, len(meshes), space, c_trav, c_int))
    else:
        check(_lib.lib().tbvh_build_batch(hs, recs, len(meshes), space, c_trav, c_int, flavour))
    for b, r in zip(bvhs, recs):
        b.vert_count = r.vert_count
    cw = [b for b in bvhs if b.layout == LAYOUT_CWBVH]
    if cw:
        convert_batch(cw)
    for b in bvhs:
        if b.layout == LAYOUT_BVH_GPU:
            check(_lib.lib().tbvh_convert(b.h, b.layout))
    return bvhs


def convert_batch(objs):
    """tbvh_convert_batch: the CWBVH of every object's BVH-layout tree, all converted in one call.  Each object then holds what
    tbvh_convert( h, LAYOUT_CWBVH ) of it alone leaves (BVH8_CWBVH.Build's conversion chain), whatever the other objects of the
    call.  A refused call raises TbvhError and leaves every object as it was."""
    objs = list(objs)
    hs = (C.c_void_p * max(len(objs), 1))(*[b.h for b in objs])
    check(_lib.lib().tbvh_convert_batch(hs, len(objs), LAYOUT_CWBVH))
    return objs


def refit_batch(objs, meshes, keep_layouts=None):
    """tbvh_refit_batch: every object refitted to its mesh's new vertices in one call.  `meshes`: numpy vertex arrays, or torch CUDA
    tensors - one space per call, the same triangles each object was built from.  keep_layouts=None applies the rule of each object's
    own Refit: BVH objects drop their derived layouts (tbvh_refit, keep_layouts=0), BVH_GPU and BVH8_CWBVH objects keep them up to date
    (tbvh_refit_layouts, keep_layouts=1); objects of both kinds in one call need an explicit keep_layouts.  A refused call raises
    TbvhError and leaves every object as it was."""
    return _refit_batch("refit_batch", objs, meshes, keep_layouts, False)


def refit_batch_indexed(objs, meshes, keep_layouts=None):
    """tbvh_refit_batch_indexed: refit_batch for a scene with indexed meshes.  For an object whose last build was indexed
    (Build( vertices, indices=.. ), build_batch with indices) its mesh holds the new positions of the vertices it was built from - the
    same number of rows -, which the engine reads through the indices it kept from the build; for any other object its mesh is the flat
    triangle soup, as in refit_batch.  Each object ends up as its refit from vertices[indices] would leave it.  `meshes`: numpy arrays
    or torch CUDA tensors, one space per call; keep_layouts as for refit_batch.  A refused call raises TbvhError and leaves every
    object as it was."""
    return _refit_batch("refit_batch_indexed", objs, meshes, keep_layouts, True)


def _refit_batch(fn, objs, meshes, keep_layouts, indexed):
    objs, meshes = list(objs), list(meshes)
    if len(objs) != len(meshes):
        raise TbvhError(f"{fn}: one object per mesh")
    if len({_is_torch(m) for m in meshes}) > 1:
        raise TbvhError(f"{fn}: host and device meshes in one call")
    if keep_layouts is None:
        rule = {b.layout != LAYOUT_BVH for b in objs}
        if len(rule) > 1:
            raise TbvhError(f"{fn}: BVH objects drop their layouts, BVH_GPU / BVH8_CWBVH objects keep them: pass keep_layouts")
        keep_layouts = rule.pop() if rule else False
    recs = (_lib.Mesh * max(len(meshes), 1))()
    keep, space = [], HOST
    for r, m, b in zip(recs, meshes, objs):
        p, stride, nv, space, k = _verts_arg(m)
        keep.append(k)
        if indexed and b.vert_count:
            r.verts, r.stride, r.vert_count, r.indices, r.prim_count = p.value, stride, nv, None, b.triCount
        else:
            r.verts, r.stride, r.vert_count, r.indices, r.prim_count = p.value, stride, 0, None, nv // 3
    hs = (C.c_void_p * max(len(objs), 1))(*[b.h for b in objs])
    entry = _lib.lib().tbvh_refit_batch_indexed if indexed else _lib.lib().tbvh_refit_batch
    check(entry(hs, recs, len(meshes), space, int(keep_layouts)))
    return objs


def pinned_empty(n: int, dtype, device: int = None, node: int = None) -> np.ndarray:
    """numpy array in page-locked host memory on the NUMA node of `device` (default: the current CUDA device): full-speed DMA
    for the host path (tbvh_host_alloc / tbvh_host_alloc_near)."""
    dtype = np.dtype(dtype)
    p = C.c_void_p()
    if node is not None:
        check(_lib.lib().tbvh_host_alloc_node(node, n * dtype.itemsize, C.byref(p)))
    elif device is None:
        check(_lib.lib().tbvh_host_alloc(n * dtype.itemsize, C.byref(p)))
    else:
        check(_lib.lib().tbvh_host_alloc_near(device, n * dtype.itemsize, C.byref(p)))
    buf = (C.c_char * (n * dtype.itemsize)).from_address(p.value)
    a = np.frombuffer(buf, dtype=dtype, count=n)
    a.flags.writeable = True
    _pinned[a.ctypes.data] = p
    return a


_pinned = {}


def pinned_free(a: np.ndarray):
    p = _pinned.pop(a.ctypes.data, None)
    if p is not None:
        check(_lib.lib().tbvh_host_free(p))


def copy_rays_to_device(rays: np.ndarray, d_rays, stream=None) -> None:
    """tbvh_copy_rays_to_device: bytes 0..63 of every host record into a [n, 64]-byte torch CUDA tensor (synchronous here)."""
    import torch
    assert rays.dtype.itemsize in (64, 128) and rays.flags.c_contiguous and d_rays.is_cuda and d_rays.is_contiguous()
    assert d_rays.numel() * d_rays.element_size() >= rays.shape[0] * 64
    st = torch.cuda.current_stream(d_rays.device)
    check(_lib.lib().tbvh_copy_rays_to_device(_np_ptr(rays), rays.dtype.itemsize, rays.shape[0], C.c_void_p(d_rays.data_ptr()), C.c_void_p(st.cuda_stream)))
    st.synchronize()


def bind_to_device(device: int = 0) -> bool:
    """Restrict the calling thread (and threads it starts later: OpenMP, the host pipeline) to the CPUs of the NUMA node `device`
    hangs off.  False when the system exposes no topology."""
    return _lib.lib().tbvh_bind_thread_to_device(device) == _lib.OK


def shard_range(n: int, part: int, parts: int):
    """tbvh_shard_range: contiguous [first, first+count) of n rays for `part`, boundaries on multiples of 32."""
    a, c = C.c_uint64(), C.c_uint64()
    _lib.lib().tbvh_shard_range(n, part, parts, C.byref(a), C.byref(c))
    return a.value, c.value


class Group:
    """Several GPUs of one process (tbvh_group_*): `replicate(bvh)` copies a BVH, or a TLAS with its BLASes, to every device over
    NVLink, `Intersect` / `IsOccluded` shard a host ray batch by index over the devices.  `layout` follows the replicated object.
    An animated scene calls `replicate(tlas)` once per frame: the replicas are refreshed in place."""

    def __init__(self, devices=None):
        self.h = C.c_void_p()
        if devices is None:
            check(_lib.lib().tbvh_group_create(None, 0, C.byref(self.h)))
        else:
            arr = (C.c_int * len(devices))(*devices)
            check(_lib.lib().tbvh_group_create(arr, len(devices), C.byref(self.h)))
        self.layout = LAYOUT_BVH
        self.src = None

    def __len__(self):
        return _lib.lib().tbvh_group_size(self.h)

    def replicate(self, bvh) -> float:
        ms = C.c_double()
        check(_lib.lib().tbvh_group_replicate(self.h, bvh.h, C.byref(ms)))
        self.src, self.layout = bvh, bvh.layout
        return ms.value

    def device_view(self, i: int, layout: int = None) -> _lib.DeviceView:
        """tbvh_device_view of device i's replica, over that device's own arrays (default layout: the replicated object's).  Valid
        until the next replicate() or close()."""
        h = _lib.lib().tbvh_group_replica(self.h, i)
        if not h:
            raise TbvhError("Group.device_view: no replica %d (replicate first)" % i)
        v = _lib.DeviceView()
        check(_lib.lib().tbvh_device_view(C.c_void_p(h), self.layout if layout is None else layout, C.byref(v)))
        return v

    def empty_rays(self, n: int, dtype) -> np.ndarray:
        """page-locked array whose index ranges sit on the NUMA node of the device that will read them (tbvh_group_host_alloc)"""
        dtype = np.dtype(dtype)
        p = C.c_void_p()
        check(_lib.lib().tbvh_group_host_alloc(self.h, dtype.itemsize, n, C.byref(p)))
        buf = (C.c_char * (n * dtype.itemsize)).from_address(p.value)
        a = np.frombuffer(buf, dtype=dtype, count=n)
        a.flags.writeable = True
        return a

    def Intersect(self, rays: np.ndarray) -> np.ndarray:
        assert rays.dtype.itemsize in (64, 128) and rays.flags.c_contiguous
        check(_lib.lib().tbvh_group_intersect(self.h, self.layout, _np_ptr(rays), rays.dtype.itemsize, rays.shape[0]))
        return rays

    def IsOccluded(self, rays: np.ndarray, bits: np.ndarray = None) -> np.ndarray:
        assert rays.dtype.itemsize in (64, 128) and rays.flags.c_contiguous
        n = rays.shape[0]
        if bits is None:
            bits = np.zeros((n + 31) // 32, np.uint32)
        check(_lib.lib().tbvh_group_occluded(self.h, self.layout, _np_ptr(rays), rays.dtype.itemsize, n, _np_ptr(bits)))
        return bits

    def close(self):
        if self.h is not None and self.h.value:
            _lib.lib().tbvh_group_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
