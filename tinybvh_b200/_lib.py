"""ctypes loader for libtinybvh_b200.so - the C-ABI of include/tinybvh_b200.h.

Fails loudly: if the shared library is missing or a call returns an error there is no CPU path to fall back to."""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "libtinybvh_b200.so")

OK, HOST, DEVICE = 0, 0, 1
E_CUDA, E_ARG, E_STATE, E_LIMIT, E_UNSUPPORTED = -1, -2, -3, -4, -5
LAYOUT_BVH, LAYOUT_BVH_GPU, LAYOUT_CWBVH = 1, 5, 10
BUILD_REFERENCE, BUILD_AVX, BUILD_HQ, BUILD_PLOC = 0, 1, 2, 3


class TbvhError(RuntimeError):
    pass


class Info(C.Structure):
    _fields_ = [("prim_count", C.c_uint32), ("idx_count", C.c_uint32), ("used_nodes", C.c_uint32),
                ("used_nodes_gpu", C.c_uint32), ("used_blocks", C.c_uint32), ("cwbvh_tri_count", C.c_uint32),
                ("max_depth", C.c_uint32), ("layouts", C.c_uint32),
                ("aabb_min", C.c_float * 3), ("aabb_max", C.c_float * 3), ("build_ms", C.c_double)]


class Mesh(C.Structure):
    """tbvh_mesh: one mesh of a tbvh_build_batch or tbvh_refit_batch call"""
    _fields_ = [("verts", C.c_void_p), ("stride", C.c_uint32), ("vert_count", C.c_uint32), ("indices", C.c_void_p), ("prim_count", C.c_uint32)]


class DeviceView(C.Structure):
    """tbvh_view: what tbvh_device_view hands a kernel that calls the device functions of include/tinybvh_b200_device.cuh (64 bytes,
    passed by value or as bytes(view))"""
    _fields_ = [("kind", C.c_int32), ("root_ref", C.c_uint32), ("root_count", C.c_uint32), ("stack", C.c_uint32),
                ("nodes", C.c_void_p), ("tris", C.c_void_p), ("prim_idx", C.c_void_p), ("inst", C.c_void_p), ("blas", C.c_void_p),
                ("cw_rd_limit", C.c_float), ("inst_shift", C.c_uint32)]


VIEW_BVH, VIEW_CWBVH, VIEW_TLAS_BVH, VIEW_TLAS_CWBVH = 1, 10, 101, 110


# every symbol include/tinybvh_b200.h declares: name -> (restype, argtypes)
vp, u32, u64, i32, f32, sz = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int, C.c_float, C.c_size_t
SYMBOLS = {
    "tbvh_ctx_create": (i32, [i32, C.POINTER(vp)]),
    "tbvh_ctx_destroy": (i32, [vp]),
    "tbvh_last_error": (C.c_char_p, []),
    "tbvh_device_count": (i32, []),
    "tbvh_set_option": (i32, [vp, C.c_char_p, i32]),
    "tbvh_host_alloc": (i32, [sz, C.POINTER(vp)]),
    "tbvh_host_free": (i32, [vp]),
    "tbvh_host_register": (i32, [vp, sz]),
    "tbvh_host_unregister": (i32, [vp]),
    "tbvh_bvh_create": (i32, [vp, C.POINTER(vp)]),
    "tbvh_bvh_destroy": (i32, [vp]),
    "tbvh_bvh_info": (i32, [vp, C.POINTER(Info)]),
    "tbvh_build": (i32, [vp, vp, u32, u32, i32, f32, f32]),
    "tbvh_build_flavour": (i32, [vp, vp, u32, u32, i32, f32, f32, i32]),
    "tbvh_sah_cost": (i32, [vp, f32, f32, vp]),
    "tbvh_sah_cost_nodes": (i32, [vp, u32, f32, f32, vp]),
    "tbvh_optimize": (i32, [vp, u32, f32, f32, vp, vp]),
    "tbvh_instance_update": (i32, [vp, vp]),
    "tbvh_instance_update_box": (i32, [vp, vp, vp]),
    "tbvh_build_tlas": (i32, [vp, vp, u32, u32, vp, u32, f32, f32]),
    "tbvh_build_tlas_update": (i32, [vp, vp, u32, u32, i32, vp, u32, f32, f32]),
    "tbvh_refit": (i32, [vp, vp, u32, u32, i32]),
    "tbvh_refit_layouts": (i32, [vp, vp, u32, u32, i32]),
    "tbvh_refit_batch": (i32, [vp, vp, u32, i32, i32]),
    "tbvh_refit_batch_indexed": (i32, [vp, vp, u32, i32, i32]),
    "tbvh_build_indexed": (i32, [vp, vp, u32, u32, vp, u32, i32, f32, f32, i32]),
    "tbvh_build_batch": (i32, [vp, vp, u32, i32, f32, f32, i32]),
    "tbvh_build_batch_hq": (i32, [vp, vp, u32, i32, f32, f32]),
    "tbvh_upload_bvh": (i32, [vp, vp, u32, vp, u32, vp, u32, u32, i32]),
    "tbvh_upload_bvh_gpu": (i32, [vp, vp, u32, vp, u32, vp, u32, u32, i32]),
    "tbvh_upload_cwbvh": (i32, [vp, vp, u32, vp, u32, i32]),
    "tbvh_convert": (i32, [vp, i32]),
    "tbvh_convert_batch": (i32, [vp, u32, i32]),
    "tbvh_download_bvh": (i32, [vp, vp, vp, i32]),
    "tbvh_download_bvh_gpu": (i32, [vp, vp, i32]),
    "tbvh_download_cwbvh": (i32, [vp, vp, vp, i32]),
    "tbvh_intersect": (i32, [vp, i32, vp, u32, u64]),
    "tbvh_intersect_packed": (i32, [vp, i32, vp, u32, u64, vp]),
    "tbvh_occluded": (i32, [vp, i32, vp, u32, u64, vp]),
    "tbvh_intersect_device": (i32, [vp, i32, vp, u32, vp, u64, vp]),
    "tbvh_occluded_device": (i32, [vp, i32, vp, u32, vp, u64, vp]),
    "tbvh_closest_point": (i32, [vp, vp, vp, u64, i32, vp]),
    "tbvh_sphere_overlap": (i32, [vp, vp, vp, u64, i32, vp]),
    "tbvh_signed_distance_prepare": (i32, [vp]),
    "tbvh_signed_distance": (i32, [vp, vp, vp, u64, i32, vp]),
    "tbvh_winding_number_prepare": (i32, [vp]),
    "tbvh_winding_number": (i32, [vp, vp, vp, u64, C.c_float, i32, vp]),
    "tbvh_mesh_overlap_pairs": (i32, [vp, vp, vp, u64, vp, i32, vp]),
    "tbvh_mesh_overlap_bits": (i32, [vp, vp, vp, i32, vp]),
    "tbvh_device_view": (i32, [vp, i32, C.POINTER(DeviceView)]),
    "tbvh_set_stats": (i32, [vp, i32]),
    "tbvh_get_stats": (i32, [vp, C.POINTER(u64), C.POINTER(u64)]),
    "tbvh_launch_count": (u64, []),
    "tbvh_get_stats_ex": (i32, [vp, C.POINTER(u64 * 4)]),
    "tbvh_copy_rays_to_device": (i32, [vp, u32, u64, vp, vp]),
    "tbvh_device_alloc": (i32, [vp, sz, C.POINTER(vp)]),
    "tbvh_device_free": (i32, [vp, vp]),
    "tbvh_device_sync": (i32, [vp]),
    "tbvh_copy_from_device": (i32, [vp, vp, sz]),
    "tbvh_device_numa_node": (i32, [i32]),
    "tbvh_bind_thread_to_device": (i32, [i32]),
    "tbvh_host_alloc_near": (i32, [i32, sz, C.POINTER(vp)]),
    "tbvh_host_alloc_node": (i32, [i32, sz, C.POINTER(vp)]),
    "tbvh_group_create": (i32, [vp, i32, C.POINTER(vp)]),
    "tbvh_group_destroy": (i32, [vp]),
    "tbvh_group_size": (i32, [vp]),
    "tbvh_group_ctx": (vp, [vp, i32]),
    "tbvh_group_replica": (vp, [vp, i32]),
    "tbvh_group_replicate": (i32, [vp, vp, C.POINTER(C.c_double)]),
    "tbvh_group_intersect": (i32, [vp, i32, vp, u32, u64]),
    "tbvh_group_occluded": (i32, [vp, i32, vp, u32, u64, vp]),
    "tbvh_group_host_alloc": (i32, [vp, u32, u64, C.POINTER(vp)]),
    "tbvh_group_host_free": (i32, [vp, vp]),
    "tbvh_shard_range": (None, [u64, u32, u32, C.POINTER(u64), C.POINTER(u64)]),
}

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.isfile(SO):
            raise TbvhError(f"{SO} not built (python -m tinybvh_b200.build); the engine has no CPU fallback")
        L = C.CDLL(SO)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = res, args
        _lib = L
    return _lib


def check(rc: int) -> None:
    if rc != OK:
        raise TbvhError(f"tinybvh_b200 error {rc}: {lib().tbvh_last_error().decode(errors='replace')}")
