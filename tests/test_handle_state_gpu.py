"""What a handle holds after each call that builds, uploads, converts or refits it, as include/tinybvh_b200.h documents it: the layout
bits and the counts of the derived layouts, which downloads succeed (the others are TBVH_E_STATE), whether a TLAS built over it still
walks in each BLAS layout or is stale, and whether tbvh_refit_layouts accepts it.  Every case starts from a BLAS that holds BVH, BVH_GPU
and CWBVH (or BVH and BVH_GPU only), under a TLAS that also covers a second BLAS."""
import ctypes as C

import numpy as np
import pytest

from tinybvh_b200 import _lib, api, rays as R, scenes
from tests.test_oracle_pin import tlas_case

pytestmark = pytest.mark.gpu

L = _lib.lib
BVH, GPU, CW = api.LAYOUT_BVH, api.LAYOUT_BVH_GPU, api.LAYOUT_CWBVH
OK, STATE = _lib.OK, _lib.E_STATE


def p(a):
    return C.c_void_p(a.ctypes.data if isinstance(a, np.ndarray) else a.data_ptr())


def on_device(a):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).cuda()
    torch.cuda.synchronize()
    return t


def state(b, v):
    """-> (layout names, which of used_nodes_gpu / used_blocks / cwbvh_tri_count are set, download codes, refit_layouts accepts)"""
    i = b.info()
    names = tuple(n for n, l in (("BVH", BVH), ("BVH_GPU", GPU), ("CWBVH", CW)) if i.layouts & (1 << l))
    counts = (i.used_nodes_gpu > 0, i.used_blocks > 0, i.cwbvh_tri_count > 0)
    n32 = np.zeros(max(i.used_nodes, 1) * 8, np.uint32)
    idx = np.zeros(max(i.idx_count, 1), np.uint32)
    n64 = np.zeros(max(i.used_nodes_gpu, 1) * 16, np.uint32)
    d8 = np.zeros(max(i.used_blocks, 1) * 4, np.uint32)
    t8 = np.zeros(max(i.cwbvh_tri_count, 1) * 12, np.uint32)
    downloads = (L().tbvh_download_bvh(b.h, p(n32), p(idx), api.HOST), L().tbvh_download_bvh_gpu(b.h, p(n64), api.HOST),
                 L().tbvh_download_cwbvh(b.h, p(d8), p(t8), api.HOST))
    # a slice of the wrong length passes every state refusal and stops at the argument check: TBVH_E_ARG means the state was accepted
    rc = L().tbvh_refit_layouts(b.h, p(v), 16, i.prim_count + 1, api.HOST)
    assert rc in (_lib.E_ARG, STATE)
    return names, counts, downloads, rc == _lib.E_ARG


FULL = (("BVH", "BVH_GPU", "CWBVH"), (True, True, True), (OK, OK, OK), True)
NO_CW = (("BVH", "BVH_GPU"), (True, False, False), (OK, OK, STATE), True)
TREE = (("BVH",), (False, False, False), (OK, STATE, STATE), True)
SBVH = TREE[:3] + (False,)
UPLOADED_GPU = (("BVH_GPU",), (True, False, False), (STATE, OK, STATE), False)
UPLOADED_CW = FULL[:3] + (False,)   # a CWBVH tbvh_convert did not produce from the resident tree


class Case:
    def __init__(self):
        v, inst, O, D = tlas_case(131, 8)
        self.v, self.other = v
        self.v2 = scenes.procedural_scene(1500, 133)
        self.moved = self.v.copy()
        self.moved[:, :3] += np.float32(0.125) * np.sin(np.arange(self.v.shape[0], dtype=np.float32))[:, None]
        self.inst, self.rays = inst, R.make_rays(O[:96], D[:96], tmax=150.0)
        src = api.BVH().Build(self.v2)
        self.nodes32, self.idx = src.download()
        api.check(L().tbvh_convert(src.h, GPU))
        self.nodes64 = api.BVH_GPU.download(src)
        api.check(L().tbvh_convert(src.h, CW))
        self.d8, self.t8 = api.BVH8_CWBVH.download(src)

    def start(self, with_cw):
        """A BLAS over v holding BVH, BVH_GPU and (with_cw) CWBVH, and a TLAS over it and a second BLAS that hold the same layouts."""
        blas = [api.BVH().Build(x) for x in (self.v, self.other)]
        for b in blas:
            api.check(L().tbvh_convert(b.h, GPU))
            if with_cw:
                api.check(L().tbvh_convert(b.h, CW))
        t = api.TLAS().Build(self.inst.copy(), blas)
        assert self.walks(t) == ((OK, OK) if with_cw else (OK, STATE))
        return blas[0], t

    def walks(self, t):
        bits = np.zeros((self.rays.shape[0] + 31) // 32, np.uint32)
        return tuple(L().tbvh_occluded(t.h, layout, p(self.rays), 128, self.rays.shape[0], p(bits)) for layout in (BVH, CW))


def upload_bvh(c, b, dev):
    a = [c.nodes32, c.idx, c.v2]
    a = [on_device(x) for x in a] if dev else a
    return L().tbvh_upload_bvh(b.h, p(a[0]), c.nodes32.shape[0], p(a[1]), c.idx.shape[0], p(a[2]), 16, c.v2.shape[0] // 3, int(dev))


def upload_bvh_gpu(c, b, dev):
    a = [c.nodes64, c.idx, c.v2]
    a = [on_device(x) for x in a] if dev else a
    return L().tbvh_upload_bvh_gpu(b.h, p(a[0]), c.nodes64.shape[0], p(a[1]), c.idx.shape[0], p(a[2]), 16, c.v2.shape[0] // 3, int(dev))


def upload_cwbvh(c, b, dev, used_blocks=None):
    a = [c.d8, c.t8]
    a = [on_device(x) for x in a] if dev else a
    return L().tbvh_upload_cwbvh(b.h, p(a[0]), used_blocks or c.d8.shape[0], p(a[1]), c.t8.shape[0] // 3, int(dev))


def build(c, b, flavour, stride=16):
    return L().tbvh_build_flavour(b.h, p(c.v2), stride, c.v2.shape[0] // 3, api.HOST, 1.0, 1.0, flavour)


def build_indexed(c, b, bad=False, dev=False):
    """bad: one index points past vert_count; dev: vertices and indices in device memory"""
    idx = np.arange(c.v2.shape[0], dtype=np.uint32)
    if bad:
        idx[7] = c.v2.shape[0]
    a = [c.v2, idx]
    a = [on_device(x) for x in a] if dev else a
    return L().tbvh_build_indexed(b.h, p(a[0]), 16, c.v2.shape[0], p(a[1]), c.v2.shape[0] // 3, int(dev), 1.0, 1.0, _lib.BUILD_REFERENCE)


def build_batch(c, b, handles=None):
    meshes = [c.v2, c.other]
    recs = (_lib.Mesh * 2)()
    for r, m in zip(recs, meshes):
        r.verts, r.stride, r.vert_count, r.indices, r.prim_count = m.ctypes.data, 16, 0, None, m.shape[0] // 3
    c.keep = api.BVH()
    hs = handles or [b.h.value, c.keep.h.value]
    return L().tbvh_build_batch((C.c_void_p * 2)(*hs), recs, 2, api.HOST, 1.0, 1.0, _lib.BUILD_REFERENCE)


def convert_batch(c, b, layout=CW):
    c.keep = api.BVH().Build(c.other)
    return L().tbvh_convert_batch((C.c_void_p * 2)(b.h.value, c.keep.h.value), 2, layout)


def refit(c, b, fn, prim_count=None, space=api.HOST):
    return fn(b.h, p(c.moved), 16, prim_count or c.moved.shape[0] // 3, space)


STALE = (STATE, STATE)
# (start holds a CWBVH, what happens, the call, its return code, the handle's state after it, the TLAS walks in BVH / CWBVH layout)
CASES = {
    "Build": (True, lambda c, b: build(c, b, _lib.BUILD_REFERENCE), OK, TREE, STALE),
    "BuildAVX": (True, lambda c, b: build(c, b, _lib.BUILD_AVX), OK, TREE, STALE),
    "BuildHQ": (True, lambda c, b: build(c, b, _lib.BUILD_HQ), OK, SBVH, STALE),
    "indexed build": (True, build_indexed, OK, TREE, STALE),
    "build_batch": (True, build_batch, OK, TREE, STALE),
    "upload_bvh host": (True, lambda c, b: upload_bvh(c, b, False), OK, TREE, STALE),
    "upload_bvh device": (True, lambda c, b: upload_bvh(c, b, True), OK, TREE, STALE),
    "upload_bvh_gpu host": (True, lambda c, b: upload_bvh_gpu(c, b, False), OK, UPLOADED_GPU, STALE),
    "upload_bvh_gpu device": (True, lambda c, b: upload_bvh_gpu(c, b, True), OK, UPLOADED_GPU, STALE),
    "upload_cwbvh host": (True, lambda c, b: upload_cwbvh(c, b, False), OK, UPLOADED_CW, STALE),
    "upload_cwbvh device": (True, lambda c, b: upload_cwbvh(c, b, True), OK, UPLOADED_CW, STALE),
    "upload_cwbvh onto no CWBVH": (False, lambda c, b: upload_cwbvh(c, b, False), OK, UPLOADED_CW, (OK, STATE)),
    # no TLAS points at d_nodes_gpu: converting to BVH_GPU leaves a TLAS over the BLAS valid
    "convert BVH_GPU": (True, lambda c, b: L().tbvh_convert(b.h, GPU), OK, FULL, (OK, OK)),
    "convert CWBVH": (True, lambda c, b: L().tbvh_convert(b.h, CW), OK, FULL, STALE),
    "convert CWBVH onto no CWBVH": (False, lambda c, b: L().tbvh_convert(b.h, CW), OK, FULL, (OK, STATE)),
    "convert_batch": (True, convert_batch, OK, FULL, STALE),
    "refit": (True, lambda c, b: refit(c, b, L().tbvh_refit), OK, TREE, STALE),
    # a refit of a BLAS without a CWBVH keeps its arrays: the TLAS is not reported stale
    "refit without CWBVH": (False, lambda c, b: refit(c, b, L().tbvh_refit), OK, TREE, (OK, STATE)),
    "refit_layouts": (True, lambda c, b: refit(c, b, L().tbvh_refit_layouts), OK, FULL, STALE),
    "refit_layouts without CWBVH": (False, lambda c, b: refit(c, b, L().tbvh_refit_layouts), OK, NO_CW, STALE),
    # refusals leave the handle and the TLAS over it as they were
    "refused build": (True, lambda c, b: build(c, b, 7), _lib.E_ARG, FULL, (OK, OK)),
    "refused build stride": (True, lambda c, b: build(c, b, _lib.BUILD_REFERENCE, stride=14), _lib.E_ARG, FULL, (OK, OK)),
    "refused indexed build host": (True, lambda c, b: build_indexed(c, b, bad=True), _lib.E_ARG, FULL, (OK, OK)),
    "refused indexed build device": (True, lambda c, b: build_indexed(c, b, bad=True, dev=True), _lib.E_ARG, FULL, (OK, OK)),
    "refused build_batch": (True, lambda c, b: build_batch(c, b, [b.h.value, b.h.value]), _lib.E_ARG, FULL, (OK, OK)),
    "refused upload_bvh": (True, lambda c, b: L().tbvh_upload_bvh(b.h, p(c.nodes32), 0, p(c.idx), c.idx.shape[0], p(c.v2), 16, c.v2.shape[0] // 3, api.HOST),
                           _lib.E_ARG, FULL, (OK, OK)),
    "refused upload_bvh_gpu": (True, lambda c, b: L().tbvh_upload_bvh_gpu(b.h, None, 1, p(c.idx), c.idx.shape[0], p(c.v2), 16, c.v2.shape[0] // 3, api.HOST),
                               _lib.E_ARG, FULL, (OK, OK)),
    "refused upload_cwbvh": (True, lambda c, b: upload_cwbvh(c, b, False, used_blocks=c.d8.shape[0] + 1), _lib.E_ARG, FULL, (OK, OK)),
    "refused convert": (True, lambda c, b: L().tbvh_convert(b.h, 7), _lib.E_UNSUPPORTED, FULL, (OK, OK)),
    "refused convert_batch": (True, lambda c, b: convert_batch(c, b, GPU), _lib.E_UNSUPPORTED, FULL, (OK, OK)),
    "refused refit": (True, lambda c, b: refit(c, b, L().tbvh_refit, c.moved.shape[0] // 3 - 1), _lib.E_ARG, FULL, (OK, OK)),
    "refused refit_layouts": (True, lambda c, b: refit(c, b, L().tbvh_refit_layouts, c.moved.shape[0] // 3 - 1), _lib.E_ARG, FULL, (OK, OK)),
    "refused refit space": (True, lambda c, b: refit(c, b, L().tbvh_refit, space=5), _lib.E_ARG, FULL, (OK, OK)),
}


@pytest.fixture(scope="module")
def case(gpu):
    return Case()


def test_start(case):
    b, _ = case.start(True)
    assert state(b, case.v) == FULL
    b, _ = case.start(False)
    assert state(b, case.v) == NO_CW


@pytest.mark.parametrize("name", list(CASES))
def test_transition(case, name):
    with_cw, call, code, want, walks = CASES[name]
    b, t = case.start(with_cw)
    assert call(case, b) == code, L().tbvh_last_error()
    assert state(b, case.v) == want
    assert case.walks(t) == walks
