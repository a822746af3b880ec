"""Handles, contexts and groups own their device arrays: every call that builds, uploads, converts, refits, optimises, builds a TLAS,
replicates or destroys a handle, and every refusal, gives back what it does not keep.  Each call is repeated often enough that one
array left behind per call would show in the device's free memory, which must come back to where it was after two warm-up calls
(the context's grow-and-keep buffers reach their size there).  No torch memory is allocated inside the loops."""
import ctypes as C

import numpy as np
import pytest

from tinybvh_b200 import _lib, api
from tests import test_handle_state_gpu as hs
from tests.test_oracle_pin import tlas_case

pytestmark = pytest.mark.gpu

L = _lib.lib
ROUNDS = 1500
# The runtime hands out small blocks from 2 MiB pages, and blocks of varying sizes freed and taken again can leave a page or two held.
# The smallest array a call here makes, 6 KB of primIdx, left behind ROUNDS times is 9 MB.
SLACK = 8 << 20


def free_bytes():
    import torch
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info()[0]


def lost(call, rounds=ROUNDS):
    """bytes of device memory `rounds` more calls of call() keep, after two warm-up calls"""
    call(), call()
    base = free_bytes()
    for _ in range(rounds):
        call()
    return base - free_bytes()


def ok(rc):
    assert rc == _lib.OK, L().tbvh_last_error()


@pytest.fixture(scope="module")
def case(gpu):
    return hs.Case()


@pytest.mark.parametrize("name", [n for n in hs.CASES if "device" not in n])
def test_transitions_and_refusals_keep_nothing(case, name):
    """every call and refusal of tests/test_handle_state_gpu.py with host inputs (device inputs would allocate torch memory)"""
    with_cw, call, code, _, _ = hs.CASES[name]
    b, t = case.start(with_cw)

    def once():
        assert call(case, b) == code, L().tbvh_last_error()
    assert lost(once) < SLACK


def meshes(c):
    recs = (_lib.Mesh * 2)()
    for r, m in zip(recs, (c.v2, c.other)):
        r.verts, r.stride, r.vert_count, r.indices, r.prim_count = m.ctypes.data, 16, 0, None, m.shape[0] // 3
    return recs


@pytest.mark.parametrize("flavour", [_lib.BUILD_REFERENCE, _lib.BUILD_AVX, _lib.BUILD_HQ, _lib.BUILD_PLOC])
def test_builds_keep_nothing(case, flavour):
    c, b, b2 = case, api.BVH(), api.BVH()
    n = c.v2.shape[0] // 3
    assert lost(lambda: ok(L().tbvh_build_flavour(b.h, hs.p(c.v2), 16, n, api.HOST, 1.0, 1.0, flavour))) < SLACK
    idx = np.arange(c.v2.shape[0], dtype=np.uint32)
    assert lost(lambda: ok(L().tbvh_build_indexed(b.h, hs.p(c.v2), 16, c.v2.shape[0], hs.p(idx), n, api.HOST, 1.0, 1.0, flavour))) < SLACK
    recs, hv = meshes(c), (C.c_void_p * 2)(b.h.value, b2.h.value)
    if flavour == _lib.BUILD_HQ:
        batch = lambda: ok(L().tbvh_build_batch_hq(hv, recs, 2, api.HOST, 1.0, 1.0))
    else:
        batch = lambda: ok(L().tbvh_build_batch(hv, recs, 2, api.HOST, 1.0, 1.0, flavour))
    assert lost(batch) < SLACK


def test_uploads_conversions_refits_and_optimize_keep_nothing(case):
    c, b, b2 = case, api.BVH(), api.BVH()
    for up in (hs.upload_bvh, hs.upload_bvh_gpu, hs.upload_cwbvh):
        assert lost(lambda: ok(up(c, b, False))) < SLACK
    n = c.v2.shape[0] // 3
    build = lambda h: ok(L().tbvh_build_flavour(h.h, hs.p(c.v2), 16, n, api.HOST, 1.0, 1.0, _lib.BUILD_REFERENCE))
    build(b)
    for layout in (hs.GPU, hs.CW):
        assert lost(lambda: ok(L().tbvh_convert(b.h, layout))) < SLACK
    moved = c.v2.copy()
    moved[:, :3] *= np.float32(1.001)
    assert lost(lambda: ok(L().tbvh_refit(b.h, hs.p(moved), 16, n, api.HOST))) < SLACK
    for h in (b, b2):
        build(h), ok(L().tbvh_convert(h.h, hs.GPU)), ok(L().tbvh_convert(h.h, hs.CW))
    assert lost(lambda: ok(L().tbvh_refit_layouts(b.h, hs.p(moved), 16, n, api.HOST))) < SLACK
    recs = (_lib.Mesh * 2)()
    for r in recs:
        r.verts, r.stride, r.vert_count, r.indices, r.prim_count = moved.ctypes.data, 16, 0, None, n
    hv = (C.c_void_p * 2)(b.h.value, b2.h.value)
    for keep in (1, 0):
        assert lost(lambda: ok(L().tbvh_refit_batch(hv, recs, 2, api.HOST, keep))) < SLACK
    rounds, sah = C.c_uint32(0), C.c_float(0)

    def optimize():
        build(b)
        ok(L().tbvh_optimize(b.h, 4, 1.0, 1.0, C.byref(rounds), C.byref(sah)))
    assert lost(optimize, ROUNDS // 3) < SLACK


def test_tlas_builds_replicas_and_destroy_keep_nothing(gpu):
    v, inst, O, D = tlas_case(141, 300)
    blas = [api.BVH().Build(x) for x in v]
    t = api.TLAS().Build(inst, blas)                 # inst now holds Update()d records
    hv = (C.c_void_p * 2)(*[b.h.value for b in blas])
    assert lost(lambda: ok(L().tbvh_build_tlas(t.h, inst.ctypes.data, 192, 300, hv, 2, 1.0, 1.0))) < SLACK
    frame = [0]

    def update():                                    # each instance count twice in a row: the second frame keeps the tables
        frame[0] += 1
        ok(L().tbvh_build_tlas_update(t.h, inst.ctypes.data, 192, 300 - ((frame[0] >> 1) & 1), api.HOST, hv, 2, 1.0, 1.0))
    assert lost(update) < SLACK
    g = C.c_void_p()
    ok(L().tbvh_group_create((C.c_int * 1)(0), 1, C.byref(g)))
    try:
        src = api.BVH().Build(v[0])
        ok(L().tbvh_convert(src.h, hs.CW))
        assert lost(lambda: ok(L().tbvh_group_replicate(g, src.h, None)), ROUNDS // 3) < SLACK
        frame[0] = 0

        def scene():                                 # the source TLAS rebuilt before each replication
            update()
            ok(L().tbvh_group_replicate(g, t.h, None))
        assert lost(scene, ROUNDS // 3) < SLACK
    finally:
        L().tbvh_group_destroy(g)
    assert lost(lambda: api.BVH().Build(v[1]), ROUNDS) < SLACK

