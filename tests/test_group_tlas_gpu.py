"""An instanced scene on a device group (tbvh_group_replicate of a TLAS): every device gets a replica TLAS over replicas of its BLASes,
and a later replicate refreshes them in place.  Group walks are held byte for byte to the source TLAS's own calls and to the oracle:
hits including hit.inst (byte 44), and occlusion words.  On a one-GPU box the group is device 0 twice."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tinybvh_b200 import _lib, api, build, rays as R, scenes
from tests import util

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FN = {_lib.VIEW_BVH: 0, _lib.VIEW_CWBVH: 1, _lib.VIEW_TLAS_BVH: 2, _lib.VIEW_TLAS_CWBVH: 3}
BLAS_CLS = {api.LAYOUT_BVH: api.BVH, api.LAYOUT_CWBVH: api.BVH8_CWBVH}


def devices():
    n = api.device_count()
    return list(range(n)) if n > 1 else [0, 0]


def rec(r):
    return r.view(np.uint8).reshape(r.shape[0], -1)[:, :64]   # the 64 bytes a walk reads and writes


def error_code(fn):
    with pytest.raises(api.TbvhError) as e:
        fn()
    return int(str(e.value).split("error ")[1].split(":")[0])


def make_blas(layout, builder, v):
    if layout == api.LAYOUT_BVH or builder == "BuildHQ":
        return getattr(BLAS_CLS[layout](), builder)(v)
    b = api.BVH8_CWBVH()                     # BVH8_CWBVH::Build converts the tree of the flavour it is given
    b.build_flavour = _lib.BUILD_REFERENCE if builder == "Build" else _lib.BUILD_AVX
    return b.Build(v)


def scene(seed, n_inst, builder="Build", layout=api.LAYOUT_BVH, n_rays=19_993):
    """two BLASes, n_inst instances; every fifth instance carries mask 0x2 only.  n_rays is not a multiple of 32 x parts."""
    v = [scenes.procedural_scene(2000, seed), scenes.procedural_scene(500, seed + 1)]
    blas = [make_blas(layout, builder, x) for x in v]
    inst = np.zeros(n_inst, api.BLAS_INSTANCE)
    inst["transform"] = util.random_transforms(n_inst, seed)
    inst["blasIdx"] = np.arange(n_inst) % 2
    inst["mask"] = np.where(np.arange(n_inst) % 5 == 0, 0x2, 0x3)
    raw = inst.copy()
    t = api.TLAS().Build(inst, blas, blas_layout=layout)
    rng = np.random.default_rng(seed)
    D = rng.normal(size=(n_rays, 3)).astype(np.float32) * 0.35 + np.array([0, 0, 1], np.float32)
    O = np.tile(np.array([[0, 0, -120]], np.float32), (n_rays, 1))
    return v, blas, raw, t, O, D


def assert_group_equals(g, t, O, D, masks=(0x1, 0x2), layout=None):
    """group Intersect / IsOccluded == the source's own calls, for every ray mask; -> the closest-hit records of the last mask"""
    g.layout = t.layout if layout is None else layout
    for mask in masks:
        rays = R.make_rays(O, D)
        rays["mask"] = mask
        want, got = rays.copy(), rays.copy()
        _lib.check(_lib.lib().tbvh_intersect(t.h, g.layout, want.ctypes.data, want.dtype.itemsize, want.shape[0]))
        g.Intersect(got)
        assert np.array_equal(rec(got), rec(want)), f"closest hits differ (ray mask {mask:#x})"
        sh = R.make_rays(O, D, tmax=150.0)
        sh["mask"] = mask
        wb = np.zeros((sh.shape[0] + 31) // 32, np.uint32)
        _lib.check(_lib.lib().tbvh_occluded(t.h, g.layout, sh.ctypes.data, sh.dtype.itemsize, sh.shape[0], wb.ctypes.data))
        assert np.array_equal(g.IsOccluded(sh), wb), f"occlusion differs (ray mask {mask:#x})"
    return got


def blas_table(view, count):
    """the BlasRef records of a TLAS view: (trav, tris, cw_nodes, cw_tris) addresses per BLAS"""
    buf = np.zeros(count * 48, np.uint8)
    _lib.check(_lib.lib().tbvh_copy_from_device(buf.ctypes.data, C.c_void_p(view.blas), buf.nbytes))
    q = buf.view(np.uint64).reshape(count, 6)
    return [tuple(int(x) for x in row[[0, 1, 4, 5]]) for row in q]


@pytest.mark.parametrize("n_inst", [1, 24, 3000])
@pytest.mark.parametrize("layout", [api.LAYOUT_BVH, api.LAYOUT_CWBVH])
@pytest.mark.parametrize("builder", ["Build", "BuildAVX", "BuildHQ"])
def test_group_tlas_equals_source_and_oracle(gpu, builder, layout, n_inst):
    v, blas, raw, t, O, D = scene(91, n_inst, builder, layout)
    g = api.Group(devices())
    assert g.replicate(t) >= 0
    for i in range(len(g)):
        assert _lib.lib().tbvh_group_replica(g.h, i)
    got = assert_group_equals(g, t, O, D)
    hit = got["t"] < 1e30
    assert n_inst == 1 or hit.sum() > 1000
    if layout == api.LAYOUT_BVH:
        ref = util.oracle_tlas(raw.copy(), v, {"Build": 0, "BuildAVX": 1, "BuildHQ": 2}[builder])
        for mask in (0x1, 0x2):
            rays = R.make_rays(O, D)
            rays["mask"] = mask
            want, got = rays.copy(), rays.copy()
            ref.intersect(want), g.Intersect(got)
            assert np.array_equal(rec(got), rec(want)), f"group hits differ from the oracle (mask {mask:#x})"
            sh = R.make_rays(O, D, tmax=150.0)
            sh["mask"] = mask
            assert np.array_equal(g.IsOccluded(sh), ref.occluded(sh))
    elif n_inst == 24:
        from oracle import portpy
        nodes, idx = t.download()
        inst = raw.copy()
        api.TLAS().Build(inst, blas, blas_layout=layout)                     # the Update()d records
        port = portpy.PortTLASCW(nodes, idx, inst, [type("CW", (), {"nodes": d[0], "tris": d[1]}) for d in (b.download() for b in blas)])
        rays = R.make_rays(O, D)
        want, got = rays.copy(), rays.copy()
        port.intersect(want), g.Intersect(got)
        assert np.array_equal(rec(got), rec(want)), "group hits differ from the CWBVH oracle"
    g.close()


def test_inst_idx_bits(gpu):
    v, blas, raw, t, O, D = scene(95, 30)
    g = api.Group(devices())
    L = _lib.lib()
    ctxs = [L.tbvh_group_ctx(g.h, i) for i in range(len(g))]
    api.set_option("inst_idx_bits", 10)
    try:
        for c in ctxs:
            _lib.check(L.tbvh_set_option(C.c_void_p(c), b"inst_idx_bits", 10))
        g.replicate(t)
        before = assert_group_equals(g, t, O, D)
        assert (before["t"] < 1e30).sum() > 1000
        _lib.check(L.tbvh_set_option(C.c_void_p(ctxs[-1]), b"inst_idx_bits", 32))
        assert error_code(lambda: g.replicate(t)) == _lib.E_STATE
        _lib.check(L.tbvh_set_option(C.c_void_p(ctxs[-1]), b"inst_idx_bits", 10))
        again = R.make_rays(O, D)
        again["mask"] = 0x2
        g.Intersect(again)
        assert np.array_equal(rec(again), rec(before)), "a refused replicate touched the replicas"
    finally:
        api.set_option("inst_idx_bits", 32)
    g.close()


def test_uploaded_cwbvh_blasses(gpu):
    v, blas, raw, t, O, D = scene(97, 40, "Build", api.LAYOUT_CWBVH)
    up = [api.BVH8_CWBVH().upload(*b.download()) for b in blas]            # bvh8Data / bvh8Tris only: no BVH-layout tree
    inst = raw.copy()
    api.TLAS().Build(inst, blas, blas_layout=api.LAYOUT_CWBVH)             # Update()s the records against the built BLASes
    t2 = api.TLAS().Build(inst, up, update=False, blas_layout=api.LAYOUT_CWBVH)
    g = api.Group(devices())
    g.replicate(t2)
    got = assert_group_equals(g, t2, O, D)
    assert (got["t"] < 1e30).sum() > 1000
    g.close()


def test_deep_blas(gpu):
    """a BLAS 64..255 levels deep with its CWBVH: the BVH-layout walk is TBVH_E_LIMIT on the replica as on the source"""
    v = util.small_scene(3000, 5)
    src = util.source_tree(v, "Build")
    tr = util.reinserted(src, 3, 50, grow_to=100)
    deep = api.BVH().upload(tr[0], tr[1], v)
    assert 64 <= deep.info().max_depth < 256
    _lib.check(_lib.lib().tbvh_convert(deep.h, api.LAYOUT_CWBVH))
    other = api.BVH8_CWBVH().Build(scenes.procedural_scene(500, 6))
    inst = np.zeros(12, api.BLAS_INSTANCE)
    inst["transform"] = util.random_transforms(12, 7)
    inst["blasIdx"] = np.arange(12) % 2
    inst["mask"] = 0x3
    t = api.TLAS().Build(inst, [deep, other], blas_layout=api.LAYOUT_CWBVH)
    g = api.Group(devices())
    g.replicate(t)
    O = np.tile(np.array([[0, 0, -120]], np.float32), (5001, 1))
    D = np.random.default_rng(1).normal(size=(5001, 3)).astype(np.float32) * 0.35 + np.array([0, 0, 1], np.float32)
    rays = R.make_rays(O, D)
    r = rays.copy()
    assert _lib.lib().tbvh_intersect(t.h, api.LAYOUT_BVH, r.ctypes.data, r.dtype.itemsize, r.shape[0]) == _lib.E_LIMIT
    g.layout = api.LAYOUT_BVH
    assert error_code(lambda: g.Intersect(rays.copy())) == _lib.E_LIMIT
    for i in range(len(g)):
        v_ = _lib.DeviceView()
        rc = _lib.lib().tbvh_device_view(C.c_void_p(_lib.lib().tbvh_group_replica(g.h, i)), api.LAYOUT_BVH, C.byref(v_))
        assert rc == _lib.E_LIMIT
    assert_group_equals(g, t, O, D, masks=(0x1,), layout=api.LAYOUT_CWBVH)
    g.close()


def test_blas_listed_twice_stale_and_destroyed_sources(gpu):
    v, blas, raw, t, O, D = scene(99, 36)
    inst = raw.copy()
    inst["blasIdx"] = np.arange(36) % 3
    t3 = api.TLAS().Build(inst, [blas[0], blas[1], blas[0]])               # BLAS 0 listed twice: one replica
    g = api.Group(devices())
    g.replicate(t3)
    before = assert_group_equals(g, t3, O, D)
    # a stale source: refused, the replicas as they were
    blas[1].Build(v[1])
    assert error_code(lambda: g.replicate(t3)) == _lib.E_STATE
    again = R.make_rays(O, D)
    again["mask"] = 0x2
    g.Intersect(again)
    assert np.array_equal(rec(again), rec(before))
    # source TLAS and BLASes destroyed: the replicas still walk
    t4 = api.TLAS().Build(raw.copy(), blas)
    g.replicate(t4)
    want = assert_group_equals(g, t4, O, D)
    for h in [t4] + blas:
        _lib.lib().tbvh_bvh_destroy(h.h)
        h.h = None
    got = R.make_rays(O, D)
    got["mask"] = 0x2
    g.Intersect(got)
    assert np.array_equal(rec(got), rec(want))
    g.close()


def test_source_in_a_group_context(gpu):
    g = api.Group(devices())
    ctx = C.c_void_p(_lib.lib().tbvh_group_ctx(g.h, 0))

    def make(cls):
        o = cls.__new__(cls)
        o.device, o.ctx, o.h, o.c_trav, o.c_int, o.vert_count = 0, ctx, C.c_void_p(), 1.0, 1.0, 0
        _lib.check(_lib.lib().tbvh_bvh_create(ctx, C.byref(o.h)))
        return o
    v = [scenes.procedural_scene(2000, 31), scenes.procedural_scene(500, 32)]
    blas = [make(api.BVH8_CWBVH).Build(x) for x in v]
    inst = np.zeros(50, api.BLAS_INSTANCE)
    inst["transform"] = util.random_transforms(50, 31)
    inst["blasIdx"] = np.arange(50) % 2
    inst["mask"] = 0x3
    for layout in (api.LAYOUT_BVH, api.LAYOUT_CWBVH):
        t = make(api.TLAS).Build(inst.copy(), blas, blas_layout=layout)
        g.replicate(t)
        assert _lib.lib().tbvh_group_replica(g.h, 0) == t.h.value
        O = np.tile(np.array([[0, 0, -120]], np.float32), (7777, 1))
        D = np.random.default_rng(2).normal(size=(7777, 3)).astype(np.float32) * 0.35 + np.array([0, 0, 1], np.float32)
        assert (assert_group_equals(g, t, O, D)["t"] < 1e30).sum() > 500
        _lib.lib().tbvh_bvh_destroy(t.h)
        t.h = None
    for b in blas:                            # the handles go before the contexts they live in
        _lib.lib().tbvh_bvh_destroy(b.h)
        b.h = None
    g.close()


def frame_transforms(n, frame):
    return util.random_transforms(n, 1000 + frame)


@pytest.mark.parametrize("kind", ["rigid", "deforming"])
@pytest.mark.parametrize("layout", [api.LAYOUT_BVH, api.LAYOUT_CWBVH])
def test_frames_refresh_in_place(gpu, kind, layout):
    v, blas, raw, t, O, D = scene(101, 200, "Build", layout)
    inst = raw.copy()
    t.Rebuild(inst)
    g = api.Group(devices())
    g.replicate(t)
    copies = [i for i in range(len(g)) if _lib.lib().tbvh_group_replica(g.h, i) != t.h.value]
    addr = {i: blas_table(g.device_view(i), 2) for i in copies}
    rng = np.random.default_rng(5)
    for frame in range(3):
        if kind == "deforming":
            moved = [(x + rng.normal(0, 0.02, x.shape).astype(np.float32) * np.array([1, 1, 1, 0], np.float32)).astype(np.float32) for x in v]
            api.refit_batch(blas, moved, keep_layouts=1)
        inst["transform"] = frame_transforms(inst.shape[0], frame)
        t.Rebuild(inst)
        g.replicate(t)
        got = assert_group_equals(g, t, O, D)
        assert (got["t"] < 1e30).sum() > 500
        for i in copies:
            assert blas_table(g.device_view(i), 2) == addr[i], f"frame {frame}: replica {i} BLAS arrays moved"


def test_launches_per_refresh_do_not_grow_with_the_blas_count(gpu):
    per = {}
    for nb in (32, 1000):
        meshes = [scenes.procedural_scene(64 + (k % 7) * 16, 400 + k) for k in range(nb)]
        blas = api.build_batch([api.BVH8_CWBVH() for _ in range(nb)], meshes)
        inst = np.zeros(2 * nb, api.BLAS_INSTANCE)
        inst["transform"] = util.random_transforms(2 * nb, nb)
        inst["blasIdx"] = np.arange(2 * nb) % nb
        inst["mask"] = 0x3
        t = api.TLAS()
        t.Rebuild(inst, blas, api.LAYOUT_CWBVH)
        g = api.Group(devices())
        g.replicate(t)
        inst["transform"] = util.random_transforms(2 * nb, nb + 1)
        t.Rebuild(inst)
        n0 = api.launch_count()
        g.replicate(t)
        rigid = api.launch_count() - n0
        api.refit_batch(blas, meshes, keep_layouts=1)
        t.Rebuild(inst)
        n0 = api.launch_count()
        g.replicate(t)
        per[nb] = (rigid, api.launch_count() - n0)
        O = np.tile(np.array([[0, 0, -120]], np.float32), (3001, 1))
        D = np.random.default_rng(3).normal(size=(3001, 3)).astype(np.float32) * 0.35 + np.array([0, 0, 1], np.float32)
        assert_group_equals(g, t, O, D, masks=(0x3,))
        g.close()
    assert per[32] == per[1000], per
    assert per[32][0] <= len(devices())


@pytest.fixture(scope="module")
def consumer(gpu, tmp_path_factory):
    nvcc = build.nvcc_path()
    assert nvcc, "nvcc is needed to build the consumer kernels"
    so = str(tmp_path_factory.mktemp("group_tlas") / "consumer.so")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I" + os.path.join(REPO, "include"),
                        "-Xcompiler", "-fPIC", "-shared", os.path.join(REPO, "tests", "device_api_consumer.cu"), "-o", so],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    L = C.CDLL(so)
    V, vp, u32, i32 = _lib.DeviceView, C.c_void_p, C.c_uint32, C.c_int
    L.dc_trace.argtypes = [V, i32, vp, vp, V, i32, vp, vp, vp, u32, i32]
    return L


@pytest.mark.parametrize("layout", [api.LAYOUT_BVH, api.LAYOUT_CWBVH])
def test_device_views_of_replicas(consumer, layout):
    import torch
    v, blas, raw, t, O, D = scene(103, 60, "BuildHQ", layout, n_rays=9_001)
    g = api.Group(devices())
    g.replicate(t)
    rays = R.make_rays(O, D)
    rays["mask"] = np.where(np.arange(rays.shape[0]) % 3 == 0, 2, 0xffffffff).astype(np.uint32)
    for i, dev in enumerate(devices()):
        h = C.c_void_p(_lib.lib().tbvh_group_replica(g.h, i))
        with torch.cuda.device(dev):
            d = torch.from_numpy(np.ascontiguousarray(rec(rays))).cuda()
            n = d.shape[0]
            want, wbits = d.clone(), torch.zeros((n + 31) // 32, dtype=torch.int32, device=d.device)
            _lib.check(_lib.lib().tbvh_intersect_device(h, layout, C.c_void_p(want.data_ptr()), 64, None, n, None))
            _lib.check(_lib.lib().tbvh_occluded_device(h, layout, C.c_void_p(d.data_ptr()), 64, C.c_void_p(wbits.data_ptr()), n, None))
            view = g.device_view(i, layout)
            got, got1, gbits, gbits1 = d.clone(), d.clone(), torch.zeros_like(wbits), torch.zeros_like(wbits)
            assert consumer.dc_trace(view, FN[view.kind], C.c_void_p(got.data_ptr()), None, view, FN[view.kind], C.c_void_p(got1.data_ptr()), None, None, n, 0) == 0
            assert consumer.dc_trace(view, FN[view.kind], C.c_void_p(d.data_ptr()), C.c_void_p(gbits.data_ptr()), view, FN[view.kind],
                                     C.c_void_p(d.data_ptr()), C.c_void_p(gbits1.data_ptr()), None, n, 1) == 0
            torch.cuda.synchronize()
            assert torch.equal(got, want), f"replica {i}: device-side hits differ from the batch call"
            assert torch.equal(gbits, wbits), f"replica {i}: device-side occlusion differs from the batch call"
            assert (got.cpu().numpy().view(np.float32)[:, 12] < 1e30).sum() > 500
        # and the batch call on the replica is the source's
        src = d.clone()
        _lib.check(_lib.lib().tbvh_intersect_device(t.h, layout, C.c_void_p(src.data_ptr()), 64, None, n, None))
        torch.cuda.synchronize()
        assert np.array_equal(src.cpu().numpy(), want.cpu().numpy())
    g.close()


def test_mixing_plain_and_scene_replicas(gpu):
    v, blas, raw, t, O, D = scene(105, 40)
    plain = api.BVH().Build(v[0])
    g = api.Group(devices())
    g.replicate(t)
    assert_group_equals(g, t, O, D)
    g.replicate(plain)                        # a plain BVH after a TLAS: the scene replicas go
    g.layout = api.LAYOUT_BVH
    rays = R.make_rays(O + np.array([0, 0, 80], np.float32), D)
    want, got = rays.copy(), rays.copy()
    plain.Intersect(want), g.Intersect(got)
    assert np.array_equal(rec(got), rec(want))
    g.replicate(t)                            # and a TLAS after a plain BVH
    assert_group_equals(g, t, O, D)
    with pytest.raises(api.TbvhError):
        g.replicate(type("R", (), {"h": C.c_void_p(_lib.lib().tbvh_group_replica(g.h, len(g) - 1)), "layout": api.LAYOUT_BVH})())
    g.close()                                 # scene replicas live
