"""Traversal from a caller's own kernels (include/tinybvh_b200_device.cuh): tests/device_api_consumer.cu is compiled here with nvcc
-I include alone and driven through ctypes.  Every result is held byte for byte to the batch calls on the same records
(tbvh_intersect_device / tbvh_occluded_device), and through them to the oracle."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tinybvh_b200 import _lib, api, build, rays as R, scenes
from tests import util

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FN = {_lib.VIEW_BVH: 0, _lib.VIEW_CWBVH: 1, _lib.VIEW_TLAS_BVH: 2, _lib.VIEW_TLAS_CWBVH: 3}

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="session")
def consumer(gpu, tmp_path_factory):
    nvcc = build.nvcc_path()
    assert nvcc, "nvcc is needed to build the consumer kernels"
    so = str(tmp_path_factory.mktemp("device_api") / "consumer.so")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I" + os.path.join(REPO, "include"),
                        "-Xcompiler", "-fPIC", "-shared", "-Xptxas", "-v", os.path.join(REPO, "tests", "device_api_consumer.cu"), "-o", so],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    print(r.stderr)   # registers, stack frame and spills of the consumer kernels
    L = C.CDLL(so)
    V, vp, u32, i32, f32 = _lib.DeviceView, C.c_void_p, C.c_uint32, C.c_int, C.c_float
    L.dc_trace.argtypes = [V, i32, vp, vp, V, i32, vp, vp, vp, u32, i32]
    L.dc_camera_shadow.argtypes = [V, i32, i32, vp, vp, vp, u32, f32, f32, f32, f32]
    api.context(0)
    return L


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def to_device(r):
    import torch
    return torch.from_numpy(np.ascontiguousarray(r.view(np.uint8).reshape(-1, 128)[:, :64])).cuda()


def batch(obj, layout, recs):
    """tbvh_intersect_device (in place) and tbvh_occluded_device on copies of the records -> (records, bits) on the host"""
    import torch
    n = recs.shape[0]
    a = recs.clone()
    bits = torch.zeros((n + 31) // 32, dtype=torch.int32, device="cuda")
    L = _lib.lib()
    _lib.check(L.tbvh_intersect_device(obj.h, layout, _p(a), 64, None, n, None))
    _lib.check(L.tbvh_occluded_device(obj.h, layout, _p(recs), 64, _p(bits), n, None))
    torch.cuda.synchronize()
    return a.cpu().numpy(), bits.cpu().numpy()


def device(L, view, recs, sel=None, view1=None, recs1=None):
    """the consumer's k_trace, closest hit then any-hit, on copies -> (records, bits[, records1, bits1])"""
    import torch
    n = recs.shape[0]
    view1 = view if view1 is None else view1
    a, a1 = recs.clone(), (recs if recs1 is None else recs1).clone()
    b, b1 = (torch.zeros((n + 31) // 32, dtype=torch.int32, device="cuda") for _ in range(2))
    s = torch.from_numpy(sel.astype(np.uint32)).cuda() if sel is not None else None
    assert L.dc_trace(view, FN[view.kind], _p(a), None, view1, FN[view1.kind], _p(a1), None, _p(s), n, 0) == 0
    h, h1 = recs.clone(), (recs if recs1 is None else recs1).clone()
    assert L.dc_trace(view, FN[view.kind], _p(h), _p(b), view1, FN[view1.kind], _p(h1), _p(b1), _p(s), n, 1) == 0
    assert torch.equal(h, recs) and (recs1 is None or torch.equal(h1, recs1)), "any-hit wrote a record"
    return a.cpu().numpy(), b.cpu().numpy(), a1.cpu().numpy(), b1.cpu().numpy()


def assert_same(obj, layout, L, recs, label):
    want, wbits = batch(obj, layout, recs)
    got, gbits, _, _ = device(L, obj.device_view(layout), recs)
    assert np.array_equal(got, want), f"{label}: {int((got != want).any(axis=1).sum())} of {got.shape[0]} records differ from the batch call"
    assert np.array_equal(gbits, wbits), f"{label}: occlusion bits differ from the batch call"
    return got


def host_hits(dev, like):
    out = like.copy()
    out.view(np.uint8).reshape(-1, 128)[:, :64] = dev
    return out


def ray_families(v):
    sets, bounds = util.ray_sets(v, res=48)
    lo, hi = bounds
    prim = sets["primary"]
    o = util.oracle_bvh(v)
    traced = prim.copy()
    o.intersect(traced)
    fams = {"primary": prim, "shadow": util.derived_sets(traced, v, bounds)["shadow"], "shadow_at_hits": util.shadow_at_hits(traced)}
    fams["axis"] = util.axis_rays(lo, hi)
    fams["octants"] = util.octant_blocks(util.octant_rays(lo, hi))
    fams["inf_rd"] = util.with_inf_rd(fams["axis"])
    fams["rd_limit"] = util.rd_limit_rays(prim, 2.0 ** 100)
    far = prim[:500].copy()
    far["O"] += np.float32(1e30)
    fams["far_origin"] = far
    return fams


@pytest.fixture(scope="module")
def scene():
    v = util.small_scene(6000, 11)
    return v, ray_families(v)


@pytest.mark.parametrize("builder", ["Build", "BuildAVX", "BuildHQ"])
def test_bvh_matches_batch_and_oracle(consumer, scene, builder):
    v, fams = scene
    b = getattr(api.BVH(), builder)(v)
    for name, r in fams.items():
        got = assert_same(b, api.LAYOUT_BVH, consumer, to_device(r), f"{builder} {name}")
        if name == "primary":
            want = r.copy()
            util.oracle_tree(v, {"Build": 0, "BuildAVX": 1, "BuildHQ": 2}[builder]).intersect(want)
            assert util.compare_hits(host_hits(got, r), want) == {"prim": 0, "t": 0, "u": 0, "v": 0}


def test_bvh_gpu_and_cwbvh_match_batch(consumer, scene):
    v, fams = scene
    g = api.BVH_GPU().Build(v)
    cw = api.BVH8_CWBVH().BuildHQ(v)
    cw2 = api.BVH8_CWBVH().Build(v)
    for name, r in fams.items():
        d = to_device(r)
        assert_same(g, api.LAYOUT_BVH_GPU, consumer, d, f"BVH_GPU {name}")
        assert_same(cw, api.LAYOUT_CWBVH, consumer, d, f"CWBVH/HQ {name}")
        assert_same(cw2, api.LAYOUT_CWBVH, consumer, d, f"CWBVH {name}")


def test_uploaded_families_and_deep_tree(consumer):
    v = util.small_scene(3000, 5)
    sets, _ = util.ray_sets(v, res=32)
    d = to_device(sets["primary"])
    src = util.source_tree(v, "Build")
    for fam in ("A0.3", "B", "C3", "DA", "DC"):
        t = util.family_tree(src, fam, 17)
        assert_same(api.BVH().upload(t[0], t[1], v), api.LAYOUT_BVH, consumer, d, f"uploaded family {fam}")
    t = util.reinserted(src, 3, 50, grow_to=100)
    b = api.BVH().upload(t[0], t[1], v)
    assert 64 <= b.info().max_depth < 256
    assert b.device_view(api.LAYOUT_BVH).stack == 256
    assert_same(b, api.LAYOUT_BVH, consumer, d, "deep BVH2")


def tlas_scene(blas_layout):
    vs = [util.small_scene(800 + 300 * k, 20 + k) for k in range(3)]
    cls = api.BVH8_CWBVH if blas_layout == api.LAYOUT_CWBVH else api.BVH
    blas = [cls().Build(x) for x in vs]
    n = 40
    inst = np.zeros(n, api.BLAS_INSTANCE)
    inst["transform"] = util.random_transforms(n, 4)
    inst["blasIdx"] = np.arange(n) % 3
    inst["mask"] = np.where(np.arange(n) % 5 == 0, 2, 1 | 4)
    t = api.TLAS().Build(inst, blas, blas_layout=blas_layout)
    lo, hi = inst["aabbMin"].min(0), inst["aabbMax"].max(0)
    eye, view = R.bounds_camera(lo, hi, "outside")
    r = R.primary_rays(eye, view, 48, 48, 4)
    r["mask"] = np.where(np.arange(r.shape[0]) % 3 == 0, 2, 0xffffffff).astype(np.uint32)
    return t, blas, inst, r


@pytest.mark.parametrize("bits", [32, 10])
@pytest.mark.parametrize("layout", [api.LAYOUT_BVH, api.LAYOUT_CWBVH])
def test_tlas_matches_batch_and_oracle(consumer, layout, bits):
    api.set_option("inst_idx_bits", bits)
    try:
        t, blas, inst, r = tlas_scene(layout)
        got = assert_same(t, layout, consumer, to_device(r), f"TLAS layout {layout} bits {bits}")
        if layout == api.LAYOUT_BVH and bits == 32:
            vs = [util.small_scene(800 + 300 * k, 20 + k) for k in range(3)]
            want = r.copy()
            util.oracle_tlas(inst.copy(), vs, 0).intersect(want)
            assert util.compare_hits(host_hits(got, r), want) == {"prim": 0, "t": 0, "u": 0, "v": 0}
            assert np.array_equal(host_hits(got, r)["pad"], want["pad"])
    finally:
        api.set_option("inst_idx_bits", 32)


def test_divergent_callers(consumer, scene):
    """seeded subsets of lanes, whole idle warps, per-lane loop trip counts, two layouts in one warp, n not a multiple of 32"""
    v, fams = scene
    b = api.BVH().Build(v)
    cw = api.BVH8_CWBVH().BuildHQ(v)
    r = np.concatenate([fams["primary"], fams["octants"], fams["axis"]])[:5000 - 7]
    d = to_device(r)
    n = d.shape[0]
    want_b, bits_b = batch(b, api.LAYOUT_BVH, d)
    want_c, bits_c = batch(cw, api.LAYOUT_CWBVH, d)
    unpack = lambda w: np.unpackbits(w.view(np.uint8), bitorder="little")[:n].astype(bool)
    base = d.cpu().numpy()
    rng = np.random.default_rng(17)
    for trial in range(4):
        trips = rng.integers(0, 4, n).astype(np.uint32)
        trips[rng.random(n) < 0.3] = 0
        idle = rng.integers(0, (n + 31) // 32, 10)
        for w in idle:
            trips[w * 32:(w + 1) * 32] = 0
        second = (rng.random(n) < 0.5).astype(np.uint32) if trial % 2 else np.zeros(n, np.uint32)
        sel = trips | (second << 4)
        got0, g0, got1, g1 = device(consumer, b.device_view(api.LAYOUT_BVH), d, sel, cw.device_view(api.LAYOUT_CWBVH), d)
        on0, on1 = (trips > 0) & (second == 0), (trips > 0) & (second == 1)
        assert np.array_equal(got0[on0], want_b[on0]) and np.array_equal(got1[on1], want_c[on1])
        assert np.array_equal(got0[~on0], base[~on0]) and np.array_equal(got1[~on1], base[~on1]), "a record no lane traced changed"
        assert np.array_equal(unpack(g0), unpack(bits_b) & on0) and np.array_equal(unpack(g1), unpack(bits_c) & on1)


@pytest.mark.parametrize("kind", ["cwbvh", "tlas"])
def test_rays_made_on_the_device(consumer, scene, kind):
    import torch
    if kind == "cwbvh":
        v, fams = scene
        obj, layout = api.BVH8_CWBVH().BuildHQ(v), api.LAYOUT_CWBVH
        cam = fams["primary"]
        lo, hi = scenes.scene_bounds(v)
    else:
        obj, _, inst, cam = tlas_scene(api.LAYOUT_CWBVH)
        layout = api.LAYOUT_CWBVH
        lo, hi = inst["aabbMin"].min(0), inst["aabbMax"].max(0)
    light = (lo + hi) * 0.5 + np.array([0, (hi - lo)[1] * 0.45, 0], np.float32)
    eps = float((hi - lo).max() * 5e-7)
    d = to_device(cam)
    n = d.shape[0]
    shadow = torch.zeros_like(d)
    bits = torch.zeros((n + 31) // 32, dtype=torch.int32, device="cuda")
    view = obj.device_view(layout)
    assert consumer.dc_camera_shadow(view, FN[view.kind], FN[view.kind], _p(d), _p(shadow), _p(bits), n, *map(float, light), eps) == 0
    torch.cuda.synchronize()
    want = torch.zeros_like(bits)
    _lib.check(_lib.lib().tbvh_occluded_device(obj.h, layout, _p(shadow), 64, _p(want), n, None))
    torch.cuda.synchronize()
    assert torch.equal(bits, want)
    assert int(torch.count_nonzero(want)) > 0


def test_views_over_the_frame_cycle(consumer):
    """refit, TLAS update and rebuild: a freshly taken view gives the new results"""
    v = util.small_scene(3000, 8)
    sets, _ = util.ray_sets(v, res=32)
    d = to_device(sets["primary"])
    b = api.BVH8_CWBVH().Build(v)
    rng = np.random.default_rng(3)
    v2 = (v + rng.normal(0, 0.01, v.shape).astype(np.float32) * np.array([1, 1, 1, 0], np.float32)).astype(np.float32)
    meshes = (_lib.Mesh * 1)(_lib.Mesh(v2.ctypes.data, 16, 0, None, v2.shape[0] // 3))
    hs = (C.c_void_p * 1)(b.h)
    _lib.check(_lib.lib().tbvh_refit_batch(hs, meshes, 1, api.HOST, 1))
    assert_same(b, api.LAYOUT_CWBVH, consumer, d, "after refit_batch")
    b.Build(v2)
    assert_same(b, api.LAYOUT_CWBVH, consumer, d, "after rebuild")
    t, blas, inst, r = tlas_scene(api.LAYOUT_CWBVH)
    inst["transform"] = util.random_transforms(inst.shape[0], 99)
    t.Rebuild(inst)
    assert_same(t, api.LAYOUT_CWBVH, consumer, to_device(r), "after tbvh_build_tlas_update")


def test_refusals_match_the_batch_calls():
    import torch
    L = _lib.lib()
    api.context(0)
    d = torch.zeros((32, 64), dtype=torch.uint8, device="cuda")
    bits = torch.zeros(1, dtype=torch.int32, device="cuda")

    def codes(obj, layout):
        n0 = api.launch_count()
        v = _lib.DeviceView()
        rc = L.tbvh_device_view(obj.h, layout, C.byref(v))
        assert api.launch_count() == n0, "taking a view launched a kernel"
        assert rc != 0 or v.kind != 0
        if rc != 0:
            assert v.kind == 0
        a = L.tbvh_intersect_device(obj.h, layout, _p(d), 64, None, 32, None)
        o = L.tbvh_occluded_device(obj.h, layout, _p(d), 64, _p(bits), 32, None)
        torch.cuda.synchronize()
        return rc, a, o

    v = util.small_scene(2000, 3)
    b = api.BVH().Build(v)
    rc, a, o = codes(b, api.LAYOUT_CWBVH)            # layout not resident
    assert rc == a == o == _lib.E_STATE
    rc, a, o = codes(b, 77)                          # unknown layout
    assert rc == a == o == _lib.E_ARG
    assert codes(b, api.LAYOUT_BVH) == (0, 0, 0)
    t = util.reinserted(util.source_tree(v, "Build"), 3, 50, max_depth=400, grow_to=300)
    db = api.BVH().upload(t[0], t[1], v)
    assert db.info().max_depth >= 256
    rc, a, o = codes(db, api.LAYOUT_BVH)             # deeper than the 256-entry stack
    assert rc == a == o == _lib.E_LIMIT
    t, blas, inst, r = tlas_scene(api.LAYOUT_BVH)
    rc, a, o = codes(t, api.LAYOUT_CWBVH)            # BLASses hold no CWBVH
    assert rc == a == o == _lib.E_STATE
    blas[0].Build(util.small_scene(900, 1))          # the TLAS is stale
    rc, a, o = codes(t, api.LAYOUT_BVH)
    assert rc == a == o == _lib.E_STATE
    from tests.test_offatrium_gpu import pending_chain
    cw = api.BVH8_CWBVH().upload(*pending_chain(129))
    rc, a, o = codes(cw, api.LAYOUT_CWBVH)           # more pending node groups than CW_STACK
    assert rc == a == o == _lib.E_LIMIT
    dd, tt = pending_chain(3)
    n = dd.view(np.uint8).reshape(-1, 80)
    n[6, 24], n[6, 15] = 0x38, 1                     # an inner child leading back to the root
    n.view(np.uint32).reshape(-1, 20)[6, 4] = 0
    rc, a, o = codes(api.BVH8_CWBVH().upload(dd, tt), api.LAYOUT_CWBVH)
    assert rc == a == o == _lib.E_ARG
    from tests.test_deep_bvh2_gpu import instances, spine
    nodes, idx, verts = spine(64, 64)
    deep_blas = api.BVH().upload(nodes, idx, verts)
    _lib.check(L.tbvh_convert(deep_blas.h, api.LAYOUT_CWBVH))
    dt = api.TLAS().Build(instances(), [deep_blas], blas_layout=api.LAYOUT_CWBVH)
    rc, a, o = codes(dt, api.LAYOUT_BVH)             # a BVH-layout walk over a BLAS too deep for the two-level stack
    assert rc == a == o == _lib.E_LIMIT
    assert codes(dt, api.LAYOUT_CWBVH) == (0, 0, 0)
    assert L.tbvh_device_view(None, api.LAYOUT_BVH, C.byref(_lib.DeviceView())) == _lib.E_ARG
    assert L.tbvh_device_view(b.h, api.LAYOUT_BVH, None) == _lib.E_ARG


def test_python_view_object(consumer, scene):
    v, fams = scene
    cw = api.BVH8_CWBVH().Build(v)
    view = cw.device_view()
    assert view.kind == _lib.VIEW_CWBVH and len(bytes(view)) == 64 and C.sizeof(view) == 64


def test_example_program_runs(gpu, tmp_path):
    """harness/device_api_b200.cu: the shim's BVH8_CWBVH, DeviceView() and a kernel of its own, checked against the batch call"""
    exe = str(tmp_path / "device_api_b200")
    lib = os.path.join(REPO, "tinybvh_b200")
    subprocess.check_call([build.nvcc_path(), "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-I" + os.path.join(REPO, "include"),
                           os.path.join(REPO, "harness", "device_api_b200.cu"), "-L" + lib, "-ltinybvh_b200", "-Xlinker", "-rpath," + lib, "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "0 mismatches against the batch call" in r.stdout
