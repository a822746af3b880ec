"""tbvh_intersect_all_tlas on the device, held bit for bit to the host restatement (tests/allhits_tlas_oracle.c, DESIGN.md §4.14 two levels): every
record, instance and count at k in {1, 2, 4, 5, 16, 17, 63, 64} over BLASses of every builder, batch-built, indexed and uploaded (a DAG and
shrunk boxes included), 1 to 3,000 instances with ray masks and the instance-update transform families, TLASes from Build and from
Rebuild frames with host and device records, after a BLAS refit, and a group replica; host and device space, strides, stream order, every
refusal in order, the cross-checks against the TLAS's tbvh_intersect_device / tbvh_occluded_device, inst_idx_bits 10, and the device
function from a caller's kernel (tests/intersect_all_tlas_consumer.cu)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import refpy
from tinybvh_b200 import _lib, api, build, rays as R, scenes
from tests import allhits_oracle as ao, allhits_tlas_oracle as tao, util
from tests.test_closest_point import family
from tests.test_closest_point_gpu import chain_tree
from tests.test_intersect_all import KS, same
from tests.test_intersect_all_gpu import torch_u8
from tests.test_intersect_all_tlas import tlas_rays
from tests.test_oracle_pin import tlas_case
from tests.test_tlas_update import update_families

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NO_PRIM = ao.NO_PRIM


def device_all(h, rays, k, stream=None):
    """the batch call in device space on handle h -> (hits (n, k, 4) float32, insts (n, k) uint32, counts uint32)"""
    import torch
    n = rays.shape[0]
    dr = torch_u8(rays)
    hits = torch.zeros((max(n, 1), k, 4), dtype=torch.float32, device="cuda")
    insts = torch.zeros((max(n, 1), k), dtype=torch.int32, device="cuda")
    counts = torch.zeros(max(n, 1), dtype=torch.int32, device="cuda")
    _lib.check(_lib.lib().tbvh_intersect_all_tlas(h, C.c_void_p(dr.data_ptr()), rays.dtype.itemsize, n, k, C.c_void_p(hits.data_ptr()),
                                                  C.c_void_p(insts.data_ptr()), C.c_void_p(counts.data_ptr()), _lib.DEVICE, stream))
    torch.cuda.synchronize()
    return hits.cpu().numpy()[:n], insts.cpu().numpy().view(np.uint32)[:n], counts.cpu().numpy().view(np.uint32)[:n]


def host_all(h, rays, k):
    n = rays.shape[0]
    r = np.ascontiguousarray(rays)
    hits = np.zeros((n, k, 4), np.float32)
    insts = np.zeros((n, k), np.uint32)
    counts = np.zeros(n, np.uint32)
    _lib.check(_lib.lib().tbvh_intersect_all_tlas(h, r.ctypes.data, r.dtype.itemsize, n, k, hits.ctypes.data, insts.ctypes.data, counts.ctypes.data,
                                                  _lib.HOST, None))
    return hits, insts, counts


def restated(t, inst, blas_objs, verts):
    """the TLAS tree, the updated instance records and every BLAS's (nodes, prim_idx, verts) as the handles hold them"""
    tn, ti = t.download()
    return tn, ti, inst, [(*b.download(), v) for b, v in zip(blas_objs, verts)]


def check_tlas(h, scene, rays, label, ks=KS, host=False, oracle="brute"):
    """every record, instance and count of the device batch call on handle h equals the restatement's, for every k"""
    for k in ks:
        want = tao.brute(*scene, rays, k)[:3] if oracle == "brute" else tao.walk(*scene, rays, k)
        got = device_all(h, rays, k)
        bad = ~(got[0].view(np.uint32) == want[0].view(np.uint32)).all((1, 2)) | ~(got[1] == want[1]).all(1) | (got[2] != want[2])
        assert not bad.any(), f"{label} k={k}: {int(bad.sum())} of {rays.shape[0]} rays differ, first {np.nonzero(bad)[0][:5]}: " \
                              f"{got[0][bad][:1]} {got[1][bad][:1]} {got[2][bad][:3]} vs {want[0][bad][:1]} {want[1][bad][:1]} {want[2][bad][:3]}"
        if host:
            hh = host_all(h, rays, k)
            assert same(hh[0], want[0]) and np.array_equal(hh[1], want[1]) and np.array_equal(hh[2], want[2]), f"{label} k={k}: host space differs"


def make_tlas(v, inst, builder="Build"):
    blas = [getattr(api.BVH(), builder)(x) for x in v]
    t = api.TLAS().Build(inst, blas)
    return t, blas


@pytest.mark.parametrize("builder", ["Build", "BuildAVX", "BuildHQ", "BuildPLOC"])
@pytest.mark.parametrize("n_inst", [1, 40, 300])
def test_builders_and_instance_counts(gpu, builder, n_inst):
    v, inst, O, D = tlas_case(91, n_inst)
    t, blas = make_tlas(v, inst, builder)
    scene = restated(t, inst, blas, v)
    for mask in (0x1, 0x2):
        rays = tlas_rays(inst, np.random.default_rng(n_inst + mask), n=500, mask=mask)
        check_tlas(t.h, scene, rays, f"{builder}/{n_inst}/{mask:#x}", ks=KS if mask == 0x2 else (1, 5, 64), host=n_inst == 40 and mask == 0x1)


def test_three_thousand_instances(gpu):
    v = [scenes.procedural_scene(n, 30 + n) for n in (300, 2000, 5000)]
    inst = refpy.make_instances(util.random_transforms(3000, 8, spread=200.0), np.arange(3000) % 3, masks=[0x3 if i % 7 else 0x2 for i in range(3000)])
    t, blas = make_tlas(v, inst)
    scene = restated(t, inst, blas, v)
    for mask in (0x1, 0x2):
        check_tlas(t.h, scene, tlas_rays(inst, np.random.default_rng(mask), n=1500, mask=mask), f"3000/{mask:#x}", ks=(1, 4, 17, 64), oracle="walk")


def test_batch_indexed_and_uploaded_blasses(gpu):
    meshes = [scenes.procedural_scene(n, 20 + n) for n in (5, 700, 4000)]
    inst = refpy.make_instances(util.random_transforms(60, 3), np.arange(60) % 3)
    for flavour in (_lib.BUILD_REFERENCE, _lib.BUILD_AVX, _lib.BUILD_PLOC, _lib.BUILD_HQ):
        objs = [api.BVH() for _ in meshes]
        api.build_batch(objs, meshes, flavour)
        i2 = inst.copy()
        t = api.TLAS().Build(i2, objs)
        check_tlas(t.h, restated(t, i2, objs, meshes), tlas_rays(i2, np.random.default_rng(flavour), n=400), f"batch-{flavour}", ks=(2, 16, 63))
    idx_objs, flat = [], []
    for v in meshes[1:]:
        uniq, invi = np.unique(v.reshape(-1, 4), axis=0, return_inverse=True)
        e = api.BVH()
        e.Build(uniq, indices=invi.astype(np.uint32).reshape(-1))
        idx_objs.append(e)
        flat.append(uniq[invi.reshape(-1)])
    i2 = refpy.make_instances(util.random_transforms(30, 4), np.arange(30) % 2)
    t = api.TLAS().Build(i2, idx_objs)
    check_tlas(t.h, restated(t, i2, idx_objs, flat), tlas_rays(i2, np.random.default_rng(2), n=400), "indexed", ks=(1, 5, 64))
    v = scenes.procedural_scene(3000, 71)
    for fam in util.FAMILIES + ["shrunk", "dag"]:
        nodes, idx = family(util.source_tree(v, "Build"), fam)
        e = api.BVH().upload(nodes, idx, v)
        i2 = refpy.make_instances(util.random_transforms(20, 5), [0] * 20)
        t = api.TLAS().Build(i2, [e])
        check_tlas(t.h, restated(t, i2, [e], [v]), tlas_rays(i2, np.random.default_rng(9), n=400), fam, ks=(1, 4, 17, 64))


@pytest.mark.parametrize("name", list(update_families().keys()))
def test_update_families(gpu, name):
    T = update_families()[name]
    v = [scenes.procedural_scene(500, 3), scenes.procedural_scene(300, 4)]
    inst = refpy.make_instances(T, np.arange(T.shape[0]) % 2)
    t, blas = make_tlas(v, inst)
    check_tlas(t.h, restated(t, inst, blas, v), tlas_rays(inst, np.random.default_rng(3), n=500), name, ks=(1, 4, 17, 64))


def test_rebuild_frames_and_refit(gpu):
    """TLAS.Rebuild frames from host records and from device records, then a BLAS refit and a rebuild over it"""
    import torch
    v, inst, O, D = tlas_case(93, 80)
    t, blas = make_tlas(v, inst)
    check_tlas(t.h, restated(t, inst, blas, v), tlas_rays(inst, np.random.default_rng(1), n=400), "build", ks=(1, 5, 64))
    for frame in (1, 2):
        rec = inst.copy()
        rec["transform"] = util.random_transforms(80, 100 + frame)
        if frame == 1:
            t.Rebuild(rec)
        else:
            d = torch.from_numpy(rec.view(np.uint8).reshape(80, 192).copy()).cuda()
            t.Rebuild(d)
            rec = d.cpu().numpy().view(rec.dtype).reshape(-1)
        check_tlas(t.h, restated(t, rec, blas, v), tlas_rays(rec, np.random.default_rng(frame), n=400), f"frame {frame}", ks=(2, 17, 63), host=True)
    moved = [x.copy() for x in v]
    for x in moved:
        x[:, :3] += np.random.default_rng(4).normal(size=(x.shape[0], 3)).astype(np.float32) * 0.05
    for b, x in zip(blas, moved):
        b.Refit(x)
    rec = inst.copy()
    t.Rebuild(rec, blas)
    check_tlas(t.h, restated(t, rec, blas, moved), tlas_rays(rec, np.random.default_rng(5), n=400), "refit + rebuild", ks=(1, 4, 64))


def test_group_replica(gpu, consumer):
    v, inst, O, D = tlas_case(95, 50)
    t, blas = make_tlas(v, inst)
    rays = tlas_rays(inst, np.random.default_rng(17), n=600)
    check_tlas(t.h, restated(t, inst, blas, v), rays, "source", ks=(5,))
    want = device_all(t.h, rays, 5)
    grp = api.Group([0])
    grp.replicate(t)
    rep = _lib.lib().tbvh_group_replica(grp.h, 0)
    assert rep and rep != t.h.value
    got = device_all(C.c_void_p(rep), rays, 5)
    assert same(got[0], want[0]) and np.array_equal(got[1], want[1]) and np.array_equal(got[2], want[2]), "replica handle"
    got = run_consumer(consumer, grp.device_view(0, api.LAYOUT_BVH), rays, np.full(rays.shape[0], 5, np.uint32))
    assert same(got[0].reshape(-1, 5, 4), want[0]) and np.array_equal(got[1].reshape(-1, 5), want[1]) and np.array_equal(got[2], want[2]), "replica view"
    grp.close()


def test_strides_host_stream_and_api(gpu):
    import torch
    v, inst, O, D = tlas_case(96, 40)
    t, blas = make_tlas(v, inst)
    rays = tlas_rays(inst, np.random.default_rng(13), n=1500)
    want = tao.brute(*restated(t, inst, blas, v), rays, 17)[:3]
    for stride in (64, 128):
        padded = np.zeros((rays.shape[0], stride), np.uint8)
        padded[:, :64] = rays.view(np.uint8).reshape(-1, 64)
        padded[:, 64:] = 0xA5
        rec = padded.view(np.dtype((np.void, stride))).reshape(-1)
        for got in (device_all(t.h, rec, 17), host_all(t.h, rec, 17)):
            assert same(got[0], want[0]) and np.array_equal(got[1], want[1]) and np.array_equal(got[2], want[2]), f"stride {stride}"
    h, ii, c = t.intersect_all(rays, 17)
    assert same(h, want[0]) and np.array_equal(ii, want[1]) and np.array_equal(c, want[2]) and c.dtype == np.uint32 and ii.dtype == np.uint32
    th, ti, tc = t.intersect_all(torch_u8(rays), 17)
    torch.cuda.synchronize()
    assert same(th.cpu().numpy(), want[0]) and np.array_equal(ti.cpu().numpy().view(np.uint32), want[1]) and np.array_equal(tc.cpu().numpy().view(np.uint32), want[2])
    # stream order: the rays are written behind a long kernel on the caller's stream
    want4 = tao.brute(*restated(t, inst, blas, v), rays, 4)[:3]
    s = torch.cuda.Stream()
    src = torch_u8(rays)
    dr = torch.zeros_like(src)
    hits = torch.zeros((rays.shape[0], 4, 4), dtype=torch.float32, device="cuda")
    insts = torch.zeros((rays.shape[0], 4), dtype=torch.int32, device="cuda")
    counts = torch.zeros(rays.shape[0], dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)
        dr.copy_(src)
    _lib.check(_lib.lib().tbvh_intersect_all_tlas(t.h, C.c_void_p(dr.data_ptr()), 64, rays.shape[0], 4, C.c_void_p(hits.data_ptr()), C.c_void_p(insts.data_ptr()),
                                                  C.c_void_p(counts.data_ptr()), _lib.DEVICE, C.c_void_p(s.cuda_stream)))
    s.synchronize()
    assert same(hits.cpu().numpy(), want4[0]) and np.array_equal(insts.cpu().numpy().view(np.uint32), want4[1]) and \
        np.array_equal(counts.cpu().numpy().view(np.uint32), want4[2]), "walked before the stream wrote the rays"
    for n in (1, 31, 33, 100):
        got = device_all(t.h, rays[:n], 4)
        assert same(got[0], want4[0][:n]) and np.array_equal(got[1], want4[1][:n]) and np.array_equal(got[2], want4[2][:n]), f"n = {n}"


def test_refusals_in_order(gpu):
    import torch
    L = _lib.lib()
    v, inst, O, D = tlas_case(97, 12)
    t, blas = make_tlas(v, inst)
    rays = torch_u8(tlas_rays(inst, np.random.default_rng(1), n=16)[:64])
    hits = torch.zeros((rays.shape[0] + 1, 64, 4), dtype=torch.float32, device="cuda")
    insts = torch.zeros((rays.shape[0] + 1, 64), dtype=torch.int32, device="cuda")
    counts = torch.zeros(rays.shape[0] + 1, dtype=torch.int32, device="cuda")
    rp, hp, ip, cp = C.c_void_p(rays.data_ptr()), C.c_void_p(hits.data_ptr()), C.c_void_p(insts.data_ptr()), C.c_void_p(counts.data_ptr())
    fn, Dv = L.tbvh_intersect_all_tlas, _lib.DEVICE
    assert fn(None, rp, 64, 4, 4, hp, ip, cp, Dv, None) == _lib.E_ARG
    assert fn(t.h, None, 64, 4, 4, hp, ip, cp, Dv, None) == _lib.E_ARG
    assert fn(t.h, rp, 64, 4, 4, None, ip, cp, Dv, None) == _lib.E_ARG
    assert fn(t.h, rp, 64, 4, 4, hp, None, cp, Dv, None) == _lib.E_ARG
    assert fn(t.h, rp, 64, 4, 4, hp, ip, None, Dv, None) == _lib.E_ARG
    assert fn(t.h, rp, 64, 4, 4, hp, ip, cp, 7, None) == _lib.E_ARG
    for stride in (0, 48, 72, 100):
        assert fn(t.h, rp, stride, 4, 4, hp, ip, cp, Dv, None) == _lib.E_ARG
    assert fn(t.h, C.c_void_p(rays.data_ptr() + 4), 64, 4, 4, hp, ip, cp, Dv, None) == _lib.E_ARG
    assert fn(t.h, rp, 64, 4, 4, C.c_void_p(hits.data_ptr() + 4), ip, cp, Dv, None) == _lib.E_ARG
    assert fn(t.h, rp, 64, 4, 4, hp, C.c_void_p(insts.data_ptr() + 2), cp, Dv, None) == _lib.E_ARG
    assert fn(t.h, rp, 64, 4, 4, hp, ip, C.c_void_p(counts.data_ptr() + 2), Dv, None) == _lib.E_ARG
    for k in (0, 65, 1 << 31):
        assert fn(t.h, rp, 64, 4, k, hp, ip, cp, Dv, None) == _lib.E_ARG
    assert fn(t.h, rp, 64, 1 << 40, 4, hp, ip, cp, Dv, None) == _lib.E_ARG
    assert fn(t.h, rp, 64, 0, 4, hp, ip, cp, Dv, None) == _lib.OK
    # a handle without a TLAS
    assert fn(blas[0].h, rp, 64, 4, 4, hp, ip, cp, Dv, None) == _lib.E_UNSUPPORTED
    assert fn(api.BVH().h, rp, 64, 4, 4, hp, ip, cp, Dv, None) == _lib.E_UNSUPPORTED
    # and tbvh_intersect_all still refuses the TLAS
    assert L.tbvh_intersect_all(t.h, rp, 64, 4, 4, hp, cp, Dv, None) == _lib.E_UNSUPPORTED
    # what tbvh_intersect_device( tlas, TBVH_LAYOUT_BVH ) refuses, with its codes: a BLAS too deep for the two-level walk
    sv = scenes.procedural_scene(300, 19)
    deep = chain_tree(sv, 100)
    d = api.BVH().upload(deep[0], deep[1], sv[:300])
    _lib.check(L.tbvh_convert(d.h, api.LAYOUT_CWBVH))
    i2 = refpy.make_instances(util.random_transforms(4, 2), [0, 1, 0, 1])
    td = api.TLAS().Build(i2, [d, blas[1]], blas_layout=api.LAYOUT_CWBVH)
    dr = torch_u8(tlas_rays(i2, np.random.default_rng(2), n=16)[:8])
    want = L.tbvh_intersect_device(td.h, _lib.LAYOUT_BVH, C.c_void_p(dr.data_ptr()), 64, None, 8, None)
    assert want == _lib.E_LIMIT and fn(td.h, rp, 64, 4, 4, hp, ip, cp, Dv, None) == _lib.E_LIMIT
    # BLASses without a BVH-layout tree
    c = api.BVH8_CWBVH().Build(sv)
    only = api.BVH8_CWBVH().upload(*c.download())
    i3 = refpy.make_instances(util.random_transforms(3, 3), [0, 0, 0])
    api.TLAS().Build(i3, [c], blas_layout=api.LAYOUT_CWBVH)     # the records updated over the same triangles' tree
    tc = api.TLAS().Build(i3, [only], update=False, blas_layout=api.LAYOUT_CWBVH)
    assert L.tbvh_intersect_device(tc.h, _lib.LAYOUT_BVH, C.c_void_p(dr.data_ptr()), 64, None, 8, None) == _lib.E_STATE
    assert fn(tc.h, rp, 64, 4, 4, hp, ip, cp, Dv, None) == _lib.E_STATE
    # a stale TLAS: a BLAS rebuilt since
    blas[0].Build(v[0])
    assert fn(t.h, rp, 64, 4, 4, hp, ip, cp, Dv, None) == _lib.E_STATE
    # the order: an argument error before a missing TLAS, a missing TLAS before a stale one
    assert fn(t.h, rp, 64, 4, 0, hp, ip, cp, Dv, None) == _lib.E_ARG
    assert fn(blas[1].h, rp, 48, 4, 4, hp, ip, cp, Dv, None) == _lib.E_ARG
    assert fn(t.h, rp, 64, 4, 4, hp, None, cp, Dv, None) == _lib.E_ARG
    torch.cuda.synchronize()
    assert not hits.any() and not insts.any() and not counts.any(), "a refused call wrote results"


def test_cross_checks_against_intersect_and_occluded(gpu):
    """k = 1: record 0's t is the TLAS's tbvh_intersect_device (BVH layout) bit for bit wherever key == t, its instance and prim differ
    only on exact-t ties; count > 0 is tbvh_occluded_device's bit (a NaN t or NaN tmax aside)"""
    import torch
    L = _lib.lib()
    v, inst, O, D = tlas_case(98, 200)
    for builder in ("Build", "BuildHQ"):
        i2 = inst.copy()
        t, blas = make_tlas(v, i2, builder)
        scene = restated(t, i2, blas, v)
        rays = tlas_rays(i2, np.random.default_rng(19), n=4000, mask=0x2)
        h, ii, c, keys = tao.brute(*scene, rays, 1)
        got = device_all(t.h, rays, 1)
        assert same(got[0], h) and np.array_equal(got[1], ii) and np.array_equal(got[2], c)
        rec = np.zeros((rays.shape[0], 64), np.uint8)
        rec[:] = rays.view(np.uint8).reshape(-1, 64)
        dr = torch.from_numpy(rec).cuda()
        bits = torch.zeros((rays.shape[0] + 31) // 32, dtype=torch.int32, device="cuda")
        _lib.check(L.tbvh_occluded_device(t.h, _lib.LAYOUT_BVH, C.c_void_p(dr.data_ptr()), 64, C.c_void_p(bits.data_ptr()), rays.shape[0], None))
        _lib.check(L.tbvh_intersect_device(t.h, _lib.LAYOUT_BVH, C.c_void_p(dr.data_ptr()), 64, None, rays.shape[0], None))
        torch.cuda.synchronize()
        ref = dr.cpu().numpy().copy().view(R.GPU_RAY_DTYPE).reshape(-1)
        occ = np.unpackbits(bits.cpu().numpy().view(np.uint8), bitorder="little")[: rays.shape[0]].astype(bool)
        nan = np.isnan(ref["t"]) | np.isnan(rays["t"])
        assert np.array_equal((c > 0)[~nan], occ[~nan]), f"{builder}: count > 0 differs from tbvh_occluded_device"
        exact = (c > 0) & (keys[:, 0].view(np.uint32) == h[:, 0, 0].view(np.uint32))
        assert exact.sum() > 0.6 * (c > 0).sum() and exact.sum() > 500
        assert same(h[exact, 0, 0], ref["t"][exact]), f"{builder}: t differs from tbvh_intersect_device"
        tie = exact & ((ao.prims(h)[:, 0] != ref["prim"]) | (ii[:, 0] != ref["pad"]))
        for i in np.nonzero(tie)[0][:50]:
            hh, hi, cc, _ = tao.brute(*scene, rays[i:i + 1], 64)
            m = min(int(cc[0]), 64)
            at = hh[0, :m, 0] == h[i, 0, 0]
            assert (int(ref["pad"][i]), int(ref["prim"][i])) in set(zip(hi[0, :m][at].tolist(), ao.prims(hh)[0, :m][at].tolist())), \
                f"{builder}: ray {i} differs without a tie"


def test_inst_idx_bits_do_not_apply(gpu):
    v, inst, O, D = tlas_case(99, 30)
    t, blas = make_tlas(v, inst)
    rays = tlas_rays(inst, np.random.default_rng(4), n=800)
    want = device_all(t.h, rays, 17)
    api.set_option("inst_idx_bits", 10)
    try:
        got = device_all(t.h, rays, 17)
        got_host = host_all(t.h, rays, 17)
    finally:
        api.set_option("inst_idx_bits", 32)
    for g in (got, got_host):
        assert same(g[0], want[0]) and np.array_equal(g[1], want[1]) and np.array_equal(g[2], want[2])


@pytest.fixture(scope="module")
def consumer(gpu, tmp_path_factory):
    nvcc = build.nvcc_path()
    so = str(tmp_path_factory.mktemp("intersect_all_tlas_consumer") / "consumer.so")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I" + os.path.join(REPO, "include"),
                        "-Xcompiler", "-fPIC", "-shared", "-Xptxas", "-v", os.path.join(REPO, "tests", "intersect_all_tlas_consumer.cu"), "-o", so],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    print(r.stderr)
    L = C.CDLL(so)
    L.iat_query.argtypes = [_lib.DeviceView] + [C.c_void_p] * 7 + [C.c_uint32, C.c_uint32]
    return L


def run_consumer(consumer, view, rays, ks, sel=None, reps=1):
    """-> (the records of every ray concatenated, their instances, counts); unselected rays keep -7 records, instances 0x5a5a5a5a and
    count 0x5a5a5a5a"""
    import torch
    n = rays.shape[0]
    offs = np.concatenate([[0], np.cumsum(ks.astype(np.uint64))[:-1]]).astype(np.uint64)
    out = torch.full((int(ks.sum()), 4), -7.0, dtype=torch.float32, device="cuda")
    insts = torch.full((int(ks.sum()),), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
    counts = torch.full((n,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
    dks = torch.from_numpy(ks.astype(np.uint32).view(np.int32)).cuda()
    doffs = torch.from_numpy(offs.view(np.int64)).cuda()
    ds = torch.from_numpy(sel.view(np.int32)).cuda() if sel is not None else None
    assert consumer.iat_query(view, torch_u8(rays).data_ptr(), dks.data_ptr(), doffs.data_ptr(), out.data_ptr(), insts.data_ptr(), counts.data_ptr(),
                              ds.data_ptr() if ds is not None else None, n, reps) == 0
    return out.cpu().numpy(), insts.cpu().numpy().view(np.uint32), counts.cpu().numpy().view(np.uint32)


def test_device_function(gpu, consumer):
    """intersect_all_tlas from divergent lanes, with a different k per lane and in a loop, gives the batch call's bytes; views of other
    kinds get empty records"""
    v, inst, O, D = tlas_case(90, 60)
    t, blas = make_tlas(v, inst)
    rays = tlas_rays(inst, np.random.default_rng(16), n=600)
    n = rays.shape[0]
    ks = np.array(KS, np.uint32)[np.random.default_rng(5).integers(0, len(KS), n)]
    want = {k: device_all(t.h, rays, k) for k in KS}
    sel = np.random.default_rng(3).integers(0, 1 << 32, (n + 31) // 32, dtype=np.uint64).astype(np.uint32)
    for s, reps in ((None, 1), (sel, 1), (None, 3)):
        got, gi, cnt = run_consumer(consumer, t.device_view(api.LAYOUT_BVH), rays, ks, s, reps)
        mask = np.ones(n, bool) if s is None else np.unpackbits(s.view(np.uint8), bitorder="little")[:n].astype(bool)
        off = 0
        for i in range(n):
            k = int(ks[i])
            rec, ri = got[off: off + k], gi[off: off + k]
            off += k
            if mask[i]:
                assert same(rec, want[k][0][i]) and np.array_equal(ri, want[k][1][i]) and cnt[i] == want[k][2][i], f"ray {i} (k={k}): differs from the batch call"
            else:
                assert (rec == -7).all() and (ri == 0x5A5A5A5A).all() and cnt[i] == 0x5A5A5A5A
    # views of other kinds: a TLAS view taken for CWBVH, a BVH view
    cw = [api.BVH8_CWBVH().Build(x) for x in v]
    tcw = api.TLAS().Build(inst.copy(), cw, blas_layout=api.LAYOUT_CWBVH)
    r = R.gpu_records(R.make_rays(np.zeros((1, 3), np.float32), np.array([[0, 0, 1]], np.float32), np.float32(5)))
    for view in (tcw.device_view(api.LAYOUT_CWBVH), blas[0].device_view()):
        got, gi, cnt = run_consumer(consumer, view, r, np.array([3], np.uint32))
        assert got.view(np.uint32).tolist() == [[np.float32(5).view(np.uint32), 0, 0, NO_PRIM]] * 3 and (gi == NO_PRIM).all() and cnt[0] == 0
