"""tbvh_intersect_all on the device, held bit for bit to the host restatement (tests/allhits_oracle.c, DESIGN.md §4.14) over the tree the
handle holds: every builder (BuildHQ with failed splits included), batch and indexed builds, uploaded families, a shrunk-box tree and a DAG,
a BVH_GPU upload and converted objects, deep and one-leaf trees, golden and off-atrium scenes, refits, tbvh_optimize and a group replica,
at k in {1, 2, 4, 5, 16, 17, 63, 64}; host and device space, strides, stream order, every refusal, the cross-checks against
tbvh_intersect_device and tbvh_occluded_device, and the device function from a caller's kernel (tests/intersect_all_consumer.cu)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import portpy
from tinybvh_b200 import _lib, api, build, rays as R, scenes
from tests import allhits_oracle as ao, util
from tests.test_closest_point import family
from tests.test_closest_point_gpu import chain_tree
from tests.test_intersect_all import KS, rays_for

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NODE32 = portpy.NODE32


def torch_u8(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(a.shape[0], -1).copy()).cuda()


def device_all(obj, rays, k, stream=None):
    """the batch call in device space -> (hits (n, k, 4) float32, counts uint32)"""
    import torch
    n = rays.shape[0]
    dr = torch_u8(rays)
    hits = torch.zeros((max(n, 1), k, 4), dtype=torch.float32, device="cuda")
    counts = torch.zeros(max(n, 1), dtype=torch.int32, device="cuda")
    _lib.check(_lib.lib().tbvh_intersect_all(obj.h, C.c_void_p(dr.data_ptr()), rays.dtype.itemsize, n, k, C.c_void_p(hits.data_ptr()),
                                             C.c_void_p(counts.data_ptr()), _lib.DEVICE, stream))
    torch.cuda.synchronize()
    return hits.cpu().numpy()[:n], counts.cpu().numpy().view(np.uint32)[:n]


def host_all(obj, rays, k):
    n = rays.shape[0]
    r = np.ascontiguousarray(rays)
    hits = np.zeros((n, k, 4), np.float32)
    counts = np.zeros(n, np.uint32)
    _lib.check(_lib.lib().tbvh_intersect_all(obj.h, r.ctypes.data, r.dtype.itemsize, n, k, hits.ctypes.data, counts.ctypes.data, _lib.HOST, None))
    return hits, counts


def same(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def check_tree(obj, nodes, idx, v, rays, label, ks=KS, host=False, oracle="brute"):
    """every record and count of the device batch call equals the restatement's, for every k"""
    for k in ks:
        want = ao.brute(nodes, idx, v, rays, k)[:2] if oracle == "brute" else ao.walk(nodes, idx, v, rays, k)
        got = device_all(obj, rays, k)
        bad = ~(np.ascontiguousarray(got[0]).view(np.uint32) == np.ascontiguousarray(want[0]).view(np.uint32)).all((1, 2)) | (got[1] != want[1])
        assert not bad.any(), f"{label} k={k}: {int(bad.sum())} of {rays.shape[0]} rays differ, first {np.nonzero(bad)[0][:5]}: " \
                              f"{got[0][bad][:1]} {got[1][bad][:3]} vs {want[0][bad][:1]} {want[1][bad][:3]}"
        if host:
            h = host_all(obj, rays, k)
            assert same(h[0], want[0]) and np.array_equal(h[1], want[1]), f"{label} k={k}: host space differs"


def scene(n, seed=5):
    return scenes.procedural_scene(n, seed)


@pytest.mark.parametrize("builder", ["Build", "BuildAVX", "BuildHQ", "BuildPLOC"])
@pytest.mark.parametrize("ntris", [1, 9, 3000, 40000])
def test_builders(gpu, builder, ntris):
    v = scene(ntris, 3 + ntris % 5)
    e = getattr(api.BVH(), builder)(v)
    nodes, idx = e.download()
    rays = rays_for(v, np.random.default_rng(ntris), n=1500)
    check_tree(e, nodes, idx, v, rays, f"{builder}-{ntris}", host=ntris == 3000, oracle="walk" if ntris == 40000 else "brute")


@pytest.mark.parametrize("name", ["snapped20k_q4", "lattice10k_k3", "clusters"])
def test_hq_failed_splits(gpu, name):
    from tests.test_build_hq_shapes import fail_scene
    v = util.long_leaf_scene(name) if name == "clusters" else fail_scene(name)
    e = api.BVH().BuildHQ(v)
    nodes, idx = e.download()
    check_tree(e, nodes, idx, v, rays_for(v, np.random.default_rng(1), n=800), f"BuildHQ-{name}", ks=(1, 4, 17, 64), oracle="walk")


def test_batch_and_indexed(gpu):
    meshes = [scene(n, 20 + n) for n in (5, 700, 4000)]
    for flavour in (_lib.BUILD_REFERENCE, _lib.BUILD_AVX, _lib.BUILD_PLOC, _lib.BUILD_HQ):
        objs = [api.BVH() for _ in meshes]
        api.build_batch(objs, meshes, flavour)
        for o, v in zip(objs, meshes):
            nodes, idx = o.download()
            check_tree(o, nodes, idx, v, rays_for(v, np.random.default_rng(2), n=400), f"batch-{flavour}-{v.shape[0] // 3}", ks=(2, 16, 63))
    v = scene(3000, 8)
    uniq, inv = np.unique(v.reshape(-1, 4), axis=0, return_inverse=True)
    e = api.BVH()
    e.Build(uniq, indices=inv.astype(np.uint32).reshape(-1))
    nodes, idx = e.download()
    check_tree(e, nodes, idx, uniq[inv.reshape(-1)], rays_for(v, np.random.default_rng(3), n=800), "indexed", ks=(1, 5, 64))


@pytest.mark.parametrize("fam", util.FAMILIES + ["shrunk", "dag"])
def test_uploaded_families(gpu, fam):
    v = scene(3000, 71)
    src = util.source_tree(v, "Build")
    nodes, idx = family(src, fam)
    e = api.BVH().upload(nodes, idx, v)
    check_tree(e, nodes, idx, v, rays_for(v, np.random.default_rng(5), n=800), fam, ks=(1, 4, 17, 64))


def test_bvh_gpu_upload_and_converted_objects(gpu):
    v = scene(3000, 9)
    o = util.oracle_tree(v, 1)
    g = api.BVH_GPU().upload(util.oracle_bvh_gpu_nodes(o), o.prim_idx, v)
    rays = rays_for(v, np.random.default_rng(6), n=800)
    check_tree(g, o.nodes, o.prim_idx, v, rays, "BVH_GPU upload", ks=(1, 5, 64))
    for cls in (api.BVH_GPU, api.BVH8_CWBVH):
        b = cls().Build(v)
        nodes = np.zeros(b.info().used_nodes, NODE32)
        idx = np.zeros(b.info().idx_count, np.uint32)
        _lib.check(_lib.lib().tbvh_download_bvh(b.h, nodes.ctypes.data, idx.ctypes.data, _lib.HOST))
        check_tree(b, nodes, idx, v, rays, cls.__name__, ks=(1, 5, 64))


def test_deep_and_one_leaf_trees(gpu):
    v = scene(400, 12)
    for m in (100, 255):
        nodes, idx = chain_tree(v, m)
        e = api.BVH().upload(nodes, idx, v[: 3 * m])
        assert e.info().max_depth == m - 1
        check_tree(e, nodes, idx, v[: 3 * m], rays_for(v[: 3 * m], np.random.default_rng(m), n=500), f"chain-{m}", ks=(1, 4, 5, 64), host=True)
    w = scene(40, 4)
    one = np.zeros(2, NODE32)
    tri = w.reshape(-1, 4)[:, :3]
    one[0] = (tri.min(0), 0, tri.max(0), 40)
    e = api.BVH().upload(one, np.arange(40, dtype=np.uint32), w)
    check_tree(e, one, np.arange(40, dtype=np.uint32), w, rays_for(w, np.random.default_rng(4), n=400), "one leaf", host=True)


@pytest.mark.parametrize("name", ["flat_500", "coincident_610", "single_tri", "atrium_3k"])
def test_golden_scenes(gpu, name):
    g = np.load(os.path.join(REPO, "tests", "golden", f"{name}.npz"))
    v = g["verts"].astype(np.float32)
    nodes = np.ascontiguousarray(g["nodes"]).view(NODE32).reshape(-1)
    e = api.BVH().upload(nodes, g["prim_idx"], v)
    rays = rays_for(v, np.random.default_rng(10), n=800)
    check_tree(e, nodes, g["prim_idx"], v, rays, name, ks=(1, 4, 17, 64))
    b = api.BVH().Build(v)
    check_tree(b, *b.download(), v, rays, name + "/Build", ks=(2, 63))


@pytest.mark.parametrize("variant", ["zero-random", "zero-order", "scale2^-20", "scale2^20", "translated"])
def test_off_atrium(gpu, variant):
    v = scene(3000, 33)
    if variant.startswith("zero"):
        v = util.signed_zero(v, variant[5:])
    elif variant.startswith("scale"):
        v = util.scaled(v, int(variant.split("^")[1]))
    else:
        v = v.copy()
        v[:, :3] += np.float32(1e4)
    for builder in ("Build", "BuildHQ"):
        e = getattr(api.BVH(), builder)(v)
        check_tree(e, *e.download(), v, rays_for(v, np.random.default_rng(11), n=800), f"{variant}/{builder}", ks=(1, 4, 17, 64))


def test_refit_and_optimize(gpu):
    v = scene(3000, 15)
    v2 = v.copy()
    v2[:, :3] += np.random.default_rng(1).normal(size=(v.shape[0], 3)).astype(np.float32) * 0.01
    rays = rays_for(v, np.random.default_rng(12), n=800)
    e = api.BVH().Build(v)
    e.Refit(v2)
    check_tree(e, *e.download(), v2, rays, "refit", ks=(1, 5, 64))
    g = api.BVH_GPU().Build(v)
    _lib.check(_lib.lib().tbvh_refit_layouts(g.h, C.c_void_p(np.ascontiguousarray(v2).ctypes.data), 16, v.shape[0] // 3, _lib.HOST))
    nodes = np.zeros(g.info().used_nodes, NODE32)
    idx = np.zeros(g.info().idx_count, np.uint32)
    _lib.check(_lib.lib().tbvh_download_bvh(g.h, nodes.ctypes.data, idx.ctypes.data, _lib.HOST))
    check_tree(g, nodes, idx, v2, rays, "refit_layouts", ks=(1, 5, 64))
    o = api.BVH().Build(v)
    o.optimize(4)
    check_tree(o, *o.download(), v, rays, "optimize", ks=(1, 5, 64))


def test_group_replica(gpu, consumer):
    import torch
    v = scene(3000, 25)
    e = api.BVH().Build(v)
    rays = rays_for(v, np.random.default_rng(17), n=800)
    want = device_all(e, rays, 5)
    check_tree(e, *e.download(), v, rays, "source", ks=(5,))
    grp = api.Group([0])
    grp.replicate(e)
    rep = _lib.lib().tbvh_group_replica(grp.h, 0)
    assert rep and rep != e.h.value
    dr = torch_u8(rays)
    hits = torch.zeros((rays.shape[0], 5, 4), dtype=torch.float32, device="cuda")
    counts = torch.zeros(rays.shape[0], dtype=torch.int32, device="cuda")
    _lib.check(_lib.lib().tbvh_intersect_all(C.c_void_p(rep), C.c_void_p(dr.data_ptr()), 64, rays.shape[0], 5, C.c_void_p(hits.data_ptr()),
                                             C.c_void_p(counts.data_ptr()), _lib.DEVICE, None))
    torch.cuda.synchronize()
    assert same(hits.cpu().numpy(), want[0]) and np.array_equal(counts.cpu().numpy().view(np.uint32), want[1]), "replica handle"
    got = run_consumer(consumer, grp.device_view(0), rays, np.full(rays.shape[0], 5, np.uint32))
    assert same(got[0].reshape(-1, 5, 4), want[0]) and np.array_equal(got[1], want[1]), "replica view"
    grp.close()


def test_strides_host_and_api(gpu):
    """strides 64, 128 and 144 (the records padded), host space, and the Python method for numpy and torch"""
    import torch
    v = scene(3000, 16)
    e = api.BVH().Build(v)
    rays = rays_for(v, np.random.default_rng(13), n=1000)
    want = ao.brute(*e.download(), v, rays, 17)[:2]
    for stride in (64, 128, 144):
        padded = np.zeros((rays.shape[0], stride), np.uint8)
        padded[:, :64] = rays.view(np.uint8).reshape(-1, 64)
        padded[:, 64:] = 0xA5
        rec = padded.view(np.dtype((np.void, stride))).reshape(-1)
        assert same(device_all(e, rec, 17)[0], want[0]) and same(host_all(e, rec, 17)[0], want[0]), f"stride {stride}"
        assert np.array_equal(host_all(e, rec, 17)[1], want[1])
    h, c = e.intersect_all(rays, 17)
    assert same(h, want[0]) and np.array_equal(c, want[1]) and c.dtype == np.uint32
    th, tc = e.intersect_all(torch_u8(rays), 17)
    torch.cuda.synchronize()
    assert same(th.cpu().numpy(), want[0]) and np.array_equal(tc.cpu().numpy().view(np.uint32), want[1])
    host128 = np.zeros(rays.shape[0], R.RAY_DTYPE)
    host128.view(np.uint8).reshape(-1, 128)[:, :64] = rays.view(np.uint8).reshape(-1, 64)
    before = host128.copy()
    h2, c2 = e.intersect_all(host128, 17)
    assert same(h2, want[0]) and np.array_equal(host128.view(np.uint8), before.view(np.uint8)), "the rays were modified"


def test_stream_order(gpu):
    import torch
    v = scene(3000, 17)
    e = api.BVH().Build(v)
    rays = rays_for(v, np.random.default_rng(14), n=2000)
    want = ao.brute(*e.download(), v, rays, 4)[:2]
    s = torch.cuda.Stream()
    src = torch_u8(rays)
    dr = torch.zeros_like(src)
    hits = torch.zeros((rays.shape[0], 4, 4), dtype=torch.float32, device="cuda")
    counts = torch.zeros(rays.shape[0], dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)   # the rays are written behind a long kernel on the caller's stream
        dr.copy_(src)
    _lib.check(_lib.lib().tbvh_intersect_all(e.h, C.c_void_p(dr.data_ptr()), 64, rays.shape[0], 4, C.c_void_p(hits.data_ptr()),
                                             C.c_void_p(counts.data_ptr()), _lib.DEVICE, C.c_void_p(s.cuda_stream)))
    s.synchronize()
    assert same(hits.cpu().numpy(), want[0]) and np.array_equal(counts.cpu().numpy().view(np.uint32), want[1]), "walked before the stream wrote the rays"
    for n in (1, 31, 33, 100):
        got = device_all(e, rays[:n], 4)
        assert same(got[0], want[0][:n]) and np.array_equal(got[1], want[1][:n]), f"n = {n}"


def test_refusals(gpu):
    import torch
    L = _lib.lib()
    v = scene(300, 18)
    e = api.BVH().Build(v)
    rays = torch_u8(rays_for(v, np.random.default_rng(1), n=16)[:64])
    hits = torch.zeros((rays.shape[0] + 1, 64, 4), dtype=torch.float32, device="cuda")
    counts = torch.zeros(rays.shape[0] + 1, dtype=torch.int32, device="cuda")
    rp, hp, cp = C.c_void_p(rays.data_ptr()), C.c_void_p(hits.data_ptr()), C.c_void_p(counts.data_ptr())
    fn, D = L.tbvh_intersect_all, _lib.DEVICE
    assert fn(None, rp, 64, 4, 4, hp, cp, D, None) == _lib.E_ARG
    assert fn(e.h, None, 64, 4, 4, hp, cp, D, None) == _lib.E_ARG
    assert fn(e.h, rp, 64, 4, 4, None, cp, D, None) == _lib.E_ARG
    assert fn(e.h, rp, 64, 4, 4, hp, None, D, None) == _lib.E_ARG
    assert fn(e.h, rp, 64, 4, 4, hp, cp, 7, None) == _lib.E_ARG
    for stride in (0, 48, 72, 100):
        assert fn(e.h, rp, stride, 4, 4, hp, cp, D, None) == _lib.E_ARG
    assert fn(e.h, C.c_void_p(rays.data_ptr() + 4), 64, 4, 4, hp, cp, D, None) == _lib.E_ARG
    assert fn(e.h, rp, 64, 4, 4, C.c_void_p(hits.data_ptr() + 4), cp, D, None) == _lib.E_ARG
    assert fn(e.h, rp, 64, 4, 4, hp, C.c_void_p(counts.data_ptr() + 2), D, None) == _lib.E_ARG
    for k in (0, 65, 1 << 31):
        assert fn(e.h, rp, 64, 4, k, hp, cp, D, None) == _lib.E_ARG
    assert fn(e.h, rp, 64, 1 << 40, 4, hp, cp, D, None) == _lib.E_ARG
    assert fn(e.h, rp, 64, 0, 4, hp, cp, D, None) == _lib.OK
    assert fn(api.BVH().h, rp, 64, 4, 4, hp, cp, D, None) == _lib.E_STATE
    c = api.BVH8_CWBVH().Build(v)
    only = api.BVH8_CWBVH().upload(*c.download())
    assert fn(only.h, rp, 64, 4, 4, hp, cp, D, None) == _lib.E_STATE
    deep = chain_tree(scene(300, 19), 300)
    d = api.BVH().upload(deep[0], deep[1], scene(300, 19))
    assert fn(d.h, rp, 64, 4, 4, hp, cp, D, None) == _lib.E_LIMIT
    inst = np.zeros(2, api.BLAS_INSTANCE)
    inst["transform"] = np.eye(4, dtype=np.float32).reshape(-1)
    inst["mask"] = 0xFFFF
    t = api.TLAS()
    t.Build(inst, [e])
    assert fn(t.h, rp, 64, 4, 4, hp, cp, D, None) == _lib.E_UNSUPPORTED
    # the order: an argument error before a TLAS, a TLAS before a missing tree
    assert fn(t.h, rp, 64, 4, 0, hp, cp, D, None) == _lib.E_ARG
    assert fn(d.h, rp, 48, 4, 4, hp, cp, D, None) == _lib.E_ARG
    torch.cuda.synchronize()
    assert not hits.any() and not counts.any(), "a refused call wrote results"


def test_cross_checks_against_intersect_and_occluded(gpu):
    """k = 1: record 0's t is tbvh_intersect_device's (BVH layout) bit for bit wherever key == t, its prim differs only on exact-t ties;
    count > 0 is tbvh_occluded_device's bit"""
    import torch
    v = scene(40000, 26)
    for builder in ("Build", "BuildHQ"):
        e = getattr(api.BVH(), builder)(v)
        nodes, idx = e.download()
        rays = rays_for(v, np.random.default_rng(19), n=6000)
        h, c, keys = ao.brute(nodes, idx, v, rays, 1)
        assert same(device_all(e, rays, 1)[0], h)
        dr = torch_u8(rays)
        hits = torch.zeros((rays.shape[0], 4), dtype=torch.float32, device="cuda")
        bits = torch.zeros((rays.shape[0] + 31) // 32, dtype=torch.int32, device="cuda")
        L = _lib.lib()
        _lib.check(L.tbvh_intersect_device(e.h, _lib.LAYOUT_BVH, C.c_void_p(dr.data_ptr()), 64, C.c_void_p(hits.data_ptr()), rays.shape[0], None))
        _lib.check(L.tbvh_occluded_device(e.h, _lib.LAYOUT_BVH, C.c_void_p(dr.data_ptr()), 64, C.c_void_p(bits.data_ptr()), rays.shape[0], None))
        torch.cuda.synchronize()
        ref = hits.cpu().numpy()
        occ = np.unpackbits(bits.cpu().numpy().view(np.uint8), bitorder="little")[: rays.shape[0]].astype(bool)
        # a NaN t is a hit for tbvh_intersect_device / tbvh_occluded_device and none here; so is any hit of a ray whose tmax is NaN (their
        # slab test's fminf drops the NaN, and no t compares above it), which gets count 0 here
        nan_t = np.isnan(ref[:, 0]) | np.isnan(rays["t"])
        assert np.array_equal((c > 0)[~nan_t], occ[~nan_t]), f"{builder}: count > 0 differs from tbvh_occluded_device"
        exact = (c > 0) & (keys[:, 0].view(np.uint32) == h[:, 0, 0].view(np.uint32))
        assert exact.sum() > 0.9 * (c > 0).sum()
        assert same(h[exact, 0, 0], ref[exact, 0]), f"{builder}: t differs from tbvh_intersect_device"
        tie = exact & (ao.prims(h)[:, 0] != ref[:, 3].view(np.uint32))
        for i in np.nonzero(tie)[0][:50]:
            hh, cc, _ = ao.brute(nodes, idx, v, rays[i:i + 1], 64)
            m = min(int(cc[0]), 64)
            assert ref[i, 3].view(np.uint32) in ao.prims(hh)[0, :m][hh[0, :m, 0] == h[i, 0, 0]], f"{builder}: ray {i} differs without a tie"


@pytest.fixture(scope="module")
def consumer(gpu, tmp_path_factory):
    nvcc = build.nvcc_path()
    so = str(tmp_path_factory.mktemp("intersect_all_consumer") / "consumer.so")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I" + os.path.join(REPO, "include"),
                        "-Xcompiler", "-fPIC", "-shared", "-Xptxas", "-v", os.path.join(REPO, "tests", "intersect_all_consumer.cu"), "-o", so],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    print(r.stderr)
    L = C.CDLL(so)
    L.ia_query.argtypes = [_lib.DeviceView, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32]
    return L


def run_consumer(consumer, view, rays, ks, sel=None, reps=1):
    """-> (the records of every ray concatenated, counts); unselected rays keep -7 records and count 0x5a5a5a5a"""
    import torch
    n = rays.shape[0]
    offs = np.concatenate([[0], np.cumsum(ks.astype(np.uint64))[:-1]]).astype(np.uint64)
    out = torch.full((int(ks.sum()), 4), -7.0, dtype=torch.float32, device="cuda")
    counts = torch.full((n,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
    dks = torch.from_numpy(ks.astype(np.uint32).view(np.int32)).cuda()
    doffs = torch.from_numpy(offs.view(np.int64)).cuda()
    ds = torch.from_numpy(sel.view(np.int32)).cuda() if sel is not None else None
    assert consumer.ia_query(view, torch_u8(rays).data_ptr(), dks.data_ptr(), doffs.data_ptr(), out.data_ptr(), counts.data_ptr(),
                             ds.data_ptr() if ds is not None else None, n, reps) == 0
    return out.cpu().numpy(), counts.cpu().numpy().view(np.uint32)


def test_device_function(gpu, consumer):
    """intersect_all_bvh from divergent lanes, with a different k per lane and in a loop, gives the batch call's bytes"""
    for m, v in ((None, scene(3000, 22)), (150, scene(400, 23))):
        if m:
            nodes, idx = chain_tree(v, m)
            v = v[: 3 * m]
            e = api.BVH().upload(nodes, idx, v)
        else:
            e = api.BVH().Build(v)
        rays = rays_for(v, np.random.default_rng(16), n=700)
        n = rays.shape[0]
        ks = np.array(KS, np.uint32)[np.random.default_rng(5).integers(0, len(KS), n)]
        want = {k: device_all(e, rays, k) for k in KS}
        sel = np.random.default_rng(3).integers(0, 1 << 32, (n + 31) // 32, dtype=np.uint64).astype(np.uint32)
        for s, reps in ((None, 1), (sel, 1), (None, 3)):
            got, cnt = run_consumer(consumer, e.device_view(), rays, ks, s, reps)
            mask = np.ones(n, bool) if s is None else np.unpackbits(s.view(np.uint8), bitorder="little")[:n].astype(bool)
            off = 0
            for i in range(n):
                k = int(ks[i])
                rec = got[off: off + k]
                off += k
                if mask[i]:
                    assert same(rec, want[k][0][i]) and cnt[i] == want[k][1][i], f"ray {i} (k={k}): device function differs from the batch call"
                else:
                    assert (rec == -7).all() and cnt[i] == 0x5A5A5A5A
    # a view of another kind: empty records and 0
    c = api.BVH8_CWBVH().Build(scene(300, 24))
    r = R.gpu_records(R.make_rays(np.zeros((1, 3), np.float32), np.array([[0, 0, 1]], np.float32), np.float32(5)))
    got, cnt = run_consumer(consumer, c.device_view(_lib.LAYOUT_CWBVH), r, np.array([3], np.uint32))
    assert got.view(np.uint32).tolist() == [[np.float32(5).view(np.uint32), 0, 0, ao.NO_PRIM]] * 3 and cnt[0] == 0
