"""tbvh_sphere_cast / tbvh_sphere_cast_occluded on the device, held bit for bit to the host restatement's brute force over every reference of
the tree the handle holds (tests/sweep_oracle.c, DESIGN.md §4.16): every builder, failed-split SBVHs, batch and indexed builds, uploaded
families and a DAG, a BVH_GPU upload, deep and one-leaf trees, golden and off-atrium scenes, refits, tbvh_optimize and a group replica; host
and device space, stream order, n = 0, every refusal, zero-length sweeps against tbvh_sphere_overlap, r = 0 against tbvh_intersect_device,
and the device functions from a caller's kernel (tests/sphere_cast_consumer.cu)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import portpy
from tinybvh_b200 import _lib, api, build, rays as R, scenes
from tests import closest_oracle as co, sweep_oracle as so, util
from tests.test_closest_point import family
from tests.test_closest_point_gpu import chain_tree, torch_f
from tests.test_sphere_cast import scene_queries

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NODE32 = portpy.NODE32


def device_query(obj, q, any_, stream=None):
    """the batch call in device space -> numpy records (cast) or words (occluded)"""
    import torch
    L = _lib.lib()
    n = q.shape[0]
    dq = torch_f(q)
    if any_:
        out = torch.zeros(max((n + 31) // 32, 1), dtype=torch.int32, device="cuda")
        _lib.check(L.tbvh_sphere_cast_occluded(obj.h, C.c_void_p(dq.data_ptr()), C.c_void_p(out.data_ptr()), n, _lib.DEVICE, stream))
    else:
        out = torch.zeros((n, 4), dtype=torch.float32, device="cuda")
        _lib.check(L.tbvh_sphere_cast(obj.h, C.c_void_p(dq.data_ptr()), C.c_void_p(out.data_ptr()), n, _lib.DEVICE, stream))
    torch.cuda.synchronize()
    o = out.cpu().numpy()
    return o.view(np.uint32) if any_ else o


def host_query(obj, q, any_):
    L = _lib.lib()
    q = np.ascontiguousarray(q, np.float32)
    n = q.shape[0]
    if any_:
        out = np.zeros(max((n + 31) // 32, 1), np.uint32)
        _lib.check(L.tbvh_sphere_cast_occluded(obj.h, q.ctypes.data, out.ctypes.data, n, _lib.HOST, None))
    else:
        out = np.zeros((n, 4), np.float32)
        _lib.check(L.tbvh_sphere_cast(obj.h, q.ctypes.data, out.ctypes.data, n, _lib.HOST, None))
    return out


def check_tree(obj, nodes, idx, v, q, label, host=False):
    """every record (16 bytes) and every bit of the device batch calls equal the brute force over (nodes, idx, v)"""
    want = so.brute(nodes, idx, v, q)
    wbits = so.brute(nodes, idx, v, q, any_=True)
    got = device_query(obj, q, False)
    bad = (got.view(np.uint32) != want.view(np.uint32)).any(1)
    assert not bad.any(), f"{label}: {int(bad.sum())} of {q.shape[0]} records differ, first {np.nonzero(bad)[0][:5]}: {got[bad][:2]} vs {want[bad][:2]}"
    gbits = device_query(obj, q, True)
    assert np.array_equal(gbits[: wbits.shape[0]], wbits), f"{label}: blocked bits differ"
    if host:
        assert np.array_equal(host_query(obj, q, False).view(np.uint32), want.view(np.uint32)), f"{label}: host space differs"
        assert np.array_equal(host_query(obj, q, True)[: wbits.shape[0]], wbits), f"{label}: host space bits differ"
    return got


def scene(n, seed=5):
    return scenes.procedural_scene(n, seed)


@pytest.mark.parametrize("builder", ["Build", "BuildAVX", "BuildHQ", "BuildPLOC"])
@pytest.mark.parametrize("ntris", [1, 9, 3000, 40000])
def test_builders(gpu, builder, ntris):
    v = scene(ntris, 3 + ntris % 5)
    e = getattr(api.BVH(), builder)(v)
    nodes, idx = e.download()
    q = scene_queries(v, np.random.default_rng(ntris), n=1000 if ntris < 40000 else 3000)
    check_tree(e, nodes, idx, v, q, f"{builder}-{ntris}", host=ntris == 3000)


@pytest.mark.parametrize("name", ["snapped20k_q4", "lattice10k_k3", "clusters"])
def test_hq_failed_splits(gpu, name):
    from tests.test_build_hq_shapes import fail_scene
    v = util.long_leaf_scene(name) if name == "clusters" else fail_scene(name)
    e = api.BVH().BuildHQ(v)
    nodes, idx = e.download()
    check_tree(e, nodes, idx, v, scene_queries(v, np.random.default_rng(1), n=800), f"BuildHQ-{name}")


def test_batch_and_indexed(gpu):
    meshes = [scene(n, 20 + n) for n in (5, 700, 4000)]
    for flavour in (_lib.BUILD_REFERENCE, _lib.BUILD_AVX, _lib.BUILD_PLOC, _lib.BUILD_HQ):
        objs = [api.BVH() for _ in meshes]
        api.build_batch(objs, meshes, flavour)
        for o, v in zip(objs, meshes):
            nodes, idx = o.download()
            check_tree(o, nodes, idx, v, scene_queries(v, np.random.default_rng(2), n=400), f"batch-{flavour}-{v.shape[0] // 3}")
    v = scene(3000, 8)
    uniq, inv = np.unique(v.reshape(-1, 4), axis=0, return_inverse=True)
    e = api.BVH()
    e.Build(uniq, indices=inv.astype(np.uint32).reshape(-1))
    nodes, idx = e.download()
    check_tree(e, nodes, idx, uniq[inv.reshape(-1)], scene_queries(v, np.random.default_rng(3), n=800), "indexed")


@pytest.mark.parametrize("fam", util.FAMILIES + ["shrunk", "dag"])
def test_uploaded_families(gpu, fam):
    v = scene(3000, 71)
    src = util.source_tree(v, "Build")
    nodes, idx = family(src, fam)
    e = api.BVH().upload(nodes, idx, v)
    check_tree(e, nodes, idx, v, scene_queries(v, np.random.default_rng(5), n=800), fam)


def test_bvh_gpu_upload_and_converted_objects(gpu):
    v = scene(3000, 9)
    o = util.oracle_tree(v, 1)
    g = api.BVH_GPU().upload(util.oracle_bvh_gpu_nodes(o), o.prim_idx, v)
    q = scene_queries(v, np.random.default_rng(6), n=800)
    check_tree(g, o.nodes, o.prim_idx, v, q, "BVH_GPU upload")
    for cls in (api.BVH_GPU, api.BVH8_CWBVH):
        b = cls().Build(v)
        nodes = np.zeros(b.info().used_nodes, NODE32)
        idx = np.zeros(b.info().idx_count, np.uint32)
        _lib.check(_lib.lib().tbvh_download_bvh(b.h, nodes.ctypes.data, idx.ctypes.data, _lib.HOST))
        check_tree(b, nodes, idx, v, q, cls.__name__)


def test_deep_and_one_leaf_trees(gpu):
    v = scene(400, 12)
    for m in (100, 255):
        nodes, idx = chain_tree(v, m)
        e = api.BVH().upload(nodes, idx, v[: 3 * m])
        assert e.info().max_depth == m - 1
        check_tree(e, nodes, idx, v[: 3 * m], scene_queries(v[: 3 * m], np.random.default_rng(m), n=400), f"chain-{m}", host=True)
    w = scene(40, 4)
    one = np.zeros(2, NODE32)
    tri = w.reshape(-1, 4)[:, :3]
    one[0] = (tri.min(0), 0, tri.max(0), 40)
    e = api.BVH().upload(one, np.arange(40, dtype=np.uint32), w)
    check_tree(e, one, np.arange(40, dtype=np.uint32), w, scene_queries(w, np.random.default_rng(4), n=300), "one leaf", host=True)


@pytest.mark.parametrize("name", ["flat_500", "coincident_610", "single_tri"])
def test_golden_scenes(gpu, name):
    g = np.load(os.path.join(REPO, "tests", "golden", f"{name}.npz"))
    v = g["verts"].astype(np.float32)
    nodes = np.ascontiguousarray(g["nodes"]).view(NODE32).reshape(-1)
    e = api.BVH().upload(nodes, g["prim_idx"], v)
    q = scene_queries(v, np.random.default_rng(10), n=800)
    check_tree(e, nodes, g["prim_idx"], v, q, name)
    b = api.BVH().Build(v)
    check_tree(b, *b.download(), v, q, name + "/Build")


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
        check_tree(e, *e.download(), v, scene_queries(v, np.random.default_rng(11), n=800), f"{variant}/{builder}")


def test_refit_and_optimize(gpu):
    v = scene(3000, 15)
    v2 = v.copy()
    v2[:, :3] += np.random.default_rng(1).normal(size=(v.shape[0], 3)).astype(np.float32) * 0.01
    q = scene_queries(v, np.random.default_rng(12), n=800)
    e = api.BVH().Build(v)
    e.Refit(v2)
    check_tree(e, *e.download(), v2, q, "refit")
    o = api.BVH().Build(v)
    o.optimize(4)
    check_tree(o, *o.download(), v, q, "optimize")


def test_group_replica(gpu, consumer):
    import torch
    v = scene(3000, 25)
    e = api.BVH().Build(v)
    q = scene_queries(v, np.random.default_rng(17), n=800)
    want = check_tree(e, *e.download(), v, q, "source")
    grp = api.Group([0])
    grp.replicate(e)
    rep = _lib.lib().tbvh_group_replica(grp.h, 0)
    assert rep and rep != e.h.value
    dq = torch_f(q)
    out = torch.zeros((q.shape[0], 4), dtype=torch.float32, device="cuda")
    _lib.check(_lib.lib().tbvh_sphere_cast(C.c_void_p(rep), C.c_void_p(dq.data_ptr()), C.c_void_p(out.data_ptr()), q.shape[0], _lib.DEVICE, None))
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy().view(np.uint32), want.view(np.uint32)), "replica handle"
    out.zero_()
    bits = torch.zeros((q.shape[0] + 31) // 32, dtype=torch.int32, device="cuda")
    assert consumer.sc_query(grp.device_view(0), dq.data_ptr(), out.data_ptr(), bits.data_ptr(), None, q.shape[0]) == 0
    assert np.array_equal(out.cpu().numpy().view(np.uint32), want.view(np.uint32)), "replica view"
    grp.close()


def test_large_batch(gpu):
    """2^18 sweeps against the restatement's pruned walk (equal to its brute force, tests/test_sphere_cast.py)"""
    v = scene(40000, 26)
    e = api.BVH().Build(v)
    nodes, idx = e.download()
    q = scene_queries(v, np.random.default_rng(18), n=1 << 17)
    assert np.array_equal(device_query(e, q, False).view(np.uint32), so.walk(nodes, idx, v, q).view(np.uint32))
    assert np.array_equal(device_query(e, q, True)[: (q.shape[0] + 31) // 32], so.walk(nodes, idx, v, q, any_=True))


def test_device_matches_host_and_api(gpu):
    import torch
    v = scene(5000, 16)
    e = api.BVH().Build(v)
    q = scene_queries(v, np.random.default_rng(13), n=2000)
    t, u, vv, prim = e.sphere_cast(q[:, :3], q[:, 4:7], q[:, 3], q[:, 7])
    tt, tu, tv, tp = e.sphere_cast(torch_f(q[:, :3]), torch_f(q[:, 4:7]), torch_f(q[:, 3]), torch_f(q[:, 7]))
    torch.cuda.synchronize()
    for a, b in ((t, tt), (u, tu), (vv, tv)):
        assert np.array_equal(a.view(np.uint32), b.cpu().numpy().view(np.uint32))
    assert np.array_equal(prim, tp.cpu().numpy().view(np.uint32))
    want = so.brute(*e.download(), v, q)
    assert np.array_equal(prim, so.record_prims(want)) and np.array_equal(t.view(np.uint32), want[:, 0].view(np.uint32))
    hits = e.sphere_cast_occluded(q[:, :3], q[:, 4:7], q[:, 3], q[:, 7])
    th = e.sphere_cast_occluded(torch_f(q[:, :3]), torch_f(q[:, 4:7]), torch_f(q[:, 3]), torch_f(q[:, 7]))
    assert np.array_equal(hits, th.cpu().numpy()) and np.array_equal(hits, prim != so.NO_PRIM)
    # (n, 4) rows and (n, 8) records, numpy and torch; the torch calls twice, so later calls reuse freed device memory
    variants = ((q[:, :4], q[:, 4:8]), (q,), (torch_f(q[:, :4]), torch_f(q[:, 4:8])), (torch_f(q),))
    for k, args in enumerate(variants + variants[2:]):
        r = e.sphere_cast(*args)
        got = r[3].cpu().numpy().view(np.uint32) if hasattr(r[3], "cpu") else r[3]
        assert np.array_equal(got, prim), k
        h = e.sphere_cast_occluded(*args)
        h = h.cpu().numpy() if hasattr(h, "cpu") else h
        bad = np.nonzero(h != hits)[0]
        assert bad.shape[0] == 0, (k, bad[:8], q[bad[:2]], got[bad[:8]], h[bad[:8]])
    # tmax defaults to inf
    r = e.sphere_cast(q[:, :3], q[:, 4:7], q[:, 3])
    qi = q.copy()
    qi[:, 7] = np.inf
    assert np.array_equal(r[3], so.record_prims(so.brute(*e.download(), v, qi)))
    with pytest.raises(api.TbvhError):
        e.sphere_cast(torch_f(q[:, :3]), torch_f(q[:, 4:7]))
    with pytest.raises(api.TbvhError):
        e.sphere_cast(q[:, :3], q[:10, 4:7], 1.0)


def test_stream_order_and_words(gpu):
    import torch
    v = scene(3000, 17)
    e = api.BVH().Build(v)
    q = scene_queries(v, np.random.default_rng(14), n=1000)
    want = so.brute(*e.download(), v, q)
    s = torch.cuda.Stream()
    src = torch_f(q)
    dq = torch.zeros_like(src)
    out = torch.zeros((q.shape[0], 4), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)   # the queries are written behind a long kernel on the caller's stream
        dq.copy_(src)
    _lib.check(_lib.lib().tbvh_sphere_cast(e.h, C.c_void_p(dq.data_ptr()), C.c_void_p(out.data_ptr()), q.shape[0], _lib.DEVICE, C.c_void_p(s.cuda_stream)))
    s.synchronize()
    assert np.array_equal(out.cpu().numpy().view(np.uint32), want.view(np.uint32)), "the query walked before the caller's stream wrote it"
    # torch inputs through the API, on a caller's stream
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)
        dq2 = src.clone()
    r = e.sphere_cast(dq2, stream=s)
    s.synchronize()
    assert np.array_equal(r[0].cpu().numpy().view(np.uint32), want[:, 0].view(np.uint32))
    for n in (0, 1, 31, 33, 100):
        if n:
            assert np.array_equal(device_query(e, q[:n], False).view(np.uint32), want[:n].view(np.uint32)), f"n = {n}"
        w = torch.full(((n + 31) // 32 + 1,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
        dq = torch_f(q[: max(n, 1)])
        _lib.check(_lib.lib().tbvh_sphere_cast_occluded(e.h, C.c_void_p(dq.data_ptr()), C.c_void_p(w.data_ptr()), n, _lib.DEVICE, None))
        got = w.cpu().numpy().view(np.uint32)
        assert got[-1] == 0x5A5A5A5A, "the word after (n+31)/32 was written"
        if n:
            bits = np.unpackbits(got[:-1].view(np.uint8), bitorder="little")
            assert not bits[n:].any(), "bits past n are set"
            assert np.array_equal(bits[:n].astype(bool), so.record_prims(want[:n]) != so.NO_PRIM)
    # n = 0 in host space writes nothing
    out0 = np.full((1, 4), 7, np.float32)
    _lib.check(_lib.lib().tbvh_sphere_cast(e.h, q.ctypes.data, out0.ctypes.data, 0, _lib.HOST, None))
    assert (out0 == 7).all()


def test_refusals(gpu):
    import torch
    L = _lib.lib()
    v = scene(300, 18)
    e = api.BVH().Build(v)
    q = torch_f(scene_queries(v, np.random.default_rng(1), n=64))
    out = torch.zeros((q.shape[0] + 1, 4), dtype=torch.float32, device="cuda")
    qp, op = C.c_void_p(q.data_ptr()), C.c_void_p(out.data_ptr())
    deep = chain_tree(scene(300, 19), 300)
    d = api.BVH().upload(deep[0], deep[1], scene(300, 19))
    c = api.BVH8_CWBVH().Build(v)
    only = api.BVH8_CWBVH().upload(*c.download())
    inst = np.zeros(2, api.BLAS_INSTANCE)
    inst["transform"] = np.eye(4, dtype=np.float32).reshape(-1)
    inst["mask"] = 0xFFFF
    t = api.TLAS()
    t.Build(inst, [e])
    for fn in (L.tbvh_sphere_cast, L.tbvh_sphere_cast_occluded):
        assert fn(None, qp, op, 4, _lib.DEVICE, None) == _lib.E_ARG
        assert fn(e.h, None, op, 4, _lib.DEVICE, None) == _lib.E_ARG
        assert fn(e.h, qp, None, 4, _lib.DEVICE, None) == _lib.E_ARG
        assert fn(e.h, qp, op, 4, 7, None) == _lib.E_ARG
        assert fn(e.h, C.c_void_p(q.data_ptr() + 4), op, 4, _lib.DEVICE, None) == _lib.E_ARG
        assert fn(e.h, C.c_void_p(q.data_ptr() + 8), op, 4, _lib.DEVICE, None) == _lib.E_ARG
        assert fn(e.h, qp, C.c_void_p(out.data_ptr() + 4), 4, _lib.DEVICE, None) == _lib.E_ARG
        assert fn(e.h, qp, op, 1 << 40, _lib.DEVICE, None) == _lib.E_ARG
        assert fn(t.h, C.c_void_p(q.data_ptr() + 4), op, 4, _lib.DEVICE, None) == _lib.E_ARG     # argument checks come first
        assert fn(t.h, qp, op, 4, _lib.DEVICE, None) == _lib.E_UNSUPPORTED
        assert fn(api.BVH().h, qp, op, 4, _lib.DEVICE, None) == _lib.E_STATE
        assert fn(only.h, qp, op, 4, _lib.DEVICE, None) == _lib.E_STATE
        assert fn(d.h, qp, op, 4, _lib.DEVICE, None) == _lib.E_LIMIT
        assert fn(e.h, qp, op, 0, _lib.DEVICE, None) == _lib.OK
    torch.cuda.synchronize()
    assert not out.any(), "a refused call wrote results"
    hq = np.zeros((4, 8), np.float32)
    ho = np.full((4, 4), 3, np.float32)
    assert L.tbvh_sphere_cast(t.h, hq.ctypes.data, ho.ctypes.data, 4, _lib.HOST, None) == _lib.E_UNSUPPORTED and (ho == 3).all()


def test_zero_length_against_sphere_overlap(gpu):
    """D = 0 on the device: t = 0 records exactly where tbvh_sphere_overlap sets the bit, except spheres touching within rounding"""
    v = scene(20000, 27)
    e = api.BVH().Build(v)
    q = scene_queries(v, np.random.default_rng(19), n=3000)[6:]
    q[:, 4:7] = 0
    got = device_query(e, q, False)
    cast = so.record_prims(got) != so.NO_PRIM
    assert (got[cast, 0] == 0).all()
    over = e.sphere_overlap(q[:, :4])
    diff = np.nonzero(cast != over)[0]
    assert cast.sum() > 100 and diff.shape[0] <= 0.001 * q.shape[0], diff
    d, _, _, _ = e.closest_point(q[diff, :3], np.inf)
    assert (np.abs(d - q[diff, 3]) <= 1e-6 * np.abs(v[:, :3]).max()).all()


def robust_rays(v, n, seed):
    """rays from inside the box of scene v with unit directions, and for each the fp64 verdict on every triangle
    (test_intersect_all_fp64.classify): robust rays have no ambiguous triangle and, when they hit, a nearest robust crossing more than
    twice the t bound before the next -> (rays, robust mask, expected prim or NO_PRIM, fp64 t, t bound)"""
    from tests.test_intersect_all_fp64 import classify
    rng = np.random.default_rng(seed)
    tri = v.reshape(-1, 3, 4)[:, :, :3].astype(np.float64)
    lo, hi = tri.reshape(-1, 3).min(0), tri.reshape(-1, 3).max(0)
    O = (lo + rng.uniform(0, 1, (n, 3)) * (hi - lo)).astype(np.float32)
    rays = R.make_rays(O, rng.normal(size=(n, 3)), np.float32(1e30))
    robust, want, t64, tb64 = np.zeros(n, bool), np.full(n, so.NO_PRIM, np.uint32), np.zeros(n), np.zeros(n)
    for i in range(0, n, 500):
        t, _, _, hit, miss, tb = classify(rays[i: i + 500], tri)
        clear = (hit | miss).all(1)
        tt = np.where(hit, t, np.inf)
        order = np.argsort(tt, axis=1)
        idx = np.arange(tt.shape[0])
        t1, t2 = tt[idx, order[:, 0]], tt[idx, order[:, 1]]
        b1 = tb[idx, order[:, 0]]
        with np.errstate(invalid="ignore"):
            sep = ~np.isfinite(t1) | (t2 - t1 > 2 * (b1 + tb[idx, order[:, 1]]))
        robust[i: i + 500] = clear & sep
        want[i: i + 500] = np.where(np.isfinite(t1), order[:, 0], so.NO_PRIM)
        t64[i: i + 500], tb64[i: i + 500] = t1, b1
    return rays, robust, want, t64, tb64


def test_zero_radius_against_intersect(gpu):
    """r = 0 on robust rays (every triangle a robust crossing or a robust miss in fp64, the nearest crossing clear of the next): the sweep
    and tbvh_intersect_device agree exactly on whether the ray hits and on the triangle, the sweep's t lies within the fp64 t bound of the
    crossing, and the ray's within twice that of the sweep's"""
    import torch
    v = scene(2000, 28)
    e = api.BVH().Build(v)
    n = 8000
    rays, robust, want, t64, tb = robust_rays(v, n, 20)
    assert robust.mean() > 0.9 and (want[robust] != so.NO_PRIM).mean() > 0.3
    g = R.gpu_records(rays)
    dr = torch.from_numpy(g.view(np.uint8).reshape(n, 64).copy()).cuda()
    e.Intersect(dr)
    torch.cuda.synchronize()
    hit = dr.cpu().numpy().reshape(-1).view(R.GPU_RAY_DTYPE)
    got = device_query(e, so.queries(g["O"], g["D"], 0.0, np.inf), False)
    prim = so.record_prims(got)
    hp = np.where(hit["t"] < 1e30, hit["prim"], so.NO_PRIM).astype(np.uint32)
    assert np.array_equal(prim[robust], want[robust]), "the sweep's triangle differs from the fp64 crossing"
    assert np.array_equal(hp[robust], want[robust]), "the ray's triangle differs from the fp64 crossing"
    h = robust & (want != so.NO_PRIM)
    assert (np.abs(got[h, 0] - t64[h]) <= tb[h]).all(), "the sweep's t is outside the fp64 bound"
    # Moeller-Trumbore's own t may stray up to about 1.2 bounds (measured on the host walk of this scene): the two within 2
    assert (np.abs(got[h, 0] - hit["t"][h]) <= 2 * tb[h]).all()


@pytest.fixture(scope="module")
def consumer(gpu, tmp_path_factory):
    nvcc = build.nvcc_path()
    so_path = str(tmp_path_factory.mktemp("sweep_consumer") / "consumer.so")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I" + os.path.join(REPO, "include"),
                        "-Xcompiler", "-fPIC", "-shared", "-Xptxas", "-v", os.path.join(REPO, "tests", "sphere_cast_consumer.cu"), "-o", so_path],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    L = C.CDLL(so_path)
    L.sc_query.argtypes = [_lib.DeviceView, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]
    return L


def test_device_functions(gpu, consumer):
    import torch
    for m, v in ((None, scene(3000, 22)), (150, scene(400, 23))):
        if m:
            nodes, idx = chain_tree(v, m)
            v = v[: 3 * m]
            e = api.BVH().upload(nodes, idx, v)
        else:
            e = api.BVH().Build(v)
        q = scene_queries(v, np.random.default_rng(16), n=800)
        want = device_query(e, q, False)
        wbits = device_query(e, q, True)
        n = q.shape[0]
        sel = np.random.default_rng(3).integers(0, 1 << 32, (n + 31) // 32, dtype=np.uint64).astype(np.uint32)
        for s in (None, sel):
            dq = torch_f(q)
            out = torch.full((n, 4), -7.0, dtype=torch.float32, device="cuda")
            bits = torch.zeros((n + 31) // 32, dtype=torch.int32, device="cuda")
            ds = torch.from_numpy(s.view(np.int32)).cuda() if s is not None else None
            assert consumer.sc_query(e.device_view(), dq.data_ptr(), out.data_ptr(), bits.data_ptr(), ds.data_ptr() if ds is not None else None, n) == 0
            got, gb = out.cpu().numpy(), bits.cpu().numpy().view(np.uint32)
            mask = np.ones(n, bool) if s is None else np.unpackbits(s.view(np.uint8), bitorder="little")[:n].astype(bool)
            assert np.array_equal(got[mask].view(np.uint32), want[mask].view(np.uint32)), "device function differs from the batch call"
            assert (got[~mask] == -7).all()
            wb = np.unpackbits(wbits.view(np.uint8), bitorder="little")[:n].astype(bool) & mask
            assert np.array_equal(np.unpackbits(gb.view(np.uint8), bitorder="little")[:n].astype(bool), wb)
    # a view of another kind: the miss record and false
    c = api.BVH8_CWBVH().Build(scene(300, 24))
    dq = torch_f(np.array([[0, 0, 0, 1, 1, 0, 0, 5]], np.float32))
    out = torch.zeros((1, 4), dtype=torch.float32, device="cuda")
    bits = torch.zeros(1, dtype=torch.int32, device="cuda")
    assert consumer.sc_query(c.device_view(_lib.LAYOUT_CWBVH), dq.data_ptr(), out.data_ptr(), bits.data_ptr(), None, 1) == 0
    assert out.cpu().numpy().view(np.uint32).tolist() == [[np.float32(5).view(np.uint32), 0, 0, so.NO_PRIM]] and int(bits[0]) == 0
