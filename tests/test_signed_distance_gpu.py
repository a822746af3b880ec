"""tbvh_signed_distance on the device, held bit for bit to the host restatement (tests/sdf_oracle.c, DESIGN.md §4.10) and to
tbvh_closest_point's records on the same queries: every builder, batch and indexed builds, uploaded families, a BVH_GPU upload, a deep
tree, golden scenes (open surfaces: bits only, no claim about the sign), tables prepared again after refits and tbvh_optimize, a group
replica, a 65,536-triangle fan, a 1 M-triangle closed mesh, host and device space, stream order, every refusal and launch counts."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import portpy
from tinybvh_b200 import _lib, api, scenes
from tests import closest_oracle as co, sdf_oracle as so, util
from tests.test_closest_point import family, queries_for
from tests.test_closest_point_gpu import chain_tree, torch_f
from tests.test_signed_distance import cone, icosphere, qrows, sample_queries, soup, star, torus, winding

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NODE32 = portpy.NODE32


def sd_device(h, q, fn="tbvh_signed_distance", stream=None):
    import torch
    dq = torch_f(q)
    out = torch.zeros((q.shape[0], 4), dtype=torch.float32, device="cuda")
    _lib.check(getattr(_lib.lib(), fn)(h, C.c_void_p(dq.data_ptr()), C.c_void_p(out.data_ptr()), q.shape[0], _lib.DEVICE, stream))
    torch.cuda.synchronize()
    return out.cpu().numpy()


def sd_host(h, q):
    q = np.ascontiguousarray(q, np.float32)
    out = np.zeros((q.shape[0], 4), np.float32)
    _lib.check(_lib.lib().tbvh_signed_distance(h, q.ctypes.data, out.ctypes.data, q.shape[0], _lib.HOST, None))
    return out


def same_bits(got, want, label):
    bad = (got.view(np.uint32) != want.view(np.uint32)).any(1)
    assert not bad.any(), f"{label}: {int(bad.sum())} of {got.shape[0]} records differ, first {np.nonzero(bad)[0][:5]}: {got[bad][:2]} vs {want[bad][:2]}"


def check_tree(obj, nodes, idx, v, q, label, host=False, walk=False, h=None):
    """prepare, then every signed record equals the restatement's and, but for the sign bit, tbvh_closest_point's"""
    h = obj.h if h is None else h
    _lib.check(_lib.lib().tbvh_signed_distance_prepare(h))
    got = sd_device(h, q)
    same_bits(got, so.brute(nodes, idx, v, q, walk=walk), label)
    cp = sd_device(h, q, "tbvh_closest_point")
    g = got.view(np.uint32).copy()
    g[g[:, 3] != co.NO_PRIM, 0] &= 0x7FFFFFFF   # a miss record is the closest-point one, r_max's sign included
    assert np.array_equal(g, cp.view(np.uint32)), f"{label}: |sd|, u, v, prim differ from tbvh_closest_point"
    if host:
        same_bits(sd_host(h, q), got, label + "/host")
    return got


def closed_meshes():
    return {"icosphere": icosphere(3), "torus": torus(), "star": star()}


def scene(n, seed=5):
    return scenes.procedural_scene(n, seed)


@pytest.mark.parametrize("builder", ["Build", "BuildAVX", "BuildHQ", "BuildPLOC"])
def test_builders(gpu, builder):
    rng = np.random.default_rng(1)
    for name, (V, F) in closed_meshes().items():
        v = soup(V, F)
        e = getattr(api.BVH(), builder)(v)
        q = qrows(sample_queries(V, F, rng, n=800))
        got = check_tree(e, *e.download(), v, q, f"{builder}/{name}", host=name == "torus")
        far = np.abs(got[:, 0]) > 1e-3 * np.ptp(V, 0).max()
        inside = np.abs(winding(V, F, q[:, :3].astype(np.float64))) > 0.5
        assert np.array_equal(np.signbit(got[far, 0]), inside[far]), f"{builder}/{name}: signs against the winding number"
    v = scene(3000, 3)
    e = getattr(api.BVH(), builder)(v)
    check_tree(e, *e.download(), v, queries_for(v, np.random.default_rng(2), n=2000), f"{builder}/soup")


@pytest.mark.parametrize("name", ["snapped20k_q4", "clusters"])
def test_hq_failed_splits(gpu, name):
    from tests.test_build_hq_shapes import fail_scene
    v = util.long_leaf_scene(name) if name == "clusters" else fail_scene(name)
    e = api.BVH().BuildHQ(v)
    check_tree(e, *e.download(), v, queries_for(v, np.random.default_rng(1), n=1500), f"BuildHQ-{name}")


def test_batch_and_indexed(gpu):
    meshes = [soup(*icosphere(2)), soup(*torus()), scene(700, 21)]
    for flavour in (_lib.BUILD_REFERENCE, _lib.BUILD_AVX, _lib.BUILD_PLOC, _lib.BUILD_HQ):
        objs = [api.BVH() for _ in meshes]
        api.build_batch(objs, meshes, flavour)
        for o, v in zip(objs, meshes):
            check_tree(o, *o.download(), v, queries_for(v, np.random.default_rng(2), n=700), f"batch-{flavour}-{v.shape[0] // 3}")
    # an indexed build and its V[I] soup: the same records
    V, F = torus()
    verts = np.zeros((V.shape[0], 4), np.float32)
    verts[:, :3] = V
    e = api.BVH()
    e.Build(verts, indices=F.astype(np.uint32).reshape(-1))
    s = api.BVH().Build(soup(V, F))
    q = qrows(sample_queries(V, F, np.random.default_rng(3), n=800))
    a = check_tree(e, *e.download(), soup(V, F), q, "indexed")
    b = check_tree(s, *s.download(), soup(V, F), q, "soup")
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("fam", util.FAMILIES + ["dag"])
def test_uploaded_families(gpu, fam):
    v = soup(*icosphere(3))
    src = util.source_tree(v, "Build")
    nodes, idx = family(src, fam)
    e = api.BVH().upload(nodes, idx, v)
    check_tree(e, nodes, idx, v, queries_for(v, np.random.default_rng(5), n=1500), fam)


def test_bvh_gpu_upload_and_deep_tree(gpu):
    v = soup(*torus())
    o = util.oracle_tree(v, 1)
    g = api.BVH_GPU().upload(util.oracle_bvh_gpu_nodes(o), o.prim_idx, v)
    check_tree(g, o.nodes, o.prim_idx, v, queries_for(v, np.random.default_rng(6), n=1500), "BVH_GPU upload")
    src = util.source_tree(v, "Build")
    deep = util.reinserted(src, 3, 50, grow_to=100)
    e = api.BVH().upload(deep[0], deep[1], v)
    assert e.info().max_depth >= 64
    check_tree(e, deep[0], deep[1], v, queries_for(v, np.random.default_rng(8), n=1500), "deep", host=True)
    w = scene(400, 12)
    nodes, idx = chain_tree(w, 255)
    c = api.BVH().upload(nodes, idx, w[: 3 * 255])
    check_tree(c, nodes, idx, w[: 3 * 255], queries_for(w[: 3 * 255], np.random.default_rng(9), n=500), "chain-255")


@pytest.mark.parametrize("name", ["flat_500", "coincident_610", "single_tri"])
def test_golden_scenes(gpu, name):
    """open surfaces: every record held bit for bit, no claim about the sign"""
    g = np.load(os.path.join(REPO, "tests", "golden", f"{name}.npz"))
    v = g["verts"].astype(np.float32)
    nodes = np.ascontiguousarray(g["nodes"]).view(NODE32).reshape(-1)
    e = api.BVH().upload(nodes, g["prim_idx"], v)
    check_tree(e, nodes, g["prim_idx"], v, queries_for(v, np.random.default_rng(10), n=1500), name)


def refused_stale(h):
    q = torch_f(np.zeros((4, 4), np.float32))
    return _lib.lib().tbvh_signed_distance(h, C.c_void_p(q.data_ptr()), C.c_void_p(q.data_ptr()), 4, _lib.DEVICE, None) == _lib.E_STATE


def test_prepared_again_after_refit_and_optimize(gpu):
    V, F = icosphere(3)
    v = soup(V, F)
    v2 = v.copy()
    v2[:, :3] *= np.float32(1.25)
    q = qrows(sample_queries(V * 1.25, F, np.random.default_rng(12), n=800))
    e = api.BVH().Build(v)
    e.prepare_signed_distance()
    e.Refit(v2)
    assert refused_stale(e.h)
    check_tree(e, *e.download(), v2, q, "refit")
    g = api.BVH_GPU().Build(v)
    _lib.check(_lib.lib().tbvh_signed_distance_prepare(g.h))
    _lib.check(_lib.lib().tbvh_refit_layouts(g.h, C.c_void_p(np.ascontiguousarray(v2).ctypes.data), 16, v.shape[0] // 3, _lib.HOST))
    assert refused_stale(g.h)
    nodes = np.zeros(g.info().used_nodes, NODE32)
    idx = np.zeros(g.info().idx_count, np.uint32)
    _lib.check(_lib.lib().tbvh_download_bvh(g.h, nodes.ctypes.data, idx.ctypes.data, _lib.HOST))
    check_tree(g, nodes, idx, v2, q, "refit_layouts")
    o = api.BVH().Build(soup(*torus()))
    o.prepare_signed_distance()
    rounds = C.c_uint32()
    _lib.check(_lib.lib().tbvh_optimize(o.h, 4, C.c_float(1.0), C.c_float(1.0), C.byref(rounds), None))
    if rounds.value:
        assert refused_stale(o.h)
    check_tree(o, *o.download(), soup(*torus()), qrows(sample_queries(*torus(), np.random.default_rng(13), n=800)), "optimize")


def test_group_replica(gpu):
    v = soup(*icosphere(3))
    e = api.BVH().Build(v)
    q = queries_for(v, np.random.default_rng(17), n=1500)
    want = check_tree(e, *e.download(), v, q, "source")
    grp = api.Group([0])
    grp.replicate(e)
    rep = _lib.lib().tbvh_group_replica(grp.h, 0)
    assert rep and rep != e.h.value
    assert refused_stale(C.c_void_p(rep)), "a replica holds no table until prepared"
    got = check_tree(None, *e.download(), v, q, "replica", h=C.c_void_p(rep))
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    grp.close()


def test_cone_fan(gpu):
    """65,536 triangles around one vertex: the apex's run is summed by one thread; signs along the axis"""
    V, F = cone()
    v = soup(V, F)
    e = api.BVH().Build(v)
    rng = np.random.default_rng(4)
    axis = np.c_[np.zeros(64), np.zeros(64), 2.0 + np.r_[rng.uniform(0.01, 0.3, 32), -rng.uniform(0.05, 1.5, 32)]]
    q = qrows(np.concatenate([axis, rng.uniform(-1.3, 1.3, (400, 3)) + [0, 0, 1]]))
    got = check_tree(e, *e.download(), v, q, "cone", walk=True)
    assert np.array_equal(np.signbit(got[:64, 0]), np.r_[np.zeros(32, bool), np.ones(32, bool)])


def big_torus(nu=1024, nv=512, R=1.0, r=0.3):
    i, j = np.meshgrid(np.arange(nu), np.arange(nv), indexing="ij")
    a, b = 2 * np.pi * i.reshape(-1) / nu, 2 * np.pi * j.reshape(-1) / nv
    V = np.stack([(R + r * np.cos(b)) * np.cos(a), (R + r * np.cos(b)) * np.sin(a), r * np.sin(b)], 1)
    idx = lambda x, y: (x % nu) * nv + (y % nv)
    i, j = i.reshape(-1), j.reshape(-1)
    A, B, Cc, D = idx(i, j), idx(i + 1, j), idx(i + 1, j + 1), idx(i, j + 1)
    F = np.concatenate([np.c_[A, B, Cc], np.c_[A, Cc, D]])
    return V, F


def test_million_triangle_mesh(gpu):
    V, F = big_torus()
    assert F.shape[0] >= 1 << 20
    v = soup(V, F)
    e = api.BVH().Build(v)
    rng = np.random.default_rng(19)
    k = rng.integers(0, F.shape[0], 4000)
    P = V[F[k]].mean(1) + rng.normal(size=(4000, 3)) * 0.01
    q = qrows(np.concatenate([P, rng.uniform(-1.4, 1.4, (4000, 3)) * [1, 1, 0.3]]))
    got = check_tree(e, *e.download(), v, q, "1M torus", walk=True)
    rho = np.hypot(np.hypot(q[:, 0], q[:, 1]) - 1.0, q[:, 2])       # distance to the core circle: inside below r = 0.3
    far = np.abs(got[:, 0]) > 1e-3
    assert np.array_equal(np.signbit(got[far, 0]), (rho < 0.3)[far])


def test_python_api_and_stream_order(gpu):
    import torch
    V, F = star()
    v = soup(V, F)
    e = api.BVH().Build(v)
    e.prepare_signed_distance()
    q = qrows(sample_queries(V, F, np.random.default_rng(14), n=600))
    want = so.brute(*e.download(), v, q)
    sd, u, vv, prim = e.signed_distance(q[:, :3], np.inf)
    same_bits(np.c_[sd, u, vv, prim.view(np.float32)], want, "numpy")
    t = e.signed_distance(torch_f(q))
    torch.cuda.synchronize()
    same_bits(np.stack([x.cpu().numpy().view(np.float32) for x in t], 1), want, "torch")
    with pytest.raises(api.TbvhError):
        e.signed_distance(q, np.inf)
    s = torch.cuda.Stream()
    src = torch_f(q)
    dq = torch.zeros_like(src)
    out = torch.zeros((q.shape[0], 4), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)   # the queries are written behind a long kernel on the caller's stream
        dq.copy_(src)
    _lib.check(_lib.lib().tbvh_signed_distance(e.h, C.c_void_p(dq.data_ptr()), C.c_void_p(out.data_ptr()), q.shape[0], _lib.DEVICE, C.c_void_p(s.cuda_stream)))
    s.synchronize()
    same_bits(out.cpu().numpy(), want, "caller's stream")
    for n in (1, 31, 33):
        same_bits(sd_device(e.h, q[:n]), want[:n], f"n = {n}")
    # misses, NaN coordinates and bad radii: the closest-point miss record
    bad = np.array([[0, 0, 0, 0.01], [np.nan, 0, 0, 1], [0, 0, 0, -1], [5, 5, 5, 0.5]], np.float32)
    assert np.array_equal(sd_device(e.h, bad).view(np.uint32), sd_device(e.h, bad, "tbvh_closest_point").view(np.uint32))
    assert (sd_device(e.h, bad).view(np.uint32)[:, 3] == co.NO_PRIM).all()


def test_refusals(gpu):
    import torch
    L = _lib.lib()
    V, F = icosphere(1)
    v = soup(V, F)
    e = api.BVH().Build(v)
    q = torch_f(qrows(V[:64] * 1.1))
    out = torch.zeros((q.shape[0] + 1, 4), dtype=torch.float32, device="cuda")
    qp, op = C.c_void_p(q.data_ptr()), C.c_void_p(out.data_ptr())
    n0 = api.launch_count()
    fn = L.tbvh_signed_distance
    # prepare
    assert L.tbvh_signed_distance_prepare(None) == _lib.E_ARG
    assert L.tbvh_signed_distance_prepare(api.BVH().h) == _lib.E_STATE
    c = api.BVH8_CWBVH().Build(v)
    only = api.BVH8_CWBVH().upload(*c.download())
    assert L.tbvh_signed_distance_prepare(only.h) == _lib.E_STATE
    # the query: tbvh_closest_point's refusals in order, then the table
    assert fn(None, qp, op, 4, _lib.DEVICE, None) == _lib.E_ARG
    assert fn(e.h, None, op, 4, _lib.DEVICE, None) == _lib.E_ARG
    assert fn(e.h, qp, None, 4, _lib.DEVICE, None) == _lib.E_ARG
    assert fn(e.h, qp, op, 4, 7, None) == _lib.E_ARG
    assert fn(e.h, C.c_void_p(q.data_ptr() + 4), op, 4, _lib.DEVICE, None) == _lib.E_ARG
    assert fn(e.h, qp, C.c_void_p(out.data_ptr() + 4), 4, _lib.DEVICE, None) == _lib.E_ARG
    assert fn(e.h, qp, op, 1 << 40, _lib.DEVICE, None) == _lib.E_ARG
    assert fn(api.BVH().h, qp, op, 4, _lib.DEVICE, None) == _lib.E_STATE
    assert fn(only.h, qp, op, 4, _lib.DEVICE, None) == _lib.E_STATE
    w = scene(300, 19)
    deep = chain_tree(w, 300)
    d = api.BVH().upload(deep[0], deep[1], w)
    assert fn(d.h, qp, op, 4, _lib.DEVICE, None) == _lib.E_LIMIT
    assert fn(e.h, qp, op, 4, _lib.DEVICE, None) == _lib.E_STATE, "a query before prepare"
    assert fn(e.h, qp, op, 0, _lib.DEVICE, None) == _lib.E_STATE
    inst = np.zeros(2, api.BLAS_INSTANCE)
    inst["transform"] = np.eye(4, dtype=np.float32).reshape(-1)
    inst["mask"] = 0xFFFF
    t = api.TLAS()
    t.Build(inst, [e])
    n1 = api.launch_count()
    assert fn(t.h, qp, op, 4, _lib.DEVICE, None) == _lib.E_UNSUPPORTED
    assert L.tbvh_signed_distance_prepare(t.h) == _lib.E_UNSUPPORTED
    assert api.launch_count() == n1, "a refusal launched work"
    torch.cuda.synchronize()
    assert not out.any(), "a refused call wrote results"
    # every call that changes the tree or its vertices makes the table stale
    stampers = {
        "Build": lambda: e.Build(v),
        "upload": lambda: e.upload(*e.download(), v),
        "refit": lambda: e.Refit(v),
        "refit_layouts": lambda: _lib.check(L.tbvh_refit_layouts(e.h, C.c_void_p(np.ascontiguousarray(v).ctypes.data), 16, v.shape[0] // 3, _lib.HOST)),
        "BuildPLOC": lambda: e.BuildPLOC(v),
    }
    for name, call in stampers.items():
        _lib.check(L.tbvh_signed_distance_prepare(e.h))
        assert fn(e.h, qp, op, 4, _lib.DEVICE, None) == _lib.OK, name
        call()
        n1 = api.launch_count()
        assert fn(e.h, qp, op, 4, _lib.DEVICE, None) == _lib.E_STATE, f"stale after {name}"
        assert api.launch_count() == n1
    assert api.launch_count() > n0


def test_conversions_keep_the_table(gpu):
    """A conversion leaves the tree and its vertices as they were, so a prepared table stays valid through it: converting a handle that
    already holds a CWBVH again (single and batched), converting to BVH_GPU, and uploading a CWBVH over it.  Every query after them gives
    the records it gave before."""
    V, F = icosphere(3)
    v = soup(V, F)
    e = api.BVH8_CWBVH().Build(v)
    other = api.BVH().Build(scene(500, 23))
    q = qrows(sample_queries(V, F, np.random.default_rng(24), n=500))
    L = _lib.lib()
    _lib.check(L.tbvh_signed_distance_prepare(e.h))
    before = sd_device(e.h, q)
    same_bits(before, so.brute(*api.BVH.download(e), v, q), "prepared")
    data, tris = e.download()
    calls = {
        "convert CWBVH again": lambda: L.tbvh_convert(e.h, api.LAYOUT_CWBVH),
        "convert_batch": lambda: L.tbvh_convert_batch((C.c_void_p * 2)(e.h.value, other.h.value), 2, api.LAYOUT_CWBVH),
        "convert BVH_GPU": lambda: L.tbvh_convert(e.h, api.LAYOUT_BVH_GPU),
        "upload_cwbvh": lambda: L.tbvh_upload_cwbvh(e.h, C.c_void_p(data.ctypes.data), data.shape[0], C.c_void_p(tris.ctypes.data), tris.shape[0] // 3, _lib.HOST),
    }
    for name, call in calls.items():
        assert call() == _lib.OK, name
        same_bits(sd_device(e.h, q), before, f"after {name}")
