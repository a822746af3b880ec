"""tbvh_closest_point / tbvh_sphere_overlap on the device, held bit for bit to the host restatement's brute force over every reference of
the tree the handle holds (tests/closest_oracle.c, DESIGN.md §4.9): every builder, batch and indexed builds, uploaded families, a BVH_GPU
upload, deep and one-leaf trees, golden and off-atrium scenes, refits, tbvh_optimize and group replicas; host and device space, stream
order, the bit words, every refusal, fp64 distances, and the device functions from a caller's kernel (tests/closest_point_consumer.cu)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import portpy
from tinybvh_b200 import _lib, api, build, scenes
from tests import closest_oracle as co, util
from tests.test_closest_point import family, fp64_closest, queries_for

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NODE32 = portpy.NODE32


def torch_f(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def device_query(obj, q, any_):
    """the batch call in device space -> numpy records (closest) or words (any)"""
    import torch
    L = _lib.lib()
    n = q.shape[0]
    dq = torch_f(q)
    if any_:
        out = torch.zeros(max((n + 31) // 32, 1), dtype=torch.int32, device="cuda")
        _lib.check(L.tbvh_sphere_overlap(obj.h, C.c_void_p(dq.data_ptr()), C.c_void_p(out.data_ptr()), n, _lib.DEVICE, None))
    else:
        out = torch.zeros((n, 4), dtype=torch.float32, device="cuda")
        _lib.check(L.tbvh_closest_point(obj.h, C.c_void_p(dq.data_ptr()), C.c_void_p(out.data_ptr()), n, _lib.DEVICE, None))
    torch.cuda.synchronize()
    o = out.cpu().numpy()
    return o.view(np.uint32) if any_ else o


def host_query(obj, q, any_):
    L = _lib.lib()
    q = np.ascontiguousarray(q, np.float32)
    n = q.shape[0]
    if any_:
        out = np.zeros(max((n + 31) // 32, 1), np.uint32)
        _lib.check(L.tbvh_sphere_overlap(obj.h, q.ctypes.data, out.ctypes.data, n, _lib.HOST, None))
    else:
        out = np.zeros((n, 4), np.float32)
        _lib.check(L.tbvh_closest_point(obj.h, q.ctypes.data, out.ctypes.data, n, _lib.HOST, None))
    return out


def check_tree(obj, nodes, idx, v, q, label, host=False):
    """every record (16 bytes) and every bit of the device batch calls equal the brute force over (nodes, idx, v)"""
    want = co.brute(nodes, idx, v, q)
    wbits = co.brute(nodes, idx, v, q, any_=True)
    got = device_query(obj, q, False)
    bad = (got.view(np.uint32) != want.view(np.uint32)).any(1)
    assert not bad.any(), f"{label}: {int(bad.sum())} of {q.shape[0]} records differ, first {np.nonzero(bad)[0][:5]}: {got[bad][:2]} vs {want[bad][:2]}"
    gbits = device_query(obj, q, True)
    assert np.array_equal(gbits[: wbits.shape[0]], wbits), f"{label}: overlap bits differ"
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
    q = queries_for(v, np.random.default_rng(ntris), n=2000 if ntris < 40000 else 6000)
    check_tree(e, nodes, idx, v, q, f"{builder}-{ntris}", host=ntris == 3000)


@pytest.mark.parametrize("name", ["snapped20k_q4", "lattice10k_k3", "clusters"])
def test_hq_failed_splits(gpu, name):
    """BuildHQ where spatial splits fail (leaves made from stale idxTmp words) and over clusters of identical triangles"""
    from tests.test_build_hq_shapes import fail_scene
    v = util.long_leaf_scene(name) if name == "clusters" else fail_scene(name)
    e = api.BVH().BuildHQ(v)
    nodes, idx = e.download()
    check_tree(e, nodes, idx, v, queries_for(v, np.random.default_rng(1), n=1500), f"BuildHQ-{name}")


def test_batch_and_indexed(gpu):
    meshes = [scene(n, 20 + n) for n in (5, 700, 4000)]
    for flavour in (_lib.BUILD_REFERENCE, _lib.BUILD_AVX, _lib.BUILD_PLOC, _lib.BUILD_HQ):
        objs = [api.BVH() for _ in meshes]
        api.build_batch(objs, meshes, flavour)
        for o, v in zip(objs, meshes):
            nodes, idx = o.download()
            check_tree(o, nodes, idx, v, queries_for(v, np.random.default_rng(2), n=700), f"batch-{flavour}-{v.shape[0] // 3}")
    v = scene(3000, 8)
    tri = v.reshape(-1, 4)
    uniq, inv = np.unique(tri, axis=0, return_inverse=True)
    e = api.BVH()
    e.Build(uniq, indices=inv.astype(np.uint32).reshape(-1))
    nodes, idx = e.download()
    check_tree(e, nodes, idx, uniq[inv.reshape(-1)], queries_for(v, np.random.default_rng(3), n=1500), "indexed")


@pytest.mark.parametrize("fam", util.FAMILIES + ["shrunk", "dag"])
def test_uploaded_families(gpu, fam):
    """util's families, a tree whose child boxes stick out of their parents, and a DAG (a slot reached on two paths, whose references
    are worth their least value over the paths)"""
    v = scene(3000, 71)
    src = util.source_tree(v, "Build")
    nodes, idx = family(src, fam)
    e = api.BVH().upload(nodes, idx, v)
    check_tree(e, nodes, idx, v, queries_for(v, np.random.default_rng(5), n=2000), fam)


def test_bvh_gpu_upload_and_converted_objects(gpu):
    v = scene(3000, 9)
    o = util.oracle_tree(v, 1)
    g = api.BVH_GPU().upload(util.oracle_bvh_gpu_nodes(o), o.prim_idx, v)
    q = queries_for(v, np.random.default_rng(6), n=2000)
    check_tree(g, o.nodes, o.prim_idx, v, q, "BVH_GPU upload")
    for cls in (api.BVH_GPU, api.BVH8_CWBVH):
        b = cls().Build(v)
        nodes = np.zeros(b.info().used_nodes, NODE32)
        idx = np.zeros(b.info().idx_count, np.uint32)
        _lib.check(_lib.lib().tbvh_download_bvh(b.h, nodes.ctypes.data, idx.ctypes.data, _lib.HOST))
        check_tree(b, nodes, idx, v, q, cls.__name__)


def chain_tree(v, m):
    """a caterpillar: interior node k's children are a one-triangle leaf and the next interior node; depth m - 1"""
    tri = v.reshape(-1, 3, 4)[:m, :, :3]
    nodes = np.zeros(2 * m, NODE32)
    lo, hi = tri.min(1), tri.max(1)
    for k in range(m - 1):
        node = 0 if k == 0 else 2 * k + 1
        leaf = 2 * k + 2
        nodes[leaf] = (lo[k], k, hi[k], 1)
        nodes[node]["leftFirst"] = leaf
    nodes[2 * m - 1] = (lo[m - 1], m - 1, hi[m - 1], 1)
    for k in range(m - 2, -1, -1):
        node, c = (0 if k == 0 else 2 * k + 1), 2 * k + 2
        nodes[node]["aabbMin"] = np.minimum(nodes[c]["aabbMin"], nodes[c + 1]["aabbMin"])
        nodes[node]["aabbMax"] = np.maximum(nodes[c]["aabbMax"], nodes[c + 1]["aabbMax"])
    return nodes, np.arange(m, dtype=np.uint32)


def test_deep_and_one_leaf_trees(gpu):
    v = scene(400, 12)
    for m in (100, 255):
        nodes, idx = chain_tree(v, m)
        e = api.BVH().upload(nodes, idx, v[: 3 * m])
        assert e.info().max_depth == m - 1
        check_tree(e, nodes, idx, v[: 3 * m], queries_for(v[: 3 * m], np.random.default_rng(m), n=700), f"chain-{m}", host=True)
    src = util.source_tree(scene(3000, 71), "Build")
    deep = util.reinserted(src, 3, 50, grow_to=100)
    e = api.BVH().upload(deep[0], deep[1], scene(3000, 71))
    assert e.info().max_depth >= 64
    check_tree(e, deep[0], deep[1], scene(3000, 71), queries_for(scene(3000, 71), np.random.default_rng(8), n=1500), "reinserted-deep")
    w = scene(40, 4)
    one = np.zeros(2, NODE32)
    tri = w.reshape(-1, 4)[:, :3]
    one[0] = (tri.min(0), 0, tri.max(0), 40)
    e = api.BVH().upload(one, np.arange(40, dtype=np.uint32), w)
    check_tree(e, one, np.arange(40, dtype=np.uint32), w, queries_for(w, np.random.default_rng(4), n=500), "one leaf", host=True)


@pytest.mark.parametrize("name", ["flat_500", "coincident_610", "single_tri"])
def test_golden_scenes(gpu, name):
    g = np.load(os.path.join(REPO, "tests", "golden", f"{name}.npz"))
    v = g["verts"].astype(np.float32)
    nodes = np.ascontiguousarray(g["nodes"]).view(NODE32).reshape(-1)
    e = api.BVH().upload(nodes, g["prim_idx"], v)
    q = queries_for(v, np.random.default_rng(10), n=1500)
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
        check_tree(e, *e.download(), v, queries_for(v, np.random.default_rng(11), n=1500), f"{variant}/{builder}")


def test_on_planes_vertices_and_edges(gpu):
    """points exactly on vertices, edge midpoints and leaf-box planes"""
    v = scene(3000, 14)
    e = api.BVH().Build(v)
    nodes, idx = e.download()
    tri = v.reshape(-1, 3, 4)[:, :, :3]
    leaves = nodes[(nodes["triCount"] > 0)]
    pts = [tri[:500, 0], (tri[:500, 0] + tri[:500, 1]) / 2, leaves["aabbMin"][:500],
           np.stack([leaves["aabbMax"][:500, 0], leaves["aabbMin"][:500, 1], (leaves["aabbMin"][:500, 2] + leaves["aabbMax"][:500, 2]) / 2], 1)]
    p = np.concatenate(pts).astype(np.float32)
    q = np.zeros((p.shape[0], 4), np.float32)
    q[:, :3] = p
    q[:, 3] = np.tile(np.array([np.inf, 0, 1e-7, 0.01], np.float32), p.shape[0] // 4 + 1)[: p.shape[0]]
    check_tree(e, nodes, idx, v, q, "planes", host=True)


def test_refit_and_optimize(gpu):
    v = scene(3000, 15)
    v2 = v.copy()
    v2[:, :3] += np.random.default_rng(1).normal(size=(v.shape[0], 3)).astype(np.float32) * 0.01
    q = queries_for(v, np.random.default_rng(12), n=1500)
    e = api.BVH().Build(v)
    e.Refit(v2)
    check_tree(e, *e.download(), v2, q, "refit")
    g = api.BVH_GPU().Build(v)
    _lib.check(_lib.lib().tbvh_refit_layouts(g.h, C.c_void_p(np.ascontiguousarray(v2).ctypes.data), 16, v.shape[0] // 3, _lib.HOST))
    nodes = np.zeros(g.info().used_nodes, NODE32)
    idx = np.zeros(g.info().idx_count, np.uint32)
    _lib.check(_lib.lib().tbvh_download_bvh(g.h, nodes.ctypes.data, idx.ctypes.data, _lib.HOST))
    check_tree(g, nodes, idx, v2, q, "refit_layouts")
    o = api.BVH().Build(v)
    o.optimize(4)
    check_tree(o, *o.download(), v, q, "optimize")


def test_group_replica(gpu, consumer):
    """a group replica's handle and its view answer as the source does"""
    import torch
    v = scene(3000, 25)
    e = api.BVH().Build(v)
    q = queries_for(v, np.random.default_rng(17), n=1500)
    want = check_tree(e, *e.download(), v, q, "source")
    grp = api.Group([0])
    grp.replicate(e)
    rep = _lib.lib().tbvh_group_replica(grp.h, 0)
    assert rep and rep != e.h.value
    dq = torch_f(q)
    out = torch.zeros((q.shape[0], 4), dtype=torch.float32, device="cuda")
    _lib.check(_lib.lib().tbvh_closest_point(C.c_void_p(rep), C.c_void_p(dq.data_ptr()), C.c_void_p(out.data_ptr()), q.shape[0], _lib.DEVICE, None))
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy().view(np.uint32), want.view(np.uint32)), "replica handle"
    out.zero_()
    bits = torch.zeros((q.shape[0] + 31) // 32, dtype=torch.int32, device="cuda")
    assert consumer.cc_query(grp.device_view(0), dq.data_ptr(), out.data_ptr(), bits.data_ptr(), None, q.shape[0]) == 0
    assert np.array_equal(out.cpu().numpy().view(np.uint32), want.view(np.uint32)), "replica view"
    grp.close()


def test_large_batch(gpu):
    """2^20 queries against the restatement's pruned walk (equal to its brute force, tests/test_closest_point.py)"""
    v = scene(40000, 26)
    e = api.BVH().Build(v)
    nodes, idx = e.download()
    q = queries_for(v, np.random.default_rng(18), n=1 << 19)[: 1 << 20]
    got = device_query(e, q, False)
    assert np.array_equal(got.view(np.uint32), co.walk(nodes, idx, v, q).view(np.uint32))
    assert np.array_equal(device_query(e, q, True), co.walk(nodes, idx, v, q, any_=True))


def test_device_matches_host_and_api(gpu):
    import torch
    v = scene(5000, 16)
    e = api.BVH().Build(v)
    q = queries_for(v, np.random.default_rng(13), n=4000)
    d, u, vv, prim = e.closest_point(q[:, :3], q[:, 3])
    td, tu, tv, tp = e.closest_point(torch_f(q[:, :3]), torch_f(q[:, 3]))
    torch.cuda.synchronize()
    for a, b in ((d, td), (u, tu), (vv, tv)):
        assert np.array_equal(a.view(np.uint32), b.cpu().numpy().view(np.uint32))
    assert np.array_equal(prim, tp.cpu().numpy().view(np.uint32))
    want = co.brute(*e.download(), v, q)
    assert np.array_equal(prim, co.record_prims(want))
    hits = e.sphere_overlap(q[:, :3], q[:, 3])
    th = e.sphere_overlap(torch_f(q[:, :3]), torch_f(q[:, 3]))
    assert np.array_equal(hits, th.cpu().numpy()) and np.array_equal(hits, prim != co.NO_PRIM)
    # (n, 4) rows are the C-ABI's {x, y, z, r} records, used as they are
    for pts in (q, torch_f(q)):
        r4 = e.closest_point(pts)
        got = r4[3].cpu().numpy().view(np.uint32) if hasattr(r4[3], "cpu") else r4[3]
        assert np.array_equal(got, prim)
        h4 = e.sphere_overlap(pts)
        assert np.array_equal(h4.cpu().numpy() if hasattr(h4, "cpu") else h4, hits)
        with pytest.raises(api.TbvhError):
            e.closest_point(pts, np.inf)
    with pytest.raises(api.TbvhError):
        e.sphere_overlap(torch_f(q[:, :3]))


def test_stream_order_and_words(gpu):
    import torch
    v = scene(3000, 17)
    e = api.BVH().Build(v)
    q = queries_for(v, np.random.default_rng(14), n=2000)
    want = co.brute(*e.download(), v, q)
    s = torch.cuda.Stream()
    src = torch_f(q)
    dq = torch.zeros_like(src)
    out = torch.zeros((q.shape[0], 4), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)   # the queries are written behind a long kernel on the caller's stream
        dq.copy_(src)
    _lib.check(_lib.lib().tbvh_closest_point(e.h, C.c_void_p(dq.data_ptr()), C.c_void_p(out.data_ptr()), q.shape[0], _lib.DEVICE, C.c_void_p(s.cuda_stream)))
    s.synchronize()
    assert np.array_equal(out.cpu().numpy().view(np.uint32), want.view(np.uint32)), "the query walked before the caller's stream wrote it"
    for n in (1, 31, 33, 100):
        assert np.array_equal(device_query(e, q[:n], False).view(np.uint32), want[:n].view(np.uint32)), f"n = {n}"
        w = torch.full(((n + 31) // 32 + 1,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
        dq = torch_f(q[:n])
        _lib.check(_lib.lib().tbvh_sphere_overlap(e.h, C.c_void_p(dq.data_ptr()), C.c_void_p(w.data_ptr()), n, _lib.DEVICE, None))
        got = w.cpu().numpy().view(np.uint32)
        assert got[-1] == 0x5A5A5A5A, "the word after (n+31)/32 was written"
        bits = np.unpackbits(got[:-1].view(np.uint8), bitorder="little")
        assert not bits[n:].any(), "bits past n are set"
        assert np.array_equal(bits[:n].astype(bool), co.record_prims(want[:n]) != co.NO_PRIM)


def test_refusals(gpu):
    import torch
    L = _lib.lib()
    v = scene(300, 18)
    e = api.BVH().Build(v)
    q = torch_f(queries_for(v, np.random.default_rng(1), n=64))
    out = torch.zeros((q.shape[0] + 1, 4), dtype=torch.float32, device="cuda")
    qp, op = C.c_void_p(q.data_ptr()), C.c_void_p(out.data_ptr())
    for fn in (L.tbvh_closest_point, L.tbvh_sphere_overlap):
        assert fn(None, qp, op, 4, _lib.DEVICE, None) == _lib.E_ARG
        assert fn(e.h, None, op, 4, _lib.DEVICE, None) == _lib.E_ARG
        assert fn(e.h, qp, None, 4, _lib.DEVICE, None) == _lib.E_ARG
        assert fn(e.h, qp, op, 4, 7, None) == _lib.E_ARG
        assert fn(e.h, C.c_void_p(q.data_ptr() + 4), op, 4, _lib.DEVICE, None) == _lib.E_ARG
        assert fn(e.h, qp, C.c_void_p(out.data_ptr() + 4), 4, _lib.DEVICE, None) == _lib.E_ARG
        assert fn(e.h, qp, op, 1 << 40, _lib.DEVICE, None) == _lib.E_ARG
        assert fn(e.h, qp, op, 0, _lib.DEVICE, None) == _lib.OK
        assert fn(api.BVH().h, qp, op, 4, _lib.DEVICE, None) == _lib.E_STATE
        c = api.BVH8_CWBVH().Build(v)
        only = api.BVH8_CWBVH().upload(*c.download())
        assert fn(only.h, qp, op, 4, _lib.DEVICE, None) == _lib.E_STATE
        deep = chain_tree(scene(300, 19), 300)
        d = api.BVH().upload(deep[0], deep[1], scene(300, 19))
        assert fn(d.h, qp, op, 4, _lib.DEVICE, None) == _lib.E_LIMIT
    inst = np.zeros(2, api.BLAS_INSTANCE)
    inst["transform"] = np.eye(4, dtype=np.float32).reshape(-1)
    inst["mask"] = 0xFFFF
    t = api.TLAS()
    t.Build(inst, [e])
    for fn in (L.tbvh_closest_point, L.tbvh_sphere_overlap):
        assert fn(t.h, qp, op, 4, _lib.DEVICE, None) == _lib.E_UNSUPPORTED
    torch.cuda.synchronize()
    assert not out.any(), "a refused call wrote results"


def test_fp64_distance(gpu):
    """builders whose leaves hold every triangle: d is the fp64 distance to the nearest triangle of the mesh within 2e-6 of the scene's
    magnitude"""
    v = scene(2000, 21)
    tri = v.reshape(-1, 3, 4)[:, :, :3].astype(np.float64)
    q = queries_for(v, np.random.default_rng(15), n=400, r_kinds=False)
    want = np.full(q.shape[0], np.inf)
    for k in range(tri.shape[0]):
        n = q.shape[0]
        want = np.minimum(want, fp64_closest(q[:, :3], np.repeat(tri[k:k + 1, 0], n, 0), np.repeat(tri[k:k + 1, 1], n, 0), np.repeat(tri[k:k + 1, 2], n, 0)))
    scale = np.maximum(np.abs(q[:, :3]).max(1), np.abs(v[:, :3]).max())
    for builder in ("Build", "BuildAVX", "BuildPLOC"):
        d, _, _, _ = getattr(api.BVH(), builder)(v).closest_point(q[:, :3], q[:, 3])
        assert (np.abs(d - want) <= 2e-6 * scale).all(), builder


@pytest.fixture(scope="module")
def consumer(gpu, tmp_path_factory):
    nvcc = build.nvcc_path()
    so = str(tmp_path_factory.mktemp("closest_consumer") / "consumer.so")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-I" + os.path.join(REPO, "include"),
                        "-Xcompiler", "-fPIC", "-shared", "-Xptxas", "-v", os.path.join(REPO, "tests", "closest_point_consumer.cu"), "-o", so],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    print(r.stderr)
    L = C.CDLL(so)
    L.cc_query.argtypes = [_lib.DeviceView, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]
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
        q = queries_for(v, np.random.default_rng(16), n=1500)
        want = device_query(e, q, False)
        wbits = device_query(e, q, True)
        n = q.shape[0]
        sel = np.random.default_rng(3).integers(0, 1 << 32, (n + 31) // 32, dtype=np.uint64).astype(np.uint32)
        for s in (None, sel):
            dq = torch_f(q)
            out = torch.full((n, 4), -7.0, dtype=torch.float32, device="cuda")
            bits = torch.zeros((n + 31) // 32, dtype=torch.int32, device="cuda")
            ds = torch.from_numpy(s.view(np.int32)).cuda() if s is not None else None
            assert consumer.cc_query(e.device_view(), dq.data_ptr(), out.data_ptr(), bits.data_ptr(), ds.data_ptr() if ds is not None else None, n) == 0
            got, gb = out.cpu().numpy(), bits.cpu().numpy().view(np.uint32)
            mask = np.ones(n, bool) if s is None else np.unpackbits(s.view(np.uint8), bitorder="little")[:n].astype(bool)
            assert np.array_equal(got[mask].view(np.uint32), want[mask].view(np.uint32)), "device function differs from the batch call"
            assert (got[~mask] == -7).all()
            wb = np.unpackbits(wbits.view(np.uint8), bitorder="little")[:n].astype(bool) & mask
            assert np.array_equal(np.unpackbits(gb.view(np.uint8), bitorder="little")[:n].astype(bool), wb)
    # a view of another kind: the miss record and false
    c = api.BVH8_CWBVH().Build(scene(300, 24))
    dq = torch_f(np.array([[0, 0, 0, 5]], np.float32))
    out = torch.zeros((1, 4), dtype=torch.float32, device="cuda")
    bits = torch.zeros(1, dtype=torch.int32, device="cuda")
    assert consumer.cc_query(c.device_view(_lib.LAYOUT_CWBVH), dq.data_ptr(), out.data_ptr(), bits.data_ptr(), None, 1) == 0
    assert out.cpu().numpy().view(np.uint32).tolist() == [[np.float32(5).view(np.uint32), 0, 0, co.NO_PRIM]] and int(bits[0]) == 0
