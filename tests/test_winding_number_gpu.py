"""tbvh_winding_number on the device, held bit for bit to the host restatement (tests/wn_oracle.c, DESIGN.md §4.11) at beta = 1.5, 2, 4
and inf: every builder (failed-split SBVHs included), batch and indexed builds, uploaded families, a BVH_GPU upload, trees 99 and 254
levels deep, golden scenes, tables prepared again after refits and tbvh_optimize, a group replica, a 65,536-triangle fan and a 1 M-triangle
mesh; host and device space, stream order, NaN queries, n = 0, every refusal and the prepare's launch count."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import portpy
from tinybvh_b200 import _lib, api, scenes
from tests import util, wn_oracle as wo
from tests.test_closest_point import family
from tests.test_closest_point_gpu import chain_tree, torch_f
from tests.test_signed_distance import cone, icosphere, soup, torus
from tests.test_signed_distance_gpu import big_torus
from tests.test_winding_number import soup_queries, two_spheres

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NODE32 = portpy.NODE32
BETAS = (1.5, 2.0, 4.0, np.inf)


def wn_device(h, q, beta, stream=None):
    import torch
    dq = torch_f(q)
    out = torch.zeros(q.shape[0], dtype=torch.float32, device="cuda")
    _lib.check(_lib.lib().tbvh_winding_number(h, C.c_void_p(dq.data_ptr()), C.c_void_p(out.data_ptr()), q.shape[0], float(beta), _lib.DEVICE, stream))
    torch.cuda.synchronize()
    return out.cpu().numpy()


def wn_host(h, q, beta):
    q = np.ascontiguousarray(q, np.float32)
    out = np.zeros(q.shape[0], np.float32)
    _lib.check(_lib.lib().tbvh_winding_number(h, q.ctypes.data, out.ctypes.data, q.shape[0], float(beta), _lib.HOST, None))
    return out


def same_bits(got, want, label):
    bad = got.view(np.uint32) != want.view(np.uint32)
    assert not bad.any(), f"{label}: {int(bad.sum())} of {got.shape[0]} differ, first {np.nonzero(bad)[0][:5]}: {got[bad][:3]} vs {want[bad][:3]}"


def check_tree(h, nodes, idx, v, q, label, host=False, betas=BETAS):
    """prepare, then every result at every beta equals the restatement's"""
    _lib.check(_lib.lib().tbvh_winding_number_prepare(h))
    t = wo.Table(nodes, idx, v)
    assert t.flag == 0, label
    out = {}
    for beta in betas:
        want = t.query(q, beta)
        out[beta] = wn_device(h, q, beta)
        same_bits(out[beta], want, f"{label} beta {beta}")
        if host:
            same_bits(wn_host(h, q, beta), want, f"{label} beta {beta} host")
    return out


def scene(n, seed=5):
    return scenes.procedural_scene(n, seed)


@pytest.mark.parametrize("builder", ["Build", "BuildAVX", "BuildHQ", "BuildPLOC"])
def test_builders(gpu, builder):
    for label, v in (("icosphere", soup(*icosphere(3))), ("two_spheres", soup(*two_spheres())), ("soup", scene(3000, 3))):
        e = getattr(api.BVH(), builder)(v)
        check_tree(e.h, *e.download(), v, soup_queries(v, np.random.default_rng(1), n=700), f"{builder}/{label}", host=label == "soup")


@pytest.mark.parametrize("name", ["snapped20k_q4", "lattice10k_k3"])
def test_hq_failed_splits(gpu, name):
    from tests.test_build_hq_shapes import fail_scene
    v = fail_scene(name)
    e = api.BVH().BuildHQ(v)
    got = check_tree(e.h, *e.download(), v, soup_queries(v, np.random.default_rng(1), n=700), f"BuildHQ-{name}")
    b = api.BVH().Build(v)
    ref = check_tree(b.h, *b.download(), v, soup_queries(v, np.random.default_rng(1), n=700), f"Build-{name}", betas=(np.inf,))
    assert np.abs(got[np.inf] - ref[np.inf]).max() <= 1e-6, "a split triangle counted twice"


def test_batch_and_indexed(gpu):
    meshes = [soup(*icosphere(2)), soup(*torus()), scene(700, 21)]
    for flavour in (_lib.BUILD_REFERENCE, _lib.BUILD_AVX, _lib.BUILD_PLOC, _lib.BUILD_HQ):
        objs = [api.BVH() for _ in meshes]
        api.build_batch(objs, meshes, flavour)
        for o, v in zip(objs, meshes):
            check_tree(o.h, *o.download(), v, soup_queries(v, np.random.default_rng(2), n=400), f"batch-{flavour}-{v.shape[0] // 3}", betas=(2.0, np.inf))
    V, F = torus()
    verts = np.zeros((V.shape[0], 4), np.float32)
    verts[:, :3] = V
    e = api.BVH()
    e.Build(verts, indices=F.astype(np.uint32).reshape(-1))
    s = api.BVH().Build(soup(V, F))
    q = soup_queries(soup(V, F), np.random.default_rng(3), n=700)
    a = check_tree(e.h, *e.download(), soup(V, F), q, "indexed")
    b = check_tree(s.h, *s.download(), soup(V, F), q, "soup")
    for beta in BETAS:
        same_bits(a[beta], b[beta], f"indexed against its V[I] soup, beta {beta}")


@pytest.mark.parametrize("fam", util.FAMILIES)
def test_uploaded_families(gpu, fam):
    v = soup(*icosphere(3))
    src = util.source_tree(v, "BuildHQ" if fam in ("C0", "C3") else "Build")
    nodes, idx = family(src, fam)
    e = api.BVH().upload(nodes, idx, v)
    check_tree(e.h, nodes, idx, v, soup_queries(v, np.random.default_rng(5), n=700), fam)


def test_bvh_gpu_upload_and_deep_trees(gpu):
    v = soup(*torus())
    o = util.oracle_tree(v, 1)
    g = api.BVH_GPU().upload(util.oracle_bvh_gpu_nodes(o), o.prim_idx, v)
    check_tree(g.h, o.nodes, o.prim_idx, v, soup_queries(v, np.random.default_rng(6), n=700), "BVH_GPU upload", host=True)
    w = scene(400, 12)
    for m in (100, 255):
        nodes, idx = chain_tree(w, m)
        c = api.BVH().upload(nodes, idx, w[: 3 * m])
        assert c.info().max_depth == m - 1
        check_tree(c.h, nodes, idx, w[: 3 * m], soup_queries(w[: 3 * m], np.random.default_rng(m), n=500), f"chain-{m}")


@pytest.mark.parametrize("name", ["flat_500", "coincident_610", "single_tri"])
def test_golden_scenes(gpu, name):
    g = np.load(os.path.join(REPO, "tests", "golden", f"{name}.npz"))
    v = g["verts"].astype(np.float32)
    nodes = np.ascontiguousarray(g["nodes"]).view(NODE32).reshape(-1)
    e = api.BVH().upload(nodes, g["prim_idx"], v)
    check_tree(e.h, nodes, g["prim_idx"], v, soup_queries(v, np.random.default_rng(10), n=700), name)


def refused_stale(h):
    q = torch_f(np.zeros((4, 4), np.float32))
    return _lib.lib().tbvh_winding_number(h, C.c_void_p(q.data_ptr()), C.c_void_p(q.data_ptr()), 4, 2.0, _lib.DEVICE, None) == _lib.E_STATE


def test_prepared_again_after_refit_and_optimize(gpu):
    V, F = icosphere(3)
    v = soup(V, F)
    v2 = v.copy()
    v2[:, :3] *= np.float32(1.25)
    q = soup_queries(v2, np.random.default_rng(12), n=600)
    e = api.BVH().Build(v)
    e.prepare_winding_number()
    e.Refit(v2)
    assert refused_stale(e.h)
    check_tree(e.h, *e.download(), v2, q, "refit")
    o = api.BVH().Build(soup(*torus()))
    o.prepare_winding_number()
    rounds = C.c_uint32()
    _lib.check(_lib.lib().tbvh_optimize(o.h, 4, C.c_float(1.0), C.c_float(1.0), C.byref(rounds), None))
    if rounds.value:
        assert refused_stale(o.h)
    check_tree(o.h, *o.download(), soup(*torus()), soup_queries(soup(*torus()), np.random.default_rng(13), n=600), "optimize")


def test_group_replica(gpu):
    v = soup(*icosphere(3))
    e = api.BVH().Build(v)
    q = soup_queries(v, np.random.default_rng(17), n=600)
    want = check_tree(e.h, *e.download(), v, q, "source")
    grp = api.Group([0])
    grp.replicate(e)
    rep = _lib.lib().tbvh_group_replica(grp.h, 0)
    assert rep and rep != e.h.value
    assert refused_stale(C.c_void_p(rep)), "a replica holds no table until prepared"
    got = check_tree(C.c_void_p(rep), *e.download(), v, q, "replica")
    for beta in BETAS:
        same_bits(got[beta], want[beta], f"replica beta {beta}")
    grp.close()


def test_cone_fan_and_million_triangles(gpu):
    V, F = cone()
    v = soup(V, F)
    e = api.BVH().Build(v)
    got = check_tree(e.h, *e.download(), v, soup_queries(v, np.random.default_rng(4), n=300), "cone")
    assert got[np.inf].shape[0] == 600
    V, F = big_torus()
    v = soup(V, F)
    e = api.BVH().Build(v)
    rng = np.random.default_rng(19)
    P = np.r_[rng.uniform(-1.4, 1.4, (300, 3)) * [1, 1, 0.3], V[F[rng.integers(0, F.shape[0], 300)]].mean(1) + rng.normal(size=(300, 3)) * 0.01]
    q = np.zeros((P.shape[0], 4), np.float32)
    q[:, :3] = P
    got = check_tree(e.h, *e.download(), v, q, "1M torus", betas=(2.0, np.inf))
    rho = np.hypot(np.hypot(q[:, 0], q[:, 1]) - 1.0, q[:, 2])
    far = np.abs(rho - 0.3) > 0.01
    assert np.array_equal((got[np.inf] > 0.5)[far], (rho < 0.3)[far])


def test_python_api_stream_nan_and_empty(gpu):
    import torch
    v = soup(*two_spheres())
    e = api.BVH().Build(v)
    e.prepare_winding_number()
    q = soup_queries(v, np.random.default_rng(14), n=600)
    t = wo.Table(*e.download(), v)
    want = t.query(q, 2.0)
    same_bits(e.winding_number(q[:, :3]), want, "numpy (n, 3)")
    same_bits(e.winding_number(q), want, "numpy (n, 4)")
    same_bits(e.winding_number(torch_f(q[:, :3])).cpu().numpy(), want, "torch")
    same_bits(e.winding_number(q, beta=np.inf), t.query(q, np.inf), "numpy exact")
    s = torch.cuda.Stream()
    src = torch_f(q)
    dq = torch.zeros_like(src)
    out = torch.zeros(q.shape[0], dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)   # the queries are written behind a long kernel on the caller's stream
        dq.copy_(src)
    _lib.check(_lib.lib().tbvh_winding_number(e.h, C.c_void_p(dq.data_ptr()), C.c_void_p(out.data_ptr()), q.shape[0], 2.0, _lib.DEVICE, C.c_void_p(s.cuda_stream)))
    s.synchronize()
    same_bits(out.cpu().numpy(), want, "caller's stream")
    for n in (1, 31, 33):
        same_bits(wn_device(e.h, q[:n], 2.0), want[:n], f"n = {n}")
    bad = np.array([[np.nan, 0, 0, 0], [0, np.nan, 0, 0], [0.4, 0, 0, np.nan], [0.4, 0, 0, 0]], np.float32)
    got = wn_device(e.h, bad, 2.0)
    assert (got.view(np.uint32)[:2] == 0x7FFFFFFF).all(), "a NaN coordinate gives NaN"
    assert got.view(np.uint32)[2] == got.view(np.uint32)[3] and abs(got[3] - 2) < 0.11, "the fourth column is ignored"
    before = api.launch_count()
    assert _lib.lib().tbvh_winding_number(e.h, C.c_void_p(src.data_ptr()), C.c_void_p(out.data_ptr()), 0, 2.0, _lib.DEVICE, None) == _lib.OK
    assert api.launch_count() == before


def test_refusals_and_launch_counts(gpu):
    import torch
    L = _lib.lib()
    V, F = icosphere(1)
    v = soup(V, F)
    e = api.BVH().Build(v)
    q = torch_f(soup_queries(v, np.random.default_rng(1), n=32))
    out = torch.zeros(q.shape[0] + 1, dtype=torch.float32, device="cuda")
    qp, op = C.c_void_p(q.data_ptr()), C.c_void_p(out.data_ptr())
    fn = lambda h, a, b, n, beta=2.0, space=_lib.DEVICE: fn0(h, a, b, n, beta, space, None)   # noqa: E731
    fn0 = L.tbvh_winding_number
    # prepare
    assert L.tbvh_winding_number_prepare(None) == _lib.E_ARG
    assert L.tbvh_winding_number_prepare(api.BVH().h) == _lib.E_STATE
    c = api.BVH8_CWBVH().Build(v)
    only = api.BVH8_CWBVH().upload(*c.download())
    assert L.tbvh_winding_number_prepare(only.h) == _lib.E_STATE
    w = scene(300, 19)
    deep = chain_tree(w, 300)
    d = api.BVH().upload(deep[0], deep[1], w)
    assert L.tbvh_winding_number_prepare(d.h) == _lib.E_LIMIT
    ball = soup(*icosphere(3))
    src = util.source_tree(ball, "Build")
    g = api.BVH().upload(family(src, "dag")[0], src[1], ball)
    before = g.download()
    assert L.tbvh_winding_number_prepare(g.h) == _lib.E_STATE
    assert refused_stale(g.h), "a refused prepare left a table"
    after = g.download()
    assert np.array_equal(before[0].view(np.uint32), after[0].view(np.uint32)) and np.array_equal(before[1], after[1])
    # the query: in proximity_query's order
    n0 = api.launch_count()
    assert fn(None, qp, op, 4) == _lib.E_ARG
    assert fn(e.h, None, op, 4) == _lib.E_ARG
    assert fn(e.h, qp, None, 4) == _lib.E_ARG
    assert fn(e.h, qp, op, 4, space=7) == _lib.E_ARG
    assert fn(e.h, C.c_void_p(q.data_ptr() + 4), op, 4) == _lib.E_ARG
    assert fn(e.h, qp, C.c_void_p(out.data_ptr() + 2), 4) == _lib.E_ARG
    for beta in (1.0, 0.5, -np.inf, np.nan):
        assert fn(e.h, qp, op, 4, beta) == _lib.E_ARG, beta
    assert fn(e.h, qp, op, 1 << 40) == _lib.E_ARG
    assert fn(api.BVH().h, qp, op, 4) == _lib.E_STATE
    assert fn(only.h, qp, op, 4) == _lib.E_STATE
    assert fn(d.h, qp, op, 4) == _lib.E_LIMIT
    assert fn(e.h, qp, op, 4) == _lib.E_STATE, "a query before prepare"
    assert fn(e.h, qp, op, 0) == _lib.E_STATE
    inst = np.zeros(2, api.BLAS_INSTANCE)
    inst["transform"] = np.eye(4, dtype=np.float32).reshape(-1)
    inst["mask"] = 0xFFFF
    t = api.TLAS()
    t.Build(inst, [e])
    n1 = api.launch_count()
    assert fn(t.h, qp, op, 4) == _lib.E_UNSUPPORTED
    assert L.tbvh_winding_number_prepare(t.h) == _lib.E_UNSUPPORTED
    assert api.launch_count() == n1 and n1 >= n0, "a refusal launched work"
    torch.cuda.synchronize()
    assert not out.any(), "a refused call wrote results"
    # a prepare launches 2 depth + 3 kernels; a misaligned result pointer 4 bytes in is fine
    k0 = api.launch_count()
    _lib.check(L.tbvh_winding_number_prepare(e.h))
    assert api.launch_count() - k0 == 2 * e.info().max_depth + 3
    assert fn(e.h, qp, C.c_void_p(out.data_ptr() + 4), 4) == _lib.OK
    # a refused query leaves the table: the same results afterwards
    a = wn_device(e.h, q.cpu().numpy(), 2.0)
    assert fn(e.h, qp, op, 4, 1.0) == _lib.E_ARG
    same_bits(wn_device(e.h, q.cpu().numpy(), 2.0), a, "after a refused query")
    # every call that changes the tree or its vertices makes the table stale
    stampers = {
        "Build": lambda: e.Build(v),
        "upload": lambda: e.upload(*e.download(), v),
        "refit": lambda: e.Refit(v),
        "refit_layouts": lambda: _lib.check(L.tbvh_refit_layouts(e.h, C.c_void_p(np.ascontiguousarray(v).ctypes.data), 16, v.shape[0] // 3, _lib.HOST)),
        "BuildPLOC": lambda: e.BuildPLOC(v),
    }
    for name, call in stampers.items():
        _lib.check(L.tbvh_winding_number_prepare(e.h))
        assert fn(e.h, qp, op, 4) == _lib.OK, name
        call()
        n1 = api.launch_count()
        assert fn(e.h, qp, op, 4) == _lib.E_STATE, f"stale after {name}"
        assert api.launch_count() == n1
