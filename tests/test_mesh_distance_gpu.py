"""tbvh_mesh_distance / tbvh_mesh_distance_pairs on the device, held bit for bit to the host restatement (tests/meshdist_oracle.c,
DESIGN.md §4.13): every nearest record, the sorted pairs and the count over every builder's tree (failed-split SBVHs included), batch and
indexed builds, uploaded families and a DAG, a BVH_GPU upload, trees 99 and 254 levels deep, golden and off-atrium scenes, refitted and
optimised trees, a group replica, a 1 M-triangle mesh against a shifted copy, and lattice meshes scaled by 2^k; host and device space,
every capacity, stream order, r_max = inf, and every refusal."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import portpy
from tinybvh_b200 import _lib, api, scenes
from tests import meshdist_oracle as md, util
from tests.test_closest_point import family
from tests.test_closest_point_gpu import chain_tree, torch_f
from tests.test_mesh_overlap import lattice_soup
from tests.test_mesh_overlap_gpu import h_of, shifted
from tests.test_signed_distance import icosphere, soup, torus
from tests.test_signed_distance_gpu import big_torus
from tests.test_winding_number import two_spheres

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NODE32 = portpy.NODE32
L = lambda: _lib.lib()  # noqa: E731


def nearest_device(a, b, n, r_max=np.inf, stream=None):
    import torch
    rec = torch.full((max(n, 1), 2), -1, dtype=torch.int32, device="cuda")
    _lib.check(L().tbvh_mesh_distance(h_of(a), h_of(b), float(r_max), C.c_void_p(rec.data_ptr()), _lib.DEVICE, stream))
    torch.cuda.synchronize()
    r = rec.cpu().numpy()[:n]
    return r[:, 0].view(np.float32), r[:, 1].view(np.uint32)


def nearest_host(a, b, n, r_max=np.inf):
    rec = np.full((max(n, 1), 2), 0xFFFFFFFF, np.uint32)
    _lib.check(L().tbvh_mesh_distance(h_of(a), h_of(b), float(r_max), rec.ctypes.data, _lib.HOST, None))
    return rec[:n, 0].view(np.float32), rec[:n, 1]


def pairs_device(a, b, r, cap, stream=None):
    import torch
    out = torch.full((max(cap, 1), 2), -1, dtype=torch.int32, device="cuda")
    count = C.c_uint64(12345)
    rc = L().tbvh_mesh_distance_pairs(h_of(a), h_of(b), float(r), C.c_void_p(out.data_ptr()), cap, C.byref(count), _lib.DEVICE, stream)
    torch.cuda.synchronize()
    return out.cpu().numpy().view(np.uint32), count.value, rc


def pairs_host(a, b, r, cap):
    out = np.full((max(cap, 1), 2), 0xFFFFFFFF, np.uint32)
    count = C.c_uint64(12345)
    rc = L().tbvh_mesh_distance_pairs(h_of(a), h_of(b), float(r), out.ctypes.data, cap, C.byref(count), _lib.HOST, None)
    return out, count.value, rc


def same_records(got, want, label):
    assert np.array_equal(got[0].view(np.uint32), want[0].view(np.uint32)), f"{label}: distances differ"
    assert np.array_equal(got[1], want[1]), f"{label}: nearest triangles differ"


def check(a, b, va, nodes, idx, vb, label, host=False, r=None):
    """a against b (a is b: the self query): nearest records at r_max = inf and r, and the pairs at r, equal the restatement's walk"""
    self = h_of(a).value == h_of(b).value
    n = va.shape[0] // 3
    ext = float(np.abs(vb[:, :3]).max()) if vb.shape[0] else 1.0
    r = 0.01 * ext if r is None else r
    want_inf = md.nearest(nodes, idx, vb, None if self else va)
    same_records(nearest_device(a, b, n), want_inf, f"{label} nearest")
    want_r = md.nearest(nodes, idx, vb, None if self else va, r_max=r)
    same_records(nearest_device(a, b, n, r), want_r, f"{label} nearest within {r}")
    want, keys, _ = md.pairs(nodes, idx, vb, None if self else va, r)
    got, count, rc = pairs_device(a, b, r, max(want.shape[0], 1))
    _lib.check(rc)
    assert count == want.shape[0] and np.array_equal(got[:count], want), f"{label}: pairs at {r} ({count}, restatement {want.shape[0]})"
    if host:
        same_records(nearest_host(a, b, n), want_inf, f"{label} host nearest")
        hp, hc, rc = pairs_host(a, b, r, max(want.shape[0], 1))
        _lib.check(rc)
        assert hc == count and np.array_equal(hp[:hc], want), f"{label}: host pairs"
    return want_inf, want


@pytest.mark.parametrize("builder", ["Build", "BuildAVX", "BuildHQ", "BuildPLOC"])
@pytest.mark.parametrize("ntris", [1, 7, 3000, 40000])
def test_builders(gpu, builder, ntris):
    va = scenes.procedural_scene(ntris, 3 + ntris)
    vb = shifted(scenes.procedural_scene(max(ntris, 2), 4 + ntris), 0.05)
    a, b = getattr(api.BVH(), builder)(va), getattr(api.BVH(), builder)(vb)
    check(a, b, va, *b.download(), vb, f"{builder}-{ntris}", host=ntris == 3000)
    check(a, a, va, *a.download(), va, f"self {builder}-{ntris}", host=ntris == 3000)
    if ntris == 3000:
        ab = pairs_device(a, b, 0.02, 1 << 20)
        ba = pairs_device(b, a, 0.02, 1 << 20)
        p, q = ab[0][: ab[1]], ba[0][: ba[1]]
        assert ab[1] > 0 and np.array_equal(p, q[np.lexsort((q[:, 0], q[:, 1]))][:, ::-1]), "swapping a and b swaps the pairs"


@pytest.mark.parametrize("name", ["snapped20k_q4", "lattice10k_k3"])
def test_hq_failed_splits(gpu, name):
    from tests.test_build_hq_shapes import fail_scene
    v = fail_scene(name)
    e = api.BVH().BuildHQ(v)
    check(e, e, v, *e.download(), v, f"BuildHQ-{name}")


def test_batch_and_indexed(gpu):
    meshes = [soup(*two_spheres()), soup(*torus()), scenes.procedural_scene(700, 21)]
    for flavour in (_lib.BUILD_REFERENCE, _lib.BUILD_AVX, _lib.BUILD_PLOC, _lib.BUILD_HQ):
        objs = [api.BVH() for _ in meshes]
        api.build_batch(objs, meshes, flavour)
        for o, v in zip(objs, meshes):
            check(o, o, v, *o.download(), v, f"batch-{flavour}-{v.shape[0] // 3}")
        check(objs[0], objs[2], meshes[0], *objs[2].download(), meshes[2], f"batch-{flavour} a/b")
    V, F = torus()
    verts = np.zeros((V.shape[0], 4), np.float32)
    verts[:, :3] = V
    e = api.BVH()
    e.Build(verts, indices=F.astype(np.uint32).reshape(-1))
    s = api.BVH().Build(soup(V, F))
    a = check(e, e, soup(V, F), *e.download(), soup(V, F), "indexed")
    b = check(s, s, soup(V, F), *s.download(), soup(V, F), "soup")
    assert np.array_equal(a[0][0], b[0][0]) and np.array_equal(a[1], b[1])


@pytest.mark.parametrize("fam", util.FAMILIES + ["dag"])
def test_uploaded_families(gpu, fam):
    v = scenes.procedural_scene(3000, 71)
    va = scenes.procedural_scene(1500, 72)
    src = util.source_tree(v, "BuildHQ" if fam in ("C0", "C3", "DB") else "Build")
    nodes, idx = family(src, fam)
    e = api.BVH().upload(nodes, idx, v)
    a = api.BVH().Build(va)
    check(a, e, va, nodes, idx, v, f"family {fam}")
    check(e, e, v, nodes, idx, v, f"family self {fam}")


def test_bvh_gpu_upload_and_deep_trees(gpu):
    v = soup(*two_spheres())
    o = util.oracle_tree(v, 1)
    g = api.BVH_GPU().upload(util.oracle_bvh_gpu_nodes(o), o.prim_idx, v)
    check(g, g, v, o.nodes, o.prim_idx, v, "BVH_GPU upload", host=True)
    w = scenes.procedural_scene(400, 12)
    for m in (100, 255):
        nodes, idx = chain_tree(w, m)
        c = api.BVH().upload(nodes, idx, w[: 3 * m])
        assert c.info().max_depth == m - 1
        check(c, c, w[: 3 * m], nodes, idx, w[: 3 * m], f"chain-{m}")
        a = api.BVH().Build(w)
        check(a, c, w, nodes, idx, w[: 3 * m], f"chain-{m} a/b")


@pytest.mark.parametrize("name", ["flat_500", "coincident_610", "single_tri", "atrium_3k"])
def test_golden_scenes(gpu, name):
    g = np.load(os.path.join(REPO, "tests", "golden", f"{name}.npz"))
    v = g["verts"].astype(np.float32)
    nodes = np.ascontiguousarray(g["nodes"]).view(NODE32).reshape(-1)
    e = api.BVH().upload(nodes, g["prim_idx"], v)
    check(e, e, v, nodes, g["prim_idx"], v, name, host=True)


def test_off_atrium(gpu):
    g = np.load(os.path.join(REPO, "tests", "golden", "atrium_3k.npz"))
    v = g["verts"].astype(np.float32)
    for d in (0.37, 1e-3):
        b = api.BVH().Build(shifted(v, d))
        a = api.BVH().Build(v)
        check(a, b, v, *b.download(), shifted(v, d), f"off-atrium {d}")


def test_refit_optimize_and_replica(gpu):
    v = soup(*two_spheres())
    v2 = v.copy()
    v2[:, :3] *= np.float32(1.25)
    e = api.BVH().Build(v)
    e.Refit(v2)
    check(e, e, v2, *e.download(), v2, "refit")
    o = api.BVH().Build(soup(*torus()))
    rounds = C.c_uint32()
    _lib.check(L().tbvh_optimize(o.h, 4, C.c_float(1.0), C.c_float(1.0), C.byref(rounds), None))
    t = soup(*torus())
    check(o, o, t, *o.download(), t, "optimize")
    s = api.BVH().Build(v)
    want_n, want = check(s, s, v, *s.download(), v, "source", r=0.05)
    grp = api.Group([0])
    grp.replicate(s)
    rep = C.c_void_p(L().tbvh_group_replica(grp.h, 0))
    same_records(nearest_device(rep, rep, v.shape[0] // 3), want_n, "group replica")
    got, count, rc = pairs_device(rep, rep, 0.05, want.shape[0] + 4)
    _lib.check(rc)
    assert count == want.shape[0] and np.array_equal(got[:count], want), "group replica pairs"
    grp.close()


def test_million_triangles_against_a_shifted_copy(gpu):
    V, F = big_torus()
    v = soup(V, F)
    w = shifted(v, 0.013)
    a, b = api.BVH().Build(v), api.BVH().Build(w)
    n = v.shape[0] // 3
    d, j = nearest_device(a, b, n)
    r = 0.004
    got, count, rc = pairs_device(a, b, r, 1 << 24)
    _lib.check(rc)
    nodes, idx = b.download()
    k = 32768
    same_records((d[:k], j[:k]), md.nearest(nodes, idx, w, v[: 3 * k]), "the first 32768 triangles of A")
    want = md.pairs(nodes, idx, w, v[: 3 * k], r)[0]
    assert np.array_equal(got[:count][got[:count, 0] < k], want), "pairs of the first 32768 triangles of A"
    assert (j != md.NO_PRIM).all()
    print(f"1M torus against its shifted copy: separation {d.min()}, {count} pairs within {r}")


def test_scaled_lattices(gpu):
    A, B = lattice_soup(3000, 4), lattice_soup(3000, 5, offset=0.5)
    ref = None
    for k in (-40, -20, 0, 20, 40):
        sa, sb = util.scaled(A, k), util.scaled(B, k)
        a, b = api.BVH().BuildHQ(sa), api.BVH().BuildHQ(sb)
        r = float(np.ldexp(np.float32(0.75), k))
        wn, wp = check(a, b, sa, *b.download(), sb, f"scale {k}", r=r)
        sn, sp = check(a, a, sa, *a.download(), sa, f"self scale {k}", r=r)
        got = (np.ldexp(wn[0], -k), wn[1], wp, np.ldexp(sn[0], -k), sn[1], sp)
        if ref is None:
            ref = got
        for x, y in zip(got, ref):
            assert np.array_equal(x, y), k
    assert ref[2].shape[0] > 100 and ref[5].shape[0] > 100


def test_capacity_python_api_and_stream_order(gpu):
    import torch
    v = soup(*two_spheres())
    w = scenes.procedural_scene(2000, 9)
    a, b = api.BVH().Build(v), api.BVH().Build(w)
    r = 0.02
    want = md.pairs(*b.download(), w, v, r)[0]
    m = want.shape[0]
    assert m > 10
    for cap in (0, 1, m // 2, m, m + 7):
        got, count, rc = pairs_device(a, b, r, cap)
        _lib.check(rc)
        assert count == m and np.array_equal(got[: min(cap, m)], want[: min(cap, m)]), cap
        assert (got[min(cap, m):] == 0xFFFFFFFF).all(), f"capacity {cap}: written past min(count, capacity)"
        hp, hc, rc = pairs_host(a, b, r, cap)
        _lib.check(rc)
        assert hc == m and np.array_equal(hp[: min(cap, m)], want[: min(cap, m)]) and (hp[min(cap, m):] == 0xFFFFFFFF).all(), cap
    count = C.c_uint64()
    _lib.check(L().tbvh_mesh_distance_pairs(a.h, b.h, C.c_float(r), None, 0, C.byref(count), _lib.DEVICE, None))
    assert count.value == m
    # the Python API: numpy and tensors
    assert np.array_equal(a.distance_pairs(b, r), want)
    s = torch.cuda.Stream()
    t = a.distance_pairs(b, r, stream=s)
    assert t.dtype == torch.int32 and t.is_cuda and np.array_equal(t.cpu().numpy().view(np.uint32), want)
    assert np.array_equal(a.distance_pairs(r=r), md.pairs(*a.download(), v, None, r)[0])
    wn = md.nearest(*b.download(), w, v)
    same_records(a.nearest_triangles(b), wn, "python numpy")
    td, tj = a.nearest_triangles(b, stream=s)
    s.synchronize()
    same_records((td.cpu().numpy(), tj.cpu().numpy().view(np.uint32)), wn, "python tensors")
    same_records(a.nearest_triangles(r_max=0.05), md.nearest(*a.download(), v, None, 0.05), "python self")
    # stream order: b's vertices refitted behind a long kernel on the caller's stream are what the calls see
    w2 = shifted(w, 0.3)
    dv = torch_f(w2)
    stage = torch.zeros_like(dv)
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)
        stage.copy_(dv)
    s.synchronize()
    _lib.check(L().tbvh_refit(b.h, C.c_void_p(stage.data_ptr()), 16, w2.shape[0] // 3, _lib.DEVICE))
    want2 = md.pairs(*b.download(), w2, v, r)[0]
    out = torch.full((want2.shape[0] + 1, 2), -1, dtype=torch.int32, device="cuda")
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)
        out.fill_(-2)   # queued behind the sleep: the pairs call must come after it
    cnt = C.c_uint64()
    _lib.check(L().tbvh_mesh_distance_pairs(a.h, b.h, C.c_float(r), C.c_void_p(out.data_ptr()), out.shape[0], C.byref(cnt), _lib.DEVICE, C.c_void_p(s.cuda_stream)))
    s.synchronize()
    o = out.cpu().numpy().view(np.uint32)
    assert cnt.value == want2.shape[0] and np.array_equal(o[: cnt.value], want2), "pairs ordered after the caller's stream"
    n = v.shape[0] // 3
    rec = torch.full((n, 2), -1, dtype=torch.int32, device="cuda")
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)
        rec.fill_(-1)
        _lib.check(L().tbvh_mesh_distance(a.h, b.h, C.c_float(np.inf), C.c_void_p(rec.data_ptr()), _lib.DEVICE, C.c_void_p(s.cuda_stream)))
    s.synchronize()
    r2 = rec.cpu().numpy()
    same_records((r2[:, 0].view(np.float32), r2[:, 1].view(np.uint32)), md.nearest(*b.download(), w2, v), "nearest queued on the caller's stream")


def test_refusals_leave_outputs_untouched(gpu):
    import torch
    v = soup(*icosphere(2))
    e = api.BVH().Build(v)
    n = v.shape[0] // 3
    out = torch.full((64, 2), -1, dtype=torch.int32, device="cuda")
    rec = torch.full((n + 2, 2), -1, dtype=torch.int32, device="cuda")
    op, rp = C.c_void_p(out.data_ptr()), C.c_void_p(rec.data_ptr())
    cnt = C.c_uint64(777)
    P = lambda a, b, o=op, r=0.1, cap=64, c=C.byref(cnt), space=_lib.DEVICE: L().tbvh_mesh_distance_pairs(a, b, C.c_float(r), o, cap, c, space, None)  # noqa: E731
    N = lambda a, b, o=rp, r=np.inf, space=_lib.DEVICE: L().tbvh_mesh_distance(a, b, C.c_float(r), o, space, None)  # noqa: E731
    assert P(None, e.h) == _lib.E_ARG and P(e.h, None) == _lib.E_ARG
    assert P(e.h, e.h, o=None) == _lib.E_ARG and P(e.h, e.h, c=None) == _lib.E_ARG and P(e.h, e.h, space=7) == _lib.E_ARG
    assert P(e.h, e.h, o=C.c_void_p(out.data_ptr() + 4)) == _lib.E_ARG
    assert N(None, e.h) == _lib.E_ARG and N(e.h, e.h, o=None) == _lib.E_ARG and N(e.h, e.h, space=7) == _lib.E_ARG
    assert N(e.h, e.h, o=C.c_void_p(rec.data_ptr() + 4)) == _lib.E_ARG
    for bad in (np.nan, -1.0, -np.inf):
        assert P(e.h, e.h, r=bad) == _lib.E_ARG and N(e.h, e.h, r=bad) == _lib.E_ARG, bad
    other_ctx = C.c_void_p()
    _lib.check(L().tbvh_ctx_create(0, C.byref(other_ctx)))
    f = C.c_void_p()
    _lib.check(L().tbvh_bvh_create(other_ctx, C.byref(f)))
    vv = np.ascontiguousarray(v)
    _lib.check(L().tbvh_build(f, vv.ctypes.data, 16, n, _lib.HOST, 1.0, 1.0))
    assert P(e.h, f) == _lib.E_ARG and N(f, e.h) == _lib.E_ARG, "handles of different contexts"
    inst = np.zeros(2, api.BLAS_INSTANCE)
    inst["transform"] = np.eye(4, dtype=np.float32).reshape(-1)
    inst["mask"] = 0xFFFF
    t = api.TLAS()
    t.Build(inst, [e])
    assert P(t.h, e.h) == _lib.E_UNSUPPORTED and N(e.h, t.h) == _lib.E_UNSUPPORTED
    assert P(t.h, e.h, r=np.nan) == _lib.E_ARG, "the distance argument is refused with the other argument errors"
    assert P(api.BVH().h, e.h) == _lib.E_STATE and N(e.h, api.BVH().h) == _lib.E_STATE
    c = api.BVH8_CWBVH().Build(v)
    only = api.BVH8_CWBVH().upload(*c.download())
    assert P(only.h, e.h) == _lib.E_STATE and N(e.h, only.h) == _lib.E_STATE
    w = scenes.procedural_scene(300, 19)
    deep = chain_tree(w, 300)
    d = api.BVH().upload(deep[0], deep[1], w)
    assert P(e.h, d.h) == _lib.E_LIMIT and N(d.h, d.h) == _lib.E_LIMIT
    torch.cuda.synchronize()
    assert (out == -1).all() and (rec == -1).all() and cnt.value == 777, "a refused call wrote its outputs"
    k0 = api.launch_count()
    assert (P(t.h, e.h), N(e.h, d.h), P(only.h, e.h), N(e.h, e.h, r=np.nan)) == (_lib.E_UNSUPPORTED, _lib.E_LIMIT, _lib.E_STATE, _lib.E_ARG)
    assert api.launch_count() == k0, "a refusal launched work"
    k0 = api.launch_count()
    _lib.check(N(e.h, e.h))
    assert api.launch_count() - k0 == 1, "the nearest query is one launch"
    # r_max = inf finds a triangle for every finite triangle; r = 0 pairs of a closed icosphere: none (neighbours share corners)
    dd, jj = nearest_device(e, e, n)
    assert (jj != md.NO_PRIM).all() and (dd > 0).all()
    assert pairs_device(e, e, 0.0, 8)[1] == 0
    _lib.check(L().tbvh_bvh_destroy(f))
    _lib.check(L().tbvh_ctx_destroy(other_ctx))
