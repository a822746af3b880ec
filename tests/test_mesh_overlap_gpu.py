"""tbvh_mesh_overlap_pairs / tbvh_mesh_overlap_bits on the device, held bit for bit to the host restatement (tests/tritri_oracle.c,
DESIGN.md §4.12): the sorted pairs, the count and every bit word over every builder's tree (failed-split SBVHs included), batch and
indexed builds, uploaded families and a DAG, a BVH_GPU upload, trees 99 and 254 levels deep, golden scenes, refitted and optimised
trees, a group replica, a 1 M-triangle mesh against a shifted copy, and lattice meshes scaled by 2^k; host and device space, every
capacity, stream order, bits against membership in the pairs, and every refusal."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import portpy
from tinybvh_b200 import _lib, api, scenes
from tests import tritri_oracle as to, util
from tests.test_closest_point import family
from tests.test_closest_point_gpu import chain_tree, torch_f
from tests.test_mesh_overlap import lattice_soup
from tests.test_signed_distance import icosphere, soup, torus
from tests.test_signed_distance_gpu import big_torus
from tests.test_winding_number import two_spheres

pytestmark = pytest.mark.gpu
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NODE32 = portpy.NODE32
L = lambda: _lib.lib()  # noqa: E731


def h_of(x):
    return x.h if hasattr(x, "h") else x


def pairs_device(a, b, cap, stream=None):
    """-> (pairs (min(count, cap), 2) uint32, count, rc)"""
    import torch
    out = torch.full((max(cap, 1), 2), -1, dtype=torch.int32, device="cuda")
    count = C.c_uint64(12345)
    rc = L().tbvh_mesh_overlap_pairs(h_of(a), h_of(b), C.c_void_p(out.data_ptr()), cap, C.byref(count), _lib.DEVICE, stream)
    torch.cuda.synchronize()
    got = out.cpu().numpy().view(np.uint32)
    return got, count.value, rc


def pairs_host(a, b, cap):
    out = np.full((max(cap, 1), 2), 0xFFFFFFFF, np.uint32)
    count = C.c_uint64(12345)
    rc = L().tbvh_mesh_overlap_pairs(h_of(a), h_of(b), out.ctypes.data, cap, C.byref(count), _lib.HOST, None)
    return out, count.value, rc


def bits_device(a, b, n):
    import torch
    w = torch.full((max((n + 31) // 32, 1),), -1, dtype=torch.int32, device="cuda")
    _lib.check(L().tbvh_mesh_overlap_bits(h_of(a), h_of(b), C.c_void_p(w.data_ptr()), _lib.DEVICE, None))
    torch.cuda.synchronize()
    return w.cpu().numpy().view(np.uint32)


def bits_host(a, b, n):
    w = np.full(max((n + 31) // 32, 1), 0xFFFFFFFF, np.uint32)
    _lib.check(L().tbvh_mesh_overlap_bits(h_of(a), h_of(b), w.ctypes.data, _lib.HOST, None))
    return w


def check(a, b, va, nodes, idx, vb, label, host=False):
    """a against b (a is b: the self query): pairs, count and bits equal the restatement's walk over b's tree"""
    self = h_of(a).value == h_of(b).value
    want, wbits, keys, _ = to.tree(nodes, idx, vb, None if self else va)
    n = va.shape[0] // 3
    cap = max(want.shape[0], 1)
    got, count, rc = pairs_device(a, b, cap)
    _lib.check(rc)
    assert count == want.shape[0], f"{label}: count {count}, restatement {want.shape[0]}"
    assert np.array_equal(got[:count], want), f"{label}: pairs differ"
    assert np.array_equal(bits_device(a, b, n), wbits), f"{label}: bits differ"
    assert np.array_equal(wbits, to.member_bits(want, n, self)) or label.startswith("family"), f"{label}: bits are not membership"
    if host:
        hp, hc, rc = pairs_host(a, b, cap)
        _lib.check(rc)
        assert hc == count and np.array_equal(hp[:hc], want), f"{label}: host pairs"
        assert np.array_equal(bits_host(a, b, n), wbits), f"{label}: host bits"
    return want, keys


def shifted(v, d):
    w = v.copy()
    w[:, :3] += np.float32(d)
    return w


@pytest.mark.parametrize("builder", ["Build", "BuildAVX", "BuildHQ", "BuildPLOC"])
@pytest.mark.parametrize("ntris", [1, 7, 3000, 40000])
def test_builders(gpu, builder, ntris):
    va = scenes.procedural_scene(ntris, 3 + ntris)
    vb = shifted(scenes.procedural_scene(max(ntris, 2), 4 + ntris), 0.05)
    a, b = getattr(api.BVH(), builder)(va), getattr(api.BVH(), builder)(vb)
    check(a, b, va, *b.download(), vb, f"{builder}-{ntris}", host=ntris == 3000)
    check(a, a, va, *a.download(), va, f"self {builder}-{ntris}", host=ntris == 3000)
    if ntris == 3000:
        ab = pairs_device(a, b, 1 << 20)
        ba = pairs_device(b, a, 1 << 20)
        p, q = ab[0][: ab[1]], ba[0][: ba[1]]
        assert np.array_equal(p, q[np.lexsort((q[:, 0], q[:, 1]))][:, ::-1]), "swapping a and b swaps the pairs"


@pytest.mark.parametrize("name", ["snapped20k_q4", "lattice10k_k3"])
def test_hq_failed_splits(gpu, name):
    from tests.test_build_hq_shapes import fail_scene
    v = fail_scene(name)
    e = api.BVH().BuildHQ(v)
    want, keys = check(e, e, v, *e.download(), v, f"BuildHQ-{name}")
    print(f"{name}: {keys.shape[0]} raw keys, {want.shape[0]} pairs")


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
    a = check(e, e, soup(V, F), *e.download(), soup(V, F), "indexed")[0]
    b = check(s, s, soup(V, F), *s.download(), soup(V, F), "soup")[0]
    assert np.array_equal(a, b)


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
    want = check(s, s, v, *s.download(), v, "source")[0]
    grp = api.Group([0])
    grp.replicate(s)
    rep = C.c_void_p(L().tbvh_group_replica(grp.h, 0))
    got, count, rc = pairs_device(rep, rep, want.shape[0] + 4)
    _lib.check(rc)
    assert count == want.shape[0] and np.array_equal(got[:count], want), "group replica"
    assert np.array_equal(bits_device(rep, rep, v.shape[0] // 3), to.member_bits(want, v.shape[0] // 3, True))
    grp.close()


def test_million_triangles_against_a_shifted_copy(gpu):
    V, F = big_torus()
    v = soup(V, F)
    w = shifted(v, 0.013)
    a, b = api.BVH().Build(v), api.BVH().Build(w)
    got, count, rc = pairs_device(a, b, 1 << 24)
    _lib.check(rc)
    bits = bits_device(a, b, v.shape[0] // 3)
    nodes, idx = b.download()
    k = 32768
    want, wbits, _, _ = to.tree(nodes, idx, w, v[: 3 * k])
    sel = got[:count][got[:count, 0] < k]
    assert np.array_equal(sel, want), "the first 32768 triangles of A"
    assert np.array_equal(bits[: k // 32], wbits[: k // 32])
    assert np.array_equal(bits, to.member_bits(got[:count], v.shape[0] // 3, False))
    print(f"1M torus against its shifted copy: {count} pairs")


def test_scaled_lattices_give_the_same_pairs(gpu):
    A, B = lattice_soup(3000, 4), lattice_soup(3000, 5)
    ref = None
    for k in (-40, -20, 0, 20, 40):
        sa, sb = util.scaled(A, k), util.scaled(B, k)
        # BuildHQ trees: the leaf boxes of BVH::Build's tree of these meshes at 2^40 do not hold their triangles, so there the reached
        # set is smaller than all pairs (the query's definition is kept, the pairs are not those of the other scales)
        a, b = api.BVH().BuildHQ(sa), api.BVH().BuildHQ(sb)
        p = check(a, b, sa, *b.download(), sb, f"scale {k}")[0]
        s = check(a, a, sa, *a.download(), sa, f"self scale {k}")[0]
        if ref is None:
            ref = (p, s)
        assert np.array_equal(p, ref[0]) and np.array_equal(s, ref[1]), k
    assert ref[0].shape[0] > 100 and ref[1].shape[0] > 100


def test_capacity_python_api_and_stream_order(gpu):
    import torch
    v = soup(*two_spheres())
    w = shifted(scenes.procedural_scene(2000, 9), 0.0)
    a, b = api.BVH().Build(v), api.BVH().Build(w)
    want = to.tree(*b.download(), w, v)[0]
    m = want.shape[0]
    assert m > 10
    for cap in (0, 1, m // 2, m, m + 7):
        got, count, rc = pairs_device(a, b, cap)
        _lib.check(rc)
        assert count == m and np.array_equal(got[: min(cap, m)], want[: min(cap, m)]), cap
        assert (got[min(cap, m):] == 0xFFFFFFFF).all(), f"capacity {cap}: written past min(count, capacity)"
        hp, hc, rc = pairs_host(a, b, cap)
        _lib.check(rc)
        assert hc == m and np.array_equal(hp[: min(cap, m)], want[: min(cap, m)]) and (hp[min(cap, m):] == 0xFFFFFFFF).all(), cap
    count = C.c_uint64()
    _lib.check(L().tbvh_mesh_overlap_pairs(a.h, b.h, None, 0, C.byref(count), _lib.DEVICE, None))
    assert count.value == m
    # the Python API: numpy and tensors, the capacity guess repeated once
    assert np.array_equal(a.overlap_pairs(b), want)
    s = torch.cuda.Stream()
    t = a.overlap_pairs(b, stream=s)
    assert t.dtype == torch.int32 and t.is_cuda and np.array_equal(t.cpu().numpy().view(np.uint32), want)
    selfp = to.tree(*a.download(), v)[0]
    assert np.array_equal(a.overlap_pairs(), selfp)
    n = v.shape[0] // 3
    member = np.zeros(n, bool)
    member[want[:, 0]] = True
    assert np.array_equal(a.overlapping(b), member)
    assert np.array_equal(a.overlapping(b, stream=s).cpu().numpy(), member)
    ms = np.zeros(n, bool)
    ms[selfp.reshape(-1)] = True
    assert np.array_equal(a.overlapping(), ms)
    # stream order: b's vertices refitted behind a long kernel on the caller's stream are what the pairs call sees
    w2 = shifted(w, 0.3)
    dv = torch_f(w2)
    stage = torch.zeros_like(dv)
    torch.cuda.synchronize()
    bits = torch.full(((n + 31) // 32,), -1, dtype=torch.int32, device="cuda")
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)
        stage.copy_(dv)
    s.synchronize()
    _lib.check(L().tbvh_refit(b.h, C.c_void_p(stage.data_ptr()), 16, w2.shape[0] // 3, _lib.DEVICE))
    want2, wbits2, _, _ = to.tree(*b.download(), w2, v)
    out = torch.full((want2.shape[0] + 1, 2), -1, dtype=torch.int32, device="cuda")
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)
        out.fill_(-2)   # queued behind the sleep: the pairs call must come after it
    cnt = C.c_uint64()
    _lib.check(L().tbvh_mesh_overlap_pairs(a.h, b.h, C.c_void_p(out.data_ptr()), out.shape[0], C.byref(cnt), _lib.DEVICE, C.c_void_p(s.cuda_stream)))
    s.synchronize()
    o = out.cpu().numpy().view(np.uint32)
    assert cnt.value == want2.shape[0] and np.array_equal(o[: cnt.value], want2), "pairs ordered after the caller's stream"
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)
        bits.fill_(-1)
        _lib.check(L().tbvh_mesh_overlap_bits(a.h, b.h, C.c_void_p(bits.data_ptr()), _lib.DEVICE, C.c_void_p(s.cuda_stream)))
    s.synchronize()
    assert np.array_equal(bits.cpu().numpy().view(np.uint32), wbits2), "bits queued on the caller's stream"


def test_refusals_leave_outputs_untouched(gpu):
    import torch
    v = soup(*icosphere(2))
    e = api.BVH().Build(v)
    n = v.shape[0] // 3
    out = torch.full((64, 2), -1, dtype=torch.int32, device="cuda")
    words = torch.full((n // 32 + 2,), -1, dtype=torch.int32, device="cuda")
    op, wp = C.c_void_p(out.data_ptr()), C.c_void_p(words.data_ptr())
    cnt = C.c_uint64(777)
    P = lambda a, b, o=op, cap=64, c=C.byref(cnt), space=_lib.DEVICE: L().tbvh_mesh_overlap_pairs(a, b, o, cap, c, space, None)  # noqa: E731
    B = lambda a, b, o=wp, space=_lib.DEVICE: L().tbvh_mesh_overlap_bits(a, b, o, space, None)  # noqa: E731
    n0 = api.launch_count()
    assert P(None, e.h) == _lib.E_ARG and P(e.h, None) == _lib.E_ARG
    assert P(e.h, e.h, o=None) == _lib.E_ARG
    assert P(e.h, e.h, c=None) == _lib.E_ARG
    assert P(e.h, e.h, space=7) == _lib.E_ARG
    assert P(e.h, e.h, o=C.c_void_p(out.data_ptr() + 4)) == _lib.E_ARG
    assert B(None, e.h) == _lib.E_ARG and B(e.h, e.h, o=None) == _lib.E_ARG and B(e.h, e.h, space=7) == _lib.E_ARG
    assert B(e.h, e.h, o=C.c_void_p(words.data_ptr() + 2)) == _lib.E_ARG
    other_ctx = C.c_void_p()
    _lib.check(L().tbvh_ctx_create(0, C.byref(other_ctx)))
    f = C.c_void_p()
    _lib.check(L().tbvh_bvh_create(other_ctx, C.byref(f)))
    vv = np.ascontiguousarray(v)
    _lib.check(L().tbvh_build(f, vv.ctypes.data, 16, n, _lib.HOST, 1.0, 1.0))
    assert P(e.h, f) == _lib.E_ARG and B(f, e.h) == _lib.E_ARG, "handles of different contexts"
    inst = np.zeros(2, api.BLAS_INSTANCE)
    inst["transform"] = np.eye(4, dtype=np.float32).reshape(-1)
    inst["mask"] = 0xFFFF
    t = api.TLAS()
    t.Build(inst, [e])
    assert P(t.h, e.h) == _lib.E_UNSUPPORTED and P(e.h, t.h) == _lib.E_UNSUPPORTED and B(e.h, t.h) == _lib.E_UNSUPPORTED
    assert P(api.BVH().h, e.h) == _lib.E_STATE and B(e.h, api.BVH().h) == _lib.E_STATE
    c = api.BVH8_CWBVH().Build(v)
    only = api.BVH8_CWBVH().upload(*c.download())
    assert P(only.h, e.h) == _lib.E_STATE and B(e.h, only.h) == _lib.E_STATE
    w = scenes.procedural_scene(300, 19)
    deep = chain_tree(w, 300)
    d = api.BVH().upload(deep[0], deep[1], w)
    assert P(e.h, d.h) == _lib.E_LIMIT and B(d.h, d.h) == _lib.E_LIMIT
    torch.cuda.synchronize()
    assert (out == -1).all() and (words == -1).all() and cnt.value == 777, "a refused call wrote its outputs"
    assert api.launch_count() >= n0
    k0 = api.launch_count()
    assert (P(t.h, e.h), P(e.h, d.h), B(only.h, e.h)) == (_lib.E_UNSUPPORTED, _lib.E_LIMIT, _lib.E_STATE)
    assert api.launch_count() == k0, "a refusal launched work"
    # one bits launch; the pairs call's launches: count, scan, fill, sort, unique, output
    k0 = api.launch_count()
    _lib.check(B(e.h, e.h))
    assert api.launch_count() - k0 == 1
    _lib.check(L().tbvh_bvh_destroy(f))
    _lib.check(L().tbvh_ctx_destroy(other_ctx))
