"""TBVH_BUILD_PLOC on the device against its host restatement (tests/ploc_oracle.c): nodes, primIdx and info byte for byte, indexed and
batched builds, the handle against an upload of the same arrays, and every downstream use of the tree (conversions, walks, refits,
tbvh_optimize, a TLAS, device views, a group replica)."""
import ctypes as C
import functools
from types import SimpleNamespace

import numpy as np
import pytest

from oracle import portpy
from tinybvh_b200 import _lib, api, scenes
from tests import util
from tests import optimize_oracle as oo
from tests import ploc_oracle as po
from tests.test_build_ploc import SCENES
from tests.test_device_api_gpu import consumer, device as device_walk, host_hits, to_device  # noqa: F401 (consumer: the fixture)

pytestmark = pytest.mark.gpu
ZERO = {"prim": 0, "t": 0, "u": 0, "v": 0}


def expo_scene(n, e0=0):
    """Triangles at doubling distances along x from 2^e0 on: every cluster's cheapest partner is the next triangle out, so the tree
    is a chain.  From the smallest subnormal (e0 = -149) 277 triangles reach 2^127 and a depth of 276."""
    x = np.ldexp(np.float32(1), np.arange(n) + e0).astype(np.float32)
    v = np.zeros((n * 3, 4), np.float32)
    v[0::3, 0], v[1::3, 0], v[2::3, 0], v[2::3, 1] = x, x * np.float32(1.01), x, 1
    return v


@functools.lru_cache(maxsize=None)
def oracle(name):
    v = SCENES[name] if name in SCENES else expo_scene(120) if name == "deep" else expo_scene(277, -149) if name == "deep255" else scenes.procedural_scene(int(name[5:]), 3)
    return v, po.build(v)


def node_bytes(nodes):
    return np.ascontiguousarray(nodes).view(np.uint8).tobytes()


def check_handle(e, v, want_nodes, want_idx):
    nodes, idx = e.download()
    assert node_bytes(nodes) == node_bytes(want_nodes)
    assert np.array_equal(idx, want_idx)
    i = e.info()
    ref = api.BVH().upload(want_nodes, want_idx, v).info()
    for f in ("used_nodes", "idx_count", "prim_count", "max_depth", "layouts"):
        assert getattr(i, f) == getattr(ref, f), f
    assert bytes(i.aabb_min) == bytes(ref.aabb_min) and bytes(i.aabb_max) == bytes(ref.aabb_max)
    assert i.build_ms > 0


@pytest.mark.parametrize("name", sorted(SCENES) + ["deep", "many_1048576"])
def test_matches_restatement(name):
    v, (nodes, idx, _, sah) = oracle(name)
    e = api.BVH().BuildPLOC(v)
    check_handle(e, v, nodes, idx)
    assert np.float32(e.SAHCost()) == sah or np.isnan(sah)
    if name == "deep":
        assert e.info().max_depth > 64 and e.device_view().stack == 256


def test_bistro_sized_scene():
    v = scenes.procedural_scene(2_840_000, 1)
    nodes, idx, _, _ = po.build(v)
    check_handle(api.BVH().BuildPLOC(v), v, nodes, idx)


def indexed_of(v):
    uniq, inv = np.unique(v.reshape(-1, 4), axis=0, return_inverse=True)
    return np.ascontiguousarray(uniq, np.float32), inv.astype(np.uint32).reshape(-1)


def test_indexed_equals_flat_and_refits():
    v = scenes.procedural_scene(20000, 13)
    uniq, ix = indexed_of(v)
    flat = np.ascontiguousarray(uniq[ix])
    a, b = api.BVH().BuildPLOC(uniq, indices=ix), api.BVH().BuildPLOC(flat)
    assert node_bytes(a.download()[0]) == node_bytes(b.download()[0]) and np.array_equal(a.download()[1], b.download()[1])
    moved = uniq.copy()
    moved[:, :3] += np.sin(np.arange(moved.shape[0], dtype=np.float32))[:, None] * 0.05
    mesh = (_lib.Mesh * 1)()
    mesh[0].verts, mesh[0].stride, mesh[0].prim_count, mesh[0].vert_count = moved.ctypes.data, 16, 20000, moved.shape[0]
    _lib.check(_lib.lib().tbvh_refit_batch_indexed((C.c_void_p * 1)(a.h), mesh, 1, api.HOST, 0))
    b.Refit(np.ascontiguousarray(moved[ix]))
    assert node_bytes(a.download()[0]) == node_bytes(b.download()[0])


def test_batches():
    names = ["seeded_3000", "seeded_1", "scaled_36", "scaled_-20", "signed_zero_order", "seeded_2", "atrium_3k", "long_leaf_identical"]
    vs = [oracle(n)[0] for n in names]
    for order in (list(range(len(names))), list(reversed(range(len(names)))), [3, 0, 6, 1, 7, 2, 5, 4]):
        es = [api.BVH() for _ in order]
        api.build_batch(es, [vs[k] for k in order], flavour=api.BUILD_PLOC)
        for e, k in zip(es, order):
            check_handle(e, vs[k], *oracle(names[k])[1][:2])
    # flat and indexed meshes in one call
    ms = [scenes.procedural_scene(n, 20 + n) for n in (500, 4000, 1)]
    u0, i0 = indexed_of(ms[0])
    es = [api.BVH() for _ in ms]
    api.build_batch(es, [u0, ms[1], ms[2]], flavour=api.BUILD_PLOC, indices=[i0, None, None])
    for e, m in zip(es, ms):
        nodes, idx, _, _ = po.build(m)
        check_handle(e, m, nodes, idx)


def download_cw(e):
    i = e.info()
    d = np.zeros((i.used_blocks, 4), np.float32)
    t = np.zeros((i.cwbvh_tri_count * 3, 4), np.float32)
    _lib.check(_lib.lib().tbvh_download_cwbvh(e.h, d.ctypes.data_as(C.c_void_p), t.ctypes.data_as(C.c_void_p), api.HOST))
    return d


def test_conversions_and_walks():
    v, (nodes, idx, _, _) = oracle("seeded_150000")
    o = portpy.PortBVH(v, nodes=nodes, prim_idx=idx)
    ocw = portpy.PortCWBVH(nodes, idx, v, idx_count=idx.shape[0])
    sets, bounds = util.ray_sets(v, res=48)
    ref = o.intersect(sets["primary"].copy())
    rays = {"primary": sets["primary"], **util.derived_sets(ref, v, bounds)}
    g = api.BVH_GPU()
    g.build_flavour = api.BUILD_PLOC
    g.Build(v)
    gn = np.zeros(g.info().used_nodes_gpu, portpy.NODE64)
    _lib.check(_lib.lib().tbvh_download_bvh_gpu(g.h, gn.ctypes.data_as(C.c_void_p), api.HOST))
    assert gn.tobytes() == o.to_bvh_gpu().tobytes()
    cw = api.BVH8_CWBVH()
    cw.build_flavour = api.BUILD_PLOC
    cw.Build(v)
    assert download_cw(cw).tobytes() == ocw.nodes.tobytes()
    # batch conversion
    es = [api.BVH().BuildPLOC(v), api.BVH().BuildPLOC(oracle("seeded_3000")[0])]
    hs = (C.c_void_p * 2)(*[e.h for e in es])
    _lib.check(_lib.lib().tbvh_convert_batch(hs, 2, api.LAYOUT_CWBVH))
    assert download_cw(es[0]).tobytes() == ocw.nodes.tobytes()
    b = api.BVH().BuildPLOC(v)
    build = portpy.PortBVH(v)
    for name, r in rays.items():
        want = o.intersect(r.copy())
        for e in (b, g):
            got = r.copy()
            e.Intersect(got)
            assert util.compare_hits(got, want) == ZERO, name
        got = r.copy()
        cw.Intersect(got)
        assert util.compare_hits(got, ocw.intersect(r.copy())) == ZERO, name
        assert np.array_equal(b.IsOccluded(r.copy()), o.occluded(r.copy())), name
        # the anchor: the Build tree of the same scene finds the same distances and occlusion bits
        assert np.array_equal(util.bits_u32(want["t"]), util.bits_u32(build.intersect(r.copy())["t"])), name
        assert np.array_equal(o.occluded(r.copy()), build.occluded(r.copy())), name


def test_refit_frames_and_optimize():
    v, (nodes, idx, _, _) = oracle("seeded_3000")
    e = api.BVH().BuildPLOC(v)
    e.Refit(v)
    assert node_bytes(e.download()[0]) == node_bytes(nodes), "a refit with the build's own vertices changes no byte"
    _lib.check(_lib.lib().tbvh_convert(e.h, api.LAYOUT_CWBVH))
    o = portpy.PortBVH(v, nodes=nodes, prim_idx=idx)
    for k in (1, 2):
        moved = np.array(v, np.float32)
        moved[:, :3] += np.cos(np.arange(moved.shape[0], dtype=np.float32) * k)[:, None] * 0.02
        o.refit(moved)
        _lib.check(_lib.lib().tbvh_refit_layouts(e.h, moved.ctypes.data_as(C.c_void_p), 16, moved.shape[0] // 3, api.HOST))
        assert node_bytes(api.BVH.download(e)[0]) == node_bytes(o.nodes)
    f = api.BVH().BuildPLOC(v)
    want, wr, wsah, _ = oo.optimize(nodes, idx, 4)
    assert f.optimize(4) == (wr, float(wsah))
    assert node_bytes(f.download()[0]) == node_bytes(want)


@pytest.mark.parametrize("layout", [api.LAYOUT_BVH, api.LAYOUT_CWBVH])
def test_tlas_over_ploc_blasses(layout):
    names = ("seeded_3000", "atrium_3k")
    vs = [oracle(n)[0] for n in names]
    bl = [api.BVH8_CWBVH() if layout == api.LAYOUT_CWBVH else api.BVH() for _ in vs]
    for b, v in zip(bl, vs):
        if layout == api.LAYOUT_CWBVH:
            b.build_flavour = api.BUILD_PLOC
            b.Build(v)
        else:
            b.BuildPLOC(v)
    inst = np.zeros(4, api.BLAS_INSTANCE)
    for i in range(4):
        m = np.eye(4, dtype=np.float32)
        m[:3, 3] = (i * 7.0, 0, i * 3.0)
        inst[i]["transform"], inst[i]["blasIdx"] = m.reshape(-1), i % 2
    tl = api.TLAS().Build(inst, bl, blas_layout=layout)   # Update()s the records in place
    sets, _ = util.ray_sets(np.concatenate(vs), res=16)
    got = sets["primary"].copy()
    tl.Intersect(got)
    tn, ti = tl.download()
    if layout == api.LAYOUT_BVH:
        o = portpy.PortTLAS(tn, ti, inst, [portpy.PortBVH(v, nodes=oracle(n)[1][0], prim_idx=oracle(n)[1][1]) for v, n in zip(vs, names)])
    else:
        o = portpy.PortTLASCW(tn, ti, inst, [portpy.PortCWBVH(oracle(n)[1][0], oracle(n)[1][1], v, idx_count=oracle(n)[1][1].shape[0]) for v, n in zip(vs, names)])
    assert util.compare_hits(got, o.intersect(sets["primary"].copy())) == ZERO
    assert np.array_equal(tl.IsOccluded(sets["primary"].copy()), o.occluded(sets["primary"].copy()))


@pytest.mark.parametrize("layout", [api.LAYOUT_BVH, api.LAYOUT_CWBVH])
def test_device_view_walks(consumer, layout):
    """The caller-kernel walks (tbvh_device_view) of a PLOC tree give the oracle's hits and occlusion bits of the same tree."""
    v, (nodes, idx, _, _) = oracle("seeded_3000")
    if layout == api.LAYOUT_BVH:
        e, o = api.BVH().BuildPLOC(v), portpy.PortBVH(v, nodes=nodes, prim_idx=idx)
    else:
        e = api.BVH8_CWBVH()
        e.build_flavour = api.BUILD_PLOC
        e.Build(v)
        o = portpy.PortCWBVH(nodes, idx, v, idx_count=idx.shape[0])
    sets, _ = util.ray_sets(v, res=32)
    r = sets["primary"]
    got, bits, _, _ = device_walk(consumer, e.device_view(layout), to_device(r))
    want = o.intersect(r.copy())
    assert util.compare_hits(host_hits(got, r), want) == ZERO
    if layout == api.LAYOUT_BVH:
        want_bits = o.occluded(r.copy())
    else:   # the CWBVH any-hit query is the closest-hit walk ending below the ray's t (FALLBACK_SHADOW_QUERY)
        hit = np.zeros(((r.shape[0] + 31) // 32) * 32, bool)
        hit[: r.shape[0]] = want["t"] < r["t"]
        want_bits = (hit.reshape(-1, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(1).astype(np.uint32)
    assert np.array_equal(bits.view(np.uint32), want_bits)


def test_group_replica():
    v, (nodes, idx, _, _) = oracle("seeded_3000")
    e = api.BVH().BuildPLOC(v)
    g = api.Group([0, 0])
    try:
        g.replicate(e)
        sets, _ = util.ray_sets(v, res=16)
        r = sets["primary"].copy()
        g.Intersect(r)
        assert util.compare_hits(r, portpy.PortBVH(v, nodes=nodes, prim_idx=idx).intersect(sets["primary"].copy())) == ZERO
    finally:
        g.close()


def test_deeper_than_255():
    """A PLOC tree 276 levels deep (the restatement says so): its BVH2 walks are refused with TBVH_E_LIMIT before a launch, as for an
    upload of the same depth, while its CWBVH converts and walks.  As for deep uploads (tests/test_deep_bvh2_gpu.py), the reference's
    SplitLeafs stack holds 64 entries, so the restatement's converter is not run on this tree; the device walk is held to the
    restatement's BVH8_CWBVH::Intersect over the downloaded bytes."""
    from tinybvh_b200 import rays as R
    v, (nodes, idx, _, _) = oracle("deep255")
    assert util.tree_depth(nodes) > 255
    e = api.BVH().BuildPLOC(v)
    check_handle(e, v, nodes, idx)
    assert e.info().max_depth == util.tree_depth(nodes)
    # one ray down onto every triangle, inside it: (x + x / 1024, 0.5) lies in the triangle (x, 0), (1.01 x, 0), (x, 1)
    x = v[0::3, 0]
    o = np.stack([x + x / np.float32(1024), np.full_like(x, 0.5), np.ones_like(x)], 1)
    d = np.tile(np.array([[0, 0, -1]], np.float32), (x.shape[0], 1))
    r = R.make_rays(o, d)
    L = _lib.lib()
    h = r.copy()
    assert L.tbvh_intersect(e.h, api.LAYOUT_BVH, h.ctypes.data_as(C.c_void_p), 128, h.shape[0]) == -4
    assert h.tobytes() == r.tobytes()
    bits = np.zeros((r.shape[0] + 31) // 32, np.uint32)
    assert L.tbvh_occluded(e.h, api.LAYOUT_BVH, h.ctypes.data_as(C.c_void_p), 128, h.shape[0], bits.ctypes.data_as(C.c_void_p)) == -4
    _lib.check(L.tbvh_convert(e.h, api.LAYOUT_CWBVH))
    i = e.info()
    d8 = np.zeros((i.used_blocks, 4), np.float32)
    t8 = np.zeros((i.cwbvh_tri_count * 3, 4), np.float32)
    _lib.check(L.tbvh_download_cwbvh(e.h, d8.ctypes.data_as(C.c_void_p), t8.ctypes.data_as(C.c_void_p), api.HOST))
    want = r.copy()
    portpy.PortCWBVH.intersect(SimpleNamespace(nodes=d8, tris=t8), want)
    got = r.copy()
    _lib.check(L.tbvh_intersect(e.h, api.LAYOUT_CWBVH, got.ctypes.data_as(C.c_void_p), 128, got.shape[0]))
    assert util.compare_hits(got, want) == ZERO
    hit = want["t"] == 1   # a ray that hits, hits its own triangle
    assert np.array_equal(want["prim"][hit], np.nonzero(hit)[0])


def test_refused_build_leaves_handle_and_tlas():
    v = scenes.procedural_scene(3000, 4)
    e = api.BVH().BuildPLOC(v)
    before = node_bytes(e.download()[0])
    inst = np.zeros(1, api.BLAS_INSTANCE)
    inst["transform"] = np.eye(4, dtype=np.float32).reshape(-1)
    tl = api.TLAS().Build(inst, [e])
    sets, _ = util.ray_sets(v, res=16)
    hits_before = tl.Intersect(sets["primary"].copy())
    rc = _lib.lib().tbvh_build_flavour(e.h, v.ctypes.data_as(C.c_void_p), 14, 3000, api.HOST, 1.0, 1.0, api.BUILD_PLOC)
    assert rc == -2
    bad = np.full(9, 10**6, np.uint32)
    rc = _lib.lib().tbvh_build_indexed(e.h, v.ctypes.data_as(C.c_void_p), 16, 9000, bad.ctypes.data_as(C.c_void_p), 3, api.HOST, 1.0, 1.0, api.BUILD_PLOC)
    assert rc == -2
    assert node_bytes(e.download()[0]) == before
    # the TLAS is not stale (a stale one refuses every walk) and finds what it found before
    hits_after = sets["primary"].copy()
    _lib.check(_lib.lib().tbvh_intersect(tl.h, api.LAYOUT_BVH, hits_after.ctypes.data_as(C.c_void_p), 128, hits_after.shape[0]))
    assert util.compare_hits(hits_after, hits_before) == ZERO
    # a successful rebuild makes it stale
    e.BuildPLOC(v)
    r = sets["primary"].copy()
    assert _lib.lib().tbvh_intersect(tl.h, api.LAYOUT_BVH, r.ctypes.data_as(C.c_void_p), 128, r.shape[0]) == -3
