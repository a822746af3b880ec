"""tbvh_optimize on the device against its host restatement (tests/optimize_oracle.c): the optimised nodes byte for byte, the handle's
bookkeeping, every downstream use of the optimised tree (walks, conversions, refits, a TLAS, a group replica), and the refusals."""
import ctypes as C
import functools

import numpy as np
import pytest

from oracle import portpy
from tinybvh_b200 import _lib, api, scenes
from tests import util
from tests import optimize_oracle as oo
from tests.cwbvh_refit_oracle import RefitCWBVH

pytestmark = pytest.mark.gpu
ZERO = {"prim": 0, "t": 0, "u": 0, "v": 0}
ROUNDS = 6
CASES = [(b, n, f) for b in ("Build", "BuildAVX", "BuildHQ") for n in (1, 2, 5, 3000) for f in ("src", "B")]
CASES += [(b, 3000, f) for b in ("Build", "BuildHQ") for f in ("A0.3", "A1", "C0", "C3", "DA", "DB", "DC")]
CASES += [("Build", 3000, "deep"), ("Build", 3000, "deep255"), ("BuildAVX", 150000, "src"), ("BuildHQ", 150000, "src"), ("Build", 400000, "src")]
IDS = [f"{b}-{n}-{f}" for b, n, f in CASES]


@functools.lru_cache(maxsize=None)
def case(builder, ntris, fam):
    v = scenes.procedural_scene(ntris, 41 + ntris % 5)
    src = util.source_tree(v, builder)
    if fam == "src":
        t = src
    elif fam.startswith("deep"):
        t = util.reinserted(src, 3, 50, grow_to=int(fam[4:] or 100))   # deep255: L = 255, the search stack's bound
    else:
        t = util.family_tree(src, fam, 23)
    rounds = 2 if ntris >= 100000 else ROUNDS
    return v, t, rounds, oo.optimize(t[0], t[1], rounds)


@pytest.fixture(scope="module", autouse=True)
def _free_cases():
    yield
    case.cache_clear()


def optimize_raw(h, rounds, c_trav=1.0, c_int=1.0):
    r, s = C.c_uint32(), C.c_float()
    rc = _lib.lib().tbvh_optimize(h, rounds, c_trav, c_int, C.byref(r), C.byref(s))
    return rc, int(r.value), np.float32(s.value)


def uploaded(v, t):
    return api.BVH().upload(t[0], t[1], v)


def node_bytes(nodes):
    return np.ascontiguousarray(nodes).view(np.uint8).tobytes()


@pytest.mark.parametrize("builder,ntris,fam", CASES, ids=IDS)
def test_matches_restatement(builder, ntris, fam):
    v, t, rounds, (want, wr, wsah, _) = case(builder, ntris, fam)
    e = uploaded(v, t)
    before = e.info()
    r, sah = e.optimize(rounds)
    assert (r, np.float32(sah)) == (wr, wsah)
    nodes, idx = e.download()
    assert node_bytes(nodes) == node_bytes(want)
    assert np.array_equal(idx, t[1])
    assert np.float32(e.SAHCost()) == wsah
    i = e.info()
    assert (i.prim_count, i.idx_count, i.layouts) == (before.prim_count, before.idx_count, 1 << api.LAYOUT_BVH)
    ref = uploaded(v, (nodes, idx, t[2])).info()
    for f in ("used_nodes", "max_depth"):
        assert getattr(i, f) == getattr(ref, f), f
    assert list(i.aabb_min) == list(ref.aabb_min) and list(i.aabb_max) == list(ref.aabb_max)
    if wr:
        assert i.build_ms > 0
        assert e.device_view().stack == (256 if i.max_depth + 1 > 64 else 64)


@pytest.mark.parametrize("builder", ["Build", "BuildAVX", "BuildHQ"])
def test_builds_on_device(builder):
    """A tree built on the device (flat and indexed) optimises to what the restatement makes of its downloaded bytes."""
    v = scenes.procedural_scene(20000, 5)
    for indexed in (False, True):
        e = api.BVH()
        if indexed:
            flat = v.reshape(-1, 4)
            uniq, inv = np.unique(flat, axis=0, return_inverse=True)
            getattr(e, builder)(np.ascontiguousarray(uniq, np.float32), indices=inv.astype(np.uint32).reshape(-1))
        else:
            getattr(e, builder)(v)
        nodes, idx = e.download()
        want, wr, wsah, _ = oo.optimize(nodes, idx, 4)
        assert e.optimize(4) == (wr, float(wsah))
        got, gidx = e.download()
        assert node_bytes(got) == node_bytes(want) and np.array_equal(gidx, idx)


def test_batch_built_trees():
    vs = [scenes.procedural_scene(n, 9 + n) for n in (500, 4000, 20000)]
    es = [api.BVH() for _ in vs]
    api.build_batch(es, vs)
    for e in es:
        nodes, idx = e.download()
        want, wr, wsah, _ = oo.optimize(nodes, idx, 3)
        assert e.optimize(3) == (wr, float(wsah))
        assert node_bytes(e.download()[0]) == node_bytes(want)


def test_max_rounds_and_no_change():
    v, t, _, _ = case("Build", 3000, "B")
    for k in (1, 2):
        e = uploaded(v, t)
        want, wr, wsah, _ = oo.optimize(t[0], t[1], k)
        assert e.optimize(k) == (wr, float(wsah)) and wr <= k
        assert node_bytes(e.download()[0]) == node_bytes(want)
    # a tree of two leaves offers no move: the handle keeps its bytes, its layouts and its generation (a TLAS over it stays valid)
    v2 = scenes.procedural_scene(2, 3)
    b = api.BVH8_CWBVH().Build(v2)
    info = b.info()
    inst = np.zeros(1, api.BLAS_INSTANCE)
    inst["transform"] = np.eye(4, dtype=np.float32).reshape(-1)
    tl = api.TLAS().Build(inst, [b], blas_layout=api.LAYOUT_CWBVH)
    rc, r, s = optimize_raw(b.h, 5)
    assert (rc, r) == (0, 0)
    assert b.info().layouts == info.layouts
    sets, _ = util.ray_sets(v2, res=8)
    tl.Intersect(sets["primary"].copy())


def test_walks_and_conversions():
    v, t, rounds, (want, wr, wsah, _) = case("Build", 3000, "B")
    assert wr > 0
    o_before = portpy.PortBVH(v, nodes=t[0], prim_idx=t[1])
    o_after = portpy.PortBVH(v, nodes=want, prim_idx=t[1])
    sets, bounds = util.ray_sets(v, res=32)
    ref = o_after.intersect(sets["primary"].copy())
    pre = o_before.intersect(sets["primary"].copy())
    assert np.array_equal(util.bits_u32(ref["t"]), util.bits_u32(pre["t"]))
    derived = util.derived_sets(ref, v, bounds)
    e = uploaded(v, t)
    e.optimize(rounds)
    got = sets["primary"].copy()
    e.Intersect(got)
    assert util.compare_hits(got, ref) == ZERO
    for name, r in derived.items():
        w = o_after.intersect(r.copy())
        g = r.copy()
        e.Intersect(g)
        assert util.compare_hits(g, w) == ZERO, name
        assert np.array_equal(e.IsOccluded(r.copy()), o_after.occluded(r.copy())), name
        assert np.array_equal(e.IsOccluded(r.copy()), o_before.occluded(r.copy())), name
    # BVH_GPU and CWBVH of the optimised tree: the conversions of the restatement's tree, and their walks
    e2 = uploaded(v, t)
    e2.optimize(rounds)
    _lib.check(_lib.lib().tbvh_convert(e2.h, api.LAYOUT_BVH_GPU))
    gn = np.zeros(e2.info().used_nodes_gpu, portpy.NODE64)
    _lib.check(_lib.lib().tbvh_download_bvh_gpu(e2.h, gn.ctypes.data_as(C.c_void_p), api.HOST))
    assert gn.tobytes() == o_after.to_bvh_gpu().tobytes()
    _lib.check(_lib.lib().tbvh_convert(e2.h, api.LAYOUT_CWBVH))
    ocw = portpy.PortCWBVH(want, t[1], v, idx_count=t[2])
    d = np.zeros((e2.info().used_blocks, 4), np.float32)
    tr = np.zeros((e2.info().cwbvh_tri_count * 3, 4), np.float32)
    _lib.check(_lib.lib().tbvh_download_cwbvh(e2.h, d.ctypes.data_as(C.c_void_p), tr.ctypes.data_as(C.c_void_p), api.HOST))
    assert d.tobytes() == ocw.nodes.tobytes()
    got = sets["primary"].copy()
    _lib.check(_lib.lib().tbvh_intersect(e2.h, api.LAYOUT_CWBVH, got.ctypes.data_as(C.c_void_p), got.dtype.itemsize, got.shape[0]))
    w = ocw.intersect(sets["primary"].copy())
    assert util.compare_hits(got, w) == ZERO


def test_refit_after_optimize():
    """An indexed BuildAVX tree keeps its indices and stays refittable: refits of the optimised tree equal orc_refit of it."""
    v = scenes.procedural_scene(20000, 13)
    flat = v.reshape(-1, 4)
    uniq, inv = np.unique(flat, axis=0, return_inverse=True)
    uniq = np.ascontiguousarray(uniq, np.float32)
    idx3 = inv.astype(np.uint32).reshape(-1)
    e = api.BVH().BuildAVX(uniq, indices=idx3)
    r, _ = e.optimize(4)
    assert r > 0
    nodes, pidx = e.download()
    moved = uniq.copy()
    moved[:, :3] += np.sin(np.arange(moved.shape[0], dtype=np.float32))[:, None] * 0.05
    o = portpy.PortBVH(moved[idx3], nodes=nodes, prim_idx=pidx)
    o.refit(moved[idx3])
    e.Refit(np.ascontiguousarray(moved[idx3]))
    assert node_bytes(e.download()[0]) == node_bytes(o.nodes)
    e2 = api.BVH().BuildAVX(uniq, indices=idx3)
    e2.optimize(4)
    mesh = (_lib.Mesh * 1)()
    mesh[0].verts, mesh[0].stride, mesh[0].prim_count, mesh[0].vert_count = moved.ctypes.data, 16, 20000, moved.shape[0]
    hs = (C.c_void_p * 1)(e2.h)
    _lib.check(_lib.lib().tbvh_refit_batch_indexed(hs, mesh, 1, api.HOST, 0))
    assert node_bytes(e2.download()[0]) == node_bytes(o.nodes)
    # tbvh_refit_layouts needs the collapse of a conversion: optimising drops the CWBVH, converting again keeps the new collapse
    e3 = api.BVH().BuildAVX(uniq, indices=idx3)
    e3.optimize(4)
    _lib.check(_lib.lib().tbvh_convert(e3.h, api.LAYOUT_CWBVH))
    flat_moved = np.ascontiguousarray(moved[idx3])
    _lib.check(_lib.lib().tbvh_refit_layouts(e3.h, flat_moved.ctypes.data_as(C.c_void_p), 16, 20000, api.HOST))
    assert node_bytes(api.BVH.download(e3)[0]) == node_bytes(o.nodes)
    want = RefitCWBVH(nodes, o.nodes, pidx, flat_moved)
    i = e3.info()
    d = np.zeros((i.used_blocks, 4), np.float32)
    tr = np.zeros((i.cwbvh_tri_count * 3, 4), np.float32)
    _lib.check(_lib.lib().tbvh_download_cwbvh(e3.h, d.ctypes.data_as(C.c_void_p), tr.ctypes.data_as(C.c_void_p), api.HOST))
    assert d.tobytes() == want.nodes.tobytes()


def test_tlas_goes_stale_then_matches():
    vs = [scenes.procedural_scene(3000, s) for s in (1, 2)]
    bl = [api.BVH().Build(v) for v in vs]
    inst = np.zeros(6, api.BLAS_INSTANCE)
    for i in range(6):
        m = np.eye(4, dtype=np.float32)
        m[:3, 3] = (i * 7.0, 0, i * 3.0)
        inst[i]["transform"], inst[i]["blasIdx"] = m.reshape(-1), i % 2
    tl = api.TLAS().Build(inst.copy(), bl)
    for b in bl:
        b.optimize(4)
    sets, _ = util.ray_sets(np.concatenate(vs), res=16)
    with pytest.raises(_lib.TbvhError):
        tl.Intersect(sets["primary"].copy())
    inst2 = inst.copy()
    tl.Build(inst2, bl)
    got = sets["primary"].copy()
    tl.Intersect(got)
    blas_o = [portpy.PortBVH(v, nodes=b.download()[0], prim_idx=b.download()[1]) for v, b in zip(vs, bl)]
    want = portpy.PortTLAS(tl.download()[0], tl.download()[1], inst2, blas_o).intersect(sets["primary"].copy())
    assert util.compare_hits(got, want) == ZERO


def test_refusals_leave_the_handle():
    v = scenes.procedural_scene(3000, 4)
    e = api.BVH().Build(v)
    before = node_bytes(e.download()[0])
    assert optimize_raw(None, 4)[0] == -2
    for args in ((0, 1.0, 1.0), (4, 0.0, 1.0), (4, 1.0, -1.0), (4, float("nan"), 1.0), (4, 1.0, float("inf"))):
        assert optimize_raw(e.h, *args)[0] == -2, args
    assert node_bytes(e.download()[0]) == before
    assert optimize_raw(api.BVH().h, 4)[0] == -3   # an empty handle
    cw = api.BVH8_CWBVH()
    d, t = api.BVH8_CWBVH().Build(v).download()
    cw.upload(d, t)
    assert optimize_raw(cw.h, 4)[0] == -3          # a CWBVH-only upload
    src = util.source_tree(v, "Build")
    g = api.BVH_GPU().upload(portpy.PortBVH(v, nodes=src[0], prim_idx=src[1]).to_bvh_gpu(), src[1], v)
    assert optimize_raw(g.h, 4)[0] == -3           # a BVH_GPU-only upload holds no BVH-layout tree
    # an upload whose node array holds slots outside the tree: two unreferenced slots after the tree, or node 1 in it
    extra = np.concatenate([src[0], src[0][-2:]])
    u = uploaded(v, (extra, src[1], src[2]))
    ub = node_bytes(u.download()[0])
    assert optimize_raw(u.h, 4)[0] == -3 and node_bytes(u.download()[0]) == ub
    swapped = src[0].copy()
    swapped[1], swapped[0]["leftFirst"] = swapped[2], 1   # the root's children at 1 and 2: node 1 in the tree, slot 3 outside it
    u1 = uploaded(v, (swapped, src[1], src[2]))
    assert optimize_raw(u1.h, 4)[0] == -3
    # deeper than the search's 255 levels
    deep = util.reinserted(src, 3, 50, grow_to=256)
    assert util.tree_depth(deep[0]) == 256
    ud = uploaded(v, deep)
    db = node_bytes(ud.download()[0])
    assert optimize_raw(ud.h, 4)[0] == -4 and node_bytes(ud.download()[0]) == db
    inst = np.zeros(2, api.BLAS_INSTANCE)
    inst["transform"] = np.eye(4, dtype=np.float32).reshape(-1)
    tl = api.TLAS().Build(inst, [e])
    tb = node_bytes(tl.download()[0])
    assert optimize_raw(tl.h, 4)[0] == -3          # a TLAS
    assert node_bytes(tl.download()[0]) == tb and node_bytes(e.download()[0]) == before


def test_group_replica_of_optimised_tree():
    if api.device_count() < 1:
        pytest.skip("no device")
    v, t, rounds, (want, wr, wsah, _) = case("BuildHQ", 3000, "src")
    e = uploaded(v, t)
    e.optimize(rounds)
    g = api.Group([0, 0])
    try:
        g.replicate(e)
        sets, _ = util.ray_sets(v, res=16)
        r = sets["primary"].copy()
        g.Intersect(r)
        w = portpy.PortBVH(v, nodes=want, prim_idx=t[1]).intersect(sets["primary"].copy())
        assert util.compare_hits(r, w) == ZERO
    finally:
        g.close()
