"""GPU parity of tbvh_convert_batch / api.convert_batch: many BVH-layout trees converted to CWBVH in one call, every handle exactly what
tbvh_convert of it alone leaves - bytes, info, traversal limits, the kept collapse - whatever the order and neighbours of its tree in
the batch, and every later call (walks, refit, TLAS, group replicas) working unchanged on batch-converted handles."""
import ctypes as C

import numpy as np
import pytest

from oracle import portpy
from tinybvh_b200 import _lib, api, rays as R, scenes
from tests import util
from tests.test_oracle_pin import tlas_case

pytestmark = pytest.mark.gpu

FLAVOURS = {"Build": _lib.BUILD_REFERENCE, "BuildAVX": _lib.BUILD_AVX, "BuildHQ": _lib.BUILD_HQ}
ORACLE_MODE = {"Build": 2, "BuildAVX": 0, "BuildHQ": 1}   # util.oracle_cwbvh: the conversion chain over that builder's tree
MIXED = [1, 2, 3, 4, 31, 128, 129, 257, 1000, 5000, 70000]


def mesh(n, seed):
    return scenes.procedural_scene(n, seed)


def built(v, name):
    b = api.BVH()
    b._build(v, 0, FLAVOURS[name])
    return b


def uploaded(tree, v):
    nodes, idx, _ = tree
    return api.BVH().upload(nodes, idx, v)


def convert(b):
    api.check(_lib.lib().tbvh_convert(b.h, api.LAYOUT_CWBVH))
    return b


def raw_batch(handles, layout=api.LAYOUT_CWBVH):
    hs = (C.c_void_p * max(len(handles), 1))(*handles)
    return _lib.lib().tbvh_convert_batch(hs, len(handles), layout)


def referenced(b):
    """bvh8Tris records the leaves reference (an SBVH's tail beyond them is left uninitialised, as the reference leaves it)."""
    nodes, _ = b.download()
    return int(nodes["triCount"][np.arange(nodes.shape[0]) != 1].sum()) * 3


def cw(b):
    i = b.info()
    d = np.zeros((i.used_blocks, 4), np.float32)
    t = np.zeros((i.cwbvh_tri_count * 3, 4), np.float32)
    api.check(_lib.lib().tbvh_download_cwbvh(b.h, d.ctypes.data, t.ctypes.data, api.HOST))
    return d.view(np.uint32), t.view(np.uint32)[: referenced(b)]


def info(b):
    return bytes(b.info())[:_lib.Info.build_ms.offset]   # every field but build_ms


def assert_same(got, want, what):
    for k, (g, w) in enumerate(zip(got, want)):
        gd, gt = cw(g)
        wd, wt = cw(w)
        assert np.array_equal(gd, wd) and np.array_equal(gt, wt), f"{what}: the CWBVH of tree {k} differs from its own conversion"
        assert info(g) == info(w), f"{what}: info of tree {k} differs"


def walk(b, v, seed=0):
    """Camera, shadow and incoherent rays through the handle's CWBVH -> (closest-hit records, shadow occlusion words)."""
    b.layout = api.LAYOUT_CWBVH
    sets, bounds = util.ray_sets(v, res=24, seed=seed)
    prim = sets["primary"].copy()
    b.Intersect(prim)
    d = util.derived_sets(prim, v, bounds)
    diffuse = d["diffuse"].copy()
    b.Intersect(diffuse)
    return np.concatenate([prim, diffuse]), b.IsOccluded(d["shadow"])


def assert_same_walks(got, want, meshes, what):
    for k, (g, w, v) in enumerate(zip(got, want, meshes)):
        gh, gb = walk(g, v, k)
        wh, wb = walk(w, v, k)
        assert util.compare_hits(util.nan_canonical(gh), util.nan_canonical(wh)) == {"prim": 0, "t": 0, "u": 0, "v": 0}, f"{what}: hits of tree {k}"
        assert np.array_equal(gb, wb), f"{what}: occlusion words of tree {k}"


@pytest.mark.parametrize("name", ["Build", "BuildAVX", "BuildHQ"])
def test_mixed_sizes_match_single_conversions_and_oracle(gpu, name):
    meshes = [mesh(n, 800 + k) for k, n in enumerate(MIXED)]
    want = [convert(built(v, name)) for v in meshes]
    for k in (0, 3, 6, 9):
        o, used = util.oracle_cwbvh(meshes[k], ORACLE_MODE[name])
        wd, wt = cw(want[k])
        assert np.array_equal(wd, np.ascontiguousarray(o.nodes).view(np.uint32).reshape(wd.shape)), f"single conversion of mesh {k} differs from the oracle"
        assert np.array_equal(wt[:used], np.ascontiguousarray(o.tris).view(np.uint32).reshape(-1, 4)[:used])
    sources = {"separately built": lambda vs: [built(v, name) for v in vs]}
    if name != "BuildHQ":
        sources["batch-built"] = lambda vs: api.build_batch([api.BVH() for _ in vs], vs, FLAVOURS[name])
    rng = np.random.default_rng(3)
    for label, make in sources.items():
        for order in (list(range(len(meshes))), list(range(len(meshes)))[::-1], list(rng.permutation(len(meshes)))):
            got = api.convert_batch(make([meshes[k] for k in order]))
            assert_same(got, [want[k] for k in order], f"{name}, {label}, order {order}")
            assert all(g.info().layouts == (1 << api.LAYOUT_BVH) | (1 << api.LAYOUT_CWBVH) for g in got)
    assert_same_walks(got, [want[k] for k in order], [meshes[k] for k in order], name)


def offatrium_meshes():
    base = mesh(3000, 31)
    out = [("plain", mesh(2500, 32)), ("plain small", mesh(90, 33))]
    for mode in ("pos", "neg", "random", "order"):
        out.append((f"signed zero {mode}", util.signed_zero(base, mode, seed=3)))
    for k in (-126, -20, 40, 90):
        out.append((f"scaled 2^{k}", util.scaled(base, k)))
    out.append(("translated", util.translated(base, 3e5)))
    return out


def test_offatrium_neighbours(gpu):
    """Signed zeros, extreme scales and far translations next to plain meshes: each tree is its own conversion, and a 2^90 tree's
    exponents change nothing for its neighbour's integer-path bound."""
    named = offatrium_meshes()
    meshes = [v for _, v in named]
    got = api.convert_batch([built(v, "Build") for v in meshes])
    want = [convert(built(v, "Build")) for v in meshes]
    for k, (label, _) in enumerate(named):
        assert_same([got[k]], [want[k]], label)
    assert_same_walks(got, want, meshes, "off-atrium")
    plain, big = meshes[0], meshes[[label for label, _ in named].index("scaled 2^90")]
    pair = api.convert_batch([built(plain, "Build"), built(big, "Build")])
    for b, v in zip(pair, (plain, big)):
        o, _ = util.oracle_cwbvh(v, 2)
        lo, hi = scenes.scene_bounds(v)
        sets, _ = util.ray_sets(v, res=16)
        rays = np.concatenate([util.rd_limit_rays(sets["primary"], util.cw_rd_limit(o.nodes)), util.axis_rays(lo, hi)])
        want_r, got_r = rays.copy(), rays.copy()
        o.intersect(want_r)
        b.layout = api.LAYOUT_CWBVH
        b.Intersect(got_r)
        assert util.compare_hits(util.nan_canonical(got_r), util.nan_canonical(want_r)) == {"prim": 0, "t": 0, "u": 0, "v": 0}


def test_uploaded_families_and_long_leaves(gpu):
    v = mesh(4000, 41)
    src = util.source_tree(v, "Build")
    trees = [(f"family {fam}", util.family_tree(src, fam, 5 + k), v) for k, fam in enumerate(util.FAMILIES)]
    for name in ("identical", "clusters", "collapsed"):
        lv = util.long_leaf_scene(name)
        trees.append((name, util.source_tree(lv, "Build"), lv))
    plain = [("plain", None, mesh(n, 900 + n)) for n in (7, 300, 20000)]
    items = plain[:1] + trees[:5] + plain[1:2] + trees[5:] + plain[2:]
    make = [(lambda t=t, x=x: uploaded(t, x) if t is not None else built(x, "Build")) for _, t, x in items]
    got = api.convert_batch([m() for m in make])
    want = [convert(m()) for m in make]
    for k, (label, _, _) in enumerate(items):
        assert_same([got[k]], [want[k]], label)
        if label in ("identical", "clusters", "collapsed") or label.startswith("family"):
            assert util.cw_depth_and_pending(cw(got[k])[0].view(np.float32)) == util.cw_depth_and_pending(cw(want[k])[0].view(np.float32)), label
    assert_same_walks(got, want, [x for _, _, x in items], "uploaded")


def test_refit_after_batch(gpu):
    meshes = [mesh(n, 60 + k) for k, n in enumerate([3, 50, 129, 6000, 30000])]
    got = api.convert_batch([built(v, "Build") for v in meshes] + [built(meshes[3], "BuildHQ")])
    want = [convert(built(v, "Build")) for v in meshes]
    for k, v in enumerate(meshes):
        moved = v.copy()
        moved[:, :3] += np.float32(0.25) * np.sin(np.arange(moved.shape[0], dtype=np.float32))[:, None]
        for b in (got[k], want[k]):
            api._refit_layouts(b, moved)
        assert_same([got[k]], [want[k]], f"refit of mesh {k}")
        gn, wn = got[k].download()[0], want[k].download()[0]
        assert np.array_equal(gn.view(np.uint32), wn.view(np.uint32))
    assert _lib.lib().tbvh_refit_layouts(got[-1].h, meshes[3].ctypes.data, 16, meshes[3].shape[0] // 3, api.HOST) == _lib.E_STATE   # an SBVH


def tlas_words(r):
    return r.view(np.uint32).reshape(-1, 32)[:, 11:16]   # hit.inst, t, u, v, prim


def test_tlas_over_batch_converted_blasses(gpu):
    v, inst, O, D = tlas_case(107, 40)
    blas = api.convert_batch([built(x, "Build") for x in v])
    t = api.TLAS().Build(inst, blas, blas_layout=api.LAYOUT_CWBVH)
    nodes, idx = t.download()

    class _CW:
        def __init__(self, b):
            self.nodes, self.tris = (a.view(np.float32) for a in cw(b))

    port = portpy.PortTLASCW(nodes, idx, inst, [_CW(b) for b in blas])
    rays = R.make_rays(O, D)
    want, got = rays.copy(), rays.copy()
    port.intersect(want), t.Intersect(got)
    assert np.array_equal(tlas_words(got), tlas_words(want)) and (want["t"] < 1e30).sum() > 1000
    sh = R.make_rays(O, D, tmax=150.0)
    assert np.array_equal(t.IsOccluded(sh), port.occluded(sh))
    # a TLAS handle is refused, alone or in a batch, before anything changes
    before = [cw(b) for b in blas[:2]]
    assert _lib.lib().tbvh_convert(t.h, api.LAYOUT_CWBVH) == _lib.E_STATE
    assert raw_batch([blas[0].h.value, t.h.value, blas[1].h.value]) == _lib.E_STATE
    for b, (d, tr) in zip(blas[:2], before):
        gd, gt = cw(b)
        assert np.array_equal(gd, d) and np.array_equal(gt, tr)
    got = rays.copy()
    t.Intersect(got)
    assert np.array_equal(tlas_words(got), tlas_words(want))
    # a batch that converts one of its BLASses again makes the TLAS stale
    api.convert_batch([blas[-1], built(v[0], "Build")])
    assert _lib.lib().tbvh_intersect(t.h, api.LAYOUT_CWBVH, got.ctypes.data, 128, 64) == _lib.E_STATE


def test_refusals_leave_handles_as_they_were(gpu):
    v, inst, O, D = tlas_case(109, 12)
    blas = api.convert_batch([built(x, "Build") for x in v])
    t = api.TLAS().Build(inst, blas, blas_layout=api.LAYOUT_CWBVH)
    rays = R.make_rays(O, D)
    want = rays.copy()
    t.Intersect(want)
    before = [cw(b) for b in blas]
    h = [b.h.value for b in blas]
    empty = api.BVH()
    only_cw = api.BVH8_CWBVH().upload(*(a.view(np.float32) for a in before[0]))
    ctx2 = C.c_void_p()
    api.check(_lib.lib().tbvh_ctx_create(0, C.byref(ctx2)))
    other = C.c_void_p()
    api.check(_lib.lib().tbvh_bvh_create(ctx2, C.byref(other)))
    try:
        cases = [("count 0", [], api.LAYOUT_CWBVH, _lib.E_ARG), ("NULL handle", [h[0], None], api.LAYOUT_CWBVH, _lib.E_ARG),
                 ("repeated handle", [h[0], h[1], h[0]], api.LAYOUT_CWBVH, _lib.E_ARG), ("two contexts", [h[0], other.value], api.LAYOUT_CWBVH, _lib.E_ARG),
                 ("no tree", [h[0], empty.h.value], api.LAYOUT_CWBVH, _lib.E_STATE), ("CWBVH only", [only_cw.h.value, h[1]], api.LAYOUT_CWBVH, _lib.E_STATE),
                 ("TLAS", [h[0], t.h.value], api.LAYOUT_CWBVH, _lib.E_STATE), ("BVH_GPU", h, api.LAYOUT_BVH_GPU, _lib.E_UNSUPPORTED),
                 ("unknown layout", h, 7, _lib.E_UNSUPPORTED)]
        for what, hs, layout, code in cases:
            if what == "count 0":
                assert _lib.lib().tbvh_convert_batch((C.c_void_p * 1)(h[0]), 0, layout) == code, what
            else:
                assert raw_batch(hs, layout) == code, what
            for b, (d, tr) in zip(blas, before):
                gd, gt = cw(b)
                assert np.array_equal(gd, d) and np.array_equal(gt, tr), f"{what}: a refused batch changed a handle"
            got = rays.copy()
            t.Intersect(got)
            assert np.array_equal(tlas_words(got), tlas_words(want)), f"{what}: a refused batch made the TLAS stale"
        with pytest.raises(api.TbvhError, match="error -3"):
            api.convert_batch([blas[0], empty])
    finally:
        _lib.lib().tbvh_bvh_destroy(other)
        _lib.lib().tbvh_ctx_destroy(ctx2)


def test_launch_count_determinism_and_replica(gpu):
    rng = np.random.default_rng(23)
    meshes = [mesh(int(n), 7000 + k) for k, n in enumerate(np.exp(rng.uniform(0, np.log(3000), 1000)).astype(int).clip(1, 3000))]
    objs = api.build_batch([api.BVH() for _ in meshes], meshes)
    n0 = api.launch_count()
    api.convert_batch(objs)
    n_batch = api.launch_count() - n0
    first = [cw(b) for b in objs]
    ten = api.build_batch([api.BVH() for _ in meshes[:10]], meshes[:10])
    n0 = api.launch_count()
    for b in ten:
        convert(b)
    n_ten = api.launch_count() - n0
    assert n_batch < n_ten, (n_batch, n_ten)
    api.convert_batch(objs)
    for k, b in enumerate(objs):
        d, t = cw(b)
        assert np.array_equal(d, first[k][0]) and np.array_equal(t, first[k][1]), f"tree {k} differs between two conversions of one batch"
    # a group replica of a batch-converted handle walks like its source
    src = objs[int(np.argmax([v.shape[0] for v in meshes]))]
    v = meshes[int(np.argmax([v.shape[0] for v in meshes]))]
    src.layout = api.LAYOUT_CWBVH
    g = api.Group([0])
    g.replicate(src)
    sets, _ = util.ray_sets(v, res=24)
    want, got = sets["primary"].copy(), sets["primary"].copy()
    src.Intersect(want)
    g.Intersect(got)
    assert util.compare_hits(got, want) == {"prim": 0, "t": 0, "u": 0, "v": 0}


def one_node_tree(n, seed):
    """An uploaded tree of one node: a leaf root over n triangles, and no node 1 (used_nodes = 1)."""
    v = mesh(n, seed)
    nodes = np.zeros(1, portpy.NODE32)
    nodes[0]["aabbMin"], nodes[0]["aabbMax"] = v[:, :3].min(0), v[:, :3].max(0)
    nodes[0]["leftFirst"], nodes[0]["triCount"] = 0, n
    return (nodes, np.arange(n, dtype=np.uint32), n), v


def test_one_node_trees_next_to_others(gpu):
    """A one-node leaf tree has no node 1 of its own to wrap its leaf root into: first, last and in the middle of a batch, each tree
    (and its refit) is still what its own conversion gives."""
    items = [one_node_tree(3, 1), (None, mesh(500, 2)), one_node_tree(2, 3), one_node_tree(7, 4), (None, mesh(40, 5)), one_node_tree(1, 6)]
    make = [(lambda t=t, x=x: uploaded(t, x) if t is not None else built(x, "Build")) for t, x in items]
    meshes = [x for _, x in items]
    got = api.convert_batch([m() for m in make])
    want = [convert(m()) for m in make]
    assert_same(got, want, "one-node trees")
    assert_same_walks(got, want, meshes, "one-node trees")
    for k, v in enumerate(meshes):
        moved = v.copy()
        moved[:, :3] += np.float32(0.125) * np.cos(np.arange(moved.shape[0], dtype=np.float32))[:, None]
        for b in (got[k], want[k]):
            api._refit_layouts(b, moved)
        assert_same([got[k]], [want[k]], f"refit of tree {k}")
