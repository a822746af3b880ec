"""GPU parity of tbvh_build_batch_hq / api.build_batch( .., BUILD_HQ ): many meshes built with BuildHQ (SBVH) in one call.  Every tree
is exactly the one a BuildHQ of its mesh alone makes - node array, the whole primIdx and info (build_ms aside) - against separate GPU
builds and the pinned restatement (portpy.build_hq), whatever the order and neighbours of the mesh in the batch, under the settings
that change which kernel and group size processes a node.  Failed spatial splits read idxTmp words an ancestor left behind, or the
initial zeros: in a batch every tree sits at its own offset of the shared index space, and those leaves must still come out as a
build of their own gives them."""
import ctypes as C
import re

import numpy as np
import pytest

from oracle import portpy
from tinybvh_b200 import _lib, api, rays as R
from tests import util
from tests.test_build_batch_gpu import info, mesh, rec, tree, words
from tests.test_build_hq_gpu import assert_same_hq_tree
from tests.test_build_hq_shapes import FAIL_SCENES, fail_scene, fail_scene_hq
from tests.test_build_hq_shapes_gpu import CONFIGS, HQ_DEFAULTS, HQ_ENV, degenerate
from tests.test_oracle_pin import tlas_case

pytestmark = pytest.mark.gpu

MIXED = [1, 2, 3, 15, 16, 17, 31, 255, 256, 257, 1000, 5000, 70000]   # around hq_small (16) and the warp kernel's cap (256)
TOTALS = re.compile(r"hq-profile failed_splits (\d+) small_roots (\d+)")


@pytest.fixture
def hq_knobs(request, monkeypatch):
    """Sets a CONFIGS entry of tests/test_build_hq_shapes_gpu.py for one test; the defaults always come back."""
    opts, env = CONFIGS[request.param]
    for k in HQ_ENV:
        monkeypatch.delenv(k, raising=False)
    for k, val in env.items():
        monkeypatch.setenv(k, val)
    try:
        for k, val in {**HQ_DEFAULTS, **opts}.items():
            api.set_option(k, val)
        yield request.param
    finally:
        for k, val in HQ_DEFAULTS.items():
            api.set_option(k, val)


def hq_batch(meshes, indices=None, cls=api.BVH):
    return api.build_batch([cls() for _ in meshes], meshes, _lib.BUILD_HQ, indices)


def separate(meshes):
    return [api.BVH().BuildHQ(v) for v in meshes]


def assert_same(got, want, what):
    for k, (g, w) in enumerate(zip(got, want)):
        gn, gi = tree(g)
        wn, wi = tree(w)
        assert gi.shape == wi.shape and np.array_equal(gn, wn) and np.array_equal(gi, wi), f"{what}: tree {k} differs from its separate BuildHQ"
        assert info(g) == info(w), f"{what}: info of tree {k} differs"


def assert_oracle(b, v, label):
    nodes, idx, ic = portpy.build_hq(v)
    assert_same_hq_tree(b, nodes, idx, ic, label)


def referenced(b):
    """primitive references the leaves of a BVH-layout tree hold: the bvh8Tris records its CWBVH writes (past them the array is
    not written, on an SBVH)"""
    return int(tree(b)[0].reshape(-1, 8)[:, 7].sum())


def raw_batch_hq(handles, recs, space=_lib.HOST):
    hs = (C.c_void_p * max(len(handles), 1))(*handles)
    arr = (_lib.Mesh * max(len(recs), 1))(*recs)
    return _lib.lib().tbvh_build_batch_hq(hs, arr, len(recs), space, 1.0, 1.0)


def test_mixed_sizes_match_oracle_and_separate_builds(gpu):
    meshes = [mesh(n, 800 + k) for k, n in enumerate(MIXED)]
    want = separate(meshes)
    for k, v in enumerate(meshes):
        assert_oracle(want[k], v, f"separate BuildHQ of mesh {k}")
    rng = np.random.default_rng(7)
    for order in (list(range(len(meshes))), list(range(len(meshes)))[::-1], list(rng.permutation(len(meshes)))):
        got = hq_batch([meshes[k] for k in order])
        assert_same(got, [want[k] for k in order], f"order {order}")
        assert all(b.info().build_ms == got[0].info().build_ms > 0 for b in got)   # the device time of the whole batch
        assert all(not b.info().layouts & ~(1 << api.LAYOUT_BVH) for b in got)
        assert_oracle(got[order.index(len(meshes) - 1)], meshes[-1], f"70k mesh in order {order}")


def profiled(monkeypatch, capfd, fn):
    """-> (fn(), failed_splits the builds it ran printed, summed)"""
    monkeypatch.setenv("TBVH_HQ_PROFILE", "1")
    capfd.readouterr()
    try:
        r = fn()
    finally:
        monkeypatch.delenv("TBVH_HQ_PROFILE")
    return r, sum(int(f) for f, _ in TOTALS.findall(capfd.readouterr().err))


@pytest.mark.parametrize("hq_knobs", ["defaults", "small8", "small256", "cluster1", "frags1_capmax", "frags_max"], indirect=True)
def test_failing_scenes_in_one_batch(gpu, hq_knobs, monkeypatch, capfd):
    """Every scene whose spatial splits fail often, interleaved with plain meshes: failed-split leaves that read stale idxTmp words sit
    in trees at nonzero batch positions.  Each tree is the restatement's; the batch fails exactly the splits the separate builds do."""
    named = []
    for k, name in enumerate(FAIL_SCENES):
        named += [(f"plain {k}", mesh(300 + 700 * k, 900 + k)), (name, fail_scene(name))]
    named.append(("plain last", mesh(20, 950)))
    meshes = [v for _, v in named]
    got, batch_failed = profiled(monkeypatch, capfd, lambda: hq_batch(meshes))
    want, separate_failed = profiled(monkeypatch, capfd, lambda: separate(meshes))
    assert_same(got, want, hq_knobs)
    assert batch_failed == separate_failed > 0, (batch_failed, separate_failed)
    for k, (name, v) in enumerate(named):
        if name in FAIL_SCENES:
            nodes, idx, ic = fail_scene_hq(name)[:3]
            assert_same_hq_tree(got[k], nodes, idx, ic, f"{name} at batch position {k}, {hq_knobs}")


def offatrium_meshes():
    base = mesh(3000, 61)
    out = [("plain", mesh(2500, 62)), ("plain small", mesh(90, 63))]
    for k in (-126, -20, 40, 90):
        out.append((f"scaled 2^{k}", util.scaled(base, k)))
    out.append(("translated", util.translated(base, 3e5)))
    out += [(name, degenerate(name)) for name in ("identical", "duplicates", "slivers")]
    out.append(("plain after", mesh(4000, 65)))
    return out


def test_offatrium_inputs_next_to_plain_meshes(gpu):
    named = offatrium_meshes()
    meshes = [v for _, v in named]
    got = hq_batch(meshes)
    want = separate(meshes)
    for k, (label, v) in enumerate(named):
        assert_same([got[k]], [want[k]], label)
    plain = [k for k, (label, _) in enumerate(named) if label.startswith("plain")]
    assert_same([got[k] for k in plain], hq_batch([meshes[k] for k in plain]), "plain meshes with and without off-atrium neighbours")


def test_signed_zero_families_match_separate_builds(gpu):
    """Meshes with -0 coordinates next to plain ones: every tree is the reference's and equals its separate GPU build, and the plain
    neighbours equal a batch of their own."""
    base = mesh(3000, 71)
    named = [("plain", mesh(1500, 72))] + [(f"signed zero {m}", util.signed_zero(base, m, seed=5)) for m in ("pos", "neg", "random", "order")]
    named += [("signed zero small", util.signed_zero(mesh(100, 73), "neg", seed=6)), ("plain after", mesh(700, 74))]
    meshes = [v for _, v in named]
    got = hq_batch(meshes)
    for k, (label, _) in enumerate(named):
        assert_oracle(got[k], meshes[k], label)
        assert_same([got[k]], separate([meshes[k]]), label)
    assert_same([got[0], got[-1]], hq_batch([meshes[0], meshes[-1]]), "plain meshes next to signed zeros")


def test_indexed_strided_and_device_inputs(gpu):
    import torch
    rng = np.random.default_rng(17)
    meshes = [mesh(int(n), 4100 + k) for k, n in enumerate([5, 200, 3000, 17, 20000])]
    want = separate(meshes)
    idx_meshes, indices = [], []
    for k, v in enumerate(meshes):
        if k % 2:
            idx_meshes.append(v), indices.append(None)
            continue
        perm = rng.permutation(v.shape[0])
        verts = np.empty_like(v)
        verts[perm] = v
        idx_meshes.append(verts), indices.append(perm.astype(np.uint32))
    assert_same(hq_batch(idx_meshes, indices=indices), want, "indexed meshes mixed with flat ones")
    d_meshes = [torch.from_numpy(v).cuda() for v in idx_meshes]
    d_indices = [None if i is None else torch.from_numpy(i.view(np.int32)).cuda() for i in indices]
    assert_same(hq_batch(d_meshes, indices=d_indices), want, "device meshes")
    # strided vertex slices: 12, 16 and 32 bytes apart
    keep, recs = [], []
    for k, v in enumerate(meshes):
        stride = (12, 16, 32)[k % 3]
        a = np.zeros((v.shape[0], stride // 4), np.float32)
        a[:, :3] = v[:, :3]
        keep.append(a), recs.append(_lib.Mesh(a.ctypes.data, stride, 0, None, v.shape[0] // 3))
    objs = [api.BVH() for _ in meshes]
    api.check(raw_batch_hq([b.h.value for b in objs], recs))
    assert_same(objs, want, "strided vertex slices")


def test_thousand_meshes_launches_and_determinism(gpu):
    rng = np.random.default_rng(23)
    sizes = np.exp(rng.uniform(0, np.log(5000), 1000)).astype(int).clip(1, 5000)
    meshes = [mesh(int(n), 6000 + k) for k, n in enumerate(sizes)]
    n0 = api.launch_count()
    got = hq_batch(meshes)
    n_batch = api.launch_count() - n0
    n0 = api.launch_count()
    want = separate(meshes[:10])
    n_ten = api.launch_count() - n0
    assert n_batch < n_ten, (n_batch, n_ten)
    assert_same(got, want + separate(meshes[10:]), "1,000 meshes")
    for k in rng.choice(len(meshes), 20, replace=False):
        assert_oracle(got[k], meshes[k], f"mesh {k}")
    assert_same(hq_batch(meshes), got, "the same batch built twice")


def test_refusals_leave_handles_as_they_were(gpu):
    meshes = [mesh(300, 81), mesh(2000, 82)]
    objs = hq_batch(meshes)
    before = [tree(b) for b in objs]
    third = api.BVH()
    h = [b.h.value for b in objs]
    h3 = h + [third.h.value]
    r = [rec(v) for v in meshes]
    ctx2 = C.c_void_p()
    api.check(_lib.lib().tbvh_ctx_create(0, C.byref(ctx2)))
    other = C.c_void_p()
    api.check(_lib.lib().tbvh_bvh_create(ctx2, C.byref(other)))
    small = np.zeros((12, 4), np.float32)   # far fewer vertices than the records claim: a refusal must come before any read
    try:
        empty = _lib.Mesh(meshes[0].ctypes.data, 16, 0, None, 0)
        badstride = _lib.Mesh(meshes[0].ctypes.data, 10, 0, None, 100)
        huge = [_lib.Mesh(small.ctypes.data, 16, 0, None, 1 << 29) for _ in range(3)]
        cases = [("count 0", h, [], _lib.HOST, _lib.E_ARG), ("NULL handle", [h[0], None], r, _lib.HOST, _lib.E_ARG),
                 ("duplicate handle", [h[0], h[0]], r, _lib.HOST, _lib.E_ARG), ("two contexts", [h[0], other.value], r, _lib.HOST, _lib.E_ARG),
                 ("prim_count 0", h, [r[0], empty], _lib.HOST, _lib.E_ARG), ("bad stride", h, [badstride, r[1]], _lib.HOST, _lib.E_ARG),
                 ("unknown space", h, r, 7, _lib.E_ARG), ("2^30 + 300 triangles", h3, huge[:2] + [r[0]], _lib.HOST, _lib.E_LIMIT),
                 ("2^32 - 1 triangles", h, [_lib.Mesh(small.ctypes.data, 16, 0, None, 0xFFFFFFFF), r[1]], _lib.HOST, _lib.E_LIMIT)]
        for what, hs, recs, space, code in cases:
            assert raw_batch_hq(hs, recs, space) == code, what
            for b, (n, i) in zip(objs, before):
                gn, gi = tree(b)
                assert np.array_equal(gn, n) and np.array_equal(gi, i), f"{what}: a refused batch changed a handle"
        # an index past its mesh's vertices, host and device
        import torch
        perm = np.arange(meshes[1].shape[0], dtype=np.uint32)
        perm[5] = meshes[1].shape[0]
        for space in ("host", "device"):
            ms = [meshes[0], meshes[1]] if space == "host" else [torch.from_numpy(v).cuda() for v in meshes]
            ix = [None, perm] if space == "host" else [None, torch.from_numpy(perm.view(np.int32)).cuda()]
            with pytest.raises(api.TbvhError, match="error -2"):
                api.build_batch(objs, ms, _lib.BUILD_HQ, ix)
            for b, (n, i) in zip(objs, before):
                gn, gi = tree(b)
                assert np.array_equal(gn, n) and np.array_equal(gi, i), f"{space} bad index: a refused batch changed a handle"
        # tbvh_build_batch itself keeps refusing BuildHQ
        hs = (C.c_void_p * 2)(*h)
        arr = (_lib.Mesh * 2)(*r)
        assert _lib.lib().tbvh_build_batch(hs, arr, 2, _lib.HOST, 1.0, 1.0, _lib.BUILD_HQ) == _lib.E_UNSUPPORTED
    finally:
        _lib.lib().tbvh_bvh_destroy(other)
        _lib.lib().tbvh_ctx_destroy(ctx2)


@pytest.mark.parametrize("cls,layout", [(api.BVH_GPU, api.LAYOUT_BVH_GPU), (api.BVH8_CWBVH, api.LAYOUT_CWBVH)])
def test_derived_layouts_from_a_batch(gpu, cls, layout):
    meshes = [mesh(n, 150 + k) for k, n in enumerate([1, 16, 100, 257, 3000, 40000])]
    got = hq_batch(meshes, cls=cls)
    for k, v in enumerate(meshes):
        want = cls().BuildHQ(v)
        g, w = got[k].download(), want.download()
        if layout == api.LAYOUT_CWBVH:
            used = 3 * referenced(api.BVH().BuildHQ(v))
            assert g[1].shape == w[1].shape and np.array_equal(g[0].view(np.uint32), w[0].view(np.uint32)), f"bvh8Data of mesh {k}"
            assert np.array_equal(g[1][:used].view(np.uint32), w[1][:used].view(np.uint32)), f"bvh8Tris of mesh {k}"
        else:
            assert np.array_equal(g.view(np.uint32), w.view(np.uint32)), f"BVH_GPU of mesh {k}"
        assert got[k].info().layouts == want.info().layouts


def test_convert_batch_and_walks_of_batch_built_trees(gpu):
    """convert_batch of batch-built SBVHs equals convert_batch of separately built ones; camera and shadow walks of the batch-built
    trees (BVH layout, leaf triangles included, and CWBVH) match the oracle walking the reference's tree."""
    v = fail_scene("snapped20k_q4")
    meshes = [mesh(500, 161), v, mesh(3000, 162)]
    got, want = hq_batch(meshes), separate(meshes)
    used = [3 * referenced(b) for b in want]
    api.convert_batch(got), api.convert_batch(want)
    for k in range(len(meshes)):
        gd, wd = got[k].info(), want[k].info()
        assert gd.used_blocks == wd.used_blocks and gd.cwbvh_tri_count == wd.cwbvh_tri_count
        for b in (got[k], want[k]):
            d8, t8 = np.zeros((b.info().used_blocks, 4), np.float32), np.zeros((b.info().cwbvh_tri_count * 3, 4), np.float32)
            api.check(_lib.lib().tbvh_download_cwbvh(b.h, d8.ctypes.data, t8.ctypes.data, api.HOST))
            b.cw = (d8, t8)
        assert np.array_equal(got[k].cw[0].view(np.uint32), want[k].cw[0].view(np.uint32)), f"bvh8Data of mesh {k}"
        assert np.array_equal(got[k].cw[1][:used[k]].view(np.uint32), want[k].cw[1][:used[k]].view(np.uint32)), f"bvh8Tris of mesh {k}"
    nodes, idx, ic = fail_scene_hq("snapped20k_q4")[:3]
    walk = portpy.PortBVH(v, nodes=nodes, prim_idx=idx)
    cw = util.oracle_cwbvh(v, mode=1)[0]
    sets, bounds = util.ray_sets(v, res=64)
    traced = sets["primary"].copy()
    walk.intersect(traced)
    sets.update(util.derived_sets(traced, v, bounds))
    for layout, oracle_walk in ((api.LAYOUT_BVH, walk.intersect), (api.LAYOUT_CWBVH, cw.intersect)):
        got[1].layout = layout
        for kind in ("primary", "shadow"):
            w_, g_ = sets[kind].copy(), sets[kind].copy()
            oracle_walk(w_), got[1].Intersect(g_)
            assert util.compare_hits(g_, w_) == {"prim": 0, "t": 0, "u": 0, "v": 0}, f"layout {layout} {kind}"
    got[1].layout = api.LAYOUT_BVH
    assert np.array_equal(got[1].IsOccluded(sets["shadow"]), walk.occluded(sets["shadow"]))


def test_refit_of_a_batch_built_sbvh_is_refused(gpu):
    meshes = [mesh(50, 171), mesh(3000, 172)]
    got = hq_batch(meshes)
    for b, v in zip(got, meshes):
        assert _lib.lib().tbvh_refit(b.h, v.ctypes.data, 16, v.shape[0] // 3, api.HOST) == _lib.E_STATE


def test_tlas_over_batch_hq_blasses(gpu):
    v, inst, O, D = tlas_case(113, 40)
    rays = R.make_rays(O, D)
    sh = R.make_rays(O, D, tmax=150.0)
    blas, sep = hq_batch(v), separate(v)
    for group in (blas, sep):
        for b in group:
            api.check(_lib.lib().tbvh_convert(b.h, api.LAYOUT_CWBVH))   # both layouts on every BLAS
    results = []
    for group in (blas, sep):
        t = api.TLAS().Build(inst.copy(), group)
        t_cw = api.TLAS().Build(inst.copy(), group, blas_layout=api.LAYOUT_CWBVH)
        hits, hits_cw = rays.copy(), rays.copy()
        t.Intersect(hits), t_cw.Intersect(hits_cw)
        results.append((t, words(hits), words(hits_cw), t.IsOccluded(sh), t_cw.IsOccluded(sh), tree(t), hits))
    a, b = results
    for k, what in enumerate(("BVH-layout hits", "CWBVH hits", "BVH-layout occlusion", "CWBVH occlusion"), start=1):
        assert np.array_equal(a[k], b[k]), what
    assert np.array_equal(a[5][0], b[5][0]) and np.array_equal(a[5][1], b[5][1]), "TLAS nodes"
    assert (a[6]["t"] < 1e30).sum() > 1000
    # a batch that rebuilds one of its BLASes makes the TLAS stale
    api.build_batch([blas[1], api.BVH()], [v[1], v[0]], _lib.BUILD_HQ)
    r = R.make_rays(O[:64], D[:64])
    assert _lib.lib().tbvh_intersect(a[0].h, api.LAYOUT_BVH, r.ctypes.data, 128, 64) == _lib.E_STATE
