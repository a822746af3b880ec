"""GPU parity of tbvh_build_batch / api.build_batch: many meshes built in one call, every tree exactly the one a build of its mesh alone
makes - against the oracle and against separate GPU builds, whatever the order and neighbours of the mesh in the batch - and every
later call (convert, refit, TLAS) working unchanged on batch-built handles."""
import ctypes as C

import numpy as np
import pytest

from tinybvh_b200 import _lib, api, rays as R, scenes
from tests import util
from tests.test_oracle_pin import tlas_case

pytestmark = pytest.mark.gpu

FLAVOURS = {"Build": _lib.BUILD_REFERENCE, "BuildAVX": _lib.BUILD_AVX}
MIXED = [1, 2, 3, 31, 128, 129, 257, 1000, 5000, 70000]   # 128 is the default small_t: the root is a warp subtree up to it


def mesh(n, seed):
    return scenes.procedural_scene(n, seed)


def tree(b):
    nodes, idx = b.download()
    return nodes.view(np.uint32).copy(), idx.copy()


def info(b):
    return bytes(b.info())[:_lib.Info.build_ms.offset]   # every field but build_ms


def separate(meshes, flavour):
    return [getattr(api.BVH(), "BuildAVX" if flavour == _lib.BUILD_AVX else "Build")(v) for v in meshes]


def assert_same(got, want, what):
    for k, (g, w) in enumerate(zip(got, want)):
        gn, gi = tree(g)
        wn, wi = tree(w)
        assert np.array_equal(gn, wn) and np.array_equal(gi, wi), f"{what}: tree {k} differs from its separate build"
        assert info(g) == info(w), f"{what}: info of tree {k} differs"


def batch(meshes, flavour=_lib.BUILD_REFERENCE, indices=None, cls=api.BVH):
    return api.build_batch([cls() for _ in meshes], meshes, flavour, indices)


def raw_batch(handles, recs, flavour=_lib.BUILD_REFERENCE, space=_lib.HOST):
    hs = (C.c_void_p * max(len(handles), 1))(*handles)
    arr = (_lib.Mesh * max(len(recs), 1))(*recs)
    return _lib.lib().tbvh_build_batch(hs, arr, len(recs), space, 1.0, 1.0, flavour)


def rec(v):
    return _lib.Mesh(v.ctypes.data, 16, 0, None, v.shape[0] // 3)


@pytest.mark.parametrize("name", ["Build", "BuildAVX"])
def test_mixed_sizes_match_oracle_and_separate_builds(gpu, name):
    flavour = FLAVOURS[name]
    meshes = [mesh(n, 500 + k) for k, n in enumerate(MIXED)]
    want = separate(meshes, flavour)
    for k, v in enumerate(meshes):
        o = util.oracle_tree(v, flavour)
        wn, wi = tree(want[k])
        assert np.array_equal(wn, o.nodes.view(np.uint32)) and np.array_equal(wi, o.prim_idx), f"separate build of mesh {k} differs from the oracle"
    rng = np.random.default_rng(5)
    for order in (list(range(len(meshes))), list(range(len(meshes)))[::-1], list(rng.permutation(len(meshes)))):
        got = batch([meshes[k] for k in order], flavour)
        assert_same(got, [want[k] for k in order], f"{name}, order {order}")
        assert all(b.info().build_ms == got[0].info().build_ms > 0 for b in got)   # the device time of the whole batch


def test_thousand_meshes(gpu):
    rng = np.random.default_rng(11)
    sizes = np.exp(rng.uniform(0, np.log(20000), 1000)).astype(int).clip(1, 20000)
    meshes = [mesh(int(n), 2000 + k) for k, n in enumerate(sizes)]
    got = batch(meshes)
    assert_same(got, separate(meshes, _lib.BUILD_REFERENCE), "1,000 meshes")
    for k in rng.choice(len(meshes), 20, replace=False):
        o = util.oracle_bvh(meshes[k])
        gn, gi = tree(got[k])
        assert np.array_equal(gn, o.nodes.view(np.uint32)) and np.array_equal(gi, o.prim_idx), f"mesh {k} differs from the oracle"


@pytest.mark.parametrize("build_mode,small_t,small_mode", [(0, 128, 0), (1, 128, 0), (0, 32, 0), (1, 32, 0), (0, 128, 1), (0, 128, 2), (0, 128, 3), (1, 32, 3)])
def test_builder_paths(gpu, build_mode, small_t, small_mode):
    """The persistent and the launch-per-stage large phase, both switch points, every warp-subtree kernel variant."""
    rng = np.random.default_rng(13)
    meshes = [mesh(400000, 21)] + [mesh(int(n), 3000 + k) for k, n in enumerate(rng.integers(1, 300, 500))]
    order = list(rng.permutation(len(meshes)))
    meshes = [meshes[k] for k in order]
    try:
        api.set_option("build_mode", build_mode), api.set_option("small_t", small_t), api.set_option("small_mode", small_mode)
        for flavour in (_lib.BUILD_REFERENCE, _lib.BUILD_AVX):
            assert_same(batch(meshes, flavour), separate(meshes, flavour), f"build_mode {build_mode}, small_t {small_t}, small_mode {small_mode}")
    finally:
        api.set_option("build_mode", 0), api.set_option("small_t", 128), api.set_option("small_mode", 0)


def offatrium_meshes():
    base = mesh(3000, 31)
    out = [("plain", mesh(2500, 32)), ("plain small", mesh(90, 33))]
    for mode in ("pos", "neg", "random", "order"):
        out.append((f"signed zero {mode}", util.signed_zero(base, mode, seed=3)))
    out.append(("signed zero small", util.signed_zero(mesh(100, 34), "neg", seed=4)))
    for k in (-126, -20, 90):
        out.append((f"scaled 2^{k}", util.scaled(base, k)))
    out.append(("translated", util.translated(base, 3e5)))
    one = np.array([[0, 0, 0, 0], [1, 0, 0, 0], [0, 1, 0, 0]], np.float32)
    flat = mesh(3000, 12)
    flat[:, 1] = 1.5
    dup = mesh(900, 13)
    out += [("identical", np.tile(one, (700, 1))), ("flat", flat), ("duplicates", np.concatenate([dup, dup, dup[:300]]))]
    out.append(("plain after", mesh(4000, 35)))
    return out


@pytest.mark.parametrize("name", ["Build", "BuildAVX"])
def test_offatrium_inputs_next_to_plain_meshes(gpu, name):
    """Signed zeros, extreme scales, far translations and degenerate meshes in one batch: each tree is its own separate build; the plain
    meshes' trees are what a batch of plain meshes alone gives them (the first -0 of the batch changes nothing for its neighbours)."""
    flavour = FLAVOURS[name]
    named = offatrium_meshes()
    meshes = [v for _, v in named]
    got = batch(meshes, flavour)
    want = separate(meshes, flavour)
    for k, (label, _) in enumerate(named):
        assert_same([got[k]], [want[k]], label)
    plain = [k for k, (label, _) in enumerate(named) if label.startswith("plain")]
    alone = batch([meshes[k] for k in plain], flavour)
    assert_same([got[k] for k in plain], alone, "plain meshes with and without off-atrium neighbours")
    o = util.oracle_tree(meshes[5], flavour)   # "signed zero order": every vertex order of -0 and +0
    gn, gi = tree(got[5])
    assert np.array_equal(gn, o.nodes.view(np.uint32)) and np.array_equal(gi, o.prim_idx)


def test_indexed_device_inputs_and_bad_index(gpu):
    import torch
    rng = np.random.default_rng(17)
    meshes = [mesh(int(n), 4000 + k) for k, n in enumerate([5, 200, 3000, 129, 20000])]
    # indexed forms: unique vertices + indices (some shuffled, so the gather matters)
    idx_meshes, indices = [], []
    for k, v in enumerate(meshes):
        if k % 2:
            idx_meshes.append(v), indices.append(None)
            continue
        perm = rng.permutation(v.shape[0])
        verts = np.empty_like(v)
        verts[perm] = v
        idx_meshes.append(verts), indices.append(perm.astype(np.uint32))
    flat = batch(meshes)
    assert_same(batch(idx_meshes, indices=indices), flat, "indexed meshes mixed with flat ones")
    d_meshes = [torch.from_numpy(v).cuda() for v in idx_meshes]
    d_indices = [None if i is None else torch.from_numpy(i.view(np.int32)).cuda() for i in indices]
    assert_same(batch(d_meshes, indices=d_indices), flat, "device meshes")
    # an index past its mesh's vertices refuses the whole batch, before any handle gave up its tree
    for space in ("host", "device"):
        objs = batch(meshes)
        before = [tree(b) for b in objs]
        bad = [None if i is None else i.copy() for i in indices]
        bad[2][7] = idx_meshes[2].shape[0]
        ms = idx_meshes if space == "host" else d_meshes
        bi = bad if space == "host" else [None if i is None else torch.from_numpy(i.view(np.int32)).cuda() for i in bad]
        with pytest.raises(api.TbvhError, match="error -2"):
            api.build_batch(objs, ms, indices=bi)
        for b, (n, i) in zip(objs, before):
            gn, gi = tree(b)
            assert np.array_equal(gn, n) and np.array_equal(gi, i), f"{space}: a refused batch changed a handle"
    with pytest.raises(api.TbvhError):
        api.build_batch([api.BVH(), api.BVH()], [meshes[0], torch.from_numpy(meshes[1]).cuda()])   # one space per call


def test_refusals_leave_handles_as_they_were(gpu):
    meshes = [mesh(300, 41), mesh(2000, 42)]
    objs = batch(meshes)
    before = [tree(b) for b in objs]
    h = [b.h.value for b in objs]
    r = [rec(v) for v in meshes]
    ctx2 = C.c_void_p()
    api.check(_lib.lib().tbvh_ctx_create(0, C.byref(ctx2)))
    other = C.c_void_p()
    api.check(_lib.lib().tbvh_bvh_create(ctx2, C.byref(other)))
    try:
        empty = _lib.Mesh(meshes[0].ctypes.data, 16, 0, None, 0)
        badstride = _lib.Mesh(meshes[0].ctypes.data, 10, 0, None, 100)
        cases = [("count 0", h, [], _lib.BUILD_REFERENCE, _lib.E_ARG), ("NULL handle", [h[0], None], r, _lib.BUILD_REFERENCE, _lib.E_ARG),
                 ("duplicate handle", [h[0], h[0]], r, _lib.BUILD_REFERENCE, _lib.E_ARG),
                 ("two contexts", [h[0], other.value], r, _lib.BUILD_REFERENCE, _lib.E_ARG),
                 ("prim_count 0", h, [r[0], empty], _lib.BUILD_REFERENCE, _lib.E_ARG), ("bad stride", h, [badstride, r[1]], _lib.BUILD_REFERENCE, _lib.E_ARG),
                 ("BuildHQ", h, r, _lib.BUILD_HQ, _lib.E_UNSUPPORTED), ("unknown flavour", h, r, 7, _lib.E_ARG)]
        for what, hs, recs, flavour, code in cases:
            assert raw_batch(hs, recs, flavour) == code, what
            for b, (n, i) in zip(objs, before):
                gn, gi = tree(b)
                assert np.array_equal(gn, n) and np.array_equal(gi, i), f"{what}: a refused batch changed a handle"
    finally:
        _lib.lib().tbvh_bvh_destroy(other)
        _lib.lib().tbvh_ctx_destroy(ctx2)


@pytest.mark.parametrize("cls,layout", [(api.BVH_GPU, api.LAYOUT_BVH_GPU), (api.BVH8_CWBVH, api.LAYOUT_CWBVH)])
def test_derived_layouts_from_a_batch(gpu, cls, layout):
    meshes = [mesh(n, 50 + k) for k, n in enumerate([1, 100, 129, 3000, 40000])]
    got = batch(meshes, _lib.BUILD_AVX, cls=cls)
    for k, v in enumerate(meshes):
        want = cls().Build(v)
        g, w = got[k].download(), want.download()
        if layout == api.LAYOUT_CWBVH:
            assert np.array_equal(g[0].view(np.uint32), w[0].view(np.uint32)) and np.array_equal(g[1].view(np.uint32), w[1].view(np.uint32)), f"CWBVH of mesh {k}"
        else:
            assert np.array_equal(g.view(np.uint32), w.view(np.uint32)), f"BVH_GPU of mesh {k}"
        assert got[k].info().layouts == want.info().layouts


def words(r):
    return r.view(np.uint32).reshape(-1, 32)[:, 11:16]   # hit.inst, t, u, v, prim


def test_tlas_over_batch_built_blasses(gpu):
    v, inst, O, D = tlas_case(103, 40)
    inst_ref = inst.copy()
    ref = util.oracle_tlas(inst_ref, v)
    blas = batch(v)
    for k in range(len(blas)):
        api.check(_lib.lib().tbvh_convert(blas[k].h, api.LAYOUT_CWBVH))   # both layouts on every BLAS
    t = api.TLAS().Build(inst, blas)
    t_cw = api.TLAS().Build(inst.copy(), blas, blas_layout=api.LAYOUT_CWBVH)
    rays = R.make_rays(O, D)
    want, got, got_cw = rays.copy(), rays.copy(), rays.copy()
    ref.intersect(want), t.Intersect(got), t_cw.Intersect(got_cw)
    assert np.array_equal(words(got), words(want))
    assert (want["t"] < 1e30).sum() > 1000
    assert (words(got_cw) == words(want)).all(axis=1).mean() > 0.999   # the CWBVH walk of the same triangles: ties aside, the same hits
    sh = R.make_rays(O, D, tmax=150.0)
    assert np.array_equal(t.IsOccluded(sh), ref.occluded(sh))
    # a batch that rebuilds one of its BLASses makes the TLAS stale
    api.build_batch([blas[1], api.BVH()], [v[1], v[0]])
    r = R.make_rays(O[:64], D[:64])
    assert _lib.lib().tbvh_intersect(t.h, api.LAYOUT_BVH, r.ctypes.data, 128, 64) == _lib.E_STATE


def test_refit_of_batch_built_handles(gpu):
    meshes = [mesh(n, 60 + k) for k, n in enumerate([50, 129, 6000, 30000])]
    got, want = batch(meshes), separate(meshes, _lib.BUILD_REFERENCE)
    for k, v in enumerate(meshes):
        moved = v.copy()
        moved[:, :3] += np.float32(0.25) * np.sin(np.arange(moved.shape[0], dtype=np.float32))[:, None]
        for b in (got[k], want[k]):
            api.check(_lib.lib().tbvh_convert(b.h, api.LAYOUT_CWBVH))
            api._refit_layouts(b, moved)
        assert_same([got[k]], [want[k]], f"refit of mesh {k}")
        gd, wd = np.zeros((got[k].info().used_blocks, 4), np.float32), np.zeros((want[k].info().used_blocks, 4), np.float32)
        for b, d in ((got[k], gd), (want[k], wd)):
            t8 = np.zeros((b.info().cwbvh_tri_count * 3, 4), np.float32)
            api.check(_lib.lib().tbvh_download_cwbvh(b.h, d.ctypes.data, t8.ctypes.data, api.HOST))
        assert np.array_equal(gd.view(np.uint32), wd.view(np.uint32)), f"refitted CWBVH of mesh {k}"


def test_launch_count_and_determinism(gpu):
    rng = np.random.default_rng(19)
    meshes = [mesh(int(n), 7000 + k) for k, n in enumerate(np.exp(rng.uniform(0, np.log(5000), 1000)).astype(int).clip(1, 5000))]
    n0 = api.launch_count()
    a = batch(meshes)
    n_batch = api.launch_count() - n0
    n0 = api.launch_count()
    separate(meshes[:10], _lib.BUILD_REFERENCE)
    n_ten = api.launch_count() - n0
    assert n_batch < n_ten, (n_batch, n_ten)
    assert_same(batch(meshes), a, "the same batch built twice")
