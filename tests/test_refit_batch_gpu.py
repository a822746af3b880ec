"""GPU parity of tbvh_refit_batch / api.refit_batch: many trees refitted in one call, every handle exactly what tbvh_refit (keep_layouts = 0)
or tbvh_refit_layouts (keep_layouts = 1) of it alone leaves - BVH2, BVH_GPU nodes, bvh8Data / bvh8Tris, info, walks - whatever the order,
the neighbours and the layouts of the other handles of the batch.  Two frames each: the second refits from the first frame's boxes."""
import ctypes as C

import numpy as np
import pytest

from oracle import portpy
from tinybvh_b200 import _lib, api, rays as R, scenes
from tests import util
from tests.cwbvh_refit_oracle import RefitCWBVH
from tests.test_convert_batch_gpu import built, convert, info, mesh, one_node_tree, uploaded
from tests.test_oracle_pin import moved, tlas_case

pytestmark = pytest.mark.gpu
ZERO = {"prim": 0, "t": 0, "u": 0, "v": 0}
SIZES = [1, 2, 3, 31, 128, 129, 257, 1000, 5000, 70000]
SUBSETS = ["bvh", "bvh+gpu", "bvh+cw", "all"]


def cw(b):
    """bvh8Data and the bvh8Tris records the leaves reference, of any handle"""
    i = b.info()
    d = np.zeros((i.used_blocks, 4), np.uint32)
    t = np.zeros((i.cwbvh_tri_count * 3, 4), np.uint32)
    api.check(_lib.lib().tbvh_download_cwbvh(b.h, d.ctypes.data, t.ctypes.data, api.HOST))
    nodes, _ = api.BVH.download(b)
    return d, t[: int(nodes["triCount"][np.arange(nodes.shape[0]) != 1].sum()) * 3]


def with_layouts(b, subset):
    if "gpu" in subset or subset == "all":
        api.check(_lib.lib().tbvh_convert(b.h, api.LAYOUT_BVH_GPU))
    if "cw" in subset or subset == "all":
        convert(b)
    return b


def frame(v, f):
    return moved(v, 70 + f, amp=0.05) if v.shape[0] > 3 else v + np.float32(0.01 * f)


def raw_refit_batch(handles, meshes, space=api.HOST, keep=1, stride=16, indices=None):
    recs = (_lib.Mesh * max(len(meshes), 1))()
    for r, m in zip(recs, meshes):
        r.verts, r.stride, r.vert_count, r.indices, r.prim_count = m.ctypes.data, stride, 0, indices, m.shape[0] // 3
    hs = (C.c_void_p * max(len(handles), 1))(*handles)
    return _lib.lib().tbvh_refit_batch(hs, recs, len(meshes), space, keep)


def single(b, v, keep):
    fn = _lib.lib().tbvh_refit_layouts if keep else _lib.lib().tbvh_refit
    api.check(fn(b.h, v.ctypes.data, 16, v.shape[0] // 3, api.HOST))


def snapshot(b):
    """every downloadable byte of a handle and its info but build_ms"""
    i = b.info()
    out = [info(b)]
    if i.layouts & (1 << api.LAYOUT_BVH):
        n, idx = api.BVH.download(b)
        out += [n.tobytes(), idx.tobytes()]
    if i.layouts & (1 << api.LAYOUT_BVH_GPU):
        out.append(api.BVH_GPU.download(b).tobytes())
    if i.layouts & (1 << api.LAYOUT_CWBVH):
        d, t = cw(b)
        out += [d.tobytes(), t.tobytes()]
    return out


def assert_same(got, want, what):
    for k, (g, w) in enumerate(zip(got, want)):
        assert snapshot(g) == snapshot(w), f"{what}: handle {k} differs from its own refit"


def walks(b, v, seed):
    """closest hit and occlusion of camera, diffuse and shadow rays in every layout the handle holds (BVH_GPU is walked through the
    BVH2 traversal view of the handle)"""
    out = []
    for layout in (api.LAYOUT_BVH, api.LAYOUT_CWBVH):
        if b.info().layouts & (1 << layout):
            b.layout = layout
            sets, bounds = util.ray_sets(v, res=24, seed=seed)
            prim = sets["primary"].copy()
            b.Intersect(prim)
            d = util.derived_sets(prim, v, bounds)
            diffuse = d["diffuse"].copy()
            b.Intersect(diffuse)
            out += [util.nan_canonical(np.concatenate([prim, diffuse])).tobytes(), b.IsOccluded(d["shadow"]).tobytes()]
    b.layout = api.LAYOUT_BVH
    return out


def check_oracle(b, v0, built_nodes, w, label):
    """BVH2 against BVH::Refit, and a kept CWBVH against the oracle's re-encode of the conversion's collapse"""
    o = portpy.PortBVH(v0, nodes=built_nodes.copy(), prim_idx=api.BVH.download(b)[1])
    o.refit(w)
    nodes, _ = api.BVH.download(b)
    assert np.array_equal(nodes.view(np.uint32), o.nodes.view(np.uint32)), f"{label}: BVH2 differs from BVH::Refit"
    if b.info().layouts & (1 << api.LAYOUT_CWBVH):
        ref = RefitCWBVH(built_nodes, o.nodes, o.prim_idx, w)
        d, t = cw(b)
        assert np.array_equal(d, np.ascontiguousarray(ref.nodes).view(np.uint32).reshape(d.shape)), f"{label}: bvh8Data differs from the oracle"
        assert np.array_equal(t, np.ascontiguousarray(ref.tris).view(np.uint32).reshape(-1, 4)[: t.shape[0]]), f"{label}: bvh8Tris differs from the oracle"


@pytest.mark.parametrize("keep", [0, 1])
@pytest.mark.parametrize("name", ["Build", "BuildAVX"])
def test_mixed_sizes_and_layouts_match_single_refits(gpu, name, keep):
    meshes = [mesh(n, 300 + k) for k, n in enumerate(SIZES)]
    rng = np.random.default_rng(5)
    orders = (list(range(len(meshes))), list(range(len(meshes)))[::-1], list(rng.permutation(len(meshes))))
    for o_i, order in enumerate(orders):
        vs = [meshes[k] for k in order]
        subsets = [SUBSETS[(k + o_i) % 4] for k in order]
        got = [with_layouts(built(v, name), s) for v, s in zip(vs, subsets)]
        want = [with_layouts(built(v, name), s) for v, s in zip(vs, subsets)]
        built_nodes = [api.BVH.download(g)[0] for g in got]
        for f in (1, 2):
            ws = [frame(v, f) for v in vs]
            api.refit_batch(got, ws, keep_layouts=keep)
            for b, w in zip(want, ws):
                single(b, w, keep)
            assert_same(got, want, f"{name}, keep {keep}, order {o_i}, frame {f}")
        if o_i == 0:
            for k in (0, 3, 7, 9):
                check_oracle(got[k], vs[k], built_nodes[k], ws[k], f"{name} mesh {k}")
            for k, (g, w, v) in enumerate(zip(got, want, ws)):
                assert walks(g, v, k) == walks(w, v, k), f"{name}, keep {keep}: walks of handle {k}"


def test_batch_converted_and_batch_built_handles(gpu):
    meshes = [mesh(n, 500 + k) for k, n in enumerate([3, 60, 400, 2500, 9000])]
    for keep in (0, 1):
        got = api.convert_batch(api.build_batch([api.BVH() for _ in meshes], meshes, _lib.BUILD_AVX))
        api.check(_lib.lib().tbvh_convert(got[1].h, api.LAYOUT_BVH_GPU))
        want = [convert(built(v, "BuildAVX")) for v in meshes]
        api.check(_lib.lib().tbvh_convert(want[1].h, api.LAYOUT_BVH_GPU))
        assert_same(got, want, "before the refit")
        for f in (1, 2):
            ws = [frame(v, f) for v in meshes]
            api.refit_batch(got, ws, keep_layouts=keep)
            for b, w in zip(want, ws):
                single(b, w, keep)
            assert_same(got, want, f"keep {keep}, frame {f}")


def test_uploaded_families_and_one_node_trees(gpu):
    v = mesh(3000, 41)
    src = util.source_tree(v, "Build")
    items = [one_node_tree(3, 1)] + [(util.family_tree(src, fam, 5 + k), v) for k, fam in enumerate(util.FAMILIES)]
    items = items[:3] + [one_node_tree(7, 4)] + items[3:] + [(None, mesh(40, 5)), one_node_tree(1, 6)]
    make = [(lambda t=t, x=x: uploaded(t, x) if t is not None else built(x, "Build")) for t, x in items]
    meshes = [x for _, x in items]
    for keep in (0, 1):
        got = [convert(m()) for m in make]
        want = [convert(m()) for m in make]
        for f in (1, 2):
            ws = [frame(x, f) for x in meshes]
            api.refit_batch(got, ws, keep_layouts=keep)
            for b, w in zip(want, ws):
                single(b, w, keep)
            assert_same(got, want, f"uploaded, keep {keep}, frame {f}")
        for k, (g, w, x) in enumerate(zip(got, want, ws)):
            assert walks(g, x, k) == walks(w, x, k), f"uploaded {k}, keep {keep}: walks"


def test_offatrium_neighbours(gpu):
    base = mesh(2000, 31)
    named = [("plain", mesh(1500, 32))]
    for mode in ("pos", "neg", "random"):
        named.append((f"signed zero {mode}", util.signed_zero(base, mode, seed=3)))
    for k in (-126, -20, 40, 90):
        named.append((f"scaled 2^{k}", util.scaled(base, k)))
    named += [("translated", util.translated(base, 3e5)), ("plain small", mesh(90, 33))]
    meshes = [x for _, x in named]
    got = [convert(built(x, "Build")) for x in meshes]
    want = [convert(built(x, "Build")) for x in meshes]
    for f in (1, 2):
        ws = [frame(x, f) for x in meshes]
        api.refit_batch(got, ws, keep_layouts=1)
        for b, w in zip(want, ws):
            single(b, w, 1)
        for k, (label, _) in enumerate(named):
            assert_same([got[k]], [want[k]], f"{label}, frame {f}")
    # axis-aligned rays with rD = 1e30: the 2^40 tree's integer-path bound moved, its neighbours' did not
    for k, (label, x) in enumerate(named):
        lo, hi = scenes.scene_bounds(ws[k])
        rays = util.axis_rays(lo, hi)
        for b in (got[k], want[k]):
            b.layout = api.LAYOUT_CWBVH
        a, c = rays.copy(), rays.copy()
        got[k].Intersect(a), want[k].Intersect(c)
        assert util.compare_hits(util.nan_canonical(a), util.nan_canonical(c)) == ZERO, label
        assert walks(got[k], ws[k], k) == walks(want[k], ws[k], k), label


@pytest.mark.parametrize("stride", [12, 16, 32])
def test_strides_host_and_device(gpu, stride):
    import torch
    meshes = [mesh(n, 600 + k) for k, n in enumerate([5, 700, 4000])]
    for device in (False, True):
        got = [with_layouts(built(v, "BuildAVX"), "all") for v in meshes]
        want = [with_layouts(built(v, "BuildAVX"), "all") for v in meshes]
        ws = [frame(v, 1) for v in meshes]
        for w in ws:
            w[:, 3] = np.arange(w.shape[0], dtype=np.float32)   # a stride below 16 leaves w alone: bvh8Tris shows it
        wide = [np.concatenate([w, np.full((w.shape[0], stride // 4 - 4), 7, np.float32)], 1) if stride > 16 else np.ascontiguousarray(w[:, : stride // 4]) for w in ws]
        if device:
            t = [torch.from_numpy(x).cuda() for x in wide]
            torch.cuda.synchronize()
            recs = (_lib.Mesh * len(t))()
            for r, x in zip(recs, t):
                r.verts, r.stride, r.vert_count, r.indices, r.prim_count = x.data_ptr(), stride, 0, None, x.shape[0] // 3
            hs = (C.c_void_p * len(got))(*[b.h for b in got])
            api.check(_lib.lib().tbvh_refit_batch(hs, recs, len(t), api.DEVICE, 1))
        else:
            api.check(raw_refit_batch([b.h for b in got], wide, stride=stride))
        for b, x in zip(want, wide):
            api.check(_lib.lib().tbvh_refit_layouts(b.h, x.ctypes.data, stride, x.shape[0] // 3, api.HOST))
        assert_same(got, want, f"stride {stride}, device {device}")


def test_refusals_leave_handles_as_they_were(gpu):
    meshes = [mesh(n, 700 + k) for k, n in enumerate([30, 800])]
    good = [with_layouts(built(v, "Build"), "all") for v in meshes]
    h = [b.h.value for b in good]
    hq = api.BVH().BuildHQ(meshes[0])
    empty = api.BVH()
    up_cw = api.BVH().upload(*api.BVH.download(good[0]), meshes[0])
    d, t = cw(good[0])
    api.check(_lib.lib().tbvh_upload_cwbvh(up_cw.h, d.ctypes.data, d.shape[0], t.ctypes.data, t.shape[0] // 3, api.HOST))
    v0, inst, O, D = tlas_case(111, 6)
    tl = api.TLAS().Build(inst, [built(x, "Build") for x in v0])
    ctx2 = C.c_void_p()
    api.check(_lib.lib().tbvh_ctx_create(0, C.byref(ctx2)))
    other = C.c_void_p()
    api.check(_lib.lib().tbvh_bvh_create(ctx2, C.byref(other)))
    ws = [frame(v, 1) for v in meshes]
    short = ws[1][:-3].copy()
    idx = (C.c_uint32 * 3)(0, 1, 2)
    try:
        everyone = good + [hq, up_cw, tl]
        before = [snapshot(b) for b in everyone]
        cases = [("count 0", [], [], {}, _lib.E_ARG), ("NULL handle", [h[0], None], ws, {}, _lib.E_ARG),
                 ("repeated handle", [h[0], h[0]], ws, {}, _lib.E_ARG), ("two contexts", [h[0], other.value], ws, {}, _lib.E_ARG),
                 ("indices", h, ws, {"indices": C.cast(idx, C.c_void_p).value}, _lib.E_ARG), ("unknown space", h, ws, {"space": 5}, _lib.E_ARG),
                 ("keep 2", h, ws, {"keep": 2}, _lib.E_ARG), ("no tree", [h[0], empty.h.value], ws, {}, _lib.E_STATE),
                 ("SBVH", [h[0], hq.h.value], [ws[0], meshes[0]], {}, _lib.E_STATE), ("TLAS", [h[1], tl.h.value], [ws[1], ws[0]], {}, _lib.E_STATE),
                 ("uploaded CWBVH", [h[1], up_cw.h.value], [ws[1], ws[0]], {}, _lib.E_STATE),
                 ("prim_count", h, [ws[0], short], {}, _lib.E_ARG), ("stride", h, ws, {"stride": 14}, _lib.E_ARG)]
        for what, hs, vs, kw, code in cases:
            if what == "count 0":
                assert _lib.lib().tbvh_refit_batch((C.c_void_p * 1)(h[0]), (_lib.Mesh * 1)(), 0, api.HOST, 1) == code, what
            else:
                assert raw_refit_batch(hs, vs, **kw) == code, what
            assert [snapshot(b) for b in everyone] == before, f"{what}: a refused batch changed a handle"
        # the same uploaded CWBVH is accepted with keep_layouts = 0, and dropped
        assert raw_refit_batch([h[1], up_cw.h.value], [ws[1], ws[0]], keep=0) == _lib.OK
        assert up_cw.info().layouts == 1 << api.LAYOUT_BVH
        with pytest.raises(api.TbvhError, match="error -3"):
            api.refit_batch([good[0], empty], ws)
    finally:
        _lib.lib().tbvh_bvh_destroy(other)
        _lib.lib().tbvh_ctx_destroy(ctx2)


def tlas_words(r):
    return r.view(np.uint32).reshape(-1, 32)[:, 11:16]   # hit.inst, t, u, v, prim


def test_tlas_staleness_and_two_level_walk(gpu):
    v, inst, O, D = tlas_case(113, 30)
    rays = R.make_rays(O, D)
    for keep in (0, 1):
        blas = [built(x, "Build") for x in v]
        for b in blas[::2]:
            convert(b)
        t = api.TLAS().Build(inst.copy(), blas)
        api.refit_batch(blas[1::2], [frame(x, 1) for x in v[1::2]], keep_layouts=keep)   # BLASes without a CWBVH
        r = rays.copy()
        assert _lib.lib().tbvh_intersect(t.h, api.LAYOUT_BVH, r.ctypes.data, 128, 64) == (_lib.E_STATE if keep else _lib.OK), f"keep {keep}: BLASes without a CWBVH"
        t = api.TLAS().Build(inst.copy(), blas)
        api.refit_batch(blas[::2], [frame(x, 1) for x in v[::2]], keep_layouts=keep)     # BLASes holding a CWBVH
        r = rays.copy()
        assert _lib.lib().tbvh_intersect(t.h, api.LAYOUT_BVH, r.ctypes.data, 128, 64) == _lib.E_STATE, f"keep {keep}: BLASes holding a CWBVH"
    # rebuilt over the refitted BLASes, the two-level walk in both layouts is the oracle's
    w = [frame(x, 2) for x in v]
    blas = [convert(built(x, "Build")) for x in v]
    api.refit_batch(blas, w, keep_layouts=1)
    for layout in (api.LAYOUT_BVH, api.LAYOUT_CWBVH):
        t = api.TLAS().Build(inst.copy(), blas, blas_layout=layout)
        want = [portpy.PortBVH(x, nodes=api.BVH.download(b)[0], prim_idx=api.BVH.download(b)[1]) for x, b in zip(w, blas)]
        if layout == api.LAYOUT_BVH:
            nodes, idx = t.download()
            port = portpy.PortTLAS(nodes, idx, t_inst(t, inst, blas), want)
        else:
            class _CW:
                def __init__(self, b):
                    self.nodes, self.tris = (a.view(np.float32) for a in cw(b))
            nodes, idx = t.download()
            port = portpy.PortTLASCW(nodes, idx, t_inst(t, inst, blas), [_CW(b) for b in blas])
        a, c = rays.copy(), rays.copy()
        port.intersect(a), t.Intersect(c)
        assert np.array_equal(tlas_words(c), tlas_words(a)), f"two-level walk, layout {layout}"


def t_inst(t, inst, blas):
    """the instance records TLAS.Build updated against the refitted BLAS boxes"""
    out = inst.copy()
    for i in range(out.shape[0]):
        api.check(_lib.lib().tbvh_instance_update(C.c_void_p(out[i:i + 1].ctypes.data), blas[int(out["blasIdx"][i])].h))
    return out


def test_launch_count_determinism_and_replica(gpu):
    v = mesh(2000, 77)
    objs = [with_layouts(built(v, "BuildAVX"), "all") for _ in range(200)]
    w = frame(v, 1)
    n0 = api.launch_count()
    api.refit_batch(objs[:2], [w] * 2, keep_layouts=1)
    n_two = api.launch_count() - n0
    n0 = api.launch_count()
    api.refit_batch(objs, [w] * 200, keep_layouts=1)
    n_all = api.launch_count() - n0
    assert n_two == n_all, (n_two, n_all)
    n0 = api.launch_count()
    for b in objs[:20]:
        single(b, w, 1)
    n_loop = api.launch_count() - n0
    assert n_all * 5 < n_loop, (n_all, n_loop)
    first = [snapshot(b) for b in objs]
    api.refit_batch(objs, [w] * 200, keep_layouts=1)
    assert [snapshot(b) for b in objs] == first, "two identical batches differ"
    # a group replica of a batch-refitted handle walks like its source
    src = objs[7]
    src.layout = api.LAYOUT_CWBVH
    g = api.Group([0])
    g.replicate(src)
    sets, _ = util.ray_sets(w, res=24)
    want, got = sets["primary"].copy(), sets["primary"].copy()
    src.Intersect(want)
    g.Intersect(got)
    assert util.compare_hits(got, want) == ZERO


def test_api_class_rule(gpu):
    v = mesh(500, 88)
    w = frame(v, 1)
    plain, wide, gpu_obj = api.BVH().Build(v), api.BVH8_CWBVH().Build(v), api.BVH_GPU().Build(v)
    convert(plain)
    api.refit_batch([plain], [w])                    # BVH: tbvh_refit drops the CWBVH
    assert plain.info().layouts == 1 << api.LAYOUT_BVH
    api.refit_batch([wide, gpu_obj], [w, w])         # BVH_GPU / BVH8_CWBVH: tbvh_refit_layouts keeps them
    assert wide.info().layouts & (1 << api.LAYOUT_CWBVH) and gpu_obj.info().layouts & (1 << api.LAYOUT_BVH_GPU)
    twin = api.BVH8_CWBVH().Build(v)
    twin.Refit(w)
    assert snapshot(wide) == snapshot(twin)
    before = [snapshot(b) for b in (plain, wide)]
    with pytest.raises(api.TbvhError, match="keep_layouts"):
        api.refit_batch([plain, wide], [v, v])
    assert [snapshot(b) for b in (plain, wide)] == before
    api.refit_batch([plain, wide], [v, v], keep_layouts=1)
    assert wide.info().layouts & (1 << api.LAYOUT_CWBVH)
