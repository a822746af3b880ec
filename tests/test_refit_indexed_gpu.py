"""GPU parity of tbvh_refit_batch_indexed / api.refit_batch_indexed: a tree built from (V, I) and refitted from the moved vertices V'
through the indices it kept is exactly its twin - built the same way and refitted by tbvh_refit / tbvh_refit_layouts from the flat soup
V'[I] at the same stride: BVH2, primIdx, BVH_GPU, bvh8Data / bvh8Tris, info, walks, generation.  The flat refit is held to the oracle
(tests/test_refit_batch_gpu.py), and so is the BVH2 here.  Two frames each: the second refits from the first frame's boxes."""
import ctypes as C

import numpy as np
import pytest

from oracle import refpy
from tinybvh_b200 import _lib, api, rays as R
from tests import util
from tests.test_convert_batch_gpu import built, convert, mesh
from tests.test_oracle_pin import tlas_case
from tests.test_refit_batch_gpu import SUBSETS, check_oracle, cw, snapshot, tlas_words, walks, with_layouts

pytestmark = pytest.mark.gpu
FLAVOUR = {"Build": _lib.BUILD_REFERENCE, "BuildAVX": _lib.BUILD_AVX}
OBJECTS = {"bvh": ("bvh", 0), "bvh_gpu": ("bvh+gpu", 1), "cwbvh": ("bvh+cw", 1)}   # layouts held by BVH / BVH_GPU / BVH8_CWBVH objects, their keep_layouts


def L():
    return _lib.lib()


def grid(nx, ny, seed, shuffle=False, unused=0):
    """A welded deformed grid around the origin: (nx + 1)(ny + 1) vertices shared by 2 nx ny triangles (about six triangles per vertex),
    random w; shuffle: triangles and their corners in random order; unused: vertices past the grid that no triangle references."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:ny + 1, 0:nx + 1].astype(np.float32)
    n = x.size
    V = np.zeros((n + unused, 4), np.float32)
    V[:n, 0], V[:n, 1] = (x.ravel() - nx / 2) * 0.25, (y.ravel() - ny / 2) * 0.25
    V[:n, 2] = np.sin(x.ravel() * 0.3) * np.cos(y.ravel() * 0.2) + rng.random(n, np.float32) * 0.05
    V[n:, :3] = rng.random((unused, 3), np.float32) * 50 - 25
    V[:, 3] = rng.random(V.shape[0], np.float32)
    a = (np.arange(ny)[:, None] * (nx + 1) + np.arange(nx)[None, :]).ravel()
    I = np.stack([a, a + 1, a + nx + 1, a + 1, a + nx + 2, a + nx + 1], 1).reshape(-1, 3)
    if shuffle:
        I = I[rng.permutation(I.shape[0])]
        I = np.take_along_axis(I, np.argsort(rng.random(I.shape), 1), 1)
    return V, np.ascontiguousarray(I.reshape(-1), np.uint32)


def same(v):
    return v


def shapes():
    """(label, base vertices, indices, family): a frame's vertices are family( moved base )"""
    out = [("welded grid", *grid(40, 30, 1), same), ("shuffled", *grid(25, 25, 2, shuffle=True), same),
           ("unused vertices", *grid(12, 9, 3, unused=50), same)]
    v = mesh(300, 4)
    out.append(("vert_count = 3 prim_count", v, np.arange(v.shape[0], dtype=np.uint32)[::-1].copy(), same))
    v, i = grid(8, 8, 5)
    i = i.reshape(-1, 3).copy()
    i[::3, 2] = i[::3, 0]
    out.append(("repeated vertex", v, np.ascontiguousarray(i.reshape(-1)), same))
    out.append(("one triangle", np.array([[0, 0, 0, 1], [1, 0, 0, 2], [0, 1, 0.5, 3]], np.float32), np.array([2, 0, 1], np.uint32), same))
    base, i = grid(30, 20, 6, shuffle=True)
    for mode in ("pos", "neg", "random"):
        out.append((f"signed zero {mode}", base, i, lambda v, m=mode: util.signed_zero(v, m, seed=3)))
    for k in (-126, 40, 90):
        out.append((f"scaled 2^{k}", base, i, lambda v, k=k: util.scaled(v, k)))
    out.append(("translated", base, i, lambda v: util.translated(v, 3e5)))
    return out


def move(v, f, seed):
    """frame f of an animation: every vertex displaced a little, new random w (frame 0: the vertices themselves)"""
    if f == 0:
        return v.copy()
    rng = np.random.default_rng(1000 * f + seed)
    w = v.copy()
    ext = float((v[:, :3].max(0) - v[:, :3].min(0)).max()) or 1.0
    w[:, :3] += (rng.random((v.shape[0], 3), np.float32) - 0.5) * np.float32(0.02 * ext)
    w[:, 3] = rng.random(v.shape[0], np.float32)
    return w


def at_stride(v, stride):
    """rows `stride` bytes apart: xyz (12), xyzw (16), xyzw and padding (32)"""
    if stride == 12:
        return np.ascontiguousarray(v[:, :3])
    if stride == 16:
        return np.ascontiguousarray(v)
    return np.ascontiguousarray(np.concatenate([v, np.full((v.shape[0], stride // 4 - 4), 7, np.float32)], 1))


def build_indexed(v, i, name="Build", stride=16):
    b = api.BVH()
    s = at_stride(v, stride)
    api.check(L().tbvh_build_indexed(b.h, s.ctypes.data, stride, v.shape[0], i.ctypes.data, i.shape[0] // 3, api.HOST, 1.0, 1.0, FLAVOUR[name]))
    b.vert_count = v.shape[0]
    return b


def build_flat(v, name="Build", stride=16):
    b = api.BVH()
    s = at_stride(v, stride)
    api.check(L().tbvh_build_flavour(b.h, s.ctypes.data, stride, v.shape[0] // 3, api.HOST, 1.0, 1.0, FLAVOUR[name]))
    return b


def build_batch(items, name, stride):
    """tbvh_build_batch of (vertices, indices or None) items at one stride"""
    bs = [api.BVH() for _ in items]
    arrays = [at_stride(v, stride) for v, _ in items]
    recs = (_lib.Mesh * len(items))()
    for r, a, (v, i) in zip(recs, arrays, items):
        if i is None:
            r.verts, r.stride, r.vert_count, r.indices, r.prim_count = a.ctypes.data, stride, 0, None, v.shape[0] // 3
        else:
            r.verts, r.stride, r.vert_count, r.indices, r.prim_count = a.ctypes.data, stride, v.shape[0], i.ctypes.data, i.shape[0] // 3
    hs = (C.c_void_p * len(bs))(*[b.h for b in bs])
    api.check(L().tbvh_build_batch(hs, recs, len(items), api.HOST, 1.0, 1.0, FLAVOUR[name]))
    for b, (v, i) in zip(bs, items):
        b.vert_count = 0 if i is None else v.shape[0]
    return bs


def raw(handles, meshes, space=api.HOST, keep=0):
    """tbvh_refit_batch_indexed; meshes: (vertex pointer, stride, vert_count, indices pointer, prim_count)"""
    recs = (_lib.Mesh * max(len(meshes), 1))(*[_lib.Mesh(*m) for m in meshes])
    hs = (C.c_void_p * max(len(handles), 1))(*handles)
    return L().tbvh_refit_batch_indexed(hs, recs, len(meshes), space, keep)


def flat_refit(b, soup, stride, keep):
    """the twin's refit: tbvh_refit / tbvh_refit_layouts of the flat soup"""
    fn = L().tbvh_refit_layouts if keep else L().tbvh_refit
    api.check(fn(b.h, soup.ctypes.data, stride, soup.shape[0] // 3, api.HOST))


def soup(v, i):
    return np.ascontiguousarray(v[i])


def ix_mesh(ptr, stride, v, i):
    return (ptr, stride, v.shape[0], None, i.shape[0] // 3)


def assert_twins(got, want, labels, what):
    for k, (g, w) in enumerate(zip(got, want)):
        assert snapshot(g) == snapshot(w), f"{what}: {labels[k]} differs from its twin"


def make_twins(items, flats, name, source, stride, subset):
    """two identical handle lists: the items built from (V, I) - by tbvh_build_indexed, or all in one tbvh_build_batch -, then the flat
    meshes, each holding the layouts of `subset`"""
    out = []
    for _ in range(2):
        if source == "batch":
            bs = build_batch([(fam(base), i) for _, base, i, fam in items] + [(v, None) for _, v in flats], name, stride)
        else:
            bs = [build_indexed(fam(base), i, name, stride) for _, base, i, fam in items] + [build_flat(v, name, stride) for _, v in flats]
        out.append([with_layouts(b, subset) for b in bs])
    return out


@pytest.mark.parametrize("obj", list(OBJECTS))
@pytest.mark.parametrize("source", ["indexed", "batch"])
@pytest.mark.parametrize("name", ["Build", "BuildAVX"])
def test_indexed_refit_is_the_flat_refit_of_the_soup(gpu, name, source, obj):
    import torch
    subset, keep = OBJECTS[obj]
    items = shapes()
    flats = [("flat plain", mesh(700, 9)), ("flat small", mesh(2, 10))]   # flat meshes of the same calls
    labels = [x[0] for x in items] + [x[0] for x in flats]
    for stride in (12, 16, 32):
        for device in (False, True):
            got, want = make_twins(items, flats, name, source, stride, subset)
            built_nodes = [api.BVH.download(b)[0] for b in got]
            for f in (1, 2):
                ws = [fam(move(base, f, k)) for k, (_, base, i, fam) in enumerate(items)]
                fs = [move(v, f, 100 + k) for k, (_, v) in enumerate(flats)]
                arrays = [at_stride(w, stride) for w in ws + fs]
                if device:
                    arrays = [torch.from_numpy(a).cuda() for a in arrays]
                    torch.cuda.synchronize()
                ptrs = [a.data_ptr() if device else a.ctypes.data for a in arrays]
                meshes = [ix_mesh(p, stride, w, i) for p, w, (_, _, i, _) in zip(ptrs, ws, items)]
                meshes += [(p, stride, 0, None, v.shape[0] // 3) for p, v in zip(ptrs[len(items):], fs)]
                handles = [b.h.value for b in got]
                space = api.DEVICE if device else api.HOST
                if f == 1:
                    api.check(raw(handles, meshes, space, keep))          # one call for the scene
                else:
                    for h, m in zip(handles, meshes):
                        api.check(raw([h], [m], space, keep))             # count = 1: a single handle
                for b, w, (_, _, i, _) in zip(want, ws, items):
                    flat_refit(b, at_stride(soup(w, i), stride), stride, keep)
                for b, v in zip(want[len(items):], fs):
                    flat_refit(b, at_stride(v, stride), stride, keep)
                what = f"{name} {source} {obj}, stride {stride}, {'device' if device else 'host'}, frame {f}"
                assert_twins(got, want, labels, what)
                if stride == 16 and not device:
                    for k in range(len(items)):
                        w_soup = soup(ws[k], items[k][2])
                        check_oracle(got[k], soup(items[k][3](items[k][1]), items[k][2]), built_nodes[k], w_soup, f"{what}: {labels[k]}")
                        assert walks(got[k], w_soup, k) == walks(want[k], w_soup, k), f"{what}: walks of {labels[k]}"


def test_batches_mixed_layouts_order_and_neighbours(gpu):
    """indexed and flat meshes of every off-atrium family and held-layout subset in one call, in three orders: every handle is its
    twin's bytes, and the same bytes whatever the order"""
    items = shapes()
    flats = [("flat plain", mesh(1500, 12)), ("flat tiny", mesh(1, 13))]
    n = len(items) + len(flats)
    labels = [x[0] for x in items] + [x[0] for x in flats]
    rng = np.random.default_rng(7)
    for keep in (0, 1):
        first = None
        for o_i, order in enumerate((list(range(n)), list(range(n))[::-1], list(rng.permutation(n)))):
            def make(k):
                if k < len(items):
                    _, base, i, fam = items[k]
                    b = build_indexed(fam(base), i, "BuildAVX")
                else:
                    b = build_flat(flats[k - len(items)][1], "BuildAVX")
                return with_layouts(b, SUBSETS[k % 4])
            got, want = [make(k) for k in order], [make(k) for k in order]
            for f in (1, 2):
                ws = [fam(move(base, f, k)) for k, (_, base, i, fam) in enumerate(items)] + [move(v, f, 50 + k) for k, (_, v) in enumerate(flats)]
                meshes = [ix_mesh(ws[k].ctypes.data, 16, ws[k], items[k][2]) if k < len(items) else (ws[k].ctypes.data, 16, 0, None, ws[k].shape[0] // 3) for k in order]
                api.check(raw([b.h.value for b in got], meshes, keep=keep))
                for b, k in zip(want, order):
                    flat_refit(b, soup(ws[k], items[k][2]) if k < len(items) else ws[k], 16, keep)
                assert_twins(got, want, [labels[k] for k in order], f"keep {keep}, order {o_i}, frame {f}")
            snaps = {k: snapshot(b) for b, k in zip(got, order)}
            if first is None:
                first = snaps
            assert snaps == first, f"keep {keep}: order {o_i} changed a tree"


def test_kept_indices_survive_refits_and_conversions_and_go_with_the_tree(gpu):
    v, i = grid(20, 20, 11, shuffle=True)
    p = i.shape[0] // 3
    got, want = build_indexed(v, i), build_indexed(v, i)
    w1, w2, w3 = (move(v, f, 0) for f in (1, 2, 3))
    for b in (got, want):
        flat_refit(b, soup(w1, i), 16, 0)                          # a flat refit
        api.check(L().tbvh_convert(b.h, api.LAYOUT_BVH_GPU))       # conversions
        convert(b)
        api.check(L().tbvh_convert_batch((C.c_void_p * 1)(b.h), 1, api.LAYOUT_CWBVH))
    api.check(raw([got.h.value], [ix_mesh(w2.ctypes.data, 16, w2, i)], keep=1))
    flat_refit(want, soup(w2, i), 16, 1)
    assert snapshot(got) == snapshot(want)
    gpu_nodes = api.BVH_GPU.download(want)
    other = build_indexed(*grid(5, 5, 12))
    inst = refpy.make_instances(util.random_transforms(4, 13), [0] * 4)
    for k in range(inst.shape[0]):
        api.check(L().tbvh_instance_update(C.c_void_p(inst[k:k + 1].ctypes.data), other.h))
    replace = [("flat rebuild", lambda b: api.check(L().tbvh_build(b.h, soup(w3, i).ctypes.data, 16, p, api.HOST, 1.0, 1.0))),
               ("flat batch rebuild", lambda b: api.check(L().tbvh_build_batch((C.c_void_p * 1)(b.h), (_lib.Mesh * 1)(_lib.Mesh(soup(w3, i).ctypes.data, 16, 0, None, p)), 1, api.HOST, 1.0, 1.0, _lib.BUILD_AVX))),
               ("upload", lambda b: b.upload(*api.BVH.download(want), soup(w3, i))),
               ("BVH_GPU upload", lambda b: api.BVH_GPU.upload(b, gpu_nodes, api.BVH.download(want)[1], soup(w3, i))),
               ("TLAS build", lambda b: api.check(L().tbvh_build_tlas(b.h, inst.ctypes.data, 192, inst.shape[0], (C.c_void_p * 1)(other.h), 1, 1.0, 1.0))),
               ("indexed BuildHQ", lambda b: b.BuildHQ(v, indices=i)),
               ("batch BuildHQ", lambda b: api.build_batch([b], [v], _lib.BUILD_HQ, indices=[i]))]
    for what, fn in replace:
        b = build_indexed(v, i)
        fn(b)
        before = snapshot(b)
        assert raw([b.h.value], [ix_mesh(w3.ctypes.data, 16, w3, i)]) == _lib.E_STATE, what
        assert snapshot(b) == before, what


def test_refusals_leave_handles_and_a_tlas_over_them_as_they_were(gpu):
    v, i = grid(15, 12, 21, shuffle=True)
    p = i.shape[0] // 3
    fv = mesh(400, 22)
    a = with_layouts(build_indexed(v, i), "all")
    fl = with_layouts(built(fv, "Build"), "all")
    hq = api.BVH().BuildHQ(v, indices=i)
    hqb = api.build_batch([api.BVH()], [v], _lib.BUILD_HQ, indices=[i])[0]
    empty = api.BVH()
    up_cw = build_indexed(v, i)
    d, t = cw(a)
    api.check(L().tbvh_upload_cwbvh(up_cw.h, d.ctypes.data, d.shape[0], t.ctypes.data, t.shape[0] // 3, api.HOST))
    _, inst, O, D = tlas_case(117, 12)
    tl = api.TLAS().Build(inst.copy(), [a, fl])
    rays = R.make_rays(O, D)
    ctx2 = C.c_void_p()
    api.check(L().tbvh_ctx_create(0, C.byref(ctx2)))
    other = C.c_void_p()
    api.check(L().tbvh_bvh_create(ctx2, C.byref(other)))
    w, wf = move(v, 1, 0), move(fv, 1, 1)
    ok_a, ok_f = ix_mesh(w.ctypes.data, 16, w, i), (wf.ctypes.data, 16, 0, None, wf.shape[0] // 3)
    idx = (C.c_uint32 * 3)(0, 1, 2)
    ip = C.cast(idx, C.c_void_p).value
    ha, hf = a.h.value, fl.h.value
    try:
        everyone = [a, fl, hq, hqb, up_cw, tl]
        before = [snapshot(b) for b in everyone]
        hits = rays.copy()
        api.check(L().tbvh_intersect(tl.h, api.LAYOUT_BVH, hits.ctypes.data, 128, hits.shape[0]))
        cases = [("NULL handle", [ha, None], [ok_a, ok_f], {}, _lib.E_ARG), ("repeated handle", [ha, ha], [ok_a, ok_a], {}, _lib.E_ARG),
                 ("two contexts", [ha, other.value], [ok_a, ok_a], {}, _lib.E_ARG), ("unknown space", [ha, hf], [ok_a, ok_f], {"space": 5}, _lib.E_ARG),
                 ("keep 2", [ha, hf], [ok_a, ok_f], {"keep": 2}, _lib.E_ARG),
                 ("indices", [ha, hf], [(w.ctypes.data, 16, v.shape[0], ip, p), ok_f], {}, _lib.E_ARG),
                 ("indices on a flat mesh", [ha, hf], [ok_a, (wf.ctypes.data, 16, 0, ip, wf.shape[0] // 3)], {}, _lib.E_ARG),
                 ("vert_count other than the build's", [hf, ha], [ok_f, (w.ctypes.data, 16, v.shape[0] - 1, None, p)], {}, _lib.E_ARG),
                 ("vert_count on a flat-built handle", [ha, hf], [ok_a, (wf.ctypes.data, 16, wf.shape[0], None, wf.shape[0] // 3)], {}, _lib.E_STATE),
                 ("no tree", [ha, empty.h.value], [ok_a, ok_a], {}, _lib.E_STATE),
                 ("indexed SBVH", [ha, hq.h.value], [ok_a, ok_a], {}, _lib.E_STATE),
                 ("batch-built SBVH", [ha, hqb.h.value], [ok_a, ok_a], {}, _lib.E_STATE),
                 ("TLAS", [hf, tl.h.value], [ok_f, ok_a], {}, _lib.E_STATE),
                 ("uploaded CWBVH", [hf, up_cw.h.value], [ok_f, ok_a], {"keep": 1}, _lib.E_STATE),
                 ("prim_count", [hf, ha], [ok_f, (w.ctypes.data, 16, v.shape[0], None, p - 1)], {}, _lib.E_ARG),
                 ("stride", [ha], [(w.ctypes.data, 14, v.shape[0], None, p)], {}, _lib.E_ARG)]
        assert L().tbvh_refit_batch_indexed((C.c_void_p * 1)(ha), (_lib.Mesh * 1)(_lib.Mesh(*ok_a)), 0, api.HOST, 0) == _lib.E_ARG, "count 0"
        for what, hs, ms, kw, code in [("count 0", None, None, None, None)] + cases:
            if hs is not None:
                assert raw(hs, ms, **kw) == code, what
            assert [snapshot(b) for b in everyone] == before, f"{what}: a refused call changed a handle"
            r = rays.copy()
            assert L().tbvh_intersect(tl.h, api.LAYOUT_BVH, r.ctypes.data, 128, r.shape[0]) == _lib.OK, f"{what}: the TLAS went stale"
            assert util.compare_hits(r, hits) == {"prim": 0, "t": 0, "u": 0, "v": 0}, what
        # the uploaded CWBVH refits with keep_layouts = 0 and is dropped; an SBVH refuses a flat slice too
        assert raw([hf, up_cw.h.value], [ok_f, ok_a], keep=0) == _lib.OK
        assert up_cw.info().layouts == 1 << api.LAYOUT_BVH
        assert raw([hq.h.value], [(soup(w, i).ctypes.data, 16, 0, None, p)]) == _lib.E_STATE
        with pytest.raises(api.TbvhError, match="error -3"):
            api.refit_batch_indexed([a, empty], [w, w])
    finally:
        L().tbvh_bvh_destroy(other)
        L().tbvh_ctx_destroy(ctx2)


def test_tlas_staleness_and_update_follow_the_twin(gpu):
    _, inst, O, D = tlas_case(119, 30)
    rays = R.make_rays(O, D)
    meshes = [grid(60, 40, 31, shuffle=True), grid(12, 12, 32)]
    for m in meshes:
        m[0][:, :3] *= 4
    for keep in (0, 1):
        got = [with_layouts(build_indexed(v, i), "bvh+cw") for v, i in meshes]
        want = [with_layouts(build_indexed(v, i), "bvh+cw") for v, i in meshes]
        tg, tw = api.TLAS().Build(inst.copy(), got), api.TLAS().Build(inst.copy(), want)
        ws = [move(v, 1, k) for k, (v, _) in enumerate(meshes)]
        api.check(raw([b.h.value for b in got], [ix_mesh(w.ctypes.data, 16, w, i) for w, (_, i) in zip(ws, meshes)], keep=keep))
        for b, w, (_, i) in zip(want, ws, meshes):
            flat_refit(b, soup(w, i), 16, keep)
        for t in (tg, tw):
            r = rays.copy()
            assert L().tbvh_intersect(t.h, api.LAYOUT_BVH, r.ctypes.data, 128, r.shape[0]) == _lib.E_STATE, f"keep {keep}: the TLAS is stale"
        ig, iw = inst.copy(), inst.copy()
        tg.Rebuild(ig, got)
        tw.Rebuild(iw, want)
        assert ig.tobytes() == iw.tobytes(), f"keep {keep}: updated records"
        assert snapshot(tg) == snapshot(tw), f"keep {keep}: TLAS"
        for layout in (api.LAYOUT_BVH, api.LAYOUT_CWBVH) if keep else (api.LAYOUT_BVH,):
            tg.layout = tw.layout = layout
            a, c = rays.copy(), rays.copy()
            tg.Intersect(a), tw.Intersect(c)
            assert np.array_equal(tlas_words(a), tlas_words(c)), f"keep {keep}: two-level walk, layout {layout}"
            assert (tlas_words(a)[:, 1].view(np.float32) < 1e30).any(), "no ray hits the scene"


def test_python_refit_batch_indexed(gpu):
    import torch
    v, i = grid(25, 18, 41, shuffle=True)
    fv = mesh(600, 42)
    for device in (False, True):
        objs = [api.BVH8_CWBVH().Build(v, indices=i), api.BVH8_CWBVH().Build(fv)]
        twins = [api.BVH8_CWBVH().Build(v, indices=i), api.BVH8_CWBVH().Build(fv)]
        assert objs[0].vert_count == v.shape[0] and objs[1].vert_count == 0
        for f in (1, 2):
            w, wf = move(v, f, 0), move(fv, f, 1)
            args = [torch.from_numpy(w).cuda(), torch.from_numpy(wf).cuda()] if device else [w, wf]
            api.refit_batch_indexed(objs, args)
            api.refit_batch(twins, [soup(w, i), wf])
            assert [snapshot(o) for o in objs] == [snapshot(t) for t in twins], f"device {device}, frame {f}"
    # batch-built objects, BVH and BVH_GPU ones in one call with an explicit keep_layouts
    bb = api.build_batch([api.BVH(), api.BVH_GPU()], [v, fv], _lib.BUILD_AVX, indices=[i, None])
    tw = api.build_batch([api.BVH(), api.BVH_GPU()], [v, fv], _lib.BUILD_AVX, indices=[i, None])
    assert bb[0].vert_count == v.shape[0] and bb[1].vert_count == 0
    with pytest.raises(api.TbvhError, match="keep_layouts"):
        api.refit_batch_indexed(bb, [w, wf])
    api.refit_batch_indexed(bb, [w, wf], keep_layouts=1)
    api.refit_batch(tw, [soup(w, i), wf], keep_layouts=1)
    assert [snapshot(o) for o in bb] == [snapshot(t) for t in tw]


def test_one_extra_launch_and_determinism(gpu):
    meshes = [grid(30 + k, 20, 60 + k, shuffle=True) for k in range(50)]
    got = [with_layouts(build_indexed(v, i, "BuildAVX"), "all") for v, i in meshes]
    want = [with_layouts(build_indexed(v, i, "BuildAVX"), "all") for v, i in meshes]
    ws = [move(v, 1, k) for k, (v, _) in enumerate(meshes)]
    soups = [soup(w, i) for w, (_, i) in zip(ws, meshes)]
    n0 = api.launch_count()
    api.check(raw([b.h.value for b in got], [ix_mesh(w.ctypes.data, 16, w, i) for w, (_, i) in zip(ws, meshes)], keep=1))
    n_ix = api.launch_count() - n0
    n0 = api.launch_count()
    api.check(raw([b.h.value for b in want], [(s.ctypes.data, 16, 0, None, s.shape[0] // 3) for s in soups], keep=1))
    n_flat = api.launch_count() - n0
    assert n_ix == n_flat + 1, (n_ix, n_flat)
    assert [snapshot(b) for b in got] == [snapshot(b) for b in want]
    first = [snapshot(b) for b in got]
    api.check(raw([b.h.value for b in got], [ix_mesh(w.ctypes.data, 16, w, i) for w, (_, i) in zip(ws, meshes)], keep=1))
    assert [snapshot(b) for b in got] == first, "two identical calls differ"
