"""tbvh_mesh_toi / tbvh_mesh_toi_pairs on the device, held bit for bit to the host restatement (tests/toi_oracle.c, DESIGN.md §4.15):
every record, pair, time and count over every builder's tree (failed-split SBVHs and PLOC included), batch and indexed builds, uploaded
families and a DAG, a BVH_GPU upload, trees 99 and 254 levels deep, one-leaf trees, refitted and optimised trees and a group replica;
end frames at strides 12, 16 and 32 from host and device; host and device space, stream order on a caller's stream, every refusal with
the outputs untouched, handles unchanged by the calls, and a three-frame loop with a refit between two steps."""
import ctypes as C

import numpy as np
import pytest

from tinybvh_b200 import _lib, api, scenes
from tests import toi_oracle as toi
from tests.test_closest_point import family
from tests.test_closest_point_gpu import chain_tree, torch_f
from tests.test_mesh_overlap_gpu import h_of
from tests.test_signed_distance import icosphere, soup, torus
from tests.test_winding_number import two_spheres

pytestmark = pytest.mark.gpu
L = lambda: _lib.lib()  # noqa: E731
ETA, XI, ITERS = 0.01, 0.004, 64


def jitter(v, seed, s=0.02):
    rng = np.random.default_rng(seed)
    out = v.copy()
    out[:, :3] += (rng.normal(size=(v.shape[0], 3)) * s).astype(np.float32)
    return out


def rows(v, stride):
    """the (n, 4) vertices as rows `stride` bytes apart (12: xyz only; 32: xyzw and four floats of padding)"""
    if stride == 12:
        return np.ascontiguousarray(v[:, :3])
    if stride == 16:
        return np.ascontiguousarray(v)
    return np.ascontiguousarray(np.concatenate([v, np.full((v.shape[0], 4), np.nan, np.float32)], 1))


def end_arg(v, stride, device):
    r = rows(v, stride)
    if not device:
        return r, C.c_void_p(r.ctypes.data)
    import torch
    t = torch.from_numpy(r).cuda()
    return t, C.c_void_p(t.data_ptr())


def nearest_call(a, a1, b, b1, n, eta=ETA, xi=XI, iters=ITERS, stride=16, device=True, stream=None):
    import torch
    ka, pa = end_arg(a1, stride, device)
    kb, pb = (ka, pa) if b1 is None else end_arg(b1, stride, device)
    if device:
        rec = torch.full((max(n, 1), 4), -1, dtype=torch.int32, device="cuda")
        _lib.check(L().tbvh_mesh_toi(h_of(a), pa, stride, h_of(b), pb, stride, C.c_float(eta), C.c_float(xi), iters, C.c_void_p(rec.data_ptr()), _lib.DEVICE, stream))
        torch.cuda.synchronize()
        r = rec.cpu().numpy()[:n]
    else:
        r = np.full((max(n, 1), 4), -1, np.int32)
        _lib.check(L().tbvh_mesh_toi(h_of(a), pa, stride, h_of(b), pb, stride, C.c_float(eta), C.c_float(xi), iters, C.c_void_p(r.ctypes.data), _lib.HOST, None))
        r = r[:n]
    return r[:, 0].view(np.float32), r[:, 1].view(np.float32), r[:, 2].view(np.uint32), r[:, 3].view(np.uint32)


def pairs_call(a, a1, b, b1, cap, eta=ETA, xi=XI, iters=ITERS, stride=16, device=True, times=True):
    import torch
    ka, pa = end_arg(a1, stride, device)
    kb, pb = (ka, pa) if b1 is None else end_arg(b1, stride, device)
    count = C.c_uint64(12345)
    if device:
        out = torch.full((max(cap, 1), 2), -1, dtype=torch.int32, device="cuda")
        tm = torch.full((max(cap, 1),), -1, dtype=torch.int32, device="cuda")
        rc = L().tbvh_mesh_toi_pairs(h_of(a), pa, stride, h_of(b), pb, stride, C.c_float(eta), C.c_float(xi), iters, C.c_void_p(out.data_ptr()),
                                     C.c_void_p(tm.data_ptr()) if times else None, cap, C.byref(count), _lib.DEVICE, None)
        torch.cuda.synchronize()
        return out.cpu().numpy().view(np.uint32), tm.cpu().numpy().view(np.float32), count.value, rc
    out = np.full((max(cap, 1), 2), 0xFFFFFFFF, np.uint32)
    tm = np.full(max(cap, 1), -1, np.int32).view(np.float32)
    rc = L().tbvh_mesh_toi_pairs(h_of(a), pa, stride, h_of(b), pb, stride, C.c_float(eta), C.c_float(xi), iters, C.c_void_p(out.ctypes.data),
                                 C.c_void_p(tm.ctypes.data) if times else None, cap, C.byref(count), _lib.HOST, None)
    return out, tm, count.value, rc


def same_records(got, want, label):
    for g, w, name in zip(got, want, ("t", "d", "j", "iters")):
        assert np.array_equal(np.asarray(g).view(np.uint32), np.asarray(w).view(np.uint32)), f"{label}: {name} differs"


def check(a, a0, a1, b, nodes, idx, b0, b1, label, host=False, stride=16, eta=ETA, xi=XI):
    """a moving from a0 to a1 against b moving from b0 to b1 (b is a: the self query, b1 None): records, pairs and times equal the
    restatement's"""
    self = h_of(a).value == h_of(b).value
    n = a0.shape[0] // 3
    bb1 = a1 if self else b1
    want = toi.nearest(nodes, idx, b0, bb1, None if self else a0, None if self else a1, eta, xi, ITERS)
    same_records(nearest_call(a, a1, b, None if self else b1, n, eta, xi, stride=stride), want, f"{label} nearest")
    wp, wt = toi.pairs(nodes, idx, b0, bb1, None if self else a0, None if self else a1, eta, xi, ITERS)
    got, gt, count, rc = pairs_call(a, a1, b, None if self else b1, max(wp.shape[0], 1), eta, xi, stride=stride)
    _lib.check(rc)
    assert count == wp.shape[0] and np.array_equal(got[:count], wp), f"{label}: pairs ({count}, restatement {wp.shape[0]})"
    assert np.array_equal(gt[:count].view(np.uint32), wt.view(np.uint32)), f"{label}: times"
    if host:
        same_records(nearest_call(a, a1, b, None if self else b1, n, eta, xi, stride=stride, device=False), want, f"{label} host nearest")
        hp, ht, hc, rc = pairs_call(a, a1, b, None if self else b1, max(wp.shape[0], 1), eta, xi, stride=stride, device=False)
        _lib.check(rc)
        assert hc == count and np.array_equal(hp[:hc], wp) and np.array_equal(ht[:hc].view(np.uint32), wt.view(np.uint32)), f"{label}: host pairs"
    return want, wp


@pytest.mark.parametrize("builder", ["Build", "BuildAVX", "BuildHQ", "BuildPLOC"])
@pytest.mark.parametrize("ntris", [1, 7, 3000])
def test_builders(gpu, builder, ntris):
    va = scenes.procedural_scene(ntris, 3 + ntris)
    vb = scenes.procedural_scene(max(ntris, 2), 4 + ntris)
    vb[:, :3] += np.float32(0.02)
    a, b = getattr(api.BVH(), builder)(va), getattr(api.BVH(), builder)(vb)
    a1, b1 = jitter(va, 1), jitter(vb, 2)
    w, p = check(a, va, a1, b, *b.download(), vb, b1, f"{builder}-{ntris}", host=ntris == 3000)
    check(a, va, a1, a, *a.download(), va, None, f"self {builder}-{ntris}", host=ntris == 3000)
    if ntris == 3000:
        assert p.shape[0] > 10 and (w[2] != toi.NO_PRIM).sum() > 10


@pytest.mark.parametrize("name", ["snapped20k_q4", "lattice10k_k3"])
def test_hq_failed_splits(gpu, name):
    from tests.test_build_hq_shapes import fail_scene
    v = fail_scene(name)
    e = api.BVH().BuildHQ(v)
    check(e, v, jitter(v, 7, 0.05), e, *e.download(), v, None, f"BuildHQ-{name}")


def test_batch_and_indexed(gpu):
    meshes = [soup(*two_spheres()), soup(*torus()), scenes.procedural_scene(700, 21)]
    for flavour in (_lib.BUILD_REFERENCE, _lib.BUILD_AVX, _lib.BUILD_PLOC, _lib.BUILD_HQ):
        objs = [api.BVH() for _ in meshes]
        api.build_batch(objs, meshes, flavour)
        for k, (o, v) in enumerate(zip(objs, meshes)):
            check(o, v, jitter(v, k), o, *o.download(), v, None, f"batch-{flavour}-{k}")
        check(objs[0], meshes[0], jitter(meshes[0], 9), objs[2], *objs[2].download(), meshes[2], jitter(meshes[2], 10), f"batch-{flavour} a/b")
    V, F = torus()
    verts = np.zeros((V.shape[0], 4), np.float32)
    verts[:, :3] = V
    e = api.BVH()
    e.Build(verts, indices=F.astype(np.uint32).reshape(-1))
    v = soup(V, F)
    check(e, v, jitter(v, 11, 0.05), e, *e.download(), v, None, "indexed")


@pytest.mark.parametrize("fam", ["A0.3", "B", "C3", "DA", "shrunk", "dag"])
def test_uploaded_families(gpu, fam):
    from tests import util
    v = scenes.procedural_scene(3000, 71)
    va = scenes.procedural_scene(1500, 72)
    src = util.source_tree(v, "BuildHQ" if fam in ("C0", "C3", "DB") else "Build")
    nodes, idx = family(src, fam)
    e = api.BVH().upload(nodes, idx, v)
    a = api.BVH().Build(va)
    check(a, va, jitter(va, 12), e, nodes, idx, v, jitter(v, 13), f"family {fam}")
    check(e, v, jitter(v, 13), e, nodes, idx, v, None, f"family self {fam}")


def test_bvh_gpu_upload_deep_and_one_leaf_trees(gpu):
    from tests import util
    v = soup(*two_spheres())
    o = util.oracle_tree(v, 1)
    g = api.BVH_GPU().upload(util.oracle_bvh_gpu_nodes(o), o.prim_idx, v)
    check(g, v, jitter(v, 14), g, o.nodes, o.prim_idx, v, None, "BVH_GPU upload", host=True)
    w = scenes.procedural_scene(400, 12)
    for m in (100, 255):
        nodes, idx = chain_tree(w, m)
        c = api.BVH().upload(nodes, idx, w[: 3 * m])
        assert c.info().max_depth == m - 1
        check(c, w[: 3 * m], jitter(w[: 3 * m], 15), c, nodes, idx, w[: 3 * m], None, f"chain-{m}")
        a = api.BVH().Build(w)
        check(a, w, jitter(w, 16), c, nodes, idx, w[: 3 * m], jitter(w[: 3 * m], 15), f"chain-{m} a/b")
    one = scenes.procedural_scene(1, 5)
    e = api.BVH().Build(one)
    assert e.info().max_depth == 0
    check(a, w, jitter(w, 16), e, *e.download(), one, jitter(one, 17, 0.3), "one-leaf B", host=True)
    check(e, one, jitter(one, 17, 0.3), a, *a.download(), w, jitter(w, 16), "one-triangle A", host=True)


@pytest.mark.parametrize("stride", [12, 16, 32])
def test_strides_host_and_device(gpu, stride):
    v = soup(*two_spheres())
    w = scenes.procedural_scene(2000, 9)
    a, b = api.BVH().Build(v), api.BVH().Build(w)
    check(a, v, jitter(v, 18), b, *b.download(), w, jitter(w, 19), f"stride {stride}", host=True, stride=stride)
    check(a, v, jitter(v, 18), a, *a.download(), v, None, f"self stride {stride}", host=True, stride=stride)


def test_refit_optimize_replica_and_three_frames(gpu):
    v = soup(*two_spheres())
    v1, v2 = jitter(v, 20), jitter(v, 21)
    e = api.BVH().Build(v)
    check(e, v, v1, e, *e.download(), v, None, "frame 0 -> 1")
    e.Refit(v1)
    check(e, v1, v2, e, *e.download(), v1, None, "frame 1 -> 2 after the refit")
    o = api.BVH().Build(soup(*torus()))
    rounds = C.c_uint32()
    _lib.check(L().tbvh_optimize(o.h, 4, C.c_float(1.0), C.c_float(1.0), C.byref(rounds), None))
    t = soup(*torus())
    check(o, t, jitter(t, 22), o, *o.download(), t, None, "optimize")
    s = api.BVH().Build(v)
    want, wp = check(s, v, v1, s, *s.download(), v, None, "source")
    grp = api.Group([0])
    grp.replicate(s)
    rep = C.c_void_p(L().tbvh_group_replica(grp.h, 0))
    same_records(nearest_call(rep, v1, rep, None, v.shape[0] // 3), want, "group replica")
    got, gt, count, rc = pairs_call(rep, v1, rep, None, wp.shape[0] + 4)
    _lib.check(rc)
    assert count == wp.shape[0] and np.array_equal(got[:count], wp), "group replica pairs"
    grp.close()


def test_handles_unchanged_python_api_and_stream_order(gpu):
    import torch
    v = soup(*two_spheres())
    w = scenes.procedural_scene(2000, 9)
    a, b = api.BVH().Build(v), api.BVH().Build(w)
    v1, w1 = jitter(v, 23), jitter(w, 24)
    info = [bytes(a.info()), bytes(b.info())]
    trees = [x.download() for x in (a, b)]
    view = [bytes(a.device_view()), bytes(b.device_view())]
    want = toi.nearest(*b.download(), w, w1, v, v1, ETA, XI, ITERS)
    wp, wt = toi.pairs(*b.download(), w, w1, v, v1, ETA, XI, ITERS)
    assert wp.shape[0] > 10
    # the Python API: numpy and tensors
    same_records(a.time_of_impact(v1, b, w1, eta=ETA, xi=XI, max_iters=ITERS), want, "python numpy")
    p, tm = a.impact_pairs(v1[:, :3], b, w1, eta=ETA, xi=XI, max_iters=ITERS)
    assert np.array_equal(p, wp) and np.array_equal(tm.view(np.uint32), wt.view(np.uint32))
    s = torch.cuda.Stream()
    r = a.time_of_impact(torch_f(v1), b, torch_f(w1), eta=ETA, xi=XI, max_iters=ITERS, stream=s)
    s.synchronize()
    same_records(tuple(x.cpu().numpy() for x in r), want, "python tensors")
    p, tm = a.impact_pairs(v1, b, w1, eta=ETA, xi=XI, max_iters=ITERS, stream=s)
    assert np.array_equal(p.cpu().numpy().view(np.uint32), wp) and np.array_equal(tm.cpu().numpy().view(np.uint32), wt.view(np.uint32))
    with pytest.raises(_lib.TbvhError):
        a.time_of_impact(v1, b, w1)
    # stream order: the end frame written behind a long kernel on the caller's stream is what the calls read
    dv = torch_f(w1)
    stage = torch.zeros_like(dv)
    av = torch_f(v1)
    n = v.shape[0] // 3
    rec = torch.full((n, 4), -1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)
        stage.copy_(dv)
        _lib.check(L().tbvh_mesh_toi(a.h, C.c_void_p(av.data_ptr()), 16, b.h, C.c_void_p(stage.data_ptr()), 16, C.c_float(ETA), C.c_float(XI), ITERS,
                                     C.c_void_p(rec.data_ptr()), _lib.DEVICE, C.c_void_p(s.cuda_stream)))
    s.synchronize()
    r2 = rec.cpu().numpy()
    same_records((r2[:, 0].view(np.float32), r2[:, 1].view(np.float32), r2[:, 2].view(np.uint32), r2[:, 3].view(np.uint32)), want, "nearest on the caller's stream")
    stage.zero_()
    out = torch.full((wp.shape[0] + 1, 2), -1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)
        stage.copy_(dv)
    cnt = C.c_uint64()
    _lib.check(L().tbvh_mesh_toi_pairs(a.h, C.c_void_p(av.data_ptr()), 16, b.h, C.c_void_p(stage.data_ptr()), 16, C.c_float(ETA), C.c_float(XI), ITERS,
                                       C.c_void_p(out.data_ptr()), None, out.shape[0], C.byref(cnt), _lib.DEVICE, C.c_void_p(s.cuda_stream)))
    s.synchronize()
    assert cnt.value == wp.shape[0] and np.array_equal(out.cpu().numpy().view(np.uint32)[: cnt.value], wp), "pairs ordered after the caller's stream"
    # the handles: same info, trees and device views (no generation change)
    assert [bytes(a.info()), bytes(b.info())] == info and [bytes(a.device_view()), bytes(b.device_view())] == view
    for x, (nodes, idx) in zip((a, b), trees):
        n2, i2 = x.download()
        assert nodes.tobytes() == n2.tobytes() and np.array_equal(idx, i2)


def test_refusals_leave_outputs_untouched(gpu):
    import torch
    v = soup(*icosphere(2))
    e = api.BVH().Build(v)
    n = v.shape[0] // 3
    ev = np.ascontiguousarray(v)
    ep = C.c_void_p(ev.ctypes.data)
    out = torch.full((64, 2), -1, dtype=torch.int32, device="cuda")
    tm = torch.full((64,), -1, dtype=torch.int32, device="cuda")
    rec = torch.full((n + 2, 4), -1, dtype=torch.int32, device="cuda")
    op, tp, rp = C.c_void_p(out.data_ptr()), C.c_void_p(tm.data_ptr()), C.c_void_p(rec.data_ptr())
    cnt = C.c_uint64(777)
    dv = torch_f(v)
    dp = C.c_void_p(dv.data_ptr())

    def P(a, b, o=op, t=tp, eta=ETA, xi=XI, it=ITERS, ae=dp, be=dp, sa=16, sb=16, cap=64, c=C.byref(cnt), space=_lib.DEVICE):
        return L().tbvh_mesh_toi_pairs(a, ae, sa, b, be, sb, C.c_float(eta), C.c_float(xi), it, o, t, cap, c, space, None)

    def N(a, b, o=rp, eta=ETA, xi=XI, it=ITERS, ae=dp, be=dp, sa=16, sb=16, space=_lib.DEVICE):
        return L().tbvh_mesh_toi(a, ae, sa, b, be, sb, C.c_float(eta), C.c_float(xi), it, o, space, None)

    for F in (P, N):
        for bad in (dict(eta=np.nan), dict(eta=-1.0), dict(eta=np.inf), dict(xi=0.0), dict(xi=-1.0), dict(xi=np.nan), dict(xi=np.inf),
                    dict(it=0), dict(it=(1 << 16) + 1), dict(ae=None), dict(be=None), dict(sa=8), dict(sb=18), dict(sa=20, sb=20, be=C.c_void_p(dv.data_ptr() + 16))):
            assert F(e.h, e.h, **bad) == _lib.E_ARG, (F.__name__, bad)
        assert F(None, e.h) == _lib.E_ARG and F(e.h, e.h, o=None) == _lib.E_ARG and F(e.h, e.h, space=7) == _lib.E_ARG
    assert N(e.h, e.h, o=C.c_void_p(rec.data_ptr() + 8)) == _lib.E_ARG and P(e.h, e.h, o=C.c_void_p(out.data_ptr() + 4)) == _lib.E_ARG
    assert P(e.h, e.h, t=C.c_void_p(tm.data_ptr() + 2)) == _lib.E_ARG and P(e.h, e.h, c=None) == _lib.E_ARG
    inst = np.zeros(2, api.BLAS_INSTANCE)
    inst["transform"] = np.eye(4, dtype=np.float32).reshape(-1)
    inst["mask"] = 0xFFFF
    t = api.TLAS()
    t.Build(inst, [e])
    assert P(t.h, e.h) == _lib.E_UNSUPPORTED and N(e.h, t.h) == _lib.E_UNSUPPORTED
    assert P(t.h, e.h, xi=0.0) == _lib.E_ARG, "the argument refusals come first"
    assert P(api.BVH().h, e.h) == _lib.E_STATE and N(e.h, api.BVH().h) == _lib.E_STATE
    w = scenes.procedural_scene(300, 19)
    deep = chain_tree(w, 300)
    d = api.BVH().upload(deep[0], deep[1], w)
    assert P(e.h, d.h) == _lib.E_LIMIT and N(d.h, d.h) == _lib.E_LIMIT
    k0 = api.launch_count()
    assert (P(t.h, e.h), N(e.h, d.h), N(e.h, e.h, it=0)) == (_lib.E_UNSUPPORTED, _lib.E_LIMIT, _lib.E_ARG)
    assert api.launch_count() == k0, "a refusal launched work"
    torch.cuda.synchronize()
    assert (out == -1).all() and (tm == -1).all() and (rec == -1).all() and cnt.value == 777, "a refused call wrote its outputs"
    # after the refusals the same handle answers: a static step in host space
    r = np.zeros((n, 4), np.float32)
    _lib.check(N(e.h, e.h, o=C.c_void_p(r.ctypes.data), ae=ep, be=ep, space=_lib.HOST))
    assert np.isinf(r[:, 0]).all(), "a closed icosphere standing still: only neighbours within eta + xi, and they are skipped"


def test_capacity_below_the_count_with_times(gpu):
    """capacity < count: the exact count, the first `capacity` pairs and their times, nothing written past them, host and device"""
    v = soup(*two_spheres())
    w = scenes.procedural_scene(2000, 9)
    a, b = api.BVH().Build(v), api.BVH().Build(w)
    v1, w1 = jitter(v, 25), jitter(w, 26)
    wp, wt = toi.pairs(*b.download(), w, w1, v, v1, ETA, XI, ITERS)
    m = wp.shape[0]
    assert m > 10
    for device in (True, False):
        for cap in (1, m // 2, m - 1, m + 7):
            got, gt, count, rc = pairs_call(a, v1, b, w1, cap, device=device)
            _lib.check(rc)
            k = min(cap, m)
            assert count == m and np.array_equal(got[:k], wp[:k]), (device, cap)
            assert np.array_equal(gt[:k].view(np.uint32), wt[:k].view(np.uint32)), f"times at capacity {cap}"
            assert (got[k:] == 0xFFFFFFFF).all() and (gt[k:].view(np.int32) == -1).all(), f"written past capacity {cap}"
        got, gt, count, rc = pairs_call(a, v1, b, w1, 0, device=device)
        _lib.check(rc)
        assert count == m and (got == 0xFFFFFFFF).all() and (gt.view(np.int32) == -1).all(), "capacity 0 writes nothing"
