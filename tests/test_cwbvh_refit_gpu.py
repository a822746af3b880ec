"""GPU parity of tbvh_refit_layouts (BVH_GPU.Refit / BVH8_CWBVH.Refit): after the vertices moved, the BVH2 is BVH::Refit's, the BVH_GPU
nodes are BVH_GPU::ConvertFrom of the refitted tree, and bvh8Data / bvh8Tris are the oracle's CWBVH over the conversion's collapse with the
refitted boxes (tests/cwbvh_refit_oracle.c), byte for byte; traversal of those bytes is the reference's CPU walk of them, bit for bit."""
import ctypes as C

import numpy as np
import pytest

from oracle import portpy
from tinybvh_b200 import api, _lib, rays as R, scenes
from tests import util
from tests.cwbvh_refit_oracle import RefitCWBVH
from tests.test_convert_gpu import diff_blob, diff_nodes
from tests.test_oracle_pin import moved, tlas_case

pytestmark = pytest.mark.gpu
ZERO = {"prim": 0, "t": 0, "u": 0, "v": 0}
E_ARG, E_STATE = -2, -3    # TBVH_E_ARG, TBVH_E_STATE (include/tinybvh_b200.h)


def engine(v, how):
    """A handle holding BVH, BVH_GPU and CWBVH: BVH8_CWBVH.Build (BuildAVX tree) or BVH.Build then tbvh_convert (BVH::Build tree)."""
    e = api.BVH8_CWBVH()
    if how == "BVH.Build":
        e.build_flavour = _lib.BUILD_REFERENCE
    e.Build(v)
    api.check(_lib.lib().tbvh_convert(e.h, api.LAYOUT_BVH_GPU))
    return e, portpy.PortBVH(v, avx=how != "BVH.Build")


def check_bytes(e, built, w, label):
    """e refitted to w; built: the oracle tree before any refit -> (refitted oracle tree, oracle CWBVH)"""
    o = portpy.PortBVH(built.verts, nodes=built.nodes.copy(), prim_idx=built.prim_idx)
    o.refit(w)
    nodes, idx = api.BVH.download(e)
    assert np.array_equal(nodes.view(np.uint32), o.nodes.view(np.uint32)) and np.array_equal(idx, o.prim_idx), f"{label}: BVH2 differs from BVH::Refit"
    diff_nodes(api.BVH_GPU.download(e), o.to_bvh_gpu(), 16)
    cw = RefitCWBVH(built.nodes, o.nodes, o.prim_idx, w)
    data, tris = e.download()
    diff_blob(data, cw.nodes, label + " bvh8Data", 80)
    diff_blob(tris, cw.tris, label + " bvh8Tris", 48)
    i = e.info()
    assert np.array_equal(np.array(i.aabb_min, np.float32), o.nodes[0]["aabbMin"]) and np.array_equal(np.array(i.aabb_max, np.float32), o.nodes[0]["aabbMax"])
    return o, cw


def occluded_bits(e, rays):
    return np.unpackbits(e.IsOccluded(rays).view(np.uint8), bitorder="little")[: rays.shape[0]].astype(bool)


def check_traversal(e, cw, rays, label):
    """host path and device tensors, closest hit and occlusion, against BVH8_CWBVH::Intersect of the same bytes"""
    import torch
    want, got = rays.copy(), rays.copy()
    cw.intersect(want), e.Intersect(got)
    assert util.compare_hits(got, want) == ZERO, label
    d = torch.from_numpy(rays.view(np.uint8).reshape(-1, 128).copy()).cuda()
    e.Intersect(d)
    torch.cuda.synchronize()
    assert util.compare_hits(d.cpu().numpy().view(R.RAY_DTYPE).reshape(-1), want) == ZERO, label + " (device rays)"
    occ_want = want["t"] < rays["t"]      # BVH8_CWBVH::IsOccluded is FALLBACK_SHADOW_QUERY: Intersect, then t < d (tiny_bvh.h:312)
    assert np.array_equal(occluded_bits(e, rays), occ_want), label + " occlusion"
    bits = e.IsOccluded(torch.from_numpy(rays.view(np.uint8).reshape(-1, 128).copy()).cuda())
    assert np.array_equal(np.unpackbits(bits.cpu().numpy().view(np.uint8), bitorder="little")[: rays.shape[0]].astype(bool), occ_want), label + " occlusion (device rays)"
    return want


@pytest.mark.parametrize("how", ["BVH8_CWBVH.Build", "BVH.Build"])
@pytest.mark.parametrize("scene", ["synthetic:1", "synthetic:5000", "synthetic:70000", "sponza"])
def test_refit_layouts_bytes(gpu, scene, how):
    v, label = scenes.load_scene(scene)
    e, built = engine(v, how)
    data0, tris0 = e.download()
    e.Refit(v)      # no motion: the conversion's own bytes
    data, tris = e.download()
    assert np.array_equal(data.view(np.uint32), data0.view(np.uint32)) and np.array_equal(tris.view(np.uint32), tris0.view(np.uint32))
    for frame in (1, 2):   # the second frame refits from the first frame's boxes, the collapse stays the conversion's
        w = moved(v, 40 + frame, amp=0.05)
        e.Refit(w)
        check_bytes(e, built, w, f"{label} frame {frame}")
        assert e.info().used_blocks == data0.shape[0]
    assert e.info().build_ms > 0


@pytest.mark.parametrize("how", ["BVH8_CWBVH.Build", "BVH.Build"])
def test_refit_layouts_traversal(gpu, how):
    v = scenes.procedural_scene(30000, 43)
    e, built = engine(v, how)
    for frame in (1, 2):
        w = moved(v, 44 + frame, amp=0.05)
        e.Refit(w)
        _, cw = check_bytes(e, built, w, f"frame {frame}")
        sets, bounds = util.ray_sets(w, res=64)
        traced = check_traversal(e, cw, sets["primary"], f"frame {frame} camera")
        assert (traced["t"] < 1e30).sum() > 1000
        for kind, rays in util.derived_sets(traced, w, bounds).items():
            check_traversal(e, cw, rays, f"frame {frame} {kind}")


def test_refit_layouts_recomputes_the_integer_path_bound(gpu):
    """Blown up by 2^40 about its centre the tree's largest exponent passes 27, and rays with rD = 1e30 (an axis-aligned D) no longer fit
    the integer-ordered slab test (cw_walk.cuh cw_ray_fits): a limit left from the normal-scale conversion would let them take it."""
    v = scenes.procedural_scene(20000, 47)
    e, built = engine(v, "BVH8_CWBVH.Build")
    lo, hi = scenes.scene_bounds(v)
    c = (lo + hi) * np.float32(0.5)
    w = v.copy()
    w[:, :3] = c + (v[:, :3] - c) * np.float32(2.0 ** 40)
    e.Refit(w)
    _, cw = check_bytes(e, built, w, "scaled")
    data, _ = e.download()
    assert data.view(np.uint8).reshape(-1, 80)[:, 12:15].view(np.int8).max() > 27    # ex, ey, ez: bytes 12..14 of every node
    wlo, whi = scenes.scene_bounds(w)
    ext = float((whi - wlo).max())
    rng = np.random.default_rng(48)
    O = (c + (rng.random((8192, 3), np.float32) - 0.5) * np.float32(0.6 * ext)).astype(np.float32)
    D = np.zeros((8192, 3), np.float32)
    D[np.arange(8192), np.arange(8192) % 3] = np.where(np.arange(8192) % 2, 1.0, -1.0)
    O[np.arange(8192), np.arange(8192) % 3] = c[np.arange(8192) % 3] - np.float32(ext) * D[np.arange(8192), np.arange(8192) % 3]
    axis = R.make_rays(O, D)
    assert (axis["rD"] == np.float32(1e30)).any(axis=1).all()
    traced = check_traversal(e, cw, axis, "axis-aligned")
    assert (traced["t"] < 1e30).sum() > 10
    sets, _ = util.ray_sets(w, res=48)
    check_traversal(e, cw, sets["primary"], "generic")


def test_refit_layouts_degenerate_motion(gpu):
    v = scenes.procedural_scene(5000, 49)
    e, built = engine(v, "BVH.Build")
    point = v.copy()
    point[:, :3] = v[0, :3]
    plane = v.copy()
    plane[:, 2] = np.float32(0.25)
    for label, w in (("point", point), ("plane", plane)):
        e.Refit(w)
        _, cw = check_bytes(e, built, w, label)
        sets, _ = util.ray_sets(v, res=48)
        check_traversal(e, cw, sets["primary"], label)


def _rc(e, verts, prim_count=None):
    v = np.ascontiguousarray(verts, np.float32)
    return _lib.lib().tbvh_refit_layouts(e.h, v.ctypes.data_as(C.c_void_p), 16, prim_count or v.shape[0] // 3, api.HOST)


def _snapshot(e):
    i = e.info()
    out = [bytes(i)]
    if i.layouts & (1 << api.LAYOUT_BVH):
        out += [x.tobytes() for x in api.BVH.download(e)]
    if i.layouts & (1 << api.LAYOUT_CWBVH):
        out += [x.tobytes() for x in api.BVH8_CWBVH.download(e)]
    return out


def test_refit_layouts_refusals_leave_the_handle_unchanged(gpu):
    v = scenes.procedural_scene(3000, 51)
    w = moved(v, 52)
    sbvh = api.BVH8_CWBVH().BuildHQ(v)
    uploaded = api.BVH8_CWBVH().Build(v)
    tree = portpy.PortBVH(v, avx=True)
    c = portpy.PortCWBVH(tree.nodes, tree.prim_idx, v)
    uploaded.upload(c.nodes, c.tris)      # bvh8Data from elsewhere over the built tree: not this handle's conversion
    x, inst, _, _ = tlas_case(53, 8)
    tlas = api.TLAS().Build(inst, [api.BVH().Build(y) for y in x])
    good = api.BVH8_CWBVH().Build(v)
    for e, verts, count, want in ((sbvh, w, None, E_STATE), (tlas, np.zeros((24, 4), np.float32), None, E_STATE),
                                  (uploaded, w, None, E_STATE), (good, w, v.shape[0] // 3 - 1, E_ARG)):
        before = _snapshot(e)
        assert _rc(e, verts, count) == want
        assert _snapshot(e) == before
    assert _rc(good, w) == _lib.OK


def test_refit_layouts_two_level(gpu):
    """A TLAS over a refitted BLAS is stale (its instance boxes are); after BLASInstance::Update and a TLAS rebuild the CWBVH walk of the
    two levels is the oracle's over the downloaded bytes."""
    from tests.test_tlas_gpu import _CW, words
    v, inst, O, D = tlas_case(55, 30)
    blas = [api.BVH8_CWBVH().Build(x) for x in v]
    t = api.TLAS().Build(inst, blas, blas_layout=api.LAYOUT_CWBVH)
    blas[0].Refit(moved(v[0], 56, amp=0.05))
    with pytest.raises(api.TbvhError, match="error -3"):
        t.Intersect(R.make_rays(O, D))
    t = api.TLAS().Build(inst, blas, blas_layout=api.LAYOUT_CWBVH)    # Update()s every instance against the new root boxes
    nodes, idx = t.download()
    port = portpy.PortTLASCW(nodes, idx, inst, [_CW(b) for b in blas])
    rays = R.make_rays(O, D)
    want, got = rays.copy(), rays.copy()
    port.intersect(want), t.Intersect(got)
    assert np.array_equal(words(got), words(want)) and (want["t"] < 1e30).sum() > 1000


def test_refit_layouts_group(gpu):
    from tests.test_group_gpu import devices
    v = scenes.procedural_scene(25000, 57)
    e = api.BVH8_CWBVH().Build(v)
    g = api.Group(devices())
    g.replicate(e)
    w = moved(v, 58, amp=0.05)
    e.Refit(w)
    g.replicate(e)
    lo, hi = scenes.scene_bounds(w)
    src = R.primary_rays(*R.bounds_camera(lo, hi, "inside"), 96, 96, 4)
    rays = g.empty_rays(src.shape[0], R.RAY_DTYPE)
    rays[:] = src
    want = src.copy()
    e.Intersect(want)
    g.Intersect(rays)
    assert util.compare_hits(rays, want) == ZERO and (want["t"] < 1e30).sum() > 1000
    g.close()
