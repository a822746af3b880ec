"""GPU parity of tbvh_build_tlas_update / api.TLAS.Rebuild: BLASInstance::Update on the device and the TLAS build in one call.  The
records, the TLAS tree, its info and its walks are those of the existing path (tbvh_instance_update per record, then tbvh_build_tlas) and
of the oracle, for host and device records of every stride, on the inputs Update is sensitive to, across the frames of an animation on
one handle; refusals leave the handle and the records as the header says."""
import ctypes as C

import numpy as np
import pytest

from oracle import portpy
from tinybvh_b200 import _lib, api, rays as R, scenes
from tests import util
from tests.test_convert_batch_gpu import convert, info
from tests.test_oracle_pin import moved, tlas_case
from tests.test_tlas_gpu import words
from tests.test_tlas_update import records, update_families

pytestmark = pytest.mark.gpu


def make_blas(builder, v):
    if builder == "CWBVH":
        return [api.BVH8_CWBVH().Build(x) for x in v]
    return [getattr(api.BVH(), builder)(x) for x in v]


def snapshot(t):
    """nodes, primIdx and every info field but build_ms"""
    nodes, idx = t.download()
    return nodes.tobytes(), idx.tobytes(), info(t)


def walks(t, O, D, layouts):
    out = []
    for layout in layouts:
        t.layout = layout
        for mask in (0x1, 0x2):
            r = R.make_rays(O, D)
            r["mask"] = mask
            t.Intersect(r)
            sh = R.make_rays(O, D, tmax=150.0)
            sh["mask"] = mask
            out += [words(r).tobytes(), t.IsOccluded(sh).tobytes()]
    return out


def raw(t, p, stride, n, space, handles, count=None):
    hs = (C.c_void_p * max(len(handles), 1))(*handles)
    return _lib.lib().tbvh_build_tlas_update(t.h if t is not None else None, p, stride, n, space, hs, len(handles) if count is None else count, 1.0, 1.0)


@pytest.mark.parametrize("n_inst", [1, 40, 300, 3000])
@pytest.mark.parametrize("builder", ["Build", "BuildAVX", "BuildHQ", "CWBVH"])
def test_equals_update_loop_and_build(gpu, builder, n_inst):
    v, inst, O, D = tlas_case(91, n_inst)
    inst["dummy"] = 0xFEED0000 + np.arange(n_inst, dtype=np.uint32)[:, None]
    blas = make_blas(builder, v)
    layouts = (api.LAYOUT_BVH, api.LAYOUT_CWBVH) if builder == "CWBVH" else (api.LAYOUT_BVH,)
    a, b = inst.copy(), inst.copy()
    old = api.TLAS().Build(a, blas)                     # tbvh_instance_update per record, then tbvh_build_tlas
    new = api.TLAS().Rebuild(b, blas)
    assert b.tobytes() == a.tobytes(), "records differ from BLASInstance::Update on the host"
    assert snapshot(new) == snapshot(old), "TLAS differs from tbvh_build_tlas"
    assert walks(new, O, D, layouts) == walks(old, O, D, layouts)


@pytest.mark.parametrize("n_inst,builder", [(40, "Build"), (1, "Build"), (300, "BuildAVX"), (3000, "Build"), (40, "BuildHQ")])
def test_equals_the_oracle(gpu, n_inst, builder):
    v, inst, O, D = tlas_case(91, n_inst)
    inst_ref = inst.copy()
    ref = util.oracle_tlas(inst_ref, v, {"Build": 0, "BuildAVX": 1, "BuildHQ": 2}[builder])
    t = api.TLAS().Rebuild(inst, make_blas(builder, v))
    assert inst.tobytes() == inst_ref.tobytes(), "BLASInstance::Update differs"
    nodes, idx = t.download()
    rb = ref.bvh()
    assert np.array_equal(nodes.view(np.uint32), rb.nodes.view(np.uint32)) and np.array_equal(idx, rb.prim_idx), "TLAS tree differs"
    for mask in (0x1, 0x2):
        rays = R.make_rays(O, D)
        rays["mask"] = mask
        want, got = rays.copy(), rays.copy()
        ref.intersect(want), t.Intersect(got)
        assert np.array_equal(words(got), words(want)), f"closest hits differ (ray mask {mask:#x})"
        sh = R.make_rays(O, D, tmax=150.0)
        sh["mask"] = mask
        assert np.array_equal(t.IsOccluded(sh), ref.occluded(sh))


def test_host_and_device_records_of_every_stride_agree(gpu):
    import torch
    n = 300
    v, inst, O, D = tlas_case(93, n)
    blas = make_blas("Build", v)
    want = inst.copy()
    want_tlas = snapshot(api.TLAS().Build(want, blas))
    want = want.view(np.uint8).reshape(n, 192)
    src = inst.view(np.uint8).reshape(n, 192)
    for stride in (192, 256, 160, 196):
        w = min(stride, 192)
        buf = np.full((n, stride), 0xA5, np.uint8)
        buf[:, :w] = src[:, :w]
        t = api.TLAS().Rebuild(buf[:, :w], blas)
        assert np.array_equal(buf[:, :w], want[:, :w]), f"host records, stride {stride}"
        assert (buf[:, w:] == 0xA5).all(), f"host stride {stride}: bytes between records changed"
        assert snapshot(t) == want_tlas, f"host stride {stride}"
    for stride in (192, 256):
        flat = torch.full((n * stride + 32,), 0xA5, dtype=torch.uint8, device="cuda")
        d = flat[16:16 + n * stride].view(n, stride)     # 16-byte aligned, not 64
        assert d.data_ptr() % 64 == 16
        d[:, :192] = torch.from_numpy(src).cuda()
        t = api.TLAS().Rebuild(d[:, :192], blas)
        got = flat.cpu().numpy()
        body = got[16:16 + n * stride].reshape(n, stride)
        assert np.array_equal(body[:, :192], want), f"device records, stride {stride}"
        assert (body[:, 192:] == 0xA5).all() and (got[:16] == 0xA5).all() and (got[16 + n * stride:] == 0xA5).all(), f"device stride {stride}: other bytes changed"
        assert snapshot(t) == want_tlas, f"device stride {stride}"


def canonical(rec):
    """record bytes with every NaN word made one pattern: an overflowing determinant (the 2^60 family: inf * 0 in invTransform) gives a NaN
    on both sides, whose sign and payload are the processor's (x86 generates 0xffc00000, the GPU 0x7fffffff)"""
    w = np.ascontiguousarray(rec).view(np.uint32).reshape(-1, 48).copy()
    w[np.isnan(w.view(np.float32))] = 0x7FC00000
    return w.tobytes()


def zero_box_blasses():
    """BLASes whose root boxes hold -0 and +0 bounds (the sign is that of the last zero folded)"""
    a, b = util.zero_tri_cases()
    v = [a, b, util.signed_zero(scenes.procedural_scene(500, 3), "neg"), util.signed_zero(scenes.procedural_scene(400, 4), "order")]
    blas = [api.BVH().Build(x) for x in v]
    boxes = np.array([list(x.info().aabb_min) + list(x.info().aabb_max) for x in blas], np.float32)
    assert util.count_neg_zero(boxes) > 0 and ((boxes == 0) & ~np.signbit(boxes)).any()
    return blas


@pytest.mark.parametrize("family", sorted(update_families()))
def test_inputs_update_is_sensitive_to(gpu, family):
    """Against the host routine bit for bit, host and device records; the TLAS over the boxes against tbvh_build_tlas's."""
    import torch
    T = update_families()[family]
    blas = zero_box_blasses()
    inst = records(np.tile(T, (len(blas), 1)), np.repeat(np.arange(len(blas), dtype=np.uint32), T.shape[0]))
    want = inst.copy()
    for i in range(want.shape[0]):
        api.check(_lib.lib().tbvh_instance_update(C.c_void_p(want[i:i + 1].ctypes.data), blas[int(want["blasIdx"][i])].h))
    if family == "singular":
        assert np.isfinite(want["invTransform"]).all()
    old = api.TLAS().Build(want.copy(), blas, update=False)
    host = inst.copy()
    t = api.TLAS().Rebuild(host, blas)
    assert canonical(host) == canonical(want), "host records"
    assert np.isnan(want["invTransform"]).any() == (family == "scale_2^60")
    assert snapshot(t) == snapshot(old)
    d = torch.from_numpy(inst.view(np.uint8).reshape(-1, 192)).cuda()
    t = api.TLAS().Rebuild(d, blas)
    assert canonical(d.cpu().numpy()) == canonical(want), "device records"
    assert snapshot(t) == snapshot(old)


@pytest.mark.parametrize("wide", [False, True])
def test_frames_on_one_handle(gpu, wide):
    """refit_batch, new transforms, Rebuild on the same TLAS object, twice: stale before the call, the oracle's walk after it.  The
    handle's device tables are not observable through the C-ABI, so their reuse is checked through results only."""
    n = 200
    v, inst, O, D = tlas_case(97, n)
    blas = [api.BVH().Build(x) for x in v]
    layout = api.LAYOUT_CWBVH if wide else api.LAYOUT_BVH
    if wide:
        for b in blas:
            convert(b)
    t = api.TLAS().Build(inst, blas, blas_layout=layout)
    rays = R.make_rays(O, D)
    for f in (1, 2):
        w = [moved(x, 70 + f, amp=0.05) for x in v]
        api.refit_batch(blas, w, keep_layouts=1)
        r = rays.copy()
        assert _lib.lib().tbvh_intersect(t.h, layout, r.ctypes.data, 128, 64) == _lib.E_STATE, "a TLAS over refitted BLASes is stale"
        inst["transform"] = util.random_transforms(n, 500 + f)
        t.Rebuild(inst)
        fresh = inst.copy()
        assert snapshot(t) == snapshot(api.TLAS().Build(fresh, blas, blas_layout=layout)) and fresh.tobytes() == inst.tobytes()
        nodes, idx = t.download()
        if wide:
            class _CW:
                def __init__(self, b):
                    i = b.info()
                    self.nodes, self.tris = np.zeros((i.used_blocks, 4), np.float32), np.zeros((i.cwbvh_tri_count * 3, 4), np.float32)
                    api.check(_lib.lib().tbvh_download_cwbvh(b.h, self.nodes.ctypes.data, self.tris.ctypes.data, api.HOST))
            port = portpy.PortTLASCW(nodes, idx, inst, [_CW(b) for b in blas])
        else:
            port = portpy.PortTLAS(nodes, idx, inst, [portpy.PortBVH(x, nodes=api.BVH.download(b)[0], prim_idx=api.BVH.download(b)[1]) for x, b in zip(w, blas)])
        want, got = rays.copy(), rays.copy()
        port.intersect(want), t.Intersect(got)
        assert np.array_equal(words(got), words(want)) and (want["t"] < 1e30).sum() > 1000, f"frame {f}"
    # another instance count on the same handle: the tables are replaced, not reused
    small = inst[:50].copy()
    t.Rebuild(small)
    assert snapshot(t) == snapshot(api.TLAS().Build(inst[:50].copy(), blas, blas_layout=layout))


def test_refusals_leave_the_tlas_and_the_records(gpu):
    import torch
    from tests.test_deep_bvh2_gpu import instances, spine
    L = _lib.lib()
    n = 60
    v, inst, O, D = tlas_case(99, n)
    blas = make_blas("Build", v)
    t = api.TLAS().Build(inst, blas)
    before, walked = snapshot(t), walks(t, O, D, (api.LAYOUT_BVH,))
    other = api.TLAS().Build(inst.copy(), blas)
    fresh = inst.copy()
    fresh["transform"] = util.random_transforms(n, 7)
    rec = fresh.copy()
    p, hs = rec.ctypes.data, [b.h for b in blas]
    past = fresh.copy()
    past["blasIdx"][17] = 2
    nodes, idx, verts = spine(64, 64)
    deep = api.BVH().upload(nodes, idx, verts)
    empty = api.BVH()
    three = instances()
    dev = torch.from_numpy(fresh.view(np.uint8).reshape(n, 192)).cuda()
    wide200 = torch.zeros((n, 200), dtype=torch.uint8, device="cuda")
    cases = [
        ("NULL BLAS", lambda: raw(t, p, 192, n, api.HOST, [blas[0].h, None]), _lib.E_ARG),
        ("the TLAS as its own BLAS", lambda: raw(t, p, 192, n, api.HOST, [blas[0].h, t.h]), _lib.E_ARG),
        ("a TLAS as BLAS", lambda: raw(t, p, 192, n, api.HOST, [blas[0].h, other.h]), _lib.E_STATE),
        ("an empty BLAS", lambda: raw(t, p, 192, n, api.HOST, [blas[0].h, empty.h]), _lib.E_STATE),
        ("blasIdx past the list", lambda: raw(t, past.ctypes.data, 192, n, api.HOST, hs), _lib.E_ARG),
        ("fewer BLASes than blasIdx names", lambda: raw(t, p, 192, n, api.HOST, hs[:1]), _lib.E_ARG),
        ("host stride not a multiple of 4", lambda: raw(t, p, 194, n - 1, api.HOST, hs), _lib.E_ARG),
        ("stride below 160", lambda: raw(t, p, 156, n, api.HOST, hs), _lib.E_ARG),
        ("device stride not a multiple of 16", lambda: raw(t, wide200.data_ptr(), 200, n, api.DEVICE, hs), _lib.E_ARG),
        ("device pointer not 16-byte aligned", lambda: raw(t, dev.data_ptr() + 8, 192, n - 1, api.DEVICE, hs), _lib.E_ARG),
        ("unknown space", lambda: raw(t, p, 192, n, 7, hs), _lib.E_ARG),
        ("no instances", lambda: raw(t, p, 192, 0, api.HOST, hs), _lib.E_ARG),
        ("no BLASes", lambda: raw(t, p, 192, n, api.HOST, hs, count=0), _lib.E_ARG),
        ("NULL records", lambda: raw(t, None, 192, n, api.HOST, hs), _lib.E_ARG),
        ("deep BLAS without its CWBVH", lambda: raw(t, three.ctypes.data, 192, 3, api.HOST, [deep.h]), _lib.E_LIMIT),
    ]
    for what, call, code in cases:
        assert call() == code, f"{what}: {L.tbvh_last_error()}"
        assert rec.tobytes() == fresh.tobytes() and dev.cpu().numpy().tobytes() == fresh.tobytes(), f"{what}: the records changed"
        assert snapshot(t) == before and walks(t, O, D, (api.LAYOUT_BVH,)) == walked, f"{what}: the TLAS on the handle changed"
    # tbvh_build_tlas gives the same codes, and it too leaves the TLAS on the handle as it was
    hs2 = lambda h: (C.c_void_p * len(h))(*h)
    cases = [
        ("NULL BLAS", lambda: L.tbvh_build_tlas(t.h, p, 192, n, hs2([blas[0].h, None]), 2, 1.0, 1.0), _lib.E_ARG),
        ("the TLAS as its own BLAS", lambda: L.tbvh_build_tlas(t.h, p, 192, n, hs2([blas[0].h, t.h]), 2, 1.0, 1.0), _lib.E_ARG),
        ("a TLAS as BLAS", lambda: L.tbvh_build_tlas(t.h, p, 192, n, hs2([blas[0].h, other.h]), 2, 1.0, 1.0), _lib.E_STATE),
        ("an empty BLAS", lambda: L.tbvh_build_tlas(t.h, p, 192, n, hs2([blas[0].h, empty.h]), 2, 1.0, 1.0), _lib.E_STATE),
        ("blasIdx past the list", lambda: L.tbvh_build_tlas(t.h, past.ctypes.data, 192, n, hs2(hs), 2, 1.0, 1.0), _lib.E_ARG),
        ("fewer BLASes than blasIdx names", lambda: L.tbvh_build_tlas(t.h, inst.ctypes.data, 192, n, hs2(hs[:1]), 1, 1.0, 1.0), _lib.E_ARG),
        ("stride below 160", lambda: L.tbvh_build_tlas(t.h, p, 156, n, hs2(hs), 2, 1.0, 1.0), _lib.E_ARG),
        ("no instances", lambda: L.tbvh_build_tlas(t.h, p, 192, 0, hs2(hs), 2, 1.0, 1.0), _lib.E_ARG),
        ("NULL records", lambda: L.tbvh_build_tlas(t.h, None, 192, n, hs2(hs), 2, 1.0, 1.0), _lib.E_ARG),
        ("deep BLAS without its CWBVH", lambda: L.tbvh_build_tlas(t.h, three.ctypes.data, 192, 3, hs2([deep.h]), 1, 1.0, 1.0), _lib.E_LIMIT),
    ]
    for what, call, code in cases:
        assert call() == code, f"tbvh_build_tlas, {what}: {L.tbvh_last_error()}"
        assert snapshot(t) == before and walks(t, O, D, (api.LAYOUT_BVH,)) == walked, f"tbvh_build_tlas, {what}: the TLAS on the handle changed"
    # device records: blasIdx is the kernel's to check - reported, never dereferenced, and the handle ends up empty
    bad = torch.from_numpy(past.view(np.uint8).reshape(n, 192)).cuda()
    torch.cuda.synchronize()
    assert raw(t, bad.data_ptr(), 192, n, api.DEVICE, hs) == _lib.E_ARG and b"past blas_count" in L.tbvh_last_error()
    assert t.info().layouts == 0 and t.info().used_nodes == 0
    r = R.make_rays(O, D)
    assert L.tbvh_intersect(t.h, api.LAYOUT_BVH, r.ctypes.data, 128, 64) != 0
    # and the handle takes the next frame
    t.Rebuild(fresh, blas)
    good = fresh.copy()
    good["transform"] = util.random_transforms(n, 7)
    assert snapshot(t) == snapshot(api.TLAS().Build(good, blas)) and good.tobytes() == fresh.tobytes()
