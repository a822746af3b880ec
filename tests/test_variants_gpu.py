"""Every tuning variant (tbvh_set_option) must give the oracle's results: the traversal-kernel variants change which
lane / code path runs a ray, never its arithmetic or order; the host-path modes change how bytes cross PCIe."""
from types import SimpleNamespace

import numpy as np
import pytest

from tinybvh_b200 import _lib, api, rays as R, scenes
from tinybvh_b200._lib import BUILD_REFERENCE
from tests import util
from tests.test_oracle_pin import tlas_case
from tests.test_tlas_gpu import words

pytestmark = pytest.mark.gpu
ZERO = {"prim": 0, "t": 0, "u": 0, "v": 0}


@pytest.fixture(scope="module")
def world():
    v = scenes.procedural_scene(40000, 71)
    o = util.oracle_bvh(v)
    sets, bounds = util.ray_sets(v, res=128)
    prim = sets["primary"].copy()
    o.intersect(prim)
    d = util.derived_sets(prim, v, bounds)
    want = {"primary": prim, "diffuse": d["diffuse"].copy(), "shadow_bits": o.occluded(d["shadow"])}
    o.intersect(want["diffuse"])
    return v, sets["primary"], d, want


@pytest.mark.parametrize("variant", [0, 3, 4])
def test_trace_variants_are_bit_exact(gpu, world, variant):
    v, primary, d, want = world
    import torch
    api.set_option("trace_variant", variant)
    try:
        e = api.BVH().Build(v)
        for name, rays in (("primary", primary), ("diffuse", d["diffuse"])):
            got = rays.copy()
            e.Intersect(got)
            assert util.compare_hits(got, want[name]) == ZERO, f"variant {variant} {name}"
            # device path with a ragged count (persistent kernel tail handling)
            m = rays.shape[0] - 37
            dev = torch.from_numpy(R.gpu_records(rays[:m]).view(np.uint8).reshape(-1, 64).copy()).cuda()
            hits = torch.zeros((m, 4), dtype=torch.float32, device="cuda")
            e.Intersect(dev, hits=hits)
            torch.cuda.synchronize()
            h = hits.cpu().numpy()
            assert np.array_equal(h[:, 0].view(np.uint32), want[name]["t"][:m].view(np.uint32))
            assert np.array_equal(h[:, 3].view(np.uint32), want[name]["prim"][:m])
        assert np.array_equal(e.IsOccluded(d["shadow"]), want["shadow_bits"]), f"variant {variant} occlusion"
        m = d["shadow"].shape[0] - 37
        assert np.array_equal(e.IsOccluded(d["shadow"][:m].copy()), util.oracle_bvh(v).occluded(d["shadow"][:m].copy()))
    finally:
        api.set_option("trace_variant", 3)


N_HOST = 65536 + 4096 + 100   # with 4096-ray chunks: 18 chunks (more than TBVH_SLOTS = 4), a ragged last chunk and occlusion word,
                              # and past d2h_mode 2's host-scatter threshold of 65,536 rays
STRIDES = (128, 64, 144, 136)  # 136 is not a multiple of 16: the gather (host_path 1) and the scatter (d2h_mode 3) must step aside
SENTINEL = np.uint32(0x5A5A5A5A)


def hit_words(records):
    """bytes 48..63 (t, u, v, prim) of every record of a [n, stride] byte array, as uint32 [n, 4]"""
    return np.ascontiguousarray(records[:, 48:64]).view(np.uint32)


@pytest.fixture(scope="module")
def host_world(world):
    """N_HOST camera and shadow rays with the oracle's hits and occlusion words in each layout, the engines, and a TLAS per layout with
    the device path's in-place results (held to the oracle in test_tlas_gpu.py)."""
    import torch
    v, primary, d, want = world
    rays, shadow = primary[:N_HOST].copy(), d["shadow"][:N_HOST].copy()
    cw, _ = util.oracle_cwbvh(v, mode=2)
    traced = rays.copy()
    cw.intersect(traced)
    tr = shadow.copy()
    cw.intersect(tr)
    occ_cw = tr["t"] < shadow["t"]   # BVH8_CWBVH::IsOccluded is FALLBACK_SHADOW_QUERY (tiny_bvh.h:312)
    bvh_words = hit_words(want["primary"][:N_HOST].view(np.uint8).reshape(-1, 128))
    bvh_bits = util.oracle_bvh(v).occluded(shadow.copy())
    cw_bits = np.packbits(np.concatenate([occ_cw, np.zeros(-N_HOST % 32, bool)]).astype(np.uint8), bitorder="little").view(np.uint32)
    engines = {}
    for name, cls in (("BVH", api.BVH), ("BVH_GPU", api.BVH_GPU), ("CWBVH", api.BVH8_CWBVH)):
        e = cls()
        e.build_flavour = BUILD_REFERENCE   # the derived layouts over BVH::Build's tree, which the oracles convert
        e.Build(v)
        engines[name] = e
    want_layout = {"BVH": (bvh_words, bvh_bits), "BVH_GPU": (bvh_words, bvh_bits), "CWBVH": (hit_words(traced.view(np.uint8).reshape(-1, 128)), cw_bits)}
    tv, inst, O, D = tlas_case(93, 24)
    blas = [api.BVH8_CWBVH().Build(x) for x in tv]
    t_bvh = api.TLAS().Build(inst.copy(), blas)
    t_cw = api.TLAS().Build(inst.copy(), blas, blas_layout=api.LAYOUT_CWBVH)
    t_rays = R.make_rays(O, D)
    tlas = {}
    for name, t in (("BVH", t_bvh), ("CWBVH", t_cw)):
        dev = torch.from_numpy(t_rays.view(np.uint8).reshape(-1, 128).copy()).cuda()
        t.Intersect(dev)
        tlas[name] = (t, words(dev.cpu().numpy().view(R.RAY_DTYPE).reshape(-1)))
    tlas["BVH_GPU"] = tlas["BVH"]
    return SimpleNamespace(rays=rays, shadow=shadow, engines=engines, want=want_layout, tlas=tlas, t_rays=t_rays, blas=blas)


def strided(rays, stride, pinned):
    """bytes 0..63 of every 128-byte record in records of `stride` bytes, page-locked or pageable; bytes 64.. carry a pattern"""
    n = rays.shape[0]
    buf = api.pinned_empty(n * stride, np.uint8).reshape(n, stride) if pinned else np.empty((n, stride), np.uint8)
    buf[:, :64] = rays.view(np.uint8).reshape(-1, 128)[:, :64]
    buf[:, 64:] = (np.arange(n)[:, None] * 13 + np.arange(stride - 64)[None, :]) & 255
    return buf


@pytest.mark.parametrize("chunk", [4096, 1 << 19])
@pytest.mark.parametrize("h2d_split", [1, 3])
@pytest.mark.parametrize("host_path", [0, 1, 2])
@pytest.mark.parametrize("layout", ["BVH", "BVH_GPU", "CWBVH"])
@pytest.mark.parametrize("mode", [0, 1, 2, 3])
def test_host_path_modes_return_the_same_hits(gpu, host_world, mode, layout, host_path, h2d_split, chunk):
    """tbvh_intersect (in place), tbvh_intersect_packed and tbvh_occluded on host records of 128, 64, 144 and 136 bytes, page-locked and
    pageable, under every d2h_mode, host_path, h2d_split and chunk size: the oracle's hits and occlusion words; in place only bytes
    48..63 of a record change, the packed call and the any-hit call change no byte of the rays, and exactly (n+31)/32 words are
    written.  A TLAS traces in place under each mode, and its packed call is refused."""
    L = _lib.lib()
    w = host_world
    e, lay = w.engines[layout], getattr(api, "LAYOUT_" + layout)
    want_hits, want_bits = w.want[layout]
    n, nw = N_HOST, (N_HOST + 31) // 32
    api.set_option("d2h_mode", mode)
    api.set_option("host_path", host_path)
    api.set_option("h2d_split", h2d_split)
    api.set_option("chunk_rays", chunk)
    try:
        for stride in STRIDES:
            for pinned in (True, False):
                label = f"{layout} d2h_mode {mode} host_path {host_path} h2d_split {h2d_split} chunk {chunk} stride {stride} {'pinned' if pinned else 'pageable'}"
                buf = strided(w.rays, stride, pinned)
                try:
                    before = buf.copy()
                    api.check(L.tbvh_intersect(e.h, lay, buf.ctypes.data, stride, n))
                    bad = np.nonzero((hit_words(buf) != want_hits).any(1))[0]
                    assert bad.size == 0, f"{label}: in-place hits differ on {bad.size} rays, first {bad[:5]}"
                    assert np.array_equal(buf[:, :48], before[:, :48]) and np.array_equal(buf[:, 64:], before[:, 64:]), f"{label}: bytes outside 48..63 changed"
                    buf[:] = before
                    hits = np.zeros((n, 4), np.uint32)
                    api.check(L.tbvh_intersect_packed(e.h, lay, buf.ctypes.data, stride, n, hits.ctypes.data))
                    assert np.array_equal(hits, want_hits), f"{label}: packed hits differ on {(hits != want_hits).any(1).sum()} rays"
                    assert np.array_equal(buf, before), f"{label}: the packed call changed the rays"
                finally:
                    if pinned:
                        api.pinned_free(buf)
                sh = strided(w.shadow, stride, pinned)
                try:
                    before = sh.copy()
                    bits = np.full(nw + 1, SENTINEL, np.uint32)
                    api.check(L.tbvh_occluded(e.h, lay, sh.ctypes.data, stride, n, bits.ctypes.data))
                    assert np.array_equal(bits[:nw], want_bits), f"{label}: {np.unpackbits((bits[:nw] ^ want_bits).view(np.uint8)).sum()} occlusion bits differ"
                    assert bits[nw] == SENTINEL, f"{label}: the word after (n+31)/32 was written"
                    assert np.array_equal(sh, before), f"{label}: the any-hit call changed the rays"
                finally:
                    if pinned:
                        api.pinned_free(sh)
        t, t_want = w.tlas[layout]
        for pinned in (True, False):
            tr = api.pinned_empty(w.t_rays.shape[0], R.RAY_DTYPE) if pinned else np.empty_like(w.t_rays)
            try:
                tr[:] = w.t_rays
                t.Intersect(tr)
                assert np.array_equal(words(tr), t_want), f"TLAS over {layout} BLASses, d2h_mode {mode} host_path {host_path}: hits differ"
            finally:
                if pinned:
                    api.pinned_free(tr)
        with pytest.raises(api.TbvhError):
            t.IntersectPacked(w.t_rays)   # TLAS hits carry the instance: in place only
    finally:
        api.set_option("d2h_mode", 1)
        api.set_option("host_path", 0)
        api.set_option("h2d_split", 1)
        api.set_option("chunk_rays", 1 << 19)
        api.set_option("trace_variant", 3)


@pytest.mark.parametrize("small_t", [8, 64, 256])
def test_builder_switch_point_does_not_change_the_tree(gpu, small_t):
    v = scenes.procedural_scene(30000, 72)
    o = util.oracle_bvh(v)
    api.set_option("small_t", small_t)
    try:
        nodes, idx = api.BVH().Build(v).download()
        assert np.array_equal(nodes.view(np.uint32), np.ascontiguousarray(o.nodes).view(np.uint32)) and np.array_equal(idx, o.prim_idx)
    finally:
        api.set_option("small_t", 128)


def test_long_host_batches_under_every_variant(gpu):
    """Host batches longer than a pipeline chunk, several chunks in flight on different streams: the persistent-warp variant pulls
    rays off a counter that must belong to ONE launch, and statistics must add up over the chunks of one call."""
    v = scenes.procedural_scene(30000, 73)
    o = util.oracle_bvh(v)
    lo, hi = scenes.scene_bounds(v)
    rays = R.primary_rays(*R.bounds_camera(lo, hi, "inside"), 384, 384, 16)   # 2,359,296 rays = 4.5 chunks of 2^19
    want = rays.copy()
    o.intersect(want, threads=0)
    sh = util.derived_sets(want, v, (lo, hi))["shadow"]
    want_bits = o.occluded(sh, threads=0)
    e = api.BVH().Build(v)
    for variant in (3, 4, 0):
        api.set_option("trace_variant", variant)
        try:
            got = rays.copy()
            e.Intersect(got)
            assert util.compare_hits(got, want) == ZERO, f"variant {variant}"
            assert np.array_equal(e.IsOccluded(sh), want_bits), f"variant {variant} occlusion"
        finally:
            api.set_option("trace_variant", 3)
    # statistics of a multi-chunk call = statistics of the same rays traced in one device launch
    import torch
    e.set_stats(True)
    got = rays.copy()
    e.Intersect(got)
    host_stats = e.get_stats()
    dev = torch.from_numpy(R.gpu_records(rays).view(np.uint8).reshape(-1, 64).copy()).cuda()
    e.Intersect(dev)
    torch.cuda.synchronize()
    assert e.get_stats() == host_stats and host_stats[0] > rays.shape[0]
    e.set_stats(False)


def test_concurrent_host_calls_on_one_handle(gpu):
    """SURVEY 8(b): batch calls are thread-safe per handle (the reference's const Intersect is called from many threads)."""
    import threading
    v = scenes.procedural_scene(20000, 74)
    o = util.oracle_bvh(v)
    lo, hi = scenes.scene_bounds(v)
    e = api.BVH().Build(v)
    sets, errs = [], []
    for k, kind in enumerate(("inside", "outside", "inside", "outside")):
        r = R.primary_rays(*R.bounds_camera(lo, hi, kind), 192 + 64 * k, 192, 16)
        w = r.copy()
        o.intersect(w, threads=0)
        sets.append((r, w))

    def work(r, w):
        try:
            for _ in range(3):
                g = r.copy()
                e.Intersect(g)
                if util.compare_hits(g, w) != ZERO:
                    errs.append("mismatch")
        except Exception as ex:  # noqa: BLE001
            errs.append(repr(ex))

    th = [threading.Thread(target=work, args=s) for s in sets]
    [t.start() for t in th]
    [t.join() for t in th]
    assert not errs, errs


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("ntris,seed", [(90000, 75), (3000, 76), (129, 77)])
def test_both_large_phase_drivers_build_the_reference_tree(gpu, mode, ntris, seed):
    """build_mode 0 = the persistent cooperative launch (k_large_phase), 1 = one launch per stage and level: same tree, byte for byte."""
    v = scenes.procedural_scene(ntris, seed)
    o = util.oracle_bvh(v)
    api.set_option("build_mode", mode)
    try:
        nodes, idx = api.BVH().Build(v).download()
        assert np.array_equal(nodes.view(np.uint32), np.ascontiguousarray(o.nodes).view(np.uint32)) and np.array_equal(idx, o.prim_idx)
        nodes2, _ = api.BVH().BuildAVX(v).download()
        from oracle import refpy
        if refpy.available():
            ra = refpy.RefBVH(v, mode=1, threaded=False)
            assert np.array_equal(nodes2.view(np.uint32), np.ascontiguousarray(ra.nodes).view(np.uint32))
    finally:
        api.set_option("build_mode", 0)
