"""The path bench.py measures, held to the oracle: the tree built and converted on the GPU with the bench's calls, 64-byte device
records, closest hits into a separate 16-byte hit array, shadow rays made from those hits and any-hit bits, the statistics pass, the
host pipeline the e2e figures time, the block-cyclic sharding and the replica a rank other than 0 uploads.  Then every instance of the
CWBVH walk (k_trace_wide<any-hit, statistics, octant switch>) under every record shape the device entry points take."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest

import bench
from tinybvh_b200 import _lib, api, multi as M, rays as R, scenes
from tests import util

pytestmark = pytest.mark.gpu

SCENE = "bistro"             # the bench's default: camera_for / light_for take the stand-in's own bounds
RES = 64                     # 64 x 64 x 16 = 65,536 camera rays per arm
BISTRO_RES = 128             # 2^18 rays on the 2.8 M-triangle scene
SHARD_RES, SHARD_BLOCK = 132, 1 << 16   # 278,784 rays = 4 whole blocks of 2^16 and a ragged fifth
ARMS = [("cwbvh", "hq"), ("cwbvh", "sah"), ("bvh", "hq"), ("bvh", "sah")]
SENTINEL = np.uint32(0x5A5A5A5A)


def _ptr(t):
    return C.c_void_p(t.data_ptr())


def bench_engine(v, layout, tree):
    """bench.py run_ours: BVH::BuildHQ or BVH::Build on the GPU, then, for the CWBVH layout, tbvh_convert on the device."""
    e = api.BVH()
    e.BuildHQ(v) if tree == "hq" else e.Build(v)
    if layout == "cwbvh":
        api.check(_lib.lib().tbvh_convert(e.h, api.LAYOUT_CWBVH))
        e.layout = api.LAYOUT_CWBVH
    return e


class Oracle:
    """The reference's walk of the layout the bench traces, over the reference's tree of the same builder."""

    def __init__(self, v, layout, tree):
        self.layout = layout
        if layout == "cwbvh":
            self.cw, self.used = util.oracle_cwbvh(v, mode=1 if tree == "hq" else 2)
            self.walk = self.cw
        else:
            self.walk = util.oracle_tree(v, 2 if tree == "hq" else 0)

    def intersect(self, rays):
        out = rays.copy()
        self.walk.intersect(out)
        return out

    def occluded(self, shadow):
        """-> bool per ray.  BVH8_CWBVH::IsOccluded is FALLBACK_SHADOW_QUERY (tiny_bvh.h:312): Intersect, then t < tmax."""
        if self.layout == "cwbvh":
            return self.intersect(shadow)["t"] < shadow["t"]
        return unpack(self.walk.occluded(shadow.copy()), shadow.shape[0])


def unpack(words, n):
    return np.unpackbits(np.ascontiguousarray(words).view(np.uint8), bitorder="little")[:n].astype(bool)


def pack(occ):
    b = np.zeros((occ.shape[0] + 31) // 32 * 32, np.uint8)
    b[: occ.shape[0]] = occ
    return np.packbits(b, bitorder="little").view(np.uint32)


def to_device(records, stride=64):
    import torch
    return torch.from_numpy(np.ascontiguousarray(records.view(np.uint8).reshape(-1, 128)[:, :stride])).cuda()


def assert_hits(h, want, label, need_hit=True):
    """t bit for bit on every ray; u, v, prim on the rays that hit (test_cwbvh_gpu.check)."""
    h = np.ascontiguousarray(h, np.float32).reshape(-1, 4)
    bad = np.nonzero(h[:, 0].view(np.uint32) != want["t"].view(np.uint32))[0]
    assert bad.size == 0, f"{label}: t differs on {bad.size} of {h.shape[0]} rays, first {bad[:5]}"
    hit = want["t"] < R.BVH_FAR
    assert hit.any() or not need_hit, f"{label}: no ray hits"
    for k, f in ((1, "u"), (2, "v"), (3, "prim")):
        bad = np.nonzero(h[hit, k].view(np.uint32) != want[f][hit].view(np.uint32))[0]
        assert bad.size == 0, f"{label}: {f} differs on {bad.size} hits"


def workload(v, layout, tree, res):
    """The bench's setup of one step (run_ours), on one GPU."""
    import torch
    e = bench_engine(v, layout, tree)
    eye, view = bench.camera_for(SCENE, v)
    n = res * res * 16
    h_prim = np.zeros(n, R.RAY_DTYPE)
    R.primary_rays_into(h_prim, eye, view, res, res, 16)
    d_prim = torch.empty((n, 64), dtype=torch.uint8, device="cuda")
    api.copy_rays_to_device(h_prim, d_prim)
    d_hits = torch.empty((n, 4), dtype=torch.float32, device="cuda")
    e.Intersect(d_prim, hits=d_hits)
    torch.cuda.synchronize()
    hits = d_hits.cpu().numpy()
    h_shadow = np.zeros(n, R.RAY_DTYPE)
    R.shadow_rays_into(h_shadow, h_prim, bench.light_for(SCENE, v), bench.shadow_eps(v), hits=hits)
    d_shadow = torch.empty((n, 64), dtype=torch.uint8, device="cuda")
    api.copy_rays_to_device(h_shadow, d_shadow)
    d_bits = torch.empty((n + 31) // 32, dtype=torch.int32, device="cuda")
    e.IsOccluded(d_shadow, bits=d_bits)
    torch.cuda.synchronize()
    return SimpleNamespace(v=v, e=e, eye=eye, view=view, n=n, h_prim=h_prim, d_prim=d_prim, hits=hits, h_shadow=h_shadow,
                           d_shadow=d_shadow, bits=d_bits.cpu().numpy().view(np.uint32))


@pytest.fixture(scope="module")
def arms(gpu):
    """(layout, tree) -> the workload and its oracle on a seeded 150,000-triangle scene, built once per module."""
    v = scenes.procedural_scene(150000, 81)
    cache = {}

    def get(layout, tree):
        if (layout, tree) not in cache:
            w = workload(v, layout, tree, RES)
            w.o = Oracle(v, layout, tree)
            cache[layout, tree] = w
        return cache[layout, tree]

    yield get
    cache.clear()


def check_workload(w, label):
    import torch
    want = w.o.intersect(w.h_prim)
    assert_hits(w.hits, want, f"{label} device hits")
    occ = w.o.occluded(w.h_shadow)
    assert 0 < occ.sum() < w.n, f"{label}: occlusion is all or nothing"
    assert np.array_equal(w.bits, pack(occ)), f"{label}: {(unpack(w.bits, w.n) != occ).sum()} occlusion bits differ"
    # the bench's node_visits pass: the statistics instance, same results
    w.e.set_stats(True)
    try:
        h = torch.empty((w.n, 4), dtype=torch.float32, device="cuda")
        w.e.Intersect(w.d_prim, hits=h)
        torch.cuda.synchronize()
        assert w.e.get_stats()[0] > w.n
        b = torch.empty((w.n + 31) // 32, dtype=torch.int32, device="cuda")
        w.e.IsOccluded(w.d_shadow, bits=b)
        torch.cuda.synchronize()
        assert_hits(h.cpu().numpy(), want, f"{label} statistics pass")
        assert np.array_equal(b.cpu().numpy().view(np.uint32), w.bits), f"{label} statistics pass: occlusion bits"
    finally:
        w.e.set_stats(False)
    # e2e: the host calls on page-locked 128-byte records, in place and packed
    p = api.pinned_empty(w.n, R.RAY_DTYPE)
    try:
        p[:] = w.h_prim
        w.e.Intersect(p)
        assert_hits(np.stack([p["t"], p["u"], p["v"], p["prim"].view(np.float32)], 1), want, f"{label} host in place")
        packed = w.e.IntersectPacked(w.h_prim)
        assert_hits(packed.view(np.float32).reshape(-1, 4), want, f"{label} host packed")
        assert np.array_equal(w.e.IsOccluded(w.h_shadow), w.bits), f"{label} host occlusion bits"
    finally:
        api.pinned_free(p)


@pytest.mark.parametrize("layout,tree", ARMS)
def test_benchmark_workload_matches_oracle(arms, layout, tree):
    check_workload(arms(layout, tree), f"{layout}/{tree}")


def test_benchmark_workload_at_bistro_size(gpu):
    """The default arm on the measured scene (the procedural stand-in of the same size in a plain checkout): the wide-tree depth,
    pending count and exponent range of the measured run."""
    v = scenes.load_scene(SCENE)[0]
    w = workload(v, "cwbvh", "hq", BISTRO_RES)
    w.o = Oracle(v, "cwbvh", "hq")
    i = w.e.info()
    d8 = np.zeros((i.used_blocks, 4), np.float32)
    t8 = np.zeros((i.cwbvh_tri_count * 3, 4), np.float32)
    api.check(_lib.lib().tbvh_download_cwbvh(w.e.h, d8.ctypes.data, t8.ctypes.data, api.HOST))
    assert d8.shape == w.o.cw.nodes.shape and np.array_equal(d8.view(np.uint32), w.o.cw.nodes.view(np.uint32)), "bvh8Data differs"
    assert np.array_equal(t8[: w.o.used].view(np.uint32), w.o.cw.tris[: w.o.used].view(np.uint32)), "bvh8Tris differs"
    check_workload(w, "bistro cwbvh/hq")


@pytest.fixture(scope="module")
def whole(arms):
    """The sharding test's ray set traced whole, as one GPU runs it."""
    a = arms("cwbvh", "hq")
    return workload(a.v, "cwbvh", "hq", SHARD_RES)


@pytest.mark.parametrize("world", [2, 3, 8])
def test_block_cyclic_shards_reassemble_the_whole_set(whole, world):
    """Every rank generates its own blocks (primary_rays_into first=), traces them and makes its shadow rays from its own hits; put
    back in place, hits and occlusion words are the whole set's, and every occlusion word comes from exactly one rank.  With world 8
    three ranks hold no block."""
    import torch
    w = whole
    hits = np.full((w.n, 4), np.nan, np.float32)
    words = np.zeros((w.n + 31) // 32, np.uint32)
    owner = np.zeros(words.shape[0], np.int64)
    light, eps = bench.light_for(SCENE, w.v), bench.shadow_eps(w.v)
    for rank in range(world):
        blocks = M.block_cyclic(w.n, rank, world, SHARD_BLOCK)
        m = sum(c for _, c in blocks)
        if m == 0:
            continue
        h = np.zeros(m, R.RAY_DTYPE)
        off = 0
        for b0, bc in blocks:
            R.primary_rays_into(h[off:off + bc], w.eye, w.view, SHARD_RES, SHARD_RES, 16, first=b0)
            off += bc
        dh = torch.empty((m, 4), dtype=torch.float32, device="cuda")
        w.e.Intersect(to_device(h), hits=dh)
        rh = dh.cpu().numpy()
        sh = np.zeros(m, R.RAY_DTYPE)
        R.shadow_rays_into(sh, h, light, eps, hits=rh)
        db = torch.full(((m + 31) // 32,), -1, dtype=torch.int32, device="cuda")
        w.e.IsOccluded(to_device(sh), bits=db)
        rb = db.cpu().numpy().view(np.uint32)
        off = 0
        for b0, bc in blocks:
            hits[b0:b0 + bc] = rh[off:off + bc]
            nw = (bc + 31) // 32
            words[b0 // 32:b0 // 32 + nw] = rb[off // 32:off // 32 + nw]
            owner[b0 // 32:b0 // 32 + nw] += 1
            off += bc
    assert (owner == 1).all(), f"occlusion words written by {set(owner.tolist())} ranks"
    assert np.array_equal(hits.view(np.uint32), w.hits.view(np.uint32)), f"world {world}: hits differ from the whole-set trace"
    assert np.array_equal(words, w.bits), f"world {world}: occlusion words differ from the whole-set trace"


def test_replica_uploaded_from_device_arrays(arms):
    """The replica of a rank other than 0: the SBVH downloaded to device tensors, uploaded from DEVICE into a new handle with the
    SBVH's idx_count (its index slack included), then converted there.  Same bvh8Data / bvh8Tris, same hits."""
    import torch
    a = arms("cwbvh", "hq")
    L = _lib.lib()
    i = a.e.info()
    d_nodes = torch.empty(i.used_nodes * 8, dtype=torch.int32, device="cuda")
    d_idx = torch.empty(i.idx_count, dtype=torch.int32, device="cuda")
    api.check(L.tbvh_download_bvh(a.e.h, _ptr(d_nodes), _ptr(d_idx), api.DEVICE))
    d_verts = torch.from_numpy(a.v.reshape(-1)).cuda()
    torch.cuda.synchronize()
    r = api.BVH()
    api.check(L.tbvh_upload_bvh(r.h, _ptr(d_nodes), d_nodes.numel() // 8, _ptr(d_idx), d_idx.numel(), _ptr(d_verts), 16, a.v.shape[0] // 3, api.DEVICE))
    api.check(L.tbvh_convert(r.h, api.LAYOUT_CWBVH))
    r.layout = api.LAYOUT_CWBVH
    j = r.info()
    assert (j.idx_count, j.used_blocks, j.cwbvh_tri_count) == (i.idx_count, i.used_blocks, i.cwbvh_tri_count)
    got, want = [api.BVH8_CWBVH.download(x) for x in (r, a.e)]
    assert np.array_equal(got[0].view(np.uint32), want[0].view(np.uint32)), "bvh8Data differs"
    used = a.o.used
    assert np.array_equal(got[1][:used].view(np.uint32), want[1][:used].view(np.uint32)), "bvh8Tris differs"
    h = torch.empty((a.n, 4), dtype=torch.float32, device="cuda")
    r.Intersect(a.d_prim, hits=h)
    assert np.array_equal(h.cpu().numpy().view(np.uint32), a.hits.view(np.uint32))


# ---- every k_trace_wide instance, every record shape ------------------------------------------------------------------------

def matrix_rays(a):
    """Camera rays, axis-aligned rays with rD = safercp(D) and with rD = +-inf, and random rays of every octant, in uniform-octant and
    mixed warps; then warps around the integer-slab-test bound (util.rd_limit_rays), some with a single lane past it.  Bytes 64..127
    carry a pattern, so a write past the 64-byte record shows."""
    lo, hi = scenes.scene_bounds(a.v)
    cam = util.ray_sets(a.v, res=32)[0]["primary"]
    ax = util.axis_rays(lo, hi, per_axis=8, seed=9)
    r = util.octant_blocks(np.concatenate([cam, ax, util.with_inf_rd(ax), util.octant_rays(lo, hi, 64, 9)]), 9)
    r = r[: r.shape[0] // 32 * 32]
    r = np.concatenate([r, util.rd_limit_rays(r, util.cw_rd_limit(a.o.cw.nodes), 9)])
    r["aux"] = (np.arange(r.shape[0])[:, None] * 7 + np.arange(64)[None, :]) & 255
    return r


@pytest.fixture(scope="module")
def matrix(arms):
    a = arms("cwbvh", "hq")
    r = matrix_rays(a)
    want = a.o.intersect(r)
    # any-hit queries: tmax unbounded, exactly the closest hit (not occluded under FALLBACK_SHADOW_QUERY), or half of it
    s = r.copy()
    k = np.arange(r.shape[0]) % 3
    s["t"] = np.where(k == 0, R.BVH_FAR, np.where(k == 1, want["t"], want["t"] * np.float32(0.5))).astype(np.float32)
    occ = a.o.occluded(s)
    assert occ.any() and not occ.all()
    return a, r, want, s, occ


def run_closest(e, r, n, shape):
    """Closest hits of r[:n] on the device in one record shape: '64' / '128' byte records, in place or '+hits' into a 16-byte array.
    -> (n, 4) float32 hits; asserts that nothing but the hit bytes of an in-place call changed."""
    import torch
    stride = int(shape.split("+")[0])
    d = to_device(r[:n], stride)
    before = d.cpu().numpy()
    hits = torch.full((n, 4), float("nan"), dtype=torch.float32, device="cuda") if shape.endswith("+hits") else None
    e.Intersect(d, hits=hits)
    torch.cuda.synchronize()
    after = d.cpu().numpy()
    if hits is not None:
        assert np.array_equal(after, before), f"{shape}: the ray records changed"
        return hits.cpu().numpy()
    assert np.array_equal(after[:, :48], before[:, :48]) and np.array_equal(after[:, 64:], before[:, 64:]), f"{shape}: bytes outside 48..63 changed"
    return np.ascontiguousarray(after[:, 48:64]).view(np.float32)


def run_anyhit(e, s, n, stride):
    """-> the (n+31)/32 occlusion words of s[:n]; asserts the records are unchanged and the word after them is not written."""
    import torch
    d = to_device(s[:n], stride)
    before = d.cpu().numpy()
    bits = torch.full(((n + 31) // 32 + 1,), int(SENTINEL), dtype=torch.int32, device="cuda")
    bits[:-1] = -1
    e.IsOccluded(d, bits=bits)
    torch.cuda.synchronize()
    assert np.array_equal(d.cpu().numpy(), before), f"{stride}-byte records changed by the any-hit walk"
    got = bits.cpu().numpy().view(np.uint32)
    assert got[-1] == SENTINEL, f"n = {n}: the word after (n+31)/32 was written"
    return got[:-1]


@pytest.mark.parametrize("which", ["1", "31", "33", "full-37", "full"])
def test_every_wide_walk_instance_and_record_shape(matrix, which):
    """k_trace_wide<closest|any, statistics off|on, per-lane|octant switch> (trace_variant 0 and 3; statistics select <., true, 0>),
    64- and 128-byte records in place or with a hit array, on a ray count that is one lane, a partial warp, one ray past a warp, a ragged
    tail or the whole set: bit for bit the reference's walk of the same bytes, occlusion bits past n zero, and the statistics the same
    for every shape and variant and for a chunked host call."""
    a, r, want, s, occ = matrix
    full = r.shape[0]
    n = {"1": 1, "31": 31, "33": 33, "full-37": full - 37, "full": full}[which]
    e = a.e
    stats = {"closest": set(), "any": set()}
    try:
        for variant in (0, 3):
            api.set_option("trace_variant", variant)
            for st in (False, True):
                e.set_stats(st)
                for shape in ("64+hits", "64", "128", "128+hits"):
                    label = f"n={n} trace_variant {variant} stats {st} {shape}"
                    assert_hits(run_closest(e, r, n, shape), want[:n], label, need_hit=False)
                    if st:
                        stats["closest"].add(e.get_stats())
                for stride in (64, 128):
                    got = run_anyhit(e, s, n, stride)
                    assert np.array_equal(got, pack(occ[:n])), f"n={n} trace_variant {variant} stats {st} {stride}-byte any-hit: " \
                        f"{(unpack(got, n) != occ[:n]).sum()} of the n bits differ, last word {got[-1]:#010x}"
                    if st:
                        stats["any"].add(e.get_stats())
        assert len(stats["closest"]) == 1 and len(stats["any"]) == 1, f"statistics differ between shapes / variants: {stats}"
        # the same statistics from a host call cut into chunks of 4096 rays
        api.set_option("chunk_rays", 4096)
        e.set_stats(True)
        h = r[:n].copy()
        e.Intersect(h)
        assert e.get_stats() in stats["closest"], f"host call statistics {e.get_stats()} != device {stats['closest']}"
        e.IsOccluded(s[:n].copy())
        assert e.get_stats() in stats["any"]
        if n == full:
            assert next(iter(stats["closest"]))[0] > n
    finally:
        e.set_stats(False)
        api.set_option("trace_variant", 3)
        api.set_option("chunk_rays", 1 << 19)


def test_trace_on_a_caller_stream(arms):
    """stream= a torch.cuda.Stream: the walk is queued behind the copy that wrote its input on that stream (the stream is kept busy
    first, so a walk queued anywhere else would read the zeros the buffers start with)."""
    import torch
    a = arms("cwbvh", "hq")
    s = torch.cuda.Stream()
    d = torch.zeros_like(a.d_prim)
    sd = torch.zeros_like(a.d_shadow)
    hits = torch.full((a.n, 4), float("nan"), dtype=torch.float32, device="cuda")
    bits = torch.full(((a.n + 31) // 32,), -1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(20_000_000)
        d.copy_(a.d_prim)
    a.e.Intersect(d, hits=hits, stream=s)
    with torch.cuda.stream(s):
        sd.copy_(a.d_shadow)
    a.e.IsOccluded(sd, bits=bits, stream=s)
    s.synchronize()
    assert np.array_equal(hits.cpu().numpy().view(np.uint32), a.hits.view(np.uint32))
    assert np.array_equal(bits.cpu().numpy().view(np.uint32), a.bits)
