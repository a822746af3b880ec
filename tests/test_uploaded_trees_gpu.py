"""Uploaded trees no builder makes (tests/util.py families: swapped children, reinserted subtrees, shuffled leaf ranges, and their
breadth-first renumbering), held to the restatement over the same bytes: the upload's info, the BVH_GPU and CWBVH conversions byte for
byte, every walk bit for bit, refits, a TLAS over such BLASses and a group replica.  The builder's own tree ("src") runs alongside.

A converted layout is only walked after its bytes matched: a wrong node array could send a walk anywhere."""
import ctypes as C
import functools

import numpy as np
import pytest

from oracle import portpy, refpy
from tinybvh_b200 import _lib, api, rays as R, scenes
from tests import util
from tests.cwbvh_refit_oracle import RefitCWBVH
from tests.test_convert_gpu import diff_blob, diff_nodes

pytestmark = pytest.mark.gpu
ZERO = {"prim": 0, "t": 0, "u": 0, "v": 0}
FAMS = ["src"] + util.FAMILIES
CASES = [(b, n, f) for b in ("Build", "BuildAVX", "BuildHQ") for n in (2, 5, 3000) for f in FAMS]
CASES += [(b, 120000, f) for b in ("Build", "BuildHQ") for f in ("src", "A0.3", "B", "C3", "DB")]
CASES += [("BuildAVX", 262267, "DB"), ("Build", 3000, "deep")]
# leaves of thousands of identical triangles: SplitLeafs turns each into a long chain of 3-triangle leaves (builder "<builder>/clusters")
CASES += [(f"{b}/clusters", 6000, f) for b in ("Build", "BuildAVX") for f in ("src", "A1", "C3", "DC")]
# where the reference is built: BVH::Build followed by the reference's own BVH::Optimize, the tree the shim's BVH::Optimize uploads
if refpy.available():
    CASES += [("Optimize", n, f) for n in (5, 3000, 30000) for f in ("src", "DB")]
IDS = [f"{b}-{n}-{f}" for b, n, f in CASES]


@pytest.fixture(scope="module", autouse=True)
def _free_cases():
    """The cases are cached for the whole module (every test function runs over all of them); freed when it ends."""
    yield
    case.cache_clear(), rays_for.cache_clear()


@functools.lru_cache(maxsize=None)
def case(builder, ntris, fam):
    """-> (verts, tree, restatement's BVH over the tree's bytes)"""
    builder, _, scene = builder.partition("/")
    v = util.long_leaf_scene(scene) if scene else scenes.procedural_scene(ntris, 71 + ntris % 7)
    assert v.shape[0] == 3 * ntris
    src = util.optimized_tree(v) if builder == "Optimize" else util.source_tree(v, builder)
    if fam == "src":
        t = src
    elif fam == "deep":
        t = util.reinserted(src, 3, 50, grow_to=100)
    else:
        t = util.family_tree(src, fam, 17)
    return v, t, portpy.PortBVH(v, nodes=t[0], prim_idx=t[1])


@functools.lru_cache(maxsize=None)
def rays_for(builder, ntris, fam):
    """camera, shadow and diffuse rays, each with the restatement's closest hits and shadow rays with their occlusion bits"""
    v, t, o = case(builder, ntris, fam)
    sets, bounds = util.ray_sets(v, res=32)
    want = o.intersect(sets["primary"].copy())
    out = {"camera": sets["primary"]}
    out.update(util.derived_sets(want, v, bounds))
    return out


def upload(t, v, space=api.HOST):
    e = api.BVH()
    if space == api.HOST:
        return e.upload(t[0], t[1], v)
    import torch
    d_nodes = torch.from_numpy(np.ascontiguousarray(t[0]).view(np.int32).copy()).cuda()
    d_idx = torch.from_numpy(t[1].view(np.int32).copy()).cuda()
    d_verts = torch.from_numpy(np.ascontiguousarray(v, np.float32).reshape(-1)).cuda()
    torch.cuda.synchronize()
    api.check(_lib.lib().tbvh_upload_bvh(e.h, C.c_void_p(d_nodes.data_ptr()), t[0].shape[0], C.c_void_p(d_idx.data_ptr()), t[2],
                                         C.c_void_p(d_verts.data_ptr()), 16, v.shape[0] // 3, api.DEVICE))
    return e


def referenced(t):
    return int(t[0]["triCount"][util.dfs_leaves(t[0])].sum())


def cw_port(t, v):
    return portpy.PortCWBVH(t[0], t[1], v, idx_count=t[2])


def check_cw_bytes(e, cw, t, label):
    d8, t8 = api.BVH8_CWBVH.download(e)
    diff_blob(d8, cw.nodes, label + " bvh8Data", 80)
    used = referenced(t) * 3
    assert t8.shape[0] >= used
    diff_blob(t8[:used], cw.tris[:used], label + " bvh8Tris", 48)


def occ_bits(o, rays):
    return np.unpackbits(o.occluded(rays.copy()).view(np.uint8), bitorder="little")[: rays.shape[0]].astype(bool)


def check_walks(e, layout, sets, closest, occluded, label):
    """Closest hit and occlusion of every set from host records and from 64-byte device records (hits into a 16-byte array), bit for bit.
    closest(rays) -> traced copy; occluded(rays) -> bool per ray."""
    from tests.test_hot_path_gpu import assert_hits, pack, run_anyhit, run_closest
    e.layout = layout
    for name, r in sets.items():
        want = closest(r.copy())
        got = r.copy()
        e.Intersect(got)
        assert util.compare_hits(got, want) == ZERO, f"{label} {name} host"
        assert_hits(run_closest(e, r, r.shape[0], "64+hits"), want, f"{label} {name} 64+hits", need_hit=False)
        s = r.copy()
        s["t"] = np.where(np.arange(r.shape[0]) % 2 == 0, R.BVH_FAR, want["t"] * np.float32(0.5)).astype(np.float32)
        occ = pack(occluded(s))
        assert np.array_equal(e.IsOccluded(s.copy()), occ), f"{label} {name} host any-hit"
        assert np.array_equal(run_anyhit(e, s, s.shape[0], 64), occ), f"{label} {name} 64-byte any-hit"


def cw_occluded(cw):
    # BVH8_CWBVH::IsOccluded is FALLBACK_SHADOW_QUERY: Intersect, then t < tmax (tiny_bvh.h:312)
    return lambda s: cw.intersect(s.copy())["t"] < s["t"]


@pytest.mark.parametrize("space", [api.HOST, api.DEVICE], ids=["host", "device"])
@pytest.mark.parametrize("builder,ntris,fam", CASES, ids=IDS)
def test_upload_info(gpu, builder, ntris, fam, space):
    v, t, o = case(builder, ntris, fam)
    e = upload(t, v, space)
    i = e.info()
    assert i.max_depth == util.tree_depth(t[0]) and (i.max_depth >= 64) == (fam == "deep")
    assert (i.used_nodes, i.idx_count, i.prim_count) == (t[0].shape[0], t[2], ntris)
    assert np.array_equal(np.array(i.aabb_min, np.float32).view(np.uint32), t[0][0]["aabbMin"].view(np.uint32))
    assert np.array_equal(np.array(i.aabb_max, np.float32).view(np.uint32), t[0][0]["aabbMax"].view(np.uint32))
    nodes, idx = e.download()
    assert nodes.tobytes() == t[0].tobytes() and idx.tobytes() == t[1].tobytes()


@pytest.mark.parametrize("builder,ntris,fam", CASES, ids=IDS)
def test_bvh_gpu_conversion(gpu, builder, ntris, fam):
    """BVH_GPU::ConvertFrom on the device: the restatement's bytes and node count; those bytes uploaded into a BVH_GPU handle walk
    like the restatement's BVH over the tree."""
    v, t, o = case(builder, ntris, fam)
    e = upload(t, v)
    api.check(_lib.lib().tbvh_convert(e.h, api.LAYOUT_BVH_GPU))
    want = o.to_bvh_gpu()
    assert e.info().used_nodes_gpu == want.shape[0] == t[0].shape[0] - 1
    got = api.BVH_GPU.download(e)
    diff_nodes(got, want, 16)
    g = api.BVH_GPU().upload(got, t[1], v)
    assert g.info().max_depth == util.tree_depth(t[0])
    check_walks(g, api.LAYOUT_BVH_GPU, rays_for(builder, ntris, fam), o.intersect, lambda s: occ_bits(o, s), f"{builder} {ntris} {fam} BVH_GPU upload")


# The depth-100 tree is left out: the restatement's conversion chain (SplitLeafs) holds a 64-entry stack, as the reference's does, so
# there is no byte oracle for the CWBVH of a tree that deep, and converted bytes are only walked after they matched one.
# (tests/test_deep_bvh2_gpu.py::test_cwbvh_of_a_deep_spine walks the CWBVH of deep builder-numbered spines.)
@pytest.mark.parametrize("builder,ntris,fam", [c for c in CASES if c[2] != "deep"], ids=[i for c, i in zip(CASES, IDS) if c[2] != "deep"])
def test_cwbvh_conversion(gpu, builder, ntris, fam):
    """SplitLeafs, 8-wide collapse and CWBVH encode of the uploaded tree: bvh8Data and the referenced bvh8Tris byte for byte, then
    the walk of those bytes."""
    v, t, o = case(builder, ntris, fam)
    e = upload(t, v)
    api.check(_lib.lib().tbvh_convert(e.h, api.LAYOUT_CWBVH))
    cw = cw_port(t, v)
    check_cw_bytes(e, cw, t, f"{builder} {ntris} {fam}")
    check_walks(e, api.LAYOUT_CWBVH, rays_for(builder, ntris, fam), cw.intersect, cw_occluded(cw), f"{builder} {ntris} {fam} CWBVH")


@pytest.mark.parametrize("builder,ntris,fam", [c for c in CASES if c[1] >= 3000], ids=[i for c, i in zip(CASES, IDS) if c[1] >= 3000])
def test_bvh_walks(gpu, builder, ntris, fam):
    """The BVH-layout walk of the uploaded tree under trace_variant 0, 3 and 4."""
    v, t, o = case(builder, ntris, fam)
    e = upload(t, v)
    try:
        for variant in (0, 3, 4):
            api.set_option("trace_variant", variant)
            check_walks(e, api.LAYOUT_BVH, rays_for(builder, ntris, fam), o.intersect, lambda s: occ_bits(o, s), f"{builder} {ntris} {fam} variant {variant}")
    finally:
        api.set_option("trace_variant", 3)


REFIT = [c for c in CASES if c[0] != "BuildHQ" and c[1] >= 5 and c[2] != "deep"]   # BVH::Refit refuses an SBVH


@pytest.mark.parametrize("builder,ntris,fam", REFIT, ids=[f"{b}-{n}-{f}" for b, n, f in REFIT])
def test_refit(gpu, builder, ntris, fam):
    """tbvh_refit with moved vertices: BVH::Refit over the uploaded nodes.  tbvh_refit_layouts on a handle holding BVH_GPU and CWBVH,
    two frames: the BVH2, BVH_GPU and CWBVH (kept collapse) bytes, then the CWBVH walk."""
    from tests.test_oracle_pin import moved
    v, t, o = case(builder, ntris, fam)
    e = upload(t, v)
    w = moved(v, 5, amp=0.05)
    ref = portpy.PortBVH(v, nodes=t[0].copy(), prim_idx=t[1])
    ref.refit(w)
    e.Refit(w)
    nodes, idx = e.download()
    assert nodes.tobytes() == ref.nodes.tobytes() and idx.tobytes() == t[1].tobytes(), "BVH2 differs from BVH::Refit"
    e = upload(t, v)
    for layout in (api.LAYOUT_BVH_GPU, api.LAYOUT_CWBVH):
        api.check(_lib.lib().tbvh_convert(e.h, layout))
    ref = portpy.PortBVH(v, nodes=t[0].copy(), prim_idx=t[1])
    for frame in (1, 2):
        w = moved(v, 50 + frame, amp=0.05)
        api._refit_layouts(e, w)
        ref.refit(w)
        label = f"{builder} {ntris} {fam} frame {frame}"
        nodes, idx = e.download()
        assert nodes.tobytes() == ref.nodes.tobytes(), f"{label}: BVH2 differs from BVH::Refit"
        diff_nodes(api.BVH_GPU.download(e), ref.to_bvh_gpu(), 16)
        cw = RefitCWBVH(t[0], ref.nodes, t[1], w, idx_count=t[2])
        check_cw_bytes(e, cw, t, label)
    if ntris >= 3000:
        sets, bounds = util.ray_sets(w, res=32)
        traced = cw.intersect(sets["primary"].copy())
        sets.update(util.derived_sets(traced, w, bounds))
        check_walks(e, api.LAYOUT_CWBVH, sets, cw.intersect, cw_occluded(cw), label)


def tlas_blasses(builder):
    """one BLAS per family, from different scenes"""
    out = []
    for k, fam in enumerate(util.FAMILIES):
        v = scenes.procedural_scene(3000, 200 + k)
        if builder == "Optimize":   # the reference's optimised trees themselves
            out.append((v, util.optimized_tree(v)))
            continue
        src = util.source_tree(v, builder)
        out.append((v, util.family_tree(src, fam, 30 + k)))
    return out


@pytest.mark.parametrize("blas_layout", [api.LAYOUT_BVH, api.LAYOUT_CWBVH], ids=["bvh", "cwbvh"])
@pytest.mark.parametrize("builder", ["Build", "BuildHQ"] + (["Optimize"] if refpy.available() else []))
def test_tlas_over_family_blasses(gpu, builder, blas_layout):
    """30 instances over BLASses of families A-D: TLAS bytes, hits and occlusion bit for bit the restatement's; SAHCost of every BLAS
    and of the TLAS BVH::SAHCost's."""
    from tests.test_tlas_gpu import words
    bl = tlas_blasses(builder)
    blas, port_blas = [], []
    for v, t in bl:
        e = upload(t, v)
        assert np.float32(e.SAHCost()).view(np.uint32) == np.float32(portpy.PortBVH(v, nodes=t[0], prim_idx=t[1]).sah_cost()).view(np.uint32)
        if blas_layout == api.LAYOUT_CWBVH:
            api.check(_lib.lib().tbvh_convert(e.h, api.LAYOUT_CWBVH))
            cw = cw_port(t, v)
            check_cw_bytes(e, cw, t, "BLAS")
            port_blas.append(cw)
        else:
            port_blas.append(portpy.PortBVH(v, nodes=t[0], prim_idx=t[1]))
        blas.append(e)
    from oracle import refpy
    n = 30
    inst = refpy.make_instances(util.random_transforms(n, 77), [i % len(blas) for i in range(n)], masks=[0xFFFF] * n)
    ref_inst = inst.copy()
    tl = api.TLAS().Build(inst, blas, blas_layout=blas_layout)
    tn, ti = tl.download()
    if blas_layout == api.LAYOUT_CWBVH:
        ref = util._PortTLAS(ref_inst, [portpy.PortBVH(v, nodes=t[0], prim_idx=t[1]) for v, t in bl])
        port = portpy.PortTLASCW(tn, ti, inst, port_blas)
        occluded = lambda s: np.unpackbits(port.occluded(s.copy()).view(np.uint8), bitorder="little")[: s.shape[0]].astype(bool)
    else:
        ref = util._PortTLAS(ref_inst, port_blas)
        port = ref
        occluded = lambda s: np.unpackbits(ref.occluded(s.copy()).view(np.uint8), bitorder="little")[: s.shape[0]].astype(bool)
    assert inst.tobytes() == ref_inst.tobytes()
    assert tn.tobytes() == ref.tree.nodes.tobytes() and np.array_equal(ti, ref.tree.prim_idx)
    assert np.float32(tl.SAHCost()).view(np.uint32) == np.float32(ref.tree.sah_cost()).view(np.uint32)
    rng = np.random.default_rng(5)
    D = rng.normal(size=(20000, 3)).astype(np.float32) * 0.35 + np.array([0, 0, 1], np.float32)
    rays = R.make_rays(np.tile(np.array([[0, 0, -120]], np.float32), (D.shape[0], 1)), D)
    want, got = port.intersect(rays.copy()), tl.Intersect(rays.copy())
    assert np.array_equal(words(got), words(want)) and (want["t"] < R.BVH_FAR).sum() > 1000
    s = rays.copy()
    s["t"] = np.where(np.arange(s.shape[0]) % 2 == 0, R.BVH_FAR, want["t"] * np.float32(0.5)).astype(np.float32)
    from tests.test_hot_path_gpu import pack
    assert np.array_equal(tl.IsOccluded(s), pack(occluded(s)))


@pytest.mark.parametrize("fam", ["A0.3", "B", "C3", "DB"])
@pytest.mark.parametrize("layout", [api.LAYOUT_BVH_GPU, api.LAYOUT_CWBVH], ids=["bvh_gpu", "cwbvh"])
def test_group_replica_of_converted_upload(gpu, layout, fam):
    """A converted uploaded handle replicated over a group: the source's converted bytes are the restatement's, and the replicas'
    hits and occlusion bits are the source's."""
    from tests.test_group_gpu import devices
    v, t, o = case("BuildAVX", 3000, fam)
    e = upload(t, v)
    api.check(_lib.lib().tbvh_convert(e.h, layout))
    if layout == api.LAYOUT_BVH_GPU:
        diff_nodes(api.BVH_GPU.download(e), o.to_bvh_gpu(), 16)
    else:
        check_cw_bytes(e, cw_port(t, v), t, fam)
    e.layout = layout
    g = api.Group(devices())
    try:
        g.replicate(e)
        for name, r in rays_for("BuildAVX", 3000, fam).items():
            want, got = e.Intersect(r.copy()), g.Intersect(r.copy())
            assert util.compare_hits(got, want) == ZERO, name
            assert np.array_equal(g.IsOccluded(r.copy()), e.IsOccluded(r.copy())), name
    finally:
        g.close()
