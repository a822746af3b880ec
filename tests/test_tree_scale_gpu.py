"""tbvh_optimize and TBVH_BUILD_PLOC on the device against their host restatements off the unit scale: signed-zero, power-of-two
scaled (2^-126 .. 2^90) and translated scenes, inside and outside the scale windows tests/test_tree_scale.py pins.  Nodes byte for
byte, rounds and SAHCost as float32 bits (NaN as NaN), the handle's info against an upload of the expected arrays, PLOC trees alone,
indexed and as neighbours in one batch, and the BVH_GPU / CWBVH conversions and walks of both producers' trees."""
import ctypes as C
import functools

import numpy as np
import pytest

from oracle import portpy
from tinybvh_b200 import _lib, api
from tests import util
from tests import optimize_oracle as oo
from tests import ploc_oracle as po
from tests.test_convert_gpu import diff_blob, diff_nodes
from tests.test_tree_scale import scale_nodes, unit_tree

pytestmark = pytest.mark.gpu
ZERO = ["zero:neg", "zero:random", "zero:order"]
SCALE = ["scale:%d" % k for k in (-126, -100, -60, -30, -6, 8, 24, 40, 60, 90)]
SHIFT = ["shift:1048576", "shift:-12582912"]
FAMS = ZERO + SCALE + SHIFT
BUILDERS = ["Build", "BuildAVX", "BuildHQ"]
LARGE = ["zero:random", "scale:-126", "scale:40", "scale:90", "shift:-12582912"]   # the 70,000-triangle subset
SIZES = [3, 40, 2000]
ROUNDS = 6
SUBSET = ["zero:random", "scale:-126", "scale:-60", "scale:40", "scale:90", "shift:-12582912"]


def grid():
    return [(f, n) for f in FAMS for n in SIZES] + [(f, 70000) for f in LARGE]


def bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


def same_f32(a, b):
    return bits(a) == bits(b) or (np.isnan(a) and np.isnan(b))


def node_bytes(nodes):
    return np.ascontiguousarray(nodes).view(np.uint8).tobytes()


@functools.lru_cache(maxsize=None)
def fam_mesh(fam, n):
    return util.family(fam, n)


@functools.lru_cache(maxsize=None)
def fam_tree(fam, n, builder):
    """The tree handed to the optimiser: the unit-scale tree with boxes times 2^k for a scaled family (the reference builder's own
    window kept out), the builder's tree of the family's mesh otherwise."""
    kind, arg = fam.split(":")
    if kind == "scale":
        t = unit_tree(n, builder, "src")
        return scale_nodes(t[0], int(arg)), t[1], t[2]
    return util.source_tree(fam_mesh(fam, n), builder)


@pytest.fixture(scope="module", autouse=True)
def _free_caches():
    yield
    fam_mesh.cache_clear(), fam_tree.cache_clear()


def check_optimized(e, v, want, wr, wsah, got_r, got_sah, idx, label):
    assert got_r == wr and same_f32(np.float32(got_sah), wsah), (label, got_r, got_sah, wr, wsah)
    nodes, gidx = e.download()
    assert node_bytes(nodes) == node_bytes(want), label
    assert np.array_equal(gidx, idx), label
    assert same_f32(np.float32(e.SAHCost()), wsah), label
    i, ref = e.info(), api.BVH().upload(want, idx, v).info()
    for f in ("used_nodes", "max_depth"):
        assert getattr(i, f) == getattr(ref, f), (label, f)
    assert bytes(i.aabb_min) == bytes(ref.aabb_min) and bytes(i.aabb_max) == bytes(ref.aabb_max), label


# ---- tbvh_optimize -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fam,n", grid(), ids=[f"{f}-{n}" for f, n in grid()])
@pytest.mark.parametrize("builder", BUILDERS)
def test_optimize_upload_matches_restatement(gpu, builder, fam, n):
    v = fam_mesh(fam, n)
    t = fam_tree(fam, n, builder)
    rounds = 2 if n >= 70000 else ROUNDS
    want, wr, wsah, _ = oo.optimize(t[0], t[1], rounds)
    e = api.BVH().upload(t[0], t[1], v)
    if wr == 0:   # 0 rounds keep the handle: its layouts and a TLAS over it stay valid
        _lib.check(_lib.lib().tbvh_convert(e.h, api.LAYOUT_CWBVH))
        layouts = e.info().layouts
        inst = np.zeros(1, api.BLAS_INSTANCE)
        inst["transform"] = np.eye(4, dtype=np.float32).reshape(-1)
        tl = api.TLAS().Build(inst, [e])
        r, s = e.optimize(rounds)
        assert e.info().layouts == layouts
        rays = util.unit_rays(fam, n)[:256]
        tl.Intersect(rays.copy())   # a stale TLAS refuses every walk
    else:
        r, s = e.optimize(rounds)
    check_optimized(e, v, want, wr, wsah, r, s, t[1], f"{builder} {fam} {n}")


@pytest.mark.parametrize("fam,n", grid(), ids=[f"{f}-{n}" for f, n in grid()])
@pytest.mark.parametrize("builder", BUILDERS)
def test_optimize_device_build_matches_restatement(gpu, builder, fam, n):
    """A device build of the family's mesh optimises to what the restatement makes of its downloaded bytes."""
    v = fam_mesh(fam, n)
    e = getattr(api.BVH(), builder)(v)
    nodes, idx = e.download()
    rounds = 2 if n >= 70000 else ROUNDS
    want, wr, wsah, _ = oo.optimize(nodes, idx, rounds)
    r, s = e.optimize(rounds)
    check_optimized(e, v, want, wr, wsah, r, s, idx, f"{builder} {fam} {n} device build")


# ---- PLOC --------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def ploc_want(fam, n):
    return po.build(fam_mesh(fam, n))


def check_ploc(e, v, want, label):
    nodes, idx, _, sah = want
    got_nodes, got_idx = e.download()
    assert node_bytes(got_nodes) == node_bytes(nodes), label
    assert np.array_equal(got_idx, idx), label
    assert same_f32(np.float32(e.SAHCost()), sah), label
    i, ref = e.info(), api.BVH().upload(nodes, idx, v).info()
    for f in ("used_nodes", "idx_count", "prim_count", "max_depth"):
        assert getattr(i, f) == getattr(ref, f), (label, f)
    assert bytes(i.aabb_min) == bytes(ref.aabb_min) and bytes(i.aabb_max) == bytes(ref.aabb_max), label


def indexed_of(v):
    """Unique vertices by their bits (np.unique on floats would merge -0 into +0) and the index buffer."""
    uniq, inv = np.unique(np.ascontiguousarray(v, np.float32).reshape(-1, 4).view(np.uint32), axis=0, return_inverse=True)
    return np.ascontiguousarray(uniq).view(np.float32), inv.astype(np.uint32).reshape(-1)


@pytest.mark.parametrize("fam,n", grid(), ids=[f"{f}-{n}" for f, n in grid()])
def test_ploc_matches_restatement(gpu, fam, n):
    v = fam_mesh(fam, n)
    want = ploc_want(fam, n)
    check_ploc(api.BVH().BuildPLOC(v), v, want, f"{fam} {n}")
    if n == 2000:
        uniq, ix = indexed_of(v)
        check_ploc(api.BVH().BuildPLOC(uniq, indices=ix), v, want, f"{fam} {n} indexed")


def test_ploc_batch_neighbours(gpu):
    """A 2^-126 mesh, a 2^90 mesh, a -0 mesh and a plain one in one batch, in two orders: each tree is its mesh's tree alone."""
    names = [("scale:-126", 2000), ("scale:90", 2000), ("zero:neg", 2000), ("scale:0", 2000)]
    vs = [fam_mesh(f, n) for f, n in names]
    wants = [po.build(v) for v in vs]
    for order in ([0, 1, 2, 3], [3, 2, 1, 0]):
        es = [api.BVH() for _ in order]
        api.build_batch(es, [vs[k] for k in order], flavour=api.BUILD_PLOC)
        for e, k in zip(es, order):
            check_ploc(e, vs[k], wants[k], f"batch {names[k]} order {order}")


# ---- downstream of both producers ---------------------------------------------------------------------------------------------
def cw_download(e):
    i = e.info()
    d = np.zeros((i.used_blocks, 4), np.float32)
    t = np.zeros((i.cwbvh_tri_count * 3, 4), np.float32)
    _lib.check(_lib.lib().tbvh_download_cwbvh(e.h, d.ctypes.data_as(C.c_void_p), t.ctypes.data_as(C.c_void_p), api.HOST))
    return d, t


def walk_layouts(e, v, nodes, idx, fam, label):
    """BVH_GPU and CWBVH of the handle's tree against the restatement's conversions of the same bytes, and the BVH, BVH_GPU and
    CWBVH walks bit for bit."""
    o = portpy.PortBVH(v, nodes=nodes, prim_idx=idx)
    _lib.check(_lib.lib().tbvh_convert(e.h, api.LAYOUT_BVH_GPU))
    diff_nodes(api.BVH_GPU.download(e), o.to_bvh_gpu(), 16)
    _lib.check(_lib.lib().tbvh_convert(e.h, api.LAYOUT_CWBVH))
    used = int(nodes["triCount"][util.dfs_leaves(nodes)].sum())
    cw = portpy.PortCWBVH(nodes, idx, v, idx_count=idx.shape[0])
    d8, t8 = cw_download(e)
    diff_blob(d8, cw.nodes, label + " bvh8Data", 80)
    diff_blob(t8[: used * 3], cw.tris[: used * 3], label + " bvh8Tris", 48)
    lim = util.cw_rd_limit(cw.nodes)
    # which slab test the CWBVH rays take: none takes the integer test at 2^-126 (a quantisation exponent reaches -128), a bound
    # of 2^(127 - e) that the rd_limit rays straddle at 2^90
    if fam == "scale:-126":
        assert lim is None
    if fam == "scale:90":
        assert lim is not None and lim < np.float32(2.0 ** 40)
    rays = util.unit_rays(fam, v.shape[0] // 3)
    finite = rays[np.isfinite(rays["rD"]).all(1)]
    for layout in (api.LAYOUT_BVH, api.LAYOUT_BVH_GPU):
        want, got = finite.copy(), finite.copy()
        o.intersect(want)
        _lib.check(_lib.lib().tbvh_intersect(e.h, layout, got.ctypes.data_as(C.c_void_p), got.dtype.itemsize, got.shape[0]))
        if fam == "scale:90":
            # A NaN distance (Moeller-Trumbore overflowing) ends every later comparison, so which triangle such a ray keeps is the
            # first one the walk reaches; the BVH2 walk's min / max drop NaN planes that the reference's ternary min / max keeps
            # (DESIGN 4.1, test_offatrium_gpu.py::test_bvh2_walk_with_infinite_rd), so the order, and the prim, can differ there.
            nan = np.isnan(want["t"])
            assert nan.any() and np.isnan(got["t"][nan]).all(), (label, layout)
            want, got = want[~nan], got[~nan]
        assert util.compare_hits(util.nan_canonical(got), util.nan_canonical(want)) == {"prim": 0, "t": 0, "u": 0, "v": 0}, (label, layout)
    cr = np.concatenate([rays, util.rd_limit_rays(rays, lim)])
    want, got = cr.copy(), cr.copy()
    cw.intersect(want)
    _lib.check(_lib.lib().tbvh_intersect(e.h, api.LAYOUT_CWBVH, got.ctypes.data_as(C.c_void_p), got.dtype.itemsize, got.shape[0]))
    assert util.compare_hits(util.nan_canonical(got), util.nan_canonical(want)) == {"prim": 0, "t": 0, "u": 0, "v": 0}, (label, "CWBVH")


@pytest.mark.parametrize("fam", SUBSET)
def test_ploc_tree_downstream(gpu, fam):
    v = fam_mesh(fam, 2000)
    nodes, idx, _, _ = ploc_want(fam, 2000)
    e = api.BVH().BuildPLOC(v)
    walk_layouts(e, v, nodes, idx, fam, f"PLOC {fam}")
    # tbvh_optimize of the PLOC tree
    f = api.BVH().BuildPLOC(v)
    want, wr, wsah, _ = oo.optimize(nodes, idx, ROUNDS)
    r, s = f.optimize(ROUNDS)
    check_optimized(f, v, want, wr, wsah, r, s, idx, f"PLOC {fam} optimised")


@pytest.mark.parametrize("fam", SUBSET)
@pytest.mark.parametrize("builder", ["Build", "BuildHQ"])
def test_optimized_tree_downstream(gpu, builder, fam):
    v = fam_mesh(fam, 2000)
    t = fam_tree(fam, 2000, builder)
    want, wr, wsah, _ = oo.optimize(t[0], t[1], ROUNDS)
    e = api.BVH().upload(t[0], t[1], v)
    assert e.optimize(ROUNDS)[0] == wr
    walk_layouts(e, v, want, t[1], fam, f"{builder} {fam} optimised")
