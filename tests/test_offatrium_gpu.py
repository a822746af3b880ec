"""GPU parity away from the procedural atrium: signed-zero coordinates, scenes scaled by powers of two far outside [-40,40],
scenes translated by millions of units, long leaves that SplitLeafs turns into chains, and rays at the edges of the walks
(axis-aligned directions with +-0 components, user-supplied rD = +-inf, |rD| around the CWBVH integer-slab bound, origins at
2^126, shadow rays with tmax equal to a hit distance).  Trees and layouts are held byte for byte, walks bit for bit, to the same
oracles as the rest of the suite (tests/util.py)."""
import numpy as np
import pytest

from tinybvh_b200 import api, rays as R, scenes
from tinybvh_b200._lib import BUILD_REFERENCE
from tests import util
from tests.test_build_gpu import assert_same_tree
from tests.test_build_hq_gpu import assert_same_hq_tree
from tests.test_convert_gpu import diff_blob, diff_nodes
from tests.test_tlas_gpu import _CW, words
from tests.util import family, unit_rays  # noqa: F401 (other test modules import them from here)

pytestmark = pytest.mark.gpu

ZERO = ["zero:pos", "zero:neg", "zero:random", "zero:order"]
SCALE = ["scale:%d" % k for k in (-126, -100, -60, -6, -4, 8, 16, 24, 30, 40, 90)]
SHIFT = ["shift:1048576", "shift:-12582912"]   # +2^20, -3 * 2^22
BUILDERS = {"Build": 0, "BuildAVX": 1, "BuildHQ": 2}


def engine_tree(v, builder):
    return getattr(api.BVH(), builder)(v)


def assert_tree(e, v, builder, label):
    if builder == "BuildHQ":
        from oracle import portpy
        nodes, idx, ic = portpy.build_hq(v)
        assert_same_hq_tree(e, nodes, idx, ic, label)
    else:
        o = util.oracle_tree(v, BUILDERS[builder])
        assert_same_tree(e, o.nodes, o.prim_idx, label)


# ---- trees ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ntris", [1, 3, 40, 2000])
@pytest.mark.parametrize("fam", ZERO + SCALE + SHIFT)
@pytest.mark.parametrize("builder", list(BUILDERS))
def test_tree_matches_oracle(gpu, builder, fam, ntris):
    v = family(fam, ntris)
    if fam.startswith("zero") and fam != "zero:pos" and ntris >= 40:
        assert util.count_neg_zero(v[:, :3]) > 0
    assert_tree(engine_tree(v, builder), v, builder, f"{builder} {fam} {ntris}")


@pytest.mark.parametrize("fam", ["zero:random", "zero:order", "scale:-126", "scale:40", "shift:1048576"])
@pytest.mark.parametrize("build_mode", [0, 1])
@pytest.mark.parametrize("builder", list(BUILDERS))
def test_tree_matches_oracle_large(gpu, builder, build_mode, fam):
    """70k triangles: the large phase (nodes above small_t) runs over several levels, in both drivers of the SAH build."""
    v = family(fam, 70000)
    api.set_option("build_mode", build_mode)
    try:
        e = engine_tree(v, builder)
    finally:
        api.set_option("build_mode", 0)
    assert_tree(e, v, builder, f"{builder} {fam} 70k mode {build_mode}")


def test_single_triangle_signed_zero_order(gpu):
    """The reference's root bound takes the sign of the last tied vertex: +0 for (-0, +0, 1), -0 once the first two are swapped."""
    a, b = util.zero_tri_cases()
    for v, neg in ((a, False), (b, True)):
        for builder in ("Build", "BuildAVX", "BuildHQ"):
            nodes, _ = engine_tree(v, builder).download()
            assert bool(np.signbit(nodes[0]["aabbMin"][0])) == neg, f"{builder}: root aabbMin.x sign"
            assert_tree(engine_tree(v, builder), v, builder, builder)


def test_tlas_signed_zero_instance_boxes(gpu):
    """Instances at the origin under exact axis-permutation and mirror matrices: BLASInstance::Update gives boxes with -0 and
    +0 bounds, and the TLAS build over them must fold their signs as the reference does."""
    v = []
    for k in range(3):
        x = util.signed_zero(scenes.procedural_scene(300, 40 + k), "random", k)
        x[:, 1] -= x[:, 1].min()                     # the floor at exactly y = 0: the BLAS box touches the plane ...
        x[:, 0] -= x[:, 0].max() + 1                 # ... and x, z < 0, so 0 * x and 0 * z in Update's transform are -0
        x[:, 2] -= x[:, 2].max() + 1
        x[:, 1][(x[:, 1] == 0) & (np.arange(x.shape[0]) % 2 == k % 2)] = util.NEG_ZERO
        v.append(x)
    perms = [(0, 1, 2), (1, 2, 0), (2, 0, 1), (1, 0, 2), (0, 2, 1), (2, 1, 0)]
    inst = np.zeros(24, api.BLAS_INSTANCE)
    for i in range(inst.shape[0]):
        m = np.zeros((4, 4), np.float32)
        p, s = perms[i % 6], (-1 if i % 4 == 1 else 1, -1 if i % 3 == 2 else 1, -1 if i % 5 == 3 else 1)
        for r in range(3):
            m[r, p[r]] = s[r]
            m[r, 3] = util.NEG_ZERO if (i + r) % 2 else 0   # a -0 translation keeps a sum of -0 terms at -0
        m[3, 3] = 1
        inst[i]["transform"] = m.reshape(-1)
        inst[i]["blasIdx"] = i % 3
        inst[i]["mask"] = 0xFFFF
    inst_ref = inst.copy()
    ref = util.oracle_tlas(inst_ref, v, 0)
    t = api.TLAS().Build(inst, [api.BVH().Build(x) for x in v])
    assert inst.tobytes() == inst_ref.tobytes(), "BLASInstance::Update differs"
    assert util.count_neg_zero(np.concatenate([inst["aabbMin"], inst["aabbMax"]])) > 0
    nodes, idx = t.download()
    rb = ref.bvh()
    assert np.array_equal(nodes.view(np.uint32), rb.nodes.view(np.uint32)) and np.array_equal(idx, rb.prim_idx), "TLAS tree differs"
    lo, hi = inst["aabbMin"].min(0), inst["aabbMax"].max(0)
    rays = util.octant_blocks(np.concatenate([util.axis_rays(lo, hi, 8, 3), util.ray_sets(np.concatenate(v), res=16)[0]["primary"]]))
    want, got = rays.copy(), rays.copy()
    ref.intersect(want), t.Intersect(got)
    assert np.array_equal(words(got), words(want))


# ---- conversions and walks ---------------------------------------------------------------------------------------------
def check_walk(e, want_fn, rays, label):
    want, got = rays.copy(), rays.copy()
    want_fn(want), e.Intersect(got)
    g, w = util.nan_canonical(got), util.nan_canonical(want)
    cmp = util.compare_hits(g, w)
    if cmp != {"prim": 0, "t": 0, "u": 0, "v": 0}:
        bad = np.nonzero((g["prim"] != w["prim"]) | (g["t"].view(np.uint32) != w["t"].view(np.uint32)) | (g["u"].view(np.uint32) != w["u"].view(np.uint32))
                         | (g["v"].view(np.uint32) != w["v"].view(np.uint32)))[0]
        k = bad[0]
        pytest.fail(f"{label}: {cmp}; first at {k} of {rays.shape[0]}: got t {got['t'][k]!r} prim {got['prim'][k]}, want t {want['t'][k]!r} "
                    f"prim {want['prim'][k]}; ray O {rays['O'][k]!r} D {rays['D'][k]!r} rD {rays['rD'][k]!r}")
    return want


def finite_rd(rays):
    """The rays without a user-supplied infinite rD: the BVH2 walk's min / max drop a NaN plane the reference keeps (DESIGN 4.1),
    test_bvh2_walk_with_infinite_rd below."""
    return rays[np.isfinite(rays["rD"]).all(1)]


@pytest.mark.xfail(strict=True, reason="the BVH2 slab test's FMNMX drops NaN planes (0 * inf) that the reference's ternary min / max keeps")
def test_bvh2_walk_with_infinite_rd(gpu):
    """Axis rays with rD = +-inf on their zero direction components and origins on the scene's zero planes."""
    v = family("zero:neg", 40)
    o = util.oracle_tree(v, 0)
    lo, hi = scenes.scene_bounds(scenes.procedural_scene(40, 5))
    r = util.with_inf_rd(util.axis_rays(lo, hi, 8, 5))
    check_walk(engine_tree(v, "Build"), o.intersect, r, "BVH rD = inf")


# families whose shadow rays (tmax = the BVH's hit distance) meet a CWBVH triangle at exactly tmax, where BVH::IsOccluded
# (t <= tmax) and BVH8_CWBVH::IsOccluded (t < tmax) differ: the check above is held at that edge
EDGE_CASES = {("scale:-6", 2000), ("scale:-4", 2000), ("shift:-12582912", 40), ("shift:-12582912", 2000)}


def occlusion_bits(rays, occ):
    return np.unpackbits(np.ascontiguousarray(occ).view(np.uint8), bitorder="little")[: rays.shape[0]].astype(bool)


@pytest.mark.parametrize("ntris", [3, 40, 2000])
@pytest.mark.parametrize("fam", ZERO[1:] + SCALE + SHIFT)
def test_layouts_and_walks_match_oracle(gpu, fam, ntris):
    """BVH_GPU and CWBVH converted on the device from the engine's BVH::Build tree: bytes as the reference converts them; the
    BVH, BVH_GPU and CWBVH walks bit for bit as the reference walks the same bytes, under every trace variant and with statistics."""
    v = family(fam, ntris)
    o = util.oracle_tree(v, 0)
    rays = unit_rays(fam, ntris)
    g = api.BVH_GPU()
    g.build_flavour = BUILD_REFERENCE
    g.Build(v)
    diff_nodes(g.download(), util.oracle_bvh_gpu_nodes(o), 16)
    cw, _ = util.oracle_cwbvh(v, mode=2)
    c = api.BVH8_CWBVH()
    c.build_flavour = BUILD_REFERENCE
    c.Build(v)
    nodes, tris = c.download()
    diff_blob(nodes, cw.nodes, f"{fam} bvh8Data", 80)
    diff_blob(tris[: cw.tris.shape[0]], cw.tris, f"{fam} bvh8Tris", 48)
    rays = np.concatenate([rays, util.rd_limit_rays(rays, util.cw_rd_limit(cw.nodes))])
    b = engine_tree(v, "Build")
    edge_rays = 0   # shadow rays on which the two reference layouts' occlusion queries differ: the t == tmax edge is reached
    for variant in (0, 3, 4):
        api.set_option("trace_variant", variant)
        try:
            for stats in (False, True):
                for x in (b, g, c):
                    x.set_stats(stats)
                traced = check_walk(b, o.intersect, finite_rd(rays), f"BVH {fam} tv{variant}")
                check_walk(g, o.intersect, finite_rd(rays), f"BVH_GPU {fam} tv{variant}")
                check_walk(c, cw.intersect, rays, f"CWBVH {fam} tv{variant}")
                # any-hit with tmax exactly at the closest hit: BVH::IsOccluded on the BVH layouts, and on the CWBVH wherever the
                # reference's own CWBVH query (Intersect, then t < tmax) agrees with it
                sh = util.shadow_at_hits(traced)
                if sh.shape[0]:
                    want = o.occluded(sh)
                    assert np.array_equal(b.IsOccluded(sh), want) and np.array_equal(g.IsOccluded(sh), want), f"{fam}: occlusion bits"
                    # the CWBVH layout: BVH8_CWBVH::IsOccluded is FALLBACK_SHADOW_QUERY (tiny_bvh.h:312), Intersect of the same bytes and
                    # then t < tmax - a triangle exactly at tmax does not occlude there, where BVH::IsOccluded (t <= tmax) says it does
                    tr = sh.copy()
                    cw.intersect(tr)
                    occ_want = tr["t"] < sh["t"]
                    got = occlusion_bits(sh, c.IsOccluded(sh))
                    bad = np.nonzero(got != occ_want)[0]
                    assert bad.size == 0, f"{fam}: {bad.size} CWBVH occlusion bits differ, first: engine {got[bad[0]]} " \
                        f"CWBVH t {tr['t'][bad[0]]!r} prim {tr['prim'][bad[0]]} ray {sh[bad[0]][['O', 'D', 'rD', 't', 'prim']]}"
                    edge_rays += int((occ_want != occlusion_bits(sh, want)).sum())
        finally:
            api.set_option("trace_variant", 3)
            for x in (b, g, c):
                x.set_stats(False)
    if (fam, ntris) in EDGE_CASES:
        assert edge_rays > 0, "no shadow ray ended exactly on a CWBVH hit"


@pytest.mark.parametrize("k", [-4, 8, 16])
@pytest.mark.parametrize("builder", list(BUILDERS))
def test_engine_is_scale_invariant_inside_the_window(gpu, builder, k):
    """Without any oracle: at 2^k the engine builds the same tree with every bound times 2^k, and its hits keep prim, u and v
    with t times 2^k exactly (the restatement does the same there, tests/test_offatrium.py)."""
    base = scenes.procedural_scene(6000, 7)
    e0, e1 = engine_tree(base, builder), engine_tree(util.scaled(base, k), builder)
    (n0, i0), (n1, i1) = e0.download(), e1.download()
    assert np.array_equal(n0["leftFirst"], n1["leftFirst"]) and np.array_equal(n0["triCount"], n1["triCount"]) and np.array_equal(i0, i1)
    for f in ("aabbMin", "aabbMax"):
        assert np.array_equal(np.ldexp(n0[f], k).view(np.uint32), n1[f].view(np.uint32)), f
    r0 = unit_rays("scale:0", 6000, seed=7)
    c0, c1 = api.BVH8_CWBVH(), api.BVH8_CWBVH()
    for layout in ("bvh", "cwbvh"):
        if layout == "bvh":
            a, b_ = e0, e1
        else:
            a, b_ = getattr(c0, builder if builder == "BuildHQ" else "Build")(base), getattr(c1, builder if builder == "BuildHQ" else "Build")(util.scaled(base, k))
        h0, h1 = r0.copy(), util.scaled_rays(r0, k)
        a.Intersect(h0), b_.Intersect(h1)
        assert np.array_equal(h0["prim"], h1["prim"]), layout
        hit = h0["t"] < 1e30
        assert np.array_equal(h0["u"][hit].view(np.uint32), h1["u"][hit].view(np.uint32)) and np.array_equal(h0["v"][hit].view(np.uint32), h1["v"][hit].view(np.uint32))
        assert np.array_equal(np.ldexp(h0["t"][hit], k).view(np.uint32), h1["t"][hit].view(np.uint32)), layout


# ---- long leaves and the pending-group limit --------------------------------------------------------------------------------
def long_leaf_rays(v):
    lo, hi = scenes.scene_bounds(v)
    c = (lo + hi) * np.float32(0.5)
    rng = np.random.default_rng(11)
    O = (c + (rng.random((512, 3)).astype(np.float32) - 0.5) * (hi - lo + 1) * 3).astype(np.float32)
    T = (lo + rng.random((512, 3)).astype(np.float32) * (hi - lo)).astype(np.float32)
    aim = R.make_rays(O, T - O)
    # axis rays straight down onto the triangles' plane (+z): the clusters sit at z = 0
    P = np.stack([lo[0] + (hi[0] - lo[0]) * rng.random(256), lo[1] + (hi[1] - lo[1]) * rng.random(256), np.full(256, lo[2] - 3)], 1)
    down = R.make_rays(P.astype(np.float32), np.tile(np.float32([0, 0, 1]), (256, 1)))
    return util.octant_blocks(np.concatenate([aim, down, util.axis_rays(lo, hi, 8, 5)]))


@pytest.mark.parametrize("name,depth,pending", [("identical", 33, 0), ("clusters", 143, 1), ("collapsed", 1792, 1)])
def test_long_leaf_trees_walk(gpu, name, depth, pending):
    """SplitLeafs makes a chain of 3-triangle leaves out of a long leaf: a deep wide tree that leaves almost nothing pending.  The
    walk holds at most one node group per ancestor with two inner children, so these trees walk as the reference walks them -
    uploaded and converted on the device, as a BLAS and under a TLAS."""
    v = util.long_leaf_scene(name)
    cw, _ = util.oracle_cwbvh(v, mode=2)
    assert util.cw_depth_and_pending(cw.nodes) == (depth, pending)
    rays = long_leaf_rays(v)
    up = api.BVH8_CWBVH().upload(cw.nodes, cw.tris)
    want = check_walk(up, cw.intersect, rays, name + " uploaded")
    if name == "clusters":
        assert (want["t"] < 1e30).sum() > 100
    if name == "collapsed":
        assert not (want["t"] < 1e30).any()   # Moeller-Trumbore's determinant overflows at 2^40
    c = api.BVH8_CWBVH()
    c.build_flavour = BUILD_REFERENCE
    c.Build(v)
    nodes, tris = c.download()
    diff_blob(nodes, cw.nodes, name + " bvh8Data", 80)
    check_walk(c, cw.intersect, rays, name + " converted")
    # under a TLAS of two instances (identity and a mirror), the BLAS walked in its CWBVH layout: as the oracle's composition
    from oracle import portpy
    inst = identity_instances(2)
    inst[1]["transform"] = np.diag(np.float32([-1, 1, 1, 1])).reshape(-1)
    t = api.TLAS().Build(inst, [c], blas_layout=api.LAYOUT_CWBVH)
    tn, ti = t.download()
    port = portpy.PortTLASCW(tn, ti, inst, [_CW(c)])
    want, got = rays.copy(), rays.copy()
    port.intersect(want), t.Intersect(got)
    assert np.array_equal(words(got), words(want))


def identity_instances(n):
    inst = np.zeros(n, api.BLAS_INSTANCE)
    for i in range(n):
        inst[i]["transform"] = inst[i]["invTransform"] = np.eye(4, dtype=np.float32).reshape(-1)
        inst[i]["mask"] = 0xFFFF
    return inst


def pending_chain(k):
    """Hand-encoded bvh8Data: a chain of k wide nodes, each with two inner children - the next chain node in slot 0, entered first by
    a ray into the +++ octant, and a node holding one one-triangle leaf in slot 1, left pending - so a walk down the chain holds k node
    groups at once.  Every child box is the unit cube (origin 0, exponents 0, quantised 0..1); the last leaf holds a real triangle at
    z = 0.5 (prim 7), every other leaf a degenerate one."""
    count = 2 * k + 2
    n = np.zeros((count, 80), np.uint8)
    w = n.view(np.uint32).reshape(-1, 20)
    n[:, 56:80:8] = 1                           # qhi.x, qhi.y, qhi.z of slot 0
    n[:, 57:80:8] = 1                           # ... and of slot 1
    for i in range(k):
        x = 2 * i
        w[x, 4] = x + 2                         # inner children: x + 2 (slot 0), x + 3 (slot 1)
        n[x, 24], n[x, 25] = 0x38 | 0, 0x38 | 1  # meta: inner children in slots 0 and 1 (0b001sssss, sssss = 24 + slot)
        n[x, 15] = 0b11                         # imask
    for x in list(range(3, 2 * k, 2)) + [2 * k, 2 * k + 1]:
        n[x, 24] = 0x20                         # one leaf child: one triangle at offset 0
    w[2 * k + 1, 5] = 3                         # the last leaf's triangle: record 1 (float4 units)
    tris = np.zeros((6, 4), np.float32)
    tris[3] = (0, 2, 0, 0)                      # e2
    tris[4] = (2, 0, 0, 0)                      # e1
    tris[5, :3] = (0, 0, 0.5)                   # v0
    tris[5, 3] = np.uint32(7).view(np.float32)  # prim
    return n.view(np.float32).reshape(-1, 4), tris


@pytest.mark.parametrize("k,ok", [(128, True), (129, False)])
def test_pending_limit_is_enforced(gpu, k, ok):
    """128 pending node groups is the reference's limit (tiny_bvh.h:7048): a tree that can need more is refused with
    TBVH_E_LIMIT, by the walk and by a TLAS build over it; one that needs exactly 128 is walked to its last leaf, holding 128
    groups on the way there."""
    d, t = pending_chain(k)
    assert util.cw_depth_and_pending(d)[1] == k
    e = api.BVH8_CWBVH().upload(d, t)
    rays = R.make_rays(np.float32([[0.5, 0.5, -1]] * 64), np.float32([[0, 0, 1]] * 64))
    inst = identity_instances(1)
    inst[0]["aabbMin"], inst[0]["aabbMax"] = 0, 1
    if ok:
        got = rays.copy()
        e.Intersect(got)
        assert (got["prim"] == 7).all() and (got["t"] == np.float32(1.5)).all()
        assert e.IsOccluded(rays.copy()).all()
        tl = api.TLAS().Build(inst, [e], update=False, blas_layout=api.LAYOUT_CWBVH)
        got = rays.copy()
        tl.Intersect(got)
        assert (got["prim"] == 7).all() and (got["t"] == np.float32(1.5)).all()
    else:
        with pytest.raises(api.TbvhError, match="pending"):
            e.Intersect(rays)
        with pytest.raises(api.TbvhError, match="pending"):
            api.TLAS().Build(inst, [e], update=False, blas_layout=api.LAYOUT_CWBVH)


def test_cwbvh_cycle_is_refused(gpu):
    """Uploaded bvh8Data whose inner-child links lead back to the root: a walk would never end, so it is refused before any launch."""
    d, t = pending_chain(3)
    n = d.view(np.uint8).reshape(-1, 80)
    n[6, 24], n[6, 15] = 0x38, 1                 # the first leaf holder of the last chain node becomes an inner node ...
    n.view(np.uint32).reshape(-1, 20)[6, 4] = 0  # ... whose child is the root
    e = api.BVH8_CWBVH().upload(d, t)
    with pytest.raises(api.TbvhError, match="cycle"):
        e.Intersect(R.make_rays(np.float32([[0.5, 0.5, -1]]), np.float32([[0, 0, 1]])))


# ---- refits at the family's own scale -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("fam", ["zero:random", "zero:order", "scale:-100", "scale:-4", "scale:24", "shift:1048576", "shift:-12582912"])
def test_refit_layouts_match_oracle(gpu, fam):
    """BVH::Refit and the CWBVH refit over the kept collapse (tbvh_refit_layouts) after the vertices moved at the family's scale
    (the signed zeros stay): bytes as BVH::Refit and tests/cwbvh_refit_oracle.py give them, walks bit for bit."""
    from tests.test_cwbvh_refit_gpu import engine, check_bytes, check_traversal
    from tests.test_oracle_pin import moved
    v = family(fam, 2000)
    e, built = engine(v, "BVH.Build")
    w = moved(v, 7, amp=0.05)
    keep = v == 0
    w[keep] = v[keep]
    e.Refit(w)
    o, cw = check_bytes(e, built, w, fam)
    check_traversal(e, cw, unit_rays(fam, 2000), fam)
