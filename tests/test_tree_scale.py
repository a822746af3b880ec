"""The two tree producers the engine defines itself - tbvh_optimize (tests/optimize_oracle.c) and TBVH_BUILD_PLOC (tests/ploc_oracle.c) -
off the unit scale, against anchors neither restatement defines: a tree scaled by an exact 2^k must optimise, and a mesh scaled by 2^k
must cluster, to the unit-scale result times 2^k bit for bit inside a window of k that is pinned here per scene; outside it the
results are well formed and what they are is asserted.  Signed-zero twins give the +0 twin's tree up to the signs of zero bounds;
translated and rebuilt far scenes never raise SAHCost and keep their walks' hits.  DESIGN.md §4.7 and §4.8 state the windows."""
import functools

import numpy as np
import pytest

from oracle import portpy
from tinybvh_b200 import scenes
from tests import util
from tests import optimize_oracle as oo
from tests import ploc_oracle as po
from tests.test_optimize import check_result, leaf_records, sah

ZERO = ["zero:neg", "zero:random", "zero:order"]
SHIFT = ["shift:1048576", "shift:-12582912"]   # +2^20, -3 * 2^22
ROUNDS = 6

# tbvh_optimize of the unit-scale source tree (procedural_scene(n, 5)) with every box scaled by 2^k: (lowest, highest) k whose result
# is the unit-scale result times 2^k with the same rounds and per-round SAHCost bits.  Below, the areas of the smallest boxes are
# subnormal (below 2^-126, with fewer significant bits) and some comparisons of the search, the gains or the acceptance go the other
# way: a different tree, still well formed and cheaper than its input.  Above, the SAH sum overflows: SAHCost is inf (the sum) or NaN
# (inf / inf, the root's area too), no round can be strictly cheaper, and the input is returned unchanged after 0 rounds.
OPT_WINDOW = {
    (40, "src"): (-67, 56), (40, "B"): (-66, 56), (40, "DB"): (-66, 56),
    (2000, "src"): (-65, 55), (2000, "B"): (-65, 54), (2000, "DB"): (-65, 54),
    (70000, "src"): (-58, 54),
}
OPT_WINDOW_OWN = {("BuildAVX", 2000, "src"): (-64, 55), ("BuildHQ", 2000, "src"): (-64, 55)}   # where a builder's tree has its own window
# the family scales of tests/test_offatrium_gpu.py and two more: 2^-30 and 2^60
KS = [-126, -100, -60, -30, -6, -4, 8, 16, 24, 30, 40, 60, 90]

# TBVH_BUILD_PLOC of procedural_scene(n, 5) scaled by 2^k: (lowest, highest) k of the run of scales around 1 whose tree is the unit tree
# times 2^k.  Below, fragment and cluster areas underflow (subnormal, then 0), the keys tie and the tie rule and the leaf collapse
# decide otherwise; above, half_area overflows to inf.  At 2^-126, 2^-100 and 2^90 every area is 0 (or inf) beside every other, so
# every leaf cost ties its interior cost and each 4-triangle subtree the clustering leaves collapses (leaf cost <= interior cost).
PLOC_WINDOW = {3: (-73, 59), 40: (-71, 58), 2000: (-64, 57), 70000: (-61, 58)}
# what the restatement leaves outside the window at n = 2000: node count of the tree, SAHCost NaN
PLOC_OUTSIDE_2000 = {-126: 1000, -100: 1000, 60: 2012, 90: 1000}


@functools.lru_cache(maxsize=None)
def unit_scene(n):
    return scenes.procedural_scene(n, 5)


@functools.lru_cache(maxsize=None)
def unit_tree(n, builder, fam):
    src = util.source_tree(unit_scene(n), builder)
    return src if fam == "src" else util.family_tree(src, fam, 5)


@functools.lru_cache(maxsize=None)
def unit_optimized(n, builder, fam):
    t = unit_tree(n, builder, fam)
    return oo.optimize(t[0], t[1], ROUNDS)


def scale_nodes(nodes, k):
    """Every box bound times 2^k (exact while the bound stays normal)."""
    out = nodes.copy()
    with np.errstate(over="ignore"):
        for f in ("aabbMin", "aabbMax"):
            out[f] = np.ldexp(out[f], k).astype(np.float32)
    return out


def is_scaled(a, b, k):
    """b is a with the same topology and every bound times 2^k, bit for bit."""
    if a.shape != b.shape or not (np.array_equal(a["leftFirst"], b["leftFirst"]) and np.array_equal(a["triCount"], b["triCount"])):
        return False
    return all(np.array_equal(util.bits_u32(scale_nodes(a, k)[f]), util.bits_u32(b[f])) for f in ("aabbMin", "aabbMax"))


def f32_bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


def opt_window(n, builder, fam):
    return OPT_WINDOW_OWN.get((builder, n, fam), OPT_WINDOW[(n, fam)])


def opt_cases():
    out = []
    for (n, fam), (lo, hi) in OPT_WINDOW.items():
        builders = ["Build", "BuildHQ"] if n == 70000 else ["Build", "BuildAVX", "BuildHQ"]
        # at 70,000 triangles the scales just below the window are left out: the rounds there spend minutes in subnormal arithmetic
        ks = {lo, hi, hi + 1, -126, 90} if n == 70000 else set(KS) | {lo - 1, lo, hi, hi + 1}
        for b in builders:
            own = OPT_WINDOW_OWN.get((b, n, fam), (lo, hi))
            out += [(n, b, fam, k) for k in sorted(ks | ({own[0] - 1, own[0], own[1], own[1] + 1} if n < 70000 else set()))]
    return out


# ---- tbvh_optimize: scale equivariance of the rounds, isolated from the builders ---------------------------------------------
@pytest.mark.parametrize("n,builder,fam,k", opt_cases(), ids=[f"{n}-{b}-{f}-2^{k}" for n, b, f, k in opt_cases()])
def test_optimize_scale_window(n, builder, fam, k):
    """The unit-scale source tree with every box times 2^k (the reference builder's own window - it builds a 4-node Build tree at
    2^40 - stays out of the way).  Inside the window: the unit result times 2^k, the same rounds and per-round SAHCost bits."""
    t = unit_tree(n, builder, fam)
    want, wr, wsah, wper = unit_optimized(n, builder, fam)
    src = scale_nodes(t[0], k)
    out, rounds, final, per = oo.optimize(src, t[1], ROUNDS)
    lo, hi = opt_window(n, builder, fam)
    inside = is_scaled(want, out, k) and rounds == wr and np.array_equal(f32_bits(per), f32_bits(wper)) and f32_bits(final) == f32_bits(wsah)
    assert inside == (lo <= k <= hi), f"2^{k} is {'inside' if lo <= k <= hi else 'outside'} the window [{lo}, {hi}]"
    if inside:
        return
    if k > hi:   # the SAH sum overflows: no round is strictly cheaper than inf, and nothing is cheaper than NaN
        assert not np.isfinite(final) and rounds == 0
    if not np.isfinite(final):
        assert rounds == 0
    if rounds == 0:
        assert out.tobytes() == src.tobytes(), "0 rounds: the input unchanged"
    else:
        check_result((src, t[1], t[2]), out, rounds, final, per, n)


@pytest.mark.parametrize("builder", ["Build", "BuildAVX", "BuildHQ"])
def test_optimize_at_2_to_minus_60_is_the_builders_window(builder):
    """At 2^-60 the optimised result of a rebuilt 2,000-triangle scene is not the unit result times 2^-60: the reference builder's
    own tree already differs there (small boxes' areas are subnormal in its SAH), while the optimiser over the unit tree scaled
    by 2^-60 is exact (test_optimize_scale_window)."""
    v = unit_scene(2000)
    rebuilt = util.source_tree(util.scaled(v, -60), builder)
    assert not is_scaled(unit_tree(2000, builder, "src")[0], rebuilt[0], -60), "the builder's tree at 2^-60"
    t = unit_tree(2000, builder, "src")
    assert is_scaled(unit_optimized(2000, builder, "src")[0], oo.optimize(scale_nodes(t[0], -60), t[1], ROUNDS)[0], -60)


# ---- PLOC: scale equivariance of the build ---------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def ploc_unit(n):
    return po.build(unit_scene(n))


def ploc_cases():
    out = []
    for n, (lo, hi) in PLOC_WINDOW.items():
        ks = {lo - 1, lo, hi, hi + 1, -126, 90} if n == 70000 else set(KS) | {lo - 1, lo, hi, hi + 1}
        out += [(n, k) for k in sorted(ks)]
    return out


@pytest.mark.parametrize("n,k", ploc_cases(), ids=[f"{n}-2^{k}" for n, k in ploc_cases()])
def test_ploc_scale_window(n, k):
    base = ploc_unit(n)
    v = util.scaled(unit_scene(n), k)
    nodes, idx, iters, cost = po.build(v)
    lo, hi = PLOC_WINDOW[n]
    inside = is_scaled(base[0], nodes, k) and np.array_equal(idx, base[1])
    assert inside == (lo <= k <= hi), f"2^{k} is {'inside' if lo <= k <= hi else 'outside'} the window [{lo}, {hi}]"
    util.check_tree((nodes, idx, n), n)
    assert np.array_equal(np.sort(idx), np.arange(n)), "every triangle exactly once"
    assert nodes.shape[0] == 2 + 2 * (util.dfs_leaves(nodes).size - 1)
    assert (nodes["triCount"][util.dfs_leaves(nodes)] <= 4).all()
    assert f32_bits(sah(nodes)) == f32_bits(cost) or (np.isnan(cost) and np.isnan(sah(nodes)))
    if inside:
        assert iters == base[2]   # SAHCost may already be inf at the top of the window: its sum overflows before the tree changes
    if n == 2000 and k in PLOC_OUTSIDE_2000:
        assert nodes.shape[0] == PLOC_OUTSIDE_2000[k] and np.isnan(cost)
    if k in (-126, -100, 90):
        # every area ties (0 or inf): the tree is collapsed into leaves of 4 triangles as far as the clustering allows
        assert np.isnan(cost) and nodes.shape[0] == 2 + 2 * ((n + 3) // 4 - 1)


# ---- signed-zero twins ------------------------------------------------------------------------------------------------------
def twin_of(v, mode):
    return util.signed_zero(v, mode, 5)


def same_up_to_zero_signs(a, b, ai, bi):
    assert np.array_equal(a["leftFirst"], b["leftFirst"]) and np.array_equal(a["triCount"], b["triCount"]), "topology"
    assert np.array_equal(ai, bi), "primIdx"
    for f in ("aabbMin", "aabbMax"):
        assert np.array_equal(util.bits_u32(a[f] + np.float32(0)), util.bits_u32(b[f] + np.float32(0))), f


@pytest.mark.parametrize("n", [40, 2000])
@pytest.mark.parametrize("mode", ["neg", "random", "order"])
@pytest.mark.parametrize("builder", ["Build", "BuildAVX", "BuildHQ"])
def test_optimize_signed_zero_twins(builder, mode, n):
    """The -0 twin's source tree optimises to the +0 twin's result up to the signs of zero bounds; -0 leaf bounds are kept."""
    base = unit_scene(n)
    pos, neg = util.source_tree(twin_of(base, "pos"), builder), util.source_tree(twin_of(base, mode), builder)
    same_up_to_zero_signs(pos[0], neg[0], pos[1], neg[1])
    a, b = oo.optimize(pos[0], pos[1], ROUNDS), oo.optimize(neg[0], neg[1], ROUNDS)
    assert a[1] == b[1] and f32_bits(a[2]) == f32_bits(b[2]) and np.array_equal(f32_bits(a[3]), f32_bits(b[3]))
    same_up_to_zero_signs(a[0], b[0], pos[1], neg[1])
    check_result(neg, b[0], b[1], b[2], b[3], n)
    boxes = lambda x: np.concatenate([x["aabbMin"], x["aabbMax"]])
    assert util.count_neg_zero(boxes(neg[0])) > 0 and util.count_neg_zero(boxes(b[0])) > 0, "a -0 bound survives"
    assert util.count_neg_zero(boxes(a[0])) == 0


@pytest.mark.parametrize("n", [40, 2000, 70000])
@pytest.mark.parametrize("mode", ["neg", "random", "order"])
def test_ploc_signed_zero_twins(mode, n):
    base = unit_scene(n)
    a, b = po.build(twin_of(base, "pos")), po.build(twin_of(base, mode))
    same_up_to_zero_signs(a[0], b[0], a[1], b[1])
    assert a[2] == b[2] and f32_bits(a[3]) == f32_bits(b[3])
    boxes = lambda x: np.concatenate([x["aabbMin"], x["aabbMax"]])
    assert util.count_neg_zero(boxes(b[0])) > 0 and util.count_neg_zero(boxes(a[0])) == 0, "a -0 bound survives"


# ---- translated and rebuilt far scenes: tbvh_optimize never raises SAHCost and keeps the walks' hits ----------------------------
FAR = SHIFT + ["scale:-126", "scale:-100", "scale:-60", "scale:40", "scale:60", "scale:90"]


@pytest.mark.parametrize("n", [40, 2000])
@pytest.mark.parametrize("fam", FAR)
@pytest.mark.parametrize("builder", ["Build", "BuildAVX", "BuildHQ"])
def test_optimize_far_scenes(builder, fam, n):
    v = util.family(fam, n)
    tree = util.source_tree(v, builder)
    out, rounds, final, per = oo.optimize(tree[0], tree[1], ROUNDS)
    before = sah(tree[0])
    if np.isnan(final) or np.isnan(before):
        assert rounds == 0 and np.isnan(final), "a NaN SAHCost: 0 rounds"
    if rounds == 0:   # the input as it came (a builder's tree at 2^40 need not hold refolded boxes)
        assert out.tobytes() == tree[0].tobytes() and f32_bits(final) == f32_bits(before) or np.isnan(final) and np.isnan(before)
        return
    check_result(tree, out, rounds, final, per, n)
    assert np.isfinite(before) and final < before
    rays = util.unit_rays(fam, n)
    rays = rays[np.isfinite(rays["rD"]).all(1)]   # the BVH2 walk's rD is finite (DESIGN 4.1)
    a, b = portpy.PortBVH(v, nodes=tree[0], prim_idx=tree[1]), portpy.PortBVH(v, nodes=out, prim_idx=tree[1])
    want, got = rays.copy(), rays.copy()
    a.intersect(want), b.intersect(got)
    bad = np.nonzero(util.bits_u32(util.nan_canonical(got)["t"]) != util.bits_u32(util.nan_canonical(want)["t"]))[0]
    if fam != "shift:-12582912":
        assert bad.size == 0
    # At -3 x 2^22 the float spacing is 1: Moeller-Trumbore's t can lie outside its leaf's box interval, and whether the walk still
    # enters that leaf depends on the t it holds by then, so on the visiting order.  Both answers are then hits of their triangles.
    assert bad.size <= rays.shape[0] // 1000
    vt = v.reshape(-1, 3, 4)
    for r in (want, got):
        for i in bad:
            p = int(r["prim"][i])
            ok, t, _, _ = portpy.tri_test(rays["O"][i], rays["D"][i], vt[p, 0, :3], vt[p, 1, :3], vt[p, 2, :3], 1e30)
            assert ok and np.float32(t).view(np.uint32) == r["t"][i].view(np.uint32)
    assert np.array_equal(b.occluded(rays.copy()), a.occluded(rays.copy()))
    sh = util.shadow_at_hits(want)
    if sh.shape[0]:
        assert np.array_equal(b.occluded(sh.copy()), a.occluded(sh.copy()))
    assert leaf_records(out) == leaf_records(tree[0])
