"""What the off-atrium GPU tests (tests/test_offatrium_gpu.py) rely on, pinned on the CPU with the plain-C restatement: its
scale-invariance window, the fold-order dependence of signed zeros, and that every input family produces what it claims."""
import numpy as np
import pytest

from oracle import portpy
from tinybvh_b200 import scenes
from tests import util


def port_tree(v, mode):
    if mode == 2:
        nodes, idx, _ = portpy.build_hq(v)
        return portpy.PortBVH(v, nodes=nodes, prim_idx=idx)
    return portpy.PortBVH(v, avx=mode == 1)


@pytest.mark.parametrize("k", [-20, -4, 8, 16, 36])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_restatement_is_scale_invariant_inside_the_window(mode, k):
    """Scaling by 2^k inside the window changes nothing but the bounds (times 2^k); for k in [-4, 16] the hits keep prim, u, v and
    t scales by exactly 2^k, in the BVH and the CWBVH walk."""
    base = scenes.procedural_scene(6000, 7)
    v = util.scaled(base, k)
    a, b = port_tree(base, mode), port_tree(v, mode)
    assert np.array_equal(a.nodes["leftFirst"], b.nodes["leftFirst"]) and np.array_equal(a.nodes["triCount"], b.nodes["triCount"])
    assert np.array_equal(a.prim_idx, b.prim_idx)
    for f in ("aabbMin", "aabbMax"):
        assert np.array_equal(np.ldexp(a.nodes[f], k).view(np.uint32), b.nodes[f].view(np.uint32))
    if not -4 <= k <= 16:
        return
    r = util.ray_sets(base, res=32)[0]["primary"]
    walks = [(a.intersect, b.intersect)]
    if mode != 1:
        walks.append((util.oracle_cwbvh(base, mode={0: 2, 2: 1}[mode])[0].intersect, util.oracle_cwbvh(v, mode={0: 2, 2: 1}[mode])[0].intersect))
    for wa, wb in walks:
        h0, h1 = r.copy(), util.scaled_rays(r, k)
        wa(h0), wb(h1)
        hit = h0["t"] < 1e30
        assert hit.sum() > 1000 and np.array_equal(h0["prim"], h1["prim"])
        assert np.array_equal(h0["u"][hit].view(np.uint32), h1["u"][hit].view(np.uint32)) and np.array_equal(h0["v"][hit].view(np.uint32), h1["v"][hit].view(np.uint32))
        assert np.array_equal(np.ldexp(h0["t"][hit], k).view(np.uint32), h1["t"][hit].view(np.uint32))


def test_restatement_changes_behaviour_outside_the_window():
    """The regimes the scaled families reach: lost hits at 2^-6 (the absolute determinant threshold), exponent bytes of -128 at
    2^-126 (no ray takes the integer slab test), the collapse at 2^40 (every SAH cost overflows BVH_FAR)."""
    base = scenes.procedural_scene(6000, 7)
    r = util.ray_sets(base, res=32)[0]["primary"]
    h0, h1 = r.copy(), util.scaled_rays(r, -6)
    portpy.PortBVH(base).intersect(h0), portpy.PortBVH(util.scaled(base, -6)).intersect(h1)
    assert not np.array_equal(h0["prim"], h1["prim"])
    cw, _ = util.oracle_cwbvh(util.scaled(base, -126), mode=2)
    assert (util.cw_exponents(cw.nodes) == -128).any() and util.cw_rd_limit(cw.nodes) is None
    cw, _ = util.oracle_cwbvh(base, mode=2)
    assert util.cw_rd_limit(cw.nodes) == np.float32(2.0 ** 127)
    big = portpy.PortBVH(util.scaled(base, 40))
    assert big.used_nodes == 4 and big.nodes["triCount"].max() > 5000
    assert (big.nodes[2:]["aabbMin"] == 0).all() and (big.nodes[2:]["aabbMax"] == 0).all()   # the children get the zero boxes


@pytest.mark.parametrize("mode", [0, 1, 2])
def test_signed_zero_bound_follows_fold_order(mode):
    """tinybvh_min returns its second operand on a tie: the root's aabbMin.x is the sign of the LAST tied vertex."""
    a, b = util.zero_tri_cases()
    assert not np.signbit(port_tree(a, mode).nodes[0]["aabbMin"][0])
    assert np.signbit(port_tree(b, mode).nodes[0]["aabbMin"][0])


def test_signed_zero_families():
    base = scenes.procedural_scene(3000, 12)
    for mode in ("pos", "neg", "random", "order"):
        v = util.signed_zero(base, mode, 1)
        xyz = v[:, :3]
        zeros, neg = int((xyz == 0).sum()), util.count_neg_zero(xyz)
        assert zeros > 500
        assert neg == {"pos": 0, "neg": zeros}.get(mode, neg) and (mode in ("pos", "neg") or 0 < neg < zeros), mode
    # in a tree of the random family the sign of zero bounds varies, so fold order matters
    n = portpy.PortBVH(util.signed_zero(base, "random", 1)).nodes
    lo = n["aabbMin"][:, 1]
    assert ((lo == 0) & np.signbit(lo)).sum() > 50 and ((lo == 0) & ~np.signbit(lo)).sum() > 50


@pytest.mark.parametrize("shift", [2.0 ** 20, -3 * 2.0 ** 22])
def test_translated_family_merges_vertices(shift):
    v = util.translated(scenes.procedural_scene(2000, 5), shift)
    t = v.reshape(-1, 3, 4)[:, :, :3]
    e1, e2 = t[:, 1] - t[:, 0], t[:, 2] - t[:, 0]
    assert (np.cross(e1, e2) == 0).all(1).sum() > 0    # zero-area triangles after rounding


@pytest.mark.parametrize("name,depth,pending", [("identical", 33, 0), ("clusters", 143, 1), ("collapsed", 1792, 1)])
def test_long_leaf_families(name, depth, pending):
    cw, _ = util.oracle_cwbvh(util.long_leaf_scene(name), mode=2)
    assert util.cw_depth_and_pending(cw.nodes) == (depth, pending)


def test_axis_rays_cover_every_octant_in_uniform_and_mixed_warps():
    lo, hi = scenes.scene_bounds(scenes.procedural_scene(2000, 5))
    r = util.octant_blocks(np.concatenate([util.axis_rays(lo, hi, 8, 5), util.octant_rays(lo, hi, 40, 5)]))
    oct_ = ((r["D"][:, 0] < 0) * 4 + (r["D"][:, 1] < 0) * 2 + (r["D"][:, 2] < 0)).astype(np.int64)
    warps = [oct_[k:k + 32] for k in range(0, oct_.shape[0] - 31, 32)]
    uniform = {int(w[0]) for w in warps if (w == w[0]).all()}
    assert uniform == set(range(8)) and any((w != w[0]).any() for w in warps)
    # +-0 direction components carry the octant's sign, and rD = safercp(D) or a user-supplied +-inf
    assert util.count_neg_zero(r["D"]) > 0 and np.isinf(util.with_inf_rd(r)["rD"]).any()


def test_rd_limit_rays_straddle_the_bound():
    lo, hi = scenes.scene_bounds(scenes.procedural_scene(200, 5))
    r = util.axis_rays(lo, hi, 4, 1)
    lim = np.float32(2.0 ** 60)
    x = np.abs(util.rd_limit_rays(r, lim)["rD"][:, 0])
    for want in (lim, np.nextafter(lim, np.float32(np.inf)), np.float32(2) * lim, np.float32(np.inf)):
        assert (x == want).any()
