"""The tree families of tests/util.py (swapped, reinserted, shuffled_ranges, their BFS renumbering) are what they claim: valid BVH2s
over the same triangles whose leaf ranges are out of DFS order, walked by the restatement exactly like the builder's tree."""
import numpy as np
import pytest

from oracle import portpy, refpy
from tinybvh_b200 import scenes
from tests import util

BUILDERS = ["Build", "BuildAVX", "BuildHQ"]
SIZES = [2, 5, 3000]


def case(builder, ntris, seed=31):
    v = scenes.procedural_scene(ntris, seed)
    return v, util.source_tree(v, builder)


@pytest.mark.parametrize("ntris", SIZES)
@pytest.mark.parametrize("builder", BUILDERS)
def test_builder_trees_are_in_dfs_leaf_order(builder, ntris):
    """The premise: every builder's tree has its leaf ranges in DFS order."""
    v, t = case(builder, ntris)
    util.check_tree(t, ntris)
    assert util.leaf_order_is_dfs(t[0])


@pytest.mark.parametrize("fam", util.FAMILIES)
@pytest.mark.parametrize("ntris", SIZES)
@pytest.mark.parametrize("builder", BUILDERS)
def test_family_is_a_valid_tree_out_of_leaf_order(builder, ntris, fam):
    v, src = case(builder, ntris)
    t = util.family_tree(src, fam, 5)
    depth = util.check_tree(t, ntris)
    assert depth < 64
    if fam not in ("B", "DB"):
        assert depth == util.tree_depth(src[0])
    nleaves = util.dfs_leaves(src[0]).size
    if nleaves > 1:
        assert not util.leaf_order_is_dfs(t[0]), "firstTri still grows along the DFS leaf order"
    if fam.startswith("D") and ntris >= 3000:
        base = util.family_tree(src, {"DA": "A0.3", "DB": "B", "DC": "C3"}[fam], 5)
        assert not np.array_equal(t[0].view(np.uint32), base[0].view(np.uint32)), "the BFS numbering differs from the DFS one"
    if fam in ("C3", "DC") and nleaves > 1:
        assert t[2] > int(t[0]["triCount"][util.dfs_leaves(t[0])].sum()), "gaps between the blocks"
    # the same multiset of primitive references in the leaves
    refs = lambda tr: np.sort(np.concatenate([tr[1][f:f + c] for f, c in zip(tr[0]["leftFirst"][util.dfs_leaves(tr[0])], tr[0]["triCount"][util.dfs_leaves(tr[0])])]))
    assert np.array_equal(refs(t), refs(src))


def test_swapped_mirror_reverses_the_leaf_order():
    v, src = case("Build", 3000)
    t = util.swapped(src, 0, 1.0)
    a, b = util.dfs_leaves(src[0]), util.dfs_leaves(t[0])
    assert np.array_equal(src[0]["leftFirst"][a], t[0]["leftFirst"][b][::-1])


@pytest.mark.parametrize("builder", ["Build", "BuildHQ"])
def test_reinserted_deep_tree(builder):
    """The one family member 64..255 levels deep (the 256-entry walk)."""
    v, src = case(builder, 3000)
    t = util.reinserted(src, 7, 50, grow_to=100)
    assert util.check_tree(t, 3000) == 100
    assert not util.leaf_order_is_dfs(t[0])


def walk_equal(v, src, t, label):
    sets, bounds = util.ray_sets(v, res=40)
    r = sets["primary"]
    a = portpy.PortBVH(v, nodes=src[0], prim_idx=src[1])
    b = portpy.PortBVH(v, nodes=t[0], prim_idx=t[1])
    want, got = a.intersect(r.copy()), b.intersect(r.copy())
    more = util.derived_sets(want, v, bounds)
    for name, rays in [("primary", r)] + list(more.items()):
        want, got = a.intersect(rays.copy()), b.intersect(rays.copy())
        assert np.array_equal(util.bits_u32(got["t"]), util.bits_u32(want["t"])), f"{label} {name}: t differs"
        assert util.classify_mismatches(got, want, v)["real"] == 0, f"{label} {name}: a different prim without a tie on t"
        assert np.array_equal(b.occluded(rays.copy()), a.occluded(rays.copy())), f"{label} {name}: occlusion differs"


@pytest.mark.parametrize("fam", util.FAMILIES)
@pytest.mark.parametrize("ntris", [5, 3000])
@pytest.mark.parametrize("builder", BUILDERS)
def test_family_walks_like_its_source(builder, ntris, fam):
    """The restatement's walk of the family tree: t bit for bit that of the builder's tree on every ray; prim differs only on ties."""
    v, src = case(builder, ntris)
    walk_equal(v, src, util.family_tree(src, fam, 5), f"{builder} {ntris} {fam}")


@pytest.mark.parametrize("fam", ["B", "C3", "DB"])
def test_family_walks_like_its_source_120k(fam):
    v, src = case("BuildAVX", 120000)
    t = util.family_tree(src, fam, 6)
    assert util.check_tree(t, 120000) < 64
    walk_equal(v, src, t, f"BuildAVX 120000 {fam}")


def test_deep_family_walks_like_its_source():
    v, src = case("Build", 3000)
    walk_equal(v, src, util.reinserted(src, 7, 50, grow_to=100), "Build 3000 deep")


if refpy.available():   # BVH::Optimize exists in the reference only
    @pytest.mark.parametrize("ntris", [5, 3000, 30000])
    def test_reference_optimize_leaves_leaf_ranges_out_of_dfs_order(ntris):
        """The reference's BVH::Optimize output is a tree of the kind the families model: valid, children behind their parent, leaf
        ranges out of DFS order; the restatement walks it like the tree it started from."""
        v = scenes.procedural_scene(ntris, 71 + ntris % 7)
        t = util.optimized_tree(v)
        util.check_tree(t, ntris)
        if util.dfs_leaves(t[0]).size > 2:
            assert not util.leaf_order_is_dfs(t[0])
        walk_equal(v, util.source_tree(v, "Build"), t, f"Optimize {ntris}")
