"""The host restatement of tbvh_optimize (tests/optimize_oracle.c) against its anchors: the reference's SAHCost never rises, the tree
stays a valid BVH2 over the same leaves, and walks find what they found on the tree before optimisation."""
import os

import numpy as np
import pytest

from oracle import portpy
from tinybvh_b200 import scenes
from tests import golden_util, util
from tests import optimize_oracle as oo

BUILDERS = ["Build", "BuildAVX", "BuildHQ"]


def _scenes():
    out = {os.path.basename(p)[:-4]: golden_util.load(p)["verts"] for p in golden_util.golden_files()}
    out["seeded_6000"] = scenes.procedural_scene(6000, 11)
    return out


SCENES = _scenes()


def sah(nodes):
    return np.float32(portpy.lib().orc_sah_cost(np.ascontiguousarray(nodes).ctypes.data, 0, 1.0, 1.0))


def leaf_records(nodes):
    leaves = util.dfs_leaves(nodes)
    return sorted(nodes[leaves].tobytes()[i * 32:(i + 1) * 32] for i in range(leaves.size))


def check_result(tree, out, rounds, final, per, ntris):
    nodes, idx, ic = tree
    depth = util.check_tree((out, idx, ic), ntris)
    assert depth <= max(util.tree_depth(nodes), 63)
    assert leaf_records(out) == leaf_records(nodes), "leaves keep firstTri, triCount and box bits"
    assert per.shape[0] == rounds and (np.diff(per) < 0).all()
    if rounds:
        assert per[0] < sah(util.refold_boxes(nodes.copy()))
        assert out.shape[0] == 2 + 2 * (util.dfs_leaves(out).size - 1), "used_nodes = 2 + 2 x interior nodes"
        assert per[-1] == final
    else:
        assert out.tobytes() == nodes.tobytes()
    assert sah(out) == final


def test_four_leaf_swap():
    """((A, C), (B, D)) with A near B and C near D becomes ((A, B), (C, D)).  No single reinsertion does that, and the two that
    do share nodes (P, S, G), so they are not taken in one round: the first round makes ((A, B), C), D), the second pairs C with D."""
    nodes = np.zeros(8, portpy.NODE32)
    lo = {"A": 0.0, "B": 0.25, "C": 10.0, "D": 10.25}
    for slot, (name, first) in zip((4, 5, 6, 7), (("A", 0), ("C", 1), ("B", 2), ("D", 3))):
        nodes[slot]["aabbMin"], nodes[slot]["aabbMax"] = lo[name], lo[name] + 1.0
        nodes[slot]["leftFirst"], nodes[slot]["triCount"] = first, 1
    nodes[0]["leftFirst"], nodes[2]["leftFirst"], nodes[3]["leftFirst"] = 2, 4, 6
    util.refold_boxes(nodes)
    one = oo.optimize(nodes, np.arange(4, dtype=np.uint32), 1)
    assert one[1] == 1 and util.tree_depth(one[0]) == 3
    out, rounds, final, per = oo.optimize(nodes, np.arange(4, dtype=np.uint32), 8)
    assert rounds == 2 and out.shape[0] == 8
    pairs = [{int(out[c]["leftFirst"]), int(out[c + 1]["leftFirst"])} for c in (int(out[2]["leftFirst"]), int(out[3]["leftFirst"]))]
    assert sorted(map(sorted, pairs)) == [[0, 2], [1, 3]]
    assert final < sah(nodes)


@pytest.mark.parametrize("builder", BUILDERS)
@pytest.mark.parametrize("scene", sorted(SCENES))
def test_builder_trees(scene, builder):
    v = SCENES[scene]
    tree = util.source_tree(v, builder)
    out, rounds, final, per = oo.optimize(tree[0], tree[1], 8)
    check_result(tree, out, rounds, final, per, v.shape[0] // 3)
    assert final <= sah(tree[0])
    again = oo.optimize(tree[0], tree[1], 8)
    assert again[0].tobytes() == out.tobytes() and again[1:3] == (rounds, final)


@pytest.mark.parametrize("fam", util.FAMILIES)
@pytest.mark.parametrize("builder", BUILDERS)
def test_family_trees(builder, fam):
    v = SCENES["atrium_3k"]
    src = util.source_tree(v, builder)
    tree = util.family_tree(src, fam, 5)
    out, rounds, final, per = oo.optimize(tree[0], tree[1], 6)
    check_result(tree, out, rounds, final, per, v.shape[0] // 3)
    if fam in ("B", "DB"):
        assert rounds > 0 and final < sah(tree[0]), "a randomly reinserted tree ends below its input cost"


@pytest.mark.parametrize("kind", ["scaled", "translated"])
@pytest.mark.parametrize("builder", BUILDERS)
def test_far_scenes(builder, kind):
    """Huge coordinates (areas overflow to inf) and a scene far off the atrium: better or unchanged, never worse or malformed."""
    v = SCENES["atrium_3k"]
    v = util.scaled(v, 90) if kind == "scaled" else util.translated(v, np.float32(3.0e6))
    tree = util.source_tree(v, builder)
    out, rounds, final, per = oo.optimize(tree[0], tree[1], 4)
    if rounds == 0:
        assert out.tobytes() == tree[0].tobytes()
        return
    check_result(tree, out, rounds, final, per, v.shape[0] // 3)
    before = sah(tree[0])
    assert final < before or not np.isfinite(before)


@pytest.mark.parametrize("builder", BUILDERS)
def test_walks_keep_their_hits(builder):
    """The same triangles under boxes that still contain their children: the closest t and the occlusion bits cannot change."""
    v = SCENES["seeded_6000"]
    nodes, idx, ic = util.source_tree(v, builder)
    out, rounds, final, per = oo.optimize(nodes, idx, 8)
    assert rounds > 0
    sets, bounds = util.ray_sets(v, res=48)
    a = portpy.PortBVH(v, nodes=nodes, prim_idx=idx)
    b = portpy.PortBVH(v, nodes=out, prim_idx=idx)
    want, got = sets["primary"].copy(), sets["primary"].copy()
    a.intersect(want), b.intersect(got)
    assert np.array_equal(util.bits_u32(got["t"]), util.bits_u32(want["t"]))
    tie = got["prim"] != want["prim"]
    assert not tie.any() or (util.classify_mismatches(got, want, v)["real"] == 0)
    for name, r in util.derived_sets(want, v, bounds).items():
        w, g = r.copy(), r.copy()
        a.intersect(w), b.intersect(g)
        assert np.array_equal(util.bits_u32(g["t"]), util.bits_u32(w["t"])), name
        assert np.array_equal(b.occluded(r.copy()), a.occluded(r.copy())), name
