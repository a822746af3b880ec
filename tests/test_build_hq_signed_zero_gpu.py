"""BuildHQ on inputs with signed zeros (tests/test_build_hq_signed_zero.py): the reference's tree byte for byte, so every zero bound
below the root - bins, clipped fragments, child boxes - carries the sign the reference's folds give it.  Under the settings that
change which kernel and group size builds a node, in batches next to meshes without -0, through the derived layouts and their
walks, and on the benchmark's path (the mirrored procedural scene through BVH8_CWBVH::BuildHQ)."""
import numpy as np
import pytest

from oracle import portpy
from tinybvh_b200 import api, scenes
from tests import util
from tests.test_build_batch_hq_gpu import assert_same, hq_batch, separate
from tests.test_build_hq_gpu import assert_same_hq_tree
from tests.test_build_hq_shapes_gpu import knobs  # noqa: F401 (fixture)
from tests.test_build_hq_signed_zero import FAMILIES, SIZES, compare_trees, family, family_hq, family_rays
from tests.test_offatrium_gpu import check_walk, finite_rd

pytestmark = pytest.mark.gpu

KNOBS = ["defaults", "small8", "small256", "cluster1", "cluster3", "frags1_capmax", "frags_max"]


def assert_hq(e, want, label):
    """The engine's tree against the restatement's (nodes, primIdx, idxCount); a mismatch names the first differing node and field
    and says whether the trees differ in the signs of zero bounds only."""
    nodes, idx, ic = want
    got_nodes, got_idx = e.download()
    first, signs_only = compare_trees((got_nodes, got_idx[: idx.shape[0]]), (nodes, idx))
    if first is not None:
        pytest.fail(f"{label}: {first}; " + ("everything else equal: only the signs of zero bounds differ" if signs_only
                                              else "the trees differ beyond the signs of zero bounds"))
    assert_same_hq_tree(e, nodes, idx, ic, label)


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("fam", FAMILIES)
def test_tree_matches_oracle(gpu, fam, n):
    v = family(fam, n)
    assert_hq(api.BVH().BuildHQ(v), family_hq(fam, n), f"{fam} {n}")


@pytest.mark.parametrize("n", SIZES[1:])
@pytest.mark.parametrize("fam", FAMILIES)
@pytest.mark.parametrize("knobs", KNOBS, indirect=True)
def test_tree_matches_oracle_under_knobs(gpu, knobs, fam, n):
    """The level kernel, cluster merges over distributed shared memory, one-CTA nodes and the warp subtrees."""
    v = family(fam, n)
    assert_hq(api.BVH().BuildHQ(v), family_hq(fam, n), f"{fam} {n} {knobs}")


def neighbours():
    base = scenes.procedural_scene(1500, 91)
    return [("plain", base), ("scaled", util.scaled(base, 8)), ("translated", util.translated(base, 1048576.0))]


@pytest.mark.parametrize("fam", FAMILIES)
def test_batch_positions_match_oracle(gpu, fam):
    """The family first, in the middle and last of a batch of plain, scaled and translated meshes: every tree is the reference's."""
    v = family(fam, 2000)
    others = neighbours()
    for pos in (0, 1, len(others)):
        named = others[:pos] + [(fam, v)] + others[pos:]
        got = hq_batch([m for _, m in named])
        for k, (label, m) in enumerate(named):
            assert_hq(got[k], family_hq(fam, 2000) if label == fam else portpy.build_hq(m), f"{label} at {k} of a batch with {fam} at {pos}")


def test_batch_with_one_signed_zero_mesh(gpu):
    """Only one mesh of the batch has a -0: the batch runs the sign pass for every tree, and each comes out as its own separate
    build and as the reference's."""
    named = neighbours() + [("straddle", family("straddle", 2000))] + [("plain 2", scenes.procedural_scene(700, 92))]
    meshes = [m for _, m in named]
    assert [util.count_neg_zero(m[:, :3]) > 0 for m in meshes] == [False, False, False, True, False]
    got = hq_batch(meshes)
    for k, (label, m) in enumerate(named):
        assert_hq(got[k], portpy.build_hq(m), label)
    assert_same(got, separate(meshes), "a batch with one signed-zero mesh")


@pytest.mark.parametrize("fam", [f for f in FAMILIES if f != "zero:pos"])
def test_derived_layouts_and_walks(gpu, fam):
    """BVH_GPU::BuildHQ and BVH8_CWBVH::BuildHQ bytes as the reference converts its SBVH; the BVH, BVH_GPU and CWBVH walks bit for bit
    on rays whose axis rays start on the zero planes."""
    v = family(fam, 2000)
    o = util.oracle_tree(v, 2)
    b = api.BVH().BuildHQ(v)
    assert_hq(b, family_hq(fam, 2000), fam)
    g = api.BVH_GPU().BuildHQ(v)
    want = util.oracle_bvh_gpu_nodes(o)
    got = g.download()
    assert got.shape == want.shape and np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"{fam}: BVH_GPU nodes differ"
    cw, used = util.oracle_cwbvh(v, mode=1)
    c = api.BVH8_CWBVH().BuildHQ(v)
    d8, t8 = c.download()
    assert d8.shape == cw.nodes.shape and np.array_equal(d8.view(np.uint32), cw.nodes.view(np.uint32)), f"{fam}: bvh8Data differs"
    assert t8.shape[0] >= used and np.array_equal(t8[:used].view(np.uint32), cw.tris[:used].view(np.uint32)), f"{fam}: bvh8Tris differs"
    rays = family_rays(v)
    check_walk(b, o.intersect, finite_rd(rays), f"BVH {fam}")
    check_walk(g, o.intersect, finite_rd(rays), f"BVH_GPU {fam}")
    check_walk(c, cw.intersect, rays, f"CWBVH {fam}")


def test_bench_path_on_the_mirrored_scene(gpu):
    """The benchmark's builder and layout on its scene mirrored through the origin (2,000+ floor zeros turned -0): BVH8_CWBVH::BuildHQ
    at 150,000 triangles, bytes and walk as the reference's."""
    v = np.array(scenes.procedural_scene(150000, 11), np.float32)
    v[:, :3] *= -1
    assert util.count_neg_zero(v[:, :3]) > 0
    cw, used = util.oracle_cwbvh(v, mode=1)
    c = api.BVH8_CWBVH().BuildHQ(v)
    d8, t8 = c.download()
    assert d8.shape == cw.nodes.shape and np.array_equal(d8.view(np.uint32), cw.nodes.view(np.uint32)), "bvh8Data differs"
    assert t8.shape[0] >= used and np.array_equal(t8[:used].view(np.uint32), cw.tris[:used].view(np.uint32)), "bvh8Tris differs"
    check_walk(c, cw.intersect, family_rays(v, res=64), "CWBVH mirrored 150k")
