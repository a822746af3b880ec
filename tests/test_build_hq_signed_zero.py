"""Input families with signed zeros for BuildHQ, on the CPU.  The reference folds bounds with `a < b ? a : b`: on a tie the second
operand wins, so of several zero bounds the one folded last gives a bin, a clipped fragment or a child box its sign.  These families
put -0 and +0 bounds in every place the SBVH builder folds them: object and spatial bins, fragments clipped per bin and by the
partition, and the child boxes refolded after a spatial split.  tests/test_build_hq_signed_zero_gpu.py holds the GPU builder to the
restatement's trees on them; here the families are pinned so that those tests can fail:
  * below the root, one field carries -0 in some node and +0 in another: no fixed-sign rule gives the tree;
  * the families meant to force spatial splits reference some triangle twice;
  * the tree is the one of the same scene with every -0 replaced by +0, except for the sign bits of zero bounds: the sign never
    changes a split, a bin or a partition;
  * an input without -0 gives no -0 bound anywhere, which is what lets the GPU builder skip the sign pass on it."""
import functools

import numpy as np
import pytest

from oracle import portpy, refpy
from tinybvh_b200 import scenes
from tests import util
from tests.test_build_hq_shapes import FAIL_SCENES, fail_scene, fail_scene_hq

SIZES = [40, 2000, 70000]
ZERO = ["zero:pos", "zero:neg", "zero:random", "zero:order"]
FAMILIES = ZERO + ["mirror:xyz", "mirror:x", "flat", "straddle"]
NEG_FAMILIES = [f for f in FAMILIES if f != "zero:pos"]
# a single-axis mirror turns that axis's zeros into -0 only; +0 bounds there come from clipping at some sizes, not at all
BOTH_SIGNS = [f for f in NEG_FAMILIES if f != "mirror:x"]
BOUNDS = [("aabbMin", k) for k in range(3)] + [("aabbMax", k) for k in range(3)]


def flat(n, seed):
    """Every triangle in the plane z = +-0 (a seeded sign per vertex): every node's z bounds are zeros."""
    rng = np.random.default_rng(seed)
    c = rng.random((n, 1, 2)) * 40 - 20
    p = c + (rng.random((n, 3, 2)) - 0.5) * 3
    v = np.zeros((n * 3, 4), np.float32)
    v[:, :2] = p.reshape(-1, 2)
    v[:, 2] = np.where(rng.random(n * 3) < 0.5, util.NEG_ZERO, np.float32(0))
    return v


def straddle(n, seed):
    """Long triangles across the wall x = 0 with two vertices on the floor y = +-0 (seeded signs), among small ones: spatial
    splits on x clip fragments whose y bounds are zeros."""
    rng = np.random.default_rng(seed)
    z = rng.random((n, 3)) * 20 - 10
    x = np.stack([-(rng.random(n) * 18 + 2), rng.random(n) * 18 + 2, rng.random(n) * 4 - 2], 1)
    y = np.stack([np.zeros(n), np.zeros(n), rng.random(n) * 6 + 0.5], 1)
    small = rng.random(n) < 0.5           # half of them short, on one side of the wall
    x[small] = rng.random((int(small.sum()), 1)) * 30 - 15 + (rng.random((int(small.sum()), 3)) - 0.5)
    v = np.zeros((n * 3, 4), np.float32)
    v[:, 0], v[:, 1], v[:, 2] = x.reshape(-1), y.reshape(-1), z.reshape(-1)
    v[:, 1][(v[:, 1] == 0) & (rng.random(n * 3) < 0.5)] = util.NEG_ZERO
    return v


@functools.lru_cache(maxsize=None)
def family(fam, n):
    seed = 7 + n % 1000
    kind, _, arg = fam.partition(":")
    if kind == "zero":
        v = util.signed_zero(scenes.procedural_scene(n, seed), arg, seed)
    elif kind == "mirror":
        v = np.array(scenes.procedural_scene(n, seed), np.float32)
        for a in {"xyz": (0, 1, 2), "x": (0,)}[arg]:
            v[:, a] *= -1
    else:
        v = flat(n, seed) if kind == "flat" else straddle(n, seed)
    v.setflags(write=False)
    return v


def family_rays(v, seed=5, res=24):
    """Camera rays, axis rays from the zero planes (with rD = +-inf on their zero components) and rays of every octant, as
    tests/test_offatrium_gpu.py unit_rays makes them, over the family's own bounds; octant-blocked."""
    lo, hi = scenes.scene_bounds(v)
    ax = util.axis_rays(lo, hi, per_axis=8, seed=seed)
    r = np.concatenate([util.ray_sets(v, res=res)[0]["primary"], ax, util.with_inf_rd(ax), util.octant_rays(lo, hi, 40, seed)])
    return util.octant_blocks(r, seed)


@functools.lru_cache(maxsize=None)
def family_hq(fam, n):
    """The restatement's BuildHQ of a family -> (nodes, primIdx, idxCount)"""
    return portpy.build_hq(family(fam, n))


def positive_zeros(v):
    v = np.array(v, np.float32)
    v[v == 0] = 0
    return v


def neg_zero(x):
    return (x == 0) & np.signbit(x)


def compare_trees(got, want):
    """Two BuildHQ trees (nodes, primIdx) -> (first differing node and field or None, whether they differ in the sign bits of zero
    bounds only)."""
    (a, ia), (b, ib) = got, want
    if a.shape != b.shape:
        return f"usedNodes {a.shape[0]} != {b.shape[0]}", False
    first = None
    for i in np.nonzero(a.view(np.uint32).reshape(-1, 8) != b.view(np.uint32).reshape(-1, 8))[0][:1]:
        for f in ("aabbMin", "leftFirst", "aabbMax", "triCount"):
            if a[i][f].tobytes() != b[i][f].tobytes():
                first = f"node {i} {f}: got {a[i][f]!r} want {b[i][f]!r}"
                break
    if first is None and not np.array_equal(ia, ib):
        k = np.nonzero(ia != ib)[0] if ia.shape == ib.shape else [min(ia.shape[0], ib.shape[0])]
        first = f"primIdx at {k[0]}"
    signs_only = (first is not None and ia.shape == ib.shape and np.array_equal(ia, ib)
                  and all(np.array_equal(a[f], b[f]) for f in ("leftFirst", "triCount", "aabbMin", "aabbMax")))
    return first, signs_only


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("fam", FAMILIES)
def test_family_is_only_a_sign_change(fam, n):
    """The tree equals the all-+0 scene's tree in leftFirst, triCount, primIdx, idxCount and every bound compared as a float."""
    v = family(fam, n)
    nodes, idx, ic = family_hq(fam, n)
    p_nodes, p_idx, p_ic = portpy.build_hq(positive_zeros(v))
    assert ic == p_ic and nodes.shape == p_nodes.shape and np.array_equal(idx, p_idx)
    for f in ("leftFirst", "triCount", "aabbMin", "aabbMax"):
        assert np.array_equal(nodes[f], p_nodes[f]), f
    assert (util.count_neg_zero(v[:, :3]) > 0) == (fam != "zero:pos")


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("fam", NEG_FAMILIES)
def test_zero_signs_below_the_root(fam, n):
    """Some node below the root has a -0 bound; on the larger scenes some bound field is -0 in one node and +0 in another."""
    nodes = family_hq(fam, n)[0][2:]
    assert neg_zero(nodes["aabbMin"]).any() or neg_zero(nodes["aabbMax"]).any(), f"{fam} {n}: no -0 bound below the root"
    if n >= 2000 and fam in BOTH_SIGNS:
        both = [(f, k) for f, k in BOUNDS if neg_zero(nodes[f][:, k]).any() and ((nodes[f][:, k] == 0) & ~np.signbit(nodes[f][:, k])).any()]
        assert both, f"{fam} {n}: no field holds both zero signs below the root"


@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("fam", FAMILIES)
def test_family_splits_references(fam, n):
    """Spatial splits: the leaves reference some triangle twice (of the 40-triangle scenes, in straddle)."""
    nodes, idx, _ = family_hq(fam, n)
    if n >= 2000 or fam == "straddle":
        assert int(nodes["triCount"].sum()) > n


def no_neg_zero_bound(nodes):
    return not neg_zero(nodes["aabbMin"]).any() and not neg_zero(nodes["aabbMax"]).any()


@pytest.mark.parametrize("n", SIZES)
def test_no_neg_zero_in_gives_no_neg_zero_out(n):
    for v in (family("zero:pos", n), scenes.procedural_scene(n, 7 + n % 1000), positive_zeros(family("straddle", n)),
              positive_zeros(family("flat", n))):
        assert util.count_neg_zero(v[:, :3]) == 0
        assert no_neg_zero_bound(portpy.build_hq(v)[0])


@pytest.mark.parametrize("name", list(FAIL_SCENES))
def test_failing_scenes_give_no_neg_zero(name):
    assert util.count_neg_zero(fail_scene(name)[:, :3]) == 0
    assert no_neg_zero_bound(fail_scene_hq(name)[0])


def test_compare_trees_names_the_field_and_sees_sign_only_differences():
    nodes, idx, _ = family_hq("zero:random", 2000)
    assert compare_trees((nodes, idx), (nodes, idx)) == (None, False)
    flipped = nodes.copy()
    i, k = next((i, k) for i in range(2, nodes.shape[0]) for k in range(3) if nodes["aabbMin"][i, k] == 0)
    flipped["aabbMin"][i, k] = -flipped["aabbMin"][i, k]
    first, signs_only = compare_trees((flipped, idx), (nodes, idx))
    assert first.startswith(f"node {i} aabbMin") and signs_only
    moved = nodes.copy()
    moved["leftFirst"][i] += 1
    first, signs_only = compare_trees((moved, idx), (nodes, idx))
    assert first.startswith(f"node {i} leftFirst") and not signs_only
