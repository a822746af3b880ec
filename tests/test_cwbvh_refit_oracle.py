"""The oracle of tbvh_refit_layouts' CWBVH (tests/cwbvh_refit_oracle.c orc_cwbvh_refit_from_bvh): the conversion chain over the collapse
of the built tree with the boxes of the refitted one.  It is a composition of pinned pieces, so it is held to two anchors: without motion
it is the conversion itself, byte for byte, and after motion the reference's CPU walk of it finds what BVH::Intersect finds on the
refitted BVH2."""
import numpy as np
import pytest

from oracle import portpy
from tinybvh_b200 import scenes
from tests import golden_util as G
from tests import util
from tests.cwbvh_refit_oracle import RefitCWBVH
from tests.test_oracle_pin import moved


def _refit_cw(tree, verts):
    """orc_refit of `tree` to `verts`, then the CWBVH over the collapse of the unrefitted tree -> (refitted PortBVH, PortCWBVH)"""
    built = tree.nodes.copy()
    r = portpy.PortBVH(tree.verts, nodes=built, prim_idx=tree.prim_idx)
    r.refit(verts)
    return r, RefitCWBVH(built, r.nodes, r.prim_idx, verts)


def _still_scenes():
    out = [(p.split("/")[-1], G.load(p)["verts"]) for p in G.golden_files()]
    out += [(f"seeded:{n}", scenes.procedural_scene(n, 80 + n % 7)) for n in (1, 3, 5000, 70000)]
    return out


@pytest.mark.parametrize("avx", [False, True], ids=["Build", "BuildAVX"])
@pytest.mark.parametrize("name,verts", _still_scenes(), ids=lambda x: x if isinstance(x, str) else "")
def test_refit_cwbvh_without_motion_is_the_conversion(name, verts, avx):
    tree = portpy.PortBVH(verts, avx=avx)
    r, cw = _refit_cw(tree, verts)
    assert np.array_equal(r.nodes.view(np.uint32), tree.nodes.view(np.uint32)), f"{name}: BVH::Refit without motion changed the tree"
    want = portpy.PortCWBVH(tree.nodes, tree.prim_idx, verts)
    assert cw.nodes.shape == want.nodes.shape and np.array_equal(cw.nodes.view(np.uint32), want.nodes.view(np.uint32)), f"{name}: bvh8Data"
    assert np.array_equal(cw.tris.view(np.uint32), want.tris.view(np.uint32)), f"{name}: bvh8Tris"


@pytest.mark.parametrize("avx", [False, True], ids=["Build", "BuildAVX"])
@pytest.mark.parametrize("ntris,seed", [(5000, 91), (70000, 92)])
def test_refit_cwbvh_walk_matches_refitted_bvh(ntris, seed, avx):
    v = scenes.procedural_scene(ntris, seed)
    tree = portpy.PortBVH(v, avx=avx)
    blocks = portpy.PortCWBVH(tree.nodes, tree.prim_idx, v).nodes.shape[0]
    for frame in (1, 2):   # every frame refits the BUILT tree's collapse, not the previous frame's
        w = moved(v, seed + frame, amp=0.05)
        r, cw = _refit_cw(tree, w)
        assert cw.nodes.shape[0] == blocks, "the wide-node count is the conversion's"
        sets, bounds = util.ray_sets(w, res=64)
        a, b = sets["primary"].copy(), sets["primary"].copy()
        r.intersect(a), cw.intersect(b)
        for kind, rays in util.derived_sets(a, w, bounds).items():
            x, y = rays.copy(), rays.copy()
            r.intersect(x), cw.intersect(y)
            assert util.classify_mismatches(y, x, w)["real"] == 0, f"frame {frame} {kind}"
        assert util.classify_mismatches(b, a, w)["real"] == 0, f"frame {frame} primary"
        assert (a["t"] < 1e30).sum() > 1000
