"""The CWBVH kernels' float slab test: a warp runs it instead of the integer-ordered one when any of its rays fails
cw_ray_fits (cw_walk.cuh), e.g. a ray whose rD was computed as 1 / D with a zero component: rD.x = +inf makes x plane values NaN
(q = 0: 0 * inf), which fminf / fmaxf skip as the reference's walk does when they come first, while the integer order would put
a NaN above every float and cull the child.  Rays with D.x = 0 and rD.x = +inf (or the safercp value 1e30) must give
BVH8_CWBVH::Intersect's hits bit for bit, whether every lane of a warp or one lane per warp carries the infinity."""
import numpy as np
import pytest

from tinybvh_b200 import api, scenes
from tests import util

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("lanes", ["every", "one_per_warp", "none"])
def test_cwbvh_infinite_rd(gpu, lanes):
    v = scenes.procedural_scene(30000, 31)
    cw, _ = util.oracle_cwbvh(v, mode=2)
    e = api.BVH8_CWBVH().upload(cw.nodes, cw.tris)
    sets, _ = util.ray_sets(v, res=64)
    rays = sets["primary"].copy()
    rays["D"][:, 0] = 0.0
    rays["rD"][:, 0] = np.float32(1e30)  # safercp( +0 )
    pick = {"every": np.ones(rays.shape[0], bool), "one_per_warp": np.arange(rays.shape[0]) % 32 == 7, "none": np.zeros(rays.shape[0], bool)}[lanes]
    rays["rD"][pick, 0] = np.float32(np.inf)
    want, got = rays.copy(), rays.copy()
    cw.intersect(want)
    e.Intersect(got)
    assert (want["t"] < 1e30).mean() > 0.5
    assert util.compare_hits(got, want) == {"prim": 0, "t": 0, "u": 0, "v": 0}
    # any-hit: BVH8_CWBVH::IsOccluded is Intersect, then t < d (tiny_bvh.h:312)
    shadow = rays.copy()
    shadow["t"] = np.float32(20.0)
    traced = shadow.copy()
    cw.intersect(traced)
    occ_want = traced["t"] < shadow["t"]
    occ_got = np.unpackbits(e.IsOccluded(shadow).view(np.uint8), bitorder="little")[: shadow.shape[0]].astype(bool)
    assert 0 < occ_want.sum() < occ_want.shape[0]
    assert np.array_equal(occ_got, occ_want)
