"""tbvh_intersect_all / tbvh_intersect_all_tlas on the device against fp64 (DESIGN.md §4.14): next to the bit-for-bit check against the
host restatement, the device's own records and counts are held to the rules of tests/test_intersect_all_fp64.py (every robust crossing
reported, no robust miss, t within 1e-6 |O - v0| / |D|, t order, robust <= count <= robust + ambiguous) on scaled, translated and
signed-zero scenes and on affine instances."""
import numpy as np
import pytest

from oracle import refpy
from tinybvh_b200 import api
from tests import util
from tests import test_intersect_all_fp64 as F
from tests import test_intersect_all_gpu as ag, test_intersect_all_tlas_gpu as tg

pytestmark = pytest.mark.gpu
KS = (1, 5, 64)


def device_rules(v, rays, builder, label):
    """the device against the restatement for every k in KS, then the rules on the device's k = 64 result"""
    e = getattr(api.BVH(), builder)(v)
    nodes, idx = e.download()
    ag.check_tree(e, nodes, idx, v, rays, label, ks=KS)
    h, c = ag.device_all(e, rays, F.K)
    res = F.check_rules(rays, v.reshape(-1, 3, 4)[:, :, :3], h, c)
    print(label, res)
    F.assert_rules(res, label)
    return h, c


@pytest.mark.parametrize("builder", ["Build", "BuildHQ"])
@pytest.mark.parametrize("fam", ["scale:-9", "scale:0", "scale:20", "shift:3e5", "shift:3e6"])
def test_scaled_and_translated(gpu, fam, builder):
    v, rays = F.scene()
    kind, x = fam.split(":")
    if kind == "scale":
        k = int(x)
        device_rules(util.scaled(v, k), util.scaled_rays(rays, k), builder, f"{fam}/{builder}")
    else:
        s = float(x)
        vt = util.translated(v, s)
        for name, r in (("near", F.near_rays(v, 300, 2)), ("inside", rays.copy())):
            r["O"] = r["O"] + np.float32(s)
            device_rules(vt, r, builder, f"{fam}/{builder}/{name}")


def test_below_the_window(gpu):
    """the device loses the same crossings below the window as the restatement: bit for bit at 2^(WINDOW_LOW - 1), some lost"""
    v, rays = F.scene()
    k = F.WINDOW_LOW - 1
    vs, rs = util.scaled(v, k), util.scaled_rays(rays, k)
    e = api.BVH().Build(vs)
    ag.check_tree(e, *e.download(), vs, rs, f"2^{k}", ks=(F.K,))
    h, c = ag.device_all(e, rs, F.K)
    assert F.check_rules(rs, vs.reshape(-1, 3, 4)[:, :, :3], h, c)["missed"] > 0


@pytest.mark.parametrize("mode", F.ZERO)
def test_signed_zero_twins(gpu, mode):
    v0, rays = F.scene()
    v, vp = util.signed_zero(v0, mode, seed=3, frac=0.2), util.signed_zero(v0, "pos", seed=3, frac=0.2)
    h, c = device_rules(v, rays, "Build", f"zero:{mode}")
    hp, cp = device_rules(vp, rays, "Build", "zero:pos")
    assert np.array_equal(c, cp) and np.array_equal(h[..., 3].view(np.uint32), hp[..., 3].view(np.uint32)), mode
    assert np.array_equal(h[..., :3], hp[..., :3]), f"{mode}: t, u or v differ in value from the +0 twin"


@pytest.mark.parametrize("name", ["rigid", "nonuniform_scale", "permutation_mirror", "translation_2^20"])
def test_tlas_affine_instances(gpu, name):
    from tinybvh_b200 import scenes
    T = F.affine_families()[name]
    v = [scenes.procedural_scene(400, 3), scenes.procedural_scene(300, 4)]
    inst = refpy.make_instances(T, np.arange(T.shape[0]) % 2)
    t, blas = tg.make_tlas(v, inst)
    scene = tg.restated(t, inst, blas, v)
    tri, offs, shift = F.world_soup(scene[2], scene[3])
    rays = F.world_rays(tri, 200, 5)
    tg.check_tlas(t.h, scene, rays, name, ks=KS)
    h, ii, c = tg.device_all(t.h, rays, F.K)
    res = F.tlas_rules(tri, offs, shift, rays, h, ii, c)
    print(name, res)
    F.assert_rules(res, name)
