"""The device's proximity queries away from the unit scale (DESIGN.md §4.9-4.11): on meshes scaled by 2^-126 to 2^90, translated by
millions of units and carrying -0 coordinates, every record and bit of tbvh_closest_point, tbvh_sphere_overlap, tbvh_signed_distance and
tbvh_winding_number (each after its prepare) equals the host restatement's, in host and device space, on the trees of Build, BuildHQ and
BuildPLOC; the device functions give the batch call's bits; and the power-of-two covariance of tests/test_proximity_scale.py holds on
the device itself."""
import numpy as np
import pytest

from tinybvh_b200 import api
from tests import util
from tests import test_closest_point_gpu as cpg, test_signed_distance_gpu as sdg, test_winding_number_gpu as wng
from tests.test_closest_point_gpu import consumer  # noqa: F401  (the module fixture that compiles the caller's kernel)
from tests.test_proximity_scale import CLOSED, base, scaled_q

pytestmark = pytest.mark.gpu

SCALES = [-126, -100, -60, -40, -36, -20, 20, 36, 40, 60, 90]
FAMILIES = ["scale:%d" % k for k in SCALES] + ["shift:1048576", "shift:-12582912", "zero:neg", "zero:random", "zero:order"]
BUILDERS = ["Build", "BuildHQ", "BuildPLOC"]


def family(name, fam):
    """(soup, queries) of a mesh in a family: scaled by 2^k (queries and radii too), translated (queries too), or zeros snapped to -0"""
    V, F, v, q = base(name)
    kind, arg = fam.split(":")
    if kind == "scale":
        return util.scaled(v, int(arg)), scaled_q(q, int(arg))
    if kind == "shift":
        v, q = util.translated(v, float(arg)), q.copy()
        q[:, :3] = q[:, :3] + np.float32(float(arg))
        return v, q
    return util.signed_zero(v, arg, seed=3, frac=0.2), util.signed_zero(q, arg, seed=5, frac=0.2)


@pytest.mark.parametrize("builder", BUILDERS)
@pytest.mark.parametrize("fam", FAMILIES)
@pytest.mark.parametrize("name", ["icosphere", "star", "two_spheres"])
def test_queries_match_restatement(gpu, name, fam, builder):
    v, q = family(name, fam)
    e = getattr(api.BVH(), builder)(v)
    nodes, idx = e.download()
    label = f"{name}/{fam}/{builder}"
    cpg.check_tree(e, nodes, idx, v, q, label, host=True)
    if name in CLOSED:
        sdg.check_tree(e, nodes, idx, v, q, label, host=True)
    wng.check_tree(e.h, nodes, idx, v, q, label, host=True)


@pytest.mark.parametrize("fam", ["scale:-40", "scale:40", "scale:90", "shift:-12582912", "zero:order"])
def test_device_functions(gpu, consumer, fam):
    """tbvh::closest_point_bvh / sphere_overlaps_bvh from a caller's kernel (tests/closest_point_consumer.cu) give the batch call's bits"""
    import torch
    v, q = family("icosphere", fam)
    e = api.BVH().Build(v)
    want, wbits = cpg.device_query(e, q, False), cpg.device_query(e, q, True)
    n = q.shape[0]
    dq = cpg.torch_f(q)
    out = torch.full((n, 4), -7.0, dtype=torch.float32, device="cuda")
    bits = torch.zeros((n + 31) // 32, dtype=torch.int32, device="cuda")
    assert consumer.cc_query(e.device_view(), dq.data_ptr(), out.data_ptr(), bits.data_ptr(), None, n) == 0
    assert np.array_equal(out.cpu().numpy().view(np.uint32), want.view(np.uint32)), f"{fam}: device function differs from the batch call"
    assert np.array_equal(bits.cpu().numpy().view(np.uint32), wbits[: (n + 31) // 32]), f"{fam}: device function bits differ"


@pytest.mark.parametrize("name", ["icosphere", "two_spheres"])
def test_covariance_on_the_device(gpu, name):
    """at k = -32, -20, 20, 40 the device's closest-point and signed distances are its k = 0 ones times 2^k with identical u, v, prim and
    sign; sphere words and winding numbers at every beta keep their bits"""
    V, F, v0, q0 = base(name)

    def run(k):
        v, q = util.scaled(v0, k), scaled_q(q0, k)
        e = api.BVH().Build(v)
        out = {"cp": cpg.device_query(e, q, False), "overlap": cpg.device_query(e, q, True)}
        if name in CLOSED:
            api.check(api._lib.lib().tbvh_signed_distance_prepare(e.h))
            out["sd"] = sdg.sd_device(e.h, q)
        api.check(api._lib.lib().tbvh_winding_number_prepare(e.h))
        for b in wng.BETAS:
            out[f"wn{b}"] = wng.wn_device(e.h, q, b)
        return out

    r0 = run(0)
    for k in (-32, -20, 20, 40):
        rk = run(k)
        for key, want in r0.items():
            want = np.array(want)
            if key in ("cp", "sd"):
                want[:, 0] = np.ldexp(want[:, 0], k)
            assert np.array_equal(np.ascontiguousarray(rk[key]).view(np.uint32), want.view(np.uint32)), f"{name} k={k}: {key} differs"
