"""tbvh_mesh_overlap_pairs / _bits and tbvh_mesh_distance / _pairs on the device away from the unit scale (DESIGN.md §4.12-4.13): held bit
for bit to the host restatements over Build and BuildHQ trees on signed-zero twins and translated meshes, and a twin's device results
equal to its +0 twin's device results (tests/test_pair_scale.py holds the restatements themselves to the twins, to exact lattices and to
fp64)."""
import numpy as np
import pytest

from tinybvh_b200 import api
from tests import tritri_oracle as to, util
from tests import test_mesh_distance_gpu as mdg, test_mesh_overlap_gpu as mog
from tests.test_pair_scale import LATTICE_SHIFT, MESHES, ZERO, lattice_pair, meshes

pytestmark = pytest.mark.gpu
BUILDERS = ["Build", "BuildHQ"]


def device_results(a, b, n, r):
    """every device result of a against b and of a against itself"""
    out = {}
    for label, x in (("", b), ("self_", a)):
        p, c, rc = mog.pairs_device(a, x, 1 << 20)
        assert rc == 0 and c < 1 << 20
        out[label + "overlap"] = p[:c].copy()
        out[label + "overlap_bits"] = mog.bits_device(a, x, n)
        d, j = mdg.nearest_device(a, x, n)
        out[label + "nearest"] = (d.view(np.uint32).copy(), j.copy())
        p, c, rc = mdg.pairs_device(a, x, r, 1 << 20)
        assert rc == 0 and c < 1 << 20
        out[label + "dist_pairs"] = p[:c].copy()
    return out


def check_overlap(a, b, va, vb, label):
    """pairs, count and bits equal the restatement's over b's tree; unlike mog.check, bits are not asked to be membership in the pairs:
    a tree whose leaf boxes do not hold their triangles (a BuildHQ tree of a mesh moved by 3e6) reaches pairs one way only"""
    self = a is b
    want, wbits, _, _ = to.tree(*b.download(), vb, None if self else va)
    got, count, rc = mog.pairs_device(a, b, max(want.shape[0], 1))
    assert rc == 0 and count == want.shape[0] and np.array_equal(got[:count], want), f"{label}: pairs differ"
    assert np.array_equal(mog.bits_device(a, b, va.shape[0] // 3), wbits), f"{label}: bits differ"


def check_both(A, B, builder, label, r):
    """both queries, two-mesh and self, against the restatements over the device's own trees -> the device results"""
    a, b = getattr(api.BVH(), builder)(A), getattr(api.BVH(), builder)(B)
    check_overlap(a, b, A, B, label)
    check_overlap(a, a, A, A, f"self {label}")
    mdg.check(a, b, A, *b.download(), B, label, r=r)
    mdg.check(a, a, A, *a.download(), A, f"self {label}", r=r)
    return device_results(a, b, A.shape[0] // 3, r)


def same(x, y):
    if isinstance(x, tuple):
        return all(np.array_equal(p, q) for p, q in zip(x, y))
    return np.array_equal(x, y)


@pytest.mark.parametrize("builder", BUILDERS)
@pytest.mark.parametrize("mode", ZERO)
@pytest.mark.parametrize("name", MESHES)
def test_signed_zero_twins(gpu, name, mode, builder):
    A0, B0 = meshes(name)
    A, B = util.signed_zero(A0, mode, seed=3, frac=0.2), util.signed_zero(B0, mode, seed=4, frac=0.2)
    Ap, Bp = util.signed_zero(A0, "pos", seed=3, frac=0.2), util.signed_zero(B0, "pos", seed=4, frac=0.2)
    r = 0.02 * float(np.abs(Ap[:, :3]).max())
    got = check_both(A, B, builder, f"{name}/{mode}/{builder}", r)
    want = check_both(Ap, Bp, builder, f"{name}/pos/{builder}", r)
    bad = [key for key in want if not same(got[key], want[key])]
    assert not bad, f"{name} {mode} {builder}: the device's twin results differ in {bad}"


@pytest.mark.parametrize("builder", BUILDERS)
@pytest.mark.parametrize("shift", LATTICE_SHIFT)
def test_translated_lattices(gpu, shift, builder):
    """exact in fp32, so the device's results are the unshifted ones as well as the restatement's"""
    A, B, S = lattice_pair()
    want = check_both(A, B, builder, f"lattice/{builder}", 1.5)
    got = check_both(util.translated(A, shift), util.translated(B, shift), builder, f"lattice+{shift}/{builder}", 1.5)
    bad = [key for key in want if not same(got[key], want[key])]
    assert not bad, f"{shift} {builder}: {bad}"
    e, et = getattr(api.BVH(), builder)(S), getattr(api.BVH(), builder)(util.translated(S, shift))
    p, c, _ = mog.pairs_device(e, e, 1 << 20)
    pt, ct, _ = mog.pairs_device(et, et, 1 << 20)
    assert c > 50 and ct == c and np.array_equal(pt[:ct], p[:c])


@pytest.mark.parametrize("builder", BUILDERS)
@pytest.mark.parametrize("shift", [3e5, 3e6])
def test_translated_meshes(gpu, shift, builder):
    """procedural meshes and the two spheres moved by 3e5 and 3e6: rounding merges corners and flattens triangles, and the device
    follows the restatement through all of it"""
    for name in ("procedural", "spheres"):
        A, B = (util.translated(x, shift) for x in meshes(name))
        check_both(A, B, builder, f"{name}+{shift}/{builder}", 0.02 * float(np.ptp(A[:, :3], 0).max()))
