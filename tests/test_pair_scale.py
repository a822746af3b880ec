"""Intersecting triangle pairs and distances between meshes away from the unit scale, on the host restatements (tests/tritri_oracle.c,
meshdist_oracle.c; DESIGN.md §4.12-4.13), without a GPU.  The unit-scale suites hold the pair test to exact arithmetic on integer lattices
and the pair distance to fp64 near the origin, and scaling by 2^k to exact covariance; this file covers what those leave open:
* signed-zero twins: a mesh whose snapped zeros are -0 (every one, a seeded sign each, or every order within a triangle) gives its +0
  twin's overlap pairs and bits, nearest records and distance pairs bit for bit, two-mesh and self, and the pair test and pair distance of
  any pair of its triangles are the twin's bits;
* translated lattices: integer soups moved by 2^20 and 3 * 2^21 stay exact in fp32, and so do their differences from T's v0, so every
  pair, bit, record and distance is the unshifted one;
* translated float pairs: the distance kinds of test_mesh_distance moved by 3e5 and 3e6 against fp64 on the exact fp32 inputs, within
  2e-6 of the pair's local magnitude max |corner - T.v0| (the coordinates' magnitude is 1e5 to 1e6 times larger), and the pair test
  against exact rationals wherever every orientation is at least 1e-3 L^3."""
from fractions import Fraction

import numpy as np
import pytest

from oracle import portpy
from tinybvh_b200 import scenes
from tests import meshdist_oracle as md, tritri_oracle as to, util
from tests.test_mesh_distance import DEGENERATE, pair_cases
from tests.test_mesh_overlap import lattice_soup
from tests.test_signed_distance import soup, torus
from tests.test_winding_number import two_spheres

ZERO = ["neg", "random", "order"]          # against the "pos" twin (util.signed_zero)
LATTICE_SHIFT = [1048576.0, 6291456.0]     # 2^20 and 3 * 2^21: lattice coordinates in [-16, 16] stay integers
FLOAT_SHIFT = [3e5, 3e6]
DIST_BOUND = 2e-6                          # of the local magnitude, as the unit-scale bound is of the inputs' magnitude


def meshes(name):
    """(A, B) float4 soups at unit scale, each crossing the planes x = 0 and y = 0 that util.signed_zero snaps to"""
    if name == "lattice":
        return lattice_soup(600, 1), lattice_soup(500, 2)
    if name == "spheres":
        return soup(*two_spheres()), soup(*torus())
    if name == "procedural":
        a = scenes.procedural_scene(3000, 33)
        b = scenes.procedural_scene(1500, 34)
        b[:, :3] += np.float32(0.05)
        return a, b
    raise ValueError(name)


MESHES = ["lattice", "spheres", "procedural"]


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def results(A, B, r):
    """every restated result over Build trees: two-mesh and self overlap pairs and bits, nearest records at r_max inf and r, distance
    pairs at r"""
    ob, oa = portpy.PortBVH(B), portpy.PortBVH(A)
    out = {}
    out["overlap"], out["overlap_bits"] = to.tree(ob.nodes, ob.prim_idx, B, A)[:2]
    out["self_overlap"], out["self_overlap_bits"] = to.tree(oa.nodes, oa.prim_idx, A)[:2]
    for label, nodes, idx, vb, va in (("", ob.nodes, ob.prim_idx, B, A), ("self_", oa.nodes, oa.prim_idx, A, None)):
        d, j = md.nearest(nodes, idx, vb, va)
        out[label + "nearest_d"], out[label + "nearest_j"] = bits(d), j
        d, j = md.nearest(nodes, idx, vb, va, r_max=r)
        out[label + "nearest_r_d"], out[label + "nearest_r_j"] = bits(d), j
        out[label + "dist_pairs"] = md.pairs(nodes, idx, vb, va, r)[0]
    return out


def wall_pairs(v, n, seed):
    """n seeded pairs of distinct triangles of v that each have a corner with a zero x or y coordinate -> (T, U) (n, 3, 3)"""
    t = v.reshape(-1, 3, 4)[:, :, :3]
    wall = np.nonzero((t[:, :, :2] == 0).any((1, 2)))[0]
    rng = np.random.default_rng(seed)
    i, j = rng.choice(wall, n), rng.choice(wall, n)
    keep = i != j
    return t[i[keep]], t[j[keep]]


def zero_signs(x, mode, seed):
    """x with its zeros made -0 as util.signed_zero's modes do: every one, a seeded sign each, or the sign triple of each corner's three
    coordinates running through every order (the pattern of (corner index / 3) % 8)"""
    x = np.array(x, np.float32)
    flat = x.reshape(-1)
    if mode == "neg":
        neg = np.ones(flat.shape[0], bool)
    elif mode == "random":
        neg = np.random.default_rng(seed).random(flat.shape[0]) < 0.5
    else:
        k = np.arange(flat.shape[0])
        neg = (((k // 3) % 8) >> (k % 3)) & 1 == 1
    flat[(flat == 0) & neg] = util.NEG_ZERO
    return x


# ---- signed-zero twins -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ZERO)
def test_pair_functions_ignore_the_sign_of_zero(mode):
    """the pair test (two-mesh and self rules) and the pair distance of pairs of triangles with corners on the snapped walls: the bits of
    the +0 twin's pairs, in both argument orders"""
    v0 = scenes.procedural_scene(3000, 33)
    v = util.signed_zero(v0, mode, seed=3, frac=0.2)
    vp = util.signed_zero(v0, "pos", seed=3, frac=0.2)
    assert util.count_neg_zero(v) > 0
    T, U = wall_pairs(v, 20000, 4)
    Tp, Up = wall_pairs(vp, 20000, 4)
    assert util.count_neg_zero(np.r_[T, U]) > 1000
    bad = []
    for label, (a, b, ap, bp) in {"T, U": (T, U, Tp, Up), "U, T": (U, T, Up, Tp)}.items():
        n = int((bits(md.dist2(a, b)) != bits(md.dist2(ap, bp))).sum())
        if n:
            bad.append(f"dist2({label}): {n} of {a.shape[0]}")
        for self in (False, True):
            n = int((to.tt(a, b, self) != to.tt(ap, bp, self)).sum())
            if n:
                bad.append(f"tt({label}, self={self}): {n}")
    # lattice pairs in {-1, 0, 1}^3: many touching, coplanar and shared-corner cases, with -0 corners
    Lp = np.random.default_rng(5).integers(-1, 2, (2, 6000, 3, 3)).astype(np.float32)
    Lz = zero_signs(Lp, mode, 6)
    assert util.count_neg_zero(Lz) > 0
    for self in (False, True):
        n = int((to.tt(Lz[0], Lz[1], self) != to.tt(Lp[0], Lp[1], self)).sum())
        if n:
            bad.append(f"lattice tt self={self}: {n}")
    n = int((bits(md.dist2(Lz[0], Lz[1])) != bits(md.dist2(Lp[0], Lp[1]))).sum())
    if n:
        bad.append(f"lattice dist2: {n}")
    assert not bad, f"{mode}: " + "; ".join(bad)


@pytest.mark.parametrize("mode", ZERO)
@pytest.mark.parametrize("name", MESHES)
def test_signed_zero_twin(name, mode):
    """overlap pairs and bits, nearest records and distance pairs (two-mesh and self) of a mesh whose zeros are -0: the +0 twin's bits"""
    A0, B0 = meshes(name)
    A, B = util.signed_zero(A0, mode, seed=3, frac=0.2), util.signed_zero(B0, mode, seed=4, frac=0.2)
    Ap, Bp = util.signed_zero(A0, "pos", seed=3, frac=0.2), util.signed_zero(B0, "pos", seed=4, frac=0.2)
    assert util.count_neg_zero(A) > 0 and util.count_neg_zero(B) > 0
    r = 0.02 * float(np.abs(Ap[:, :3]).max())
    got, want = results(A, B, r), results(Ap, Bp, r)
    bad = [f"{key}: {got[key].shape} vs {want[key].shape}, {int((got[key] != want[key]).sum()) if got[key].shape == want[key].shape else '-'} differ"
           for key in want if not np.array_equal(got[key], want[key])]
    assert not bad, f"{name} {mode}: " + "; ".join(bad)
    assert want["dist_pairs"].shape[0] > 0 and want["self_dist_pairs"].shape[0] > 0


# ---- translated lattices: exact ----------------------------------------------------------------------------------------------------
def lattice_pair():
    """integer soups in [-11, 11] and a self mesh of three of them, with repeated, touching and crossing triangles"""
    A, B = lattice_soup(400, 21), lattice_soup(350, 22)
    S = np.concatenate([A, lattice_soup(250, 23, lo=-4, hi=4)])
    return A, B, S


@pytest.mark.parametrize("shift", LATTICE_SHIFT)
def test_translated_lattices_are_exact(shift):
    """every coordinate and every difference stays exact in fp32, so the pairs, bits, records and distances are the unshifted ones"""
    A, B, S = lattice_pair()
    At, Bt, St = (util.translated(x, shift) for x in (A, B, S))
    for x, xt in ((A, At), (B, Bt), (S, St)):
        assert np.array_equal(xt[:, :3].astype(np.float64) - shift, x[:, :3].astype(np.float64)), "not exact"
    want, got = results(A, B, 1.5), results(At, Bt, 1.5)
    bad = [key for key in want if not np.array_equal(got[key], want[key])]
    assert not bad, f"{shift}: {bad}"
    assert want["overlap"].shape[0] > 50 and want["dist_pairs"].shape[0] > want["overlap"].shape[0]
    sp, sbits = to.all_pairs(S)
    tp, tbits = to.all_pairs(St)
    assert sp.shape[0] > 50 and np.array_equal(tp, sp) and np.array_equal(tbits, sbits)
    T, U = S.reshape(-1, 3, 4)[:325, :, :3], S.reshape(-1, 3, 4)[325:650, :, :3]
    Tt, Ut = St.reshape(-1, 3, 4)[:325, :, :3], St.reshape(-1, 3, 4)[325:650, :, :3]
    assert np.array_equal(bits(md.dist2(Tt, Ut)), bits(md.dist2(T, U)))
    for self in (False, True):
        assert np.array_equal(to.tt(Tt, Ut, self), to.tt(T, U, self))


# ---- translated float pairs: fp64 ----------------------------------------------------------------------------------------------
def local_mag(T, U):
    """max |corner - T.v0| over the six corners, T the canonical triangle (the pair test's frame); fp64 on the fp32 inputs"""
    T, U = np.asarray(T, np.float64), np.asarray(U, np.float64)
    out = np.zeros(T.shape[0])
    for a, b in ((T, U), (U, T)):
        m = np.maximum(np.abs(a - a[:, :1]).max((1, 2)), np.abs(b - a[:, :1]).max((1, 2)))
        out = np.maximum(out, m)
    return out


@pytest.mark.parametrize("shift", FLOAT_SHIFT)
def test_translated_pair_distance_against_fp64(shift):
    """sqrt( tt_dist2 ) within 2e-6 of the local magnitude of the fp64 distance on the exact fp32 inputs (0 where exact rationals say the
    triangles meet), every kind of pair_cases moved by 3e5 and 3e6; the pair test agrees with exact rationals on every pair whose
    orientations are all at least 1e-3 L^3 (L^2 in the plane)"""
    worst, checked, total = {}, 0, 0
    for kind, (T0, U0) in pair_cases(seed=15, n=500).items():
        T, U = T0 + np.float32(shift), U0 + np.float32(shift)
        got = np.sqrt(md.dist2(T, U).astype(np.float64))
        want = md.fp64_tt(T, U)
        meet = np.array([to.exact_tt(t, u, num=Fraction) for t, u in zip(T, U)])
        tt = to.tt(T, U)
        want = np.where(meet & tt, 0.0, want)
        # a pair the fp32 test does not report although it meets exactly is a degenerate one (zero scaled normal), or one within rounding
        # of touching: its distance is the least candidate, the fp64 fifteen-feature distance
        L = local_mag(T, U)
        tol = DIST_BOUND * L
        err = np.abs(got - want)
        worst[kind] = float((err / L).max())
        assert (err <= tol).all(), f"{kind} + {shift}: worst error {(err / tol).max():.3g} x the tolerance"
        if kind not in DEGENERATE:
            for k in range(T.shape[0]):
                tr = to._Track()
                e = to.exact_tt(T[k], U[k], num=Fraction, track=tr)
                Lk = Fraction(float(L[k]))
                if (tr.m3 is None or tr.m3 >= Fraction(1, 1000) * Lk ** 3) and (tr.m2 is None or tr.m2 >= Fraction(1, 1000) * Lk ** 2):
                    checked += 1
                    assert e == tt[k], f"{kind} + {shift}: pair {k} is well conditioned and differs from exact rationals"
            total += T.shape[0]
    print(f"+{shift}: worst error of the local magnitude " + ", ".join(f"{k} {v:.3g}" for k, v in worst.items()))
    assert checked > 0.5 * total, (checked, total)
