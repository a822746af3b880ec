"""The host restatement of tbvh_mesh_distance / tbvh_mesh_distance_pairs (tests/meshdist_oracle.c, DESIGN.md §4.13): the pair distance
against an independent fp64 distance (all fifteen features, clamped segment-segment, 0 where exact arithmetic says the triangles meet) on
random, degenerate, nearly parallel and coplanar pairs; exact zeros on the lattice families of the overlap test; symmetry; exact scaling by
2^k for every k in [-40, 40]; consistency with the overlap query; the pruned walk against the definition on every builder's tree, the
uploaded families, a DAG and failed-split SBVHs; and the self rules."""
from fractions import Fraction

import numpy as np
import pytest

from oracle import portpy
from tinybvh_b200 import scenes
from tests import meshdist_oracle as md, tritri_oracle as to, util
from tests.test_closest_point import builder_trees, family
from tests.test_mesh_overlap import degenerate, lattice_families, lattice_soup, swapped_pairs
from tests.test_signed_distance import icosphere, soup


def tt_d(T, U):
    return np.sqrt(md.dist2(T, U).astype(np.float64))


def truth(T, U):
    """fp64 distance, 0 where exact rationals say the closed triangles meet"""
    want = md.fp64_tt(T, U)
    meet = np.array([to.exact_tt(t, u, num=Fraction) for t, u in zip(T, U)])
    return np.where(meet, 0.0, want), meet


def pair_cases(seed=5, n=1500):
    """{kind: (T, U)}: random pairs near each other, the degenerate kinds of §4.9 against random triangles, nearly parallel crossing
    edges, and coplanar disjoint pairs"""
    rng = np.random.default_rng(seed)
    out = {}
    c = rng.normal(size=(n, 1, 3)) * 3
    out["random"] = (c + rng.normal(size=(n, 3, 3)) * 0.5, c + rng.normal(size=(n, 3, 3)) * 0.5)
    out["random_apart"] = (c + rng.normal(size=(n, 3, 3)) * 0.5, c + 2 + rng.normal(size=(n, 3, 3)) * 0.5)
    a, d = c[:, 0], rng.normal(size=(n, 3))
    U = c + rng.normal(size=(n, 3, 3))
    out["sliver"] = (np.stack([a, a + d, a + d * rng.uniform(0.2, 0.8, (n, 1)) + rng.normal(size=(n, 3)) * 1e-5], 1), U)
    out["collinear"] = (np.stack([a, a + d, a + d * rng.uniform(-2, 2, (n, 1))], 1), U)
    out["zero_area"] = (np.stack([a, a + d, a], 1), U)
    out["zero_edge"] = (np.stack([a, a, a + d], 1), U)     # v0 == v1: Ericson's regions put the point at v0
    out["coincident"] = (np.stack([a, a, a], 1), U)
    # an edge of U nearly parallel to an edge of T, crossing over it at a small height: the edge-edge solution is badly conditioned
    ang = rng.uniform(1e-6, 1e-2, n) * rng.choice([-1, 1], n)
    h = rng.uniform(0, 1e-2, n)
    T = np.stack([np.c_[-np.ones(n), np.zeros(n), np.zeros(n)], np.c_[np.ones(n), np.zeros(n), np.zeros(n)], np.c_[np.zeros(n), -np.ones(n), -np.ones(n)]], 1)
    dirn = np.c_[np.cos(ang), np.sin(ang), np.zeros(n)]
    p = np.c_[rng.uniform(-0.5, 0.5, n), np.zeros(n), h]
    U = np.stack([p - dirn, p + dirn, p + np.c_[np.zeros(n), np.ones(n), np.ones(n)]], 1)
    out["near_parallel"] = (T, U)
    # coplanar and disjoint: U beyond an edge of T in T's plane
    z = rng.normal(size=(n, 1, 1))
    T2 = np.concatenate([rng.uniform(-1, 0, (n, 3, 2)), np.broadcast_to(z, (n, 3, 1))], 2)
    U2 = np.concatenate([rng.uniform(0.01, 1, (n, 3, 2)), np.broadcast_to(z, (n, 3, 1))], 2)
    out["coplanar_disjoint"] = (T2, U2)
    return {k: (np.asarray(x, np.float32), np.asarray(y, np.float32)) for k, (x, y) in out.items()}


DEGENERATE = ("sliver", "collinear", "zero_area", "zero_edge", "coincident")


def test_pair_distance_matches_fp64():
    """sqrt( tt_dist2 ) is within 2e-6 of the inputs' magnitude of the fp64 distance (0 where the triangles meet), on the degenerate kinds
    too: the vertex-edge candidates are exact where the per-triangle function of §4.9 is only held to the triangle's width"""
    worst = {}
    for kind, (T, U) in pair_cases().items():
        got = tt_d(T, U)
        want, meet = truth(T, U)
        scale = np.abs(np.concatenate([T.reshape(-1, 9), U.reshape(-1, 9)], 1)).max(1)
        tol = 2e-6 * scale
        if kind in DEGENERATE:
            # a triangle whose fp32 normal is 0 (collinear within rounding) is never reported by the pair test (§4.12 item 4), so where it
            # pierces the other exactly its distance is the least of the fifteen candidates, which the fp64 features give
            lost = meet & ~to.tt(T, U)
            want = np.where(lost, md.fp64_tt(T, U), want)
            print(f"{kind}: {int(lost.sum())} exact crossings of a triangle the pair test takes as zero-area")
        err = np.abs(got - want)
        worst[kind] = float((err / scale).max())
        assert (err <= tol).all(), f"{kind}: worst error {(err / tol).max():.3g} x the tolerance"
        assert np.isfinite(got).all() and (got >= 0).all(), kind
        print(f"{kind}: {int(meet.sum())} of {T.shape[0]} meet; worst error {worst[kind]:.3g} of the magnitude")


def test_lattice_families_zero_exactly_where_they_meet():
    """on the integer lattice families of the overlap test: d == 0 on every meeting pair (exact arithmetic: the pair test is exact there)
    and d > 0 on every disjoint pair of non-degenerate triangles"""
    for fam, (T, U, _, _) in lattice_families().items():
        d2 = md.dist2(T, U)
        meet = to.tt(T, U, False)
        ok = ~(degenerate(T) | degenerate(U))
        assert (d2[meet] == 0).all(), f"{fam}: a meeting pair at a distance"
        assert (d2[ok & ~meet] > 0).all(), f"{fam}: {int((d2[ok & ~meet] == 0).sum())} disjoint pairs at 0"
        want = md.fp64_tt(T, U)
        assert np.allclose(np.sqrt(d2[ok & ~meet].astype(np.float64)), want[ok & ~meet], rtol=1e-5, atol=1e-5), fam


def test_non_finite_pairs_are_skipped():
    T = np.array([[[0, 0, 0], [1, 0, 0], [0, 1, 0]]] * 3, np.float32)
    U = T.copy() + np.float32(2)
    U[0, 1, 2], U[1, 0, 0], U[2, 2, 1] = np.nan, np.inf, -np.inf
    assert np.isnan(md.dist2(T, U)).all() and np.isnan(md.dist2(U, T)).all()
    v = np.zeros((6, 4), np.float32)
    v[:3, :3] = T[0]
    v[3:, :3] = U[0]
    o = portpy.PortBVH(v)
    d, j = md.nearest(o.nodes, o.prim_idx, v, v[:3], r_max=np.inf)
    assert j[0] == 0 and d[0] == 0     # itself, not the non-finite triangle
    d, j = md.nearest(o.nodes, o.prim_idx, v, v[3:], r_max=np.inf)
    assert j[0] == md.NO_PRIM and d[0] == np.inf, "a non-finite triangle gets the miss record"


def test_symmetry():
    for kind, (T, U) in pair_cases(9, 600).items():
        assert np.array_equal(md.dist2(T, U).view(np.uint32), md.dist2(U, T).view(np.uint32)), kind
    for fam, (T, U, _, _) in lattice_families().items():
        assert np.array_equal(md.dist2(T, U).view(np.uint32), md.dist2(U, T).view(np.uint32)), fam
    A, B = lattice_soup(500, 1), lattice_soup(400, 2, offset=0.25)
    oa, ob = portpy.PortBVH(A), portpy.PortBVH(B)
    for r in (0.0, 0.3, 1.0):
        ab = md.pairs(ob.nodes, ob.prim_idx, B, A, r)[0]
        ba = md.pairs(oa.nodes, oa.prim_idx, A, B, r)[0]
        assert ab.shape[0] > 50 and np.array_equal(ab, swapped_pairs(ba)), r


def test_scale_gives_the_same_prims_pairs_and_scaled_distances_for_every_k():
    """BuildHQ trees (the BVH::Build leaf boxes of such meshes at 2^40 do not hold their triangles, §4.12)"""
    A, B = lattice_soup(200, 4), lattice_soup(200, 5, offset=0.5)
    ref = None
    for k in range(-40, 41):
        sa, sb = util.scaled(A, k), util.scaled(B, k)
        bn, bi, _ = portpy.build_hq(sb)
        an, ai, _ = portpy.build_hq(sa)
        d, j = md.nearest(bn, bi, sb, sa)
        ds, js = md.nearest(an, ai, sa)
        p = md.pairs(bn, bi, sb, sa, np.ldexp(np.float32(0.75), k))[0]
        s = md.pairs(an, ai, sa, None, np.ldexp(np.float32(0.75), k))[0]
        got = (np.ldexp(d, -k), j, np.ldexp(ds, -k), js, p, s)
        if ref is None:
            ref = got
            assert (d > 0).any() and p.shape[0] > 20 and s.shape[0] > 20
        for x, y in zip(got, ref):
            assert np.array_equal(x, y), k


def test_overlap_pairs_are_distance_pairs_at_zero():
    A, B = lattice_soup(600, 7), lattice_soup(500, 8, offset=0.5)
    ob = portpy.PortBVH(B)
    ov = to.tree(ob.nodes, ob.prim_idx, B, A)[0]
    dp = md.pairs(ob.nodes, ob.prim_idx, B, A, 0.0)[0]
    assert ov.shape[0] > 50
    assert set(map(tuple, ov)) <= set(map(tuple, dp)), "an overlapping pair is not within distance 0"
    d, j = md.nearest(ob.nodes, ob.prim_idx, B, A)
    assert (d[ov[:, 0]] == 0).all()
    # self: overlapping pairs that share no corner are self distance pairs at 0
    S = np.concatenate([A, lattice_soup(300, 9, offset=0.25)])
    os_ = portpy.PortBVH(S)
    sov = to.tree(os_.nodes, os_.prim_idx, S)[0]
    t = S.reshape(-1, 3, 4)[:, :, :3]
    share = np.array([(t[i][:, None] == t[k][None]).all(2).any() for i, k in sov]).reshape(-1)
    sdp = md.pairs(os_.nodes, os_.prim_idx, S, None, 0.0)[0]
    assert (~share).sum() > 20
    assert set(map(tuple, sov[~share])) <= set(map(tuple, sdp))


def check_walk(nodes, idx, vb, va, label, holds=True, r=0.05):
    """pruned walk == definition (nearest records bit for bit, pairs); where boxes hold their triangles, the nearest distance is the least
    pair distance over all triangles of B (the bounds raise nothing beyond rounding)"""
    d, j = md.nearest(nodes, idx, vb, va)
    bd, bj = md.nearest(nodes, idx, vb, va, brute=True)
    assert np.array_equal(d.view(np.uint32), bd.view(np.uint32)) and np.array_equal(j, bj), f"{label}: nearest walk differs from the definition"
    for rm in (0.0, r):
        dm, jm = md.nearest(nodes, idx, vb, va, r_max=rm)
        bdm, bjm = md.nearest(nodes, idx, vb, va, r_max=rm, brute=True)
        assert np.array_equal(dm.view(np.uint32), bdm.view(np.uint32)) and np.array_equal(jm, bjm), f"{label}: r_max {rm}"
        p = md.pairs(nodes, idx, vb, va, rm)[0]
        bp = md.pairs(nodes, idx, vb, va, rm, brute=True)[0]
        assert np.array_equal(p, bp), f"{label}: pairs at {rm} differ from the definition"
        found = jm != md.NO_PRIM
        assert np.array_equal(np.unique(p[:, 0]), np.nonzero(found)[0]) or va is None, f"{label}: nearest within r is not 'has a pair'"
    if holds:
        tb = vb.reshape(-1, 3, 4)[:, :, :3]
        ta = (vb if va is None else va).reshape(-1, 3, 4)[:, :, :3]
        rng = np.random.default_rng(0)
        for i in rng.choice(ta.shape[0], min(40, ta.shape[0]), replace=False):
            d2 = md.dist2(np.broadcast_to(ta[i], tb.shape), tb)
            if va is None:
                shared = (tb[:, :, None, :] == ta[i][None, None, :, :]).all(3).any((1, 2))
                d2[shared] = np.nan
            d2 = np.where(np.isnan(d2), np.inf, d2)
            assert np.isclose(float(d[i]) ** 2, float(d2.min()), rtol=1e-5, atol=1e-12), f"{label}: triangle {i}"
    return d, j


@pytest.mark.parametrize("ntris", [1, 7, 800])
def test_pruned_walk_equals_definition_on_every_builder(ntris):
    A = scenes.procedural_scene(ntris, 11 + ntris)
    B = scenes.procedural_scene(max(ntris, 2), 12 + ntris)
    B[:, :3] += np.float32(0.05)
    for label, nodes, idx in builder_trees(B):
        check_walk(nodes, idx, B, A, f"{label}-{ntris}", holds=label != "BuildHQ")
    for label, nodes, idx in builder_trees(A):
        check_walk(nodes, idx, A, None, f"self {label}-{ntris}", holds=label != "BuildHQ")


def test_failed_split_sbvh():
    from tests.test_build_hq_shapes import fail_scene, fail_scene_hq
    v = fail_scene("snapped3k_q4")
    nodes, idx = fail_scene_hq("snapped3k_q4")[:2]
    check_walk(nodes, idx, v, v[: 3 * 600], "snapped3k_q4", holds=False)
    check_walk(nodes, idx, v, None, "snapped3k_q4 self", holds=False)


@pytest.mark.parametrize("fam", util.FAMILIES + ["shrunk", "dag"])
def test_uploaded_families(fam):
    v = scenes.procedural_scene(1500, 71)
    a = scenes.procedural_scene(600, 72)
    src = util.source_tree(v, "BuildHQ" if fam in ("A1", "DB") else "Build")
    nodes, idx = family(src, fam)
    holds = fam not in ("shrunk", "dag", "A1", "DB")
    check_walk(nodes, idx, v, a, fam, holds=holds)
    check_walk(nodes, idx, v, None, f"self {fam}", holds=holds)


def test_self_rules():
    """corner-sharing pairs are never reported; two parallel sheets at distance h appear at r >= h and not below it"""
    V, F = icosphere(3)
    ball = soup(V, F)
    o = portpy.PortBVH(ball)
    p = md.pairs(o.nodes, o.prim_idx, ball, None, 0.5)[0]
    t = ball.reshape(-1, 3, 4)[:, :, :3]
    assert p.shape[0] > 100 and (p[:, 0] < p[:, 1]).all()
    assert not np.array([(t[i][:, None] == t[k][None]).all(2).any() for i, k in p]).any(), "a corner-sharing pair"
    d, j = md.nearest(o.nodes, o.prim_idx, ball)
    assert (j != md.NO_PRIM).all() and (d > 0).all()
    assert not np.array([(t[i][:, None] == t[k][None]).all(2).any() for i, k in enumerate(j)]).any()
    g = np.stack(np.meshgrid(np.arange(9), np.arange(9), indexing="ij"), -1).reshape(-1, 2)
    idx = np.arange(81).reshape(9, 9)
    Fg = np.r_[np.c_[idx[:-1, :-1].ravel(), idx[1:, :-1].ravel(), idx[1:, 1:].ravel()], np.c_[idx[:-1, :-1].ravel(), idx[1:, 1:].ravel(), idx[:-1, 1:].ravel()]]
    h = np.float32(0.125)
    lo, hi = soup(np.c_[g * 0.5, np.zeros(81)], Fg), soup(np.c_[g * 0.5, np.full(81, h)], Fg)
    sheets = np.concatenate([lo, hi])
    n = lo.shape[0] // 3
    o = portpy.PortBVH(sheets)
    assert md.pairs(o.nodes, o.prim_idx, sheets, None, float(np.nextafter(h, np.float32(0))))[0].shape[0] == 0
    at = md.pairs(o.nodes, o.prim_idx, sheets, None, float(h))[0]
    assert at.shape[0] >= n and ((at[:, 0] < n) & (at[:, 1] >= n)).all()
    d, j = md.nearest(o.nodes, o.prim_idx, sheets)
    assert (d == h).all() and ((j >= n) == (np.arange(2 * n) < n)).all()
