"""The host restatement of tbvh_mesh_overlap_pairs / tbvh_mesh_overlap_bits (tests/tritri_oracle.c, DESIGN.md §4.12): the fp32 pair test
against exact arithmetic on integer lattices (the same predicates in Python ints, and an independent separating-axis test), seeded float
pairs against exact rationals, symmetry, scaling by 2^k for every k in [-40, 40], the pruned walk against the definition and against all
pairs on every builder's tree and the uploaded families, and self-intersection scenes."""
from fractions import Fraction

import numpy as np
import pytest

from oracle import portpy
from tinybvh_b200 import scenes
from tests import tritri_oracle as to, util
from tests.test_closest_point import builder_trees, family
from tests.test_signed_distance import icosphere, soup
from tests.test_winding_number import two_spheres


def rand_tri(rng, lo=-16, hi=16, n=1):
    return rng.integers(lo, hi + 1, (n, 3, 3)).astype(np.float32)


def lattice_families(seed=3):
    """{family: (T, U, self, expected or None)} of integer-cornered pairs in [-16, 16]; expected: the geometric truth where the
    construction fixes it"""
    rng = np.random.default_rng(seed)
    out = {}
    n = 3000
    T, U = rand_tri(rng, n=n), rand_tri(rng, n=n)
    out["general"] = (T, U, False, None)
    # small triangles near each other: many touching and crossing cases
    c = rng.integers(-12, 13, (n, 1, 3))
    out["near"] = ((c + rng.integers(-2, 3, (n, 3, 3))).astype(np.float32), (c + rng.integers(-2, 3, (n, 3, 3))).astype(np.float32), False, None)
    # a corner of U on the face of T (T in z = 0 with integer interior points), the rest of U above
    T = np.tile(np.array([[-8, -8, 0], [8, -8, 0], [-8, 8, 0]], np.float32), (n, 1, 1))
    p = np.c_[rng.integers(-7, 1, (n, 1)), rng.integers(-7, 1, (n, 1)), np.zeros((n, 1))]
    U = np.stack([p, p + np.c_[rng.integers(-3, 4, (n, 2)), rng.integers(1, 5, (n, 1))], p + np.c_[rng.integers(-3, 4, (n, 2)), rng.integers(1, 5, (n, 1))]], 1)
    out["vertex_on_face"] = (T, U.astype(np.float32), False, None)
    # edge on edge: U's edge crosses T's edge x = 0 at an integer point, U leaning away
    T = np.tile(np.array([[0, -8, -8], [0, 8, -8], [0, 0, 8]], np.float32), (n, 1, 1))
    y = rng.integers(-7, 8, n)
    U = np.stack([np.c_[-np.ones(n), y, np.full(n, -8)], np.c_[np.ones(n), y, np.full(n, -8)], np.c_[np.zeros(n), y + 3, np.full(n, -12)]], 1)
    out["edge_on_edge"] = (T, U.astype(np.float32), False, np.ones(n, bool))
    # an edge of U through the face of T
    T = np.tile(np.array([[-10, -10, 0], [10, -10, 0], [-10, 10, 0]], np.float32), (n, 1, 1))
    q = rng.integers(-8, 0, (n, 2))
    U = np.stack([np.c_[q, -np.ones(n) * 3], np.c_[q, np.ones(n) * 3], np.c_[q + rng.integers(1, 5, (n, 2)), rng.integers(-3, 4, n)]], 1)
    out["edge_through_face"] = (T, U.astype(np.float32), False, np.ones(n, bool))
    # coplanar on z = const: overlapping, contained and touching (a corner on an edge, shared edges, disjoint)
    z = rng.integers(-16, 17, (n, 1, 1)).astype(np.float32)
    T2, U2 = rng.integers(-6, 7, (n, 3, 2)), rng.integers(-6, 7, (n, 3, 2))
    out["coplanar"] = (np.concatenate([T2, np.broadcast_to(z, (n, 3, 1))], 2).astype(np.float32),
                       np.concatenate([U2, np.broadcast_to(z, (n, 3, 1))], 2).astype(np.float32), False, None)
    big = np.array([[-9, -9], [9, -9], [-9, 9]])
    inner = rng.integers(-8, 0, (n, 1, 2)) + np.array([[0, 0], [1, 0], [0, 1]])
    out["coplanar_contained"] = (np.concatenate([np.broadcast_to(big, (n, 3, 2)), np.broadcast_to(z, (n, 3, 1))], 2).astype(np.float32),
                                 np.concatenate([inner, np.broadcast_to(z, (n, 3, 1))], 2).astype(np.float32), False, np.ones(n, bool))
    touch = np.stack([np.c_[np.zeros(n), rng.integers(-8, 1, n)], np.c_[-rng.integers(1, 5, n), rng.integers(-4, 4, n)], np.c_[-rng.integers(1, 5, n), rng.integers(4, 9, n)]], 1)
    edge = np.array([[0, -8], [0, 8], [6, 0]])
    out["coplanar_touching"] = (np.concatenate([np.broadcast_to(edge, (n, 3, 2)), np.broadcast_to(z, (n, 3, 1))], 2).astype(np.float32),
                                np.concatenate([touch, np.broadcast_to(z, (n, 3, 1))], 2).astype(np.float32), False, np.ones(n, bool))
    # self mode: shared corner, shared edge folded both ways, duplicate faces
    a, b, c2 = (rng.integers(-8, 9, (n, 3)) for _ in range(3))
    d, e = rng.integers(-8, 9, (n, 3)), rng.integers(-8, 9, (n, 3))
    out["self_shared_corner"] = (np.stack([a, b, c2], 1).astype(np.float32), np.stack([d, a, e], 1).astype(np.float32), True, None)
    out["self_shared_edge"] = (np.stack([a, b, c2], 1).astype(np.float32), np.stack([b, a, d], 1).astype(np.float32), True, None)
    # coplanar folds across a shared edge on z = const: third corners on the same side (a fold, reported) or on opposite sides (not)
    s = np.c_[rng.integers(1, 8, n), rng.integers(-6, 7, n)]
    e0, e1 = np.array([0, -8]), np.array([0, 8])
    tri_a = np.stack([np.broadcast_to(e0, (n, 2)), np.broadcast_to(e1, (n, 2)), s], 1)
    same = np.stack([np.broadcast_to(e1, (n, 2)), np.broadcast_to(e0, (n, 2)), s + [rng.integers(0, 3), 1]], 1)
    flip = np.stack([np.broadcast_to(e1, (n, 2)), np.broadcast_to(e0, (n, 2)), -s], 1)
    zz = np.broadcast_to(z, (n, 3, 1))
    out["self_fold_same_side"] = (np.concatenate([tri_a, zz], 2).astype(np.float32), np.concatenate([same, zz], 2).astype(np.float32), True, np.ones(n, bool))
    out["self_fold_opposite"] = (np.concatenate([tri_a, zz], 2).astype(np.float32), np.concatenate([flip, zz], 2).astype(np.float32), True, np.zeros(n, bool))
    perm = rng.permutation(3)
    out["self_duplicate"] = (np.stack([a, b, c2], 1).astype(np.float32), np.stack([a, b, c2], 1)[:, perm].astype(np.float32), True, None)
    return out


def degenerate(T):
    return ~np.cross(T[:, 1] - T[:, 0], T[:, 2] - T[:, 0]).astype(np.float64).any(1)


@pytest.mark.parametrize("fam", list(lattice_families().keys()))
def test_lattice_pairs_equal_exact_arithmetic(fam):
    T, U, self, expected = lattice_families()[fam]
    got = to.tt(T, U, self)
    exact = np.array([to.exact_tt(t, u, self) for t, u in zip(T, U)])
    assert np.array_equal(got, exact), f"{fam}: {int((got != exact).sum())} of {T.shape[0]} differ from exact arithmetic"
    ok = ~(degenerate(T) | degenerate(U))
    if expected is not None:
        assert np.array_equal(got[ok], expected[ok]), fam
    if not self:
        sat = np.array([to.sat_tt(t.astype(int).tolist(), u.astype(int).tolist()) if k else False for t, u, k in zip(T, U, ok)])
        assert np.array_equal(got, sat), f"{fam}: {int((got != sat).sum())} differ from the separating-axis test"
    else:
        dup = (T[:, None, :, :] == U[:, :, None, :]).all(3).any(1).sum(1) == 3
        assert got[dup & ok].all(), "a duplicate face is always reported"
        assert not got[~ok].any(), "a degenerate triangle is never reported"
    print(f"{fam}: {int(got.sum())} of {T.shape[0]} pairs overlap")


def test_self_rules_on_one_shared_corner():
    """sharing one corner: reported exactly when the triangles meet elsewhere - checked against the separating-axis test on the
    triangles with the shared corner pulled a tenth of the way towards each triangle's centroid (meeting elsewhere survives a small pull
    for these lattice pairs, touching only at the corner does not)"""
    T, U, _, _ = lattice_families()["self_shared_corner"]
    ok = ~(degenerate(T) | degenerate(U))
    got = to.tt(T, U, True)
    agree = 0
    for k in np.nonzero(ok)[0][:1500]:
        t, u = [Fraction(int(x)) for x in T[k].reshape(-1)], [Fraction(int(x)) for x in U[k].reshape(-1)]
        t, u = np.array(t, object).reshape(3, 3), np.array(u, object).reshape(3, 3)
        # the shared corner is T[0] == U[1]
        tc, uc = t.sum(0) / 3, u.sum(0) / 3
        t2, u2 = t.copy(), u.copy()
        t2[0] = t[0] + (tc - t[0]) * Fraction(1, 1000)
        u2[1] = u[1] + (uc - u[1]) * Fraction(1, 1000)
        meet = to.sat_tt(t2.tolist(), u2.tolist())
        agree += meet == got[k]
    assert agree >= 0.99 * min(1500, int(ok.sum())), agree


def float_pairs(seed, n=3000):
    rng = np.random.default_rng(seed)
    c = rng.normal(size=(n, 1, 3))
    T = (c + rng.normal(size=(n, 3, 3)) * 0.5).astype(np.float32)
    U = (c + rng.normal(size=(n, 3, 3)) * 0.5).astype(np.float32)
    return T, U


def test_seeded_float_pairs_against_exact_rationals():
    T, U = float_pairs(7)
    got = to.tt(T, U)
    checked = bad = 0
    for k in range(T.shape[0]):
        tr = to._Track()
        e = to.exact_tt(T[k], U[k], num=Fraction, track=tr)
        L = Fraction(float(np.abs(np.r_[T[k], U[k]] - T[k][0]).max()))
        conditioned = (tr.m3 is None or tr.m3 >= Fraction(1, 1000) * L ** 3) and (tr.m2 is None or tr.m2 >= Fraction(1, 1000) * L ** 2)
        if conditioned:
            checked += 1
            bad += e != got[k]
    assert bad == 0 and checked > 0.8 * T.shape[0], (checked, bad)
    # near-touching pairs: U's corner jittered onto T's face; disagreements are counted, with no claim
    rng = np.random.default_rng(8)
    w = rng.dirichlet((1, 1, 1), T.shape[0])
    U2 = U.copy()
    U2[:, 0] = (w[:, :, None] * T.astype(np.float64)).sum(1).astype(np.float32) + rng.normal(size=(T.shape[0], 3)).astype(np.float32) * 1e-7
    got2 = to.tt(T, U2)
    dis = sum(to.exact_tt(T[k], U2[k], num=Fraction) != got2[k] for k in range(T.shape[0]))
    print(f"conditioned pairs: {checked} of {T.shape[0]}, all agree; near-touching pairs: {dis} of {T.shape[0]} disagree with exact rationals")


def lattice_soup(n, seed, lo=-8, hi=8, size=3, offset=0.0):
    rng = np.random.default_rng(seed)
    c = rng.integers(lo, hi + 1, (n, 1, 3))
    t = (c + rng.integers(-size, size + 1, (n, 3, 3))).astype(np.float32) + np.float32(offset)
    v = np.zeros((3 * n, 4), np.float32)
    v[:, :3] = t.reshape(-1, 3)
    return v


def swapped_pairs(p):
    return p[np.lexsort((p[:, 0], p[:, 1]))][:, ::-1]


def test_symmetry():
    for fam, (T, U, self, _) in lattice_families().items():
        assert np.array_equal(to.tt(T, U, self), to.tt(U, T, self)), fam
    T, U = float_pairs(9)
    assert np.array_equal(to.tt(T, U), to.tt(U, T))
    A, B = lattice_soup(700, 1), lattice_soup(600, 2)
    ab, abits = to.all_pairs(A, B)
    ba, _ = to.all_pairs(B, A)
    assert ab.shape[0] > 100
    assert np.array_equal(ab, swapped_pairs(ba))
    nA, iA = portpy.PortBVH(A).nodes, None
    oa, ob = portpy.PortBVH(A), portpy.PortBVH(B)
    wab = to.tree(ob.nodes, ob.prim_idx, B, A)[0]
    wba = to.tree(oa.nodes, oa.prim_idx, A, B)[0]
    assert np.array_equal(wab, ab) and np.array_equal(wba, ba)
    del nA, iA


def test_scale_gives_the_same_pairs_for_every_k():
    A, B = lattice_soup(300, 4), lattice_soup(300, 5)
    S = np.concatenate([A, lattice_soup(200, 6, offset=0.5)])
    ref_ab, ref_bits = to.all_pairs(A, B)
    ref_s, ref_sbits = to.all_pairs(S)
    assert ref_ab.shape[0] > 50 and ref_s.shape[0] > 50
    for k in range(-40, 41):
        ab, bits = to.all_pairs(util.scaled(A, k), util.scaled(B, k))
        assert np.array_equal(ab, ref_ab) and np.array_equal(bits, ref_bits), k
        s, sbits = to.all_pairs(util.scaled(S, k))
        assert np.array_equal(s, ref_s) and np.array_equal(sbits, ref_sbits), k
        if k % 20 == 0:
            o = portpy.PortBVH(util.scaled(B, k))
            assert np.array_equal(to.tree(o.nodes, o.prim_idx, util.scaled(B, k), util.scaled(A, k))[0], ref_ab), k


def check_walk(nodes, idx, vb, va, label, holds=True):
    """pruned walk == definition (pairs and bits); with boxes that hold their triangles, == all pairs; returns the walk's pairs"""
    w, wbits, wkeys, _ = to.tree(nodes, idx, vb, va)
    b, bbits, _, _ = to.tree(nodes, idx, vb, va, brute=True)
    assert np.array_equal(w, b), f"{label}: pruned walk differs from the definition"
    assert np.array_equal(wbits, bbits), f"{label}: bits"
    assert wkeys.shape[0] >= w.shape[0]
    if holds:
        ap, apbits = to.all_pairs(vb if va is None else va, None if va is None else vb)
        assert np.array_equal(w, ap), f"{label}: the reached set is not all pairs"
        assert np.array_equal(wbits, apbits), f"{label}: bits against all pairs"
        n = (vb if va is None else va).shape[0] // 3
        assert np.array_equal(wbits, to.member_bits(w, n, va is None)), f"{label}: bits are not 'appears in pairs'"
    return w, wkeys


@pytest.mark.parametrize("ntris", [1, 7, 2000])
def test_pruned_walk_equals_all_pairs_on_every_builder(ntris):
    A = scenes.procedural_scene(ntris, 11 + ntris)
    B = scenes.procedural_scene(max(ntris, 2), 12 + ntris)
    B[:, :3] += np.float32(0.05)
    for label, nodes, idx in builder_trees(B):
        check_walk(nodes, idx, B, A, f"{label}-{ntris}")
    for label, nodes, idx in builder_trees(A):
        check_walk(nodes, idx, A, None, f"self {label}-{ntris}")


def test_failed_split_sbvh_and_duplicates():
    """an SBVH whose spatial splits fail, and BuildHQ trees that reference a triangle from several leaves: the repeats are removed"""
    from tests.test_build_hq_shapes import fail_scene, fail_scene_hq
    v = fail_scene("snapped3k_q4")
    nodes, idx = fail_scene_hq("snapped3k_q4")[:2]
    w, keys = check_walk(nodes, idx, v, None, "snapped3k_q4 self", holds=False)
    b = scenes.procedural_scene(3000, 5)
    hn, hi, _ = portpy.build_hq(b)
    w, keys = check_walk(hn, hi, b, v, "BuildHQ")
    print(f"BuildHQ: {keys.shape[0]} raw keys, {w.shape[0]} pairs")


@pytest.mark.parametrize("fam", util.FAMILIES + ["shrunk", "dag"])
def test_uploaded_families(fam):
    v = scenes.procedural_scene(3000, 71)
    a = scenes.procedural_scene(1500, 72)
    src = util.source_tree(v, "BuildHQ" if fam in ("A1", "DB") else "Build")
    nodes, idx = family(src, fam)
    # shrunk boxes and the DAG's lost subtree need not reach every pair: the definition only
    holds = fam not in ("shrunk", "dag")
    check_walk(nodes, idx, v, a, fam, holds=holds)
    check_walk(nodes, idx, v, None, f"self {fam}", holds=holds)


def exact_self_pairs(v):
    """every pair i < j of a soup by exact_tt in Fractions (for small meshes)"""
    t = v.reshape(-1, 3, 4)[:, :, :3]
    out = []
    for i in range(t.shape[0]):
        lo, hi = t[i].min(0), t[i].max(0)
        for j in range(i + 1, t.shape[0]):
            if (t[j].max(0) < lo).any() or (t[j].min(0) > hi).any():
                continue
            if to.exact_tt(t[i], t[j], True, num=Fraction):
                out.append((i, j))
    return np.array(out, np.uint32).reshape(-1, 2)


def fan_fold():
    """a flat fan around the origin, and one triangle that shares a corner with its neighbour but is folded down through it"""
    a = np.linspace(0, 2 * np.pi, 9)[:-1]
    rim = np.c_[np.cos(a), np.sin(a), np.zeros(8)]
    V = np.r_[[[0, 0, 0]], rim]
    F = [(0, 1 + k, 1 + (k + 1) % 8) for k in range(8)]
    v = soup(V, F)
    # a triangle sharing rim corner 1 with the fan, dipping through triangle 0
    extra = np.array([[rim[0], [0.2, 0.3, -0.5], [0.3, 0.2, 0.5]]], np.float32)
    e = np.zeros((3, 4), np.float32)
    e[:, :3] = extra.reshape(-1, 3)
    return np.r_[v, e]


def test_self_intersection_scenes():
    V, F = icosphere(3)
    ball = soup(V, F)
    o = portpy.PortBVH(ball)
    assert to.tree(o.nodes, o.prim_idx, ball)[0].shape[0] == 0, "a closed icosphere has no self-intersections"
    two = soup(*two_spheres())
    o = portpy.PortBVH(two)
    got = to.tree(o.nodes, o.prim_idx, two)[0]
    want = exact_self_pairs(two)
    assert want.shape[0] > 20 and np.array_equal(got, want), (got.shape, want.shape)
    fan = fan_fold()
    o = portpy.PortBVH(fan)
    got = to.tree(o.nodes, o.prim_idx, fan)[0]
    assert (8 in got[:, 1]) and np.array_equal(got, exact_self_pairs(fan)), got
    # a coplanar fold across a shared edge: triangle 1 folded flat onto triangle 0
    fold = np.zeros((6, 4), np.float32)
    fold[:, :3] = [[0, 0, 0], [4, 0, 0], [0, 4, 0], [4, 0, 0], [0, 0, 0], [1, 1, 0]]
    o = portpy.PortBVH(fold)
    assert np.array_equal(to.tree(o.nodes, o.prim_idx, fold)[0], [[0, 1]])
    unfolded = fold.copy()
    unfolded[5, :3] = [1, -1, 0]
    assert to.tree(portpy.PortBVH(unfolded).nodes, portpy.PortBVH(unfolded).prim_idx, unfolded)[0].shape[0] == 0
    # a flat grid: neighbours share edges and corners, nothing crosses
    g = np.stack(np.meshgrid(np.arange(33), np.arange(33), indexing="ij"), -1).reshape(-1, 2)
    Vg = np.c_[g, np.zeros(g.shape[0])] * 0.25
    idx = np.arange(33 * 33).reshape(33, 33)
    Fg = np.r_[np.c_[idx[:-1, :-1].ravel(), idx[1:, :-1].ravel(), idx[1:, 1:].ravel()], np.c_[idx[:-1, :-1].ravel(), idx[1:, 1:].ravel(), idx[:-1, 1:].ravel()]]
    grid = soup(Vg, Fg)
    o = portpy.PortBVH(grid)
    assert to.tree(o.nodes, o.prim_idx, grid)[0].shape[0] == 0, "a flat grid has no self-intersections"
    assert not to.tree(o.nodes, o.prim_idx, grid)[1].any()
