"""The host restatement of tbvh_mesh_toi / tbvh_mesh_toi_pairs (tests/toi_oracle.c, DESIGN.md §4.15): the time of impact of one pair
against an independent fp64 conservative advancement on random, sliver, nearly parallel and coplanar sliding pairs (the bracket
TOI(eta + xi) <= t <= TOI(eta)); analytic families (a vertex falling onto a face, edges crossing at right angles, a sheet tunnelling
through a plate within one step); static and rigid steps; symmetry, -0 twins, exact scaling by 2^k and the max_iters and no-progress
paths, bit for bit; and the pruned walk against the definition on every builder's tree, the uploaded families, a DAG and a failed-split
SBVH, two-mesh and self."""
import numpy as np
import pytest

from oracle import portpy
from tinybvh_b200 import scenes
from tests import meshdist_oracle as md, toi_oracle as toi, tritri_oracle as to, util
from tests.test_closest_point import builder_trees, family
from tests.test_mesh_distance import pair_cases
from tests.test_signed_distance import icosphere, soup

ETA, XI = 0.05, 0.01


def moving_pairs(seed=9, n=300):
    """{kind: (T0, T1, U0, U1)}: the static pair kinds of test_mesh_distance with U driven towards T (plus a little deformation of both),
    and coplanar pairs sliding within their plane"""
    rng = np.random.default_rng(seed)
    out = {}
    cases = pair_cases(seed, n)
    for kind in ("random_apart", "sliver", "near_parallel"):
        T0, U0 = (np.asarray(x, np.float64) for x in cases[kind])
        push = (T0.mean(1) - U0.mean(1))[:, None, :] * rng.uniform(0.5, 2.0, (n, 1, 1))
        if kind == "near_parallel":   # U lifted off T's edge, then lowered onto it, nearly parallel throughout
            U0 = U0 + [0, 0, 0.3]
            push = np.c_[np.zeros((n, 2)), -rng.uniform(0.1, 0.6, n)][:, None, :]
        T1 = T0 + rng.normal(size=(n, 1, 3)) * 0.2 + rng.normal(size=(n, 3, 3)) * 0.02
        U1 = U0 + push + rng.normal(size=(n, 3, 3)) * 0.02
        out[kind] = (T0, T1, U0, U1)
    T0, U0 = (np.asarray(x, np.float64) for x in cases["coplanar_disjoint"])
    slide = np.c_[rng.uniform(-1.5, -0.2, n), rng.uniform(-1.5, -0.2, n), np.zeros(n)][:, None, :]
    out["coplanar_sliding"] = (T0, T0, U0, U0 + slide)
    return {k: tuple(np.asarray(x, np.float32) for x in v) for k, v in out.items()}


def tol_of(*frames):
    return 2e-6 * (1.0 + max(float(np.abs(f).max()) for f in frames))


@pytest.mark.parametrize("kind", ["random_apart", "sliver", "near_parallel", "coplanar_sliding"])
def test_bracket_against_fp64(kind):
    T0, T1, U0, U1 = moving_pairs()[kind]
    for eta, xi, iters in ((ETA, XI, 64), (0.0, 1e-3, 64), (ETA, XI, 3)):
        hit, t, d, it = toi.pair(T0, T1, U0, U1, eta, xi, iters)
        tol = tol_of(T0, T1, U0, U1)
        hi = toi.toi64(T0, T1, U0, U1, max(eta - tol, 0.0))
        lo = toi.toi64(T0, T1, U0, U1, eta + xi + tol)
        # contact at t = 0 is the start frame's distance (§4.13, held to fp64 there; its overlap test misjudges some slivers)
        moved = t > 0
        res, unres = hit & (it < iters) & moved, hit & (it == iters) & moved
        assert hit.sum() > 20 and (~hit).sum() > 20 or kind == "coplanar_sliding", (kind, hit.sum())
        assert (t[res] >= lo[res] - 1e-9).all(), f"{kind}: a resolved contact before the first time at eta + xi"
        assert (t[hit & moved] <= hi[hit & moved] + 1e-9).all(), f"{kind}: a contact after the first time at eta"
        assert np.isinf(hi[~hit]).all(), f"{kind}: no contact reported where fp64 reaches eta"
        assert (d[res] <= np.float32(eta + xi) * (1 + 1e-6)).all(), f"{kind}: a resolved contact farther than eta + xi"
        if iters == 3:
            assert unres.sum() > 0 or kind == "coplanar_sliding"


def test_vertex_falling_onto_a_face():
    """a triangle whose lowest corner falls at speed v onto a face h below it: t within the bracket around (h - eta) / v"""
    rng = np.random.default_rng(4)
    n = 200
    face = np.array([[-4, -4, 0], [4, -4, 0], [0, 4, 0]], np.float32)
    h, v = rng.uniform(0.2, 2, n).astype(np.float32), rng.uniform(0.5, 4, n).astype(np.float32)
    p = np.c_[rng.uniform(-1, 1, (n, 2)), h].astype(np.float32)
    T0 = np.stack([p, p + [0.5, 0, 1], p + [0, 0.5, 1]], 1).astype(np.float32)
    T1 = T0 - np.c_[np.zeros((n, 2)), v][:, None, :].astype(np.float32)
    U = np.broadcast_to(face, (n, 3, 3))
    hit, t, d, it = toi.pair(T0, T1, U, U, ETA, XI, 64)
    exact = (h.astype(np.float64) - ETA) / v
    reach = exact <= 1
    assert reach.sum() > 50 and (~reach).sum() > 20
    assert (hit == ((h - ETA - XI) / v <= 1 + 1e-6) | hit).all()
    assert not hit[(h.astype(np.float64) - ETA) / v > 1 + 1e-5].any()
    r = hit & (it < 64)
    lo = (h.astype(np.float64) - ETA - XI) / v
    assert (t[r] >= lo[r] - 1e-6).all() and (t[r] <= exact[r] + 1e-6).all()


def test_edges_crossing_at_right_angles():
    """two thin triangles whose long edges cross at right angles, closing at speed 1 from height h: contact at (h - eta) / 1"""
    n = 64
    h = np.linspace(0.1, 1.5, n).astype(np.float32)
    T = np.broadcast_to(np.array([[-2, 0, 0], [2, 0, 0], [0, 0, -1]], np.float32), (n, 3, 3))
    U0 = np.stack([np.c_[np.zeros(n), -2 * np.ones(n), h], np.c_[np.zeros(n), 2 * np.ones(n), h], np.c_[np.zeros(n), np.zeros(n), h + 1]], 1).astype(np.float32)
    U1 = U0 - np.array([0, 0, 1], np.float32)
    hit, t, d, it = toi.pair(T, T, U0, U1, ETA, XI, 64)
    exact = (h.astype(np.float64) - ETA) / 1.0
    assert (hit == (h - ETA - XI <= 1)).all() or (hit[exact <= 1]).all()
    r = hit & (it < 64)
    assert r.sum() > 30
    assert (t[r] >= exact[r] - XI - 1e-6).all() and (t[r] <= exact[r] + 1e-6).all()
    assert (np.abs(d[r] - (h[r] - t[r])) <= 1e-5).all(), "the distance at t is the gap of the two edges"


def plate_and_sheet():
    """a plate at z = 0 and a thin sheet above it at z = 1 that ends the step at z = -1: it passes through the plate within the step"""
    g = np.stack(np.meshgrid(np.arange(5), np.arange(5), indexing="ij"), -1).reshape(-1, 2).astype(np.float32)
    idx = np.arange(25).reshape(5, 5)
    F = np.r_[np.c_[idx[:-1, :-1].ravel(), idx[1:, :-1].ravel(), idx[1:, 1:].ravel()], np.c_[idx[:-1, :-1].ravel(), idx[1:, 1:].ravel(), idx[:-1, 1:].ravel()]]
    plate = soup(np.c_[g, np.zeros(25)], F)
    sheet0 = soup(np.c_[g * 0.5 + 0.6, np.ones(25)], F)
    sheet1 = soup(np.c_[g * 0.5 + 0.6, -np.ones(25)], F)
    return plate, sheet0, sheet1


def test_tunnelling_sheet_is_found():
    plate, s0, s1 = plate_and_sheet()
    o = portpy.PortBVH(plate)
    for s in (s0, s1):
        assert to.all_pairs(s, plate)[0].shape[0] == 0, "the discrete check at either end finds nothing"
    p, times = toi.pairs(o.nodes, o.prim_idx, plate, plate, s0, s1, eta=0.0, xi=1e-3)
    assert p.shape[0] > 10
    assert (np.abs(times - 0.5) <= 1e-3).all(), times
    t, d, j, it = toi.nearest(o.nodes, o.prim_idx, plate, plate, s0, s1, eta=0.0, xi=1e-3)
    assert (j != toi.NO_PRIM).sum() > 0 and (np.abs(t[j != toi.NO_PRIM] - 0.5) <= 1e-3).all()


def test_static_step_is_distance_pairs_at_time_zero():
    """end == start: t = 0 exactly on the distance pairs at eta + xi and no contact elsewhere (L = 0), on every builder's tree: a
    reference is reached in both queries by the same bound, swept boxes being the triangles' own boxes, and the pair test at t = 0 is
    tt_dist2 on the input corners (x(0) is x0 up to the sign of zero, which tt_dist2 ignores); the one rounding difference, distance
    pairs comparing r^2 = fl( fl( eta + xi )^2 ) against max( tt_dist2, LBtri, P ) where this query compares tt_dist2 alone, changes
    nothing where boxes hold their triangles, as every builder's do"""
    A = scenes.procedural_scene(700, 31)
    B = scenes.procedural_scene(700, 32)
    B[:, :3] += np.float32(0.05)
    r = np.float32(ETA) + np.float32(XI)
    for label, nodes, idx in builder_trees(B):
        want = md.pairs(nodes, idx, B, A, float(r))[0]
        p, times = toi.pairs(nodes, idx, B, B, A, A, ETA, XI)
        assert want.shape[0] > 10 and np.array_equal(p, want), label
        assert (times == 0).all()
        t, d, j, it = toi.nearest(nodes, idx, B, B, A, A, ETA, XI)
        has = np.zeros(A.shape[0] // 3, bool)
        has[want[:, 0]] = True
        assert ((t == 0) == has).all() and np.isinf(t[~has]).all() and (it == 0).all(), label
        assert np.array_equal(j[has], np.array([want[want[:, 0] == i, 1].min() for i in np.nonzero(has)[0]])), label


def test_rigid_translation_gives_zero_or_inf():
    """a common translation moves every corner by the same exact amount (dyadic coordinates): L = 0, so t is 0 or inf"""
    A = np.round(scenes.procedural_scene(600, 41) * 64) / 64
    B = np.round(scenes.procedural_scene(600, 42) * 64) / 64
    A[900:, 0] += 64   # the second half of A far from B
    shift = np.array([0.25, -0.5, 0.125, 0], np.float32)
    o = portpy.PortBVH(B)
    t, d, j, it = toi.nearest(o.nodes, o.prim_idx, B, B + shift, A, A + shift, ETA, XI)
    assert ((t == 0) | np.isinf(t)).all() and (t == 0).sum() > 10 and np.isinf(t).sum() > 10
    t2 = toi.nearest(o.nodes, o.prim_idx, B, B, A, A, ETA, XI)[0]
    assert np.array_equal(t, t2), "a rigid step finds the contacts of the start frame"


def test_pair_properties_bit_for_bit():
    """symmetry under swapping the triangles, -0 twins, scaling by 2^k for k in [-40, 40], the max_iters and no-progress paths"""
    cases = moving_pairs(n=200)
    for kind, (T0, T1, U0, U1) in cases.items():
        a = toi.pair(T0, T1, U0, U1, ETA, XI)
        b = toi.pair(U0, U1, T0, T1, ETA, XI)
        for x, y in zip(a, b):
            assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8)), f"{kind}: not symmetric"
        z = [x.copy() for x in (T0, T1, U0, U1)]
        for x in z:
            x[np.abs(x) < 0.3] = 0.0
        neg = [np.where(x == 0, np.float32(-0.0), x).astype(np.float32) for x in z]
        p, q = toi.pair(*z, ETA, XI), toi.pair(*neg, ETA, XI)
        for x, y in zip(p, q):
            assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8)), f"{kind}: -0 twin differs"
        for k in (-40, -17, 3, 40):
            s = [np.ldexp(x, k).astype(np.float32) for x in (T0, T1, U0, U1)]
            e, x_ = float(np.ldexp(np.float32(ETA), k)), float(np.ldexp(np.float32(XI), k))
            h, t, d, it = toi.pair(*s, e, x_)
            assert np.array_equal(h, a[0]) and np.array_equal(t.view(np.uint32), a[1].view(np.uint32)) and np.array_equal(it, a[3]), (kind, k)
            assert np.array_equal(np.ldexp(d, -k).view(np.uint32), a[2].view(np.uint32)), (kind, k)
    # max_iters: every iteration count up to the cap, and the cap reported as unresolved at an earlier t
    T0, T1, U0, U1 = cases["near_parallel"]
    full = toi.pair(T0, T1, U0, U1, 0.0, 1e-6, 1 << 16)
    assert full[3][full[0]].max() > 4
    for m in (1, 2, 4):
        h, t, d, it = toi.pair(T0, T1, U0, U1, 0.0, 1e-6, m)
        same = (h == full[0]) & (t.view(np.uint32) == full[1].view(np.uint32)) & (it == full[3])
        cut = h & (it == m) & (t <= full[1])
        assert (same | cut).all() and (cut & ~same).sum() > 0, m
        assert same[full[0] & (full[3] < m)].all()
    # no progress: a step below half an ulp of t leaves t where it is -> unresolved at that t
    f = np.float32
    T = np.array([[[0, 0, 0], [1, 0, 0], [0, 1, 0]]], f)
    U0 = np.array([[[0, 0, 1], [1, 0, 1], [0, 1, 1]]], f) * f(1)
    U1 = U0.copy()
    U1[:, :, 2] = f(1) - f(2.0 ** -30)
    U0b = U0.copy()
    U0b[:, :, 2] = f(0.75) + f(2.0 ** -23)
    U1b = U0b - np.array([0, 0, 2.0 ** -4], f)
    h, t, d, it = toi.pair(T, T, U0b, U1b, 0.5, 0.25, 64)
    assert not h[0], "moving too slowly to reach the margin within the step"
    h, t, d, it = toi.pair(T, T, U0, U0 - np.array([0, 0, 1.5], f), 0.0, 2.0 ** -24, 1 << 16)
    assert h[0] and abs(float(t[0]) - 2 / 3) < 1e-5


def check_walk(nodes, idx, B0, B1, A0, A1, label):
    """the pruned walk with abandonment == the definition: nearest records bit for bit, and the pairs"""
    for eta, xi in ((ETA, XI), (0.0, 1e-3)):
        w = toi.nearest(nodes, idx, B0, B1, A0, A1, eta, xi)
        b = toi.nearest(nodes, idx, B0, B1, A0, A1, eta, xi, brute=True)
        for x, y in zip(w, b):
            assert np.array_equal(x.view(np.uint32), y.view(np.uint32)), f"{label}: nearest walk differs from the definition"
        p, tp = toi.pairs(nodes, idx, B0, B1, A0, A1, eta, xi)
        bp, _ = toi.pairs(nodes, idx, B0, B1, A0, A1, eta, xi, brute=True)
        assert np.array_equal(p, bp), f"{label}: pairs differ from the definition"
        hit = w[2] != toi.NO_PRIM
        assert np.array_equal(np.unique(p[:, 0]), np.nonzero(hit)[0]) or A0 is None, f"{label}: a nearest record without a pair"
    return w, p


def jitter(v, seed, s=0.02):
    rng = np.random.default_rng(seed)
    out = v.copy()
    out[:, :3] += (rng.normal(size=(v.shape[0], 3)) * s).astype(np.float32)
    return out


@pytest.mark.parametrize("ntris", [1, 7, 600])
def test_pruned_walk_equals_definition_on_every_builder(ntris):
    A = scenes.procedural_scene(ntris, 11 + ntris)
    B = scenes.procedural_scene(max(ntris, 2), 12 + ntris)
    B[:, :3] += np.float32(0.05)
    B1, A1 = jitter(B, 1), jitter(A, 2)
    for label, nodes, idx in builder_trees(B):
        check_walk(nodes, idx, B, B1, A, A1, f"{label}-{ntris}")
    for label, nodes, idx in builder_trees(A):
        w, p = check_walk(nodes, idx, A, A1, None, None, f"self {label}-{ntris}")
        assert (p[:, 0] < p[:, 1]).all()


def test_failed_split_sbvh():
    from tests.test_build_hq_shapes import fail_scene, fail_scene_hq
    v = fail_scene("snapped3k_q4")
    nodes, idx = fail_scene_hq("snapped3k_q4")[:2]
    check_walk(nodes, idx, v, jitter(v, 3, 0.05), v[: 3 * 600], jitter(v[: 3 * 600], 4, 0.05), "snapped3k_q4")
    check_walk(nodes, idx, v, jitter(v, 3, 0.05), None, None, "snapped3k_q4 self")


@pytest.mark.parametrize("fam", util.FAMILIES + ["shrunk", "dag"])
def test_uploaded_families(fam):
    v = scenes.procedural_scene(1500, 71)
    a = scenes.procedural_scene(600, 72)
    src = util.source_tree(v, "BuildHQ" if fam in ("A1", "DB") else "Build")
    nodes, idx = family(src, fam)
    check_walk(nodes, idx, v, jitter(v, 5), a, jitter(a, 6), fam)
    check_walk(nodes, idx, v, jitter(v, 5), None, None, f"self {fam}")


def test_self_rules():
    """corner-sharing pairs (equal in both frames) are never reported; a ball squashed flat within the step finds its far sides"""
    V, F = icosphere(3)
    ball = soup(V, F)
    flat = ball.copy()
    flat[:, 2] *= np.float32(0.01)
    o = portpy.PortBVH(ball)
    p, times = toi.pairs(o.nodes, o.prim_idx, ball, flat, eta=0.0, xi=0.02)
    t = ball.reshape(-1, 3, 4)[:, :, :3]
    assert p.shape[0] > 100 and (p[:, 0] < p[:, 1]).all() and (times > 0).all() and (times <= 1).all()
    assert not np.array([(t[i][:, None] == t[k][None]).all(2).any() for i, k in p]).any(), "a corner-sharing pair"
    tt, d, j, it = toi.nearest(o.nodes, o.prim_idx, ball, flat, eta=0.0, xi=0.02)
    assert (j != toi.NO_PRIM).sum() > 100 and (j != np.arange(j.shape[0])).all()
